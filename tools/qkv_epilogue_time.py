"""GPU microbenchmark: the fused QKV GEMM of one DiT block alone, with EPI_QKV_ROPE and with EPI_QKV_NORM_ROPE
(qk_norm="rms_norm"), at the F5TTS Base shape (K = 1024, N = 3 x 1024) and M = 1876 (cfg2: 938 frames, CFG-packed).

    python tools/qkv_epilogue_time.py            # QKV_M=<rows>, QKV_ROUNDS=<n> override the defaults

Each epilogue's launches are captured into a CUDA graph (so host-side planning is not timed); every round replays
each graph with CUDA events around it, alternating the variants, at the planner's tile width (bn = 0) and at every
instantiated width.  Prints the card name and power limit of the run."""
import os
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from f5_tts_b200 import ops  # noqa: E402

dev = "cuda:0"
M, D, inner = int(os.environ.get("QKV_M", "1876")), 1024, 1024
rounds, iters = int(os.environ.get("QKV_ROUNDS", "7")), 100
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = torch.cuda.get_device_name(0)
print(f"device: {card}")

g = torch.Generator().manual_seed(0)
a = torch.randn(M, D, generator=g).half().to(dev)
w = (torch.randn(3 * inner, D, generator=g) / 32).half().to(dev)
bias = (0.05 * torch.randn(3 * inner, generator=g)).to(dev)
qg, kg = (1 + 0.1 * torch.randn(64, generator=g)).to(dev), (1 + 0.1 * torch.randn(64, generator=g)).to(dev)
seq = M // 2
cs, sn = ops.rope_tables(seq, dev)
base = dict(seq=seq, rope=(cs, sn), inner=inner, pe_heads=16, static_w=True)
variants = {}
for bn in (0, 128, 192, 256):
    variants[f"rope bn{bn}"] = dict(epi=ops.EPI_QKV_ROPE, bn=bn)
    variants[f"norm_rope bn{bn}"] = dict(epi=ops.EPI_QKV_NORM_ROPE, bn=bn, qk_norm=(qg, kg))
print("planner width:", {e: ops.gemm_tile(M, 3 * inner, D, epi=e)[0] for e in (ops.EPI_QKV_ROPE, ops.EPI_QKV_NORM_ROPE)})


graphs = {}
for k, kw in variants.items():
    ops.linear(a, w, bias, **base, **kw)  # warm-up outside the capture
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        for _ in range(iters):
            ops.linear(a, w, bias, **base, **kw)
    graphs[k] = gr


def time_us(gr):
    gr.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    gr.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


res = {k: [] for k in variants}
for r in range(rounds):
    for k in variants:
        res[k].append(time_us(graphs[k]))
flop = 2.0 * M * D * 3 * inner
for k, v in res.items():
    v = sorted(v)
    med = v[len(v) // 2]
    print(f"M={M} {k:16s} median {med:7.2f} us  min {v[0]:7.2f}  max {v[-1]:7.2f}  ({flop / med * 1e-6:.0f} TFLOP/s)")
