"""GPU timing: 128-wide attention heads against 64-wide ones at the same attention width (inner 1024).

1. The attention kernel alone at the cfg2 shape (CFG-packed batch Be = 2, N = 938): 16 heads of 64 against 8 heads of
   128, CUDA-graph timed (ATTN_REPS launches per replay), alternating for ATTN_ROUNDS rounds.
2. One cfg2 sampler call (tools/step_time.py's measurement, vocoder included) of F5TTS_v1_Base against the same model
   with `heads: 8, dim_head: 128`, alternating within every round (STEP_ROUNDS, default 3).

The card's name, power limit and max SM clock are printed with the times.  Run from the repository root:
    python tools/dim_head_time.py
"""
import os
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from f5_tts_b200 import ops  # noqa: E402

dev = "cuda:0"
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                           "0"], capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = torch.cuda.get_device_name(0)
print(f"device: {card}")

Be, N, inner = 2, 938, 1024
reps, rounds = int(os.environ.get("ATTN_REPS", "50")), int(os.environ.get("ATTN_ROUNDS", "5"))
g = torch.Generator().manual_seed(0)
qkv = torch.randn(Be * N, 3 * inner, generator=g).half().to(dev)
graphs = {}
for dh in (64, 128):
    heads = inner // dh
    ops.attention(qkv, Be, N, heads, dim_head=dh)  # configure + warm
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(gr, stream=s):
            for _ in range(reps):
                ops.attention(qkv, Be, N, heads, dim_head=dh)
    graphs[dh] = gr
flop = 4.0 * Be * N * N * inner  # QK^T + PV
for r in range(rounds):
    for dh, gr in graphs.items():
        gr.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        gr.replay()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / reps
        print(f"attention Be={Be} N={N} heads={inner // dh} x dim_head={dh} round={r}: {us:.2f} us  "
              f"{flop / us * 1e-6:.1f} TFLOP/s")

os.environ.setdefault("STEP_ARCH", "f5tts_v1_base,f5tts_v1_base_dh128")
os.environ.setdefault("STEP_ROUNDS", "3")
import tools.step_time  # noqa: E402,F401  (runs the alternating sampler-call timing)
