"""GPU timing of the MMDiT path.

1. The joint attention kernel alone at the cfg2 shape (CFG-packed batch Be = 2, N = 938 audio rows, nt = 150 text
   rows, 16 heads of 64) against f5_attention_dh over one contiguous sequence of 938 + 150 = 1088 rows (the same
   FLOPs), CUDA-graph timed (ATTN_REPS launches per replay), alternating for ATTN_ROUNDS rounds; median and range.
2. What one MMDiT block adds to a DiT block at that shape: the text stream's kernels alone (two AdaLN norms, the text
   QKV, out-projection and FF pair over Be * nt = 300 rows, D = 1024) and the joint attention against the DiT
   attention over the 938 audio rows, timed the same way.
3. One cfg2 call (mel front-end, 32 Euler steps, Vocos) of an MMDiT at F5TTS_v1_Base widths (depth 22) against
   F5TTS_v1_Base, alternating within every round (STEP_ROUNDS, default 5); median and range.

The card's name, power limit and max SM clock are printed with the times.  Run from the repository root:
    python tools/mmdit_time.py
"""
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
import bench  # noqa: E402
import synthdata as SD  # noqa: E402
from f5_tts_b200 import ops  # noqa: E402

dev = "cuda:0"
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                           "0"], capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = torch.cuda.get_device_name(0)
print(f"device: {card}")


def summary(xs):
    return f"median {statistics.median(xs):.2f}  range [{min(xs):.2f}, {max(xs):.2f}]  (n={len(xs)})"


# ---- 1. and 2. kernels -----------------------------------------------------------------------------------------------
Be, N, nt, H, dh = 2, 938, 150, 16, 64
inner = H * dh
reps, rounds = int(os.environ.get("ATTN_REPS", "50")), int(os.environ.get("ATTN_ROUNDS", "9"))
g = torch.Generator().manual_seed(0)
qkv = torch.randn(Be * N, 3 * inner, generator=g).half().to(dev)
qkv_c = torch.randn(Be * nt, 3 * inner, generator=g).half().to(dev)
qkv_1 = torch.randn(Be * (N + nt), 3 * inner, generator=g).half().to(dev)
D, F = inner, 2 * inner
c32 = torch.randn(Be * nt, D, generator=g).to(dev)
a16 = c32.half()
mod = torch.randn(D, generator=g).mul(0.02).to(dev)
w_qkv, w_out, w_ff1, w_ff2 = ((torch.randn(n, k, generator=g) / k ** 0.5).half().to(dev)
                              for n, k in ((3 * D, D), (D, D), (F, D), (D, F)))
bias3, bias1, bias2 = (torch.zeros(n, device=dev) for n in (3 * D, D, F))
rope = ops.rope_tables(nt, dev)
ao_c = torch.randn(Be * nt, D, generator=g).half().to(dev)


def text_stream():
    ops.row_norm(c32, 0, mod, mod)
    ops.linear(a16, w_qkv, bias3, epi=ops.EPI_QKV_ROPE, seq=nt, rope=rope, inner=D, pe_heads=H, static_w=True)
    ops.linear(ao_c, w_out, bias1, epi=ops.EPI_RESID, resid=c32, gate=mod, static_w=True)
    ops.row_norm(c32, 0, mod, mod)
    h = ops.linear(a16, w_ff1, bias2, epi=ops.EPI_F16, act=ops.ACT_GELU_TANH, static_w=True)
    ops.linear(h, w_ff2, bias1, epi=ops.EPI_RESID, resid=c32, gate=mod, static_w=True)


calls = {"joint N=938 + nt=150": lambda: ops.attention_joint(qkv, qkv_c, Be, N, nt, H),
         "single seq=1088": lambda: ops.attention(qkv_1, Be, N + nt, H),
         "DiT single seq=938": lambda: ops.attention(qkv, Be, N, H),
         "text stream of one block (Be*nt=300 rows)": text_stream}
graphs = {}
for name, fn in calls.items():
    fn()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(gr, stream=s):
            for _ in range(reps):
                fn()
    graphs[name] = gr
times = {name: [] for name in graphs}
for r in range(rounds):
    for name, gr in graphs.items():
        gr.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        gr.replay()
        e1.record()
        torch.cuda.synchronize()
        times[name].append(e0.elapsed_time(e1) * 1e3 / reps)
flop = 4.0 * Be * (N + nt) ** 2 * inner  # QK^T + PV over N + nt queries and keys
for name, xs in times.items():
    rate = f"  {flop / statistics.median(xs) * 1e-6:.1f} TFLOP/s" if "1088" in name or "joint" in name else ""
    print(f"Be={Be} H={H} dh={dh} {name}: us {summary(xs)}{rate}")

# ---- 3. one cfg2 call -------------------------------------------------------------------------------------------------
import f5_tts_b200 as F5  # noqa: E402

w = bench.WORKLOADS["cfg2"]
base, voc, _ = bench.build_gpu_model("f5tts_v1_base", dev)
cfg = SD.mmdit_v1_base_widths()
mm = F5.CFM(transformer=F5.MMDiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult, mel_dim=100,
                                 text_num_embeds=cfg.text_num_embeds, text_mask_padding=cfg.text_mask_padding),
            vocab_char_map=base.vocab_char_map)
mm.load_state_dict(SD.synthetic_state_dict(cfg, seed=1234), strict=True)
mm = mm.to(dev)
wav, text, duration, lens = (t.to(dev) for t in bench.synth_inputs(w))
models = {"F5TTS_v1_Base": base, "MMDiT at v1_Base widths": mm}


def time_call(model, n=5):
    fn = lambda: bench.hot_path(model, voc, wav, text, duration, lens, w["nfe"])  # noqa: E731
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


for m in models.values():
    for _ in range(3):
        bench.hot_path(m, voc, wav, text, duration, lens, w["nfe"])
call = {k: [] for k in models}
for r in range(int(os.environ.get("STEP_ROUNDS", "5"))):
    for k, m in models.items():
        call[k].append(time_call(m))
for k, xs in call.items():
    print(f"cfg2 call (B=1, N={int(duration[0])}, nt={text.shape[1]}, NFE {w['nfe']}, vocoder) {k}: ms {summary(xs)}")
