"""GPU timing of UNetT skip_connect_type "concat", "add" and "none".

One cfg5-shaped call per model (E2TTS_Base widths and depth, B = 8 x 938 frames, 150 text tokens, 32 Euler steps with
CFG, mel front-end + CFM.sample + Vocos, as bench.py's cfg5 record), the three models alternating within every round
(ROUNDS, default 5; CALLS calls per timed window, default 3); median and range per model.  The three models share every
weight but the concat model's skip projections.  The card's name, power limit and max SM clock are read and printed in
the same run.  Run from the repository root:
    python tools/unett_skip_time.py
"""
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
import bench  # noqa: E402
import synthdata as SD  # noqa: E402

dev = "cuda:0"
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                           "0"], capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = torch.cuda.get_device_name(0)
print(f"device: {card}")

import f5_tts_b200 as F5  # noqa: E402
from f5_tts_b200.vocoder import Vocos  # noqa: E402


def summary(xs):
    return f"median {statistics.median(xs):.2f}  range [{min(xs):.2f}, {max(xs):.2f}]  (n={len(xs)})"


w = bench.WORKLOADS["cfg5"]
sd = SD.synthetic_state_dict(SD.e2tts_base(), seed=1234)  # concat: a superset of the add / none keys
models = {}
for t in ("concat", "add", "none"):
    cfg = SD.e2tts_base()
    cfg.skip_connect_type = t
    m = F5.CFM(transformer=F5.UNetT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult,
                                    text_dim=cfg.text_dim, text_mask_padding=cfg.text_mask_padding,
                                    conv_layers=cfg.conv_layers, pe_attn_head=cfg.pe_attn_head,
                                    text_num_embeds=cfg.text_num_embeds, mel_dim=100, skip_connect_type=t))
    keys = {k for k, _, _ in SD.state_dict_spec(cfg)}
    m.load_state_dict({k: v for k, v in sd.items() if k in keys}, strict=True)
    models[t] = m.to(dev)
voc = Vocos()
voc.load_state_dict(SD.synthetic_vocos_state_dict(), strict=False)
voc = voc.to(dev)
wav, text, duration, lens = (t.to(dev) for t in bench.synth_inputs(w))


def call(m):
    return bench.hot_path(m, voc, wav, text, duration, lens, w["nfe"])


def time_calls(m, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        call(m)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


for m in models.values():
    for _ in range(2):
        call(m)
n = int(os.environ.get("CALLS", "3"))
ms = {k: [] for k in models}
for r in range(int(os.environ.get("ROUNDS", "5"))):
    for k, m in models.items():
        ms[k].append(time_calls(m, n))
B, N = w["B"], w["frames"][0]
for k, xs in ms.items():
    fl = models[k].transformer.sample_flops(B, N, w["nfe"], bench.CFG_STRENGTH, nt=text.shape[1])
    print(f"cfg5 call (B={B}, N={N}, nt={text.shape[1]}, NFE {w['nfe']}, mel + sample + vocoder) {k}: ms {summary(xs)}"
          f"  sample FLOPs {fl:.4e}")
print(f"device: {card}")
