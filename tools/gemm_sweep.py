"""GPU tool: time the persistent wgmma GEMM per (shape, epilogue, tile) from a CUDA graph (rotating weights > L2).

Every row ends with the same shape through cuBLAS (torch.matmul fp16, no epilogue) as a comparator.
SWEEP_M=<M,...> picks the row counts; SWEEP_TILES=auto times only the planner's pick.  With the instrumented library
(F5_LIB=f5_tts_b200/libf5tts_b200_trace.so) and F5_GEMM_EPI=none the times are of the main loop alone.
SWEEP_CONV=1 instead times the conv position embedding pair (Conv1d(k=31, groups=16) + Mish to fp16, then the same
with the fp32 residual add) at B = 2, N = 938 for dim 768 (48 channels per group) and dim 1024 (64 per group).
"""
import os
import sys

import torch

sys.path.insert(0, ".")
from bench import _graph_time_us  # noqa: E402
from f5_tts_b200 import ops  # noqa: E402
from f5_tts_b200.ops import *  # noqa: E402,F403

DEV = "cuda:0"
torch.cuda.init()
g = torch.Generator().manual_seed(0)


def bench(M, N, K, epi, act, bn, nw=24):
    a = [torch.randn(M, K, generator=g).half().to(DEV) for _ in range(2)]
    w = [(torch.randn(N, K, generator=g) / 32).half().to(DEV) for _ in range(nw)]
    b = torch.randn(N, generator=g).to(DEV)
    kw = dict(epi=epi, act=act, bn=bn, static_w=True)
    if epi == EPI_RESID:
        kw["resid"] = torch.zeros(M, N, device=DEV)
        kw["gate"] = torch.randn(N, generator=g).to(DEV)
    if epi == EPI_QKV_ROPE:
        seq = M // 2
        kw.update(seq=seq, rope=ops.rope_tables(seq, DEV), inner=N // 3, pe_heads=1)
    us = _graph_time_us(lambda: [ops.linear(a[i % 2], w[i], b, **kw) for i in range(nw)], nw, rounds=4)
    return us, 2.0 * M * N * K / (us * 1e-6) / 1e12


def cublas(M, N, K, nw):
    a = [torch.randn(M, K, generator=g).half().to(DEV) for _ in range(2)]
    wt = [(torch.randn(N, K, generator=g) / 32).half().to(DEV).t() for _ in range(nw)]
    return _graph_time_us(lambda: [torch.matmul(a[i % 2], wt[i]) for i in range(nw)], nw, rounds=4)


def conv_pair(D, B=2, N=938, nw=8):
    G = D // 16
    x = torch.randn(B, N, D, generator=g).half().to(DEV)
    w = [(torch.randn(31, D, G, generator=g) / (G * 31) ** 0.5).half().to(DEV) for _ in range(2 * nw)]
    b = torch.randn(D, generator=g).to(DEV)
    r = torch.zeros(B, N, D, device=DEV)

    def pair(i):
        c = ops.grouped_conv31(x, w[2 * i], b)
        ops.grouped_conv31(c, w[2 * i + 1], b, resid=r)

    us = _graph_time_us(lambda: [pair(i) for i in range(nw)], nw, rounds=20)
    return us, 2 * 2.0 * B * N * D * G * 31 / (us * 1e-6) / 1e12


if os.environ.get("SWEEP_CONV"):
    for D in (768, 1024):
        us, tf = conv_pair(D)
        print(f"conv pair D={D} G={D // 16} B=2 N=938: {us:6.1f}us per pair  {tf:5.1f} algorithmic TF", flush=True)
    sys.exit(0)

Ms = [int(x) for x in os.environ.get("SWEEP_M", "1876,3752,7504,15008").split(",")]
pick_only = os.environ.get("SWEEP_TILES", "all") == "auto"
for M in Ms:
    for (N, K, epi, act, tag) in ((3072, 1024, EPI_QKV_ROPE, ACT_NONE, "QKV"), (1024, 1024, EPI_RESID, ACT_NONE, "out"),
                                  (2048, 1024, EPI_F16, ACT_GELU_TANH, "FF1"), (1024, 2048, EPI_RESID, ACT_NONE, "FF2"),
                                  (4096, 1024, EPI_F16, ACT_GELU_TANH, "FF1-e2"), (1024, 4096, EPI_RESID, ACT_NONE, "FF2-e2")):
        if M > 2000 and "e2" in tag:
            continue
        nw = -(-200_000_000 // (N * K * 2))  # distinct weights > L2 (50 MB), as in the real step
        nw = nw if M < 8000 else max(6, nw // 4)
        auto = ops.gemm_tile(M, N, K, epi, act)[0]
        row = []
        for bn in [auto] if pick_only else (128, 192, 256):
            us, tf = bench(M, N, K, epi, act, bn, nw=nw)
            row.append(f"bn{bn}: {us:6.1f}us {tf:5.0f}TF")
        print(f"M={M:6d} {tag:7s} N={N:5d} K={K:5d} | " + " | ".join(row) + f" | auto={auto}"
              f" | cuBLAS {cublas(M, N, K, nw):6.1f}us", flush=True)
