"""GPU tool: the dh-64 attention kernel at 128 queries per CTA (2 consumer warpgroups) against 256 (4), forced through
f5_attention_qwg / f5_attention_joint_qwg, at the tools/attn_bench.py shapes and the MMDiT joint shape (Be 2, N 938,
nt 150).  Each width is a CUDA graph of REPS launches over three rotating QKV buffers; the two graphs are replayed
alternately for ROUNDS rounds.  Prints median and range per launch, what the planner picks (qwg = 0), and checks that
both widths give the same output bit for bit.  The card's name and power limit are read in the same run.
    python tools/attn_qwg_time.py
"""
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from f5_tts_b200 import _lib  # noqa: E402

DEV = "cuda:0"
REPS, ROUNDS = int(os.environ.get("ATTN_REPS", "30")), int(os.environ.get("ATTN_ROUNDS", "11"))
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                           "0"], capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = torch.cuda.get_device_name(0)
print(f"device: {card}, {torch.cuda.get_device_properties(0).multi_processor_count} SMs", flush=True)
L = _lib.lib()


def stream():
    return torch.cuda.current_stream().cuda_stream


def plain(qkv, out, Be, seq, H, qwg):
    _lib.check(L.f5_attention_qwg(qkv.data_ptr(), out.data_ptr(), Be, seq, H, 64, None, 0.125, qwg, stream()),
               "f5_attention_qwg")


def joint(qkv, qkv_c, out, out_c, Be, seq, nt, H, qwg):
    _lib.check(L.f5_attention_joint_qwg(qkv.data_ptr(), qkv_c.data_ptr(), out.data_ptr(), out_c.data_ptr(), Be, seq,
                                        nt, H, 64, None, None, 1, 0.125, qwg, stream()), "f5_attention_joint_qwg")


def graph(fn):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def time_pair(make):
    """{qwg: [us per launch per round]} for qwg 2 and 4, graphs replayed alternately."""
    graphs = {q: graph(make(q)) for q in (2, 4)}
    ts = {2: [], 4: []}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(ROUNDS):
        for q in ((2, 4) if r % 2 == 0 else (4, 2)):
            e0.record()
            graphs[q].replay()
            e1.record()
            torch.cuda.synchronize()
            ts[q].append(e0.elapsed_time(e1) * 1e3 / REPS)
    return ts


def fmt(xs):
    return f"median {statistics.median(xs):7.2f} us  range [{min(xs):7.2f}, {max(xs):7.2f}]"


gen = torch.Generator().manual_seed(0)
for Be, seq, H in ((2, 938, 16), (16, 938, 16), (16, 1875, 16), (2, 1875, 16), (2, 469, 16), (16, 939, 16)):
    qkvs = [torch.randn(Be * seq, 3 * H * 64, generator=gen).half().to(DEV) for _ in range(3)]
    outs = {q: torch.empty(Be * seq, H * 64, dtype=torch.float16, device=DEV) for q in (0, 2, 4)}
    ts = time_pair(lambda q: lambda: [plain(qkvs[i % 3], outs[q], Be, seq, H, q) for i in range(REPS)])
    for q in (0, 2, 4):
        plain(qkvs[0], outs[q], Be, seq, H, q)
    torch.cuda.synchronize()
    pick = [q for q in (2, 4) if torch.equal(outs[0].view(torch.int16), outs[q].view(torch.int16))]
    same = torch.equal(outs[2].view(torch.int16), outs[4].view(torch.int16))
    fl = 4.0 * Be * H * seq * seq * 64
    print(f"attention Be={Be} seq={seq} H={H}: qwg 2 {fmt(ts[2])} | qwg 4 {fmt(ts[4])} | "
          f"{fl / statistics.median(ts[4]) / 1e6:6.1f} TFLOP/s at 4 | planner output equals qwg {pick} | "
          f"bit-equal {same}", flush=True)

Be, N, nt, H = 2, 938, 150, 16
qkvs = [torch.randn(Be * N, 3 * H * 64, generator=gen).half().to(DEV) for _ in range(3)]
qkvc = [torch.randn(Be * nt, 3 * H * 64, generator=gen).half().to(DEV) for _ in range(3)]
outs = {q: (torch.empty(Be * N, H * 64, dtype=torch.float16, device=DEV),
            torch.empty(Be * nt, H * 64, dtype=torch.float16, device=DEV)) for q in (2, 4)}
ts = time_pair(lambda q: lambda: [joint(qkvs[i % 3], qkvc[i % 3], *outs[q], Be, N, nt, H, q) for i in range(REPS)])
for q in (2, 4):
    joint(qkvs[0], qkvc[0], *outs[q], Be, N, nt, H, q)
torch.cuda.synchronize()
same = all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(outs[2], outs[4]))
print(f"joint attention Be={Be} N={N} nt={nt} H={H}: qwg 2 {fmt(ts[2])} | qwg 4 {fmt(ts[4])} | bit-equal {same}",
      flush=True)
