"""GPU timing of concurrent CFM.sample callers with batching off and on (CFM.enable_batching).

Workload: K client threads (KS, default 1,2,4,8), each issuing CALLS (default 4) cfg2-like calls one after another:
B = 1, a 282-frame prompt, 100-200 text tokens, 700-1100 frames in all, 32 Euler steps, cfg 2, sway -1, at
F5TTS_v1_Base widths (synthetic weights).  Lengths are drawn once per (round, K) and used by both modes; the two modes
alternate within each round (ROUNDS, default 3).  A call's latency runs from its start to its result being complete on
the GPU (a synchronise of the caller's stream).  Per K and mode: requests/s, generated frames/s (frames past the
prompt), p50 / p95 latency over all rounds, the batch sizes that ran and the mean GPU idle gap when a queued batch took
over.  Then, with graphs warm: a lone caller with batching off and on (the same call alternating), and the engine
time of 8 single-sample calls against one merged exact_varlen call of the same 8 samples.  Last, the cost of a new graph
key: the first engine call at a (B, N) the engine has not seen (workspace, graph capture and instantiation) against
the next call with that key.  The card's name, power limit and max SM clock are printed with
the numbers.  Run from the repository root:
    python tools/concurrent_sample_time.py
"""
import collections
import os
import random
import statistics
import subprocess
import sys
import threading
import time

import torch

sys.path.insert(0, ".")
import synthdata as SD  # noqa: E402

dev = "cuda:0"
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                           "0"], capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = torch.cuda.get_device_name(0)
print(f"device: {card}")

import f5_tts_b200 as F5  # noqa: E402

PROMPT, NFE = 282, 32
KS = [int(k) for k in os.environ.get("KS", "1,2,4,8").split(",")]
CALLS = int(os.environ.get("CALLS", "4"))
ROUNDS = int(os.environ.get("ROUNDS", "3"))

cfg = SD.f5tts_v1_base()
model = F5.CFM(transformer=F5.DiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, ff_mult=cfg.ff_mult,
                                  text_dim=cfg.text_dim, text_mask_padding=cfg.text_mask_padding,
                                  conv_layers=cfg.conv_layers, pe_attn_head=cfg.pe_attn_head,
                                  text_num_embeds=cfg.text_num_embeds, mel_dim=100))
model.load_state_dict(SD.synthetic_state_dict(cfg, seed=1234), strict=True)
model = model.to(dev)
g = torch.Generator().manual_seed(0)
cond = torch.randn(1, PROMPT, 100, generator=g).to(dev)
texts = [torch.randint(0, cfg.text_num_embeds, (1, n), generator=g).to(dev) for n in range(100, 201)]


def one_call(duration, seed):
    t0 = time.perf_counter()
    model.sample(cond, texts[seed % len(texts)], duration, steps=NFE, cfg_strength=2.0, sway_sampling_coef=-1.0,
                 seed=seed)
    torch.cuda.current_stream().synchronize()
    return time.perf_counter() - t0


def run(plan):
    """plan[k] = [durations of thread k's calls] -> (wall seconds, [latency seconds])"""
    lat, go = [], threading.Barrier(len(plan) + 1)

    def client(k):
        go.wait()
        for i, d in enumerate(plan[k]):
            lat.append(one_call(d, 1000 * k + i))

    threads = [threading.Thread(target=client, args=(k,)) for k in range(len(plan))]
    for t in threads:
        t.start()
    go.wait()
    t0 = time.perf_counter()
    for t in threads:
        t.join()
    return time.perf_counter() - t0, lat


def pct(xs, p):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(round(p / 100 * (len(xs) - 1))))]


rng = random.Random(1)
res = collections.defaultdict(lambda: dict(wall=0.0, calls=0, frames=0, lat=[], sizes=collections.Counter(),
                                           handoffs=0, gap=0.0))
for r in range(ROUNDS + 1):  # round 0 warms up every shape (graph capture) and is not reported
    for K in KS:
        plan = [[rng.randint(700, 1100) for _ in range(CALLS)] for _ in range(K)]
        for mode in ("off", "on"):
            stats = model.enable_batching() if mode == "on" else None
            try:
                wall, lat = run(plan)
            finally:
                model.disable_batching()
            if r == 0:
                continue
            a = res[(K, mode)]
            a["wall"] += wall
            a["calls"] += len(lat)
            a["frames"] += sum(d - PROMPT for p in plan for d in p)
            a["lat"] += lat
            if stats is not None:
                a["sizes"] += stats.batch_sizes
                a["handoffs"] += stats.handoffs
                a["gap"] += stats.handoff_gap_ms

print(f"workload: K threads x {CALLS} calls, B = 1, {PROMPT}-frame prompt, 700-1100 frames, NFE {NFE}, cfg 2, sway -1, "
      f"F5TTS_v1_Base widths; {ROUNDS} rounds, modes alternating")
for K in KS:
    for mode in ("off", "on"):
        a = res[(K, mode)]
        line = (f"K={K} batching {mode:3s}: {a['calls'] / a['wall']:6.2f} req/s  {a['frames'] / a['wall']:8.0f} frames/s  "
                f"latency p50 {1e3 * statistics.median(a['lat']):7.1f} ms  p95 {1e3 * pct(a['lat'], 95):7.1f} ms")
        if mode == "on":
            gap = a["gap"] / a["handoffs"] if a["handoffs"] else float("nan")
            line += f"  calls per run {dict(sorted(a['sizes'].items()))}  idle gap at hand-off {gap:.2f} ms"
        print(line)

tr = model.transformer
grid = torch.linspace(0, 1, NFE + 1).tolist()


def engine_ms(B, N, durs=None):
    """host time of one engine call, ending in a device synchronise"""
    y = torch.randn(B, N, 100, device=dev)
    sc = torch.zeros_like(y)
    text = torch.randint(0, cfg.text_num_embeds, (B, 150), device=dev)
    dur = None if durs is None else torch.tensor(durs, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tr.run(y.clone(), sc, text, grid, dur, 2.0, exact_varlen=dur is not None)
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


# a lone caller: the same call alternately with batching off and on, graphs warm
lone = {"off": [], "on": []}
for i in range(2 * int(os.environ.get("LONE_CALLS", "10")) + 2):
    mode = ("off", "on")[i % 2]
    if mode == "on":
        model.enable_batching()
    try:
        ms = 1e3 * one_call(938, 7)
    finally:
        model.disable_batching()
    if i >= 2:
        lone[mode].append(ms)
print(f"lone caller, 938 frames: batching off median {statistics.median(lone['off']):.2f} ms "
      f"[{min(lone['off']):.2f}, {max(lone['off']):.2f}], on {statistics.median(lone['on']):.2f} ms "
      f"[{min(lone['on']):.2f}, {max(lone['on']):.2f}]")

# what merging buys on the GPU: 8 single-sample engine calls against one exact_varlen call of the 8, graphs warm
durs = [rng.randint(700, 1024) for _ in range(8)]
for _ in range(2):
    solo_ms = [engine_ms(1, d) for d in durs]
    merged_ms = engine_ms(8, 1024, durs)
print(f"engine time of 8 samples ({min(durs)}-{max(durs)} frames, NFE {NFE}): 8 single calls {sum(solo_ms):.1f} ms, "
      f"one merged call (B = 8, padded to 1024) {merged_ms:.1f} ms, ratio {merged_ms / sum(solo_ms):.3f}")

# cost of a new graph key: the first engine call at a (B, N) the engine has not seen against the next one
for B, N in ((1, 1133), (8, 1280)):
    durs = None if B == 1 else [N - 37 * i for i in range(B)]
    first = engine_ms(B, N, durs)
    nxt = engine_ms(B, N, durs)
    print(f"new graph key B={B} N={N}: first call {first:.1f} ms, next call {nxt:.1f} ms, difference {first - nxt:.1f} ms")
print(f"device: {card}")
