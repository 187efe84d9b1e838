"""GPU timing of the backbone operator transformer(x, cond, text, time, ..., cfg_infer=True) at the cfg2 shape
(F5TTS_Base, B = 1, N = 938, cond | uncond packed) against one backbone evaluation inside a sampler call.

Arms, alternating in every round for ROUNDS rounds (default 7) after two warm-up rounds:
  * "one-step f5_sample": what the operator ran before f5_forward existed, a one-step eager f5_sample call with v_out;
  * "forward cache=False": f5_forward with the text embeddings recomputed, graph replay;
  * "forward cache=True": f5_forward reusing the text embeddings, graph replay;
  * "forward cache=True, B = 3": three samples at three different times in one call (the per-sample AdaLN kernels);
  * "engine evaluation": one 32-step Euler sampler call (graph) divided by its 32 evaluations;
  * "RK4 8 steps": a torchdiffeq-style RK4 (3/8 rule) loop over forward(cache=True), 32 evaluations plus the torch
    updates, against "Euler 32 steps", the sampler call itself.
Operator arms time CALLS back-to-back calls between two synchronises (default 32) and report per call;
"host enqueue" is the host time of those cached calls up to the last return, before the synchronise.  Printed: median
and range per arm over the rounds, with the card's name, power limit and max SM clock, then, from a torch.profiler run of
its own, the kernels and copies per cached operator call and per sampler evaluation with their durations summed
(kernels that overlap under programmatic dependent launch count in full, so the sum exceeds the elapsed time).  Run
from the repository root:
    python tools/forward_time.py
"""
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, ".")
import synthdata as SD  # noqa: E402
from bench import build_gpu_model  # noqa: E402

DEV = "cuda:0"
ROUNDS = int(os.environ.get("ROUNDS", "7"))
CALLS = int(os.environ.get("CALLS", "32"))
CFG = 2.0


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def enqueue(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    ms = (time.perf_counter() - t0) * 1e3 / reps
    torch.cuda.synchronize()
    return ms


def device_time(fn, reps):
    """Summed kernel, memcpy and memset durations per call, and the number of such activities per call"""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    ev = [e for e in trace.get("traceEvents", []) if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    return sum(float(e.get("dur", 0.0)) for e in ev) / 1e3 / reps, len(ev) / reps


def timed(fn, reps=1):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def main():
    print(f"device 0: {card()}")
    w = SD.WORKLOADS["cfg2"]
    model, _, _ = build_gpu_model(w["arch"], DEV)
    tr = model.transformer
    N, B, nt = 938, 1, 220
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, N, 100, generator=g).to(DEV)
    cond = torch.randn(B, N, 100, generator=g).to(DEV)
    cond[:, 282:] = 0  # the prompt's frames, zeros past them (cfm.py:151-153)
    text = torch.randint(0, 2545, (B, nt), generator=g).to(DEV)
    t_grid = torch.linspace(0, 1, 33)
    t_grid = (t_grid + SD.SWAY * (torch.cos(torch.pi / 2 * t_grid) - 1 + t_grid)).tolist()
    t1 = torch.full((B,), 0.4, device=DEV)
    v = torch.empty(2 * B, N, 100, device=DEV)
    x3, cond3 = torch.randn(3, N, 100, generator=g).to(DEV), cond.expand(3, -1, -1).contiguous()
    text3 = torch.randint(0, 2545, (3, nt), generator=g).to(DEV)
    t3 = torch.tensor([0.1, 0.4, 0.8], device=DEV)

    def old_operator():
        tr._run_local(x.clone(), cond, text, [0.4, 1.4], None, 1.0, None, v, use_graph=False)

    def fwd(cache):
        return lambda: tr(x, cond, text, t1, cfg_infer=True, cache=cache)

    def fwd3():
        tr(x3, cond3, text3, t3, cfg_infer=True, cache=True)

    def euler32():
        tr._run_local(x.clone(), cond, text, t_grid, None, CFG, None, None, use_graph=True)

    def flow(tk, y):
        o = tr(y, cond, text, torch.full((B,), float(tk), device=DEV), cfg_infer=True, cache=True)
        return o[:B] + (o[:B] - o[B:]) * CFG

    def rk4():
        t = torch.linspace(0, 1, 9)
        y = x
        for k in range(8):
            t0, dt = t[k], t[k + 1] - t[k]
            k1 = flow(t0, y)
            k2 = flow(t0 + dt / 3, y + dt * k1 / 3)
            k3 = flow(t0 + dt * 2 / 3, y + dt * (k2 - k1 / 3))
            k4 = flow(t[k + 1], y + dt * (k1 - k2 + k3))
            y = y + (k1 + 3 * (k2 + k3) + k4) * dt * 0.125
        return y

    arms = {
        "one-step f5_sample (ms/call)": lambda: timed(old_operator, CALLS),
        "forward cache=False (ms/call)": lambda: timed(fwd(False), CALLS),
        "forward cache=True (ms/call)": lambda: timed(fwd(True), CALLS),
        "forward cache=True, host enqueue (ms/call)": lambda: enqueue(fwd(True), CALLS),
        "forward cache=True, B = 3 (ms/call)": lambda: timed(fwd3, CALLS),
        "engine evaluation (ms/eval)": lambda: timed(euler32) / 32,
        "RK4 8 steps over forward (ms/call)": lambda: timed(rk4),
        "Euler 32 steps, sampler (ms/call)": lambda: timed(euler32),
    }
    res = {k: [] for k in arms}
    for r in range(ROUNDS + 2):
        tr.clear_cache()
        for k, fn in arms.items():
            ms = fn()
            if r >= 2:
                res[k].append(ms)
    a = tr(x, cond, text, t1, cfg_infer=True, cache=False)
    old_operator()
    print(f"forward == one-step f5_sample evaluation: {bool(torch.equal(a, v))}")
    print(f"{ROUNDS} rounds, median [min, max]:")
    for k, v_ in res.items():
        print(f"  {k:44s} {statistics.median(v_):8.3f}  [{min(v_):.3f}, {max(v_):.3f}]")
    ms, n = device_time(fwd(True), 8)
    print(f"forward(cache=True) call: {n:.0f} kernels and copies, durations summed {ms:.3f} ms")
    ms, n = device_time(fwd(False), 8)
    print(f"forward(cache=False) call: {n:.0f} kernels and copies, durations summed {ms:.3f} ms")
    ms, n = device_time(euler32, 2)
    print(f"sampler evaluation: {n / 32:.1f} kernels and copies, durations summed {ms / 32:.3f} ms")


if __name__ == "__main__":
    main()
