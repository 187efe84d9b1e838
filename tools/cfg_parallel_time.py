"""GPU timing of one sampler call on one GPU against the same call with its unconditional CFG half on a second GPU
(CFM.enable_cfg_parallel).

Workloads (synthetic weights, BASELINE.json sizes): cfg2 (F5TTS_Base, B = 1, 938 frames, NFE 32), cfg3 (F5TTS_Base,
B = 8 variable length, exact_varlen), cfg5 (E2TTS_Base, B = 8 x 938 frames), and one chunked request through
infer_batch_process (four text chunks in one batched sampler call, plus the vocoder).  Per workload the two modes
alternate call by call (ROUNDS, default 7, after a warm-up of each) with one peer kept for the whole run, so every timed
split call is warm (no weight copy, workspace allocation or graph capture: checked); a call runs from its start to a
synchronise of the caller's stream.  Printed: median and range per mode, the split result's bit equality with the one-GPU result, and,
from a torch.profiler trace of one split cfg2 and cfg3 call (a run of its own), the per-evaluation exchange copies
(count and mean time per device).  The card's name, power limit and max SM clock are printed with the numbers.

With one visible GPU the "pair" is loopback (both halves on cuda:0, two streams): that measures the cost of the split's
extra launches and copies, not the gain of a second GPU, and the output says so.  Run from the repository root:
    python tools/cfg_parallel_time.py
"""
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, ".")
import synthdata as SD  # noqa: E402
from bench import build_gpu_model  # noqa: E402

DEV = "cuda:0"
N_GPUS = torch.cuda.device_count()
PEER = "cuda:1" if N_GPUS >= 2 else DEV
ROUNDS = int(os.environ.get("ROUNDS", "7"))


def card(i):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                               "-i", str(i)], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(i)


print(f"device 0: {card(0)}")
if N_GPUS >= 2:
    print(f"device 1: {card(1)}")
else:
    print("one visible GPU: the 'pair' below is LOOPBACK (both halves on cuda:0), not two GPUs")


def sampler_call(model, name):
    w = SD.WORKLOADS[name]
    wav, text, duration, lens = SD.synth_inputs(w)
    wav, text, duration, lens = wav.to(DEV), text.to(DEV), duration.to(DEV), lens.to(DEV)
    cond = model.mel_spec(wav, frames_last=False)
    if w["B"] == 1:
        return lambda: model.sample(wav, text, int(duration[0]), steps=w["nfe"], cfg_strength=SD.CFG_STRENGTH,
                                    sway_sampling_coef=SD.SWAY, seed=0)[0]
    return lambda: model.sample(cond, text, duration, lens=lens, steps=w["nfe"], cfg_strength=SD.CFG_STRENGTH,
                                sway_sampling_coef=SD.SWAY, seed=0, exact_varlen=name == "cfg3")[0]


def chunked_call(model, voc):
    from f5_tts_b200 import infer

    g = torch.Generator().manual_seed(3)
    ref = (0.1 * torch.randn(1, 4 * 24000, generator=g), 24000)
    chunks = ["I don't really care what you call me.", "I've been a silent spectator, watching species evolve.",
              "Empires rise and fall.", "But always remember, I am mighty and enduring, whatever you call me."]

    def run():
        torch.manual_seed(0)
        wav, _, _ = next(infer.infer_batch_process(ref, "Some call me nature, others call me mother nature. ", chunks,
                                                   model, voc, nfe_step=32, device=DEV))
        return torch.from_numpy(wav)

    return run


def timed(fn):
    s = torch.cuda.current_stream(DEV)
    s.synchronize()
    t0 = time.perf_counter()
    out = fn()
    s.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


_peers = {}


def set_split(model, on):
    """Switches the split on or off without dropping the peer: one peer per model for the whole run, so its weight
    copy, stream, workspace and captured graphs stay warm, as in a user's steady state."""
    if id(model) not in _peers:
        _peers[id(model)] = model.enable_cfg_parallel(PEER)
    model.transformer.cfg_peer = _peers[id(model)] if on else None


def compare(model, fn, label, lengths=None):
    """`lengths`: exact_varlen defines each sample's first lengths[b] frames only; the bit check compares those."""
    for split in (False, True):  # warm-up: engines, replica, workspaces, graphs
        set_split(model, split)
        timed(fn)
    peer = _peers[id(model)]
    made, pooled = peer.replications, len(peer._ws_free)
    times = {False: [], True: []}
    outs = {}
    for _ in range(ROUNDS):
        for split in (False, True):
            set_split(model, split)
            ms, outs[split] = timed(fn)
            times[split].append(ms)
    set_split(model, False)
    # steady state: the timed split calls made no new weight copy and no new peer workspace
    assert peer.replications == made and len(peer._ws_free) == pooled, "split calls were not warm"
    one, two = times[False], times[True]
    a, b = outs[False].cpu(), outs[True].cpu()
    same = all(torch.equal(a[i, :d], b[i, :d]) for i, d in enumerate(lengths)) if lengths else torch.equal(a, b)
    print(f"{label:9s} one GPU {statistics.median(one):8.1f} ms [{min(one):.1f}, {max(one):.1f}]   "
          f"{'pair' if N_GPUS >= 2 else 'loopback'} {statistics.median(two):8.1f} ms [{min(two):.1f}, {max(two):.1f}]   "
          f"speed-up {statistics.median(one) / statistics.median(two):.2f}x   bit-equal {same}")


def exchange_trace(model, fn, label, evals):
    from torch.profiler import ProfilerActivity, profile

    set_split(model, True)
    timed(fn)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        timed(fn)
        torch.cuda.synchronize(PEER)
    set_split(model, False)
    groups = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" in ev.name and ("PtoP" in ev.name or
                                                                                         "DtoD" in ev.name):
            groups.setdefault((ev.name, ev.device_index), []).append(ev.device_time)
    # the exchange is one copy per evaluation and device; the few others (inputs to the peer, trajectory row 0) are
    # outnumbered, so the median is the exchange copy's time
    for (name, dev), ts in sorted(groups.items()):
        print(f"  [{label}] {name} on device {dev}: {len(ts)} copies ({evals} evaluations), median "
              f"{statistics.median(ts):.1f} us, max {max(ts):.1f} us, sum {sum(ts) / 1e3:.2f} ms")


model, voc, _ = build_gpu_model("f5tts_base", DEV)
for name in ("cfg2", "cfg3"):
    compare(model, sampler_call(model, name), name, SD.WORKLOADS[name]["frames"] if name == "cfg3" else None)
compare(model, chunked_call(model, voc), "chunked")
for name in ("cfg2", "cfg3"):
    exchange_trace(model, sampler_call(model, name), name, SD.WORKLOADS[name]["nfe"])
del model, voc
torch.cuda.empty_cache()
e2, _, _ = build_gpu_model("e2tts_base", DEV)
compare(e2, sampler_call(e2, "cfg5"), "cfg5")
