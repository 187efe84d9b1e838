"""GPU timing of one batched sampler call on one GPU against the same call with its samples split into groups
(CFM.enable_sample_parallel).

Workloads (synthetic weights, BASELINE.json sizes): cfg3 (F5TTS_Base, B = 8 variable length, exact_varlen), cfg5
(E2TTS_Base, B = 8 x 938 frames, faithful) and one request of 16 text chunks through infer_batch_process (one
exact_varlen sampler call of B = 16, plus the vocoder).  Modes, alternating call by call for ROUNDS rounds (default 5)
after two warm-up rounds:

  * "one GPU": the call unsplit on cuda:0;
  * "loopback x2": two groups, both on cuda:0 (each on its own stream and workspace);
  * "G GPUs" for G = 2, 4, 8 where that many GPUs are visible: one group per GPU;
  * "... full N" (exact_varlen workloads only): the same split with every group at the call's frame count, which
    measures what running each group at its own bucketed length saves.

Each split keeps its peers for the whole run, so every timed call is warm (no weight copy, workspace allocation or
graph capture: checked).  A call runs from its start to a synchronise of the caller's stream (and of every device the
split used).  Printed: median and range per mode, the speed-up against one GPU, and whether the result is bit-equal to
the one-GPU result (exact_varlen: each sample's valid frames, the only ones the mode defines).  The cards' name, power
limit and max SM clock are printed with the numbers.  Run from the repository root:
    python tools/sample_parallel_time.py
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
from f5_tts_b200 import sample_parallel  # noqa: E402

DEV = "cuda:0"
N_GPUS = torch.cuda.device_count()
ROUNDS = int(os.environ.get("ROUNDS", "5"))


def card(i):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                               "-i", str(i)], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(i)


for i in range(N_GPUS):
    print(f"device {i}: {card(i)}")
if N_GPUS < 2:
    print("one visible GPU: splits over several GPUs are not measured; 'loopback' runs both groups on cuda:0")

_plan = sample_parallel.plan_sample_split


def _full_frames(durations, N, exact_varlen, n_devices):
    """The same groups, every one at the call's frame count."""
    return [(b0, b1, N) for b0, b1, _ in _plan(durations, N, exact_varlen, n_devices)]


def modes(varlen):
    """[(label, device list or None, full N)]"""
    out = [("one GPU", None, False), ("loopback x2", [DEV, DEV], False)]
    out += [(f"{g} GPUs", [f"cuda:{i}" for i in range(g)], False) for g in (2, 4, 8) if g <= N_GPUS]
    if varlen:
        out += [(label + " full N", devs, True) for label, devs, _ in out[1:]]
    return out


def sampler_call(model, name):
    w = SD.WORKLOADS[name]
    wav, text, duration, lens = SD.synth_inputs(w)
    wav, text, duration, lens = wav.to(DEV), text.to(DEV), duration.to(DEV), lens.to(DEV)
    cond = model.mel_spec(wav, frames_last=False)
    return lambda: model.sample(cond, text, duration, lens=lens, steps=w["nfe"], cfg_strength=SD.CFG_STRENGTH,
                                sway_sampling_coef=SD.SWAY, seed=0, exact_varlen=name == "cfg3")[0]


CHUNKS = ["I don't really care what you call me.", "I've been a silent spectator, watching species evolve.",
          "Empires rise and fall.", "But always remember, I am mighty and enduring.",
          "Respect me and I'll nurture you; ignore me and you shall face the consequences.", "Yes.",
          "The quick brown fox jumps over the lazy dog, twice, before breakfast.", "Short one.",
          "A rainbow is a meteorological phenomenon caused by reflection, refraction and dispersion of light.",
          "Hello there.", "Some call me nature, others call me mother nature.", "One more sentence of middle length.",
          "It is what it is.", "Numbers like three hundred and twelve are spelled out.", "Almost done now.",
          "And this is the sixteenth and last chunk of the request, a little longer than most of the others."]


def chunked_call(model, voc):
    from f5_tts_b200 import infer

    g = torch.Generator().manual_seed(3)
    ref = (0.1 * torch.randn(1, 4 * 24000, generator=g), 24000)

    def run():
        torch.manual_seed(0)
        wav, _, _ = next(infer.infer_batch_process(ref, "Some call me nature, others call me mother nature. ", CHUNKS,
                                                   model, voc, nfe_step=32, device=DEV))
        return torch.from_numpy(wav)

    return run


def timed(fn, devs):
    s = torch.cuda.current_stream(DEV)
    s.synchronize()
    t0 = time.perf_counter()
    out = fn()
    s.synchronize()
    for d in devs or ():  # the caller's stream already waits for every group; this only guards the clock
        torch.cuda.synchronize(d)
    return (time.perf_counter() - t0) * 1e3, out


def compare(model, fn, label, varlen, lengths=None):
    """`lengths`: exact_varlen defines each sample's first lengths[b] frames only; the bit check compares those."""
    ms = modes(varlen)
    splits = {}

    def run(mode):
        _, devs, full = mode
        key = tuple(devs or ())
        if devs is not None and key not in splits:
            model.enable_sample_parallel(devs)
            splits[key] = model.transformer.sample_split
        model.transformer.sample_split = splits.get(key)
        sample_parallel.plan_sample_split = _full_frames if full else _plan
        try:
            return timed(fn, devs)
        finally:
            model.transformer.sample_split = None
            sample_parallel.plan_sample_split = _plan

    for _ in range(2):  # warm-up: engines, replicas, workspaces, graphs; "full N" reuses its split's peers
        for m in ms:
            run(m)
    warm = {k: [(p.replications, len(p._ws_free)) for p in s.peers] for k, s in splits.items()}
    times = {m[0]: [] for m in ms}
    outs = {}
    for _ in range(ROUNDS):
        for m in ms:
            t, outs[m[0]] = run(m)
            times[m[0]].append(t)
    assert {k: [(p.replications, len(p._ws_free)) for p in s.peers] for k, s in splits.items()} == warm, \
        "split calls were not warm"
    one = statistics.median(times["one GPU"])
    ref = outs["one GPU"].cpu()
    for name, _, _ in ms:
        t = times[name]
        o = outs[name].cpu()
        same = (all(torch.equal(ref[i, :d], o[i, :d]) for i, d in enumerate(lengths)) if lengths
                else torch.equal(ref, o))
        print(f"{label:8s} {name:22s} {statistics.median(t):8.1f} ms [{min(t):.1f}, {max(t):.1f}]   "
              f"speed-up {one / statistics.median(t):.2f}x   bit-equal {same}")


model, voc, _ = build_gpu_model("f5tts_base", DEV)
compare(model, sampler_call(model, "cfg3"), "cfg3", True, SD.WORKLOADS["cfg3"]["frames"])
compare(model, chunked_call(model, voc), "chunks16", True)
del model
torch.cuda.empty_cache()
e2, _, _ = build_gpu_model("e2tts_base", DEV)
compare(e2, sampler_call(e2, "cfg5"), "cfg5", False)
