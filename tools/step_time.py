"""GPU diagnostic: device time of one CFM.sample call (default cfg2, NFE 32) — used with the instrumented build and
F5_DIAG_SKIP=<kernel class> to read the in-situ cost of that class as the difference to the full step.

STEP_ODE=<method>:<steps>[,<method>:<steps>...] times each ODE solver setting in turn (default euler:<workload NFE>),
STEP_ROUNDS=<n> repeats the whole list n times, alternating, so that settings are compared within one process
(e.g. STEP_ODE=euler:32,midpoint:16 — both make 32 backbone evaluations).
STEP_ARCH=<preset>[,<preset>...] (synthdata presets, default the workload's arch) times each architecture on the same
inputs, alternating within every round (e.g. STEP_ARCH=f5tts_v1_base,f5tts_v1_small)."""
import os
import subprocess
import sys

import torch

sys.path.insert(0, ".")
import bench  # noqa: E402

dev = "cuda:0"
name = os.environ.get("STEP_WORKLOAD", "cfg2")
w = bench.WORKLOADS[name]
runs = [(m, int(s)) for m, s in (p.split(":") for p in os.environ.get("STEP_ODE", f"euler:{w['nfe']}").split(","))]
rounds = int(os.environ.get("STEP_ROUNDS", "1"))
archs = os.environ.get("STEP_ARCH", w["arch"]).split(",")
models = {}
for a in archs:
    models[a], voc, _ = bench.build_gpu_model(a, dev)
wav, text, duration, lens = (t.to(dev) for t in bench.synth_inputs(w))
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = torch.cuda.get_device_name(0)
print(f"device: {card}")


def time_call(model, method, steps, n=5):
    model.odeint_kwargs = dict(method=method)
    fn = lambda: bench.hot_path(model, voc, wav, text, duration, lens, steps)  # noqa: E731
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


for r in range(rounds):
    for arch in archs:
        for method, steps in runs:
            nfe = 2 * steps if method == "midpoint" else steps
            ms = time_call(models[arch], method, steps)
            print(f"{name} arch={arch} ode={method} steps={steps} nfe={nfe} round={r} ms_per_call {ms:.3f}  "
                  f"per_NFE_us {ms * 1e3 / nfe:.1f}  skip={os.environ.get('F5_DIAG_SKIP', '')}")
