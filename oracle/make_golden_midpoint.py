"""Generate the midpoint-solver fixtures by running the UNMODIFIED reference's CFM.sample with
odeint_kwargs=dict(method="midpoint") (TEST INFRASTRUCTURE).  Needs the reference checkout (F5_REFERENCE_SRC = its
src directory); runs on the CPU:

    F5_REFERENCE_SRC=<reference>/src python -m oracle.make_golden_midpoint

torchdiffeq is not installed, so the midpoint step is oracle/ode_midpoint.odeint's restatement of torchdiffeq's
fixed-grid midpoint method (parity unpinned, DESIGN.md §2), registered as the `torchdiffeq` stand-in before the
reference is imported.  Writes new files only:

* tests/golden/reference_tiny_dit_varlen_midpoint.npz: the tiny DiT var-len case of
  oracle/make_golden_reference_checks.tiny_dit_varlen_case (inputs and noise regenerate from seeds);
* tests/golden/f5base_b2_varlen_midpoint.npz: F5TTS_Base width, B = 2, variable length, 3 steps, CFG 2, sway -1,
  stored with the keys of the oracle/make_golden.py fixtures (weights regenerate from (cfg, wseed)).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import f5_oracle as O  # noqa: E402
from oracle import make_golden as MG  # noqa: E402
from oracle import make_golden_reference_checks as MR  # noqa: E402
from oracle import ode_midpoint as OM  # noqa: E402
from oracle import ref_shims  # noqa: E402

TINY = "reference_tiny_dit_varlen_midpoint"
FULL = "f5base_b2_varlen_midpoint"


def full_width_case():
    """(cfg, wseed, cond, text, duration, lens, sample kwargs) of the F5TTS_Base fixture, shared with the tests."""
    cfg = O.f5tts_base()
    g = torch.Generator().manual_seed(123)
    cond = torch.randn(2, 48, 100, generator=g)
    text = torch.randint(0, cfg.text_num_embeds, (2, 30), generator=g)
    text[1, 22:] = -1
    return (cfg, 1234, cond, text, torch.tensor([184, 152]), torch.tensor([48, 40]),
            dict(steps=3, cfg_strength=2.0, sway_sampling_coef=-1.0, seed=11))


def midpoint_reference(cfg, sd):
    # cfm.py binds `odeint` from torchdiffeq when it is imported, and ref_shims.install() keeps a stand-in that is
    # already registered: register the restatement that knows the midpoint method first
    if "f5_tts.model.cfm" not in sys.modules:
        ref_shims._stub("torchdiffeq", odeint=OM.odeint)
    model = MG.build_reference(cfg, sd)
    assert sys.modules["f5_tts.model.cfm"].odeint is OM.odeint, "the reference was imported with another odeint"
    model.odeint_kwargs = dict(method="midpoint")  # what CFM(odeint_kwargs=dict(method="midpoint")) stores (cfm.py:74)
    return model


def main():
    if not ref_shims.reference_available():
        raise SystemExit("set F5_REFERENCE_SRC to the reference checkout's src directory")
    torch.set_num_threads(os.cpu_count() or 8)

    cfg, sd, cond, text, dur, kw = MR.tiny_dit_varlen_case()
    with torch.no_grad():
        out, traj = midpoint_reference(cfg, sd).sample(cond=cond, text=text, duration=dur, **kw)
    res = OM.sample(sd, cfg, cond, text, dur, method="midpoint", **kw)
    print(f"[{TINY}] out {tuple(out.shape)} traj rows {traj.shape[0]} oracle rel-L2 {MG.rel_l2(res.out, out):.3e}")
    np.savez_compressed(os.path.join(MG.GOLD, TINY + ".npz"), out=out.numpy(), y0=traj[0].numpy(),
                        traj_1=traj[1].numpy())

    cfg, wseed, cond, text, dur, lens, kw = full_width_case()
    sd = O.synthetic_state_dict(cfg, seed=wseed)
    with torch.no_grad():
        out, traj = midpoint_reference(cfg, sd).sample(cond=cond, text=text, duration=dur, lens=lens, **kw)
    res = OM.sample(sd, cfg, cond, text, dur, lens=lens, method="midpoint", **kw)
    print(f"[{FULL}] out {tuple(out.shape)} traj rows {traj.shape[0]} oracle rel-L2 {MG.rel_l2(res.out, out):.3e}")
    np.savez_compressed(os.path.join(MG.GOLD, FULL + ".npz"), out=out.numpy(), y0=traj[0].numpy(),
                        traj_1=traj[1].numpy())


if __name__ == "__main__":
    main()
