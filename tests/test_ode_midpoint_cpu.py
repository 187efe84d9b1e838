"""CPU: the midpoint ODE solver (odeint_kwargs=dict(method="midpoint")) of the oracle (oracle/ode_midpoint.py) against
fixtures written by the unmodified reference's CFM.sample (oracle/make_golden_midpoint.py), a closed form and the Euler
oracle, and the host-side surface of the sampler (constructor check, C-ABI argument block)."""
import os

import numpy as np
import pytest
import torch

from oracle import f5_oracle as O
from oracle import ode_midpoint as OM

TOL = 1e-5  # fp32 vs fp32 on the same host, as in test_oracle_vs_golden.py


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _load(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    return {k: torch.from_numpy(z[k]) for k in ("out", "y0", "traj_1")}


def test_oracle_midpoint_vs_reference_tiny_dit_varlen(golden_dir):
    from oracle import make_golden_midpoint as MM
    from oracle import make_golden_reference_checks as MR

    cfg, sd, cond, text, dur, kw = MR.tiny_dit_varlen_case()
    want = _load(golden_dir, MM.TINY)
    res = OM.sample(sd, cfg, cond, text, dur, method="midpoint", **kw)
    assert torch.equal(res.y0, want["y0"])
    assert res.trajectory.shape[0] == kw["steps"] + 1
    assert _rel(res.trajectory[1], want["traj_1"]) <= TOL
    assert _rel(res.out, want["out"]) <= TOL
    # the fixture is not the Euler result under another name
    euler = O.sample(sd, cfg, cond, text, dur, **kw)
    assert _rel(euler.out, want["out"]) > 100 * TOL


def test_midpoint_oracle_euler_equals_oracle():
    """oracle/ode_midpoint.sample restates oracle/f5_oracle.sample around its own odeint: with method="euler" the two
    agree bit for bit (var-len DiT and UNetT, CFG and no CFG)."""
    from oracle import make_golden as MG
    from oracle import make_golden_reference_checks as MR

    cfg, sd, cond, text, dur, kw = MR.tiny_dit_varlen_case()
    a, b = O.sample(sd, cfg, cond, text, dur, **kw), OM.sample(sd, cfg, cond, text, dur, method="euler", **kw)
    assert torch.equal(a.trajectory, b.trajectory) and torch.equal(a.out, b.out)
    cfg = MG.tiny_unett()
    sd = O.synthetic_state_dict(cfg, seed=3)
    kw = dict(lens=torch.tensor([20, 12]), steps=2, cfg_strength=0.0, sway_sampling_coef=None, seed=2)
    a, b = O.sample(sd, cfg, cond, text, dur, **kw), OM.sample(sd, cfg, cond, text, dur, method="euler", **kw)
    assert torch.equal(a.trajectory, b.trajectory) and torch.equal(a.out, b.out)


@pytest.mark.slow
def test_oracle_midpoint_vs_reference_f5base_b2_varlen(golden_dir):
    from oracle import make_golden_midpoint as MM

    cfg, wseed, cond, text, dur, lens, kw = MM.full_width_case()
    want = _load(golden_dir, MM.FULL)
    res = OM.sample(O.synthetic_state_dict(cfg, seed=wseed), cfg, cond, text, dur, lens=lens, method="midpoint", **kw)
    assert torch.equal(res.y0, want["y0"])
    assert _rel(res.trajectory[1], want["traj_1"]) <= TOL
    assert _rel(res.out, want["out"]) <= TOL


def test_odeint_midpoint_linear_ode_closed_form():
    """dy/dt = a*y: one midpoint step multiplies y by 1 + a*dt + (a*dt)^2/2 exactly (in exact arithmetic)."""
    a = -1.7
    t = torch.tensor([0.0, 0.05, 0.2, 0.23, 0.6, 1.0], dtype=torch.float32)  # non-uniform grid
    y0 = torch.randn(3, 4, generator=torch.Generator().manual_seed(0))
    calls = []

    def f(tt, y):
        calls.append(float(tt))
        return a * y

    traj = OM.odeint(f, y0, t, method="midpoint")
    assert traj.shape == (t.shape[0], 3, 4)
    assert len(calls) == 2 * (t.shape[0] - 1)
    want = y0.double()
    for k in range(t.shape[0] - 1):
        dt = float(t[k + 1] - t[k])
        assert calls[2 * k] == float(t[k])
        assert calls[2 * k + 1] == pytest.approx(float(t[k]) + 0.5 * dt, abs=1e-7)
        want = want * (1 + a * dt + (a * dt) ** 2 / 2)
        assert torch.allclose(traj[k + 1].double(), want, rtol=1e-6, atol=1e-7)


def test_cfm_accepts_euler_and_midpoint_only():
    import f5_tts_b200 as F5

    def make(**kw):
        return F5.CFM(transformer=F5.DiT(dim=1024, depth=1, heads=16, ff_mult=2, text_dim=512, conv_layers=1,
                                         text_num_embeds=10), **kw)

    for m in ("rk4", "dopri5", "heun2"):
        with pytest.raises(NotImplementedError, match="midpoint") as ei:
            make(odeint_kwargs=dict(method=m))
        assert "euler" in str(ei.value)
    assert make(odeint_kwargs=dict(method="midpoint")).odeint_kwargs["method"] == "midpoint"
    assert make().odeint_kwargs["method"] == "euler"


def test_sample_args_ends_in_method():
    from f5_tts_b200 import _lib

    name, ctype = _lib.SampleArgs._fields_[-1]
    assert name == "method" and ctype is _lib.C.c_int
    assert _lib.SampleArgs().method == 0  # a zeroed argument block keeps Euler
    assert _lib.ODE_METHODS == {"euler": 0, "midpoint": 1}


def test_nfe_counts_backbone_evaluations():
    """Host-only: the Python wrapper sizes the workspace and the FLOP count for 2 * steps evaluations with midpoint."""
    from f5_tts_b200 import model as M

    assert M._nfe(16, "euler") == 16 and M._nfe(16, "midpoint") == 32
    with pytest.raises(NotImplementedError):
        M._nfe(4, "rk4")
