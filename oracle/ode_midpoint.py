"""CPU ORACLE for the midpoint ODE solver — TEST INFRASTRUCTURE ONLY (same rules as oracle/f5_oracle.py).

The reference passes ``odeint_kwargs`` straight to ``torchdiffeq.odeint`` (cfm.py:39-43, 218) and names two methods,
``euler`` and ``midpoint`` (cfm.py:42, infer/speech_edit.py:40).  torchdiffeq is not installed and the reference does
not pin its version, so both fixed-grid methods are restated here from its published algorithm (**parity unpinned**,
like the Euler step of oracle/f5_oracle.py and oracle/ref_shims.py).  Per grid interval (t0, t1), dt = t1 - t0:

    euler:    y1 = y0 + dt * f(t0, y0)
    midpoint: half_dt = 0.5 * dt;  y_mid = y0 + f(t0, y0) * half_dt;  y1 = y0 + dt * f(t0 + half_dt, y_mid)

Both return y at the grid points only (t.shape[0] rows).

* ``odeint`` is the restatement.  oracle/make_golden_midpoint.py registers it as the ``torchdiffeq`` stand-in before
  the unmodified reference is imported (cfm.py binds ``odeint`` at import time), so the reference's own
  ``CFM.sample`` runs the midpoint method through it.
* ``sample`` is oracle/f5_oracle.sample (model/cfm.py:83-229) with the ODE loop delegated to ``odeint``; it reuses
  every backbone function of oracle/f5_oracle.py unchanged.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import f5_oracle as O

METHODS = ("euler", "midpoint")


def odeint(func, y0, t, *, method="euler", **_unused):
    if method not in METHODS:
        raise NotImplementedError(f"odeint method {method!r}: only the fixed-grid 'euler' and 'midpoint' are restated")
    ys = [y0]
    y = y0
    for k in range(t.shape[0] - 1):
        t0, t1 = t[k], t[k + 1]
        dt = t1 - t0
        if method == "midpoint":
            half_dt = 0.5 * dt
            y_mid = y + func(t0, y) * half_dt
            y = y + dt * func(t0 + half_dt, y_mid)
        else:
            y = y + dt * func(t0, y)
        ys.append(y)
    return torch.stack(ys, dim=0)


@torch.no_grad()
def sample(sd, cfg: O.ArchConfig, cond, text, duration, *, lens=None, steps=32, cfg_strength=1.0,
           sway_sampling_coef=None, seed=None, max_duration=65536, use_epss=True, no_ref_audio=False,
           edit_mask=None, y0=None, method="midpoint") -> O.SampleResult:
    """oracle/f5_oracle.sample with ``odeint_kwargs=dict(method=method)``; same arguments and result."""
    if cond.ndim == 2:
        cond = O.mel_spectrogram(cond).permute(0, 2, 1)
    cond = cond.float()
    B, n_cond = cond.shape[:2]
    if lens is None:
        lens = torch.full((B,), n_cond, dtype=torch.long)
    cond_mask = O.lens_to_mask(lens)
    if edit_mask is not None:
        cond_mask = cond_mask & edit_mask
    if isinstance(duration, int):
        duration = torch.full((B,), duration, dtype=torch.long)
    duration = torch.maximum(torch.maximum((text != -1).sum(dim=-1), lens) + 1, duration).clamp(max=max_duration)
    N = int(duration.amax())
    cond = F.pad(cond, (0, 0, 0, N - n_cond), value=0.0)
    if no_ref_audio:
        cond = torch.zeros_like(cond)
    cond_mask = F.pad(cond_mask, (0, N - cond_mask.shape[-1]), value=False)[..., None]
    step_cond = torch.where(cond_mask, cond, torch.zeros_like(cond))
    mask = O.lens_to_mask(duration) if B > 1 else None

    if cfg.backbone == "DiT":
        seq_len = N if mask is None else mask.sum(dim=1)
        te = (O.text_embedding_dit(sd, cfg, text, seq_len, False), O.text_embedding_dit(sd, cfg, text, seq_len, True))
        fwd = O.dit_forward
    else:
        te = (O.text_embedding_unett(sd, cfg, text, N, False), O.text_embedding_unett(sd, cfg, text, N, True))
        fwd = O.unett_forward

    def fn(t, x):
        if cfg_strength < 1e-5:
            return fwd(sd, cfg, x, step_cond, te, t, mask, False)
        pred, null = fwd(sd, cfg, x, step_cond, te, t, mask, True).chunk(2, dim=0)
        return pred + (pred - null) * cfg_strength

    if y0 is None:
        rows = []
        for dur in duration.tolist():
            if seed is not None:
                torch.manual_seed(seed)
            rows.append(torch.randn(dur, cfg.mel_dim, dtype=torch.float32))
        y0 = torch.nn.utils.rnn.pad_sequence(rows, padding_value=0, batch_first=True)
    t = O.time_grid(steps, sway_sampling_coef, use_epss)
    traj = odeint(fn, y0, t, method=method)
    out = torch.where(cond_mask, cond, traj[-1])
    return O.SampleResult(out=out, trajectory=traj, y0=y0, t=t,
                          extras={"text_cond": te[0], "text_uncond": te[1], "mask": mask, "step_cond": step_cond})
