"""CPU ORACLE for UNetT's ``skip_connect_type`` — TEST INFRASTRUCTURE ONLY (same rules as oracle/f5_oracle.py and
oracle/arch_options.py, whose functions it reuses unchanged).

The reference's UNetT (backbones/unett.py:127, 286-297) takes ``skip_connect_type`` in ("add", "concat", "none"): each
later-half layer pops the x its mirror first-half layer pushed and, before attn_norm, runs
``x = skip_proj(cat(x, skip))`` ("concat", the default and every shipped config), ``x = x + skip`` ("add") or nothing
("none").  It is read from synthdata.ArchConfig.skip_connect_type.  With "concat", ``unett_forward`` computes exactly
what oracle/arch_options.unett_forward does, and the other options (qk_norm, dim_head, attn_mask_enabled) are those of
oracle/arch_options.attention.  ``sample`` is oracle/arch_options.sample for a UNetT over this module's forward.
oracle/make_golden_unett_skip.py pins "add" and "none" against the unmodified reference.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import arch_options as OA
from oracle import f5_oracle as O
from oracle import ode_midpoint as OM


def unett_forward(sd, cfg, x, cond, text_emb, time, mask, cfg_infer: bool):
    """backbones/unett.py:244-307 with qk_norm and skip_connect_type"""
    B, N, _ = x.shape
    t = time.reshape(-1).expand(B) if time.ndim == 0 or time.numel() == 1 else time
    t_emb = O.timestep_embedding(sd, t)
    if cfg_infer:
        h = O._pack_cfg(sd, cfg, x, cond, text_emb[0], text_emb[1], None)
        t_emb = torch.cat((t_emb, t_emb), dim=0)
        mask = None if mask is None else torch.cat((mask, mask), dim=0)
    else:
        h = O.input_embedding(sd, x, cond, text_emb[0], False, None)
    h = torch.cat((t_emb[:, None], h), dim=1)
    if mask is not None:
        mask = F.pad(mask, (1, 0), value=True)
    ang = O.rope_angles(N + 1, cfg.dim_head, dtype=h.dtype)
    skips = []
    half = cfg.depth // 2
    for i in range(cfg.depth):
        p = f"transformer.layers.{i}."
        if i < half:
            skips.append(h)
        else:
            skip = skips.pop()
            if cfg.skip_connect_type == "concat":
                h = F.linear(torch.cat((h, skip), dim=-1), sd[p + "0.weight"])
            elif cfg.skip_connect_type == "add":
                h = h + skip
        h = OA.attention(sd, cfg, p + "2.", O.x_rmsnorm(h, sd[p + "1.g"]), mask, ang) + h
        h = O.feed_forward(sd, p + "4.", O.x_rmsnorm(h, sd[p + "3.g"])) + h
    h = O.x_rmsnorm(h, sd["transformer.norm_out.g"])[:, 1:]
    return O._linear(sd, "transformer.proj_out", h)


@torch.no_grad()
def sample(sd, cfg, cond, text, duration, *, lens=None, steps=32, cfg_strength=1.0, sway_sampling_coef=None, seed=None,
           max_duration=65536, use_epss=True, y0=None, method="euler") -> O.SampleResult:
    """model/cfm.py:83-229 for a UNetT (cond: raw wave [B, nw] or mel [B, n, mel]), as oracle/arch_options.sample, over
    this module's unett_forward."""
    assert cfg.backbone == "UNetT", cfg.backbone
    if cond.ndim == 2:
        cond = O.mel_spectrogram(cond).permute(0, 2, 1)
    cond = cond.float()
    B, n_cond = cond.shape[:2]
    if lens is None:
        lens = torch.full((B,), n_cond, dtype=torch.long)
    cond_mask = O.lens_to_mask(lens)
    if isinstance(duration, int):
        duration = torch.full((B,), duration, dtype=torch.long)
    duration = torch.maximum(torch.maximum((text != -1).sum(dim=-1), lens) + 1, duration).clamp(max=max_duration)
    N = int(duration.amax())
    cond = F.pad(cond, (0, 0, 0, N - n_cond), value=0.0)
    cond_mask = F.pad(cond_mask, (0, N - cond_mask.shape[-1]), value=False)[..., None]
    step_cond = torch.where(cond_mask, cond, torch.zeros_like(cond))
    mask = O.lens_to_mask(duration) if B > 1 else None
    te = (O.text_embedding_unett(sd, cfg, text, N, False), O.text_embedding_unett(sd, cfg, text, N, True))

    def fn(t, x):
        if cfg_strength < 1e-5:
            return unett_forward(sd, cfg, x, step_cond, te, t, mask, False)
        pred, null = unett_forward(sd, cfg, x, step_cond, te, t, mask, True).chunk(2, dim=0)
        return pred + (pred - null) * cfg_strength

    if y0 is None:
        rows = []
        for dur in duration.tolist():
            if seed is not None:
                torch.manual_seed(seed)
            rows.append(torch.randn(dur, cfg.mel_dim, dtype=torch.float32))
        y0 = torch.nn.utils.rnn.pad_sequence(rows, padding_value=0, batch_first=True)
    t = O.time_grid(steps, sway_sampling_coef, use_epss)
    traj = OM.odeint(fn, y0, t, method=method)
    out = torch.where(cond_mask, cond, traj[-1])
    return O.SampleResult(out=out, trajectory=traj, y0=y0, t=t,
                          extras={"text_cond": te[0], "text_uncond": te[1], "mask": mask, "step_cond": step_cond})
