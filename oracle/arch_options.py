"""CPU ORACLE for the backbone options no shipped config turns on — TEST INFRASTRUCTURE ONLY (same rules as
oracle/f5_oracle.py, whose functions it reuses unchanged).

The reference's constructors build three switches that are off in every configs/*.yaml:

* ``qk_norm="rms_norm"`` (DiT and UNetT): per-head RMSNorm(dim_head, eps 1e-6, learned gain) of q and k, before RoPE
  (model/modules.py:286-305, 402-409, 492-496);
* ``long_skip_connection`` (DiT): ``x = Linear(2D -> D, bias=False)(cat(x after the last block, x after the input
  embedding))`` before norm_out (backbones/dit.py:228, 354-365);
* ``text_embedding_average_upsampling`` (DiT): after the text blocks, each sample's valid text rows are spread evenly
  over its audio length (backbones/dit.py:41-43, 55-84, 131-137).

They are read from the ``qk_norm`` / ``long_skip_connection`` / ``text_embedding_average_upsampling`` fields of
synthdata.ArchConfig.  With all three off, every function here computes exactly what its oracle/f5_oracle.py
counterpart does.  ``sample`` is oracle/ode_midpoint.sample (euler or midpoint) over these backbone functions.
oracle/make_golden_arch_options.py pins all of it against the unmodified reference.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import f5_oracle as O
from oracle import ode_midpoint as OM


def rms_norm(x, w, eps=1e-6):
    """modules.py:286-305 RMSNorm over the last axis, fp32: x * rsqrt(mean(x^2) + eps) * w"""
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w


def average_upsample(h, text_mask, audio_len):
    """backbones/dit.py:55-84: sample b's valid text rows (text_mask) spread evenly over its first audio_len[b] rows,
    token j repeated audio_len // T times plus once more for the last audio_len % T tokens; other rows 0."""
    out = torch.zeros_like(h)
    for b in range(h.shape[0]):
        rows = h[b, text_mask[b]]
        T, A = rows.shape[0], int(audio_len[b])
        if T == 0 or A <= 0:
            continue
        base, rem = divmod(A, T)
        reps = torch.full((T,), base, dtype=torch.long)
        reps[T - rem:] += 1
        out[b, :A] = rows.repeat_interleave(reps, dim=0)[:A]
    return out


def text_embedding_dit(sd, cfg, text, seq_len, drop_text: bool):
    """backbones/dit.py:86-139: oracle/f5_oracle.text_embedding_dit, then average upsampling when it is on.  The mask
    is the cond row's (text == 0 after the +1 shift, the crop to N and the per-sample length), taken before drop_text."""
    h = O.text_embedding_dit(sd, cfg, text, seq_len, drop_text)
    if not cfg.text_embedding_average_upsampling:
        return h
    per_sample = torch.is_tensor(seq_len)
    n = h.shape[1]
    ids = F.pad((text + 1)[:, :n], (0, max(0, n - text.shape[1])), value=0)
    if per_sample:
        ids = ids.masked_fill(~(torch.arange(n)[None, :] < seq_len.long()[:, None]), 0)
    audio = seq_len.long() if per_sample else torch.full((h.shape[0],), n, dtype=torch.long)
    return average_upsample(h, ids != 0, audio)


def attention(sd, cfg, p: str, x, mask, ang):
    """modules.py:471-556 AttnProcessor (torch backend) with qk_norm.  x [Be, N, D]"""
    B, N, _ = x.shape
    H, dh = cfg.heads, cfg.dim_head
    q = O._linear(sd, p + "to_q", x).view(B, N, H, dh).transpose(1, 2)
    k = O._linear(sd, p + "to_k", x).view(B, N, H, dh).transpose(1, 2)
    v = O._linear(sd, p + "to_v", x).view(B, N, H, dh).transpose(1, 2)
    if cfg.qk_norm == "rms_norm":
        q = rms_norm(q, sd[p + "q_norm.weight"])
        k = rms_norm(k, sd[p + "k_norm.weight"])
    pn = H if cfg.pe_attn_head is None else cfg.pe_attn_head
    q = torch.cat((O.apply_rope(q[:, :pn], ang), q[:, pn:]), dim=1)
    k = torch.cat((O.apply_rope(k[:, :pn], ang), k[:, pn:]), dim=1)
    key_mask = None
    if cfg.attn_mask_enabled and mask is not None:
        key_mask = mask[:, None, None, :].expand(B, H, N, N)
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=key_mask, dropout_p=0.0, is_causal=False)
    o = O._linear(sd, p + "to_out.0", o.transpose(1, 2).reshape(B, N, H * dh))
    if mask is not None:
        o = o.masked_fill(~mask[..., None], 0.0)
    return o


def dit_block(sd, cfg, i: int, x, t_emb, mask, ang):
    """modules.py:743-757 DiTBlock.forward + AdaLayerNorm 312-326"""
    p = f"transformer.transformer_blocks.{i}."
    mod = O._linear(sd, p + "attn_norm.linear", F.silu(t_emb))
    shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = mod.chunk(6, dim=1)
    h = O._ln_noaffine(x) * (1 + scale_msa[:, None]) + shift_msa[:, None]
    x = x + gate_msa[:, None] * attention(sd, cfg, p + "attn.", h, mask, ang)
    h = O._ln_noaffine(x) * (1 + scale_mlp[:, None]) + shift_mlp[:, None]
    return x + gate_mlp[:, None] * O.feed_forward(sd, p + "ff.", h)


def dit_forward(sd, cfg, x, cond, text_emb, time, mask, cfg_infer: bool):
    """backbones/dit.py:319-370 with qk_norm and the long skip connection"""
    B, N, _ = x.shape
    t = time.reshape(-1).expand(B) if time.ndim == 0 or time.numel() == 1 else time
    t_emb = O.timestep_embedding(sd, t)
    if cfg_infer:
        h = O._pack_cfg(sd, cfg, x, cond, text_emb[0], text_emb[1], mask)
        t_emb = torch.cat((t_emb, t_emb), dim=0)
        mask = None if mask is None else torch.cat((mask, mask), dim=0)
    else:
        h = O.input_embedding(sd, x, cond, text_emb[0], False, mask)
    ang = O.rope_angles(N, cfg.dim_head, dtype=h.dtype)
    residual = h
    for i in range(cfg.depth):
        h = dit_block(sd, cfg, i, h, t_emb, mask, ang)
    if cfg.long_skip_connection:
        h = F.linear(torch.cat((h, residual), dim=-1), sd["transformer.long_skip_connection.weight"])
    mod = O._linear(sd, "transformer.norm_out.linear", F.silu(t_emb))
    scale, shift = mod.chunk(2, dim=1)
    h = O._ln_noaffine(h) * (1 + scale)[:, None] + shift[:, None]
    return O._linear(sd, "transformer.proj_out", h)


def unett_forward(sd, cfg, x, cond, text_emb, time, mask, cfg_infer: bool):
    """backbones/unett.py:244-307 with qk_norm"""
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
            h = F.linear(torch.cat((h, skips.pop()), dim=-1), sd[p + "0.weight"])
        h = attention(sd, cfg, p + "2.", O.x_rmsnorm(h, sd[p + "1.g"]), mask, ang) + h
        h = O.feed_forward(sd, p + "4.", O.x_rmsnorm(h, sd[p + "3.g"])) + h
    h = O.x_rmsnorm(h, sd["transformer.norm_out.g"])[:, 1:]
    return O._linear(sd, "transformer.proj_out", h)


@torch.no_grad()
def sample(sd, cfg, cond, text, duration, *, lens=None, steps=32, cfg_strength=1.0, sway_sampling_coef=None, seed=None,
           max_duration=65536, use_epss=True, y0=None, method="euler") -> O.SampleResult:
    """model/cfm.py:83-229 as oracle/ode_midpoint.sample (cond: raw wave [B, nw] or mel [B, n, mel]), over the backbone
    functions of this module."""
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
    if cfg.backbone == "DiT":
        seq_len = N if mask is None else mask.sum(dim=1)
        te = (text_embedding_dit(sd, cfg, text, seq_len, False), text_embedding_dit(sd, cfg, text, seq_len, True))
        fwd = dit_forward
    else:
        te = (O.text_embedding_unett(sd, cfg, text, N, False), O.text_embedding_unett(sd, cfg, text, N, True))
        fwd = unett_forward

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
    traj = OM.odeint(fn, y0, t, method=method)
    out = torch.where(cond_mask, cond, traj[-1])
    return O.SampleResult(out=out, trajectory=traj, y0=y0, t=t,
                          extras={"text_cond": te[0], "text_uncond": te[1], "mask": mask, "step_cond": step_cond})
