"""CPU ORACLE of the MMDiT backbone — TEST INFRASTRUCTURE ONLY (same rules as oracle/f5_oracle.py, whose functions it
reuses unchanged).

backbones/mmdit.py builds a backbone with two residual streams, audio ``x`` [B, N, D] and text ``c`` [B, nt, D] (the
text is not padded to N), and one joint attention per block over the keys [audio | text] (MMDiTBlock and
JointAttnProcessor, model/modules.py:563-705, 763-846).  The last block (context_pre_only) normalises the text with an
AdaLayerNorm_Final and discards its text output.  ``sample`` is oracle/ode_midpoint.sample's CFM.sample (euler or
midpoint) over ``mmdit_forward``.  oracle/make_golden_mmdit.py pins all of it against the unmodified reference.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import arch_options as OA
from oracle import f5_oracle as O
from oracle import ode_midpoint as OM

P = "transformer."


def text_embedding(sd, cfg, text, drop_text: bool):
    """backbones/mmdit.py:31-63.  text int[B, nt] (pad -1) -> [B, nt, D]"""
    ids = text + 1
    pad = ids == 0
    if drop_text:
        ids = torch.zeros_like(ids)
    h = sd[P + "text_embed.text_embed.weight"][ids]
    pos = torch.arange(text.shape[1]).clamp(max=1023)  # get_pos_embed_indices, modules.py:221-230
    h = h + O.abs_pos_table(cfg.dim, 1024, dtype=h.dtype)[pos]
    if cfg.text_mask_padding:
        h = h.masked_fill(pad[..., None], 0.0)
    return h


def audio_embedding(sd, x, cond, drop_audio_cond: bool):
    """backbones/mmdit.py:67-78: Linear(2 mel -> D), then ConvPositionEmbedding WITHOUT a mask"""
    if drop_audio_cond:
        cond = torch.zeros_like(cond)
    h = O._linear(sd, P + "audio_embed.linear", torch.cat((x, cond), dim=-1))
    return O.conv_position_embedding(sd, h, None, p=P + "audio_embed.conv_pos_embed.") + h


def _heads(sd, cfg, p, x, names, norms):
    B, n, _ = x.shape
    q, k, v = (O._linear(sd, p + nm, x).view(B, n, cfg.heads, cfg.dim_head).transpose(1, 2) for nm in names)
    if cfg.qk_norm == "rms_norm":
        q, k = OA.rms_norm(q, sd[p + norms[0]]), OA.rms_norm(k, sd[p + norms[1]])
    ang = O.rope_angles(n, cfg.dim_head, dtype=x.dtype)  # every head, positions 0.. per stream
    return O.apply_rope(q, ang), O.apply_rope(k, ang), v


def joint_attention(sd, cfg, p, x, c, mask, c_mask, last: bool):
    """modules.py:563-705 JointAttnProcessor (torch backend) -> (x_out, c_out or None)"""
    B, N, _ = x.shape
    q, k, v = _heads(sd, cfg, p, x, ("to_q", "to_k", "to_v"), ("q_norm.weight", "k_norm.weight"))
    qc, kc, vc = _heads(sd, cfg, p, c, ("to_q_c", "to_k_c", "to_v_c"), ("c_q_norm.weight", "c_k_norm.weight"))
    q, k, v = torch.cat((q, qc), dim=2), torch.cat((k, kc), dim=2), torch.cat((v, vc), dim=2)
    key_mask = None
    if cfg.attn_mask_enabled and mask is not None:
        key_mask = torch.cat((mask, c_mask), dim=1)[:, None, None, :].expand(B, cfg.heads, q.shape[2], k.shape[2])
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=key_mask, dropout_p=0.0, is_causal=False)
    o = o.transpose(1, 2).reshape(B, -1, cfg.heads * cfg.dim_head)
    xo = O._linear(sd, p + "to_out.0", o[:, :N])
    if mask is not None:
        xo = xo.masked_fill(~mask[..., None], 0.0)
    if last:
        return xo, None
    co = O._linear(sd, p + "to_out_c", o[:, N:]).masked_fill(~c_mask[..., None], 0.0)
    return xo, co


def mmdit_block(sd, cfg, i: int, x, c, t_emb, mask, c_mask):
    """modules.py:806-846 MMDiTBlock.forward"""
    p = f"{P}transformer_blocks.{i}."
    last = i == cfg.depth - 1
    st = F.silu(t_emb)
    mc = O._linear(sd, p + "attn_norm_c.linear", st)
    if last:  # AdaLayerNorm_Final: (scale, shift)
        scale, shift = mc.chunk(2, dim=1)
        nc = O._ln_noaffine(c) * (1 + scale[:, None]) + shift[:, None]
    else:
        c_shift_msa, c_scale_msa, c_gate_msa, c_shift_mlp, c_scale_mlp, c_gate_mlp = mc.chunk(6, dim=1)
        nc = O._ln_noaffine(c) * (1 + c_scale_msa[:, None]) + c_shift_msa[:, None]
    shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = O._linear(sd, p + "attn_norm_x.linear",
                                                                                st).chunk(6, dim=1)
    nx = O._ln_noaffine(x) * (1 + scale_msa[:, None]) + shift_msa[:, None]
    xo, co = joint_attention(sd, cfg, p + "attn.", nx, nc, mask, c_mask, last)
    if not last:
        c = c + c_gate_msa[:, None] * co
        h = O._ln_noaffine(c) * (1 + c_scale_mlp[:, None]) + c_shift_mlp[:, None]
        c = c + c_gate_mlp[:, None] * O.feed_forward(sd, p + "ff_c.", h)
    x = x + gate_msa[:, None] * xo
    h = O._ln_noaffine(x) * (1 + scale_mlp[:, None]) + shift_mlp[:, None]
    return x + gate_mlp[:, None] * O.feed_forward(sd, p + "ff_x.", h), c


def mmdit_forward(sd, cfg, x, cond, text, text_emb, time, mask, cfg_infer: bool):
    """backbones/mmdit.py:198-246.  text_emb = (cond_variant, uncond_variant) text embeddings"""
    B = x.shape[0]
    t = time.reshape(-1).expand(B) if time.ndim == 0 or time.numel() == 1 else time
    t_emb = O.timestep_embedding(sd, t)
    c_mask = text != -1
    if cfg_infer:
        h = torch.cat((audio_embedding(sd, x, cond, False), audio_embedding(sd, x, cond, True)), dim=0)
        c = torch.cat(text_emb, dim=0)
        t_emb = torch.cat((t_emb, t_emb), dim=0)
        mask = None if mask is None else torch.cat((mask, mask), dim=0)
        c_mask = torch.cat((c_mask, c_mask), dim=0)
    else:
        h, c = audio_embedding(sd, x, cond, False), text_emb[0]
    for i in range(cfg.depth):
        h, c = mmdit_block(sd, cfg, i, h, c, t_emb, mask, c_mask)
    scale, shift = O._linear(sd, P + "norm_out.linear", F.silu(t_emb)).chunk(2, dim=1)
    h = O._ln_noaffine(h) * (1 + scale[:, None]) + shift[:, None]
    return O._linear(sd, P + "proj_out", h)


@torch.no_grad()
def sample(sd, cfg, cond, text, duration, *, lens=None, steps=32, cfg_strength=1.0, sway_sampling_coef=None, seed=None,
           max_duration=65536, use_epss=True, y0=None, method="euler") -> O.SampleResult:
    """model/cfm.py:83-229 over an MMDiT (cond: mel [B, n, mel] or raw wave [B, nw])."""
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
    te = (text_embedding(sd, cfg, text, False), text_embedding(sd, cfg, text, True))

    def fn(t, x):
        if cfg_strength < 1e-5:
            return mmdit_forward(sd, cfg, x, step_cond, text, te, t, mask, False)
        pred, null = mmdit_forward(sd, cfg, x, step_cond, text, te, t, mask, True).chunk(2, dim=0)
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
