"""CPU ORACLE — TEST INFRASTRUCTURE ONLY.  Not the product, not a fallback.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this file.  The product package
(``f5_tts_b200``) never does, and raises if its CUDA library is missing.

What it is: a plain PyTorch **fp32, CPU** functional restatement of the
reference's ODE-sampling hot path (SURVEY.md §8a rows a1-a18), operating on a
flat ``state_dict`` with the *released checkpoint key names*
(SURVEY.md §8b "Checkpoint layout").  Each function cites the reference
file:line it follows (paths relative to /root/reference/src/f5_tts).

How it is pinned: ``oracle/make_golden.py`` runs the UNMODIFIED reference
modules (imported through ``oracle/ref_shims.py``) on seeded synthetic weights
and inputs and commits their outputs under ``tests/golden/``;
``tests/test_oracle_vs_golden.py`` checks this restatement against those
vectors (and against the live reference when /root/reference is present).
The reference itself has no tests or golden vectors for this path
(SURVEY.md §4).  Pieces that live in third-party packages absent from the
reference tree are restated from their published algorithm and are
**parity unpinned**: torchdiffeq Euler (cfm.py:218), x_transformers rotary /
RMSNorm (modules.py:499-509, unett.py:154), vocos.Vocos.decode
(infer/utils_infer.py:118-129,511).  The mel front-end is pinned against
torchaudio.transforms.MelSpectrogram, ISTFT against torch.istft.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Optional

import torch
import torch.nn.functional as F


# configuration presets + synthetic weights live in the neutral module `synthdata` (shared with bench.py / smoke());
# re-exported here so tests keep a single import.
from synthdata import (ArchConfig, e2tts_base, f5tts_base, f5tts_v1_base, state_dict_spec, synthetic_state_dict,  # noqa: E402,F401
                       synthetic_vocos_state_dict, vocos_state_dict_spec)


# ---------------------------------------------------------------------------
# mel front-end (a7): model/modules.py:80-109 -> torchaudio MelSpectrogram
# ---------------------------------------------------------------------------
def hz_to_mel_htk(f):
    return 2595.0 * math.log10(1.0 + f / 700.0)


def mel_filterbank(n_freqs=513, f_min=0.0, f_max=12000.0, n_mels=100, sample_rate=24000) -> torch.Tensor:
    """HTK-scale triangular filters, norm=None — torchaudio.functional.melscale_fbanks semantics. [n_freqs, n_mels]"""
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs)
    m_pts = torch.linspace(hz_to_mel_htk(f_min), hz_to_mel_htk(f_max), n_mels + 2)
    f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    down = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    return torch.clamp(torch.min(down, up), min=0.0)


def mel_spectrogram(wav: torch.Tensor, n_fft=1024, hop=256, win=1024, n_mels=100, sr=24000) -> torch.Tensor:
    """wav [B, nw] f32 -> log-mel [B, n_mels, 1 + nw//hop]   (modules.py:80-109; SURVEY.md §9.2)"""
    assert wav.ndim == 2 and win == n_fft
    xp = F.pad(wav.unsqueeze(1), (n_fft // 2, n_fft // 2), mode="reflect").squeeze(1)
    frames = xp.unfold(-1, n_fft, hop)  # [B, T, n_fft]
    window = torch.hann_window(win, periodic=True, dtype=wav.dtype)
    spec = torch.fft.rfft(frames * window, dim=-1).abs()  # power=1 magnitude
    fb = mel_filterbank(n_fft // 2 + 1, 0.0, sr / 2, n_mels, sr).to(wav.dtype)
    mel = spec @ fb  # [B, T, n_mels]
    return mel.clamp(min=1e-5).log().transpose(1, 2)


# ---------------------------------------------------------------------------
# small ops
# ---------------------------------------------------------------------------
def _linear(sd, prefix, x):
    return F.linear(x, sd[prefix + ".weight"], sd.get(prefix + ".bias"))


def _ln_noaffine(x, eps=1e-6):
    return F.layer_norm(x, (x.shape[-1],), eps=eps)


def sinus_time_features(t: torch.Tensor, dim=256, scale=1000.0, dtype=torch.float32) -> torch.Tensor:
    """modules.py:157-169 — [B] -> [B, dim] = cat(sin, cos), computed in `dtype`"""
    half = dim // 2
    k = math.log(10000.0) / (half - 1)
    freqs = torch.exp(torch.arange(half, dtype=dtype) * -k)
    arg = scale * t.to(dtype)[:, None] * freqs[None, :]
    return torch.cat((arg.sin(), arg.cos()), dim=-1)


def timestep_embedding(sd, t: torch.Tensor, p="transformer.time_embed.") -> torch.Tensor:
    """modules.py:852-862, in the dtype of the time MLP's weights"""
    h = sinus_time_features(t, dtype=sd[p + "time_mlp.0.weight"].dtype)
    h = _linear(sd, p + "time_mlp.0", h)
    return _linear(sd, p + "time_mlp.2", F.silu(h))


def abs_pos_table(dim: int, end: int, theta=10000.0, dtype=torch.float32) -> torch.Tensor:
    """modules.py:207-218 precompute_freqs_cis — [end, dim] = cat(cos, sin), computed in `dtype`"""
    freqs = 1.0 / (theta ** (torch.arange(0, dim, 2)[: dim // 2].to(dtype) / dim))
    ang = torch.outer(torch.arange(end).to(dtype), freqs)
    return torch.cat((ang.cos(), ang.sin()), dim=-1)


def convnext_v2_block(sd, p, x):
    """modules.py:252-280 (+ GRN 236-245).  x [B, N, C]"""
    h = F.conv1d(x.transpose(1, 2), sd[p + "dwconv.weight"], sd[p + "dwconv.bias"], padding=3,
                 groups=x.shape[-1]).transpose(1, 2)
    h = F.layer_norm(h, (h.shape[-1],), sd[p + "norm.weight"], sd[p + "norm.bias"], eps=1e-6)
    h = F.gelu(_linear(sd, p + "pwconv1", h))
    gx = torch.linalg.vector_norm(h, ord=2, dim=1, keepdim=True)  # over the SEQUENCE axis (incl. padded rows)
    nx = gx / (gx.mean(dim=-1, keepdim=True) + 1e-6)
    h = sd[p + "grn.gamma"] * (h * nx) + sd[p + "grn.beta"] + h
    return x + _linear(sd, p + "pwconv2", h)


def text_embedding_dit(sd, cfg: ArchConfig, text, seq_len, drop_text: bool):
    """backbones/dit.py:86-139.  text int[B, nt] (pad -1); seq_len int or int[B] -> [B, N, Td]"""
    p = "transformer.text_embed."
    text = text + 1
    per_sample = torch.is_tensor(seq_len)
    n = int(seq_len.max()) if per_sample else int(seq_len)
    text = text[:, :n]
    text = F.pad(text, (0, n - text.shape[1]), value=0)
    valid = None
    if per_sample:
        valid = torch.arange(n)[None, :] < seq_len.long()[:, None]
        text = text.masked_fill(~valid, 0)
    filler = text == 0  # taken BEFORE drop_text zeroing (dit.py:103-107)
    if drop_text:
        text = torch.zeros_like(text)
    h = F.embedding(text, sd[p + "text_embed.weight"])
    if valid is not None:
        h = h.masked_fill(~valid[..., None], 0.0)
    if cfg.conv_layers > 0:
        pos = abs_pos_table(cfg.tdim, n, dtype=h.dtype)
        if valid is not None:
            pos = pos[None] * valid[..., None].to(pos.dtype)
        h = h + pos
        for i in range(cfg.conv_layers):
            if cfg.text_mask_padding:
                h = h.masked_fill(filler[..., None], 0.0)
            h = convnext_v2_block(sd, f"{p}text_blocks.{i}.", h)
        if cfg.text_mask_padding:
            h = h.masked_fill(filler[..., None], 0.0)
    return h


def text_embedding_unett(sd, cfg: ArchConfig, text, seq_len: int, drop_text: bool):
    """backbones/unett.py:55-84"""
    p = "transformer.text_embed."
    text = (text + 1)[:, :seq_len]
    text = F.pad(text, (0, seq_len - text.shape[1]), value=0)
    filler = text == 0
    if drop_text:
        text = torch.zeros_like(text)
    h = F.embedding(text, sd[p + "text_embed.weight"])
    if cfg.conv_layers > 0:
        h = h + abs_pos_table(cfg.tdim, 4096, dtype=h.dtype)[:seq_len]
        for i in range(cfg.conv_layers):
            if cfg.text_mask_padding:
                h = h.masked_fill(filler[..., None], 0.0)
            h = convnext_v2_block(sd, f"{p}text_blocks.{i}.", h)
        if cfg.text_mask_padding:
            h = h.masked_fill(filler[..., None], 0.0)
    return h


def conv_position_embedding(sd, x, mask, p="transformer.input_embed.conv_pos_embed."):
    """modules.py:175-201.  x [B, N, D], mask bool[B, N] | None"""
    h = x.transpose(1, 2)
    m = None if mask is None else mask[:, None, :]
    if m is not None:
        h = h.masked_fill(~m, 0.0)
    for i in (0, 2):
        h = F.conv1d(h, sd[f"{p}conv1d.{i}.weight"], sd[f"{p}conv1d.{i}.bias"], padding=15, groups=16)
        if m is not None:
            h = h.masked_fill(~m, 0.0)
        h = F.mish(h)
    return h.transpose(1, 2)


def input_embedding(sd, x, cond, text_emb, drop_audio_cond: bool, mask):
    """backbones/dit.py:151-164 (unett.py:90-102 passes mask=None)"""
    if drop_audio_cond:
        cond = torch.zeros_like(cond)
    h = _linear(sd, "transformer.input_embed.proj", torch.cat((x, cond, text_emb), dim=-1))
    return conv_position_embedding(sd, h, mask) + h


def rope_angles(n: int, dim_head=64, base=10000.0, dtype=torch.float32) -> torch.Tensor:
    """x_transformers RotaryEmbedding.forward_from_seq_len (dit.py:207,352): [n, dim_head], interleaved duplicate,
    computed in `dtype`"""
    inv = 1.0 / (base ** (torch.arange(0, dim_head, 2).to(dtype) / dim_head))
    ang = torch.outer(torch.arange(n).to(dtype), inv)
    return torch.stack((ang, ang), dim=-1).flatten(-2)


def apply_rope(t: torch.Tensor, ang: torch.Tensor) -> torch.Tensor:
    """x_transformers apply_rotary_pos_emb (modules.py:499-509): pairs (x0,x1)->(x0 c - x1 s, x1 c + x0 s)"""
    tp = t.unflatten(-1, (-1, 2))
    rot = torch.stack((-tp[..., 1], tp[..., 0]), dim=-1).flatten(-2)
    return t * ang.cos() + rot * ang.sin()


def attention(sd, cfg: ArchConfig, p: str, x, mask, ang):
    """modules.py:471-556 AttnProcessor (torch backend).  x [Be, N, D]"""
    B, N, _ = x.shape
    H, dh = cfg.heads, cfg.dim_head
    q = _linear(sd, p + "to_q", x).view(B, N, H, dh).transpose(1, 2)
    k = _linear(sd, p + "to_k", x).view(B, N, H, dh).transpose(1, 2)
    v = _linear(sd, p + "to_v", x).view(B, N, H, dh).transpose(1, 2)
    pn = H if cfg.pe_attn_head is None else cfg.pe_attn_head
    q = torch.cat((apply_rope(q[:, :pn], ang), q[:, pn:]), dim=1)
    k = torch.cat((apply_rope(k[:, :pn], ang), k[:, pn:]), dim=1)
    key_mask = None
    if cfg.attn_mask_enabled and mask is not None:
        key_mask = mask[:, None, None, :].expand(B, H, N, N)
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=key_mask, dropout_p=0.0, is_causal=False)
    o = o.transpose(1, 2).reshape(B, N, H * dh)
    o = _linear(sd, p + "to_out.0", o)
    if mask is not None:
        o = o.masked_fill(~mask[..., None], 0.0)
    return o


def feed_forward(sd, p: str, x):
    """modules.py:353-364 with approximate='tanh' (modules.py:741; unett.py:168)"""
    return _linear(sd, p + "ff.2", F.gelu(_linear(sd, p + "ff.0.0", x), approximate="tanh"))


def dit_block(sd, cfg, i: int, x, t_emb, mask, ang):
    """modules.py:743-757 DiTBlock.forward + AdaLayerNorm 312-326"""
    p = f"transformer.transformer_blocks.{i}."
    mod = _linear(sd, p + "attn_norm.linear", F.silu(t_emb))
    shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = mod.chunk(6, dim=1)
    h = _ln_noaffine(x) * (1 + scale_msa[:, None]) + shift_msa[:, None]
    x = x + gate_msa[:, None] * attention(sd, cfg, p + "attn.", h, mask, ang)
    h = _ln_noaffine(x) * (1 + scale_mlp[:, None]) + shift_mlp[:, None]
    return x + gate_mlp[:, None] * feed_forward(sd, p + "ff.", h)


def _pack_cfg(sd, cfg, x, cond, text_c, text_u, mask):
    xc = input_embedding(sd, x, cond, text_c, False, mask)
    xu = input_embedding(sd, x, cond, text_u, True, mask)
    return torch.cat((xc, xu), dim=0)


def dit_forward(sd, cfg: ArchConfig, x, cond, text_emb, time, mask, cfg_infer: bool):
    """backbones/dit.py:319-370.  text_emb = (cond_variant, uncond_variant) cached text embeddings.

    cfg_infer=True packs cond/uncond on the batch axis; otherwise only text_emb[0] with the
    undropped audio condition is evaluated (cfm.py:166-177).
    """
    B, N, _ = x.shape
    t = time.reshape(-1).expand(B) if time.ndim == 0 or time.numel() == 1 else time
    t_emb = timestep_embedding(sd, t)
    if cfg_infer:
        h = _pack_cfg(sd, cfg, x, cond, text_emb[0], text_emb[1], mask)
        t_emb = torch.cat((t_emb, t_emb), dim=0)
        mask = None if mask is None else torch.cat((mask, mask), dim=0)
    else:
        h = input_embedding(sd, x, cond, text_emb[0], False, mask)
    ang = rope_angles(N, cfg.dim_head, dtype=h.dtype)
    for i in range(cfg.depth):
        h = dit_block(sd, cfg, i, h, t_emb, mask, ang)
    mod = _linear(sd, "transformer.norm_out.linear", F.silu(t_emb))  # modules.py:342-347
    scale, shift = mod.chunk(2, dim=1)
    h = _ln_noaffine(h) * (1 + scale)[:, None] + shift[:, None]
    return _linear(sd, "transformer.proj_out", h)


def x_rmsnorm(x, g):
    """x_transformers.RMSNorm (unett.py:19,154): F.normalize(x) * sqrt(dim) * g"""
    return F.normalize(x, dim=-1) * (x.shape[-1] ** 0.5) * g


def unett_forward(sd, cfg: ArchConfig, x, cond, text_emb, time, mask, cfg_infer: bool):
    """backbones/unett.py:244-307"""
    B, N, _ = x.shape
    t = time.reshape(-1).expand(B) if time.ndim == 0 or time.numel() == 1 else time
    t_emb = timestep_embedding(sd, t)
    if cfg_infer:
        h = _pack_cfg(sd, cfg, x, cond, text_emb[0], text_emb[1], None)  # unett.py:101 — conv-pos unmasked
        t_emb = torch.cat((t_emb, t_emb), dim=0)
        mask = None if mask is None else torch.cat((mask, mask), dim=0)
    else:
        h = input_embedding(sd, x, cond, text_emb[0], False, None)
    h = torch.cat((t_emb[:, None], h), dim=1)
    if mask is not None:
        mask = F.pad(mask, (1, 0), value=True)
    ang = rope_angles(N + 1, cfg.dim_head, dtype=h.dtype)
    skips = []
    half = cfg.depth // 2
    for i in range(cfg.depth):
        p = f"transformer.layers.{i}."
        if i < half:
            skips.append(h)
        else:
            h = F.linear(torch.cat((h, skips.pop()), dim=-1), sd[p + "0.weight"])
        h = attention(sd, cfg, p + "2.", x_rmsnorm(h, sd[p + "1.g"]), mask, ang) + h
        h = feed_forward(sd, p + "4.", x_rmsnorm(h, sd[p + "3.g"])) + h
    h = x_rmsnorm(h, sd["transformer.norm_out.g"])[:, 1:]
    return _linear(sd, "transformer.proj_out", h)


# ---------------------------------------------------------------------------
# sampler (a1-a6): model/cfm.py:83-229
# ---------------------------------------------------------------------------
EPSS = {  # model/utils.py:205-218
    5: [0, 2, 4, 8, 16, 32],
    6: [0, 2, 4, 6, 8, 16, 32],
    7: [0, 2, 4, 6, 8, 16, 24, 32],
    10: [0, 2, 4, 6, 8, 12, 16, 20, 24, 28, 32],
    12: [0, 2, 4, 6, 8, 10, 12, 14, 16, 20, 24, 28, 32],
    16: [0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 32],
}


def time_grid(steps: int, sway: Optional[float], use_epss=True, t_start=0.0) -> torch.Tensor:
    """cfm.py:203-216"""
    if t_start == 0 and use_epss and steps in EPSS:
        t = (1.0 / 32.0) * torch.tensor(EPSS[steps], dtype=torch.float32)
    else:
        t = torch.linspace(t_start, 1, steps + 1, dtype=torch.float32)
    if sway is not None:
        t = t + sway * (torch.cos(torch.pi / 2 * t) - 1 + t)
    return t


def lens_to_mask(lens: torch.Tensor, length: Optional[int] = None) -> torch.Tensor:
    """model/utils.py:53-58"""
    length = int(lens.amax()) if length is None else length
    return torch.arange(length)[None, :] < lens[:, None]


@dataclass
class SampleResult:
    out: torch.Tensor
    trajectory: torch.Tensor
    y0: torch.Tensor
    t: torch.Tensor
    extras: dict = field(default_factory=dict)


@torch.no_grad()
def sample(sd, cfg: ArchConfig, cond, text, duration, *, lens=None, steps=32, cfg_strength=1.0,
           sway_sampling_coef=None, seed=None, max_duration=65536, use_epss=True, no_ref_audio=False,
           edit_mask=None, y0=None) -> SampleResult:
    """model/cfm.py:83-229 (vocoder hook, duplicate_test omitted: off the measured path).

    cond: [B, nw] raw wave or [B, n, mel]; text: int[B, nt] padded with -1.
    y0: optional injected noise [B, N, mel] (SURVEY.md §8c RNG caveat); default follows cfm.py:196-201.
    """
    if cond.ndim == 2:
        cond = mel_spectrogram(cond).permute(0, 2, 1)
    cond = cond.float()
    B, n_cond = cond.shape[:2]
    if lens is None:
        lens = torch.full((B,), n_cond, dtype=torch.long)
    cond_mask = lens_to_mask(lens)
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
    mask = lens_to_mask(duration) if B > 1 else None

    # text embeddings are computed once per sample() and cached (dit.py:294-310; unett.py:219-232)
    if cfg.backbone == "DiT":
        seq_len = N if mask is None else mask.sum(dim=1)
        te = (text_embedding_dit(sd, cfg, text, seq_len, False), text_embedding_dit(sd, cfg, text, seq_len, True))
        fwd = dit_forward
    else:
        te = (text_embedding_unett(sd, cfg, text, N, False), text_embedding_unett(sd, cfg, text, N, True))
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
    t = time_grid(steps, sway_sampling_coef, use_epss)
    traj = [y0]
    y = y0
    for k in range(t.shape[0] - 1):  # torchdiffeq fixed-grid Euler (cfm.py:218)
        y = y + (t[k + 1] - t[k]) * fn(t[k], y)
        traj.append(y)
    out = torch.where(cond_mask, cond, y)
    return SampleResult(out=out, trajectory=torch.stack(traj, 0), y0=y0, t=t,
                        extras={"text_cond": te[0], "text_uncond": te[1], "mask": mask, "step_cond": step_cond})


# ---------------------------------------------------------------------------
# Vocos back-end (a18) — third-party `vocos` package, restated (parity unpinned)
# ---------------------------------------------------------------------------
def istft_center(spec: torch.Tensor, n_fft=1024, hop=256, window=None) -> torch.Tensor:
    """== torch.istft(spec, n_fft, hop, n_fft, hann, center=True)  (SURVEY.md §9.3).  spec complex [B, F, T]"""
    B, _, T = spec.shape
    window = torch.hann_window(n_fft, periodic=True) if window is None else window
    frames = torch.fft.irfft(spec, n=n_fft, dim=1) * window[None, :, None]  # [B, n_fft, T]
    L = n_fft + hop * (T - 1)
    y = F.fold(frames, output_size=(1, L), kernel_size=(1, n_fft), stride=(1, hop))[:, 0, 0]
    env = F.fold((window ** 2)[None, :, None].expand(1, n_fft, T), output_size=(1, L), kernel_size=(1, n_fft),
                 stride=(1, hop))[:, 0, 0]
    pad = n_fft // 2
    return y[:, pad:L - pad] / env[:, pad:L - pad]


@torch.no_grad()
def vocos_decode(vsd, mel: torch.Tensor, layers=8) -> torch.Tensor:
    """vocos.Vocos.decode as constructed at infer/utils_infer.py:118-129 (charactr/vocos-mel-24khz):
    VocosBackbone + ISTFTHead(padding='center').  mel [B, 100, n] -> wav [B, 256 (n-1)].
    Head restated in-tree at runtime/triton_trtllm/scripts/export_vocoder_to_onnx.py:45-59.
    """
    h = F.conv1d(mel.float(), vsd["backbone.embed.weight"], vsd["backbone.embed.bias"], padding=3)
    h = F.layer_norm(h.transpose(1, 2), (h.shape[1],), vsd["backbone.norm.weight"], vsd["backbone.norm.bias"], 1e-6)
    for i in range(layers):
        p = f"backbone.convnext.{i}."
        r = h
        h = F.conv1d(h.transpose(1, 2), vsd[p + "dwconv.weight"], vsd[p + "dwconv.bias"], padding=3,
                     groups=h.shape[-1]).transpose(1, 2)
        h = F.layer_norm(h, (h.shape[-1],), vsd[p + "norm.weight"], vsd[p + "norm.bias"], 1e-6)
        h = F.linear(F.gelu(F.linear(h, vsd[p + "pwconv1.weight"], vsd[p + "pwconv1.bias"])),
                     vsd[p + "pwconv2.weight"], vsd[p + "pwconv2.bias"])
        h = r + vsd[p + "gamma"] * h
    h = F.layer_norm(h, (h.shape[-1],), vsd["backbone.final_layer_norm.weight"],
                     vsd["backbone.final_layer_norm.bias"], 1e-6)
    o = F.linear(h, vsd["head.out.weight"], vsd["head.out.bias"]).transpose(1, 2)
    mag, ph = o.chunk(2, dim=1)
    mag = torch.clip(torch.exp(mag), max=1e2)
    spec = torch.complex(mag * torch.cos(ph), mag * torch.sin(ph))
    return istft_center(spec, window=vsd["head.istft.window"])
