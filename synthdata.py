"""Synthetic model weights, architecture presets and inputs of the BASELINE.json workloads (NEUTRAL test data).

Shared by the product-side measurement (`bench.py`, `__graft_entry__.smoke()`), the tests and the CPU oracle so that
every arm sees bit-identical weights and inputs; it contains no arithmetic of the hot path and imports neither the
product package nor `oracle/`.  Weights follow the released checkpoint key layout (SURVEY.md §8b); every tensor the
reference zero-initialises (AdaLN linears, norm_out, proj_out, GRN gamma/beta — backbones/dit.py:264-274,
modules.py:239-240) is re-randomised so that the synthetic model exercises every kernel (SURVEY.md §0.4, §8d).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch


# ---------------------------------------------------------------------------
# configuration (mirrors yaml `model.arch`, configs/F5TTS_Base.yaml:25-35 etc.)
# ---------------------------------------------------------------------------
@dataclass
class ArchConfig:
    backbone: str = "DiT"  # "DiT" | "UNetT"
    dim: int = 1024
    depth: int = 22
    heads: int = 16
    dim_head: int = 64
    ff_mult: int = 2
    mel_dim: int = 100
    text_num_embeds: int = 2545
    text_dim: Optional[int] = 512
    text_mask_padding: bool = False
    conv_layers: int = 4
    pe_attn_head: Optional[int] = 1
    attn_mask_enabled: bool = False

    @property
    def tdim(self) -> int:
        return self.mel_dim if self.text_dim is None else self.text_dim


def f5tts_base() -> ArchConfig:  # configs/F5TTS_Base.yaml:25-35
    return ArchConfig()


def f5tts_v1_base() -> ArchConfig:  # configs/F5TTS_v1_Base.yaml:26-36
    return ArchConfig(text_mask_padding=True, pe_attn_head=None)


def e2tts_base() -> ArchConfig:  # configs/E2TTS_Base.yaml:25-31
    return ArchConfig(backbone="UNetT", depth=24, ff_mult=4, text_dim=None, conv_layers=0,
                      text_mask_padding=False, pe_attn_head=1)


def f5tts_small() -> ArchConfig:  # configs/F5TTS_Small.yaml:25-35
    return ArchConfig(dim=768, depth=18, heads=12)


def f5tts_v1_small() -> ArchConfig:  # configs/F5TTS_v1_Small.yaml:26-36
    return ArchConfig(dim=768, depth=18, heads=12, text_mask_padding=True, pe_attn_head=None)


def e2tts_small() -> ArchConfig:  # configs/E2TTS_Small.yaml:25-31
    return ArchConfig(backbone="UNetT", dim=768, depth=20, heads=12, ff_mult=4, text_dim=None, conv_layers=0,
                      text_mask_padding=False, pe_attn_head=1)


# ---------------------------------------------------------------------------
# synthetic weights in the released checkpoint layout
# ---------------------------------------------------------------------------
def state_dict_spec(cfg: ArchConfig) -> list[tuple[str, tuple[int, ...], str]]:
    """(key, shape, kind) for every tensor of CFM(transformer=DiT|UNetT) — SURVEY.md §8b.

    kind selects the synthetic distribution only.
    """
    D, T, M = cfg.dim, cfg.tdim, cfg.mel_dim
    inner = cfg.heads * cfg.dim_head
    ff = int(D * cfg.ff_mult)
    spec: list[tuple[str, tuple[int, ...], str]] = []

    def lin(prefix, out_f, in_f, kind="linear", bias=True):
        spec.append((prefix + ".weight", (out_f, in_f), kind))
        if bias:
            spec.append((prefix + ".bias", (out_f,), "bias"))

    p = "transformer."
    lin(p + "time_embed.time_mlp.0", D, 256)
    lin(p + "time_embed.time_mlp.2", D, D)
    spec.append((p + "text_embed.text_embed.weight", (cfg.text_num_embeds + 1, T), "embed"))
    for i in range(cfg.conv_layers):
        b = f"{p}text_embed.text_blocks.{i}."
        spec.append((b + "dwconv.weight", (T, 1, 7), "conv"))
        spec.append((b + "dwconv.bias", (T,), "bias"))
        spec.append((b + "norm.weight", (T,), "ln_w"))
        spec.append((b + "norm.bias", (T,), "bias"))
        lin(b + "pwconv1", 2 * T, T)
        spec.append((b + "grn.gamma", (1, 1, 2 * T), "grn_g"))
        spec.append((b + "grn.beta", (1, 1, 2 * T), "grn_b"))
        lin(b + "pwconv2", T, 2 * T)
    lin(p + "input_embed.proj", D, 2 * M + T)
    for i in (0, 2):
        spec.append((f"{p}input_embed.conv_pos_embed.conv1d.{i}.weight", (D, D // 16, 31), "conv"))
        spec.append((f"{p}input_embed.conv_pos_embed.conv1d.{i}.bias", (D,), "bias"))
    spec.append((p + "rotary_embed.inv_freq", (cfg.dim_head // 2,), "inv_freq"))
    if cfg.backbone == "DiT":
        for i in range(cfg.depth):
            b = f"{p}transformer_blocks.{i}."
            lin(b + "attn_norm.linear", 6 * D, D, kind="adaln")
            for nm in ("to_q", "to_k", "to_v"):
                lin(b + "attn." + nm, inner, D)
            lin(b + "attn.to_out.0", D, inner)
            lin(b + "ff.ff.0.0", ff, D)
            lin(b + "ff.ff.2", D, ff)
        lin(p + "norm_out.linear", 2 * D, D, kind="adaln")
        lin(p + "proj_out", M, D)
    elif cfg.backbone == "UNetT":
        for i in range(cfg.depth):
            b = f"{p}layers.{i}."
            if i >= cfg.depth // 2:
                lin(b + "0", D, 2 * D, bias=False)
            spec.append((b + "1.g", (D,), "ln_w"))
            for nm in ("to_q", "to_k", "to_v"):
                lin(b + "2." + nm, inner, D)
            lin(b + "2.to_out.0", D, inner)
            spec.append((b + "3.g", (D,), "ln_w"))
            lin(b + "4.ff.0.0", ff, D)
            lin(b + "4.ff.2", D, ff)
        spec.append((p + "norm_out.g", (D,), "ln_w"))
        lin(p + "proj_out", M, D)
    else:
        raise ValueError(cfg.backbone)
    return spec


def _draw(shape, kind, gen, dim_head=64):
    if kind == "inv_freq":
        return 1.0 / (10000.0 ** (torch.arange(0, dim_head, 2).float() / dim_head))
    z = torch.randn(shape, generator=gen, dtype=torch.float32)
    if kind == "linear":
        return z / math.sqrt(shape[1])
    if kind == "adaln":  # zero-init in the reference (dit.py:264-274): MUST be re-randomised, SURVEY.md §0.4
        return z * 0.02
    if kind == "conv":
        return z / math.sqrt(shape[1] * shape[2])
    if kind == "embed":
        return z
    if kind == "bias":
        return z * 0.05
    if kind == "ln_w":
        return 1.0 + 0.1 * z
    if kind == "grn_g":  # zero-init in the reference (modules.py:239-240)
        return 0.3 * z
    if kind == "grn_b":
        return 0.1 * z
    raise ValueError(kind)


def synthetic_state_dict(cfg: ArchConfig, seed: int = 1234) -> dict[str, torch.Tensor]:
    gen = torch.Generator(device="cpu").manual_seed(seed)
    return {k: _draw(shape, kind, gen, cfg.dim_head) for k, shape, kind in state_dict_spec(cfg)}


def vocos_state_dict_spec(dim=512, inter=1536, layers=8, n_mels=100, n_fft=1024):
    spec = [("backbone.embed.weight", (dim, n_mels, 7), "conv"), ("backbone.embed.bias", (dim,), "bias"),
            ("backbone.norm.weight", (dim,), "ln_w"), ("backbone.norm.bias", (dim,), "bias")]
    for i in range(layers):
        b = f"backbone.convnext.{i}."
        spec += [(b + "dwconv.weight", (dim, 1, 7), "conv"), (b + "dwconv.bias", (dim,), "bias"),
                 (b + "norm.weight", (dim,), "ln_w"), (b + "norm.bias", (dim,), "bias"),
                 (b + "pwconv1.weight", (inter, dim), "linear"), (b + "pwconv1.bias", (inter,), "bias"),
                 (b + "pwconv2.weight", (dim, inter), "linear"), (b + "pwconv2.bias", (dim,), "bias"),
                 (b + "gamma", (dim,), "layer_scale")]
    spec += [("backbone.final_layer_norm.weight", (dim,), "ln_w"), ("backbone.final_layer_norm.bias", (dim,), "bias"),
             ("head.out.weight", (n_fft + 2, dim), "linear"), ("head.out.bias", (n_fft + 2,), "bias"),
             ("head.istft.window", (n_fft,), "hann")]
    return spec


def synthetic_vocos_state_dict(seed: int = 4321, **kw) -> dict[str, torch.Tensor]:
    gen = torch.Generator(device="cpu").manual_seed(seed)
    out = {}
    layers = kw.get("layers", 8)
    for k, shape, kind in vocos_state_dict_spec(**kw):
        if kind == "hann":
            out[k] = torch.hann_window(shape[0], periodic=True)
        elif kind == "layer_scale":
            out[k] = torch.full(shape, 1.0 / layers) * (1.0 + 0.1 * torch.randn(shape, generator=gen))
        else:
            out[k] = _draw(shape, kind, gen)
    return out


# ---------------------------------------------------------------------------
# synthetic inputs of the BASELINE.json workloads (SURVEY.md §8d)
# ---------------------------------------------------------------------------
WORKLOADS = {
    # name: backbone, B (per GPU), frames, prompt frames, text tokens, NFE
    "cfg2": dict(arch="f5tts_base", B=1, frames=[938], ref=[282], nt=150, nfe=32),
    "cfg3": dict(arch="f5tts_base", B=8, frames=[469, 670, 871, 1072, 1272, 1473, 1674, 1875],
                 ref=[141, 201, 261, 322, 382, 442, 502, 562], nt=300, nfe=32),
    "cfg4": dict(arch="f5tts_base", B=8, frames=[938] * 8, ref=[282] * 8, nt=150, nfe=16),
    "cfg5": dict(arch="e2tts_base", B=8, frames=[938] * 8, ref=[282] * 8, nt=150, nfe=32),
}
CFG_STRENGTH, SWAY = 2.0, -1.0


def synth_inputs(w: dict, seed: int = 7):
    """(wav [B, n_ref*256] 0.1*randn, text ids [B, nt], duration [B], lens [B]) — same draw order for every arm."""
    g = torch.Generator().manual_seed(seed)
    B = w["B"]
    n_ref = max(w["ref"])
    wav = 0.1 * torch.randn(B, n_ref * 256, generator=g)
    text = torch.randint(0, 2545, (B, w["nt"]), generator=g)
    duration = torch.tensor(w["frames"], dtype=torch.long)
    lens = torch.tensor(w["ref"], dtype=torch.long)
    return wav, text, duration, lens
