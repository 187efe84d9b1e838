"""MMDiT on the CPU: the oracle against the reference fixtures, the checkpoint keys, the constructor surface, and the
DiT / UNetT parameter specs and packed-cache keys, which the MMDiT backbone must leave as they were."""
from __future__ import annotations

import glob
import hashlib
import importlib
import json
import os
import sys
import warnings

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import synthdata as SD  # noqa: E402
from f5_tts_b200 import model as M  # noqa: E402
from f5_tts_b200 import weights as W  # noqa: E402
from oracle import mmdit as OMM  # noqa: E402
from oracle import ref_shims  # noqa: E402

FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "mmdit_*.npz")))
NAMES = [os.path.basename(p)[:-4] for p in FIXTURES]


def load_case(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    cfg = SD.ArchConfig(**json.loads(str(z["cfg"])))
    return z, cfg


def case_args(z):
    dur = z["duration"]
    duration = int(dur) if dur.ndim == 0 else torch.from_numpy(dur).long()
    lens = torch.from_numpy(z["lens"]).long() if z["lens"].size else None
    sway = float(z["sway"])
    return dict(cond=torch.from_numpy(z["cond"]), text=torch.from_numpy(z["text"]).long(), duration=duration,
                lens=lens, steps=int(z["steps"]), cfg_strength=float(z["cfg_strength"]),
                sway_sampling_coef=None if np.isnan(sway) else sway, seed=int(z["seed"]), method=str(z["method"]))


def rel_l2(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-12))


def test_fixtures_cover_the_cases():
    assert len(NAMES) >= 9
    cfgs = [load_case(n)[1] for n in NAMES]
    assert any(c.attn_mask_enabled for c in cfgs) and any(c.qk_norm for c in cfgs)
    assert any(not c.text_mask_padding for c in cfgs) and any(c.dim_head == 128 for c in cfgs)
    assert any(c.dim == 1024 and c.heads == 16 for c in cfgs)
    assert any(load_case(n)[0]["text"].shape[1] > 128 for n in NAMES)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_reference_fixture(name):
    z, cfg = load_case(name)
    a = case_args(z)
    sd = SD.synthetic_state_dict(cfg, seed=int(z["wseed"]))
    torch.manual_seed(0)
    res = OMM.sample(sd, cfg, a.pop("cond"), a.pop("text"), a.pop("duration"), **a)
    assert rel_l2(res.trajectory[1], torch.from_numpy(z["traj_1"])) <= 1e-6
    assert rel_l2(res.out, torch.from_numpy(z["out"])) <= 1e-6


def test_attention_mask_mode_changes_the_output():
    a, _ = load_case("mmdit_b2_varlen")
    b, _ = load_case("mmdit_b2_attnmask")
    assert rel_l2(torch.from_numpy(a["out"]), torch.from_numpy(b["out"])) > 1e-4


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_keys_equal_the_reference(name):
    z, cfg = load_case(name)
    ref = [str(k) for k in z["ref_keys"]]
    assert [k for k, _, _ in SD.state_dict_spec(cfg)] == ref
    m = M.MMDiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
                mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds, text_mask_padding=cfg.text_mask_padding,
                qk_norm=cfg.qk_norm, attn_mask_enabled=cfg.attn_mask_enabled)
    pre = "transformer."
    assert set(m.state_dict()) == {k[len(pre):] for k in ref if k.startswith(pre)}
    sd = {k[len(pre):]: v for k, v in SD.synthetic_state_dict(cfg).items() if k.startswith(pre)}
    res = m.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys


REJECTED = [dict(text_dim=512), dict(conv_layers=4), dict(pe_attn_head=1), dict(long_skip_connection=True),
            dict(text_embedding_average_upsampling=True)]
ACCEPTED = dict(dropout=0.0, checkpoint_activations=True, attn_backend="torch", attn_mask_enabled=True,
                text_mask_padding=False, qk_norm="rms_norm", dim_head=128, heads=2)


def _constructors():
    yield M.MMDiT
    if ref_shims.reference_available():
        ref_shims.import_reference()
        yield importlib.import_module("f5_tts.model.backbones.mmdit").MMDiT


@pytest.mark.parametrize("bad", REJECTED, ids=lambda d: next(iter(d)))
def test_constructor_rejects_what_the_reference_rejects(bad):
    for cls in _constructors():
        with pytest.raises(TypeError):
            cls(dim=128, depth=2, heads=2, **bad)


def test_constructor_accepts_the_reference_arguments():
    for cls in _constructors():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            cls(dim=256, depth=2, ff_mult=2, mel_dim=100, text_num_embeds=50, **ACCEPTED)
        with pytest.raises(ValueError):
            cls(dim=128, depth=2, heads=2, qk_norm="layer_norm")


@pytest.mark.skipif(not ref_shims.reference_available(), reason="reference checkout not available")
def test_constructor_signature_matches_the_reference():
    import inspect

    ref_shims.import_reference()
    ref = importlib.import_module("f5_tts.model.backbones.mmdit").MMDiT
    assert list(inspect.signature(M.MMDiT.__init__).parameters) == list(inspect.signature(ref.__init__).parameters)


# Parameter specs and packed-cache keys of DiT / UNetT models, as they were before MMDiT was added.
OTHER_MODELS = [
    ("dit_v1", M.DiT, dict(dim=128, depth=2, heads=2, ff_mult=2, text_dim=64, conv_layers=2, text_mask_padding=True,
                           pe_attn_head=None), "93b54f80454f4e4f",
     "('DiT', 128, 2, 2, 64, 256, 100, 64, 50, 2, True, None)"),
    ("dit_opts", M.DiT, dict(dim=128, depth=2, heads=2, ff_mult=2, text_dim=64, conv_layers=2, qk_norm="rms_norm",
                             long_skip_connection=True), "8fe97f0798845a46",
     "('DiT', 128, 2, 2, 64, 256, 100, 64, 50, 2, True, None, 'rms_norm', True, False)"),
    ("unett", M.UNetT, dict(dim=128, depth=4, heads=2, ff_mult=4, text_dim=None, conv_layers=0, pe_attn_head=1),
     "d723d501ee6216d9", "('UNetT', 128, 4, 2, 64, 512, 100, 100, 50, 0, True, 1)"),
]


@pytest.mark.parametrize("name,cls,kw,spec_digest,arch", OTHER_MODELS, ids=[o[0] for o in OTHER_MODELS])
def test_dit_unett_specs_and_cache_keys_unchanged(tmp_path, name, cls, kw, spec_digest, arch):
    m = cls(**kw, text_num_embeds=50)
    spec = M._backbone_spec(m.KIND, dim=m.dim, depth=m.depth, heads=m.heads, dim_head=m.dim_head,
                            ff_mult=kw["ff_mult"], mel_dim=100, text_num_embeds=50, text_dim=m.text_dim,
                            conv_layers=m.conv_layers, qk_norm=m.qk_norm, long_skip_connection=m.long_skip)
    assert hashlib.sha256(repr(spec).encode()).hexdigest()[:16] == spec_digest
    ckpt = tmp_path / "model.pt"
    ckpt.write_bytes(b"x" * 1000)
    st = os.stat(ckpt)
    raw = f"{os.path.abspath(ckpt)}|{st.st_size}|{st.st_mtime_ns}|{arch}|fmt1"
    assert W.cache_key(str(ckpt), m) == hashlib.sha256(raw.encode()).hexdigest()[:24]


def test_mmdit_cache_key_covers_backbone_and_architecture(tmp_path):
    ckpt = tmp_path / "model.pt"
    ckpt.write_bytes(b"x" * 1000)
    base = dict(dim=128, depth=2, heads=2, ff_mult=2, text_num_embeds=50)
    keys = {W.cache_key(str(ckpt), M.MMDiT(**base)),
            W.cache_key(str(ckpt), M.MMDiT(**dict(base, depth=3))),
            W.cache_key(str(ckpt), M.MMDiT(**base, qk_norm="rms_norm")),
            W.cache_key(str(ckpt), M.MMDiT(**base, text_mask_padding=False)),
            W.cache_key(str(ckpt), M.DiT(**base, text_dim=0, conv_layers=0, pe_attn_head=None))}
    assert len(keys) == 5
