"""CPU: the dim-768 Small configs (F5TTS_v1_Small, F5TTS_Small, E2TTS_Small).

  * the oracle reproduces the unmodified reference's CFM.sample at Small width (tests/golden/*small*.npz, written by
    oracle/make_golden_small.py; rel-L2 0.0 at generation time, bound 1e-6 here);
  * api.MODEL_ARCH names exactly the six configs the reference ships;
  * the package's DiT / UNetT built from the Small entries have the released checkpoint layout of the Small presets.
"""
import ast
import json
import os

import numpy as np
import pytest
import torch

import synthdata as SD
from f5_tts_b200 import api
from oracle import f5_oracle as O

TOL = 1e-6
FIXTURES = ["f5v1small_b2_varlen", "f5small_b1_n192", "e2small_b2_varlen"]
PRESETS = {"F5TTS_v1_Small": SD.f5tts_v1_small, "F5TTS_Small": SD.f5tts_small, "E2TTS_Small": SD.e2tts_small}


def _cfg_from_repr(s: str) -> O.ArchConfig:
    body = s[s.index("(") + 1: s.rindex(")")]
    return O.ArchConfig(**{k: ast.literal_eval(v) for k, v in (p.split("=") for p in body.split(", "))})


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_small_reference_fixture(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg = _cfg_from_repr(str(z["cfg"]))
    assert cfg.dim == 768 and cfg.heads == 12
    sd = O.synthetic_state_dict(cfg, seed=int(z["wseed"]))
    dur = z["duration"]
    duration = int(dur) if dur.ndim == 0 else torch.from_numpy(dur).long()
    lens = torch.from_numpy(z["lens"]).long() if z["lens"].size else None
    sway = None if np.isnan(z["sway"]) else float(z["sway"])
    res = O.sample(sd, cfg, torch.from_numpy(z["cond"]), torch.from_numpy(z["text"]), duration, lens=lens,
                   steps=int(z["steps"]), cfg_strength=float(z["cfg_strength"]), sway_sampling_coef=sway,
                   seed=int(z["seed"]))
    assert torch.equal(res.y0, torch.from_numpy(z["y0"]))
    r1, rn = _rel(res.trajectory[1], torch.from_numpy(z["traj_1"])), _rel(res.out, torch.from_numpy(z["out"]))
    print(f"[{name}] oracle vs reference: step-1 rel-L2 {r1:.3e}  final {rn:.3e}")
    assert r1 <= TOL and rn <= TOL


def test_model_arch_names_the_six_shipped_configs(golden_dir):
    with open(os.path.join(golden_dir, "reference_model_configs.json")) as f:
        ref = json.load(f)
    assert set(api.MODEL_ARCH) == set(ref)
    assert len(api.MODEL_ARCH) == 6


@pytest.mark.parametrize("name", sorted(PRESETS))
def test_small_model_keys_match_preset_layout(name):
    """The package's backbone built from the MODEL_ARCH entry has the released key layout of the synthdata preset, so
    a Small checkpoint loads with strict=True."""
    import f5_tts_b200 as F5

    cls, arch = api.MODEL_ARCH[name]
    cfg = PRESETS[name]()
    assert cls.__name__ == cfg.backbone and arch["dim"] == cfg.dim == 768
    model = F5.CFM(transformer=cls(**arch, text_num_embeds=cfg.text_num_embeds, mel_dim=cfg.mel_dim))
    got = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    want = {k: shape for k, shape, _ in SD.state_dict_spec(cfg)}
    assert got == want
    # the grouped conv position embedding has dim / 16 = 48 channels per group
    assert want["transformer.input_embed.conv_pos_embed.conv1d.0.weight"] == (768, 48, 31)
