"""CPU: DiT / UNetT checkpoints built with 128-wide attention heads (dim_head=128).

  * the oracle reproduces the unmodified reference on the fixtures of oracle/make_golden_dim_head.py (rel-L2 0.0 at
    generation time, bound 1e-6 here, as for the other fixtures);
  * the package's constructors accept dim_head 64 and 128 and refuse any other width, and their state-dict keys and
    shapes equal synthdata.state_dict_spec, so a dim_head=128 checkpoint loads with strict=True;
  * the packed-weight cache key of a dim_head=64 model is what it was before 128 was accepted.
"""
import hashlib
import os

import numpy as np
import pytest
import torch

import synthdata as SD
from oracle import arch_options as OA
from oracle import f5_oracle as O
from oracle import make_golden as MG
from oracle import make_golden_dim_head as MD
from test_arch_options_cpu import cfg_from_repr

TOL = 1e-6


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("name", sorted(MD.CASES))
def test_oracle_reproduces_dim_head_fixture(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg, kw = MD.CASES[name]
    assert cfg.dim_head == 128
    assert cfg_from_repr(str(z["cfg"])) == cfg and str(z["method"]) == kw.get("method", "euler")
    sd = O.synthetic_state_dict(cfg, seed=int(z["wseed"]))
    cond, text, duration, lens = MD.MA.case_inputs(cfg, **kw)
    res = OA.sample(sd, cfg, cond, text, duration, lens=lens, method=kw.get("method", "euler"), steps=kw["steps"],
                    cfg_strength=kw["cfg_strength"], sway_sampling_coef=kw["sway"], seed=kw["seed"])
    assert torch.equal(res.y0, torch.from_numpy(z["y0"]))
    r1, rn = _rel(res.trajectory[1], torch.from_numpy(z["traj_1"])), _rel(res.out, torch.from_numpy(z["out"]))
    print(f"[{name}] oracle vs reference: step-1 rel-L2 {r1:.3e}  final {rn:.3e}")
    assert r1 <= TOL and rn <= TOL


def _model(cls_name, dim_head, **kw):
    import f5_tts_b200 as F5

    return getattr(F5, cls_name)(dim=128, depth=2, heads=2, dim_head=dim_head, **kw)


@pytest.mark.parametrize("cls_name", ["DiT", "UNetT"])
def test_constructors_accept_64_and_128(cls_name):
    for dh in (64, 128):
        m = _model(cls_name, dh, qk_norm="rms_norm")
        assert m.dim_head == dh
        sd = m.state_dict()
        q = "transformer_blocks.0.attn." if cls_name == "DiT" else "layers.0.2."
        assert tuple(sd[q + "to_q.weight"].shape) == (2 * dh, 128)
        assert tuple(sd[q + "q_norm.weight"].shape) == (dh,)
        assert tuple(sd["rotary_embed.inv_freq"].shape) == (dh // 2,)


@pytest.mark.parametrize("cls_name", ["DiT", "UNetT"])
@pytest.mark.parametrize("dim_head", [32, 96, 256])
def test_constructors_reject_other_widths(cls_name, dim_head):
    with pytest.raises(NotImplementedError, match="64, 128"):
        _model(cls_name, dim_head)


def test_attention_width_over_1024_is_rejected():
    import f5_tts_b200 as F5

    F5.DiT(dim=1024, depth=1, heads=8, dim_head=128)
    with pytest.raises(NotImplementedError):
        F5.DiT(dim=1024, depth=1, heads=16, dim_head=128)


@pytest.mark.parametrize("name", sorted(MD.CASES))
def test_state_dict_keys_equal_spec(name):
    import f5_tts_b200 as F5

    cfg, _ = MD.CASES[name]
    cls = F5.DiT if cfg.backbone == "DiT" else F5.UNetT
    kw = dict(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
              mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim,
              text_mask_padding=cfg.text_mask_padding, conv_layers=cfg.conv_layers, pe_attn_head=cfg.pe_attn_head,
              qk_norm=cfg.qk_norm)
    model = F5.CFM(transformer=cls(**kw))
    got = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    assert got == {k: shape for k, shape, _ in SD.state_dict_spec(cfg)}
    model.load_state_dict(SD.synthetic_state_dict(cfg, seed=1234), strict=True)


def test_cache_key_dim_head(tmp_path):
    """dim_head = 64: the key is the one packed caches were written under before 128 was accepted; 128 gets its own."""
    from f5_tts_b200 import weights as Wt

    ck = tmp_path / "model.safetensors"
    ck.write_bytes(b"x")
    st = os.stat(ck)
    m64 = _model("DiT", 64)
    arch = (m64.KIND, m64.dim, m64.depth, m64.heads, 64, m64.ff_inner, m64.mel_dim, m64.text_dim,
            m64.text_num_embeds, m64.conv_layers, m64.text_mask_padding, m64.pe_attn_head)
    raw = f"{os.path.abspath(ck)}|{st.st_size}|{st.st_mtime_ns}|{arch}|fmt{Wt.PACK_FORMAT}"
    assert Wt.cache_key(str(ck), m64) == hashlib.sha256(raw.encode()).hexdigest()[:24]
    assert Wt.cache_key(str(ck), _model("DiT", 128)) != Wt.cache_key(str(ck), m64)
    assert Wt.cache_key(str(ck), _model("UNetT", 128)) != Wt.cache_key(str(ck), _model("UNetT", 64))


def test_tiny_fixture_inner_differs_from_dim():
    """The tiny fixtures run an attention width (heads * 128) that is not the model width."""
    cfg, _ = MD.CASES["dh128_dit_b2_varlen"]
    assert cfg.heads * cfg.dim_head != cfg.dim
    assert MG.tiny_dit().dim_head == 64
