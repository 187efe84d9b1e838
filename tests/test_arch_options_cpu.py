"""CPU: the architecture options no shipped config turns on — qk_norm="rms_norm" (DiT, UNetT), long_skip_connection and
text_embedding_average_upsampling (DiT).

  * the oracle (oracle/arch_options.py) reproduces the unmodified reference on the fixtures of oracle/make_golden_arch_options.py (rel-L2 0.0 at
    generation time, bound 1e-6 here), and each option changes the result;
  * the package's DiT / UNetT accept and reject the options as the reference's constructors do, and their state-dict
    keys equal synthdata.state_dict_spec, so checkpoints trained with the options load with strict=True;
  * with the options off, the synthetic weights and the packed-weight cache key are what they were before the options
    existed.
"""
import ast
import hashlib
import os

import numpy as np
import pytest
import torch

import synthdata as SD
from oracle import f5_oracle as O
from oracle import make_golden as MG
from oracle import make_golden_arch_options as MA
from oracle import arch_options as OA

TOL = 1e-6


def cfg_from_repr(s: str) -> O.ArchConfig:
    body = s[s.index("(") + 1: s.rindex(")")]
    return O.ArchConfig(**{k: ast.literal_eval(v) for k, v in (p.split("=") for p in body.split(", "))})


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _oracle(cfg, kw, sd=None):
    sd = O.synthetic_state_dict(cfg, seed=1234) if sd is None else sd
    cond, text, duration, lens = MA.case_inputs(cfg, **kw)
    return OA.sample(sd, cfg, cond, text, duration, lens=lens, method=kw.get("method", "euler"), steps=kw["steps"],
                     cfg_strength=kw["cfg_strength"], sway_sampling_coef=kw["sway"], seed=kw["seed"])


@pytest.mark.parametrize("name", sorted(MA.CASES))
def test_oracle_reproduces_arch_option_fixture(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg, kw = MA.CASES[name]
    assert cfg_from_repr(str(z["cfg"])) == cfg and str(z["method"]) == kw.get("method", "euler")
    res = _oracle(cfg, kw)
    assert torch.equal(res.y0, torch.from_numpy(z["y0"]))
    r1, rn = _rel(res.trajectory[1], torch.from_numpy(z["traj_1"])), _rel(res.out, torch.from_numpy(z["out"]))
    print(f"[{name}] oracle vs reference: step-1 rel-L2 {r1:.3e}  final {rn:.3e}")
    assert r1 <= TOL and rn <= TOL


@pytest.mark.parametrize("option", ["qk_norm", "long_skip_connection", "text_embedding_average_upsampling"])
def test_each_option_changes_the_result(option):
    """The fixtures would not notice a dropped option if it had no effect on them (compared on the generated state: the
    prompt frames of `out` are copied from the condition)."""
    name = {"qk_norm": "opt_dit_qknorm_b2_varlen", "long_skip_connection": "opt_dit_longskip_b2_varlen",
            "text_embedding_average_upsampling": "opt_dit_avgup_b2_varlen"}[option]
    cfg, kw = MA.CASES[name]
    sd = O.synthetic_state_dict(cfg, seed=1234)
    on = _oracle(cfg, kw, sd).trajectory[-1]
    off_cfg = O.ArchConfig(**{**cfg.__dict__, option: None if option == "qk_norm" else False})
    off = _oracle(off_cfg, kw, sd).trajectory[-1]
    print(f"[{option}] on vs off rel-L2 {_rel(off, on):.3e}")
    assert _rel(off, on) > 1e-3


def test_average_upsample_repeats():
    """audio 7 over 3 valid tokens: 7 // 3 = 2 repeats each, the last 7 % 3 = 1 token once more; filler rows skipped."""
    h = torch.arange(1.0, 9.0)[None, :, None]  # rows 1..8
    mask = torch.tensor([[True, False, True, True, False, False, False, False]])
    out = OA.average_upsample(h, mask, torch.tensor([7]))[0, :, 0]
    assert out.tolist() == [1, 1, 3, 3, 4, 4, 4, 0]
    assert OA.average_upsample(h, mask, torch.tensor([2]))[0, :, 0].tolist() == [3, 4, 0, 0, 0, 0, 0, 0]
    assert not OA.average_upsample(h, torch.zeros_like(mask), torch.tensor([7])).any()


# ---------------------------------------------------------------------------------------------------------------------
# constructors and checkpoint layout
# ---------------------------------------------------------------------------------------------------------------------
def _package_model(cfg, **extra):
    import f5_tts_b200 as F5

    cls = F5.DiT if cfg.backbone == "DiT" else F5.UNetT
    kw = dict(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
              mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim,
              text_mask_padding=cfg.text_mask_padding, conv_layers=cfg.conv_layers, pe_attn_head=cfg.pe_attn_head,
              qk_norm=cfg.qk_norm)
    if cfg.backbone == "DiT":
        kw.update(long_skip_connection=cfg.long_skip_connection,
                  text_embedding_average_upsampling=cfg.text_embedding_average_upsampling)
    kw.update(extra)
    return F5.CFM(transformer=cls(**kw))


@pytest.mark.parametrize("name", sorted(MA.CASES))
def test_state_dict_keys_equal_spec(name):
    cfg, _ = MA.CASES[name]
    model = _package_model(cfg)
    got = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    assert got == {k: shape for k, shape, _ in SD.state_dict_spec(cfg)}
    model.load_state_dict(SD.synthetic_state_dict(cfg, seed=1234), strict=True)
    tr = model.transformer
    assert (tr.qk_norm, tr.long_skip, tr.text_embedding_average_upsampling) == (
        cfg.qk_norm, cfg.long_skip_connection, cfg.text_embedding_average_upsampling)


def test_checkpoint_activations_is_accepted_and_ignored():
    cfg = MG.tiny_dit()
    a = _package_model(cfg, checkpoint_activations=True)
    b = _package_model(cfg)
    assert a.state_dict().keys() == b.state_dict().keys()


def test_constructor_rejections_match_reference():
    import f5_tts_b200 as F5

    with pytest.raises(ValueError):  # modules.py:408-409
        F5.DiT(dim=128, depth=2, heads=2, qk_norm="layer_norm")
    with pytest.raises(ValueError):
        F5.UNetT(dim=128, depth=2, heads=2, qk_norm="layer_norm")
    with pytest.raises(AssertionError):  # dit.py:41-43
        F5.DiT(dim=128, depth=2, heads=2, text_mask_padding=False, text_embedding_average_upsampling=True)
    for k in ("long_skip_connection", "text_embedding_average_upsampling"):  # not UNetT arguments (unett.py:109-128)
        with pytest.raises(TypeError):
            F5.UNetT(dim=128, depth=2, heads=2, **{k: True})
    F5.UNetT(dim=128, depth=2, heads=2, qk_norm="rms_norm")


@pytest.mark.skipif(not os.path.isdir(os.path.join(os.environ.get("F5_REFERENCE_SRC", "/nonexistent"), "f5_tts")),
                    reason="needs the reference checkout (F5_REFERENCE_SRC)")
def test_constructor_rejections_on_the_reference_itself():
    from oracle import ref_shims

    _, dit, unett, _, _ = ref_shims.import_reference()
    with pytest.raises(ValueError):
        dit.DiT(dim=128, depth=2, heads=2, qk_norm="layer_norm")
    with pytest.raises(AssertionError):
        dit.DiT(dim=128, depth=2, heads=2, text_mask_padding=False, text_embedding_average_upsampling=True)
    with pytest.raises(TypeError):
        unett.UNetT(dim=128, depth=2, heads=2, long_skip_connection=True)


# ---------------------------------------------------------------------------------------------------------------------
# options off: nothing moved
# ---------------------------------------------------------------------------------------------------------------------
# sha256 (first 16 hex digits) of synthetic_state_dict(cfg, 1234) — keys and float32 bytes — before the options existed
OFF_DIGESTS = {"tiny_dit": "94f01382c20a671f", "tiny_unett": "b4604bd29aac3f33",
               "f5tts_v1_small": "79ec23ab712dfb5b", "e2tts_small": "4a4759acb7fa7f31"}


@pytest.mark.parametrize("name", sorted(OFF_DIGESTS))
def test_options_off_state_dict_unchanged(name):
    cfg = {"tiny_dit": MG.tiny_dit, "tiny_unett": MG.tiny_unett, "f5tts_v1_small": SD.f5tts_v1_small,
           "e2tts_small": SD.e2tts_small}[name]()
    m = hashlib.sha256()
    for k, v in SD.synthetic_state_dict(cfg, seed=1234).items():
        m.update(k.encode())
        m.update(v.contiguous().numpy().tobytes())
    assert m.hexdigest()[:16] == OFF_DIGESTS[name]


def test_cache_key_arch_tuple(tmp_path):
    from f5_tts_b200 import weights as Wt

    ck = tmp_path / "model.safetensors"
    ck.write_bytes(b"x")
    st = os.stat(ck)
    off = _package_model(MG.tiny_dit()).transformer
    arch = (off.KIND, off.dim, off.depth, off.heads, off.dim_head, off.ff_inner, off.mel_dim, off.text_dim,
            off.text_num_embeds, off.conv_layers, off.text_mask_padding, off.pe_attn_head)
    raw = f"{os.path.abspath(ck)}|{st.st_size}|{st.st_mtime_ns}|{arch}|fmt{Wt.PACK_FORMAT}"
    assert Wt.cache_key(str(ck), off) == hashlib.sha256(raw.encode()).hexdigest()[:24]
    keys = {Wt.cache_key(str(ck), off)}
    for over in (dict(qk_norm="rms_norm"), dict(long_skip_connection=True),
                 dict(text_mask_padding=True, text_embedding_average_upsampling=True)):
        keys.add(Wt.cache_key(str(ck), _package_model(MG.tiny_dit(**over)).transformer))
    keys.add(Wt.cache_key(str(ck), _package_model(MG.tiny_dit(text_mask_padding=True)).transformer))
    assert len(keys) == 5
