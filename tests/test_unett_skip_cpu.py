"""CPU: UNetT checkpoints built with skip_connect_type="add" or "none" (backbones/unett.py:127, 286-297).

  * the oracle (oracle/unett_skip.py) reproduces the unmodified reference on the fixtures of
    oracle/make_golden_unett_skip.py (rel-L2 0.0 at generation time, bound 1e-6 here), and the three types give three
    different results;
  * the package's UNetT accepts the three values and rejects any other with ValueError; DiT and MMDiT reject the
    argument with TypeError;
  * the state-dict keys of each type are the reference module's (no `layers.{i}.0.weight` without concat), so such a
    checkpoint loads with strict=True;
  * the packed-weight cache key tells the types apart and is unchanged for concat.
"""
import hashlib
import os
import re

import numpy as np
import pytest
import torch

import synthdata as SD
from oracle import f5_oracle as O
from oracle import make_golden as MG
from oracle import make_golden_arch_options as MA
from oracle import make_golden_unett_skip as MU
from oracle import unett_skip as OU
from test_arch_options_cpu import cfg_from_repr

TOL = 1e-6
TYPES = ("concat", "add", "none")
HAS_REFERENCE = os.path.isdir(os.path.join(os.environ.get("F5_REFERENCE_SRC", "/nonexistent"), "f5_tts"))


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _oracle(cfg, kw, sd=None):
    sd = O.synthetic_state_dict(cfg, seed=1234) if sd is None else sd
    cond, text, duration, lens = MA.case_inputs(cfg, **kw)
    return OU.sample(sd, cfg, cond, text, duration, lens=lens, method=kw.get("method", "euler"), steps=kw["steps"],
                     cfg_strength=kw["cfg_strength"], sway_sampling_coef=kw["sway"], seed=kw["seed"])


@pytest.mark.parametrize("name", sorted(MU.CASES))
def test_oracle_reproduces_unett_skip_fixture(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg, kw = MU.CASES[name]
    assert cfg_from_repr(str(z["cfg"])) == cfg and str(z["method"]) == kw.get("method", "euler")
    res = _oracle(cfg, kw)
    assert torch.equal(res.y0, torch.from_numpy(z["y0"]))
    r1, rn = _rel(res.trajectory[1], torch.from_numpy(z["traj_1"])), _rel(res.out, torch.from_numpy(z["out"]))
    print(f"[{name}] oracle vs reference: step-1 rel-L2 {r1:.3e}  final {rn:.3e}")
    assert r1 <= TOL and rn <= TOL


def test_the_three_types_differ():
    """Same weights apart from the concat projections: add, none and concat give three different generated states."""
    _, kw = MU.CASES["unett_skip_add_b2_varlen"]
    sd = O.synthetic_state_dict(MG.tiny_unett(), seed=1234)  # concat: a superset of the add / none keys
    out = {t: _oracle(MG.tiny_unett(skip_connect_type=t), kw, sd).trajectory[-1] for t in TYPES}
    for a, b in (("add", "none"), ("add", "concat"), ("none", "concat")):
        print(f"[{a} vs {b}] rel-L2 {_rel(out[a], out[b]):.3e}")
        assert _rel(out[a], out[b]) > 1e-3


def test_concat_default_unchanged():
    """The field's default is concat, and with concat this oracle computes exactly what oracle/arch_options.py (which
    the existing UNetT fixtures pin) does."""
    from oracle import arch_options as OA

    assert SD.ArchConfig().skip_connect_type == "concat"
    assert MG.tiny_unett() == MG.tiny_unett(skip_connect_type="concat")
    cfg, (_, kw) = MG.tiny_unett(qk_norm="rms_norm"), MU.CASES["unett_skip_add_b2_varlen"]
    sd = O.synthetic_state_dict(cfg, seed=1234)
    cond, text, duration, lens = MA.case_inputs(cfg, **kw)
    skw = dict(lens=lens, steps=2, cfg_strength=2.0, sway_sampling_coef=-1.0, seed=3)
    ours, theirs = OU.sample(sd, cfg, cond, text, duration, **skw), OA.sample(sd, cfg, cond, text, duration, **skw)
    assert torch.equal(ours.trajectory, theirs.trajectory)


# ---------------------------------------------------------------------------------------------------------------------
# constructors and checkpoint layout
# ---------------------------------------------------------------------------------------------------------------------
def _unett(cfg):
    import f5_tts_b200 as F5

    return F5.CFM(transformer=F5.UNetT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head,
                                       ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds,
                                       text_dim=cfg.text_dim, text_mask_padding=cfg.text_mask_padding,
                                       conv_layers=cfg.conv_layers, pe_attn_head=cfg.pe_attn_head,
                                       attn_mask_enabled=cfg.attn_mask_enabled, qk_norm=cfg.qk_norm,
                                       skip_connect_type=cfg.skip_connect_type))


def test_constructor_accepts_the_three_types():
    import f5_tts_b200 as F5

    for t in TYPES:
        assert F5.UNetT(dim=128, depth=2, heads=2, skip_connect_type=t).skip_connect_type == t
    assert F5.UNetT(dim=128, depth=2, heads=2).skip_connect_type == "concat"
    assert F5.DiT(dim=128, depth=2, heads=2).skip_connect_type is None


@pytest.mark.parametrize("bad", ["Add", "concatenate", "", None, 1])
def test_constructor_rejects_other_values(bad):
    """The reference runs any other value like "none" (it compares against "concat" and "add" only); here it raises."""
    import f5_tts_b200 as F5

    with pytest.raises(ValueError):
        F5.UNetT(dim=128, depth=2, heads=2, skip_connect_type=bad)


@pytest.mark.parametrize("t", TYPES)
def test_dit_and_mmdit_reject_the_argument(t):
    import f5_tts_b200 as F5

    with pytest.raises(TypeError):
        F5.DiT(dim=128, depth=2, heads=2, skip_connect_type=t)
    with pytest.raises(TypeError):
        F5.MMDiT(dim=128, depth=2, heads=2, skip_connect_type=t)


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("depth", [4, 3])
def test_state_dict_keys_equal_spec(t, depth):
    cfg = MG.tiny_unett(depth=depth, skip_connect_type=t)
    model = _unett(cfg)
    got = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    assert got == {k: shape for k, shape, _ in SD.state_dict_spec(cfg)}
    skip_proj = {k for k in got if re.fullmatch(r"transformer\.layers\.\d+\.0\.weight", k)}
    assert len(skip_proj) == (depth - depth // 2 if t == "concat" else 0)
    model.load_state_dict(SD.synthetic_state_dict(cfg, seed=1234), strict=True)


@pytest.mark.skipif(not HAS_REFERENCE, reason="needs the reference checkout (F5_REFERENCE_SRC)")
@pytest.mark.parametrize("t", TYPES)
def test_state_dict_keys_equal_the_reference_module(t):
    from oracle import ref_shims

    _, _, unett, _, _ = ref_shims.import_reference()
    kw = dict(dim=128, depth=4, heads=2, ff_mult=4, mel_dim=100, text_num_embeds=50, text_mask_padding=False,
              pe_attn_head=1, qk_norm="rms_norm")
    ref = unett.UNetT(**kw, skip_connect_type=t)
    cfg = MG.tiny_unett(qk_norm="rms_norm", skip_connect_type=t)
    ours = _unett(cfg).transformer
    want = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    assert {k: tuple(v.shape) for k, v in ours.state_dict().items()} == want


@pytest.mark.skipif(not HAS_REFERENCE, reason="needs the reference checkout (F5_REFERENCE_SRC)")
def test_reference_runs_an_unknown_type_like_none():
    """The deviation this package makes on purpose: the reference builds no skip_proj for any value but "concat" and
    then combines nothing unless the value is "add"."""
    from oracle import ref_shims

    _, _, unett, _, _ = ref_shims.import_reference()
    kw = dict(dim=128, depth=2, heads=2, mel_dim=100, text_num_embeds=50)
    assert unett.UNetT(**kw, skip_connect_type="bogus").state_dict().keys() == \
        unett.UNetT(**kw, skip_connect_type="none").state_dict().keys()


# ---------------------------------------------------------------------------------------------------------------------
# packed-weight cache key and C ABI struct
# ---------------------------------------------------------------------------------------------------------------------
def test_cache_key_tells_the_types_apart(tmp_path):
    from f5_tts_b200 import weights as Wt

    ck = tmp_path / "model.safetensors"
    ck.write_bytes(b"x")
    st = os.stat(ck)
    concat = _unett(MG.tiny_unett()).transformer
    arch = (concat.KIND, concat.dim, concat.depth, concat.heads, concat.dim_head, concat.ff_inner, concat.mel_dim,
            concat.text_dim, concat.text_num_embeds, concat.conv_layers, concat.text_mask_padding, concat.pe_attn_head)
    raw = f"{os.path.abspath(ck)}|{st.st_size}|{st.st_mtime_ns}|{arch}|fmt{Wt.PACK_FORMAT}"
    assert Wt.cache_key(str(ck), concat) == hashlib.sha256(raw.encode()).hexdigest()[:24], "concat keys unchanged"
    keys = {t: Wt.cache_key(str(ck), _unett(MG.tiny_unett(skip_connect_type=t)).transformer) for t in TYPES}
    keys["add+qk"] = Wt.cache_key(str(ck), _unett(MG.tiny_unett(skip_connect_type="add", qk_norm="rms_norm")).transformer)
    keys["concat+qk"] = Wt.cache_key(str(ck), _unett(MG.tiny_unett(qk_norm="rms_norm")).transformer)
    assert len(set(keys.values())) == len(keys), keys


def test_arch_struct_ends_with_skip_type():
    """f5_arch.skip_type is the struct's last field, so a zeroed struct (a caller that never sets it) gets concat."""
    from f5_tts_b200 import _lib

    assert _lib.Arch._fields_[-1] == ("skip_type", _lib.c_int)
    assert _lib.Arch().skip_type == 0 and _lib.SKIP_TYPES == {"concat": 0, "add": 1, "none": 2}
