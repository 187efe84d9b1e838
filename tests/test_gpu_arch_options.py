"""GPU: the architecture options no shipped config turns on — qk_norm="rms_norm" (DiT, UNetT), long_skip_connection and
text_embedding_average_upsampling (DiT).

  * EPI_QKV_NORM_ROPE (per-head RMSNorm + RoPE in the QKV GEMM epilogue) element by element against a float64
    reference on the same fp16 operands, at every instantiated tile width; its v section is bit-identical to
    EPI_QKV_ROPE's; malformed arguments are rejected;
  * end to end against the unmodified reference: the fixtures of oracle/make_golden_arch_options.py, rel-L2 <= 5e-3
    after step 1 and at the end;
  * exact_varlen with average upsampling and with the long skip equals a loop of B = 1 calls; two calls are
    bit-identical and graph replay equals eager launches; f5_sample_flops counts the long-skip GEMM;
  * infer.load_model on a checkpoint in the released layout with the options in the arch dict, and the packed-weight
    cache round trip of such a model.
"""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import f5_tts_b200 as F5  # noqa: E402
import synthdata as SD  # noqa: E402
from f5_tts_b200 import _lib, infer, ops  # noqa: E402
from f5_tts_b200.ops import EPI_QKV_NORM_ROPE, EPI_QKV_ROPE  # noqa: E402
from oracle import arch_options as OA  # noqa: E402
from oracle import f5_oracle as O  # noqa: E402
from oracle import make_golden as MG  # noqa: E402
from oracle import make_golden_arch_options as MA  # noqa: E402
from oracle import step_increment as SI  # noqa: E402

DEV = "cuda:0"
TOL = 5e-3
_models = {}


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def gen(shape, seed, scale=1.0, dtype=torch.float16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).to(DEV)


# ---------------------------------------------------------------------------------------------------------------------
# kernel
# ---------------------------------------------------------------------------------------------------------------------
def qkv_norm_rope_ref64(a, w, bias, cs, sn, seq, inner, pe_heads, qg, kg, lens):
    """float64 [M, 3 inner]: acc + bias; q and k heads RMSNorm(64, eps 1e-6) * gain, then RoPE on the first pe_heads
    heads (pairs (2i, 2i + 1) rotated by cos / sin[pos, i]); rows at or past their sample's length 0."""
    y = a.double().cpu() @ w.double().cpu().t() + bias.double().cpu()
    M, H = y.shape[0], inner // 64
    pos = torch.arange(M) % seq
    c, s = cs.double().cpu()[pos][:, None], sn.double().cpu()[pos][:, None]
    parts = []
    for sec, g in ((0, qg), (1, kg)):
        t = y[:, sec * inner:(sec + 1) * inner].reshape(M, H, 64)
        t = t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6) * g.double().cpu()
        x0, x1 = t[:, :pe_heads, 0::2], t[:, :pe_heads, 1::2]
        rot = torch.stack((x0 * c - x1 * s, x1 * c + x0 * s), dim=-1).flatten(-2)
        parts.append(torch.cat((rot, t[:, pe_heads:]), dim=1).reshape(M, inner))
    out = torch.cat(parts + [y[:, 2 * inner:]], dim=1)
    if lens is not None:
        keep = pos < lens.cpu().long()[torch.arange(M) // seq]
        out = torch.where(keep[:, None], out, torch.zeros_like(out))
    return out


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("pe", ["all", 1, 0])
@pytest.mark.parametrize("inner", [768, 1024])
@pytest.mark.parametrize("bn", [128, 192, 256])
def test_gemm_qkv_norm_rope(bn, inner, pe, masked):
    """Bound: one fp16 rounding of the output (2^-11 relative) over an fp32-accumulated, fp32-normalised value:
    |d| <= 2^-10 |ref| + 1e-4 max|ref| element by element.  M = 2 x 150 is not a multiple of 128."""
    seq, B = 150, 2
    M, K = B * seq, inner
    H = inner // 64
    pe_heads = H if pe == "all" else pe
    a = gen((M, K), 70)
    w = gen((3 * inner, K), 71, 1 / math.sqrt(K))
    bias = gen((3 * inner,), 72, 0.2, torch.float32)
    qg = gen((64,), 73, 0.1, torch.float32) + 1.0
    kg = gen((64,), 74, 0.1, torch.float32) + 1.0
    cs, sn = ops.rope_tables(seq, DEV)
    lens = torch.tensor([seq, 97], dtype=torch.int32, device=DEV) if masked else None
    kw = dict(bn=bn, seq=seq, rope=(cs, sn), inner=inner, pe_heads=pe_heads, row_len=lens)
    out = ops.linear(a, w, bias, epi=EPI_QKV_NORM_ROPE, qk_norm=(qg, kg), **kw)
    ref = qkv_norm_rope_ref64(a, w, bias, cs, sn, seq, inner, pe_heads, qg, kg, lens)
    d = (out.double().cpu() - ref).abs()
    bound = 2.0 ** -10 * ref.abs() + 1e-4 * float(ref.abs().max())
    print(f"[qkv_norm_rope bn{bn} inner{inner} pe{pe} masked{masked}] rel-L2 {rel(out, ref):.3e} "
          f"max|d| {float(d.max()):.3e} worst d/bound {float((d / bound).max()):.3f}")
    assert torch.isfinite(out).all() and bool((d <= bound).all())
    plain = ops.linear(a, w, bias, epi=EPI_QKV_ROPE, **kw)
    assert torch.equal(out[:, 2 * inner:], plain[:, 2 * inner:]), "the v section is EPI_QKV_ROPE's"


def test_gemm_qkv_norm_rope_planner_width():
    """bn = 0: the planner's width gives the same result as a forced one."""
    seq, inner = 469, 1024
    a, w = gen((2 * seq, inner), 75), gen((3 * inner, inner), 76, 1 / 32)
    bias, qg, kg = gen((3 * inner,), 77, 0.2, torch.float32), gen((64,), 78, 1.0, torch.float32), gen((64,), 79, 1.0,
                                                                                                     torch.float32)
    cs, sn = ops.rope_tables(seq, DEV)
    kw = dict(seq=seq, rope=(cs, sn), inner=inner, pe_heads=16, qk_norm=(qg, kg))
    bn, _ = ops.gemm_tile(2 * seq, 3 * inner, inner, epi=EPI_QKV_NORM_ROPE)
    assert bn in (128, 192, 256)
    o0 = ops.linear(a, w, bias, epi=EPI_QKV_NORM_ROPE, bn=0, **kw)
    o1 = ops.linear(a, w, bias, epi=EPI_QKV_NORM_ROPE, bn=bn, **kw)
    assert torch.equal(o0, o1)


def test_gemm_qkv_norm_rope_rejects_missing_operands():
    seq, inner = 64, 128
    a, w = gen((seq, inner), 80), gen((3 * inner, inner), 81)
    g = gen((64,), 82, 1.0, torch.float32)
    cs, sn = ops.rope_tables(seq, DEV)
    kw = dict(epi=EPI_QKV_NORM_ROPE, seq=seq, rope=(cs, sn), pe_heads=1)
    with pytest.raises(_lib.F5LibraryError):
        ops.linear(a, w, inner=inner, qk_norm=(g, None), **kw)
    with pytest.raises(_lib.F5LibraryError):
        ops.linear(a, w, inner=96, qk_norm=(g, g), **kw)
    ops.linear(a, w, inner=inner, qk_norm=(g, g), **kw)


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
def arch_kwargs(cfg):
    kw = dict(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
              mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim,
              text_mask_padding=cfg.text_mask_padding, conv_layers=cfg.conv_layers, pe_attn_head=cfg.pe_attn_head,
              attn_mask_enabled=cfg.attn_mask_enabled, qk_norm=cfg.qk_norm)
    if cfg.backbone == "DiT":
        kw.update(long_skip_connection=cfg.long_skip_connection,
                  text_embedding_average_upsampling=cfg.text_embedding_average_upsampling)
    return kw


def build(cfg: O.ArchConfig, wseed: int = 1234):
    key = (repr(cfg), wseed)
    if key not in _models:
        _models.clear()
        cls = F5.DiT if cfg.backbone == "DiT" else F5.UNetT
        model = F5.CFM(transformer=cls(**arch_kwargs(cfg)))
        sd = O.synthetic_state_dict(cfg, seed=wseed)
        model.load_state_dict(sd, strict=True)
        _models[key] = (model.to(DEV), sd)
    model, sd = _models[key]
    model.odeint_kwargs = dict(method="euler")
    model.use_cuda_graph = True
    return model, sd


@pytest.mark.parametrize("name", sorted(MA.CASES))
def test_sample_vs_reference_fixture(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg, kw = MA.CASES[name]
    model, _ = build(cfg, int(z["wseed"]))
    model.odeint_kwargs = dict(method=str(z["method"]))
    dur = z["duration"]
    duration = int(dur) if dur.ndim == 0 else torch.from_numpy(dur).long().to(DEV)
    lens = torch.from_numpy(z["lens"]).long().to(DEV) if z["lens"].size else None
    try:
        out, traj = model.sample(cond=torch.from_numpy(z["cond"]).to(DEV), text=torch.from_numpy(z["text"]).to(DEV),
                                 duration=duration, lens=lens, steps=int(z["steps"]),
                                 cfg_strength=float(z["cfg_strength"]), sway_sampling_coef=float(z["sway"]),
                                 seed=int(z["seed"]), y0=torch.from_numpy(z["y0"]).to(DEV))
    finally:
        model.odeint_kwargs = dict(method="euler")
    assert traj.shape[0] == int(z["steps"]) + 1 and out.shape == z["out"].shape
    SI.check(traj[1], z["y0"], z["traj_1"], z["duration"] if cfg.attn_mask_enabled else None, name)
    r1, rn = rel(traj[1], z["traj_1"]), rel(out, z["out"])
    print(f"[{name}] step-1 rel-L2 {r1:.3e}  final rel-L2 {rn:.3e}")
    assert r1 <= TOL and rn <= TOL


@pytest.mark.parametrize("option", ["text_embedding_average_upsampling", "long_skip_connection"])
def test_exact_varlen_batch_equals_single_calls(option):
    over = dict(text_mask_padding=True, text_embedding_average_upsampling=True) if option.startswith("text") else \
        dict(long_skip_connection=True)
    model, _ = build(MG.tiny_dit(**over))
    g = torch.Generator().manual_seed(90)
    n_ref, durs = 30, [211, 97, 150]
    cond = torch.randn(1, n_ref, 100, generator=g)
    text = torch.randint(0, 50, (3, 44), generator=g)
    text[1, 29:] = -1
    text[2, 37:] = -1
    y0 = [torch.randn(1, d, 100, generator=g) for d in durs]
    kw = dict(steps=3, cfg_strength=2.0, sway_sampling_coef=-1.0)
    singles = []
    for b, d in enumerate(durs):
        tb = text[b: b + 1, : int((text[b] != -1).sum())]
        o, _ = model.sample(cond.to(DEV), tb.to(DEV), d, **kw, y0=y0[b].to(DEV))
        singles.append(o)
    y0b = torch.zeros(3, max(durs), 100)
    for b, d in enumerate(durs):
        y0b[b, :d] = y0[b][0]
    out, _ = model.sample(cond.expand(3, -1, -1).contiguous().to(DEV), text.to(DEV), torch.tensor(durs).to(DEV),
                          lens=torch.full((3,), n_ref).to(DEV), **kw, y0=y0b.to(DEV), exact_varlen=True)
    for b, d in enumerate(durs):
        md = float((out[b, :d] - singles[b][0]).abs().max())
        print(f"[{option} exact_varlen] sample {b} ({d} frames): batched vs single max|d| {md:.3e}")
        assert torch.equal(out[b, :d], singles[b][0])


def test_all_options_graph_equals_eager_and_deterministic():
    model, _ = build(MA.big_all_options())
    g = torch.Generator().manual_seed(91)
    cond = torch.randn(2, 50, 100, generator=g).to(DEV)
    text = torch.randint(0, 2545, (2, 40), generator=g)
    text[1, 27:] = -1
    dur = torch.tensor([200, 163]).to(DEV)
    kw = dict(steps=3, cfg_strength=2.0, sway_sampling_coef=-1.0, lens=torch.tensor([50, 41]).to(DEV),
              y0=torch.randn(2, 200, 100, generator=g).to(DEV))
    try:
        model.odeint_kwargs = dict(method="midpoint")
        a, ta = model.sample(cond, text.to(DEV), dur, **kw)
        b, tb = model.sample(cond, text.to(DEV), dur, **kw)
        model.use_cuda_graph = False
        c, tc = model.sample(cond, text.to(DEV), dur, **kw)
    finally:
        model.use_cuda_graph = True
        model.odeint_kwargs = dict(method="euler")
    assert torch.isfinite(a).all()
    assert torch.equal(a, b) and torch.equal(ta, tb), "same inputs must be bit-identical run to run"
    assert torch.equal(a, c) and torch.equal(ta, tc), "graph replay and eager launches run the same kernels"


def test_sample_flops_count_the_long_skip_gemm():
    """long_skip_connection adds one Linear(2D -> D) per sample-forward: 2 n D (2 D) FLOPs, times NFE and the CFG batch."""
    plain, _ = build(MG.tiny_dit())
    f_plain = {c: plain.transformer.sample_flops(*c) for c in ((1, 300, 8, 2.0), (3, 128, 5, 0.0))}
    model, _ = build(MG.tiny_dit(long_skip_connection=True))
    D = 128
    for (B, N, nfe, cfg), base in f_plain.items():
        Be = 2 * B if cfg > 0 else B
        want = base + nfe * Be * 2 * N * D * 2 * D
        got = model.transformer.sample_flops(B, N, nfe, cfg)
        print(f"[long skip flops] B{B} N{N} nfe{nfe} cfg{cfg}: {got:.6e} vs {want:.6e}")
        assert abs(got - want) <= 1e-9 * want


# ---------------------------------------------------------------------------------------------------------------------
# loading: released checkpoint layout with the options in the arch dict, packed-weight cache
# ---------------------------------------------------------------------------------------------------------------------
ARCH = dict(dim=768, depth=4, heads=12, ff_mult=2, text_dim=512, text_mask_padding=True, conv_layers=4,
            pe_attn_head=None, qk_norm="rms_norm", long_skip_connection=True, text_embedding_average_upsampling=True,
            checkpoint_activations=True)  # a training config's arch block, passed as is


@pytest.fixture(scope="module")
def options_ckpt(tmp_path_factory):
    from safetensors.torch import save_file

    cfg = SD.ArchConfig(dim=768, depth=4, heads=12, text_mask_padding=True, pe_attn_head=None, qk_norm="rms_norm",
                        long_skip_connection=True, text_embedding_average_upsampling=True)
    sd = SD.synthetic_state_dict(cfg, seed=1234)
    ema = {"ema_model." + k: v for k, v in sd.items()}
    ema["initted"], ema["step"] = torch.tensor(True), torch.tensor(1)
    ckpt = str(tmp_path_factory.mktemp("f5opts") / "model_1.safetensors")
    save_file(ema, ckpt)
    return dict(cfg=cfg, sd=sd, ckpt=ckpt)


def test_load_model_with_options_vs_oracle(options_ckpt, golden_dir):
    _models.clear()
    a = options_ckpt
    m = infer.load_model(F5.DiT, ARCH, a["ckpt"], vocab_file=os.path.join(golden_dir, "vocab.txt"), device=DEV)
    tr = m.transformer
    assert (tr.qk_norm, tr.long_skip, tr.text_embedding_average_upsampling) == ("rms_norm", True, True)
    g = torch.Generator().manual_seed(92)
    cond = torch.randn(2, 40, 100, generator=g)
    text = torch.randint(0, 2545, (2, 30), generator=g)
    text[0, 21:] = -1
    dur, lens = torch.tensor([170, 139]), torch.tensor([40, 35])
    kw = dict(steps=3, cfg_strength=2.0, sway_sampling_coef=-1.0)
    ref = OA.sample(a["sd"], a["cfg"], cond, text, dur, lens=lens, **kw, seed=5)
    out, _ = m.sample(cond.to(DEV), text.to(DEV), dur.to(DEV), lens=lens.to(DEV), **kw, y0=ref.y0.to(DEV))
    r = rel(out, ref.out)
    print(f"[load_model options] final rel-L2 {r:.3e}")
    assert r <= TOL


def test_packed_cache_roundtrip_qk_norm(options_ckpt, golden_dir, tmp_path):
    import glob

    from f5_tts_b200 import weights as Wt

    _models.clear()
    a = options_ckpt
    vocab = os.path.join(golden_dir, "vocab.txt")
    cache = str(tmp_path / "pack")
    m1 = infer.load_model(F5.DiT, ARCH, a["ckpt"], vocab_file=vocab, device=DEV, packed_cache_dir=cache)
    files = glob.glob(os.path.join(cache, "f5pack_*.safetensors"))
    assert len(files) == 1
    from safetensors import safe_open

    with safe_open(files[0], framework="pt") as f:
        names = set(f.keys())
    assert {"L0.q_norm_w", "L0.k_norm_w", "L3.k_norm_w", "long_skip_w"} <= names
    calls = {"n": 0}
    orig = Wt.packed_tensors

    def counting(m):
        calls["n"] += 1
        return orig(m)

    Wt.packed_tensors = counting
    try:
        m2 = infer.load_model(F5.DiT, ARCH, a["ckpt"], vocab_file=vocab, device=DEV, packed_cache_dir=cache)
        g = torch.Generator().manual_seed(93)
        cond = torch.randn(1, 40, 100, generator=g).to(DEV)
        text = torch.randint(0, 2545, (1, 30), generator=g).to(DEV)
        y0 = torch.randn(1, 150, 100, generator=g).to(DEV)
        kw = dict(steps=2, cfg_strength=2.0, sway_sampling_coef=-1.0)
        o2, _ = m2.sample(cond, text, 150, **kw, y0=y0)
        assert calls["n"] == 0, "the second load must not re-pack"
    finally:
        Wt.packed_tensors = orig
    o1, _ = m1.sample(cond, text, 150, **kw, y0=y0)
    assert torch.equal(o1, o2)
