"""GPU: DiT / UNetT checkpoints built with 128-wide attention heads (dim_head=128).

  * attention (f5_attention_dh at 128) against a float64 softmax(q k^T / sqrt(128)) v on the same fp16 operands, with
    and without a key mask, at sequence and key lengths that are not multiples of the 128-key tile;
  * the QKV GEMM epilogues (RoPE, RMSNorm + RoPE) over 128-column heads element by element against float64, at every
    tile width the planner can pick for them, with rotary on all heads and on the first one only;
  * end to end against the unmodified reference: the fixtures of oracle/make_golden_dim_head.py, rel-L2 <= 5e-3 after
    step 1 and at the end; exact_varlen equals a loop of B = 1 calls bit for bit; graph replay equals eager launches;
  * f5_sample_flops counts the attention width heads * dim_head.
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
from f5_tts_b200 import _lib, ops  # noqa: E402
from f5_tts_b200.ops import EPI_QKV_NORM_ROPE, EPI_QKV_ROPE  # noqa: E402
from oracle import f5_oracle as O  # noqa: E402
from oracle import make_golden as MG  # noqa: E402
from oracle import make_golden_dim_head as MD  # noqa: E402
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
# attention
# ---------------------------------------------------------------------------------------------------------------------
def attention_ref64(qkv, B, seq, H, dh, kv_len):
    x = qkv.double().cpu().view(B, seq, 3, H, dh).permute(2, 0, 3, 1, 4)  # [3, B, H, seq, dh]
    q, k, v = x[0], x[1], x[2]
    s = q @ k.transpose(-1, -2) / math.sqrt(dh)
    if kv_len is not None:
        keep = torch.arange(seq)[None, :] < kv_len.cpu().long()[:, None]  # [B, seq keys]
        s = s.masked_fill(~keep[:, None, None, :], float("-inf"))
    o = torch.softmax(s, dim=-1) @ v  # [B, H, seq, dh]
    return o.permute(0, 2, 1, 3).reshape(B * seq, H * dh)


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("seq", [90, 469, 1875])
def test_attention_dh128_vs_float64(seq, masked):
    B, H, dh = 2, 8, 128
    qkv = gen((B * seq, 3 * H * dh), 200 + seq, 1.0)
    # key lengths that end inside a 128-key tile; one sample keeps all its keys
    kv = torch.tensor([seq, max(1, seq - 77)], dtype=torch.int32, device=DEV) if masked else None
    out = ops.attention(qkv, B, seq, H, kv_len=kv, dim_head=dh)
    ref = attention_ref64(qkv, B, seq, H, dh, kv)
    r = rel(out, ref)
    print(f"[attention dh128 seq{seq} masked{masked}] rel-L2 {r:.3e}")
    assert torch.isfinite(out).all() and r <= 3e-3


def test_attention_dh64_through_dh_entry_point_is_f5_attention():
    B, seq, H = 2, 469, 16
    qkv = gen((B * seq, 3 * H * 64), 210)
    kv = torch.tensor([469, 300], dtype=torch.int32, device=DEV)
    a = ops.attention(qkv, B, seq, H, kv_len=kv)
    out = torch.empty_like(a)
    with torch.cuda.device(DEV):
        _lib.check(_lib.lib().f5_attention_dh(qkv.data_ptr(), out.data_ptr(), B, seq, H, 64, kv.data_ptr(), 0.125,
                                              torch.cuda.current_stream().cuda_stream), "f5_attention_dh")
    torch.cuda.synchronize()
    assert torch.equal(a, out)


def test_attention_rejects_other_widths():
    qkv = gen((128, 3 * 2 * 96), 211)
    out = torch.empty((128, 2 * 96), dtype=torch.float16, device=DEV)
    rc = _lib.lib().f5_attention_dh(qkv.data_ptr(), out.data_ptr(), 1, 128, 2, 96, None, 0.1,
                                    torch.cuda.current_stream().cuda_stream)
    assert rc == -1 and b"dim_head" in _lib.lib().f5_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# QKV epilogues over 128-column heads
# ---------------------------------------------------------------------------------------------------------------------
def qkv_ref64(a, w, bias, cs, sn, seq, inner, pe_heads, dh, norm, lens):
    """float64 [M, 3 inner]: acc + bias; with norm, q and k heads RMSNorm(dh, eps 1e-6) * gain; RoPE on the first
    pe_heads heads of q and k (pairs (2i, 2i + 1) rotated by cos / sin[pos, i], i < dh / 2); rows at or past their
    sample's length 0."""
    y = a.double().cpu() @ w.double().cpu().t() + bias.double().cpu()
    M, H = y.shape[0], inner // dh
    pos = torch.arange(M) % seq
    c, s = cs.double().cpu()[pos][:, None], sn.double().cpu()[pos][:, None]
    parts = []
    for sec in (0, 1):
        t = y[:, sec * inner:(sec + 1) * inner].reshape(M, H, dh)
        if norm is not None:
            t = t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6) * norm[sec].double().cpu()
        x0, x1 = t[:, :pe_heads, 0::2], t[:, :pe_heads, 1::2]
        rot = torch.stack((x0 * c - x1 * s, x1 * c + x0 * s), dim=-1).flatten(-2)
        parts.append(torch.cat((rot, t[:, pe_heads:]), dim=1).reshape(M, inner))
    out = torch.cat(parts + [y[:, 2 * inner:]], dim=1)
    if lens is not None:
        keep = pos < lens.cpu().long()[torch.arange(M) // seq]
        out = torch.where(keep[:, None], out, torch.zeros_like(out))
    return out


QKV_CASES = [(EPI_QKV_ROPE, bn) for bn in (128, 192, 256)] + [(EPI_QKV_NORM_ROPE, 128)]


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("pe", ["all", 1])
@pytest.mark.parametrize("inner", [512, 1024])
@pytest.mark.parametrize("epi,bn", QKV_CASES)
def test_gemm_qkv_epilogue_dh128(epi, bn, inner, pe, masked):
    """Bound: one fp16 rounding of the output (2^-11 relative) over an fp32-accumulated value:
    |d| <= 2^-10 |ref| + 1e-4 max|ref| element by element, and rel-L2 <= 1.5e-3.  M = 2 x 150 is not a multiple of
    128."""
    seq, B, dh, K = 150, 2, 128, 1024
    M = B * seq
    H = inner // dh
    pe_heads = H if pe == "all" else pe
    a = gen((M, K), 220)
    w = gen((3 * inner, K), 221, 1 / math.sqrt(K))
    bias = gen((3 * inner,), 222, 0.2, torch.float32)
    norm = None
    if epi == EPI_QKV_NORM_ROPE:
        norm = (gen((dh,), 223, 0.1, torch.float32) + 1.0, gen((dh,), 224, 0.1, torch.float32) + 1.0)
    cs, sn = ops.rope_tables(seq, DEV, dim_head=dh)
    lens = torch.tensor([seq, 97], dtype=torch.int32, device=DEV) if masked else None
    out = ops.linear(a, w, bias, epi=epi, bn=bn, seq=seq, rope=(cs, sn), inner=inner, pe_heads=pe_heads, row_len=lens,
                     qk_norm=norm, dim_head=dh)
    ref = qkv_ref64(a, w, bias, cs, sn, seq, inner, pe_heads, dh, norm, lens)
    d = (out.double().cpu() - ref).abs()
    bound = 2.0 ** -10 * ref.abs() + 1e-4 * float(ref.abs().max())
    r = rel(out, ref)
    print(f"[qkv epi{epi} dh128 bn{bn} inner{inner} pe{pe} masked{masked}] rel-L2 {r:.3e} "
          f"worst d/bound {float((d / bound).max()):.3f}")
    assert torch.isfinite(out).all() and bool((d <= bound).all()) and r <= 1.5e-3


def test_gemm_qkv_dh128_planner_and_rejections():
    seq, inner, dh = 469, 1024, 128
    M = 2 * seq
    bn, _ = ops.gemm_tile(M, 3 * inner, inner, epi=EPI_QKV_NORM_ROPE, dim_head=dh)
    assert bn == 128, "a head must not straddle a tile"
    assert ops.gemm_tile(M, 3 * inner, inner, epi=EPI_QKV_ROPE, dim_head=dh)[0] in (128, 192, 256)
    a, w = gen((M, inner), 230), gen((3 * inner, inner), 231, 1 / 32)
    g = gen((dh,), 232, 1.0, torch.float32)
    cs, sn = ops.rope_tables(seq, DEV, dim_head=dh)
    kw = dict(seq=seq, rope=(cs, sn), inner=inner, pe_heads=8, dim_head=dh)
    o0 = ops.linear(a, w, epi=EPI_QKV_NORM_ROPE, qk_norm=(g, g), **kw)
    o1 = ops.linear(a, w, epi=EPI_QKV_NORM_ROPE, qk_norm=(g, g), bn=128, **kw)
    assert torch.equal(o0, o1)
    for bad in (dict(bn=192), dict(bn=256)):
        with pytest.raises(_lib.F5LibraryError):
            ops.linear(a, w, epi=EPI_QKV_NORM_ROPE, qk_norm=(g, g), **kw, **bad)
    with pytest.raises(_lib.F5LibraryError):  # inner not a multiple of 128
        ops.linear(a, w[: 3 * 960], epi=EPI_QKV_ROPE, **{**kw, "inner": 960})
    with pytest.raises(_lib.F5LibraryError):  # 128 only for the QKV epilogues
        ops.linear(a, w, dim_head=128)


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
def build(cfg: O.ArchConfig, wseed: int = 1234):
    key = (repr(cfg), wseed)
    if key not in _models:
        _models.clear()
        cls = F5.DiT if cfg.backbone == "DiT" else F5.UNetT
        kw = dict(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
                  mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim,
                  text_mask_padding=cfg.text_mask_padding, conv_layers=cfg.conv_layers,
                  pe_attn_head=cfg.pe_attn_head, attn_mask_enabled=cfg.attn_mask_enabled, qk_norm=cfg.qk_norm)
        model = F5.CFM(transformer=cls(**kw))
        sd = O.synthetic_state_dict(cfg, seed=wseed)
        model.load_state_dict(sd, strict=True)
        _models[key] = model.to(DEV)
    model = _models[key]
    model.odeint_kwargs = dict(method="euler")
    model.use_cuda_graph = True
    return model


@pytest.mark.parametrize("name", sorted(MD.CASES))
def test_sample_vs_reference_fixture(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg, _ = MD.CASES[name]
    model = build(cfg, int(z["wseed"]))
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


@pytest.mark.parametrize("backbone", ["DiT", "UNetT"])
def test_exact_varlen_batch_equals_single_calls(backbone):
    cfg = (MG.tiny_dit if backbone == "DiT" else MG.tiny_unett)(dim_head=128, qk_norm="rms_norm")
    model = build(cfg)
    g = torch.Generator().manual_seed(240)
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
        print(f"[{backbone} dh128 exact_varlen] sample {b} ({d} frames): batched vs single max|d| {md:.3e}")
        assert torch.equal(out[b, :d], singles[b][0])


def test_graph_equals_eager_and_attn_mask_nocfg():
    """Full width (8 heads of 128), midpoint, key-masked attention, with and without CFG: graph replay and eager
    launches give the same bits, and two calls agree."""
    cfg = MD.full_width()
    cfg.attn_mask_enabled = True
    model = build(cfg)
    g = torch.Generator().manual_seed(241)
    cond = torch.randn(2, 50, 100, generator=g).to(DEV)
    text = torch.randint(0, 2545, (2, 40), generator=g)
    text[1, 27:] = -1
    dur = torch.tensor([200, 163]).to(DEV)
    y0 = torch.randn(2, 200, 100, generator=g).to(DEV)
    for cfg_strength in (2.0, 0.0):
        kw = dict(steps=3, cfg_strength=cfg_strength, sway_sampling_coef=-1.0, lens=torch.tensor([50, 41]).to(DEV),
                  y0=y0)
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
        assert torch.equal(a, b) and torch.equal(ta, tb)
        assert torch.equal(a, c) and torch.equal(ta, tc)


def test_sample_flops_count_the_attention_width():
    """DiT: 8 n D I for QKV and the out-projection and 4 n^2 I for attention, I = heads * dim_head."""
    m64 = build(MG.tiny_dit(heads=4)).transformer  # I = 256 = 2 D
    f64 = {c: m64.sample_flops(*c) for c in ((1, 300, 8, 2.0), (3, 128, 5, 0.0))}
    m128 = build(MG.tiny_dit(heads=2, dim_head=128)).transformer  # the same I
    D, Ld = 128, 2
    for (B, N, nfe, cfg), base in f64.items():
        Be = 2 * B if cfg > 0 else B
        # the dim_head 64 count takes I = D
        want = base + nfe * Be * Ld * (8.0 * N * D * (256 - D) + 4.0 * N * N * (256 - D))
        got = m128.sample_flops(B, N, nfe, cfg)
        print(f"[dh128 flops] B{B} N{N} nfe{nfe} cfg{cfg}: {got:.6e} vs {want:.6e}")
        assert abs(got - want) <= 1e-9 * want
