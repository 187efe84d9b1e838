"""The per-element bounds of oracle/kernel_bounds.py against an fp32 emulation of the GEMM and attention kernels'
arithmetic, and against broken variants of it (CPU).

The emulation follows the error model the bounds are derived from: fp16 operands, each k16 step adding 16 exact
products to an fp32 accumulator with truncation toward zero, the epilogue in fp32, fp16 stores rounding to nearest.
It must lie within every bound.  Each mutant is one mistake a rewrite of an epilogue or of the softmax could make
(a stray fp16 rounding, a lost bias, a lost K tail, an off-by-one row or column, a wrong rotary position, the gate row
of the wrong ODE evaluation, unnormalised P) and must fall outside its bound somewhere.  A bound loose enough to let
one of them through would let the same bug through on the GPU.
"""
import math

import pytest
import torch

from oracle import kernel_bounds as KB

F32, F64 = torch.float32, torch.float64


def rnd(shape, seed, scale=1.0, dtype=torch.float16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=F64) * scale).to(dtype)


def trunc32(x):
    """float64 -> fp32 rounded toward zero."""
    f = x.to(F32)
    over = f.to(F64).abs() > x.abs()
    return torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f)


def emu_acc(a, w, k_end=None):
    """fp32 accumulator of the wgmma main loop: k16 steps of exact products, truncated to fp32 after each step.
    k_end: stop before this column (a mutant that loses the K tail)."""
    K = a.shape[1] if k_end is None else k_end
    a64, w64 = a.to(F64), w.to(F64)
    acc = torch.zeros((a.shape[0], w.shape[0]), dtype=F32)
    for k0 in range(0, K, 16):
        k1 = min(k0 + 16, K)
        acc = trunc32(acc.to(F64) + a64[:, k0:k1] @ w64[:, k0:k1].t())
    return acc


def emu_gelu_tanh(x):
    c0, c1 = torch.tensor(-2.3022081981, dtype=F32), torch.tensor(-0.1029432396, dtype=F32)
    return x / (1.0 + torch.exp2(x * (x * x * c1 + c0)))


def emu_gelu_erf(x):
    return 0.5 * x * (1.0 + torch.erf(x * torch.tensor(0.7071067811865476, dtype=F32)))


def emu_rope(v, cos, sin, pos, inner, pe_heads, dh):
    out = v.clone()
    c, s = cos[pos][:, None, :], sin[pos][:, None, :]
    for sec in (0, 1):
        cols = slice(sec * inner, sec * inner + pe_heads * dh)
        t = v[:, cols].reshape(v.shape[0], pe_heads, dh)
        x0, x1 = t[..., 0::2], t[..., 1::2]
        out[:, cols] = torch.stack((x0 * c - x1 * s, x1 * c + x0 * s), -1).reshape(v.shape[0], -1)
    return out


def emu_rms_norm(v, qg, kg, inner, dh):
    out = v.clone()
    for sec, g in ((0, qg), (1, kg)):
        cols = slice(sec * inner, (sec + 1) * inner)
        t = v[:, cols].reshape(v.shape[0], -1, dh)
        r = torch.rsqrt((t * t).sum(-1, keepdim=True) * (1.0 / dh) + torch.tensor(1e-6, dtype=F32))
        out[:, cols] = (t * r * g).reshape(v.shape[0], inner)
    return out


def rope_tables(seq, dh):
    inv = 1.0 / (10000 ** (torch.arange(0, dh, 2).float() / dh))
    ang = torch.outer(torch.arange(seq).float(), inv)
    return ang.cos(), ang.sin()


def check(good, mutants, ref, bound):
    """good within the bound, every mutant outside it; returns (good ratio, {mutant: ratio})."""
    r = KB.worst_ratio(good, ref, bound)
    assert r <= 1.0, f"the emulated kernel is outside its bound (worst err / bound {r:.3f})"
    out = {}
    for name, m in mutants.items():
        out[name] = KB.worst_ratio(m, ref, bound)
        print(f"  mutant {name}: worst err / bound {out[name]:.3g}")
        assert out[name] > 1.0, f"mutant '{name}' passes the bound (worst err / bound {out[name]:.3f})"
    print(f"  emulation: worst err / bound {r:.3f}")
    return r, out


# ---------------------------------------------------------------------------------------------------------------------
# GEMM epilogues
# ---------------------------------------------------------------------------------------------------------------------
def test_resid_gate_mask_mutants():
    """The shapes of the rel-L2 test of the residual epilogue (K = 2048, gate, bias, row mask) at fewer rows and
    columns: four mutants that pass its rel-L2 <= 2e-4 fall outside the per-element bound."""
    seq, lens, N, K = 64, [64, 50, 1], 256, 2048
    M = seq * len(lens)
    a, w = rnd((M, K), 7), rnd((N, K), 8, 1 / math.sqrt(K))
    bias, gate = rnd((N,), 9, 0.3, F32), rnd((N,), 10, 0.5, F32)
    x0 = rnd((M, N), 11, 1.0, F32)
    keep = KB.row_mask(M, seq, torch.tensor(lens), "cpu")[:, None]
    y, e = KB.linear_ref(a, w, bias)
    ref, bound = KB.resid_ref(x0, gate, y, e)
    ref, bound = torch.where(keep, ref, x0.to(F64)), torch.where(keep, bound, 0.0)

    acc = emu_acc(a, w)
    v = acc + bias

    def resid(x, g, v):
        return torch.where(keep, x + g * v, x)

    nb = v.clone()
    j = int(bias.abs().argmax())
    nb[M // 2, j] = acc[M // 2, j]
    mutants = {
        "GEMM result rounded to fp16": resid(x0, gate, v.half().float()),
        "residual read through fp16": resid(x0.half().float(), gate, v),
        "gate rounded to fp16": resid(x0, gate.half().float(), v),
        "one element missing its bias": resid(x0, gate, nb),
        "K tail block missing": resid(x0, gate, emu_acc(a, w, K - 64) + bias),
    }
    check(resid(x0, gate, v), mutants, ref, bound)


def test_f32_and_f16_epilogue_mutants():
    """EPI_F32 with an N and K tail (K = 712, the input projection's width): an output rounded through fp16, a lost K
    tail (the 8 columns past 704), the last row or column written off by one.  EPI_F16 with GELU (tanh and erf)."""
    M, N, K = 200, 100, 712
    a, w = rnd((M, K), 20), rnd((N, K), 21, 1 / math.sqrt(K))
    bias = rnd((N,), 22, 0.5, F32)
    y, e = KB.linear_ref(a, w, bias)
    v = emu_acc(a, w) + bias
    row = v.clone()
    row[-1] = v[-2]
    col = v.clone()
    col[:, -1] = 0.0
    mutants = {
        "fp32 output rounded to fp16": v.half().float(),
        "K tail (8 columns) missing": emu_acc(a, w, 704) + bias,
        "last tail row from the row before": row,
        "last tail column not stored": col,
    }
    check(v, mutants, y, e)
    for ref_fn, emu in ((KB.gelu_tanh_ref, emu_gelu_tanh), (KB.gelu_erf_ref, emu_gelu_erf)):
        z, ez = ref_fn(y, e)
        out = emu(v).half()
        check(out, {"no bias": emu(v - bias).half(), "activation of the fp16-rounded input": emu(v.half().float()).half()},
              z, KB.half_bound(z, ez))


def test_mish_bound_holds():
    M, N, K = 128, 64, 31 * 64
    a, w = rnd((M, K), 30, 1.0), rnd((N, K), 31, 2 / math.sqrt(K))
    bias = rnd((N,), 32, 0.5, F32)
    y, e = KB.linear_ref(a, w, bias)
    v = emu_acc(a, w) + bias
    z, ez = KB.mish_ref(y, e)
    out = (v * torch.tanh(torch.where(v > 20.0, v, torch.log1p(torch.exp(v))))).half()
    check(out, {"no activation": v.half()}, z, KB.half_bound(z, ez))


@pytest.mark.parametrize("dh,norm", [(64, False), (64, True), (128, False), (128, True)])
def test_qkv_epilogue_mutants(dh, norm):
    """QKV + (RMSNorm) + RoPE with masked rows: a rotary position off by one, and (RMSNorm) the norm taken before the
    bias, fall outside the bound."""
    seq, lens, H, K = 40, [40, 23], 2, 256
    inner = H * dh
    M = seq * len(lens)
    a, w = rnd((M, K), 40 + dh), rnd((3 * inner, K), 41, 1 / math.sqrt(K))
    bias = rnd((3 * inner,), 42, 0.2, F32)
    gains = (rnd((dh,), 43, 0.1, F32) + 1.0, rnd((dh,), 44, 0.1, F32) + 1.0) if norm else None
    cos, sin = rope_tables(seq, dh)
    row_len = torch.tensor(lens)
    ref, e = KB.qkv_ref(a, w, bias, cos, sin, seq, inner, H, dh, gains, row_len)
    keep = KB.row_mask(M, seq, row_len, "cpu")[:, None]
    pos = torch.arange(M) % seq

    def epi(acc, b, pos):
        v = acc + b
        if norm:
            v = emu_rms_norm(v, gains[0], gains[1], inner, dh)
        v = emu_rope(v, cos, sin, pos, inner, H, dh)
        return torch.where(keep, v, 0.0).half()

    acc = emu_acc(a, w)
    mutants = {"RoPE position + 1": epi(acc, bias, (pos + 1) % seq)}
    if norm:
        mutants["norm before the bias"] = epi(acc, 0.0, pos) + torch.where(keep, bias, 0.0).half()
    check(epi(acc, bias, pos), mutants, ref, KB.half_bound(ref, e))


def test_gate_of_the_wrong_step():
    """step_ptr selects row k of a [S, N] gate table: the gate of row k - 1 falls outside the bound."""
    M, N, K, k = 128, 192, 512, 2
    a, w = rnd((M, K), 50), rnd((N, K), 51, 1 / math.sqrt(K))
    table = rnd((4, N), 52, 0.5, F32)
    x0 = rnd((M, N), 53, 1.0, F32)
    y, e = KB.linear_ref(a, w)
    ref, bound = KB.resid_ref(x0, table[k], y, e)
    v = emu_acc(a, w)
    check(x0 + table[k] * v, {"gate row k - 1": x0 + table[k - 1] * v}, ref, bound)


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
def emu_attention(q, k, v, kv_len, scale, rescale=True, normalise=True):
    """The kernel's online softmax over 128-key tiles, per (sample, head): fp32 scores from the k16 model, exponents
    relative to the running max in log2 units, P rounded to fp16 for P V, l from the unrounded exponentials."""
    B, H, seq, dh = q.shape
    out = torch.zeros((B, H, seq, dh), dtype=torch.float16)
    sl2 = torch.tensor(scale, dtype=F32) * torch.tensor(1.4426950408889634, dtype=F32)
    for b in range(B):
        n = int(kv_len[b])
        for h in range(H):
            m = torch.full((seq, 1), -math.inf, dtype=F32)
            l = torch.zeros((seq, 1), dtype=F32)
            o = torch.zeros((seq, dh), dtype=F32)
            for j0 in range(0, n, 128):
                j1 = min(j0 + 128, n)
                sc = emu_acc(q[b, h], k[b, h, j0:j1])
                m_new = torch.maximum(m, sc.amax(-1, keepdim=True) * sl2)
                alpha = torch.exp2(m - m_new)
                p = torch.exp2(sc * sl2 - m_new)
                l = l * alpha + p.sum(-1, keepdim=True)
                if rescale:
                    o = o * alpha
                pv = emu_acc(p.half(), v[b, h, j0:j1].t().contiguous())
                o = trunc32(o.to(F64) + pv.to(F64))
                m = m_new
            out[b, h] = (o / l if normalise else o).half()
    return out


@pytest.mark.parametrize("mode", ["plain", "rising"])
def test_attention_bound_and_mutants(mode):
    """Two key tiles, one sample with a key length inside the second: the emulation lies within the bound; P V without
    the rescale by exp2(m_old - m_new) when the running max grows, or without the division by l, lies outside."""
    B, H, seq, dh = 2, 1, 200, 64
    q, k, v = (rnd((B, H, seq, dh), 60 + i) for i in range(3))
    if mode == "rising":  # every key tile larger than the one before: the running max moves at the second tile
        k = (k.double() * (1.0 + torch.arange(seq, dtype=F64)[:, None] / 64.0)).half()
    kv_len = torch.tensor([seq, 150])
    scale = dh ** -0.5
    ref, bound = KB.attention_ref(q, k, v, kv_len, scale)
    good = emu_attention(q, k, v, kv_len, scale)
    mutants = {"P not renormalised (no division by l)": emu_attention(q, k, v, kv_len, scale, normalise=False)}
    if mode == "rising":
        mutants["no rescale when the running max grows"] = emu_attention(q, k, v, kv_len, scale, rescale=False)
    check(good, mutants, ref, bound)


def test_bounds_reject_nan_and_accept_exact():
    ref = torch.tensor([1.0, -2.0, 0.0], dtype=F64)
    bound = torch.tensor([1e-3, 1e-3, 0.0], dtype=F64)
    assert KB.worst_ratio(ref, ref, bound) == 0.0
    assert KB.worst_ratio(torch.tensor([1.0, float("nan"), 0.0]), ref, bound) == math.inf
    assert KB.worst_ratio(torch.tensor([1.0, -2.0, 1e-30]), ref, bound) > 1.0  # a zero bound demands equality
    with pytest.raises(AssertionError):
        KB.assert_within(torch.tensor([1.0, float("nan"), 0.0]), ref, bound, "nan")
