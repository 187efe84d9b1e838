"""float64 references of the GEMM epilogues, of attention and of the bandwidth-bound kernels' row norms, positions and
text embeddings, each with a per-element error bound for the sm_90a kernels.

Pure torch: the references run on whichever device their inputs are on (the GPU tests keep them on the H100, the CPU
test rehearses the bounds against an fp32 emulation of the kernels' arithmetic and against deliberately broken
variants of it).  Every function returns (value, bound): `value` is the exact result of the operation on the kernel's
own fp16 / fp32 inputs, evaluated in float64, and `bound` is the largest |kernel - value| the kernel's arithmetic can
produce under the error model in the docstring.  u = 2^-24 is the fp32 unit roundoff.

The bounds are first-order: products of two error terms (u^2 S and the like) are left out, and `SLACK` (one part in a
thousand of each bound) stands for them.  A bound is a worst case, so a correct kernel on random data stays well below
it; a result above it is either a kernel bug or a flaw in the error model, never a tolerance to widen.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import f5_oracle as O

U = 2.0 ** -24
F64 = torch.float64
SLACK = 1.001  # second-order terms of the first-order bounds below
# MUFU.EX2 (ex2.approx.ftz.f32): relative error taken as 2^-21, twice the 2^-22 the PTX ISA documents
EX2_REL = 2.0 ** -21
GELU_DMAX = 1.13  # max |d/dx gelu(x)| (1.1289 at x = 1.5, both forms)
MISH_DMAX = 1.1   # max |d/dx mish(x)| (1.0886 at x = 1.22)


# ---------------------------------------------------------------------------------------------------------------------
# comparison helpers
# ---------------------------------------------------------------------------------------------------------------------
def ulp16(x):
    """fp16 ulp at |x| (subnormal spacing 2^-24 below 2^-14)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


def half_bound(ref, e32):
    """Bound of an fp16 result: the fp32 bound e32 plus half an fp16 ulp, taken at |ref| + e32 (which covers a rounding
    across a binade)."""
    return e32 + 0.5 * ulp16(ref.abs() + e32)


def worst_ratio(got, ref, bound):
    """max |got - ref| / bound over all elements (NaN counts as infinitely far; a zero bound demands equality)."""
    got, ref = got.to(F64), ref.to(F64)
    err = (got - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))
    r = torch.where(torch.isnan(err), torch.full_like(err, math.inf), r)
    return float(r.max()) if r.numel() else 0.0


def assert_within(got, ref, bound, what):
    """Every element of got within bound of ref; returns the worst err / bound."""
    got, ref = got.to(F64), ref.to(F64)
    err = (got - ref).abs()
    bad = ~(err <= bound)  # also catches NaN
    if bool(bad.any()):
        i = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound; first at flat index "
                             f"{i}: got {float(got.flatten()[i])!r} ref {float(ref.flatten()[i])!r} "
                             f"bound {float(bound.flatten()[i]):.3e}")
    return worst_ratio(got, ref, bound)


def assert_half(got, ref, e32, what):
    """fp16 result: the fp32 bound plus half an fp16 ulp (taken at |ref| + e32, which covers a rounding across a binade)."""
    assert got.dtype == torch.float16
    return assert_within(got, ref, half_bound(ref, e32), what)


# ---------------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------------
def acc_bound(S, k16_steps):
    """Accumulation error of a wgmma GEMM over `k16_steps` k16 steps, S = sum_k |a_k| |w_k| (float64).

    Model: a k16 step adds 16 exact fp16 x fp16 products to the fp32 accumulator and truncates the sum to fp32 (round
    toward zero, not to nearest): one step errs by less than one fp32 ulp of the partial sum, <= 2u |partial sum| <=
    2u S.  The steps accumulate in fp32, so nothing is assumed about IEEE fp32 summation.  Two extra steps of slack
    cover the tails of the fragment.  How close Hopper's tensor cores come to this model has not been measured: the
    bound is a model of the hardware, and a ratio above 1 on the device would mean the model is wrong as much as that
    the kernel is.
        e_acc = (k16_steps + 2) * 2u * S"""
    return (k16_steps + 2) * 2.0 * U * S


def k16_steps(K):
    return -(-K // 16)


def linear_ref(a, w, bias=None, k16=None):
    """(y, e): y = a . w^T (+ bias) in float64 on the fp16 operands, and the bound of the kernel's fp32 value acc (+ bias).

    e = e_acc(S) + u (|y| + e_acc), S = |a| . |w|^T (+ |bias|): the accumulation bound of acc_bound, then one fp32
    rounding of the bias add.  k16: number of k16 steps (default ceil(K / 16))."""
    a64, w64 = a.to(F64), w.to(F64)
    y = a64 @ w64.t()
    S = a64.abs() @ w64.abs().t()
    if bias is not None:
        b = bias.to(F64)
        y = y + b
        S = S + b.abs()
    e = acc_bound(S, k16_steps(a.shape[-1]) if k16 is None else k16)
    return y, e + U * (y.abs() + e)


def gelu_tanh_ref(y, e):
    """(gelu_tanh(y), bound) for the kernel's x / (1 + 2^t), t = x (c0 + c1 x^2) (ex2.approx, __fdividef).

    Propagated input error: |gelu'| <= 1.13.  Arithmetic: t = x * fmaf(x^2, c1, c0) with c0, c1 rounded to fp32 is off
    by at most 6u |t|, and MUFU.EX2 adds EX2_REL relative; an error d in ln(1 + 2^t)'s exponent moves the result by
    |x| s (1 - s) |d ln 2|, s = 1 / (1 + 2^t).  1 + e and __fdividef (2 ulp) add 5u |result|.  Where 2^t overflows the
    result is 0 against a true value below 2^-120 |x|."""
    t = y * (-2.0 * math.sqrt(2.0 / math.pi) / math.log(2.0)) * (1.0 + 0.044715 * y * y)
    s = torch.sigmoid(-t * math.log(2.0))
    z = y * s
    arith = y.abs() * s * (1.0 - s) * (6.0 * U * t.abs() * math.log(2.0) + EX2_REL) + 5.0 * U * z.abs() + 1e-30
    return z, GELU_DMAX * e + arith


def gelu_erf_ref(y, e):
    """(gelu_erf(y), bound) for the kernel's 0.5 x (1 + erff(x * 0.70710678f)).

    Propagated input error: |gelu'| <= 1.13.  Arithmetic: the argument z is off by 2u |z| (rounded constant and
    product), which moves erf by 2/sqrt(pi) e^-z^2 2u |z|; erff errs by at most 2 ulp <= 4u |erf z|; 1 + erf rounds
    once (u |1 + erf|); the products by 0.5 and x round once (u |result|)."""
    z = y * math.sqrt(0.5)
    ez = torch.erf(z)
    out = 0.5 * y * (1.0 + ez)
    d_erf = 2.0 / math.sqrt(math.pi) * torch.exp(-z * z) * 2.0 * U * z.abs() + 4.0 * U * ez.abs()
    arith = 0.5 * y.abs() * (d_erf + U * (1.0 + ez).abs()) + 2.0 * U * out.abs()
    return out, GELU_DMAX * e + arith


def mish_ref(y, e):
    """(mish(y), bound) for the kernel's x tanhf(log1pf(__expf(x))) (softplus = x above 20).

    Propagated input error: |mish'| <= 1.1.  Arithmetic: __expf errs by 2 + 1.173 |x| ulp (CUDA programming guide),
    <= (4 + 2.35 |x|) u relative, which moves softplus by that times e^x / (1 + e^x); log1pf adds 1 ulp (2u |sp|);
    tanhf (1 - tanh^2) times the softplus error plus 2 ulp (4u |tanh|); the product u |result|."""
    sp = torch.nn.functional.softplus(y)
    th = torch.tanh(sp)
    out = y * th
    sig = torch.sigmoid(y)
    e_sp = torch.where(y > 20.0, torch.zeros_like(y), (4.0 + 2.35 * y.abs()) * U * sig + 2.0 * U * sp)
    e_th = (1.0 - th * th) * e_sp + 4.0 * U * th.abs()
    return out, MISH_DMAX * e + y.abs() * e_th + U * out.abs()


def resid_ref(x, g, y, e):
    """(x + g y, bound) of the residual epilogue: x, g fp32 (g = 1 for no gate), y with bound e.

    g (y + d) is rounded once and added to x with one more rounding (or one fused rounding):
        |g| e + 2u (|x| + |g y|)"""
    x64 = x.to(F64)
    g64 = torch.ones((), dtype=F64, device=y.device) if g is None else g.to(F64)
    gy = g64 * y
    return x64 + gy, g64.abs() * e + 2.0 * U * (x64.abs() + gy.abs())


def rope_ref(y, e, cos, sin, pos, inner, pe_heads, dh):
    """(rope(y), bound) of the QKV epilogue's rotary step over y [M, 3 inner]: the first pe_heads heads of the q and k
    sections have column pairs (2i, 2i + 1) rotated by cos / sin[pos, i] (fp32 tables, taken as exact inputs).

        v0 = x0 c - x1 s, v1 = x1 c + x0 s:   |c| e0 + |s| e1 + 2u (|x0 c| + |x1 s|)     (two products, one sum)
    Other columns pass through unchanged."""
    M = y.shape[0]
    H = inner // dh
    c = cos.to(F64)[pos][:, None, :]  # [M, 1, dh / 2]
    s = sin.to(F64)[pos][:, None, :]
    out, eo = y.clone(), e.clone()
    for sec in (0, 1):
        cols = slice(sec * inner, sec * inner + pe_heads * dh)
        t = y[:, cols].reshape(M, pe_heads, dh)
        te = e[:, cols].reshape(M, pe_heads, dh)
        x0, x1, e0, e1 = t[..., 0::2], t[..., 1::2], te[..., 0::2], te[..., 1::2]
        r0, r1 = x0 * c - x1 * s, x1 * c + x0 * s
        ar = 2.0 * U * ((x0 * c).abs() + (x1 * s).abs())
        ar1 = 2.0 * U * ((x1 * c).abs() + (x0 * s).abs())
        out[:, cols] = torch.stack((r0, r1), -1).reshape(M, -1)
        eo[:, cols] = torch.stack((c.abs() * e0 + s.abs() * e1 + ar, c.abs() * e1 + s.abs() * e0 + ar1), -1).reshape(M, -1)
    return out, eo


def rms_norm_heads_ref(y, e, q_gain, k_gain, inner, dh):
    """(norm(y), bound) of the QKV epilogue's per-head RMSNorm of the q and k sections of y [M, 3 inner]:
    v * rsqrt(mean(v^2) + 1e-6) * gain over each dh-column head.

    With ss = sum y^2 over the head: the kernel's fp32 sum of squares of y + d (|d| <= e) errs by at most
    2 sum |y| e + sum e^2 + (dh + 1) u sum y^2 (products, then a sum of dh terms); dividing by dh is exact (a power of
    two), adding the fp32 1e-6 rounds once and differs from 1e-6 by |1e-6f - 1e-6|.  rsqrtf errs by 2 ulp (4u
    relative), and half of m's relative error reaches r = m^-1/2.  The two products round once each:
        |v r g - y r g| <= |y r g| (rel_r + 2u) + |g| r e (1 + rel_r)"""
    M = y.shape[0]
    H = inner // dh
    out, eo = y.clone(), e.clone()
    eps32 = float(torch.tensor(1e-6, dtype=torch.float32))
    for sec, gain in ((0, q_gain), (1, k_gain)):
        cols = slice(sec * inner, (sec + 1) * inner)
        t = y[:, cols].reshape(M, H, dh)
        te = e[:, cols].reshape(M, H, dh)
        g = gain.to(F64)
        ss = (t * t).sum(-1, keepdim=True)
        d_ss = 2.0 * (t.abs() * te).sum(-1, keepdim=True) + (te * te).sum(-1, keepdim=True) + (dh + 1) * U * ss
        m = ss / dh + 1e-6
        rel_m = (d_ss / dh + U * m + abs(eps32 - 1e-6)) / m
        r = torch.rsqrt(m)
        rel_r = 0.5 * rel_m + 4.0 * U
        z = t * r * g
        out[:, cols] = z.reshape(M, inner)
        eo[:, cols] = (z.abs() * (rel_r + 2.0 * U) + g.abs() * r * te * (1.0 + rel_r)).reshape(M, inner)
    return out, eo


def row_mask(M, seq, row_len, device):
    """[M] bool: row m (sample m // seq, position m % seq) lies before its sample's length."""
    pos = torch.arange(M, device=device) % seq
    return pos < row_len.to(device).long()[torch.arange(M, device=device) // seq]


def qkv_ref(a, w, bias, cos, sin, seq, inner, pe_heads, dh, norm=None, row_len=None):
    """(out, bound) of the QKV epilogues before the fp16 store: linear_ref, the optional per-head RMSNorm
    (norm = (q gain, k gain)), RoPE at position m % seq, rows at or past their sample's length exactly 0."""
    y, e = linear_ref(a, w, bias)
    M = y.shape[0]
    if norm is not None:
        y, e = rms_norm_heads_ref(y, e, norm[0], norm[1], inner, dh)
    pos = torch.arange(M, device=y.device) % seq
    y, e = rope_ref(y, e, cos, sin, pos, inner, pe_heads, dh)
    if row_len is not None:
        keep = row_mask(M, seq, row_len, y.device)[:, None]
        y, e = torch.where(keep, y, 0.0), torch.where(keep, e, 0.0)
    return y, e


def conv31_ref(x, w_packed, bias, G):
    """(y, e) of the grouped conv GEMM before its activation: y[b, n, c] = sum_t sum_i x[b, n + t - 15, g G + i]
    w_packed[t, c, i] + bias[c] (zero outside [0, N)), g = c // G, in float64.

    Each tap is one 64-column k-block (G <= 64 channels, the rest zero-filled), so 31 ceil(G / 16) k16 steps carry
    non-zero products; the bound is linear_ref's with that count."""
    B, N, D = x.shape
    taps = w_packed.shape[0]
    pad = taps // 2
    x64 = torch.nn.functional.pad(x.to(F64), (0, 0, pad, pad))
    w64 = w_packed.to(F64).view(taps, D // G, G, G)  # [t, group, out in group, in]
    y = torch.zeros((B, N, D // G, G), dtype=F64, device=x.device)
    S = torch.zeros_like(y)
    for t in range(taps):
        xs = x64[:, t:t + N].reshape(B, N, D // G, G)
        y += torch.einsum("bngi,goi->bngo", xs, w64[t])
        S += torch.einsum("bngi,goi->bngo", xs.abs(), w64[t].abs())
    b = bias.to(F64)
    y = y.reshape(B, N, D) + b
    S = S.reshape(B, N, D) + b.abs()
    e = acc_bound(S, taps * k16_steps(G))
    return y, e + U * (y.abs() + e)


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
def attention_ref(q, k, v, kv_len=None, scale=None, block_kv=128):
    """(o, bound) of softmax(scale q k^T) v over the first kv_len[b] keys, float64 on the fp16 q, k, v [B, H, seq, dh].

    Error model of the flash-attention kernel (fp32 scores from wgmma, online softmax with MUFU.EX2 in log2 units, P
    rounded to fp16 for P V, the row sum l of the unrounded exponentials, o / l rounded to fp16):
      * score error δs_j (natural-log units): the GEMM model at K = dh on scale |q| |k|, 3u |s_j| for scale * log2(e)
        rounded to fp32 and the product, u (m - s_j) for rounding the exponent relative to the running max m
        (subtracting m is exact in effect: the same m scales the numerator and l, as does every rescale factor), and
        EX2_REL for MUFU.EX2.  To first order it moves o by  sum_j p_j |δs_j| |v_j - o|  <=  sum_j p_j |δs_j| (|v_j| + |o|).
      * P to fp16 (in P V only, not in l):  sum_j (2^-11 p_j + 2^-25) |v_j|,  the 2^-25 for fp16 subnormals (P is at
        most 1 per tile, and l >= 1).
      * ε_pv, the P V accumulation: the GEMM model over ceil(kv / 16) k16 steps plus two roundings per rescaled key
        tile, on sum_j p_j |v_j|.
      * l: a 32-term fp32 sum per thread and tile, a rescale and add per tile, two quad shuffles; then 1 / l and the
        product (IEEE): (36 + 2 tiles) u |o|.
      * the fp16 store: half an fp16 ulp of |o| + e.
    Keys at or past kv_len have p = 0 exactly (their scores are -inf) and contribute nothing."""
    B, H, seq, dh = q.shape
    scale = dh ** -0.5 if scale is None else scale
    q64, k64, v64 = q.to(F64), k.to(F64), v.to(F64)
    dev = q.device
    if kv_len is None:
        kv = torch.full((B,), seq, dtype=torch.long, device=dev)
    else:
        kv = kv_len.to(dev).long().clamp(1, seq)
    keep = (torch.arange(seq, device=dev)[None, :] < kv[:, None])[:, None, None, :]  # [B, 1, 1, keys]
    s = scale * (q64 @ k64.transpose(-1, -2))
    s = s.masked_fill(~keep, -math.inf)
    p = torch.softmax(s, dim=-1)
    v0 = torch.where(keep[..., 0, :, None], v64, 0.0)  # [B, 1, keys, 1] mask: rows past kv_len are not inputs
    o = p @ v0
    sabs = q64.abs() @ k64.abs().transpose(-1, -2)
    smax = s.amax(-1, keepdim=True)
    ds = scale * acc_bound(sabs, k16_steps(dh)) + 3.0 * U * s.abs() + U * (smax - s) + EX2_REL
    ds = torch.where(keep, ds, 0.0)
    pd = p * ds
    av = v0.abs()
    b1 = pd @ av + pd.sum(-1, keepdim=True) * o.abs()
    b2 = (2.0 ** -11) * (p @ av) + (2.0 ** -25) * (keep.to(F64) @ av)
    tiles = (-(-kv // block_kv)).to(F64)[:, None, None, None]
    steps = (kv.to(F64) / 16.0).ceil()[:, None, None, None]
    b3 = (steps + 2.0 * tiles + 2.0) * 2.0 * U * (p @ av)
    b4 = (36.0 + 2.0 * tiles) * U * o.abs()
    e = SLACK * (b1 + b2 + b3 + b4)
    return o, half_bound(o, e)


# ---------------------------------------------------------------------------------------------------------------------
# bandwidth-bound kernels: row norms, depthwise conv, sinusoidal positions, text embeddings
# ---------------------------------------------------------------------------------------------------------------------
def gam(n):
    return n * U / (1.0 - n * U)


def ln_ref_bound(a, e_a, w, b, eps, depth):
    """LayerNorm over the last axis of the exact pre-norm values `a` (float64), y = (a - mean) * rstd * w + b, and a
    per-element bound on the kernel's fp32 y when its fp32 copy of `a` is off by at most `e_a`.

    The kernel sums in fp32 with `depth` = terms per lane + 5 warp-shuffle levels:
      mean:  e_mean = mean(e_a) + g(depth + 1) * mean|a|                  (sum of C terms, one division)
      d:     e_d    = e_a + e_mean + u |d|                                (subtraction)
      var:   e_var  = mean(2 |d| e_d + e_d^2) + g(depth + 2) * var        (squares, sum, division)
      rstd:  rho    = (e_var / (var + eps) + u) / 2 + 4 u                 (relative; +eps, rsqrtf within 2 ulp)
      y:     e_y    = |w| rstd (e_d + |d| rho) + 3 u |d rstd w| + u |y|   (two products, w itself rounded once, + b)
    """
    mean = a.mean(-1, keepdim=True)
    d = a - mean
    var = (d * d).mean(-1, keepdim=True)
    rstd = (var + eps).rsqrt()
    y = d * rstd * w + b
    e_mean = e_a.mean(-1, keepdim=True) + gam(depth + 1) * a.abs().mean(-1, keepdim=True)
    e_d = e_a + e_mean + U * d.abs()
    e_var = (2 * d.abs() * e_d + e_d * e_d).mean(-1, keepdim=True) + gam(depth + 2) * var
    rho = 0.5 * (e_var / (var + eps) + U) + 4 * U
    e_y = w.abs() * rstd * (e_d + d.abs() * rho) + 3 * U * (d * rstd * w).abs() + U * y.abs()
    return y, e_y


def pos_bound(ang):
    """cos / sin of ang = n * 10000^(-2i/dim), fp32: the exponent 2i/dim (u, times ln 1e4 < 9.3), powf (2 ulp = 4u), the
    reciprocal (u) and the product n * freq (u) give |d ang| <= 16 u * ang; cosf / sinf add 2 ulp <= 4 u.  Bound used:
    20 u * ang + 8 u."""
    return 20 * U * ang + 8 * U


def dwconv7_ref(x, w, wb):
    """Depthwise Conv1d(k=7, pad=3) along the sequence of x [B, N, C] (float64), w [C, 7]; returns (a, sum|terms|)."""
    B, N, C = x.shape
    xp = F.pad(x, (0, 0, 3, 3))
    a = wb.expand(B, N, C).clone()
    s = wb.abs().expand(B, N, C).clone()
    for t in range(7):
        a = a + w[:, t] * xp[:, t:t + N]
        s = s + (w[:, t] * xp[:, t:t + N]).abs()
    return a, s


def mmdit_text_embed_ref(table, ids, Be, mask_padding):
    """(out, bound) of the MMDiT text embedding (backbones/mmdit.py:31-63) of ids [B, nt] (-1 padded) over the fp32
    table [V + 1, D]; out [Be, nt, D] with Be = B (cond) or 2 B (cond, then uncond, whose ids are all 0):
        out[v, b, n] = table[id + 1] + cat(cos, sin)(ang),   ang = min(n, 1023) * 10000^(-2i/D)
    (precompute_freqs_cis(D, 1024), get_pos_embed_indices clamps at 1023), and 0 where the real text's id is -1 when
    mask_padding, in both variants.  Bound: pos_bound(ang) for the fp32 angle and cosf / sinf, plus u |out| for the one
    rounded addition; zeroed rows are exact (bound 0)."""
    B, nt = ids.shape
    D = table.shape[1]
    dev = table.device
    ids = ids.to(dev).long()
    idx = torch.cat((ids + 1, torch.zeros_like(ids)), 0)[:Be]
    freq = 10000.0 ** (-torch.arange(D // 2, dtype=F64, device=dev) * 2 / D)
    a = torch.arange(nt, dtype=F64, device=dev).clamp(max=1023)[:, None] * freq[None]
    out = table.to(F64)[idx] + torch.cat((a.cos(), a.sin()), -1)
    keep = (ids != -1) if mask_padding else torch.ones_like(ids, dtype=torch.bool)
    keep = torch.cat((keep, keep), 0)[:Be, :, None]
    bound = pos_bound(torch.cat((a, a), -1)) + U * out.abs()
    return torch.where(keep, out, 0.0), torch.where(keep, bound, 0.0)


def avg_upsample_index(valid, audio_len, N):
    """[B, N] source row of every output row of text average upsampling (backbones/dit.py:55-84), -1 where the row is 0.
    Sample b's T valid text rows (the positions set in valid [B, K], in order) are spread over its first
    A = min(audio_len[b], N) rows with dit.py's own loop: token j repeated A // T times, once more when
    j >= T - A % T, cut at A.  Rows at or past A, and every row when T = 0, are 0.  Pure index arithmetic: the kernel's
    copy of the selected rows must match bit for bit."""
    B = valid.shape[0]
    src = torch.full((B, N), -1, dtype=torch.long)
    for b in range(B):
        rows = torch.nonzero(valid[b].cpu()).flatten()
        T, A = rows.numel(), min(int(audio_len[b]), N)
        if T == 0 or A <= 0:
            continue
        base, rem = divmod(A, T)
        reps = torch.tensor([base + (1 if j >= T - rem else 0) for j in range(T)], dtype=torch.long)
        src[b, :A] = rows.repeat_interleave(reps)[:A]
    return src


def istft_ref(head, T):
    """(wav, bound) of the Vocos ISTFT head (istft_frames + istft_ola) over head [B T, 1026] (log-magnitude | phase of
    T >= 2 frames per sample, float64): the oracle's istft_center (== torch.istft(center=True)) of the spectrum
    clipped at magnitude 100, wav [B, 256 (T - 1)].

    Bound: per frame, A_t = (|X_0| + |X_512| + 2 sum_k |X_k|) / 1024 bounds |x_n|.  The input (expf, sincosf: 3 x 4 u)
    and ten radix-2 stages (about 6 u each with table twiddles) put at most 100 u A_t on each frame sample; the window,
    the <= 4-term overlap-add and the division by the envelope add 8 u of sum_t |w_n x_t,n| / env.  So
    |d wav_i| <= (sum_t w_n (100 u A_t + 8 u |x_t,n|)) / env_i."""
    nb = 513
    B = head.shape[0] // T
    mag = torch.exp(head[:, :nb]).clamp(max=100.0)
    spec = torch.polar(mag, head[:, nb:]).view(B, T, nb).transpose(1, 2)  # [B, F, T]
    win = torch.hann_window(1024, periodic=True, dtype=F64)
    ref = O.istft_center(spec, window=win)
    a = (mag[:, 0] + mag[:, nb - 1] + 2 * mag[:, 1:nb - 1].sum(-1)) / 1024  # [B T]
    x = torch.fft.irfft(spec, n=1024, dim=1)  # [B, 1024, T]
    per = win[None, :, None] * (100 * U * a.view(B, 1, T) + 8 * U * x.abs())
    L = 1024 + 256 * (T - 1)
    num = F.fold(per, output_size=(1, L), kernel_size=(1, 1024), stride=(1, 256))[:, 0, 0, 512:L - 512]
    env = F.fold((win ** 2)[None, :, None].expand(1, 1024, T), output_size=(1, L), kernel_size=(1, 1024),
                 stride=(1, 256))[:, 0, 0, 512:L - 512]
    return ref, num / env
