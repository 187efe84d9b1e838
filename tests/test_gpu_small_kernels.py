"""Element-by-element GPU tests of the bandwidth-bound and FFT kernels (csrc/elementwise.cuh, csrc/fft.cuh) against
float64 references of the same operation.

The kernels are launched one at a time through libf5tts_b200_kernels.so (csrc/kernel_hooks.cu): the product's own
objects and launchers plus one extern "C" wrapper per launcher.  The mel front-end is tested through the public
f5_mel_spectrogram of libf5tts_b200.so.

Tolerances, per element (u = 2^-24, the fp32 unit roundoff; g(n) = n u / (1 - n u)):
- data movement (pack / concat / prepend / mask / im2col / gather without positions) is bit-exact; fp32 -> fp16 is
  __float2half_rn, which equals torch's .half();
- fp32 results: a bound derived from the operation in each test's docstring, e.g. g(n) * sum|terms| for an n-term sum;
- fp16 results: that bound plus half an fp16 ulp of the reference (one rounding).
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from f5_tts_b200 import _lib, ops  # noqa: E402
from oracle import f5_oracle as O  # noqa: E402
from oracle.kernel_bounds import (assert_half, assert_within, dwconv7_ref, gam, istft_ref,  # noqa: E402,F401
                                  ln_ref_bound, pos_bound, ulp16)

DEV = "cuda:0"
U = 2.0 ** -24
F64 = torch.float64


# ---------------------------------------------------------------------------------------------------------------------
# ctypes binding of the kernel hooks
# ---------------------------------------------------------------------------------------------------------------------
_P, _I, _F, _LL = C.c_void_p, C.c_int, C.c_float, C.c_longlong
_SIGS = {
    "f5k_row_norm": [_I, _P, _P, _I, _I, _F, _P, _P, _P, _LL, _I],
    "f5k_dwconv7_ln": [_P, _P, _I, _I, _I, _P, _P, _P, _P, _F],
    "f5k_text_gather": [_P, _I, _I, _I, _I, _P, _P, _I, _I, _P, _P],
    "f5k_mask_rows": [_P, _P, _I, _I, _I],
    "f5k_mask_rows_len": [_P, _I, _P, _I, _I, _I, _I],
    "f5k_grn": [_P, _P, _P, _P, _P, _I, _I, _I],
    "f5k_pack_input": [_P, _I, _I, _I, _I, _I, _I, _P, _P, _P],
    "f5k_cfg_euler": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I],
    "f5k_small_linear": [_I, _P, _P, _P, _P, _I, _I, _I],
    "f5k_time_features": [_P, _P, _I, _I],
    "f5k_silu_to_half": [_P, _P, _LL],
    "f5k_rope_table": [_P, _P, _I, _I],
    "f5k_prepend_time_token": [_P, _P, _P, _P, _I, _I, _LL],
    "f5k_concat_half": [_P, _P, _P, _LL, _I],
    "f5k_vocos_im2col": [_P, _I, _I, _I, _P, _I],
    "f5k_ln_affine_f32": [_P, _P, _I, _I, _F, _P, _P],
    "f5k_istft": [_P, _I, _P, _P, _I, _I],
}
_hooks = None


def hooks():
    global _hooks
    if _hooks is None:
        L = C.CDLL(_lib.KERNELS_LIB_PATH)
        L.f5k_last_error.restype = C.c_char_p
        L.f5k_grn_rows.restype = _I
        for name, args in _SIGS.items():
            getattr(L, name).argtypes = args + [_P]  # + stream
            getattr(L, name).restype = _I
        _hooks = L
    return _hooks


def launch(name, *args):
    """Call hook `name` on the current stream; tensors pass their data pointer, None a null pointer."""
    conv = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    rc = getattr(hooks(), name)(*conv, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, f"{name} failed (rc={rc}): {hooks().f5k_last_error().decode()}"


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def rnd(shape, seed, scale=1.0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=F64) * scale).to(dtype).to(DEV)


def assert_equal(got, ref, what):
    if not torch.equal(got, ref):
        d = torch.nonzero(got != ref)
        raise AssertionError(f"{what}: {d.shape[0]} elements differ, first at {d[0].tolist()}: "
                             f"got {got[tuple(d[0])].item()!r} ref {ref[tuple(d[0])].item()!r}")


def grn_ref(v, gamma, beta):
    """modules.py:236-245 (oracle convnext_v2_block): Gx = ||v[b, :, c]||_2 over the sequence, Nx = Gx / (mean_c Gx + 1e-6)"""
    gx = torch.linalg.vector_norm(v, ord=2, dim=1, keepdim=True)
    nx = gx / (gx.mean(dim=-1, keepdim=True) + 1e-6)
    return gamma * (v * nx) + beta + v, nx


# ---------------------------------------------------------------------------------------------------------------------
# references vs the oracle
# ---------------------------------------------------------------------------------------------------------------------
def test_references_match_oracle():
    """The float64 restatements used below equal the oracle's convnext_v2_block (dwconv + LN, GRN) run in float64, and
    the fp32-only oracle tables (abs_pos_table, sinus_time_features) lie within the stated position bounds."""
    g = torch.Generator().manual_seed(0)
    C, N = 64, 9
    sd = {"p.dwconv.weight": torch.randn(C, 1, 7, generator=g, dtype=F64), "p.dwconv.bias": torch.randn(C, generator=g, dtype=F64),
          "p.norm.weight": torch.randn(C, generator=g, dtype=F64), "p.norm.bias": torch.randn(C, generator=g, dtype=F64),
          "p.pwconv1.weight": torch.randn(2 * C, C, generator=g, dtype=F64) / 8, "p.pwconv1.bias": torch.randn(2 * C, generator=g, dtype=F64),
          "p.grn.gamma": torch.randn(2 * C, generator=g, dtype=F64), "p.grn.beta": torch.randn(2 * C, generator=g, dtype=F64),
          "p.pwconv2.weight": torch.randn(C, 2 * C, generator=g, dtype=F64) / 11, "p.pwconv2.bias": torch.randn(C, generator=g, dtype=F64)}
    x = torch.randn(2, N, C, generator=g, dtype=F64)
    ref = O.convnext_v2_block(sd, "p.", x)
    a, _ = dwconv7_ref(x, sd["p.dwconv.weight"][:, 0], sd["p.dwconv.bias"])
    h, _ = ln_ref_bound(a, torch.zeros_like(a), sd["p.norm.weight"], sd["p.norm.bias"], 1e-6, 1)
    h = F.gelu(F.linear(h, sd["p.pwconv1.weight"], sd["p.pwconv1.bias"]))
    h, _ = grn_ref(h, sd["p.grn.gamma"], sd["p.grn.beta"])
    mine = x + F.linear(h, sd["p.pwconv2.weight"], sd["p.pwconv2.bias"])
    assert float((mine - ref).abs().max()) <= 1e-12 * float(ref.abs().max())
    for dim, n in ((512, 4096), (100, 4096)):
        freq = 10000.0 ** (-torch.arange(dim // 2, dtype=F64) * 2 / dim)
        ang = torch.arange(n, dtype=F64)[:, None] * freq[None]
        pos = torch.cat((ang.cos(), ang.sin()), -1)
        assert_within(O.abs_pos_table(dim, n), pos, pos_bound(torch.cat((ang, ang), -1)), f"abs_pos_table {dim}")


# ---------------------------------------------------------------------------------------------------------------------
# text path
# ---------------------------------------------------------------------------------------------------------------------
V = 2545  # text_num_embeds: table rows V + 1


@pytest.mark.parametrize("Td,B,nt,N,lens,add_pos", [
    (512, 3, 40, 300, "mixed", 1),   # nt < N, per-sample valid lengths 1 / mid / N
    (512, 2, 500, 300, None, 1),     # nt > N: crop
    (100, 3, 40, 300, "mixed", 0),
    (100, 2, 500, 300, None, 0),
    (100, 2, 4100, 4000, None, 1),   # positions up to 3999
    (512, 2, 3000, 4000, "long", 1),
])
def test_text_gather(Td, B, nt, N, lens, add_pos):
    """text_gather_kernel against a float64 gather of the same table.  Without positions the fp32 output is the table
    row itself (bit-exact).  With positions, out = table[id] + cos/sin(n * 10000^(-2i/Td)): pos_bound(ang) for the
    fp32 angle and cosf / sinf, plus u |out| for the addition.  Rows past a sample's valid length are exactly 0 and the
    filler mask (id == 0 before the drop) is exact."""
    g = torch.Generator().manual_seed(Td + N + nt)
    table = rnd((V + 1, Td), 1, 0.5)
    ids = torch.randint(0, V, (B, nt), generator=g)
    ids[0, 0], ids[0, 1], ids[-1, 2] = 0, V - 1, V - 1  # id 0 and the largest valid id (table row V)
    for b in range(B):
        ids[b, nt - 5 * b - 3:] = -1  # -1 padding, a different amount per sample
    vl = None
    if lens == "mixed":
        vl = torch.tensor([1, N // 2, N], dtype=torch.int32)
    elif lens == "long":
        vl = torch.tensor([N, 2777], dtype=torch.int32)
    out = torch.full((2 * B, N, Td), 777.0, device=DEV)
    filler = torch.full((B, N), 9, dtype=torch.uint8, device=DEV)
    launch("f5k_text_gather", ids.to(DEV), B, nt, N, Td, None if vl is None else vl.to(DEV), table, V + 1, add_pos, out, filler)
    # reference
    n = torch.arange(N)
    idx = torch.zeros(B, N, dtype=torch.long)
    idx[:, :min(nt, N)] = ids[:, :N] + 1
    valid = torch.ones(B, N, dtype=torch.bool) if vl is None else n[None] < vl.long()[:, None]
    idx = torch.where(valid, idx, 0)
    assert_equal(filler.cpu(), (idx == 0).to(torch.uint8), "filler")
    tab = table.cpu().double()
    ref = torch.cat((tab[idx], tab[torch.zeros_like(idx)].expand(B, N, Td)), 0)  # cond, then uncond (all ids 0)
    ref = torch.where(torch.cat((valid, valid), 0)[..., None], ref, 0.0)
    got = out.cpu()
    if not add_pos:
        assert_equal(got, ref.float(), "text_gather")
        return
    half = Td // 2
    freq = 10000.0 ** (-torch.arange(half, dtype=F64) * 2 / Td)
    ang = n.double()[:, None] * freq[None]
    pos = torch.cat((ang.cos(), ang.sin()), -1)
    vv = torch.cat((valid, valid), 0)[..., None]
    ref = torch.where(vv, ref + pos, 0.0)
    bound = torch.where(vv, pos_bound(torch.cat((ang, ang), -1)) + U * ref.abs(), 0.0)
    assert_within(got, ref, bound, f"text_gather Td{Td} N{N}")


def test_mask_rows():
    """mask_rows_kernel and mask_rows_len_kernel<float / half>: rows are either untouched or exactly zero."""
    B, N, C = 3, 50, 512
    g = torch.Generator().manual_seed(3)
    filler = (torch.randint(0, 3, (B * N,), generator=g) * 3).to(torch.uint8)  # 0, 3, 6: any non-zero value masks
    for rows in (2 * B * N, B * N):
        x0 = rnd((2 * B * N, C), 4)
        x = x0.clone()
        launch("f5k_mask_rows", x, filler.to(DEV), B * N, rows, C)
        ref = x0.clone()
        r = torch.arange(rows, device=DEV)
        ref[:rows][filler.to(DEV)[r % (B * N)] != 0] = 0.0
        assert_equal(x, ref, f"mask_rows rows={rows}")
    vl = torch.tensor([1, 25, N], dtype=torch.int32, device=DEV)  # rows on both sides of every sample's end
    for dt, is_half in ((torch.float32, 0), (torch.float16, 1)):
        for variants in (1, 2):
            rows = variants * B * N
            x0 = rnd((rows + 7, C), 5, dtype=dt)  # 7 rows past `rows` must stay untouched
            x = x0.clone()
            launch("f5k_mask_rows_len", x, is_half, vl, B, N, rows, C)
            r = torch.arange(rows + 7, device=DEV)
            dead = (r < rows) & ((r % N) >= vl.long()[(r // N) % B])
            assert_equal(x, torch.where(dead[:, None], torch.zeros_like(x0), x0), f"mask_rows_len {dt} x{variants}")


@pytest.mark.parametrize("C", [64, 512])
@pytest.mark.parametrize("N", [1, 2, 3, 7, 300])
def test_dwconv7_ln(N, C):
    """dwconv7_ln_kernel: a = wb + sum_t w[c, t] x[n + t - 3] is an 8-term fp32 sum, |d a| <= g(8) * sum|terms|; the
    LayerNorm over C is bounded by ln_ref_bound with C / 32 + 5 terms per sum; the fp16 store adds half an ulp.  Each
    sample carries its own large offset and scale, so a tap that reads across a sample boundary shows."""
    B = 6
    x = rnd((B, N, C), 10)
    x = x * torch.arange(1, B + 1, device=DEV)[:, None, None] + 40.0 * torch.tensor([1, -2, 3, -4, 5, -6], device=DEV)[:, None, None]
    w, wb = rnd((C, 7), 11, 0.3), rnd((C,), 12, 0.3)
    lw, lb = rnd((C,), 13, 0.5) + 1.0, rnd((C,), 14, 0.3)
    out = torch.empty((B * N, C), dtype=torch.float16, device=DEV)
    launch("f5k_dwconv7_ln", x, out, B, N, C, w, wb, lw, lb, 1e-6)
    a, s = dwconv7_ref(x.double(), w.double(), wb.double())
    y, e = ln_ref_bound(a, gam(8) * s, lw.double(), lb.double(), 1e-6, C // 32 + 5)
    assert_half(out, y.reshape(B * N, C), e.reshape(B * N, C), f"dwconv7_ln N{N} C{C}")


@pytest.mark.parametrize("N", [1, 63, 64, 65, 938])
def test_grn(N):
    """GRN (grn_sumsq / grn_finalize / grn_apply via run_grn) on fp16 g [B, N, C].  v^2 of an fp16 value is exact in
    fp32; per channel the sum over the sequence is a sum of <= 64 terms per block plus ceil(N / 64) block partials, so
    Gx = sqrtf(sum) has relative error r_g = g(64 + nblk) / 2 + u.  mean_c Gx sums C / 256 terms per thread and two
    5-level shuffle trees: r_m = g(C / 256 + 11) + r_g.  Nx = Gx / (mean + 1e-6): r_n = r_g + r_m + 2 u.
    out = gamma (v Nx) + beta + v: |d| <= |gamma v Nx| (r_n + 2 u) + u (|gamma v Nx| + |beta|) + u |out|, then one fp16
    rounding.  Channel 5 is zero in every sample and sample 1 is zero everywhere (Gx = 0, Nx = 0)."""
    B, C = 16, 1024
    rows = hooks().f5k_grn_rows()
    assert rows == 64
    g16 = rnd((B, N, C), 20, 1.0, torch.float16)
    g16[:, :, 5] = 0
    g16[1] = 0
    g0 = g16.clone()
    gamma, beta = rnd((C,), 21, 0.7), rnd((C,), 22, 0.5)
    nblk = (N + rows - 1) // rows
    partial = torch.full((B * nblk * C,), float("nan"), device=DEV)
    nx = torch.full((B * C,), float("nan"), device=DEV)
    launch("f5k_grn", g16, partial, nx, gamma, beta, B, N, C)
    v = g0.double()
    ref, nx_ref = grn_ref(v, gamma.double(), beta.double())
    r_g = 0.5 * gam(rows + nblk) + U
    r_n = r_g + (gam(C // 256 + 11) + r_g) + 2 * U
    assert_within(nx.view(B, 1, C), nx_ref, nx_ref * r_n, f"grn Nx N{N}")
    t = (gamma.double() * v * nx_ref).abs()
    e = t * (r_n + 2 * U) + U * (t + beta.double().abs()) + U * ref.abs()
    assert_half(g16, ref, e, f"grn N{N}")


# ---------------------------------------------------------------------------------------------------------------------
# step path
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("packed", [0, 1])
def test_pack_input(packed):
    """pack_input_kernel: xin = fp16([y | cond (cond half) or 0 | text | 0]) for every row, bit-exact, zero columns
    past 2 mel + Td included."""
    B, N, mel, Td, Kpad = 2, 300, 100, 512, 744
    Be = 2 * B if packed else B
    y, cond, text = rnd((B, N, mel), 30), rnd((B, N, mel), 31), rnd((2 * B, N, Td), 32)
    xin = rnd((Be * N, Kpad), 33, 1.0, torch.float16)
    launch("f5k_pack_input", xin, B, N, mel, Td, Kpad, packed, y, cond, text)
    ref = torch.zeros((Be // B, B * N, Kpad), device=DEV)  # [half, b * N + n, column]
    ref[:, :, :mel] = y.view(1, B * N, mel)
    ref[0, :, mel:2 * mel] = cond.view(B * N, mel)
    ref[:, :, 2 * mel:2 * mel + Td] = text.view(2, B * N, Td)[:Be // B]
    assert_equal(xin, ref.view(Be * N, Kpad).half(), f"pack_input packed={packed}")


class _SampleIo(C.Structure):
    _fields_ = [("y", C.c_void_p), ("traj", C.c_void_p), ("cfg", C.c_float)]


def _dev_bytes(b):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to(DEV)


@pytest.mark.parametrize("tok_off", [0, 1])
@pytest.mark.parametrize("packed", [0, 1])
def test_cfg_euler(packed, tok_off):
    """cfg_euler_kernel through a 3-step Euler stage table, then a 2-step midpoint table, launched in order as sample()
    does.  B N mel = 200000 > 256 * 148 * 4, so the grid-stride loop runs more than once.

    Each launch is checked against float64 on the kernel's own fp32 inputs (y, v):  g = pr + (pr - nu) cfg costs at most
    2 u (|pr - nu| cfg + |g|); y' = y + coef g adds 2 u (|coef g| + |y'|).  A committing stage stores y' in y and in its
    trajectory row (bit-identical to y); a midpoint half stage leaves y and the trajectory alone.  Both fp16 x halves of
    xin hold fp16(y') (bit-identical to y.half() on a commit), every other xin column and trajectory row is untouched,
    and the evaluation counter is k + 1 with the CTA done counter back at 0."""
    B, N, mel, Kpad, cfg = 2, 1000, 100, 728, 2.0
    assert B * N * mel > 256 * 148 * 4
    Be = 2 * B if packed else B
    seq_tok = N + tok_off
    BN = B * N
    t = O.time_grid(3, -1.0).tolist()
    tm = O.time_grid(2, -1.0).tolist()
    phases = [("euler", 3, [(t[k + 1] - t[k], k + 1) for k in range(3)]),
              ("midpoint", 2, [s for k in range(2) for s in (((tm[k + 1] - tm[k]) * 0.5, -1), (tm[k + 1] - tm[k], k + 1))])]
    y = rnd((BN, mel), 40)
    xin = rnd((Be * N, Kpad), 41, 1.0, torch.float16)
    seed = 42
    for phase, steps, stages in phases:
        stage_np = np.array([(np.float32(c), r) for c, r in stages], dtype=[("coef", "<f4"), ("row", "<i4")])
        stage = _dev_bytes(stage_np.tobytes())
        traj = torch.full((steps + 1, BN, mel), -12345.0, device=DEV)
        io = _dev_bytes(bytes(_SampleIo(y.data_ptr(), traj.data_ptr(), cfg)))
        step = torch.zeros(2, dtype=torch.int32, device=DEV)
        for k, (coef, row) in enumerate(stages):
            coef = float(np.float32(coef))
            seed += 1
            v = rnd((Be * seq_tok, mel), seed)
            if tok_off:
                v.view(Be, seq_tok, mel)[:, 0] = 1e4  # the time-token rows must not be read
            y0, traj0, xin0 = y.clone(), traj.clone(), xin.clone()
            launch("f5k_cfg_euler", io, v, xin, stage, step, BN, mel, Kpad, packed, N, seq_tok, tok_off, B)
            what = f"{phase} stage {k} packed={packed} tok_off={tok_off}"
            vv = v.double().view(Be, seq_tok, mel)[:, tok_off:tok_off + N].reshape(Be // B, BN, mel)
            pr = vv[0]
            if packed:
                nu = vv[1]
                gref = pr + (pr - nu) * cfg
                e_g = 2 * U * ((pr - nu).abs() * cfg + gref.abs())
            else:
                gref, e_g = pr, torch.zeros_like(pr)
            yref = y0.double() + coef * gref
            e_y = abs(coef) * e_g + 2 * U * ((coef * gref).abs() + yref.abs())
            if row >= 0:
                assert_within(y, yref, e_y, what + " y")
                expect_traj = traj0.clone()
                expect_traj[row] = y
                assert_equal(traj, expect_traj, what + " trajectory")
                assert_equal(xin[:BN, :mel], y.half(), what + " xin x (cond half) vs y")
            else:
                assert_equal(y, y0, what + " y untouched")
                assert_equal(traj, traj0, what + " trajectory untouched")
            assert_half(xin[:BN, :mel], yref, e_y, what + " xin x")
            if packed:
                assert_equal(xin[BN:, :mel], xin[:BN, :mel], what + " xin x (uncond half)")
            assert_equal(xin[:, mel:], xin0[:, mel:], what + " other xin columns")
            assert step.tolist() == [k + 1, 0], what + f" counters {step.tolist()}"


# ---------------------------------------------------------------------------------------------------------------------
# time path
# ---------------------------------------------------------------------------------------------------------------------
def silu64(x):
    return x / (1.0 + torch.exp(-x))


def silu_rel(x):
    """silu = x / (1 + __expf(-x)) in fp32: __expf is within 2 + 1.2 |x| ulp (<= 2 u each), the sum and the quotient
    add u each, and e / (1 + e) <= 1 carries the exponential's relative error to the result.  Past |x| = 90 the
    exponential is exactly 0 or inf, so the ulp count stops growing there."""
    return (2 + 1.2 * x.abs().clamp(max=90.0)) * 2 * U + 2 * U


@pytest.mark.parametrize("K", [256, 1024, 1000, 1056])
@pytest.mark.parametrize("act", [0, 1])
def test_small_linear(act, K):
    """small_linear_kernel: K in {256, 1024} takes the register path, {1000, 1056} the generic path.  Per lane the dot
    product sums ceil(K / 32) products (fused), then 5 shuffle levels and the bias: |d acc| <= g(ceil(K/32) + 7) *
    (|x| . |W| + |b|).  silu: 1.1 |d acc| (|silu'| < 1.1) + silu_rel(acc) |silu(acc)|."""
    Nout = 1003  # not a multiple of 8: the last CTA has idle warps
    W = rnd((Nout, K), 50, 1.0 / math.sqrt(K), torch.float16)
    for S in (1, 64):
        x = rnd((S, K), 51 + S, 2.0)
        for use_bias in (False, True):
            bias = rnd((Nout,), 53, 0.5) if use_bias else None
            out = torch.full((S, Nout), float("nan"), device=DEV)
            launch("f5k_small_linear", act, x, W, bias, out, S, K, Nout)
            xd, Wd = x.double(), W.double()
            acc = xd @ Wd.t()
            mag = xd.abs() @ Wd.abs().t()
            if use_bias:
                acc = acc + bias.double()
                mag = mag + bias.double().abs()
            e = gam(-(-K // 32) + 7) * mag
            ref = acc
            if act == 1:
                ref = silu64(acc)
                e = 1.1 * e + silu_rel(acc) * ref.abs()
            assert_within(out, ref, e, f"small_linear act{act} K{K} S{S} bias={use_bias}")


def time_args():
    return torch.cat((torch.tensor([0.0, 1.0]), O.time_grid(32, -1.0), O.time_grid(16, None)))  # 52 <= 64 rows


def test_time_features():
    """time_features_kernel: arg = 1000 t exp(-ln(1e4) / (half - 1) * i).  k = logf(1e4) / 127 is within 3 u, k i adds
    u (|k i| <= 9.3, so 4 u relative turns into 37 u of exp's argument), expf adds 2 ulp (4 u), the two products 2 u:
    |d arg| <= 47 u |arg|; sinf / cosf add 4 u.  Bound: 48 u |arg| + 4 u.  Times: 0, 1, the sway grid of 32 steps and
    the EPSS grid of 16 steps.  The oracle's fp32 sinus_time_features lies within the same bound."""
    t = time_args()
    S, dim = t.shape[0], 256
    feat = torch.full((S, dim), float("nan"), device=DEV)
    launch("f5k_time_features", t.to(DEV), feat, S, dim)
    half = dim // 2
    arg = 1000.0 * t.double()[:, None] * torch.exp(-math.log(10000.0) / (half - 1) * torch.arange(half, dtype=F64))[None]
    ref = torch.cat((arg.sin(), arg.cos()), -1)
    bound = torch.cat((arg, arg), -1).abs() * 48 * U + 4 * U
    assert_within(feat.cpu(), ref, bound, "time_features")
    assert_within(O.sinus_time_features(t, dim), ref, bound, "oracle sinus_time_features")


def test_silu_to_half():
    """silu_to_half_kernel over more elements than one pass of the capped grid: fp16(silu(x)), bounded by silu_rel
    plus one fp16 rounding.  silu(1e5) = 1e5 overflows fp16 to +inf, as torch's .half() does; silu(-80) and silu(-1e5)
    round to (-)0."""
    special = torch.tensor([80.0, -80.0, 1e5, -1e5, 0.0, 11.0, -11.0, 65504.0, 65519.0, 65520.0])
    x = torch.cat((special, torch.randn(700_000, generator=torch.Generator().manual_seed(60)) * 6.0)).to(DEV)
    n = x.numel()
    out = torch.full((n,), float("nan"), dtype=torch.float16, device=DEV)
    launch("f5k_silu_to_half", x, out, n)
    ref = silu64(x.double())
    e = silu_rel(x.double()) * ref.abs()
    ovf = (ref.abs() + e) >= 65520.0
    assert bool(ovf[2]) and float(out[2]) == math.inf, "silu(1e5) must overflow to +inf"
    assert_equal(out[ovf], ref[ovf].half(), "silu overflow to inf")
    ok = ~ovf
    assert_half(out[ok], ref[ok], e[ok], "silu_to_half")


def test_rope_table():
    """rope_table_kernel for seq 4096: cos / sin of pos * 10000^(-2i/64), pos_bound(ang) against float64; ops.rope_tables
    (torch fp32) lies within the same bound of float64, so the two differ by at most twice it."""
    seq, half = 4096, 32
    cs = torch.full((seq, half), float("nan"), device=DEV)
    sn = torch.full((seq, half), float("nan"), device=DEV)
    launch("f5k_rope_table", cs, sn, seq, half)
    ang = torch.arange(seq, dtype=F64)[:, None] * (10000.0 ** (-torch.arange(half, dtype=F64) * 2 / (2 * half)))[None]
    b = pos_bound(ang)
    assert_within(cs.cpu(), ang.cos(), b, "rope cos")
    assert_within(sn.cpu(), ang.sin(), b, "rope sin")
    tc, ts = ops.rope_tables(seq, "cpu")
    assert_within(tc, ang.cos(), b, "ops.rope_tables cos")
    assert_within(cs.cpu(), tc, 2 * b, "rope cos vs ops.rope_tables")
    assert_within(sn.cpu(), ts, 2 * b, "rope sin vs ops.rope_tables")


# ---------------------------------------------------------------------------------------------------------------------
# row norm (AdaLN modulation from the per-evaluation table)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [128, 768, 1024])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_row_norm_hook(mode, D):
    """row_norm_kernel<mode> with scale / shift read from a modulation table at row *step_ptr, stride modW = 6 D, both
    before (params_static = 1) and after the dependency wait.  x has a common offset of 300.  Modes 0 / 1: ln_ref_bound
    with D / 32 + 5 terms per sum (mode 0 uses w = 1 + scale, rounded once).  Mode 2: rstd = sqrt(D) / ||x||, the sum of
    squares within g(D / 32 + 6), sqrtf twice and the quotient: r = g(D / 32 + 6) / 2 + 3 u; out = x rstd g:
    |d| <= |out| (r + 2 u).  One fp16 rounding."""
    modW, kmax = 6 * D, 4
    mod = rnd((kmax + 1, modW), 70, 0.4)
    a_off, b_off = 2 * D, 4 * D  # scale / weight at column 2D, shift / bias at 4D of each row
    for rows in (1, 5, 1877):
        x = rnd((rows, D), 71 + rows, 2.0) + 300.0
        for k in (0, kmax):
            step = torch.tensor([k], dtype=torch.int32, device=DEV)
            a = mod[k, a_off:a_off + D].double()
            b = mod[k, b_off:b_off + D].double()
            xd = x.double()
            if mode == 2:
                nrm = xd.norm(dim=-1, keepdim=True)
                ref = xd / nrm * math.sqrt(D) * a
                e = ref.abs() * (0.5 * gam(D // 32 + 6) + 5 * U)
            else:
                w = (1.0 + a) if mode == 0 else a
                ref, e = ln_ref_bound(xd, torch.zeros_like(xd), w, b, 1e-6, D // 32 + 5)
            for static in (0, 1):
                out = torch.full((rows, D), float("nan"), dtype=torch.float16, device=DEV)
                bp = mod.data_ptr() + 4 * b_off if mode != 2 else None
                launch("f5k_row_norm", mode, x, out, rows, D, 1e-6, mod.data_ptr() + 4 * a_off, bp, step, modW, static)
                assert_half(out, ref, e, f"row_norm mode{mode} D{D} rows{rows} k{k} static{static}")


# ---------------------------------------------------------------------------------------------------------------------
# UNetT
# ---------------------------------------------------------------------------------------------------------------------
def test_prepend_time_token_and_concat_half():
    """prepend_time_token_kernel: h[b, 0] = t_emb[k], h[b, 1:] = src[b] (fp32, exact) at evaluation k = 5;
    concat_half_kernel: fp16([x | skip]) (exact, values beyond the fp16 range become inf as in torch)."""
    B, N, D, S, k = 2, 300, 1024, 8, 5
    src, temb = rnd((B * N, D), 80), rnd((S, D), 81)
    step = torch.tensor([k], dtype=torch.int32, device=DEV)
    rows_out = B * (N + 1)
    dst = torch.full((rows_out + 3, D), -1.0, device=DEV)  # 3 rows past rows_out stay untouched
    launch("f5k_prepend_time_token", dst, src, temb, step, N, D, rows_out)
    ref = torch.full_like(dst, -1.0)
    ref[:rows_out].view(B, N + 1, D)[:, 0] = temb[k]
    ref[:rows_out].view(B, N + 1, D)[:, 1:] = src.view(B, N, D)
    assert_equal(dst, ref, "prepend_time_token")
    M = rows_out
    x, skip = rnd((M, D), 82, 3.0), rnd((M, D), 83, 3.0)
    x[0, :4] = torch.tensor([1e5, -1e5, 65519.0, 6e-8], device=DEV)
    out = torch.full((M, 2 * D), float("nan"), dtype=torch.float16, device=DEV)
    launch("f5k_concat_half", x, skip, out, M, D)
    assert_equal(out, torch.cat((x, skip), -1).half(), "concat_half")


# ---------------------------------------------------------------------------------------------------------------------
# Vocos: im2col, LayerNorm (fp32 out), ISTFT
# ---------------------------------------------------------------------------------------------------------------------
VOCOS_CASES = [(B, T) for B in (1, 3) for T in (2, 3, 5, 200)]


@pytest.mark.parametrize("B,T", VOCOS_CASES)
def test_vocos_im2col_ln(B, T):
    """vocos_im2col_kernel: A[b T + t, tap 100 + c] = fp16(mel[b, c, t + tap - 3]) (0 outside, 0 in the pad columns),
    bit-exact.  ln_affine_f32_kernel (D = 512): ln_ref_bound with 512 / 32 + 5 terms per sum, fp32 output."""
    Cm, Kpad, D = 100, 704, 512
    mel = rnd((B, Cm, T), 90, 2.0) - 1.0
    A = torch.full((B * T, Kpad), float("nan"), dtype=torch.float16, device=DEV)
    launch("f5k_vocos_im2col", mel, B, Cm, T, A, Kpad)
    mp = F.pad(mel, (3, 3))
    ref = torch.zeros((B, T, Kpad), device=DEV)
    for tap in range(7):
        ref[:, :, tap * Cm:(tap + 1) * Cm] = mp[:, :, tap:tap + T].transpose(1, 2)
    assert_equal(A, ref.view(B * T, Kpad).half(), f"vocos_im2col B{B} T{T}")
    R = B * T
    x = rnd((R, D), 91, 1.5) + 7.0
    w, b = rnd((D,), 92, 0.5) + 1.0, rnd((D,), 93, 0.5)
    out = torch.full((R, D), float("nan"), device=DEV)
    launch("f5k_ln_affine_f32", x, out, R, D, 1e-6, w, b)
    xd = x.double()
    y, e = ln_ref_bound(xd, torch.zeros_like(xd), w.double(), b.double(), 1e-6, D // 32 + 5)
    assert_within(out, y, e, f"ln_affine_f32 B{B} T{T}")


@pytest.mark.parametrize("B,T", VOCOS_CASES)
def test_istft(B, T):
    """run_istft (istft_frames + istft_ola) against kernel_bounds.istft_ref: the oracle's istft_center in float64 of
    the clipped spectrum mag = min(exp(logmag), 100), under istft_ref's bound, with log-magnitudes above ln 100 and
    non-zero DC / Nyquist phases (whose imaginary parts the inverse real FFT ignores)."""
    ld, nb = 1026, 513
    g = torch.Generator().manual_seed(100 + T + B)
    logmag = torch.randn(B * T, nb, generator=g, dtype=F64) * 1.5 + 2.0
    logmag[:, 200:260] = 5.5  # above ln 100 = 4.605: clipped to 100
    logmag[::2, 0] = 6.0
    phase = (torch.rand(B * T, nb, generator=g, dtype=F64) * 2 - 1) * math.pi
    phase[:, 0], phase[:, nb - 1] = 1.1, -2.3  # DC / Nyquist phases
    head = torch.cat((logmag, phase), -1).float().to(DEV)
    frames = torch.full((B * T, 1024), float("nan"), device=DEV)
    wav = torch.full((B, 256 * (T - 1)), float("nan"), device=DEV)
    launch("f5k_istft", head, ld, frames, wav, B, T)
    ref, bound = istft_ref(head.cpu().double(), T)
    assert ref.shape == (B, 256 * (T - 1))
    assert_within(wav.cpu(), ref, bound, f"istft B{B} T{T}")


# ---------------------------------------------------------------------------------------------------------------------
# mel front-end (public C ABI)
# ---------------------------------------------------------------------------------------------------------------------
FLOOR = 1e-5


def mel_ref(wav, fb):
    """float64 |STFT| (reflect pad 512, periodic Hann 1024, hop 256) @ fb -> linear mel [B, T, n_mels], and the per
    (b, t) L2 norm of the windowed frame."""
    xp = F.pad(wav.double()[:, None], (512, 512), mode="reflect")[:, 0]
    fr = xp.unfold(-1, 1024, 256) * torch.hann_window(1024, periodic=True, dtype=F64)
    return torch.fft.rfft(fr, dim=-1).abs() @ fb.double(), fr.norm(dim=-1)


def mel_call(wav, fb, n_mels, out_btc):
    B, nw = wav.shape
    T = 1 + nw // 256
    out = torch.full((B, T, n_mels) if out_btc else (B, n_mels, T), float("nan"), device=DEV)
    _lib.check(_lib.lib().f5_mel_spectrogram(wav.data_ptr(), B, nw, fb.data_ptr(), n_mels, out.data_ptr(), out_btc,
                                             torch.cuda.current_stream().cuda_stream), "f5_mel_spectrogram")
    torch.cuda.synchronize()
    return out if out_btc else out.transpose(1, 2)


def check_mel(got, wav, fb, what):
    """got: log-mel [B, T, n_mels] from the kernel.  The real-input FFT is one 512-point complex radix-2 FFT (9 stages,
    at most ~8 u each in the L2 norm with table twiddles) plus the split, so every bin's |X_k| is within
    160 u sqrt(512) ||windowed frame||_2 (the L2 error bound of the transform applied per bin); the filter sum adds
    colsum(fb) times that plus g(513) of the mel value.  max(., 1e-5) is 1-Lipschitz, and logf then expf-back cost
    4 u |log|.  Bins whose reference is below the floor by more than the bound must equal log(1e-5) exactly."""
    lin, l2 = mel_ref(wav.cpu(), fb.cpu())
    e_bin = 160 * U * math.sqrt(512) * l2  # [B, T]
    e = e_bin[..., None] * fb.cpu().double().sum(0) + gam(513) * lin
    floor_val = torch.full((), FLOOR, device=DEV).log().cpu()  # the device logf of fp32 1e-5
    g = got.cpu()
    at_floor = (lin + e) < FLOOR
    assert_equal(g[at_floor], floor_val.expand(int(at_floor.sum())), what + " floor bins")
    ref = lin.clamp(min=FLOOR)
    gl = torch.exp(g.double())
    assert_within(gl, ref, e + ref * 4 * U * ref.log().abs() + 2 * U * ref, what)
    return int(at_floor.sum())


@pytest.mark.parametrize("nw", [513, 767, 768, 769, 48017])
@pytest.mark.parametrize("B", [1, 3])
def test_mel_spectrogram(B, nw):
    """f5_mel_spectrogram in both layouts: sample 0 is noise, sample 1 silence (exactly log 1e-5 everywhere), sample 2 a
    tone at the centre of bin 100."""
    fb = O.mel_filterbank(513, 0.0, 12000.0, 100, 24000).contiguous().to(DEV)
    g = torch.Generator().manual_seed(nw)
    wav = 0.1 * torch.randn(B, nw, generator=g)
    if B == 3:
        wav[1] = 0.0
        wav[2] = 0.5 * torch.sin(2 * math.pi * 100 * torch.arange(nw, dtype=F64) / 1024).float()
    wav = wav.to(DEV)
    got = mel_call(wav, fb, 100, 0)
    assert_equal(mel_call(wav, fb, 100, 1), got, "out_btc layouts")
    check_mel(got, wav, fb, f"mel B{B} nw{nw}")
    if B == 3:
        assert bool((got[1].cpu() == torch.full((), FLOOR, device=DEV).log().cpu()).all()), "silence must be log(1e-5)"


def test_mel_filterbank_reuse():
    """One filterbank buffer used three times: filterbank A (f_max 12 kHz, 100 mels), the same storage rewritten in place
    with B (f_max 8 kHz, 100 mels), then with an 80-mel filterbank.  Each call must use the filterbank as it is at
    launch time, and match its own float64 reference."""
    nw = 24000
    wav = (0.1 * torch.randn(2, nw, generator=torch.Generator().manual_seed(7))).to(DEV)
    buf = torch.zeros(513 * 100, device=DEV)
    for what, n_mels, f_max in (("A", 100, 12000.0), ("B in place", 100, 8000.0), ("80 mels in place", 80, 12000.0)):
        fb = O.mel_filterbank(513, 0.0, f_max, n_mels, 24000)
        buf[:513 * n_mels].copy_(fb.reshape(-1).to(DEV))
        view = buf[:513 * n_mels].view(513, n_mels)
        check_mel(mel_call(wav, view, n_mels, 1), wav, view, f"filterbank {what}")
