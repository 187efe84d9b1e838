"""Element-by-element GPU tests of the launchers the engine and the Vocos decode use beyond test_gpu_small_kernels.py:
the MMDiT text embedding, text average upsampling, the per-sample AdaLN row norm (mode 4) and time token of
f5_forward, and the length-aware dwconv7_ln, vocos_im2col and istft of the different-length Vocos decode, each against
a float64 reference of the same operation.

The kernels are launched one at a time through libf5tts_b200_kernels.so (csrc/kernel_hooks.cu).  Every output is
pre-filled with NaN or a sentinel, so a value the kernel should have written and did not, or wrote and should not
have, shows.  Inputs past a length (rows past a sample's end, filler rows, frames past a sample's frame count) hold
NaN, +-inf and 1e4, so a read past a length shows as well.  Data movement is bit-exact; every other bound is derived
in its test's docstring (u = 2^-24, g(n) = n u / (1 - n u)).
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from f5_tts_b200 import _lib  # noqa: E402
from oracle import kernel_bounds as KB  # noqa: E402
from oracle.kernel_bounds import (assert_half, assert_within, dwconv7_ref, gam, istft_ref, ln_ref_bound,  # noqa: E402
                                  mmdit_text_embed_ref)

DEV = "cuda:0"
F64 = torch.float64
POISON = (math.nan, math.inf, -math.inf, 1e4)

# ---------------------------------------------------------------------------------------------------------------------
# ctypes binding of the kernel hooks
# ---------------------------------------------------------------------------------------------------------------------
_P, _I, _F, _LL = C.c_void_p, C.c_int, C.c_float, C.c_longlong
_SIGS = {
    "f5k_mmdit_text_embed": [_P, _I, _I, _I, _I, _P, _I, _I, _P, _P],
    "f5k_text_avg_upsample": [_P, _P, _P, _P, _I, _I, _I, _I],
    "f5k_row_norm_sample": [_P, _P, _I, _I, _F, _P, _P, _LL, _I, _I, _I],
    "f5k_prepend_time_token_sample": [_P, _P, _P, _I, _I, _I, _LL],
    "f5k_dwconv7_ln": [_P, _P, _I, _I, _I, _P, _P, _P, _P, _F],
    "f5k_dwconv7_ln_len": [_P, _P, _I, _I, _I, _P, _P, _P, _P, _F, _P],
    "f5k_vocos_im2col": [_P, _I, _I, _I, _P, _I],
    "f5k_vocos_im2col_len": [_P, _I, _I, _I, _P, _I, _P],
    "f5k_istft": [_P, _I, _P, _P, _I, _I],
    "f5k_istft_len": [_P, _I, _P, _P, _I, _I, _P],
}
_hooks = None


def hooks():
    global _hooks
    if _hooks is None:
        L = C.CDLL(_lib.KERNELS_LIB_PATH)
        L.f5k_last_error.restype = C.c_char_p
        for name, args in _SIGS.items():
            getattr(L, name).argtypes = args + [_P]  # + stream
            getattr(L, name).restype = _I
        _hooks = L
    return _hooks


def call(name, *args):
    """Call hook `name` on the current stream (tensors pass their data pointer, None a null pointer), wait for it, and
    return (rc, error message)."""
    conv = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    rc = getattr(hooks(), name)(*conv, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, hooks().f5k_last_error().decode() if rc else ""


def launch(name, *args):
    rc, msg = call(name, *args)
    assert rc == 0, f"{name} failed (rc={rc}): {msg}"


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def rnd(shape, seed, scale=1.0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=F64) * scale).to(dtype).to(DEV)


def assert_equal(got, ref, what):
    if not torch.equal(got, ref):
        d = torch.nonzero(~((got == ref) | (torch.isnan(got) & torch.isnan(ref))))
        raise AssertionError(f"{what}: {d.shape[0]} elements differ, first at {d[0].tolist()}: "
                             f"got {got[tuple(d[0])].item()!r} ref {ref[tuple(d[0])].item()!r}")


def poison(x, dead):
    """x [..., R, C] with the rows where dead [..., R] is set overwritten by NaN, +inf, -inf, 1e4 (cycling by row)."""
    vals = torch.tensor(POISON, dtype=x.dtype, device=x.device)[torch.arange(dead.shape[-1], device=x.device) % 4]
    return torch.where(dead[..., None], vals[:, None].expand(x.shape[-2:]), x)


def report(what, worst):
    print(f"{what}: worst err / bound {worst:.3f}")


# ---------------------------------------------------------------------------------------------------------------------
# MMDiT text embedding
# ---------------------------------------------------------------------------------------------------------------------
V = 2545  # text_num_embeds: table rows V + 1


def mmdit_ids(nt, seed):
    """Three samples: no padding (ids 0 and V - 1 included), all -1 (c_len 0), trailing -1 padding after 2 nt / 3."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, V, (3, nt), generator=g)
    ids[0, 0], ids[0, -1] = 0, V - 1
    ids[1] = -1
    keep = max(1, 2 * nt // 3)
    ids[2, keep:] = -1
    ids[2, 0] = V - 1
    if keep > 1:
        ids[2, 1] = 0
    return ids


@pytest.mark.parametrize("nt", [1, 17, 300, 1500])
@pytest.mark.parametrize("D", [1024, 768, 128])
def test_mmdit_text_embed(D, nt):
    """mmdit_text_embed_kernel for Be = B (cond) and 2B (cond, uncond), mask_padding 0 and 1, against
    kernel_bounds.mmdit_text_embed_ref: out = table[id + 1] + cat(cos, sin)(min(n, 1023) * 10000^(-2i/D)) (uncond: id 0,
    the real text's mask), within pos_bound(ang) + u |out| (fp32 angle and cosf / sinf, one rounded addition).  Masked
    rows must be exactly 0 and c_len[v B + b] (ids that are not -1) exact.  At nt = 1500 every row from 1023 on carries
    position 1023.  Rows past Be * nt and c_len entries past Be keep their sentinels."""
    B = 3
    table = rnd((V + 1, D), D + nt, 0.5)
    ids = mmdit_ids(nt, nt)
    n_valid = (ids != -1).sum(1).tolist()
    assert n_valid[1] == 0 and n_valid[0] == nt
    worst = 0.0
    for Be in (B, 2 * B):
        for mp in (0, 1):
            what = f"mmdit_text_embed D{D} nt{nt} Be{Be} mask_padding{mp}"
            out = torch.full((2 * B * nt + 1, D), math.nan, device=DEV)
            c_len = torch.full((2 * B + 1,), -7, dtype=torch.int32, device=DEV)
            launch("f5k_mmdit_text_embed", ids.to(DEV), B, Be, nt, D, table, V + 1, mp, out, c_len)
            ref, bound = mmdit_text_embed_ref(table, ids, Be, mp)
            worst = max(worst, assert_within(out[:Be * nt].view(Be, nt, D), ref, bound, what))
            assert bool(torch.isnan(out[Be * nt:]).all()), what + ": rows past Be * nt were written"
            assert c_len.tolist() == (n_valid * 2)[:Be] + [-7] * (2 * B + 1 - Be), what + f" c_len {c_len.tolist()}"
    report(f"mmdit_text_embed D{D} nt{nt}", worst)


# ---------------------------------------------------------------------------------------------------------------------
# text average upsampling
# ---------------------------------------------------------------------------------------------------------------------
UPSAMPLE_CASES = [
    # N, nt, Td, valid text rows T per sample, valid_len (None: null, A = N)
    (100, 40, 512, (0, 1, 30, 25, 12), (100, 77, 10, 25, 36)),  # T = 0, T = 1, A < T, A = T, A = 3 T
    (100, 40, 100, (0, 1, 25, 33, 7), None),                    # A = N = 4 * 25, 3 * 33 + 1, 14 * 7 + 2
    (61, 200, 512, (61, 20, 20, 13), (61, 0, 1000, 39)),        # nt > N (K = N = 61); A = 0; valid_len > N; A = 3 T
    (1000, 700, 512, (500, 350, 699, 1), (1000, 300, 5000, 999)),  # K = 700 > 256: three ballot passes
    (3000, 2900, 100, (2000, 2900), None),                      # twelve ballot passes
]


def upsample_case(N, nt, Td, Ts, vl, seed):
    """tx [2B, N, Td], filler [B, N] with Ts[b] valid rows scattered over the first K = min(nt, N) positions.  Filler
    flags are any non-zero value; positions at or past K are 0 (they must never be read: the kernel treats them as
    filler), and tx rows that are not valid text rows hold NaN / inf / 1e4 in both variants."""
    B, K = len(Ts), min(nt, N)
    g = torch.Generator().manual_seed(seed)
    valid = torch.zeros(B, N, dtype=torch.bool)
    for b, T in enumerate(Ts):
        valid[b, torch.randperm(K, generator=g)[:T]] = True
    filler = torch.randint(1, 256, (B, N), generator=g, dtype=torch.uint8)
    filler[valid] = 0
    filler[:, K:] = 0
    tx = poison(rnd((2 * B, N, Td), seed + 1), torch.cat((~valid, ~valid), 0).to(DEV))
    return tx, filler.to(DEV), valid


def upsample_ref(tx, valid, A, N):
    """The kernel copies rows, so the reference is a copy of the rows avg_upsample_index picks (0 where it picks none)."""
    B = valid.shape[0]
    src = KB.avg_upsample_index(valid, A, N).to(tx.device)  # [B, N]
    ref = torch.zeros_like(tx)
    for var in (0, 1):
        for b in range(B):
            keep = src[b] >= 0
            ref[var * B + b, keep] = tx[var * B + b, src[b, keep]]
    return ref


@pytest.mark.parametrize("N,nt,Td,Ts,vl", UPSAMPLE_CASES)
def test_text_avg_upsample(N, nt, Td, Ts, vl):
    """text_avg_upsample_kernel against kernel_bounds.avg_upsample_index (dit.py:55-84's own repeat loop), bit-exact:
    sample b's T valid rows fill its A = min(valid_len[b], N) rows (N when valid_len is null), token j repeated A // T
    times and once more for the last A % T tokens; rows at or past A, and every row when T = 0, are exactly 0; both CFG
    variants use the same source rows.  Every output element starts as NaN."""
    B = len(Ts)
    tx, filler, valid = upsample_case(N, nt, Td, Ts, vl, N + nt)
    A = [N] * B if vl is None else list(vl)
    out = torch.full_like(tx, math.nan)
    launch("f5k_text_avg_upsample", tx, out, filler, None if vl is None else torch.tensor(vl, dtype=torch.int32, device=DEV),
           B, N, nt, Td)
    assert_equal(out, upsample_ref(tx, valid, A, N), f"text_avg_upsample N{N} nt{nt} valid_len={vl}")


def test_text_avg_upsample_token_limit():
    """A block keeps its sample's valid-row list and 8 warp counts in the 48 KB of shared memory it gets without an
    opt-in, so K = min(nt, N) is limited to 48 KB / 4 - 8 = 12280 tokens: K = 12280 runs and is exact like the cases
    above, K = 12281 is rejected with an error before anything is launched (the output keeps its NaN)."""
    kmax = 12280
    N, Td = kmax + 1, 4
    tx, filler, valid = upsample_case(N, kmax, Td, (9000,), None, 5)
    out = torch.full_like(tx, math.nan)
    launch("f5k_text_avg_upsample", tx, out, filler, None, 1, N, kmax, Td)
    assert_equal(out, upsample_ref(tx, valid, [N], N), f"text_avg_upsample K = {kmax}")
    out = torch.full_like(tx, math.nan)
    rc, msg = call("f5k_text_avg_upsample", tx, out, filler, None, 1, N, N, Td)
    assert rc != 0 and str(kmax) in msg, f"K = {kmax + 1} must be rejected (rc={rc}, {msg!r})"
    assert bool(torch.isnan(out).all()), "a rejected call wrote its output"


# ---------------------------------------------------------------------------------------------------------------------
# f5_forward: per-sample AdaLN (row norm mode 4) and time token
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stream", ["N", "N+1", "nt"])
@pytest.mark.parametrize("D", [128, 768, 1024])
def test_row_norm_sample(D, stream):
    """row_norm_kernel<4>: mode 0's LayerNorm * (1 + scale) + shift with scale / shift read from row
    (row / sample_seq) % samples of a modulation table of stride modW = 6 D (scale at column 2D, shift at 4D), for
    sample_seq = N (DiT audio stream), N + 1 (UNetT, time token) and nt (MMDiT text stream), rows = 2 B seq (cond and
    uncond) and B seq, B = 1, 2, 3, params_static 0 and 1.  Bound: test_row_norm_hook's for mode 0, ln_ref_bound with
    D / 32 + 5 terms per sum and w = 1 + scale, plus one fp16 rounding.  Every table row differs, and the row after the
    last sample's is NaN, so a wrong modulation row shows; 4 rows past `rows` keep their NaN."""
    N, nt = 45, 19
    seq = {"N": N, "N+1": N + 1, "nt": nt}[stream]
    modW, a_off, b_off = 6 * D, 2 * D, 4 * D
    worst = 0.0
    for B in (1, 2, 3):
        mod = rnd((B + 1, modW), 70 + B, 0.4)
        mod[B] = math.nan
        for variants in (2, 1):
            rows = variants * B * seq
            x = rnd((rows, D), 71 + rows, 2.0) + 300.0
            sample = (torch.arange(rows, device=DEV) // seq) % B
            a = mod[sample, a_off:a_off + D].double()
            b = mod[sample, b_off:b_off + D].double()
            xd = x.double()
            ref, e = ln_ref_bound(xd, torch.zeros_like(xd), 1.0 + a, b, 1e-6, D // 32 + 5)
            for static in (0, 1):
                what = f"row_norm mode 4 D{D} seq{seq} B{B} rows{rows} static{static}"
                out = torch.full((rows + 4, D), math.nan, dtype=torch.float16, device=DEV)
                launch("f5k_row_norm_sample", x, out, rows, D, 1e-6, mod.data_ptr() + 4 * a_off,
                       mod.data_ptr() + 4 * b_off, modW, seq, B, static)
                worst = max(worst, assert_half(out[:rows], ref, e, what))
                assert bool(torch.isnan(out[rows:]).all()), what + ": rows past `rows` were written"
    report(f"row_norm mode 4 D{D} seq {stream}", worst)


def test_row_norm_sample_rejects_bad_samples():
    """Mode 4 with samples <= 0 or sample_seq <= 0 is an error, and nothing is launched."""
    D, rows = 128, 8
    x = rnd((rows, D), 72)
    mod = rnd((2, 6 * D), 73)
    for samples, seq in ((0, 4), (-1, 4), (2, 0), (2, -3)):
        out = torch.full((rows, D), math.nan, dtype=torch.float16, device=DEV)
        rc, msg = call("f5k_row_norm_sample", x, out, rows, D, 1e-6, mod, mod, 6 * D, seq, samples, 1)
        assert rc != 0 and "mode 4" in msg, f"samples={samples} sample_seq={seq} must be rejected (rc={rc}, {msg!r})"
        assert bool(torch.isnan(out).all()), "a rejected call wrote its output"


@pytest.mark.parametrize("B", [1, 2, 3])
def test_prepend_time_token_sample(B):
    """prepend_time_token_sample_kernel, bit-exact: for rows_out = 2B (N + 1) (cond and uncond) and B (N + 1), row
    b (N + 1) is t_emb[b % B] (each sample's own time, shared by its cond and uncond rows) and the next N rows are
    src[b N : (b + 1) N].  The t_emb row after the last sample's is NaN; 3 rows past rows_out keep their sentinel."""
    N = 300
    for D in (768, 1024):
        src, temb = rnd((2 * B * N, D), 80 + D), rnd((B + 1, D), 81 + D)
        temb[B] = math.nan
        for variants in (2, 1):
            Be = variants * B
            rows_out = Be * (N + 1)
            dst = torch.full((rows_out + 3, D), -1.0, device=DEV)
            launch("f5k_prepend_time_token_sample", dst, src, temb, B, N, D, rows_out)
            ref = torch.full_like(dst, -1.0)
            ref[:rows_out].view(Be, N + 1, D)[:, 0] = temb[torch.arange(Be, device=DEV) % B]
            ref[:rows_out].view(Be, N + 1, D)[:, 1:] = src[:Be * N].view(Be, N, D)
            assert_equal(dst, ref, f"prepend_time_token_sample B{B} D{D} rows_out{rows_out}")


# ---------------------------------------------------------------------------------------------------------------------
# Vocos decode of different-length mels: dwconv7_ln, im2col and ISTFT with per-sample lengths
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [64, 512])
@pytest.mark.parametrize("N", [9, 300])
def test_dwconv7_ln_len(N, C):
    """dwconv7_ln_kernel with len = 0, 1, 2, 3, 4, N - 1, N: sample b against dwconv7_ref of its first len[b] rows (the
    conv's zero padding starts at len[b]) under test_dwconv7_ln's bound (an 8-term fp32 sum, g(8) sum|terms|; LayerNorm
    by ln_ref_bound with C / 32 + 5 terms per sum; one fp16 rounding).  Rows at or past len[b] hold NaN / inf / 1e4 in x
    and keep the output sentinel.  Each sample carries its own offset and scale.  With every len = N the output equals
    the null-len launch bit for bit."""
    lens = [0, 1, 2, 3, 4, N - 1, N]
    B = len(lens)
    x0 = rnd((B, N, C), 10) * torch.arange(1, B + 1, device=DEV)[:, None, None]
    x0 = x0 + 40.0 * torch.tensor([1, -2, 3, -4, 5, -6, 7], device=DEV, dtype=torch.float32)[:, None, None]
    w, wb = rnd((C, 7), 11, 0.3), rnd((C,), 12, 0.3)
    lw, lb = rnd((C,), 13, 0.5) + 1.0, rnd((C,), 14, 0.3)
    ln = torch.tensor(lens, dtype=torch.int32, device=DEV)
    x = poison(x0, torch.arange(N, device=DEV)[None] >= ln[:, None].long())
    sentinel = 1234.0  # exact in fp16
    out = torch.full((B * N, C), sentinel, dtype=torch.float16, device=DEV)
    launch("f5k_dwconv7_ln_len", x, out, B, N, C, w, wb, lw, lb, 1e-6, ln)
    worst = 0.0
    for b, L in enumerate(lens):
        rows = out[b * N:(b + 1) * N]
        if L:
            a, s = dwconv7_ref(x[b:b + 1, :L].double(), w.double(), wb.double())
            y, e = ln_ref_bound(a, gam(8) * s, lw.double(), lb.double(), 1e-6, C // 32 + 5)
            worst = max(worst, assert_half(rows[:L], y[0], e[0], f"dwconv7_ln_len N{N} C{C} len{L}"))
        assert bool((rows[L:] == sentinel).all()), f"dwconv7_ln_len N{N} C{C}: rows at or past len {L} were written"
    report(f"dwconv7_ln_len N{N} C{C}", worst)
    a_null = torch.full((B * N, C), sentinel, dtype=torch.float16, device=DEV)
    a_len = a_null.clone()
    launch("f5k_dwconv7_ln", x0, a_null, B, N, C, w, wb, lw, lb, 1e-6)
    launch("f5k_dwconv7_ln_len", x0, a_len, B, N, C, w, wb, lw, lb, 1e-6, torch.full_like(ln, N))
    assert_equal(a_len, a_null, f"dwconv7_ln N{N} C{C}: len = N vs null")


@pytest.mark.parametrize("T", [7, 200])
def test_vocos_im2col_len(T):
    """vocos_im2col_kernel with lengths 1, 2, 3, T - 1, T, bit-exact: A[b T + t, tap 100 + c] = fp16(mel[b, c, t + tap
    - 3]) when 0 <= t + tap - 3 < lengths[b], else 0 (0 in the pad columns too), for every row t < T.  Frames at or past
    lengths[b] hold NaN / inf / 1e4 in mel, so a tap that reads one shows.  With every length = T the output equals the
    null-lengths launch bit for bit."""
    Cm, Kpad = 100, 704
    lens = [1, 2, 3, T - 1, T]
    B = len(lens)
    ln = torch.tensor(lens, dtype=torch.int32, device=DEV)
    mel0 = rnd((B, Cm, T), 90, 2.0) - 1.0
    dead = torch.arange(T, device=DEV)[None] >= ln[:, None].long()  # [B, T]
    mel = poison(mel0.transpose(1, 2), dead).transpose(1, 2).contiguous()
    A = torch.full((B * T, Kpad), math.nan, dtype=torch.float16, device=DEV)
    launch("f5k_vocos_im2col_len", mel, B, Cm, T, A, Kpad, ln)
    mp = F.pad(torch.where(dead[:, None, :], 0.0, mel0), (3, 3))
    ref = torch.zeros((B, T, Kpad), device=DEV)
    for tap in range(7):
        ref[:, :, tap * Cm:(tap + 1) * Cm] = mp[:, :, tap:tap + T].transpose(1, 2)
    assert_equal(A, ref.view(B * T, Kpad).half(), f"vocos_im2col_len T{T}")
    a_null = torch.full((B * T, Kpad), math.nan, dtype=torch.float16, device=DEV)
    a_len = a_null.clone()
    launch("f5k_vocos_im2col", mel0, B, Cm, T, a_null, Kpad)
    launch("f5k_vocos_im2col_len", mel0, B, Cm, T, a_len, Kpad, torch.full_like(ln, T))
    assert_equal(a_len, a_null, f"vocos_im2col T{T}: lengths = T vs null")


@pytest.mark.parametrize("T", [2, 5, 200])
def test_istft_len(T):
    """run_istft with lengths Tb = 1 (an all-zero waveform), 2, T - 1 and T: sample b is the float64 ISTFT of its
    first Tb frames under kernel_bounds.istft_ref's bound, followed by exact zeros up to 256 (T - 1).  Head rows of
    frames at or past Tb hold NaN / inf / 1e4, and those frames keep the sentinel of the frames scratch (they are not
    computed).  With every length = T, frames and waveform equal the null-lengths launch bit for bit."""
    ld, nb = 1026, 513
    lens = [1, 2, T - 1, T]
    B = len(lens)
    ln = torch.tensor(lens, dtype=torch.int32, device=DEV)
    g = torch.Generator().manual_seed(200 + T)
    logmag = torch.randn(B * T, nb, generator=g, dtype=F64) * 1.5 + 2.0
    logmag[:, 200:260] = 5.5  # above ln 100: clipped to 100
    phase = (torch.rand(B * T, nb, generator=g, dtype=F64) * 2 - 1) * math.pi
    phase[:, 0], phase[:, nb - 1] = 1.1, -2.3  # DC / Nyquist phases
    head0 = torch.cat((logmag, phase), -1).float().to(DEV)
    dead = (torch.arange(T, device=DEV)[None] >= ln[:, None].long()).reshape(B * T)
    head = poison(head0, dead)
    sentinel = -5.0
    frames = torch.full((B * T, 1024), sentinel, device=DEV)
    wav = torch.full((B, 256 * (T - 1)), math.nan, device=DEV)
    launch("f5k_istft_len", head, ld, frames, wav, B, T, ln)
    assert bool((frames[dead] == sentinel).all()), f"istft T{T}: a frame at or past its sample's length was computed"
    h = head.cpu().double()
    worst = 0.0
    for b, Tb in enumerate(lens):
        L = 256 * (Tb - 1)
        if Tb >= 2:
            ref, bound = istft_ref(h[b * T:b * T + Tb], Tb)
            worst = max(worst, assert_within(wav[b, :L].cpu(), ref[0], bound[0], f"istft_len T{T} Tb{Tb}"))
        assert bool((wav[b, L:] == 0).all()), f"istft_len T{T} Tb{Tb}: the tail past 256 (Tb - 1) is not exactly 0"
    report(f"istft_len T{T}", worst)
    f_null, w_null = torch.full_like(frames, sentinel), torch.full_like(wav, math.nan)
    f_len, w_len = f_null.clone(), w_null.clone()
    launch("f5k_istft", head0, ld, f_null, w_null, B, T)
    launch("f5k_istft_len", head0, ld, f_len, w_len, B, T, torch.full_like(ln, T))
    assert_equal(f_len, f_null, f"istft T{T}: frames, lengths = T vs null")
    assert_equal(w_len, w_null, f"istft T{T}: waveform, lengths = T vs null")
