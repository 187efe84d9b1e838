"""Every GEMM instantiation, the GEMM options the engine and the vocoder set, and the attention kernel, element by
element against float64 references with the derived error bounds of oracle/kernel_bounds.py.

f5_gemm is called through `gemm()` below, which fills _lib.GemmArgs directly: the engine's options (step_ptr,
skip_padded_tiles, out16b, ldo > n_out, weights_static, the conv GEMM's tile skip) are not reachable from ops.linear and
have no product caller in Python.  The float64 references run on the device.

Every output lives inside a guard band: sentinel rows before and after it, and columns between n_out and ldo.  No
kernel may change a sentinel bit.  Each test prints its worst err / bound; the module prints the worst per group at the
end.  A worst ratio above 1 is a finding (a kernel bug or a flaw in the error model), not a tolerance to raise.
"""
import math
import os
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import ctypes as C  # noqa: E402

from f5_tts_b200 import _lib, ops  # noqa: E402
from oracle import kernel_bounds as KB  # noqa: E402

DEV = "cuda:0"
F64 = torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPI = {"EPI_F16": 0, "EPI_F32": 1, "EPI_RESID": 2, "EPI_QKV_ROPE": 3, "EPI_QKV_NORM_ROPE": 4,
       "EPI_QKV_ROPE_DH128": 3, "EPI_QKV_NORM_ROPE_DH128": 4}
ACT = {"ACT_NONE": 0, "ACT_GELU_TANH": 1, "ACT_GELU_ERF": 2, "ACT_MISH": 3}
STAGES = {64: 7, 128: 5, 192: 4, 256: 3}  # gemm_stages(bn)
SMS = torch.cuda.get_device_properties(0).multi_processor_count

# every entry of kGemmKernels (gemm.cu), as (bn, epilogue, activation, conv)
PLAIN = [(bn, e, a, False) for bn in (64, 128, 192, 256)
         for e, a in (("EPI_F16", "ACT_NONE"), ("EPI_F16", "ACT_GELU_TANH"), ("EPI_F16", "ACT_GELU_ERF"),
                      ("EPI_F32", "ACT_NONE"), ("EPI_RESID", "ACT_NONE"))
         if not (bn == 192 and (a == "ACT_GELU_ERF" or e == "EPI_F32"))]
QKV = ([(bn, "EPI_QKV_ROPE", "ACT_NONE", False) for bn in (128, 192, 256)]
       + [(bn, "EPI_QKV_NORM_ROPE", "ACT_NONE", False) for bn in (128, 192, 256)]
       + [(bn, "EPI_QKV_ROPE_DH128", "ACT_NONE", False) for bn in (128, 192, 256)]
       + [(128, "EPI_QKV_NORM_ROPE_DH128", "ACT_NONE", False)])
CONV = [(64, "EPI_F16", "ACT_MISH", True), (64, "EPI_RESID", "ACT_MISH", True)]

_worst = {}


def record(group, what, r):
    print(f"[{group}] {what}: worst err / bound {r:.3f}")
    _worst[group] = max(_worst.get(group, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    print("\nworst err / bound per group: " + ", ".join(f"{g} {r:.3f}" for g, r in sorted(_worst.items())))


def gen(shape, seed, scale=1.0, dtype=torch.float16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=F64) * scale).to(dtype).to(DEV)


# ---------------------------------------------------------------------------------------------------------------------
# guarded outputs and the raw f5_gemm call
# ---------------------------------------------------------------------------------------------------------------------
_SENTINEL = {torch.float16: (torch.int16, 0x7E5A), torch.float32: (torch.int32, 0x7FC5A5A5)}  # NaN payloads


class Guarded:
    """[rows, n] output at leading dimension ldo inside a buffer with `pad` sentinel rows on each side; `init` fills
    [rows, :n] (the residual of EPI_RESID), otherwise the whole buffer holds the sentinel."""

    def __init__(self, rows, n, ldo, dtype, init=None, pad=3):
        self.rows, self.n, self.pad, self.dtype = rows, n, pad, dtype
        it, bits = _SENTINEL[dtype]
        self.buf = torch.full((rows + 2 * pad, ldo), bits, dtype=it, device=DEV).view(dtype)
        if init is not None:
            self.buf[pad:pad + rows, :n] = init
        self.before = self.buf.clone()

    def ptr(self):
        return self.buf[self.pad].data_ptr()

    def out(self):
        return self.buf[self.pad:self.pad + self.rows, :self.n]

    def bits(self):
        return self.buf.view(_SENTINEL[self.dtype][0])

    def untouched(self):
        """[rows, n] bool: the element kept the bits it had before the launch."""
        same = self.bits() == self.before.view(_SENTINEL[self.dtype][0])
        return same[self.pad:self.pad + self.rows, :self.n]

    def check_guard(self, what):
        same = self.bits() == self.before.view(_SENTINEL[self.dtype][0])
        same[self.pad:self.pad + self.rows, :self.n] = True
        if not bool(same.all()):
            r, c = torch.nonzero(~same)[0].tolist()
            raise AssertionError(f"{what}: {int((~same).sum())} guard elements changed, first at buffer row {r} col {c} "
                                 f"(output rows {self.pad}..{self.pad + self.rows - 1}, columns < {self.n})")


def gemm(a, w, *, epi, act="ACT_NONE", bn=0, rows, n_out, k, lda=None, batches=1, bias=None, out=None, out16b=None,
         resid=None, ldo=0, gate=None, step_ptr=None, gate_step_stride=0, row_len=None, seq=0, rope=None, inner=0,
         pe_heads=0, norm=None, dim_head=0, weights_static=0, skip=0, conv_taps=0):
    g = _lib.GemmArgs()
    g.rows, g.batches, g.n_out, g.k = rows, batches, n_out, k
    g.lda, g.ldw = (k if lda is None else lda), k
    g.bn, g.epi, g.act, g.conv_taps = bn, EPI[epi], ACT[act], conv_taps
    ptr = lambda t: None if t is None else (t.ptr() if isinstance(t, Guarded) else t.data_ptr())  # noqa: E731
    g.bias, g.out, g.out16b, g.resid, g.ldo = ptr(bias), ptr(out), ptr(out16b), ptr(resid), ldo
    g.gate, g.step_ptr, g.gate_step_stride = ptr(gate), ptr(step_ptr), gate_step_stride
    g.row_len, g.seq = ptr(row_len), seq
    if rope is not None:
        g.rope_cos, g.rope_sin = rope[0].data_ptr(), rope[1].data_ptr()
    g.inner, g.pe_heads = inner, pe_heads
    if norm is not None:
        g.q_norm, g.k_norm = norm[0].data_ptr(), norm[1].data_ptr()
    g.dim_head = 128 if epi.endswith("DH128") else dim_head
    g.weights_static, g.skip_padded_tiles = weights_static, skip
    _lib.check(_lib.lib().f5_gemm(a.data_ptr(), w.data_ptr(), C.byref(g), torch.cuda.current_stream().cuda_stream),
               "f5_gemm")
    torch.cuda.synchronize()


def planner_bn(M, N, K, epi, act="ACT_NONE"):
    return ops.gemm_tile(M, N, K, epi=EPI[epi], act=ACT[act], dim_head=128 if epi.endswith("DH128") else 64)[0]


def round_up(x, m):
    return (x + m - 1) // m * m


# ---------------------------------------------------------------------------------------------------------------------
# one GEMM case: inputs, launch, reference, checks
# ---------------------------------------------------------------------------------------------------------------------
def gemm_case(group, *, bn, epi, act="ACT_NONE", M, N, K, seed, has_bias=True, gate="none", seq=0, lens=None,
              ldo_extra=None, out16b=False, skip=0, H=0, pe_heads=0, weights_static=1, a_scale=1.0):
    """Run one plain or QKV GEMM inside guard bands and check every element against its float64 bound.  gate: "none",
    "vector" or "step" (row k of a [4, N + 16] table through step_ptr).  Returns (launch, outputs): launch(ws) runs the
    same GEMM again with weights_static = ws into fresh guarded outputs."""
    qkv = epi.startswith("EPI_QKV")
    dh = 128 if epi.endswith("DH128") else 64
    a = gen((M, K), seed, a_scale)
    w = gen((N, K), seed + 1, 1 / math.sqrt(K))
    bias = gen((N,), seed + 2, 0.3, torch.float32) if has_bias else None
    align = {"EPI_F32": 1, "EPI_RESID": 4}.get(epi, 8)
    ldo = round_up(N, align) + (align if ldo_extra is None else ldo_extra)
    row_len = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=DEV)
    kw = dict(epi=epi, act=act, bn=bn, rows=M, n_out=N, k=K, bias=bias, ldo=ldo, row_len=row_len, seq=seq, skip=skip)
    x0 = gv = step = None
    if epi == "EPI_RESID":
        x0 = gen((M, N), seed + 3, 1.0, torch.float32)
        if gate == "vector":
            gv = gen((N,), seed + 4, 0.5, torch.float32)
            kw["gate"] = gv
        elif gate == "step":
            table = gen((4, N + 16), seed + 4, 0.5, torch.float32)
            step = torch.tensor([2], dtype=torch.int32, device=DEV)
            kw.update(gate=table, step_ptr=step, gate_step_stride=N + 16)
            gv = table[2, :N]
    norm = None
    if qkv:
        inner = N // 3
        cs, sn = ops.rope_tables(seq, DEV, dim_head=dh)
        kw.update(rope=(cs, sn), inner=inner, pe_heads=pe_heads)
        if "NORM" in epi:
            norm = (gen((dh,), seed + 5, 0.1, torch.float32) + 1.0, gen((dh,), seed + 6, 0.1, torch.float32) + 1.0)
            kw["norm"] = norm

    def launch(ws):
        outs = {}
        if epi == "EPI_RESID":
            outs["resid"] = Guarded(M, N, ldo, torch.float32, init=x0)
            kw["resid"] = outs["resid"]
        else:
            outs["out"] = Guarded(M, N, ldo, torch.float16 if epi != "EPI_F32" else torch.float32)
            kw["out"] = outs["out"]
            if out16b:
                outs["out16b"] = Guarded(M, N, ldo, torch.float16)
                kw["out16b"] = outs["out16b"]
        gemm(a, w, weights_static=ws, **kw)
        return outs

    outs = launch(weights_static)
    what = f"{epi} {act} bn{bn} {M}x{N}x{K}"
    for name, gd in outs.items():
        gd.check_guard(f"{what} {name}")
    # rows of tiles the kernel skips: 128-row tiles all past one sample's length (skip_padded_tiles)
    skipped = torch.zeros(M, dtype=torch.bool, device=DEV)
    if skip and lens is not None:
        for m0 in range(0, M, 128):
            last = min(m0 + 128, M) - 1
            if m0 // seq == last // seq and m0 % seq >= lens[m0 // seq]:
                skipped[m0:last + 1] = True
    keep = torch.ones(M, dtype=torch.bool, device=DEV) if lens is None else KB.row_mask(M, seq, row_len, DEV)
    if qkv:
        ref, e = KB.qkv_ref(a, w, bias, cs, sn, seq, inner, pe_heads, dh, norm, row_len)
        got, bound = outs["out"].out(), KB.half_bound(ref, e)
    else:
        y, e = KB.linear_ref(a, w, bias)
        if act == "ACT_GELU_TANH":
            y, e = KB.gelu_tanh_ref(y, e)
        elif act == "ACT_GELU_ERF":
            y, e = KB.gelu_erf_ref(y, e)
        if epi == "EPI_RESID":
            ref, bound = KB.resid_ref(x0, gv, y, e)
            ref = torch.where(keep[:, None], ref, x0.to(F64))  # masked rows keep their residual bit for bit
            bound = torch.where(keep[:, None], bound, 0.0)
            got = outs["resid"].out()
        elif epi == "EPI_F16":
            ref, bound = torch.where(keep[:, None], y, 0.0), torch.where(keep[:, None], KB.half_bound(y, e), 0.0)
            got = outs["out"].out()
        else:  # EPI_F32: unmasked; the fp16 copy is the fp32 result rounded, masked rows 0
            ref, bound, got = y, e, outs["out"].out()
    computed = ~skipped[:, None]
    if bool(skipped.any()):
        for name, gd in outs.items():
            assert bool(gd.untouched()[skipped].all()), f"{what} {name}: a skipped tile was written"
    r = KB.assert_within(got[computed.expand_as(got)], ref[computed.expand_as(ref)], bound[computed.expand_as(bound)],
                         what)
    if "out16b" in outs:
        o16 = outs["out16b"].out()
        want = torch.where(keep[:, None], got.half(), torch.zeros_like(o16))
        assert torch.equal(o16[~skipped].view(torch.int16), want[~skipped].view(torch.int16)), \
            f"{what}: out16b is not the fp32 result rounded to fp16 with masked rows 0"
    record(group, what, r)
    return launch, outs


def assert_same_bits(o1, o2, what):
    for name in o1:
        assert torch.equal(o1[name].bits(), o2[name].bits()), f"{what}: {name} differs"


# ---------------------------------------------------------------------------------------------------------------------
# completeness
# ---------------------------------------------------------------------------------------------------------------------
def test_every_instantiation_has_a_test():
    """Each F5_GEMM_KERNEL(...) line of gemm.cu is a parameter of this module: an instantiation added without a test
    fails here."""
    with open(os.path.join(ROOT, "f5_tts_b200", "csrc", "gemm.cu")) as f:
        src = f.read()
    table = src[src.index("kGemmKernels[]"):src.index("#undef F5_GEMM_KERNEL")]
    found = {(int(bn), e, a, c == "true")
             for bn, e, a, c in re.findall(r"F5_GEMM_KERNEL\((\d+),\s*(\w+),\s*(\w+),\s*(true|false)\)", table)}
    assert len(found) == 30
    tested = set(PLAIN) | set(QKV) | set(CONV)
    assert found == tested, f"untested: {sorted(found - tested)}; not instantiated: {sorted(tested - found)}"


# ---------------------------------------------------------------------------------------------------------------------
# plain instantiations at edge shapes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bn,epi,act,conv", PLAIN)
def test_plain_instantiation_edges(bn, epi, act, conv):
    """Edge shapes of one instantiation:
      * M = 77 < 128, n_out = 100 (< bn from 128 up, a tail at 64), K = 8 (one k-block, mostly zero fill);
      * M = 300 (tail), an n_out tail, K = 712 (the input projection's width), no bias, rows masked by length;
      * M = 1876, more tiles than SMs (the persistent loop runs several rounds), K = 704 (Vocos' embedding width);
      * K = 64 (STAGES - 1) - 24 (fewer k-blocks than ring stages) with a K tail.
    EPI_F32 takes odd n_out and odd ldo (the scalar store path).  weights_static = 1 (W prefetched before the
    dependency wait) gives the bits of weights_static = 0, and a second launch repeats them."""
    odd = 1 if epi == "EPI_F32" else 0
    n_tiles = SMS // 15 + 1  # column tiles at M = 1876 (15 row tiles) for more tiles than SMs
    cases = [dict(M=77, N=100 + odd, K=8, ldo_extra=2 if odd else None),
             dict(M=300, N=3 * bn + 36 + odd, K=712, has_bias=False, seq=100, lens=[100, 37, 1]),
             dict(M=1876, N=(n_tiles - 1) * bn + 40 + odd, K=704, ldo_extra=3 if odd else None),
             dict(M=200, N=bn + 8 + odd, K=64 * (STAGES[bn] - 1) - 24)]
    for i, c in enumerate(cases):
        gate = "vector" if i != 1 else "none"
        launch, o1 = gemm_case("plain edges", bn=bn, epi=epi, act=act, seed=100 + 10 * i, gate=gate,
                               out16b=(epi == "EPI_F32" and i == 1), **c)
        what = f"bn{bn} {epi} {act} case {i}"
        assert_same_bits(o1, launch(0), what + " weights_static 1 vs 0")
        assert_same_bits(o1, launch(1), what + " repeated launch")


@pytest.mark.parametrize("bn,epi,act,conv", QKV)
def test_qkv_instantiation_edges(bn, epi, act, conv):
    """QKV (+ RMSNorm) + RoPE: M = 77 with n_out < bn where the head width allows it and K = 8; M = 2 x 150 with an
    n_out tail, K = 712, masked rows, rotary on the first head only, no bias; M = 1876 over more tiles than SMs at
    K = 704 with rotary on every head."""
    dh = 128 if epi.endswith("DH128") else 64
    h3 = 5 if dh == 64 else 3  # 3 inner = 960 / 1152: a tail at 128 / 256
    cases = [dict(M=77, seq=77, H=1, K=8, pe=1),
             dict(M=300, seq=150, H=h3, K=712, pe=1, lens=[150, 97], has_bias=False),
             dict(M=1876, seq=938, H=1024 // dh, K=704, pe=1024 // dh)]
    for i, c in enumerate(cases):
        H, pe = c.pop("H"), c.pop("pe")
        launch, o1 = gemm_case("qkv edges", bn=bn, epi=epi, N=3 * H * dh, H=H, pe_heads=pe, seed=200 + 10 * i, **c)
        what = f"bn{bn} {epi} case {i}"
        assert_same_bits(o1, launch(0), what + " weights_static 1 vs 0")
        assert_same_bits(o1, launch(1), what + " repeated launch")


# ---------------------------------------------------------------------------------------------------------------------
# the conv GEMM
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("epi,G,masked", [("EPI_F16", 64, True), ("EPI_RESID", 64, True), ("EPI_F16", 48, False),
                                          ("EPI_RESID", 48, True), ("EPI_F16", 8, True)])
def test_conv_gemm(epi, G, masked):
    """Grouped Conv1d(k=31, groups=16) + bias + Mish as 31 accumulated GEMMs per (row tile, group), G channels per group
    (64: the base model, 48: the Small configs, 8: the smallest allowed), batches = 3, N = 300, ldo > D.  Masked: row
    lengths [300, 100, 1] with skip_padded_tiles, input rows past a length zero (the engine clears them): row tiles
    all past their sample's length keep the output sentinel (F16) or the residual (RESID), rows past the length in
    computed tiles are 0 (F16) or keep their residual."""
    B, N, taps = 3, 300, 31
    D = 16 * G
    x = gen((B, N, D), 300 + G, 1.0)
    wp = gen((taps, D, G), 301 + G, 1 / math.sqrt(G * taps))
    bias = gen((D,), 302, 0.1, torch.float32)
    lens = [300, 100, 1] if masked else None
    row_len = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=DEV)
    keep = torch.ones((B, N), dtype=torch.bool, device=DEV)
    if masked:
        keep = torch.arange(N, device=DEV)[None, :] < row_len[:, None]
        x = torch.where(keep[..., None], x, torch.zeros_like(x))
    ldo = D + (8 if epi == "EPI_F16" else 4)
    x0 = gen((B * N, D), 303, 1.0, torch.float32)

    def launch(ws):
        if epi == "EPI_F16":
            o = Guarded(B * N, D, ldo, torch.float16)
            kw = dict(out=o)
        else:
            o = Guarded(B * N, D, ldo, torch.float32, init=x0)
            kw = dict(resid=o)
        gemm(x, wp, epi=epi, act="ACT_MISH", rows=N, batches=B, n_out=D, k=G, lda=D, bias=bias, ldo=ldo, seq=N,
             row_len=row_len, skip=1 if masked else 0, conv_taps=taps, weights_static=ws, **kw)
        return {"out": o}

    o = launch(1)["out"]
    what = f"conv {epi} G{G} masked{masked}"
    o.check_guard(what)
    y, e = KB.conv31_ref(x, wp, bias, G)
    y, e = KB.mish_ref(y, e)
    y, e = y.reshape(B * N, D), e.reshape(B * N, D)
    keep = keep.reshape(B * N)
    skipped = torch.zeros((B, N), dtype=torch.bool, device=DEV)
    if masked:
        for b, n in enumerate(lens):
            skipped[b, round_up(n, 128):] = True
    skipped = skipped.reshape(B * N)
    if epi == "EPI_F16":
        ref, bound = torch.where(keep[:, None], y, 0.0), torch.where(keep[:, None], KB.half_bound(y, e), 0.0)
        assert bool(o.untouched()[skipped].all()), what + ": a skipped tile was written"
    else:
        ref, bound = KB.resid_ref(x0, None, y, e)
        ref, bound = torch.where(keep[:, None], ref, x0.to(F64)), torch.where(keep[:, None], bound, 0.0)
        skipped[:] = False  # the residual of every masked row is unchanged, skipped tile or not
    r = KB.assert_within(o.out()[~skipped], ref[~skipped], bound[~skipped], what)
    record("conv", what, r)
    # with tile skipping the plan turns the W prefetch off (the first tile may be skipped): the bits still agree
    assert_same_bits({"out": o}, launch(0), what + " weights_static 1 vs 0")


# ---------------------------------------------------------------------------------------------------------------------
# production shapes
# ---------------------------------------------------------------------------------------------------------------------
PROD = {  # name: (M, N, K, epi, act, bn, extra)
    "proj F32 + out16b": (1876, 1024, 712, "EPI_F32", "ACT_NONE", 128, dict(out16b=True, seq=938, lens=[938, 500])),
    "mod": (32, 6144, 1024, "EPI_F32", "ACT_NONE", 128, {}),
    "qkv planner": (1876, 3072, 1024, "EPI_QKV_ROPE", "ACT_NONE", 0, dict(seq=938, H=16)),
    "qkv bn128": (1876, 3072, 1024, "EPI_QKV_ROPE", "ACT_NONE", 128, dict(seq=938, H=16)),
    "qkv bn192": (1876, 3072, 1024, "EPI_QKV_ROPE", "ACT_NONE", 192, dict(seq=938, H=16)),
    "qkv bn256": (1876, 3072, 1024, "EPI_QKV_ROPE", "ACT_NONE", 256, dict(seq=938, H=16)),
    "qkv norm planner": (1876, 3072, 1024, "EPI_QKV_NORM_ROPE", "ACT_NONE", 0, dict(seq=938, H=16)),
    "oproj": (1876, 1024, 1024, "EPI_RESID", "ACT_NONE", 0, dict(gate="step", seq=938, lens=[938, 700])),
    "ff1 2D": (1876, 2048, 1024, "EPI_F16", "ACT_GELU_TANH", 0, {}),
    "ff1 4D": (1876, 4096, 1024, "EPI_F16", "ACT_GELU_TANH", 0, {}),
    "ff2": (1876, 1024, 2048, "EPI_RESID", "ACT_NONE", 0, dict(gate="step")),
    "out_proj": (1876, 100, 1024, "EPI_F32", "ACT_NONE", 128, {}),
    "text pw1": (1876, 1024, 512, "EPI_F16", "ACT_GELU_ERF", 128, {}),
    "text pw2": (1876, 512, 1024, "EPI_RESID", "ACT_NONE", 64, {}),
    "vocos embed": (1200, 512, 704, "EPI_F32", "ACT_NONE", 64, {}),
    "vocos pw1": (1200, 1536, 512, "EPI_F16", "ACT_GELU_ERF", 128, {}),
    "vocos pw2": (1200, 512, 1536, "EPI_RESID", "ACT_NONE", 64, dict(gate="vector")),
    "vocos head": (1200, 1026, 512, "EPI_F32", "ACT_NONE", 128, {}),
}


@pytest.mark.parametrize("name", list(PROD))
def test_production_shapes(name):
    """One GEMM per engine and Vocos call site at its real shape (base model: D = 1024, 16 heads, 938-frame batch of
    two; Vocos: 1200 frames), with the output leading dimension the call site uses (ldo = n_out) and the planner's tile
    where the call site leaves it to the planner."""
    M, N, K, epi, act, bn, extra = PROD[name]
    extra = dict(extra)
    if bn == 0:
        bn = planner_bn(M, N, K, epi, act)
    H = extra.pop("H", 0)
    gemm_case("production", bn=bn, epi=epi, act=act, M=M, N=N, K=K, seed=400 + len(name), ldo_extra=0, H=H,
              pe_heads=H, **extra)


# ---------------------------------------------------------------------------------------------------------------------
# engine options
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("epi,act", [("EPI_F16", "ACT_GELU_TANH"), ("EPI_QKV_ROPE", "ACT_NONE"),
                                     ("EPI_QKV_NORM_ROPE_DH128", "ACT_NONE"), ("EPI_RESID", "ACT_NONE"),
                                     ("EPI_F32", "ACT_NONE")])
def test_skip_padded_tiles(epi, act):
    """skip_padded_tiles over the flattened [samples x seq] rows (batches = 1), seq = 300 (not a multiple of 128),
    lengths [300, 40, 150]: rows 384-511 (all in sample 1, past 40) and 768-899 (sample 2, past 150) are skipped tiles
    and keep the sentinel bit for bit; tile 512-639 straddles samples 1 and 2 and is computed; rows past a length in a
    computed tile are 0 (fp16 outputs, the fp16 copy of EPI_F32) or keep their residual (EPI_RESID); EPI_F32's fp32
    rows are not masked."""
    seq, lens = 300, [300, 40, 150]
    M = seq * len(lens)
    dh = 128 if epi.endswith("DH128") else 64
    qkv = epi.startswith("EPI_QKV")
    H = 4 if qkv else 0
    N = 3 * H * dh if qkv else 640
    bn = 128
    gemm_case("skip padded tiles", bn=bn, epi=epi, act=act, M=M, N=N, K=256, seed=500, seq=seq, lens=lens, skip=1,
              H=H, pe_heads=H, out16b=epi == "EPI_F32", gate="step" if epi == "EPI_RESID" else "none")


@pytest.mark.parametrize("bn", [64, 128, 192, 256])
def test_gate_row_from_step_ptr(bn):
    """EPI_RESID with step_ptr -> k = 2 and a [4, N + 16] gate table whose rows differ: only row k is used."""
    gemm_case("step_ptr gate", bn=bn, epi="EPI_RESID", M=333, N=2 * bn + 8, K=320, seed=600, gate="step")


def test_plans_rejected_before_launch():
    """Arguments gemm_plan and attn_plan refuse before anything is launched."""
    a, w = gen((128, 64), 700), gen((128, 64), 701)
    o = torch.empty((128, 128), dtype=torch.float16, device=DEV)
    L = _lib.lib()
    for epi, ldo in (("EPI_F16", 132), ("EPI_RESID", 130)):
        with pytest.raises(_lib.F5LibraryError, match="ldo"):
            gemm(a, w, epi=epi, bn=128, rows=128, n_out=128, k=64, out=o, resid=o.float(), ldo=ldo)
    with pytest.raises(_lib.F5LibraryError, match="cta_pair"):
        ops.linear(a, w, epi=EPI["EPI_F16"], bn=128, pair=1)
    qkv = gen((128, 3 * 64), 702)
    assert L.f5_attention_dh(qkv.data_ptr(), o.data_ptr(), 1, 128, 1, 96, None, 0.1,
                             torch.cuda.current_stream().cuda_stream) == -1
    assert L.f5_attention_dh(qkv.data_ptr(), o.data_ptr(), 0, 128, 1, 64, None, 0.1,
                             torch.cuda.current_stream().cuda_stream) == -1


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
def attention_case(group, *, dh, Be, seq, H, kv, seed, scale=None, pattern=None):
    """Attention over a fused [Be * seq, 3 inner] QKV buffer followed by NaN rows (outside its tensor map, never read),
    into an output with sentinel rows before and after it.

    Contract on key and value rows at or past a sample's kv_len: inside the last key tile they are loaded and multiplied
    by P = 0, so they must be finite (the engine clears the QKV buffer before a key-masked call); here they hold
    +-6e4.  Rows in key tiles past the last one are never loaded: here they hold NaN.  Neither may change the output."""
    inner = H * dh
    x = gen((Be * seq, 3 * inner), seed, 1.0).double().view(Be, seq, 3, H, dh)
    if pattern is not None:
        pos = torch.arange(seq, device=DEV, dtype=F64)[None, :, None, None]
        if pattern == "wide":
            x[:, :, 0] *= 3.0
            x[:, :, 1] *= 3.0
        elif pattern == "rising":
            x[:, :, 1] *= 1.0 + pos / 128.0
        elif pattern == "falling":
            x[:, :, 1] *= 6.0 / (1.0 + pos / 64.0)
        elif pattern == "spike":
            x[:, :, 0] = x[:, :, 0].abs()
            x[:, min(600, seq - 1), 1] = 12.0
    x = x.half()
    kv_len = None if kv is None else torch.tensor(kv, dtype=torch.int32, device=DEV)
    q, k, v = (x[:, :, i].permute(0, 2, 1, 3) for i in range(3))  # [Be, H, seq, dh]
    ref, bound = KB.attention_ref(q, k, v, kv_len, scale)
    buf = torch.full((Be * seq + 5, 3 * inner), float("nan"), dtype=torch.float16, device=DEV)
    xb = buf[:Be * seq].view(Be, seq, 3, H, dh)
    xb.copy_(x)
    if kv is not None:
        g = torch.Generator().manual_seed(seed + 1)
        for b, n in enumerate(kv):
            end = min(round_up(n, 128), seq)
            sign = torch.randint(0, 2, (end - n, 2, H, dh), generator=g).to(DEV) * 2.0 - 1.0
            xb[b, n:end, 1:] = (6e4 * sign).half()
            xb[b, end:, 1:] = float("nan")
    out = Guarded(Be * seq, inner, inner, torch.float16)
    sc = dh ** -0.5 if scale is None else scale
    _lib.check(_lib.lib().f5_attention_dh(buf.data_ptr(), out.ptr(), Be, seq, H, dh,
                                          None if kv_len is None else kv_len.data_ptr(), sc,
                                          torch.cuda.current_stream().cuda_stream), "f5_attention_dh")
    torch.cuda.synchronize()
    what = f"attention dh{dh} Be{Be} seq{seq} H{H} kv{kv} scale{scale} {pattern or ''}"
    out.check_guard(what)
    got = out.out().view(Be, seq, H, dh).permute(0, 2, 1, 3)
    r = KB.assert_within(got, ref, bound, what)
    record(group, what, r)


@pytest.mark.parametrize("kvset", ["a", "b"])
@pytest.mark.parametrize("seq", [1, 77, 127, 128, 129, 469, 1876])
@pytest.mark.parametrize("dh", [64, 128])
def test_attention_shapes(dh, seq, kvset):
    """Be = 3 samples with different key lengths from {1, 127, 128, 129, seq} (clamped to seq), H = 2; set "b" with
    a non-default scale."""
    kv = [seq, 1, 129] if kvset == "a" else [127, 128, seq]
    kv = [min(n, seq) for n in kv]
    attention_case("attention", dh=dh, Be=3, seq=seq, H=2, kv=kv, seed=800 + seq + dh,
                   scale=0.09 if kvset == "b" else None)


@pytest.mark.parametrize("pattern", ["wide", "rising", "falling", "spike"])
@pytest.mark.parametrize("dh", [64, 128])
def test_attention_logit_patterns(dh, pattern):
    """Logits with large jumps between key tiles, rising and falling across tiles, and one key far above all before it
    (the running max and the rescale of o and l), without a key mask."""
    attention_case("attention patterns", dh=dh, Be=2, seq=700, H=2, kv=None, seed=900 + dh, pattern=pattern)
