"""GPU: EPI_RESID_SAMPLE, the gated residual epilogue f5_forward runs (each output row reads the gate row of its sample,
(row / gate_seq) % gate_samples), against the EPI_RESID kernel launched once per sample through f5_gemm with that
sample's gate row.  EPI_RESID is checked element by element against float64 in tests/test_gpu_gemm_attn_exact.py; here
every element must equal it bit for bit, at every width of gemm.cu's kGemmSampleKernels, with cond | uncond packing
(rows b and B + b share a gate row), n_out tails, rows masked by length and padded tiles skipped."""
import ctypes as C
import os
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from f5_tts_b200 import _lib  # noqa: E402

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDTHS = [128, 192, 256]
_hooks = None


def hooks():
    global _hooks
    if _hooks is None:
        L = C.CDLL(_lib.KERNELS_LIB_PATH)
        L.f5k_last_error.restype = C.c_char_p
        L.f5k_gemm_resid_sample.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(_lib.GemmArgs), C.c_int, C.c_int,
                                            C.c_void_p]
        _hooks = L
    return _hooks


def test_every_sample_gate_width_has_a_test():
    with open(os.path.join(ROOT, "f5_tts_b200", "csrc", "gemm.cu")) as f:
        src = f.read()
    line = src[src.index("kGemmSampleKernels[]"):]
    line = line[:line.index(";")]
    assert sorted(int(w) for w in re.findall(r"sample_gate_kernel<(\d+)>", line)) == WIDTHS


def args(*, bn, rows, n_out, k, bias, resid, ldo, gate, stride, row_len=None, seq=0, skip=0):
    a = _lib.GemmArgs()
    a.rows, a.batches, a.n_out, a.k, a.lda, a.ldw, a.bn = rows, 1, n_out, k, k, k, bn
    a.epi, a.act = _lib.EPI_RESID, _lib.ACT_NONE
    a.bias, a.resid, a.ldo = bias.data_ptr(), resid, ldo
    a.gate, a.gate_step_stride = gate, stride
    a.row_len, a.seq, a.skip_padded_tiles, a.weights_static = row_len, seq, skip, 1
    return a


@pytest.mark.parametrize("bn", WIDTHS)
@pytest.mark.parametrize("case", ["packed", "cond", "masked"])
def test_sample_gates_equal_per_sample_launches(bn, case):
    g = torch.Generator().manual_seed(bn + len(case))
    S, seq, K = 3, 300, 712
    Be = 2 * S if case != "cond" else S
    M, N = Be * seq, 3 * bn + 36
    ldo, stride = N + 4, N + 20
    A = (torch.randn(M, K, generator=g)).half().to(DEV)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).half().to(DEV)
    bias = (0.3 * torch.randn(N, generator=g)).to(DEV)
    table = (0.5 * torch.randn(S, stride, generator=g)).to(DEV)
    x0 = torch.randn(M, ldo, generator=g).to(DEV)
    lens = skip = None
    if case == "masked":
        lens = torch.tensor([300, 37, 171, 300, 37, 171], dtype=torch.int32, device=DEV)
        skip = 1
    stream = torch.cuda.current_stream().cuda_stream

    got = x0.clone()
    a = args(bn=bn, rows=M, n_out=N, k=K, bias=bias, resid=got.data_ptr(), ldo=ldo, gate=table.data_ptr(),
             stride=stride, row_len=None if lens is None else lens.data_ptr(), seq=seq, skip=skip or 0)
    rc = hooks().f5k_gemm_resid_sample(A.data_ptr(), W.data_ptr(), C.byref(a), seq, S, stream)
    assert rc == 0, hooks().f5k_last_error().decode()

    want = x0.clone()
    for b in range(Be):
        r0 = b * seq
        a = args(bn=bn, rows=seq, n_out=N, k=K, bias=bias, resid=want[r0:].data_ptr(), ldo=ldo,
                 gate=table[b % S].data_ptr(), stride=0, row_len=None if lens is None else lens[b:].data_ptr(),
                 seq=seq, skip=skip or 0)
        _lib.check(_lib.lib().f5_gemm(A[r0:].data_ptr(), W.data_ptr(), C.byref(a), stream), "f5_gemm")
    torch.cuda.synchronize()
    assert torch.equal(got, want), f"bn {bn} {case}: {int((got != want).sum())} elements differ"
    assert not torch.equal(got[:, :N], x0[:, :N])  # the epilogue wrote
    if lens is not None:  # rows past a sample's length keep their residual
        for b in range(Be):
            assert torch.equal(got[b * seq + int(lens[b]):(b + 1) * seq], x0[b * seq + int(lens[b]):(b + 1) * seq])
