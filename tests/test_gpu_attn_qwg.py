"""GPU: the dh-64 attention kernels at 256 queries per CTA (4 consumer warpgroups) against 128 (2).

  * f5_attention_qwg forced to 4, element by element against the float64 reference of oracle/kernel_bounds.py, at
    sequence lengths whose last 256-row block leaves 0, 1, 2 or 3 warpgroups without a query row, with and without
    per-sample key lengths, Be 1 to 3, and the logit patterns of test_gpu_gemm_attn_exact.py;
  * the same call forced to 2 gives the same output bit for bit, and so does the joint (MMDiT) kernel;
  * the planner picks 4 where the 128-query grid needs two waves and 2 where it fits in one.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from f5_tts_b200 import _lib, ops  # noqa: E402
from oracle import kernel_bounds as KB  # noqa: E402

DEV = "cuda:0"
F64 = torch.float64


def stream():
    return torch.cuda.current_stream().cuda_stream


def make_qkv(Be, seq, H, seed, pattern):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(Be, seq, 3, H, 64, generator=g, dtype=F64).to(DEV)
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
    return x.half()


def attention(x, kv_len, qwg, scale):
    Be, seq, _, H, dh = x.shape
    out = torch.full((Be * seq, H * dh), float("nan"), dtype=torch.float16, device=DEV)
    _lib.check(_lib.lib().f5_attention_qwg(x.data_ptr(), out.data_ptr(), Be, seq, H, dh, ops._ptr(kv_len), scale, qwg,
                                           stream()), "f5_attention_qwg")
    torch.cuda.synchronize()
    return out


# seq -> warpgroups of the last 256-row block with no query row: 90 (2), 200 (0), 257 (3), 469 (0), 700 (1), 938 (1),
# 1875 (2)
@pytest.mark.parametrize("pattern", [None, "wide", "rising", "falling", "spike"])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("seq", [90, 200, 257, 469, 700, 938, 1875])
def test_attention_qwg4(seq, masked, pattern):
    Be = 1 + seq % 3
    H = 2
    x = make_qkv(Be, seq, H, 1000 + seq, pattern)
    kv = [max(1, seq - 131 * b) for b in range(Be)] if masked else None
    kv_len = None if kv is None else torch.tensor(kv, dtype=torch.int32, device=DEV)
    got4 = attention(x, kv_len, 4, 0.125)
    got2 = attention(x, kv_len, 2, 0.125)
    assert torch.equal(got4.view(torch.int16), got2.view(torch.int16)), "qwg 4 and qwg 2 differ"
    q, k, v = (x[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    ref, bound = KB.attention_ref(q, k, v, kv_len, 0.125)
    KB.assert_within(got4.view(Be, seq, H, 64).permute(0, 2, 1, 3), ref, bound,
                     f"attention qwg4 Be{Be} seq{seq} kv{kv} {pattern}")


@pytest.mark.parametrize("lens", ["none", "lengths", "c_len0"])
@pytest.mark.parametrize("N,nt", [(90, 17), (257, 130), (938, 150), (1875, 300)])
def test_attention_joint_qwg4_equals_qwg2(N, nt, lens):
    Be, H, dh = 2, 4, 64
    inner = H * dh
    g = torch.Generator().manual_seed(N + nt)
    qkv = torch.randn(Be * N, 3 * inner, generator=g).half().to(DEV)
    qkv_c = torch.randn(Be * nt, 3 * inner, generator=g).half().to(DEV)
    if lens == "none":
        kv_t = kc_t = None
    else:
        kc = [nt - 5, 0] if lens == "c_len0" else [nt, max(1, nt - 13)]
        kv_t = torch.tensor([N, max(1, N - 77)], dtype=torch.int32, device=DEV)
        kc_t = torch.tensor(kc, dtype=torch.int32, device=DEV)
    res = {}
    for qwg in (2, 4):
        out = torch.full((Be * N, inner), float("nan"), dtype=torch.float16, device=DEV)
        out_c = torch.full((Be * nt, inner), float("nan"), dtype=torch.float16, device=DEV)
        _lib.check(_lib.lib().f5_attention_joint_qwg(qkv.data_ptr(), qkv_c.data_ptr(), out.data_ptr(), out_c.data_ptr(),
                                                     Be, N, nt, H, dh, ops._ptr(kv_t), ops._ptr(kc_t), 1, dh ** -0.5,
                                                     qwg, stream()), "f5_attention_joint_qwg")
        torch.cuda.synchronize()
        res[qwg] = (out, out_c)
    ref_out, ref_c = ops.attention_joint(qkv, qkv_c, Be, N, nt, H, kv_len=kv_t, c_len=kc_t, dim_head=dh)
    torch.cuda.synchronize()
    for a, b, r in zip(res[4], res[2], (ref_out, ref_c)):
        assert not bool(a.isnan().any())
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
        assert torch.equal(a.view(torch.int16), r.view(torch.int16))


def test_qwg_arguments_rejected():
    qkv = torch.zeros(128, 3 * 128, dtype=torch.float16, device=DEV)
    o = torch.zeros(128, 128, dtype=torch.float16, device=DEV)
    L = _lib.lib()
    assert L.f5_attention_qwg(qkv.data_ptr(), o.data_ptr(), 1, 128, 1, 128, None, 0.1, 4, stream()) == -1  # dh 128
    assert L.f5_attention_qwg(qkv.data_ptr(), o.data_ptr(), 1, 128, 2, 64, None, 0.1, 3, stream()) == -1


@pytest.mark.skipif(torch.cuda.get_device_properties(0).multi_processor_count != 132, reason="shapes checked on 132 SMs")
def test_planner_choice():
    L = _lib.lib()
    assert L.f5_attention_qwg_choice(2, 938, 16, 64) == 4  # 256 CTAs of 128 queries: two waves
    assert L.f5_attention_qwg_choice(2, 469, 16, 64) == 2  # 128 CTAs: one wave
    assert L.f5_attention_qwg_choice(16, 1875, 16, 64) == 4
    assert L.f5_attention_qwg_choice(2, 938, 16, 128) == 2  # head width 128 stays at 2
