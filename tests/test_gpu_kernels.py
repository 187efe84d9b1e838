"""GPU parity of the individual sm_90a kernels (called through the C ABI) against plain PyTorch fp32 references of the
same op evaluated on the SAME fp16-rounded operands.  Tolerances (written here, per the north star's "stated fp
tolerance"): fp32 outputs rel-L2 <= 2e-4 (fp32 accumulation-order noise), fp16 outputs rel-L2 <= 1.5e-3 and
max-abs <= 4e-3 * max|ref| (one fp16 rounding), attention rel-L2 <= 3e-3 (P is rounded to fp16 before P.V).
"""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from f5_tts_b200 import _lib, ops  # noqa: E402
from f5_tts_b200.ops import (ACT_GELU_ERF, ACT_GELU_TANH, ACT_NONE, EPI_F16, EPI_F32, EPI_QKV_ROPE,  # noqa: E402
                             EPI_RESID)

DEV = "cuda:0"


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20))


def report(name, got, ref):
    d = (got.float() - ref.float()).abs()
    print(f"[{name}] rel-L2 {rel(got, ref):.3e} max|d| {float(d.max()):.3e} max|ref| {float(ref.abs().max()):.3e}")


def gen(shape, seed, scale=1.0, dtype=torch.float16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).to(DEV)


@pytest.mark.parametrize("M,N,K,bn", [(128, 128, 64, 128), (128, 128, 256, 128), (256, 256, 128, 64), (1876, 1024, 1024, 64),
                                      (1876, 2048, 1024, 128), (333, 100, 1024, 128), (1000, 512, 768, 64),
                                      (77, 3072, 1024, 128), (32, 4096, 1024, 128), (1876, 1024, 712 // 8 * 8, 128)])
def test_gemm_f32(M, N, K, bn):
    a, w = gen((M, K), 1), gen((N, K), 2, 1 / math.sqrt(K))
    bias = gen((N,), 3, 1.0, torch.float32)
    out = ops.linear(a, w, bias, epi=EPI_F32, bn=bn)
    ref = a.float() @ w.float().t() + bias
    report(f"gemm_f32 {M}x{N}x{K} bn{bn}", out, ref)
    assert rel(out, ref) <= 2e-4


@pytest.mark.parametrize("M,N,K,bn", [(256, 256, 64, 256), (1876, 2048, 1024, 256), (1876, 3072, 1024, 128), (700, 1024, 2048, 128),
                                      (129, 512, 192, 256), (30000 // 8, 2048, 1024, 256), (1876, 3072, 1024, 192),
                                      (500, 1024, 2048, 192)])
def test_gemm_wide_tiles(M, N, K, bn):
    """128-, 192- and 256-wide tiles, including M not a multiple of 128 and K = 2048: fp16+GELU, fp32 residual add and
    QKV+RoPE epilogues."""
    a, w = gen((M, K), 31), gen((N, K), 32, 1 / math.sqrt(K))
    bias = gen((N,), 33, 0.5, torch.float32)
    ref = a.float() @ w.float().t() + bias
    out = ops.linear(a, w, bias, epi=EPI_F16, act=ACT_GELU_TANH, bn=bn)
    report(f"f16 gelu {M}x{N}x{K} bn{bn}", out, F.gelu(ref, approximate="tanh"))
    assert rel(out, F.gelu(ref, approximate="tanh")) <= 1.5e-3
    x0 = gen((M, N), 34, 1.0, torch.float32)
    gate = gen((N,), 35, 0.5, torch.float32)
    x = x0.clone()
    ops.linear(a, w, bias, epi=EPI_RESID, bn=bn, resid=x, gate=gate)
    assert rel(x, x0 + gate * ref) <= 2e-4
    if N % 192 == 0:
        seq, inner = M // 2, N // 3
        cs, sn = ops.rope_tables(seq, DEV)
        o = ops.linear(a[: 2 * seq], w, bias, epi=EPI_QKV_ROPE, bn=bn, seq=seq, rope=(cs, sn), inner=inner, pe_heads=1)
        o1 = ops.linear(a[: 2 * seq], w, bias, epi=EPI_QKV_ROPE, bn=128, seq=seq, rope=(cs, sn), inner=inner, pe_heads=1)
        assert rel(o, o1) <= 1e-6  # the tile width does not change the arithmetic


def test_gemm_rejects_cta_pair():
    """There are no cluster-pair tiles: a request for one is an error, not a silent single-CTA run."""
    a, w = gen((256, 128), 36), gen((256, 128), 37)
    with pytest.raises(_lib.F5LibraryError):
        ops.linear(a, w, epi=EPI_F16, bn=128, pair=1)


@pytest.mark.parametrize("act", [ACT_NONE, ACT_GELU_TANH, ACT_GELU_ERF])
@pytest.mark.parametrize("bn", [64, 128, 192, 256, 0])
def test_gemm_f16_act(act, bn):
    if act == ACT_GELU_ERF and bn == 192:
        pytest.skip("not instantiated")
    M, N, K = 700, 2048, 1024
    a, w = gen((M, K), 4), gen((N, K), 5, 1 / math.sqrt(K))
    bias = gen((N,), 6, 0.5, torch.float32)
    out = ops.linear(a, w, bias, epi=EPI_F16, act=act, bn=bn)
    # model weights may be fetched ahead of the programmatic-launch dependency wait: same bits either way
    assert torch.equal(out, ops.linear(a, w, bias, epi=EPI_F16, act=act, bn=bn, static_w=True))
    ref = a.float() @ w.float().t() + bias
    if act == ACT_GELU_TANH:
        ref = F.gelu(ref, approximate="tanh")
    elif act == ACT_GELU_ERF:
        ref = F.gelu(ref)
    report(f"gemm_f16 act{act} bn{bn}", out, ref)
    assert rel(out, ref) <= 1.5e-3
    assert float((out.float() - ref).abs().max()) <= 4e-3 * float(ref.abs().max())


@pytest.mark.parametrize("bn", [64, 128, 192, 0])
def test_gemm_resid_gate_mask(bn):
    M, N, K, seq = 3 * 200, 1024, 2048, 200
    a, w = gen((M, K), 7), gen((N, K), 8, 1 / math.sqrt(K))
    bias, gate = gen((N,), 9, 0.3, torch.float32), gen((N,), 10, 0.5, torch.float32)
    x0 = gen((M, N), 11, 1.0, torch.float32)
    row_len = torch.tensor([200, 150, 1], dtype=torch.int32, device=DEV)
    x = x0.clone()
    ops.linear(a, w, bias, epi=EPI_RESID, bn=bn, resid=x, gate=gate, row_len=row_len, seq=seq)
    y = a.float() @ w.float().t() + bias
    mask = (torch.arange(seq, device=DEV)[None, :] < row_len[:, None]).reshape(M, 1)
    ref = x0 + gate[None, :] * torch.where(mask, y, torch.zeros_like(y))
    report(f"gemm_resid bn{bn}", x, ref)
    assert rel(x, ref) <= 2e-4
    # no gate, no mask
    x = x0.clone()
    ops.linear(a, w, bias, epi=EPI_RESID, bn=bn, resid=x)
    assert rel(x, x0 + y) <= 2e-4


@pytest.mark.parametrize("pe_heads,bn", [(1, 128), (16, 256), (1, 256), (1, 192), (16, 192), (1, 0)])
def test_gemm_qkv_rope(pe_heads, bn):
    Be, seq, D, H = 2, 300, 1024, 16
    inner = H * 64
    a, w = gen((Be * seq, D), 12), gen((3 * inner, D), 13, 1 / math.sqrt(D))
    bias = gen((3 * inner,), 14, 0.2, torch.float32)
    cs, sn = ops.rope_tables(seq, DEV)
    out = ops.linear(a, w, bias, epi=EPI_QKV_ROPE, bn=bn, seq=seq, rope=(cs, sn), inner=inner, pe_heads=pe_heads)
    y = (a.float() @ w.float().t() + bias).view(Be, seq, 3, H, 32, 2)
    c, s = cs.view(1, seq, 1, 1, 32), sn.view(1, seq, 1, 1, 32)
    rot = torch.stack((y[..., 0] * c - y[..., 1] * s, y[..., 1] * c + y[..., 0] * s), dim=-1)
    ref = y.clone()
    ref[:, :, :2, :pe_heads] = rot[:, :, :2, :pe_heads]
    ref = ref.reshape(Be * seq, 3 * inner)
    report(f"qkv_rope pe{pe_heads} bn{bn}", out, ref)
    assert rel(out, ref) <= 1.5e-3


@pytest.mark.parametrize("B,N,masked", [(1, 256, False), (2, 300, True), (1, 938, False), (3, 77, True)])
def test_grouped_conv31(B, N, masked):
    D = 1024
    x = gen((B, N, D), 15)
    w = gen((D, 64, 31), 16, 1 / math.sqrt(64 * 31))
    bias = gen((D,), 17, 0.1, torch.float32)
    lens = None
    if masked:
        lens = torch.tensor([N, max(1, N // 2), 5][:B], dtype=torch.int32, device=DEV)
        m = (torch.arange(N, device=DEV)[None, :] < lens[:, None])[..., None]
        x = torch.where(m, x, torch.zeros_like(x))
    wp = w.permute(2, 0, 1).contiguous()
    out = ops.grouped_conv31(x.contiguous(), wp, bias, row_len=lens)
    # reference on the CPU: cuDNN's grouped fp32 conv1d can stall for minutes on first use
    y = F.conv1d(x.float().cpu().transpose(1, 2), w.float().cpu(), bias.cpu(), padding=15, groups=16).transpose(1, 2)
    y = y.to(DEV)
    if masked:
        y = torch.where(m, y, torch.zeros_like(y))
    ref = F.mish(y)
    report(f"conv31 B{B} N{N} masked{masked}", out, ref)
    assert rel(out, ref) <= 1.5e-3
    r0 = gen((B, N, D), 18, 1.0, torch.float32)
    r = r0.clone()
    ops.grouped_conv31(x.contiguous(), wp, bias, resid=r, row_len=lens)
    assert rel(r, r0 + ref) <= 2e-4


@pytest.mark.parametrize("Be,seq,H,kv", [(1, 128, 1, None), (2, 128, 2, None), (2, 300, 16, None), (2, 938, 16, None),
                                         (3, 200, 4, [200, 131, 7]), (1, 1876, 2, None), (2, 129, 3, [129, 128])])
def test_attention(Be, seq, H, kv):
    inner = H * 64
    qkv = gen((Be * seq, 3 * inner), 19, 1.0)
    kv_len = None if kv is None else torch.tensor(kv, dtype=torch.int32, device=DEV)
    out = ops.attention(qkv, Be, seq, H, kv_len)
    q, k, v = qkv.float().view(Be, seq, 3, H, 64).permute(2, 0, 3, 1, 4)
    mask = None
    if kv is not None:
        mask = (torch.arange(seq, device=DEV)[None, :] < kv_len[:, None])[:, None, None, :].expand(Be, H, seq, seq)
    ref = F.scaled_dot_product_attention(q, k, v, attn_mask=mask).transpose(1, 2).reshape(Be * seq, inner)
    report(f"attention Be{Be} seq{seq} H{H} kv{kv}", out, ref)
    assert rel(out, ref) <= 3e-3


@pytest.mark.parametrize("mode", ["wide", "rising", "falling", "spike"])
def test_attention_reference_tracking(mode):
    """The attention kernel folds the softmax reference into the Q K^T accumulator one tile ahead and only checks row
    sums on its fast path: scores that outgrow the reference (slowly, abruptly, by more than the fp16 range) must take
    the rescale / exact-path branches and still match the fp32 softmax."""
    Be, seq, H = 2, 700, 2
    inner = H * 64
    qkv = gen((Be * seq, 3 * inner), 23, 1.0).float().view(Be, seq, 3, H, 64)
    pos = torch.arange(seq, device=DEV, dtype=torch.float32)[None, :, None, None]
    if mode == "wide":       # logits with a standard deviation of ~13 (log2 units): large jumps between key tiles
        qkv[:, :, 0] *= 3.0
        qkv[:, :, 1] *= 3.0
    elif mode == "rising":   # every key tile is larger than the one before
        qkv[:, :, 1] *= 1.0 + pos / 128.0
    elif mode == "falling":  # the first tile dominates: later probabilities underflow exactly like the reference's
        qkv[:, :, 1] *= 6.0 / (1.0 + pos / 64.0)
    elif mode == "spike":    # one key in the fifth tile with a score far above everything before it
        qkv[:, :, 0] = qkv[:, :, 0].abs()
        qkv[:, 600, 1] = 12.0
    qkv = qkv.half().reshape(Be * seq, 3 * inner).contiguous()
    out = ops.attention(qkv, Be, seq, H)
    q, k, v = qkv.float().view(Be, seq, 3, H, 64).permute(2, 0, 3, 1, 4)
    ref = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(Be * seq, inner)
    report(f"attention reference tracking: {mode}", out, ref)
    assert torch.isfinite(out.float()).all()
    assert rel(out, ref) <= 5e-3  # one more fp16 rounding of the scaled queries shows at logits of this size


@pytest.mark.parametrize("D", [1024, 512, 128])
def test_row_norm(D):
    rows = 1000
    x = gen((rows, D), 20, 2.0, torch.float32) + 0.5
    a, b = gen((D,), 21, 0.3, torch.float32), gen((D,), 22, 0.3, torch.float32)
    ln = F.layer_norm(x, (D,), eps=1e-6)
    assert rel(ops.row_norm(x, 0, a, b), ln * (1 + a) + b) <= 1e-3
    assert rel(ops.row_norm(x, 1, a, b), ln * a + b) <= 1e-3
    assert rel(ops.row_norm(x, 2, a), F.normalize(x, dim=-1) * D ** 0.5 * a) <= 1e-3


def test_mel_frontend_vs_golden(golden_dir):
    from f5_tts_b200.model import MelSpec

    z = np.load(os.path.join(golden_dir, "mel_vocos.npz"))
    wav = torch.from_numpy(z["wav"]).to(DEV)
    ms = MelSpec().to(DEV)
    mel = ms(wav)
    ref = torch.from_numpy(z["mel"]).to(DEV)
    report("mel", mel, ref)
    assert mel.shape == ref.shape
    # log-mel of a random signal: absolute tolerance on the log value (fp32 FFT, different summation order)
    assert float((mel - ref).abs().max()) <= 2e-3
    mel_t = ms(wav, frames_last=False)
    assert torch.equal(mel_t.permute(0, 2, 1), mel)
    # odd length + short clip
    w2 = wav[:, :5000].contiguous()
    import torchaudio

    ta = torchaudio.transforms.MelSpectrogram(sample_rate=24000, n_fft=1024, win_length=1024, hop_length=256, n_mels=100,
                                              power=1, center=True, normalized=False, norm=None).to(DEV)
    assert float((ms(w2) - ta(w2).clamp(min=1e-5).log()).abs().max()) <= 2e-3


def test_vocos_decode(golden_dir):
    from f5_tts_b200.vocoder import Vocos
    from oracle import f5_oracle as O

    z = np.load(os.path.join(golden_dir, "vocos_oracle_frozen.npz"))
    voc = Vocos()
    voc.load_state_dict(O.synthetic_vocos_state_dict(), strict=False)
    voc = voc.to(DEV)
    mel = torch.from_numpy(z["mel"]).to(DEV)
    wav = voc.decode(mel)
    ref = torch.from_numpy(z["wav"]).to(DEV)
    report("vocos", wav, ref)
    assert wav.shape == ref.shape
    assert rel(wav, ref) <= 1e-2  # fp16 GEMM operands through 8 ConvNeXt blocks + exp() head (SURVEY.md §8c gate)
    # batch of 2, different length
    g = torch.Generator().manual_seed(5)
    mel2 = (torch.randn(2, 100, 33, generator=g) * 1.5 - 2.0)
    ref2 = O.vocos_decode(O.synthetic_vocos_state_dict(), mel2)
    assert rel(voc.decode(mel2.to(DEV)).cpu(), ref2) <= 1e-2
