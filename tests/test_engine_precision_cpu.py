"""CPU: oracle/engine_precision, the fp16-storage model of the engine, and the stress weights of the frame tests
(tests/test_gpu_forward_frames_f64.py).

  * with identity rounding the float64 path equals the fp32 oracle to within fp32 rounding, for every backbone;
  * the fp16 emulation sits at the distance from float64 that fp16 storage predicts (a few 1e-4), uniformly over
    frames, and each of its two parts (weights, activations) contributes;
  * leaving the context restores the oracle modules' `F`, also when the block raises;
  * the stress weights, per config, in float64: zeroing attention moves the output by a large fraction, a one-position
    RoPE shift of the rows >= 128 moves it by at least 10x the emulated fp16 noise, and every fp16-stored value stays
    far inside the fp16 range.
"""
import pytest
import torch
import torch.nn.functional as TF

from oracle import engine_precision as EP
from oracle import f5_oracle as O

CONFIGS = EP.stress_configs()
IDENT = lambda v: v  # noqa: E731


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def inputs(cfg, B, N, nt, seed=3):
    g = torch.Generator().manual_seed(seed)
    x, cond = torch.randn(B, N, 100, generator=g), torch.randn(B, N, 100, generator=g)
    text = torch.randint(0, cfg.text_num_embeds, (B, nt), generator=g)
    text[-1, nt // 2:] = -1
    t = torch.linspace(0.0, 0.996, B)
    return x, cond, text, t


def run(sd, cfg, args, rnd=IDENT, mask=None, patch=None):
    """float64 forward (CFG-packed) with the engine's fp16 storage emulated by `rnd` (IDENT: plain float64)"""
    sd64 = EP.engine_state_dict(sd, rnd=rnd)
    with EP.fp16_storage(sd64, rnd=rnd) as ns:
        if patch:
            patch(ns)
        return EP.forward(sd64, cfg, *args, mask, True)


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_identity_rounding_equals_fp32_oracle(name):
    cfg = CONFIGS[name]
    sd = EP.stress_state_dict(cfg)
    args = inputs(cfg, 2, 70, 30)
    mask = O.lens_to_mask(torch.tensor([70, 41]))
    for m in (None, mask):
        ref32 = EP.forward(sd, cfg, *args, m, True)
        got = run(sd, cfg, args, mask=m)
        assert got.dtype == torch.float64 and ref32.dtype == torch.float32
        r = rel(got, ref32)
        print(f"[{name} mask={m is not None}] float64 path vs fp32 oracle rel-L2 {r:.2e}")
        assert r <= 2e-5


def test_emulation_error_order():
    """F5TTS_Base widths: the emulation's rel-L2 from float64 is that of fp16 storage through a few blocks (about
    3 * 2^-11 / sqrt(3) per stored operand, compounded over the blocks), far above fp32 rounding, and spread evenly over
    frames.  Rounding only the weights or only the activations gives a smaller but clearly nonzero error."""
    cfg = CONFIGS["f5base"]
    sd = EP.stress_state_dict(cfg)
    args = inputs(cfg, 2, 200, 80)
    ref = run(sd, cfg, args)
    emu = run(sd, cfg, args, rnd=EP.to_fp16)
    r = rel(emu, ref)
    sd64 = EP.engine_state_dict(sd, rnd=EP.to_fp16)
    with EP.fp16_storage(sd64, rnd=IDENT):
        r_w = rel(EP.forward(sd64, cfg, *args, None, True), ref)
    sd64 = EP.engine_state_dict(sd, rnd=IDENT)
    with EP.fp16_storage(sd64, rnd=EP.to_fp16):
        r_a = rel(EP.forward(sd64, cfg, *args, None, True), ref)
    frames = ((emu - ref).pow(2).mean(-1).sqrt() / ref.pow(2).mean((1, 2), keepdim=True).sqrt()[..., 0])
    spread = float((frames.amax(1) / frames.median(1).values).max())
    print(f"emulation rel-L2 {r:.2e} (weights only {r_w:.2e}, activations only {r_a:.2e}), worst frame / median "
          f"{spread:.2f}")
    assert 2e-4 <= r <= 2e-3
    assert 5e-5 <= r_w < r and 5e-5 <= r_a < r
    assert spread <= 3.0


def test_rounding_removed_on_exit():
    cfg = CONFIGS["e2_add"]
    sd = EP.engine_state_dict(EP.stress_state_dict(cfg), rnd=IDENT)
    args = inputs(cfg, 1, 40, 20)
    before = EP.forward(sd, cfg, *args, None, True)
    with EP.fp16_storage(sd) as ns:
        assert all(m.F is ns for m in EP.MODULES)
        inside = EP.forward(sd, cfg, *args, None, True)
    assert all(m.F is TF for m in EP.MODULES)
    with pytest.raises(RuntimeError, match="inside"):
        with EP.fp16_storage(sd):
            raise RuntimeError("inside")
    assert all(m.F is TF for m in EP.MODULES)
    after = EP.forward(sd, cfg, *args, None, True)
    assert torch.equal(before, after) and not torch.equal(before, inside)


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_stress_weights(name, monkeypatch):
    cfg = CONFIGS[name]
    sd = EP.stress_state_dict(cfg)
    N = 257
    args = inputs(cfg, 2, N, 120 if cfg.backbone == "MMDiT" else 150)
    ref = run(sd, cfg, args)
    peak = [0.0]

    def rnd_peak(v):
        peak[0] = max(peak[0], float(v.abs().max()))
        return EP.to_fp16(v)

    noise = rel(run(sd, cfg, args, rnd=rnd_peak), ref)

    def zero_attention(ns):
        ns.scaled_dot_product_attention = lambda q, k, v, *a, **kw: torch.zeros_like(q)

    no_attn = rel(run(sd, cfg, args, patch=zero_attention), ref)
    real = O.rope_angles

    def shifted(n, dim_head=64, base=10000.0, dtype=torch.float32):  # positions >= 128 one further on
        idx = torch.arange(n)
        idx[128:] += 1
        return real(n + 1, dim_head, base, dtype)[idx]

    monkeypatch.setattr(O, "rope_angles", shifted)
    shift = rel(run(sd, cfg, args), ref)
    monkeypatch.undo()
    print(f"[{name}] fp16 noise {noise:.2e}; zero attention {no_attn:.2e}; RoPE shift {shift:.2e} "
          f"({shift / noise:.1f}x the noise); largest fp16-stored |value| {peak[0]:.1f}")
    assert no_attn >= 0.3
    assert shift >= 10 * noise
    assert peak[0] <= 65504 / 64
