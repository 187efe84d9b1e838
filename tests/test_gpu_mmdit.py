"""GPU: MMDiT (backbones/mmdit.py) on the H100 path.

  * f5_attention_joint element by element against a float64 softmax over the concatenated keys [audio | text]
    (oracle/kernel_bounds.attention_ref), dim_head 64 and 128, with and without per-segment key lengths (c_len = 0
    included), and the last-block flag that leaves the text output unwritten;
  * end to end against the unmodified reference: the fixtures of oracle/make_golden_mmdit.py, rel-L2 <= 5e-3 after
    step 1 and at the end;
  * exact_varlen with ragged text equals a loop of B = 1 calls on the trimmed text; two calls are bit-identical and
    graph replay equals eager launches; two calls on one workspace that differ only in the text length are both right;
  * f5_sample_flops_nt counts the text stream and the joint attention;
  * infer.load_model(MMDiT, ...) on a checkpoint in the released layout, and the packed-weight cache round trip.
"""
import json
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import f5_tts_b200 as F5  # noqa: E402
import synthdata as SD  # noqa: E402
from f5_tts_b200 import _lib, infer, ops  # noqa: E402
from oracle import kernel_bounds as KB  # noqa: E402
from oracle import mmdit as OMM  # noqa: E402
from oracle import step_increment as SI  # noqa: E402

DEV = "cuda:0"
TOL = 5e-3
_models = {}


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ---------------------------------------------------------------------------------------------------------------------
# kernel
# ---------------------------------------------------------------------------------------------------------------------
def joint_ref(x, xc, kv, kc, b):
    """(o, bound) of sample b: float64 softmax over the valid keys of both segments, for the queries [audio | text].
    The valid keys are moved to the front (a softmax does not depend on the key order) so that attention_ref's
    prefix mask applies; block_kv is chosen so that its tile count is at least the kernel's, which tiles each segment
    separately."""
    q = torch.cat((x[b, :, 0], xc[b, :, 0]), dim=0)  # [N + nt, H, dh]
    n, m = x.shape[1], xc.shape[1]
    order = torch.cat((torch.arange(kv), n + torch.arange(kc), torch.arange(kv, n), n + torch.arange(kc, m)))
    k = torch.cat((x[b, :, 1], xc[b, :, 1]), dim=0)[order.to(DEV)]
    v = torch.cat((x[b, :, 2], xc[b, :, 2]), dim=0)[order.to(DEV)]
    tiles = -(-kv // 128) + -(-kc // 128)
    kv_len = torch.tensor([kv + kc], dtype=torch.int32, device=DEV)
    t = lambda a: a.permute(1, 0, 2)[None]  # noqa: E731  [1, H, seq, dh]
    return KB.attention_ref(t(q), t(k), t(v), kv_len, block_kv=max(1, (kv + kc) // tiles))


@pytest.mark.parametrize("lens", ["none", "lengths", "c_len0"])
@pytest.mark.parametrize("N,nt", [(90, 17), (469, 150), (938, 150), (1875, 300), (203, 130)])
@pytest.mark.parametrize("dh", [64, 128])
def test_attention_joint(dh, N, nt, lens):
    Be, H = 2, 4
    inner = H * dh
    g = torch.Generator().manual_seed(N + nt + dh)
    x = torch.randn(Be, N, 3, H, dh, generator=g).half().to(DEV)
    xc = torch.randn(Be, nt, 3, H, dh, generator=g).half().to(DEV)
    if lens == "none":
        kv, kc = [N] * Be, [nt] * Be
    else:
        kv, kc = [N, max(1, N - 77)], [nt - 5, 0] if lens == "c_len0" else [nt, max(1, nt - 13)]
    kv_t = None if lens == "none" else torch.tensor(kv, dtype=torch.int32, device=DEV)
    kc_t = None if lens == "none" else torch.tensor(kc, dtype=torch.int32, device=DEV)
    qkv, qkv_c = x.reshape(Be * N, 3 * inner).contiguous(), xc.reshape(Be * nt, 3 * inner).contiguous()
    out, out_c = ops.attention_joint(qkv, qkv_c, Be, N, nt, H, kv_len=kv_t, c_len=kc_t, dim_head=dh)
    torch.cuda.synchronize()
    got = torch.cat((out.view(Be, N, H, dh), out_c.view(Be, nt, H, dh)), dim=1).permute(0, 2, 1, 3)
    for b in range(Be):
        ref, bound = joint_ref(x, xc, kv[b], kc[b], b)
        KB.assert_within(got[b:b + 1], ref, bound, f"joint attention dh{dh} N{N} nt{nt} {lens} b{b}")
    # last block: only the audio queries; out_c stays as it was and out is the same
    fill = torch.full((Be * nt, inner), 7.0, dtype=torch.float16, device=DEV)
    out2 = torch.empty_like(out)
    _lib.check(_lib.lib().f5_attention_joint(qkv.data_ptr(), qkv_c.data_ptr(), out2.data_ptr(), fill.data_ptr(), Be,
                                             N, nt, H, dh, ops._ptr(kv_t), ops._ptr(kc_t), 0, dh ** -0.5,
                                             torch.cuda.current_stream().cuda_stream), "f5_attention_joint")
    torch.cuda.synchronize()
    assert torch.equal(out2, out) and bool((fill == 7.0).all())


def test_attention_joint_rejects_bad_arguments():
    qkv = torch.zeros(2 * 64, 3 * 128, dtype=torch.float16, device=DEV)
    with pytest.raises(_lib.F5LibraryError):
        ops.attention_joint(qkv, torch.zeros(0, 3 * 128, dtype=torch.float16, device=DEV), 2, 64, 0, 2)
    with pytest.raises(_lib.F5LibraryError):
        ops.attention_joint(torch.zeros(2 * 64, 3 * 96, dtype=torch.float16, device=DEV),
                            torch.zeros(2 * 8, 3 * 96, dtype=torch.float16, device=DEV), 2, 64, 8, 1, dim_head=96)


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
FIXTURES = sorted(n[:-4] for n in os.listdir(os.path.join(os.path.dirname(__file__), "golden"))
                  if n.startswith("mmdit_") and n.endswith(".npz"))


def tiny(**over):
    base = dict(backbone="MMDiT", dim=128, depth=3, heads=2, dim_head=64, ff_mult=2, mel_dim=100, text_num_embeds=50,
                text_dim=None, conv_layers=0, text_mask_padding=True, pe_attn_head=None, attn_mask_enabled=False)
    base.update(over)
    return SD.ArchConfig(**base)


def build(cfg: SD.ArchConfig, wseed: int = 1234):
    key = (repr(cfg), wseed)
    if key not in _models:
        _models.clear()
        model = F5.CFM(transformer=F5.MMDiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head,
                                            ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim,
                                            text_num_embeds=cfg.text_num_embeds,
                                            text_mask_padding=cfg.text_mask_padding, qk_norm=cfg.qk_norm,
                                            attn_mask_enabled=cfg.attn_mask_enabled))
        sd = SD.synthetic_state_dict(cfg, seed=wseed)
        model.load_state_dict(sd, strict=True)
        _models[key] = (model.to(DEV), sd)
    model, sd = _models[key]
    model.odeint_kwargs = dict(method="euler")
    model.use_cuda_graph = True
    return model, sd


@pytest.mark.parametrize("name", FIXTURES)
def test_sample_vs_reference_fixture(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg = SD.ArchConfig(**json.loads(str(z["cfg"])))
    model, _ = build(cfg, int(z["wseed"]))
    model.odeint_kwargs = dict(method=str(z["method"]))
    dur = z["duration"]
    duration = int(dur) if dur.ndim == 0 else torch.from_numpy(dur).long().to(DEV)
    lens = torch.from_numpy(z["lens"]).long().to(DEV) if z["lens"].size else None
    sway = float(z["sway"])
    try:
        out, traj = model.sample(cond=torch.from_numpy(z["cond"]).to(DEV), text=torch.from_numpy(z["text"]).to(DEV),
                                 duration=duration, lens=lens, steps=int(z["steps"]),
                                 cfg_strength=float(z["cfg_strength"]),
                                 sway_sampling_coef=None if math.isnan(sway) else sway, seed=int(z["seed"]),
                                 y0=torch.from_numpy(z["y0"]).to(DEV))
    finally:
        model.odeint_kwargs = dict(method="euler")
    assert traj.shape[0] == int(z["steps"]) + 1 and out.shape == z["out"].shape
    SI.check(traj[1], z["y0"], z["traj_1"], z["duration"] if cfg.attn_mask_enabled else None, name)
    r1, rn = rel(traj[1], z["traj_1"]), rel(out, z["out"])
    print(f"[{name}] step-1 rel-L2 {r1:.3e}  final rel-L2 {rn:.3e}")
    assert r1 <= TOL and rn <= TOL


@pytest.mark.parametrize("attn_mask", [False, True])
def test_exact_varlen_batch_equals_single_calls(attn_mask):
    model, _ = build(tiny(attn_mask_enabled=attn_mask))
    g = torch.Generator().manual_seed(95)
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
        print(f"[mmdit exact_varlen attn_mask={attn_mask}] sample {b} ({d} frames): batched vs single max|d| {md:.3e}")
        assert torch.equal(out[b, :d], singles[b][0])


def test_graph_equals_eager_and_deterministic():
    cfg = SD.mmdit_v1_base_widths()
    cfg.depth = 3
    model, _ = build(cfg)
    g = torch.Generator().manual_seed(96)
    cond = torch.randn(2, 50, 100, generator=g).to(DEV)
    text = torch.randint(0, 2545, (2, 40), generator=g)
    text[1, 27:] = -1
    dur = torch.tensor([200, 163]).to(DEV)
    kw = dict(steps=3, cfg_strength=2.0, sway_sampling_coef=-1.0, lens=torch.tensor([50, 41]).to(DEV),
              y0=torch.randn(2, 200, 100, generator=g).to(DEV))
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
    assert torch.equal(a, b) and torch.equal(ta, tb), "same inputs must be bit-identical run to run"
    assert torch.equal(a, c) and torch.equal(ta, tc), "graph replay and eager launches run the same kernels"


def test_text_length_is_part_of_the_graph_key():
    """Two calls on one workspace with the same N but different text lengths: the second must not replay the first's
    graph (its text-stream plans have the other nt)."""
    model, sd = build(tiny())
    cfg = tiny()
    g = torch.Generator().manual_seed(97)
    cond = torch.randn(1, 30, 100, generator=g)
    kw = dict(steps=3, cfg_strength=2.0, sway_sampling_coef=-1.0)
    ptrs = []
    for nt in (60, 23):  # the larger first: the pooled workspace also fits the second call
        text = torch.randint(0, 50, (1, nt), generator=g)
        ref = OMM.sample(sd, cfg, cond, text, 120, **kw, seed=3)
        out, _ = model.sample(cond.to(DEV), text.to(DEV), 120, **kw, y0=ref.y0.to(DEV))
        ptrs.append([w.data_ptr() for pool in model.transformer._ws_free.values() for w in pool])
        r = rel(out, ref.out)
        print(f"[graph key] nt {nt}: final rel-L2 {r:.3e}")
        assert r <= TOL
    assert ptrs[0] == ptrs[1] and len(ptrs[0]) == 1, "both calls ran on one workspace"


def test_sample_flops_count_text_stream_and_joint_attention():
    cfg = tiny(dim=256, heads=4, depth=3)
    model, _ = build(cfg)
    D, F, I, Ld, mel = 256, 512, 256, 3, 100
    for B, N, nt, steps, cfgs in ((1, 300, 40, 8, 2.0), (3, 128, 100, 5, 0.0)):
        n, m = float(N), float(nt)
        blocks = Ld * (6 * n * D * I + 2 * n * I * D + 4 * n * D * F + 6 * m * D * I + 4 * n * (n + m) * I) + \
            (Ld - 1) * (2 * m * I * D + 4 * m * D * F + 4 * m * (n + m) * I)
        embed = 2 * n * 2 * mel * D + 2 * (2 * n * D * (D // 16) * 31) + 2 * n * D * mel
        modw = (Ld - 1) * 12 * D + 8 * D + 2 * D
        Be = 2 * B if cfgs > 0 else B
        want = steps * Be * (blocks + embed) + steps * (2 * 256 * D + 2 * D * D + 2 * D * modw)
        got = model.transformer.sample_flops(B, N, steps, cfgs, nt=nt)
        print(f"[mmdit flops] B{B} N{N} nt{nt} steps{steps} cfg{cfgs}: {got:.6e} vs {want:.6e}")
        assert abs(got - want) <= 1e-9 * want
        assert model.transformer.sample_flops(B, N, steps, cfgs) == model.transformer.sample_flops(B, N, steps, cfgs,
                                                                                                   nt=N)


def test_workspace_bytes_nt():
    model, _ = build(tiny())
    L, h = _lib.lib(), model.transformer.engine()["handle"]
    assert L.f5_sample_workspace_bytes(h, 2, 200, 8, 2.0) == L.f5_sample_workspace_bytes_nt(h, 2, 200, 200, 8, 2.0)
    assert L.f5_sample_workspace_bytes_nt(h, 2, 200, 50, 8, 2.0) < L.f5_sample_workspace_bytes_nt(h, 2, 200, 150, 8, 2.0)


# ---------------------------------------------------------------------------------------------------------------------
# loading: released checkpoint layout, packed-weight cache
# ---------------------------------------------------------------------------------------------------------------------
ARCH = dict(dim=256, depth=3, heads=4, ff_mult=2, text_mask_padding=True, qk_norm="rms_norm",
            checkpoint_activations=False)


@pytest.fixture(scope="module")
def mmdit_ckpt(tmp_path_factory):
    from safetensors.torch import save_file

    cfg = SD.ArchConfig(backbone="MMDiT", dim=256, depth=3, heads=4, ff_mult=2, text_dim=None, conv_layers=0,
                        text_mask_padding=True, pe_attn_head=None, qk_norm="rms_norm")
    sd = SD.synthetic_state_dict(cfg, seed=1234)
    ema = {"ema_model." + k: v for k, v in sd.items()}
    ema["initted"], ema["step"] = torch.tensor(True), torch.tensor(1)
    ckpt = str(tmp_path_factory.mktemp("f5mmdit") / "model_1.safetensors")
    save_file(ema, ckpt)
    return dict(cfg=cfg, sd=sd, ckpt=ckpt)


def test_load_model_vs_oracle(mmdit_ckpt, golden_dir):
    _models.clear()
    a = mmdit_ckpt
    m = infer.load_model(F5.MMDiT, ARCH, a["ckpt"], vocab_file=os.path.join(golden_dir, "vocab.txt"), device=DEV)
    assert isinstance(m.transformer, F5.MMDiT) and m.transformer.qk_norm == "rms_norm"
    g = torch.Generator().manual_seed(98)
    cond = torch.randn(2, 40, 100, generator=g)
    text = torch.randint(0, 2545, (2, 30), generator=g)
    text[0, 21:] = -1
    dur, lens = torch.tensor([170, 139]), torch.tensor([40, 35])
    kw = dict(steps=3, cfg_strength=2.0, sway_sampling_coef=-1.0)
    ref = OMM.sample(a["sd"], a["cfg"], cond, text, dur, lens=lens, **kw, seed=5)
    out, _ = m.sample(cond.to(DEV), text.to(DEV), dur.to(DEV), lens=lens.to(DEV), **kw, y0=ref.y0.to(DEV))
    r = rel(out, ref.out)
    print(f"[load_model mmdit] final rel-L2 {r:.3e}")
    assert r <= TOL


def test_packed_cache_roundtrip(mmdit_ckpt, golden_dir, tmp_path):
    import glob

    from safetensors import safe_open

    from f5_tts_b200 import weights as Wt

    _models.clear()
    a = mmdit_ckpt
    vocab = os.path.join(golden_dir, "vocab.txt")
    cache = str(tmp_path / "pack")
    m1 = infer.load_model(F5.MMDiT, ARCH, a["ckpt"], vocab_file=vocab, device=DEV, packed_cache_dir=cache)
    files = glob.glob(os.path.join(cache, "f5pack_*.safetensors"))
    assert len(files) == 1
    with safe_open(files[0], framework="pt") as f:
        names = set(f.keys())
    assert {"C0.w_qkv_c", "C0.w_out_c", "C1.w_ff2_c", "C2.w_qkv_c", "C2.q_norm_c", "mod_w"} <= names
    assert "C2.w_out_c" not in names, "the last block has no text out-projection"
    calls = {"n": 0}
    orig = Wt.packed_tensors

    def counting(m):
        calls["n"] += 1
        return orig(m)

    Wt.packed_tensors = counting
    try:
        m2 = infer.load_model(F5.MMDiT, ARCH, a["ckpt"], vocab_file=vocab, device=DEV, packed_cache_dir=cache)
        g = torch.Generator().manual_seed(99)
        cond = torch.randn(1, 40, 100, generator=g).to(DEV)
        text = torch.randint(0, 2545, (1, 30), generator=g).to(DEV)
        y0 = torch.randn(1, 150, 100, generator=g).to(DEV)
        kw = dict(steps=2, cfg_strength=2.0, sway_sampling_coef=-1.0)
        o2, _ = m2.sample(cond, text, 150, **kw, y0=y0)
        assert calls["n"] == 0, "the second load must not re-pack"
    finally:
        Wt.packed_tensors = orig
    o1, _ = m1.sample(cond, text, 150, **kw, y0=y0)
    assert torch.equal(o1, o2)
