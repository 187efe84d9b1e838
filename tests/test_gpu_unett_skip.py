"""GPU: UNetT checkpoints built with skip_connect_type="add" or "none" (backbones/unett.py:127, 286-297).

  * row_norm_kernel<3> (x += skip, written back, then RMSNorm of the sum) element by element: the written x equals
    x + skip bit for bit, the fp16 output is within the fp16-rounding bound of a float64 reference;
  * end to end against the unmodified reference: the fixtures of oracle/make_golden_unett_skip.py, rel-L2 <= 5e-3
    after step 1 and at the end;
  * exact_varlen equals a loop of B = 1 calls; two calls are bit-identical and graph replay equals eager launches;
  * f5_sample_flops drops the combiner GEMM, the "none" workspace drops the saved rows, an odd depth is refused;
  * infer.load_model on a checkpoint in the released layout with skip_connect_type in the arch dict, and the
    packed-weight cache round trip of such a model.
"""
import ctypes as C
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
from f5_tts_b200 import _lib, infer  # noqa: E402
from oracle import f5_oracle as O  # noqa: E402
from oracle import make_golden as MG  # noqa: E402
from oracle import make_golden_unett_skip as MU  # noqa: E402
from oracle import unett_skip as OU  # noqa: E402
from oracle.kernel_bounds import assert_half  # noqa: E402
from oracle import step_increment as SI  # noqa: E402

DEV = "cuda:0"
TOL = 5e-3
U = 2.0 ** -24
_models = {}


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ---------------------------------------------------------------------------------------------------------------------
# kernel: row norm mode 3
# ---------------------------------------------------------------------------------------------------------------------
_hooks = None


def hooks():
    global _hooks
    if _hooks is None:
        L = C.CDLL(_lib.KERNELS_LIB_PATH)
        L.f5k_last_error.restype = C.c_char_p
        L.f5k_row_norm_add_skip.argtypes = [C.c_void_p] * 3 + [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.f5k_row_norm_add_skip.restype = C.c_int
        L.f5k_row_norm.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_void_p]
        L.f5k_row_norm.restype = C.c_int
        _hooks = L
    return _hooks


def row_norm_add_skip(x, skip, out, g):
    rows, D = x.shape
    rc = hooks().f5k_row_norm_add_skip(x.data_ptr(), skip.data_ptr(), out.data_ptr(), rows, D, g.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream)
    assert rc == 0, hooks().f5k_last_error().decode()


def unett_rows(B, N, D, seed):
    """[B * (N + 1), D] fp32 in the UNetT residual layout: row 0 of every sample is the time token (here ~10x the scale
    of the frame rows), rows 1..N the frames."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N + 1, D, generator=g, dtype=torch.float64) * 2.0
    x[:, 0] *= 10.0
    return x.reshape(B * (N + 1), D).float().to(DEV)


@pytest.mark.parametrize("D", [128, 768, 1024])
@pytest.mark.parametrize("shape", [(1, 0), (2, 300), (3, 625)])
def test_row_norm_add_skip(D, shape):
    """x <- x + skip (fp32, one IEEE addition: equal to torch's bit for bit); out = RMSNorm(x + skip) * g in fp16.
    Bound of out as row_norm mode 2 (tests/test_gpu_small_kernels.py): the sum of squares within g(D / 32 + 6), sqrtf
    twice and the quotient, |d| <= |out| (g(D / 32 + 6) / 2 + 5 u), plus one fp16 rounding."""
    B, N = shape
    x, skip = unett_rows(B, N, D, 60 + D + N), unett_rows(B, N, D, 61 + D + N)
    gen = torch.Generator().manual_seed(62)
    gain = (1.0 + 0.1 * torch.randn(D, generator=gen)).to(DEV)
    want_x = x + skip
    out = torch.full(x.shape, float("nan"), dtype=torch.float16, device=DEV)
    row_norm_add_skip(x, skip, out, gain)
    torch.cuda.synchronize()
    assert torch.equal(x, want_x), "the written x is x + skip bit for bit"
    sd = want_x.double()
    ref = sd / sd.norm(dim=-1, keepdim=True) * math.sqrt(D) * gain.double()
    n = (D // 32 + 6) * U / (1 - (D // 32 + 6) * U)
    worst = assert_half(out, ref, ref.abs() * (0.5 * n + 5 * U), f"row_norm_add_skip D{D} B{B} N{N}")
    # the same fp16 output as mode 2 over the materialised sum: the fusion changes nothing downstream
    out2 = torch.full_like(out, float("nan"))
    rc = hooks().f5k_row_norm(2, want_x.data_ptr(), out2.data_ptr(), x.shape[0], D, 1e-6, gain.data_ptr(), None, None,
                              0, 1, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    print(f"[row_norm_add_skip D{D} B{B} N{N}] worst err/bound {worst:.3f}")
    assert torch.equal(out, out2)


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
def arch_kwargs(cfg):
    return dict(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
                mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim,
                text_mask_padding=cfg.text_mask_padding, conv_layers=cfg.conv_layers, pe_attn_head=cfg.pe_attn_head,
                attn_mask_enabled=cfg.attn_mask_enabled, qk_norm=cfg.qk_norm, skip_connect_type=cfg.skip_connect_type)


def build(cfg: O.ArchConfig, wseed: int = 1234):
    key = (repr(cfg), wseed)
    if key not in _models:
        _models.clear()
        model = F5.CFM(transformer=F5.UNetT(**arch_kwargs(cfg)))
        sd = O.synthetic_state_dict(cfg, seed=wseed)
        model.load_state_dict(sd, strict=True)
        _models[key] = (model.to(DEV), sd)
    model, sd = _models[key]
    model.odeint_kwargs = dict(method="euler")
    model.use_cuda_graph = True
    return model, sd


@pytest.mark.parametrize("name", sorted(MU.CASES))
def test_sample_vs_reference_fixture(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg, kw = MU.CASES[name]
    model, _ = build(cfg, int(z["wseed"]))
    model.odeint_kwargs = dict(method=str(z["method"]))
    duration = torch.from_numpy(z["duration"]).long().to(DEV)
    lens = torch.from_numpy(z["lens"]).long().to(DEV)
    try:
        out, traj = model.sample(cond=torch.from_numpy(z["cond"]).to(DEV), text=torch.from_numpy(z["text"]).to(DEV),
                                 duration=duration, lens=lens, steps=int(z["steps"]),
                                 cfg_strength=float(z["cfg_strength"]), sway_sampling_coef=float(z["sway"]),
                                 seed=int(z["seed"]), y0=torch.from_numpy(z["y0"]).to(DEV))
    finally:
        model.odeint_kwargs = dict(method="euler")
    assert traj.shape[0] == int(z["steps"]) + 1 and out.shape == z["out"].shape
    SI.check(traj[1], z["y0"], z["traj_1"], z["duration"] if cfg.attn_mask_enabled else None, name)
    r1, rn = rel(traj[1], z["traj_1"]), rel(out, z["out"])
    print(f"[{name}] step-1 rel-L2 {r1:.3e}  final rel-L2 {rn:.3e}")
    assert r1 <= TOL and rn <= TOL


@pytest.mark.parametrize("over", [dict(skip_connect_type="add"), dict(skip_connect_type="none"),
                                  dict(skip_connect_type="add", attn_mask_enabled=True, dim_head=128)],
                         ids=["add", "none", "add-attnmask-dh128"])
def test_exact_varlen_batch_equals_single_calls(over):
    model, _ = build(MG.tiny_unett(**over))
    g = torch.Generator().manual_seed(94)
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
        print(f"[{over} exact_varlen] sample {b} ({d} frames): batched vs single max|d| {md:.3e}")
        assert torch.equal(out[b, :d], singles[b][0])


@pytest.mark.parametrize("skip", ["add", "none"])
def test_graph_equals_eager_and_deterministic(skip):
    """E2TTS_Small widths at depth 4 with qk_norm, midpoint, ragged batch."""
    cfg = SD.e2tts_small()
    cfg.depth, cfg.skip_connect_type, cfg.qk_norm = 4, skip, "rms_norm"
    model, _ = build(cfg)
    g = torch.Generator().manual_seed(95)
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


def test_sample_flops_drop_the_combiner_gemm():
    """concat runs Linear(2D -> D) on the n + 1 rows of every later-half layer: 2 (n + 1) D (2 D) FLOPs each, times NFE
    and the CFG batch.  add and none count the same."""
    depth, D = 4, 128
    flops = {}
    for t in ("concat", "add", "none"):
        m, _ = build(MG.tiny_unett(skip_connect_type=t))
        flops[t] = {c: m.transformer.sample_flops(*c) for c in ((1, 300, 8, 2.0), (3, 128, 5, 0.0))}
    for (B, N, nfe, cfg), f_concat in flops["concat"].items():
        Be = 2 * B if cfg > 0 else B
        want = nfe * Be * (depth // 2) * 2.0 * (N + 1) * D * 2 * D
        got = f_concat - flops["add"][(B, N, nfe, cfg)]
        print(f"[skip flops] B{B} N{N} nfe{nfe} cfg{cfg}: concat - add {got:.6e} vs {want:.6e}")
        assert abs(got - want) <= 1e-9 * f_concat
        assert flops["add"][(B, N, nfe, cfg)] == flops["none"][(B, N, nfe, cfg)]


def test_workspace_sizes():
    """none keeps no saved rows: depth/2 * M1 * D * 4 bytes less than add; add has no [x | skip] fp16 operand: M1 * 2D * 2
    bytes less than concat (M1 = Be * (N + 1); every buffer is a multiple of 256 bytes at D % 128 == 0)."""
    depth, D = 4, 128
    ws = {}
    for t in ("concat", "add", "none"):
        m, _ = build(MG.tiny_unett(skip_connect_type=t))
        h = m.transformer.engine()["handle"]
        ws[t] = {c: _lib.lib().f5_sample_workspace_bytes(h, *c) for c in ((1, 300, 8, 2.0), (3, 127, 5, 0.0))}
    for (B, N, nfe, cfg) in ws["concat"]:
        M1 = (2 * B if cfg > 0 else B) * (N + 1)
        c, a, n = (ws[t][(B, N, nfe, cfg)] for t in ("concat", "add", "none"))
        print(f"[workspace] B{B} N{N} cfg{cfg}: concat {c} add {a} none {n}")
        assert a - n == depth // 2 * M1 * D * 4
        assert c - a == M1 * 2 * D * 2


@pytest.mark.parametrize("skip", ["add", "none"])
def test_odd_depth_raises(skip):
    """Every first-half layer pushes x and every later-half layer pops one: an odd depth would pop more than it pushed
    (the reference's constructor asserts an even depth).  The engine refuses it before anything is launched."""
    cfg = MG.tiny_unett(depth=3, skip_connect_type=skip)
    model, _ = build(cfg)
    y0 = torch.randn(1, 80, 100).to(DEV)
    with pytest.raises(_lib.F5LibraryError, match="even depth"):
        model.sample(torch.randn(1, 20, 100).to(DEV), torch.randint(0, 50, (1, 12)).to(DEV), 80, steps=2,
                     cfg_strength=2.0, y0=y0)


def test_engine_create_checks_skip_type():
    """skip_type only on UNetT, w_skip only with concat (checked by the C ABI itself)."""
    model, _ = build(MG.tiny_unett(skip_connect_type="add"))
    st = model.transformer.engine()
    A, W = st["arch"], st["weights"]
    L = _lib.lib()

    def create():
        h = C.c_void_p()
        rc = L.f5_engine_create(C.byref(A), C.byref(W), C.byref(h))
        if rc == 0:
            L.f5_engine_destroy(h)
        return rc

    assert create() == 0
    saved = (A.backbone, A.skip_type, st["layers"][3].w_skip)
    try:
        A.skip_type = 3
        assert create() != 0
        A.skip_type, A.backbone = 1, 0
        assert create() != 0 and b"UNetT" in L.f5_last_error()
        A.backbone = 1
        st["layers"][3].w_skip = st["layers"][3].w_qkv  # any pointer: add takes no skip projection
        assert create() != 0 and b"w_skip" in L.f5_last_error()
        A.skip_type = 0  # concat needs it in every later-half layer: layer 2 has none
        assert create() != 0 and b"w_skip" in L.f5_last_error()
    finally:
        A.backbone, A.skip_type, st["layers"][3].w_skip = saved
    assert create() == 0


# ---------------------------------------------------------------------------------------------------------------------
# loading: released checkpoint layout with skip_connect_type in the arch dict, packed-weight cache
# ---------------------------------------------------------------------------------------------------------------------
ARCH = dict(dim=768, depth=4, heads=12, ff_mult=4, text_dim=None, text_mask_padding=False, conv_layers=0,
            pe_attn_head=1, skip_connect_type="add")


@pytest.fixture(scope="module")
def add_ckpt(tmp_path_factory):
    from safetensors.torch import save_file

    cfg = SD.ArchConfig(backbone="UNetT", dim=768, depth=4, heads=12, ff_mult=4, text_dim=None, conv_layers=0,
                        text_mask_padding=False, pe_attn_head=1, skip_connect_type="add")
    sd = SD.synthetic_state_dict(cfg, seed=1234)
    ema = {"ema_model." + k: v for k, v in sd.items()}
    ema["initted"], ema["step"] = torch.tensor(True), torch.tensor(1)
    ckpt = str(tmp_path_factory.mktemp("f5skip") / "model_1.safetensors")
    save_file(ema, ckpt)
    return dict(cfg=cfg, sd=sd, ckpt=ckpt)


def test_load_model_add_vs_oracle(add_ckpt, golden_dir):
    _models.clear()
    a = add_ckpt
    m = infer.load_model(F5.UNetT, ARCH, a["ckpt"], vocab_file=os.path.join(golden_dir, "vocab.txt"), device=DEV)
    assert m.transformer.skip_connect_type == "add"
    g = torch.Generator().manual_seed(96)
    cond = torch.randn(2, 40, 100, generator=g)
    text = torch.randint(0, 2545, (2, 30), generator=g)
    text[0, 21:] = -1
    dur, lens = torch.tensor([170, 139]), torch.tensor([40, 35])
    kw = dict(steps=3, cfg_strength=2.0, sway_sampling_coef=-1.0)
    ref = OU.sample(a["sd"], a["cfg"], cond, text, dur, lens=lens, **kw, seed=5)
    out, _ = m.sample(cond.to(DEV), text.to(DEV), dur.to(DEV), lens=lens.to(DEV), **kw, y0=ref.y0.to(DEV))
    r = rel(out, ref.out)
    print(f"[load_model add] final rel-L2 {r:.3e}")
    assert r <= TOL


def test_packed_cache_roundtrip_add(add_ckpt, golden_dir, tmp_path):
    import glob

    from safetensors import safe_open

    from f5_tts_b200 import weights as Wt

    _models.clear()
    a = add_ckpt
    vocab = os.path.join(golden_dir, "vocab.txt")
    cache = str(tmp_path / "pack")
    m1 = infer.load_model(F5.UNetT, ARCH, a["ckpt"], vocab_file=vocab, device=DEV, packed_cache_dir=cache)
    files = glob.glob(os.path.join(cache, "f5pack_*.safetensors"))
    assert len(files) == 1
    with safe_open(files[0], framework="pt") as f:
        assert not any(k.endswith("w_skip") for k in f.keys())
    calls = {"n": 0}
    orig = Wt.packed_tensors

    def counting(m):
        calls["n"] += 1
        return orig(m)

    Wt.packed_tensors = counting
    try:
        m2 = infer.load_model(F5.UNetT, ARCH, a["ckpt"], vocab_file=vocab, device=DEV, packed_cache_dir=cache)
        g = torch.Generator().manual_seed(97)
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
    # a concat model of the same widths and checkpoint path never reads the add model's file
    concat = dict(ARCH, skip_connect_type="concat")
    mc = F5.CFM(transformer=F5.UNetT(**concat, text_num_embeds=m1.transformer.text_num_embeds, mel_dim=100))
    assert Wt.cache_key(a["ckpt"], mc.transformer) != Wt.cache_key(a["ckpt"], m1.transformer)
