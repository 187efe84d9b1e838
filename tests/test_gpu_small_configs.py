"""GPU: the dim-768 Small configs (F5TTS_v1_Small, F5TTS_Small, E2TTS_Small) and the grouped conv position embedding
with G = dim / 16 channels per group.

  * conv kernel, G in {8, 16, 32, 48, 64}: both epilogues element by element against a float64 grouped conv1d of the
    same fp16 operands; channels of the other groups filled with NaN leave a group's outputs unchanged; bad G rejected;
  * end to end against the unmodified reference: the three Small fixtures (oracle/make_golden_small.py) and the six
    tiny fixtures (dim 128, G = 8) of oracle/make_golden.py — rel-L2 <= 5e-3 after step 1 and at the end;
  * against the CPU oracle on fresh inputs (var-len, attn-mask, no-CFG, raw wave + EPSS, midpoint, E2TTS_Small);
  * exact_varlen, graph replay, determinism, FLOP accounting;
  * F5TTS(model="F5TTS_v1_Small").infer, the packed-weight cache and the serving processor.
"""
import ast
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F
import yaml

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import f5_tts_b200 as F5  # noqa: E402
import synthdata as SD  # noqa: E402
from f5_tts_b200 import _lib, api, infer, ops  # noqa: E402
from f5_tts_b200.model import list_str_to_idx  # noqa: E402
from oracle import f5_oracle as O  # noqa: E402
from oracle import ode_midpoint as OM  # noqa: E402
from oracle import step_increment as SI  # noqa: E402

DEV = "cuda:0"
TOL = 5e-3
_models = {}


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def gen(shape, seed, scale=1.0, dtype=torch.float16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).to(DEV)


# ---------------------------------------------------------------------------------------------------------------------
# conv kernel
# ---------------------------------------------------------------------------------------------------------------------
def conv_ref64(x, w, bias, lens):
    """float64 Mish(mask(Conv1d(k=31, groups=16, padding=15)(x) + bias)) on the same fp16 operands, [B, N, D]."""
    y = F.conv1d(x.double().cpu().transpose(1, 2), w.double().cpu(), bias.double().cpu(), padding=15,
                 groups=16).transpose(1, 2)
    if lens is not None:
        m = (torch.arange(x.shape[1])[None, :] < lens.cpu()[:, None])[..., None]
        y = torch.where(m, y, torch.zeros_like(y))
    return F.mish(y)


def conv_case(G, B, N, masked, seed=0):
    D = 16 * G
    x = gen((B, N, D), 50 + seed)
    w = gen((D, G, 31), 51 + seed, 1 / math.sqrt(G * 31))
    bias = gen((D,), 52 + seed, 0.1, torch.float32)
    lens = None
    if masked:
        lens = torch.tensor([N, max(1, N // 2), 5][:B], dtype=torch.int32, device=DEV)
        m = (torch.arange(N, device=DEV)[None, :] < lens[:, None])[..., None]
        x = torch.where(m, x, torch.zeros_like(x))
    return x.contiguous(), w, w.permute(2, 0, 1).contiguous(), bias, lens


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("N", [77, 300])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("G", [8, 16, 32, 48, 64])
def test_grouped_conv_any_group_width(G, B, N, masked):
    """Bounds: the fp16 output is one fp16 rounding of an fp32-accumulated sum of 31 G fp16 products (relative error
    <= 2^-11 of the output plus the accumulation's ~31 G 2^-24 sum |terms|), hence rel-L2 <= 1.5e-3 and max|d| <=
    4e-3 max|ref| as in test_grouped_conv31; the fp32 residual has no output rounding: rel-L2 <= 2e-4."""
    x, w, wp, bias, lens = conv_case(G, B, N, masked)
    ref = conv_ref64(x, w, bias, lens)
    out = ops.grouped_conv31(x, wp, bias, row_len=lens)
    r = rel(out, ref)
    md = float((out.double().cpu() - ref).abs().max())
    print(f"[conv G{G} B{B} N{N} masked{masked}] fp16 rel-L2 {r:.3e} max|d| {md:.3e} max|ref| {float(ref.abs().max()):.3e}")
    assert torch.isfinite(out).all()
    assert r <= 1.5e-3 and md <= 4e-3 * float(ref.abs().max())
    r0 = gen((B, N, 16 * G), 53, 1.0, torch.float32)
    res = r0.clone()
    ops.grouped_conv31(x, wp, bias, resid=res, row_len=lens)
    want = r0.double().cpu() + ref
    rr = rel(res, want)
    print(f"[conv G{G} B{B} N{N} masked{masked}] resid rel-L2 {rr:.3e}")
    assert rr <= 2e-4


@pytest.mark.parametrize("G", [8, 16, 32, 48, 64])
def test_grouped_conv_groups_are_isolated(G):
    """Every channel outside group gi (activations, weights' output rows, bias) is NaN: the TMA box of a group reaches
    64 columns into its neighbours' channels, which must arrive as zeros or only feed columns that are never stored.
    The group's outputs stay finite and bit-identical to the clean run."""
    B, N = 2, 300
    D = 16 * G
    x, w, wp, bias, _ = conv_case(G, B, N, False, seed=7)
    clean = ops.grouped_conv31(x, wp, bias)
    r0 = gen((B, N, D), 54, 1.0, torch.float32)
    clean_r = r0.clone()
    ops.grouped_conv31(x, wp, bias, resid=clean_r)
    for gi in sorted({0, 7, 15}):
        sl = slice(gi * G, (gi + 1) * G)
        xn = torch.full_like(x, float("nan"))
        xn[..., sl] = x[..., sl]
        wn = torch.full_like(wp, float("nan"))
        wn[:, sl, :] = wp[:, sl, :]
        bn = torch.full_like(bias, float("nan"))
        bn[sl] = bias[sl]
        out = ops.grouped_conv31(xn.contiguous(), wn.contiguous(), bn)
        assert torch.isfinite(out[..., sl]).all(), f"group {gi}: NaN leaked in"
        assert torch.equal(out[..., sl], clean[..., sl])
        rr = r0.clone()
        ops.grouped_conv31(xn.contiguous(), wn.contiguous(), bn, resid=rr)
        assert torch.isfinite(rr[..., sl]).all() and torch.equal(rr[..., sl], clean_r[..., sl])


@pytest.mark.parametrize("G,D", [(12, 192), (72, 1152), (16, 200), (24, 392)])
def test_grouped_conv_rejects_bad_group_width(G, D):
    """G must be a multiple of 8, at most 64, and divide the channel count."""
    x = gen((1, 64, D), 55)
    wp = gen((31, D, G), 56)
    bias = gen((D,), 57, 0.1, torch.float32)
    with pytest.raises(_lib.F5LibraryError):
        ops.grouped_conv31(x, wp, bias)


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
def cfg_from_repr(s: str) -> O.ArchConfig:
    body = s[s.index("(") + 1: s.rindex(")")]
    return O.ArchConfig(**{k: ast.literal_eval(v) for k, v in (p.split("=") for p in body.split(", "))})


def build(cfg: O.ArchConfig, wseed: int = 1234):
    key = (repr(cfg), wseed)
    if key not in _models:
        _models.clear()
        cls = F5.DiT if cfg.backbone == "DiT" else F5.UNetT
        kw = dict(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
                  mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim,
                  text_mask_padding=cfg.text_mask_padding, conv_layers=cfg.conv_layers, pe_attn_head=cfg.pe_attn_head,
                  attn_mask_enabled=cfg.attn_mask_enabled)
        model = F5.CFM(transformer=cls(**kw))
        sd = O.synthetic_state_dict(cfg, seed=wseed)
        model.load_state_dict(sd, strict=True)
        _models[key] = (model.to(DEV), sd)
    model, sd = _models[key]
    model.odeint_kwargs = dict(method="euler")
    return model, sd


SMALL_FIXTURES = ["f5v1small_b2_varlen", "f5small_b1_n192", "e2small_b2_varlen"]
TINY_FIXTURES = ["dit_tiny_b1_wave", "dit_tiny_b3_varlen", "dit_tiny_b3_attnmask", "dit_tiny_v1style_b2",
                 "dit_tiny_nocfg_nosway", "unett_tiny_b2"]


@pytest.mark.parametrize("name", SMALL_FIXTURES + TINY_FIXTURES)
def test_sample_vs_reference_fixture(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg = cfg_from_repr(str(z["cfg"]))
    assert cfg.dim in (128, 768)
    model, _ = build(cfg, int(z["wseed"]))
    dur = z["duration"]
    duration = int(dur) if dur.ndim == 0 else torch.from_numpy(dur).long().to(DEV)
    lens = torch.from_numpy(z["lens"]).long().to(DEV) if z["lens"].size else None
    sway = None if np.isnan(z["sway"]) else float(z["sway"])
    out, traj = model.sample(cond=torch.from_numpy(z["cond"]).to(DEV), text=torch.from_numpy(z["text"]).to(DEV),
                             duration=duration, lens=lens, steps=int(z["steps"]), cfg_strength=float(z["cfg_strength"]),
                             sway_sampling_coef=sway, seed=int(z["seed"]), y0=torch.from_numpy(z["y0"]).to(DEV))
    assert traj.shape[0] == int(z["steps"]) + 1 and out.shape == z["out"].shape
    SI.check(traj[1], z["y0"], z["traj_1"], z["duration"] if cfg.attn_mask_enabled else None, name)
    want, want1, t1 = torch.from_numpy(z["out"]), torch.from_numpy(z["traj_1"]), traj[1]
    if cfg.attn_mask_enabled:  # key-masked mode: padded rows are not computed, compare every sample's valid rows
        durs = z["duration"].tolist()
        out = torch.cat([out[b, :d].cpu() for b, d in enumerate(durs)])
        want = torch.cat([want[b, :d] for b, d in enumerate(durs)])
        t1 = torch.cat([t1[b, :d].cpu() for b, d in enumerate(durs)])
        want1 = torch.cat([want1[b, :d] for b, d in enumerate(durs)])
    r1, rn = rel(t1, want1), rel(out, want)
    print(f"[{name}] step-1 rel-L2 {r1:.3e}  final rel-L2 {rn:.3e}")
    assert r1 <= TOL and rn <= TOL


@pytest.mark.parametrize("variant", ["mask_faithful", "attn_mask", "no_cfg", "wave_epss", "midpoint", "e2_varlen"])
def test_small_sample_vs_oracle(variant):
    cfg = SD.e2tts_small() if variant == "e2_varlen" else SD.f5tts_v1_small()
    if variant == "attn_mask":
        cfg.attn_mask_enabled = True
    model, sd = build(cfg)
    g = torch.Generator().manual_seed(61)
    kw = dict(steps=3, cfg_strength=2.0, sway_sampling_coef=-1.0, seed=7)
    if variant in ("mask_faithful", "attn_mask", "midpoint"):
        cond = torch.randn(3, 40, 100, generator=g)
        text = torch.randint(0, 2545, (3, 30), generator=g)
        text[1, 20:] = -1
        args = (cond, text, torch.tensor([150, 97, 131]))
        kw["lens"] = torch.tensor([40, 25, 33])
        if variant == "midpoint":
            kw["steps"] = 2
    elif variant == "e2_varlen":
        cond = torch.randn(2, 36, 100, generator=g)
        text = torch.randint(0, 2545, (2, 28), generator=g)
        text[1, 18:] = -1
        args = (cond, text, torch.tensor([140, 104]))
        kw["lens"] = torch.tensor([36, 30])
    elif variant == "no_cfg":
        args = (torch.randn(1, 30, 100, generator=g), torch.randint(0, 2545, (1, 25), generator=g), 130)
        kw.update(cfg_strength=0.0, sway_sampling_coef=None)
    else:  # raw wave in (mel kernel) + the EPSS grid of 5 steps
        args = (0.1 * torch.randn(1, 30 * 256, generator=g), torch.randint(0, 2545, (1, 25), generator=g), 140)
        kw["steps"] = 5
    if variant == "midpoint":
        ref = OM.sample(sd, cfg, *args, method="midpoint", **kw)
        model.odeint_kwargs = dict(method="midpoint")
    else:
        ref = O.sample(sd, cfg, *args, **kw)
    dargs = tuple(a.to(DEV) if torch.is_tensor(a) else a for a in args)
    dkw = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in kw.items()}
    try:
        out, traj = model.sample(*dargs, **dkw, y0=ref.y0.to(DEV))
    finally:
        model.odeint_kwargs = dict(method="euler")
    assert traj.shape[0] == kw["steps"] + 1
    if variant == "attn_mask":
        durs = args[2].tolist()
        r = rel(torch.cat([out[b, :d].cpu() for b, d in enumerate(durs)]),
                torch.cat([ref.out[b, :d] for b, d in enumerate(durs)]))
    else:
        r = rel(out, ref.out)
    print(f"[small oracle:{variant}] final rel-L2 {r:.3e}")
    assert r <= TOL


def test_small_exact_varlen_batch_equals_single_calls():
    model, _ = build(SD.f5tts_v1_small())
    g = torch.Generator().manual_seed(62)
    n_ref, durs = 60, [420, 150, 297]
    cond = torch.randn(1, n_ref, 100, generator=g)
    text = torch.randint(0, 2545, (3, 50), generator=g)
    text[1, 30:] = -1
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
        print(f"[small exact_varlen] sample {b} ({d} frames): batched vs single max|d| {md:.3e}")
        assert torch.equal(out[b, :d], singles[b][0])


def test_small_graph_equals_eager_and_deterministic():
    model, _ = build(SD.f5tts_v1_small())
    g = torch.Generator().manual_seed(63)
    cond = torch.randn(1, 50, 100, generator=g).to(DEV)
    text = torch.randint(0, 2545, (1, 40), generator=g).to(DEV)
    kw = dict(steps=4, cfg_strength=2.0, sway_sampling_coef=-1.0, y0=torch.randn(1, 200, 100, generator=g).to(DEV))
    try:
        model.use_cuda_graph = True
        a, ta = model.sample(cond, text, 200, **kw)
        b, tb = model.sample(cond, text, 200, **kw)
        model.use_cuda_graph = False
        c, tc = model.sample(cond, text, 200, **kw)
    finally:
        model.use_cuda_graph = True
    assert torch.equal(a, b) and torch.equal(ta, tb), "same inputs must be bit-identical run to run"
    assert torch.equal(a, c) and torch.equal(ta, tc), "graph replay and eager launches run the same kernels"


def test_small_sample_flops_formula():
    """SURVEY.md §8d: per DiT sample-forward L (8 n D^2 + 4 n D F + 4 n^2 D) + input projection 2 n (2 mel + Td) D + two
    grouped convs 2 * 2 n D (D / 16) 31 + output projection 2 n D mel; times NFE and the CFG batch; plus the text
    embedding once per sample and CFG branch and the per-evaluation conditioning (time MLP, AdaLN table)."""
    model, _ = build(SD.f5tts_v1_small())
    L, D, Fi, mel, Td, V = 18, 768, 1536, 100, 512, 4
    for B, N, nfe, cfg in ((1, 938, 32, 2.0), (3, 300, 7, 0.0)):
        Be = 2 * B if cfg > 0 else B
        fwd = L * (8 * N * D * D + 4 * N * D * Fi + 4 * N * N * D) + 2 * N * (2 * mel + Td) * D \
            + 2 * (2 * N * D * (D // 16) * 31) + 2 * N * D * mel
        text = 2 * B * V * (2 * 2 * N * Td * 2 * Td)
        modw = L * 6 * D + 2 * D
        cond = nfe * (2 * 256 * D + 2 * D * D + 2 * D * modw)
        want = nfe * Be * fwd + text + cond
        got = model.transformer.sample_flops(B, N, nfe, cfg)
        print(f"[small flops] B{B} N{N} nfe{nfe} cfg{cfg}: {got:.6e} vs {want:.6e}")
        assert abs(got - want) <= 1e-9 * want


# ---------------------------------------------------------------------------------------------------------------------
# top level: F5TTS.infer, packed-weight cache, serving
# ---------------------------------------------------------------------------------------------------------------------
REF_TEXT = "Some call me nature, others call me mother nature."
GEN_SHORT = "I don't really care what you call me."
NFE = 4


@pytest.fixture(scope="module")
def small_tts(tmp_path_factory, golden_dir):
    """F5TTS(model="F5TTS_v1_Small") over an EMA checkpoint and a vocoder folder in the released on-disk layouts."""
    from safetensors.torch import save_file

    _models.clear()
    d = tmp_path_factory.mktemp("f5assets_small")
    cfg = SD.f5tts_v1_small()
    sd = SD.synthetic_state_dict(cfg, seed=1234)
    ema = {"ema_model." + k: v for k, v in sd.items()}
    ema["initted"], ema["step"] = torch.tensor(True), torch.tensor(1)
    ckpt = str(d / "model_1.safetensors")
    save_file(ema, ckpt)
    vcfg = {"feature_extractor": {"class_path": "vocos.feature_extractors.MelSpectrogramFeatures",
                                  "init_args": {"sample_rate": 24000, "n_fft": 1024, "hop_length": 256, "n_mels": 100,
                                                "padding": "center"}},
            "backbone": {"class_path": "vocos.models.VocosBackbone",
                         "init_args": {"input_channels": 100, "dim": 512, "intermediate_dim": 1536, "num_layers": 8}},
            "head": {"class_path": "vocos.heads.ISTFTHead",
                     "init_args": {"dim": 512, "n_fft": 1024, "hop_length": 256, "padding": "center"}}}
    vdir = d / "vocos"
    vdir.mkdir()
    (vdir / "config.yaml").write_text(yaml.safe_dump(vcfg))
    vsd = SD.synthetic_vocos_state_dict()
    full = dict(vsd)
    full["feature_extractor.mel_spec.spectrogram.window"] = torch.hann_window(1024)
    full["feature_extractor.mel_spec.mel_scale.fb"] = O.mel_filterbank()
    torch.save(full, str(vdir / "pytorch_model.bin"))
    vocab = os.path.join(golden_dir, "vocab.txt")
    tts = api.F5TTS(model="F5TTS_v1_Small", ckpt_file=ckpt, vocab_file=vocab, vocoder_local_path=str(vdir), device=DEV)
    return dict(tts=tts, sd=sd, vsd=vsd, cfg=cfg, ckpt=ckpt, vocab=vocab, ref=os.path.join(golden_dir, "basic_ref_en.wav"))


def test_f5tts_small_infer_vs_oracle(small_tts):
    """test_gpu_infer.py's recipe: the expected chunk is the reference's formulas on top of the CPU oracle with the noise
    `sample` drew on the device after seed_everything(seed)."""
    a = small_tts
    seed = 1234
    wav, sr, spec = a["tts"].infer(a["ref"], REF_TEXT, GEN_SHORT, nfe_step=NFE, seed=seed, show_info=lambda *_: None)
    audio, asr = infer._load_wav(a["ref"])
    assert sr == asr == 24000
    rms = float(torch.sqrt(torch.mean(torch.square(audio))))
    if rms < 0.1:
        audio = audio * 0.1 / rms
    ref_text = REF_TEXT + "  "  # preprocess_ref_audio_text and infer_batch_process each append one space
    ref_len = audio.shape[-1] // 256
    duration = ref_len + int(ref_len / len(ref_text.encode("utf-8")) * len(GEN_SHORT.encode("utf-8")))
    api.seed_everything(seed)
    y0 = torch.randn(duration, 100, device=DEV, dtype=torch.float16).float().cpu()[None]
    ids = list_str_to_idx(infer.convert_char_to_pinyin([ref_text + GEN_SHORT]), a["tts"].ema_model.vocab_char_map)
    cond = O.mel_spectrogram(audio).permute(0, 2, 1).half().float()
    res = O.sample(a["sd"], a["cfg"], cond, ids, duration, steps=NFE, cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y0)
    s_ref = res.out.half().float()[:, ref_len:, :].permute(0, 2, 1)
    w_ref = O.vocos_decode(a["vsd"], s_ref)
    if rms < 0.1:
        w_ref = w_ref * rms / 0.1
    s_ref, w_ref = s_ref[0].numpy(), w_ref.squeeze().numpy()
    assert spec.shape == s_ref.shape and wav.shape == w_ref.shape
    rs, rw = rel(spec, s_ref), rel(wav, w_ref)
    print(f"[F5TTS_v1_Small.infer] {duration} frames ({ref_len} prompt): spectrogram rel-L2 {rs:.3e}, waveform {rw:.3e}")
    assert rs <= 5e-3 and rw <= 2e-2


def test_small_packed_weight_cache_roundtrip(small_tts, tmp_path):
    import glob

    from f5_tts_b200 import weights as Wt

    a = small_tts
    cls, arch = api.MODEL_ARCH["F5TTS_v1_Small"]
    cache = str(tmp_path / "pack")
    m1 = infer.load_model(cls, arch, a["ckpt"], vocab_file=a["vocab"], device=DEV, packed_cache_dir=cache)
    assert len(glob.glob(os.path.join(cache, "f5pack_*.safetensors"))) == 1
    calls = {"n": 0}
    orig = Wt.packed_tensors

    def counting(m):
        calls["n"] += 1
        return orig(m)

    Wt.packed_tensors = counting
    try:
        m2 = infer.load_model(cls, arch, a["ckpt"], vocab_file=a["vocab"], device=DEV, packed_cache_dir=cache)
        g = torch.Generator().manual_seed(64)
        cond = torch.randn(1, 40, 100, generator=g).to(DEV)
        text = torch.randint(0, 2545, (1, 30), generator=g).to(DEV)
        y0 = torch.randn(1, 150, 100, generator=g).to(DEV)
        kw = dict(steps=2, cfg_strength=2.0, sway_sampling_coef=-1.0)
        o2, _ = m2.sample(cond.half(), text, 150, **kw, y0=y0)
        assert calls["n"] == 0, "the second load must not re-pack"
    finally:
        Wt.packed_tensors = orig
    o1, _ = m1.sample(cond.half(), text, 150, **kw, y0=y0)
    assert m2.transformer.dim == 768 and torch.equal(o1, o2)


def test_small_serving_batched_equals_single(small_tts):
    from f5_tts_b200 import serving

    a = small_tts
    audio, _ = infer._load_wav(a["ref"])
    wav = audio.numpy()
    reqs = [{"reference_wav": wav, "reference_text": REF_TEXT, "target_text": "Hello there."},
            {"reference_wav": wav[:, :60000], "reference_wav_len": np.array([60000], np.int32),
             "reference_text": "Some call me nature,", "target_text": "I am mighty and enduring."}]
    proc = serving.F5TTSRequestProcessor(a["tts"].ema_model, a["tts"].vocoder, device=DEV, nfe_step=NFE, seed=11)
    batched = proc.execute(reqs)
    singles = [proc.execute([r])[0] for r in reqs]
    for b, s in zip(batched, singles):
        assert np.isfinite(b).all() and float(np.abs(b).max()) > 0
        assert np.array_equal(b, s)


def test_small_socket_server_loads_by_model_name(small_tts):
    """socket_server's `--model F5TTS_v1_Small` resolves through api.MODEL_ARCH and loads the Small checkpoint."""
    from f5_tts_b200 import socket_server

    a = small_tts
    proc = socket_server.TTSStreamingProcessor("F5TTS_v1_Small", a["ckpt"], a["vocab"], a["ref"], REF_TEXT, device=DEV,
                                               vocoder=a["tts"].vocoder)
    tr = proc.model.transformer
    assert (tr.dim, tr.depth, tr.heads) == (768, 18, 12)
