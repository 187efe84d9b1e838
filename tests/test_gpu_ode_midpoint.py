"""GPU: CFM.sample with torchdiffeq's fixed-grid midpoint solver (odeint_kwargs=dict(method="midpoint")), which makes
two backbone evaluations per grid interval through the same captured step graph as Euler.

  * the engine against the unmodified reference's midpoint sample (tests/golden/f5base_b2_varlen_midpoint.npz, made by
    oracle/make_golden_midpoint.py) and against the CPU oracle on fresh inputs — rel-L2 <= 5e-3 as for Euler
    (test_gpu_sample.py);
  * exact_varlen, graph replay vs eager launches, determinism, Euler/midpoint alternation on one model, launch and FLOP
    accounting;
  * the top-level F5TTS(ode_method="midpoint").infer and the serving processor.
"""
import os

import numpy as np
import pytest
import torch
import yaml

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import f5_tts_b200 as F5  # noqa: E402
import synthdata as SD  # noqa: E402
from f5_tts_b200 import _lib  # noqa: E402
from oracle import f5_oracle as O  # noqa: E402
from oracle import ode_midpoint as OM  # noqa: E402

DEV = "cuda:0"
TOL = 5e-3
_models = {}


def build(cfg: O.ArchConfig, wseed: int):
    """One CFM per (config, seed) kept resident; its ODE method is set per call by `with_method`."""
    key = (repr(cfg), wseed)
    if key not in _models:
        _models.clear()
        cls = F5.DiT if cfg.backbone == "DiT" else F5.UNetT
        kw = dict(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
                  mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim,
                  text_mask_padding=cfg.text_mask_padding, conv_layers=cfg.conv_layers, pe_attn_head=cfg.pe_attn_head,
                  attn_mask_enabled=cfg.attn_mask_enabled)
        model = F5.CFM(transformer=cls(**kw), odeint_kwargs=dict(method="midpoint"))
        sd = O.synthetic_state_dict(cfg, seed=wseed)
        model.load_state_dict(sd, strict=True)
        _models[key] = (model.to(DEV), sd)
    return _models[key]


def with_method(model, method):
    model.odeint_kwargs = dict(method=method)  # a fresh dict: never mutate the constructor's default argument
    return model


def rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm())


def test_midpoint_vs_reference_golden(golden_dir):
    from oracle import make_golden_midpoint as MM

    cfg, wseed, cond, text, dur, lens, kw = MM.full_width_case()
    z = np.load(os.path.join(golden_dir, MM.FULL + ".npz"))
    model = with_method(build(cfg, wseed)[0], "midpoint")
    out, traj = model.sample(cond.to(DEV), text.to(DEV), dur.to(DEV), lens=lens.to(DEV), **kw,
                             y0=torch.from_numpy(z["y0"]).to(DEV))
    r1, rN = rel(traj[1], torch.from_numpy(z["traj_1"])), rel(out, torch.from_numpy(z["out"]))
    print(f"[midpoint golden] step-1 rel-L2 {r1:.3e}  final rel-L2 {rN:.3e}")
    assert traj.shape[0] == kw["steps"] + 1 and out.shape == z["out"].shape
    assert r1 <= TOL and rN <= TOL


@pytest.mark.parametrize("variant", ["mask_faithful", "attn_mask", "no_cfg", "wave_epss", "unett"])
def test_midpoint_vs_oracle(variant):
    cfg = O.e2tts_base() if variant == "unett" else O.f5tts_base()
    if variant == "attn_mask":
        cfg.attn_mask_enabled = True
    model, sd = build(cfg, 1234)
    model = with_method(model, "midpoint")
    g = torch.Generator().manual_seed(43)
    kw = dict(steps=2, cfg_strength=2.0, sway_sampling_coef=-1.0, seed=7)
    if variant in ("mask_faithful", "attn_mask"):
        cond = torch.randn(3, 40, 100, generator=g)
        text = torch.randint(0, 2545, (3, 30), generator=g)
        text[1, 20:] = -1
        args = (cond, text, torch.tensor([150, 97, 131]))
        kw["lens"] = torch.tensor([40, 25, 33])
    elif variant == "unett":
        cond = torch.randn(2, 36, 100, generator=g)
        text = torch.randint(0, 2545, (2, 28), generator=g)
        text[1, 18:] = -1
        args = (cond, text, torch.tensor([140, 104]))
        kw["lens"] = torch.tensor([36, 30])
    elif variant == "no_cfg":
        args = (torch.randn(1, 30, 100, generator=g), torch.randint(0, 2545, (1, 25), generator=g), 130)
        kw.update(steps=3, cfg_strength=0.0, sway_sampling_coef=None)
    else:  # raw wave in (mel kernel) + the EPSS grid of 5 steps
        args = (0.1 * torch.randn(1, 30 * 256, generator=g), torch.randint(0, 2545, (1, 25), generator=g), 140)
        kw["steps"] = 5
    ref = OM.sample(sd, cfg, *args, method="midpoint", **kw)
    dargs = tuple(a.to(DEV) if torch.is_tensor(a) else a for a in args)
    dkw = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in kw.items()}
    out, traj = model.sample(*dargs, **dkw, y0=ref.y0.to(DEV))
    assert traj.shape[0] == kw["steps"] + 1
    if variant == "attn_mask":  # key-masked mode: padded rows are not computed, compare every sample's valid rows
        durs = args[2].tolist()
        got = torch.cat([out[b, :d].cpu() for b, d in enumerate(durs)])
        want = torch.cat([ref.out[b, :d] for b, d in enumerate(durs)])
        r = rel(got, want)
    else:
        r = rel(out, ref.out)
    print(f"[midpoint oracle:{variant}] final rel-L2 {r:.3e}")
    assert r <= TOL


def test_midpoint_exact_varlen_batch_equals_single_calls():
    cfg = O.f5tts_base()
    model = with_method(build(cfg, 1234)[0], "midpoint")
    g = torch.Generator().manual_seed(34)
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
        r = rel(out[b, :d], singles[b][0])
        print(f"[midpoint exact_varlen] sample {b} ({d} frames): batched vs single rel-L2 {r:.3e}")
        assert r <= 1e-3


def _inputs(seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(1, 50, 100, generator=g).to(DEV), torch.randint(0, 2545, (1, 40), generator=g).to(DEV),
            torch.randn(1, 200, 100, generator=g).to(DEV))


def test_midpoint_graph_equals_eager_and_deterministic():
    model = with_method(build(O.f5tts_base(), 1234)[0], "midpoint")
    cond, text, y0 = _inputs(1)
    kw = dict(steps=4, cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y0)
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


def test_euler_midpoint_alternation_keeps_euler_bit_identical():
    """One model, one workspace, same shapes: Euler, midpoint, Euler.  A midpoint call between them (which may replay or
    capture a step graph on the same workspace) leaves the Euler result bit-identical, and the two methods differ."""
    model = build(O.f5tts_base(), 1234)[0]
    cond, text, y0 = _inputs(2)
    kw = dict(steps=4, cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y0)
    e1, te1 = with_method(model, "euler").sample(cond, text, 200, **kw)
    m, tm = with_method(model, "midpoint").sample(cond, text, 200, **kw)
    e2, te2 = with_method(model, "euler").sample(cond, text, 200, **kw)
    # Euler over 8 steps has as many evaluations as midpoint over 4 and shares its step graph
    with_method(model, "euler").sample(cond, text, 200, **dict(kw, steps=8))
    m2, _ = with_method(model, "midpoint").sample(cond, text, 200, **kw)
    e3, _ = with_method(model, "euler").sample(cond, text, 200, **kw)
    with_method(model, "midpoint")
    assert torch.equal(e1, e2) and torch.equal(te1, te2) and torch.equal(e1, e3)
    assert torch.equal(m, m2)
    assert tm.shape == te1.shape and rel(m, e1) > 1e-3


def test_midpoint_launches_and_flops_match_euler_with_twice_the_steps():
    model = build(O.f5tts_base(), 1234)[0]
    cond, text, y0 = _inputs(3)
    kw = dict(cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y0)
    counts = {}
    try:
        for graph in (True, False):
            model.use_cuda_graph = graph
            for method, steps in (("midpoint", 3), ("euler", 6)):
                with_method(model, method).sample(cond, text, 200, steps=steps, **kw)  # warm (captures the graph)
                torch.cuda.synchronize()
                n0 = _lib.launch_count()
                with_method(model, method).sample(cond, text, 200, steps=steps, **kw)
                torch.cuda.synchronize()
                counts[(graph, method)] = _lib.launch_count() - n0
    finally:
        model.use_cuda_graph = True
        with_method(model, "midpoint")
    print(f"[midpoint launches] {counts}")
    for graph in (True, False):
        assert counts[(graph, "midpoint")] == counts[(graph, "euler")] > 0
    tr = model.transformer
    mid, e1, e2 = tr.sample_flops(2, 300, 16, 2.0, "midpoint"), tr.sample_flops(2, 300, 16, 2.0), tr.sample_flops(2, 300, 32, 2.0)
    assert mid == e2  # 32 backbone evaluations either way
    assert 1.95 * e1 < mid <= 2 * e1  # twice Euler's backbone and conditioning work; the text embedding runs once


@pytest.fixture(scope="module")
def tts_midpoint(tmp_path_factory, golden_dir):
    """Checkpoint + vocoder folder in the released on-disk layouts (as in test_gpu_infer.py), loaded by
    F5TTS(ode_method="midpoint")."""
    from safetensors.torch import save_file

    from f5_tts_b200 import api

    _models.clear()
    d = tmp_path_factory.mktemp("f5assets_midpoint")
    sd = SD.synthetic_state_dict(SD.f5tts_base(), seed=1234)
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
    full = dict(SD.synthetic_vocos_state_dict())
    full["feature_extractor.mel_spec.spectrogram.window"] = torch.hann_window(1024)
    full["feature_extractor.mel_spec.mel_scale.fb"] = O.mel_filterbank()
    torch.save(full, str(vdir / "pytorch_model.bin"))
    tts = api.F5TTS(model="F5TTS_Base", ckpt_file=ckpt, vocab_file=os.path.join(golden_dir, "vocab.txt"),
                    vocoder_local_path=str(vdir), device=DEV, ode_method="midpoint")
    return tts, os.path.join(golden_dir, "basic_ref_en.wav")


def test_f5tts_infer_midpoint_end_to_end(tts_midpoint):
    tts, ref = tts_midpoint
    assert tts.ema_model.odeint_kwargs["method"] == "midpoint"
    ref_text, gen = "Some call me nature, others call me mother nature.", "I don't really care what you call me."
    wm, sr, spec_m = tts.infer(ref, ref_text, gen, nfe_step=4, seed=5, show_info=lambda *_: None)
    tts.ema_model.odeint_kwargs = dict(method="euler")
    try:
        we, _, spec_e = tts.infer(ref, ref_text, gen, nfe_step=4, seed=5, show_info=lambda *_: None)
    finally:
        tts.ema_model.odeint_kwargs = dict(method="midpoint")
    print(f"[F5TTS midpoint] {len(wm)} samples, spectrogram midpoint vs euler rel-L2 {rel(torch.from_numpy(spec_m), torch.from_numpy(spec_e)):.3e}")
    assert sr == 24000 and np.isfinite(wm).all() and float(np.abs(wm).max()) > 0
    assert wm.shape == we.shape and spec_m.shape == spec_e.shape
    assert not np.array_equal(spec_m, spec_e)


def test_serving_midpoint_batched_equals_single(tts_midpoint):
    from f5_tts_b200 import infer, serving

    tts, ref = tts_midpoint
    audio, _ = infer._load_wav(ref)
    wav = audio.numpy()
    reqs = [{"reference_wav": wav, "reference_text": "Some call me nature, others call me mother nature.",
             "target_text": "Hello there."},
            {"reference_wav": wav[:, :60000], "reference_wav_len": np.array([60000], np.int32),
             "reference_text": "Some call me nature,", "target_text": "I am mighty and enduring."}]
    proc = serving.F5TTSRequestProcessor(tts.ema_model, tts.vocoder, device=DEV, nfe_step=4, seed=11)
    batched = proc.execute(reqs)
    singles = [proc.execute([r])[0] for r in reqs]
    for b, s in zip(batched, singles):
        assert np.isfinite(b).all() and float(np.abs(b).max()) > 0
        assert np.array_equal(b, s)
