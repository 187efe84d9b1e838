"""GPU: the samples of one CFM.sample call run in groups on several engines (CFM.enable_sample_parallel).

  * Loopback (every group on cuda:0, each on its own stream and workspace: the same code path as several devices), with
    2 and 3 groups.  The split call's final mel and full trajectory equal the unsplit call bit for bit for DiT at B = 3
    and B = 5 in the faithful, attn_mask and exact_varlen modes; midpoint; UNetT with concat and add skips; MMDiT;
    dim_head 128; cfg_strength 0; eager against graph; more devices than samples; repeated calls (no new workspace, no
    weight copy); a peer with its own weight copy on the same GPU that follows a weight edit; concurrent threads; merged
    runs of enable_batching; infer_batch_process and F5TTS.infer end to end.  Under exact_varlen the trajectory's rows
    past each sample's duration are zero and y keeps its input there.
  * Two devices (skipped with fewer than two): the same equalities against the single-device call, and the caller's
    stream sees finished results without a synchronise.
"""
import os
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import f5_tts_b200 as F5  # noqa: E402
import synthdata as SD  # noqa: E402
from f5_tts_b200 import infer, sample_parallel  # noqa: E402

DEV = "cuda:0"
TWO_GPUS = torch.cuda.device_count() >= 2
DURATIONS = [300, 250, 101, 90, 133]  # under exact_varlen the groups run at 300, 256 or 128 frames instead of 300


def cfg(backbone="DiT", **kw):
    base = dict(dim=128, depth=2, heads=2, ff_mult=2, text_num_embeds=50, text_dim=64, text_mask_padding=True,
                conv_layers=2, pe_attn_head=None)
    if backbone == "UNetT":
        base.update(depth=4, text_dim=None, text_mask_padding=False, conv_layers=0, pe_attn_head=1)
    if backbone == "MMDiT":
        base.update(depth=3, text_dim=None, conv_layers=0)
    base.update(kw)
    return SD.ArchConfig(backbone=backbone, **base)


def build(c: SD.ArchConfig, device=DEV, method="euler") -> F5.CFM:
    kw = dict(dim=c.dim, depth=c.depth, heads=c.heads, dim_head=c.dim_head, ff_mult=c.ff_mult, mel_dim=c.mel_dim,
              text_num_embeds=c.text_num_embeds, text_mask_padding=c.text_mask_padding,
              attn_mask_enabled=c.attn_mask_enabled)
    if c.backbone != "MMDiT":
        kw.update(text_dim=c.text_dim, conv_layers=c.conv_layers, pe_attn_head=c.pe_attn_head)
    if c.backbone == "UNetT":
        kw.update(skip_connect_type=c.skip_connect_type)
    model = F5.CFM(transformer=getattr(F5, c.backbone)(**kw), odeint_kwargs=dict(method=method))
    model.load_state_dict(SD.synthetic_state_dict(c, seed=1234), strict=True)
    return model.to(device)


def inputs(b=3, seed=5, pad_text=False, **extra):
    """(args, kwargs) of one sample() call: b samples of different durations, seeded noise."""
    g = torch.Generator().manual_seed(seed)
    cond = torch.randn(b, 40, 100, generator=g).to(DEV)
    text = torch.randint(0, 50, (b, 24), generator=g)
    if pad_text:
        text[-1, 15:] = -1
    duration = torch.tensor(DURATIONS[:b]).to(DEV) if b > 1 else DURATIONS[0]
    return (cond, text.to(DEV), duration), dict(steps=8, cfg_strength=2.0, sway_sampling_coef=-1.0, seed=seed, **extra)


def split_and_solo(model, args, kw, devices):
    want = model.sample(*args, **kw)
    peers = model.enable_sample_parallel(devices)
    try:
        got = model.sample(*args, **kw)
    finally:
        model.disable_sample_parallel()
    assert sum(len(p._ws_free) > 0 for p in peers) >= 2, "the call did not run as two or more groups"
    return got, want


def assert_same(got, want, what, lengths=None):
    """Bit equality of final mel and trajectory.  `lengths`: compare each sample's first lengths[b] frames only — with
    attn_mask_enabled (DiT, UNetT concat) or exact_varlen the engine skips tiles that hold only padding, so the frames
    past a sample's duration are not defined, in the unsplit call as in the split one."""
    (out, traj), (wout, wtraj) = got, want
    assert out.shape == wout.shape and traj.shape == wtraj.shape
    if lengths is not None:
        pairs = [((out[b, :d], traj[:, b, :d]), (wout[b, :d], wtraj[:, b, :d])) for b, d in enumerate(lengths)]
    else:
        pairs = [((out, traj), (wout, wtraj))]
    for (o, t), (wo, wt) in pairs:
        assert torch.isfinite(t).all()
        assert torch.equal(o, wo), f"{what}: final mel differs from the unsplit call"
        assert torch.equal(t, wt), f"{what}: trajectory differs from the unsplit call"


def assert_zero_past_duration(traj, lengths):
    """exact_varlen: the split writes zeros to the trajectory rows the mode does not define."""
    for b, d in enumerate(lengths):
        assert not traj[:, b, d:].any()


# ---------------------------------------------------------------------------------------------------------------------
# loopback
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b,groups", [(3, 2), (5, 3)])
@pytest.mark.parametrize("mode", ["faithful", "attn_mask", "exact_varlen"])
def test_dit(mode, b, groups):
    model = build(cfg(attn_mask_enabled=mode == "attn_mask", text_mask_padding=False, pe_attn_head=1))
    args, kw = inputs(b=b, exact_varlen=mode == "exact_varlen")
    got, want = split_and_solo(model, args, kw, [DEV] * groups)
    lengths = None if mode == "faithful" else args[2].tolist()
    assert_same(got, want, f"DiT B={b} {mode}", lengths=lengths)
    if mode == "exact_varlen":
        assert_zero_past_duration(got[1], lengths)


def test_exact_varlen_rows_past_duration():
    """Through the backbone's run: the valid rows equal the unsplit call, y keeps its input past each duration and the
    trajectory is zero there."""
    model = build(cfg())
    bb = model.transformer
    g = torch.Generator().manual_seed(3)
    B, N = 5, 300
    y0 = torch.randn(B, N, 100, generator=g).to(DEV)
    sc = torch.randn(B, N, 100, generator=g).to(DEV)
    text = torch.randint(0, 50, (B, 24), generator=g).to(DEV)
    dur = torch.tensor(DURATIONS, dtype=torch.int32, device=DEV)
    t = [k / 8 for k in range(9)]
    y_a, traj_a = y0.clone(), torch.empty(9, B, N, 100, device=DEV)
    bb.run(y_a, sc, text, t, dur, 2.0, trajectory=traj_a, exact_varlen=True)
    model.enable_sample_parallel([DEV] * 3)
    try:
        y_b, traj_b = y0.clone(), torch.full((9, B, N, 100), float("nan"), device=DEV)
        bb.run(y_b, sc, text, t, dur, 2.0, trajectory=traj_b, exact_varlen=True)
    finally:
        model.disable_sample_parallel()
    torch.cuda.synchronize()
    for b, d in enumerate(DURATIONS):
        assert torch.equal(y_b[b, :d], y_a[b, :d]) and torch.equal(traj_b[:, b, :d], traj_a[:, b, :d])
        assert torch.equal(y_b[b, d:], y0[b, d:])
    assert_zero_past_duration(traj_b, DURATIONS)


def test_midpoint():
    model = build(cfg(), method="midpoint")
    got, want = split_and_solo(model, *inputs(b=3), [DEV] * 2)
    assert_same(got, want, "midpoint")


@pytest.mark.parametrize("skip", ["concat", "add"])
def test_unett(skip):
    model = build(cfg("UNetT", skip_connect_type=skip))
    got, want = split_and_solo(model, *inputs(b=3), [DEV] * 3)
    assert_same(got, want, f"UNetT {skip}")


@pytest.mark.parametrize("mode", ["faithful", "exact_varlen"])
def test_mmdit(mode):
    model = build(cfg("MMDiT"))
    args, kw = inputs(b=3, pad_text=True, exact_varlen=mode == "exact_varlen")
    got, want = split_and_solo(model, args, kw, [DEV] * 2)
    assert_same(got, want, f"MMDiT {mode}", lengths=args[2].tolist() if mode == "exact_varlen" else None)


@pytest.mark.parametrize("backbone", ["DiT", "UNetT"])
def test_dim_head_128(backbone):
    model = build(cfg(backbone, dim=256, heads=2, dim_head=128))
    got, want = split_and_solo(model, *inputs(b=3), [DEV] * 2)
    assert_same(got, want, f"{backbone} dim_head 128")


def test_cfg_strength_zero_splits():
    model = build(cfg())
    args, kw = inputs(b=3)
    got, want = split_and_solo(model, args, dict(kw, cfg_strength=0.0), [DEV] * 2)
    assert_same(got, want, "cfg 0")


def test_one_sample_and_forward_stay_local():
    model = build(cfg())
    args, kw = inputs(b=1)
    want = model.sample(*args, **kw)
    peers = model.enable_sample_parallel([DEV] * 2)
    try:
        got = model.sample(*args, **kw)
        bb = model.transformer
        x = torch.randn(2, 60, 100, device=DEV)
        text = torch.randint(0, 50, (2, 20), device=DEV)
        got_v = bb(x, torch.zeros_like(x), text, torch.tensor([0.3], device=DEV), cfg_infer=True)
    finally:
        model.disable_sample_parallel()
    assert all(not p._ws_free for p in peers)  # no group ran
    assert_same(got, want, "B = 1")
    want_v = bb(x, torch.zeros_like(x), text, torch.tensor([0.3], device=DEV), cfg_infer=True)
    assert torch.equal(got_v, want_v)


def test_more_devices_than_samples():
    model = build(cfg())
    args, kw = inputs(b=2, exact_varlen=True)
    got, want = split_and_solo(model, args, kw, [DEV] * 4)
    assert_same(got, want, "4 devices, 2 samples", lengths=args[2].tolist())


def test_eager_graph_and_repeats():
    """Split eager, split graph (three times: capture, then replay) and unsplit graph: one answer."""
    model = build(cfg())
    args, kw = inputs(b=5)
    want = model.sample(*args, **kw)
    model.enable_sample_parallel([DEV] * 3)
    try:
        model.use_cuda_graph = False
        eager = model.sample(*args, **kw)
        model.use_cuda_graph = True
        graph = [model.sample(*args, **kw) for _ in range(3)]
    finally:
        model.disable_sample_parallel()
    assert_same(eager, want, "eager split")
    for g in graph:
        assert_same(g, want, "graph split")


def test_steady_state_calls_stay_warm():
    """Enabling again keeps the peers; repeated calls reuse one workspace per peer (so its captured graph) and copy no
    weights."""
    model = build(cfg())
    args, kw = inputs(b=5, exact_varlen=True)
    want = model.sample(*args, **kw)
    peers = model.enable_sample_parallel([DEV] * 3)
    try:
        got = [model.sample(*args, **kw)]
        ws = [[w.data_ptr() for w in p._ws_free] for p in peers]
        for _ in range(3):
            assert model.enable_sample_parallel([DEV] * 3) is peers
            got.append(model.sample(*args, **kw))
        assert [[w.data_ptr() for w in p._ws_free] for p in peers] == ws
        assert all(len(w) == 1 for w in ws) and all(p.replications == 0 for p in peers)
    finally:
        model.disable_sample_parallel()
    for g in got:
        assert_same(g, want, "steady state", lengths=args[2].tolist())


def test_weight_copy_on_one_gpu_follows_edits():
    """Peers with their own weight copies on the same GPU: the path a second device takes (replication, another engine,
    its graph cache).  Equal to the unsplit call, and a weight edit on the primary is copied again before the next
    split call."""
    model = build(cfg())
    args, kw = inputs(b=3)
    want = model.sample(*args, **kw)
    split = sample_parallel.SampleSplit([DEV, DEV], copy_weights=True)
    model.transformer.sample_split = split
    try:
        got = model.sample(*args, **kw)
        primary = model.transformer.engine()["handle"].value
        assert [p.replications for p in split.peers] == [1, 1]
        assert all(p._state["handle"].value != primary for p in split.peers)
        with torch.no_grad():
            model.transformer.proj_out.weight.mul_(1.5)  # in place: the fingerprint changes
        edited = model.sample(*args, **kw)
        assert [p.replications for p in split.peers] == [2, 2]
    finally:
        model.disable_sample_parallel()
    want_edited = model.sample(*args, **kw)
    assert_same(got, want, "weight copy")
    assert not torch.equal(edited[0], want[0])
    assert_same(edited, want_edited, "weight copy after an edit")


def test_concurrent_threads():
    model = build(cfg())
    cases = [inputs(b=3, seed=s, exact_varlen=True) for s in (21, 22, 23)]
    want = [model.sample(*a, **k) for a, k in cases]
    model.enable_sample_parallel([DEV] * 2)
    results, errors = {}, []

    def work(i):
        try:
            s = torch.cuda.Stream(DEV)
            with torch.cuda.stream(s):
                results[i] = [model.sample(*cases[i][0], **cases[i][1]) for _ in range(2)]
            s.synchronize()
        except Exception as e:  # noqa: BLE001 — reported by the main thread
            errors.append(e)

    try:
        th = [threading.Thread(target=work, args=(i,)) for i in range(len(cases))]
        for t in th:
            t.start()
        for t in th:
            t.join(120)
    finally:
        model.disable_sample_parallel()
    assert not errors, errors
    for i, w in enumerate(want):
        for got in results[i]:
            assert_same(got, w, f"thread {i}", lengths=cases[i][0][2].tolist())


def test_with_batching():
    """enable_batching's merged runs go through the backbone's run: a run of two or more samples splits, and each caller
    gets its solo answer."""
    model = build(cfg())
    cases = [inputs(b=1, seed=s) for s in (31, 32, 33)] + [inputs(b=3, seed=34, exact_varlen=True)]
    want = [model.sample(*a, **k) for a, k in cases]
    stats = model.enable_batching()
    peers = model.enable_sample_parallel([DEV] * 2)
    results, errors = {}, []

    def work(i):
        try:
            results[i] = model.sample(*cases[i][0], **cases[i][1])
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    try:
        th = [threading.Thread(target=work, args=(i,)) for i in range(len(cases))]
        for t in th:
            t.start()
        for t in th:
            t.join(120)
    finally:
        model.disable_sample_parallel()
        model.disable_batching()
    assert not errors, errors
    assert stats.calls == len(cases) and any(p._ws_free for p in peers)
    for i, w in enumerate(want):
        lengths = None if i < 3 else cases[i][0][2].tolist()
        assert_same(results[i], w, f"batched call {i}", lengths=lengths)


def test_infer_batch_process_and_f5tts_infer(tmp_path, golden_dir):
    """A chunked request through infer_batch_process, and F5TTS(sample_parallel_devices=...).infer of a text long enough
    for several chunks, equal their unsplit runs."""
    import yaml
    from safetensors.torch import save_file

    from f5_tts_b200 import api
    from oracle import f5_oracle as O

    sd = SD.synthetic_state_dict(SD.f5tts_v1_small(), seed=1234)
    ema = {"ema_model." + k: v for k, v in sd.items()}
    ema["initted"], ema["step"] = torch.tensor(True), torch.tensor(1)
    ckpt = str(tmp_path / "model_1.safetensors")
    save_file(ema, ckpt)
    vcfg = {"feature_extractor": {"class_path": "vocos.feature_extractors.MelSpectrogramFeatures",
                                  "init_args": {"sample_rate": 24000, "n_fft": 1024, "hop_length": 256, "n_mels": 100,
                                                "padding": "center"}},
            "backbone": {"class_path": "vocos.models.VocosBackbone",
                         "init_args": {"input_channels": 100, "dim": 512, "intermediate_dim": 1536, "num_layers": 8}},
            "head": {"class_path": "vocos.heads.ISTFTHead",
                     "init_args": {"dim": 512, "n_fft": 1024, "hop_length": 256, "padding": "center"}}}
    vdir = tmp_path / "vocos"
    vdir.mkdir()
    (vdir / "config.yaml").write_text(yaml.safe_dump(vcfg))
    full = dict(SD.synthetic_vocos_state_dict())
    full["feature_extractor.mel_spec.spectrogram.window"] = torch.hann_window(1024)
    full["feature_extractor.mel_spec.mel_scale.fb"] = O.mel_filterbank()
    torch.save(full, str(vdir / "pytorch_model.bin"))
    vocab = os.path.join(golden_dir, "vocab.txt")
    ref = os.path.join(golden_dir, "basic_ref_en.wav")
    ref_text = "Some call me nature, others call me mother nature."
    plain = api.F5TTS(model="F5TTS_v1_Small", ckpt_file=ckpt, vocab_file=vocab, vocoder_local_path=str(vdir), device=DEV)
    split = api.F5TTS(model="F5TTS_v1_Small", ckpt_file=ckpt, vocab_file=vocab, vocoder_local_path=str(vdir), device=DEV,
                      sample_parallel_devices=[DEV, DEV, DEV])
    assert plain.ema_model.transformer.sample_split is None
    ss = split.ema_model.transformer.sample_split
    split_calls, run = [], ss.run
    ss.run = lambda *a, **k: (split_calls.append(a[1].shape[0]), run(*a, **k))[1]

    audio, sr = infer._load_wav(ref)
    chunks = ["I don't really care what you call me.", "Short one.", "And I will be here long after you are gone."]
    outs = []
    for t in (plain, split):
        torch.manual_seed(77)
        outs.append(next(infer.infer_batch_process((audio, sr), ref_text + " ", chunks, t.ema_model, t.vocoder,
                                                   nfe_step=6, device=DEV)))
    (w1, _, s1), (w2, _, s2) = outs
    assert np.isfinite(w1).all() and np.array_equal(w1, w2) and np.array_equal(s1, s2)
    assert split_calls == [3]

    gen = ("I don't really care what you call me. I've been a silent spectator, watching species evolve, empires rise "
           "and fall. But always remember, I am mighty and enduring. Respect me and I'll nurture you; ignore me and "
           "you shall face the consequences.")
    outs = [t.infer(ref, ref_text, gen, nfe_step=6, seed=5, show_info=lambda *_: None) for t in (plain, split)]
    assert len(split_calls) == 2 and split_calls[1] >= 2  # the text went into one call of several chunks
    (w1, _, s1), (w2, _, s2) = outs
    assert np.isfinite(w1).all() and np.array_equal(w1, w2) and np.array_equal(s1, s2)


# ---------------------------------------------------------------------------------------------------------------------
# two devices
# ---------------------------------------------------------------------------------------------------------------------
two_gpus = pytest.mark.skipif(not TWO_GPUS, reason="needs two CUDA devices (a group runs on cuda:1)")


@two_gpus
@pytest.mark.parametrize("case", ["dit_faithful", "dit_varlen", "unett_add", "mmdit_varlen"])
def test_two_devices_equal_single_device(case):
    c = {"dit_faithful": cfg(), "dit_varlen": cfg(), "unett_add": cfg("UNetT", skip_connect_type="add"),
         "mmdit_varlen": cfg("MMDiT")}[case]
    model = build(c)
    varlen = case.endswith("varlen")
    args, kw = inputs(b=5, pad_text=case.startswith("mmdit"), exact_varlen=varlen)
    got, want = split_and_solo(model, args, kw, ["cuda:0", "cuda:1", "cuda:1"])
    assert_same(got, want, case, lengths=args[2].tolist() if varlen else None)
    if varlen:
        assert_zero_past_duration(got[1], args[2].tolist())


@two_gpus
def test_two_devices_caller_stream_sees_results():
    """Work queued on the caller's stream after sample() reads the finished result: no synchronise in between."""
    model = build(cfg())
    args, kw = inputs(b=3)
    want = model.sample(*args, **kw)
    model.enable_sample_parallel(["cuda:1", "cuda:0"])
    s = torch.cuda.Stream(DEV)
    try:
        with torch.cuda.stream(s):
            for _ in range(3):
                out, traj = model.sample(*args, **kw)
                copies = (out.clone(), traj.clone())  # queued right behind the call on the same stream
        s.synchronize()
    finally:
        model.disable_sample_parallel()
    assert_same(copies, want, "caller stream")


@two_gpus
def test_two_devices_weight_edit_reaches_replica():
    model = build(cfg())
    args, kw = inputs(b=3)
    model.enable_sample_parallel(["cuda:0", "cuda:1"])
    try:
        before = model.sample(*args, **kw)
        with torch.no_grad():
            model.transformer.proj_out.weight.mul_(1.5)  # in place: the fingerprint changes
        after = model.sample(*args, **kw)
    finally:
        model.disable_sample_parallel()
    want = model.sample(*args, **kw)
    assert not torch.equal(before[0], after[0])
    assert_same(after, want, "after a weight edit")
