"""GPU: one CFM.sample call with its conditional and unconditional CFG halves on two engines (CFM.enable_cfg_parallel,
f5_sample_cfg_split).

  * Loopback (both halves on cuda:0, two workspaces and two streams: the same code path as two devices).  The split
    call's final mel and full trajectory equal the unsplit call bit for bit for DiT at B = 1; B = 3 faithful padded,
    with attn_mask_enabled and with exact_varlen; midpoint; UNetT with concat and add skips; MMDiT; dim_head 128; eager
    against graph; repeated calls; concurrent threads; merged runs of enable_batching; infer_batch_process and
    F5TTS.infer end to end.  Through the C ABI directly, both sides end with the same y.  Enabling again keeps the peer
    and repeated calls reuse its workspace; a peer with its own weight copy on the same GPU (the replica path of a
    second device) gives the same answer and follows weight edits.
  * Two devices (skipped with fewer than two): the same equalities against the single-device call, y equal on both
    devices, the caller's stream sees finished results without a synchronise, and a weight edit on the primary reaches
    the replica.
"""
import ctypes as C
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
from f5_tts_b200 import _lib, cfg_parallel, infer  # noqa: E402

DEV = "cuda:0"
TWO_GPUS = torch.cuda.device_count() >= 2
PEER = "cuda:1" if TWO_GPUS else DEV


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


def inputs(b=1, seed=5, device=DEV, pad_text=False):
    """(args, kwargs) of one sample() call: b samples of different durations (b > 1), seeded noise."""
    g = torch.Generator().manual_seed(seed)
    cond = torch.randn(b, 40, 100, generator=g).to(device)
    text = torch.randint(0, 50, (b, 24), generator=g)
    if pad_text:
        text[-1, 15:] = -1
    duration = 180 if b == 1 else torch.tensor([180, 133, 101][:b])
    if b > 1:
        duration = duration.to(device)
    return (cond, text.to(device), duration), dict(steps=8, cfg_strength=2.0, sway_sampling_coef=-1.0, seed=seed)


def split_and_solo(model, args, kw, peer=PEER):
    want = model.sample(*args, **kw)
    model.enable_cfg_parallel(peer)
    try:
        got = model.sample(*args, **kw)
    finally:
        model.disable_cfg_parallel()
    return got, want


def assert_same(got, want, what, lengths=None):
    """Bit equality of final mel and trajectory.  `lengths`: compare each sample's first lengths[b] frames only — with
    attn_mask_enabled or exact_varlen the engine skips tiles that hold only padding, so the frames past a sample's
    duration keep whatever the workspace held, in the unsplit call as in the split one; the modes define only the valid
    frames."""
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


# ---------------------------------------------------------------------------------------------------------------------
# loopback
# ---------------------------------------------------------------------------------------------------------------------
def test_dit_b1():
    model = build(cfg())
    got, want = split_and_solo(model, *inputs(), peer=DEV)
    assert_same(got, want, "DiT B=1")


@pytest.mark.parametrize("mode", ["faithful", "attn_mask", "exact_varlen"])
def test_dit_b3(mode):
    model = build(cfg(attn_mask_enabled=mode == "attn_mask", text_mask_padding=False, pe_attn_head=1))
    args, kw = inputs(b=3)
    got, want = split_and_solo(model, args, dict(kw, exact_varlen=mode == "exact_varlen"), peer=DEV)
    assert_same(got, want, f"DiT B=3 {mode}", lengths=None if mode == "faithful" else args[2].tolist())


def test_midpoint():
    model = build(cfg(), method="midpoint")
    args, kw = inputs(b=2)
    got, want = split_and_solo(model, args, kw, peer=DEV)
    assert_same(got, want, "midpoint")


@pytest.mark.parametrize("skip", ["concat", "add"])
def test_unett(skip):
    model = build(cfg("UNetT", skip_connect_type=skip))
    args, kw = inputs(b=2)
    got, want = split_and_solo(model, args, kw, peer=DEV)
    assert_same(got, want, f"UNetT {skip}")


@pytest.mark.parametrize("b", [1, 2])
def test_mmdit(b):
    model = build(cfg("MMDiT", attn_mask_enabled=b == 2))
    got, want = split_and_solo(model, *inputs(b=b, pad_text=b == 2), peer=DEV)
    assert_same(got, want, f"MMDiT B={b}")


@pytest.mark.parametrize("backbone", ["DiT", "UNetT"])
def test_dim_head_128(backbone):
    model = build(cfg(backbone, dim=256, heads=2, dim_head=128))
    got, want = split_and_solo(model, *inputs(b=2), peer=DEV)
    assert_same(got, want, f"{backbone} dim_head 128")


def test_eager_graph_and_repeats():
    """Split eager, split graph (twice: capture, then replay) and unsplit graph: one answer."""
    model = build(cfg())
    args, kw = inputs(b=2)
    want = model.sample(*args, **kw)
    model.enable_cfg_parallel(DEV)
    try:
        model.use_cuda_graph = False
        eager = model.sample(*args, **kw)
        model.use_cuda_graph = True
        graph = [model.sample(*args, **kw) for _ in range(3)]
    finally:
        model.disable_cfg_parallel()
    assert_same(eager, want, "eager split")
    for g in graph:
        assert_same(g, want, "graph split")


def test_steady_state_calls_stay_warm():
    """Enabling again keeps the peer; repeated calls reuse one peer workspace (so its captured graph) and copy no
    weights."""
    model = build(cfg())
    args, kw = inputs(b=2)
    want = model.sample(*args, **kw)
    peer = model.enable_cfg_parallel(DEV)
    try:
        got = [model.sample(*args, **kw)]
        ws = [w.data_ptr() for w in peer._ws_free]
        for _ in range(3):
            assert model.enable_cfg_parallel(DEV) is peer
            got.append(model.sample(*args, **kw))
        assert [w.data_ptr() for w in peer._ws_free] == ws and len(ws) == 1 and peer.replications == 0
    finally:
        model.disable_cfg_parallel()
    for g in got:
        assert_same(g, want, "steady state")


def test_weight_copy_on_one_gpu_follows_edits():
    """A peer with its own weight copy on the same GPU: two engines over two copies of the packed weights, the path a
    second device takes (replication, a second engine, its graph cache).  Equal to the unsplit call, and a weight edit
    on the primary is copied again before the next split call."""
    model = build(cfg())
    args, kw = inputs(b=2)
    want = model.sample(*args, **kw)
    peer = cfg_parallel.CfgPeer(DEV, copy_weights=True)
    model.transformer.cfg_peer = peer
    try:
        got = model.sample(*args, **kw)
        assert peer.replications == 1 and peer._state["handle"].value != model.transformer.engine()["handle"].value
        with torch.no_grad():
            model.transformer.proj_out.weight.mul_(1.5)  # in place: the fingerprint changes
        edited = model.sample(*args, **kw)
        assert peer.replications == 2
    finally:
        model.disable_cfg_parallel()
    want_edited = model.sample(*args, **kw)
    assert_same(got, want, "weight copy")
    assert not torch.equal(edited[0], want[0])
    assert_same(edited, want_edited, "weight copy after an edit")


def test_cfg_strength_zero_and_forward_stay_local():
    """No packed half to split off: the call runs unsplit and returns what it returns without the peer."""
    model = build(cfg())
    args, kw = inputs()
    kw = dict(kw, cfg_strength=0.0)
    got, want = split_and_solo(model, args, kw, peer=DEV)
    assert_same(got, want, "cfg 0")
    bb = model.transformer
    x = torch.randn(1, 60, 100, device=DEV)
    text = torch.randint(0, 50, (1, 20), device=DEV)
    want_v = bb(x, torch.zeros_like(x), text, torch.tensor([0.3], device=DEV), cfg_infer=True)
    model.enable_cfg_parallel(DEV)
    try:
        got_v = bb(x, torch.zeros_like(x), text, torch.tensor([0.3], device=DEV), cfg_infer=True)
    finally:
        model.disable_cfg_parallel()
    assert torch.equal(got_v, want_v)


def test_concurrent_threads():
    model = build(cfg())
    cases = [inputs(b=1, seed=s) for s in (21, 22, 23)]
    want = [model.sample(*a, **k) for a, k in cases]
    model.enable_cfg_parallel(DEV)
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
        model.disable_cfg_parallel()
    assert not errors, errors
    for i, w in enumerate(want):
        for got in results[i]:
            assert_same(got, w, f"thread {i}")


def test_with_batching():
    """enable_batching's merged runs go through the backbone's run: they split too, and each caller gets its solo answer."""
    model = build(cfg())
    cases = [inputs(b=1, seed=s) for s in (31, 32, 33)]
    want = [model.sample(*a, **k) for a, k in cases]
    stats = model.enable_batching()
    model.enable_cfg_parallel(DEV)
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
        model.disable_cfg_parallel()
        model.disable_batching()
    assert not errors, errors
    assert stats.calls == len(cases)
    for i, w in enumerate(want):
        assert_same(results[i], w, f"batched call {i}")


def split_abi(model, args, kw, peer):
    """f5_sample_cfg_split called directly: (y of side 0, y of side 1, trajectory) after a whole call."""
    bb = model.transformer
    cond, text, duration = args
    out, traj = model.sample(*args, **kw)  # unsplit reference: shapes, grid
    B, N = traj.shape[1], traj.shape[2]
    g = torch.Generator().manual_seed(9)
    y0 = torch.randn(B, N, 100, generator=g).to(DEV)
    sc = torch.randn(B, N, 100, generator=g).to(DEV)
    text = text.to(torch.int64).contiguous()
    dur = duration.to(torch.int32).contiguous() if torch.is_tensor(duration) else None
    t = [k / 8 for k in range(9)]
    st0 = bb.engine()
    peer_obj = cfg_parallel.CfgPeer(peer)
    st1 = peer_obj.engine(bb, st0, torch.device(DEV))
    y1 = y0.to(peer, copy=True)
    y_a = y0.clone()
    traj_a = torch.empty((9, B, N, 100), device=DEV)
    L = _lib.lib()
    need = L.f5_sample_cfg_split_workspace_bytes(st0["handle"], B, N, text.shape[1], 8)
    ws0 = torch.empty(need, dtype=torch.uint8, device=DEV)
    ws1 = torch.empty(need, dtype=torch.uint8, device=peer)
    s0, s1 = torch.cuda.Stream(DEV), torch.cuda.Stream(peer)
    torch.cuda.synchronize(DEV)
    torch.cuda.synchronize(peer)
    tg = (C.c_float * 9)(*t)
    a0 = _lib.sample_args(y_a, sc, text, dur, tg, 8, 2.0, traj_a, True, False, "euler")
    a1 = _lib.sample_args(y1, sc.to(peer), text.to(peer), None if dur is None else dur.to(peer), tg, 8, 2.0, None,
                          True, False, "euler")
    torch.cuda.synchronize(peer)
    _lib.check(L.f5_sample_cfg_split(st0["handle"], C.byref(a0), ws0.data_ptr(), need, s0.cuda_stream, st1["handle"],
                                     C.byref(a1), ws1.data_ptr(), need, s1.cuda_stream), "f5_sample_cfg_split")
    s0.synchronize()
    s1.synchronize()
    # the same problem unsplit
    y_b = y0.clone()
    traj_b = torch.empty_like(traj_a)
    bb.run(y_b, sc, text, t, dur, 2.0, trajectory=traj_b)
    torch.cuda.synchronize(DEV)
    return y_a, y1.to(DEV), traj_a, y_b, traj_b


def test_abi_both_sides_end_with_the_same_y():
    model = build(cfg())
    y_a, y1, traj_a, y_b, traj_b = split_abi(model, *inputs(b=2), DEV)
    assert torch.equal(y_a, y1) and torch.equal(y_a, y_b) and torch.equal(traj_a, traj_b)
    assert torch.equal(traj_a[-1], y_a)


def test_abi_rejects_mismatched_sides():
    model = build(cfg())
    bb = model.transformer
    st = bb.engine()
    y = torch.zeros(1, 64, 100, device=DEV)
    sc = torch.zeros_like(y)
    text = torch.zeros(1, 10, dtype=torch.int64, device=DEV)
    tg = (C.c_float * 3)(0.0, 0.5, 1.0)
    L = _lib.lib()
    need = L.f5_sample_cfg_split_workspace_bytes(st["handle"], 1, 64, 10, 2)
    ws0 = torch.empty(need, dtype=torch.uint8, device=DEV)
    ws1 = torch.empty(need, dtype=torch.uint8, device=DEV)
    s0, s1 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
    y1 = y.clone()

    def call(a0, a1, st1=s1):
        return L.f5_sample_cfg_split(st["handle"], C.byref(a0), ws0.data_ptr(), need, s0.cuda_stream, st["handle"],
                                     C.byref(a1), ws1.data_ptr(), need, st1.cuda_stream)

    args = lambda yy, steps=2, cfg_s=2.0: _lib.sample_args(yy, sc, text, None, tg, steps, cfg_s, None, True,  # noqa
                                                           False, "euler")
    assert call(args(y), args(y1, cfg_s=0.0)) != 0  # the two sides disagree
    assert call(args(y, cfg_s=0.0), args(y1, cfg_s=0.0)) != 0  # no unconditional half
    assert call(args(y), args(y)) != 0  # one y for both sides
    assert call(args(y), args(y1), st1=s0) != 0  # one stream for both sides
    torch.cuda.synchronize()


def test_infer_batch_process_and_f5tts_infer(tmp_path, golden_dir):
    """A chunked request through infer_batch_process, and F5TTS(cfg_parallel_device=...).infer, equal their unsplit runs."""
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
                      cfg_parallel_device=PEER)
    assert split.ema_model.transformer.cfg_peer is not None and plain.ema_model.transformer.cfg_peer is None

    audio, sr = infer._load_wav(ref)
    chunks = ["I don't really care what you call me.", "Short one.", "And I will be here long after you are gone."]
    outs = []
    for t in (plain, split):
        torch.manual_seed(77)
        outs.append(next(infer.infer_batch_process((audio, sr), ref_text + " ", chunks, t.ema_model, t.vocoder,
                                                   nfe_step=6, device=DEV)))
    (w1, _, s1), (w2, _, s2) = outs
    assert np.isfinite(w1).all() and np.array_equal(w1, w2) and np.array_equal(s1, s2)

    outs = [t.infer(ref, ref_text, "I don't really care what you call me.", nfe_step=6, seed=5,
                    show_info=lambda *_: None) for t in (plain, split)]
    (w1, _, s1), (w2, _, s2) = outs
    assert np.isfinite(w1).all() and np.array_equal(w1, w2) and np.array_equal(s1, s2)


# ---------------------------------------------------------------------------------------------------------------------
# two devices
# ---------------------------------------------------------------------------------------------------------------------
two_gpus = pytest.mark.skipif(not TWO_GPUS, reason="needs two CUDA devices (the peer half runs on cuda:1)")


@two_gpus
@pytest.mark.parametrize("case", ["dit_b1", "dit_b3_varlen", "unett_add", "mmdit_b2"])
def test_two_devices_equal_single_device(case):
    c = {"dit_b1": cfg(), "dit_b3_varlen": cfg(), "unett_add": cfg("UNetT", skip_connect_type="add"),
         "mmdit_b2": cfg("MMDiT")}[case]
    model = build(c)
    args, kw = inputs(b={"dit_b1": 1, "dit_b3_varlen": 3}.get(case, 2), pad_text=case == "mmdit_b2")
    if case == "dit_b3_varlen":
        kw = dict(kw, exact_varlen=True)
    got, want = split_and_solo(model, args, kw, peer="cuda:1")
    assert_same(got, want, case, lengths=args[2].tolist() if case == "dit_b3_varlen" else None)


@two_gpus
def test_two_devices_y_equal_on_both():
    model = build(cfg())
    y_a, y1, traj_a, y_b, traj_b = split_abi(model, *inputs(b=2), "cuda:1")
    assert torch.equal(y_a, y1) and torch.equal(y_a, y_b) and torch.equal(traj_a, traj_b)


@two_gpus
def test_two_devices_caller_stream_sees_results():
    """Work queued on the caller's stream after sample() reads the finished result: no synchronise in between."""
    model = build(cfg())
    args, kw = inputs(b=2)
    want = model.sample(*args, **kw)
    model.enable_cfg_parallel("cuda:1")
    s = torch.cuda.Stream(DEV)
    try:
        with torch.cuda.stream(s):
            for _ in range(3):
                out, traj = model.sample(*args, **kw)
                copies = (out.clone(), traj.clone())  # queued right behind the call on the same stream
        s.synchronize()
    finally:
        model.disable_cfg_parallel()
    assert_same(copies, want, "caller stream")


@two_gpus
def test_two_devices_weight_edit_reaches_replica():
    model = build(cfg())
    args, kw = inputs()
    model.enable_cfg_parallel("cuda:1")
    try:
        before = model.sample(*args, **kw)
        with torch.no_grad():
            model.transformer.proj_out.weight.mul_(1.5)  # in place: the fingerprint changes
        after = model.sample(*args, **kw)
    finally:
        model.disable_cfg_parallel()
    want = model.sample(*args, **kw)
    assert not torch.equal(before[0], after[0])
    assert_same(after, want, "after a weight edit")
