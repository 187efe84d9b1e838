"""GPU: concurrent CFM.sample calls merged into shared engine calls (CFM.enable_batching, f5_tts_b200/batching.py).

  * Small synthetic DiT v1 (rope on every head), DiT v0 (pe_attn_head = 1), UNetT and MMDiT models.  Threads make
    calls that differ in prompt length, text and duration (frame counts on and off the 128-frame bucket), one with
    `edit_mask`, one with `no_ref_audio`, each with its own seed, plus one two-sample exact_varlen call.  With batching
    on, every thread's `out` and trajectory equal the same call made alone with batching off, bit for bit (for the
    exact_varlen call: its valid rows, the only rows exact_varlen defines).
  * The first call's engine run is held until every other call has queued, so the merge is forced: the stats show one
    run for all the compatible calls.  Calls with other steps or another cfg_strength run on their own and still equal
    their solo results; a two-sample faithful call bypasses the batcher; a call with an out-of-range token gets its
    IndexError and the others finish.
  * The socket server with batching on: three concurrent clients get complete streams of the expected lengths, and
    their sampler calls shared engine runs.
"""
import contextlib
import os
import socket
import threading
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import f5_tts_b200 as F5  # noqa: E402
import synthdata as SD  # noqa: E402

DEV = "cuda:0"
CONFIGS = {
    "dit_v1": SD.ArchConfig(backbone="DiT", dim=128, depth=2, heads=2, ff_mult=2, text_num_embeds=50, text_dim=64,
                            text_mask_padding=True, conv_layers=2, pe_attn_head=None),
    "dit_v0": SD.ArchConfig(backbone="DiT", dim=128, depth=2, heads=2, ff_mult=2, text_num_embeds=50, text_dim=64,
                            text_mask_padding=False, conv_layers=2, pe_attn_head=1),
    "unett": SD.ArchConfig(backbone="UNetT", dim=128, depth=4, heads=2, ff_mult=4, text_num_embeds=50, text_dim=None,
                           text_mask_padding=False, conv_layers=0, pe_attn_head=1),
    "mmdit": SD.ArchConfig(backbone="MMDiT", dim=128, depth=3, heads=2, ff_mult=2, text_num_embeds=50, text_dim=None,
                           text_mask_padding=True, conv_layers=0, pe_attn_head=None),
}


def build(cfg: SD.ArchConfig, vocab_char_map=None) -> F5.CFM:
    kw = dict(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
              mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds, text_mask_padding=cfg.text_mask_padding)
    if cfg.backbone != "MMDiT":
        kw.update(text_dim=cfg.text_dim, conv_layers=cfg.conv_layers, pe_attn_head=cfg.pe_attn_head)
    model = F5.CFM(transformer=getattr(F5, cfg.backbone)(**kw), vocab_char_map=vocab_char_map)
    model.load_state_dict(SD.synthetic_state_dict(cfg, seed=1234), strict=True)
    return model.to(DEV)


def calls():
    """name -> (args, kwargs) of one sample() call each.  "hold" goes first; the merged calls share its time grid."""
    g = torch.Generator().manual_seed(5)
    kw = dict(steps=8, cfg_strength=2.0, sway_sampling_coef=-1.0)

    def ids(*shape):
        return torch.randint(0, 50, shape, generator=g).to(DEV)

    def mel(n, b=1):
        return torch.randn(b, n, 100, generator=g).to(DEV)

    text2 = ids(2, 33)
    text2[1, 21:] = -1
    edit = torch.ones(1, 90, dtype=torch.bool)
    edit[0, 30:55] = False
    return {
        "hold": ((mel(40), ids(1, 20), 180), dict(kw, seed=10)),
        "long": ((mel(70), ids(1, 40), 403), dict(kw, seed=11)),
        "bucket": ((mel(50), ids(1, 25), 256), dict(kw, seed=12)),
        "edit": ((mel(90), ids(1, 31), 203), dict(kw, seed=13, edit_mask=edit.to(DEV))),
        "no_ref": ((mel(30), ids(1, 17), 150), dict(kw, seed=14, no_ref_audio=True)),
        "varlen2": ((mel(44, 2), text2, torch.tensor([230, 121]).to(DEV)), dict(kw, seed=15, exact_varlen=True)),
        "steps6": ((mel(35), ids(1, 22), 140), dict(kw, seed=16, steps=6)),
        "cfg15": ((mel(35), ids(1, 22), 160), dict(kw, seed=17, cfg_strength=1.5)),
        "faithful2": ((mel(40, 2), ids(2, 26), torch.tensor([170, 133]).to(DEV)), dict(kw, seed=18)),
        "bad_token": ((mel(30), torch.full((1, 12), 60, device=DEV), 120), dict(kw, seed=19)),
    }


@contextlib.contextmanager
def first_run_held(model, stats, n_calls, sleep_cycles=0):
    """The batcher's first engine run waits (on the host) until `n_calls` calls have reached the batcher, so the calls
    behind it queue; `sleep_cycles` also puts a spin kernel on the batcher's stream ahead of it.  Yields an event set
    when the first run has started."""
    real_run = model.transformer.run
    held = threading.Event()

    def gated_run(*a, **k):
        if not held.is_set():
            if sleep_cycles:
                torch.cuda._sleep(sleep_cycles)
            held.set()
            for _ in range(2000):
                if stats.calls >= n_calls:
                    break
                threading.Event().wait(0.005)
        return real_run(*a, **k)

    model.transformer.run = gated_run
    try:
        yield held
    finally:
        del model.transformer.run


MERGED = ("long", "bucket", "edit", "no_ref", "varlen2")  # one run after "hold"'s
ALONE = ("steps6", "cfg15")  # queued, but each with its own key
BYPASSED = ("faithful2",)


def valid_rows(name, out, traj, args):
    """exact_varlen leaves the rows past a sample's duration undefined: compare the rows it defines."""
    if name != "varlen2":
        return [(out, traj)]
    return [(out[b, :d], traj[:, b, :d]) for b, d in enumerate(args[2].tolist())]


@pytest.mark.parametrize("arch", sorted(CONFIGS))
def test_concurrent_calls_equal_solo_calls(arch):
    model = build(CONFIGS[arch])
    cs = calls()
    solo = {}
    for name, (args, kw) in cs.items():
        if name == "bad_token":
            with pytest.raises(IndexError):
                model.sample(*args, **kw)
            continue
        solo[name] = model.sample(*args, **kw)
    stats = model.enable_batching()
    queued = len(MERGED) + len(ALONE)
    results, errors = {}, {}

    def worker(name):
        args, kw = cs[name]
        try:
            results[name] = model.sample(*args, **kw)
        except Exception as e:  # noqa: BLE001
            errors[name] = e

    try:
        with first_run_held(model, stats, 1 + queued) as held:
            first = threading.Thread(target=worker, args=("hold",))
            first.start()
            assert held.wait(30)
            rest = [threading.Thread(target=worker, args=(n,)) for n in cs if n != "hold"]
            for t in rest:
                t.start()
            for t in [first] + rest:
                t.join(120)
    finally:
        model.disable_batching()
    assert set(errors) == {"bad_token"} and isinstance(errors["bad_token"], IndexError), errors
    print(f"[batching {arch}] {stats}")
    assert stats.calls == 1 + queued and stats.bypassed == len(BYPASSED)
    assert stats.runs == 2 + len(ALONE) < stats.calls
    assert stats.batch_sizes == {1: 1 + len(ALONE), len(MERGED): 1}
    for name, (out, traj) in results.items():
        want_out, want_traj = solo[name]
        assert out.shape == want_out.shape and traj.shape == want_traj.shape
        for (o, t), (wo, wt) in zip(valid_rows(name, out, traj, cs[name][0]),
                                    valid_rows(name, want_out, want_traj, cs[name][0])):
            assert torch.equal(o, wo), f"{arch} {name}: out differs from the solo call"
            assert torch.equal(t, wt), f"{arch} {name}: trajectory differs from the solo call"


def test_lone_call_runs_at_once_and_equals_unbatched():
    """A call that finds the batcher idle runs as it is: one run of one call, the same answer."""
    model = build(CONFIGS["dit_v1"])
    args, kw = calls()["long"]
    want = model.sample(*args, **kw)
    stats = model.enable_batching()
    try:
        got = model.sample(*args, **kw)
    finally:
        model.disable_batching()
    assert stats.calls == 1 and stats.runs == 1 and stats.handoffs == 0
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_caller_sync_does_not_wait_for_a_running_batch():
    """Runs go to the batcher's own stream: while one is busy on the GPU (a spin kernel of about a second ahead of it),
    a synchronisation on another caller's stream, like the `.tolist()` of every sample() prologue, returns at once."""
    model = build(CONFIGS["dit_v1"])
    args, kw = calls()["long"]
    stats = model.enable_batching()
    model.sample(*args, **kw)  # the engine, the batcher's stream, its workspace and graph exist before the timed part
    out = {}
    try:
        with first_run_held(model, stats, 2, sleep_cycles=2_000_000_000) as held:
            th = threading.Thread(target=lambda: out.setdefault("r", model.sample(*args, **kw)))
            th.start()
            assert held.wait(30)
            t0 = time.perf_counter()
            torch.arange(3, device=DEV).sum().tolist()
            waited = time.perf_counter() - t0
            busy = th.is_alive()
            th.join(60)
    finally:
        model.disable_batching()
    print(f"[batching] caller sync took {waited * 1e3:.2f} ms while a run was in flight: {busy}")
    assert busy and waited < 0.3 and "r" in out


def test_socket_server_batch_clients(golden_dir):
    """Three concurrent clients of the streaming server with batching on: each stream is complete (its length equals
    the same request served alone) and the clients' sampler calls shared engine runs."""
    from f5_tts_b200 import infer, socket_server as SS
    from f5_tts_b200.vocoder import Vocos

    vocab, n_vocab = infer.get_tokenizer(os.path.join(golden_dir, "vocab.txt"), "custom")
    cfg = SD.ArchConfig(backbone="DiT", dim=1024, depth=4, heads=16, ff_mult=2, text_num_embeds=n_vocab, text_dim=512,
                        text_mask_padding=False, conv_layers=4, pe_attn_head=1)
    model = build(cfg, vocab_char_map=vocab)
    voc = Vocos()
    voc.load_state_dict(SD.synthetic_vocos_state_dict(), strict=False)
    voc = voc.to(DEV)
    sr = infer.target_sample_rate
    ref = 0.1 * torch.randn(1, 3 * sr, generator=torch.Generator().manual_seed(3))
    proc = SS.TTSStreamingProcessor("F5TTS_Base", "", "", (ref, sr), "A short reference sentence for the voice.",
                                    device=DEV, model_obj=model, vocoder=voc)
    texts = ["Hello there, how are you?", "The weather is nice today.", "Batching merges these calls."]
    assert all(len(t) < proc.min_chars for t in texts)  # one chunk per request, first package or not
    expect = [sum(len(w) for w, _ in proc._stream(proc.plan_chunks(t))) for t in texts]
    stats = model.enable_batching()
    ready, stop = threading.Event(), threading.Event()
    server = threading.Thread(target=SS.start_server, args=("127.0.0.1", 0, proc, ready, stop), daemon=True)
    server.start()
    got = [None] * len(texts)

    def client(i):
        with socket.create_connection(("127.0.0.1", ready.port), timeout=120) as c:
            c.sendall(texts[i].encode("utf-8"))
            got[i] = SS.receive_stream(c)

    try:
        assert ready.wait(10)
        with first_run_held(model, stats, len(texts)):
            threads = [threading.Thread(target=client, args=(i,)) for i in range(len(texts))]
            for t in threads:
                t.start()
            for t in threads:
                t.join(180)
    finally:
        stop.set()
        server.join(5)
        model.disable_batching()
    print(f"[socket batching] lengths {[None if g is None else len(g) for g in got]} expected {expect}; {stats}")
    for g, n in zip(got, expect):
        assert g is not None and len(g) == n and bool(torch.isfinite(torch.from_numpy(g.copy())).all())
    assert stats.calls == len(texts) and stats.runs == 2 and stats.batch_sizes == {1: 1, 2: 1}
