"""GPU: the backbone operator transformer(x, cond, text, time, mask, drop_audio_cond, drop_text, cfg_infer, cache) through
f5_forward, with a time per sample.

  * per-sample times against the CPU oracle forwards (DiT and UNetT at F5TTS_Base / E2TTS_Base widths, a tiny MMDiT):
    B = 3 distinct times, cfg_infer on and off, the joint drop, with and without a mask, rel-L2 <= 3e-3;
  * a batch of distinct times equals each sample evaluated alone at its own time, bit for bit (DiT, UNetT, MMDiT);
  * a uniform time tensor, a scalar time and the one-step f5_sample evaluation the operator ran before agree bit for bit;
  * cache=True over five calls with changing x and time equals cache=False bit for bit (DiT, UNetT, MMDiT);
    clear_cache() lets a new text in; two threads with different texts each get their own answer;
  * graph replay equals eager launches bit for bit, and repeated calls capture nothing new; the first call on a freshly
    built model, which captures its graph, is right too;
  * an Euler loop over forward(cfg_infer=True, cache=True) follows CFM.sample's trajectory, and a torchdiffeq-style RK4
    (3/8 rule) loop over the operator matches the same loop over the CPU oracle operator.
"""
import ctypes as C
import threading

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import f5_tts_b200 as F5  # noqa: E402
import synthdata as SD  # noqa: E402
from f5_tts_b200 import _lib  # noqa: E402
from oracle import f5_oracle as O  # noqa: E402
from oracle import mmdit as OMM  # noqa: E402

DEV = "cuda:0"
TOL = 3e-3  # test_backbone_operator_seam's bound
_models = {}


def configs():
    dit = SD.f5tts_base()
    dit.depth = 4  # F5TTS_Base widths, a short stack: the CPU oracle stays at a few seconds
    unett = SD.e2tts_base()
    unett.depth = 4
    mmdit = SD.ArchConfig(backbone="MMDiT", dim=128, depth=3, heads=2, dim_head=64, ff_mult=2, mel_dim=100,
                          text_num_embeds=50, text_dim=None, conv_layers=0, text_mask_padding=True, pe_attn_head=None,
                          attn_mask_enabled=False)
    return {"dit": dit, "unett": unett, "mmdit": mmdit}


def build(kind: str, wseed: int = 1234):
    key = (kind, wseed)
    if key not in _models:
        _models.clear()
        cfg = configs()[kind]
        if kind == "mmdit":
            tr = F5.MMDiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
                          mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds,
                          text_mask_padding=cfg.text_mask_padding)
        else:
            cls = F5.DiT if kind == "dit" else F5.UNetT
            tr = cls(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
                     mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim,
                     text_mask_padding=cfg.text_mask_padding, conv_layers=cfg.conv_layers,
                     pe_attn_head=cfg.pe_attn_head)
        model = F5.CFM(transformer=tr)
        sd = SD.synthetic_state_dict(cfg, seed=wseed)
        model.load_state_dict(sd, strict=True)
        _models[key] = (model.to(DEV), sd, cfg)
    return _models[key]


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


def inputs(B, N, nt, seed, vocab):
    g = torch.Generator().manual_seed(seed)
    x, cond = torch.randn(B, N, 100, generator=g), torch.randn(B, N, 100, generator=g)
    text = torch.randint(0, vocab, (B, nt), generator=g)
    return x, cond, text


def oracle_forward(kind, sd, cfg, x, cond, text, t, mask, cfg_infer):
    N = x.shape[1]
    if kind == "dit":
        seq = mask.sum(1) if mask is not None else N
        te = (O.text_embedding_dit(sd, cfg, text, seq, False), O.text_embedding_dit(sd, cfg, text, seq, True))
        return O.dit_forward(sd, cfg, x, cond, te, t, mask, cfg_infer)
    if kind == "unett":
        te = (O.text_embedding_unett(sd, cfg, text, N, False), O.text_embedding_unett(sd, cfg, text, N, True))
        return O.unett_forward(sd, cfg, x, cond, te, t, mask, cfg_infer)
    te = (OMM.text_embedding(sd, cfg, text, False), OMM.text_embedding(sd, cfg, text, True))
    return OMM.mmdit_forward(sd, cfg, x, cond, text, te, t, mask, cfg_infer)


def op(model, x, cond, text, t, mask=None, mode="cond", cache=False):
    kw = {"cond": {}, "cfg": {"cfg_infer": True}, "drop": {"drop_audio_cond": True, "drop_text": True}}[mode]
    tt = t.to(DEV) if torch.is_tensor(t) else t
    return model.transformer(x.to(DEV), cond.to(DEV), text.to(DEV), tt, mask=None if mask is None else mask.to(DEV),
                             cache=cache, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# per-sample times against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["dit", "unett", "mmdit"])
@pytest.mark.parametrize("masked", [False, True])
def test_per_sample_times_vs_oracle(kind, masked):
    model, sd, cfg = build(kind)
    B, N = 3, 96
    x, cond, text = inputs(B, N, 40 if kind != "mmdit" else 30, 7, cfg.text_num_embeds)
    text[1, 25:] = -1
    t = torch.tensor([0.05, 0.47, 0.93])
    mask = O.lens_to_mask(torch.tensor([96, 70, 81])) if masked else None
    ref_cfg = oracle_forward(kind, sd, cfg, x, cond, text, t, mask, True)
    ref_cond = oracle_forward(kind, sd, cfg, x, cond, text, t, mask, False)
    for mode, ref in (("cfg", ref_cfg), ("cond", ref_cond), ("drop", ref_cfg[B:])):
        got = op(model, x, cond, text, t, mask, mode)
        r = rel(got, ref)
        print(f"[forward {kind} masked={masked} {mode}] rel-L2 {r:.3e}")
        assert got.shape == ref.shape and r <= TOL


# ---------------------------------------------------------------------------------------------------------------------
# bit-for-bit properties
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["dit", "unett", "mmdit"])
def test_batch_equals_single_calls(kind):
    model, _, cfg = build(kind)
    B, N = 3, 150
    x, cond, text = inputs(B, N, 50, 8, cfg.text_num_embeds)
    t = torch.tensor([0.12, 0.55, 0.81])
    for mode in ("cfg", "cond", "drop"):
        got = op(model, x, cond, text, t, None, mode)
        for b in range(B):
            one = op(model, x[b:b + 1], cond[b:b + 1], text[b:b + 1], t[b:b + 1], None, mode)
            rows = [b, B + b] if mode == "cfg" else [b]
            assert torch.equal(got[rows], one), (kind, mode, b)


@pytest.mark.parametrize("kind", ["dit", "unett", "mmdit"])
def test_uniform_time_matches_scalar_and_sample_evaluation(kind):
    """A [b] tensor of one time, a float and a 0-d tensor agree bit for bit, and equal the raw output of a one-step
    f5_sample evaluation at that time (the operator's previous implementation)."""
    model, _, cfg = build(kind)
    B, N, t0 = 2, 128, 0.3125
    x, cond, text = inputs(B, N, 40, 9, cfg.text_num_embeds)
    mask = O.lens_to_mask(torch.tensor([128, 100]))
    for m in (None, mask):
        for mode in ("cfg", "cond", "drop"):
            a = op(model, x, cond, text, torch.full((B,), t0), m, mode)
            assert torch.equal(a, op(model, x, cond, text, t0, m, mode))
            assert torch.equal(a, op(model, x, cond, text, torch.tensor(t0), m, mode))
            assert torch.equal(a, op(model, x, cond, text, torch.tensor([t0]), m, mode))
            packed = mode != "cond"
            v = torch.empty((2 * B if packed else B, N, 100), device=DEV)
            dur = None if m is None else m.sum(1).to(torch.int32).to(DEV)
            model.transformer._run_local(x.to(DEV).clone(), cond.to(DEV), text.to(DEV), [t0, t0 + 1.0], dur,
                                         1.0 if packed else 0.0, None, v, use_graph=False)
            ref = v[B:] if mode == "drop" else v
            assert torch.equal(a, ref), (kind, m is None, mode)


@pytest.mark.parametrize("kind", ["dit", "unett", "mmdit"])
def test_cache_equals_no_cache_and_clear_cache(kind):
    model, _, cfg = build(kind)
    tr = model.transformer
    B, N = 2, 120
    x, cond, text = inputs(B, N, 40, 10, cfg.text_num_embeds)
    g = torch.Generator().manual_seed(3)
    tr.clear_cache()
    for k in range(5):
        xk = x + 0.1 * k * torch.randn(x.shape, generator=g)
        tk = torch.rand(B, generator=g)
        a = op(model, xk, cond, text, tk, None, "cfg", cache=True)
        b = op(model, xk, cond, text, tk, None, "cfg", cache=False)
        assert torch.equal(a, b), k
    # the reference's cache: a new text at the same shapes reuses the first text's embeddings until clear_cache()
    _, _, text2 = inputs(B, N, 40, 11, cfg.text_num_embeds)
    t = torch.tensor([0.2, 0.6])
    old = op(model, x, cond, text, t, None, "cfg")
    new = op(model, x, cond, text2, t, None, "cfg")
    assert not torch.equal(old, new)
    assert torch.equal(op(model, x, cond, text2, t, None, "cfg", cache=True), old)
    assert tr.clear_cache() is None
    assert torch.equal(op(model, x, cond, text2, t, None, "cfg", cache=True), new)
    # another mode or shape recomputes
    assert torch.equal(op(model, x, cond, text, t, None, "cond", cache=True), op(model, x, cond, text, t, None, "cond"))
    tr.clear_cache()


def test_cache_is_per_thread():
    model, _, cfg = build("dit")
    B, N = 1, 100
    x, cond, text_a = inputs(B, N, 40, 12, cfg.text_num_embeds)
    _, _, text_b = inputs(B, N, 40, 13, cfg.text_num_embeds)
    t = torch.tensor([0.4])
    want = {"a": op(model, x, cond, text_a, t, None, "cfg"), "b": op(model, x, cond, text_b, t, None, "cfg")}
    got, errors = {}, []
    barrier = threading.Barrier(2)

    def worker(name, text):
        try:
            torch.cuda.set_device(0)
            op(model, x, cond, text, t, None, "cfg", cache=True)  # fills this thread's cache
            barrier.wait()
            outs = [op(model, x + 0.0, cond, text, t, None, "cfg", cache=True) for _ in range(3)]
            torch.cuda.current_stream().synchronize()
            got[name] = outs
            model.transformer.clear_cache()
        except Exception as e:  # reported below
            errors.append(e)
            barrier.abort()

    th = [threading.Thread(target=worker, args=("a", text_a)), threading.Thread(target=worker, args=("b", text_b))]
    for h in th:
        h.start()
    for h in th:
        h.join()
    assert not errors, errors
    for name in ("a", "b"):
        for o in got[name]:
            assert torch.equal(o, want[name]), name


def abi_forward(model, ws, x, cond, text, t, mode, use_graph, reuse_text=0):
    handle = model.transformer.engine()["handle"]
    B, N, _ = x.shape
    v = torch.empty((2 * B if mode == _lib.FORWARD_CFG else B, N, 100), device=DEV)
    a = _lib.ForwardArgs()
    a.B, a.N, a.nt = B, N, text.shape[1]
    a.x, a.step_cond, a.text, a.time = x.data_ptr(), cond.data_ptr(), text.data_ptr(), t.data_ptr()
    a.duration = None
    a.mode, a.v_out, a.use_graph, a.reuse_text = mode, v.data_ptr(), use_graph, reuse_text
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(_lib.lib().f5_forward(handle, C.byref(a), ws.data_ptr(), ws.numel(), stream), "f5_forward")
    return v


@pytest.mark.parametrize("kind", ["dit", "unett", "mmdit"])
def test_graph_replay_equals_eager_and_captures_once(kind):
    """Graph calls on one workspace against eager calls on another, with new x and times every call: the capturing
    call and each replay equal the eager launches bit for bit."""
    model, _, cfg = build(kind)
    L = _lib.lib()
    handle = model.transformer.engine()["handle"]
    B, N = 2, 130
    x, cond, text = inputs(B, N, 45, 14, cfg.text_num_embeds)
    x, cond, text = x.to(DEV), cond.to(DEV), text.to(DEV)
    need = L.f5_forward_workspace_bytes(handle, B, N, 45, _lib.FORWARD_CFG)
    ws_eager = torch.empty(need, dtype=torch.uint8, device=DEV)
    ws_graph = torch.empty(need, dtype=torch.uint8, device=DEV)
    g = torch.Generator().manual_seed(5)
    graphs = None
    for k in range(4):
        t = torch.rand(B, generator=g).to(DEV)
        xk = x + 0.05 * k
        eager = abi_forward(model, ws_eager, xk, cond, text, t, _lib.FORWARD_CFG, 0)
        replay = abi_forward(model, ws_graph, xk, cond, text, t, _lib.FORWARD_CFG, 1, reuse_text=int(k > 0))
        assert torch.equal(eager, replay), k
        if graphs is None:
            graphs = L.f5_engine_graph_count(handle)
        assert L.f5_engine_graph_count(handle) == graphs  # new x and times replay the graph captured at k = 0
    # operator calls at one shape: one capture, then replays
    model.transformer.clear_cache()
    before = L.f5_engine_graph_count(handle)
    for k in range(3):
        op(model, x.cpu(), cond.cpu(), text.cpu(), torch.rand(B, generator=g), None, "cfg", cache=True)
        assert L.f5_engine_graph_count(handle) == min(before + 1, 16)


def test_first_call_on_a_fresh_model():
    """A small DiT (dim 128, two text blocks, 60 frames), new for the test: the first call, which captures the graph,
    and every later call with a new time equal the one-step f5_sample evaluation, with and without the cache."""
    cfg = SD.ArchConfig(dim=128, depth=2, heads=2, ff_mult=2, text_num_embeds=50, text_dim=64, text_mask_padding=True,
                        conv_layers=2, pe_attn_head=None)
    model = F5.CFM(transformer=F5.DiT(dim=128, depth=2, heads=2, ff_mult=2, text_num_embeds=50, text_dim=64,
                                      text_mask_padding=True, conv_layers=2, pe_attn_head=None))
    model.load_state_dict(SD.synthetic_state_dict(cfg, seed=1234), strict=True)
    model = model.to(DEV)
    tr = model.transformer
    g = torch.Generator().manual_seed(18)
    x = torch.randn(1, 60, 100, generator=g).to(DEV)
    cond = torch.zeros_like(x)
    text = torch.randint(0, 50, (1, 20), generator=g).to(DEV)
    for cache in (False, True):
        for t0 in (0.3, 0.3, 0.7, 0.1):
            got = tr(x, cond, text, torch.tensor([t0], device=DEV), cfg_infer=True, cache=cache)
            want = torch.empty(2, 60, 100, device=DEV)
            tr._run_local(x.clone(), cond, text, [t0, t0 + 1.0], None, 1.0, None, want, use_graph=False)
            assert torch.equal(got, want), (cache, t0)
    tr.clear_cache()


def test_reuse_text_needs_held_embeddings():
    model, _, cfg = build("dit")
    L = _lib.lib()
    handle = model.transformer.engine()["handle"]
    B, N = 1, 100
    x, cond, text = (a.to(DEV) for a in inputs(B, N, 40, 15, cfg.text_num_embeds))
    ws = torch.empty(L.f5_forward_workspace_bytes(handle, B, N, 40, _lib.FORWARD_CFG), dtype=torch.uint8, device=DEV)
    t = torch.tensor([0.5], device=DEV)
    with pytest.raises(_lib.F5LibraryError, match="reuse_text"):
        abi_forward(model, ws, x, cond, text, t, _lib.FORWARD_CFG, 1, reuse_text=1)
    abi_forward(model, ws, x, cond, text, t, _lib.FORWARD_CFG, 1)
    abi_forward(model, ws, x, cond, text, t, _lib.FORWARD_CFG, 1, reuse_text=1)
    with pytest.raises(_lib.F5LibraryError, match="reuse_text"):  # another mode
        abi_forward(model, ws, x, cond, text, t, _lib.FORWARD_COND, 1, reuse_text=1)


# ---------------------------------------------------------------------------------------------------------------------
# samplers over the operator
# ---------------------------------------------------------------------------------------------------------------------
def test_euler_loop_follows_sample():
    model, _, cfg = build("dit")
    seen = {}
    real_run = model.transformer.run

    def spy(y, step_cond, text, t_grid, duration, cfg_strength, **kw):
        seen.update(y0=y.clone(), step_cond=step_cond.clone(), text=text.clone(), t=list(t_grid), duration=duration,
                    cfg=float(cfg_strength))
        out = real_run(y, step_cond, text, t_grid, duration, cfg_strength, **kw)
        seen["traj"] = kw["trajectory"].clone()
        return out

    model.transformer.run = spy
    try:
        g = torch.Generator().manual_seed(16)
        cond = torch.randn(1, 60, 100, generator=g)
        text = torch.randint(0, cfg.text_num_embeds, (1, 40), generator=g)
        model.sample(cond.to(DEV), text.to(DEV), 300, steps=16, cfg_strength=2.0, sway_sampling_coef=-1.0, seed=0)
    finally:
        del model.transformer.run
    y, B = seen["y0"], seen["y0"].shape[0]
    t = torch.tensor(seen["t"], dtype=torch.float32)
    tr = model.transformer
    tr.clear_cache()
    worst = 0.0
    mask = None
    if seen["duration"] is not None:
        mask = torch.arange(y.shape[1], device=DEV)[None, :] < seen["duration"].to(DEV)[:, None]
    for k in range(len(t) - 1):
        v = tr(y, seen["step_cond"], seen["text"], t[k].to(DEV), mask=mask, cfg_infer=True, cache=True)
        pred, null = v[:B], v[B:]
        y = y + (t[k + 1] - t[k]).to(DEV) * (pred + (pred - null) * seen["cfg"])
        worst = max(worst, rel(y, seen["traj"][k + 1]))
    tr.clear_cache()
    print(f"[euler loop] worst rel-L2 against CFM.sample's trajectory over {len(t) - 1} steps: {worst:.3e}")
    assert worst <= 1e-3


def rk4_38(f, y, t):
    """torchdiffeq's fixed-grid rk4 (rk4_alt_step_func, the 3/8 rule) over the grid t"""
    for k in range(len(t) - 1):
        t0, dt = t[k], t[k + 1] - t[k]
        k1 = f(t0, y)
        k2 = f(t0 + dt / 3, y + dt * k1 / 3)
        k3 = f(t0 + dt * 2 / 3, y + dt * (k2 - k1 / 3))
        k4 = f(t[k + 1], y + dt * (k1 - k2 + k3))
        y = y + (k1 + 3 * (k2 + k3) + k4) * dt * 0.125
    return y


@pytest.mark.parametrize("kind", ["dit", "mmdit"])
def test_rk4_loop_vs_oracle(kind):
    model, sd, cfg = build(kind)
    B, N, cfg_s = 2, 110, 2.0
    x0, cond, text = inputs(B, N, 40, 17, cfg.text_num_embeds)
    t = torch.linspace(0, 1, 9)  # 8 steps, 32 evaluations

    def f_gpu(tk, y):
        v = model.transformer(y, cond.to(DEV), text.to(DEV), torch.full((B,), float(tk)).to(DEV), cfg_infer=True,
                              cache=True)
        return v[:B] + (v[:B] - v[B:]) * cfg_s

    def f_ref(tk, y):
        v = oracle_forward(kind, sd, cfg, y, cond, text, torch.full((B,), float(tk)), None, True)
        return v[:B] + (v[:B] - v[B:]) * cfg_s

    model.transformer.clear_cache()
    got = rk4_38(f_gpu, x0.to(DEV), t)
    model.transformer.clear_cache()
    ref = rk4_38(f_ref, x0, t)
    r = rel(got, ref)
    print(f"[rk4 {kind}] final state rel-L2 {r:.3e}")
    assert r <= 5e-3
