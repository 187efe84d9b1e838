"""GPU end-to-end parity of CFM.sample (C ABI engine) against
  (a) golden vectors produced by the UNMODIFIED reference in fp32 (tests/golden/*.npz), and
  (b) the CPU oracle on fresh seeded inputs (masked / attn-mask / UNetT variants),
plus size-independent properties at the BASELINE.json sizes (N = 938, NFE 32).

Tolerance (SURVEY.md §8c, BASELINE.md §2): final-mel rel-L2 <= 5e-3 vs the fp32 reference with identical injected y0
(fp16 tensor-core operands, fp32 accumulation / residual / ODE state).  The reference's own fp16 path sits at 1.5e-3.
"""
import ast
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import f5_tts_b200 as F5  # noqa: E402
from oracle import f5_oracle as O  # noqa: E402
from oracle import step_increment as SI  # noqa: E402

DEV = "cuda:0"
TOL = 5e-3
_models = {}


def cfg_from_repr(s: str) -> O.ArchConfig:
    body = s[s.index("(") + 1: s.rindex(")")]
    return O.ArchConfig(**{k: ast.literal_eval(v) for k, v in (p.split("=") for p in body.split(", "))})


def build(cfg: O.ArchConfig, wseed: int):
    key = (repr(cfg), wseed)
    if key not in _models:
        _models.clear()  # keep one ~1.3 GB model resident at a time
        cls = F5.DiT if cfg.backbone == "DiT" else F5.UNetT
        kw = dict(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
                  mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim,
                  text_mask_padding=cfg.text_mask_padding, conv_layers=cfg.conv_layers, pe_attn_head=cfg.pe_attn_head,
                  attn_mask_enabled=cfg.attn_mask_enabled)
        model = F5.CFM(transformer=cls(**kw))
        sd = O.synthetic_state_dict(cfg, seed=wseed)
        model.load_state_dict(sd, strict=True)
        _models[key] = (model.to(DEV), sd)
    return _models[key]


def rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm())


@pytest.mark.parametrize("name", ["f5base_b1_n192", "f5base_b2_varlen", "f5v1base_b1_n128", "e2base_b1_n128"])
def test_sample_vs_reference_golden(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    cfg = cfg_from_repr(str(z["cfg"]))
    model, _ = build(cfg, int(z["wseed"]))
    dur = z["duration"]
    duration = int(dur) if dur.ndim == 0 else torch.from_numpy(dur).long().to(DEV)
    lens = torch.from_numpy(z["lens"]).long().to(DEV) if z["lens"].size else None
    out, traj = model.sample(cond=torch.from_numpy(z["cond"]).to(DEV), text=torch.from_numpy(z["text"]).to(DEV),
                             duration=duration, lens=lens, steps=int(z["steps"]), cfg_strength=float(z["cfg_strength"]),
                             sway_sampling_coef=float(z["sway"]), seed=int(z["seed"]),
                             y0=torch.from_numpy(z["y0"]).to(DEV))
    SI.check(traj[1], z["y0"], z["traj_1"], z["duration"] if cfg.attn_mask_enabled else None, name)
    r1, rN = rel(traj[1], torch.from_numpy(z["traj_1"])), rel(out, torch.from_numpy(z["out"]))
    print(f"[{name}] step-1 rel-L2 {r1:.3e}  final rel-L2 {rN:.3e}")
    assert traj.shape[0] == int(z["steps"]) + 1 and out.shape == z["out"].shape
    assert r1 <= TOL and rN <= TOL


@pytest.mark.parametrize("variant", ["mask_faithful", "attn_mask", "no_cfg", "wave_epss"])
def test_sample_vs_oracle(variant):
    cfg = O.f5tts_base()
    if variant == "attn_mask":
        cfg.attn_mask_enabled = True
    model, sd = build(cfg, 1234)
    g = torch.Generator().manual_seed(42)
    kw = dict(steps=3, cfg_strength=2.0, sway_sampling_coef=-1.0, seed=7)
    if variant in ("mask_faithful", "attn_mask"):
        cond = torch.randn(3, 40, 100, generator=g)
        text = torch.randint(0, 2545, (3, 30), generator=g)
        text[1, 20:] = -1
        args = (cond, text, torch.tensor([150, 97, 131]))
        kw["lens"] = torch.tensor([40, 25, 33])
    elif variant == "no_cfg":
        args = (torch.randn(1, 30, 100, generator=g), torch.randint(0, 2545, (1, 25), generator=g), 130)
        kw["cfg_strength"] = 0.0
        kw["sway_sampling_coef"] = None
    else:  # raw wave in (mel kernel) + EPSS grid (16 steps would be slow on the CPU oracle: use 5)
        args = (0.1 * torch.randn(1, 30 * 256, generator=g), torch.randint(0, 2545, (1, 25), generator=g), 140)
        kw["steps"] = 5
    ref = O.sample(sd, cfg, *args, **kw)
    dargs = tuple(a.to(DEV) if torch.is_tensor(a) else a for a in args)
    dkw = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in kw.items()}
    out, traj = model.sample(*dargs, **dkw, y0=ref.y0.to(DEV))
    if variant == "attn_mask":
        # key-masked mode: rows past a sample's duration influence nothing and are not computed at all (padded tiles
        # are skipped) — compare the valid rows of every sample
        durs = args[2].tolist()
        got = torch.cat([out[b, :d].cpu() for b, d in enumerate(durs)])
        want = torch.cat([ref.out[b, :d] for b, d in enumerate(durs)])
        t1g = torch.cat([traj[1][b, :d].cpu() for b, d in enumerate(durs)])
        t1w = torch.cat([ref.trajectory[1][b, :d] for b, d in enumerate(durs)])
        r, r1 = rel(got, want), rel(t1g, t1w)
    else:
        r, r1 = rel(out, ref.out), rel(traj[1], ref.trajectory[1])
    print(f"[oracle:{variant}] final rel-L2 {r:.3e}  step-1 {r1:.3e}")
    assert r <= TOL


def test_large_batch_step():
    """B = 8 x 938 frames (BASELINE config 4 shape per GPU, M = 15008): the large-batch GEMM tile shapes; one Euler
    step against the CPU oracle."""
    cfg = O.f5tts_base()
    model, sd = build(cfg, 1234)
    g = torch.Generator().manual_seed(21)
    cond = torch.randn(8, 282, 100, generator=g)
    text = torch.randint(0, 2545, (8, 150), generator=g)
    kw = dict(steps=1, cfg_strength=2.0, sway_sampling_coef=-1.0, seed=5, use_epss=False)
    ref = O.sample(sd, cfg, cond, text, 938, **kw)
    out, traj = model.sample(cond.to(DEV), text.to(DEV), 938, **kw, y0=ref.y0.to(DEV))
    r = rel(traj[1], ref.trajectory[1])
    print(f"[large-batch] step rel-L2 {r:.3e}")
    assert r <= TOL


def test_graph_equals_eager_and_deterministic():
    cfg = O.f5tts_base()
    model, _ = build(cfg, 1234)
    g = torch.Generator().manual_seed(1)
    cond = torch.randn(1, 50, 100, generator=g).to(DEV)
    text = torch.randint(0, 2545, (1, 40), generator=g).to(DEV)
    kw = dict(steps=4, cfg_strength=2.0, sway_sampling_coef=-1.0, seed=3)
    model.use_cuda_graph = True
    a, _ = model.sample(cond, text, 200, **kw)
    b, _ = model.sample(cond, text, 200, **kw)
    model.use_cuda_graph = False
    c, _ = model.sample(cond, text, 200, **kw)
    model.use_cuda_graph = True
    assert torch.equal(a, b), "same inputs + seed must be bit-identical run to run"
    assert torch.equal(a, c), "graph replay and eager launches run the same kernels"


def test_properties_at_baseline_size():
    """BASELINE config 2 shape (B=1, N=938, NFE 32) is too slow for the CPU oracle inside a test; check properties."""
    cfg = O.f5tts_base()
    model, _ = build(cfg, 1234)
    g = torch.Generator().manual_seed(9)
    cond = torch.randn(1, 282, 100, generator=g).to(DEV)
    text = torch.randint(0, 2545, (1, 150), generator=g).to(DEV)
    y0 = torch.randn(1, 938, 100, generator=g).to(DEV)
    # (1) one Euler step is affine in cfg_strength: y(s) = y0 + dt (p + (p - n) s)
    outs = []
    for s in (1.0, 2.0, 3.0):
        _, tr = model.sample(cond, text, 938, steps=1, cfg_strength=s, sway_sampling_coef=None, y0=y0, use_epss=False)
        outs.append(tr[1].double())
    lin = float(((outs[2] - outs[1]) - (outs[1] - outs[0])).norm() / (outs[1] - outs[0]).norm())
    print(f"[prop] cfg affinity residual {lin:.3e}")
    assert lin <= 1e-4
    # (2) trajectory composition: 32 steps in one call == 16 + 16 steps chained through the state
    out32, tr32 = model.sample(cond, text, 938, steps=32, cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y0)
    assert tr32.shape == (33, 1, 938, 100)
    assert torch.isfinite(out32).all()
    assert torch.equal(out32[:, :282], cond), "prompt frames are copied through (cfm.py:221-223)"
    # (3) batch consistency: two identical samples in a batch produce identical rows, equal to the B=1 result
    cond2, text2, y02 = cond.repeat(2, 1, 1), text.repeat(2, 1), y0.repeat(2, 1, 1)
    out2, _ = model.sample(cond2, text2, 938, steps=2, cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y02)
    out1, _ = model.sample(cond, text, 938, steps=2, cfg_strength=2.0, sway_sampling_coef=-1.0, y0=y0)
    assert torch.equal(out2[0], out2[1])
    assert rel(out2[0:1], out1) <= 1e-5


def test_backbone_operator_seam():
    """transformer(x, cond, text, time, mask, cfg_infer=True) == the reference operator (dit.py:319-370)."""
    cfg = O.f5tts_base()
    model, sd = build(cfg, 1234)
    g = torch.Generator().manual_seed(11)
    x, cond = torch.randn(2, 90, 100, generator=g), torch.randn(2, 90, 100, generator=g)
    text = torch.randint(0, 2545, (2, 40), generator=g)
    mask = O.lens_to_mask(torch.tensor([90, 61]))
    t = torch.tensor(0.43)
    te = (O.text_embedding_dit(sd, cfg, text, mask.sum(1), False), O.text_embedding_dit(sd, cfg, text, mask.sum(1), True))
    ref = O.dit_forward(sd, cfg, x, cond, te, t, mask, True)
    got = model.transformer(x.to(DEV), cond.to(DEV), text.to(DEV), t.to(DEV), mask=mask.to(DEV), cfg_infer=True)
    r = rel(got, ref)
    print(f"[seam] dit forward rel-L2 {r:.3e}")
    assert got.shape == (4, 90, 100) and r <= 3e-3


def test_errors_are_loud():
    from f5_tts_b200 import _lib

    with pytest.raises(_lib.F5LibraryError):
        F5.MelSpec()(torch.zeros(1, 4000))  # CPU tensor: no fallback
    model, _ = build(O.f5tts_base(), 1234)
    with pytest.raises(NotImplementedError):
        model(torch.zeros(1, 10, 100), torch.zeros(1, 10, dtype=torch.long))


@pytest.mark.parametrize("arch", ["f5tts_base", "f5tts_v1_base"])
def test_exact_varlen_batch_equals_single_calls(arch):
    """exact_varlen (f5_sample_args): one batched call over samples of different lengths == a loop of B = 1 calls, which
    is what the reference's infer_batch_process computes per text chunk (utils_infer.py:540-541).  Also against the CPU
    oracle run sample by sample.  Covers the strict text-block masking, per-sample conv padding, key masking and the
    skipping of padded tiles (lengths chosen to leave whole 128-row tiles of padding)."""
    cfg = getattr(O, arch)()
    model, sd = build(cfg, 1234)
    g = torch.Generator().manual_seed(33)
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
        if b == 1:  # one sample against the fp32 oracle as well
            ref = O.sample(sd, cfg, cond, tb, d, **kw, y0=y0[b])
            assert rel(o, ref.out) <= TOL
    y0b = torch.zeros(3, max(durs), 100)
    for b, d in enumerate(durs):
        y0b[b, :d] = y0[b][0]
    out, _ = model.sample(cond.expand(3, -1, -1).contiguous().to(DEV), text.to(DEV), torch.tensor(durs).to(DEV),
                          lens=torch.full((3,), n_ref).to(DEV), **kw, y0=y0b.to(DEV), exact_varlen=True)
    for b, d in enumerate(durs):
        r = rel(out[b, :d], singles[b][0])
        print(f"[exact_varlen {arch}] sample {b} ({d} frames): batched vs single rel-L2 {r:.3e}")
        assert r <= 1e-3
