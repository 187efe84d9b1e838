"""GPU parity of CFM.sample at the REAL sizes of the BASELINE.json configurations.

  cfg2  B=1, 938 frames, NFE 32 in full — against tests/golden/cfg2_full_nfe32.npz, produced by the UNMODIFIED reference
        in fp32 (oracle/make_golden_baseline.py); drift reported at steps 1 / 8 / 16 / 32 next to the reference's own
        fp16-vs-fp32 drift on the same inputs (stored in the fixture; SURVEY.md §9.4 measured 1.5e-3 at N = 400).
  cfg3  B=8 variable length 469..1875 frames (padded), NFE 8 of 32, faithful mode (padded keys attended,
        attn_mask_enabled=False) and masked mode (attn_mask_enabled=True)
  cfg4  B=8 x 938 frames (one GPU's shard of the 64-utterance config), the full EPSS-16 grid
  cfg5  E2-TTS UNetT, B=8 x 938 frames, NFE 8 of 32 — the batched UNetT path (time token, row_len + 1)
cfg3-5 compare with golden vectors of the CPU oracle (tests/golden/fullsize_*.npz, written by
oracle/make_golden_fullsize.py: every third generated row of every utterance after step 1 and after the last step, fp32;
the oracle is pinned bit-exactly to the reference by tests/test_oracle_vs_golden.py).  Computing the oracle live took half
of the suite's 12 minutes on the GPU box's host; the initial noise is re-drawn from the seed exactly as cfm.py:196-201
does and checked against the fixture's checksum.  Identical injected y0 everywhere.

Tolerance (BASELINE.md §2, SURVEY.md §8c): rel-L2 of the generated region <= 5e-3 at every checked step.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.fullsize]

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import f5_tts_b200 as F5  # noqa: E402
import synthdata as SD  # noqa: E402
from oracle import f5_oracle as O  # noqa: E402
from oracle import step_increment as SI  # noqa: E402

DEV = "cuda:0"
TOL = 5e-3
_cache = {}


def build(cfg, wseed=1234):
    key = (repr(cfg), wseed)
    if key not in _cache:
        _cache.clear()  # one 1.3 GB model at a time
        cls = F5.DiT if cfg.backbone == "DiT" else F5.UNetT
        model = F5.CFM(transformer=cls(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head,
                                       ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds,
                                       text_dim=cfg.text_dim, text_mask_padding=cfg.text_mask_padding,
                                       conv_layers=cfg.conv_layers, pe_attn_head=cfg.pe_attn_head,
                                       attn_mask_enabled=cfg.attn_mask_enabled))
        sd = SD.synthetic_state_dict(cfg, seed=wseed)
        model.load_state_dict(sd, strict=True)
        _cache[key] = (model.to(DEV), sd)
    return _cache[key]


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / b.norm())


def test_cfg2_full_nfe32_vs_reference(golden_dir):
    z = np.load(os.path.join(golden_dir, "cfg2_full_nfe32.npz"))
    w = SD.WORKLOADS["cfg2"]
    cfg = SD.f5tts_base()
    model, _ = build(cfg, int(z["wseed"]))
    wav, text, duration, _ = SD.synth_inputs(w)
    out, traj = model.sample(wav.to(DEV), text.to(DEV), int(duration[0]), steps=int(z["steps"]),
                             cfg_strength=float(z["cfg_strength"]), sway_sampling_coef=float(z["sway"]), seed=int(z["seed"]),
                             y0=torch.from_numpy(z["y0"]).to(DEV))
    SI.check(traj[1], z["y0"], z["traj_1"], None, "cfg2_full_nfe32")  # every row: B = 1, no mask
    n_ref = int(z["n_ref"])
    gen = slice(n_ref, None)
    drift = {int(k): rel(traj[int(k)][:, gen], torch.from_numpy(z[f"traj_{int(k)}"])[:, gen]) for k in z["kept"]}
    ref16 = dict(zip([int(k) for k in z["kept"]], z["ref_fp16_drift"].tolist()))
    print("[cfg2 full NFE 32] rel-L2 of the generated region vs the fp32 reference, per step:")
    for k in sorted(drift):
        print(f"   step {k:2d}: H100 path {drift[k]:.3e}   reference's own fp16 path {ref16[k]:.3e}")
    final = rel(out, torch.from_numpy(z["out"]))
    print(f"   final mel (all rows) {final:.3e}   gate {TOL:.0e}")
    # prompt rows are the prompt mel itself (cfm.py:221-223): CUDA mel kernel vs torchaudio on the CPU, fp32 rounding only
    assert torch.allclose(out[:, :n_ref].float().cpu(), torch.from_numpy(z["out"])[:, :n_ref], atol=2e-4), "prompt rows"
    assert all(v <= TOL for v in drift.values()) and final <= TOL
    # fp32 state / residual / statistics: the H100 path must not drift more than the reference's fp16 path does
    assert drift[32] <= ref16[32]


def _golden_vs_gpu(name, golden_dir):
    from oracle.make_golden_fullsize import draw_y0

    z = np.load(os.path.join(golden_dir, f"fullsize_{name}.npz"))
    cfg = getattr(SD, str(z["arch"]))()
    cfg.attn_mask_enabled = bool(z["attn_mask_enabled"])
    w, steps, stride = SD.WORKLOADS[str(z["workload"])], int(z["steps"]), int(z["stride"])
    model, _ = build(cfg, int(z["wseed"]))
    wav, text, duration, lens = SD.synth_inputs(w)
    cond = O.mel_spectrogram(wav).permute(0, 2, 1).contiguous()  # [B, n_ref, 100]; prompt lengths via `lens`
    y0 = draw_y0(duration, cfg.mel_dim, seed=int(z["seed"]))
    chk = np.array([float(y0.double().sum()), float(y0.double().abs().sum())])
    assert np.allclose(chk, z["y0_checksum"], rtol=1e-12), "the CPU generator drew different noise than the fixture's"
    out, traj = model.sample(cond.to(DEV), text.to(DEV), duration.to(DEV), lens=lens.to(DEV), steps=steps,
                             cfg_strength=SD.CFG_STRENGTH, sway_sampling_coef=SD.SWAY, seed=int(z["seed"]), y0=y0.to(DEV))
    g1, gN = torch.from_numpy(z["step1"]), torch.from_numpy(z["final"])
    worst, at = 0.0, 0
    inc = ([], [], [])  # the first increment's rows: engine, y0, fixture
    for b in range(w["B"]):  # every `stride`-th valid generated row of each utterance
        sl = slice(int(lens[b]), int(duration[b]), stride)
        n = len(range(*sl.indices(int(duration[b]))))
        for rows, t in zip(inc, (traj[1][b, sl], y0[b, sl], g1[at: at + n])):
            rows.append(t)
        r1 = rel(traj[1][b, sl], g1[at: at + n])
        rN = rel(out[b, sl], gN[at: at + n])
        at += n
        worst = max(worst, r1, rN)
        print(f"[{name}] utt {b} frames {int(duration[b])}: step-1 {r1:.3e}  final({steps} steps) {rN:.3e}")
    assert at == g1.shape[0] == gN.shape[0]
    SI.check_rows(*inc, tag=f"fullsize_{name}")
    assert worst <= TOL
    return worst


@pytest.mark.parametrize("mode", ["faithful", "masked"])
def test_cfg3_varlen_b8_nfe8(mode, golden_dir):
    _golden_vs_gpu(f"cfg3_{mode}", golden_dir)


def test_cfg4_b8_epss16(golden_dir):
    _golden_vs_gpu("cfg4_epss16", golden_dir)


def test_cfg5_unett_b8_nfe8(golden_dir):
    _golden_vs_gpu("cfg5_unett", golden_dir)
