"""Generate the fixtures of UNetT checkpoints built with skip_connect_type="add" or "none" by running the UNMODIFIED
reference's CFM.sample (TEST INFRASTRUCTURE).  Needs the reference checkout (F5_REFERENCE_SRC = its src directory); runs
on the CPU:

    F5_REFERENCE_SRC=<reference>/src python -m oracle.make_golden_unett_skip   # prints oracle-vs-reference rel-L2

Same recipe as oracle/make_golden_arch_options.py, whose case inputs it reuses: synthetic weights loaded with
load_state_dict(strict=True), which also pins the checkpoint layout of these types (no `layers.{i}.0.weight`: the
reference's skip_proj slot is None).  The oracle side is oracle/unett_skip.sample.  Each case is first checked: the
oracle must reproduce the reference within 1e-6 rel-L2 before its fixture is written.
"""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import synthdata as SD  # noqa: E402
from oracle import f5_oracle as O  # noqa: E402
from oracle import make_golden as MG  # noqa: E402
from oracle import make_golden_arch_options as MA  # noqa: E402
from oracle import ode_midpoint as OM  # noqa: E402
from oracle import ref_shims  # noqa: E402
from oracle import unett_skip as OU  # noqa: E402

ADD, NONE = dict(skip_connect_type="add"), dict(skip_connect_type="none")
TOL = 1e-6


def small_widths() -> O.ArchConfig:
    """E2TTS_Small widths (dim 768, 12 heads, ff 4x) at depth 4 with the additive skip."""
    cfg = SD.e2tts_small()
    cfg.depth, cfg.skip_connect_type = 4, "add"
    return cfg


# name -> (config, inputs).  Every case is a ragged batch of two with ragged text.
CASES = {
    "unett_skip_add_b2_varlen": (MG.tiny_unett(**ADD),
                                 dict(B=2, n_ref=24, nt=30, durations=[77, 52], lens=[24, 20], steps=4,
                                      cfg_strength=2.0, sway=-1.0, seed=41, text_pad=[30, 21])),
    "unett_skip_none_b2_varlen": (MG.tiny_unett(**NONE),
                                  dict(B=2, n_ref=24, nt=30, durations=[74, 55], lens=[24, 20], steps=4,
                                       cfg_strength=2.0, sway=-1.0, seed=42, text_pad=[30, 19])),
    "unett_skip_add_b2_attnmask": (MG.tiny_unett(attn_mask_enabled=True, **ADD),
                                   dict(B=2, n_ref=24, nt=30, durations=[81, 50], lens=[24, 20], steps=4,
                                        cfg_strength=2.0, sway=-1.0, seed=43, text_pad=[30, 22])),
    "unett_skip_add_qknorm_b2_midpoint": (MG.tiny_unett(qk_norm="rms_norm", **ADD),
                                          dict(B=2, n_ref=24, nt=30, durations=[70, 57], lens=[24, 20], steps=2,
                                               cfg_strength=2.0, sway=-1.0, seed=44, text_pad=[30, 20],
                                               method="midpoint")),
    "unett_skip_add_dh128_b2": (MG.tiny_unett(dim_head=128, **ADD),
                                dict(B=2, n_ref=24, nt=30, durations=[133, 71], lens=[24, 20], steps=4,
                                     cfg_strength=2.0, sway=-1.0, seed=45, text_pad=[30, 24])),
    "unett_skip_add_d768_b2": (small_widths(),
                               dict(B=2, n_ref=40, nt=36, durations=[171, 130], lens=[40, 33], steps=2,
                                    cfg_strength=2.0, sway=-1.0, seed=46, text_pad=[36, 25])),
}


def build_reference(cfg, sd, method):
    """The unmodified reference CFM over UNetT(skip_connect_type=cfg.skip_connect_type), weights loaded strict."""
    if "f5_tts.model.cfm" not in sys.modules:
        ref_shims._stub("torchdiffeq", odeint=OM.odeint)
    cfm, _, unett, _, _ = ref_shims.import_reference()
    assert cfm.odeint is OM.odeint, "the reference was imported with another odeint"
    backbone = unett.UNetT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head, ff_mult=cfg.ff_mult,
                           mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds, text_dim=cfg.text_dim,
                           text_mask_padding=cfg.text_mask_padding, conv_layers=cfg.conv_layers,
                           pe_attn_head=cfg.pe_attn_head, attn_backend="torch",
                           attn_mask_enabled=cfg.attn_mask_enabled, qk_norm=cfg.qk_norm,
                           skip_connect_type=cfg.skip_connect_type)
    model = cfm.CFM(transformer=backbone,
                    mel_spec_kwargs=dict(n_fft=1024, hop_length=256, win_length=1024, n_mel_channels=100,
                                         target_sample_rate=24000, mel_spec_type="vocos"),
                    odeint_kwargs=dict(method=method), vocab_char_map=None)
    res = model.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    return model.eval()


def run(name, cfg, kw, wseed=1234):
    t0 = time.time()
    method = kw.get("method", "euler")
    sd = O.synthetic_state_dict(cfg, seed=wseed)
    model = build_reference(cfg, sd, method)
    cond, text, duration, lens = MA.case_inputs(cfg, **kw)
    skw = dict(steps=kw["steps"], cfg_strength=kw["cfg_strength"], sway_sampling_coef=kw["sway"], seed=kw["seed"])
    with torch.no_grad():
        out, traj = model.sample(cond=cond, text=text, duration=duration, lens=lens, **skw)
    res = OU.sample(sd, cfg, cond, text, duration, lens=lens, method=method, **skw)
    d = max(MG.rel_l2(res.out, out), MG.rel_l2(res.trajectory[1], traj[1]))
    print(f"[{name}] out {tuple(out.shape)} oracle-vs-ref rel-L2 {d:.3e}  ({time.time() - t0:.1f}s)")
    if d > TOL:
        raise SystemExit(f"[{name}] the oracle does not reproduce the reference (rel-L2 {d:.3e} > {TOL}): not written")
    np.savez_compressed(os.path.join(MG.GOLD, name + ".npz"), cond=cond.numpy(), text=text.numpy(),
                        duration=np.asarray(kw["durations"]), lens=np.asarray(kw.get("lens") or []),
                        steps=kw["steps"], cfg_strength=kw["cfg_strength"], sway=np.asarray(kw["sway"]),
                        seed=kw["seed"], wseed=wseed, method=np.asarray(method), out=out.numpy(),
                        y0=traj[0].numpy(), traj_1=traj[1].numpy(), cfg=np.asarray(repr(cfg)))
    return d


def main():
    if not ref_shims.reference_available():
        raise SystemExit("set F5_REFERENCE_SRC to the reference checkout's src directory")
    torch.set_num_threads(os.cpu_count() or 8)
    worst = max(run(name, cfg, kw) for name, (cfg, kw) in CASES.items())
    print(f"largest oracle-vs-reference rel-L2: {worst:.3e}")


if __name__ == "__main__":
    main()
