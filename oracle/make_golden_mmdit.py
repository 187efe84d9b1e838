"""Generate the MMDiT fixtures tests/golden/mmdit_*.npz by running the UNMODIFIED reference's CFM.sample over its
backbones/mmdit.py MMDiT (TEST INFRASTRUCTURE).  Needs the reference checkout (F5_REFERENCE_SRC = its src directory);
runs on the CPU:

    F5_REFERENCE_SRC=<reference>/src python -m oracle.make_golden_mmdit   # prints oracle-vs-reference rel-L2

Same recipe as oracle/make_golden_arch_options.py: weights are synthdata.synthetic_state_dict(config, seed) loaded
with load_state_dict(strict=True) into the reference module, and the fixtures store the inputs, the reference's step-1
and final outputs and the reference's state-dict key list, not the weights.  The oracle side is oracle/mmdit.sample.
"""
from __future__ import annotations

import dataclasses
import importlib
import json
import os
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import synthdata as SD  # noqa: E402
from oracle import make_golden as MG  # noqa: E402
from oracle import make_golden_arch_options as MGA  # noqa: E402
from oracle import mmdit as OMM  # noqa: E402
from oracle import ode_midpoint as OM  # noqa: E402
from oracle import ref_shims  # noqa: E402


def tiny_mmdit(**over) -> SD.ArchConfig:
    base = dict(backbone="MMDiT", dim=128, depth=3, heads=2, dim_head=64, ff_mult=2, mel_dim=100, text_num_embeds=50,
                text_dim=None, conv_layers=0, text_mask_padding=True, pe_attn_head=None, attn_mask_enabled=False)
    base.update(over)
    return SD.ArchConfig(**base)


def v1base_widths_mmdit() -> SD.ArchConfig:
    cfg = SD.mmdit_v1_base_widths()
    cfg.depth = 3
    return cfg


VARLEN = dict(B=2, n_ref=24, nt=30, durations=[80, 57], lens=[24, 20], steps=4, cfg_strength=2.0, sway=-1.0,
              text_pad=[30, 19])
# name -> (config, inputs).  B > 1 cases are variable length with ragged (trailing-padded) text.
CASES = {
    "mmdit_b1_epss_sway": (tiny_mmdit(), dict(B=1, n_ref=20, nt=24, durations=70, steps=5, cfg_strength=2.0,
                                              sway=-1.0, seed=41)),
    "mmdit_b2_varlen": (tiny_mmdit(), dict(VARLEN, seed=42)),
    "mmdit_b2_attnmask": (tiny_mmdit(attn_mask_enabled=True), dict(VARLEN, seed=43)),
    "mmdit_qknorm_b2_midpoint": (tiny_mmdit(qk_norm="rms_norm"), dict(VARLEN, steps=2, seed=44, method="midpoint")),
    "mmdit_nocfg_b1": (tiny_mmdit(), dict(B=1, n_ref=20, nt=24, durations=66, steps=4, cfg_strength=0.0, sway=None,
                                          seed=45)),
    "mmdit_nomaskpad_b2": (tiny_mmdit(text_mask_padding=False), dict(VARLEN, seed=46)),
    "mmdit_dh128_b2": (tiny_mmdit(dim=256, heads=2, dim_head=128), dict(VARLEN, seed=47)),
    # text over two key tiles (nt 140 > 128), N = 203 not a multiple of 128; per-segment key lengths in masked mode
    "mmdit_nt140_b2_attnmask": (tiny_mmdit(attn_mask_enabled=True),
                                dict(B=2, n_ref=30, nt=140, durations=[203, 170], lens=[30, 26], steps=3,
                                     cfg_strength=2.0, sway=-1.0, seed=48, text_pad=[140, 131])),
    # F5TTS_v1_Base widths (dim 1024, 16 heads, ff_mult 2) at depth 3: the full-size GEMM tiles
    "mmdit_v1base_d3_b2": (v1base_widths_mmdit(),
                           dict(B=2, n_ref=40, nt=36, durations=[171, 130], lens=[40, 33], steps=2, cfg_strength=2.0,
                                sway=-1.0, seed=49, text_pad=[36, 25])),
}


def config_json(cfg: SD.ArchConfig) -> str:
    return json.dumps(dataclasses.asdict(cfg), sort_keys=True)


def build_reference(cfg: SD.ArchConfig, sd, method):
    """The unmodified reference CFM over its MMDiT, weights loaded with strict=True."""
    if "f5_tts.model.cfm" not in sys.modules:
        ref_shims._stub("torchdiffeq", odeint=OM.odeint)
    cfm = ref_shims.import_reference()[0]
    assert cfm.odeint is OM.odeint, "the reference was imported with another odeint"
    mmdit = importlib.import_module("f5_tts.model.backbones.mmdit")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        backbone = mmdit.MMDiT(dim=cfg.dim, depth=cfg.depth, heads=cfg.heads, dim_head=cfg.dim_head,
                               ff_mult=cfg.ff_mult, mel_dim=cfg.mel_dim, text_num_embeds=cfg.text_num_embeds,
                               text_mask_padding=cfg.text_mask_padding, qk_norm=cfg.qk_norm, attn_backend="torch",
                               attn_mask_enabled=cfg.attn_mask_enabled)
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
    sd = SD.synthetic_state_dict(cfg, seed=wseed)
    model = build_reference(cfg, sd, method)
    keys = list(model.state_dict().keys())
    cond, text, duration, lens = MGA.case_inputs(cfg, **kw)
    skw = dict(steps=kw["steps"], cfg_strength=kw["cfg_strength"], sway_sampling_coef=kw["sway"], seed=kw["seed"])
    with torch.no_grad():
        out, traj = model.sample(cond=cond, text=text, duration=duration, lens=lens, **skw)
    res = OMM.sample(sd, cfg, cond, text, duration, lens=lens, method=method, **skw)
    d = max(MG.rel_l2(res.out, out), MG.rel_l2(res.trajectory[1], traj[1]))
    print(f"[{name}] out {tuple(out.shape)} oracle-vs-ref rel-L2 {d:.3e}  ({time.time() - t0:.1f}s)")
    np.savez_compressed(os.path.join(MG.GOLD, name + ".npz"), cond=cond.numpy(), text=text.numpy(),
                        duration=np.asarray(kw["durations"]), lens=np.asarray(kw.get("lens") or []),
                        steps=kw["steps"], cfg_strength=kw["cfg_strength"],
                        sway=np.asarray(np.nan if kw["sway"] is None else kw["sway"]), seed=kw["seed"], wseed=wseed,
                        method=np.asarray(method), out=out.numpy(), y0=traj[0].numpy(), traj_1=traj[1].numpy(),
                        cfg=np.asarray(config_json(cfg)), ref_keys=np.asarray(keys))
    return d


def main():
    if not ref_shims.reference_available():
        raise SystemExit("set F5_REFERENCE_SRC to the reference checkout's src directory")
    torch.set_num_threads(os.cpu_count() or 8)
    worst = max(run(name, cfg, kw) for name, (cfg, kw) in CASES.items())
    print(f"largest oracle-vs-reference rel-L2: {worst:.3e}")


if __name__ == "__main__":
    main()
