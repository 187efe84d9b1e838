"""Generate the fixtures of DiT / UNetT checkpoints built with 128-wide attention heads (dim_head=128) by running the
UNMODIFIED reference's CFM.sample (TEST INFRASTRUCTURE).  Needs the reference checkout (F5_REFERENCE_SRC = its src
directory); runs on the CPU:

    F5_REFERENCE_SRC=<reference>/src python -m oracle.make_golden_dim_head   # prints oracle-vs-reference rel-L2

Same recipe as oracle/make_golden_arch_options.py, whose reference builder and writer it reuses: synthetic weights
loaded with load_state_dict(strict=True), which also pins the shapes a dim_head=128 checkpoint has (to_q / to_k / to_v
[heads * 128, dim], q_norm / k_norm [128]).  The oracle side is oracle/arch_options.sample over oracle/f5_oracle.py,
both of which take dim_head from the config.
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import synthdata as SD  # noqa: E402
from oracle import f5_oracle as O  # noqa: E402
from oracle import make_golden as MG  # noqa: E402
from oracle import make_golden_arch_options as MA  # noqa: E402
from oracle import ref_shims  # noqa: E402

DH = dict(dim_head=128)


def full_width() -> O.ArchConfig:
    """F5TTS_v1_Base widths (dim 1024, text_dim 512, 4 text blocks) with 8 heads of 128, at depth 2."""
    cfg = SD.f5tts_v1_base()
    cfg.heads, cfg.dim_head, cfg.depth = 8, 128, 2
    return cfg


# name -> (config, inputs).  The tiny configs keep 2 heads, so the attention width heads * 128 = 256 is not dim = 128.
CASES = {
    "dh128_dit_b2_varlen": (MG.tiny_dit(**DH),
                            dict(B=2, n_ref=24, nt=30, durations=[150, 97], lens=[24, 20], steps=4,
                                 cfg_strength=2.0, sway=-1.0, seed=31, text_pad=[30, 19])),
    "dh128_dit_qknorm_b2_varlen": (MG.tiny_dit(text_mask_padding=True, pe_attn_head=None, qk_norm="rms_norm", **DH),
                                   dict(B=2, n_ref=24, nt=30, durations=[140, 83], lens=[24, 20], steps=4,
                                        cfg_strength=2.0, sway=-1.0, seed=32, text_pad=[30, 21])),
    "dh128_unett_b2_varlen": (MG.tiny_unett(**DH),
                              dict(B=2, n_ref=24, nt=30, durations=[131, 70], lens=[24, 20], steps=4,
                                   cfg_strength=2.0, sway=-1.0, seed=33, text_pad=[30, 23])),
    "dh128_f5v1_d2_b2_midpoint": (full_width(),
                                  dict(B=2, n_ref=40, nt=36, durations=[171, 130], lens=[40, 33], steps=2,
                                       cfg_strength=2.0, sway=-1.0, seed=34, text_pad=[36, 25], method="midpoint")),
}


def main():
    if not ref_shims.reference_available():
        raise SystemExit("set F5_REFERENCE_SRC to the reference checkout's src directory")
    torch.set_num_threads(os.cpu_count() or 8)
    worst = max(MA.run(name, cfg, kw) for name, (cfg, kw) in CASES.items())
    print(f"largest oracle-vs-reference rel-L2: {worst:.3e}")


if __name__ == "__main__":
    main()
