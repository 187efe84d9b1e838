"""Generate the Small-config fixtures (dim 768: F5TTS_v1_Small, F5TTS_Small, E2TTS_Small) by running the UNMODIFIED
reference's CFM.sample (TEST INFRASTRUCTURE).  Needs the reference checkout (F5_REFERENCE_SRC = its src directory);
runs on the CPU:

    F5_REFERENCE_SRC=<reference>/src python -m oracle.make_golden_small   # prints oracle-vs-reference rel-L2

Same recipe as oracle/make_golden.py (its run_case / build_reference are reused): weights are
synthetic_state_dict(config, seed) loaded with load_state_dict(strict=True), which also pins the Small checkpoint key
layout; the fixtures store the inputs and the reference outputs, not the weights.  At dim 768 the reference's
ConvPositionEmbedding has 768 / 16 = 48 channels per group.
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import synthdata as SD  # noqa: E402
from oracle.make_golden import GOLD, run_case  # noqa: E402

# name -> (config, run_case keyword arguments)
CASES = {
    "f5v1small_b2_varlen": (SD.f5tts_v1_small, dict(B=2, n_ref=50, nt=28, durations=[160, 120], lens=[50, 36],
                                                   steps=3, cfg_strength=2.0, sway=-1.0, seed=11, text_pad=[28, 19])),
    "f5small_b1_n192": (SD.f5tts_small, dict(B=1, n_ref=58, nt=31, durations=192, steps=4, cfg_strength=2.0, sway=-1.0,
                                            seed=12)),
    "e2small_b2_varlen": (SD.e2tts_small, dict(B=2, n_ref=36, nt=28, durations=[140, 104], lens=[36, 30], steps=2,
                                              cfg_strength=2.0, sway=-1.0, seed=13, text_pad=[28, 18], wseed=99)),
}


def main():
    os.makedirs(GOLD, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 8)
    for name, (cfg, kw) in CASES.items():
        run_case(name, cfg(), **kw)


if __name__ == "__main__":
    main()
