"""The first ODE step's increment against a committed fixture — TEST INFRASTRUCTURE ONLY.

traj[1] = y0 + dt * v, so a rel-L2 on traj[1] divides the velocity's error by |traj[1] - y0| / |traj[1]|, which is
2e-3 to 1e-2 on fixtures with a small first step (cfg2_full_nfe32, mmdit_b1_epss_sway, dit_tiny_*): a step-1 gate of
5e-3 there lets the velocity be off by 50 % or more.  This compares the increments traj[1] - y0 themselves (the same y0
on both sides), per sample and per frame.

Every GPU test that samples an end-to-end fixture with y0 and traj_1 calls it: the reference fixtures of
test_gpu_sample, test_gpu_small_configs, test_gpu_arch_options, test_gpu_dim_head, test_gpu_unett_skip, test_gpu_mmdit
and test_gpu_ode_midpoint, and the real-size fixtures of test_gpu_fullsize (cfg2_full_nfe32 over all 938 rows; the
fullsize_cfg3/4/5 fixtures over the every-third generated rows they store, with y0 re-drawn by
make_golden_fullsize.draw_y0).  reference_tiny_dit_varlen_midpoint is the one such fixture left out: no GPU test samples
it (it pins the CPU midpoint oracle, tests/test_ode_midpoint_cpu.py; the GPU midpoint path is checked on
f5base_b2_varlen_midpoint).

Measured on an H100 80GB HBM3 (700 W power limit), worst per-sample increment rel-L2 / worst frame over its sample's
median: cfg2_full_nfe32 1.15e-3 / 1.48, fullsize_cfg3_faithful 1.72e-3 / 1.56, fullsize_cfg3_masked 1.65e-3 / 1.50,
fullsize_cfg4_epss16 1.67e-3 / 1.33, fullsize_cfg5_unett 1.33e-3 / 1.29; over the 39 smaller fixtures 4.4e-4 to 1.57e-3
(e2base_b1_n128) and up to 2.33 (the dh128 qk_norm and midpoint fixtures).  Each test prints its fixture's worst values.
"""
from __future__ import annotations

import torch

SAMPLE_TOL = 5e-3  # the project's end-to-end rel-L2, now on dt * v
FRAME_FACTOR = 3.5  # a frame's error over its sample's median frame error: 1.5x the worst measured (2.33)


def check(traj1, y0, want1, lengths=None, tag: str = "", sample_tol: float = SAMPLE_TOL,
          frame_factor: float = FRAME_FACTOR) -> tuple[float, float]:
    """Gate the increments traj1 - y0 (engine) against want1 - y0 (fixture), [B, N, mel] each.  lengths: compare each
    sample's first lengths[b] frames only (key-masked and exact_varlen fixtures, whose padded rows are not computed).
    See check_rows for the gates."""
    y0 = torch.as_tensor(y0).double().cpu()
    got, want = torch.as_tensor(traj1).double().cpu(), torch.as_tensor(want1).double().cpu()
    B, N = y0.shape[:2]
    n = [N] * B if lengths is None else [int(v) for v in torch.as_tensor(lengths).reshape(-1).expand(B)]
    return check_rows([got[b, :n[b]] for b in range(B)], [y0[b, :n[b]] for b in range(B)],
                      [want[b, :n[b]] for b in range(B)], tag, sample_tol, frame_factor)


def check_rows(traj1, y0, want1, tag: str = "", sample_tol: float = SAMPLE_TOL,
               frame_factor: float = FRAME_FACTOR) -> tuple[float, float]:
    """The same gates over per-sample lists of compared frames, [n_b, mel] each (e.g. the strided rows a fullsize
    fixture keeps).  Per sample: rel-L2 of the increment <= sample_tol.  Per frame: the rms error over the mel channels
    <= frame_factor * the sample's median frame error (floored at 1e-6 of the sample's rms increment).  Returns (worst
    rel-L2, worst frame ratio)."""
    worst_rel = worst_frame = 0.0
    for b, (g, y, w) in enumerate(zip(traj1, y0, want1)):
        g, y, w = (torch.as_tensor(a).double().cpu() for a in (g, y, w))
        assert torch.isfinite(g).all(), f"{tag} sample {b}: non-finite increment"
        d, w = g - w, w - y
        r = float(d.norm() / w.norm())
        fe = d.pow(2).mean(-1).sqrt()
        floor = max(float(fe.median()), 1e-6 * float(w.pow(2).mean().sqrt()))
        fr = float(fe.max()) / floor
        worst_rel, worst_frame = max(worst_rel, r), max(worst_frame, fr)
        assert r <= sample_tol, f"{tag} sample {b}: step-1 increment rel-L2 {r:.3e} > {sample_tol}"
        assert fr <= frame_factor, (f"{tag} sample {b}: frame {int(fe.argmax())} increment error {fr:.2f}x the median "
                                    f"frame's (> {frame_factor})")
    print(f"[{tag}] step-1 increment: worst rel-L2 {worst_rel:.3e}, worst frame / median {worst_frame:.2f}")
    return worst_rel, worst_frame
