"""The kernel hooks keep up with the launchers (CPU, no GPU needed).

libf5tts_b200_kernels.so (csrc/kernel_hooks.cu) gives the element-by-element GPU tests one extern "C" entry point per
launcher of internal.h.  A launcher without a hook, a launch mode no hook reaches, a hook that build() does not check
for, or a hook no GPU test calls is a kernel only the end-to-end tests see.  This file parses the sources to keep that
from happening quietly, and checks the float64 text-embedding references of oracle/kernel_bounds.py, which the GPU
tests compare the kernels with, against the CPU oracle.
"""
import ast
import glob
import os
import re
import types

import pytest
import torch

from f5_tts_b200 import _lib
from oracle import arch_options as OA
from oracle import kernel_bounds as KB
from oracle import mmdit as OM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "f5_tts_b200", "csrc")
F64 = torch.float64

# Launchers the hooks need not reach: the public C ABI tests (test_gpu_gemm_attn_exact.py and the attention tests)
# already launch them element by element through f5_gemm / f5_attention*, and fft_tables only builds constant tables.
ALLOWED_WITHOUT_HOOK = {"gemm_run", "attn_run", "fft_tables"}


def source(path):
    """C++ source without comments."""
    with open(path) as f:
        s = f.read()
    s = re.sub(r"/\*.*?\*/", " ", s, flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def launchers():
    """Functions declared in internal.h that take a cudaStream_t: every kernel launcher (run_*, gemm_run, attn_run,
    fft_tables)."""
    decls = re.findall(r"\bint\s+(\w+)\s*\(([^;{]*?)\)\s*;", source(os.path.join(CSRC, "internal.h")), flags=re.S)
    return {name for name, params in decls if "cudaStream_t" in params}


def hooks_source():
    return source(os.path.join(CSRC, "kernel_hooks.cu"))


def hook_definitions():
    return set(re.findall(r"^\s*(?:int|const char\*)\s+(f5k_\w+)\s*\(", hooks_source(), flags=re.M))


def gpu_tests():
    return {os.path.basename(p): open(p).read() for p in sorted(glob.glob(os.path.join(ROOT, "tests", "test_gpu_*.py")))}


def test_every_launcher_has_a_hook():
    found = launchers()
    assert {"run_row_norm", "run_istft", "run_mmdit_text_embed", "gemm_run"} <= found, f"parsed launchers: {found}"
    assert ALLOWED_WITHOUT_HOOK <= found, f"stale allow-list entries: {ALLOWED_WITHOUT_HOOK - found}"
    called = set(re.findall(r"\b(\w+)\s*\(", hooks_source()))
    missing = sorted(found - called - ALLOWED_WITHOUT_HOOK)
    assert not missing, f"launchers of internal.h that no hook in kernel_hooks.cu calls: {missing}"


def _int_list(node):
    try:
        v = ast.literal_eval(node)
    except ValueError:
        return []
    return [x for x in v if isinstance(x, int)] if isinstance(v, (list, tuple)) else []


def _row_norm_modes_from_tests():
    """Modes the GPU tests pass to the pass-through hook f5k_row_norm(mode, ...): a literal first argument of a direct
    call, or the values of a `mode` parametrization of a test that launches it."""
    modes = set()
    for name, text in gpu_tests().items():
        for fn in ast.walk(ast.parse(text)):
            if not isinstance(fn, ast.FunctionDef):
                continue
            launches = False
            for node in ast.walk(fn):
                if not isinstance(node, ast.Call):
                    continue
                f = node.func
                if isinstance(f, ast.Attribute) and f.attr == "f5k_row_norm":
                    launches = True
                    if node.args and isinstance(node.args[0], ast.Constant) and isinstance(node.args[0].value, int):
                        modes.add(node.args[0].value)
                if any(isinstance(a, ast.Constant) and a.value == "f5k_row_norm" for a in node.args):
                    launches = True
            if not launches:
                continue
            for dec in fn.decorator_list:
                if (isinstance(dec, ast.Call) and isinstance(dec.func, ast.Attribute) and dec.func.attr == "parametrize"
                        and dec.args and isinstance(dec.args[0], ast.Constant) and dec.args[0].value == "mode"):
                    modes.update(_int_list(dec.args[1]))
    return modes


def test_every_row_norm_mode_is_reached():
    """run_row_norm selects a kernel instantiation by its mode argument.  Each mode it accepts is reached either by a
    hook that fixes the mode (a literal argument) or through f5k_row_norm by a GPU test."""
    ops = source(os.path.join(CSRC, "ops.cu"))
    body = ops[ops.index("int run_row_norm("):]
    body = body[:body.index("\n}\n")]
    accepted = {int(m) for m in re.findall(r"\bmode\s*==\s*(\d+)", body)}
    assert accepted == {0, 1, 2, 3, 4}, f"modes run_row_norm accepts: {accepted}"
    fixed = {int(m) for m in re.findall(r"\brun_row_norm\s*\(\s*(\d+)\s*,", hooks_source())}
    passed = re.findall(r"\brun_row_norm\s*\(\s*([A-Za-z_]\w*)\s*,", hooks_source())
    assert passed == ["mode"], f"hooks passing a variable mode to run_row_norm: {passed}"
    reached = fixed | _row_norm_modes_from_tests()
    assert accepted <= reached, f"row norm modes no hook and no GPU test reaches: {sorted(accepted - reached)}"


def test_hook_symbols_are_listed_and_called():
    """Every f5k_* definition is in _lib.KERNEL_HOOK_SYMBOLS (which build() checks the library for) and the other way
    round, and every hook is called by at least one tests/test_gpu_*.py."""
    defined = hook_definitions()
    listed = set(_lib.KERNEL_HOOK_SYMBOLS)
    assert len(listed) == len(_lib.KERNEL_HOOK_SYMBOLS), "KERNEL_HOOK_SYMBOLS lists a symbol twice"
    assert defined - listed == set(), f"hooks missing from KERNEL_HOOK_SYMBOLS: {sorted(defined - listed)}"
    assert listed - defined == set(), f"KERNEL_HOOK_SYMBOLS entries kernel_hooks.cu does not define: {sorted(listed - defined)}"
    tests = "\n".join(gpu_tests().values())
    uncalled = sorted(h for h in defined if not re.search(rf"\b{h}\b", tests))
    assert not uncalled, f"hooks no tests/test_gpu_*.py calls: {uncalled}"


# ---------------------------------------------------------------------------------------------------------------------
# the float64 references of the GPU tests against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 1])
def test_avg_upsample_index_matches_oracle(seed):
    """kernel_bounds.avg_upsample_index picks the same rows as oracle/arch_options.average_upsample (dit.py:55-84) for
    T = 0 and 1, A < T, A = T, A a multiple of T, A with a remainder, A = 0, and fillers scattered through the text."""
    g = torch.Generator().manual_seed(seed)
    N, Td = 50, 6
    Ts = [0, 1, 30, 12, 12, 7, 5, 40]
    As = [50, 37, 11, 12, 36, 50, 0, 49]
    valid = torch.zeros(len(Ts), N, dtype=torch.bool)
    for b, T in enumerate(Ts):
        valid[b, torch.randperm(45, generator=g)[:T]] = True
    h = torch.randn(len(Ts), N, Td, generator=g, dtype=F64)
    want = OA.average_upsample(h, valid, torch.tensor(As))
    src = KB.avg_upsample_index(valid, As, N)
    got = torch.zeros_like(h)
    for b in range(len(Ts)):
        keep = src[b] >= 0
        got[b, keep] = h[b, src[b, keep]]
    assert torch.equal(got, want)
    assert (src >= 0).sum(1).tolist() == [0 if T == 0 else A for T, A in zip(Ts, As)]


@pytest.mark.parametrize("mask_padding", [0, 1])
@pytest.mark.parametrize("D", [128, 1024])
def test_mmdit_text_ref_matches_oracle(D, mask_padding):
    """kernel_bounds.mmdit_text_embed_ref against oracle/mmdit.text_embedding (fp32, both CFG variants) for 1100 text
    positions, past the 1023 clamp: the oracle's fp32 position table lies within pos_bound of the exact angle (as
    test_references_match_oracle shows for abs_pos_table) and its sum is rounded once, so it must lie within the
    reference's own bound."""
    g = torch.Generator().manual_seed(D)
    V, nt = 40, 1100
    table = torch.randn(V + 1, D, generator=g)
    ids = torch.randint(0, V, (3, nt), generator=g)
    ids[0, 0], ids[0, 1] = 0, V - 1
    ids[1] = -1
    ids[2, 700:] = -1
    sd = {"transformer.text_embed.text_embed.weight": table}
    cfg = types.SimpleNamespace(dim=D, text_mask_padding=mask_padding)
    ref, bound = KB.mmdit_text_embed_ref(table, ids, 6, mask_padding)
    want = torch.cat((OM.text_embedding(sd, cfg, ids, False), OM.text_embedding(sd, cfg, ids, True)), 0)
    KB.assert_within(want, ref, bound, f"oracle mmdit text_embedding D{D} mask_padding{mask_padding}")
