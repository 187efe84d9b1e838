"""CPU: the backbone operator's argument handling and the f5_forward C ABI block.

  * `time` is a number, a 0-d tensor, [1] or [b]; any other shape raises ValueError before anything reaches the GPU;
  * drop_audio_cond != drop_text still raises;
  * _lib.ForwardArgs has the field order, offsets and size of f5_forward_args in include/f5tts_b200.h (checked against
    the C compiler when one is installed);
  * the built library reports f5_version() 110 and exports f5_forward, f5_forward_workspace_bytes and
    f5_engine_graph_count.
"""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch

from f5_tts_b200 import _lib
from f5_tts_b200.model import forward_times

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ["B", "N", "nt", "x", "step_cond", "text", "duration", "time", "mode", "v_out", "use_graph", "reuse_text"]
OFFSETS = [0, 4, 8, 16, 24, 32, 40, 48, 56, 64, 72, 76]


def tiny_dit():
    import f5_tts_b200 as F5

    return F5.DiT(dim=128, depth=1, heads=2, ff_mult=2, text_dim=64, conv_layers=0, text_num_embeds=10)


def test_forward_times_shapes():
    assert torch.equal(forward_times(0.25, 3, "cpu"), torch.full((3,), 0.25))
    assert torch.equal(forward_times(1, 2, "cpu"), torch.ones(2))
    assert torch.equal(forward_times(torch.tensor(0.5), 3, "cpu"), torch.full((3,), 0.5))
    assert torch.equal(forward_times(torch.tensor([0.5]), 3, "cpu"), torch.full((3,), 0.5))
    t = torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64)
    got = forward_times(t, 3, "cpu")
    assert got.dtype == torch.float32 and got.is_contiguous() and torch.equal(got, t.float())
    assert torch.equal(forward_times(torch.tensor([0.7]), 1, "cpu"), torch.tensor([0.7]))


@pytest.mark.parametrize("bad", [torch.zeros(2), torch.zeros(4), torch.zeros(3, 1), torch.zeros(1, 3), torch.zeros(0),
                                 "0.5", None, [0.1, 0.2, 0.3]])
def test_forward_times_rejects(bad):
    with pytest.raises(ValueError):
        forward_times(bad, 3, "cpu")


def test_forward_rejects_time_shape_before_the_gpu():
    m = tiny_dit()
    x = torch.zeros(3, 16, 100)
    text = torch.zeros(3, 8, dtype=torch.long)
    for bad in (torch.zeros(2), torch.zeros(3, 1), torch.zeros(2, 2)):
        with pytest.raises(ValueError):
            m(x, x, text, bad)
    with pytest.raises(NotImplementedError):
        m(x, x, text, 0.5, drop_audio_cond=True, drop_text=False)


def test_forward_args_layout():
    assert [n for n, _ in _lib.ForwardArgs._fields_] == FIELDS
    assert [getattr(_lib.ForwardArgs, n).offset for n in FIELDS] == OFFSETS
    assert C.sizeof(_lib.ForwardArgs) == 80
    assert (_lib.FORWARD_COND, _lib.FORWARD_CFG, _lib.FORWARD_UNCOND) == (0, 1, 2)


def test_forward_args_layout_matches_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "off.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"f5tts_b200.h\"\nint main(void) {\n"
                   "  printf(\"%zu\", sizeof(f5_forward_args));\n"
                   + "".join(f"  printf(\" %zu\", offsetof(f5_forward_args, {n}));\n" for n in FIELDS)
                   + "  printf(\" %d %d %d\\n\", F5_FORWARD_COND, F5_FORWARD_CFG, F5_FORWARD_UNCOND);\n  return 0;\n}\n")
    exe = tmp_path / "off"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out == [80] + OFFSETS + [0, 1, 2]


def test_library_version_and_symbols():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built (run __graft_entry__.build())")
    lib = _lib.lib()
    assert lib.f5_version() == 110
    for n in ("f5_forward", "f5_forward_workspace_bytes", "f5_engine_graph_count"):
        assert hasattr(lib, n) and n in _lib.EXPORTED_SYMBOLS


def test_clear_cache_without_state():
    m = tiny_dit()
    assert m.clear_cache() is None
    m._op_states()[("k",)] = {"ws": None}
    assert m.clear_cache() is None
    assert m._op_states() == {}
