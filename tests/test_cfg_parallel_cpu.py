"""CPU: host logic of the CFG split (CFM.enable_cfg_parallel, f5_tts_b200/cfg_parallel.py, f5_sample_cfg_split).

  * a CPU device and an unknown device are refused;
  * a call without guidance (cfg_strength < 1e-5) and the backbone's forward stay on the primary, a guided call goes to
    the peer;
  * the new C entry points are declared, exported and bound, and the SampleArgs layout is the one f5_sample has;
  * the peer's replica is copied once per primary fingerprint and again when it changes;
  * load_model / F5TTS take the option.
"""
import ctypes as C
import inspect
import os

import pytest
import torch

import f5_tts_b200 as F5
from f5_tts_b200 import _lib, api, cfg_parallel, infer


def small_model():
    return F5.CFM(transformer=F5.DiT(dim=128, depth=1, heads=2, ff_mult=2, text_dim=64, conv_layers=1,
                                     text_num_embeds=10))


def test_cpu_and_unknown_devices_refused():
    model = small_model()
    for dev in ("cpu", torch.device("cpu"), "cuda:99", "not-a-device"):
        with pytest.raises(ValueError):
            model.enable_cfg_parallel(dev)
    assert model.transformer.cfg_peer is None
    if torch.cuda.device_count() == 0:
        with pytest.raises(ValueError):
            model.enable_cfg_parallel("cuda:0")


class RecordingPeer:
    def __init__(self):
        self.calls = 0

    def run(self, *a, **k):
        self.calls += 1


def test_only_guided_calls_split(monkeypatch):
    model = small_model()
    bb = model.transformer
    local = []
    monkeypatch.setattr(bb, "_run_local", lambda *a, **k: local.append(a[5] if len(a) > 5 else k["cfg_strength"]))
    peer = RecordingPeer()
    bb.cfg_peer = peer
    y = torch.zeros(1, 16, 100)
    sc = torch.zeros_like(y)
    text = torch.zeros(1, 4, dtype=torch.int64)
    bb.run(y, sc, text, [0.0, 1.0], None, 0.0)
    bb.run(y, sc, text, [0.0, 1.0], None, 5e-6)
    assert peer.calls == 0 and local == [0.0, 5e-6]
    bb.run(y, sc, text, [0.0, 1.0], None, 2.0)
    assert peer.calls == 1 and len(local) == 2
    # the operator seam asks for the raw backbone output: it stays on the primary
    bb(torch.zeros(1, 16, 100), torch.zeros(1, 16, 100), text, torch.tensor([0.5]), cfg_infer=True)
    assert peer.calls == 1 and len(local) == 3
    model.disable_cfg_parallel()
    assert bb.cfg_peer is None


def test_sample_cfg_zero_does_not_split(monkeypatch):
    """CFM.sample with cfg_strength = 0 reaches the backbone's run without the peer being asked."""
    model = small_model()
    bb = model.transformer
    seen = []
    monkeypatch.setattr(bb, "_run_local", lambda *a, **k: seen.append("local"))
    peer = RecordingPeer()
    bb.cfg_peer = peer
    monkeypatch.setattr(F5.model, "lens_to_mask", lambda t, length=None: torch.ones(t.shape[0], int(t.amax()),
                                                                                    dtype=torch.bool))
    model.sample(torch.zeros(1, 8, 100), torch.zeros(1, 4, dtype=torch.long), 20, steps=2, cfg_strength=0.0, seed=1)
    assert seen == ["local"] and peer.calls == 0
    model.sample(torch.zeros(1, 8, 100), torch.zeros(1, 4, dtype=torch.long), 20, steps=2, cfg_strength=2.0, seed=1)
    assert seen == ["local"] and peer.calls == 1


def test_header_declares_and_library_exports_the_split():
    src = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "include", "f5tts_b200.h")).read()
    for name in ("f5_sample_cfg_split", "f5_sample_cfg_split_workspace_bytes"):
        assert f"{name}(" in src and name in _lib.EXPORTED_SYMBOLS
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built (run __graft_entry__.build())")
    lib = _lib.lib()
    assert hasattr(lib, "f5_sample_cfg_split") and hasattr(lib, "f5_sample_cfg_split_workspace_bytes")
    assert lib.f5_version() >= 109
    assert lib.f5_sample_cfg_split.argtypes[1] is C.POINTER(_lib.SampleArgs)
    assert lib.f5_sample_cfg_split.argtypes[6] is C.POINTER(_lib.SampleArgs)


def test_sample_args_layout_unchanged():
    names = [n for n, _ in _lib.SampleArgs._fields_]
    assert names == ["B", "N", "nt", "steps", "text", "step_cond", "y", "duration", "t", "cfg_strength", "trajectory",
                     "use_graph", "v_out", "exact_varlen", "method"]
    assert C.sizeof(_lib.SampleArgs) == 96


def test_replica_follows_fingerprint(monkeypatch):
    copies, destroyed = [], []

    def fake_replicate(primary, backbone, device, stream):
        copies.append(primary["fp"])
        return {"handle": len(copies)}

    monkeypatch.setattr(cfg_parallel, "replicate", fake_replicate)
    monkeypatch.setattr(cfg_parallel, "destroy", lambda st: destroyed.append(st["handle"]))
    monkeypatch.setattr(cfg_parallel, "peer_device", lambda d: torch.device(d))
    peer = cfg_parallel.CfgPeer("cuda:1")

    class Stream:
        def synchronize(self):
            pass

    monkeypatch.setattr(peer, "stream", lambda: Stream())
    prim = torch.device("cuda", 0)
    st_a = {"fp": ("a",), "handle": "primary"}
    r1 = peer.engine(None, st_a, prim)
    r2 = peer.engine(None, st_a, prim)
    assert r1 is r2 and copies == [("a",)] and r1["fp"] == ("a",)
    st_b = {"fp": ("b",), "handle": "primary"}
    r3 = peer.engine(None, st_b, prim)
    assert copies == [("a",), ("b",)] and destroyed == [1] and r3["handle"] == 2 and peer.replications == 2
    # loopback: the primary's own engine, no copy
    assert peer.engine(None, st_b, torch.device("cuda", 1)) is st_b and len(copies) == 2
    peer._state = None  # a stand-in handle: nothing for the library to destroy


def test_enable_again_keeps_the_peer(monkeypatch):
    """Enabling the split again for the same device keeps the peer (weight copy, stream, workspaces); another device
    or disable_cfg_parallel drops it."""
    monkeypatch.setattr(cfg_parallel, "peer_device", lambda d: torch.device(d))
    model = small_model()
    p1 = model.enable_cfg_parallel("cuda:1")
    assert model.enable_cfg_parallel("cuda:1") is p1 and model.transformer.cfg_peer is p1
    p2 = model.enable_cfg_parallel("cuda:2")
    assert p2 is not p1 and p2.device == torch.device("cuda:2")
    model.disable_cfg_parallel()
    assert model.transformer.cfg_peer is None


def test_real_fingerprint_changes_on_weight_edit():
    """The primary's fingerprint (what the replica is keyed on) changes when a weight is edited in place."""
    bb = small_model().transformer
    fp = bb._fingerprint()
    with torch.no_grad():
        bb.proj_out.weight.add_(1.0)
    assert bb._fingerprint() != fp


def test_load_model_and_f5tts_take_the_option():
    assert inspect.signature(infer.load_model).parameters["cfg_parallel_device"].default is None
    assert inspect.signature(api.F5TTS.__init__).parameters["cfg_parallel_device"].default is None
