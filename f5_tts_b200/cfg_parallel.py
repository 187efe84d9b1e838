"""One `CFM.sample` call on two GPUs: the conditional and unconditional CFG halves on separate devices
(`CFM.enable_cfg_parallel`).

With classifier-free guidance on, every backbone evaluation runs two independent problems stacked on the batch axis:
the conditional rows and the unconditional rows.  They meet only in the update g = pred + (pred - null) * cfg.  A split
call runs the conditional half on the model's own device and the unconditional half on a peer device, and after every
evaluation each device copies the other's half of the flow (B * N * mel fp32 values) before the unchanged update kernel
runs on both (f5_sample_cfg_split in include/f5tts_b200.h; the ordering argument is in DESIGN.md §4).  Each caller gets
bit for bit what the unsplit call returns.

The peer holds a replica of the backbone's packed operands, copied again whenever the primary's weight fingerprint
changes, its own stream and its own workspace pool.  The peer may be the model's own device ("loopback": two workspaces
on one GPU, the same engine); that runs the same code path and is how one GPU tests it.  Whether the pair is faster than
one GPU depends on the size of the call (DESIGN.md §8), which is why it is off by default.

`DevicePeer` is that per-device state on its own; the sample split (`sample_parallel.py`) runs its groups on it too.
"""
from __future__ import annotations

import ctypes as C
import threading

import torch

from . import _lib


def peer_device(device, what: str = "cfg_parallel device") -> torch.device:
    """The CUDA device `device` names; ValueError for a CPU or unknown device.  `what` names the argument in the
    message."""
    try:
        dev = torch.device(device)
    except (RuntimeError, TypeError) as e:
        raise ValueError(f"{what} {device!r}: {e}") from None
    if dev.type != "cuda":
        raise ValueError(f"{what} {device!r} is not a CUDA device: split calls run on a GPU")
    count = torch.cuda.device_count() if torch.cuda.is_available() else 0
    index = dev.index if dev.index is not None else (torch.cuda.current_device() if count else 0)
    if index >= count:
        raise ValueError(f"{what} {device!r}: this process sees {count} CUDA device(s)")
    return torch.device("cuda", index)


def replicate(primary: dict, backbone, device: torch.device, stream: torch.cuda.Stream) -> dict:
    """An engine over a copy of the primary engine's packed operands on `device`; complete when this returns.  The copies
    are allocated on `stream` (the peer's), so when a later replica replaces them their memory is reused in that
    stream's order, after the peer's last use."""
    from .weights import engine_from_packed

    src = next(iter(primary["keep"].values())).device
    with torch.cuda.device(device), torch.cuda.stream(stream):
        T = {k: v.to(device, copy=True) for k, v in primary["keep"].items()}
    torch.cuda.synchronize(src)
    torch.cuda.synchronize(device)
    return engine_from_packed(backbone, T)


def destroy(state: dict) -> None:
    _lib.lib().f5_engine_destroy(state["handle"])


class DevicePeer:
    """One device's side of split calls for one backbone: the device, the replica engine, a stream, a workspace pool.

    `copy_weights`: None (default) replicates the weights when the peer is another device and runs loopback on the
    primary's own engine; True replicates them even on the primary's device (two engines on one GPU, which exercises
    the replica path where only one GPU is available)."""

    def __init__(self, device, copy_weights=None):
        self.device = peer_device(device)
        self.copy_weights = copy_weights
        self._lock = threading.Lock()
        self._stream_lock = threading.Lock()
        self._state = None  # replica engine state {"handle", "keep", ..., "fp"}; None until the first split call
        self._stream = None
        self._ws_free: list = []  # peer workspaces not in use by a call, all allocated on the peer stream
        self.replications = 0  # replicas made so far (one per primary fingerprint the peer has served)

    def engine(self, backbone, primary: dict, primary_device: torch.device) -> dict:
        """The engine the peer's work runs on: the primary's own for loopback, else the replica, copied again when the
        primary's fingerprint (the `fp` its engine state was packed at) has changed."""
        if primary_device == self.device and not self.copy_weights:
            return primary
        with self._lock:
            st = self._state
            if st is None or st["fp"] != primary["fp"]:
                if st is not None:
                    self._state = None
                    self.stream().synchronize()  # the old replica's last split call is done with it
                    destroy(st)
                st = replicate(primary, backbone, self.device, self.stream())
                st["fp"] = primary["fp"]
                self._state = st
                self.replications += 1
            return st

    def stream(self) -> torch.cuda.Stream:
        with self._stream_lock:
            if self._stream is None:
                self._stream = torch.cuda.Stream(self.device)
            return self._stream

    def _ws_acquire(self, nbytes: int) -> torch.Tensor:
        """A peer workspace of at least `nbytes`, allocated on the peer stream: reuse (by later calls, or by the
        allocator after the pool lets a buffer go) is ordered after the peer's work on it.  A finished call returns its
        buffer, so the next call reuses the address and hits the peer engine's graph cache."""
        with self._lock:
            for i, ws in enumerate(self._ws_free):
                if ws.numel() >= nbytes:
                    return self._ws_free.pop(i)
            self._ws_free.clear()  # too small for the current shapes: let them go
        with torch.cuda.device(self.device), torch.cuda.stream(self.stream()):
            return torch.empty(int(nbytes * 1.05) + 4096, dtype=torch.uint8, device=self.device)

    def _ws_release(self, ws: torch.Tensor) -> None:
        with self._lock:
            self._ws_free.append(ws)

    def __del__(self):
        st = getattr(self, "_state", None)
        if st is not None:
            try:
                destroy(st)
            except Exception:
                pass


class CfgPeer(DevicePeer):
    """The peer side of CFG-split calls: a `DevicePeer` that runs the unconditional half."""

    def run(self, backbone, y, step_cond, text, t_grid, duration, cfg_strength, trajectory, use_graph, exact_varlen,
            method):
        """`backbone.run` with the unconditional half on the peer device.  Returns when the launches are queued; the
        caller's stream is ordered after them."""
        from .model import _nfe

        st0 = backbone.engine()
        dev0 = y.device
        st1 = self.engine(backbone, st0, dev0)
        L = _lib.lib()
        steps = len(t_grid) - 1
        assert y.is_contiguous() and step_cond.is_contiguous() and text.is_contiguous()
        assert y.dtype == torch.float32 and step_cond.dtype == torch.float32 and text.dtype == torch.int64
        B, N, _ = y.shape
        nt = text.shape[1]
        need = L.f5_sample_cfg_split_workspace_bytes(st0["handle"], B, N, nt, _nfe(steps, method))
        caller = torch.cuda.current_stream(dev0)
        ps = self.stream()
        # the peer's stream starts after the caller's prologue; the inputs the peer half reads are copied to its device
        ready = torch.cuda.Event()
        ready.record(caller)
        ps.wait_event(ready)
        with torch.cuda.device(self.device), torch.cuda.stream(ps):
            y1 = torch.empty_like(y, device=self.device)  # a state of its own, also for loopback
            y1.copy_(y)
            sc1, text1 = step_cond.to(self.device), text.to(self.device)
            dur1 = duration.to(self.device) if duration is not None else None
        tg = (C.c_float * (steps + 1))(*[float(v) for v in t_grid])
        a0 = _lib.sample_args(y, step_cond, text, duration, tg, steps, cfg_strength, trajectory, use_graph,
                              exact_varlen, method)
        a1 = _lib.sample_args(y1, sc1, text1, dur1, tg, steps, cfg_strength, None, use_graph, exact_varlen, method)
        ws0 = backbone._ws_acquire(need, dev0, caller.cuda_stream)
        ws1 = self._ws_acquire(need)
        try:
            with torch.cuda.device(dev0):
                _lib.check(L.f5_sample_cfg_split(st0["handle"], C.byref(a0), ws0.data_ptr(), ws0.numel(),
                                                 caller.cuda_stream, st1["handle"], C.byref(a1), ws1.data_ptr(),
                                                 ws1.numel(), ps.cuda_stream), "f5_sample_cfg_split")
        finally:
            # also after a failure: the caller's stream (and whatever it frees next) waits for everything the peer queued
            done = torch.cuda.Event()
            done.record(ps)
            caller.wait_event(done)
            self._ws_release(ws1)
            backbone._ws_release(ws0, dev0, caller.cuda_stream)
