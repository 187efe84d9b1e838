"""One `CFM.sample` call on several GPUs: its samples cut into groups, one group per device
(`CFM.enable_sample_parallel`).

The samples of a batched call never interact: each sample's rows depend only on its own inputs and on the call's shapes.
So a call of B >= 2 samples can run as contiguous groups of samples, each an ordinary `f5_sample` call on its own engine,
stream and workspace, with no exchange inside the NFE loop, and each caller still gets what the one-GPU call returns
(DESIGN.md §4):

* faithful mode and `attn_mask_enabled`: a sample's rows depend on N (padded rows are computed, padded keys attended),
  so every group runs at the call's N and text length, and the result is the unsplit call's bit for bit;
* `exact_varlen`: every sample is computed as if it were alone, so a group runs at its own longest duration rounded up
  to `batching.bucket_frames`.  The mode does not define the rows at or past a sample's duration: the split writes zeros
  to those rows of the trajectory and leaves `y` there as it was.

Each entry of the device list is a `cfg_parallel.DevicePeer`: a replica of the packed weights (refreshed when the weights
change), its own stream, ordered against the caller's by events both ways, and its own workspace pool.  A device may be
named more than once and may be the model's own ("loopback": more streams and workspaces on one GPU), which is how one
GPU tests the split.  Whether it pays depends on the size of the call (DESIGN.md §8), which is why it is off by default.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib, cfg_parallel
from .batching import bucket_frames


def _fill(costs: list[int], cap: int) -> list[tuple[int, int]]:
    """Contiguous groups [(b0, b1)] of `costs`, each filled left to right while its sum stays within `cap`: the fewest
    groups any contiguous plan within `cap` can have."""
    groups, b0, acc = [], 0, 0
    for b, c in enumerate(costs):
        if b > b0 and acc + c > cap:
            groups.append((b0, b))
            b0, acc = b, 0
        acc += c
    groups.append((b0, len(costs)))
    return groups


def plan_sample_split(durations, N: int, exact_varlen: bool, n_devices: int) -> list[tuple[int, int, int]]:
    """Groups [(b0, b1, frames)] of a call's samples: contiguous, none empty, at most `n_devices`, chosen so that the
    largest group cost is as small as possible (with the fewest groups among such plans).  A sample costs N, or under
    `exact_varlen` its duration rounded up to `batching.bucket_frames`.  `frames` is the frame count the group runs at:
    N, or under `exact_varlen` its longest duration rounded up the same way, at most N."""
    N = int(N)
    durations = [min(max(int(d), 1), N) for d in durations]
    if not durations or int(n_devices) < 1:
        raise ValueError(f"nothing to split: {len(durations)} sample(s) over {n_devices} device(s)")
    costs = [bucket_frames(d) for d in durations] if exact_varlen else [N] * len(durations)
    lo, hi = max(costs), sum(costs)  # the optimum lies in between; _fill's group count falls as the cap grows
    while lo < hi:
        mid = (lo + hi) // 2
        if len(_fill(costs, mid)) <= n_devices:
            hi = mid
        else:
            lo = mid + 1
    return [(b0, b1, min(N, bucket_frames(max(durations[b0:b1]))) if exact_varlen else N)
            for b0, b1 in _fill(costs, lo)]


def split_devices(devices) -> list[torch.device]:
    """The CUDA devices of a sample split's device list; ValueError for an empty list, a CPU or an unknown device."""
    if devices is None or isinstance(devices, (str, int, torch.device)):
        raise ValueError(f"sample_parallel devices must be a list of CUDA devices, got {devices!r}")
    devs = [cfg_parallel.peer_device(d, "sample_parallel device") for d in devices]
    if not devs:
        raise ValueError("sample_parallel devices: the list is empty")
    return devs


class SampleSplit:
    """The devices of a sample split for one backbone: one `DevicePeer` per entry of the device list, in order."""

    def __init__(self, devices, copy_weights=None):
        self.peers = [cfg_parallel.DevicePeer(d, copy_weights) for d in split_devices(devices)]

    def run(self, backbone, y, step_cond, text, t_grid, duration, cfg_strength, trajectory, use_graph, exact_varlen,
            method):
        """`backbone.run` with the samples cut into groups (`plan_sample_split`), group g on peer g.  Returns when the
        launches are queued; the caller's stream is ordered after them."""
        from .model import _nfe

        assert y.is_contiguous() and step_cond.is_contiguous() and text.is_contiguous()
        assert y.dtype == torch.float32 and step_cond.dtype == torch.float32 and text.dtype == torch.int64
        B, N, mel = y.shape
        strict = bool(exact_varlen) and duration is not None  # what f5_sample_args.exact_varlen means
        lengths = [min(max(int(d), 0), N) for d in duration.tolist()] if strict else [N] * B
        groups = plan_sample_split(lengths, N, strict, len(self.peers))
        st0 = backbone.engine()
        dev0 = y.device
        caller = torch.cuda.current_stream(dev0)
        L = _lib.lib()
        steps = len(t_grid) - 1
        nfe = _nfe(steps, method)
        tg = (C.c_float * (steps + 1))(*[float(v) for v in t_grid])
        if strict and trajectory is not None:
            for b, d in enumerate(lengths):  # rows exact_varlen does not define: no group copies anything there
                if d < N:
                    trajectory[:, b, d:].zero_()
        # the groups start after the caller's prologue; each group's inputs are copied to its device on its stream
        ready = torch.cuda.Event()
        ready.record(caller)
        jobs = []  # [peer, workspace, b0, group y, group trajectory] of every group whose stream has work queued
        try:
            for peer, (b0, b1, n) in zip(self.peers, groups):
                ps = peer.stream()
                ps.wait_event(ready)
                job = [peer, None, b0, None, None]
                jobs.append(job)
                st = peer.engine(backbone, st0, dev0)
                with torch.cuda.device(peer.device), torch.cuda.stream(ps):
                    yg = torch.empty((b1 - b0, n, mel), dtype=torch.float32, device=peer.device)
                    yg.copy_(y[b0:b1, :n])
                    scg = torch.empty_like(yg)
                    scg.copy_(step_cond[b0:b1, :n])
                    textg = text[b0:b1].to(peer.device)
                    durg = duration[b0:b1].to(peer.device) if duration is not None else None
                    trg = None
                    if trajectory is not None:
                        trg = torch.empty((steps + 1, b1 - b0, n, mel), dtype=torch.float32, device=peer.device)
                job[3], job[4] = yg, trg
                need = L.f5_sample_workspace_bytes_nt(st["handle"], b1 - b0, n, text.shape[1], nfe, float(cfg_strength))
                job[1] = ws = peer._ws_acquire(need)
                a = _lib.sample_args(yg, scg, textg, durg, tg, steps, cfg_strength, trg, use_graph, exact_varlen, method)
                with torch.cuda.device(peer.device):
                    _lib.check(L.f5_sample(st["handle"], C.byref(a), ws.data_ptr(), ws.numel(), ps.cuda_stream),
                               "f5_sample")
            # results back into the caller's tensors, on each group's stream, once every group is queued
            for peer, _, b0, yg, trg in jobs:
                with torch.cuda.device(peer.device), torch.cuda.stream(peer.stream()):
                    for i in range(yg.shape[0]):
                        d = lengths[b0 + i]
                        y[b0 + i, :d].copy_(yg[i, :d])
                        if trg is not None:
                            trajectory[:, b0 + i, :d].copy_(trg[:, i, :d])
        finally:
            # also after a failure: the caller's stream (and whatever it frees next) waits for everything the groups
            # queued
            for peer, ws, *_ in jobs:
                done = torch.cuda.Event()
                done.record(peer.stream())
                caller.wait_event(done)
                if ws is not None:
                    peer._ws_release(ws)
