"""Concurrent `CFM.sample` calls merged into one engine call (`CFM.enable_batching`).

Servers, thread pools and Gradio apps call `sample()` from many threads at once, mostly with B = 1, and calls on one
stream run one after another.  This module lets such calls share engine calls.  Whether that pays depends on how well
one call fills the GPU: at cfg2-like lengths on an H100 it does not (DESIGN.md §8), which is why it is off by default.

Each caller still runs its own prologue (mel, tokens, duration, masks, seeded noise, time grid) and its own epilogue
(prompt copy, vocoder).  Only the `transformer.run(...)` call in between goes through a `SampleBatcher`: calls that agree
on the time grid, the CFG scale, the ODE method and the graph setting are stacked into one
`run(..., exact_varlen=True)`.  exact_varlen computes every sample exactly as if it were alone in the batch, so every
caller gets the final state and trajectory its own call would have produced.

Scheduling is leader / follower; the batcher owns no thread.  A call that finds the batcher idle leads: it runs at once,
so a lone caller waits for nothing.  Calls that arrive while a run is in flight queue up in arrival order.  When the
run's completion event has fired on the GPU, its leader hands the oldest queued call, with every compatible queued call
up to `max_batch` samples and `max_frames` padded rows, to the oldest call's thread, which leads the next run.  Runs go to
a stream kept for them, ordered after each caller's prologue by an event recorded on the caller's stream, and each
caller's stream waits on the run's completion event.  Callers' own streams never wait on other callers' runs, so a
caller's prologue synchronisation (`.tolist()`) does not queue behind a batch.
"""
from __future__ import annotations

import collections
import threading
from dataclasses import dataclass, field

import torch

FRAME_BUCKET = 128  # merged frame counts are padded to the GEMM row tile: samples start on a tile, fewer graph keys
DEFAULT_MAX_BATCH = 8
DEFAULT_MAX_FRAMES = 8192  # samples x padded frames of one merged run (bounds its workspace and trajectory)


def bucket_frames(n: int) -> int:
    return -(-int(n) // FRAME_BUCKET) * FRAME_BUCKET


def plan_batch(shapes) -> tuple[int, list[int]]:
    """(padded frame count, first row of each call) for calls of shapes [(B, N), ...] stacked in order."""
    offsets, b0 = [], 0
    for b, _ in shapes:
        offsets.append(b0)
        b0 += b
    return bucket_frames(max(n for _, n in shapes)), offsets


def mergeable(kind: str, y: torch.Tensor, text: torch.Tensor, duration, exact_varlen: bool) -> bool:
    """Whether a call may share an engine call with others without changing its answer.

    B > 1 without exact_varlen (the reference's batched semantics) attends its own padded keys by design: it runs alone.
    An MMDiT call of one sample whose text holds -1 padding attends those text keys when alone, while exact_varlen masks
    them (the text length of a sample is its count of ids other than -1): it runs alone too."""
    if y.shape[0] > 1:
        return bool(exact_varlen) and duration is not None
    if kind == "MMDiT":
        return not bool((text == -1).any())
    return True


def select_batch(queue: list, max_batch: int, max_frames: int) -> list:
    """Removes and returns the next run's calls from `queue` (arrival order): the oldest call, then every later call with
    its key that keeps the run within `max_batch` samples and `max_frames` padded rows.  The oldest call always goes,
    even when it alone exceeds a cap."""
    if not queue:
        return []
    key = queue[0].key
    chosen, rest, b, n = [], [], 0, 0
    for c in queue:
        nb, nn_ = b + c.B, max(n, c.N)
        if c.key == key and (not chosen or (nb <= max_batch and nb * bucket_frames(nn_) <= max_frames)):
            chosen.append(c)
            b, n = nb, nn_
        else:
            rest.append(c)
    queue[:] = rest
    return chosen


def stack_calls(calls: list, n_pad: int, offsets: list[int]):
    """Merged (y, step_cond, text, duration int32, trajectory) of `calls`: rows zero-padded to n_pad frames, text padded
    with -1 to the longest, each sample's duration its own (a call without durations: its frame count)."""
    c0 = calls[0]
    B = offsets[-1] + calls[-1].B
    mel, dev = c0.y.shape[-1], c0.y.device
    nt = max(c.text.shape[1] for c in calls)
    y = torch.zeros((B, n_pad, mel), dtype=c0.y.dtype, device=dev)
    step_cond = torch.zeros((B, n_pad, mel), dtype=c0.step_cond.dtype, device=dev)
    text = torch.full((B, nt), -1, dtype=torch.int64, device=dev)
    duration = torch.empty((B,), dtype=torch.int32, device=dev)
    for c, b0 in zip(calls, offsets):
        rows = slice(b0, b0 + c.B)
        y[rows, : c.N] = c.y
        step_cond[rows, : c.N] = c.step_cond
        text[rows, : c.text.shape[1]] = c.text
        if c.duration is None:
            duration[rows] = c.N
        else:
            duration[rows] = c.duration
    trajectory = None
    if any(c.trajectory is not None for c in calls):
        trajectory = torch.empty((len(c0.t_grid), B, n_pad, mel), dtype=torch.float32, device=dev)
    return y, step_cond, text, duration, trajectory


def split_results(calls: list, offsets: list[int], y: torch.Tensor, trajectory) -> None:
    """Copies each call's rows of the merged final state and trajectory into the caller's own tensors."""
    for c, b0 in zip(calls, offsets):
        c.y.copy_(y[b0: b0 + c.B, : c.N])
        if c.trajectory is not None:
            c.trajectory.copy_(trajectory[:, b0: b0 + c.B, : c.N])


@dataclass
class BatchStats:
    """Counters of one batcher, for operators and tests.  Updated under the batcher's lock."""

    calls: int = 0  # calls served by merged-capable runs
    bypassed: int = 0  # calls that could not merge and ran alone on the caller's stream
    runs: int = 0  # engine runs the served calls took (failed runs included)
    samples: int = 0  # samples over those runs
    batch_sizes: collections.Counter = field(default_factory=collections.Counter)  # calls per run -> runs
    handoffs: int = 0  # runs started by a queued call when the previous run completed
    handoff_gap_ms: float = 0.0  # GPU idle time over those hand-offs: previous run's end to this run's first launch


_streams: dict = {}
_streams_lock = threading.Lock()


def _batch_stream(dev: torch.device) -> torch.cuda.Stream:
    """The stream merged runs go to on `dev`, one per process: a batcher enabled again, or another model's, reuses it,
    and with it the engine workspace pooled for that stream and the CUDA graphs captured on that workspace."""
    with _streams_lock:
        if dev not in _streams:
            _streams[dev] = torch.cuda.Stream(dev)
        return _streams[dev]


class _Call:
    """One caller's engine call, with the arguments `transformer.run` takes."""

    def __init__(self, y, step_cond, text, t_grid, duration, cfg_strength, trajectory, use_graph, exact_varlen, method):
        self.y, self.step_cond, self.text, self.duration, self.trajectory = y, step_cond, text, duration, trajectory
        self.t_grid, self.cfg_strength, self.use_graph, self.method = list(t_grid), cfg_strength, use_graph, method
        self.exact_varlen = exact_varlen
        self.B, self.N = int(y.shape[0]), int(y.shape[1])
        # the merge key (the batcher belongs to one model): what every sample of one engine call must share
        self.key = (y.device, tuple(float(v) for v in t_grid), float(cfg_strength), method, bool(use_graph))
        self.ready = None  # event on the caller's stream after its prologue
        self.done = None  # completion event of the run that served the call
        self.error = None
        self.lead_batch = None  # set when this call's thread is to lead the next run
        self.wake = threading.Event()


class SampleBatcher:
    """Merges concurrent engine calls of one model (see the module docstring).  `run` takes `transformer.run`'s
    arguments and returns when the call's rows are in its `y` and `trajectory`."""

    def __init__(self, transformer, max_batch: int = DEFAULT_MAX_BATCH, max_frames: int = DEFAULT_MAX_FRAMES):
        if int(max_batch) < 1 or int(max_frames) < FRAME_BUCKET:
            raise ValueError(f"max_batch must be >= 1 and max_frames >= {FRAME_BUCKET}, got {max_batch}, {max_frames}")
        self.transformer = transformer
        self.max_batch, self.max_frames = int(max_batch), int(max_frames)
        self.stats = BatchStats()
        self._lock = threading.Lock()
        self._queue: list[_Call] = []
        self._busy = False
        self._last_done = None  # completion event of the previous run (idle-gap accounting)

    def run(self, y, step_cond, text, t_grid, duration, cfg_strength, trajectory=None, use_graph=True,
            exact_varlen=False, method="euler"):
        if not mergeable(self.transformer.KIND, y, text, duration, exact_varlen):
            with self._lock:
                self.stats.bypassed += 1
            return self.transformer.run(y, step_cond, text, t_grid, duration, cfg_strength, trajectory=trajectory,
                                        use_graph=use_graph, exact_varlen=exact_varlen, method=method)
        call = _Call(y, step_cond, text, t_grid, duration, cfg_strength, trajectory, use_graph, exact_varlen, method)
        if y.is_cuda:
            call.ready = torch.cuda.Event()
            call.ready.record(torch.cuda.current_stream(y.device))
        with self._lock:
            self.stats.calls += 1
            lead = not self._busy
            if lead:
                self._busy = True
            else:
                self._queue.append(call)
        if lead:
            self._lead([call], handoff=False)
        else:
            call.wake.wait()
            if call.lead_batch is not None:
                self._lead(call.lead_batch, handoff=True)
        if call.error is not None:
            raise call.error
        if call.done is not None:
            torch.cuda.current_stream(y.device).wait_event(call.done)

    # -- leader side ------------------------------------------------------------------------------------------------
    def _lead(self, batch: list, handoff: bool) -> None:
        done, error = None, None
        try:
            done = self._execute(batch, handoff)
        except BaseException as e:  # noqa: BLE001 — the error belongs to every caller of the run; the batcher goes on
            error = e
        finally:
            with self._lock:
                nxt = select_batch(self._queue, self.max_batch, self.max_frames)
                if not nxt:
                    self._busy = False
            for c in batch:
                c.done, c.error = done, error
                c.wake.set()
            if nxt:
                nxt[0].lead_batch = nxt
                nxt[0].wake.set()

    def _execute(self, batch: list, handoff: bool):
        """Runs one engine call for `batch` and waits for it to complete.  Returns its completion event (None for host
        tensors, which only a stand-in transformer accepts)."""
        dev = batch[0].y.device
        if dev.type != "cuda":
            try:
                self._run(batch)
            finally:
                self._count(batch, handoff, 0.0)
            return None
        stream = _batch_stream(dev)
        start, done = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.device(dev), torch.cuda.stream(stream), torch.inference_mode():
            for c in batch:
                stream.wait_event(c.ready)
            start.record(stream)
            try:
                self._run(batch)
            finally:  # also after a failed launch: nothing of the run may still use the callers' tensors
                done.record(stream)
                done.synchronize()
                prev, self._last_done = self._last_done, done
                self._count(batch, handoff, prev.elapsed_time(start) if handoff and prev is not None else 0.0)
        return done

    def _run(self, batch: list) -> None:
        c0 = batch[0]
        kw = dict(use_graph=c0.use_graph, method=c0.method)
        if len(batch) == 1:  # the call exactly as the caller made it
            self.transformer.run(c0.y, c0.step_cond, c0.text, c0.t_grid, c0.duration, c0.cfg_strength,
                                 trajectory=c0.trajectory, exact_varlen=c0.exact_varlen, **kw)
            return
        n_pad, offsets = plan_batch([(c.B, c.N) for c in batch])
        y, step_cond, text, duration, trajectory = stack_calls(batch, n_pad, offsets)
        self.transformer.run(y, step_cond, text, c0.t_grid, duration, c0.cfg_strength, trajectory=trajectory,
                             exact_varlen=True, **kw)
        split_results(batch, offsets, y, trajectory)

    def _count(self, batch: list, handoff: bool, gap_ms: float) -> None:
        with self._lock:
            s = self.stats
            s.runs += 1
            s.samples += sum(c.B for c in batch)
            s.batch_sizes[len(batch)] += 1
            if handoff:
                s.handoffs += 1
                s.handoff_gap_ms += gap_ms
