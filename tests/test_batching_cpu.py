"""CPU: the host side of merging concurrent sample() calls (f5_tts_b200/batching.py): the merge key and the bypass rules,
the 128-frame padding plan, the choice of the next run from the queue under the caps, stacking the callers' tensors
and splitting the result back, and the leader / follower scheduling with a stand-in transformer: queued calls merge
into one run, each caller gets its own rows, an error in a run reaches exactly that run's callers and the batcher
keeps serving."""
import threading
from types import SimpleNamespace

import pytest
import torch

import f5_tts_b200 as F5
from f5_tts_b200 import batching as BT


def call(B=1, N=100, nt=10, grid=(0.0, 0.5, 1.0), cfg=2.0, method="euler", graph=True, duration=None, varlen=False,
         device="cpu", seed=0):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(B, N, 100, generator=g, device="cpu").to(device)
    return BT._Call(y, torch.randn(B, N, 100, generator=g).to(device), torch.randint(0, 50, (B, nt), generator=g),
                    list(grid), duration, cfg, torch.empty(len(grid), B, N, 100), graph, varlen, method)


def test_bucket_and_plan():
    assert [BT.bucket_frames(n) for n in (1, 127, 128, 129, 938, 1024)] == [128, 128, 128, 256, 1024, 1024]
    assert BT.plan_batch([(1, 403), (2, 230), (1, 150)]) == (512, [0, 1, 3])
    assert BT.plan_batch([(1, 256)]) == (256, [0])


def test_merge_key():
    base = call()
    assert call(seed=1, N=300, nt=40).key == base.key  # shapes and contents do not enter the key
    for other in (call(grid=(0.0, 0.25, 1.0)), call(grid=(0.0, 0.5, 0.75, 1.0)), call(cfg=1.5), call(method="midpoint"),
                  call(graph=False)):
        assert other.key != base.key
    assert call(device="meta").key != base.key


def test_bypass_rules():
    y1, y2 = torch.zeros(1, 10, 100), torch.zeros(2, 10, 100)
    text, padded = torch.zeros(1, 5, dtype=torch.long), torch.tensor([[3, 4, -1]])
    dur = torch.tensor([10, 7], dtype=torch.int32)
    for kind in ("DiT", "UNetT", "MMDiT"):
        assert BT.mergeable(kind, y1, text, None, False)
        assert not BT.mergeable(kind, y2, text.expand(2, -1), dur, False), "a B > 1 faithful call runs alone"
        assert BT.mergeable(kind, y2, text.expand(2, -1), dur, True)
    # one MMDiT sample with -1 text padding attends those keys alone; exact_varlen would not
    assert not BT.mergeable("MMDiT", y1, padded, None, False)
    assert BT.mergeable("DiT", y1, padded, None, False) and BT.mergeable("UNetT", y1, padded, None, False)


def test_select_batch_order_key_and_caps():
    a, b, c = call(N=400), call(N=200, cfg=1.5), call(N=300)
    d, e = call(B=3, N=900), call(N=120)
    q = [a, b, c, d, e]
    # a's key: a, c, then d would make 5 x 1024 > 4096 rows, e fits; b keeps its place for the next run
    assert BT.select_batch(q, max_batch=8, max_frames=4096) == [a, c, e]
    assert q == [b, d]
    assert BT.select_batch(q, max_batch=8, max_frames=4096) == [b]
    assert BT.select_batch(q, max_batch=2, max_frames=128) == [d], "the oldest call goes even above the caps"
    assert q == [] and BT.select_batch(q, 8, 4096) == []
    q = [call(), call(), call(), call()]
    assert len(BT.select_batch(q, max_batch=3, max_frames=1 << 20)) == 3 and len(q) == 1


def test_stack_and_split():
    cs = [call(N=403, nt=40, seed=1), call(B=2, N=230, nt=33, duration=torch.tensor([230, 121], dtype=torch.int32),
                                          varlen=True, seed=2), call(N=150, nt=17, seed=3)]
    n_pad, offsets = BT.plan_batch([(c.B, c.N) for c in cs])
    y, sc, text, dur, traj = BT.stack_calls(cs, n_pad, offsets)
    assert y.shape == sc.shape == (4, 512, 100) and text.shape == (4, 40) and traj.shape == (3, 4, 512, 100)
    assert dur.dtype == torch.int32 and dur.tolist() == [403, 230, 121, 150]
    for c, b0 in zip(cs, offsets):
        assert torch.equal(y[b0: b0 + c.B, : c.N], c.y) and not y[b0: b0 + c.B, c.N:].any()
        assert torch.equal(sc[b0: b0 + c.B, : c.N], c.step_cond) and not sc[b0: b0 + c.B, c.N:].any()
        assert torch.equal(text[b0: b0 + c.B, : c.text.shape[1]], c.text)
        assert (text[b0: b0 + c.B, c.text.shape[1]:] == -1).all()
    y_out, traj_out = torch.randn_like(y), torch.randn_like(traj)
    BT.split_results(cs, offsets, y_out, traj_out)
    for c, b0 in zip(cs, offsets):
        assert torch.equal(c.y, y_out[b0: b0 + c.B, : c.N])
        assert torch.equal(c.trajectory, traj_out[:, b0: b0 + c.B, : c.N])


class StandIn:
    """transformer.run with a per-sample answer that does not depend on the batch: y[b, :d] = step_cond * cfg + steps,
    trajectory[k] = k * y.  Runs whose text holds the id 99 raise.  The first run waits until `gate` is set."""

    KIND = "DiT"

    def __init__(self):
        self.runs, self.gate = [], threading.Event()

    def run(self, y, step_cond, text, t_grid, duration, cfg_strength, trajectory=None, use_graph=True,
            exact_varlen=False, method="euler"):
        if not self.runs:
            assert self.gate.wait(10)
        self.runs.append((y.shape[0], y.shape[1], exact_varlen))
        if bool((text == 99).any()):
            raise RuntimeError("engine failure")
        lens = duration.tolist() if duration is not None else [y.shape[1]] * y.shape[0]
        for b, d in enumerate(lens):
            y[b, :d] = step_cond[b, :d] * cfg_strength + len(t_grid)
            if trajectory is not None:
                for k in range(len(t_grid)):
                    trajectory[k, b, :d] = k * y[b, :d]


def solo(c):
    y = c.step_cond * c.cfg_strength + len(c.t_grid)
    return y, torch.stack([k * y for k in range(len(c.t_grid))])


def test_leader_follower_merges_and_isolates_errors():
    t = StandIn()
    batcher = BT.SampleBatcher(t, max_batch=8, max_frames=4096)
    first = call(N=64, seed=9)
    queued = [call(N=100 + 37 * i, nt=5 + i, seed=10 + i) for i in range(4)] + [call(cfg=1.0, seed=20)]
    failing = [call(N=90, grid=(0.0, 0.3, 1.0), seed=30), call(N=60, grid=(0.0, 0.3, 1.0), seed=31)]
    failing[0].text[0, 0] = 99  # the run of these two fails
    errors = {}

    def go(c):
        try:
            batcher.run(c.y, c.step_cond, c.text, c.t_grid, c.duration, c.cfg_strength, trajectory=c.trajectory,
                        use_graph=c.use_graph, exact_varlen=c.exact_varlen, method=c.method)
        except Exception as e:  # noqa: BLE001
            errors[id(c)] = e

    lead = threading.Thread(target=go, args=(first,))
    lead.start()
    for _ in range(200):
        if batcher._busy:
            break
        threading.Event().wait(0.01)
    rest = [threading.Thread(target=go, args=(c,)) for c in queued + failing]
    for th in rest:
        th.start()
    for _ in range(500):
        if batcher.stats.calls == 1 + len(queued) + len(failing):
            break
        threading.Event().wait(0.01)
    t.gate.set()
    for th in [lead] + rest:
        th.join(20)
    assert not batcher._busy and not batcher._queue
    assert set(errors) == {id(c) for c in failing}, [repr(e) for e in errors.values()]
    assert all(str(e) == "engine failure" for e in errors.values())
    s = batcher.stats
    assert s.calls == 8 and s.runs == 4 and s.handoffs == 3 and s.bypassed == 0
    assert s.batch_sizes == {1: 2, 4: 1, 2: 1}
    assert t.runs[0] == (1, 64, False) and (4, 256, True) in t.runs  # 100..211 frames padded to 256
    for c in [first] + queued:
        want_y, want_traj = solo(c)
        assert torch.equal(c.y, want_y) and torch.equal(c.trajectory, want_traj)
    # the batcher keeps serving after a failed run: a lone call runs at once
    c = call(seed=40)
    batcher.run(c.y, c.step_cond, c.text, c.t_grid, None, c.cfg_strength, trajectory=c.trajectory)
    assert batcher.stats.runs == 5 and torch.equal(c.y, solo(c)[0])


def test_cfm_switches_and_bypass():
    model = F5.CFM(transformer=F5.DiT(dim=128, depth=2, heads=2, text_dim=64, conv_layers=1))
    assert model.batcher is None
    stats = model.enable_batching(max_batch=4, max_frames=2048)
    assert isinstance(stats, BT.BatchStats) and model.batcher.stats is stats
    assert (model.batcher.max_batch, model.batcher.max_frames) == (4, 2048)
    model.disable_batching()
    assert model.batcher is None
    with pytest.raises(ValueError):
        model.enable_batching(max_batch=0)
    # a call that cannot merge goes straight to the transformer, on the caller's thread
    seen = []
    batcher = BT.SampleBatcher(SimpleNamespace(KIND="DiT", run=lambda *a, **k: seen.append(k["exact_varlen"])))
    batcher.run(torch.zeros(2, 10, 100), torch.zeros(2, 10, 100), torch.zeros(2, 3, dtype=torch.long), [0.0, 1.0],
                torch.tensor([10, 8], dtype=torch.int32), 2.0, exact_varlen=False)
    assert seen == [False] and batcher.stats.bypassed == 1 and batcher.stats.calls == 0
