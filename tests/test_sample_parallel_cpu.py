"""CPU: host logic of the sample split (CFM.enable_sample_parallel, f5_tts_b200/sample_parallel.py).

  * the plan: every sample in exactly one group, groups contiguous and never more than the devices or the samples, the
    largest group cost optimal (brute force over small cases), the frame count smaller than N only under exact_varlen;
  * refused arguments: an empty list, a CPU or unknown device, a bare device instead of a list, both splits at once;
  * which calls split: B >= 2 calls (cfg_strength 0 included, merged runs of enable_batching included); B = 1 calls,
    the backbone's forward and calls with the split off stay local;
  * enabling again with the same list keeps the peers; load_model / F5TTS take the option.
"""
import inspect
import itertools
import random

import pytest
import torch

import f5_tts_b200 as F5
from f5_tts_b200 import api, batching, cfg_parallel, infer, sample_parallel
from f5_tts_b200.batching import bucket_frames
from f5_tts_b200.sample_parallel import plan_sample_split


def small_model():
    return F5.CFM(transformer=F5.DiT(dim=128, depth=1, heads=2, ff_mult=2, text_dim=64, conv_layers=1,
                                     text_num_embeds=10))


# ---------------------------------------------------------------------------------------------------------------------
# the plan
# ---------------------------------------------------------------------------------------------------------------------
def costs_of(durations, N, exact_varlen):
    return [bucket_frames(d) for d in durations] if exact_varlen else [N] * len(durations)


def brute_force_best(costs, n_devices):
    """The smallest largest-group cost over every contiguous plan of at most n_devices groups."""
    B = len(costs)
    best = None
    for k in range(1, min(B, n_devices) + 1):
        for cuts in itertools.combinations(range(1, B), k - 1):
            edges = (0, *cuts, B)
            worst = max(sum(costs[a:b]) for a, b in zip(edges, edges[1:]))
            best = worst if best is None else min(best, worst)
    return best


def check_plan(durations, N, exact_varlen, n_devices):
    plan = plan_sample_split(durations, N, exact_varlen, n_devices)
    B = len(durations)
    assert 1 <= len(plan) <= min(B, n_devices)
    assert plan[0][0] == 0 and plan[-1][1] == B
    for (a0, a1, _), (b0, _, _) in zip(plan, plan[1:]):
        assert a1 == b0  # contiguous, so every sample is in exactly one group
    costs = costs_of(durations, N, exact_varlen)
    for b0, b1, frames in plan:
        assert b0 < b1
        if exact_varlen:
            assert frames == min(N, bucket_frames(max(durations[b0:b1])))
            assert frames >= max(durations[b0:b1])
        else:
            assert frames == N
    assert max(sum(costs[b0:b1]) for b0, b1, _ in plan) == brute_force_best(costs, n_devices)
    return plan


@pytest.mark.parametrize("exact_varlen", [False, True])
def test_plan_random_small_cases_are_optimal(exact_varlen):
    rng = random.Random(11)
    for _ in range(400):
        B = rng.randint(1, 9)
        durations = [rng.randint(1, 1900) for _ in range(B)]
        N = max(durations) + rng.choice([0, 0, 5, 130])
        check_plan(durations, N, exact_varlen, rng.randint(1, 10))


def test_plan_faithful_balances_counts():
    assert plan_sample_split([500] * 5, 938, False, 2) == [(0, 3, 938), (3, 5, 938)]
    assert plan_sample_split([500] * 5, 938, False, 3) == [(0, 2, 938), (2, 4, 938), (4, 5, 938)]
    assert plan_sample_split([938] * 8, 938, False, 8) == [(b, b + 1, 938) for b in range(8)]


def test_plan_more_devices_than_samples():
    assert plan_sample_split([100, 200], 200, False, 5) == [(0, 1, 200), (1, 2, 200)]
    assert plan_sample_split([100, 200], 200, True, 5) == [(0, 1, 128), (1, 2, 200)]
    assert plan_sample_split([300], 300, True, 4) == [(0, 1, 300)]


def test_plan_exact_varlen_balances_bucketed_durations():
    frames = [469, 670, 871, 1072, 1272, 1473, 1674, 1875]  # cfg3
    plan = check_plan(frames, 1875, True, 2)
    assert plan == [(0, 5, 1280), (5, 8, 1875)]  # costs 512+768+896+1152+1280 = 4608 against 1536+1792+1920 = 5248
    # one very long sample takes a group of its own; the rest share one
    assert check_plan([1900, 100, 100, 100], 1900, True, 3) == [(0, 1, 1900), (1, 4, 128)]


def test_frame_count_shrinks_only_under_exact_varlen():
    durations = [200, 300, 1000, 1100]
    faithful = plan_sample_split(durations, 1100, False, 2)
    varlen = plan_sample_split(durations, 1100, True, 2)
    assert all(f == 1100 for _, _, f in faithful)
    assert [f for _, _, f in varlen] == [1024, 1100]  # the first group at 1000 -> 1024, the last one capped at N


def test_plan_refuses_nothing_to_split():
    with pytest.raises(ValueError):
        plan_sample_split([], 100, False, 2)
    with pytest.raises(ValueError):
        plan_sample_split([100], 100, False, 0)


# ---------------------------------------------------------------------------------------------------------------------
# arguments
# ---------------------------------------------------------------------------------------------------------------------
def test_refused_devices():
    model = small_model()
    for devs in ([], ["cpu"], [torch.device("cpu")], ["cuda:99"], ["not-a-device"], "cuda:0", None, 0,
                 torch.device("cuda", 0)):
        with pytest.raises(ValueError):
            model.enable_sample_parallel(devs)
    assert model.transformer.sample_split is None
    if torch.cuda.device_count() == 0:
        with pytest.raises(ValueError):
            model.enable_sample_parallel(["cuda:0"])


def test_both_splits_refused(monkeypatch):
    monkeypatch.setattr(cfg_parallel, "peer_device", lambda d, what=None: torch.device(d))
    model = small_model()
    peers = model.enable_sample_parallel(["cuda:0", "cuda:1"])
    with pytest.raises(ValueError):
        model.enable_cfg_parallel("cuda:1")
    assert model.transformer.cfg_peer is None and model.transformer.sample_split.peers is peers
    model.disable_sample_parallel()
    model.enable_cfg_parallel("cuda:1")
    with pytest.raises(ValueError):
        model.enable_sample_parallel(["cuda:0", "cuda:1"])
    assert model.transformer.sample_split is None
    model.disable_cfg_parallel()


def test_enable_again_keeps_the_peers(monkeypatch):
    """The same list keeps the peers (weight copies, streams, workspaces); another list or disable drops them.  A device
    named twice gets two peers."""
    monkeypatch.setattr(cfg_parallel, "peer_device", lambda d, what=None: torch.device(d))
    model = small_model()
    p1 = model.enable_sample_parallel(["cuda:0", "cuda:0"])
    assert len(p1) == 2 and p1[0] is not p1[1] and all(isinstance(p, cfg_parallel.DevicePeer) for p in p1)
    assert [p.device for p in p1] == [torch.device("cuda:0")] * 2
    assert model.enable_sample_parallel(["cuda:0", "cuda:0"]) is p1
    p2 = model.enable_sample_parallel(["cuda:0", "cuda:1"])
    assert p2 is not p1 and [p.device for p in p2] == [torch.device("cuda:0"), torch.device("cuda:1")]
    model.disable_sample_parallel()
    assert model.transformer.sample_split is None


def test_load_model_and_f5tts_take_the_option():
    assert inspect.signature(infer.load_model).parameters["sample_parallel_devices"].default is None
    assert inspect.signature(api.F5TTS.__init__).parameters["sample_parallel_devices"].default is None


# ---------------------------------------------------------------------------------------------------------------------
# routing
# ---------------------------------------------------------------------------------------------------------------------
class RecordingSplit:
    def __init__(self):
        self.calls = []

    def run(self, backbone, y, step_cond, text, t_grid, duration, cfg_strength, trajectory, use_graph, exact_varlen,
            method):
        self.calls.append((y.shape[0], float(cfg_strength), bool(exact_varlen)))


def routed(monkeypatch):
    model = small_model()
    bb = model.transformer
    local = []
    monkeypatch.setattr(bb, "_run_local", lambda y, *a, **k: local.append(y.shape[0]))
    split = RecordingSplit()
    bb.sample_split = split
    return model, bb, split, local


def call(bb, B, cfg_strength=2.0, exact_varlen=False):
    y = torch.zeros(B, 16, 100)
    text = torch.zeros(B, 4, dtype=torch.int64)
    bb.run(y, torch.zeros_like(y), text, [0.0, 1.0], torch.full((B,), 16, dtype=torch.int32), cfg_strength,
           exact_varlen=exact_varlen)


def test_only_batched_calls_split(monkeypatch):
    model, bb, split, local = routed(monkeypatch)
    call(bb, 1)
    assert split.calls == [] and local == [1]
    call(bb, 2)
    call(bb, 5, exact_varlen=True)
    call(bb, 3, cfg_strength=0.0)  # no guidance: the samples still split
    assert split.calls == [(2, 2.0, False), (5, 2.0, True), (3, 0.0, False)] and local == [1]
    # the operator seam asks for the raw backbone output: it stays local
    bb(torch.zeros(2, 16, 100), torch.zeros(2, 16, 100), torch.zeros(2, 4, dtype=torch.int64), torch.tensor([0.5]),
       cfg_infer=True)
    assert len(split.calls) == 3 and local == [1, 2]
    model.disable_sample_parallel()
    call(bb, 4)
    assert len(split.calls) == 3 and local == [1, 2, 4]


def test_sample_calls_route_by_batch(monkeypatch):
    """CFM.sample: a batched call reaches the split, with and without guidance; a one-sample call does not."""
    model, bb, split, local = routed(monkeypatch)
    monkeypatch.setattr(F5.model, "lens_to_mask", lambda t, length=None: torch.ones(t.shape[0], int(t.amax()),
                                                                                    dtype=torch.bool))
    model.sample(torch.zeros(1, 8, 100), torch.zeros(1, 4, dtype=torch.long), 20, steps=2, seed=1)
    assert local == [1] and split.calls == []
    for cfg_strength in (2.0, 0.0):
        model.sample(torch.zeros(3, 8, 100), torch.zeros(3, 4, dtype=torch.long), 20, steps=2,
                     cfg_strength=cfg_strength, seed=1, exact_varlen=True)
    assert local == [1] and split.calls == [(3, 2.0, True), (3, 0.0, True)]


def test_batcher_runs_split(monkeypatch):
    """enable_batching's runs call the backbone's run: a run of two or more samples splits."""
    model, bb, split, local = routed(monkeypatch)
    batcher = batching.SampleBatcher(bb)
    y = torch.zeros(2, 16, 100)
    batcher.run(y, torch.zeros_like(y), torch.zeros(2, 4, dtype=torch.int64), [0.0, 1.0],
                torch.tensor([16, 9], dtype=torch.int32), 2.0, exact_varlen=True)
    y1 = torch.zeros(1, 16, 100)
    batcher.run(y1, torch.zeros_like(y1), torch.zeros(1, 4, dtype=torch.int64), [0.0, 1.0], None, 2.0)
    assert split.calls == [(2, 2.0, True)] and local == [1] and batcher.stats.runs == 2


def test_sample_split_is_built_from_device_peers(monkeypatch):
    monkeypatch.setattr(cfg_parallel, "peer_device", lambda d, what=None: torch.device(d))
    split = sample_parallel.SampleSplit(["cuda:0", "cuda:1"], copy_weights=True)
    assert [type(p) for p in split.peers] == [cfg_parallel.DevicePeer] * 2
    assert all(p.copy_weights and p.replications == 0 and p._state is None for p in split.peers)
    assert issubclass(cfg_parallel.CfgPeer, cfg_parallel.DevicePeer)
