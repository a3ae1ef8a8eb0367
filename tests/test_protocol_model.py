"""Exhaustive interleaving check of the fused engine's mailbox protocol (dist_mnist_b200/utils/protocol_model.py).

The deferred-publish guard of csrc/fused_step_sm90.cu (`deferred = ... && (nxt - cur) < (nslots >> 1)`) exists because
the unguarded version deadlocked on the GPU; the model reproduces that deadlock and shows that the guarded protocol, the
immediate-publish protocol and `--strict_steps` have none, never overwrite an unconsumed mailbox slot and apply every push
exactly once, in order — for every interleaving of every small configuration."""
import pytest

from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
from dist_mnist_b200.utils.protocol_model import Config, check

SMALL = [(lanes, nslots, steps) for lanes in (1, 2, 3) for nslots in range(max(2, lanes), 7) for steps in (5, 8)
         if not (lanes == 3 and steps == 8 and nslots > 4)]


@pytest.mark.parametrize("lanes,nslots,steps", SMALL)
def test_guarded_deferred_publish_has_no_deadlock_and_no_slot_hazard(lanes, nslots, steps):
    r = check(Config(lanes, nslots, steps, guard=True))
    assert r.ok, (r.reason, r.trace)


@pytest.mark.parametrize("lanes,nslots,steps", [(2, 4, 8), (3, 4, 8), (2, 2, 6), (3, 6, 9)])
def test_unguarded_deferred_publish_deadlocks_like_the_first_gpu_version(lanes, nslots, steps):
    r = check(Config(lanes, nslots, steps, guard=False))
    assert not r.ok and r.reason.startswith("deadlock"), r.reason
    # the cycle: some lane's flow control waits for an acknowledgement the ps cannot give because the push it needs
    # next is still unpublished
    assert "ps waits for push" in r.reason and r.trace


@pytest.mark.parametrize("lanes,nslots,steps", [(1, 2, 6), (2, 2, 7), (2, 4, 8), (3, 3, 7), (3, 6, 8)])
def test_strict_and_immediate_publish_variants(lanes, nslots, steps):
    assert check(Config(lanes, nslots, steps, strict=True)).ok
    assert check(Config(lanes, nslots, steps, defer=False)).ok


def test_single_lane_needs_no_guard():
    # one lane claims consecutive steps: (nxt - cur) == 1 < nslots, its deferred push is never what its own flow control
    # waits for as long as the ring has at least 2 slots
    assert check(Config(1, 2, 8, guard=False)).ok
    assert check(Config(1, 4, 8, guard=False)).ok


def test_engine_config_keeps_the_ring_at_least_as_deep_as_the_lanes():
    # the model's precondition nslots >= lanes is what EngineConfig.validate enforces for the real engine
    with pytest.raises(ValueError):
        EngineConfig(backend="cpu", lanes=4, nslots=2).validate(OptimizerConfig("adam", 1e-4))


@pytest.mark.parametrize("lanes,nslots", [(12, 48), (12, 12), (8, 16), (4, 8), (16, 64)])
def test_random_schedules_of_production_sized_configurations(lanes, nslots):
    """The CLI / bench default (12 lanes, 48 mailbox slots) is far too large to enumerate: random schedules, also with a
    starved ps (maximal back-pressure on the flow control), a straggling lane (holds an old sequence number while the
    others race ahead) and an eager ps."""
    from dist_mnist_b200.utils.protocol_model import simulate

    for bias in ("uniform", "slow_ps", "slow_lane", "fast_ps"):
        for seed in range(6):
            r = simulate(Config(lanes, nslots, 400), seed, bias)
            assert r.ok, (bias, seed, r.reason)
    # and the unguarded variant is caught by random schedules too (it deadlocks as soon as a lane's next claim is
    # >= nslots ahead of its deferred push)
    bad = [simulate(Config(lanes, nslots, 400, guard=False), seed, "slow_lane") for seed in range(6)]
    assert any(not r.ok and r.reason.startswith("deadlock") for r in bad) or lanes < 4


@pytest.mark.parametrize("lanes,nslots,steps,shards", [(2, 4, 7, 2), (2, 2, 6, 3), (3, 4, 6, 2), (1, 2, 6, 3)])
def test_several_ps_shards_acknowledging_independently(lanes, nslots, steps, shards):
    """row_split / multi-ps: every push has a part on every shard, each shard consumes and acknowledges on its own and the
    worker's flow control waits for the slowest one."""
    assert check(Config(lanes, nslots, steps, shards=shards)).ok
    assert check(Config(lanes, nslots, steps, shards=shards, strict=True)).ok
    if lanes >= 2:
        r = check(Config(lanes, nslots, steps, shards=shards, guard=False))
        assert not r.ok and r.reason.startswith("deadlock")
