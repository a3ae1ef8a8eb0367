"""Explicit-state model checker for the worker <-> ps mailbox protocol of the fused step engine.

The reference has no race detection of any kind (SURVEY §5 "Race detection / sanitizers": TF's runtime owns every
queue); here the hand-off between a worker's step clusters and the persistent ps kernel is a hand-written lock-free
protocol, so besides compute-sanitizer runs on the GPU its *design* is checked exhaustively:
this module enumerates every interleaving of a small configuration and verifies that none deadlocks, none overwrites a
mailbox slot the ps has not consumed, and every push is applied exactly once and in order.

What is modelled (csrc/fused_step_sm90.cu, csrc/ps_apply_sm90.cu):

* a launch runs ``lanes`` clusters; steps are claimed from one atomic counter (``claim()``, kernel line "first step of
  this cluster"), the *next* step of a lane is claimed in the prologue of its current one;
* push ``seq`` (= step + 1) goes to mailbox slot ``seq % nslots``; the step's prologue waits for the ps
  acknowledgement of push ``seq - nslots`` (flow control: the slot's previous occupant has been applied);
* the ps consumes one worker's pushes strictly in sequence order (it polls the flags of slot ``next % nslots`` for the
  value ``next``) and acknowledges with the highest sequence number applied;
* *publishing* a push (completion of the TMA stores, a system-scope fence, the flag stores) is expensive, so the
  publisher warp defers it into the head phase of the lane's next step — i.e. until after that step's flow-control wait —
  unless ``strict`` is set, the lane has no next step, or the guard ``(next - cur) < nslots // 2`` fails.

The guard is what this model is about: the first deferred-publish version of the kernel had no guard and deadlocked on
the GPU (``ack timeout need=21 ack=15``): lane A's next step waited for an acknowledgement that could only follow the
publication A itself had deferred behind that very wait. ``check(..., guard=False)`` reproduces that deadlock; with the
guard every edge "X waits for Y's deferred publish" implies ``seq_Y < seq_X - nslots / 2``, so waits-for cycles cannot
close (tests/test_protocol_model.py checks all small configurations).
"""
from __future__ import annotations

from collections import deque
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

# lane phases
CLAIM, FLOW, HEAD, PUSH, ACKWAIT, DONE = range(6)


@dataclass(frozen=True)
class Config:
    lanes: int
    nslots: int
    n_steps: int
    guard: bool = True        # the kernel's deferral guard (nxt - cur) < nslots // 2
    defer: bool = True        # deferred publishing at all (False: publish right after the push)
    strict: bool = False      # --strict_steps: publish at once and wait for the acknowledgement before the next step
    shards: int = 1           # ps tasks the worker pushes to (row_split: every push has a tile on every shard); each
                              # shard consumes and acknowledges on its own, the worker waits for the slowest


@dataclass
class Result:
    ok: bool
    states: int
    reason: str = ""
    trace: Optional[List[str]] = None


# state = (counter, acks(per shard), ps_next(per shard), published(frozenset), slots(tuple),
#          lanes(tuple of (phase, cur, nxt, pend)))
def _initial(cfg: Config):
    lanes = []
    counter = 0
    for _ in range(cfg.lanes):   # every cluster claims its first step when it starts
        if counter < cfg.n_steps:
            lanes.append((CLAIM, counter, -1, -1))
            counter += 1
        else:
            lanes.append((DONE, -1, -1, -1))
    return (counter, tuple([0] * cfg.shards), tuple([1] * cfg.shards), frozenset(), tuple([0] * cfg.nslots), tuple(lanes))


def _successors(cfg: Config, st) -> List[Tuple[str, tuple, Optional[str]]]:
    counter, acks, ps_nexts, published, slots, lanes = st
    ack = min(acks)          # what the worker's flow control / strict wait sees: the slowest shard
    ps_next = min(ps_nexts)
    out = []
    # ---- ps shards: each applies the next push of this worker once it has been published ----
    for k in range(cfg.shards):
        nk = ps_nexts[k]
        if nk in published:
            err = None
            if slots[nk % cfg.nslots] != nk:
                err = f"ps {k} reads slot {nk % cfg.nslots} for push {nk} but it holds push {slots[nk % cfg.nslots]}"
            a2 = acks[:k] + (nk,) + acks[k + 1:]
            n2 = ps_nexts[:k] + (nk + 1,) + ps_nexts[k + 1:]
            out.append((f"ps {k} applies {nk}" if cfg.shards > 1 else f"ps applies {nk}", (counter, a2, n2, published, slots, lanes), err))
    # ---- lanes ----
    for i, (phase, cur, nxt, pend) in enumerate(lanes):
        def put(new_lane, **kw):
            l2 = list(lanes)
            l2[i] = new_lane
            return (kw.get("counter", counter), acks, ps_nexts, kw.get("published", published), kw.get("slots", slots),
                    tuple(l2))
        seq = cur + 1
        if phase == CLAIM:       # prologue: claim the lane's next step
            if counter < cfg.n_steps:
                out.append((f"lane {i} claims step {counter}", put((FLOW, cur, counter, pend), counter=counter + 1), None))
            else:
                out.append((f"lane {i} finds no further step", put((FLOW, cur, -1, pend)), None))
        elif phase == FLOW:      # flow control: the slot's previous occupant must have been applied
            if seq <= cfg.nslots or ack >= seq - cfg.nslots:
                out.append((f"lane {i} passes flow control of push {seq}", put((HEAD, cur, nxt, pend)), None))
        elif phase == HEAD:      # head phase: the publisher warp publishes the deferred previous push of this lane
            pub = published | {pend} if pend > 0 else published
            out.append((f"lane {i} head phase" + (f", publishes deferred {pend}" if pend > 0 else ""),
                        put((PUSH, cur, nxt, -1), published=pub), None))
        elif phase == PUSH:      # the gradient push into the mailbox slot, then publish now or defer
            err = None
            prev = slots[seq % cfg.nslots]
            if prev != 0 and ack < prev:
                err = f"lane {i} overwrites slot {seq % cfg.nslots} (push {prev} not applied yet, ack {ack}) with push {seq}"
            s2 = list(slots)
            s2[seq % cfg.nslots] = seq
            s2 = tuple(s2)
            deferred = (cfg.defer and not cfg.strict and nxt >= 0
                        and (not cfg.guard or (nxt - cur) < (cfg.nslots >> 1)))
            if deferred:
                out.append((f"lane {i} pushes {seq}, defers its publication",
                            put((CLAIM, nxt, -1, seq), slots=s2), err))
            else:
                if nxt < 0:
                    nl = (DONE, -1, -1, -1)
                elif cfg.strict:
                    nl = (ACKWAIT, cur, nxt, -1)     # the next pull starts only after this push has been applied
                else:
                    nl = (CLAIM, nxt, -1, -1)
                out.append((f"lane {i} pushes and publishes {seq}", put(nl, slots=s2, published=published | {seq}), err))
        elif phase == ACKWAIT:
            if ack >= seq:
                out.append((f"lane {i} sees push {seq} acknowledged", put((CLAIM, nxt, -1, -1)), None))
    return out


def check(cfg: Config, max_states: int = 2_000_000) -> Result:
    """Breadth-first search over every interleaving. ok == no deadlock, no slot overwritten early, no stale slot read,
    and every terminal state has all pushes applied in order."""
    if cfg.nslots < 1 or cfg.lanes < 1:
        raise ValueError("need lanes >= 1 and nslots >= 1")
    init = _initial(cfg)
    parent: Dict[tuple, Tuple[Optional[tuple], str]] = {init: (None, "start")}
    q = deque([init])

    def trace_of(st, extra=None):
        steps = []
        while st is not None:
            par, label = parent[st]
            steps.append(label)
            st = par
        steps.reverse()
        if extra:
            steps.append(extra)
        return steps

    while q:
        st = q.popleft()
        succ = _successors(cfg, st)
        counter, acks, ps_nexts, published, slots, lanes = st
        ack, ps_next = min(acks), min(ps_nexts)
        if not succ:
            if ack == cfg.n_steps and all(l[0] == DONE for l in lanes):
                continue   # proper termination
            waiting = [f"lane {i} waits for ack >= {l[1] + 1 - cfg.nslots}" for i, l in enumerate(lanes) if l[0] == FLOW]
            waiting += [f"lane {i} waits for ack >= {l[1] + 1}" for i, l in enumerate(lanes) if l[0] == ACKWAIT]
            return Result(False, len(parent), f"deadlock: ack={ack}, ps waits for push {ps_next}, " + "; ".join(waiting),
                          trace_of(st))
        for label, nst, err in succ:
            if err:
                parent.setdefault(nst, (st, label))
                return Result(False, len(parent), err, trace_of(st, label))
            if nst not in parent:
                parent[nst] = (st, label)
                if len(parent) > max_states:
                    return Result(False, len(parent), "state limit exceeded")
                q.append(nst)
    return Result(True, len(parent))


def simulate(cfg: Config, seed: int, bias: str = "uniform", max_moves: int = 10_000_000) -> Result:
    """One random schedule of a configuration that is too large to enumerate (the production default is 12 lanes x 48
    slots). `bias` skews the scheduler: "uniform", "slow_ps" (the ps moves only when nothing else can or with 2 %
    probability: maximal back-pressure), "slow_lane" (lane 0 is starved the same way: a straggler holding an old
    sequence number), "fast_ps". Same checks as `check`."""
    import random
    rnd = random.Random(seed)
    st = _initial(cfg)
    moves = 0
    while moves < max_moves:
        succ = _successors(cfg, st)
        counter, acks, ps_nexts, published, slots, lanes = st
        ack, ps_next = min(acks), min(ps_nexts)
        if not succ:
            if ack == cfg.n_steps and all(l[0] == DONE for l in lanes):
                return Result(True, moves)
            return Result(False, moves, f"deadlock after {moves} moves: ack={ack}, ps waits for push {ps_next}")
        pick = None
        if bias != "uniform" and len(succ) > 1:
            slow = "ps " if bias == "slow_ps" else "lane 0 " if bias == "slow_lane" else None
            fast = "ps " if bias == "fast_ps" else None
            if slow is not None and rnd.random() > 0.02:
                others = [x for x in succ if not x[0].startswith(slow)]
                if others:
                    pick = rnd.choice(others)
            if fast is not None:
                f = [x for x in succ if x[0].startswith(fast)]
                if f and rnd.random() < 0.9:
                    pick = f[0]
        if pick is None:
            pick = rnd.choice(succ)
        label, st, err = pick
        if err:
            return Result(False, moves, err)
        # the set of published-and-applied pushes is never consulted again: keep the state small
        counter, acks, ps_nexts, published, slots, lanes = st
        if len(published) > 4 * cfg.nslots:
            st = (counter, acks, ps_nexts, frozenset(x for x in published if x >= min(ps_nexts)), slots, lanes)
        moves += 1
    return Result(False, moves, "move limit exceeded")


def main() -> int:   # python -m dist_mnist_b200.utils.protocol_model LANES NSLOTS STEPS [noguard]
    import sys
    a = sys.argv[1:]
    shards = next((int(x.split("=")[1]) for x in a if x.startswith("shards=")), 1)
    cfg = Config(int(a[0]), int(a[1]), int(a[2]), guard="noguard" not in a, strict="strict" in a, shards=shards)
    r = check(cfg)
    print(cfg, "->", "OK" if r.ok else "FAILED: " + r.reason, f"({r.states} states)")
    if r.trace:
        print("\n".join("  " + t for t in r.trace))
    return 0 if r.ok else 1


if __name__ == "__main__":
    raise SystemExit(main())
