"""Both GPU engines' pushed gradients, reported loss and correct count, element by element against the fp64 step, on
inputs that tf32 cannot round (bench_tools/fused_push_ref: the case builder, the bound and its derivation, proved on
the CPU by tests/test_fused_push_bound_cpu.py). SGD at learning rate 0 keeps the variables, so every step pulls the
same tf32-exact hidden weight; pushes are read out of the mailbox.

Fused engine: one strict step at every shape of the matrix; 3 x nslots steps in one cluster, strict and pulling ahead,
with every mailbox slot reused; 4 lanes in flight (pushes matched to batches as a multiset); both 2-shard layouts;
push == apply (atomic); and a push against the next batch's reference, which must fail. Graph engine: the same checker
at 784-H-10. Every check prints the worst err / bound per variable."""
import _harness
import pytest

from bench_tools import fused_push_ref as R

pytestmark = pytest.mark.gpu

MATRIX = R.shape_matrix()


@pytest.mark.parametrize("name,shape,saturate", MATRIX, ids=[m[0] for m in MATRIX])
def test_fused_push_is_inside_the_fp64_bound(name, shape, saturate):
    case = R.case_for(shape, saturate)
    x, y = case.batches[0]
    with _harness.cluster(case) as cl:
        got = _harness.step(cl.worker, x, y)
    _harness.check(f"fused {name} seed {case.seed} (random shapes from seed {R.RANDOM_SEED})", got, case, x, y)
    if shape[1] == 1:   # one class: softmax is 1, every gradient and the loss are exactly zero
        assert all(float(g.abs().max()) == 0.0 for g in got.grads.values()) and got.loss == 0.0


def _loader_batches(w, case, seed=0):
    """A native loader over the case's batches in order (no shuffle: batch i of an epoch is case.batches[i]) and a
    twin that hands the same batches to the host."""
    import torch

    xs = torch.cat([x for x, _ in case.batches])
    ys = torch.cat([y for _, y in case.batches])
    return w.make_loader(xs, ys, seed=seed, shuffle=False), w.make_loader(xs, ys, seed=seed, shuffle=False,
                                                                           epoch_feed=False)


@pytest.mark.parametrize("B", [32, 33, 100, 256])
def test_fused_pushes_of_consecutive_steps_in_one_launch(B):
    """Three launches of nslots steps at one lane, each step on a batch of its own: strict, strict again (every mailbox
    slot reused), then pulling the next step's W ahead of the push (non-strict). Each push is checked against its
    batch: the running sums of the row tiles restart with every step, and every slot holds its own step's push. A slot
    that kept its previous push (that of the batch nslots steps earlier) would fail the bound, and that is checked too."""
    import torch

    ns = 4
    case = R.case_for((100, 10, 784, B, "book"), n_batches=3 * ns, seed=2)
    with _harness.cluster(case, nslots=ns) as cl:
        w = cl.worker
        loader, twin = _loader_batches(w, case)
        seq = 0
        for strict in (True, True, False):
            if not strict:
                w.set_lanes(1, strict=False)
            outs = list(w.run_steps(ns, loader, wait_applied=True))
            assert [o.seq for o in outs] == list(range(seq + 1, seq + ns + 1))
            for o in outs:
                i = o.seq - 1                       # push s trains on batch s - 1 of the unshuffled loader
                x, y = twin.next_batch()
                assert torch.equal(x, case.batches[i][0])
                got = R.Step(R.pushed(w, o.seq), float(o.loss), int(o.correct))
                _harness.check(f"fused B{B} step {o.seq} strict={strict}", got, case, x, y)
                if i >= ns:   # what the slot held before this push: it must not pass for this step's
                    _harness.check(f"fused B{B} step {o.seq} vs the batch of the slot's previous push (must fail)",
                                   got, case, *case.batches[i - ns], expect_ok=False)
            seq += ns


@pytest.mark.parametrize("B", [32, 256])
def test_fused_pipelined_pushes_match_their_batches(B):
    """4 lanes in flight, not strict, 8 steps into 8 mailbox slots: the 8 pushes and the 8 batches match one to one,
    whichever lane ran which step."""
    case = R.case_for((100, 10, 784, B, "book"), n_batches=8, seed=3)
    with _harness.cluster(case, lanes=4, nslots=8, strict=False) as cl:
        w = cl.worker
        loader, twin = _loader_batches(w, case)
        outs = list(w.run_steps(8, loader, wait_applied=True))
        assert sorted(o.seq for o in outs) == list(range(1, 9))
        batches = [twin.next_batch() for _ in range(8)]
        refs = [R.reference(case.spec, case.params, x, y) for x, y in batches]
        pushes = [(o.seq, R.Step(R.pushed(w, o.seq), float(o.loss), int(o.correct))) for o in outs]
    match = {}
    for s, got in pushes:
        verdicts = [R.compare(got, r) for r in refs]
        hits = [i for i, v in enumerate(verdicts) if v.ok]
        print(f"[fused pipelined B{B} push {s}] matches batches {hits}; "
              f"{verdicts[hits[0]].line() if hits else [round(v.max, 2) for v in verdicts]}", flush=True)
        assert len(hits) == 1, (s, [v.max for v in verdicts])
        match[s] = hits[0]
    assert sorted(match.values()) == list(range(8))


SHARDED = [((100, 10, 784, 100, "book"), 2, "row_split"), ((72, 10, 1024, 256, "book"), 2, "row_split"),
           ((100, 10, 784, 32, "book"), 2, "round_robin")]


@pytest.mark.parametrize("shape,nps,sharding", SHARDED, ids=[f"H{s[0]}-I{s[2]}-B{s[3]}-{n}ps-{m}" for s, n, m in SHARDED])
def test_fused_sharded_push_is_inside_the_fp64_bound(shape, nps, sharding):
    case = R.case_for(shape)
    x, y = case.batches[0]
    with _harness.cluster(case, nps=nps, sharding=sharding) as cl:
        got = _harness.step(cl.worker, x, y)
    _harness.check(f"fused {sharding} over {nps} ps {shape}", got, case, x, y)


@pytest.mark.parametrize("shape", [(100, 10, 784, 32, "book"), (128, 11, 1024, 256, "xent")],
                         ids=["H100-C10-I784-B32-book", "H128-C11-I1024-B256-xent"])
def test_fused_atomic_push_is_inside_the_fp64_bound(shape):
    """push_mode "atomic": the kernel adds -lr * g into the master copy (push == apply). At lr = 1, -lr * g is exact;
    g = p0 - p1 is recovered from the master copy, p1 = fl(p0 - g) adding at most 2^-24 max(|p0|, |p1|)."""
    import torch

    case = R.case_for(shape)
    x, y = case.batches[0]
    with _harness.cluster(case, push_mode="atomic", lr=1.0) as cl:
        w = cl.worker
        out = w.step(x, y)
        w.wait_applied()
        p1 = w.read_variables()
    p0 = case.params
    g = {n: p0[n].double() - p1[n].double() for n in R.VARS}
    ref = R.reference(case.spec, p0, x, y)
    for n in R.VARS:
        ref.bounds[n] = ref.bounds[n] + 2.0 ** -24 * torch.maximum(p0[n].double().abs(), p1[n].double().abs())
    v = R.compare(R.Step(g, float(out.loss), int(out.correct)), ref)
    print(f"[fused atomic {shape}] {v.line()}", flush=True)
    assert v.ok, (v.worst, v.where)


GRAPH = [(100, 1), (100, 32), (100, 100), (128, 256)]


@pytest.mark.parametrize("H,B", GRAPH, ids=[f"H{h}-B{b}" for h, b in GRAPH])
def test_graph_push_is_inside_the_fp64_bound(H, B):
    """The per-layer graph engine (`engine="auto"` takes it for batches above 32): forward GEMM on the same exact
    operands, head with IEEE division, dW GEMM on tf32 dpre. The bound needs no change (see the module docstring)."""
    case = R.case_for((H, 10, 784, B, "book"))
    x, y = case.batches[0]
    with _harness.cluster(case, engine="graph") as cl:
        got = _harness.step(cl.worker, x, y)
    _harness.check(f"graph H{H} B{B}", got, case, x, y)


def test_push_against_the_next_batch_fails_the_bound():
    """Negative control on real pushes: a fused push is far outside the bound of the batch after it."""
    case = R.case_for((100, 10, 784, 32, "book"), n_batches=2, seed=4)
    (x0, y0), (x1, y1) = case.batches
    with _harness.cluster(case) as cl:
        got = _harness.step(cl.worker, x0, y0)
    _harness.check("fused push of batch 0 vs its own batch", got, case, x0, y0)
    v = _harness.check("fused push of batch 0 vs batch 1 (must fail)", got, case, x1, y1, expect_ok=False)
    assert v.max > 10.0, v.worst
