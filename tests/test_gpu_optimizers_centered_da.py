"""Centered RMSProp and AdagradDA on the GPU parameter server: the serve kernel alone against the TF1 formulas in fp64
(both math modes, per push and merged, default and register-resident geometry, constant rate, scheduled and averaging;
AdagradDA from a sched_step where fp32 T starts to round), the fused engine in lock-step with fp32 PyTorch, 8 lanes over
2 ps on the graph engine and with row_split, a 1 ps + 2 worker run in three processes, and a checkpoint resume that
keeps the mg slot."""
import dataclasses
import re
import tempfile

import _harness
import pytest
import torch

pytestmark = pytest.mark.gpu


def _opts():
    from dist_mnist_b200.parallel.config import OptimizerConfig
    return {
        "centered": OptimizerConfig("rmsprop", 1e-3, centered=True),
        "centered_momentum": OptimizerConfig("rmsprop", 1e-3, centered=True, momentum=0.9, decay=0.8, eps=1e-6),
        "centered_momentum_lr1e4": OptimizerConfig("rmsprop", 1e-4, centered=True, momentum=0.9, decay=0.8, eps=1e-6),
        "adagrad_da": OptimizerConfig("adagrad_da", 0.1),
        "adagrad_da_l1_l2": OptimizerConfig("adagrad_da", 0.1, l1_regularization_strength=1e-4,
                                            l2_regularization_strength=1e-2),
        "adagrad_da_l2": OptimizerConfig("adagrad_da", 0.1, l2_regularization_strength=1e-2),
    }


def _serve_checks(opt, sched_step=0):
    from bench_tools import gpu_check
    from dist_mnist_b200 import _native as N

    ok = True
    for math in ("fast", "ieee"):
        for mode in (N.APPLY_PER_PUSH, N.APPLY_MERGED):
            for resident in (False, True):
                ok &= gpu_check.check_ps_serve_tf1(dataclasses.replace(opt, math=math), mode, resident=resident,
                                                   sched_step=sched_step)
    return ok


@pytest.mark.parametrize("rule", ["centered", "centered_momentum", "adagrad_da", "adagrad_da_l1_l2", "adagrad_da_l2"])
def test_serve_kernel_alone_matches_tf1_formulas(rule):
    """Constant rate (AdagradDA: its scheduled instantiation), from sched_step 0 and 5."""
    assert _serve_checks(_opts()[rule]) and _serve_checks(_opts()[rule], 5)


@pytest.mark.parametrize("rule", ["centered_momentum", "adagrad_da_l1_l2"])
def test_scheduled_and_averaging_serve_kernels_match_fp64(rule):
    from dist_mnist_b200.parallel.config import LrSchedule

    sched = LrSchedule("exponential_decay", decay_steps=4, decay_rate=0.75)
    opt = _opts()[rule]
    assert _serve_checks(dataclasses.replace(opt, schedule=sched), 1)
    assert _serve_checks(dataclasses.replace(opt, moving_average_decay=0.99))
    assert _serve_checks(dataclasses.replace(opt, schedule=sched, moving_average_decay=0.99), 3)


@pytest.mark.parametrize("rule", ["adagrad_da", "adagrad_da_l1_l2"])
def test_adagrad_da_T_counts_past_2_24(rule):
    """Every item starts at sched_step 2^24 - 4, so the 9 pushes take T past 2^24. The check catches an off-by-one or a
    wrap in T, and the final sched_step must be 2^24 + 5. T's fp32 rounding there moves p by ~6e-8 relative, below the
    check's 1e-5 bound, so this does not test the rounding: the kernel casts T exactly as the cpu loop does, and
    tests/test_optimizers_centered_da_cpu.py::test_adagrad_da_T_is_rounded_to_fp32 checks that cast."""
    assert _serve_checks(_opts()[rule], (1 << 24) - 4)


@pytest.mark.parametrize("rule", ["centered", "centered_momentum_lr1e4", "adagrad_da", "adagrad_da_l2"])
def test_strict_fused_native_loop_is_lock_step_with_fp32_torch(rule):
    """300 strict steps (lanes=1) against an un-rounded fp32 PyTorch step on the same `next_batch` sequence, with the
    bounds of tests/test_gpu_optimizers.py. T is the global step here: one worker, one lane, strict. l1 is 0: the tf32
    forward moves g_acc enough to put an element on the other side of the T * l1 threshold; the serve kernels are
    checked with l1 against fp64 above. Centered RMSProp with momentum 0.9 runs at lr 1e-4: its normalised update,
    accumulated by the momentum, turns the tf32 forward's rounding into whole steps, and at lr 1e-3 it ended 6.5e-3
    from fp32 PyTorch on an H100, above the parameter bound."""
    from bench_tools.gpu_e2e import ref_slots, ref_step
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    opt = _opts()[rule]
    ds = data.synthetic_mnist(8192, seed=5)
    spec = mlp.book_model(100)
    params = mlp.init_params(spec, seed=11)
    ref_p = {k: t.clone() for k, t in params.items()}
    ref_m, ref_v, ref_g = ref_slots(opt, params, with_mg=True)
    cfg = EngineConfig(backend="cuda", engine="fused", lanes=1, nslots=8, strict_steps=True)
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=1, params=params) as cl:
        w = cl.worker
        assert w.engine == "fused"
        loader = w.make_loader(ds.images, ds.labels, seed=7)
        twin = w.make_loader(ds.images, ds.labels, seed=7, epoch_feed=False)
        outs = []
        for n in (7, 93, 200):
            outs += list(w.run_steps(n, loader, wait_applied=True))
        assert len(outs) == 300 and w.read_global_step() == 300
        if opt.kind == "adagrad_da":
            assert set(w.read_sched_steps(0)) == {300}
        t, worst = 0, 0.0
        for o in outs:
            x, y = twin.next_batch()
            lref, t = ref_step(spec, ref_p, ref_m, ref_v, t, x, y, opt, mg=ref_g)
            assert o.global_step == o.seq
            if lref > 1e-6:
                worst = max(worst, abs(o.loss - lref) / abs(lref))
        got = w.read_variables()
    perr = max(float((got[k] - ref_p[k]).norm() / (ref_p[k].norm() + 1e-9)) for k in got)
    print(f"[lock-step {rule}] 300 steps: worst per-step loss rel err {worst:.2e}, param rel err {perr:.2e}")
    assert worst < 1e-2
    assert perr < 5e-3


# (layout, rule, lr, whether the loss must halve). AdagradDA at lr 0.5 halved the loss on the graph engine, but with
# row_split 8 lanes took it from 0.225 to 2.06 on an H100 (as FTRL at lr 0.5 does); there it runs at its default 0.1 and
# the loss has to fall.
EIGHT_LANES = [("graph", "centered_momentum", 1e-3, True), ("row_split", "centered", 1e-3, True),
               ("graph", "adagrad_da_l2", 0.5, True), ("row_split", "adagrad_da", 0.1, False)]


@pytest.mark.parametrize("case", EIGHT_LANES)
def test_eight_lanes_over_two_ps(case):
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    layout, rule, lr, halves = case
    opt = dataclasses.replace(_opts()[rule], lr=lr)
    kw = {"engine": "graph"} if layout == "graph" else {"sharding": "row_split"}
    cfg = EngineConfig(backend="cuda", lanes=8, nslots=16, **kw)
    ds = data.synthetic_mnist(8192, seed=6)
    with InProcessCluster(mlp.book_model(100), opt, cfg, batch_size=32, num_ps=2) as cl:
        w = cl.worker
        assert w.engine == ("graph" if layout == "graph" else "fused")
        loader = w.make_loader(ds.images, ds.labels, seed=0)
        outs = list(w.run_steps(300, loader, wait_applied=True)) + list(w.run_steps(97, loader, wait_applied=True))
        assert len(outs) == 397 and w.read_global_step() == 397
        assert sorted(o.seq for o in outs) == list(range(1, 398))
        assert all(torch.isfinite(torch.tensor(o.loss)) for o in outs)
        if opt.kind == "adagrad_da":   # one T step per applied push on every item
            assert set(w.read_sched_steps(0)) == set(w.read_sched_steps(1)) == {397}
        first = sum(o.loss for o in outs[:20]) / 20
        last = sum(o.loss for o in outs[-20:]) / 20
        print(f"[8 lanes {layout} {rule} lr {lr}] loss {first:.4f} -> {last:.4f}")
        assert last < (0.5 if halves else 1.0) * first, (first, last)


def test_checkpoint_resume_keeps_mg():
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig
    from dist_mnist_b200.session import InProcessCluster, train_loop
    from dist_mnist_b200.utils import data

    opt = _opts()["centered_momentum"]
    spec = mlp.book_model(100)
    cfg = EngineConfig(backend="cuda", lanes=1, nslots=2)
    ds = data.synthetic_mnist(4096, seed=3)
    d = tempfile.mkdtemp()
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=2) as cl:
        train_loop(cl.worker, ds, train_steps=60, log_every=0, checkpoint_dir=d, chunk=20)
        before = {r: cl.worker.read_variables(r) for r in ("params", "adam_m", "adam_v", "mg")}
    assert any(float(t.abs().max()) > 0 for t in before["mg"].values())
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=2, restore_dir=d) as cl:
        assert cl.worker.read_global_step() == 60
        for r, vals in before.items():
            got = cl.worker.read_variables(r)
            for k in vals:
                assert torch.equal(got[k].cpu(), vals[k].cpu()), (r, k)
        res = train_loop(cl.worker, ds, train_steps=100, log_every=0, chunk=20)
        assert res.steps_run == 40
        after = cl.worker.read_variables("mg")
        assert any(not torch.equal(after[k].cpu(), before["mg"][k].cpu()) for k in after)


@pytest.mark.timeout(420)
def test_centered_rmsprop_one_ps_two_workers_three_processes_one_gpu():
    """As tests/test_gpu_multiproc_one_gpu.py: every push applied exactly once, the loss falls, the ps exits. At lr
    1e-3 one such run on an H100 logged 0.23 then 0.97: with 8 pushes in flight, ms - mg^2 of an element whose gradient
    barely varies falls towards epsilon (1e-10) and the normalised step grows, as it can in TF. The run uses the
    reference's default rate, 1e-4, and the batch losses logged every 40 steps must dip below the first."""
    common = ["--train_steps", "240", "--learning_rate", "0.0001", "--log_every", "40", "--lanes", "4",
              "--optimizer", "rmsprop", "--centered"]
    with _harness.Tasks(backend="cuda", gpu=0) as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done"])
        ws = [t.spawn("worker", i, common) for i in range(2)]
        outs_w = [t.finish(w, 300) for w in ws]
        out_p = t.finish(ps, 90)
    for w, o in zip(ws, outs_w):
        assert w.returncode == 0, o
        assert "engine=fused" in o, o
    assert ps.returncode == 0, out_p
    total = sum(int(re.search(r"local_steps=(\d+)", o).group(1)) for o in outs_w)
    assert total >= 240
    m = re.search(r"exiting: global_step=(\d+) owns_global_step=1", out_p)
    assert m and int(m.group(1)) == total, (out_p, total)
    losses = [float(l.split("loss: ")[1]) for o in outs_w for l in o.splitlines() if l.startswith("Train step ")]
    assert len(losses) >= 2 and min(losses[1:]) < losses[0], losses
