"""Adadelta, FTRL (V1 and V2), ProximalAdagrad and ProximalGradientDescent on the GPU parameter server: the serve
kernel's new instantiations alone against the TF1 formulas in fp64 (constant-rate, scheduled and averaging), the fused
engine in lock-step with fp32 PyTorch, pipelined runs on the graph engine and with row_split sharding, and a 1 ps + 2
worker multi-process run on one GPU."""
import re

import _harness
import pytest
import torch

pytestmark = pytest.mark.gpu


def _opts():
    """Every rule and branch: l1 > 0 and == 0, lr_power -0.5 and -0.25, shrinkage on and off."""
    from dist_mnist_b200.parallel.config import OptimizerConfig
    return {
        "adadelta": OptimizerConfig("adadelta", 1.0),
        "adadelta_rho": OptimizerConfig("adadelta", 0.5, rho=0.9, eps=1e-6),
        "ftrl": OptimizerConfig("ftrl", 0.05),
        "adadelta_lr01": OptimizerConfig("adadelta", 0.1),
        "adadelta_rho_lr01": OptimizerConfig("adadelta", 0.1, rho=0.9, eps=1e-6),
        "ftrl_l1": OptimizerConfig("ftrl", 0.05, l1_regularization_strength=1e-3, l2_regularization_strength=1e-2),
        "ftrl_pow": OptimizerConfig("ftrl", 0.05, learning_rate_power=-0.25, l1_regularization_strength=1e-3),
        "ftrl_v2": OptimizerConfig("ftrl", 0.05, l1_regularization_strength=1e-3, l2_regularization_strength=1e-3,
                                   l2_shrinkage_regularization_strength=1e-2),
        "ftrl_pow_v2": OptimizerConfig("ftrl", 0.05, learning_rate_power=-0.25, l2_regularization_strength=1e-3,
                                       l2_shrinkage_regularization_strength=1e-2),
        "proximal_adagrad": OptimizerConfig("proximal_adagrad", 0.05),
        "proximal_adagrad_l1": OptimizerConfig("proximal_adagrad", 0.05, l1_regularization_strength=1e-3,
                                               l2_regularization_strength=1e-2),
        "proximal_adagrad_l2": OptimizerConfig("proximal_adagrad", 0.05, l2_regularization_strength=1e-3),
        "proximal_sgd": OptimizerConfig("proximal_sgd", 0.05),
        "proximal_sgd_l1": OptimizerConfig("proximal_sgd", 0.05, l1_regularization_strength=1e-3,
                                           l2_regularization_strength=1e-2),
        "proximal_sgd_l2": OptimizerConfig("proximal_sgd", 0.05, l2_regularization_strength=1e-3),
    }


SERVE_RULES = ["adadelta", "adadelta_rho", "ftrl", "ftrl_l1", "ftrl_pow", "ftrl_v2", "ftrl_pow_v2", "proximal_adagrad",
               "proximal_adagrad_l1", "proximal_sgd", "proximal_sgd_l1"]


def _serve_checks(opt, sched_step=0):
    from bench_tools import gpu_check
    from dist_mnist_b200 import _native as N

    ok = True
    for mode in (N.APPLY_PER_PUSH, N.APPLY_MERGED):
        for resident in (False, True):
            ok &= gpu_check.check_ps_serve_tf1(opt, mode, resident=resident, sched_step=sched_step)
    return ok


@pytest.mark.parametrize("rule", SERVE_RULES)
def test_serve_kernel_alone_matches_tf1_formulas(rule):
    """Both math modes, per push and merged, with the default geometry and with the register-resident one."""
    import dataclasses

    ok = True
    for math in ("fast", "ieee"):
        ok &= _serve_checks(dataclasses.replace(_opts()[rule], math=math))
    assert ok


@pytest.mark.parametrize("rule", ["adadelta", "ftrl_pow_v2", "ftrl_l1", "proximal_adagrad_l1", "proximal_sgd_l1"])
def test_scheduled_serve_kernel_matches_fp64(rule):
    """The scheduled instantiations in both math modes, every item starting just below 2^24 and crossing a staircase
    boundary in the middle of a pass."""
    import dataclasses

    from dist_mnist_b200.parallel.config import LrSchedule

    sched = LrSchedule("exponential_decay", decay_steps=1 << 20, decay_rate=0.96875, staircase=True)
    ok = True
    for math in ("fast", "ieee"):
        ok &= _serve_checks(dataclasses.replace(_opts()[rule], math=math, schedule=sched), (1 << 24) - 4)
    assert ok


@pytest.mark.parametrize("rule", ["adadelta_rho", "ftrl_v2", "ftrl_pow", "proximal_adagrad_l1", "proximal_sgd_l1"])
def test_averaging_serve_kernel_matches_fp64(rule):
    """The averaging instantiations in both math modes, at a constant rate and under a schedule."""
    import dataclasses

    from dist_mnist_b200.parallel.config import LrSchedule

    ok = True
    for math in ("fast", "ieee"):
        opt = dataclasses.replace(_opts()[rule], math=math, moving_average_decay=0.99)
        ok &= _serve_checks(opt)
        ok &= _serve_checks(dataclasses.replace(opt, schedule=LrSchedule("exponential_decay", decay_steps=4,
                                                                         decay_rate=0.75)), 1)
    assert ok


@pytest.mark.parametrize("rule", ["adadelta_lr01", "adadelta_rho_lr01", "ftrl", "ftrl_pow_v2", "proximal_adagrad",
                                  "proximal_adagrad_l2", "proximal_sgd", "proximal_sgd_l2"])
def test_strict_fused_native_loop_is_lock_step_with_fp32_torch(rule):
    """300 strict steps (lanes=1) against an un-rounded fp32 PyTorch step on the same `next_batch` sequence, with the
    bounds of tests/test_gpu_optimizers.py::test_strict_fused_native_loop_is_lock_step_with_fp32_torch. l1 is 0: the
    tf32 forward moves the gradient enough to put an element on the other side of an l1 threshold. Adadelta runs at lr
    0.1: its normalised update turns the tf32 forward's rounding into whole steps, as Adam's does, and at lr 1.0 it ended
    1.4e-2 from fp32 PyTorch here (0.5 with rho 0.9: 5.2e-3), above the parameter bound; its serve kernels are checked
    against fp64 above."""
    from bench_tools.gpu_e2e import ref_slots, ref_step
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    opt = _opts()[rule]
    assert not opt.l1_regularization_strength
    ds = data.synthetic_mnist(8192, seed=5)
    spec = mlp.book_model(100)
    params = mlp.init_params(spec, seed=11)
    ref_p = {k: t.clone() for k, t in params.items()}
    ref_m, ref_v = ref_slots(opt, params)
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
        t, worst = 0, 0.0
        for o in outs:
            x, y = twin.next_batch()
            lref, t = ref_step(spec, ref_p, ref_m, ref_v, t, x, y, opt)
            assert o.global_step == o.seq
            if lref > 1e-6:
                worst = max(worst, abs(o.loss - lref) / abs(lref))
        got = w.read_variables()
    perr = max(float((got[k] - ref_p[k]).norm() / (ref_p[k].norm() + 1e-9)) for k in got)
    print(f"[lock-step {rule}] 300 steps: worst per-step loss rel err {worst:.2e}, param rel err {perr:.2e}")
    assert worst < 1e-2
    assert perr < 5e-3


# Whether the loss must halve: Adadelta, ProximalAdagrad and ProximalGradientDescent were seen to take the batch loss of
# this MLP from about 0.2 to below a fifth of that within 400 single-worker steps on the cpu backend. FTRL was not: at
# lr 0.05 it went 0.230 -> 0.223 there, and at lr 0.5, which trains on one lane, 8 lanes here went 0.225 -> 2.1. Its
# curve is reported.
TRAINS = {"adadelta": True, "ftrl": False, "proximal_adagrad_l2": True, "proximal_sgd": True}


@pytest.mark.parametrize("case", [("graph", "adadelta"), ("row_split", "ftrl"), ("row_split", "proximal_adagrad_l2"),
                                  ("graph", "proximal_sgd")])
def test_eight_lanes_over_two_ps(case):
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    layout, rule = case
    kw = {"engine": "graph"} if layout == "graph" else {"sharding": "row_split"}
    cfg = EngineConfig(backend="cuda", lanes=8, nslots=16, **kw)
    ds = data.synthetic_mnist(8192, seed=6)
    with InProcessCluster(mlp.book_model(100), _opts()[rule], cfg, batch_size=32, num_ps=2) as cl:
        w = cl.worker
        assert w.engine == ("graph" if layout == "graph" else "fused")
        loader = w.make_loader(ds.images, ds.labels, seed=0)
        outs = list(w.run_steps(300, loader, wait_applied=True)) + list(w.run_steps(97, loader, wait_applied=True))
        assert len(outs) == 397 and w.read_global_step() == 397
        assert sorted(o.seq for o in outs) == list(range(1, 398))
        assert all(torch.isfinite(torch.tensor(o.loss)) for o in outs)
        first = sum(o.loss for o in outs[:20]) / 20
        last = sum(o.loss for o in outs[-20:]) / 20
        print(f"[8 lanes {layout} {rule}] loss {first:.4f} -> {last:.4f}")
        if TRAINS[rule]:
            assert last < 0.5 * first, (first, last)


@pytest.mark.timeout(420)
def test_proximal_adagrad_one_ps_two_workers_three_processes_one_gpu():
    """As tests/test_gpu_multiproc_one_gpu.py: every push applied exactly once, the loss falls, the ps exits."""
    common = ["--train_steps", "240", "--learning_rate", "0.05", "--log_every", "80", "--lanes", "4",
              "--optimizer", "proximal_adagrad", "--l2_regularization_strength", "0.001"]
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
    losses = [float(l.split("loss: ")[1]) for l in outs_w[0].splitlines() if l.startswith("Train step ")]
    if len(losses) >= 2:
        assert losses[-1] < losses[0]
