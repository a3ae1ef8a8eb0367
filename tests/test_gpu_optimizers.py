"""Momentum (and Nesterov), Adagrad and RMSProp on the GPU parameter server: the serve kernel's new instantiations
alone against the TF1 formulas in fp64, the fused engine in lock-step with fp32 PyTorch, pipelined runs on the graph
engine and with row_split sharding, and a 1 ps + 2 worker multi-process run on one GPU."""
import re

import _harness
import pytest
import torch

pytestmark = pytest.mark.gpu


def _opts():
    from dist_mnist_b200.parallel.config import OptimizerConfig
    return {
        "momentum": OptimizerConfig("momentum", 1e-2),
        "nesterov": OptimizerConfig("momentum", 1e-2, use_nesterov=True),
        "adagrad": OptimizerConfig("adagrad", 5e-2),
        "rmsprop": OptimizerConfig("rmsprop", 1e-3),
        "rmsprop_mom": OptimizerConfig("rmsprop", 1e-3, momentum=0.9),
    }


@pytest.mark.parametrize("rule", ["momentum", "nesterov", "adagrad", "rmsprop_mom"])
def test_serve_kernel_alone_matches_tf1_formulas(rule):
    """Both math modes, per push and merged, with the default geometry and with the register-resident one."""
    import dataclasses

    from bench_tools import gpu_check
    from dist_mnist_b200 import _native as N

    ok = True
    for math in ("fast", "ieee"):
        opt = dataclasses.replace(_opts()[rule], math=math)
        for mode in (N.APPLY_PER_PUSH, N.APPLY_MERGED):
            for resident in (False, True):
                ok &= gpu_check.check_ps_serve_tf1(opt, mode, resident=resident)
    assert ok


@pytest.mark.parametrize("rule", ["momentum", "nesterov", "adagrad", "rmsprop", "rmsprop_mom"])
def test_strict_fused_native_loop_is_lock_step_with_fp32_torch(rule):
    """300 strict steps (lanes=1) against an un-rounded fp32 PyTorch step on the same `next_batch` sequence, with the
    bounds of tests/test_gpu_fused_batches.py::test_strict_native_loop_is_lock_step_with_fp32_torch_at_batch."""
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


@pytest.mark.parametrize("case", [("graph", "rmsprop_mom"), ("row_split", "nesterov"), ("row_split", "adagrad")])
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
        first = sum(o.loss for o in outs[:20]) / 20
        last = sum(o.loss for o in outs[-20:]) / 20
        assert last < 0.5 * first, (first, last)


@pytest.mark.timeout(420)
def test_nesterov_one_ps_two_workers_three_processes_one_gpu():
    """As tests/test_gpu_multiproc_one_gpu.py: every push applied exactly once, the loss falls, the ps exits."""
    common = ["--train_steps", "240", "--learning_rate", "0.01", "--log_every", "80", "--lanes", "4",
              "--optimizer", "momentum", "--use_nesterov"]
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
