"""Learning-rate schedules on the GPU parameter server: the scheduled serve-kernel instantiations alone against fp64,
the fused engine in lock-step with fp32 PyTorch while the rate changes, pipelined runs on the graph engine and with
row_split sharding that end with every item at the global step, and a 1 ps + 2 worker multi-process run on one GPU."""
import json
import os
import re
import tempfile

import _harness
import pytest

pytestmark = pytest.mark.gpu


def _schedules():
    """(schedule, starting sched_step) per case. Decay rates are exact in fp32, so the fp32 kernel and the fp64
    reference differ by rounding only. The first starts just below 2^24 and crosses a staircase boundary (at 2^24)
    in the middle of a pass."""
    from dist_mnist_b200.parallel.config import LrSchedule
    return {
        "exponential_staircase_2p24": (LrSchedule("exponential_decay", decay_steps=1 << 20, decay_rate=0.96875,
                                                  staircase=True), (1 << 24) - 4),
        "exponential": (LrSchedule("exponential_decay", decay_steps=4, decay_rate=0.75), 1),
        "inverse_time": (LrSchedule("inverse_time_decay", decay_steps=4, decay_rate=0.5), 3),
        "natural_exp_staircase": (LrSchedule("natural_exp_decay", decay_steps=5, decay_rate=0.25, staircase=True), 0),
        "polynomial_cycle": (LrSchedule("polynomial_decay", decay_steps=4, end_learning_rate=1e-4, power=2.0,
                                        cycle=True), 0),
        "cosine": (LrSchedule("cosine_decay", decay_steps=7, alpha=0.125), 2),
        "piecewise": (LrSchedule("piecewise_constant", boundaries=(3, 5, 7), values=(1e-2, 5e-3, 2e-3, 1e-3)), 0),
    }


def _run_serve_checks(opt, sched_step):
    from bench_tools import gpu_check
    from dist_mnist_b200 import _native as N

    ok = True
    for mode in (N.APPLY_PER_PUSH, N.APPLY_MERGED):
        for resident in (False, True):
            ok &= gpu_check.check_ps_serve_tf1(opt, mode, resident=resident, sched_step=sched_step)
    return ok


@pytest.mark.parametrize("sched", list(_schedules()))
def test_scheduled_serve_kernel_adam_and_sgd_match_fp64(sched):
    """Adam (fast and IEEE) and SGD, per push and merged, default and register-resident geometry, with the bounds of
    check_ps_serve_tf1; every item ends at its starting schedule step plus the 9 pushes."""
    from dist_mnist_b200.parallel.config import OptimizerConfig

    schedule, s0 = _schedules()[sched]
    ok = True
    for opt in (OptimizerConfig("adam", 1e-2, schedule=schedule), OptimizerConfig("adam", 1e-2, math="ieee",
                                                                                  schedule=schedule),
                OptimizerConfig("sgd", 5e-2, schedule=schedule)):
        ok &= _run_serve_checks(opt, s0)
    assert ok


@pytest.mark.parametrize("case", [("momentum", "exponential_staircase_2p24"), ("nesterov", "piecewise"),
                                  ("adagrad", "cosine"), ("rmsprop_mom", "polynomial_cycle"),
                                  ("rmsprop", "inverse_time")])
def test_scheduled_serve_kernel_tf1_rules_match_fp64(case):
    """Momentum / Nesterov, Adagrad and RMSProp in both math modes."""
    import dataclasses

    from dist_mnist_b200.parallel.config import OptimizerConfig

    rule, sched = case
    schedule, s0 = _schedules()[sched]
    base = {"momentum": OptimizerConfig("momentum", 1e-2), "nesterov": OptimizerConfig("momentum", 1e-2,
                                                                                        use_nesterov=True),
            "adagrad": OptimizerConfig("adagrad", 5e-2), "rmsprop": OptimizerConfig("rmsprop", 1e-3),
            "rmsprop_mom": OptimizerConfig("rmsprop", 1e-3, momentum=0.9)}[rule]
    ok = True
    for math in ("fast", "ieee"):
        ok &= _run_serve_checks(dataclasses.replace(base, math=math, schedule=schedule), s0)
    assert ok


def test_check_ps_serve_takes_a_schedule():
    from bench_tools import gpu_check

    schedule, s0 = _schedules()["exponential_staircase_2p24"]
    assert gpu_check.check_ps_serve(schedule=schedule, sched_step=(1 << 24) - 2)
    assert gpu_check.check_ps_serve(ieee=True, schedule=_schedules()["cosine"][0], sched_step=5)


@pytest.mark.parametrize("rule", ["sgd", "momentum"])
def test_strict_fused_native_loop_under_a_schedule_is_lock_step_with_fp32_torch(rule):
    """300 strict steps (lanes=1): step i is applied at lr(i). Bounds of
    tests/test_gpu_optimizers.py::test_strict_fused_native_loop_is_lock_step_with_fp32_torch. Adam is not among the
    rules: at a constant rate of 1e-3 it already ends 6.9e-3 from fp32 PyTorch here, above the parameter bound (its
    normalised update amplifies rounding); its scheduled serve kernels are checked against fp64 above."""
    from bench_tools.gpu_e2e import ref_slots, ref_step
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, LrSchedule, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    if rule == "sgd":
        opt = OptimizerConfig("sgd", 5e-2, schedule=LrSchedule("piecewise_constant", boundaries=(60, 150, 230),
                                                                values=(5e-2, 2e-2, 1e-2, 5e-3)))
    else:
        opt = OptimizerConfig("momentum", 1e-2, schedule=LrSchedule("exponential_decay", decay_steps=50,
                                                                     decay_rate=0.75, staircase=True))
    assert len({opt.lr_at(i) for i in range(300)}) >= 4
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
        assert set(w.read_sched_steps(0)) == {300}
        t, worst = 0, 0.0
        for i, o in enumerate(outs):
            x, y = twin.next_batch()
            lref, t = ref_step(spec, ref_p, ref_m, ref_v, t, x, y, opt, lr=opt.lr_at(i))
            assert o.global_step == o.seq
            if lref > 1e-6:
                worst = max(worst, abs(o.loss - lref) / abs(lref))
        got = w.read_variables()
    perr = max(float((got[k] - ref_p[k]).norm() / (ref_p[k].norm() + 1e-9)) for k in got)
    print(f"[lock-step {rule} scheduled] 300 steps: worst per-step loss rel err {worst:.2e}, param rel err {perr:.2e}")
    assert worst < 1e-2
    assert perr < 5e-3


@pytest.mark.parametrize("layout", ["graph", "row_split"])
def test_eight_lanes_over_two_ps_end_at_the_global_step(layout):
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, LrSchedule, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    if layout == "graph":
        opt = OptimizerConfig("rmsprop", 1e-3, momentum=0.9,
                              schedule=LrSchedule("exponential_decay", decay_steps=200, decay_rate=0.5))
        kw = {"engine": "graph"}
    else:
        opt = OptimizerConfig("momentum", 1e-2, use_nesterov=True,
                              schedule=LrSchedule("cosine_decay", decay_steps=400, alpha=0.25))
        kw = {"sharding": "row_split"}
    cfg = EngineConfig(backend="cuda", lanes=8, nslots=16, **kw)
    ds = data.synthetic_mnist(8192, seed=6)
    with InProcessCluster(mlp.book_model(100), opt, cfg, batch_size=32, num_ps=2) as cl:
        w = cl.worker
        assert w.engine == ("graph" if layout == "graph" else "fused")
        loader = w.make_loader(ds.images, ds.labels, seed=0)
        outs = list(w.run_steps(300, loader, wait_applied=True)) + list(w.run_steps(97, loader, wait_applied=True))
        assert len(outs) == 397 and w.read_global_step() == 397
        assert sorted(o.seq for o in outs) == list(range(1, 398))
        for k in range(2):
            assert set(w.read_sched_steps(k)) == {397}, k
        first = sum(o.loss for o in outs[:20]) / 20
        last = sum(o.loss for o in outs[-20:]) / 20
        assert last < 0.5 * first, (first, last)


@pytest.mark.timeout(420)
def test_cosine_decay_one_ps_two_workers_three_processes_one_gpu():
    """As tests/test_gpu_optimizers.py::test_nesterov_one_ps_two_workers_three_processes_one_gpu, and the metrics
    file's learning_rate is lr_at(global_step)."""
    from dist_mnist_b200.parallel.config import LrSchedule

    common = ["--train_steps", "240", "--learning_rate", "0.01", "--log_every", "80", "--lanes", "4",
              "--optimizer", "momentum", "--lr_schedule", "cosine_decay", "--decay_steps", "240", "--alpha", "0.1"]
    d = tempfile.mkdtemp()
    files = [os.path.join(d, f"w{i}.jsonl") for i in range(2)]
    with _harness.Tasks(backend="cuda", gpu=0) as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done"])
        ws = [t.spawn("worker", i, common + ["--metrics_file", files[i]]) for i in range(2)]
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
    sched = LrSchedule("cosine_decay", decay_steps=240, alpha=0.1)
    recs = [json.loads(l) for f in files for l in open(f)]
    assert recs
    for r in recs:
        assert r["learning_rate"] == sched.lr_at(r["global_step"], 0.01), r
    losses = [float(l.split("loss: ")[1]) for l in outs_w[0].splitlines() if l.startswith("Train step ")]
    if len(losses) >= 2:
        assert losses[-1] < losses[0]
