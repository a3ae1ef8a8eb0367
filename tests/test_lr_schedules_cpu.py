"""Learning-rate schedules on the parameter server, cpu backend: `LrSchedule.lr_at` against hand-computed TF1 values
and torch.optim.lr_scheduler, validation, lock-step runs that check parameters, both slot buffers and every item's
schedule step after every step, the ps / worker agreement on the schedule, checkpoint round trips and a multi-process
CLI run with a metrics file."""
import json
import math
import os
import tempfile

import _harness
import pytest
import torch

from bench_tools.gpu_e2e import ref_slots, ref_step
from dist_mnist_b200 import cli
from dist_mnist_b200.cluster import ClusterSpec
from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.config import EngineConfig, LrSchedule, OptimizerConfig
from dist_mnist_b200.parallel.ps import ParameterServer
from dist_mnist_b200.parallel.worker import Worker
from dist_mnist_b200.session import InProcessCluster, free_port, train_loop
from dist_mnist_b200.utils import ckpt, data
from dist_mnist_b200.utils.metrics import TrainMetricsWriter


def _close(a, b, rel=1e-6):
    return a == pytest.approx(b, rel=rel, abs=1e-12)


# (schedule, lr0, step, hand-computed TF1 rate)
HAND = [
    (LrSchedule("exponential_decay", decay_steps=1000, decay_rate=0.96, staircase=True), 0.1, 0, 0.1),
    (LrSchedule("exponential_decay", decay_steps=1000, decay_rate=0.96, staircase=True), 0.1, 999, 0.1),
    (LrSchedule("exponential_decay", decay_steps=1000, decay_rate=0.96, staircase=True), 0.1, 1000, 0.096),
    (LrSchedule("exponential_decay", decay_steps=1000, decay_rate=0.96, staircase=True), 0.1, 2999, 0.09216),
    (LrSchedule("exponential_decay", decay_steps=1000, decay_rate=0.96), 0.1, 500, 0.1 * 0.96 ** 0.5),
    (LrSchedule("exponential_decay", decay_steps=3, decay_rate=0.9999995, staircase=True), 0.1, 2 ** 24 + 3,
     0.1 * 0.9999995 ** 5592406),
    (LrSchedule("inverse_time_decay", decay_steps=10, decay_rate=0.5), 0.1, 15, 0.1 / 1.75),
    (LrSchedule("inverse_time_decay", decay_steps=10, decay_rate=0.5, staircase=True), 0.1, 15, 0.1 / 1.5),
    (LrSchedule("inverse_time_decay", decay_steps=10, decay_rate=0.5, staircase=True), 0.1, 20, 0.05),
    (LrSchedule("natural_exp_decay", decay_steps=10, decay_rate=0.5), 0.1, 20, 0.1 * math.exp(-1.0)),
    (LrSchedule("natural_exp_decay", decay_steps=10, decay_rate=0.5, staircase=True), 0.1, 29, 0.1 * math.exp(-1.0)),
    (LrSchedule("polynomial_decay", decay_steps=100, end_learning_rate=0.01, power=2.0), 0.1, 50, 0.0325),
    (LrSchedule("polynomial_decay", decay_steps=100, end_learning_rate=0.01, power=2.0), 0.1, 150, 0.01),
    (LrSchedule("polynomial_decay", decay_steps=100), 0.1, 25, (0.1 - 1e-4) * 0.75 + 1e-4),
    (LrSchedule("polynomial_decay", decay_steps=100, end_learning_rate=0.01, power=2.0, cycle=True), 0.1, 0, 0.1),
    (LrSchedule("polynomial_decay", decay_steps=100, end_learning_rate=0.01, power=2.0, cycle=True), 0.1, 100, 0.01),
    (LrSchedule("polynomial_decay", decay_steps=100, end_learning_rate=0.01, power=2.0, cycle=True), 0.1, 150,
     0.09 * 0.25 ** 2 + 0.01),
    (LrSchedule("polynomial_decay", decay_steps=100, end_learning_rate=0.01, power=2.0, cycle=True), 0.1, 200, 0.01),
    (LrSchedule("polynomial_decay", decay_steps=100, end_learning_rate=0.01, power=2.0, cycle=True), 0.1, 201,
     0.09 * (99 / 300) ** 2 + 0.01),
    (LrSchedule("cosine_decay", decay_steps=100, alpha=0.1), 0.1, 0, 0.1),
    (LrSchedule("cosine_decay", decay_steps=100, alpha=0.1), 0.1, 50, 0.055),
    (LrSchedule("cosine_decay", decay_steps=100, alpha=0.1), 0.1, 100, 0.01),
    (LrSchedule("cosine_decay", decay_steps=100, alpha=0.1), 0.1, 1000, 0.01),
    (LrSchedule("cosine_decay", decay_steps=100), 0.1, 100, 0.0),
    (LrSchedule("piecewise_constant", boundaries=(100, 200), values=(1.0, 0.5, 0.1)), None, 100, 1.0),
    (LrSchedule("piecewise_constant", boundaries=(100, 200), values=(1.0, 0.5, 0.1)), None, 101, 0.5),
    (LrSchedule("piecewise_constant", boundaries=(100, 200), values=(1.0, 0.5, 0.1)), None, 200, 0.5),
    (LrSchedule("piecewise_constant", boundaries=(100, 200), values=(1.0, 0.5, 0.1)), None, 201, 0.1),
    # exact past 2^24, where a float32 cast of the step would make 2^24 + 3 and 2^24 + 4 equal
    (LrSchedule("piecewise_constant", boundaries=(2 ** 24 + 3,), values=(1.0, 0.5)), None, 2 ** 24 + 3, 1.0),
    (LrSchedule("piecewise_constant", boundaries=(2 ** 24 + 3,), values=(1.0, 0.5)), None, 2 ** 24 + 4, 0.5),
    (LrSchedule(), 0.1, 12345, 0.1),
]


@pytest.mark.parametrize("case", range(len(HAND)))
def test_lr_at_matches_hand_computed_tf1_values(case):
    sched, lr0, step, want = HAND[case]
    assert _close(sched.lr_at(step, lr0), want), (sched, step)


def _torch_lrs(make, lr0, n):
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=lr0)
    sch = make(opt)
    out = []
    for _ in range(n):
        out.append(opt.param_groups[0]["lr"])
        opt.step()
        sch.step()
    return out


@pytest.mark.parametrize("case", ["step", "exponential", "polynomial", "multistep", "cosine"])
def test_lr_at_agrees_with_torch_lr_scheduler(case):
    S = torch.optim.lr_scheduler
    lr0 = 0.1
    if case == "step":      # staircase exponential_decay = StepLR
        sched, ref = LrSchedule("exponential_decay", decay_steps=7, decay_rate=0.5, staircase=True), \
            _torch_lrs(lambda o: S.StepLR(o, step_size=7, gamma=0.5), lr0, 40)
    elif case == "exponential":   # decay_steps = 1: ExponentialLR
        sched, ref = LrSchedule("exponential_decay", decay_steps=1, decay_rate=0.9), \
            _torch_lrs(lambda o: S.ExponentialLR(o, gamma=0.9), lr0, 40)
    elif case == "polynomial":    # end_learning_rate 0, no cycle: PolynomialLR
        sched, ref = LrSchedule("polynomial_decay", decay_steps=25, end_learning_rate=0.0, power=2.0), \
            _torch_lrs(lambda o: S.PolynomialLR(o, total_iters=25, power=2.0), lr0, 40)
    elif case == "multistep":     # TF's `s <= b` keeps values[i] at the boundary: milestone b + 1
        sched = LrSchedule("piecewise_constant", boundaries=(5, 12, 20), values=(0.1, 0.01, 0.001, 0.0001))
        ref = _torch_lrs(lambda o: S.MultiStepLR(o, milestones=[6, 13, 21], gamma=0.1), lr0, 40)
    else:                         # cosine_decay up to decay_steps: CosineAnnealingLR with eta_min = alpha lr0
        sched, ref = LrSchedule("cosine_decay", decay_steps=30, alpha=0.2), \
            _torch_lrs(lambda o: S.CosineAnnealingLR(o, T_max=30, eta_min=0.02), lr0, 31)
    for s, want in enumerate(ref):
        assert sched.lr_at(s, lr0) == pytest.approx(want, rel=1e-5, abs=1e-9), (case, s)


def test_schedule_validation():
    ok = LrSchedule("polynomial_decay", decay_steps=10)
    assert (ok.end_learning_rate, ok.power, ok.cycle) == (1e-4, 1.0, False)
    assert LrSchedule("cosine_decay", decay_steps=10).alpha == 0.0
    assert LrSchedule().constant and OptimizerConfig("adam", 1e-3).schedule == LrSchedule()
    bad = [
        dict(kind="exponential_decay", decay_rate=0.5),                       # decay_steps missing
        dict(kind="exponential_decay", decay_steps=10),                       # decay_rate missing
        dict(kind="inverse_time_decay", decay_steps=0, decay_rate=0.5),
        dict(kind="cosine_decay", decay_steps=-3),
        dict(kind="polynomial_decay"),
        dict(kind="linear_decay", decay_steps=3),
        dict(kind="cosine_decay", decay_steps=10, decay_rate=0.5),            # a parameter it does not use
        dict(kind="cosine_decay", decay_steps=10, staircase=True),
        dict(kind="exponential_decay", decay_steps=10, decay_rate=0.5, cycle=True),
        dict(kind="constant", decay_steps=10),
        dict(kind="constant", alpha=0.0),
        dict(kind="piecewise_constant", boundaries=(), values=(0.1,)),
        dict(kind="piecewise_constant", boundaries=(5, 5), values=(0.1, 0.2, 0.3)),
        dict(kind="piecewise_constant", boundaries=(5, 4), values=(0.1, 0.2, 0.3)),
        dict(kind="piecewise_constant", boundaries=(5,), values=(0.1,)),
        dict(kind="piecewise_constant", boundaries=tuple(range(1, 10)), values=(0.1,) * 10),   # > 8 boundaries
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            LrSchedule(**kw)
    LrSchedule("piecewise_constant", boundaries=tuple(range(1, 9)), values=(0.1,) * 9)


def test_atomic_push_mode_refuses_a_schedule():
    sched = LrSchedule("exponential_decay", decay_steps=10, decay_rate=0.5)
    EngineConfig(backend="cuda", push_mode="atomic").validate(OptimizerConfig("sgd", 0.05))
    with pytest.raises(ValueError, match="schedule"):
        EngineConfig(backend="cuda", push_mode="atomic").validate(OptimizerConfig("sgd", 0.05, schedule=sched))


def _opt(argv):
    return cli.optimizer_config_from_args(cli.build_parser().parse_args(argv))


def test_cli_schedule_flags():
    assert _opt([]).schedule == LrSchedule()
    o = _opt(["--learning_rate", "0.1", "--lr_schedule", "exponential_decay", "--decay_steps", "1000",
              "--decay_rate", "0.96", "--staircase"])
    assert o.lr == 0.1 and o.schedule == LrSchedule("exponential_decay", decay_steps=1000, decay_rate=0.96,
                                                    staircase=True)
    o = _opt(["--lr_schedule", "polynomial_decay", "--decay_steps", "50", "--end_learning_rate", "0.001",
              "--power", "0.5", "--cycle"])
    assert o.schedule == LrSchedule("polynomial_decay", decay_steps=50, end_learning_rate=0.001, power=0.5, cycle=True)
    assert _opt(["--lr_schedule", "cosine_decay", "--decay_steps", "9", "--alpha", "0.1"]).schedule.alpha == 0.1
    o = _opt(["--lr_schedule", "piecewise_constant", "--lr_boundaries", "1000,2000", "--lr_values", "0.1,0.01,0.001"])
    assert o.schedule.boundaries == (1000, 2000) and o.schedule.values == (0.1, 0.01, 0.001)
    for argv in (["--lr_schedule", "cosine_decay", "--decay_steps", "9", "--decay_rate", "0.5"],
                 ["--staircase"], ["--decay_steps", "10"], ["--lr_values", "0.1"],
                 ["--lr_schedule", "exponential_decay", "--decay_rate", "0.5"],
                 ["--lr_schedule", "exponential_decay", "--decay_steps", "10", "--decay_rate", "0.5", "--alpha", "0"],
                 ["--lr_schedule", "polynomial_decay", "--decay_steps", "10", "--staircase"],
                 ["--lr_schedule", "piecewise_constant", "--lr_boundaries", "10", "--lr_values", "0.1,0.01",
                  "--learning_rate", "0.1"],
                 ["--lr_schedule", "piecewise_constant", "--lr_boundaries", "1,2,3,4,5,6,7,8,9",
                  "--lr_values", "1,1,1,1,1,1,1,1,1,1"]):
        with pytest.raises(ValueError):
            _opt(argv)


def test_metrics_lines_gain_learning_rate_only_with_a_schedule():
    class O:
        def __init__(self, gs):
            self.loss, self.correct, self.global_step = 0.5, 10, gs

    sched = LrSchedule("exponential_decay", decay_steps=10, decay_rate=0.5, staircase=True)
    for lr_at in (None, lambda s: sched.lr_at(s, 0.1)):
        with tempfile.NamedTemporaryFile("r", suffix=".jsonl") as f:
            m = TrainMetricsWriter(f.name, 0, 32, every_steps=5, lr_at=lr_at)
            m.update([O(g) for g in range(1, 31)])
            m.close()
            recs = [json.loads(l) for l in open(f.name)]
        assert [r["global_step"] for r in recs] == [5, 10, 15, 20, 25, 30]
        for r in recs:
            if lr_at is None:
                assert "learning_rate" not in r
            else:
                assert r["learning_rate"] == sched.lr_at(r["global_step"], 0.1)


RULES = {"sgd": ("sgd", 5e-2), "adam": ("adam", 1e-3), "momentum": ("momentum", 1e-2), "rmsprop": ("rmsprop", 1e-3)}
# every one changes the rate inside an 8-step run
SCHEDULES = {
    "exponential_staircase": LrSchedule("exponential_decay", decay_steps=3, decay_rate=0.5, staircase=True),
    "polynomial_cycle": LrSchedule("polynomial_decay", decay_steps=3, end_learning_rate=1e-4, power=2.0, cycle=True),
    "cosine": LrSchedule("cosine_decay", decay_steps=6, alpha=0.125),
    "piecewise": None,   # values relative to the rule's lr, built in the test
}


def _schedule(name, lr):
    if name == "piecewise":
        return LrSchedule("piecewise_constant", boundaries=(2, 5), values=(lr, lr / 2, lr / 8))
    return SCHEDULES[name]


@pytest.mark.parametrize("mode", [(1, "per_push"), (2, "merged"), (2, "per_push"), (1, "merged")])
@pytest.mark.parametrize("sched", list(SCHEDULES))
@pytest.mark.parametrize("rule", list(RULES))
def test_lockstep_trajectory_under_a_schedule(rule, sched, mode):
    """Tolerances of tests/test_optimizers_cpu.py::test_lockstep_trajectory_matches_tf1_formulas; push i (0-based) is
    applied at schedule step i on every item."""
    nps, apply_mode = mode
    kind, lr = RULES[rule]
    opt = OptimizerConfig(kind, lr, schedule=_schedule(sched, lr))
    spec = mlp.book_model(100)
    cfg = EngineConfig(backend="cpu", apply_mode=apply_mode)
    ds = data.synthetic_mnist(512, seed=2)
    it = data.BatchIterator(ds, seed=0)
    params = mlp.init_params(spec, seed=5)
    rp = {k: v.clone() for k, v in params.items()}
    rm, rv = ref_slots(opt, params)
    t = 0
    rates = {opt.lr_at(i) for i in range(8)}
    assert len(rates) >= 3, rates
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=nps, params=params) as cl:
        w = cl.worker
        for k in range(nps):
            assert set(w.read_sched_steps(k)) == {0}
        for i in range(8):
            x, y = it.next_batch(32)
            r = w.step(x, y)
            w.wait_applied()
            lref, t = ref_step(spec, rp, rm, rv, t, x, y, opt, lr=opt.lr_at(i))
            assert r.loss == pytest.approx(lref, rel=1e-4)
            got, gm, gv = w.read_variables(), w.read_variables("adam_m"), w.read_variables("adam_v")
            for k in got:
                assert torch.allclose(got[k], rp[k], rtol=1e-4, atol=1e-6), (i, k)
                assert torch.allclose(gm[k], rm[k], rtol=1e-4, atol=1e-7), (i, k)
                assert torch.allclose(gv[k], rv[k], rtol=1e-4, atol=1e-7), (i, k)
            for k in range(nps):
                assert set(w.read_sched_steps(k)) == {i + 1}, (i, k)
        assert w.read_global_step() == 8


@pytest.mark.parametrize("ps_sched,w_sched", [
    (LrSchedule("exponential_decay", decay_steps=10, decay_rate=0.5), LrSchedule()),
    (LrSchedule(), LrSchedule("cosine_decay", decay_steps=10)),
    (LrSchedule("exponential_decay", decay_steps=10, decay_rate=0.5),
     LrSchedule("exponential_decay", decay_steps=10, decay_rate=0.25)),
    (LrSchedule("piecewise_constant", boundaries=(3,), values=(0.1, 0.01)),
     LrSchedule("piecewise_constant", boundaries=(4,), values=(0.1, 0.01))),
])
def test_worker_refuses_a_ps_with_another_schedule(ps_sched, w_sched):
    spec = mlp.book_model(32)
    cfg = EngineConfig(backend="cpu")
    cluster = ClusterSpec((f"127.0.0.1:{free_port()}",), (f"127.0.0.1:{free_port()}",))
    ps = ParameterServer(cluster, 0, spec, OptimizerConfig("adam", 1e-3, schedule=ps_sched), cfg)
    try:
        w = Worker(cluster, 0, spec, OptimizerConfig("adam", 1e-3, schedule=w_sched), cfg)
        with pytest.raises(RuntimeError, match="different engine configuration"):
            w.connect()
    finally:
        ps.close()


def test_worker_accepts_a_ps_with_the_same_schedule():
    spec = mlp.book_model(32)
    cfg = EngineConfig(backend="cpu")
    sched = LrSchedule("piecewise_constant", boundaries=(3, 9), values=(0.1, 0.01, 0.001))
    opt = OptimizerConfig("momentum", 1e-3, schedule=sched)
    with InProcessCluster(spec, opt, cfg, batch_size=16) as cl:
        assert cl.worker.opt.schedule == sched


# a schedule whose rate at the checkpoint's step (30) differs from its rate at step 0
CKPT_SCHED = LrSchedule("piecewise_constant", boundaries=(20,), values=(0.05, 0.005))


@pytest.mark.parametrize("restore_num_ps", [2, 1])
def test_checkpoint_restore_continues_the_schedule_at_the_global_step(restore_num_ps):
    """Saved with 2 ps; restored with 2 (item state restored) or 1 (another tiling: item state restarts): either way
    every item is at schedule step 30 and the next push is applied at lr(30), not lr(0)."""
    spec = mlp.book_model(64)
    opt = OptimizerConfig("sgd", 0.05, schedule=CKPT_SCHED)
    cfg = EngineConfig(backend="cpu")
    ds = data.synthetic_mnist(512, seed=0)
    d = tempfile.mkdtemp()
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=2) as cl:
        train_loop(cl.worker, ds, train_steps=30, log_every=0, checkpoint_dir=d, chunk=10)
    state = torch.load(ckpt.latest_checkpoint(d), weights_only=False)
    assert state["global_step"] == 30
    assert LrSchedule.from_dict(state["optimizer"]["schedule"]) == CKPT_SCHED
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=restore_num_ps, restore_dir=d) as cl:
        w = cl.worker
        assert w.read_global_step() == 30
        for k in range(restore_num_ps):
            assert set(w.read_sched_steps(k)) == {30}
        before = w.read_variables()
        x, y = data.BatchIterator(ds, seed=3).next_batch(32)
        w.step(x, y)
        w.wait_applied()
        after = w.read_variables()
        for k in range(restore_num_ps):
            assert set(w.read_sched_steps(k)) == {31}
    _, grads, _ = mlp.manual_loss_and_grads(spec, before, x, y)
    for k in after:
        want = before[k] - opt.lr_at(30) * grads[k]
        assert torch.allclose(after[k], want, rtol=1e-5, atol=1e-7), k
        assert not torch.allclose(after[k], before[k] - opt.lr_at(0) * grads[k], rtol=1e-5, atol=1e-7), k


def test_restore_under_another_schedule_is_allowed():
    spec = mlp.book_model(32)
    cfg = EngineConfig(backend="cpu")
    ds = data.synthetic_mnist(256, seed=0)
    d = tempfile.mkdtemp()
    with InProcessCluster(spec, OptimizerConfig("adam", 1e-3), cfg, batch_size=16) as cl:
        train_loop(cl.worker, ds, train_steps=10, log_every=0, checkpoint_dir=d, chunk=10)
    opt = OptimizerConfig("adam", 1e-3, schedule=LrSchedule("cosine_decay", decay_steps=100))
    with InProcessCluster(spec, opt, cfg, batch_size=16, restore_dir=d) as cl:
        assert cl.worker.read_global_step() == 10
        assert set(cl.worker.read_sched_steps(0)) == {10}


@pytest.mark.timeout(180)
def test_cli_exponential_staircase_one_ps_two_workers_metrics_learning_rate():
    sched_flags = ["--lr_schedule", "exponential_decay", "--decay_steps", "100", "--decay_rate", "0.5", "--staircase"]
    common = ["--train_steps", "400", "--learning_rate", "0.05", "--optimizer", "sgd", "--log_every", "50",
              *sched_flags]
    d = tempfile.mkdtemp()
    files = [os.path.join(d, f"w{i}.jsonl") for i in range(2)]
    with _harness.Tasks() as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done"])
        ws = [t.spawn("worker", i, common + ["--metrics_file", files[i]]) for i in (1, 0)]
        outs = [t.finish(w, 120) for w in ws]
        outp = t.finish(ps, 60)
    for w, o in zip(ws, outs):
        assert w.returncode == 0, o
    assert ps.returncode == 0, outp
    logged = [l for o in outs for l in o.splitlines() if l.startswith("Train step ")]
    assert logged and all(", loss: " in l for l in logged)      # the stdout contract is unchanged
    gstep = int(outp.split("exiting: global_step=")[1].split()[0])
    total = sum(int(l.split("local_steps=")[1].split()[0]) for o in outs for l in o.splitlines() if "local_steps=" in l)
    assert gstep == total
    sched = LrSchedule("exponential_decay", decay_steps=100, decay_rate=0.5, staircase=True)
    recs = [json.loads(l) for f in files for l in open(f)]
    assert recs
    for r in recs:
        assert r["learning_rate"] == sched.lr_at(r["global_step"], 0.05), r
    assert len({r["learning_rate"] for r in recs}) >= 3      # the rate fell during the run
