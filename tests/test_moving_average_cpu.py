"""Exponential moving averages of the model variables on the parameter server (TF1 `ExponentialMovingAverage.apply`
after every optimizer step), cpu backend: `ema_decay_at` against hand-computed TF1 values, validation of the config and
the CLI flags, lock-step runs that check parameters, both slot buffers, the shadows and every item's step count after
every step, the ps / worker agreement on averaging, checkpoint round trips, `evaluate(moving_averages=True)` and a
multi-process CLI run whose checkpoint holds the shadows."""
import tempfile

import _harness
import pytest
import torch

from bench_tools.gpu_e2e import ref_ema, ref_slots, ref_step
from dist_mnist_b200 import cli
from dist_mnist_b200.cluster import ClusterSpec
from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.config import EngineConfig, LrSchedule, OptimizerConfig
from dist_mnist_b200.parallel.ps import ParameterServer
from dist_mnist_b200.parallel.worker import Worker
from dist_mnist_b200.session import InProcessCluster, free_port, train_loop
from dist_mnist_b200.utils import ckpt, data


def _f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def test_ema_decay_at_matches_tf1():
    # TF1: decay = min(decay, (1 + num_updates) / (10 + num_updates)), in float32
    o = OptimizerConfig("sgd", 0.1, moving_average_decay=0.999)
    assert o.ema_decay_at(0) == _f32(0.1)              # (1 + 0) / (10 + 0)
    assert o.ema_decay_at(1) == _f32(2 / 11)
    assert o.ema_decay_at(10) == _f32(0.55)
    assert o.ema_decay_at(990) == _f32(991 / 1000)      # warm-up: (1+n)/(10+n) < decay
    assert o.ema_decay_at(8990) == _f32(0.999)          # (1+n)/(10+n) = 0.999 exactly: the threshold
    assert o.ema_decay_at(100000) == _f32(0.999)
    assert o.ema_decay_at(2 ** 32 - 1) == _f32(0.999)
    o = OptimizerConfig("adam", 1e-3, moving_average_decay=0.9999)
    assert o.ema_decay_at(5000) == _f32(5001 / 5010)
    assert o.ema_decay_at(89990) == _f32(0.9999)
    # without num_updates the decay never warms up
    o = OptimizerConfig("sgd", 0.1, moving_average_decay=0.99, moving_average_num_updates=False)
    assert [o.ema_decay_at(n) for n in (0, 1, 10, 10 ** 6)] == [_f32(0.99)] * 4
    with pytest.raises(ValueError):
        OptimizerConfig("sgd", 0.1).ema_decay_at(1)


def test_config_validation_and_as_dict():
    assert not OptimizerConfig("adam").moving_averages
    o = OptimizerConfig("momentum", 0.01, moving_average_decay=0.99, moving_average_num_updates=False)
    assert o.moving_averages
    d = o.as_dict()
    assert d["moving_average_decay"] == 0.99 and d["moving_average_num_updates"] is False
    assert OptimizerConfig("adam").as_dict()["moving_average_decay"] is None
    for bad in (0.0, 1.0, -0.5, 1.5, float("nan"), True):
        with pytest.raises(ValueError):
            OptimizerConfig("sgd", 0.1, moving_average_decay=bad)


def test_atomic_push_mode_refuses_averaging():
    opt = OptimizerConfig("sgd", 0.1, moving_average_decay=0.99)
    with pytest.raises(ValueError, match="moving_average_decay"):
        EngineConfig(backend="cuda", push_mode="atomic").validate(opt)
    EngineConfig(backend="cuda", push_mode="mailbox").validate(opt)


def _opt(argv):
    return cli.optimizer_config_from_args(cli.build_parser().parse_args(argv))


def test_cli_moving_average_flags():
    o = _opt([])
    assert o.moving_average_decay is None and o.moving_average_num_updates
    o = _opt(["--moving_average_decay", "0.9999"])
    assert o.moving_average_decay == 0.9999 and o.moving_average_num_updates
    o = _opt(["--moving_average_decay", "0.999", "--moving_average_num_updates", "none"])
    assert o.moving_average_decay == 0.999 and not o.moving_average_num_updates
    o = _opt(["--moving_average_decay", "0.999", "--moving_average_num_updates", "global_step"])
    assert o.moving_average_num_updates
    for argv in (["--moving_average_num_updates", "global_step"], ["--moving_average_num_updates", "none"],
                 ["--moving_average_decay", "1.0"], ["--moving_average_decay", "0"]):
        with pytest.raises(ValueError):
            _opt(argv)
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["--moving_average_num_updates", "sometimes"])


RULES = {"sgd": ("sgd", 5e-2), "adam": ("adam", 1e-3), "momentum": ("momentum", 1e-2), "rmsprop": ("rmsprop", 1e-3)}
# (rule, schedule): RMSProp runs both with a constant rate and under a schedule
CASES = [("sgd", None), ("adam", None), ("momentum", None), ("rmsprop", None),
         ("rmsprop", LrSchedule("exponential_decay", decay_steps=3, decay_rate=0.5, staircase=True))]


@pytest.mark.parametrize("mode", [(1, "per_push"), (2, "merged"), (2, "per_push"), (1, "merged")])
@pytest.mark.parametrize("case", range(len(CASES)), ids=[f"{r}-{'sched' if s else 'const'}" for r, s in CASES])
def test_lockstep_trajectory_with_moving_averages(case, mode):
    """Tolerances of tests/test_lr_schedules_cpu.py::test_lockstep_trajectory_under_a_schedule; push i (0-based) is
    followed by the shadow update with decay ema_decay_at(i + 1) on every item, and every item has counted i + 1
    pushes afterwards, also at a constant rate. The warm-up (decay 0.99 reaches its bound only at step 890) makes the
    decay change at every step."""
    rule, sched = CASES[case]
    nps, apply_mode = mode
    kind, lr = RULES[rule]
    opt = OptimizerConfig(kind, lr, schedule=sched or LrSchedule(), moving_average_decay=0.99)
    spec = mlp.book_model(100)
    cfg = EngineConfig(backend="cpu", apply_mode=apply_mode)
    ds = data.synthetic_mnist(512, seed=2)
    it = data.BatchIterator(ds, seed=0)
    params = mlp.init_params(spec, seed=5)
    rp = {k: v.clone() for k, v in params.items()}
    re = {k: v.clone() for k, v in params.items()}
    rm, rv = ref_slots(opt, params)
    t = 0
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=nps, params=params) as cl:
        w = cl.worker
        shadows = w.read_variables("ema")
        for k in params:      # the shadows start at the initial values
            assert torch.equal(shadows[k], params[k]), k
        for k in range(nps):
            assert set(w.read_sched_steps(k)) == {0}
        for i in range(8):
            x, y = it.next_batch(32)
            r = w.step(x, y)
            w.wait_applied()
            lref, t = ref_step(spec, rp, rm, rv, t, x, y, opt, lr=opt.lr_at(i))
            ref_ema(opt, rp, re, i + 1)
            assert r.loss == pytest.approx(lref, rel=1e-4)
            got, gm, gv = w.read_variables(), w.read_variables("adam_m"), w.read_variables("adam_v")
            ge = w.read_variables("ema")
            for k in got:
                assert torch.allclose(got[k], rp[k], rtol=1e-4, atol=1e-6), (i, k)
                assert torch.allclose(gm[k], rm[k], rtol=1e-4, atol=1e-7), (i, k)
                assert torch.allclose(gv[k], rv[k], rtol=1e-4, atol=1e-7), (i, k)
                assert torch.allclose(ge[k], re[k], rtol=1e-4, atol=1e-6), (i, k)
            for k in range(nps):
                assert set(w.read_sched_steps(k)) == {i + 1}, (i, k)
        assert w.read_global_step() == 8
        moved = w.read_variables("ema")
        assert any(not torch.equal(moved[k], params[k]) for k in params)
        assert any(not torch.equal(moved[k], got[k]) for k in params)


def test_constant_rate_without_averaging_keeps_the_step_counter_at_zero():
    """Without averaging (and at a constant rate) the serve loop runs exactly as before: no step counting."""
    opt = OptimizerConfig("sgd", 0.05)
    with InProcessCluster(mlp.book_model(32), opt, EngineConfig(backend="cpu"), batch_size=16) as cl:
        x, y = data.BatchIterator(data.synthetic_mnist(64, seed=0), seed=0).next_batch(16)
        cl.worker.step(x, y)
        cl.worker.wait_applied()
        assert set(cl.worker.read_sched_steps(0)) == {0}
        with pytest.raises(ValueError, match="moving averages are off"):
            cl.worker.read_variables("ema")
        with pytest.raises(ValueError, match="moving averages are off"):
            cl.worker.write_variables(mlp.init_params(mlp.book_model(32), 0), "ema")
        with pytest.raises(ValueError, match="moving averages are off"):
            cl.worker.evaluate(x, y, moving_averages=True)


@pytest.mark.parametrize("ps_avg,w_avg", [
    ({"moving_average_decay": 0.99}, {}),
    ({}, {"moving_average_decay": 0.99}),
    ({"moving_average_decay": 0.99}, {"moving_average_decay": 0.999}),
    ({"moving_average_decay": 0.99}, {"moving_average_decay": 0.99, "moving_average_num_updates": False}),
])
def test_worker_refuses_a_ps_with_other_moving_averages(ps_avg, w_avg):
    spec = mlp.book_model(32)
    cfg = EngineConfig(backend="cpu")
    cluster = ClusterSpec((f"127.0.0.1:{free_port()}",), (f"127.0.0.1:{free_port()}",))
    ps = ParameterServer(cluster, 0, spec, OptimizerConfig("adam", 1e-3, **ps_avg), cfg)
    try:
        w = Worker(cluster, 0, spec, OptimizerConfig("adam", 1e-3, **w_avg), cfg)
        with pytest.raises(RuntimeError, match="different engine configuration"):
            w.connect()
    finally:
        ps.close()


def test_worker_accepts_a_ps_with_the_same_moving_averages():
    spec = mlp.book_model(32)
    opt = OptimizerConfig("momentum", 1e-2, moving_average_decay=0.999, moving_average_num_updates=False)
    with InProcessCluster(spec, opt, EngineConfig(backend="cpu"), batch_size=16) as cl:
        assert cl.worker.opt.moving_average_decay == 0.999
        assert set(cl.worker.read_variables("ema")) == set(cl.worker.read_variables())


AVG = OptimizerConfig("momentum", 1e-2, moving_average_decay=0.99)


def _train_and_save(opt, steps=30, num_ps=2):
    spec = mlp.book_model(64)
    ds = data.synthetic_mnist(512, seed=0)
    d = tempfile.mkdtemp()
    with InProcessCluster(spec, opt, EngineConfig(backend="cpu"), batch_size=32, num_ps=num_ps) as cl:
        train_loop(cl.worker, ds, train_steps=steps, log_every=0, checkpoint_dir=d, chunk=10)
        before = {r: cl.worker.read_variables(r) for r in ("params", "adam_m", "adam_v")}
        if opt.moving_averages:
            before["ema"] = cl.worker.read_variables("ema")
    return spec, ds, d, before


@pytest.mark.parametrize("restore_num_ps", [2, 1])
def test_checkpoint_roundtrip_keeps_the_moving_averages(restore_num_ps):
    spec, ds, d, before = _train_and_save(AVG)
    state = torch.load(ckpt.latest_checkpoint(d), weights_only=False)
    assert state["optimizer"]["moving_average_decay"] == 0.99 and state["optimizer"]["moving_average_num_updates"]
    assert set(state["ema"]) == set(state["variables"])
    for k in before["ema"]:
        assert torch.equal(state["ema"][k], before["ema"][k]), k
        assert not torch.equal(state["ema"][k], state["variables"][k]), k
    with InProcessCluster(spec, AVG, EngineConfig(backend="cpu"), batch_size=32, num_ps=restore_num_ps,
                          restore_dir=d) as cl:
        w = cl.worker
        assert w.read_global_step() == 30
        for k in range(restore_num_ps):
            assert set(w.read_sched_steps(k)) == {30}      # num_updates continues at the global step
        for r, vals in before.items():
            got = w.read_variables(r)
            for k in vals:
                assert torch.equal(got[k], vals[k]), (r, k)
        # the next step moves the shadows with the decay of step 31
        p0, e0 = w.read_variables(), w.read_variables("ema")
        x, y = data.BatchIterator(ds, seed=3).next_batch(32)
        w.step(x, y)
        w.wait_applied()
        p1, e1 = w.read_variables(), w.read_variables("ema")
        want = {k: v.clone() for k, v in e0.items()}
        ref_ema(AVG, p1, want, 31)
        for k in e1:
            assert torch.allclose(e1[k], want[k], rtol=1e-6, atol=1e-8), k
            assert not torch.equal(e1[k], e0[k]), k


def test_averaging_run_refuses_a_checkpoint_without_moving_averages():
    off = OptimizerConfig("momentum", 1e-2)
    spec, _, d, _ = _train_and_save(off, steps=10, num_ps=1)
    assert "ema" not in torch.load(ckpt.latest_checkpoint(d), weights_only=False)
    with InProcessCluster(spec, AVG, EngineConfig(backend="cpu"), batch_size=32) as cl:
        with pytest.raises(RuntimeError, match="no moving averages"):
            ckpt.restore_latest(cl.worker, d)
    with pytest.raises(RuntimeError, match="no moving averages"):
        ckpt.load_variables(d, moving_averages=True)


def test_run_without_averaging_ignores_saved_moving_averages():
    spec, _, d, before = _train_and_save(AVG, steps=10, num_ps=1)
    off = OptimizerConfig("momentum", 1e-2)
    with InProcessCluster(spec, off, EngineConfig(backend="cpu"), batch_size=32) as cl:
        assert ckpt.restore_latest(cl.worker, d) == 10
        got = cl.worker.read_variables()
        for k in got:
            assert torch.equal(got[k], before["params"][k]), k


def test_evaluate_moving_averages_is_the_forward_of_the_shadows():
    spec = mlp.book_model(64)
    opt = OptimizerConfig("sgd", 0.1, moving_average_decay=0.9)
    ds = data.synthetic_mnist(512, seed=1)
    with InProcessCluster(spec, opt, EngineConfig(backend="cpu"), batch_size=32) as cl:
        train_loop(cl.worker, ds, train_steps=20, log_every=0, chunk=10)
        images, labels = ds.images[:256], ds.labels[:256]
        shadows = cl.worker.read_variables("ema")
        loss, acc = cl.worker.evaluate(images, labels, moving_averages=True)
        loss_p, acc_p = cl.worker.evaluate(images, labels)
    logits, _ = mlp.forward_logits(spec, shadows, images.float())
    assert loss == pytest.approx(float(mlp.loss_from_logits(spec, logits, labels.float())), rel=1e-6)
    assert acc == mlp.accuracy_count(logits, labels) / 256
    assert loss != loss_p


def test_load_variables_reads_either_set():
    spec, _, d, before = _train_and_save(AVG, steps=10, num_ps=1)
    path = ckpt.latest_checkpoint(d)
    for src in (d, path):
        v, e = ckpt.load_variables(src), ckpt.load_variables(src, moving_averages=True)
        for k in before["params"]:
            assert torch.equal(v[k], before["params"][k]) and torch.equal(e[k], before["ema"][k]), k


@pytest.mark.timeout(180)
def test_cli_moving_averages_one_ps_two_workers_checkpoint():
    d = tempfile.mkdtemp()
    common = ["--train_steps", "300", "--learning_rate", "0.05", "--optimizer", "sgd", "--log_every", "100",
              "--moving_average_decay", "0.99"]
    with _harness.Tasks() as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done"])
        ws = [t.spawn("worker", i, common + ["--checkpoint_dir", d]) for i in (1, 0)]
        outs = [t.finish(w, 120) for w in ws]
        outp = t.finish(ps, 60)
    for w, o in zip(ws, outs):
        assert w.returncode == 0, o
    assert ps.returncode == 0, outp
    logged = [l for o in outs for l in o.splitlines() if l.startswith("Train step ")]
    assert logged and all(", loss: " in l for l in logged)      # the stdout contract is unchanged
    state = torch.load(ckpt.latest_checkpoint(d), weights_only=False)
    assert state["optimizer"]["moving_average_decay"] == 0.99
    params, shadows = ckpt.load_variables(d), ckpt.load_variables(d, moving_averages=True)
    assert set(shadows) == set(params)
    for k in params:
        assert torch.isfinite(shadows[k]).all(), k
        assert not torch.equal(shadows[k], params[k]), k
        assert torch.equal(shadows[k], state["ema"][k]), k
