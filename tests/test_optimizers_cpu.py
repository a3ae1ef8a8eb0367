"""Momentum (with and without Nesterov), Adagrad and RMSProp on the parameter server, cpu backend: the TF1
`training_ops` formulas step by step (parameters and both slot buffers), their defaults and flags, slot
initialisation, the ps / worker and checkpoint agreement on the optimizer, and a multi-process CLI run."""
import tempfile

import _harness
import pytest
import torch

from bench_tools.gpu_e2e import ref_slots, ref_step, tf1_apply
from dist_mnist_b200 import cli
from dist_mnist_b200.cluster import ClusterSpec
from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
from dist_mnist_b200.parallel.ps import ParameterServer
from dist_mnist_b200.parallel.worker import Worker
from dist_mnist_b200.session import InProcessCluster, free_port, train_loop
from dist_mnist_b200.utils import ckpt, data


RULES = {
    "momentum": OptimizerConfig("momentum", 1e-2),
    "nesterov": OptimizerConfig("momentum", 1e-2, use_nesterov=True),
    "adagrad": OptimizerConfig("adagrad", 5e-2),
    "rmsprop": OptimizerConfig("rmsprop", 1e-3),
    "rmsprop_mom": OptimizerConfig("rmsprop", 1e-3, momentum=0.9),
}


@pytest.mark.parametrize("apply_mode", ["per_push", "merged"])
@pytest.mark.parametrize("nps", [1, 2])
@pytest.mark.parametrize("rule", list(RULES))
def test_lockstep_trajectory_matches_tf1_formulas(rule, nps, apply_mode):
    """Tolerances of tests/test_cpu_engine.py::test_lockstep_trajectory_matches_reference_math."""
    opt = RULES[rule]
    spec = mlp.book_model(100)
    cfg = EngineConfig(backend="cpu", apply_mode=apply_mode)
    ds = data.synthetic_mnist(512, seed=2)
    it = data.BatchIterator(ds, seed=0)
    params = mlp.init_params(spec, seed=5)
    rp = {k: v.clone() for k, v in params.items()}
    rm, rv = ref_slots(opt, params)
    t = 0
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=nps, params=params) as cl:
        w = cl.worker
        for i in range(8):
            x, y = it.next_batch(32)
            r = w.step(x, y)
            w.wait_applied()
            lref, t = ref_step(spec, rp, rm, rv, t, x, y, opt)
            assert r.loss == pytest.approx(lref, rel=1e-4)
            assert r.seq == i + 1
            got, gm, gv = w.read_variables(), w.read_variables("adam_m"), w.read_variables("adam_v")
            for k in got:
                assert torch.allclose(got[k], rp[k], rtol=1e-4, atol=1e-6), (i, k)
                assert torch.allclose(gm[k], rm[k], rtol=1e-4, atol=1e-7), (i, k)
                assert torch.allclose(gv[k], rv[k], rtol=1e-4, atol=1e-7), (i, k)
        assert w.read_global_step() == 8


@pytest.mark.parametrize("case", ["momentum", "nesterov", "adagrad"])
def test_reference_formulas_agree_with_torch_optim(case):
    """Where TF1 and torch.optim coincide: SGD momentum with dampening 0 (plain and Nesterov), and Adagrad with
    eps=0 and initial_accumulator_value=0.1."""
    torch.manual_seed(0)
    p0 = torch.randn(1000, dtype=torch.float64)
    opt = {"momentum": OptimizerConfig("momentum", 0.05), "nesterov": OptimizerConfig("momentum", 0.05, use_nesterov=True),
           "adagrad": OptimizerConfig("adagrad", 0.05)}[case]
    ref = torch.nn.Parameter(p0.clone())
    if case == "adagrad":
        o = torch.optim.Adagrad([ref], lr=0.05, eps=0.0, initial_accumulator_value=0.1)
    else:
        o = torch.optim.SGD([ref], lr=0.05, momentum=0.9, dampening=0, nesterov=case == "nesterov")
    m0, v0 = opt.slot_init()
    p, m, v = p0.clone(), torch.full_like(p0, m0), torch.full_like(p0, v0)
    for _ in range(6):
        g = torch.randn(1000, dtype=torch.float64)
        p, m, v = tf1_apply(opt, p, m, v, g)
        ref.grad = g.clone()
        o.step()
    assert torch.allclose(p, ref.detach(), rtol=1e-12, atol=1e-12)


def test_defaults_per_kind():
    assert OptimizerConfig("adam", 1e-4) == OptimizerConfig("adam", 1e-4, 0.9, 0.999, 1e-8, "fast")
    assert OptimizerConfig("sgd", 1e-2).eps == 1e-8
    m = OptimizerConfig("momentum", 1e-2)
    assert (m.momentum, m.use_nesterov, m.decay, m.initial_accumulator_value) == (0.9, False, None, None)
    a = OptimizerConfig("adagrad", 1e-2)
    assert (a.initial_accumulator_value, a.momentum, a.decay) == (0.1, None, None)
    r = OptimizerConfig("rmsprop", 1e-2)
    assert (r.decay, r.momentum, r.eps) == (0.9, 0.0, 1e-10)
    assert OptimizerConfig("adam").slot_init() == OptimizerConfig("momentum").slot_init() == (0.0, 0.0)
    assert a.slot_init() == (0.0, 0.1) and r.slot_init() == (0.0, 1.0)
    for bad in ({"kind": "adam", "momentum": 0.9}, {"kind": "sgd", "use_nesterov": True},
                {"kind": "momentum", "decay": 0.9}, {"kind": "rmsprop", "initial_accumulator_value": 0.1},
                {"kind": "adagrad", "initial_accumulator_value": 0.0}):
        with pytest.raises(ValueError):
            OptimizerConfig(**bad)


def _opt(argv):
    return cli.optimizer_config_from_args(cli.build_parser().parse_args(argv))


def test_cli_optimizer_flags():
    assert _opt([]) == OptimizerConfig("adam", 1e-4, math="fast")
    assert _opt(["--optimizer", "adam"]) == OptimizerConfig("adam", 1e-4)
    assert _opt(["--optimizer", "adam", "--epsilon", "1e-7"]).eps == 1e-7
    assert _opt(["--optimizer", "sgd", "--learning_rate", "0.05"]) == OptimizerConfig("sgd", 0.05)
    assert _opt(["--optimizer", "momentum"]) == OptimizerConfig("momentum", 1e-4, momentum=0.9)
    o = _opt(["--optimizer", "momentum", "--use_nesterov", "--momentum", "0.5"])
    assert o.use_nesterov and o.momentum == 0.5
    assert _opt(["--optimizer", "adagrad", "--initial_accumulator_value", "0.3"]).initial_accumulator_value == 0.3
    r = _opt(["--optimizer", "rmsprop", "--rmsprop_decay", "0.95", "--momentum", "0.9", "--epsilon", "1e-6",
              "--adam_math", "ieee"])
    assert (r.decay, r.momentum, r.eps, r.math) == (0.95, 0.9, 1e-6, "ieee")
    assert _opt(["--optimizer", "rmsprop"]).eps == 1e-10
    for argv in (["--momentum", "0.9"], ["--optimizer", "sgd", "--epsilon", "1e-6"], ["--use_nesterov"],
                 ["--optimizer", "rmsprop", "--use_nesterov"], ["--optimizer", "adagrad", "--epsilon", "1e-6"],
                 ["--optimizer", "momentum", "--rmsprop_decay", "0.9"],
                 ["--optimizer", "rmsprop", "--initial_accumulator_value", "0.1"]):
        with pytest.raises(ValueError):
            _opt(argv)


@pytest.mark.parametrize("kind", ["momentum", "adagrad", "rmsprop", "adam"])
def test_atomic_push_mode_stays_sgd_only(kind):
    with pytest.raises(ValueError):
        EngineConfig(backend="cuda", push_mode="atomic").validate(OptimizerConfig(kind))


@pytest.mark.parametrize("kind,m0,v0", [("adam", 0.0, 0.0), ("sgd", 0.0, 0.0), ("momentum", 0.0, 0.0),
                                        ("adagrad", 0.0, 0.25), ("rmsprop", 0.0, 1.0)])
def test_slot_initialisation(kind, m0, v0):
    opt = OptimizerConfig(kind, 1e-2, **({"initial_accumulator_value": 0.25} if kind == "adagrad" else {}))
    with InProcessCluster(mlp.book_model(32), opt, EngineConfig(backend="cpu"), batch_size=16, num_ps=2) as cl:
        for region, want in (("adam_m", m0), ("adam_v", v0)):
            for k, t in cl.worker.read_variables(region).items():
                assert torch.equal(t, torch.full_like(t, want)), (region, k)


@pytest.mark.parametrize("ps_kind,w_kind", [("rmsprop", "adam"), ("adam", "momentum"), ("adagrad", "rmsprop")])
def test_worker_refuses_a_ps_with_another_optimizer(ps_kind, w_kind):
    spec = mlp.book_model(32)
    cfg = EngineConfig(backend="cpu")
    cluster = ClusterSpec((f"127.0.0.1:{free_port()}",), (f"127.0.0.1:{free_port()}",))
    ps = ParameterServer(cluster, 0, spec, OptimizerConfig(ps_kind, 1e-3), cfg)
    try:
        w = Worker(cluster, 0, spec, OptimizerConfig(w_kind, 1e-3), cfg)
        with pytest.raises(RuntimeError, match="different engine configuration"):
            w.connect()
        if ps_kind != "adam":     # same kind, another learning rate
            w = Worker(cluster, 0, spec, OptimizerConfig(ps_kind, 2e-3), cfg)
            with pytest.raises(RuntimeError, match="different engine configuration"):
                w.connect()
    finally:
        ps.close()


@pytest.mark.parametrize("kind", ["momentum", "rmsprop"])
def test_checkpoint_roundtrip_keeps_slots_bit_identical(kind):
    spec = mlp.book_model(64)
    opt = OptimizerConfig(kind, 1e-2 if kind == "momentum" else 1e-3, momentum=0.9)
    cfg = EngineConfig(backend="cpu")
    ds = data.synthetic_mnist(512, seed=0)
    d = tempfile.mkdtemp()
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=2) as cl:
        train_loop(cl.worker, ds, train_steps=30, log_every=0, checkpoint_dir=d, chunk=10)
        before = {r: cl.worker.read_variables(r) for r in ("params", "adam_m", "adam_v")}
    state = torch.load(ckpt.latest_checkpoint(d), weights_only=False)
    assert state["optimizer"]["kind"] == kind and state["optimizer"]["momentum"] == 0.9
    assert set(state) >= {"adam_m", "adam_v"} and state["format_version"] == ckpt.FORMAT_VERSION
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=2, restore_dir=d) as cl:
        assert cl.worker.read_global_step() == 30
        for r, vals in before.items():
            got = cl.worker.read_variables(r)
            for k in vals:
                assert torch.equal(got[k], vals[k]), (r, k)
        res = train_loop(cl.worker, ds, train_steps=40, log_every=0, chunk=10)
        assert res.steps_run == 10


def test_adam_checkpoint_is_refused_by_an_rmsprop_run():
    spec = mlp.book_model(32)
    cfg = EngineConfig(backend="cpu")
    ds = data.synthetic_mnist(256, seed=0)
    d = tempfile.mkdtemp()
    with InProcessCluster(spec, OptimizerConfig("adam", 1e-3), cfg, batch_size=16) as cl:
        train_loop(cl.worker, ds, train_steps=10, log_every=0, checkpoint_dir=d, chunk=10)
    with InProcessCluster(spec, OptimizerConfig("rmsprop", 1e-3), cfg, batch_size=16) as cl:
        with pytest.raises(RuntimeError, match="optimizer slots"):
            ckpt.restore_latest(cl.worker, d)
    with InProcessCluster(spec, OptimizerConfig("sgd", 1e-2), cfg, batch_size=16) as cl:
        assert ckpt.restore_latest(cl.worker, d) == 10      # Adam <-> SGD restores as before


@pytest.mark.timeout(180)
def test_cli_rmsprop_one_ps_two_worker_processes():
    common = ["--train_steps", "400", "--learning_rate", "0.001", "--optimizer", "rmsprop"]
    with _harness.Tasks() as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done"])
        ws = [t.spawn("worker", i, common) for i in (1, 0)]
        outs = [t.finish(w, 120) for w in ws]
        outp = t.finish(ps, 60)
    for w, o in zip(ws, outs):
        assert w.returncode == 0, o
        assert o.splitlines()[:2] == ["job name : worker", f"task index : {1 if w is ws[0] else 0}"]
    assert ps.returncode == 0, outp
    logged = [l for o in outs for l in o.splitlines() if l.startswith("Train step ")]
    assert logged and all(int(l.split(",")[0].split()[-1]) % 100 == 0 and ", loss: " in l for l in logged)
    last = [int(l.split("last_global_step=")[1].split()[0]) for o in outs for l in o.splitlines()
            if "last_global_step=" in l]
    assert len(last) == 2 and min(last) >= 400            # both stop at the shared global step
    gstep = int(outp.split("exiting: global_step=")[1].split()[0])
    total = sum(int(l.split("local_steps=")[1].split()[0]) for o in outs for l in o.splitlines() if "local_steps=" in l)
    assert gstep == total                                 # every push applied exactly once
    losses = [float(l.split("loss: ")[1]) for l in logged]
    assert min(losses) < 0.05                             # trained (an untrained batch loss is ~0.23)
