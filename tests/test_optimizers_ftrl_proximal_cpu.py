"""Adadelta, FTRL (V1 and V2), ProximalAdagrad and ProximalGradientDescent on the parameter server, cpu backend: the
TF1 `training_ops` formulas pinned by hand-computed one-element values and cross-checked against `torch.optim`, their
defaults, validation and flags, slot initialisation, lock-step runs (parameters and both slot buffers after every step,
also under a learning-rate schedule and with moving averages), the exact zeros of a large l1, the ps / worker and
checkpoint agreement on the optimizer, and a multi-process CLI run."""
import tempfile

import _harness
import pytest
import torch

from bench_tools.gpu_e2e import tf1_apply
from dist_mnist_b200 import cli
from dist_mnist_b200.cluster import ClusterSpec
from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.config import EngineConfig, LrSchedule, OptimizerConfig
from dist_mnist_b200.parallel.ps import ParameterServer
from dist_mnist_b200.parallel.worker import Worker
from dist_mnist_b200.session import InProcessCluster, free_port, train_loop
from dist_mnist_b200.utils import ckpt, data

# every rule and branch: l1 > 0 and == 0, lr_power -0.5 and -0.25, shrinkage on and off
RULES = {
    "adadelta": OptimizerConfig("adadelta", 1.0),
    "adadelta_rho": OptimizerConfig("adadelta", 0.5, rho=0.9, eps=1e-6),
    "ftrl": OptimizerConfig("ftrl", 0.05),
    "ftrl_l1": OptimizerConfig("ftrl", 0.05, l1_regularization_strength=1e-3, l2_regularization_strength=1e-2),
    "ftrl_pow": OptimizerConfig("ftrl", 0.05, learning_rate_power=-0.25, l1_regularization_strength=1e-3),
    "ftrl_v2": OptimizerConfig("ftrl", 0.05, l1_regularization_strength=1e-3, l2_regularization_strength=1e-3,
                               l2_shrinkage_regularization_strength=1e-2),
    "proximal_adagrad": OptimizerConfig("proximal_adagrad", 0.05),
    "proximal_adagrad_l1": OptimizerConfig("proximal_adagrad", 0.05, l1_regularization_strength=1e-3,
                                           l2_regularization_strength=1e-2),
    "proximal_sgd": OptimizerConfig("proximal_sgd", 0.05),
    "proximal_sgd_l1": OptimizerConfig("proximal_sgd", 0.05, l1_regularization_strength=1e-3,
                                       l2_regularization_strength=1e-2),
}


def _one(x):
    return torch.tensor([x], dtype=torch.float64)


# (optimizer, p, m, v, g) -> (p, m, v) after one step, computed by hand from TF 1.15's training_ops formulas
HAND = [
    # Adadelta, rho 0.9, eps 0.01: accum = 0.025; update = sqrt(0.01) / sqrt(0.035) * 0.5 = 0.26726...
    (OptimizerConfig("adadelta", 1.0, rho=0.9, eps=0.01), (1.0, 0.0, 0.0, 0.5),
     (0.7327387580875756, 0.007142857142857144, 0.025)),
    # the same, second step with g = -0.25 from there
    (OptimizerConfig("adadelta", 1.0, rho=0.9, eps=0.01), (0.7327387580875756, 0.007142857142857144, 0.025, -0.25),
     (0.8990209567296836, 0.009193548387096776, 0.02875)),
    # ProximalAdagrad, lr 0.2, l2 0.25: accum = 0.35, a = 0.2 / sqrt(0.35); l1 0.5 / 0 / 3 (|prox| < a l1: zero)
    (OptimizerConfig("proximal_adagrad", 0.2, l1_regularization_strength=0.5, l2_regularization_strength=0.25),
     (1.0, 0.0, 0.1, 0.5), (0.6103539724388765, 0.0, 0.35)),
    (OptimizerConfig("proximal_adagrad", 0.2, l2_regularization_strength=0.25), (1.0, 0.0, 0.1, 0.5),
     (0.7662123834633259, 0.0, 0.35)),
    (OptimizerConfig("proximal_adagrad", 0.2, l1_regularization_strength=3.0, l2_regularization_strength=0.25),
     (1.0, 0.0, 0.1, 0.5), (0.0, 0.0, 0.35)),
    # ProximalGradientDescent, lr 0.2, l2 0.25: prox = p - 0.1; l1 0.5 / 0; a negative prox; a zeroed one
    (OptimizerConfig("proximal_sgd", 0.2, l1_regularization_strength=0.5, l2_regularization_strength=0.25),
     (1.0, 0.0, 0.0, 0.5), (0.7619047619047619, 0.0, 0.0)),
    (OptimizerConfig("proximal_sgd", 0.2, l2_regularization_strength=0.25), (1.0, 0.0, 0.0, 0.5),
     (0.8571428571428571, 0.0, 0.0)),
    (OptimizerConfig("proximal_sgd", 0.2, l1_regularization_strength=0.5, l2_regularization_strength=0.25),
     (-1.0, 0.0, 0.0, 0.5), (-0.9523809523809523, 0.0, 0.0)),
    (OptimizerConfig("proximal_sgd", 0.2, l1_regularization_strength=1.0, l2_regularization_strength=0.25),
     (-0.05, 0.0, 0.0, 0.5), (0.0, 0.0, 0.0)),
    # FTRL, lr 0.2, l2 0.25, accum 0.1 -> 0.35, linear 0 -> 0.5 - (sqrt(0.35) - sqrt(0.1)) / 0.2 = -0.87690...
    (OptimizerConfig("ftrl", 0.2, l1_regularization_strength=0.1, l2_regularization_strength=0.25),
     (1.0, 0.0, 0.1, 0.5), (0.22466515304351517, -0.8769010614656181, 0.35)),
    # |linear| <= l1: the weight becomes exactly 0
    (OptimizerConfig("ftrl", 0.2, l1_regularization_strength=1.0, l2_regularization_strength=0.25),
     (1.0, 0.0, 0.1, 0.5), (0.0, -0.8769010614656181, 0.35)),
    # lr_power -0.25: x^0.25 in place of sqrt
    (OptimizerConfig("ftrl", 0.2, l1_regularization_strength=0.1, l2_regularization_strength=0.25,
                     learning_rate_power=-0.25), (1.0, 0.0, 0.1, 0.5), (0.09988861136609606, -0.5340962106155482, 0.35)),
    # V2, shrinkage 0.5: linear gets g + 2 * 0.5 * p = 1.5 (accum still gets g^2); the threshold in the other direction
    (OptimizerConfig("ftrl", 0.2, l1_regularization_strength=0.1, l2_regularization_strength=0.25,
                     l2_shrinkage_regularization_strength=0.5), (1.0, 0.0, 0.1, 0.5),
     (-0.006679777925878565, 0.12309893853438192, 0.35)),
    (OptimizerConfig("ftrl", 0.2, l1_regularization_strength=1.0, l2_regularization_strength=0.25,
                     l2_shrinkage_regularization_strength=0.5, learning_rate_power=-0.25), (1.0, 0.0, 0.1, 0.5),
     (0.0, 0.46590378938445176, 0.35)),
]


@pytest.mark.parametrize("case", range(len(HAND)))
def test_reference_matches_hand_computed_tf1_values(case):
    opt, (p, m, v, g), want = HAND[case]
    got = tf1_apply(opt, _one(p), _one(m), _one(v), _one(g))
    for x, w in zip(got, want):
        assert float(x) == pytest.approx(w, rel=1e-12, abs=1e-15), (opt.kind, got, want)


@pytest.mark.parametrize("case", ["adadelta", "adadelta_rho", "proximal_adagrad"])
def test_reference_formulas_agree_with_torch_optim(case):
    """Adadelta against torch.optim.Adadelta with matched lr, rho and eps; ProximalAdagrad at l1 = l2 = 0 against
    torch.optim.Adagrad(eps=0, initial_accumulator_value=...)."""
    torch.manual_seed(0)
    p0 = torch.randn(1000, dtype=torch.float64)
    ref = torch.nn.Parameter(p0.clone())
    if case == "adadelta":
        opt = OptimizerConfig("adadelta", 1.0)
        o = torch.optim.Adadelta([ref], lr=1.0, rho=0.95, eps=1e-8)
    elif case == "adadelta_rho":
        opt = OptimizerConfig("adadelta", 0.3, rho=0.8, eps=1e-4)
        o = torch.optim.Adadelta([ref], lr=0.3, rho=0.8, eps=1e-4)
    else:
        opt = OptimizerConfig("proximal_adagrad", 0.05, initial_accumulator_value=0.3)
        o = torch.optim.Adagrad([ref], lr=0.05, eps=0.0, initial_accumulator_value=0.3)
    m0, v0 = opt.slot_init()
    p, m, v = p0.clone(), torch.full_like(p0, m0), torch.full_like(p0, v0)
    for _ in range(6):
        g = torch.randn(1000, dtype=torch.float64)
        p, m, v = tf1_apply(opt, p, m, v, g)
        ref.grad = g.clone()
        o.step()
    assert torch.allclose(p, ref.detach(), rtol=1e-12, atol=1e-12)


def test_defaults_and_validation():
    d = OptimizerConfig("adadelta", 1e-3)
    assert (d.rho, d.eps, d.l1_regularization_strength, d.initial_accumulator_value) == (0.95, 1e-8, None, None)
    f = OptimizerConfig("ftrl", 1e-3)
    assert (f.initial_accumulator_value, f.l1_regularization_strength, f.l2_regularization_strength,
            f.l2_shrinkage_regularization_strength, f.learning_rate_power, f.rho) == (0.1, 0.0, 0.0, 0.0, -0.5, None)
    a = OptimizerConfig("proximal_adagrad", 1e-3)
    assert (a.initial_accumulator_value, a.l1_regularization_strength, a.l2_regularization_strength,
            a.l2_shrinkage_regularization_strength, a.learning_rate_power) == (0.1, 0.0, 0.0, None, None)
    s = OptimizerConfig("proximal_sgd", 1e-3)
    assert (s.initial_accumulator_value, s.l1_regularization_strength, s.l2_regularization_strength) == (None, 0.0, 0.0)
    assert OptimizerConfig("adam").rho is None and OptimizerConfig("adam").learning_rate_power is None
    assert OptimizerConfig("ftrl", 1e-3, initial_accumulator_value=0.0).initial_accumulator_value == 0.0
    assert OptimizerConfig("ftrl", 1e-3, learning_rate_power=0.0).learning_rate_power == 0.0
    for bad in ({"kind": "adam", "rho": 0.9}, {"kind": "adagrad", "l1_regularization_strength": 0.1},
                {"kind": "sgd", "l2_regularization_strength": 0.1}, {"kind": "rmsprop", "learning_rate_power": -0.5},
                {"kind": "adadelta", "l1_regularization_strength": 0.1}, {"kind": "adadelta", "momentum": 0.9},
                {"kind": "adadelta", "initial_accumulator_value": 0.1}, {"kind": "proximal_sgd", "rho": 0.9},
                {"kind": "proximal_sgd", "initial_accumulator_value": 0.1},
                {"kind": "proximal_adagrad", "learning_rate_power": -0.5},
                {"kind": "proximal_adagrad", "l2_shrinkage_regularization_strength": 0.1},
                {"kind": "ftrl", "decay": 0.9}, {"kind": "ftrl", "use_nesterov": True},
                # a positive lr_power, a negative l1 / l2 / shrinkage, a non-positive ProximalAdagrad accumulator
                {"kind": "ftrl", "learning_rate_power": 0.5}, {"kind": "ftrl", "l1_regularization_strength": -1e-3},
                {"kind": "ftrl", "l2_regularization_strength": -1e-3},
                {"kind": "ftrl", "l2_shrinkage_regularization_strength": -1e-3},
                {"kind": "proximal_adagrad", "l1_regularization_strength": -1e-3},
                {"kind": "proximal_sgd", "l2_regularization_strength": -1e-3},
                {"kind": "proximal_adagrad", "initial_accumulator_value": 0.0},
                {"kind": "proximal_adagrad", "initial_accumulator_value": -0.1},
                {"kind": "ftrl", "initial_accumulator_value": -0.1},
                # every hyper-parameter finite, and a positive rate where TF's kernels require one
                {"kind": "ftrl", "l1_regularization_strength": float("inf")},
                {"kind": "adadelta", "rho": float("nan")}, {"kind": "adadelta", "eps": float("inf")},
                {"kind": "ftrl", "learning_rate_power": float("-inf")}, {"kind": "proximal_sgd", "lr": float("inf")},
                {"kind": "ftrl", "lr": 0.0}, {"kind": "proximal_adagrad", "lr": -0.1}):
        with pytest.raises(ValueError):
            OptimizerConfig(**bad)


def _opt(argv):
    return cli.optimizer_config_from_args(cli.build_parser().parse_args(argv))


def test_cli_optimizer_flags():
    assert _opt(["--optimizer", "adadelta"]) == OptimizerConfig("adadelta", 1e-4)   # --learning_rate keeps its default
    d = _opt(["--optimizer", "adadelta", "--rho", "0.9", "--epsilon", "1e-6", "--learning_rate", "1.0"])
    assert (d.rho, d.eps, d.lr) == (0.9, 1e-6, 1.0)
    f = _opt(["--optimizer", "ftrl", "--l1_regularization_strength", "0.01", "--l2_regularization_strength", "0.02",
              "--l2_shrinkage_regularization_strength", "0.03", "--learning_rate_power", "-0.25",
              "--initial_accumulator_value", "0.5", "--adam_math", "ieee"])
    assert (f.l1_regularization_strength, f.l2_regularization_strength, f.l2_shrinkage_regularization_strength,
            f.learning_rate_power, f.initial_accumulator_value, f.math) == (0.01, 0.02, 0.03, -0.25, 0.5, "ieee")
    a = _opt(["--optimizer", "proximal_adagrad", "--l1_regularization_strength", "0.01",
              "--initial_accumulator_value", "0.2"])
    assert (a.l1_regularization_strength, a.l2_regularization_strength, a.initial_accumulator_value) == (0.01, 0.0, 0.2)
    s = _opt(["--optimizer", "proximal_sgd", "--l2_regularization_strength", "0.5"])
    assert (s.l1_regularization_strength, s.l2_regularization_strength) == (0.0, 0.5)
    # the ps-side l2 strength and the worker-side L2 loss term are separate settings; both may be given
    b = _opt(["--optimizer", "ftrl", "--l2_regularization_strength", "0.5", "--l2_regularization", "1e-4"])
    assert b.l2_regularization_strength == 0.5 and b.l2.scale == 1e-4
    for argv in (["--rho", "0.9"], ["--optimizer", "sgd", "--l1_regularization_strength", "0.1"],
                 ["--optimizer", "adagrad", "--l2_regularization_strength", "0.1"],
                 ["--optimizer", "proximal_adagrad", "--learning_rate_power", "-0.5"],
                 ["--optimizer", "proximal_sgd", "--initial_accumulator_value", "0.1"],
                 ["--optimizer", "proximal_sgd", "--epsilon", "1e-6"], ["--optimizer", "ftrl", "--rho", "0.9"],
                 ["--optimizer", "ftrl", "--epsilon", "1e-6"], ["--optimizer", "adadelta", "--momentum", "0.9"],
                 ["--optimizer", "adadelta", "--l2_shrinkage_regularization_strength", "0.1"],
                 ["--optimizer", "ftrl", "--learning_rate_power", "0.5"],
                 ["--optimizer", "ftrl", "--l1_regularization_strength", "-0.1"],
                 ["--optimizer", "proximal_adagrad", "--initial_accumulator_value", "0"]):
        with pytest.raises(ValueError):
            _opt(argv)


@pytest.mark.parametrize("kind", ["adadelta", "ftrl", "proximal_adagrad", "proximal_sgd"])
def test_atomic_push_mode_stays_sgd_only(kind):
    with pytest.raises(ValueError):
        EngineConfig(backend="cuda", push_mode="atomic").validate(OptimizerConfig(kind, 1e-2))


@pytest.mark.parametrize("kind,m0,v0", [("adadelta", 0.0, 0.0), ("ftrl", 0.0, 0.25), ("proximal_adagrad", 0.0, 0.25),
                                        ("proximal_sgd", 0.0, 0.0)])
def test_slot_initialisation(kind, m0, v0):
    kw = {"initial_accumulator_value": 0.25} if kind in ("ftrl", "proximal_adagrad") else {}
    opt = OptimizerConfig(kind, 1e-2, **kw)
    assert opt.slot_init() == (m0, v0)
    with InProcessCluster(mlp.book_model(32), opt, EngineConfig(backend="cpu"), batch_size=16, num_ps=2) as cl:
        for region, want in (("adam_m", m0), ("adam_v", v0)):
            for k, t in cl.worker.read_variables(region).items():
                assert torch.equal(t, torch.full_like(t, want)), (region, k)


@pytest.mark.parametrize("apply_mode", ["per_push", "merged"])
@pytest.mark.parametrize("nps", [1, 2])
@pytest.mark.parametrize("rule", list(RULES))
def test_lockstep_trajectory_matches_tf1_formulas(rule, nps, apply_mode):
    _harness.cpu_optimizer_lockstep(RULES[rule], nps, apply_mode)


@pytest.mark.parametrize("rule,apply_mode", [("ftrl_pow", "per_push"), ("proximal_adagrad_l1", "merged"),
                                             ("adadelta", "per_push")])
def test_lockstep_under_a_learning_rate_schedule(rule, apply_mode):
    import dataclasses

    opt = dataclasses.replace(RULES[rule], schedule=LrSchedule("exponential_decay", decay_steps=2, decay_rate=0.5))
    assert len({opt.lr_at(i) for i in range(8)}) == 8
    _harness.cpu_optimizer_lockstep(opt, 2, apply_mode)


@pytest.mark.parametrize("rule", ["ftrl_v2", "proximal_sgd_l1", "adadelta_rho"])
def test_lockstep_with_moving_averages(rule):
    import dataclasses

    _harness.cpu_optimizer_lockstep(dataclasses.replace(RULES[rule], moving_average_decay=0.9), 1, "per_push", ema=True)


@pytest.mark.parametrize("kind", ["proximal_adagrad", "ftrl"])
def test_large_l1_leaves_the_same_exact_zeros_as_the_reference(kind):
    """A large l1 sets most of hid_w to exact zeros (the proximal step's soft threshold; FTRL's |linear| <= l1), and they
    sit where the reference's are, element for element."""
    opt = OptimizerConfig(kind, 0.05, l1_regularization_strength=0.05 if kind == "ftrl" else 0.5)
    got, ref = _harness.cpu_optimizer_lockstep(opt, 2, "per_push", steps=6)
    zg, zr = got["hid_w"] == 0, ref["hid_w"] == 0
    assert zr.float().mean() > 0.5, float(zr.float().mean())
    assert torch.equal(zg, zr), int((zg != zr).sum())


@pytest.mark.parametrize("ps_kind,w_kind", [("ftrl", "adam"), ("adam", "proximal_sgd"), ("adadelta", "rmsprop"),
                                            ("proximal_adagrad", "ftrl")])
def test_worker_refuses_a_ps_with_another_optimizer(ps_kind, w_kind):
    spec = mlp.book_model(32)
    cfg = EngineConfig(backend="cpu")
    cluster = ClusterSpec((f"127.0.0.1:{free_port()}",), (f"127.0.0.1:{free_port()}",))
    ps = ParameterServer(cluster, 0, spec, OptimizerConfig(ps_kind, 1e-3), cfg)
    try:
        w = Worker(cluster, 0, spec, OptimizerConfig(w_kind, 1e-3), cfg)
        with pytest.raises(RuntimeError, match="different engine configuration"):
            w.connect()
        if ps_kind != "adam":     # same kind, another hyper-parameter
            kw = {"rho": 0.9} if ps_kind == "adadelta" else {"l1_regularization_strength": 0.1}
            w = Worker(cluster, 0, spec, OptimizerConfig(ps_kind, 1e-3, **kw), cfg)
            with pytest.raises(RuntimeError, match="different engine configuration"):
                w.connect()
    finally:
        ps.close()


@pytest.mark.parametrize("kind", ["ftrl", "adadelta"])
def test_checkpoint_roundtrip_keeps_slots_bit_identical(kind):
    spec = mlp.book_model(64)
    opt = (OptimizerConfig("ftrl", 0.05, l1_regularization_strength=1e-3, learning_rate_power=-0.25)
           if kind == "ftrl" else OptimizerConfig("adadelta", 1.0, rho=0.9))
    cfg = EngineConfig(backend="cpu")
    ds = data.synthetic_mnist(512, seed=0)
    d = tempfile.mkdtemp()
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=2) as cl:
        train_loop(cl.worker, ds, train_steps=30, log_every=0, checkpoint_dir=d, chunk=10)
        before = {r: cl.worker.read_variables(r) for r in ("params", "adam_m", "adam_v")}
    state = torch.load(ckpt.latest_checkpoint(d), weights_only=False)
    saved = state["optimizer"]
    assert saved["kind"] == kind
    if kind == "ftrl":
        assert (saved["l1_regularization_strength"], saved["learning_rate_power"]) == (1e-3, -0.25)
    else:
        assert saved["rho"] == 0.9
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=2, restore_dir=d) as cl:
        assert cl.worker.read_global_step() == 30
        for r, vals in before.items():
            got = cl.worker.read_variables(r)
            for k in vals:
                assert torch.equal(got[k], vals[k]), (r, k)
        res = train_loop(cl.worker, ds, train_steps=40, log_every=0, chunk=10)
        assert res.steps_run == 10


def test_checkpoints_of_other_kinds_are_refused_and_older_ones_restore():
    spec = mlp.book_model(32)
    cfg = EngineConfig(backend="cpu")
    ds = data.synthetic_mnist(256, seed=0)
    d = tempfile.mkdtemp()
    with InProcessCluster(spec, OptimizerConfig("adagrad", 5e-2), cfg, batch_size=16) as cl:
        train_loop(cl.worker, ds, train_steps=10, log_every=0, checkpoint_dir=d, chunk=10)
    for kind in ("ftrl", "proximal_adagrad", "proximal_sgd", "adadelta"):
        with InProcessCluster(spec, OptimizerConfig(kind, 1e-2), cfg, batch_size=16) as cl:
            with pytest.raises(RuntimeError, match="optimizer slots"):
                ckpt.restore_latest(cl.worker, d)
    # a checkpoint written before these optimizers existed has none of their keys in its `optimizer` entry
    path = ckpt.latest_checkpoint(d)
    state = torch.load(path, weights_only=False)
    for key in ("rho", "l1_regularization_strength", "l2_regularization_strength",
                "l2_shrinkage_regularization_strength", "learning_rate_power"):
        del state["optimizer"][key]
    torch.save(state, path)
    with InProcessCluster(spec, OptimizerConfig("adagrad", 5e-2), cfg, batch_size=16) as cl:
        assert ckpt.restore_latest(cl.worker, d) == 10
    d2 = tempfile.mkdtemp()
    with InProcessCluster(spec, OptimizerConfig("proximal_sgd", 1e-2), cfg, batch_size=16) as cl:
        train_loop(cl.worker, ds, train_steps=10, log_every=0, checkpoint_dir=d2, chunk=10)
    with InProcessCluster(spec, OptimizerConfig("sgd", 1e-2), cfg, batch_size=16) as cl:
        with pytest.raises(RuntimeError, match="optimizer slots"):
            ckpt.restore_latest(cl.worker, d2)


@pytest.mark.timeout(180)
def test_cli_ftrl_one_ps_two_worker_processes():
    common = ["--train_steps", "400", "--learning_rate", "0.5", "--optimizer", "ftrl"]
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
