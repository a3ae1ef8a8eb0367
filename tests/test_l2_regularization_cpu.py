"""L2 weight regularization on the worker (TF1's `loss + S * sum(tf.nn.l2_loss(v))` before `compute_gradients`), cpu
backend: the fp32 reference against hand-computed TF1 values, validation of `L2Regularization` and the CLI flags, an
unset or zero scale leaving trajectories bit-identical, lock-step runs checked after every step against an fp32 torch
loop that regularizes (and clips) with the reference, an L2 worker against a ps started without it, and a
multi-process CLI run."""
import _harness
import pytest
import torch

from bench_tools.gpu_e2e import ref_slots, tf1_apply
from dist_mnist_b200 import cli
from dist_mnist_b200.cluster import ClusterSpec
from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.config import EngineConfig, GradClip, L2Regularization, OptimizerConfig
from dist_mnist_b200.parallel.ps import ParameterServer
from dist_mnist_b200.parallel.worker import Worker
from dist_mnist_b200.session import InProcessCluster, free_port
from dist_mnist_b200.utils import data

F32 = torch.float32


def _t(*v):
    return torch.tensor(v, dtype=F32)


# ---------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------
def test_l2_regularize_matches_tf1():
    params = {"w": _t(1.0, -2.0, 3.0).view(1, 3), "b": _t(0.5, 4.0)}
    grads = {"w": _t(0.25, 0.5, -1.0).view(1, 3), "b": _t(1.0, -1.0)}
    # weights only: l2_loss(w) = (1 + 4 + 9) / 2 = 7, S * 7 = 0.7 in fp32; g + S*w
    loss, out = mlp.l2_regularize(params, grads, L2Regularization(0.1))
    s = _t(0.1)[0]
    assert float(loss) == float(s * _t(7.0)[0])
    assert torch.equal(out["w"], grads["w"] + s * params["w"]) and torch.equal(out["b"], grads["b"])
    assert torch.equal(out["w"], _t(0.25 + float(s * 1), 0.5 + float(s * -2), -1.0 + float(s * 3)).view(1, 3))
    # "all" (convolutional.py): the biases too, l2_loss(b) = (0.25 + 16) / 2 = 8.125
    loss, out = mlp.l2_regularize(params, grads, L2Regularization(0.5, "all"))
    assert float(loss) == 0.5 * (7.0 + 8.125)
    assert torch.equal(out["b"], _t(1.25, 1.0)) and torch.equal(out["w"], _t(0.75, -0.5, 0.5).view(1, 3))


def test_l2_product_and_sum_round_separately():
    """fl(g + fl(S * w)), no FMA: S * w = 1 + 2^-22 + 2^-46 rounds to 1 + 2^-22, so g = -(1 + 2^-22) leaves 0, where
    one rounding of the whole expression (an FMA) would keep 2^-46."""
    g, w = _t(-(1.0 + 2.0 ** -22)), _t(1.0 + 2.0 ** -23)
    _, out = mlp.l2_regularize({"w": w.view(1, 1)}, {"w": g.view(1, 1)}, L2Regularization(1.0 + 2.0 ** -23))
    assert float(out["w"]) == 0.0
    assert float(torch.tensor(-(1.0 + 2.0 ** -22) + (1.0 + 2.0 ** -23) ** 2, dtype=torch.float64).to(F32)) == 2.0 ** -46


def test_l2_off_and_loss():
    p = {"w": _t(3.0, 4.0).view(1, 2), "b": _t(2.0)}
    g = {"w": _t(1.0, 1.0).view(1, 2), "b": _t(1.0)}
    for off in (L2Regularization(), L2Regularization(0.0), L2Regularization(0, "all")):
        assert not off.enabled
        loss, out = off.apply(p, g)
        assert loss == 0.0 and out is g
        assert off.loss(p) == 0.0
    assert L2Regularization(2.0).loss(p) == 25.0 and L2Regularization(2.0, "all").loss(p) == 29.0


# ---------------------------------------------------------------------------------------------------------------
# configuration and CLI
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [
    {"scale": -1e-4}, {"scale": float("nan")}, {"scale": float("inf")}, {"scale": float("-inf")}, {"scale": True},
    {"scale": "0.1"}, {"scale": 1e-4, "variables": "biases"}, {"variables": "none"},
])
def test_l2_validation(kw):
    with pytest.raises(ValueError):
        L2Regularization(**kw)


def test_l2_in_optimizer_config():
    assert OptimizerConfig("adam").l2 == L2Regularization()
    o = OptimizerConfig("sgd", 0.1, l2=L2Regularization(5e-4, "all"))
    assert o.l2.scale == 5e-4 and o.as_dict()["l2"] == {"scale": 5e-4, "variables": "all"}
    assert L2Regularization.from_dict(o.as_dict()["l2"]) == o.l2 and L2Regularization.from_dict(None) == L2Regularization()
    assert isinstance(L2Regularization(1).scale, float)
    with pytest.raises(ValueError):
        OptimizerConfig("sgd", 0.1, l2={"scale": 1e-4})


def test_atomic_push_mode_refuses_l2():
    opt = OptimizerConfig("sgd", 0.1, l2=L2Regularization(1e-4))
    with pytest.raises(ValueError, match="L2 regularization needs push_mode='mailbox'"):
        EngineConfig(backend="cuda", push_mode="atomic").validate(opt)
    EngineConfig(backend="cuda", push_mode="mailbox").validate(opt)
    # a zero scale is off
    EngineConfig(backend="cuda", push_mode="atomic").validate(OptimizerConfig("sgd", 0.1, l2=L2Regularization(0.0)))


def _opt(argv):
    return cli.optimizer_config_from_args(cli.build_parser().parse_args(argv))


def test_cli_l2_flags():
    assert _opt([]).l2 == L2Regularization()
    assert _opt(["--l2_regularization", "5e-4"]).l2 == L2Regularization(5e-4)
    assert _opt(["--l2_regularization", "5e-4", "--l2_variables", "all"]).l2 == L2Regularization(5e-4, "all")
    assert _opt(["--l2_regularization", "0"]).l2 == L2Regularization(0.0)
    for argv in (["--l2_variables", "all"], ["--l2_variables", "weights"],           # no --l2_regularization
                 ["--l2_regularization=-1e-4"], ["--l2_regularization", "nan"], ["--l2_regularization", "inf"]):
        with pytest.raises(ValueError):
            _opt(argv)
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["--l2_regularization", "1e-4", "--l2_variables", "biases"])
    args = cli.build_parser().parse_args(["--push_mode", "atomic", "--optimizer", "sgd", "--l2_regularization", "1e-4"])
    with pytest.raises(ValueError, match="L2 regularization"):
        cli.engine_config_from_args(args, "cuda").validate(cli.optimizer_config_from_args(args))


# ---------------------------------------------------------------------------------------------------------------
# lock-step runs
# ---------------------------------------------------------------------------------------------------------------
def _run(opt, steps, nps=1, sharding="round_robin"):
    """(losses, variables after every step) of a 1-worker --lanes 1 --strict_steps cpu run."""
    spec = mlp.book_model(100)
    ds = data.synthetic_mnist(512, seed=2)
    it = data.BatchIterator(ds, seed=0)
    losses, ends = [], []
    with InProcessCluster(spec, opt, EngineConfig(backend="cpu", lanes=1, strict_steps=True, sharding=sharding),
                          batch_size=32, num_ps=nps, params=mlp.init_params(spec, seed=5)) as cl:
        for _ in range(steps):
            losses.append(cl.worker.step(*it.next_batch(32)).loss)
            cl.worker.wait_applied()
            ends.append(cl.worker.read_variables())
    return losses, ends


def test_unset_and_zero_scale_leave_the_trajectory_bit_identical():
    base = _run(OptimizerConfig("momentum", 1e-2), 4)
    for l2 in (L2Regularization(), L2Regularization(0.0), L2Regularization(0.0, "all")):
        losses, ends = _run(OptimizerConfig("momentum", 1e-2, l2=l2), 4)
        assert losses == base[0]
        for a, b in zip(ends, base[1]):
            assert all(torch.equal(a[k], b[k]) for k in a)


def test_l2_changes_the_trajectory():
    base = _run(OptimizerConfig("sgd", 0.5), 3)
    losses, ends = _run(OptimizerConfig("sgd", 0.5, l2=L2Regularization(0.05)), 3)
    assert losses[0] > base[0][0]   # the same first pull: the L2 term is added to the reported loss
    assert not torch.allclose(ends[-1]["hid_w"], base[1][-1]["hid_w"], rtol=1e-4, atol=1e-6)


def _apply(opt, params, m, v, t, grads):
    t += 1
    for k in params:
        g = grads[k]
        if opt.kind == "sgd":
            params[k] = params[k] - opt.lr * g
        elif opt.kind == "adam":
            m[k] = opt.beta1 * m[k] + (1 - opt.beta1) * g
            v[k] = opt.beta2 * v[k] + (1 - opt.beta2) * g * g
            lr_t = opt.lr * (1 - opt.beta2 ** t) ** 0.5 / (1 - opt.beta1 ** t)
            params[k] = params[k] - lr_t * m[k] / (v[k].sqrt() + opt.eps)
        else:
            params[k], m[k], v[k] = tf1_apply(opt, params[k], m[k], v[k], g)
    return t


RATES = {"sgd": 0.5, "adam": 1e-3, "momentum": 1e-2}
CLIPS = {"off": GradClip(), "global_norm": GradClip("global_norm", clip_norm=0.17),
         "norm": GradClip("norm", clip_norm=0.16), "value": GradClip("value", value_min=-0.012, value_max=0.0105)}
SHARDINGS = [(1, "round_robin"), (2, "row_split")]


@pytest.mark.parametrize("shards", SHARDINGS, ids=[f"{n}ps-{s}" for n, s in SHARDINGS])
@pytest.mark.parametrize("kind", list(RATES))
@pytest.mark.parametrize("clip", list(CLIPS))
def test_lockstep_trajectory_with_l2(clip, kind, shards):
    """1 worker, --lanes 1 --strict_steps: the step pulls exactly what read_variables() shows before it, so its loss is
    the fp32 reference's (data loss + L2 term) bit for bit; the parameters after every step match fp32 torch applying
    the reference's regularized (and clipped) gradient (the tolerances of tests/test_grad_clip_cpu.py: the ps applies
    in its own native code)."""
    nps, sharding = shards
    l2 = L2Regularization(0.05, "all" if kind == "momentum" else "weights")
    opt = OptimizerConfig(kind, RATES[kind], clip=CLIPS[clip], l2=l2)
    spec = mlp.book_model(100)
    ds = data.synthetic_mnist(512, seed=2)
    it = data.BatchIterator(ds, seed=0)
    params = mlp.init_params(spec, seed=5)
    rp = {k: v.clone() for k, v in params.items()}
    rm, rv = ref_slots(opt, params)
    t = 0
    with InProcessCluster(spec, opt, EngineConfig(backend="cpu", lanes=1, strict_steps=True, sharding=sharding),
                          batch_size=32, num_ps=nps, params=params) as cl:
        w = cl.worker
        for i in range(8):
            x, y = it.next_batch(32)
            pulled = w.read_variables()
            r = w.step(x, y)
            w.wait_applied()
            loss, grads, _ = mlp.manual_loss_and_grads(spec, pulled, x, y)
            reg, grads = mlp.l2_regularize(pulled, grads, l2)
            assert float(reg) > 0
            assert r.loss == float(loss + reg), i
            # the torch loop regularizes its own parameters (within the tolerance of the ps's)
            _, g_ref, _ = mlp.manual_loss_and_grads(spec, rp, x, y)
            _, g_ref = mlp.l2_regularize(rp, g_ref, l2)
            t = _apply(opt, rp, rm, rv, t, mlp.clip_gradients(g_ref, opt.clip) if opt.clip.enabled else g_ref)
            got = w.read_variables()
            for k in got:
                assert torch.allclose(got[k], rp[k], rtol=1e-4, atol=1e-6), (i, k)


# ---------------------------------------------------------------------------------------------------------------
# ps / worker agreement and the CLI
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["adam", "momentum"])   # momentum: the ps / worker optimizer dicts are compared
def test_l2_worker_connects_to_a_ps_without_l2(kind):
    spec = mlp.book_model(32)
    cfg = EngineConfig(backend="cpu")
    cluster = ClusterSpec((f"127.0.0.1:{free_port()}",), (f"127.0.0.1:{free_port()}",))
    ps = ParameterServer(cluster, 0, spec, OptimizerConfig(kind, 1e-3), cfg)
    try:
        w = Worker(cluster, 0, spec, OptimizerConfig(kind, 1e-3, l2=L2Regularization(5e-4, "all")), cfg)
        try:
            w.connect()
        finally:
            w.close()
    finally:
        ps.close()


@pytest.mark.timeout(900)
def test_cli_l2_one_ps_two_workers():
    common = ["--learning_rate", "0.001", "--log_every", "1000", "--lanes", "1", "--l2_regularization", "5e-4",
              "--l2_variables", "all"]
    with _harness.Tasks() as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done"])
        ws = [t.spawn("worker", i, common) for i in (1, 0)]
        outs = [t.finish(w, 780) for w in ws]
        outp = t.finish(ps, 60)
    for w, o in zip(ws, outs):
        assert w.returncode == 0, o
        assert "done: local_steps=" in o, o
    assert ps.returncode == 0, outp
    assert int(outp.split("global_step=")[1].split()[0]) >= 4000, outp
