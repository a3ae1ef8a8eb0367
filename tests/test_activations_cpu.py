"""Hidden-layer activations (`--activation`, TF 1.15's tf.nn functors and registered gradients), cpu backend: f and f'
against hand-computed TF1 values at the kinks, at +-0 and at saturation; the hand-derived backward against autograd
in fp64; flag and config validation; the fp64 push checker's bound and its activation mutants; lock-step cpu runs;
and a multi-process CLI run."""
import math

import _harness
import pytest
import torch

from bench_tools import fused_push_ref as R
from bench_tools.gpu_e2e import ref_slots, tf1_apply
from dist_mnist_b200 import cli
from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
from dist_mnist_b200.session import InProcessCluster
from dist_mnist_b200.utils import data

F32 = torch.float32
S, SA = mlp.SELU_SCALE, mlp.SELU_SCALE_ALPHA


def _f32(v):
    return float(torch.tensor(v, dtype=F32))


# ---------------------------------------------------------------------------------------------------------------
# f and f'
# ---------------------------------------------------------------------------------------------------------------
# (activation, x, TF1's f(x) in fp32)
FORWARD = [
    ("relu", -1.0, 0.0), ("relu", 0.0, 0.0), ("relu", -0.0, 0.0), ("relu", 2.5, 2.5),
    ("relu6", -1.0, 0.0), ("relu6", 0.0, 0.0), ("relu6", 3.0, 3.0), ("relu6", 6.0, 6.0), ("relu6", 7.5, 6.0),
    ("leaky_relu", -1.0, _f32(-0.2)), ("leaky_relu", 0.0, 0.0), ("leaky_relu", -0.0, 0.0), ("leaky_relu", 2.0, 2.0),
    ("elu", -1.0, math.exp(-1.0) - 1.0), ("elu", 0.0, 0.0), ("elu", -0.0, 0.0), ("elu", 1.5, 1.5),
    ("elu", -20.0, -1.0), ("elu", -30.0, -1.0),
    ("selu", -1.0, SA * (math.exp(-1.0) - 1.0)), ("selu", 0.0, 0.0), ("selu", 2.0, S * 2.0), ("selu", -25.0, -SA),
    ("sigmoid", 0.0, 0.5), ("sigmoid", -0.0, 0.5), ("sigmoid", 20.0, 1.0), ("sigmoid", -20.0, 1.0 / (1.0 + math.exp(20.0))),
    ("sigmoid", 2.0, 1.0 / (1.0 + math.exp(-2.0))),
    ("tanh", 0.0, 0.0), ("tanh", -0.0, 0.0), ("tanh", 20.0, 1.0), ("tanh", -20.0, -1.0), ("tanh", 0.5, math.tanh(0.5)),
]

# (activation, y, dy, TF1's dx): the registered gradients take the layer's output y
BACKWARD = [
    ("relu", 0.0, 3.0, 0.0), ("relu", 2.5, 3.0, 3.0),
    ("relu6", 0.0, 3.0, 0.0), ("relu6", 6.0, 3.0, 0.0), ("relu6", 3.0, 3.0, 3.0),
    ("leaky_relu", _f32(-0.2), 3.0, _f32(0.2) * 3.0), ("leaky_relu", 0.0, 3.0, _f32(0.2) * 3.0), ("leaky_relu", 2.0, 3.0, 3.0),
    ("elu", -1.0, 3.0, 0.0), ("elu", -0.5, 3.0, 1.5), ("elu", 0.0, 3.0, 3.0), ("elu", 1.5, 3.0, 3.0),
    ("selu", -SA, 3.0, 0.0), ("selu", -1.0, 2.0, 2.0 * (SA - 1.0)), ("selu", 0.0, 3.0, 3.0 * S), ("selu", 2.0, 3.0, 3.0 * S),
    ("sigmoid", 0.5, 3.0, 0.75), ("sigmoid", 1.0, 3.0, 0.0), ("sigmoid", 0.0, 3.0, 0.0),
    ("tanh", 0.0, 3.0, 3.0), ("tanh", 1.0, 3.0, 0.0), ("tanh", -1.0, 3.0, 0.0), ("tanh", 0.5, 2.0, 1.5),
]


@pytest.mark.parametrize("name,x,want", FORWARD)
def test_forward_matches_tf1(name, x, want):
    got = float(mlp.activate(name, torch.tensor([x], dtype=F32))[0])
    assert got == pytest.approx(_f32(want), rel=2 ** -22, abs=0.0), (name, x, got, want)


@pytest.mark.parametrize("name,y,dy,want", BACKWARD)
def test_gradient_from_the_output_matches_tf1(name, y, dy, want):
    got = float(mlp.activation_grad(name, torch.tensor([y], dtype=F32), torch.tensor([dy], dtype=F32))[0])
    assert got == pytest.approx(_f32(want), rel=2 ** -22, abs=0.0), (name, y, got, want)


def test_saturated_units_keep_finite_gradients():
    x = torch.tensor([-200.0, -20.0, 20.0, 200.0], dtype=F32)
    for name in mlp.ACTIVATIONS:
        y = mlp.activate(name, x)
        g = mlp.activation_grad(name, y, torch.ones_like(y))
        assert bool(torch.isfinite(y).all() and torch.isfinite(g).all()), name
    assert mlp.activate("sigmoid", x).tolist()[2:] == [1.0, 1.0]
    assert mlp.activate("elu", x).tolist()[:2] == [-1.0, -1.0]


# ---------------------------------------------------------------------------------------------------------------
# the hand-derived backward against autograd
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hidden", [(7,), (7, 5)], ids=["1-hidden", "2-hidden"])
@pytest.mark.parametrize("loss", ["book", "xent"])
@pytest.mark.parametrize("name", mlp.ACTIVATIONS)
def test_manual_gradients_match_autograd_in_fp64(name, loss, hidden):
    spec = mlp.MLPSpec(name="t", in_features=20, hidden=hidden, num_classes=4, loss=loss, init="glorot",
                       activation=name)
    g = torch.Generator().manual_seed(3)
    params = {k: v.double() for k, v in mlp.init_params(spec, seed=4).items()}
    for k in params:   # biases away from zero, weights wide enough that pre-activations cross every kink
        params[k] = params[k] * 4 + (0.5 * torch.randn(params[k].shape, generator=g, dtype=torch.float64)
                                     if params[k].dim() == 1 else 0)
    x = 3 * torch.randn(16, 20, generator=g, dtype=torch.float64)
    y = torch.nn.functional.one_hot(torch.randint(0, 4, (16,), generator=g), 4).double()
    pre = x @ params[spec.variable_names()[0][0]].t() + params[spec.variable_names()[0][1]]
    assert bool((pre < 0).any() and (pre > 0).any())
    if name == "relu6":
        assert bool((pre > 6).any())
    l_m, g_m, _ = mlp.manual_loss_and_grads(spec, params, x, y)
    l_a, g_a, _ = mlp.loss_and_grads(spec, params, x, y)
    assert float(l_m) == pytest.approx(float(l_a), rel=1e-12)
    for k in g_a:
        assert torch.allclose(g_m[k], g_a[k], rtol=1e-10, atol=1e-13), (k, float((g_m[k] - g_a[k]).abs().max()))


# ---------------------------------------------------------------------------------------------------------------
# flag and config
# ---------------------------------------------------------------------------------------------------------------
def test_flag_default_choices_and_validation():
    p = cli.build_parser()
    assert p.parse_args([]).activation == "relu"
    for name in mlp.ACTIVATIONS:
        assert p.parse_args(["--activation", name]).activation == name
    for bad in ("swish", "softplus", "RELU", ""):
        with pytest.raises(SystemExit):
            p.parse_args(["--activation", bad])
    with pytest.raises(ValueError, match="unknown activation"):
        mlp.MLPSpec(activation="crelu")
    with pytest.raises(ValueError, match="unknown activation"):
        mlp.get_model("book", 100, "softsign")


def test_models_take_the_activation():
    assert mlp.get_model("book", 100) == mlp.get_model("book", 100, "relu") == mlp.book_model(100)
    for model in ("book", "zhihu", "wide"):
        spec = mlp.get_model(model, 64, "tanh")
        assert spec.activation == "tanh"
        assert spec.variables() == mlp.get_model(model, 64).variables()   # the same variables, as TF stores them
    assert [mlp.activation_code(a) for a in mlp.ACTIVATIONS] == list(range(1, 8))


def _run(spec, opt, steps, nps=1, sharding="round_robin"):
    """(losses, variables after every step) of a 1-worker --lanes 1 --strict_steps cpu run."""
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


def test_explicit_relu_is_bit_identical_and_other_activations_differ():
    opt = OptimizerConfig("momentum", 1e-2)
    base = _run(mlp.book_model(100), opt, 4)
    explicit = _run(mlp.MLPSpec(name="book", hidden=(100,), loss="book", init="book", activation="relu"), opt, 4)
    assert explicit[0] == base[0]
    for a, b in zip(explicit[1], base[1]):
        assert all(torch.equal(a[k], b[k]) for k in a)
    other = _run(mlp.get_model("book", 100, "tanh"), opt, 4)
    assert other[0][0] != base[0][0]


# ---------------------------------------------------------------------------------------------------------------
# the fp64 push checker under every activation
# ---------------------------------------------------------------------------------------------------------------
SUBSET = [(100, 10, 784, b, "book") for b in (1, 31, 32, 33, 63, 64, 100, 255, 256)]
SUBSET += [(1, 2, 228, 32, "book"), (17, 3, 260, 33, "xent"), (128, 11, 1024, 256, "xent"), (1, 11, 784, 33, "xent")]


@pytest.mark.parametrize("shape", SUBSET, ids=[f"H{h}-C{c}-I{i}-B{b}-{l}" for h, c, i, b, l in SUBSET])
@pytest.mark.parametrize("name", mlp.ACTIVATIONS[1:])
def test_emulated_kernel_is_inside_the_bound_and_activation_mutants_are_not(name, shape):
    case = R.case_for(shape, activation=name)
    x, y = case.batches[0]
    assert R.check_case(case, x, y) == [] and R.exact_inputs(case) == []
    ref = R.reference(case.spec, case.params, x, y)
    for mode in ("trunc", "rne"):
        v = R.compare(R.emulate(case.spec, case.params, x, y, mode), ref)
        print(f"[{case.name} seed {case.seed}] emulated, tf32 {mode}: {v.line()}")
        assert v.ok and v.max < 0.6, (mode, v.worst, v.where)
    muts = R.mutant_instances(case, ref)
    assert "relu_missing" not in {m for m, _ in muts}
    for mode in ("trunc", "rne"):
        for mut, arg in muts:
            v = R.compare(R.emulate(case.spec, case.params, x, y, mode, mut, arg), ref)
            assert v.max > (20.0 if mut in R.ACT_MUTANTS else 4.0), (mode, mut, arg, v.worst)


def test_every_activation_mutant_is_admitted_somewhere():
    want = {"relu6": {"act_forward_missing", "act_grad_missing", "relu6_upper_kink_missing"},
            "leaky_relu": {"act_forward_missing", "act_grad_missing"}}
    for name in mlp.ACTIVATIONS[1:]:
        seen = set()
        for shape in ((100, 10, 784, 32, "book"), (128, 11, 1024, 256, "xent")):
            case = R.case_for(shape, activation=name)
            seen |= {m for m, _ in R.mutant_instances(case, R.reference(case.spec, case.params, *case.batches[0]))}
        # leaky_relu's and relu6's f' is piecewise constant with the sign of y: f' of pre is f' of y
        assert want.get(name, {"act_forward_missing", "act_grad_missing", "act_grad_from_pre"}) <= seen, (name, seen)


def test_relu_cases_are_unchanged_by_the_activation_argument():
    for shape in ((100, 10, 784, 33, "book"), (17, 3, 260, 33, "xent")):
        a, b = R.case_for(shape), R.case_for(shape, activation="relu")
        assert a.seed == b.seed and a.name == b.name
        assert all(torch.equal(a.params[k], b.params[k]) for k in a.params)


# ---------------------------------------------------------------------------------------------------------------
# lock-step runs
# ---------------------------------------------------------------------------------------------------------------
RATES = {"adam": 1e-3, "momentum": 1e-2}
SHARDINGS = [(1, "round_robin"), (2, "row_split")]


@pytest.mark.parametrize("shards", SHARDINGS, ids=[f"{n}ps-{s}" for n, s in SHARDINGS])
@pytest.mark.parametrize("kind", list(RATES))
@pytest.mark.parametrize("name", ["tanh", "selu"])
def test_lockstep_trajectory(name, kind, shards):
    """1 worker, --lanes 1 --strict_steps: the step pulls exactly what read_variables() shows before it, so its loss is
    the fp32 reference's bit for bit; the parameters after every step match fp32 torch applying the reference's
    gradient."""
    nps, sharding = shards
    opt = OptimizerConfig(kind, RATES[kind])
    spec = mlp.get_model("book", 100, name)
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
            loss, _, _ = mlp.manual_loss_and_grads(spec, pulled, x, y)
            assert r.loss == float(loss), i
            _, g_ref, _ = mlp.manual_loss_and_grads(spec, rp, x, y)
            t += 1
            for k in rp:
                if kind == "adam":
                    rm[k] = opt.beta1 * rm[k] + (1 - opt.beta1) * g_ref[k]
                    rv[k] = opt.beta2 * rv[k] + (1 - opt.beta2) * g_ref[k] * g_ref[k]
                    lr_t = opt.lr * (1 - opt.beta2 ** t) ** 0.5 / (1 - opt.beta1 ** t)
                    rp[k] = rp[k] - lr_t * rm[k] / (rv[k].sqrt() + opt.eps)
                else:
                    rp[k], rm[k], rv[k] = tf1_apply(opt, rp[k], rm[k], rv[k], g_ref[k])
            got = w.read_variables()
            for k in got:
                assert torch.allclose(got[k], rp[k], rtol=1e-4, atol=1e-6), (i, k)


# ---------------------------------------------------------------------------------------------------------------
# the CLI
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
def test_cli_sigmoid_one_ps_two_workers():
    common = ["--learning_rate", "0.001", "--log_every", "1000", "--lanes", "1", "--activation", "sigmoid"]
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
