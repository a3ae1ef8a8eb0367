"""The workers' classification losses (`--loss`, `--label_smoothing`) on the cpu backend and in the fp64 push checker:
TF 1.15's tf.losses values, the hand-derived gradients against autograd, the flags, lock-step runs and the CLI."""
import math

import _harness
import pytest
import torch
import torch.nn.functional as F

from bench_tools import fused_push_ref as R
from bench_tools.gpu_e2e import ref_slots, tf1_apply
from dist_mnist_b200 import cli
from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.config import EngineConfig, GradClip, L2Regularization, OptimizerConfig
from dist_mnist_b200.session import InProcessCluster
from dist_mnist_b200.utils import data


def _head(loss, z, y, ls=0.0):
    """(mean loss, dz) of `loss` on logits z and labels y [B, C] from the cpu backend's hand-derived step: a model whose
    logits are its sm_b (sm_w = 0), so that the gradient of sm_b, summed over a one-row batch, is dz."""
    z, y = torch.tensor([z], dtype=torch.float32), torch.tensor([y], dtype=torch.float32)
    C = z.shape[1]
    spec = mlp.MLPSpec(in_features=4, hidden=(3,), num_classes=C, loss=loss, label_smoothing=ls)
    params = mlp.init_params(spec, seed=0)
    params["sm_w"].zero_()
    params["sm_b"] = z[0].clone()
    loss_v, grads, logits = mlp.manual_loss_and_grads(spec, params, torch.ones(1, 4), y)
    assert torch.equal(logits, z)
    assert float(mlp.loss_from_logits(spec, z, y)) == pytest.approx(float(loss_v), rel=1e-6, abs=1e-30)
    return float(loss_v), grads["sm_b"].tolist()


LN2 = math.log(2.0)
# (loss, ls, z, y, TF1 loss, TF1 dz) on one row; values from the tf.losses formulas with weight 1
TF1_VALUES = [
    ("sigmoid_xent", 0.0, [0.0], [1.0], LN2, [-0.5]),
    ("sigmoid_xent", 0.0, [100.0], [1.0], 0.0, [0.0]),            # exp(-100) underflows to a denormal, no overflow
    ("sigmoid_xent", 0.0, [-100.0], [1.0], 100.0, [-1.0]),
    ("sigmoid_xent", 0.0, [100.0], [0.0], 100.0, [1.0]),
    ("sigmoid_xent", 0.0, [-100.0], [0.0], 0.0, [0.0]),
    ("sigmoid_xent", 0.1, [0.0], [1.0], LN2, [0.5 - 0.95]),       # y' = 0.9 + 0.05
    ("sigmoid_xent", 1.0, [0.0, 2.0], [1.0, 0.0], (LN2 + 2.0 - 1.0 + math.log1p(math.exp(-2.0))) / 2,
     [0.0, (1 / (1 + math.exp(-2.0)) - 0.5) / 2]),                 # every y' = 0.5
    ("mse", 0.0, [3.0, -1.0], [1.0, 0.0], (4.0 + 1.0) / 2, [2.0, -1.0]),
    ("mse", 0.0, [100.0], [0.0], 1e4, [200.0]),
    ("hinge", 0.0, [1.0], [1.0], 0.0, [0.0]),                      # the kink: 1 - z = 0 takes no gradient
    ("hinge", 0.0, [-1.0], [0.0], 0.0, [0.0]),                     # the kink on the negative side
    ("hinge", 0.0, [0.5, 0.0], [1.0, 0.0], (0.5 + 1.0) / 2, [-0.5, 0.5]),
    ("hinge", 0.0, [-100.0, 100.0], [0.0, 1.0], 0.0, [0.0, 0.0]),
    ("hinge", 0.0, [100.0], [0.0], 101.0, [1.0]),
    ("xent", 0.1, [0.0] * 10, [1.0] + [0.0] * 9, math.log(10.0), [0.1 - 0.91] + [0.1 - 0.01] * 9),
    ("xent", 1.0, [0.0] * 10, [1.0] + [0.0] * 9, math.log(10.0), [0.0] * 10),
    ("xent", 0.0, [100.0, -100.0], [0.0, 1.0], 200.0, [1.0, -1.0]),
]


@pytest.mark.parametrize("loss,ls,z,y,want_loss,want_dz", TF1_VALUES,
                         ids=[f"{t[0]}-ls{t[1]}-{i}" for i, t in enumerate(TF1_VALUES)])
def test_losses_match_tf1(loss, ls, z, y, want_loss, want_dz):
    got_loss, got_dz = _head(loss, z, y, ls)
    assert math.isfinite(got_loss) and all(math.isfinite(v) for v in got_dz)
    assert got_loss == pytest.approx(want_loss, rel=1e-6, abs=1e-7)
    assert got_dz == pytest.approx(want_dz, rel=1e-6, abs=1e-7)


def test_smoothing_rounds_as_tf1_and_zero_keeps_the_labels():
    y = torch.tensor([[1.0, 0.0, 0.0]])
    for loss in ("xent", "sigmoid_xent"):
        assert mlp.smooth_labels(mlp.MLPSpec(num_classes=3, loss=loss), y) is y
    ls = 0.1
    keep = torch.tensor(1.0 - float(torch.tensor(ls, dtype=torch.float32)), dtype=torch.float32)
    xent = mlp.smooth_labels(mlp.MLPSpec(num_classes=3, loss="xent", label_smoothing=ls), y)
    assert torch.equal(xent, y * keep + torch.tensor(ls, dtype=torch.float32) / torch.tensor(3.0))
    sig = mlp.smooth_labels(mlp.MLPSpec(num_classes=3, loss="sigmoid_xent", label_smoothing=ls), y)
    assert torch.equal(sig, y * keep + torch.tensor(0.5 * float(torch.tensor(ls, dtype=torch.float32))))
    one = mlp.smooth_labels(mlp.MLPSpec(num_classes=3, loss="xent", label_smoothing=1.0), y)
    assert torch.equal(one, torch.full_like(y, float(torch.tensor(1.0) / 3)))


def _independent_loss(spec, z, y):
    """torch's own losses, whose autograd derivatives are independent of `manual_loss_and_grads`. The smoothed labels
    are the fp32 ones every engine uses (their rounding is checked on its own above)."""
    ys = mlp.smooth_labels(spec, y.float()).to(y.dtype)
    if spec.loss == "xent":
        return F.cross_entropy(z, ys)
    if spec.loss == "sigmoid_xent":
        return F.binary_cross_entropy_with_logits(z, ys)
    if spec.loss == "mse":
        return F.mse_loss(z, y)
    if spec.loss == "hinge":
        return torch.clamp(1 - (2 * y - 1) * z, min=0).mean()
    return mlp.loss_from_logits(spec, z, y)


LOSS_SETTINGS = [("xent", 0.0), ("xent", 0.1), ("xent", 1.0), ("sigmoid_xent", 0.0), ("sigmoid_xent", 0.1),
                 ("sigmoid_xent", 1.0), ("mse", 0.0), ("hinge", 0.0)]


@pytest.mark.parametrize("hidden", [(7,), (7, 5)], ids=["1-hidden", "2-hidden"])
@pytest.mark.parametrize("loss,ls", LOSS_SETTINGS, ids=[f"{l}-ls{s:g}" for l, s in LOSS_SETTINGS])
def test_manual_gradients_match_autograd_in_fp64(loss, ls, hidden):
    spec = mlp.MLPSpec(name="t", in_features=12, hidden=hidden, num_classes=4, loss=loss, init="glorot",
                       activation="tanh", label_smoothing=ls)
    g = torch.Generator().manual_seed(3)
    params = {k: v.double() * 3 for k, v in mlp.init_params(spec, seed=1).items()}   # logits past +-1 for the hinge
    x = torch.rand(6, 12, generator=g, dtype=torch.float64)
    y = torch.zeros(6, 4, dtype=torch.float64)
    y[torch.arange(6), torch.randint(0, 4, (6,), generator=g)] = 1.0
    loss_m, g_m, logits = mlp.manual_loss_and_grads(spec, params, x, y)
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    z, _ = mlp.forward_logits(spec, leaves, x, act_fn=mlp._activate_autograd)
    loss_a = _independent_loss(spec, z, y)
    g_a = dict(zip(leaves, torch.autograd.grad(loss_a, list(leaves.values()))))
    if loss == "hinge":   # no margin sits at the kink, where the two may pick different one-sided derivatives
        assert float((1 - (2 * y - 1) * logits).abs().min()) > 1e-6
    assert float(loss_m) == pytest.approx(float(loss_a.detach()), rel=1e-12)
    if loss == "xent":   # torch's own smoothing, in exact arithmetic: equal up to the fp32 rounding of y'
        assert float(loss_m) == pytest.approx(float(F.cross_entropy(z.detach(), y.argmax(dim=1), label_smoothing=ls)), rel=1e-6)
    for k in g_m:
        assert torch.allclose(g_m[k], g_a[k], rtol=1e-10, atol=1e-13), (k, float((g_m[k] - g_a[k]).abs().max()))


def test_accuracy_uses_the_raw_labels_under_full_smoothing():
    """With ls = 1 every smoothed label is equal; the correct count must still compare with the raw argmax."""
    spec = mlp.MLPSpec(num_classes=3, loss="xent", label_smoothing=1.0)
    logits = torch.tensor([[0.0, 5.0, 0.0], [0.0, 0.0, 5.0]])
    y = torch.tensor([[0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])
    assert mlp.accuracy_count(logits, y) == 2
    assert mlp.accuracy_count(logits, mlp.smooth_labels(spec, y)) == 0   # what a count of y' would give


# ---------------------------------------------------------------------------------------------------------------
# flags and config
# ---------------------------------------------------------------------------------------------------------------
def _loss_args(argv):
    return cli.loss_from_args(cli.build_parser().parse_args(argv))


def test_flag_defaults_choices_and_refusals():
    p = cli.build_parser()
    a = p.parse_args([])
    assert a.loss is None and a.label_smoothing is None
    assert _loss_args([]) == (None, 0.0)
    for name in mlp.LOSSES:
        assert p.parse_args(["--loss", name]).loss == name
    for bad in ("huber", "softmax", "XENT", ""):
        with pytest.raises(SystemExit):
            p.parse_args(["--loss", bad])
    assert _loss_args(["--loss", "sigmoid_xent", "--label_smoothing", "0.1"]) == ("sigmoid_xent", 0.1)
    assert _loss_args(["--model", "zhihu", "--label_smoothing", "0.2"]) == (None, 0.2)   # zhihu's own loss is xent
    with pytest.raises(ValueError, match=r"--label_smoothing does not apply to --loss book \(only xent, sigmoid_xent\)"):
        _loss_args(["--label_smoothing", "0.1"])                                           # book's own loss
    for loss in ("book", "mse", "hinge"):
        with pytest.raises(ValueError, match=f"does not apply to --loss {loss}"):
            _loss_args(["--loss", loss, "--label_smoothing", "0"])
    for bad in ("-0.1", "1.5", "nan", "inf"):
        with pytest.raises(ValueError, match="finite and in"):
            _loss_args(["--loss", "xent", "--label_smoothing", bad])
    with pytest.raises(ValueError, match="unknown loss"):
        mlp.MLPSpec(loss="huber")
    with pytest.raises(ValueError, match="unknown loss"):
        mlp.get_model("book", 100, loss="l1")
    with pytest.raises(ValueError, match="does not apply to loss mse"):
        mlp.get_model("book", 100, loss="mse", label_smoothing=0.1)
    with pytest.raises(ValueError, match="finite"):
        mlp.MLPSpec(loss="xent", label_smoothing=float("nan"))


def test_models_keep_their_own_loss_unless_given():
    assert mlp.get_model("book", 100) == mlp.book_model(100)
    assert mlp.get_model("zhihu").loss == mlp.get_model("wide").loss == "xent"
    assert mlp.get_model("book", 100, loss="book", label_smoothing=0.0) == mlp.book_model(100)
    for model in ("book", "zhihu", "wide"):
        spec = mlp.get_model(model, 64, loss="hinge")
        assert spec.loss == "hinge" and spec.variables() == mlp.get_model(model, 64).variables()
    assert [mlp.loss_code(n) for n in mlp.LOSSES] == list(range(5))


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


def test_explicit_own_loss_is_bit_identical_and_other_losses_differ():
    opt = OptimizerConfig("momentum", 1e-2)
    for model in ("book", "zhihu"):
        base = _run(mlp.get_model(model, 100), opt, 3)
        explicit = _run(mlp.get_model(model, 100, loss=mlp.get_model(model).loss, label_smoothing=0.0), opt, 3)
        assert explicit[0] == base[0]
        for a, b in zip(explicit[1], base[1]):
            assert all(torch.equal(a[k], b[k]) for k in a)
    base = _run(mlp.book_model(100), opt, 1)
    for loss, ls in (("xent", 0.0), ("sigmoid_xent", 0.1), ("mse", 0.0), ("hinge", 0.0)):
        assert _run(mlp.get_model("book", 100, loss=loss, label_smoothing=ls), opt, 1)[0][0] != base[0][0]


# ---------------------------------------------------------------------------------------------------------------
# the fp64 push checker under every loss
# ---------------------------------------------------------------------------------------------------------------
SUBSET = [(100, 10, 784, b) for b in (1, 31, 32, 33, 100, 256)] + [(1, 2, 228, 32), (17, 3, 260, 33),
                                                                    (128, 11, 1024, 256)]


@pytest.mark.parametrize("shape", SUBSET, ids=[f"H{h}-C{c}-I{i}-B{b}" for h, c, i, b in SUBSET])
@pytest.mark.parametrize("loss,ls", LOSS_SETTINGS, ids=[f"{l}-ls{s:g}" for l, s in LOSS_SETTINGS])
def test_emulated_kernel_is_inside_the_bound_and_loss_mutants_are_not(loss, ls, shape):
    case = R.case_for((*shape, loss), label_smoothing=ls)
    x, y = case.batches[0]
    assert R.check_case(case, x, y) == [] and R.exact_inputs(case) == []
    ref = R.reference(case.spec, case.params, x, y)
    for mode in ("trunc", "rne"):
        v = R.compare(R.emulate(case.spec, case.params, x, y, mode), ref)
        print(f"[{case.name} seed {case.seed}] emulated, tf32 {mode}: {v.line()}")
        assert v.ok and v.max < 0.6, (mode, v.worst, v.where)
    for mode in ("trunc", "rne"):
        for mut, arg in R.mutant_instances(case, ref):
            v = R.compare(R.emulate(case.spec, case.params, x, y, mode, mut, arg), ref)
            assert v.max > (20.0 if mut in R.LOSS_MUTANTS + R.ACT_MUTANTS else 4.0), (mode, mut, arg, v.worst)


def test_every_loss_mutant_is_admitted_somewhere():
    seen = set()
    for loss, ls in LOSS_SETTINGS:
        for shape in ((100, 10, 784, 32), (128, 11, 1024, 256)):
            case = R.case_for((*shape, loss), label_smoothing=ls)
            seen |= {m for m, _ in R.mutant_instances(case, R.reference(case.spec, case.params, *case.batches[0]))}
    assert set(R.LOSS_MUTANTS) <= seen, set(R.LOSS_MUTANTS) - seen


def test_unsmoothed_cases_are_unchanged_by_the_smoothing_argument():
    for shape in ((100, 10, 784, 33, "book"), (17, 3, 260, 33, "xent")):
        a, b = R.case_for(shape), R.case_for(shape, label_smoothing=0.0)
        assert a.seed == b.seed and a.name == b.name
        assert all(torch.equal(a.params[k], b.params[k]) for k in a.params)


# ---------------------------------------------------------------------------------------------------------------
# lock-step runs
# ---------------------------------------------------------------------------------------------------------------
SHARDINGS = [(1, "round_robin"), (2, "row_split")]
EXTRAS = {"plain": {}, "l2-clip": {"l2": L2Regularization(1e-3), "clip": GradClip("global_norm", clip_norm=0.05)}}


@pytest.mark.parametrize("extra", list(EXTRAS))
@pytest.mark.parametrize("shards", SHARDINGS, ids=[f"{n}ps-{s}" for n, s in SHARDINGS])
@pytest.mark.parametrize("loss,ls", [("sigmoid_xent", 0.1), ("mse", 0.0), ("hinge", 0.0), ("xent", 0.1)],
                         ids=["sigmoid_xent-ls0.1", "mse", "hinge", "xent-ls0.1"])
def test_lockstep_trajectory(loss, ls, shards, extra):
    """1 worker, --lanes 1 --strict_steps: the step pulls exactly what read_variables() shows before it, so its loss
    (with the L2 term) is the fp32 reference's bit for bit; the parameters after every step match fp32 torch applying
    the reference's (regularized, clipped) gradient."""
    nps, sharding = shards
    opt = OptimizerConfig("momentum", 1e-2, **EXTRAS[extra])
    spec = mlp.get_model("book", 100, loss=loss, label_smoothing=ls)
    ds = data.synthetic_mnist(512, seed=2)
    it = data.BatchIterator(ds, seed=0)
    params = mlp.init_params(spec, seed=5)
    rp = {k: v.clone() for k, v in params.items()}
    rm, rv = ref_slots(opt, params)
    with InProcessCluster(spec, opt, EngineConfig(backend="cpu", lanes=1, strict_steps=True, sharding=sharding),
                          batch_size=32, num_ps=nps, params=params) as cl:
        w = cl.worker
        for i in range(6):
            x, y = it.next_batch(32)
            pulled = w.read_variables()
            r = w.step(x, y)
            w.wait_applied()
            loss_ref, g_ref, logits = mlp.manual_loss_and_grads(spec, pulled, x, y)
            if opt.l2.enabled:
                reg, _ = opt.l2.apply(pulled, g_ref)
                loss_ref = loss_ref + reg
            assert r.loss == float(loss_ref), i
            assert r.correct == mlp.accuracy_count(logits, y)
            _, g, _ = mlp.manual_loss_and_grads(spec, rp, x, y)
            if opt.l2.enabled:
                _, g = opt.l2.apply(rp, g)
            g = opt.clip.apply(g)
            for k in rp:
                rp[k], rm[k], rv[k] = tf1_apply(opt, rp[k], rm[k], rv[k], g[k])
            got = w.read_variables()
            for k in got:
                assert torch.allclose(got[k], rp[k], rtol=1e-4, atol=1e-6), (i, k)


def test_evaluate_reports_the_smoothed_loss():
    spec = mlp.get_model("book", 100, loss="sigmoid_xent", label_smoothing=0.1)
    ds = data.synthetic_mnist(256, seed=4)
    with InProcessCluster(spec, OptimizerConfig("sgd", 0.0), EngineConfig(backend="cpu", lanes=1), batch_size=32,
                          params=mlp.init_params(spec, seed=5)) as cl:
        loss, acc = cl.worker.evaluate(ds.images, ds.labels)
        params = cl.worker.read_variables()
    logits, _ = mlp.forward_logits(spec, params, ds.images.float())
    assert loss == float(mlp.loss_from_logits(spec, logits, ds.labels.float()))
    assert loss != float(mlp.loss_from_logits(mlp.get_model("book", 100, loss="sigmoid_xent"), logits,
                                              ds.labels.float()))
    assert acc == mlp.accuracy_count(logits, ds.labels) / 256


# ---------------------------------------------------------------------------------------------------------------
# the CLI
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
def test_cli_sigmoid_xent_smoothed_one_ps_two_workers():
    """The workers train with sigmoid_xent smoothed by 0.1; the ps is given a combination a worker would refuse (mse
    takes no smoothing) and ignores it."""
    common = ["--learning_rate", "0.001", "--log_every", "1000", "--lanes", "1"]
    with _harness.Tasks() as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done", "--loss", "mse", "--label_smoothing", "0.5"])
        ws = [t.spawn("worker", i, common + ["--loss", "sigmoid_xent", "--label_smoothing", "0.1"]) for i in (1, 0)]
        outs = [t.finish(w, 780) for w in ws]
        outp = t.finish(ps, 60)
    for w, o in zip(ws, outs):
        assert w.returncode == 0, o
        assert "done: local_steps=" in o, o
    assert ps.returncode == 0, outp
    assert int(outp.split("global_step=")[1].split()[0]) >= 4000, outp
