"""The workers' classification losses and label smoothing on both GPU engines: the head kernel per loss against torch
(bench_tools/gpu_check); every pushed element and the reported loss against the fp64 step within the bound of
bench_tools/fused_push_ref, at fused batches 32, 100 and 256, 4 pipelined lanes, a 2-shard row split, the atomic push,
a clip and L2, under the ReLU and tanh (so that every general-head instantiation of the fused kernel runs), and the graph
engine at 784-H-10; lock-step trajectories against fp32 torch (300 strict fused steps, 100 graph-engine zhihu steps, one
bf16 run); and `evaluate` on both engines and of the moving averages."""
import _harness
import pytest

from bench_tools import fused_push_ref as R
from dist_mnist_b200.models import mlp

pytestmark = pytest.mark.gpu

# (loss, label_smoothing): each new loss, and the smoothing of both cross-entropies
SETTINGS = [("sigmoid_xent", 0.0), ("sigmoid_xent", 0.1), ("mse", 0.0), ("hinge", 0.0), ("xent", 0.1), ("xent", 1.0)]
IDS = [f"{l}-ls{s:g}" for l, s in SETTINGS]


@pytest.mark.parametrize("loss,ls", SETTINGS, ids=IDS)
def test_head_kernel(loss, ls):
    from bench_tools import gpu_check

    assert gpu_check.check_head("relu", loss, ls)
    assert gpu_check.check_head("tanh", loss, ls)


# ---------------------------------------------------------------------------------------------------------------
# pushes against fp64
# ---------------------------------------------------------------------------------------------------------------
SHAPES = [(100, 10, 784, b) for b in (32, 100, 256)] + [(1, 2, 228, 1), (128, 11, 1024, 33)]


@pytest.mark.parametrize("act", ["relu", "tanh"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"H{h}-C{c}-I{i}-B{b}" for h, c, i, b in SHAPES])
@pytest.mark.parametrize("loss,ls", SETTINGS, ids=IDS)
def test_fused_push_is_inside_the_fp64_bound(loss, ls, shape, act):
    case = R.case_for((*shape, loss), activation=act, label_smoothing=ls)
    x, y = case.batches[0]
    with _harness.cluster(case) as cl:
        got = _harness.step(cl.worker, x, y)
    _harness.check(f"fused {case.name} seed {case.seed}", got, case, x, y)


@pytest.mark.parametrize("loss,ls", SETTINGS, ids=IDS)
def test_fused_pipelined_sharded_and_atomic_pushes(loss, ls):
    """4 lanes in flight matched to their batches one to one; a 2-shard row split; push == apply at lr 1."""
    import torch

    case = R.case_for((100, 10, 784, 100, loss), n_batches=8, seed=3, label_smoothing=ls)
    with _harness.cluster(case, lanes=4, nslots=8, strict=False) as cl:
        w = cl.worker
        loader = w.make_loader(torch.cat([b[0] for b in case.batches]), torch.cat([b[1] for b in case.batches]),
                               seed=0, shuffle=False)
        outs = list(w.run_steps(8, loader, wait_applied=True))
        assert sorted(o.seq for o in outs) == list(range(1, 9))
        pushes = [R.Step(R.pushed(w, o.seq), float(o.loss), int(o.correct)) for o in outs]
    refs = [R.reference(case.spec, case.params, x, y) for x, y in case.batches]
    hits = sorted(next(i for i, r in enumerate(refs) if R.compare(p, r).ok) for p in pushes)
    assert hits == list(range(8)), hits

    x, y = case.batches[0]
    with _harness.cluster(case, nps=2, sharding="row_split") as cl:
        got = _harness.step(cl.worker, x, y)
    _harness.check(f"fused row_split 2 ps {case.name}", got, case, x, y)

    with _harness.cluster(case, push_mode="atomic", lr=1.0) as cl:
        w = cl.worker
        out = w.step(x, y)
        w.wait_applied()
        p1 = w.read_variables()
    p0 = case.params
    ref = R.reference(case.spec, p0, x, y)
    for n in R.VARS:
        ref.bounds[n] = ref.bounds[n] + 2.0 ** -24 * torch.maximum(p0[n].double().abs(), p1[n].double().abs())
    g = {n: p0[n].double() - p1[n].double() for n in R.VARS}
    _harness.check(f"fused atomic {case.name}", R.Step(g, float(out.loss), int(out.correct)), case, x, y, ref)


@pytest.mark.parametrize("act", ["relu", "tanh"])
@pytest.mark.parametrize("B", [32, 33])
@pytest.mark.parametrize("loss,ls", SETTINGS, ids=IDS)
def test_fused_clip_and_l2_instantiations(loss, ls, B, act):
    """The clip, L2 and clip + L2 general-head instantiations: a clip by value that does not bind leaves the push as it
    is, and L2 adds fl(S w) to it (2 u of |g| + |S w| more in the bound) and its term to the reported loss."""
    import torch

    from dist_mnist_b200.parallel.config import GradClip, L2Regularization

    case = R.case_for((100, 10, 784, B, loss), activation=act, label_smoothing=ls)
    x, y = case.batches[0]
    wide = GradClip("value", value_min=-1e3, value_max=1e3)
    l2 = L2Regularization(1e-3, "all")
    for clip, reg in ((wide, None), (None, l2), (wide, l2)):
        with _harness.cluster(case, clip=clip, l2=reg) as cl:
            got = _harness.step(cl.worker, x, y)
        ref = R.reference(case.spec, case.params, x, y)
        if reg is not None:
            for n in R.VARS:
                sw = reg.scale * case.params[n].double()
                ref.grads[n] = ref.grads[n] + sw
                ref.bounds[n] = ref.bounds[n] + 2.0 ** -23 * (ref.grads[n].abs() + sw.abs())
            term = reg.scale * sum(float((case.params[n].double() ** 2).sum()) / 2 for n in R.VARS)
            ref.loss += term
            ref.loss_bound += 2.0 ** -16 * (term + abs(ref.loss))   # the fp32 sum of S w w / 2 over the variables
        _harness.check(f"fused clip={clip and clip.kind} l2={reg is not None} {case.name}", got, case, x, y, ref)
        assert torch.isfinite(got.grads["hid_w"]).all()


@pytest.mark.parametrize("H,B", [(100, 32), (128, 100)], ids=["H100-B32", "H128-B100"])
@pytest.mark.parametrize("loss,ls", SETTINGS, ids=IDS)
def test_graph_push_is_inside_the_fp64_bound(loss, ls, H, B):
    case = R.case_for((H, 10, 784, B, loss), label_smoothing=ls)
    x, y = case.batches[0]
    with _harness.cluster(case, engine="graph") as cl:
        got = _harness.step(cl.worker, x, y)
    _harness.check(f"graph {case.name}", got, case, x, y)


# ---------------------------------------------------------------------------------------------------------------
# trajectories and evaluate
# ---------------------------------------------------------------------------------------------------------------
def _lockstep(loss, ls, engine, model, steps, dtype="fp32", loss_tol=1e-2, param_tol=5e-3):
    from dist_mnist_b200.parallel.config import OptimizerConfig

    spec = mlp.get_model(model, 100, loss=loss, label_smoothing=ls)
    worst, errs = _harness.gpu_lockstep(spec, OptimizerConfig("sgd", 5e-2), engine, steps, dtype)
    perr = max(errs.values())
    print(f"[{engine} {model} {dtype} {loss} ls {ls}] {steps} steps: worst per-step loss rel err {worst:.2e}, "
          f"param rel err {perr:.2e} ({max(errs, key=errs.get)})")
    assert worst < loss_tol
    assert perr < param_tol


# The hinge's gradient jumps by k wherever a margin crosses its kink, so a tf32 rounding that moves one margin across
# changes the step by a whole k, and its mean loss falls towards the few margins left positive: on one H100 the hinge
# runs drifted to 10 % (fused) and 7 % (graph) in the per-step loss and 1.3 % / 2 % in the parameters. Each step's push
# is checked against fp64 above; these are 2x those drifts.
HINGE_TOL = {"fused": {"loss_tol": 0.2, "param_tol": 3e-2}, "graph": {"loss_tol": 0.15, "param_tol": 5e-2}}


@pytest.mark.parametrize("loss,ls", SETTINGS, ids=IDS)
def test_strict_fused_trajectory_is_lock_step_with_fp32_torch(loss, ls):
    _lockstep(loss, ls, "fused", "book", 300, **(HINGE_TOL["fused"] if loss == "hinge" else {}))


@pytest.mark.parametrize("loss,ls", SETTINGS, ids=IDS)
def test_graph_zhihu_trajectory_is_lock_step_with_fp32_torch(loss, ls):
    """The tolerances of the activations' zhihu runs: the tf32 GEMMs over the 500-wide layers drift further from fp32
    torch than the book model's."""
    _lockstep(loss, ls, "graph", "zhihu", 100,
              **(HINGE_TOL["graph"] if loss == "hinge" else {"loss_tol": 2e-2, "param_tol": 3e-2}))


def test_graph_zhihu_bf16_trajectory():
    _lockstep("sigmoid_xent", 0.1, "graph", "zhihu", 100, dtype="bf16", loss_tol=5e-2, param_tol=3e-2)


@pytest.mark.parametrize("engine,model,ema", [("fused", "book", False), ("graph", "book", False),
                                              ("graph", "zhihu", False), ("fused", "book", True),
                                              ("graph", "zhihu", True)])
@pytest.mark.parametrize("loss,ls", SETTINGS, ids=IDS)
def test_evaluate_reports_the_chosen_loss(loss, ls, engine, model, ema):
    from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    ds = data.synthetic_mnist(1024, seed=9)
    spec = mlp.get_model(model, 100, loss=loss, label_smoothing=ls)
    params = mlp.init_params(spec, seed=4)
    cfg = EngineConfig(backend="cuda", engine=engine, lanes=1, nslots=4)
    opt = OptimizerConfig("sgd", 0.0, **({"moving_average_decay": 0.99} if ema else {}))
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=1, params=params) as cl:
        loss_v, acc = cl.worker.evaluate(ds.images, ds.labels, moving_averages=ema)
    logits, _ = mlp.forward_logits(spec, params, ds.images.float())
    want_loss = float(mlp.loss_from_logits(spec, logits, ds.labels.float()))
    want_acc = mlp.accuracy_count(logits, ds.labels) / ds.images.shape[0]
    own = float(mlp.loss_from_logits(mlp.get_model(model, 100), logits, ds.labels.float()))
    print(f"[evaluate {engine} {model} ema={ema} {loss} ls {ls}] loss {loss_v:.6f} / {want_loss:.6f} (own loss "
          f"{own:.6f}), accuracy {acc} / {want_acc}")
    assert loss_v == pytest.approx(want_loss, rel=2e-3)
    assert abs(acc - want_acc) <= 4 / ds.images.shape[0]
    assert abs(own - want_loss) > 1e-3


@pytest.mark.parametrize("loss,ls", SETTINGS, ids=IDS)
def test_lane_cap_of_the_general_head(loss, ls):
    """The lane-cap query answers for the general head the selector picks for this loss, which fits as many clusters
    as the ReLU book head."""
    import ctypes as C

    from dist_mnist_b200 import _native as N

    lib = N.lib()
    N.ensure_prepared(0)

    def lanes(B, head):
        out = C.c_int(0)
        N.check(lib.dm_fused_max_lanes(0, B, 0, 0, head, C.byref(out)))
        return out.value

    for B in (1, 32, 33, 256):
        relu = lanes(B, N.fused_head_code(N.ACT_RELU, N.LOSS_BOOK, 0.0))
        assert relu > 0
        assert lanes(B, N.fused_head_code(N.ACT_RELU, mlp.loss_code(loss), ls)) == relu
