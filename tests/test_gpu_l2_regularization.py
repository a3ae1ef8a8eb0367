"""L2 weight regularization on both GPU engines: the regularized push against the unregularized push of the same step
plus fl(S * w) (isolating the L2 term from tf32 error), alone and under every clip kind, over the fused engine's batch
sizes, hidden sizes and shardings and on the graph engine (book and zhihu, fp32 and bf16); the reported loss against
the unregularized one plus the fp64 L2 term; lock-step trajectories against fp32 PyTorch with the reference L2 (300
fused steps, 100 graph steps); bit-identical repeated runs; and group graphs."""
import _harness
import pytest

from bench_tools.fused_push_ref import pushed

pytestmark = pytest.mark.gpu


def _one_step(H, B, nps, sharding, l2, clip=None, model="book", engine="fused", dtype="fp32"):
    """One strict step from fixed variables (seed 3, biases set) on batch 0 of a fixed dataset: (loss, pushed gradient,
    those variables)."""
    import torch

    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, GradClip, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    spec = mlp.get_model(model, H)
    ds = data.synthetic_mnist(512, seed=4)
    opt = OptimizerConfig("sgd", 1e-2, clip=clip or GradClip(), l2=l2)
    kw = {"strict_steps": True} if engine == "fused" else {}
    cfg = EngineConfig(backend="cuda", engine=engine, lanes=1, nslots=4, sharding=sharding, dtype=dtype, **kw)
    params = mlp.init_params(spec, seed=3)
    for k, v in params.items():   # nonzero biases (they start at zero), so that "all" has a term for them
        if v.dim() == 1:
            params[k] = torch.linspace(-0.05, 0.05, v.numel(), dtype=torch.float32)
    with InProcessCluster(spec, opt, cfg, batch_size=B, num_ps=nps, params=params) as cl:
        w = cl.worker
        assert w.engine == engine
        r = w.step(ds.images[:B], ds.labels[:B])
        w.wait_applied()
        return r.loss, pushed(w), params


def _clip_ref(g, clip):
    """The reference clip of `g` with its scale / divisors computed in fp64 and rounded to fp32."""
    import torch

    f32 = torch.float32
    if clip.kind == "value":
        lo, hi = torch.tensor(clip.value_min, dtype=f32), torch.tensor(clip.value_max, dtype=f32)
        return {k: torch.maximum(torch.minimum(v, hi), lo) for k, v in g.items()}
    c = torch.tensor(clip.clip_norm, dtype=f32)
    if clip.kind == "global_norm":
        n = float(sum((v.double() ** 2).sum() for v in g.values())) ** 0.5
        scale = torch.tensor(clip.clip_norm * min(1.0 / n, 1.0 / clip.clip_norm), dtype=f32)
        return {k: v * scale for k, v in g.items()}
    out = {}
    for k, v in g.items():
        l2 = float((v.double() ** 2).sum())
        den = torch.tensor(max(l2 ** 0.5 if l2 > 0 else l2, clip.clip_norm), dtype=f32)
        out[k] = (v * c) / den
    return out


def _check(H, B, nps, sharding, clips=False, **kw):
    import torch

    from dist_mnist_b200.parallel.config import GradClip, L2Regularization

    f32 = torch.float32
    loss0, g, params = _one_step(H, B, nps, sharding, L2Regularization(), **kw)
    for l2 in (L2Regularization(5e-3), L2Regularization(5e-3, "all")):
        s = torch.tensor(l2.scale, dtype=f32)
        reg = {k: (l2.variables == "all" or v.dim() == 2) for k, v in params.items()}
        exp = {k: g[k] + s * params[k] if reg[k] else g[k] for k in g}   # fl(g + fl(S * w))
        loss, got, _ = _one_step(H, B, nps, sharding, l2, **kw)
        # g is this step's unregularized push, recomputed in a run of its own: both engines compute it bit for bit
        # the same, so the one rounding of the addition is all that separates got from exp. The bound allows one more
        # ulp of each term for a summation order that differs between the two runs.
        for k in g:
            err = (got[k] - exp[k]).abs()
            tol = 2.0 ** -23 * (g[k].abs() + (s * params[k]).abs() * reg[k])
            assert bool((err <= tol).all()), (l2, k, float(err.max()))
            if reg[k]:
                assert not torch.equal(got[k], g[k]), (l2, k)
            else:
                assert torch.equal(got[k], g[k]), (l2, k)
        # the reported loss: data loss + S * sum(w*w) / 2, the term summed in fp64 and rounded to fp32; relative bound:
        # fp32 sums of up to 10^5 positive squares (~1e-6) and the fp32 addition
        term = l2.scale * sum(float((params[k].double() ** 2).sum()) / 2 for k in params if reg[k])
        want = float(torch.tensor(loss0 + term, dtype=torch.float64).to(f32))
        assert loss == pytest.approx(want, rel=1e-5), (l2, loss, loss0, term)
        if not clips:
            continue
        norms = {k: float(v.double().norm()) for k, v in exp.items()}
        gn = sum(n * n for n in norms.values()) ** 0.5
        top = max(float(v.abs().max()) for v in exp.values())
        for clip in (GradClip("global_norm", clip_norm=0.5 * gn),
                     GradClip("norm", clip_norm=sorted(norms.values())[len(norms) // 2]),
                     GradClip("value", value_min=-0.5 * top, value_max=0.25 * top)):
            _, got, _ = _one_step(H, B, nps, sharding, l2, clip=clip, **kw)
            ce = _clip_ref(exp, clip)
            for k in g:
                err = (got[k] - ce[k]).abs()
                # the clip's fp32 rounding + summation order (tests/test_gpu_grad_clip.py) on top of the bound above
                tol = 2e-6 * ce[k].abs() + 1e-9 * float(ce[k].abs().max()) + 2.0 ** -23 * ce[k].abs()
                if clip.kind == "value":
                    tol = 2.0 ** -23 * (g[k].abs() + (s * params[k]).abs() * reg[k])
                assert bool((err <= tol).all()), (l2, clip, k, float(err.max()))


# (H, B, #ps, sharding, with the clip kinds): every batch size at H = 100, both hidden sizes, both 2-shard layouts
SHAPES = ([(100, b, 1, "round_robin", b in (32, 256)) for b in (1, 32, 64, 100, 256)]
          + [(128, 32, 1, "round_robin", False), (128, 256, 1, "round_robin", False),
             (100, 100, 2, "round_robin", False), (100, 64, 2, "row_split", True), (128, 256, 2, "row_split", False)])


@pytest.mark.parametrize("shape", SHAPES, ids=[f"H{h}-B{b}-{n}ps-{s}{'-clips' if c else ''}" for h, b, n, s, c in SHAPES])
def test_fused_l2_push_is_the_unregularized_push_plus_s_w(shape):
    H, B, nps, sharding, clips = shape
    _check(H, B, nps, sharding, clips=clips)


GRAPH_CASES = [("book", "fp32", True), ("zhihu", "fp32", False), ("zhihu", "bf16", False), ("book", "bf16", False)]


@pytest.mark.parametrize("case", GRAPH_CASES, ids=[f"{m}-{d}{'-clips' if c else ''}" for m, d, c in GRAPH_CASES])
def test_graph_l2_push_is_the_unregularized_push_plus_s_w(case):
    """The graph engine's tail (csrc/clip_sm90.cu): w is read from the shard at the end of the step, which with one
    worker and lanes 1 is the value the step pulled (the ps applies nothing before the tail releases the flags)."""
    model, dtype, clips = case
    _check(100, 32, 1, "round_robin", clips=clips, model=model, engine="graph", dtype=dtype)


def _ref_l2_step(spec, params, x, y, lr, l2):
    from dist_mnist_b200.models import mlp

    loss, grads, _ = mlp.manual_loss_and_grads(spec, params, x, y)
    reg, grads = l2.apply(params, grads)
    for k in params:
        params[k] = params[k] - lr * grads[k]
    return float(loss + reg)


def _lockstep(engine, steps):
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import L2Regularization, OptimizerConfig

    spec = mlp.book_model(100)
    l2 = L2Regularization(5e-3, "all")
    opt = OptimizerConfig("sgd", 5e-2, l2=l2)
    worst, errs = _harness.gpu_lockstep(spec, opt, engine, steps,
                                        ref_update=lambda p, x, y: _ref_l2_step(spec, p, x, y, opt.lr, l2))
    perr = max(errs.values())
    print(f"[{engine} lock-step L2] {steps} steps: worst per-step loss rel err {worst:.2e}, param rel err {perr:.2e}")
    assert worst < 1e-2
    assert perr < 5e-3


def test_strict_fused_l2_trajectory_is_lock_step_with_fp32_torch():
    """300 strict steps: the bounds of tests/test_gpu_grad_clip.py's lock-step trajectories."""
    _lockstep("fused", 300)


def test_graph_l2_trajectory_is_lock_step_with_fp32_torch():
    """100 graph-engine steps, each followed by wait_applied (the read-your-writes order)."""
    _lockstep("graph", 100)


@pytest.mark.parametrize("B", [32, 100])
def test_strict_fused_l2_runs_are_bit_identical(B):
    import torch

    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, GradClip, L2Regularization, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    spec = mlp.book_model(100)
    ds = data.synthetic_mnist(8192, seed=8)
    opt = OptimizerConfig("adam", 1e-3, clip=GradClip("global_norm", clip_norm=0.1), l2=L2Regularization(1e-3, "all"))
    cfg = EngineConfig(backend="cuda", engine="fused", lanes=1, nslots=8, strict_steps=True)
    runs = []
    for _ in range(2):
        with InProcessCluster(spec, opt, cfg, batch_size=B, num_ps=1, params=mlp.init_params(spec, seed=2)) as cl:
            w = cl.worker
            outs = list(w.run_steps(200, w.make_loader(ds.images, ds.labels, seed=1), wait_applied=True))
            assert len(outs) == 200
            runs.append(([o.loss for o in outs], w.read_variables()))
    assert runs[0][0] == runs[1][0]
    for k in runs[0][1]:
        assert torch.equal(runs[0][1][k], runs[1][1][k]), k


@pytest.mark.parametrize("model,dtype", [("zhihu", "bf16"), ("book", "fp32")])
def test_graph_l2_pipelined_runs_with_group_graphs(model, dtype):
    """4 lanes in group graphs of 2 steps: every push lands and is applied, and training makes progress."""
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, L2Regularization, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    opt = OptimizerConfig("adam", 1e-3, l2=L2Regularization(1e-4))
    cfg = EngineConfig(backend="cuda", engine="graph", lanes=4, graph_steps=2, nslots=8, dtype=dtype)
    ds = data.synthetic_mnist(8192, seed=6)
    with InProcessCluster(mlp.get_model(model, 100), opt, cfg, batch_size=64, num_ps=2) as cl:
        w = cl.worker
        assert w.engine == "graph"
        loader = w.make_loader(ds.images, ds.labels, seed=0)
        outs = list(w.run_steps(300, loader, wait_applied=True)) + list(w.run_steps(96, loader, wait_applied=True))
        assert len(outs) == 396 and w.read_global_step() == 396
        assert sorted(o.seq for o in outs) == list(range(1, 397))
        first = sum(o.loss for o in outs[:20]) / 20
        last = sum(o.loss for o in outs[-20:]) / 20
        assert last < 0.7 * first, (first, last)

