"""Gradient clipping on both GPU engines: the clipped push against the unclipped push of the same step transformed by
the reference clip (isolating the clip from tf32 error), for every kind over the fused engine's batch sizes, hidden
sizes and shardings and on the graph engine (zhihu in fp32 and bf16); lock-step trajectories against fp32 PyTorch
with the reference clip (300 fused steps, 100 graph steps); pipelined graph-engine runs with several steps per graph;
bit-identical repeated runs; and the fused lanes staying resident beside the ps."""
import pytest

from bench_tools.fused_push_ref import pushed

pytestmark = pytest.mark.gpu


def _one_step_push(H, B, nps, sharding, clip, model="book", engine="fused", dtype="fp32"):
    """One strict step from the initial variables (seed 3) on batch 0 of a fixed dataset; the pushed gradient."""
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    spec = mlp.get_model(model, H)
    ds = data.synthetic_mnist(512, seed=4)
    opt = OptimizerConfig("sgd", 1e-2, clip=clip)
    kw = {"strict_steps": True} if engine == "fused" else {}
    cfg = EngineConfig(backend="cuda", engine=engine, lanes=1, nslots=4, sharding=sharding, dtype=dtype, **kw)
    with InProcessCluster(spec, opt, cfg, batch_size=B, num_ps=nps, params=mlp.init_params(spec, seed=3)) as cl:
        w = cl.worker
        assert w.engine == engine
        w.step(ds.images[:B], ds.labels[:B])
        w.wait_applied()
        return pushed(w)


def _expected(g, clip):
    """The reference clip of the unclipped push `g` with its scale / divisors computed in fp64 and rounded to fp32."""
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


# (H, B, #ps, sharding): every batch size at H = 100, every hidden size at B = 32, both 2-shard layouts at B = 100
SHAPES = ([(100, b, 1, "round_robin") for b in (1, 32, 100, 256)] + [(h, 32, 1, "round_robin") for h in (128, 72)]
          + [(100, 100, 2, "round_robin"), (100, 100, 2, "row_split"), (72, 256, 2, "row_split")])


@pytest.mark.parametrize("shape", SHAPES, ids=[f"H{h}-B{b}-{n}ps-{s}" for h, b, n, s in SHAPES])
def test_fused_clipped_push_is_the_reference_clip_of_the_unclipped_push(shape):
    _check_clipped_pushes(*shape)


GRAPH_CASES = [("fp32", 32, 1), ("bf16", 32, 1), ("fp32", 100, 2)]


@pytest.mark.parametrize("case", GRAPH_CASES, ids=[f"zhihu-{d}-B{b}-{n}ps" for d, b, n in GRAPH_CASES])
def test_graph_clipped_push_is_the_reference_clip_of_the_unclipped_push(case):
    """The graph engine's clip tail (csrc/clip_sm90.cu) on the zhihu model: the epilogues push into the slot's local
    buffer, the tail writes the clipped gradient into the mailbox and releases the flags."""
    dtype, B, nps = case
    _check_clipped_pushes(100, B, nps, "round_robin", model="zhihu", engine="graph", dtype=dtype)


def _check_clipped_pushes(H, B, nps, sharding, **kw):
    import torch

    from dist_mnist_b200.parallel.config import GradClip

    g = _one_step_push(H, B, nps, sharding, GradClip(), **kw)
    norms = {k: float(v.double().norm()) for k, v in g.items()}
    gn = sum(n * n for n in norms.values()) ** 0.5
    top = max(float(v.abs().max()) for v in g.values())
    clips = [GradClip("global_norm", clip_norm=0.5 * gn),                       # clipped
             GradClip("global_norm", clip_norm=41.0 * gn),                      # not clipped: scale 41 * fl(1/41)
             # between the variables' norms: some variables are clipped, the others not
             GradClip("norm", clip_norm=sorted(norms.values())[len(norms) // 2]),
             GradClip("value", value_min=-0.5 * top, value_max=0.25 * top)]
    for clip in clips:
        got = _one_step_push(H, B, nps, sharding, clip, **kw)
        exp = _expected(g, clip)
        for k in g:
            if clip.kind == "value":
                assert torch.equal(got[k], exp[k]), (clip, k)
                continue
            err = (got[k] - exp[k]).abs()
            tol = 2e-6 * exp[k].abs() + 1e-9 * float(exp[k].abs().max())   # fp32 rounding + summation order
            assert bool((err <= tol).all()), (clip, k, float(err.max()), float((err / exp[k].abs()).nan_to_num().max()))
        if clip.kind != "global_norm" or clip.clip_norm < gn:
            assert not all(torch.equal(got[k], g[k]) for k in g), clip   # the clip did something


def _ref_clip_step(spec, params, x, y, lr, clip):
    from dist_mnist_b200.models import mlp

    loss, grads, _ = mlp.manual_loss_and_grads(spec, params, x, y)
    n = float(sum((g.double() ** 2).sum() for g in grads.values())) ** 0.5
    grads = clip.apply(grads)
    for k in params:
        params[k] = params[k] - lr * grads[k]
    return float(loss), n


def test_strict_fused_clipped_trajectory_is_lock_step_with_fp32_torch():
    """300 strict steps with clip_by_global_norm active on some steps: the bounds of
    tests/test_gpu_lr_schedules.py::test_strict_fused_native_loop_under_a_schedule_is_lock_step_with_fp32_torch."""
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, GradClip, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    ds = data.synthetic_mnist(8192, seed=5)
    spec = mlp.book_model(100)
    params = mlp.init_params(spec, seed=11)
    ref_p = {k: t.clone() for k, t in params.items()}
    # clip_norm: the median global norm of the first batches at the initial variables, so that clipping is active on
    # some steps and not on others (asserted below)
    probe = data.BatchIterator(ds, seed=0)
    norms = sorted(_ref_clip_step(spec, dict(params), *probe.next_batch(32), 0.0, GradClip())[1] for _ in range(21))
    clip = GradClip("global_norm", clip_norm=norms[10])
    opt = OptimizerConfig("sgd", 5e-2, clip=clip)
    cfg = EngineConfig(backend="cuda", engine="fused", lanes=1, nslots=8, strict_steps=True)
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=1, params=params) as cl:
        w = cl.worker
        loader = w.make_loader(ds.images, ds.labels, seed=7)
        twin = w.make_loader(ds.images, ds.labels, seed=7, epoch_feed=False)
        outs = []
        for n in (7, 93, 200):
            outs += list(w.run_steps(n, loader, wait_applied=True))
        assert len(outs) == 300 and w.read_global_step() == 300
        worst, clipped = 0.0, []
        for o in outs:
            x, y = twin.next_batch()
            lref, gn = _ref_clip_step(spec, ref_p, x, y, opt.lr, clip)
            clipped.append(gn > clip.clip_norm)
            if lref > 1e-6:
                worst = max(worst, abs(o.loss - lref) / abs(lref))
        got = w.read_variables()
    perr = max(float((got[k] - ref_p[k]).norm() / (ref_p[k].norm() + 1e-9)) for k in got)
    print(f"[lock-step clipped] 300 steps, {sum(clipped)} clipped: worst per-step loss rel err {worst:.2e}, "
          f"param rel err {perr:.2e}")
    assert any(clipped) and not all(clipped)
    assert worst < 1e-2
    assert perr < 5e-3


@pytest.mark.parametrize("B", [32, 100])
def test_strict_fused_clipped_runs_are_bit_identical(B):
    import torch

    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, GradClip, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    spec = mlp.book_model(100)
    ds = data.synthetic_mnist(8192, seed=8)
    opt = OptimizerConfig("adam", 1e-3, clip=GradClip("global_norm", clip_norm=0.1))
    cfg = EngineConfig(backend="cuda", engine="fused", lanes=1, nslots=8, strict_steps=True)
    ends = []
    for _ in range(2):
        with InProcessCluster(spec, opt, cfg, batch_size=B, num_ps=1, params=mlp.init_params(spec, seed=2)) as cl:
            w = cl.worker
            outs = list(w.run_steps(200, w.make_loader(ds.images, ds.labels, seed=1), wait_applied=True))
            assert len(outs) == 200
            ends.append(w.read_variables())
    for k in ends[0]:
        assert torch.equal(ends[0][k], ends[1][k]), k


def test_clipping_lanes_stay_resident_beside_the_ps():
    """tests/test_gpu_lane_residency.py with the clip instantiation."""
    from bench_tools import lane_residency

    from dist_mnist_b200.parallel.config import GradClip
    from dist_mnist_b200.parallel.ps import serve_geometry

    res = lane_residency.run(lanes=12, steps=20000, warmup=50, batch=32, clip=GradClip("global_norm", clip_norm=0.1))
    lanes = res["lanes"]
    n_ctas, cluster = serve_geometry(35, 0, True, "fused")
    assert res["ps_ctas"] == n_ctas
    assert lanes == min(12, res["fused_max_active_clusters_before_ps"] - n_ctas // cluster)
    claims = [c["steps"] for c in res["clusters"]]
    assert len(claims) == lanes and sum(claims) == 20000
    assert min(claims) > 0, claims
    step_us = res["us_per_step_per_lane"]
    late = [c for c in res["clusters"] if c["first_claim_us"] > step_us]
    assert not late, (step_us, late)


def test_graph_clipped_trajectory_is_lock_step_with_fp32_torch():
    """100 graph-engine steps, each followed by wait_applied (the read-your-writes order), with clip_by_global_norm
    active on some steps: the bounds of the fused trajectory above."""
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, GradClip, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    ds = data.synthetic_mnist(8192, seed=5)
    spec = mlp.book_model(100)
    params = mlp.init_params(spec, seed=11)
    ref_p = {k: t.clone() for k, t in params.items()}
    it = data.BatchIterator(ds, seed=0)
    norms = sorted(_ref_clip_step(spec, dict(params), *it.next_batch(32), 0.0, GradClip())[1] for _ in range(21))
    clip = GradClip("global_norm", clip_norm=norms[10])
    opt = OptimizerConfig("sgd", 5e-2, clip=clip)
    cfg = EngineConfig(backend="cuda", engine="graph", lanes=1, nslots=8)
    it = data.BatchIterator(ds, seed=3)
    worst, clipped = 0.0, []
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=1, params=params) as cl:
        w = cl.worker
        assert w.engine == "graph"
        for _ in range(100):
            x, y = it.next_batch(32)
            o = w.step(x, y)
            w.wait_applied()
            lref, gn = _ref_clip_step(spec, ref_p, x, y, opt.lr, clip)
            clipped.append(gn > clip.clip_norm)
            if lref > 1e-6:
                worst = max(worst, abs(o.loss - lref) / abs(lref))
        assert w.read_global_step() == 100
        got = w.read_variables()
    perr = max(float((got[k] - ref_p[k]).norm() / (ref_p[k].norm() + 1e-9)) for k in got)
    print(f"[graph lock-step clipped] 100 steps, {sum(clipped)} clipped: worst per-step loss rel err {worst:.2e}, "
          f"param rel err {perr:.2e}")
    assert any(clipped) and not all(clipped)
    assert worst < 1e-2
    assert perr < 5e-3


@pytest.mark.parametrize("model,dtype", [("zhihu", "bf16"), ("book", "fp32")])
def test_graph_clipped_pipelined_runs_with_group_graphs(model, dtype):
    """4 lanes in group graphs of 2 steps (graph_steps > 1: each chain clips through its own slot's buffer): every
    push lands and is applied, and training makes progress under clip_by_norm."""
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, GradClip, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    opt = OptimizerConfig("adam", 1e-3, clip=GradClip("norm", clip_norm=0.05))
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
