"""Fused step engine at batches of 33..256 rows (ceil(B / 32) row tiles per step) on one H100: agreement with the
per-layer graph engine, lock-step parity with un-rounded fp32 PyTorch, and the native loop with several lanes,
row_split sharding, the epoch feed, StopAtStep semantics and evaluation. Batch 32 (one tile) runs alongside as the
yardstick. `engine="auto"` keeps the graph engine above 32 rows, so these tests ask for the fused engine."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BATCHES = [32, 33, 64, 100, 128, 256]


def _cluster(cfg_kw, opt, batch, num_ps=1, params=None):
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster

    spec = mlp.book_model(100)
    cfg = EngineConfig(backend="cuda", **cfg_kw)
    return spec, InProcessCluster(spec, OptimizerConfig(*opt), cfg, batch_size=batch, num_ps=num_ps, params=params)


@pytest.mark.parametrize("batch", BATCHES)
def test_fused_and_graph_engines_agree_at_batch(batch):
    """Same parameters, same batches, 50 SGD steps with one step in flight: the tolerances of
    tests/test_gpu_fused.py::test_fused_and_graph_engines_agree."""
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.utils import data

    ds = data.synthetic_mnist(4096, seed=1)
    params = mlp.init_params(mlp.book_model(100), seed=3)
    out = {}
    for engine in ("fused", "graph"):
        _, cl = _cluster({"engine": engine, "lanes": 1, "nslots": 8}, ("sgd", 0.05), batch, params=params)
        with cl:
            w = cl.worker
            assert w.engine == engine
            it = data.BatchIterator(ds, seed=9)
            losses = []
            for _ in range(50):
                x, y = it.next_batch(batch)
                losses.append(w.step(x, y).loss)
                w.wait_applied()
            out[engine] = (losses, w.read_variables())
    lf, lg = out["fused"][0], out["graph"][0]
    worst = max(abs(a - b) / (abs(b) + 1e-9) for a, b in zip(lf, lg))
    perr = max(float((out["fused"][1][k] - out["graph"][1][k]).norm() / (out["graph"][1][k].norm() + 1e-9))
               for k in out["fused"][1])
    print(f"[fused vs graph, batch {batch}] worst per-step loss rel err {worst:.2e}, param rel err {perr:.2e}")
    assert worst < 2e-3
    assert perr < 5e-3


@pytest.mark.parametrize("batch", BATCHES)
def test_strict_native_loop_is_lock_step_with_fp32_torch_at_batch(batch):
    """300 strict steps of the native loop (lanes=1: every pull follows the acknowledgement of the previous push)
    against an un-rounded fp32 PyTorch step on the same `next_batch` sequence; the bounds of
    tests/test_gpu_fused.py::test_long_horizon_loss_and_accuracy_parity_with_fp32_torch for SGD."""
    from bench_tools.gpu_e2e import ref_step
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import OptimizerConfig
    from dist_mnist_b200.utils import data

    steps = 300
    ds = data.synthetic_mnist(8192, seed=5)
    spec = mlp.book_model(100)
    params = mlp.init_params(spec, seed=11)
    opt = OptimizerConfig("sgd", 0.05)
    ref_p = {k: t.clone() for k, t in params.items()}
    ref_m = {k: torch.zeros_like(t) for k, t in params.items()}
    ref_v = {k: torch.zeros_like(t) for k, t in params.items()}
    _, cl = _cluster({"engine": "fused", "lanes": 1, "nslots": 8, "strict_steps": True}, ("sgd", 0.05), batch,
                     params=params)
    with cl:
        w = cl.worker
        assert w.engine == "fused"
        loader = w.make_loader(ds.images, ds.labels, seed=7)
        twin = w.make_loader(ds.images, ds.labels, seed=7, epoch_feed=False)   # same sequence
        outs = []
        for n in (7, 93, 200):
            outs += list(w.run_steps(n, loader, wait_applied=True))
        assert len(outs) == steps and w.read_global_step() == steps
        t, worst = 0, 0.0
        for o in outs:
            x, y = twin.next_batch()
            lref, t = ref_step(spec, ref_p, ref_m, ref_v, t, x, y, opt)
            assert o.global_step == o.seq
            if lref > 1e-6:
                worst = max(worst, abs(o.loss - lref) / abs(lref))
        got = w.read_variables()
    perr = max(float((got[k] - ref_p[k]).norm() / (ref_p[k].norm() + 1e-9)) for k in got)
    print(f"[lock-step, batch {batch}] {steps} steps: worst per-step loss rel err {worst:.2e}, param rel err {perr:.2e}")
    assert worst < 1e-2
    assert perr < 5e-3


def test_eight_lanes_row_split_at_batch_128():
    """lanes=8, row_split over 2 ps tasks (which selects the fused engine), batch 128 (four tiles, a dense ring slot:
    the epoch feed applies)."""
    from dist_mnist_b200.utils import data

    ds = data.synthetic_mnist(4096, seed=6)
    _, cl = _cluster({"sharding": "row_split", "lanes": 8, "nslots": 16}, ("adam", 1e-3), 128, num_ps=2)
    with cl:
        w = cl.worker
        assert w.engine == "fused" and w.fused_lanes == 8
        loader = w.make_loader(ds.images, ds.labels, seed=0)
        assert loader.epoch_feed
        outs = w.run_steps(300, loader, wait_applied=True)
        assert len(outs) == 300 and w.read_global_step() == 300
        assert sorted(int(s) for s in outs.seq) == list(range(1, 301))
        loss = outs.loss
        assert float(loss[-20:].mean()) < 0.5 * float(loss[:20].mean())
        assert w.feed_stats()["direct_chunks"] > 0


def test_stop_at_global_step_and_evaluate_at_batch_100():
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.utils import data

    ds = data.synthetic_mnist(4096, seed=6)
    spec, cl = _cluster({"engine": "fused", "lanes": 4, "nslots": 16}, ("adam", 1e-3), 100)
    with cl:
        w = cl.worker
        assert w.engine == "fused" and w.B_pad == 128
        loader = w.make_loader(ds.images, ds.labels, seed=0)
        assert not loader.epoch_feed                       # 100 rows in a 128-row slot: the row-gather path
        a = w.run_steps(100, loader)
        # StopAtStepHook semantics (DS:101): the native loop stops claiming steps once a step reports the target
        d = w.run_steps(5000, loader, stop_at_global_step=300)
        w.wait_applied()
        gs = w.read_global_step()
        assert 300 <= gs <= 300 + 64 and len(a) + len(d) == gs
        assert max(int(g) for g in d.global_step) >= 300
        assert sorted(int(s) for s in list(a.seq) + list(d.seq)) == list(range(1, gs + 1))
        loss_e, acc_e = w.evaluate(ds.images[:2000], ds.labels[:2000])
        params = w.read_variables()
    logits, _ = mlp.forward_logits(spec, params, ds.images[:2000])
    assert abs(loss_e - float(mlp.loss_from_logits(spec, logits, ds.labels[:2000]))) < 1e-4
    assert abs(acc_e - mlp.accuracy_count(logits, ds.labels[:2000]) / 2000) < 1e-9
    assert acc_e > 0.5
