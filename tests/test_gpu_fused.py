"""Fused step engine on one H100: long-horizon parity with fp32 PyTorch, agreement with the per-layer graph engine,
checkpoint / resume, lane and strictness switching, StopAtStep semantics of the native loop."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _cluster(cfg_kw=None, opt=("adam", 1e-3), num_ps=1, batch=32, params=None, restore_dir=None, hidden=100):
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster

    spec = mlp.book_model(hidden)
    cfg = EngineConfig(backend="cuda", **(cfg_kw or {}))
    return spec, InProcessCluster(spec, OptimizerConfig(*opt), cfg, batch_size=batch, num_ps=num_ps, params=params,
                                  restore_dir=restore_dir)


@pytest.mark.parametrize("okind,lr,steps", [("sgd", 0.05, 4000), ("adam", 1e-3, 2000)])
def test_long_horizon_loss_and_accuracy_parity_with_fp32_torch(okind, lr, steps):
    """The reference computes in fp32 (DS:41-47, 92-93); the kernels multiply in tf32 with fp32 accumulation. Thousands
    of lock-step optimizer steps on identical batches: the loss curve and the final accuracy must stay on the fp32
    PyTorch trajectory (an *un-rounded* fp32 reference, not a tf32-emulating one)."""
    from bench_tools.gpu_e2e import ref_step
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import OptimizerConfig
    from dist_mnist_b200.utils import data

    ds = data.synthetic_mnist(8192, seed=5)
    spec = mlp.book_model(100)
    params = mlp.init_params(spec, seed=11)
    opt = OptimizerConfig(okind, lr)
    ref_p = {k: t.clone() for k, t in params.items()}
    ref_m = {k: torch.zeros_like(t) for k, t in params.items()}
    ref_v = {k: torch.zeros_like(t) for k, t in params.items()}
    t = 0
    it = data.BatchIterator(ds, seed=2)
    _, cl = _cluster({"lanes": 1, "nslots": 8, "strict_steps": True}, (okind, lr), params=params)
    worst, checks = 0.0, []
    with cl:
        w = cl.worker
        for i in range(steps):
            x, y = it.next_batch(32)
            r = w.step(x, y)
            w.wait_applied()
            lref, t = ref_step(spec, ref_p, ref_m, ref_v, t, x, y, opt)
            rel = abs(r.loss - lref) / (abs(lref) + 1e-12)
            if (i + 1) % 500 == 0:
                checks.append((i + 1, r.loss, lref, rel))
            worst = max(worst, rel) if lref > 1e-6 else worst
        loss_e, acc_e = w.evaluate(ds.images[:4096], ds.labels[:4096])
        got = w.read_variables()
    logits, _ = mlp.forward_logits(spec, ref_p, ds.images[:4096])
    acc_r = mlp.accuracy_count(logits, ds.labels[:4096]) / 4096
    loss_r = float(mlp.loss_from_logits(spec, logits, ds.labels[:4096]))
    perr = max(float((got[k] - ref_p[k]).norm() / (ref_p[k].norm() + 1e-9)) for k in got)
    print(f"[parity {okind}] {steps} steps: worst per-step loss rel err {worst:.2e}; checkpoints {checks}; "
          f"eval loss engine {loss_e:.5f} vs fp32 {loss_r:.5f}; accuracy {acc_e:.4f} vs {acc_r:.4f}; param rel err {perr:.2e}")
    # tf32 MMAs against fp32 PyTorch: the bounds leave room for tf32 rounding accumulated over these horizons
    assert abs(acc_e - acc_r) <= 0.005
    assert abs(loss_e - loss_r) <= 0.02 * abs(loss_r) + 1e-6
    assert worst < 1e-2
    assert perr < (5e-3 if okind == "sgd" else 3e-2)


def test_fused_and_graph_engines_agree():
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.utils import data

    ds = data.synthetic_mnist(2048, seed=1)
    spec = mlp.book_model(100)
    params = mlp.init_params(spec, seed=3)
    out = {}
    for engine in ("fused", "graph"):
        _, cl = _cluster({"engine": engine, "lanes": 1, "nslots": 8}, ("sgd", 0.05), params=params)
        with cl:
            w = cl.worker
            assert w.engine == engine
            it = data.BatchIterator(ds, seed=9)
            losses = []
            for _ in range(50):
                x, y = it.next_batch(32)
                losses.append(w.step(x, y).loss)
                w.wait_applied()
            out[engine] = (losses, w.read_variables(), w.kernels_per_step)
    lf, lg = out["fused"][0], out["graph"][0]
    assert max(abs(a - b) / (abs(b) + 1e-9) for a, b in zip(lf, lg)) < 2e-3
    for k in out["fused"][1]:
        a, b = out["fused"][1][k], out["graph"][1][k]
        assert float((a - b).norm() / (b.norm() + 1e-9)) < 5e-3, k
    assert out["fused"][2] == 1 and out["graph"][2] == 3


def test_checkpoint_resume_row_split_two_ps(tmp_path):
    from dist_mnist_b200.utils import ckpt, data

    ds = data.synthetic_mnist(2048, seed=4)
    _, cl = _cluster({"sharding": "row_split", "lanes": 4, "nslots": 16}, num_ps=2)
    with cl:
        w = cl.worker
        loader = w.make_loader(ds.images, ds.labels, seed=0)
        outs = w.run_steps(300, loader)
        assert len(outs) == 300
        path = ckpt.save_checkpoint(w, str(tmp_path))
        saved = w.read_variables()
        gs = w.read_global_step()
        assert gs == 300
    _, cl2 = _cluster({"sharding": "row_split", "lanes": 4, "nslots": 16}, num_ps=2, restore_dir=str(tmp_path))
    with cl2:
        w = cl2.worker
        assert w.read_global_step() == 300
        got = w.read_variables()
        for k in saved:
            assert torch.equal(saved[k], got[k]), k
        loader = w.make_loader(ds.images, ds.labels, seed=1)
        outs = w.run_steps(100, loader)
        w.wait_applied()
        assert w.read_global_step() == 400 and outs[-1].loss < 0.1
    assert path.endswith("model.ckpt-300.pt")


def test_set_lanes_strict_and_stop_at_global_step():
    from dist_mnist_b200.utils import data

    ds = data.synthetic_mnist(4096, seed=6)
    _, cl = _cluster({"lanes": 8, "nslots": 32})
    with cl:
        w = cl.worker
        loader = w.make_loader(ds.images, ds.labels, seed=0)
        a = w.run_steps(200, loader)
        w.set_lanes(1, strict=True)
        b = w.run_steps(100, loader)
        w.set_lanes(4, strict=False)
        c = w.run_steps(100, loader)
        w.wait_applied()
        assert w.read_global_step() == 400
        seqs = sorted(o.seq for o in list(a) + list(b) + list(c))
        assert seqs == list(range(1, 401))
        # strict lanes=1: every step saw all previous pushes applied -> global_step reported == its own seq
        assert [o.global_step for o in b] == [o.seq for o in b]
        # StopAtStepHook semantics (DS:101): the native loop stops claiming steps once a step reports the target
        d = w.run_steps(5000, loader, stop_at_global_step=1000)
        w.wait_applied()
        gs = w.read_global_step()
        assert 1000 <= gs <= 1000 + 64 and len(d) == gs - 400
        assert max(o.global_step for o in d) >= 1000
