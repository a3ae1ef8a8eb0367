"""Moving averages of the variables on the GPU parameter server: the averaging serve-kernel instantiations alone against
fp64, the fused engine in lock-step with fp32 PyTorch plus an fp32 shadow reference, pipelined runs on the graph
engine and with row_split sharding that end with every item at the global step and evaluate the shadows, and a
1 ps + 2 worker multi-process run on one GPU whose checkpoint holds the shadows."""
import re
import tempfile

import _harness
import pytest

pytestmark = pytest.mark.gpu


def _rules():
    """Every family of serve kernels in both math modes (Momentum has one instantiation: plain and Nesterov)."""
    from dist_mnist_b200.parallel.config import OptimizerConfig
    return [OptimizerConfig("adam", 1e-2), OptimizerConfig("adam", 1e-2, math="ieee"), OptimizerConfig("sgd", 5e-2),
            OptimizerConfig("momentum", 1e-2), OptimizerConfig("momentum", 1e-2, use_nesterov=True),
            OptimizerConfig("adagrad", 5e-2), OptimizerConfig("adagrad", 5e-2, math="ieee"),
            OptimizerConfig("rmsprop", 1e-3, momentum=0.9), OptimizerConfig("rmsprop", 1e-3, math="ieee")]


# (schedule, starting step): warm-up from 0, where the decay changes at every push, and just below 2^24, where it is
# the bound; the schedule crosses a staircase boundary at 2^24 inside the pass
def _starts():
    from dist_mnist_b200.parallel.config import LrSchedule
    sched = LrSchedule("exponential_decay", decay_steps=1 << 20, decay_rate=0.96875, staircase=True)
    return {"const-0": (None, 0), "const-2p24": (None, (1 << 24) - 4),
            "sched-0": (LrSchedule("exponential_decay", decay_steps=4, decay_rate=0.75), 0),
            "sched-2p24": (sched, (1 << 24) - 4)}


@pytest.mark.parametrize("start", list(_starts()))
def test_averaging_serve_kernels_match_fp64(start):
    """Every family and math mode, per push and merged, default and register-resident geometry: parameters, slots and
    shadows within 1e-5 of fp64; bf16 shadow, global_step, acks and the final step count exact."""
    import dataclasses

    from bench_tools import gpu_check
    from dist_mnist_b200 import _native as N
    from dist_mnist_b200.parallel.config import LrSchedule

    schedule, s0 = _starts()[start]
    ok = True
    for base in _rules():
        opt = dataclasses.replace(base, schedule=schedule or LrSchedule(), moving_average_decay=0.99)
        for mode in (N.APPLY_PER_PUSH, N.APPLY_MERGED):
            for resident in (False, True):
                ok &= gpu_check.check_ps_serve_tf1(opt, mode, resident=resident, sched_step=s0)
    assert ok


def test_averaging_serve_kernels_without_num_updates():
    import dataclasses

    from bench_tools import gpu_check
    from dist_mnist_b200 import _native as N

    ok = True
    for base in _rules()[:4]:
        opt = dataclasses.replace(base, moving_average_decay=0.9, moving_average_num_updates=False)
        for mode in (N.APPLY_PER_PUSH, N.APPLY_MERGED):
            ok &= gpu_check.check_ps_serve_tf1(opt, mode, resident=mode == N.APPLY_MERGED, sched_step=7)
    assert ok


def test_check_ps_serve_takes_an_averaging_config():
    from bench_tools import gpu_check
    from dist_mnist_b200.parallel.config import LrSchedule

    assert gpu_check.check_ps_serve(moving_average_decay=0.99)
    assert gpu_check.check_ps_serve(ieee=True, schedule=LrSchedule("cosine_decay", decay_steps=7), sched_step=3,
                                    moving_average_decay=0.999)


@pytest.mark.parametrize("rule", ["sgd", "momentum"])
def test_strict_fused_native_loop_with_moving_averages_is_lock_step_with_fp32_torch(rule):
    """300 strict steps (lanes=1): step i is followed by the shadow update with ema_decay_at(i + 1). Bounds of
    tests/test_gpu_lr_schedules.py::test_strict_fused_native_loop_under_a_schedule_is_lock_step_with_fp32_torch, the
    parameter bound also for the shadows."""
    from bench_tools.gpu_e2e import ref_ema, ref_slots, ref_step
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    opt = OptimizerConfig(rule, 5e-2 if rule == "sgd" else 1e-2, moving_average_decay=0.99)
    ds = data.synthetic_mnist(8192, seed=5)
    spec = mlp.book_model(100)
    params = mlp.init_params(spec, seed=11)
    ref_p = {k: t.clone() for k, t in params.items()}
    ref_e = {k: t.clone() for k, t in params.items()}
    ref_m, ref_v = ref_slots(opt, params)
    cfg = EngineConfig(backend="cuda", engine="fused", lanes=1, nslots=8, strict_steps=True)
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=1, params=params) as cl:
        w = cl.worker
        assert w.engine == "fused"
        loader = w.make_loader(ds.images, ds.labels, seed=7)
        twin = w.make_loader(ds.images, ds.labels, seed=7, epoch_feed=False)
        outs = []
        for n in (7, 93, 200):
            outs += list(w.run_steps(n, loader, wait_applied=True))
        assert len(outs) == 300 and w.read_global_step() == 300
        assert set(w.read_sched_steps(0)) == {300}
        t, worst = 0, 0.0
        for i, o in enumerate(outs):
            x, y = twin.next_batch()
            lref, t = ref_step(spec, ref_p, ref_m, ref_v, t, x, y, opt)
            ref_ema(opt, ref_p, ref_e, i + 1)
            assert o.global_step == o.seq
            if lref > 1e-6:
                worst = max(worst, abs(o.loss - lref) / abs(lref))
        got, got_e = w.read_variables(), w.read_variables("ema")
    perr = max(float((got[k] - ref_p[k]).norm() / (ref_p[k].norm() + 1e-9)) for k in got)
    eerr = max(float((got_e[k] - ref_e[k]).norm() / (ref_e[k].norm() + 1e-9)) for k in got_e)
    # how far the shadows moved from the initial values, relative (all variables together)
    moved = (sum(float((ref_e[k] - params[k]).norm()) ** 2 for k in ref_e)
             / sum(float(ref_e[k].norm()) ** 2 for k in ref_e)) ** 0.5
    print(f"[lock-step {rule} ema] 300 steps: worst per-step loss rel err {worst:.2e}, param rel err {perr:.2e}, "
          f"shadow rel err {eerr:.2e} (shadows moved {moved:.2e})")
    assert worst < 1e-2
    assert perr < 5e-3
    assert eerr < 5e-3
    assert moved > 2 * eerr


@pytest.mark.parametrize("layout", ["graph", "row_split"])
def test_eight_lanes_over_two_ps_with_moving_averages(layout):
    import torch

    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    if layout == "graph":
        opt = OptimizerConfig("rmsprop", 1e-3, momentum=0.9, moving_average_decay=0.99)
        kw = {"engine": "graph"}
    else:
        opt = OptimizerConfig("momentum", 1e-2, use_nesterov=True, moving_average_decay=0.99)
        kw = {"sharding": "row_split"}
    cfg = EngineConfig(backend="cuda", lanes=8, nslots=16, **kw)
    ds = data.synthetic_mnist(8192, seed=6)
    spec = mlp.book_model(100)
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=2) as cl:
        w = cl.worker
        assert w.engine == ("graph" if layout == "graph" else "fused")
        loader = w.make_loader(ds.images, ds.labels, seed=0)
        outs = list(w.run_steps(300, loader, wait_applied=True)) + list(w.run_steps(97, loader, wait_applied=True))
        assert len(outs) == 397 and w.read_global_step() == 397
        for k in range(2):
            assert set(w.read_sched_steps(k)) == {397}, k
        params, shadows = w.read_variables(), w.read_variables("ema")
        for k in shadows:
            assert torch.isfinite(shadows[k]).all(), k
            assert not torch.equal(shadows[k], params[k]), k
        images, labels = ds.images[:1024], ds.labels[:1024]
        loss, acc = w.evaluate(images, labels, moving_averages=True)
        loss_p, acc_p = w.evaluate(images, labels)
    logits, _ = mlp.forward_logits(spec, shadows, images.float())
    assert loss == pytest.approx(float(mlp.loss_from_logits(spec, logits, labels.float())), rel=1e-5)
    assert acc == mlp.accuracy_count(logits, labels) / 1024
    print(f"[{layout} ema] eval loss {loss:.4f} acc {acc:.3f}; parameters: loss {loss_p:.4f} acc {acc_p:.3f}")


@pytest.mark.timeout(420)
def test_moving_averages_one_ps_two_workers_three_processes_one_gpu():
    """As tests/test_gpu_lr_schedules.py::test_cosine_decay_one_ps_two_workers_three_processes_one_gpu, with
    --moving_average_decay: the chief's checkpoint holds finite shadows that differ from the parameters."""
    import torch

    from dist_mnist_b200.utils import ckpt

    d = tempfile.mkdtemp()
    common = ["--train_steps", "240", "--learning_rate", "0.01", "--log_every", "80", "--lanes", "4",
              "--optimizer", "momentum", "--moving_average_decay", "0.99"]
    with _harness.Tasks(backend="cuda", gpu=0) as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done"])
        ws = [t.spawn("worker", i, common + ["--checkpoint_dir", d]) for i in range(2)]
        outs_w = [t.finish(w, 300) for w in ws]
        out_p = t.finish(ps, 90)
    for w, o in zip(ws, outs_w):
        assert w.returncode == 0, o
        assert "engine=fused" in o, o
    assert ps.returncode == 0, out_p
    total = sum(int(re.search(r"local_steps=(\d+)", o).group(1)) for o in outs_w)
    assert total >= 240
    m = re.search(r"exiting: global_step=(\d+) owns_global_step=1", out_p)
    assert m and int(m.group(1)) == total, (out_p, total)
    params, shadows = ckpt.load_variables(d), ckpt.load_variables(d, moving_averages=True)
    assert set(shadows) == set(params)
    for k in params:
        assert torch.isfinite(shadows[k]).all(), k
        assert not torch.equal(shadows[k], params[k]), k
