"""Epoch feed of the fused executor on a real H100 (csrc/fused_exec.cu, csrc/loader.h): steps fed as contiguous slices of
the pinned epoch buffer must see exactly the `next_batch` sequence (/root/reference/distributed_server-basic.py:111).
The host-side logic is covered on CPU by tests/test_fexec_emulated.py; this is the same check through the real DMA
engine and the real kernel. (Sorted last on purpose: it is the newest GPU test.)"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_epoch_feed_steps_see_the_next_batch_sequence():
    from bench_tools.gpu_e2e import ref_step
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    ds = data.synthetic_mnist(2048, seed=9)          # 64 steps per epoch
    spec = mlp.book_model(100)
    params = mlp.init_params(spec, seed=3)
    opt = OptimizerConfig("sgd", 0.05)
    cfg = EngineConfig(backend="cuda", lanes=1, nslots=8, strict_steps=True)   # lock-step: comparable step by step
    ref_p = {k: t.clone() for k, t in params.items()}
    ref_m = {k: torch.zeros_like(t) for k, t in params.items()}
    ref_v = {k: torch.zeros_like(t) for k, t in params.items()}
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=1, params=params) as cl:
        w = cl.worker
        fed = w.make_loader(ds.images, ds.labels, seed=7)
        plain = w.make_loader(ds.images, ds.labels, seed=7, epoch_feed=False)   # same sequence, row-gather path
        assert fed.epoch_feed and not plain.epoch_feed
        losses = []
        for n in (5, 20, 50, 16, 109, 200):          # 400 steps = 6.25 epochs, boundaries inside and between runs
            outs = w.run_steps(n, fed, wait_applied=True)
            assert len(outs) == n
            losses += [o.loss for o in outs]
        stats = w.feed_stats()
        assert w.read_global_step() == 400
        t, worst = 0, 0.0
        for i, got in enumerate(losses):
            x, y = plain.next_batch()
            lref, t = ref_step(spec, ref_p, ref_m, ref_v, t, x, y, opt)
            rel = abs(got - lref) / (abs(lref) + 1e-12)
            worst = max(worst, rel)
            assert rel < 2e-2, (i, got, lref)
        assert fed.epochs == plain.epochs == 6
    print(f"[epoch feed] 400 lock-step steps, worst loss rel err vs fp32 reference on the next_batch sequence {worst:.2e}; {stats}")
    # 36 chunks in all; the 6 that contain an epoch boundary are row-gathered, the rest are slices of an epoch buffer
    # (unless a fill could not be posted in time, which only costs speed)
    assert stats["direct_chunks"] > 0 and stats["gathered_chunks"] >= 6 and stats["fills_posted"] >= 3


def test_ps_serve_kernel_ieee_adam_math():
    """`--adam_math ieee` (PsServeParams::ieee_math): the second instantiation of ps_serve_kernel, with correctly
    rounded sqrt / divide like TF's ApplyAdam, against the same PyTorch fp32 reference as the default fast path
    (tests/test_gpu_kernels.py::test_persistent_ps_serve_kernel)."""
    from bench_tools import gpu_check
    assert gpu_check.check_ps_serve(ieee=True)
