"""Batches of 33..256 rows on the fused step engine, on CPU: engine selection, the fused tiling's protocol at batch 100
on the cpu backend, and the fused executor's ring geometry for batches that are not one 32-row tile (the executor runs
on the emulated CUDA runtime of tests/native/fake_cuda with tests/native/fexec_emulated_batches.cpp, built with
AddressSanitizer + UBSan)."""
import os
import shutil
import subprocess

import pytest
import torch

from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel import sharding
from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dist_mnist_b200", "csrc")


@pytest.mark.parametrize("batch", [33, 64, 100, 128, 200, 256])
def test_fused_engine_runs_batches_up_to_256_rows(batch):
    spec = mlp.book_model(100)
    assert sharding.fused_eligible(spec, batch)
    assert EngineConfig(engine="fused").resolve_engine(spec, batch) == "fused"
    assert EngineConfig(engine="graph").resolve_engine(spec, batch) == "graph"
    # auto keeps the graph engine above one row tile (host-fed training is not faster on the fused engine there, see
    # sharding.FUSED_AUTO_MAX_BATCH) unless row_split needs the fused tiling
    assert EngineConfig().resolve_engine(spec, batch) == "graph"
    assert EngineConfig(sharding="row_split").resolve_engine(spec, batch) == "fused"


def test_fused_batch_limit_and_row_split():
    spec = mlp.book_model(100)
    assert sharding.FUSED_MAX_BATCH == 256 and sharding.FUSED_AUTO_MAX_BATCH == 32
    assert EngineConfig().resolve_engine(spec, 32) == "fused"
    assert not sharding.fused_eligible(spec, 257)
    with pytest.raises(ValueError, match="batch <= 256"):
        EngineConfig(engine="fused").resolve_engine(spec, 257)
    lay = sharding.build_layout(spec, 2, "row_split", engine="fused")
    assert {sl.ps for sl in lay.fused_slices} == {0, 1}
    with pytest.raises(ValueError, match="row_split"):
        EngineConfig(sharding="row_split").resolve_engine(spec, 257)


def test_row_split_two_ps_at_batch_100_is_lock_step_with_the_fp32_reference():
    """cpu backend, fused tiling (`row_split` over 2 ps tasks), batch 100: every strict step matches an fp32 PyTorch
    step on the same `next_batch` sequence, and global_step counts the pushes."""
    from bench_tools.gpu_e2e import ref_step
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    ds = data.synthetic_mnist(1000, seed=9)            # 10 steps per epoch
    spec = mlp.book_model(100)
    params = mlp.init_params(spec, seed=3)
    opt = OptimizerConfig("adam", 1e-3)
    cfg = EngineConfig(backend="cpu", lanes=1, nslots=4, strict_steps=True, sharding="row_split")
    ref_p = {k: t.clone() for k, t in params.items()}
    ref_m = {k: torch.zeros_like(t) for k, t in params.items()}
    ref_v = {k: torch.zeros_like(t) for k, t in params.items()}
    with InProcessCluster(spec, opt, cfg, batch_size=100, num_ps=2, params=params) as cl:
        w = cl.worker
        assert w.engine == "fused" and w.B_pad == 128
        assert all(s.n_items > 0 for s in w.layout.shards)
        loader = w.make_loader(ds.images, ds.labels, seed=7)
        twin = w.make_loader(ds.images, ds.labels, seed=7)
        t = 0
        outs = list(w.run_steps(25, loader))
        assert len(outs) == 25
        for o in outs:
            x, y = twin.next_batch()
            assert x.shape[0] == 100
            lref, t = ref_step(spec, ref_p, ref_m, ref_v, t, x, y, opt)
            assert abs(o.loss - lref) <= 2e-4 * abs(lref), (o.seq, o.loss, lref)
            assert o.global_step == o.seq
        assert w.read_global_step() == 25
        got = w.read_variables()
        loss_e, acc_e = w.evaluate(ds.images[:500], ds.labels[:500])
    for k in got:
        assert float((got[k] - ref_p[k]).norm() / (ref_p[k].norm() + 1e-12)) < 1e-3, k
    logits, _ = mlp.forward_logits(spec, ref_p, ds.images[:500])
    assert abs(loss_e - float(mlp.loss_from_logits(spec, logits, ds.labels[:500]))) < 1e-4
    assert abs(acc_e - mlp.accuracy_count(logits, ds.labels[:500]) / 500) < 1e-9


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(cuda_inc, "cuda.h")):
        pytest.skip("no cuda.h (CUtensorMap type)")
    exe = str(tmp_path_factory.mktemp("fexec_batches") / "fexec_emulated_batches")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
           "-x", "c++", "-I", os.path.join(ROOT, "tests", "native", "fake_cuda"), "-I", CSRC, "-I", cuda_inc,
           os.path.join(ROOT, "tests", "native", "fexec_emulated_batches.cpp"), os.path.join(CSRC, "fused_exec.cu"),
           os.path.join(CSRC, "loader_api.cpp"), "-o", exe, "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return exe


def _run(exe, n, feed, steps, batch, delay_us=50, threads=3):
    env = dict(os.environ, FAKE_CUDA_DELAY_US=str(delay_us), DM_GATHER_THREADS=str(threads),
               ASAN_OPTIONS="detect_leaks=1")
    r = subprocess.run([exe, str(n), str(feed), str(steps), str(batch)], capture_output=True, text=True, env=env,
                       timeout=600)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])
    line = r.stdout.strip().splitlines()[-1]
    assert line.startswith("OK"), line
    return dict(kv.split("=") for kv in line.split()[1:])


def test_batch_100_gather_path_feeds_every_step_its_batch(harness):
    # 100 rows in a 128-row slot: never a dense slice of the epoch buffer, so every chunk is gathered
    s = _run(harness, 3000, 1, 600, 100)
    assert int(s["direct_chunks"]) == 0 and int(s["gathered_chunks"]) > 0 and int(s["epochs"]) >= 19


def test_batch_128_epoch_feed_feeds_every_step_its_batch(harness):
    s = _run(harness, 4096 + 17, 1, 600, 128)
    assert int(s["direct_chunks"]) > 0 and int(s["gathered_chunks"]) > 0 and int(s["epochs"]) >= 18


@pytest.mark.parametrize("batch", [1, 33, 256])
def test_batch_edges_on_the_gather_path(harness, batch):
    s = _run(harness, 3000, 0, 300, batch, delay_us=20)
    assert int(s["direct_chunks"]) == 0 and int(s["gathered_chunks"]) > 0
