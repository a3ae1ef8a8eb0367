"""GPU-side distributed correctness on ONE GPU: the reference's documented topology (1 ps + 2 workers,
/root/reference/README.md:7-9) as separate OS processes that share cuda:0 — the ps shard is exported with CUDA IPC,
the workers' kernels push into it and the persistent serve kernel of the ps process applies (the GPU time-slices the
three contexts, so this is slow but exercises exactly the multi-process protocol of a multi-GPU run).

Asserted: the shared step counter equals the number of pushes the workers made (every push applied exactly once),
training converges, the ps exits once the workers are done; with 2 ps tasks; with async-SGD red.add pushes; and the
failure path on the cuda backend: a worker crashes (fault injection), is declared dead after --worker_timeout, is
started again and re-admitted (stop / patch / relaunch of the serve kernel)."""
import re

import _harness
import pytest

pytestmark = pytest.mark.gpu


def _local_steps(out):
    m = re.search(r"local_steps=(\d+)", out)
    assert m, out
    return int(m.group(1))


def _ps_gstep(out):
    m = re.search(r"exiting: global_step=(\d+) owns_global_step=(\d+)", out)
    assert m, out
    return int(m.group(1)), int(m.group(2))


@pytest.mark.timeout(420)
@pytest.mark.parametrize("mode", ["mailbox_adam", "atomic_sgd", "two_ps_row_split"])
def test_one_ps_two_workers_three_processes_one_gpu(mode):
    n_ps = 2 if mode == "two_ps_row_split" else 1
    common = ["--train_steps", "240", "--learning_rate", "0.001", "--log_every", "80", "--lanes", "4"]
    if mode == "atomic_sgd":
        common += ["--optimizer", "sgd", "--push_mode", "atomic", "--learning_rate", "0.05"]
    if mode == "two_ps_row_split":
        common += ["--sharding", "row_split"]
    with _harness.Tasks(backend="cuda", n_ps=n_ps, gpu=0) as t:
        pss = [t.spawn("ps", k, common + ["--ps_exit_when_done"]) for k in range(n_ps)]
        ws = [t.spawn("worker", i, common) for i in range(2)]
        outs_w = [t.finish(w, 300) for w in ws]
        outs_p = [t.finish(p, 90) for p in pss]
    for w, o in zip(ws, outs_w):
        assert w.returncode == 0, o
        assert "engine=fused" in o, o
    for p, o in zip(pss, outs_p):
        assert p.returncode == 0, o
    total = sum(_local_steps(o) for o in outs_w)
    assert total >= 240
    gsteps = [_ps_gstep(o) for o in outs_p]
    owner = [g for g, owns in gsteps if owns]
    if mode != "atomic_sgd" or True:
        # every push of every worker was applied exactly once: the shared counter equals the number of pushes
        assert owner and owner[0] == total, (gsteps, total, outs_w, outs_p)
    logged = [l for o in outs_w for l in o.splitlines() if l.startswith("Train step ")]
    assert logged, outs_w
    losses = [float(l.split("loss: ")[1]) for l in outs_w[0].splitlines() if l.startswith("Train step ")]
    if len(losses) >= 2:
        assert losses[-1] < losses[0]


@pytest.mark.timeout(600)
def test_worker_crash_timeout_and_restart_on_cuda_one_gpu():
    # --chunk_sleep throttles the workers to <= 1000 steps/s each, so the run (40 000 global steps) outlives the
    # crash, the 6 s failure-detection window and the restart whatever the GPU's time-slicing speed is
    common = ["--train_steps", "40000", "--learning_rate", "0.001", "--log_every", "10000", "--lanes", "2",
              "--chunk_sleep", "0.05"]
    with _harness.Tasks(backend="cuda", gpu=0) as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done", "--worker_timeout", "6"])
        w0 = t.spawn("worker", 0, common)
        w1 = t.spawn("worker", 1, common + ["--inject_fault", "40"])
        out1 = t.finish(w1, 240)
        assert w1.returncode == 42 and "[fault injection] worker 1 dies" in out1, out1
        import time
        time.sleep(9)      # > --worker_timeout: the ps declares worker 1 dead (mark_worker_dead on the cuda backend)
        w1b = t.spawn("worker", 1, common)
        out1b = t.finish(w1b, 300)
        out0 = t.finish(w0, 300)
        outp = t.finish(ps, 90)
    assert w1b.returncode == 0, out1b
    assert w0.returncode == 0, out0
    assert ps.returncode == 0, outp
    assert "worker 1 presumed dead" in outp, outp
    assert "worker 1 re-registered (incarnation 2): re-admitting it" in outp, outp
    assert _local_steps(out1b) > 0
