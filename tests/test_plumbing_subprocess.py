"""The README recipe of the reference (1 ps + 2 workers as separate OS processes on 127.0.0.1 ports) on the CPU
backend: real processes, TCP rendezvous, POSIX-shm peer memory. BASELINE.json config 1 / SURVEY §4 item 2."""
import os
import subprocess
import sys
import time

import _harness
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "distributed_server-basic.py")


@pytest.mark.timeout(180)
def test_one_ps_two_workers_processes():
    common = ["--train_steps", "300", "--learning_rate", "0.001"]
    with _harness.Tasks() as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done"])
        time.sleep(0.5)
        w1 = t.spawn("worker", 1, common)      # non-chief first: must wait for the chief's init
        time.sleep(0.5)
        w0 = t.spawn("worker", 0, common)
        out0, out1 = t.finish(w0, 120), t.finish(w1, 120)
        outp = t.finish(ps, 60)
    assert w0.returncode == 0, out0
    assert w1.returncode == 0, out1
    assert ps.returncode == 0, outp
    assert out0.splitlines()[:2] == ["job name : worker", "task index : 0"]
    assert outp.splitlines()[:2] == ["job name : ps", "task index : 0"]
    logged = [l for l in (out0 + out1).splitlines() if l.startswith("Train step ")]
    assert logged, (out0, out1)
    steps = sorted({int(l.split(",")[0].split()[-1]) for l in logged})
    assert all(s % 100 == 0 for s in steps)
    losses = [float(l.split("loss: ")[1]) for l in logged]
    assert min(losses) < 0.05


@pytest.mark.timeout(120)
def test_ps_blocks_forever_like_server_join():
    """Reference ps never exits (server.join(), DS:83): without --ps_exit_when_done it must still be alive after
    the only worker has finished."""
    with _harness.Tasks(n_workers=1) as t:
        ps = t.spawn("ps", 0, ["--train_steps", "40"])
        w0 = t.spawn("worker", 0, ["--train_steps", "40", "--log_every", "20"])
        out0 = t.finish(w0, 90)
        assert w0.returncode == 0, out0
        assert "Train step 20, loss:" in out0 and "Train step 40, loss:" in out0
        time.sleep(1.0)
        assert ps.poll() is None, "ps task exited although the reference's ps blocks forever"


def test_bad_invocations():
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, SCRIPT, "--task_index", "0", "--ps_hosts", "a:1", "--worker_hosts", "a:2"],
                       capture_output=True, text=True, env=env)
    assert r.returncode != 0 and "Must specify the job name explicitly" in r.stderr
    r = subprocess.run([sys.executable, SCRIPT, "--job_name", "worker", "--ps_hosts", "a:1", "--worker_hosts", "a:2"],
                       capture_output=True, text=True, env=env)
    assert r.returncode != 0 and "Must specify a valid task index" in r.stderr
    assert "job name : worker" in r.stdout


@pytest.mark.timeout(240)
def test_worker_crash_is_detected_and_training_continues():
    """Failure detection (SURVEY §5): worker 1 crashes mid-run (fault injection); the ps declares it dead after
    `--worker_timeout` seconds without a heartbeat, worker 0 trains on to the target global step, and the ps
    (asked to exit when done) does not wait for the dead worker forever."""
    common = ["--train_steps", "600", "--learning_rate", "0.001"]
    with _harness.Tasks() as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done", "--worker_timeout", "3"])
        w0 = t.spawn("worker", 0, common)
        w1 = t.spawn("worker", 1, common + ["--inject_fault", "50"])
        out1 = t.finish(w1, 120)
        assert w1.returncode == 42 and "[fault injection] worker 1 dies" in out1, out1
        out0 = t.finish(w0, 150)
        assert w0.returncode == 0, out0
        assert "Train step 600, loss:" in out0 or "Train step 500, loss:" in out0, out0
        outp = t.finish(ps, 60)
    assert ps.returncode == 0, outp
    assert "worker 1 presumed dead" in outp, outp


@pytest.mark.timeout(300)
def test_crashed_worker_can_be_restarted_and_rejoins():
    """Elastic recovery (the reference's `_RecoverableSession`, SURVEY §3.4 / §5): worker 1 crashes, is started
    again with the same task index, the ps re-admits it (new incarnation: fresh push sequence and inbox) and it
    trains on with worker 0 until the shared global step reaches the target."""
    common = ["--train_steps", "2500", "--learning_rate", "0.001", "--log_every", "500"]
    with _harness.Tasks() as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done", "--worker_timeout", "30"])
        w0 = t.spawn("worker", 0, common)
        w1 = t.spawn("worker", 1, common + ["--inject_fault", "30"])
        out1 = t.finish(w1, 120)
        assert w1.returncode == 42, out1
        w1b = t.spawn("worker", 1, common + ["--metrics_file", os.devnull, "--log_steps_per_sec"])
        out1b = t.finish(w1b, 200)
        out0 = t.finish(w0, 200)
        outp = t.finish(ps, 60)
    assert w1b.returncode == 0, out1b
    assert w0.returncode == 0, out0
    assert ps.returncode == 0, outp
    assert "worker 1 re-registered (incarnation 2): re-admitting it" in outp, outp
    # the restarted worker really trained: it reported steps of its own
    assert "INFO global_step/sec" in out1b, out1b
    assert "Train step 2500, loss:" in (out0 + out1b) or "Train step 2000, loss:" in (out0 + out1b)


@pytest.mark.timeout(300)
def test_restarted_chief_does_not_reinitialize_live_variables():
    """Round-1 advisor finding: a restarted chief (worker 0) used to run the initialisers again on the live ps shards
    (parameters and Adam slots reset while global_step and the per-item step counts kept running, loss jumped from
    ~4e-5 to 0.08). It must see that the variables are live and simply rejoin."""
    common = ["--train_steps", "4000", "--learning_rate", "0.001", "--log_every", "100", "--chunk_sleep", "0.1"]
    with _harness.Tasks() as t:
        ps = t.spawn("ps", 0, common + ["--ps_exit_when_done"])
        w0 = t.spawn("worker", 0, common + ["--inject_fault", "200"])
        w1 = t.spawn("worker", 1, common)
        out0 = t.finish(w0, 120)
        assert w0.returncode == 42, out0
        w0b = t.spawn("worker", 0, common + ["--metrics_file", os.devnull, "--log_steps_per_sec"])
        out0b = t.finish(w0b, 240)
        out1 = t.finish(w1, 240)
        outp = t.finish(ps, 60)
    assert w0b.returncode == 0, out0b
    assert w1.returncode == 0, out1
    assert ps.returncode == 0, outp
    assert "variables are live on the ps, not re-initialising" in out0b, out0b
    # training continued from the live state: whatever the restarted chief logged is far below the fresh-init loss
    # (~0.23) — after a re-initialisation its first logged losses would be back up there
    losses = [float(l.split("loss: ")[1]) for l in out0b.splitlines() if l.startswith("Train step ")]
    assert all(v < 0.02 for v in losses), out0b
    assert "done: local_steps=" in out0b and "done: local_steps=" in out1


def test_more_ps_tasks_than_variables_global_step_and_exit():
    """Round-1 advisor finding: with 5 ps tasks round-robin placement leaves ps 0 with `global_step` only (no variable,
    no item); its counter is never incremented and it never saw `worker_done`. The counter of the first shard that
    owns items is authoritative, every shard hears `worker_done`, and an item-less shard exits with the others."""
    import torch  # noqa: F401
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data

    ds = data.synthetic_mnist(512, seed=0)
    spec = mlp.book_model(100)
    cfg = EngineConfig(backend="cpu", nslots=4)
    with InProcessCluster(spec, OptimizerConfig("adam", 1e-3), cfg, batch_size=32, num_ps=5) as cl:
        w = cl.worker
        assert cl.ps[0].shard.n_items == 0 and w.gs_owner != 0
        for i in range(7):
            out = w.step(ds.images[32 * i:32 * i + 32], ds.labels[32 * i:32 * i + 32])
        w.wait_applied()
        assert out.global_step == 7 and w.read_global_step() == 7
        w.finish()
        t0 = time.time()
        while any(p.kernel_running() for p in cl.ps):
            assert time.time() - t0 < 20, "a ps shard (the item-less one?) did not exit after every worker was done"
            time.sleep(0.01)


@pytest.mark.timeout(180)
def test_two_ps_row_split_two_workers_processes():
    """`--ps_hosts` is a list in the reference (DS:73-77); with `--sharding row_split` the hidden weight itself is
    split over both ps processes, so every push of every worker goes to two shards. The exit lines give the counters:
    the shard that owns the step counter must have seen exactly the sum of the workers' steps."""
    common = ["--train_steps", "240", "--learning_rate", "0.001", "--sharding", "row_split"]
    with _harness.Tasks(n_ps=2) as t:
        ps0 = t.spawn("ps", 0, common + ["--ps_exit_when_done"])
        ps1 = t.spawn("ps", 1, common + ["--ps_exit_when_done"])
        time.sleep(0.5)
        w1 = t.spawn("worker", 1, common)
        w0 = t.spawn("worker", 0, common)
        out0, out1 = t.finish(w0, 120), t.finish(w1, 120)
        outp0, outp1 = t.finish(ps0, 60), t.finish(ps1, 60)
    for p, o in ((w0, out0), (w1, out1), (ps0, outp0), (ps1, outp1)):
        assert p.returncode == 0, o
    done = [int(l.split("local_steps=")[1].split()[0].rstrip(",")) for l in (out0 + out1).splitlines() if "local_steps=" in l]
    assert len(done) == 2 and sum(done) >= 240
    gsteps = [int(l.split("global_step=")[1].split()[0].rstrip(",")) for l in (outp0 + outp1).splitlines()
              if "exiting: global_step=" in l]
    assert gsteps and max(gsteps) == sum(done), (gsteps, done)
