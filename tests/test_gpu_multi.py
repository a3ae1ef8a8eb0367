"""Multi-GPU tests (need >= 2 H100s on one machine; skipped otherwise): separate OS processes exchange CUDA IPC
handles through the rendezvous and train over NVLink peer memory."""
import json
import os
import socket
import subprocess
import sys
import time

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "distributed_server-basic.py")


def _need_gpus(n):
    if not torch.cuda.is_available() or torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs")


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _spawn(job, idx, ps_hosts, worker_hosts, extra=()):
    cmd = [sys.executable, SCRIPT, "--job_name", job, "--task_index", str(idx), "--ps_hosts", ps_hosts,
           "--worker_hosts", worker_hosts, "--backend", "cuda", *extra]
    env = dict(os.environ, PYTHONPATH=ROOT, PYTHONUNBUFFERED="1")
    return subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, cwd=ROOT)


@pytest.mark.parametrize("extra", [[], ["--optimizer", "sgd", "--push_mode", "atomic", "--learning_rate", "0.05"]])
def test_cli_one_ps_one_worker_two_gpus(extra):
    _need_gpus(2)
    ps_hosts, worker_hosts = f"127.0.0.1:{_free_port()}", f"127.0.0.1:{_free_port()}"
    common = ["--train_steps", "400", "--learning_rate", "0.001", *extra]
    ps = _spawn("ps", 0, ps_hosts, worker_hosts, common + ["--ps_exit_when_done"])
    w0 = _spawn("worker", 0, ps_hosts, worker_hosts, common)
    out0, _ = w0.communicate(timeout=240)
    outp, _ = ps.communicate(timeout=60)
    assert w0.returncode == 0, out0
    assert ps.returncode == 0, outp
    logged = [l for l in out0.splitlines() if l.startswith("Train step ")]
    assert [int(l.split(",")[0].split()[-1]) for l in logged] == [100, 200, 300, 400], out0
    losses = [float(l.split("loss: ")[1]) for l in logged]
    assert losses[-1] < losses[0]


def test_bench_two_gpus_contract():
    _need_gpus(2)
    port = _free_port()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "bench.py"), "--gpus", "2", "--steps", "300",
           "--warmup", "10"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    line = [l for l in r.stdout.splitlines() if l.startswith("{")][-1]
    d = json.loads(line)
    assert d["n_gpus"] == 2 and d["value"] > 0 and d["e2e"]["value"] > 0
    # fused engine: one persistent kernel launch runs all 300 steps (the acknowledgement wait is its tail)
    assert d["gpu_launches"] >= 1 and d["gpu_launches"] * d["steps_per_launch"] >= 300
    assert d["config"]["global_step_after_run"] >= 300 and d["config"]["engine"] == "fused"
    assert d["parity"]["value_device_timed"] > 0


def _local_steps(out):
    import re
    m = re.search(r"local_steps=(\d+)", out)
    assert m, out
    return int(m.group(1))


@pytest.mark.parametrize("n_ps,extra", [(1, []), (2, ["--sharding", "row_split"])])
def test_documented_topology_one_process_per_gpu(n_ps, extra):
    """The reference's README topology (1 ps + 2 workers, /root/reference/README.md:7-9) with every task on its own
    GPU (3 GPUs; 4 with two row-split ps shards): the shared step counter equals the number of pushes."""
    import re
    _need_gpus(n_ps + 2)
    ps_hosts = ",".join(f"127.0.0.1:{_free_port()}" for _ in range(n_ps))
    worker_hosts = f"127.0.0.1:{_free_port()},127.0.0.1:{_free_port()}"
    common = ["--train_steps", "2000", "--learning_rate", "0.001", "--log_every", "500", *extra]
    pss = [_spawn("ps", k, ps_hosts, worker_hosts, common + ["--ps_exit_when_done"]) for k in range(n_ps)]
    ws = [_spawn("worker", i, ps_hosts, worker_hosts, common) for i in range(2)]
    outs_w = [w.communicate(timeout=300)[0] for w in ws]
    outs_p = [p.communicate(timeout=90)[0] for p in pss]
    for w, o in zip(ws, outs_w):
        assert w.returncode == 0 and "engine=fused" in o, o
    for p, o in zip(pss, outs_p):
        assert p.returncode == 0, o
    total = sum(_local_steps(o) for o in outs_w)
    owner = [int(m.group(1)) for o in outs_p for m in [re.search(r"global_step=(\d+) owns_global_step=1", o)] if m]
    assert owner and owner[0] == total >= 2000, (owner, total, outs_p)


def test_nvls_multicast_publish_and_in_switch_reduce():
    """NVSwitch multicast over every visible GPU of this process (csrc/nvls_sm90.cu): `multimem.st` publish lands bit
    for bit in every replica, `multimem.ld_reduce` returns the exact sum over the replicas. Run in a fresh process
    (the probe creates VMM mappings and enables peer access itself)."""
    _need_gpus(2)
    n = min(torch.cuda.device_count(), 8)
    code = ("from dist_mnist_b200 import _native as N\n"
            f"ok, log = N.nvls_probe({n}, 318032, 20)\n"
            "print(log)\n"
            "raise SystemExit(0 if ok else 1)\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT), timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "PROBE OK" in r.stdout, (r.stdout[-3000:], r.stderr[-2000:])
    assert "0 of 79508 floats differ" in r.stdout
