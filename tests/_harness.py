"""What the test files share: the tasks of a CLI cluster as OS processes, the in-process GPU push check against the fp64
step, and the lock-step drivers of the GPU engines and of the cpu-backend optimizers. Test modules import it as
`import _harness` (pytest puts tests/ on sys.path; the leading underscore keeps it from being collected)."""
import os
import subprocess
import sys

import pytest
import torch

from bench_tools import fused_push_ref as R
from bench_tools.gpu_e2e import ref_ema, ref_slots, ref_step
from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.config import EngineConfig, GradClip, L2Regularization, OptimizerConfig
from dist_mnist_b200.session import InProcessCluster, free_port
from dist_mnist_b200.utils import data

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "distributed_server-basic.py")


# ---------------------------------------------------------------------------------------------------------------
# CLI tasks as OS processes
# ---------------------------------------------------------------------------------------------------------------
class Tasks:
    """The ps and worker tasks of one CLI cluster on 127.0.0.1 ports. Every task it started that is still running when
    the `with` block exits, by an assertion, a timeout or a normal return, is killed and reaped, so that no ps (and on
    the cuda backend no persistent serve kernel) outlives the test."""

    def __init__(self, backend="cpu", n_ps=1, n_workers=2, gpu=None):
        self.ps_hosts = ",".join(f"127.0.0.1:{free_port()}" for _ in range(n_ps))
        self.worker_hosts = ",".join(f"127.0.0.1:{free_port()}" for _ in range(n_workers))
        self.backend = ["--backend", backend] + ([] if gpu is None else ["--gpu", str(gpu)])
        self.procs = []

    def spawn(self, job, idx, extra=()):
        cmd = [sys.executable, SCRIPT, "--job_name", job, "--task_index", str(idx), "--ps_hosts", self.ps_hosts,
               "--worker_hosts", self.worker_hosts, *self.backend, *extra]
        env = dict(os.environ, PYTHONPATH=ROOT, PYTHONUNBUFFERED="1")
        p = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, cwd=ROOT)
        self.procs.append(p)
        return p

    @staticmethod
    def finish(p, timeout):
        """The task's output once it has exited; a task still running after `timeout` seconds is killed and fails
        the test with its output so far."""
        try:
            out, _ = p.communicate(timeout=timeout)
        except subprocess.TimeoutExpired:
            p.kill()
            out, _ = p.communicate()
            pytest.fail(f"process timed out; output so far:\n{out}")
        return out

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        for p in self.procs:
            if p.poll() is None:
                p.kill()
                p.communicate()
        return False


# ---------------------------------------------------------------------------------------------------------------
# one GPU step's push against the fp64 step (bench_tools/fused_push_ref)
# ---------------------------------------------------------------------------------------------------------------
def cluster(case, nps=1, sharding="round_robin", engine="fused", lanes=1, nslots=4, strict=True,
            push_mode="mailbox", lr=0.0, clip=None, l2=None):
    """An in-process cuda cluster on the case's model and variables, SGD at `lr` (0 keeps the variables)."""
    kw = {"strict_steps": strict} if engine == "fused" else {}
    cfg = EngineConfig(backend="cuda", engine=engine, lanes=lanes, nslots=nslots, sharding=sharding,
                       push_mode=push_mode, **kw)
    opt = OptimizerConfig("sgd", lr, clip=clip or GradClip(), l2=l2 or L2Regularization())
    cl = InProcessCluster(case.spec, opt, cfg, batch_size=case.batch, num_ps=nps, params=case.params)
    assert cl.worker.engine == engine
    return cl


def step(w, x, y):
    """One step; what it pushed, the loss and the correct count it reported."""
    out = w.step(x, y)
    w.wait_applied()
    return R.Step(R.pushed(w, out.seq), float(out.loss), int(out.correct))


def check(tag, got, case, x, y, ref=None, expect_ok=True):
    """`got` against `ref` (by default the fp64 step of the case's variables on x, y): inside the bound, or with
    `expect_ok=False` outside it. Prints the worst err / bound per variable and returns the verdict."""
    assert R.check_case(case, x, y) == [], tag
    v = R.compare(got, ref or R.reference(case.spec, case.params, x, y))
    print(f"[{tag}] {v.line()}", flush=True)
    assert v.ok == expect_ok, (tag, v.worst, v.where)
    return v


# ---------------------------------------------------------------------------------------------------------------
# lock-step trajectories
# ---------------------------------------------------------------------------------------------------------------
def gpu_lockstep(spec, opt, engine, steps, dtype="fp32", ref_update=None):
    """`steps` SGD steps of one cuda worker at batch 32 from init_params(seed 11) on synthetic data (seed 5): the fused
    engine strict through its native loader, whose batches a twin loader hands to the reference, the graph engine one
    `step()` and `wait_applied()` at a time. `ref_update(params, x, y)` applies one fp32 reference step to `params`
    in place and returns its loss; by default the plain SGD step of `mlp.manual_loss_and_grads` at `opt.lr`.
    Returns the worst per-step relative loss error and each variable's relative parameter error at the end."""
    if ref_update is None:
        def ref_update(p, x, y):
            loss, grads, _ = mlp.manual_loss_and_grads(spec, p, x, y)
            for k in p:
                p[k] = p[k] - opt.lr * grads[k]
            return float(loss)

    ds = data.synthetic_mnist(8192, seed=5)
    params = mlp.init_params(spec, seed=11)
    ref_p = {k: t.clone() for k, t in params.items()}
    kw = {"strict_steps": True} if engine == "fused" else {}
    cfg = EngineConfig(backend="cuda", engine=engine, lanes=1, nslots=8, dtype=dtype, **kw)
    worst = 0.0
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=1, params=params) as cl:
        w = cl.worker
        assert w.engine == engine
        if engine == "fused":
            loader = w.make_loader(ds.images, ds.labels, seed=7)
            twin = w.make_loader(ds.images, ds.labels, seed=7, epoch_feed=False)
            outs = []
            for n in (7, 93, steps - 100):
                outs += list(w.run_steps(n, loader, wait_applied=True))
            batches = [twin.next_batch() for _ in outs]
        else:
            it = data.BatchIterator(ds, seed=3)
            outs, batches = [], []
            for _ in range(steps):
                batches.append(it.next_batch(32))
                outs.append(w.step(*batches[-1]))
                w.wait_applied()
        assert len(outs) == steps and w.read_global_step() == steps
        for o, (x, y) in zip(outs, batches):
            lref = ref_update(ref_p, x, y)
            worst = max(worst, abs(o.loss - lref) / abs(lref))
        got = w.read_variables()
    return worst, {k: float((got[k] - ref_p[k]).norm() / (ref_p[k].norm() + 1e-9)) for k in got}


def cpu_optimizer_lockstep(opt, nps, apply_mode, steps=8, ema=False):
    """`steps` cpu-backend steps of book_model(100) at batch 32, each checked right after it against the fp32 reference
    step of bench_tools/gpu_e2e: the loss, the push sequence, and the parameters and both slot buffers; centered
    RMSProp's third slot when the rule keeps one; AdagradDA's step count on every shard; with `ema`, the moving
    averages. Returns (got, reference) params."""
    spec = mlp.book_model(100)
    cfg = EngineConfig(backend="cpu", apply_mode=apply_mode)
    ds = data.synthetic_mnist(512, seed=2)
    it = data.BatchIterator(ds, seed=0)
    params = mlp.init_params(spec, seed=5)
    rp = {k: v.clone() for k, v in params.items()}
    re = {k: v.clone() for k, v in params.items()}
    rm, rv, rg = ref_slots(opt, params, with_mg=True)
    t = 0
    with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=nps, params=params) as cl:
        w = cl.worker
        for i in range(steps):
            x, y = it.next_batch(32)
            r = w.step(x, y)
            w.wait_applied()
            lref, t = ref_step(spec, rp, rm, rv, t, x, y, opt, lr=opt.lr_at(i), mg=rg)
            assert r.loss == pytest.approx(lref, rel=1e-4)
            assert r.seq == i + 1
            got, gm, gv = w.read_variables(), w.read_variables("adam_m"), w.read_variables("adam_v")
            gg = w.read_variables("mg") if opt.uses_mg else None
            for k in got:
                assert torch.allclose(got[k], rp[k], rtol=1e-4, atol=1e-6), (i, k)
                assert torch.allclose(gm[k], rm[k], rtol=1e-4, atol=1e-7), (i, k)
                assert torch.allclose(gv[k], rv[k], rtol=1e-4, atol=1e-7), (i, k)
                if gg is not None:
                    assert torch.allclose(gg[k], rg[k], rtol=1e-4, atol=1e-7), (i, k)
            if opt.kind == "adagrad_da":
                for k in range(nps):
                    assert set(w.read_sched_steps(k)) == {i + 1}
            if ema:
                ref_ema(opt, rp, re, i + 1)
                ge = w.read_variables("ema")
                for k in ge:
                    assert torch.allclose(ge[k], re[k], rtol=1e-4, atol=1e-6), (i, k)
        assert w.read_global_step() == steps
    return got, rp
