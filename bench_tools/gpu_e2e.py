"""Single-GPU end-to-end checks of the engine (ps + worker in one process on cuda:0).

    python -m bench_tools.gpu_e2e traj        # lock-step trajectory vs a plain PyTorch fp32 re-implementation
    python -m bench_tools.gpu_e2e throughput  # pipelined native loop, steps/s
    python -m bench_tools.gpu_e2e all
"""
from __future__ import annotations

import dataclasses
import struct
import subprocess
import sys
import os
import time
import traceback

import torch

from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
from dist_mnist_b200.session import InProcessCluster
from dist_mnist_b200.utils import data


def _prox_shrink(prox, a, l1, l2):
    """ApplyProximalAdagrad / ApplyProximalGradientDescent's proximal step at step size `a` (a tensor)."""
    if l1 > 0:
        return prox.sign() * (prox.abs() - a * l1).clamp_min(0) / (1 + l2 * a)
    return prox / (1 + l2 * a)


def _f32(x: float) -> float:
    return struct.unpack("f", struct.pack("f", float(x)))[0]


def tf1_apply(opt, p, m, v, g, mg=None, global_step=None):
    """One TF1 `training_ops` step of Momentum / Adagrad / RMSProp / Adadelta / FTRL (V2 with l2_shrinkage) /
    ProximalAdagrad / ProximalGradientDescent / AdagradDA on tensors, in their own dtype: `m` is the slot kept in
    adam_m (momentum accumulator, RMSProp mom, Adadelta accum_update, FTRL linear, AdagradDA gradient_accumulator), `v`
    the one in adam_v (Adagrad, FTRL and ProximalAdagrad accumulator, RMSProp ms, Adadelta accum, AdagradDA
    gradient_squared_accumulator). Returns the new (p, m, v).

    `mg`: centered RMSProp's third slot (needed when opt.centered); the result is then (p, m, v, mg).
    `global_step`: AdagradDA's T, the applied steps including this one (an integer; converted to fp32 once, as TF's
    static_cast<float> and the ps do)."""
    if opt.kind == "rmsprop" and opt.centered:
        if mg is None:
            raise ValueError("centered rmsprop needs its mg slot")
        v = v + (g * g - v) * (1 - opt.decay)
        mg = mg + (g - mg) * (1 - opt.decay)
        m = m * opt.momentum + (g * opt.lr) / ((v - mg * mg) + opt.eps).sqrt()
        return p - m, m, v, mg
    if opt.kind == "adagrad_da":
        if global_step is None:
            raise ValueError("adagrad_da needs the global step T")
        T = _f32(int(global_step))
        l1, l2, lr = opt.l1_regularization_strength, opt.l2_regularization_strength, opt.lr
        m = m + g
        v = v + g * g
        if l1 > 0:
            p = -lr * m.sign() * (m.abs() - T * l1).clamp_min(0) / (l2 * (T * lr) + v.sqrt())
        else:
            p = -lr * m / ((T * lr) * l2 + v.sqrt())
    elif opt.kind == "momentum":
        m = opt.momentum * m + g
        p = p - (g * opt.lr + m * opt.momentum * opt.lr) if opt.use_nesterov else p - opt.lr * m
    elif opt.kind == "adagrad":
        v = v + g * g
        p = p - opt.lr * g / v.sqrt()
    elif opt.kind == "rmsprop":
        v = v + (g * g - v) * (1 - opt.decay)
        m = opt.momentum * m + opt.lr * g / (v + opt.eps).sqrt()
        p = p - m
    elif opt.kind == "adadelta":
        rho = opt.rho
        v = v * rho + g * g * (1 - rho)
        upd = (m + opt.eps).sqrt() * (v + opt.eps).rsqrt() * g
        p = p - upd * opt.lr
        m = m * rho + upd * upd * (1 - rho)
    elif opt.kind == "proximal_adagrad":
        v = v + g * g
        a = opt.lr * v.rsqrt()
        p = _prox_shrink(p - g * a, a, opt.l1_regularization_strength, opt.l2_regularization_strength)
    elif opt.kind == "proximal_sgd":
        a = torch.full_like(p, opt.lr)
        p = _prox_shrink(p - g * a, a, opt.l1_regularization_strength, opt.l2_regularization_strength)
    elif opt.kind == "ftrl":
        l1, l2, lrp = opt.l1_regularization_strength, opt.l2_regularization_strength, opt.learning_rate_power
        gs = g + 2 * opt.l2_shrinkage_regularization_strength * p
        n = v + g * g
        pn, pa = (n.sqrt(), v.sqrt()) if lrp == -0.5 else (n.pow(-lrp), v.pow(-lrp))
        m = m + (gs - (pn - pa) / opt.lr * p)
        y = pn / opt.lr + 2 * l2
        p = torch.where(m.abs() > l1, (m.sign() * l1 - m) / y, torch.zeros_like(p))
        v = n
    else:
        raise ValueError(opt.kind)
    return (p, m, v) if mg is None else (p, m, v, mg)


def ref_slots(opt, params, with_mg=False):
    """Initial (m, v) slot dicts of `opt` for `params` (Worker.initialize_variables writes the same values).
    `with_mg`: (m, v, mg), with centered RMSProp's third slot (zeros)."""
    m0, v0 = opt.slot_init()
    m, v = {k: torch.full_like(t, m0) for k, t in params.items()}, {k: torch.full_like(t, v0) for k, t in params.items()}
    return (m, v, {k: torch.zeros_like(t) for k, t in params.items()}) if with_mg else (m, v)


def ref_step(spec, params, m, v, t, x, y, opt, lr=None, mg=None, global_step=None):
    """One reference training step in place; `lr`: this step's rate (a learning-rate schedule's), else opt.lr.
    `mg`: centered RMSProp's third slot dict (updated in place). `global_step`: AdagradDA's T for this step, by default
    the returned step count (one worker, starting from step 0)."""
    if lr is not None:
        opt = dataclasses.replace(opt, lr=lr)
    loss, grads, _ = mlp.manual_loss_and_grads(spec, params, x, y)
    t += 1
    for k in params:
        g = grads[k]
        if opt.kind == "sgd":
            params[k] = params[k] - opt.lr * g
        elif opt.kind == "rmsprop" and opt.centered:
            params[k], m[k], v[k], mg[k] = tf1_apply(opt, params[k], m[k], v[k], g, mg=mg[k])
        elif opt.kind != "adam":
            params[k], m[k], v[k] = tf1_apply(opt, params[k], m[k], v[k], g,
                                              global_step=t if global_step is None else global_step)
        else:
            m[k] = opt.beta1 * m[k] + (1 - opt.beta1) * g
            v[k] = opt.beta2 * v[k] + (1 - opt.beta2) * g * g
            lr_t = opt.lr * (1 - opt.beta2 ** t) ** 0.5 / (1 - opt.beta1 ** t)
            params[k] = params[k] - lr_t * m[k] / (v[k].sqrt() + opt.eps)
    return float(loss), t


def ref_ema(opt, params, ema, n):
    """TF1 `ExponentialMovingAverage.apply` in place, after the optimizer step that brought the global step to `n`:
    shadow -= (shadow - p) * (1 - d) with d = opt.ema_decay_at(n), every op in fp32 as TF1's graph does it."""
    omd = torch.tensor(1.0, dtype=torch.float32) - torch.tensor(opt.ema_decay_at(n), dtype=torch.float32)
    for k in params:
        ema[k] = ema[k] - (ema[k] - params[k]) * omd


def wait_gstep(worker, target, timeout=10.0):
    t0 = time.time()
    while worker.read_global_step() < target:
        if time.time() - t0 > timeout:
            raise TimeoutError(f"global_step stuck at {worker.read_global_step()} < {target}")
        time.sleep(0.0005)


# (model, optimizer, dtype, push mode, #ps, batch, tolerance). SGD is linear in the gradient, so its parameter
# error directly reflects kernel numerics (tf32 / bf16 rounding); Adam's normalised step m/sqrt(v) turns a
# rounding-level gradient difference on a near-zero gradient into a full +-lr step, hence the looser bound there.
TRAJ_CASES = [
        # --- fused step engine (the reference's live configuration: 784-100-10, batch 32, fp32) ---
        ("book", "adam", "fp32", "mailbox", 1, 32, 5e-2),
        ("book", "sgd", "fp32", "mailbox", 1, 32, 2e-2),
        ("book", "sgd", "fp32", "atomic", 1, 32, 2e-2),
        ("book", "adam", "fp32", "mailbox", 2, 32, 5e-2),
        # --- per-layer kernels in a CUDA graph (deeper / wider / bf16 models) ---
        ("zhihu", "sgd", "fp32", "mailbox", 2, 100, 2e-2),
        ("zhihu", "adam", "fp32", "mailbox", 2, 100, 2.5e-1),
        ("wide", "sgd", "bf16", "mailbox", 2, 64, 5e-2),
        ("wide", "adam", "bf16", "mailbox", 2, 64, 2.5e-1),
        ("book", "adam", "bf16", "mailbox", 1, 32, 2e-1),
        # --- fused engine: intra-variable (row-split) sharding over 2 and 8 ps shards, strict pull order, xent loss,
        #     a partial batch and a narrower hidden layer ---
        ("book", "sgd", "fp32", "mailbox", 2, 32, 2e-2, {"sharding": "row_split"}),
        ("book", "adam", "fp32", "mailbox", 8, 32, 5e-2, {"sharding": "row_split", "strict_steps": True}),
        ("book", "sgd", "fp32", "mailbox", 1, 20, 2e-2, {"loss": "xent", "hidden": 64}),
        # --- the same flagship model through the graph engine (kept as the general path) ---
        ("book", "adam", "fp32", "mailbox", 1, 32, 5e-2, {"engine": "graph"}),
        ("book", "sgd", "fp32", "atomic", 1, 32, 2e-2, {"engine": "graph"}),
]


def check_traj(only=None) -> bool:
    ok = True
    ds = data.synthetic_mnist(4096, seed=3)
    cases = TRAJ_CASES if only is None else [TRAJ_CASES[only]]
    for case in cases:
        (model, okind, dtype, push, nps, batch, tol), extra = case[:7], (case[7] if len(case) > 7 else {})
        name = f"traj model={model} opt={okind} dtype={dtype} push={push} ps={nps} B={batch} {extra or ''}"
        try:
            spec = mlp.get_model(model, extra.get("hidden", 100)) if model == "book" else mlp.get_model(model)
            if extra.get("loss"):
                import dataclasses
                spec = dataclasses.replace(spec, loss=extra["loss"])
            lr = 1e-3 if okind == "adam" else 5e-2
            opt = OptimizerConfig(okind, lr)
            cfg = EngineConfig(backend="cuda", dtype=dtype, push_mode=push, sharding=extra.get("sharding", "round_robin"),
                               engine=extra.get("engine", "auto"), strict_steps=extra.get("strict_steps", False))
            params = mlp.init_params(spec, seed=7)
            ref_p = {k: t.clone() for k, t in params.items()}
            ref_m = {k: torch.zeros_like(t) for k, t in params.items()}
            ref_v = {k: torch.zeros_like(t) for k, t in params.items()}
            t = 0
            it = data.BatchIterator(ds, seed=1)
            with InProcessCluster(spec, opt, cfg, batch_size=batch, num_ps=nps, params=params) as cl:
                w = cl.worker
                worst = 0.0
                n_steps = 12
                for i in range(n_steps):
                    x, y = it.next_batch(batch)
                    r = w.step(x, y)
                    if os.environ.get("DM_TRAJ_WAIT", "applied") == "applied":
                        w.wait_applied()   # every shard has applied the push (global_step lives on shard 0 only)
                    wait_gstep(w, i + 1)
                    lref, t = ref_step(spec, ref_p, ref_m, ref_v, t, x, y, opt)
                    worst = max(worst, abs(r.loss - lref) / (abs(lref) + 1e-9))
                    if os.environ.get("DM_TRAJ_VERBOSE"):
                        print(f"      step {i}: loss {r.loss!r} ref {lref!r}", flush=True)
                got = w.read_variables()
                perrs = {k: float((got[k] - ref_p[k]).norm() / (ref_p[k].norm() + 1e-9)) for k in got}
                perr = max(perrs.values())
                if os.environ.get("DM_TRAJ_VERBOSE"):
                    print("    per-variable rel err: " + " ".join(f"{k}={v:.2e}" for k, v in perrs.items()), flush=True)
                gs = w.read_global_step()
                acc_loss, acc = w.evaluate(ds.images[:512], ds.labels[:512])
            good = worst < tol and perr < tol and gs == n_steps
            print(f"[{'PASS' if good else 'FAIL'}] {name}: engine={w.engine} worst_loss_rel={worst:.2e} "
                  f"param_rel={perr:.2e} global_step={gs} eval_loss={acc_loss:.4f} acc={acc:.3f}", flush=True)
            ok &= good
        except Exception:
            traceback.print_exc()
            print(f"[FAIL] {name}: exception", flush=True)
            ok = False
    return ok


TP_CASES = [("book", "adam", "fp32", "mailbox", 32), ("book", "sgd", "fp32", "atomic", 32),
            ("book", "sgd", "fp32", "mailbox", 32), ("wide", "adam", "bf16", "mailbox", 32)]


def check_throughput(only=None) -> bool:
    ok = True
    ds = data.synthetic_mnist(data.TRAIN_SIZE, seed=0)
    for (model, okind, dtype, push, batch) in (TP_CASES if only is None else [TP_CASES[only]]):
        name = f"throughput model={model} opt={okind} dtype={dtype} push={push} B={batch}"
        try:
            spec = mlp.get_model(model)
            opt = OptimizerConfig(okind, 1e-4 if okind == "adam" else 1e-2)
            cfg = EngineConfig(backend="cuda", dtype=dtype, push_mode=push)
            with InProcessCluster(spec, opt, cfg, batch_size=batch) as cl:
                w = cl.worker
                loader = w.make_loader(ds.images, ds.labels, seed=0)
                outs = w.run_steps(200, loader)  # warm-up
                first_loss = outs[0].loss
                torch.cuda.synchronize() if False else None
                t0 = time.perf_counter()
                n = 4000
                outs = w.run_steps(n, loader)
                dt = time.perf_counter() - t0
                w.drain()
                time.sleep(0.05)
                gs = w.read_global_step()
                print(f"[PASS] {name}: {n / dt:.0f} steps/s e2e (wall), {dt / n * 1e6:.1f} us/step, loss {first_loss:.4f} -> "
                      f"{outs[-1].loss:.4f}, global_step={gs} (expected {n + 200}), kernels/step={w.kernels_per_step}",
                      flush=True)
                ok &= gs == n + 200
        except Exception:
            traceback.print_exc()
            print(f"[FAIL] {name}: exception", flush=True)
            ok = False
    return ok


PIPE_CASES = [
    # graph engine (lanes / group graphs / PDL)
    ("book", "adam", "fp32", "mailbox", 2, 1, False, False, {"engine": "graph"}),
    ("book", "adam", "fp32", "mailbox", 4, 2, True, False, {"engine": "graph"}),
    ("book", "sgd", "fp32", "atomic", 4, 4, True, False, {"engine": "graph"}),
    ("wide", "adam", "bf16", "mailbox", 4, 2, True),
    ("zhihu", "sgd", "fp32", "mailbox", 2, 2, False),
    # fused engine: lanes = clusters of one launch, chunked executor
    ("book", "adam", "fp32", "mailbox", 1, 1, True, False, {}),
    ("book", "adam", "fp32", "mailbox", 8, 1, True, False, {}),
    ("book", "sgd", "fp32", "atomic", 4, 1, True, False, {}),
    ("book", "adam", "fp32", "mailbox", 8, 1, True, False, {"sharding": "row_split", "num_ps": 2}),
    ("book", "adam", "fp32", "mailbox", 2, 1, True, False, {"strict_steps": True}),
]


def check_pipelined(only=None) -> bool:
    """Several steps in flight (lanes) and several steps per graph launch (graph_steps): every step gets a unique
    push sequence number, every push is applied exactly once (global_step == steps), results come back in
    submission order and training still converges; mixes odd-sized runs so that the single-step head / tail paths
    of the native loop are exercised next to the group launches."""
    ok = True
    ds = data.synthetic_mnist(8192, seed=0)
    for case in (PIPE_CASES if only is None else [PIPE_CASES[only]]):
        (model, okind, dtype, push, lanes, gsteps, pdl), fuse = case[:7], (len(case) > 7 and case[7])
        extra = case[8] if len(case) > 8 else {}
        name = (f"pipelined model={model} opt={okind} dtype={dtype} push={push} lanes={lanes} graph_steps={gsteps} "
                f"pdl={pdl} {extra or ''}")
        try:
            spec = mlp.get_model(model)
            opt = OptimizerConfig(okind, 1e-3 if okind == "adam" else 1e-2)
            cfg = EngineConfig(backend="cuda", dtype=dtype, push_mode=push, lanes=lanes, graph_steps=gsteps,
                               nslots=max(2, lanes), pipeline_slots=max(4, 2 * lanes), pdl=pdl,
                               engine=extra.get("engine", "auto"), sharding=extra.get("sharding", "round_robin"),
                               strict_steps=extra.get("strict_steps", False))
            with InProcessCluster(spec, opt, cfg, batch_size=32, num_ps=extra.get("num_ps", 1)) as cl:
                w = cl.worker
                loader = w.make_loader(ds.images, ds.labels, seed=0)
                outs = []
                for n in (3, 301, 1, 200, 7):
                    outs += w.run_steps(n, loader)
                x, y = loader.next_batch()
                outs.append(w.step(x, y))          # synchronous API on the same executor
                outs += w.run_steps(88, loader)
                total = 3 + 301 + 1 + 200 + 7 + 1 + 88
                w.wait_applied()
                gs = w.read_global_step()
                seqs = sorted(o.seq for o in outs)
                first = sum(o.loss for o in outs[:20]) / 20
                last = sum(o.loss for o in outs[-20:]) / 20
                good_fused = True
                good = (good_fused and len(outs) == total and gs == total and seqs == list(range(1, total + 1))
                        and last < first and all(o.loss == o.loss for o in outs))
                print(f"[{'PASS' if good else 'FAIL'}] {name}: engine={w.engine} steps={len(outs)} global_step={gs} "
                      f"seqs unique={seqs == list(range(1, total + 1))} loss {first:.4f} -> {last:.4f}", flush=True)
                ok &= good
        except Exception:
            traceback.print_exc()
            print(f"[FAIL] {name}: exception", flush=True)
            ok = False
    return ok


CHECKS = {"traj": check_traj, "throughput": check_throughput, "pipelined": check_pipelined}


def main(argv) -> int:
    which = argv[0] if argv else "all"
    if which == "all":
        rc = 0
        jobs = [f"traj:{i}" for i in range(len(TRAJ_CASES))] + [f"throughput:{i}" for i in range(len(TP_CASES))]
        for g in jobs:
            try:
                code = subprocess.run([sys.executable, "-m", "bench_tools.gpu_e2e", g], timeout=120).returncode
            except subprocess.TimeoutExpired:
                code = 124
            if code != 0:
                print(f"===== {g}: exit {code} =====", flush=True)
            rc |= int(code != 0)
        return rc
    import faulthandler
    faulthandler.dump_traceback_later(75, exit=True)  # a hang prints the Python stack of every thread, then exits
    group, _, idx = which.partition(":")
    return 0 if CHECKS[group](int(idx) if idx else None) else 1


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
