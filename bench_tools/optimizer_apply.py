"""What each ps optimizer costs in the flagship configuration: Adam, SGD, Momentum, Nesterov momentum, Adagrad,
RMSProp, Adadelta, FTRL (at lr_power -0.5, the square-root path, and as `ftrl_pow` at -0.25, the general power),
ProximalAdagrad and ProximalGradientDescent, one after the other, in bench.py's single-GPU setup (ps and worker sharing the GPU, fused engine, default
lanes, device-resident data).

Per optimizer, two in-process clusters: one for the device-timed steps/s of `Worker.run_resident` (the serve kernel's
counters off, as in bench.py), one with DM_PS_STATS=1 for the serve kernel's apply cycles per push
(`ParameterServer.serve_stats()`). The card's name and power limit are read in the same call. One JSON line per
optimizer, then a table.

`--lr_schedule KIND` measures every optimizer twice, under that learning-rate schedule (the scheduled serve kernels)
and at a constant rate, alternated in the same call: the cost of the rate table the scheduled kernels build per pass.
`--moving_average_decay D` likewise measures every optimizer with moving averages of that decay (the averaging serve
kernels) and without, alternated in the same call: the cost of the shadow load, update and store.

`--rounds N` repeats the whole sequence N times, so that every rule is measured N times, alternated with the others.

    python bench_tools/optimizer_apply.py [--steps 20000] [--warmup 50] [--only rmsprop,adam] [--lr_schedule KIND]
                                          [--moving_average_decay D] [--rounds N]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

RULES = ["adam", "sgd", "momentum", "nesterov", "adagrad", "rmsprop", "adadelta", "ftrl", "ftrl_pow", "proximal_adagrad",
         "proximal_sgd"]


def schedule(kind: str, lr: float):
    """A schedule of `kind` that changes the rate many times within a measured run."""
    from dist_mnist_b200.parallel.config import LrSchedule

    if kind in ("exponential_decay", "inverse_time_decay", "natural_exp_decay"):
        return LrSchedule(kind, decay_steps=1000, decay_rate=0.96)
    if kind in ("polynomial_decay", "cosine_decay"):
        return LrSchedule(kind, decay_steps=100000)
    if kind == "piecewise_constant":
        return LrSchedule(kind, boundaries=(5000, 10000), values=(lr, lr / 10, lr / 100))
    return LrSchedule()


def optimizer(rule: str, lr: float, sched: str = "constant", ema=None):
    from dist_mnist_b200.parallel.config import OptimizerConfig

    if rule == "nesterov":
        return OptimizerConfig("momentum", lr, use_nesterov=True, schedule=schedule(sched, lr),
                               moving_average_decay=ema)
    if rule == "ftrl_pow":
        return OptimizerConfig("ftrl", lr, learning_rate_power=-0.25, schedule=schedule(sched, lr),
                               moving_average_decay=ema)
    return OptimizerConfig(rule, lr, schedule=schedule(sched, lr), moving_average_decay=ema)


def run_one(rule: str, steps: int, warmup: int, stats: bool, dev: int = 0, sched: str = "constant",
            ema=None) -> dict:
    """One cluster in the bench configuration: warm-up, then one timed run_resident region after a ps restart."""
    import torch

    import bench
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data as data_utils

    args = bench.parse_args(["--gpus", "1"])
    spec = mlp.get_model(args.model, args.hidden_units)
    cfg = bench.engine_config(args)
    opt = optimizer(rule, args.learning_rate, sched, ema)
    torch.cuda.set_device(dev)
    ds = data_utils.synthetic_mnist(data_utils.TRAIN_SIZE, seed=0)
    dev_x = ds.images.to(torch.float32).to(f"cuda:{dev}").contiguous()
    dev_y = ds.labels.to(f"cuda:{dev}").contiguous()
    old = os.environ.get("DM_PS_STATS")
    os.environ["DM_PS_STATS"] = "1" if stats else "0"
    cl = InProcessCluster(spec, opt, cfg, batch_size=args.batch_size, device=dev, seed=0)
    try:
        w, ps = cl.worker, cl.ps[0]
        n_rows = dev_x.shape[0] - w.B_pad
        xrow, yrow = dev_x.shape[1] * 4, dev_y.shape[1] * 4
        w.run_resident(warmup, dev_x.data_ptr(), dev_y.data_ptr(), xrow, yrow, n_rows, 0)
        w.wait_applied()
        ps.stop()
        ps.serve_stats(reset=True)
        ps.restart()
        w.run_resident(steps, dev_x.data_ptr(), dev_y.data_ptr(), xrow, yrow, n_rows, warmup, wait_applied=True,
                       timed=True)
        ms = w.last_elapsed_ms()
        w.wait_applied()
        ps.stop()
        st = ps.serve_stats()
        gs = w.read_global_step()
        ps.restart()
        res = {"engine": w.engine, "lanes": w.fused_lanes if w.engine == "fused" else cfg.lanes,
               "elapsed_ms": round(ms, 3), "steps_per_s": round(steps / (ms / 1e3)), "global_step": gs}
        if st is not None:
            res.update({k: st[k] for k in ("apply_cycles_per_push", "pushes_per_pass", "apply_us_per_pass",
                                           "busy_fraction")})
        return res
    finally:
        cl.close()
        if old is None:
            del os.environ["DM_PS_STATS"]
        else:
            os.environ["DM_PS_STATS"] = old


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=20000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--only", type=str, default="", help="comma-separated subset of " + ",".join(RULES))
    ap.add_argument("--lr_schedule", type=str, default="constant",
                    help="also run every optimizer under this learning-rate schedule, alternated with constant")
    ap.add_argument("--moving_average_decay", type=float, default=None,
                    help="also run every optimizer with moving averages of this decay, alternated with none")
    ap.add_argument("--rounds", type=int, default=1, help="repeat the whole sequence of optimizers this many times")
    a = ap.parse_args(argv)
    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"error": "optimizer_apply needs a CUDA device"}))
        return 1
    from bench_tools.lane_residency import card_info

    rules = [r for r in a.only.split(",") if r] or RULES
    for r in rules:
        if r not in RULES:
            raise SystemExit(f"unknown rule {r!r} ({', '.join(RULES)})")
    from dist_mnist_b200.parallel.config import LR_SCHEDULES
    if a.lr_schedule not in LR_SCHEDULES:
        raise SystemExit(f"unknown lr_schedule {a.lr_schedule!r} ({', '.join(LR_SCHEDULES)})")
    scheds = [a.lr_schedule, "constant"] if a.lr_schedule != "constant" else ["constant"]
    emas = [a.moving_average_decay, None] if a.moving_average_decay is not None else [None]
    card = card_info(0)
    rows = []
    for r in [r for _ in range(a.rounds) for r in rules]:
        for sc, ema in [(sc, e) for sc in scheds for e in emas]:
            timed = run_one(r, a.steps, a.warmup, stats=False, sched=sc, ema=ema)
            counted = run_one(r, a.steps, a.warmup, stats=True, sched=sc, ema=ema)
            row = {"optimizer": r, "lr_schedule": sc, "moving_average_decay": ema, **timed,
                   "apply_cycles_per_push": counted.get("apply_cycles_per_push"),
                   "pushes_per_pass": counted.get("pushes_per_pass"), "ps_busy_fraction": counted.get("busy_fraction"),
                   "steps_per_s_with_counters": counted["steps_per_s"], "card": card}
            rows.append(row)
            print(json.dumps(row), flush=True)
    print(f"card {card}; {a.steps} timed steps per optimizer, schedule and averaging; {a.rounds} round(s)")
    print(f"{'optimizer':>10} {'lr_schedule':>18} {'ema decay':>10} {'steps/s':>9} {'apply cycles/push':>18} "
          f"{'pushes/pass':>12} {'ps busy':>8}")
    for row in rows:
        print(f"{row['optimizer']:>10} {row['lr_schedule']:>18} {str(row['moving_average_decay']):>10} "
              f"{row['steps_per_s']:>9} "
              f"{str(row['apply_cycles_per_push']):>18} {str(row['pushes_per_pass']):>12} "
              f"{str(row['ps_busy_fraction']):>8}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
