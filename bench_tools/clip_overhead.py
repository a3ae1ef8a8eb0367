"""What gradient clipping costs: steps/s with clipping off and with each kind on, on both GPU engines.

Runs the bench configuration in-process (ps and worker on one GPU, device-resident data, 12 lanes) on the fused engine
at batch 32 and at batch 256 and on the graph engine with the zhihu model (784-500-500-10, batch 32), once per clip
setting, and alternates the settings over `--rounds` rounds in one call so that clock and thermal drift fall on all of
them alike. A fused measurement is one launch of `--steps` steps after a warm-up, timed with CUDA events around the
launch (Worker.last_elapsed_ms); a graph-engine measurement is the native loop over `--graph_steps` steps, timed with
CUDA events on the worker's compute stream up to the ps acknowledgement of its last push, as bench.py times it. Prints the card name and power limit and one JSON line with the median
steps/s per setting.

    python bench_tools/clip_overhead.py [--steps 20000] [--warmup 200] [--rounds 3] [--lanes 12]
"""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SETTINGS = ("off", "global_norm", "norm", "value")


def _clip(name):
    from dist_mnist_b200.parallel.config import GradClip

    if name == "off":
        return GradClip()
    if name == "value":
        return GradClip("value", value_min=-0.01, value_max=0.01)
    return GradClip(name, clip_norm=0.1)


def measure(batch: int, lanes: int, steps: int, warmup: int, clip_name: str, dev: int = 0, engine: str = "fused",
            model: str = None, l2=None, activation: str = "relu", loss: str = None, label_smoothing: float = 0.0) -> float:
    """Device-timed steps/s of `steps` steps beside the resident ps (`l2`: an L2Regularization, default off;
    `activation`: of the hidden layers; `loss`, `label_smoothing`: of the head, default the model's own loss)."""

    import torch

    import bench
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data as data_utils
    from dist_mnist_b200.utils.metrics import StreamTimer

    args = bench.parse_args(["--gpus", "1", "--lanes", str(lanes), "--batch_size", str(batch)])
    spec = mlp.get_model(model or args.model, args.hidden_units, activation, loss, label_smoothing)
    opt = OptimizerConfig(args.optimizer, args.learning_rate, clip=_clip(clip_name),
                          **({"l2": l2} if l2 is not None else {}))
    cfg = dataclasses.replace(bench.engine_config(args), engine=engine)
    ds = data_utils.synthetic_mnist(data_utils.TRAIN_SIZE, seed=0)
    # (every tensor is made before the cluster starts: no new CUDA work while a persistent ps kernel is resident)
    dev_x = ds.images.to(torch.float32 if cfg.dtype == "fp32" else torch.bfloat16).to(f"cuda:{dev}").contiguous()
    dev_y = ds.labels.to(f"cuda:{dev}").contiguous()
    cl = InProcessCluster(spec, opt, cfg, batch_size=batch, device=dev, seed=0)
    try:
        w = cl.worker
        n_rows = dev_x.shape[0] - w.B_pad
        xrow, yrow = dev_x.shape[1] * dev_x.element_size(), dev_y.shape[1] * 4
        if engine == "graph":
            w.run_resident(warmup, dev_x.data_ptr(), dev_y.data_ptr(), xrow, yrow, n_rows, 0)
            w.wait_applied()
            timer = StreamTimer(w.compute_stream, dev)
            timer.start()
            w.fork_lanes()   # no lane starts a timed step before the start event
            w.run_resident(steps, dev_x.data_ptr(), dev_y.data_ptr(), xrow, yrow, n_rows, warmup)
            w.enqueue_wait_ack()
            timer.stop()
            ms = timer.elapsed_ms()
            w.wait_applied()
            return steps / (ms / 1e3)
        w.run_resident(warmup, dev_x.data_ptr(), dev_y.data_ptr(), xrow, yrow, n_rows, 0, wait_applied=True)
        w.run_resident(steps, dev_x.data_ptr(), dev_y.data_ptr(), xrow, yrow, n_rows, warmup, wait_applied=True,
                       timed=True)
        ms = w.last_elapsed_ms()
        w.wait_applied()
    finally:
        cl.close()
    return steps / (ms / 1e3)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=20000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--lanes", type=int, default=12)
    ap.add_argument("--batches", type=str, default="32,256")
    ap.add_argument("--graph_steps", type=int, default=5000)
    a = ap.parse_args(argv)
    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"error": "clip_overhead needs a CUDA device"}))
        return 1
    from bench_tools.lane_residency import card_info

    card = card_info(0)
    print(f"card {card}")
    res = {}
    for batch in (int(b) for b in a.batches.split(",")):
        runs = {s: [] for s in SETTINGS}
        for r in range(a.rounds):
            order = SETTINGS if r % 2 == 0 else tuple(reversed(SETTINGS))
            for s in order:
                runs[s].append(measure(batch, a.lanes, a.steps, a.warmup, s))
        med = {s: statistics.median(v) for s, v in runs.items()}
        for s in SETTINGS:
            print(f"fused batch {batch:>3} lanes {a.lanes} clip {s:>11}: {med[s]:>10.0f} steps/s "
                  f"({100.0 * (med['off'] / med[s] - 1.0):+.1f}% time per step)  runs {[round(v) for v in runs[s]]}")
        res[f"fused_b{batch}"] = {s: round(med[s]) for s in SETTINGS}
    runs = {s: [] for s in SETTINGS}
    for r in range(a.rounds):
        for s in (SETTINGS if r % 2 == 0 else tuple(reversed(SETTINGS))):
            runs[s].append(measure(32, a.lanes, a.graph_steps, a.warmup, s, engine="graph", model="zhihu"))
    med = {s: statistics.median(v) for s, v in runs.items()}
    for s in SETTINGS:
        print(f"graph zhihu batch 32 lanes {a.lanes} clip {s:>11}: {med[s]:>10.0f} steps/s "
              f"({100.0 * (med['off'] / med[s] - 1.0):+.1f}% time per step)  runs {[round(v) for v in runs[s]]}")
    res["graph_zhihu_b32"] = {s: round(med[s]) for s in SETTINGS}
    print(json.dumps({"card": card, "lanes": a.lanes, "steps": a.steps, "steps_per_s": res}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
