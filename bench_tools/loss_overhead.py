"""What each `--loss` and a label smoothing cost: steps/s under each loss on both GPU engines.

The configurations, timing, alternation and output of bench_tools/activation_overhead.py (ps and worker on one GPU,
device-resident data, 12 lanes; fused engine at batch 32 and 256, graph engine with the zhihu model at batch 32): the
settings alternate over `--rounds` rounds in one call (forward, then backward order) so that clock and thermal drift
fall on all of them alike. On the fused engine the model's own loss (book) runs the ReLU instantiations and every other
setting the general-head ones; the graph engine has one head kernel for all. The percentages are the time per step
relative to the model's own loss. Prints the card name, power limit and clock and one JSON line with the median
steps/s per setting.

    python bench_tools/loss_overhead.py [--steps 20000] [--warmup 200] [--rounds 3] [--lanes 12]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SMOOTHING = 0.1
# (setting, loss, label_smoothing)
SETTINGS = [("book", "book", 0.0), ("xent", "xent", 0.0), (f"xent_ls{SMOOTHING:g}", "xent", SMOOTHING),
            ("sigmoid_xent", "sigmoid_xent", 0.0), ("mse", "mse", 0.0), ("hinge", "hinge", 0.0)]


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
        print(json.dumps({"error": "loss_overhead needs a CUDA device"}))
        return 1
    from bench_tools.clip_overhead import measure
    from bench_tools.lane_residency import card_info

    card = card_info(0)
    print(f"card {card}")
    names = [s for s, _, _ in SETTINGS]
    cases = [(f"fused_b{b}", f"fused batch {b:>3}", int(b), "book", {}) for b in a.batches.split(",")]
    cases.append(("graph_zhihu_b32", "graph zhihu batch 32", 32, "xent",
                  {"engine": "graph", "model": "zhihu", "steps": a.graph_steps}))
    res = {}
    for key, label, batch, own, kw in cases:
        runs = {s: [] for s in names}
        for r in range(a.rounds):
            for s, loss, ls in (SETTINGS if r % 2 == 0 else list(reversed(SETTINGS))):
                k = dict(kw)
                runs[s].append(measure(batch, a.lanes, k.pop("steps", a.steps), a.warmup, "off", loss=loss,
                                       label_smoothing=ls, **k))
        med = {s: statistics.median(v) for s, v in runs.items()}
        for s in names:
            print(f"{label} lanes {a.lanes} {s:>12}: {med[s]:>10.0f} steps/s "
                  f"({100.0 * (med[own] / med[s] - 1.0):+.1f}% time per step)  runs {[round(v) for v in runs[s]]}")
        res[key] = {s: round(med[s]) for s in names}
    print(json.dumps({"card": card, "lanes": a.lanes, "steps": a.steps, "steps_per_s": res}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
