"""Where the fused step's lanes and the ps serve kernel run on one shared GPU, and whether every lane takes part.

Runs the flagship bench configuration in-process (ps and worker on one GPU, fused engine, device-resident data): a
warm-up, then one long launch of `--steps` steps after a ps restart, the way bench.py's timed region runs. The fused
kernel writes its lane residency record (FusedParams::lane_rec) and the serve kernel its per-CTA SM ids
(DM_PS_STATS=1). Printed: per cluster its SMs, the steps it claimed and when it started and finished relative to the
first cluster; the ps CTAs' SMs and serve statistics; the device's cluster capacity for the fused kernel before the
ps starts; and a JSON summary line.

    python bench_tools/lane_residency.py [--lanes 12] [--steps 20000] [--warmup 50] [--batch_size 32]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card_info(dev: int) -> dict:
    import torch

    props = torch.cuda.get_device_properties(dev)
    info = {"name": props.name, "sm_count": props.multi_processor_count}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_and_max_sm_clock"] = out
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable ({e})"
    return info


def run(lanes: int, steps: int, warmup: int, batch: int, dev: int = 0, clip=None) -> dict:
    """One long fused launch beside the resident ps; returns the residency record as a dict. `clip`: a GradClip, which
    runs the gradient-clipping instantiation of the fused kernel."""
    import torch

    import bench
    from dist_mnist_b200 import _native as N
    from dist_mnist_b200.models import mlp
    from dist_mnist_b200.parallel.config import OptimizerConfig
    from dist_mnist_b200.session import InProcessCluster
    from dist_mnist_b200.utils import data as data_utils

    args = bench.parse_args(["--gpus", "1", "--lanes", str(lanes), "--batch_size", str(batch)])
    spec = mlp.get_model(args.model, args.hidden_units)
    opt = OptimizerConfig(args.optimizer, args.learning_rate, **({"clip": clip} if clip is not None else {}))
    cfg = bench.engine_config(args)
    torch.cuda.set_device(dev)
    lib = N.lib()
    N.ensure_prepared(dev)
    max_lanes = C.c_int(0)
    N.check(lib.dm_fused_max_lanes(dev, batch, int(opt.clip.enabled), int(opt.l2.enabled),
                                   mlp.activation_code(spec.activation), C.byref(max_lanes)), "fused occupancy")

    ds = data_utils.synthetic_mnist(data_utils.TRAIN_SIZE, seed=0)
    dev_x = ds.images.to(torch.float32).to(f"cuda:{dev}").contiguous()
    dev_y = ds.labels.to(f"cuda:{dev}").contiguous()
    held = {}

    def hook(w):   # allocated before the ps kernel is resident
        held["rec"] = torch.zeros(w.fused_lanes * N.LANE_REC_WORDS, dtype=torch.int64, device=f"cuda:{dev}")

    stats_env = os.environ.get("DM_PS_STATS")
    os.environ["DM_PS_STATS"] = "1"   # serve statistics, which carry the ps CTAs' SM ids
    cl = InProcessCluster(spec, opt, cfg, batch_size=batch, device=dev, seed=0, setup_hook=hook)
    try:
        w, ps = cl.worker, cl.ps[0]
        if w.engine != "fused":
            raise SystemExit(f"the probe needs the fused engine (got {w.engine})")
        rec = held["rec"]
        w._fx_params.lane_rec = rec.data_ptr()
        N.check(lib.dm_fexec_set_params(w._fexec, C.addressof(w._fx_maps), C.addressof(w._fx_params)), "set params")
        n_rows = dev_x.shape[0] - w.B_pad
        xrow, yrow = dev_x.shape[1] * 4, dev_y.shape[1] * 4
        w.run_resident(warmup, dev_x.data_ptr(), dev_y.data_ptr(), xrow, yrow, n_rows, 0)

        # quiesce, clear the record and the counters, relaunch the ps (as bench.py does before a timed region)
        w.wait_applied()
        ps.stop()
        ps.serve_stats(reset=True)
        torch.cuda.synchronize()
        rec.zero_()
        torch.cuda.synchronize()
        ps.restart()
        w.run_resident(steps, dev_x.data_ptr(), dev_y.data_ptr(), xrow, yrow, n_rows, warmup, wait_applied=True,
                       timed=True)
        ms = w.last_elapsed_ms()
        w.wait_applied()
        ps.stop()
        ps_stats = ps.serve_stats()
        torch.cuda.synchronize()
        r = rec.cpu().view(-1, N.LANE_REC_WORDS).tolist()
        ps.restart()
    finally:
        cl.close()
        if stats_env is None:
            del os.environ["DM_PS_STATS"]
        else:
            os.environ["DM_PS_STATS"] = stats_env

    t0 = min(row[9] for row in r if row[8] > 0)
    clusters = [{"lane": i, "smids": row[:8], "steps": row[8],
                 "entry_us": round((row[11] - t0) / 1e3, 1),
                 "first_claim_us": round((row[9] - t0) / 1e3, 1) if row[8] else None,
                 "end_us": round((row[10] - t0) / 1e3, 1)} for i, row in enumerate(r)]
    return {"lanes": w.fused_lanes, "steps": steps, "elapsed_ms": round(ms, 3),
            "steps_per_s": round(steps / (ms / 1e3)), "us_per_step_per_lane": round(ms * 1e3 * w.fused_lanes / steps, 2),
            "fused_max_active_clusters_before_ps": max_lanes.value,
            "ps_ctas": (ps_stats or {}).get("ctas"), "ps_smids": (ps_stats or {}).get("smids"),
            "ps_busy_fraction": (ps_stats or {}).get("busy_fraction"), "ps_stats": ps_stats, "clusters": clusters}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lanes", type=int, default=12)
    ap.add_argument("--steps", type=int, default=20000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--batch_size", type=int, default=32)
    a = ap.parse_args(argv)
    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"error": "lane_residency needs a CUDA device"}))
        return 1
    res = run(a.lanes, a.steps, a.warmup, a.batch_size)
    res["card"] = card_info(0)
    print(f"card {res['card']}; fused max active clusters before the ps starts: "
          f"{res['fused_max_active_clusters_before_ps']}; ps CTAs {res['ps_ctas']} on SMs {res['ps_smids']}")
    print(f"{res['lanes']} lanes, {res['steps']} steps in {res['elapsed_ms']} ms = {res['steps_per_s']} steps/s "
          f"({res['us_per_step_per_lane']} us per step per lane); ps busy fraction {res['ps_busy_fraction']}")
    print(f"{'lane':>4} {'steps':>6} {'entry_us':>10} {'first_us':>10} {'end_us':>10}  SMs")
    for c in res["clusters"]:
        print(f"{c['lane']:>4} {c['steps']:>6} {c['entry_us']:>10} {str(c['first_claim_us']):>10} {c['end_us']:>10}  "
              f"{c['smids']}")
    print(json.dumps({k: v for k, v in res.items() if k not in ("clusters", "ps_stats")}
                     | {"claims": [c["steps"] for c in res["clusters"]],
                        "first_claim_us": [c["first_claim_us"] for c in res["clusters"]]}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
