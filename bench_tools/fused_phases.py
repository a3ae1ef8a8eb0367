"""In-kernel phase stamps of the fused step kernel (DM_FUSED_DEBUG_TS=1): clock64() of cluster 0 / CTA 0 at
step start, forward accumulator ready, after the reduce-scatter barrier, head done, after the all-gather barrier,
dW accumulator ready, tile pushed, step end — for the first 8 steps of the last launch. lanes=1 and lanes=8."""
import os
import sys

import torch

from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.config import EngineConfig, OptimizerConfig
from dist_mnist_b200.session import InProcessCluster
from dist_mnist_b200.utils import data

NAMES = ["start", "acc1", "rs_bar", "head_in", "softmax", "grads_sent", "ag_bar", "acc2", "staged", "bar3",
         "tile_published(w0)", "result(w0)"]
KTS = 16
SM_MHZ = 1980   # H100 SXM maximum SM clock: cycle counts are converted at this rate (a power-limited card runs slower)


def print_stamps(buf, tag):
    """Epilogue thread 0 of cluster 0 / CTA 0 stamps 0..9, warp 0 (publisher) stamps 10, 11; first 4 steps."""
    ts = buf.view(4, KTS)
    t0 = int(ts[0, 0])
    print(f"{tag}: cluster 0, SM cycles ({SM_MHZ} MHz -> /{SM_MHZ} = us); deltas to the previous stamp")
    for j in range(4):
        row = [int(ts[j, k]) - t0 for k in range(12)]
        d = [row[k] - row[k - 1] if k else 0 for k in range(10)]
        nxt = (int(ts[j + 1, 0]) - t0 - row[0]) if j + 1 < 4 else None
        print(f"  step {j}: " + " ".join(f"{NAMES[k]}=+{d[k]}" for k in range(1, 10)) +
              f" | publisher: tile at +{row[10] - row[9]} after bar3, result at +{row[11] - row[9]}"
              f" | step {row[9] - row[0]} cyc = {(row[9] - row[0]) / SM_MHZ:.2f} us"
              + (f", next step starts {nxt} cyc after this one" if nxt is not None else ""))


    g = [int(buf[60]), int(buf[61]), int(buf[63])]
    if g[0] and g[1]:
        print(f"  globaltimer: kernel entry -> first step claimed {(g[1] - g[0]) / 1e3:.2f} us"
              + (f"; entry -> last cluster re-armed / acks in {(g[2] - g[0]) / 1e3:.2f} us" if g[2] > g[0] else ""))


def main():
    os.environ["DM_FUSED_DEBUG_TS"] = "1"
    ds = data.synthetic_mnist(8192, seed=0)
    spec = mlp.book_model(100)
    opt = OptimizerConfig("adam", 1e-4)
    for lanes in (1, 8):
        cfg = EngineConfig(backend="cuda", lanes=lanes, nslots=2 * lanes, pipeline_slots=max(4, 2 * lanes))
        with InProcessCluster(spec, opt, cfg, batch_size=32) as cl:
            w = cl.worker
            dev_x = ds.images.cuda().contiguous()
            dev_y = ds.labels.cuda().contiguous()
            n_rows = dev_x.shape[0] - 32
            for rep in range(3):
                w.run_resident(64, dev_x.data_ptr(), dev_y.data_ptr(), 784 * 4, 40, n_rows, rep * 64)
                w.wait_applied()
            print_stamps(w._fx_dbg.cpu(), f"lanes={lanes}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
