"""Checkpoint / resume of the parameter-server state.

Reference parity: the chief's `MonitoredTrainingSession` owns a default `CheckpointSaverHook` that writes
all PS-resident variables (model, Adam slots, beta powers, `global_step`) to `checkpoint_dir` every 600 s and
at the end, and restores the latest checkpoint found there at session start
(/root/reference/distributed_server-basic.py:106-109; `checkpoint_dir = tempfile.mkdtemp()` makes resume
impossible in practice there — here `--checkpoint_dir` can be given, default stays a temp dir).

The chief reads the shards through peer memory (X6 in SURVEY.md): the PS task itself is not involved.
Files: `<dir>/model.ckpt-<global_step>.pt` plus a TF-style `<dir>/checkpoint` index naming the latest one.
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import torch

from ..parallel.config import TF1_SLOT_KINDS

FORMAT_VERSION = 1


def save_checkpoint(worker, directory: str) -> str:
    os.makedirs(directory, exist_ok=True)
    worker.wait_applied()  # our own pushes are in; other workers may still race (Hogwild, as in the reference)
    gstep = worker.read_global_step()
    state = {
        "format_version": FORMAT_VERSION,
        "model": worker.spec.name,
        "hidden": tuple(worker.spec.hidden),
        "global_step": gstep,
        "optimizer": {"kind": worker.opt.kind, "lr": worker.opt.lr, "beta1": worker.opt.beta1,
                      "beta2": worker.opt.beta2, "eps": worker.opt.eps, "momentum": worker.opt.momentum,
                      "use_nesterov": worker.opt.use_nesterov, "decay": worker.opt.decay,
                      "initial_accumulator_value": worker.opt.initial_accumulator_value,
                      "rho": worker.opt.rho,
                      "l1_regularization_strength": worker.opt.l1_regularization_strength,
                      "l2_regularization_strength": worker.opt.l2_regularization_strength,
                      "l2_shrinkage_regularization_strength": worker.opt.l2_shrinkage_regularization_strength,
                      "learning_rate_power": worker.opt.learning_rate_power,
                      "schedule": worker.opt.schedule.as_dict(),
                      "moving_average_decay": worker.opt.moving_average_decay,
                      "moving_average_num_updates": worker.opt.moving_average_num_updates},
        "variables": worker.read_variables("params"),       # [out, in] layout, see models/mlp.py
        "adam_m": worker.read_variables("adam_m"),
        "adam_v": worker.read_variables("adam_v"),
        "item_state": {k: worker.read_item_state(k) for k in range(worker.cluster.num_ps)},
        "sharding": worker.cfg.sharding,
        "num_ps": worker.cluster.num_ps,
        "dw_tile_n": worker.layout.dw_tile_n,    # item tables (hence item_state) depend on the dW tile width
    }
    if worker.opt.moving_averages:   # the shadow variables (TF1 saves `<var>/ExponentialMovingAverage`)
        state["ema"] = worker.read_variables("ema")
    name = f"model.ckpt-{gstep}.pt"
    path = os.path.join(directory, name)
    tmp = path + ".tmp"
    torch.save(state, tmp)
    os.replace(tmp, path)
    index = os.path.join(directory, "checkpoint")   # TF-style index file, replaced atomically like the checkpoint itself
    with open(index + ".tmp", "w") as f:
        f.write(f'model_checkpoint_path: "{name}"\n')
    os.replace(index + ".tmp", index)
    return path


def latest_checkpoint(directory: Optional[str]) -> Optional[str]:
    if not directory:
        return None
    index = os.path.join(directory, "checkpoint")
    if not os.path.exists(index):
        return None
    with open(index) as f:
        line = f.readline().strip()
    if not line.startswith("model_checkpoint_path:"):
        return None
    name = line.split(":", 1)[1].strip().strip('"')
    path = os.path.join(directory, name)
    return path if os.path.exists(path) else None


def restore_latest(worker, directory: Optional[str]) -> Optional[int]:
    """Chief-side restore into the PS shards. Returns the restored global step, or None if nothing to restore."""
    path = latest_checkpoint(directory)
    if path is None:
        return None
    state = torch.load(path, map_location="cpu", weights_only=False)
    if state.get("format_version") != FORMAT_VERSION:
        raise RuntimeError(f"unsupported checkpoint format in {path}")
    if tuple(state["hidden"]) != tuple(worker.spec.hidden):
        raise RuntimeError(f"checkpoint {path} is for hidden={state['hidden']}, model has {worker.spec.hidden}")
    # adam_m / adam_v hold a different optimizer's state under every kind but Adam and SGD (TF fails on the missing
    # slot variables in this case); only the kind is read, so checkpoints without the later hyper-parameters restore
    kind = state.get("optimizer", {}).get("kind")
    if kind != worker.opt.kind and (kind in TF1_SLOT_KINDS or worker.opt.kind in TF1_SLOT_KINDS):
        raise RuntimeError(f"checkpoint {path} holds {kind!r} optimizer slots, this run uses {worker.opt.kind!r}")
    # moving averages: restored when this run keeps them (TF1's Saver restores only the variables its graph has, so
    # saved shadows are ignored without them), and a run that keeps them cannot start from a checkpoint without them
    # (TF1 fails on the missing `.../ExponentialMovingAverage` variables)
    if worker.opt.moving_averages and "ema" not in state:
        raise RuntimeError(f"checkpoint {path} has no moving averages, this run keeps them "
                           f"(moving_average_decay={worker.opt.moving_average_decay})")
    worker.write_variables(state["variables"], "params")
    worker.write_variables(state["adam_m"], "adam_m")
    worker.write_variables(state["adam_v"], "adam_v")
    if worker.opt.moving_averages:
        worker.write_variables(state["ema"], "ema")
    # per-item optimizer state (Adam step count / beta powers) is only meaningful for the same item table; with a
    # different shard count, placement or dW tile width the variables and Adam slots are restored and the
    # per-item step counters restart (bias correction re-warms, as after a TF slot-variable reset)
    if (state.get("num_ps") == worker.cluster.num_ps and state.get("sharding") == worker.cfg.sharding
            and state.get("dw_tile_n", 64) == worker.layout.dw_tile_n):
        for k, st in state["item_state"].items():
            worker.write_item_state(int(k), st)
    # the learning-rate schedule continues at the restored global_step on every item, whether or not the item state
    # was restored (TF1 evaluates it from global_step; like TF1 the schedule itself may change across a restore)
    worker.set_sched_step(int(state["global_step"]))
    worker.write_global_step(int(state["global_step"]))
    return int(state["global_step"])


def load_variables(path: str, moving_averages: bool = False) -> Dict[str, torch.Tensor]:
    """The model variables of a checkpoint file (or of the latest checkpoint of a directory), by name in the [out, in]
    layout of models/mlp.py, for evaluating a finished run offline. `moving_averages`: the shadow variables instead,
    as TF1's `saver = tf.train.Saver(ema.variables_to_restore())` loads them into the model variables."""
    if os.path.isdir(path):
        latest = latest_checkpoint(path)
        if latest is None:
            raise FileNotFoundError(f"no checkpoint in {path}")
        path = latest
    state = torch.load(path, map_location="cpu", weights_only=False)
    if state.get("format_version") != FORMAT_VERSION:
        raise RuntimeError(f"unsupported checkpoint format in {path}")
    if not moving_averages:
        return state["variables"]
    if "ema" not in state:
        raise RuntimeError(f"checkpoint {path} has no moving averages (the run had no moving_average_decay)")
    return state["ema"]
