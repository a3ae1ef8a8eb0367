"""Command-line entry point: the reference's flag surface on the new engine.

Reference parity (`/root/reference/distributed_server-basic.py`):
  * DS:9-24    nine flags: data_dir, hidden_units, train_steps, batch_size, learning_rate, ps_hosts,
               worker_hosts, job_name, task_index — same names and types here.
  * DS:59-67   validation + echo: `job name : {}` / `task index : {}`, `ValueError('Must specify the job name
               explicitly')`, `ValueError('Must specify a valid task index')`.
  * DS:82-83   `ps`  -> `server.join()` (never returns).
  * DS:85-116  `worker` -> build replica, chief init, train until global step 4000, print every 100 steps.

Documented divergences: the three flags that are dead in the reference are live here but default to the
values the reference *effectively* uses (`--train_steps` 4000 because of the hard-coded StopAtStepHook DS:101,
`--batch_size` 32 because of `next_batch(32)` DS:111, `--data_dir` falls back to synthetic data because the
image has no network). New flags select what the reference cannot express (optimizer, model, dtype, ...).

    python -m dist_mnist_b200.cli --job_name ps --task_index 0 --ps_hosts 127.0.0.1:9910 \
        --worker_hosts 127.0.0.1:9900,127.0.0.1:9901
"""
from __future__ import annotations

import argparse
import sys
from typing import List, Optional

import torch

from .cluster import ClusterSpec, Rendezvous, default_device_index
from .models import mlp
from .parallel.config import (CLIP_KINDS, CLIP_PARAMS, L2_VARIABLES, LR_SCHEDULES, SCHEDULE_PARAMS, EngineConfig,
                              GradClip, L2Regularization, LrSchedule, OptimizerConfig)
from .parallel.ps import ParameterServer
from .parallel.worker import Worker
from .session import train_loop
from .utils import ckpt as ckpt_utils
from .utils import data as data_utils
from .utils.metrics import TrainMetricsWriter


DEFAULT_LANES = 12   # the engine's default (bench.py uses the same); --lanes 1 reproduces the reference's sequential loop


def engine_config_from_args(args, backend: str) -> EngineConfig:
    """The engine configuration every task derives from the command line (ps and worker tasks must agree)."""
    lanes = max(1, args.lanes)
    nslots = args.nslots or max(4 * lanes, 8)
    gsteps = args.graph_steps or next(u for u in (4, 3, 2, 1) if lanes % u == 0)   # largest divisor of lanes <= 4
    return EngineConfig(backend=backend, dtype=args.dtype, nslots=nslots, apply_mode=args.apply_mode,
                        push_mode=args.push_mode, sharding=args.sharding, colocate=args.colocate, lanes=lanes,
                        graph_steps=gsteps, pipeline_slots=max(4, 2 * lanes), engine=args.engine,
                        strict_steps=args.strict_steps, ps_row_blocks=args.ps_row_blocks)


# optimizer flag -> the optimizers that use it
_PROXIMAL_OPTS = ("ftrl", "proximal_adagrad", "proximal_sgd")
_OPT_FLAGS = {"momentum": ("momentum", "rmsprop"), "use_nesterov": ("momentum",), "rmsprop_decay": ("rmsprop",),
              "initial_accumulator_value": ("adagrad", "ftrl", "proximal_adagrad"),
              "epsilon": ("adam", "rmsprop", "adadelta"), "rho": ("adadelta",),
              "l1_regularization_strength": _PROXIMAL_OPTS, "l2_regularization_strength": _PROXIMAL_OPTS,
              "l2_shrinkage_regularization_strength": ("ftrl",), "learning_rate_power": ("ftrl",)}


# learning-rate schedule flag -> LrSchedule parameter
_SCHED_FLAGS = {"decay_steps": "decay_steps", "decay_rate": "decay_rate", "staircase": "staircase",
                "end_learning_rate": "end_learning_rate", "power": "power", "cycle": "cycle", "alpha": "alpha",
                "lr_boundaries": "boundaries", "lr_values": "values"}


class _StoreLearningRate(argparse.Action):
    """--learning_rate, remembering that it was given (piecewise_constant takes its rates from --lr_values)."""

    def __call__(self, parser, namespace, values, option_string=None):
        setattr(namespace, self.dest, values)
        namespace.learning_rate_given = True


def _int_list(text: str):
    return tuple(int(x) for x in text.split(",") if x.strip())


def _float_list(text: str):
    return tuple(float(x) for x in text.split(",") if x.strip())


def lr_schedule_from_args(args) -> LrSchedule:
    """The learning-rate schedule of `--lr_schedule` and its parameters; a parameter flag the chosen schedule does not
    use is an error, and so is --learning_rate with piecewise_constant."""
    kind = args.lr_schedule
    given = {flag: getattr(args, flag) for flag in _SCHED_FLAGS
             if getattr(args, flag) is not None and getattr(args, flag) is not False}
    for flag in given:
        name = _SCHED_FLAGS[flag]
        if kind not in SCHEDULE_PARAMS[name]:
            raise ValueError(f"--{flag} does not apply to --lr_schedule {kind} "
                             f"(only {', '.join(SCHEDULE_PARAMS[name])})")
    if kind == "piecewise_constant" and getattr(args, "learning_rate_given", False):
        raise ValueError("--lr_schedule piecewise_constant takes its rates from --lr_values, not --learning_rate")
    return LrSchedule(kind, **{_SCHED_FLAGS[flag]: v for flag, v in given.items()})


# gradient-clip flag -> GradClip parameter
_CLIP_FLAGS = {"clip_norm": "clip_norm", "clip_value_min": "value_min", "clip_value_max": "value_max"}


def grad_clip_from_args(args) -> GradClip:
    """The gradient clip of `--clip_gradients` and its parameters; a parameter flag the chosen kind does not use, or any
    of them without --clip_gradients, is an error."""
    kind = args.clip_gradients
    given = {flag: getattr(args, flag) for flag in _CLIP_FLAGS if getattr(args, flag) is not None}
    for flag in given:
        kinds = CLIP_PARAMS[_CLIP_FLAGS[flag]]
        if kind is None:
            raise ValueError(f"--{flag} needs --clip_gradients (gradient clipping is off)")
        if kind not in kinds:
            raise ValueError(f"--{flag} does not apply to --clip_gradients {kind} (only {', '.join(kinds)})")
    return GradClip(kind, **{_CLIP_FLAGS[flag]: v for flag, v in given.items()})


def l2_regularization_from_args(args) -> L2Regularization:
    """The L2 weight regularization of `--l2_regularization` and `--l2_variables`; the second without the first is an
    error."""
    if args.l2_variables is not None and args.l2_regularization is None:
        raise ValueError("--l2_variables needs --l2_regularization (L2 regularization is off)")
    return L2Regularization(args.l2_regularization, args.l2_variables or "weights")


def optimizer_config_from_args(args) -> OptimizerConfig:
    """The optimizer every task derives from the command line; a hyper-parameter flag the chosen optimizer does not
    use is an error."""
    for flag, kinds in _OPT_FLAGS.items():
        if getattr(args, flag) not in (None, False) and args.optimizer not in kinds:
            raise ValueError(f"--{flag} does not apply to --optimizer {args.optimizer} (only {', '.join(kinds)})")
    if args.moving_average_num_updates is not None and args.moving_average_decay is None:
        raise ValueError("--moving_average_num_updates needs --moving_average_decay (moving averages are off)")
    return OptimizerConfig(args.optimizer, args.learning_rate, eps=args.epsilon, math=args.adam_math,
                           momentum=args.momentum, use_nesterov=args.use_nesterov, decay=args.rmsprop_decay,
                           initial_accumulator_value=args.initial_accumulator_value, rho=args.rho,
                           l1_regularization_strength=args.l1_regularization_strength,
                           l2_regularization_strength=args.l2_regularization_strength,
                           l2_shrinkage_regularization_strength=args.l2_shrinkage_regularization_strength,
                           learning_rate_power=args.learning_rate_power,
                           schedule=lr_schedule_from_args(args),
                           moving_average_decay=args.moving_average_decay,
                           moving_average_num_updates=args.moving_average_num_updates != "none",
                           clip=grad_clip_from_args(args), l2=l2_regularization_from_args(args))


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(prog="distributed_server-basic", description=__doc__,
                                formatter_class=argparse.RawDescriptionHelpFormatter)
    # ---- the reference's flags (DS:11-24) ----
    p.add_argument("--data_dir", type=str, default=None, help="Directory for mnist data (idx files); synthetic if absent")
    p.add_argument("--hidden_units", type=int, default=100)
    p.add_argument("--train_steps", type=int, default=4000,
                   help="stop at this *global* step (reference: flag default 10000 is dead, hook hard-codes 4000)")
    p.add_argument("--batch_size", type=int, default=32,
                   help="per-worker batch (reference: flag default 100 is dead, next_batch(32) is hard-coded)")
    p.add_argument("--learning_rate", type=float, default=0.0001, action=_StoreLearningRate)
    p.add_argument("--ps_hosts", type=str, default=None)
    p.add_argument("--worker_hosts", type=str, default=None)
    p.add_argument("--job_name", type=str, default=None, help="worker or ps")
    p.add_argument("--task_index", type=int, default=None)
    # ---- new-engine flags ----
    p.add_argument("--optimizer", choices=["adam", "sgd", "momentum", "adagrad", "rmsprop", "adadelta", "ftrl",
                                           "proximal_adagrad", "proximal_sgd"], default="adam",
                   help="reference uses Adam (DS:102); momentum / adagrad / rmsprop / adadelta / ftrl / "
                        "proximal_adagrad / proximal_sgd are TF1's MomentumOptimizer, AdagradOptimizer, (non-centered) "
                        "RMSPropOptimizer, AdadeltaOptimizer, FtrlOptimizer, ProximalAdagradOptimizer and "
                        "ProximalGradientDescentOptimizer, applied on the ps")
    p.add_argument("--adam_math", choices=["fast", "ieee"], default="fast",
                   help="ps-side arithmetic of every optimizer with a square root or a power (cuda): MUFU "
                        "sqrt/reciprocal/power (default) or correctly rounded like TF's Apply* kernels")
    # optimizer hyper-parameters: unset = the chosen optimizer's TF1 default; one it does not use is an error
    p.add_argument("--momentum", type=float, default=None, help="momentum (0.9) and rmsprop (0.0)")
    p.add_argument("--use_nesterov", action="store_true", help="momentum: Nesterov momentum")
    p.add_argument("--rmsprop_decay", type=float, default=None, help="rmsprop: decay of the mean square (0.9)")
    p.add_argument("--initial_accumulator_value", type=float, default=None,
                   help="adagrad, ftrl and proximal_adagrad: starting value of the accumulator (0.1)")
    p.add_argument("--epsilon", type=float, default=None, help="adam (1e-8), rmsprop (1e-10) and adadelta (1e-8)")
    p.add_argument("--rho", type=float, default=None, help="adadelta: decay of both accumulators (0.95)")
    p.add_argument("--l1_regularization_strength", type=float, default=None,
                   help="ftrl, proximal_adagrad and proximal_sgd: l1 strength of the ps-side proximal step, which "
                        "sets weights to exact zeros (0.0)")
    p.add_argument("--l2_regularization_strength", type=float, default=None,
                   help="ftrl, proximal_adagrad and proximal_sgd: l2 strength of the ps-side proximal step (0.0). This "
                        "is the optimizer's own term, not the worker-side --l2_regularization loss term; both may be "
                        "given")
    p.add_argument("--l2_shrinkage_regularization_strength", type=float, default=None,
                   help="ftrl: magnitude shrinkage added to the gradient, TF's FTRL V2 (0.0: off)")
    p.add_argument("--learning_rate_power", type=float, default=None,
                   help="ftrl: power of the per-coordinate rate, <= 0 (-0.5)")
    # learning-rate schedule over the global step (TF1's tf.train.*_decay / piecewise_constant), evaluated on the ps
    # when a push is applied; a parameter flag the schedule does not use is an error
    p.add_argument("--lr_schedule", choices=list(LR_SCHEDULES), default="constant",
                   help="rate of a push at global step s, from lr0 = --learning_rate (constant: lr0)")
    p.add_argument("--decay_steps", type=int, default=None,
                   help="exponential / inverse_time / natural_exp / polynomial / cosine decay (required)")
    p.add_argument("--decay_rate", type=float, default=None,
                   help="exponential_decay / inverse_time_decay / natural_exp_decay (required)")
    p.add_argument("--staircase", action="store_true",
                   help="exponential / inverse_time / natural_exp decay: decay at whole multiples of decay_steps")
    p.add_argument("--end_learning_rate", type=float, default=None, help="polynomial_decay (1e-4)")
    p.add_argument("--power", type=float, default=None, help="polynomial_decay (1.0)")
    p.add_argument("--cycle", action="store_true", help="polynomial_decay: restart past decay_steps")
    p.add_argument("--alpha", type=float, default=None, help="cosine_decay: final rate as a fraction of lr0 (0.0)")
    p.add_argument("--lr_boundaries", type=_int_list, default=None,
                   help="piecewise_constant: 1..8 increasing global steps, e.g. 1000,2000")
    p.add_argument("--lr_values", type=_float_list, default=None,
                   help="piecewise_constant: one rate more than boundaries, e.g. 0.1,0.01,0.001")
    # TF1's ExponentialMovingAverage of every model variable, updated on the ps after each optimizer step and saved
    # in checkpoints (utils/ckpt.load_variables(..., moving_averages=True) reads them back)
    p.add_argument("--moving_average_decay", type=float, default=None,
                   help="keep moving averages of the variables with this decay, in (0, 1), e.g. 0.9999 (unset: off)")
    p.add_argument("--moving_average_num_updates", choices=["global_step", "none"], default=None,
                   help="global_step (default): decay = min(D, (1 + step) / (10 + step)), TF1's num_updates=global_step;"
                        " none: decay = D")
    # gradient clipping on the worker before the push (TF1's compute_gradients -> clip_by_* -> apply_gradients)
    p.add_argument("--clip_gradients", choices=list(CLIP_KINDS), default=None,
                   help="global_norm: tf.clip_by_global_norm; norm: tf.clip_by_norm per variable; value: "
                        "tf.clip_by_value (unset: off; fused engine and cpu backend)")
    p.add_argument("--clip_norm", type=float, default=None, help="global_norm / norm (required): finite, > 0")
    p.add_argument("--clip_value_min", type=float, default=None, help="value (required): finite, <= --clip_value_max")
    p.add_argument("--clip_value_max", type=float, default=None, help="value (required): finite")
    # L2 weight regularization on the worker (TF1's loss + S * sum(tf.nn.l2_loss(v))), before the clip
    p.add_argument("--l2_regularization", type=float, default=None,
                   help="scale S of the L2 term added to the loss and S * w to the gradient: finite, >= 0 "
                        "(unset or 0: off)")
    p.add_argument("--l2_variables", choices=list(L2_VARIABLES), default=None,
                   help="weights (default): every layer's weight matrix; all: the weights and the biases")
    p.add_argument("--model", choices=["book", "zhihu", "wide"], default="book")
    p.add_argument("--dtype", choices=["fp32", "bf16"], default="fp32")
    p.add_argument("--backend", choices=["auto", "cuda", "cpu"], default="auto")
    p.add_argument("--push_mode", choices=["mailbox", "atomic"], default="mailbox")
    p.add_argument("--apply_mode", choices=["per_push", "merged"], default="per_push")
    p.add_argument("--sharding", choices=["round_robin", "byte_balanced", "row_split"], default="round_robin",
                   help="variable -> ps placement: round_robin = the reference's replica_device_setter; row_split also "
                        "splits the hidden weight along its input features over every ps task (fused engine)")
    p.add_argument("--engine", choices=["auto", "fused", "graph"], default="auto",
                   help="fused: one persistent kernel runs whole steps (784-H-10, H <= 128, batch <= 256, fp32); "
                        "graph: per-layer kernels in a CUDA graph (any model / dtype); auto: fused for eligible "
                        "models up to batch 32 (any eligible batch with --sharding row_split), graph otherwise")
    p.add_argument("--nslots", type=int, default=0, help="mailbox slots per worker (0 = max(4 x lanes, 8))")
    p.add_argument("--lanes", type=int, default=DEFAULT_LANES,
                   help="steps of this worker in flight at once: bounded-staleness asynchronous SGD inside one worker "
                        "(1 = strictly one step after the other, like the reference's sess.run loop)")
    p.add_argument("--strict_steps", action="store_true",
                   help="fused engine: pull the weights of a lane's next step only after the ps acknowledged its "
                        "previous push (with --lanes 1: exactly the reference's read-your-writes order)")
    p.add_argument("--graph_steps", type=int, default=0,
                   help="graph engine: steps per CUDA-graph launch in the native train loop (0 = min(lanes, 4))")
    p.add_argument("--ps_row_blocks", type=int, default=4,
                   help="fused tiling: ps items (serve-kernel CTAs) per pushed column slice of the hidden weight")
    p.add_argument("--checkpoint_dir", type=str, default=None, help="chief checkpoints here (default: mkdtemp, DS:106)")
    p.add_argument("--save_checkpoint_secs", type=float, default=600.0)
    p.add_argument("--gpu", type=int, default=None, help="CUDA device for this task (default: ps k -> k, worker i -> num_ps+i)")
    p.add_argument("--colocate", action="store_true", help="worker i shares GPU i with ps i")
    p.add_argument("--log_every", type=int, default=100)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--metrics_file", type=str, default=None,
                   help="worker: append one JSON line per --log_every local steps (loss, batch accuracy, steps/sec)")
    p.add_argument("--log_steps_per_sec", action="store_true",
                   help="worker: also print the reference's implicit StepCounterHook line (global_step/sec)")
    p.add_argument("--worker_timeout", type=float, default=0.0,
                   help="ps: declare a worker dead after this many seconds without a heartbeat and stop waiting for "
                        "it (0 = never, like the reference)")
    p.add_argument("--inject_fault", type=int, default=0,
                   help="worker: crash (os._exit) after this many local steps — fault-injection hook for tests")
    p.add_argument("--chunk_sleep", type=float, default=0.0,
                   help="worker: sleep this many seconds after every chunk of 50 steps — slows a worker down (tests of "
                        "the failure / restart path need a run that outlives a crash and a restart)")
    p.add_argument("--ps_exit_when_done", action="store_true",
                   help="let a ps task return once every worker has finished (reference ps blocks forever)")
    p.add_argument("--rendezvous_timeout", type=float, default=300.0)
    return p


def validate_task(job_name: Optional[str], task_index: Optional[int]) -> None:
    """Exact reference behaviour of DS:59-67."""
    if job_name is not None and len(job_name) > 0:
        print("job name : {}".format(job_name))
    else:
        raise ValueError("Must specify the job name explicitly")
    if task_index is not None and task_index >= 0:
        print("task index : {}".format(task_index))
    else:
        raise ValueError("Must specify a valid task index")


def resolve_backend(name: str) -> str:
    if name == "auto":
        return "cuda" if torch.cuda.is_available() else "cpu"
    return name


def run(args: argparse.Namespace) -> int:
    validate_task(args.job_name, args.task_index)
    cluster = ClusterSpec.from_flags(args.ps_hosts, args.worker_hosts)
    if args.job_name not in ("ps", "worker"):
        # the reference silently does nothing for other job names (neither branch DS:82/85 fires) after starting
        # a server that fails for an unknown job; be explicit instead.
        raise ValueError(f"unknown job name {args.job_name!r} (expected 'ps' or 'worker')")
    cluster.task_endpoint(args.job_name, args.task_index)
    backend = resolve_backend(args.backend)
    spec = mlp.get_model(args.model, args.hidden_units)
    opt = optimizer_config_from_args(args)
    cfg = engine_config_from_args(args, backend)
    cfg.validate(opt)
    device = -1
    if backend == "cuda":
        n_dev = torch.cuda.device_count()
        device = args.gpu if args.gpu is not None else default_device_index(
            cluster, args.job_name, args.task_index, n_dev, args.colocate)
    rdv = Rendezvous(cluster, args.job_name, args.task_index, timeout_s=args.rendezvous_timeout)

    if args.job_name == "ps":
        ps = ParameterServer(cluster, args.task_index, spec, opt, cfg, device=device, rdv=rdv,
                             batch_size=args.batch_size)
        ps.start()
        try:
            # DS:83 — blocks forever unless asked otherwise
            ps.join(exit_when_done=args.ps_exit_when_done, worker_timeout_s=args.worker_timeout)
        except KeyboardInterrupt:
            pass
        finally:
            try:
                print(f"[ps {args.task_index}] exiting: global_step={ps.global_step()} "
                      f"owns_global_step={int(ps.shard.owns_global_step)} items={ps.shard.n_items}", flush=True)
            except Exception:
                pass
            ps.close()
        return 0

    worker = Worker(cluster, args.task_index, spec, opt, cfg, batch_size=args.batch_size, device=device, rdv=rdv)
    dataset = data_utils.get_dataset(args.data_dir, seed=args.seed)  # DS:69 (every worker holds the full set)
    worker.connect()
    if worker.is_chief:
        if worker.variables_are_live():
            # a restarted chief (incarnation > 1): the ps tasks still hold the live training state the other workers
            # keep updating — re-running the initialisers (or restoring an older checkpoint) would reset parameters
            # and Adam slots under them while global_step and the per-item step counts keep running
            print(f"[worker 0] restarted (incarnation {worker.incarnation}): variables are live on the ps, "
                  f"not re-initialising", flush=True)
        else:
            restored = ckpt_utils.restore_latest(worker, args.checkpoint_dir)
            if restored is None:
                worker.initialize_variables(seed=args.seed)
            else:
                worker.mark_initialized()
    worker.wait_ready()
    metrics = None
    if args.metrics_file or args.log_steps_per_sec:
        metrics = TrainMetricsWriter(args.metrics_file, args.task_index, args.batch_size,
                                     every_steps=max(1, args.log_every), echo=args.log_steps_per_sec,
                                     lr_at=None if opt.schedule.constant else opt.lr_at)
    try:
        res = train_loop(worker, dataset, train_steps=args.train_steps, log_every=args.log_every,
                         checkpoint_dir=args.checkpoint_dir, save_checkpoint_secs=args.save_checkpoint_secs,
                         seed=args.seed, inject_fault_after=args.inject_fault, metrics=metrics,
                         chunk_sleep_s=args.chunk_sleep)
        print(f"[worker {args.task_index}] done: local_steps={res.steps_run} last_global_step={res.last_global_step} "
              f"engine={worker.engine}", flush=True)
    finally:
        if metrics is not None:
            metrics.close()
        worker.close()
    return 0


def main(argv: Optional[List[str]] = None) -> int:
    args = build_parser().parse_args(argv)
    return run(args)


if __name__ == "__main__":
    sys.exit(main())
