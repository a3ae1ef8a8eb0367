"""Engine configuration shared by ps and worker tasks."""
from __future__ import annotations

import os
from dataclasses import dataclass, asdict

from .. import _native as N


MAX_SLOTS = 32   # executor ring depth limit (one push-sequence word per slot in the worker segment)


def _env_flag(name: str, default: bool) -> bool:
    v = os.environ.get(name)
    return default if v is None else v not in ("0", "", "false", "False")


@dataclass(frozen=True)
class OptimizerConfig:
    """Reference: `tf.train.AdamOptimizer(FLAGS.learning_rate)` with TF defaults (DS:102); SGD is the
    north-star "async-SGD" variant."""
    kind: str = "adam"          # "adam" | "sgd"
    lr: float = 1e-4            # --learning_rate default (DS:15)
    beta1: float = 0.9
    beta2: float = 0.999
    eps: float = 1e-8
    math: str = "fast"          # ps-side Adam arithmetic on the cuda backend: "fast" (MUFU sqrt / reciprocal, <= 2 ulp,
                                # the measured configuration) | "ieee" (correctly rounded sqrt and divide, like TF's
                                # ApplyAdam; ~4x the per-push apply cost). The cpu backend is always IEEE.

    def __post_init__(self):
        if self.math not in ("fast", "ieee"):
            raise ValueError(f"unknown adam math {self.math!r} (fast | ieee)")

    @property
    def native_kind(self) -> int:
        if self.kind == "adam":
            return N.OPT_ADAM
        if self.kind == "sgd":
            return N.OPT_SGD
        raise ValueError(f"unknown optimizer {self.kind!r} (adam | sgd)")


@dataclass(frozen=True)
class EngineConfig:
    backend: str = "cuda"            # "cuda" (sm_90a kernels over NVLink peer memory) | "cpu" (shm plumbing backend)
    dtype: str = "fp32"              # compute dtype of the dense layers: "fp32" (tf32 tensor cores) | "bf16"
    nslots: int = 2                  # mailbox slots per worker (pushes in flight before the worker waits for an ack)
    apply_mode: str = "per_push"     # "per_push" (reference semantics) | "merged"
    push_mode: str = "mailbox"       # "mailbox" (PS kernel applies; Adam or SGD) | "atomic" (SGD red.add, no PS kernel)
    sharding: str = "round_robin"    # "round_robin" (reference parity) | "byte_balanced" | "row_split" (the hidden
                                     # weight is split along its input features over every ps task; fused engine)
    engine: str = "auto"             # "fused": one persistent kernel runs whole steps (784-H-10 models, H <= 128,
                                     # batch <= 32, fp32) | "graph": per-layer kernels chained in a CUDA graph (any
                                     # model / dtype) | "auto": fused when the model is eligible
    strict_steps: bool = False       # fused engine and cpu backend: a lane pulls the weights of its next step only
                                     # after the ps has acknowledged its previous push (the reference's read-your-writes
                                     # order inside one worker); default: the pull overlaps the previous step's backward
                                     # half. (The per-layer graph engine has no strict mode: use step() + wait_applied().)
    ps_row_blocks: int = 4           # fused tiling: ps items (CTAs) per pushed column slice of the hidden weight
    ps_mode: str = "persistent"      # "persistent": resident serve kernel | "oneshot": the serve kernel is launched
                                     # after the workers' kernels, applies what is pending and exits (in-process
                                     # clusters under profilers / sanitizers; `smoke()`)
    ps_ctas: int = 0                 # CTAs of the persistent PS kernel (0 = auto: 120 on a dedicated ps GPU,
                                     # 32 when a worker shares the GPU)
    pipeline_slots: int = 0          # graph engine: worker executor ring depth (0 = auto: max(4, 2 x lanes))
    lanes: int = 1                   # steps of one worker in flight on the GPU at once. 1 = each step starts after
                                     # the previous one's kernels (reference-like); n = step i+1's pull/forward
                                     # overlaps step i's backward/push (asynchronous SGD; needs nslots >= lanes)
    graph_steps: int = 1             # steps per CUDA-graph launch in the native loops (U parallel step chains in
                                     # one graph: one input transfer + one launch per U steps); divides lanes
    pdl: bool = _env_flag("DM_PDL", True)   # programmatic dependent launch between the kernels of a step graph
    colocate: bool = False           # worker i shares GPU i with ps i (N workers on N GPUs)

    @property
    def native_dtype(self) -> int:
        if self.dtype == "fp32":
            return N.DT_F32
        if self.dtype == "bf16":
            return N.DT_BF16
        raise ValueError(f"unknown dtype {self.dtype!r} (fp32 | bf16)")

    @property
    def native_apply_mode(self) -> int:
        if self.apply_mode == "per_push":
            return N.APPLY_PER_PUSH
        if self.apply_mode == "merged":
            return N.APPLY_MERGED
        raise ValueError(f"unknown apply_mode {self.apply_mode!r}")

    def validate(self, opt: OptimizerConfig) -> None:
        if self.backend not in ("cuda", "cpu"):
            raise ValueError(f"unknown backend {self.backend!r}")
        if self.push_mode not in ("mailbox", "atomic"):
            raise ValueError(f"unknown push_mode {self.push_mode!r}")
        if self.engine not in ("auto", "fused", "graph"):
            raise ValueError(f"unknown engine {self.engine!r} (auto | fused | graph)")
        if self.ps_mode not in ("persistent", "oneshot"):
            raise ValueError(f"unknown ps_mode {self.ps_mode!r} (persistent | oneshot)")
        if self.sharding not in ("round_robin", "byte_balanced", "row_split"):
            raise ValueError(f"unknown sharding {self.sharding!r}")
        if self.ps_row_blocks < 1 or self.ps_row_blocks > 16:
            raise ValueError("ps_row_blocks must be in [1, 16]")
        if self.push_mode == "atomic":
            if opt.kind != "sgd":
                raise ValueError("push_mode='atomic' fuses the push with an SGD apply (red.add); use --optimizer sgd")
            if self.dtype != "fp32":
                raise ValueError("push_mode='atomic' updates only the fp32 master copy; use dtype fp32")
            if self.backend != "cuda":
                raise ValueError("push_mode='atomic' needs the cuda backend")
        if self.nslots < 1:
            raise ValueError("nslots must be >= 1")
        u = self.graph_steps
        if self.lanes < 1 or u < 1 or self.lanes % u != 0:
            raise ValueError("lanes must be a positive multiple of graph_steps")
        if self.push_mode == "mailbox" and self.lanes > self.nslots:
            raise ValueError("lanes (steps in flight) cannot exceed nslots (mailbox slots per worker)")
        ring = self.ring_slots
        if not (self.lanes <= ring <= MAX_SLOTS) or ring % u != 0 or (ring // u) % (self.lanes // u) != 0:
            raise ValueError(f"pipeline_slots must be <= {MAX_SLOTS}, a multiple of graph_steps, and hold a whole "
                             "number of rounds of lanes")
        _ = self.native_dtype, self.native_apply_mode, opt.native_kind

    @property
    def ring_slots(self) -> int:
        """Executor ring depth of the graph engine: `pipeline_slots`, or two rounds of lanes when left at 0."""
        return self.pipeline_slots or max(4, 2 * self.lanes)

    def as_dict(self) -> dict:
        return asdict(self)

    def resolve_engine(self, spec, batch_size: int) -> str:
        """Which step engine (and therefore which shard tiling) ps and worker tasks use. Both sides evaluate the
        same rule from the same flags; the rendezvous descriptor check catches a mismatch."""
        from .sharding import fused_eligible

        ok = fused_eligible(spec, batch_size, self.dtype)
        if self.engine == "fused" and not ok:
            raise ValueError("engine 'fused' needs one hidden layer of <= 128 units, <= 11 classes, batch <= 32, fp32 "
                             "and 8 <= ceil(in_features / 32) <= 32")
        if self.engine == "graph" or not ok:
            if self.sharding == "row_split":
                raise ValueError("sharding 'row_split' needs the fused engine")
            return "graph"
        return "fused"
