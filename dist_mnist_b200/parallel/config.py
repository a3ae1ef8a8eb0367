"""Engine configuration shared by ps and worker tasks."""
from __future__ import annotations

import math
import os
import struct
from dataclasses import dataclass, asdict
from typing import Optional, Tuple

from .. import _native as N


MAX_SLOTS = 32   # executor ring depth limit (one push-sequence word per slot in the worker segment)


def _env_flag(name: str, default: bool) -> bool:
    v = os.environ.get(name)
    return default if v is None else v not in ("0", "", "false", "False")


_NATIVE_KINDS = {"adam": N.OPT_ADAM, "sgd": N.OPT_SGD, "momentum": N.OPT_MOMENTUM, "adagrad": N.OPT_ADAGRAD,
                 "rmsprop": N.OPT_RMSPROP, "adadelta": N.OPT_ADADELTA, "ftrl": N.OPT_FTRL,
                 "proximal_adagrad": N.OPT_PROXIMAL_ADAGRAD, "proximal_sgd": N.OPT_PROXIMAL_SGD,
                 "adagrad_da": N.OPT_ADAGRAD_DA}
# the kinds after Adam / SGD: their slot buffers hold other state, so ps, chief and checkpoints must agree on the kind
TF1_SLOT_KINDS = ("momentum", "adagrad", "rmsprop", "adadelta", "ftrl", "proximal_adagrad", "proximal_sgd",
                  "adagrad_da")
_PROXIMAL = ("ftrl", "proximal_adagrad", "proximal_sgd")
_L1_L2 = _PROXIMAL + ("adagrad_da",)   # the kinds with l1 / l2 regularization strengths
_FTRL_PROX_HPARAMS = ("rho", "l1_regularization_strength", "l2_regularization_strength",
                      "l2_shrinkage_regularization_strength", "learning_rate_power")
# hyper-parameters beyond lr / beta1 / beta2 / eps, the kinds that use each, and the TF1 default per kind
# (TF1's MomentumOptimizer has no default momentum; 0.9 here)
_EXTRA_DEFAULTS = {
    "momentum": {"momentum": 0.9, "rmsprop": 0.0},
    "decay": {"rmsprop": 0.9},
    "initial_accumulator_value": {"adagrad": 0.1, "ftrl": 0.1, "proximal_adagrad": 0.1, "adagrad_da": 0.1},
    "rho": {"adadelta": 0.95},
    "l1_regularization_strength": {k: 0.0 for k in _L1_L2},
    "l2_regularization_strength": {k: 0.0 for k in _L1_L2},
    "l2_shrinkage_regularization_strength": {"ftrl": 0.0},
    "learning_rate_power": {"ftrl": -0.5},
}


_NATIVE_SCHEDULES = {"constant": N.LR_CONSTANT, "exponential_decay": N.LR_EXPONENTIAL,
                     "inverse_time_decay": N.LR_INVERSE_TIME, "natural_exp_decay": N.LR_NATURAL_EXP,
                     "polynomial_decay": N.LR_POLYNOMIAL, "cosine_decay": N.LR_COSINE,
                     "piecewise_constant": N.LR_PIECEWISE}
LR_SCHEDULES = tuple(_NATIVE_SCHEDULES)
_DECAY3 = ("exponential_decay", "inverse_time_decay", "natural_exp_decay")
# schedule parameter -> the schedules that use it
SCHEDULE_PARAMS = {
    "decay_steps": _DECAY3 + ("polynomial_decay", "cosine_decay"),
    "decay_rate": _DECAY3,
    "staircase": _DECAY3,
    "end_learning_rate": ("polynomial_decay",),
    "power": ("polynomial_decay",),
    "cycle": ("polynomial_decay",),
    "alpha": ("cosine_decay",),
    "boundaries": ("piecewise_constant",),
    "values": ("piecewise_constant",),
}
_SCHEDULE_DEFAULTS = {"end_learning_rate": 1e-4, "power": 1.0, "alpha": 0.0}   # TF1's defaults


@dataclass(frozen=True)
class LrSchedule:
    """TF1's `tf.train.*_decay(learning_rate, global_step, ...)` / `piecewise_constant(global_step, ...)` on the ps.

    The rate of a push is `lr_at(s, lr0)` for the number `s` of pushes its item had already applied (the global step at
    apply time; `lr0` is the optimizer's `lr`). A parameter left at None takes TF1's default; one that the kind does not
    use is an error. The ps evaluates the rate in fp32; `lr_at` is the fp64 reference of that, rounded once to fp32."""
    kind: str = "constant"
    decay_steps: Optional[int] = None
    decay_rate: Optional[float] = None
    staircase: bool = False
    end_learning_rate: Optional[float] = None
    power: Optional[float] = None
    cycle: bool = False
    alpha: Optional[float] = None
    boundaries: Optional[Tuple[int, ...]] = None
    values: Optional[Tuple[float, ...]] = None

    def __post_init__(self):
        if self.kind not in _NATIVE_SCHEDULES:
            raise ValueError(f"unknown lr_schedule {self.kind!r} ({' | '.join(LR_SCHEDULES)})")
        for name, kinds in SCHEDULE_PARAMS.items():
            v = getattr(self, name)
            if v is not None and v is not False and self.kind not in kinds:
                raise ValueError(f"lr_schedule {self.kind!r} has no parameter {name!r}")
            if self.kind in kinds and getattr(self, name) is None and name in _SCHEDULE_DEFAULTS:
                object.__setattr__(self, name, _SCHEDULE_DEFAULTS[name])
        if self.boundaries is not None:
            object.__setattr__(self, "boundaries", tuple(int(b) for b in self.boundaries))
        if self.values is not None:
            object.__setattr__(self, "values", tuple(float(v) for v in self.values))
        k = self.kind
        if k in SCHEDULE_PARAMS["decay_steps"]:
            if self.decay_steps is None or int(self.decay_steps) != self.decay_steps or not 0 < self.decay_steps < 2 ** 32:
                raise ValueError(f"lr_schedule {k!r} needs an integer decay_steps in [1, 2^32)")
            object.__setattr__(self, "decay_steps", int(self.decay_steps))
        if k in _DECAY3 and (self.decay_rate is None or not math.isfinite(self.decay_rate)):
            raise ValueError(f"lr_schedule {k!r} needs a decay_rate")
        if k == "polynomial_decay" and not (math.isfinite(self.end_learning_rate) and math.isfinite(self.power)):
            raise ValueError("polynomial_decay needs a finite end_learning_rate and power")
        if k == "cosine_decay" and not math.isfinite(self.alpha):
            raise ValueError("cosine_decay needs a finite alpha")
        if k == "piecewise_constant":
            b, v = self.boundaries, self.values
            if not b or len(b) > N.MAX_LR_BOUNDARIES:
                raise ValueError(f"piecewise_constant needs 1..{N.MAX_LR_BOUNDARIES} boundaries")
            if any(x < 0 or x >= 2 ** 32 for x in b) or any(b[i] >= b[i + 1] for i in range(len(b) - 1)):
                raise ValueError("piecewise_constant boundaries must be strictly increasing steps in [0, 2^32)")
            if v is None or len(v) != len(b) + 1:
                raise ValueError("piecewise_constant needs len(boundaries) + 1 values")

    @property
    def native_kind(self) -> int:
        return _NATIVE_SCHEDULES[self.kind]

    @property
    def constant(self) -> bool:
        return self.kind == "constant"

    def lr_at(self, step: int, lr0: float) -> float:
        """The rate at step `step`: TF1's formula in fp64 (the step ratio is exact), rounded once to fp32."""
        s, k = int(step), self.kind
        if k == "piecewise_constant":
            i = 0
            while i < len(self.boundaries) and s > self.boundaries[i]:
                i += 1
            return _f32(self.values[i])
        if k == "constant":
            return _f32(lr0)
        d = self.decay_steps
        if k in _DECAY3:
            p = float(s // d) if self.staircase else s / d
            if k == "exponential_decay":
                r = lr0 * self.decay_rate ** p
            elif k == "inverse_time_decay":
                r = lr0 / (1.0 + self.decay_rate * p)
            else:
                r = lr0 * math.exp(-self.decay_rate * p)
        elif k == "polynomial_decay":
            if self.cycle:
                sp, dp = s, d * max(1, -(-s // d))
            else:
                sp, dp = min(s, d), d
            r = (lr0 - self.end_learning_rate) * (1.0 - sp / dp) ** self.power + self.end_learning_rate
        else:   # cosine_decay
            f = min(s, d) / d
            r = lr0 * ((1.0 - self.alpha) * 0.5 * (1.0 + math.cos(math.pi * f)) + self.alpha)
        return _f32(r)

    def fill_native(self, P) -> None:
        """Write this schedule into a PsServeParams."""
        P.lr_schedule = self.native_kind
        P.decay_steps = int(self.decay_steps or 0)
        P.decay_rate = self.decay_rate or 0.0
        P.end_lr = self.end_learning_rate or 0.0
        P.power = self.power or 0.0
        P.alpha = self.alpha or 0.0
        P.staircase, P.cycle = int(self.staircase), int(self.cycle)
        b, v = self.boundaries or (), self.values or ()
        P.n_boundaries = len(b)
        for i, x in enumerate(b):
            P.boundaries[i] = x
        for i, x in enumerate(v):
            P.values[i] = x

    def as_dict(self) -> dict:
        d = asdict(self)
        for name in ("boundaries", "values"):   # JSON-shaped (rendezvous descriptors, checkpoints)
            if d[name] is not None:
                d[name] = list(d[name])
        return d

    @classmethod
    def from_dict(cls, d: Optional[dict]) -> "LrSchedule":
        return cls(**d) if d else cls()


def _f32(x: float) -> float:
    return struct.unpack("f", struct.pack("f", x))[0]


CLIP_KINDS = ("global_norm", "norm", "value")
_NATIVE_CLIPS = {None: N.CLIP_OFF, "global_norm": N.CLIP_GLOBAL_NORM, "norm": N.CLIP_NORM, "value": N.CLIP_VALUE}
# clip parameter -> the kinds that use it
CLIP_PARAMS = {"clip_norm": ("global_norm", "norm"), "value_min": ("value",), "value_max": ("value",)}


@dataclass(frozen=True)
class GradClip:
    """Gradient clipping on the worker, between TF1's `opt.compute_gradients(loss)` and `opt.apply_gradients(...)`:
    "global_norm" is `tf.clip_by_global_norm(grads, clip_norm)`, "norm" is `tf.clip_by_norm(g, clip_norm)` applied to
    every model variable separately, "value" is `tf.clip_by_value(g, value_min, value_max)`. `kind` None = off.

    The clip applies to the gradient of the mean loss over the whole batch, the one that is pushed. The ps never sees
    it: it combines with every optimizer, schedule, moving average, apply mode and sharding. `mlp.clip_gradients` is
    the fp32 reference. A parameter the kind does not use is an error."""
    kind: Optional[str] = None
    clip_norm: Optional[float] = None
    value_min: Optional[float] = None
    value_max: Optional[float] = None

    def __post_init__(self):
        if self.kind not in _NATIVE_CLIPS:
            raise ValueError(f"unknown gradient clip {self.kind!r} ({' | '.join(CLIP_KINDS)})")
        for name, kinds in CLIP_PARAMS.items():
            v = getattr(self, name)
            if v is None:
                if self.kind in kinds:
                    raise ValueError(f"gradient clip {self.kind!r} needs {name}")
                continue
            if self.kind not in kinds:
                what = "gradient clipping is off" if self.kind is None else f"gradient clip {self.kind!r}"
                raise ValueError(f"{what}: {name} does not apply (only {', '.join(kinds)})")
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v):
                raise ValueError(f"{name} must be a finite number, got {v!r}")
            object.__setattr__(self, name, float(v))
        if self.clip_norm is not None and not self.clip_norm > 0:
            raise ValueError(f"clip_norm must be > 0, got {self.clip_norm!r}")
        if self.kind == "value" and not self.value_min <= self.value_max:
            raise ValueError(f"value_min ({self.value_min}) must not exceed value_max ({self.value_max})")

    @property
    def enabled(self) -> bool:
        return self.kind is not None

    @property
    def native_kind(self) -> int:
        return _NATIVE_CLIPS[self.kind]

    def apply(self, grads):
        """The reference clip (mlp.clip_gradients) of a {variable name: gradient} dict; unchanged when off."""
        from ..models import mlp

        return mlp.clip_gradients(grads, self) if self.enabled else grads

    def fill_native(self, P) -> None:
        """Write this clip into a FusedParams."""
        P.clip_kind = self.native_kind
        P.clip_norm = self.clip_norm or 0.0
        P.clip_min = self.value_min or 0.0
        P.clip_max = self.value_max or 0.0

    def as_dict(self) -> dict:
        return asdict(self)

    @classmethod
    def from_dict(cls, d: Optional[dict]) -> "GradClip":
        return cls(**d) if d else cls()


L2_VARIABLES = ("weights", "all")


@dataclass(frozen=True)
class L2Regularization:
    """TF1's L2 weight regularization on the worker: `loss += scale * sum(tf.nn.l2_loss(v) for v in V)` before
    `opt.compute_gradients(loss)` (equivalently `tf.contrib.layers.l2_regularizer(scale)`, or cifar10's
    `wd * l2_loss(w)`). V is every layer's weight matrix ("weights") or the weights and the biases ("all", as in the
    MNIST `convolutional.py` example). `scale` None or 0.0 = off.

    The gradient pushed for a variable in V is fl(g + fl(scale * w)), with w the variable as the step read it; gradient
    clipping applies to that sum. The ps never sees it: it combines with every optimizer, schedule, moving average,
    apply mode and sharding. `mlp.l2_regularize` is the fp32 reference."""
    scale: Optional[float] = None
    variables: str = "weights"

    def __post_init__(self):
        if self.variables not in L2_VARIABLES:
            raise ValueError(f"unknown L2 variable set {self.variables!r} ({' | '.join(L2_VARIABLES)})")
        s = self.scale
        if s is None:
            return
        if isinstance(s, bool) or not isinstance(s, (int, float)) or not math.isfinite(s) or s < 0:
            raise ValueError(f"L2 regularization scale must be a finite number >= 0, got {s!r}")
        object.__setattr__(self, "scale", float(s))

    @property
    def enabled(self) -> bool:
        return bool(self.scale)

    def apply(self, params, grads):
        """(reg_loss, grads') of the reference (mlp.l2_regularize) for {variable name: tensor} dicts; (0.0, grads)
        unchanged when off."""
        from ..models import mlp

        if not self.enabled:
            return 0.0, grads
        return mlp.l2_regularize(params, grads, self)

    def loss(self, params) -> float:
        """The regularization term scale * sum over V of l2_loss(v) (fp32 reference) of {variable name: tensor}, 0.0
        when off."""
        return float(self.apply(params, {k: v * 0 for k, v in params.items()})[0])

    def fill_native(self, P) -> None:
        """Write this regularization into a FusedParams (l2_scale 0: the unregularized kernels)."""
        P.l2_scale = self.scale or 0.0
        P.l2_biases = int(self.enabled and self.variables == "all")

    def as_dict(self) -> dict:
        return asdict(self)

    @classmethod
    def from_dict(cls, d: Optional[dict]) -> "L2Regularization":
        return cls(**d) if d else cls()


@dataclass(frozen=True)
class OptimizerConfig:
    """Reference: `tf.train.AdamOptimizer(FLAGS.learning_rate)` with TF defaults (DS:102); SGD is the
    north-star "async-SGD" variant. "momentum", "adagrad" and "rmsprop" are TF1's `MomentumOptimizer`,
    `AdagradOptimizer` and (non-centered) `RMSPropOptimizer`, applied on the ps with the `training_ops` formulas;
    "adadelta", "ftrl", "proximal_adagrad" and "proximal_sgd" likewise are `AdadeltaOptimizer`, `FtrlOptimizer` (V2
    when l2_shrinkage_regularization_strength > 0), `ProximalAdagradOptimizer` and `ProximalGradientDescentOptimizer`,
    and "adagrad_da" is `AdagradDAOptimizer`, whose global step T is the ps's count of pushes applied to each variable.
    Their l1 / l2 strengths are the ps-side terms of those optimizers, not the worker-side loss term `l2`.
    `centered` is RMSPropOptimizer(centered=True), which keeps a third slot (the mean gradient, `uses_mg`).

    A hyper-parameter left at None takes the kind's TF1 default; giving one that the kind does not use is an error."""
    kind: str = "adam"          # "adam" | "sgd" | "momentum" | "adagrad" | "rmsprop" | "adadelta" | "ftrl" |
                                # "proximal_adagrad" | "proximal_sgd" | "adagrad_da"
    lr: float = 1e-4            # --learning_rate default (DS:15)
    beta1: float = 0.9
    beta2: float = 0.999
    eps: Optional[float] = None   # Adam and Adadelta 1e-8 (also kept for the kinds without an epsilon), RMSProp 1e-10
    math: str = "fast"          # ps-side arithmetic of every rule with a square root (all but SGD, Momentum and
                                # ProximalGradientDescent; FTRL's general power too) on the
                                # cuda backend: "fast" (MUFU, <= 2 ulp, the measured configuration) | "ieee" (correctly
                                # rounded sqrt and divide, like TF's Apply* kernels; ~4x the per-push apply cost for
                                # Adam). The cpu backend is always IEEE.
    momentum: Optional[float] = None    # "momentum" (0.9), "rmsprop" (0.0)
    use_nesterov: bool = False          # "momentum"
    centered: bool = False              # "rmsprop": normalise by the variance estimate ms - mg^2 (a third slot, mg)
    decay: Optional[float] = None       # "rmsprop" (0.9)
    initial_accumulator_value: Optional[float] = None   # "adagrad", "ftrl", "proximal_adagrad", "adagrad_da" (0.1):
                                                        # the (squared) accumulator slot starts here, not at 0
    rho: Optional[float] = None                         # "adadelta" (0.95)
    l1_regularization_strength: Optional[float] = None  # "ftrl", "proximal_adagrad", "proximal_sgd", "adagrad_da" (0.0)
    l2_regularization_strength: Optional[float] = None  # the same four (0.0)
    l2_shrinkage_regularization_strength: Optional[float] = None   # "ftrl" (0.0; > 0: ApplyFtrlV2)
    learning_rate_power: Optional[float] = None         # "ftrl" (-0.5)
    schedule: LrSchedule = LrSchedule()   # learning-rate schedule over the global step (default: constant `lr`)
    # TF1 `tf.train.ExponentialMovingAverage(decay, num_updates=global_step).apply(tf.trainable_variables())`, run on
    # the ps after every optimizer step (zero_debias=False): every model variable gets a shadow that starts at the
    # variable's initial value and moves by shadow -= (shadow - p) * (1 - d). None = off.
    moving_average_decay: Optional[float] = None
    moving_average_num_updates: bool = True   # d = min(decay, (1 + n) / (10 + n)), n = global step; False: d = decay
    # gradient clipping on the worker before the push (TF1 clip_by_global_norm / clip_by_norm / clip_by_value); the
    # ps does not use it, and workers of one session may clip differently
    clip: GradClip = GradClip()
    # L2 weight regularization on the worker (TF1 scale * l2_loss(w) added to the loss); like the clip, the ps does not
    # use it, and it is part of the model's loss, not of the optimizer state a checkpoint restores
    l2: L2Regularization = L2Regularization()

    def __post_init__(self):
        if self.math not in ("fast", "ieee"):
            raise ValueError(f"unknown adam math {self.math!r} (fast | ieee)")
        if self.eps is None:
            object.__setattr__(self, "eps", 1e-10 if self.kind == "rmsprop" else 1e-8)
        for name, defaults in _EXTRA_DEFAULTS.items():
            if getattr(self, name) is None:
                object.__setattr__(self, name, defaults.get(self.kind))
            elif self.kind not in defaults:
                raise ValueError(f"optimizer {self.kind!r} has no hyper-parameter {name!r}")
        if self.use_nesterov and self.kind != "momentum":
            raise ValueError(f"use_nesterov applies to the momentum optimizer, not {self.kind!r}")
        if not isinstance(self.centered, bool):
            raise ValueError(f"centered must be a bool, got {self.centered!r}")
        if self.centered and self.kind != "rmsprop":
            raise ValueError(f"centered applies to the rmsprop optimizer, not {self.kind!r}")
        if self.kind in ("adagrad", "proximal_adagrad", "adagrad_da") and not self.initial_accumulator_value > 0:
            raise ValueError(f"initial_accumulator_value must be positive ({self.kind} divides by its square root)")
        if self.kind in ("adadelta", "adagrad_da") + _PROXIMAL or self.centered:   # every hyper-parameter finite
            for name in ("lr", "eps", "initial_accumulator_value", "momentum", "decay") + _FTRL_PROX_HPARAMS:
                x = getattr(self, name)
                if x is not None and (isinstance(x, bool) or not isinstance(x, (int, float)) or not math.isfinite(x)):
                    raise ValueError(f"{name} must be a finite number, got {x!r}")
            if self.kind in _PROXIMAL and not self.lr > 0:   # TF's Apply{Ftrl,Proximal*} kernels: "lr is not positive"
                raise ValueError(f"optimizer {self.kind!r} needs a positive learning rate, got {self.lr!r}")
        for name in ("l1_regularization_strength", "l2_regularization_strength", "l2_shrinkage_regularization_strength"):
            if getattr(self, name) is not None and getattr(self, name) < 0:
                raise ValueError(f"{name} must be >= 0, got {getattr(self, name)!r}")
        if self.kind == "ftrl":
            if self.initial_accumulator_value < 0:
                raise ValueError(f"initial_accumulator_value must be >= 0 for ftrl, got {self.initial_accumulator_value!r}")
            if self.learning_rate_power > 0:
                raise ValueError(f"learning_rate_power must be <= 0, got {self.learning_rate_power!r}")
        if not isinstance(self.schedule, LrSchedule):
            raise ValueError(f"schedule must be an LrSchedule, got {type(self.schedule).__name__}")
        if not isinstance(self.clip, GradClip):
            raise ValueError(f"clip must be a GradClip, got {type(self.clip).__name__}")
        if not isinstance(self.l2, L2Regularization):
            raise ValueError(f"l2 must be an L2Regularization, got {type(self.l2).__name__}")
        d = self.moving_average_decay
        if d is not None:
            if isinstance(d, bool) or not isinstance(d, (int, float)) or not 0.0 < d < 1.0:
                raise ValueError(f"moving_average_decay must lie in (0, 1), got {d!r}")
            object.__setattr__(self, "moving_average_decay", float(d))
        object.__setattr__(self, "moving_average_num_updates", bool(self.moving_average_num_updates))

    def lr_at(self, step: int) -> float:
        """The learning rate of a push applied at global step `step` (LrSchedule.lr_at with lr0 = lr)."""
        return self.schedule.lr_at(step, self.lr)

    @property
    def moving_averages(self) -> bool:
        return self.moving_average_decay is not None

    def ema_decay_at(self, n: int) -> float:
        """The moving-average decay of the optimizer step that brings the global step to `n` (the step included, as
        TF1's `num_updates` after the apply op the average depends on): min(decay, (1 + n) / (10 + n)) in fp64,
        rounded once to fp32 (what the ps computes in fp32), or the decay without num_updates."""
        if self.moving_average_decay is None:
            raise ValueError("moving averages are off (moving_average_decay is None)")
        d = self.moving_average_decay
        if self.moving_average_num_updates:
            n = int(n)
            d = min(d, (1.0 + n) / (10.0 + n))
        return _f32(d)

    @property
    def native_kind(self) -> int:
        if self.kind in _NATIVE_KINDS:
            return _NATIVE_KINDS[self.kind]
        raise ValueError(f"unknown optimizer {self.kind!r} ({' | '.join(_NATIVE_KINDS)})")

    @property
    def uses_mg(self) -> bool:
        """Whether the rule has the third slot buffer "mg" (centered RMSProp's mean gradient, which starts at 0)."""
        return self.kind == "rmsprop" and self.centered

    def slot_init(self) -> Tuple[float, float]:
        """Initial values of the two slot buffers (adam_m, adam_v): the accumulator of Adagrad, FTRL and
        ProximalAdagrad and AdagradDA's squared accumulator start at initial_accumulator_value and RMSProp's ms at 1
        (TF1's `ones_initializer`); every other slot (FTRL's linear, both of Adadelta's, AdagradDA's gradient
        accumulator, centered RMSProp's mg) at 0."""
        if self.kind in ("adagrad", "ftrl", "proximal_adagrad", "adagrad_da"):
            return 0.0, float(self.initial_accumulator_value)
        if self.kind == "rmsprop":
            return 0.0, 1.0
        return 0.0, 0.0

    def fill_native_rule(self, P) -> None:
        """Write the rule's hyper-parameters beyond lr / beta1 / beta2 / eps into a PsServeParams (Adadelta's rho rides
        in `decay`). The mg slot's pointer is the caller's."""
        P.momentum = self.momentum or 0.0
        P.decay = self.rho if self.kind == "adadelta" else (self.decay or 0.0)
        P.nesterov = int(self.use_nesterov)
        P.l1 = self.l1_regularization_strength or 0.0
        P.l2 = self.l2_regularization_strength or 0.0
        P.l2_shrinkage = self.l2_shrinkage_regularization_strength or 0.0
        P.lr_power = self.learning_rate_power or 0.0
        P.centered = int(self.centered)

    def as_dict(self) -> dict:
        d = asdict(self)
        d["schedule"] = self.schedule.as_dict()
        return d


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
                                     # batch <= 256, fp32) | "graph": per-layer kernels chained in a CUDA graph (any
                                     # model / dtype) | "auto": fused when the model is eligible and the batch is
                                     # <= 32 rows (any eligible batch with sharding "row_split")
    strict_steps: bool = False       # fused engine and cpu backend: a lane pulls the weights of its next step only
                                     # after the ps has acknowledged its previous push (the reference's read-your-writes
                                     # order inside one worker); default: the pull overlaps the previous step's backward
                                     # half. (The per-layer graph engine has no strict mode: use step() + wait_applied().)
    ps_row_blocks: int = 4           # fused tiling: ps items (CTAs) per pushed column slice of the hidden weight
    ps_mode: str = "persistent"      # "persistent": resident serve kernel | "oneshot": the serve kernel is launched
                                     # after the workers' kernels, applies what is pending and exits (in-process
                                     # clusters under profilers / sanitizers; `smoke()`)
    ps_ctas: int = 0                 # CTAs of the persistent PS kernel (0 = auto, ps.serve_geometry: 128 on a
                                     # dedicated ps GPU, 40 beside a worker, in clusters of <= 8 beside a
                                     # fused-engine worker; one item per CTA where possible)
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
            if not opt.schedule.constant:
                raise ValueError("push_mode='atomic' folds a constant -lr into the worker's push; a learning-rate "
                                 "schedule needs push_mode='mailbox'")
            if opt.moving_averages:
                raise ValueError("push_mode='atomic' has no ps-side apply to update moving averages after; "
                                 "moving_average_decay needs push_mode='mailbox'")
            if opt.clip.enabled:
                raise ValueError("push_mode='atomic' applies every gradient tile as it is produced, before a clip "
                                 "could know its scale; gradient clipping needs push_mode='mailbox'")
            if opt.l2.enabled:
                raise ValueError("push_mode='atomic' applies every gradient tile as it is produced (the graph engine's "
                                 "dW epilogue red.add is the apply), with no place to add the L2 term; L2 "
                                 "regularization needs push_mode='mailbox'")
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
        from .sharding import FUSED_AUTO_MAX_BATCH, FUSED_MAX_BATCH, fused_eligible

        ok = fused_eligible(spec, batch_size, self.dtype)
        if self.engine == "fused" and not ok:
            raise ValueError(f"engine 'fused' needs one hidden layer of <= 128 units, <= 11 classes, "
                             f"batch <= {FUSED_MAX_BATCH}, fp32 and 8 <= ceil(in_features / 32) <= 32")
        if self.engine == "graph" or not ok:
            if self.sharding == "row_split":
                raise ValueError("sharding 'row_split' needs the fused engine")
            return "graph"
        if self.engine == "auto" and batch_size > FUSED_AUTO_MAX_BATCH and self.sharding != "row_split":
            return "graph"   # host-fed training is not faster on the fused engine there (sharding.FUSED_AUTO_MAX_BATCH)
        return "fused"
