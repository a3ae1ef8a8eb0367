"""MLP model family of the reference, as framework-level specs plus a plain-PyTorch fp32 implementation.

Two models exist in the reference (`/root/reference/distributed_server-basic.py`):

* **book**  (live, DS:39-54):  784-H-10, `hid_w ~ TruncNormal(sigma=1/28)`, `sm_w ~ TruncNormal(sigma=1/sqrt(H))`,
  zero biases, `loss = -mean_{B x 10}(labels * log(clip(softmax(logits), 1e-10, 1)))`  (note: mean over all
  B*10 elements, i.e. per-sample cross-entropy / 10).
* **zhihu** (dead code, DS:30-36): 784-500-500-10 via `tf.layers.dense` (glorot-uniform kernels, zero biases),
  `loss = mean_B(softmax_cross_entropy_with_logits)`.

plus the bf16 784-1024-1024-10 configuration named in BASELINE.json. Everything here is generic over the
hidden-layer list. Weights are stored `[out_features, in_features]` (row-major, `in` contiguous) — the
K-major operand layout of the forward wgmma GEMM — i.e. the transpose of the reference's `[in, out]`
variables; `to_reference_layout` converts for checkpoints that want TF's orientation.

The torch implementation in this file is the numerical reference for every CUDA kernel test and the compute
path of the CPU plumbing backend; it is *not* the GPU hot path (that is `ops/` + `csrc/`).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, replace
from typing import Dict, List, Tuple

import torch

IMAGE_PIXELS = 28  # reference DS:27


@dataclass(frozen=True)
class VarSpec:
    name: str
    shape: Tuple[int, ...]  # weights: (out, in); biases: (out,)
    kind: str               # "weight" | "bias"
    layer: int              # 0-based dense layer index

    @property
    def numel(self) -> int:
        n = 1
        for s in self.shape:
            n *= s
        return n


# Activations of the hidden layers (`--activation`), TF 1.15's tf.nn functors and registered gradients. The index of a
# name is its protocol.h ActivationKind code minus one (code 0 is "none").
ACTIVATIONS = ("relu", "relu6", "leaky_relu", "elu", "selu", "sigmoid", "tanh")
LEAKY_RELU_ALPHA = 0.2                                 # tf.nn.leaky_relu's default
SELU_SCALE = 1.0507009873554804934193349852946         # TF's selu constants: scale
SELU_SCALE_ALPHA = 1.7580993408473768599402175208123   # and scale * alpha


def activation_code(name: str) -> int:
    """protocol.h ActivationKind of a hidden-layer activation (ACT_RELU = 1, ...)."""
    return ACTIVATIONS.index(name) + 1


# Losses of the classifier head (`--loss`). The index of a name is its protocol.h LossKind code. "book" is the
# reference's clipped log loss (DS:52-53), the others are TF 1.15's tf.losses functions on the logits with weight 1:
# softmax_cross_entropy, sigmoid_cross_entropy, mean_squared_error and hinge_loss.
LOSSES = ("book", "xent", "sigmoid_xent", "mse", "hinge")
SMOOTHED_LOSSES = ("xent", "sigmoid_xent")   # the losses that take a label_smoothing


def loss_code(name: str) -> int:
    """protocol.h LossKind of a loss (LOSS_BOOK = 0, LOSS_XENT = 1, ...)."""
    return LOSSES.index(name)


@dataclass(frozen=True)
class MLPSpec:
    name: str = "book"
    in_features: int = IMAGE_PIXELS * IMAGE_PIXELS
    hidden: Tuple[int, ...] = (100,)
    num_classes: int = 10
    loss: str = "book"   # one of LOSSES
    init: str = "book"   # "book" (truncated normal, DS:41-47) | "glorot" (tf.layers.dense default)
    activation: str = "relu"   # of every hidden layer, one of ACTIVATIONS (the logits layer has none)
    label_smoothing: float = 0.0   # xent / sigmoid_xent: tf.losses' label_smoothing, in [0, 1]

    def __post_init__(self):
        if self.activation not in ACTIVATIONS:
            raise ValueError(f"unknown activation {self.activation!r} (expected {' | '.join(ACTIVATIONS)})")
        if self.loss not in LOSSES:
            raise ValueError(f"unknown loss {self.loss!r} (expected {' | '.join(LOSSES)})")
        if not (math.isfinite(self.label_smoothing) and 0.0 <= self.label_smoothing <= 1.0):
            raise ValueError(f"label_smoothing must be finite and in [0, 1], got {self.label_smoothing}")
        if self.label_smoothing != 0.0 and self.loss not in SMOOTHED_LOSSES:
            raise ValueError(f"label_smoothing does not apply to loss {self.loss} (only {', '.join(SMOOTHED_LOSSES)})")

    @property
    def layer_sizes(self) -> List[Tuple[int, int]]:
        """[(in, out)] per dense layer, last one is the classifier."""
        dims = [self.in_features, *self.hidden, self.num_classes]
        return [(dims[i], dims[i + 1]) for i in range(len(dims) - 1)]

    def variable_names(self) -> List[Tuple[str, str]]:
        n = len(self.layer_sizes)
        if self.name == "book" and n == 2:
            return [("hid_w", "hid_b"), ("sm_w", "sm_b")]  # DS:41-47
        names = []
        for i in range(n):
            suffix = "" if i == 0 else f"_{i}"
            names.append((f"dense{suffix}/kernel", f"dense{suffix}/bias"))  # tf.layers.dense naming
        return names

    def variables(self) -> List[VarSpec]:
        """Trainable variables in the reference's creation order (w then b per layer)."""
        out = []
        for i, ((fin, fout), (wn, bn)) in enumerate(zip(self.layer_sizes, self.variable_names())):
            out.append(VarSpec(wn, (fout, fin), "weight", i))
            out.append(VarSpec(bn, (fout,), "bias", i))
        return out

    @property
    def num_params(self) -> int:
        return sum(v.numel for v in self.variables())

    def flops_per_step(self, batch: int) -> int:
        """fwd + bwd multiply-add FLOPs of one training step (dX of the first layer is not needed)."""
        f = 0
        for i, (fin, fout) in enumerate(self.layer_sizes):
            f += 2 * batch * fin * fout          # forward
            f += 2 * batch * fin * fout          # dW
            if i > 0:
                f += 2 * batch * fin * fout      # dX
        return f


def book_model(hidden_units: int = 100) -> MLPSpec:
    """The live model of the reference (`model_from_book_example`, DS:39-54)."""
    return MLPSpec(name="book", hidden=(hidden_units,), loss="book", init="book")


def zhihu_model() -> MLPSpec:
    """The dead-code model of the reference (`model_from_zhihu`, DS:30-36)."""
    return MLPSpec(name="zhihu", hidden=(500, 500), loss="xent", init="glorot")


def wide_model() -> MLPSpec:
    """784-1024-1024-10 configuration named in BASELINE.json (config 4, run in bf16)."""
    return MLPSpec(name="wide", hidden=(1024, 1024), loss="xent", init="glorot")


def get_model(name: str, hidden_units: int = 100, activation: str = "relu", loss: str | None = None,
              label_smoothing: float = 0.0) -> MLPSpec:
    """The model `name` with a hidden-layer activation and a loss (None: the model's own, book for book, xent for
    zhihu and wide) smoothed by `label_smoothing`."""
    if name == "book":
        spec = book_model(hidden_units)
    elif name == "zhihu":
        spec = zhihu_model()
    elif name == "wide":
        spec = wide_model()
    else:
        raise ValueError(f"unknown model {name!r} (expected book | zhihu | wide)")
    return replace(spec, activation=activation, loss=spec.loss if loss is None else loss,
                   label_smoothing=float(label_smoothing))


# ----------------------------------------------------------------------------------------------
# initialisation (SURVEY K9)
# ----------------------------------------------------------------------------------------------
def truncated_normal_(t: torch.Tensor, std: float, generator: torch.Generator | None = None) -> torch.Tensor:
    """tf.truncated_normal semantics: N(0, std) with values beyond 2 std re-drawn."""
    with torch.no_grad():
        t.normal_(0.0, 1.0, generator=generator)
        bad = t.abs() > 2.0
        while bool(bad.any()):
            redraw = torch.empty(int(bad.sum()), dtype=t.dtype, device=t.device).normal_(0.0, 1.0, generator=generator)
            t[bad] = redraw
            bad = t.abs() > 2.0
        t.mul_(std)
    return t


def init_params(spec: MLPSpec, seed: int = 0, device: str | torch.device = "cpu") -> Dict[str, torch.Tensor]:
    """fp32 initial values keyed by variable name, weights in [out, in] layout."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    params: Dict[str, torch.Tensor] = {}
    n_layers = len(spec.layer_sizes)
    for v in spec.variables():
        if v.kind == "bias":
            params[v.name] = torch.zeros(v.shape, dtype=torch.float32)
            continue
        fout, fin = v.shape
        w = torch.empty(fin, fout, dtype=torch.float32)  # drawn in the reference's [in, out] orientation
        if spec.init == "book":
            # DS:41-42: hid_w stddev 1/IMAGE_PIXELS ; DS:45-46: sm_w stddev 1/sqrt(hidden_units)
            std = 1.0 / IMAGE_PIXELS if v.layer == 0 and n_layers == 2 else 1.0 / math.sqrt(fin)
            truncated_normal_(w, std, g)
        else:
            limit = math.sqrt(6.0 / (fin + fout))  # glorot_uniform
            w.uniform_(-limit, limit, generator=g)
        params[v.name] = w.t().contiguous()
    return {k: t.to(device) for k, t in params.items()}


def to_reference_layout(params: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """[out, in] weights -> the reference's [in, out] orientation (biases unchanged)."""
    return {k: (v.t().contiguous() if v.dim() == 2 else v.clone()) for k, v in params.items()}


# ----------------------------------------------------------------------------------------------
# plain-PyTorch model (numerical reference + CPU backend compute)
# ----------------------------------------------------------------------------------------------
def activate(name: str, x: torch.Tensor) -> torch.Tensor:
    """y = f(x), TF 1.15's functor of `name`, each operation rounded in x's dtype (no fused multiply-add, exp - 1 rather
    than expm1): what every engine computes."""
    if name == "relu":
        return torch.relu(x)
    if name == "relu6":
        return torch.clamp(torch.clamp(x, min=0.0), max=6.0)
    if name == "leaky_relu":
        return torch.where(x > 0, x, LEAKY_RELU_ALPHA * x)
    if name == "elu":
        return torch.where(x < 0, torch.exp(x) - 1, x)
    if name == "selu":
        return torch.where(x < 0, SELU_SCALE_ALPHA * (torch.exp(x) - 1), SELU_SCALE * x)
    if name == "sigmoid":
        return 1 / (1 + torch.exp(-x))
    if name == "tanh":
        return torch.tanh(x)
    raise ValueError(f"unknown activation {name!r}")


def activation_grad(name: str, y: torch.Tensor, dy: torch.Tensor) -> torch.Tensor:
    """dx = dy * f'(x), computed from the layer's output y as TF's *Grad ops compute it."""
    if name == "relu":
        return dy * (y > 0).to(dy.dtype)
    if name == "relu6":
        return dy * ((y > 0) & (y < 6)).to(dy.dtype)
    if name == "leaky_relu":
        return torch.where(y > 0, dy, LEAKY_RELU_ALPHA * dy)
    if name == "elu":
        return torch.where(y < 0, dy * (y + 1), dy)
    if name == "selu":
        return torch.where(y < 0, dy * (y + SELU_SCALE_ALPHA), dy * SELU_SCALE)
    if name == "sigmoid":
        return dy * y * (1 - y)
    if name == "tanh":
        return dy * (1 - y * y)
    raise ValueError(f"unknown activation {name!r}")


def _activate_autograd(name: str, x: torch.Tensor) -> torch.Tensor:
    """torch's own activations (their autograd derivatives are independent of `activation_grad`)."""
    F = torch.nn.functional
    fns = {"relu": torch.relu, "relu6": F.relu6, "leaky_relu": lambda t: F.leaky_relu(t, LEAKY_RELU_ALPHA),
           "elu": F.elu, "selu": F.selu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}
    return fns[name](x)


def forward_logits(spec: MLPSpec, params: Dict[str, torch.Tensor], x: torch.Tensor,
                   act_fn=activate) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    """(logits, [x, hidden activations...]); `act_fn(name, z)` applies the hidden layers' activation."""
    acts = [x]
    h = x
    names = spec.variable_names()
    for i, (wn, bn) in enumerate(names):
        z = h @ params[wn].t() + params[bn]
        if i < len(names) - 1:
            h = act_fn(spec.activation, z)
            acts.append(h)
        else:
            return z, acts
    raise AssertionError("unreachable")


def smooth_labels(spec: MLPSpec, labels: torch.Tensor) -> torch.Tensor:
    """The labels the loss sees: tf.losses' label smoothing of `spec.loss`, in fp32, with ls its fp32 value:
    y' = y * fl(1 - ls) + ls / C (xent, an fp32 division) or y * fl(1 - ls) + fl(0.5 * ls) (sigmoid_xent), the constants
    formed in double as TF forms them, the multiply and the add rounded separately (so fp64 labels get the fp32 y' as
    well). ls = 0 returns the labels."""
    if spec.label_smoothing == 0.0:
        return labels
    f32 = torch.float32
    ls = torch.tensor(spec.label_smoothing, dtype=f32)
    keep = torch.tensor(1.0 - float(ls), dtype=f32)
    if spec.loss == "xent":
        add = ls / torch.tensor(float(labels.shape[-1]), dtype=f32)
    else:
        add = torch.tensor(0.5 * float(ls), dtype=f32)
    return (labels.to(f32) * keep + add).to(labels.dtype)


def _sigmoid_xent_terms(z: torch.Tensor, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(per-element loss, sigmoid(z)) of tf.nn.sigmoid_cross_entropy_with_logits: max(z, 0) - z y + log1p(exp(-|z|)),
    and the sigmoid formed from the same e = exp(-|z|) <= 1 (1 / (1 + e) for z >= 0, e / (1 + e) below), so nothing
    overflows."""
    e = torch.exp(-z.abs())
    d = 1 + e
    return torch.clamp(z, min=0.0) - z * y + torch.log1p(e), torch.where(z >= 0, 1 / d, e / d)


def loss_from_logits(spec: MLPSpec, logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """The mean loss of `spec.loss` (labels smoothed by `spec.label_smoothing`), as TF's loss tensor computes it."""
    y = smooth_labels(spec, labels)
    if spec.loss == "book":
        p = torch.softmax(logits, dim=-1)
        return -(labels * torch.log(torch.clamp(p, 1e-10, 1.0))).mean()  # DS:52-53 (mean over B x C)
    if spec.loss == "xent":
        return -(y * torch.log_softmax(logits, dim=-1)).sum(dim=-1).mean()  # DS:35
    if spec.loss == "sigmoid_xent":
        return _sigmoid_xent_terms(logits, y)[0].mean()
    if spec.loss == "mse":
        return ((logits - y) * (logits - y)).mean()
    if spec.loss == "hinge":
        return torch.relu(1 - (2 * y - 1) * logits).mean()
    raise ValueError(spec.loss)


def accuracy_count(logits: torch.Tensor, labels: torch.Tensor) -> int:
    return int((logits.argmax(dim=-1) == labels.argmax(dim=-1)).sum())


def loss_and_grads(spec: MLPSpec, params: Dict[str, torch.Tensor], x: torch.Tensor, labels: torch.Tensor):
    """Autograd reference: returns (loss, grads by name, logits)."""
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    logits, _ = forward_logits(spec, leaves, x, act_fn=_activate_autograd)
    loss = loss_from_logits(spec, logits, labels)
    grads = torch.autograd.grad(loss, list(leaves.values()))
    return loss.detach(), {k: g for k, g in zip(leaves.keys(), grads)}, logits.detach()


def manual_loss_and_grads(spec: MLPSpec, params: Dict[str, torch.Tensor], x: torch.Tensor, labels: torch.Tensor):
    """Hand-derived backward (no autograd) — the math the CUDA kernels implement, used by the CPU worker."""
    names = spec.variable_names()
    logits, acts = forward_logits(spec, params, x)
    B, Cn = logits.shape
    p = torch.softmax(logits, dim=-1)
    y = smooth_labels(spec, labels)
    k = 1.0 / (B * Cn)   # the elementwise losses' 1 / (B C)
    if spec.loss == "book":
        loss = -(labels * torch.log(torch.clamp(p, 1e-10, 1.0))).sum() * k
        passes = (p >= 1e-10) & (p <= 1.0)
        g = torch.where(passes, -k * labels / p.clamp_min(1e-38), torch.zeros_like(p))
        dz = p * (g - (g * p).sum(dim=-1, keepdim=True))
    elif spec.loss == "xent":
        loss = -(y * torch.log_softmax(logits, dim=-1)).sum(dim=-1).mean()
        dz = (p * y.sum(dim=-1, keepdim=True) - y) / B
    elif spec.loss == "sigmoid_xent":
        elem, sig = _sigmoid_xent_terms(logits, y)
        loss = elem.mean()
        dz = k * (sig - y)
    elif spec.loss == "mse":
        d = logits - y
        loss = (d * d).mean()
        dz = (2 * k) * d   # TF's SquaredDifference gradient: (2 grad)(z - y)
    elif spec.loss == "hinge":
        ypm = 2 * y - 1
        m = 1 - ypm * logits
        loss = torch.relu(m).mean()
        dz = torch.where(m > 0, (-k) * ypm, torch.zeros_like(m))
    else:
        raise ValueError(spec.loss)
    grads: Dict[str, torch.Tensor] = {}
    d = dz
    for i in range(len(names) - 1, -1, -1):
        wn, bn = names[i]
        grads[wn] = d.t() @ acts[i]
        grads[bn] = d.sum(dim=0)
        if i > 0:
            d = activation_grad(spec.activation, acts[i], d @ params[wn])
    return loss, grads, logits


def clip_gradients(grads: Dict[str, torch.Tensor], clip) -> Dict[str, torch.Tensor]:
    """TF1's gradient clipping in fp32 (the reference of every engine's clip), applied to the gradients of the mean
    loss over the whole batch, keyed by variable name. `clip` is a `parallel.config.GradClip`:

    * "global_norm" (`tf.clip_by_global_norm`): n = sqrt(sum over the variables of sum(g*g)),
      scale = clip_norm * min(1/n, 1/clip_norm) (NaN when n is inf or NaN), g' = g * scale. An unclipped step is still
      multiplied by clip_norm * fl(1/clip_norm), which need not be 1.
    * "norm" (`tf.clip_by_norm`, each variable on its own): l2 = sum(g*g), norm = sqrt(l2) if l2 > 0 else l2,
      g' = (g * clip_norm) / max(norm, clip_norm).
    * "value" (`tf.clip_by_value`): g' = max(min(g, value_max), value_min)."""
    f32 = torch.float32
    g32 = {k: g.detach().to(f32) for k, g in grads.items()}
    if clip.kind == "value":
        lo, hi = torch.tensor(clip.value_min, dtype=f32), torch.tensor(clip.value_max, dtype=f32)
        return {k: torch.maximum(torch.minimum(g, hi), lo) for k, g in g32.items()}
    c = torch.tensor(clip.clip_norm, dtype=f32)
    if clip.kind == "global_norm":
        total = torch.zeros((), dtype=f32)
        for g in g32.values():
            total = total + (g * g).sum()
        n = torch.sqrt(total)
        scale = c * torch.minimum(1.0 / n, 1.0 / c) + (n - n)
        return {k: g * scale for k, g in g32.items()}
    if clip.kind == "norm":
        out = {}
        for k, g in g32.items():
            l2 = (g * g).sum()
            norm = torch.sqrt(l2) if bool(l2 > 0) else l2
            out[k] = (g * c) / torch.maximum(norm, c)
        return out
    raise ValueError(f"unknown gradient clip {clip.kind!r}")


def l2_regularize(params: Dict[str, torch.Tensor], grads: Dict[str, torch.Tensor],
                  reg) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """TF1's L2 weight regularization in fp32 (the reference of every engine's L2 term), keyed by variable name.
    `reg` is a `parallel.config.L2Regularization` with scale S and variable set V: the weight matrices (2-D
    variables) for "weights", every variable for "all".

    Returns (reg_loss, grads'): reg_loss = S * sum over V of l2_loss(v), l2_loss(v) = sum(v*v) / 2 as in
    `tf.nn.l2_loss`, the term added to the data loss; grads' = g + fl(S * w) for a variable in V (TF's `L2LossGrad`
    followed by the ADD_N of the two gradients: the product and the sum each rounded, no FMA), g unchanged otherwise.
    `w` is the variable as the step read it (the fp32 master copy under bf16), `g` the gradient of the mean data loss
    over the whole batch."""
    f32 = torch.float32
    s = torch.tensor(reg.scale, dtype=f32)
    total = torch.zeros((), dtype=f32)
    out = {}
    for name, g in grads.items():
        g = g.detach().to(f32)
        w = params[name].detach().to(f32)
        if reg.variables == "all" or w.dim() == 2:
            total = total + (w * w).sum() / 2
            g = g + s * w
        out[name] = g
    return s * total, out
