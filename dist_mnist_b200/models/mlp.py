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
from dataclasses import dataclass
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


@dataclass(frozen=True)
class MLPSpec:
    name: str = "book"
    in_features: int = IMAGE_PIXELS * IMAGE_PIXELS
    hidden: Tuple[int, ...] = (100,)
    num_classes: int = 10
    loss: str = "book"   # "book" | "xent"
    init: str = "book"   # "book" (truncated normal, DS:41-47) | "glorot" (tf.layers.dense default)

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


def get_model(name: str, hidden_units: int = 100) -> MLPSpec:
    if name == "book":
        return book_model(hidden_units)
    if name == "zhihu":
        return zhihu_model()
    if name == "wide":
        return wide_model()
    raise ValueError(f"unknown model {name!r} (expected book | zhihu | wide)")


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
def forward_logits(spec: MLPSpec, params: Dict[str, torch.Tensor], x: torch.Tensor) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    acts = [x]
    h = x
    names = spec.variable_names()
    for i, (wn, bn) in enumerate(names):
        z = h @ params[wn].t() + params[bn]
        if i < len(names) - 1:
            h = torch.relu(z)
            acts.append(h)
        else:
            return z, acts
    raise AssertionError("unreachable")


def loss_from_logits(spec: MLPSpec, logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    if spec.loss == "book":
        y = torch.softmax(logits, dim=-1)
        return -(labels * torch.log(torch.clamp(y, 1e-10, 1.0))).mean()  # DS:52-53 (mean over B x C)
    if spec.loss == "xent":
        return -(labels * torch.log_softmax(logits, dim=-1)).sum(dim=-1).mean()  # DS:35
    raise ValueError(spec.loss)


def accuracy_count(logits: torch.Tensor, labels: torch.Tensor) -> int:
    return int((logits.argmax(dim=-1) == labels.argmax(dim=-1)).sum())


def loss_and_grads(spec: MLPSpec, params: Dict[str, torch.Tensor], x: torch.Tensor, labels: torch.Tensor):
    """Autograd reference: returns (loss, grads by name, logits)."""
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    logits, _ = forward_logits(spec, leaves, x)
    loss = loss_from_logits(spec, logits, labels)
    grads = torch.autograd.grad(loss, list(leaves.values()))
    return loss.detach(), {k: g for k, g in zip(leaves.keys(), grads)}, logits.detach()


def manual_loss_and_grads(spec: MLPSpec, params: Dict[str, torch.Tensor], x: torch.Tensor, labels: torch.Tensor):
    """Hand-derived backward (no autograd) — the math the CUDA kernels implement, used by the CPU worker."""
    names = spec.variable_names()
    logits, acts = forward_logits(spec, params, x)
    B, Cn = logits.shape
    p = torch.softmax(logits, dim=-1)
    if spec.loss == "book":
        k = 1.0 / (B * Cn)
        loss = -(labels * torch.log(torch.clamp(p, 1e-10, 1.0))).sum() * k
        passes = (p >= 1e-10) & (p <= 1.0)
        g = torch.where(passes, -k * labels / p.clamp_min(1e-38), torch.zeros_like(p))
        dz = p * (g - (g * p).sum(dim=-1, keepdim=True))
    else:
        loss = -(labels * torch.log_softmax(logits, dim=-1)).sum(dim=-1).mean()
        dz = (p * labels.sum(dim=-1, keepdim=True) - labels) / B
    grads: Dict[str, torch.Tensor] = {}
    d = dz
    for i in range(len(names) - 1, -1, -1):
        wn, bn = names[i]
        grads[wn] = d.t() @ acts[i]
        grads[bn] = d.sum(dim=0)
        if i > 0:
            d = (d @ params[wn]) * (acts[i] > 0).to(d.dtype)
    return loss, grads, logits
