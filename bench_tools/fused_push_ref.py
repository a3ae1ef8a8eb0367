"""Element-wise check of a worker step's pushed gradient against fp64, for the fused step kernel
(csrc/fused_step_sm90.cu) and the graph engine (gemm_sm90.cu + head_sm90.cu).

Inputs that tf32 cannot round
-----------------------------
Both engines feed fp32 bits to `wgmma ... .tf32`, which reads the top 19 bits of each operand. The case builder makes
both operands of the forward GEMM exact in tf32: x holds values k/256 (k = 0..255, 8 significant bits, sparse like
MNIST) and the hidden weight W is `mlp.init_params(...)["hid_w"]` with its low 13 mantissa bits cleared. Every product
of the forward is then exact whether the hardware truncates or rounds, and only fp32 accumulation error is left. The
one tf32 conversion left in a step is dpre = (dlogits . W_last) * relu', the operand of the dW GEMM that x multiplies.

The bound
---------
`reference` computes the step in fp64 (`mlp.manual_loss_and_grads` on the same inputs) and a per-element bound on
|pushed - reference| for the four variables, and bounds for the loss and the correct count. Below, u = 2^-24 (fp32
unit roundoff), k the loss normalisation (1 / (B C) for the book loss, 1 / B for xent), and all |.| products are in fp64.

* Forward: pre = x W^T + b. Each CTA sums <= 128 exact products in the tensor core's fp32 accumulator, then 8 partials
  and the bias are added in fp32. A truncating accumulator errs by <= 2 ulp per k8 MMA, all with the same sign: <= 16 *
  2 + 8 + 1 ulp of the magnitude A = |x| |W|^T + |b|, i.e. < 2^-17 A = EPS_FWD A =: band. That bounds |pre_kernel -
  pre| and, ReLU being 1-Lipschitz, the error of every hidden activation hv. Pairs (b, j) with |pre_bj| <= AMBIG A
  (AMBIG = 2^-14, 8x wider: a wider band costs nothing but a few more ambiguous pairs) are *ambiguous*: the kernel may
  take either ReLU branch there.
* Logits: z = hv W_last^T + b_last in fp32 FMAs over <= 128 terms: dz_bc = band_b . |W_last_c| + EPS_F (hv_b . |W_last_c|
  + |b_last_c|), with EPS_F = 2^-16 = 256 u for every fp32 sum of at most a few hundred terms (worst case H u = 2^-17
  for H = 128; the sums of the small gradients run over <= 256 rows and 8 partials in a fixed order). dz_b = max_c dz_bc.
* Softmax: p_c = __expf(z_c - zmax) / esum (`__fdividef` in the fused kernel, IEEE division in the graph head). CUDA's
  documented maximum errors: __expf(t) <= 2 + floor(1.173 |t|) ulp, __fdividef <= 2 ulp, __logf <= 2^-21.41 absolute
  on [0.5, 2] and <= 3 ulp elsewhere. With e_c's relative error ee_c = (2 + 1.173 |z_c - zmax|) 2^-23 the rounding
  part of p_c's relative error is ep_c = ee_c + sum_c' p_c' ee_c' + 16 u + 2^-22 (the sum of <= 16 terms and the
  division); the logit error adds |dp_c| <= 2 p_c dz_b to first order. So |dp_c| <= p_c (2 dz_b + ep_c) (the 2^-20 per
  row in EXP_SLACK covers the second-order terms and fl(z - zmax)).
* dlogits: for one-hot labels both losses give dl = k (p - y), except that the book loss's clamp zeroes a row whose
  true-class p is below 1e-10 (no other p meets the clamp: y = 0 there). The kernel's dl (book: p (g - sum g p) with
  g = -k y / p; xent: k (p sum(y) - y)) has a cancellation where p_true is near 1, so its rounding is absolute:
  E_bc = k (p_c (2 dz_b + ep_c) + EPS_F (p_c + y_c)). Rows are asserted to keep p_true outside [1e-10 / 2, 2e-10],
  so the clamp branch is the same in both (`check_case`).
* dh = dl . W_last (FMAs over 16 classes): ddh_bj = sum_c E_bc |W_last_cj| + EPS_F sum_c |dl_bc| |W_last_cj|; the
  error of dpre_bj is ddh_bj where the unit is active, 0 where it is inactive, and |dh_bj| + ddh_bj where it is
  ambiguous. Call that ddp_bj.
* hid_w: dW = dpre^T x, dpre converted to tf32 (relative error < 2^-10 truncated, <= 2^-11 rounded to nearest) and x
  exact: |dW - ref| <= TF32 (|dpre|^T |x|) + ((1 + TF32) ddp + EPS_F |dpre|)^T |x|, TF32 = 2^-9 (2x the truncation
  error). Over the shape matrix the fp32 terms are a median 0.07-0.35 of the tf32 term (mostly the worst-case sum of
  the forward's error over the hidden units in dz); only ambiguous pairs and the saturated case, whose logits and so
  dz are 100x larger, are dominated by them. The emulation below reaches at most 0.45 of the bound, every mutant at
  least 20x it.
* hid_b = sum_b dpre: sum_b (ddp + EPS_F |dpre|). sm_w = dl^T hv: sum_b (E hv + |dl| band + EPS_F |dl| hv).
  sm_b = sum_b dl: sum_b (E + EPS_F |dl|).
* loss, per row (then times k, plus EPS_F of the total for the sum): xent  2 dz_b + 2^-20 (1 + ln esum) + EPS_F
  (|z_true| + |zmax| + ln esum); book  2 dz_b + ep_true + 2^-20 + EPS_F |ln p_true| (a clamped row: EPS_F ln 1e10).
* correct count: exact over rows whose top two logits are further apart than 2 dz_b + EPS_F max|z_b|; each other row
  may go either way.

Other activations (`--activation`, case builder and bound take `activation`; relu is the derivation above exactly)
-----------------------------------------------------------------------------------------------------------------
hv = f(pre) and dpre = dh * f'(hv), f' taken of the output as TF's *Grad ops take it (csrc/activation.cuh). With L_f
the Lipschitz constant of f (1; selu sa = 1.7581; sigmoid 1/4) the kernel's hv errs by ey = L_f band + f's own
rounding. CUDA 12.9's documented maximum errors are 2 ulp for expf and for tanhf and 0 for the IEEE divide, so f
rounds by at most (2 ulp + 2 u) |y| for sigmoid and tanh, by 2^-22 K e^pre + u |y| on the negative branch of elu (K
= 1) and selu (K = sa), and by u |y| for leaky_relu's and selu's products (their fp32 constants differ from the fp64
ones by < u relative); RND_ACT = 2^-20 times (|y| + K e^pre [pre < 0]) covers each with a 4x margin (relu and relu6
do not round). ey replaces band in dz and in the sm_w bound, |hv| replaces hv.
f' as a function of y has slope S (0 for the piecewise constant relu, relu6 and leaky_relu; 1 for elu and selu on y <
0 and for sigmoid's y (1 - y); 2 |y| for tanh's 1 - y y), so the kernel's f' errs by S ey + RND_ACT |f'|, and outside
the ambiguity bands ddp = |f'| ddh + |dh| (S ey + RND_ACT |f'|). The ambiguity bands sit at the kinks of f', where
the kernel may take either branch: 0 for relu, leaky_relu and selu (whose f' jumps from sa to s there), 0 and 6 for
relu6; elu's f' is continuous at 0 and sigmoid and tanh have none. There ddp = jump |dh| + max|f'| ddh + |dh| (S ey +
RND_ACT |f'|), with the jump of f' across the kink (relu: 1, giving the |dh| + ddh above). The builder moves biases so
that every branch is taken: both signs for leaky_relu, elu and selu, pre above 6 for relu6, |pre| > 3 in saturated
units for sigmoid and tanh (`_cover_activation`, asserted by `check_case`).

Other losses (`--loss`, `--label_smoothing`; case builder and bound take `loss` and `label_smoothing`)
--------------------------------------------------------------------------------------------------
The labels the loss sees are y' = smooth(y), formed in fp32 exactly as the kernels form them (csrc/loss.cuh); that
rounding is TF's too, so the fp64 reference takes the fp32 y' as its labels. The correct count uses the raw y. For
the elementwise losses k = 1 / (B C), and dz_bc (not its row maximum) bounds the error of logit z_bc.
* xent on smoothed labels: y' is no longer one-hot, so the cancellation in p S - y' (S = sum_c y'_c, about 1) sits at
  every class where p_c is near y'_c, not only at the true one; the rounding stays absolute: E_bc = k (p_c (2 dz_b +
  ep_c) S + EPS_F (p_c S + y'_c)) plus EPS_F p_c S for fl(S) (exact for one-hot labels). Loss per row: sum_c y'_c (2 dz_b + 2^-20 (1 + ln esum)
  + EPS_F (|z_c| + |zmax| + ln esum)), the one-hot terms above at every class.
* sigmoid_xent: dl = k (s - y') with s = sigmoid(z) from e = expf(-|z|) (2 ulp), 1 + e and an IEEE divide, so s errs
  by s' dz_bc <= dz_bc / 4 plus RND_LOSS s (RND_LOSS = 2^-20, 4x the roundings); the subtraction adds EPS_F (s + y'):
  E = k (dz / 4 + RND_LOSS s + EPS_F (s + y')). Loss element: its slope in z is s - y' in [-1, 1], so dz, plus
  log1pf's 2 ulp and the roundings, EPS_F (|z| (1 + y') + 1).
* mse: dl = 2k (z - y), so the error is absolute in |z - y|: E = 2k (dz + EPS_F |z - y|) (the fp32 k and the exact
  doubling add u). Loss element (z - y)^2: 2 |z - y| dz + dz^2 + EPS_F (z - y)^2.
* hinge: dl = -k y+- where m = 1 - y+- z > 0 (y+- = 2y - 1 = +-1), else 0. m errs by hedge = dz + EPS_F (|z| + 1),
  so, as at the ReLU's kink, pairs with |m| <= 2 hedge are *ambiguous*: the kernel may take either branch, E = k (the
  jump); elsewhere only k's fp32 rounding, E = EPS_F k. Loss element relu(m), 1-Lipschitz: hedge + EPS_F relu(m). A
  kernel that took m >= 0 for m > 0 differs only at m = 0 exactly, inside the band, so no mutant can show it; the
  hinge mutant drops the mask instead. The builder scales W_last by HINGE_SCALE so that logits pass +-1 and both
  branches are taken beyond the band (`check_case`).

The graph engine computes the same quantities with the same or tighter fp32 operations (IEEE division in the head, an
fp32 dW GEMM on tf32 operands), so the same bound applies to it unchanged.

Measured on one H100 80GB HBM3 (700 W power limit) over tests/test_gpu_fused_push_exact.py, whose `-s` log prints the
worst err / bound of every check: the pushes of both engines reach at most 0.45 of the hid_w bound (0.58 with the
atomic push, whose update rounding is added to the bound), every other variable and the loss at most 0.03 of theirs,
and every reported correct count lies in its range.

`emulate` runs the kernel's arithmetic in fp32 on the CPU, with dpre converted to tf32 by truncation or by
round-to-nearest; tests/test_fused_push_bound_cpu.py shows it inside the bound and each of a set of mutants (a dropped
batch row, a zeroed k-chunk, ...) far outside it at every case whose coverage admits the mutant, and
tests/test_activations_cpu.py does the same for every activation with the activation's own mutants (f or f' not
applied, f' of the pre-activation, relu6's f' without its upper kink), and tests/test_losses_cpu.py for every loss
and smoothing (LOSS_MUTANTS: smoothing not applied, the correct count taken of the smoothed labels, the sigmoid's
gradient negated, mse's factor 2 dropped, hinge's mask dropped).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field, replace
from typing import Dict, List, Optional, Tuple

import torch

from dist_mnist_b200.models import mlp

EPS_FWD = 2.0 ** -17     # forward accumulation: error of pre and of the hidden activations
AMBIG = 2.0 ** -14       # the ReLU's ambiguity band, 8x EPS_FWD
EPS_F = 2.0 ** -16       # every other fp32 sum and rounding
TF32 = 2.0 ** -9         # tf32 conversion of dpre, 2x margin over truncation
EXP_SLACK = 2.0 ** -20   # per-row second-order and fl(z - zmax) terms of the softmax
ULP1 = 2.0 ** -23
U = 2.0 ** -24
CLAMP = 1e-10            # the book loss's clip of p
CHUNK = 32               # features per k-chunk of the fused kernel
VARS = ("hid_w", "hid_b", "sm_w", "sm_b")
RND_ACT = 2.0 ** -20     # relative rounding of f and f' (expf / tanhf 2 ulp + a few roundings, 4x margin)
RND_LOSS = 2.0 ** -20    # relative rounding of the sigmoid of sigmoid_xent (expf 2 ulp + two roundings, 4x margin)
HINGE_SCALE = 10.0       # W_last scale of hinge cases: logits past +-1, so that both branches of the hinge are taken
ELEMENTWISE = ("sigmoid_xent", "mse", "hinge")


@dataclass(frozen=True)
class ActBound:
    """What the bound needs of an activation f: its Lipschitz constant, max |f'|, the jump of f' at its kinks (where
    the kernel may take either branch), the slope of f' as a function of y (tanh: 2 |y|, `slope_y` True), whether f
    and f' round at all, and the factor K of expf's absolute error term K e^x on the negative branch."""
    lip: float
    fmax: float
    jump: float
    kinks: Tuple[float, ...]
    slope: float
    slope_y: bool = False
    rounds: bool = True
    exp_k: float = 0.0


ACT_BOUNDS = {
    "relu": ActBound(1.0, 1.0, 1.0, (0.0,), 0.0, rounds=False),
    "relu6": ActBound(1.0, 1.0, 1.0, (0.0, 6.0), 0.0, rounds=False),
    "leaky_relu": ActBound(1.0, 1.0, 1.0 - mlp.LEAKY_RELU_ALPHA, (0.0,), 0.0),
    "elu": ActBound(1.0, 1.0, 0.0, (), 1.0, exp_k=1.0),
    "selu": ActBound(mlp.SELU_SCALE_ALPHA, mlp.SELU_SCALE_ALPHA, mlp.SELU_SCALE_ALPHA - mlp.SELU_SCALE, (0.0,), 1.0,
                     exp_k=mlp.SELU_SCALE_ALPHA),
    "sigmoid": ActBound(0.25, 0.25, 0.0, (), 1.0),
    "tanh": ActBound(1.0, 1.0, 0.0, (), 2.0, slope_y=True),
}


@dataclass
class Case:
    """A model, its variables (hid_w exact in tf32, nonzero biases) and one or more batches (x exact in tf32)."""
    name: str
    spec: mlp.MLPSpec
    params: Dict[str, torch.Tensor]
    batches: List[Tuple[torch.Tensor, torch.Tensor]]
    seed: int
    saturated: bool = False

    @property
    def batch(self) -> int:
        return self.batches[0][0].shape[0]

    @property
    def shape(self) -> Tuple[int, int, int, int, str]:
        (I, H), (_, C) = self.spec.layer_sizes
        return H, C, I, self.batch, self.spec.loss


def spec_for(H: int, C: int, I: int, loss: str, activation: str = "relu", label_smoothing: float = 0.0) -> mlp.MLPSpec:
    return mlp.MLPSpec(name="book", in_features=I, hidden=(H,), num_classes=C, loss=loss, init="book",
                       activation=activation, label_smoothing=label_smoothing)


def tf32_exact(t: torch.Tensor) -> torch.Tensor:
    """fp32 values with the 13 mantissa bits tf32 drops cleared (truncation: exact in tf32 by construction)."""
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def to_tf32(t: torch.Tensor, mode: str) -> torch.Tensor:
    """What the tensor core reads of fp32 operand bits: "trunc" drops the low 13 bits, "rne" rounds to nearest even."""
    b = t.contiguous().view(torch.int32)
    if mode == "rne":
        b = b + 0xFFF + ((b >> 13) & 1)
    elif mode != "trunc":
        raise ValueError(mode)
    return (b & ~0x1FFF).view(torch.float32)


def _draw_batch(g: torch.Generator, protos: torch.Tensor, B: int) -> Tuple[torch.Tensor, torch.Tensor]:
    C, I = protos.shape
    lab = torch.randint(0, C, (B,), generator=g)
    x = protos[lab] * (0.6 + 0.4 * torch.rand(B, 1, generator=g))
    x = x + (torch.rand(B, I, generator=g) < 0.1).float() * 0.35 * torch.rand(B, I, generator=g)
    x = torch.floor(x.clamp(0.0, 1.0) * 256.0).clamp(max=255.0) / 256.0      # k / 256, k = 0..255
    y = torch.zeros(B, C)
    y[torch.arange(B), lab] = 1.0
    return x.contiguous(), y


def make_case(H: int, C: int, I: int, B: int, loss: str, seed: int, n_batches: int = 1, saturate: float = 0.0,
              name: Optional[str] = None, activation: str = "relu", label_smoothing: float = 0.0) -> Case:
    """A tf32-exact case at shape (H, C, I, B, loss), redrawn from `seed` until `check_case` passes (coverage, the
    clamp margin). `saturate` scales W_last so that some rows' true-class p fall far below the clamp (hinge cases
    scale it by HINGE_SCALE). Under an activation other than relu, biases are then moved so that every branch of it is
    taken (`_cover_activation`); relu cases are drawn exactly as they were before activations existed."""
    spec = spec_for(H, C, I, loss, activation, label_smoothing)
    if loss == "hinge" and not saturate:
        saturate = HINGE_SCALE
    for attempt in range(64):
        sub = seed * 1000 + attempt
        g = torch.Generator().manual_seed(sub)
        params = mlp.init_params(spec, seed=sub)
        params["hid_w"] = tf32_exact(params["hid_w"])
        params["hid_b"] = (torch.rand(H, generator=g) * 0.2 - 0.05).float()
        params["sm_b"] = (torch.rand(C, generator=g) * 0.2 - 0.1).float()
        if saturate:
            params["sm_w"] = (params["sm_w"] * saturate).float()
        protos = (torch.rand(C, I, generator=g) < 0.2).float() * (0.5 + 0.5 * torch.rand(C, I, generator=g))
        batches = [_draw_batch(g, protos, B) for _ in range(n_batches)]
        # a dead unit hides a zeroed hidden row: raise a bias where needed so that every unit is active in some row
        # of every batch (small batches end up with every unit active, larger ones keep inactive pairs)
        top = torch.stack([(x.double() @ params["hid_w"].double().t()).amax(dim=0) for x, _ in batches]).amin(dim=0)
        params["hid_b"] = torch.maximum(params["hid_b"], (0.02 - top).float())
        if activation != "relu":
            _cover_activation(activation, params, batches)
        case = Case(name or f"H{H}-C{C}-I{I}-B{B}-{loss}" + ("-sat" if saturate and loss != "hinge" else "") +
                    ("" if activation == "relu" else f"-{activation}") +
                    (f"-ls{label_smoothing:g}" if label_smoothing else ""), spec, params, batches, sub,
                    saturated=bool(saturate) and loss != "hinge")
        if all(not check_case(case, x, y) for x, y in batches):
            assert exact_inputs(case) == [], exact_inputs(case)
            return case
    raise RuntimeError(f"no covered case at {(H, C, I, B, loss)} from seed {seed}")


def _cover_activation(activation: str, params: Dict[str, torch.Tensor],
                      batches: List[Tuple[torch.Tensor, torch.Tensor]]) -> None:
    """Move hidden biases so that the batches reach every branch of `activation` (`check_case` asserts it): relu6's
    upper kink (every third unit but the last tops out at 6.25 in some row; one unit alone is left below 6, where it
    can show every other mutant), and saturated sigmoid / tanh units (every third unit
    at least 3.5 in every row, the next one at most -3.5). The other units keep pre-activations of both signs, which
    leaky_relu, elu and selu need."""
    pre = [x.double() @ params["hid_w"].double().t() for x, _ in batches]
    top = torch.stack([p.amax(dim=0) for p in pre]).amin(dim=0)
    low = torch.stack([p.amin(dim=0) for p in pre]).amax(dim=0)
    b = params["hid_b"].clone()
    H, B = b.numel(), batches[0][0].shape[0]
    if activation == "relu6" and H > 1:
        up = torch.arange(0, H - 1, 3)   # the last unit stays below 6 (it shows a zeroed last hidden row)
        b[up] = (6.25 - top[up]).float()
    elif activation in ("sigmoid", "tanh"):
        b[0::3] = (3.5 - low[0::3]).float()
        b[1::3] = (-3.5 - top[1::3]).float()
    elif activation in ("leaky_relu", "elu", "selu"):
        if H > 1:
            b[1::3] = (-0.5 - top[1::3]).float()                    # every row of these units negative
        elif B > 1:
            b[0] = (0.02 - top[0]).float()                          # one unit: its top row positive, the others not
    params["hid_b"] = b


def exact_inputs(case: Case) -> List[str]:
    """What breaks the premise of the bound: empty when hid_w and every x are exact in tf32 under either conversion
    (truncation and round-to-nearest leave them unchanged) and both biases are nonzero somewhere."""
    bad = []
    for what, t in [("hid_w", case.params["hid_w"])] + [(f"x of batch {i}", x) for i, (x, _) in enumerate(case.batches)]:
        for mode in ("trunc", "rne"):
            if not bool((to_tf32(t, mode) == t).all()):
                bad.append(f"{what} is not exact in tf32 ({mode})")
    for b in ("hid_b", "sm_b"):
        if not bool((case.params[b] != 0).any()):
            bad.append(f"{b} is all zero")
    return bad


RANDOM_SEED = 20261017
SATURATE = 100.0   # W_last scale of the saturated case: about half its rows' true-class p lie far below 1e-10


def shape_matrix() -> List[Tuple[str, Tuple[int, int, int, int, str], float]]:
    """(id, (H, C, I, B, loss), saturate) of every case the element-wise checks run: the flagship at every batch
    edge, hidden-size edges, input edges (the last k-chunk partial or whole; 1, 2 or 4 k-chunks per CTA), class edges
    with both losses, corners, a saturated book-loss case, and 8 random shapes (from RANDOM_SEED) of the fused
    engine's domain (`sharding.fused_eligible`)."""
    shapes = [(100, 10, 784, b, "book") for b in (1, 31, 32, 33, 63, 64, 100, 255, 256)]
    shapes += [(h, 10, 784, 32, "book") for h in (1, 15, 16, 17, 64, 113, 127, 128)]
    shapes += [(100, 10, i, 32, "book") for i in (228, 256, 260, 1020, 1024)]
    shapes += [(100, c, 784, 32, loss) for c in (1, 2, 11) for loss in ("book", "xent")]
    shapes += [(128, 11, 1024, 256, "xent"), (1, 1, 228, 1, "book"), (17, 3, 260, 33, "xent")]
    out = [(f"H{h}-C{c}-I{i}-B{b}-{l}", (h, c, i, b, l), 0.0) for h, c, i, b, l in shapes]
    out.append(("H100-C10-I784-B32-book-saturated", (100, 10, 784, 32, "book"), SATURATE))
    g = torch.Generator().manual_seed(RANDOM_SEED)
    for n in range(8):
        h, c = int(torch.randint(1, 129, (1,), generator=g)), int(torch.randint(1, 12, (1,), generator=g))
        i, b = 4 * int(torch.randint(57, 257, (1,), generator=g)), int(torch.randint(1, 257, (1,), generator=g))
        loss = ("book", "xent")[int(torch.randint(0, 2, (1,), generator=g))]
        out.append((f"random{n}-H{h}-C{c}-I{i}-B{b}-{loss}", (h, c, i, b, loss), 0.0))
    return out


def case_for(shape: Tuple[int, int, int, int, str], saturate: float = 0.0, n_batches: int = 1, seed: int = 1,
             activation: str = "relu", label_smoothing: float = 0.0) -> Case:
    return make_case(*shape, seed=seed, n_batches=n_batches, saturate=saturate, activation=activation,
                     label_smoothing=label_smoothing)


# ----------------------------------------------------------------------------------------------
# fp64 reference and bounds
# ----------------------------------------------------------------------------------------------
@dataclass
class Reference:
    grads: Dict[str, torch.Tensor]          # fp64
    bounds: Dict[str, torch.Tensor]         # fp64, same shapes
    loss: float
    loss_bound: float
    correct_lo: int                          # rows surely correct
    correct_hi: int                          # + rows whose top two logits are within the error
    # intermediates for coverage, mutants and localisation
    x: torch.Tensor = field(repr=False, default=None)
    pre: torch.Tensor = field(repr=False, default=None)
    edge: torch.Tensor = field(repr=False, default=None)     # half-width of the ambiguity band at f's kinks
    dh: torch.Tensor = field(repr=False, default=None)
    dpre: torch.Tensor = field(repr=False, default=None)
    dl: torch.Tensor = field(repr=False, default=None)
    p_true: torch.Tensor = field(repr=False, default=None)
    active: torch.Tensor = field(repr=False, default=None)   # f' != 0, away from every kink
    hv: torch.Tensor = field(repr=False, default=None)       # f(pre)
    z: torch.Tensor = field(repr=False, default=None)        # logits
    hinge_m: torch.Tensor = field(repr=False, default=None)  # hinge: 1 - y+- z
    hinge_edge: torch.Tensor = field(repr=False, default=None)  # hinge: half-width of the ambiguity band at m = 0


def _k(spec: mlp.MLPSpec, B: int) -> float:
    return 1.0 / B if spec.loss == "xent" else 1.0 / (B * spec.num_classes)


def reference(spec: mlp.MLPSpec, params: Dict[str, torch.Tensor], x: torch.Tensor, y: torch.Tensor) -> Reference:
    """The fp64 step on (x, y) and the per-element bounds of the module docstring."""
    d = torch.float64
    P = {k: v.to(d) for k, v in params.items()}
    yraw = y.to(d)
    # the smoothed labels are rounded to fp32 as TF (and the kernels) round them: they are the fp64 step's labels
    spec0 = replace(spec, label_smoothing=0.0)
    x64, y64 = x.to(d), mlp.smooth_labels(spec, y.float()).to(d)
    loss, grads, logits = mlp.manual_loss_and_grads(spec0, P, x64, y64)
    W, b, Wl, bl = P["hid_w"], P["hid_b"], P["sm_w"], P["sm_b"]
    B, C = y.shape
    k = _k(spec, B)
    ax, aWl = x64.abs(), Wl.abs()
    pre = x64 @ W.t() + b
    A = ax @ W.abs().t() + b.abs()
    band, edge = EPS_FWD * A, AMBIG * A
    ab = ACT_BOUNDS[spec.activation]
    amb = torch.zeros_like(pre, dtype=torch.bool)
    for kink in ab.kinks:
        amb |= (pre - kink).abs() <= edge
    hv = mlp.activate(spec.activation, pre)
    fp = mlp.activation_grad(spec.activation, hv, torch.ones_like(hv))      # f'(pre), from y as the kernels do
    act = ~amb & (fp != 0)
    ahv = hv.abs()
    ey = ab.lip * band                                                        # error of the kernel's hv
    if ab.rounds:
        ey = ey + RND_ACT * (ahv + ab.exp_k * torch.exp(pre.clamp(max=0.0)) * (pre < 0).to(d))
    z = logits
    dzc = ey @ aWl.t() + EPS_F * (ahv @ aWl.t() + bl.abs())
    dz = dzc.amax(dim=1, keepdim=True)
    p = torch.softmax(z, dim=1)
    zmax = z.amax(dim=1, keepdim=True)
    ee = (2.0 + 1.173 * (zmax - z)) * ULP1
    ep = ee + (p * ee).sum(dim=1, keepdim=True) + 16 * U + 2.0 ** -22 + EXP_SLACK
    p_true = (p * yraw).sum(dim=1)
    live = p_true >= CLAMP if spec.loss == "book" else torch.ones(B, dtype=torch.bool)
    S = y64.sum(dim=1, keepdim=True)
    hm = hedge = None
    if spec.loss == "book":
        E = k * (p * (2 * dz + ep) + EPS_F * (p + y64)) * live[:, None].to(d)
        passes = p >= CLAMP
        g = torch.where(passes, -k * y64 / p.clamp_min(1e-300), torch.zeros_like(p))
        dl = p * (g - (g * p).sum(dim=1, keepdim=True))
    elif spec.loss == "xent":
        fl_s = EPS_F * p * S if spec.label_smoothing else 0.0   # fl(S): exact for one-hot labels
        E = k * (p * (2 * dz + ep) * S + EPS_F * (p * S + y64) + fl_s)
        dl = (p * S - y64) * k
    elif spec.loss == "sigmoid_xent":
        sig = torch.sigmoid(z)
        E = k * (dzc / 4 + RND_LOSS * sig + EPS_F * (sig + y64))
        dl = k * (sig - y64)
    elif spec.loss == "mse":
        E = 2 * k * (dzc + EPS_F * (z - y64).abs())
        dl = 2 * k * (z - y64)
    else:   # hinge
        ypm = 2 * y64 - 1
        hm = 1 - ypm * z
        hedge = 2 * (dzc + EPS_F * (z.abs() + 1))
        E = k * torch.where(hm.abs() <= hedge, torch.ones_like(hm), torch.full_like(hm, EPS_F))
        dl = torch.where(hm > 0, -k * ypm, torch.zeros_like(hm))
    dh = dl @ Wl
    dpre = mlp.activation_grad(spec.activation, hv, dh)
    ddh = E @ aWl + EPS_F * (dl.abs() @ aWl)
    # f' of the kernel's y: off by slope * ey (tanh: 2 |y| ey), plus its own rounding
    dfp = (ab.slope * ahv if ab.slope_y else torch.full_like(hv, ab.slope)) * ey
    if ab.rounds:
        dfp = dfp + RND_ACT * fp.abs()
    ddp = ((~amb).to(d) * (fp.abs() * ddh + dh.abs() * dfp) +
           amb.to(d) * (ab.jump * dh.abs() + ab.fmax * ddh + dh.abs() * dfp))
    bounds = {
        "hid_w": (TF32 * dpre.abs() + (1 + TF32) * ddp + EPS_F * dpre.abs()).t() @ ax,
        "hid_b": (ddp + EPS_F * dpre.abs()).sum(dim=0),
        "sm_w": E.t() @ ahv + dl.abs().t() @ ey + EPS_F * (dl.abs().t() @ ahv),
        "sm_b": (E + EPS_F * dl.abs()).sum(dim=0),
    }
    esum = torch.exp(z - zmax).sum(dim=1)
    dzr = dz[:, 0]
    if spec.loss == "xent":
        lrow = (y64 * (2 * dz + EXP_SLACK * (1 + esum.log()[:, None]) +
                       EPS_F * (z.abs() + zmax.abs() + esum.log()[:, None]))).sum(dim=1)
    elif spec.loss == "sigmoid_xent":
        lrow = (dzc + EPS_F * (z.abs() * (1 + y64) + 1)).sum(dim=1)
    elif spec.loss == "mse":
        lrow = (2 * (z - y64).abs() * dzc + dzc * dzc + EPS_F * (z - y64) ** 2).sum(dim=1)
    elif spec.loss == "hinge":
        lrow = (hedge / 2 + EPS_F * hm.clamp(min=0.0)).sum(dim=1)
    else:
        ep_t = (ep * y64).sum(dim=1)
        lrow = torch.where(live, 2 * dzr + ep_t + EXP_SLACK + EPS_F * p_true.clamp_min(CLAMP).log().abs(),
                           torch.full_like(dzr, EPS_F * math.log(1e10)))
    loss_bound = float(k * lrow.sum()) + EPS_F * abs(float(loss))
    top2 = z.topk(min(2, C), dim=1).values
    gap = top2[:, 0] - top2[:, 1] if C > 1 else torch.full((B,), math.inf, dtype=d)
    unsure = gap <= 2 * dzr + EPS_F * z.abs().amax(dim=1)
    right = z.argmax(dim=1) == yraw.argmax(dim=1)
    lo = int((right & ~unsure).sum())
    return Reference({n: grads[n] for n in VARS}, bounds, float(loss), loss_bound, lo, lo + int(unsure.sum()),
                     x64, pre, edge, dh, dpre, dl, p_true, act, hv, z, hm, hedge)


def check_case(case: Case, x: torch.Tensor, y: torch.Tensor) -> List[str]:
    """What keeps a batch from testing every edge of the kernel: empty when covered. Every hidden unit is active
    (beyond the ReLU's ambiguity band) in some row, every batch row has a nonzero x and a nonzero dlogits row (so it
    moves sm_b and the loss at least) unless it is a clamped row of the saturated case or there is one class, every
    k-chunk has a nonzero x under an active unit, and the book
    loss keeps every true-class p outside [1e-10 / 2, 2e-10]; the saturated case has clamped and unclamped rows.
    "Active" is f' != 0 outside the ambiguity bands (the ReLU: pre above the band). Each branch of the activation is
    taken (beyond the band) where a single pre-activation does not rule it out: both signs for leaky_relu, elu and
    selu, pre above 6 for relu6 (with H > 1), saturated |pre| > 3 for sigmoid and tanh. The hinge has margins on both
sides of its kink, beyond the ambiguity band."""
    spec = case.spec
    r = reference(spec, case.params, x, y)
    act = r.pre > r.edge if spec.activation == "relu6" else r.active   # (units above 6 are not dead)
    bad = []
    a = spec.activation
    several = r.pre.numel() > 1
    if a in ("leaky_relu", "elu", "selu") and several and not (bool((r.pre > r.edge).any()) and
                                                               bool((r.pre < -r.edge).any())):
        bad.append(f"{a}: pre-activations of one sign only")
    if a == "relu6" and spec.hidden[0] > 1 and not bool((r.pre > 6 + r.edge).any()):
        bad.append("relu6: no pre-activation above 6")
    if a in ("sigmoid", "tanh") and not bool((r.pre.abs() > 3).any()):
        bad.append(f"{a}: no saturated pre-activation")
    if not bool(act.any(dim=0).all()):
        bad.append(f"hidden units never active: {(~act.any(dim=0)).nonzero().flatten().tolist()}")
    live = r.p_true >= CLAMP if spec.loss == "book" else torch.ones(x.shape[0], dtype=torch.bool)
    if spec.loss == "hinge" and r.z.numel() > 1 and not (bool((r.hinge_m > r.hinge_edge).any()) and
                                                          bool((r.hinge_m < -r.hinge_edge).any())):
        bad.append("hinge: margins of one side only")
    rows_ok = (x.abs().sum(dim=1) > 0) & (~live | (r.dl.abs().sum(dim=1) > 0) | torch.tensor(spec.num_classes == 1))
    if not bool(rows_ok.all()):
        bad.append(f"batch rows without a contribution: {(~rows_ok).nonzero().flatten().tolist()}")
    I = spec.in_features
    seen = (act.to(torch.float64).t() @ r.x.abs()).sum(dim=0)   # [I]: x under an active unit
    for c in range((I + CHUNK - 1) // CHUNK):
        if not float(seen[c * CHUNK:(c + 1) * CHUNK].sum()) > 0:
            bad.append(f"k-chunk {c} sees no input")
    if spec.loss == "book":
        near = (r.p_true >= CLAMP / 2) & (r.p_true <= 2 * CLAMP)
        if bool(near.any()):
            bad.append(f"true-class p near the clamp in rows {near.nonzero().flatten().tolist()}")
        clamped = int((~live).sum())
        if case.saturated and not (0 < clamped < x.shape[0]):
            bad.append(f"saturated case with {clamped} clamped rows of {x.shape[0]}")
    return bad


# ----------------------------------------------------------------------------------------------
# the kernel's arithmetic in fp32 on the CPU, and mutants of it
# ----------------------------------------------------------------------------------------------
@dataclass
class Step:
    """What one step reports: the pushed gradient by variable, the loss and the correct count."""
    grads: Dict[str, torch.Tensor]
    loss: float
    correct: int


def emulate(spec: mlp.MLPSpec, params: Dict[str, torch.Tensor], x: torch.Tensor, y: torch.Tensor,
            tf32: str = "trunc", mutant: Optional[str] = None, arg: int = 0) -> Step:
    """One fused step in fp32 with dpre converted to tf32 (`tf32` = "trunc" | "rne"), under spec.activation. `mutant`
    (with `arg`) is one of MUTANTS: a plausible kernel bug, applied where the kernel would make it."""
    f = torch.float32
    W, b, Wl, bl = (params[n].to(f) for n in VARS)
    x, y = x.to(f), y.to(f)
    B, C = y.shape
    live = torch.ones(B, 1)
    if mutant == "drop_row":
        live[arg] = 0.0
    elif mutant == "drop_tile":
        live[32 * arg:32 * (arg + 1)] = 0.0
    nb = 32 * ((B + 31) // 32) if mutant == "loss_32T" else B
    ys = y if mutant == "smoothing_missing" else mlp.smooth_labels(spec, y)
    pre = x @ W.t() + b
    a = spec.activation
    hv = pre if mutant == "act_forward_missing" else mlp.activate(a, pre)
    z = hv @ Wl.t() + bl
    p = torch.softmax(z, dim=1)
    k = torch.tensor(1.0, dtype=f) / (torch.tensor(float(nb), dtype=f) * torch.tensor(float(C), dtype=f))
    if spec.loss == "book":
        g = torch.where((p >= 1e-10) & (p <= 1.0), -k * y / p, torch.zeros_like(p))
        dl = p * (g - (g * p).sum(dim=1, keepdim=True))
        lc = -k * y * torch.log(p.clamp(1e-10, 1.0))
    elif spec.loss == "xent":
        k = torch.tensor(1.0, dtype=f) / torch.tensor(float(nb), dtype=f)
        dl = k * (p * ys.sum(dim=1, keepdim=True) - ys)
        lc = -k * ys * torch.log_softmax(z, dim=1)
    elif spec.loss == "sigmoid_xent":
        elem, sig = mlp._sigmoid_xent_terms(z, ys)
        dl = k * (ys - sig) if mutant == "sigmoid_grad_sign" else k * (sig - ys)
        lc = k * elem
    elif spec.loss == "mse":
        dz = z - ys
        dl = (k if mutant == "mse_factor_two_missing" else 2 * k) * dz
        lc = k * (dz * dz)
    else:   # hinge
        ypm = 2 * ys - 1
        m = 1 - ypm * z
        dl = (-k) * ypm if mutant == "hinge_mask_missing" else torch.where(m > 0, (-k) * ypm, torch.zeros_like(m))
        lc = k * torch.relu(m)
    dl = dl * live
    if a == "relu":
        mask = (hv > 0).to(f)
        if mutant == "relu_missing":
            mask[:, arg] = 1.0
        dpre = (dl @ Wl) * mask
    elif mutant == "act_grad_missing":
        dpre = dl @ Wl
    elif mutant == "act_grad_from_pre":
        dpre = mlp.activation_grad(a, pre, dl @ Wl)
    elif mutant == "relu6_upper_kink_missing":
        dpre = mlp.activation_grad("relu", hv, dl @ Wl)
    else:
        dpre = mlp.activation_grad(a, hv, dl @ Wl)
    dW = to_tf32(dpre, tf32).t() @ x
    if mutant == "zero_chunk":
        dW[:, arg * CHUNK:(arg + 1) * CHUNK] = 0.0
    elif mutant == "zero_hidden_row":
        dW[arg] = 0.0
    dWl = dl.t() @ hv
    if mutant == "sm_w_transposed":
        dWl = dWl.t().contiguous().reshape(dWl.shape)
    elif mutant == "sm_w_class_shift":
        dWl = torch.roll(dWl, 1, dims=0)
    yc = ys if mutant == "smoothing_in_accuracy" else y
    correct = int(((z.argmax(dim=1) == yc.argmax(dim=1)) & (live[:, 0] > 0)).sum())
    return Step({"hid_w": dW, "hid_b": dpre.sum(dim=0), "sm_w": dWl, "sm_b": dl.sum(dim=0)},
                float((lc * live).sum()), correct)


MUTANTS = ("drop_row", "drop_tile", "zero_chunk", "zero_hidden_row", "relu_missing", "loss_32T", "sm_w_transposed",
           "sm_w_class_shift", "act_forward_missing", "act_grad_missing", "act_grad_from_pre", "relu6_upper_kink_missing",
           "smoothing_missing", "smoothing_in_accuracy", "sigmoid_grad_sign", "mse_factor_two_missing",
           "hinge_mask_missing")
ACT_MUTANTS = MUTANTS[8:12]  # the activation's own: f not applied, f' not applied, f' of pre, relu6's f' without its
                             # upper kink
LOSS_MUTANTS = MUTANTS[12:]  # the loss's own: labels not smoothed, the correct count of the smoothed labels, the
                             # sigmoid's gradient negated, mse's factor 2 dropped, the hinge's mask dropped


def mutant_instances(case: Case, ref: Reference) -> List[Tuple[str, int]]:
    """(mutant, arg) pairs that this batch's coverage admits, i.e. that change the step beyond rounding: every
    mutant needs >= 2 classes (one class pushes exact zeros); a dropped tile and the last row of tile 0 need > 32
    rows; the 32 T normalisation needs B % 32 != 0; a transposed sm_w needs H >= 2; the missing ReLU mask needs an
    inactive (b, j) under a nonzero dh and x (it takes the unit with the most such weight). Under another activation
    than relu, the missing mask is replaced by ACT_MUTANTS, each admitted where it changes the step: f not applied
    where f(pre) differs from pre by more than 0.02, f' not applied or taken of pre where that changes some |dpre| |x|
    by 5 % of the largest, relu6's upper kink likewise where a pre lies above 6."""
    H, C, I, B, _ = case.shape
    if C < 2:
        return []
    out = [("drop_row", 0), ("drop_row", B - 1), ("zero_chunk", 0), ("zero_chunk", (I + CHUNK - 1) // CHUNK - 1),
           ("zero_hidden_row", H - 1), ("sm_w_class_shift", 0)]
    if B > 32:
        out += [("drop_row", 31), ("drop_tile", 0), ("drop_tile", (B + 31) // 32 - 1)]
    if B % 32:
        out.append(("loss_32T", 0))
    if H >= 2:
        out.append(("sm_w_transposed", 0))
    a = case.spec.activation
    rows = ref.x.abs().sum(dim=1, keepdim=True)

    def moves(change: torch.Tensor) -> bool:   # f' changed by `change`, by 5 % of the largest |dpre| |x| somewhere
        return float(((change.abs() * ref.dh.abs()) * rows).max()) > 0.05 * float((ref.dpre.abs() * rows).max())

    out += _loss_mutants(case, ref)
    if a == "relu":
        off = (ref.pre < -ref.edge).to(torch.float64)
        weight = ((off * ref.dh.abs()) * rows).sum(dim=0)
        if float(weight.max()) > 0:
            out.append(("relu_missing", int(weight.argmax())))
        return out
    one = torch.ones_like(ref.hv)
    fp = mlp.activation_grad(a, ref.hv, one)
    if float((ref.hv - ref.pre).abs().max()) > 0.02:
        out.append(("act_forward_missing", 0))
    if moves(fp - 1):
        out.append(("act_grad_missing", 0))
    if moves(mlp.activation_grad(a, ref.pre, one) - fp):
        out.append(("act_grad_from_pre", 0))
    if a == "relu6" and moves((ref.pre > 6 + ref.edge).to(torch.float64)):
        out.append(("relu6_upper_kink_missing", 0))
    return out


def _loss_mutants(case: Case, ref: Reference) -> List[Tuple[str, int]]:
    """LOSS_MUTANTS this batch admits: the smoothing ones under a smoothing (the correct count of the smoothed labels
    only where it falls outside the reference's range: ls = 1, where every y' is equal and argmax says class 0), each
    loss's own mutant under that loss (the hinge's dropped mask where some margin lies beyond the band on the inactive
    side)."""
    spec, out = case.spec, []
    if spec.label_smoothing:
        out.append(("smoothing_missing", 0))
        z0 = int((ref.z.argmax(dim=1) == 0).sum())
        if not ref.correct_lo <= z0 <= ref.correct_hi and spec.label_smoothing == 1.0:
            out.append(("smoothing_in_accuracy", 0))
    if spec.loss == "sigmoid_xent":
        out.append(("sigmoid_grad_sign", 0))
    elif spec.loss == "mse":
        out.append(("mse_factor_two_missing", 0))
    elif spec.loss == "hinge" and bool((ref.hinge_m < -ref.hinge_edge).any()):
        out.append(("hinge_mask_missing", 0))
    return out


# ----------------------------------------------------------------------------------------------
# comparison
# ----------------------------------------------------------------------------------------------
@dataclass
class Verdict:
    worst: Dict[str, float]                      # err / bound per variable, "loss", "correct" (0 or inf)
    where: Dict[str, Tuple[int, ...]]            # element of the worst ratio (+ its dominant batch row for hid_w)
    got_correct: int = 0
    ref_correct: Tuple[int, int] = (0, 0)

    @property
    def ok(self) -> bool:
        return all(v <= 1.0 for v in self.worst.values())

    @property
    def max(self) -> float:
        return max(self.worst.values())

    def line(self) -> str:
        parts = []
        for n in VARS + ("loss",):
            w = self.where.get(n)
            parts.append(f"{n} {self.worst[n]:.3g}" + (f"@{w}" if w and self.worst[n] > 0.5 else ""))
        parts.append(f"correct {self.got_correct} in [{self.ref_correct[0]}, {self.ref_correct[1]}]")
        return "err/bound: " + ", ".join(parts)


def compare(got: Step, ref: Reference) -> Verdict:
    """The worst |got - ref| / bound of each variable, the loss and the correct count, and where it occurs: (row,
    column, batch row with the largest |dpre x| there) for hid_w, the element index otherwise. A zero bound demands an
    exact zero difference."""
    worst, where = {}, {}
    for n in VARS:
        g = got.grads[n].to(torch.float64).reshape(ref.grads[n].shape)
        err = (g - ref.grads[n]).abs()
        bnd = ref.bounds[n]
        ratio = torch.where(bnd > 0, err / bnd.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
        ratio = torch.nan_to_num(ratio, nan=math.inf)
        i = int(ratio.flatten().argmax())
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), ratio.shape))
        if n == "hid_w":
            j, f = idx
            idx = (j, f, int((ref.dpre[:, j].abs() * ref.x[:, f].abs()).argmax()))
        worst[n], where[n] = float(ratio.flatten()[i]), idx
    lerr = abs(got.loss - ref.loss)
    worst["loss"] = lerr / ref.loss_bound if ref.loss_bound > 0 else (0.0 if lerr == 0 else math.inf)
    if not math.isfinite(got.loss):
        worst["loss"] = math.inf
    worst["correct"] = 0.0 if ref.correct_lo <= got.correct <= ref.correct_hi else math.inf
    return Verdict(worst, where, got.correct, (ref.correct_lo, ref.correct_hi))


# ----------------------------------------------------------------------------------------------
# reading a push on the GPU
# ----------------------------------------------------------------------------------------------
def pushed(w, seq: int = 1) -> Dict[str, torch.Tensor]:
    """The gradient worker `w` pushed with push `seq`, read out of its mailbox slot in the ps segments (and put
    together from the pieces of a row-split variable)."""
    ns = w.cfg.nslots
    slot = seq % ns
    out = {}
    for name, vl in w.layout.by_name.items():
        owners = list(dict.fromkeys((pc.ps, pc.offset) for pc in vl.pieces))
        spans = {}
        for k, off in owners:
            base = (w.task_index * ns + slot) * w.ps_desc[k]["arena_elems"]
            spans[(k, off)] = w._unpack(vl, w._copy_from_ps(k, "mailbox", base + off, vl.span, torch.float32))
        if len(owners) == 1:
            out[name] = spans[owners[0]]
            continue
        full = torch.empty(vl.rows, vl.cols)
        for pc in vl.pieces:
            if pc.c1 > pc.c0:
                full[:, pc.c0:pc.c1] = spans[(pc.ps, pc.offset)][:, pc.c0:pc.c1]
        out[name] = full
    return out
