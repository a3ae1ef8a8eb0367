// Classification losses after the two softmax ones (protocol.h LossKind), and the label smoothing of the two
// cross-entropies, as TF 1.15's tf.losses functions compute them in fp32 with weight 1 (SUM_BY_NONZERO_WEIGHTS: the mean
// over the B x C elements). Every operation is rounded on its own (no contraction into FMAs) and uses the accurate
// expf / log1pf and an IEEE divide, as activation.cuh does; models/mlp.py holds the reference. Both heads call these only
// for real classes: a padded class carries z = -inf, and 0 * inf would be NaN.
#pragma once
#include <cuda_runtime.h>

#include "protocol.h"

namespace dm {

// y' = y (1 - ls) + ls / C (LOSS_XENT) or y (1 - ls) + 0.5 ls (LOSS_SIGMOID_XENT): TF forms 1 - ls and 0.5 ls in double
// and rounds them to fp32, ls / C is an fp32 division; the multiply and the add round separately. ls = 0 keeps y.
__device__ __forceinline__ float smooth_label(int loss_kind, float y, float ls, int C) {
  const float keep = static_cast<float>(1.0 - static_cast<double>(ls));
  const float add = loss_kind == LOSS_SIGMOID_XENT ? static_cast<float>(0.5 * static_cast<double>(ls))
                                                   : __fdiv_rn(ls, static_cast<float>(C));
  return __fadd_rn(__fmul_rn(y, keep), add);
}

// One element of LOSS_SIGMOID_XENT, LOSS_MSE or LOSS_HINGE: logit z, label y (smoothed for the sigmoid), k = 1 / (B C).
// `lc` is k times the element's loss, `dl` the gradient of the mean loss with respect to z.
__device__ __forceinline__ void elementwise_loss(int loss_kind, float z, float y, float k, float& dl, float& lc) {
  if (loss_kind == LOSS_SIGMOID_XENT) {
    // max(z, 0) - z y + log1p(exp(-|z|));  dz = k (sigmoid(z) - y), sigmoid from e = exp(-|z|) <= 1
    const float e = expf(-fabsf(z));
    const float d = __fadd_rn(1.f, e);
    const float sig = z >= 0.f ? __fdiv_rn(1.f, d) : __fdiv_rn(e, d);
    dl = __fmul_rn(k, __fsub_rn(sig, y));
    lc = __fmul_rn(k, __fadd_rn(__fsub_rn(fmaxf(z, 0.f), __fmul_rn(z, y)), log1pf(e)));
  } else if (loss_kind == LOSS_MSE) {
    // (z - y)^2;  dz = (2 k)(z - y), the order of TF's SquaredDifference gradient
    const float d = __fsub_rn(z, y);
    dl = __fmul_rn(__fmul_rn(2.f, k), d);
    lc = __fmul_rn(k, __fmul_rn(d, d));
  } else {
    // LOSS_HINGE: relu(1 - y' z) with y' = 2 y - 1;  dz = -k y' where 1 - y' z > 0 (ReluGrad on the output), else 0
    const float ypm = __fsub_rn(__fmul_rn(2.f, y), 1.f);
    const float m = __fsub_rn(1.f, __fmul_rn(ypm, z));
    dl = m > 0.f ? __fmul_rn(-k, ypm) : 0.f;
    lc = __fmul_rn(k, fmaxf(m, 0.f));
  }
}

inline bool loss_valid(int loss_kind) { return loss_kind >= LOSS_BOOK && loss_kind <= LOSS_HINGE; }

// A label smoothing `ls` a loss accepts: finite and in [0, 1], and 0 unless the loss is a cross-entropy on y'
inline bool label_smoothing_valid(int loss_kind, float ls) {
  return ls >= 0.f && ls <= 1.f && (ls == 0.f || loss_kind == LOSS_XENT || loss_kind == LOSS_SIGMOID_XENT);
}

}  // namespace dm
