// Gradient clipping arithmetic shared by the fused step's clip instantiations (fused_step_sm90.cu) and the graph
// engine's clip tail (clip_sm90.cu): TF1 1.15's clip_by_global_norm / clip_by_norm / clip_by_value in fp32, with
// TF's NaN behaviour (models/mlp.py clip_gradients is the reference).
#pragma once
#include "protocol.h"

namespace dm {

// clip_by_global_norm: scale = clip_norm * min(1 / n, 1 / clip_norm) with n = sqrt(sum of squares), plus (n - n),
// which makes the scale NaN when n is inf or NaN, as TF does.
__device__ __forceinline__ float clip_global_scale(float ssq, float clip_norm) {
  const float n = __fsqrt_rn(ssq);
  return __fadd_rn(__fmul_rn(clip_norm, fminf(__fdiv_rn(1.f, n), __fdiv_rn(1.f, clip_norm))), __fsub_rn(n, n));
}
// clip_by_norm: the divisor max(norm, clip_norm), norm = sqrt(l2) if l2 > 0 else l2. A NaN norm stays NaN (TF's
// maximum propagates it), so a variable with a NaN element becomes NaN as a whole.
__device__ __forceinline__ float clip_norm_divisor(float l2, float clip_norm) {
  const float norm = l2 > 0.f ? __fsqrt_rn(l2) : l2;
  return norm != norm ? norm : fmaxf(norm, clip_norm);
}
// One element: CLIP_GLOBAL_NORM g * f (f = the scale); CLIP_NORM (g * clip_norm) / f (f = the divisor);
// CLIP_VALUE max(min(g, hi), lo), a NaN element staying NaN as under TF's minimum / maximum.
__device__ __forceinline__ float clip_element(int kind, float g, float f, float clip_norm, float lo, float hi) {
  if (kind == CLIP_GLOBAL_NORM) return __fmul_rn(g, f);
  if (kind == CLIP_NORM) return __fdiv_rn(__fmul_rn(g, clip_norm), f);
  return g != g ? g : fmaxf(fminf(g, hi), lo);
}

}  // namespace dm
