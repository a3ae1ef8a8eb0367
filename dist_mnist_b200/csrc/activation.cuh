// Hidden-layer activations (protocol.h ActivationKind): f and its derivative as TF 1.15's functors and registered
// gradients compute them, in fp32. The derivative takes the layer's output y, as TF's *Grad ops do (the graph engine
// keeps only the activations). Every operation is rounded on its own (no contraction into FMAs) and uses the accurate
// expf / tanhf and an IEEE divide, so the result equals models/mlp.py's fp32 torch arithmetic up to expf / tanhf's
// ulp error. Units and rows the callers mask out stay exactly as they were: f is applied only to values they keep.
#pragma once
#include <cuda_runtime.h>

#include "protocol.h"

namespace dm {

constexpr float kLeakyReluAlpha = 0.2f;
constexpr float kSeluScale = 1.0507009873554804934193349852946f;
constexpr float kSeluScaleAlpha = 1.7580993408473768599402175208123f;

__device__ __forceinline__ float act_forward(int act, float x) {
  switch (act) {
    case ACT_RELU: return fmaxf(x, 0.f);
    case ACT_RELU6: return fminf(fmaxf(x, 0.f), 6.f);
    case ACT_LEAKY_RELU: return x > 0.f ? x : __fmul_rn(kLeakyReluAlpha, x);
    case ACT_ELU: return x < 0.f ? __fsub_rn(expf(x), 1.f) : x;
    case ACT_SELU: return x < 0.f ? __fmul_rn(kSeluScaleAlpha, __fsub_rn(expf(x), 1.f)) : __fmul_rn(kSeluScale, x);
    case ACT_SIGMOID: return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x)));
    case ACT_TANH: return tanhf(x);
    default: return x;   // ACT_NONE
  }
}

// dx = dy * f'(x), from y = f(x)
__device__ __forceinline__ float act_backward(int act, float y, float dy) {
  switch (act) {
    case ACT_RELU: return y > 0.f ? dy : 0.f;
    case ACT_RELU6: return (y > 0.f && y < 6.f) ? dy : 0.f;
    case ACT_LEAKY_RELU: return y > 0.f ? dy : __fmul_rn(kLeakyReluAlpha, dy);   // y > 0 iff x > 0 (alpha > 0)
    case ACT_ELU: return y < 0.f ? __fmul_rn(dy, __fadd_rn(y, 1.f)) : dy;
    case ACT_SELU: return y < 0.f ? __fmul_rn(dy, __fadd_rn(y, kSeluScaleAlpha)) : __fmul_rn(dy, kSeluScale);
    case ACT_SIGMOID: return __fmul_rn(__fmul_rn(dy, y), __fsub_rn(1.f, y));
    case ACT_TANH: return __fmul_rn(dy, __fsub_rn(1.f, __fmul_rn(y, y)));
    default: return dy;   // ACT_NONE
  }
}

inline bool act_valid(int act) { return act >= ACT_NONE && act <= ACT_TANH; }

}  // namespace dm
