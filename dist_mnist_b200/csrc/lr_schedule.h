// Learning-rate schedules of the parameter server: TF1's tf.train.{exponential,inverse_time,natural_exp,polynomial,
// cosine}_decay and piecewise_constant, evaluated at a step count `s` (PsItemState::sched_step), and the decay of
// TF1's ExponentialMovingAverage. Shared by the scheduled and averaging serve kernels (ps_apply_sm90.cu) and the cpu
// backend's serve loop (host_runtime.cpp).
//
// The rate is fp32 like TF1's float32 graph ops (powf / expf / cosf, IEEE division). The step becomes an exponent
// through integer arithmetic, p = q + r / decay_steps with q = s / decay_steps, r = s % decay_steps (q alone with
// staircase), so it stays exact past 2^24 steps, where TF1's float cast of global_step would not.
#pragma once
#include <math.h>
#include <stdint.h>

#include "protocol.h"

#ifdef __CUDACC__
#define DM_LR_HD __host__ __device__ __forceinline__
#else
#define DM_LR_HD inline
#endif

namespace dm {

// s / d as q + r / d in fp32 (`floor_only`: q)
template <typename T>
DM_LR_HD float lr_sched_ratio(T s, T d, bool floor_only) {
  const T q = s / d, r = s - q * d;
  return floor_only ? static_cast<float>(q) : static_cast<float>(q) + static_cast<float>(r) / static_cast<float>(d);
}

DM_LR_HD float scheduled_lr(const PsServeParams& P, uint32_t s) {
  const float lr0 = P.lr;
  const uint32_t d = P.decay_steps;
  switch (P.lr_schedule) {
    case LR_EXPONENTIAL:
      return lr0 * powf(P.decay_rate, lr_sched_ratio(s, d, P.staircase != 0));
    case LR_INVERSE_TIME:
      return lr0 / (1.f + P.decay_rate * lr_sched_ratio(s, d, P.staircase != 0));
    case LR_NATURAL_EXP:
      return lr0 * expf(-P.decay_rate * lr_sched_ratio(s, d, P.staircase != 0));
    case LR_POLYNOMIAL: {
      float f;
      if (P.cycle) {   // d' = d * max(1, ceil(s / d)) may pass 2^32
        const uint64_t c = (static_cast<uint64_t>(s) + d - 1) / d;
        f = lr_sched_ratio<uint64_t>(s, static_cast<uint64_t>(d) * (c > 1 ? c : 1), false);
      } else {
        f = lr_sched_ratio<uint32_t>(s < d ? s : d, d, false);
      }
      return (lr0 - P.end_lr) * powf(1.f - f, P.power) + P.end_lr;
    }
    case LR_COSINE: {
      const float f = lr_sched_ratio(s < d ? s : d, d, false);
      return lr0 * ((1.f - P.alpha) * 0.5f * (1.f + cosf(3.14159265358979323846f * f)) + P.alpha);
    }
    case LR_PIECEWISE: {
      int i = 0;
      while (i < P.n_boundaries && s > P.boundaries[i]) ++i;
      return P.values[i];
    }
    default:
      return lr0;
  }
}

// Decay of TF1's ExponentialMovingAverage for the optimizer step that brings an item to `n` applied pushes:
// min(decay, (1 + n) / (10 + n)) from the float cast of n, in fp32 with IEEE division like TF1's graph. For
// n >= (10 decay - 1) / (1 - decay) the min is `decay`; that bound lies below 2^24 for every decay <= 0.99999, so
// the cast's rounding past 2^24 cannot change d there.
DM_LR_HD float ema_decay(const PsServeParams& P, uint32_t n) {
  if (!P.ema_num_updates) return P.ema_decay;
  const float nf = static_cast<float>(n);
  const float r = (1.f + nf) / (10.f + nf);
  return P.ema_decay < r ? P.ema_decay : r;
}

}  // namespace dm
