// Parameter-server shard kernels for sm_90a.
//
// ps_serve_kernel is the PS "process" of the reference (tf.train.Server(...).join(),
// /root/reference/distributed_server-basic.py:80-83) turned into a persistent GPU kernel: it owns the
// shard (params + Adam slots + global_step, DS:88-91,102-103), polls the per-item flags that workers
// publish with st.release.sys after their in-kernel P2P gradient stores, reduces whatever is ready
// (many-to-one) and applies the optimizer in the same pass (ApplyAdam / SGD, SURVEY K7; or TF1's
// ApplyMomentum / ApplyAdagrad / ApplyRMSProp / ApplyAdadelta / ApplyFtrl(V2) / ApplyProximalAdagrad /
// ApplyProximalGradientDescent in their own instantiations), bumps global_step (K8) and acknowledges into the
// worker's inbox over NVLink. No host, NCCL or gRPC in the loop.
//
// Work decomposition: items (2-D blocks of the arena) are dealt round-robin to CTAs; a CTA never shares
// an item, so item state (Adam step count / beta powers) needs no synchronisation. Pushes of one worker
// are consumed in order per item; different workers interleave arbitrarily (Hogwild, like the reference's
// unlocked async apply).
#include "common.cuh"
#include "lr_schedule.h"
#include "protocol.h"

namespace dm {

constexpr int kPsThreads = 512;
constexpr int kMaxOwn = 32;   // items one CTA may own (their descriptors / state / cursors live in shared memory)
constexpr int kQuads = 2;     // element quads per thread per pass
constexpr int kMaxPending = 32;

// MUFU approximations (<= 2 ulp): the Adam update is issue-bound on the one SM that owns an item (IEEE sqrt and
// divide expand to ~15 instructions each: 3.9 us per push and item measured, 4x the SGD path).
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sqrt_approx(float x) {
  float y;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// kIeee (`--adam_math ieee`, PsServeParams::ieee_math): correctly rounded sqrt and divide like TF's ApplyAdam CPU /
// CUDA kernels (Eigen), at ~4x the per-push cost; the default instantiation is the MUFU fast path, unchanged.
template <bool kIeee = false>
__device__ __forceinline__ void adam_step(float& p, float& m, float& v, float g, float lr_t, float beta1,
                                          float beta2, float eps) {
  // TF1 AdamOptimizer: m <- b1 m + (1-b1) g ; v <- b2 v + (1-b2) g^2 ; p <- p - lr_t m / (sqrt(v) + eps)
  m = fmaf(beta1, m, (1.f - beta1) * g);
  v = fmaf(beta2, v, (1.f - beta2) * g * g);
  if constexpr (kIeee) p = p - __fdiv_rn(lr_t * m, __fsqrt_rn(v) + eps);
  else p = fmaf(-lr_t * m, rcp_approx(sqrt_approx(v) + eps), p);
}
template <bool kIeee = false>
__device__ __forceinline__ float adam_lr_t(float lr, float b1p, float b2p) {
  if constexpr (kIeee) return __fdiv_rn(lr * __fsqrt_rn(1.f - b2p), 1.f - b1p);
  else return lr * sqrt_approx(1.f - b2p) * rcp_approx(1.f - b1p);   // lr * sqrt(1 - b2^t) / (1 - b1^t)
}

// The other TF1 `training_ops` rules (Apply{Momentum,Adagrad,RMSProp}). Slots: adam_m holds the momentum accumulator /
// RMSProp's mom, adam_v holds Adagrad's accumulator / RMSProp's ms (m and v below).
__device__ __forceinline__ float rsqrt_approx(float x) {
  float y;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
template <bool kIeee>
__device__ __forceinline__ float div_sqrt(float a, float x) {   // a / sqrt(x)
  if constexpr (kIeee) return __fdiv_rn(a, __fsqrt_rn(x));
  else return a * rsqrt_approx(x);
}
// Adadelta, FTRL and the proximal rules (Apply{Adadelta,Ftrl,FtrlV2,ProximalAdagrad,ProximalGradientDescent}): fast =
// the MUFU helpers above (and __powf for FTRL's general power), IEEE = correctly rounded sqrt / divide (rsqrt as 1 /
// sqrt) and powf.
template <bool kIeee>
__device__ __forceinline__ float sqrt_m(float x) {
  if constexpr (kIeee) return __fsqrt_rn(x);
  else return sqrt_approx(x);
}
template <bool kIeee>
__device__ __forceinline__ float rsqrt_m(float x) {
  if constexpr (kIeee) return __fdiv_rn(1.f, __fsqrt_rn(x));
  else return rsqrt_approx(x);
}
template <bool kIeee>
__device__ __forceinline__ float div_m(float a, float b) {
  if constexpr (kIeee) return __fdiv_rn(a, b);
  else return a * rcp_approx(b);
}
template <bool kIeee>
__device__ __forceinline__ float pow_m(float x, float y) {
  if constexpr (kIeee) return powf(x, y);
  else return __powf(x, y);
}
// The proximal step of ApplyProximalAdagrad / ApplyProximalGradientDescent at step size `a`:
//   l1 > 0: sign(prox) max(|prox| - a l1, 0) / (1 + l2 a) ; else prox / (1 + l2 a)
template <bool kIeee>
__device__ __forceinline__ float prox_shrink(float prox, float a, float l1, float l2) {
  const float num = l1 > 0.f ? copysignf(fmaxf(fabsf(prox) - a * l1, 0.f), prox) : prox;
  return div_m<kIeee>(num, fmaf(l2, a, 1.f));
}
// kSched: the step's rate is `lr_sched`; else P.lr (read from the parameter block as the measured instantiations do).
// `mg`: centered RMSProp's third slot. `da_t` (kSched): AdagradDA's global step T, the item's applied pushes with this
// step's included, converted to fp32 once.
template <int kOpt, bool kIeee, bool kSched>
__device__ __forceinline__ void tf1_step(float& p, float& m, float& v, float& mg, float g, const PsServeParams& P,
                                         const float& lr_sched, float da_t) {
  const float& lr = kSched ? lr_sched : P.lr;
  if constexpr (kOpt == OPT_MOMENTUM) {
    // accum <- momentum accum + g ; p <- p - lr accum  (Nesterov: p <- p - lr g - lr momentum accum)
    m = fmaf(P.momentum, m, g);
    if (P.nesterov) p = p - fmaf(g, lr, m * P.momentum * lr);
    else p = fmaf(-lr, m, p);
  } else if constexpr (kOpt == OPT_ADAGRAD) {
    bool da = false;
    if constexpr (kSched) da = P.opt == OPT_ADAGRAD_DA;
    if (da) {
      // ApplyAdagradDA (m = gradient_accumulator, v = gradient_squared_accumulator): g_acc <- g_acc + g ;
      // gg_acc <- gg_acc + g^2 ; p <- -lr sign(g_acc) max(|g_acc| - T l1, 0) / (l2 (T lr) + sqrt(gg_acc))
      //                              (l1 = 0: -lr g_acc / ((T lr) l2 + sqrt(gg_acc)))
      m = m + g;
      v = fmaf(g, g, v);
      const float tl = da_t * lr;
      if (P.l1 > 0.f)
        p = div_m<kIeee>(-lr * copysignf(fmaxf(fabsf(m) - da_t * P.l1, 0.f), m), fmaf(P.l2, tl, sqrt_m<kIeee>(v)));
      else
        p = div_m<kIeee>(-lr * m, fmaf(tl, P.l2, sqrt_m<kIeee>(v)));
    } else {
      // accum <- accum + g^2 ; p <- p - lr g / sqrt(accum)   (no epsilon)
      v = fmaf(g, g, v);
      p = p - div_sqrt<kIeee>(lr * g, v);
    }
  } else if constexpr (kOpt == OPT_RMSPROP) {
    // ms <- ms + (g^2 - ms)(1 - decay) ; mom <- momentum mom + lr g / sqrt(ms + eps) ; p <- p - mom
    // centered: mg <- mg + (g - mg)(1 - decay) ; mom <- momentum mom + g lr / sqrt((ms - mg^2) + eps)  (not clamped: a
    // negative denominator gives NaN, as in TF)
    v = fmaf(fmaf(g, g, -v), 1.f - P.decay, v);
    if (P.centered) {
      mg = fmaf(g - mg, 1.f - P.decay, mg);
      m = fmaf(P.momentum, m, div_sqrt<kIeee>(g * lr, fmaf(-mg, mg, v) + P.eps));
    } else {
      m = fmaf(P.momentum, m, div_sqrt<kIeee>(lr * g, v + P.eps));
    }
    p = p - m;
  } else if constexpr (kOpt == OPT_ADADELTA) {
    // accum <- rho accum + (1 - rho) g^2 ; update = sqrt(accum_update + eps) rsqrt(accum + eps) g ; p <- p - lr update ;
    // accum_update <- rho accum_update + (1 - rho) update^2   (rho rides in P.decay; v = accum, m = accum_update)
    const float rho = P.decay;
    v = fmaf(v, rho, g * g * (1.f - rho));
    const float upd = sqrt_m<kIeee>(m + P.eps) * rsqrt_m<kIeee>(v + P.eps) * g;
    p = fmaf(-upd, lr, p);
    m = fmaf(m, rho, upd * upd * (1.f - rho));
  } else if constexpr (kOpt == OPT_PROXIMAL_ADAGRAD) {
    // accum <- accum + g^2 ; a = lr rsqrt(accum) ; p <- shrink(p - g a, a)
    v = fmaf(g, g, v);
    const float a = lr * rsqrt_m<kIeee>(v);
    p = prox_shrink<kIeee>(fmaf(-g, a, p), a, P.l1, P.l2);
  } else if constexpr (kOpt == OPT_PROXIMAL_SGD) {
    // p <- shrink(p - lr g, lr)   (no square root: one instantiation, IEEE divide)
    p = prox_shrink<true>(fmaf(-lr, g, p), lr, P.l1, P.l2);
  } else {
    static_assert(kOpt == OPT_FTRL, "unknown optimizer family");
    // ApplyFtrlV2 (l2_shrinkage 0: ApplyFtrl, gs = g exactly). v = accum, m = linear.
    //   n = accum + g^2 ; linear += gs - (n^-lr_power - accum^-lr_power) / lr p ;
    //   p <- |linear| > l1 ? (sign(linear) l1 - linear) / (n^-lr_power / lr + 2 l2) : 0 ; accum <- n
    const float gs = fmaf(2.f * P.l2_shrinkage, p, g);
    const float n = fmaf(g, g, v);
    float pn, pa;
    if (P.lr_power == -0.5f) {   // TF's special case: sqrt
      pn = sqrt_m<kIeee>(n);
      pa = sqrt_m<kIeee>(v);
    } else {
      pn = pow_m<kIeee>(n, -P.lr_power);
      pa = pow_m<kIeee>(v, -P.lr_power);
    }
    m = m + (gs - div_m<kIeee>(pn - pa, lr) * p);
    const float y = div_m<kIeee>(pn, lr) + 2.f * P.l2;
    p = fabsf(m) > P.l1 ? div_m<kIeee>(copysignf(P.l1, m) - m, y) : 0.f;
    v = n;
  }
}

// Optimizer family of a serve-kernel instantiation. Adam and SGD share theirs (P.opt picks the rule at run time); every
// other kind gets its own.
constexpr int kFamAdamSgd = -1;

// Apply every pending push to one item. s_pend[0..n_pend) lists the mailbox slots (element offset of the slot
// inside P.mailbox) in application order — round k = the k-th pending push of every worker, oldest round first —
// and s_round[i] is the round of entry i. One optimizer step per push, or per round in APPLY_MERGED mode
// (concurrent pushes of different workers are summed; consecutive pushes of one worker stay separate steps).
// Parameters and Adam slots stay in registers for the whole pass; the gradient loads of kCh pushes are issued
// together (a mailbox line costs an L2/HBM round trip of ~1-2 us: issuing them one push at a time made the
// pass, and with it the push->ack latency that throttles the workers, proportional to 5 us x pending pushes).
// Optimizer state of an item held in registers across passes (see ps_serve_kernel): valid when the CTA owns exactly one
// item that fits one sweep of the CTA (<= kPsThreads * kQuads * 4 elements, vectorisable).
struct ResidentState {
  float p[kQuads][4], m[kQuads][4], v[kQuads][4];
  bool loaded;
};
// The moving averages of that item (the averaging instantiations) and, in the RMSProp family, centered RMSProp's mean
// gradients (P.centered), valid whenever ResidentState::loaded is.
template <int kFam>
struct ResidentExtra {
  float e[kQuads][4];
};
template <>
struct ResidentExtra<OPT_RMSPROP> {
  float e[kQuads][4];
  float g[kQuads][4];
};
// Pending pushes whose gradient loads are in flight together, per instantiation: the largest chunk that ptxas compiles
// without a spill under __launch_bounds__(kPsThreads, 1) (IEEE Adam / SGD at a constant rate keeps the fast one's 8 and
// spills 28 bytes; four RMSProp entries and the Adagrad family's IEEE scheduled / averaging ones are one below their
// earlier values, so that centered RMSProp's third slot and AdagradDA fit). Indexed [family row][kIeee][constant rate,
// scheduled, averaging]; the family rows are Adam / SGD, then OPT_MOMENTUM .. OPT_PROXIMAL_SGD in enum order. 0: no
// such instantiation (see serve_kernel).
constexpr int kServeChunk[8][2][3] = {
    {{8, 7, 6}, {8, 6, 5}},   // Adam / SGD
    {{7, 7, 7}, {0, 0, 0}},   // Momentum
    {{7, 7, 6}, {7, 6, 5}},   // Adagrad (the scheduled / averaging ones also run AdagradDA)
    {{7, 7, 6}, {6, 6, 5}},   // RMSProp (with centered RMSProp's third slot)
    {{7, 8, 6}, {7, 7, 6}},   // Adadelta
    {{8, 8, 6}, {7, 7, 6}},   // FTRL
    {{7, 7, 7}, {7, 7, 5}},   // ProximalAdagrad
    {{0, 0, 0}, {7, 7, 5}},   // ProximalGradientDescent
};
constexpr int serve_family_row(int fam) { return fam == kFamAdamSgd ? 0 : fam - OPT_MOMENTUM + 1; }

// kSched (the scheduled instantiations): the rate of the optimizer step whose pushes sit at positions i0..i1 of the
// application order is s_lr[i0], the pass's rate table (lr(sched_step + i), built by the serve loop); else P.lr.
// kEma (the averaging instantiations, which are also kSched): the item's moving averages P.ema stay in registers for
// the pass like the parameters, and after the optimizer step that ends at position i every element's shadow moves
// toward the new parameter by 1 - s_ema[i], the pass's decay table (ema_decay(sched_step + i + 1)).
// The RMSProp family with P.centered also keeps the third slot P.mg (resident beside the others, in res_extra->g);
// the Adagrad family's scheduled instantiations also run AdagradDA (P.opt), whose T at the step that ends at position i
// is sched_step + i + 1.
template <int kFam, bool kIeee, bool kSched, bool kEma>
__device__ void apply_item(const PsServeParams& P, const PsItem it, const PsItemState st, const uint64_t* s_pend,
                           const uint32_t* s_round, const int n_pend, ResidentState* res, const float* s_lr,
                           const float* s_ema, ResidentExtra<kFam>* res_extra) {
  const int tid = threadIdx.x;
  const int total = it.rows * it.cols;
  const bool vec = ((it.cols & 3) == 0) && ((it.ld & 3) == 0) && ((it.offset & 3) == 0);
  const int step = vec ? 4 : 1;
  const bool adam = kFam == kFamAdamSgd && P.opt == OPT_ADAM;
  // the slot buffers this rule reads and writes
  bool use_m = kFam == kFamAdamSgd ? adam : opt_uses_m(kFam);
  const bool use_v = kFam == kFamAdamSgd ? adam : opt_uses_v(kFam);
  if constexpr (kFam == OPT_ADAGRAD && kSched) use_m = opt_uses_m(P.opt);   // AdagradDA's gradient_accumulator
  bool use_mg = false;   // centered RMSProp's mean gradient
  if constexpr (kFam == OPT_RMSPROP) use_mg = P.centered != 0u;
  const bool merged = P.apply_mode == APPLY_MERGED;
  for (int e0 = tid * step; e0 < total; e0 += kPsThreads * step * kQuads) {
    uint64_t a[kQuads];
    bool ok[kQuads];
    float pv[kQuads][4], mv[kQuads][4], vv[kQuads][4];
    float ev[kQuads][4];   // kEma: the shadows
    float gv[kQuads][4];   // use_mg: the mean gradients
#pragma unroll
    for (int q = 0; q < kQuads; ++q) {
      const int e = e0 + q * kPsThreads * step;
      ok[q] = e < total;
      const int r = ok[q] ? e / it.cols : 0;
      const int c = ok[q] ? e - r * it.cols : 0;
      a[q] = it.offset + static_cast<uint64_t>(r) * it.ld + c;
#pragma unroll
      for (int j = 0; j < 4; ++j) { pv[q][j] = 0.f; mv[q][j] = 0.f; vv[q][j] = 0.f; }
      if constexpr (kEma) {
#pragma unroll
        for (int j = 0; j < 4; ++j) ev[q][j] = 0.f;
      }
      if constexpr (kFam == OPT_RMSPROP) {
#pragma unroll
        for (int j = 0; j < 4; ++j) gv[q][j] = 0.f;
      }
    }
    if (res != nullptr && res->loaded) {
      // the item's parameters and Adam slots never left this thread's registers: no load round trip in this pass
#pragma unroll
      for (int q = 0; q < kQuads; ++q)
#pragma unroll
        for (int j = 0; j < 4; ++j) { pv[q][j] = res->p[q][j]; mv[q][j] = res->m[q][j]; vv[q][j] = res->v[q][j]; }
      if constexpr (kEma) {
#pragma unroll
        for (int q = 0; q < kQuads; ++q)
#pragma unroll
          for (int j = 0; j < 4; ++j) ev[q][j] = res_extra->e[q][j];
      }
      if constexpr (kFam == OPT_RMSPROP) {
        if (use_mg) {
#pragma unroll
          for (int q = 0; q < kQuads; ++q)
#pragma unroll
            for (int j = 0; j < 4; ++j) gv[q][j] = res_extra->g[q][j];
        }
      }
    } else {
#pragma unroll
      for (int q = 0; q < kQuads; ++q) {
        if (!ok[q]) continue;
        if (vec) {
          const float4 t = __ldcg(reinterpret_cast<const float4*>(P.params + a[q]));
          pv[q][0] = t.x; pv[q][1] = t.y; pv[q][2] = t.z; pv[q][3] = t.w;
          if (use_m) {
            const float4 tm = __ldcg(reinterpret_cast<const float4*>(P.adam_m + a[q]));
            mv[q][0] = tm.x; mv[q][1] = tm.y; mv[q][2] = tm.z; mv[q][3] = tm.w;
          }
          if (use_v) {
            const float4 tv = __ldcg(reinterpret_cast<const float4*>(P.adam_v + a[q]));
            vv[q][0] = tv.x; vv[q][1] = tv.y; vv[q][2] = tv.z; vv[q][3] = tv.w;
          }
          if constexpr (kEma) {
            const float4 te = __ldcg(reinterpret_cast<const float4*>(P.ema + a[q]));
            ev[q][0] = te.x; ev[q][1] = te.y; ev[q][2] = te.z; ev[q][3] = te.w;
          }
          if constexpr (kFam == OPT_RMSPROP) {
            if (use_mg) {
              const float4 tg = __ldcg(reinterpret_cast<const float4*>(P.mg + a[q]));
              gv[q][0] = tg.x; gv[q][1] = tg.y; gv[q][2] = tg.z; gv[q][3] = tg.w;
            }
          }
        } else {
          pv[q][0] = __ldcg(P.params + a[q]);
          if (use_m) mv[q][0] = __ldcg(P.adam_m + a[q]);
          if (use_v) vv[q][0] = __ldcg(P.adam_v + a[q]);
          if constexpr (kEma) ev[q][0] = __ldcg(P.ema + a[q]);
          if constexpr (kFam == OPT_RMSPROP) {
            if (use_mg) gv[q][0] = __ldcg(P.mg + a[q]);
          }
        }
      }
    }
    float b1p = st.beta1_pow, b2p = st.beta2_pow;
    float gsum[kQuads][4];
#pragma unroll
    for (int q = 0; q < kQuads; ++q)
#pragma unroll
      for (int j = 0; j < 4; ++j) gsum[q][j] = 0.f;

    constexpr int kCh = kServeChunk[serve_family_row(kFam)][kIeee][kEma ? 2 : kSched ? 1 : 0];
    static_assert(kCh > 0, "no serve-kernel instantiation of this family and math");
    int r0 = 0;   // kSched, merged: position of the first push of the current round
    for (int i0 = 0; i0 < n_pend; i0 += kCh) {
      float g[kCh][kQuads][4];
#pragma unroll
      for (int ci = 0; ci < kCh; ++ci) {
        const bool live = i0 + ci < n_pend;
        const float* gbase = P.mailbox + s_pend[live ? i0 + ci : i0];
#pragma unroll
        for (int q = 0; q < kQuads; ++q) {
          g[ci][q][0] = g[ci][q][1] = g[ci][q][2] = g[ci][q][3] = 0.f;
          if (!ok[q] || !live) continue;
          if (vec) {
            const float4 t = __ldcg(reinterpret_cast<const float4*>(gbase + a[q]));  // L2: written over NVLink
            g[ci][q][0] = t.x; g[ci][q][1] = t.y; g[ci][q][2] = t.z; g[ci][q][3] = t.w;
          } else {
            g[ci][q][0] = __ldcg(gbase + a[q]);
          }
        }
      }
#pragma unroll
      for (int ci = 0; ci < kCh; ++ci) {
        const int i = i0 + ci;
        if (i >= n_pend) break;
        bool do_step = true;
        if (merged) {
#pragma unroll
          for (int q = 0; q < kQuads; ++q)
#pragma unroll
            for (int j = 0; j < 4; ++j) gsum[q][j] += g[ci][q][j];
          do_step = (i + 1 == n_pend) || (s_round[i + 1] != s_round[i]);   // last push of its round
        }
        if (!do_step) continue;
        float lr = P.lr;
        if constexpr (kSched) {
          lr = s_lr[merged ? r0 : i];
          r0 = i + 1;
        }
        float lr_t = lr;
        if (adam) {
          b1p *= P.beta1;
          b2p *= P.beta2;
          lr_t = adam_lr_t<kIeee>(lr, b1p, b2p);
        }
        float ema_omd = 0.f;   // kEma: 1 - d of this step, in fp32 like TF1's `1.0 - decay`
        if constexpr (kEma) ema_omd = 1.f - s_ema[i];
        float da_t = 0.f;   // AdagradDA: T = pushes applied to the item after this step (TF's static_cast<float>)
        if constexpr (kFam == OPT_ADAGRAD && kSched) da_t = static_cast<float>(st.sched_step + static_cast<uint32_t>(i) + 1u);
#pragma unroll
        for (int q = 0; q < kQuads; ++q) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (j >= step) continue;
            const float gr = merged ? gsum[q][j] : g[ci][q][j];
            if constexpr (kFam != kFamAdamSgd)
              tf1_step<kFam, kIeee, kSched>(pv[q][j], mv[q][j], vv[q][j], gv[q][j], gr, P, lr, da_t);
            else if (adam) adam_step<kIeee>(pv[q][j], mv[q][j], vv[q][j], gr, lr_t, P.beta1, P.beta2, P.eps);
            else pv[q][j] = fmaf(-lr, gr, pv[q][j]);
            // assign_moving_average: shadow -= (shadow - p) * (1 - d), each op rounded as TF1's graph does
            if constexpr (kEma) ev[q][j] = ev[q][j] - __fmul_rn(ev[q][j] - pv[q][j], ema_omd);
            if (merged) gsum[q][j] = 0.f;
          }
        }
      }
    }
    if (res != nullptr) {
#pragma unroll
      for (int q = 0; q < kQuads; ++q)
#pragma unroll
        for (int j = 0; j < 4; ++j) { res->p[q][j] = pv[q][j]; res->m[q][j] = mv[q][j]; res->v[q][j] = vv[q][j]; }
      if constexpr (kEma) {
#pragma unroll
        for (int q = 0; q < kQuads; ++q)
#pragma unroll
          for (int j = 0; j < 4; ++j) res_extra->e[q][j] = ev[q][j];
      }
      if constexpr (kFam == OPT_RMSPROP) {
        if (use_mg) {
#pragma unroll
          for (int q = 0; q < kQuads; ++q)
#pragma unroll
            for (int j = 0; j < 4; ++j) res_extra->g[q][j] = gv[q][j];
        }
      }
      res->loaded = true;
    }
#pragma unroll
    for (int q = 0; q < kQuads; ++q) {
      if (!ok[q]) continue;
      const bool shadow = P.shadow_bf16 != nullptr && (it.flags & 1);
      if (vec) {
        *reinterpret_cast<float4*>(P.params + a[q]) = make_float4(pv[q][0], pv[q][1], pv[q][2], pv[q][3]);
        if (use_m) *reinterpret_cast<float4*>(P.adam_m + a[q]) = make_float4(mv[q][0], mv[q][1], mv[q][2], mv[q][3]);
        if (use_v) *reinterpret_cast<float4*>(P.adam_v + a[q]) = make_float4(vv[q][0], vv[q][1], vv[q][2], vv[q][3]);
        if constexpr (kEma) *reinterpret_cast<float4*>(P.ema + a[q]) = make_float4(ev[q][0], ev[q][1], ev[q][2], ev[q][3]);
        if constexpr (kFam == OPT_RMSPROP) {
          if (use_mg) *reinterpret_cast<float4*>(P.mg + a[q]) = make_float4(gv[q][0], gv[q][1], gv[q][2], gv[q][3]);
        }
        if (shadow) {
          __nv_bfloat162 lo = __floats2bfloat162_rn(pv[q][0], pv[q][1]);
          __nv_bfloat162 hi = __floats2bfloat162_rn(pv[q][2], pv[q][3]);
          uint2 pk;
          pk.x = *reinterpret_cast<uint32_t*>(&lo);
          pk.y = *reinterpret_cast<uint32_t*>(&hi);
          *reinterpret_cast<uint2*>(P.shadow_bf16 + a[q]) = pk;
        }
      } else {
        P.params[a[q]] = pv[q][0];
        if (use_m) P.adam_m[a[q]] = mv[q][0];
        if (use_v) P.adam_v[a[q]] = vv[q][0];
        if constexpr (kEma) P.ema[a[q]] = ev[q][0];
        if constexpr (kFam == OPT_RMSPROP) {
          if (use_mg) P.mg[a[q]] = gv[q][0];
        }
        if (shadow) {
          __nv_bfloat16 b = __float2bfloat16(pv[q][0]);
          P.shadow_bf16[a[q]] = *reinterpret_cast<uint16_t*>(&b);
        }
      }
    }
  }
}

// kFam: optimizer family; kIeee: correctly rounded sqrt / divide. kSched: a non-constant learning-rate schedule
// (P.lr_schedule != LR_CONSTANT). kEma: moving averages of the parameters (P.ema != null), under any schedule: the rate
// table is compiled in as with kSched (scheduled_lr is lr0 for LR_CONSTANT), so one instantiation serves a constant rate
// and every schedule. Everything a schedule adds sits behind `if constexpr (kSched)`, everything averaging adds behind
// `if constexpr (kEma)`, so the constant-rate instantiations carry none of it.
template <int kFam, bool kIeee, bool kSched, bool kEma>
__global__ void __launch_bounds__(kPsThreads, 1) ps_serve_kernel(const __grid_constant__ PsServeParams P) {
  static_assert(kSched || !kEma, "the averaging instantiations read the rate table too");
  // Everything the poll loop needs about this CTA's items lives in shared memory: the only global traffic of an
  // idle poll is one acquire load of a flag word per (worker, look-ahead slot).
  __shared__ PsItem s_item[kMaxOwn];
  __shared__ PsItemState s_state[kMaxOwn];
  __shared__ uint32_t s_next[kMaxOwn][kMaxWorkers];  // next expected push seq per (owned item, worker)
  __shared__ uint64_t s_pend[kMaxPending];
  __shared__ uint32_t s_round[kMaxPending];
  __shared__ uint32_t s_npend;
  __shared__ uint32_t s_any;
  __shared__ uint32_t s_exit;
  __shared__ float s_lr[kMaxPending];   // kSched: rate of the pass's i-th push, lr(sched_step + i)
  __shared__ float s_ema[kMaxPending];  // kEma: decay of the step ending at the i-th push, ema_decay(sched_step + i + 1)
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  uint32_t iter = 0;
  int n_own = 0;
  for (int item = blockIdx.x; item < P.n_items && n_own < kMaxOwn; item += gridDim.x) ++n_own;
  for (int i = tid; i < n_own; i += kPsThreads) {
    const int item = blockIdx.x + i * gridDim.x;
    s_item[i] = P.items[item];
    s_state[i] = P.item_state[item];
  }
  for (int i = tid; i < n_own * kMaxWorkers; i += kPsThreads) {
    const int own = i / kMaxWorkers, w = i - own * kMaxWorkers;
    s_next[own][w] = w < P.n_workers ? P.next_seq[static_cast<size_t>(w) * P.n_items + blockIdx.x + own * gridDim.x] : 0u;
  }
  __syncthreads();
  // poll lanes, round-major: lane = k * n_workers + w checks push s_next[w] + k of worker w. Pushes of one worker
  // are consumed in order, so only its contiguous ready prefix k = 0 .. cnt-1 is taken in a pass; lane order is
  // then exactly the application order (round k = k-th pending push of every worker, oldest round first).
  const int nw = P.n_workers;
  int kdepth = max(1, min(min(P.nslots, 16), 32 / nw));
  if (P.lookahead != 0u) kdepth = min(kdepth, static_cast<int>(P.lookahead));
  const int pk = lane / nw, pw = lane - pk * nw;
  const bool pvalid = pk < kdepth;
  const uint64_t wstride = static_cast<uint64_t>(P.nslots) * P.arena_elems;

  // Register-resident optimizer state: a CTA that owns exactly one vectorisable item of at most one sweep keeps the
  // item's parameters and Adam slots in registers from pass to pass (it is the only writer while it runs; the host
  // writes variables only while no serve kernel is resident). Results are still stored every pass — the workers pull
  // the parameters, checkpoints read the slots — but the three load round trips (~1 us of a ~6.7 us pass) are gone.
  ResidentState resident;
  resident.loaded = false;
  ResidentExtra<kFam> resident_extra;   // beside them: the shadows (kEma), centered RMSProp's mean gradients
  bool use_resident = false;
  if (n_own == 1) {
    const PsItem it0 = s_item[0];
    use_resident = ((it0.cols & 3) == 0) && ((it0.ld & 3) == 0) && ((it0.offset & 3) == 0) &&
                   (it0.rows * it0.cols <= kPsThreads * kQuads * 4);
  }

  // serve statistics (thread 0's view; the CTA barriers make it representative)
  unsigned long long st_pass = 0, st_push = 0, st_apply = 0, st_book = 0, st_idle_n = 0, st_idle = 0, st_max = 0,
                     st_poll = 0;
  const bool stats_on = P.stats != nullptr;

  for (;;) {
    bool sweep_any = false;   // (uniform over the CTA: s_any is read after a barrier)
    for (int own = 0; own < n_own; ++own) {
      const int item = blockIdx.x + own * gridDim.x;
      const long long c0 = stats_on ? clock64() : 0;
      uint32_t p_seq = 0, p_cnt = 0, p_taken = 0;   // warp 0: this lane's push seq, its worker's prefix, all taken
      bool p_take = false;
      if (warp == 0) {
        uint32_t ready = 0, slot = 0;
        if (pvalid) {
          p_seq = s_next[own][pw] + pk;
          slot = p_seq % P.nslots;
          const uint32_t f = ld_acquire_scoped_u32(
              P.flags + (static_cast<size_t>(pw) * P.nslots + slot) * P.n_flags + s_item[own].flag_index, P.gpu_scope);
          ready = (f == p_seq) ? 1u : 0u;
        }
        const uint32_t b = __ballot_sync(0xffffffffu, ready);
        if (pvalid)
          while (p_cnt < static_cast<uint32_t>(kdepth) && ((b >> (p_cnt * nw + pw)) & 1u)) ++p_cnt;
        p_take = pvalid && static_cast<uint32_t>(pk) < p_cnt;
        p_taken = __ballot_sync(0xffffffffu, p_take);
        if (p_take) {
          const int pos = __popc(p_taken & ((1u << lane) - 1u));
          s_pend[pos] = static_cast<uint64_t>(pw) * wstride + static_cast<uint64_t>(slot) * P.arena_elems;
          s_round[pos] = pk;
        }
        if (lane == 0) {
          s_any = p_taken;
          s_npend = __popc(p_taken);
        }
        if constexpr (kSched) {
          // the pass's rate table (one fp32 evaluation per lane): the i-th push of the application order is applied
          // at schedule step sched_step + i; published to apply_item by the barrier below
          if (lane < __popc(p_taken)) s_lr[lane] = scheduled_lr(P, s_state[own].sched_step + lane);
        }
        if constexpr (kEma) {
          // the pass's decay table: the step that ends at the i-th push leaves the item at sched_step + i + 1
          // applied pushes, TF1's num_updates = global_step after the apply_gradients op the average follows
          if (lane < __popc(p_taken)) s_ema[lane] = ema_decay(P, s_state[own].sched_step + lane + 1);
        }
      }
      __syncthreads();
      const long long c1 = stats_on ? clock64() : 0;
      if (!s_any && stats_on) { ++st_idle_n; st_idle += c1 - c0; }
      if (s_any) {
        sweep_any = true;
        const PsItemState st = s_state[own];
        apply_item<kFam, kIeee, kSched, kEma>(P, s_item[own], st, s_pend, s_round, static_cast<int>(s_npend),
                                              use_resident ? &resident : nullptr, s_lr, s_ema,
                                              use_resident ? &resident_extra : nullptr);
        __syncthreads();   // every thread's parameter stores precede warp 0's release operations below
        const long long c2 = stats_on ? clock64() : 0;
        if (stats_on) {
          ++st_pass; st_push += s_npend; st_apply += c2 - c1; st_poll += c1 - c0;
          st_max = max(st_max, static_cast<unsigned long long>(s_npend));
        }
        if (warp == 0) {
          if (lane == 0) {
            const uint32_t npush = __popc(p_taken);
            const uint32_t rounds = (31u - __clz(p_taken)) / nw + 1u;   // lanes are round-major
            const uint32_t nsteps = (P.apply_mode == APPLY_MERGED) ? rounds : npush;
            PsItemState ns = st;
            ns.t += nsteps;
            for (uint32_t k = 0; k < nsteps; ++k) { ns.beta1_pow *= P.beta1; ns.beta2_pow *= P.beta2; }
            // one schedule step per push, in both apply modes (also the num_updates of the averaging kernels)
            if constexpr (kSched) ns.sched_step += npush;
            s_state[own] = ns;
            P.item_state[item] = ns;   // persisted for checkpoints / a relaunch (never read back in this loop)
          }
          if (p_take) {
            const uint32_t slot = p_seq % P.nslots;
            const uint32_t done = atomicAdd(&P.consumed[pw * P.nslots + slot], 1u) + 1u;
            if (done == static_cast<uint32_t>(P.n_items)) {
              // this worker's push `p_seq` is fully applied: one global step (reference DS:91,103)
              P.consumed[pw * P.nslots + slot] = 0;
              const uint32_t gs = atomicAdd(P.global_step, 1u) + 1u;
              uint32_t* ib = P.inbox_table[pw];
              if (ib != nullptr) {
                red_max_relaxed_scoped_u32(ib + 1, gs, P.gpu_scope);
                red_max_release_scoped_u32(ib, p_seq, P.gpu_scope);  // ack: the mailbox slot may be reused
              }
            }
          }
          if (pvalid && pk == 0 && p_cnt > 0) {
            const uint32_t nx = p_seq + p_cnt;
            s_next[own][pw] = nx;
            P.next_seq[static_cast<size_t>(pw) * P.n_items + item] = nx;
          }
        }
        if (stats_on) { __syncwarp(); st_book += clock64() - c2; }
      }
      __syncthreads();
    }
    // ---- exit protocol: host stop request, or every worker has left and all their pushes are applied ----
    // (checked every 32nd poll round only: the check itself costs several system-scope loads, and the poll
    //  loop's period is the PS's reaction latency)
    if (tid == 0) {
      uint32_t ex = 0;
      // one-shot mode: everything that will ever be pushed was pushed before this launch (stream order), so a
      // full sweep without work means the shard is up to date
      if (P.oneshot && !sweep_any) ex = 1;
      const bool check = !P.oneshot && (iter & 31u) == 0u;
      if (check && *P.host_stop != 0u) ex = 1;
      if (check && !ex) {
        bool all_done = true;
        for (int w = 0; w < P.n_workers && all_done; ++w) {
          const uint32_t d = ld_acquire_sys_u32(P.worker_done + w);  // = last push seq + 1, 0 while active
          if (d == 0) { all_done = false; break; }
          if (d == kWorkerDead) continue;   // presumed dead: whatever it left half-pushed is dropped
          for (int own = 0; own < n_own; ++own)
            if (s_next[own][w] != d) { all_done = false; break; }
        }
        if (all_done) ex = 1;
      }
      s_exit = ex;
    }
    __syncthreads();
    if (s_exit) break;
    ++iter;
  }
  if (tid == 0) {
    if (stats_on) {
      unsigned long long* o = P.stats + static_cast<size_t>(blockIdx.x) * 8;
      o[0] += st_pass; o[1] += st_push; o[2] += st_apply; o[3] += st_book; o[4] += st_idle_n; o[5] += st_idle;
      o[6] = max(o[6], st_max); o[7] += st_poll;
      P.stats[kPsStatsCtas * 8 + blockIdx.x] = sm_id();
    }
    atomicAdd(P.exit_counter, 1u);
  }
}

using ServeKernel = void (*)(PsServeParams);
template <int kFam, bool kIeee>
ServeKernel serve_kernel_at(bool sched, bool ema) {
  if (ema) return ps_serve_kernel<kFam, kIeee, true, true>;
  if (sched) return ps_serve_kernel<kFam, kIeee, true, false>;
  return ps_serve_kernel<kFam, kIeee, false, false>;
}
template <int kFam>
ServeKernel serve_kernel_of(bool ieee, bool sched, bool ema) {
  // Momentum has no square root or divide: its one instantiation serves both math modes. ProximalGradientDescent has no
  // square root: its one has the IEEE divide.
  if constexpr (kFam == OPT_MOMENTUM) return serve_kernel_at<kFam, false>(sched, ema);
  else if constexpr (kFam == OPT_PROXIMAL_SGD) return serve_kernel_at<kFam, true>(sched, ema);
  else return ieee ? serve_kernel_at<kFam, true>(sched, ema) : serve_kernel_at<kFam, false>(sched, ema);
}
// The serve-kernel instantiation for optimizer `opt` (OptimizerKind) in math mode `ieee`, with a non-constant schedule
// (`sched`) and moving averages (`ema`, which takes the scheduled path whatever `sched` is); null for an unknown `opt`.
ServeKernel serve_kernel(int opt, bool ieee, bool sched, bool ema) {
  switch (opt) {
    case OPT_SGD:
    case OPT_ADAM: return serve_kernel_of<kFamAdamSgd>(ieee, sched, ema);
    case OPT_MOMENTUM: return serve_kernel_of<OPT_MOMENTUM>(ieee, sched, ema);
    case OPT_ADAGRAD: return serve_kernel_of<OPT_ADAGRAD>(ieee, sched, ema);
    // AdagradDA's T is the item's sched_step, which only the scheduled and averaging instantiations advance
    case OPT_ADAGRAD_DA: return serve_kernel_of<OPT_ADAGRAD>(ieee, true, ema);
    case OPT_RMSPROP: return serve_kernel_of<OPT_RMSPROP>(ieee, sched, ema);
    case OPT_ADADELTA: return serve_kernel_of<OPT_ADADELTA>(ieee, sched, ema);
    case OPT_FTRL: return serve_kernel_of<OPT_FTRL>(ieee, sched, ema);
    case OPT_PROXIMAL_ADAGRAD: return serve_kernel_of<OPT_PROXIMAL_ADAGRAD>(ieee, sched, ema);
    case OPT_PROXIMAL_SGD: return serve_kernel_of<OPT_PROXIMAL_SGD>(ieee, sched, ema);
    default: return nullptr;
  }
}

// `cluster` > 1: the grid is launched as clusters of that many CTAs. The kernel has no cluster-scope code; the
// clusters only make the hardware place the CTAs GPC by GPC (a cluster lives inside one GPC), so that they leave
// whole GPCs' worth of SMs to the 8-CTA clusters of a fused worker step kernel on the same GPU.
cudaError_t launch_ps_serve(const PsServeParams& p, int n_ctas, int cluster, cudaStream_t stream) {
  if (p.n_workers > kMaxWorkers || p.n_workers < 1 || cluster < 1 || cluster > 8) return cudaErrorInvalidValue;
  const int max_ctas = (p.n_items + cluster - 1) / cluster * cluster;   // whole clusters: a CTA may own no item
  if (n_ctas > max_ctas) n_ctas = max_ctas;
  const int min_ctas = (p.n_items + kMaxOwn - 1) / kMaxOwn;  // a CTA caches at most kMaxOwn items
  if (n_ctas < min_ctas) n_ctas = min_ctas;
  if (n_ctas < 1) n_ctas = 1;
  if (n_ctas % cluster != 0) return cudaErrorInvalidValue;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(n_ctas);
  cfg.blockDim = dim3(kPsThreads);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = cluster > 1 ? 1 : 0;
  const ServeKernel k = serve_kernel(p.opt, p.ieee_math != 0u, p.lr_schedule != LR_CONSTANT, p.ema != nullptr);
  if (k == nullptr) return cudaErrorInvalidValue;
  return cudaLaunchKernelEx(&cfg, k, p);
}

// ------------------------------------------------------------------------------------------
// One-shot dense optimizer apply over a flat range (synchronous baselines: NCCL reduce + apply,
// host-staged gRPC stand-in on the GPU, unit tests of the update rule).
// ------------------------------------------------------------------------------------------
__global__ void dense_apply_kernel(float* __restrict__ params, float* __restrict__ m, float* __restrict__ v,
                                   const float* __restrict__ grad, uint16_t* __restrict__ shadow, size_t n, int opt,
                                   float lr, float beta1, float beta2, float eps, float lr_t) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float p = params[i];
    const float g = grad[i];
    if (opt == OPT_ADAM) {
      float mm = m[i], vv = v[i];
      adam_step(p, mm, vv, g, lr_t, beta1, beta2, eps);
      m[i] = mm;
      v[i] = vv;
    } else {
      p = fmaf(-lr, g, p);
    }
    params[i] = p;
    if (shadow != nullptr) {
      __nv_bfloat16 b = __float2bfloat16(p);
      shadow[i] = *reinterpret_cast<uint16_t*>(&b);
    }
  }
}

cudaError_t launch_dense_apply(float* params, float* m, float* v, const float* grad, uint16_t* shadow, size_t n,
                               int opt, float lr, float beta1, float beta2, float eps, uint32_t t,
                               cudaStream_t stream) {
  float lr_t = lr;
  if (opt == OPT_ADAM) lr_t = lr * sqrtf(1.f - powf(beta2, static_cast<float>(t))) / (1.f - powf(beta1, static_cast<float>(t)));
  const int threads = 256;
  int blocks = static_cast<int>((n + threads - 1) / threads);
  if (blocks > device_sm_count() * 8) blocks = device_sm_count() * 8;
  if (blocks < 1) blocks = 1;
  dense_apply_kernel<<<blocks, threads, 0, stream>>>(params, m, v, grad, shadow, n, opt, lr, beta1, beta2, eps, lr_t);
  return cudaGetLastError();
}

// fp32 -> bf16 shadow refresh for a flat range (chief init / checkpoint restore).
__global__ void shadow_refresh_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    __nv_bfloat16 b = __float2bfloat16(src[i]);
    dst[i] = *reinterpret_cast<uint16_t*>(&b);
  }
}
cudaError_t launch_shadow_refresh(const float* src, uint16_t* dst, size_t n, cudaStream_t stream) {
  const int threads = 256;
  int blocks = static_cast<int>((n + threads - 1) / threads);
  if (blocks > device_sm_count() * 8) blocks = device_sm_count() * 8;
  if (blocks < 1) blocks = 1;
  shadow_refresh_kernel<<<blocks, threads, 0, stream>>>(src, dst, n);
  return cudaGetLastError();
}

// Stream-ordered "all my pushes are applied" fence on the worker: spins (locally — the PS writes the inbox
// into the worker's HBM) until every shard has acknowledged the worker's latest push. Lets a CUDA-event
// timed region include the PS-side apply of its last step.
__global__ void wait_ack_kernel(const uint32_t* inbox, uint32_t n_inbox, const uint32_t* seq_ptr) {
  const uint32_t seq = *reinterpret_cast<const volatile uint32_t*>(seq_ptr);
  const uint64_t t0 = globaltimer_ns();
  for (uint32_t i = 0; i < n_inbox; ++i) {
    while (static_cast<int32_t>(ld_acquire_sys_u32(inbox + 2 * i) - seq) < 0) {
      if (globaltimer_ns() - t0 > DM_SPIN_TIMEOUT_NS) {
        printf("[dm] wait_ack: shard %u stuck at ack=%u, seq=%u\n", i, inbox[2 * i], seq);
        __trap();
      }
    }
  }
}
cudaError_t launch_wait_ack(const uint32_t* inbox, uint32_t n_inbox, const uint32_t* seq_ptr, cudaStream_t stream) {
  wait_ack_kernel<<<1, 1, 0, stream>>>(inbox, n_inbox, seq_ptr);
  return cudaGetLastError();
}

// Worker leaves the session: publish last_seq + 1 into the PS's worker_done slot (peer store).
__global__ void worker_done_kernel(uint32_t* done_slot, const uint32_t* seq_ptr) {
  __threadfence_system();
  st_release_sys_u32(done_slot, *seq_ptr + 1u);
}
cudaError_t launch_worker_done(uint32_t* done_slot, const uint32_t* seq_ptr, cudaStream_t stream) {
  worker_done_kernel<<<1, 1, 0, stream>>>(done_slot, seq_ptr);
  return cudaGetLastError();
}

}  // namespace dm

namespace dm {
// Force-load every kernel of this translation unit (DESIGN §7). The serve kernels are enumerated through serve_kernel,
// so every one that launch_ps_serve can pick is loaded here.
cudaError_t prepare_ps_kernels() {
  cudaFuncAttributes a;
  cudaError_t e;
  for (int opt = OPT_SGD; opt <= OPT_ADAGRAD_DA; ++opt)
    for (const bool ieee : {false, true})
      for (const bool sched : {false, true})
        for (const bool ema : {false, true})
          if ((e = cudaFuncGetAttributes(&a, serve_kernel(opt, ieee, sched, ema))) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, dense_apply_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, shadow_refresh_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, wait_ack_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, worker_done_kernel)) != cudaSuccess) return e;
  return cudaSuccess;
}
}  // namespace dm
