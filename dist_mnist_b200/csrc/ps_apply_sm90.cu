// Parameter-server shard kernels for sm_90a.
//
// ps_serve_kernel is the PS "process" of the reference (tf.train.Server(...).join(),
// /root/reference/distributed_server-basic.py:80-83) turned into a persistent GPU kernel: it owns the
// shard (params + Adam slots + global_step, DS:88-91,102-103), polls the per-item flags that workers
// publish with st.release.sys after their in-kernel P2P gradient stores, reduces whatever is ready
// (many-to-one) and applies the optimizer in the same pass (ApplyAdam / SGD, SURVEY K7; or TF1's
// ApplyMomentum / ApplyAdagrad / ApplyRMSProp in their own instantiations), bumps
// global_step (K8) and acknowledges into the worker's inbox over NVLink. No host, NCCL or gRPC in the loop.
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
constexpr int kChunk = 8;     // pending pushes whose gradient loads are in flight together
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
// kSched: the step's rate is `lr_sched`; else P.lr (read from the parameter block as the measured instantiations do)
template <int kOpt, bool kIeee, bool kSched>
__device__ __forceinline__ void tf1_step(float& p, float& m, float& v, float g, const PsServeParams& P,
                                         const float& lr_sched) {
  const float& lr = kSched ? lr_sched : P.lr;
  if constexpr (kOpt == OPT_MOMENTUM) {
    // accum <- momentum accum + g ; p <- p - lr accum  (Nesterov: p <- p - lr g - lr momentum accum)
    m = fmaf(P.momentum, m, g);
    if (P.nesterov) p = p - fmaf(g, lr, m * P.momentum * lr);
    else p = fmaf(-lr, m, p);
  } else if constexpr (kOpt == OPT_ADAGRAD) {
    // accum <- accum + g^2 ; p <- p - lr g / sqrt(accum)   (no epsilon)
    v = fmaf(g, g, v);
    p = p - div_sqrt<kIeee>(lr * g, v);
  } else {
    static_assert(kOpt == OPT_RMSPROP, "unknown optimizer family");
    // ms <- ms + (g^2 - ms)(1 - decay) ; mom <- momentum mom + lr g / sqrt(ms + eps) ; p <- p - mom
    v = fmaf(fmaf(g, g, -v), 1.f - P.decay, v);
    m = fmaf(P.momentum, m, div_sqrt<kIeee>(lr * g, v + P.eps));
    p = p - m;
  }
}

// Optimizer family of a serve-kernel instantiation. Adam and SGD share the two instantiations that were measured (P.opt
// picks the rule at run time; their SASS is unchanged by the other families); every other kind gets its own.
constexpr int kFamAdamSgd = -1;

// Apply every pending push to one item. s_pend[0..n_pend) lists the mailbox slots (element offset of the slot
// inside P.mailbox) in application order — round k = the k-th pending push of every worker, oldest round first —
// and s_round[i] is the round of entry i. One optimizer step per push, or per round in APPLY_MERGED mode
// (concurrent pushes of different workers are summed; consecutive pushes of one worker stay separate steps).
// Parameters and Adam slots stay in registers for the whole pass; the gradient loads of kChunk pushes are issued
// together (a mailbox line costs an L2/HBM round trip of ~1-2 us: issuing them one push at a time made the
// pass, and with it the push->ack latency that throttles the workers, proportional to 5 us x pending pushes).
// Optimizer state of an item held in registers across passes (see ps_serve_kernel): valid when the CTA owns exactly one
// item that fits one sweep of the CTA (<= kPsThreads * kQuads * 4 elements, vectorisable).
struct ResidentState {
  float p[kQuads][4], m[kQuads][4], v[kQuads][4];
  bool loaded;
};
// The moving averages of that item (the averaging instantiations), valid whenever ResidentState::loaded is.
struct ResidentEma {
  float e[kQuads][4];
};
// Gradient loads in flight in the averaging instantiations (see kCh in apply_item).
template <int kFam, bool kIeee>
constexpr int kChEma() {
  if constexpr (kFam == kFamAdamSgd) return kIeee ? kChunk - 3 : kChunk - 2;
  else return (kFam == OPT_ADAGRAD || kIeee) ? kChunk - 2 : kChunk - 1;
}

// kSched (the scheduled instantiations): the rate of the optimizer step whose pushes sit at positions i0..i1 of the
// application order is s_lr[i0], the pass's rate table (lr(sched_step + i), built by the serve loop); else P.lr.
// kEma (the averaging instantiations, which are also kSched): the item's moving averages P.ema stay in registers for
// the pass like the parameters, and after the optimizer step that ends at position i every element's shadow moves
// toward the new parameter by 1 - s_ema[i], the pass's decay table (ema_decay(sched_step + i + 1)).
template <bool kIeee, int kFam, bool kSched = false, bool kEma = false>
__device__ void apply_item(const PsServeParams& P, const PsItem it, const PsItemState st, const uint64_t* s_pend,
                           const uint32_t* s_round, const int n_pend, ResidentState* res = nullptr,
                           const float* s_lr = nullptr, const float* s_ema = nullptr,
                           ResidentEma* res_ema = nullptr) {
  const int tid = threadIdx.x;
  const int total = it.rows * it.cols;
  const bool vec = ((it.cols & 3) == 0) && ((it.ld & 3) == 0) && ((it.offset & 3) == 0);
  const int step = vec ? 4 : 1;
  const bool adam = kFam == kFamAdamSgd && P.opt == OPT_ADAM;
  // the slot buffers this rule reads and writes
  const bool use_m = kFam == kFamAdamSgd ? adam : (kFam == OPT_MOMENTUM || kFam == OPT_RMSPROP);
  const bool use_v = kFam == kFamAdamSgd ? adam : (kFam == OPT_ADAGRAD || kFam == OPT_RMSPROP);
  const bool merged = P.apply_mode == APPLY_MERGED;
  for (int e0 = tid * step; e0 < total; e0 += kPsThreads * step * kQuads) {
    uint64_t a[kQuads];
    bool ok[kQuads];
    float pv[kQuads][4], mv[kQuads][4], vv[kQuads][4];
    float ev[kQuads][4];   // kEma: the shadows
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
          for (int j = 0; j < 4; ++j) ev[q][j] = res_ema->e[q][j];
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
        } else {
          pv[q][0] = __ldcg(P.params + a[q]);
          if (use_m) mv[q][0] = __ldcg(P.adam_m + a[q]);
          if (use_v) vv[q][0] = __ldcg(P.adam_v + a[q]);
          if constexpr (kEma) ev[q][0] = __ldcg(P.ema + a[q]);
        }
      }
    }
    float b1p = st.beta1_pow, b2p = st.beta2_pow;
    float gsum[kQuads][4];
#pragma unroll
    for (int q = 0; q < kQuads; ++q)
#pragma unroll
      for (int j = 0; j < 4; ++j) gsum[q][j] = 0.f;

    // the other families' straight-line update keeps more values live: a chunk of 8 spills there, 7 does not. The
    // scheduled Adam / SGD instantiations (rate-table read, round start) spill at 8 too, and the IEEE one still at 7:
    // 7 and 6 there; the scheduled Momentum / Adagrad / RMSProp ones do not spill at 7.
    constexpr int kChNoEma = kFam != kFamAdamSgd ? kChunk - 1 : !kSched ? kChunk : kIeee ? kChunk - 2 : kChunk - 1;
    // The averaging instantiations hold 8 shadows more per thread (kChEma): Momentum and fast RMSProp do not spill at
    // 7; Adagrad (both), IEEE RMSProp and fast Adam / SGD spill at 7 and take 6; IEEE Adam / SGD spills at 6 and
    // takes 5.
    constexpr int kCh = kEma ? kChEma<kFam, kIeee>() : kChNoEma;
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
#pragma unroll
        for (int q = 0; q < kQuads; ++q) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (j >= step) continue;
            const float gv = merged ? gsum[q][j] : g[ci][q][j];
            if constexpr (kFam != kFamAdamSgd) tf1_step<kFam, kIeee, kSched>(pv[q][j], mv[q][j], vv[q][j], gv, P, lr);
            else if (adam) adam_step<kIeee>(pv[q][j], mv[q][j], vv[q][j], gv, lr_t, P.beta1, P.beta2, P.eps);
            else pv[q][j] = fmaf(-lr, gv, pv[q][j]);
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
          for (int j = 0; j < 4; ++j) res_ema->e[q][j] = ev[q][j];
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
        if (shadow) {
          __nv_bfloat16 b = __float2bfloat16(pv[q][0]);
          P.shadow_bf16[a[q]] = *reinterpret_cast<uint16_t*>(&b);
        }
      }
    }
  }
}

// Adam / SGD: ps_serve_kernel<kIeee>, the two instantiations that were measured.
template <bool kIeee>
__global__ void __launch_bounds__(kPsThreads, 1) ps_serve_kernel(const __grid_constant__ PsServeParams P) {
  constexpr int kFam = kFamAdamSgd;
  constexpr bool kSched = false;
  constexpr bool kEma = false;
#include "ps_serve_body.cuh"
}
// Momentum / Adagrad / RMSProp: ps_serve_kernel<kOpt, kIeee>.
template <int kOpt, bool kIeee>
__global__ void __launch_bounds__(kPsThreads, 1) ps_serve_kernel(const __grid_constant__ PsServeParams P) {
  constexpr int kFam = kOpt;
  constexpr bool kSched = false;
  constexpr bool kEma = false;
#include "ps_serve_body.cuh"
}
// Any family under a non-constant learning-rate schedule (P.lr_schedule != LR_CONSTANT): ps_serve_sched_kernel<kFam,
// kIeee>. Separate instantiations keep the seven above, and with them every constant-rate run, exactly as measured.
template <int kFamT, bool kIeee>
__global__ void __launch_bounds__(kPsThreads, 1) ps_serve_sched_kernel(const __grid_constant__ PsServeParams P) {
  constexpr int kFam = kFamT;
  constexpr bool kSched = true;
  constexpr bool kEma = false;
#include "ps_serve_body.cuh"
}
// Any family with moving averages of the parameters (P.ema != null), under any schedule: ps_serve_ema_kernel<kFam,
// kIeee>. The rate table is compiled in as in the scheduled kernels (scheduled_lr is lr0 for LR_CONSTANT), so one
// set serves a constant rate and every schedule; the fourteen above stay exactly as measured.
template <int kFamT, bool kIeee>
__global__ void __launch_bounds__(kPsThreads, 1) ps_serve_ema_kernel(const __grid_constant__ PsServeParams P) {
  constexpr int kFam = kFamT;
  constexpr bool kSched = true;
  constexpr bool kEma = true;
#include "ps_serve_body.cuh"
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
  if (p.ema != nullptr) {
    switch (p.opt) {
      case OPT_SGD:
      case OPT_ADAM:
        if (p.ieee_math) return cudaLaunchKernelEx(&cfg, ps_serve_ema_kernel<kFamAdamSgd, true>, p);
        return cudaLaunchKernelEx(&cfg, ps_serve_ema_kernel<kFamAdamSgd, false>, p);
      case OPT_MOMENTUM:
        return cudaLaunchKernelEx(&cfg, ps_serve_ema_kernel<OPT_MOMENTUM, false>, p);
      case OPT_ADAGRAD:
        if (p.ieee_math) return cudaLaunchKernelEx(&cfg, ps_serve_ema_kernel<OPT_ADAGRAD, true>, p);
        return cudaLaunchKernelEx(&cfg, ps_serve_ema_kernel<OPT_ADAGRAD, false>, p);
      case OPT_RMSPROP:
        if (p.ieee_math) return cudaLaunchKernelEx(&cfg, ps_serve_ema_kernel<OPT_RMSPROP, true>, p);
        return cudaLaunchKernelEx(&cfg, ps_serve_ema_kernel<OPT_RMSPROP, false>, p);
      default:
        return cudaErrorInvalidValue;
    }
  }
  if (p.lr_schedule != LR_CONSTANT) {
    switch (p.opt) {
      case OPT_SGD:
      case OPT_ADAM:
        if (p.ieee_math) return cudaLaunchKernelEx(&cfg, ps_serve_sched_kernel<kFamAdamSgd, true>, p);
        return cudaLaunchKernelEx(&cfg, ps_serve_sched_kernel<kFamAdamSgd, false>, p);
      case OPT_MOMENTUM:
        return cudaLaunchKernelEx(&cfg, ps_serve_sched_kernel<OPT_MOMENTUM, false>, p);
      case OPT_ADAGRAD:
        if (p.ieee_math) return cudaLaunchKernelEx(&cfg, ps_serve_sched_kernel<OPT_ADAGRAD, true>, p);
        return cudaLaunchKernelEx(&cfg, ps_serve_sched_kernel<OPT_ADAGRAD, false>, p);
      case OPT_RMSPROP:
        if (p.ieee_math) return cudaLaunchKernelEx(&cfg, ps_serve_sched_kernel<OPT_RMSPROP, true>, p);
        return cudaLaunchKernelEx(&cfg, ps_serve_sched_kernel<OPT_RMSPROP, false>, p);
      default:
        return cudaErrorInvalidValue;
    }
  }
  switch (p.opt) {
    case OPT_SGD:
    case OPT_ADAM:
      if (p.ieee_math) return cudaLaunchKernelEx(&cfg, ps_serve_kernel<true>, p);
      return cudaLaunchKernelEx(&cfg, ps_serve_kernel<false>, p);
    case OPT_MOMENTUM:   // no square root: one instantiation serves both math modes
      return cudaLaunchKernelEx(&cfg, ps_serve_kernel<OPT_MOMENTUM, false>, p);
    case OPT_ADAGRAD:
      if (p.ieee_math) return cudaLaunchKernelEx(&cfg, ps_serve_kernel<OPT_ADAGRAD, true>, p);
      return cudaLaunchKernelEx(&cfg, ps_serve_kernel<OPT_ADAGRAD, false>, p);
    case OPT_RMSPROP:
      if (p.ieee_math) return cudaLaunchKernelEx(&cfg, ps_serve_kernel<OPT_RMSPROP, true>, p);
      return cudaLaunchKernelEx(&cfg, ps_serve_kernel<OPT_RMSPROP, false>, p);
    default:
      return cudaErrorInvalidValue;
  }
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
// Force-load every kernel of this translation unit. With CUDA's lazy module loading the *first* launch of a
// kernel may need a context-wide synchronisation; if that first launch happens while the persistent serve
// kernel is resident (and the serve kernel is waiting for the new kernel's flags) the process deadlocks.
cudaError_t preload_ps_kernels() {
  cudaFuncAttributes a;
  cudaError_t e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_kernel<false>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_kernel<true>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_kernel<OPT_MOMENTUM, false>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_kernel<OPT_ADAGRAD, false>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_kernel<OPT_ADAGRAD, true>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_kernel<OPT_RMSPROP, false>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_kernel<OPT_RMSPROP, true>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_sched_kernel<kFamAdamSgd, false>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_sched_kernel<kFamAdamSgd, true>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_sched_kernel<OPT_MOMENTUM, false>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_sched_kernel<OPT_ADAGRAD, false>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_sched_kernel<OPT_ADAGRAD, true>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_sched_kernel<OPT_RMSPROP, false>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_sched_kernel<OPT_RMSPROP, true>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_ema_kernel<kFamAdamSgd, false>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_ema_kernel<kFamAdamSgd, true>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_ema_kernel<OPT_MOMENTUM, false>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_ema_kernel<OPT_ADAGRAD, false>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_ema_kernel<OPT_ADAGRAD, true>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_ema_kernel<OPT_RMSPROP, false>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, ps_serve_ema_kernel<OPT_RMSPROP, true>)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, dense_apply_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, shadow_refresh_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, wait_ack_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, worker_done_kernel)) != cudaSuccess) return e;
  return cudaSuccess;
}
}  // namespace dm
