// Parameter-server shard kernels for sm_90a.
//
// ps_serve_kernel is the PS "process" of the reference (tf.train.Server(...).join(),
// /root/reference/distributed_server-basic.py:80-83) turned into a persistent GPU kernel: it owns the
// shard (params + Adam slots + global_step, DS:88-91,102-103), polls the per-item flags that workers
// publish with st.release.sys after their in-kernel P2P gradient stores, reduces whatever is ready
// (many-to-one) and applies the optimizer in the same pass (ApplyAdam / SGD, SURVEY K7), bumps
// global_step (K8) and acknowledges into the worker's inbox over NVLink. No host, NCCL or gRPC in the loop.
//
// Work decomposition: items (2-D blocks of the arena) are dealt round-robin to CTAs; a CTA never shares
// an item, so item state (Adam step count / beta powers) needs no synchronisation. Pushes of one worker
// are consumed in order per item; different workers interleave arbitrarily (Hogwild, like the reference's
// unlocked async apply).
#include "common.cuh"
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

template <bool kIeee>
__device__ void apply_item(const PsServeParams& P, const PsItem it, const PsItemState st, const uint64_t* s_pend,
                           const uint32_t* s_round, const int n_pend, ResidentState* res = nullptr) {
  const int tid = threadIdx.x;
  const int total = it.rows * it.cols;
  const bool vec = ((it.cols & 3) == 0) && ((it.ld & 3) == 0) && ((it.offset & 3) == 0);
  const int step = vec ? 4 : 1;
  const bool adam = P.opt == OPT_ADAM;
  const bool merged = P.apply_mode == APPLY_MERGED;
  for (int e0 = tid * step; e0 < total; e0 += kPsThreads * step * kQuads) {
    uint64_t a[kQuads];
    bool ok[kQuads];
    float pv[kQuads][4], mv[kQuads][4], vv[kQuads][4];
#pragma unroll
    for (int q = 0; q < kQuads; ++q) {
      const int e = e0 + q * kPsThreads * step;
      ok[q] = e < total;
      const int r = ok[q] ? e / it.cols : 0;
      const int c = ok[q] ? e - r * it.cols : 0;
      a[q] = it.offset + static_cast<uint64_t>(r) * it.ld + c;
#pragma unroll
      for (int j = 0; j < 4; ++j) { pv[q][j] = 0.f; mv[q][j] = 0.f; vv[q][j] = 0.f; }
    }
    if (res != nullptr && res->loaded) {
      // the item's parameters and Adam slots never left this thread's registers: no load round trip in this pass
#pragma unroll
      for (int q = 0; q < kQuads; ++q)
#pragma unroll
        for (int j = 0; j < 4; ++j) { pv[q][j] = res->p[q][j]; mv[q][j] = res->m[q][j]; vv[q][j] = res->v[q][j]; }
    } else {
#pragma unroll
      for (int q = 0; q < kQuads; ++q) {
        if (!ok[q]) continue;
        if (vec) {
          const float4 t = __ldcg(reinterpret_cast<const float4*>(P.params + a[q]));
          pv[q][0] = t.x; pv[q][1] = t.y; pv[q][2] = t.z; pv[q][3] = t.w;
          if (adam) {
            const float4 tm = __ldcg(reinterpret_cast<const float4*>(P.adam_m + a[q]));
            const float4 tv = __ldcg(reinterpret_cast<const float4*>(P.adam_v + a[q]));
            mv[q][0] = tm.x; mv[q][1] = tm.y; mv[q][2] = tm.z; mv[q][3] = tm.w;
            vv[q][0] = tv.x; vv[q][1] = tv.y; vv[q][2] = tv.z; vv[q][3] = tv.w;
          }
        } else {
          pv[q][0] = __ldcg(P.params + a[q]);
          if (adam) { mv[q][0] = __ldcg(P.adam_m + a[q]); vv[q][0] = __ldcg(P.adam_v + a[q]); }
        }
      }
    }
    float b1p = st.beta1_pow, b2p = st.beta2_pow;
    float gsum[kQuads][4];
#pragma unroll
    for (int q = 0; q < kQuads; ++q)
#pragma unroll
      for (int j = 0; j < 4; ++j) gsum[q][j] = 0.f;

    for (int i0 = 0; i0 < n_pend; i0 += kChunk) {
      float g[kChunk][kQuads][4];
#pragma unroll
      for (int ci = 0; ci < kChunk; ++ci) {
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
      for (int ci = 0; ci < kChunk; ++ci) {
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
        float lr_t = P.lr;
        if (adam) {
          b1p *= P.beta1;
          b2p *= P.beta2;
          lr_t = adam_lr_t<kIeee>(P.lr, b1p, b2p);
        }
#pragma unroll
        for (int q = 0; q < kQuads; ++q) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (j >= step) continue;
            const float gv = merged ? gsum[q][j] : g[ci][q][j];
            if (adam) adam_step<kIeee>(pv[q][j], mv[q][j], vv[q][j], gv, lr_t, P.beta1, P.beta2, P.eps);
            else pv[q][j] = fmaf(-P.lr, gv, pv[q][j]);
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
      res->loaded = true;
    }
#pragma unroll
    for (int q = 0; q < kQuads; ++q) {
      if (!ok[q]) continue;
      const bool shadow = P.shadow_bf16 != nullptr && (it.flags & 1);
      if (vec) {
        *reinterpret_cast<float4*>(P.params + a[q]) = make_float4(pv[q][0], pv[q][1], pv[q][2], pv[q][3]);
        if (adam) {
          *reinterpret_cast<float4*>(P.adam_m + a[q]) = make_float4(mv[q][0], mv[q][1], mv[q][2], mv[q][3]);
          *reinterpret_cast<float4*>(P.adam_v + a[q]) = make_float4(vv[q][0], vv[q][1], vv[q][2], vv[q][3]);
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
        if (adam) { P.adam_m[a[q]] = mv[q][0]; P.adam_v[a[q]] = vv[q][0]; }
        if (shadow) {
          __nv_bfloat16 b = __float2bfloat16(pv[q][0]);
          P.shadow_bf16[a[q]] = *reinterpret_cast<uint16_t*>(&b);
        }
      }
    }
  }
}

template <bool kIeee>
__global__ void __launch_bounds__(kPsThreads, 1) ps_serve_kernel(const __grid_constant__ PsServeParams P) {
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
      }
      __syncthreads();
      const long long c1 = stats_on ? clock64() : 0;
      if (!s_any && stats_on) { ++st_idle_n; st_idle += c1 - c0; }
      if (s_any) {
        sweep_any = true;
        const PsItemState st = s_state[own];
        apply_item<kIeee>(P, s_item[own], st, s_pend, s_round, static_cast<int>(s_npend), use_resident ? &resident : nullptr);
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
    }
    atomicAdd(P.exit_counter, 1u);
  }
}

cudaError_t launch_ps_serve(const PsServeParams& p, int n_ctas, cudaStream_t stream) {
  if (p.n_workers > kMaxWorkers || p.n_workers < 1) return cudaErrorInvalidValue;
  if (n_ctas > p.n_items) n_ctas = p.n_items;
  const int min_ctas = (p.n_items + kMaxOwn - 1) / kMaxOwn;  // a CTA caches at most kMaxOwn items
  if (n_ctas < min_ctas) n_ctas = min_ctas;
  if (n_ctas < 1) n_ctas = 1;
  if (p.ieee_math) ps_serve_kernel<true><<<n_ctas, kPsThreads, 0, stream>>>(p);
  else ps_serve_kernel<false><<<n_ctas, kPsThreads, 0, stream>>>(p);
  return cudaGetLastError();
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
  if ((e = cudaFuncGetAttributes(&a, dense_apply_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, shadow_refresh_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, wait_ack_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, worker_done_kernel)) != cudaSuccess) return e;
  return cudaSuccess;
}
}  // namespace dm
