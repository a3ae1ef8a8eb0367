// Gradient clipping tail of the graph engine's step (sm_90a).
//
// With clipping on, every push target of a step graph (the head, the dX colsum and the dW epilogues) points at a
// worker-local gradient buffer of the step's ring slot instead of the ps mailbox (a PUSH_MAILBOX target with slot
// stride 0 and worker-local flags, so the epilogues themselves are unchanged). The global norm is known only after
// the last of them, so three kernels close the step:
//
//   grad_clip_ssq_kernel      per-block partial sums of squares of every variable (grid-stride over its elements,
//                             a fixed block reduction): no float atomics, the same partials on every run
//   grad_clip_apply_kernel    every block adds the partials in the same fixed order and derives the factor of every
//                             variable (grad_clip.cuh), then writes g' into this worker's mailbox slot of the owning
//                             shard and zeroes the local buffer for the slot's next step (the colsum epilogue
//                             accumulates when it runs more than one batch tile)
//   grad_clip_release_kernel  once every store of the apply kernel has completed (stream order, no programmatic
//                             early launch): a fence at the flags' scope, then every flag of this worker's slot on every
//                             shard it pushes to is released with the step's push sequence number
//
// CLIP_VALUE needs no sums: the ssq kernel is not captured and the apply kernel clamps.
//
// L2 weight regularization (the <true> instantiations; GradClipParams::l2_scale != 0, with or without a clip) takes the
// same route: the ssq kernel also sums w*w per block and, for the clip norms, squares g' = fl(g + fl(S * w)) instead of
// g, where w is read from the owning shard (as the dX GEMM pulls W a second time); the apply kernel writes the clipped
// g' (or g' itself under CLIP_OFF), and its block 0 adds S * sum(w*w) / 2 to the slot's StepResult loss, the partials
// summed in a fixed order.
#include "common.cuh"
#include "grad_clip.cuh"

namespace dm {

constexpr int kClipThreads = 256;
constexpr int kClipBlocks = 132;

// the block sum of v (warp shuffles, then the warps in order) into *out from thread 0
template <typename F>
__device__ __forceinline__ void clip_block_sum(float v, float* s_warp, F&& store) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float b = 0.f;
#pragma unroll
    for (int w = 0; w < kClipThreads / 32; ++w) b += s_warp[w];
    store(b);
  }
  __syncthreads();
}

// g' = fl(g + fl(S * w)), as TF's L2LossGrad followed by the ADD_N of the two gradients
__device__ __forceinline__ float l2_grad(float g, float s, float w) { return __fadd_rn(g, __fmul_rn(s, w)); }

template <bool kL2>
__global__ void __launch_bounds__(kClipThreads) grad_clip_ssq_kernel(const __grid_constant__ GradClipParams p) {
  __shared__ float s_warp[kClipThreads / 32];
  for (int v = 0; v < p.n_vars; ++v) {
    const GradClipVar& var = p.var[v];
    const uint64_t n = static_cast<uint64_t>(var.rows) * var.cols;
    float acc = 0.f;
    if constexpr (kL2) {
      const float* w = p.l2_w[v];
      const bool norms = p.kind == CLIP_GLOBAL_NORM || p.kind == CLIP_NORM;
      float reg = 0.f;
      for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kClipThreads + threadIdx.x; i < n;
           i += static_cast<uint64_t>(gridDim.x) * kClipThreads) {
        const uint64_t e = (i / var.cols) * var.ld + i % var.cols;
        float g = var.local[e];
        if (w != nullptr) {
          const float wv = w[e];
          g = l2_grad(g, p.l2_scale, wv);
          reg = fmaf(wv, wv, reg);
        }
        if (norms) acc = fmaf(g, g, acc);
      }
      clip_block_sum(reg, s_warp, [&](float b) { p.l2_partials[blockIdx.x * kGradClipMaxVars + v] = b; });
    } else {
      for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kClipThreads + threadIdx.x; i < n;
           i += static_cast<uint64_t>(gridDim.x) * kClipThreads) {
        const float g = var.local[(i / var.cols) * var.ld + i % var.cols];
        acc = fmaf(g, g, acc);
      }
    }
    clip_block_sum(acc, s_warp, [&](float b) { p.partials[blockIdx.x * kGradClipMaxVars + v] = b; });
  }
}

template <bool kL2>
__global__ void __launch_bounds__(kClipThreads) grad_clip_apply_kernel(const __grid_constant__ GradClipParams p) {
  __shared__ float s_fac[kGradClipMaxVars];
  const uint32_t seq = *reinterpret_cast<const volatile uint32_t*>(p.seq_ptr);
  const uint64_t slot = seq % p.nslots;
  if constexpr (kL2) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      float r = 0.f;
      for (int v = 0; v < p.n_vars; ++v)
        for (int b = 0; b < kClipBlocks; ++b) r += p.l2_partials[b * kGradClipMaxVars + v];
      p.result->loss = __fadd_rn(p.result->loss, __fmul_rn(p.l2_scale, __fmul_rn(0.5f, r)));
    }
  }
  if (kL2 ? (p.kind == CLIP_GLOBAL_NORM || p.kind == CLIP_NORM) : p.kind != CLIP_VALUE) {
    __shared__ float s_tot[kGradClipMaxVars];
    if (threadIdx.x < static_cast<unsigned>(p.n_vars)) {
      float t = 0.f;
      for (int b = 0; b < kClipBlocks; ++b) t += p.partials[b * kGradClipMaxVars + threadIdx.x];
      s_tot[threadIdx.x] = t;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      if (p.kind == CLIP_GLOBAL_NORM) {
        float t = 0.f;
        for (int v = 0; v < p.n_vars; ++v) t += s_tot[v];
        const float sc = clip_global_scale(t, p.clip_norm);
        for (int v = 0; v < p.n_vars; ++v) s_fac[v] = sc;
      } else {
        for (int v = 0; v < p.n_vars; ++v) s_fac[v] = clip_norm_divisor(s_tot[v], p.clip_norm);
      }
    }
    __syncthreads();
  }
  for (int v = 0; v < p.n_vars; ++v) {
    const GradClipVar& var = p.var[v];
    const float f = (kL2 ? (p.kind == CLIP_GLOBAL_NORM || p.kind == CLIP_NORM) : p.kind != CLIP_VALUE) ? s_fac[v] : 1.f;
    float* mb = var.mailbox + slot * var.mailbox_slot_stride;
    const uint64_t n = static_cast<uint64_t>(var.rows) * var.cols;
    if constexpr (kL2) {
      const float* w = p.l2_w[v];
      for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kClipThreads + threadIdx.x; i < n;
           i += static_cast<uint64_t>(gridDim.x) * kClipThreads) {
        const uint64_t e = (i / var.cols) * var.ld + i % var.cols;
        float g = var.local[e];
        if (w != nullptr) g = l2_grad(g, p.l2_scale, w[e]);
        mb[e] = p.kind == CLIP_OFF ? g : clip_element(p.kind, g, f, p.clip_norm, p.clip_min, p.clip_max);
        var.local[e] = 0.f;
      }
    } else {
      for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kClipThreads + threadIdx.x; i < n;
           i += static_cast<uint64_t>(gridDim.x) * kClipThreads) {
        const uint64_t e = (i / var.cols) * var.ld + i % var.cols;
        mb[e] = clip_element(p.kind, var.local[e], f, p.clip_norm, p.clip_min, p.clip_max);
        var.local[e] = 0.f;
      }
    }
  }
}

__global__ void __launch_bounds__(kClipThreads) grad_clip_release_kernel(const __grid_constant__ GradClipParams p) {
  const uint32_t seq = *reinterpret_cast<const volatile uint32_t*>(p.seq_ptr);
  const uint64_t slot = seq % p.nslots;
  fence_acq_rel_scoped(p.gpu_scope);   // every mailbox store of the apply kernel (completed before this grid started)
  for (int k = 0; k < p.n_shards; ++k) {
    uint32_t* f = p.flags[k] + slot * p.flag_slot_stride[k];
    for (uint32_t i = threadIdx.x; i < p.n_flags[k]; i += kClipThreads) st_relaxed_sys_u32(f + i, seq);
  }
}

using GradClipKernel = void (*)(const GradClipParams);

// The kernel of clip stage `stage` (0 sums of squares, 1 clip into the mailbox, 2 flags), with or without the L2 term;
// null for an unknown stage.
static GradClipKernel grad_clip_kernel(int stage, bool l2) {
  if (stage == 0 || stage == 1) {
    if (!l2) return stage == 0 ? grad_clip_ssq_kernel<false> : grad_clip_apply_kernel<false>;
    return stage == 0 ? grad_clip_ssq_kernel<true> : grad_clip_apply_kernel<true>;
  }
  return stage == 2 ? grad_clip_release_kernel : nullptr;
}

cudaError_t prepare_grad_clip_kernels() {
  cudaFuncAttributes a;
  for (const bool l2 : {false, true})
    for (const int stage : {0, 1})
      if (cudaError_t e = cudaFuncGetAttributes(&a, grad_clip_kernel(stage, l2)); e != cudaSuccess) return e;
  return cudaFuncGetAttributes(&a, grad_clip_kernel(2, false));
}

cudaError_t launch_grad_clip(const GradClipParams& p, int stage, cudaStream_t stream) {
  const bool l2 = p.l2_scale != 0.f;
  if (p.n_vars < 1 || p.n_vars > kGradClipMaxVars || p.n_shards < 0 || p.n_shards > kGradClipMaxShards ||
      p.nslots < 1 || p.kind < (l2 ? CLIP_OFF : CLIP_GLOBAL_NORM) || p.kind > CLIP_VALUE ||
      !(p.l2_scale >= 0.f && p.l2_scale < INFINITY) || (l2 && (p.l2_partials == nullptr || p.result == nullptr)))
    return cudaErrorInvalidValue;
  const GradClipKernel k = grad_clip_kernel(stage, l2);
  if (k == nullptr) return cudaErrorInvalidValue;
  k<<<stage == 2 ? 1 : kClipBlocks, kClipThreads, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace dm
