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
#include "common.cuh"
#include "grad_clip.cuh"

namespace dm {

constexpr int kClipThreads = 256;
constexpr int kClipBlocks = 132;

__global__ void __launch_bounds__(kClipThreads) grad_clip_ssq_kernel(const __grid_constant__ GradClipParams p) {
  __shared__ float s_warp[kClipThreads / 32];
  for (int v = 0; v < p.n_vars; ++v) {
    const GradClipVar& var = p.var[v];
    const uint64_t n = static_cast<uint64_t>(var.rows) * var.cols;
    float acc = 0.f;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kClipThreads + threadIdx.x; i < n;
         i += static_cast<uint64_t>(gridDim.x) * kClipThreads) {
      const float g = var.local[(i / var.cols) * var.ld + i % var.cols];
      acc = fmaf(g, g, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float b = 0.f;
#pragma unroll
      for (int w = 0; w < kClipThreads / 32; ++w) b += s_warp[w];
      p.partials[blockIdx.x * kGradClipMaxVars + v] = b;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kClipThreads) grad_clip_apply_kernel(const __grid_constant__ GradClipParams p) {
  __shared__ float s_fac[kGradClipMaxVars];
  const uint32_t seq = *reinterpret_cast<const volatile uint32_t*>(p.seq_ptr);
  const uint64_t slot = seq % p.nslots;
  if (p.kind != CLIP_VALUE) {
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
    const float f = p.kind != CLIP_VALUE ? s_fac[v] : 1.f;
    float* mb = var.mailbox + slot * var.mailbox_slot_stride;
    const uint64_t n = static_cast<uint64_t>(var.rows) * var.cols;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kClipThreads + threadIdx.x; i < n;
         i += static_cast<uint64_t>(gridDim.x) * kClipThreads) {
      const uint64_t e = (i / var.cols) * var.ld + i % var.cols;
      mb[e] = clip_element(p.kind, var.local[e], f, p.clip_norm, p.clip_min, p.clip_max);
      var.local[e] = 0.f;
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

cudaError_t preload_grad_clip_kernels() {
  cudaFuncAttributes a;
  cudaError_t e = cudaFuncGetAttributes(&a, grad_clip_ssq_kernel);   // force-load (see preload_ps_kernels)
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&a, grad_clip_apply_kernel);
  return e != cudaSuccess ? e : cudaFuncGetAttributes(&a, grad_clip_release_kernel);
}

cudaError_t launch_grad_clip(const GradClipParams& p, int stage, cudaStream_t stream) {
  if (p.n_vars < 1 || p.n_vars > kGradClipMaxVars || p.n_shards < 0 || p.n_shards > kGradClipMaxShards ||
      p.nslots < 1 || p.kind < CLIP_GLOBAL_NORM || p.kind > CLIP_VALUE)
    return cudaErrorInvalidValue;
  if (stage == 0) {
    grad_clip_ssq_kernel<<<kClipBlocks, kClipThreads, 0, stream>>>(p);
  } else if (stage == 1) {
    grad_clip_apply_kernel<<<kClipBlocks, kClipThreads, 0, stream>>>(p);
  } else if (stage == 2) {
    grad_clip_release_kernel<<<1, kClipThreads, 0, stream>>>(p);
  } else {
    return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace dm
