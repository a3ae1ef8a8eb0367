// NVLink peer-memory microbenchmark / utility kernels (BASELINE.json config 5: PS push/pull bandwidth
// sweep 1 KB - 1 GB; SURVEY X3/X4 transports in isolation).
//
//   p2p_copy (mode 0)  : vectorised ld.global.v4 / st.global.v4 copy; either side may be a peer pointer
//                        (push = remote dst, pull = remote src).
//   p2p_copy (mode 1)  : TMA bulk copy  global -> smem -> global  (cp.async.bulk), 4 x 16 KB ring per CTA.
//   p2p_reduce_apply   : many-to-one pull-reduce fused with SGD apply: params -= lr * sum_s grads[s]
//                        where grads[s] are peer pointers into the workers' HBM.
//   pingpong           : flag round-trip latency between two GPUs (st.release.sys / ld.acquire.sys).
#include "common.cuh"

namespace dm {

__global__ void __launch_bounds__(512) p2p_copy_ldst_kernel(int4* __restrict__ dst, const int4* __restrict__ src,
                                                            size_t n16, uint32_t* flag) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  // 4 independent 16-byte loads in flight per thread
  for (; i + 3 * stride < n16; i += 4 * stride) {
    int4 v0 = __ldcg(src + i);
    int4 v1 = __ldcg(src + i + stride);
    int4 v2 = __ldcg(src + i + 2 * stride);
    int4 v3 = __ldcg(src + i + 3 * stride);
    dst[i] = v0;
    dst[i + stride] = v1;
    dst[i + 2 * stride] = v2;
    dst[i + 3 * stride] = v3;
  }
  for (; i < n16; i += stride) dst[i] = __ldcg(src + i);
  if (flag != nullptr) {
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) atom_add_sys_u32(flag, 1u);  // arrival counter: receiver waits for gridDim.x arrivals
  }
}

constexpr int kBulkChunk = 16384;
constexpr int kBulkRing = 4;

__global__ void __launch_bounds__(32) p2p_copy_tma_kernel(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src,
                                                          size_t bytes, uint32_t* flag) {
  extern __shared__ __align__(128) uint8_t ring[];
  __shared__ uint64_t bar[kBulkRing];
  if (threadIdx.x == 0) {
    for (int i = 0; i < kBulkRing; ++i) mbar_init(&bar[i], 1);
    fence_mbar_init();
    const size_t nchunks = (bytes + kBulkChunk - 1) / kBulkChunk;
    // chunks are dealt round-robin to CTAs
    auto chunk_of = [&](size_t k) { return blockIdx.x + k * gridDim.x; };
    size_t mine = 0;
    for (size_t c = blockIdx.x; c < nchunks; c += gridDim.x) ++mine;
    auto issue_load = [&](size_t k) {
      const int s = k % kBulkRing;
      const size_t off = chunk_of(k) * kBulkChunk;
      const uint32_t n = static_cast<uint32_t>(min(static_cast<size_t>(kBulkChunk), bytes - off));
      mbar_arrive_expect_tx(&bar[s], n);
      bulk_load_1d(ring + s * kBulkChunk, src + off, n, &bar[s]);
    };
    for (size_t k = 0; k < mine && k < kBulkRing; ++k) issue_load(k);
    for (size_t k = 0; k < mine; ++k) {
      const int s = k % kBulkRing;
      mbar_wait(&bar[s], (k / kBulkRing) & 1);
      const size_t off = chunk_of(k) * kBulkChunk;
      const uint32_t n = static_cast<uint32_t>(min(static_cast<size_t>(kBulkChunk), bytes - off));
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst + off),
                   "r"(smem_u32(ring + s * kBulkChunk)), "r"(n)
                   : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      if (k + kBulkRing < mine) {
        // the store must have finished reading this buffer before the next load lands in it;
        // the other ring slots' loads stay in flight meanwhile.
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        issue_load(k + kBulkRing);
      }
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    if (flag != nullptr) {
      __threadfence_system();
      atom_add_sys_u32(flag, 1u);
    }
  }
}

cudaError_t launch_p2p_copy(void* dst, const void* src, size_t bytes, int mode, int ctas, uint32_t* flag,
                            uint32_t /*flag_value*/, cudaStream_t stream) {
  if (ctas < 1) ctas = 1;
  if (mode == 0) {
    if (bytes % 16 != 0) return cudaErrorInvalidValue;
    p2p_copy_ldst_kernel<<<ctas, 512, 0, stream>>>(static_cast<int4*>(dst), static_cast<const int4*>(src), bytes / 16,
                                                   flag);
  } else {
    if (bytes % 16 != 0) return cudaErrorInvalidValue;
    const int smem = kBulkChunk * kBulkRing;
    cudaError_t e = cudaFuncSetAttribute(p2p_copy_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    p2p_copy_tma_kernel<<<ctas, 32, smem, stream>>>(static_cast<uint8_t*>(dst), static_cast<const uint8_t*>(src), bytes,
                                                    flag);
  }
  return cudaGetLastError();
}

__global__ void __launch_bounds__(512) p2p_reduce_apply_kernel(float4* __restrict__ params,
                                                               const float* const* __restrict__ grads, int n_src,
                                                               size_t n4, float lr) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4; i += stride) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < n_src; ++s) {
      const float4 g = __ldcg(reinterpret_cast<const float4*>(grads[s]) + i);
      acc.x += g.x; acc.y += g.y; acc.z += g.z; acc.w += g.w;
    }
    float4 p = params[i];
    p.x = fmaf(-lr, acc.x, p.x); p.y = fmaf(-lr, acc.y, p.y);
    p.z = fmaf(-lr, acc.z, p.z); p.w = fmaf(-lr, acc.w, p.w);
    params[i] = p;
  }
}

cudaError_t launch_p2p_reduce_apply(float* params, const float* const* grads, int n_src, size_t n, float lr, int ctas,
                                    cudaStream_t stream) {
  if (n % 4 != 0) return cudaErrorInvalidValue;
  if (ctas < 1) ctas = 1;
  p2p_reduce_apply_kernel<<<ctas, 512, 0, stream>>>(reinterpret_cast<float4*>(params), grads, n_src, n / 4, lr);
  return cudaGetLastError();
}

__global__ void pingpong_kernel(uint32_t* local_flag, uint32_t* remote_flag, int iters, int role, uint64_t* out_ns) {
  const uint64_t t0 = globaltimer_ns();
  for (int i = 1; i <= iters; ++i) {
    if (role == 0) st_release_sys_u32(remote_flag, static_cast<uint32_t>(i));
    const uint64_t w0 = globaltimer_ns();
    while (ld_acquire_sys_u32(local_flag) != static_cast<uint32_t>(i)) {
      if (globaltimer_ns() - w0 > DM_SPIN_TIMEOUT_NS) { printf("[dm] pingpong timeout i=%d\n", i); __trap(); }
    }
    if (role == 1) st_release_sys_u32(remote_flag, static_cast<uint32_t>(i));
  }
  out_ns[0] = globaltimer_ns() - t0;
}

cudaError_t launch_pingpong(uint32_t* local_flag, uint32_t* remote_flag, int iters, int role, uint64_t* out_ns,
                            cudaStream_t stream) {
  pingpong_kernel<<<1, 1, 0, stream>>>(local_flag, remote_flag, iters, role, out_ns);
  return cudaGetLastError();
}

}  // namespace dm

namespace dm {
cudaError_t prepare_p2p_kernels() {
  cudaFuncAttributes a;
  cudaError_t e;
  if ((e = cudaFuncGetAttributes(&a, p2p_copy_ldst_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, p2p_copy_tma_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, p2p_reduce_apply_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, pingpong_kernel)) != cudaSuccess) return e;
  return cudaSuccess;
}
}  // namespace dm
