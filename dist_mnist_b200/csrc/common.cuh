// Shared device-side primitives for the sm_90a kernels: mbarrier, TMA, wgmma,
// system-scope flag loads/stores for the NVLink peer-memory protocol.
//
// Everything here is raw PTX for sm_90a (compile with -gencode arch=compute_90a,code=sm_90a).
// No CUTLASS/CuTe dependency: the descriptor encoding below follows the PTX ISA table of the
// wgmma shared-memory matrix descriptor.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

namespace dm {

// ------------------------------------------------------------------------------------------
// misc
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ uint32_t sm_id() {
  uint32_t s;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
  return s;
}

// Spin-wait guard: a kernel that waits longer than this traps instead of hanging the GPU
// (a trap is a failed call the host can report; a hang is not).
#ifndef DM_SPIN_TIMEOUT_NS
#define DM_SPIN_TIMEOUT_NS (4000000000ull)
#endif

// SM count of the current device: grid-stride kernels cap their grid at a few CTAs per SM (132 on an H100 SXM, the
// fallback if the query fails).
inline int device_sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      n <= 0)
    return 132;
  return n;
}

// One entry per translation unit: opt its kernels into their dynamic shared memory where they need it and force-load
// every kernel its launchers can pick, so that no first launch needs a lazy load while a persistent serve kernel is
// resident (DESIGN §7). dm_prepare_kernels calls each once per device.
cudaError_t prepare_gemm_kernels();
cudaError_t prepare_head_kernels();
cudaError_t prepare_grad_clip_kernels();
cudaError_t prepare_ps_kernels();
cudaError_t prepare_p2p_kernels();
cudaError_t prepare_fused_kernels();
cudaError_t prepare_nvls_kernels();

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  while (!mbar_try_wait(bar, parity)) {
    if (globaltimer_ns() - t0 > DM_SPIN_TIMEOUT_NS) {
      printf("[dm] mbarrier wait timeout block=(%d,%d,%d) thread=%d parity=%u\n", blockIdx.x, blockIdx.y,
             blockIdx.z, threadIdx.x, parity);
      __trap();
    }
  }
}

// ------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) — global (local HBM *or* NVLink peer-mapped HBM) -> shared
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* t) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(t)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// 1-D bulk copy global -> shared (no tensor map): used for contiguous parameter slabs.
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
// Restricted to shared memory: orders this thread's shared-memory writes (own CTA / whole cluster) against later
// async-proxy accesses without waiting for its outstanding *global* (possibly NVLink peer) stores.
__device__ __forceinline__ void fence_proxy_async_smem_cta() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem_cluster() {
  asm volatile("fence.proxy.async.shared::cluster;" ::: "memory");
}
// TMA store (shared -> global, possibly NVLink peer memory): 3-D tile {c0, c1, c2} of the tensor map, bulk-group
// completion. The reduce variant adds (fp32) instead of overwriting: push == apply for asynchronous SGD.
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tmap, const void* smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tmap)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap* tmap, const void* smem_src, int c0, int c1, int c2) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tmap)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_group0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// only the *source* (shared memory) of every committed bulk group has been read: the staging tile may be reused
__device__ __forceinline__ void bulk_wait_group_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

// ------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, sm_90a): D[64 x N] (fp32, registers of the 128 threads of one aligned warpgroup)
//   += A[64 x K] * B[N x K]^T, B from a shared-memory matrix descriptor (K-major), A from registers.
// ------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, SWIZZLE_128B, K-major (sm_90 layout):
//   bits [0,14) start address >> 4   [16,30) leading byte offset >> 4 (unused for swizzled K-major)
//   bits [32,46) stride byte offset >> 4 (8 rows x 128 B = 1024)   [62,64) layout type (1 = SWIZZLE_128B)
// The tile base is 1024-byte aligned; a k-step inside the 128-byte swizzle atom advances the start address by
// its byte offset (32 B per k8 tf32 / k16 bf16 step).
__device__ __forceinline__ uint64_t make_wgmma_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr >> 4) & 0x3FFFu);
  d |= static_cast<uint64_t>(1u) << 16;
  d |= static_cast<uint64_t>(1024u >> 4) << 32;
  d |= static_cast<uint64_t>(1u) << 62;
  return d;
}
// Byte offset of element `c` (element size `es`) of row `r` in a 128-byte-swizzled tile (TMA SWIZZLE_128B,
// 1024-byte aligned base): the 16-byte chunk j of row r sits at chunk position j ^ (r & 7).
__device__ __forceinline__ uint32_t sw128_offset(uint32_t r, uint32_t c, uint32_t es) {
  const uint32_t b = c * es;
  return r * 128u + ((((b >> 4) ^ (r & 7u)) << 4) | (b & 15u));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keep the accumulator registers of an asynchronous wgmma live across the fence / wait
__device__ __forceinline__ void wgmma_reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }

template <typename T>
struct Wgmma;
template <>
struct Wgmma<float> {  // fp32 storage consumed as tf32: k = 8 per instruction
  static constexpr int kK = 8;
  // A fragment (m64 x k8, per warp 16 rows): a0 (r, c), a1 (r + 8, c), a2 (r, c + 4), a3 (r + 8, c + 4)
  // with r = 16 * warp + lane / 4, c = lane % 4
  __device__ static __forceinline__ void mma(float (&d)[8], const uint32_t (&a)[4], uint64_t bdesc, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc));
  }
};
template <>
struct Wgmma<__nv_bfloat16> {  // k = 16 per instruction
  static constexpr int kK = 16;
  // A fragment: pairs of consecutive k; a0 (r, 2c..2c+1), a1 (r + 8, 2c..), a2 (r, 2c + 8..), a3 (r + 8, 2c + 8..)
  __device__ static __forceinline__ void mma(float (&d)[8], const uint32_t (&a)[4], uint64_t bdesc, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc));
  }
};

// ------------------------------------------------------------------------------------------
// system-scope flags (NVLink peer-memory protocol)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_acq_rel_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
__device__ __forceinline__ void st_relaxed_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// Scope-selectable variants: when every party of a flag protocol runs on the *same* GPU (ps and worker sharing
// a device), gpu scope is sufficient and several times cheaper than the system-scope fence NVLink peers need.
__device__ __forceinline__ void st_release_scoped_u32(uint32_t* p, uint32_t v, uint32_t gpu_scope) {
  if (gpu_scope) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
  else st_release_sys_u32(p, v);
}
__device__ __forceinline__ uint32_t ld_acquire_scoped_u32(const uint32_t* p, uint32_t gpu_scope) {
  uint32_t v;
  if (gpu_scope) asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  else v = ld_acquire_sys_u32(p);
  return v;
}
__device__ __forceinline__ void fence_acq_rel_scoped(uint32_t gpu_scope) {
  if (gpu_scope) asm volatile("fence.acq_rel.gpu;" ::: "memory");
  else fence_acq_rel_sys();
}
__device__ __forceinline__ uint32_t ld_relaxed_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t atom_add_sys_u32(uint32_t* p, uint32_t v) {
  uint32_t old;
  asm volatile("atom.add.relaxed.sys.global.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}
// Monotone publication of a counter into (possibly peer) memory: several CTAs may acknowledge consecutive
// pushes of one worker at almost the same time, and a plain store of the older value landing last would move
// the acknowledged sequence number backwards. `release` orders the publisher's earlier writes before it.
__device__ __forceinline__ void red_max_release_scoped_u32(uint32_t* p, uint32_t v, uint32_t gpu_scope) {
  if (gpu_scope) asm volatile("red.release.gpu.global.max.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
  else asm volatile("red.release.sys.global.max.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_max_relaxed_scoped_u32(uint32_t* p, uint32_t v, uint32_t gpu_scope) {
  if (gpu_scope) asm volatile("red.relaxed.gpu.global.max.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
  else asm volatile("red.relaxed.sys.global.max.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Fire-and-forget fp32 reduction into (possibly peer) global memory: the SGD "push == apply" path.
__device__ __forceinline__ void red_add_sys_f32(float* p, float v) {
  asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ void red_add_sys_v4f32(float* p, float a, float b, float c, float d) {
  asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c),
               "f"(d)
               : "memory");
}
__device__ __forceinline__ void st_global_v4f32(float* p, float a, float b, float c, float d) {
  asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// ------------------------------------------------------------------------------------------
// thread-block clusters / distributed shared memory
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// shared::cta address of this CTA -> shared::cluster address of the same offset in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_shared_cluster(uint32_t cta_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(cta_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_shared_cluster_f32(uint32_t cluster_addr, float v) {
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(cluster_addr), "f"(v) : "memory");
}
__device__ __forceinline__ void st_shared_cluster_v4f32(uint32_t cluster_addr, float a, float b, float c, float d) {
  asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(cluster_addr), "f"(a), "f"(b), "f"(c), "f"(d)
               : "memory");
}
__device__ __forceinline__ void st_shared_cluster_v2f32(uint32_t cluster_addr, float a, float b) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(cluster_addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void st_shared_cluster_u32(uint32_t cluster_addr, uint32_t v) {
  asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(cluster_addr), "r"(v) : "memory");
}
__device__ __forceinline__ void cluster_barrier_arrive_release() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_barrier_wait_acquire() {
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Named barrier among a subset of warps (id 1..15; 0 is __syncthreads).
// Programmatic dependent launch (PDL): a kernel launched with the programmatic-stream-serialization attribute
// may start while its predecessor in the stream is still running; `grid_dep_wait` blocks until the predecessor
// grid has completed and its memory is visible, `grid_dep_launch` lets the successor start being scheduled.
// Both are no-ops for kernels launched without the attribute.
__device__ __forceinline__ void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void grid_dep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// Non-blocking arrival at a named barrier that other warps bar.sync on (producer side of a hand-off).
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

}  // namespace dm
