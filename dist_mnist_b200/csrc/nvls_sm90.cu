// NVLS multicast parameter publish — measured prototype (SURVEY X3 variant (a); not yet wired into the ps shard).
//
// The reference re-sends every variable to every worker on every step (each `sess.run` fetches the variables of
// /root/reference/distributed_server-basic.py:41-47 from the ps over gRPC, DS:112). With NVSwitch multicast ("NVLS")
// the ps can instead *publish* an updated parameter tile once: one `multimem.st` to a multicast address is replicated
// by the switch into the bound memory of every GPU of the team, so the workers' TMA pulls become local reads and the
// ps egress carries one copy instead of one per worker.
//
// This file holds the two kernels of that path and a self-contained probe (`dm_nvls_probe`) that builds a multicast
// team over the visible GPUs *of one process* (cuMulticastCreate / AddDevice / BindMem + VMM mappings), publishes a
// buffer from GPU 0 with `multimem.st`, verifies every replica bit for bit and times the publish against per-replica
// unicast peer stores. The driver entry points are fetched with cudaGetDriverEntryPoint (the library does not link
// libcuda). Engine integration (a multicast team across the ps / worker *processes*: fd passing of the multicast and
// allocation handles, `multimem.st` in `apply_item`'s store phase, workers' tensor maps on their local replica) is
// described in DESIGN.md section 8.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

namespace dm {

// dst is a *multicast* address: every 16-byte store lands in the replica of every GPU of the team.
__global__ void multimem_publish_kernel(const float4* __restrict__ src, float4* mc_dst, size_t n4) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 v = src[i];
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_dst + i), "f"(v.x), "f"(v.y),
                 "f"(v.z), "f"(v.w)
                 : "memory");
  }
  __threadfence_system();
}

// The same publish with plain peer stores: one store per replica (what a ps without multicast has to do).
__global__ void unicast_publish_kernel(const float4* __restrict__ src, float4* const* __restrict__ dsts, int n_dst,
                                       size_t n4) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 v = src[i];
    for (int d = 0; d < n_dst; ++d) dsts[d][i] = v;
  }
  __threadfence_system();
}

// In-switch reduction: one `multimem.ld_reduce` returns the SUM over the replicas of every GPU of the team — the
// gradient aggregation of a merged / synchronous apply (`--apply_mode merged`; the reference itself only has the
// asynchronous per-push apply, /root/reference/distributed_server-basic.py:102-103) done by the NVSwitch instead of
// the ps: the ps reads each aggregated gradient element once instead of once per worker.
__global__ void multimem_reduce_kernel(const float4* mc_src, float4* __restrict__ out, size_t n4) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(mc_src + i)
                 : "memory");
    out[i] = v;
  }
}

// The same aggregation with peer loads: one load per replica.
__global__ void unicast_reduce_kernel(float4* const* __restrict__ srcs, int n_src, float4* __restrict__ out, size_t n4) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int d = 0; d < n_src; ++d) {
      const float4 v = __ldcv(srcs[d] + i);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    out[i] = acc;
  }
}

cudaError_t prepare_nvls_kernels() {
  cudaFuncAttributes a;
  cudaError_t e;
  if ((e = cudaFuncGetAttributes(&a, multimem_publish_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, multimem_reduce_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, unicast_reduce_kernel)) != cudaSuccess) return e;
  return cudaFuncGetAttributes(&a, unicast_publish_kernel);
}

}  // namespace dm

namespace {

struct Log {
  std::string s;
  void add(const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    s += buf;
    s += "\n";
  }
};

template <typename F>
bool load_entry(const char* name, F& fn, Log& log) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || p == nullptr) {
    log.add("FAIL: cudaGetDriverEntryPoint(%s): %s (query result %d)", name, cudaGetErrorName(e), static_cast<int>(q));
    cudaGetLastError();
    return false;
  }
  fn = reinterpret_cast<F>(p);
  return true;
}

#define CU_TRY(call)                                                              \
  do {                                                                            \
    CUresult r__ = (call);                                                        \
    if (r__ != CUDA_SUCCESS) {                                                    \
      log.add("FAIL: %s -> CUresult %d", #call, static_cast<int>(r__));         \
      return finish(false);                                                       \
    }                                                                             \
  } while (0)
#define RT_TRY(call)                                                              \
  do {                                                                            \
    cudaError_t e__ = (call);                                                     \
    if (e__ != cudaSuccess) {                                                     \
      log.add("FAIL: %s -> %s", #call, cudaGetErrorName(e__));                  \
      return finish(false);                                                       \
    }                                                                             \
  } while (0)

}  // namespace

extern "C" {

// Probe: multicast team over devices 0..n_dev-1 of this process; GPU 0 publishes `bytes` (rounded up to the multicast
// granularity) `iters` times. Writes a human-readable log (one finding per line, "RESULT key=value" lines for the
// numbers) into out_log. Returns 0 when multicast publishing worked and every replica verified, 1 otherwise.
int dm_nvls_probe(int n_dev, size_t bytes, int iters, char* out_log, size_t log_cap) {
  Log log;
  auto finish = [&](bool ok) -> int {
    log.add(ok ? "PROBE OK" : "PROBE FAILED");
    if (out_log != nullptr && log_cap > 0) {
      strncpy(out_log, log.s.c_str(), log_cap - 1);
      out_log[log_cap - 1] = 0;
    }
    return ok ? 0 : 1;
  };
  int visible = 0;
  RT_TRY(cudaGetDeviceCount(&visible));
  if (n_dev < 2 || n_dev > visible || n_dev > 8) {
    log.add("FAIL: need 2..8 devices in this process (asked %d, visible %d)", n_dev, visible);
    return finish(false);
  }
  decltype(&cuDeviceGet) pDeviceGet = nullptr;
  decltype(&cuDeviceGetAttribute) pDeviceGetAttribute = nullptr;
  decltype(&cuMulticastCreate) pMulticastCreate = nullptr;
  decltype(&cuMulticastAddDevice) pMulticastAddDevice = nullptr;
  decltype(&cuMulticastBindMem) pMulticastBindMem = nullptr;
  decltype(&cuMulticastGetGranularity) pMulticastGetGranularity = nullptr;
  decltype(&cuMemCreate) pMemCreate = nullptr;
  decltype(&cuMemGetAllocationGranularity) pMemGetAllocationGranularity = nullptr;
  decltype(&cuMemAddressReserve) pMemAddressReserve = nullptr;
  decltype(&cuMemMap) pMemMap = nullptr;
  decltype(&cuMemSetAccess) pMemSetAccess = nullptr;
  if (!load_entry("cuDeviceGet", pDeviceGet, log) || !load_entry("cuDeviceGetAttribute", pDeviceGetAttribute, log) ||
      !load_entry("cuMulticastCreate", pMulticastCreate, log) ||
      !load_entry("cuMulticastAddDevice", pMulticastAddDevice, log) ||
      !load_entry("cuMulticastBindMem", pMulticastBindMem, log) ||
      !load_entry("cuMulticastGetGranularity", pMulticastGetGranularity, log) ||
      !load_entry("cuMemCreate", pMemCreate, log) ||
      !load_entry("cuMemGetAllocationGranularity", pMemGetAllocationGranularity, log) ||
      !load_entry("cuMemAddressReserve", pMemAddressReserve, log) || !load_entry("cuMemMap", pMemMap, log) ||
      !load_entry("cuMemSetAccess", pMemSetAccess, log))
    return finish(false);

  std::vector<CUdevice> dev(n_dev);
  for (int d = 0; d < n_dev; ++d) {
    RT_TRY(cudaSetDevice(d));
    RT_TRY(cudaFree(nullptr));   // make sure the primary context exists
    CU_TRY(pDeviceGet(&dev[d], d));
    int mc = 0;
    CU_TRY(pDeviceGetAttribute(&mc, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev[d]));
    log.add("device %d: CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED = %d", d, mc);
    if (!mc) return finish(false);
  }
  for (int a = 0; a < n_dev; ++a) {   // peer access both ways (unicast comparison + fabric reachability)
    RT_TRY(cudaSetDevice(a));
    for (int b = 0; b < n_dev; ++b) {
      if (a == b) continue;
      cudaError_t e = cudaDeviceEnablePeerAccess(b, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
        log.add("FAIL: cudaDeviceEnablePeerAccess(%d -> %d): %s", a, b, cudaGetErrorName(e));
        return finish(false);
      }
      cudaGetLastError();
    }
  }
  RT_TRY(cudaSetDevice(0));

  // ---- multicast object ----
  CUmulticastObjectProp mp;
  memset(&mp, 0, sizeof(mp));
  mp.numDevices = static_cast<unsigned int>(n_dev);
  mp.size = bytes;
  mp.handleTypes = 0;
  mp.flags = 0;
  size_t gran_min = 0, gran = 0;
  CU_TRY(pMulticastGetGranularity(&gran_min, &mp, CU_MULTICAST_GRANULARITY_MINIMUM));
  CU_TRY(pMulticastGetGranularity(&gran, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED));
  log.add("multicast granularity: minimum %zu B, recommended %zu B", gran_min, gran);
  if (gran == 0) gran = gran_min ? gran_min : (2u << 20);
  const size_t size = (bytes + gran - 1) / gran * gran;
  mp.size = size;
  CUmemGenericAllocationHandle mc = 0;
  CU_TRY(pMulticastCreate(&mc, &mp));
  for (int d = 0; d < n_dev; ++d) CU_TRY(pMulticastAddDevice(mc, dev[d]));
  log.add("multicast object created: %d devices, %zu bytes per replica", n_dev, size);

  // ---- one physical replica per device, bound to the object and mapped for unicast access ----
  std::vector<CUmemGenericAllocationHandle> h(n_dev);
  std::vector<CUdeviceptr> va(n_dev);
  for (int d = 0; d < n_dev; ++d) {
    CUmemAllocationProp ap;
    memset(&ap, 0, sizeof(ap));
    ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ap.location.id = d;
    ap.requestedHandleTypes = CU_MEM_HANDLE_TYPE_NONE;
    size_t ag = 0;
    CU_TRY(pMemGetAllocationGranularity(&ag, &ap, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    if (size % ag != 0) {
      log.add("FAIL: replica size %zu is not a multiple of the allocation granularity %zu of device %d", size, ag, d);
      return finish(false);
    }
    RT_TRY(cudaSetDevice(d));
    CU_TRY(pMemCreate(&h[d], size, &ap, 0));
    CU_TRY(pMulticastBindMem(mc, 0, h[d], 0, size, 0));
    CU_TRY(pMemAddressReserve(&va[d], size, gran, 0, 0));
    CU_TRY(pMemMap(va[d], size, 0, h[d], 0));
    CUmemAccessDesc ad[2];
    memset(ad, 0, sizeof(ad));
    ad[0].location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ad[0].location.id = d;
    ad[0].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    ad[1].location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ad[1].location.id = 0;       // GPU 0 (the publisher) may also store into every replica directly: unicast baseline
    ad[1].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    CU_TRY(pMemSetAccess(va[d], size, ad, d == 0 ? 1 : 2));
  }
  RT_TRY(cudaSetDevice(0));
  CUdeviceptr mcva = 0;
  CU_TRY(pMemAddressReserve(&mcva, size, gran, 0, 0));
  CU_TRY(pMemMap(mcva, size, 0, mc, 0));
  {
    CUmemAccessDesc ad;
    memset(&ad, 0, sizeof(ad));
    ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ad.location.id = 0;
    ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    CU_TRY(pMemSetAccess(mcva, size, &ad, 1));
  }
  log.add("replicas bound and mapped; multicast address mapped on GPU 0");

  // ---- publish from GPU 0 ----
  const size_t n4 = bytes / 16;
  std::vector<float> host(n4 * 4);
  for (size_t i = 0; i < host.size(); ++i) host[i] = static_cast<float>((i * 2654435761u) % 100003);  // exact integers
  float4* src = nullptr;
  RT_TRY(cudaMalloc(reinterpret_cast<void**>(&src), n4 * 16));
  RT_TRY(cudaMemcpy(src, host.data(), n4 * 16, cudaMemcpyHostToDevice));
  for (int d = 0; d < n_dev; ++d) {
    RT_TRY(cudaSetDevice(d));
    RT_TRY(cudaMemset(reinterpret_cast<void*>(va[d]), 0, size));
    RT_TRY(cudaDeviceSynchronize());
  }
  RT_TRY(cudaSetDevice(0));
  const int threads = 256;
  int blocks = static_cast<int>((n4 + threads - 1) / threads);
  int sms = 0;
  RT_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  if (blocks > sms * 4) blocks = sms * 4;
  if (blocks < 1) blocks = 1;
  cudaEvent_t t0, t1;
  RT_TRY(cudaEventCreate(&t0));
  RT_TRY(cudaEventCreate(&t1));
  dm::multimem_publish_kernel<<<blocks, threads>>>(src, reinterpret_cast<float4*>(mcva), n4);
  RT_TRY(cudaGetLastError());
  RT_TRY(cudaDeviceSynchronize());
  // verify every replica bit for bit
  std::vector<float> back(n4 * 4);
  for (int d = 0; d < n_dev; ++d) {
    RT_TRY(cudaSetDevice(d));
    RT_TRY(cudaMemcpy(back.data(), reinterpret_cast<void*>(va[d]), n4 * 16, cudaMemcpyDeviceToHost));
    size_t bad = 0;
    for (size_t i = 0; i < back.size(); ++i) bad += memcmp(&back[i], &host[i], 4) != 0;
    log.add("replica on GPU %d after multimem.st publish: %zu of %zu floats differ", d, bad, back.size());
    if (bad != 0) return finish(false);
  }
  RT_TRY(cudaSetDevice(0));
  float ms_mc = 0.f, ms_uc = 0.f;
  RT_TRY(cudaEventRecord(t0));
  for (int i = 0; i < iters; ++i) dm::multimem_publish_kernel<<<blocks, threads>>>(src, reinterpret_cast<float4*>(mcva), n4);
  RT_TRY(cudaEventRecord(t1));
  RT_TRY(cudaEventSynchronize(t1));
  RT_TRY(cudaEventElapsedTime(&ms_mc, t0, t1));
  // unicast baseline: one peer store per remote replica (+ the local copy)
  float4** dsts = nullptr;
  std::vector<float4*> hd(n_dev);
  for (int d = 0; d < n_dev; ++d) hd[d] = reinterpret_cast<float4*>(va[d]);
  RT_TRY(cudaMalloc(reinterpret_cast<void**>(&dsts), sizeof(float4*) * n_dev));
  RT_TRY(cudaMemcpy(dsts, hd.data(), sizeof(float4*) * n_dev, cudaMemcpyHostToDevice));
  dm::unicast_publish_kernel<<<blocks, threads>>>(src, dsts, n_dev, n4);
  RT_TRY(cudaGetLastError());
  RT_TRY(cudaDeviceSynchronize());
  RT_TRY(cudaEventRecord(t0));
  for (int i = 0; i < iters; ++i) dm::unicast_publish_kernel<<<blocks, threads>>>(src, dsts, n_dev, n4);
  RT_TRY(cudaEventRecord(t1));
  RT_TRY(cudaEventSynchronize(t1));
  RT_TRY(cudaEventElapsedTime(&ms_uc, t0, t1));
  const double us_mc = ms_mc * 1e3 / iters, us_uc = ms_uc * 1e3 / iters;
  log.add("RESULT devices=%d bytes=%zu multicast_publish_us=%.2f unicast_publish_us=%.2f", n_dev, n4 * 16, us_mc, us_uc);
  log.add("RESULT multicast: %.1f GB/s leaving GPU 0, %.1f GB/s delivered to %d remote replicas; unicast: %.1f GB/s leaving "
          "GPU 0 for the same delivery", n4 * 16 / us_mc * 1e-3, n4 * 16.0 * (n_dev - 1) / us_mc * 1e-3, n_dev - 1,
          n4 * 16.0 * (n_dev - 1) / us_uc * 1e-3);

  // ---- in-switch reduction: replica d holds host + d; GPU 0 reads the sum with multimem.ld_reduce ----
  {
    std::vector<float> rep(n4 * 4);
    for (int d = 0; d < n_dev; ++d) {
      for (size_t i = 0; i < rep.size(); ++i) rep[i] = host[i] + static_cast<float>(d);
      RT_TRY(cudaSetDevice(d));
      RT_TRY(cudaMemcpy(reinterpret_cast<void*>(va[d]), rep.data(), n4 * 16, cudaMemcpyHostToDevice));
      RT_TRY(cudaDeviceSynchronize());
    }
    RT_TRY(cudaSetDevice(0));
    float4* out = nullptr;
    RT_TRY(cudaMalloc(reinterpret_cast<void**>(&out), n4 * 16));
    RT_TRY(cudaMemset(out, 0, n4 * 16));
    dm::multimem_reduce_kernel<<<blocks, threads>>>(reinterpret_cast<const float4*>(mcva), out, n4);
    cudaError_t le = cudaGetLastError();
    cudaError_t se = cudaDeviceSynchronize();
    if (le != cudaSuccess || se != cudaSuccess) {
      log.add("FAIL: multimem.ld_reduce kernel: launch %s, sync %s", cudaGetErrorName(le), cudaGetErrorName(se));
      return finish(false);
    }
    RT_TRY(cudaMemcpy(back.data(), out, n4 * 16, cudaMemcpyDeviceToHost));
    size_t bad = 0;
    const float tri = static_cast<float>(n_dev * (n_dev - 1) / 2);
    for (size_t i = 0; i < back.size(); ++i) bad += back[i] != host[i] * static_cast<float>(n_dev) + tri;
    log.add("multimem.ld_reduce.add over %d replicas: %zu of %zu floats differ from the exact sum", n_dev, bad, back.size());
    if (bad != 0) return finish(false);
    float ms_mr = 0.f, ms_ur = 0.f;
    RT_TRY(cudaEventRecord(t0));
    for (int i = 0; i < iters; ++i)
      dm::multimem_reduce_kernel<<<blocks, threads>>>(reinterpret_cast<const float4*>(mcva), out, n4);
    RT_TRY(cudaEventRecord(t1));
    RT_TRY(cudaEventSynchronize(t1));
    RT_TRY(cudaEventElapsedTime(&ms_mr, t0, t1));
    dm::unicast_reduce_kernel<<<blocks, threads>>>(dsts, n_dev, out, n4);
    RT_TRY(cudaGetLastError());
    RT_TRY(cudaDeviceSynchronize());
    RT_TRY(cudaMemcpy(back.data(), out, n4 * 16, cudaMemcpyDeviceToHost));
    bad = 0;
    for (size_t i = 0; i < back.size(); ++i) bad += back[i] != host[i] * static_cast<float>(n_dev) + tri;
    if (bad != 0) {
      log.add("FAIL: unicast reduce baseline: %zu floats differ", bad);
      return finish(false);
    }
    RT_TRY(cudaEventRecord(t0));
    for (int i = 0; i < iters; ++i) dm::unicast_reduce_kernel<<<blocks, threads>>>(dsts, n_dev, out, n4);
    RT_TRY(cudaEventRecord(t1));
    RT_TRY(cudaEventSynchronize(t1));
    RT_TRY(cudaEventElapsedTime(&ms_ur, t0, t1));
    const double us_mr = ms_mr * 1e3 / iters, us_ur = ms_ur * 1e3 / iters;
    log.add("RESULT devices=%d bytes=%zu multicast_reduce_us=%.2f unicast_reduce_us=%.2f", n_dev, n4 * 16, us_mr, us_ur);
    log.add("RESULT in-switch reduce: %.1f GB/s of aggregated gradient into GPU 0 (%.1f GB/s of replica data reduced); "
            "peer-load reduce: %.1f GB/s aggregated", n4 * 16 / us_mr * 1e-3, n4 * 16.0 * n_dev / us_mr * 1e-3,
            n4 * 16 / us_ur * 1e-3);
  }
  return finish(true);
}

}  // extern "C"
