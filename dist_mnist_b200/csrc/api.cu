// C ABI of the native runtime (loaded from Python with ctypes; see dist_mnist_b200/_native.py).
//
// The ABI is deliberately flat: kernel parameter blocks are passed as raw bytes that mirror the structs
// in protocol.h (the Python side keeps ctypes mirrors and checks sizeof at import), pointers travel as
// integers, streams as cudaStream_t handles taken from torch.cuda.current_stream().
#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>
#include <stdint.h>
#include <string.h>
#include <stdio.h>
#include <string>

#include "activation.cuh"
#include "common.cuh"
#include "fused.h"
#include "loss.cuh"
#include "protocol.h"

namespace dm {
size_t gemm_smem_bytes(int bn, int stages, int cluster);
cudaError_t launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int dtype, bool a_mn,
                        bool b_mn, int splits, cudaStream_t stream);
size_t head_smem_bytes(int B_pad, int H, int C);
cudaError_t launch_head(const HeadParams& p, cudaStream_t stream);
cudaError_t launch_grad_clip(const GradClipParams& p, int stage, cudaStream_t stream);
cudaError_t launch_accuracy(const float* logits, const float* labels, int B, int C, uint32_t* correct,
                            cudaStream_t stream);
cudaError_t launch_ps_serve(const PsServeParams& p, int n_ctas, int cluster, cudaStream_t stream);
cudaError_t launch_dense_apply(float* params, float* m, float* v, const float* grad, uint16_t* shadow, size_t n,
                               int opt, float lr, float beta1, float beta2, float eps, uint32_t t,
                               cudaStream_t stream);
cudaError_t launch_shadow_refresh(const float* src, uint16_t* dst, size_t n, cudaStream_t stream);
cudaError_t launch_worker_done(uint32_t* done_slot, const uint32_t* seq_ptr, cudaStream_t stream);
cudaError_t launch_wait_ack(const uint32_t* inbox, uint32_t n_inbox, const uint32_t* seq_ptr, cudaStream_t stream);
cudaError_t launch_p2p_copy(void* dst, const void* src, size_t bytes, int mode, int ctas, uint32_t* flag,
                            uint32_t flag_value, cudaStream_t stream);
cudaError_t launch_p2p_reduce_apply(float* params, const float* const* grads, int n_src, size_t n, float lr,
                                    int ctas, cudaStream_t stream);
cudaError_t launch_pingpong(uint32_t* local_flag, uint32_t* remote_flag, int iters, int role, uint64_t* out_ns,
                            cudaStream_t stream);
}  // namespace dm

static thread_local std::string g_err;

static int fail(const char* what, cudaError_t e) {
  g_err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
  return static_cast<int>(e) ? static_cast<int>(e) : -1;
}
#define DM_CUDA(call)                          \
  do {                                         \
    cudaError_t e__ = (call);                  \
    if (e__ != cudaSuccess) return fail(#call, e__); \
  } while (0)

extern "C" {

const char* dm_last_error() { return g_err.c_str(); }

int dm_sizeof(const char* name) {
  using namespace dm;
  if (!strcmp(name, "PushTarget")) return sizeof(PushTarget);
  if (!strcmp(name, "GemmParams")) return sizeof(GemmParams);
  if (!strcmp(name, "HeadParams")) return sizeof(HeadParams);
  if (!strcmp(name, "StepResult")) return sizeof(StepResult);
  if (!strcmp(name, "PsItem")) return sizeof(PsItem);
  if (!strcmp(name, "PsItemState")) return sizeof(PsItemState);
  if (!strcmp(name, "PsServeParams")) return sizeof(PsServeParams);
  if (!strcmp(name, "CUtensorMap")) return sizeof(CUtensorMap);
  if (!strcmp(name, "FusedSlice")) return sizeof(FusedSlice);
  if (!strcmp(name, "FusedShard")) return sizeof(FusedShard);
  if (!strcmp(name, "FusedParams")) return sizeof(FusedParams);
  if (!strcmp(name, "FusedMaps")) return sizeof(FusedMaps);
  if (!strcmp(name, "GradClipVar")) return sizeof(GradClipVar);
  if (!strcmp(name, "GradClipParams")) return sizeof(GradClipParams);
  return -1;
}

// ------------------------------------------------------------------------------------------
// device / memory
// ------------------------------------------------------------------------------------------
int dm_device_count(int* n) {
  cudaError_t e = cudaGetDeviceCount(n);
  if (e != cudaSuccess) { *n = 0; cudaGetLastError(); }
  return 0;
}
int dm_set_device(int dev) { DM_CUDA(cudaSetDevice(dev)); return 0; }
int dm_device_sm_count(int dev, int* n) {
  DM_CUDA(cudaDeviceGetAttribute(n, cudaDevAttrMultiProcessorCount, dev));
  return 0;
}
int dm_device_clock_khz(int dev, int* khz) {
  DM_CUDA(cudaDeviceGetAttribute(khz, cudaDevAttrClockRate, dev));
  return 0;
}
int dm_device_cc(int dev, int* major, int* minor) {
  DM_CUDA(cudaDeviceGetAttribute(major, cudaDevAttrComputeCapabilityMajor, dev));
  DM_CUDA(cudaDeviceGetAttribute(minor, cudaDevAttrComputeCapabilityMinor, dev));
  return 0;
}
int dm_cuda_malloc(int dev, size_t bytes, void** out) {
  DM_CUDA(cudaSetDevice(dev));
  DM_CUDA(cudaMalloc(out, bytes));
  DM_CUDA(cudaMemset(*out, 0, bytes));
  return 0;
}
int dm_cuda_free(void* p) { DM_CUDA(cudaFree(p)); return 0; }
int dm_host_alloc(size_t bytes, void** out) {
  DM_CUDA(cudaHostAlloc(out, bytes, cudaHostAllocPortable));
  memset(*out, 0, bytes);
  return 0;
}
int dm_host_free(void* p) { DM_CUDA(cudaFreeHost(p)); return 0; }
int dm_ipc_get_handle(void* ptr, void* out64) {
  cudaIpcMemHandle_t h;
  DM_CUDA(cudaIpcGetMemHandle(&h, ptr));
  static_assert(sizeof(h) == 64, "ipc handle size");
  memcpy(out64, &h, 64);
  return 0;
}
int dm_ipc_open_handle(int dev, const void* handle64, void** out) {
  DM_CUDA(cudaSetDevice(dev));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  DM_CUDA(cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}
int dm_ipc_close(void* p) { DM_CUDA(cudaIpcCloseMemHandle(p)); return 0; }
int dm_can_access_peer(int dev, int peer, int* ok) { DM_CUDA(cudaDeviceCanAccessPeer(ok, dev, peer)); return 0; }
int dm_enable_peer_access(int dev, int peer) {
  DM_CUDA(cudaSetDevice(dev));
  cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return 0; }
  if (e != cudaSuccess) return fail("cudaDeviceEnablePeerAccess", e);
  return 0;
}
int dm_memcpy_async(void* dst, const void* src, size_t bytes, void* stream) {
  DM_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, static_cast<cudaStream_t>(stream)));
  return 0;
}
int dm_memset_async(void* dst, int value, size_t bytes, void* stream) {
  DM_CUDA(cudaMemsetAsync(dst, value, bytes, static_cast<cudaStream_t>(stream)));
  return 0;
}
int dm_stream_create(void** out) {
  cudaStream_t s;
  DM_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  *out = s;
  return 0;
}
int dm_stream_destroy(void* s) { DM_CUDA(cudaStreamDestroy(static_cast<cudaStream_t>(s))); return 0; }
int dm_stream_sync(void* s) { DM_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(s))); return 0; }
// `waiter` does not run anything enqueued after this call until everything enqueued on `other` so far has finished
int dm_stream_wait_stream(void* waiter, void* other) {
  cudaEvent_t e;
  DM_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  DM_CUDA(cudaEventRecord(e, static_cast<cudaStream_t>(other)));
  DM_CUDA(cudaStreamWaitEvent(static_cast<cudaStream_t>(waiter), e, 0));
  DM_CUDA(cudaEventDestroy(e));
  return 0;
}
int dm_stream_query(void* s) {  // 0 = idle, 1 = busy, <0 error
  cudaError_t e = cudaStreamQuery(static_cast<cudaStream_t>(s));
  if (e == cudaSuccess) return 0;
  if (e == cudaErrorNotReady) { cudaGetLastError(); return 1; }
  fail("cudaStreamQuery", e);
  return -1;
}

// ------------------------------------------------------------------------------------------
// TMA tensor maps. dtype: 0 = fp32, 1 = bf16. 2-D, 128-byte swizzle, zero fill out of bounds.
// The global address may be a peer-mapped (cudaIpcOpenMemHandle) pointer: the resulting TMA loads
// then travel over NVLink from the PS shard straight into the consumer's shared memory.
// ------------------------------------------------------------------------------------------
int dm_make_tensor_map_2d(void* out, void* gptr, int dtype, uint64_t dim0, uint64_t dim1, uint64_t stride1_bytes,
                          uint32_t box0, uint32_t box1) {
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || fn == nullptr) {
      g_err = "cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed";
      return -1;
    }
    encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }
  CUtensorMap tm;
  cuuint64_t dims[2] = {dim0, dim1};
  cuuint64_t strides[1] = {stride1_bytes};
  cuuint32_t box[2] = {box0, box1};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMapDataType dt = dtype == 0 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUresult r = encode(&tm, dt, 2, gptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf),
             "cuTensorMapEncodeTiled failed: CUresult %d (ptr=%p dims=%llu,%llu stride=%llu box=%u,%u); "
             "row strides must be multiples of 16 bytes", int(r), gptr,
             (unsigned long long)dim0, (unsigned long long)dim1, (unsigned long long)stride1_bytes, box0, box1);
    g_err = buf;
    return -1;
  }
  memcpy(out, &tm, sizeof(tm));
  return 0;
}

// 3-D fp32 tensor map [dim2][dim1][dim0] (dim0 contiguous), box {box0, box1, 1}, 128-byte swizzle: the mailbox slots
// of one variable ([slot][row][col]) as the destination of the fused kernel's TMA-store gradient push.
int dm_make_tensor_map_3d(void* out, void* gptr, uint64_t dim0, uint64_t dim1, uint64_t dim2, uint64_t stride1_bytes,
                          uint64_t stride2_bytes, uint32_t box0, uint32_t box1) {
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || fn == nullptr) {
      g_err = "cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed";
      return -1;
    }
    encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }
  CUtensorMap tm;
  cuuint64_t dims[3] = {dim0, dim1, dim2};
  cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
  cuuint32_t box[3] = {box0, box1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = encode(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, gptr, dims, strides, box, estr,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled(3d) failed: CUresult %d (ptr=%p dims=%llu,%llu,%llu strides=%llu,%llu "
             "box=%u,%u)", int(r), gptr, (unsigned long long)dim0, (unsigned long long)dim1, (unsigned long long)dim2,
             (unsigned long long)stride1_bytes, (unsigned long long)stride2_bytes, box0, box1);
    g_err = buf;
    return -1;
  }
  memcpy(out, &tm, sizeof(tm));
  return 0;
}

// ------------------------------------------------------------------------------------------
// kernel launches
// ------------------------------------------------------------------------------------------
int dm_gemm_smem_bytes(int bn, int stages, int cluster) {
  return static_cast<int>(dm::gemm_smem_bytes(bn, stages, cluster));
}

// Once per device, before any launch / graph capture: opt the big-smem kernels into their dynamic smem sizes and
// force-load every kernel (DESIGN §7). The order is where each kernel's code lands, which the flagship rate depends on
// (DESIGN §4): kernels added to the list go after the fused ones.
int dm_prepare_kernels(int dev) {
  DM_CUDA(cudaSetDevice(dev));
  DM_CUDA(dm::prepare_gemm_kernels());
  DM_CUDA(dm::prepare_head_kernels());
  DM_CUDA(dm::prepare_grad_clip_kernels());
  DM_CUDA(dm::prepare_ps_kernels());
  DM_CUDA(dm::prepare_p2p_kernels());
  DM_CUDA(dm::prepare_fused_kernels());
  DM_CUDA(dm::prepare_nvls_kernels());
  return 0;
}

// Fused worker-step kernel (fused_step_sm90.cu): direct launch (tests / tools; the engine goes through fused_exec.cu)
int dm_launch_fused(const void* maps, const void* params, int lanes, void* stream) {
  dm::FusedMaps m;
  dm::FusedParams p;
  memcpy(&m, maps, sizeof(m));
  memcpy(&p, params, sizeof(p));
  DM_CUDA(dm::launch_fused_step(m, p, lanes, static_cast<cudaStream_t>(stream)));
  return 0;
}
// How many clusters of the fused step a batch of `batch` rows runs can be co-resident on the device: with (clip != 0)
// or without gradient clipping, with (l2 != 0) or without L2 regularization, and with the head `head` selects:
// head = act + 256 loss_kind + 65536 smoothed, the ActivationKind of the hidden layer, the LossKind, and 1 if the labels
// are smoothed (so a plain ActivationKind asks for LOSS_BOOK without smoothing)
int dm_fused_max_lanes(int dev, int batch, int clip, int l2, int head, int* out) {
  const int act = head & 255, loss_kind = (head >> 8) & 255, smoothed = head >> 16;
  if (!dm::act_valid(act) || !dm::loss_valid(loss_kind) || (smoothed != 0 && smoothed != 1))
    return fail("dm_fused_max_lanes(head)", cudaErrorInvalidValue);
  DM_CUDA(cudaSetDevice(dev));
  DM_CUDA(dm::fused_max_lanes(batch, clip != 0, l2 != 0, dm::fused_general_head(act, loss_kind, smoothed), out));
  return 0;
}
int dm_fused_smem_bytes(int batch) { return static_cast<int>(dm::fused_smem_bytes(batch)); }

int dm_launch_gemm(const void* tmA, const void* tmB, const void* params, int dtype, int a_mn, int b_mn, int splits,
                   void* stream) {
  CUtensorMap a, b;
  dm::GemmParams p;
  memcpy(&a, tmA, sizeof(a));
  memcpy(&b, tmB, sizeof(b));
  memcpy(&p, params, sizeof(p));
  DM_CUDA(dm::launch_gemm(a, b, p, dtype, a_mn != 0, b_mn != 0, splits, static_cast<cudaStream_t>(stream)));
  return 0;
}
// Graph engine gradient clipping tail (clip_sm90.cu): stage 0 sums of squares, 1 clip into the mailbox, 2 flags
int dm_launch_grad_clip(const void* params, int stage, void* stream) {
  dm::GradClipParams p;
  memcpy(&p, params, sizeof(p));
  DM_CUDA(dm::launch_grad_clip(p, stage, static_cast<cudaStream_t>(stream)));
  return 0;
}
int dm_launch_head(const void* params, void* stream) {
  dm::HeadParams p;
  memcpy(&p, params, sizeof(p));
  DM_CUDA(dm::launch_head(p, static_cast<cudaStream_t>(stream)));
  return 0;
}
int dm_launch_accuracy(const void* logits, const void* labels, int B, int C, void* correct, void* stream) {
  DM_CUDA(dm::launch_accuracy(static_cast<const float*>(logits), static_cast<const float*>(labels), B, C,
                              static_cast<uint32_t*>(correct), static_cast<cudaStream_t>(stream)));
  return 0;
}
int dm_launch_ps_serve(const void* params, int n_ctas, int cluster, void* stream) {
  dm::PsServeParams p;
  memcpy(&p, params, sizeof(p));
  DM_CUDA(dm::launch_ps_serve(p, n_ctas, cluster, static_cast<cudaStream_t>(stream)));
  return 0;
}
int dm_launch_dense_apply(void* params, void* m, void* v, const void* grad, void* shadow, size_t n, int opt, float lr,
                          float beta1, float beta2, float eps, uint32_t t, void* stream) {
  DM_CUDA(dm::launch_dense_apply(static_cast<float*>(params), static_cast<float*>(m), static_cast<float*>(v),
                                 static_cast<const float*>(grad), static_cast<uint16_t*>(shadow), n, opt, lr, beta1,
                                 beta2, eps, t, static_cast<cudaStream_t>(stream)));
  return 0;
}
int dm_launch_shadow_refresh(const void* src, void* dst, size_t n, void* stream) {
  DM_CUDA(dm::launch_shadow_refresh(static_cast<const float*>(src), static_cast<uint16_t*>(dst), n,
                                    static_cast<cudaStream_t>(stream)));
  return 0;
}
int dm_launch_worker_done(void* done_slot, const void* seq_ptr, void* stream) {
  DM_CUDA(dm::launch_worker_done(static_cast<uint32_t*>(done_slot), static_cast<const uint32_t*>(seq_ptr),
                                 static_cast<cudaStream_t>(stream)));
  return 0;
}
int dm_launch_wait_ack(const void* inbox, uint32_t n_inbox, const void* seq_ptr, void* stream) {
  DM_CUDA(dm::launch_wait_ack(static_cast<const uint32_t*>(inbox), n_inbox, static_cast<const uint32_t*>(seq_ptr),
                              static_cast<cudaStream_t>(stream)));
  return 0;
}
int dm_launch_p2p_copy(void* dst, const void* src, size_t bytes, int mode, int ctas, void* flag, uint32_t flag_value,
                       void* stream) {
  DM_CUDA(dm::launch_p2p_copy(dst, src, bytes, mode, ctas, static_cast<uint32_t*>(flag), flag_value,
                              static_cast<cudaStream_t>(stream)));
  return 0;
}
int dm_launch_p2p_reduce_apply(void* params, const void* grads_ptr_array_dev, int n_src, size_t n, float lr, int ctas,
                               void* stream) {
  DM_CUDA(dm::launch_p2p_reduce_apply(static_cast<float*>(params),
                                      static_cast<const float* const*>(grads_ptr_array_dev), n_src, n, lr, ctas,
                                      static_cast<cudaStream_t>(stream)));
  return 0;
}
int dm_launch_pingpong(void* local_flag, void* remote_flag, int iters, int role, void* out_ns, void* stream) {
  DM_CUDA(dm::launch_pingpong(static_cast<uint32_t*>(local_flag), static_cast<uint32_t*>(remote_flag), iters, role,
                              static_cast<uint64_t*>(out_ns), static_cast<cudaStream_t>(stream)));
  return 0;
}

}  // extern "C"
