// Fused classifier head for sm_90a: last dense layer + softmax + loss + accuracy + every gradient that
// does not need a big GEMM, with the small-variable gradient push fused in.
//
// One launch computes, for h = activations of the last hidden layer [B][H]:
//   logits = h . W_last^T + b_last              (W_last/b_last read straight from the PS shard: peer loads)
//   p      = softmax(logits)
//   loss   = LOSS_BOOK: -mean_{B x C}(labels * log(clip(p, 1e-10, 1)))     reference DS:52-53
//            LOSS_XENT: mean_B(softmax_cross_entropy_with_logits)           reference DS:35
//   correct= #(argmax logits == argmax labels)                              (accuracy numerator, SURVEY K12)
//   dlogits, dW_last = dlogits^T . h, db_last = sum_B dlogits
//   dpre   = (dlogits . W_last) * relu'(h)      -> [B][H] buffer consumed by the wgmma dW / dX GEMMs
//   db_hid = sum_B dpre
// and pushes dW_last / db_last / db_hid to the parameter server (mailbox + flags, or red.add for SGD).
//
// grid = ceil(H / 128) CTAs x 512 threads. Every CTA recomputes the (tiny) logits/softmax phase and then
// owns a 128-wide slice of H for the gradient phase, so no inter-CTA synchronisation is needed.
// The kernel is latency- not throughput-bound (~0.2 MFLOP), so it is organised to keep every phase a handful
// of dependent instructions deep: operands are staged in shared memory once, all global loads of a phase are
// independent, 16 warps hide the shared-memory latency.
// Replaces reference ops DS:52-53 + their gradients from DS:103 (SURVEY K3, K4, K5, part of K6, K12).
#include "common.cuh"
#include "protocol.h"

namespace dm {

constexpr int kHeadThreads = 512;
constexpr int kHeadSlice = 128;
constexpr int kHeadGroups = kHeadThreads / kHeadSlice;  // batch-row groups in the gradient phase
constexpr int kMaxC = 16;
constexpr int kMaxB = 256;
constexpr int kPartStride = kMaxC + 1;

__device__ __forceinline__ float ld_act(const void* __restrict__ p, size_t idx, int is_bf16) {
  return is_bf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[idx])
                 : reinterpret_cast<const float*>(p)[idx];
}
__device__ __forceinline__ void st_act(void* __restrict__ p, size_t idx, int is_bf16, float v) {
  if (is_bf16) reinterpret_cast<__nv_bfloat16*>(p)[idx] = __float2bfloat16(v);
  else reinterpret_cast<float*>(p)[idx] = v;
}
// 4 consecutive activations (16-byte aligned for fp32, 8-byte for bf16)
__device__ __forceinline__ float4 ld_act4(const void* __restrict__ p, size_t idx, int is_bf16) {
  if (is_bf16) {
    const uint2 raw = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(p) + idx);
    const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(&raw.x);
    const __nv_bfloat162 hi = *reinterpret_cast<const __nv_bfloat162*>(&raw.y);
    const float2 a = __bfloat1622float2(lo), b = __bfloat1622float2(hi);
    return make_float4(a.x, a.y, b.x, b.y);
  }
  return *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p) + idx);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct ResolvedPushH {
  float* base;
  uint32_t* flags;
};
__device__ __forceinline__ ResolvedPushH resolve_push_h(const PushTarget& t, uint32_t seq) {
  ResolvedPushH r{t.base, t.flags};
  if (t.mode == PUSH_MAILBOX) {
    const uint32_t slot = seq % t.nslots;
    r.base = t.base + static_cast<uint64_t>(slot) * t.slot_stride;
    r.flags = t.flags + static_cast<uint64_t>(slot) * t.flag_slot_stride;
  }
  return r;
}
__device__ __forceinline__ void push_value(const PushTarget& t, float* dst, float v) {
  if (t.mode == PUSH_ATOMIC) red_add_sys_f32(dst, t.scale * v);
  else *dst = v;
}

// shared-memory row stride of W_last: multiple of 4 floats with (stride/4) odd, so that the 16 class rows
// read by one half-warp land in distinct bank groups.
__host__ __device__ __forceinline__ int head_w_stride(int H) {
  int s = (H + 3) & ~3;
  if (((s >> 2) & 1) == 0) s += 4;
  return s;
}

__global__ void __launch_bounds__(kHeadThreads, 1) head_kernel(const __grid_constant__ HeadParams p) {
  extern __shared__ __align__(16) float hsm[];
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int C = p.C, H = p.H, B = p.B;
  const int ldw = head_w_stride(H);
  const int h0 = blockIdx.x * kHeadSlice;

  // smem carve-up. region0 holds W_last, later (gradient phase) the cross-group partial sums.
  const int region0 = max(kMaxC * ldw, (kHeadGroups - 1) * kHeadSlice * kPartStride);
  float* sW = hsm;                               // [kMaxC][ldw] (rows >= C are zero)
  float* sPart = hsm;                            // aliases sW once the W columns are in registers
  float* sLogit = hsm + region0;                 // [B_pad][kMaxC] logits, then dlogits
  float* sHs = sLogit + p.B_pad * kMaxC;         // [B_pad][kHeadSlice] this CTA's slice of h
  float* sRed = sHs + p.B_pad * kHeadSlice;      // [64] block reductions
  __shared__ uint32_t s_seq;
  __shared__ uint32_t s_gstep;
  long long* dbg = (p.debug_ts != nullptr && blockIdx.x == 0) ? p.debug_ts : nullptr;
  if (dbg && tid == 0) dbg[0] = clock64();
  grid_dep_launch();  // PDL: the dW kernel may set itself up (barriers, tensor-map prefetch) while we run

  // ---- phase A.1: stage W_last (peer loads from the PS shard) — independent of the forward kernels, so under
  //      PDL it overlaps their tail ----
  for (int i = tid; i < kMaxC * ldw; i += kHeadThreads) {
    const int c = i / ldw, k = i - c * ldw;
    sW[i] = (c < C && k < H) ? p.w_last[static_cast<size_t>(c) * H + k] : 0.f;
  }
  grid_dep_wait();    // the forward kernels' activations and the step's sequence number are visible from here

  if (tid == 0) {
    uint32_t seq = p.seq_ptr ? *reinterpret_cast<volatile uint32_t*>(p.seq_ptr) : 1u;
    s_seq = seq;
    uint32_t gstep = seq;
    if (p.compute_grads && p.push.mode == PUSH_MAILBOX && p.inbox != nullptr) {
      // flow control: the mailbox slot we are about to overwrite was used by push (seq - nslots);
      // wait until the PS has acknowledged it. The PS writes the inbox into *our* HBM, so this spins locally.
      const volatile uint32_t* inbox = reinterpret_cast<const volatile uint32_t*>(p.inbox);
      if (seq > p.nslots) {
        const uint64_t t0 = globaltimer_ns();
        for (uint32_t i = 0; i < p.n_inbox; ++i) {
          while (static_cast<int32_t>(inbox[2 * i] - (seq - p.nslots)) < 0) {
            if (globaltimer_ns() - t0 > DM_SPIN_TIMEOUT_NS) {
              printf("[dm] head: PS %u ack timeout (seq=%u ack=%u)\n", i, seq, inbox[2 * i]);
              __trap();
            }
          }
        }
      }
      // entry 0 belongs to the shard that owns global_step (first variable created, reference DS:91).
      // global_step as of our last acknowledged push + our own pushes since then: exact with one worker,
      // a lower bound under concurrency (the reference's fetched value is equally unordered w.r.t. peers).
      const uint32_t ack = inbox[0];
      __threadfence();
      gstep = inbox[1] + (seq - ack);
    }
    s_gstep = gstep;
    if (dbg) dbg[1] = clock64();   // seq read + ack wait done
  }

  // ---- phase A.2: this CTA's slice of h ----
  for (int i = tid; i < p.B_pad * kHeadSlice; i += kHeadThreads) {
    const int b = i / kHeadSlice, hh = i - b * kHeadSlice;
    sHs[i] = (b < B && h0 + hh < H) ? ld_act(p.h, static_cast<size_t>(b) * p.ldh + h0 + hh, p.act_bf16) : 0.f;
  }
  __syncthreads();
  if (dbg && tid == 0) dbg[2] = clock64();
  const uint32_t seq = s_seq;

  // ---- phase B+C: logits, softmax, loss, accuracy and dlogits. thread -> (row b, class c): the 16 lanes of a
  //      half-warp own one batch row, so every per-row reduction is four xor-shuffles and the logits never
  //      leave registers. ----
  float loss_part = 0.f;
  float corr_part = 0.f;
  {
    const int c = lane & (kMaxC - 1);
    const bool c_ok = c < C;
    const float bias = c_ok ? p.b_last[c] : 0.f;
    const float* wrow = sW + c * ldw;
    const bool h_smem = gridDim.x == 1;          // the staged slice is the whole of h
    const int H4 = (h_smem || (p.ldh & 3) == 0) ? (H & ~3) : 0;
    for (int b0 = warp * 2; b0 < B; b0 += (kHeadThreads / 32) * 2) {   // warp-uniform trip count
      const int b = b0 + (lane >> 4);
      const bool row_ok = b < B;
      const int bs = row_ok ? b : B - 1;
      const float y = (c_ok && row_ok) ? p.labels[static_cast<size_t>(bs) * C + c] : 0.f;  // in flight during the dot
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      if (h_smem) {
        const float* hrow = sHs + bs * kHeadSlice;
#pragma unroll 4
        for (int k = 0; k < H4; k += 4) {
          const float4 hv = *reinterpret_cast<const float4*>(hrow + k);
          const float4 wv = *reinterpret_cast<const float4*>(wrow + k);
          a0 = fmaf(hv.x, wv.x, a0); a1 = fmaf(hv.y, wv.y, a1);
          a2 = fmaf(hv.z, wv.z, a2); a3 = fmaf(hv.w, wv.w, a3);
        }
        for (int k = H4; k < H; ++k) a0 = fmaf(hrow[k], wrow[k], a0);
      } else {
        const size_t rowoff = static_cast<size_t>(bs) * p.ldh;
#pragma unroll 8
        for (int k = 0; k < H4; k += 4) {
          const float4 hv = ld_act4(p.h, rowoff + k, p.act_bf16);
          const float4 wv = *reinterpret_cast<const float4*>(wrow + k);
          a0 = fmaf(hv.x, wv.x, a0); a1 = fmaf(hv.y, wv.y, a1);
          a2 = fmaf(hv.z, wv.z, a2); a3 = fmaf(hv.w, wv.w, a3);
        }
        for (int k = H4; k < H; ++k) a0 = fmaf(ld_act(p.h, rowoff + k, p.act_bf16), wrow[k], a0);
      }
      const float z = c_ok ? (a0 + a1) + (a2 + a3) + bias : -INFINITY;
      // row reductions over the 16-lane group
      float zmax = z, ybest = c_ok ? y : -INFINITY, ysum = y;
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {
        zmax = fmaxf(zmax, __shfl_xor_sync(0xffffffffu, zmax, o));
        ybest = fmaxf(ybest, __shfl_xor_sync(0xffffffffu, ybest, o));
        ysum += __shfl_xor_sync(0xffffffffu, ysum, o);
      }
      int zarg = (c_ok && z == zmax) ? c : kMaxC, yarg = (c_ok && y == ybest) ? c : kMaxC;  // first maximum wins
      const float e = c_ok ? __expf(z - zmax) : 0.f;
      float esum = e;
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {
        zarg = min(zarg, __shfl_xor_sync(0xffffffffu, zarg, o));
        yarg = min(yarg, __shfl_xor_sync(0xffffffffu, yarg, o));
        esum += __shfl_xor_sync(0xffffffffu, esum, o);
      }
      const float pc = e / esum;
      float dl = 0.f, lc = 0.f;
      if (p.loss_kind == LOSS_BOOK) {
        // L = -(1/(B*C)) sum y*log(clip(p,1e-10,1));  dL/dp = -y/(B*C*p) where the clip passes gradient
        const float k = 1.f / (static_cast<float>(B) * static_cast<float>(C));
        const bool pass = c_ok && (pc >= 1e-10f) && (pc <= 1.0f);
        const float g = pass ? (-k * y / pc) : 0.f;
        float gp = g * pc;
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) gp += __shfl_xor_sync(0xffffffffu, gp, o);
        dl = pc * (g - gp);
        lc = c_ok ? -k * y * __logf(fminf(fmaxf(pc, 1e-10f), 1.0f)) : 0.f;
      } else {
        // L = (1/B) sum_b -sum_c y*log_softmax(z);  dz = (p*sum(y) - y)/B
        const float k = 1.f / static_cast<float>(B);
        dl = k * (pc * ysum - y);
        lc = c_ok ? -k * y * (z - (zmax + __logf(esum))) : 0.f;
      }
      if (row_ok) {
        sLogit[b * kMaxC + c] = c_ok ? dl : 0.f;
        loss_part += lc;
        if (c == 0) corr_part += (zarg == yarg) ? 1.f : 0.f;
      }
    }
  }
  // block-reduce loss / correct (only CTA 0 reports them)
  loss_part = warp_sum(loss_part);
  corr_part = warp_sum(corr_part);
  if (lane == 0) { sRed[warp] = loss_part; sRed[32 + warp] = corr_part; }

  // this thread's column of W_last, before region0 is recycled for the partial sums
  const int hh = tid & (kHeadSlice - 1);
  const int grp = tid >> 7;  // kHeadGroups groups split the batch rows
  const int h = h0 + hh;
  const bool h_ok = h < H;
  float wcol[kMaxC];
#pragma unroll
  for (int c = 0; c < kMaxC; ++c) wcol[c] = sW[c * ldw + min(h, H - 1)];
  __syncthreads();
  if (dbg && tid == 0) dbg[3] = clock64();

  if (blockIdx.x == 0 && tid == 0) {
    float l = 0.f, cr = 0.f;
    for (int w = 0; w < kHeadThreads / 32; ++w) { l += sRed[w]; cr += sRed[32 + w]; }
    uint32_t gstep = s_gstep;
    if (p.compute_grads && p.push.mode == PUSH_ATOMIC && p.ps_global_step != nullptr)
      gstep = atom_add_sys_u32(p.ps_global_step, 1u) + 1u;  // async SGD: this push *is* global step gstep
    StepResult r;
    r.loss = l;
    r.global_step = gstep;
    r.correct = static_cast<uint32_t>(cr + 0.5f);
    r.seq = seq;
    *p.result = r;
  }
  if (!p.compute_grads) return;

  // ---- phase D: gradients for this CTA's 128-wide slice of H; thread -> (column hh, row group grp) ----
  float dw[kMaxC];
#pragma unroll
  for (int c = 0; c < kMaxC; ++c) dw[c] = 0.f;
  float dbh = 0.f;
  for (int b = grp; b < B; b += kHeadGroups) {
    const float hv = sHs[b * kHeadSlice + hh];
    const float4* dl4 = reinterpret_cast<const float4*>(sLogit + b * kMaxC);  // broadcast reads
    float dh = 0.f;
#pragma unroll
    for (int c4 = 0; c4 < kMaxC / 4; ++c4) {
      const float4 d = dl4[c4];
      dw[4 * c4 + 0] = fmaf(d.x, hv, dw[4 * c4 + 0]); dh = fmaf(d.x, wcol[4 * c4 + 0], dh);
      dw[4 * c4 + 1] = fmaf(d.y, hv, dw[4 * c4 + 1]); dh = fmaf(d.y, wcol[4 * c4 + 1], dh);
      dw[4 * c4 + 2] = fmaf(d.z, hv, dw[4 * c4 + 2]); dh = fmaf(d.z, wcol[4 * c4 + 2], dh);
      dw[4 * c4 + 3] = fmaf(d.w, hv, dw[4 * c4 + 3]); dh = fmaf(d.w, wcol[4 * c4 + 3], dh);
    }
    const float dp = hv > 0.f ? dh : 0.f;
    dbh += dp;
    if (h_ok) st_act(p.dpre, static_cast<size_t>(b) * p.ldh + h, p.act_bf16, dp);
  }
  // zero the padding rows of dpre so the dW GEMM's batch reduction sees zeros
  for (int b = B + grp; b < p.B_pad; b += kHeadGroups)
    if (h_ok) st_act(p.dpre, static_cast<size_t>(b) * p.ldh + h, p.act_bf16, 0.f);

  if (grp > 0) {
    float* dst = sPart + ((grp - 1) * kHeadSlice + hh) * kPartStride;
#pragma unroll
    for (int c = 0; c < kMaxC; ++c) dst[c] = dw[c];
    dst[kMaxC] = dbh;
  }
  __syncthreads();
  if (dbg && tid == 0) dbg[4] = clock64();
  const ResolvedPushH r = resolve_push_h(p.push, seq);
  const ResolvedPushH rb = resolve_push_h(p.push_bh, seq);
  const ResolvedPushH rl = resolve_push_h(p.push_bl, seq);
  if (grp == 0 && h_ok) {
#pragma unroll
    for (int g = 0; g < kHeadGroups - 1; ++g) {
      const float* src = sPart + (g * kHeadSlice + hh) * kPartStride;
#pragma unroll
      for (int c = 0; c < kMaxC; ++c) dw[c] += src[c];
      dbh += src[kMaxC];
    }
#pragma unroll
    for (int c = 0; c < kMaxC; ++c)
      if (c < C) push_value(p.push, r.base + p.off_w_last + static_cast<size_t>(c) * H + h, dw[c]);
    push_value(p.push_bh, rb.base + p.off_b_hidden + h, dbh);
  }
  if (blockIdx.x == 0 && grp == 1 && hh < C) {
    float s0 = 0.f, s1 = 0.f;
    int b = 0;
    for (; b + 1 < B; b += 2) { s0 += sLogit[b * kMaxC + hh]; s1 += sLogit[(b + 1) * kMaxC + hh]; }
    if (b < B) s0 += sLogit[b * kMaxC + hh];
    push_value(p.push_bl, rl.base + p.off_b_last + hh, s0 + s1);
  }
  if (p.push.mode == PUSH_MAILBOX) {
    // the CTA barrier orders every thread's P2P stores before thread 0's cumulative system-scope release
    __syncthreads();
    if (dbg && tid == 0) dbg[5] = clock64();
    if (tid == 0) {
      fence_acq_rel_scoped(p.push.gpu_scope);
      st_relaxed_sys_u32(r.flags + p.item_w_last_base + blockIdx.x, seq);
      st_relaxed_sys_u32(rb.flags + p.item_b_hidden_base + blockIdx.x, seq);
      if (blockIdx.x == 0) st_relaxed_sys_u32(rl.flags + p.item_b_last, seq);
    }
  }
  if (dbg && tid == 0) dbg[6] = clock64();
}

size_t head_smem_bytes(int B_pad, int H, int C) {
  (void)C;
  const int ldw = head_w_stride(H);
  const size_t region0 = static_cast<size_t>(
      kMaxC * ldw > (kHeadGroups - 1) * kHeadSlice * kPartStride ? kMaxC * ldw
                                                                 : (kHeadGroups - 1) * kHeadSlice * kPartStride);
  return sizeof(float) * (region0 + static_cast<size_t>(B_pad) * kMaxC + static_cast<size_t>(B_pad) * kHeadSlice + 64);
}

constexpr int kHeadMaxSmem = 224 * 1024;

cudaError_t prepare_head_kernel() {
  return cudaFuncSetAttribute(head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kHeadMaxSmem);
}

cudaError_t launch_head(const HeadParams& p, cudaStream_t stream) {
  if (p.C > kMaxC || p.B > kMaxB || p.B_pad > kMaxB) return cudaErrorInvalidValue;
  const size_t smem = head_smem_bytes(p.B_pad, p.H, p.C);
  if (smem > static_cast<size_t>(kHeadMaxSmem)) return cudaErrorInvalidValue;
  const int grid = (p.H + kHeadSlice - 1) / kHeadSlice;
  if (!p.pdl) {
    head_kernel<<<grid, kHeadThreads, smem, stream>>>(p);
    return cudaGetLastError();
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kHeadThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, head_kernel, p);
}

// ------------------------------------------------------------------------------------------
// Stand-alone accuracy reduction (evaluation path): count argmax(logits) == argmax(labels).
// One warp per row, block partial -> one atomic per block. SURVEY K12.
// ------------------------------------------------------------------------------------------
__global__ void accuracy_kernel(const float* __restrict__ logits, const float* __restrict__ labels, int B, int C,
                                uint32_t* __restrict__ correct) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  uint32_t local = 0;
  for (int b = warp; b < B; b += nwarps) {
    float zb = -INFINITY, yb = -INFINITY;
    int za = 0x7fffffff, ya = 0x7fffffff;
    for (int c = lane; c < C; c += 32) {
      const float z = logits[static_cast<size_t>(b) * C + c];
      const float y = labels[static_cast<size_t>(b) * C + c];
      if (z > zb) { zb = z; za = c; }
      if (y > yb) { yb = y; ya = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float zo = __shfl_xor_sync(0xffffffffu, zb, o);
      const int zao = __shfl_xor_sync(0xffffffffu, za, o);
      const float yo = __shfl_xor_sync(0xffffffffu, yb, o);
      const int yao = __shfl_xor_sync(0xffffffffu, ya, o);
      if (zo > zb || (zo == zb && zao < za)) { zb = zo; za = zao; }
      if (yo > yb || (yo == yb && yao < ya)) { yb = yo; ya = yao; }
    }
    if (lane == 0 && za == ya) ++local;
  }
  __shared__ uint32_t s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  if (lane == 0 && local) atomicAdd(&s_cnt, local);
  __syncthreads();
  if (threadIdx.x == 0 && s_cnt) atomicAdd(correct, s_cnt);
}

cudaError_t launch_accuracy(const float* logits, const float* labels, int B, int C, uint32_t* correct,
                            cudaStream_t stream) {
  const int threads = 256;
  int blocks = (B * 32 + threads - 1) / threads;
  if (blocks > device_sm_count() * 4) blocks = device_sm_count() * 4;
  if (blocks < 1) blocks = 1;
  accuracy_kernel<<<blocks, threads, 0, stream>>>(logits, labels, B, C, correct);
  return cudaGetLastError();
}

cudaError_t preload_head_kernels() {
  cudaFuncAttributes a;
  cudaError_t e;
  if ((e = cudaFuncGetAttributes(&a, head_kernel)) != cudaSuccess) return e;
  if ((e = cudaFuncGetAttributes(&a, accuracy_kernel)) != cudaSuccess) return e;
  return cudaSuccess;
}

}  // namespace dm
