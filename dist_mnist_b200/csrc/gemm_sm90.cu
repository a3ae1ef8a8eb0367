// wgmma / TMA dense-layer GEMM for sm_90a, with the parameter-server transfers fused in.
//
//   D[M, N] (fp32) = A[M, K] * B[N, K]^T            one 128 x bn output tile per CTA
//
// Operand roles in the MLP (all tensors keep their natural row-major layout; no transposes in global memory):
//   forward   : A = W[out][in]   (K-major, *pulled straight from the PS shard over NVLink by TMA*)
//               B = x[batch][in] (K-major)          D = pre-activation^T      -> EPI_TRANSPOSED (+bias, act)
//   dW        : A = dy[batch][out] (MN-major)  B = x[batch][in] (MN-major)   reduction over batch
//               D = dW[out][in]                     -> EPI_ROWMAJOR_PUSH: the epilogue *is* the gradient
//               push (P2P stores into the PS mailbox + release flag, or red.add for async SGD)
//   dX        : A = W[out][in] (MN-major, pulled from the PS)  B = dy[batch][out] (K-major)
//               D = dx^T                            -> EPI_TRANSPOSED (* act'(mask), bias-grad sums)
//
// These replace the MatMul/BiasAdd/Relu (+grads) ops of the reference training script and the implicit gRPC
// variable fetch / gradient send around them (SURVEY.md K1,K2,K6,X3,X4).
//
// Warp roles (256 threads): two consumer warpgroups issuing wgmma for tile rows [0, 64) and [64, 128); thread 0 also
// issues the TMA loads. wgmma takes A from registers (loaded from the stage in whatever layout TMA left it, so the
// MN-major operands need no transpose) and B from shared memory, K-major only: an MN-major B stage is first copied
// into a K-major tile. After the K loop the accumulators are written to a [128][bn + 4] fp32 tile over the idle
// operand ring, and warps 0..3 run the epilogue with one tile row per thread.
//
// Split-K (forward / dX, whose K loop is TMA-issue bound on one SM): the splits of a tile form a thread-block
// cluster and reduce-scatter their partial accumulators through distributed shared memory (global-scratch
// variants remain for tiles wider than 64 columns). Kernels of one training step are chained with programmatic
// dependent launch (griddepcontrol). (The 784-H-10 models run the whole step in fused_step_sm90.cu instead.)
#include "activation.cuh"
#include "common.cuh"
#include "protocol.h"

namespace dm {

// Two consumer warpgroups (wgmma) and nothing else: a block of 256 threads may use 255 registers per thread, which the
// up to 128 fp32 accumulators per thread need (a separate producer warp would round the block up to 384 threads for
// register allocation, i.e. 168 registers, and make the accumulators spill). Thread 0 also issues the TMA loads.
constexpr int kGemmThreads = 256;
constexpr int kMaxNB = 16;           // n16 blocks per tile: bn <= 256
constexpr int kTileM = 128;
constexpr int kABytes = kTileM * 128;  // one A stage: 128 rows x 128 B (K-major) or slabs x BK rows x 128 B

// Resolve a push target for the current sequence number: returns the destination base pointer
// (slot applied) and the flag array for that slot.
struct ResolvedPush {
  float* base;
  uint32_t* flags;
  uint32_t seq;
};
__device__ __forceinline__ ResolvedPush resolve_push(const PushTarget& t) {
  ResolvedPush r;
  r.seq = t.seq_ptr ? *reinterpret_cast<const volatile uint32_t*>(t.seq_ptr) : 1u;
  r.base = t.base;
  r.flags = t.flags;
  if (t.mode == PUSH_MAILBOX) {
    const uint32_t slot = r.seq % t.nslots;
    r.base = t.base + static_cast<uint64_t>(slot) * t.slot_stride;
    r.flags = t.flags + static_cast<uint64_t>(slot) * t.flag_slot_stride;
  }
  return r;
}

// Bias gradient of an EPI_TRANSPOSED tile: lane m owns feature m and has summed it over the batch tile.
// Called by all 128 epilogue threads of the (finalizing) CTA.
__device__ __forceinline__ void epilogue_colsum(const GemmParams& p, float colsum, int m, bool m_ok) {
  if (!p.has_colsum) return;
  const ResolvedPush r = resolve_push(p.colsum);
  if (m_ok) {
    float* dst = r.base + p.colsum_offset + m;
    if (p.colsum.mode == PUSH_ATOMIC) red_add_sys_f32(dst, p.colsum.scale * colsum);
    else if (gridDim.y > 1) atomicAdd(dst, colsum);
    else *dst = colsum;
  }
  if (p.colsum.mode == PUSH_MAILBOX) {
    named_bar_sync(1, 128);  // orders every lane's P2P store before the one cumulative st.release.sys below
    if (threadIdx.x == 64) st_release_scoped_u32(r.flags + p.colsum_item_base + blockIdx.x, r.seq, p.colsum.gpu_scope);
  }
}

// Byte offset of A element (m, k) inside one operand stage: K-major = 128 rows of 128 B; MN-major = 128 / SLAB
// slabs of BKE k-rows x 128 B (SLAB = BKE m-elements per row). Both 128-byte swizzled (TMA SWIZZLE_128B).
template <typename T, bool MN>
__device__ __forceinline__ uint32_t a_offset(int m, int k) {
  constexpr uint32_t es = sizeof(T);
  constexpr int BKE = 128 / es;
  return MN ? static_cast<uint32_t>(m / BKE) * (BKE * 128u) + sw128_offset(k, m % BKE, es) : sw128_offset(m, k, es);
}

// wgmma A fragment of k-step j for rows r, r + 8 (r = 16 * warp-in-group + lane / 4; c = lane % 4), read from the
// stage with its own layout: the MN-major operands (dW, dX) need no transpose in shared memory.
template <typename T, bool MN>
__device__ __forceinline__ void load_a_frag(const uint8_t* sa, int r, int c, int j, uint32_t (&a)[4]) {
  if constexpr (sizeof(T) == 4) {
    const int k = 8 * j + c;
    a[0] = *reinterpret_cast<const uint32_t*>(sa + a_offset<T, MN>(r, k));
    a[1] = *reinterpret_cast<const uint32_t*>(sa + a_offset<T, MN>(r + 8, k));
    a[2] = *reinterpret_cast<const uint32_t*>(sa + a_offset<T, MN>(r, k + 4));
    a[3] = *reinterpret_cast<const uint32_t*>(sa + a_offset<T, MN>(r + 8, k + 4));
  } else {
    const int k = 16 * j + 2 * c;
    auto pair = [&](int m, int kk) -> uint32_t {
      if constexpr (!MN) return *reinterpret_cast<const uint32_t*>(sa + a_offset<T, MN>(m, kk));
      const uint32_t lo = *reinterpret_cast<const uint16_t*>(sa + a_offset<T, MN>(m, kk));
      const uint32_t hi = *reinterpret_cast<const uint16_t*>(sa + a_offset<T, MN>(m, kk + 1));
      return lo | (hi << 16);
    };
    a[0] = pair(r, k);
    a[1] = pair(r + 8, k);
    a[2] = pair(r, k + 8);
    a[3] = pair(r + 8, k + 8);
  }
}

// this thread's 16 consecutive accumulator columns [c0, c0 + 16) of its tile row, out of the staged tile
__device__ __forceinline__ void acc_ld16(const float* row, int c0, float (&v)[16]) {
#pragma unroll
  for (int j = 0; j < 16; j += 4) {
    const float4 t = *reinterpret_cast<const float4*>(row + c0 + j);
    v[j] = t.x; v[j + 1] = t.y; v[j + 2] = t.z; v[j + 3] = t.w;
  }
}

template <typename T, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint32_t s_last;  // split-K: "this CTA arrived last at the tile counter"
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  constexpr int BKE = 128 / sizeof(T);       // k elements per stage chunk (32 tf32 / 64 bf16) == 128 bytes
  constexpr int KSTEPS = BKE / Wgmma<T>::kK; // 4
  constexpr int SLAB = BKE;                  // MN-major: elements per 128-byte wide slab
  constexpr uint32_t es = sizeof(T);

  const int bn = p.bn;
  const int b_bytes = bn * 128;
  const int stage_bytes = kABytes + b_bytes;
  const int stages = p.stages;

  // the operand ring doubles as the accumulator tile (128 x (bn + 4) fp32) the epilogue reads; keep in sync with
  // gemm_smem_bytes()
  int ring_bytes = stages * stage_bytes;
  const int tile_bytes = (kTileM * (bn + 4) * 4 + 1023) & ~1023;
  if (ring_bytes < tile_bytes) ring_bytes = tile_bytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + ring_bytes);
  uint64_t* empty_bar = full_bar + stages;
  // cluster split-K: landing zone for the partial columns the *other* CTAs of the cluster send us through
  // distributed shared memory: red[src rank][my column][tile row], then csum[src rank][tile row]
  float* red = reinterpret_cast<float*>(smem + ring_bytes + 256);
  float* csum = red + (bn + 8) * kTileM;   // nsplit * ceil(bn / nsplit) <= bn + 8 landing columns
  const bool cluster_mode = p.splitk_cluster != 0 && gridDim.z > 1;
  // MN-major B: K-major copy of the stage's B tile (wgmma reads B from shared memory K-major only)
  const int cl_bytes = cluster_mode ? ((bn + 8) * kTileM + 8 * kTileM) * 4 : 0;
  uint8_t* bt = smem + ((ring_bytes + 256 + cl_bytes + 1023) & ~1023);
  const float* sacc = reinterpret_cast<const float*>(smem);
  const int ldc = bn + 4;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  grid_dep_launch();  // PDL: the next kernel of the step may set itself up while this one runs
  // optional phase timestamps (SM cycle counter) of CTA (0,0,0) — bench_tools/profile_kernels.py --phases
  long long* dbg = (p.debug_ts != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) ? p.debug_ts : nullptr;
  if (dbg && threadIdx.x == 0) dbg[0] = clock64();
  // every CTA: wall-clock (globaltimer, ns) entry/exit stamps, to see stragglers and launch skew
  const int cta_lin = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
  if (p.debug_ts != nullptr && threadIdx.x == 0 && cta_lin < 120) p.debug_ts[16 + 2 * cta_lin] = static_cast<long long>(globaltimer_ns());
  const int m0 = blockIdx.x * kTileM;
  const int n0 = blockIdx.y * bn;
  const int kc_total = (p.K + BKE - 1) / BKE;
  const int kc_begin = blockIdx.z * p.kc_per_split;
  const int kc_end = min(kc_total, kc_begin + p.kc_per_split);
  const int nkc = kc_end - kc_begin;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&tmA);
    prefetch_tensormap(&tmB);
    // The first kernel of a training step opens a new push sequence number (it does not read it itself;
    // every later kernel of the step does, after this kernel has completed). Steps of different lanes may be
    // in flight concurrently, hence the atomic draw from the worker-wide counter.
    if (p.bump_seq != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
      const uint32_t sq = atomicAdd(p.seq_counter, 1u) + 1u;
      *p.bump_seq = sq;
    }
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  grid_dep_wait();    // PDL: everything above overlapped the previous kernel; its outputs are visible from here
  // Distributed shared memory of a peer CTA may only be touched once that CTA is known to be running:
  // everybody arrives here, and waits right before its first remote access / at the end of its role.
  if (cluster_mode) cluster_barrier_arrive_release();
  if (dbg && threadIdx.x == 0) dbg[1] = clock64();
  // the epilogue warps request the bias (a peer load from the PS shard) before the K loop so that its NVLink round
  // trip overlaps it
  const int m_pref = m0 + (warp & 3) * 32 + lane;
  const float bias_pref =
      (warp < 4 && p.epi == EPI_TRANSPOSED && p.bias != nullptr && m_pref < p.M) ? p.bias[m_pref] : 0.f;

  // ===================== TMA producer (thread 0) =====================
  // Up to `stages` k-chunks are in flight: stage s is refilled with chunk i + stages once both consumer warpgroups
  // have released chunk i (empty_bar[s]).
  auto issue = [&](int i) {
    const int s = i % stages;
    mbar_arrive_expect_tx(&full_bar[s], stage_bytes);
    const int k0 = (kc_begin + i) * BKE;
    uint8_t* sa = smem + s * stage_bytes;
    uint8_t* sb = sa + kABytes;
    if constexpr (!A_MN) {
      tma_load_2d(sa, &tmA, &full_bar[s], k0, m0);  // box {BKE, 128}
    } else {
#pragma unroll
      for (int slab = 0; slab < kTileM / SLAB; ++slab)  // box {SLAB, BKE}: BKE k-rows of 128 B
        tma_load_2d(sa + slab * (BKE * 128), &tmA, &full_bar[s], m0 + slab * SLAB, k0);
    }
    if constexpr (!B_MN) {
      tma_load_2d(sb, &tmB, &full_bar[s], k0, n0);  // box {BKE, bn}
    } else {
      for (int slab = 0; slab < bn / SLAB; ++slab)
        tma_load_2d(sb + slab * (BKE * 128), &tmB, &full_bar[s], n0 + slab * SLAB, k0);
    }
  };
  if (threadIdx.x == 0) {
    for (int i = 0; i < min(stages, nkc); ++i) issue(i);
    if (dbg) dbg[2] = clock64();
  }
  {
    // ===================== two consumer warpgroups: wgmma, 64 tile rows each =====================
    const int wg = warp >> 2;
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows r, r + 8
    const int c = lane & 3;
    const int nbn = bn >> 4;                                  // n16 blocks of the tile
    float acc[kMaxNB][8];
#pragma unroll
    for (int nb = 0; nb < kMaxNB; ++nb)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[nb][e] = 0.f;
    for (int i = 0; i < nkc; ++i) {
      const int s = i % stages;
      const uint32_t ph = (i / stages) & 1;
      mbar_wait(&full_bar[s], ph);
      const uint8_t* sa = smem + s * stage_bytes;
      uint32_t b_addr = smem_u32(sa + kABytes);
      if constexpr (B_MN) {
        named_bar_sync(3, 256);   // both warpgroups are done with the previous chunk's K-major copy
        const uint8_t* sb = sa + kABytes;
        for (int idx = threadIdx.x; idx < bn * BKE; idx += 256) {
          const int n = idx / BKE, k = idx - n * BKE;
          const uint32_t src = static_cast<uint32_t>(n / SLAB) * (BKE * 128u) + sw128_offset(k, n % SLAB, es);
          *reinterpret_cast<T*>(bt + sw128_offset(n, k, es)) = *reinterpret_cast<const T*>(sb + src);
        }
        fence_proxy_async_smem_cta();   // generic-proxy writes -> tensor-core (async proxy) reads
        named_bar_sync(3, 256);
        b_addr = smem_u32(bt);
      }
      uint32_t a[KSTEPS][4];
#pragma unroll
      for (int j = 0; j < KSTEPS; ++j) load_a_frag<T, A_MN>(sa, r, c, j, a[j]);
      if (dbg && threadIdx.x == 0 && i == 0) dbg[3] = clock64();
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < KSTEPS; ++j) {
#pragma unroll
        for (int nb = 0; nb < kMaxNB; ++nb) {
          // K-major B: n16 block = 16 rows x 128 B (2048 B); k-step = 32 B inside the 128 B swizzle atom
          if (nb < nbn) Wgmma<T>::mma(acc[nb], a[j], make_wgmma_desc_sw128(b_addr + nb * 2048 + j * 32), (i > 0 || j > 0) ? 1u : 0u);
        }
      }
      wgmma_commit();
      wgmma_wait0();
#pragma unroll
      for (int nb = 0; nb < kMaxNB; ++nb)
#pragma unroll
        for (int e = 0; e < 8; ++e) wgmma_reg_fence(acc[nb][e]);
      if ((warp & 3) == 0 && lane == 0) mbar_arrive(&empty_bar[s]);
      if (threadIdx.x == 0 && i + stages < nkc) {
        mbar_wait(&empty_bar[s], ph);   // both warpgroups are done with chunk i
        issue(i + stages);
      }
    }
    if (dbg && threadIdx.x == 0) dbg[4] = clock64();
    // accumulators -> the [128][bn + 4] fp32 tile over the (now idle) operand ring: the epilogues below own one tile
    // row per thread. Fragment element e of n16 block nb: row r + 8 * ((e >> 1) & 1), column 16 nb + 8 (e >> 2) +
    // 2 c + (e & 1).
    named_bar_sync(3, 256);   // both warpgroups' MMAs have finished reading the ring
    float* st = reinterpret_cast<float*>(smem);
#pragma unroll
    for (int nb = 0; nb < kMaxNB; ++nb) {
      if (nb < nbn) {
#pragma unroll
        for (int e = 0; e < 8; e += 2) {
          const int row = r + 8 * ((e >> 1) & 1);
          const int col = 16 * nb + 8 * (e >> 2) + 2 * c;
          *reinterpret_cast<float2*>(st + row * ldc + col) = make_float2(acc[nb][e], acc[nb][e + 1]);
        }
      }
    }
    named_bar_sync(3, 256);
  }
  if (warp < 4) {
    // ===================== epilogue warps (accumulator tile -> registers -> global / peer) =====================
    if (dbg && threadIdx.x == 64) dbg[5] = clock64();
    const int q = warp;
    const int m = m0 + q * 32 + lane;
    const bool m_ok = m < p.M;
    const float* arow = sacc + (q * 32 + lane) * ldc;   // this thread's accumulator row

    if (p.epi == EPI_TRANSPOSED) {
      // ---- split-K: every CTA parks its fp32 partial tile in scratch; the CTA that arrives last at the tile's
      //      counter sums the partials and runs the real epilogue (one SM's TMA front-end only sustains ~16 B/clk
      //      with 128-byte-wide boxes, so the K loop is spread over several SMs).
      const int nsplit = gridDim.z;
      bool finalize = true;
      float* part_base = nullptr;
      if (cluster_mode) {
        // ---- cluster split-K, phase 1 (reduce-scatter): CTA r of the cluster owns columns [r*cw, (r+1)*cw) of
        // the tile. Every lane sends each of its accumulator values to the owner's shared memory with
        // st.shared::cluster (coalesced over the 32 lanes of a warp); after the cluster barrier every CTA sums
        // the nsplit contributions for its own columns. No global-memory round trip, no atomics.
        cluster_barrier_wait_acquire();   // all CTAs of the cluster are up (arrived after their prologue)
        const uint32_t crank = cluster_ctarank();
        const int cw = (bn + nsplit - 1) / nsplit;
        const uint32_t red_local = smem_u32(red) + ((crank * cw) * kTileM + q * 32 + lane) * 4u;
        int dest = 0, cc = 0;
        for (int c0 = 0; c0 < bn; c0 += 16) {
          float v[16];
          acc_ld16(arow, c0, v);   // (a CTA without k-chunks — K not a multiple of the split — holds zeros)
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const uint32_t ra = mapa_shared_cluster(red_local + static_cast<uint32_t>(cc * kTileM) * 4u, dest);
            st_shared_cluster_f32(ra, v[j]);
            if (++cc == cw) { cc = 0; ++dest; }
          }
        }
        finalize = false;  // phase 2 runs after the cluster barrier below
      } else if (nsplit > 1) {
        // scratch layout [mtile][split][n][128] with the tile row (= lane) fastest: every warp store / load below
        // is one fully used 128-byte line (the row-per-thread layout cost 32 line transactions per instruction
        // and made the fix-up take 8 us).
        part_base = p.splitk_scratch + static_cast<size_t>(blockIdx.x) * nsplit * bn * kTileM + q * 32 + lane;
        float* mine = part_base + static_cast<size_t>(blockIdx.z) * bn * kTileM;
        for (int c0 = 0; c0 < bn; c0 += 16) {
          float v[16];
          acc_ld16(arow, c0, v);
#pragma unroll
          for (int j = 0; j < 16; ++j) mine[static_cast<size_t>(c0 + j) * kTileM] = v[j];
        }
        __threadfence();
        named_bar_sync(1, 128);
        if (!p.has_colsum) {
          // ---- distributed fix-up (forward GEMMs): wait until all splits of this tile have parked their
          // partials (the grid is far smaller than one wave, so all CTAs are co-resident), then every CTA
          // finishes its own slice of the tile's columns: bn/nsplit columns x nsplit partials per lane, all
          // loads independent and coalesced — instead of one CTA re-reading every partial tile.
          if (threadIdx.x == 64) {
            uint32_t* ctr = p.splitk_counter + blockIdx.x;      // monotonic: nsplit arrivals per launch
            const uint32_t old = atomicAdd(ctr, 1u);
            const uint32_t target = (old / nsplit + 1u) * nsplit;
            const uint64_t t0 = globaltimer_ns();
            while (static_cast<int32_t>(ld_acquire_scoped_u32(ctr, 1u) - target) < 0) {
              if (globaltimer_ns() - t0 > DM_SPIN_TIMEOUT_NS) {
                printf("[dm] split-K barrier timeout tile=%d split=%d\n", blockIdx.x, blockIdx.z);
                __trap();
              }
            }
          }
          named_bar_sync(1, 128);
          const int cw = (bn + nsplit - 1) / nsplit;
          const int c_begin = blockIdx.z * cw;
          const int c_end = min(bn, c_begin + cw);
          const float* col0 = part_base;  // + (z * bn + c) * kTileM
          for (int c = c_begin; c < c_end; ++c) {
            float acc = 0.f;
#pragma unroll 8
            for (int z = 0; z < nsplit; ++z) acc += __ldcg(col0 + (static_cast<size_t>(z) * bn + c) * kTileM);
            const int n = n0 + c;
            if (n < p.N && m_ok) {
              float val = acc + bias_pref;
              if (p.mask != nullptr) {
                const float a = p.mask_bf16
                                    ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(
                                          p.mask)[static_cast<size_t>(n) * p.ldmask + m])
                                    : reinterpret_cast<const float*>(p.mask)[static_cast<size_t>(n) * p.ldmask + m];
                val = act_backward(p.act, a, val);   // dX: act'(y) from the layer's output
              } else {
                val = act_forward(p.act, val);
              }
              const size_t o = static_cast<size_t>(n) * p.ldo + m;
              if (p.out_bf16) reinterpret_cast<__nv_bfloat16*>(p.out)[o] = __float2bfloat16(val);
              else reinterpret_cast<float*>(p.out)[o] = val;
            }
          }
          finalize = false;
        } else {
          // ---- last-arriver fix-up (dX GEMMs, whose bias-gradient column sums need the whole tile) ----
          if (threadIdx.x == 64) {
            const uint32_t old = atomicAdd(p.splitk_counter + blockIdx.x, 1u);
            s_last = ((old + 1u) % static_cast<uint32_t>(nsplit)) == 0u;
          }
          named_bar_sync(1, 128);
          finalize = s_last != 0;
          if (finalize) __threadfence();
        }
      }
      if (finalize) {
        const float bias = bias_pref;
        float colsum = 0.f;
        for (int c0 = 0; c0 < bn; c0 += 16) {
          float v[16];
          if (nsplit == 1) {
            acc_ld16(arow, c0, v);
          } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = 0.f;
            // 8 partial tiles (32 independent 16-byte L2 loads) in flight per round: the fix-up is a latency
            // chain of ceil(nsplit / 8) L2 round trips instead of nsplit.
            for (int z0 = 0; z0 < nsplit; z0 += 8) {
              float t[8][16];
#pragma unroll
              for (int zz = 0; zz < 8; ++zz) {
                const int z = min(z0 + zz, nsplit - 1);
                const float* src = part_base + (static_cast<size_t>(z) * bn + c0) * kTileM;
#pragma unroll
                for (int j = 0; j < 16; ++j) t[zz][j] = __ldcg(src + static_cast<size_t>(j) * kTileM);
              }
#pragma unroll
              for (int zz = 0; zz < 8; ++zz) {
                if (z0 + zz < nsplit) {
#pragma unroll
                  for (int j = 0; j < 16; ++j) v[j] += t[zz][j];
                }
              }
            }
          }
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int n = n0 + c0 + j;
            if (n < p.N && m_ok) {
              float val = v[j] + bias;
              if (p.mask != nullptr) {
                const float a = p.mask_bf16
                                    ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(
                                          p.mask)[static_cast<size_t>(n) * p.ldmask + m])
                                    : reinterpret_cast<const float*>(p.mask)[static_cast<size_t>(n) * p.ldmask + m];
                val = act_backward(p.act, a, val);   // dX: act'(y) from the layer's output
              } else {
                val = act_forward(p.act, val);
              }
              colsum += val;
              const size_t o = static_cast<size_t>(n) * p.ldo + m;
              if (p.out_bf16) reinterpret_cast<__nv_bfloat16*>(p.out)[o] = __float2bfloat16(val);
              else reinterpret_cast<float*>(p.out)[o] = val;
            }
          }
        }
        epilogue_colsum(p, colsum, m, m_ok);  // (the arrival counter is monotonic: no reset needed)
      }
    } else {
      // EPI_ROWMAJOR_PUSH: the gradient push. Thread m owns row m of the dW tile; pushing row runs per thread
      // makes every 16-byte store of a warp hit a different row (32 partial lines per instruction, and 16-byte
      // packets on NVLink). The staged variant reads the shared-memory tile so that each warp instruction writes
      // whole 256-byte row segments: lanes 0..15 one row, lanes 16..31 the next.
      const ResolvedPush r = resolve_push(p.push);
      float* gbase = r.base + p.push_offset;
      const bool vec_ok = ((p.ldo & 3) == 0) && ((p.push_offset & 3) == 0) && ((p.N & 3) == 0);
      if (p.push_staged) {
        // the accumulator tile is already row-major in shared memory (row stride ldc)
        const float* sC = sacc + static_cast<size_t>(q * 32) * ldc;   // this warp's 32 rows
        __syncwarp();
        const int vec_per_row = bn >> 2;
        const float sc = p.push.scale;
        for (int idx = lane; idx < 32 * vec_per_row; idx += 32) {
          const int rl = idx / vec_per_row;
          const int c4 = (idx - rl * vec_per_row) << 2;
          const int mm = m0 + q * 32 + rl;
          const int n = n0 + c4;
          if (mm >= p.M || n >= p.N) continue;
          const float4 t = *reinterpret_cast<const float4*>(sC + rl * ldc + c4);
          float* dstp = gbase + static_cast<size_t>(mm) * p.ldo + n;
          if (vec_ok) {
            if (p.push.mode == PUSH_ATOMIC) red_add_sys_v4f32(dstp, sc * t.x, sc * t.y, sc * t.z, sc * t.w);
            else st_global_v4f32(dstp, t.x, t.y, t.z, t.w);
          } else {
            const float tv[4] = {t.x, t.y, t.z, t.w};
  #pragma unroll
            for (int j = 0; j < 4; ++j) {
              if (n + j < p.N) {
                if (p.push.mode == PUSH_ATOMIC) red_add_sys_f32(dstp + j, sc * tv[j]);
                else dstp[j] = tv[j];
              }
            }
          }
        }
      } else {
        // direct variant: lane m pushes its own row run (16-byte stores, one row per lane)
        float* row = gbase + static_cast<size_t>(m) * p.ldo + n0;
        const float sc = p.push.scale;
        for (int c0 = 0; c0 < bn; c0 += 16) {
          float v[16];
          acc_ld16(arow, c0, v);
          if (!m_ok) continue;
          const int n = n0 + c0;
          if (vec_ok && n + 16 <= p.N) {
#pragma unroll
            for (int j = 0; j < 16; j += 4) {
              if (p.push.mode == PUSH_ATOMIC)
                red_add_sys_v4f32(row + c0 + j, sc * v[j], sc * v[j + 1], sc * v[j + 2], sc * v[j + 3]);
              else
                st_global_v4f32(row + c0 + j, v[j], v[j + 1], v[j + 2], v[j + 3]);
            }
          } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              if (n + j < p.N) {
                if (p.push.mode == PUSH_ATOMIC) red_add_sys_f32(row + c0 + j, sc * v[j]);
                else row[c0 + j] = v[j];
              }
            }
          }
        }
      }
      if (p.push.mode == PUSH_MAILBOX) {
        // Publish the tile: the CTA barrier orders every lane's P2P stores before the single st.release.sys
        // (release is cumulative over what the barrier made visible to the releasing thread), so only one
        // thread pays for a system-scope fence instead of all 128 (measured: 14 us -> 4 us for this kernel).
        named_bar_sync(1, 128);
        if (threadIdx.x == 64)
          st_release_scoped_u32(r.flags + p.push_item_base + blockIdx.x * gridDim.y + blockIdx.y, r.seq,
                                p.push.gpu_scope);
      }
    }
  } else if (cluster_mode) {
    cluster_barrier_wait_acquire();   // second consumer warpgroup: end of its role
  }

  if (cluster_mode) {
    // every thread of every CTA of the cluster: partial columns have landed after this barrier
    cluster_barrier_arrive_release();
    cluster_barrier_wait_acquire();
    const int nsplit = gridDim.z;
    const uint32_t crank = cluster_ctarank();
    const int cw = (bn + nsplit - 1) / nsplit;
    float colsum = 0.f;
    if (warp < 4) {
      // ---- phase 2: sum the nsplit contributions of my columns and run the real epilogue on them ----
      const int q = warp & 3;
      const int mrow = q * 32 + lane;
      const int m = m0 + mrow;
      const bool m_ok = m < p.M;
      const float bias = (p.bias != nullptr && m_ok) ? p.bias[m] : 0.f;
      for (int cc = 0; cc < cw; ++cc) {
        const int c = static_cast<int>(crank) * cw + cc;
        if (c >= bn) break;
        float acc = 0.f;
        for (int src = 0; src < nsplit; ++src) acc += red[(src * cw + cc) * kTileM + mrow];
        const int n = n0 + c;
        if (n < p.N && m_ok) {
          float val = acc + bias;
          if (p.mask != nullptr) {
            const float a = p.mask_bf16
                                ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(
                                      p.mask)[static_cast<size_t>(n) * p.ldmask + m])
                                : reinterpret_cast<const float*>(p.mask)[static_cast<size_t>(n) * p.ldmask + m];
            val = act_backward(p.act, a, val);   // dX: act'(y) from the layer's output
          } else {
            val = act_forward(p.act, val);
          }
          colsum += val;
          const size_t o = static_cast<size_t>(n) * p.ldo + m;
          if (p.out_bf16) reinterpret_cast<__nv_bfloat16*>(p.out)[o] = __float2bfloat16(val);
          else reinterpret_cast<float*>(p.out)[o] = val;
        }
      }
      if (p.has_colsum) {
        // bias-gradient partial sums of my columns -> CTA 0 of the cluster
        const uint32_t ca = mapa_shared_cluster(smem_u32(csum) + (crank * kTileM + mrow) * 4u, 0);
        st_shared_cluster_f32(ca, colsum);
      }
    }
    if (p.has_colsum) {
      cluster_barrier_arrive_release();
      cluster_barrier_wait_acquire();
      if (crank == 0 && warp < 4) {
        const int mrow = warp * 32 + lane;
        float tot = 0.f;
        for (int src = 0; src < nsplit; ++src) tot += csum[src * kTileM + mrow];
        epilogue_colsum(p, tot, m0 + mrow, m0 + mrow < p.M);
      }
    }
  }

  if (dbg && threadIdx.x == 64) dbg[7] = clock64();
  __syncthreads();
  if (dbg && threadIdx.x == 0) dbg[8] = clock64();
  if (p.debug_ts != nullptr && threadIdx.x == 0 && cta_lin < 120) p.debug_ts[17 + 2 * cta_lin] = static_cast<long long>(globaltimer_ns());
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
size_t gemm_smem_bytes(int bn, int stages, int cluster) {
  size_t ring = static_cast<size_t>(stages) * (kABytes + bn * 128);
  const size_t stage_tile = static_cast<size_t>(kTileM) * (bn + 4) * sizeof(float);  // push-epilogue transpose tile
  if (ring < stage_tile) ring = (stage_tile + 1023) & ~size_t(1023);
  size_t total = ring + 256 /* barriers */ + 1024 /* alignment slack */;
  if (cluster) total += static_cast<size_t>(bn + 8) * kTileM * sizeof(float) + 8 * kTileM * sizeof(float);  // red + csum
  return total;
}

// MN-major B operands: the K-major copy of one stage's B tile (+ its 1024-byte alignment)
size_t gemm_bt_bytes(int bn) { return static_cast<size_t>(bn) * 128 + 1024; }

constexpr int kMaxDynSmem = 226 * 1024;  // 227 KB per-block limit minus the kernel's static shared memory

using GemmKernel = void (*)(const CUtensorMap, const CUtensorMap, const GemmParams);

template <typename T>
static GemmKernel gemm_kernel_of(bool a_mn, bool b_mn) {
  if (!a_mn && !b_mn) return gemm_wgmma_kernel<T, false, false>;
  if (a_mn && b_mn) return gemm_wgmma_kernel<T, true, true>;
  if (a_mn) return gemm_wgmma_kernel<T, true, false>;
  return gemm_wgmma_kernel<T, false, true>;
}

// The instantiation for operands of `dtype` (0 = fp32 (tf32 MMA), 1 = bf16), A and B MN-major or K-major.
static GemmKernel gemm_kernel(int dtype, bool a_mn, bool b_mn) {
  return dtype == 0 ? gemm_kernel_of<float>(a_mn, b_mn) : gemm_kernel_of<__nv_bfloat16>(a_mn, b_mn);
}

// Opt every instantiation into the full 227 KB of dynamic shared memory once per device, outside of any
// stream capture (launches themselves then carry no attribute calls and are graph-capturable), and force-load it.
cudaError_t prepare_gemm_kernels() {
  static const bool kLayouts[4][2] = {{false, false}, {true, true}, {true, false}, {false, true}};   // (A, B) MN-major
  for (const int dtype : {0, 1})
    for (const auto& mn : kLayouts) {
      const GemmKernel k = gemm_kernel(dtype, mn[0], mn[1]);
      cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem);
      cudaFuncAttributes a;
      if (e == cudaSuccess) e = cudaFuncGetAttributes(&a, k);
      if (e != cudaSuccess) return e;
    }
  return cudaSuccess;
}

static cudaError_t launch_one(GemmKernel kern, bool b_mn, const CUtensorMap& tmA, const CUtensorMap& tmB,
                              const GemmParams& p, dim3 grid, cudaStream_t stream) {
  const bool cluster = p.splitk_cluster != 0 && grid.z > 1;
  const size_t smem = gemm_smem_bytes(p.bn, p.stages, cluster ? 1 : 0) + (b_mn ? gemm_bt_bytes(p.bn) : 0);
  if (smem > static_cast<size_t>(kMaxDynSmem) || p.bn < 16 || p.bn > 16 * kMaxNB || (p.bn & 15)) return cudaErrorInvalidValue;
  if (!cluster && !p.pdl) {
    kern<<<grid, kGemmThreads, smem, stream>>>(tmA, tmB, p);
    return cudaGetLastError();
  }
  if (cluster && (grid.z > 8 || (2 * p.stages + 1) * sizeof(uint64_t) + 16 > 256)) return cudaErrorInvalidValue;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  unsigned na = 0;
  if (cluster) {
    attr[na].id = cudaLaunchAttributeClusterDimension;   // the K-splits of one output tile form a cluster
    attr[na].val.clusterDim.x = 1;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = grid.z;
    ++na;
  }
  if (p.pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kern, tmA, tmB, p);
}

// dtype: 0 = fp32 (tf32 MMA), 1 = bf16
cudaError_t launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int dtype, bool a_mn,
                        bool b_mn, int splits, cudaStream_t stream) {
  if (!act_valid(p.act)) return cudaErrorInvalidValue;
  dim3 grid((p.M + kTileM - 1) / kTileM, (p.N + p.bn - 1) / p.bn, splits);
  return launch_one(gemm_kernel(dtype, a_mn, b_mn), b_mn, tmA, tmB, p, grid, stream);
}

}  // namespace dm
