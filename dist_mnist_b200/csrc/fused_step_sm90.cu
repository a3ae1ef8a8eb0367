// Fused worker step for sm_90a: whole training steps of the 784-H-10 MLP inside ONE persistent kernel.
//
// The reference's hot loop is `sess.run([train_op, loss, global_step], feed_dict)`
// (distributed_server-basic.py:110-113 of the reference): fetch the variables from the ps (DS:41-47 placed by
// DS:88-89), forward (DS:49-51), loss (DS:52-53), backward + send the gradients to the ps (DS:103). Here that whole
// iteration is one pass of one 8-CTA thread-block cluster, repeated for as many steps as the launch was given —
// no kernel boundary, no host round trip and no global-memory hand-off between the phases of a step:
//
//   pull + forward   CTA r of the cluster owns input features [32 kb_r, 32 ke_r): warp 0 TMA-loads that K-slice of
//                    W *straight out of the owning ps shard's HBM* (NVLink peer mapping) and of x into 128B-swizzled
//                    shared memory (warp 4); warps 0..3 (one warpgroup) issue wgmma (tf32, fp32 accumulators in
//                    registers): a split-K partial of pre^T [128 hidden x 32 batch].
//   reduce-scatter   the partial accumulators are scattered from registers through distributed shared memory
//                    (st.shared::cluster.v2): CTA r ends up with batch rows 4r..4r+3 for all hidden
//                    units, adds the bias (peer load) and applies the ReLU.
//   head             logits / softmax / loss (book or xent) / accuracy / dlogits for those 4 rows, then
//                    dpre = (dlogits . W_last) * relu' and the partial dW_last / db_hidden / db_last sums.
//   all-gather       dpre^T is the A operand of the dW GEMM: every CTA writes its 16-byte chunk of each 128-byte
//                    row (K-major, SWIZZLE_128B) into the shared memory of all 8 CTAs; the small-gradient partials
//                    are reduce-scattered the same way (16 hidden units per CTA).
//   dW + push        CTA r computes dW[:, its K-slice]^T = x^T (slice x 32) . dpre (32 x 128) with wgmma (x^T is the
//                    register operand, read from a second copy of the x tile; dpre^T is the shared-memory operand)
//                    and its epilogue *is the gradient push*: registers -> swizzled staging tile in shared memory -> TMA store (cp.async.bulk.tensor, whole 128-byte
//                    lines over NVLink) into this worker's mailbox slot in the ps shard's HBM — or a TMA *reduce-add*
//                    into the master copy for async SGD (push == apply) — then one cumulative st.release flag per tile.
//   publish          everything that waits for a round trip (store completion, the release of the tile flag, the small
//                    variables' flags, the 16-byte step result into pinned host memory) is done by warp 4 *after* the
//                    step's last cluster barrier, i.e. while the other warps already run the next step's forward.
//   small variables  bias / W_last / b_last are pulled with cp.async.bulk on the same mbarrier as the W tiles: no
//                    synchronous peer load is ever on the critical path.
//
// Steps are claimed dynamically (atomic counter), so `lanes` = gridDim.y clusters of one launch work on different
// steps concurrently and a cluster that is scheduled late simply takes fewer steps. Within a cluster the next
// step's W / x loads are issued as soon as the forward MMAs of the current step have drained the buffers
// (`strict` = 0), i.e. the pull of step s+1 overlaps the backward half of step s.
//
// Batches of 33..256 rows (fused_step_kernel<kFsMaxTiles>): a step is T = ceil(B / 32) row tiles of 32 rows. W and the
// small variables are pulled once per step and stay resident for all T tiles (the next step's pull is issued after
// barrier #1 of the last tile); each tile loads its own x rows (row0 + 32 t, same tensor map) and runs the phases above
// with barriers #1 and #2, and #3 closes the step. The forward's x of tile t + 1 goes into Xk after barrier #1 of tile
// t, the dW GEMM's copy into Xmn once tile t's dW MMAs are done (bar_xmn_empty). The dW staging tile and the small
// gradients / loss / correct count add up over the tiles in shared memory and are pushed once per step, the loss
// normalised by the whole batch. B <= 32 runs fused_step_kernel<1>, whose code is that of the one-tile kernel.
//
// SURVEY K1-K6, K12, X3-X5 for the flagship model; deeper / wider / bf16 models use the per-layer kernels
// (gemm_sm90.cu, head_sm90.cu) chained in a CUDA graph.
#include "common.cuh"
#include "activation.cuh"
#include "fused.h"
#include "grad_clip.cuh"
#include "loss.cuh"

namespace dm {

constexpr int kFsThreads = 160;        // warps 0..3: wgmma + head warpgroup; warp 4: TMA producer + publisher
constexpr int kFsProducerWarp = 4;
constexpr int kFsRows = 4;             // batch rows per CTA (32 / kFusedCluster)
constexpr int kFsMaxC = 16;            // classes, padded
constexpr int kFsPart = 12;            // floats per (source CTA, hidden unit): dW_last[0..10], db_hidden
constexpr int kFsWlStride = 132;       // smem row stride of W_last: 16 class rows land in distinct bank groups
constexpr uint32_t kFsWChunk = 128 * 128;   // one k-chunk of W: 128 rows x 128 B
constexpr uint32_t kFsXChunk = 32 * 128;    // one k-chunk of x: 32 rows x 128 B

// shared-memory carve-up (byte offsets from the 1024-aligned base; identical in every CTA of the cluster)
constexpr uint32_t kOffW = 0;                                        // 4 x 16 KB   W k-chunks (A of the forward)
constexpr uint32_t kOffXk = kOffW + kFusedMaxChunks * kFsWChunk;     // 4 x 4 KB    x k-chunks (B of the forward)
constexpr uint32_t kOffXmn = kOffXk + kFusedMaxChunks * kFsXChunk;   // 4 x 4 KB    x k-chunks (A of the dW GEMM)
constexpr uint32_t kOffA = kOffXmn + kFusedMaxChunks * kFsXChunk;    // 16 KB       dpre^T     (B of the dW GEMM)
constexpr uint32_t kOffRed = kOffA + 128 * 128;                      // [8][128][4] reduce-scatter landing zone
constexpr uint32_t kOffSg = kOffRed + 8 * 128 * 4 * 4;               // [8][16][12] small-gradient landing zone
constexpr uint32_t kOffVal = kOffSg + 8 * 16 * kFsPart * 4;          // [4][128]    activations of my rows
constexpr uint32_t kOffWl = kOffVal + kFsRows * 128 * 4;             // [16][132]   W_last
constexpr uint32_t kOffDl = kOffWl + kFsMaxC * kFsWlStride * 4;      // [4][16]     dlogits of my rows
constexpr uint32_t kOffDbl = kOffDl + kFsRows * kFsMaxC * 4;         // [8][16]     db_last partials (CTA 0)
constexpr uint32_t kOffScal = kOffDbl + 8 * kFsMaxC * 4;             // [8][2]      loss / correct partials (CTA 0)
constexpr uint32_t kOffRedw = kOffScal + 8 * 2 * 4;                  // [8]         warp partials
constexpr uint32_t kOffCtl = kOffRedw + 8 * 4;                       // next-step words [2]
constexpr uint32_t kOffBar = kOffCtl + 32;                           // mbarriers (2; the multi-tile kernel: 4)
constexpr uint32_t kOffRawWl = (kOffBar + 64 + 127) & ~127u;         // W_last as it sits in the arena [C][H] (bulk copy)
constexpr uint32_t kOffRawB = kOffRawWl + (kFsPart - 1) * 128 * 4;   // hidden bias [H]
constexpr uint32_t kOffRawBl = kOffRawB + 128 * 4;                   // b_last [C]
constexpr uint32_t kOffStage = (kOffRawBl + 64 + 1023) & ~1023u;     // 4 x 16 KB  dW tile staging for the TMA store
constexpr uint32_t kFsSmemUsed = kOffStage + kFusedMaxChunks * kFsWChunk;
constexpr uint32_t kFsSmemBytes = kFsSmemUsed + 1024;                // + alignment slack
static_assert(kOffA % 1024 == 0 && kOffXk % 1024 == 0 && kOffXmn % 1024 == 0, "swizzled tiles need 1024-byte alignment");
static_assert(kOffBar % 8 == 0 && kOffRed % 16 == 0 && kOffSg % 16 == 0 && kOffRawWl % 16 == 0 && kOffRawB % 16 == 0 &&
              kOffRawBl % 16 == 0 && kOffStage % 1024 == 0, "alignment");
static_assert(kFsSmemBytes <= 227 * 1024, "shared memory budget");
// Batches of more than 32 rows run as several 32-row tiles per step (the multi-tile instantiation). Its running sums
// of the small gradients over the tiles of a step live behind the one-tile layout, which is left exactly as it is.
constexpr int kFsMaxTiles = 8;                                       // 256 rows
constexpr uint32_t kOffAcc = kFsSmemUsed;                            // [12][128]   dW_last / db_hidden of unit et
constexpr uint32_t kOffAccDbl = kOffAcc + kFsPart * 128 * 4;         // [16]        db_last of my rows
constexpr uint32_t kOffAccScal = kOffAccDbl + kFsMaxC * 4;           // [2]         loss / correct of my rows
constexpr uint32_t kFsMultiSmemBytes = kOffAccScal + 2 * 4 + 1024;
static_assert(kFsMultiSmemBytes <= 227 * 1024, "shared memory budget (multi-tile)");
template <int kMaxTiles>
constexpr uint32_t fs_smem_bytes() { return kMaxTiles == 1 ? kFsSmemBytes : kFsMultiSmemBytes; }
// Gradient clipping (fused_step_kernel<*, true>): the per-variable sums of squares of a step sit in the alignment gap
// before the staging tile, so that the clip instantiations have the shared-memory footprint (and the residency beside
// the ps serve kernel) of the unclipped ones.
constexpr int kFsClipVars = 4;                                        // hid_w, hid_b, sm_w, sm_b
constexpr uint32_t kOffClipWarp = (kOffRawBl + 64 + 15) & ~15u;       // [4][4]      warp partials of this CTA
constexpr uint32_t kOffClipPart = kOffClipWarp + 4 * kFsClipVars * 4; // [8][4]      CTA partials (DSMEM all-gather)
static_assert(kOffClipPart + kFusedCluster * kFsClipVars * 4 <= kOffStage, "the clip partials fit before the staging tile");
// L2 regularization (fused_step_kernel<*, *, true>): the sums of w*w of a step sit in the same gap, behind the clip
// partials: per warp of this CTA {hid_w, small variables}, and the CTA partials that CTA 0's publisher adds up.
constexpr uint32_t kOffL2Warp = kOffClipPart + kFusedCluster * kFsClipVars * 4;   // [4][2]  warp partials of this CTA
constexpr uint32_t kOffL2Part = kOffL2Warp + 4 * 2 * 4;                           // [8]     CTA partials (CTA 0)
static_assert(kOffL2Part + kFusedCluster * 4 <= kOffStage, "the L2 partials fit before the staging tile");

// pre^T block [64 x 32] += W [64 x k8] . x [32 x k8]^T, both operands from shared memory (tf32)
__device__ __forceinline__ void fs_mma_m64n32(float (&d)[4][4], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]),
        "+f"(d[1][3]), "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[3][0]), "+f"(d[3][1]),
        "+f"(d[3][2]), "+f"(d[3][3])
      : "l"(adesc), "l"(bdesc), "r"(acc));
}
// dW^T block [64 x 128] += x^T [64 x k8] (registers) . dpre [k8 x 128] (shared memory, dpre^T K-major)
__device__ __forceinline__ void fs_mma_m64n128(float (&d)[16][4], const uint32_t (&a)[4], uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]),
        "+f"(d[1][3]), "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[3][0]), "+f"(d[3][1]),
        "+f"(d[3][2]), "+f"(d[3][3]), "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]), "+f"(d[5][0]),
        "+f"(d[5][1]), "+f"(d[5][2]), "+f"(d[5][3]), "+f"(d[6][0]), "+f"(d[6][1]), "+f"(d[6][2]), "+f"(d[6][3]),
        "+f"(d[7][0]), "+f"(d[7][1]), "+f"(d[7][2]), "+f"(d[7][3]), "+f"(d[8][0]), "+f"(d[8][1]), "+f"(d[8][2]),
        "+f"(d[8][3]), "+f"(d[9][0]), "+f"(d[9][1]), "+f"(d[9][2]), "+f"(d[9][3]), "+f"(d[10][0]), "+f"(d[10][1]),
        "+f"(d[10][2]), "+f"(d[10][3]), "+f"(d[11][0]), "+f"(d[11][1]), "+f"(d[11][2]), "+f"(d[11][3]),
        "+f"(d[12][0]), "+f"(d[12][1]), "+f"(d[12][2]), "+f"(d[12][3]), "+f"(d[13][0]), "+f"(d[13][1]),
        "+f"(d[13][2]), "+f"(d[13][3]), "+f"(d[14][0]), "+f"(d[14][1]), "+f"(d[14][2]), "+f"(d[14][3]),
        "+f"(d[15][0]), "+f"(d[15][1]), "+f"(d[15][2]), "+f"(d[15][3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc));
}

__device__ __forceinline__ void cluster_sync_all() {
  cluster_barrier_arrive_release();
  cluster_barrier_wait_acquire();
}

struct FsPush {
  float* base;
  uint32_t* flags;
};
__device__ __forceinline__ FsPush fs_resolve(const PushTarget& t, uint32_t seq) {
  FsPush r{t.base, t.flags};
  if (t.mode == PUSH_MAILBOX) {
    const uint32_t slot = seq % t.nslots;
    r.base = t.base + static_cast<uint64_t>(slot) * t.slot_stride;
    r.flags = t.flags + static_cast<uint64_t>(slot) * t.flag_slot_stride;
  }
  return r;
}
__device__ __forceinline__ void fs_push_value(const PushTarget& t, float* dst, float v) {
  if (t.mode == PUSH_ATOMIC) red_add_sys_f32(dst, t.scale * v);
  else *dst = v;
}

__device__ __forceinline__ uint64_t fs_row0(const FusedParams& p, uint32_t step) {
  return (p.row_start + static_cast<uint64_t>(step) * p.row_stride) % p.row_wrap;
}

// spin until every shard has acknowledged push `need` of this worker (acks are written into local memory by the ps)
__device__ __forceinline__ void fs_wait_acks(const FusedParams& p, uint32_t need, const char* who) {
  const uint64_t t0 = globaltimer_ns();
  for (int k = 0; k < p.n_shards; ++k) {
    const volatile uint32_t* ib = reinterpret_cast<const volatile uint32_t*>(p.shard[k].inbox);
    if (ib == nullptr) continue;
    while (static_cast<int32_t>(ib[0] - need) < 0) {
      if (globaltimer_ns() - t0 > DM_SPIN_TIMEOUT_NS) {
        printf("[dm] fused step (%s): ps shard %d ack timeout (need=%u ack=%u)\n", who, k, need, ib[0]);
        __trap();
      }
    }
  }
}

// kMaxTiles == 1: B <= 32, one row tile per step. kMaxTiles > 1: T = ceil(B / 32) row tiles per step (see the header).
// kClip: the pushed gradient is clipped first (FusedParams::clip_kind, TF1's clip_by_global_norm / clip_by_norm per
// variable / clip_by_value). In the last row tile every CTA sums the squares of the gradient elements it pushes, per
// variable: hid_w over its staging tile, sm_w / hid_b over its 16 hidden units, sm_b on CTA 0. The 4 partials go to
// every CTA through DSMEM, one more cluster barrier (the norm barrier) follows, and every CTA adds the 8 x 4 partials
// in the same order, so all agree on the scale bit for bit. The staging tile is then scaled in place before warp 4
// stores it, and the small gradients are pushed after the norm barrier (still before barrier #3). CLIP_VALUE clamps
// element-wise and needs neither the sums nor the barrier.
// kL2: L2 weight regularization (FusedParams::l2_scale, l2_biases), before the clip: the pushed gradient of a
// regularized variable is fl(g + fl(S * w)), with w the copy this step pulled. W is read out of its forward tile and the
// small variables out of their landing zones, so warp 4 issues the next step's pull only once the last row tile has
// handed the staging tile over (named barrier 2) instead of after its barrier #1. Every CTA sums w*w over what it
// owns (its W k-slice, W_last / b of its 16 hidden units, b_last on CTA 0) into one partial on CTA 0, whose publisher
// adds the 8 partials in a fixed order and reports loss + S * sum / 2.
// kGeneral: the general head. The hidden layer's activation is FusedParams::act (activation.cuh) instead of the ReLU:
// f where the hidden values hv are formed, f'(hv) where dpre is. Units >= H stay 0; padding rows (>= B) hold f(bias),
// which nothing reads: their dlogits are 0, so they add 0 to dpre and to every sum, and the loss and correct count mask
// them. The loss is any LossKind (loss.cuh) and the labels the head reads are smoothed by FusedParams::label_smoothing;
// the correct count compares with the raw labels. Without it the head runs LOSS_BOOK or an unsmoothed LOSS_XENT.
template <int kMaxTiles, bool kClip, bool kL2, bool kGeneral>
__global__ void __launch_bounds__(kFsThreads, 1)
fused_step_kernel(const __grid_constant__ FusedMaps maps, const __grid_constant__ FusedParams p) {
  constexpr bool kMulti = kMaxTiles > 1;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sbase = smem_u32(smem);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();
  const FusedSlice sl = p.slice[rank];
  const int nkc = sl.kc_count;

  uint64_t* bar_w = reinterpret_cast<uint64_t*>(smem + kOffBar);   // W + x (K-major) of a step have landed
  uint64_t* bar_xmn = bar_w + 1;                                    // the dW GEMM's copy of x of a tile has landed
  uint64_t* bar_xk = bar_w + 2;          // multi-tile: the forward's x of tile t >= 1 has landed (W stays resident)
  uint64_t* bar_xmn_empty = bar_w + 3;   // multi-tile: the dW MMAs of tile t < T - 1 are done with Xmn
  volatile uint32_t* ctl_next = reinterpret_cast<volatile uint32_t*>(smem + kOffCtl);

  if (p.debug_ts != nullptr && blockIdx.y == 0 && rank == 0 && threadIdx.x == 0)
    p.debug_ts[60] = static_cast<long long>(globaltimer_ns());                                 // kernel entry
  if (p.lane_rec != nullptr && threadIdx.x == 0) {
    unsigned long long* rec = p.lane_rec + blockIdx.y * kLaneRecWords;
    rec[rank] = sm_id();
    if (rank == 0) rec[11] = globaltimer_ns();
  }
  if (warp == kFsProducerWarp && lane == 0) {
    prefetch_tensormap(&maps.w[rank]);
    prefetch_tensormap(&maps.xk);
    mbar_init(bar_w, 1);
    mbar_init(bar_xmn, 1);
    if constexpr (kMulti) {
      mbar_init(bar_xk, 1);
      mbar_init(bar_xmn_empty, 128);
    }
    fence_mbar_init();
  }
  __syncthreads();

  // Distributed shared memory of a peer CTA may only be touched once that CTA is known to be running.
  cluster_sync_all();
  // ---- first step of this cluster: claimed by CTA 0, broadcast to everybody ----
  auto claim = [&]() -> uint32_t {
    if (*reinterpret_cast<volatile uint32_t*>(p.stop_word) != 0u) return kFusedNoStep;
    const uint32_t g = atomicAdd(p.step_counter, 1u);
    if (g >= p.n_steps) return kFusedNoStep;
    if (p.lane_rec != nullptr) {
      unsigned long long* rec = p.lane_rec + blockIdx.y * kLaneRecWords;
      if (rec[8]++ == 0) rec[9] = globaltimer_ns();
    }
    return g;
  };
  auto broadcast_next = [&](uint32_t which, uint32_t g) {
#pragma unroll
    for (uint32_t d = 0; d < kFusedCluster; ++d)
      st_shared_cluster_u32(mapa_shared_cluster(sbase + kOffCtl + which * 4u, d), g);
  };
  const bool is_claimer = rank == 0 && threadIdx.x == 0;    // head thread et == 0 of CTA 0
  if (is_claimer) broadcast_next(0, claim());
  cluster_sync_all();
  uint32_t cur = ctl_next[0];

  const bool dbg = p.debug_ts != nullptr && blockIdx.y == 0 && rank == 0;
  if (dbg && threadIdx.x == 0) p.debug_ts[61] = static_cast<long long>(globaltimer_ns());   // first step claimed
  const bool mailbox = p.shard[0].push.mode == PUSH_MAILBOX;
  const int H = p.H, C = p.C, B = p.B;
  const int T = kMulti ? (B + 31) >> 5 : 1;   // row tiles per step
  const uint32_t wl_bytes = (static_cast<uint32_t>(C * H) * 4u + 15u) & ~15u;   // bulk copies move 16-byte multiples
  const uint32_t b_bytes = (static_cast<uint32_t>(H) * 4u + 15u) & ~15u;        // (the arena pads every variable)
  const uint32_t bl_bytes = (static_cast<uint32_t>(C) * 4u + 15u) & ~15u;
  constexpr int kTs = 16;   // debug stamps per step

  if (warp == kFsProducerWarp) {
    // =========================== TMA producer + publisher ===========================
    auto issue_wx = [&](uint32_t step) {
      const int row0 = static_cast<int>(fs_row0(p, step));
      mbar_arrive_expect_tx(bar_w, static_cast<uint32_t>(nkc) * (kFsWChunk + kFsXChunk) + wl_bytes + b_bytes + bl_bytes);
      for (int i = 0; i < nkc; ++i) {
        const int k0 = (sl.kc_begin + i) * 32;
        tma_load_2d(smem + kOffW + i * kFsWChunk, &maps.w[rank], bar_w, k0, 0);      // peer HBM -> smem (the pull)
        tma_load_2d(smem + kOffXk + i * kFsXChunk, &maps.xk, bar_w, k0, row0);
      }
      // the small variables ride on the same barrier: no synchronous peer load anywhere in the step
      bulk_load_1d(smem + kOffRawWl, p.w_last, wl_bytes, bar_w);
      bulk_load_1d(smem + kOffRawB, p.bias_h, b_bytes, bar_w);
      bulk_load_1d(smem + kOffRawBl, p.b_last, bl_bytes, bar_w);
    };
    // x rows of row tile t of a step into one of the two x buffers (Xmn: the dW GEMM's copy; Xk: the forward's copy
    // of tiles t >= 1 — tile 0's rides on bar_w with W)
    auto issue_x = [&](uint32_t step, int t, uint32_t off, uint64_t* bar) {
      if (nkc == 0) { mbar_arrive(bar); return; }
      const int row0 = static_cast<int>(fs_row0(p, step)) + 32 * t;
      mbar_arrive_expect_tx(bar, static_cast<uint32_t>(nkc) * kFsXChunk);
      for (int i = 0; i < nkc; ++i)
        tma_load_2d(smem + off + i * kFsXChunk, &maps.xk, bar, (sl.kc_begin + i) * 32, row0);
    };
    auto issue_xmn = [&](uint32_t step, int t) { issue_x(step, t, kOffXmn, bar_xmn); };
    if (lane == 0 && cur != kFusedNoStep) {
      issue_wx(cur);
      issue_xmn(cur, 0);
    }
    __syncwarp();
    const float* scal = reinterpret_cast<const float*>(smem + kOffScal);
    // ---- publishing a finished step (lane 0): everything that costs memory round trips — an NVLink round trip when the
    // ps is remote — and that nothing inside the step depends on
    struct Pending { uint32_t step, seq; float loss, corr; uint32_t ts_slot; };
    Pending pend{0u, 0u, 0.f, 0.f, 0u};
    auto publish = [&](const Pending& d) {
      const PushTarget& tw = p.shard[sl.shard].push;
      const bool tile = nkc > 0;
      if (tile) bulk_wait_group0();                       // my tile has reached the ps shard's memory
      if (dbg && d.ts_slot < 4) p.debug_ts[d.ts_slot * kTs + 10] = clock64();
      if (mailbox && (tile || rank == 0)) {
        // one cumulative fence: my TMA-stored tile (async proxy) and — through cluster barrier #3 — every CTA's
        // small-gradient stores are ordered before the flags below
        fence_proxy_async();
        fence_acq_rel_scoped(tw.gpu_scope);
        if (tile) st_relaxed_sys_u32(fs_resolve(tw, d.seq).flags + sl.flag_index, d.seq);
        if (rank == 0) {
          st_relaxed_sys_u32(fs_resolve(p.shard[p.shard_wl].push, d.seq).flags + p.flag_wl, d.seq);
          st_relaxed_sys_u32(fs_resolve(p.shard[p.shard_bh].push, d.seq).flags + p.flag_bh, d.seq);
          st_relaxed_sys_u32(fs_resolve(p.shard[p.shard_bl].push, d.seq).flags + p.flag_bl, d.seq);
        }
      }
      if (rank == 0) {
        uint32_t gstep = d.seq;
        if (mailbox) {
          const volatile unsigned long long* ib = reinterpret_cast<const volatile unsigned long long*>(p.shard[0].inbox);
          if (ib != nullptr) {
            // {acked push, global_step} in one 8-byte load. global_step as of our last acknowledged push + our own
            // pushes since then: exact with one worker, a lower bound under concurrency (the reference's fetched
            // value is equally unordered w.r.t. peers)
            const unsigned long long v = *ib;
            gstep = static_cast<uint32_t>(v >> 32) + (d.seq - static_cast<uint32_t>(v));
          }
        } else if (p.shard[0].push.mode == PUSH_ATOMIC && p.ps_global_step != nullptr) {
          gstep = atom_add_sys_u32(p.ps_global_step, 1u) + 1u;   // async SGD: this push *is* global step gstep
        }
        StepResult res;
        res.loss = d.loss;
        res.global_step = gstep;
        res.correct = static_cast<uint32_t>(d.corr + 0.5f);
        res.seq = d.seq;
        p.results[d.step] = res;                              // pinned host memory: a 16-byte posted write
        atomicAdd(p.seq_word, 1u);
        if (p.stop_at != 0u && gstep >= p.stop_at) *reinterpret_cast<volatile uint32_t*>(p.stop_word) = 1u;
        if (dbg && d.ts_slot < 4) p.debug_ts[d.ts_slot * kTs + 11] = clock64();
      }
    };
    bool arrived1 = false;   // barrier #1 of the coming step already arrived at (early, see below)
    bool deferred = false;   // `pend` holds a finished step whose publishing was deferred into this step's head phase
    for (uint32_t jl = 0; cur != kFusedNoStep; ++jl) {
      const uint32_t seq = p.seq_base + cur + 1u;
      uint32_t nxt = kFusedNoStep;
      // Row tiles: barriers #1 and #2 are passed once per tile (cluster barriers count every thread), #3 once per step.
      for (int t = 0; t < T; ++t) {
        const bool last = t == T - 1;
        if (t > 0 || !arrived1) cluster_barrier_arrive_release();
        cluster_barrier_wait_acquire();                     // #1: the forward MMAs have drained the W / x tiles
        if (t == 0) nxt = ctl_next[(jl + 1) & 1];
        if (!last) {
          if (lane == 0) issue_x(cur, t + 1, kOffXk, bar_xk);   // x of the next tile (W stays for the whole step)
        } else if (!kL2 && lane == 0 && !p.strict && nxt != kFusedNoStep) {
          issue_wx(nxt);                                    // W / x buffers are free: pull ahead
        }
        __syncwarp();
        if (t == 0 && deferred) {
          // EARLY ARRIVAL at barrier #2, then the previous step is published while the other warps run this step's
          // head: nothing they do before their staging writes (which come after barrier #2) involves this warp.
          cluster_barrier_arrive_release();                 // #2 (arrive)
          if (lane == 0) publish(pend);
          __syncwarp();
          cluster_barrier_wait_acquire();                   // #2 (wait)
          deferred = false;
        } else {
          cluster_sync_all();                               // #2
        }
        if (!last) {
          // the next tile's copy of x for the dW GEMM, once this tile's dW MMAs have read Xmn
          if (lane == 0) {
            if (nkc > 0) mbar_wait(bar_xmn_empty, (jl * static_cast<uint32_t>(T - 1) + static_cast<uint32_t>(t)) & 1u);
            issue_xmn(cur, t + 1);
          }
          __syncwarp();
        }
      }
      if constexpr (kClip) {
        if (p.clip_kind != CLIP_VALUE) cluster_sync_all();   // the norm barrier (see the head warpgroup)
      }
      // ---- the gradient push: the epilogue warps have staged the dW tile (swizzled, fence.proxy.async'ed) ----
      named_bar_sync(2, 160);
      if constexpr (kL2) {
        // the warpgroup has read W and the small variables for the L2 term (and fenced those generic reads before the
        // hand-off): the pull-ahead may overwrite them now
        if (lane == 0 && !p.strict && nxt != kFusedNoStep) issue_wx(nxt);
      }
      {
        const PushTarget& tw = p.shard[sl.shard].push;
        const uint32_t slot = tw.mode == PUSH_MAILBOX ? seq % tw.nslots : 0u;
        if (lane == 0 && nkc > 0) {
          fence_proxy_async_smem_cta();
          for (int i = 0; i < nkc; ++i) {
            const void* src = smem + kOffStage + i * kFsWChunk;
            const int c0 = (sl.kc_begin + i) * 32;
            if (tw.mode == PUSH_ATOMIC) tma_reduce_add_3d(&maps.push[rank], src, c0, 0, 0);   // push == apply (SGD)
            else tma_store_3d(&maps.push[rank], src, c0, 0, static_cast<int>(slot));          // rows >= H / cols >= I clipped
          }
          bulk_commit_group();
        }
      }
      __syncwarp();
      cluster_sync_all();                                   // #3: dW MMAs done, every CTA's small-gradient stores issued
      // What the publisher needs of this step is read now: once this warp has arrived at the next step's barriers the
      // other warps run ahead and overwrite the per-step shared-memory state.
      pend.step = cur;
      pend.seq = seq;
      pend.ts_slot = jl;
      pend.loss = pend.corr = 0.f;
      if (rank == 0 && lane == 0) {
#pragma unroll
        for (int src = 0; src < kFusedCluster; ++src) { pend.loss += scal[src * 2]; pend.corr += scal[src * 2 + 1]; }
        if constexpr (kL2) {
          const float* l2p = reinterpret_cast<const float*>(smem + kOffL2Part);
          float r = 0.f;
#pragma unroll
          for (int src = 0; src < kFusedCluster; ++src) r += l2p[src];
          pend.loss = __fadd_rn(pend.loss, __fmul_rn(p.l2_scale, __fmul_rn(0.5f, r)));
        }
      }
      if (lane == 0 && nxt != kFusedNoStep) issue_xmn(nxt, 0);   // (the dW MMAs that read the second x tile are complete)
      // Publishing costs several memory round trips (an NVLink round trip when the ps is remote): store completion,
      // a system-scope fence, the flags, the step result. It is deferred into the next step's head phase (see above)
      // unless (a) strict mode wants the acknowledgement before the next pull, (b) this was the cluster's last step,
      // or (c) the next step's mailbox flow control could wait for an acknowledgement that depends on these very
      // flags: the ps acknowledges in push order, the next step waits for push (next_seq - nslots), and that is at or
      // beyond this push only if the two claims are >= nslots apart — publish first whenever they are >= nslots / 2.
      deferred = !p.strict && nxt != kFusedNoStep && (nxt - cur) < (p.nslots >> 1);
      if (deferred && lane == 0 && nkc > 0) bulk_wait_group_read0();   // staging tile read: the next step may refill it
      __syncwarp();
      // EARLY ARRIVAL at barrier #1 of the next step: the other warps' next forward / reduce-scatter never waits for
      // this warp; it only *waits* for that barrier when it gets back to the loop top.
      arrived1 = nxt != kFusedNoStep;
      if (arrived1) cluster_barrier_arrive_release();
      if (!deferred && lane == 0) {
        publish(pend);
        if (nxt != kFusedNoStep && p.strict) {
          // strict: reference-exact read-your-writes — the next pull starts only after this step's push is applied
          if (mailbox) fs_wait_acks(p, seq, "strict pull");
          issue_wx(nxt);
        }
      }
      __syncwarp();
      cur = nxt;
    }
  } else {
    // =========================== wgmma / head warpgroup ===========================
    const int q = warp;                           // warp of the warpgroup
    const int et = threadIdx.x;                   // hidden unit of the head / small-gradient roles
    const bool unit_ok = et < H;
    // wgmma fragments: rows fr, fr + 8 of each m64 block, columns 8 (e >> 2) + 2 fc + (e & 1) of element e
    const int fr = q * 16 + (lane >> 2);
    const int fc = lane & 3;
    float* red = reinterpret_cast<float*>(smem + kOffRed);
    float* sg = reinterpret_cast<float*>(smem + kOffSg);
    float* val = reinterpret_cast<float*>(smem + kOffVal);
    float* wls = reinterpret_cast<float*>(smem + kOffWl);
    float* dls = reinterpret_cast<float*>(smem + kOffDl);
    float* dbl = reinterpret_cast<float*>(smem + kOffDbl);
    float* redw = reinterpret_cast<float*>(smem + kOffRedw);
    const float* raw_wl = reinterpret_cast<const float*>(smem + kOffRawWl);
    const float* raw_b = reinterpret_cast<const float*>(smem + kOffRawB);
    const float* raw_bl = reinterpret_cast<const float*>(smem + kOffRawBl);
    // head role of this thread: warp q handles batch row q of this CTA; lane -> (class hc, k-half kh)
    const int hc = lane >> 1, kh = lane & 1;
    const bool hc_ok = hc < C;
    const int brow = static_cast<int>(rank) * kFsRows + q;   // row of the head role inside a 32-row tile
    float* acc = reinterpret_cast<float*>(smem + kOffAcc);   // multi-tile running sums (see kOffAcc)
    float* acc_dbl = reinterpret_cast<float*>(smem + kOffAccDbl);
    float* acc_scal = reinterpret_cast<float*>(smem + kOffAccScal);
    // kClip: this thread's small gradients out of the landing zones (the same sums, in the same order, as the unclipped
    // push): sm_w value vg of unit u, value vg + 8 of it or hid_b (vg == 3), and sm_b (CTA 0, et < C). They are read
    // once for the norms and again for the push, so that no register holds them across the dW GEMM.
    // kL2: g + S * w of one small-gradient element, w out of its landing zone; `r` adds up w * w
    auto l2_add = [&](float g, float w, float& r) -> float {
      r = fmaf(w, w, r);
      return __fadd_rn(g, __fmul_rn(p.l2_scale, w));
    };
    // kL2: the L2 terms of this thread's small gradients (the elements the push below writes); returns the sum of w*w
    auto l2_small = [&](float& s0, float& s1, float& sbl) -> float {
      const int u = et & 15, vg = et >> 4;
      const int unit = static_cast<int>(rank) * 16 + u;
      float r = 0.f;
      if (unit < H) {
        if (vg < C) s0 = l2_add(s0, raw_wl[vg * H + unit], r);
        if (vg < 3 && vg + 8 < C) s1 = l2_add(s1, raw_wl[(vg + 8) * H + unit], r);
        if (vg == 3 && p.l2_biases) s1 = l2_add(s1, raw_b[unit], r);
      }
      if (rank == 0 && et < C && p.l2_biases) sbl = l2_add(sbl, raw_bl[et], r);
      return r;
    };
    // kL2: the per-warp sum of v into L2 warp partial `var` of this CTA (hid_w 0, small variables 1)
    float* l2_warp = reinterpret_cast<float*>(smem + kOffL2Warp);
    auto l2_warp_sum = [&](float v, int var) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) l2_warp[q * 2 + var] = v;
    };
    auto small_grads = [&](float& s0, float& s1, float& sbl) {
      const int u = et & 15, vg = et >> 4;
      s0 = 0.f;
      s1 = 0.f;
#pragma unroll
      for (int s = 0; s < kFusedCluster; ++s) {
        s0 += sg[(s * 16 + u) * kFsPart + vg];
        if (vg < 4) s1 += sg[(s * 16 + u) * kFsPart + vg + 8];
      }
      sbl = 0.f;
      if (rank == 0 && et < C) {
#pragma unroll
        for (int src = 0; src < kFusedCluster; ++src) sbl += dbl[src * kFsMaxC + et];
      }
      if constexpr (kL2) return l2_small(s0, s1, sbl);
      else return 0.f;
    };
    // kClip: the per-warp sum of v into warp partial `var` of this CTA (hid_w 0, hid_b 1, sm_w 2, sm_b 3)
    float* clip_warp = reinterpret_cast<float*>(smem + kOffClipWarp);
    auto clip_warp_sum = [&](float v, int var) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) clip_warp[q * kFsClipVars + var] = v;
    };
    // kClip: the clip factor of each variable (hid_w, hid_b, sm_w, sm_b) once every warp has stored its partials of
    // the small variables (after barrier #2) and this thread's sum of squares of its hid_w elements is `ssq_w`.
    // CLIP_GLOBAL_NORM: the common scale; CLIP_NORM: max(norm, clip_norm) per variable; CLIP_VALUE: unused.
    auto clip_factors = [&](float ssq_w) -> float4 {
      float4 fac = make_float4(1.f, 1.f, 1.f, 1.f);
      if (p.clip_kind == CLIP_VALUE) return fac;
      const float* cw = clip_warp;
      const float* cp = reinterpret_cast<const float*>(smem + kOffClipPart);
      clip_warp_sum(ssq_w, 0);
      named_bar_sync(1, 128);
      if (et < kFsClipVars) {
        const float c = (cw[et] + cw[kFsClipVars + et]) + (cw[2 * kFsClipVars + et] + cw[3 * kFsClipVars + et]);
#pragma unroll
        for (uint32_t d = 0; d < kFusedCluster; ++d)
          st_shared_cluster_f32(mapa_shared_cluster(sbase + kOffClipPart + (rank * kFsClipVars + et) * 4u, d), c);
      }
      cluster_sync_all();   // the norm barrier: every CTA's partials have landed in every CTA
      float tot[kFsClipVars];
#pragma unroll
      for (int v = 0; v < kFsClipVars; ++v) {
        float a = 0.f;
#pragma unroll
        for (int src = 0; src < kFusedCluster; ++src) a += cp[src * kFsClipVars + v];
        tot[v] = a;
      }
      const float cn = p.clip_norm;
      if (p.clip_kind == CLIP_GLOBAL_NORM) {
        const float sc = clip_global_scale(((tot[0] + tot[1]) + tot[2]) + tot[3], cn);
        fac = make_float4(sc, sc, sc, sc);
      } else {
        fac = make_float4(clip_norm_divisor(tot[0], cn), clip_norm_divisor(tot[1], cn), clip_norm_divisor(tot[2], cn),
                          clip_norm_divisor(tot[3], cn));
      }
      return fac;
    };
    auto clip_value = [&](float g, float f) -> float {
      return clip_element(p.clip_kind, g, f, p.clip_norm, p.clip_min, p.clip_max);
    };

    for (uint32_t jl = 0; cur != kFusedNoStep; ++jl) {
      const uint32_t seq = p.seq_base + cur + 1u;
      if (dbg && et == 0 && jl < 4) p.debug_ts[jl * kTs + 0] = clock64();
      // ---- step prologue ----
      if (is_claimer) broadcast_next((jl + 1) & 1, claim());
      // ---- row tiles of the step (the debug stamps below record the last tile's phases) ----
      for (int t = 0; t < T; ++t) {
        const bool last = t == T - 1;
        // Multi-tile: the step number is re-read from ctl_next[jl & 1], where it stays until barrier #3 of the step —
        // one register fewer across the tile loop, which keeps the kernel free of spills.
        uint32_t step = cur, push_seq = seq;
        if constexpr (kMulti) {
          step = ctl_next[jl & 1];
          push_seq = p.seq_base + step + 1u;
        }
        const int trow = 32 * t + brow;
        const bool hrow_ok = trow < B;
        float ylab = 0.f;
        if (hrow_ok && hc_ok) ylab = p.y_base[(fs_row0(p, step) + static_cast<uint64_t>(trow)) * C + hc];
        if (t == 0 && et == 127 && mailbox && push_seq > p.nslots) fs_wait_acks(p, push_seq - p.nslots, "flow control");

        // ---- forward partial: pre^T [128 hidden x 32 batch] over my K-slice ----
        if (t == 0) mbar_wait(bar_w, jl & 1);      // this step's W / x of tile 0 / small variables have landed
        else mbar_wait(bar_xk, (jl * static_cast<uint32_t>(T - 1) + static_cast<uint32_t>(t - 1)) & 1u);   // x of tile t
        float fa[2][4][4];             // [m64 block][n8 group][element]
#pragma unroll
        for (int mb = 0; mb < 2; ++mb)
#pragma unroll
          for (int g = 0; g < 4; ++g)
#pragma unroll
            for (int e = 0; e < 4; ++e) fa[mb][g][e] = 0.f;
        if (nkc > 0) {
          wgmma_fence();
          for (int i = 0; i < nkc; ++i) {
            const uint32_t a_addr = sbase + kOffW + i * kFsWChunk;
            const uint32_t b_addr = sbase + kOffXk + i * kFsXChunk;
#pragma unroll
            for (int j = 0; j < 4; ++j)   // K-major: advance 32 B inside the 128 B swizzle atom; SBO = 8 rows x 128 B
#pragma unroll
              for (int mb = 0; mb < 2; ++mb)
                fs_mma_m64n32(fa[mb], make_wgmma_desc_sw128(a_addr + mb * 64 * 128 + j * 32),
                              make_wgmma_desc_sw128(b_addr + j * 32), (i > 0 || j > 0) ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait0();
#pragma unroll
          for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int g = 0; g < 4; ++g)
#pragma unroll
              for (int e = 0; e < 4; ++e) wgmma_reg_fence(fa[mb][g][e]);
        }
        if (dbg && et == 0 && jl < 4) p.debug_ts[jl * kTs + 1] = clock64();
        // small variables out of the bulk-copied image, before barrier #1 lets warp 0 overwrite it with the next pull
        const float bias = unit_ok ? raw_b[et] : 0.f;
        float wl[kFsMaxC];
#pragma unroll
        for (int c = 0; c < kFsMaxC; ++c) wl[c] = (unit_ok && c < C) ? raw_wl[c * H + et] : 0.f;
        const float blast = hc_ok ? raw_bl[hc] : 0.f;
        {
          // reduce-scatter: batch columns 4d..4d+3 go to CTA d; element pair (e, e + 1) of n8 group g is columns
          // 8 g + 2 fc, +1 of row fr + 8 (e >> 1): CTA 2 g + (fc >> 1), at column offset 2 (fc & 1) of its float4
#pragma unroll
          for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int g = 0; g < 4; ++g)
#pragma unroll
              for (int e = 0; e < 4; e += 2) {
                const uint32_t row = static_cast<uint32_t>(mb * 64 + fr + 8 * (e >> 1));
                const uint32_t d = static_cast<uint32_t>(2 * g + (fc >> 1));
                const uint32_t off = kOffRed + ((rank * 128u + row) << 4) + static_cast<uint32_t>(fc & 1) * 8u;
                st_shared_cluster_v2f32(mapa_shared_cluster(sbase + off, d), fa[mb][g][e], fa[mb][g][e + 1]);
              }
        }
        cluster_sync_all();                                   // #1
        if (dbg && et == 0 && jl < 4) p.debug_ts[jl * kTs + 2] = clock64();
        float hv[kFsRows];
        {
          float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int s = 0; s < kFusedCluster; ++s) {
            const float4 t = *reinterpret_cast<const float4*>(red + (s * 128 + et) * 4);
            acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
          }
          if constexpr (kGeneral) {
            hv[0] = unit_ok ? act_forward(p.act, acc.x + bias) : 0.f;
            hv[1] = unit_ok ? act_forward(p.act, acc.y + bias) : 0.f;
            hv[2] = unit_ok ? act_forward(p.act, acc.z + bias) : 0.f;
            hv[3] = unit_ok ? act_forward(p.act, acc.w + bias) : 0.f;
          } else {
            hv[0] = unit_ok ? fmaxf(acc.x + bias, 0.f) : 0.f;
            hv[1] = unit_ok ? fmaxf(acc.y + bias, 0.f) : 0.f;
            hv[2] = unit_ok ? fmaxf(acc.z + bias, 0.f) : 0.f;
            hv[3] = unit_ok ? fmaxf(acc.w + bias, 0.f) : 0.f;
          }
        }
        // ---- head on my 4 batch rows ----
#pragma unroll
        for (int i = 0; i < kFsRows; ++i) val[i * 128 + et] = hv[i];
#pragma unroll
        for (int c = 0; c < kFsMaxC; ++c) wls[c * kFsWlStride + et] = wl[c];
        named_bar_sync(1, 128);
        if (dbg && et == 0 && jl < 4) p.debug_ts[jl * kTs + 3] = clock64();
        {
          // logits: warp q = row q of this CTA, lane = (class, half of the hidden units)
          float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
          const float* hrow = val + q * 128 + kh * 64;
          const float* wrow = wls + hc * kFsWlStride + kh * 64;
#pragma unroll
          for (int k = 0; k < 64; k += 4) {   // units >= H are zero in both operands
            const float4 hvv = *reinterpret_cast<const float4*>(hrow + k);
            const float4 wv = *reinterpret_cast<const float4*>(wrow + k);
            a0 = fmaf(hvv.x, wv.x, a0); a1 = fmaf(hvv.y, wv.y, a1);
            a2 = fmaf(hvv.z, wv.z, a2); a3 = fmaf(hvv.w, wv.w, a3);
          }
          float dot = (a0 + a1) + (a2 + a3);
          dot += __shfl_xor_sync(0xffffffffu, dot, 1);
          // the label the loss sees: smoothed (general head) for real classes, still 0 for padded ones
          float y = ylab;
          if constexpr (kGeneral) y = hc_ok ? smooth_label(p.loss_kind, ylab, p.label_smoothing, C) : 0.f;
          const float z = hc_ok ? dot + blast : -INFINITY;
          float zmax = z, ybest = hc_ok ? ylab : -INFINITY, ysum = y;
#pragma unroll
          for (int o = 16; o > 1; o >>= 1) {   // over the 16 classes (lane bit 0 is the k-half: both halves hold the same)
            zmax = fmaxf(zmax, __shfl_xor_sync(0xffffffffu, zmax, o));
            ybest = fmaxf(ybest, __shfl_xor_sync(0xffffffffu, ybest, o));
            ysum += __shfl_xor_sync(0xffffffffu, ysum, o);
          }
          int zarg = (hc_ok && z == zmax) ? hc : kFsMaxC, yarg = (hc_ok && ylab == ybest) ? hc : kFsMaxC;  // first maximum wins
          const float e = hc_ok ? __expf(z - zmax) : 0.f;
          float esum = e;
#pragma unroll
          for (int o = 16; o > 1; o >>= 1) {
            zarg = min(zarg, __shfl_xor_sync(0xffffffffu, zarg, o));
            yarg = min(yarg, __shfl_xor_sync(0xffffffffu, yarg, o));
            esum += __shfl_xor_sync(0xffffffffu, esum, o);
          }
          const float pc = __fdividef(e, esum);
          float dl = 0.f, lc = 0.f;
          if (p.loss_kind == LOSS_BOOK) {
            // L = -(1/(B*C)) sum y*log(clip(p,1e-10,1));  dL/dp = -y/(B*C*p) where the clip passes gradient (DS:52-53)
            const float k = 1.f / (static_cast<float>(B) * static_cast<float>(C));
            const bool pass = hc_ok && (pc >= 1e-10f) && (pc <= 1.0f);
            const float g = pass ? (-k * y / pc) : 0.f;
            float gp = g * pc;
#pragma unroll
            for (int o = 16; o > 1; o >>= 1) gp += __shfl_xor_sync(0xffffffffu, gp, o);
            dl = pc * (g - gp);
            lc = hc_ok ? -k * y * __logf(fminf(fmaxf(pc, 1e-10f), 1.0f)) : 0.f;
          } else if (!kGeneral || p.loss_kind == LOSS_XENT) {
            // L = (1/B) sum_b -sum_c y*log_softmax(z);  dz = (p*sum(y) - y)/B   (DS:35)
            const float k = 1.f / static_cast<float>(B);
            dl = k * (pc * ysum - y);
            lc = hc_ok ? -k * y * (z - (zmax + __logf(esum))) : 0.f;
          } else if (hc_ok) {
            elementwise_loss(p.loss_kind, z, y, 1.f / (static_cast<float>(B) * static_cast<float>(C)), dl, lc);
          }
          if (kh == 0) dls[q * kFsMaxC + hc] = (hrow_ok && hc_ok) ? dl : 0.f;
          float loss_part = (hrow_ok && kh == 0) ? lc : 0.f;
          float corr_part = (hrow_ok && lane == 0 && zarg == yarg) ? 1.f : 0.f;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) loss_part += __shfl_xor_sync(0xffffffffu, loss_part, o);
          corr_part = __shfl_sync(0xffffffffu, corr_part, 0);
          if (lane == 0) { redw[q] = loss_part; redw[4 + q] = corr_part; }
        }
        named_bar_sync(1, 128);
        if (dbg && et == 0 && jl < 4) p.debug_ts[jl * kTs + 4] = clock64();
        // ---- gradients of my rows; thread -> hidden unit et ----
        float dw[kFsPart];
#pragma unroll
        for (int c = 0; c < kFsPart; ++c) dw[c] = 0.f;
        float dp[kFsRows];
        float dbh = 0.f;
#pragma unroll
        for (int i = 0; i < kFsRows; ++i) {
          float dh = 0.f;
#pragma unroll
          for (int c4 = 0; c4 < kFsMaxC / 4; ++c4) {
            const float4 d = *reinterpret_cast<const float4*>(dls + i * kFsMaxC + 4 * c4);   // broadcast reads
            dh = fmaf(d.x, wl[4 * c4 + 0], dh); dh = fmaf(d.y, wl[4 * c4 + 1], dh);
            dh = fmaf(d.z, wl[4 * c4 + 2], dh); dh = fmaf(d.w, wl[4 * c4 + 3], dh);
            if (4 * c4 + 0 < kFsPart - 1) dw[4 * c4 + 0] = fmaf(d.x, hv[i], dw[4 * c4 + 0]);
            if (4 * c4 + 1 < kFsPart - 1) dw[4 * c4 + 1] = fmaf(d.y, hv[i], dw[4 * c4 + 1]);
            if (4 * c4 + 2 < kFsPart - 1) dw[4 * c4 + 2] = fmaf(d.z, hv[i], dw[4 * c4 + 2]);
            if (4 * c4 + 3 < kFsPart - 1) dw[4 * c4 + 3] = fmaf(d.w, hv[i], dw[4 * c4 + 3]);
          }
          if constexpr (kGeneral) dp[i] = act_backward(p.act, hv[i], dh);   // (finite f': 0 for rows >= B as well)
          else dp[i] = hv[i] > 0.f ? dh : 0.f;       // rows >= B carry dlogits == 0 -> dp == 0
          dbh += dp[i];
        }
        dw[kFsPart - 1] = dbh;
        // Multi-tile: the small gradients, loss and correct count add up over the row tiles in shared memory (the
        // same thread owns the same words in every tile) and are reduce-scattered once, in the last tile.
        auto carry = [&](float v, float* run) -> float {
          if (t > 0) v += *run;
          if (!last) *run = v;
          return v;
        };
        if constexpr (kMulti) {
#pragma unroll
          for (int c = 0; c < kFsPart; ++c) dw[c] = carry(dw[c], acc + c * 128 + et);
        }
        {
          // all-gather of dpre^T: row et (128 B = 32 batch values), my 16-byte chunk is number `rank`; K-major
          // SWIZZLE_128B: chunk j of row r sits at r * 128 + ((j ^ (r & 7)) << 4)
          const uint32_t a_off = kOffA + static_cast<uint32_t>(et) * 128u + ((rank ^ (static_cast<uint32_t>(et) & 7u)) << 4);
#pragma unroll
          for (uint32_t d = 0; d < kFusedCluster; ++d)
            st_shared_cluster_v4f32(mapa_shared_cluster(sbase + a_off, d), dp[0], dp[1], dp[2], dp[3]);
          if (last) {
            // reduce-scatter of the small-gradient partials: hidden units [16 d, 16 d + 16) are summed by CTA d
            const uint32_t sg_off = kOffSg + ((rank * 16u + (static_cast<uint32_t>(et) & 15u)) * kFsPart) * 4u;
            const uint32_t sg_dst = mapa_shared_cluster(sbase + sg_off, static_cast<uint32_t>(et) >> 4);
            st_shared_cluster_v4f32(sg_dst, dw[0], dw[1], dw[2], dw[3]);
            st_shared_cluster_v4f32(sg_dst + 16u, dw[4], dw[5], dw[6], dw[7]);
            st_shared_cluster_v4f32(sg_dst + 32u, dw[8], dw[9], dw[10], dw[11]);
          }
          if (et < kFsMaxC) {
            float sdl = 0.f;
#pragma unroll
            for (int i = 0; i < kFsRows; ++i) sdl += dls[i * kFsMaxC + et];
            if constexpr (kMulti) sdl = carry(sdl, acc_dbl + et);
            if (last) st_shared_cluster_f32(mapa_shared_cluster(sbase + kOffDbl + (rank * kFsMaxC + et) * 4u, 0), sdl);
          }
          if (et == 0) {
            float ls = (redw[0] + redw[1]) + (redw[2] + redw[3]);
            if constexpr (kMulti) ls = carry(ls, acc_scal);
            if (last) st_shared_cluster_f32(mapa_shared_cluster(sbase + kOffScal + (rank * 2u) * 4u, 0), ls);
            float cs = (redw[4] + redw[5]) + (redw[6] + redw[7]);
            if constexpr (kMulti) cs = carry(cs, acc_scal + 1);
            if (last) st_shared_cluster_f32(mapa_shared_cluster(sbase + kOffScal + (rank * 2u + 1u) * 4u, 0), cs);
          }
        }
        fence_proxy_async_smem_cluster();
        if (dbg && et == 0 && jl < 4) p.debug_ts[jl * kTs + 5] = clock64();
        cluster_sync_all();                                   // #2
        if (dbg && et == 0 && jl < 4) p.debug_ts[jl * kTs + 6] = clock64();

        // ---- small gradients: sum the 8 sources for my 16 hidden units and push them ----
        if (!kClip && last) {
          const FsPush pw_l = fs_resolve(p.shard[p.shard_wl].push, push_seq);
          const FsPush pb_h = fs_resolve(p.shard[p.shard_bh].push, push_seq);
          const int u = et & 15, vg = et >> 4;   // values vg (0..7) and vg + 8 (8..11) of unit u
          float s0 = 0.f, s1 = 0.f;
#pragma unroll
          for (int s = 0; s < kFusedCluster; ++s) {
            s0 += sg[(s * 16 + u) * kFsPart + vg];
            if (vg < 4) s1 += sg[(s * 16 + u) * kFsPart + vg + 8];
          }
          const int unit = static_cast<int>(rank) * 16 + u;
          float s = 0.f;
          if constexpr (kL2) {
            if (rank == 0 && et < C) {
#pragma unroll
              for (int src = 0; src < kFusedCluster; ++src) s += dbl[src * kFsMaxC + et];
            }
            l2_warp_sum(l2_small(s0, s1, s), 1);
          }
          if (unit < H) {
            if (vg < C) fs_push_value(p.shard[p.shard_wl].push, pw_l.base + p.off_wl + static_cast<size_t>(vg) * H + unit, s0);
            if (vg < 3 && vg + 8 < C)
              fs_push_value(p.shard[p.shard_wl].push, pw_l.base + p.off_wl + static_cast<size_t>(vg + 8) * H + unit, s1);
            if (vg == 3) fs_push_value(p.shard[p.shard_bh].push, pb_h.base + p.off_bh + unit, s1);
          }
          if (rank == 0 && et < C) {
            const FsPush pb_l = fs_resolve(p.shard[p.shard_bl].push, push_seq);
            if constexpr (!kL2) {
#pragma unroll
              for (int src = 0; src < kFusedCluster; ++src) s += dbl[src * kFsMaxC + et];
            }
            fs_push_value(p.shard[p.shard_bl].push, pb_l.base + p.off_bl + et, s);
          }
        }
        // kClip: only their squares count now (warp partials of hid_b / sm_w / sm_b); they are pushed once the clip is
        // known, after the norm barrier
        if (kClip && last && p.clip_kind != CLIP_VALUE) {
          const int u = et & 15, vg = et >> 4;
          const int unit = static_cast<int>(rank) * 16 + u;
          float s0, s1, sbl, ssq_bh = 0.f, ssq_wl = 0.f, ssq_bl = 0.f;
          small_grads(s0, s1, sbl);
          if (unit < H) {
            if (vg < C) ssq_wl = s0 * s0;
            if (vg < 3 && vg + 8 < C) ssq_wl += s1 * s1;
            if (vg == 3) ssq_bh = s1 * s1;
          }
          if (rank == 0 && et < C) ssq_bl = sbl * sbl;
          clip_warp_sum(ssq_bh, 1);
          clip_warp_sum(ssq_wl, 2);
          clip_warp_sum(ssq_bl, 3);
        }

        // ---- dW^T tile of my K-slice: wgmma -> registers -> swizzled staging tile; warp 4 TMA-stores it (the push) ----
        fence_proxy_async_smem_cta();   // generic-proxy (DSMEM) writes of dpre^T -> tensor-core reads
        mbar_wait(bar_xmn, (jl * static_cast<uint32_t>(T) + static_cast<uint32_t>(t)) & 1u);
        if (dbg && et == 0 && jl < 4) p.debug_ts[jl * kTs + 7] = clock64();
        float4 cfac = make_float4(1.f, 1.f, 1.f, 1.f);   // kClip: clip_factors of this step
        if (nkc > 0) {
          // D[feature f][hidden h] = sum_b x[b][f] dpre^T[h][b]: M = my features (m64 blocks), N = 128 hidden units,
          // K = 32 batch rows. A = x^T from registers, read out of the K-major x tile ([b][f], 128-byte swizzled);
          // B = dpre^T, K-major in shared memory. Rows of a block beyond my slice compute garbage and are not stored.
          const int nmb = (nkc * 32 + 63) >> 6;
          const uint8_t* xs = smem + kOffXmn;
          float da[2][16][4];
#pragma unroll
          for (int mb = 0; mb < 2; ++mb) {
            if (mb < nmb) {
              uint32_t a[4][4];
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const int f0 = mb * 64 + fr, b0 = 8 * j + fc;
                auto xat = [&](int f, int b) -> uint32_t {   // x[b][f]: chunk f / 32 of the x tile
                  const uint32_t o = static_cast<uint32_t>(f >> 5) * kFsXChunk + sw128_offset(b, f & 31, 4);
                  return (f >> 5) < nkc ? *reinterpret_cast<const uint32_t*>(xs + o) : 0u;
                };
                a[j][0] = xat(f0, b0);
                a[j][1] = xat(f0 + 8, b0);
                a[j][2] = xat(f0, b0 + 4);
                a[j][3] = xat(f0 + 8, b0 + 4);
              }
              wgmma_fence();
#pragma unroll
              for (int j = 0; j < 4; ++j)
                fs_mma_m64n128(da[mb], a[j], make_wgmma_desc_sw128(sbase + kOffA + j * 32), j > 0 ? 1u : 0u);
              wgmma_commit();
              wgmma_wait0();
#pragma unroll
              for (int g = 0; g < 16; ++g)
#pragma unroll
                for (int e = 0; e < 4; ++e) wgmma_reg_fence(da[mb][g][e]);
            }
          }
          if constexpr (kMulti) {
            if (!last) mbar_arrive(bar_xmn_empty);   // Xmn is read: warp 4 may load the next tile's x into it
          }
          const PushTarget& tw = p.shard[sl.shard].push;
          const float sc = tw.mode == PUSH_ATOMIC ? tw.scale : 1.f;
          // staging tile of chunk i: [128 hidden rows][32 features] fp32, SWIZZLE_128B (the TMA store's box); row
          // tiles after the first add into it (every thread owns the same elements in every tile)
#pragma unroll
          for (int mb = 0; mb < 2; ++mb) {
            if (mb < nmb) {
#pragma unroll
              for (int g = 0; g < 16; ++g)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const int f = mb * 64 + fr + 8 * (e >> 1);
                  const int h = 8 * g + 2 * fc + (e & 1);
                  if ((f >> 5) < nkc) {
                    float* st = reinterpret_cast<float*>(smem + kOffStage + (f >> 5) * kFsWChunk + sw128_offset(h, f & 31, 4));
                    if (kMulti && t > 0) *st += sc * da[mb][g][e];
                    else *st = sc * da[mb][g][e];
                  }
                }
            }
          }
          if constexpr (kL2) {
            if (last) {
              // g + S * w over the staging tile, rolled like the clip passes below. The forward's W tile has the
              // staging tile's layout ([128 hidden rows][32 features] per chunk, SWIZZLE_128B), so element o of one is
              // element o of the other. Only the elements the TMA store pushes count toward the sum of w*w.
              const int n4 = nkc * static_cast<int>(kFsWChunk / 16);
              named_bar_sync(1, 128);   // every thread's part of the tile is in place (the pass crosses threads)
              const float S = p.l2_scale;
              float r = 0.f;
              for (int i4 = et; i4 < n4; i4 += 128) {
                const int i = i4 / static_cast<int>(kFsWChunk / 16), o = (i4 % static_cast<int>(kFsWChunk / 16)) * 16;
                const int h = o >> 7, fl = (((o >> 4) & 7) ^ (h & 7)) << 2;   // inverse of sw128_offset
                const float4 w = *reinterpret_cast<const float4*>(smem + kOffW + i * kFsWChunk + o);
                float4* st = reinterpret_cast<float4*>(smem + kOffStage + i * kFsWChunk + o);
                float4 v = *st;
                v.x = __fadd_rn(v.x, __fmul_rn(S, w.x));
                v.y = __fadd_rn(v.y, __fmul_rn(S, w.y));
                v.z = __fadd_rn(v.z, __fmul_rn(S, w.z));
                v.w = __fadd_rn(v.w, __fmul_rn(S, w.w));
                *st = v;
                if (h < H && (sl.kc_begin + i) * 32 + fl < p.I) {   // I % 4 == 0: a float4 is in or out as a whole
                  r = fmaf(w.x, w.x, r);
                  r = fmaf(w.y, w.y, r);
                  r = fmaf(w.z, w.z, r);
                  r = fmaf(w.w, w.w, r);
                }
              }
              l2_warp_sum(r, 0);
            }
          }
          if constexpr (kClip) {
            if (last) {
              // Only the elements the TMA store pushes (hidden rows < H, features < I) count toward the norms. The loop
              // above has written the step's dW (summed over the row tiles) into the staging tile, which is read and
              // scaled in place as float4s by a rolled loop: an unrolled pass over the wgmma fragments instead costs
              // more than twice the step time at batch 32 (measured), from the code it adds to the step loop.
              const int n4 = nkc * static_cast<int>(kFsWChunk / 16);
              named_bar_sync(1, 128);   // every thread's part of the tile is in place (the passes below cross threads)
              if (p.clip_kind != CLIP_VALUE) {   // (value clamps each element: no sums, no norm barrier)
                float ssq_w = 0.f;
                for (int i4 = et; i4 < n4; i4 += 128) {
                  const int i = i4 / static_cast<int>(kFsWChunk / 16), o = (i4 % static_cast<int>(kFsWChunk / 16)) * 16;
                  const int h = o >> 7, fl = (((o >> 4) & 7) ^ (h & 7)) << 2;   // inverse of sw128_offset
                  const float4 v = *reinterpret_cast<const float4*>(smem + kOffStage + i * kFsWChunk + o);
                  if (h < H && (sl.kc_begin + i) * 32 + fl < p.I) {   // I % 4 == 0: a float4 is in or out as a whole
                    ssq_w = fmaf(v.x, v.x, ssq_w);
                    ssq_w = fmaf(v.y, v.y, ssq_w);
                    ssq_w = fmaf(v.z, v.z, ssq_w);
                    ssq_w = fmaf(v.w, v.w, ssq_w);
                  }
                }
                cfac = clip_factors(ssq_w);
              }
              for (int i4 = et; i4 < n4; i4 += 128) {
                const int i = i4 / static_cast<int>(kFsWChunk / 16), o = (i4 % static_cast<int>(kFsWChunk / 16)) * 16;
                float4* st = reinterpret_cast<float4*>(smem + kOffStage + i * kFsWChunk + o);
                float4 v = *st;
                v.x = clip_value(v.x, cfac.x);
                v.y = clip_value(v.y, cfac.x);
                v.z = clip_value(v.z, cfac.x);
                v.w = clip_value(v.w, cfac.x);
                *st = v;
              }
            }
          }
        }
        if constexpr (kClip) {
          if (last) {
            if (nkc == 0) cfac = clip_factors(0.f);   // no dW tile, the same norm barrier
            // the small gradients, clipped, after the norm barrier and before barrier #3 (the publisher's flags)
            const FsPush pw_l = fs_resolve(p.shard[p.shard_wl].push, push_seq);
            const FsPush pb_h = fs_resolve(p.shard[p.shard_bh].push, push_seq);
            const int u = et & 15, vg = et >> 4;
            float cg0, cg1, cgl;
            const float l2_r = small_grads(cg0, cg1, cgl);
            if constexpr (kL2) l2_warp_sum(l2_r, 1);
            const int unit = static_cast<int>(rank) * 16 + u;
            if (unit < H) {
              if (vg < C)
                fs_push_value(p.shard[p.shard_wl].push, pw_l.base + p.off_wl + static_cast<size_t>(vg) * H + unit,
                              clip_value(cg0, cfac.z));
              if (vg < 3 && vg + 8 < C)
                fs_push_value(p.shard[p.shard_wl].push, pw_l.base + p.off_wl + static_cast<size_t>(vg + 8) * H + unit,
                              clip_value(cg1, cfac.z));
              if (vg == 3) fs_push_value(p.shard[p.shard_bh].push, pb_h.base + p.off_bh + unit, clip_value(cg1, cfac.y));
            }
            if (rank == 0 && et < C) {
              const FsPush pb_l = fs_resolve(p.shard[p.shard_bl].push, push_seq);
              fs_push_value(p.shard[p.shard_bl].push, pb_l.base + p.off_bl + et, clip_value(cgl, cfac.w));
            }
          }
        }
        if constexpr (kL2) {
          if (last) {
            if (nkc == 0) l2_warp_sum(0.f, 0);   // no W k-slice
            named_bar_sync(1, 128);              // every warp's L2 partials are in place
            if (et == 0) {
              const float r = ((l2_warp[0] + l2_warp[2]) + (l2_warp[4] + l2_warp[6])) +
                              ((l2_warp[1] + l2_warp[3]) + (l2_warp[5] + l2_warp[7]));
              st_shared_cluster_f32(mapa_shared_cluster(sbase + kOffL2Part + rank * 4u, 0), r);   // before barrier #3
            }
          }
        }
        if (last) {
          fence_proxy_async_smem_cta();  // staging writes -> visible to the TMA engine (shared memory only: does not
                                         // wait for the small-gradient peer stores issued above)
          named_bar_arrive(2, 160);      // hand the tile to warp 4 (non-blocking) ...
          if (dbg && et == 0 && jl < 4) p.debug_ts[jl * kTs + 8] = clock64();
          cluster_sync_all();            // #3 ... and go on to the next step
          if (dbg && et == 0 && jl < 4) p.debug_ts[jl * kTs + 9] = clock64();
        }
      }
      cur = ctl_next[(jl + 1) & 1];
    }
  }

  // ---- teardown ----
  __syncthreads();
  cluster_sync_all();   // nobody leaves while a peer might still address its shared memory
  if (rank == 0 && threadIdx.x == 0) {
    if (p.lane_rec != nullptr) p.lane_rec[blockIdx.y * kLaneRecWords + 10] = globaltimer_ns();
    // The last cluster to finish re-arms the launch state (no host-side memset / copy between launches) and, when asked
    // to, waits for the ps acknowledgement of every push made so far — every other cluster has published its steps
    // before it got here, so *seq_word is final.
    __threadfence();
    if (atomicAdd(p.exit_counter, 1u) + 1u == gridDim.y) {
      __threadfence();
      if (p.wait_acks && p.shard[0].push.mode == PUSH_MAILBOX)
        fs_wait_acks(p, *reinterpret_cast<volatile uint32_t*>(p.seq_word), "end of launch");
      *p.step_counter = 0u;
      *p.exit_counter = 0u;
      if (p.clear_stop) *p.stop_word = 0u;
      if (dbg) p.debug_ts[63] = static_cast<long long>(globaltimer_ns());
    }
  }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static bool fused_multi_tile(int B) { return B > 32; }

size_t fused_smem_bytes(int B) { return fused_multi_tile(B) ? fs_smem_bytes<kFsMaxTiles>() : fs_smem_bytes<1>(); }

// One launch config for every instantiation: `lanes` clusters of 8 CTAs.
static cudaLaunchConfig_t fused_launch_config(int lanes, int B, cudaStream_t stream, cudaLaunchAttribute* attr) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(kFusedCluster, lanes, 1);
  cfg.blockDim = dim3(kFsThreads);
  cfg.dynamicSmemBytes = fused_smem_bytes(B);
  cfg.stream = stream;
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kFusedCluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cfg;
}

using FusedKernel = void (*)(const FusedMaps, const FusedParams);

// The instantiation that runs batch B, with or without the clip, the L2 term and the general head (fused_general_head).
static FusedKernel fused_kernel(int B, bool clip, bool l2, bool general) {
  static const FusedKernel table[2][2][2][2] = {   // [general][l2][clip][multi-tile], in load order
      {{{fused_step_kernel<1, false, false, false>, fused_step_kernel<kFsMaxTiles, false, false, false>},
        {fused_step_kernel<1, true, false, false>, fused_step_kernel<kFsMaxTiles, true, false, false>}},
       {{fused_step_kernel<1, false, true, false>, fused_step_kernel<kFsMaxTiles, false, true, false>},
        {fused_step_kernel<1, true, true, false>, fused_step_kernel<kFsMaxTiles, true, true, false>}}},
      {{{fused_step_kernel<1, false, false, true>, fused_step_kernel<kFsMaxTiles, false, false, true>},
        {fused_step_kernel<1, true, false, true>, fused_step_kernel<kFsMaxTiles, true, false, true>}},
       {{fused_step_kernel<1, false, true, true>, fused_step_kernel<kFsMaxTiles, false, true, true>},
        {fused_step_kernel<1, true, true, true>, fused_step_kernel<kFsMaxTiles, true, true, true>}}}};
  return table[general][l2][clip][fused_multi_tile(B)];
}

// Every instantiation: shared-memory opt-in + force-load (DESIGN §7). A one-tile (32) and a multi-tile batch, with and
// without the general head, stand for all.
cudaError_t prepare_fused_kernels() {
  for (const bool general : {false, true})
    for (const bool l2 : {false, true})
      for (const bool clip : {false, true})
        for (const int B : {32, 32 * kFsMaxTiles}) {
          const FusedKernel k = fused_kernel(B, clip, l2, general);
          cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(fused_smem_bytes(B)));
          cudaFuncAttributes a;
          if (e == cudaSuccess) e = cudaFuncGetAttributes(&a, k);
          if (e != cudaSuccess) return e;
        }
  return cudaSuccess;
}

cudaError_t launch_fused_step(const FusedMaps& maps, const FusedParams& p, int lanes, cudaStream_t stream) {
  if (lanes < 1 || p.B < 1 || p.B > 32 * kFsMaxTiles || p.H < 1 || p.H > 128 || p.C < 1 || p.C > kFsPart - 1 ||
      (p.I & 3) || p.n_shards < 1 || p.n_shards > kFusedMaxShards || p.nslots < 1 || p.clip_kind < CLIP_OFF ||
      p.clip_kind > CLIP_VALUE || !(p.l2_scale >= 0.f && p.l2_scale < INFINITY) ||
      (p.l2_scale != 0.f && p.shard[0].push.mode == PUSH_ATOMIC) || !act_valid(p.act) || !loss_valid(p.loss_kind) ||
      !label_smoothing_valid(p.loss_kind, p.label_smoothing))
    return cudaErrorInvalidValue;
  for (int r = 0; r < kFusedCluster; ++r)
    if (p.slice[r].kc_count < 0 || p.slice[r].kc_count > kFusedMaxChunks) return cudaErrorInvalidValue;
  cudaLaunchAttribute attr[1];
  const cudaLaunchConfig_t cfg = fused_launch_config(lanes, p.B, stream, attr);
  const bool general = fused_general_head(p.act, p.loss_kind, p.label_smoothing);
  return cudaLaunchKernelEx(&cfg, fused_kernel(p.B, p.clip_kind != CLIP_OFF, p.l2_scale != 0.f, general), maps, p);
}

cudaError_t fused_max_lanes(int B, bool clip, bool l2, bool general, int* out) {
  cudaLaunchAttribute attr[1];
  const cudaLaunchConfig_t cfg = fused_launch_config(1, B, nullptr, attr);
  return cudaOccupancyMaxActiveClusters(out, fused_kernel(B, clip, l2, general), &cfg);
}

}  // namespace dm
