// Host/device shared structures: kernel parameter blocks and the parameter-server shard layout.
//
// Terminology
//   arena     : one PS shard's flat fp32 parameter buffer (all variables placed on that ps task,
//               each at an aligned element offset) plus same-shaped Adam m/v buffers and an optional
//               bf16 shadow copy that workers pull when computing in bf16.
//   mailbox   : per (worker, slot) gradient staging area living in the *PS's* HBM, same layout as the
//               arena. Workers write gradient tiles into it with P2P stores from inside their backward
//               kernels; the PS kernel polls per-item flags and applies.
//   item      : the unit of push/apply hand-off: a 2-D block {offset, rows, cols, ld} of the arena.
//               One flag per (worker, slot, item); flag value == push sequence number when ready.
//   inbox     : tiny buffer in each *worker's* HBM that the PS writes (P2P) so the worker can poll
//               locally: {acked push seq, global_step}.
#pragma once
#include <stdint.h>

namespace dm {

constexpr int kMaxWorkers = 32;
// worker_done[w] sentinel written by the ps host when worker w is presumed dead (no heartbeat): the serve kernel /
// loop stops waiting for its pushes when it decides whether every worker has left.
constexpr uint32_t kWorkerDead = 0xFFFFFFFFu;

enum PushMode : int {
  PUSH_LOCAL = 0,    // plain store into a local fp32 gradient buffer (tests, NCCL baseline)
  PUSH_MAILBOX = 1,  // P2P store into the PS mailbox slot + release flag (Adam / SGD via PS kernel)
  PUSH_ATOMIC = 2,   // red.add(scale * g) straight into the PS master params (async SGD, no PS kernel)
};

struct PushTarget {
  int mode;
  float scale;              // PUSH_ATOMIC: -lr ; else 1
  float* base;              // LOCAL: grad arena; MAILBOX: this worker's slot-0 mailbox on the PS; ATOMIC: PS params
  uint64_t slot_stride;     // elements between mailbox slots
  uint32_t* flags;          // MAILBOX: this worker's slot-0 flag array on the PS
  uint32_t flag_slot_stride;
  uint32_t nslots;
  uint32_t gpu_scope;       // 1: the PS shard lives on this worker's own GPU -> gpu-scope release is enough
  uint32_t pad_;
  const uint32_t* seq_ptr;  // device-local current push sequence number (1-based); null => seq 1 / slot 0
};

// Epilogue selection for the wgmma GEMM  D[M,N] = A[M,K] * B[N,K]^T  (fp32 accumulators)
enum GemmEpilogue : int {
  // out[n * ldo + m] = f(acc[m][n]) — lanes write consecutive m (coalesced). Forward and dX GEMMs.
  //   f = (+bias[m]) -> (relu) -> (* (mask[n*ldmask+m] > 0)), optional sums over n (bias grads).
  EPI_TRANSPOSED = 0,
  // out[m * ldo + n] = acc[m][n] — each lane owns a row run. dW GEMMs, fused with the gradient push.
  EPI_ROWMAJOR_PUSH = 1,
};

struct GemmParams {
  int M, N, K;          // real extents (tiles are masked against them)
  int bn;               // N tile, multiple of 16, <= 256
  int stages;           // smem ring depth
  int kc_per_split;     // k-chunks handled per blockIdx.z
  int epi;              // GemmEpilogue
  int out_bf16;         // EPI_TRANSPOSED: output element type (0 = fp32, 1 = bf16)
  int relu;
  int ldo;
  int ldmask;
  int mask_bf16;
  void* out;            // EPI_TRANSPOSED destination
  const float* bias;    // [M] or null (may be a peer pointer into the PS arena)
  const void* mask;     // [N][ldmask] activations (relu' = mask > 0) or null
  PushTarget colsum;    // EPI_TRANSPOSED: optional sum over n of the stored value -> vector[m] (bias grads)
  uint64_t colsum_offset;  // element offset of the vector inside colsum.base
  int colsum_item_base; // flag item index of mtile 0 of the vector
  int has_colsum;
  PushTarget push;      // EPI_ROWMAJOR_PUSH destination
  uint64_t push_offset; // element offset of the variable inside push.base
  int push_item_base;   // first flag item index for this variable's tiles (tile = mtile * ntiles + ntile)
  int push_staged;      // 1: transpose the dW tile through smem so each warp store covers whole 256-byte row runs
  uint32_t* bump_seq;   // if set, CTA (0,0,0) opens a new push sequence number for this step: it draws
  uint32_t* seq_counter;//   atomicAdd(seq_counter, 1) + 1 and stores it to *bump_seq (the step lane's seq word,
                        //   which every later kernel of the same step reads through PushTarget::seq_ptr)
  float* splitk_scratch;     // gridDim.z > 1: [mtiles][splits][128][bn] fp32 partial tiles
  uint32_t* splitk_counter;  // gridDim.z > 1: [mtiles] arrival counters (self-resetting)
  long long* debug_ts;       // optional: 9 clock64() phase stamps of CTA (0,0,0); null in production
  int splitk_cluster;        // 1: the gridDim.z splits of a tile form one thread-block cluster and reduce
  int pdl;                   //    their partial accumulators through distributed shared memory
                             // pdl = 1: launch with programmatic stream serialization (prologue overlaps the
                             //    previous kernel of the step; data reads wait on griddepcontrol.wait)
  int pad2_, pad3_;
};

// Softmax-cross-entropy head (last dense layer + loss + its gradients), see head_sm90.cu
enum LossKind : int {
  LOSS_BOOK = 0,  // -mean over B x C of labels * log(clip(softmax, 1e-10, 1))   (reference DS:52-53)
  LOSS_XENT = 1,  // mean over B of softmax_cross_entropy_with_logits               (reference DS:35)
};

struct StepResult {  // written once per worker step, read back by the host (D2H)
  float loss;
  uint32_t global_step;
  uint32_t correct;   // argmax(logits) == argmax(labels) count over the batch (accuracy numerator)
  uint32_t seq;       // push sequence number of this step
};

struct HeadParams {
  int B;            // real batch
  int B_pad;        // rows allocated in h / dpre (multiple of 16)
  int H;            // last hidden width
  int C;            // classes
  int loss_kind;
  int act_bf16;     // h / dpre element type
  int ldh;
  int compute_grads;  // 0 = eval only (loss + accuracy)
  const void* h;        // [B_pad][ldh]
  const float* labels;  // [B_pad][C] one-hot (or soft) labels
  const float* w_last;  // [C][H] fp32 master on the PS (peer pointer)
  const float* b_last;  // [C]
  void* dpre;           // [B_pad][ldh] gradient wrt last hidden pre-activation (relu' applied)
  PushTarget push;      // dW_last   — each small gradient goes to the shard that owns its variable
  PushTarget push_bl;   // db_last     (round-robin placement puts sm_w and sm_b on different ps tasks)
  PushTarget push_bh;   // db of the last hidden layer
  uint64_t off_w_last, off_b_last, off_b_hidden;
  int item_w_last_base; // + blockIdx.x
  int item_b_last;
  int item_b_hidden_base;  // + blockIdx.x
  int pdl;                 // 1: launch with programmatic stream serialization (see GemmParams::pdl)
  StepResult* result;      // device buffer (copied D2H by the step graph)
  // PS bookkeeping
  uint32_t* seq_ptr;         // local; bumped by the first kernel of the step (GemmParams::bump_seq), read here
  const uint32_t* inbox;     // local [n_inbox][2] = {ack_seq, global_step} per PS shard, written by the PS; or null
  uint32_t* ps_global_step;  // peer pointer (atomic mode: atom.add; local mode: null)
  uint32_t nslots;
  uint32_t n_inbox;          // number of PS shards this worker pushes to
  long long* debug_ts;       // optional clock64() phase stamps of CTA 0; null in production
};

// One unit of PS apply work.
struct PsItem {
  uint64_t offset;  // element offset inside the arena
  int rows, cols;
  int ld;
  int flags;        // bit0: refresh bf16 shadow for this block
  int flag_index;   // which of the worker's per-push flags announces this block (several items may share one
  int pad_;         //   flag: a pushed tile is applied by several ps CTAs, one sub-block each)
};

struct PsItemState {  // persisted across serve-kernel launches and checkpointed
  uint32_t t;        // number of pushes applied to this item (Adam step count)
  float beta1_pow;
  float beta2_pow;
  uint32_t sched_step;  // pushes applied to this item under a non-constant learning-rate schedule or with moving
                        // averages on: the schedule step, and TF1's num_updates of ExponentialMovingAverage
                        // (set to the restored global_step by a checkpoint restore)
};

// TF1 `training_ops` rules applied per push (or per round, APPLY_MERGED). Slot buffers: adam_m = Adam m / momentum
// accumulator / RMSProp mom / Adadelta accum_update / FTRL linear; adam_v = Adam v / Adagrad accumulator / RMSProp ms /
// Adadelta accum / FTRL accum / ProximalAdagrad accumulator. ProximalGradientDescent has no slot.
enum OptimizerKind : int {
  OPT_SGD = 0,
  OPT_ADAM = 1,
  OPT_MOMENTUM = 2,
  OPT_ADAGRAD = 3,
  OPT_RMSPROP = 4,
  OPT_ADADELTA = 5,
  OPT_FTRL = 6,
  OPT_PROXIMAL_ADAGRAD = 7,
  OPT_PROXIMAL_SGD = 8,
};
enum ApplyMode : int {
  APPLY_PER_PUSH = 0,  // reference semantics: every worker push is its own optimizer step
  APPLY_MERGED = 1,    // pushes that are ready at the same poll are summed and applied as one step
};

constexpr int kMaxLrBoundaries = 8;   // PsServeParams::boundaries (piecewise_constant)

struct PsServeParams {
  float* params;
  float* adam_m;
  float* adam_v;
  uint16_t* shadow_bf16;       // null if unused
  const PsItem* items;
  PsItemState* item_state;
  int n_items;
  int n_flags;                 // flags per (worker, slot); PsItem::flag_index < n_flags
  int n_workers;
  int nslots;
  int opt;
  int apply_mode;
  float lr, beta1, beta2, eps;
  const float* mailbox;        // [n_workers][nslots][arena_elems]
  uint64_t arena_elems;
  uint32_t* flags;             // [n_workers][nslots][n_flags]
  uint32_t* next_seq;          // [n_workers][n_items] next expected push seq (persisted)
  uint32_t* consumed;          // [n_workers][nslots] items consumed of the in-flight push
  uint32_t* global_step;       // shard-local step counter (only shard 0's is authoritative)
  uint32_t* worker_done;       // [n_workers] set remotely by workers when they leave the session
  volatile uint32_t* host_stop;  // host-mapped stop request
  // Table (in the PS's own memory) of peer pointers to each worker's inbox {ack_seq, global_step}; the host
  // patches entries while the kernel runs when a worker attaches late, so it is read with volatile loads.
  uint32_t* volatile* inbox_table;
  uint32_t* exit_counter;      // CTAs increment on exit (debug / clean shutdown)
  uint32_t gpu_scope;          // 1: every worker runs on the PS's own GPU (flags / acks at gpu scope)
  uint32_t lookahead;          // max pushes of one worker consumed per item pass (0 = auto: up to nslots)
  uint32_t oneshot;            // 1: apply whatever is pending and exit after the first full sweep that finds nothing
  uint32_t ieee_math;          //    (stream-ordered after the workers' kernels: profiler / sanitizer safe)
                               // ieee_math 1: correctly rounded sqrt / divide in Adam, Adagrad and RMSProp
                               //   (`--adam_math ieee`)
  // Optional per-CTA serve statistics [kPsStatsCtas][8] (accumulated over launches, written when a CTA exits):
  // passes with work, pushes applied, cycles in apply, cycles in bookkeeping, idle poll rounds, cycles idle,
  // largest number of pushes taken in one pass, poll cycles of working passes; then [kPsStatsCtas] the SM each CTA
  // of the last launch ran on. Null = off.
  unsigned long long* stats;
  // hyper-parameters of the rules after Adam / SGD (appended, so that no earlier field moves); `eps` above is also
  // RMSProp's epsilon
  float momentum;              // OPT_MOMENTUM, OPT_RMSPROP
  float decay;                 // OPT_RMSPROP (TF1 `decay`), OPT_ADADELTA (TF1 `rho`)
  uint32_t nesterov;           // OPT_MOMENTUM: 1 = use_nesterov
  uint32_t pad_;
  // learning-rate schedule (TF1 tf.train.*_decay / piecewise_constant; appended, so that no earlier field moves).
  // The rate of a push is lr(s), s = the item's PsItemState::sched_step when the push is applied; `lr` above is lr0.
  int lr_schedule;             // LrScheduleKind; LR_CONSTANT runs the unscheduled instantiations
  uint32_t decay_steps;        // > 0 for every decay schedule
  float decay_rate;            // exponential / inverse_time / natural_exp
  float end_lr;                // polynomial: end_learning_rate
  float power;                 // polynomial
  float alpha;                 // cosine: floor of the rate as a fraction of lr0
  uint32_t staircase;          // exponential / inverse_time / natural_exp: p = floor(s / decay_steps)
  uint32_t cycle;              // polynomial
  int n_boundaries;            // piecewise: 1 .. kMaxLrBoundaries
  uint32_t boundaries[kMaxLrBoundaries];  // piecewise: strictly increasing steps
  float values[kMaxLrBoundaries + 1];     // piecewise: n_boundaries + 1 rates
  // exponential moving averages of the parameters (TF1 tf.train.ExponentialMovingAverage.apply, zero_debias=False;
  // appended, so that no earlier field moves). After every optimizer step of an element:
  //   shadow -= (shadow - p) * (1 - d),  d = min(ema_decay, (1 + n) / (10 + n))  (d = ema_decay without num_updates)
  // with n = the item's pushes applied, this step's included (PsItemState::sched_step after the step).
  float* ema;                  // [arena] shadow variables of the fp32 parameters; null = off (unaveraged kernels)
  float ema_decay;
  uint32_t ema_num_updates;    // 1: d warms up with n (TF1 num_updates=global_step); 0: d = ema_decay
  // hyper-parameters of FTRL and the proximal rules (appended, so that no earlier field moves); `eps` above is also
  // Adadelta's epsilon, `decay` its rho
  float l1;                    // OPT_FTRL, OPT_PROXIMAL_ADAGRAD, OPT_PROXIMAL_SGD: l1_regularization_strength (>= 0)
  float l2;                    //   the same three: l2_regularization_strength (>= 0)
  float l2_shrinkage;          // OPT_FTRL: l2_shrinkage_regularization_strength (>= 0; 0 = ApplyFtrl, else ApplyFtrlV2)
  float lr_power;              // OPT_FTRL: learning_rate_power (<= 0; -0.5 takes the square-root path)
};
enum LrScheduleKind : int {
  LR_CONSTANT = 0,
  LR_EXPONENTIAL = 1,
  LR_INVERSE_TIME = 2,
  LR_NATURAL_EXP = 3,
  LR_POLYNOMIAL = 4,
  LR_COSINE = 5,
  LR_PIECEWISE = 6,
};
constexpr int kPsStatsCtas = 160;

// ------------------------------------------------------------------------------------------------
// Fused worker step (fused_step_sm90.cu): one 8-CTA thread-block cluster runs whole training steps of the
// 784-H-10 MLP (H <= 128, batch <= 256) back to back inside one launch: TMA pull of its K-slice of W from the ps
// shard, wgmma forward (split-K over the cluster, DSMEM reduce-scatter), classifier head, DSMEM all-gather of
// the pre-activation gradient, wgmma dW of its own column slice, gradient push + flag. `lanes` clusters of one
// launch work on different steps concurrently.
// ------------------------------------------------------------------------------------------------
constexpr int kFusedCluster = 8;
constexpr int kFusedMaxChunks = 4;   // 32-feature k-chunks per CTA  (in_features <= 8 * 4 * 32)
constexpr int kFusedMaxShards = 8;
constexpr uint32_t kFusedNoStep = 0xFFFFFFFFu;
constexpr int kLaneRecWords = 16;   // FusedParams::lane_rec: [0, 8) SM ids, 8 steps, 9 first claim, 10 end, 11 entry

struct FusedSlice {        // what CTA `rank` of every cluster owns
  int kc_begin;            // first k-chunk (x 32 input features)
  int kc_count;            // 0 .. kFusedMaxChunks
  int shard;               // index into FusedParams::shard of the ps shard that owns this column slice of W
  int flag_index;          // flag (on that shard) announcing this CTA's dW tile
  uint64_t w_offset;       // element offset of the hidden weight inside that shard's arena
};

struct FusedShard {        // one ps shard this worker pushes to
  PushTarget push;         // mailbox / flags / mode of this worker on that shard (seq_ptr unused)
  const uint32_t* inbox;   // local {ack_seq, global_step} pair the shard writes; null in atomic mode
};

struct FusedParams {
  int B, H, C, I;          // batch (<= 32), hidden units (<= 128), classes (<= 11), input features
  int loss_kind;
  int ldw;                 // leading dimension of the hidden weight in the arena
  int n_shards;
  int strict;              // 1: pull W for a step only after every shard acknowledged this lane's previous push
  FusedSlice slice[kFusedCluster];
  FusedShard shard[kFusedMaxShards];
  // small variables: where they live (peer pointers into the owning shard's params) and where their grads go
  const float* bias_h; const float* w_last; const float* b_last;
  int shard_bh, shard_wl, shard_bl;          // FusedParams::shard index owning hid_b / sm_w / sm_b
  int flag_bh, flag_wl, flag_bl;             // their flag indices on those shards
  uint64_t off_bh, off_wl, off_bl;           // element offsets inside those shards' arenas
  // inputs: batch of step s = rows [(row_start + s * row_stride) % row_wrap, +B) of the x / y matrices (x is read in
  // whole 32-row tiles: the x map must cover round_up(B, 32) rows from there)
  const float* y_base;
  uint64_t row_start, row_stride, row_wrap;
  // bookkeeping
  uint32_t n_steps;        // steps of this launch (claimed dynamically by the clusters)
  uint32_t seq_base;       // push sequence number of step s is seq_base + s + 1
  uint32_t nslots;
  uint32_t stop_at;        // > 0: no further steps are claimed once a step reports global_step >= stop_at
  uint32_t* step_counter;  // device word: next unclaimed step of the launch; the last cluster to exit zeroes it again
  uint32_t* stop_word;     // device word, zeroed by the last cluster to exit when `clear_stop` is set
  uint32_t* seq_word;      // device word: total pushes made by this worker (advanced at the end of every step)
  uint32_t* ps_global_step;  // atomic mode: peer pointer to the shared step counter
  StepResult* results;     // [n_steps] pinned host memory, written by the kernel
  long long* debug_ts;     // optional phase stamps of cluster 0 / CTA 0
  // optional lane residency record, [lanes][kLaneRecWords] (null in production): the SM of each CTA of the cluster,
  // then steps the cluster claimed, globaltimer at its first claim, after its last step, and at kernel entry
  unsigned long long* lane_rec;
  uint32_t* exit_counter;  // device word: clusters that have finished (self-resetting)
  uint32_t clear_stop;     // 1: the last cluster to exit zeroes *stop_word (last launch of a run)
  uint32_t wait_acks;      // 1: the last cluster to exit returns only after every shard has acknowledged every push made
                           //    so far (the launch then covers the ps-side apply of its last step: timed regions)
  // gradient clipping before the push (TF1 clip_by_global_norm / clip_by_norm per variable / clip_by_value; appended,
  // so that no earlier field moves). CLIP_OFF runs the unclipped instantiations.
  int clip_kind;           // GradClipKind
  float clip_norm;         // CLIP_GLOBAL_NORM, CLIP_NORM: > 0
  float clip_min, clip_max;  // CLIP_VALUE
  // L2 weight regularization (TF1 loss + l2_scale * sum l2_loss(v); appended): g' = fl(g + fl(l2_scale * w)) for the
  // weights (and, with l2_biases, the biases) before the clip. 0 runs the unregularized instantiations.
  float l2_scale;          // finite, >= 0
  uint32_t l2_biases;      // 1: the biases are regularized too
};
enum GradClipKind : int {
  CLIP_OFF = 0,
  CLIP_GLOBAL_NORM = 1,
  CLIP_NORM = 2,
  CLIP_VALUE = 3,
};

// Gradient clipping tail of the graph engine (clip_sm90.cu): the step's epilogues push into worker-local buffers, these
// kernels clip them into this worker's mailbox slot on every shard and release the slot's flags.
constexpr int kGradClipMaxVars = 8;
constexpr int kGradClipMaxShards = 16;
constexpr int kGradClipBlocks = 132;     // blocks of the sum-of-squares and apply kernels (partials: [blocks][vars])
struct GradClipVar {
  float* local;                  // the variable in this slot's local gradient buffer (arena layout of its shard)
  float* mailbox;                // the variable in slot 0 of this worker's mailbox on its shard
  uint64_t mailbox_slot_stride;  // elements between mailbox slots (the shard's arena)
  uint32_t rows, cols, ld, pad_;
};
struct GradClipParams {
  int kind;                      // GradClipKind (not CLIP_OFF)
  float clip_norm, clip_min, clip_max;
  int n_vars, n_shards;
  uint32_t nslots;               // mailbox slots: the slot of push seq is seq % nslots
  uint32_t gpu_scope;            // 1: every shard is on this GPU (gpu-scope fence suffices)
  const uint32_t* seq_ptr;       // this ring slot's current push sequence number
  float* partials;               // [kGradClipBlocks][kGradClipMaxVars] worker-local scratch
  GradClipVar var[kGradClipMaxVars];
  uint32_t* flags[kGradClipMaxShards];          // slot-0 flags of this worker on each shard
  uint32_t flag_slot_stride[kGradClipMaxShards];
  uint32_t n_flags[kGradClipMaxShards];
  // L2 weight regularization (appended; the tail runs with l2_scale != 0 even when kind is CLIP_OFF): g' = fl(local +
  // fl(l2_scale * w)) before the clip for every variable with an l2_w, and loss += l2_scale * sum(w*w) / 2
  const float* l2_w[kGradClipMaxVars];          // the variable's fp32 values on its shard (nullptr: not regularized)
  float l2_scale;
  uint32_t l2_pad_;
  float* l2_partials;                           // [kGradClipBlocks][kGradClipMaxVars] worker-local scratch: sums of w*w
  StepResult* result;                           // this ring slot's step result (the head has written the data loss)
};

}  // namespace dm
