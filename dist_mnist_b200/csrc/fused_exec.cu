// Native worker-side executor for the fused step kernel (fused_step_sm90.cu).
//
// The reference worker loop is `next_batch(32)` -> `sess.run(train_op, feed_dict)` -> read loss / global_step
// (/root/reference/distributed_server-basic.py:110-116). Here the steps themselves run inside one persistent
// kernel launch per *chunk* of steps; the executor's job is to keep that kernel fed:
//
//   gather pool  persistent helper threads run the `next_batch` loader (row gather into pinned staging memory;
//                DRAM-latency bound, ~20 us per batch on one core) — created once, spinning only while a run is
//                active, parked on a condition variable otherwise. No thread is spawned per call.
//   chunks       a run of n steps is cut into chunks (4, 8, 16, 16, ... steps). Chunk c: gather -> one H2D copy of
//                its x rows + one of its labels into a device ring buffer (copy stream) -> event -> one launch of
//                the fused kernel for the chunk's steps (compute stream). Four chunk buffers rotate, so the gather
//                and the transfer of chunk c+1 overlap the kernel of chunk c.
//   epoch feed   with a loader whose epoch feed is enabled (loader.h) no row is gathered on the training thread at all:
//                the current epoch's rows sit in permutation order in a pinned buffer, so a chunk that does not
//                straddle an epoch boundary is ONE contiguous H2D copy straight out of that buffer, issued as soon
//                as the chunk's ring buffer is free. The helper threads fill the next epoch's buffer in the
//                background (low priority: they serve gather tasks first); only the chunk that contains the boundary
//                goes through the gather path above.
//   results      every step's {loss, global_step, correct, seq} is written by the kernel straight into pinned host
//                memory (posted PCIe write); a chunk's results are valid once its completion event has fired.
//   resident     `run_resident`: one launch for any number of steps over a device-resident dataset (the kernel's TMA
//                reads the batch rows directly out of the dataset; no staging copies at all).
//
// Everything is stream ordered — there is no kernel that waits for the host — so the path is safe under profilers
// and sanitizers that serialise kernels.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdlib>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "fused.h"
#include "loader.h"
#include "trace.h"

namespace {

thread_local std::string g_fx_err;

int fxfail(const char* what, cudaError_t e) {
  g_fx_err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
  return -1;
}
#define FX_CUDA(call)                                   \
  do {                                                  \
    cudaError_t e__ = (call);                           \
    if (e__ != cudaSuccess) return fxfail(#call, e__);  \
  } while (0)

inline void cpu_relax() {
#if defined(__x86_64__)
  __builtin_ia32_pause();
#endif
}

// ---------------------------------------------------------------------------------------------
// persistent gather pool
// ---------------------------------------------------------------------------------------------
struct GatherTask {
  const dm::BatchLoader* loader;
  std::shared_ptr<std::vector<uint32_t>> idx;   // batch row indices (planned by the submitting thread: the loader
                                                // stays sequential); shared by the sub-tasks of one batch
  int r0, r1;                   // rows of the batch this task copies (a batch is split over several threads: the
                                // gather is DRAM-latency bound, ~2 us per 3 KB row)
  uint8_t* x_dst;
  uint8_t* y_dst;
  std::atomic<uint32_t>* done;  // += rows copied
};

// Background job: materialise one epoch of the loader's epoch feed (rows idx[0..n) of the dataset, in that order, into
// x_dst / y_dst). Threads claim blocks of kFillBlock rows; between blocks they go back to the gather queue first.
constexpr uint32_t kFillBlock = 64;
struct FillJob {
  const dm::BatchLoader* loader;
  std::shared_ptr<std::vector<uint32_t>> idx;
  uint8_t* x_dst;
  uint8_t* y_dst;
  uint32_t n;
  std::atomic<uint32_t> next{0};   // first unclaimed row
  std::atomic<uint32_t>* done;     // += rows copied (BatchLoader::feed_rows[b])
};

struct GatherPool {
  std::vector<std::thread> threads;
  std::mutex mu;
  std::condition_variable cv;
  std::deque<GatherTask*> queue;
  std::deque<std::shared_ptr<FillJob>> fills;
  std::atomic<bool> fill_active{false};
  std::atomic<int> active{0};     // > 0 while some run is in progress: workers spin instead of sleeping
  std::atomic<uint64_t> posted{0}, taken{0};
  bool quit = false;
  int spin_grace_ms = 1;

  void start(int n) {
    for (int t = 0; t < n; ++t) threads.emplace_back([this] { loop(); });
  }
  void stop() {
    {
      std::lock_guard<std::mutex> lk(mu);
      quit = true;
    }
    cv.notify_all();
    for (auto& t : threads) t.join();
    threads.clear();
  }
  GatherTask* try_pop() {
    if (taken.load(std::memory_order_acquire) >= posted.load(std::memory_order_acquire)) return nullptr;
    std::lock_guard<std::mutex> lk(mu);
    if (queue.empty()) return nullptr;
    GatherTask* t = queue.front();
    queue.pop_front();
    taken.fetch_add(1, std::memory_order_release);
    return t;
  }
  void post(GatherTask* t) {
    {
      std::lock_guard<std::mutex> lk(mu);
      queue.push_back(t);
      posted.fetch_add(1, std::memory_order_release);
    }
    cv.notify_one();
  }
  void post_fill(std::shared_ptr<FillJob> j) {
    {
      std::lock_guard<std::mutex> lk(mu);
      fills.push_back(std::move(j));
      fill_active.store(true, std::memory_order_release);
    }
    cv.notify_all();
  }
  // One block of the oldest fill job; false when there is no fill work. Any thread may call it (the training thread
  // does while it waits for an epoch buffer).
  bool fill_step() {
    if (!fill_active.load(std::memory_order_acquire)) return false;
    std::shared_ptr<FillJob> j;
    {
      std::lock_guard<std::mutex> lk(mu);
      if (fills.empty()) { fill_active.store(false, std::memory_order_release); return false; }
      j = fills.front();
    }
    const uint32_t r0 = j->next.fetch_add(kFillBlock, std::memory_order_relaxed);
    if (r0 >= j->n) {   // every block is claimed (some may still be in flight on other threads): retire the job
      std::lock_guard<std::mutex> lk(mu);
      if (!fills.empty() && fills.front() == j) fills.pop_front();
      if (fills.empty()) fill_active.store(false, std::memory_order_release);
      return true;
    }
    const uint32_t r1 = std::min(j->n, r0 + kFillBlock);
    j->loader->copy_rows(j->idx->data(), static_cast<int>(r0), static_cast<int>(r1), j->x_dst, j->y_dst);
    j->done->fetch_add(r1 - r0, std::memory_order_release);
    return true;
  }
  static void run_task(GatherTask* t) {
    t->loader->copy_rows(t->idx->data(), t->r0, t->r1, t->x_dst, t->y_dst);
    std::atomic<uint32_t>* d = t->done;
    const uint32_t rows = static_cast<uint32_t>(t->r1 - t->r0);
    delete t;
    d->fetch_add(rows, std::memory_order_release);
  }
  void loop() {
    // Spin while a run is active and for a grace period after the last one (a training loop calls run() back to back:
    // waking a parked thread costs tens of microseconds — more than gathering a whole batch); park on the condition
    // variable only when the executor has really gone idle.
    auto last_active = std::chrono::steady_clock::now();
    for (;;) {
      GatherTask* t = try_pop();
      if (t != nullptr) { run_task(t); last_active = std::chrono::steady_clock::now(); continue; }
      if (fill_step()) { last_active = std::chrono::steady_clock::now(); continue; }
      if (active.load(std::memory_order_acquire) > 0) { cpu_relax(); last_active = std::chrono::steady_clock::now(); continue; }
      if (std::chrono::steady_clock::now() - last_active < std::chrono::milliseconds(spin_grace_ms)) { cpu_relax(); continue; }
      std::unique_lock<std::mutex> lk(mu);
      cv.wait(lk, [this] { return quit || !queue.empty() || !fills.empty() || active.load(std::memory_order_acquire) > 0; });
      if (quit && queue.empty() && fills.empty()) return;   // posted work is always finished, also during shutdown
      last_active = std::chrono::steady_clock::now();
    }
  }
};

constexpr int kChunkMax = 16;   // steps per chunk buffer
constexpr int kBuffers = 4;     // chunk buffers in rotation
constexpr int kRowTile = 32;         // rows of one row tile of the fused kernel
constexpr int kMaxBatch = 256;       // 8 row tiles
constexpr int kRowsPerTask = 8;   // rows of a batch gathered by one pool task

struct ChunkBuf {
  cudaEvent_t copied = nullptr, done = nullptr;
  std::atomic<uint32_t> gathered{0};
  uint32_t n = 0;              // steps of the chunk currently occupying the buffer
  bool in_flight = false;
  bool direct = false;         // fed straight from the loader's epoch buffer: its H2D copies are already enqueued
  uint64_t first_step = 0;     // index (within the run) of the chunk's first step
};

struct FusedExec {
  int device = 0, lanes = 1, n_threads = 4;
  int I = 0, C = 0, batch = 0;
  int rows = 0;                // rows of a ring slot: the batch rounded up to whole 32-row tiles (rows >= batch zero)
  size_t x_slot_bytes = 0, y_slot_bytes = 0;
  uint8_t *x_dev = nullptr, *y_dev = nullptr, *x_stage = nullptr, *y_stage = nullptr;
  dm::StepResult* res_chunks = nullptr;   // pinned [kBuffers][kChunkMax]
  dm::StepResult* res_big = nullptr;      // pinned, grown on demand (run_resident / single steps)
  size_t res_big_cap = 0;
  uint32_t* ctl_dev = nullptr;            // [0] step counter, [1] stop word, [2] seq word (pushes made)
  uint32_t* zeros_pin = nullptr;          // pinned zeros: control words are reset with a DMA copy, never a memset —
                                          // a memset may be a driver kernel whose lazy first load deadlocks against
                                          // a resident persistent ps kernel
  cudaStream_t compute = nullptr, copy = nullptr;
  dm::FusedMaps maps{};
  dm::FusedParams params{};
  bool have_params = false;
  bool warmed = false;
  uint64_t steps_done = 0;    // steps completed over the executor's lifetime == push sequence numbers used
  uint64_t launches = 0;
  uint64_t direct_chunks = 0, gathered_chunks = 0, fills_posted = 0;   // feed statistics (dm_fexec_feed_stats)
  bool feed_broken = false;   // a copy out of an epoch buffer was refused: this executor stays on the row-gather path
  ChunkBuf bufs[kBuffers];
  GatherPool pool;
  cudaEvent_t feed_read[2] = {nullptr, nullptr};     // epoch feed: last H2D copy that reads epoch buffer b (copy stream)
  bool feed_read_valid[2] = {false, false};
  cudaEvent_t t_start = nullptr, t_stop = nullptr;   // timing events of a timed resident launch
  cudaEvent_t last_done = nullptr;  // completion of the most recent launch
  uint64_t last_n = 0;              // steps requested by the most recent resident launch
  dm::StepResult* last_results = nullptr;

  // The kernel re-arms its own launch state (step counter, exit counter, optionally the stop word) when its last cluster
  // exits, so a launch is exactly one stream operation. `clear_stop`: last launch of a run; `wait_acks`: the launch
  // returns only after the ps has applied every push made so far.
  int launch(const dm::FusedMaps& m, dm::FusedParams p, uint32_t n_steps, dm::StepResult* results, uint32_t stop_at,
             bool clear_stop, bool wait_acks = false) {
    p.n_steps = n_steps;
    p.seq_base = static_cast<uint32_t>(steps_done);
    p.stop_at = stop_at;
    p.step_counter = ctl_dev;
    p.stop_word = ctl_dev + 1;
    p.seq_word = ctl_dev + 2;
    p.exit_counter = ctl_dev + 3;
    p.clear_stop = clear_stop ? 1u : 0u;
    p.wait_acks = wait_acks ? 1u : 0u;
    p.results = results;
    FX_CUDA(dm::launch_fused_step(m, p, lanes, compute));
    ++launches;
    return 0;
  }
  int ensure_big(size_t n) {
    if (n <= res_big_cap) return 0;
    if (res_big) cudaFreeHost(res_big);
    res_big = nullptr;
    res_big_cap = 0;
    size_t cap = 1024;
    while (cap < n) cap <<= 1;
    FX_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&res_big), cap * sizeof(dm::StepResult),
                          cudaHostAllocMapped | cudaHostAllocPortable));
    res_big_cap = cap;
    return 0;
  }
};

// Epoch feed: start materialising epoch `epochs + 1` into its buffer once that buffer is free — the fill of the epoch
// that used it before has completed and no H2D copy is still reading it (every copy out of it was enqueued on the copy
// stream before the loader crossed into the current epoch). Called often; does nothing most of the time.
// Returns -1 on a CUDA error.
int maybe_post_fill(FusedExec* ex, dm::BatchLoader* ld) {
  const uint64_t e1 = ld->epochs + 1;
  const int nb = static_cast<int>(e1 & 1);
  if (ld->feed_epoch[nb] == e1) return 0;   // already posted
  // whatever was last materialised in that buffer (normally epoch e1 - 2, long complete) must be complete: two fill
  // jobs never write one buffer at the same time
  if (ld->feed_epoch[nb] != dm::BatchLoader::kNoEpoch && ld->feed_rows[nb].load(std::memory_order_acquire) < ld->n) return 0;
  // ... and no H2D copy may still be reading it: every copy out of that buffer was enqueued before the loader crossed
  // into the current epoch, the last of them followed by feed_read[nb]. (Asking whether the whole copy stream is idle
  // would almost never succeed in a pipelined run: the current epoch's copies keep it busy.)
  if (ex->feed_read_valid[nb]) {
    const cudaError_t q = cudaEventQuery(ex->feed_read[nb]);
    if (q == cudaErrorNotReady) { cudaGetLastError(); return 0; }
    if (q != cudaSuccess) return fxfail("cudaEventQuery(feed_read)", q);
    ex->feed_read_valid[nb] = false;
  }
  auto j = std::make_shared<FillJob>();
  j->loader = ld;
  j->idx = ld->draw_next_perm();
  j->x_dst = ld->feed_x[nb];
  j->y_dst = ld->feed_y[nb];
  j->n = static_cast<uint32_t>(ld->n);
  j->done = &ld->feed_rows[nb];
  ld->feed_epoch[nb] = e1;
  ld->feed_rows[nb].store(0, std::memory_order_release);
  ex->pool.post_fill(std::move(j));
  ++ex->fills_posted;
  dm::nvtx_mark("dm.fexec.epoch_fill.posted");
  return 0;
}

}  // namespace

extern "C" {

const char* dm_fexec_last_error() { return g_fx_err.c_str(); }

int dm_fexec_create(int device, int lanes, int I, int C, int batch, void** out) {
  FX_CUDA(cudaSetDevice(device));
  if (lanes < 1 || batch < 1 || batch > kMaxBatch || (I & 3) != 0) {
    g_fx_err = "fused executor: need lanes >= 1, 1 <= batch <= 256, in_features % 4 == 0";
    return -1;
  }
  FusedExec* ex = new FusedExec();
  ex->device = device;
  ex->lanes = lanes;
  ex->I = I;
  ex->C = C;
  ex->batch = batch;
  ex->rows = (batch + kRowTile - 1) / kRowTile * kRowTile;
  ex->x_slot_bytes = static_cast<size_t>(ex->rows) * I * 4;
  ex->y_slot_bytes = static_cast<size_t>(ex->rows) * C * 4;
  const size_t slots = static_cast<size_t>(kBuffers) * kChunkMax;
  FX_CUDA(cudaMalloc(reinterpret_cast<void**>(&ex->x_dev), slots * ex->x_slot_bytes));
  FX_CUDA(cudaMalloc(reinterpret_cast<void**>(&ex->y_dev), slots * ex->y_slot_bytes));
  FX_CUDA(cudaMemset(ex->x_dev, 0, slots * ex->x_slot_bytes));
  FX_CUDA(cudaMemset(ex->y_dev, 0, slots * ex->y_slot_bytes));
  FX_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&ex->x_stage), slots * ex->x_slot_bytes, cudaHostAllocDefault));
  FX_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&ex->y_stage), slots * ex->y_slot_bytes, cudaHostAllocDefault));
  memset(ex->x_stage, 0, slots * ex->x_slot_bytes);
  memset(ex->y_stage, 0, slots * ex->y_slot_bytes);
  FX_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&ex->res_chunks), slots * sizeof(dm::StepResult),
                        cudaHostAllocMapped | cudaHostAllocPortable));
  memset(ex->res_chunks, 0, slots * sizeof(dm::StepResult));
  FX_CUDA(cudaMalloc(reinterpret_cast<void**>(&ex->ctl_dev), 64));
  FX_CUDA(cudaMemset(ex->ctl_dev, 0, 64));
  FX_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&ex->zeros_pin), 64, cudaHostAllocDefault));
  memset(ex->zeros_pin, 0, 64);
  FX_CUDA(cudaStreamCreateWithFlags(&ex->compute, cudaStreamNonBlocking));
  FX_CUDA(cudaStreamCreateWithFlags(&ex->copy, cudaStreamNonBlocking));
  for (auto& b : ex->bufs) {
    FX_CUDA(cudaEventCreateWithFlags(&b.copied, cudaEventDisableTiming));
    FX_CUDA(cudaEventCreateWithFlags(&b.done, cudaEventDisableTiming));
  }
  FX_CUDA(cudaEventCreateWithFlags(&ex->last_done, cudaEventDisableTiming));
  for (auto& e : ex->feed_read) FX_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  FX_CUDA(cudaEventCreate(&ex->t_start));
  FX_CUDA(cudaEventCreate(&ex->t_stop));
  if (ex->ensure_big(1u << 16) != 0) return -1;   // up front: no pinned allocation while a persistent ps kernel is resident
  if (const char* e = getenv("DM_GATHER_THREADS")) ex->n_threads = std::max(1, atoi(e));
  else ex->n_threads = static_cast<int>(std::min<unsigned>(8u, std::max(2u, std::thread::hardware_concurrency() / 4)));
  if (const char* e = getenv("DM_GATHER_SPIN_MS")) ex->pool.spin_grace_ms = std::max(0, atoi(e));
  ex->pool.start(ex->n_threads);
  *out = ex;
  return 0;
}

// Device / staging ring buffers: [kBuffers * kChunkMax slots][rows][I] fp32 and [..][rows][C] fp32 (rows: the batch
// rounded up to a multiple of 32), and the control words.
int dm_fexec_buffers(void* h, void** x_dev, void** y_dev, void** x_stage, void** y_stage, void** ctl_dev, int* slots) {
  FusedExec* ex = static_cast<FusedExec*>(h);
  *x_dev = ex->x_dev;
  *y_dev = ex->y_dev;
  *x_stage = ex->x_stage;
  *y_stage = ex->y_stage;
  *ctl_dev = ex->ctl_dev;
  *slots = kBuffers * kChunkMax;
  return 0;
}

// The launch template for steps fed through the ring: tensor maps over x_dev, y_base == y_dev, row geometry of the ring.
int dm_fexec_set_params(void* h, const void* maps, const void* params) {
  FusedExec* ex = static_cast<FusedExec*>(h);
  memcpy(&ex->maps, maps, sizeof(dm::FusedMaps));
  memcpy(&ex->params, params, sizeof(dm::FusedParams));
  ex->have_params = true;
  // Dry launch (0 steps: every cluster finds nothing to claim and exits). The first real launch of a kernel can make
  // the driver allocate per-context resources (local-memory pool for its stack frame, the device printf FIFO, cluster
  // launch state), which needs a context-wide synchronisation — and would deadlock once a persistent ps kernel is
  // resident on this GPU. Callers set the launch template before any ps kernel is started (Worker.prepare()).
  if (!ex->warmed) {
    if (ex->launch(ex->maps, ex->params, 0, ex->res_chunks, 0, true) != 0) return -1;
    FX_CUDA(cudaStreamSynchronize(ex->compute));
    --ex->launches;
    ex->warmed = true;
  }
  return 0;
}

void* dm_fexec_compute_stream(void* h) { return static_cast<FusedExec*>(h)->compute; }
uint64_t dm_fexec_steps_done(void* h) { return static_cast<FusedExec*>(h)->steps_done; }
uint64_t dm_fexec_launches(void* h) { return static_cast<FusedExec*>(h)->launches; }
int dm_fexec_lanes(void* h) { return static_cast<FusedExec*>(h)->lanes; }
// Clusters per launch from now on (steps of this worker in flight at once); the caller keeps it <= nslots.
int dm_fexec_set_lanes(void* h, int lanes) {
  if (lanes < 1) { g_fx_err = "set_lanes: lanes must be >= 1"; return -1; }
  static_cast<FusedExec*>(h)->lanes = lanes;
  return 0;
}
int dm_fexec_gather_threads(void* h) { return static_cast<FusedExec*>(h)->n_threads; }
// Epoch-feed statistics: chunks fed straight from an epoch buffer, chunks that went through the gather path, epoch
// fills posted to the helper threads.
void dm_fexec_feed_stats(void* h, uint64_t* direct_chunks, uint64_t* gathered_chunks, uint64_t* fills_posted) {
  FusedExec* ex = static_cast<FusedExec*>(h);
  *direct_chunks = ex->direct_chunks;
  *gathered_chunks = ex->gathered_chunks;
  *fills_posted = ex->fills_posted;
}

// Debug aid (hang analysis): control words {step counter, stop word, pushes made} read through a side stream while
// kernels may be running, plus seq / global_step of the first result slot of the chunk ring.
int dm_fexec_debug(void* h, uint32_t* out8) {
  FusedExec* ex = static_cast<FusedExec*>(h);
  cudaStream_t s;
  FX_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  uint32_t* pin = nullptr;
  FX_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&pin), 64, cudaHostAllocDefault));
  FX_CUDA(cudaMemcpyAsync(pin, ex->ctl_dev, 16, cudaMemcpyDeviceToHost, s));
  FX_CUDA(cudaStreamSynchronize(s));
  for (int i = 0; i < 4; ++i) out8[i] = pin[i];
  out8[4] = ex->res_chunks[0].seq;
  out8[5] = ex->res_chunks[0].global_step;
  out8[6] = static_cast<uint32_t>(ex->steps_done);
  out8[7] = cudaStreamQuery(ex->compute) == cudaSuccess ? 0u : 1u;
  cudaGetLastError();
  cudaFreeHost(pin);
  cudaStreamDestroy(s);
  return 0;
}

int dm_fexec_drain(void* h) {
  FusedExec* ex = static_cast<FusedExec*>(h);
  FX_CUDA(cudaStreamSynchronize(ex->copy));
  FX_CUDA(cudaStreamSynchronize(ex->compute));
  return 0;
}

// n steps (n <= kChunkMax) on host batches laid out like the staging ring (x [n][rows][I], y [n][rows][C]; rows >= batch
// zero): H2D + one launch + wait. Results to out[n]. The `step()` / `submit` path of the public API.
int dm_fexec_steps_host(void* h, const void* x_host, const void* y_host, uint32_t n, void* out, uint32_t* n_done) {
  FusedExec* ex = static_cast<FusedExec*>(h);
  if (!ex->have_params || n < 1 || n > kChunkMax) { g_fx_err = "steps_host: bad arguments"; return -1; }
  dm::NvtxRange nvtx_steps("dm.fexec.steps_host");
  FX_CUDA(cudaStreamSynchronize(ex->compute));   // buffer 0 must be free
  memcpy(ex->x_stage, x_host, n * ex->x_slot_bytes);
  memcpy(ex->y_stage, y_host, n * ex->y_slot_bytes);
  memset(ex->res_chunks, 0, n * sizeof(dm::StepResult));
  FX_CUDA(cudaMemcpyAsync(ex->x_dev, ex->x_stage, n * ex->x_slot_bytes, cudaMemcpyHostToDevice, ex->compute));
  FX_CUDA(cudaMemcpyAsync(ex->y_dev, ex->y_stage, n * ex->y_slot_bytes, cudaMemcpyHostToDevice, ex->compute));
  dm::FusedParams p = ex->params;
  p.row_start = 0;
  if (ex->launch(ex->maps, p, n, ex->res_chunks, 0, true) != 0) return -1;
  FX_CUDA(cudaStreamSynchronize(ex->compute));
  uint32_t done = 0;
  dm::StepResult* o = static_cast<dm::StepResult*>(out);
  for (uint32_t i = 0; i < n; ++i)
    if (ex->res_chunks[i].seq != 0) o[done++] = ex->res_chunks[i];
  ex->steps_done += done;
  if (n_done) *n_done = done;
  return 0;
}

// The native train loop: n_steps x { next_batch -> pinned staging -> H2D -> fused step -> result }, chunked and
// pipelined as described in the file header. stop_at_global_step > 0: StopAtStepHook semantics (reference DS:101) —
// no step is started once a finished step has reported global_step >= that value; *n_done = steps actually run.
// wait_acks != 0 (and no stop condition): the last chunk's launch returns only after the ps has acknowledged every push.
int dm_fexec_run(void* h, void* loader, uint64_t n_steps, void* out_results, uint32_t stop_at_global_step,
                 uint64_t* n_done, int wait_acks) {
  FusedExec* ex = static_cast<FusedExec*>(h);
  dm::BatchLoader* ld = static_cast<dm::BatchLoader*>(loader);
  dm::StepResult* out = static_cast<dm::StepResult*>(out_results);
  if (!ex->have_params) { g_fx_err = "run: launch template not set"; return -1; }
  if (ld->batch != ex->batch) { g_fx_err = "run: loader batch size differs from the executor's"; return -1; }
  dm::NvtxRange nvtx_run("dm.fexec.run");
  FX_CUDA(cudaSetDevice(ex->device));
  FX_CUDA(cudaStreamSynchronize(ex->compute));
  for (auto& b : ex->bufs) b.in_flight = false;
  // chunk schedule: a short first chunk gets the GPU going while the bigger ones are being gathered
  std::vector<uint32_t> sizes;
  {
    uint64_t left = n_steps;
    uint32_t sz = 4;
    while (left > 0) {
      const uint32_t n = static_cast<uint32_t>(std::min<uint64_t>(left, sz));
      sizes.push_back(n);
      left -= n;
      sz = std::min<uint32_t>(sz * 2, kChunkMax);
    }
  }
  // epoch feed usable with this executor's ring geometry: a slot is exactly one dense batch (the batch is a multiple of
  // 32 rows, so no slot has padding rows)
  bool feed_ok = ld->feed && !ex->feed_broken && ld->batch == ex->rows &&
                 ld->x_row_bytes * ex->rows == ex->x_slot_bytes && ld->y_row_bytes * ex->rows == ex->y_slot_bytes;
  const size_t nchunks = sizes.size();
  std::vector<uint64_t> first(nchunks + 1, 0);
  for (size_t c = 0; c < nchunks; ++c) first[c + 1] = first[c] + sizes[c];
  const bool trace = getenv("DM_FEXEC_TRACE") != nullptr;
  const auto t_begin = std::chrono::steady_clock::now();
  auto us_since = [&] { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_begin).count(); };
  // The helper threads are woken (and kept spinning for the rest of the run) only when a chunk actually needs rows
  // gathered: a run fed entirely from the epoch buffer never touches them — waking a dozen parked threads costs the
  // training thread tens of microseconds, a sizeable part of a 20-step call.
  bool pool_active = false;
  auto activate_pool = [&] {
    if (pool_active) return;
    pool_active = true;
    ex->pool.active.fetch_add(1, std::memory_order_release);
    ex->pool.cv.notify_all();
  };
  uint64_t total_done = 0;
  bool stop = false;
  size_t next_gather = 0, next_launch = 0, next_harvest = 0;
  int rc = 0;
  auto harvest = [&](size_t c, bool wait) -> int {   // 1 = harvested, 0 = not ready, -1 = error
    ChunkBuf& b = ex->bufs[c % kBuffers];
    if (wait) {
      if (cudaEventSynchronize(b.done) != cudaSuccess) return fxfail("cudaEventSynchronize", cudaGetLastError());
    } else {
      cudaError_t q = cudaEventQuery(b.done);
      if (q == cudaErrorNotReady) { cudaGetLastError(); return 0; }
      if (q != cudaSuccess) return fxfail("cudaEventQuery", q);
    }
    const dm::StepResult* r = ex->res_chunks + (c % kBuffers) * kChunkMax;
    for (uint32_t i = 0; i < b.n; ++i) {
      if (r[i].seq == 0) continue;   // never claimed (stop)
      if (out) out[total_done] = r[i];
      ++total_done;
      if (stop_at_global_step && r[i].global_step >= stop_at_global_step) stop = true;
    }
    b.in_flight = false;
    return 1;
  };
  while (next_launch < nchunks && !stop) {
    // ---- post gathers ahead (a buffer is free once the chunk that used it has been harvested) ----
    while (next_gather < nchunks && next_gather < next_launch + kBuffers - 1) {
      const size_t c = next_gather;
      ChunkBuf& b = ex->bufs[c % kBuffers];
      dm::NvtxRange nvtx_plan("dm.fexec.chunk.plan");
      if (b.in_flight) {
        while (next_harvest + kBuffers <= c) {   // the previous occupant must be complete before it is overwritten
          const int hr = harvest(next_harvest, true);
          if (hr < 0) { rc = -1; break; }
          ++next_harvest;
        }
        if (rc != 0 || stop) break;
      }
      b.n = sizes[c];
      b.first_step = first[c];
      b.gathered.store(0, std::memory_order_relaxed);
      b.in_flight = true;
      b.direct = false;
      const size_t slot0 = (c % kBuffers) * kChunkMax;
      memset(ex->res_chunks + slot0, 0, sizes[c] * sizeof(dm::StepResult));
      if (feed_ok) {
        const size_t rows = static_cast<size_t>(sizes[c]) * ld->batch;
        // the current epoch's buffer is still being filled (start of a run right after a boundary, or the consumer
        // is faster than the helpers): help finishing it — cheaper than gathering the same rows batch by batch
        if (ld->cursor + rows <= ld->n && ld->feed_fill_in_progress()) {
          const auto t_wait = std::chrono::steady_clock::now();
          while (ld->feed_fill_in_progress()) {
            if (ex->pool.fill_step()) continue;
            cpu_relax();
            // (all blocks are claimed, the last ones are in flight on helper threads: microseconds. The deadline only
            // keeps a stuck helper from stalling training — the chunk then takes the gather path.)
            if (std::chrono::steady_clock::now() - t_wait > std::chrono::seconds(2)) break;
          }
        }
        if (maybe_post_fill(ex, ld) != 0) { rc = -1; break; }
        if (ld->feed_slice_ready(rows)) {
          const int eb = static_cast<int>(ld->epochs & 1);
          cudaError_t e = cudaMemcpyAsync(ex->x_dev + slot0 * ex->x_slot_bytes, ld->feed_x[eb] + ld->cursor * ld->x_row_bytes,
                                          rows * ld->x_row_bytes, cudaMemcpyHostToDevice, ex->copy);
          if (e == cudaSuccess)
            e = cudaMemcpyAsync(ex->y_dev + slot0 * ex->y_slot_bytes, ld->feed_y[eb] + ld->cursor * ld->y_row_bytes,
                                rows * ld->y_row_bytes, cudaMemcpyHostToDevice, ex->copy);
          if (e == cudaSuccess) e = cudaEventRecord(b.copied, ex->copy);
          if (e == cudaSuccess) e = cudaEventRecord(ex->feed_read[eb], ex->copy);
          if (e == cudaSuccess) {
            ex->feed_read_valid[eb] = true;
            ld->skip_rows(rows);
            b.direct = true;
            b.gathered.store(static_cast<uint32_t>(rows), std::memory_order_release);
            ++ex->direct_chunks;
            ++next_gather;
            // nothing to wait for: launch what is planned before planning further ahead (the copies of the following
            // chunk are enqueued right after this chunk's launch and still overlap its kernel); planning three chunks
            // ahead first would only delay the first launch of a short run by the host time of six copy calls
            break;
          }
          // The runtime refused a copy out of the epoch buffer (a synchronous, non-sticky error: nothing was consumed
          // from the loader yet). Training must not die of an input-path optimisation: say so once, stay on the
          // row-gather path from here on — this chunk included (its ring slots are simply copied again, in order, on
          // the same stream).
          fprintf(stderr, "[dm] fused executor: epoch feed switched off (%s: %s); using the row-gather path\n",
                  cudaGetErrorName(e), cudaGetErrorString(e));
          cudaGetLastError();
          ex->feed_broken = true;
          ex->feed_read_valid[eb] = true;   // (conservative: an x copy may have been enqueued before the failure)
          cudaEventRecord(ex->feed_read[eb], ex->copy);
          feed_ok = false;
        }
      }
      ++ex->gathered_chunks;
      activate_pool();
      for (uint32_t i = 0; i < sizes[c]; ++i) {
        auto idx = std::make_shared<std::vector<uint32_t>>(ld->batch);
        ld->plan(idx->data());
        for (int r0 = 0; r0 < ld->batch; r0 += kRowsPerTask) {
          GatherTask* t = new GatherTask();
          t->loader = ld;
          t->idx = idx;
          t->r0 = r0;
          t->r1 = std::min(ld->batch, r0 + kRowsPerTask);
          t->x_dst = ex->x_stage + (slot0 + i) * ex->x_slot_bytes;
          t->y_dst = ex->y_stage + (slot0 + i) * ex->y_slot_bytes;
          t->done = &b.gathered;
          ex->pool.post(t);
        }
      }
      ++next_gather;
    }
    if (rc != 0 || stop) break;
    // ---- launch the next chunk as soon as its batches are in place (this thread helps gathering meanwhile) ----
    {
      const size_t c = next_launch;
      ChunkBuf& b = ex->bufs[c % kBuffers];
      dm::NvtxRange nvtx_launch("dm.fexec.chunk.launch");
      while (b.gathered.load(std::memory_order_acquire) < b.n * static_cast<uint32_t>(ld->batch)) {
        GatherTask* t = ex->pool.try_pop();
        if (t != nullptr) GatherPool::run_task(t);
        else cpu_relax();
      }
      const size_t slot0 = (c % kBuffers) * kChunkMax;
      cudaError_t e = cudaSuccess;
      if (!b.direct) {   // (a chunk fed from the epoch buffer had its copies enqueued when it was planned)
        e = cudaMemcpyAsync(ex->x_dev + slot0 * ex->x_slot_bytes, ex->x_stage + slot0 * ex->x_slot_bytes,
                            b.n * ex->x_slot_bytes, cudaMemcpyHostToDevice, ex->copy);
        if (e == cudaSuccess)
          e = cudaMemcpyAsync(ex->y_dev + slot0 * ex->y_slot_bytes, ex->y_stage + slot0 * ex->y_slot_bytes,
                              b.n * ex->y_slot_bytes, cudaMemcpyHostToDevice, ex->copy);
        if (e == cudaSuccess) e = cudaEventRecord(b.copied, ex->copy);
      }
      if (e == cudaSuccess) e = cudaStreamWaitEvent(ex->compute, b.copied, 0);
      if (e != cudaSuccess) { rc = fxfail("chunk transfer", e); break; }
      dm::FusedParams p = ex->params;
      p.row_start = static_cast<uint64_t>(slot0) * ex->rows;
      // seq_base of this chunk assumes every earlier chunk of the run completes all its steps; if one is cut short
      // by the stop condition the (persistent) stop word keeps every later chunk from claiming anything
      const uint64_t saved = ex->steps_done;
      ex->steps_done = saved + first[c];
      const int lrc = ex->launch(ex->maps, p, b.n, ex->res_chunks + slot0, stop_at_global_step,
                                 /*clear_stop=*/stop_at_global_step == 0,
                                 /*wait_acks=*/wait_acks != 0 && stop_at_global_step == 0 && c + 1 == nchunks);
      ex->steps_done = saved;
      if (lrc != 0) { rc = -1; break; }
      if (trace) fprintf(stderr, "[fexec] chunk %zu (%u steps) launched at +%.1f us\n", c, b.n, us_since());
      e = cudaEventRecord(b.done, ex->compute);
      if (e != cudaSuccess) { rc = fxfail("cudaEventRecord", e); break; }
      ++next_launch;
    }
    // ---- non-blocking harvest (keeps the stop condition timely) ----
    while (next_harvest < next_launch) {
      const int hr = harvest(next_harvest, false);
      if (hr < 0) { rc = -1; break; }
      if (hr == 0) break;
      ++next_harvest;
    }
    if (rc != 0) break;
  }
  // drain: batches gathered ahead of an early stop are dropped (their chunks were never launched)
  while (rc == 0 && next_harvest < next_launch) {
    if (harvest(next_harvest, true) < 0) { rc = -1; break; }
    ++next_harvest;
  }
  for (size_t c = next_launch; c < next_gather; ++c) {   // wait for outstanding gather tasks of unlaunched chunks
    ChunkBuf& b = ex->bufs[c % kBuffers];
    while (b.gathered.load(std::memory_order_acquire) < b.n * static_cast<uint32_t>(ld->batch)) {
      GatherTask* t = ex->pool.try_pop();
      if (t != nullptr) GatherPool::run_task(t);
      else cpu_relax();
    }
    b.in_flight = false;
  }
  if (pool_active) ex->pool.active.fetch_sub(1, std::memory_order_release);
  if (rc != 0) return rc;
  FX_CUDA(cudaStreamSynchronize(ex->compute));
  if (trace) fprintf(stderr, "[fexec] run of %llu steps drained at +%.1f us (%d gather threads)\n",
                     static_cast<unsigned long long>(n_steps), us_since(), ex->n_threads);
  if (stop_at_global_step != 0)   // the stop word had to survive across the chunks of this run: clear it now
    FX_CUDA(cudaMemcpyAsync(ex->ctl_dev + 1, ex->zeros_pin, 4, cudaMemcpyHostToDevice, ex->compute));
  ex->steps_done += total_done;
  if (n_done) *n_done = total_done;
  return 0;
}

// One launch for n_steps over a device-resident dataset: `maps` are tensor maps over the dataset, the batch of step s
// is rows [(row_start + s * row_stride) % row_wrap, + batch); the kernel reads whole 32-row tiles, so the maps must
// cover `rows` rows from there. Asynchronous: returns after enqueueing (dm_fexec_drain /
// dm_fexec_resident_results complete it).
// `timed` != 0: the launch is bracketed by two CUDA events recorded on the compute stream immediately before and after
// it (no interpreter time in between); dm_fexec_last_elapsed_ms returns their distance.
int dm_fexec_run_resident(void* h, const void* maps, const void* y_base, uint64_t row_start, uint64_t row_stride,
                          uint64_t row_wrap, uint64_t n_steps, int wait_acks, int timed) {
  FusedExec* ex = static_cast<FusedExec*>(h);
  if (!ex->have_params || n_steps == 0 || n_steps > 0xFFFFFFF0ull) { g_fx_err = "run_resident: bad arguments"; return -1; }
  dm::NvtxRange nvtx_res("dm.fexec.run_resident");
  if (ex->last_results == ex->res_big && ex->last_n != 0) FX_CUDA(cudaEventSynchronize(ex->last_done));
  if (ex->ensure_big(n_steps) != 0) return -1;
  memset(ex->res_big, 0, n_steps * sizeof(dm::StepResult));
  dm::FusedMaps m;
  memcpy(&m, maps, sizeof(m));
  dm::FusedParams p = ex->params;
  p.y_base = static_cast<const float*>(y_base);
  p.row_start = row_start;
  p.row_stride = row_stride;
  p.row_wrap = row_wrap;
  if (timed) FX_CUDA(cudaEventRecord(ex->t_start, ex->compute));
  if (ex->launch(m, p, static_cast<uint32_t>(n_steps), ex->res_big, 0, true, wait_acks != 0) != 0) return -1;
  if (timed) FX_CUDA(cudaEventRecord(ex->t_stop, ex->compute));
  FX_CUDA(cudaEventRecord(ex->last_done, ex->compute));
  ex->steps_done += n_steps;   // no stop condition on this path: every step runs
  ex->last_n = n_steps;
  ex->last_results = ex->res_big;
  return 0;
}

// Device time of the most recent timed resident launch (waits for it).
int dm_fexec_last_elapsed_ms(void* h, float* ms) {
  FusedExec* ex = static_cast<FusedExec*>(h);
  FX_CUDA(cudaEventSynchronize(ex->t_stop));
  FX_CUDA(cudaEventElapsedTime(ms, ex->t_start, ex->t_stop));
  return 0;
}

// Wait for the most recent resident launch and copy its results (out may be null: just wait).
int dm_fexec_resident_results(void* h, void* out, uint64_t max_n, uint64_t* n) {
  FusedExec* ex = static_cast<FusedExec*>(h);
  if (ex->last_n == 0) { if (n) *n = 0; return 0; }
  FX_CUDA(cudaEventSynchronize(ex->last_done));
  const uint64_t k = std::min<uint64_t>(ex->last_n, max_n);
  if (out) memcpy(out, ex->last_results, k * sizeof(dm::StepResult));
  if (n) *n = k;
  return 0;
}

int dm_fexec_destroy(void* h) {
  FusedExec* ex = static_cast<FusedExec*>(h);
  cudaSetDevice(ex->device);
  ex->pool.stop();
  cudaStreamSynchronize(ex->copy);
  cudaStreamSynchronize(ex->compute);
  for (auto& b : ex->bufs) {
    cudaEventDestroy(b.copied);
    cudaEventDestroy(b.done);
  }
  cudaEventDestroy(ex->last_done);
  for (auto& e : ex->feed_read) cudaEventDestroy(e);
  cudaEventDestroy(ex->t_start);
  cudaEventDestroy(ex->t_stop);
  cudaFree(ex->x_dev);
  cudaFree(ex->y_dev);
  cudaFree(ex->ctl_dev);
  cudaFreeHost(ex->x_stage);
  cudaFreeHost(ex->y_stage);
  cudaFreeHost(ex->res_chunks);
  cudaFreeHost(ex->zeros_pin);
  if (ex->res_big) cudaFreeHost(ex->res_big);
  cudaStreamDestroy(ex->compute);
  cudaStreamDestroy(ex->copy);
  delete ex;
  return 0;
}

}  // extern "C"
