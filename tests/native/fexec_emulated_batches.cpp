// Host-only test of the fused executor (csrc/fused_exec.cu) at batch sizes that are not one 32-row tile, on the
// emulated CUDA runtime (fake_cuda/cuda_runtime.h).
//
// A ring slot holds the batch rounded up to whole 32-row tiles. The step kernel is replaced by a function that reads
// each step's batch out of the device ring where the real kernel's TMA would (row (row_start + s * row_stride) %
// row_wrap), checksums its B x I inputs and its labels, and also checks that the slot's padding rows are zero. The test
// replays the same `next_batch` sequence with a second loader and checks that every step of every run saw exactly its
// batch, over the gather path, the epoch feed (batch a multiple of 32) and epoch boundaries.
//
//   fexec_emulated_batches <dataset rows> <epoch feed 0|1> <steps> <batch>
#include <cuda_runtime.h>
#include <stdio.h>

#include <cmath>
#include <vector>

#include "fused.h"
#include "loader.h"

extern "C" {
void* dm_loader_create(const void*, const void*, size_t, size_t, size_t, size_t, size_t, int, uint64_t, int);
void dm_loader_next(void*, void*, void*);
uint64_t dm_loader_epochs(void*);
int dm_loader_enable_feed(void*, void*, void*, void*, void*, int);
void dm_loader_destroy(void*);
int dm_fexec_create(int, int, int, int, int, void**);
int dm_fexec_buffers(void*, void**, void**, void**, void**, void**, int*);
int dm_fexec_set_params(void*, const void*, const void*);
int dm_fexec_run(void*, void*, uint64_t, void*, uint32_t, uint64_t*, int);
void dm_fexec_feed_stats(void*, uint64_t*, uint64_t*, uint64_t*);
int dm_fexec_destroy(void*);
const char* dm_fexec_last_error();
}

namespace {
const float* g_x_dev = nullptr;
std::atomic<uint32_t> g_global_step{0};
std::atomic<uint32_t> g_dirty_padding{0};
int g_I = 0, g_C = 0, g_rows = 0;

float checksum(const float* p, size_t n) {
  double a = 0;
  for (size_t i = 0; i < n; ++i) a += p[i] * static_cast<double>((i % 7) + 1);
  return static_cast<float>(a);
}
}  // namespace

namespace dm {
// Stand-in for the kernel: same launch-state protocol as fused_step_kernel (step claiming is sequential here).
cudaError_t launch_fused_step(const FusedMaps&, const FusedParams& p, int, cudaStream_t stream) {
  const FusedParams q = p;
  stream->push([q] {
    fakecuda::random_delay();
    for (uint32_t s = 0; s < q.n_steps; ++s) {
      if (*q.stop_word != 0) break;
      const uint64_t row = (q.row_start + s * q.row_stride) % q.row_wrap;
      const float* x = g_x_dev + row * g_I;
      const float* y = q.y_base + row * g_C;
      for (size_t i = static_cast<size_t>(q.B) * g_I; i < static_cast<size_t>(g_rows) * g_I; ++i)
        if (x[i] != 0.f) g_dirty_padding.fetch_add(1);   // the kernel reads whole tiles: padding rows must be zero
      StepResult r;
      r.loss = checksum(x, static_cast<size_t>(q.B) * g_I);
      r.correct = static_cast<uint32_t>(std::lround(checksum(y, static_cast<size_t>(q.B) * g_C)));
      r.global_step = g_global_step.fetch_add(1) + 1;
      r.seq = q.seq_base + s + 1;
      q.results[s] = r;
    }
    if (q.clear_stop) *q.stop_word = 0;
  });
  return cudaSuccess;
}
}  // namespace dm

#define CHECK(c)                                                                                      \
  do {                                                                                                \
    if (!(c)) {                                                                                       \
      fprintf(stderr, "CHECK FAILED %s:%d: %s (%s)\n", __FILE__, __LINE__, #c, dm_fexec_last_error()); \
      return 1;                                                                                       \
    }                                                                                                 \
  } while (0)

int main(int argc, char** argv) {
  if (argc < 5) {
    fprintf(stderr, "usage: %s rows feed steps batch\n", argv[0]);
    return 2;
  }
  const size_t n = static_cast<size_t>(atoi(argv[1]));
  const int feed = atoi(argv[2]);
  const uint64_t total = static_cast<uint64_t>(atoll(argv[3]));
  const int B = atoi(argv[4]);
  const int I = 16, C = 10;
  const int rows = (B + 31) / 32 * 32;
  g_I = I;
  g_C = C;
  g_rows = rows;
  std::vector<float> images(n * I), labels(n * C, 0.f);
  for (size_t r = 0; r < n; ++r) {
    for (int k = 0; k < I; ++k) images[r * I + k] = static_cast<float>(r + 1) + 0.001f * k;   // no all-zero row
    labels[r * C + r % C] = static_cast<float>(1 + r % 5);
  }
  void* ld = dm_loader_create(images.data(), labels.data(), n, I * 4, C * 4, I * 4, C * 4, B, 1234, 1);
  void* ref = dm_loader_create(images.data(), labels.data(), n, I * 4, C * 4, I * 4, C * 4, B, 1234, 1);
  std::vector<float> fx[2], fy[2];
  if (feed) {
    for (int b = 0; b < 2; ++b) { fx[b].assign(n * I, -1.f); fy[b].assign(n * C, -1.f); }
    CHECK(dm_loader_enable_feed(ld, fx[0].data(), fy[0].data(), fx[1].data(), fy[1].data(), 3) == (n >= 1024 ? 1 : 0));
  }
  void* ex = nullptr;
  CHECK(dm_fexec_create(0, 4, I, C, B, &ex) == 0);
  void *xd, *yd, *xs, *ys, *ctl;
  int slots = 0;
  CHECK(dm_fexec_buffers(ex, &xd, &yd, &xs, &ys, &ctl, &slots) == 0);
  g_x_dev = static_cast<const float*>(xd);
  dm::FusedMaps maps;
  memset(&maps, 0, sizeof(maps));
  dm::FusedParams p;
  memset(&p, 0, sizeof(p));
  p.B = B; p.I = I; p.C = C;
  p.y_base = static_cast<const float*>(yd);
  p.row_start = 0; p.row_stride = rows; p.row_wrap = static_cast<uint64_t>(slots) * rows;
  CHECK(dm_fexec_set_params(ex, &maps, &p) == 0);

  std::vector<float> bx(static_cast<size_t>(B) * I), by(static_cast<size_t>(B) * C);
  const uint64_t run_sizes[] = {5, 20, 1, 50, 16, 37, 100, 4, 333};
  uint64_t done_total = 0, seq_expected = 0;
  for (size_t k = 0; done_total < total; ++k) {
    const uint64_t want = run_sizes[k % (sizeof(run_sizes) / sizeof(run_sizes[0]))];
    std::vector<dm::StepResult> out(want);
    uint64_t n_done = 0;
    CHECK(dm_fexec_run(ex, ld, want, out.data(), 0, &n_done, 0) == 0);
    CHECK(n_done == want);
    for (uint64_t s = 0; s < want; ++s) {
      dm_loader_next(ref, bx.data(), by.data());
      const float ex_loss = checksum(bx.data(), bx.size());
      const uint32_t ex_corr = static_cast<uint32_t>(std::lround(checksum(by.data(), by.size())));
      ++seq_expected;
      if (out[s].loss != ex_loss || out[s].correct != ex_corr || out[s].seq != seq_expected) {
        fprintf(stderr, "MISMATCH at run %zu step %llu: loss %.3f vs %.3f, y %u vs %u, seq %u vs %llu\n", k,
                (unsigned long long)s, out[s].loss, ex_loss, out[s].correct, ex_corr, out[s].seq,
                (unsigned long long)seq_expected);
        return 1;
      }
    }
    done_total += want;
  }
  CHECK(dm_loader_epochs(ld) == dm_loader_epochs(ref));
  CHECK(g_dirty_padding.load() == 0);
  uint64_t direct = 0, gathered = 0, fills = 0;
  dm_fexec_feed_stats(ex, &direct, &gathered, &fills);
  printf("OK n=%zu feed=%d batch=%d steps=%llu epochs=%llu direct_chunks=%llu gathered_chunks=%llu fills_posted=%llu\n",
         n, feed, B, (unsigned long long)done_total, (unsigned long long)dm_loader_epochs(ld),
         (unsigned long long)direct, (unsigned long long)gathered, (unsigned long long)fills);
  dm_loader_destroy(ld);
  dm_loader_destroy(ref);
  CHECK(dm_fexec_destroy(ex) == 0);
  return 0;
}
