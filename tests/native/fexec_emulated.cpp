// Host-only test of the fused executor (csrc/fused_exec.cu) on the emulated CUDA runtime (fake_cuda/cuda_runtime.h).
//
// The fused step kernel is replaced by a function that runs on the emulated compute stream, reads each step's batch out
// of the device ring exactly where the real kernel's TMA would (row (row_start + s * row_stride) % row_wrap) and writes
// a checksum of the 32 x I inputs and of the labels into the step's result. The test replays the same `next_batch`
// sequence with a second loader and checks that every step of every run saw exactly its batch — through the gather
// path, the epoch-feed path, across epoch boundaries, with early stop, and with the loader also used from outside.
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
int g_I = 0, g_C = 0;

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
      StepResult r;
      r.loss = checksum(x, static_cast<size_t>(q.B) * g_I);
      r.correct = static_cast<uint32_t>(std::lround(checksum(y, static_cast<size_t>(q.B) * g_C)));
      r.global_step = g_global_step.fetch_add(1) + 1;
      r.seq = q.seq_base + s + 1;
      q.results[s] = r;
      if (q.stop_at != 0 && r.global_step >= q.stop_at) *q.stop_word = 1;
    }
    if (q.clear_stop) *q.stop_word = 0;
  });
  return cudaSuccess;
}
}  // namespace dm

#define CHECK(c)                                                                     \
  do {                                                                               \
    if (!(c)) {                                                                      \
      fprintf(stderr, "CHECK FAILED %s:%d: %s (%s)\n", __FILE__, __LINE__, #c, dm_fexec_last_error()); \
      return 1;                                                                      \
    }                                                                                \
  } while (0)

int main(int argc, char** argv) {
  const size_t n = argc > 1 ? atoi(argv[1]) : 3000;   // dataset rows
  const int feed = argc > 2 ? atoi(argv[2]) : 1;
  const uint64_t total = argc > 3 ? atoll(argv[3]) : 1200;   // steps
  const int I = 16, C = 10, B = 32;
  g_I = I;
  g_C = C;
  std::vector<float> images(n * I), labels(n * C, 0.f);
  for (size_t r = 0; r < n; ++r) {
    for (int k = 0; k < I; ++k) images[r * I + k] = static_cast<float>(r) + 0.001f * k;
    labels[r * C + r % C] = static_cast<float>(1 + r % 5);
  }
  void* ld = dm_loader_create(images.data(), labels.data(), n, I * 4, C * 4, I * 4, C * 4, B, 1234, 1);
  void* ref = dm_loader_create(images.data(), labels.data(), n, I * 4, C * 4, I * 4, C * 4, B, 1234, 1);
  std::vector<float> fx[2], fy[2];
  if (feed) {
    for (int b = 0; b < 2; ++b) { fx[b].assign(n * I, -1.f); fy[b].assign(n * C, -1.f); }
    const int en = dm_loader_enable_feed(ld, fx[0].data(), fy[0].data(), fx[1].data(), fy[1].data(), 3);
    CHECK(en == (n >= 1024 ? 1 : 0));
  }
  if (const char* e = getenv("FAKE_FAIL_FEED_COPY")) {   // refuse copies out of the epoch buffers after `e` good ones
    fakecuda::fail_countdown() = atoi(e);
    fakecuda::fail_pred() = [&](const void* src) {
      for (int b = 0; b < 2; ++b) {
        const char* p = static_cast<const char*>(src);
        if (!fx[b].empty() && p >= reinterpret_cast<const char*>(fx[b].data()) && p < reinterpret_cast<const char*>(fx[b].data() + fx[b].size())) return true;
        if (!fy[b].empty() && p >= reinterpret_cast<const char*>(fy[b].data()) && p < reinterpret_cast<const char*>(fy[b].data() + fy[b].size())) return true;
      }
      return false;
    };
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
  p.row_start = 0; p.row_stride = 32; p.row_wrap = static_cast<uint64_t>(slots) * 32;
  CHECK(dm_fexec_set_params(ex, &maps, &p) == 0);

  std::vector<float> bx(B * I), by(B * C);
  uint64_t done_total = 0, seq_expected = 0;
  const unsigned seed = argc > 4 ? static_cast<unsigned>(atoi(argv[4])) : 0u;   // != 0: random run lengths
  std::mt19937 rng(seed ? seed : 7u);
  const uint64_t run_sizes[] = {5, 20, 1, 50, 16, 37, 100, 4, 333};
  size_t k = 0;
  while (done_total < total) {
    const uint64_t want = seed != 0 ? 1 + rng() % 120 : run_sizes[k % (sizeof(run_sizes) / sizeof(run_sizes[0]))];
    ++k;
    if (k % 5 == 0) {   // the loader is also used from outside the executor (Python's next_batch): must stay coherent
      dm_loader_next(ld, bx.data(), by.data());
      std::vector<float> rx(B * I), ry(B * C);
      dm_loader_next(ref, rx.data(), ry.data());
      CHECK(memcmp(bx.data(), rx.data(), rx.size() * 4) == 0 && memcmp(by.data(), ry.data(), ry.size() * 4) == 0);
    }
    // now and then an early stop: the executor plans ahead, so the loader may have been advanced past the steps run;
    // the reference loader cannot know by how much -> only done on the last run
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
        fprintf(stderr, "MISMATCH at run %zu step %llu (global %llu): loss %.3f vs %.3f, y %u vs %u, seq %u vs %llu, epochs %llu\n", k,
                (unsigned long long)s, (unsigned long long)(done_total + s), out[s].loss, ex_loss, out[s].correct, ex_corr,
                out[s].seq, (unsigned long long)seq_expected, (unsigned long long)dm_loader_epochs(ref));
        return 1;
      }
    }
    done_total += want;
  }
  CHECK(dm_loader_epochs(ld) == dm_loader_epochs(ref));
  // early stop: global_step is at done_total (+ nothing else): stop 10 steps into a 64-step run
  {
    const uint32_t stop_at = g_global_step.load() + 10;
    std::vector<dm::StepResult> out(64);
    uint64_t n_done = 0;
    CHECK(dm_fexec_run(ex, ld, 64, out.data(), stop_at, &n_done, 0) == 0);
    CHECK(n_done >= 10 && n_done <= 64);
    for (uint64_t s = 0; s < n_done; ++s) CHECK(out[s].seq == seq_expected + s + 1);
    // and the executor is usable afterwards
    uint64_t n2 = 0;
    CHECK(dm_fexec_run(ex, ld, 8, out.data(), 0, &n2, 0) == 0);
    CHECK(n2 == 8);
  }
  uint64_t direct = 0, gathered = 0, fills = 0;
  dm_fexec_feed_stats(ex, &direct, &gathered, &fills);
  printf("OK n=%zu feed=%d steps=%llu epochs=%llu direct_chunks=%llu gathered_chunks=%llu fills_posted=%llu\n", n, feed,
         (unsigned long long)done_total, (unsigned long long)dm_loader_epochs(ld), (unsigned long long)direct,
         (unsigned long long)gathered, (unsigned long long)fills);
  // destroy the loader while a fill may still be running, then the executor
  dm_loader_destroy(ld);
  dm_loader_destroy(ref);
  CHECK(dm_fexec_destroy(ex) == 0);
  return 0;
}
