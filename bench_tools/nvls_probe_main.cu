// Standalone driver of dm_nvls_probe (dist_mnist_b200/csrc/nvls_sm90.cu): no Python, no torch import, so a run on a
// fresh GPU box costs seconds. Built by bench_tools/build_nvls_probe.sh into bench_tools/bin/nvls_probe.
//   nvls_probe [n_dev] -> probes the 318 KB parameter set of the 784-100-10 MLP and a 64 MiB buffer.
#include <cstdio>
#include <cstdlib>
#include <vector>

extern "C" int dm_nvls_probe(int n_dev, size_t bytes, int iters, char* out_log, size_t log_cap);

int main(int argc, char** argv) {
  const int n_dev = argc > 1 ? atoi(argv[1]) : 2;
  std::vector<char> log(1 << 16);
  int rc = 0;
  const size_t sizes[2] = {79510 * 4 / 16 * 16, size_t(64) << 20};
  const int iters[2] = {200, 20};
  for (int k = 0; k < 2; ++k) {
    printf("=== nvls probe: %d devices, %zu bytes, %d iterations ===\n", n_dev, sizes[k], iters[k]);
    const int r = dm_nvls_probe(n_dev, sizes[k], iters[k], log.data(), log.size());
    fputs(log.data(), stdout);
    fflush(stdout);
    rc |= r;
    if (r != 0) break;   // the second size would fail the same way
  }
  return rc;
}
