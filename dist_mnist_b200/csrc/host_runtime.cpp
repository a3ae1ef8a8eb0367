// Host-side native runtime (no CUDA): POSIX shared-memory "peer memory" for the CPU plumbing backend and
// the CPU parameter-server serve loop.
//
// The CPU backend (BASELINE.json config 1: 1 ps + 1 worker on CPU) runs the *same* shard protocol as the
// GPU path — arena / mailbox / per-item flags / inbox acks (protocol.h) — with POSIX shm standing in for
// NVLink peer memory and a native thread standing in for the persistent PS kernel. It mirrors
// ps_serve_kernel in ps_apply_sm90.cu line for line so the protocol logic can be tested without a GPU.
//
// Reference parity: tf.train.Server(...).join() serving variable reads / ApplyAdam on the ps task
// (/root/reference/distributed_server-basic.py:80-83, 102-103).
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <cerrno>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>

#include "protocol.h"

namespace {

thread_local std::string g_err_host;

inline uint32_t load_acquire(const uint32_t* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
inline void store_release(uint32_t* p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }

inline uint16_t f32_to_bf16(float f) {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x40);  // NaN
  u += 0x7fffu + ((u >> 16) & 1u);                                                     // round to nearest even
  return static_cast<uint16_t>(u >> 16);
}

struct CpuPs {
  dm::PsServeParams P;
  std::thread th;
  std::atomic<int> running{0};
  std::atomic<uint64_t> applied{0};
};

void apply_item_cpu(const dm::PsServeParams& P, const dm::PsItem& it, dm::PsItemState st, uint32_t mask,
                    const uint32_t* seqs) {
  const uint64_t wstride = static_cast<uint64_t>(P.nslots) * P.arena_elems;
  for (int r = 0; r < it.rows; ++r) {
    for (int c = 0; c < it.cols; ++c) {
      const uint64_t a = it.offset + static_cast<uint64_t>(r) * it.ld + c;
      float p = P.params[a];
      float m = 0.f, v = 0.f;
      if (P.opt == dm::OPT_ADAM) { m = P.adam_m[a]; v = P.adam_v[a]; }
      float b1p = st.beta1_pow, b2p = st.beta2_pow;
      float gsum = 0.f;
      uint32_t mm = mask;
      while (mm) {
        const int w = __builtin_ffs(mm) - 1;
        mm &= mm - 1;
        const uint32_t slot = seqs[w] % P.nslots;
        const float g = P.mailbox[static_cast<uint64_t>(w) * wstride + static_cast<uint64_t>(slot) * P.arena_elems + a];
        if (P.apply_mode == dm::APPLY_MERGED) { gsum += g; continue; }
        if (P.opt == dm::OPT_ADAM) {
          b1p *= P.beta1; b2p *= P.beta2;
          const float lr_t = P.lr * std::sqrt(1.f - b2p) / (1.f - b1p);
          m = P.beta1 * m + (1.f - P.beta1) * g;
          v = P.beta2 * v + (1.f - P.beta2) * g * g;
          p -= lr_t * m / (std::sqrt(v) + P.eps);
        } else {
          p -= P.lr * g;
        }
      }
      if (P.apply_mode == dm::APPLY_MERGED) {
        if (P.opt == dm::OPT_ADAM) {
          b1p *= P.beta1; b2p *= P.beta2;
          const float lr_t = P.lr * std::sqrt(1.f - b2p) / (1.f - b1p);
          m = P.beta1 * m + (1.f - P.beta1) * gsum;
          v = P.beta2 * v + (1.f - P.beta2) * gsum * gsum;
          p -= lr_t * m / (std::sqrt(v) + P.eps);
        } else {
          p -= P.lr * gsum;
        }
      }
      P.params[a] = p;
      if (P.opt == dm::OPT_ADAM) { P.adam_m[a] = m; P.adam_v[a] = v; }
      if (P.shadow_bf16 != nullptr && (it.flags & 1)) P.shadow_bf16[a] = f32_to_bf16(p);
    }
  }
}

void serve_loop(CpuPs* ps) {
  const dm::PsServeParams& P = ps->P;
  uint32_t seqs[dm::kMaxWorkers];
  int idle = 0;
  for (;;) {
    bool any = false;
    for (int item = 0; item < P.n_items; ++item) {
      uint32_t mask = 0;
      for (int w = 0; w < P.n_workers; ++w) {
        const uint32_t seq = P.next_seq[static_cast<size_t>(w) * P.n_items + item];
        const uint32_t slot = seq % P.nslots;
        seqs[w] = seq;
        if (load_acquire(P.flags + (static_cast<size_t>(w) * P.nslots + slot) * P.n_flags + P.items[item].flag_index) == seq)
          mask |= 1u << w;
      }
      if (!mask) continue;
      any = true;
      const dm::PsItem it = P.items[item];
      const dm::PsItemState st = P.item_state[item];
      apply_item_cpu(P, it, st, mask, seqs);
      const int npush = __builtin_popcount(mask);
      const int nsteps = (P.apply_mode == dm::APPLY_MERGED) ? 1 : npush;
      dm::PsItemState ns = st;
      ns.t += nsteps;
      for (int k = 0; k < nsteps; ++k) { ns.beta1_pow *= P.beta1; ns.beta2_pow *= P.beta2; }
      P.item_state[item] = ns;
      uint32_t mm = mask;
      while (mm) {
        const int w = __builtin_ffs(mm) - 1;
        mm &= mm - 1;
        const uint32_t seq = seqs[w];
        const uint32_t slot = seq % P.nslots;
        P.next_seq[static_cast<size_t>(w) * P.n_items + item] = seq + 1;
        const uint32_t done = ++P.consumed[w * P.nslots + slot];
        if (done == static_cast<uint32_t>(P.n_items)) {
          P.consumed[w * P.nslots + slot] = 0;
          const uint32_t gs = __atomic_add_fetch(P.global_step, 1u, __ATOMIC_ACQ_REL);
          ps->applied.fetch_add(1);
          uint32_t* ib = P.inbox_table[w];
          if (ib != nullptr) {
            __atomic_store_n(ib + 1, gs, __ATOMIC_RELAXED);
            store_release(ib, seq);
          }
        }
      }
    }
    if (load_acquire(const_cast<const uint32_t*>(P.host_stop)) != 0) break;
    bool all_done = true;
    for (int w = 0; w < P.n_workers && all_done; ++w) {
      const uint32_t d = load_acquire(P.worker_done + w);
      if (d == 0) { all_done = false; break; }
      if (d == dm::kWorkerDead) continue;   // presumed dead (ps host failure detector)
      for (int item = 0; item < P.n_items; ++item)
        if (P.next_seq[static_cast<size_t>(w) * P.n_items + item] != d) { all_done = false; break; }
    }
    if (all_done) break;
    if (any) {
      idle = 0;
    } else if (++idle > 64) {
      std::this_thread::sleep_for(std::chrono::microseconds(20));
    } else {
      std::this_thread::yield();
    }
  }
  __atomic_add_fetch(P.exit_counter, 1u, __ATOMIC_ACQ_REL);
  ps->running.store(0);
}

}  // namespace

extern "C" {

const char* dm_host_last_error() { return g_err_host.c_str(); }

// ---- POSIX shared memory -----------------------------------------------------------------
int dm_shm_create(const char* name, size_t bytes, void** out) {
  shm_unlink(name);
  int fd = shm_open(name, O_CREAT | O_EXCL | O_RDWR, 0600);
  if (fd < 0) { g_err_host = std::string("shm_open(create) failed for ") + name + ": " + strerror(errno); return -1; }
  if (ftruncate(fd, static_cast<off_t>(bytes)) != 0) {
    g_err_host = std::string("ftruncate failed: ") + strerror(errno);
    close(fd);
    return -1;
  }
  void* p = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (p == MAP_FAILED) { g_err_host = std::string("mmap failed: ") + strerror(errno); return -1; }
  std::memset(p, 0, bytes);
  *out = p;
  return 0;
}
int dm_shm_open(const char* name, size_t bytes, void** out) {
  int fd = shm_open(name, O_RDWR, 0600);
  if (fd < 0) { g_err_host = std::string("shm_open failed for ") + name + ": " + strerror(errno); return -1; }
  void* p = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (p == MAP_FAILED) { g_err_host = std::string("mmap failed: ") + strerror(errno); return -1; }
  *out = p;
  return 0;
}
int dm_shm_unmap(void* p, size_t bytes) { return munmap(p, bytes); }
int dm_shm_unlink(const char* name) { return shm_unlink(name); }

// ---- flags --------------------------------------------------------------------------------
void dm_store_release_u32(void* p, uint32_t v) { store_release(static_cast<uint32_t*>(p), v); }
uint32_t dm_load_acquire_u32(const void* p) { return load_acquire(static_cast<const uint32_t*>(p)); }
uint32_t dm_atomic_add_u32(void* p, uint32_t v) {
  return __atomic_fetch_add(static_cast<uint32_t*>(p), v, __ATOMIC_ACQ_REL);
}
// Spin (with yield) until *p == v or the timeout expires. Returns 0 on success, 1 on timeout.
int dm_wait_ge_u32(const void* p, uint32_t v, double timeout_s) {
  const auto t0 = std::chrono::steady_clock::now();
  int spins = 0;
  while (static_cast<int32_t>(load_acquire(static_cast<const uint32_t*>(p)) - v) < 0) {
    if (++spins > 64) {
      std::this_thread::sleep_for(std::chrono::microseconds(20));
      if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > timeout_s) return 1;
    } else {
      std::this_thread::yield();
    }
  }
  return 0;
}

// ---- CPU parameter-server serve loop --------------------------------------------------------
void* dm_cpu_ps_start(const void* params_bytes) {
  CpuPs* ps = new CpuPs();
  std::memcpy(&ps->P, params_bytes, sizeof(dm::PsServeParams));
  ps->running.store(1);
  ps->th = std::thread(serve_loop, ps);
  return ps;
}
int dm_cpu_ps_running(void* h) { return static_cast<CpuPs*>(h)->running.load(); }
uint64_t dm_cpu_ps_applied(void* h) { return static_cast<CpuPs*>(h)->applied.load(); }
int dm_cpu_ps_join(void* h) {
  CpuPs* ps = static_cast<CpuPs*>(h);
  if (ps->th.joinable()) ps->th.join();
  delete ps;
  return 0;
}

}  // extern "C"
