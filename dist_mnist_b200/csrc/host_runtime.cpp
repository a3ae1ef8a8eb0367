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

#include "lr_schedule.h"
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

// ApplyProximalAdagrad / ApplyProximalGradientDescent's proximal step at step size a (ps_apply_sm90.cu prox_shrink)
float prox_shrink_cpu(float prox, float a, float l1, float l2) {
  const float num = l1 > 0.f ? std::copysign(std::fmax(std::fabs(prox) - a * l1, 0.f), prox) : prox;
  return num / (1.f + l2 * a);
}

// TF1 Apply{Momentum,Adagrad,RMSProp,Adadelta,FtrlV2,ProximalAdagrad,ProximalGradientDescent} with IEEE arithmetic and
// the C library's float functions (ps_apply_sm90.cu tf1_step)
void tf1_step_cpu(const dm::PsServeParams& P, float lr, float& p, float& m, float& v, float g) {
  if (P.opt == dm::OPT_MOMENTUM) {
    m = P.momentum * m + g;
    if (P.nesterov) p -= g * lr + m * P.momentum * lr;
    else p -= lr * m;
  } else if (P.opt == dm::OPT_ADAGRAD) {
    v += g * g;
    p -= lr * g / std::sqrt(v);
  } else if (P.opt == dm::OPT_RMSPROP) {
    v += (g * g - v) * (1.f - P.decay);
    m = P.momentum * m + lr * g / std::sqrt(v + P.eps);
    p -= m;
  } else if (P.opt == dm::OPT_ADADELTA) {   // v = accum, m = accum_update, rho = P.decay
    v = v * P.decay + g * g * (1.f - P.decay);
    const float upd = std::sqrt(m + P.eps) * (1.f / std::sqrt(v + P.eps)) * g;
    p -= upd * lr;
    m = m * P.decay + upd * upd * (1.f - P.decay);
  } else if (P.opt == dm::OPT_PROXIMAL_ADAGRAD) {   // v = accumulator
    v += g * g;
    const float a = lr * (1.f / std::sqrt(v));
    p = prox_shrink_cpu(p - g * a, a, P.l1, P.l2);
  } else if (P.opt == dm::OPT_PROXIMAL_SGD) {
    p = prox_shrink_cpu(p - lr * g, lr, P.l1, P.l2);
  } else {   // OPT_FTRL: v = accum, m = linear
    const float gs = g + 2.f * P.l2_shrinkage * p;
    const float n = v + g * g;
    const bool half = P.lr_power == -0.5f;
    const float pn = half ? std::sqrt(n) : std::pow(n, -P.lr_power);
    const float pa = half ? std::sqrt(v) : std::pow(v, -P.lr_power);
    m += gs - (pn - pa) / lr * p;
    const float y = pn / lr + 2.f * P.l2;
    p = std::fabs(m) > P.l1 ? (std::copysign(P.l1, m) - m) / y : 0.f;
    v = n;
  }
}

void apply_item_cpu(const dm::PsServeParams& P, const dm::PsItem& it, dm::PsItemState st, uint32_t mask,
                    const uint32_t* seqs) {
  const uint64_t wstride = static_cast<uint64_t>(P.nslots) * P.arena_elems;
  const bool tf1 = P.opt != dm::OPT_ADAM && P.opt != dm::OPT_SGD;
  const bool use_m = P.opt == dm::OPT_ADAM || P.opt == dm::OPT_MOMENTUM || P.opt == dm::OPT_RMSPROP ||
                     P.opt == dm::OPT_ADADELTA || P.opt == dm::OPT_FTRL;
  const bool use_v = P.opt == dm::OPT_ADAM || P.opt == dm::OPT_ADAGRAD || P.opt == dm::OPT_RMSPROP ||
                     P.opt == dm::OPT_ADADELTA || P.opt == dm::OPT_FTRL || P.opt == dm::OPT_PROXIMAL_ADAGRAD;
  // rate of the k-th push of the pass (workers in order), lr(sched_step + k); a merged step uses lr(sched_step)
  float lrs[dm::kMaxWorkers];
  for (int k = 0; k < __builtin_popcount(mask); ++k)
    lrs[k] = P.lr_schedule == dm::LR_CONSTANT ? P.lr : dm::scheduled_lr(P, st.sched_step + k);
  // moving averages: 1 - d of the step that ends at the k-th push, d = ema_decay(sched_step + k + 1); a merged step
  // ends at the last push of the pass
  const bool ema = P.ema != nullptr;
  const int npush = __builtin_popcount(mask);
  float ema_omd[dm::kMaxWorkers];
  for (int k = 0; ema && k < npush; ++k) ema_omd[k] = 1.f - dm::ema_decay(P, st.sched_step + k + 1);
  for (int r = 0; r < it.rows; ++r) {
    for (int c = 0; c < it.cols; ++c) {
      const uint64_t a = it.offset + static_cast<uint64_t>(r) * it.ld + c;
      float p = P.params[a];
      float m = 0.f, v = 0.f, e = 0.f;
      if (use_m) m = P.adam_m[a];
      if (use_v) v = P.adam_v[a];
      if (ema) e = P.ema[a];
      float b1p = st.beta1_pow, b2p = st.beta2_pow;
      float gsum = 0.f;
      uint32_t mm = mask;
      int k = 0;
      while (mm) {
        const int w = __builtin_ffs(mm) - 1;
        mm &= mm - 1;
        const uint32_t slot = seqs[w] % P.nslots;
        const float g = P.mailbox[static_cast<uint64_t>(w) * wstride + static_cast<uint64_t>(slot) * P.arena_elems + a];
        if (P.apply_mode == dm::APPLY_MERGED) { gsum += g; continue; }
        const float omd = ema ? ema_omd[k] : 0.f;
        const float lr = lrs[k++];
        if (tf1) {
          tf1_step_cpu(P, lr, p, m, v, g);
        } else if (P.opt == dm::OPT_ADAM) {
          b1p *= P.beta1; b2p *= P.beta2;
          const float lr_t = lr * std::sqrt(1.f - b2p) / (1.f - b1p);
          m = P.beta1 * m + (1.f - P.beta1) * g;
          v = P.beta2 * v + (1.f - P.beta2) * g * g;
          p -= lr_t * m / (std::sqrt(v) + P.eps);
        } else {
          p -= lr * g;
        }
        if (ema) e -= (e - p) * omd;   // assign_moving_average
      }
      if (P.apply_mode == dm::APPLY_MERGED) {
        const float lr = lrs[0];
        if (tf1) {
          tf1_step_cpu(P, lr, p, m, v, gsum);
        } else if (P.opt == dm::OPT_ADAM) {
          b1p *= P.beta1; b2p *= P.beta2;
          const float lr_t = lr * std::sqrt(1.f - b2p) / (1.f - b1p);
          m = P.beta1 * m + (1.f - P.beta1) * gsum;
          v = P.beta2 * v + (1.f - P.beta2) * gsum * gsum;
          p -= lr_t * m / (std::sqrt(v) + P.eps);
        } else {
          p -= lr * gsum;
        }
        if (ema) e -= (e - p) * ema_omd[npush - 1];
      }
      P.params[a] = p;
      if (use_m) P.adam_m[a] = m;
      if (use_v) P.adam_v[a] = v;
      if (ema) P.ema[a] = e;
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
      // one schedule step per push, both apply modes (also the moving averages' num_updates)
      if (P.lr_schedule != dm::LR_CONSTANT || P.ema != nullptr) ns.sched_step += npush;
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
