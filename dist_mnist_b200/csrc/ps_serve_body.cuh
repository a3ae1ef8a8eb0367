// Body of ps_serve_kernel, included once per kernel template (ps_apply_sm90.cu): it expects the kernel parameter
// block `P` and the compile-time `kIeee` (correctly rounded sqrt / divide), `kFam` (optimizer family), `kSched`
// (non-constant learning-rate schedule) and `kEma` (moving averages; implies kSched) in scope. A shared device
// function called by both kernels would give the Adam / SGD instantiations different SASS from the one that was
// measured; included textually they compile exactly as before. Everything a schedule adds sits behind
// `if constexpr (kSched)`, everything averaging adds behind `if constexpr (kEma)`.
  // Everything the poll loop needs about this CTA's items lives in shared memory: the only global traffic of an
  // idle poll is one acquire load of a flag word per (worker, look-ahead slot).
  __shared__ PsItem s_item[kMaxOwn];
  __shared__ PsItemState s_state[kMaxOwn];
  __shared__ uint32_t s_next[kMaxOwn][kMaxWorkers];  // next expected push seq per (owned item, worker)
  __shared__ uint64_t s_pend[kMaxPending];
  __shared__ uint32_t s_round[kMaxPending];
  __shared__ uint32_t s_npend;
  __shared__ uint32_t s_any;
  __shared__ uint32_t s_exit;
  __shared__ float s_lr[kMaxPending];   // kSched: rate of the pass's i-th push, lr(sched_step + i)
  __shared__ float s_ema[kMaxPending];  // kEma: decay of the step ending at the i-th push, ema_decay(sched_step + i + 1)
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  uint32_t iter = 0;
  int n_own = 0;
  for (int item = blockIdx.x; item < P.n_items && n_own < kMaxOwn; item += gridDim.x) ++n_own;
  for (int i = tid; i < n_own; i += kPsThreads) {
    const int item = blockIdx.x + i * gridDim.x;
    s_item[i] = P.items[item];
    s_state[i] = P.item_state[item];
  }
  for (int i = tid; i < n_own * kMaxWorkers; i += kPsThreads) {
    const int own = i / kMaxWorkers, w = i - own * kMaxWorkers;
    s_next[own][w] = w < P.n_workers ? P.next_seq[static_cast<size_t>(w) * P.n_items + blockIdx.x + own * gridDim.x] : 0u;
  }
  __syncthreads();
  // poll lanes, round-major: lane = k * n_workers + w checks push s_next[w] + k of worker w. Pushes of one worker
  // are consumed in order, so only its contiguous ready prefix k = 0 .. cnt-1 is taken in a pass; lane order is
  // then exactly the application order (round k = k-th pending push of every worker, oldest round first).
  const int nw = P.n_workers;
  int kdepth = max(1, min(min(P.nslots, 16), 32 / nw));
  if (P.lookahead != 0u) kdepth = min(kdepth, static_cast<int>(P.lookahead));
  const int pk = lane / nw, pw = lane - pk * nw;
  const bool pvalid = pk < kdepth;
  const uint64_t wstride = static_cast<uint64_t>(P.nslots) * P.arena_elems;

  // Register-resident optimizer state: a CTA that owns exactly one vectorisable item of at most one sweep keeps the
  // item's parameters and Adam slots in registers from pass to pass (it is the only writer while it runs; the host
  // writes variables only while no serve kernel is resident). Results are still stored every pass — the workers pull
  // the parameters, checkpoints read the slots — but the three load round trips (~1 us of a ~6.7 us pass) are gone.
  ResidentState resident;
  resident.loaded = false;
  ResidentEma resident_ema;   // kEma: the shadows beside them
  bool use_resident = false;
  if (n_own == 1) {
    const PsItem it0 = s_item[0];
    use_resident = ((it0.cols & 3) == 0) && ((it0.ld & 3) == 0) && ((it0.offset & 3) == 0) &&
                   (it0.rows * it0.cols <= kPsThreads * kQuads * 4);
  }

  // serve statistics (thread 0's view; the CTA barriers make it representative)
  unsigned long long st_pass = 0, st_push = 0, st_apply = 0, st_book = 0, st_idle_n = 0, st_idle = 0, st_max = 0,
                     st_poll = 0;
  const bool stats_on = P.stats != nullptr;

  for (;;) {
    bool sweep_any = false;   // (uniform over the CTA: s_any is read after a barrier)
    for (int own = 0; own < n_own; ++own) {
      const int item = blockIdx.x + own * gridDim.x;
      const long long c0 = stats_on ? clock64() : 0;
      uint32_t p_seq = 0, p_cnt = 0, p_taken = 0;   // warp 0: this lane's push seq, its worker's prefix, all taken
      bool p_take = false;
      if (warp == 0) {
        uint32_t ready = 0, slot = 0;
        if (pvalid) {
          p_seq = s_next[own][pw] + pk;
          slot = p_seq % P.nslots;
          const uint32_t f = ld_acquire_scoped_u32(
              P.flags + (static_cast<size_t>(pw) * P.nslots + slot) * P.n_flags + s_item[own].flag_index, P.gpu_scope);
          ready = (f == p_seq) ? 1u : 0u;
        }
        const uint32_t b = __ballot_sync(0xffffffffu, ready);
        if (pvalid)
          while (p_cnt < static_cast<uint32_t>(kdepth) && ((b >> (p_cnt * nw + pw)) & 1u)) ++p_cnt;
        p_take = pvalid && static_cast<uint32_t>(pk) < p_cnt;
        p_taken = __ballot_sync(0xffffffffu, p_take);
        if (p_take) {
          const int pos = __popc(p_taken & ((1u << lane) - 1u));
          s_pend[pos] = static_cast<uint64_t>(pw) * wstride + static_cast<uint64_t>(slot) * P.arena_elems;
          s_round[pos] = pk;
        }
        if (lane == 0) {
          s_any = p_taken;
          s_npend = __popc(p_taken);
        }
        if constexpr (kSched) {
          // the pass's rate table (one fp32 evaluation per lane): the i-th push of the application order is applied
          // at schedule step sched_step + i; published to apply_item by the barrier below
          if (lane < __popc(p_taken)) s_lr[lane] = scheduled_lr(P, s_state[own].sched_step + lane);
        }
        if constexpr (kEma) {
          // the pass's decay table: the step that ends at the i-th push leaves the item at sched_step + i + 1
          // applied pushes, TF1's num_updates = global_step after the apply_gradients op the average follows
          if (lane < __popc(p_taken)) s_ema[lane] = ema_decay(P, s_state[own].sched_step + lane + 1);
        }
      }
      __syncthreads();
      const long long c1 = stats_on ? clock64() : 0;
      if (!s_any && stats_on) { ++st_idle_n; st_idle += c1 - c0; }
      if (s_any) {
        sweep_any = true;
        const PsItemState st = s_state[own];
        if constexpr (kEma)
          apply_item<kIeee, kFam, true, true>(P, s_item[own], st, s_pend, s_round, static_cast<int>(s_npend),
                                              use_resident ? &resident : nullptr, s_lr, s_ema,
                                              use_resident ? &resident_ema : nullptr);
        else if constexpr (kSched)
          apply_item<kIeee, kFam, true>(P, s_item[own], st, s_pend, s_round, static_cast<int>(s_npend),
                                        use_resident ? &resident : nullptr, s_lr);
        else
          apply_item<kIeee, kFam>(P, s_item[own], st, s_pend, s_round, static_cast<int>(s_npend),
                                  use_resident ? &resident : nullptr);
        __syncthreads();   // every thread's parameter stores precede warp 0's release operations below
        const long long c2 = stats_on ? clock64() : 0;
        if (stats_on) {
          ++st_pass; st_push += s_npend; st_apply += c2 - c1; st_poll += c1 - c0;
          st_max = max(st_max, static_cast<unsigned long long>(s_npend));
        }
        if (warp == 0) {
          if (lane == 0) {
            const uint32_t npush = __popc(p_taken);
            const uint32_t rounds = (31u - __clz(p_taken)) / nw + 1u;   // lanes are round-major
            const uint32_t nsteps = (P.apply_mode == APPLY_MERGED) ? rounds : npush;
            PsItemState ns = st;
            ns.t += nsteps;
            for (uint32_t k = 0; k < nsteps; ++k) { ns.beta1_pow *= P.beta1; ns.beta2_pow *= P.beta2; }
            // one schedule step per push, in both apply modes (also the num_updates of the averaging kernels)
            if constexpr (kSched) ns.sched_step += npush;
            s_state[own] = ns;
            P.item_state[item] = ns;   // persisted for checkpoints / a relaunch (never read back in this loop)
          }
          if (p_take) {
            const uint32_t slot = p_seq % P.nslots;
            const uint32_t done = atomicAdd(&P.consumed[pw * P.nslots + slot], 1u) + 1u;
            if (done == static_cast<uint32_t>(P.n_items)) {
              // this worker's push `p_seq` is fully applied: one global step (reference DS:91,103)
              P.consumed[pw * P.nslots + slot] = 0;
              const uint32_t gs = atomicAdd(P.global_step, 1u) + 1u;
              uint32_t* ib = P.inbox_table[pw];
              if (ib != nullptr) {
                red_max_relaxed_scoped_u32(ib + 1, gs, P.gpu_scope);
                red_max_release_scoped_u32(ib, p_seq, P.gpu_scope);  // ack: the mailbox slot may be reused
              }
            }
          }
          if (pvalid && pk == 0 && p_cnt > 0) {
            const uint32_t nx = p_seq + p_cnt;
            s_next[own][pw] = nx;
            P.next_seq[static_cast<size_t>(pw) * P.n_items + item] = nx;
          }
        }
        if (stats_on) { __syncwarp(); st_book += clock64() - c2; }
      }
      __syncthreads();
    }
    // ---- exit protocol: host stop request, or every worker has left and all their pushes are applied ----
    // (checked every 32nd poll round only: the check itself costs several system-scope loads, and the poll
    //  loop's period is the PS's reaction latency)
    if (tid == 0) {
      uint32_t ex = 0;
      // one-shot mode: everything that will ever be pushed was pushed before this launch (stream order), so a
      // full sweep without work means the shard is up to date
      if (P.oneshot && !sweep_any) ex = 1;
      const bool check = !P.oneshot && (iter & 31u) == 0u;
      if (check && *P.host_stop != 0u) ex = 1;
      if (check && !ex) {
        bool all_done = true;
        for (int w = 0; w < P.n_workers && all_done; ++w) {
          const uint32_t d = ld_acquire_sys_u32(P.worker_done + w);  // = last push seq + 1, 0 while active
          if (d == 0) { all_done = false; break; }
          if (d == kWorkerDead) continue;   // presumed dead: whatever it left half-pushed is dropped
          for (int own = 0; own < n_own; ++own)
            if (s_next[own][w] != d) { all_done = false; break; }
        }
        if (all_done) ex = 1;
      }
      s_exit = ex;
    }
    __syncthreads();
    if (s_exit) break;
    ++iter;
  }
  if (tid == 0) {
    if (stats_on) {
      unsigned long long* o = P.stats + static_cast<size_t>(blockIdx.x) * 8;
      o[0] += st_pass; o[1] += st_push; o[2] += st_apply; o[3] += st_book; o[4] += st_idle_n; o[5] += st_idle;
      o[6] = max(o[6], st_max); o[7] += st_poll;
      P.stats[kPsStatsCtas * 8 + blockIdx.x] = sm_id();
    }
    atomicAdd(P.exit_counter, 1u);
  }
