// resident.cu — delta scatter for device-resident state records (SURVEY.md row f2, incremental state upload).
//
// One thread per delta.  Bit-sliced fields (phase 4 planes, cond / decision 2 planes) flip one bit per plane with
// atomicOr / atomicAnd on the record's u32 words, so deltas of different steps that share a word compose; byte
// fields use a word-wide atomic on the containing u32.  At most one delta per (run, field, index) per launch
// (contract in include/bobrafrontier.h), so no ordering between threads is needed.
#include "stages.cuh"

namespace bf {


DI void set_planes(uint8_t* rec, uint32_t off, uint32_t words, uint32_t nbits, uint32_t idx, uint32_t code) {
  uint32_t* w = reinterpret_cast<uint32_t*>(rec + off) + (idx >> 5);
  const uint32_t bit = 1u << (idx & 31u);
  for (uint32_t b = 0; b < nbits; ++b, w += words) {
    if ((code >> b) & 1u) atomicOr(w, bit);
    else atomicAnd(w, ~bit);
  }
}
DI void set_byte(uint8_t* rec, uint32_t byte_off, uint32_t mask, uint32_t value) {  // (byte & ~mask) | value
  uint32_t* w = reinterpret_cast<uint32_t*>(rec + (byte_off & ~3u));
  const uint32_t sh = (byte_off & 3u) * 8u;
  atomicAnd(w, ~(mask << sh));
  atomicOr(w, value << sh);
}

// ---- run control (bf_resident_runctl*): stops and run-level deadlines --------------------------------------------------------
DI bool runctl_default(const bf_run_ctl& c) {
  const uint4 v = *reinterpret_cast<const uint4*>(&c);
  return v.x == BF_TIMER_NONE && v.y == BF_TIMER_NONE && v.z == 0u && v.w == 0u;
}
DI bool deadline_due(uint32_t d, uint32_t now) { return d != BF_TIMER_NONE && d <= now; }

// ---- a run's side areas (RunAreasView) in the launches that move or reset runs: one warp per run ------------------------------
// The lanes share the timer slots (lane t takes slots t, t + 32); lane 0 writes the one-record areas.
DI void drop_baseline(const RunAreasView& A, uint32_t r) {   // run r's schedule record has no baseline
  if (A.sched_rec) *reinterpret_cast<uint32_t*>(A.sched_rec + (size_t)r * A.sched_stride + 12) = kSchedNoBase;
}
DI void empty_timers(const RunAreasView& A, uint32_t r, uint32_t lane) {
  for (uint32_t k = lane; A.timers && k < A.timer_k; k += 32u) A.timers[(size_t)r * A.timer_k + k] = kTimerEmpty;
}
// Run r is vacated: its timer slots empty, its limiter inputs and run control at the defaults.
DI void vacate_areas(const RunAreasView& A, uint32_t r, uint32_t lane) {
  empty_timers(A, r, lane);
  if (lane == 0 && A.sched_in) A.sched_in[r] = kSchedDefault;
  if (lane == 0 && A.runctl) A.runctl[r] = kRunCtlDefault;
}
// Run r of S arrives at index `to` of D (S may be D: a move within a batch).  Its armed slots lead its slots and number at most
// D.timer_k (transfer_fit): they are copied in order, empty slots behind them.  Its limiter inputs and run control are copied,
// or set to the defaults where S has no area, and its schedule record at `to` has no baseline.  Each lane reads the same slots
// of r that vacate_areas has it empty, so a move may vacate r behind it.
DI void arrive_areas(const RunAreasView& S, uint32_t r, const RunAreasView& D, uint32_t to, uint32_t lane) {
  for (uint32_t k = lane; D.timers && k < D.timer_k; k += 32u)
    D.timers[(size_t)to * D.timer_k + k] = S.timers && k < S.timer_k ? S.timers[(size_t)r * S.timer_k + k] : kTimerEmpty;
  if (lane != 0) return;
  if (D.sched_in) {
    D.sched_in[to] = S.sched_in ? S.sched_in[r] : kSchedDefault;
    drop_baseline(D, to);
  }
  if (D.runctl) D.runctl[to] = S.runctl ? S.runctl[r] : kRunCtlDefault;
}
// Reshape (lane 0): run r of the new limiter inputs and run control keeps its old entries (keep), else takes the defaults.
DI void keep_areas(const RunAreasView& from, const RunAreasView& to, uint32_t r, bool keep) {
  if (to.sched_in) to.sched_in[r] = keep ? from.sched_in[r] : kSchedDefault;
  if (to.runctl) to.runctl[r] = keep ? from.runctl[r] : kRunCtlDefault;
}

// Stops run `run` (record rec, run-control record ctl) for `reason`, unless it is stopped already: saves its flags byte, writes
// the stopped byte, empties its step-timer slots, marks the run touched and, for a timeout, sets its limiter inputs' run_phase.
// The caller is the only thread writing this run's records in its launch.  -> 1 when the run was stopped now
DI uint32_t stop_run(uint8_t* rec, bf_run_ctl* ctl, uint32_t run, uint32_t reason, const StopParams& S) {
  if (ctl->stop) return 0u;
  ctl->saved_flags = rec[4];
  ctl->stop = (uint8_t)reason;
  set_byte(rec, 4u, 0xFFu, kStoppedFlags);
  const RunAreasView& A = S.areas;
  for (uint32_t k = 0; A.timers && k < A.timer_k; ++k) A.timers[(size_t)run * A.timer_k + k] = kTimerEmpty;
  if (reason == BF_STOP_TIMEOUT && A.sched_in) A.sched_in[run].run_phase = BF_PHASE_TIMEOUT;
  atomicMax(S.mark + run, S.mark_value);   // max: an upload's "must list" bit stays
  return 1u;
}

// Put: one thread per request (one request per run).  Deadlines are stored, then the stop applies.
__global__ void __launch_bounds__(256) runctl_put(const RunCtlPutParams P) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  const bf_run_ctl_put q = P.req[i];
  bf_run_ctl* ctl = P.area + q.run;
  ctl->story_deadline = q.story_deadline;
  ctl->drain_deadline = q.drain_deadline;
  if (q.stop) stop_run(P.state + (size_t)q.run * P.state_stride, ctl, q.run, q.stop, P.stop);
}

cudaError_t launch_runctl_put(const RunCtlPutParams& P, cudaStream_t stream) {
  if (P.n == 0) return cudaSuccess;
  runctl_put<<<(P.n + 255) / 256, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

// After an upload: one thread per uploaded run; a stopped one keeps the uploaded byte as its saved flags and is stopped again.
__global__ void __launch_bounds__(256) runctl_restop(const RunCtlRestopParams P) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  bf_run_ctl* ctl = P.area + P.first + i;
  if (!ctl->stop) return;
  uint8_t* rec = P.state + (size_t)(P.first + i) * P.state_stride;
  ctl->saved_flags = rec[4];
  set_byte(rec, 4u, 0xFFu, kStoppedFlags);
}

cudaError_t launch_runctl_restop(const RunCtlRestopParams& P, cudaStream_t stream) {
  if (P.n == 0) return cudaSuccess;
  runctl_restop<<<(P.n + 255) / 256, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

__device__ __forceinline__ void apply_delta(const DeltaParams& P, const bf_delta d) {
  bool ok = d.run < P.n_runs;
  if (ok) atomicMax(P.mark + d.run, P.mark_value);   // touch mark (Resident in ctx.h, touched ticks); max: an upload's "must list" bit stays
  uint8_t* rec = P.state + (size_t)d.run * P.state_stride;
  const uint32_t S_max = P.words * 32u;
  if (ok) switch (d.field) {
    case BF_DELTA_PHASE:
      ok = d.index < S_max && d.code < 15u;
      if (ok) set_planes(rec, P.off_phase, P.words, 4, d.index, d.code);
      break;
    case BF_DELTA_COND:
      ok = P.off_cond != BF_OFF_NONE && d.index < S_max && d.code < 4u;
      if (ok) set_planes(rec, P.off_cond, P.words, 2, d.index, d.code);
      break;
    case BF_DELTA_DECISION:
      ok = P.off_decision != BF_OFF_NONE && d.index < S_max && d.code < 4u;
      if (ok) set_planes(rec, P.off_decision, P.words, 2, d.index, d.code);
      break;
    case BF_DELTA_CHILD:
      ok = P.off_child != BF_OFF_NONE && d.index < P.child_nibbles && d.code < 15u;
      if (ok) set_byte(rec, P.off_child + (d.index >> 1), 0xFu << ((d.index & 1u) * 4u), (uint32_t)d.code << ((d.index & 1u) * 4u));
      break;
    case BF_DELTA_RUN_FLAGS:   // a stopped run keeps its stop: the byte is what a redrive restores
      if (P.runctl && P.runctl[d.run].stop) set_byte(reinterpret_cast<uint8_t*>(P.runctl + d.run), 9u, 0xFFu, d.code);
      else set_byte(rec, 4u, 0xFFu, d.code);
      break;
    case BF_DELTA_REGISTERED: {
      ok = d.index < BF_MAX_PARALLEL;
      if (ok) {
        uint32_t* w = reinterpret_cast<uint32_t*>(rec + 8) + (d.index >> 5);
        const uint32_t bit = 1u << (d.index & 31u);
        if (d.code) atomicOr(w, bit); else atomicAnd(w, ~bit);
      }
      break;
    }
    case BF_DELTA_TOPO_SLOT:
      *reinterpret_cast<uint32_t*>(rec) = (uint32_t)d.index | ((uint32_t)d.code << 16);
      break;
    default:
      ok = false;
  }
  if (!ok) atomicAdd(P.rejected, 1u);
}

__global__ void __launch_bounds__(256) apply_deltas(const DeltaParams P) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  apply_delta(P, P.deltas[i]);
}

// The deltas of several batches in one launch (bf_resident_tick_touched_many): delta i of the launch is delta i - first[k] of
// batch k for the last k with first[k] <= i; first[n_parts] is the total
__global__ void __launch_bounds__(256) apply_deltas_many(const DeltaParams* __restrict__ parts, const uint32_t* __restrict__ first,
                                                         uint32_t n_parts) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= first[n_parts]) return;
  uint32_t lo = 0, hi = n_parts;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (first[mid] <= i) lo = mid; else hi = mid;
  }
  const DeltaParams& P = parts[lo];
  apply_delta(P, P.deltas[i - first[lo]]);
}

// Touch marks of runs [first, first + n) after an upload: epoch << 1 | 1 ("must list", Resident in ctx.h)
__global__ void __launch_bounds__(256) mark_runs(uint32_t* mark, uint32_t first, uint32_t n, uint32_t value) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) mark[first + i] = value;
}

cudaError_t launch_mark_runs(uint32_t* mark, uint32_t first, uint32_t n, uint32_t value, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  mark_runs<<<(n + 255) / 256, 256, 0, stream>>>(mark, first, n, value);
  return cudaGetLastError();
}

// Arena compaction (topology.cu): record i moves from src + moves[i].x to dst + moves[i].y (moves[i].z bytes, multiples of 16).
// One warp per record, 16 bytes per lane per trip.
__global__ void __launch_bounds__(256) move_records(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, const ulonglong4* __restrict__ moves,
                                                    uint32_t n) {
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
  if (w >= n) return;
  const ulonglong4 m = moves[w];
  const uint4* s = reinterpret_cast<const uint4*>(src + m.x);
  uint4* d = reinterpret_cast<uint4*>(dst + m.y);
  for (unsigned long long i = lane; i < m.z / 16; i += 32) d[i] = s[i];
}

cudaError_t launch_move_records(const uint8_t* src, uint8_t* dst, const void* moves, uint32_t n, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  move_records<<<(n + 7) / 8, 256, 0, stream>>>(src, dst, static_cast<const ulonglong4*>(moves), n);
  return cudaGetLastError();
}

cudaError_t launch_apply_deltas_many(const DeltaParams* parts, const uint32_t* first, uint32_t n_parts, uint32_t n, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  apply_deltas_many<<<(n + 255) / 256, 256, 0, stream>>>(parts, first, n_parts);
  return cudaGetLastError();
}

cudaError_t launch_apply_deltas(const DeltaParams& P, cudaStream_t stream) {
  if (P.n == 0) return cudaSuccess;
  apply_deltas<<<(P.n + 255) / 256, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

// Migration of the runs of one topology slot to another (bf_resident_migrate).  One warp per run: a run of another slot leaves
// after reading its header word.  A run of old_slot stages the code planes its layout has (phase, then cond, then decision) and
// its child area in shared memory, then rebuilds every plane word in place: lane t gathers the codes of new step 32w + t from the
// old step the inverse map names, and one ballot per plane assembles the word.  The child area is zeroed and each kept parallel
// desc's words are copied to their new place (child_first is a multiple of 8 nibbles); the children_registered bits follow their
// descs.  All shared memory is dynamic: word 0 is the CTA's count, the warps' stages start at word 4 (migrate_stage_words each).
__host__ __device__ inline uint32_t migrate_planes(const MigrateParams& P) {
  return 4u + (P.off_cond != BF_OFF_NONE ? 2u : 0u) + (P.off_decision != BF_OFF_NONE ? 2u : 0u);
}
__host__ __device__ inline uint32_t migrate_child_words(const MigrateParams& P) {
  return P.off_child != BF_OFF_NONE ? (P.child_nibbles + 7) / 8 : 0u;
}
__host__ __device__ inline uint32_t migrate_stage_words(const MigrateParams& P) {
  return migrate_planes(P) * P.words + migrate_child_words(P);
}

// The timer slots of a migrated run (whole warp): lane t holds slots t and t + 32, maps each armed step through the step map (a
// gone step, or one past the map, cancels the slot), ranks the survivors by their new step (the map is injective: no ties) and,
// after every lane has read, stores them in that order with empty slots behind.
DI void migrate_timers(const MigrateParams& P, uint32_t run, uint32_t lane) {
  const uint32_t K = P.areas.timer_k;
  unsigned long long* t = P.areas.timers + (size_t)run * K;
  unsigned long long v[2];
  uint32_t to[2];
  for (uint32_t h = 0; h < 2; ++h) {
    const uint32_t k = lane + 32u * h;
    v[h] = k < K ? t[k] : kTimerEmpty;
    to[h] = BF_MIGRATE_GONE;
    if (timer_armed(v[h])) {
      const uint32_t s = timer_step(v[h]);
      to[h] = s < P.n_old_steps ? P.fwd[s] : BF_MIGRATE_GONE;
    }
  }
  uint32_t rank[2] = {0u, 0u}, kept = 0u;
  for (uint32_t j = 0; j < 64u; ++j) {
    const uint32_t tj = __shfl_sync(FULL, to[j >> 5], j & 31u);
    if (tj == BF_MIGRATE_GONE) continue;
    ++kept;
    for (uint32_t h = 0; h < 2; ++h) rank[h] += tj < to[h] ? 1u : 0u;   // a gone slot's rank is never used
  }
  __syncwarp();
  for (uint32_t h = 0; h < 2; ++h) {
    const uint32_t k = lane + 32u * h;
    if (to[h] != BF_MIGRATE_GONE) t[rank[h]] = (v[h] & ~(0xFFFFull << 32)) | (unsigned long long)to[h] << 32;
    if (k >= kept && k < K) t[k] = kTimerEmpty;
  }
}

__global__ void __launch_bounds__(256) migrate_runs(const MigrateParams P) {
  extern __shared__ uint32_t smem[];
  uint32_t& block_count = smem[0];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u, W = P.words;
  const uint32_t np = migrate_planes(P), child_words = migrate_child_words(P);
  if (threadIdx.x == 0) block_count = 0;
  __syncthreads();
  const uint32_t run = blockIdx.x * (blockDim.x >> 5) + warp;
  uint8_t* rec = P.state + (size_t)run * P.state_stride;
  if (run < P.n_runs && *reinterpret_cast<const uint32_t*>(rec) == P.old_slot) {
    uint32_t* st = smem + 4u + warp * migrate_stage_words(P);   // np planes of W words | child words
    const bool has_cond = P.off_cond != BF_OFF_NONE, has_dec = P.off_decision != BF_OFF_NONE;
    // plane k lives at plane_of(k) in the record: 0-3 phase, then cond's two planes, then decision's
    auto plane_of = [&](uint32_t k) -> uint32_t* {
      if (k < 4u) return reinterpret_cast<uint32_t*>(rec + P.off_phase) + k * W;
      if (has_cond && k < 6u) return reinterpret_cast<uint32_t*>(rec + P.off_cond) + (k - 4u) * W;
      return reinterpret_cast<uint32_t*>(rec + P.off_decision) + (k - (has_cond ? 6u : 4u)) * W;
    };
    for (uint32_t i = lane; i < np * W; i += 32u) st[i] = plane_of(i / W)[i % W];   // all lanes load, plane after plane
    uint32_t* child = child_words ? reinterpret_cast<uint32_t*>(rec + P.off_child) : nullptr;
    uint32_t* st_child = st + np * W;
    for (uint32_t i = lane; i < child_words; i += 32u) st_child[i] = child[i];
    const uint64_t reg_old = *reinterpret_cast<const uint64_t*>(rec + 8);
    __syncwarp();
    uint32_t* dst = lane < np ? plane_of(lane) : nullptr;   // lane k stores plane k's words
    for (uint32_t w = 0; w < W; ++w) {
      const uint32_t o = P.inv[w * 32u + lane];
      uint32_t code = 0;
      if (o != BF_MIGRATE_GONE)
        for (uint32_t k = 0; k < np; ++k) code |= ((st[k * W + (o >> 5)] >> (o & 31u)) & 1u) << k;
      uint32_t word = 0;
      for (uint32_t k = 0; k < np; ++k) {
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, (code >> k) & 1u);
        if (lane == k) word = b;
      }
      if (dst) dst[w] = word;
    }
    // child area: nibbles past the layout's child_nibbles (the last word's padding) are kept
    for (uint32_t i = lane; i < child_words; i += 32u) {
      const uint32_t used = P.child_nibbles - i * 8u;
      child[i] = used >= 8u ? 0u : st_child[i] & ~((1u << (4u * used)) - 1u);
    }
    __syncwarp();
    uint64_t reg_new = 0;
    for (uint32_t d = 0; d < P.n_desc; ++d) {
      const MigrateDesc md = P.desc[d];
      reg_new |= ((reg_old >> md.old_p) & 1ull) << md.new_p;
      if (!child_words) continue;
      const uint32_t nw = (md.branches + 7u) / 8u, tail = md.branches & 7u;
      for (uint32_t i = lane; i < nw; i += 32u) {
        uint32_t v = st_child[md.old_first / 8u + i];
        if (i == nw - 1u && tail) v &= (1u << (4u * tail)) - 1u;
        child[md.new_first / 8u + i] = v;
      }
    }
    if (P.areas.timers) migrate_timers(P, run, lane);
    if (lane == 0) {
      drop_baseline(P.areas, run);
      *reinterpret_cast<uint32_t*>(rec) = P.new_slot;
      *reinterpret_cast<uint64_t*>(rec + 8) = reg_new;
      P.mark[run] = P.mark_value;
      atomicAdd(&block_count, 1u);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && block_count) atomicAdd(P.migrated, block_count);
}

// Warps per CTA: 8, fewer when their stages and the 16-byte count header pass the 48 KiB a launch gets without an opt-in.  One
// warp always fits: its stage is at most 8 * 32 + 8192 words (33 KiB).
uint32_t migrate_warps_per_block(const MigrateParams& P) {
  const uint32_t warp_bytes = migrate_stage_words(P) * 4u;
  uint32_t wpb = 8;
  while (wpb > 1 && 16u + wpb * warp_bytes > (48u << 10)) --wpb;
  return wpb;
}

cudaError_t launch_migrate(const MigrateParams& P, cudaStream_t stream) {
  if (P.n_runs == 0) return cudaSuccess;
  const uint32_t wpb = migrate_warps_per_block(P);
  migrate_runs<<<(P.n_runs + wpb - 1) / wpb, wpb * 32, 16u + wpb * migrate_stage_words(P) * 4u, stream>>>(P);
  return cudaGetLastError();
}

// Redrive (bf_resident_redrive).  One warp per request: a run holding another slot leaves after reading its header word.  Lane w
// takes plane word w: it reads word w of the request's reset set R (a closure mask, or the low S bits for BF_REDRIVE_ALL) and
// clears those bits in every phase and decision plane and in cond plane 0; on cond plane 1 it clears them and then sets the ones
// of steps with an `if` (HOLD), read from the topology's HAS_IF plane.  Lane p (and p + 32) takes parallel desc p: when its step
// is in R it zeroes the desc's child nibbles (whole words up to the last, whose padding nibbles a masked AND keeps), and one
// ballot per half gives the children_registered bits lane 0 clears, with BF_RF_TOPOLOGY_TERMINATED, by one atomicAnd each.
// Requests are not sorted by run, and two requests of one run may run at once: every operation drives a bit to a value fixed per
// (run, step) (0, or HAS_IF on cond plane 1), and each request's OR follows its own AND, so any interleaving of two requests
// leaves the same word as applying them one after the other.  Child words outside a desc's tail are only ever stored as 0.
__global__ void __launch_bounds__(256) redrive_runs(const RedriveParams P) {
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
  if (i >= P.n) return;
  const bf_redrive q = P.req[i];
  uint8_t* rec = P.state + (size_t)q.run * P.state_stride;
  const bool hit = *reinterpret_cast<const uint32_t*>(rec) == q.slot;   // no request of this launch writes the slot word
  if (lane == 0) P.status[i] = hit ? 1u : 0u;
  if (!hit) return;
  empty_timers(P.areas, q.run, lane);   // the whole step-timer annotation goes (storyrun_controller.go:477-478, :524-525)
  const uint8_t* topo = reinterpret_cast<const uint8_t*>(P.slots[q.slot].addr);
  const TopoHeader* th = reinterpret_cast<const TopoHeader*>(topo);
  const uint32_t S = th->S, TW = th->W, W = P.words, key = P.key[i];
  uint32_t m = 0;   // word `lane` of R (TW <= W: the topology fits the layout)
  if (lane < TW)
    m = key == BF_REDRIVE_ALL ? (S - lane * 32u >= 32u ? ~0u : (1u << (S - lane * 32u)) - 1u) : P.masks[(size_t)key * W + lane];
  if (m) {
    uint32_t* ph = reinterpret_cast<uint32_t*>(rec + P.off_phase) + lane;
    for (uint32_t b = 0; b < 4; ++b) atomicAnd(ph + b * W, ~m);
    if (P.off_decision != BF_OFF_NONE) {
      uint32_t* dc = reinterpret_cast<uint32_t*>(rec + P.off_decision) + lane;
      atomicAnd(dc, ~m);
      atomicAnd(dc + W, ~m);
    }
    if (P.off_cond != BF_OFF_NONE) {
      uint32_t* cd = reinterpret_cast<uint32_t*>(rec + P.off_cond) + lane;
      const uint32_t hold = m & reinterpret_cast<const uint32_t*>(topo + th->off_planes)[PL_HASIF * TW + lane];
      atomicAnd(cd, ~m);
      atomicAnd(cd + W, ~m);
      if (hold) atomicOr(cd + W, hold);
    }
  }
  const ParDesc* pd = reinterpret_cast<const ParDesc*>(topo + th->off_par);
  const uint32_t n_par = th->P;
  uint32_t reg[2];
  for (uint32_t h = 0; h < 2; ++h) {   // BF_MAX_PARALLEL = 64 descs: lane p and lane p + 32
    const uint32_t p = lane + 32u * h;
    const ParDesc d = p < n_par ? pd[p] : ParDesc{};
    const uint32_t mw = __shfl_sync(0xFFFFFFFFu, m, (d.step >> 5) & 31u);
    const bool in = p < n_par && ((mw >> (d.step & 31u)) & 1u);
    reg[h] = __ballot_sync(0xFFFFFFFFu, in);
    if (in && P.off_child != BF_OFF_NONE) {
      uint32_t* cw = reinterpret_cast<uint32_t*>(rec + P.off_child) + d.child_first / 8u;   // child_first: a multiple of 8 nibbles
      const uint32_t nw = (d.branches + 7u) / 8u, tail = d.branches & 7u;
      for (uint32_t k = 0; k < nw; ++k) {
        if (k == nw - 1u && tail) atomicAnd(cw + k, ~((1u << (4u * tail)) - 1u));
        else cw[k] = 0u;
      }
    }
  }
  if (lane == 0) {
    const unsigned long long gone = (unsigned long long)reg[1] << 32 | reg[0];
    if (gone) atomicAnd(reinterpret_cast<unsigned long long*>(rec + 8), ~gone);
    if (P.areas.runctl) {   // the stop goes (one exchange: of two requests of a run, one restores), the drain deadline too
      bf_run_ctl* ctl = P.areas.runctl + q.run;
      const uint32_t was = atomicExch(reinterpret_cast<uint32_t*>(ctl) + 2, 0u);   // stop | saved_flags << 8
      if (was & 0xFFu) set_byte(rec, 4u, 0xFFu, (was >> 8) & 0xFFu);
      ctl->drain_deadline = BF_TIMER_NONE;
      if (key == BF_REDRIVE_ALL) ctl->story_deadline = BF_TIMER_NONE;   // StartedAt = nil (storyrun_controller.go:414-438)
    }
    atomicAnd(reinterpret_cast<uint32_t*>(rec + 4), ~(uint32_t)BF_RF_TOPOLOGY_TERMINATED);   // run_flags is the low byte
    atomicMax(P.mark + q.run, P.mark_value);   // max: an upload's "must list" bit stays
  }
}

cudaError_t launch_redrive(const RedriveParams& P, cudaStream_t stream) {
  if (P.n == 0) return cudaSuccess;
  redrive_runs<<<(P.n + 7) / 8, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

// Reshape (bf_resident_reshape).  Each new record word is computed from its byte offset o alone, so any pair of layouts that
// pass check_layout works and every word is stored once.  A plane field [to_off, to_off + planes * Wn * 4): word w of plane p
// is word w of plane p at from_off when w < Wo and the old layout has the field, else 0.
DI bool reshape_planes(const uint32_t* src, uint32_t o, uint32_t to_off, uint32_t from_off, uint32_t planes, uint32_t Wn,
                       uint32_t Wo, uint32_t& v) {
  if (to_off == BF_OFF_NONE || o < to_off || o >= to_off + planes * Wn * 4u) return false;
  const uint32_t k = (o - to_off) >> 2, p = k / Wn, w = k - p * Wn;
  v = from_off != BF_OFF_NONE && w < Wo ? src[(from_off >> 2) + p * Wo + w] : 0u;
  return true;
}
DI uint32_t child_area_words(const bf_layout& L) { return ((L.child_nibbles + 1u) / 2u + 3u) / 4u; }

DI uint32_t reshape_state_word(const uint32_t* s, uint32_t o, const bf_layout& F, const bf_layout& T) {
  if (o < 16u) return s[o >> 2];   // bf_run_header
  uint32_t v = 0;
  if (reshape_planes(s, o, T.off_phase, F.off_phase, 4, T.words, F.words, v) ||
      reshape_planes(s, o, T.off_cond, F.off_cond, 2, T.words, F.words, v) ||
      reshape_planes(s, o, T.off_decision, F.off_decision, 2, T.words, F.words, v))
    return v;
  if (T.off_child != BF_OFF_NONE && o >= T.off_child && o < T.off_child + child_area_words(T) * 4u) {
    const uint32_t k = (o - T.off_child) >> 2;   // child_first does not depend on the layout: the old bytes stay in place
    return F.off_child != BF_OFF_NONE && k < child_area_words(F) ? s[(F.off_child >> 2) + k] : 0u;
  }
  return 0u;   // padding
}

DI uint32_t reshape_result_word(const uint32_t* s, uint32_t o, const bf_layout& F, const bf_layout& T) {
  if (o < 16u) return s[o >> 2];   // bf_result_header
  uint32_t v = 0;
  if (reshape_planes(s, o, T.off_ready, F.off_ready, 1, T.words, F.words, v) ||
      reshape_planes(s, o, T.off_skip, F.off_skip, 1, T.words, F.words, v) ||
      reshape_planes(s, o, T.off_fail, F.off_fail, 1, T.words, F.words, v) ||
      reshape_planes(s, o, T.off_needs_cond, F.off_needs_cond, 1, T.words, F.words, v) ||
      reshape_planes(s, o, T.off_skip_dep, F.off_skip_dep, 1, T.words, F.words, v) ||
      reshape_planes(s, o, T.off_phase_out, F.off_phase_out, 4, T.words, F.words, v))
    return v;
  return 0u;   // stride padding, as store_words leaves it
}

// One warp per run of the new capacity; lane t stores words t, t + 32, ... of the new state record, then of the new result
// record (coalesced 4-byte stores; planes start on 8-byte boundaries with an odd word count, so no 16-byte vectors).
// Runs at or above n_old get zero records.
__global__ void __launch_bounds__(256) reshape_runs(const ReshapeParams P) {
  const uint32_t r = blockIdx.x * 8u + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
  if (r >= P.n_new) return;
  const bool keep = r < P.n_old;
  const uint32_t* s = reinterpret_cast<const uint32_t*>(P.old_state + (size_t)r * P.from.state_stride);
  uint32_t* d = reinterpret_cast<uint32_t*>(P.state + (size_t)r * P.to.state_stride);
  for (uint32_t o = lane * 4u; o < P.to.state_stride; o += 128u) d[o >> 2] = keep ? reshape_state_word(s, o, P.from, P.to) : 0u;
  s = reinterpret_cast<const uint32_t*>(P.old_result + (size_t)r * P.from.result_stride);
  d = reinterpret_cast<uint32_t*>(P.result + (size_t)r * P.to.result_stride);
  for (uint32_t o = lane * 4u; o < P.to.result_stride; o += 128u) d[o >> 2] = keep ? reshape_result_word(s, o, P.from, P.to) : 0u;
  if (lane == 0) keep_areas(P.old_areas, P.areas, r, keep);
}

cudaError_t launch_reshape(const ReshapeParams& P, cudaStream_t stream) {
  if (P.n_new == 0) return cudaSuccess;
  reshape_runs<<<(P.n_new - 1u) / 8u + 1u, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

// Retire (bf_resident_retire).  One warp per vacated index m + i: when the run there lives on, the warp copies its state record
// and current result record to its target (16-byte accesses, lane t takes vectors t, t + 32, ...) and its side areas, and lane 0
// marks the target; then the warp zeroes the vacated state record and its mark and vacates its areas.  Targets lie below m and
// vacated indices at or above it, and each lane zeroes only the vectors and slots it read itself, so no warp reads what another
// writes.
__global__ void __launch_bounds__(256) retire_runs(const RetireParams P) {
  const uint32_t i = blockIdx.x * 8u + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
  if (i >= P.n) return;
  const uint32_t from = P.m + i, to = P.to[i], sv = P.state_stride >> 4;
  uint4* s = reinterpret_cast<uint4*>(P.state + (size_t)from * P.state_stride);
  if (to != kRetireNoMove) {
    uint4* d = reinterpret_cast<uint4*>(P.state + (size_t)to * P.state_stride);
    for (uint32_t k = lane; k < sv; k += 32u) d[k] = s[k];
    const uint4* rs = reinterpret_cast<const uint4*>(P.result + (size_t)from * P.result_stride);
    uint4* rd = reinterpret_cast<uint4*>(P.result + (size_t)to * P.result_stride);
    for (uint32_t k = lane; k < (P.result_stride >> 4); k += 32u) rd[k] = rs[k];
    if (lane == 0) P.mark[to] = P.mark_value;
    arrive_areas(P.areas, from, P.areas, to, lane);
  }
  for (uint32_t k = lane; k < sv; k += 32u) s[k] = make_uint4(0u, 0u, 0u, 0u);
  if (lane == 0) P.mark[from] = 0u;
  vacate_areas(P.areas, from, lane);
}

cudaError_t launch_retire(const RetireParams& P, cudaStream_t stream) {
  if (P.n == 0) return cudaSuccess;
  retire_runs<<<(P.n - 1u) / 8u + 1u, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

// Extent (bf_resident_extent, bf_resident_narrow).  Word o of a record lies in the plane field at `off` (planes * W words): w is
// its word within its plane.
DI bool in_planes(uint32_t o, uint32_t off, uint32_t planes, uint32_t W, uint32_t& w) {
  if (off == BF_OFF_NONE || o < off || o >= off + planes * W * 4u) return false;
  w = ((o - off) >> 2) % W;
  return true;
}
// steps needed by plane word w holding v: one past its highest set bit
DI uint32_t word_extent(uint32_t w, uint32_t v) { return v ? 32u * w + 32u - __clz(v) : 0u; }

// State word o holding v: the steps its codes need, the nibbles of the child area it needs, the input fields it needs.
DI void state_word_extent(const bf_layout& L, uint32_t o, uint32_t v, uint32_t& steps, uint32_t& child, uint32_t& fields) {
  if (o < 16u || v == 0u) return;   // bf_run_header
  uint32_t w;
  if (in_planes(o, L.off_phase, 4, L.words, w)) {
    steps = max(steps, word_extent(w, v));
  } else if (in_planes(o, L.off_cond, 2, L.words, w)) {
    steps = max(steps, word_extent(w, v));
    fields |= BF_F_COND;
  } else if (in_planes(o, L.off_decision, 2, L.words, w)) {
    steps = max(steps, word_extent(w, v));
    fields |= BF_F_DECISION;
  } else if (L.off_child != BF_OFF_NONE && o >= L.off_child && o < L.off_child + child_area_words(L) * 4u) {
    const uint32_t first = ((o - L.off_child) >> 2) * 8u;   // nibbles first .. first + 7, those below child_nibbles count
    if (first >= L.child_nibbles) return;
    const uint32_t n = min(8u, L.child_nibbles - first), m = n == 8u ? v : v & ((1u << (4u * n)) - 1u);
    if (m) { child = max(child, first + (31u - __clz(m)) / 4u + 1u); fields |= BF_F_CHILD; }
  }
}

// Result word o holding v: the steps its masks need (only the fields R places count).
DI uint32_t result_word_extent(const bf_layout& R, uint32_t o, uint32_t v) {
  uint32_t w;
  if (o >= 16u && v && (in_planes(o, R.off_ready, 1, R.words, w) || in_planes(o, R.off_skip, 1, R.words, w) ||
                        in_planes(o, R.off_fail, 1, R.words, w) || in_planes(o, R.off_needs_cond, 1, R.words, w) ||
                        in_planes(o, R.off_skip_dep, 1, R.words, w) || in_planes(o, R.off_phase_out, 4, R.words, w)))
    return word_extent(w, v);
  return 0u;
}

// The timer slots of one run (lane t reads slots t, t + 32): an armed step s needs s + 1 steps, a code that writes needs the
// decision planes.  -> the armed slots this lane saw
DI uint32_t timer_extent(const unsigned long long* t, uint32_t K, uint32_t lane, uint32_t& steps, uint32_t& fields) {
  uint32_t armed = 0u;
  for (uint32_t k = lane; k < K; k += 32u) {
    const unsigned long long v = t[k];
    if (!timer_armed(v)) continue;
    ++armed;
    steps = max(steps, timer_step(v) + 1u);
    if (timer_code(v) != BF_DEC_PENDING) fields |= BF_F_DECISION;
  }
  return armed;
}

// The extent of run r of B (one warp; each lane's part, which the caller reduces): lane t reads the 16-byte vectors t, t + 32, ...
// of its state record and slots t, t + 32 of its timers; when r is a run, also of its result record when a later tick compares
// with it (the fields B.R places), and lane 0 adds the S and the child area of its topology when its slot is alive.  -> the
// armed slots this lane saw
DI uint32_t run_extent(const ExtentBatch& B, uint32_t r, bool is_run, uint32_t lane, uint32_t& steps, uint32_t& child, uint32_t& fields) {
  const uint8_t* s = B.state + (size_t)r * B.L.state_stride;
  for (uint32_t o = lane * 16u; o < B.L.state_stride; o += 512u) {
    const uint4 q = *reinterpret_cast<const uint4*>(s + o);
    state_word_extent(B.L, o, q.x, steps, child, fields);
    state_word_extent(B.L, o + 4u, q.y, steps, child, fields);
    state_word_extent(B.L, o + 8u, q.z, steps, child, fields);
    state_word_extent(B.L, o + 12u, q.w, steps, child, fields);
  }
  const RunAreasView& A = B.areas;
  const uint32_t armed = A.timers ? timer_extent(A.timers + (size_t)r * A.timer_k, A.timer_k, lane, steps, fields) : 0u;
  if (!is_run) return armed;
  const uint32_t m = B.mark[r];
  const bool baseline = r < B.prev_runs || (r < B.eval_runs && !((m & 1u) && (m >> 1) > B.full_epoch));
  const uint8_t* res = B.result + (size_t)r * B.L.result_stride;
  for (uint32_t o = lane * 16u; baseline && o < B.L.result_stride; o += 512u) {
    const uint4 q = *reinterpret_cast<const uint4*>(res + o);
    steps = max(steps, max(max(result_word_extent(B.R, o, q.x), result_word_extent(B.R, o + 4u, q.y)),
                           max(result_word_extent(B.R, o + 8u, q.z), result_word_extent(B.R, o + 12u, q.w))));
  }
  if (lane == 0) {
    const uint32_t slot = *reinterpret_cast<const uint32_t*>(s);
    const Slot sl = slot < B.n_slots ? B.slots[slot] : Slot{};
    if (sl.addr) {
      steps = max(steps, sl.meta & 0xFFFFu);
      child = max(child, (uint32_t)reinterpret_cast<const TopoHeader*>(sl.addr)->child_nibbles);
    }
  }
  return armed;
}

// One warp per record, grid-stride, each record streamed once with coalesced loads (run_extent; the runs are those below n_runs).
// Warp reductions, then each warp folds its record's extents into its running maxima (its records ascend, so the running maximum
// keeps the lowest index), the CTA's warps meet in shared memory and one thread per CTA adds the CTA's three words to P.out.
__global__ void __launch_bounds__(256) extent_runs(const ExtentParams P) {
  __shared__ unsigned long long cta[3];
  if (threadIdx.x < 3) cta[threadIdx.x] = 0ull;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31u, warps = gridDim.x * 8u;
  unsigned long long best_steps = 0ull, best_child = 0ull;
  uint32_t all_fields = 0u;
  for (uint32_t r = blockIdx.x * 8u + (threadIdx.x >> 5); r < P.n_records; r += warps) {
    uint32_t steps = 0u, child = 0u, fields = 0u;
    run_extent(P.B, r, r < P.n_runs, lane, steps, child, fields);
    steps = __reduce_max_sync(FULL, steps);
    child = __reduce_max_sync(FULL, child);
    all_fields |= __reduce_or_sync(FULL, fields);
    const unsigned long long idx = ~r & 0xFFFFFFFFull;
    if (steps) best_steps = max(best_steps, (unsigned long long)steps << 32 | idx);
    if (child) best_child = max(best_child, (unsigned long long)child << 32 | idx);
  }
  if (lane == 0) {
    if (best_steps) atomicMax(&cta[0], best_steps);
    if (best_child) atomicMax(&cta[1], best_child);
    if (all_fields) atomicOr(&cta[2], (unsigned long long)all_fields);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (cta[0]) atomicMax(P.out, cta[0]);
    if (cta[1]) atomicMax(P.out + 1, cta[1]);
    if (cta[2]) atomicOr(P.out + 2, cta[2]);
  }
}

cudaError_t launch_extent(const ExtentParams& P, uint32_t sm_count, cudaStream_t stream) {
  if (P.n_records == 0) return cudaSuccess;
  const uint32_t grid = min((P.n_records - 1u) / 8u + 1u, max(sm_count, 1u) * 8u);   // 8 CTAs of 8 warps per SM at most
  extent_runs<<<grid, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

// Transfer (bf_resident_transfer), fit check.  One warp per listed run: its extent as extent_runs takes it (run_extent, counting
// the result planes T keeps).  Lane 0 stores the run's extent and, when T cannot hold it, lowers P.unfit to its position.
__global__ void __launch_bounds__(256) transfer_fit(const TransferParams P) {
  const uint32_t i = blockIdx.x * 8u + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
  if (i >= P.n) return;
  const uint32_t r = P.runs[i];
  uint32_t steps = 0u, child = 0u, fields = 0u;
  uint32_t armed = run_extent(P.src, r, true, lane, steps, child, fields);
  steps = __reduce_max_sync(FULL, steps);
  child = __reduce_max_sync(FULL, child);
  fields = __reduce_or_sync(FULL, fields);
  armed = __reduce_add_sync(FULL, armed);
  if (lane == 0) {
    const bf_layout& T = P.T;
    const uint32_t placed = (T.off_cond != BF_OFF_NONE ? BF_F_COND : 0u) | (T.off_decision != BF_OFF_NONE ? BF_F_DECISION : 0u) |
                            (T.off_child != BF_OFF_NONE ? BF_F_CHILD : 0u);
    const bf_run_ctl* ctl = P.src.areas.runctl;
    const bool ctl_lost = ctl && !P.dst_areas.runctl && !runctl_default(ctl[r]);   // no area to arrive in
    P.extent[i] = make_uint4(steps, child, fields, armed | (ctl_lost ? 0x80000000u : 0u));
    if (steps > T.steps_max || (T.off_child != BF_OFF_NONE && child > T.child_nibbles) || (fields & ~placed) ||
        armed > P.dst_areas.timer_k || ctl_lost)
      atomicMin(P.unfit, i);
  }
}

// Transfer, the move.  One warp per listed run: lane t stores words t, t + 32, ... of destination record dst_first + i, each
// re-laid from src.L to T by its byte offset as reshape_runs does (state, then current result), lane 0 marks the arrival, and
// the run's side areas arrive with it.  The source records are only read; retire_runs compacts the source behind this launch on
// the same stream.
__global__ void __launch_bounds__(256) transfer_runs(const TransferParams P) {
  const uint32_t i = blockIdx.x * 8u + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
  if (i >= P.n) return;
  const uint32_t r = P.runs[i], to = P.dst_first + i;
  const bf_layout& F = P.src.L;
  const uint32_t* s = reinterpret_cast<const uint32_t*>(P.src.state + (size_t)r * F.state_stride);
  uint32_t* d = reinterpret_cast<uint32_t*>(P.dst_state + (size_t)to * P.T.state_stride);
  for (uint32_t o = lane * 4u; o < P.T.state_stride; o += 128u) d[o >> 2] = reshape_state_word(s, o, F, P.T);
  s = reinterpret_cast<const uint32_t*>(P.src.result + (size_t)r * F.result_stride);
  d = reinterpret_cast<uint32_t*>(P.dst_result + (size_t)to * P.T.result_stride);
  for (uint32_t o = lane * 4u; o < P.T.result_stride; o += 128u) d[o >> 2] = reshape_result_word(s, o, F, P.T);
  if (lane == 0) P.dst_mark[to] = P.mark_value;
  arrive_areas(P.src.areas, r, P.dst_areas, to, lane);
}

cudaError_t launch_transfer_fit(const TransferParams& P, cudaStream_t stream) {
  if (P.n == 0) return cudaSuccess;
  transfer_fit<<<(P.n - 1u) / 8u + 1u, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

cudaError_t launch_transfer(const TransferParams& P, cudaStream_t stream) {
  if (P.n == 0) return cudaSuccess;
  transfer_runs<<<(P.n - 1u) / 8u + 1u, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

// Transfer to another ctx (bf_resident_transfer_ctx), the gather on the source.  One warp per listed run: lane t copies the
// 16-byte vectors t, t + 32, ... of its state and current result records into staged run i, the header's slot mapped to the
// destination's, and timer slots t, t + 32; lane 0 copies its limiter inputs and run control and writes its identity index, its
// baseline mark and its slot verdict (GatherParams).  The source is only read, so a refusal later leaves it as it was.
__global__ void __launch_bounds__(256) gather_runs(const GatherParams P) {
  const uint32_t i = blockIdx.x * 8u + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
  if (i >= P.n) return;
  const ExtentBatch& B = P.src;
  const uint32_t r = P.runs[i];
  const uint4* s = reinterpret_cast<const uint4*>(B.state + (size_t)r * B.L.state_stride);
  const uint32_t slot = s[0].x;
  const uint32_t to = slot < P.n_slot_map ? P.slot_map[slot] : BF_SLOT_NONE;
  const uint32_t why = slot >= P.n_slot_map ? (uint32_t)BF_UNFIT_SLOT_PAST_MAP
                       : to == BF_SLOT_NONE ? (uint32_t)BF_UNFIT_SLOT_UNMAPPED
                       : to == kSlotDead    ? (uint32_t)BF_UNFIT_SLOT_DEAD
                                            : (uint32_t)BF_UNFIT_NONE;
  uint4* d = reinterpret_cast<uint4*>(P.state + (size_t)i * B.L.state_stride);
  for (uint32_t k = lane; k < (B.L.state_stride >> 4); k += 32u) {
    uint4 v = s[k];
    if (k == 0 && why == BF_UNFIT_NONE) v.x = to;
    d[k] = v;
  }
  const uint4* rs = reinterpret_cast<const uint4*>(B.result + (size_t)r * B.L.result_stride);
  uint4* rd = reinterpret_cast<uint4*>(P.result + (size_t)i * B.L.result_stride);
  for (uint32_t k = lane; k < (B.L.result_stride >> 4); k += 32u) rd[k] = rs[k];
  const RunAreasView& A = B.areas;
  for (uint32_t k = lane; A.timers && k < A.timer_k; k += 32u) P.areas.timers[(size_t)i * A.timer_k + k] = A.timers[(size_t)r * A.timer_k + k];
  if (lane != 0) return;
  if (A.sched_in) P.areas.sched_in[i] = A.sched_in[r];
  if (A.runctl) P.areas.runctl[i] = A.runctl[r];
  const uint32_t m = B.mark[r];
  const bool baseline = r < B.prev_runs || (r < B.eval_runs && !((m & 1u) && (m >> 1) > B.full_epoch));
  P.mark[i] = baseline ? 0u : 3u;
  P.ident[i] = i;
  P.reason[i] = why;
  if (why != BF_UNFIT_NONE) atomicMin(P.unfit, i);
}

cudaError_t launch_gather(const GatherParams& P, cudaStream_t stream) {
  if (P.n == 0) return cudaSuccess;
  gather_runs<<<(P.n - 1u) / 8u + 1u, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

// ---- step timers (bf_resident_timers*, bf_resident_fire) ----------------------------------------------------------------------
// Relay (bf_resident_timers, reshape): one thread per slot of the new area.
__global__ void __launch_bounds__(256) relay_timers(const TimerRelayParams P) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)P.n * P.dst_k) return;
  const uint32_t r = (uint32_t)(i / P.dst_k), k = (uint32_t)(i % P.dst_k);
  P.dst[i] = P.src && r < P.n_src && k < P.src_k ? P.src[(size_t)r * P.src_k + k] : kTimerEmpty;
}

cudaError_t launch_relay_timers(const TimerRelayParams& P, cudaStream_t stream) {
  const size_t n = (size_t)P.n * P.dst_k;
  if (n == 0) return cudaSuccess;
  relay_timers<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(P);
  return cudaGetLastError();
}

// the first index of req[lo, hi) whose step is >= s (requests of one group ascend by step)
DI uint32_t req_lower_bound(const bf_timer* req, uint32_t lo, uint32_t hi, uint32_t s) {
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (req[mid].step < s) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Arm, both launches: one warp per request group (one run).  The warp stages the run's slots in shared memory and marks the armed
// slots a request names (replaced or cancelled).  The check launch counts the run's armed slots after the merge and lowers
// P.overflow to its group when they pass timer_k; the merge launch, which runs only when no group overflows, stores every kept
// slot and every arming request at its rank by step: a kept slot at its index among the kept slots plus the arming requests of
// lower steps, a request at its index among the arming requests plus the kept slots of lower steps.  Empty slots follow.
template <bool kMerge>
__global__ void __launch_bounds__(256) arm_timers(const TimerArmParams P) {
  __shared__ unsigned long long stage[8][BF_TIMER_MAX_SLOTS];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u, g = blockIdx.x * 8u + warp;
  if (g >= P.n_groups) return;
  const uint32_t lo = P.first[g], hi = P.first[g + 1], K = P.timer_k, run = P.req[lo].run;
  unsigned long long* t = P.timers + (size_t)run * K;
  unsigned long long* st = stage[warp];
  uint32_t matched[2], armed[2];
  for (uint32_t h = 0; h < 2; ++h) {
    const uint32_t k = lane + 32u * h;
    const unsigned long long v = k < K ? t[k] : kTimerEmpty;
    st[k] = v;
    const bool a = timer_armed(v);
    const uint32_t j = a ? req_lower_bound(P.req, lo, hi, timer_step(v)) : hi;
    armed[h] = __ballot_sync(FULL, a);
    matched[h] = __ballot_sync(FULL, a && j < hi && P.req[j].step == timer_step(v));
  }
  const uint32_t arms = P.arm_before[hi] - P.arm_before[lo];
  const uint32_t E = __popc(armed[0]) + __popc(armed[1]), M = __popc(matched[0]) + __popc(matched[1]), total = E - M + arms;
  if (!kMerge) {
    if (lane == 0 && total > K) atomicMin(P.overflow, g);
    return;
  }
  __syncwarp();
  auto matched_below = [&](uint32_t k) {   // matched slots among [0, k)
    return k <= 32u ? __popc(matched[0] & (k == 32u ? FULL : (1u << k) - 1u))
                    : __popc(matched[0]) + __popc(matched[1] & (k == 64u ? FULL : (1u << (k - 32u)) - 1u));
  };
  for (uint32_t h = 0; h < 2; ++h) {   // kept slots
    const uint32_t k = lane + 32u * h;
    if (k >= E || ((matched[h] >> lane) & 1u)) continue;
    const unsigned long long v = st[k];
    const uint32_t j = req_lower_bound(P.req, lo, hi, timer_step(v));
    t[k - matched_below(k) + P.arm_before[j] - P.arm_before[lo]] = v;
  }
  for (uint32_t j = lo + lane; j < hi; j += 32u) {   // arming requests
    const bf_timer q = P.req[j];
    if (q.deadline == BF_TIMER_NONE) continue;
    uint32_t a = 0, b = E;   // kept or matched slots of lower steps: the first staged slot at or above q.step
    while (a < b) {
      const uint32_t mid = (a + b) >> 1;
      if (timer_step(st[mid]) < q.step) a = mid + 1; else b = mid;
    }
    t[P.arm_before[j] - P.arm_before[lo] + a - matched_below(a)] =
        (unsigned long long)q.deadline | (unsigned long long)q.step << 32 | (unsigned long long)q.code << 48;
  }
  for (uint32_t k = total + lane; k < K; k += 32u) t[k] = kTimerEmpty;
}

cudaError_t launch_arm_timers(const TimerArmParams& P, bool merge, cudaStream_t stream) {
  if (P.n_groups == 0) return cudaSuccess;
  const uint32_t grid = (P.n_groups - 1u) / 8u + 1u;
  if (merge) arm_timers<true><<<grid, 256, 0, stream>>>(P);
  else arm_timers<false><<<grid, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

// the code of step s in the nbits planes at `off`
DI uint32_t get_planes(const uint8_t* rec, uint32_t off, uint32_t words, uint32_t nbits, uint32_t s) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(rec + off) + (s >> 5);
  uint32_t code = 0;
  for (uint32_t b = 0; b < nbits; ++b) code |= ((w[b * words] >> (s & 31u)) & 1u) << b;
  return code;
}

// One run's armed slots against `now`: fired (due, step not terminal) -> 1, pruned (step terminal) -> 2, kept -> 0
DI uint32_t fire_kind(const FireParams& P, const uint8_t* rec, unsigned long long v) {
  if ((BF_LUT_TERMINAL >> get_planes(rec, P.off_phase, P.words, 4, timer_step(v))) & 1u) return 2u;
  return timer_deadline(v) <= P.now ? 1u : 0u;
}
// a run whose story timeout fires now: not stopped and its story deadline due
DI bool story_fires(const FireParams& P, const bf_run_ctl& c) { return !c.stop && deadline_due(c.story_deadline, P.now); }
DI uint32_t fired_of_run(const FireParams& P, uint32_t r) {
  if (r >= P.n_runs) return 0u;
  uint32_t n = 0;
  if (P.areas.runctl) {   // run level: the drain deadline, and a story timeout, which stands for every step slot
    const bf_run_ctl c = P.areas.runctl[r];
    n = deadline_due(c.drain_deadline, P.now) ? 1u : 0u;
    if (story_fires(P, c)) return n + 1u;
  }
  const uint8_t* rec = P.state + (size_t)r * P.state_stride;
  const unsigned long long* t = P.areas.timers + (size_t)r * P.areas.timer_k;
  for (uint32_t k = 0; k < P.areas.timer_k; ++k) {
    const unsigned long long v = t[k];
    if (!timer_armed(v)) break;   // armed slots lead
    n += fire_kind(P, rec, v) == 1u ? 1u : 0u;
  }
  return n;
}

// Fire, first launch: one thread per run (a warp per chunk of 32 runs) counts its fired timers; each CTA stores its total.  CTA 0
// initialises the four output words, which the second launch accumulates into.
__global__ void __launch_bounds__(256) fire_count(const FireParams P) {
  __shared__ uint32_t warp_sum[8];
  const uint32_t r = blockIdx.x * 256u + threadIdx.x, lane = threadIdx.x & 31u;
  const uint32_t n = __reduce_add_sync(FULL, fired_of_run(P, r));
  if (lane == 0) warp_sum[threadIdx.x >> 5] = n;
  if (blockIdx.x == 0 && threadIdx.x < 4) P.out[threadIdx.x] = threadIdx.x == 3 ? BF_TIMER_NONE : 0u;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t sum = 0;
    for (uint32_t w = 0; w < 8; ++w) sum += warp_sum[w];
    P.block_sums[blockIdx.x] = sum;
  }
}

// Fire, second launch: each CTA sums the totals of the CTAs before it, scans its runs' counts (the same counts: nothing changed
// in between) and each thread walks its run's slots once: a pruned slot goes, a fired one is listed at its place in run order
// (written when its code writes and the decision code is still PENDING: the planes of the delta scatter, and the touch mark), a
// kept one moves down over the gaps; empty slots close the run.  Warp sums and a warp minimum go to the four output words.
__global__ void __launch_bounds__(256) fire_apply(const FireParams P) {
  __shared__ uint32_t base_part[8], warp_incl[8];
  const uint32_t r = blockIdx.x * 256u + threadIdx.x, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t before = 0;   // fired timers of the CTAs before this one: each warp sums a strided share
  for (uint32_t b = threadIdx.x; b < blockIdx.x; b += 256u) before += P.block_sums[b];
  before = __reduce_add_sync(FULL, before);
  const uint32_t mine = fired_of_run(P, r);
  uint32_t incl = mine;   // inclusive warp scan
  for (uint32_t d = 1; d < 32; d <<= 1) {
    const uint32_t x = __shfl_up_sync(FULL, incl, d);
    if (lane >= d) incl += x;
  }
  if (lane == 31) warp_incl[warp] = incl;
  if (lane == 0) base_part[warp] = before;
  __syncthreads();
  uint32_t pos = incl - mine;
  for (uint32_t w = 0; w < 8; ++w) pos += base_part[w] + (w < warp ? warp_incl[w] : 0u);
  uint32_t written = 0, pruned = 0, next = BF_TIMER_NONE, touched = 0;
  if (r < P.n_runs && P.areas.runctl && story_fires(P, P.areas.runctl[r])) {   // the story timeout: no step slot fires, each is pruned
    uint8_t* rec = P.state + (size_t)r * P.state_stride;
    bf_run_ctl* ctl = P.areas.runctl + r;
    for (uint32_t k = 0; k < P.areas.timer_k && timer_armed(P.areas.timers[(size_t)r * P.areas.timer_k + k]); ++k) ++pruned;
    const uint32_t drain = ctl->drain_deadline;
    stop_run(rec, ctl, r, BF_STOP_TIMEOUT, StopParams{P.areas, P.mark, P.mark_value});
    written = 1u;
    if (deadline_due(drain, P.now)) {   // BF_FIRED_DRAIN < BF_FIRED_STORY: listed first
      ctl->drain_deadline = BF_TIMER_NONE;
      if (pos < P.fired_cap) P.fired[pos] = bf_fired{r, (uint16_t)BF_FIRED_DRAIN, (uint8_t)BF_DEC_PENDING, 0u};
      ++pos;
    } else if (drain != BF_TIMER_NONE) {
      next = drain;
    }
    if (pos < P.fired_cap) P.fired[pos] = bf_fired{r, (uint16_t)BF_FIRED_STORY, (uint8_t)BF_DEC_TIMED_OUT, 1u};
  } else if (r < P.n_runs) {
    uint8_t* rec = P.state + (size_t)r * P.state_stride;
    unsigned long long* t = P.areas.timers + (size_t)r * P.areas.timer_k;
    uint32_t keep = 0, k = 0;
    for (; k < P.areas.timer_k; ++k) {
      const unsigned long long v = t[k];
      if (!timer_armed(v)) break;
      const uint32_t kind = fire_kind(P, rec, v);
      if (kind == 2u) { ++pruned; continue; }
      if (kind == 0u) { t[keep++] = v; next = min(next, timer_deadline(v)); continue; }
      const uint32_t s = timer_step(v), code = timer_code(v);
      bool w = false;
      if (code != BF_DEC_PENDING && P.off_decision != BF_OFF_NONE && get_planes(rec, P.off_decision, P.words, 2, s) == BF_DEC_PENDING) {
        set_planes(rec, P.off_decision, P.words, 2, s, code);
        w = true;
      }
      written += w ? 1u : 0u;
      touched |= w ? 1u : 0u;
      if (pos < P.fired_cap) P.fired[pos] = bf_fired{r, (uint16_t)s, (uint8_t)code, (uint8_t)(w ? 1u : 0u)};
      ++pos;
    }
    for (uint32_t e = keep; e < k; ++e) t[e] = kTimerEmpty;
    if (touched) atomicMax(P.mark + r, P.mark_value);   // max: an upload's "must list" bit stays
    if (P.areas.runctl) {   // after the steps (BF_FIRED_DRAIN sorts above every step); a stopped run's story deadline is dormant
      bf_run_ctl* ctl = P.areas.runctl + r;
      const uint32_t drain = ctl->drain_deadline;
      if (deadline_due(drain, P.now)) {
        ctl->drain_deadline = BF_TIMER_NONE;
        if (pos < P.fired_cap) P.fired[pos] = bf_fired{r, (uint16_t)BF_FIRED_DRAIN, (uint8_t)BF_DEC_PENDING, 0u};
      } else {
        next = min(next, drain);
      }
      if (!ctl->stop) next = min(next, ctl->story_deadline);
    }
  }
  const uint32_t f = __reduce_add_sync(FULL, mine), wr = __reduce_add_sync(FULL, written), pr = __reduce_add_sync(FULL, pruned);
  next = __reduce_min_sync(FULL, next);
  if (lane == 0) {
    if (f) atomicAdd(P.out, f);
    if (wr) atomicAdd(P.out + 1, wr);
    if (pr) atomicAdd(P.out + 2, pr);
    if (next != BF_TIMER_NONE) atomicMin(P.out + 3, next);
  }
}

cudaError_t launch_fire(const FireParams& P, cudaStream_t stream) {
  if (P.n_runs == 0) return cudaSuccess;
  const uint32_t grid = (P.n_runs - 1u) / 256u + 1u;
  fire_count<<<grid, 256, 0, stream>>>(P);
  fire_apply<<<grid, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

// One CTA: for each of K arrays of n_ctas per-CTA totals (array k at cta + k * n_ctas), the totals become the sums of the CTAs
// before each (exclusive scan in place); array k's sum goes to total[k].  The K arrays are walked together in chunks of 1024, a
// warp scan and a scan of the warp totals per chunk, carrying the running sums.  bf_resident_status scans its events (K = 1),
// bf_resident_schedule its listed runs and events, bf_resident_resync its items and drifted runs, bf_resident_commit_journal its
// items and written runs (K = 2).
template <uint32_t K>
DI void cta_scan_body(unsigned long long* cta, unsigned long long* total, uint32_t n_ctas) {
  __shared__ unsigned long long s_e[K][32];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  unsigned long long carry[K] = {};
  for (uint32_t base = 0; base < n_ctas; base += 1024u) {
    const uint32_t i = base + threadIdx.x;
    unsigned long long e[K], ie[K];
    for (uint32_t k = 0; k < K; ++k) ie[k] = e[k] = i < n_ctas ? cta[(size_t)k * n_ctas + i] : 0ull;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1)
      for (uint32_t k = 0; k < K; ++k) {
        const unsigned long long b = __shfl_up_sync(FULL, ie[k], d);
        if ((int)lane >= d) ie[k] += b;
      }
    if (lane == 31)
      for (uint32_t k = 0; k < K; ++k) s_e[k][warp] = ie[k];
    __syncthreads();
    if (warp == 0) {   // the warp totals' inclusive scans
      for (uint32_t k = 0; k < K; ++k) {
        unsigned long long we = s_e[k][lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const unsigned long long b = __shfl_up_sync(FULL, we, d);
          if ((int)lane >= d) we += b;
        }
        s_e[k][lane] = we;
      }
    }
    __syncthreads();
    for (uint32_t k = 0; k < K; ++k) {
      if (i < n_ctas) cta[(size_t)k * n_ctas + i] = carry[k] + (warp ? s_e[k][warp - 1] : 0ull) + ie[k] - e[k];
      carry[k] += s_e[k][31];
    }
    __syncthreads();   // s_e is rewritten by the next chunk
  }
  if (threadIdx.x == 0)
    for (uint32_t k = 0; k < K; ++k) total[k] = carry[k];
}
template <uint32_t K>
__global__ void __launch_bounds__(1024) cta_scan(unsigned long long* cta, unsigned long long* total, uint32_t n_ctas) {
  cta_scan_body<K>(cta, total, n_ctas);
}
// The journal scan of a touched commit: one total per block of 8 list positions, ceil(*n_list / 8) of them
template <uint32_t K>
__global__ void __launch_bounds__(1024) cta_scan_list(unsigned long long* cta, unsigned long long* total, const unsigned long long* n_list) {
  cta_scan_body<K>(cta, total, (uint32_t)((*n_list + 7u) / 8u));
}

cudaError_t launch_cta_scan(unsigned long long* cta, unsigned long long* total, uint32_t n_ctas, uint32_t K, cudaStream_t stream) {
  if (K == 1) cta_scan<1><<<1, 1024, 0, stream>>>(cta, total, n_ctas);
  else cta_scan<2><<<1, 1024, 0, stream>>>(cta, total, n_ctas);
  return cudaGetLastError();
}

// Past 48 KiB of dynamic shared memory a kernel opts in before its launch.
template <class... Params>
static cudaError_t allow_smem(void (*kernel)(Params...), uint32_t smem_bytes) {
  return smem_bytes > 48u * 1024u ? cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes)
                                  : cudaSuccess;
}

// The count launch, cta_scan over its K arrays of CTA totals and the list launch of P.n runs, P.warps_per_block warps and
// smem_bytes of shared stages per CTA (bf_resident_status, bf_resident_resync).
template <uint32_t K, class Params>
static cudaError_t launch_listing(void (*count)(Params), void (*list)(Params), const Params& P, uint32_t smem_bytes, cudaStream_t stream) {
  if (P.n == 0) return cudaSuccess;
  cudaError_t e = allow_smem(count, smem_bytes);
  if (e == cudaSuccess) e = allow_smem(list, smem_bytes);
  if (e != cudaSuccess) return e;
  const uint32_t grid = (P.n - 1u) / P.warps_per_block + 1u, threads = 32u * P.warps_per_block;
  count<<<grid, threads, smem_bytes, stream>>>(P);
  cta_scan<K><<<1, 1024, 0, stream>>>(P.cta, P.total, grid);
  list<<<grid, threads, smem_bytes, stream>>>(P);
  return cudaGetLastError();
}

// ---- tick commits (bf_resident_commit*) -------------------------------------------------------------------------------------
// One warp per run; lane w holds word w of the run's masks and codes (words <= 32).  Both launches read a run the same way: its
// topology's step types, the masks of its current result record (and of its schedule record), and its entries [lo, hi), found by
// a binary search every lane runs alike.  A run with no mask bit, no entry and (kRewrite) no rewrite leaves at once.
struct CommitRun {
  const uint8_t* topo;          // nullptr: dead slot, or a topology wider than the layout (no masks)
  uint32_t TW, VALID;
  uint32_t launched, queued, skip, fail;
  uint32_t T_COND, SYNC_T, T_PAR, T_STOP;
  uint32_t lo, hi, slot;
};

template <bool kRewrite>
DI bool commit_run(const CommitParams& P, uint32_t r, uint32_t lane, CommitRun& c) {
  const uint32_t slot = c.slot = *reinterpret_cast<const uint32_t*>(P.state + (size_t)r * P.state_stride);
  const Slot sl = slot < P.n_slots ? P.slots[slot] : Slot{};
  const TopoHeader* th = reinterpret_cast<const TopoHeader*>(sl.addr);
  c.topo = sl.addr && th->W <= P.words ? reinterpret_cast<const uint8_t*>(sl.addr) : nullptr;
  c.TW = c.topo ? th->W : 0u;
  c.VALID = c.launched = c.queued = c.skip = c.fail = 0u;
  uint32_t t0 = 0u, t1 = 0u, t2 = 0u;
  if (lane < c.TW) {
    c.VALID = bmsk_clamp(0u, th->S - lane * 32u);
    const uint32_t* pl = reinterpret_cast<const uint32_t*>(c.topo + th->off_planes) + lane;
    t0 = pl[PL_T0 * c.TW]; t1 = pl[PL_T1 * c.TW]; t2 = pl[PL_T2 * c.TW];
    const uint8_t* res = P.result + (size_t)r * P.result_stride;
    const uint32_t ready = reinterpret_cast<const uint32_t*>(res + P.off_ready)[lane];
    c.skip = reinterpret_cast<const uint32_t*>(res + P.off_skip)[lane];
    if (P.off_fail != BF_OFF_NONE) c.fail = reinterpret_cast<const uint32_t*>(res + P.off_fail)[lane];
    c.launched = ready;
    if (P.sched_rec) {
      const uint32_t* sr = reinterpret_cast<const uint32_t*>(P.sched_rec + (size_t)r * P.sched_stride + 16) + lane;
      c.launched = sr[0];
      c.queued = sr[P.words] | sr[2u * P.words];
    }
  }
  c.T_COND = t0 & ~t1 & ~t2;
  c.SYNC_T = t0 & (t1 | t2);
  c.T_PAR = ~t0 & t1 & ~t2 & c.VALID;
  c.T_STOP = ~t0 & ~t1 & t2 & c.VALID;
  uint32_t a = 0u, b = P.n_entries;
  while (a < b) { const uint32_t m = (a + b) >> 1; if (P.entries[m].run < r) a = m + 1u; else b = m; }
  c.lo = a; b = P.n_entries;
  while (a < b) { const uint32_t m = (a + b) >> 1; if (P.entries[m].run <= r) a = m + 1u; else b = m; }
  c.hi = a;
  return __any_sync(FULL, (c.launched | c.queued | c.skip | c.fail) != 0u) || c.lo != c.hi || (kRewrite && P.rw_runs[r]);
}

// The entries of a run: lane w collects the HOLD and PHASE bits of its word; err: the run has an ERROR entry.  With check, the
// lowest offending entry's key (entries ascend by step) is returned, else ~0.
DI unsigned long long commit_entries(const CommitParams& P, uint32_t r, uint32_t lane, const CommitRun& c, bool check,
                                     uint32_t& hold, uint32_t& phased, bool& err) {
  hold = phased = 0u; err = false;
  unsigned long long bad = ~0ull;
  for (uint32_t i = c.lo; i < c.hi; ++i) {   // warp-uniform trip count
    const bf_commit_entry e = P.entries[i];
    const uint32_t w = e.step >> 5, bit = 1u << (e.step & 31u);   // step < steps_max: w < words <= 32
    if (lane == w) {
      if (e.kind == BF_COMMIT_HOLD) hold |= bit;
      if (e.kind == BF_COMMIT_PHASE) phased |= bit;
    }
    err = err || e.kind == BF_COMMIT_ERROR;
    if (!check) continue;
    const uint32_t lw = __shfl_sync(FULL, c.launched, w), sw = __shfl_sync(FULL, c.T_STOP, w);
    const uint32_t why = !(lw & bit) ? kCommitNotLaunched : (e.kind == BF_COMMIT_PHASE && !(sw & bit)) ? kCommitNotStop : 0u;
    if (why && bad == ~0ull) bad = (unsigned long long)r << 32 | (unsigned long long)e.step << 8 | why;
  }
  return bad;
}

// Where commit_apply<true> lists a run's new arms: its TIMER items start at items[at] (nullptr: no journal, nothing listed)
struct ArmItems {
  bf_commit_write* items;
  unsigned long long at, cap;
};

// The timer arms of run r (whole warp, with a timing table): each timing of the run's slot whose step is in ARM (lane w holds
// word w: the launched sleep / gate / wait steps) and that no armed slot of the run names is a new arm; an armed slot stays.
// Lane t holds slots t and t + 32 (armed slots lead, ascending by step).  The timings ascend by step and are walked 32 at a time,
// so new arms come in step order: a new arm's rank is the new arms before it plus the armed slots of lower steps (counted over
// the slots, read through shuffles, which also finds a stored slot), a kept slot's is its index plus the new arms of lower
// steps, as arm_timers ranks them.  Check: -> the key of the run's first arming offence (a non-PENDING code without decision
// planes at its step, more than timer_k slots at the lowest new step), else ~0; nothing is written; n_armed: the new arms.
// Apply (after a check that found none): stores the moved and the new slots, lists the new arms in step order at J, and adds
// the arms and their earliest deadline to A.out.
DI unsigned long long commit_arms(const CommitTimings& A, uint32_t r, uint32_t lane, uint32_t slot, uint32_t ARM, bool apply,
                                  uint32_t& n_armed, const ArmItems& J) {
  n_armed = 0;
  if (slot >= A.n_slots || !__any_sync(FULL, ARM != 0u)) return ~0ull;
  const uint32_t lo = A.first[slot], hi = A.first[slot + 1], K = A.timer_k;
  if (lo == hi) return ~0ull;
  unsigned long long* t = A.timers + (size_t)r * K;
  const unsigned long long v0 = lane < K ? t[lane] : kTimerEmpty, v1 = lane + 32u < K ? t[lane + 32u] : kTimerEmpty;
  const uint32_t s0 = timer_step(v0), s1 = timer_step(v1);
  const uint32_t E = __popc(__ballot_sync(FULL, timer_armed(v0))) + __popc(__ballot_sync(FULL, timer_armed(v1)));
  uint32_t n_new = 0, first_new = 0, first_dec = ~0u, nb0 = 0, nb1 = 0, next = BF_TIMER_NONE;
  for (uint32_t j0 = lo; j0 < hi; j0 += 32u) {   // warp-uniform trip count
    const uint32_t j = j0 + lane;
    const bf_step_timing q = j < hi ? A.tim[j] : bf_step_timing{0, 0, 0, 0};
    const uint32_t s = q.step;
    uint32_t below = 0;   // armed slots of lower steps; a run holds few, so each lane compares with every one
    bool stored = false;
    for (uint32_t k = 0; k < E; ++k) {
      const uint32_t sk = __shfl_sync(FULL, k < 32u ? s0 : s1, k & 31u);
      below += sk < s ? 1u : 0u;
      stored = stored || sk == s;
    }
    const uint32_t aw = __shfl_sync(FULL, ARM, (s >> 5) & 31u);   // every lane shuffles, also those past hi
    const bool fresh = j < hi && ((aw >> (s & 31u)) & 1u) && !stored;
    const uint32_t m = __ballot_sync(FULL, fresh);
    if (!m) continue;
    if (n_new == 0) first_new = __shfl_sync(FULL, s, __ffs(m) - 1);
    if (!apply) {
      const uint32_t nd = A.decision ? 0u : __ballot_sync(FULL, fresh && q.code != BF_DEC_PENDING);
      if (nd && first_dec == ~0u) first_dec = __shfl_sync(FULL, s, __ffs(nd) - 1);
    } else {
      if (fresh) {
        const uint32_t dl = (uint32_t)min((unsigned long long)A.now + q.delay, (unsigned long long)BF_TIMER_NONE - 1ull);
        const uint32_t rank = n_new + __popc(m & ((1u << lane) - 1u));
        t[rank + below] = (unsigned long long)dl | (unsigned long long)s << 32 | (unsigned long long)q.code << 48;
        next = min(next, dl);
        if (J.items && J.at + rank < J.cap)
          reinterpret_cast<uint4*>(J.items)[J.at + rank] = make_uint4(r, s | BF_COMMIT_WRITE_TIMER << 16 | (uint32_t)q.code << 24, BF_TIMER_NONE, dl);
      }
      for (uint32_t x = m; x; x &= x - 1u) {   // each new arm moves the kept slots of higher steps up one
        const uint32_t sn = __shfl_sync(FULL, s, __ffs(x) - 1);
        nb0 += timer_armed(v0) && s0 > sn ? 1u : 0u;
        nb1 += timer_armed(v1) && s1 > sn ? 1u : 0u;
      }
    }
    n_new += __popc(m);
  }
  n_armed = n_new;
  if (!apply) {   // a decision offence at the lowest new step wins over the overflow there
    if (first_dec != ~0u && (first_dec == first_new || E + n_new <= K))
      return (unsigned long long)r << 32 | (unsigned long long)first_dec << 8 | kCommitNoDecision;
    return E + n_new > K ? (unsigned long long)r << 32 | (unsigned long long)first_new << 8 | kCommitOverflow : ~0ull;
  }
  if (nb0) t[lane + nb0] = v0;   // the slots read above were loaded before any store (the ballots order them)
  if (nb1) t[lane + 32u + nb1] = v1;
  next = __reduce_min_sync(FULL, next);
  if (lane == 0 && n_new) {
    atomicAdd(A.out, n_new);
    atomicMin(A.out + 1, next);
  }
  return ~0ull;
}

// The writes of run r (no ERROR entry, a slot that fits: c.topo set) on the codes as the pass reads them (code 15 as 0): lane w's
// stored planes p, new codes n and the steps whose code changes (dirty), and the disjoint masks; commit_registered adds the
// registered bits newly set (lanes p and p + 32 look at the launched parallel descs; reg_only counts the steps whose bit alone
// changes).  commit_apply stores them; commit_check<true> counts them, so that both launches agree on every item.  between(LA)
// runs once the masks are known (commit_apply arms there).  With kRewrite the masks write over the base codes rewrite_runs left
// for run r when it flagged it (the codes after a single pass's stages), else over the stored codes; dirty stays the steps whose
// stored code changes.
struct CommitWrites {
  uint32_t p[4], n0, n1, n2, n3, dirty;
  uint32_t SK, FA, LA, QU;
  unsigned long long reg, newly;
  uint32_t reg_only;
};
template <bool kRewrite, typename Between>
DI void commit_writes(const CommitParams& P, uint32_t r, uint32_t lane, const CommitRun& c, const uint8_t* rec, uint32_t hold,
                      CommitWrites& w, Between between) {
  const uint32_t* ph = reinterpret_cast<const uint32_t*>(rec + P.off_phase) + lane;
  for (uint32_t b = 0; b < 4; ++b) w.p[b] = 0u;
  if (lane < c.TW)
    for (uint32_t b = 0; b < 4; ++b) w.p[b] = ph[b * P.words];
  const uint32_t keep = c.VALID & ~(w.p[0] & w.p[1] & w.p[2] & w.p[3]);
  const uint32_t m0 = w.p[0] & keep, m1 = w.p[1] & keep, m2 = w.p[2] & keep, m3 = w.p[3] & keep;
  uint32_t n0 = m0, n1 = m1, n2 = m2, n3 = m3;
  if (kRewrite && P.rw_runs[r] && lane < c.TW) {   // warp-uniform flag
    const uint32_t* b = P.rw_planes + (size_t)r * 4u * P.words + lane;
    n0 = b[0]; n1 = b[P.words]; n2 = b[2u * P.words]; n3 = b[3u * P.words];
  }
  w.SK = c.skip; w.FA = c.fail & ~w.SK; w.LA = c.launched & ~w.SK & ~w.FA & ~hold; w.QU = c.queued & ~w.SK & ~w.FA & ~c.launched;
  between(w.LA);
  pset<BF_PHASE_FAILED>(w.FA, n0, n1, n2, n3);
  launch_effects(w.SK, w.LA, c.T_COND, c.SYNC_T, c.T_PAR, c.T_STOP, n0, n1, n2, n3);
  pset<BF_PHASE_PENDING_QUEUED>(w.QU, n0, n1, n2, n3);
  for (uint32_t i = c.lo; i < c.hi; ++i) {   // the stop steps' phases (a PHASE entry names a launched stop step)
    const bf_commit_entry e = P.entries[i];
    const uint32_t bit = 1u << (e.step & 31u);
    if (e.kind != BF_COMMIT_PHASE || lane != (e.step >> 5u) || !(w.LA & bit)) continue;
    n0 = (e.code & 1u) ? n0 | bit : n0 & ~bit;
    n1 = (e.code & 2u) ? n1 | bit : n1 & ~bit;
    n2 = (e.code & 4u) ? n2 | bit : n2 & ~bit;
    n3 = (e.code & 8u) ? n3 | bit : n3 & ~bit;
  }
  w.n0 = n0; w.n1 = n1; w.n2 = n2; w.n3 = n3;
  w.dirty = (n0 ^ m0) | (n1 ^ m1) | (n2 ^ m2) | (n3 ^ m3);
}
// launched parallel steps register their children (step_executor.go:808-809)
DI void commit_registered(uint32_t lane, const CommitRun& c, const uint8_t* rec, CommitWrites& w) {
  const TopoHeader* th = reinterpret_cast<const TopoHeader*>(c.topo);
  const ParDesc* pd = reinterpret_cast<const ParDesc*>(c.topo + th->off_par);
  w.reg = *reinterpret_cast<const unsigned long long*>(rec + 8);
  const uint32_t n_par = th->P;
  uint32_t set[2];
  w.reg_only = 0u;
  for (uint32_t h = 0; h < 2; ++h) {   // BF_MAX_PARALLEL = 64 descs: lane p and lane p + 32
    const uint32_t q = lane + 32u * h;
    const uint32_t stp = q < n_par ? pd[q].step : 0u;
    const uint32_t lw = __shfl_sync(FULL, w.LA, (stp >> 5) & 31u), dw = __shfl_sync(FULL, w.dirty, (stp >> 5) & 31u);
    const bool in = q < n_par && ((lw >> (stp & 31u)) & 1u);
    set[h] = __ballot_sync(FULL, in);
    if (in && !((w.reg >> q) & 1ull) && !((dw >> (stp & 31u)) & 1u)) ++w.reg_only;   // counted once per step
  }
  w.newly = ((unsigned long long)set[1] << 32 | set[0]) & ~w.reg;
}

// a word's share of each total when the word is the total (one array of CTA totals)
struct WordPart {
  DI uint32_t operator()(uint32_t w, uint32_t) const { return w; }
};
// a run's journal word's share of the items (k = 0) and of the written runs (k = 1)
struct JournalPart {
  DI uint32_t operator()(uint32_t w, uint32_t k) const { return k ? w & 1u : w >> kJournalItemsShift; }
};

// The per-run part of commit_check: lane 0 lowers P.offender to the run's first offence.  -> with kJournal, the run's journal
// word (its items, new arms and whether its record changes; 0 for a run that writes nothing), else 0.
template <bool kJournal, bool kRewrite>
DI uint32_t check_run(const CommitParams& P, uint32_t r, uint32_t lane) {
  CommitRun c;
  if (!commit_run<kRewrite>(P, r, lane, c)) return 0u;
  uint32_t hold, phased;
  bool err;
  unsigned long long bad = commit_entries(P, r, lane, c, true, hold, phased, err);
  const uint32_t miss = err ? 0u : c.launched & c.T_STOP & ~hold & ~phased;
  const uint32_t lanes = __ballot_sync(FULL, miss != 0u);
  if (lanes) {
    const uint32_t w = __ffs(lanes) - 1u;
    const uint32_t step = w * 32u + __ffs(__shfl_sync(FULL, miss, w)) - 1u;
    bad = min(bad, (unsigned long long)r << 32 | (unsigned long long)step << 8 | kCommitNoPhase);
  }
  if (lane == 0 && bad != ~0ull) atomicMin(P.offender, bad);
  if (err) return 0u;
  uint32_t armed = 0;
  if (P.arm.tim) {
    bad = commit_arms(P.arm, r, lane, c.slot, c.launched & ~c.skip & ~c.fail & ~hold & c.SYNC_T, false, armed, ArmItems{});
    if (lane == 0 && bad != ~0ull) atomicMin(P.offender, bad);
  }
  if (!kJournal || !c.topo) return 0u;   // a dead or too-wide slot has no masks: it writes nothing (an entry on it is refused)
  const uint8_t* rec = P.state + (size_t)r * P.state_stride;
  CommitWrites w;
  commit_writes<kRewrite>(P, r, lane, c, rec, hold, w, [](uint32_t) {});
  commit_registered(lane, c, rec, w);
  const uint32_t items = redux_add(__popc(w.dirty)) + __popcll(w.newly) + armed;
  const bool written = __any_sync(FULL, w.dirty != 0u) || w.newly != 0ull;
  return items << kJournalItemsShift | armed << kJournalArmsShift | (written ? 1u : 0u);
}

// Check: every entry names a launched step (a PHASE entry a stop step), and every launched stop step of a run without an ERROR
// entry has a HOLD or PHASE entry; with a timing table, the arming offences too.  Lane 0 lowers P.offender to the run's first
// offence.  Nothing is written but, with kJournal, each run's journal word and each CTA's items and written runs.  The kernels
// commit_check (kRewrite = false) and commit_check_rewrites (both true) are this body.
// commit_check_at: warp position i (its journal word and block total) takes run r when `has`.
template <bool kJournal, bool kRewrite>
DI void commit_check_at(const CommitParams& P, uint32_t i, uint32_t r, bool has, uint32_t block, uint32_t n_blocks) {
  const uint32_t lane = threadIdx.x & 31u;
  if (!kJournal) {
    if (has) check_run<false, kRewrite>(P, r, lane);
    return;
  }
  const uint32_t jw = has ? check_run<true, kRewrite>(P, r, lane) : 0u;
  if (lane == 0 && has) P.run_items[i] = jw;
  store_cta_totals_at<2>(jw, P.cta, JournalPart{}, block, n_blocks);
}
template <bool kJournal, bool kRewrite>
DI void commit_check_body(const CommitParams& P) {
  const uint32_t r = blockIdx.x * 8u + (threadIdx.x >> 5);
  commit_check_at<kJournal, kRewrite>(P, r, r, r < P.n_runs, blockIdx.x, gridDim.x);
}
template <bool kJournal>
__global__ void __launch_bounds__(256) commit_check(const CommitParams P) { commit_check_body<kJournal, false>(P); }
__global__ void __launch_bounds__(256) commit_check_rewrites(const CommitParams P) { commit_check_body<true, true>(P); }

// Apply (after a check that found no offender): the writes of commit_writes, stored only where a code changed; the registered
// bits of launched parallel descs; with a timing table, the arms of the launched sleep / gate / wait steps.  With kJournal each
// run with a journal word lists its items (PHASE by step, REGISTERED by desc, TIMER by step) from the offset of the CTAs before
// and the warps before in its CTA, and its entry in runs when its record changed.  With kRewrite a PHASE item of a step without
// a mask bit (its code comes from the stages) carries BF_COMMIT_WRITE_REWRITE, and those steps are added to *P.rewritten.  The
// kernels commit_apply (kRewrite = false) and commit_apply_rewrites (both true) are this body.
// commit_apply_at: warp position i (its journal word, in block `block` of n_blocks) takes run r.
template <bool kJournal, bool kRewrite>
DI void commit_apply_at(const CommitParams& P, uint32_t i, uint32_t r, uint32_t block, uint32_t n_blocks) {
  const uint32_t lane = threadIdx.x & 31u;
  CommitRun c;
  if (!commit_run<kRewrite>(P, r, lane, c)) return;
  uint32_t hold, phased;
  bool err;
  commit_entries(P, r, lane, c, false, hold, phased, err);
  if (err) return;   // Execute failed: nothing of this reconcile is persisted
  uint8_t* rec = P.state + (size_t)r * P.state_stride;
  uint32_t jw = 0, armed;
  unsigned long long pos = 0;
  if (kJournal && (jw = P.run_items[i]) != 0u) {
    unsigned long long base[2];
    run_offsets_at<2>(P.cta, P.run_items, block * 8u, i, JournalPart{}, base, block, n_blocks);
    pos = base[0];
    if (lane == 0 && (jw & 1u) && base[1] < P.runs_cap) P.runs[base[1]] = r;
  }
  CommitWrites w;
  commit_writes<kRewrite>(P, r, lane, c, rec, hold, w, [&](uint32_t LA) {
    if (!P.arm.tim) return;
    const uint32_t n_arms = (jw >> kJournalArmsShift) & ((1u << (kJournalItemsShift - kJournalArmsShift)) - 1u);
    const ArmItems J{kJournal && jw ? P.items : nullptr, pos + (jw >> kJournalItemsShift) - n_arms, P.items_cap};
    commit_arms(P.arm, r, lane, c.slot, LA & c.SYNC_T, true, armed, J);
  });
  const uint32_t dirty = w.dirty;
  uint32_t* ph = reinterpret_cast<uint32_t*>(rec + P.off_phase) + lane;
  if (dirty) {
    ph[0] = (w.p[0] & ~dirty) | (w.n0 & dirty);
    ph[P.words] = (w.p[1] & ~dirty) | (w.n1 & dirty);
    ph[2u * P.words] = (w.p[2] & ~dirty) | (w.n2 & dirty);
    ph[3u * P.words] = (w.p[3] & ~dirty) | (w.n3 & dirty);
  }
  commit_registered(lane, c, rec, w);
  if (kJournal && jw) {   // PHASE items lane by lane in step order, then REGISTERED items by desc
    const uint32_t staged = kRewrite ? ~(w.SK | w.FA | w.LA | w.QU) : 0u;
    const unsigned long long reg_at = emit_bits(dirty, pos, P.items_cap, [&](uint32_t b, unsigned long long at) {
      const uint32_t was = ((w.p[0] >> b) & 1u) | ((w.p[1] >> b) & 1u) << 1 | ((w.p[2] >> b) & 1u) << 2 | ((w.p[3] >> b) & 1u) << 3;
      const uint32_t now = ((w.n0 >> b) & 1u) | ((w.n1 >> b) & 1u) << 1 | ((w.n2 >> b) & 1u) << 2 | ((w.n3 >> b) & 1u) << 3;
      const uint32_t code = ((staged >> b) & 1u) ? BF_COMMIT_WRITE_REWRITE << 24 : 0u;
      reinterpret_cast<uint4*>(P.items)[at] = make_uint4(r, (lane * 32u + b) | (uint32_t)BF_DELTA_PHASE << 16 | code, was, now);
    });
    for (uint32_t h = 0; h < 2; ++h) {
      const uint32_t q = lane + 32u * h;
      if (!((w.newly >> q) & 1ull)) continue;
      const unsigned long long a = reg_at + __popcll(w.newly & ((1ull << q) - 1ull));
      if (a < P.items_cap) reinterpret_cast<uint4*>(P.items)[a] = make_uint4(r, q | (uint32_t)BF_DELTA_REGISTERED << 16, 0u, 1u);
    }
  }
  const unsigned long long newly = w.newly;
  const uint32_t written = __any_sync(FULL, dirty != 0u) || newly != 0ull;
  const uint32_t n_skip = redux_add(__popc(dirty & w.SK)), n_launch = redux_add(__popc(dirty & w.LA) + w.reg_only);
  const uint32_t n_queue = redux_add(__popc(dirty & w.QU)), n_fail = redux_add(__popc(dirty & w.FA));
  if (lane == 0 && written) {
    if (newly) *reinterpret_cast<unsigned long long*>(rec + 8) = w.reg | newly;
    atomicMax(P.mark + r, P.mark_value);   // max: an upload's "must list" bit stays
    atomicAdd(P.counts, 1u);
    if (n_skip) atomicAdd(P.counts + 1, n_skip);
    if (n_launch) atomicAdd(P.counts + 2, n_launch);
    if (n_queue) atomicAdd(P.counts + 3, n_queue);
    if (n_fail) atomicAdd(P.counts + 4, n_fail);
  }
  if (kRewrite) {
    const uint32_t n_rw = redux_add(__popc(dirty & ~(w.SK | w.FA | w.LA | w.QU)));
    if (lane == 0 && n_rw) atomicAdd(P.rewritten, n_rw);
  }
}
template <bool kJournal, bool kRewrite>
DI void commit_apply_body(const CommitParams& P) {
  const uint32_t r = blockIdx.x * 8u + (threadIdx.x >> 5);
  if (r >= P.n_runs) return;
  commit_apply_at<kJournal, kRewrite>(P, r, r, blockIdx.x, gridDim.x);
}
template <bool kJournal>
__global__ void __launch_bounds__(256) commit_apply(const CommitParams P) { commit_apply_body<kJournal, false>(P); }
__global__ void __launch_bounds__(256) commit_apply_rewrites(const CommitParams P) { commit_apply_body<true, true>(P); }

// Without a journal: the check, or the apply.  With one (P.run_items set): the check and the scan, or the apply; with P.rw_runs
// set (after rewrite_runs) their rewriting builds.
cudaError_t launch_commit(const CommitParams& P, bool apply, cudaStream_t stream) {
  if (P.n_runs == 0) return cudaSuccess;
  const uint32_t grid = (P.n_runs - 1u) / 8u + 1u;
  if (!P.run_items) {
    if (apply) commit_apply<false><<<grid, 256, 0, stream>>>(P);
    else commit_check<false><<<grid, 256, 0, stream>>>(P);
  } else if (apply) {
    if (P.rw_runs) commit_apply_rewrites<<<grid, 256, 0, stream>>>(P);
    else commit_apply<true><<<grid, 256, 0, stream>>>(P);
  } else {
    if (P.rw_runs) commit_check_rewrites<<<grid, 256, 0, stream>>>(P);
    else commit_check<true><<<grid, 256, 0, stream>>>(P);
    return launch_cta_scan(P.cta, P.total, grid, 2, stream);
  }
  return cudaGetLastError();
}

// ---- touched commits (bf_resident_commit_touched) ------------------------------------------------------------------------------
// The list-mode builds of both launches (CommitListParams): each CTA walks blocks b = blockIdx.x, + gridDim.x, ... of 8 list
// positions while 8 b < *n_list; warp w of block b takes position 8 b + w, and runs the full form's per-run body on run list[i]
// with the journal's words and block totals indexed by position.  The list ascends, so items and runs come out ordered by run
// as in the full form.
DI uint32_t list_run(const CommitListParams& L, uint32_t i) { return L.list ? L.list[i] : i; }
template <bool kJournal, bool kRewrite>
__global__ void __launch_bounds__(256) commit_check_list(const CommitListParams L) {
  const uint32_t n = (uint32_t)*L.n_list, n_blocks = (n + 7u) / 8u;
  for (uint32_t b = blockIdx.x; b < n_blocks; b += gridDim.x) {   // CTA-uniform
    const uint32_t i = b * 8u + (threadIdx.x >> 5);
    commit_check_at<kJournal, kRewrite>(L.P, i, i < n ? list_run(L, i) : 0u, i < n, b, n_blocks);
    if (kJournal) __syncthreads();   // the block's warp words are read before the next block stores its own
  }
}
// The apply also keeps the commit-due bits of the runs it takes: a run an entry names stays due (the next commit checks it
// again), every other one is cleared.
template <bool kJournal, bool kRewrite>
__global__ void __launch_bounds__(256) commit_apply_list(const CommitListParams L) {
  const uint32_t n = (uint32_t)*L.n_list, n_blocks = (n + 7u) / 8u, lane = threadIdx.x & 31u;
  for (uint32_t b = blockIdx.x; b < n_blocks; b += gridDim.x) {
    const uint32_t i = b * 8u + (threadIdx.x >> 5);
    if (i >= n) break;
    const uint32_t r = list_run(L, i);
    if (lane == 0) {
      uint32_t a = 0u, e = L.P.n_entries;
      while (a < e) { const uint32_t m = (a + e) >> 1; if (L.P.entries[m].run < r) a = m + 1u; else e = m; }
      const uint32_t bit = 1u << (r & 31u);
      if (a < L.P.n_entries && L.P.entries[a].run == r) atomicOr(L.due + (r >> 5), bit);
      else atomicAnd(L.due + (r >> 5), ~bit);
    }
    commit_apply_at<kJournal, kRewrite>(L.P, i, r, b, n_blocks);
  }
}

// The check (and with a journal its scan), or the apply, of a touched commit over at most max_n list positions, `ctas` CTAs
cudaError_t launch_commit_list(const CommitListParams& L, bool apply, uint32_t max_n, uint32_t ctas, cudaStream_t stream) {
  if (max_n == 0) return cudaSuccess;
  const uint32_t grid = std::min((max_n - 1u) / 8u + 1u, std::max(ctas, 1u));
  if (!L.P.run_items) {
    if (apply) commit_apply_list<false, false><<<grid, 256, 0, stream>>>(L);
    else commit_check_list<false, false><<<grid, 256, 0, stream>>>(L);
  } else if (apply) {
    if (L.P.rw_runs) commit_apply_list<true, true><<<grid, 256, 0, stream>>>(L);
    else commit_apply_list<true, false><<<grid, 256, 0, stream>>>(L);
  } else {
    if (L.P.rw_runs) commit_check_list<true, true><<<grid, 256, 0, stream>>>(L);
    else commit_check_list<true, false><<<grid, 256, 0, stream>>>(L);
    cta_scan_list<2><<<1, 1024, 0, stream>>>(L.P.cta, L.P.total, L.n_list);
  }
  return cudaGetLastError();
}

// The due word w of a touched commit's list: its commit-due bits and the runs entries name, below n_runs
DI uint32_t due_word(const DueListParams& D, uint32_t w) {
  const uint32_t first = w * 32u;
  if (first >= D.n_runs) return 0u;
  uint32_t bits = D.due[w];
  uint32_t a = 0u, e = D.n_entries;
  while (a < e) { const uint32_t m = (a + e) >> 1; if (D.entries[m].run < first) a = m + 1u; else e = m; }
  for (; a < D.n_entries && D.entries[a].run < first + 32u; ++a) bits |= 1u << (D.entries[a].run & 31u);
  const uint32_t left = D.n_runs - first;
  return left < 32u ? bits & ((1u << left) - 1u) : bits;
}
// Count: group g (warp) takes due words 32 g + lane; its runs, and each CTA's total.  List (after cta_scan<1>): the same groups
// again, each writing its runs from its offset, lane by lane and bit by bit (ascending).
template <bool kList>
__global__ void __launch_bounds__(256) due_runs(const DueListParams D) {
  const uint32_t g = blockIdx.x * 8u + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
  const uint32_t w = g * 32u + lane, bits = g < D.n ? due_word(D, w) : 0u;
  if (!kList) {
    const uint32_t k = redux_add((uint32_t)__popc(bits));
    if (lane == 0 && g < D.n) D.group_runs[g] = k;
    store_cta_totals<1>(k, D.cta, WordPart{});
    return;
  }
  if (g >= D.n) return;
  unsigned long long base[1];
  run_offsets<1>(D.cta, D.group_runs, blockIdx.x * 8u, g, WordPart{}, base);
  emit_bits(bits, base[0], D.n_runs, [&](uint32_t b, unsigned long long at) { D.list[at] = w * 32u + b; });
}
cudaError_t launch_due_list(const DueListParams& D, cudaStream_t stream) {
  return launch_listing<1>(due_runs<false>, due_runs<true>, D, 0u, stream);
}

// The touched tick's evaluated runs (list[0, min(*count, bound))) become commit-due; a grid-stride loop of `ctas` CTAs
__global__ void __launch_bounds__(256) due_mark_list(uint32_t* due, const uint32_t* list, const uint32_t* count, uint32_t bound) {
  const uint32_t n = min(*count, bound);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t r = list[i];
    atomicOr(due + (r >> 5), 1u << (r & 31u));
  }
}
cudaError_t launch_due_mark_list(uint32_t* due, const uint32_t* list, const uint32_t* count, uint32_t bound, uint32_t ctas,
                                 cudaStream_t stream) {
  if (bound == 0) return cudaSuccess;
  due_mark_list<<<std::min((bound - 1u) / 256u + 1u, std::max(ctas, 1u)), 256, 0, stream>>>(due, list, count, bound);
  return cudaGetLastError();
}

// The runs whose schedule record bf_resident_schedule changed (listed: run_events[r] != kSchedUnlisted) become commit-due; one
// thread per run, one word per warp
__global__ void __launch_bounds__(256) due_mark_sched(uint32_t* due, const uint32_t* run_events, uint32_t n_runs) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t m = __ballot_sync(FULL, r < n_runs && run_events[r] != kSchedUnlisted);
  if ((threadIdx.x & 31u) == 0 && m) atomicOr(due + (r >> 5), m);
}
cudaError_t launch_due_mark_sched(uint32_t* due, const uint32_t* run_events, uint32_t n_runs, cudaStream_t stream) {
  if (n_runs == 0) return cudaSuccess;
  due_mark_sched<<<(n_runs - 1u) / 256u + 1u, 256, 0, stream>>>(due, run_events, n_runs);
  return cudaGetLastError();
}

// ---- a single pass's stages over one state record (bf_resident_status, bf_resident_resync) ------------------------------------
// One warp per run; lane w holds word w of its codes (words <= 32).  The topology planes of lane word w that stages G, H and I read.
struct PassTopo {
  uint32_t VALID, AF, TS, G1, G2, SYNC_T, T_PAR;
};
DI PassTopo pass_topo(const uint8_t* topo, const TopoHeader& th, uint32_t lane, bool act) {
  uint32_t t0 = 0, t1 = 0, t2 = 0;
  PassTopo T{};
  if (act) {
    const uint32_t Wt = th.W;
    const uint32_t* pl = reinterpret_cast<const uint32_t*>(topo + th.off_planes) + lane;
    t0 = pl[PL_T0 * Wt]; t1 = pl[PL_T1 * Wt]; t2 = pl[PL_T2 * Wt];
    T.AF = pl[PL_AF * Wt]; T.TS = pl[PL_TS * Wt]; T.G1 = pl[PL_G1 * Wt]; T.G2 = pl[PL_G2 * Wt];
    T.VALID = bmsk_clamp(0u, th.S - lane * 32u);
  }
  T.SYNC_T = t0 & (t1 | t2);
  T.T_PAR = ~t0 & t1 & ~t2 & T.VALID;
  return T;
}
// Word `lane` of the 4 phase planes (p) or the 2 planes (p0, p1) of a code at `off` of a record, masked to `valid`; a phase code
// 15 reads as 0.
DI void load_phases(const uint8_t* rec, uint32_t off, uint32_t words, uint32_t lane, uint32_t valid, uint32_t& p0, uint32_t& p1,
                    uint32_t& p2, uint32_t& p3) {
  const uint32_t* ph = reinterpret_cast<const uint32_t*>(rec + off) + lane;
  p0 = ph[0]; p1 = ph[words]; p2 = ph[2u * words]; p3 = ph[3u * words];
  const uint32_t keep = valid & ~(p0 & p1 & p2 & p3);
  p0 &= keep; p1 &= keep; p2 &= keep; p3 &= keep;
}
DI void load_codes2(const uint8_t* rec, uint32_t off, uint32_t words, uint32_t lane, uint32_t valid, uint32_t& c0, uint32_t& c1) {
  const uint32_t* cw = reinterpret_cast<const uint32_t*>(rec + off) + lane;
  c0 = cw[0] & valid; c1 = cw[words] & valid;
}

// Stages H, G and I of a single pass over the codes p (decisions d0, d1) of a run with flags byte rflags, as bf_resident_status
// applies them.  Stage H runs only when a registered parallel step is live: the warp first copies the state record `rec` and the
// topology record into its shared stage at stage_a (P.topo_bytes for the topology record, 256 scratch bytes behind it); with
// `over`, the children_registered bits (sel & 1) and the child area (sel & 2) are taken from that record instead.
template <class Params>
DI RunClass single_pass(const Params& P, uint32_t lane, bool act, const TopoHeader& th, const uint8_t* topo, const PassTopo& T,
                        uint32_t rflags, const uint8_t* rec, const uint8_t* over, uint32_t sel, uint32_t stage_a, uint32_t d0,
                        uint32_t d1, uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3) {
  if (P.off_child != BF_OFF_NONE && th.P != 0 &&
      __any_sync(FULL, (T.T_PAR & (p0 | p1 | p2 | p3) & ~plut<BF_LUT_TERMINAL>(p0, p1, p2, p3)) != 0u)) {
    const uint32_t sr_a = stage_a, tr_a = stage_a + P.state_stride;
    __syncwarp();   // a stage H before this one may still read the stage
    for (uint32_t x = lane; x < P.state_stride / 16u; x += 32u) {
      const uint4 v = reinterpret_cast<const uint4*>(rec)[x];
      sts_v4(sr_a + 16u * x, v.x, v.y, v.z, v.w);
    }
    for (uint32_t x = lane; x < th.rec_bytes / 16u; x += 32u) {
      const uint4 v = reinterpret_cast<const uint4*>(topo)[x];
      sts_v4(tr_a + 16u * x, v.x, v.y, v.z, v.w);
    }
    if (over) {
      __syncwarp();
      if ((sel & 1u) && lane < 2u) sts_u32(sr_a + 8u + 4u * lane, reinterpret_cast<const uint32_t*>(over + 8)[lane]);
      for (uint32_t x = lane; (sel & 2u) && x < (P.state_stride - P.off_child) / 4u; x += 32u)
        sts_u32(sr_a + P.off_child + 4u * x, reinterpret_cast<const uint32_t*>(over + P.off_child)[x]);
    }
    __syncwarp();
    stage_h(P, lane, act, th.W, th.P, T.T_PAR, sr_a, tr_a, th.off_par, tr_a + P.topo_bytes, false, p0, p1, p2, p3);   // the codes, not whether they changed
    __syncwarp();
  }
  if (P.off_decision != BF_OFF_NONE) stage_g(T.SYNC_T, T.TS, d0, d1, p0, p1, p2, p3);
  return stage_bi<true>([](uint32_t v) { return redux_or(v); }, rflags, th.n_main, th.n_comp, th.n_final, T.AF, T.VALID & ~T.G1 & ~T.G2, T.G1, T.G2, p0, p1, p2, p3);
}

// ---- run status (bf_resident_status) ------------------------------------------------------------------------------------------
// The codes of the state record take the stages of a single pass (single_pass).  The counts, the failed set and the allowed
// failures are bit-plane tables over the result.
struct RunStatus {
  bf_status_rec rec;   // every field but first_event (warp-uniform)
  uint32_t EV, FL;     // this lane's word of the listed steps, and of those the ones in the failed set
  uint32_t p0, p1, p2, p3;
};

DI void run_status(const StatusParams& P, uint32_t i, uint32_t lane, uint32_t stage_a, RunStatus& s) {
  const uint32_t r = P.runs ? P.runs[i] : i;
  const uint8_t* rec = P.state + (size_t)r * P.state_stride;
  const uint32_t slot = *reinterpret_cast<const uint32_t*>(rec);
  const uint8_t* topo = slot < P.n_slots ? reinterpret_cast<const uint8_t*>(P.slots[slot].addr) : nullptr;
  s.rec = bf_status_rec{};
  s.rec.run = r;
  s.rec.first_failed = BF_STATUS_NO_STEP;
  s.EV = s.FL = s.p0 = s.p1 = s.p2 = s.p3 = 0u;
  const TopoHeader th = topo ? *reinterpret_cast<const TopoHeader*>(topo) : TopoHeader{};
  if (th.W - 1u >= P.words) {   // dead slot, or wider than the layout
    s.rec.outcome = BF_OUTCOME_DEAD;
    return;
  }
  const bool act = lane < th.W;
  const uint32_t rflags = rec[4];
  const PassTopo T = pass_topo(topo, th, lane, act);
  uint32_t p0 = 0, p1 = 0, p2 = 0, p3 = 0, d0 = 0, d1 = 0;
  if (act) {
    load_phases(rec, P.off_phase, P.words, lane, T.VALID, p0, p1, p2, p3);
    if (P.off_decision != BF_OFF_NONE) load_codes2(rec, P.off_decision, P.words, lane, ~0u, d0, d1);
  }
  const uint32_t AF = T.AF, G1 = T.G1, G2 = T.G2, GM = T.VALID & ~G1 & ~G2;
  const RunClass rc = single_pass(P, lane, act, th, topo, T, rflags, rec, nullptr, 0u, stage_a, d0, d1, p0, p1, p2, p3);

  const uint32_t TERM = plut<BF_LUT_TERMINAL>(p0, p1, p2, p3) & ~plut<BF_LUT_COMPLETED0>(p0, p1, p2, p3);
  const uint32_t FAILED = TERM & ~AF, ALLOWED = TERM & AF;
  const uint32_t ac = redux_add((uint32_t)__popc(plut<0x0104u>(p0, p1, p2, p3)) | (uint32_t)__popc(plut<0x0008u>(p0, p1, p2, p3)) << 16);
  const uint32_t fk = redux_add((uint32_t)__popc(plut<0x0010u>(p0, p1, p2, p3)) | (uint32_t)__popc(plut<0x2000u>(p0, p1, p2, p3)) << 16);
  const uint32_t fb = redux_or(((FAILED & G2) ? 1u : 0u) | ((FAILED & G1) ? 2u : 0u) | ((FAILED & GM) ? 4u : 0u));
  const uint32_t stop = P.runctl ? P.runctl[r].stop : BF_STOP_NONE;
  uint32_t outcome, FL = 0u;
  if (stop != BF_STOP_NONE) outcome = stop == BF_STOP_TIMEOUT ? BF_OUTCOME_TIMED_OUT : stop == BF_STOP_CANCEL ? BF_OUTCOME_CANCELED : BF_OUTCOME_STOPPED;
  else if (rc.group != BF_GROUP_DONE) outcome = BF_OUTCOME_NONE;
  else if (fb & 1u) { outcome = BF_OUTCOME_CLEANUP_FAILED; FL = FAILED & G2; }
  else if (fb & 2u) { outcome = BF_OUTCOME_COMPENSATION_FAILED; FL = FAILED & G1; }
  else if (fb & 4u) { outcome = th.n_comp ? BF_OUTCOME_COMPENSATED : BF_OUTCOME_DEPENDENCY_FAILED; FL = FAILED & GM; }
  else outcome = BF_OUTCOME_SUCCEEDED;
  const uint32_t phase = outcome == BF_OUTCOME_SUCCEEDED ? BF_PHASE_SUCCEEDED
                         : outcome == BF_OUTCOME_COMPENSATED ? BF_PHASE_COMPENSATED
                         : outcome == BF_OUTCOME_TIMED_OUT ? BF_PHASE_TIMEOUT
                         : outcome == BF_OUTCOME_CANCELED ? BF_PHASE_FINISHED
                         : outcome >= BF_OUTCOME_DEPENDENCY_FAILED && outcome <= BF_OUTCOME_CLEANUP_FAILED ? BF_PHASE_FAILED : 0u;
  s.EV = FL | ALLOWED;
  s.FL = FL;
  s.p0 = p0; s.p1 = p1; s.p2 = p2; s.p3 = p3;
  s.rec.n_events = (uint16_t)redux_add((uint32_t)__popc(s.EV));
  s.rec.first_failed = (uint16_t)__reduce_min_sync(FULL, FL ? lane * 32u + (uint32_t)__ffs(FL) - 1u : BF_STATUS_NO_STEP);
  s.rec.summary = (uint16_t)(rc.sum | rc.group);
  s.rec.group = (uint8_t)rc.group;
  s.rec.outcome = (uint8_t)outcome;
  s.rec.story_phase = (uint8_t)phase;
  s.rec.active = (uint16_t)(ac & 0xFFFFu); s.rec.completed = (uint16_t)(ac >> 16);
  s.rec.failed = (uint16_t)(fk & 0xFFFFu); s.rec.skipped = (uint16_t)(fk >> 16);
}

// Count (kList = false): each listed run's events, and each CTA's total.  List (kList = true, after cta_scan): the same runs
// again, each record with the offset of its first event (the CTAs before, then the warps before in its CTA) and its events, lane by
// lane in step order.

template <bool kList>
__global__ void __launch_bounds__(256, 1) status_runs(const StatusParams P) {
  extern __shared__ __align__(16) uint8_t status_stage[];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const uint32_t i = blockIdx.x * P.warps_per_block + warp;
  const uint32_t stage_a = smem_u32(status_stage) + warp * pass_stage_bytes(P.off_child, P.state_stride, P.topo_bytes);
  RunStatus s;
  if (!kList) {
    uint32_t ne = 0;
    if (i < P.n) {
      run_status(P, i, lane, stage_a, s);
      ne = s.rec.n_events;
      if (lane == 0) P.run_events[i] = ne;
    }
    store_cta_totals<1>(ne, P.cta, WordPart{});
    return;
  }
  if (i >= P.n) return;
  run_status(P, i, lane, stage_a, s);
  unsigned long long base[1];
  run_offsets<1>(P.cta, P.run_events, blockIdx.x * P.warps_per_block, i, WordPart{}, base);
  s.rec.first_event = (uint32_t)base[0];
  if (lane == 0) {
    const uint4* v = reinterpret_cast<const uint4*>(&s.rec);
    uint4* o = reinterpret_cast<uint4*>(P.records + i);
    o[0] = v[0]; o[1] = v[1];
  }
  emit_bits(s.EV, base[0], P.events_cap, [&](uint32_t b, unsigned long long at) {
    const uint32_t ph = ((s.p0 >> b) & 1u) | ((s.p1 >> b) & 1u) << 1 | ((s.p2 >> b) & 1u) << 2 | ((s.p3 >> b) & 1u) << 3;
    const uint32_t kind = ((s.FL >> b) & 1u) ? BF_STATUS_EVT_FAILED : BF_STATUS_EVT_ALLOWED;
    P.events[at] = (uint16_t)((lane * 32u + b) | ph << 10 | kind << 14);
  });
}

cudaError_t launch_status(const StatusParams& P, uint32_t smem_bytes, cudaStream_t stream) {
  return launch_listing<1>(status_runs<false>, status_runs<true>, P, smem_bytes, stream);
}

// ---- rewrites of a single pass (bf_resident_commit_rewrites) ------------------------------------------------------------------
// One warp per run of [0, n_runs), the shared stage of status_runs.  Only a run whose pass rewrote a phase (BF_SUM_PHASE_CHANGED in
// its current result record, which the pass that left it derived from the same codes) can have a rewrite; a stopped run, a dead
// slot and a slot wider than the layout have none.  Such a run takes single_pass (stages H, G and I, no stage-D cond FAIL), and is
// flagged with its planes stored when a code (15 read as 0) changed.
DI void rewrite_run(const RewriteParams& P, uint32_t r, uint32_t stage_a) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint8_t* rec = P.state + (size_t)r * P.state_stride;
  const uint32_t summary = *reinterpret_cast<const uint32_t*>(P.result + (size_t)r * P.result_stride);
  const uint32_t slot = *reinterpret_cast<const uint32_t*>(rec);
  const uint8_t* topo = slot < P.n_slots ? reinterpret_cast<const uint8_t*>(P.slots[slot].addr) : nullptr;
  const TopoHeader th = topo ? *reinterpret_cast<const TopoHeader*>(topo) : TopoHeader{};
  const bool stopped = P.runctl && P.runctl[r].stop != BF_STOP_NONE;
  uint32_t changed = 0u;
  if ((summary & BF_SUM_PHASE_CHANGED) && th.W - 1u < P.words && !stopped) {   // warp-uniform
    const bool act = lane < th.W;
    const PassTopo T = pass_topo(topo, th, lane, act);
    uint32_t p0 = 0, p1 = 0, p2 = 0, p3 = 0, d0 = 0, d1 = 0;
    if (act) {
      load_phases(rec, P.off_phase, P.words, lane, T.VALID, p0, p1, p2, p3);
      if (P.off_decision != BF_OFF_NONE) load_codes2(rec, P.off_decision, P.words, lane, ~0u, d0, d1);
    }
    const uint32_t m0 = p0, m1 = p1, m2 = p2, m3 = p3;
    single_pass(P, lane, act, th, topo, T, rec[4], rec, nullptr, 0u, stage_a, d0, d1, p0, p1, p2, p3);
    changed = __any_sync(FULL, ((p0 ^ m0) | (p1 ^ m1) | (p2 ^ m2) | (p3 ^ m3)) != 0u) ? 1u : 0u;
    if (changed && lane < P.words) {
      uint32_t* b = P.rw_planes + (size_t)r * 4u * P.words + lane;
      b[0] = p0; b[P.words] = p1; b[2u * P.words] = p2; b[3u * P.words] = p3;
    }
  }
  if (lane == 0) P.rw_runs[r] = changed;
}
__global__ void __launch_bounds__(256, 1) rewrite_runs(const RewriteParams P) {
  extern __shared__ __align__(16) uint8_t rewrite_stage[];
  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t r = blockIdx.x * P.warps_per_block + warp;
  if (r >= P.n_runs) return;
  rewrite_run(P, r, smem_u32(rewrite_stage) + warp * pass_stage_bytes(P.off_child, P.state_stride, P.topo_bytes));
}
// The list-mode build (bf_resident_commit_touched): the warps walk the list positions below *n_list, `ctas` CTAs of them, and
// take run list[i] (list == nullptr: run i); rw_runs and rw_planes stay indexed by run.
__global__ void __launch_bounds__(256, 1) rewrite_runs_list(const RewriteParams P, const uint32_t* list, const unsigned long long* n_list) {
  extern __shared__ __align__(16) uint8_t rewrite_stage[];
  const uint32_t warp = threadIdx.x >> 5, n = (uint32_t)*n_list;
  const uint32_t stage_a = smem_u32(rewrite_stage) + warp * pass_stage_bytes(P.off_child, P.state_stride, P.topo_bytes);
  for (uint32_t i = blockIdx.x * P.warps_per_block + warp; i < n; i += gridDim.x * P.warps_per_block)   // warp-uniform
    rewrite_run(P, list ? list[i] : i, stage_a);
}

cudaError_t launch_rewrites(const RewriteParams& P, uint32_t smem_bytes, cudaStream_t stream) {
  if (P.n_runs == 0) return cudaSuccess;
  if (const cudaError_t e = allow_smem(rewrite_runs, smem_bytes)) return e;
  const uint32_t grid = (P.n_runs - 1u) / P.warps_per_block + 1u;
  rewrite_runs<<<grid, 32u * P.warps_per_block, smem_bytes, stream>>>(P);
  return cudaGetLastError();
}
cudaError_t launch_rewrites_list(const RewriteParams& P, const uint32_t* list, const unsigned long long* n_list, uint32_t ctas,
                                 uint32_t smem_bytes, cudaStream_t stream) {
  if (P.n_runs == 0) return cudaSuccess;
  if (const cudaError_t e = allow_smem(rewrite_runs_list, smem_bytes)) return e;
  const uint32_t grid = std::min((P.n_runs - 1u) / P.warps_per_block + 1u, std::max(ctas, 1u));
  rewrite_runs_list<<<grid, 32u * P.warps_per_block, smem_bytes, stream>>>(P, list, n_list);
  return cudaGetLastError();
}

// ---- resyncs (bf_resident_resync) -------------------------------------------------------------------------------------------
// One warp per listed run; lane w holds word w of its codes.  The device's record and the caller's record as the repair would leave
// it (the device's codes in the fields not selected) both take single_pass on a live slot; each field is compared by XOR of its
// plane words under the mask of the steps compared (the phases' 15 -> 0 is applied as they are loaded).
constexpr uint32_t kSelPhase = 1u << BF_DELTA_PHASE, kSelCond = 1u << BF_DELTA_COND, kSelDecision = 1u << BF_DELTA_DECISION,
                   kSelChild = 1u << BF_DELTA_CHILD, kSelFlags = 1u << BF_DELTA_RUN_FLAGS, kSelRegistered = 1u << BF_DELTA_REGISTERED;

struct RunDrift {
  uint32_t r, slot_dev, slot_rec;
  const uint8_t *dev, *rec, *topo;
  TopoHeader th;
  bool live, stopped;
  uint32_t PH, CO, DE;                        // this lane's word of the differing steps of each selected field
  uint32_t a0, a1, a2, a3, b0, b1, b2, b3;    // device / record phases (after the stages on a live slot)
  uint32_t c0, c1, k0, k1, d0, d1, e0, e1;    // device / record cond and decision codes
  unsigned long long descs, reg;              // descs whose nibbles and bits are compared; the differing registered bits
  uint32_t flags_dev, flags_rec;
  uint32_t n;                                 // items of the run (warp-uniform)
};

// The nibbles (bit k: nibble 8x + k) of child word x that are compared and differ: every nibble of the layout on a dead slot, else
// those of the descs in `descs`.  vd, vr: the device's and the caller's word, each nibble 15 read as 0.
DI uint32_t child_diff(const ResyncParams& P, const RunDrift& d, uint32_t x, uint32_t& vd, uint32_t& vr) {
  auto canon = [](uint32_t w) {
    const uint32_t f = w & (w >> 1) & (w >> 2) & (w >> 3) & 0x11111111u;
    return w & ~(f * 0xFu);
  };
  vd = canon(reinterpret_cast<const uint32_t*>(d.dev + P.off_child)[x]);
  vr = canon(reinterpret_cast<const uint32_t*>(d.rec + P.off_child)[x]);
  const uint32_t lo = 8u * x, hi = min(lo + 8u, P.child_nibbles);
  uint32_t cm = 0;
  if (!d.live) {
    cm = hi > lo ? (1u << (hi - lo)) - 1u : 0u;
  } else {
    const ParDesc* pd = reinterpret_cast<const ParDesc*>(d.topo + d.th.off_par);
    for (unsigned long long q = d.descs; q; q &= q - 1ull) {
      const ParDesc dq = pd[__ffsll((long long)q) - 1];
      const uint32_t a = max(dq.child_first, lo), b = min(dq.child_first + dq.branches, hi);
      if (a < b) cm |= ((1u << (b - a)) - 1u) << (a - lo);
    }
  }
  const uint32_t x4 = vd ^ vr;
  return squeeze4((x4 | (x4 >> 1) | (x4 >> 2) | (x4 >> 3)) & 0x11111111u) & cm;
}

DI void run_drift(const ResyncParams& P, uint32_t i, uint32_t lane, uint32_t stage_a, RunDrift& d) {
  d.r = P.runs ? P.runs[i] : i;
  d.dev = P.state + (size_t)d.r * P.state_stride;
  d.rec = P.records + (size_t)i * P.state_stride;
  d.slot_dev = *reinterpret_cast<const uint32_t*>(d.dev);
  d.slot_rec = *reinterpret_cast<const uint32_t*>(d.rec);
  d.PH = d.CO = d.DE = 0u;
  d.a0 = d.a1 = d.a2 = d.a3 = d.b0 = d.b1 = d.b2 = d.b3 = 0u;
  d.c0 = d.c1 = d.k0 = d.k1 = d.d0 = d.d1 = d.e0 = d.e1 = 0u;
  d.descs = d.reg = 0ull;
  d.stopped = P.runctl && P.runctl[d.r].stop;
  if (d.slot_dev != d.slot_rec) {   // codes of two topologies are not comparable
    d.n = 1u;
    return;
  }
  const uint32_t sel = P.fields;
  d.topo = d.slot_dev < P.n_slots ? reinterpret_cast<const uint8_t*>(P.slots[d.slot_dev].addr) : nullptr;
  d.th = d.topo ? *reinterpret_cast<const TopoHeader*>(d.topo) : TopoHeader{};
  d.live = d.th.W - 1u < P.words;
  d.flags_dev = d.stopped ? P.runctl[d.r].saved_flags : d.dev[4];
  d.flags_rec = d.rec[4];
  const bool act = lane < (d.live ? (uint32_t)d.th.W : P.words);
  const PassTopo T = d.live ? pass_topo(d.topo, d.th, lane, act) : PassTopo{};
  const uint32_t VAL = d.live ? T.VALID : (act ? ~0u : 0u);
  const uint8_t* rp = (sel & kSelPhase) ? d.rec : d.dev;   // where the caller's side takes each code from
  const uint8_t* rd = (sel & kSelDecision) ? d.rec : d.dev;
  if (act) {
    load_phases(d.dev, P.off_phase, P.words, lane, VAL, d.a0, d.a1, d.a2, d.a3);
    load_phases(rp, P.off_phase, P.words, lane, VAL, d.b0, d.b1, d.b2, d.b3);
    if (P.off_cond != BF_OFF_NONE) {
      load_codes2(d.dev, P.off_cond, P.words, lane, VAL, d.c0, d.c1);
      load_codes2(d.rec, P.off_cond, P.words, lane, VAL, d.k0, d.k1);
    }
    if (P.off_decision != BF_OFF_NONE) {
      load_codes2(d.dev, P.off_decision, P.words, lane, VAL, d.d0, d.d1);
      load_codes2(rd, P.off_decision, P.words, lane, VAL, d.e0, d.e1);
    }
  }
  uint32_t NT = VAL;   // the steps whose input codes are compared
  if (d.live) {
    const uint32_t rflags_rec = d.stopped ? d.dev[4] : (sel & kSelFlags) ? d.flags_rec : d.dev[4];
    single_pass(P, lane, act, d.th, d.topo, T, d.dev[4], d.dev, nullptr, 0u, stage_a, d.d0, d.d1, d.a0, d.a1, d.a2, d.a3);
    single_pass(P, lane, act, d.th, d.topo, T, rflags_rec, d.dev, d.rec,
                ((sel & kSelRegistered) ? 1u : 0u) | ((sel & kSelChild) ? 2u : 0u), stage_a, d.e0, d.e1, d.b0, d.b1, d.b2, d.b3);
    NT &= ~(plut<BF_LUT_TERMINAL>(d.a0, d.a1, d.a2, d.a3) & plut<BF_LUT_TERMINAL>(d.b0, d.b1, d.b2, d.b3));
    const ParDesc* pd = reinterpret_cast<const ParDesc*>(d.topo + d.th.off_par);
    for (uint32_t q0 = 0; q0 < d.th.P; q0 += 32u) {   // desc q <-> lane q - q0
      const uint32_t q = q0 + lane;
      const uint32_t step = q < d.th.P ? pd[q].step : 0u;
      const uint32_t ntw = __shfl_sync(FULL, NT, (step >> 5) & 31u);
      const uint32_t m = __ballot_sync(FULL, q < d.th.P && ((ntw >> (step & 31u)) & 1u));
      d.descs |= (unsigned long long)m << q0;
    }
  } else {
    d.descs = ~0ull;
  }
  if (sel & kSelPhase) d.PH = VAL & ((d.a0 ^ d.b0) | (d.a1 ^ d.b1) | (d.a2 ^ d.b2) | (d.a3 ^ d.b3));
  if (sel & kSelCond) d.CO = NT & ((d.c0 ^ d.k0) | (d.c1 ^ d.k1));
  if (sel & kSelDecision) d.DE = NT & ((d.d0 ^ d.e0) | (d.d1 ^ d.e1));
  if (sel & kSelRegistered)
    d.reg = (*reinterpret_cast<const unsigned long long*>(d.dev + 8) ^ *reinterpret_cast<const unsigned long long*>(d.rec + 8)) & d.descs;
  uint32_t n_child = 0;
  if (sel & kSelChild) {
    const uint32_t cw = (P.child_nibbles + 7u) / 8u;
    for (uint32_t x = lane; x < cw; x += 32u) {
      uint32_t vd, vr;
      n_child += (uint32_t)__popc(child_diff(P, d, x, vd, vr));
    }
  }
  d.n = redux_add((uint32_t)(__popc(d.PH) + __popc(d.CO) + __popc(d.DE)) + n_child) + (uint32_t)__popcll((long long)d.reg) +
        ((sel & kSelFlags) && d.flags_dev != d.flags_rec ? 1u : 0u);
}

// One item per set bit of this lane's `bits` (index lane * 32 + bit; values bit b of the planes a and b), from item position pos
// -> the position after the warp's items.
DI unsigned long long emit_words(const ResyncParams& P, uint32_t lane, uint32_t run, uint32_t field, uint32_t bits,
                                 unsigned long long pos, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1,
                                 uint32_t b2, uint32_t b3) {
  return emit_bits(bits, pos, P.items_cap, [&](uint32_t b, unsigned long long at) {
    const uint32_t dv = ((a0 >> b) & 1u) | ((a1 >> b) & 1u) << 1 | ((a2 >> b) & 1u) << 2 | ((a3 >> b) & 1u) << 3;
    const uint32_t rv = ((b0 >> b) & 1u) | ((b1 >> b) & 1u) << 1 | ((b2 >> b) & 1u) << 2 | ((b3 >> b) & 1u) << 3;
    reinterpret_cast<uint4*>(P.items)[at] = make_uint4(run, (lane * 32u + b) | field << 16, dv, rv);
  });
}

// a listed run's item count's share of the items (k = 0) and of the drifted runs (k = 1)
struct DriftPart {
  DI uint32_t operator()(uint32_t w, uint32_t k) const { return k ? (w ? 1u : 0u) : w; }
};

// Count (kList = false): each listed run's items, and each CTA's items and drifted runs.  List (kList = true, after cta_scan): the
// runs with items again, their items from the offset of the CTAs before and the warps before in the CTA, their drifted entries and,
// unless the call only checks, their repair.
template <bool kList>
__global__ void __launch_bounds__(256, 1) resync_runs(const ResyncParams P) {
  extern __shared__ __align__(16) uint8_t resync_stage[];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const uint32_t i = blockIdx.x * P.warps_per_block + warp;
  const uint32_t stage_a = smem_u32(resync_stage) + warp * pass_stage_bytes(P.off_child, P.state_stride, P.topo_bytes);
  RunDrift d;
  if (!kList) {
    uint32_t ni = 0;
    if (i < P.n) {
      run_drift(P, i, lane, stage_a, d);
      ni = d.n;
      if (lane == 0) P.run_items[i] = ni;
    }
    store_cta_totals<2>(ni, P.cta, DriftPart{});
    return;
  }
  if (i >= P.n || P.run_items[i] == 0u) return;
  run_drift(P, i, lane, stage_a, d);
  unsigned long long base[2];
  run_offsets<2>(P.cta, P.run_items, blockIdx.x * P.warps_per_block, i, DriftPart{}, base);
  unsigned long long pos = base[0];
  if (lane == 0 && base[1] < P.drifted_cap) P.drifted[base[1]] = d.r;
  const uint32_t sel = P.fields;
  const bool slot = d.slot_dev != d.slot_rec;
  if (slot) {
    if (lane == 0 && pos < P.items_cap)
      reinterpret_cast<uint4*>(P.items)[pos] = make_uint4(d.r, (uint32_t)BF_DELTA_TOPO_SLOT << 16, d.slot_dev, d.slot_rec);
  } else {
    pos = emit_words(P, lane, d.r, BF_DELTA_PHASE, d.PH, pos, d.a0, d.a1, d.a2, d.a3, d.b0, d.b1, d.b2, d.b3);
    pos = emit_words(P, lane, d.r, BF_DELTA_COND, d.CO, pos, d.c0, d.c1, 0u, 0u, d.k0, d.k1, 0u, 0u);
    pos = emit_words(P, lane, d.r, BF_DELTA_DECISION, d.DE, pos, d.d0, d.d1, 0u, 0u, d.e0, d.e1, 0u, 0u);
    if (sel & kSelChild) {
      const uint32_t cw = (P.child_nibbles + 7u) / 8u;
      for (uint32_t x0 = 0; x0 < cw; x0 += 32u) {   // warp-uniform: the shuffles below take every lane
        const uint32_t x = x0 + lane;
        uint32_t vd = 0, vr = 0;
        const uint32_t m = x < cw ? child_diff(P, d, x, vd, vr) : 0u;
        pos = emit_bits(m, pos, P.items_cap, [&](uint32_t k, unsigned long long a) {
          reinterpret_cast<uint4*>(P.items)[a] =
              make_uint4(d.r, (8u * x + k) | (uint32_t)BF_DELTA_CHILD << 16, (vd >> (4u * k)) & 0xFu, (vr >> (4u * k)) & 0xFu);
        });
      }
    }
    if (lane == 0) {
      if ((sel & kSelFlags) && d.flags_dev != d.flags_rec) {
        if (pos < P.items_cap)
          reinterpret_cast<uint4*>(P.items)[pos] = make_uint4(d.r, (uint32_t)BF_DELTA_RUN_FLAGS << 16, d.flags_dev, d.flags_rec);
        ++pos;
      }
      const unsigned long long rd = *reinterpret_cast<const unsigned long long*>(d.dev + 8);
      const unsigned long long rr = *reinterpret_cast<const unsigned long long*>(d.rec + 8);
      for (unsigned long long y = d.reg; y && pos < P.items_cap; y &= y - 1ull, ++pos) {
        const uint32_t q = (uint32_t)__ffsll((long long)y) - 1u;
        reinterpret_cast<uint4*>(P.items)[pos] =
            make_uint4(d.r, q | (uint32_t)BF_DELTA_REGISTERED << 16, (uint32_t)(rd >> q) & 1u, (uint32_t)(rr >> q) & 1u);
      }
    }
  }
  if (P.check) return;
  __syncwarp();   // every read of the device's record above is done
  uint8_t* dev = P.state + (size_t)d.r * P.state_stride;
  if (slot) {   // the caller's whole record; a stopped run keeps its stop, the caller's flags byte becomes its saved byte
    for (uint32_t x = lane; x < P.state_stride / 16u; x += 32u) {
      uint4 v = reinterpret_cast<const uint4*>(d.rec)[x];
      if (x == 0 && d.stopped) {
        P.runctl[d.r].saved_flags = (uint8_t)v.y;
        v.y = (v.y & ~0xFFu) | kStoppedFlags;
      }
      reinterpret_cast<uint4*>(dev)[x] = v;
    }
    if (lane == 0) {
      atomicMax(P.mark + d.r, P.mark_must_list);
      drop_baseline(P.areas, d.r);
    }
    return;
  }
  uint32_t* dw = reinterpret_cast<uint32_t*>(dev);
  const uint32_t* rw = reinterpret_cast<const uint32_t*>(d.rec);
  if (lane < P.words) {
    if (sel & kSelPhase)
      for (uint32_t b = 0; b < 4u; ++b) dw[P.off_phase / 4u + b * P.words + lane] = rw[P.off_phase / 4u + b * P.words + lane];
    if (sel & kSelCond)
      for (uint32_t b = 0; b < 2u; ++b) dw[P.off_cond / 4u + b * P.words + lane] = rw[P.off_cond / 4u + b * P.words + lane];
    if (sel & kSelDecision)
      for (uint32_t b = 0; b < 2u; ++b) dw[P.off_decision / 4u + b * P.words + lane] = rw[P.off_decision / 4u + b * P.words + lane];
  }
  if (sel & kSelChild)
    for (uint32_t x = lane; x < (P.child_nibbles + 7u) / 8u; x += 32u) dw[P.off_child / 4u + x] = rw[P.off_child / 4u + x];
  if (lane == 0) {
    if (sel & kSelRegistered) { dw[2] = rw[2]; dw[3] = rw[3]; }
    if (sel & kSelFlags) {
      if (d.stopped) P.runctl[d.r].saved_flags = d.rec[4];
      else dev[4] = d.rec[4];
    }
    atomicMax(P.mark + d.r, P.mark_touched);   // max: an upload's "must list" bit stays
  }
}

cudaError_t launch_resync(const ResyncParams& P, uint32_t smem_bytes, cudaStream_t stream) {
  return launch_listing<2>(resync_runs<false>, resync_runs<true>, P, smem_bytes, stream);
}

// ---- side-area resyncs (bf_resident_resync_areas) ---------------------------------------------------------------------------
// One warp per listed run; lane t holds slots t and t + 32 of both sides (armed slots lead, ascending by step), as commit_arms holds
// them.  One warp-uniform walk over the longer armed list matches each slot with the other side's slot of its step by shuffles.  The
// item flags of each slot kind are then ballots, and an item's rank among its field's items is the ballot below it plus, for a TIMER
// item, the other side's TIMER items of lower steps (a walk over those items alone: a run without timer drift walks nothing).  A
// slot step's stored phase and decision are read straight from the device's state record.  Lanes 0-4 take the limiter inputs,
// lanes 0-2 the story deadline, drain deadline and stop.
struct AreaDrift {
  uint32_t r;
  bf_run_ctl dc, rc;                   // the device's and the caller's run control (the device's where RUNCTL is not selected)
  bool stopped;                        // stopped on the device or by the caller's run control: no timers compared or written
  unsigned long long dv[2], cv[2];     // this lane's device / caller slots t, t + 32
  unsigned long long dev_of_c[2];      // the device's slot at the step of cv[j], or kTimerEmpty
  unsigned long long TD, TC, CC, KEEP; // ballots over slot indices: device-only TIMER items, caller-side TIMER items, TIMER_CODE
                                       // items, caller slots the repair keeps (not taken as fired)
  uint32_t SM, RM;                     // differing limiter inputs (bit f), differing story deadline / drain deadline / stop (bits 0-2)
  uint32_t nT, nC, n;                  // TIMER items, TIMER_CODE items, all items (warp-uniform)
};

DI unsigned long long ballot64(bool lo, bool hi) {
  return (unsigned long long)__ballot_sync(FULL, lo) | (unsigned long long)__ballot_sync(FULL, hi) << 32;
}
DI unsigned long long below64(unsigned long long m, uint32_t k) { return m & ((1ull << k) - 1ull); }

DI void area_drift(const ResyncAreasParams& P, uint32_t i, uint32_t lane, AreaDrift& d) {
  d.r = P.runs ? P.runs[i] : i;
  d.dc = P.areas.runctl ? P.areas.runctl[d.r] : kRunCtlDefault;
  d.rc = (P.sel & BF_RESYNC_AREA_RUNCTL) ? P.runctl[i] : d.dc;
  d.stopped = d.dc.stop || d.rc.stop;
  const uint8_t* rec = P.state + (size_t)d.r * P.state_stride;
  const uint32_t K = P.areas.timer_k;
  const bool timers = (P.sel & BF_RESYNC_AREA_TIMERS) && !d.stopped;
  bool tc[2] = {false, false}, cc[2] = {false, false}, keep[2] = {false, false}, td[2] = {false, false};
  for (uint32_t j = 0; j < 2; ++j) {
    const uint32_t k = lane + 32u * j;
    d.dv[j] = timers && k < K ? P.areas.timers[(size_t)d.r * K + k] : kTimerEmpty;
    d.cv[j] = timers && k < K ? P.timers[(size_t)i * K + k] : kTimerEmpty;
    d.dev_of_c[j] = kTimerEmpty;
  }
  if (timers) {
    const uint32_t Ed = (uint32_t)__popcll((long long)ballot64(timer_armed(d.dv[0]), timer_armed(d.dv[1])));
    const uint32_t Ec = (uint32_t)__popcll((long long)ballot64(timer_armed(d.cv[0]), timer_armed(d.cv[1])));
    bool rec_at[2] = {false, false};   // the caller has a slot at the step of dv[j]
    for (uint32_t k = 0; k < max(Ed, Ec); ++k) {   // warp-uniform trip count
      const unsigned long long a = __shfl_sync(FULL, k < 32u ? d.dv[0] : d.dv[1], k & 31u);
      const unsigned long long b = __shfl_sync(FULL, k < 32u ? d.cv[0] : d.cv[1], k & 31u);
      for (uint32_t j = 0; j < 2; ++j) {
        if (timer_armed(a) && timer_armed(d.cv[j]) && timer_step(a) == timer_step(d.cv[j])) d.dev_of_c[j] = a;
        if (timer_armed(b) && timer_armed(d.dv[j]) && timer_step(b) == timer_step(d.dv[j])) rec_at[j] = true;
      }
    }
    for (uint32_t j = 0; j < 2; ++j) {
      const unsigned long long c = d.cv[j], v = d.dv[j], m = d.dev_of_c[j];
      if (timer_armed(c)) {
        const uint32_t s = timer_step(c);
        const bool live = !((BF_LUT_TERMINAL >> get_planes(rec, P.off_phase, P.words, 4, s)) & 1u);
        const bool matched = timer_armed(m);
        const uint32_t dec = P.off_decision != BF_OFF_NONE ? get_planes(rec, P.off_decision, P.words, 2, s) : (uint32_t)BF_DEC_PENDING;
        const bool fired = !matched && P.fired_now != BF_TIMER_NONE && timer_deadline(c) <= P.fired_now &&
                           (timer_code(c) == BF_DEC_PENDING || dec != BF_DEC_PENDING);
        tc[j] = live && (matched ? timer_deadline(m) != timer_deadline(c) : !fired);
        cc[j] = live && matched && timer_code(m) != timer_code(c);
        keep[j] = !fired;
      }
      if (timer_armed(v) && !rec_at[j])
        td[j] = !((BF_LUT_TERMINAL >> get_planes(rec, P.off_phase, P.words, 4, timer_step(v))) & 1u);
    }
  }
  d.TD = ballot64(td[0], td[1]);
  d.TC = ballot64(tc[0], tc[1]);
  d.CC = ballot64(cc[0], cc[1]);
  d.KEEP = ballot64(keep[0], keep[1]);
  bool sm = false, rm = false;
  if ((P.sel & BF_RESYNC_AREA_SCHED) && lane < 5u)
    sm = reinterpret_cast<const uint32_t*>(P.areas.sched_in + d.r)[lane] != reinterpret_cast<const uint32_t*>(P.sched + i)[1u + lane];
  if ((P.sel & BF_RESYNC_AREA_RUNCTL) && lane < 3u) {
    const uint32_t dd = d.dc.drain_deadline, rd = d.rc.drain_deadline;
    rm = lane == 0u ? d.dc.story_deadline != d.rc.story_deadline
       : lane == 1u ? dd != rd && !(dd == BF_TIMER_NONE && deadline_due(rd, P.fired_now) && P.fired_now != BF_TIMER_NONE)
                    : d.dc.stop != d.rc.stop;
  }
  d.SM = __ballot_sync(FULL, sm);
  d.RM = __ballot_sync(FULL, rm);
  d.nT = (uint32_t)(__popcll((long long)d.TD) + __popcll((long long)d.TC));
  d.nC = (uint32_t)__popcll((long long)d.CC);
  d.n = d.nT + d.nC + (uint32_t)(__popc(d.SM) + __popc(d.RM));
}

DI void put_drift(const ResyncAreasParams& P, unsigned long long at, uint32_t run, uint32_t index, uint32_t field, uint32_t dv, uint32_t rv) {
  if (at < P.items_cap) reinterpret_cast<uint4*>(P.items)[at] = make_uint4(run, index | field << 16, dv, rv);
}

// Count (kList = false): each listed run's items, and each CTA's items and drifted runs.  List (kList = true, after cta_scan): the
// runs with items again, their items from the offsets of the CTAs and warps before them, their drifted entries and, unless the
// call only checks, their repair.
template <bool kList>
__global__ void __launch_bounds__(256) resync_area_runs(const ResyncAreasParams P) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const uint32_t i = blockIdx.x * P.warps_per_block + warp;
  AreaDrift d;
  if (!kList) {
    if (blockIdx.x == 0 && threadIdx.x < 2) P.total[2 + threadIdx.x] = 0ull;   // the list launch adds into them
    uint32_t ni = 0;
    if (i < P.n) {
      area_drift(P, i, lane, d);
      ni = d.n;
      if (lane == 0) P.run_items[i] = ni;
    }
    store_cta_totals<2>(ni, P.cta, DriftPart{});
    return;
  }
  if (i >= P.n || P.run_items[i] == 0u) return;
  area_drift(P, i, lane, d);
  unsigned long long base[2];
  run_offsets<2>(P.cta, P.run_items, blockIdx.x * P.warps_per_block, i, DriftPart{}, base);
  if (lane == 0 && base[1] < P.drifted_cap) P.drifted[base[1]] = d.r;
  const unsigned long long pos = base[0];
  // TIMER items of lower steps on the other side: a walk over the set bits of the other side's (warp-uniform) item ballot
  uint32_t cross_c[2] = {0u, 0u}, cross_d[2] = {0u, 0u};
  for (unsigned long long m = d.TD; m; m &= m - 1ull) {
    const uint32_t k = (uint32_t)__ffsll((long long)m) - 1u;
    const uint32_t s = timer_step(__shfl_sync(FULL, k < 32u ? d.dv[0] : d.dv[1], k & 31u));
    for (uint32_t j = 0; j < 2; ++j) cross_c[j] += s < timer_step(d.cv[j]) ? 1u : 0u;
  }
  for (unsigned long long m = d.TC; m; m &= m - 1ull) {
    const uint32_t k = (uint32_t)__ffsll((long long)m) - 1u;
    const uint32_t s = timer_step(__shfl_sync(FULL, k < 32u ? d.cv[0] : d.cv[1], k & 31u));
    for (uint32_t j = 0; j < 2; ++j) cross_d[j] += s < timer_step(d.dv[j]) ? 1u : 0u;
  }
  for (uint32_t j = 0; j < 2; ++j) {
    const uint32_t k = lane + 32u * j;
    const unsigned long long c = d.cv[j], v = d.dv[j], m = d.dev_of_c[j];
    if ((d.TC >> k) & 1ull)
      put_drift(P, pos + __popcll((long long)below64(d.TC, k)) + cross_c[j], d.r, timer_step(c), BF_DRIFT_TIMER,
                timer_armed(m) ? timer_deadline(m) : BF_TIMER_NONE, timer_deadline(c));
    if ((d.TD >> k) & 1ull)
      put_drift(P, pos + __popcll((long long)below64(d.TD, k)) + cross_d[j], d.r, timer_step(v), BF_DRIFT_TIMER, timer_deadline(v),
                BF_TIMER_NONE);
    if ((d.CC >> k) & 1ull)
      put_drift(P, pos + d.nT + __popcll((long long)below64(d.CC, k)), d.r, timer_step(c), BF_DRIFT_TIMER_CODE, timer_code(m),
                timer_code(c));
  }
  const unsigned long long at_sched = pos + d.nT + d.nC, at_ctl = at_sched + __popc(d.SM);
  const uint32_t below = (1u << lane) - 1u;
  if ((d.SM >> lane) & 1u)
    put_drift(P, at_sched + __popc(d.SM & below), d.r, 0u, BF_DRIFT_SCHED_STORY_KEY + lane,
              reinterpret_cast<const uint32_t*>(P.areas.sched_in + d.r)[lane], reinterpret_cast<const uint32_t*>(P.sched + i)[1u + lane]);
  if ((d.RM >> lane) & 1u) {
    const uint32_t dv = lane == 0u ? d.dc.story_deadline : lane == 1u ? d.dc.drain_deadline : d.dc.stop;
    const uint32_t rv = lane == 0u ? d.rc.story_deadline : lane == 1u ? d.rc.drain_deadline : d.rc.stop;
    put_drift(P, at_ctl + __popc(d.RM & below), d.r, 0u, BF_DRIFT_STORY_DEADLINE + lane, dv, rv);
  }
  if (P.check) return;
  __syncwarp();   // every read of the device's areas above is done
  bool wrote = false;
  if ((P.sel & BF_RESYNC_AREA_TIMERS) && !d.stopped && d.nT + d.nC) {   // the caller's slots minus those taken as fired
    const uint32_t K = P.areas.timer_k, n_keep = (uint32_t)__popcll((long long)d.KEEP);
    unsigned long long* t = P.areas.timers + (size_t)d.r * K;
    for (uint32_t j = 0; j < 2; ++j) {
      const uint32_t k = lane + 32u * j;
      if (k < K && timer_armed(d.cv[j]) && ((d.KEEP >> k) & 1ull)) t[__popcll((long long)below64(d.KEEP, k))] = d.cv[j];
      if (k < K && k >= n_keep) t[k] = kTimerEmpty;
    }
    wrote = true;
  }
  if (lane != 0) return;
  if ((P.sel & BF_RESYNC_AREA_SCHED) && d.SM) {
    const bf_sched_put q = P.sched[i];
    P.areas.sched_in[d.r] = bf_sched_run{q.story_key, q.queue_key, q.priority, q.queued_since, q.run_phase, {0u, 0u, 0u}};
    wrote = true;
  }
  bf_run_ctl* ctl = P.areas.runctl ? P.areas.runctl + d.r : nullptr;
  if (d.RM & 1u) ctl->story_deadline = d.rc.story_deadline;
  if (d.RM & 2u) ctl->drain_deadline = d.rc.drain_deadline;
  wrote = wrote || (d.RM & 3u);
  const bool stop = (P.sel & BF_RESYNC_AREA_RUNCTL) && d.rc.stop && !d.dc.stop;
  if (stop) stop_run(P.state + (size_t)d.r * P.state_stride, ctl, d.r, d.rc.stop, StopParams{P.areas, P.mark, P.mark_touched});
  if (wrote || stop) atomicAdd(P.total + 2, 1ull);
  if (stop) atomicAdd(P.total + 3, 1ull);
}

cudaError_t launch_resync_areas(const ResyncAreasParams& P, cudaStream_t stream) {
  return launch_listing<2>(resync_area_runs<false>, resync_area_runs<true>, P, 0u, stream);
}

}  // namespace bf
