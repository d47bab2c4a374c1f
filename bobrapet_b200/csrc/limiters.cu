// limiters.cu — the concurrency limiters that consume the ready sets (SURVEY.md rows a9 / f4).
//
// Reference: findAndLaunchReadySteps (internal/controller/runs/dag.go:1709-1728) applies
// enforceStoryConcurrency (:1780-1799) and enforceSchedulingLimits (:1801-1861; enforcePriorityOrdering
// :1910-1946, effectivePriority :1948-1961, storyRunHasDemand :1981-1999) to each run's ready LIST and keeps a
// prefix.  The counts it reads from cluster LISTs are reductions over the batch here (contract in
// include/bobrafrontier.h):
//
//   sched_count  one warp per run: Running StepRuns of the run (engram steps in phase Running + Running children
//                of registered parallel steps) and its demand flag from the bit-sliced state record and the
//                topology's type planes; integer atomics by story key / queue key / global, atomicMax of the
//                effective priority by queue.  Integer sums and maxima are order-free: bit-exact.
//   sched_apply  one warp per run: prefix truncation of the ready mask ("first k set bits" = readySteps[:slots])
//                against the totals; writes launch / queued_story / queued_sched masks + header.
#include <limits.h>

#include "kernel_common.cuh"

namespace bf {


DI int32_t effective_priority(int32_t base, uint32_t elapsed_s, int32_t aging) {  // dag.go:1948-1961
  if (elapsed_s == BF_SCHED_NONE || aging <= 0 || elapsed_s == 0u) return base;
  const uint32_t e = elapsed_s > 0x7FFFFFFFu ? 0x7FFFFFFFu : elapsed_s;  // int32(elapsed.Seconds())
  const int32_t steps = (int32_t)e / aging;
  return steps > 0 ? (int32_t)((uint32_t)base + (uint32_t)steps) : base;   // Go's int32 sum wraps; signed overflow is UB here
}

// queued_elapsed_s of a run whose field holds `v`: the elapsed time itself (now == BF_SCHED_NONE, bf_schedule), or its queue
// origin on the clock of `now` (bf_resident_schedule): BF_SCHED_NONE stays none, an origin at or past `now` is 0 (Go's
// elapsed <= 0), else the whole clock units between them
DI uint32_t queued_elapsed(uint32_t v, uint32_t now) {
  if (now == BF_SCHED_NONE || v == BF_SCHED_NONE) return v;
  return now > v ? now - v : 0u;
}

// totals start from the host's base counts (StepRuns of stories / queues the batch does not hold)
__global__ void sched_init(const SchedParams P) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.n_stories) P.story_running[i] = P.story_base ? P.story_base[i] : 0u;
  if (i < P.n_queues) {
    P.queue_running[i] = P.queue_base ? P.queue_base[i] : 0u;
    P.queue_maxprio[i] = P.queue_maxprio_base ? P.queue_maxprio_base[i] : INT32_MIN;
  }
  if (i == 0) *P.global_running = P.global_base;
}

__global__ void __launch_bounds__(256) sched_count(const SchedParams P) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, G = (gridDim.x * blockDim.x) >> 5;
  uint32_t block_total = 0;  // lane 0 of each warp accumulates the global count
  for (uint32_t r = gw; r < P.n_runs; r += G) {
    const uint8_t* sr = P.state + (size_t)r * P.state_stride;
    const uint32_t sid = __ldg(reinterpret_cast<const uint32_t*>(sr));
    const bf_sched_run sc = P.runs[r];
    uint32_t cnt = 0;
    bool dem = false;
    if (sid < P.n_slots) {
      const Slot e = P.slots[sid];
      if (e.addr != 0) {
        const uint8_t* tr = reinterpret_cast<const uint8_t*>(e.addr);
        const uint4 h0 = __ldg(reinterpret_cast<const uint4*>(tr));
        const uint4 h1 = __ldg(reinterpret_cast<const uint4*>(tr + 16));
        const uint32_t S = h0.x & 0xFFFFu, Wt = h0.x >> 16, nP = h0.y >> 16;
        if (Wt <= P.words && lane < Wt) {
          const uint32_t* pw = reinterpret_cast<const uint32_t*>(sr + P.off_phase) + lane;
          uint32_t p0 = __ldg(pw), p1 = __ldg(pw + P.words), p2 = __ldg(pw + 2 * P.words), p3 = __ldg(pw + 3 * P.words);
          const uint32_t rem = S - lane * 32;
          const uint32_t valid = rem >= 32 ? 0xFFFFFFFFu : ((1u << rem) - 1u);
          const uint32_t* sp = reinterpret_cast<const uint32_t*>(tr + h1.y) + lane;
          const uint32_t t0 = __ldg(sp + PL_T0 * Wt), t1 = __ldg(sp + PL_T1 * Wt), t2 = __ldg(sp + PL_T2 * Wt);
          const uint32_t running = ~p0 & p1 & ~p2 & ~p3 & valid;   // BF_PHASE_RUNNING (2)
          const uint32_t queued = ~p0 & p1 & p2 & p3 & valid;      // 14: Pending with a "Queued due to ..." message
          cnt = (uint32_t)__popc(running & ~t0 & ~t1 & ~t2);       // engram steps own a StepRun
          dem = (running | queued) != 0;
        }
        if (P.off_child != BF_OFF_NONE && nP != 0 && Wt <= P.words) {  // children of registered parallel steps
          const uint64_t registered = *reinterpret_cast<const uint64_t*>(sr + 8);
          const ParDesc* pd = reinterpret_cast<const ParDesc*>(tr + h1.z);
          const uint8_t* child = sr + P.off_child;
          for (uint32_t q = 0; q < nP; ++q) {
            if (!((registered >> q) & 1ull)) continue;
            const ParDesc d = pd[q];
            if ((uint64_t)d.child_first + d.branches > P.child_nibbles) continue;  // child area shorter than the topology's: nothing to read
            for (uint32_t b = lane; b < d.branches; b += 32) cnt += get_nibble(child, d.child_first + b) == BF_PHASE_RUNNING;
          }
        }
      }
    }
    cnt = redux_add(cnt);
    dem = __any_sync(FULL, dem);
    if (lane == 0) {
      if (cnt) {
        if (sc.story_key < P.n_stories) atomicAdd(&P.story_running[sc.story_key], cnt);
        if (sc.queue_key < P.n_queues) atomicAdd(&P.queue_running[sc.queue_key], cnt);
        block_total += cnt;
      }
      const uint32_t ph = sc.run_phase & 0xFu;
      const bool terminal = (BF_LUT_TERMINAL >> ph) & 1u;
      const bool demand = ph == BF_PHASE_RUNNING || ph == BF_PHASE_PENDING || dem;   // dag.go:1985-1998
      if (!terminal && demand && sc.queue_key < P.n_queues)
        atomicMax(&P.queue_maxprio[sc.queue_key],
                  effective_priority(sc.priority, queued_elapsed(sc.queued_elapsed_s, P.now), P.queue_aging[sc.queue_key]));
    }
  }
  if (lane == 0 && block_total) atomicAdd(P.global_running, block_total);
}

// first `keep` set bits of the warp-wide mask (word `lane` in each lane), list order = LSB first
DI uint32_t keep_prefix(uint32_t word, uint32_t lane, uint32_t keep) {
  const uint32_t c = (uint32_t)__popc(word);
  uint32_t incl = c;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t v = __shfl_up_sync(FULL, incl, d);
    if ((int)lane >= d) incl += v;
  }
  const uint32_t excl = incl - c;
  if (excl >= keep) return 0u;
  if (incl <= keep) return word;
  const uint32_t pos = __fns(word, 0u, (int)(keep - excl) + 1);  // position of the first bit to drop
  return word & ((1u << pos) - 1u);
}

// One run's limits against the totals (whole warp; word `lane` of each mask in lane `lane`): the launch, queued_story and
// queued_sched masks and the header words n_launch, n_queued_story, n_queued_sched, reason (equal in every lane)
struct RunSchedule {
  uint32_t launch, q_story, q_sched;
  uint4 head;
};

DI RunSchedule limit_run(const SchedParams& P, uint32_t r, uint32_t lane, uint32_t global_running) {
  const bf_sched_run sc = P.runs[r];
  const uint32_t elapsed = queued_elapsed(sc.queued_elapsed_s, P.now);
  uint32_t cur = lane < P.words ? __ldg(reinterpret_cast<const uint32_t*>(P.result + (size_t)r * P.result_stride + P.off_ready) + lane) : 0u;
  uint32_t cnt = redux_add((uint32_t)__popc(cur));
  uint32_t q_story = 0, q_sched = 0, reason = BF_QUEUED_NONE;
  const bool ks = sc.story_key < P.n_stories, kq = sc.queue_key < P.n_queues;
  // enforceStoryConcurrency, dag.go:1780-1799
  const int32_t lim = ks ? P.story_limit[sc.story_key] : 0;
  if (cnt != 0 && lim > 0) {
    const uint32_t running = P.story_running[sc.story_key];
    const uint32_t slots = (uint32_t)lim > running ? (uint32_t)lim - running : 0u;
    if (slots < cnt) {
      const uint32_t kept = keep_prefix(cur, lane, slots);
      q_story = cur & ~kept;
      cur = kept;
      cnt = slots;
    }
  }
  // enforceSchedulingLimits, dag.go:1801-1861
  if (cnt != 0) {
    const int32_t mine = effective_priority(sc.priority, elapsed, kq ? P.queue_aging[sc.queue_key] : 0);
    if (kq && P.queue_maxprio[sc.queue_key] > mine) {  // some other run with demand outranks this one (:1928-1942)
      q_sched = cur;
      cur = 0;
      reason = BF_QUEUED_PRIORITY;
    } else {
      const int32_t gl = P.global_limit, ql = kq ? P.queue_limit[sc.queue_key] : 0;
      uint32_t gslots = cnt, qslots = cnt;
      if (gl > 0) gslots = (uint32_t)gl > global_running ? (uint32_t)gl - global_running : 0u;
      if (ql > 0) {
        const uint32_t rq = P.queue_running[sc.queue_key];
        qslots = (uint32_t)ql > rq ? (uint32_t)ql - rq : 0u;
      }
      const uint32_t slots = min(cnt, min(gslots, qslots));
      if (slots < cnt) {
        const uint32_t kept = keep_prefix(cur, lane, slots);
        q_sched = cur & ~kept;
        cur = kept;
        reason = (gl > 0 && (ql <= 0 || gslots <= qslots)) ? BF_QUEUED_GLOBAL : (ql > 0 ? BF_QUEUED_QUEUE : BF_QUEUED_OTHER);
      }
    }
  }
  const uint32_t n_launch = redux_add((uint32_t)__popc(cur)), n_qs = redux_add((uint32_t)__popc(q_story)),
                 n_qd = redux_add((uint32_t)__popc(q_sched));
  return {cur, q_story, q_sched, make_uint4(n_launch, n_qs, n_qd, reason)};
}

__global__ void __launch_bounds__(256) sched_apply(const SchedParams P) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, G = (gridDim.x * blockDim.x) >> 5;
  const uint32_t global_running = *P.global_running;
  for (uint32_t r = gw; r < P.n_runs; r += G) {
    const RunSchedule o = limit_run(P, r, lane, global_running);
    uint8_t* rec = P.records + (size_t)r * P.stride;
    if (lane == 0) *reinterpret_cast<uint4*>(rec) = o.head;
    if (lane < P.words) {
      uint32_t* m = reinterpret_cast<uint32_t*>(rec + 16);
      m[lane] = o.launch;
      m[P.words + lane] = o.q_story;
      m[2 * P.words + lane] = o.q_sched;
    }
    const uint32_t tail = 16u + 12u * P.words;
    for (uint32_t x = tail / 4 + lane; x < P.stride / 4; x += 32) reinterpret_cast<uint32_t*>(rec)[x] = 0u;
  }
}

// phases (kSched*, ctx.h): the totals' start (sched_init), the counting into them (sched_count) and the truncation against them
// (sched_apply).  bf_schedule and bf_schedule_device take all three; a sharded batch all-reduces the totals between counting and
// truncation (bf_group_schedule: sums of the running counts, maximum of the priorities); bf_resident_schedule starts the totals
// once and counts each of its batches into them.
cudaError_t launch_schedule(const SchedParams& P, uint32_t sm_count, cudaStream_t stream, uint32_t phases) {
  const uint32_t wpb = 8;
  uint32_t grid = (P.n_runs + wpb - 1) / wpb;
  if (grid == 0) grid = 1;
  if (grid > sm_count * 8) grid = sm_count * 8;
  const uint32_t n_tab = P.n_stories > P.n_queues ? P.n_stories : P.n_queues;
  if (phases & kSchedInit) sched_init<<<(n_tab + 255) / 256 + 1, 256, 0, stream>>>(P);
  if (phases & kSchedCount) sched_count<<<grid, wpb * 32, 0, stream>>>(P);
  if (phases & kSchedApply) sched_apply<<<grid, wpb * 32, 0, stream>>>(P);
  return cudaGetLastError();
}

// ---- bf_resident_schedule -------------------------------------------------------------------------------------------------
// Limit and compare: warp w of CTA b takes runs 256 b + 32 w + j, j = 0..31, one after the other.  Each run's new record goes
// over its stored one in the batch's schedule-record area; the run is listed when there was no baseline (at or above base_runs,
// or kSchedNoBase in the stored reason) or some header or mask word differs.  Every lane reads the words it then writes, so the
// comparison needs no staging.  run_events[r] and the CTA's listed runs and events feed cta_scan and sched_list_runs.
// A warp's word for the CTA's totals is its events << 8 | its listed runs (at most 32 runs of 3 * 1024 events).
struct SchedPart {
  DI uint32_t operator()(uint32_t w, uint32_t k) const { return k ? w >> 8 : w & 0xFFu; }
};
__global__ void __launch_bounds__(256) sched_limit_runs(const ResSchedParams R) {
  const SchedParams& P = R.S;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t global_running = *P.global_running;
  uint32_t listed = 0, events = 0;
  for (uint32_t j = 0; j < 32u; ++j) {
    const uint32_t r = blockIdx.x * 256u + warp * 32u + j;
    if (r >= P.n_runs) break;
    const RunSchedule o = limit_run(P, r, lane, global_running);
    uint8_t* rec = P.records + (size_t)r * P.stride;
    uint32_t* m = reinterpret_cast<uint32_t*>(rec + 16);
    bool differs = false;
    if (lane == 0) {
      const uint4 h = *reinterpret_cast<const uint4*>(rec);
      differs = r >= R.base_runs || h.w == kSchedNoBase || h.x != o.head.x || h.y != o.head.y || h.z != o.head.z || h.w != o.head.w;
      *reinterpret_cast<uint4*>(rec) = o.head;
    }
    if (lane < P.words) {
      differs |= m[lane] != o.launch || m[P.words + lane] != o.q_story || m[2 * P.words + lane] != o.q_sched;
      m[lane] = o.launch;
      m[P.words + lane] = o.q_story;
      m[2 * P.words + lane] = o.q_sched;
    }
    const uint32_t tail = 16u + 12u * P.words;
    for (uint32_t x = tail / 4 + lane; x < P.stride / 4; x += 32) reinterpret_cast<uint32_t*>(rec)[x] = 0u;
    const bool list = __any_sync(FULL, differs);
    const uint32_t ev = o.head.x + o.head.y + o.head.z;
    if (lane == 0) {
      R.run_events[r] = list ? ev : kSchedUnlisted;
      if (list) { ++listed; events += ev; }
    }
  }
  store_cta_totals<2>(events << 8 | listed, R.cta, SchedPart{});
}

// List: the same partition.  Each CTA reads the listed runs and events of the CTAs before it (cta_scan), scans its own 256 runs,
// and each warp writes its listed runs in order: lane 0 the index and the header, the lanes of the mask words their steps'
// events (ascending: word by lane, bit by bit).
__global__ void __launch_bounds__(256) sched_list_runs(const ResSchedParams R) {
  __shared__ uint32_t s_l[8];
  __shared__ unsigned long long s_e[8];
  const SchedParams& P = R.S;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  // this thread's run, and the inclusive scans of listed runs and events over the warp
  const uint32_t r = blockIdx.x * 256u + threadIdx.x;
  const uint32_t v = r < P.n_runs ? R.run_events[r] : kSchedUnlisted;
  const uint32_t mine_l = v != kSchedUnlisted ? 1u : 0u;
  const unsigned long long mine_e = v != kSchedUnlisted ? v : 0u;
  uint32_t il = mine_l;
  unsigned long long ie = mine_e;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t a = __shfl_up_sync(FULL, il, d);
    const unsigned long long b = __shfl_up_sync(FULL, ie, d);
    if ((int)lane >= d) { il += a; ie += b; }
  }
  if (lane == 31) { s_l[warp] = il; s_e[warp] = ie; }
  __syncthreads();
  unsigned long long wl = R.cta[blockIdx.x], we = R.cta[gridDim.x + blockIdx.x];
  for (uint32_t w = 0; w < warp; ++w) { wl += s_l[w]; we += s_e[w]; }
  const unsigned long long pos_mine = wl + il - mine_l, off_mine = we + ie - mine_e;
  for (uint32_t j = 0; j < 32u; ++j) {
    const bool listed = __shfl_sync(FULL, mine_l, j) != 0u;
    if (!listed) continue;
    const uint32_t rj = blockIdx.x * 256u + warp * 32u + j;
    const unsigned long long pos = __shfl_sync(FULL, pos_mine, j);
    const unsigned long long off = __shfl_sync(FULL, off_mine, j);
    const uint8_t* rec = P.records + (size_t)rj * P.stride;
    if (lane == 0 && pos < R.runs_cap) {
      R.runs[pos] = rj;
      R.heads[pos] = *reinterpret_cast<const bf_sched_header*>(rec);
    }
    const uint32_t* m = reinterpret_cast<const uint32_t*>(rec + 16);
    const uint32_t launch = lane < P.words ? m[lane] : 0u, qs = lane < P.words ? m[P.words + lane] : 0u,
                   qd = lane < P.words ? m[2 * P.words + lane] : 0u;
    emit_bits(launch | qs | qd, off, R.events_cap, [&](uint32_t b, unsigned long long e) {
      const uint32_t kind = (launch >> b) & 1u ? BF_SEVT_LAUNCH : ((qs >> b) & 1u ? BF_SEVT_QUEUED_STORY : BF_SEVT_QUEUED_SCHED);
      R.events[e] = (uint16_t)((lane * 32u + b) | kind << 10);
    });
  }
}

cudaError_t launch_resident_schedule(const ResSchedParams& R, cudaStream_t stream) {
  if (R.S.n_runs == 0) return cudaSuccess;
  const uint32_t grid = (R.S.n_runs - 1u) / 256u + 1u;
  sched_limit_runs<<<grid, 256, 0, stream>>>(R);
  if (const cudaError_t e = launch_cta_scan(R.cta, R.totals, grid, 2, stream)) return e;
  sched_list_runs<<<grid, 256, 0, stream>>>(R);
  return cudaGetLastError();
}

// bf_resident_sched_put: one thread per request (the host checked that no two name the same run)
__global__ void __launch_bounds__(256) sched_put(const SchedPutParams P) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  const bf_sched_put q = P.req[i];
  P.area[q.run] = bf_sched_run{q.story_key, q.queue_key, q.priority, q.queued_since, q.run_phase, {0u, 0u, 0u}};
}

cudaError_t launch_sched_put(const SchedPutParams& P, cudaStream_t stream) {
  if (P.n == 0) return cudaSuccess;
  sched_put<<<(P.n - 1u) / 256u + 1u, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

}  // namespace bf
