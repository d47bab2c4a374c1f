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
        atomicMax(&P.queue_maxprio[sc.queue_key], effective_priority(sc.priority, sc.queued_elapsed_s, P.queue_aging[sc.queue_key]));
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

__global__ void __launch_bounds__(256) sched_apply(const SchedParams P) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, G = (gridDim.x * blockDim.x) >> 5;
  const uint32_t global_running = *P.global_running;
  for (uint32_t r = gw; r < P.n_runs; r += G) {
    const bf_sched_run sc = P.runs[r];
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
      const int32_t mine = effective_priority(sc.priority, sc.queued_elapsed_s, kq ? P.queue_aging[sc.queue_key] : 0);
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
    uint8_t* rec = P.records + (size_t)r * P.stride;
    if (lane == 0) *reinterpret_cast<uint4*>(rec) = make_uint4(n_launch, n_qs, n_qd, reason);
    if (lane < P.words) {
      uint32_t* m = reinterpret_cast<uint32_t*>(rec + 16);
      m[lane] = cur;
      m[P.words + lane] = q_story;
      m[2 * P.words + lane] = q_sched;
    }
    const uint32_t tail = 16u + 12u * P.words;
    for (uint32_t x = tail / 4 + lane; x < P.stride / 4; x += 32) reinterpret_cast<uint32_t*>(rec)[x] = 0u;
  }
}

// phases: 1 = totals (sched_init + sched_count), 2 = truncation against the totals (sched_apply), 3 = both.  A sharded
// batch all-reduces the totals between the two (bf_group_schedule): sums of the running counts, maximum of the priorities.
cudaError_t launch_schedule(const SchedParams& P, uint32_t sm_count, cudaStream_t stream, uint32_t phases) {
  const uint32_t wpb = 8;
  uint32_t grid = (P.n_runs + wpb - 1) / wpb;
  if (grid == 0) grid = 1;
  if (grid > sm_count * 8) grid = sm_count * 8;
  const uint32_t n_tab = P.n_stories > P.n_queues ? P.n_stories : P.n_queues;
  if (phases & 1u) {
    sched_init<<<(n_tab + 255) / 256 + 1, 256, 0, stream>>>(P);
    sched_count<<<grid, wpb * 32, 0, stream>>>(P);
  }
  if (phases & 2u) sched_apply<<<grid, wpb * 32, 0, stream>>>(P);
  return cudaGetLastError();
}

}  // namespace bf
