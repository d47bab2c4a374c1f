// compact.cu — result records -> compact lists, on the device (SURVEY.md rows a9 / d).
//
// The consumer of a pass (findAndLaunchReadySteps, dag.go:1735-1775) wants LISTS: the ready steps to hand to
// StepExecutor.Execute and the skipped steps to mark.  A frontier pass over 100k runs x 256 steps leaves ~3 such steps
// per run, yet the dense result records are 80 bytes per run (16-byte header + two 256-bit masks): 8 MB per pass over
// PCIe.  Here every run gets one head word (summary flags | listed | event count) and every (run, step) with a result
// bit one 16-bit event (step | kind << 10), run-major and step-ascending — the order of the reference's lists — so a pass
// ships 4 bytes per run + 2 bytes per event.  In changed-only mode a run whose record equals the previous tick's is not
// listed at all.  Two launches: heads + per-block event totals, then every block sums the totals before it, scans its
// own runs and emits through shared memory (deterministic order: bit-exact against the oracle's masks).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/bobrafrontier.h"
#include "device_record.h"

namespace bf {

constexpr int CB = 512;                  // runs per block (one thread per run)
constexpr uint32_t STAGE_EVENTS = 8192;  // events of a block staged in shared memory (16 KB)

struct RunWords { uint32_t rd, sk, fl, nc, sd; };
__device__ __forceinline__ RunWords load_words(const CompactParams& P, const uint8_t* rr, uint32_t w) {
  RunWords x;
  x.rd = reinterpret_cast<const uint32_t*>(rr + P.off_ready)[w];
  x.sk = reinterpret_cast<const uint32_t*>(rr + P.off_skip)[w];
  x.fl = P.off_fail != BF_OFF_NONE ? reinterpret_cast<const uint32_t*>(rr + P.off_fail)[w] : 0u;
  x.nc = P.off_needs_cond != BF_OFF_NONE ? reinterpret_cast<const uint32_t*>(rr + P.off_needs_cond)[w] : 0u;
  x.sd = P.off_skip_dep != BF_OFF_NONE ? reinterpret_cast<const uint32_t*>(rr + P.off_skip_dep)[w] : 0u;
  return x;
}

__global__ void __launch_bounds__(CB) compact_heads(const CompactParams P) {
  __shared__ uint32_t sh[CB / 32], shl[CB / 32];
  const uint32_t r = blockIdx.x * CB + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t c = 0, listed = 0;
  if (r < P.n_runs) {
    const uint8_t* rr = P.result + (size_t)r * P.result_stride;
    const uint32_t summary = *reinterpret_cast<const uint32_t*>(rr);
    const bool dead = summary == 0xFFFFFFFFu;   // a dead slot's record is empty by contract
    listed = 1;
    if (P.prev_result) {   // changed-only: the run is listed when any word of its record differs from the previous tick's
      const uint32_t* a = reinterpret_cast<const uint32_t*>(rr);
      const uint32_t* b = reinterpret_cast<const uint32_t*>(P.prev_result + (size_t)r * P.result_stride);
      uint32_t diff = 0;
      for (uint32_t x = 0; x < P.result_tail / 4; ++x) diff |= a[x] ^ b[x];
      listed = diff != 0;
    }
    if (listed && !dead)
      for (uint32_t w = 0; w < P.words; ++w) {
        const RunWords x = load_words(P, rr, w);
        c += __popc(x.rd | x.sk | x.fl | x.nc | x.sd);
      }
    const uint32_t hw = (dead ? BF_HEAD_DEAD : (summary & BF_HEAD_SUMMARY_MASK)) | (listed ? BF_HEAD_LISTED : 0u) | (c << BF_HEAD_COUNT_SHIFT);
    P.head[r] = hw;
    if (P.host_head) P.host_head[r] = hw;   // posted, coalesced 128-byte writes over PCIe; visible after the stream's synchronise
  }
  const uint32_t wc = __reduce_add_sync(0xffffffffu, c), wl = __reduce_add_sync(0xffffffffu, listed);
  if (lane == 0) { sh[warp] = wc; shl[warp] = wl; }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t tc = 0, tl = 0;
    for (int k = 0; k < CB / 32; ++k) { tc += sh[k]; tl += shl[k]; }
    P.block_sums[blockIdx.x] = tc;
    if (tl) atomicAdd(&P.total[1], (unsigned long long)tl);   // integer sum: order-free
  }
}

// sum of v[0 .. b): what the blocks before mine (block b of its launch or of its part) produced (every thread of the block gets it)
__device__ __forceinline__ unsigned long long blocks_before(const unsigned long long* v, uint32_t b = blockIdx.x) {
  __shared__ unsigned long long sh64[CB / 32];
  __shared__ unsigned long long base_s;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  unsigned long long part = 0;
  for (uint32_t k = threadIdx.x; k < b; k += CB) part += v[k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_down_sync(0xffffffffu, part, o);
  if (lane == 0) sh64[warp] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int k = 0; k < CB / 32; ++k) t += sh64[k];
    base_s = t;
  }
  __syncthreads();
  return base_s;
}

// exclusive scan of c over the block: returns the sum of the threads before mine; *tot = the block's sum
__device__ __forceinline__ uint32_t block_scan(uint32_t c, uint32_t* tot) {
  __shared__ uint32_t sh[32];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t inc = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= (uint32_t)o) inc += n;
  }
  if (lane == 31) sh[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    uint32_t v = lane < CB / 32 ? sh[lane] : 0u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t n = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= (uint32_t)o) v += n;
    }
    sh[lane] = v;
  }
  __syncthreads();
  *tot = sh[CB / 32 - 1];
  return inc - c + (warp ? sh[warp - 1] : 0u);
}

// the events of one run (result record rr) from position `at` of the block's slice: into the stage, or straight to P.events
__device__ __forceinline__ void emit_run(const CompactParams& P, const uint8_t* rr, uint32_t at, unsigned long long base, bool staged,
                                         uint16_t* stage) {
  for (uint32_t w = 0; w < P.words; ++w) {
    const RunWords x = load_words(P, rr, w);
    for (uint32_t u = x.rd | x.sk | x.fl | x.nc | x.sd; u; u &= u - 1) {
      const uint32_t b = __ffs(u) - 1;
      const uint32_t kind = ((x.rd >> b) & 1u) * BF_EVT_READY | ((x.sk >> b) & 1u) * BF_EVT_SKIP | ((x.fl >> b) & 1u) * BF_EVT_FAIL |
                            ((x.nc >> b) & 1u) * BF_EVT_NEEDS_COND | ((x.sd >> b) & 1u) * BF_EVT_SKIP_DEP;
      const uint16_t e = (uint16_t)((w * 32u + b) | (kind << 10));
      if (staged) stage[at] = e;
      else if (base + at < P.cap) P.events[base + at] = e;
      ++at;
    }
  }
}

// a staged slice of btot events goes out as 32-bit words (two events each: a warp writes 128 contiguous bytes — whole PCIe
// packets when the list is posted straight to the caller's pinned buffer), with a single 16-bit store at an odd start and at
// an odd end
__device__ __forceinline__ void write_slice(const CompactParams& P, unsigned long long base, uint32_t btot, const uint16_t* stage) {
  const unsigned long long room = P.cap > base ? P.cap - base : 0ull;
  const uint32_t n = btot < room ? btot : (uint32_t)room;          // events of my slice that fit the caller's capacity
  const uint32_t lead = (uint32_t)(base & 1ull) < n ? (uint32_t)(base & 1ull) : n;
  if (threadIdx.x == 0 && lead) P.events[base] = stage[0];
  const uint32_t pairs = (n - lead) >> 1;
  uint32_t* out32 = reinterpret_cast<uint32_t*>(P.events + base + lead);
  for (uint32_t i = threadIdx.x; i < pairs; i += CB) out32[i] = (uint32_t)stage[lead + 2 * i] | ((uint32_t)stage[lead + 2 * i + 1] << 16);
  if (threadIdx.x == 0 && ((n - lead) & 1u)) P.events[base + n - 1] = stage[n - 1];
}

__global__ void __launch_bounds__(CB) compact_emit(const CompactParams P) {
  __shared__ uint16_t stage[STAGE_EVENTS];
  // events of the blocks before mine
  const unsigned long long base = blocks_before(P.block_sums);
  const uint32_t r = blockIdx.x * CB + threadIdx.x;
  const uint32_t hw = r < P.n_runs ? P.head[r] : 0u;
  const uint32_t c = hw >> BF_HEAD_COUNT_SHIFT;
  if (P.heads_done && P.host_head && r < P.n_runs) P.host_head[r] = hw;   // the pass left the heads on the device: post them here
  // the next tick's pass adds into the OTHER totals buffer: leave all of it zeroed (ticks may differ in size)
  if (P.zero_sums)
    for (uint32_t i = blockIdx.x * CB + threadIdx.x; i < P.zero_len; i += gridDim.x * CB) P.zero_sums[i] = 0ull;
  // exclusive scan of c over the block
  uint32_t btot;
  const uint32_t before = block_scan(c, &btot);
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
    P.total[0] = base + btot;  // the batch's event count
    if (P.host_tail) {         // posted writes to pinned host memory; visible to the host once the stream has been synchronised
      P.host_tail->events = base + btot;
      for (int k = 0; k < 4; ++k) P.host_tail->counts[k] = P.counts ? P.counts[k] : 0ull;
      P.host_tail->rejected = P.rejected ? (unsigned long long)*P.rejected : 0ull;
      P.host_tail->listed = P.heads_done ? (unsigned long long)P.n_runs : P.total[1];   // (total[1]: every compact_heads block has finished)
    }
    // leave the scratch the way the next tick expects it (no memset launches in the steady state): the listed-runs total
    // and the rejected-delta counter have been delivered
    P.total[1] = 0ull;
    if (P.host_tail && P.rejected) *const_cast<uint32_t*>(P.rejected) = 0u;
  }
  // A block's slice of the list is staged in shared memory and written out by consecutive threads (coalesced 64-byte
  // segments per warp instead of 2-byte scatters); a slice larger than the stage goes out directly.
  const bool staged = btot <= STAGE_EVENTS;
  if (c != 0) emit_run(P, P.result + (size_t)r * P.result_stride, before, base, staged, stage);
  if (!staged) return;
  __syncthreads();
  write_slice(P, base, btot, stage);
}

// ---- touched ticks: the run list in front of the pass, and its compaction behind it ----------------------------------
constexpr uint32_t SCAN_RUNS = 4;   // runs per thread of the list build (one 16-byte load of marks)

// touched runs of my SCAN_RUNS runs: bit k = run r0 + k, below n_scan in the low nibble, at or above it in the high one
__device__ __forceinline__ uint32_t touched_bits(const TouchedParams& P, uint32_t r0) {
  uint32_t bits = 0;
  if (r0 < P.n_marks) {
    const uint4 m = *reinterpret_cast<const uint4*>(P.mark + r0);   // the mark array is padded to a multiple of 4
    const uint32_t mv[4] = {m.x, m.y, m.z, m.w};
#pragma unroll
    for (uint32_t k = 0; k < SCAN_RUNS; ++k)
      if (r0 + k < P.n_marks && (mv[k] >> 1) > P.full_epoch) bits |= 1u << (k + (r0 + k < P.n_scan ? 0u : SCAN_RUNS));
  }
  return bits;
}

// touched runs per block of CB * SCAN_RUNS runs: below n_scan (the list) and at or above it (carried to a later tick)
// (each body runs as block b of nblocks of its tick: the whole launch for one tick, the tick's blocks of a launch over several)
__device__ __forceinline__ void touched_count_body(const TouchedParams& P, uint32_t b) {
  const uint32_t bits = touched_bits(P, (b * CB + threadIdx.x) * SCAN_RUNS);
  uint32_t tot;   // a block counts at most 2048 runs of each kind: one packed scan
  block_scan(__popc(bits & 0xFu) | (__popc(bits >> SCAN_RUNS) << 16), &tot);
  if (threadIdx.x == 0) { P.scan_sums[b] = tot & 0xFFFFu; P.carry_sums[b] = tot >> 16; }
}

// the ascending list: every block writes its touched runs after those of the blocks before it; the last block stores the count
__device__ __forceinline__ void touched_list_body(const TouchedParams& P, uint32_t b, uint32_t nblocks) {
  const unsigned long long base = blocks_before(P.scan_sums, b);
  const uint32_t r0 = (b * CB + threadIdx.x) * SCAN_RUNS;
  uint32_t bits = touched_bits(P, r0) & 0xFu;
  uint32_t btot;
  unsigned long long at = base + block_scan(__popc(bits), &btot);
  for (; bits; bits &= bits - 1, ++at)
    if (at < P.bound) P.list[at] = r0 + __ffs(bits) - 1;   // (the host's bound holds: every touched run has a delta or upload behind it)
  if (b == nblocks - 1) {
    // the touched runs this tick leaves for a later one: the host's next bound starts from them (posted to the pinned tail)
    const unsigned long long carried = blocks_before(P.carry_sums, b) + P.carry_sums[b];
    if (threadIdx.x == 0) {
      *P.list_count = (uint32_t)min(base + btot, (unsigned long long)P.bound);
      P.C.host_tail->carried = carried;
    }
  }
}

// per list position: compare the run's new record with its current one (the bytes compact_heads compares), list it when they
// differ or it must be listed, bring the current record up to date and clear the run's mark; head word and events as compact_heads
__device__ __forceinline__ void touched_heads_body(const TouchedParams& P, uint32_t b) {
  const CompactParams& C = P.C;
  const uint32_t i = b * CB + threadIdx.x;
  const uint32_t n = min(*P.list_count, P.bound);
  uint32_t c = 0, listed = 0;
  if (i < n) {
    const uint32_t r = P.list[i];
    const uint8_t* nr = C.result + (size_t)r * C.result_stride;
    uint8_t* cr = const_cast<uint8_t*>(C.prev_result) + (size_t)r * C.result_stride;
    const uint32_t summary = *reinterpret_cast<const uint32_t*>(nr);
    const bool dead = summary == 0xFFFFFFFFu;
    // 16 bytes at a time: the bytes between result_tail and the next multiple of 16 are padding, zero in every record
    uint32_t diff = 0;
#pragma unroll 4
    for (uint32_t x = 0; x < (C.result_tail + 15) / 16; ++x) {
      const uint4 u = reinterpret_cast<const uint4*>(nr)[x], v = reinterpret_cast<const uint4*>(cr)[x];
      diff |= (u.x ^ v.x) | (u.y ^ v.y) | (u.z ^ v.z) | (u.w ^ v.w);
    }
    listed = (diff != 0 || (P.mark[r] & 1u)) ? 1u : 0u;
    if (diff)
#pragma unroll 4
      for (uint32_t x = 0; x < C.result_stride / 16; ++x) reinterpret_cast<uint4*>(cr)[x] = reinterpret_cast<const uint4*>(nr)[x];
    P.mark[r] = 0u;   // evaluated: untouched until its next delta or upload
    if (listed && !dead)
      for (uint32_t w = 0; w < C.words; ++w) {
        const RunWords x = load_words(C, nr, w);
        c += __popc(x.rd | x.sk | x.fl | x.nc | x.sd);
      }
    P.pos_head[i] = (dead ? BF_HEAD_DEAD : (summary & BF_HEAD_SUMMARY_MASK)) | (listed ? BF_HEAD_LISTED : 0u) | (c << BF_HEAD_COUNT_SHIFT);
  }
  // events of a block <= 512 * 1024 < 2^20, listed runs <= 512: one packed scan
  uint32_t tot;
  block_scan(c | (listed << 20), &tot);
  if (threadIdx.x == 0) { P.sums[b] = tot & 0xFFFFFu; P.sums_listed[b] = tot >> 20; }
}

// the listed runs in list order: runs[] and head[] (first runs_cap), events as compact_emit (same staging and capacity rules)
__device__ __forceinline__ void touched_emit_body(const TouchedParams& P, uint32_t b, uint32_t nblocks) {
  __shared__ uint16_t stage[STAGE_EVENTS];
  const CompactParams& C = P.C;
  const unsigned long long base = blocks_before(P.sums, b), base_l = blocks_before(P.sums_listed, b);
  const uint32_t i = b * CB + threadIdx.x;
  const uint32_t n = min(*P.list_count, P.bound);
  const uint32_t hw = i < n ? P.pos_head[i] : 0u;
  const uint32_t listed = (hw & BF_HEAD_LISTED) ? 1u : 0u, c = hw >> BF_HEAD_COUNT_SHIFT;
  uint32_t tot;
  const uint32_t before_p = block_scan(c | (listed << 20), &tot);
  const uint32_t before = before_p & 0xFFFFFu, btot = tot & 0xFFFFFu;
  const uint32_t r = listed ? P.list[i] : 0u;
  if (listed) {
    const unsigned long long k = base_l + (before_p >> 20);
    if (k < P.runs_cap) { P.out_runs[k] = r; P.out_head[k] = hw; }
  }
  if (b == nblocks - 1 && threadIdx.x == 0) {
    ResultTail& t = *C.host_tail;   // pinned host memory: visible to the host once the stream has been synchronised
    t.events = base + btot;
    for (int k = 0; k < 4; ++k) t.counts[k] = C.counts ? C.counts[k] : 0ull;
    t.rejected = C.rejected ? (unsigned long long)*C.rejected : 0ull;
    t.listed = base_l + (tot >> 20);
    t.evaluated = n;
    if (C.rejected) *const_cast<uint32_t*>(C.rejected) = 0u;   // delivered: clean for the next tick
  }
  const bool staged = btot <= STAGE_EVENTS;
  if (c != 0) emit_run(C, C.result + (size_t)r * C.result_stride, before, base, staged, stage);
  if (!staged) return;
  __syncthreads();
  write_slice(C, base, btot, stage);
}

__global__ void __launch_bounds__(CB) touched_count(const TouchedParams P) { touched_count_body(P, blockIdx.x); }
__global__ void __launch_bounds__(CB) touched_list(const TouchedParams P) { touched_list_body(P, blockIdx.x, gridDim.x); }
__global__ void __launch_bounds__(CB) touched_heads(const TouchedParams P) { touched_heads_body(P, blockIdx.x); }
__global__ void __launch_bounds__(CB) touched_emit(const TouchedParams P) { touched_emit_body(P, blockIdx.x, gridDim.x); }

// ---- several touched ticks in one launch per stage (bf_resident_tick_touched_many): the blocks of tick k are
// [first[k], first[k + 1]) of the launch; each runs the single tick's body as block blockIdx.x - first[k] of its tick
struct PartBlock { uint32_t k, b, n; };
__device__ __forceinline__ PartBlock part_block(const uint32_t* first, uint32_t n_parts) {
  uint32_t lo = 0, hi = n_parts;   // the last k with first[k] <= blockIdx.x
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (first[mid] <= blockIdx.x) lo = mid; else hi = mid;
  }
  return {lo, blockIdx.x - first[lo], first[lo + 1] - first[lo]};
}
__global__ void __launch_bounds__(CB) touched_count_many(const TouchedParams* __restrict__ T, const uint32_t* __restrict__ first, uint32_t n) {
  const PartBlock p = part_block(first, n);
  touched_count_body(T[p.k], p.b);
}
__global__ void __launch_bounds__(CB) touched_list_many(const TouchedParams* __restrict__ T, const uint32_t* __restrict__ first, uint32_t n) {
  const PartBlock p = part_block(first, n);
  touched_list_body(T[p.k], p.b, p.n);
}
__global__ void __launch_bounds__(CB) touched_heads_many(const TouchedParams* __restrict__ T, const uint32_t* __restrict__ first, uint32_t n) {
  const PartBlock p = part_block(first, n);
  touched_heads_body(T[p.k], p.b);
}
__global__ void __launch_bounds__(CB) touched_emit_many(const TouchedParams* __restrict__ T, const uint32_t* __restrict__ first, uint32_t n) {
  const PartBlock p = part_block(first, n);
  touched_emit_body(T[p.k], p.b, p.n);
}

// T, list_first and compact_first are device arrays of n ticks; list_first / compact_first hold the block starts of each tick
// (ceil(n_marks / 2048) list blocks, ceil(bound / 512) compaction blocks, every tick at least one) and the total at [n]
cudaError_t launch_touched_list_many(const TouchedParams* T, const uint32_t* list_first, uint32_t n, uint32_t blocks, cudaStream_t stream) {
  touched_count_many<<<blocks, CB, 0, stream>>>(T, list_first, n);
  touched_list_many<<<blocks, CB, 0, stream>>>(T, list_first, n);
  return cudaGetLastError();
}
cudaError_t launch_touched_compact_many(const TouchedParams* T, const uint32_t* compact_first, uint32_t n, uint32_t blocks,
                                        cudaStream_t stream) {
  touched_heads_many<<<blocks, CB, 0, stream>>>(T, compact_first, n);
  touched_emit_many<<<blocks, CB, 0, stream>>>(T, compact_first, n);
  return cudaGetLastError();
}

cudaError_t launch_touched_list(const TouchedParams& P, cudaStream_t stream) {
  const uint32_t nb = (P.n_marks + CB * SCAN_RUNS - 1) / (CB * SCAN_RUNS);
  touched_count<<<nb, CB, 0, stream>>>(P);
  touched_list<<<nb, CB, 0, stream>>>(P);
  return cudaGetLastError();
}

cudaError_t launch_touched_compact(const TouchedParams& P, cudaStream_t stream) {
  const uint32_t nb = (P.bound + CB - 1) / CB;
  touched_heads<<<nb, CB, 0, stream>>>(P);
  touched_emit<<<nb, CB, 0, stream>>>(P);
  return cudaGetLastError();
}

// scratch: block_sums needs ceil(n / 512) u64; total[2] is zero on entry (the caller zeroes it once, compact_emit leaves it zeroed)
cudaError_t launch_compact(const CompactParams& P, cudaStream_t stream) {
  if (P.n_runs == 0) {
    if (P.host_tail) *P.host_tail = ResultTail{};   // pinned host memory: plain store (caller synchronised)
    return cudaSuccess;
  }
  const uint32_t nb = (P.n_runs + CB - 1) / CB;
  if (!P.heads_done) compact_heads<<<nb, CB, 0, stream>>>(P);
  compact_emit<<<nb, CB, 0, stream>>>(P);
  return cudaGetLastError();
}

}  // namespace bf
