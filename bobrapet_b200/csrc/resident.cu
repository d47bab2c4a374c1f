// resident.cu — delta scatter for device-resident state records (SURVEY.md row f2, incremental state upload).
//
// One thread per delta.  Bit-sliced fields (phase 4 planes, cond / decision 2 planes) flip one bit per plane with
// atomicOr / atomicAnd on the record's u32 words, so deltas of different steps that share a word compose; byte
// fields use a word-wide atomic on the containing u32.  At most one delta per (run, field, index) per launch
// (contract in include/bobrafrontier.h), so no ordering between threads is needed.
#include "kernel_common.cuh"

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

__global__ void __launch_bounds__(256) apply_deltas(const DeltaParams P) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n) return;
  const bf_delta d = P.deltas[i];
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
    case BF_DELTA_RUN_FLAGS:
      set_byte(rec, 4u, 0xFFu, d.code);
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
    if (lane == 0) {
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
}

cudaError_t launch_reshape(const ReshapeParams& P, cudaStream_t stream) {
  if (P.n_new == 0) return cudaSuccess;
  reshape_runs<<<(P.n_new - 1u) / 8u + 1u, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

// Retire (bf_resident_retire).  One warp per vacated index m + i: when the run there lives on, the warp copies its state record
// and current result record to its target (16-byte accesses, lane t takes vectors t, t + 32, ...) and lane 0 marks the target;
// then the warp zeroes the vacated state record and its mark.  Targets lie below m and vacated indices at or above it, and
// each lane zeroes only the vectors it read itself, so no warp reads what another writes.
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
  }
  for (uint32_t k = lane; k < sv; k += 32u) s[k] = make_uint4(0u, 0u, 0u, 0u);
  if (lane == 0) P.mark[from] = 0u;
}

cudaError_t launch_retire(const RetireParams& P, cudaStream_t stream) {
  if (P.n == 0) return cudaSuccess;
  retire_runs<<<(P.n - 1u) / 8u + 1u, 256, 0, stream>>>(P);
  return cudaGetLastError();
}

}  // namespace bf
