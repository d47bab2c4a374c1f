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
  if (ok) atomicMax(P.mark + d.run, P.mark_value);   // touch mark (abi.cu, touched ticks); max: an upload's "must list" bit stays
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

// Touch marks of runs [first, first + n) after an upload: epoch << 1 | 1 ("must list", abi.cu)
__global__ void __launch_bounds__(256) mark_runs(uint32_t* mark, uint32_t first, uint32_t n, uint32_t value) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) mark[first + i] = value;
}

cudaError_t launch_mark_runs(uint32_t* mark, uint32_t first, uint32_t n, uint32_t value, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  mark_runs<<<(n + 255) / 256, 256, 0, stream>>>(mark, first, n, value);
  return cudaGetLastError();
}

// Arena compaction (abi.cu): record i moves from src + moves[i].x to dst + moves[i].y (moves[i].z bytes, multiples of 16).
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

}  // namespace bf
