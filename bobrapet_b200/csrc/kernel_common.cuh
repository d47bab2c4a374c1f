// kernel_common.cuh — PTX / bit-plane helpers shared by the frontier kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/bobrafrontier.h"
#include "device_record.h"

namespace bf {

#define DI __device__ __forceinline__
constexpr uint32_t FULL = 0xffffffffu;

// ------------------------------------------------------------------ PTX helpers
DI uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
DI void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
DI void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
DI uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok;
}
DI void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// TMA bulk copy global -> shared, completion counted in bytes on an mbarrier.
DI void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
DI void sts_zero16(uint32_t a) { asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(a), "r"(0u) : "memory"); }
DI void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

template <int IMM>
DI uint32_t lop3(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t r;
  asm("lop3.b32 %0, %1, %2, %3, %4;" : "=r"(r) : "r"(a), "r"(b), "r"(c), "n"(IMM));
  return r;
}
// 16-entry boolean table over a bit-sliced 4-bit code: 3 LOP3 for 32 steps.
template <uint32_t T16>
DI uint32_t plut(uint32_t p0, uint32_t p1, uint32_t p2, uint32_t p3) {
  const uint32_t lo = lop3<(T16 & 0xFF)>(p2, p1, p0);
  const uint32_t hi = lop3<((T16 >> 8) & 0xFF)>(p2, p1, p0);
  return lop3<0xCA>(p3, hi, lo);  // p3 ? hi : lo
}
// set the code of the steps in mask m to the constant CODE
template <int CODE>
DI void pset(uint32_t m, uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3) {
  p0 = (CODE & 1) ? (p0 | m) : (p0 & ~m);
  p1 = (CODE & 2) ? (p1 | m) : (p1 & ~m);
  p2 = (CODE & 4) ? (p2 | m) : (p2 & ~m);
  p3 = (CODE & 8) ? (p3 | m) : (p3 & ~m);
}
// Launch effects of Execute (dag.go:1735-1775, step_executor.go:132-185) on one word of codes: the skipped steps become Skipped,
// launched condition steps Succeeded, sleep / wait / gate steps Paused, parallel steps Running, and the other launched steps but
// stop steps Running when their code is 0 or 14.  The fixpoint applies them in registers between iterations; bf_resident_commit
// writes them into the records.
DI void launch_effects(uint32_t skip, uint32_t launched, uint32_t T_COND, uint32_t SYNC_T, uint32_t T_PAR, uint32_t T_STOP,
                       uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3) {
  pset<BF_PHASE_SKIPPED>(skip, p0, p1, p2, p3);
  const uint32_t none_or_q = ~(p0 | p1 | p2 | p3) | (~p0 & p1 & p2 & p3);  // code 0 or 14
  pset<BF_PHASE_SUCCEEDED>(launched & T_COND, p0, p1, p2, p3);
  pset<BF_PHASE_PAUSED>(launched & SYNC_T, p0, p1, p2, p3);
  pset<BF_PHASE_RUNNING>(launched & T_PAR, p0, p1, p2, p3);
  pset<BF_PHASE_RUNNING>(launched & ~T_COND & ~SYNC_T & ~T_PAR & ~T_STOP & none_or_q, p0, p1, p2, p3);
}
DI uint32_t squeeze4(uint32_t x) {  // bits 0,4,..,28 -> low byte
  x = (x | (x >> 3)) & 0x03030303u;
  x = (x | (x >> 6)) & 0x000F000Fu;
  x = (x | (x >> 12)) & 0xFFu;
  return x;
}
DI uint32_t squeeze2(uint32_t x) {  // bits 0,2,..,30 -> low half
  x = (x | (x >> 1)) & 0x33333333u;
  x = (x | (x >> 2)) & 0x0F0F0F0Fu;
  x = (x | (x >> 4)) & 0x00FF00FFu;
  x = (x | (x >> 8)) & 0xFFFFu;
  return x;
}
DI uint32_t spread4(uint32_t x) {  // inverse of squeeze4
  x = (x | (x << 12)) & 0x000F000Fu;
  x = (x | (x << 6)) & 0x03030303u;
  x = (x | (x << 3)) & 0x11111111u;
  return x;
}
DI uint32_t bits4_to_bytes(uint32_t nib) { return (nib * 0x00204081u) & 0x01010101u; }  // 4 bits -> 4 0/1 bytes
DI uint32_t get_nibble(const uint8_t* base, uint32_t i) {
  const uint32_t v = (base[i >> 1] >> ((i & 1u) * 4u)) & 0xFu;
  return v == 15u ? 0u : v;
}
DI uint32_t redux_or(uint32_t v) { return __reduce_or_sync(FULL, v); }
DI uint32_t redux_add(uint32_t v) { return __reduce_add_sync(FULL, v); }
// Segmented reductions: every lane gets the OR / sum / max of the aligned segment of 2^lg lanes that holds it (lg warp-uniform,
// at most 5), by a butterfly of full-mask shuffles.  A __reduce_*_sync over a sub-warp mask is one REDUX only when the mask is
// the same in every lane; with a different mask per segment ptxas runs it once per distinct mask in a divergent fallback
// block (WARPSYNC.COLLECTIVE on the mask register) far from the loop.  tests/test_sass_collectives.py keeps that block out of
// the frontier kernels.
DI uint32_t seg_or(uint32_t v, uint32_t lg) {
  for (uint32_t o = (1u << lg) >> 1; o; o >>= 1) v |= __shfl_xor_sync(FULL, v, o);
  return v;
}
DI uint32_t seg_add(uint32_t v, uint32_t lg) {
  for (uint32_t o = (1u << lg) >> 1; o; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
DI uint32_t seg_max(uint32_t v, uint32_t lg) {
  for (uint32_t o = (1u << lg) >> 1; o; o >>= 1) v = max(v, __shfl_xor_sync(FULL, v, o));
  return v;
}

// ---- per-run lists (bf_resident_schedule, _status, _resync, _commit_journal): count, scan, list ------------------------------
// A count launch gives each warp one word for its run (or runs) and stores each CTA's K totals; cta_scan (resident.cu) turns each
// of the K arrays of CTA totals into the totals of the CTAs before each and posts the sums; the list launch rebuilds each run's
// offsets from them and writes its items.  part(word, k) is a word's share of total k, the same in both launches.
cudaError_t launch_cta_scan(unsigned long long* cta, unsigned long long* total, uint32_t n_ctas, uint32_t K, cudaStream_t stream);

// Count (every thread of the CTA): lane 0 of each warp passes its word (0 for a warp without a run); thread 0 stores total k of
// the CTA's words at cta[k * gridDim.x + blockIdx.x].  Its 32 bytes of static shared memory are kStatusStaticSmem.
// The _at forms take the block and the number of blocks in place of the CTA's own: a launch whose CTAs walk several blocks of
// runs (the touched commit's list-mode builds) stores and reads one total per block.
template <uint32_t K, class Part>
DI void store_cta_totals_at(uint32_t word, unsigned long long* cta, Part part, uint32_t block, uint32_t n_blocks) {
  __shared__ uint32_t warp_word[8];
  if ((threadIdx.x & 31u) == 0) warp_word[threadIdx.x >> 5] = word;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (uint32_t k = 0; k < K; ++k) {
    unsigned long long sum = 0;
    for (uint32_t w = 0; w < (blockDim.x >> 5); ++w) sum += part(warp_word[w], k);
    cta[k * n_blocks + block] = sum;
  }
}
template <uint32_t K, class Part>
DI void store_cta_totals(uint32_t word, unsigned long long* cta, Part part) {
  store_cta_totals_at<K>(word, cta, part, blockIdx.x, gridDim.x);
}

// List (whole warp): the offsets of the run whose word is run_words[i], the CTA's runs starting at run_words[first]: the totals of
// the CTAs before (after cta_scan) and of the warps before it in its CTA.
template <uint32_t K, class Part>
DI void run_offsets_at(const unsigned long long* cta, const uint32_t* run_words, uint32_t first, uint32_t i, Part part,
                       unsigned long long (&base)[K], uint32_t block, uint32_t n_blocks) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t before = first + lane < i ? run_words[first + lane] : 0u;
  for (uint32_t k = 0; k < K; ++k) base[k] = cta[k * n_blocks + block] + redux_add(part(before, k));
}
template <uint32_t K, class Part>
DI void run_offsets(const unsigned long long* cta, const uint32_t* run_words, uint32_t first, uint32_t i, Part part,
                    unsigned long long (&base)[K]) {
  run_offsets_at<K>(cta, run_words, first, i, part, base, blockIdx.x, gridDim.x);
}

// Emit (whole warp): one item per set bit of this lane's `bits`, lane by lane and bit by bit (step order when lane w holds word
// w of the steps), from position pos; store(b, at) writes bit b's item at `at`, for every at below cap.  -> the position after
// the warp's items
template <class Store>
DI unsigned long long emit_bits(uint32_t bits, unsigned long long pos, unsigned long long cap, Store store) {
  const uint32_t lane = threadIdx.x & 31u, mine = (uint32_t)__popc(bits);
  uint32_t incl = mine;
  for (uint32_t d = 1; d < 32; d <<= 1) {
    const uint32_t x = __shfl_up_sync(FULL, incl, d);
    if (lane >= d) incl += x;
  }
  unsigned long long at = pos + incl - mine;
  for (uint32_t x = bits; x && at < cap; x &= x - 1u, ++at) store((uint32_t)__ffs(x) - 1u, at);
  return pos + __shfl_sync(FULL, incl, 31);
}

DI uint32_t bmsk_clamp(uint32_t pos, uint32_t width) {
  uint32_t r;
  asm("bmsk.clamp.b32 %0, %1, %2;" : "=r"(r) : "r"(pos), "r"(width));
  return r;
}

// ---- shared-space accessors on 32-bit addresses (keeps the walk's address math in 32 bits) ----
DI uint32_t lds_u8(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
DI uint32_t lds_u16(uint32_t a) { uint32_t v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
DI uint32_t lds_u32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
// polling load of a word another warp publishes: volatile at the PTX level and a compiler barrier (a plain asm-volatile load
// in an empty loop was dropped by the compiler together with the loop)
DI uint32_t lds_poll_u32(uint32_t a) { uint32_t v; asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
DI uint4 lds_v4(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
  return v;
}
DI void sts_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
DI void sts_v4(uint32_t a, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
DI void red_or_shared(uint32_t a, uint32_t v) { asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
DI void sts_v2(uint32_t a, uint32_t x, uint32_t y) { asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y) : "memory"); }// generic pointer of a shared-window address (rare paths only: parallel join, in-loop failure fix-up)
DI const uint8_t* gptr(uint32_t a) { return static_cast<const uint8_t*>(__cvta_shared_to_generic(a)); }
// keep a loop-invariant value in a register instead of letting the compiler rematerialise it from constants
DI uint32_t pin(uint32_t v) { asm volatile("" : "+r"(v)); return v; }

// ------------------------------------------------------------------ stage D: the dependency walk
// findReadySteps' inner loop (dag.go:2711-2733): one step per lane over the `needs` row of every candidate step,
// visiting only the 32-step words that hold a candidate.  The row formats and their fetch (row_locate, row_fetch) are
// shared; how a dependency's status is kept is each kernel's own: the one-run-per-warp kernel (frontier_kernel.cu, the
// walks below) keeps one status byte per step, bit0 = not satisfied, bit1 = failed dependency, with the byte at index
// PAD = 32*W (just past the last step word) always 0; the packed-lanes kernel keeps bit words (frontier_pack.cu).
//
// Row formats (device_record.h), a compile-time parameter of the hot walks:
//   FMT_CSR4   CSR, no row longer than 4: the first four entries are fetched branch-free and clamp-free (col_idx carries
//              four zero entries of padding, so whatever lies past a short row is a valid step index; the verdict is
//              masked with the row length)
//   FMT_CSRL   CSR with longer rows: the same plus a tail loop
//   FMT_ELL2 / FMT_ELL4   fixed-width rows of 2 / 4 entries, unused entries = PAD: no row_ptr, no mask
//   FMT_ELL2B / FMT_ELL4B the same with BYTE entries (S <= 256): a row is ONE 16- / 32-bit load; short rows repeat their
//              first entry, rows without needs are kept out of the walk by the NODEP plane (device_record.h)
//   FMT_ELL4P  four 10-BIT entries (S > 512, the one-run-per-warp kernel only): one 32-bit load + one byte load per row; the
//              `rp_addr` argument of the walks carries the address of the block's high-byte array (there is no row_ptr)
enum : int { FMT_CSR4 = 0, FMT_CSRL = 1, FMT_ELL2 = 2, FMT_ELL4 = 4, FMT_ELL2B = 0x102, FMT_ELL4B = 0x104, FMT_ELL4P = 0x204 };
template <int FMT> struct fmt_traits {
  static constexpr bool byte_rows = (FMT & 0x100) != 0;
  static constexpr bool packed10 = (FMT & 0x200) != 0;
  static constexpr bool fixed = FMT >= 2;
  static constexpr uint32_t row_bytes = packed10 ? 4u : (byte_rows ? (uint32_t)(FMT & 0xFF) : 2u * (uint32_t)(FMT & 0xFF));  // fixed formats (10-bit: the lo words)
};

DI int fmt_of(uint32_t ell, uint32_t max_deg) { return ell ? (int)ell : (max_deg > 4 ? FMT_CSRL : FMT_CSR4); }

// phase 1 of an item: where the row of step `i` starts (shared address) and, for CSR, its length
template <int FMT>
DI void row_locate(bool cand, uint32_t i, uint32_t rp_addr, uint32_t col_addr, uint32_t& p, uint32_t& n) {
  if (fmt_traits<FMT>::packed10) { p = col_addr + i * 4u; n = rp_addr + i; }   // n carries the address of the row's high byte
  else if (fmt_traits<FMT>::fixed) { p = col_addr + i * fmt_traits<FMT>::row_bytes; n = (uint32_t)(FMT & 0xFF); }  // rows exist for every step of the word (padded to 32*W)
  else {
    uint32_t e0 = 0;
    n = 0;
    if (cand) { const uint32_t a = rp_addr + i * 2u; e0 = lds_u16(a); n = lds_u16(a + 2u) - e0; }
    p = col_addr + e0 * 2u;
  }
}
// phase 2: the first entries of the row (may run past a short CSR row: valid indices, masked in phase 3)
template <int FMT>
DI void row_fetch(uint32_t p, uint32_t n, uint32_t (&x)[4]) {
  if (FMT == FMT_ELL4P) {
    const uint32_t lo = lds_u32(p), hi = lds_u8(n);
    x[0] = lo & 0x3FFu; x[1] = (lo >> 10) & 0x3FFu; x[2] = (lo >> 20) & 0x3FFu; x[3] = (lo >> 30) | (hi << 2);
    return;
  }
  if (FMT == FMT_ELL4B) {
    const uint32_t r = lds_u32(p);
    x[0] = r & 0xFFu; x[1] = (r >> 8) & 0xFFu; x[2] = (r >> 16) & 0xFFu; x[3] = r >> 24;
    return;
  }
  if (FMT == FMT_ELL2B) {
    const uint32_t r = lds_u16(p);
    x[0] = r & 0xFFu; x[1] = r >> 8;
    return;
  }
  x[0] = lds_u16(p); x[1] = lds_u16(p + 2u);
  if (FMT != FMT_ELL2) { x[2] = lds_u16(p + 4u); x[3] = lds_u16(p + 6u); }
}
// phase 3, one-run-per-warp kernel: OR of the status bytes of the row's dependencies (CSR: one byte lane per entry, masked by
// the row length)
template <int FMT>
DI uint32_t row_status_bytes(uint32_t p, uint32_t n, const uint32_t (&x)[4], uint32_t st_addr) {
  if (FMT == FMT_ELL2 || FMT == FMT_ELL2B) return lds_u8(st_addr + x[0]) | lds_u8(st_addr + x[1]);
  const uint32_t s0 = lds_u8(st_addr + x[0]), s1 = lds_u8(st_addr + x[1]), s2 = lds_u8(st_addr + x[2]), s3 = lds_u8(st_addr + x[3]);
  if (FMT == FMT_ELL4 || FMT == FMT_ELL4B || FMT == FMT_ELL4P) return s0 | s1 | s2 | s3;
  uint32_t w = (((s3 * 256u + s2) * 256u + s1) * 256u + s0) & bmsk_clamp(0u, n * 8u);
  if (FMT == FMT_CSRL)
    for (uint32_t q = 4; q < n; ++q) w |= lds_u8(st_addr + lds_u16(p + q * 2u));
  return w;
}

// ---- one run per warp (frontier_kernel.cu): K candidate words at once = K independent load chains in flight.
// All K words exist (the driver below only calls it with at least K left).
template <int K, int FMT, bool NEED_FD>
DI void walk_group(uint32_t lane, uint32_t CAND, uint32_t& todo, uint32_t rp_addr, uint32_t col_addr, uint32_t st_addr,
                   uint32_t& met_w, uint32_t& fd_w) {
  uint32_t j[K], p[K], n[K], w[K], cw[K], x[K][4];
  bool c[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    j[k] = __ffs(todo) - 1;
    todo &= todo - 1;
  }
#pragma unroll
  for (int k = 0; k < K; ++k) {
    cw[k] = __shfl_sync(FULL, CAND, j[k]);
    c[k] = (cw[k] >> lane) & 1u;
    row_locate<FMT>(c[k], j[k] * 32u + lane, rp_addr, col_addr, p[k], n[k]);
  }
#pragma unroll
  for (int k = 0; k < K; ++k) row_fetch<FMT>(p[k], n[k], x[k]);
#pragma unroll
  for (int k = 0; k < K; ++k) w[k] = row_status_bytes<FMT>(p[k], n[k], x[k], st_addr);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    if (fmt_traits<FMT>::fixed) {   // every lane holds a real row: the (lane-uniform) candidate word masks the ballot
      const uint32_t m = __ballot_sync(FULL, (w[k] & 0x01010101u) == 0) & cw[k];
      if (lane == j[k]) met_w = m;
      if (NEED_FD) {
        const uint32_t f = __ballot_sync(FULL, (w[k] & 0x02020202u) != 0) & cw[k];
        if (lane == j[k]) fd_w = f;
      }
    } else {
      const uint32_t m = __ballot_sync(FULL, c[k] && (w[k] & 0x01010101u) == 0);
      if (lane == j[k]) met_w = m;
      if (NEED_FD) {
        const uint32_t f = __ballot_sync(FULL, c[k] && (w[k] & 0x02020202u) != 0);
        if (lane == j[k]) fd_w = f;
      }
    }
  }
}

// Stage D driver: the candidate words of a run, KMAX at a time while that many are left, then 2, then 1.
// KMAX = 1 is the plain walk; 2 is used at two CTAs per SM, 4 where one CTA per SM leaves little else to hide
// latency.
template <int KMAX, int FMT, bool NEED_FD>
DI void walk_words(uint32_t lane, uint32_t CAND, uint32_t rp_addr, uint32_t col_addr, uint32_t st_addr, uint32_t& met_w,
                   uint32_t& fd_w) {
  met_w = 0;
  fd_w = 0;
  uint32_t todo = __ballot_sync(FULL, CAND != 0);  // words with at least one candidate step
  if (KMAX >= 4)
    while (__popc(todo) >= 4) walk_group<4, FMT, NEED_FD>(lane, CAND, todo, rp_addr, col_addr, st_addr, met_w, fd_w);
  if (KMAX >= 2) {
    if (KMAX >= 4) {
      if (__popc(todo) >= 2) walk_group<2, FMT, NEED_FD>(lane, CAND, todo, rp_addr, col_addr, st_addr, met_w, fd_w);
    } else {
      while (__popc(todo) >= 2) walk_group<2, FMT, NEED_FD>(lane, CAND, todo, rp_addr, col_addr, st_addr, met_w, fd_w);
    }
  }
  if (KMAX >= 2) {
    if (todo) walk_group<1, FMT, NEED_FD>(lane, CAND, todo, rp_addr, col_addr, st_addr, met_w, fd_w);
  } else {
    while (todo) walk_group<1, FMT, NEED_FD>(lane, CAND, todo, rp_addr, col_addr, st_addr, met_w, fd_w);
  }
}

template <int KMAX, bool NEED_FD>
DI void walk_words_fmt(int fmt, uint32_t lane, uint32_t CAND, uint32_t rp_addr, uint32_t col_addr, uint32_t st_addr,
                       uint32_t& met_w, uint32_t& fd_w) {  // fmt is warp-uniform
  if (fmt == FMT_ELL4P) walk_words<KMAX, FMT_ELL4P, NEED_FD>(lane, CAND, rp_addr, col_addr, st_addr, met_w, fd_w);
  else if (fmt == FMT_ELL4B) walk_words<KMAX, FMT_ELL4B, NEED_FD>(lane, CAND, rp_addr, col_addr, st_addr, met_w, fd_w);
  else if (fmt == FMT_ELL4) walk_words<KMAX, FMT_ELL4, NEED_FD>(lane, CAND, rp_addr, col_addr, st_addr, met_w, fd_w);
  else if (fmt == FMT_ELL2B) walk_words<KMAX, FMT_ELL2B, NEED_FD>(lane, CAND, rp_addr, col_addr, st_addr, met_w, fd_w);
  else if (fmt == FMT_CSR4) walk_words<KMAX, FMT_CSR4, NEED_FD>(lane, CAND, rp_addr, col_addr, st_addr, met_w, fd_w);
  else if (fmt == FMT_ELL2) walk_words<KMAX, FMT_ELL2, NEED_FD>(lane, CAND, rp_addr, col_addr, st_addr, met_w, fd_w);
  else walk_words<KMAX, FMT_CSRL, NEED_FD>(lane, CAND, rp_addr, col_addr, st_addr, met_w, fd_w);
}

// ---- the fix-up walk (rare): a step set Failed earlier in this same loop (dag.go:2744/2810 mutate stepStates while
// `completed` stays as built at :497) is visible to LATER steps of the list only.  Plain loop over every entry of the
// row, any format.  The item (word j of the run whose CAND word is held by lane `owner`) is given by the caller, and so is
// `status(d)`: dependency d's status in the kernel's own representation, as bit0 = not satisfied, bit1 = failed dependency.
template <class Status>
DI void fixup_item(uint32_t lane, uint32_t candw, uint32_t j, uint32_t ell, uint32_t rp_addr, uint32_t col_addr, Status status,
                   uint32_t mfail_addr, uint32_t failed_class, uint32_t& metb, uint32_t& fdb) {
  const bool cand = (candw >> lane) & 1u;
  const uint32_t i = j * 32u + lane;
  uint32_t acc = 0;
  if (cand) {
    uint32_t p, n;
    const uint32_t eb = (ell & ELL_BYTE) ? 1u : 2u;   // bytes per entry (the caller keeps NODEP steps out of candw)
    uint32_t lo10 = 0, hi10 = 0;
    if (ell & ELL_PACK10) { n = 4u; p = 0; lo10 = lds_u32(col_addr + i * 4u); hi10 = lds_u8(rp_addr + i); }  // rp_addr: the high-byte array
    else if (ell) { n = ell_k(ell); p = col_addr + i * n * eb; }
    else { const uint32_t a = rp_addr + i * 2u; const uint32_t e0 = lds_u16(a); n = lds_u16(a + 2u) - e0; p = col_addr + e0 * 2u; }
    for (uint32_t e = 0; e < n; ++e) {
      const uint32_t d = (ell & ELL_PACK10) ? (e < 3u ? (lo10 >> (10u * e)) & 0x3FFu : (lo10 >> 30) | (hi10 << 2))
                                            : (eb == 1u ? lds_u8(p + e) : lds_u16(p + e * 2u));
      uint32_t sb = status(d);
      if (d < i && ((lds_u32(mfail_addr + (d >> 5) * 4u) >> (d & 31u)) & 1u)) sb = failed_class;  // PAD >= i: never
      acc |= sb;
    }
  }
  fdb = __ballot_sync(FULL, cand && (acc & 2u) != 0);
  metb = __ballot_sync(FULL, cand && (acc & 1u) == 0);
}

}  // namespace bf
