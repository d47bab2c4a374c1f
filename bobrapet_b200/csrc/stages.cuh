// stages.cuh — the bit-plane stages of a frontier pass around the dependency walk, one definition for both kernels:
// frontier_kernel.cu (one run per warp) and frontier_pack.cu (a group of R = 32 / Wq runs per warp).
//
// A lane holds word w (32 steps) of one run: w = lane in the general kernel, lane = g * Wq + w in the packed-lanes kernel.
// Per-run reductions run over `gmask`, the lanes of the caller's run (FULL in the general kernel).  No collective sits under
// a per-run branch: a run that does not take a step still takes part in every vote.
#pragma once
#include "kernel_common.cuh"

namespace bf {

// ------------------------------------------------------------------ conditions the packed-lanes producer relies on
// Any edit to stages G, I, D-prep or the cond-FAIL fix-up below must keep all three.
//
// (1) No stage of a single pass makes a candidate of a step whose INPUT code (15 read as 0) lies in TERMINAL ∪ RUNNING_Q:
//     stage G rewrites only RUNNING sync steps, into 8 or a terminal code; stage I and the fix-up only set Skipped /
//     Failed; GSEL and NODEP only narrow.  The producer (the cut, frontier_pack.cu) stages a run's rows only from its first
//     word with a code outside that set, so the rows below are never read.
// (2) A fail-fast run whose group the host does not set, with a code of TERMINAL \ COMPLETED0 (4, 5, 6, 7, 11, 12) on a
//     main step without allowFailure, in a topology with G1 = G2 = 0, has CAND = 0 in every word.  Stage G rewrites only
//     RUNNING sync steps, so that code survives it and the step is FAILED & GM: amf holds, and stage I marks mark_ff =
//     GM & ~COMPL & ~RUNQ & ~TERM Skipped.  With G1 = G2 = 0, GSEL is GM (CAND0 = GM minus what mark_ff just covered:
//     empty) or the group is DONE (CAND0 = 0); the topology-terminated branch only adds Failed steps.  The producer stages
//     none of such a run's rows (the fail-fast skip of the cut).
// (3) In a pass without cond and decision codes, a run without BF_RF_TOPOLOGY_TERMINATED in a topology with G1 = G2 = 0
//     that condition (2) does not exempt has every step that is satisfied or a failed dependency ((VALID & ~U) | FD) among
//     the steps whose INPUT code is TERMINAL, or TERMINAL ∪ RT_SAT for a realtime run: without stage G and the fix-up,
//     SAT ⊆ COMPLETED0 ∪ TERM ∪ RT_SAT and FD ⊆ TERM; mark_cs needs a compensation step, mark_ff fires only under
//     condition (2), and only the topology-terminated branch sets other Failed codes.  The producer stages and the walk
//     reads no rows of a word whose dependency floor lies above the highest such step (the floor cut, frontier_pack.cu).

// ------------------------------------------------------------------ stage G: gate / sleep / wait sync
// dag.go:1469-1533, 1235-1277, 1327-1437.  A RUNNING sync step (SYNC_T: sleep, wait, gate) takes the code its decision
// (d0, d1; TS per step) names.  Returns the steps whose code really changed: a rewrite may write the code a step already has.
DI uint32_t stage_g(uint32_t SYNC_T, uint32_t TS, uint32_t d0, uint32_t d1, uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3) {
  const uint32_t syn = SYNC_T & plut<BF_LUT_RUNNING>(p0, p1, p2, p3);
  const uint32_t n0 = d0;
  const uint32_t n1 = d0 & ~(d1 & TS);
  const uint32_t n2 = d1 & (~d0 | TS);
  const uint32_t n3 = ~(d0 ^ d1);
  const uint32_t dirty = syn & ((p0 ^ n0) | (p1 ^ n1) | (p2 ^ n2) | (p3 ^ n3));
  p0 = (p0 & ~syn) | (n0 & syn);
  p1 = (p1 & ~syn) | (n1 & syn);
  p2 = (p2 & ~syn) | (n2 & syn);
  p3 = (p3 & ~syn) | (n3 & syn);
  return dirty;
}

// ------------------------------------------------------------------ stages B and I
// What stage I leaves for the rest of the pass: the classes of this lane's word after its markings, and the run's group
// selection.
struct RunClass {
  uint32_t TERM, COMPL, RUNQ;
  uint32_t group;  // BF_GROUP_*
  uint32_t sum;    // BF_SUM_* bits (0 when the host sets the group)
  bool marked;     // a marking rewrote a code
};

// Stage B, classification (dag.go:3377-3388, 2020-2033), then stage I: fail-fast / compensation marking and group selection
// (dag.go:422-495), all per-run reductions in one sub-warp redux.or.  Host-group runs take part in every vote, never qualify
// for a marking, and get the host's group.
// SUM_FIRST orders two independent results and changes nothing else.  ptxas schedules the packed-lanes kernel differently
// with each order, and each build is fastest with its own (H100 SXM at 400 W, µs per pipelined pass in three rounds): with
// cond / decision codes, cfg4 took 56.1 - 56.3 group first and 55.0 - 55.2 summary first; without them, cfg3 took
// 49.6 - 49.7 group first and 50.3 - 50.9 summary first (the latter with a 4-byte spill).
template <bool SUM_FIRST>
DI RunClass stage_bi(uint32_t gmask, uint32_t rflags, uint32_t n_main, uint32_t n_comp, uint32_t n_final, uint32_t AF,
                     uint32_t GM, uint32_t G1, uint32_t G2, uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3) {
  bool marked = false;
  const bool fail_fast = rflags & BF_RF_FAIL_FAST;
  const bool realtime = rflags & BF_RF_REALTIME;
  const bool topo_term = rflags & BF_RF_TOPOLOGY_TERMINATED;
  const bool auto_group = !(rflags & BF_RF_HOST_GROUP);
  // stage B
  uint32_t TERM = plut<BF_LUT_TERMINAL>(p0, p1, p2, p3);
  uint32_t COMPL = plut<BF_LUT_COMPLETED0>(p0, p1, p2, p3) | (TERM & AF);
  uint32_t RUNQ = plut<BF_LUT_RUNNING_Q>(p0, p1, p2, p3);
  uint32_t FAILED = TERM & ~COMPL;
  // stage I
  uint32_t RUN = plut<BF_LUT_RUNNING>(p0, p1, p2, p3);
  const uint32_t DONE = COMPL | FAILED;
  const uint32_t mark_ff = GM & ~COMPL & ~RUNQ & ~TERM;           // markFailFastSkipped candidates (:3289-3312)
  const uint32_t mark_cs = G1 & ~COMPL & ~RUN & ~FAILED & ~TERM;   // markCompensationsSkipped candidates (:3314-3342)
  uint32_t bits = ((FAILED & GM) != 0 ? 1u : 0u)                   // any main failed
                  | ((GM & ~DONE) != 0 ? 2u : 0u)                  // main not done (no marking)
                  | ((GM & ~DONE & ~mark_ff) != 0 ? 4u : 0u)       // main not done even after fail-fast marking
                  | ((G1 & ~DONE) != 0 ? 8u : 0u)                  // comp not done (no marking)
                  | ((G1 & ~DONE & ~mark_cs) != 0 ? 16u : 0u)      // comp not done after comp-skip marking
                  | ((G2 & ~DONE) != 0 ? 32u : 0u)                 // finally not done
                  | ((FAILED & G1) != 0 ? 64u : 0u)
                  | ((FAILED & G2) != 0 ? 128u : 0u)
                  | (mark_ff != 0 ? 256u : 0u)
                  | (mark_cs != 0 ? 512u : 0u);
  bits = __reduce_or_sync(gmask, bits);
  bool amf = bits & 1u;
  const bool do_ff = auto_group && fail_fast && amf;
  if (do_ff) {
    marked = marked || (bits & 256u);
    pset<BF_PHASE_SKIPPED>(mark_ff, p0, p1, p2, p3);
    TERM |= mark_ff; COMPL |= mark_ff; RUN &= ~mark_ff;
  }
  bool main_done = n_main == 0 || !(bits & (do_ff ? 4u : 2u));
  const bool acf = bits & 64u;
  // dag.go:436-464 (rare)
  const bool tt = auto_group && !main_done && realtime && topo_term;
  if (__any_sync(FULL, tt)) {
    const uint32_t mtt = tt ? (GM & (p0 | p1 | p2 | p3) & ~TERM) : 0u;
    pset<BF_PHASE_FAILED>(mtt, p0, p1, p2, p3);
    TERM |= mtt; COMPL |= mtt & AF; FAILED |= mtt & ~AF; RUN &= ~mtt; RUNQ &= ~mtt;
    const uint32_t b2 = __reduce_or_sync(gmask, (mtt != 0 ? 1u : 0u) | ((FAILED & GM) != 0 ? 2u : 0u));
    if (tt) {
      marked = marked || (b2 & 1u);
      main_done = true;
      amf = b2 & 2u;
    }
  }
  bool comp_done;
  if (auto_group && main_done && !amf && n_comp != 0) {
    marked = marked || (bits & 512u);
    pset<BF_PHASE_SKIPPED>(mark_cs, p0, p1, p2, p3);
    TERM |= mark_cs; COMPL |= mark_cs;
    comp_done = !(bits & 16u);
  } else {
    comp_done = n_comp == 0 || !(bits & 8u);
  }
  const bool final_done = n_final == 0 || !(bits & 32u);
  const bool aff = bits & 128u;
  RunClass c{TERM, COMPL, RUNQ, BF_GROUP_DONE, 0u, marked};
  auto summary = [&]() {
    c.sum = (main_done ? BF_SUM_MAIN_DONE : 0u) | (amf ? BF_SUM_MAIN_FAILED : 0u) | (comp_done ? BF_SUM_COMP_DONE : 0u) |
            (final_done ? BF_SUM_FINAL_DONE : 0u) | (acf ? BF_SUM_COMP_FAILED : 0u) | (aff ? BF_SUM_FINAL_FAILED : 0u);
  };
  if (SUM_FIRST) summary();
  if (!main_done) c.group = BF_GROUP_MAIN;
  else if (amf && n_comp != 0 && !comp_done) c.group = BF_GROUP_COMPENSATION;
  else if (n_final != 0 && !final_done) c.group = BF_GROUP_FINALLY;
  if (!SUM_FIRST) summary();
  if (!auto_group) {
    c.group = (rflags >> BF_RF_HOST_GROUP_SHIFT) & 3u;
    c.sum = 0;
  }
  return c;
}

// ------------------------------------------------------------------ D-prep: dependency classes under the pass's policy
// dag.go:499-502.  A run whose group is DONE has no candidate.
struct DepClass {
  uint32_t U;      // not satisfied: status bit 0 (& VALID: the bytes past the last step read "satisfied")
  uint32_t FD;     // failed dependency under skip-on-failed: status bit 1
  uint32_t CAND;   // candidates whose rows are walked
  uint32_t FREE;   // candidates without needs: met by definition (byte-entry rows only)
  bool allow_failed, skip_on_failed;
};

DI DepClass stage_dprep(const RunClass& c, uint32_t rflags, uint32_t VALID, uint32_t GM, uint32_t G1, uint32_t G2,
                        uint32_t NODEP, uint32_t p0, uint32_t p1, uint32_t p2, uint32_t p3) {
  DepClass d;
  d.allow_failed = c.group != BF_GROUP_MAIN;
  d.skip_on_failed = c.group == BF_GROUP_MAIN && !(rflags & BF_RF_FAIL_FAST);
  const uint32_t GSEL = c.group == BF_GROUP_MAIN ? GM : (c.group == BF_GROUP_COMPENSATION ? G1 : G2);
  const uint32_t SAT = c.COMPL | ((rflags & BF_RF_REALTIME) ? plut<BF_LUT_RT_SAT>(p0, p1, p2, p3) : 0u) |
                       (d.allow_failed ? c.TERM : 0u);
  d.U = VALID & ~SAT;
  d.FD = d.skip_on_failed ? (c.TERM & ~SAT) : 0u;
  const uint32_t CAND0 = c.group != BF_GROUP_DONE ? (GSEL & ~c.COMPL & ~c.RUNQ & ~c.TERM) : 0u;
  d.FREE = CAND0 & NODEP;
  d.CAND = CAND0 & ~NODEP;
  return d;
}

// ------------------------------------------------------------------ cond masking and the in-loop FAIL fixed point
// dag.go:2741-2843.  A met step is ready (BF_COND_PASS), skipped (BF_COND_SKIP) or failed (BF_COND_FAIL) by its cond code
// (c0, c1); HOLD (c1 & ~c0) does nothing.  A step set Failed inside the loop is visible to LATER steps of the list only
// (dag.go:2745, :497): while the failures change, every candidate item is walked again with the failures so far, to the
// unique fixed point (one extra round per chained failure; at most round_cap + 1 rounds).  `fixup(L, candw, fclass, metb,
// fdb)` walks item L, whose CAND word candw lane L holds, against the fail words at mfail_a, a failed dependency reading as
// status byte fclass; `own` says this lane's fail word has a place there.  Sets the failed steps Failed (dag.go:2745-2747,
// 2810-2812) and returns whether the warp has any.
template <class Fixup>
DI bool stage_cond(uint32_t lane, uint32_t c0, uint32_t c1, const DepClass& d, uint32_t mfail_a, bool own, uint32_t round_cap,
                   Fixup fixup, uint32_t& met_w, uint32_t& fd_w, uint32_t& ready_w, uint32_t& skipc_w, uint32_t& fail_w,
                   uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3) {
  ready_w = met_w & ~c0 & ~c1;   // BF_COND_PASS
  skipc_w = met_w & c0 & ~c1;    // BF_COND_SKIP
  fail_w = met_w & c0 & c1;      // BF_COND_FAIL
  const bool any_fail = __any_sync(FULL, fail_w != 0);
  if (any_fail) {
    const uint32_t fclass = d.allow_failed ? 0u : (d.skip_on_failed ? 3u : 1u);
    for (uint32_t round = 0; round <= round_cap; ++round) {
      __syncwarp();
      if (own) sts_u32(mfail_a + lane * 4u, fail_w);
      __syncwarp();
      met_w = 0; fd_w = 0;
      for (uint32_t todo = __ballot_sync(FULL, d.CAND != 0); todo; todo &= todo - 1) {
        const uint32_t L = __ffs(todo) - 1;
        uint32_t mb, fb;
        fixup(L, __shfl_sync(FULL, d.CAND, L), __shfl_sync(FULL, fclass, L), mb, fb);
        if (lane == L) { met_w = mb; fd_w = fb; }
      }
      met_w |= d.FREE;
      const uint32_t nf = met_w & c0 & c1;
      const bool same = !__any_sync(FULL, nf != fail_w);
      fail_w = nf;
      if (same) break;
    }
    ready_w = met_w & ~c0 & ~c1;
    skipc_w = met_w & c0 & ~c1;
  }
  pset<BF_PHASE_FAILED>(fail_w, p0, p1, p2, p3);
  return any_fail;
}

// ------------------------------------------------------------------ stage E: the result words of word w
// Lanes with w < P.words write the masks the layout carries; then the lanes w = 0 .. wstride - 1 of the run zero the record's
// padding from result_tail to the stride.
template <bool XO>
DI void store_words(const KParams& P, uint8_t* rr, uint32_t w, uint32_t wstride, uint32_t ready, uint32_t skip, uint32_t fail,
                    uint32_t needs, uint32_t skipdep, uint32_t p0, uint32_t p1, uint32_t p2, uint32_t p3) {
  const uint32_t Wmax = P.words;
  if (w < Wmax) {
    reinterpret_cast<uint32_t*>(rr + P.off_ready)[w] = ready;
    reinterpret_cast<uint32_t*>(rr + P.off_skip)[w] = skip;
    if (XO) {
      if (P.off_fail != BF_OFF_NONE) reinterpret_cast<uint32_t*>(rr + P.off_fail)[w] = fail;
      if (P.off_needs_cond != BF_OFF_NONE) reinterpret_cast<uint32_t*>(rr + P.off_needs_cond)[w] = needs;
      if (P.off_skip_dep != BF_OFF_NONE) reinterpret_cast<uint32_t*>(rr + P.off_skip_dep)[w] = skipdep;
      if (P.off_phase_out != BF_OFF_NONE) {
        uint32_t* po = reinterpret_cast<uint32_t*>(rr + P.off_phase_out) + w;
        po[0] = p0; po[Wmax] = p1; po[2 * Wmax] = p2; po[3 * Wmax] = p3;
      }
    }
  }
  if (P.result_tail != P.result_stride)
    for (uint32_t x = P.result_tail / 4 + w; x < P.result_stride / 4; x += wstride) reinterpret_cast<uint32_t*>(rr)[x] = 0u;
}

// ------------------------------------------------------------------ host side: dispatch shared by the two launchers
typedef void (*KernelFn)(const KParams);

// Variant bits every kernel has: CD (cond and/or decision codes present) = 2, XO (any of fail / needs_cond / skip_dep /
// phase_out requested) = 1.
inline uint32_t variant_bits(const KParams& P) {
  const bool cd = P.off_cond != BF_OFF_NONE || P.off_decision != BF_OFF_NONE;
  const bool xo = P.off_fail != BF_OFF_NONE || P.off_needs_cond != BF_OFF_NONE || P.off_skip_dep != BF_OFF_NONE ||
                  P.off_phase_out != BF_OFF_NONE;
  return (cd ? 2u : 0u) | (xo ? 1u : 0u);
}

// Lets `fn` use the whole 227 KB of dynamic shared memory, once per (device, function).
inline cudaError_t allow_max_smem(KernelFn fn) {
  static KernelFn configured[8][64] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const bool cached = dev >= 0 && dev < 8;
  if (cached)
    for (int i = 0; i < 64; ++i)
      if (configured[dev][i] == fn) return cudaSuccess;
  e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (e == cudaSuccess && cached)
    for (int i = 0; i < 64; ++i)
      if (configured[dev][i] == nullptr) { configured[dev][i] = fn; break; }
  return e;
}

}  // namespace bf
