// frontier_kernel.cu — the StoryRun ready-frontier pass for sm_90a (H100).
//
// One WARP evaluates one StoryRun per trip of a persistent loop.  For every run two cp.async.bulk (TMA) copies —
// the run's dynamic state record and its Story topology record (CSR + bit-sliced static flags) — land in a
// per-warp, multi-stage shared-memory ring guarded by mbarriers; the copies of the next runs are in flight while
// the current one is evaluated, so HBM streams with no register staging.  The chain run -> slot id -> slot entry
// is prefetched for 32 runs at a time (one run per lane) and the lane that owns a run issues its copies.
//
// Evaluation is BIT-SLICED: the 4-bit phase codes of a run arrive as four bit planes (one u32 word = 32 steps),
// so every classification of buildStateMaps (dag.go:3358-3391), the gate/sleep/wait rewrite (dag.go:1455-1547),
// fail-fast / compensation marking and group selection (dag.go:422-511) are a handful of LOP3s per 32 steps,
// held by lanes 0..W-1, and the per-run reductions of group selection are ONE redux.or.  The dependency walk of
// findReadySteps (dag.go:2711-2733) then runs one step per lane over the CSR row in shared memory against a
// per-step status byte, several candidate words at a time (independent load chains), and __ballot_sync folds
// the 32 per-step verdicts of a word straight into one word of the ready / skip bit masks.
//
// All shared-memory traffic of the loop uses 32-bit shared-window addresses (ld.shared / st.shared through inline
// PTX).  The kernel is compiled in variants <CD, CH, FX, XO, LIST, RB> (cond/decision codes present, parallel
// steps present, device fixpoint, extra outputs, run-list tier, register budget of the build) so the common
// pass carries no dead work.  Integer only; no tensor cores.  ~3 KB in, 80 B out per run at the BASELINE
// configuration (measured rates: DESIGN.md section 5).  The bit-plane stages are shared with frontier_pack.cu (stages.cuh).
#include "stages.cuh"

namespace bf {

extern __shared__ __align__(128) uint8_t smem_raw[];

// CD: cond and/or decision codes present   CH: topologies with `parallel` steps may occur (stage H, expansion count)
// FX: device-side fixpoint (BF_EVAL_FIXPOINT)   XO: any of fail/needs_cond/skip_dep/phase_out requested
// LIST: second-tier run over P.run_list (runs deferred by the packed-lanes kernel)
// RB: register budget of the build, chosen by the host plan from what fits shared memory (the pass is bound by per-warp
//       instruction latency: resident warps first) —
//       0: one CTA of up to 16 warps per SM (<= 128 registers)
//       1: two resident CTAs of up to 16 warps (<= 64 registers)
//       2: one CTA of up to 24 warps (<= 80 registers)
template <bool CD, bool CH, bool FX, bool XO, bool LIST, int RB>
__global__ void __launch_bounds__(RB == 2 ? 768 : 512, RB == 1 ? 2 : 1) frontier_kernel(const KParams P) {
  const uint32_t lane = pin(threadIdx.x & 31u);  // pinned: otherwise rematerialised from S2R inside the loop
  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t ST = P.stages;

  // ---- shared memory carve-up ----
  unsigned long long* blk_counts = reinterpret_cast<unsigned long long*>(smem_raw);
  // [128 B counters][mbarriers: 64 B per warp][warp regions: ST stages of (state record | topology record), scratch].
  // The stages' mbarriers live in one block for the whole CTA, AWAY from the TMA destinations: a barrier placed
  // right behind a record's tail slowed the pass (A/B on one card).
  const uint32_t ring_bytes = ST * P.stage_bytes;
  const uint32_t per_warp = ring_bytes + P.work_bytes;
  uint8_t* const wbase = smem_raw + 128 + P.warps_per_block * 64u + warp * per_warp;
  const uint32_t wb = pin(smem_u32(wbase));  // pinned: otherwise rematerialised from S2R inside the loop
  const uint32_t bar_base = pin(smem_u32(smem_raw) + 128u + warp * 64u);

  if (threadIdx.x < 4) blk_counts[threadIdx.x] = 0ull;
  if (lane == 0) {
    for (uint32_t s = 0; s < ST; ++s) mbar_init(bar_base + 8 * s, 1);
    fence_barrier_init();
  }
  __syncthreads();

  const uint32_t gw = blockIdx.x * P.warps_per_block + warp;
  const uint32_t G = gridDim.x * P.warps_per_block;
  // run-list mode (second tier after the packed-lanes kernel): the runs to take are run_list[0..count)
  const uint32_t* const rlist = LIST ? P.run_list : nullptr;
  const uint32_t N = LIST ? min(*reinterpret_cast<const volatile uint32_t*>(P.run_list_count), P.n_runs) : P.n_runs;
  // This warp's n-th run is run (or list position) rbase + n * rstride: a contiguous block of the batch
  // (run_blocked) or every G-th run.
  uint32_t rbase, rstride, my_runs;
  if (P.run_blocked) {
    const uint32_t lo = (uint32_t)((uint64_t)N * gw / G), hi = (uint32_t)((uint64_t)N * (gw + 1) / G);
    rbase = lo; rstride = 1; my_runs = hi - lo;
  } else {
    rbase = gw; rstride = G; my_runs = gw < N ? (N - gw + G - 1) / G : 0;
  }
  auto run_of = [&](uint32_t n) -> uint32_t {  // global run index of this warp's n-th run
    const uint32_t idx = rbase + n * rstride;
    return LIST ? __ldg(rlist + idx) : idx;
  };

  // ---- producer: the warp prefetches slot ids and slot entries 32 runs at a time (lane l holds issue index
  //      32*b + l), so the chain run -> slot id -> slot entry -> TMA costs two coalesced loads per 32 runs and
  //      the lane that owns an index issues its copies from its own registers ----
  uint32_t ni = 0;                          // next issue index (lane-uniform)
  uint32_t nx_rid = 0, nx_sid = 0xFFFFFFFFu;  // lane l: run / slot id of index (next batch) + l
  uint32_t pf_rid = 0, pf_lo = 0, pf_hi = 0, pf_bytes = 0;  // lane l: run, record address, record bytes of index (this batch) + l
  auto load_sids = [&](uint32_t n0) {
    const uint32_t n = n0 + lane;
    nx_rid = 0; nx_sid = 0xFFFFFFFFu;
    if (n < my_runs) {
      nx_rid = run_of(n);
      nx_sid = __ldg(reinterpret_cast<const uint32_t*>(P.state + (size_t)nx_rid * P.state_stride));
    }
  };
  auto load_ents = [&]() {
    pf_rid = nx_rid; pf_lo = 0; pf_hi = 0; pf_bytes = 0;
    if (nx_sid < P.n_slots) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(P.slots + nx_sid));
      pf_lo = v.x; pf_hi = v.y; pf_bytes = v.z;
    }
  };
  // issue the copies of index ni into the stage at shared address `buf` guarded by mbarrier `bar`
  auto issue = [&](uint32_t buf, uint32_t bar) {
    if (lane == (ni & 31u) && ni < my_runs) {
      const bool ok = (pf_lo | pf_hi) != 0 && pf_bytes <= P.topo_buf_bytes;
      if (!ok) sts_zero16(buf + P.state_stride);  // dead / oversized slot: a zero header (W = 0) marks the stage
      mbar_expect_tx(bar, P.state_stride + (ok ? pf_bytes : 0u));
      bulk_g2s(buf, P.state + (size_t)pf_rid * P.state_stride, P.state_stride, bar);
      if (ok) bulk_g2s(buf + P.state_stride, reinterpret_cast<const void*>((uint64_t)pf_lo | ((uint64_t)pf_hi << 32)), pf_bytes, bar);
    }
    ++ni;
    if ((ni & 31u) == 16u) load_sids((ni & ~31u) + 32u);  // half a batch ahead
    if ((ni & 31u) == 0u) load_ents();                    // consumed from the next issue on
  };
  if (my_runs != 0) {
    load_sids(0);
    load_ents();
    for (uint32_t s = 0; s < ST; ++s) issue(wb + s * P.stage_bytes, bar_base + 8 * s);
  }

  // scratch (per warp): fix-up fail mask words, then one status byte per step (+16 guard bytes)
  // (all shared-memory traffic of the loop below goes through 32-bit shared-window addresses: no generic
  //  pointers, no cvta, no 64-bit address arithmetic)
  const uint32_t Wmax = P.words;
  const uint32_t mfail_a = wb + ring_bytes;
  const uint32_t st_a = mfail_a + ((4u * Wmax + 15u) & ~15u);

  const bool has_cond = CD && P.off_cond != BF_OFF_NONE;
  const bool has_dec = CD && P.off_decision != BF_OFF_NONE;
  const bool has_child = CH && P.off_child != BF_OFF_NONE;

  uint32_t tot_ready = 0, tot_skip = 0, tot_exp = 0, tot_evals = 0;  // lane-uniform
  uint32_t cs = 0, cpar = 0;                                         // consumer stage index / parity
  uint32_t stage_a = wb;                                             // shared address of the consumer stage
  const size_t result_step = (size_t)rstride * P.result_stride;
  uint8_t* rr_inc = P.result + (size_t)rbase * P.result_stride;
  uint32_t r_inc = rbase;

  for (uint32_t k = 0; k < my_runs; ++k, rr_inc += result_step, r_inc += rstride) {
    const uint32_t r = LIST ? run_of(k) : r_inc;
    uint8_t* const rr = LIST ? P.result + (size_t)r * P.result_stride : rr_inc;
    const uint32_t cur_stage = stage_a, cur_bar = bar_base + 8u * cs;
    mbar_wait(cur_bar, cpar);  // the stage index ni = k + ST will be copied into
    const uint32_t sr_a = cur_stage, tr_a = cur_stage + P.state_stride;  // state record / topology record
    stage_a += P.stage_bytes; ++cs;
    if (cs == ST) { cs = 0; stage_a = wb; cpar ^= 1u; }

    const uint4 h0 = lds_v4(tr_a);                               // TopoHeader, first half
    const uint32_t S = h0.x & 0xFFFFu, Wt = h0.x >> 16;          // S, W
    const uint32_t max_deg = h0.y & 0xFFFFu, nP = h0.y >> 16;    // max_deg, P
    const uint32_t n_main = h0.z & 0xFFFFu, n_comp = h0.z >> 16, n_final = h0.w & 0xFFFFu;
    if (Wt - 1u >= Wmax) {  // dead slot (zero header) / out-of-range record: empty result, summary all-ones
      for (uint32_t x = lane; x < P.result_stride / 4; x += 32) reinterpret_cast<uint32_t*>(rr)[x] = x == 0 ? 0xFFFFFFFFu : 0u;
      if (CH && P.exp_counts && lane == 0) P.exp_counts[r] = 0;
      __syncwarp();
      issue(cur_stage, cur_bar);
      continue;
    }
    const uint4 h1 = lds_v4(tr_a + 16);                          // off_col | ell << 16, off_planes, off_par, rec_bytes
    const uint32_t rflags = lds_u8(sr_a + 4);
    const uint32_t ell = h1.x >> 16;                             // 0 = CSR, 2 / 4 = fixed-width rows (device_record.h)
    const int fmt = fmt_of(ell, max_deg);

    // ---------------- planes of word `lane`: dynamic codes (state record) + static flags (topology) ----------------
    const bool act = lane < Wt;
    uint32_t t0 = 0, t1 = 0, t2 = 0, AF = 0, TS = 0, HASIF = 0, G1 = 0, G2 = 0, VALID = 0, NODEP = 0;
    uint32_t c0 = 0, c1 = 0, d0 = 0, d1 = 0;
    uint32_t p0 = 0, p1 = 0, p2 = 0, p3 = 0;
    if (act) {
      const uint32_t sp = tr_a + h1.y + lane * 4u, ps = Wt * 4u;  // static planes: word `lane`, plane stride
      if (CD || FX || CH) { t0 = lds_u32(sp + PL_T0 * ps); t1 = lds_u32(sp + PL_T1 * ps); t2 = lds_u32(sp + PL_T2 * ps); }
      AF = lds_u32(sp + PL_AF * ps);
      if (CD) TS = lds_u32(sp + PL_TS * ps);
      if (XO) HASIF = lds_u32(sp + PL_HASIF * ps);
      if (ell_has_nodep(ell)) NODEP = lds_u32(sp + PL_NODEP * ps);   // byte-entry rows: steps without needs stay out of the walk
      G1 = lds_u32(sp + PL_G1 * ps); G2 = lds_u32(sp + PL_G2 * ps);
      VALID = bmsk_clamp(0u, S - lane * 32u);  // the word's steps below S (width clamps at 32)
      const uint32_t pw = sr_a + P.off_phase + lane * 4u, ds = Wmax * 4u;  // dynamic planes: stride of the layout
      p0 = lds_u32(pw); p1 = lds_u32(pw + ds); p2 = lds_u32(pw + 2u * ds); p3 = lds_u32(pw + 3u * ds);
      const uint32_t keep = VALID & ~(p0 & p1 & p2 & p3);   // steps >= S and the reserved code 15 read as 0
      p0 &= keep; p1 &= keep; p2 &= keep; p3 &= keep;
      if (CD) {
        if (has_cond) { const uint32_t cw = sr_a + P.off_cond + lane * 4u; c0 = lds_u32(cw); c1 = lds_u32(cw + ds); }
        if (has_dec) { const uint32_t dw = sr_a + P.off_decision + lane * 4u; d0 = lds_u32(dw); d1 = lds_u32(dw + ds); }
      }
    }
    uint32_t gdirty = 0;  // steps whose code a stage-G rewrite really changed (for the "changed" flag; every other
                          // rewrite of the pass sets `marked` and always changes the code)
    const uint32_t GM = VALID & ~G1 & ~G2;
    const uint32_t SYNC_T = t0 & (t1 | t2);          // sleep(3) | wait(5) | gate(7)
    const uint32_t T_COND = t0 & ~t1 & ~t2;          // 1
    const uint32_t T_PAR = ~t0 & t1 & ~t2 & VALID;   // 2
    const uint32_t T_STOP = ~t0 & ~t1 & t2 & VALID;  // 4

    const bool realtime = rflags & BF_RF_REALTIME;

    uint32_t acc_ready = 0, acc_skip = 0, acc_fail = 0, acc_needs = 0, acc_skipdep = 0;
    uint32_t summary = 0, iters = 0;
    bool marked = false;  // some phase was rewritten (lane-uniform)
    const uint32_t cap = FX ? (P.max_iter ? P.max_iter : S + 1) : 1u;
    const uint32_t col_a = tr_a + (h1.x & 0xFFFFu);   // col_idx / the fixed-width block
    // row_ptr u16[S+1] (CSR); the walks' row_ptr argument carries the high-byte array of a 10-bit block instead
    const uint32_t rp_a = (ell & ELL_PACK10) ? col_a + 128u * Wt : tr_a + (uint32_t)sizeof(TopoHeader);
    if (ell && lane == 0) sts_u32(st_a + 32u * Wt, 0u);  // status byte PAD = 32*W: what unused row entries point at

    for (uint32_t it = 0; it < cap; ++it) {
      ++iters;
      // ---------------- stage H: parallel join (dag.go:1131-1198) ----------------
      // A registered parallel step that is neither absent nor terminal joins when every child is terminal: Failed if a
      // terminal child neither succeeded / was skipped nor is an allowFailure branch, else Succeeded.  Child phases are
      // nibbles, eight per word: one lane classifies eight children with the bit-plane tables (SWAR), a sub-warp of SW
      // lanes covers one descriptor, 32 / SW descriptors per round, and the verdicts reach the lanes that own the parents'
      // words through two scratch words per step word (the status-byte area is not in use yet at this point).
      if (CH && has_child && nP != 0) {
        const uint32_t ACTIVE = T_PAR & (p0 | p1 | p2 | p3) & ~plut<BF_LUT_TERMINAL>(p0, p1, p2, p3);
        if (__any_sync(FULL, ACTIVE != 0)) {
          const uint32_t pd_a = tr_a + h1.z, child_a = sr_a + P.off_child;
          // which descriptors join at all: registered, with children, parent neither absent nor terminal (lane q <-> desc q,
          // second round for descs 32..63), and the widest of them — usually none or a few of the run's descriptors
          uint32_t take_lo = 0, take_hi = 0, mb = 0;
          for (uint32_t q0 = 0; q0 < nP; q0 += 32) {
            const uint32_t q = q0 + lane;
            const uint32_t sb = q < nP ? lds_u32(pd_a + q * 16u) : 0u;   // step | branches << 16
            const uint32_t actw = __shfl_sync(FULL, ACTIVE, ((sb & 0xFFFFu) >> 5) & 31u);
            const uint32_t reg = lds_u32(sr_a + 8u + (q0 >> 3));          // children_registered, 32 descs per word
            const bool tk = q < nP && (sb >> 16) != 0u && ((reg >> lane) & 1u) != 0u && ((actw >> (sb & 31u)) & 1u) != 0u;
            const uint32_t m = __ballot_sync(FULL, tk);
            if (q0 == 0) take_lo = m; else take_hi = m;
            if (tk) mb = max(mb, sb >> 16);
          }
          mb = __reduce_max_sync(FULL, mb);
          const uint32_t mw = (mb + 7u) >> 3;   // child words of the widest joining descriptor
          if ((take_lo | take_hi) == 0u) {
            // nothing to join in this pass
          } else if (mw <= 32u) {
            const uint32_t lgs = mw > 1u ? 32u - (uint32_t)__clz(mw - 1u) : 0u;   // sub-warp of SW = 2^lgs >= mw lanes per descriptor
            const uint32_t SW = 1u << lgs, DPI = 32u >> lgs, sub = lane >> lgs, wi = lane & (SW - 1u);
            const uint32_t gm = (SW == 32u ? FULL : ((1u << SW) - 1u)) << (sub << lgs);
            const uint32_t dmask = DPI == 32u ? FULL : ((1u << DPI) - 1u);
            const uint32_t tS = st_a, tF = st_a + 4u * Wt;
            __syncwarp();
            if (act) { sts_u32(tS + lane * 4u, 0u); sts_u32(tF + lane * 4u, 0u); }
            __syncwarp();
            for (uint32_t q0 = 0; q0 < nP; q0 += DPI) {
              const uint32_t tw = q0 < 32u ? take_lo >> q0 : take_hi >> (q0 - 32u);   // DPI divides 32: a round never straddles the words
              if ((tw & dmask) == 0u) continue;                                       // warp-uniform
              const uint32_t q = q0 + sub;
              const bool take = (tw >> sub) & 1u;
              uint4 d = make_uint4(0u, 0u, 0u, 0u);
              if (take) d = lds_v4(pd_a + q * 16u);          // step | branches << 16, child_first, allow_off, -
              const uint32_t step = d.x & 0xFFFFu, br = d.x >> 16, wj = step >> 5, wb = step & 31u;
              bool nd = false, fl = false;
              if (take && wi * 8u < br) {
                const uint32_t cw = lds_u32(child_a + (d.y >> 1) + wi * 4u);   // child_first is a multiple of 8 nibbles
                const uint32_t vm = 0x11111111u & bmsk_clamp(0u, min(8u, br - wi * 8u) * 4u);
                uint32_t x0 = cw & 0x11111111u, x1 = (cw >> 1) & 0x11111111u, x2 = (cw >> 2) & 0x11111111u, x3 = (cw >> 3) & 0x11111111u;
                const uint32_t keep = ~(x0 & x1 & x2 & x3);                     // the reserved code 15 reads as 0
                x0 &= keep; x1 &= keep; x2 &= keep; x3 &= keep;
                const uint32_t done = plut<BF_LUT_TERMINAL>(x0, x1, x2, x3);
                const uint32_t ab = (lds_u32(tr_a + d.z + (wi >> 2) * 4u) >> ((wi & 3u) * 8u)) & 0xFFu;   // allowFailure bits of my 8 branches
                const uint32_t okc = plut<BF_LUT_COMPLETED0>(x0, x1, x2, x3) | spread4(ab);
                nd = (vm & ~done) != 0u;
                fl = (vm & done & ~okc) != 0u;
              }
              const uint32_t ndm = __ballot_sync(FULL, nd), flm = __ballot_sync(FULL, fl);
              if (take && wi == 0u && (ndm & gm) == 0u) red_or_shared(((flm & gm) ? tF : tS) + wj * 4u, 1u << wb);
            }
            __syncwarp();
            uint32_t sS = 0, sF = 0;
            if (act) { sS = lds_u32(tS + lane * 4u); sF = lds_u32(tF + lane * 4u); }
            if (__any_sync(FULL, (sS | sF) != 0u)) marked = true;
            pset<BF_PHASE_SUCCEEDED>(sS, p0, p1, p2, p3);
            pset<BF_PHASE_FAILED>(sF, p0, p1, p2, p3);
            __syncwarp();
          } else {   // more than 256 branches on one step: one descriptor at a time, one child per lane
            const uint8_t* sr = gptr(sr_a);
            const uint8_t* tr = gptr(tr_a);
            const uint64_t registered = *reinterpret_cast<const uint64_t*>(sr + 8);
            const ParDesc* pd = reinterpret_cast<const ParDesc*>(tr + h1.z);
            const uint8_t* child = sr + P.off_child;
            for (uint32_t q = 0; q < nP; ++q) {
              if (!((registered >> q) & 1ull)) continue;
              const ParDesc d = pd[q];
              if (d.branches == 0) continue;  // no children to wait for (dag.go:1140-1143)
              const uint32_t wj = d.step >> 5, wb = d.step & 31u;
              if (!((__shfl_sync(FULL, ACTIVE, wj) >> wb) & 1u)) continue;
              const uint32_t* allow = reinterpret_cast<const uint32_t*>(tr + d.allow_off);
              bool all_done = true, any_failed = false;
              for (uint32_t b = lane; b < d.branches; b += 32) {
                const uint32_t cph = get_nibble(child, d.child_first + b);
                const bool done = cph != 0 && ((BF_LUT_TERMINAL >> cph) & 1u);
                const bool okc = cph == BF_PHASE_SUCCEEDED || cph == BF_PHASE_SKIPPED || ((allow[b >> 5] >> (b & 31u)) & 1u);
                all_done = all_done && done;
                any_failed = any_failed || (done && !okc);
              }
              all_done = __all_sync(FULL, all_done);
              any_failed = __any_sync(FULL, any_failed);
              if (all_done) {
                marked = true;
                if (lane == wj) {  // the lane that owns word wj rewrites its planes
                  const uint32_t m = 1u << wb;
                  if (any_failed) pset<BF_PHASE_FAILED>(m, p0, p1, p2, p3); else pset<BF_PHASE_SUCCEEDED>(m, p0, p1, p2, p3);
                }
              }
            }
          }
        }
      }

      // ---------------- stages G, B, I and D-prep (stages.cuh) ----------------
      if (has_dec) gdirty |= stage_g(SYNC_T, TS, d0, d1, p0, p1, p2, p3);
      const RunClass rc = stage_bi<CD>(FULL, rflags, n_main, n_comp, n_final, AF, GM, G1, G2, p0, p1, p2, p3);
      marked = marked || rc.marked;
      summary = rc.sum | rc.group;

      uint32_t it_ready = 0, it_skip = 0, it_fail = 0;
      if (rc.group != BF_GROUP_DONE) {
        const DepClass dc = stage_dprep(rc, rflags, VALID, GM, G1, G2, NODEP, p0, p1, p2, p3);
        const bool skip_on_failed = dc.skip_on_failed;
        const uint32_t U = dc.U, FD = dc.FD, CAND = dc.CAND;
        // ------------- stage C: masks -> one status byte per step (bit0 unmet, bit1 failed-dep) -------------
        __syncwarp();
        uint32_t m0 = 0;
#pragma unroll 1
        do {  // uniform trip count (one trip per 256 steps): every lane takes part in the shuffles
          const uint32_t m = m0 + lane;
          const uint32_t src = (m >> 2) & 31u, sh = (m & 3u) * 8u;
          const uint32_t ub = __shfl_sync(FULL, U, src) >> sh;
          uint2 v;
          v.x = bits4_to_bytes(ub & 0xFu);
          v.y = bits4_to_bytes((ub >> 4) & 0xFu);
          if (skip_on_failed) {  // lane-uniform: FD is empty under every other policy
            const uint32_t fb = __shfl_sync(FULL, FD, src) >> sh;
            v.x |= bits4_to_bytes(fb & 0xFu) << 1;
            v.y |= bits4_to_bytes((fb >> 4) & 0xFu) << 1;
          }
          if (m < 4 * Wt) sts_v2(st_a + m * 8u, v.x, v.y);
          m0 += 32;
        } while (m0 < 4 * Wt);
        __syncwarp();
        // ------------- stage D: walk the needs rows (dag.go:2711-2733) -------------
        uint32_t met_w, fd_w;
        // candidate words per walk group (walk_words, kernel_common.cuh): 2 at two CTAs per SM, 4 where one CTA per
        // SM leaves little else to hide latency
        constexpr int WK = RB == 1 ? 2 : 4;
        if (skip_on_failed) walk_words_fmt<WK, true>(fmt, lane, CAND, rp_a, col_a, st_a, met_w, fd_w);  // warp-uniform dispatch
        else walk_words_fmt<WK, false>(fmt, lane, CAND, rp_a, col_a, st_a, met_w, fd_w);
        met_w |= dc.FREE;
        uint32_t ready_w = met_w, skipc_w = 0, fail_w = 0;
        if (CD) {
          // item j: word j of the run; the scratch holds fail words for the run's words only (the lanes of `act`)
          auto fixup = [&](uint32_t j, uint32_t candw, uint32_t fclass, uint32_t& mb, uint32_t& fb) {
            fixup_item(lane, candw, j, ell, rp_a, col_a, [&](uint32_t d) { return lds_u8(st_a + d); }, mfail_a, fclass, mb, fb);
          };
          if (stage_cond(lane, c0, c1, dc, mfail_a, act, S, fixup, met_w, fd_w, ready_w, skipc_w, fail_w, p0, p1, p2, p3)) marked = true;
        }
        it_ready = ready_w;
        it_skip = fd_w | skipc_w;
        it_fail = fail_w;
        if (XO) {
          acc_needs |= realtime ? 0u : (met_w & HASIF);
          acc_skipdep |= fd_w;
        }
      }
      acc_ready |= it_ready; acc_skip |= it_skip; acc_fail |= it_fail;

      if (!FX) break;
      if (rc.group == BF_GROUP_DONE) break;
      // ------------- launch effects (dag.go:1735-1775, step_executor.go:132-185) -------------
      const uint32_t o0 = p0, o1 = p1, o2 = p2, o3 = p3;
      launch_effects(it_skip, it_ready, T_COND, SYNC_T, T_PAR, T_STOP, p0, p1, p2, p3);
      const uint32_t fl = redux_or(((it_ready | it_skip) != 0 ? 1u : 0u) | ((it_ready & T_STOP) != 0 ? 2u : 0u) |
                                   (((p0 ^ o0) | (p1 ^ o1) | (p2 ^ o2) | (p3 ^ o3)) != 0 ? 4u : 0u));
      marked = marked || (fl & 4u);
      if ((fl & 3u) != 1u) break;  // no progress, or a ready `stop` step hands the run to the host
    }

    // ---------------- stage E: result record ----------------
    const uint32_t n_rs = redux_add((uint32_t)__popc(acc_ready) | ((uint32_t)__popc(acc_skip) << 16));  // both <= S <= 1024
    const uint32_t n_ready = n_rs & 0xFFFFu, n_skip = n_rs >> 16;
    uint32_t n_exp = 0;
    if (CH && nP != 0) {
      const ParDesc* pd = reinterpret_cast<const ParDesc*>(gptr(tr_a + h1.z));
      uint32_t mine = 0;
      for (uint32_t q0i = 0; q0i < nP; q0i += 32) {  // uniform trip count (shuffles inside)
        const uint32_t q = q0i + lane;
        const uint32_t stp = q < nP ? pd[q].step : 0u;
        const uint32_t w = __shfl_sync(FULL, acc_ready, stp >> 5);
        if (q < nP && ((w >> (stp & 31u)) & 1u)) mine += pd[q].branches;
      }
      n_exp = redux_add(mine);
    }
    // G rewrites (decision codes) may write the code a step already has: `gdirty` holds the ones that really changed
    bool changed = marked;
    if (CD) changed = __any_sync(FULL, gdirty != 0) || marked;
    summary |= (changed ? BF_SUM_PHASE_CHANGED : 0u) | (iters << BF_SUM_ITER_SHIFT);
    if (lane == 0) {
      *reinterpret_cast<uint4*>(rr) = make_uint4(summary, n_ready, n_skip, n_exp);
      if (CH && P.exp_counts) P.exp_counts[r] = n_exp;
    }
    store_words<XO>(P, rr, lane, 32u, acc_ready, acc_skip, acc_fail, acc_needs, acc_skipdep, p0, p1, p2, p3);
    tot_ready += n_ready; tot_skip += n_skip; tot_exp += n_exp; tot_evals += S;

    __syncwarp();  // every lane is done with this stage's buffers
    issue(cur_stage, cur_bar);
  }

  // ---- counters: warp -> block (shared atomics) -> one global atomic per block ----
  if (P.counts) {
    if (lane == 0 && my_runs != 0) {
      atomicAdd(&blk_counts[0], (unsigned long long)tot_ready);
      atomicAdd(&blk_counts[1], (unsigned long long)tot_skip);
      atomicAdd(&blk_counts[2], (unsigned long long)tot_exp);
      atomicAdd(&blk_counts[3], (unsigned long long)tot_evals);
    }
    __syncthreads();
    if (threadIdx.x < 4 && blk_counts[threadIdx.x] != 0ull) atomicAdd(&P.counts[threadIdx.x], blk_counts[threadIdx.x]);
  }
}

// ------------------------------------------------------------------ host-side dispatch
// index: variant_bits (CD, XO) | CH << 2 | FX << 3; the fixpoint variants exist as RB = 0 only
template <int RB>
static KernelFn pick_kernel(uint32_t v) {
  static const KernelFn table[16] = {
      frontier_kernel<false, false, false, false, false, RB>, frontier_kernel<false, false, false, true, false, RB>,
      frontier_kernel<true, false, false, false, false, RB>,  frontier_kernel<true, false, false, true, false, RB>,
      frontier_kernel<false, true, false, false, false, RB>,  frontier_kernel<false, true, false, true, false, RB>,
      frontier_kernel<true, true, false, false, false, RB>,   frontier_kernel<true, true, false, true, false, RB>,
      frontier_kernel<false, false, true, false, false, 0>,   frontier_kernel<false, false, true, true, false, 0>,
      frontier_kernel<true, false, true, false, false, 0>,    frontier_kernel<true, false, true, true, false, 0>,
      frontier_kernel<false, true, true, false, false, 0>,    frontier_kernel<false, true, true, true, false, 0>,
      frontier_kernel<true, true, true, false, false, 0>,     frontier_kernel<true, true, true, true, false, 0>,
  };
  return table[v];
}

// rb: the build (template parameter RB)
static KernelFn kernel_for(const KParams& P, uint32_t rb) {
  uint32_t v = variant_bits(P);
  v |= (P.any_parallel != 0 ? 4u : 0u)            // CH: the join needs the child area; the expansion count needs only the descs
       | ((P.flags & BF_EVAL_FIXPOINT) ? 8u : 0u);  // FX
  if (P.run_list) {
    // Run lists reach this kernel in two ways, both planned as the 16-warp build (RB = 0, plan_general in abi.cu):
    //  - the second tier of a two-tier pass, after the packed-lanes kernel: a single pass (FX = 0) of a batch with some
    //    topology that has parallel steps (CH = 1) — indices 4-7;
    //  - a touched tick (bf_resident_tick_touched) that the packed-lanes kernel cannot take: S > 512, the device fixpoint or
    //    BF_KERNEL=general, with or without parallel topologies — every index.
    static const KernelFn list_table[16] = {
        frontier_kernel<false, false, false, false, true, 0>, frontier_kernel<false, false, false, true, true, 0>,
        frontier_kernel<true, false, false, false, true, 0>,  frontier_kernel<true, false, false, true, true, 0>,
        frontier_kernel<false, true, false, false, true, 0>,  frontier_kernel<false, true, false, true, true, 0>,
        frontier_kernel<true, true, false, false, true, 0>,   frontier_kernel<true, true, false, true, true, 0>,
        frontier_kernel<false, false, true, false, true, 0>,  frontier_kernel<false, false, true, true, true, 0>,
        frontier_kernel<true, false, true, false, true, 0>,   frontier_kernel<true, false, true, true, true, 0>,
        frontier_kernel<false, true, true, false, true, 0>,   frontier_kernel<false, true, true, true, true, 0>,
        frontier_kernel<true, true, true, false, true, 0>,    frontier_kernel<true, true, true, true, true, 0>};
    return list_table[v];
  }
  return rb == 2 ? pick_kernel<2>(v) : rb == 1 ? pick_kernel<1>(v) : pick_kernel<0>(v);
}

cudaError_t launch_frontier(const KParams& P, uint32_t grid, uint32_t smem_bytes, cudaStream_t stream) {
  const KernelFn fn = kernel_for(P, P.occ2);
  const cudaError_t e = allow_max_smem(fn);
  if (e != cudaSuccess) return e;
  fn<<<grid, P.warps_per_block * 32, smem_bytes, stream>>>(P);
  return cudaGetLastError();
}

// Resident CTAs per SM for this launch shape; *occ2 says which build to launch (the 64-register one when two
// CTAs fit in shared memory, else the unconstrained one).
int frontier_max_blocks_per_sm(const KParams& P, uint32_t threads, uint32_t smem_bytes, uint32_t* occ2) {
  int n = 0;
  *occ2 = 0;
  if (threads > 512) {   // more than 16 warps per CTA: the 80-register build, one CTA per SM (no fixpoint variants)
    if (P.flags & BF_EVAL_FIXPOINT) return 0;
    KernelFn fn3 = kernel_for(P, 2);
    allow_max_smem(fn3);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn3, (int)threads, smem_bytes) != cudaSuccess || n < 1) return 0;
    *occ2 = 2;
    return 1;
  }
  KernelFn fn2 = kernel_for(P, 1);
  allow_max_smem(fn2);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn2, (int)threads, smem_bytes) == cudaSuccess && n >= 2) {
    *occ2 = 1;
    return n;
  }
  KernelFn fn = kernel_for(P, 0);
  allow_max_smem(fn);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, (int)threads, smem_bytes) != cudaSuccess) return 1;
  return n;
}

}  // namespace bf
