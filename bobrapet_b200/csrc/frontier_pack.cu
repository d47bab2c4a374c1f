// frontier_pack.cu — packed-lanes frontier pass: one warp evaluates a GROUP of R = 32 / Wq StoryRuns per trip
// (Wq = words per run rounded up to a power of two; R = 4 at S = 256, 16 at S = 64).  It is the default kernel of
// single-pass batches whose runs have at most 512 steps; frontier_kernel.cu (one run per warp) covers S > 512,
// the device fixpoint and, as a second tier, the runs whose topology has `parallel` steps.
//
// Why: at S = 256 the one-run-per-warp kernel spends most of its warp instructions per run on per-word work that
// keeps 8 of 32 lanes busy.
// Here lane l = g * Wq + w holds word w (32 steps) of run g of the group, so every bit-plane stage (gate / sleep /
// wait rewrite dag.go:1455-1547, buildStateMaps :3358-3391, fail-fast / compensation marking and group selection
// :422-511, cond masking :2741-2843, result words) runs on all 32 lanes and its instructions are shared by R runs;
// per-run reductions are ballots masked to the run's lanes and segmented butterflies of full-mask shuffles (seg_or / seg_add,
// kernel_common.cuh), so the warp stays converged: a sub-warp __reduce_*_sync took a divergent fallback, once per run, on every
// trip.  Only the dependency walk (dag.go:2711-2733, one step per lane
// over a `needs` row) stays per (run, word).
//
// Data movement: the CTA (one per SM, persistent) owns a ring of NG slot groups in shared memory, each holding the R
// state records (adjacent in HBM: ONE bulk copy) and R topology records (one bulk copy each) of a group, guarded by
// one mbarrier per slot group.  The ring is shared by all warps of the CTA: groups are consumed in ticket order (a free
// warp draws the CTA's next group from a shared counter), and the warp that finishes group t re-arms the slot group it
// just read with the copies of group t + NG, which whichever warp draws that ticket will consume — so the number of
// groups in flight adapts by itself (a warp waiting at a barrier IS a group in flight), and a CTA keeps 24 warps fed
// from 33 slot groups where a private double-buffered ring per warp would allow only 16 warps.  The chain run ->
// slot id -> slot entry of group t + NG is fetched by the R lanes that own its runs while the warp works on group t
// (first link before the barrier wait, second after it), and those lanes issue the copies from their own registers.
// A dead / oversized slot is marked by a zero header written before the arrive, a run deferred to the general kernel by
// an all-ones header word.  A record with fixed-width rows arrives as two copies, its header and the part from the rows of
// the run's first word that can hold a candidate step on (the cut, at issue() below): finished prefixes are not moved.
//
// Start-up and tail: a cold CTA needs three dependent DRAM round trips (slot id, slot entry, bulk copy; tools/trace_probe.py
// shows them) before its first group can be evaluated, and the CTAs of a grid do not finish together.
// BF_EVAL_PIPELINED (a caller's promise that consecutive passes are independent) launches the pass as a
// programmatic dependent of the preceding kernel: its CTAs take the SMs that kernel has already left, so start-up,
// launch gap and tail overlap; griddepcontrol.wait sits in front of the counters.
//
// All shared-memory traffic goes through 32-bit shared-window addresses.  Integer only; no tensor cores.
#include "stages.cuh"

namespace bf {

extern __shared__ __align__(128) uint8_t smem_p[];

#ifndef WALK_K
#define WALK_K 4   // (run, word) items walked at once: independent load chains per warp (H100 SXM at 400 W, cfg3, us per
#endif             // pipelined pass in two rounds: 2: 58.4 / 57.7, 3: 58.4 / 58.0, 4: 57.8 / 58.6 — within the spread)
#ifndef PACK_MAX_WARPS
#define PACK_MAX_WARPS 24   // warps per CTA the kernel is compiled for (registers: 65536 / (32 * PACK_MAX_WARPS) per thread = 80).
#endif                      // H100 SXM at 400 W, cfg3, us per pipelined pass in two rounds: 16: 59.8 / 62.0, 20: 58.1 / 58.5,
                            // 24: 57.8 / 58.6, 28: 58.0 / 57.4 (spills at 72 registers), 32: 65.9 / 66.0

#ifdef PACK_TRACE   // timeline probe (tools/trace_probe.py, lib_ab builds only): per launch and CTA {start, first group landed, last group done, end}
__device__ unsigned long long g_trace[8][160][4];
__device__ unsigned int g_launch;
DI unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#endif
#ifdef PACK_STAGES  // stage probe (tools/stage_probe.py, lib_ab builds only): SM cycles per region of a group trip, summed over all warps:
// 0 ticket + barrier wait, 1 planes + stages G / B / I / D-prep, 2 stage C, 3 walk (with the second link's load issue),
// 4 load_cut + cond fix-up + stage E, 5 issue; 6 counts trips.  Lane i accumulates region i (one register).
__device__ unsigned long long g_stages[8];
#define PROBE(i) do { const uint32_t t_ = (uint32_t)clock(); pr_acc += lane == (i) ? t_ - pr_t : 0u; pr_t = t_; } while (0)
#else
#define PROBE(i) do { } while (0)
#endif

// ---- status of the steps of a group: bit words, not bytes.
// Stage C stores each lane's U (not satisfied) and FD (failed dependency) words once per trip, interleaved by half words into
// a pair of 32-bit status words, one per 16 steps: the word of steps 0 - 15 holds U in its low half and FD in its high half,
// the word of steps 16 - 31 FD in its low half and U in its high half.  Rotated right by d & 31 (shf.r.wrap takes the low 5
// bits of d by itself), the status word of step d has d's U bit at bit 0 and its FD bit at bit 16 in either half, so one 32-bit
// load serves both tests.  Word pair w of run g lies at st0 + g * 16 Wq + 8 w: a run's pairs start on a 16 Wq-byte boundary
// and pairs Wq .. 2 Wq - 1 stay zero, so dependency d's status word is at base | ((d >> 2) & ~3) (a shift and one LOP3).
// The PAD entry of u16 fixed-width rows (d = 32 W, device_record.h) reads pair W: a lane of the run with w >= W (U = FD = 0),
// or for W = Wq the zero pair behind the run's words — "satisfied".  All lanes of one item read the status of the same run,
// at most 2 Wq distinct words in 8 Wq contiguous bytes: broadcast loads without bank conflicts.
constexpr uint32_t ST_BYTES = 512;   // status of the R runs of a group: R * 16 * Wq = 512 bytes at every Wq
constexpr uint32_t ST_U = 1u, ST_FD = 1u << 16;   // the bits of a rotated status word (dep_status)

// dependency d of the run whose status starts at st, rotated: bit 0 not satisfied, bit 16 failed dependency, the other bits
// without meaning.  Only the low 5 bits of d and the bits `off_mask` keeps of d >> 2 are read.
DI uint32_t dep_status(uint32_t st, uint32_t d, uint32_t off_mask) {
  const uint32_t v = lds_u32(st | ((d >> 2) & off_mask));
  return __funnelshift_r(v, v, d);
}

// phase 3 of an item (phases 1 and 2: row_locate / row_fetch, kernel_common.cuh): OR of the rotated status words of the row's
// dependencies (CSR: masked by the row length)
template <int FMT>
DI uint32_t row_status_bits(uint32_t p, uint32_t n, const uint32_t (&x)[4], uint32_t st) {
  constexpr int E = (FMT == FMT_ELL2 || FMT == FMT_ELL2B) ? 2 : 4;
  uint32_t s[E], r = 0;
#pragma unroll
  for (int e = 0; e < E; ++e) s[e] = dep_status(st, x[e], ~3u);
#pragma unroll
  for (int e = 0; e < E; ++e) r |= (fmt_traits<FMT>::fixed || (uint32_t)e < n) ? s[e] : 0u;
  if (FMT == FMT_CSRL)
    for (uint32_t q = 4; q < n; ++q) r |= dep_status(st, lds_u16(p + q * 2u), ~3u);
  return r;
}

// ---- stage D over the (run, word) items of a group.
// Where the rows and status pairs of run g live: CSR formats read the per-run table {col_a, rp_a, st_a, max_deg | ell << 16}
// written in stage C; fixed-width rows always start 32 bytes into the run's topology buffer, so their addresses are
// computed (two multiply-adds, no dependent shared-memory load in front of the row fetch).
struct WalkCtx {
  uint32_t tab_a;      // per-run table (16 B entries)
  uint32_t col0;       // fixed-width formats: col_idx of run 0 of the group (topology buffer 0 + 32)
  uint32_t topo_buf;   // bytes between the topology buffers of consecutive runs
  uint32_t st0;        // status pairs of run 0
  uint32_t st_run;     // bytes between the status of consecutive runs (16 * Wq)
};

// K items at once (independent load chains); FMT as in kernel_common.cuh — the caller guarantees that every live run
// of the group has this row format (else it takes walk_items_any).
// AL (byte-entry rows of four, 8 words per run): the row word shifted right by 8 e is entry e as far as dep_status reads it
// (its low 5 bits, and bits 4 .. 7 through the offset mask 0x3C), so no entry is extracted.
// Fixed-width rows exist for every step of a word, so all 32 lanes fetch and the candidate word (the same in every lane
// after the shuffle) masks the ballot instead of every lane's predicate.
template <int K, int FMT, bool NEED_FD, bool AL = false>
DI void walk_items_k(uint32_t lane, uint32_t CAND, uint32_t& todo, uint32_t lg, const WalkCtx& C, uint32_t& met_w, uint32_t& fd_w) {
  const uint32_t wmask = (1u << lg) - 1u;
  uint32_t L[K], p[K], n[K], wv[K], st[K], cw[K], x[K][4];
  bool c[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    L[k] = __ffs(todo) - 1;
    todo &= todo - 1;
  }
  if (AL && FMT == FMT_ELL4B) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      cw[k] = __shfl_sync(FULL, CAND, L[k]);
      const uint32_t g = L[k] >> 3, i = (L[k] & 7u) * 32u + lane;
      st[k] = C.st0 + g * 128u;
      p[k] = C.col0 + g * C.topo_buf + i * 4u;
    }
#pragma unroll
    for (int k = 0; k < K; ++k) n[k] = lds_u32(p[k]);   // the row: four byte entries
#pragma unroll
    for (int k = 0; k < K; ++k)
      wv[k] = dep_status(st[k], n[k], 0x3Cu) | dep_status(st[k], n[k] >> 8, 0x3Cu) | dep_status(st[k], n[k] >> 16, 0x3Cu) |
              dep_status(st[k], n[k] >> 24, 0x3Cu);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const uint32_t m = __ballot_sync(FULL, (wv[k] & ST_U) == 0) & cw[k];
      if (lane == L[k]) met_w = m;
      if (NEED_FD) {
        const uint32_t f = __ballot_sync(FULL, (wv[k] & ST_FD) != 0) & cw[k];
        if (lane == L[k]) fd_w = f;
      }
    }
    return;
  }
#pragma unroll
  for (int k = 0; k < K; ++k) {
    cw[k] = __shfl_sync(FULL, CAND, L[k]);
    const uint32_t g = L[k] >> lg, i = (L[k] & wmask) * 32u + lane;
    c[k] = (cw[k] >> lane) & 1u;
    if (fmt_traits<FMT>::fixed) {
      st[k] = C.st0 + g * C.st_run;
      p[k] = C.col0 + g * C.topo_buf + i * fmt_traits<FMT>::row_bytes;   // rows exist for every step of the word (device_record.h)
      n[k] = (uint32_t)(FMT & 0xFF);
    } else {
      const uint4 t = lds_v4(C.tab_a + g * 16u);
      st[k] = t.z;
      row_locate<FMT>(c[k], i, t.y, t.x, p[k], n[k]);
    }
  }
#pragma unroll
  for (int k = 0; k < K; ++k) row_fetch<FMT>(p[k], n[k], x[k]);
#pragma unroll
  for (int k = 0; k < K; ++k) wv[k] = row_status_bits<FMT>(p[k], n[k], x[k], st[k]);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    if (fmt_traits<FMT>::fixed) {   // every lane holds a real row: mask the ballot with the (lane-uniform) candidate word
      const uint32_t m = __ballot_sync(FULL, (wv[k] & ST_U) == 0) & cw[k];
      if (lane == L[k]) met_w = m;
      if (NEED_FD) {
        const uint32_t f = __ballot_sync(FULL, (wv[k] & ST_FD) != 0) & cw[k];
        if (lane == L[k]) fd_w = f;
      }
    } else {
      const uint32_t m = __ballot_sync(FULL, c[k] && (wv[k] & ST_U) == 0);
      if (lane == L[k]) met_w = m;
      if (NEED_FD) {
        const uint32_t f = __ballot_sync(FULL, c[k] && (wv[k] & ST_FD) != 0);
        if (lane == L[k]) fd_w = f;
      }
    }
  }
}

template <int FMT, bool NEED_FD, bool AL = false>
DI void walk_items(uint32_t lane, uint32_t CAND, uint32_t lg, const WalkCtx& C, uint32_t& met_w, uint32_t& fd_w) {
  met_w = 0;
  fd_w = 0;
  uint32_t todo = __ballot_sync(FULL, CAND != 0);  // (run, word) pairs with at least one candidate step
  while (__popc(todo) >= WALK_K) walk_items_k<WALK_K, FMT, NEED_FD, AL>(lane, CAND, todo, lg, C, met_w, fd_w);
  if (WALK_K > 2)
    if (__popc(todo) >= 2) walk_items_k<2, FMT, NEED_FD, AL>(lane, CAND, todo, lg, C, met_w, fd_w);
  if (todo) walk_items_k<1, FMT, NEED_FD, AL>(lane, CAND, todo, lg, C, met_w, fd_w);
}

// mixed row formats inside one group (rare): one item at a time, format read from the item's table entry
template <bool NEED_FD>
DI void walk_items_any(uint32_t lane, uint32_t CAND, uint32_t lg, const WalkCtx& C, uint32_t& met_w, uint32_t& fd_w) {
  met_w = 0;
  fd_w = 0;
  for (uint32_t todo = __ballot_sync(FULL, CAND != 0); todo;) {
    const uint32_t L = __ffs(todo) - 1;
    const uint32_t meta = lds_u32(C.tab_a + (L >> lg) * 16u + 12u);
    const int fmt = fmt_of(meta >> 16, meta & 0xFFFFu);  // warp-uniform
    uint32_t one = todo & (0u - todo);
    todo ^= one;
    if (fmt == FMT_ELL4B) walk_items_k<1, FMT_ELL4B, NEED_FD>(lane, CAND, one, lg, C, met_w, fd_w);
    else if (fmt == FMT_ELL2B) walk_items_k<1, FMT_ELL2B, NEED_FD>(lane, CAND, one, lg, C, met_w, fd_w);
    else if (fmt == FMT_ELL4) walk_items_k<1, FMT_ELL4, NEED_FD>(lane, CAND, one, lg, C, met_w, fd_w);
    else if (fmt == FMT_CSR4) walk_items_k<1, FMT_CSR4, NEED_FD>(lane, CAND, one, lg, C, met_w, fd_w);
    else if (fmt == FMT_ELL2) walk_items_k<1, FMT_ELL2, NEED_FD>(lane, CAND, one, lg, C, met_w, fd_w);
    else walk_items_k<1, FMT_CSRL, NEED_FD>(lane, CAND, one, lg, C, met_w, fd_w);
  }
}

// CD: cond and/or decision codes present   XO: any of fail/needs_cond/skip_dep/phase_out requested
// LIST: run-list mode (touched ticks, resident_abi.cu): group t takes the runs at list positions [t * R, t * R + R) of P.run_list, whose
//       length the list build left at *P.run_list_count (P.n_runs is the host's bound on it).  The runs' state records are not
//       adjacent, so the lane that owns a run copies its record itself; results go to each run's own index, and no fused head
//       words are written.
template <bool CD, bool XO, bool LIST>
#ifndef PACK_MIN_BLOCKS
#define PACK_MIN_BLOCKS 1   // resident CTAs per SM the build is compiled for (BF_PACK_CTAS experiments)
#endif
__global__ void __launch_bounds__(32 * PACK_MAX_WARPS, PACK_MIN_BLOCKS) frontier_pack_kernel(const KParams P) {
  // BF_EVAL_PIPELINED: let the next kernel of the stream (launched as a programmatic dependent) take the SMs this grid leaves
  // as its CTAs run out of groups; a no-op otherwise
  if (P.flags & BF_EVAL_PIPELINED) asm volatile("griddepcontrol.launch_dependents;");
  const uint32_t lane = pin(threadIdx.x & 31u);  // pinned: otherwise rematerialised from S2R inside the loop
  const uint32_t warp = __shfl_sync(FULL, threadIdx.x >> 5, 0);  // through a shuffle: the compiler then treats it as warp-uniform
  const uint32_t NW = P.warps_per_block, NG = P.slot_groups;
  const uint32_t Wq = P.wq, lg = P.wq_log2, R = 32u >> lg;
  const uint32_t g = pin(lane >> lg), w = pin(lane & (Wq - 1u));
  const uint32_t wq_mask = Wq == 32u ? FULL : ((1u << Wq) - 1u);
  const uint32_t gmask = wq_mask << (g << lg);
  const uint32_t Wmax = P.words;
  constexpr bool FF = !CD;   // the fail-fast skip and the floor cut below

#ifdef PACK_TRACE
  const unsigned long long tr_start = gtime();
  const unsigned int tr_launch = *((volatile unsigned int*)&g_launch) & 7u;
  unsigned long long tr_first = 0, tr_last = 0;
#endif
  // ---- shared memory carve-up: [block counters 128 B][mbarriers, one per slot group][NG slot groups][warp scratch]
  // slot group: R state records (contiguous, as in HBM) then R topology buffers of topo_buf_bytes each.
  // The mbarriers sit in one block AWAY from the TMA destinations (a barrier next to a record tail slowed the pass).
  unsigned long long* blk_counts = reinterpret_cast<unsigned long long*>(smem_p);
  const uint32_t smem_base = smem_u32(smem_p);
  const uint32_t bars = pin(smem_base + 128u);
  const uint32_t armed_a = bars + NG * 8u;                        // u32 per slot group: uses armed so far (see the wait below)
  const uint32_t bars_bytes = (NG * 12u + 127u) & ~127u;
  const uint32_t group_bytes = R * (P.state_stride + P.topo_buf_bytes);
  const uint32_t groups_a = pin(smem_base + 128u + bars_bytes);
  // scratch (per warp, 256-byte aligned, work_bytes a multiple of 256, at least ST_BYTES + 128 + 16 R): [status pairs: R x 16 Wq]
  // [fix-up fail words 128 B][walk table: R x 16 B]
  const uint32_t st_run = 16u * Wq;
  const uint32_t scratch_a = ((groups_a + NG * group_bytes + 255u) & ~255u) + warp * P.work_bytes;
  const uint32_t st0_a = scratch_a;
  const uint32_t mfail_a = st0_a + ST_BYTES;
  const uint32_t tab_a = mfail_a + 128u;
  // !CD passes (no fix-up): the fix-up words of the NW warps hold the needed word of slot group sg (issue(); NG <= 32 NW)
  // at word sg % 32 of warp sg / 32, an address recomputed from the parameters at each use (a register more spills)
  auto need_a = [&](uint32_t sg) {
    return ((groups_a + NG * (R * (P.state_stride + P.topo_buf_bytes)) + 255u) & ~255u) + (sg >> 5) * P.work_bytes + ST_BYTES + (sg & 31u) * 4u;
  };

  if (threadIdx.x < 5) blk_counts[threadIdx.x] = 0ull;   // four counters + the group ticket
  if (threadIdx.x < NG) {   // NG <= blockDim.x: the planner (plan_pack, abi.cu) gives a CTA no more slot groups than threads
    mbar_init(bars + 8u * threadIdx.x, R);
    sts_u32(armed_a + 4u * threadIdx.x, 0u);
    fence_barrier_init();
  }
  for (uint32_t x = lane * 4u; x < P.work_bytes; x += 128u) sts_u32(scratch_a + x, 0u);  // the PAD pairs start as 0 and stay 0
  __syncthreads();

  // ---- the CTA's groups: global group id = blockIdx.x + t * gridDim.x, runs R * gid .. R * gid + R - 1
  const uint32_t N = LIST ? min(*reinterpret_cast<const volatile uint32_t*>(P.run_list_count), P.n_runs) : P.n_runs;
  const uint32_t n_groups = (N + R - 1) >> (5 - lg);
  const uint32_t T = blockIdx.x < n_groups ? (n_groups - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  // Schedule: groups are CONSUMED in ticket order — a warp that is free takes the next group of the CTA from a shared
  // counter (a static t -> warp map left the warps with one group more than the others running alone at the end).
  // Group t lives in slot group t % NG, use number t / NG; groups t < NG are issued in the prologue (by warp t % NW), group t >= NG by the warp that consumed t - NG and thereby freed the slot.
  const uint32_t n_pro = warp < NG ? (NG - warp + NW - 1) / NW : 0;   // my prologue issues: t = warp + q * NW < NG

  // ---- producer side: the chain run -> slot id -> slot entry of a group is fetched by the R lanes that own its runs.
  // Prologue: lane l holds (issue q0 + l / R, run l % R) of a batch of GB = 32 / R issues; steady state: the lanes of
  // issue 0 (lq == 0) hold the group my warp will issue when it is done with the current one.
  const uint32_t GB = 32u >> (5 - lg);        // = Wq: issues per prologue batch
  const uint32_t lq = lane >> (5 - lg), lr = lane & (R - 1u);   // my pair inside a batch: issue lq, run lr
  // A lane without a run keeps pf_sid all ones, so load_ent leaves its entry zero and issue() writes a dead marker.
  uint32_t pf_sid = 0xFFFFFFFFu, pf_rf = 0, pf_lo = 0, pf_hi = 0, pf_bytes = 0, pf_meta = 0;
  uint32_t pf_run = 0xFFFFFFFFu;   // LIST: my run of the group I shall issue (all ones: none)
  auto load_sid = [&](uint32_t t, bool mine) {   // first link: my run's topology slot id and run flags (bf_run_header)
    pf_sid = 0xFFFFFFFFu; pf_rf = 0;
    if (LIST) pf_run = 0xFFFFFFFFu;
    if (mine && t < T) {
      uint32_t r = ((blockIdx.x + t * gridDim.x) << (5 - lg)) + lr;
      if (r < N) {
        if (LIST) { r = __ldg(P.run_list + r); pf_run = r; }
        const uint8_t* sr = P.state + (size_t)r * P.state_stride;
        const uint2 hv = __ldg(reinterpret_cast<const uint2*>(sr));
        pf_sid = hv.x; pf_rf = hv.y;
        // the phase words load_cut() reads for this run: into L2 now, so that they are there when it asks
        asm volatile("prefetch.global.L2 [%0];" ::"l"(sr + P.off_phase));
        asm volatile("prefetch.global.L2 [%0];" ::"l"(sr + P.off_phase + 16u * Wmax - 4u));
      }
    }
  };
  // second link: the slot entry (address, bytes, meta).  From here on pf_sid is the slot whose cut-table row load_cut() reads,
  // with SID_NO_FF for a run that is not fail-fast or whose group the host sets (stage I does not mark it), SID_NO_FLOOR for
  // a topology-terminated run (condition (3) in stages.cuh) and SID_RT for a realtime one; all ones: no row (a run without a
  // live slot, slot ids above SID_SLOT, passes with cond or decision codes).
  constexpr uint32_t SID_NO_FF = 1u << 31, SID_NO_FLOOR = 1u << 30, SID_RT = 1u << 29, SID_SLOT = SID_RT - 1u;
  auto load_ent = [&]() {
    pf_lo = 0; pf_hi = 0; pf_bytes = 0; pf_meta = 0;
    if (pf_sid < P.n_slots) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(P.slots + pf_sid));
      pf_lo = v.x; pf_hi = v.y; pf_bytes = v.z; pf_meta = v.w;
    }
    if (FF && pf_sid < P.n_slots && pf_sid <= SID_SLOT) {
      asm volatile("prefetch.global.L2 [%0];" ::"l"(P.ff_mask + (size_t)pf_sid * FF_STRIDE));
      pf_sid |= ((pf_rf & (BF_RF_FAIL_FAST | BF_RF_HOST_GROUP)) != BF_RF_FAIL_FAST ? SID_NO_FF : 0u) |
                ((pf_rf & BF_RF_TOPOLOGY_TERMINATED) ? SID_NO_FLOOR : 0u) | ((pf_rf & BF_RF_REALTIME) ? SID_RT : 0u);
    } else {
      pf_sid = 0xFFFFFFFFu;
    }
  };
  // The cut: a run's topology buffer receives its header and the rows from the run's first word that can hold a candidate
  // step on; the rows below stay whatever an earlier group left there.  Stage D and the cond-FAIL fix-up read the rows of
  // the words with CAND != 0 only, and by condition (1) at the top of stages.cuh a candidate's input code lies outside
  // TERMINAL and RUNNING_Q.  Should the stages ever break that condition, this cut must go.  The phase words of the group's
  // runs are read from global memory (lane g * Wq + w: word w of run g; load_sid prefetches them into L2): the same lines
  // the group's state copy reads, and like it before griddepcontrol.wait.
  // A run that cannot have a candidate at all receives no rows: a fail-fast run (stage I chooses its group) with a code of
  // TERMINAL \ COMPLETED0 on a step of its topology's fail-fast mask (FF_STRIDE, device_record.h: main steps without
  // allowFailure, and only in topologies with G1 = G2 = 0).  Condition (2) in stages.cuh says why such a run has CAND = 0
  // in every word; should the stages ever break it, this skip must go.  Only passes without cond and
  // decision codes (!CD) test for such runs: with them the test cost more than the rows it saved (H100 SXM at 700 W, cfg4,
  // µs per pipelined pass in three rounds: 52.3 - 52.5 without the test, 52.8 - 53.1 with it).
  // Passes without decision codes read neither T0, T1, T2 nor TS: a run that receives no rows then receives its planes from
  // AF on (rounded down to 16 B).
  // The floor cut, also in !CD passes only: word w of a run is NEEDED when it can hold a candidate and its dependency floor
  // (FF_STRIDE, device_record.h) is at most hs_p = 1 + the highest step with a TERMINAL code (or an RT_SAT code, realtime
  // runs).  In any other word every dependency of a candidate lies at or above hs_p, on a step that is unsatisfied and not a
  // failed dependency by condition (3) in stages.cuh, so the walk would find met = fd = 0 for every candidate: the producer stages the
  // rows of the needed words lo .. hi only (with the planes a third copy when hi is not the last word) and leaves the group's
  // needed words at need_a for the consumer, whose walk takes CAND of those words alone.  Should the stages ever break condition
  // (3), this cut must go.
  constexpr uint32_t LUT_CAND_POSSIBLE = ~(BF_LUT_TERMINAL | BF_LUT_RUNNING_Q) & 0xFFFFu;   // codes 0, 9, 10, 14, 15
  constexpr uint32_t LUT_FAILED = BF_LUT_TERMINAL & ~BF_LUT_COMPLETED0;                       // codes 4, 5, 6, 7, 11, 12
  const bool trim_planes = P.off_decision == BF_OFF_NONE;
  uint32_t cp0 = 0, cp1 = 0, cp2 = 0, cp3 = 0, ffm = 0, flr = 0;
  // the phase words, fail-fast mask word and dependency floor (| SID_RT for a realtime run; 0 = never cut) of lane g * Wq + w
  // for group t, whose slot entries the lanes of issue k hold (load_ent has run)
  auto load_cut = [&](uint32_t t, uint32_t k) {
    cp0 = 0; cp1 = 0; cp2 = 0; cp3 = 0; ffm = 0; flr = 0;
    uint32_t r = ((blockIdx.x + t * gridDim.x) << (5 - lg)) + g;
    const bool mine = t < T && r < N && w < Wmax;
    if (mine) {
      if (LIST) r = __ldg(P.run_list + r);
      const uint32_t* pw = reinterpret_cast<const uint32_t*>(P.state + (size_t)r * P.state_stride + P.off_phase) + w;
      cp0 = __ldg(pw); cp1 = __ldg(pw + Wmax); cp2 = __ldg(pw + 2u * Wmax); cp3 = __ldg(pw + 3u * Wmax);
    }
    if (!FF) return;
    const uint32_t sid = __shfl_sync(FULL, pf_sid, (k << (5 - lg)) + g);
    const uint32_t* row = P.ff_mask + (size_t)(sid & SID_SLOT) * FF_STRIDE;   // a clear SID_NO_* bit: a live slot
    if (mine && !(sid & SID_NO_FF)) ffm = __ldg(row + w);
    if (mine && !(sid & SID_NO_FLOOR)) flr = __ldg(row + FF_WORDS + w) | (sid & SID_RT);
  };
  // issue the copies of group t into slot group `sg`, which thereby starts its use number `use`; the lanes of issue `k`
  // (lq == k) own its runs and hold their slot entries, load_cut(t, k) has been called
  auto issue = [&](uint32_t t, uint32_t sg, uint32_t use, uint32_t k) {
    const uint32_t Sg = __shfl_sync(FULL, pf_meta, (k << (5 - lg)) + g) & 0xFFFFu;   // steps of run g
    const uint32_t cpw = w * 32u < Sg ? bmsk_clamp(0u, Sg - w * 32u) & plut<LUT_CAND_POSSIBLE>(cp0, cp1, cp2, cp3) : 0u;
    const uint32_t cand_b = __ballot_sync(FULL, cpw != 0);
    uint32_t need_b = cand_b;   // bit g * Wq + w: word w of run g is staged (and walked)
    if (FF) {
      const uint32_t ff_b = __ballot_sync(FULL, (plut<LUT_FAILED>(cp0, cp1, cp2, cp3) & ffm) != 0);
      const uint32_t bp = plut<BF_LUT_TERMINAL>(cp0, cp1, cp2, cp3) | (plut<BF_LUT_RT_SAT>(cp0, cp1, cp2, cp3) & (0u - ((flr >> 29) & 1u)));   // bit 29: SID_RT
      // the run's highest word with such a code (the highest lane of its segment in the ballot) and that word's highest step
      const uint32_t tb = __ballot_sync(FULL, bp != 0) & gmask;
      const uint32_t hl = 31u - __clz(tb), hb = __shfl_sync(FULL, bp, hl);   // tb = 0: any lane, result unused
      const uint32_t hs_p = tb ? (hl & (Wq - 1u)) * 32u + 32u - __clz(hb) : 0u;
      need_b = __ballot_sync(FULL, cpw != 0 && (flr & 0xFFFFu) <= hs_p && (ff_b & gmask) == 0);
    }
    const uint32_t cand_words = (need_b >> (lr << lg)) & wq_mask;   // of my run (issuing lanes)
    if (t < T && lq == k) {
      const uint32_t buf = groups_a + sg * group_bytes;
      const uint32_t bar = bars + 8u * sg;
      const uint32_t tb = buf + R * P.state_stride + lr * P.topo_buf_bytes;   // my run's topology buffer
      const bool dfr = P.defer_list != nullptr && ((pf_meta >> 16) & 0xFFu) != 0;  // topology with parallel steps
      const bool ok = !dfr && (pf_lo | pf_hi) != 0 && pf_bytes <= P.topo_buf_bytes;
      if (!ok) sts_v4(tb, dfr ? 0xFFFFFFFFu : 0u, 0u, 0u, 0u);   // marker header (W = 0: dead, all-ones: deferred)
      uint32_t sbytes = 0;
      const uint32_t first = (blockIdx.x + t * gridDim.x) << (5 - lg);
      if (LIST) sbytes = pf_run != 0xFFFFFFFFu ? P.state_stride : 0u;   // my run's record: a copy of its own
      if (lr == 0) {
        if (!LIST) sbytes = min(R, N - first) * P.state_stride;   // the group's state records are adjacent: one copy
        sts_u32(armed_a + 4u * sg, use + 1u);          // published before my arrive: the previous use is over, this one is armed
        if (FF) sts_u32(need_a(sg), need_b);           // likewise, as a marker header
      }
      // fixed-width rows (rb = row bytes per step; 0 for CSR and formats not cut: one copy of the whole record): the header,
      // then the rows of the needed words lo .. hi (!CD; else from the first word that can hold a candidate on) and the
      // planes, from AF when the pass reads no decision codes.  Up to the last word that is one copy, as is a run without
      // rows (header and planes); a run whose hi is below its last word takes a third copy for the planes (on H100 the
      // extra copy cost more than the 96 B of T0 - T2 it would save alone).
      const uint32_t Wr = ((pf_meta & 0xFFFFu) + 31u) >> 5, rb = ok ? pf_meta >> 24 : 0u;
      const uint32_t lo_word = cand_words ? __ffs(cand_words) - 1u : Wr;
      const uint32_t hi_end = FF && cand_words ? 32u - __clz(cand_words) : Wr;   // one past the last word staged
      const uint32_t hdr = (uint32_t)sizeof(TopoHeader), rows_end = hdr + 32u * rb * Wr;   // rows_end = off_planes
      const uint32_t planes_from = trim_planes ? (rows_end + PL_AF * 4u * Wr) & ~15u : rows_end;
      uint32_t from = hdr + 32u * rb * lo_word, mid = pf_bytes, rest = pf_bytes;   // copies [0, hdr), [from, mid), [rest, pf_bytes)
      if (rb && from == rows_end) from = planes_from;
      else if (rb && hi_end < Wr) { mid = hdr + 32u * rb * hi_end; rest = planes_from; }
      mbar_expect_tx(bar, (ok ? pf_bytes - (from - hdr) - (rest - mid) : 0u) + sbytes);
      if (LIST) {
        if (sbytes) bulk_g2s(buf + lr * P.state_stride, P.state + (size_t)pf_run * P.state_stride, sbytes, bar);
      } else if (lr == 0) {
        bulk_g2s(buf, P.state + (size_t)first * P.state_stride, sbytes, bar);
      }
      if (ok) {
        const uint8_t* src = reinterpret_cast<const uint8_t*>((uint64_t)pf_lo | ((uint64_t)pf_hi << 32));
        const uint32_t at = from != hdr ? from : 0u;
        if (at) bulk_g2s(tb, src, hdr, bar);
        bulk_g2s(tb + at, src + at, mid - at, bar);
        if (rest != mid) bulk_g2s(tb + rest, src + rest, pf_bytes - rest, bar);
      }
    }
  };
  for (uint32_t q0 = 0; q0 < n_pro; q0 += GB) {      // prologue: GB of my issues at a time (both links of all of them in flight together)
    const bool in_pro = q0 + lq < n_pro;
    load_sid(warp + (q0 + lq) * NW, in_pro);
    load_ent();
    load_cut(warp + q0 * NW, 0u);                    // the batch's first issue: its phase words beside the second link
    for (uint32_t k = 0; k < GB && q0 + k < n_pro; ++k) {
      const uint32_t t = warp + (q0 + k) * NW;       // < NG: its slot group is t itself, use 0
      if (k) load_cut(t, k);
      issue(t, t, 0u, k);
    }
  }

  const bool has_cond = CD && P.off_cond != BF_OFF_NONE;
  const bool has_dec = CD && P.off_decision != BF_OFF_NONE;
  uint32_t lane_ready = 0, lane_skip = 0, lane_evals = 0;  // per-lane running totals, reduced once at the end

  // the next group to consume: a CTA-wide ticket counter behind the four block counters (smem_p + 32)
  const uint32_t ng_magic = NG > 1u ? (uint32_t)(0x100000000ull / NG) + 1u : 0u;   // t / NG = umulhi(t, ng_magic), exact for t < 2^32 / NG (NG = 1: T <= 1, t = 0)
#ifdef PACK_STAGES
  uint32_t pr_acc = 0, pr_t = (uint32_t)clock();
#endif
  for (;;) {
    uint32_t t = 0;
    if (lane == 0) t = atomicAdd(reinterpret_cast<uint32_t*>(smem_p + 32), 1u);
    t = __shfl_sync(FULL, t, 0);
    if (t >= T) break;
    const uint32_t cur_use = __umulhi(t, ng_magic), cur_sg = t - cur_use * NG;   // t / NG, t % NG
    uint32_t r_list = 0;   // LIST: my run, fetched before the waits
    if (LIST) {
      const uint32_t pos = ((blockIdx.x + t * gridDim.x) << (5 - lg)) + g;
      if (pos < N) r_list = __ldg(P.run_list + pos);
    }
    load_sid(t + NG, lq == 0);   // first link of the group I shall issue into this slot group when I am done with it
    // The slot group is shared between warps: its use `cur_use` is armed by the warp that consumed the previous use.
    // A parity wait alone cannot tell "use u - 1 still pending" from "use u complete" (the parity then names the phase
    // before), so first wait until the arming warp has published use u; from then on the barrier is in phase u.
    while ((int32_t)(lds_poll_u32(armed_a + 4u * cur_sg) - (cur_use + 1u)) < 0) __nanosleep(32);
    mbar_wait(bars + 8u * cur_sg, cur_use & 1u);
    PROBE(0);
#ifdef PACK_TRACE
    if (t == 0) tr_first = gtime();
#endif

    const uint32_t gid = blockIdx.x + t * gridDim.x;
    const uint32_t pos = (gid << (5 - lg)) + g;               // my run (LIST: my list position)
    const uint32_t r = LIST ? r_list : pos;
    uint8_t* const rr = P.result + (size_t)r * P.result_stride;
    const uint32_t grp_a = groups_a + cur_sg * group_bytes;
    const uint32_t sr_a = grp_a + g * P.state_stride;                                   // my run's state record
    const uint32_t tr_a = grp_a + R * P.state_stride + g * P.topo_buf_bytes;            // my run's topology record

    const bool in_batch = pos < N;
    const uint4 h0 = lds_v4(tr_a);
    const uint4 h1 = lds_v4(tr_a + 16);
    const bool deferred = in_batch && h0.x == 0xFFFFFFFFu;
    uint32_t S = h0.x & 0xFFFFu, Wt = h0.x >> 16;
    const uint32_t max_deg = h0.y & 0xFFFFu;
    uint32_t n_main = h0.z & 0xFFFFu, n_comp = h0.z >> 16, n_final = h0.w & 0xFFFFu;
    const bool live = in_batch && Wt - 1u < Wmax;  // group-uniform (a marker header has W = 0 or 0xFFFF)
    if (!live) { S = 0; Wt = 0; n_main = n_comp = n_final = 0; }
    const uint32_t ell = live ? (h1.x >> 16) : 0u;
    const uint32_t rflags = live ? lds_u8(sr_a + 4) : (uint32_t)BF_RF_HOST_GROUP | (BF_GROUP_DONE << BF_RF_HOST_GROUP_SHIFT);

    // ---------------- planes of my word ----------------
    const bool act = w < Wt;
    uint32_t AF = 0, TS = 0, HASIF = 0, G1 = 0, G2 = 0, VALID = 0, SYNC_T = 0, NODEP = 0;
    uint32_t c0 = 0, c1 = 0, d0 = 0, d1 = 0;
    uint32_t p0 = 0, p1 = 0, p2 = 0, p3 = 0;
    if (act) {
      const uint32_t sp = tr_a + h1.y + w * 4u, ps = Wt * 4u;   // static planes: my word, plane stride
      AF = lds_u32(sp + PL_AF * ps);
      G1 = lds_u32(sp + PL_G1 * ps); G2 = lds_u32(sp + PL_G2 * ps);
      if (XO) HASIF = lds_u32(sp + PL_HASIF * ps);
      if (ell_has_nodep(ell)) NODEP = lds_u32(sp + PL_NODEP * ps);   // byte-entry rows: steps without needs stay out of the walk
      VALID = bmsk_clamp(0u, S - w * 32u);
      const uint32_t pw = sr_a + P.off_phase + w * 4u, ds = Wmax * 4u;  // dynamic planes: stride of the layout
      p0 = lds_u32(pw); p1 = lds_u32(pw + ds); p2 = lds_u32(pw + 2u * ds); p3 = lds_u32(pw + 3u * ds);
      const uint32_t keep = VALID & ~(p0 & p1 & p2 & p3);  // steps >= S and the reserved code 15 read as 0
      p0 &= keep; p1 &= keep; p2 &= keep; p3 &= keep;
      if (CD) {
        if (has_cond) { const uint32_t cw = sr_a + P.off_cond + w * 4u; c0 = lds_u32(cw); c1 = lds_u32(cw + ds); }
        if (has_dec) {
          const uint32_t dw = sr_a + P.off_decision + w * 4u; d0 = lds_u32(dw); d1 = lds_u32(dw + ds);
          const uint32_t t0 = lds_u32(sp + PL_T0 * ps), t1 = lds_u32(sp + PL_T1 * ps), t2 = lds_u32(sp + PL_T2 * ps);
          TS = lds_u32(sp + PL_TS * ps);
          SYNC_T = t0 & (t1 | t2);  // sleep(3) | wait(5) | gate(7)
        }
      }
    }
    const uint32_t q0 = p0, q1 = p1, q2 = p2, q3 = p3;
    const uint32_t GM = VALID & ~G1 & ~G2;
    const bool realtime = rflags & BF_RF_REALTIME;

    // ---------------- stages G, B, I and D-prep (stages.cuh); U & VALID: the PAD entry of a narrower run reads "satisfied"
    if (has_dec) stage_g(SYNC_T, TS, d0, d1, p0, p1, p2, p3);
    const RunClass rc = stage_bi<CD>([&](uint32_t v) { return seg_or(v, lg); }, rflags, n_main, n_comp, n_final, AF, GM, G1, G2, p0, p1, p2, p3);
    uint32_t summary = rc.sum | rc.group;
    const DepClass dc = stage_dprep(rc, rflags, VALID, GM, G1, G2, NODEP, p0, p1, p2, p3);
    const uint32_t U = dc.U, FD = dc.FD;
    // the floor cut: the walk takes the words the producer staged (bit `lane` of the slot group's needed word); a word it
    // left out has met = FREE, fd = 0
    const uint32_t CAND = FF ? ((lds_u32(need_a(cur_sg)) >> lane) & 1u ? dc.CAND : 0u) : dc.CAND;
    // ------------- stage C: each lane's status word pair (U and FD interleaved by half words), all R runs -------------
    const bool any_fd = __any_sync(FULL, dc.skip_on_failed);           // some run of the group has a failed-dependency class
    const int my_fmt = fmt_of(ell, max_deg);
    const int fmt0 = __shfl_sync(FULL, live ? my_fmt : -1, __ffs(__ballot_sync(FULL, live) | 0x80000000u) - 1);  // format of the first live run
    const bool mixed = __any_sync(FULL, live && my_fmt != fmt0);
    PROBE(1);
    __syncwarp();
    const uint32_t my_st = st0_a + g * st_run;
    sts_v2(my_st + w * 8u, __byte_perm(U, FD, 0x5410), __byte_perm(U, FD, 0x3276));   // {U lo, FD lo}, {FD hi, U hi}
    // per-run walk entry: CSR / row bases, status base, longest row and row format
    const uint32_t col_a = tr_a + (h1.x & 0xFFFFu);
    if (w == 0) sts_v4(tab_a + g * 16u, col_a, tr_a + (uint32_t)sizeof(TopoHeader), my_st, max_deg | (ell << 16));
    __syncwarp();
    PROBE(2);
    // second link of the group I shall issue (its slot id, requested when I drew my ticket, has arrived by now — asking for
    // it right behind the barrier wait stalled every trip for a DRAM round trip); consumed by issue() at the end of the trip
    load_ent();
    // ------------- stage D: walk the needs rows (dag.go:2711-2733) -------------
    uint32_t met_w, fd_w;
    const WalkCtx wctx{tab_a, grp_a + R * P.state_stride + (uint32_t)sizeof(TopoHeader), P.topo_buf_bytes, st0_a, st_run};
    if (mixed) {
      if (any_fd) walk_items_any<true>(lane, CAND, lg, wctx, met_w, fd_w);
      else walk_items_any<false>(lane, CAND, lg, wctx, met_w, fd_w);
    } else if (fmt0 == FMT_ELL4B && Wq == 8u) {   // 129 .. 256 steps: entries used in place in the row word
      if (any_fd) walk_items<FMT_ELL4B, true, true>(lane, CAND, lg, wctx, met_w, fd_w);
      else walk_items<FMT_ELL4B, false, true>(lane, CAND, lg, wctx, met_w, fd_w);
    } else if (fmt0 == FMT_ELL4B) {
      if (any_fd) walk_items<FMT_ELL4B, true>(lane, CAND, lg, wctx, met_w, fd_w);
      else walk_items<FMT_ELL4B, false>(lane, CAND, lg, wctx, met_w, fd_w);
    } else if (fmt0 == FMT_ELL2B) {
      if (any_fd) walk_items<FMT_ELL2B, true>(lane, CAND, lg, wctx, met_w, fd_w);
      else walk_items<FMT_ELL2B, false>(lane, CAND, lg, wctx, met_w, fd_w);
    } else if (fmt0 == FMT_ELL4) {
      if (any_fd) walk_items<FMT_ELL4, true>(lane, CAND, lg, wctx, met_w, fd_w);
      else walk_items<FMT_ELL4, false>(lane, CAND, lg, wctx, met_w, fd_w);
    } else if (fmt0 == FMT_CSR4) {
      if (any_fd) walk_items<FMT_CSR4, true>(lane, CAND, lg, wctx, met_w, fd_w);
      else walk_items<FMT_CSR4, false>(lane, CAND, lg, wctx, met_w, fd_w);
    } else if (fmt0 == FMT_ELL2) {
      if (any_fd) walk_items<FMT_ELL2, true>(lane, CAND, lg, wctx, met_w, fd_w);
      else walk_items<FMT_ELL2, false>(lane, CAND, lg, wctx, met_w, fd_w);
    } else {
      if (any_fd) walk_items<FMT_CSRL, true>(lane, CAND, lg, wctx, met_w, fd_w);
      else walk_items<FMT_CSRL, false>(lane, CAND, lg, wctx, met_w, fd_w);
    }
    met_w |= dc.FREE;
    PROBE(3);
    load_cut(t + NG, 0u);   // the phase words and masks for the cut of the group I shall issue (issue() reduces them)
    uint32_t ready_w = met_w, skipc_w = 0, fail_w = 0;
    if (CD) {
      // item L: word L & (Wq - 1) of run L >> lg, its rows and status pairs from the run's walk-table entry
      auto fixup = [&](uint32_t L, uint32_t candw, uint32_t fclass, uint32_t& mb, uint32_t& fb) {
        const uint4 te = lds_v4(tab_a + (L >> lg) * 16u);
        auto status = [&](uint32_t d) { const uint32_t s = dep_status(te.z, d, ~3u); return (s & ST_U) | ((s >> 15) & 2u); };
        fixup_item(lane, candw, L & ((1u << lg) - 1u), te.w >> 16, te.y, te.x, status, mfail_a + ((L >> lg) << lg) * 4u, fclass, mb, fb);
      };
      stage_cond(lane, c0, c1, dc, mfail_a, true, 32u * Wmax, fixup, met_w, fd_w, ready_w, skipc_w, fail_w, p0, p1, p2, p3);
    }
    const uint32_t acc_ready = ready_w, acc_skip = fd_w | skipc_w;

    // ---------------- stage E: result records ----------------
    const uint32_t cnt = seg_add((uint32_t)__popc(acc_ready) | ((uint32_t)__popc(acc_skip) << 16), lg);   // both <= S <= 512
    bool changed = rc.marked;   // with cond / decision codes: stage G may write the code a step already has
    if (CD) changed = (__ballot_sync(FULL, ((p0 ^ q0) | (p1 ^ q1) | (p2 ^ q2) | (p3 ^ q3)) != 0) & gmask) != 0;
    // fused compaction head (compact.cu): events of the run = steps with a bit in any result mask the layout carries
    uint32_t n_events = 0;
    if (P.head) {
      uint32_t u = acc_ready | acc_skip;
      if (XO) {
        if (P.off_fail != BF_OFF_NONE) u |= fail_w;
        if (P.off_needs_cond != BF_OFF_NONE) u |= realtime ? 0u : (met_w & HASIF);
        if (P.off_skip_dep != BF_OFF_NONE) u |= fd_w;
      }
      n_events = seg_add((uint32_t)__popc(u), lg);
    }
    if (deferred) {
      if (w == 0) P.defer_list[atomicAdd(P.defer_count, 1u)] = r;  // the general kernel writes this run's record
    } else if (in_batch) {
      if (w == 0) {
        summary = live ? (summary | (changed ? BF_SUM_PHASE_CHANGED : 0u) | (1u << BF_SUM_ITER_SHIFT)) : 0xFFFFFFFFu;
        *reinterpret_cast<uint4*>(rr) = make_uint4(summary, cnt & 0xFFFFu, cnt >> 16, 0u);
        if (P.exp_counts) P.exp_counts[r] = 0;
        if (P.head) {
          P.head[r] = live ? ((summary & BF_HEAD_SUMMARY_MASK) | BF_HEAD_LISTED | (n_events << BF_HEAD_COUNT_SHIFT)) : (BF_HEAD_DEAD | BF_HEAD_LISTED);
          if (live && n_events) atomicAdd(&P.head_sums[r >> 9], (unsigned long long)n_events);
        }
      }
      store_words<XO>(P, rr, w, Wq, acc_ready, acc_skip, fail_w, realtime ? 0u : (met_w & HASIF), fd_w, p0, p1, p2, p3);
    }
    lane_ready += (uint32_t)__popc(acc_ready);
    lane_skip += (uint32_t)__popc(acc_skip);
    lane_evals += (w == 0 && live) ? S : 0u;

    __syncwarp();  // every lane is done with this slot group's buffers
    PROBE(4);
    issue(t + NG, cur_sg, cur_use + 1u, 0u);  // re-arm it with group t + NG (consumed by whichever warp draws that ticket)
    PROBE(5);
#ifdef PACK_STAGES
    pr_acc += lane == 6u ? 1u : 0u;   // trips
#endif
#ifdef PACK_TRACE
    if (t == 0 && lane == 0 && blockIdx.x < 160) g_trace[tr_launch][blockIdx.x][1] = tr_first;
    tr_last = gtime();
#endif
  }
#ifdef PACK_TRACE
  if (lane == 0 && blockIdx.x < 160) atomicMax(&g_trace[tr_launch][blockIdx.x][2], tr_last);
#endif
#ifdef PACK_STAGES
  if (lane < 7u) atomicAdd(&g_stages[lane], (unsigned long long)pr_acc);
#endif

  // ---- BF_EVAL_PIPELINED: this grid may have started before the preceding kernel of the stream ended (it reads and writes
  // nothing of that kernel's); from here on it touches the counts and then completes, so that kernel must be complete.
  if (P.flags & BF_EVAL_PIPELINED) asm volatile("griddepcontrol.wait;" ::: "memory");
  // ---- counters: lane -> warp (redux) -> block (shared atomics) -> one global atomic per block ----
  if (P.counts) {
    const uint32_t wr = redux_add(lane_ready), ws = redux_add(lane_skip), we = redux_add(lane_evals);
    if (lane == 0) {
      atomicAdd(&blk_counts[0], (unsigned long long)wr);
      atomicAdd(&blk_counts[1], (unsigned long long)ws);
      atomicAdd(&blk_counts[3], (unsigned long long)we);
    }
    __syncthreads();
    if (P.acc == nullptr) {
      if (threadIdx.x < 4 && blk_counts[threadIdx.x] != 0ull) atomicAdd(&P.counts[threadIdx.x], blk_counts[threadIdx.x]);
    } else {
      // BF_EVAL_COUNTS_SET: totals gathered in this launch's block of the ctx scratch ring; the last CTA out writes them to
      // `counts` and clears the block for the launch that gets it next
      if (threadIdx.x < 4 && blk_counts[threadIdx.x] != 0ull) atomicAdd(&P.acc[threadIdx.x], blk_counts[threadIdx.x]);
      __threadfence();
      __syncthreads();
      volatile unsigned int* last_out = reinterpret_cast<volatile unsigned int*>(smem_p + 40);   // free word of the counter block
      if (threadIdx.x == 0) *last_out = atomicAdd(reinterpret_cast<unsigned int*>(&P.acc[4]), 1u) == gridDim.x - 1u;
      __syncthreads();
      if (*last_out) {
        __threadfence();
        if (threadIdx.x < 4) P.counts[threadIdx.x] = atomicExch(&P.acc[threadIdx.x], 0ull);
        if (threadIdx.x == 4) P.acc[4] = 0ull;
      }
    }
  }
#ifdef PACK_TRACE
  __syncthreads();
  if (threadIdx.x == 0 && blockIdx.x < 160) {
    g_trace[tr_launch][blockIdx.x][0] = tr_start;
    g_trace[tr_launch][blockIdx.x][3] = gtime();
    __threadfence();
    if (atomicAdd(reinterpret_cast<unsigned int*>(&g_trace[tr_launch][159][0]), 1u) == gridDim.x - 1) {   // last CTA out
      *reinterpret_cast<unsigned int*>(&g_trace[tr_launch][159][0]) = 0u;
      atomicAdd(&g_launch, 1u);
      for (int b = 0; b < 160; ++b) g_trace[(tr_launch + 1) & 7u][b][2] = 0ull;   // next launch's atomicMax cells
    }
  }
#endif
}


uint32_t frontier_pack_max_warps() { return PACK_MAX_WARPS; }
#ifdef PACK_TRACE
extern "C" int bf_debug_pack_trace(unsigned long long* out, unsigned int* launch) {
  cudaDeviceSynchronize();
  if (cudaMemcpyFromSymbol(out, g_trace, sizeof(g_trace)) != cudaSuccess) return -1;
  return cudaMemcpyFromSymbol(launch, g_launch, sizeof(unsigned int)) == cudaSuccess ? 0 : -1;
}
#endif
#ifdef PACK_STAGES
extern "C" int bf_debug_pack_stages(unsigned long long* out) {   // the totals since the last call, then zeroed
  static const unsigned long long zero[8] = {};
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(out, g_stages, sizeof(g_stages)) != cudaSuccess) return -1;
  return cudaMemcpyToSymbol(g_stages, zero, sizeof(g_stages)) == cudaSuccess ? 0 : -1;
}
#endif

cudaError_t launch_frontier_pack(const KParams& P, uint32_t grid, uint32_t smem_bytes, cudaStream_t stream) {
  static const KernelFn table[8] = {frontier_pack_kernel<false, false, false>, frontier_pack_kernel<false, true, false>,
                                    frontier_pack_kernel<true, false, false>,  frontier_pack_kernel<true, true, false>,
                                    frontier_pack_kernel<false, false, true>,  frontier_pack_kernel<false, true, true>,
                                    frontier_pack_kernel<true, false, true>,   frontier_pack_kernel<true, true, true>};
  const KernelFn fn = table[variant_bits(P) | (P.run_list ? 4u : 0u)];
  const cudaError_t e = allow_max_smem(fn);
  if (e != cudaSuccess) return e;
  if (P.flags & BF_EVAL_PIPELINED) {   // programmatic dependent launch: may start while the preceding kernel drains
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(P.warps_per_block * 32); cfg.dynamicSmemBytes = smem_bytes; cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, fn, P);
  }
  fn<<<grid, P.warps_per_block * 32, smem_bytes, stream>>>(P);
  return cudaGetLastError();
}

}  // namespace bf
