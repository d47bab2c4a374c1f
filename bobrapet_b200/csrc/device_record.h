// device_record.h — HBM layouts shared by the host packer (topology.cu) and the kernels.
//
// A topology (one Story generation: needs-adjacency + static step flags) is one
// contiguous, 16-byte aligned, 16-byte padded record in the arena so that a warp
// stages it into shared memory with ONE cp.async.bulk (TMA) copy.  Two adjacency formats,
// chosen per topology when it is uploaded (plan_record, topology.cu):
//
//   CSR (ell = 0)
//   +0            TopoHeader (32 B)
//   +32           row_ptr   u16[S+1]          CSR over allStorySteps (dag.go:3270), pad 16
//   +off_col      col_idx   u16[E]            dependency step indices, then >= 4 zero entries, pad 16
//
//   fixed-width rows (ell = K in {2, 4}; taken when no step has more than K needs and S*K entries are not
//   larger than the CSR block they replace; S > 256): row_ptr is implicit (row i starts at entry i*K)
//   +32 = off_col col_idx   u16[32*W][K]      the needs of step i, unused entries (and the rows past S) = PAD
//                                             PAD = 32*W: the status just past the last step word, always
//                                             "satisfied, not failed", so a padded entry never changes a verdict
//
//   fixed-width rows with BYTE entries (ell = 0x100 | K; taken for every topology of at most 256 steps that qualifies
//   for fixed-width rows): a step index fits a byte, so the adjacency is HALF the size again
//   +32 = off_col col_idx   u8[32*W][K]       the needs of step i; a row shorter than K repeats its first entry (the OR
//                                             over a row's statuses is idempotent); there is no PAD index (32*W = 256
//                                             does not fit a byte at S = 256), so a row WITHOUT needs holds its own index
//                                             and its step is flagged in a ninth static plane, NODEP: flagged steps never
//                                             enter the walk, their dependencies are trivially met
//
//   fixed-width rows with 10-BIT entries (ell = 0x200 | 4; taken for topologies of more than 512 steps — the ones only the
//   one-run-per-warp kernel stages — whose rows have at most 4 needs): a step index below 1024 fits 10 bits
//   +32 = off_col lo        u32[32*W]         entries 0, 1, 2 in bits 0-9, 10-19, 20-29; the low 2 bits of entry 3 in bits 30-31
//   +32 + 128*W   hi        u8[32*W]          the high 8 bits of entry 3          (5 bytes per row against 8)
//                                             short rows, rows without needs and NODEP as for byte entries
//
//   all
//   +off_planes   planes    u32[8 or 9][W]    static step flags, BIT-SLICED (W = ceil(S/32)):
//                                             t0,t1,t2 (type), AF, TS, HAS_IF, G1 (comp), G2 (finally)
//                                             = S bytes, same size as the canonical u8 step_flags[S];
//                                             byte-entry and 10-bit rows: + NODEP
//   +off_par      ParDesc[P] (16 B each) followed by the branch allowFailure bit words
//
// Canonical ("algorithmic") bytes per topology, SURVEY.md section 8(d):
//   2*(S+1) + 2*E + S  (u16 CSR + u8 flags).  The CSR record adds the header and the 16-byte paddings
//   (~1.5% at cfg3); the fixed-width record drops row_ptr, so it is SMALLER than the canonical figure
//   (cfg3: 2 336 B with u16 entries, 1 344 B with byte entries, against 2 798 B).
#pragma once
#include <stdint.h>

namespace bf {

struct TopoHeader {
  uint16_t S;          // steps
  uint16_t W;          // ceil(S/32)
  uint16_t max_deg;    // largest in-degree (the kernel's straight-line walk covers <= 4; E = row_ptr[S])
  uint16_t P;          // parallel descs
  uint16_t n_main, n_comp, n_final;
  uint16_t child_nibbles;  // total child nibbles of all descs
  uint16_t off_col;    // byte offset of col_idx
  uint16_t ell;        // 0 = CSR (row_ptr at +32), K = 2 / 4: fixed-width rows of K u16 entries, no row_ptr; 0x100 | K: byte entries; 0x204: 10-bit entries
  uint32_t off_planes;
  uint32_t off_par;
  uint32_t rec_bytes;  // multiple of 16
};
static_assert(sizeof(TopoHeader) == 32, "TopoHeader must be 32 bytes");

enum Plane { PL_T0 = 0, PL_T1, PL_T2, PL_AF, PL_TS, PL_HASIF, PL_G1, PL_G2, PL_COUNT, PL_NODEP = PL_COUNT };
constexpr uint32_t ELL_BYTE = 0x100u;                                                   // TopoHeader::ell flag: byte entries
constexpr uint32_t ELL_PACK10 = 0x200u;                                                 // TopoHeader::ell flag: 10-bit entries (K = 4)
__host__ __device__ inline uint32_t ell_k(uint32_t ell) { return ell & 0xFFu; }                      // entries per row
__host__ __device__ inline uint32_t ell_row_bytes(uint32_t ell) {
  return (ell & ELL_PACK10) ? 5u : ((ell & ELL_BYTE) ? (ell & 0xFFu) : 2u * ell);
}
__host__ __device__ inline bool ell_has_nodep(uint32_t ell) { return (ell & (ELL_BYTE | ELL_PACK10)) != 0; }
__host__ __device__ inline uint32_t plane_count(uint32_t ell) { return ell_has_nodep(ell) ? PL_COUNT + 1u : PL_COUNT; }
// entry e of row i of a fixed-width block at `col` (any of the three entry widths); W = words of the topology
__host__ __device__ inline uint32_t ell_entry(const uint8_t* col, uint32_t ell, uint32_t W, uint32_t i, uint32_t e) {
  if (ell & ELL_PACK10) {
    const uint32_t lo = reinterpret_cast<const uint32_t*>(col)[i];
    return e < 3u ? (lo >> (10u * e)) & 0x3FFu : (lo >> 30) | ((uint32_t)col[128u * W + i] << 2);
  }
  if (ell & ELL_BYTE) return col[i * (ell & 0xFFu) + e];
  return reinterpret_cast<const uint16_t*>(col)[i * ell + e];
}

struct ParDesc {
  uint16_t step;
  uint16_t branches;
  uint32_t child_first;  // nibble offset in the run's child area
  uint32_t allow_off;    // byte offset (from record start) of this desc's allowFailure bit words
  uint32_t reserved;
};
static_assert(sizeof(ParDesc) == 16, "ParDesc must be 16 bytes");

struct Slot {          // device slot table entry
  uint64_t addr;       // device address of the record (0 = dead slot)
  uint32_t bytes;      // rec_bytes
  uint32_t meta;       // S | P << 16 | row_bytes << 24 (P = number of parallel descs; row_bytes = bytes of one needs row of a
                       // byte-entry or u16 fixed-width record, whose rows of a 32-step word are row_bytes * 32 bytes, else 0)
};
// bits 24-31 of Slot::meta (topology.cu writes them, the packed-lanes kernel reads them to stage only the rows it can walk)
__host__ __device__ inline uint32_t slot_row_bytes(uint32_t ell) { return (ell != 0 && !(ell & ELL_PACK10)) ? ell_row_bytes(ell) : 0u; }
static_assert(sizeof(Slot) == 16, "Slot must be 16 bytes");
// Cut table beside the slot table: FF_STRIDE words per slot id, filled for a topology of at most FF_WORDS words (512
// steps) that has no compensation or finally step; every other topology (and a dead slot) has an all-zero row.  The
// packed-lanes kernel reads it to stage fewer needs rows (the cut, frontier_pack.cu).
//   words 0 .. FF_WORDS - 1          fail-fast mask: word w holds the bits of word w of the main steps without allowFailure.
//                                    A fail-fast run with a Failed step under its mask has no candidate step in its pass,
//                                    so none of its rows are staged.
//   words FF_WORDS .. FF_STRIDE - 1  dependency floor of word w: 1 + the smallest real dependency index of the steps of word
//                                    w that are walked (PAD entries and NODEP steps do not count), or 0 ("never") when such
//                                    a step has no real dependency, or FF_FLOOR_NONE when no step of the word is walked.  A
//                                    run none of whose steps at or above floor_w is satisfied or failed cannot meet or fail
//                                    a dependency of a candidate of word w, so that word is neither staged nor walked.
constexpr uint32_t FF_WORDS = 16;
constexpr uint32_t FF_STRIDE = 2 * FF_WORDS;
constexpr uint32_t FF_FLOOR_NONE = 0xFFFFu;

struct KParams {
  const uint8_t* state;
  uint8_t* result;
  const Slot* slots;
  const uint32_t* ff_mask;      // [n_slots][FF_STRIDE] cut table: fail-fast masks and dependency floors (packed-lanes kernel only)
  unsigned long long* counts;   // bf_counts (4 x u64) or nullptr
  // compact ticks whose pass is the packed-lanes kernel alone: the pass itself leaves every run's head word (summary | listed |
  // event count) and adds the counts to the per-512-run totals the emit kernel scans — no separate heads kernel
  uint32_t* head;               // [n_runs] or nullptr
  unsigned long long* head_sums;   // [ceil(n_runs / 512)], zero on entry
  unsigned long long* acc;      // BF_EVAL_COUNTS_SET, packed-lanes kernel alone: ctx scratch {4 totals, CTA ticket}; the last CTA
                                // out copies the totals to `counts` and clears the scratch (nullptr: add to `counts`)
  uint32_t* exp_counts;         // [n_runs] compact per-run expansion counts or nullptr
  // two-tier dispatch: the packed-lanes kernel appends the runs it cannot take (topologies with
  // parallel steps) to defer_list; the general kernel then runs over run_list[0..*run_list_count)
  uint32_t* defer_list;
  uint32_t* defer_count;
  const uint32_t* run_list;
  const uint32_t* run_list_count;
  uint32_t n_slots;
  uint32_t n_runs;
  uint32_t flags;               // BF_EVAL_*
  uint32_t max_iter;
  uint32_t any_parallel;        // some live topology has `parallel` steps (selects the CH kernel variants)
  // layout (bf_layout)
  uint32_t words;
  uint32_t state_stride, off_phase, off_cond, off_decision, off_child;
  uint32_t result_tail;         // first byte after the last result field (padding up to the stride is zeroed)
  uint32_t result_stride, off_ready, off_skip, off_fail, off_needs_cond, off_skip_dep, off_phase_out;
  // shared-memory plan
  uint32_t stages;              // general kernel: ring depth per warp
  uint32_t topo_buf_bytes;      // per-run room for a topology record
  uint32_t stage_bytes;         // general kernel: state_stride + topo_buf_bytes (multiple of 16)
  uint32_t work_bytes;          // per-warp scratch
  uint32_t warps_per_block;
  uint32_t occ2;                // general kernel: launch the build compiled for two resident CTAs per SM
  uint32_t run_blocked;         // general kernel: 1: a warp takes a contiguous block of runs, 0: every G-th run
  // packed-lanes kernel (frontier_pack.cu): words per run rounded up to a power of two, slot groups per CTA
  uint32_t wq, wq_log2;
  uint32_t slot_groups;
};

// a pass's small results, posted to pinned host memory by the last block of a compaction (no separate small D2H copies)
struct ResultTail {
  unsigned long long events;      // events of the batch (touched ticks: of the listed runs)
  unsigned long long counts[4];   // bf_counts of the pass, or zero
  unsigned long long rejected;    // rejected deltas, or zero without a counter
  unsigned long long listed;      // listed runs
  unsigned long long evaluated;   // touched ticks: runs evaluated (touched_emit)
  unsigned long long carried;     // touched ticks: touched runs in [n_scan, n_marks), left for a later tick (touched_list)
};
static_assert(offsetof(ResultTail, counts) == 8 && offsetof(ResultTail, rejected) == 40 && offsetof(ResultTail, listed) == 48 &&
              offsetof(ResultTail, evaluated) == 56 && offsetof(ResultTail, carried) == 64, "ResultTail: word k at byte 8 * k");

// compact.cu: result records -> one head word per run + 16-bit (step | kind << 10) events
struct CompactParams {
  const uint8_t* result;
  const uint8_t* prev_result;        // previous tick's records (changed-only mode) or nullptr: every run is listed
  uint32_t* head;                    // [n_runs]
  uint32_t* host_head;               // the caller's pinned head buffer (device-visible address) or nullptr: heads are also posted
                                     // straight to it, no separate download
  uint16_t* events;                  // [cap]
  unsigned long long cap;
  unsigned long long* block_sums;    // scratch: ceil(n_runs / 512)
  unsigned long long* zero_sums;     // the OTHER totals buffer: the emit kernel leaves it zeroed for the next tick's pass to add into
  uint32_t zero_len;                 // entries of zero_sums
  uint32_t heads_done;               // the pass wrote head words and block totals itself (every run listed): no compact_heads
  unsigned long long* total;         // out: [0] events of the batch, [1] listed runs
  ResultTail* host_tail;             // device-visible address of the pinned tail (all but evaluated and carried), or nullptr
  const unsigned long long* counts;  // device bf_counts of the pass
  const uint32_t* rejected;          // device counter of rejected deltas, or nullptr
  uint32_t n_runs, words, result_stride, result_tail, off_ready, off_skip, off_fail, off_needs_cond, off_skip_dep;
};

// compact.cu, touched ticks (bf_resident_tick_touched, resident_abi.cu): the list build in front of the pass and the list-mode compaction
// behind it.  Every scratch array is written before it is read in the same tick (no self-cleaning needed).
struct TouchedParams {
  CompactParams C;               // result = the pass's new records (the batch's second buffer), prev_result = the batch's current
                                 // records (brought up to date here); events, cap, host_tail, counts, rejected as for compact_emit
  uint32_t* mark;                // [n_marks rounded up to 4] touch marks: touched when mark >> 1 > full_epoch, bit 0 = must list
  uint32_t full_epoch;
  uint32_t n_scan;               // the list takes the touched runs of [0, n_scan)
  uint32_t n_marks;              // the list build counts the touched runs of [n_scan, n_marks) too (they stay touched)
  uint32_t bound;                // the host's bound on the list length: list capacity, grid of the compaction
  uint32_t* list;                // [bound] touched runs, ascending
  uint32_t* list_count;          // [1] their number
  uint32_t* pos_head;            // [bound] head word per list position
  unsigned long long* sums;      // [ceil(bound / 512)] events per compaction block
  unsigned long long* sums_listed;  // [ceil(bound / 512)] listed runs per compaction block
  unsigned long long* scan_sums; // [ceil(n_marks / 2048)] touched runs below n_scan per list-build block
  unsigned long long* carry_sums;   // [ceil(n_marks / 2048)] touched runs at or above n_scan per list-build block
  uint32_t* out_runs;            // [runs_cap] listed runs (device scratch or the caller's pinned buffer)
  uint32_t* out_head;            // [runs_cap]
  uint32_t runs_cap;
};

// resident.cu (row f2)
struct DeltaParams {
  uint8_t* state;
  const bf_delta* deltas;
  uint32_t n, n_runs;
  uint32_t words, state_stride, off_phase, off_cond, off_decision, off_child, child_nibbles;
  uint32_t* rejected;  // count of deltas outside the record (bad run / index / absent field)
  uint32_t* mark;      // [n_runs] touch marks (Resident in ctx.h, touched ticks): every delta of a run in range raises its mark to mark_value
  uint32_t mark_value;
  bf_run_ctl* runctl;  // [n_runs] run-control records, or nullptr: no area (a RUN_FLAGS delta of a stopped run goes to saved_flags)
};

// bf_resident_migrate (resident.cu): the records of the runs on old_slot are re-indexed in place to new_slot's step indices
struct MigrateDesc {   // a parallel desc of the new topology whose step is the image of a parallel step of the old one
  uint32_t old_first, new_first;   // child_first of the old / new desc: multiples of 8 nibbles, so whole u32 words of the child area
  uint16_t branches, old_p, new_p, reserved;
};
static_assert(sizeof(MigrateDesc) == 16, "MigrateDesc must be 16 bytes");
struct MigrateParams {
  uint8_t* state;
  uint32_t* mark;                // touch marks: a migrated run's is set to mark_value (touched and must be listed)
  uint32_t mark_value;
  uint32_t* migrated;            // [1] runs migrated (zeroed by the caller)
  const uint16_t* inv;           // [words * 32] old index of new step j, or BF_MIGRATE_GONE
  const MigrateDesc* desc;       // [n_desc]
  uint32_t n_desc;
  uint32_t n_runs, old_slot, new_slot;
  uint32_t words, state_stride, off_phase, off_cond, off_decision, off_child;
  uint32_t child_nibbles;        // of the layout; the child area is ceil(child_nibbles / 8) u32 words
  unsigned long long* timers;    // [capacity][timer_k] the batch's timer slots (bf_timer_slot), or nullptr: no area
  const uint16_t* fwd;           // [n_old_steps] the step map (new index of old step i, or BF_MIGRATE_GONE), for the timers
  uint32_t timer_k, n_old_steps;
  uint8_t* sched_rec;            // [capacity][sched_stride] the last schedule records (kSchedNoBase), or nullptr: no area
  uint32_t sched_stride;
};

// bf_resident_redrive (resident.cu): the reset sets of the requests are cleared in the records of their runs
struct RedriveParams {
  uint8_t* state;
  uint32_t* mark;                // touch marks: an applied request raises its run's to mark_value (touched, as by a delta)
  uint32_t mark_value;
  const bf_redrive* req;         // [n]
  const uint32_t* key;           // [n] row of `masks` holding request i's reset set, or BF_REDRIVE_ALL
  const uint32_t* masks;         // [keys][words] closure masks (launch_closure)
  uint8_t* status;               // [n] out: 1 = the run held the request's slot and was reset
  const Slot* slots;
  uint32_t n;
  uint32_t words, state_stride, off_phase, off_cond, off_decision, off_child;
  unsigned long long* timers;    // [capacity][timer_k] timer slots, or nullptr: an applied request empties its run's
  uint32_t timer_k;
  bf_run_ctl* runctl;            // [capacity] run-control records, or nullptr: an applied request lifts its run's stop
};

// bf_resident_reshape (resident.cu): both record arrays re-laid from layout `from` into new buffers at layout `to`
struct ReshapeParams {
  const uint8_t* old_state;
  const uint8_t* old_result;
  uint8_t* state;                // [n_new][to.state_stride]
  uint8_t* result;               // [n_new][to.result_stride]
  uint32_t n_old, n_new;         // runs r >= n_old get zero records
  bf_layout from, to;
  const bf_sched_run* old_sched_in;   // the limiter inputs, or nullptr: no area (runs r >= n_old get kSchedDefault)
  bf_sched_run* sched_in;             // [n_new]
  const bf_run_ctl* old_runctl;       // run-control records, or nullptr: no area (runs r >= n_old get kRunCtlDefault)
  bf_run_ctl* runctl;                 // [n_new]
};

// bf_resident_retire (resident.cu): the runs [m, m + n) vacate their indices; the live ones among them move below m
constexpr uint32_t kRetireNoMove = 0xFFFFFFFFu;
struct RetireParams {
  uint8_t* state;
  uint8_t* result;               // the current result records
  uint32_t* mark;                // touch marks: a target's becomes mark_value (touched and must be listed), a vacated one 0
  uint32_t mark_value;
  const uint32_t* to;            // [n] the new index of run m + i, or kRetireNoMove for a retired run
  uint32_t m, n;
  uint32_t state_stride, result_stride;   // multiples of 16
  unsigned long long* timers;    // [capacity][timer_k] timer slots, or nullptr: a mover's slots move with it, vacated ones empty
  uint32_t timer_k;
  bf_sched_run* sched_in;        // [capacity] limiter inputs, or nullptr: a mover's move with it, vacated ones get kSchedDefault
  uint8_t* sched_rec;            // [capacity][sched_stride] last schedule records: a mover's target loses its baseline
  uint32_t sched_stride;
  bf_run_ctl* runctl;            // [capacity] run-control records, or nullptr: a mover's move with it, vacated ones get kRunCtlDefault
};

// bf_resident_extent / _narrow (resident.cu): the smallest layout a batch's records and the topologies of its runs allow.  Each
// extent is reduced into out[] as extent << 32 | ~index, so that one 64-bit atomicMax keeps the largest extent and the lowest
// index that needs it.
struct ExtentParams {
  const uint8_t* state;          // [n_records][L.state_stride]
  const uint8_t* result;         // [n_runs][L.result_stride]: the current result records
  const uint32_t* mark;          // touch marks (Resident in ctx.h)
  const Slot* slots;
  uint32_t n_slots;
  uint32_t n_records;            // state records scanned (the capacity)
  uint32_t n_runs;               // runs whose slot counts, and whose result record counts when a later tick may compare with it:
  uint32_t prev_runs;            //   run r < prev_runs (the changed-only baseline), or
  uint32_t eval_runs;            //   run r < eval_runs (the touched baseline) not marked "must list" after full_epoch
  uint32_t full_epoch;
  bf_layout L;                   // the batch's layout
  bf_layout R;                   // L with the result fields that do not count set to BF_OFF_NONE
  unsigned long long* out;       // [3], zeroed by the caller: steps, child nibbles (both extent << 32 | ~index), BF_F_* input fields
  const unsigned long long* timers;   // [n_records][timer_k] timer slots, or nullptr: an armed step s counts s + 1, a non-PENDING
  uint32_t timer_k;                   //   code BF_F_DECISION
};

// bf_resident_transfer (resident.cu): runs[i] of the source batch (layout F) is checked against the destination layout T
// (transfer_fit), then re-laid into destination record dst_first + i (transfer_runs).  The source's compaction is retire_runs.
struct TransferParams {
  const uint8_t* src_state;
  const uint8_t* src_result;     // the source's current result records
  const uint32_t* src_mark;
  uint8_t* dst_state;
  uint8_t* dst_result;
  uint32_t* dst_mark;            // an arrival's becomes mark_value (touched and must be listed)
  uint32_t mark_value;
  const uint32_t* runs;          // [n] source indices
  uint32_t n, dst_first;
  const Slot* slots;
  uint32_t n_slots;
  uint32_t prev_runs, eval_runs, full_epoch;   // the source's baselines: which result records count (ExtentParams)
  bf_layout F, T;
  bf_layout R;                   // F with the result fields T lacks set to BF_OFF_NONE
  uint4* extent;                 // [n] out: steps, child nibbles, BF_F_* input fields of each run
  uint32_t* unfit;               // [1] the lowest i that T cannot hold (atomicMin; 0xFFFFFFFF from the caller)
  const unsigned long long* src_timers;   // [src capacity][src_k] or nullptr
  unsigned long long* dst_timers;         // [dst capacity][dst_k] or nullptr: an arrival's armed slots, the rest empty
  uint32_t src_k, dst_k;                  // a run with more armed slots than dst_k is unfit
  const bf_sched_run* src_sched_in;       // limiter inputs, or nullptr (an arrival gets kSchedDefault)
  bf_sched_run* dst_sched_in;             // or nullptr: the destination has no area (then neither has the source)
  uint8_t* dst_sched_rec;                 // [dst capacity][dst_sched_stride]: an arrival has no baseline
  uint32_t dst_sched_stride;
  const bf_run_ctl* src_runctl;           // run-control records, or nullptr (an arrival gets kRunCtlDefault)
  bf_run_ctl* dst_runctl;                 // or nullptr: a run whose record is not the default is unfit (extent.w bit 31)
};

// step timers (resident.cu): slot = deadline | step << 32 | code << 48 (bf_timer_slot read as one little-endian u64); an empty
// slot is kTimerEmpty.  A run's armed slots come first, ascending by step.
constexpr unsigned long long kTimerEmpty = 0xFFFFFFFFull;
__host__ __device__ inline uint32_t timer_deadline(unsigned long long v) { return (uint32_t)v; }
__host__ __device__ inline uint32_t timer_step(unsigned long long v) { return (uint32_t)(v >> 32) & 0xFFFFu; }
__host__ __device__ inline uint32_t timer_code(unsigned long long v) { return (uint32_t)(v >> 48) & 0xFFu; }
__host__ __device__ inline bool timer_armed(unsigned long long v) { return (uint32_t)v != 0xFFFFFFFFu; }

// bf_resident_timers / _reshape: run r < n of the new area gets the first min(src_k, dst_k) slots of run r of the old one (when
// r < n_src), the rest empty
struct TimerRelayParams {
  const unsigned long long* src;   // or nullptr: every slot empty
  unsigned long long* dst;
  uint32_t n, n_src, src_k, dst_k;
};

// bf_resident_timers_arm: requests sorted by (run, step), grouped by run.  Group g is requests [first[g], first[g + 1]) of
// run run[g]; arm_before[j] is the number of arming (not cancelling) requests of j's group before j.
struct TimerArmParams {
  unsigned long long* timers;
  uint32_t timer_k;
  const bf_timer* req;
  const uint32_t* first;           // [n_groups + 1]
  const uint32_t* arm_before;      // [n]
  uint32_t n_groups;
  uint32_t* overflow;              // [1] lowest group whose run would hold more than timer_k armed slots (atomicMin)
};

// bf_resident_fire: one thread per run, a warp per chunk of 32 runs
struct FireParams {
  uint8_t* state;
  unsigned long long* timers;
  uint32_t* mark;                  // a run whose code was written is raised to mark_value, as by a delta
  uint32_t mark_value;
  uint32_t n_runs, timer_k, now;
  uint32_t words, state_stride, off_phase, off_decision;
  uint32_t* block_sums;            // [blocks] fired timers per block (fire_count), read by fire_apply for its offsets
  uint32_t* out;                   // [4] n_fired, n_written, n_pruned, next_deadline (fire_count initialises them)
  bf_fired* fired;                 // [fired_cap]
  uint32_t fired_cap;
  bf_run_ctl* runctl;              // [n_runs] run-control records, or nullptr: no story or drain deadlines (timers must be set)
  bf_sched_run* sched_in;          // limiter inputs, or nullptr: a story timeout sets its run's run_phase to BF_PHASE_TIMEOUT
};

// limiters.cu (rows a9 / f4)
struct SchedParams {
  const uint8_t* state;
  const uint8_t* result;
  const Slot* slots;
  const bf_sched_run* runs;
  uint8_t* records;            // [n_runs][stride]
  uint32_t* story_running;     // totals (pre-loaded with the base counts)
  uint32_t* queue_running;
  int32_t* queue_maxprio;      // pre-loaded with INT32_MIN
  uint32_t* global_running;
  const int32_t* story_limit;
  const int32_t* queue_limit;
  const int32_t* queue_aging;
  const uint32_t* story_base;  // StepRuns the batch does not hold, or nullptr
  const uint32_t* queue_base;
  const int32_t* queue_maxprio_base;  // highest effective priority among runs with demand OUTSIDE the batch, or nullptr
  uint32_t global_base;
  int32_t global_limit;
  uint32_t n_stories, n_queues, n_slots, n_runs;
  uint32_t words, state_stride, off_phase, off_child, child_nibbles, result_stride, off_ready, stride;
  uint32_t now;                // BF_SCHED_NONE: runs[r].queued_elapsed_s holds the elapsed time; else its queue origin
};

// the phases of launch_schedule (limiters.cu): the totals' start, the counting into them, the truncation against them
enum : uint32_t { kSchedInit = 1, kSchedCount = 2, kSchedApply = 4, kSchedTotals = kSchedInit | kSchedCount };

// The limiter inputs of a run never put (bf_resident_sched): no keys, priority 0, nothing queued, phase 0
constexpr bf_sched_run kSchedDefault = {BF_SCHED_NONE, BF_SCHED_NONE, 0, BF_SCHED_NONE, 0, {0u, 0u, 0u}};
// The reason word of a stored schedule record whose run has no baseline: no limiter writes it, so every new record differs
constexpr uint32_t kSchedNoBase = 0xFFFFFFFFu;

// bf_resident_schedule, per part (limiters.cu): S holds the part's batch (state, current result, inputs area as runs, the now of
// the call) and the shared tables and totals; S.records is the batch's schedule-record area, compared and overwritten in place.
// Runs are taken in CTAs of 256 (8 warps of 32 consecutive runs), the same partition in both launches.
struct ResSchedParams {
  SchedParams S;
  uint32_t base_runs;              // the previous schedule's n_runs: runs at or above it have no baseline
  uint32_t* run_events;            // [n_runs] events of a listed run, kSchedUnlisted for the others (sched_limit_runs)
  uint32_t* cta_listed;            // [CTAs] listed runs per CTA, then (sched_scan_ctas) those of the CTAs before it
  unsigned long long* cta_events;  // [CTAs] their events, likewise
  unsigned long long* totals;      // [2] out: n_listed, n_events (written by the last CTA of sched_list_runs)
  uint32_t* runs;                  // [runs_cap]
  bf_sched_header* heads;          // [runs_cap]
  uint16_t* events;                // [events_cap]
  uint32_t runs_cap;
  unsigned long long events_cap;
};
constexpr uint32_t kSchedUnlisted = 0xFFFFFFFFu;

// run control (resident.cu): the record of a run never put, and the run_flags byte of a stopped run
constexpr bf_run_ctl kRunCtlDefault = {0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u, {0u, 0u, 0u, 0u, 0u, 0u}};
constexpr uint32_t kStoppedFlags = BF_RF_HOST_GROUP | (uint32_t)BF_GROUP_DONE << BF_RF_HOST_GROUP_SHIFT;

// What a stop needs besides the record and its run-control record: the batch's timer slots (emptied), its limiter inputs (a
// timeout's run_phase), its touch marks (touched as by a delta).  Each may be nullptr but mark.
struct StopParams {
  unsigned long long* timers;
  uint32_t timer_k;
  bf_sched_run* sched_in;
  uint32_t* mark;
  uint32_t mark_value;
};

// bf_resident_runctl_put: req[i] is written into area[req[i].run], and a request with a stop stops its run (record r of state)
struct RunCtlPutParams {
  bf_run_ctl* area;
  const bf_run_ctl_put* req;
  uint32_t n;
  uint8_t* state;
  uint32_t state_stride;
  StopParams stop;
};

// bf_resident_upload of a batch with run control: every stopped run of [first, first + n) saves its uploaded flags byte and is
// stopped again
struct RunCtlRestopParams {
  bf_run_ctl* area;
  uint8_t* state;
  uint32_t state_stride, first, n;
};

// bf_resident_commit (resident.cu): commit_check over runs [0, n_runs) lowers *offender, then commit_apply writes the records.
// Entries are sorted by (run, step).  The offender key is run << 32 | step << 8 | reason (kCommitNotLaunched, ...).
enum : uint32_t { kCommitNotLaunched = 1, kCommitNotStop = 2, kCommitNoPhase = 3 };
struct CommitParams {
  uint8_t* state;
  const uint8_t* result;         // the current result records
  const uint8_t* sched_rec;      // [n_runs][sched_stride] the last schedule records, or nullptr: launched = ready, nothing queued
  const Slot* slots;
  uint32_t n_slots;
  const bf_commit_entry* entries;   // [n_entries], ascending by (run, step)
  uint32_t n_entries;
  uint32_t n_runs;
  uint32_t words, state_stride, off_phase, result_stride, off_ready, off_skip, off_fail, sched_stride;
  uint32_t* mark;                // a written run's is raised to mark_value, as by a delta
  uint32_t mark_value;
  unsigned long long* offender;  // [1] commit_check: lowest key (atomicMin; ~0 from the caller)
  uint32_t* counts;              // [5] commit_apply: runs written, skipped, launched, queued, failed (zeroed by the caller)
};

// bf_resident_sched_put: req[i] is written into area[req[i].run]
struct SchedPutParams {
  bf_sched_run* area;
  const bf_sched_put* req;
  uint32_t n;
};

}  // namespace bf
