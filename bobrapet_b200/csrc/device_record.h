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

#include "retire_moves.h"   // kRetireNoMove

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
// A resident batch's per-run side areas (RunAreas in ctx.h), as the launches that move, re-key or reset runs see them.  An
// absent area is nullptr (and timer_k 0); sched_rec is present exactly when sched_in is.
struct RunAreasView {
  unsigned long long* timers;    // [capacity][timer_k] step-timer slots (bf_timer_slot)
  uint32_t timer_k;
  bf_sched_run* sched_in;        // [capacity] limiter inputs
  uint8_t* sched_rec;            // [capacity][sched_stride] the last schedule records (reason kSchedNoBase: no baseline)
  uint32_t sched_stride;
  bf_run_ctl* runctl;            // [capacity] run-control records
};

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
  RunAreasView areas;            // a migrated run's timer slots are re-keyed through fwd, and its schedule record has no baseline
  const uint16_t* fwd;           // [n_old_steps] the step map (new index of old step i, or BF_MIGRATE_GONE), for the timers
  uint32_t n_old_steps;
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
  RunAreasView areas;            // an applied request empties its run's timer slots and lifts its stop
};

// bf_resident_reshape (resident.cu): both record arrays re-laid from layout `from` into new buffers at layout `to`
struct ReshapeParams {
  const uint8_t* old_state;
  const uint8_t* old_result;
  uint8_t* state;                // [n_new][to.state_stride]
  uint8_t* result;               // [n_new][to.result_stride]
  uint32_t n_old, n_new;         // runs r >= n_old get zero records
  bf_layout from, to;
  RunAreasView old_areas;        // areas holds the limiter inputs and run control of a new capacity, or none: runs r < n_old keep
  RunAreasView areas;            // theirs, the others get the defaults (its timers and schedule records are filled by the host)
};

// bf_resident_retire (resident.cu): the runs [m, m + n) vacate their indices; the live ones among them move below m
struct RetireParams {
  uint8_t* state;
  uint8_t* result;               // the current result records
  uint32_t* mark;                // touch marks: a target's becomes mark_value (touched and must be listed), a vacated one 0
  uint32_t mark_value;
  const uint32_t* to;            // [n] the new index of run m + i, or kRetireNoMove for a retired run
  uint32_t m, n;
  uint32_t state_stride, result_stride;   // multiples of 16
  RunAreasView areas;            // a mover's entries move with it (its target has no schedule baseline), vacated ones are reset
};

// bf_resident_extent / _narrow (resident.cu): the smallest layout a batch's records and the topologies of its runs allow.  Each
// extent is reduced into out[] as extent << 32 | ~index, so that one 64-bit atomicMax keeps the largest extent and the lowest
// index that needs it.
// The batch whose runs' extents are taken (extent_runs, transfer_fit): a run's state record and timer slots always count (an armed
// step s needs s + 1 steps, a non-PENDING code BF_F_DECISION); its result record counts when a later tick may compare with it.
struct ExtentBatch {
  const uint8_t* state;          // [capacity][L.state_stride]
  const uint8_t* result;         // [capacity][L.result_stride]: the current result records
  const uint32_t* mark;          // touch marks (Resident in ctx.h)
  RunAreasView areas;
  const Slot* slots;
  uint32_t n_slots;
  uint32_t prev_runs;            // a result record counts for run r < prev_runs (the changed-only baseline), or for
  uint32_t eval_runs;            //   run r < eval_runs (the touched baseline) not marked "must list" after full_epoch
  uint32_t full_epoch;
  bf_layout L;                   // the batch's layout
  bf_layout R;                   // L with the result fields that do not count set to BF_OFF_NONE
};

struct ExtentParams {
  ExtentBatch B;
  uint32_t n_records;            // state records scanned (the capacity)
  uint32_t n_runs;               // runs whose slot and result record count
  unsigned long long* out;       // [3], zeroed by the caller: steps, child nibbles (both extent << 32 | ~index), BF_F_* input fields
};

// bf_resident_transfer (resident.cu): runs[i] of the source batch (layout src.L) is checked against the destination layout T
// (transfer_fit), then re-laid into destination record dst_first + i (transfer_runs).  The source's compaction is retire_runs.
struct TransferParams {
  ExtentBatch src;               // src.R: the result fields T keeps
  uint8_t* dst_state;
  uint8_t* dst_result;
  uint32_t* dst_mark;            // an arrival's becomes mark_value (touched and must be listed)
  uint32_t mark_value;
  RunAreasView dst_areas;        // an arrival's entries, or the defaults where the source has no area.  A run with more armed slots
                                 // than dst_areas.timer_k, or with run control other than the default and no area here, is unfit
  const uint32_t* runs;          // [n] source indices
  uint32_t n, dst_first;
  bf_layout T;
  uint4* extent;                 // [n] out: steps, child nibbles, BF_F_* input fields, armed slots | 1 << 31 for lost run control
  uint32_t* unfit;               // [1] the lowest i that T cannot hold (atomicMin; 0xFFFFFFFF from the caller)
};

// bf_resident_transfer_ctx (resident.cu): runs[i] of the source batch is packed into staged run i, in the source layout (gather_runs).
// The staging, copied to the destination ctx, is the source view of transfer_fit and transfer_runs there: its state records carry
// the destination slot, ident[i] = i stands for runs, and mark[i] is 0 when the run's result record is a baseline of the source
// (run_extent's rule) and 3 (must list after epoch 0) when not, for an ExtentBatch with prev_runs 0, eval_runs n, full_epoch 0.
// A run whose slot the map does not carry sets reason[i] (BF_UNFIT_SLOT_*) and lowers *unfit, which transfer_fit lowers further.
constexpr uint32_t kSlotDead = 0xFFFFFFFEu;   // slot_map entry of a slot that is not live in the source ctx
struct GatherParams {
  ExtentBatch src;               // the source batch, its baselines as transfer_fit would read them
  const uint32_t* runs;          // [n] source indices
  uint32_t n;
  const uint32_t* slot_map;      // [n_slot_map] destination slot, BF_SLOT_NONE or kSlotDead
  uint32_t n_slot_map;
  uint32_t* unfit;               // [1] BF_EXTENT_NO_RUN from the caller
  uint32_t* reason;              // [n]
  uint32_t* ident;               // [n]
  uint32_t* mark;                // [n]
  uint8_t* state;                // [n][src.L.state_stride]
  uint8_t* result;               // [n][src.L.result_stride]
  RunAreasView areas;            // [n] entries of each area the source has (sched_rec unused)
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
  RunAreasView areas;              // timer slots; run control, or none: no story or drain deadlines (then timers are set); limiter
                                   // inputs, or none: a story timeout sets its run's run_phase to BF_PHASE_TIMEOUT
  uint32_t* mark;                  // a run whose code was written is raised to mark_value, as by a delta
  uint32_t mark_value;
  uint32_t n_runs, now;
  uint32_t words, state_stride, off_phase, off_decision;
  uint32_t* block_sums;            // [blocks] fired timers per block (fire_count), read by fire_apply for its offsets
  uint32_t* out;                   // [4] n_fired, n_written, n_pruned, next_deadline (fire_count initialises them)
  bf_fired* fired;                 // [fired_cap]
  uint32_t fired_cap;
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
  unsigned long long* cta;         // [2][CTAs] listed runs and events of each CTA, then (cta_scan) of the CTAs before it
  unsigned long long* totals;      // [2] out: n_listed, n_events (cta_scan)
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
// timeout's run_phase), its touch marks (touched as by a delta).
struct StopParams {
  RunAreasView areas;
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
// Entries are sorted by (run, step).  The offender key is run << 32 | step << 8 | reason (kCommitNotLaunched, ...).  With a
// timing table (bf_resident_commit_timed) both launches also take the arms: the check adds kCommitNoDecision and
// kCommitOverflow, the apply merges the new slots into the timer area.
enum : uint32_t { kCommitNotLaunched = 1, kCommitNotStop = 2, kCommitNoPhase = 3, kCommitNoDecision = 4, kCommitOverflow = 5 };
// the step timings of every topology slot (bf_topology_timings), one table: slot s has tim[first[s], first[s + 1]), ascending by step
struct CommitTimings {
  const bf_step_timing* tim;     // or nullptr: the commit arms nothing
  const uint32_t* first;         // [n_slots + 1]
  uint32_t n_slots;              // slots at or above it have no timings
  unsigned long long* timers;    // the batch's timer area, timer_k slots per run
  uint32_t timer_k, now;
  bool decision;                 // the layout has decision planes
  uint32_t* out;                 // [2] commit_apply: slots armed (atomicAdd), earliest deadline armed (atomicMin; NONE from the caller)
};
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
  CommitTimings arm;             // arm.tim = nullptr: no arming
  // bf_resident_commit_journal (the <true> builds of both launches): commit_check stores each run's journal word and each CTA's
  // items and written runs (cta: [2][CTAs]), cta_scan turns them into those of the CTAs before each and posts the sums
  // (total[2]), commit_apply writes each run's items and its entry in runs at those offsets
  uint32_t* run_items;           // [n_runs] items << 8 | new arms << 1 | written
  unsigned long long* cta;       // [2][CTAs] items and written runs of each CTA, then (cta_scan) of the CTAs before it
  unsigned long long* total;     // [2] items and written runs of the call
  bf_commit_write* items;        // [items_cap]
  unsigned long long items_cap;
  uint32_t* runs;                // [runs_cap]
  uint32_t runs_cap;
  // bf_resident_commit_rewrites (the rewriting builds of both launches): the writes of a run flagged in rw_runs start from its
  // codes after the stages G / H / I of a single pass, which rewrite_runs left in rw_planes; commit_apply adds the steps written
  // from them (no mask bit) to *rewritten
  const uint32_t* rw_runs;       // [n_runs] 1: the stages rewrote a code of the run, 0: its stored codes are the base
  const uint32_t* rw_planes;     // [n_runs][4][words] the phase planes after the stages (flagged runs only)
  uint32_t* rewritten;           // [1] steps written from the stages (zeroed by the caller)
};
static_assert(sizeof(bf_commit_write) == 16, "bf_commit_write must be 16 bytes");
constexpr uint32_t kJournalArmsShift = 1, kJournalItemsShift = 8;   // new arms <= BF_TIMER_MAX_SLOTS < 128

// bf_resident_commit_touched (resident.cu): the list-mode builds of the commit launches.  Warp i of the list takes run list[i]
// (list == nullptr: run i), i below *n_list; the launch's CTAs walk blocks of 8 list positions, so the journal's words and CTA
// totals are those of list positions, ceil(*n_list / 8) blocks of them.  The apply clears the commit-due bit of each run it
// takes that no entry names and sets the bit of one that an entry names.  A separate parameter block, so the full-form builds
// keep theirs.
struct CommitListParams {
  CommitParams P;
  const uint32_t* list;                 // [*n_list] ascending runs, or nullptr: [0, *n_list)
  const unsigned long long* n_list;     // [1] the list length (the list build's scan, or uploaded)
  uint32_t* due;                        // [ceil(capacity / 32)] the batch's commit-due bits (apply)
};
// The run list of a touched commit (launch_listing over groups of 32 due words, one warp per group and lane w on word w): the
// due bits of [0, n_runs) and the runs the entries name.  due_count stores each group's runs (group_runs) and each CTA's total,
// cta_scan<1> turns those into the runs of the CTAs before each and posts the list length (total), due_list writes the runs.
struct DueListParams {
  const uint32_t* due;
  const bf_commit_entry* entries;       // [n_entries], ascending by (run, step)
  uint32_t n_entries, n_runs;
  uint32_t n, warps_per_block;          // groups (launch_listing's runs) and 8
  uint32_t* group_runs;                 // [n]
  unsigned long long* cta;              // [CTAs]
  unsigned long long* total;            // [1] out: the list length
  uint32_t* list;                       // [n_runs] out
};

// bf_resident_commit_rewrites (resident.cu): rewrite_runs, one warp per run of [0, n_runs) and the shared stage of StatusParams,
// takes a run through the stages of a single pass when its current result record carries BF_SUM_PHASE_CHANGED, it is not stopped
// and its slot is live and fits the layout; a run whose codes the stages changed is flagged in rw_runs and its planes stored in
// rw_planes, every other run is flagged 0.
struct RewriteParams {
  const uint8_t* state;
  const uint8_t* result;            // the current result records (their summary word)
  const Slot* slots;
  uint32_t n_slots;
  const bf_run_ctl* runctl;         // or nullptr: no run is stopped
  uint32_t n_runs, warps_per_block;
  uint32_t words, state_stride, off_phase, off_decision, off_child, topo_bytes, result_stride;
  uint32_t* rw_runs;                // [n_runs]
  uint32_t* rw_planes;              // [n_runs][4][words]
};

// bf_resident_status (resident.cu): one warp per listed run.  status_runs<false> stores each listed run's event count and each
// CTA's total, cta_scan turns the CTA totals into the events of the CTAs before each and posts the sum, status_runs<true> writes
// the records and the events.
static_assert(sizeof(bf_status_rec) == 32, "bf_status_rec must be 32 bytes");
// The single-pass launches (status_runs, resync_runs, rewrite_runs): their static shared memory (one word per warp,
// store_cta_totals), beside the warps' shared stages.  With a child area each warp has a stage for stage H: the state record,
// the topology record (topo_bytes: the largest record the layout fits) and 256 scratch bytes; without one, none.
constexpr uint32_t kStatusStaticSmem = 32;
__host__ __device__ inline uint32_t pass_stage_bytes(uint32_t off_child, uint32_t state_stride, uint32_t topo_bytes) {
  return off_child != BF_OFF_NONE ? state_stride + topo_bytes + 256u : 0u;
}
struct StatusParams {
  const uint8_t* state;
  const Slot* slots;
  uint32_t n_slots;
  const bf_run_ctl* runctl;         // or nullptr: no run is stopped
  const uint32_t* runs;             // [n] ascending, or nullptr: listed run i is run i
  uint32_t n, warps_per_block;
  uint32_t words, state_stride, off_phase, off_decision, off_child, topo_bytes;
  uint32_t* run_events;             // [n] events of each listed run (status_runs<false>)
  unsigned long long* cta;          // [CTAs] events of each CTA, then (cta_scan) of the CTAs before it
  unsigned long long* total;        // [1] events of the call (cta_scan)
  bf_status_rec* records;           // [n]
  uint16_t* events;                 // [events_cap]
  unsigned long long events_cap;
};

// bf_resident_resync (resident.cu): one warp per listed run, the shared stage of StatusParams.  resync_runs<false> stores each
// listed run's item count and each CTA's items and drifted runs (cta: [2][CTAs]), cta_scan turns them into the items and drifted
// runs of the CTAs before each and posts the sums (total[2]), resync_runs<true> visits the runs with items: their items, their
// drifted entries and, unless check, their repair.
static_assert(sizeof(bf_drift) == 16, "bf_drift must be 16 bytes");
struct ResyncParams {
  uint8_t* state;
  const Slot* slots;
  uint32_t n_slots;
  bf_run_ctl* runctl;               // or nullptr: no run is stopped
  RunAreasView areas;               // a slot-drifted run's schedule baseline is dropped
  uint32_t* mark;
  uint32_t mark_touched, mark_must_list;
  const uint32_t* runs;             // [n] ascending, or nullptr: listed run i is run i
  const uint8_t* records;           // [n] the caller's records, list order
  uint32_t n, warps_per_block;
  uint32_t words, state_stride, off_phase, off_cond, off_decision, off_child, child_nibbles, topo_bytes;
  uint32_t fields;                  // BF_RESYNC_FIELD bits of the fields the layout places
  bool check;
  uint32_t* run_items;              // [n] items of each listed run
  unsigned long long* cta;          // [2][CTAs] items and drifted runs of each CTA, then (cta_scan) of the CTAs before it
  unsigned long long* total;        // [2] items and drifted runs of the call
  uint32_t* drifted;                // [drifted_cap]
  uint32_t drifted_cap;
  bf_drift* items;                  // [items_cap]
  unsigned long long items_cap;
};

// bf_resident_resync_areas (resident.cu): one warp per listed run, no shared stage.  resync_area_runs<false> stores each listed
// run's item count and each CTA's items and drifted runs, cta_scan turns them into those of the CTAs before each and posts the sums
// (total[0..1]), resync_area_runs<true> visits the runs with items: their items, their drifted entries and, unless check, their
// repair, adding the runs written and the runs stopped to total[2] and total[3] (zeroed by the count launch).
static_assert(sizeof(bf_timer_slot) == 8 && sizeof(bf_sched_put) == 32 && sizeof(bf_run_ctl) == 16, "resync area rows");
struct ResyncAreasParams {
  uint8_t* state;
  RunAreasView areas;               // the device's areas; those the call selects are present
  uint32_t* mark;                   // a run the repair stops is raised to mark_touched, as by a delta
  uint32_t mark_touched;
  const uint32_t* runs;             // [n] ascending, or nullptr: listed run i is run i
  const unsigned long long* timers; // [n][areas.timer_k] the caller's slots, list order (TIMERS selected)
  const bf_sched_put* sched;        // [n] (SCHED selected)
  const bf_run_ctl* runctl;         // [n] (RUNCTL selected)
  uint32_t n, warps_per_block;
  uint32_t words, state_stride, off_phase, off_decision;
  uint32_t sel;                     // BF_RESYNC_AREA_* bits
  uint32_t fired_now;
  bool check;
  uint32_t* run_items;              // [n] items of each listed run
  unsigned long long* cta;          // [2][CTAs] items and drifted runs of each CTA, then (cta_scan) of the CTAs before it
  unsigned long long* total;        // [4] items, drifted runs, written runs, stopped runs
  uint32_t* drifted;                // [drifted_cap]
  uint32_t drifted_cap;
  bf_drift* items;                  // [items_cap]
  unsigned long long items_cap;
};

// bf_resident_sched_put: req[i] is written into area[req[i].run]
struct SchedPutParams {
  bf_sched_run* area;
  const bf_sched_put* req;
  uint32_t n;
};

}  // namespace bf
