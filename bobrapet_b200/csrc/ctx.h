// ctx.h — what the C ABI's translation units share (abi.cu: context, batch evaluation, limiters; topology.cu: topology
// arena; resident_abi.cu: resident batches; group.cu: device groups): bf_ctx and the records it keeps, the device-buffer
// owner, the error helpers, the kernel launchers and the host helpers of a pass.  Private to the library:
// include/bobrafrontier.h is the public surface.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "../../include/bobrafrontier.h"
#include "device_record.h"

namespace bf {
cudaError_t launch_frontier(const KParams& P, uint32_t grid, uint32_t smem_bytes, cudaStream_t stream);
cudaError_t launch_expansion(const KParams& P, unsigned long long* block_sums, unsigned long long* offsets,
                             bf_expansion* out, unsigned long long cap, cudaStream_t stream, uint32_t* launches);
int frontier_max_blocks_per_sm(const KParams& P, uint32_t threads, uint32_t smem_bytes, uint32_t* occ2);
cudaError_t launch_frontier_pack(const KParams& P, uint32_t grid, uint32_t smem_bytes, cudaStream_t stream);
uint32_t frontier_pack_max_warps();
cudaError_t launch_apply_deltas(const DeltaParams& P, cudaStream_t stream);
cudaError_t launch_compact(const CompactParams& P, cudaStream_t stream);
cudaError_t launch_touched_list(const TouchedParams& P, cudaStream_t stream);
cudaError_t launch_touched_compact(const TouchedParams& P, cudaStream_t stream);
cudaError_t launch_apply_deltas_many(const DeltaParams* parts, const uint32_t* first, uint32_t n_parts, uint32_t n, cudaStream_t stream);
cudaError_t launch_touched_list_many(const TouchedParams* T, const uint32_t* list_first, uint32_t n, uint32_t blocks, cudaStream_t stream);
cudaError_t launch_touched_compact_many(const TouchedParams* T, const uint32_t* compact_first, uint32_t n, uint32_t blocks,
                                        cudaStream_t stream);
cudaError_t launch_mark_runs(uint32_t* mark, uint32_t first, uint32_t n, uint32_t value, cudaStream_t stream);
cudaError_t launch_move_records(const uint8_t* src, uint8_t* dst, const void* moves, uint32_t n, cudaStream_t stream);
cudaError_t launch_migrate(const MigrateParams& P, cudaStream_t stream);
cudaError_t launch_redrive(const RedriveParams& P, cudaStream_t stream);
cudaError_t launch_reshape(const ReshapeParams& P, cudaStream_t stream);
cudaError_t launch_retire(const RetireParams& P, cudaStream_t stream);
cudaError_t launch_extent(const ExtentParams& P, uint32_t sm_count, cudaStream_t stream);
cudaError_t launch_transfer_fit(const TransferParams& P, cudaStream_t stream);
cudaError_t launch_transfer(const TransferParams& P, cudaStream_t stream);
cudaError_t launch_gather(const GatherParams& P, cudaStream_t stream);
cudaError_t launch_relay_timers(const TimerRelayParams& P, cudaStream_t stream);
cudaError_t launch_arm_timers(const TimerArmParams& P, bool merge, cudaStream_t stream);
cudaError_t launch_fire(const FireParams& P, cudaStream_t stream);
cudaError_t launch_schedule(const SchedParams& P, uint32_t sm_count, cudaStream_t stream, uint32_t phases = kSchedTotals | kSchedApply);
cudaError_t launch_resident_schedule(const ResSchedParams& R, cudaStream_t stream);
cudaError_t launch_sched_put(const SchedPutParams& P, cudaStream_t stream);
cudaError_t launch_runctl_put(const RunCtlPutParams& P, cudaStream_t stream);
cudaError_t launch_runctl_restop(const RunCtlRestopParams& P, cudaStream_t stream);
cudaError_t launch_commit(const CommitParams& P, bool apply, cudaStream_t stream);
cudaError_t launch_status(const StatusParams& P, uint32_t smem_bytes, cudaStream_t stream);
cudaError_t launch_rewrites(const RewriteParams& P, uint32_t smem_bytes, cudaStream_t stream);
cudaError_t launch_commit_list(const CommitListParams& L, bool apply, uint32_t max_n, uint32_t ctas, cudaStream_t stream);
cudaError_t launch_rewrites_list(const RewriteParams& P, const uint32_t* list, const unsigned long long* n_list, uint32_t ctas,
                                 uint32_t smem_bytes, cudaStream_t stream);
cudaError_t launch_due_list(const DueListParams& D, cudaStream_t stream);
cudaError_t launch_due_mark_list(uint32_t* due, const uint32_t* list, const uint32_t* count, uint32_t bound, uint32_t ctas,
                                 cudaStream_t stream);
cudaError_t launch_due_mark_sched(uint32_t* due, const uint32_t* run_events, uint32_t n_runs, cudaStream_t stream);
cudaError_t launch_resync(const ResyncParams& P, uint32_t smem_bytes, cudaStream_t stream);
cudaError_t launch_resync_areas(const ResyncAreasParams& P, cudaStream_t stream);
cudaError_t launch_closure(const Slot* slots, const uint32_t* slot_ids, const uint32_t* starts, uint32_t n, uint32_t n_slots,
                           uint32_t words_out, uint32_t* masks, cudaStream_t stream);
cudaError_t launch_validate(const Slot* slots, const uint32_t* slot_ids, uint32_t n, uint32_t n_slots, uint32_t* status,
                            cudaStream_t stream);

inline uint32_t round_up(uint32_t v, uint32_t a) { return (v + a - 1) / a * a; }
inline size_t round_up_sz(size_t v, size_t a) { return (v + a - 1) / a * a; }
inline int fail(bf_ctx* c, int code, const std::string& msg);

// The launch-shape knobs of a pass (A/B timing and the launch-shape tests, DESIGN.md), read at the start of every pass so
// that a changed knob takes effect on the same ctx.  A number that is unset, 0 or not a number is 0: the planner's choice.
struct Knobs {
  bool general = false;    // BF_KERNEL=general: the one-run-per-warp kernel for every pass
  bool blocked = false;    // BF_ASSIGN=blocked: each CTA takes a block of consecutive runs (KParams::run_blocked)
  int warps = 0;           // BF_WARPS: warps per CTA of the packed-lanes kernel, else of the general kernel alone
  int groups = 0;          // BF_GROUPS: slot groups of the packed-lanes ring (taken when it fits)
  int stages = 0;          // BF_STAGES: ring stages of the general kernel
  int blocks_per_sm = 0;   // BF_BLOCKS_PER_SM: at most this many general-kernel CTAs per SM
  int wq = 0;              // BF_WQ: at least this many lanes per run in the packed-lanes kernel
  int pack_ctas = 0;       // BF_PACK_CTAS: packed-lanes CTAs per SM, 1..4 (a build with -DPACK_MIN_BLOCKS; else 1)
  auto tie() const { return std::tie(general, blocked, warps, groups, stages, blocks_per_sm, wq, pack_ctas); }
  bool operator==(const Knobs& o) const { return tie() == o.tie(); }
};

// A compact tick's head words and per-block event totals, offered to its pass: a packed-lanes pass may write them itself
// (device_record.h) and then sets done, so that the compaction skips its head kernel
struct FusedHeads {
  uint32_t* head;
  unsigned long long* sums;
  bool done;
};
}  // namespace bf

// The owner of one device allocation: a pointer and a capacity in elements, freed by the destructor.  It converts to its
// pointer, so kernel parameters and address arithmetic read it as a plain T*.
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;

  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { reset(); p = std::exchange(o.p, nullptr); cap = std::exchange(o.cap, 0); }
    return *this;
  }
  ~DevBuf() { reset(); }

  operator T*() const { return p; }
  void reset() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  // Exactly n elements, which replace the old ones once they exist (no old contents kept).  A failed allocation changes
  // nothing and clears the error it left behind: an allocation failure is not a launch failure of the next call.
  cudaError_t alloc(size_t n) {
    T* np = nullptr;
    const cudaError_t e = cudaMalloc(&np, n * sizeof(T));
    if (e != cudaSuccess) { cudaGetLastError(); return e; }
    reset();
    p = np; cap = n;
    return e;
  }
  // At least n elements: doubles from the current capacity (or 1).  BF_ENOMEM on failure.
  int ensure(bf_ctx* c, size_t n) {
    if (n <= cap) return BF_OK;
    size_t ncap = cap ? cap : 1;
    while (ncap < n) ncap *= 2;
    const cudaError_t e = alloc(ncap);
    return e == cudaSuccess ? BF_OK : bf::fail(c, BF_ENOMEM, std::string("cudaMalloc: ") + cudaGetErrorString(e));
  }
};

struct Resident;

// The device scratch of one touched tick: [0] = list length, [1..] = the list | head word per list position | listed runs and
// their heads (when the caller's buffers are not pinned) | per-block sums | the event list (bf_resident_tick_touched_many's
// pageable event buffers; the single call stages them in bf_ctx::d_events)
struct TouchScratch {
  DevBuf<uint32_t> list, pos_head, runs, head;
  DevBuf<unsigned long long> sums;
  DevBuf<uint16_t> events;
};

struct TopoMeta {
  bool alive = false;
  uint32_t S = 0, E = 0, P = 0, bytes = 0;
  size_t offset = 0;  // in arena
  std::vector<uint32_t> child_first;
  std::vector<uint16_t> par_step, par_branches;   // step and branch count of each parallel desc (bf_resident_migrate)
  uint32_t child_nibbles = 0;
  std::vector<uint8_t> types;            // BF_STEP_* of each step (bf_topology_timings checks the codes against them)
  std::vector<bf_step_timing> timings;   // bf_topology_timings, ascending by step
  bool fits(const bf_layout& L) const { return S <= L.steps_max && (L.off_child == BF_OFF_NONE || child_nibbles <= L.child_nibbles); }
};

struct bf_ctx {
  int device = 0;
  int sm_count = 0;                    // SMs the frontier kernels spread over (device SMs minus the reserved ones)
  cudaStream_t stream = nullptr;
  // the chunked pipeline that bf_eval and the full resident ticks share (abi.cu): H2D copies (bf_eval only), kernels and D2H
  // copies of consecutive run chunks overlap on three streams
  static constexpr uint32_t kMaxChunks = 32;
  cudaStream_t s_in = nullptr, s_out = nullptr;
  cudaEvent_t ev_in[kMaxChunks] = {}, ev_k[kMaxChunks] = {};
  bool pipe_ready = false;
  std::mutex mu;
  std::string err;

  DevBuf<uint8_t> arena;               // capacity: arena.cap bytes
  size_t arena_used = 0;
  size_t arena_dead = 0;               // bytes of dropped records below arena_used (reclaimed by compact_arena)
  uint64_t arena_compactions = 0;
  std::vector<TopoMeta> meta;
  std::vector<uint32_t> free_slots;
  std::vector<bf::Slot> slots_host;
  DevBuf<bf::Slot> slots_dev;
  bool slots_dirty = true;
  std::vector<uint32_t> ff_host;       // cut table (fail-fast masks, dependency floors), bf::FF_STRIDE words per slot (device_record.h), mirrored with the slots
  DevBuf<uint32_t> ff_dev;             // capacity: slots_dev.cap rows
  uint32_t max_rec_by_w[33] = {};      // largest live record among the topologies of W = ceil(S/32) words (bf::largest_record)
  bool rec_max_dirty = false;          // a drop may have lowered the maxima: recomputed at the next plan
  uint32_t n_alive = 0;
  uint32_t n_with_parallel = 0;  // live topologies that have parallel steps
  uint64_t slot_changes = 0;     // slot drops and reuses so far: either changes what the runs holding the slot evaluate
                                 // to, so a touched tick after one evaluates every run
  // step timings of every slot (bf_topology_timings) as one table, slot s at [tim_first[s], tim_first[s + 1]), built and copied
  // to the device by the first arming commit after a change (sync_timings); nothing is allocated until a slot has timings
  bool timings_dirty = false;
  uint64_t timing_changes = 0;   // timings calls and drops that changed a slot's timings: a touched commit after one that arms is full
  std::vector<uint32_t> tim_first_host;
  std::vector<bf_step_timing> tim_host;
  DevBuf<uint32_t> tim_first_dev;
  DevBuf<bf_step_timing> tim_dev;

  // host-API staging
  DevBuf<uint8_t> d_state, d_result;
  DevBuf<unsigned long long> d_counts;
  // BF_EVAL_COUNTS_SET scratch of the packed-lanes kernel (device_record.h): a ring of kAccSlots blocks of 8 u64, one per launch
  // in turn (launches of different streams may overlap; a block is left zeroed by the launch that used it)
  static constexpr uint32_t kAccSlots = 256;
  DevBuf<unsigned long long> d_acc;
  uint32_t acc_seq = 0;
  // where a pass's small results land on the host, pinned (a pageable target would make a copy synchronous)
  struct Pinned {
    uint32_t word;         // a 4-byte device counter: rejected deltas where no compaction delivers them, migrated runs
    bf::ResultTail tail;   // written by a compaction's last kernel; a pass without one copies its counts into tail.counts
    uint32_t fire[4];      // bf_resident_fire: n_fired, n_written, n_pruned, next_deadline
    uint32_t commit[8];    // bf_resident_commit: the offender key (two words), then the five counts
    // the totals of a call's lists: bf_resident_status its events; bf_resident_resync its items and drifted runs;
    // bf_resident_commit_journal its items and written runs; bf_resident_resync_areas its items, drifted, written and stopped runs
    // (every call holds the ctx lock, so they share the words)
    unsigned long long list_totals[4];
    bf_counts counts() const { return {tail.counts[0], tail.counts[1], tail.counts[2], tail.counts[3]}; }
  }* pinned = nullptr;
  DevBuf<bf_expansion> d_exp;
  // compact results (bf_eval_compact / bf_resident_tick_compact)
  DevBuf<uint32_t> d_head;
  DevBuf<uint16_t> d_events;
  // [0] = events, [1] = listed runs, then TWO buffers of per-512-run event totals used in turn: a tick's emit kernel leaves the
  // other one zeroed, so a pass that adds its runs' counts itself (fused heads, device_record.h) finds a clean buffer
  DevBuf<unsigned long long> d_cblock;
  uint32_t cblock_flip = 0;
  uint64_t last_events = 0;                                          // events of the previous compact pass (sizes the first D2H)
  // scratch shared by both entry points
  DevBuf<uint32_t> d_exp_counts;
  DevBuf<unsigned long long> d_offsets, d_block_sums;
  DevBuf<uint32_t> d_defer;  // [0] = count, [1..] = run ids
  // touched ticks: [0] for bf_resident_tick_touched, one per part for bf_resident_tick_touched_many (whose parts are all in
  // flight before its one synchronisation)
  std::vector<TouchScratch> touch = std::vector<TouchScratch>(1);
  uint64_t last_touched_events = 0;   // events of the previous touched tick (sizes the first D2H)
  // bf_resident_tick_touched_many: the small results of each part, pinned (the single call uses pinned->tail)
  bf::ResultTail* part_tails = nullptr;
  uint32_t part_tails_cap = 0;
  // bf_resident_schedule_ctxs: this ctx's own Running counts and queue priority maxima (phase 1), pinned
  uint32_t* span_totals = nullptr;
  size_t span_totals_cap = 0;
  // The device inputs and outputs of one resident call that is not a tick (migrate, redrive, retire, extent, narrow, transfer,
  // timers_arm, fire, sched_put, schedule, runctl_put, commit, status, resync), laid out by the call (CallStage, resident_abi.cu).  They are
  // valid from the call's staging until it returns: a call reads only bytes it uploaded, set or had a kernel write during the
  // same call, so every counter or sentinel word it reads is written by that call.  ensure only grows it, so the largest call
  // sizes it and a steady-state call allocates nothing.
  DevBuf<uint8_t> d_call;

  // limiters (bf_schedule): the records the last pass evaluated (bf_eval's staging or a resident batch), read in place.  Cleared
  // (valid = false) when a pass starts or a call changes those records (end_snapshot); assigned whole once a pass went through.
  struct Snapshot {
    bool valid = false;
    uint32_t n_runs = 0;
    bf_layout layout{};
    const uint8_t *state = nullptr, *result = nullptr;
    bool holds(const uint8_t* st) const { return valid && state == st; }
    bool matches(uint32_t n, const bf_layout& L) const { return valid && n_runs == n && memcmp(&layout, &L, sizeof L) == 0; }
  } snap;
  DevBuf<uint8_t> d_sched;                              // runs | records | tables, one allocation
  // resident batches (row f2)
  std::vector<Resident> resident;
  DevBuf<bf_delta> d_deltas;
  DevBuf<uint32_t> d_rejected;
  // small device scratch that its consumers leave zeroed (the compaction's tail block reads and clears the rejected-delta
  // counter and the listed-runs total), so the steady-state tick carries no memset launches; a failed call marks it dirty
  bool rejected_clean = false, cblock_clean = false;

  // cached shared-memory plans of the general kernel (recomputed when the layout, the largest record or a launch-shape knob
  // changes): [0] for passes over whole batches, [1] for passes over a run list (touched ticks), so that a batch that mixes
  // full and touched ticks keeps both
  struct Plan {
    uint32_t key_stride = 0, key_words = 0, key_rec = 0, key_variant = 0xFFFFFFFFu;
    bf::Knobs key_knobs;   // as last planned
    uint32_t stages = 0, wpb = 0, per_sm = 0, occ2 = 0, smem = 0;
  } plan[2];

  bf_stats stats{};
};

namespace bf {
inline int fail(bf_ctx* c, int code, const std::string& msg) {
  if (c) c->err = msg;
  return code;
}
inline int cuda_fail(bf_ctx* c, cudaError_t e, const char* what) {
  return fail(c, BF_ECUDA, std::string(what) + ": " + cudaGetErrorString(e));
}
// The synchronisation that ends a call, so that it never returns with work or copies into the caller's buffers in flight.  The
// first error, of the call's own work (e) or of the synchronisation, fails the call as `what`.
inline int end_call(bf_ctx* c, cudaError_t e, const char* what) {
  const cudaError_t es = cudaStreamSynchronize(c->stream);
  if (e == cudaSuccess) e = es;
  return e == cudaSuccess ? BF_OK : cuda_fail(c, e, what);
}
}  // namespace bf
#define BF_CUDA(c, call)                                       \
  do {                                                         \
    cudaError_t e__ = (call);                                  \
    if (e__ != cudaSuccess) return bf::cuda_fail(c, e__, #call); \
  } while (0)

// The per-run side areas of a resident batch, each with one entry per run of the capacity, or absent:
//   d_timers, timer_k  step-timer slots (bf_resident_timers): timer_k slots per run, or none (timer_k = 0).  Arm and fire change
//                      them.
//   d_sched_in         limiter inputs (bf_resident_sched), or none.  Put changes them.
//   d_sched_rec,       with the inputs: the records of the last bf_resident_schedule, BF_SCHED_STRIDE(words) bytes per run.  A run
//   sched_base_runs    at or above sched_base_runs, or whose stored reason is kSchedNoBase, has no baseline.
//   d_runctl           run-control records (bf_resident_runctl), or none.  Put and fire change them (a stop also rewrites the run's
//                      flags byte, empties its timers and, for a timeout, sets its inputs' run_phase); deltas, uploads and redrives
//                      honour them.
//   d_due              commit-due bits (bf_resident_commit_marks), one per run in words of 32, or none.  Touched ticks set the bits
//                      of the runs they evaluate, bf_resident_schedule those of the runs whose record changed, a touched commit
//                      clears those of the runs it considered that no entry named.  Bits at or past the capacity stay set.  Only
//                      ever too many bits cost anything (work, not results), so moves need not re-key them.
// The calls that move or reset runs carry every area in the launches that handle the records, through view() (resident.cu):
// retire and transfer move a run's entries with it and reset the ones it leaves, migrate re-keys its timers, redrive empties its
// timers and lifts its stop, and a run that is moved, migrated or uploaded has no schedule baseline.  Reshape and a retire to a
// new capacity allocate the areas anew (alloc_resized), fill them and adopt them; narrow keeps them (the capacity stays, and a
// smaller stride fits the schedule records).  A change of words drops every schedule baseline (Resident::adopt).
struct RunAreas {
  DevBuf<unsigned long long> d_timers;
  uint32_t timer_k = 0;
  DevBuf<bf_sched_run> d_sched_in;
  DevBuf<uint8_t> d_sched_rec;
  uint32_t sched_base_runs = 0;
  DevBuf<bf_run_ctl> d_runctl;
  DevBuf<uint32_t> d_due;

  static size_t due_words(uint32_t capacity) { return ((size_t)capacity + 31) / 32; }
  bf::RunAreasView view(uint32_t words) const {
    return {d_timers, timer_k, d_sched_in, d_sched_rec, BF_SCHED_STRIDE(words), d_runctl};
  }
  // schedule records for `capacity` runs of `words` words, every run without a baseline (all bytes 0xFF: reason kSchedNoBase)
  static cudaError_t alloc_sched_rec(DevBuf<uint8_t>& rec, uint32_t capacity, uint32_t words, cudaStream_t s) {
    const size_t bytes = (size_t)capacity * BF_SCHED_STRIDE(words);
    cudaError_t e = rec.alloc(bytes);
    return e == cudaSuccess ? cudaMemsetAsync(rec, 0xFF, bytes, s) : e;
  }
  // Allocates into the empty set n, for `capacity` runs of `words` words, each area this set holds whose size changes from `cap`
  // runs of `old_words`.  Schedule records that no copy from here fills (relay, copy_prefix) start without a baseline.  -> "" or
  // the error of the failed allocation, naming its area; this set is unchanged either way.
  std::string alloc_resized(RunAreas& n, uint32_t cap, uint32_t capacity, uint32_t old_words, uint32_t words, cudaStream_t s) const {
    const bool resize = capacity != cap, relaid = resize || words != old_words;
    cudaError_t e = cudaSuccess;
    const char* area = "timers";
    if (resize && timer_k) { e = n.d_timers.alloc((size_t)capacity * timer_k); n.timer_k = timer_k; }
    if (e == cudaSuccess && resize && d_sched_in) { area = "limiter inputs"; e = n.d_sched_in.alloc(capacity); }
    if (e == cudaSuccess && resize && d_runctl) { area = "run control"; e = n.d_runctl.alloc(capacity); }
    if (e == cudaSuccess && resize && d_due) {   // every bit set: copy_due keeps the old runs' below them
      area = "commit-due bits";
      e = n.d_due.alloc(due_words(capacity));
      if (e == cudaSuccess) e = cudaMemsetAsync(n.d_due, 0xFF, n.d_due.cap * 4, s);
    }
    if (e == cudaSuccess && relaid && d_sched_in) {
      area = "schedule records";
      e = capacity < cap && words == old_words ? n.d_sched_rec.alloc((size_t)capacity * BF_SCHED_STRIDE(words))
                                               : alloc_sched_rec(n.d_sched_rec, capacity, words, s);
    }
    return e == cudaSuccess ? std::string() : std::string("(") + area + "): " + cudaGetErrorString(e);
  }
  // Reshape: the timers of n (alloc_resized from `cap` runs of `old_words`) take each run's slots from here, empty past cap (one
  // relay launch, counted in launches), and with the words unchanged n's schedule records take the first cap runs' records.
  // reshape_runs fills n's limiter inputs and run control.
  cudaError_t relay(RunAreas& n, uint32_t cap, uint32_t capacity, uint32_t old_words, uint32_t words, cudaStream_t s,
                    uint64_t& launches) const {
    cudaError_t e = cudaSuccess;
    if (n.d_sched_rec && words == old_words)
      e = cudaMemcpyAsync(n.d_sched_rec, d_sched_rec, (size_t)cap * BF_SCHED_STRIDE(words), cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess && n.d_timers) {
      e = bf::launch_relay_timers({d_timers, n.d_timers, capacity, cap, timer_k, timer_k}, s);
      launches += 1;
    }
    return e == cudaSuccess ? copy_due(n, std::min(cap, capacity), s) : e;
  }
  // Retire to a smaller capacity: the first `capacity` runs of every area into n (alloc_resized), device to device.
  cudaError_t copy_prefix(RunAreas& n, uint32_t capacity, uint32_t words, cudaStream_t s) const {
    const auto copy = [&](void* to, const void* from, size_t per_run) {
      return cudaMemcpyAsync(to, from, capacity * per_run, cudaMemcpyDeviceToDevice, s);
    };
    cudaError_t e = cudaSuccess;
    if (timer_k) e = copy(n.d_timers, d_timers, (size_t)timer_k * 8);
    if (e == cudaSuccess && d_sched_in) e = copy(n.d_sched_in, d_sched_in, sizeof(bf_sched_run));
    if (e == cudaSuccess && d_sched_in) e = copy(n.d_sched_rec, d_sched_rec, BF_SCHED_STRIDE(words));
    if (e == cudaSuccess && d_runctl) e = copy(n.d_runctl, d_runctl, sizeof(bf_run_ctl));
    return e == cudaSuccess ? copy_due(n, capacity, s) : e;
  }
  // Reshape and retire to a new capacity: n's commit-due bits (alloc_resized, all set) take this set's whole words below `runs`,
  // the runs both capacities hold; the runs of a partial last word stay due.
  cudaError_t copy_due(RunAreas& n, uint32_t runs, cudaStream_t s) const {
    if (!n.d_due || runs < 32) return cudaSuccess;
    return cudaMemcpyAsync(n.d_due, d_due, (size_t)(runs / 32) * 4, cudaMemcpyDeviceToDevice, s);
  }
  // takes every area n holds in place of this set's
  void adopt(RunAreas&& n) {
    if (n.d_timers) d_timers = std::move(n.d_timers);
    if (n.d_sched_in) d_sched_in = std::move(n.d_sched_in);
    if (n.d_sched_rec) d_sched_rec = std::move(n.d_sched_rec);
    if (n.d_runctl) d_runctl = std::move(n.d_runctl);
    if (n.d_due) d_due = std::move(n.d_due);
  }
};

// A device-resident batch (row f2), with the bookkeeping of touched ticks that tests/resident_model.py restates under the
// same names.  Each field and the calls that change it:
//   L, cap, d_state,   create, and reshape / retire / narrow (adopt).  d_state also: upload, deltas, migrate, redrive, retire.
//   d_result           full ticks write it; a touched tick's list-mode compaction updates the runs it evaluated; reshape and
//                      narrow re-lay it out; retire moves records with their runs.
//   d_result_prev      result_prev allocates it on first use, adopt drops it; a changed-only tick swaps it with d_result and a
//                      touched tick passes into it, so it is never read before a pass writes it.
//   prev_valid, _runs  d_result holds a pass over the current state lineage of prev_runs runs: full_tick_done sets it; an upload
//                      and records_unknown clear it; compact_to follows the run count; narrowed clears it past its n_runs.
//   d_mark, epoch,     deltas and redrives raise a run's mark to mark_touched() (epoch << 1); uploads, migrations and retires to
//   full_epoch         mark_must_list() (| 1: listed even if unchanged).  full_tick_done records the ending epoch in full_epoch
//                      and opens the next, so older marks are stale by comparison alone (no clear, no launch), and zeroes the
//                      marks on epoch wrap.  A touched tick evaluates the runs marked after full_epoch and zeroes their marks.
//   full_runs          runs of the last full tick (full_tick_done); compact_to and narrowed clamp it.
//   need_full          the current records are not known to be complete: no tick yet, a failed call (records_unknown, a failed
//                      touched tick), a reshape that added decision planes or output fields, or a narrow that dropped decision
//                      planes, the child area or output fields.  full_tick_done clears it.
//   last_fixpoint, last_max_iter, slot_changes_seen: BF_EVAL_FIXPOINT, max_iterations and bf_ctx::slot_changes at the last
//                      full tick.  A touched tick with other parameters, or after a slot drop or reuse, is full (full_due).
//   pending            bound on the touched runs: those the last touched tick left at or above its n_runs, plus the deltas,
//                      uploaded, migrated, redriven, moved and received runs since.  full_tick_done zeroes it.
//   (transfer)         the source compacts as by retire (compact_to); the destination takes the arrivals as uploads (received).
//   uploaded           merged [first, end) ranges, keyed by first, of the runs at or above full_runs uploaded since the last full
//                      tick (note_uploaded); compact_to clips them; full_tick_done clears them.
//   areas              the per-run side areas (RunAreas): step timers, limiter inputs and schedule records, run control, commit-due
//                      bits.
//   commit_all,        with the commit-due bits: the next touched commit considers every run of [0, n_runs) (and sets the bits
//   commit_form,       at or past n_runs).  Set by enabling the bits, a full tick (resident_tick_locked), a failed tick or commit;
//   commit_timings     a touched commit is full also when its form (arm, journal, rewrites: commit_form) or, arming, the ctx's
//                      timing_changes (commit_timings) differ from the last touched commit's.  A touched commit clears it.
//   ticked             runs covered by a tick since the last call that changed d_state (state_changed), or -1: none since.  A
//                      resident schedule over n runs needs ticked >= n.
//   single_ticked      runs covered by single-pass ticks since the last tick with BF_EVAL_FIXPOINT, or -1.  scheduled: runs covered
//                      by a bf_resident_schedule since the last tick, or -1.  A commit over n runs needs ticked, single_ticked and,
//                      with a limiter area, scheduled >= n; a commit that writes changes d_state.
// A call that changes d_state ends the evaluated snapshot (end_snapshot): bf_schedule must follow a new pass.
struct Resident {
  bool alive = false, prev_valid = false, need_full = true;
  bf_layout L{};
  uint32_t cap = 0, prev_runs = 0, epoch = 1, full_epoch = 0, full_runs = 0, last_fixpoint = 0, last_max_iter = 0;
  DevBuf<uint8_t> d_state, d_result, d_result_prev;
  DevBuf<uint32_t> d_mark;
  RunAreas areas;
  int64_t ticked = -1, single_ticked = -1, scheduled = -1;
  bool commit_all = true;
  uint32_t commit_form = ~0u;
  uint64_t commit_timings = 0;
  uint64_t slot_changes_seen = 0, pending = 0;
  std::map<uint32_t, uint32_t> uploaded;

  uint32_t mark_touched() const { return epoch << 1; }
  uint32_t mark_must_list() const { return epoch << 1 | 1u; }
  void end_snapshot(bf_ctx* c) const { if (c->snap.holds(d_state)) c->snap.valid = false; }
  // a call changes d_state: bf_schedule and bf_resident_schedule must both follow a new tick
  void state_changed(bf_ctx* c) { end_snapshot(c); ticked = -1; }
  void tick_done(uint32_t n_runs, uint32_t flags) {
    ticked = std::max<int64_t>(ticked, n_runs);
    single_ticked = (flags & BF_EVAL_FIXPOINT) ? -1 : std::max<int64_t>(single_ticked, n_runs);
    scheduled = -1;
  }
  bf::RunAreasView areas_view() const { return areas.view(L.words); }
  // the runs [first, end) were uploaded: the part at or above full_runs, merged with the ranges it touches
  void note_uploaded(uint32_t first, uint32_t end) {
    uint32_t lo = std::max(first, full_runs), hi = end;
    if (lo >= hi) return;
    auto it = uploaded.upper_bound(lo);
    if (it != uploaded.begin() && std::prev(it)->second >= lo) {
      --it;
      lo = it->first; hi = std::max(hi, it->second);
      it = uploaded.erase(it);
    }
    while (it != uploaded.end() && it->first <= hi) { hi = std::max(hi, it->second); it = uploaded.erase(it); }
    uploaded.emplace(lo, hi);
  }
  // Were all runs of [lo, hi) uploaded since the last full tick?  (The ranges are merged: one of them must hold all of it.)
  bool uploads_cover(uint32_t lo, uint32_t hi) const {
    auto it = uploaded.upper_bound(lo);
    if (it == uploaded.begin()) return false;
    --it;
    return it->first <= lo && it->second >= hi;
  }
  // must a touched tick over n_runs with these parameters be full?  Also just before the epoch wraps (full_tick_done)
  bool full_due(const bf_ctx* c, uint32_t n_runs, uint32_t flags, uint32_t max_iter) const {
    return need_full || c->slot_changes != slot_changes_seen || (flags & BF_EVAL_FIXPOINT) != last_fixpoint ||
           max_iter != last_max_iter || epoch >= 0x7FFFFFFEu || (n_runs > full_runs && !uploads_cover(full_runs, n_runs));
  }
  int full_tick_done(bf_ctx* c, uint32_t n_runs, uint32_t flags, uint32_t max_iter, cudaStream_t s) {
    prev_valid = true; prev_runs = n_runs; need_full = false;
    full_epoch = epoch++; full_runs = n_runs;
    last_fixpoint = flags & BF_EVAL_FIXPOINT; last_max_iter = max_iter; slot_changes_seen = c->slot_changes;
    pending = 0; uploaded.clear();
    if (epoch >= 0x7FFFFFFFu) {   // the epoch must fit mark >> 1: once per 2^31 full ticks the marks start over
      BF_CUDA(c, cudaMemsetAsync(d_mark, 0, d_mark.cap * sizeof(uint32_t), s));
      epoch = 1; full_epoch = 0;
    }
    return BF_OK;
  }
  void records_unknown() { need_full = true; prev_valid = false; }
  // the end of a call rewriting records in place (bf::end_call): after a failure some records may have changed, so the next
  // touched tick evaluates and lists every run
  int sync_in_place(bf_ctx* c, cudaError_t e, const char* what) {
    const int rc = bf::end_call(c, e, what);
    if (rc != BF_OK) records_unknown();
    return rc;
  }
  int result_prev(bf_ctx* c) {
    const cudaError_t e = d_result_prev ? cudaSuccess : d_result_prev.alloc((size_t)cap * L.result_stride);
    return e == cudaSuccess ? BF_OK : bf::fail(c, BF_ENOMEM, std::string("resident batch (second result buffer): ") + cudaGetErrorString(e));
  }
  // the state, result and touch-mark buffers of a new batch (create), or of new ones a batch adopts (reshape, retire, narrow): a
  // call that fails first frees them with its locals
  cudaError_t alloc(const bf_layout& layout, uint32_t capacity) {
    cudaError_t e = d_state.alloc((size_t)capacity * layout.state_stride);
    if (e == cudaSuccess) e = d_result.alloc((size_t)capacity * layout.result_stride);
    return e == cudaSuccess ? d_mark.alloc(((size_t)capacity + 3) / 4 * 4) : e;   // padded: the list build reads four marks at a time
  }
  // new buffers at a new layout and capacity, with the side areas b holds (the others stay); the second result buffer is
  // allocated at the new size when next used
  void adopt(Resident&& b, const bf_layout& layout, uint32_t capacity) {
    d_state = std::move(b.d_state); d_result = std::move(b.d_result); d_result_prev.reset(); d_mark = std::move(b.d_mark);
    areas.adopt(std::move(b.areas));
    if (layout.words != L.words) areas.sched_base_runs = 0;
    L = layout; cap = capacity;
  }
  // retire left the runs [0, m) of [0, N); moves[i] is the new index of run m + i, or kRetireNoMove.  A moved run counts as
  // uploaded at its new index, and its result record moved with it (a changed-only tick compares it with its own record).
  void compact_to(uint32_t m, uint32_t N, const std::vector<uint32_t>& moves) {
    full_runs = std::min(full_runs, m);
    areas.sched_base_runs = std::min(areas.sched_base_runs, m);
    uploaded.erase(uploaded.lower_bound(m), uploaded.end());
    for (auto& u : uploaded) u.second = std::min(u.second, m);
    for (uint32_t to : moves)
      if (to != bf::kRetireNoMove) { note_uploaded(to, to + 1); ++pending; }
    if (prev_valid && prev_runs == N) prev_runs = m;
    else prev_valid = false;
  }
  // The runs below this bound whose current result record a touched tick may compare with: none while the next touched tick is
  // full; else those of the last full tick, and the runs uploaded since in one range from there on that a touched tick has
  // evaluated (a touched tick over more runs than full_runs is full unless such a range covers them).  Runs still marked
  // "must list" are listed whatever their record holds, and records past the bound were never written by a pass or are not
  // compared any more: neither limits a narrow.
  uint32_t touched_baseline_runs() const {
    if (need_full) return 0;
    auto it = uploaded.find(full_runs);
    return it == uploaded.end() ? full_runs : it->second;
  }
  // narrow re-laid every record at a smaller layout (adopt) after checking the result records of [0, n_runs) only: those above
  // may have lost bits, so neither a full tick nor a changed-only baseline reaches past n_runs.  results_may_change: decision
  // planes, the child area or an output field were dropped, which may change any run's result.
  void narrowed(uint32_t n_runs, bool results_may_change) {
    full_runs = std::min(full_runs, n_runs);
    if (prev_runs > n_runs) prev_valid = false;
    if (results_may_change) need_full = true;
  }
  // transfer wrote n arrivals at [first, first + n), marked "must list": they count as uploaded.  The changed-only baseline
  // reaches over them when it covered exactly `first` runs and their result records were a baseline of their source
  // (src_baseline), else the next changed-only tick lists every run.
  void received(uint32_t first, uint32_t n, bool src_baseline) {
    note_uploaded(first, first + n);
    pending += n;
    if (prev_valid && prev_runs == first && src_baseline) prev_runs = first + n;
    else prev_valid = false;
  }
};

namespace bf {
// the topology arena (topology.cu)
int grow_arena(bf_ctx* c, size_t need_total);
int sync_slots(bf_ctx* c, cudaStream_t stream);
// the timing table of a commit that arms (one copy when a timing changed since the last): P.tim stays nullptr when no slot has one
int sync_timings(bf_ctx* c, cudaStream_t stream, CommitTimings& P);
uint32_t largest_record(bf_ctx* c, uint32_t w);

// host helpers of a pass, defined in abi.cu and used by resident_abi.cu too
int check_layout(bf_ctx* c, const bf_layout& L);
int run_pass(bf_ctx* c, const bf_batch& b, const uint8_t* d_state, uint8_t* d_result, bf_expansion* d_exp,
             unsigned long long* d_counts, cudaStream_t stream, const uint32_t* run_list = nullptr,
             const uint32_t* run_list_count = nullptr, FusedHeads* heads = nullptr);
void* pinned_dev(const void* p);
CompactParams compact_params(bf_ctx* c, const bf_layout& L, uint32_t n_runs, bool want_counts, bool want_rejected);
int events_first(bf_ctx* c, uint16_t* events, uint64_t prev, uint64_t slack, uint64_t cap, bool posted, cudaStream_t s, uint64_t& first);
int compact_prepare(bf_ctx* c, uint32_t n_runs, cudaStream_t s);
unsigned long long* cblock_sums(bf_ctx* c, uint32_t which);
int compact_enqueue(bf_ctx* c, const bf_layout& L, const uint8_t* d_result, const uint8_t* d_prev, uint32_t n_runs, bf_compact_out* out,
                    cudaStream_t s, uint64_t& first_slice, bool with_rejected, bool heads_done = false);
int compact_finish(bf_ctx* c, bf_compact_out* out, uint64_t first_slice, uint64_t& prev);
// the chunked pipeline of bf_eval and the full resident ticks: chunk count, the chunks' passes and copies, the results behind
// them, the synchronise that ends the call, and what a pass that went through publishes
int plan_chunks(bf_ctx* c, size_t bytes, size_t per_chunk, uint32_t at_least, uint32_t& chunks);
int chunked_pass(bf_ctx* c, bf_batch db, uint32_t chunks, bool taper, uint8_t* d_state, uint8_t* d_result, const uint8_t* h_state,
                 uint8_t* h_result, bf_expansion* d_exp, FusedHeads* heads);
int pass_results(bf_ctx* c, const bf_layout& L, const uint8_t* d_result, const uint8_t* d_prev, uint32_t n_runs, bf_compact_out* co,
                 uint64_t& first_slice, bool with_rejected, bool heads_done);
int pass_end(bf_ctx* c, int rc, uint32_t chunks, bool uploaded, bool compacted);
int publish_pass(bf_ctx* c, uint32_t n_runs, const bf_layout& L, const uint8_t* d_state, const uint8_t* d_result, bf_counts* counts,
                 bf_compact_out* co, uint64_t first_slice, uint64_t& prev);

// host-buffer evaluation and scheduling (abi.cu), which a device group (group.cu) runs once per shard
int eval_host(bf_ctx* c, const bf_batch* b, bf_compact_out* co);
// totals hook of a sharded schedule: called between the counting and the truncation kernels with the device totals
struct SchedTotals { uint32_t* story_running; uint32_t* queue_running; int32_t* queue_maxprio; uint32_t* global_running; uint32_t ns, nq; };
typedef int (*sched_between_fn)(void* user, const SchedTotals& t, cudaStream_t s);
int schedule_host(bf_ctx* c, const bf_batch* b, const bf_sched_run* runs, const bf_sched_tables* t, bf_sched_out* out,
                  sched_between_fn between, void* user, bool with_bases);
}  // namespace bf
