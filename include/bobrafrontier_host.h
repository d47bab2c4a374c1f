/*
 * bobrafrontier_host.h — host-side mirror of the reference's objects for the frontier path (SURVEY.md 8 row f2).
 *
 * What the Go batcher would otherwise re-implement: turning Story / StoryRun objects (names, `needs`, template
 * strings, StepState phases and messages, GateStatus, child StepRuns) into the packed records of
 * bobrafrontier.h, and result records back into step names.  Reference functions mirrored (paths relative to
 * /root/reference/internal/controller/runs):
 *
 *   buildDependencyGraphs / findAndAddDeps / addDependency   dag.go:3024-3073, 3223-3268  (bfh_story_finalize)
 *   sanitizeStepIdentifier (alias map)                       step_executor.go:1652-1670
 *   validateRuntimeDependencyGraph (unknown deps)            dag.go:3076-3098            (cycles: bf_topology_put)
 *   allStorySteps (index space main ++ comp ++ finally)      dag.go:3270-3280
 *   isConcurrencyQueued (message prefixes -> code 14)        dag.go:2035-2051            (bfh_run_set_phase)
 *   checkSyncGates decision order                            dag.go:1489-1533            (bfh_run_set_gate)
 *   syncStateFromStepRuns-style incremental updates          dag.go:965-1009             (bfh_run_set_* are O(1))
 *
 * State records live in pinned host memory owned by the batch and are updated IN PLACE (a phase change flips at
 * most four bits), so a tick's host work is O(changes) and bf_eval's upload is one contiguous copy.
 *
 * Same ABI rules as bobrafrontier.h: flat C, negative bf_status on error, nothing retained but what is documented.
 */
#ifndef BOBRAFRONTIER_HOST_H_
#define BOBRAFRONTIER_HOST_H_

#include "bobrafrontier.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ Story (definition side) */
typedef struct bfh_story bfh_story;

bfh_story* bfh_story_new(void);
void bfh_story_free(bfh_story* s);
const char* bfh_story_error(const bfh_story* s);

/* Append a step in list order within its group.  group: BF_GROUP_MAIN / _COMPENSATION / _FINALLY;
 * type: BF_STEP_* (BF_STEP_ENGRAM = step.Ref set).  if_expr / with_raw may be NULL.  Returns the step's
 * insertion handle (>= 0) or a negative status. */
int bfh_story_add_step(bfh_story* s, const char* name, int group, int type, int allow_failure, int on_timeout_skip,
                       const char* if_expr, const char* with_raw);
int bfh_step_add_need(bfh_story* s, int step, const char* dep_name);
int bfh_step_add_branch(bfh_story* s, int step, const char* branch_name, int allow_failure); /* parallel: with.steps */
/* continue_on_step_failure: -1 unset, 0, 1 (Policy.Retries.ContinueOnStepFailure, dag.go:3504-3511) */
int bfh_story_set_policy(bfh_story* s, int continue_on_step_failure, int realtime);

/* Resolve names, extract template references, build the CSR over allStorySteps.  BF_ETOPO on unknown deps. */
int bfh_story_finalize(bfh_story* s);
int bfh_story_dims(const bfh_story* s, uint32_t* n_steps, uint32_t* n_edges, uint32_t* n_parallel);
/* Copy out the packed form (row_ptr[S+1], col_idx[E], step_flags[S]); any pointer may be NULL. */
int bfh_story_csr(const bfh_story* s, uint32_t* row_ptr, uint16_t* col_idx, uint8_t* step_flags);
/* The timing of a sleep, gate or wait step (insertion handle `step`) that bfh_story_upload puts after the topology
 * (bf_topology_timings: code BF_DEC_*, delay in clock units after the arming commit's `now`); code -1 removes it.  Parsing
 * `with` (duration, timeout, pollInterval) stays with the caller, as on_timeout_skip does.  BF_EINVAL when the step's type
 * does not take the code (the rules of bf_topology_timings). */
int bfh_story_set_step_timing(bfh_story* s, int step, int code, uint32_t delay);
int bfh_story_upload(bfh_story* s, bf_ctx* ctx, uint32_t* slot_out); /* bf_topology_put of the packed form, then its timings */
int bfh_story_step_index(const bfh_story* s, const char* name);      /* index in allStorySteps order, or -1 */
const char* bfh_story_step_name(const bfh_story* s, uint32_t index);
uint32_t bfh_story_run_flags(const bfh_story* s);                     /* BF_RF_FAIL_FAST / BF_RF_REALTIME from the policy */

/* One pass of the template-reference scanner (exposed for tests): writes up to cap names, '\n'-separated. */
int bfh_scan_step_refs(const char* expression, char* out, size_t cap);

/* ------------------------------------------------------------------ Batch of live StoryRuns */
typedef struct bfh_batch bfh_batch;

/* ctx may be NULL (CPU-side packing only: bfh_batch_eval then returns BF_ENODEV). */
bfh_batch* bfh_batch_new(bf_ctx* ctx, uint32_t steps_max, uint32_t child_nibbles, uint32_t fields, uint32_t capacity);
void bfh_batch_free(bfh_batch* b);
const char* bfh_batch_error(const bfh_batch* b);
const bf_layout* bfh_batch_layout(const bfh_batch* b);
uint32_t bfh_batch_size(const bfh_batch* b);
const void* bfh_batch_state(const bfh_batch* b);   /* [size * state_stride]  */
const void* bfh_batch_result(const bfh_batch* b);  /* [size * result_stride] */

/* Add a StoryRun of `story` (finalized; `slot` from bfh_story_upload or any caller-chosen slot id).  Returns the
 * run index.  The run starts with no StepStates, run flags from the Story policy. */
int bfh_batch_add_run(bfh_batch* b, const bfh_story* story, uint32_t slot);
int bfh_batch_remove_last_run(bfh_batch* b);

/* StepState update.  phase: "", "Pending", ... ; message only matters for Pending (queued prefixes -> code 14). */
int bfh_run_set_phase(bfh_batch* b, uint32_t run, uint32_t step, const char* phase, const char* message);
int bfh_run_set_phase_code(bfh_batch* b, uint32_t run, uint32_t step, int code);
int bfh_run_set_cond(bfh_batch* b, uint32_t run, uint32_t step, int cond_code);         /* BF_COND_* */
int bfh_run_set_decision(bfh_batch* b, uint32_t run, uint32_t step, int decision_code); /* BF_DEC_*  */
/* Gate decision exactly as checkSyncGates orders it: Approved > Rejected > timed-out > pending. */
int bfh_run_set_gate(bfh_batch* b, uint32_t run, uint32_t step, const char* gate_state, int timed_out);
int bfh_run_set_run_flags(bfh_batch* b, uint32_t run, int topology_terminated, int host_group /* -1 none, else BF_GROUP_* */);
int bfh_run_register_children(bfh_batch* b, uint32_t run, uint32_t parallel_index, int registered);
int bfh_run_set_child_phase(bfh_batch* b, uint32_t run, uint32_t parallel_index, uint32_t branch, const char* phase);

/* Resident mode (row f2, incremental state upload): the device keeps the state records; from then on every
 * bfh_run_set_* also logs a delta (coalesced per (run, field, index): the last value of a tick wins) and
 * bfh_batch_eval sends the records of NEW runs plus the tick's deltas instead of the whole batch — H2D is
 * O(changes), what syncStateFromStepRuns (dag.go:965-1009) produces per reconcile.  Needs a device ctx.        */
int bfh_batch_set_resident(bfh_batch* b, int on);
/* bytes sent so far as full records / as deltas, and the deltas logged since the last eval */
int bfh_batch_traffic(const bfh_batch* b, uint64_t* full_record_bytes, uint64_t* delta_bytes, uint32_t* pending_deltas);

/* A Story edited while its runs are live (see bf_resident_migrate).  bfh_story_migration_map writes, for each step i of `old_story`
 * (finalized, allStorySteps order), the index of the step of the same name in `new_story`, or BF_MIGRATE_GONE, into map[i] for
 * i < cap, and returns the step count of old_story.  bfh_batch_migrate moves every run whose record holds old_slot (each must be
 * a run of old_story) to new_story / new_slot: the mirror re-packs its own records by step name (parallel steps keep their
 * registered bit and child phases, branches by index; a kept parallel step whose branch count changed is BF_EINVAL), rewrites
 * the step, child and desc indices of the pending deltas of those runs and drops the ones of removed steps; in resident mode it
 * first calls bf_resident_migrate over the uploaded runs, so that the device and the mirror stay identical.  Nothing changes
 * on an error, with one exception: when the device copy had diverged from the mirror and bf_resident_migrate moved a different
 * number of runs than the mirror holds, the mirror stays unchanged, its pending deltas are discarded and the next
 * bfh_batch_eval uploads every record in full (BF_EINVAL reports it).  Returns the number of runs moved.  Steps new to this generation start with no state; re-send what they had
 * if their name existed in an earlier generation.                                                                         */
int bfh_story_migration_map(const bfh_story* old_story, const bfh_story* new_story, uint16_t* map, uint32_t cap);
int bfh_batch_migrate(bfh_batch* b, const bfh_story* old_story, const bfh_story* new_story, uint32_t old_slot, uint32_t new_slot);

/* An operator redrive of live runs (see bf_resident_redrive).  Request i resets run runs[i] from step steps[i] (an index of the
 * run's story) or, for steps[i] = -1, the whole run.  The mirror re-packs its own records by the rules of bf_resident_redrive,
 * with the reset set computed here from the story's dependency rows; it drops the pending deltas that would undo the reset when
 * sent (phase / cond / decision of reset steps, child phases and registered bits of reset parallel steps) and clears
 * BF_RF_TOPOLOGY_TERMINATED in a pending run-flags delta; other pending deltas still apply after the reset.  In resident mode it
 * also calls bf_resident_redrive once for the uploaded runs, so that the device and the mirror stay identical; should a device
 * record not hold the slot the mirror holds (a copy changed behind the mirror's back), the next bfh_batch_eval uploads every
 * record in full.  A run or step out of range is BF_EINVAL and changes nothing.  Returns BF_OK.                            */
int bfh_batch_redrive(bfh_batch* b, const uint32_t* runs, const int32_t* steps, uint32_t n);

/* Grow the batch (see bf_resident_reshape): the layout becomes bf_layout_init(steps_max, child_nibbles, fields) and the capacity
 * `capacity`, by the same growth rules.  The mirror re-lays its own state and result records as bf_resident_reshape re-lays the
 * device's, and keeps its pending deltas (their run, step and child indices do not change).  In resident mode it calls
 * bf_resident_reshape first; when that fails, the mirror changes nothing either.  A shrinking or invalid shape is BF_EINVAL, a
 * failed allocation BF_ENOMEM, and both change nothing.  Afterwards bfh_batch_add_run takes the larger Stories and the
 * additional runs.                                                                                                         */
int bfh_batch_reshape(bfh_batch* b, uint32_t steps_max, uint32_t child_nibbles, uint32_t fields, uint32_t capacity);

/* Narrow the batch (see bf_resident_narrow): the layout becomes bf_layout_init(steps_max, child_nibbles, fields), the capacity
 * stays.  The same acceptance test is applied to the mirror's own records (every record below the capacity, the Story of every
 * run, the result record of every run) and to its pending deltas: a pending delta whose step, child index or field the new
 * layout lacks blocks the call, so nothing is dropped silently.  The mirror re-lays its records as bf_resident_narrow re-lays
 * the device's and keeps its pending deltas.  In resident mode it first uploads its runs not yet on the device, then calls
 * bf_resident_narrow over its runs; when that fails, the mirror changes nothing.  A growing, invalid or blocked shape is
 * BF_EINVAL, a failed allocation BF_ENOMEM, and both change nothing.                                                       */
int bfh_batch_narrow(bfh_batch* b, uint32_t steps_max, uint32_t child_nibbles, uint32_t fields);

/* Retire runs (see bf_resident_retire): `runs` lists n distinct runs below bfh_batch_size; the last live runs move into the
 * indices they free, by the same rule, and the size becomes size - n.  capacity 0 keeps the capacity, else it becomes
 * `capacity` (size - n <= capacity <= current).  The mirror moves its own records, drops the pending deltas of retired runs and
 * re-keys those of moved runs, which then apply at the new index.  In resident mode it first uploads its runs not yet on the
 * device, then calls bf_resident_retire; when that fails, the mirror's records and deltas do not change.  moves_from / moves_to
 * ([n] each, may be NULL) receive the moves, ascending by target.  Returns the number of moves, or BF_EINVAL (bad arguments,
 * nothing changed), BF_ENOMEM or the device's error.                                                                        */
int bfh_batch_retire(bfh_batch* b, const uint32_t* runs, uint32_t n, uint32_t capacity, uint32_t* moves_from, uint32_t* moves_to);

/* Move runs to another batch (see bf_resident_transfer): `runs` lists n distinct runs below bfh_batch_size(src); runs[i] becomes
 * run bfh_batch_size(dst) + i of dst, with its Story, its records re-laid at dst's layout as bf_resident_transfer re-lays the
 * device's, and its pending deltas, re-keyed to the new index.  src then equals bfh_batch_retire of the same runs with capacity
 * 0 (the same moves into moves_from / moves_to, [n] each, may be NULL; the other pending deltas re-keyed likewise).  Each run
 * must fit dst's layout by bf_resident_narrow's test applied to it alone (its record, its Story, its result record when the last
 * eval covered it), and a pending delta of a moved run whose step, child index or field dst's layout lacks blocks the call.
 * Both batches must be of one ctx (or both without one) and in the same mode.  In resident mode it first uploads the runs of
 * both batches not yet on the device, then calls bf_resident_transfer; when that fails, neither mirror changes.  Returns the
 * number of moves, or BF_EINVAL (bad arguments or a refusal, nothing changed) or the device's error.                       */
int bfh_batch_transfer(bfh_batch* src, bfh_batch* dst, const uint32_t* runs, uint32_t n, uint32_t* moves_from, uint32_t* moves_to);

/* One frontier pass over the batch through bf_eval (or, in resident mode, bf_resident_*) (eval_flags: BF_EVAL_*). */
int bfh_batch_eval(bfh_batch* b, uint32_t eval_flags, bf_counts* counts);

/* A tick commit in resident mode (see bf_resident_commit), after bfh_batch_eval: bf_resident_commit_journal over the runs of that
 * eval on the device, whose PHASE and REGISTERED items the mirror applies to its own records.  It logs no delta.  An item whose
 * (run, field, index) a delta logged since the eval covers is not applied: the next eval applies that delta after the commit on
 * the device as well, so it wins on both sides.  The journal is sized from the mirror's last results (ready, skip and fail steps
 * and ready parallel steps), so it is never cut short.  Timers are not armed (the mirror holds no timer area).  After the call
 * and the next eval the mirror's records equal the device's for every uploaded run.  Not resident: BF_EINVAL.  A refusal
 * (bad_run / bad_step in out, which may be NULL) changes neither the device nor the mirror.                                 */
int bfh_batch_commit(bfh_batch* b, const bf_commit_entry* entries, uint32_t n, bf_commit_out* out);

/* bfh_batch_commit through bf_resident_commit_rewrites: the device also stores the phases a single pass's stages G, H and I
 * rewrite, and the mirror applies those PHASE items as the others (pending deltas win the same way).  The journal is sized as
 * bfh_batch_commit's, with every step of the Story for a run whose last result carries BF_SUM_PHASE_CHANGED.  *n_rewritten
 * (may be NULL) is the call's count of steps written from the stages.                                                       */
int bfh_batch_commit_rewrites(bfh_batch* b, const bf_commit_entry* entries, uint32_t n, bf_commit_out* out, uint32_t* n_rewritten);

/* Results of the last pass.  Step lists come back in list order (ascending index), the order the
 * concurrency limiters' readySteps[:slots] relies on (dag.go:1796-1798). */
uint32_t bfh_run_summary(const bfh_batch* b, uint32_t run);
int bfh_run_ready(const bfh_batch* b, uint32_t run, uint32_t* steps_out, uint32_t cap);
int bfh_run_skipped(const bfh_batch* b, uint32_t run, uint32_t* steps_out, uint32_t cap);
int bfh_run_failed(const bfh_batch* b, uint32_t run, uint32_t* steps_out, uint32_t cap);
int bfh_run_needs_cond(const bfh_batch* b, uint32_t run, uint32_t* steps_out, uint32_t cap);
int bfh_run_phase_out(const bfh_batch* b, uint32_t run, uint32_t step); /* phase code after the pass, or -1 */
/* "Skipped due to failed dependency: <name>" names the first dep in CSR order that is failed (SURVEY 8.0-F). */
int bfh_run_skip_reason(const bfh_batch* b, uint32_t run, uint32_t step, char* out, size_t cap);

/* ------------------------------------------------------------------ limiters (rows a9 / f4)
 * Host side of bf_schedule: what stays on the host in the batch contract of bobrafrontier.h —
 *   resolveSchedulingDecision / queueLabelValue / normalizeQueueName   scheduling.go:21-35, 130-163
 *   queueConfigForName (a queue without an entry = zero config)        scheduling.go:101-112
 *   storyConcurrencyLimit                                              dag.go:1863-1868
 *   storyRunQueuedSince -> elapsed seconds for effectivePriority       dag.go:1948-1979
 *   the "Queued due to ... (%d running, limit %d)" messages            dag.go:103-108, 1797, 1849-1855
 * Keys: a story key per (namespace, Story name) — countRunningStepRuns lists by namespace + story label,
 * dag.go:1874-1877 — and a queue key per queue label.  One bf_sched_run per run of the batch.              */
typedef struct bfh_sched bfh_sched;

bfh_sched* bfh_sched_new(bfh_batch* batch);
void bfh_sched_free(bfh_sched* s);
const char* bfh_sched_error(const bfh_sched* s);
/* scheduling.globalConcurrency + Running StepRuns the batch does not hold */
int bfh_sched_set_global(bfh_sched* s, int32_t global_concurrency, uint32_t running_base);
/* scheduling.queues[name]; returns the queue key.  Queues named by a Story but never configured read as zeros. */
int bfh_sched_set_queue(bfh_sched* s, const char* name, int32_t concurrency, int32_t default_priority,
                        int32_t priority_aging_seconds, uint32_t running_base);
/* Running StepRuns of (namespace, story) held by StoryRuns outside the batch; returns the story key. */
int bfh_sched_set_story_base(bfh_sched* s, const char* story_namespace, const char* story_name, uint32_t running_base);
/* One run: its Story's policy (policy_queue NULL/"" = unset, has_priority 0 = unset, story_concurrency <= 0 = none),
 * StoryRun.Status.Phase, and the earliest StartedAt among its queued steps (Unix nanoseconds; queued_since_ns < 0:
 * none) against now_ns: the elapsed seconds are int32((now - since).Seconds()) as in effectivePriority, dag.go:1952-1956. */
int bfh_sched_set_run(bfh_sched* s, uint32_t run, const char* story_namespace, const char* story_name, int32_t story_concurrency,
                      const char* policy_queue, int has_priority, int32_t policy_priority, const char* run_phase,
                      int64_t queued_since_ns, int64_t now_ns);
/* the packed inputs (for inspection / CPU-side checks): bf_sched_run[size], tables valid until the next set_* call */
const bf_sched_run* bfh_sched_runs(const bfh_sched* s);
int bfh_sched_tables(const bfh_sched* s, bf_sched_tables* out);
const char* bfh_sched_queue_name(const bfh_sched* s, uint32_t queue_key);
/* bf_schedule over the batch's last bfh_batch_eval */
int bfh_sched_apply(bfh_sched* s);
/* results of the last apply: step lists in list order; which = 0 launch, 1 queued by the Story limit, 2 queued by scheduling */
int bfh_sched_steps(const bfh_sched* s, uint32_t run, int which, uint32_t* steps_out, uint32_t cap);
/* the reference's message text for which = 1 / 2 ("" when nothing was queued that way) */
int bfh_sched_message(const bfh_sched* s, uint32_t run, int which, char* out, size_t cap);
/* message text from a reason code and the totals (exposed for CPU-side tests) */
int bfh_sched_format_message(int reason /* 0 = story limit, else BF_QUEUED_* */, uint32_t running, int32_t limit, char* out, size_t cap);

#ifdef __cplusplus
}
#endif
#endif /* BOBRAFRONTIER_HOST_H_ */
