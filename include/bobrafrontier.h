/*
 * bobrafrontier.h — C ABI of the H100-native (sm_90a) StoryRun DAG ready-frontier engine.
 *
 * This is the drop-in boundary for ONE hot path of bubustack/bobrapet: the
 * per-reconcile "which steps are ready now?" computation
 *
 *     DAGReconciler.findReadySteps      internal/controller/runs/dag.go:2631-2848
 *     buildStateMaps                    internal/controller/runs/dag.go:3358-3391
 *     clearConcurrencyQueuedSteps       internal/controller/runs/dag.go:2020-2051
 *     checkSyncGates/Sleep/Wait         internal/controller/runs/dag.go:1455-1547, 1217-1288, 1291-1452
 *     checkSyncParallelSteps            internal/controller/runs/dag.go:1112-1200
 *     group selection, fail-fast,       internal/controller/runs/dag.go:422-511, 3289-3342
 *       compensation skipping
 *     launch effects of Execute         internal/controller/runs/step_executor.go:132-185,
 *                                       internal/controller/runs/dag.go:1735-1775
 *
 * evaluated for a whole BATCH of live StoryRuns in one pass on the GPU.  The
 * reference has no FFI for this path (it is Go-internal); these entry points
 * are what a cgo shim (go/frontier/frontier.go, INTEGRATION.md) binds.
 *
 * Rules of the ABI: flat PODs, caller-owned buffers, no callbacks, no C++
 * types, never aborts, never throws; every function returns 0 or a negative
 * bf_status.  The library retains nothing the caller passed except the
 * topologies (copied to HBM by bf_topology_put*).
 *
 * Everything here is integer/bit work; results are bit-exact against the
 * oracle (oracle/), see DESIGN.md.
 */
#ifndef BOBRAFRONTIER_H_
#define BOBRAFRONTIER_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BF_ABI_VERSION 3u

/* ------------------------------------------------------------------ status */
typedef enum bf_status {
  BF_OK = 0,
  BF_EINVAL = -1, /* bad argument / malformed batch                              */
  BF_ENOMEM = -2, /* host or device allocation failed                            */
  BF_ECUDA = -3,  /* CUDA runtime error (bf_last_error has the text)             */
  BF_ENCCL = -4,  /* collective error (multi-GPU count exchange)                 */
  BF_ETOPO = -5,  /* topology rejected: unknown dep, cycle, too large, bad slot  */
  BF_ENODEV = -6  /* no usable sm_90 device / extension built without CUDA       */
} bf_status;

/* ---------------------------------------------------------- phase encoding */
/* 4-bit code per (run, step), stored bit-sliced (see "record layout").  Order = declaration order of enums.Phase
 * (pkg/enums/enums.go:44-97); 0 = "no StepState entry".  Code 14 folds the
 * "queued" bit into the nibble: phase Pending whose message starts with one of
 * the four "Queued due to ..." prefixes (dag.go:103-108, isConcurrencyQueued
 * dag.go:2035-2051).  It is Pending for every purpose except that
 * clearConcurrencyQueuedSteps removes it from the running set.               */
enum {
  BF_PHASE_NONE = 0,
  BF_PHASE_PENDING = 1,
  BF_PHASE_RUNNING = 2,
  BF_PHASE_SUCCEEDED = 3,
  BF_PHASE_FAILED = 4,
  BF_PHASE_FINISHED = 5,
  BF_PHASE_CANCELED = 6,
  BF_PHASE_COMPENSATED = 7,
  BF_PHASE_PAUSED = 8,
  BF_PHASE_BLOCKED = 9,
  BF_PHASE_SCHEDULING = 10,
  BF_PHASE_TIMEOUT = 11,
  BF_PHASE_ABORTED = 12,
  BF_PHASE_SKIPPED = 13,
  BF_PHASE_PENDING_QUEUED = 14,
  BF_PHASE_RESERVED = 15 /* invalid on input; rejected by BF_EVAL_VALIDATE */
};

/* 16-entry boolean tables over the phase code (bit v = value for code v).   */
#define BF_LUT_TERMINAL 0x38F8u   /* Phase.IsTerminal, enums.go:101-115          */
#define BF_LUT_COMPLETED0 0x2008u /* Succeeded|Skipped, dag.go:3377              */
#define BF_LUT_RUNNING 0x4106u    /* Running|Pending|Paused (+queued), :3379     */
#define BF_LUT_RUNNING_Q 0x0106u  /* ... minus concurrency-queued, :2020-2033    */
#define BF_LUT_RT_SAT 0x410Eu     /* dependencySatisfiedForRealtime, :3457-3473  */

/* ------------------------------------------------------------- step flags  */
/* One byte per step, static per Story generation (bf_topology_put).         */
enum {
  BF_STEP_ENGRAM = 0, /* step.Ref != nil                         */
  BF_STEP_CONDITION = 1,
  BF_STEP_PARALLEL = 2,
  BF_STEP_SLEEP = 3,
  BF_STEP_STOP = 4,
  BF_STEP_WAIT = 5,
  BF_STEP_EXECUTE_STORY = 6,
  BF_STEP_GATE = 7
};
#define BF_SF_TYPE_MASK 0x07u
#define BF_SF_ALLOW_FAILURE 0x08u   /* step.AllowFailure, story_types.go:193      */
#define BF_SF_ON_TIMEOUT_SKIP 0x10u /* with.onTimeout == "skip", dag.go:1655-1668 */
#define BF_SF_HAS_IF 0x20u          /* step.If != nil && != "", dag.go:2741       */
#define BF_SF_GROUP_SHIFT 6         /* 0 main (spec.steps), 1 compensations, 2 finally */
#define BF_SF_GROUP_MASK 0xC0u
enum { BF_GROUP_MAIN = 0, BF_GROUP_COMPENSATION = 1, BF_GROUP_FINALLY = 2, BF_GROUP_DONE = 3 };

/* -------------------------------------------------------------- run flags  */
#define BF_RF_FAIL_FAST 0x01u           /* shouldFailFast, dag.go:3504-3511             */
#define BF_RF_REALTIME 0x02u            /* story.Spec.Pattern.IsRealtime()              */
#define BF_RF_TOPOLOGY_TERMINATED 0x04u /* Degraded/TopologyTerminated, dag.go:436-464  */
#define BF_RF_HOST_GROUP 0x08u          /* tier K1: group given by host, skip stage I   */
#define BF_RF_HOST_GROUP_SHIFT 4        /* bits 4-5: BF_GROUP_* when BF_RF_HOST_GROUP   */

/* ----------------------------------------------------- cond / decision codes */
/* 2 bits per (run, step), stored as 2 bit planes.                            */
enum {
  BF_COND_PASS = 0, /* no `if`, realtime, or evaluated true and `with` refs fresh (dag.go:2741,2837,2844) */
  BF_COND_SKIP = 1, /* evaluated false and refs not stale (dag.go:2820-2832)                            */
  BF_COND_HOLD = 2, /* blocked / eval error / offloaded wait / stale refs (dag.go:2801-2842)            */
  BF_COND_FAIL = 3  /* template-safety violation or offloaded under fail policy (dag.go:2744,2810)      */
};
enum {
  BF_DEC_PENDING = 0,   /* keep waiting -> Paused                                      */
  BF_DEC_SUCCEED = 1,   /* gate approved / sleep elapsed / wait satisfied -> Succeeded  */
  BF_DEC_FAIL = 2,      /* gate rejected / invalid config / fail policy  -> Failed      */
  BF_DEC_TIMED_OUT = 3  /* timeout elapsed while pending -> Skipped|Timeout (dag.go:1655) */
};

/* ---------------------------------------------------------------- limits   */
#define BF_MAX_STEPS 1024u   /* steps per topology (CRD caps at 100+50+50, story_types.go:129-140) */
#define BF_MAX_EDGES 65535u  /* u16 row_ptr on device                                             */
#define BF_MAX_PARALLEL 64u  /* parallel steps per topology (children_registered is a u64)        */
#define BF_OFF_NONE 0xFFFFFFFFu

/* ------------------------------------------------------------- topologies  */
typedef struct bf_parallel_desc {
  uint16_t step;        /* index of the `parallel` step                                       */
  uint16_t branches;    /* B = len(with.steps), step_executor.go:745-806                      */
  uint32_t allow_first; /* index of branch 0's bit in branch_allow_bits (bit i -> branch i)   */
} bf_parallel_desc;

typedef struct bf_topology {
  uint32_t n_steps;                /* S: main ++ compensations ++ finally (allStorySteps, dag.go:3270) */
  uint32_t n_edges;                /* E                                                               */
  const uint32_t* row_ptr;         /* [S+1], row_ptr[0]=0, row_ptr[S]=E; deps of step i = col_idx[row_ptr[i]..row_ptr[i+1]) */
  const uint16_t* col_idx;         /* [E] dependency step indices (buildDependencyGraphs, dag.go:3024-3073) */
  const uint8_t* step_flags;       /* [S] BF_SF_*                                                     */
  const bf_parallel_desc* parallel; /* [n_parallel], ascending by step                                */
  uint32_t n_parallel;
  const uint8_t* branch_allow_bits; /* branch allowFailure bits (dag.go:1145-1158); may be NULL       */
  uint32_t n_branch_allow_bits;
} bf_topology;

/* ------------------------------------------------------------ record layout */
/* Dynamic state travels as ONE record per run (so the host->device copy is a
 * single contiguous transfer and the kernel stages a run with one bulk copy).
 * Per-step codes are BIT-SLICED: a k-bit code is stored as k bit planes of
 * `words` u32 each, step i = bit (i%32) of word i/32 of every plane, plane b
 * holding bit b of the code.  Same size as nibble packing (4 bits/step for the
 * phase), but 32 steps are classified by a handful of bitwise ops and no
 * transposition is ever needed on either side.
 *
 *   offset 0     bf_run_header (16 B)
 *   off_phase    phase code, 4 planes: plane b at off_phase + b*words*4     (words*16 B)
 *   off_cond     cond code, 2 planes                                        (words*8 B)  optional
 *   off_decision decision code, 2 planes                                    (words*8 B)  optional
 *   off_child    child StepRun phase NIBBLES of parallel steps (branch order), desc p
 *                starts at nibble child_first[p] (assigned by bf_topology_put),
 *                child c at byte c/2, low nibble first                                   optional
 *
 * Results likewise, one record per run:
 *
 *   offset 0   bf_result_header (16 B)
 *   off_ready / off_skip / off_fail / off_needs_cond / off_skip_dep  bit masks,
 *              step i = bit (i%32) of u32 word i/32  (words*4 B each)
 *   off_phase_out  phase code after this pass's status mutations, 4 planes  (words*16 B)
 *
 * All strides are multiples of 16 bytes.                                      */
typedef struct bf_run_header {
  uint32_t topo_slot;           /* from bf_topology_put                                          */
  uint8_t run_flags;            /* BF_RF_*                                                       */
  uint8_t reserved[3];
  uint64_t children_registered; /* bit p: PrimitiveChildren[parallel p] non-empty, dag.go:1140   */
} bf_run_header;

typedef struct bf_result_header {
  uint32_t summary;      /* BF_SUM_*                                                             */
  uint32_t n_ready;      /* popcount(ready)                                                      */
  uint32_t n_skip;       /* popcount(skip)                                                       */
  uint32_t n_expansion;  /* child StepRuns to create for ready `parallel` steps                   */
} bf_result_header;

#define BF_SUM_GROUP_MASK 0x3u       /* BF_GROUP_* evaluated this pass (3 = finalize on host, dag.go:490-495) */
#define BF_SUM_MAIN_DONE 0x4u        /* dag.go:431                                                        */
#define BF_SUM_MAIN_FAILED 0x8u      /* len(mainFailed) > 0                                               */
#define BF_SUM_COMP_DONE 0x10u
#define BF_SUM_FINAL_DONE 0x20u
#define BF_SUM_COMP_FAILED 0x40u
#define BF_SUM_FINAL_FAILED 0x80u
#define BF_SUM_PHASE_CHANGED 0x100u  /* some phase nibble was rewritten (needsPersist, dag.go:409-470)    */
#define BF_SUM_ITER_SHIFT 16         /* bits 16-27: iterations run (fixpoint mode), dag.go:393            */

/* field selection for bf_layout_init */
#define BF_F_COND 0x1u
#define BF_F_DECISION 0x2u
#define BF_F_CHILD 0x4u
#define BF_F_OUT_FAIL 0x10u
#define BF_F_OUT_NEEDS_COND 0x20u
#define BF_F_OUT_SKIP_DEP 0x40u
#define BF_F_OUT_PHASE 0x80u

typedef struct bf_layout {
  uint32_t steps_max; /* max S over the topologies of the batch                      */
  uint32_t words;     /* ceil(steps_max/32)                                          */
  uint32_t fields;    /* BF_F_*                                                      */
  uint32_t child_nibbles;
  uint32_t state_stride;
  uint32_t off_phase, off_cond, off_decision, off_child;
  uint32_t result_stride;
  uint32_t off_ready, off_skip, off_fail, off_needs_cond, off_skip_dep, off_phase_out;
} bf_layout;

/* ------------------------------------------------------------------ batch  */
#define BF_EVAL_VALIDATE 0x1u   /* host API only: check slots / reserved nibbles before launch   */
#define BF_EVAL_FIXPOINT 0x2u   /* iterate runDagIterations on device (dag.go:393-540), applying
                                   launch effects of instantly-completing primitives             */
#define BF_EVAL_EXPANSION 0x4u  /* emit (run, step, branch) tuples for ready parallel steps      */
#define BF_EVAL_NO_COUNTS 0x8u  /* skip the global counters                                      */
/* bf_eval_device only (0x10 is BF_EVAL_CHANGED_ONLY below):                                                          */
#define BF_EVAL_COUNTS_SET 0x20u /* counts are OVERWRITTEN with this pass's totals (no zeroing by the caller, no memset
                                   launch between passes: the last CTA out publishes the totals)                      */
#define BF_EVAL_PIPELINED 0x40u  /* caller's promise: this pass reads nothing the preceding kernel of the stream writes
                                   and writes nothing it reads or writes (other batch, other result / counts buffers).
                                   The pass is then launched as a programmatic dependent of that kernel: its CTAs start
                                   on SMs the previous pass has already left, so its start-up (slot ids -> slot entries
                                   -> first bulk copies) overlaps the previous pass's tail.  Completion order is
                                   kept (the pass completes after the preceding kernel).  Needs BF_EVAL_COUNTS_SET or
                                   BF_EVAL_NO_COUNTS; ignored where it does not apply                               */

typedef struct bf_expansion {
  uint32_t run;    /* index in the batch                      */
  uint16_t step;   /* the parallel step                       */
  uint16_t branch; /* branch index in with.steps              */
} bf_expansion;

typedef struct bf_counts {
  uint64_t ready;     /* sum n_ready over the batch                                   */
  uint64_t skip;      /* sum n_skip                                                   */
  uint64_t expansion; /* sum n_expansion                                              */
  uint64_t evals;     /* (run, step) pairs visited = sum of S over runs (dag.go:2647) */
} bf_counts;

typedef struct bf_batch {
  uint32_t struct_size; /* sizeof(bf_batch)                                            */
  uint32_t n_runs;
  uint32_t flags;       /* BF_EVAL_*                                                   */
  uint32_t max_iterations; /* fixpoint cap; 0 = S+1 (dag.go:393)                        */
  bf_layout layout;
  const void* state;    /* [n_runs * state_stride]                                     */
  void* result;         /* [n_runs * result_stride]                                    */
  bf_expansion* expansion; /* [expansion_cap], run-major/step/branch order; may be NULL */
  uint64_t expansion_cap;
  bf_counts* counts;    /* out; may be NULL                                            */
} bf_batch;

/* ------------------------------------------------------------------- ctx   */
typedef struct bf_ctx bf_ctx;

typedef struct bf_config {
  uint32_t struct_size;
  int32_t device;          /* CUDA ordinal; one ctx drives one GPU (one process per GPU) */
  uint64_t arena_bytes;    /* initial topology arena in HBM (grows on demand); 0 = default */
  uint32_t max_topologies; /* initial slot table size; 0 = default                       */
  uint32_t flags;          /* BF_CFG_*                                                   */
} bf_config;
/* The frontier kernels are persistent (one CTA per SM holding nearly all of its shared memory), so a kernel of ANOTHER
 * stream — the NCCL all-gather of the counts — finds no SM until a pass ends and queues behind it.  Leaving k SMs out of
 * the grid (k = flags & 0xFF) lets the collective run beside the next pass; it costs k / (SM count) of the pass: k / 132 on H100. */
#define BF_CFG_RESERVE_SMS(k) ((uint32_t)(k) & 0xFFu)

uint32_t bf_abi_version(void);
const char* bf_strerror(int status);
/* Last error text of this ctx (valid until the next call on the ctx). */
const char* bf_last_error(const bf_ctx* ctx);

int bf_create(bf_ctx** out, const bf_config* cfg);
void bf_destroy(bf_ctx* ctx);

/* Upload one topology; returns its slot in *slot_out.  Validates what
 * validateRuntimeDependencyGraph (dag.go:3076-3146) validates: every col_idx
 * < S (no unknown dep) and acyclicity (Kahn), else BF_ETOPO.                  */
int bf_topology_put(bf_ctx* ctx, const bf_topology* topo, uint32_t* slot_out);
/* Bulk form: `count` topologies, one bf_topology each; slots_out[count].      */
int bf_topology_put_many(bf_ctx* ctx, const bf_topology* topos, uint32_t count, uint32_t* slots_out);
/* Device-validated bulk upload (SURVEY 8 row f3): unknown deps are still checked on the host, acyclicity is
 * checked by a kernel over the uploaded records (one warp per topology, level-synchronous peeling) instead of
 * the host's Kahn pass.  status_out[i]: bit 0 = cycle detected (the topology is dropped, slots_out[i] =
 * 0xFFFFFFFF), bits 8.. = number of dependency levels.  Returns BF_OK even when some topologies are cyclic. */
int bf_topology_put_many_checked_on_device(bf_ctx* ctx, const bf_topology* topos, uint32_t count, uint32_t* slots_out,
                                           uint32_t* status_out);
/* Re-validate already uploaded topologies on the device (status words as above; 0xFFFFFFFF = unknown slot). */
int bf_topology_check(bf_ctx* ctx, const uint32_t* slots, uint32_t count, uint32_t* status_out);

/* Redrive closure (row f3): for each query (topology slot, step index) the set of steps a redrive from that step
 * resets — the step plus everything downstream of it inside its own group (resolveRedriveFromStepSet,
 * internal/controller/runs/storyrun_controller.go:535-558; findStepGroup :560-577).  masks_out[q][words], same bit
 * order as the ready masks.  BF_EINVAL for a step index >= S ("step %q not found", :541).  Host buffers, synchronous. */
int bf_topology_closure(bf_ctx* ctx, const uint32_t* slots, const uint32_t* steps, uint32_t count, uint32_t words,
                        uint32_t* masks_out);

int bf_topology_drop(bf_ctx* ctx, uint32_t slot);

/* Step timings of a topology slot: how long each sleep sleeps and when each gate or wait times out, for the tick commits that
 * arm the step timers of the steps they launch (bf_resident_commit_timed).  The reference sets a step's StartedAt when it
 * launches it (markStepState, step_executor.go:171-179; ensureStepStateTimes, step_state.go:25-33) and the deadline is StartedAt
 * plus the step's with.duration / with.timeout / with.pollInterval, so the timing is static per Story generation: `delay` in
 * clock units after the `now` of the arming commit, and `code` what the armed timer writes when it fires.
 * bf_topology_timings(slot, t, n) replaces the slot's set; n = 0 clears it.  Checked before anything changes, else BF_EINVAL and
 * nothing changed: the slot is alive; each step is below the slot's S and named at most once (any order); reserved is 0; the
 * step's type (its BF_SF_* flags at the put) allows the code:
 *   sleep: BF_DEC_SUCCEED or BF_DEC_FAIL;  gate: BF_DEC_TIMED_OUT or BF_DEC_FAIL;
 *   wait:  BF_DEC_TIMED_OUT, BF_DEC_PENDING (wake-only: its pollInterval) or BF_DEC_FAIL;  every other type: none.
 * Timings belong to the slot: bf_topology_drop discards them and a put that reuses the slot starts with none.  They change no
 * pass result, so the topology record, bf_topology_record_build and the touched ticks' slot bookkeeping ignore them.  The ctx
 * keeps them on the host and copies one table of all of them to the device at the first arming commit after a change; a ctx
 * that never calls this allocates and copies nothing for them.                                                              */
typedef struct bf_step_timing {  /* 8 B                                                                                       */
  uint16_t step;                 /* allStorySteps index, < S of the slot                                                     */
  uint8_t code;                  /* BF_DEC_*: what the armed timer writes when it fires                                      */
  uint8_t reserved;              /* 0                                                                                        */
  uint32_t delay;                /* clock units after `now` of the arming commit                                             */
} bf_step_timing;
int bf_topology_timings(bf_ctx* ctx, uint32_t slot, const bf_step_timing* timings, uint32_t n);
/* Nibble offset of parallel desc p's children inside the child area.          */
int bf_topology_child_first(const bf_ctx* ctx, uint32_t slot, uint32_t* child_first_out, uint32_t cap);

int bf_layout_init(bf_layout* out, uint32_t steps_max, uint32_t child_nibbles, uint32_t fields);

/* Synchronous pass over HOST buffers: H2D(state) -> kernels -> D2H(result),
 * returns when result/expansion/counts are filled.  Thread-safe per ctx.      */
int bf_eval(bf_ctx* ctx, const bf_batch* batch);

/* Asynchronous pass over DEVICE buffers on `stream` (a cudaStream_t): state,
 * result, expansion and counts are device pointers; nothing is synchronised.
 * counts must be zeroed by the caller unless BF_EVAL_NO_COUNTS or
 * BF_EVAL_COUNTS_SET (without them the library only adds).                    */
int bf_eval_device(bf_ctx* ctx, const bf_batch* batch, void* stream);

/* ------------------------------------------------------------------ limiters (SURVEY.md rows a9 / f4)
 * The consumer of the ready sets: findAndLaunchReadySteps applies enforceStoryConcurrency (dag.go:1780-1799)
 * and enforceSchedulingLimits (:1801-1861, with enforcePriorityOrdering :1910-1946 and effectivePriority
 * :1948-1961) to each run's ready LIST and keeps a prefix (readySteps[:slots]); the rest is marked
 * "Queued due to ...".  Ready masks are LSB-first = list order, so the prefix is "the first k set bits".
 *
 * Batch contract (one consistent snapshot per tick): first the counts the reference obtains from cluster LISTs
 * are REDUCED over the batch on the device —
 *   running StepRuns of a run = engram steps in phase Running + Running children of registered parallel steps
 *                               (StepState mirrors StepRun.Status.Phase after syncStateFromStepRuns, :965-1009),
 *   per story key / per queue key / global totals = host-supplied base (StepRuns the batch does not hold) + sum,
 *   per queue the highest effective priority among non-terminal runs with demand (storyRunHasDemand :1981-1999:
 *   run phase Running/Pending, or a step Running or queued) —
 * then every run is limited independently against them (StepRuns created in the same tick have no phase yet
 * and do not count, exactly as in the reference).  Host work that stays on the host: label -> key mapping,
 * time (queued_elapsed_s = int32((now - storyRunQueuedSince).Seconds()), BF_SCHED_NONE when nothing is queued
 * with a StartedAt), formatting "(%d running, limit %d)" from the totals returned here.
 * A run's own label priority is the priority its Story resolves to (ensureSchedulingLabels, scheduling.go:48-70).
 *
 * Edges (pinned by tests/test_gpu_schedule.py against oracle/limiters.py):
 *   - a story_key >= n_stories / queue_key >= n_queues is counted in no story / queue total and gets no story limit,
 *     no queue limit, no aging and no priority ordering; its Running steps still count globally, and the global
 *     limit still applies to it;
 *   - only the low 4 bits of run_phase are read;
 *   - a run whose slot was dropped or never put contributes no Running steps and no step demand; its run_phase
 *     still makes demand.  The slot table is read as it stands at the bf_schedule call: a slot dropped after the
 *     pass counts nothing, a slot reused since counts its new topology;
 *   - nothing is counted for phase codes at or past the topology's S, for registered bits >= its parallel step
 *     count, or for a parallel step whose children lie past the layout's child area; a topology wider than the
 *     layout (more words) counts nothing;
 *   - the reduction reads the state records as stored, also after BF_EVAL_FIXPOINT: the counts stand for the
 *     StepRuns of the cluster LISTs, which the in-memory iterations of runDagIterations do not change;
 *   - effective priority = priority + aging steps in int32 arithmetic that wraps, as in Go (dag.go:1960).
 */
#define BF_SCHED_NONE 0xFFFFFFFFu
enum {                       /* why the steps in queued_sched were queued                               */
  BF_QUEUED_NONE = 0,
  BF_QUEUED_PRIORITY = 1,    /* "Queued due to higher-priority work"      dag.go:1807-1811               */
  BF_QUEUED_GLOBAL = 2,      /* "Queued due to global concurrency limit"  dag.go:1849-1850               */
  BF_QUEUED_QUEUE = 3,       /* "Queued due to queue concurrency limit"   dag.go:1851-1852               */
  BF_QUEUED_OTHER = 4        /* "Queued due to scheduling limits"         dag.go:1853-1855               */
};

typedef struct bf_sched_run { /* 32 B per run                                                           */
  uint32_t story_key;         /* index into the story tables (namespace + Story name)                    */
  uint32_t queue_key;         /* index into the queue tables (queueLabelValue of the scheduling decision)*/
  int32_t priority;           /* schedulingDecision.Priority == the run's priority label                 */
  uint32_t queued_elapsed_s;  /* seconds queued, BF_SCHED_NONE if no queued step has a StartedAt         */
  uint32_t run_phase;         /* BF_PHASE_* of StoryRun.Status.Phase                                     */
  uint32_t reserved[3];
} bf_sched_run;

typedef struct bf_sched_tables {
  uint32_t struct_size;
  uint32_t n_stories, n_queues;
  int32_t global_limit;                /* scheduling.globalConcurrency, <= 0: none                       */
  uint32_t global_running_base;
  const int32_t* story_limit;          /* [n_stories] Story.spec.policy.concurrency, <= 0: none          */
  const uint32_t* story_running_base;  /* [n_stories] or NULL (zeros)                                     */
  const int32_t* queue_limit;          /* [n_queues]  queues[q].concurrency, <= 0: none                  */
  const int32_t* queue_aging_s;        /* [n_queues]  queues[q].priorityAgingSeconds, <= 0: no aging      */
  const uint32_t* queue_running_base;  /* [n_queues] or NULL (zeros)                                      */
  const int32_t* queue_max_priority_base; /* [n_queues] highest effective priority among non-terminal runs with demand that the
                                          batch does NOT hold (other shards, runs the batcher left out), INT32_MIN where none;
                                          NULL = none anywhere.  enforcePriorityOrdering (dag.go:1917-1944) compares against
                                          EVERY non-terminal StoryRun of the queue, so a sharded / partial batch must be given
                                          the rest here (bf_group_schedule does the exchange between shards itself)          */
} bf_sched_tables;

typedef struct bf_sched_header { /* first 16 B of a schedule record                                     */
  uint32_t n_launch;             /* popcount(launch): steps to hand to StepExecutor.Execute              */
  uint32_t n_queued_story;       /* queued by the Story's own concurrency limit                          */
  uint32_t n_queued_sched;       /* queued by priority ordering / queue / global limits                  */
  uint32_t sched_reason;         /* BF_QUEUED_*                                                          */
} bf_sched_header;

/* schedule record of a run: bf_sched_header, then launch[words], queued_story[words], queued_sched[words]
 * (u32 bit masks, same bit order as ready); stride = BF_SCHED_STRIDE(words), a multiple of 16.           */
#define BF_SCHED_STRIDE(words) ((16u + 12u * (uint32_t)(words) + 15u) & ~15u)

typedef struct bf_sched_out {
  uint32_t struct_size;
  uint32_t reserved;
  void* records;                 /* [n_runs][BF_SCHED_STRIDE(layout.words)]                               */
  uint32_t* story_running;       /* [n_stories] totals used (base + batch), or NULL                       */
  uint32_t* queue_running;       /* [n_queues] or NULL                                                    */
  int32_t* queue_max_priority;   /* [n_queues] INT32_MIN when no run of the queue has demand, or NULL     */
  uint32_t* global_running;      /* [1] or NULL                                                           */
} bf_sched_out;

/* Host buffers.  Limits the ready sets of the batch evaluated by the IMMEDIATELY PRECEDING bf_eval on this
 * ctx (same n_runs and layout; its state and result records are still on the device).  Synchronous.      */
int bf_schedule(bf_ctx* ctx, const bf_batch* batch, const bf_sched_run* runs, const bf_sched_tables* tables,
                bf_sched_out* out);
/* Device buffers: batch->state / batch->result as for bf_eval_device, runs / table arrays / out arrays are
 * device pointers (totals arrays are required here: they are the reduction scratch).  Asynchronous on `stream`. */
int bf_schedule_device(bf_ctx* ctx, const bf_batch* batch, const bf_sched_run* runs, const bf_sched_tables* tables,
                       bf_sched_out* out, void* stream);


/* ------------------------------------------------------------------ resident batches (SURVEY.md row f2)
 * Incremental state upload: the state records of a batch stay on the device and the host sends DELTAS — what
 * syncStateFromStepRuns (dag.go:965-1009) and the StepRun watch events (storyrun_controller.go:2116-2129) amount
 * to per tick: a handful of (run, step) phase changes — so the H2D traffic of a tick is O(changes), not O(N*S).
 * A delta rewrites one code of one record in place (bit-sliced fields: one bit per plane, by integer atomics).
 * Contract: within ONE bf_resident_apply call at most one delta per (run, field, index) — the host mirror
 * coalesces (the last value of a tick wins); deltas of different steps that share a word are fine.              */
enum {
  BF_DELTA_PHASE = 0,       /* index = step, code = BF_PHASE_* (0..14)                                           */
  BF_DELTA_COND = 1,        /* index = step, code = BF_COND_*                                                    */
  BF_DELTA_DECISION = 2,    /* index = step, code = BF_DEC_*                                                     */
  BF_DELTA_CHILD = 3,       /* index = child nibble (child_first[p] + branch), code = BF_PHASE_*                 */
  BF_DELTA_RUN_FLAGS = 4,   /* index ignored, code = BF_RF_* byte                                                */
  BF_DELTA_REGISTERED = 5,  /* index = parallel desc p, code = 0 / 1 (children_registered bit)                   */
  BF_DELTA_TOPO_SLOT = 6    /* index = low 16 bits, code = bits 16-23 of the new topology slot (slot < 2^24)     */
};
typedef struct bf_delta { /* 8 B */
  uint32_t run;
  uint16_t index;
  uint8_t field; /* BF_DELTA_* */
  uint8_t code;
} bf_delta;

/* A resident batch of up to `capacity` runs with the given layout; *handle_out identifies it on this ctx.       */
int bf_resident_create(bf_ctx* ctx, const bf_layout* layout, uint32_t capacity, uint32_t* handle_out);
int bf_resident_destroy(bf_ctx* ctx, uint32_t handle);
/* Full records for runs [first_run, first_run + n_runs) (new StoryRuns, or a resync): host buffer, synchronous.  */
int bf_resident_upload(bf_ctx* ctx, uint32_t handle, uint32_t first_run, uint32_t n_runs, const void* state_records);
/* Apply n deltas (host buffer; copied and scattered on the ctx stream, synchronous).                            */
int bf_resident_apply(bf_ctx* ctx, uint32_t handle, const bf_delta* deltas, uint32_t n);
/* One pass over runs [0, n_runs) of the resident state: kernels + D2H of the result records (host buffer) and
 * counts.  flags = BF_EVAL_* (expansion is not offered on this path).  Also the batch bf_schedule refers to.     */
int bf_resident_eval(bf_ctx* ctx, uint32_t handle, uint32_t n_runs, uint32_t flags, uint32_t max_iterations, void* result,
                     bf_counts* counts);
/* A whole tick in one call and one synchronisation: apply n_deltas deltas (may be 0), run the pass, read the results
 * (the kernels of later run chunks overlap the download of earlier ones).                                       */
int bf_resident_tick(bf_ctx* ctx, uint32_t handle, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs, uint32_t flags,
                     uint32_t max_iterations, void* result, bf_counts* counts);
/* Read the device copy back (tests / resync checks).                                                            */
int bf_resident_download(bf_ctx* ctx, uint32_t handle, uint32_t first_run, uint32_t n_runs, void* state_records);

/* ------------------------------------------------------------------ compact results
 * What the consumer of a pass needs (findAndLaunchReadySteps, dag.go:1735-1775) is two short LISTS per run — the
 * ready steps to hand to StepExecutor.Execute and the skipped steps to mark — plus the run's summary flags, not 80+
 * bytes of masks per run.  The compact entry points turn the result masks into lists ON THE DEVICE and ship only
 * those:
 *   head[r]   one u32 per run: low 15 bits = low bits of the run's BF_SUM_* word (group, done / failed flags,
 *             PHASE_CHANGED; 0x7FFF = dead topology slot), bit 15 = the run's events are in this call's list,
 *             high 16 bits = how many.  The fixpoint iteration count of the summary word is not carried.
 *   events[]  one u16 per (run, step) that has any result bit set: step | kind << 10, run-major in batch order and
 *             step-ascending inside a run (the order of the reference's lists); run r's events are the next
 *             head[r] >> 16 entries.
 * At BASELINE configs[2] that is 0.4 MB + ~0.6 MB per pass instead of 8 MB of mask records.  The dense records stay
 * on the device (bf_schedule may follow).
 * BF_EVAL_CHANGED_ONLY (resident ticks): only runs whose result record differs from the PREVIOUS tick's carry
 * BF_HEAD_LISTED and events — the batcher keeps the last row of every run anyway (INTEGRATION.md), so a steady-state
 * tick returns O(changes) in both directions.  The first tick after bf_resident_create / _upload lists every run.   */
#define BF_EVT_READY 0x1u      /* step is in `ready`                                                            */
#define BF_EVT_SKIP 0x2u       /* step is in `skip`  (failed dependency or `if` false)                          */
#define BF_EVT_FAIL 0x4u       /* step is in `fail`        (only when the layout has BF_F_OUT_FAIL)              */
#define BF_EVT_NEEDS_COND 0x8u /* step is in `needs_cond`  (only with BF_F_OUT_NEEDS_COND)                       */
#define BF_EVT_SKIP_DEP 0x10u  /* step is in `skip_dep`    (only with BF_F_OUT_SKIP_DEP)                         */
#define BF_EVENT_STEP(e) ((uint32_t)(e) & 0x3FFu)
#define BF_EVENT_KIND(e) ((uint32_t)(e) >> 10)
#define BF_HEAD_SUMMARY_MASK 0x7FFFu
#define BF_HEAD_DEAD 0x7FFFu   /* low bits of a run whose topology slot is dead: no events                       */
#define BF_HEAD_LISTED 0x8000u
#define BF_HEAD_COUNT_SHIFT 16
#define BF_EVAL_CHANGED_ONLY 0x10u /* flag of bf_resident_tick_compact                                           */

typedef struct bf_compact_out {
  uint32_t struct_size;
  uint32_t n_listed;           /* out: runs that carry BF_HEAD_LISTED                                            */
  uint32_t* head;              /* [n_runs]                                                                       */
  uint16_t* events;            /* [events_cap]                                                                   */
  uint64_t events_cap;
  uint64_t n_events;           /* out: events the pass produced; when > events_cap only the first events_cap were written
                                  (heads always carry the true counts)                                           */
} bf_compact_out;

/* bf_eval with compact results: H2D(state) -> kernels -> D2H(heads + events).  batch->result is ignored
 * (may be NULL).  Host buffers, synchronous.                                                                     */
int bf_eval_compact(bf_ctx* ctx, const bf_batch* batch, bf_compact_out* out);
/* bf_resident_tick with compact results: deltas -> scatter -> pass -> heads + events.  This is the steady-state
 * tick of the operator: both directions are proportional to what changed.  Buffers in PINNED host memory
 * (bf_alloc_pinned, cudaHostAlloc, cudaHostRegister) are used in place: the scatter kernel reads the deltas from
 * them and the compaction kernel posts head words and events into them, with no staging copy on either side;
 * any other buffer goes through the upload / download copies.  Either way the call returns when they are filled. */
int bf_resident_tick_compact(bf_ctx* ctx, uint32_t handle, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs,
                             uint32_t flags, uint32_t max_iterations, bf_compact_out* out, bf_counts* counts);

/* ------------------------------------------------------------------ touched ticks
 * The steady-state tick of a batcher that ticks often: only the runs that changed are evaluated and listed, so both the work
 * and the traffic of a tick follow the number of changes, not n_runs.  A run's result is a function of its state record, its
 * topology and the pass parameters alone, and the state changes only through deltas and uploads, so a run that received
 * neither since it was last evaluated would not be listed by a BF_EVAL_CHANGED_ONLY tick either.
 *   touched run   a run in [0, n_runs) that received a delta (this call's, bf_resident_apply's or an earlier tick's; applied
 *                 or rejected) or an upload since the last tick that evaluated it.  Touched runs at or above n_runs stay
 *                 touched for a later tick that covers them.
 *   listed run    a touched run whose new result record differs from the one it had (the bytes BF_EVAL_CHANGED_ONLY compares),
 *                 or that was uploaded since it was last listed (the batcher has no row for it).
 * With full == 0, runs / head / events are exactly what a BF_EVAL_CHANGED_ONLY compact tick on the same device state gives for
 * its listed runs: the same head words and the same events in the same order (ascending run index).  counts covers the
 * evaluated runs only (evals = sum of S over them).
 * The tick evaluates every run in [0, n_runs), lists them all (runs[i] = i) and sets full = 1 when: no tick has run on the batch
 * yet (or the last one failed); a slot of the ctx was dropped, or a put reused a dropped slot, since the last tick (a dropped
 * slot kills its runs, a reused one re-points them); BF_EVAL_FIXPOINT or max_iterations differs from the last tick's; bf_resident_reshape added
 * decision planes or an output field since, or bf_resident_narrow dropped decision planes, the child area or an output field
 * (each may change any run's result); or n_runs exceeds the run count of the last full evaluation and not
 * every run beyond it was uploaded since.  A run may hold only a slot a put has returned (alive or dropped since): a put that
 * creates a new slot index is not a change, so runs that already held that index (by a delta or an upload) keep the dead
 * result of their last evaluation until they are touched again.  Any tick of the other kinds (bf_resident_tick,
 * _eval, _tick_compact) may come between touched ticks, and bf_schedule may follow a touched tick.
 * flags: BF_EVAL_FIXPOINT and BF_EVAL_NO_COUNTS only (else BF_EINVAL).  Pinned buffers are used in place as by
 * bf_resident_tick_compact; the call returns when they are filled.                                                  */
typedef struct bf_touched_out {
  uint32_t struct_size;
  uint32_t full;               /* out: 1 when the tick evaluated and listed every run in [0, n_runs) (see above)         */
  uint32_t* runs;              /* [runs_cap] out: ascending indices of the listed runs                                  */
  uint32_t* head;              /* [runs_cap] out: head word of runs[i], same bits as bf_compact_out.head                */
  uint32_t runs_cap;
  uint32_t n_listed;           /* out: listed runs; only the first runs_cap are written when larger                      */
  uint32_t n_evaluated;        /* out: runs the pass evaluated                                                           */
  uint32_t reserved;
  uint16_t* events;            /* [events_cap] out: events of the listed runs, same format and order as the compact lists */
  uint64_t events_cap;
  uint64_t n_events;           /* out: as bf_compact_out.n_events                                                        */
} bf_touched_out;

int bf_resident_tick_touched(bf_ctx* ctx, uint32_t handle, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs,
                             uint32_t flags, uint32_t max_iterations, bf_touched_out* out, bf_counts* counts);

/* Touched ticks of several resident batches of one ctx in one call, e.g. one batch per width class (INTEGRATION.md step 5).
 * Each part is one bf_resident_tick_touched: its handle, deltas, n_runs, out and counts mean what that call's arguments mean;
 * flags and max_iterations are shared.
 *   - Equivalence: every batch and touch mark, every counts block, the out fields and the listed entries of runs / head /
 *     events (the first min(n_listed, runs_cap) and min(n_events, events_cap)) end as after calling bf_resident_tick_touched
 *     once per part in array order, including the full rules, the truncation at the caps with true counts and the tick that
 *     bf_resident_schedule and the commits read.  Entries past those are not defined by either call.
 *   - Refusals come first: flags (as bf_resident_tick_touched takes them) and parts, then every part (struct_size, a live
 *     handle, n_runs within the batch, the out, runs, head and events pointers, null deltas), and no two parts may name one
 *     batch.  On a refusal the call returns BF_EINVAL, *bad_part names the first bad part (BF_COMMIT_NONE for bad flags, null
 *     parts or a null ctx) and nothing changed.
 *   - Deltas are handled as by the single call: a rejected delta still touches its run and the others are applied; every part
 *     still ticks, and the call returns BF_EINVAL with *bad_part = the first part that had a rejected delta.
 *   - Any other failure (BF_ECUDA, BF_ENOMEM) returns with *bad_part = the part it was met in.  Parts may then have ticked, in
 *     part or not at all: the next touched tick of every part is full, and the caller resends every part's deltas (a delta
 *     writes a code, so one applied twice changes nothing).
 *   - The parts whose ticks are not full run together: one scatter launch over all their deltas, one list build over all their
 *     touch marks, one pass per part back to back, one compaction over all their lists, one synchronisation.  Pinned buffers
 *     are written in place; pageable ones are copied back once their lengths are known.  A part whose tick is full (see above)
 *     runs as its single call does, with a synchronisation of its own.
 * n_parts == 0 is a no-op; *bad_part = BF_COMMIT_NONE on success (bad_part may be NULL).                                      */
typedef struct bf_tick_part {
  uint32_t struct_size;          /* sizeof(bf_tick_part)                                                                 */
  uint32_t handle;               /* resident batch of this ctx                                                           */
  const bf_delta* deltas;        /* as bf_resident_tick_touched                                                          */
  uint32_t n_deltas;
  uint32_t n_runs;
  bf_touched_out* out;           /* as bf_resident_tick_touched (full, runs, head, events)                               */
  bf_counts* counts;             /* may be NULL                                                                          */
} bf_tick_part;

int bf_resident_tick_touched_many(bf_ctx* ctx, uint32_t flags, uint32_t max_iterations, bf_tick_part* parts, uint32_t n_parts,
                                  uint32_t* bad_part);

/* ------------------------------------------------------------------ migrations (a Story edited while its runs are live)
 * The reference does not pin a StoryRun to the Story generation it started with: every reconcile loads the current Story
 * (getStoryForRun, storyrun_controller.go:1297-1313) and walks allStorySteps of that spec, with StepStates, Gates and
 * PrimitiveChildren keyed by step name (buildStateMaps ignores names the list no longer has, dag.go:3373-3376).  Here state is
 * kept by step INDEX, and an edit moves indices.  bf_resident_migrate re-indexes, in place on the device, every run in
 * [0, n_runs) whose header holds old_slot, so that its record equals what packing its by-name state against new_slot gives:
 *   - new step j carries the phase / cond / decision codes of the old step mapped to j; steps without one carry 0;
 *   - a parallel desc of new_slot whose step is the image of an old parallel step takes that step's children_registered bit
 *     and child nibbles (branches matched by index); other descs start unregistered with zero nibbles;
 *   - topo_slot = new_slot; run_flags and every other run are untouched (a changed policy travels as BF_DELTA_RUN_FLAGS).
 * Checked before anything runs, else BF_EINVAL / BF_ETOPO and nothing changed: both slots alive and different; n_old_steps ==
 * S of old_slot; the map injective with targets below S of new_slot; both topologies fit the batch layout (steps_max,
 * child_nibbles); every surviving parallel step keeps its branch count (else BF_EINVAL: re-pack those runs on the host).
 * Migrated runs are touched and must be listed by the next bf_resident_tick_touched, as uploaded runs are; a changed-only
 * compact tick lists them when their result record changed.  Like an upload, the call ends the evaluated snapshot (bf_schedule
 * must follow a new pass).  A step name removed in an earlier generation and re-added now starts at 0: the caller sends deltas
 * for it.  One launch and one synchronisation.                                                                        */
#define BF_MIGRATE_GONE 0xFFFFu
typedef struct bf_migration {
  uint32_t struct_size;        /* sizeof(bf_migration)                                                         */
  uint32_t old_slot, new_slot;
  uint32_t n_runs;             /* runs [0, n_runs) of the resident batch are considered                        */
  const uint16_t* step_map;    /* [n_old_steps]: new index of old step i, or BF_MIGRATE_GONE; injective         */
  uint32_t n_old_steps;        /* must equal S of old_slot                                                     */
  uint32_t migrated;           /* out: runs whose header held old_slot and were moved                          */
} bf_migration;

int bf_resident_migrate(bf_ctx* ctx, uint32_t handle, bf_migration* m);

/* ------------------------------------------------------------------ redrives (an operator re-drives a live run)
 * Redrive from a step (annotation <step>:<token>, handleRedriveFromStepIfRequested, storyrun_controller.go:293-348): the reset
 * set R is the step plus everything downstream of it inside its own group (resolveRedriveFromStepSet :535-558, the set
 * bf_topology_closure returns), and resetStoryRunForStepRedrive (:740-789) deletes StepStates, Gates and PrimitiveChildren of
 * every step of R and clears Conditions.  Redrive of the whole run (token annotation, resetStoryRunForRedrive :415-439) clears
 * all four for every step: step = BF_REDRIVE_ALL, R = every step of the topology.
 * For each request whose run's header holds `slot` (status_out[i] = 1) bf_resident_redrive sets, in place on the device:
 *   - the phase code of every step of R to 0 (delete(StepStates, ...));
 *   - the decision code to BF_DEC_PENDING (delete(Gates, ...)), when the layout has decision planes;
 *   - the cond code, when the layout has cond planes, to BF_COND_HOLD for steps with BF_SF_HAS_IF and BF_COND_PASS for the
 *     others.  Cond codes are host inputs, not reference state: those of R were computed from outputs the redrive discards
 *     (their StepRuns are deleted).  HOLD is what the lazy needs_cond protocol gives an `if` the host has not evaluated yet,
 *     so no redriven `if` step launches on a stale verdict; the host sends the fresh cond code as a delta when it has one;
 *   - the children_registered bit of every parallel desc whose step is in R to 0, and that desc's child nibbles to 0
 *     (delete(PrimitiveChildren, ...)); nibbles past the desc's branches (padding) are kept;
 *   - BF_RF_TOPOLOGY_TERMINATED in run_flags to 0 (Conditions = nil: the Degraded/TopologyTerminated condition, dag.go:436-464).
 * Every other run_flags bit, the slot and every step outside R are unchanged.  A request whose run holds another slot (stale
 * request, dead slot, never uploaded) changes nothing and gets status_out[i] = 0.  Several requests may name the same run: the
 * result is the union of their resets (each reset is idempotent, as the reference's annotations applied one at a time are).
 * Checked before anything runs, else BF_EINVAL / BF_ETOPO and nothing changed: the handle; run < capacity; slot alive;
 * step < S of slot or BF_REDRIVE_ALL ("step %q not found", :539-541); reserved == 0; the slot's topology fits the batch layout
 * (steps_max, child_nibbles).  *applied_out = the requests with status 1.
 * Ordering: a redrive applies at the call; deltas given afterwards (bf_resident_apply, the next tick) apply after it.  Applied
 * runs are touched as by a delta: the next bf_resident_tick_touched evaluates them and lists those whose result changed.  Like
 * an upload, the call ends the evaluated snapshot (bf_schedule must follow a new pass).  One H2D copy, the closure launch
 * (when a request names a step), one redrive launch, one D2H copy and one synchronisation.                              */
#define BF_REDRIVE_ALL 0xFFFFFFFFu
typedef struct bf_redrive {    /* 16 B, no pointers                                                                   */
  uint32_t run;                /* index in the resident batch                                                         */
  uint32_t slot;               /* topology slot the caller holds the run on                                           */
  uint32_t step;               /* allStorySteps index of the redrive-from step, or BF_REDRIVE_ALL (the whole run)     */
  uint32_t reserved;           /* 0                                                                                   */
} bf_redrive;

int bf_resident_redrive(bf_ctx* ctx, uint32_t handle, const bf_redrive* requests, uint32_t n, uint8_t* status_out,
                        uint32_t* applied_out);

/* ------------------------------------------------------------------ reshapes (a live batch outgrows its shape)
 * bf_resident_create fixes a batch's capacity and layout.  bf_resident_reshape grows both in place, keeping every run's state,
 * the current result records and the touch marks, so that a batcher can keep the tightest layout its live Stories allow and
 * widen it when a larger Story, a parallel step with more branches, the first `if` or gate, or more runs arrive.
 * Growth only.  `layout` passes the checks of bf_resident_create, and else BF_EINVAL and nothing changed: a known handle;
 * capacity >= the current capacity; layout->steps_max >= the current steps_max; layout->fields a superset of the current
 * fields (input and output fields alike), and every field the current layout places is placed by the new one too;
 * layout->child_nibbles >= the current child_nibbles when the batch has BF_F_CHILD.  Should an allocation fail, BF_ENOMEM and
 * nothing changed: the new buffers are allocated before the old ones are freed, and those are freed after the copy completed.
 * Afterwards, by the bytes:
 *   - state record r < old capacity equals pack_state of the same codes at the new layout: the header (slot, run flags,
 *     children_registered) as it was; each phase / cond / decision plane its old words, zero words above them; the planes of
 *     an added field zero (the host sends the real codes as deltas); the child area its old bytes, the rest zero (child_first
 *     does not depend on the layout: child delta indices stay valid); every other byte zero.  Records r >= old capacity are
 *     zero, as after create.  Zero cond planes are BF_COND_PASS, which is how a pass reads absent ones; zero decision planes
 *     are BF_DEC_PENDING, which a pass applies to RUNNING gate / sleep / wait steps where absent planes leave them alone;
 *   - the current result records (those BF_EVAL_CHANGED_ONLY and touched ticks compare with) are re-laid out the same way:
 *     header kept; each mask and phase_out plane its old words, zeros above them (exactly what a pass at the new layout
 *     writes for an unchanged run); the masks of an added output field zero;
 *   - touch marks and the touched-tick bookkeeping are kept; the runs of the new capacity start untouched.
 * So with neither decision planes nor an output field added, the next touched tick is not full and evaluates only the runs
 * touched before or after the call, and the next changed-only tick lists what it would have listed without it.  With
 * decision planes or an output field added (e.g. BF_F_OUT_NEEDS_COND with BF_F_COND) the next touched tick is full; a
 * changed-only tick lists the runs whose result changed, the zeroed new masks and planes included.  Like an upload, the call ends the evaluated snapshot (bf_schedule must follow a new pass).  bf_stats and the
 * ctx's staging buffers are unaffected.  One launch, one device copy of the marks and one synchronisation.
 * Shrinking a batch or dropping a field is bf_resident_retire's (capacity) and bf_resident_narrow's (layout) job.         */
int bf_resident_reshape(bf_ctx* ctx, uint32_t handle, const bf_layout* layout, uint32_t capacity);

/* ------------------------------------------------------------------ retirements (runs leave a live batch)
 * The reference stops evaluating a StoryRun once it is terminal (handleTerminalStoryRun, storyrun_controller.go:282-288) and
 * retention deletes it later.  bf_resident_retire takes such runs out of a live batch, so that passes, ticks and memory follow
 * the live runs instead of every run the batch ever held.  The batch's runs are [0, n_runs); `runs` lists n of them.  The last
 * live runs move into the indices the retired ones free, by a rule the host can compute itself: with m = n_runs - n, the
 * retired indices below m ("holes", ascending) receive the live indices of [m, n_runs) ("sources", ascending), hole k source k.
 * Runs below m that are not retired keep their index.  moves_from / moves_to (each may be NULL) receive the n_moves moves,
 * ascending by target (and by source); a batcher re-keys its rows by them.  Afterwards, by the bytes:
 *   - the state record and the current result record (those BF_EVAL_CHANGED_ONLY and touched ticks compare with) at each target
 *     equal the source's; state records and touch marks in [m, old n_runs) are zero, as after bf_resident_create;
 *   - records at or above the old n_runs are not runs for this call: they keep their bytes and marks below the capacity;
 *   - with capacity != 0 the buffers are reallocated at that size (new ones are allocated and filled before the old ones are
 *     freed); records from the capacity on are released.  The layout does not change.
 * Touched ticks: every moved run is touched and must be listed by the next bf_resident_tick_touched, as an uploaded run is, so
 * the batcher gets a row under its new index.  The call never makes the next touched tick full by itself: the run count of the
 * last full evaluation drops to m at most, the runs uploaded since are kept below m only, and the moved runs count as uploaded.
 * A later tick over more than m runs is full unless uploads cover the difference, as before.  A BF_EVAL_CHANGED_ONLY tick over
 * [0, m) right after the call lists what it would list had every moved run always had its new index (when the last tick
 * covered the old n_runs; otherwise it lists every run).  Like an upload, the call ends the evaluated snapshot (bf_schedule must
 * follow a new pass).
 * Checked before anything changes, else BF_EINVAL and nothing changed: struct_size and the handle; n_runs <= capacity of the
 * batch; runs not NULL when n > 0; every index below n_runs, none twice; capacity 0 or within [m, current capacity].  A failed
 * allocation is BF_ENOMEM and changes nothing.  n == 0 with capacity set only trims the capacity; n == 0 without is a no-op.
 * One H2D copy of the move table, one launch and one synchronisation, plus the copies into the new buffers of a new capacity.
 * What is terminal is the host's decision: the device does not retire runs by itself.                                    */
typedef struct bf_retire {
  uint32_t struct_size;        /* sizeof(bf_retire)                                                                   */
  uint32_t n_runs;             /* in: the batch's runs are [0, n_runs); out: n_runs - n                               */
  const uint32_t* runs;        /* [n] indices to retire: distinct, each < n_runs, any order                           */
  uint32_t n;
  uint32_t capacity;           /* 0 = keep; else the new capacity, new n_runs <= capacity <= current                  */
  uint32_t* moves_from;        /* [n] out, may be NULL: run moves_from[i] now lives at moves_to[i]                    */
  uint32_t* moves_to;          /* [n] out, may be NULL                                                                */
  uint32_t n_moves;            /* out                                                                                 */
} bf_retire;

int bf_resident_retire(bf_ctx* ctx, uint32_t handle, bf_retire* r);

/* ------------------------------------------------------------------ narrowings (a live batch sheds the shape its wide Stories needed)
 * bf_resident_reshape only grows a layout, so one 200-step Story, one `if` or one `parallel` step would cost every later pass its
 * width, planes and child area for the life of the batch.  bf_resident_extent reports the smallest layout the batch's contents
 * allow, and bf_resident_narrow re-lays the batch to a smaller one in place once the Stories that needed the width have left.
 * The extent of runs [0, n_runs) is taken over three sets:
 *   - the topology slot of each run below n_runs whose slot is alive: its S counts towards steps_max, its child area towards
 *     child_nibbles (what bf_resident_migrate and _redrive require of a slot: it fits the layout);
 *   - every state record below the capacity, records at or above n_runs included (a batcher may upload ahead): the highest step
 *     with a non-zero phase, cond or decision code sets steps_max, the highest non-zero child nibble below the layout's
 *     child_nibbles sets child_nibbles; a non-PASS cond code, a non-PENDING decision code and a non-zero child nibble set
 *     BF_F_COND, BF_F_DECISION and BF_F_CHILD in `fields`;
 *   - the current result record of each run below n_runs that a later tick compares with: the runs a BF_EVAL_CHANGED_ONLY tick
 *     would compare over (when one would), and, unless the next touched tick is full, the runs of the last full evaluation and
 *     the runs uploaded since that a touched tick has evaluated, except runs uploaded, migrated or moved since their last
 *     evaluation (a touched tick lists those whatever their record holds).  Records never written by a pass (a batch before its
 *     first tick) therefore never count.  The highest set bit of a mask or phase_out plane counts towards steps_max;
 *     bf_resident_narrow counts only the planes the new layout keeps, bf_resident_extent all of them.
 * widest_run is the lowest index of a run (or a record, when it lies at or above n_runs) that needs all of steps_max.
 * bf_resident_narrow(layout T) accepts exactly this region.  Checked before anything changes, else BF_EINVAL, nothing changed and
 * `e` still filled (so that the caller sees why): n_runs <= capacity; T passes the checks of bf_resident_create; T grows no
 * dimension (T.steps_max <= the current steps_max, T.fields a subset of the current fields, every field T places placed by the
 * current layout too, T.child_nibbles <= the current child_nibbles when both have BF_F_CHILD); T.steps_max >= e.steps_max;
 * T.child_nibbles >= e.child_nibbles when T has BF_F_CHILD; T.fields a superset of e.fields (an input plane holding a
 * non-default code is never dropped).  Output fields may always be dropped: they hold results, not codes.  T equal to the
 * current layout is BF_OK and changes nothing.  Should an allocation fail, BF_ENOMEM and nothing changed.
 * Afterwards, by the bytes (the capacity does not change: bf_resident_retire owns it):
 *   - every state record equals pack_state of the same codes at T: the header as it was, each plane its low T.words words, the
 *     child area its low bytes;
 *   - every current result record equals what a pass at T writes for an unchanged run: the header as it was, each kept mask and
 *     phase_out plane its low T.words words, dropped masks gone.
 * Touched ticks: narrowing steps_max or child_nibbles, and dropping cond planes (all PASS, as absent planes read), keep the touch
 * marks and the touched-tick bookkeeping, so the next touched tick stays incremental.  Dropping decision planes (zero planes are
 * PENDING, which a pass applies; absent ones skip it), the child area (a registered parallel step without branches joins with an
 * area and not without one) or an output field (the event kinds change) makes the next touched tick full.  Result records at or
 * above n_runs were not checked, so the run count of the last full evaluation drops to n_runs at most and a BF_EVAL_CHANGED_ONLY
 * tick over more than n_runs runs lists every run, as after bf_resident_retire.  Like an upload, the call ends the evaluated
 * snapshot (bf_schedule must follow a new pass).  bf_resident_narrow: the extent launch, the re-layout launch and a device copy
 * of the marks into new buffers, one synchronisation; the new buffers replace the old ones only when the extent passes.
 * bf_resident_extent: one launch, one synchronisation, nothing changed.                                                   */
#define BF_EXTENT_NO_RUN 0xFFFFFFFFu
typedef struct bf_extent {
  uint32_t struct_size;        /* sizeof(bf_extent)                                                                   */
  uint32_t n_runs;             /* in: the batch's runs are [0, n_runs), n_runs <= capacity                            */
  uint32_t steps_max;          /* out: the smallest steps_max a narrow accepts (>= 1)                                 */
  uint32_t child_nibbles;      /* out: the smallest child_nibbles a narrow that keeps BF_F_CHILD accepts              */
  uint32_t fields;             /* out: input fields (BF_F_COND / _DECISION / _CHILD) holding a non-default code       */
  uint32_t widest_run;         /* out: the lowest run index that needs steps_max, BF_EXTENT_NO_RUN when none does     */
  uint32_t reserved[2];        /* 0                                                                                   */
} bf_extent;

int bf_resident_extent(bf_ctx* ctx, uint32_t handle, bf_extent* e);
int bf_resident_narrow(bf_ctx* ctx, uint32_t handle, const bf_layout* layout, bf_extent* e);

/* ------------------------------------------------------------------ transfers (live runs move between batches of one ctx)
 * A batch has one layout, and every run in it pays for that layout on every pass: one Story of more than 512 steps moves the
 * whole batch from the packed-lanes kernel to the one-run-per-warp one.  A batcher keeps width classes instead (several batches
 * in one ctx, e.g. <= 64, <= 512 and <= 1024 steps, with and without decision planes or a child area; topology slots belong to
 * the ctx, so a slot is valid in every batch of it).  bf_resident_transfer moves live runs from the batch src_handle to the
 * batch dst_handle of the same ctx: when a Story edit changes a run's class, or a straggler holds a batch's width.
 * The source's runs are [0, src_n_runs), the destination's [0, dst_n_runs); `runs` lists n distinct source runs, any order.
 * Afterwards, by the bytes, with F the source layout and T the destination's:
 *   - runs[i] lives at destination index dst_n_runs + i.  Its state record equals pack_state of the same codes at T: the header
 *     as it was, each plane its low words with zero words above them, planes F lacks zero (cond PASS; decision PENDING, which a
 *     pass applies where absent planes do not, exactly as after bf_resident_reshape), the child area its low bytes.  Its
 *     current result record is what a pass at T writes for an unchanged run: the header as it was, each mask and phase_out plane
 *     its low words, masks T lacks dropped, masks only T has zero.  Records at or above dst_n_runs before the call are not runs
 *     and the arrivals overwrite them; records from dst_n_runs + n on keep their bytes.
 *   - the source is byte-identical to bf_resident_retire of the same runs with capacity 0, and moves_from / moves_to receive
 *     the same moves.
 * Fit: each moved run must fit T under bf_resident_narrow's acceptance test applied to that run alone: the S and the child
 * area of its slot when alive; its state record (highest non-zero code, non-PASS cond and non-PENDING decision codes, non-zero
 * child nibbles); its current result record when a later tick of the source compares with it (the rule of bf_resident_extent),
 * counting the planes T keeps.  unfit is the position in runs[] of the first run T cannot hold, and `why` that run's own extent
 * (widest_run = its source index, or BF_EXTENT_NO_RUN when it needs no step).
 * Checked before anything changes, else BF_EINVAL and both batches byte-identical: struct_size and both handles, src_handle !=
 * dst_handle; src_n_runs <= the source capacity; dst_n_runs + n <= the destination capacity (bf_resident_reshape grows it
 * first); runs not NULL when n > 0, every index below src_n_runs, none twice; every run fits.  A failed allocation is BF_ENOMEM
 * and changes nothing.  n == 0 is a no-op.
 * Touched ticks: the source follows bf_resident_retire (moved runs are listed, the call never forces a full tick by itself).
 * In the destination the arrivals count as uploaded: the next bf_resident_tick_touched lists them and is not full because of
 * them.  A BF_EVAL_CHANGED_ONLY tick of the destination over [0, dst_n_runs + n) right after the call lists what it would list
 * had the arrivals always been there, when its last tick covered dst_n_runs and the source's last tick covered every moved
 * run (else it lists every run).  Both batches end their evaluated snapshot (bf_schedule must follow a new pass).
 * Cost: one H2D copy (runs and moves), the fit launch, one D2H copy and one synchronisation before anything is written; then
 * the transfer and retire launches and one synchronisation.  bf_resident_transfer_ctx moves runs to a batch of another ctx.  */
typedef struct bf_transfer {
  uint32_t struct_size;        /* sizeof(bf_transfer)                                                                 */
  uint32_t src_n_runs;         /* in: source runs are [0, src_n_runs); out: src_n_runs - n                            */
  uint32_t dst_n_runs;         /* in: destination runs are [0, dst_n_runs); out: dst_n_runs + n                      */
  const uint32_t* runs;        /* [n] source indices: distinct, each < src_n_runs, any order                          */
  uint32_t n;
  uint32_t* moves_from;        /* [n] out, may be NULL: the source's compaction moves, exactly bf_retire's            */
  uint32_t* moves_to;          /* [n] out, may be NULL                                                                */
  uint32_t n_moves;            /* out                                                                                 */
  uint32_t unfit;              /* out: position in runs[] of the first run T cannot hold, BF_EXTENT_NO_RUN when all fit */
  bf_extent why;               /* out on a fit refusal: that run's own extent                                         */
} bf_transfer;

int bf_resident_transfer(bf_ctx* ctx, uint32_t src_handle, uint32_t dst_handle, bf_transfer* t);

/* ------------------------------------------------------------------ transfers between ctxs (live runs move to another GPU)
 * bf_resident_transfer_ctx moves live runs from the batch src_handle of src_ctx to the batch dst_handle of dst_ctx, which may live
 * on another device: to rebalance a batcher's runs over its GPUs, or to drain one.  The contract is bf_resident_transfer's, for
 * two ctxs: afterwards both batches are byte for byte what bf_resident_transfer leaves when both live in one ctx (state and
 * current result records re-laid to the destination layout, timer slots, limiter inputs, run control, touch and commit
 * bookkeeping, the changed-only baseline rule, no schedule baseline for the arrivals, the moves), except one field: the topology
 * slot in each arrival's bf_run_header is slot_map[its source slot].
 * Slots belong to a ctx, so the caller puts the same Story generations into both ctxs and passes the map: slot_map[s] is the
 * destination slot of source slot s, or BF_SLOT_NONE.  Every entry other than BF_SLOT_NONE whose source slot is live must name a
 * live destination slot whose packed topology record (bf_topology_record) equals the source slot's byte for byte; the host
 * reads both records once per call for these entries.  A moved run whose slot is at or past n_slot_map, unmapped, or dead in the
 * source is unfit, as is every run bf_resident_transfer finds unfit; unfit_reason (BF_UNFIT_*) tells which.
 * Refused, with BF_EINVAL and both ctxs byte-identical: everything bf_resident_transfer refuses; src_ctx == dst_ctx (that is
 * bf_resident_transfer); a bad struct_size; slot_map NULL with n_slot_map > 0; a bad map entry as above.
 * Cost: on the source stream one H2D copy (runs, map, moves) and the gather launch (one warp per moved run packs its state and
 * result records and side-area entries, in the source layout, into the source ctx's scratch); one peer copy of that staging into
 * the destination ctx's scratch (cudaMemcpyPeerAsync, ordered by an event; a device-to-device copy when both ctxs share a
 * device); on the destination stream the fit launch, one D2H copy and one synchronisation before anything is written; then the
 * transfer launch on the destination stream and the retire launch on the source stream, and one synchronisation of each.  The
 * call holds both ctxs' locks, taken in address order.                                                                        */
#define BF_SLOT_NONE 0xFFFFFFFFu
enum {                          /* bf_ctx_transfer.unfit_reason                                                               */
  BF_UNFIT_NONE = 0,            /* every run fits                                                                             */
  BF_UNFIT_LAYOUT = 1,          /* the destination layout or its areas cannot hold the run (bf_resident_transfer's test)      */
  BF_UNFIT_SLOT_UNMAPPED = 2,   /* slot_map[slot] is BF_SLOT_NONE                                                             */
  BF_UNFIT_SLOT_PAST_MAP = 3,   /* slot >= n_slot_map                                                                         */
  BF_UNFIT_SLOT_DEAD = 4        /* the run's slot is not live in the source ctx                                               */
};
typedef struct bf_ctx_transfer {
  uint32_t struct_size;         /* sizeof(bf_ctx_transfer)                                                                    */
  uint32_t src_n_runs;          /* in / out, as bf_transfer                                                                   */
  uint32_t dst_n_runs;          /* in / out, as bf_transfer                                                                   */
  const uint32_t* runs;         /* [n] as bf_transfer                                                                         */
  uint32_t n;
  const uint32_t* slot_map;     /* [n_slot_map] source slot -> destination slot, BF_SLOT_NONE                                 */
  uint32_t n_slot_map;
  uint32_t* moves_from;         /* [n] out, may be NULL, as bf_transfer                                                       */
  uint32_t* moves_to;           /* [n] out, may be NULL                                                                       */
  uint32_t n_moves;             /* out                                                                                        */
  uint32_t unfit;               /* out: position in runs[] of the first unfit run, BF_EXTENT_NO_RUN when all fit              */
  uint32_t unfit_reason;        /* out: BF_UNFIT_* of that run                                                                */
  bf_extent why;                /* out on a fit refusal: that run's own extent                                                */
} bf_ctx_transfer;

int bf_resident_transfer_ctx(bf_ctx* src_ctx, uint32_t src_handle, bf_ctx* dst_ctx, uint32_t dst_handle, bf_ctx_transfer* t);

/* ------------------------------------------------------------------ step timers (time-driven transitions of a resident batch)
 * The reference compares `now` with each run's step timers on every reconcile: sleepUntil fires a sleep step (checkSyncSleepSteps,
 * dag.go:1217-1288), gateTimeoutAt and waitTimeoutAt time out a gate or a wait (dag.go:1455-1547, :1291-1452), the timers live per
 * step in the runs.bubustack.io/step-timers annotation (stepTimerStore, dag.go:64,110-171) and the nearest one sets the requeue
 * (setPollInterval :201-208, RequeueAfter :366-370).  A resident batch keeps these timers itself, in a side area of K slots per
 * run, so that retire, transfer, migrate and redrive re-key them with the runs and a batcher keeps no timer table of its own.
 * The area is separate from the state records: bf_layout and the record bytes do not change, and a batch that never calls
 * bf_resident_timers launches nothing more than before for any call.
 * Time is a u32 in units the host chooses, one clock for deadlines and `now` (suggested: seconds since the batcher's epoch; the
 * annotation's metav1.Time values have second resolution).  A timer is DUE iff deadline <= now (`remaining <= 0`, :1266;
 * `!now.Before(timeoutAt)`, :1434, :1529).
 * Slot layout, canonical so that downloads compare byte for byte: a run's armed slots first, ascending by step; an empty slot is
 * deadline = BF_TIMER_NONE with every other byte 0.
 *
 * bf_resident_timers(handle, K): creates the area (every slot empty) or grows K, keeping every armed slot.  1 <= K <= 64; a smaller
 *   K than the current one is BF_EINVAL.  bf_resident_destroy frees the area.
 * bf_resident_timers_arm(handle, req, n) (host buffer, synchronous): arms the timer of (run, step), replacing an armed one;
 *   deadline = BF_TIMER_NONE cancels it.  `code` is what firing writes as the step's decision code: BF_DEC_SUCCEED (a sleep),
 *   BF_DEC_TIMED_OUT (a gate or wait timeout), BF_DEC_FAIL, or BF_DEC_PENDING = wake-only (reported when due, writes nothing: a
 *   wait step's pollInterval, :1440, where the host re-evaluates `until`).  Checked before anything changes, else BF_EINVAL and
 *   nothing changed: the handle; the area exists; run < capacity, step < steps_max; code <= 3, reserved fields 0; a non-PENDING
 *   code needs decision planes (BF_F_DECISION); at most one request per (run, step).  A run whose K slots would overflow is
 *   BF_ENOMEM and nothing changed (bf_last_error names the run).  Arming touches no run.
 * bf_resident_fire(handle, now, out) over runs [0, out->n_runs), for each armed slot:
 *   - the step's phase code is terminal (BF_LUT_TERMINAL): the slot is disarmed ("pruned") and written nowhere, due or not
 *     (pruneTerminal, dag.go:173-190);
 *   - else, when due: disarmed and listed in `fired`.  When code != BF_DEC_PENDING and the step's decision code is still
 *     BF_DEC_PENDING, the code is written exactly as a BF_DELTA_DECISION delta writes it and the run is touched as by a delta
 *     (written = 1); an approve / reject already delivered takes precedence over a timeout (:1501-1533).  A due timer whose
 *     decision code is already set, or a wake-only one, is listed with written = 0 and touches nothing.
 *   Slots of runs at or above n_runs are untouched.  Deltas given later apply after the fire.  Like a delta, the fire ends the
 *   evaluated snapshot (bf_schedule must follow a new pass).  next_deadline is the batcher's next wake-up: the batch form of
 *   RequeueAfter.  Two launches, one D2H copy of the counts and one synchronisation; a fired list in pinned memory is written by
 *   the kernel in place, any other gets the entries that fired copied after the synchronisation.
 * bf_resident_timers_download(handle, first_run, n_runs, slots): the raw slots (n_runs * K of them), for tests and resyncs.
 *
 * What the other calls do to the area (each launches nothing more when the batch has none):
 *   upload: nothing.  retire: retired runs' slots are emptied, moved runs' slots move with them byte for byte, slots of
 *   [m, old n_runs) are emptied; a new capacity re-allocates the area.  transfer: the moved runs' armed slots arrive in the
 *   destination's canonical layout and the source follows retire; a moved run with more armed slots than the destination's K (0
 *   without an area) is unfit (BF_EINVAL, both batches byte-identical).  migrate: each slot of a migrated run is re-indexed
 *   through step_map and the run's slots re-sorted; a slot of a BF_MIGRATE_GONE step, or of a step at or above n_old_steps, is
 *   cancelled.  redrive: every slot of a run with status_out = 1 is emptied, for both kinds of request (the reference deletes
 *   the whole annotation, storyrun_controller.go:456-525).  reshape: a larger capacity extends the area with empty slots.
 *   extent / narrow / transfer fit: an armed slot at step s counts s + 1 towards steps_max (over every record below the
 *   capacity, as state records count) and a non-PENDING one sets BF_F_DECISION in `fields`, so a narrow never drops the decision
 *   planes a pending timeout needs nor the width of an armed step.                                                         */
#define BF_TIMER_NONE 0xFFFFFFFFu
#define BF_TIMER_MAX_SLOTS 64u
typedef struct bf_timer_slot {  /* 8 B                                                                                    */
  uint32_t deadline;            /* BF_TIMER_NONE: empty                                                                  */
  uint16_t step;
  uint8_t code;                 /* BF_DEC_*                                                                              */
  uint8_t reserved;
} bf_timer_slot;
typedef struct bf_timer {       /* 16 B arm request                                                                      */
  uint32_t run;
  uint16_t step;
  uint8_t code;                 /* BF_DEC_*: what firing writes; BF_DEC_PENDING = wake-only                             */
  uint8_t reserved;             /* 0                                                                                     */
  uint32_t deadline;            /* BF_TIMER_NONE cancels                                                                 */
  uint32_t reserved2;           /* 0                                                                                     */
} bf_timer;
typedef struct bf_fired {       /* 8 B                                                                                   */
  uint32_t run;
  uint16_t step;
  uint8_t code;                 /* the slot's code                                                                       */
  uint8_t written;              /* 1: the code was written into the decision planes and the run touched                 */
} bf_fired;
typedef struct bf_fire_out {
  uint32_t struct_size;         /* sizeof(bf_fire_out)                                                                   */
  uint32_t n_runs;              /* in: runs [0, n_runs) are fired, n_runs <= capacity                                    */
  uint32_t n_fired;             /* out: due timers listed (the true count, also past fired_cap)                          */
  uint32_t n_written;           /* out: of those, the ones that wrote their code                                         */
  uint32_t n_pruned;            /* out: slots disarmed because their step is terminal                                    */
  uint32_t next_deadline;       /* out: earliest deadline still armed in [0, n_runs), or BF_TIMER_NONE                   */
  bf_fired* fired;              /* [fired_cap] out: ascending by run, then by step                                       */
  uint32_t fired_cap;
  uint32_t reserved;            /* 0                                                                                     */
} bf_fire_out;

int bf_resident_timers(bf_ctx* ctx, uint32_t handle, uint32_t slots_per_run);
int bf_resident_timers_arm(bf_ctx* ctx, uint32_t handle, const bf_timer* requests, uint32_t n);
/* bf_resident_fire needs a timer area or a run-control area (bf_resident_runctl, which adds the run-level entries).          */
int bf_resident_fire(bf_ctx* ctx, uint32_t handle, uint32_t now, bf_fire_out* out);
int bf_resident_timers_download(bf_ctx* ctx, uint32_t handle, uint32_t first_run, uint32_t n_runs, void* slots);

/* ------------------------------------------------------------------ resident limiters (the schedule of resident batches)
 * bf_schedule uploads one bf_sched_run per run and downloads one schedule record per run on every call, and limits one batch
 * against bases the host supplies.  A resident batch may instead keep its limiter inputs on the device, and one call limits
 * several resident batches of the ctx (width classes) against ONE set of totals and lists only the runs whose schedule changed.
 * The inputs are kept in a side area of one bf_sched_run-sized record per run, like the timer slots: bf_layout and the state
 * records do not change, and a batch that never calls bf_resident_sched launches nothing more than before for any call.
 *
 * bf_resident_sched(handle): creates the area, every run at the defaults: both keys BF_SCHED_NONE, priority 0, queued_since
 *   BF_SCHED_NONE, run_phase 0 (counted in no story or queue total; only the global limit applies).  Again on a batch that has
 *   one: BF_OK, nothing changes.  bf_resident_destroy frees it.
 * bf_resident_sched_put(handle, req, n) (host buffer, synchronous): writes the inputs of each req[i].run.  Checked before
 *   anything changes, else BF_EINVAL and nothing changed: the area exists; run < capacity; reserved fields 0; at most one
 *   request per run.  A put touches no run and changes no state record, so it neither needs nor ends a tick.
 * bf_resident_sched_download(handle, first_run, n_runs, out): the stored inputs (out[i].run = first_run + i), for tests and resyncs.
 *
 * Time: queued_since is the origin of the run's queueing on the same u32 clock as `now` (the step timers' clock, suggested: seconds
 *   since the batcher's epoch).  The device derives queued_elapsed_s of bf_sched_run as: BF_SCHED_NONE when queued_since is
 *   BF_SCHED_NONE, else now - queued_since when now > queued_since, else 0 (Go's `elapsed <= 0` keeps the base priority).  The
 *   difference is taken in whole clock units: a host that wants Go's truncation of sub-second differences picks a clock of that
 *   resolution.  The clamp at INT32_MAX and the wrapping int32 sum of the limiter block apply as for bf_schedule.  So aging
 *   advances with `now` alone, and a host puts a run only when its keys, priority, StoryRun phase or queue origin change.
 *
 * bf_resident_schedule(tables, now, parts, n_parts, totals): one schedule over the resident batches parts[i].handle.
 *   Totals: the table bases, plus the Running StepRuns and the queue priority maxima of every run [0, n_runs) of every part, under
 *   the count rules of the limiter block.  Each run is then limited against these shared totals: its record is bit for bit what
 *   bf_schedule gives that run for a batch whose bf_sched_run records are the stored inputs (elapsed derived as above) and whose
 *   bases are the tables' plus the other parts' contributions (Running counts added, queue priority maxima by maximum).
 *   totals->story_running, queue_running, queue_max_priority, global_running (host arrays, each may be NULL) receive the totals;
 *   totals->records is not used.
 *   Listing: each batch keeps the records of its last schedule on the device.  A run is listed when its new record differs from
 *   the one the batch's previous schedule gave that index, or when there is no such record: the batch's first schedule, runs at or
 *   above the previous schedule's n_runs, runs uploaded, migrated, moved by retire or transfer, or received by transfer since, and
 *   every run after a reshape or narrow changed `words`.  full = 1 when every run of [0, n_runs) was listed.  A listed run's head
 *   is its record's bf_sched_header, and its events are the steps of its launch, queued_story and queued_sched masks, one
 *   (step | kind << 10) per step, kind BF_SEVT_*, run-major and step-ascending.  runs / heads / events receive the first
 *   runs_cap / runs_cap / events_cap entries; n_listed and n_events are the true counts.  Pinned buffers are written by the
 *   kernels in place; any other gets the entries copied after the synchronisation.
 *   Checked before anything is written, else BF_EINVAL and nothing changed (inputs, state records, schedule records): the struct
 *   sizes and tables (as bf_schedule); now != BF_SCHED_NONE; each handle live, listed once, with an inputs area; n_runs <=
 *   capacity; null runs / heads / events with a non-zero cap; and a tick of any kind over at least n_runs ran on the batch since
 *   the last call that changed its state records (apply, upload, migrate, redrive, retire, transfer, reshape, narrow, a tick's
 *   deltas, a fire that wrote a code); bf_last_error names the batch.  The call changes no state record and leaves bf_schedule's
 *   snapshot as it was.  The slot table is read as it stands at the call.  Launches: one for the totals' start, then four per
 *   part (count, limit and compare, scan of the per-CTA counts, list), one synchronisation.
 *
 * What the other calls do to the area (each launches nothing more when the batch has none): upload, migrate, redrive: nothing
 *   (the inputs are per run, not per step).  retire: moved runs carry their inputs; retired and vacated indices return to the
 *   defaults; a new capacity re-allocates the area.  transfer: the inputs arrive with their runs (the defaults from a source
 *   without an area); a destination without an area refuses a source that has one (BF_EINVAL, both batches byte-identical).
 *   reshape: a larger capacity extends the area with defaults.  narrow: keeps the area.                                     */
typedef struct bf_sched_put {   /* 32 B                                                                                    */
  uint32_t run;
  uint32_t story_key, queue_key;  /* as bf_sched_run; BF_SCHED_NONE (or any key past the tables) = none                    */
  int32_t priority;
  uint32_t queued_since;          /* clock of `now`; BF_SCHED_NONE = no queued step with a StartedAt                          */
  uint32_t run_phase;             /* BF_PHASE_* of StoryRun.Status.Phase                                                      */
  uint32_t reserved[2];           /* 0                                                                                        */
} bf_sched_put;

#define BF_SEVT_LAUNCH 0x1u         /* in launch: hand to StepExecutor.Execute                                               */
#define BF_SEVT_QUEUED_STORY 0x2u   /* in queued_story                                                                       */
#define BF_SEVT_QUEUED_SCHED 0x4u   /* in queued_sched                                                                       */

typedef struct bf_resident_sched_part {
  uint32_t struct_size;         /* sizeof(bf_resident_sched_part)                                                          */
  uint32_t handle;
  uint32_t n_runs;              /* runs [0, n_runs) of the batch are counted and limited                                   */
  uint32_t runs_cap;
  uint32_t* runs;               /* [runs_cap] out: ascending indices of the listed runs                                    */
  bf_sched_header* heads;       /* [runs_cap] out: the schedule header of runs[i]                                          */
  uint16_t* events;             /* [events_cap] out: step | kind << 10, run-major, step-ascending                          */
  uint64_t events_cap;
  uint32_t n_listed;            /* out: listed runs (the true count, also past runs_cap)                                   */
  uint32_t full;                /* out: 1 when every run of [0, n_runs) was listed                                          */
  uint64_t n_events;            /* out: events of the listed runs (the true count, also past events_cap)                   */
} bf_resident_sched_part;

int bf_resident_sched(bf_ctx* ctx, uint32_t handle);
int bf_resident_sched_put(bf_ctx* ctx, uint32_t handle, const bf_sched_put* requests, uint32_t n);
int bf_resident_sched_download(bf_ctx* ctx, uint32_t handle, uint32_t first_run, uint32_t n_runs, bf_sched_put* out);
int bf_resident_schedule(bf_ctx* ctx, const bf_sched_tables* tables, uint32_t now, bf_resident_sched_part* parts, uint32_t n_parts,
                         bf_sched_out* totals);

/* bf_resident_schedule_ctxs(tables, now, parts, n_parts, totals): one schedule over resident batches of several ctxs (one per
 *   GPU, e.g. the shards of a group through bf_group_ctx), so that the Story, queue and global limits and priority ordering hold
 *   over all of them.  Story and queue keys and the tables are global to the call.  Every part's records, lists, full flag and
 *   commit-due marks, and the totals, equal those of one bf_resident_schedule over the same batches held in one ctx; with one
 *   ctx the call is bf_resident_schedule.  Each part is checked on its own ctx as bf_resident_schedule checks it (a batch may
 *   appear once), with n_parts >= 1, non-null ctx and part pointers and struct_size; a refusal is BF_EINVAL with nothing changed,
 *   and bf_last_error of the first part's ctx says why (also of the refused part's own ctx).  Afterwards each batch
 *   is scheduled for its commits as after bf_resident_schedule; a failure leaves every part as after a failed bf_resident_schedule.
 *   Plan: the distinct ctxs are locked in address order.  Phase 1, per ctx on its stream: the totals' start without bases, a count
 *   launch per part, one D2H copy of the four totals arrays into pinned memory, one synchronisation per ctx.  The host gives ctx k
 *   the table bases plus every other ctx's counts (uint32 sums, as the device atomics add them; queue priority maxima by maximum,
 *   INT32_MIN for none).  Phase 2, per ctx: bf_resident_schedule of its parts with those bases.  The exchange is
 *   n_stories + 2 * n_queues + 1 words per ctx through the host; no collective library is involved.                            */
typedef struct bf_ctx_sched_part {
  uint32_t struct_size;         /* sizeof(bf_ctx_sched_part)                                                               */
  uint32_t reserved;            /* 0                                                                                         */
  bf_ctx* ctx;
  bf_resident_sched_part* part; /* a part of bf_resident_schedule, of a batch of ctx                                         */
} bf_ctx_sched_part;

int bf_resident_schedule_ctxs(const bf_sched_tables* tables, uint32_t now, bf_ctx_sched_part* parts, uint32_t n_parts, bf_sched_out* totals);

/* ------------------------------------------------------------------ StoryRun stops and deadlines (run control of a resident batch)
 * Above the steps, the reference stops DAG-evaluating a StoryRun for three reasons: its story timeout (enforceStoryTimeout,
 * dag.go:544-578, checked at the start of every iteration :393-398, before the gate / sleep / wait syncs :409-420: once
 * now - Status.StartedAt >= policy.timeouts.story the run becomes Timeout), a graceful cancel (spec.cancelRequested returns from
 * Reconcile before the DAG, storyrun_controller.go:279-280; handleGracefulCancel :1517-1578 force-deletes the StepRuns once
 * !now.Before(observedAt + gracefulShutdownTimeout)) and a terminal phase (:281-287).  A resident batch keeps the stop and both
 * deadlines itself, in a side area of one 16-byte record per run, so that its runs stop producing ready steps and launches on the
 * device and bf_resident_fire reports the run-level deadlines with the step timers.  bf_layout, the record bytes and the pass
 * do not change, and a batch that never calls bf_resident_runctl launches nothing more than before for any call.
 * Time is the step timers' clock (a u32 the host chooses; `now` of bf_resident_fire).  A deadline is DUE iff it is not
 * BF_TIMER_NONE and deadline <= now.
 *
 * Stop.  Stopping a run saves its run_flags byte in saved_flags and writes BF_RF_HOST_GROUP | BF_GROUP_DONE << BF_RF_HOST_GROUP_SHIFT
 *   into the record: both frontier kernels evaluate such a run as "finalize on host" (BF_GROUP_DONE) with no candidates, so it
 *   lists no ready step, no event and no launch.  The pass may still apply its stage G/H phase rewrites to the result record of a
 *   host-group run (phase_out, BF_SUM_PHASE_CHANGED); the host ignores those for a stopped run.  A stop also empties the run's
 *   step-timer slots (the reference never applies them again), touches the run as a delta does (the next touched tick evaluates
 *   it and lists it when its result changed), ends the evaluated snapshot and the schedule's tick (bf_resident_schedule must follow
 *   a new tick).  A BF_STOP_TIMEOUT stop also writes run_phase = BF_PHASE_TIMEOUT into the run's limiter inputs when the batch has
 *   that area: the run makes no demand in priority ordering (storyRunHasDemand, dag.go:1981-1999), while its Running steps still
 *   count in the totals (its StepRuns still exist).  A stopped run keeps its stop until a redrive: a put cannot clear it, and
 *   stopping it again changes nothing (the first reason and the saved byte stay).
 *
 * bf_resident_runctl(handle): creates the area, every record at the default {BF_TIMER_NONE, BF_TIMER_NONE, BF_STOP_NONE, 0}.
 *   Again on a batch that has one: BF_OK, nothing changes.  bf_resident_destroy frees it.
 * bf_resident_runctl_put(handle, req, n) (host buffer, synchronous): writes both deadlines of each req[i].run; stop != BF_STOP_NONE
 *   stops the run now.  Checked before anything changes, else BF_EINVAL and nothing changed: the area exists; run < capacity;
 *   stop <= BF_STOP_HOST; reserved fields 0; at most one request per run.  A put that only changes deadlines touches no run.
 * bf_resident_runctl_download(handle, first_run, n_runs, out): the raw records, for tests and resyncs.
 * bf_resident_fire (step timers section) also runs on a batch with this area and no timer area.  For each run below n_runs:
 *   1. not stopped and story_deadline due: the run is stopped with BF_STOP_TIMEOUT and listed as (run, BF_FIRED_STORY,
 *      BF_DEC_TIMED_OUT, written = 1); its armed step slots are disarmed and counted in n_pruned, none listed or written (the
 *      story timeout precedes the step syncs, dag.go:393-409);
 *   2. otherwise its step slots fire as described there;
 *   3. drain_deadline due: disarmed and listed as (run, BF_FIRED_DRAIN, BF_DEC_PENDING, written = 0), wake-only (the host's
 *      force-delete).
 *   The list stays ascending by run, then step; n_written counts the timeouts.  next_deadline is the minimum over the armed step
 *   slots, the drain deadlines and the story deadlines of runs not stopped (a stopped run's story deadline is kept, dormant).
 *
 * What the other calls do to the area (each launches nothing more when the batch has none):
 *   delta scatter: a BF_DELTA_RUN_FLAGS delta of a stopped run is written into saved_flags; the record keeps the stop.
 *   upload: deadlines and stops persist; a stopped run's uploaded flags byte becomes saved_flags and the record is stopped again
 *     (one more launch over the uploaded range), so a resync from a host mirror that knows nothing of stops keeps them.
 *   redrive (both kinds, runs with status_out = 1): a stopped run's record gets saved_flags without BF_RF_TOPOLOGY_TERMINATED and
 *     the stop is cleared; the drain deadline is disarmed; BF_REDRIVE_ALL also disarms the story deadline (resetStoryRunForRedrive
 *     sets StartedAt = nil, storyrun_controller.go:414-438), a step redrive keeps it (resetStoryRunForStepRedrive keeps StartedAt:
 *     a timed-out run redriven from a step times out again at the next fire, as in the reference).
 *   retire: records move with their runs, retired and vacated indices get the default; a new capacity re-allocates the area.
 *   transfer: records arrive with their runs (the default from a source without an area); a destination without an area refuses a
 *     moved run whose record is not the default (BF_EINVAL, both batches byte-identical).
 *   reshape: a larger capacity extends the area with defaults.  narrow: keeps the area; extent and the fit do not change (a stop
 *     needs no width and no planes).  migrate: nothing.                                                                     */
enum { BF_STOP_NONE = 0, BF_STOP_TIMEOUT = 1, BF_STOP_CANCEL = 2, BF_STOP_HOST = 3 };
typedef struct bf_run_ctl {     /* 16 B; the default is {BF_TIMER_NONE, BF_TIMER_NONE, 0, 0, {0}}                           */
  uint32_t story_deadline;      /* StartedAt + policy.timeouts.story on the timers' clock, BF_TIMER_NONE: none               */
  uint32_t drain_deadline;      /* graceful-cancel force-delete time, wake-only, BF_TIMER_NONE: none                         */
  uint8_t stop;                 /* BF_STOP_*                                                                                 */
  uint8_t saved_flags;          /* the run's own run_flags byte while stopped, else 0                                        */
  uint8_t reserved[6];
} bf_run_ctl;
typedef struct bf_run_ctl_put { /* 16 B                                                                                      */
  uint32_t run;
  uint32_t story_deadline, drain_deadline;   /* BF_TIMER_NONE: none                                                          */
  uint8_t stop;                 /* BF_STOP_NONE: deadlines only; else stop the run now                                       */
  uint8_t reserved[3];          /* 0                                                                                         */
} bf_run_ctl_put;
#define BF_FIRED_DRAIN 0xFFFEu  /* bf_fired.step of a drain deadline                                                         */
#define BF_FIRED_STORY 0xFFFFu  /* bf_fired.step of a story timeout                                                          */

int bf_resident_runctl(bf_ctx* ctx, uint32_t handle);
int bf_resident_runctl_put(bf_ctx* ctx, uint32_t handle, const bf_run_ctl_put* requests, uint32_t n);
int bf_resident_runctl_download(bf_ctx* ctx, uint32_t handle, uint32_t first_run, uint32_t n_runs, bf_run_ctl* out);

/* ------------------------------------------------------------------ tick commits (the decisions of a tick written back)
 * After a tick the reference writes, in the same reconcile, what the decisions of that iteration did to StepStates: skipped steps
 * become Skipped (dag.go:1734-1746), queued steps Pending with a "Queued due to ..." message (markQueuedSteps, :1999-2018; code 14
 * here), and each launched step what StepExecutor.Execute writes for its type (step_executor.go:132-185).  bf_resident_commit makes
 * these writes in the stored state records of runs [0, n_runs), so that a batcher sends no echo deltas for its own decisions: a step
 * downstream of a skip becomes ready at the next tick, and a launched step is no longer listed as ready.
 *
 * The writes, from the current result record of each run (the one the last tick left) and, when the batch has a limiter area
 * (bf_resident_sched), its last schedule record:
 *   skip mask                                      -> BF_PHASE_SKIPPED
 *   fail mask (cond FAIL, dag.go:2744-2748)        -> BF_PHASE_FAILED
 *   launched condition step                        -> BF_PHASE_SUCCEEDED                          (step_executor.go:168-170)
 *   launched sleep / gate / wait step              -> BF_PHASE_PAUSED                             (:171-179)
 *   launched parallel step                         -> BF_PHASE_RUNNING and its children_registered bit set (:808-809)
 *   launched stop step                             -> the code of its BF_COMMIT_PHASE entry        (:1096-1106)
 *   launched engram / executeStory step            -> BF_PHASE_RUNNING when its code is 0 or 14, else unchanged (dag.go:1770-1774)
 *   queued step (queued_story | queued_sched)      -> BF_PHASE_PENDING_QUEUED                      (dag.go:1999-2018)
 * The launched steps are the schedule record's launch mask when the batch has a limiter area, else the ready mask (nothing is then
 * queued).  The masks are taken disjoint in this order: fail without skip, launched and queued without either.  A run whose topology
 * slot is dead, or does not fit the layout, has no masks.  A phase code 15 reads as 0, as the pass reads it; a step the commit does
 * not write keeps its bytes.
 *
 * Entries report what the host's Execute did, at most one per (run, step), each naming a launched step:
 *   BF_COMMIT_HOLD   Execute was blocked on template evaluation (dag.go:1750-1761): that step gets no launch write.
 *   BF_COMMIT_ERROR  Execute failed: the reference returns the error and persists nothing of that reconcile (dag.go:1763-1768,
 *                    :342-345), so the whole run gets no write.
 *   BF_COMMIT_PHASE  the with.phase of a launched stop step (code: BF_PHASE_PENDING .. BF_PHASE_SKIPPED).  Every launched stop step
 *                    of a run without a BF_COMMIT_ERROR entry needs one, or a BF_COMMIT_HOLD entry.
 * Checked before anything changes, else BF_EINVAL, nothing changed, and bad_run / bad_step name the first offender (BF_COMMIT_NONE
 * for a refusal of the whole call).  In this order: struct_size and the handle; n_runs <= capacity; entries not NULL when n > 0;
 * the layout has cond planes but no BF_F_OUT_FAIL (the device cannot know the cond-FAIL steps); the batch's state records changed
 * since its last tick over n_runs (the rule of bf_resident_schedule); a topology slot of the ctx was dropped, or a dropped one
 * reused, since the batch's last tick (the masks were evaluated against the step types the slot had then); a tick with BF_EVAL_FIXPOINT ran since the last single-pass
 * tick over n_runs (the fixpoint applies these effects in memory, under unlimited limiters); the batch has a limiter area and no
 * bf_resident_schedule over at least n_runs of it ran since its last tick.  Then each entry in array order: run < n_runs,
 * step < steps_max, kind and code (0 for HOLD and ERROR); then the lowest (run, step) named twice; then, on the device, the lowest
 * (run, step) that is an entry naming a step not launched, a BF_COMMIT_PHASE entry of a step that is not a stop step, or a
 * launched stop step without an entry.
 *
 * Idempotent: a run whose writes are in place is not changed.  A run whose record changed is touched as by a delta (the next
 * bf_resident_tick_touched evaluates it), and a commit that changed anything ends the evaluated snapshot and the tick a schedule
 * or a commit needs.  bf_resident_commit arms no step timer (bf_resident_commit_timed below arms those of the launched sleeps,
 * gates and waits), and a stopped run (bf_resident_runctl) has no candidates, so it gets nothing.  The counts are steps whose code the commit changed (a
 * launched parallel step also when only its registered bit was set).  Stage G / H / I rewrites (gate syncs, joins, fail-fast and
 * compensation skips) are not persisted by this call, _timed or _journal: each pass recomputes them from the state
 * (bf_resident_commit_rewrites below stores them).  One H2D copy of the sorted entries, the check
 * launch, one D2H copy and one synchronisation before anything is written; then the apply launch, one D2H copy and one
 * synchronisation.                                                                                                          */
enum { BF_COMMIT_HOLD = 1, BF_COMMIT_ERROR = 2, BF_COMMIT_PHASE = 3 };
#define BF_COMMIT_NONE 0xFFFFFFFFu
typedef struct bf_commit_entry { /* 8 B, one per (run, step) the host's Execute did not launch normally                        */
  uint32_t run;
  uint16_t step;
  uint8_t kind;                  /* BF_COMMIT_*                                                                               */
  uint8_t code;                  /* BF_COMMIT_PHASE: the phase code executeStopStep writes; else 0                            */
} bf_commit_entry;
typedef struct bf_commit_out {
  uint32_t struct_size;          /* sizeof(bf_commit_out)                                                                     */
  uint32_t n_runs_written;       /* out: runs whose state record changed (touched)                                            */
  uint32_t n_skipped;            /* out: steps written as BF_PHASE_SKIPPED                                                    */
  uint32_t n_launched;           /* out: launched steps written                                                               */
  uint32_t n_queued;             /* out: steps written as BF_PHASE_PENDING_QUEUED                                             */
  uint32_t n_failed;             /* out: steps written as BF_PHASE_FAILED by a cond FAIL                                      */
  uint32_t bad_run;              /* out on a refusal: the offending run, or BF_COMMIT_NONE                                    */
  uint32_t bad_step;             /* out on a refusal: the offending step, or BF_COMMIT_NONE                                   */
} bf_commit_out;

int bf_resident_commit(bf_ctx* ctx, uint32_t handle, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n_entries,
                       bf_commit_out* out);

/* bf_resident_commit_timed(..., out, arm) is bf_resident_commit (arm = NULL is exactly that call) that also arms the step timers of
 * the steps it launches, as the reference arms them when it launches a step (ensureSleepUntil / ensureWaitTimeoutAt /
 * ensureGateTimeoutAt, dag.go:128-171).  For each run the commit writes (no BF_COMMIT_ERROR entry), each launched step after the
 * commit's masks (launched, not skipped, not cond-FAIL, no BF_COMMIT_HOLD entry) that is a sleep, gate or wait step and has a
 * timing in the run's slot (bf_topology_timings):
 *   - no armed slot of the run names the step: {deadline = min(now + delay, BF_TIMER_NONE - 1), step, code} is armed into the
 *     run's slots in the canonical order (a delay of 0 is due at `now`: the next bf_resident_fire fires it);
 *   - an armed slot names it: that slot stays as it is and is not counted (the stored deadline wins, dag.go:128-171).
 * Checked before anything changes, in addition to bf_resident_commit's checks, with bad_run / bad_step as there: arm->struct_size,
 * arm->now != BF_TIMER_NONE and the batch's timer area (bf_resident_timers), BF_EINVAL for the whole call; then, on the device
 * and together with the entry offences (the lowest (run, step) of all of them), a run that would arm a non-PENDING code on a
 * batch without decision planes (BF_EINVAL, at that step), and a run whose armed slots plus its new arms exceed K (BF_ENOMEM,
 * at the lowest step it would newly arm; grow K with bf_resident_timers and repeat the commit).  Arming touches no run (every
 * armed step is a written step); stopped runs, dead slots and slots wider than the layout have no masks and arm nothing.  The
 * arms are made by the same two launches; the copies of the counts carry two more words.                                      */
typedef struct bf_commit_arm {
  uint32_t struct_size;          /* sizeof(bf_commit_arm)                                                                     */
  uint32_t now;                  /* in: the clock of bf_resident_fire; != BF_TIMER_NONE                                       */
  uint32_t n_armed;              /* out: slots this call armed                                                                */
  uint32_t next_deadline;        /* out: earliest deadline this call armed, or BF_TIMER_NONE                                  */
} bf_commit_arm;
int bf_resident_commit_timed(bf_ctx* ctx, uint32_t handle, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n_entries,
                             bf_commit_out* out, bf_commit_arm* arm);

/* bf_resident_commit_journal(..., out, arm, journal) is bf_resident_commit_timed (arm = NULL: bf_resident_commit) that also lists
 * what it wrote, so that a batcher persists the same writes to StepStates (and a host mirror applies them) without a second copy of
 * the commit's rules.  Checks, refusals, writes, touches, arms and counts are exactly those of the call it extends.  Items
 * (bf_commit_write), one per changed byte or slot:
 *   BF_DELTA_PHASE         a step whose stored code changed: before = the stored nibble (15 as stored), after = the code written
 *   BF_DELTA_REGISTERED    a parallel desc whose children_registered bit the commit set: before = 0, after = 1
 *   BF_COMMIT_WRITE_TIMER  a timer slot `arm` newly armed: code = the armed code, before = BF_TIMER_NONE, after = the deadline (a
 *                          kept stored slot is not listed, so these items number arm->n_armed)
 * ordered by (run, field in that order, index); nothing else is listed: a second commit of the same tick, BF_COMMIT_ERROR runs,
 * HOLD steps, stopped runs and dead or too-wide slots list nothing.  runs: the ascending runs whose state record changed (the
 * touched runs; n_runs_listed == out->n_runs_written).  n_items and n_runs_listed are the true counts; only the first items_cap /
 * runs_cap are written.  A refusal writes nothing and leaves both counts 0.  A NULL journal or a wrong struct_size, and items /
 * runs NULL with a non-zero cap, are BF_EINVAL before anything else is checked or written.
 * Cost: the check launch also counts each run's items, one scan launch (as bf_resident_status) turns the counts into offsets, and
 * the apply launch writes the items there: one launch more than bf_resident_commit_timed and no further synchronisation.  Pinned
 * buffers (items 16-byte aligned) are written in place; others are staged in the ctx's device scratch, sized after the check
 * launch to what will be copied (16 B per item of min(n_items, items_cap), 4 B per run of min(n_runs_listed, runs_cap)), and
 * copied before the final synchronisation.  A scratch that has to grow for them waits for the device once.                  */
#define BF_COMMIT_WRITE_TIMER 0x10u   /* field of a timer-arm item; PHASE and REGISTERED items use BF_DELTA_PHASE / _REGISTERED       */
typedef struct bf_commit_write { /* 16 B                                                                                        */
  uint32_t run;
  uint16_t index;                /* step (PHASE, TIMER) or parallel desc (REGISTERED)                                           */
  uint8_t field;                 /* BF_DELTA_PHASE, BF_DELTA_REGISTERED, BF_COMMIT_WRITE_TIMER                                  */
  uint8_t code;                  /* TIMER: the armed code; PHASE: 0 or BF_COMMIT_WRITE_REWRITE (_rewrites); else 0              */
  uint32_t before, after;        /* PHASE: stored nibble / code written; REGISTERED: 0 / 1; TIMER: BF_TIMER_NONE / deadline     */
} bf_commit_write;
typedef struct bf_commit_journal {
  uint32_t struct_size;          /* sizeof(bf_commit_journal)                                                                   */
  uint32_t reserved;
  bf_commit_write* items;        /* [items_cap] out                                                                             */
  uint64_t items_cap;
  uint64_t n_items;              /* out: the true count; only the first items_cap are written                                   */
  uint32_t* runs;                /* [runs_cap] out: ascending runs whose record changed                                         */
  uint32_t runs_cap;
  uint32_t n_runs_listed;        /* out: the true count, == bf_commit_out.n_runs_written                                        */
} bf_commit_journal;
int bf_resident_commit_journal(bf_ctx* ctx, uint32_t handle, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n_entries,
                               bf_commit_out* out, bf_commit_arm* arm, bf_commit_journal* journal);

/* bf_resident_commit_rewrites(..., out, arm, journal, n_rewritten) is bf_resident_commit_journal (arm = NULL allowed) that also
 * stores the phases a single pass's stages G, H and I rewrite, as the reference persists the StepStates its checkSync* and
 * markFailFastSkipped / markCompensationsSkipped wrote (persistMergedStates, dag.go:774-793): a fired sleep, an approved, rejected
 * or timed-out gate or wait (stage G), a joined parallel step (stage H), fail-fast and compensation skips and the Failed codes of a
 * terminated realtime topology (stage I).  The journal is required (a rewrite the batcher never hears of is not persisted in the
 * cluster); NULL, or a wrong struct_size, is BF_EINVAL as for bf_resident_commit_journal, and so is a NULL n_rewritten.
 *
 * The writes of a run start from its codes after the stages bf_resident_status applies (no stage-D cond-FAIL write: the fail mask
 * still writes those) instead of its stored codes, and are stored where they differ from the stored codes (15 read as 0, as
 * always).  A run with a BF_COMMIT_ERROR entry, a stopped run, and a run on a dead or too-wide slot get no rewrite (nor, as before,
 * any other write); a HOLD step takes no launch write, and the rest of its run takes its rewrites.  Checks, refusals, entries,
 * arms and touches are those of bf_resident_commit_journal.  A run whose only writes are rewrites is a written run: touched,
 * listed in journal->runs and counted in out->n_runs_written, and a commit that wrote ends the tick as any other.
 *
 * Items as bf_resident_commit_journal, in the same order; a PHASE item of a step that has no mask bit (not skipped, cond-FAIL,
 * launched or queued: its new code comes from the stages) carries code = BF_COMMIT_WRITE_REWRITE, every other item code 0 (or
 * the armed code of a TIMER item).  The counts of out keep counting the mask writes; *n_rewritten is the number of steps written
 * from the stages (the items marked BF_COMMIT_WRITE_REWRITE).  A commit that wrote ends the tick, so a second call needs a new
 * tick; that tick evaluates the written records, and a run whose stages rewrite again over them (a fail-fast skip after stored
 * Failed codes, say) is flagged by its new result record and takes those rewrites at the next call.
 *
 * Precondition that makes it cheap and exact: only a run whose current result record carries BF_SUM_PHASE_CHANGED can have a
 * rewrite, because the tick that left that record took the same stages over the same stored codes and flags any phase they
 * change (a commit or any other write in between is refused, or ends the tick, as for every commit).  So one more launch, one warp
 * per run, evaluates the stages of those runs alone and stages their planes in the ctx's device scratch (16 B per run and word,
 * plus 4 B per run); the check and apply launches read them there.  One launch more than bf_resident_commit_journal and no further
 * synchronisation.                                                                                                            */
#define BF_COMMIT_WRITE_REWRITE 0x1u  /* bf_commit_write.code of a PHASE item whose code comes from the stages G / H / I          */
int bf_resident_commit_rewrites(bf_ctx* ctx, uint32_t handle, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n_entries,
                                bf_commit_out* out, bf_commit_arm* arm, bf_commit_journal* journal, uint32_t* n_rewritten);

/* Touched commits.  Every commit form walks all of [0, n_runs), although after the first commit almost every run's writes are
 * already in place.  bf_resident_commit_touched considers only the runs whose writes may not be in place, and its results are
 * those of the matching full form.
 *
 * bf_resident_commit_marks(ctx, handle) enables the batch's commit-due area: one bit per run, every bit set.  Reshape and a
 * retire to a new capacity keep the bits of the runs both capacities hold; a batch that never enables the area launches, copies
 * and writes what it did before.  Calling it again sets every bit again.
 *
 * The form: arm, journal and BF_COMMIT_SCOPE_REWRITES in scope->flags pick the full form the call matches, with that form's
 * argument rules:
 *   arm NULL, journal NULL                      bf_resident_commit
 *   arm set,  journal NULL                      bf_resident_commit_timed
 *   journal set, no BF_COMMIT_SCOPE_REWRITES    bf_resident_commit_journal
 *   journal set, BF_COMMIT_SCOPE_REWRITES       bf_resident_commit_rewrites (n_rewritten required)
 * n_rewritten is ignored without BF_COMMIT_SCOPE_REWRITES, and BF_COMMIT_SCOPE_REWRITES without a journal is BF_EINVAL.  A batch
 * without the area is BF_EINVAL (bad_run = bad_step = BF_COMMIT_NONE).
 *
 * Equivalence guarantee: for any sequence of resident calls, the return code, bad_run and bad_step, every bf_commit_out and
 * bf_commit_arm field, n_rewritten, the journal's items and runs and their true counts, the state records, timer slots and touch
 * marks, and the batch's bookkeeping (the tick a schedule or commit needs, the touched-list bound, what the next touched tick
 * lists) are exactly those the matching full form would have given at the same point.
 *
 * Why it holds: a commit is idempotent (over records whose writes are in place it writes nothing and refuses nothing), and what
 * it writes or checks for a run is a function of that run's state record, current result record, schedule record, timer slots
 * and run-control record, the slot's step types and timings, the run's entries and the form.  A run is due unless the last
 * touched commit that considered it found no entry on it and none of those inputs changed since:
 *   - a touched tick (single or _many) sets the bit of every run it evaluates, bf_resident_schedule that of every run whose
 *     schedule record changed;
 *   - the call considers every run of [0, n_runs) ("full") after a full tick (bf_resident_tick, _tick_compact, _eval, a touched
 *     tick that ran full), after enabling the area, after a tick, schedule or commit that failed (CUDA or allocation), when its
 *     form differs from the last touched commit's, and, for a form that arms, after a bf_topology_timings or a drop changed the
 *     ctx's timings since the last touched commit;
 *   - a run that an entry names is considered, and stays due after the commit.
 * Every other call that changes a run's records (deltas, uploads, moves, migrations, redrives, resyncs, fires that write, stops,
 * commits that write) touches the run, and a commit must follow a tick over n_runs (the rule of every form), which evaluates
 * and so marks every touched run.  A commit of another form, a refused commit and a commit that fails clear no bit.
 *
 * Device work: without full, one count, scan and list launch triple builds the ascending list of the due runs below n_runs and
 * the runs the entries name; the check (with a journal, and its scan over the list's blocks of 8 positions), the rewrites and the
 * apply launches are list-mode builds of the full form's, one warp per listed run; the apply also clears the due bits.  With
 * full, no list is built: every bit is set once the check passed (a memset, no launch) and the list-mode builds take
 * [0, n_runs).  Launches: the full form's, plus 3 without full (so 5, 5, 6 and 7 for the four forms; 2, 2, 3 and 4 with full),
 * none when n_runs == 0.  The
 * commit's two synchronisations stay.  A touched tick on a batch with the area adds one launch (one per part for _many), and
 * bf_resident_schedule one per batch with the area.
 *
 * scope (required): struct_size = sizeof(bf_commit_scope), flags; out: full (1: every run of [0, n_runs) was considered) and
 * n_considered (the runs considered; n_runs with full).  Both are 0 for n_runs == 0 and on a refusal before the device. */
#define BF_COMMIT_SCOPE_REWRITES 0x1u
typedef struct bf_commit_scope {
  uint32_t struct_size;          /* sizeof(bf_commit_scope)                                                                     */
  uint32_t flags;                /* BF_COMMIT_SCOPE_REWRITES or 0                                                               */
  uint32_t full;                 /* out                                                                                         */
  uint32_t n_considered;         /* out                                                                                         */
} bf_commit_scope;
int bf_resident_commit_marks(bf_ctx* ctx, uint32_t handle);
int bf_resident_commit_touched(bf_ctx* ctx, uint32_t handle, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n_entries,
                               bf_commit_out* out, bf_commit_arm* arm, bf_commit_journal* journal, uint32_t* n_rewritten,
                               bf_commit_scope* scope);

/* ------------------------------------------------------------------ run status (what a batcher persists of a run's status)
 * When group selection finds nothing left to run (BF_GROUP_DONE, dag.go:482-495) the reference finalizes the StoryRun
 * (finalizeStoryRun, dag.go:693-754): the failed set of the finally, compensation or main group, in that order, decides its phase
 * and condition reason, the message names the set's first failed step, and status.error lists every step of the set with its
 * phase (BuildStoryRunError, pkg/runs/status/storyrun.go:165).  On every persist it also writes status.allowedFailures
 * (syncAllowedFailures, dag.go:478, :3393-3430) and the step counters (updateStepProgress / summarizeStepProgress, :904-942).  All
 * of these read the phases after the pass's rewrites, which only the device holds.  bf_resident_status reports them for the
 * listed runs of a resident batch.
 *
 * The phases are those of the run's state record after stages G (gate / sleep / wait decisions), H (parallel join) and I
 * (fail-fast and compensation-skip marking, topology-terminated fails): the stages, with the parameters, a single-pass tick
 * applies to the record now.  Stage D's cond-FAIL writes are not among them (they reach the record through a commit).
 *
 * runs[n]: strictly ascending, each below n_runs; runs == NULL with n == n_runs lists every run of [0, n_runs).  One record per
 * listed run, in list order:
 *   group      the BF_GROUP_* of that pass (the host's group for host-group runs, BF_GROUP_DONE for a stopped run)
 *   summary    its BF_SUM_* group, done and failed bits (no BF_SUM_PHASE_CHANGED, no iteration count; 0 besides the group for a
 *              host-group run)
 *   outcome    BF_OUTCOME_NONE when the group is not BF_GROUP_DONE; else from the failed sets (failed: terminal and not completed
 *              under allowFailure, as buildStateMaps): finally's -> CLEANUP_FAILED, else compensation's -> COMPENSATION_FAILED, else
 *              main's -> COMPENSATED when the topology has compensation steps, else DEPENDENCY_FAILED; none -> SUCCEEDED.  A run
 *              stopped in the batch's run control (bf_resident_runctl) takes TIMED_OUT, CANCELED or STOPPED from its stop reason
 *              and lists no failed set.  A dead topology slot, or one wider than the layout (of more words than L.words): DEAD,
 *              group and summary 0, counts 0, no events.  A topology of more than L.steps_max steps but no more words is live and
 *              lists events up to 32 * L.words, as many as its steps.
 *   story_phase  the BF_PHASE_* the reference writes for the outcome: SUCCEEDED -> Succeeded (provisional: the host still
 *              evaluates the Story's output template, finalizeSuccessfulRun, dag.go:2871, which can block or fail), the three
 *              failures -> Failed, COMPENSATED -> Compensated, TIMED_OUT -> Timeout (dag.go:566-571), CANCELED -> Finished
 *              (storyrun_controller.go:1557; the host sets it once its drain ends), otherwise 0
 *   first_failed  the lowest step of the listed failed set, or BF_STATUS_NO_STEP
 *   active / completed / failed / skipped   steps whose code is Running or Paused / Succeeded / Failed / Skipped (code 14 and
 *              code 0 count in none, as summarizeStepProgress)
 *   n_events, first_event   the run's events are events[first_event .. first_event + n_events) of the call's list
 * events: one u16 per listed step, step | phase << 10 | kind << 14, run-major and step-ascending:
 *   BF_STATUS_EVT_FAILED    a step of the listed failed set (the failedSteps of status.error)
 *   BF_STATUS_EVT_ALLOWED   a terminal step with allowFailure that is neither Succeeded nor Skipped (collectAllowedFailures),
 *                           in every run that is not dead, finished or not
 * n_events is the true count; only the first events_cap events are written (as bf_compact_out); a run has at most
 * 32 * L.words events.
 * Read-only: no record, result, side area, touch mark or tick state changes, so the call may sit anywhere in the per-tick loop.
 * Refused before any launch with BF_EINVAL and nothing written: struct_size, the handle, n_runs > capacity, runs not strictly
 * ascending or not below n_runs, runs == NULL with n != n_runs, records == NULL with n > 0, events == NULL with events_cap > 0.
 * Pinned buffers (runs, records, events) are used in place; others go through the call's staging.  One synchronisation, and with
 * events not in pinned memory a second one: their copy follows the synchronisation that brings back their number.            */
enum {
  BF_OUTCOME_NONE = 0, BF_OUTCOME_SUCCEEDED = 1, BF_OUTCOME_DEPENDENCY_FAILED = 2, BF_OUTCOME_COMPENSATED = 3,
  BF_OUTCOME_COMPENSATION_FAILED = 4, BF_OUTCOME_CLEANUP_FAILED = 5, BF_OUTCOME_TIMED_OUT = 6, BF_OUTCOME_CANCELED = 7,
  BF_OUTCOME_STOPPED = 8, BF_OUTCOME_DEAD = 9
};
#define BF_STATUS_EVT_FAILED 0x1u
#define BF_STATUS_EVT_ALLOWED 0x2u
#define BF_STATUS_EVENT_STEP(e) ((uint32_t)(e) & 0x3FFu)
#define BF_STATUS_EVENT_PHASE(e) (((uint32_t)(e) >> 10) & 0xFu)
#define BF_STATUS_EVENT_KIND(e) ((uint32_t)(e) >> 14)
#define BF_STATUS_NO_STEP 0xFFFFu
typedef struct bf_status_rec {   /* 32 B                                                                                         */
  uint32_t run;
  uint32_t first_event;
  uint16_t n_events;
  uint16_t first_failed;         /* BF_STATUS_NO_STEP: none                                                                    */
  uint16_t summary;
  uint8_t group;
  uint8_t outcome;               /* BF_OUTCOME_*                                                                               */
  uint8_t story_phase;           /* BF_PHASE_*                                                                                 */
  uint8_t reserved[7];
  uint16_t active, completed, failed, skipped;
} bf_status_rec;
typedef struct bf_status_out {
  uint32_t struct_size;          /* sizeof(bf_status_out)                                                                      */
  uint32_t reserved;
  bf_status_rec* records;        /* [n] out                                                                                    */
  uint16_t* events;              /* [events_cap] out                                                                           */
  uint64_t events_cap;
  uint64_t n_events;             /* out: events of the listed runs; when > events_cap only the first events_cap were written  */
} bf_status_out;

int bf_resident_status(bf_ctx* ctx, uint32_t handle, uint32_t n_runs, const uint32_t* runs, uint32_t n, bf_status_out* out);

/* ------------------------------------------------------------------ resyncs (does the device still agree with the cluster?)
 * The reference rebuilds its state from the StepRuns and the fresh status on every reconcile (syncStateFromStepRuns, dag.go:965-1009)
 * and merges its writes back into the cluster object (persistMergedStates, :774-793), so drift never outlives one reconcile.  A
 * resident batch keeps state across ticks, so a lost watch event or a failed status PATCH persists until something overwrites it.
 * bf_resident_resync compares the device's state records of the listed runs with records the caller packed from the cluster (same
 * format and layout as bf_resident_upload), lists every difference and, without BF_RESYNC_CHECK, repairs only the runs that drifted.
 *
 * What is compared (record = the caller's record as the repair would leave it on the device: the device's record with the caller's
 * codes in the selected fields; for a stopped run the flags byte the stages read is the stopped byte on both sides):
 *   - slot: topo_slot, always.  A run whose slot differs has exactly one item, BF_DELTA_TOPO_SLOT (index 0), and nothing else.
 *   - a live slot that fits the layout: both sides take the stages of a single pass that bf_resident_status applies (H, G, I; no
 *     stage D cond-FAIL writes; a stopped run evaluated with its stopped flags byte).  Then for each field selected in `fields`:
 *       PHASE      the resulting codes of steps < S (code 15 read as 0 before the stages);
 *       COND, DECISION   the input codes of steps whose resulting phase is not terminal on at least one side (a step terminal on
 *                  both no longer reads them);
 *       CHILD      the nibbles (15 read as 0) of the slot's parallel descs whose step is not terminal on at least one side;
 *       REGISTERED the children_registered bits of those same descs;
 *       RUN_FLAGS  the byte; for a stopped run the device's saved byte (bf_run_ctl.saved_flags), not the stopped byte.
 *   - a dead slot, or one wider than the layout: no stages.  Every code of the layout as stored (words * 32 steps, phases and
 *     nibbles with 15 read as 0), every child nibble of the layout, all 64 registered bits and the flags byte.
 *   - never compared: the reserved header bytes, codes at or past S of a live slot, nibbles and registered bits outside its descs,
 *     padding.  A field the layout does not place (cond, decision, child area) is neither compared nor written.
 * Items (bf_drift) are ordered by (run, field, index); device and record are the compared values (a PHASE item carries the phases
 * after the stages).  Why the stages come first: their rewrites are never stored (a fired sleep is Paused with decision SUCCEED on
 * the device and Succeeded in the cluster; a joined parallel step Running here and Succeeded / Failed there; a fail-fast skip 0
 * here and Skipped there), so equal states differ as bytes and agree only after them.
 *
 * Repair (without BF_RESYNC_CHECK), of the drifted runs only:
 *   - slot drift: the whole record becomes the caller's bytes; the run is touched as by a migrate (listed by the next touched tick
 *     even if its result is unchanged) and its schedule baseline is dropped (listed by the next bf_resident_schedule);
 *   - otherwise: each selected field's storage (all of its planes' words, the whole child area, all 64 registered bits, the flags
 *     byte) becomes the caller's and the rest stays the device's; the run is touched as by a delta (the next touched tick evaluates
 *     it and lists it when its result changed) and keeps its schedule baseline;
 *   - a stopped run stays stopped: the caller's flags byte becomes its saved byte and the record keeps the stopped byte;
 *   - timers, limiter inputs, result records and the changed-only baseline are not touched.  pending grows by n_written.
 * A resync that wrote something ends the evaluated snapshot and the tick (bf_resident_schedule and bf_resident_commit must follow a
 * new tick), as a commit that wrote.  One that wrote nothing, and every BF_RESYNC_CHECK call, changes nothing at all.
 * Refused before anything is written, BF_EINVAL and nothing changed: struct_size or the handle; n_runs > capacity; runs not strictly
 * ascending or not below n_runs; runs == NULL with n != n_runs; records == NULL with n > 0; drifted / items NULL with a non-zero
 * cap; unknown flags or fields bits; a record naming a slot no put has returned (bad_run names its run, else BF_RESYNC_NONE).
 * One H2D copy of the records (and one of a run list not in pinned memory), three launches (count, scan, list and repair), one D2H
 * copy of the totals, one synchronisation.  Pinned drifted / items buffers are written in place; others are staged in the ctx's
 * device scratch (16 B per item of items_cap, clamped to what the listed runs can have; the scratch keeps its largest size for
 * the ctx's lifetime, so size items_cap to the drift expected: n_items is the true count) and copied after the synchronisation. */
#define BF_RESYNC_CHECK 0x1u                 /* flags: compare and list only; nothing changes                                   */
#define BF_RESYNC_FIELD(f) (1u << (f))       /* fields: BF_DELTA_PHASE .. BF_DELTA_REGISTERED; the slot is always compared       */
#define BF_RESYNC_ALL_FIELDS 0x3Fu
#define BF_RESYNC_NONE 0xFFFFFFFFu
typedef struct bf_drift {        /* 16 B                                                                                       */
  uint32_t run;
  uint16_t index;                /* step (PHASE / COND / DECISION), child nibble (CHILD), desc (REGISTERED), else 0             */
  uint8_t field;                 /* BF_DELTA_*                                                                                 */
  uint8_t reserved;
  uint32_t device, record;       /* the compared values: the device's and the caller's                                        */
} bf_drift;
typedef struct bf_resync {
  uint32_t struct_size;          /* sizeof(bf_resync)                                                                          */
  uint32_t n_runs;               /* in: the batch's runs are [0, n_runs)                                                       */
  const uint32_t* runs;          /* in: [n] strictly ascending, below n_runs; NULL with n == n_runs: every run of [0, n_runs)  */
  uint32_t n;
  uint32_t fields;               /* in: BF_RESYNC_FIELD(BF_DELTA_*) bits                                                       */
  const void* records;           /* in: n state records in list order, the batch's layout                                      */
  uint32_t flags;                /* in: BF_RESYNC_CHECK                                                                        */
  uint32_t drifted_cap;
  uint32_t* drifted;             /* [drifted_cap] out: ascending runs with at least one item                                   */
  uint32_t n_drifted;            /* out: the true count                                                                        */
  uint32_t n_written;            /* out: runs repaired (0 with BF_RESYNC_CHECK)                                                */
  bf_drift* items;               /* [items_cap] out                                                                            */
  uint64_t items_cap;
  uint64_t n_items;              /* out: the true count; only the first items_cap were written                                */
  uint32_t bad_run;              /* out on a refusal: the run whose record names an unknown slot, else BF_RESYNC_NONE          */
  uint32_t reserved;
} bf_resync;

int bf_resident_resync(bf_ctx* ctx, uint32_t handle, bf_resync* r);

/* bf_resident_resync_areas: the same for the per-run side areas a batcher persists outside the state records: the step timers (the
 * runs.bubustack.io/step-timers annotation, stepTimerStore dag.go:64,110-190), the limiter inputs (labels, priority, queue origin
 * and StoryRun phase) and the run control (StartedAt + policy.timeouts.story, spec.cancelRequested).  The caller packs each selected
 * area (`areas`) for the listed runs, in list order, as the upload calls take them; the device compares them with its own, lists
 * every difference and, without BF_RESYNC_CHECK, repairs only the runs that drifted.  Resync the records first: the timer rules read
 * the device's phases and decisions.
 *
 * What is compared: what the device's next bf_resident_fire and bf_resident_schedule would do, not raw bytes.
 *   - TIMERS (run not stopped on the device, and not stopped by the caller's run control when RUNCTL is selected: a stopped run's slots
 *     are empty by the stop rule, so such a run compares and writes no timers).  The slots of a step are compared only when the
 *     device's STORED phase code at that step is not terminal (BF_LUT_TERMINAL): a slot at a terminal step is dormant and the next
 *     fire prunes it (pruneTerminal, dag.go:173-190).  A step with a slot on both sides lists BF_DRIFT_TIMER when the deadlines
 *     differ and BF_DRIFT_TIMER_CODE when the codes differ.  A step with a slot on one side lists BF_DRIFT_TIMER with BF_TIMER_NONE
 *     on the other side, except a caller slot TAKEN AS FIRED: the device has no slot at its step, fired_now != BF_TIMER_NONE, its
 *     deadline <= fired_now, and its code is BF_DEC_PENDING (wake-only) or the device's decision code at the step is not
 *     BF_DEC_PENDING.  The fire disarms a due slot while the annotation keeps it until the step is terminal, so such a slot is
 *     equal.  A due caller slot whose step still has decision PENDING on the device is drift: the stuck step the repair re-arms.
 *   - SCHED: the five stored inputs (story_key, queue_key, priority, queued_since, run_phase), one item each (index 0).
 *   - RUNCTL: story_deadline as stored (a stopped run keeps it, dormant); drain_deadline by the taken-as-fired rule (a caller drain
 *     deadline the device no longer has, due at fired_now, is equal: the fire disarms it); the stop by reason (BF_DRIFT_STOP).
 * Items (bf_drift) are ordered by (run, field, index); device and record are the compared values (deadlines, codes, inputs, stop
 * reasons).  The field codes below are disjoint from BF_DELTA_*, so one loop consumes the items of both resync calls.
 *
 * Repair (without BF_RESYNC_CHECK), of the drifted runs and, in a run, of the areas it lists items for:
 *   - timers: the run's K slots become the caller's slots minus those taken as fired, in the canonical layout.  Touches no run;
 *   - limiter inputs: the run's inputs become the caller's.  Touches no run and needs no new tick: the next schedule lists the run
 *     when its schedule changes;
 *   - deadlines: each drifted deadline takes the caller's value;
 *   - a caller stop on a run the device has not stopped stops the run exactly as bf_resident_runctl_put does (saved flags byte,
 *     stopped byte, timers emptied, run_phase = BF_PHASE_TIMEOUT for BF_STOP_TIMEOUT with a limiter area, the run touched, the
 *     evaluated snapshot and the schedule's tick ended).  This runs after the inputs are written.  A device stop the caller lacks,
 *     or a stop of another reason, is listed and kept: only a redrive lifts a stop, and stopping again changes nothing.
 *   n_written counts the runs whose areas or record the repair changed (a run whose only items are a kept stop is not one).  A call
 *   that wrote no stop changes no state record and ends nothing; every BF_RESYNC_CHECK call changes nothing at all.
 * Refused before anything is written, BF_EINVAL and nothing changed, bad_run naming the first offending run where there is one (else
 * BF_RESYNC_NONE): struct_size or the handle; n_runs > capacity, runs not strictly ascending or not below n_runs, runs == NULL with
 * n != n_runs; unknown flags or areas bits; a selected area the batch has no area for (bf_resident_timers / _sched / _runctl: a caller
 * packing an area for a batch without one has a bug); a NULL array of a selected area with n > 0; drifted / items NULL with a
 * non-zero cap; a timer row that is not canonical (armed slots first, strictly ascending by step, step < steps_max, code <= 3, a
 * non-PENDING code only with decision planes, reserved 0; an empty slot is deadline BF_TIMER_NONE with every other byte 0); a sched
 * row whose run is not the listed run, or with non-zero reserved words; a runctl row with stop > BF_STOP_HOST or non-zero
 * saved_flags / reserved bytes.
 * Cost: one H2D copy per selected area straight from the caller's array (and one of a run list not in pinned memory), three launches
 * (count, scan, list and repair: one warp per listed run, lane t on slots t and t + 32, no shared stage), one D2H copy of the totals,
 * one synchronisation.  Pinned drifted / items buffers are written in place, others staged and copied after it.  A batch that never
 * calls this launches nothing more than before.                                                                                  */
#define BF_RESYNC_AREA_TIMERS 0x1u
#define BF_RESYNC_AREA_SCHED 0x2u
#define BF_RESYNC_AREA_RUNCTL 0x4u
#define BF_RESYNC_ALL_AREAS 0x7u
enum {                            /* bf_drift.field of bf_resident_resync_areas (BF_DELTA_* end at 6)                           */
  BF_DRIFT_TIMER = 8,             /* index = step; the deadlines, BF_TIMER_NONE for a side without a slot at the step            */
  BF_DRIFT_TIMER_CODE = 9,        /* index = step; the codes of the two slots at the step                                        */
  BF_DRIFT_SCHED_STORY_KEY = 10,  /* index 0; the five stored limiter inputs, in bf_sched_put order                              */
  BF_DRIFT_SCHED_QUEUE_KEY = 11,
  BF_DRIFT_SCHED_PRIORITY = 12,
  BF_DRIFT_SCHED_QUEUED_SINCE = 13,
  BF_DRIFT_SCHED_RUN_PHASE = 14,
  BF_DRIFT_STORY_DEADLINE = 15,   /* index 0; the deadlines                                                                      */
  BF_DRIFT_DRAIN_DEADLINE = 16,
  BF_DRIFT_STOP = 17              /* index 0; the BF_STOP_* reasons                                                              */
};
typedef struct bf_resync_areas {
  uint32_t struct_size;           /* sizeof(bf_resync_areas)                                                                     */
  uint32_t n_runs;                /* in: the batch's runs are [0, n_runs)                                                        */
  const uint32_t* runs;           /* in: [n] strictly ascending, below n_runs; NULL with n == n_runs: every run of [0, n_runs)   */
  uint32_t n;
  uint32_t areas;                 /* in: BF_RESYNC_AREA_* bits                                                                   */
  uint32_t flags;                 /* in: BF_RESYNC_CHECK                                                                         */
  uint32_t fired_now;             /* in: `now` of the last bf_resident_fire on this batch, BF_TIMER_NONE: none                   */
  const bf_timer_slot* timers;    /* in: [n * K] each run's K slots (K: the batch's current K), canonical, list order            */
  const bf_sched_put* sched;      /* in: [n] .run = the listed run, reserved 0                                                   */
  const bf_run_ctl* runctl;       /* in: [n] saved_flags and reserved 0                                                          */
  uint32_t drifted_cap;
  uint32_t n_drifted;             /* out: the true count                                                                         */
  uint32_t* drifted;              /* [drifted_cap] out: ascending runs with at least one item                                    */
  uint32_t n_written;             /* out: runs the repair changed (0 with BF_RESYNC_CHECK)                                       */
  uint32_t bad_run;               /* out on a refusal: the offending run, else BF_RESYNC_NONE                                    */
  bf_drift* items;                /* [items_cap] out                                                                             */
  uint64_t items_cap;
  uint64_t n_items;               /* out: the true count; only the first items_cap were written                                 */
} bf_resync_areas;

int bf_resident_resync_areas(bf_ctx* ctx, uint32_t handle, bf_resync_areas* r);

/* ------------------------------------------------------------------ device groups (SURVEY.md row e)
 * The reference is ONE operator process (cmd/main.go:220, StoryRunReconciler storyrun_controller.go:216), so the
 * multi-GPU path must be reachable from one process through this ABI: a group owns one ctx per device and an NCCL
 * communicator over them (ncclCommInitAll; libnccl.so.2 is loaded at bf_group_create, the library itself does not
 * link it).  StoryRuns are independent, so a batch shards into contiguous blocks of ceil(N / G) runs with NO
 * data-path collective; the one exchange of a pass is an ncclAllGather of each shard's 32-byte counts block, which
 * gives every shard the global totals and the offsets of its compacted lists.  Topologies live where their runs
 * are: put them through the shard's own ctx (bf_group_ctx + bf_topology_put_many; slot ids are per shard) or
 * replicate a shared set on every device with bf_group_topology_put_many (same slot ids everywhere).
 * Collective failures come back as BF_ENCCL with the NCCL text in bf_group_last_error.                            */
typedef struct bf_group bf_group;

int bf_group_create(bf_group** out, const int32_t* devices, uint32_t n_devices, const bf_config* cfg /* device field ignored; may be NULL */);
void bf_group_destroy(bf_group* g);
uint32_t bf_group_size(const bf_group* g);
bf_ctx* bf_group_ctx(bf_group* g, uint32_t shard);
const char* bf_group_last_error(const bf_group* g);
/* Runs [*first, *first + *count) of an n_runs batch belong to `shard`.                                            */
int bf_group_shard_range(const bf_group* g, uint32_t n_runs, uint32_t shard, uint32_t* first, uint32_t* count);
/* The same topologies on every device; fails with BF_ETOPO if the shards' slot tables have diverged (mixing
 * replicated and per-shard uploads is allowed only when the replicated ones come first).                          */
int bf_group_topology_put_many(bf_group* g, const bf_topology* topos, uint32_t count, uint32_t* slots_out);
/* One pass over a HOST batch sharded across the group: every shard runs bf_eval on its block of runs (its own H2D /
 * kernels / D2H pipeline, all shards concurrently), then the counts are all-gathered on the devices.
 * shard_counts[n_devices] (may be NULL) receives the gathered per-shard counts, batch->counts the global totals.
 * BF_EVAL_EXPANSION is not offered here (per-shard lists: call bf_eval on bf_group_ctx).                           */
int bf_group_eval(bf_group* g, const bf_batch* batch, bf_counts* shard_counts);
/* bf_schedule for a batch evaluated by the IMMEDIATELY PRECEDING bf_group_eval: every shard counts its own Running
 * StepRuns and demand, the per-story / per-queue / global totals are all-reduced (sum) and the per-queue highest
 * effective priority (max) across the shards, then every shard truncates its ready sets against the GLOBAL totals —
 * the limits and the priority ordering hold across the whole batch, as enforcePriorityOrdering / enforceSchedulingLimits
 * (dag.go:1801-1946) hold across the cluster.  runs[n_runs] and out->records cover the whole batch; the totals arrays
 * of `out` receive the global values.                                                                             */
int bf_group_schedule(bf_group* g, const bf_batch* batch, const bf_sched_run* runs, const bf_sched_tables* tables, bf_sched_out* out);

/* Pinned host memory for batches (cgo: memory with no Go pointers).           */
int bf_alloc_pinned(bf_ctx* ctx, size_t bytes, void** out);
int bf_free_pinned(bf_ctx* ctx, void* p);

/* Introspection used by bench/roofline accounting.                            */
typedef struct bf_stats {
  uint64_t kernel_launches;   /* kernels launched by this ctx so far            */
  uint64_t arena_used_bytes;  /* HBM bytes of topology records                  */
  uint64_t arena_cap_bytes;
  uint32_t n_topologies;
  uint32_t sm_count;
  uint32_t last_grid, last_block, last_smem_bytes, last_stages;
  uint32_t last_kernel;        /* 0 = one run per warp (general), 1 = packed lanes, 2 = packed lanes + deferred general;
                                  3, 4, 5: the same over the run list of a touched tick                                   */
  uint32_t last_runs_per_trip; /* StoryRuns evaluated per warp trip by the last pass                                   */
  uint32_t last_eval_chunks;   /* run chunks the last bf_eval pipelined over its copy/compute streams (1 = serial)      */
  uint32_t arena_compactions;  /* times the topology arena was re-packed (dropped records reclaimed)                             */
} bf_stats;
int bf_get_stats(const bf_ctx* ctx, bf_stats* out);
/* Device address + byte size of a topology record (for traffic accounting).   */
int bf_topology_record(const bf_ctx* ctx, uint32_t slot, uint64_t* dev_addr, uint32_t* bytes);
/* Host-only (no ctx, no GPU): validates `topo` exactly as bf_topology_put does and writes the device record it would upload
 * (the row format chosen for it, device_record.h) into out[cap]; *bytes_out = the record's size, also when cap is too
 * small (then nothing is written and BF_ENOMEM is returned).  For tests and for sizing an arena.                          */
int bf_topology_record_build(const bf_topology* topo, void* out, uint32_t cap, uint32_t* bytes_out);

#ifdef __cplusplus
}
#endif
#endif /* BOBRAFRONTIER_H_ */
