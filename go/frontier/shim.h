/*
 * shim.h — flat C wrappers over include/bobrafrontier.h for the cgo binding (go/frontier/frontier.go).
 *
 * cgo forbids passing a pointer to Go memory that itself contains Go pointers ("cgo argument has Go pointer to
 * unpinned Go pointer").  The ABI's argument structs (bf_topology, bf_batch, bf_sched_tables, bf_sched_out,
 * bf_compact_out) hold pointers, so they must never be built in Go memory.  Every wrapper below takes the scalars and
 * the buffer pointers as FLAT arguments — a Go caller passes &slice[0] of slices that hold no pointers, which is legal —
 * and builds the struct here, on the C stack.
 *
 * The same header is compiled by tests/c_abi_harness.c (gcc, no Go needed), which performs the call sequence of
 * frontier.go against the real library on a GPU: the struct layouts and the argument order the Go side relies on are
 * exercised even though this image has no Go toolchain.
 */
#ifndef BOBRAFRONTIER_GO_SHIM_H_
#define BOBRAFRONTIER_GO_SHIM_H_

#include <stdlib.h>
#include <string.h>

#include "bobrafrontier.h"

static inline int bfgo_create(int32_t device, bf_ctx** out) {
  bf_config cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.struct_size = (uint32_t)sizeof cfg;
  cfg.device = device;
  return bf_create(out, &cfg);
}

static inline int bfgo_topology_put(bf_ctx* c, uint32_t n_steps, uint32_t n_edges, const uint32_t* row_ptr, const uint16_t* col_idx,
                                    const uint8_t* step_flags, const bf_parallel_desc* parallel, uint32_t n_parallel,
                                    const uint8_t* allow_bits, uint32_t n_allow_bits, uint32_t* slot_out) {
  bf_topology t;
  memset(&t, 0, sizeof t);
  t.n_steps = n_steps; t.n_edges = n_edges; t.row_ptr = row_ptr; t.col_idx = col_idx; t.step_flags = step_flags;
  t.parallel = parallel; t.n_parallel = n_parallel; t.branch_allow_bits = allow_bits; t.n_branch_allow_bits = n_allow_bits;
  return bf_topology_put(c, &t, slot_out);
}

static inline void bfgo_batch(bf_batch* b, const bf_layout* L, uint32_t n_runs, uint32_t flags, uint32_t max_iterations, const void* state,
                              void* result, bf_counts* counts) {
  memset(b, 0, sizeof *b);
  b->struct_size = (uint32_t)sizeof *b;
  b->n_runs = n_runs; b->flags = flags; b->max_iterations = max_iterations; b->layout = *L;
  b->state = state; b->result = result; b->counts = counts;
}

static inline int bfgo_eval(bf_ctx* c, const bf_layout* L, uint32_t n_runs, uint32_t flags, uint32_t max_iterations, const void* state,
                            void* result, bf_counts* counts) {
  bf_batch b;
  bfgo_batch(&b, L, n_runs, flags, max_iterations, state, result, counts);
  return bf_eval(c, &b);
}

static inline void bfgo_compact(bf_compact_out* co, uint32_t* head, uint16_t* events, uint64_t events_cap) {
  memset(co, 0, sizeof *co);
  co->struct_size = (uint32_t)sizeof *co;
  co->head = head; co->events = events; co->events_cap = events_cap;
}

static inline int bfgo_eval_compact(bf_ctx* c, const bf_layout* L, uint32_t n_runs, uint32_t flags, uint32_t max_iterations,
                                    const void* state, uint32_t* head, uint16_t* events, uint64_t events_cap,
                                    uint64_t* n_events, uint32_t* n_listed, bf_counts* counts) {
  bf_batch b;
  bf_compact_out co;
  bfgo_batch(&b, L, n_runs, flags, max_iterations, state, NULL, counts);
  bfgo_compact(&co, head, events, events_cap);
  const int rc = bf_eval_compact(c, &b, &co);
  *n_events = co.n_events;
  *n_listed = co.n_listed;
  return rc;
}

static inline int bfgo_resident_tick_compact(bf_ctx* c, uint32_t handle, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs,
                                             uint32_t flags, uint32_t max_iterations, uint32_t* head, uint16_t* events,
                                             uint64_t events_cap, uint64_t* n_events, uint32_t* n_listed, bf_counts* counts) {
  bf_compact_out co;
  bfgo_compact(&co, head, events, events_cap);
  const int rc = bf_resident_tick_compact(c, handle, deltas, n_deltas, n_runs, flags, max_iterations, &co, counts);
  *n_events = co.n_events;
  *n_listed = co.n_listed;
  return rc;
}

static inline int bfgo_resident_tick_touched(bf_ctx* c, uint32_t handle, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs,
                                             uint32_t flags, uint32_t max_iterations, uint32_t* runs, uint32_t* head, uint32_t runs_cap,
                                             uint16_t* events, uint64_t events_cap, uint32_t* full, uint32_t* n_listed,
                                             uint32_t* n_evaluated, uint64_t* n_events, bf_counts* counts) {
  bf_touched_out to;
  memset(&to, 0, sizeof to);
  to.struct_size = (uint32_t)sizeof to;
  to.runs = runs; to.head = head; to.runs_cap = runs_cap; to.events = events; to.events_cap = events_cap;
  const int rc = bf_resident_tick_touched(c, handle, deltas, n_deltas, n_runs, flags, max_iterations, &to, counts);
  *full = to.full;
  *n_listed = to.n_listed;
  *n_evaluated = to.n_evaluated;
  *n_events = to.n_events;
  return rc;
}

/* bf_resident_tick_touched_many over flat arrays: part k is batch handles[k] over n_runs[k] runs, its deltas are
 * deltas[delta_first[k] .. delta_first[k + 1]), its runs / head lists runs[runs_first[k] ..] and head[runs_first[k] ..] up to
 * runs_first[k + 1], its events events[events_first[k] .. events_first[k + 1]); its outputs land at index k of full, n_listed,
 * n_evaluated, n_events and counts.  The part and out structs are built here, in C memory.                                 */
static inline int bfgo_resident_tick_touched_many(bf_ctx* c, uint32_t flags, uint32_t max_iterations, uint32_t n_parts,
                                                  const uint32_t* handles, const uint32_t* n_runs, const bf_delta* deltas,
                                                  const uint32_t* delta_first, uint32_t* runs, uint32_t* head,
                                                  const uint32_t* runs_first, uint16_t* events, const uint64_t* events_first,
                                                  uint32_t* full, uint32_t* n_listed, uint32_t* n_evaluated, uint64_t* n_events,
                                                  bf_counts* counts, uint32_t* bad_part) {
  bf_tick_part* parts = (bf_tick_part*)calloc(n_parts ? n_parts : 1, sizeof(bf_tick_part));
  bf_touched_out* outs = (bf_touched_out*)calloc(n_parts ? n_parts : 1, sizeof(bf_touched_out));
  if (!parts || !outs) {
    free(parts);
    free(outs);
    *bad_part = 0xFFFFFFFFu;
    return BF_ENOMEM;
  }
  for (uint32_t k = 0; k < n_parts; ++k) {
    bf_touched_out* o = &outs[k];
    o->struct_size = (uint32_t)sizeof *o;
    o->runs_cap = runs_first[k + 1] - runs_first[k];
    o->runs = o->runs_cap ? runs + runs_first[k] : NULL;
    o->head = o->runs_cap ? head + runs_first[k] : NULL;
    o->events_cap = events_first[k + 1] - events_first[k];
    o->events = o->events_cap ? events + events_first[k] : NULL;
    bf_tick_part* p = &parts[k];
    p->struct_size = (uint32_t)sizeof *p;
    p->handle = handles[k];
    p->n_deltas = delta_first[k + 1] - delta_first[k];
    p->deltas = p->n_deltas ? deltas + delta_first[k] : NULL;
    p->n_runs = n_runs[k];
    p->out = o;
    p->counts = &counts[k];
  }
  const int rc = bf_resident_tick_touched_many(c, flags, max_iterations, parts, n_parts, bad_part);
  for (uint32_t k = 0; k < n_parts; ++k) {
    full[k] = outs[k].full;
    n_listed[k] = outs[k].n_listed;
    n_evaluated[k] = outs[k].n_evaluated;
    n_events[k] = outs[k].n_events;
  }
  free(parts);
  free(outs);
  return rc;
}

static inline int bfgo_resident_migrate(bf_ctx* c, uint32_t handle, uint32_t old_slot, uint32_t new_slot, const uint16_t* step_map,
                                        uint32_t n_old_steps, uint32_t n_runs, uint32_t* migrated) {
  bf_migration m;
  memset(&m, 0, sizeof m);
  m.struct_size = (uint32_t)sizeof m;
  m.old_slot = old_slot; m.new_slot = new_slot; m.n_runs = n_runs; m.step_map = step_map; m.n_old_steps = n_old_steps;
  const int rc = bf_resident_migrate(c, handle, &m);
  *migrated = m.migrated;
  return rc;
}

static inline int bfgo_resident_redrive(bf_ctx* c, uint32_t handle, const bf_redrive* requests, uint32_t n, uint8_t* status,
                                        uint32_t* applied) {
  *applied = 0;
  return bf_resident_redrive(c, handle, requests, n, status, applied);
}

/* bf_resident_reshape with the new layout built here by bf_layout_init; *layout_out receives it when the reshape succeeded. */
static inline int bfgo_resident_reshape(bf_ctx* c, uint32_t handle, uint32_t steps_max, uint32_t child_nibbles, uint32_t fields,
                                        uint32_t capacity, bf_layout* layout_out) {
  bf_layout L;
  const int rc = bf_layout_init(&L, steps_max, child_nibbles, fields);
  if (rc != BF_OK) return rc;
  const int rc2 = bf_resident_reshape(c, handle, &L, capacity);
  if (rc2 == BF_OK) *layout_out = L;
  return rc2;
}

/* bf_resident_retire with the bf_retire built here on the C stack (a Go struct holding Go pointers may not be passed to C). */
static inline int bfgo_resident_retire(bf_ctx* c, uint32_t handle, uint32_t n_runs, const uint32_t* runs, uint32_t n, uint32_t capacity,
                                       uint32_t* moves_from, uint32_t* moves_to, uint32_t* n_runs_out, uint32_t* n_moves_out) {
  bf_retire r;
  memset(&r, 0, sizeof r);
  r.struct_size = (uint32_t)sizeof r;
  r.n_runs = n_runs; r.runs = runs; r.n = n; r.capacity = capacity; r.moves_from = moves_from; r.moves_to = moves_to;
  const int rc = bf_resident_retire(c, handle, &r);
  *n_runs_out = rc == BF_OK ? r.n_runs : n_runs;
  *n_moves_out = rc == BF_OK ? r.n_moves : 0;
  return rc;
}

/* bf_resident_extent / bf_resident_narrow with the bf_extent built here on the C stack; narrow builds the new layout with
 * bf_layout_init and *layout_out receives it when the narrow succeeded.  out[4] = steps_max, child_nibbles, fields, widest_run
 * (filled by a rejected narrow too, so that the caller sees why). */
static inline int bfgo_resident_extent(bf_ctx* c, uint32_t handle, uint32_t n_runs, uint32_t* out) {
  bf_extent e;
  memset(&e, 0, sizeof e);
  e.struct_size = (uint32_t)sizeof e;
  e.n_runs = n_runs;
  const int rc = bf_resident_extent(c, handle, &e);
  out[0] = e.steps_max; out[1] = e.child_nibbles; out[2] = e.fields; out[3] = e.widest_run;
  return rc;
}

static inline int bfgo_resident_narrow(bf_ctx* c, uint32_t handle, uint32_t steps_max, uint32_t child_nibbles, uint32_t fields,
                                       uint32_t n_runs, uint32_t* out, bf_layout* layout_out) {
  bf_layout L;
  int rc = bf_layout_init(&L, steps_max, child_nibbles, fields);
  if (rc != BF_OK) return rc;
  bf_extent e;
  memset(&e, 0, sizeof e);
  e.struct_size = (uint32_t)sizeof e;
  e.n_runs = n_runs;
  rc = bf_resident_narrow(c, handle, &L, &e);
  out[0] = e.steps_max; out[1] = e.child_nibbles; out[2] = e.fields; out[3] = e.widest_run;
  if (rc == BF_OK) *layout_out = L;
  return rc;
}

/* bf_resident_transfer with the bf_transfer built here on the C stack.  counts[4] = src_n_runs, dst_n_runs, n_moves, unfit
 * (the n_runs given back and BF_EXTENT_NO_RUN moves on a refusal); why[4] = steps_max, child_nibbles, fields, widest_run of
 * the run a fit refusal names. */
static inline int bfgo_resident_transfer(bf_ctx* c, uint32_t src, uint32_t dst, uint32_t src_n_runs, uint32_t dst_n_runs,
                                         const uint32_t* runs, uint32_t n, uint32_t* moves_from, uint32_t* moves_to,
                                         uint32_t* counts, uint32_t* why) {
  bf_transfer t;
  memset(&t, 0, sizeof t);
  t.struct_size = (uint32_t)sizeof t;
  t.src_n_runs = src_n_runs; t.dst_n_runs = dst_n_runs; t.runs = runs; t.n = n; t.moves_from = moves_from; t.moves_to = moves_to;
  const int rc = bf_resident_transfer(c, src, dst, &t);
  counts[0] = rc == BF_OK ? t.src_n_runs : src_n_runs;
  counts[1] = rc == BF_OK ? t.dst_n_runs : dst_n_runs;
  counts[2] = rc == BF_OK ? t.n_moves : 0;
  counts[3] = t.unfit;
  why[0] = t.why.steps_max; why[1] = t.why.child_nibbles; why[2] = t.why.fields; why[3] = t.why.widest_run;
  return rc;
}

/* Step timers.  bf_resident_timers and bf_resident_timers_arm are called directly (flat arguments already); bf_resident_fire with
 * the bf_fire_out built here on the C stack.  counts[5] = n_fired, n_written, n_pruned, next_deadline, entries written into
 * fired (min(n_fired, fired_cap)). */
/* bf_resident_transfer_ctx with the bf_ctx_transfer built here on the C stack.  counts[5] = src_n_runs, dst_n_runs, n_moves,
 * unfit, unfit_reason (the n_runs given back and no moves on a refusal); why[4] as bfgo_resident_transfer. */
static inline int bfgo_resident_transfer_ctx(bf_ctx* sc, uint32_t src, bf_ctx* dc, uint32_t dst, uint32_t src_n_runs,
                                             uint32_t dst_n_runs, const uint32_t* runs, uint32_t n, const uint32_t* slot_map,
                                             uint32_t n_slot_map, uint32_t* moves_from, uint32_t* moves_to, uint32_t* counts,
                                             uint32_t* why) {
  bf_ctx_transfer t;
  memset(&t, 0, sizeof t);
  t.struct_size = (uint32_t)sizeof t;
  t.src_n_runs = src_n_runs; t.dst_n_runs = dst_n_runs; t.runs = runs; t.n = n; t.slot_map = slot_map; t.n_slot_map = n_slot_map;
  t.moves_from = moves_from; t.moves_to = moves_to;
  const int rc = bf_resident_transfer_ctx(sc, src, dc, dst, &t);
  counts[0] = rc == BF_OK ? t.src_n_runs : src_n_runs;
  counts[1] = rc == BF_OK ? t.dst_n_runs : dst_n_runs;
  counts[2] = rc == BF_OK ? t.n_moves : 0;
  counts[3] = t.unfit;
  counts[4] = t.unfit_reason;
  why[0] = t.why.steps_max; why[1] = t.why.child_nibbles; why[2] = t.why.fields; why[3] = t.why.widest_run;
  return rc;
}

static inline int bfgo_resident_fire(bf_ctx* c, uint32_t handle, uint32_t n_runs, uint32_t now, bf_fired* fired, uint32_t fired_cap,
                                     uint32_t* counts) {
  bf_fire_out o;
  memset(&o, 0, sizeof o);
  o.struct_size = (uint32_t)sizeof o;
  o.n_runs = n_runs; o.fired = fired; o.fired_cap = fired_cap;
  const int rc = bf_resident_fire(c, handle, now, &o);
  counts[0] = o.n_fired; counts[1] = o.n_written; counts[2] = o.n_pruned; counts[3] = o.next_deadline;
  counts[4] = o.n_fired < fired_cap ? o.n_fired : fired_cap;
  return rc;
}

/* StoryRun stops and deadlines.  bf_resident_runctl is called directly; a put of one run's deadlines and stop is built here on
 * the C stack (bf_resident_runctl_put takes any number: a batcher with many sends them through bf_resident_runctl_put itself). */
static inline int bfgo_resident_runctl_put1(bf_ctx* c, uint32_t handle, uint32_t run, uint32_t story_deadline, uint32_t drain_deadline,
                                            uint8_t stop) {
  bf_run_ctl_put q;
  memset(&q, 0, sizeof q);
  q.run = run; q.story_deadline = story_deadline; q.drain_deadline = drain_deadline; q.stop = stop;
  return bf_resident_runctl_put(c, handle, &q, 1);
}

/* Tick commits.  The entries are passed as they are (bf_commit_entry holds no pointers); the out block comes back flat:
 * counts[0..6] = runs written, skipped, launched, queued, failed, bad_run, bad_step. */
static inline int bfgo_resident_commit(bf_ctx* c, uint32_t handle, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n,
                                       uint32_t* counts) {
  bf_commit_out o;
  memset(&o, 0, sizeof o);
  o.struct_size = (uint32_t)sizeof o;
  const int rc = bf_resident_commit(c, handle, n_runs, entries, n, &o);
  counts[0] = o.n_runs_written; counts[1] = o.n_skipped; counts[2] = o.n_launched; counts[3] = o.n_queued; counts[4] = o.n_failed;
  counts[5] = o.bad_run; counts[6] = o.bad_step;
  return rc;
}

/* Tick commits that arm step timers: as bfgo_resident_commit, and counts[7..8] = slots armed, earliest deadline armed. */
static inline int bfgo_resident_commit_timed(bf_ctx* c, uint32_t handle, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n,
                                             uint32_t now, uint32_t* counts) {
  bf_commit_out o;
  memset(&o, 0, sizeof o);
  o.struct_size = (uint32_t)sizeof o;
  bf_commit_arm a;
  memset(&a, 0, sizeof a);
  a.struct_size = (uint32_t)sizeof a;
  a.now = now;
  const int rc = bf_resident_commit_timed(c, handle, n_runs, entries, n, &o, &a);
  counts[0] = o.n_runs_written; counts[1] = o.n_skipped; counts[2] = o.n_launched; counts[3] = o.n_queued; counts[4] = o.n_failed;
  counts[5] = o.bad_run; counts[6] = o.bad_step; counts[7] = a.n_armed; counts[8] = a.next_deadline;
  return rc;
}

/* Tick commits that list their writes: as bfgo_resident_commit_timed when now != BF_TIMER_NONE, else as bfgo_resident_commit (no
 * arming), and the journal's items and runs land in the caller's buffers (bf_commit_write holds no pointers).  counts[9] = runs
 * listed (the true count), *n_items = items (the true count); only the first items_cap / runs_cap are written. */
static inline int bfgo_resident_commit_journal(bf_ctx* c, uint32_t handle, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n,
                                               uint32_t now, bf_commit_write* items, uint64_t items_cap, uint32_t* runs,
                                               uint32_t runs_cap, uint32_t* counts, uint64_t* n_items) {
  bf_commit_out o;
  memset(&o, 0, sizeof o);
  o.struct_size = (uint32_t)sizeof o;
  bf_commit_arm a;
  memset(&a, 0, sizeof a);
  a.struct_size = (uint32_t)sizeof a;
  a.now = now;
  bf_commit_journal j;
  memset(&j, 0, sizeof j);
  j.struct_size = (uint32_t)sizeof j;
  j.items = items; j.items_cap = items_cap; j.runs = runs; j.runs_cap = runs_cap;
  const int rc = bf_resident_commit_journal(c, handle, n_runs, entries, n, &o, now == BF_TIMER_NONE ? NULL : &a, &j);
  counts[0] = o.n_runs_written; counts[1] = o.n_skipped; counts[2] = o.n_launched; counts[3] = o.n_queued; counts[4] = o.n_failed;
  counts[5] = o.bad_run; counts[6] = o.bad_step;
  counts[7] = now == BF_TIMER_NONE ? 0u : a.n_armed; counts[8] = now == BF_TIMER_NONE ? BF_TIMER_NONE : a.next_deadline;
  counts[9] = j.n_runs_listed;
  *n_items = j.n_items;
  return rc;
}

/* bfgo_resident_commit_journal through bf_resident_commit_rewrites: counts[10] = the steps written from the stages G / H / I. */
static inline int bfgo_resident_commit_rewrites(bf_ctx* c, uint32_t handle, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n,
                                                uint32_t now, bf_commit_write* items, uint64_t items_cap, uint32_t* runs,
                                                uint32_t runs_cap, uint32_t* counts, uint64_t* n_items) {
  bf_commit_out o;
  memset(&o, 0, sizeof o);
  o.struct_size = (uint32_t)sizeof o;
  bf_commit_arm a;
  memset(&a, 0, sizeof a);
  a.struct_size = (uint32_t)sizeof a;
  a.now = now;
  bf_commit_journal j;
  memset(&j, 0, sizeof j);
  j.struct_size = (uint32_t)sizeof j;
  j.items = items; j.items_cap = items_cap; j.runs = runs; j.runs_cap = runs_cap;
  uint32_t nrw = 0;
  const int rc = bf_resident_commit_rewrites(c, handle, n_runs, entries, n, &o, now == BF_TIMER_NONE ? NULL : &a, &j, &nrw);
  counts[0] = o.n_runs_written; counts[1] = o.n_skipped; counts[2] = o.n_launched; counts[3] = o.n_queued; counts[4] = o.n_failed;
  counts[5] = o.bad_run; counts[6] = o.bad_step;
  counts[7] = now == BF_TIMER_NONE ? 0u : a.n_armed; counts[8] = now == BF_TIMER_NONE ? BF_TIMER_NONE : a.next_deadline;
  counts[9] = j.n_runs_listed;
  counts[10] = nrw;
  *n_items = j.n_items;
  return rc;
}

/* Touched commits (bf_resident_commit_touched) of the form the arguments pick: arming when now != BF_TIMER_NONE, journaled when
 * journal != 0 (items and runs as bfgo_resident_commit_journal), rewriting when flags carries BF_COMMIT_SCOPE_REWRITES (needs the
 * journal).  counts as bfgo_resident_commit_rewrites (counts[7..10] zero / BF_TIMER_NONE where the form has no such field), and
 * counts[11] = full, counts[12] = runs considered.  bf_resident_commit_marks enables the batch's commit-due bits first. */
static inline int bfgo_resident_commit_touched(bf_ctx* c, uint32_t handle, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n,
                                               uint32_t now, uint32_t flags, uint32_t journal, bf_commit_write* items,
                                               uint64_t items_cap, uint32_t* runs, uint32_t runs_cap, uint32_t* counts,
                                               uint64_t* n_items) {
  bf_commit_out o;
  memset(&o, 0, sizeof o);
  o.struct_size = (uint32_t)sizeof o;
  bf_commit_arm a;
  memset(&a, 0, sizeof a);
  a.struct_size = (uint32_t)sizeof a;
  a.now = now;
  bf_commit_journal j;
  memset(&j, 0, sizeof j);
  j.struct_size = (uint32_t)sizeof j;
  j.items = items; j.items_cap = items_cap; j.runs = runs; j.runs_cap = runs_cap;
  bf_commit_scope sc;
  memset(&sc, 0, sizeof sc);
  sc.struct_size = (uint32_t)sizeof sc;
  sc.flags = flags;
  uint32_t nrw = 0;
  const int rc = bf_resident_commit_touched(c, handle, n_runs, entries, n, &o, now == BF_TIMER_NONE ? NULL : &a, journal ? &j : NULL,
                                            &nrw, &sc);
  counts[0] = o.n_runs_written; counts[1] = o.n_skipped; counts[2] = o.n_launched; counts[3] = o.n_queued; counts[4] = o.n_failed;
  counts[5] = o.bad_run; counts[6] = o.bad_step;
  counts[7] = now == BF_TIMER_NONE ? 0u : a.n_armed; counts[8] = now == BF_TIMER_NONE ? BF_TIMER_NONE : a.next_deadline;
  counts[9] = journal ? j.n_runs_listed : 0u;
  counts[10] = (flags & BF_COMMIT_SCOPE_REWRITES) ? nrw : 0u;
  counts[11] = sc.full; counts[12] = sc.n_considered;
  *n_items = journal ? j.n_items : 0u;
  return rc;
}

/* Run status.  The records (bf_status_rec holds no pointers) and events land in the caller's buffers; *n_events = the events of
 * the listed runs, of which the first events_cap were written.  runs == NULL with n == n_runs lists every run of [0, n_runs). */
static inline int bfgo_resident_status(bf_ctx* c, uint32_t handle, uint32_t n_runs, const uint32_t* runs, uint32_t n,
                                       bf_status_rec* records, uint16_t* events, uint64_t events_cap, uint64_t* n_events) {
  bf_status_out o;
  memset(&o, 0, sizeof o);
  o.struct_size = (uint32_t)sizeof o;
  o.records = records; o.events = events; o.events_cap = events_cap;
  const int rc = bf_resident_status(c, handle, n_runs, runs, n, &o);
  *n_events = o.n_events;
  return rc;
}

/* Resync.  The records, the run list and the outputs (bf_drift holds no pointers) are the caller's buffers; the counts and, on a
 * refusal that names a run, *bad_run come back through the pointers.  runs == NULL with n == n_runs lists every run of [0, n_runs). */
static inline int bfgo_resident_resync(bf_ctx* c, uint32_t handle, uint32_t n_runs, const uint32_t* runs, uint32_t n,
                                       const void* records, uint32_t fields, uint32_t flags, uint32_t* drifted, uint32_t drifted_cap,
                                       bf_drift* items, uint64_t items_cap, uint32_t* n_drifted, uint32_t* n_written,
                                       uint64_t* n_items, uint32_t* bad_run) {
  bf_resync q;
  memset(&q, 0, sizeof q);
  q.struct_size = (uint32_t)sizeof q;
  q.n_runs = n_runs; q.runs = runs; q.n = n; q.records = records; q.fields = fields; q.flags = flags;
  q.drifted = drifted; q.drifted_cap = drifted_cap; q.items = items; q.items_cap = items_cap;
  const int rc = bf_resident_resync(c, handle, &q);
  *n_drifted = q.n_drifted; *n_written = q.n_written; *n_items = q.n_items; *bad_run = q.bad_run;
  return rc;
}

/* Side-area resync.  The caller's rows of each area in `areas` (bf_timer_slot, bf_sched_put, bf_run_ctl: no pointers), the run
 * list and the outputs are the caller's buffers; the counts and, on a refusal that names a run, *bad_run come back through the
 * pointers. */
static inline int bfgo_resident_resync_areas(bf_ctx* c, uint32_t handle, uint32_t n_runs, const uint32_t* runs, uint32_t n,
                                             uint32_t areas, const bf_timer_slot* timers, const bf_sched_put* sched,
                                             const bf_run_ctl* runctl, uint32_t fired_now, uint32_t flags, uint32_t* drifted,
                                             uint32_t drifted_cap, bf_drift* items, uint64_t items_cap, uint32_t* n_drifted,
                                             uint32_t* n_written, uint64_t* n_items, uint32_t* bad_run) {
  bf_resync_areas q;
  memset(&q, 0, sizeof q);
  q.struct_size = (uint32_t)sizeof q;
  q.n_runs = n_runs; q.runs = runs; q.n = n; q.areas = areas; q.flags = flags; q.fired_now = fired_now;
  q.timers = timers; q.sched = sched; q.runctl = runctl;
  q.drifted = drifted; q.drifted_cap = drifted_cap; q.items = items; q.items_cap = items_cap;
  const int rc = bf_resident_resync_areas(c, handle, &q);
  *n_drifted = q.n_drifted; *n_written = q.n_written; *n_items = q.n_items; *bad_run = q.bad_run;
  return rc;
}

/* Step timings of a topology slot (bf_step_timing holds no pointers): passed as they are. */
static inline int bfgo_topology_timings(bf_ctx* c, uint32_t slot, const bf_step_timing* t, uint32_t n) {
  return bf_topology_timings(c, slot, t, n);
}

static inline void bfgo_tables(bf_sched_tables* t, uint32_t n_stories, uint32_t n_queues, int32_t global_limit, uint32_t global_base,
                               const int32_t* story_limit, const uint32_t* story_base, const int32_t* queue_limit,
                               const int32_t* queue_aging_s, const uint32_t* queue_base, const int32_t* queue_max_priority_base) {
  memset(t, 0, sizeof *t);
  t->struct_size = (uint32_t)sizeof *t;
  t->n_stories = n_stories; t->n_queues = n_queues; t->global_limit = global_limit; t->global_running_base = global_base;
  t->story_limit = story_limit; t->story_running_base = story_base; t->queue_limit = queue_limit; t->queue_aging_s = queue_aging_s;
  t->queue_running_base = queue_base; t->queue_max_priority_base = queue_max_priority_base;
}

static inline void bfgo_sched_out(bf_sched_out* o, void* records, uint32_t* story_running, uint32_t* queue_running,
                                  int32_t* queue_max_priority, uint32_t* global_running) {
  memset(o, 0, sizeof *o);
  o->struct_size = (uint32_t)sizeof *o;
  o->records = records; o->story_running = story_running; o->queue_running = queue_running;
  o->queue_max_priority = queue_max_priority; o->global_running = global_running;
}

static inline int bfgo_schedule(bf_ctx* c, const bf_layout* L, uint32_t n_runs, const bf_sched_run* runs, uint32_t n_stories,
                                uint32_t n_queues, int32_t global_limit, uint32_t global_base, const int32_t* story_limit,
                                const uint32_t* story_base, const int32_t* queue_limit, const int32_t* queue_aging_s,
                                const uint32_t* queue_base, const int32_t* queue_max_priority_base, void* records,
                                uint32_t* story_running, uint32_t* queue_running, int32_t* queue_max_priority, uint32_t* global_running) {
  bf_batch b;
  bf_sched_tables t;
  bf_sched_out o;
  bfgo_batch(&b, L, n_runs, 0, 0, NULL, NULL, NULL);
  bfgo_tables(&t, n_stories, n_queues, global_limit, global_base, story_limit, story_base, queue_limit, queue_aging_s, queue_base,
              queue_max_priority_base);
  bfgo_sched_out(&o, records, story_running, queue_running, queue_max_priority, global_running);
  return bf_schedule(c, &b, runs, &t, &o);
}

/* Resident limiters.  bf_resident_sched, _sched_put and _sched_download are called directly (flat arguments already); a part of
 * bf_resident_schedule is filled here (its list buffers are C memory, pinned for the kernels to write them in place), and the call
 * takes the tables flat as bfgo_schedule does. */
static inline void bfgo_sched_part(bf_resident_sched_part* p, uint32_t handle, uint32_t n_runs, uint32_t* runs, bf_sched_header* heads,
                                   uint32_t runs_cap, uint16_t* events, uint64_t events_cap) {
  memset(p, 0, sizeof *p);
  p->struct_size = (uint32_t)sizeof *p;
  p->handle = handle; p->n_runs = n_runs;
  p->runs = runs; p->heads = heads; p->runs_cap = runs_cap; p->events = events; p->events_cap = events_cap;
}

static inline int bfgo_resident_schedule(bf_ctx* c, uint32_t now, uint32_t n_stories, uint32_t n_queues, int32_t global_limit,
                                         uint32_t global_base, const int32_t* story_limit, const uint32_t* story_base,
                                         const int32_t* queue_limit, const int32_t* queue_aging_s, const uint32_t* queue_base,
                                         const int32_t* queue_max_priority_base, bf_resident_sched_part* parts, uint32_t n_parts,
                                         uint32_t* story_running, uint32_t* queue_running, int32_t* queue_max_priority,
                                         uint32_t* global_running) {
  bf_sched_tables t;
  bf_sched_out o;
  bfgo_tables(&t, n_stories, n_queues, global_limit, global_base, story_limit, story_base, queue_limit, queue_aging_s, queue_base,
              queue_max_priority_base);
  bfgo_sched_out(&o, NULL, story_running, queue_running, queue_max_priority, global_running);
  return bf_resident_schedule(c, &t, now, parts, n_parts, &o);
}

/* bf_resident_schedule_ctxs: part i is parts[i] (filled by bfgo_sched_part) of a batch of ctxs[i]; the bf_ctx_sched_part array
 * that points at them is built here in C memory, so the Go side passes only C pointers. */
static inline int bfgo_resident_schedule_ctxs(uint32_t now, uint32_t n_stories, uint32_t n_queues, int32_t global_limit,
                                              uint32_t global_base, const int32_t* story_limit, const uint32_t* story_base,
                                              const int32_t* queue_limit, const int32_t* queue_aging_s, const uint32_t* queue_base,
                                              const int32_t* queue_max_priority_base, bf_ctx* const* ctxs,
                                              bf_resident_sched_part* parts, uint32_t n_parts, uint32_t* story_running,
                                              uint32_t* queue_running, int32_t* queue_max_priority, uint32_t* global_running) {
  bf_sched_tables t;
  bf_sched_out o;
  bfgo_tables(&t, n_stories, n_queues, global_limit, global_base, story_limit, story_base, queue_limit, queue_aging_s, queue_base,
              queue_max_priority_base);
  bfgo_sched_out(&o, NULL, story_running, queue_running, queue_max_priority, global_running);
  bf_ctx_sched_part* cp = (bf_ctx_sched_part*)calloc(n_parts ? n_parts : 1, sizeof *cp);
  if (!cp) return BF_ENOMEM;
  for (uint32_t i = 0; i < n_parts; ++i) {
    cp[i].struct_size = (uint32_t)sizeof *cp;
    cp[i].ctx = ctxs[i];
    cp[i].part = &parts[i];
  }
  const int rc = bf_resident_schedule_ctxs(&t, now, cp, n_parts, &o);
  free(cp);
  return rc;
}

static inline int bfgo_group_eval(bf_group* g, const bf_layout* L, uint32_t n_runs, uint32_t flags, uint32_t max_iterations,
                                  const void* state, void* result, bf_counts* shard_counts, bf_counts* global_counts) {
  bf_batch b;
  bfgo_batch(&b, L, n_runs, flags, max_iterations, state, result, global_counts);
  return bf_group_eval(g, &b, shard_counts);
}

static inline int bfgo_group_schedule(bf_group* g, const bf_layout* L, uint32_t n_runs, const bf_sched_run* runs, uint32_t n_stories,
                                      uint32_t n_queues, int32_t global_limit, uint32_t global_base, const int32_t* story_limit,
                                      const uint32_t* story_base, const int32_t* queue_limit, const int32_t* queue_aging_s,
                                      const uint32_t* queue_base, const int32_t* queue_max_priority_base, void* records,
                                      uint32_t* story_running, uint32_t* queue_running, int32_t* queue_max_priority,
                                      uint32_t* global_running) {
  bf_batch b;
  bf_sched_tables t;
  bf_sched_out o;
  bfgo_batch(&b, L, n_runs, 0, 0, NULL, NULL, NULL);
  bfgo_tables(&t, n_stories, n_queues, global_limit, global_base, story_limit, story_base, queue_limit, queue_aging_s, queue_base,
              queue_max_priority_base);
  bfgo_sched_out(&o, records, story_running, queue_running, queue_max_priority, global_running);
  return bf_group_schedule(g, &b, runs, &t, &o);
}

#endif /* BOBRAFRONTIER_GO_SHIM_H_ */
