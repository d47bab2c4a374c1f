/*
 * c_commit_touched_harness.c — plain C caller of libbobrafrontier.so that performs the per-tick loop of the cgo binding with a
 * touched rewriting commit (go/frontier/frontier.go) through the same entry points and flat wrappers (go/frontier/shim.h):
 * Resident.EnableCommitMarks once, then Fire -> TickTouched -> Ctx.ScheduleResident -> (Execute) -> Resident.CommitTouched
 * (journal, rewrites) -> Status -> Resync check, twice.  The first commit considers both runs (the marks were just enabled), the
 * second only run 0, the one run the touched tick evaluated; run 1 keeps its writes in place and is not considered.
 * The Story: S (sleep, 1 unit), E (engram), F (engram) needs E.  Run 0 launches S and E at the first tick: the commit pauses S,
 * arms its timer and runs E.  At the second tick the timer fires, the pass's stage G turns S Succeeded, and the rewriting commit
 * stores that and lists it as a rewrite item, as bf_resident_commit_rewrites would.  Run 1 arrives with every step Succeeded.  After each commit the cluster view (the
 * uploaded records with every journal item applied, as a batcher persists them) resyncs without drift, and Status reports run 0.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_commit_touched_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_commit_touched_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 2, CAP_EV = 64, CAP_ITEMS = 16, NOW = 100 };

static uint32_t phase_of(const uint8_t* rec, const bf_layout* L, uint32_t step) {
  const uint32_t* ph = (const uint32_t*)(rec + L->off_phase);
  uint32_t code = 0;
  for (uint32_t b = 0; b < 4; ++b) code |= ((ph[b * L->words + step / 32] >> (step % 32)) & 1u) << b;
  return code;
}

static void set_phase(uint8_t* rec, const bf_layout* L, uint32_t step, uint32_t code) {
  uint32_t* ph = (uint32_t*)(rec + L->off_phase);
  for (uint32_t b = 0; b < 4; ++b) {
    uint32_t* w = &ph[b * L->words + step / 32];
    *w = ((code >> b) & 1u) ? *w | 1u << (step % 32) : *w & ~(1u << (step % 32));
  }
}

/* what the batcher persists of a journal: each PHASE item's code and each REGISTERED bit, into its copy of the records */
static void persist(uint8_t* view, const bf_layout* L, const bf_commit_write* items, uint64_t n) {
  for (uint64_t i = 0; i < n; ++i) {
    uint8_t* r = view + (size_t)items[i].run * L->state_stride;
    if (items[i].field == BF_DELTA_PHASE) set_phase(r, L, items[i].index, items[i].after);
    else if (items[i].field == BF_DELTA_REGISTERED) ((bf_run_header*)r)->children_registered |= 1ull << items[i].index;
  }
}

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  const uint32_t rp[4] = {0, 0, 0, 1};
  const uint16_t ci[1] = {1};
  const uint8_t fl[3] = {BF_STEP_SLEEP, BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, 3, 1, rp, ci, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  bf_step_timing tim;
  memset(&tim, 0, sizeof tim);
  tim.step = 0; tim.code = BF_DEC_SUCCEED; tim.delay = 1;
  CHECK(bfgo_topology_timings(ctx, slot, &tim, 1) == BF_OK);                          /* PutTimings */
  bf_layout L;
  CHECK(bf_layout_init(&L, 32, 0, BF_F_DECISION | BF_F_OUT_FAIL) == BF_OK);
  uint8_t* rec = (uint8_t*)calloc(N, L.state_stride);
  for (uint32_t r = 0; r < N; ++r) ((bf_run_header*)(rec + (size_t)r * L.state_stride))->topo_slot = slot;
  for (uint32_t s = 0; s < 3; ++s) set_phase(rec + (size_t)L.state_stride, &L, s, BF_PHASE_SUCCEEDED);
  uint32_t h;
  CHECK(bf_resident_create(ctx, &L, N, &h) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, rec) == BF_OK);
  CHECK(bf_resident_timers(ctx, h, 2) == BF_OK);                                      /* EnableTimers */
  CHECK(bf_resident_sched(ctx, h) == BF_OK);                                          /* EnableSched */
  CHECK(bf_resident_commit_marks(ctx, h) == BF_OK);                                   /* EnableCommitMarks */
  bf_sched_put put[N];
  memset(put, 0, sizeof put);
  for (uint32_t r = 0; r < N; ++r) {
    put[r].run = r; put[r].story_key = BF_SCHED_NONE; put[r].queue_key = BF_SCHED_NONE;
    put[r].queued_since = BF_SCHED_NONE; put[r].run_phase = BF_PHASE_RUNNING;
  }
  CHECK(bf_resident_sched_put(ctx, h, put, N) == BF_OK);
  uint32_t* runs;
  bf_sched_header* heads;
  uint16_t* events;
  CHECK(bf_alloc_pinned(ctx, N * sizeof(uint32_t), (void**)&runs) == BF_OK);
  CHECK(bf_alloc_pinned(ctx, N * sizeof(bf_sched_header), (void**)&heads) == BF_OK);
  CHECK(bf_alloc_pinned(ctx, CAP_EV * sizeof(uint16_t), (void**)&events) == BF_OK);
  uint8_t* view = (uint8_t*)malloc((size_t)N * L.state_stride);   /* the cluster's copy, from the journals */
  memcpy(view, rec, (size_t)N * L.state_stride);
  uint8_t* got = (uint8_t*)malloc((size_t)N * L.state_stride);

  for (uint32_t tick = 0; tick < 2; ++tick) {
    const uint32_t now = NOW + tick;
    /* Fire -> TickTouched -> ScheduleResident */
    bf_fired fired[8];
    uint32_t fc[5];
    CHECK(bfgo_resident_fire(ctx, h, N, now, fired, 8, fc) == BF_OK && fc[0] == tick);
    uint32_t runs_t[N], head_t[N], full, n_listed, n_eval;
    uint16_t ev_t[CAP_EV];
    uint64_t n_ev;
    bf_counts k;
    CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, CAP_EV, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
    if (tick == 1) CHECK(n_listed == 1 && runs_t[0] == 0 && (head_t[0] & BF_SUM_PHASE_CHANGED));   /* the fired sleep */
    bf_resident_sched_part part;
    bfgo_sched_part(&part, h, N, runs, heads, N, events, CAP_EV);
    uint32_t gr;
    CHECK(bfgo_resident_schedule(ctx, now, 0, 0, 0, 0, NULL, NULL, NULL, NULL, NULL, NULL, &part, 1, NULL, NULL, NULL, &gr) == BF_OK);

    /* CommitRewrites */
    bf_commit_write items[CAP_ITEMS];
    uint32_t written[N], c[13];
    uint64_t n_items = 99;
    CHECK(bfgo_resident_commit_touched(ctx, h, N, NULL, 0, now, BF_COMMIT_SCOPE_REWRITES, 1, items, CAP_ITEMS, written, N, c,
                                       &n_items) == BF_OK);
    CHECK(c[0] == 1 && c[9] == 1 && written[0] == 0);
    CHECK(tick ? (c[11] == 0 && c[12] == 1) : (c[11] == 1 && c[12] == N));   /* full once, then the evaluated run alone */
    if (tick == 0) {   /* the launch writes: S paused and armed, E running; nothing from the stages */
      CHECK(c[2] == 2 && c[7] == 1 && c[10] == 0 && n_items == 3);
      CHECK(items[0].index == 0 && items[0].after == BF_PHASE_PAUSED && items[0].code == 0);
      CHECK(items[1].index == 1 && items[1].after == BF_PHASE_RUNNING && items[1].code == 0);
      CHECK(items[2].field == BF_COMMIT_WRITE_TIMER && items[2].after == NOW + 1);
    } else {           /* stage G: the fired sleep is stored Succeeded, marked as a rewrite */
      CHECK(c[2] == 0 && c[10] == 1 && n_items == 1);
      CHECK(items[0].run == 0 && items[0].field == BF_DELTA_PHASE && items[0].index == 0 && items[0].code == BF_COMMIT_WRITE_REWRITE &&
            items[0].before == BF_PHASE_PAUSED && items[0].after == BF_PHASE_SUCCEEDED);
    }
    persist(view, &L, items, n_items);
    CHECK(bf_resident_download(ctx, h, 0, N, got) == BF_OK);
    CHECK(phase_of(got, &L, 0) == (tick ? BF_PHASE_SUCCEEDED : BF_PHASE_PAUSED) && phase_of(got, &L, 1) == BF_PHASE_RUNNING);

    /* Status over the written run */
    bf_status_rec st[1];
    uint16_t sev[CAP_EV];
    uint64_t n_sev;
    CHECK(bfgo_resident_status(ctx, h, N, written, 1, st, sev, CAP_EV, &n_sev) == BF_OK);
    CHECK(st[0].run == 0 && st[0].outcome == BF_OUTCOME_NONE && st[0].active == (tick ? 1 : 2) && st[0].completed == tick);

    /* Resync check of the cluster's copy: phases and registered bits, as persisted from the journals, list no drift */
    uint32_t drifted[N], n_drifted = 9, n_written = 9, bad = 0;
    bf_drift ditems[8];
    uint64_t n_ditems = 9;
    CHECK(bfgo_resident_resync(ctx, h, N, NULL, N, view, BF_RESYNC_FIELD(BF_DELTA_PHASE) | BF_RESYNC_FIELD(BF_DELTA_REGISTERED),
                               BF_RESYNC_CHECK, drifted, N, ditems, 8, &n_drifted, &n_written, &n_ditems, &bad) == BF_OK);
    CHECK(n_drifted == 0 && n_ditems == 0);
  }

  free(got);
  free(view);
  CHECK(bf_free_pinned(ctx, runs) == BF_OK && bf_free_pinned(ctx, heads) == BF_OK && bf_free_pinned(ctx, events) == BF_OK);
  CHECK(bf_resident_destroy(ctx, h) == BF_OK);
  free(rec);
  bf_destroy(ctx);
  printf("c_commit_touched_harness: ok\n");
  return 0;
}
