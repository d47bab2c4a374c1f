/*
 * c_resync_harness.c — plain C caller of libbobrafrontier.so that performs the per-tick loop of the cgo binding
 * (go/frontier/frontier.go) through the same entry points and flat wrappers (go/frontier/shim.h) up to a resync check:
 * Resident.Fire -> TickTouched -> Ctx.ScheduleResident -> (Execute) -> Resident.Commit -> Resident.Status, then the records a
 * batcher packs from the cluster -> Resident.Resync(ResyncCheck) lists nothing; one lost event later Resync repairs that run and
 * the next TickTouched evaluates and lists it alone.  The Story: A (engram), B (sleep), C (engram) needs B.
 *   run 0: A Succeeded, B Paused with its timer due: Fire writes SUCCEED, the pass syncs B to Succeeded and C launches.  The
 *          device keeps B Paused with decision SUCCEED; the cluster has B Succeeded and no decision.
 *   run 1: fail-fast, A Failed: the pass skips B and C, which the device never stores; the cluster has them Skipped.
 *   run 2: nothing yet: A and B launch (Running, Paused).
 *   run 3: every step Succeeded.
 * A touched tick after the commit evaluates the runs it wrote, as the next round of the loop does.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_resync_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_resync_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 4, S = 3, CAP_EV = 64, CAP_ITEMS = 64 };

static void set_code(uint8_t* rec, uint32_t off, uint32_t words, uint32_t nbits, uint32_t step, uint32_t code) {
  uint32_t* pl = (uint32_t*)(rec + off);
  for (uint32_t b = 0; b < nbits; ++b) {
    uint32_t* w = &pl[b * words + step / 32];
    *w = ((code >> b) & 1u) ? (*w | (1u << (step % 32))) : (*w & ~(1u << (step % 32)));
  }
}

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  const uint32_t rp[S + 1] = {0, 0, 0, 1};
  const uint16_t ci[1] = {1};
  const uint8_t fl[S] = {BF_STEP_ENGRAM, BF_STEP_SLEEP, BF_STEP_ENGRAM};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, S, 1, rp, ci, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  bf_layout L;
  CHECK(bf_layout_init(&L, 32, 0, BF_F_DECISION | BF_F_OUT_FAIL | BF_F_OUT_PHASE) == BF_OK);
  uint8_t* rec = (uint8_t*)calloc(N, L.state_stride);
  const uint32_t codes[N][S] = {{BF_PHASE_SUCCEEDED, BF_PHASE_PAUSED, 0},
                                {BF_PHASE_FAILED, 0, 0},
                                {0, 0, 0},
                                {BF_PHASE_SUCCEEDED, BF_PHASE_SUCCEEDED, BF_PHASE_SUCCEEDED}};
  for (uint32_t r = 0; r < N; ++r) {
    uint8_t* x = rec + (size_t)r * L.state_stride;
    ((bf_run_header*)x)->topo_slot = slot;
    ((bf_run_header*)x)->run_flags = r == 1 ? BF_RF_FAIL_FAST : 0;
    for (uint32_t s = 0; s < S; ++s) set_code(x, L.off_phase, L.words, 4, s, codes[r][s]);
  }
  uint32_t h;
  CHECK(bf_resident_create(ctx, &L, N, &h) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, rec) == BF_OK);
  CHECK(bf_resident_timers(ctx, h, 1) == BF_OK);                                      /* EnableTimers */
  bf_timer t;
  memset(&t, 0, sizeof t);
  t.run = 0; t.step = 1; t.code = BF_DEC_SUCCEED; t.deadline = 0;
  CHECK(bf_resident_timers_arm(ctx, h, &t, 1) == BF_OK);                              /* ArmTimers */
  CHECK(bf_resident_sched(ctx, h) == BF_OK);                                          /* EnableSched */
  bf_sched_put put[N];
  memset(put, 0, sizeof put);
  for (uint32_t r = 0; r < N; ++r) {
    put[r].run = r; put[r].story_key = BF_SCHED_NONE; put[r].queue_key = BF_SCHED_NONE;
    put[r].queued_since = BF_SCHED_NONE; put[r].run_phase = BF_PHASE_RUNNING;
  }
  CHECK(bf_resident_sched_put(ctx, h, put, N) == BF_OK);

  /* Fire -> TickTouched -> ScheduleResident -> Commit -> Status */
  bf_fired fired[4];
  uint32_t fc[5];
  CHECK(bfgo_resident_fire(ctx, h, N, 1, fired, 4, fc) == BF_OK && fc[0] == 1 && fc[1] == 1);
  uint32_t runs_t[N], head_t[N], full, n_listed, n_eval;
  uint16_t ev_t[CAP_EV];
  uint64_t n_ev;
  bf_counts k;
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, CAP_EV, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  CHECK(full == 1 && n_listed == N && k.ready == 3);   /* C of run 0, A and B of run 2 */
  uint32_t* runs;
  bf_sched_header* heads;
  uint16_t* events;
  CHECK(bf_alloc_pinned(ctx, N * sizeof(uint32_t), (void**)&runs) == BF_OK);
  CHECK(bf_alloc_pinned(ctx, N * sizeof(bf_sched_header), (void**)&heads) == BF_OK);
  CHECK(bf_alloc_pinned(ctx, CAP_EV * sizeof(uint16_t), (void**)&events) == BF_OK);
  bf_resident_sched_part part;
  bfgo_sched_part(&part, h, N, runs, heads, N, events, CAP_EV);
  const int32_t sl[1] = {0};
  uint32_t sr[1], gr;
  CHECK(bfgo_resident_schedule(ctx, 1, 1, 0, 0, 0, sl, NULL, NULL, NULL, NULL, NULL, &part, 1, sr, NULL, NULL, &gr) == BF_OK);
  uint32_t c[7];
  CHECK(bfgo_resident_commit(ctx, h, N, NULL, 0, c) == BF_OK && c[0] == 2 && c[2] == 3);
  bf_status_rec st[N];
  uint16_t sev[CAP_EV];
  uint64_t n_sev = 0;
  CHECK(bfgo_resident_status(ctx, h, N, NULL, N, st, sev, CAP_EV, &n_sev) == BF_OK);
  CHECK(st[0].completed == 2 && st[0].active == 1);                                    /* B synced: Succeeded */
  CHECK(st[1].outcome == BF_OUTCOME_DEPENDENCY_FAILED && st[1].skipped == 2);          /* B, C skipped by fail-fast */
  CHECK(st[3].outcome == BF_OUTCOME_SUCCEEDED);
  /* the next tick evaluates the runs the commit wrote (0 and 2); nothing else is touched afterwards */
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, CAP_EV, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  CHECK(full == 0 && n_eval == 2);

  /* What the batcher persisted, packed as it packs new runs: the phases after the rewrites, no decision on a terminal step */
  uint8_t* dev = (uint8_t*)malloc((size_t)N * L.state_stride);
  uint8_t* view = (uint8_t*)malloc((size_t)N * L.state_stride);
  CHECK(bf_resident_download(ctx, h, 0, N, dev) == BF_OK);
  memcpy(view, dev, (size_t)N * L.state_stride);
  uint8_t* v0 = view;
  uint8_t* v1 = view + L.state_stride;
  set_code(v0, L.off_phase, L.words, 4, 1, BF_PHASE_SUCCEEDED);
  set_code(v0, L.off_decision, L.words, 2, 1, BF_DEC_PENDING);
  set_code(v1, L.off_phase, L.words, 4, 1, BF_PHASE_SKIPPED);
  set_code(v1, L.off_phase, L.words, 4, 2, BF_PHASE_SKIPPED);
  CHECK(memcmp(view, dev, (size_t)N * L.state_stride) != 0);
  uint32_t drifted[N], n_drifted, n_written, bad_run;
  bf_drift items[CAP_ITEMS];
  uint64_t n_items;
  CHECK(bfgo_resident_resync(ctx, h, N, NULL, N, view, BF_RESYNC_ALL_FIELDS, BF_RESYNC_CHECK, drifted, N, items, CAP_ITEMS,
                             &n_drifted, &n_written, &n_items, &bad_run) == BF_OK);
  CHECK(n_items == 0 && n_drifted == 0 && n_written == 0 && bad_run == BF_RESYNC_NONE);

  /* A lost watch event: run 2's A Succeeded in the cluster, Running here.  The resync lists and repairs run 2 alone */
  uint8_t* v2 = view + 2 * (size_t)L.state_stride;
  set_code(v2, L.off_phase, L.words, 4, 0, BF_PHASE_SUCCEEDED);
  CHECK(bfgo_resident_resync(ctx, h, N, NULL, N, view, BF_RESYNC_ALL_FIELDS, 0, drifted, N, items, CAP_ITEMS, &n_drifted,
                             &n_written, &n_items, &bad_run) == BF_OK);
  CHECK(n_drifted == 1 && n_written == 1 && drifted[0] == 2 && n_items == 1);
  CHECK(items[0].run == 2 && items[0].index == 0 && items[0].field == BF_DELTA_PHASE && items[0].device == BF_PHASE_RUNNING &&
        items[0].record == BF_PHASE_SUCCEEDED);
  CHECK(bf_resident_download(ctx, h, 0, N, dev) == BF_OK);
  CHECK(memcmp(dev + 2 * (size_t)L.state_stride, v2, L.state_stride) == 0);
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, CAP_EV, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  CHECK(full == 0 && n_eval == 1 && n_listed == 1 && runs_t[0] == 2);
  /* a record naming a slot no put has returned is refused and names its run */
  ((bf_run_header*)v1)->topo_slot = 4000;
  CHECK(bfgo_resident_resync(ctx, h, N, NULL, N, view, BF_RESYNC_ALL_FIELDS, 0, drifted, N, items, CAP_ITEMS, &n_drifted,
                             &n_written, &n_items, &bad_run) == BF_EINVAL && bad_run == 1);

  free(dev);
  free(view);
  CHECK(bf_free_pinned(ctx, runs) == BF_OK && bf_free_pinned(ctx, heads) == BF_OK && bf_free_pinned(ctx, events) == BF_OK);
  CHECK(bf_resident_destroy(ctx, h) == BF_OK);
  free(rec);
  bf_destroy(ctx);
  printf("c_resync_harness: ok\n");
  return 0;
}
