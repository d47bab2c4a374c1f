/*
 * c_status_harness.c — plain C caller of libbobrafrontier.so that performs the per-tick loop of the cgo binding
 * (go/frontier/frontier.go) through the same entry points and flat wrappers (go/frontier/shim.h) up to the status a batcher
 * persists: Resident.Fire -> TickTouched -> Ctx.ScheduleResident -> (Execute) -> Resident.Commit -> Resident.Status (the runs
 * the tick listed as done, and the runs the commit wrote) -> Resident.Retire of the finished runs.  The Story: A (engram,
 * allowFailure), B (engram), C (engram) needs B; every run fail-fast.  Run 0 has A Failed, B and C Succeeded: finished,
 * Succeeded, A an allowed failure.  Run 1 has A Succeeded, B Failed: fail-fast skips C, finished, DependencyFailed naming B.
 * Run 2 has nothing yet (A and B launch), run 3 has A and B Succeeded (C launches).  After the retire the two live runs report
 * under their new indices.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_status_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_status_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 4, S = 3, CAP_EV = 64 };

static void set_phase(uint8_t* rec, const bf_layout* L, uint32_t step, uint32_t code) {
  uint32_t* ph = (uint32_t*)(rec + L->off_phase);
  for (uint32_t b = 0; b < 4; ++b) {
    uint32_t* w = &ph[b * L->words + step / 32];
    *w = ((code >> b) & 1u) ? (*w | (1u << (step % 32))) : (*w & ~(1u << (step % 32)));
  }
}

static uint16_t event(uint32_t step, uint32_t phase, uint32_t kind) { return (uint16_t)(step | phase << 10 | kind << 14); }

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  const uint32_t rp[S + 1] = {0, 0, 0, 1};
  const uint16_t ci[1] = {1};
  const uint8_t fl[S] = {BF_STEP_ENGRAM | BF_SF_ALLOW_FAILURE, BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, S, 1, rp, ci, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  bf_layout L;
  CHECK(bf_layout_init(&L, 32, 0, BF_F_OUT_FAIL) == BF_OK);
  uint8_t* rec = (uint8_t*)calloc(N, L.state_stride);
  const uint32_t codes[N][S] = {{BF_PHASE_FAILED, BF_PHASE_SUCCEEDED, BF_PHASE_SUCCEEDED},
                                {BF_PHASE_SUCCEEDED, BF_PHASE_FAILED, 0},
                                {0, 0, 0},
                                {BF_PHASE_SUCCEEDED, BF_PHASE_SUCCEEDED, 0}};
  for (uint32_t r = 0; r < N; ++r) {
    uint8_t* x = rec + (size_t)r * L.state_stride;
    ((bf_run_header*)x)->topo_slot = slot;
    ((bf_run_header*)x)->run_flags = BF_RF_FAIL_FAST;
    for (uint32_t s = 0; s < S; ++s) set_phase(x, &L, s, codes[r][s]);
  }
  uint32_t h;
  CHECK(bf_resident_create(ctx, &L, N, &h) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, rec) == BF_OK);
  CHECK(bf_resident_timers(ctx, h, 1) == BF_OK);                                      /* EnableTimers */
  CHECK(bf_resident_sched(ctx, h) == BF_OK);                                          /* EnableSched */
  bf_sched_put put[N];
  memset(put, 0, sizeof put);
  for (uint32_t r = 0; r < N; ++r) {
    put[r].run = r; put[r].story_key = BF_SCHED_NONE; put[r].queue_key = BF_SCHED_NONE;
    put[r].queued_since = BF_SCHED_NONE; put[r].run_phase = BF_PHASE_RUNNING;
  }
  CHECK(bf_resident_sched_put(ctx, h, put, N) == BF_OK);

  /* Fire -> TickTouched -> ScheduleResident -> Commit */
  bf_fired fired[4];
  uint32_t fc[5];
  CHECK(bfgo_resident_fire(ctx, h, N, 1, fired, 4, fc) == BF_OK && fc[0] == 0);
  uint32_t runs_t[N], head_t[N], full, n_listed, n_eval;
  uint16_t ev_t[CAP_EV];
  uint64_t n_ev;
  bf_counts k;
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, CAP_EV, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  CHECK(full == 1 && n_listed == N && k.ready == 3);
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

  /* Status: the runs the tick listed as done (0 and 1) and the runs the commit wrote (2 and 3), ascending */
  uint32_t list[N];
  uint32_t n_list = 0;
  for (uint32_t i = 0; i < n_listed; ++i)
    if ((head_t[i] & BF_SUM_GROUP_MASK) == BF_GROUP_DONE) list[n_list++] = runs_t[i];
  CHECK(n_list == 2 && list[0] == 0 && list[1] == 1);
  list[n_list++] = 2;
  list[n_list++] = 3;
  uint8_t* before = (uint8_t*)malloc((size_t)N * L.state_stride);
  uint8_t* after = (uint8_t*)malloc((size_t)N * L.state_stride);
  CHECK(bf_resident_download(ctx, h, 0, N, before) == BF_OK);
  bf_status_rec st[N];
  uint16_t sev[CAP_EV];
  uint64_t n_sev = 0;
  CHECK(bfgo_resident_status(ctx, h, N, list, n_list, st, sev, CAP_EV, &n_sev) == BF_OK);
  CHECK(bf_resident_download(ctx, h, 0, N, after) == BF_OK && memcmp(before, after, (size_t)N * L.state_stride) == 0);
  CHECK(n_sev == 2);
  CHECK(st[0].run == 0 && st[0].group == BF_GROUP_DONE && st[0].outcome == BF_OUTCOME_SUCCEEDED && st[0].story_phase == BF_PHASE_SUCCEEDED);
  CHECK(st[0].first_failed == BF_STATUS_NO_STEP && st[0].completed == 2 && st[0].failed == 1 && st[0].n_events == 1);
  CHECK(sev[st[0].first_event] == event(0, BF_PHASE_FAILED, BF_STATUS_EVT_ALLOWED));
  CHECK(st[1].run == 1 && st[1].outcome == BF_OUTCOME_DEPENDENCY_FAILED && st[1].story_phase == BF_PHASE_FAILED && st[1].first_failed == 1);
  CHECK(st[1].completed == 1 && st[1].failed == 1 && st[1].skipped == 1 && st[1].n_events == 1);
  CHECK(sev[st[1].first_event] == event(1, BF_PHASE_FAILED, BF_STATUS_EVT_FAILED));
  CHECK(st[2].outcome == BF_OUTCOME_NONE && st[2].group == BF_GROUP_MAIN && st[2].active == 2 && st[2].n_events == 0);
  CHECK(st[3].outcome == BF_OUTCOME_NONE && st[3].active == 1 && st[3].completed == 2 && st[3].n_events == 0);
  /* a list that does not ascend is refused */
  const uint32_t bad[2] = {3, 1};
  CHECK(bfgo_resident_status(ctx, h, N, bad, 2, st, sev, CAP_EV, &n_sev) == BF_EINVAL);

  /* Retire the finished runs; the live ones report under their new indices */
  uint32_t from[2], to[2], n_after, n_moves;
  CHECK(bfgo_resident_retire(ctx, h, N, list, 2, 0, from, to, &n_after, &n_moves) == BF_OK && n_after == 2);
  CHECK(bfgo_resident_status(ctx, h, n_after, NULL, n_after, st, sev, 0, &n_sev) == BF_OK && n_sev == 0);
  for (uint32_t i = 0; i < n_moves; ++i) {
    const bf_status_rec* m = &st[to[i]];
    CHECK(m->run == to[i] && m->outcome == BF_OUTCOME_NONE && m->active == (from[i] == 2 ? 2 : 1));
  }
  CHECK(n_moves == 2);

  free(before);
  free(after);
  CHECK(bf_free_pinned(ctx, runs) == BF_OK && bf_free_pinned(ctx, heads) == BF_OK && bf_free_pinned(ctx, events) == BF_OK);
  CHECK(bf_resident_destroy(ctx, h) == BF_OK);
  free(rec);
  bf_destroy(ctx);
  printf("c_status_harness: ok\n");
  return 0;
}
