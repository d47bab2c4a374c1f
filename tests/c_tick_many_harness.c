/*
 * c_tick_many_harness.c — plain C caller of libbobrafrontier.so that performs the per-tick loop of INTEGRATION.md step 5 over
 * three width-class batches (32, 512 and 1024 steps) with the flat wrappers of go/frontier/shim.h, as Ctx.TickTouched in the
 * cgo binding (go/frontier/frontier.go) calls them: Fire on each batch -> one bf_resident_tick_touched_many over all three ->
 * one ScheduleResident over all three -> Commit on each.  Every run holds one Story of two independent engram steps.  The first
 * tick is full and lists both steps of every run as ready; the commit launches them, so the next tick lists every run again with
 * no events; a delta on one run of the widest batch is then the only thing listed.  A repeated handle is refused, naming the part.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_tick_many_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_tick_many_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 4, B = 3, EV = 64 };

static bf_ctx* ctx = NULL;
static uint32_t h[B];
static uint32_t runs[B * N], head[B * N], full[B], n_listed[B], n_eval[B];
static uint16_t events[B * EV];
static uint64_t n_ev[B];
static bf_counts counts[B];

/* Fire on each batch, then the touched ticks of all three in one call; part b's deltas are d[dfirst[b] .. dfirst[b + 1]) */
static int tick(const bf_delta* d, const uint32_t* dfirst, uint32_t* bad) {
  uint32_t fc[5];
  bf_fired fired[4];
  for (int b = 0; b < B; ++b)
    if (bfgo_resident_fire(ctx, h[b], N, 100, fired, 4, fc) != BF_OK) return -1;
  const uint32_t nr[B] = {N, N, N}, rf[B + 1] = {0, N, 2 * N, 3 * N};
  const uint64_t ef[B + 1] = {0, EV, 2 * EV, 3 * EV};
  return bfgo_resident_tick_touched_many(ctx, 0, 0, B, h, nr, d, dfirst, runs, head, rf, events, ef, full, n_listed, n_eval, n_ev,
                                         counts, bad);
}

/* one ScheduleResident over the three batches, then Commit on each: every ready step launches (no limits) */
static int schedule_and_commit(void) {
  static uint32_t sr[B][N];
  static bf_sched_header sh[B][N];
  static uint16_t se[B][EV];
  bf_resident_sched_part parts[B];
  for (int b = 0; b < B; ++b) bfgo_sched_part(&parts[b], h[b], N, sr[b], sh[b], N, se[b], EV);
  uint32_t gr;
  if (bfgo_resident_schedule(ctx, 100, 0, 0, 0, 0, NULL, NULL, NULL, NULL, NULL, NULL, parts, B, NULL, NULL, NULL, &gr) != BF_OK) return -1;
  for (int b = 0; b < B; ++b) {
    uint32_t cc[7];
    if (bfgo_resident_commit(ctx, h[b], N, NULL, 0, cc) != BF_OK || cc[2] == 0) return -1;
  }
  return 0;
}

int main(void) {
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  const uint32_t rp[3] = {0, 0, 0};
  const uint8_t fl[2] = {BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, 2, 0, rp, NULL, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  const uint32_t widths[B] = {32, 512, 1024};
  for (int b = 0; b < B; ++b) {
    bf_layout L;
    CHECK(bf_layout_init(&L, widths[b], 0, b == 1 ? BF_F_COND | BF_F_DECISION | BF_F_OUT_FAIL : 0) == BF_OK);
    uint8_t* rec = (uint8_t*)calloc(N, L.state_stride);
    for (uint32_t r = 0; r < N; ++r) ((bf_run_header*)(rec + (size_t)r * L.state_stride))->topo_slot = slot;
    CHECK(bf_resident_create(ctx, &L, N, &h[b]) == BF_OK);
    CHECK(bf_resident_upload(ctx, h[b], 0, N, rec) == BF_OK);
    CHECK(bf_resident_runctl(ctx, h[b]) == BF_OK);                                    /* EnableRunCtl: Fire's deadlines */
    CHECK(bf_resident_sched(ctx, h[b]) == BF_OK);                                     /* EnableSched */
    bf_sched_put put[N];
    memset(put, 0, sizeof put);
    for (uint32_t r = 0; r < N; ++r) {
      put[r].run = r; put[r].story_key = BF_SCHED_NONE; put[r].queue_key = BF_SCHED_NONE;
      put[r].queued_since = BF_SCHED_NONE; put[r].run_phase = BF_PHASE_RUNNING;
    }
    CHECK(bf_resident_sched_put(ctx, h[b], put, N) == BF_OK);
    free(rec);
  }
  const uint32_t none[B + 1] = {0, 0, 0, 0};
  uint32_t bad = 0;
  /* tick 1: full, both steps of every run ready */
  CHECK(tick(NULL, none, &bad) == BF_OK && bad == BF_COMMIT_NONE);
  for (int b = 0; b < B; ++b) {
    CHECK(full[b] == 1 && n_listed[b] == N && n_ev[b] == 2 * N && counts[b].ready == 2 * N);
    CHECK(runs[b * N + 3] == 3 && (head[b * N] >> BF_HEAD_COUNT_SHIFT) == 2);
    CHECK(events[b * EV] == (0 | BF_EVT_READY << 10) && events[b * EV + 1] == (1 | BF_EVT_READY << 10));
  }
  CHECK(schedule_and_commit() == 0);
  /* tick 2: the commit wrote every run (both steps launched): every run evaluated and listed, nothing ready */
  CHECK(tick(NULL, none, &bad) == BF_OK);
  for (int b = 0; b < B; ++b) CHECK(full[b] == 0 && n_eval[b] == N && n_listed[b] == N && n_ev[b] == 0);
  /* tick 3: step 0 of run 2 of the widest batch back to not started (code 0): that run alone is listed, step 0 ready again */
  bf_delta d;
  memset(&d, 0, sizeof d);
  d.run = 2; d.index = 0; d.field = BF_DELTA_PHASE; d.code = 0;
  const uint32_t df[B + 1] = {0, 0, 0, 1};
  CHECK(tick(&d, df, &bad) == BF_OK);
  CHECK(n_eval[0] == 0 && n_eval[1] == 0 && n_listed[0] == 0 && n_listed[1] == 0);
  CHECK(n_eval[2] == 1 && n_listed[2] == 1 && runs[2 * N] == 2 && n_ev[2] == 1 && events[2 * EV] == (0 | BF_EVT_READY << 10));
  /* one batch named twice: refused before anything runs, naming the second part */
  const uint32_t twice[B] = {h[0], h[1], h[0]}, nr[B] = {N, N, N}, rf[B + 1] = {0, N, 2 * N, 3 * N};
  const uint64_t ef[B + 1] = {0, EV, 2 * EV, 3 * EV};
  CHECK(bfgo_resident_tick_touched_many(ctx, 0, 0, B, twice, nr, NULL, none, runs, head, rf, events, ef, full, n_listed, n_eval, n_ev,
                                        counts, &bad) == BF_EINVAL && bad == 2);
  for (int b = 0; b < B; ++b) CHECK(bf_resident_destroy(ctx, h[b]) == BF_OK);
  bf_destroy(ctx);
  printf("c_tick_many_harness: ok\n");
  return 0;
}
