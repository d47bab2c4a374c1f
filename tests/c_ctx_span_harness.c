/*
 * c_ctx_span_harness.c — plain C caller of libbobrafrontier.so that performs the per-tick loop of INTEGRATION.md step 9 over two
 * ctxs with the flat wrappers of go/frontier/shim.h, as the cgo binding (go/frontier/frontier.go) calls them: Fire on each batch
 * -> TickTouched per ctx -> one ScheduleResidentCtxs over both -> Commit on each -> TickTouched per ctx -> TransferToCtx from
 * one ctx to the other -> TickTouched per ctx.  Each ctx holds one batch of N runs of one Story of two independent engram steps, step 0 Running; the
 * Story sits at slot 1 of ctx 0 (a filler Story takes slot 0) and at slot 0 of ctx 1, so the slot map is not the identity.
 * The span schedule counts the Running steps of both ctxs (2N for the Story and in all); a Story limit of 2N + 1 leaves each
 * run one slot, which its one ready step takes.  The transfer moves runs 0 and 2 with their slot mapped, and an unmapped slot
 * is refused with nothing changed.  Both ctxs live on device 0, or on devices 0 and 1 when two are visible.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_ctx_span_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                                                                   \
  do {                                                                                                                                \
    if (!(cond)) {                                                                                                                    \
      fprintf(stderr, "c_ctx_span_harness: FAILED %s (line %d): %s | %s\n", #cond, __LINE__, ctx[0] ? bf_last_error(ctx[0]) : "",  \
              ctx[1] ? bf_last_error(ctx[1]) : "");                                                                                   \
      return 1;                                                                                                                       \
    }                                                                                                                                 \
  } while (0)

enum { N = 4, CAP = 8, EV = 64 };

static bf_ctx* ctx[2] = {NULL, NULL};
static uint32_t h[2], n_runs[2] = {N, N};
static uint32_t runs[CAP], head[CAP], full, n_listed, n_eval;
static uint16_t events[EV];
static uint64_t n_ev;
static bf_counts counts;
static bf_layout L;

/* Fire, then the touched tick of ctx k's batch (TickTouched with one part) */
static int tick(int k) {
  uint32_t fc[5], bad = 0;
  bf_fired fired[4];
  if (bfgo_resident_fire(ctx[k], h[k], n_runs[k], 100, fired, 4, fc) != BF_OK) return -1;
  const uint32_t none[2] = {0, 0}, rf[2] = {0, CAP};
  const uint64_t ef[2] = {0, EV};
  return bfgo_resident_tick_touched_many(ctx[k], 0, 0, 1, &h[k], &n_runs[k], NULL, none, runs, head, rf, events, ef, &full, &n_listed,
                                         &n_eval, &n_ev, &counts, &bad);
}

int main(void) {
  CHECK(bfgo_create(0, &ctx[0]) == BF_OK);
  if (bfgo_create(1, &ctx[1]) != BF_OK) CHECK(bfgo_create(0, &ctx[1]) == BF_OK);   /* a second device when there is one */
  const uint32_t rp[3] = {0, 0, 0}, rp1[2] = {0, 0};
  const uint8_t fl[2] = {BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t filler = 99, slot[2] = {99, 99};
  CHECK(bfgo_topology_put(ctx[0], 1, 0, rp1, NULL, fl, NULL, 0, NULL, 0, &filler) == BF_OK);
  CHECK(bfgo_topology_put(ctx[0], 2, 0, rp, NULL, fl, NULL, 0, NULL, 0, &slot[0]) == BF_OK);
  CHECK(bfgo_topology_put(ctx[1], 2, 0, rp, NULL, fl, NULL, 0, NULL, 0, &slot[1]) == BF_OK);
  CHECK(filler == 0 && slot[0] == 1 && slot[1] == 0);
  CHECK(bf_layout_init(&L, 32, 0, 0) == BF_OK);
  uint8_t* rec = (uint8_t*)calloc(CAP, L.state_stride);
  for (int k = 0; k < 2; ++k) {
    for (uint32_t r = 0; r < N; ++r) {
      uint8_t* x = rec + (size_t)r * L.state_stride;
      ((bf_run_header*)x)->topo_slot = slot[k];
      ((uint32_t*)(x + L.off_phase))[1 * L.words] = 1u;   /* step 0: BF_PHASE_RUNNING (2), plane 1 */
    }
    CHECK(bf_resident_create(ctx[k], &L, CAP, &h[k]) == BF_OK);
    CHECK(bf_resident_upload(ctx[k], h[k], 0, N, rec) == BF_OK);
    CHECK(bf_resident_runctl(ctx[k], h[k]) == BF_OK);   /* EnableRunCtl: Fire's deadlines */
    CHECK(bf_resident_sched(ctx[k], h[k]) == BF_OK);    /* EnableSched */
    bf_sched_put put[N];
    memset(put, 0, sizeof put);
    for (uint32_t r = 0; r < N; ++r) {
      put[r].run = r; put[r].story_key = 0; put[r].queue_key = BF_SCHED_NONE;
      put[r].queued_since = BF_SCHED_NONE; put[r].run_phase = BF_PHASE_RUNNING;
    }
    CHECK(bf_resident_sched_put(ctx[k], h[k], put, N) == BF_OK);
  }
  /* tick 1 per ctx: full, step 1 of every run ready */
  for (int k = 0; k < 2; ++k) {
    CHECK(tick(k) == BF_OK);
    CHECK(full == 1 && n_listed == N && n_ev == N && counts.ready == N && events[0] == (1 | BF_EVT_READY << 10));
  }
  /* one ScheduleResidentCtxs over both batches: the Story's Running count is both ctxs' */
  static uint32_t sr[2][N];
  static bf_sched_header sh[2][N];
  static uint16_t se[2][EV];
  bf_resident_sched_part parts[2];
  for (int k = 0; k < 2; ++k) bfgo_sched_part(&parts[k], h[k], N, sr[k], sh[k], N, se[k], EV);
  const int32_t story_limit[1] = {2 * N + 1};
  uint32_t story_running = 0, gr = 0;
  CHECK(bfgo_resident_schedule_ctxs(100, 1, 0, 0, 0, story_limit, NULL, NULL, NULL, NULL, NULL, ctx, parts, 2, &story_running, NULL,
                                    NULL, &gr) == BF_OK);
  CHECK(story_running == 2 * N && gr == 2 * N);
  for (int k = 0; k < 2; ++k) CHECK(parts[k].n_listed == N && parts[k].full == 1 && sh[k][0].n_launch == 1 && se[k][0] == (1 | BF_SEVT_LAUNCH << 10));
  /* Commit on each: every run launches its ready step */
  for (int k = 0; k < 2; ++k) {
    uint32_t cc[7];
    CHECK(bfgo_resident_commit(ctx[k], h[k], N, NULL, 0, cc) == BF_OK && cc[2] == N);
  }
  /* TickTouched per ctx: the commit wrote every run, so each is listed, with nothing ready */
  for (int k = 0; k < 2; ++k) {
    CHECK(tick(k) == BF_OK);
    CHECK(full == 0 && n_listed == N && n_ev == 0);
  }
  /* TransferToCtx: an unmapped slot is refused and changes nothing; then runs 0 and 2 move with their slot mapped */
  const uint32_t moved[2] = {0, 2}, map_none[2] = {BF_SLOT_NONE, BF_SLOT_NONE}, map[2] = {BF_SLOT_NONE, 0};
  uint32_t from[2], to[2], tc[5], why[4];
  CHECK(bfgo_resident_transfer_ctx(ctx[0], h[0], ctx[1], h[1], N, N, moved, 2, map_none, 2, from, to, tc, why) == BF_EINVAL);
  CHECK(tc[0] == N && tc[1] == N && tc[3] == 0 && tc[4] == BF_UNFIT_SLOT_UNMAPPED);
  CHECK(bfgo_resident_transfer_ctx(ctx[0], h[0], ctx[1], h[1], N, N, moved, 2, map, 2, from, to, tc, why) == BF_OK);
  CHECK(tc[0] == N - 2 && tc[1] == N + 2 && tc[2] == 1 && from[0] == 3 && to[0] == 0);
  n_runs[0] = N - 2; n_runs[1] = N + 2;
  CHECK(bf_resident_download(ctx[1], h[1], 0, N + 2, rec) == BF_OK);
  for (uint32_t r = 0; r < N + 2; ++r) CHECK(((bf_run_header*)(rec + (size_t)r * L.state_stride))->topo_slot == slot[1]);
  /* TickTouched per ctx: the source lists its moved run, the destination its two arrivals; neither tick is full */
  CHECK(tick(0) == BF_OK);
  CHECK(full == 0 && n_listed == 1 && runs[0] == 0);
  CHECK(tick(1) == BF_OK);
  CHECK(full == 0 && n_listed == 2 && runs[0] == N && runs[1] == N + 1);
  free(rec);
  for (int k = 0; k < 2; ++k) {
    CHECK(bf_resident_destroy(ctx[k], h[k]) == BF_OK);
    bf_destroy(ctx[k]);
    ctx[k] = NULL;
  }
  printf("c_ctx_span_harness: ok\n");
  return 0;
}
