/*
 * c_commit_harness.c — plain C caller of libbobrafrontier.so that performs the per-tick loop of the cgo binding
 * (go/frontier/frontier.go) through the same entry points and flat wrappers (go/frontier/shim.h): Resident.Fire ->
 * TickTouched -> Ctx.ScheduleResident -> (Execute) -> Resident.Commit.  The Story: A (engram), B (condition), C (stop), D
 * (engram) needs B.  Four runs: run 3's Story limit of 1 launches A alone and queues B and C; the others launch A, B and C.
 * Run 1's Execute held A, run 2's failed.  Commits without C's phase, with a PHASE entry on a step that is not a stop step and
 * with an entry on a queued step are refused, naming the offender; the commit then writes A Running, B Succeeded, C the phase
 * of its entry and run 3's B and C code 14, a second commit is refused until a tick, and the next touched tick evaluates the
 * three written runs and lists D ready in run 0 without any delta.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_commit_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_commit_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 4, CAP_EV = 64 };

static uint32_t phase_of(const uint8_t* rec, const bf_layout* L, uint32_t step) {
  const uint32_t* ph = (const uint32_t*)(rec + L->off_phase);
  uint32_t code = 0;
  for (uint32_t b = 0; b < 4; ++b) code |= ((ph[b * L->words + step / 32] >> (step % 32)) & 1u) << b;
  return code;
}

static bf_commit_entry entry(uint32_t run, uint16_t step, uint8_t kind, uint8_t code) {
  bf_commit_entry e;
  e.run = run; e.step = step; e.kind = kind; e.code = code;
  return e;
}

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  const uint32_t rp[5] = {0, 0, 0, 0, 1};
  const uint16_t ci[1] = {1};
  const uint8_t fl[4] = {BF_STEP_ENGRAM, BF_STEP_CONDITION, BF_STEP_STOP, BF_STEP_ENGRAM};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, 4, 1, rp, ci, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  bf_layout L;
  CHECK(bf_layout_init(&L, 32, 0, BF_F_DECISION | BF_F_OUT_FAIL) == BF_OK);
  uint8_t* rec = (uint8_t*)calloc(N, L.state_stride);
  for (uint32_t r = 0; r < N; ++r) ((bf_run_header*)(rec + (size_t)r * L.state_stride))->topo_slot = slot;
  uint32_t h;
  CHECK(bf_resident_create(ctx, &L, N, &h) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, rec) == BF_OK);
  CHECK(bf_resident_timers(ctx, h, 1) == BF_OK);                                      /* EnableTimers */
  CHECK(bf_resident_sched(ctx, h) == BF_OK);                                          /* EnableSched */
  bf_sched_put put[N];
  memset(put, 0, sizeof put);
  for (uint32_t r = 0; r < N; ++r) {
    put[r].run = r; put[r].story_key = r == 3 ? 0 : BF_SCHED_NONE; put[r].queue_key = BF_SCHED_NONE;
    put[r].queued_since = BF_SCHED_NONE; put[r].run_phase = BF_PHASE_RUNNING;
  }
  CHECK(bf_resident_sched_put(ctx, h, put, N) == BF_OK);

  /* Fire -> TickTouched -> ScheduleResident */
  bf_fired fired[4];
  uint32_t fc[5];
  CHECK(bfgo_resident_fire(ctx, h, N, 1, fired, 4, fc) == BF_OK && fc[0] == 0);
  uint32_t runs_t[N], head_t[N], full, n_listed, n_eval;
  uint16_t ev_t[CAP_EV];
  uint64_t n_ev;
  bf_counts k;
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, CAP_EV, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  CHECK(full == 1 && k.ready == 3 * N);
  uint32_t* runs;
  bf_sched_header* heads;
  uint16_t* events;
  CHECK(bf_alloc_pinned(ctx, N * sizeof(uint32_t), (void**)&runs) == BF_OK);
  CHECK(bf_alloc_pinned(ctx, N * sizeof(bf_sched_header), (void**)&heads) == BF_OK);
  CHECK(bf_alloc_pinned(ctx, CAP_EV * sizeof(uint16_t), (void**)&events) == BF_OK);
  bf_resident_sched_part part;
  bfgo_sched_part(&part, h, N, runs, heads, N, events, CAP_EV);
  const int32_t sl[1] = {1};
  uint32_t sr[1], gr;
  CHECK(bfgo_resident_schedule(ctx, 1, 1, 0, 0, 0, sl, NULL, NULL, NULL, NULL, NULL, &part, 1, sr, NULL, NULL, &gr) == BF_OK);
  CHECK(part.n_listed == N && heads[3].n_launch == 1 && heads[3].n_queued_story == 2 && heads[0].n_launch == 3);

  /* refusals: nothing changes, the first offender is named */
  uint32_t c[7];
  CHECK(bfgo_resident_commit(ctx, h, N, NULL, 0, c) == BF_EINVAL && c[5] == 0 && c[6] == 2);            /* C has no phase */
  bf_commit_entry e[5];
  e[0] = entry(0, 2, BF_COMMIT_PHASE, BF_PHASE_SUCCEEDED);
  e[1] = entry(1, 0, BF_COMMIT_HOLD, 0);
  e[2] = entry(1, 2, BF_COMMIT_PHASE, BF_PHASE_FAILED);
  e[3] = entry(2, 1, BF_COMMIT_ERROR, 0);
  e[4] = entry(3, 0, BF_COMMIT_PHASE, BF_PHASE_SUCCEEDED);
  CHECK(bfgo_resident_commit(ctx, h, N, e, 5, c) == BF_EINVAL && c[5] == 3 && c[6] == 0);               /* A is no stop step */
  e[4] = entry(3, 2, BF_COMMIT_HOLD, 0);
  CHECK(bfgo_resident_commit(ctx, h, N, e, 5, c) == BF_EINVAL && c[5] == 3 && c[6] == 2);               /* run 3's C is queued */
  uint8_t* got = (uint8_t*)malloc((size_t)N * L.state_stride);
  CHECK(bf_resident_download(ctx, h, 0, N, got) == BF_OK && memcmp(got, rec, (size_t)N * L.state_stride) == 0);

  /* Commit: runs 0, 1 and 3 written; run 2's Execute failed */
  CHECK(bfgo_resident_commit(ctx, h, N, e, 4, c) == BF_OK);
  CHECK(c[0] == 3 && c[1] == 0 && c[2] == 3 + 2 + 1 && c[3] == 2 && c[4] == 0);
  CHECK(bf_resident_download(ctx, h, 0, N, got) == BF_OK);
  const uint8_t* g0 = got;
  const uint8_t* g1 = got + L.state_stride;
  const uint8_t* g2 = got + 2 * (size_t)L.state_stride;
  const uint8_t* g3 = got + 3 * (size_t)L.state_stride;
  CHECK(phase_of(g0, &L, 0) == BF_PHASE_RUNNING && phase_of(g0, &L, 1) == BF_PHASE_SUCCEEDED && phase_of(g0, &L, 2) == BF_PHASE_SUCCEEDED);
  CHECK(phase_of(g1, &L, 0) == 0 && phase_of(g1, &L, 1) == BF_PHASE_SUCCEEDED && phase_of(g1, &L, 2) == BF_PHASE_FAILED);
  CHECK(memcmp(g2, rec + 2 * (size_t)L.state_stride, L.state_stride) == 0);
  CHECK(phase_of(g3, &L, 0) == BF_PHASE_RUNNING && phase_of(g3, &L, 1) == BF_PHASE_PENDING_QUEUED &&
        phase_of(g3, &L, 2) == BF_PHASE_PENDING_QUEUED && phase_of(g3, &L, 3) == 0);
  /* the commit wrote: the tick is over */
  CHECK(bfgo_resident_commit(ctx, h, N, e, 4, c) == BF_EINVAL && c[5] == BF_COMMIT_NONE && c[6] == BF_COMMIT_NONE);

  /* the next touched tick evaluates the written runs alone; D is ready in run 0 with no delta sent */
  CHECK(bfgo_resident_fire(ctx, h, N, 2, fired, 4, fc) == BF_OK);
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, CAP_EV, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  CHECK(full == 0 && n_eval == 3 && n_listed >= 1 && runs_t[0] == 0);
  CHECK((head_t[0] >> BF_HEAD_COUNT_SHIFT) == 1 && ev_t[0] == (3 | BF_EVT_READY << 10));

  free(got);
  CHECK(bf_free_pinned(ctx, runs) == BF_OK && bf_free_pinned(ctx, heads) == BF_OK && bf_free_pinned(ctx, events) == BF_OK);
  CHECK(bf_resident_destroy(ctx, h) == BF_OK);
  free(rec);
  bf_destroy(ctx);
  printf("c_commit_harness: ok\n");
  return 0;
}
