/*
 * c_sched_harness.c — plain C caller of libbobrafrontier.so that performs the call sequence of Resident.{EnableSched, PutSched} and
 * Ctx.ScheduleResident in the cgo binding (go/frontier/frontier.go) through the same entry points and flat wrappers
 * (go/frontier/shim.h), with the lists in pinned memory as NewSchedBuffers allocates them.  Two batches of one engram Story with
 * two independent steps share one queue: the first schedule lists every run, with caps smaller than the lists; a later `now`
 * ages the low-priority run past the high one; a put that changes nothing lists nothing; a delta without a tick is refused.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_sched_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_sched_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 4 };

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  const uint32_t rp[3] = {0, 0, 0};
  const uint8_t fl[2] = {BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, 2, 0, rp, NULL, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  bf_layout L;
  CHECK(bf_layout_init(&L, 32, 0, 0) == BF_OK);
  uint8_t* rec = (uint8_t*)calloc(N, L.state_stride);
  for (uint32_t r = 0; r < N; ++r) ((bf_run_header*)(rec + (size_t)r * L.state_stride))->topo_slot = slot;   /* both steps ready */
  uint32_t h[2];
  uint32_t runs_t[N], head_t[N], full, n_listed, n_eval;
  uint16_t ev_t[64];
  uint64_t n_ev;
  bf_counts k;
  for (int b = 0; b < 2; ++b) {
    CHECK(bf_resident_create(ctx, &L, N, &h[b]) == BF_OK);
    CHECK(bf_resident_upload(ctx, h[b], 0, N, rec) == BF_OK);
    CHECK(bf_resident_sched(ctx, h[b]) == BF_OK);                                    /* EnableSched */
    CHECK(bfgo_resident_tick_touched(ctx, h[b], NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, 64, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  }
  /* PutSched: every run in queue 0; batch 0 run 0 has priority 5, the others 1, batch 1 run 2 queued since t = 0 */
  bf_sched_put put[N];
  for (int b = 0; b < 2; ++b) {
    memset(put, 0, sizeof put);
    for (uint32_t r = 0; r < N; ++r) {
      put[r].run = r; put[r].story_key = BF_SCHED_NONE; put[r].queue_key = 0;
      put[r].priority = (b == 0 && r == 0) ? 5 : 1;
      put[r].queued_since = (b == 1 && r == 2) ? 0 : BF_SCHED_NONE;
      put[r].run_phase = BF_PHASE_RUNNING;
    }
    CHECK(bf_resident_sched_put(ctx, h[b], put, N) == BF_OK);
  }
  /* the list buffers in pinned memory, caps below the lists: 3 of 4 runs, 5 events per part */
  uint32_t* runs[2];
  bf_sched_header* heads[2];
  uint16_t* events[2];
  for (int b = 0; b < 2; ++b) {
    CHECK(bf_alloc_pinned(ctx, 3 * sizeof(uint32_t), (void**)&runs[b]) == BF_OK);
    CHECK(bf_alloc_pinned(ctx, 3 * sizeof(bf_sched_header), (void**)&heads[b]) == BF_OK);
    CHECK(bf_alloc_pinned(ctx, 5 * sizeof(uint16_t), (void**)&events[b]) == BF_OK);
  }
  const int32_t ql[1] = {0}, qa[1] = {1};
  uint32_t qr[1], gr;
  int32_t mp[1];
  bf_resident_sched_part parts[2];
  for (int b = 0; b < 2; ++b) bfgo_sched_part(&parts[b], h[b], N, runs[b], heads[b], 3, events[b], 5);
  CHECK(bfgo_resident_schedule(ctx, 3, 0, 1, 0, 0, NULL, NULL, ql, qa, NULL, NULL, parts, 2, NULL, qr, mp, &gr) == BF_OK);
  /* at now = 3 the aged run has priority 4 < 5: only batch 0 run 0 launches; every run is listed, true counts past the caps */
  CHECK(mp[0] == 5 && gr == 0);
  CHECK(parts[0].full == 1 && parts[0].n_listed == N && parts[0].n_events == 2 * N);
  CHECK(runs[0][0] == 0 && runs[0][1] == 1 && runs[0][2] == 2);
  CHECK(heads[0][0].n_launch == 2 && heads[0][1].n_launch == 0 && heads[0][1].n_queued_sched == 2 && heads[0][1].sched_reason == BF_QUEUED_PRIORITY);
  CHECK(events[0][0] == (0 | BF_SEVT_LAUNCH << 10) && events[0][1] == (1 | BF_SEVT_LAUNCH << 10) &&
        events[0][2] == (0 | BF_SEVT_QUEUED_SCHED << 10) && events[0][4] == (0 | BF_SEVT_QUEUED_SCHED << 10));
  CHECK(parts[1].n_listed == N && heads[1][2].n_launch == 0);
  /* at now = 10 the aged run (priority 11) outranks everyone: it alone launches, and every run whose record changed is listed */
  for (int b = 0; b < 2; ++b) bfgo_sched_part(&parts[b], h[b], N, runs[b], heads[b], 3, events[b], 5);
  CHECK(bfgo_resident_schedule(ctx, 10, 0, 1, 0, 0, NULL, NULL, ql, qa, NULL, NULL, parts, 2, NULL, qr, mp, &gr) == BF_OK);
  CHECK(mp[0] == 11 && parts[0].n_listed == 1 && runs[0][0] == 0 && heads[0][0].n_launch == 0 && heads[0][0].n_queued_sched == 2);
  CHECK(parts[1].n_listed == 1 && runs[1][0] == 2 && heads[1][0].n_launch == 2 && parts[1].full == 0);
  /* a put that changes nothing lists nothing */
  CHECK(bf_resident_sched_put(ctx, h[1], put, N) == BF_OK);
  for (int b = 0; b < 2; ++b) bfgo_sched_part(&parts[b], h[b], N, runs[b], heads[b], 3, events[b], 5);
  CHECK(bfgo_resident_schedule(ctx, 10, 0, 1, 0, 0, NULL, NULL, ql, qa, NULL, NULL, parts, 2, NULL, qr, mp, &gr) == BF_OK);
  CHECK(parts[0].n_listed == 0 && parts[1].n_listed == 0 && parts[1].n_events == 0);
  /* a delta without a tick: refused, naming the batch; after the tick the schedule goes through */
  bf_delta d;
  memset(&d, 0, sizeof d);
  d.run = 1; d.index = 0; d.field = BF_DELTA_PHASE; d.code = BF_PHASE_RUNNING;
  CHECK(bf_resident_apply(ctx, h[0], &d, 1) == BF_OK);
  CHECK(bfgo_resident_schedule(ctx, 10, 0, 1, 0, 0, NULL, NULL, ql, qa, NULL, NULL, parts, 2, NULL, qr, mp, &gr) == BF_EINVAL);
  CHECK(strstr(bf_last_error(ctx), "batch") != NULL);
  CHECK(bfgo_resident_tick_touched(ctx, h[0], NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, 64, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  CHECK(bfgo_resident_schedule(ctx, 10, 0, 1, 0, 0, NULL, NULL, ql, qa, NULL, NULL, parts, 2, NULL, qr, mp, &gr) == BF_OK);
  CHECK(gr == 1 && parts[0].n_listed == 1 && runs[0][0] == 1 && heads[0][0].n_queued_sched == 1);

  for (int b = 0; b < 2; ++b) {
    CHECK(bf_free_pinned(ctx, runs[b]) == BF_OK && bf_free_pinned(ctx, heads[b]) == BF_OK && bf_free_pinned(ctx, events[b]) == BF_OK);
    CHECK(bf_resident_destroy(ctx, h[b]) == BF_OK);
  }
  free(rec);
  bf_destroy(ctx);
  printf("c_sched_harness: ok\n");
  return 0;
}
