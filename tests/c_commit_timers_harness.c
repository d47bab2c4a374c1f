/*
 * c_commit_timers_harness.c — plain C caller of libbobrafrontier.so that performs the per-tick loop of the cgo binding with
 * timed commits (go/frontier/frontier.go) through the same entry points and flat wrappers (go/frontier/shim.h):
 * Ctx.PutTimings -> Resident.Fire -> TickTouched -> Ctx.ScheduleResident -> (Execute) -> Resident.CommitTimed.  The Story: S
 * (sleep, 1 unit), E (engram) needs S, G (gate, timeout 5 units).  Two runs launch S and G.  With one timer slot per run the
 * timed commit is refused with BF_ENOMEM at run 0's S and nothing changes; with two it pauses S and G and arms both in each
 * run (next deadline now + 1).  Fire at now fires nothing, Fire at now + 1 writes both sleeps, and the next touched tick lists
 * E ready in both runs with no delta sent.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_commit_timers_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_commit_timers_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 2, CAP_EV = 64, NOW = 100 };

static uint32_t phase_of(const uint8_t* rec, const bf_layout* L, uint32_t step) {
  const uint32_t* ph = (const uint32_t*)(rec + L->off_phase);
  uint32_t code = 0;
  for (uint32_t b = 0; b < 4; ++b) code |= ((ph[b * L->words + step / 32] >> (step % 32)) & 1u) << b;
  return code;
}

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  const uint32_t rp[4] = {0, 0, 1, 1};
  const uint16_t ci[1] = {0};
  const uint8_t fl[3] = {BF_STEP_SLEEP, BF_STEP_ENGRAM, BF_STEP_GATE};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, 3, 1, rp, ci, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  bf_step_timing tim[2];
  memset(tim, 0, sizeof tim);
  tim[0].step = 2; tim[0].code = BF_DEC_TIMED_OUT; tim[0].delay = 5;
  tim[1].step = 0; tim[1].code = BF_DEC_SUCCEED; tim[1].delay = 1;
  tim[1].reserved = 1;
  CHECK(bfgo_topology_timings(ctx, slot, tim, 2) == BF_EINVAL);                       /* reserved must be 0 */
  tim[1].reserved = 0;
  tim[1].code = BF_DEC_TIMED_OUT;
  CHECK(bfgo_topology_timings(ctx, slot, tim, 2) == BF_EINVAL);                       /* a sleep does not time out */
  tim[1].code = BF_DEC_SUCCEED;
  CHECK(bfgo_topology_timings(ctx, slot, tim, 2) == BF_OK);                           /* PutTimings */
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
    put[r].run = r; put[r].story_key = BF_SCHED_NONE; put[r].queue_key = BF_SCHED_NONE;
    put[r].queued_since = BF_SCHED_NONE; put[r].run_phase = BF_PHASE_RUNNING;
  }
  CHECK(bf_resident_sched_put(ctx, h, put, N) == BF_OK);

  /* Fire -> TickTouched -> ScheduleResident */
  bf_fired fired[8];
  uint32_t fc[5];
  CHECK(bfgo_resident_fire(ctx, h, N, NOW, fired, 8, fc) == BF_OK && fc[0] == 0);
  uint32_t runs_t[N], head_t[N], full, n_listed, n_eval;
  uint16_t ev_t[CAP_EV];
  uint64_t n_ev;
  bf_counts k;
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, CAP_EV, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  CHECK(full == 1 && k.ready == 2 * N);
  uint32_t* runs;
  bf_sched_header* heads;
  uint16_t* events;
  CHECK(bf_alloc_pinned(ctx, N * sizeof(uint32_t), (void**)&runs) == BF_OK);
  CHECK(bf_alloc_pinned(ctx, N * sizeof(bf_sched_header), (void**)&heads) == BF_OK);
  CHECK(bf_alloc_pinned(ctx, CAP_EV * sizeof(uint16_t), (void**)&events) == BF_OK);
  bf_resident_sched_part part;
  bfgo_sched_part(&part, h, N, runs, heads, N, events, CAP_EV);
  uint32_t gr;
  CHECK(bfgo_resident_schedule(ctx, NOW, 0, 0, 0, 0, NULL, NULL, NULL, NULL, NULL, NULL, &part, 1, NULL, NULL, NULL, &gr) == BF_OK);
  CHECK(part.n_listed == N && heads[0].n_launch == 2 && heads[1].n_launch == 2);

  /* CommitTimed: one slot per run cannot hold S and G, so nothing changes; two can */
  uint32_t c[9];
  CHECK(bfgo_resident_commit_timed(ctx, h, N, NULL, 0, NOW, c) == BF_ENOMEM && c[5] == 0 && c[6] == 0 && c[7] == 0 &&
        c[8] == BF_TIMER_NONE);
  CHECK(bfgo_resident_commit_timed(ctx, h, N, NULL, 0, BF_TIMER_NONE, c) == BF_EINVAL && c[5] == BF_COMMIT_NONE);
  uint8_t* got = (uint8_t*)malloc((size_t)N * L.state_stride);
  CHECK(bf_resident_download(ctx, h, 0, N, got) == BF_OK && memcmp(got, rec, (size_t)N * L.state_stride) == 0);
  bf_timer_slot ts[2 * N];
  CHECK(bf_resident_timers_download(ctx, h, 0, N, ts) == BF_OK && ts[0].deadline == BF_TIMER_NONE && ts[1].deadline == BF_TIMER_NONE);
  CHECK(bf_resident_timers(ctx, h, 2) == BF_OK);
  CHECK(bfgo_resident_commit_timed(ctx, h, N, NULL, 0, NOW, c) == BF_OK);
  CHECK(c[0] == N && c[2] == 2 * N && c[7] == 2 * N && c[8] == NOW + 1);
  CHECK(bf_resident_download(ctx, h, 0, N, got) == BF_OK);
  for (uint32_t r = 0; r < N; ++r) {
    const uint8_t* g = got + (size_t)r * L.state_stride;
    CHECK(phase_of(g, &L, 0) == BF_PHASE_PAUSED && phase_of(g, &L, 1) == 0 && phase_of(g, &L, 2) == BF_PHASE_PAUSED);
  }
  CHECK(bf_resident_timers_download(ctx, h, 0, N, ts) == BF_OK);
  for (uint32_t r = 0; r < N; ++r) {
    CHECK(ts[2 * r].deadline == NOW + 1 && ts[2 * r].step == 0 && ts[2 * r].code == BF_DEC_SUCCEED);
    CHECK(ts[2 * r + 1].deadline == NOW + 5 && ts[2 * r + 1].step == 2 && ts[2 * r + 1].code == BF_DEC_TIMED_OUT);
  }

  /* the next ticks: nothing due at now, both sleeps at now + 1, and E is ready with no delta sent */
  CHECK(bfgo_resident_fire(ctx, h, N, NOW, fired, 8, fc) == BF_OK && fc[0] == 0 && fc[3] == NOW + 1);
  CHECK(bfgo_resident_fire(ctx, h, N, NOW + 1, fired, 8, fc) == BF_OK && fc[0] == N && fc[1] == N && fc[3] == NOW + 5);
  CHECK(fired[0].run == 0 && fired[0].step == 0 && fired[0].written == 1 && fired[1].run == 1);
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, CAP_EV, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  CHECK(full == 0 && n_eval == N && n_listed == N && k.ready == N);
  CHECK((head_t[0] >> BF_HEAD_COUNT_SHIFT) == 1 && ev_t[0] == (1 | BF_EVT_READY << 10));

  free(got);
  CHECK(bf_free_pinned(ctx, runs) == BF_OK && bf_free_pinned(ctx, heads) == BF_OK && bf_free_pinned(ctx, events) == BF_OK);
  CHECK(bf_resident_destroy(ctx, h) == BF_OK);
  free(rec);
  bf_destroy(ctx);
  printf("c_commit_timers_harness: ok\n");
  return 0;
}
