/*
 * c_runctl_harness.c — plain C caller of libbobrafrontier.so that performs the call sequence of Resident.{EnableRunCtl, PutRunCtl,
 * Fire} in the cgo binding (go/frontier/frontier.go) through the same entry points and flat wrappers (go/frontier/shim.h): run 3
 * gets a story deadline and a sleep timer, run 9 is cancelled with a drain deadline; a fire before anything is due reports the
 * next wake-up; at the story deadline run 3 is stopped (its sleep pruned, not listed) and the next touched tick evaluates the two
 * stopped runs and lists no event for either; the drain deadline is then listed wake-only; a redrive of the whole run lifts run
 * 3's stop and gives back its flags byte.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_runctl_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_runctl_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 16, CAP_EV = 4096 };

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  /* the Story: A; B (sleep) needs A; C needs nothing */
  const uint32_t rp[4] = {0, 0, 1, 1};
  const uint16_t ci[1] = {0};
  const uint8_t fl[3] = {0, BF_STEP_SLEEP, 0};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, 3, 1, rp, ci, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  bf_layout L;
  CHECK(bf_layout_init(&L, 32, 0, BF_F_DECISION) == BF_OK);
  uint8_t* rec = (uint8_t*)calloc(N, L.state_stride);
  for (uint32_t r = 0; r < N; ++r) {   /* A Succeeded (code 3: planes 0 and 1), B Running (code 2: plane 1), C Pending */
    uint8_t* p = rec + (size_t)r * L.state_stride;
    ((bf_run_header*)p)->topo_slot = slot;
    ((bf_run_header*)p)->run_flags = BF_RF_FAIL_FAST;
    uint32_t* ph = (uint32_t*)(p + L.off_phase);
    ph[0] = 0x1u;
    ph[L.words] = 0x3u;
  }
  uint32_t h = 0;
  CHECK(bf_resident_create(ctx, &L, N, &h) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, rec) == BF_OK);
  uint32_t runs[N], head[N], full, n_listed, n_eval;
  uint16_t events[CAP_EV];
  uint64_t n_events;
  bf_counts k;
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(full == 1);

  /* EnableTimers, EnableRunCtl, PutRunCtl: run 3's story deadline, run 9's cancel */
  CHECK(bf_resident_timers(ctx, h, 2) == BF_OK);
  bf_timer t;
  memset(&t, 0, sizeof t);
  t.run = 3; t.step = 1; t.code = BF_DEC_SUCCEED; t.deadline = 100;   /* sleepUntil, due with the story timeout */
  CHECK(bf_resident_timers_arm(ctx, h, &t, 1) == BF_OK);
  CHECK(bf_resident_runctl(ctx, h) == BF_OK);
  CHECK(bfgo_resident_runctl_put1(ctx, h, 3, 100, BF_TIMER_NONE, BF_STOP_NONE) == BF_OK);
  CHECK(bfgo_resident_runctl_put1(ctx, h, 9, BF_TIMER_NONE, 300, BF_STOP_CANCEL) == BF_OK);
  bf_run_ctl rc[N];
  CHECK(bf_resident_runctl_download(ctx, h, 0, N, rc) == BF_OK);
  CHECK(rc[9].stop == BF_STOP_CANCEL && rc[9].saved_flags == BF_RF_FAIL_FAST && rc[3].story_deadline == 100);

  /* Fire before anything is due: the next wake-up */
  bf_fired fired[8];
  uint32_t c[5];
  CHECK(bfgo_resident_fire(ctx, h, N, 99, fired, 8, c) == BF_OK);
  CHECK(c[0] == 0 && c[3] == 100);

  /* Fire at the story deadline: run 3 stopped, its sleep pruned; TickTouched evaluates runs 3 and 9, no events */
  CHECK(bfgo_resident_fire(ctx, h, N, 100, fired, 8, c) == BF_OK);
  CHECK(c[0] == 1 && c[1] == 1 && c[2] == 1 && c[3] == 300);
  CHECK(fired[0].run == 3 && fired[0].step == BF_FIRED_STORY && fired[0].code == BF_DEC_TIMED_OUT && fired[0].written == 1);
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(full == 0 && n_eval == 2 && n_events == 0);
  for (uint32_t i = 0; i < n_listed; ++i) CHECK((head[i] & BF_SUM_GROUP_MASK) == BF_GROUP_DONE && (head[i] >> BF_HEAD_COUNT_SHIFT) == 0);

  /* the drain deadline: listed wake-only, nothing armed after it */
  CHECK(bfgo_resident_fire(ctx, h, N, 300, fired, 8, c) == BF_OK);
  CHECK(c[0] == 1 && c[1] == 0 && c[3] == BF_TIMER_NONE && fired[0].run == 9 && fired[0].step == BF_FIRED_DRAIN && fired[0].written == 0);

  /* a redrive of the whole run lifts run 3's stop */
  bf_redrive rd;
  memset(&rd, 0, sizeof rd);
  rd.run = 3; rd.slot = slot; rd.step = BF_REDRIVE_ALL;
  uint8_t st = 0;
  uint32_t applied = 0;
  CHECK(bf_resident_redrive(ctx, h, &rd, 1, &st, &applied) == BF_OK && applied == 1);
  CHECK(bf_resident_runctl_download(ctx, h, 3, 1, rc) == BF_OK);
  CHECK(rc[0].stop == BF_STOP_NONE && rc[0].story_deadline == BF_TIMER_NONE);
  CHECK(bf_resident_download(ctx, h, 3, 1, rec) == BF_OK);
  CHECK(((bf_run_header*)rec)->run_flags == BF_RF_FAIL_FAST);

  CHECK(bf_resident_destroy(ctx, h) == BF_OK);
  free(rec);
  bf_destroy(ctx);
  printf("c_runctl_harness: ok\n");
  return 0;
}
