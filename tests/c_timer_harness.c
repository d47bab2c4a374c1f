/*
 * c_timer_harness.c — plain C caller of libbobrafrontier.so that performs the call sequence of Resident.{EnableTimers, ArmTimers,
 * Fire} in the cgo binding (go/frontier/frontier.go) through the same entry points and flat wrapper (go/frontier/shim.h): a gate
 * timeout, a sleep and a wake-only poll are armed; a fire before any is due reports the next wake-up; a fire at the gate's
 * deadline writes BF_DEC_TIMED_OUT and the next touched tick evaluates exactly that run; a retire moves the sleep's timer with
 * its run; the last fire lists the sleep (written) and the poll (wake-only) and leaves nothing armed.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_timer_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_timer_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 16, CAP_EV = 4096 };

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  /* the Story: A (gate); B (sleep) needs A; C (wait) needs nothing */
  const uint32_t rp[4] = {0, 0, 1, 1};
  const uint16_t ci[1] = {0};
  const uint8_t fl[3] = {BF_STEP_GATE, BF_STEP_SLEEP, BF_STEP_WAIT};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, 3, 1, rp, ci, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  bf_layout L;
  CHECK(bf_layout_init(&L, 32, 0, BF_F_DECISION) == BF_OK);
  uint8_t* rec = (uint8_t*)calloc(N, L.state_stride);
  for (uint32_t r = 0; r < N; ++r) {
    uint8_t* p = rec + (size_t)r * L.state_stride;
    ((bf_run_header*)p)->topo_slot = slot;
    uint32_t* ph = (uint32_t*)(p + L.off_phase);   /* every step Running (code 2: plane 1) */
    ph[L.words] = 0x7u;
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

  /* EnableTimers, ArmTimers */
  CHECK(bf_resident_timers(ctx, h, 2) == BF_OK);
  bf_timer t[3];
  memset(t, 0, sizeof t);
  t[0].run = 3; t[0].step = 0; t[0].code = BF_DEC_TIMED_OUT; t[0].deadline = 100;   /* gate timeout */
  t[1].run = 15; t[1].step = 1; t[1].code = BF_DEC_SUCCEED; t[1].deadline = 200;    /* sleepUntil */
  t[2].run = 15; t[2].step = 2; t[2].code = BF_DEC_PENDING; t[2].deadline = 150;    /* pollInterval: wake-only */
  CHECK(bf_resident_timers_arm(ctx, h, t, 3) == BF_OK);

  /* Fire before anything is due: the next wake-up */
  bf_fired fired[8];
  uint32_t c[5];
  CHECK(bfgo_resident_fire(ctx, h, N, 99, fired, 8, c) == BF_OK);
  CHECK(c[0] == 0 && c[3] == 100);

  /* Fire at the gate's deadline, then TickTouched: run 3 alone is evaluated */
  CHECK(bfgo_resident_fire(ctx, h, N, 100, fired, 8, c) == BF_OK);
  CHECK(c[0] == 1 && c[1] == 1 && c[3] == 150 && fired[0].run == 3 && fired[0].step == 0 && fired[0].written == 1);
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(full == 0 && n_eval == 1);

  /* Retire run 0: run 15 moves to index 0 with its timers */
  bf_retire rt;
  memset(&rt, 0, sizeof rt);
  const uint32_t gone[1] = {0};
  rt.struct_size = (uint32_t)sizeof rt; rt.n_runs = N; rt.runs = gone; rt.n = 1;
  CHECK(bf_resident_retire(ctx, h, &rt) == BF_OK && rt.n_runs == N - 1);
  bf_timer_slot s[2 * N];
  CHECK(bf_resident_timers_download(ctx, h, 0, N, s) == BF_OK);
  CHECK(s[0].step == 1 && s[0].deadline == 200 && s[1].step == 2 && s[1].deadline == 150);
  CHECK(s[2 * 15].deadline == BF_TIMER_NONE && s[2 * 15 + 1].deadline == BF_TIMER_NONE);

  /* the last fire: the sleep (written) and the poll (wake-only); nothing stays armed */
  CHECK(bfgo_resident_fire(ctx, h, N - 1, 250, fired, 8, c) == BF_OK);
  CHECK(c[0] == 2 && c[1] == 1 && c[3] == BF_TIMER_NONE);
  CHECK(fired[0].run == 0 && fired[0].step == 1 && fired[0].written == 1 && fired[1].step == 2 && fired[1].written == 0);

  CHECK(bf_resident_destroy(ctx, h) == BF_OK);
  free(rec);
  bf_destroy(ctx);
  printf("c_timer_harness: ok\n");
  return 0;
}
