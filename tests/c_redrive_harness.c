/*
 * c_redrive_harness.c — plain C caller of libbobrafrontier.so that performs the call sequence of Resident.Redrive in the cgo binding
 * (go/frontier/frontier.go) through the same flat wrapper (go/frontier/shim.h): live runs are uploaded, an operator redrives some
 * of them (from a step, and whole runs), a stale and a duplicate request among them, and the next touched tick lists the reset runs.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_redrive_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_redrive_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 64, CAP_EV = 1024 };

static uint32_t phase_of(const uint8_t* rec, const bf_layout* L, uint32_t step) {
  const uint32_t* w = (const uint32_t*)(rec + L->off_phase);
  uint32_t v = 0;
  for (uint32_t b = 0; b < 4; ++b) v |= ((w[b * L->words + step / 32] >> (step % 32)) & 1u) << b;
  return v;
}

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  /* A; B needs A; C needs B; D needs nothing.  Every step has Succeeded in every run.  */
  const uint32_t rp[5] = {0, 0, 1, 2, 2};
  const uint16_t ci[2] = {0, 1};
  const uint8_t fl[4] = {BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t s_run = 99, s_other = 99;
  CHECK(bfgo_topology_put(ctx, 4, 2, rp, ci, fl, NULL, 0, NULL, 0, &s_run) == BF_OK);
  CHECK(bfgo_topology_put(ctx, 4, 2, rp, ci, fl, NULL, 0, NULL, 0, &s_other) == BF_OK);   /* another Story, same shape */
  bf_layout L;
  CHECK(bf_layout_init(&L, 4, 0, BF_F_OUT_SKIP_DEP) == BF_OK);
  uint8_t* state = (uint8_t*)calloc(N, L.state_stride);
  uint8_t* back = (uint8_t*)calloc(N, L.state_stride);
  for (uint32_t r = 0; r < N; ++r) {   /* even runs on s_run, odd ones on s_other; all TopologyTerminated */
    uint8_t* rec = state + (size_t)r * L.state_stride;
    ((bf_run_header*)rec)->topo_slot = (r % 2) ? s_other : s_run;
    ((bf_run_header*)rec)->run_flags = BF_RF_TOPOLOGY_TERMINATED;
    uint32_t* ph = (uint32_t*)(rec + L.off_phase);
    ph[0 * L.words] = 0xFu; ph[1 * L.words] = 0xFu;   /* steps 0-3: code 3 (Succeeded) */
  }
  uint32_t h = 0;
  CHECK(bf_resident_create(ctx, &L, N, &h) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, state) == BF_OK);
  uint32_t runs[N], head[N], full = 9, n_listed = 0, n_eval = 0;
  uint16_t events[CAP_EV];
  uint64_t n_events = 0;
  bf_counts k;
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(full == 1 && n_listed == N && n_events == 0);

  /* a step past S is rejected and changes nothing */
  uint8_t status[8];
  uint32_t applied = 77;
  const bf_redrive bad[1] = {{0, s_run, 4, 0}};
  CHECK(bfgo_resident_redrive(ctx, h, bad, 1, status, &applied) == BF_EINVAL);
  CHECK(bf_resident_download(ctx, h, 0, N, back) == BF_OK && memcmp(back, state, (size_t)N * L.state_stride) == 0);
  /* run 0 from B; run 2 entirely and again from B (a duplicate); run 1 is not on s_run (stale); run 4 from D */
  const bf_redrive req[5] = {{0, s_run, 1, 0}, {2, s_run, BF_REDRIVE_ALL, 0}, {2, s_run, 1, 0}, {1, s_run, 0, 0}, {4, s_run, 3, 0}};
  CHECK(bfgo_resident_redrive(ctx, h, req, 5, status, &applied) == BF_OK && applied == 4);
  CHECK(status[0] == 1 && status[1] == 1 && status[2] == 1 && status[3] == 0 && status[4] == 1);
  CHECK(bf_resident_download(ctx, h, 0, N, back) == BF_OK);
  const uint32_t want[5][4] = {{3, 0, 0, 3}, {0}, {0, 0, 0, 0}, {0}, {3, 3, 3, 0}};   /* phases of runs 0, 2 and 4 */
  for (uint32_t r = 0; r < N; ++r) {
    const uint8_t* rec = back + (size_t)r * L.state_stride;
    if (r % 2 || r > 4) {   /* the runs of s_other (run 1: the stale request) and every run not named */
      CHECK(memcmp(rec, state + (size_t)r * L.state_stride, L.state_stride) == 0);
      continue;
    }
    CHECK(((const bf_run_header*)rec)->topo_slot == s_run && ((const bf_run_header*)rec)->run_flags == 0);
    for (uint32_t s = 0; s < 4; ++s) CHECK(phase_of(rec, &L, s) == want[r][s]);
  }
  /* the next touched tick evaluates the three reset runs and lists them: B ready in run 0, A and D in run 2, D in run 4 */
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(full == 0 && n_listed == 3 && n_eval == 3 && n_events == 4);
  CHECK(runs[0] == 0 && runs[1] == 2 && runs[2] == 4);
  CHECK((head[0] >> BF_HEAD_COUNT_SHIFT) == 1 && (head[1] >> BF_HEAD_COUNT_SHIFT) == 2 && (head[2] >> BF_HEAD_COUNT_SHIFT) == 1);
  const uint32_t ev_step[4] = {1, 0, 3, 3};
  for (uint32_t i = 0; i < 4; ++i) CHECK(BF_EVENT_STEP(events[i]) == ev_step[i] && BF_EVENT_KIND(events[i]) == BF_EVT_READY);

  CHECK(bf_resident_destroy(ctx, h) == BF_OK);
  free(state);
  free(back);
  bf_destroy(ctx);
  printf("c_redrive_harness: ok\n");
  return 0;
}
