/*
 * c_touched_harness.c — plain C caller of libbobrafrontier.so that performs the call sequence of Resident.TickTouched in the cgo
 * binding (go/frontier/frontier.go) through the same flat wrapper (go/frontier/shim.h), with pinned buffers as the Go side
 * uses them, and checks every touched tick against a changed-only compact tick of a twin batch that received the same deltas.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_touched_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_touched_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 64, CAP_EV = 1024 };

/* the touched tick's lists equal the changed-only tick's lists of the listed runs */
static int same_lists(const uint32_t* runs, const uint32_t* head, const uint16_t* events, uint32_t n_listed, const uint32_t* chead,
                      const uint16_t* cevents) {
  uint32_t k = 0, pos = 0, cpos = 0;
  for (uint32_t r = 0; r < N; ++r) {
    const uint32_t cn = chead[r] >> BF_HEAD_COUNT_SHIFT;
    if (chead[r] & BF_HEAD_LISTED) {
      if (k >= n_listed || runs[k] != r || head[k] != chead[r]) return 0;
      if (memcmp(events + pos, cevents + cpos, cn * sizeof(uint16_t)) != 0) return 0;
      pos += cn;
      ++k;
    }
    cpos += cn;
  }
  return k == n_listed;
}

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  /* story A; B needs A; C needs B */
  const uint32_t row_ptr[4] = {0, 0, 1, 2};
  const uint16_t col_idx[2] = {0, 1};
  const uint8_t flags[3] = {BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, 3, 2, row_ptr, col_idx, flags, NULL, 0, NULL, 0, &slot) == BF_OK);
  bf_layout L;
  CHECK(bf_layout_init(&L, 3, 0, BF_F_OUT_SKIP_DEP) == BF_OK);
  uint8_t* state = (uint8_t*)calloc(N, L.state_stride);
  for (uint32_t r = 0; r < N; ++r) ((bf_run_header*)(state + (size_t)r * L.state_stride))->topo_slot = slot;

  uint32_t hT = 0, hC = 0;
  CHECK(bf_resident_create(ctx, &L, N, &hT) == BF_OK && bf_resident_create(ctx, &L, N, &hC) == BF_OK);
  CHECK(bf_resident_upload(ctx, hT, 0, N, state) == BF_OK && bf_resident_upload(ctx, hC, 0, N, state) == BF_OK);
  void *runs_v = NULL, *head_v = NULL, *ev_v = NULL;
  CHECK(bf_alloc_pinned(ctx, N * 4, &runs_v) == BF_OK && bf_alloc_pinned(ctx, N * 4, &head_v) == BF_OK &&
        bf_alloc_pinned(ctx, CAP_EV * 2, &ev_v) == BF_OK);
  uint32_t* runs = (uint32_t*)runs_v;
  uint32_t* head = (uint32_t*)head_v;
  uint16_t* events = (uint16_t*)ev_v;
  uint32_t chead[N];
  uint16_t cevents[CAP_EV];
  uint32_t full = 9, n_listed = 0, n_eval = 0, c_listed = 0;
  uint64_t n_events = 0, c_events = 0;
  bf_counts k, kc;

  /* the first tick evaluates and lists every run: A is ready in each */
  CHECK(bfgo_resident_tick_touched(ctx, hT, NULL, 0, N, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(bfgo_resident_tick_compact(ctx, hC, NULL, 0, N, BF_EVAL_CHANGED_ONLY, 0, chead, cevents, CAP_EV, &c_events, &c_listed, &kc) == BF_OK);
  CHECK(full == 1 && n_listed == N && n_eval == N && n_events == N && runs[N - 1] == N - 1 && k.ready == N && k.evals == 3 * N);
  CHECK(same_lists(runs, head, events, n_listed, chead, cevents));

  /* run 3: A Succeeded (B ready); run 40: A Running (nothing ready); run 41: A Failed (B skipped); run 50: run flags rewritten
     to the value they had (touched, evaluated, not listed) */
  bf_delta d[4];
  memset(d, 0, sizeof d);
  d[0].run = 3;  d[0].index = 0; d[0].field = BF_DELTA_PHASE; d[0].code = BF_PHASE_SUCCEEDED;
  d[1].run = 40; d[1].index = 0; d[1].field = BF_DELTA_PHASE; d[1].code = BF_PHASE_RUNNING;
  d[2].run = 41; d[2].index = 0; d[2].field = BF_DELTA_PHASE; d[2].code = BF_PHASE_FAILED;
  d[3].run = 50; d[3].index = 0; d[3].field = BF_DELTA_RUN_FLAGS; d[3].code = 0;
  CHECK(bfgo_resident_tick_touched(ctx, hT, d, 4, N, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(bfgo_resident_tick_compact(ctx, hC, d, 4, N, BF_EVAL_CHANGED_ONLY, 0, chead, cevents, CAP_EV, &c_events, &c_listed, &kc) == BF_OK);
  CHECK(full == 0 && n_eval == 4 && n_listed == 3 && c_listed == 3 && n_events == c_events);
  CHECK(runs[0] == 3 && runs[1] == 40 && runs[2] == 41);
  CHECK(BF_EVENT_STEP(events[0]) == 1 && BF_EVENT_KIND(events[0]) == BF_EVT_READY);
  CHECK(k.evals == 4 * 3 && k.ready == 2 && k.skip == 1);   /* run 3: B, run 50: A ready; run 41: B skipped */
  CHECK(same_lists(runs, head, events, n_listed, chead, cevents));

  /* deltas through bf_resident_apply count too; a tick without deltas then evaluates their run alone */
  d[0].run = 3; d[0].index = 1; d[0].code = BF_PHASE_SUCCEEDED;
  CHECK(bf_resident_apply(ctx, hT, d, 1) == BF_OK && bf_resident_apply(ctx, hC, d, 1) == BF_OK);
  CHECK(bfgo_resident_tick_touched(ctx, hT, NULL, 0, N, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(bfgo_resident_tick_compact(ctx, hC, NULL, 0, N, BF_EVAL_CHANGED_ONLY, 0, chead, cevents, CAP_EV, &c_events, &c_listed, &kc) == BF_OK);
  CHECK(full == 0 && n_eval == 1 && n_listed == 1 && runs[0] == 3 && BF_EVENT_STEP(events[0]) == 2);
  CHECK(same_lists(runs, head, events, n_listed, chead, cevents));

  /* nothing touched: nothing evaluated, nothing listed */
  CHECK(bfgo_resident_tick_touched(ctx, hT, NULL, 0, N, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(full == 0 && n_eval == 0 && n_listed == 0 && n_events == 0 && k.evals == 0);

  /* an unknown flag is rejected */
  CHECK(bfgo_resident_tick_touched(ctx, hT, NULL, 0, N, BF_EVAL_CHANGED_ONLY, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval,
                                   &n_events, &k) == BF_EINVAL);

  CHECK(bf_resident_destroy(ctx, hT) == BF_OK && bf_resident_destroy(ctx, hC) == BF_OK);
  CHECK(bf_free_pinned(ctx, runs_v) == BF_OK && bf_free_pinned(ctx, head_v) == BF_OK && bf_free_pinned(ctx, ev_v) == BF_OK);
  free(state);
  bf_destroy(ctx);
  printf("c_touched_harness: ok\n");
  return 0;
}
