/*
 * c_retire_harness.c — plain C caller of libbobrafrontier.so that performs the call sequence of Resident.Retire in the cgo binding
 * (go/frontier/frontier.go) through the same flat wrapper (go/frontier/shim.h): a batch ticks, retires four runs while shrinking its
 * capacity, reports the moves of the rule, and its next touched tick lists the moved runs and leaves the records a batch uploaded
 * in the new order holds.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_retire_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_retire_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 32, CAP = 40, NEW_CAP = 30, M = 28, CAP_EV = 4096 };

/* the record of run r (of the original order): step k Succeeded when bit k of r is set */
static void pack(uint8_t* p, const bf_layout* L, uint32_t slot, uint32_t r) {
  memset(p, 0, L->state_stride);
  ((bf_run_header*)p)->topo_slot = slot;
  uint32_t* ph = (uint32_t*)(p + L->off_phase);
  for (uint32_t k = 0; k < 4; ++k)
    if ((r >> k) & 1u) { ph[0] |= 1u << k; ph[L->words] |= 1u << k; }   /* code 3 = bits 0 and 1 */
}

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  /* A; B needs A; C needs B; D needs nothing */
  const uint32_t rp[5] = {0, 0, 1, 2, 2};
  const uint16_t ci[2] = {0, 1};
  const uint8_t fl[4] = {BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, 4, 2, rp, ci, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  bf_layout L;
  CHECK(bf_layout_init(&L, 8, 0, BF_F_DECISION | BF_F_OUT_SKIP_DEP) == BF_OK);
  uint8_t* rec = (uint8_t*)calloc(CAP, L.state_stride);
  uint8_t* want = (uint8_t*)calloc(CAP, L.state_stride);
  uint8_t* back = (uint8_t*)calloc(CAP, L.state_stride);
  for (uint32_t r = 0; r < N; ++r) pack(rec + (size_t)r * L.state_stride, &L, slot, r);

  /* 1: the batch and its first (full) touched tick */
  uint32_t h = 0, g = 0;
  CHECK(bf_resident_create(ctx, &L, CAP, &h) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, rec) == BF_OK);
  uint32_t runs[CAP], head[CAP], full = 0, n_listed = 0, n_eval = 0;
  uint16_t events[CAP_EV];
  uint64_t n_events = 0;
  bf_counts k;
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs, head, CAP, events, CAP_EV, &full, &n_listed, &n_eval,
                                   &n_events, &k) == BF_OK);
  CHECK(full == 1 && n_listed == N);

  /* 2: a rejected call (a run named twice) changes nothing */
  uint32_t from[4], to[4], n_runs = 0, n_moves = 0;
  const uint32_t twice[2] = {3, 3};
  CHECK(bfgo_resident_retire(ctx, h, N, twice, 2, 0, from, to, &n_runs, &n_moves) == BF_EINVAL);
  CHECK(n_runs == N && n_moves == 0);
  CHECK(bf_resident_download(ctx, h, 0, N, back) == BF_OK && memcmp(back, rec, (size_t)N * L.state_stride) == 0);

  /* 3: retire 30, 5, 29 and 1, the capacity shrinks to 30: runs 28 and 31 move into 1 and 5 */
  const uint32_t gone[4] = {30, 5, 29, 1};
  CHECK(bfgo_resident_retire(ctx, h, N, gone, 4, NEW_CAP, from, to, &n_runs, &n_moves) == BF_OK);
  CHECK(n_runs == M && n_moves == 2 && from[0] == 28 && to[0] == 1 && from[1] == 31 && to[1] == 5);
  memcpy(want, rec, (size_t)M * L.state_stride);
  memcpy(want + 1 * L.state_stride, rec + 28 * L.state_stride, L.state_stride);
  memcpy(want + 5 * L.state_stride, rec + 31 * L.state_stride, L.state_stride);
  CHECK(bf_resident_download(ctx, h, 0, NEW_CAP, back) == BF_OK && memcmp(back, want, (size_t)NEW_CAP * L.state_stride) == 0);
  CHECK(bf_resident_download(ctx, h, 0, NEW_CAP + 1, back) == BF_EINVAL);

  /* 4: a twin uploaded in the new order; a delta on an unmoved run; the touched tick lists it and both moved runs */
  CHECK(bf_resident_create(ctx, &L, NEW_CAP, &g) == BF_OK);
  CHECK(bf_resident_upload(ctx, g, 0, M, want) == BF_OK);
  bf_delta d;
  memset(&d, 0, sizeof d);
  d.run = 0; d.index = 0; d.field = BF_DELTA_PHASE; d.code = 3;   /* run 0: A Succeeded, B becomes ready */
  CHECK(bfgo_resident_tick_touched(ctx, h, &d, 1, M, 0, 0, runs, head, CAP, events, CAP_EV, &full, &n_listed, &n_eval,
                                   &n_events, &k) == BF_OK);
  CHECK(full == 0 && n_eval == 3 && n_listed == 3 && runs[0] == 0 && runs[1] == 1 && runs[2] == 5);
  CHECK(bf_resident_apply(ctx, g, &d, 1) == BF_OK);
  uint8_t* back2 = (uint8_t*)calloc(CAP, L.state_stride);
  CHECK(bf_resident_download(ctx, h, 0, M, back) == BF_OK && bf_resident_download(ctx, g, 0, M, back2) == BF_OK);
  CHECK(memcmp(back, back2, (size_t)M * L.state_stride) == 0);

  CHECK(bf_resident_destroy(ctx, h) == BF_OK && bf_resident_destroy(ctx, g) == BF_OK);
  free(rec); free(want); free(back); free(back2);
  bf_destroy(ctx);
  printf("c_retire_harness: ok\n");
  return 0;
}
