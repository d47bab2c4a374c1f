/*
 * c_narrow_harness.c — plain C caller of libbobrafrontier.so that performs the call sequence of Resident.Extent and Resident.Narrow
 * in the cgo binding (go/frontier/frontier.go) through the same flat wrappers (go/frontier/shim.h): a batch laid out for wide
 * Stories holds only small ones, reports its extent, refuses a narrow below it, narrows to the extent's width without its all-PASS
 * cond planes, and the next touched tick gives what a batch created at the narrow layout from the start gives.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_narrow_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_narrow_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 32, CAP_EV = 4096 };

/* records of n runs on `slot` at layout L, phase code `code` at step 0 (everything else 0) */
static void pack(uint8_t* rec, const bf_layout* L, uint32_t n, uint32_t slot, uint32_t code) {
  memset(rec, 0, (size_t)n * L->state_stride);
  for (uint32_t r = 0; r < n; ++r) {
    uint8_t* p = rec + (size_t)r * L->state_stride;
    ((bf_run_header*)p)->topo_slot = slot;
    uint32_t* ph = (uint32_t*)(p + L->off_phase);
    for (uint32_t b = 0; b < 4; ++b)
      if ((code >> b) & 1u) ph[b * L->words] |= 1u;
  }
}

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  /* the Story: A; B needs A; C needs B; D needs nothing */
  const uint32_t rp[5] = {0, 0, 1, 2, 2};
  const uint16_t ci[2] = {0, 1};
  const uint8_t fl[4] = {BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t s_small = 99;
  CHECK(bfgo_topology_put(ctx, 4, 2, rp, ci, fl, NULL, 0, NULL, 0, &s_small) == BF_OK);
  /* the wide batch once held 200-step Stories with `if` steps; its runs now all hold the 4-step Story and every cond code is
     PASS, so it narrows to 8 steps without cond planes, which keeps the next touched tick incremental */
  const uint32_t tight_fields = BF_F_DECISION | BF_F_OUT_SKIP_DEP, wide_fields = tight_fields | BF_F_COND;
  bf_layout Lt, Lw;
  CHECK(bf_layout_init(&Lt, 8, 0, tight_fields) == BF_OK);
  CHECK(bf_layout_init(&Lw, 200, 0, wide_fields) == BF_OK);
  uint8_t* tight = (uint8_t*)malloc((size_t)N * Lt.state_stride);
  uint8_t* wide = (uint8_t*)malloc((size_t)N * Lw.state_stride);
  uint8_t* back = (uint8_t*)malloc((size_t)N * Lw.state_stride);
  uint8_t* back2 = (uint8_t*)malloc((size_t)N * Lw.state_stride);
  pack(tight, &Lt, N, s_small, 0);
  pack(wide, &Lw, N, s_small, 0);

  /* 1-2: the wide batch and a tight twin, each with its first (full) touched tick */
  uint32_t h = 0, g = 0;
  CHECK(bf_resident_create(ctx, &Lw, N, &h) == BF_OK);
  CHECK(bf_resident_create(ctx, &Lt, N, &g) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, wide) == BF_OK);
  CHECK(bf_resident_upload(ctx, g, 0, N, tight) == BF_OK);
  uint32_t runs[2][N], head[2][N], full[2], n_listed[2], n_eval[2];
  uint16_t events[2][CAP_EV];
  uint64_t n_events[2];
  bf_counts k;
  const uint32_t hg[2] = {h, g};
  for (int i = 0; i < 2; ++i) {
    CHECK(bfgo_resident_tick_touched(ctx, hg[i], NULL, 0, N, 0, 0, runs[i], head[i], N, events[i], CAP_EV, &full[i], &n_listed[i],
                                     &n_eval[i], &n_events[i], &k) == BF_OK);
    CHECK(full[i] == 1 && n_listed[i] == N);
  }

  /* 3: the extent: 4 steps (the Story), no input field in use, run 0 the first that needs them */
  uint32_t ext[4];
  CHECK(bfgo_resident_extent(ctx, h, N, ext) == BF_OK);
  CHECK(ext[0] == 4 && ext[1] == 0 && ext[2] == 0 && ext[3] == 0);

  /* 4: a narrow below the extent is rejected, reports the extent and changes nothing; the one above it keeps every code */
  bf_layout L2;
  memset(&L2, 0, sizeof L2);
  memset(ext, 0, sizeof ext);
  CHECK(bfgo_resident_narrow(ctx, h, 3, 0, tight_fields, N, ext, &L2) == BF_EINVAL);
  CHECK(ext[0] == 4 && ext[3] == 0);
  CHECK(bf_resident_download(ctx, h, 0, N, back) == BF_OK && memcmp(back, wide, (size_t)N * Lw.state_stride) == 0);
  CHECK(bfgo_resident_narrow(ctx, h, 8, 0, tight_fields, N, ext, &L2) == BF_OK);
  CHECK(memcmp(&L2, &Lt, sizeof Lt) == 0);
  CHECK(bf_resident_download(ctx, h, 0, N, back) == BF_OK && bf_resident_download(ctx, g, 0, N, back2) == BF_OK);
  CHECK(memcmp(back, back2, (size_t)N * Lt.state_stride) == 0);

  /* 5-6: deltas and the touched tick: incremental, and what the tight twin gives */
  bf_delta d[2];
  memset(d, 0, sizeof d);
  d[0].run = 0; d[0].index = 0; d[0].field = BF_DELTA_PHASE; d[0].code = 3;       /* A Succeeded: B becomes ready */
  d[1].run = 5; d[1].index = 3; d[1].field = BF_DELTA_DECISION; d[1].code = BF_DEC_PENDING;   /* touched, result unchanged */
  for (int i = 0; i < 2; ++i)
    CHECK(bfgo_resident_tick_touched(ctx, hg[i], d, 2, N, 0, 0, runs[i], head[i], N, events[i], CAP_EV, &full[i], &n_listed[i],
                                     &n_eval[i], &n_events[i], &k) == BF_OK);
  CHECK(full[0] == 0 && n_eval[0] == 2 && n_listed[0] == 1);
  CHECK(full[1] == full[0] && n_eval[1] == n_eval[0] && n_listed[1] == n_listed[0] && n_events[1] == n_events[0]);
  CHECK(memcmp(runs[0], runs[1], n_listed[0] * 4) == 0 && memcmp(head[0], head[1], n_listed[0] * 4) == 0);
  CHECK(memcmp(events[0], events[1], n_events[0] * 2) == 0);
  CHECK(runs[0][0] == 0 && BF_EVENT_STEP(events[0][0]) == 1 && BF_EVENT_KIND(events[0][0]) == BF_EVT_READY);

  CHECK(bf_resident_destroy(ctx, h) == BF_OK && bf_resident_destroy(ctx, g) == BF_OK);
  free(tight); free(wide); free(back); free(back2);
  bf_destroy(ctx);
  printf("c_narrow_harness: ok\n");
  return 0;
}
