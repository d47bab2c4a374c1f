/*
 * c_reshape_harness.c — plain C caller of libbobrafrontier.so that performs the call sequence of Resident.Reshape in the cgo binding
 * (go/frontier/frontier.go) through the same flat wrapper (go/frontier/shim.h): a tight batch ticks, grows everything at once
 * (capacity, steps_max, cond planes and a child area), takes runs of a larger Story into the new capacity and deltas, and the next
 * touched tick gives what a batch created at the wide layout from the start gives.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_reshape_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_reshape_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 32, CAP = 64, BIG_S = 40, CAP_EV = 4096 };

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
  /* the small Story: A; B needs A; C needs B; D needs nothing.  The large one: a chain of BIG_S steps.  */
  const uint32_t rp[5] = {0, 0, 1, 2, 2};
  const uint16_t ci[2] = {0, 1};
  const uint8_t fl[4] = {BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t brp[BIG_S + 1];
  uint16_t bci[BIG_S - 1];
  uint8_t bfl[BIG_S];
  brp[0] = 0;
  for (uint32_t i = 0; i < BIG_S; ++i) {
    brp[i + 1] = i;   /* step i needs step i - 1 */
    if (i) bci[i - 1] = (uint16_t)(i - 1);
    bfl[i] = BF_STEP_ENGRAM;
  }
  uint32_t s_small = 99, s_big = 99;
  CHECK(bfgo_topology_put(ctx, 4, 2, rp, ci, fl, NULL, 0, NULL, 0, &s_small) == BF_OK);
  CHECK(bfgo_topology_put(ctx, BIG_S, BIG_S - 1, brp, bci, bfl, NULL, 0, NULL, 0, &s_big) == BF_OK);
  /* the tight batch has decision planes (gates) already: the reshape adds cond planes and a child area, which keeps the next
     touched tick incremental (added decision planes or output fields would make it a full one) */
  const uint32_t tight_fields = BF_F_DECISION | BF_F_OUT_SKIP_DEP, wide_fields = tight_fields | BF_F_COND | BF_F_CHILD;
  bf_layout Lt, Lw;
  CHECK(bf_layout_init(&Lt, 8, 0, tight_fields) == BF_OK);
  CHECK(bf_layout_init(&Lw, 64, 16, wide_fields) == BF_OK);
  uint8_t* tight = (uint8_t*)malloc((size_t)N * Lt.state_stride);
  uint8_t* wide = (uint8_t*)malloc((size_t)CAP * Lw.state_stride);
  uint8_t* back = (uint8_t*)malloc((size_t)CAP * Lw.state_stride);
  uint8_t* back2 = (uint8_t*)malloc((size_t)CAP * Lw.state_stride);
  pack(tight, &Lt, N, s_small, 0);
  pack(wide, &Lw, N, s_small, 0);

  /* 1-2: the tight batch and the wide one, each with its first (full) touched tick */
  uint32_t h = 0, g = 0;
  CHECK(bf_resident_create(ctx, &Lt, N, &h) == BF_OK);
  CHECK(bf_resident_create(ctx, &Lw, CAP, &g) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, tight) == BF_OK);
  CHECK(bf_resident_upload(ctx, g, 0, N, wide) == BF_OK);
  uint32_t runs[2][CAP], head[2][CAP], full[2], n_listed[2], n_eval[2];
  uint16_t events[2][CAP_EV];
  uint64_t n_events[2];
  bf_counts k;
  const uint32_t hg[2] = {h, g};
  for (int i = 0; i < 2; ++i) {
    CHECK(bfgo_resident_tick_touched(ctx, hg[i], NULL, 0, N, 0, 0, runs[i], head[i], CAP, events[i], CAP_EV, &full[i], &n_listed[i],
                                     &n_eval[i], &n_events[i], &k) == BF_OK);
    CHECK(full[i] == 1 && n_listed[i] == N);
  }

  /* 3: a shrinking reshape is rejected and changes nothing; the growing one keeps every record */
  bf_layout L2;
  memset(&L2, 0, sizeof L2);
  CHECK(bfgo_resident_reshape(ctx, h, 8, 0, tight_fields, N - 1, &L2) == BF_EINVAL);
  CHECK(bf_resident_download(ctx, h, 0, N, back) == BF_OK && memcmp(back, tight, (size_t)N * Lt.state_stride) == 0);
  CHECK(bfgo_resident_reshape(ctx, h, 64, 16, wide_fields, CAP, &L2) == BF_OK);
  CHECK(memcmp(&L2, &Lw, sizeof Lw) == 0);
  CHECK(bf_resident_download(ctx, h, 0, CAP, back) == BF_OK && bf_resident_download(ctx, g, 0, CAP, back2) == BF_OK);
  CHECK(memcmp(back, back2, (size_t)CAP * Lw.state_stride) == 0);

  /* 4: runs of the larger Story in the added capacity, step 0 Succeeded */
  pack(wide + (size_t)N * Lw.state_stride, &Lw, 16, s_big, 3);
  for (int i = 0; i < 2; ++i) CHECK(bf_resident_upload(ctx, hg[i], N, 16, wide + (size_t)N * Lw.state_stride) == BF_OK);

  /* 5-6: deltas (one on a cond plane the tight layout did not have) and the touched tick */
  bf_delta d[3];
  memset(d, 0, sizeof d);
  d[0].run = 0; d[0].index = 0; d[0].field = BF_DELTA_PHASE; d[0].code = 3;     /* A Succeeded: B becomes ready       */
  d[1].run = 2; d[1].index = 3; d[1].field = BF_DELTA_COND; d[1].code = BF_COND_PASS;   /* touched, result unchanged */
  d[2].run = 33; d[2].index = 1; d[2].field = BF_DELTA_PHASE; d[2].code = 3;    /* chain step 1 Succeeded             */
  for (int i = 0; i < 2; ++i)
    CHECK(bfgo_resident_tick_touched(ctx, hg[i], d, 3, N + 16, 0, 0, runs[i], head[i], CAP, events[i], CAP_EV, &full[i], &n_listed[i],
                                     &n_eval[i], &n_events[i], &k) == BF_OK);
  CHECK(full[0] == 0 && n_eval[0] == 18 && n_listed[0] == 17);   /* runs 0, 2 and the 16 uploaded; run 2 is not listed */
  CHECK(full[1] == full[0] && n_eval[1] == n_eval[0] && n_listed[1] == n_listed[0] && n_events[1] == n_events[0]);
  CHECK(memcmp(runs[0], runs[1], n_listed[0] * 4) == 0 && memcmp(head[0], head[1], n_listed[0] * 4) == 0);
  CHECK(memcmp(events[0], events[1], n_events[0] * 2) == 0);
  CHECK(runs[0][0] == 0 && runs[0][1] == N && BF_EVENT_STEP(events[0][0]) == 1 && BF_EVENT_KIND(events[0][0]) == BF_EVT_READY);
  CHECK(bf_resident_download(ctx, h, 0, CAP, back) == BF_OK && bf_resident_download(ctx, g, 0, CAP, back2) == BF_OK);
  CHECK(memcmp(back, back2, (size_t)CAP * Lw.state_stride) == 0);

  CHECK(bf_resident_destroy(ctx, h) == BF_OK && bf_resident_destroy(ctx, g) == BF_OK);
  free(tight); free(wide); free(back); free(back2);
  bf_destroy(ctx);
  printf("c_reshape_harness: ok\n");
  return 0;
}
