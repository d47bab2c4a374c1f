/*
 * c_transfer_harness.c — plain C caller of libbobrafrontier.so that performs the call sequence of Resident.TransferTo in the cgo
 * binding (go/frontier/frontier.go) through the same flat wrapper (go/frontier/shim.h): a batch of the wide class holds runs of a
 * small Story; a run holding a cond code the narrow class has no plane for is refused and nothing changes; three runs move to the
 * narrow class, the wide batch compacts by the retire rule, and the next touched tick of each batch is incremental and lists the
 * runs that moved.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_transfer_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_transfer_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 32, CAP_EV = 4096 };

/* records of n runs on `slot` at layout L, every code 0 */
static void pack(uint8_t* rec, const bf_layout* L, uint32_t n, uint32_t slot) {
  memset(rec, 0, (size_t)n * L->state_stride);
  for (uint32_t r = 0; r < n; ++r) ((bf_run_header*)(rec + (size_t)r * L->state_stride))->topo_slot = slot;
}

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  /* the Story: A; B needs A; C needs B; D needs nothing */
  const uint32_t rp[5] = {0, 0, 1, 2, 2};
  const uint16_t ci[2] = {0, 1};
  const uint8_t fl[4] = {BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, 4, 2, rp, ci, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  /* two width classes of one ctx: 200 steps with cond planes, 8 steps without */
  bf_layout Lw, Ln;
  CHECK(bf_layout_init(&Lw, 200, 0, BF_F_COND | BF_F_OUT_SKIP_DEP) == BF_OK);
  CHECK(bf_layout_init(&Ln, 8, 0, BF_F_OUT_SKIP_DEP) == BF_OK);
  uint8_t* wide = (uint8_t*)malloc((size_t)N * Lw.state_stride);
  uint8_t* back = (uint8_t*)malloc((size_t)N * Lw.state_stride);
  uint8_t* want = (uint8_t*)malloc((size_t)N * Ln.state_stride);
  pack(wide, &Lw, N, slot);
  uint32_t h = 0, g = 0;
  CHECK(bf_resident_create(ctx, &Lw, N, &h) == BF_OK);
  CHECK(bf_resident_create(ctx, &Ln, N, &g) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, wide) == BF_OK);

  /* 1: the first touched tick of each batch (the narrow one holds no run yet) */
  uint32_t runs[N], head[N], full, n_listed, n_eval;
  uint16_t events[CAP_EV];
  uint64_t n_events;
  bf_counts k;
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(full == 1 && n_listed == N);
  CHECK(bfgo_resident_tick_touched(ctx, g, NULL, 0, 0, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);

  /* 2: run 2 holds a SKIP cond code: its move is refused, names it, and changes nothing */
  bf_delta d;
  memset(&d, 0, sizeof d);
  d.run = 2; d.index = 3; d.field = BF_DELTA_COND; d.code = BF_COND_SKIP;
  CHECK(bf_resident_apply(ctx, h, &d, 1) == BF_OK);
  CHECK(bf_resident_download(ctx, h, 0, N, wide) == BF_OK);
  uint32_t from[4], to[4], counts[4], why[4];
  const uint32_t bad[2] = {7, 2};
  CHECK(bfgo_resident_transfer(ctx, h, g, N, 0, bad, 2, from, to, counts, why) == BF_EINVAL);
  CHECK(counts[0] == N && counts[1] == 0 && counts[3] == 1 && why[0] == 4 && why[2] == BF_F_COND && why[3] == 2);
  CHECK(bf_resident_download(ctx, h, 0, N, back) == BF_OK && memcmp(back, wide, (size_t)N * Lw.state_stride) == 0);

  /* 3: three runs move; the wide batch compacts by the retire rule (29 -> 0, 30 -> 5) */
  const uint32_t mv[3] = {5, 0, 31};
  CHECK(bfgo_resident_transfer(ctx, h, g, N, 0, mv, 3, from, to, counts, why) == BF_OK);
  CHECK(counts[0] == N - 3 && counts[1] == 3 && counts[2] == 2 && counts[3] == BF_EXTENT_NO_RUN);
  CHECK(from[0] == 29 && to[0] == 0 && from[1] == 30 && to[1] == 5);
  pack(want, &Ln, 3, slot);
  CHECK(bf_resident_download(ctx, g, 0, 3, back) == BF_OK && memcmp(back, want, (size_t)3 * Ln.state_stride) == 0);

  /* 4: the next touched tick of each batch: incremental; the narrow one lists its three arrivals, the wide one its moved runs */
  CHECK(bfgo_resident_tick_touched(ctx, g, NULL, 0, 3, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(full == 0 && n_listed == 3 && runs[0] == 0 && runs[1] == 1 && runs[2] == 2);
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N - 3, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(full == 0 && n_listed >= 2 && runs[0] == 0);

  CHECK(bf_resident_destroy(ctx, h) == BF_OK && bf_resident_destroy(ctx, g) == BF_OK);
  free(wide); free(back); free(want);
  bf_destroy(ctx);
  printf("c_transfer_harness: ok\n");
  return 0;
}
