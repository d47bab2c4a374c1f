/*
 * c_migrate_harness.c — plain C caller of libbobrafrontier.so that performs the call sequence of Resident.Migrate in the cgo binding
 * (go/frontier/frontier.go) through the same flat wrapper (go/frontier/shim.h): a Story is edited while its runs are live, the new
 * generation is put, the runs move to it, and the next touched tick lists them.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_migrate_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_migrate_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
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
  /* generation 1: A; B needs A; C needs B.  Generation 2: B needs A; A; D (new); C needs B.  */
  const uint32_t rp1[4] = {0, 0, 1, 2};
  const uint16_t ci1[2] = {0, 1};
  const uint8_t fl1[3] = {BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  const uint32_t rp2[5] = {0, 1, 1, 1, 2};
  const uint16_t ci2[2] = {1, 0};
  const uint8_t fl2[4] = {BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t s_old = 99, s_other = 99, s_new = 99;
  CHECK(bfgo_topology_put(ctx, 3, 2, rp1, ci1, fl1, NULL, 0, NULL, 0, &s_old) == BF_OK);
  CHECK(bfgo_topology_put(ctx, 3, 2, rp1, ci1, fl1, NULL, 0, NULL, 0, &s_other) == BF_OK);   /* another Story, same shape */
  CHECK(bfgo_topology_put(ctx, 4, 2, rp2, ci2, fl2, NULL, 0, NULL, 0, &s_new) == BF_OK);
  bf_layout L;
  CHECK(bf_layout_init(&L, 4, 0, BF_F_OUT_SKIP_DEP) == BF_OK);
  uint8_t* state = (uint8_t*)calloc(N, L.state_stride);
  uint8_t* back = (uint8_t*)calloc(N, L.state_stride);
  for (uint32_t r = 0; r < N; ++r) {   /* even runs on the edited Story: A Succeeded, B Running */
    uint8_t* rec = state + (size_t)r * L.state_stride;
    ((bf_run_header*)rec)->topo_slot = (r % 2) ? s_other : s_old;
    uint32_t* ph = (uint32_t*)(rec + L.off_phase);
    ph[0 * L.words] |= 1u << 0; ph[1 * L.words] |= 1u << 0;   /* step 0: code 3 */
    ph[1 * L.words] |= 1u << 1;                               /* step 1: code 2 */
  }
  uint32_t h = 0;
  CHECK(bf_resident_create(ctx, &L, N, &h) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, state) == BF_OK);
  uint32_t runs[N], head[N], full = 9, n_listed = 0, n_eval = 0;
  uint16_t events[CAP_EV];
  uint64_t n_events = 0;
  bf_counts k;
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(full == 1 && n_listed == N);

  /* the map by name: A -> 1, B -> 0, C -> 3; a map that is not injective is rejected and changes nothing */
  const uint16_t bad[3] = {1, 1, 3};
  uint32_t migrated = 77;
  CHECK(bfgo_resident_migrate(ctx, h, s_old, s_new, bad, 3, N, &migrated) == BF_EINVAL);
  CHECK(bf_resident_download(ctx, h, 0, N, back) == BF_OK && memcmp(back, state, (size_t)N * L.state_stride) == 0);
  const uint16_t map[3] = {1, 0, 3};
  CHECK(bfgo_resident_migrate(ctx, h, s_old, s_new, map, 3, N, &migrated) == BF_OK && migrated == N / 2);
  CHECK(bf_resident_download(ctx, h, 0, N, back) == BF_OK);
  for (uint32_t r = 0; r < N; ++r) {
    const uint8_t* rec = back + (size_t)r * L.state_stride;
    if (r % 2) { CHECK(memcmp(rec, state + (size_t)r * L.state_stride, L.state_stride) == 0); continue; }
    CHECK(((const bf_run_header*)rec)->topo_slot == s_new);
    CHECK(phase_of(rec, &L, 0) == BF_PHASE_RUNNING && phase_of(rec, &L, 1) == BF_PHASE_SUCCEEDED);
    CHECK(phase_of(rec, &L, 2) == BF_PHASE_NONE && phase_of(rec, &L, 3) == BF_PHASE_NONE);
  }
  /* the old generation may go now; the next touched tick lists every migrated run (D is ready in each: it needs nothing) */
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs, head, N, events, CAP_EV, &full, &n_listed, &n_eval, &n_events, &k) == BF_OK);
  CHECK(full == 0 && n_listed == N / 2 && n_eval == N / 2 && n_events == N / 2);
  for (uint32_t i = 0; i < N / 2; ++i) {
    CHECK(runs[i] == 2 * i && (head[i] & BF_HEAD_LISTED) && (head[i] >> BF_HEAD_COUNT_SHIFT) == 1);
    CHECK(BF_EVENT_STEP(events[i]) == 2 && BF_EVENT_KIND(events[i]) == BF_EVT_READY);
  }
  CHECK(bf_topology_drop(ctx, s_old) == BF_OK);

  CHECK(bf_resident_destroy(ctx, h) == BF_OK);
  free(state);
  free(back);
  bf_destroy(ctx);
  printf("c_migrate_harness: ok\n");
  return 0;
}
