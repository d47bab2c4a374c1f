/*
 * c_resync_areas_harness.c — plain C caller of libbobrafrontier.so that performs the call sequence of the cgo binding
 * (go/frontier/frontier.go) through the same entry points and flat wrappers (go/frontier/shim.h) for a side-area resync:
 * Resident.Fire -> TickTouched -> Resync (the records agree) -> ResyncAreas, then a Fire that fires the slot the resync re-armed.
 * The Story: A (engram), B (sleep), C (engram) needs B.  Both runs: A Succeeded, B Paused with decision PENDING.
 *   run 0: the sleep's arm was lost: the device has no slot, the step-timers annotation has B due at 5.  No fire and no tick lists
 *          the run (the stuck step); the resync re-arms B, the next Fire writes SUCCEED and the next tick readies C.
 *   run 1: armed on both sides; the cluster has spec.cancelRequested, which the device missed: the resync stops the run.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_resync_areas_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_resync_areas_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 2, S = 3, K = 2, CAP_EV = 64, CAP_ITEMS = 16 };

static void set_code(uint8_t* rec, uint32_t off, uint32_t words, uint32_t nbits, uint32_t step, uint32_t code) {
  uint32_t* pl = (uint32_t*)(rec + off);
  for (uint32_t b = 0; b < nbits; ++b) {
    uint32_t* w = &pl[b * words + step / 32];
    *w = ((code >> b) & 1u) ? (*w | (1u << (step % 32))) : (*w & ~(1u << (step % 32)));
  }
}

static void empty_slots(bf_timer_slot* row) {
  memset(row, 0, K * sizeof *row);
  for (uint32_t k = 0; k < K; ++k) row[k].deadline = BF_TIMER_NONE;
}

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  const uint32_t rp[S + 1] = {0, 0, 0, 1};
  const uint16_t ci[1] = {1};
  const uint8_t fl[S] = {BF_STEP_ENGRAM, BF_STEP_SLEEP, BF_STEP_ENGRAM};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, S, 1, rp, ci, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  bf_layout L;
  CHECK(bf_layout_init(&L, 32, 0, BF_F_DECISION | BF_F_OUT_FAIL | BF_F_OUT_PHASE) == BF_OK);
  uint8_t* rec = (uint8_t*)calloc(N, L.state_stride);
  for (uint32_t r = 0; r < N; ++r) {
    uint8_t* x = rec + (size_t)r * L.state_stride;
    ((bf_run_header*)x)->topo_slot = slot;
    set_code(x, L.off_phase, L.words, 4, 0, BF_PHASE_SUCCEEDED);
    set_code(x, L.off_phase, L.words, 4, 1, BF_PHASE_PAUSED);
  }
  uint32_t h;
  CHECK(bf_resident_create(ctx, &L, N, &h) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, rec) == BF_OK);
  CHECK(bf_resident_timers(ctx, h, K) == BF_OK);                                      /* EnableTimers */
  CHECK(bf_resident_runctl(ctx, h) == BF_OK);                                         /* EnableRunCtl */
  bf_timer t;
  memset(&t, 0, sizeof t);
  t.run = 1; t.step = 1; t.code = BF_DEC_SUCCEED; t.deadline = 50;
  CHECK(bf_resident_timers_arm(ctx, h, &t, 1) == BF_OK);                              /* run 0's arm is lost */

  /* Fire -> TickTouched: nothing is due on the device, and run 0 waits for good */
  bf_fired fired[4];
  uint32_t fc[5];
  CHECK(bfgo_resident_fire(ctx, h, N, 5, fired, 4, fc) == BF_OK && fc[0] == 0);
  uint32_t runs_t[N], head_t[N], full, n_listed, n_eval;
  uint16_t ev_t[CAP_EV];
  uint64_t n_ev;
  bf_counts k;
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, CAP_EV, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  CHECK(full == 1 && k.ready == 0);

  /* Resync: the records the batcher packs from the cluster agree */
  uint8_t* dev = (uint8_t*)malloc((size_t)N * L.state_stride);
  CHECK(bf_resident_download(ctx, h, 0, N, dev) == BF_OK);
  uint32_t drifted[N], n_drifted, n_written, bad_run;
  bf_drift items[CAP_ITEMS];
  uint64_t n_items;
  CHECK(bfgo_resident_resync(ctx, h, N, NULL, N, dev, BF_RESYNC_ALL_FIELDS, BF_RESYNC_CHECK, drifted, N, items, CAP_ITEMS,
                             &n_drifted, &n_written, &n_items, &bad_run) == BF_OK && n_items == 0);

  /* ResyncAreas: the annotation (run 0: B due at 5; run 1: B at 50) and the run control (run 1 cancel-requested), with the now of
   * the last Fire.  Run 0's slot is due but B is still undecided on the device: the stuck step, listed and re-armed.  Run 1 lists
   * its stop and compares no timers (the stop empties them). */
  bf_timer_slot slots[N * K];
  empty_slots(slots);
  empty_slots(slots + K);
  slots[0].deadline = 5; slots[0].step = 1; slots[0].code = BF_DEC_SUCCEED;
  slots[K].deadline = 50; slots[K].step = 1; slots[K].code = BF_DEC_SUCCEED;
  bf_run_ctl ctl[N];
  memset(ctl, 0, sizeof ctl);
  for (uint32_t r = 0; r < N; ++r) ctl[r].story_deadline = ctl[r].drain_deadline = BF_TIMER_NONE;
  ctl[1].stop = BF_STOP_CANCEL;
  const uint32_t areas = BF_RESYNC_AREA_TIMERS | BF_RESYNC_AREA_RUNCTL;
  CHECK(bfgo_resident_resync_areas(ctx, h, N, NULL, N, areas, slots, NULL, ctl, 5, BF_RESYNC_CHECK, drifted, N, items, CAP_ITEMS,
                                   &n_drifted, &n_written, &n_items, &bad_run) == BF_OK);
  CHECK(n_items == 2 && n_drifted == 2 && n_written == 0);
  CHECK(items[0].run == 0 && items[0].index == 1 && items[0].field == BF_DRIFT_TIMER && items[0].device == BF_TIMER_NONE &&
        items[0].record == 5);
  CHECK(items[1].run == 1 && items[1].field == BF_DRIFT_STOP && items[1].device == BF_STOP_NONE && items[1].record == BF_STOP_CANCEL);
  CHECK(bfgo_resident_resync_areas(ctx, h, N, NULL, N, areas, slots, NULL, ctl, 5, 0, drifted, N, items, CAP_ITEMS, &n_drifted,
                                   &n_written, &n_items, &bad_run) == BF_OK);
  CHECK(n_items == 2 && n_drifted == 2 && n_written == 2 && drifted[0] == 0 && drifted[1] == 1);
  bf_timer_slot got[N * K];
  CHECK(bf_resident_timers_download(ctx, h, 0, N, got) == BF_OK);
  CHECK(got[0].deadline == 5 && got[0].step == 1 && got[1].deadline == BF_TIMER_NONE && got[K].deadline == BF_TIMER_NONE);
  bf_run_ctl area[N];
  CHECK(bf_resident_runctl_download(ctx, h, 0, N, area) == BF_OK && area[1].stop == BF_STOP_CANCEL && area[0].stop == BF_STOP_NONE);

  /* the next Fire fires the re-armed sleep, and the next tick readies C of run 0 (run 1 is stopped: no candidates) */
  CHECK(bfgo_resident_fire(ctx, h, N, 5, fired, 4, fc) == BF_OK && fc[0] == 1 && fc[1] == 1);
  CHECK(fired[0].run == 0 && fired[0].step == 1 && fired[0].code == BF_DEC_SUCCEED && fired[0].written == 1);
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, CAP_EV, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  CHECK(full == 0 && n_eval == 2 && k.ready == 1);
  uint32_t c_ready = 0;
  for (uint64_t e = 0; e < n_ev && e < CAP_EV; ++e)
    if (BF_EVENT_STEP(ev_t[e]) == 2 && (BF_EVENT_KIND(ev_t[e]) & BF_EVT_READY)) ++c_ready;
  CHECK(c_ready == 1);
  /* repaired: a check lists nothing more; a caller row naming another run is refused and names its run */
  CHECK(bfgo_resident_resync_areas(ctx, h, N, NULL, N, BF_RESYNC_AREA_RUNCTL, NULL, NULL, ctl, 5, BF_RESYNC_CHECK, drifted, N,
                                   items, CAP_ITEMS, &n_drifted, &n_written, &n_items, &bad_run) == BF_OK && n_items == 0);
  ctl[0].saved_flags = 1;
  CHECK(bfgo_resident_resync_areas(ctx, h, N, NULL, N, BF_RESYNC_AREA_RUNCTL, NULL, NULL, ctl, 5, 0, drifted, N, items,
                                   CAP_ITEMS, &n_drifted, &n_written, &n_items, &bad_run) == BF_EINVAL && bad_run == 0);

  free(dev);
  CHECK(bf_resident_destroy(ctx, h) == BF_OK);
  free(rec);
  bf_destroy(ctx);
  printf("c_resync_areas_harness: ok\n");
  return 0;
}
