/*
 * c_commit_journal_harness.c — plain C caller of libbobrafrontier.so that performs the per-tick loop of the cgo binding with a
 * journaled commit (go/frontier/frontier.go) through the same entry points and flat wrappers (go/frontier/shim.h):
 * Resident.Fire -> TickTouched -> Ctx.ScheduleResident -> (Execute) -> Resident.CommitJournal -> Status(journal runs and done
 * runs) -> Retire.  The Story: S (sleep, 1 unit), E (engram), F (engram) needs E.  Run 0 launches S and E, run 1 launches them
 * too but its Execute fails, run 2 arrives with every step Succeeded.  A refused commit lists nothing and changes nothing; the
 * commit lists run 0's two phase writes and its timer arm, and only run 0 as written.  Status over run 0 and the done run 2
 * reports S and E active in run 0 and run 2 succeeded, and retiring run 2 leaves run 0's record as the commit wrote it.
 *
 *   gcc -O1 -Wall -Iinclude -Igo/frontier tests/c_commit_journal_harness.c -Lbobrapet_b200/lib -lbobrafrontier -Wl,-rpath,... -o harness
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "shim.h"

#define CHECK(cond)                                                                 \
  do {                                                                              \
    if (!(cond)) { fprintf(stderr, "c_commit_journal_harness: FAILED %s (line %d): %s\n", #cond, __LINE__, ctx ? bf_last_error(ctx) : ""); return 1; } \
  } while (0)

enum { N = 3, CAP_EV = 64, CAP_ITEMS = 16, NOW = 100 };

static uint32_t phase_of(const uint8_t* rec, const bf_layout* L, uint32_t step) {
  const uint32_t* ph = (const uint32_t*)(rec + L->off_phase);
  uint32_t code = 0;
  for (uint32_t b = 0; b < 4; ++b) code |= ((ph[b * L->words + step / 32] >> (step % 32)) & 1u) << b;
  return code;
}

static void set_phase(uint8_t* rec, const bf_layout* L, uint32_t step, uint32_t code) {
  uint32_t* ph = (uint32_t*)(rec + L->off_phase);
  for (uint32_t b = 0; b < 4; ++b) {
    uint32_t* w = &ph[b * L->words + step / 32];
    *w = ((code >> b) & 1u) ? *w | 1u << (step % 32) : *w & ~(1u << (step % 32));
  }
}

int main(void) {
  bf_ctx* ctx = NULL;
  CHECK(bfgo_create(0, &ctx) == BF_OK);
  const uint32_t rp[4] = {0, 0, 0, 1};
  const uint16_t ci[1] = {1};
  const uint8_t fl[3] = {BF_STEP_SLEEP, BF_STEP_ENGRAM, BF_STEP_ENGRAM};
  uint32_t slot = 99;
  CHECK(bfgo_topology_put(ctx, 3, 1, rp, ci, fl, NULL, 0, NULL, 0, &slot) == BF_OK);
  bf_step_timing tim;
  memset(&tim, 0, sizeof tim);
  tim.step = 0; tim.code = BF_DEC_SUCCEED; tim.delay = 1;
  CHECK(bfgo_topology_timings(ctx, slot, &tim, 1) == BF_OK);                          /* PutTimings */
  bf_layout L;
  CHECK(bf_layout_init(&L, 32, 0, BF_F_DECISION | BF_F_OUT_FAIL) == BF_OK);
  uint8_t* rec = (uint8_t*)calloc(N, L.state_stride);
  for (uint32_t r = 0; r < N; ++r) ((bf_run_header*)(rec + (size_t)r * L.state_stride))->topo_slot = slot;
  for (uint32_t s = 0; s < 3; ++s) set_phase(rec + 2 * (size_t)L.state_stride, &L, s, BF_PHASE_SUCCEEDED);
  uint32_t h;
  CHECK(bf_resident_create(ctx, &L, N, &h) == BF_OK);
  CHECK(bf_resident_upload(ctx, h, 0, N, rec) == BF_OK);
  CHECK(bf_resident_timers(ctx, h, 2) == BF_OK);                                      /* EnableTimers */
  CHECK(bf_resident_sched(ctx, h) == BF_OK);                                          /* EnableSched */
  bf_sched_put put[N];
  memset(put, 0, sizeof put);
  for (uint32_t r = 0; r < N; ++r) {
    put[r].run = r; put[r].story_key = BF_SCHED_NONE; put[r].queue_key = BF_SCHED_NONE;
    put[r].queued_since = BF_SCHED_NONE; put[r].run_phase = BF_PHASE_RUNNING;
  }
  CHECK(bf_resident_sched_put(ctx, h, put, N) == BF_OK);

  /* Fire -> TickTouched -> ScheduleResident */
  bf_fired fired[8];
  uint32_t fc[5];
  CHECK(bfgo_resident_fire(ctx, h, N, NOW, fired, 8, fc) == BF_OK && fc[0] == 0);
  uint32_t runs_t[N], head_t[N], full, n_listed, n_eval;
  uint16_t ev_t[CAP_EV];
  uint64_t n_ev;
  bf_counts k;
  CHECK(bfgo_resident_tick_touched(ctx, h, NULL, 0, N, 0, 0, runs_t, head_t, N, ev_t, CAP_EV, &full, &n_listed, &n_eval, &n_ev, &k) == BF_OK);
  CHECK(full == 1 && n_listed == N && k.ready == 4);
  uint32_t done[N], n_done = 0;   /* the runs whose group selection found nothing left: the batcher finalizes them */
  for (uint32_t i = 0; i < n_listed; ++i)
    if ((head_t[i] & BF_HEAD_SUMMARY_MASK & BF_SUM_GROUP_MASK) == BF_GROUP_DONE) done[n_done++] = runs_t[i];
  CHECK(n_done == 1 && done[0] == 2);
  uint32_t* runs;
  bf_sched_header* heads;
  uint16_t* events;
  CHECK(bf_alloc_pinned(ctx, N * sizeof(uint32_t), (void**)&runs) == BF_OK);
  CHECK(bf_alloc_pinned(ctx, N * sizeof(bf_sched_header), (void**)&heads) == BF_OK);
  CHECK(bf_alloc_pinned(ctx, CAP_EV * sizeof(uint16_t), (void**)&events) == BF_OK);
  bf_resident_sched_part part;
  bfgo_sched_part(&part, h, N, runs, heads, N, events, CAP_EV);
  uint32_t gr;
  CHECK(bfgo_resident_schedule(ctx, NOW, 0, 0, 0, 0, NULL, NULL, NULL, NULL, NULL, NULL, &part, 1, NULL, NULL, NULL, &gr) == BF_OK);
  CHECK(heads[0].n_launch == 2 && heads[1].n_launch == 2);

  /* CommitJournal: a PHASE entry on an engram step is refused, lists nothing and changes nothing */
  bf_commit_write items[CAP_ITEMS];
  uint32_t written[N], c[10];
  uint64_t n_items = 99;
  bf_commit_entry ents[2];
  memset(ents, 0, sizeof ents);
  ents[0].run = 0; ents[0].step = 1; ents[0].kind = BF_COMMIT_PHASE; ents[0].code = BF_PHASE_SUCCEEDED;
  CHECK(bfgo_resident_commit_journal(ctx, h, N, ents, 1, NOW, items, CAP_ITEMS, written, N, c, &n_items) == BF_EINVAL);
  CHECK(c[5] == 0 && c[6] == 1 && c[9] == 0 && n_items == 0);
  uint8_t* got = (uint8_t*)malloc((size_t)N * L.state_stride);
  CHECK(bf_resident_download(ctx, h, 0, N, got) == BF_OK && memcmp(got, rec, (size_t)N * L.state_stride) == 0);
  /* run 1's Execute failed: nothing of it is written or listed */
  ents[0].run = 1; ents[0].step = 1; ents[0].kind = BF_COMMIT_ERROR; ents[0].code = 0;
  CHECK(bfgo_resident_commit_journal(ctx, h, N, ents, 1, NOW, items, CAP_ITEMS, written, N, c, &n_items) == BF_OK);
  CHECK(c[0] == 1 && c[2] == 2 && c[7] == 1 && c[8] == NOW + 1 && c[9] == 1 && written[0] == 0 && n_items == 3);
  CHECK(items[0].run == 0 && items[0].field == BF_DELTA_PHASE && items[0].index == 0 && items[0].before == 0 && items[0].after == BF_PHASE_PAUSED);
  CHECK(items[1].run == 0 && items[1].field == BF_DELTA_PHASE && items[1].index == 1 && items[1].before == 0 && items[1].after == BF_PHASE_RUNNING);
  CHECK(items[2].run == 0 && items[2].field == BF_COMMIT_WRITE_TIMER && items[2].index == 0 && items[2].code == BF_DEC_SUCCEED &&
        items[2].before == BF_TIMER_NONE && items[2].after == NOW + 1);
  CHECK(bf_resident_download(ctx, h, 0, N, got) == BF_OK);
  CHECK(phase_of(got, &L, 0) == BF_PHASE_PAUSED && phase_of(got, &L, 1) == BF_PHASE_RUNNING && phase_of(got, &L, 2) == 0);
  CHECK(memcmp(got + L.state_stride, rec + L.state_stride, 2 * (size_t)L.state_stride) == 0);

  /* Status over the journal's runs and the done runs (ascending), then Retire the done run */
  const uint32_t status_runs[2] = {written[0], done[0]};
  bf_status_rec st[2];
  uint16_t sev[CAP_EV];
  uint64_t n_sev;
  CHECK(bfgo_resident_status(ctx, h, N, status_runs, 2, st, sev, CAP_EV, &n_sev) == BF_OK);
  CHECK(st[0].run == 0 && st[0].outcome == BF_OUTCOME_NONE && st[0].active == 2 && st[0].completed == 0);
  CHECK(st[1].run == 2 && st[1].outcome == BF_OUTCOME_SUCCEEDED && st[1].story_phase == BF_PHASE_SUCCEEDED && st[1].completed == 3);
  uint32_t from[1], to[1], n_out, n_moves;
  CHECK(bfgo_resident_retire(ctx, h, N, done, n_done, 0, from, to, &n_out, &n_moves) == BF_OK && n_out == 2 && n_moves == 0);
  CHECK(bf_resident_download(ctx, h, 0, 1, got + 2 * (size_t)L.state_stride) == BF_OK);
  CHECK(memcmp(got, got + 2 * (size_t)L.state_stride, L.state_stride) == 0);

  free(got);
  CHECK(bf_free_pinned(ctx, runs) == BF_OK && bf_free_pinned(ctx, heads) == BF_OK && bf_free_pinned(ctx, events) == BF_OK);
  CHECK(bf_resident_destroy(ctx, h) == BF_OK);
  free(rec);
  bf_destroy(ctx);
  printf("c_commit_journal_harness: ok\n");
  return 0;
}
