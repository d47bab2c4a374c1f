// resident_abi.cu — the C ABI of include/bobrafrontier.h for resident batches (row f2): a batch's records stay on the device
// between ticks; uploads, deltas, migrations, redrives, reshapes and retirements change them in place, and full, compact,
// changed-only and touched ticks evaluate them.  The bookkeeping of touched ticks lives in Resident (ctx.h).
#include <stdlib.h>
#include <string.h>

#include <unordered_map>

#include "ctx.h"

using bf::cuda_fail; using bf::fail; using bf::round_up_sz;

// the bf_resident_* definitions take their C linkage from include/bobrafrontier.h
// ---- resident batches (row f2: incremental state upload) --------------------------------------------------
// The ctx lock, which the caller holds for the call, and the live batch of handle h.  The batch is nullptr for a null ctx (no
// lock then) and for an unknown handle (its error set; an argument check that fails after this one sets its own instead).
static std::pair<std::unique_lock<std::mutex>, Resident*> lock_resident(bf_ctx* c, uint32_t h) {
  if (!c) return {};
  std::unique_lock<std::mutex> g(c->mu);
  Resident* r = h < c->resident.size() && c->resident[h].alive ? &c->resident[h] : nullptr;
  if (!r) fail(c, BF_EINVAL, "unknown resident batch");
  return {std::move(g), r};
}

int bf_resident_create(bf_ctx* c, const bf_layout* L, uint32_t capacity, uint32_t* handle_out) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  if (!L || !handle_out || capacity == 0) return fail(c, BF_EINVAL, "null layout / handle or zero capacity");
  if (int rc = bf::check_layout(c, *L)) return rc;
  BF_CUDA(c, cudaSetDevice(c->device));
  Resident r;
  cudaError_t e = r.alloc(*L, capacity);
  if (e == cudaSuccess) e = cudaMemsetAsync(r.d_state, 0, (size_t)capacity * L->state_stride, c->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(r.d_mark, 0, r.d_mark.cap * sizeof(uint32_t), c->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  if (e != cudaSuccess) return fail(c, BF_ENOMEM, std::string("resident batch: ") + cudaGetErrorString(e));
  r.L = *L; r.cap = capacity; r.alive = true;
  uint32_t h = 0;
  while (h < c->resident.size() && c->resident[h].alive) ++h;
  if (h == c->resident.size()) c->resident.push_back(std::move(r)); else c->resident[h] = std::move(r);
  *handle_out = h;
  return BF_OK;
}

int bf_resident_destroy(bf_ctx* c, uint32_t h) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaStreamSynchronize(c->stream);
  r->end_snapshot(c);
  *r = Resident();
  return BF_OK;
}

int bf_resident_upload(bf_ctx* c, uint32_t h, uint32_t first, uint32_t n, const void* records) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if ((uint64_t)first + n > r->cap || (n && !records)) return fail(c, BF_EINVAL, "run range outside the resident batch");
  if (n == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  r->end_snapshot(c);
  r->prev_valid = false;   // full records arrived: the next changed-only tick lists every run
  BF_CUDA(c, cudaMemcpyAsync(r->d_state + (size_t)first * r->L.state_stride, records, (size_t)n * r->L.state_stride, cudaMemcpyHostToDevice, c->stream));
  BF_CUDA(c, bf::launch_mark_runs(r->d_mark, first, n, r->mark_must_list(), c->stream));
  c->stats.kernel_launches += 1;
  r->pending += n;
  r->note_uploaded(first, first + n);
  BF_CUDA(c, cudaStreamSynchronize(c->stream));
  return BF_OK;
}

int bf_resident_download(bf_ctx* c, uint32_t h, uint32_t first, uint32_t n, void* records) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if ((uint64_t)first + n > r->cap || (n && !records)) return fail(c, BF_EINVAL, "run range outside the resident batch");
  if (n == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  BF_CUDA(c, cudaMemcpyAsync(records, r->d_state + (size_t)first * r->L.state_stride, (size_t)n * r->L.state_stride, cudaMemcpyDeviceToHost, c->stream));
  BF_CUDA(c, cudaStreamSynchronize(c->stream));
  return BF_OK;
}

// H2D of the deltas + the scatter kernel on the ctx stream, no synchronisation; the rejected counter is read by the caller
static int resident_apply_async(bf_ctx* c, Resident* r, const bf_delta* deltas, uint32_t n) {
  if (int rc = c->d_deltas.ensure(c, n ? n : 1)) return rc;
  if (!c->d_rejected) { BF_CUDA(c, c->d_rejected.alloc(4)); c->rejected_clean = false; }
  cudaStream_t s = c->stream;
  if (!c->rejected_clean) { BF_CUDA(c, cudaMemsetAsync(c->d_rejected, 0, 4, s)); c->rejected_clean = true; }
  if (n == 0) return BF_OK;
  c->rejected_clean = false;   // the scatter kernel may count; whoever reads the counter decides whether it is clean again
  // deltas in pinned host memory are read by the scatter kernel itself over PCIe (one launch instead of a copy and a launch:
  // BF_NO_ZC_DELTAS restores the upload), any other buffer is uploaded first
  const bf_delta* d_src = c->d_deltas;
  bool direct = false;
  if (!getenv("BF_NO_ZC_DELTAS")) {
    if (void* d = bf::pinned_dev(deltas)) {
      d_src = static_cast<const bf_delta*>(d);
      direct = true;
    }
  }
  if (!direct) BF_CUDA(c, cudaMemcpyAsync(c->d_deltas, deltas, (size_t)n * sizeof(bf_delta), cudaMemcpyHostToDevice, s));
  bf::DeltaParams P{};
  P.state = r->d_state; P.deltas = d_src; P.n = n; P.n_runs = r->cap;
  P.words = r->L.words; P.state_stride = r->L.state_stride; P.off_phase = r->L.off_phase; P.off_cond = r->L.off_cond;
  P.off_decision = r->L.off_decision; P.off_child = r->L.off_child; P.child_nibbles = r->L.child_nibbles;
  P.rejected = c->d_rejected;
  P.mark = r->d_mark; P.mark_value = r->mark_touched();
  BF_CUDA(c, bf::launch_apply_deltas(P, s));
  c->stats.kernel_launches += 1;
  return BF_OK;
}

// the end of a call whose scatter rejected n deltas: the others were applied (and the call's pass ran over them)
static int rejected_deltas(bf_ctx* c, uint64_t n, bool pass_ran) {
  if (n == 0) return BF_OK;
  return fail(c, BF_EINVAL, std::to_string(n) + " delta(s) outside the record (run, index, code or absent field); the others were applied" +
                                (pass_ran ? " and the pass ran" : ""));
}

int bf_resident_apply(bf_ctx* c, uint32_t h, const bf_delta* deltas, uint32_t n) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if (n && !deltas) return fail(c, BF_EINVAL, "null deltas");
  if (n == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  r->end_snapshot(c);
  r->pending += n;
  const int rc = resident_apply_async(c, r, deltas, n);
  cudaError_t e = rc == BF_OK ? cudaMemcpyAsync(&c->pinned->word, c->d_rejected, 4, cudaMemcpyDeviceToHost, c->stream) : cudaSuccess;
  const cudaError_t es = cudaStreamSynchronize(c->stream);  // the caller's delta buffer may be reused after return
  if (rc != BF_OK) return rc;
  if (e != cudaSuccess) return cuda_fail(c, e, "bf_resident_apply");
  if (es != cudaSuccess) return cuda_fail(c, es, "cudaStreamSynchronize");
  return rejected_deltas(c, c->pinned->word, false);
}

// deltas (optional) + one pass + results, one synchronisation: the pass goes through the chunked pipeline of bf_eval (abi.cu)
// without its upload, the state being on the device already, so each chunk's pass overlaps the download of the chunk before
static int resident_tick_locked(bf_ctx* c, Resident* r, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs, uint32_t flags,
                                uint32_t max_iterations, void* result, bf_counts* counts, bf_compact_out* co = nullptr) {
  c->snap.valid = false;
  if (co && co->struct_size != sizeof(bf_compact_out)) return fail(c, BF_EINVAL, "bad bf_compact_out.struct_size");
  if (co && co->events_cap && !co->events) return fail(c, BF_EINVAL, "null events with a non-zero events_cap");
  if (n_runs > r->cap || (n_runs && !result && !co)) return fail(c, BF_EINVAL, "n_runs exceeds the resident batch / null result");
  if (flags & BF_EVAL_EXPANSION) return fail(c, BF_EINVAL, "expansion is not offered on the resident path");
  if (n_deltas && !deltas) return fail(c, BF_EINVAL, "null deltas");
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  const bf_layout& L = r->L;
  const bool changed_only = co && (flags & BF_EVAL_CHANGED_ONLY);
  flags &= ~(uint32_t)BF_EVAL_CHANGED_ONLY;
  const uint8_t* d_prev = nullptr;
  if (changed_only) {   // this pass writes the other buffer; the one it leaves behind is what "changed" is measured against
    if (int rc = r->result_prev(c)) return rc;
    std::swap(r->d_result, r->d_result_prev);
    if (r->prev_valid && r->prev_runs == n_runs) d_prev = r->d_result_prev;
  }
  // ~2 MB of result records per chunk; compact results stay on the device, so one chunk
  uint32_t chunks = 1;
  if (int rc = bf::plan_chunks(c, co ? 0 : (size_t)n_runs * L.result_stride, 2u << 20, 1, chunks)) return rc;
  uint64_t first_slice = 0;
  // a compaction over runs delivers the rejected-delta counter in the pinned tail and clears it; otherwise a counter that may have
  // counted lands in the pinned word and is zeroed before its next use
  const bool tail_delivers = co && n_runs;
  auto body = [&]() -> int {
    if (int rc = resident_apply_async(c, r, deltas, n_deltas)) return rc;
    const bool may_fuse = co && chunks == 1 && !d_prev && !changed_only && !getenv("BF_NO_FUSED_HEADS");
    bf::FusedHeads heads{};
    if (may_fuse) {
      if (int rc = bf::compact_prepare(c, n_runs, s)) return rc;
      heads = {c->d_head, bf::cblock_sums(c, c->cblock_flip), false};
    }
    bf_batch db{};
    db.struct_size = sizeof(bf_batch);
    db.flags = flags & ~(uint32_t)(BF_EVAL_VALIDATE | BF_EVAL_COUNTS_SET | BF_EVAL_PIPELINED); db.max_iterations = max_iterations; db.layout = L;
    db.n_runs = n_runs;
    // one chunk: the pass overwrites the counts block itself (no memset in front of it); several chunks add into a zeroed block
    if (chunks == 1) db.flags |= BF_EVAL_COUNTS_SET;
    else BF_CUDA(c, cudaMemsetAsync(c->d_counts, 0, sizeof(bf_counts), s));
    if (int rc = bf::chunked_pass(c, db, chunks, false, r->d_state, r->d_result, nullptr, static_cast<uint8_t*>(result), nullptr,
                                  may_fuse ? &heads : nullptr))
      return rc;
    if (int rc = bf::pass_results(c, L, r->d_result, d_prev, n_runs, co, first_slice, true, heads.done)) return rc;
    if (!tail_delivers && (!co || n_deltas)) BF_CUDA(c, cudaMemcpyAsync(&c->pinned->word, c->d_rejected, 4, cudaMemcpyDeviceToHost, s));
    return BF_OK;
  };
  const int rc = bf::pass_end(c, body(), chunks, false, co != nullptr);
  r->records_unknown();
  if (rc != BF_OK) return rc;
  if (int rc2 = r->full_tick_done(c, n_runs, flags, max_iterations, s)) return rc2;
  if (tail_delivers) c->rejected_clean = true;
  const uint64_t rejected = tail_delivers ? c->pinned->tail.rejected : c->pinned->word;
  if (int rc2 = bf::publish_pass(c, n_runs, L, r->d_state, r->d_result, counts, co, first_slice, c->last_events)) return rc2;
  return rejected_deltas(c, n_deltas ? rejected : 0, true);
}

int bf_resident_eval(bf_ctx* c, uint32_t h, uint32_t n_runs, uint32_t flags, uint32_t max_iterations, void* result, bf_counts* counts) {
  return bf_resident_tick(c, h, nullptr, 0, n_runs, flags, max_iterations, result, counts);
}

int bf_resident_tick(bf_ctx* c, uint32_t h, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs, uint32_t flags,
                     uint32_t max_iterations, void* result, bf_counts* counts) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  return resident_tick_locked(c, r, deltas, n_deltas, n_runs, flags, max_iterations, result, counts);
}

int bf_resident_tick_compact(bf_ctx* c, uint32_t h, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs, uint32_t flags,
                             uint32_t max_iterations, bf_compact_out* out, bf_counts* counts) {
  auto [g, r] = lock_resident(c, h);
  if (!out) return fail(c, BF_EINVAL, "null bf_compact_out");
  if (!r) return BF_EINVAL;
  return resident_tick_locked(c, r, deltas, n_deltas, n_runs, flags, max_iterations, nullptr, counts, out);
}

// A touched tick: scatter -> list build -> pass over the list (into the second result buffer) -> list-mode compaction, which
// brings the current result records up to date.  Falls back to a full compact tick where the baseline rules require one.
static int touched_tick_locked(bf_ctx* c, Resident* r, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs, uint32_t flags,
                               uint32_t max_iterations, bf_touched_out* out, bf_counts* counts) {
  if (out->struct_size != sizeof(bf_touched_out)) return fail(c, BF_EINVAL, "bad bf_touched_out.struct_size");
  if (flags & ~(uint32_t)(BF_EVAL_FIXPOINT | BF_EVAL_NO_COUNTS)) return fail(c, BF_EINVAL, "touched ticks take BF_EVAL_FIXPOINT and BF_EVAL_NO_COUNTS only");
  if (out->runs_cap && (!out->runs || !out->head)) return fail(c, BF_EINVAL, "null runs / head with a non-zero runs_cap");
  if (out->events_cap && !out->events) return fail(c, BF_EINVAL, "null events with a non-zero events_cap");
  if (n_runs > r->cap) return fail(c, BF_EINVAL, "n_runs exceeds the resident batch");
  if (n_deltas && !deltas) return fail(c, BF_EINVAL, "null deltas");
  BF_CUDA(c, cudaSetDevice(c->device));
  bf_compact_out co{};   // the event list, as a compact tick returns it
  co.struct_size = sizeof co; co.events = out->events; co.events_cap = out->events_cap;
  if (r->full_due(c, n_runs, flags, max_iterations)) {   // a plain compact tick: every run evaluated and listed, heads in run order
    const int rc = resident_tick_locked(c, r, deltas, n_deltas, n_runs, flags, max_iterations, nullptr, counts, &co);
    if (!c->snap.holds(r->d_state)) return rc;   // no results (rejected deltas alone still deliver them)
    const uint32_t n = std::min(n_runs, out->runs_cap);
    if (n) BF_CUDA(c, cudaMemcpy(out->head, c->d_head, (size_t)n * 4, cudaMemcpyDeviceToHost));
    for (uint32_t i = 0; i < n; ++i) out->runs[i] = i;
    out->full = 1; out->n_listed = n_runs; out->n_evaluated = n_runs; out->n_events = co.n_events;
    return rc;
  }

  c->snap.valid = false;
  cudaStream_t s = c->stream;
  const bf_layout& L = r->L;
  const uint32_t bound = (uint32_t)std::min<uint64_t>(n_runs, r->pending + n_deltas);   // >= the touched runs below n_runs
  r->pending += n_deltas;
  const uint64_t cap = out->events ? out->events_cap : 0;
  const uint32_t runs_n = std::min(bound, out->runs_cap);
  if (int rc = r->result_prev(c)) return rc;
  const uint32_t nb = (bound + 511) / 512, nbl = (r->cap + 2047) / 2048;
  if (int rc = c->d_tlist.ensure(c, (size_t)bound + 1)) return rc;
  if (int rc = c->d_tpos_head.ensure(c, bound ? bound : 1)) return rc;
  if (int rc = c->d_tsums.ensure(c, 2 * (size_t)nb + 2 * (size_t)nbl + 1)) return rc;
  if (int rc = c->d_events.ensure(c, cap ? (size_t)cap : 1)) return rc;
  // the caller's pinned buffers get the lists posted by the emit kernel, any other buffer gets them by a download
  uint32_t* p_runs = static_cast<uint32_t*>(bf::pinned_dev(out->runs));
  uint32_t* p_head = static_cast<uint32_t*>(bf::pinned_dev(out->head));
  uint16_t* p_events = cap ? static_cast<uint16_t*>(bf::pinned_dev(out->events)) : nullptr;
  if (!p_runs || !p_head) {
    if (int rc = c->d_truns.ensure(c, runs_n ? runs_n : 1)) return rc;
    if (int rc = c->d_thead.ensure(c, runs_n ? runs_n : 1)) return rc;
  }
  uint64_t first_slice = 0;
  auto body = [&]() -> int {
    if (int rc = resident_apply_async(c, r, deltas, n_deltas)) return rc;
    if (bound == 0) {   // nothing below n_runs can be touched: no launch beyond the scatter
      if (n_deltas) BF_CUDA(c, cudaMemcpyAsync(&c->pinned->word, c->d_rejected, 4, cudaMemcpyDeviceToHost, s));
      return BF_OK;
    }
    bf::TouchedParams T{};
    T.C = bf::compact_params(c, L, bound, !(flags & BF_EVAL_NO_COUNTS), true);
    T.C.result = r->d_result_prev; T.C.prev_result = r->d_result;
    T.C.events = p_events ? p_events : c->d_events; T.C.cap = cap;
    T.mark = r->d_mark; T.full_epoch = r->full_epoch; T.n_scan = n_runs; T.n_marks = r->cap; T.bound = bound;
    T.list = c->d_tlist + 1; T.list_count = c->d_tlist; T.pos_head = c->d_tpos_head;
    T.sums = c->d_tsums; T.sums_listed = c->d_tsums + nb; T.scan_sums = c->d_tsums + 2 * (size_t)nb;
    T.carry_sums = T.scan_sums + nbl;
    T.out_runs = p_runs && p_head ? p_runs : c->d_truns; T.out_head = p_runs && p_head ? p_head : c->d_thead; T.runs_cap = runs_n;
    c->rejected_clean = false;   // the emit kernel delivers and clears the counter; a failed call leaves it to be zeroed
    BF_CUDA(c, bf::launch_touched_list(T, s));
    bf_batch db{};
    db.struct_size = sizeof(bf_batch);
    db.flags = flags | BF_EVAL_COUNTS_SET; db.max_iterations = max_iterations; db.layout = L; db.n_runs = bound;
    if (int rc = bf::run_pass(c, db, r->d_state, r->d_result_prev, nullptr, c->d_counts, s, c->d_tlist + 1, c->d_tlist)) return rc;
    BF_CUDA(c, bf::launch_touched_compact(T, s));
    c->stats.kernel_launches += 4;
    if (runs_n && !(p_runs && p_head)) {
      BF_CUDA(c, cudaMemcpyAsync(out->runs, c->d_truns, (size_t)runs_n * 4, cudaMemcpyDeviceToHost, s));
      BF_CUDA(c, cudaMemcpyAsync(out->head, c->d_thead, (size_t)runs_n * 4, cudaMemcpyDeviceToHost, s));
    }
    return bf::events_first(c, out->events, c->last_touched_events, 1024, cap, p_events != nullptr, s, first_slice);
  };
  const int rc = body();
  const cudaError_t es = cudaStreamSynchronize(s);
  if (rc != BF_OK || es != cudaSuccess) {   // marks and current records may be half updated: the next touched tick is a full one
    r->need_full = true; c->rejected_clean = false;
    if (rc != BF_OK) return rc;
    return cuda_fail(c, es, "cudaStreamSynchronize");
  }
  bf::ResultTail& tail = c->pinned->tail;
  uint64_t rejected = tail.rejected;
  if (bound == 0) {   // no kernel ran: the counter is zeroed before its next use
    rejected = n_deltas ? c->pinned->word : 0u;
    tail = bf::ResultTail{};   // no kernel wrote the tail: compact_finish and the counts read nothing evaluated or listed
  } else {
    r->pending = tail.carried;   // every touched run below n_runs was evaluated: the ones above it are all that is left
    c->rejected_clean = true;    // delivered and cleared by the emit kernel
  }
  if (int rc2 = bf::publish_pass(c, n_runs, L, r->d_state, r->d_result, counts, &co, first_slice, c->last_touched_events)) return rc2;
  out->full = 0; out->n_listed = co.n_listed; out->n_evaluated = (uint32_t)tail.evaluated; out->n_events = co.n_events;
  return rejected_deltas(c, rejected, true);
}

int bf_resident_tick_touched(bf_ctx* c, uint32_t h, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs, uint32_t flags,
                             uint32_t max_iterations, bf_touched_out* out, bf_counts* counts) {
  auto [g, r] = lock_resident(c, h);
  if (!out) return fail(c, BF_EINVAL, "null bf_touched_out");
  if (!r) return BF_EINVAL;
  return touched_tick_locked(c, r, deltas, n_deltas, n_runs, flags, max_iterations, out, counts);
}

// A Story edited while its runs are live: re-index the runs of old_slot to new_slot's step indices in place (resident.cu).  All
// checks come first, so a rejected call changes nothing; then one upload of the tables, one launch, one synchronisation.
int bf_resident_migrate(bf_ctx* c, uint32_t h, bf_migration* m) {
  auto [g, r] = lock_resident(c, h);
  if (!m || m->struct_size != sizeof(bf_migration)) return fail(c, BF_EINVAL, "null bf_migration or bad struct_size");
  if (!r) return BF_EINVAL;
  const bf_layout& L = r->L;
  if (m->n_runs > r->cap) return fail(c, BF_EINVAL, "n_runs exceeds the resident batch");
  auto alive = [&](uint32_t s) { return s < c->meta.size() && c->meta[s].alive; };
  if (!alive(m->old_slot) || !alive(m->new_slot)) return fail(c, BF_ETOPO, "migration between unknown topology slots");
  if (m->old_slot == m->new_slot) return fail(c, BF_EINVAL, "migration from a slot to itself");
  const TopoMeta& mo = c->meta[m->old_slot];
  const TopoMeta& mn = c->meta[m->new_slot];
  if (m->n_old_steps != mo.S || !m->step_map) return fail(c, BF_EINVAL, "step_map must have one entry per step of old_slot");
  if (!mo.fits(L) || !mn.fits(L)) return fail(c, BF_ETOPO, "topology does not fit the batch layout (steps_max / child_nibbles)");
  std::vector<uint16_t> inv((size_t)L.words * 32, (uint16_t)BF_MIGRATE_GONE);
  for (uint32_t i = 0; i < mo.S; ++i) {
    const uint32_t t = m->step_map[i];
    if (t == BF_MIGRATE_GONE) continue;
    if (t >= mn.S) return fail(c, BF_EINVAL, "step_map[" + std::to_string(i) + "] is not a step of new_slot");
    if (inv[t] != BF_MIGRATE_GONE) return fail(c, BF_EINVAL, "step_map is not injective (new step " + std::to_string(t) + ")");
    inv[t] = (uint16_t)i;
  }
  std::vector<bf::MigrateDesc> descs;
  for (uint32_t q = 0; q < mn.P; ++q) {
    const uint32_t o = inv[mn.par_step[q]];
    if (o == BF_MIGRATE_GONE) continue;
    const auto it = std::lower_bound(mo.par_step.begin(), mo.par_step.end(), (uint16_t)o);   // descs ascend by step
    if (it == mo.par_step.end() || *it != o) continue;   // the old step was not parallel: the desc starts unregistered
    const uint32_t p = (uint32_t)(it - mo.par_step.begin());
    if (mo.par_branches[p] != mn.par_branches[q])
      return fail(c, BF_EINVAL, "parallel step " + std::to_string(o) + " changes its branch count: re-pack its runs on the host");
    bf::MigrateDesc d{};
    d.old_first = mo.child_first[p]; d.new_first = mn.child_first[q];
    d.branches = mn.par_branches[q]; d.old_p = (uint16_t)p; d.new_p = (uint16_t)q;
    descs.push_back(d);
  }
  m->migrated = 0;
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  const size_t o_inv = 16, o_desc = round_up_sz(o_inv + inv.size() * 2, 16), bytes = o_desc + descs.size() * sizeof(bf::MigrateDesc);
  if (int rc = c->d_mig.ensure(c, bytes)) return rc;
  std::vector<uint8_t> blob(bytes, 0);   // the counter starts at zero
  memcpy(blob.data() + o_inv, inv.data(), inv.size() * 2);
  if (!descs.empty()) memcpy(blob.data() + o_desc, descs.data(), descs.size() * sizeof(bf::MigrateDesc));
  r->end_snapshot(c);   // as after an upload
  bf::MigrateParams P{};
  P.state = r->d_state; P.mark = r->d_mark; P.mark_value = r->mark_must_list();
  P.migrated = reinterpret_cast<uint32_t*>(c->d_mig.p);
  P.inv = reinterpret_cast<const uint16_t*>(c->d_mig + o_inv);
  P.desc = reinterpret_cast<const bf::MigrateDesc*>(c->d_mig + o_desc); P.n_desc = (uint32_t)descs.size();
  P.n_runs = m->n_runs; P.old_slot = m->old_slot; P.new_slot = m->new_slot;
  P.words = L.words; P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.off_cond = L.off_cond;
  P.off_decision = L.off_decision; P.off_child = L.off_child; P.child_nibbles = L.child_nibbles;
  cudaError_t e = cudaMemcpyAsync(c->d_mig, blob.data(), bytes, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = bf::launch_migrate(P, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&c->pinned->word, c->d_mig, 4, cudaMemcpyDeviceToHost, s);
  if (int rc = r->sync_in_place(c, e, "bf_resident_migrate")) return rc;
  c->stats.kernel_launches += m->n_runs ? 1 : 0;
  m->migrated = c->pinned->word;
  r->pending += m->migrated;   // the touched-list bound counts the migrated runs as it counts uploaded ones
  return BF_OK;
}

// An operator redrive of live runs (resident.cu).  All checks come first, so a rejected call changes nothing.  The distinct
// (slot, step) keys get one closure mask each from the closure kernel (a mass redrive of one Story from one step costs one
// closure), then one launch resets every request's set.  One H2D copy, at most two launches, one D2H copy, one synchronisation.
int bf_resident_redrive(bf_ctx* c, uint32_t h, const bf_redrive* req, uint32_t n, uint8_t* status_out, uint32_t* applied_out) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if (n && !req) return fail(c, BF_EINVAL, "null requests");
  const bf_layout& L = r->L;
  std::unordered_map<uint64_t, uint32_t> key_of;   // (slot, step) -> key index
  std::vector<uint32_t> key(n), key_slot, key_step;
  for (uint32_t i = 0; i < n; ++i) {
    const bf_redrive& q = req[i];
    auto at = [i] { return "request " + std::to_string(i) + ": "; };   // built on failure only
    if (q.run >= r->cap) return fail(c, BF_EINVAL, at() + "run outside the resident batch");
    if (q.reserved != 0) return fail(c, BF_EINVAL, at() + "reserved must be 0");
    if (q.slot >= c->meta.size() || !c->meta[q.slot].alive) return fail(c, BF_ETOPO, at() + "unknown topology slot");
    const TopoMeta& m = c->meta[q.slot];
    if (q.step != BF_REDRIVE_ALL && q.step >= m.S) return fail(c, BF_EINVAL, at() + "step index out of range");  // "step %q not found", :541
    if (!m.fits(L)) return fail(c, BF_ETOPO, at() + "topology does not fit the batch layout (steps_max / child_nibbles)");
    key[i] = BF_REDRIVE_ALL;
    if (q.step == BF_REDRIVE_ALL) continue;
    const auto it = key_of.emplace((uint64_t)q.slot << 32 | q.step, (uint32_t)key_slot.size());
    if (it.second) { key_slot.push_back(q.slot); key_step.push_back(q.step); }
    key[i] = it.first->second;
  }
  if (applied_out) *applied_out = 0;
  if (n == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  if (int rc = bf::sync_slots(c, c->stream)) return rc;
  const size_t K = key_slot.size();
  const size_t o_req = round_up_sz(n, 16), o_key = o_req + (size_t)n * sizeof(bf_redrive), o_ks = o_key + (size_t)n * 4,
               o_mask = round_up_sz(o_ks + K * 8, 16), bytes = o_mask + K * L.words * 4;
  if (int rc = c->d_redrive.ensure(c, bytes)) return rc;
  std::vector<uint8_t> blob(o_mask - o_req);   // requests | keys | key slots | key steps (the statuses are written by the kernel)
  memcpy(blob.data(), req, (size_t)n * sizeof(bf_redrive));
  memcpy(blob.data() + (o_key - o_req), key.data(), (size_t)n * 4);
  if (K) {
    memcpy(blob.data() + (o_ks - o_req), key_slot.data(), K * 4);
    memcpy(blob.data() + (o_ks - o_req) + K * 4, key_step.data(), K * 4);
  }
  r->end_snapshot(c);   // as after an upload
  uint8_t* d = c->d_redrive;
  uint32_t* d_ks = reinterpret_cast<uint32_t*>(d + o_ks);
  uint32_t* d_mask = reinterpret_cast<uint32_t*>(d + o_mask);
  bf::RedriveParams P{};
  P.state = r->d_state; P.mark = r->d_mark; P.mark_value = r->mark_touched();   // as by a delta
  P.req = reinterpret_cast<const bf_redrive*>(d + o_req); P.key = reinterpret_cast<const uint32_t*>(d + o_key);
  P.masks = d_mask; P.status = d; P.slots = c->slots_dev; P.n = n;
  P.words = L.words; P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.off_cond = L.off_cond;
  P.off_decision = L.off_decision; P.off_child = L.off_child;
  std::vector<uint8_t> status(n);
  cudaStream_t s = c->stream;
  cudaError_t e = cudaMemcpyAsync(d + o_req, blob.data(), blob.size(), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess)
    e = bf::launch_closure(c->slots_dev, d_ks, d_ks + K, (uint32_t)K, (uint32_t)c->slots_host.size(), L.words, d_mask, s);
  if (e == cudaSuccess) e = bf::launch_redrive(P, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(status.data(), d, n, cudaMemcpyDeviceToHost, s);
  if (int rc = r->sync_in_place(c, e, "bf_resident_redrive")) return rc;
  c->stats.kernel_launches += K ? 2 : 1;
  uint32_t applied = 0;
  for (uint32_t i = 0; i < n; ++i) applied += status[i];
  if (status_out) memcpy(status_out, status.data(), n);
  if (applied_out) *applied_out = applied;
  r->pending += applied;   // the touched-list bound counts the reset runs as it counts deltas
  return BF_OK;
}

// A live batch grows its capacity and / or layout (resident.cu).  All checks come first, and the new buffers are allocated and
// filled before the old ones are freed, so a rejected or failed call changes nothing.  One launch (both record arrays), one
// device copy of the touch marks, one synchronisation.
int bf_resident_reshape(bf_ctx* c, uint32_t h, const bf_layout* layout, uint32_t capacity) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if (!layout) return fail(c, BF_EINVAL, "null layout");
  if (int rc = bf::check_layout(c, *layout)) return rc;
  const bf_layout F = r->L, T = *layout;
  if (capacity < r->cap) return fail(c, BF_EINVAL, "reshape cannot lower the capacity");
  if (T.steps_max < F.steps_max) return fail(c, BF_EINVAL, "reshape cannot lower steps_max");
  if (F.fields & ~T.fields) return fail(c, BF_EINVAL, "reshape cannot drop a field");
  if (F.off_child != BF_OFF_NONE && T.child_nibbles < F.child_nibbles) return fail(c, BF_EINVAL, "reshape cannot shrink the child area");
  // the kernel follows the offsets: every field the batch places must have a place in the new layout
  const uint32_t from[] = {F.off_cond, F.off_decision, F.off_child, F.off_fail, F.off_needs_cond, F.off_skip_dep, F.off_phase_out};
  const uint32_t to[] = {T.off_cond, T.off_decision, T.off_child, T.off_fail, T.off_needs_cond, T.off_skip_dep, T.off_phase_out};
  // zero decision planes are PENDING, which a pass applies to RUNNING gate / sleep / wait steps (an absent plane leaves them
  // alone), and added output masks may gain bits: either may change a result the touch marks know nothing of
  bool results_may_change = false;
  for (int i = 0; i < 7; ++i) {
    if (from[i] != BF_OFF_NONE && to[i] == BF_OFF_NONE) return fail(c, BF_EINVAL, "the new layout drops a field the batch has");
    if (i != 0 && i != 2 && from[i] == BF_OFF_NONE && to[i] != BF_OFF_NONE) results_may_change = true;
  }
  BF_CUDA(c, cudaSetDevice(c->device));
  Resident nb;
  if (cudaError_t e = nb.alloc(T, capacity)) return fail(c, BF_ENOMEM, std::string("resident reshape: ") + cudaGetErrorString(e));
  const size_t old_mark = r->d_mark.cap * sizeof(uint32_t), new_mark = nb.d_mark.cap * sizeof(uint32_t);
  bf::ReshapeParams P{};
  P.old_state = r->d_state; P.old_result = r->d_result; P.state = nb.d_state; P.result = nb.d_result;
  P.n_old = r->cap; P.n_new = capacity; P.from = F; P.to = T;
  cudaStream_t s = c->stream;
  cudaError_t e = bf::launch_reshape(P, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(nb.d_mark, r->d_mark, old_mark, cudaMemcpyDeviceToDevice, s);   // with the list-build padding
  if (e == cudaSuccess && new_mark > old_mark) e = cudaMemsetAsync(reinterpret_cast<uint8_t*>(nb.d_mark.p) + old_mark, 0, new_mark - old_mark, s);
  const cudaError_t es = cudaStreamSynchronize(s);
  if (e == cudaSuccess) e = es;
  if (e != cudaSuccess) return cuda_fail(c, e, "bf_resident_reshape");   // the old buffers were only read: the batch is as it was
  r->end_snapshot(c);   // as after an upload
  r->adopt(std::move(nb), T, capacity);
  if (results_may_change) r->need_full = true;
  return BF_OK;
}

// Runs leave a live batch (resident.cu): the last live runs move into the indices the retired ones free, so the batch's runs
// stay [0, n_runs - n).  All checks and allocations come first, so a rejected call or a failed allocation changes nothing.
// One H2D copy of the move table, one launch, one synchronisation; a new capacity adds the prefix copies into its buffers.
int bf_resident_retire(bf_ctx* c, uint32_t h, bf_retire* rt) {
  auto [g, r] = lock_resident(c, h);
  if (!rt || rt->struct_size != sizeof(bf_retire)) return fail(c, BF_EINVAL, "null bf_retire or bad struct_size");
  if (!r) return BF_EINVAL;
  const uint32_t N = rt->n_runs, n = rt->n;
  if (N > r->cap) return fail(c, BF_EINVAL, "n_runs exceeds the resident batch");
  if (n && !rt->runs) return fail(c, BF_EINVAL, "null runs");
  std::vector<uint8_t> gone(N, 0);
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t q = rt->runs[i];
    if (q >= N) return fail(c, BF_EINVAL, "runs[" + std::to_string(i) + "] is not below n_runs");
    if (gone[q]) return fail(c, BF_EINVAL, "runs[" + std::to_string(i) + "] is retired twice");
    gone[q] = 1;
  }
  const uint32_t m = N - n, cap = rt->capacity ? rt->capacity : r->cap;
  if (cap < m || cap > r->cap) return fail(c, BF_EINVAL, "capacity must be 0 or within [n_runs - n, the current capacity]");
  const bool resize = cap != r->cap;
  if (n == 0 && !resize) { rt->n_moves = 0; return BF_OK; }
  // the move rule: the k-th retired index below m (ascending) receives the k-th live index of [m, N); there are as many of each
  std::vector<uint32_t> to(n, bf::kRetireNoMove);   // new index of run m + i
  uint32_t n_moves = 0;
  for (uint32_t i = 0, hole = 0; i < n; ++i) {
    if (gone[m + i]) continue;
    while (!gone[hole]) ++hole;
    to[i] = hole++;
    ++n_moves;
  }
  BF_CUDA(c, cudaSetDevice(c->device));
  if (int rc = c->d_retire.ensure(c, n ? n : 1)) return rc;
  const bf_layout& L = r->L;
  Resident nb;
  if (resize)
    if (cudaError_t e = nb.alloc(L, cap)) return fail(c, BF_ENOMEM, std::string("resident retire: ") + cudaGetErrorString(e));
  r->end_snapshot(c);   // as after an upload
  bf::RetireParams P{};
  P.state = r->d_state; P.result = r->d_result; P.mark = r->d_mark; P.mark_value = r->mark_must_list();
  P.to = c->d_retire; P.m = m; P.n = n; P.state_stride = L.state_stride; P.result_stride = L.result_stride;
  cudaStream_t s = c->stream;
  cudaError_t e = n ? cudaMemcpyAsync(c->d_retire, to.data(), (size_t)n * 4, cudaMemcpyHostToDevice, s) : cudaSuccess;
  if (e == cudaSuccess) e = bf::launch_retire(P, s);
  if (resize) {   // in place first, then the prefix into the new buffers (the mark padding past cap is never read)
    if (e == cudaSuccess) e = cudaMemcpyAsync(nb.d_state, r->d_state, (size_t)cap * L.state_stride, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(nb.d_result, r->d_result, (size_t)cap * L.result_stride, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(nb.d_mark, r->d_mark, nb.d_mark.cap * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s);
  }
  if (int rc = r->sync_in_place(c, e, "bf_resident_retire")) return rc;
  c->stats.kernel_launches += n ? 1 : 0;
  if (resize) r->adopt(std::move(nb), L, cap);
  r->compact_to(m, N, to);
  for (uint32_t i = 0, k = 0; i < n && (rt->moves_from || rt->moves_to); ++i) {
    if (to[i] == bf::kRetireNoMove) continue;
    if (rt->moves_from) rt->moves_from[k] = m + i;
    if (rt->moves_to) rt->moves_to[k] = to[i];
    ++k;
  }
  rt->n_runs = m; rt->n_moves = n_moves;
  return BF_OK;
}
