// resident_abi.cu — the C ABI of include/bobrafrontier.h for resident batches (row f2): a batch's records stay on the device
// between ticks; uploads, deltas, migrations, redrives, reshapes, retirements and narrowings change them in place, transfers move
// runs between batches, and full, compact, changed-only and touched ticks evaluate them.  The bookkeeping of touched ticks lives in Resident (ctx.h).
#include <stdlib.h>
#include <string.h>

#include <array>
#include <functional>
#include <type_traits>
#include <unordered_map>

#include "ctx.h"

using bf::cuda_fail; using bf::fail; using bf::round_up_sz;

// the bf_resident_* definitions take their C linkage from include/bobrafrontier.h
// ---- resident batches (row f2: incremental state upload) --------------------------------------------------
// the live batch of handle h, or nullptr (the caller holds the ctx lock)
static Resident* live_batch(bf_ctx* c, uint32_t h) { return h < c->resident.size() && c->resident[h].alive ? &c->resident[h] : nullptr; }

// The ctx lock, which the caller holds for the call, and the live batch of handle h.  The batch is nullptr for a null ctx (no
// lock then) and for an unknown handle (its error set; an argument check that fails after this one sets its own instead).
static std::pair<std::unique_lock<std::mutex>, Resident*> lock_resident(bf_ctx* c, uint32_t h) {
  if (!c) return {};
  std::unique_lock<std::mutex> g(c->mu);
  Resident* r = live_batch(c, h);
  if (!r) fail(c, BF_EINVAL, "unknown resident batch");
  return {std::move(g), r};
}

// The sections of one call's device inputs and outputs in c->d_call (ctx.h), each 16-byte aligned (the uint4 extents, the
// 8-byte words) in the order taken.  up() takes a section the call uploads, copied into the host image at once; out() takes one
// that only the device writes.  A call takes its uploaded sections first, so that one H2D copy carries them.  send() ensures
// d_call, points each taken pointer at its section and issues that copy (none when nothing is uploaded).
struct CallStage {
  std::vector<uint8_t> image;   // the uploaded sections, as the copy carries them
  size_t size = 0;
  std::vector<std::function<void(uint8_t*)>> points;   // each points a taken pointer into d_call

  template <typename T>
  size_t take(T*& p, size_t bytes) {
    const size_t o = size;
    size = round_up_sz(o + bytes, 16);
    points.push_back([&p, o](uint8_t* d) { p = reinterpret_cast<T*>(d + o); });
    return o;
  }
  template <typename T>
  void up(T*& p, const std::remove_const_t<T>* src, size_t n) {
    const size_t o = take(p, n * sizeof(T));
    image.resize(o + n * sizeof(T));
    if (n) memcpy(image.data() + o, src, n * sizeof(T));
  }
  template <typename T>
  void out(T*& p, size_t n) { take(p, n * sizeof(T)); }
  int send(bf_ctx* c, const char* what) {
    if (int rc = c->d_call.ensure(c, std::max<size_t>(size, 16))) return rc;
    for (const auto& point : points) point(c->d_call);
    if (image.empty()) return BF_OK;
    const cudaError_t e = cudaMemcpyAsync(c->d_call, image.data(), image.size(), cudaMemcpyHostToDevice, c->stream);
    return e == cudaSuccess ? BF_OK : cuda_fail(c, e, what);
  }
};

// Request i names `run` (below cap); each run may be named once.  seen holds request index + 1 per run named so far.
static int name_run_once(bf_ctx* c, std::vector<uint32_t>& seen, uint32_t cap, uint32_t run, uint32_t i) {
  if (seen.empty()) seen.assign(cap, 0u);
  if (seen[run]) return fail(c, BF_EINVAL, "requests " + std::to_string(seen[run] - 1) + " and " + std::to_string(i) + " name the same run");
  seen[run] = i + 1;
  return BF_OK;
}

// The order of n requests by (run, step), ties by index.  -> false when two name the same (run, step): the first such pair of
// that order, as (earlier, later) in it, is in clash.
template <typename Q>
static bool order_by_run_step(const Q* q, uint32_t n, std::vector<uint32_t>& order, std::pair<uint32_t, uint32_t>& clash) {
  order.resize(n);
  for (uint32_t i = 0; i < n; ++i) order[i] = i;
  auto key = [&](uint32_t i) { return (uint64_t)q[i].run << 16 | q[i].step; };
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return key(a) < key(b); });
  for (uint32_t j = 1; j < n; ++j)
    if (key(order[j]) == key(order[j - 1])) { clash = {order[j - 1], order[j]}; return false; }
  return true;
}

// The runs [first, first + n) of a per-run device array (the state records or a side area), per_run bytes each, into the
// caller's buffer: the range check, one D2H copy, one synchronisation
static int download_runs(bf_ctx* c, const Resident* r, uint32_t first, uint32_t n, void* out, const void* area, size_t per_run) {
  if ((uint64_t)first + n > r->cap || (n && !out)) return fail(c, BF_EINVAL, "run range outside the resident batch");
  if (n == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  BF_CUDA(c, cudaMemcpyAsync(out, static_cast<const uint8_t*>(area) + first * per_run, n * per_run, cudaMemcpyDeviceToHost, c->stream));
  BF_CUDA(c, cudaStreamSynchronize(c->stream));
  return BF_OK;
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
  r->state_changed(c);
  r->prev_valid = false;   // full records arrived: the next changed-only tick lists every run
  BF_CUDA(c, cudaMemcpyAsync(r->d_state + (size_t)first * r->L.state_stride, records, (size_t)n * r->L.state_stride, cudaMemcpyHostToDevice, c->stream));
  const bf::RunAreasView A = r->areas_view();
  if (A.sched_rec)   // the uploaded runs have no schedule baseline: kSchedNoBase in the reason word of each stored record
    BF_CUDA(c, cudaMemset2DAsync(A.sched_rec + (size_t)first * A.sched_stride + 12, A.sched_stride, 0xFF, 4, n, c->stream));
  BF_CUDA(c, bf::launch_mark_runs(r->d_mark, first, n, r->mark_must_list(), c->stream));
  c->stats.kernel_launches += 1;
  if (A.runctl) {   // stops persist: a stopped run's uploaded flags byte is its saved one
    BF_CUDA(c, bf::launch_runctl_restop({A.runctl, r->d_state, r->L.state_stride, first, n}, c->stream));
    c->stats.kernel_launches += 1;
  }
  r->pending += n;
  r->note_uploaded(first, first + n);
  BF_CUDA(c, cudaStreamSynchronize(c->stream));
  return BF_OK;
}

int bf_resident_download(bf_ctx* c, uint32_t h, uint32_t first, uint32_t n, void* records) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  return download_runs(c, r, first, n, records, r->d_state, r->L.state_stride);
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
  P.runctl = r->areas.d_runctl;
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
  r->state_changed(c);
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
  if (n_deltas) r->ticked = -1;
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
  r->tick_done(n_runs, flags);
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
  if (n_deltas) r->ticked = -1;
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
  r->tick_done(n_runs, flags);
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
  bf::MigrateParams P{};
  const uint32_t zero = 0;
  CallStage st;
  st.up(P.migrated, &zero, 1);
  st.up(P.inv, inv.data(), inv.size());
  st.up(P.desc, descs.data(), descs.size());
  st.up(P.fwd, m->step_map, r->areas.timer_k ? mo.S : 0);   // the timers are re-keyed forwards
  if (int rc = st.send(c, "bf_resident_migrate")) return rc;
  r->state_changed(c);   // as after an upload
  P.state = r->d_state; P.mark = r->d_mark; P.mark_value = r->mark_must_list();
  P.n_desc = (uint32_t)descs.size();
  P.n_runs = m->n_runs; P.old_slot = m->old_slot; P.new_slot = m->new_slot;
  P.words = L.words; P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.off_cond = L.off_cond;
  P.off_decision = L.off_decision; P.off_child = L.off_child; P.child_nibbles = L.child_nibbles;
  P.areas = r->areas_view(); P.n_old_steps = mo.S;
  cudaError_t e = bf::launch_migrate(P, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&c->pinned->word, P.migrated, 4, cudaMemcpyDeviceToHost, s);
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
  bf::RedriveParams P{};
  const uint32_t *d_key_slot, *d_key_step;
  uint32_t* d_mask;
  CallStage st;   // the statuses and the closure masks are written by the kernels
  st.up(P.req, req, n);
  st.up(P.key, key.data(), n);
  st.up(d_key_slot, key_slot.data(), K);
  st.up(d_key_step, key_step.data(), K);
  st.out(P.status, n);
  st.out(d_mask, K * L.words);
  if (int rc = st.send(c, "bf_resident_redrive")) return rc;
  r->state_changed(c);   // as after an upload
  P.state = r->d_state; P.mark = r->d_mark; P.mark_value = r->mark_touched();   // as by a delta
  P.masks = d_mask; P.slots = c->slots_dev; P.n = n;
  P.words = L.words; P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.off_cond = L.off_cond;
  P.off_decision = L.off_decision; P.off_child = L.off_child;
  P.areas = r->areas_view();
  std::vector<uint8_t> status(n);
  cudaStream_t s = c->stream;
  cudaError_t e = bf::launch_closure(c->slots_dev, d_key_slot, d_key_step, (uint32_t)K, (uint32_t)c->slots_host.size(), L.words, d_mask, s);
  if (e == cudaSuccess) e = bf::launch_redrive(P, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(status.data(), P.status, n, cudaMemcpyDeviceToHost, s);
  if (int rc = r->sync_in_place(c, e, "bf_resident_redrive")) return rc;
  c->stats.kernel_launches += K ? 2 : 1;
  uint32_t applied = 0;
  for (uint32_t i = 0; i < n; ++i) applied += status[i];
  if (status_out) memcpy(status_out, status.data(), n);
  if (applied_out) *applied_out = applied;
  r->pending += applied;   // the touched-list bound counts the reset runs as it counts deltas
  return BF_OK;
}

// the offsets of the fields a layout may leave out, in one order: cond, decision, child, then the optional output fields
static std::array<uint32_t, 7> optional_fields(const bf_layout& L) {
  return {L.off_cond, L.off_decision, L.off_child, L.off_fail, L.off_needs_cond, L.off_skip_dep, L.off_phase_out};
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
  const auto from = optional_fields(F), to = optional_fields(T);
  // zero decision planes are PENDING, which a pass applies to RUNNING gate / sleep / wait steps (an absent plane leaves them
  // alone), and added output masks may gain bits: either may change a result the touch marks know nothing of
  bool results_may_change = false;
  for (size_t i = 0; i < from.size(); ++i) {
    if (from[i] != BF_OFF_NONE && to[i] == BF_OFF_NONE) return fail(c, BF_EINVAL, "the new layout drops a field the batch has");
    if (i != 0 && i != 2 && from[i] == BF_OFF_NONE && to[i] != BF_OFF_NONE) results_may_change = true;
  }
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Resident nb;
  if (cudaError_t e = nb.alloc(T, capacity)) return fail(c, BF_ENOMEM, std::string("resident reshape: ") + cudaGetErrorString(e));
  // the side areas follow the capacity (the new runs' entries empty or the defaults); the schedule records follow the words too,
  // and keep their baselines when the words stay
  if (std::string e = r->areas.alloc_resized(nb.areas, r->cap, capacity, F.words, T.words, s); !e.empty())
    return fail(c, BF_ENOMEM, "resident reshape " + e);
  const size_t old_mark = r->d_mark.cap * sizeof(uint32_t), new_mark = nb.d_mark.cap * sizeof(uint32_t);
  bf::ReshapeParams P{};
  P.old_state = r->d_state; P.old_result = r->d_result; P.state = nb.d_state; P.result = nb.d_result;
  P.n_old = r->cap; P.n_new = capacity; P.from = F; P.to = T;
  P.old_areas = r->areas_view(); P.areas = nb.areas.view(T.words);
  cudaError_t e = bf::launch_reshape(P, s);
  if (e == cudaSuccess) e = r->areas.relay(nb.areas, r->cap, capacity, F.words, T.words, s, c->stats.kernel_launches);
  if (e == cudaSuccess) e = cudaMemcpyAsync(nb.d_mark, r->d_mark, old_mark, cudaMemcpyDeviceToDevice, s);   // with the list-build padding
  if (e == cudaSuccess && new_mark > old_mark) e = cudaMemsetAsync(reinterpret_cast<uint8_t*>(nb.d_mark.p) + old_mark, 0, new_mark - old_mark, s);
  if (int rc = bf::end_call(c, e, "bf_resident_reshape")) return rc;   // the old buffers were only read: the batch is as it was
  r->state_changed(c);   // as after an upload
  r->adopt(std::move(nb), T, capacity);
  if (results_may_change) r->need_full = true;
  return BF_OK;
}

// Batch r as the extent kernels read it (after sync_slots), counting the result planes of its layout that layout T keeps.  Only
// result records a later tick compares with count: the changed-only baseline and the touched one (ctx.h).
static bf::ExtentBatch extent_batch(bf_ctx* c, const Resident* r, const bf_layout& T) {
  bf::ExtentBatch B{};
  B.state = r->d_state; B.result = r->d_result; B.mark = r->d_mark; B.areas = r->areas_view();
  B.slots = c->slots_dev; B.n_slots = (uint32_t)c->slots_host.size();
  B.prev_runs = r->prev_valid ? r->prev_runs : 0u; B.eval_runs = r->touched_baseline_runs(); B.full_epoch = r->full_epoch;
  B.L = B.R = r->L;
  if (T.off_fail == BF_OFF_NONE) B.R.off_fail = BF_OFF_NONE;
  if (T.off_needs_cond == BF_OFF_NONE) B.R.off_needs_cond = BF_OFF_NONE;
  if (T.off_skip_dep == BF_OFF_NONE) B.R.off_skip_dep = BF_OFF_NONE;
  if (T.off_phase_out == BF_OFF_NONE) B.R.off_phase_out = BF_OFF_NONE;
  return B;
}

// The extent kernel over the batch, counting the result fields layout T keeps, on the ctx stream, into three words at the start
// of c->d_call; the caller downloads them (download_extent) behind whatever else it launches.  Nothing of the batch changes.
static int extent_async(bf_ctx* c, Resident* r, uint32_t n_runs, const bf_layout& T) {
  cudaStream_t s = c->stream;
  if (int rc = c->d_call.ensure(c, 3 * sizeof(unsigned long long))) return rc;
  if (int rc = bf::sync_slots(c, s)) return rc;
  const bf::ExtentParams P{extent_batch(c, r, T), r->cap, n_runs, reinterpret_cast<unsigned long long*>(c->d_call.p)};
  BF_CUDA(c, cudaMemsetAsync(c->d_call, 0, 3 * sizeof(unsigned long long), s));
  BF_CUDA(c, bf::launch_extent(P, c->sm_count, s));
  c->stats.kernel_launches += 1;
  return BF_OK;
}

static cudaError_t download_extent(bf_ctx* c, unsigned long long* out) {
  return cudaMemcpyAsync(out, c->d_call, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream);
}

static void fill_extent(const unsigned long long* out, bf_extent* e) {
  e->steps_max = std::max(1u, (uint32_t)(out[0] >> 32));
  e->widest_run = out[0] ? ~(uint32_t)out[0] : BF_EXTENT_NO_RUN;
  e->child_nibbles = (uint32_t)(out[1] >> 32);
  e->fields = (uint32_t)out[2];
}

int bf_resident_extent(bf_ctx* c, uint32_t h, bf_extent* e) {
  auto [g, r] = lock_resident(c, h);
  if (!e || e->struct_size != sizeof(bf_extent)) return fail(c, BF_EINVAL, "null bf_extent or bad struct_size");
  if (!r) return BF_EINVAL;
  if (e->n_runs > r->cap) return fail(c, BF_EINVAL, "n_runs exceeds the resident batch");
  BF_CUDA(c, cudaSetDevice(c->device));
  unsigned long long out[3] = {};
  if (int rc = extent_async(c, r, e->n_runs, r->L)) return rc;
  BF_CUDA(c, download_extent(c, out));
  BF_CUDA(c, cudaStreamSynchronize(c->stream));
  fill_extent(out, e);
  return BF_OK;
}

// A live batch narrows its layout (resident.cu).  The layout checks come first; then the new buffers are allocated, the extent
// kernel, the re-layout into the new buffers and the copy of the marks run back to back, and after the one synchronisation the
// new buffers replace the old ones only when the extent passes.  A rejected or failed call changes nothing: the old buffers were
// only read.
int bf_resident_narrow(bf_ctx* c, uint32_t h, const bf_layout* layout, bf_extent* e) {
  auto [g, r] = lock_resident(c, h);
  if (!e || e->struct_size != sizeof(bf_extent)) return fail(c, BF_EINVAL, "null bf_extent or bad struct_size");
  if (!r) return BF_EINVAL;
  const uint32_t N = e->n_runs;
  if (N > r->cap) return fail(c, BF_EINVAL, "n_runs exceeds the resident batch");
  BF_CUDA(c, cudaSetDevice(c->device));
  unsigned long long out[3] = {};
  // a layout rejected before the extent is known still reports the extent (over every result plane), so the caller sees what fits
  auto reject = [&](const std::string& why) {
    if (extent_async(c, r, N, r->L) == BF_OK && download_extent(c, out) == cudaSuccess && cudaStreamSynchronize(c->stream) == cudaSuccess)
      fill_extent(out, e);
    return fail(c, BF_EINVAL, why);
  };
  if (!layout) return reject("null layout");
  if (bf::check_layout(c, *layout)) return reject(std::string(c->err));
  const bf_layout F = r->L, T = *layout;
  if (T.steps_max > F.steps_max) return reject("narrow cannot raise steps_max (reshape grows a batch)");
  if (T.fields & ~F.fields) return reject("narrow cannot add a field (reshape grows a batch)");
  if (F.off_child != BF_OFF_NONE && T.off_child != BF_OFF_NONE && T.child_nibbles > F.child_nibbles)
    return reject("narrow cannot enlarge the child area (reshape grows a batch)");
  // the kernel follows the offsets: every field the new layout places must be placed by the batch's.  Dropping decision planes
  // (zero ones are PENDING, which a pass applies; absent ones skip it), the child area (a registered parallel step without
  // branches joins with an area and not without one) or an output mask (the event kinds change) may change any run's result
  const auto from = optional_fields(F), to = optional_fields(T);
  bool results_may_change = false;
  for (size_t i = 0; i < from.size(); ++i) {
    if (from[i] == BF_OFF_NONE && to[i] != BF_OFF_NONE) return reject("the new layout places a field the batch lacks");
    if (i != 0 && from[i] != BF_OFF_NONE && to[i] == BF_OFF_NONE) results_may_change = true;
  }
  const bool same = memcmp(&F, &T, sizeof T) == 0;
  Resident nb;
  if (!same)
    if (cudaError_t e2 = nb.alloc(T, r->cap)) return fail(c, BF_ENOMEM, std::string("resident narrow: ") + cudaGetErrorString(e2));
  if (int rc = extent_async(c, r, N, T)) { cudaStreamSynchronize(c->stream); return rc; }
  cudaStream_t s = c->stream;
  cudaError_t err = cudaSuccess;
  if (!same) {
    bf::ReshapeParams P{};
    P.old_state = r->d_state; P.old_result = r->d_result; P.state = nb.d_state; P.result = nb.d_result;
    P.n_old = r->cap; P.n_new = r->cap; P.from = F; P.to = T;
    err = bf::launch_reshape(P, s);
    if (err == cudaSuccess) err = cudaMemcpyAsync(nb.d_mark, r->d_mark, r->d_mark.cap * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s);
    c->stats.kernel_launches += 1;
  }
  if (err == cudaSuccess) err = download_extent(c, out);
  if (int rc = bf::end_call(c, err, "bf_resident_narrow")) return rc;   // the old buffers were only read: the batch is as it was
  fill_extent(out, e);
  if (same) return BF_OK;
  const uint32_t placed = (T.off_cond != BF_OFF_NONE ? BF_F_COND : 0u) | (T.off_decision != BF_OFF_NONE ? BF_F_DECISION : 0u) |
                          (T.off_child != BF_OFF_NONE ? BF_F_CHILD : 0u);
  if (T.steps_max < e->steps_max)
    return fail(c, BF_EINVAL, "run " + std::to_string(e->widest_run) + " needs steps_max " + std::to_string(e->steps_max));
  if (T.off_child != BF_OFF_NONE && T.child_nibbles < e->child_nibbles)
    return fail(c, BF_EINVAL, "the batch needs child_nibbles " + std::to_string(e->child_nibbles));
  if (e->fields & ~placed) return fail(c, BF_EINVAL, "the new layout drops an input field holding a non-default code");
  r->state_changed(c);   // as after an upload
  r->adopt(std::move(nb), T, r->cap);
  r->narrowed(N, results_may_change);
  return BF_OK;
}

// The move rule of a retirement, shared with transfers: the k-th retired index below m (ascending) receives the k-th live index
// of [m, m + n); there are as many of each.  to[i] is the new index of run m + i, or kRetireNoMove.  -> the number of moves
static uint32_t retire_moves(const std::vector<uint8_t>& gone, uint32_t m, uint32_t n, std::vector<uint32_t>& to) {
  to.assign(n, bf::kRetireNoMove);
  uint32_t n_moves = 0;
  for (uint32_t i = 0, hole = 0; i < n; ++i) {
    if (gone[m + i]) continue;
    while (!gone[hole]) ++hole;
    to[i] = hole++;
    ++n_moves;
  }
  return n_moves;
}

// the moves of `to` into the caller's arrays (either may be NULL), ascending by target
static void write_moves(const std::vector<uint32_t>& to, uint32_t m, uint32_t* moves_from, uint32_t* moves_to) {
  for (uint32_t i = 0, k = 0; i < to.size() && (moves_from || moves_to); ++i) {
    if (to[i] == bf::kRetireNoMove) continue;
    if (moves_from) moves_from[k] = m + i;
    if (moves_to) moves_to[k] = to[i];
    ++k;
  }
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
  std::vector<uint32_t> to;
  const uint32_t n_moves = retire_moves(gone, m, n, to);
  BF_CUDA(c, cudaSetDevice(c->device));
  const bf_layout& L = r->L;
  cudaStream_t s = c->stream;
  Resident nb;
  if (resize) {
    if (cudaError_t e = nb.alloc(L, cap)) return fail(c, BF_ENOMEM, std::string("resident retire: ") + cudaGetErrorString(e));
    if (std::string e = r->areas.alloc_resized(nb.areas, r->cap, cap, L.words, L.words, s); !e.empty())
      return fail(c, BF_ENOMEM, "resident retire " + e);
  }
  bf::RetireParams P{};
  CallStage st;
  st.up(P.to, to.data(), n);
  if (int rc = st.send(c, "bf_resident_retire")) return rc;
  r->state_changed(c);   // as after an upload
  P.state = r->d_state; P.result = r->d_result; P.mark = r->d_mark; P.mark_value = r->mark_must_list();
  P.m = m; P.n = n; P.state_stride = L.state_stride; P.result_stride = L.result_stride;
  P.areas = r->areas_view();
  cudaError_t e = bf::launch_retire(P, s);
  if (resize) {   // in place first, then the prefix into the new buffers (the mark padding past cap is never read)
    if (e == cudaSuccess) e = cudaMemcpyAsync(nb.d_state, r->d_state, (size_t)cap * L.state_stride, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(nb.d_result, r->d_result, (size_t)cap * L.result_stride, cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(nb.d_mark, r->d_mark, nb.d_mark.cap * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s);
    if (e == cudaSuccess) e = r->areas.copy_prefix(nb.areas, cap, L.words, s);
  }
  if (int rc = r->sync_in_place(c, e, "bf_resident_retire")) return rc;
  c->stats.kernel_launches += n ? 1 : 0;
  if (resize) r->adopt(std::move(nb), L, cap);
  r->compact_to(m, N, to);
  write_moves(to, m, rt->moves_from, rt->moves_to);
  rt->n_runs = m; rt->n_moves = n_moves;
  return BF_OK;
}

// Live runs move from one batch of the ctx to another (resident.cu), re-laid to the destination's layout.  Both batches are
// looked up under one hold of the ctx lock.  All argument checks, the allocation and the fit check (one H2D copy, one launch,
// one D2H copy, one synchronisation) come before anything is written, so a refused or failed call changes nothing; then the
// transfer launch, the source's retire launch and one synchronisation.
int bf_resident_transfer(bf_ctx* c, uint32_t hs, uint32_t hd, bf_transfer* t) {
  auto [g, src] = lock_resident(c, hs);
  if (!t || t->struct_size != sizeof(bf_transfer)) return fail(c, BF_EINVAL, "null bf_transfer or bad struct_size");
  t->unfit = BF_EXTENT_NO_RUN;
  t->why = bf_extent{};
  if (!src) return BF_EINVAL;
  Resident* dst = live_batch(c, hd);
  if (!dst) return fail(c, BF_EINVAL, "unknown resident batch");
  if (hs == hd) return fail(c, BF_EINVAL, "a transfer from a batch to itself");
  const uint32_t N = t->src_n_runs, D = t->dst_n_runs, n = t->n;
  if (N > src->cap) return fail(c, BF_EINVAL, "src_n_runs exceeds the source batch");
  if ((uint64_t)D + n > dst->cap) return fail(c, BF_EINVAL, "dst_n_runs + n exceeds the destination batch (reshape it first)");
  if (n && !t->runs) return fail(c, BF_EINVAL, "null runs");
  std::vector<uint8_t> gone(N, 0);
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t q = t->runs[i];
    if (q >= N) return fail(c, BF_EINVAL, "runs[" + std::to_string(i) + "] is not below src_n_runs");
    if (gone[q]) return fail(c, BF_EINVAL, "runs[" + std::to_string(i) + "] is moved twice");
    gone[q] = 1;
  }
  if (n == 0) { t->n_moves = 0; return BF_OK; }
  if (src->areas.d_sched_in && !dst->areas.d_sched_in)
    return fail(c, BF_EINVAL, "the source batch has limiter inputs and the destination has no area for them (bf_resident_sched)");
  const uint32_t m = N - n;
  std::vector<uint32_t> to;
  const uint32_t n_moves = retire_moves(gone, m, n, to);
  BF_CUDA(c, cudaSetDevice(c->device));
  if (int rc = bf::sync_slots(c, c->stream)) return rc;
  bf::TransferParams P{};
  bf::RetireParams Q{};   // the source's compaction behind the transfer
  const uint32_t none = BF_EXTENT_NO_RUN;
  CallStage st;
  st.up(P.unfit, &none, 1);
  st.up(P.runs, t->runs, n);
  st.up(Q.to, to.data(), n);
  st.out(P.extent, n);
  if (int rc = st.send(c, "bf_resident_transfer")) return rc;
  const bf_layout F = src->L;
  P.src = extent_batch(c, src, dst->L);   // the source's result records as a later tick of it compares them (bf_resident_extent)
  P.dst_state = dst->d_state; P.dst_result = dst->d_result; P.dst_mark = dst->d_mark; P.mark_value = dst->mark_must_list();
  P.dst_areas = dst->areas_view();
  P.n = n; P.dst_first = D; P.T = dst->L;
  cudaStream_t s = c->stream;
  BF_CUDA(c, bf::launch_transfer_fit(P, s));
  BF_CUDA(c, cudaMemcpyAsync(&c->pinned->word, P.unfit, 4, cudaMemcpyDeviceToHost, s));
  BF_CUDA(c, cudaStreamSynchronize(s));
  c->stats.kernel_launches += 1;
  const uint32_t unfit = c->pinned->word;
  if (unfit != BF_EXTENT_NO_RUN) {   // the refused run's extent, read on this path only
    uint32_t x[4] = {};
    BF_CUDA(c, cudaMemcpy(x, P.extent + unfit, sizeof x, cudaMemcpyDeviceToHost));
    t->unfit = unfit;
    t->why.struct_size = sizeof(bf_extent); t->why.n_runs = N;
    t->why.steps_max = std::max(1u, x[0]); t->why.child_nibbles = x[1]; t->why.fields = x[2];
    t->why.widest_run = x[0] ? t->runs[unfit] : BF_EXTENT_NO_RUN;
    return fail(c, BF_EINVAL, "runs[" + std::to_string(unfit) + "] (run " + std::to_string(t->runs[unfit]) +
                                  ") does not fit the destination layout: it needs steps_max " + std::to_string(x[0]) +
                                  ", child_nibbles " + std::to_string(x[1]) + ", fields " + std::to_string(x[2]) + ", " +
                                  std::to_string(x[3] & 0x7FFFFFFFu) + " timer slot(s) of the destination's " + std::to_string(P.dst_areas.timer_k) +
                                  ((x[3] >> 31) ? ", and a run-control area (bf_resident_runctl) for its stop or deadlines" : ""));
  }
  // every arrival's record is a changed-only baseline of the source: the destination's may reach over them
  bool src_baseline = src->prev_valid;
  for (uint32_t i = 0; i < n && src_baseline; ++i) src_baseline = t->runs[i] < src->prev_runs;
  src->state_changed(c);   // as after an upload, both batches
  dst->state_changed(c);
  Q.state = src->d_state; Q.result = src->d_result; Q.mark = src->d_mark; Q.mark_value = src->mark_must_list();
  Q.m = m; Q.n = n; Q.state_stride = F.state_stride; Q.result_stride = F.result_stride; Q.areas = P.src.areas;
  cudaError_t e = bf::launch_transfer(P, s);
  if (e == cudaSuccess) e = bf::launch_retire(Q, s);   // behind the transfer on the stream: the sources are read first
  if (int rc = src->sync_in_place(c, e, "bf_resident_transfer")) { dst->records_unknown(); return rc; }
  c->stats.kernel_launches += 2;
  src->compact_to(m, N, to);
  dst->received(D, n, src_baseline);
  write_moves(to, m, t->moves_from, t->moves_to);
  t->src_n_runs = m; t->dst_n_runs = D + n; t->n_moves = n_moves;
  return BF_OK;
}

// ---- step timers (resident.cu) ------------------------------------------------------------------------------------------------
// The area of K slots per run: created with every slot empty, or grown to a larger K with each run's slots kept in place (one
// relay launch into new slots, one synchronisation; the old area is freed once the new one is filled).
int bf_resident_timers(bf_ctx* c, uint32_t h, uint32_t K) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if (K < 1 || K > BF_TIMER_MAX_SLOTS) return fail(c, BF_EINVAL, "slots_per_run must be within [1, 64]");
  if (K < r->areas.timer_k) return fail(c, BF_EINVAL, "slots_per_run cannot shrink (" + std::to_string(r->areas.timer_k) + " now)");
  if (K == r->areas.timer_k) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  DevBuf<unsigned long long> area;
  if (cudaError_t e = area.alloc((size_t)r->cap * K)) return fail(c, BF_ENOMEM, std::string("timer area: ") + cudaGetErrorString(e));
  const cudaError_t e = bf::launch_relay_timers({r->areas.d_timers, area, r->cap, r->cap, r->areas.timer_k, K}, c->stream);
  if (int rc = bf::end_call(c, e, "bf_resident_timers")) return rc;   // the old area was only read
  c->stats.kernel_launches += 1;
  r->areas.d_timers = std::move(area);
  r->areas.timer_k = K;
  return BF_OK;
}

// Arms and cancels: every argument is checked on the host (the requests sorted by (run, step), which also finds duplicates), then
// one H2D copy, the check launch, one D2H copy of the overflow word and one synchronisation before anything is written; then the
// merge launch and one synchronisation.
int bf_resident_timers_arm(bf_ctx* c, uint32_t h, const bf_timer* req, uint32_t n) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if (!r->areas.timer_k) return fail(c, BF_EINVAL, "the batch has no timer area (bf_resident_timers)");
  if (n && !req) return fail(c, BF_EINVAL, "null requests");
  const bf_layout& L = r->L;
  for (uint32_t i = 0; i < n; ++i) {
    const bf_timer& q = req[i];
    auto at = [i] { return "request " + std::to_string(i) + ": "; };
    if (q.run >= r->cap) return fail(c, BF_EINVAL, at() + "run outside the resident batch");
    if (q.step >= L.steps_max) return fail(c, BF_EINVAL, at() + "step outside the batch layout (steps_max)");
    if (q.code > BF_DEC_TIMED_OUT) return fail(c, BF_EINVAL, at() + "code is not a BF_DEC_* code");
    if (q.reserved || q.reserved2) return fail(c, BF_EINVAL, at() + "reserved fields must be 0");
    if (q.code != BF_DEC_PENDING && L.off_decision == BF_OFF_NONE)
      return fail(c, BF_EINVAL, at() + "a code that writes needs decision planes (BF_F_DECISION)");
  }
  if (n == 0) return BF_OK;
  std::vector<uint32_t> order;
  std::pair<uint32_t, uint32_t> clash;
  if (!order_by_run_step(req, n, order, clash))
    return fail(c, BF_EINVAL, "requests " + std::to_string(clash.first) + " and " + std::to_string(clash.second) + " name the same (run, step)");
  std::vector<bf_timer> sorted(n);
  std::vector<uint32_t> first, arm_before(n + 1, 0);
  for (uint32_t j = 0; j < n; ++j) {
    sorted[j] = req[order[j]];
    if (j == 0 || sorted[j].run != sorted[j - 1].run) first.push_back(j);
    arm_before[j + 1] = arm_before[j] + (sorted[j].deadline != BF_TIMER_NONE ? 1u : 0u);
  }
  const uint32_t G = (uint32_t)first.size();
  first.push_back(n);
  BF_CUDA(c, cudaSetDevice(c->device));
  bf::TimerArmParams P{};
  const uint32_t none = 0xFFFFFFFFu;
  CallStage st;
  st.up(P.overflow, &none, 1);
  st.up(P.first, first.data(), G + 1);
  st.up(P.arm_before, arm_before.data(), n + 1);
  st.up(P.req, sorted.data(), n);
  if (int rc = st.send(c, "bf_resident_timers_arm")) return rc;
  P.timers = r->areas.d_timers; P.timer_k = r->areas.timer_k; P.n_groups = G;
  cudaStream_t s = c->stream;
  BF_CUDA(c, bf::launch_arm_timers(P, false, s));
  BF_CUDA(c, cudaMemcpyAsync(&c->pinned->word, P.overflow, 4, cudaMemcpyDeviceToHost, s));
  BF_CUDA(c, cudaStreamSynchronize(s));
  c->stats.kernel_launches += 1;
  if (c->pinned->word != none)
    return fail(c, BF_ENOMEM, "run " + std::to_string(sorted[first[c->pinned->word]].run) + " would hold more than " +
                                  std::to_string(r->areas.timer_k) + " armed timers");
  if (int rc = bf::end_call(c, bf::launch_arm_timers(P, true, s), "bf_resident_timers_arm")) return rc;
  c->stats.kernel_launches += 1;
  return BF_OK;
}

// Due timers against `now` (resident.cu): the count and apply launches, the D2H copy of the four output words, one
// synchronisation.  A pinned list is posted to by the kernel itself; any other gets the entries that fired copied after it.
int bf_resident_fire(bf_ctx* c, uint32_t h, uint32_t now, bf_fire_out* out) {
  auto [g, r] = lock_resident(c, h);
  if (!out || out->struct_size != sizeof(bf_fire_out)) return fail(c, BF_EINVAL, "null bf_fire_out or bad struct_size");
  if (!r) return BF_EINVAL;
  const bf::RunAreasView A = r->areas_view();
  if (!A.timers && !A.runctl) return fail(c, BF_EINVAL, "the batch has neither a timer area (bf_resident_timers) nor run control (bf_resident_runctl)");
  const uint32_t N = out->n_runs;
  if (N > r->cap) return fail(c, BF_EINVAL, "n_runs exceeds the resident batch");
  if (out->fired_cap && !out->fired) return fail(c, BF_EINVAL, "null fired with a non-zero fired_cap");
  out->n_fired = out->n_written = out->n_pruned = 0;
  out->next_deadline = BF_TIMER_NONE;
  if (N == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  const uint32_t grid = (N - 1) / 256 + 1;
  // the list is at most N * (K + 2) long (with run control: a drain and a story entry per run): a larger fired_cap stages no more
  const uint32_t cap = (uint32_t)std::min<uint64_t>(out->fired_cap, (uint64_t)N * (A.timer_k + (A.runctl ? 2u : 0u)));
  bf::FireParams P{};
  P.fired = static_cast<bf_fired*>(bf::pinned_dev(out->fired));   // a pinned list is posted to in place
  const bool staged = !P.fired;
  CallStage st;
  st.out(P.out, 4);
  st.out(P.block_sums, grid);
  if (staged) st.out(P.fired, cap);
  if (int rc = st.send(c, "bf_resident_fire")) return rc;
  r->end_snapshot(c);   // as a delta
  P.state = r->d_state; P.areas = A; P.mark = r->d_mark; P.mark_value = r->mark_touched();
  P.n_runs = N; P.now = now;
  P.words = r->L.words; P.state_stride = r->L.state_stride; P.off_phase = r->L.off_phase; P.off_decision = r->L.off_decision;
  P.fired_cap = cap;
  cudaStream_t s = c->stream;
  uint32_t* words = c->pinned->fire;
  cudaError_t e = bf::launch_fire(P, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(words, P.out, 16, cudaMemcpyDeviceToHost, s);
  if (int rc = r->sync_in_place(c, e, "bf_resident_fire")) return rc;
  c->stats.kernel_launches += 2;
  if (const uint32_t listed = std::min(words[0], cap); listed && staged)
    BF_CUDA(c, cudaMemcpy(out->fired, P.fired, (size_t)listed * 8, cudaMemcpyDeviceToHost));
  out->n_fired = words[0]; out->n_written = words[1]; out->n_pruned = words[2]; out->next_deadline = words[3];
  r->pending += out->n_written;   // the touched-list bound counts the written codes and the timeouts as it counts deltas
  if (out->n_written) r->ticked = -1;
  return BF_OK;
}

int bf_resident_timers_download(bf_ctx* c, uint32_t h, uint32_t first, uint32_t n, void* slots) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if (!r->areas.timer_k) return fail(c, BF_EINVAL, "the batch has no timer area (bf_resident_timers)");
  return download_runs(c, r, first, n, slots, r->areas.d_timers, (size_t)r->areas.timer_k * 8);
}

// ---- resident limiters (limiters.cu) ------------------------------------------------------------------------------------------
// The inputs area: one upload of the defaults and the schedule records' fill, one synchronisation.
int bf_resident_sched(bf_ctx* c, uint32_t h) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if (r->areas.d_sched_in) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  DevBuf<bf_sched_run> in;
  DevBuf<uint8_t> rec;
  const std::vector<bf_sched_run> defaults(r->cap, bf::kSchedDefault);
  cudaError_t e = in.alloc(r->cap);
  if (e == cudaSuccess) e = RunAreas::alloc_sched_rec(rec, r->cap, r->L.words, c->stream);
  if (e != cudaSuccess) return fail(c, BF_ENOMEM, std::string("limiter inputs: ") + cudaGetErrorString(e));
  e = cudaMemcpyAsync(in, defaults.data(), (size_t)r->cap * sizeof(bf_sched_run), cudaMemcpyHostToDevice, c->stream);
  if (int rc = bf::end_call(c, e, "bf_resident_sched")) return rc;
  r->areas.d_sched_in = std::move(in);
  r->areas.d_sched_rec = std::move(rec);
  r->areas.sched_base_runs = 0;
  return BF_OK;
}

// Puts: every request checked on the host first, then one H2D copy, one launch, one synchronisation.  No state record changes.
int bf_resident_sched_put(bf_ctx* c, uint32_t h, const bf_sched_put* req, uint32_t n) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if (!r->areas.d_sched_in) return fail(c, BF_EINVAL, "the batch has no limiter inputs (bf_resident_sched)");
  if (n && !req) return fail(c, BF_EINVAL, "null requests");
  std::vector<uint32_t> seen;
  for (uint32_t i = 0; i < n; ++i) {
    const bf_sched_put& q = req[i];
    auto at = [i] { return "request " + std::to_string(i) + ": "; };
    if (q.run >= r->cap) return fail(c, BF_EINVAL, at() + "run outside the resident batch");
    if (q.reserved[0] || q.reserved[1]) return fail(c, BF_EINVAL, at() + "reserved fields must be 0");
    if (int rc = name_run_once(c, seen, r->cap, q.run, i)) return rc;
  }
  if (n == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  bf::SchedPutParams P{r->areas.d_sched_in, nullptr, n};
  CallStage st;
  st.up(P.req, req, n);
  if (int rc = st.send(c, "bf_resident_sched_put")) return rc;
  if (int rc = bf::end_call(c, bf::launch_sched_put(P, c->stream), "bf_resident_sched_put")) return rc;
  c->stats.kernel_launches += 1;
  return BF_OK;
}

int bf_resident_sched_download(bf_ctx* c, uint32_t h, uint32_t first, uint32_t n, bf_sched_put* out) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if (!r->areas.d_sched_in) return fail(c, BF_EINVAL, "the batch has no limiter inputs (bf_resident_sched)");
  // the inputs land in the caller's buffer and become puts there, one record at a time
  static_assert(sizeof(bf_sched_run) == sizeof(bf_sched_put), "a put takes the place of its run's inputs");
  if (int rc = download_runs(c, r, first, n, out, r->areas.d_sched_in, sizeof(bf_sched_run))) return rc;
  for (uint32_t i = 0; i < n; ++i) {
    bf_sched_run in;
    memcpy(&in, &out[i], sizeof in);
    out[i] = bf_sched_put{first + i, in.story_key, in.queue_key, in.priority, in.queued_elapsed_s, in.run_phase, {0u, 0u}};
  }
  return BF_OK;
}

// One schedule over several resident batches: every check first; then the tables' upload, the totals' start, a count launch per
// part into the shared totals, the limit-and-compare, CTA-scan and list launches per part, the D2H copies of the totals and of each part's
// two counts, one synchronisation, and the lists of parts whose buffers are not pinned.
int bf_resident_schedule(bf_ctx* c, const bf_sched_tables* t, uint32_t now, bf_resident_sched_part* parts, uint32_t n_parts,
                         bf_sched_out* totals) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  if (!t || t->struct_size != sizeof(bf_sched_tables)) return fail(c, BF_EINVAL, "bad bf_sched_tables.struct_size");
  if ((t->n_stories && !t->story_limit) || (t->n_queues && (!t->queue_limit || !t->queue_aging_s)))
    return fail(c, BF_EINVAL, "null limit table");
  if (!totals || totals->struct_size != sizeof(bf_sched_out)) return fail(c, BF_EINVAL, "bad bf_sched_out.struct_size");
  if (now == BF_SCHED_NONE) return fail(c, BF_EINVAL, "now must be below BF_SCHED_NONE");
  if (n_parts && !parts) return fail(c, BF_EINVAL, "null parts");
  std::vector<Resident*> rs(n_parts);
  for (uint32_t i = 0; i < n_parts; ++i) {
    const bf_resident_sched_part& p = parts[i];
    auto at = [&] { return "part " + std::to_string(i) + " (batch " + std::to_string(p.handle) + "): "; };
    if (p.struct_size != sizeof(bf_resident_sched_part)) return fail(c, BF_EINVAL, "part " + std::to_string(i) + ": bad struct_size");
    Resident* r = live_batch(c, p.handle);
    if (!r) return fail(c, BF_EINVAL, at() + "unknown resident batch");
    for (uint32_t k = 0; k < i; ++k)
      if (parts[k].handle == p.handle) return fail(c, BF_EINVAL, at() + "the batch is also part " + std::to_string(k));
    if (!r->areas.d_sched_in) return fail(c, BF_EINVAL, at() + "the batch has no limiter inputs (bf_resident_sched)");
    if (p.n_runs > r->cap) return fail(c, BF_EINVAL, at() + "n_runs exceeds the resident batch");
    if (p.runs_cap && (!p.runs || !p.heads)) return fail(c, BF_EINVAL, at() + "null runs / heads with a non-zero runs_cap");
    if (p.events_cap && !p.events) return fail(c, BF_EINVAL, at() + "null events with a non-zero events_cap");
    if (r->ticked < (int64_t)p.n_runs)
      return fail(c, BF_EINVAL, at() + "its state records changed since its last tick over " + std::to_string(p.n_runs) +
                                    " runs: a tick must come between them and the schedule");
    rs[i] = r;
  }
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  if (int rc = bf::sync_slots(c, s)) return rc;   // topology puts and drops since the ticks count as they stand now
  // tables | totals | per part: run events | CTA listed | CTA events | two totals | staged lists
  const size_t ns = t->n_stories, nq = t->n_queues;
  bf::SchedParams S{};
  CallStage st;
  st.up(S.story_limit, t->story_limit, ns);
  st.up(S.queue_limit, t->queue_limit, nq);
  st.up(S.queue_aging, t->queue_aging_s, nq);
  if (t->story_running_base) st.up(S.story_base, t->story_running_base, ns);
  if (t->queue_running_base) st.up(S.queue_base, t->queue_running_base, nq);
  if (t->queue_max_priority_base) st.up(S.queue_maxprio_base, t->queue_max_priority_base, nq);
  st.out(S.story_running, ns); st.out(S.queue_running, nq); st.out(S.queue_maxprio, nq); st.out(S.global_running, 1);
  // each part's lists go straight into the caller's buffers when they are pinned, else into staged ones copied after the call
  struct Plan { bf::ResSchedParams R; bool stage_runs, stage_events; };
  std::vector<Plan> plan(n_parts);
  for (uint32_t i = 0; i < n_parts; ++i) {
    const bf_resident_sched_part& p = parts[i];
    Plan& q = plan[i];
    bf::ResSchedParams& R = q.R;
    const size_t grid = ((size_t)p.n_runs + 255) / 256;
    R.runs_cap = std::min(p.runs_cap, p.n_runs);
    R.events_cap = std::min<uint64_t>(p.events_cap, (uint64_t)p.n_runs * rs[i]->L.words * 32);
    R.runs = R.runs_cap ? static_cast<uint32_t*>(bf::pinned_dev(p.runs)) : nullptr;
    R.heads = R.runs_cap ? static_cast<bf_sched_header*>(bf::pinned_dev(p.heads)) : nullptr;
    R.events = R.events_cap ? static_cast<uint16_t*>(bf::pinned_dev(p.events)) : nullptr;
    q.stage_runs = R.runs_cap && !(R.runs && R.heads);
    q.stage_events = R.events_cap && !R.events;
    st.out(R.run_events, p.n_runs); st.out(R.cta_listed, grid); st.out(R.cta_events, grid); st.out(R.totals, 2);
    if (q.stage_runs) { st.out(R.runs, R.runs_cap); st.out(R.heads, R.runs_cap); }
    if (q.stage_events) st.out(R.events, R.events_cap);
  }
  if (int rc = st.send(c, "bf_resident_schedule")) return rc;
  S.n_stories = t->n_stories; S.n_queues = t->n_queues; S.global_limit = t->global_limit; S.global_base = t->global_running_base;
  S.n_slots = (uint32_t)c->slots_host.size(); S.slots = c->slots_dev; S.now = now;
  auto part_params = [&](uint32_t i) {
    const Resident* r = rs[i];
    const bf_layout& L = r->L;
    bf::SchedParams P = S;
    const bf::RunAreasView A = r->areas_view();
    P.state = r->d_state; P.result = r->d_result; P.runs = A.sched_in; P.records = A.sched_rec; P.n_runs = parts[i].n_runs;
    P.words = L.words; P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.off_child = L.off_child;
    P.child_nibbles = L.child_nibbles; P.result_stride = L.result_stride; P.off_ready = L.off_ready; P.stride = A.sched_stride;
    return P;
  };
  std::vector<unsigned long long> part_tot((size_t)n_parts * 2, 0ull);
  uint64_t launches = 1;
  auto body = [&]() -> cudaError_t {
    cudaError_t e = bf::launch_schedule(S, (uint32_t)c->sm_count, s, bf::kSchedInit);
    for (uint32_t i = 0; i < n_parts && e == cudaSuccess; ++i)
      if (parts[i].n_runs) { e = bf::launch_schedule(part_params(i), (uint32_t)c->sm_count, s, bf::kSchedCount); ++launches; }
    for (uint32_t i = 0; i < n_parts && e == cudaSuccess; ++i) {
      bf::ResSchedParams R = plan[i].R;
      R.S = part_params(i);
      R.base_runs = rs[i]->areas.sched_base_runs;
      if (parts[i].n_runs) {
        e = bf::launch_resident_schedule(R, s);
        launches += 3;
        if (e == cudaSuccess) e = cudaMemcpyAsync(&part_tot[2 * i], R.totals, 16, cudaMemcpyDeviceToHost, s);
      }
    }
    auto down = [&](void* dst, const void* from, size_t bytes) -> cudaError_t {
      return (dst && bytes) ? cudaMemcpyAsync(dst, from, bytes, cudaMemcpyDeviceToHost, s) : cudaSuccess;
    };
    if (e == cudaSuccess) e = down(totals->story_running, S.story_running, ns * 4);
    if (e == cudaSuccess) e = down(totals->queue_running, S.queue_running, nq * 4);
    if (e == cudaSuccess) e = down(totals->queue_max_priority, S.queue_maxprio, nq * 4);
    if (e == cudaSuccess) e = down(totals->global_running, S.global_running, 4);
    return e;
  };
  for (Resident* r : rs) r->scheduled = -1;   // a commit reads the records this call writes
  const cudaError_t e = body();
  c->stats.kernel_launches += launches;
  if (int rc = bf::end_call(c, e, "bf_resident_schedule")) {   // the schedule records may be half written: no baseline survives
    for (Resident* r : rs) r->areas.sched_base_runs = 0;
    return rc;
  }
  for (uint32_t i = 0; i < n_parts; ++i) {
    bf_resident_sched_part& p = parts[i];
    const Plan& q = plan[i];
    p.n_listed = (uint32_t)part_tot[2 * i];
    p.n_events = part_tot[2 * i + 1];
    p.full = p.n_listed == p.n_runs ? 1u : 0u;
    rs[i]->areas.sched_base_runs = p.n_runs;
    rs[i]->scheduled = std::max<int64_t>(rs[i]->scheduled, p.n_runs);
    const uint32_t nl = std::min(p.n_listed, q.R.runs_cap);
    if (nl && q.stage_runs) {
      BF_CUDA(c, cudaMemcpy(p.runs, q.R.runs, (size_t)nl * 4, cudaMemcpyDeviceToHost));
      BF_CUDA(c, cudaMemcpy(p.heads, q.R.heads, (size_t)nl * sizeof(bf_sched_header), cudaMemcpyDeviceToHost));
    }
    const uint64_t ne = std::min<uint64_t>(p.n_events, q.R.events_cap);
    if (ne && q.stage_events) BF_CUDA(c, cudaMemcpy(p.events, q.R.events, (size_t)ne * 2, cudaMemcpyDeviceToHost));
  }
  return BF_OK;
}

// ---- StoryRun stops and deadlines (resident.cu) -------------------------------------------------------------------------------
// The area: every record at the default (deadlines BF_TIMER_NONE, the rest 0) by two memsets, one synchronisation.
int bf_resident_runctl(bf_ctx* c, uint32_t h) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if (r->areas.d_runctl) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  DevBuf<bf_run_ctl> area;
  if (cudaError_t e = area.alloc(r->cap)) return fail(c, BF_ENOMEM, std::string("run control: ") + cudaGetErrorString(e));
  cudaError_t e = cudaMemsetAsync(area, 0, (size_t)r->cap * sizeof(bf_run_ctl), c->stream);
  if (e == cudaSuccess) e = cudaMemset2DAsync(area, sizeof(bf_run_ctl), 0xFF, 8, r->cap, c->stream);   // both deadlines
  if (int rc = bf::end_call(c, e, "bf_resident_runctl")) return rc;
  r->areas.d_runctl = std::move(area);
  return BF_OK;
}

// Puts: every request checked on the host first, then one H2D copy, one launch, one synchronisation.  A put with a stop changes
// state records: it ends the snapshot and the schedule's tick, and its runs count towards the touched-list bound.
int bf_resident_runctl_put(bf_ctx* c, uint32_t h, const bf_run_ctl_put* req, uint32_t n) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if (!r->areas.d_runctl) return fail(c, BF_EINVAL, "the batch has no run-control area (bf_resident_runctl)");
  if (n && !req) return fail(c, BF_EINVAL, "null requests");
  std::vector<uint32_t> seen;
  uint32_t stops = 0;
  for (uint32_t i = 0; i < n; ++i) {
    const bf_run_ctl_put& q = req[i];
    auto at = [i] { return "request " + std::to_string(i) + ": "; };
    if (q.run >= r->cap) return fail(c, BF_EINVAL, at() + "run outside the resident batch");
    if (q.stop > BF_STOP_HOST) return fail(c, BF_EINVAL, at() + "stop is not a BF_STOP_* code");
    if (q.reserved[0] || q.reserved[1] || q.reserved[2]) return fail(c, BF_EINVAL, at() + "reserved fields must be 0");
    if (int rc = name_run_once(c, seen, r->cap, q.run, i)) return rc;
    stops += q.stop ? 1u : 0u;
  }
  if (n == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  bf::RunCtlPutParams P{};
  CallStage st;
  st.up(P.req, req, n);
  if (int rc = st.send(c, "bf_resident_runctl_put")) return rc;
  if (stops) r->state_changed(c);   // as a delta
  P.area = r->areas.d_runctl; P.n = n; P.state = r->d_state; P.state_stride = r->L.state_stride;
  P.stop = bf::StopParams{r->areas_view(), r->d_mark, r->mark_touched()};
  if (int rc = r->sync_in_place(c, bf::launch_runctl_put(P, c->stream), "bf_resident_runctl_put")) return rc;
  c->stats.kernel_launches += 1;
  r->pending += stops;   // the touched-list bound counts the stopped runs as it counts deltas
  return BF_OK;
}

int bf_resident_runctl_download(bf_ctx* c, uint32_t h, uint32_t first, uint32_t n, bf_run_ctl* out) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  if (!r->areas.d_runctl) return fail(c, BF_EINVAL, "the batch has no run-control area (bf_resident_runctl)");
  return download_runs(c, r, first, n, out, r->areas.d_runctl, sizeof(bf_run_ctl));
}

// ---- tick commits (resident.cu) -----------------------------------------------------------------------------------------------
// The host checks the call and the entries, sorts them by (run, step) and uploads them; the check launch lowers the first
// offender, which one D2H copy and one synchronisation bring back before anything is written; then the apply launch and the
// counts.  A commit that wrote a run changes the state records: it ends the snapshot and the tick a schedule or a commit needs.
int bf_resident_commit(bf_ctx* c, uint32_t h, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n, bf_commit_out* out) {
  auto [g, r] = lock_resident(c, h);
  if (!out || out->struct_size != sizeof(bf_commit_out)) return fail(c, BF_EINVAL, "null bf_commit_out or bad struct_size");
  *out = bf_commit_out{};
  out->struct_size = sizeof(bf_commit_out);
  out->bad_run = out->bad_step = BF_COMMIT_NONE;
  if (!r) return BF_EINVAL;
  auto refuse = [&](uint32_t run, uint32_t step, const std::string& msg) {
    out->bad_run = run; out->bad_step = step;
    return fail(c, BF_EINVAL, msg);
  };
  const bf_layout& L = r->L;
  if (n_runs > r->cap) return refuse(BF_COMMIT_NONE, BF_COMMIT_NONE, "n_runs exceeds the resident batch");
  if (n && !entries) return refuse(BF_COMMIT_NONE, BF_COMMIT_NONE, "null entries");
  if (L.off_cond != BF_OFF_NONE && L.off_fail == BF_OFF_NONE)
    return refuse(BF_COMMIT_NONE, BF_COMMIT_NONE, "the layout has cond planes but no BF_F_OUT_FAIL: the cond-FAIL steps are unknown");
  const std::string over = " over " + std::to_string(n_runs) + " runs";
  if (r->ticked < (int64_t)n_runs)
    return refuse(BF_COMMIT_NONE, BF_COMMIT_NONE, "the state records changed since the last tick" + over + ": a tick must come between them and the commit");
  if (c->slot_changes != r->slot_changes_seen)   // every tick that went through left them equal (a change makes the next tick full)
    return refuse(BF_COMMIT_NONE, BF_COMMIT_NONE, "a topology slot was dropped or reused since the last tick: the masks may not fit the slot's steps");
  if (r->single_ticked < (int64_t)n_runs)
    return refuse(BF_COMMIT_NONE, BF_COMMIT_NONE, "no single-pass tick" + over + " since the last BF_EVAL_FIXPOINT tick: commits follow single-pass ticks");
  const bf::RunAreasView A = r->areas_view();
  if (A.sched_in && r->scheduled < (int64_t)n_runs)
    return refuse(BF_COMMIT_NONE, BF_COMMIT_NONE, "the batch has limiter inputs and no bf_resident_schedule" + over + " ran since its last tick");
  for (uint32_t i = 0; i < n; ++i) {
    const bf_commit_entry& e = entries[i];
    auto at = [i] { return "entry " + std::to_string(i) + ": "; };
    if (e.run >= n_runs) return refuse(e.run, e.step, at() + "run outside [0, n_runs)");
    if (e.step >= L.steps_max) return refuse(e.run, e.step, at() + "step outside the layout");
    if (e.kind < BF_COMMIT_HOLD || e.kind > BF_COMMIT_PHASE) return refuse(e.run, e.step, at() + "kind is not a BF_COMMIT_* code");
    if (e.kind == BF_COMMIT_PHASE ? (e.code < BF_PHASE_PENDING || e.code > BF_PHASE_SKIPPED) : e.code != 0)
      return refuse(e.run, e.step, at() + "bad code (a BF_COMMIT_PHASE entry takes BF_PHASE_PENDING .. BF_PHASE_SKIPPED, the others 0)");
  }
  std::vector<uint32_t> order;
  std::pair<uint32_t, uint32_t> clash;
  if (!order_by_run_step(entries, n, order, clash)) {
    const bf_commit_entry& e = entries[clash.second];
    return refuse(e.run, e.step, "entries " + std::to_string(clash.first) + " and " + std::to_string(clash.second) + " name the same (run, step)");
  }
  if (n_runs == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  if (int rc = bf::sync_slots(c, s)) return rc;   // the slot table as it stands now
  std::vector<bf_commit_entry> sorted(n);
  for (uint32_t i = 0; i < n; ++i) sorted[i] = entries[order[i]];
  bf::CommitParams P{};
  const unsigned long long no_offender = ~0ull;
  const uint32_t zero_counts[5] = {};
  CallStage st;
  st.up(P.offender, &no_offender, 1);
  st.up(P.counts, zero_counts, 5);
  st.up(P.entries, sorted.data(), n);
  if (int rc = st.send(c, "bf_resident_commit (check)")) return rc;
  P.state = r->d_state; P.result = r->d_result; P.sched_rec = A.sched_rec;
  P.slots = c->slots_dev; P.n_slots = (uint32_t)c->slots_host.size();
  P.n_entries = n; P.n_runs = n_runs;
  P.words = L.words; P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.result_stride = L.result_stride;
  P.off_ready = L.off_ready; P.off_skip = L.off_skip; P.off_fail = L.off_fail; P.sched_stride = A.sched_stride;
  P.mark = r->d_mark; P.mark_value = r->mark_touched();
  uint32_t* host = c->pinned->commit;
  cudaError_t e = bf::launch_commit(P, false, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(host, P.offender, 8, cudaMemcpyDeviceToHost, s);
  if (int rc = bf::end_call(c, e, "bf_resident_commit (check)")) return rc;
  c->stats.kernel_launches += 1;
  uint64_t key;
  memcpy(&key, host, 8);
  if (key != ~0ull) {
    const uint32_t run = (uint32_t)(key >> 32), step = (uint32_t)(key >> 8) & 0xFFFFFFu, why = (uint32_t)key & 0xFFu;
    const std::string at = "run " + std::to_string(run) + " step " + std::to_string(step) + ": ";
    return refuse(run, step, at + (why == bf::kCommitNotLaunched ? "an entry names a step the tick did not launch"
                                   : why == bf::kCommitNotStop   ? "a BF_COMMIT_PHASE entry names a step that is not a stop step"
                                                                 : "a launched stop step has no BF_COMMIT_PHASE entry"));
  }
  e = bf::launch_commit(P, true, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(host, P.counts, 20, cudaMemcpyDeviceToHost, s);
  if (int rc = r->sync_in_place(c, e, "bf_resident_commit")) { r->state_changed(c); return rc; }
  c->stats.kernel_launches += 1;
  uint32_t k[5];
  memcpy(k, host, sizeof k);
  out->n_runs_written = k[0]; out->n_skipped = k[1]; out->n_launched = k[2]; out->n_queued = k[3]; out->n_failed = k[4];
  if (k[0]) {   // as a delta: the written runs are touched, and the tick a schedule or a commit needs is over
    r->state_changed(c);
    r->pending += k[0];
  }
  return BF_OK;
}
