// resident_abi.cu — the C ABI of include/bobrafrontier.h for resident batches (row f2): a batch's records stay on the device
// between ticks; uploads, deltas, migrations, redrives, reshapes, retirements and narrowings change them in place, transfers move
// runs between batches, and full, compact, changed-only and touched ticks evaluate them.  The bookkeeping of touched ticks lives in Resident (ctx.h).
#include <stdlib.h>
#include <string.h>

#include <array>
#include <functional>
#include <memory>
#include <type_traits>
#include <unordered_map>

#include "ctx.h"

using bf::cuda_fail; using bf::fail; using bf::retire_moves; using bf::round_up_sz; using bf::write_moves;

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
  // After send(), for out() sections sized from what the call's first launches found: d_call grows to hold them, keeping the
  // first `kept` bytes (the sections taken before), and every taken pointer is pointed at its section again.  A growth frees
  // the old scratch, which waits for the device; a scratch already large enough costs nothing.
  int grow(bf_ctx* c, size_t kept, const char* what) {
    if (size > c->d_call.cap) {
      decltype(c->d_call) grown;
      if (int rc = grown.ensure(c, size)) return rc;
      const cudaError_t e = cudaMemcpyAsync(grown, c->d_call, kept, cudaMemcpyDeviceToDevice, c->stream);
      if (e != cudaSuccess) return cuda_fail(c, e, what);
      c->d_call = std::move(grown);
    }
    for (const auto& point : points) point(c->d_call);
    return BF_OK;
  }
};

// One output list of a call (bf_resident_schedule, _status, _resync, _commit_journal): the kernels write it in place when the
// caller's buffer is pinned, and, for items the kernels store as uint4 (vec16), 16-byte aligned; else into the call's scratch
// (stage(), or stage_at() once the number of items is known), from where copy() or copy_async() bring min(total, cap) items back.
template <typename T>
struct OutList {
  T* host;
  uint64_t cap;          // clamped by the caller
  T* dev = nullptr;      // where the kernels write
  bool staged = false;
  OutList(void* buf, uint64_t cap, bool vec16 = false) : host(static_cast<T*>(buf)), cap(cap) {
    if (cap && (!vec16 || reinterpret_cast<uintptr_t>(buf) % 16 == 0)) dev = static_cast<T*>(bf::pinned_dev(buf));
    staged = cap && !dev;
  }
  // a and b are written in place only together: when one is staged, both are
  template <typename U>
  void pair(OutList<U>& b) {
    if (staged == b.staged) return;
    dev = nullptr; b.dev = nullptr;
    staged = cap != 0; b.staged = b.cap != 0;
  }
  void stage(CallStage& st) { if (staged) st.out(dev, cap); }
  void stage_at(CallStage& st, uint64_t total) {   // the staging holds what the list gets and the copy brings back, no more
    if (!staged) return;
    cap = std::min(total, cap);
    if (cap) st.out(dev, cap);
  }
  size_t bytes(uint64_t total) const { return staged ? (size_t)std::min(total, cap) * sizeof(T) : 0; }
  cudaError_t copy_async(uint64_t total, cudaStream_t s) const {
    const size_t b = bytes(total);
    return b ? cudaMemcpyAsync(host, dev, b, cudaMemcpyDeviceToHost, s) : cudaSuccess;
  }
  cudaError_t copy(uint64_t total) const {
    const size_t b = bytes(total);
    return b ? cudaMemcpy(host, dev, b, cudaMemcpyDeviceToHost) : cudaSuccess;
  }
};

// The shared stage of the single-pass launches (status, resync, the rewriting commit): per warp pass_stage_bytes, up to 8 warps
// per CTA within the 227 KiB a CTA can opt in to beside the launches' static words.
struct PassStage {
  uint32_t wpb = 8, topo = 0, per_warp = 0;
  uint32_t smem() const { return wpb * per_warp; }
};
static int plan_pass_stage(bf_ctx* c, const bf_layout& L, PassStage& ps) {
  if (L.off_child == BF_OFF_NONE) return BF_OK;   // no stage H, no stage
  ps.topo = bf::largest_record(c, L.words);
  ps.per_warp = bf::pass_stage_bytes(L.off_child, L.state_stride, ps.topo);
  ps.wpb = std::min<uint32_t>(8u, (227u * 1024u - bf::kStatusStaticSmem) / ps.per_warp);
  return ps.wpb ? BF_OK : fail(c, BF_ENOMEM, "a topology record and a state record do not fit one warp's shared memory");
}

// The listed runs of a status or resync call: n_runs within the batch, and runs ascending below n_runs, or runs == NULL for
// every run of [0, n_runs)
static int check_run_list(bf_ctx* c, const Resident* r, uint32_t n_runs, const uint32_t* runs, uint32_t n) {
  if (n_runs > r->cap) return fail(c, BF_EINVAL, "n_runs exceeds the resident batch");
  if (!runs && n != n_runs) return fail(c, BF_EINVAL, "runs == NULL lists every run of [0, n_runs): n must equal n_runs");
  for (uint32_t i = 0; runs && i < n; ++i) {
    if (runs[i] >= n_runs) return fail(c, BF_EINVAL, "runs[" + std::to_string(i) + "] is not below n_runs");
    if (i && runs[i] <= runs[i - 1]) return fail(c, BF_EINVAL, "runs[" + std::to_string(i) + "] does not ascend");
  }
  return BF_OK;
}

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

// The scatter of n deltas (device-visible) into batch r, counting rejected ones in *rejected
static bf::DeltaParams delta_params(const Resident* r, const bf_delta* d_src, uint32_t n, uint32_t* rejected) {
  bf::DeltaParams P{};
  P.state = r->d_state; P.deltas = d_src; P.n = n; P.n_runs = r->cap;
  P.words = r->L.words; P.state_stride = r->L.state_stride; P.off_phase = r->L.off_phase; P.off_cond = r->L.off_cond;
  P.off_decision = r->L.off_decision; P.off_child = r->L.off_child; P.child_nibbles = r->L.child_nibbles;
  P.rejected = rejected;
  P.mark = r->d_mark; P.mark_value = r->mark_touched();
  P.runctl = r->areas.d_runctl;
  return P;
}

// The device address the scatter reads n deltas from in place: pinned host memory (one launch instead of a copy and a launch;
// BF_NO_ZC_DELTAS restores the upload), else nullptr
static const bf_delta* deltas_in_place(const bf_delta* deltas) {
  return getenv("BF_NO_ZC_DELTAS") ? nullptr : static_cast<const bf_delta*>(bf::pinned_dev(deltas));
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
  const bf_delta* d_src = deltas_in_place(deltas);
  const bool direct = d_src != nullptr;
  if (!direct) d_src = c->d_deltas;
  if (!direct) BF_CUDA(c, cudaMemcpyAsync(c->d_deltas, deltas, (size_t)n * sizeof(bf_delta), cudaMemcpyHostToDevice, s));
  BF_CUDA(c, bf::launch_apply_deltas(delta_params(r, d_src, n, c->d_rejected), s));
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
  r->commit_all = true;   // a full tick may change any run's result: the next touched commit considers every run
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

// The argument checks of a touched tick, made before anything changes: bf_resident_tick_touched's, and each part's of
// bf_resident_tick_touched_many (whose flags are the call's, checked once)
static int check_touched_flags(bf_ctx* c, uint32_t flags) {
  if (flags & ~(uint32_t)(BF_EVAL_FIXPOINT | BF_EVAL_NO_COUNTS)) return fail(c, BF_EINVAL, "touched ticks take BF_EVAL_FIXPOINT and BF_EVAL_NO_COUNTS only");
  return BF_OK;
}
static int check_touched(bf_ctx* c, const Resident* r, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs,
                         const bf_touched_out* out) {
  if (out->struct_size != sizeof(bf_touched_out)) return fail(c, BF_EINVAL, "bad bf_touched_out.struct_size");
  if (out->runs_cap && (!out->runs || !out->head)) return fail(c, BF_EINVAL, "null runs / head with a non-zero runs_cap");
  if (out->events_cap && !out->events) return fail(c, BF_EINVAL, "null events with a non-zero events_cap");
  if (n_runs > r->cap) return fail(c, BF_EINVAL, "n_runs exceeds the resident batch");
  if (n_deltas && !deltas) return fail(c, BF_EINVAL, "null deltas");
  return BF_OK;
}

// A touched tick that is not full: what its launches and its end need
struct TouchedTick {
  Resident* r;
  uint32_t n_runs, n_deltas;
  bf_touched_out* out;
  TouchScratch* ts;
  uint32_t bound = 0, runs_n = 0;
  bool posted_lists = false, posted_events = false;   // written in place by the kernels (the caller's buffers are pinned)
  bf::TouchedParams T{};   // the list build and the compaction, with bound > 0
};

// The host side of a touched tick that is not full, before its launches: the batch's bookkeeping, the bound on its list, its
// scratch, and the parameters of its list build and compaction (host tail, counts and rejected counter as for a single tick;
// bf_resident_tick_touched_many points them elsewhere).  Lists go to the caller's pinned buffers in place, else to t.ts (runs,
// head) and `events`, for the caller to download.  With t.bound == 0 nothing below n_runs can be touched: no launch beyond the
// scatter.
static int touched_prepare(bf_ctx* c, TouchedTick& t, uint32_t flags, DevBuf<uint16_t>& events) {
  Resident* r = t.r;
  TouchScratch& ts = *t.ts;
  c->snap.valid = false;
  if (t.n_deltas) r->ticked = -1;
  const uint32_t bound = t.bound = (uint32_t)std::min<uint64_t>(t.n_runs, r->pending + t.n_deltas);   // >= the touched runs below n_runs
  r->pending += t.n_deltas;
  const uint64_t cap = t.out->events ? t.out->events_cap : 0;
  const uint32_t runs_n = t.runs_n = std::min(bound, t.out->runs_cap);
  if (int rc = r->result_prev(c)) return rc;
  const uint32_t nb = (bound + 511) / 512, nbl = (r->cap + 2047) / 2048;
  if (int rc = ts.list.ensure(c, (size_t)bound + 1)) return rc;
  if (int rc = ts.pos_head.ensure(c, bound ? bound : 1)) return rc;
  if (int rc = ts.sums.ensure(c, 2 * (size_t)nb + 2 * (size_t)nbl + 1)) return rc;
  if (int rc = events.ensure(c, cap ? (size_t)cap : 1)) return rc;
  uint32_t* p_runs = static_cast<uint32_t*>(bf::pinned_dev(t.out->runs));
  uint32_t* p_head = static_cast<uint32_t*>(bf::pinned_dev(t.out->head));
  uint16_t* p_events = cap ? static_cast<uint16_t*>(bf::pinned_dev(t.out->events)) : nullptr;
  t.posted_lists = p_runs && p_head; t.posted_events = p_events != nullptr;
  if (!t.posted_lists) {
    if (int rc = ts.runs.ensure(c, runs_n ? runs_n : 1)) return rc;
    if (int rc = ts.head.ensure(c, runs_n ? runs_n : 1)) return rc;
  }
  bf::TouchedParams& T = t.T;
  T.C = bf::compact_params(c, r->L, bound, !(flags & BF_EVAL_NO_COUNTS), true);
  T.C.result = r->d_result_prev; T.C.prev_result = r->d_result;
  T.C.events = p_events ? p_events : events.p; T.C.cap = cap;
  T.mark = r->d_mark; T.full_epoch = r->full_epoch; T.n_scan = t.n_runs; T.n_marks = r->cap; T.bound = bound;
  T.list = ts.list + 1; T.list_count = ts.list; T.pos_head = ts.pos_head;
  T.sums = ts.sums; T.sums_listed = ts.sums + nb; T.scan_sums = ts.sums + 2 * (size_t)nb;
  T.carry_sums = T.scan_sums + nbl;
  T.out_runs = t.posted_lists ? p_runs : ts.runs.p; T.out_head = t.posted_lists ? p_head : ts.head.p; T.runs_cap = runs_n;
  return BF_OK;
}

// The pass of a touched tick over its list (into the batch's second result buffer), adding its counts into `counts`
static int touched_pass(bf_ctx* c, const TouchedTick& t, uint32_t flags, uint32_t max_iterations, unsigned long long* counts) {
  bf_batch db{};
  db.struct_size = sizeof(bf_batch);
  db.flags = flags | BF_EVAL_COUNTS_SET; db.max_iterations = max_iterations; db.layout = t.r->L; db.n_runs = t.bound;
  return bf::run_pass(c, db, t.r->d_state, t.r->d_result_prev, nullptr, counts, c->stream, t.ts->list + 1, t.ts->list);
}

// The end of a touched tick that is not full, once the stream is synchronised, from the tail its last kernel posted (zero where
// no kernel ran): the batch's pending runs and tick, the evaluated snapshot, the counts and the out fields.  Both touched calls
// end their list-mode ticks here.
static void touched_end(bf_ctx* c, const TouchedTick& t, uint32_t flags, const bf::ResultTail& tail, bf_counts* counts) {
  Resident* r = t.r;
  if (t.bound) r->pending = tail.carried;   // every touched run below n_runs was evaluated: the ones above it are all that is left
  r->tick_done(t.n_runs, flags);
  c->snap = {true, t.n_runs, r->L, r->d_state, r->d_result};
  if (counts) *counts = {tail.counts[0], tail.counts[1], tail.counts[2], tail.counts[3]};
  t.out->full = 0; t.out->n_listed = (uint32_t)tail.listed; t.out->n_evaluated = (uint32_t)tail.evaluated; t.out->n_events = tail.events;
}

// With commit-due bits (bf_resident_commit_marks), the runs a touched tick evaluates become due: one launch over its list, behind
// the list build
static int mark_commit_due(bf_ctx* c, const TouchedTick& t) {
  uint32_t* due = t.r->areas.d_due;
  if (!due) return BF_OK;
  BF_CUDA(c, bf::launch_due_mark_list(due, t.T.list, t.T.list_count, t.bound, (uint32_t)c->sm_count * 4u, c->stream));
  c->stats.kernel_launches += 1;
  return BF_OK;
}

// A touched tick: scatter -> list build -> pass over the list -> list-mode compaction, which brings the current result records up
// to date; or a full compact tick where the baseline rules require one.
static int touched_tick_locked(bf_ctx* c, Resident* r, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs, uint32_t flags,
                               uint32_t max_iterations, bf_touched_out* out, bf_counts* counts) {
  if (int rc = check_touched_flags(c, flags)) return rc;
  if (int rc = check_touched(c, r, deltas, n_deltas, n_runs, out)) return rc;
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

  cudaStream_t s = c->stream;
  TouchedTick t{r, n_runs, n_deltas, out, &c->touch[0]};
  uint64_t first_slice = 0;
  auto body = [&]() -> int {
    if (int rc = touched_prepare(c, t, flags, c->d_events)) return rc;
    if (int rc = resident_apply_async(c, r, deltas, n_deltas)) return rc;
    if (t.bound == 0) {   // no launch beyond the scatter
      if (n_deltas) BF_CUDA(c, cudaMemcpyAsync(&c->pinned->word, c->d_rejected, 4, cudaMemcpyDeviceToHost, s));
      return BF_OK;
    }
    c->rejected_clean = false;   // the emit kernel delivers and clears the counter; a failed call leaves it to be zeroed
    BF_CUDA(c, bf::launch_touched_list(t.T, s));
    if (int rc = mark_commit_due(c, t)) return rc;
    if (int rc = touched_pass(c, t, flags, max_iterations, c->d_counts)) return rc;
    BF_CUDA(c, bf::launch_touched_compact(t.T, s));
    c->stats.kernel_launches += 4;
    if (t.runs_n && !t.posted_lists) {
      BF_CUDA(c, cudaMemcpyAsync(out->runs, t.ts->runs, (size_t)t.runs_n * 4, cudaMemcpyDeviceToHost, s));
      BF_CUDA(c, cudaMemcpyAsync(out->head, t.ts->head, (size_t)t.runs_n * 4, cudaMemcpyDeviceToHost, s));
    }
    return bf::events_first(c, out->events, c->last_touched_events, 1024, co.events ? co.events_cap : 0, t.posted_events, s, first_slice);
  };
  const int rc = body();
  const cudaError_t es = cudaStreamSynchronize(s);
  if (rc != BF_OK || es != cudaSuccess) {   // marks and current records may be half updated: the next touched tick is a full one
    r->need_full = true; r->commit_all = true; c->rejected_clean = false;
    if (rc != BF_OK) return rc;
    return cuda_fail(c, es, "cudaStreamSynchronize");
  }
  bf::ResultTail& tail = c->pinned->tail;
  uint64_t rejected = tail.rejected;
  if (t.bound == 0) {   // no kernel ran: the counter is zeroed before its next use
    rejected = n_deltas ? c->pinned->word : 0u;
    tail = bf::ResultTail{};   // no kernel wrote the tail: nothing evaluated or listed
  } else {
    c->rejected_clean = true;    // delivered and cleared by the emit kernel
  }
  touched_end(c, t, flags, tail, counts);
  if (int rc2 = bf::compact_finish(c, &co, first_slice, c->last_touched_events)) return rc2;   // the events the first slice missed
  return rejected_deltas(c, rejected, true);
}

int bf_resident_tick_touched(bf_ctx* c, uint32_t h, const bf_delta* deltas, uint32_t n_deltas, uint32_t n_runs, uint32_t flags,
                             uint32_t max_iterations, bf_touched_out* out, bf_counts* counts) {
  auto [g, r] = lock_resident(c, h);
  if (!out) return fail(c, BF_EINVAL, "null bf_touched_out");
  if (!r) return BF_EINVAL;
  return touched_tick_locked(c, r, deltas, n_deltas, n_runs, flags, max_iterations, out, counts);
}

// Several touched ticks, one per part, with one synchronisation.  Every part is checked first.  A part whose tick is full runs as
// its single call does (own synchronisation).  The other parts tick together: one upload of their part tables, deltas and zeroed
// counters; one scatter launch over every part's deltas; one list-build launch pair over every part's touch marks; one pass per
// part (each batch has its own kernel build and launch plan), back to back; one compaction launch pair over every part's list;
// one D2H of the parts' rejected-delta counters; one synchronisation.  Each part has its own list scratch, counts block, pinned
// tail and counter, so no part's results are overwritten before the host reads them.  The parts then end in part order as
// single ticks end (touched_end), pageable lists are downloaded now that their lengths are known, and the evaluated snapshot is
// the last part's, as after the per-part calls.
int bf_resident_tick_touched_many(bf_ctx* c, uint32_t flags, uint32_t max_iterations, bf_tick_part* parts, uint32_t n_parts,
                                  uint32_t* bad_part) {
  if (bad_part) *bad_part = BF_COMMIT_NONE;
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  if (n_parts && !parts) return fail(c, BF_EINVAL, "null parts");
  if (int rc = check_touched_flags(c, flags)) return rc;
  auto name = [&](uint32_t k, int rc) {   // a refusal or failure of part k
    if (bad_part) *bad_part = k;
    c->err = "parts[" + std::to_string(k) + "]: " + c->err;
    return rc;
  };
  std::vector<Resident*> rs(n_parts);
  std::unordered_map<uint32_t, uint32_t> named;   // handle -> the part naming it
  for (uint32_t k = 0; k < n_parts; ++k) {
    const bf_tick_part& p = parts[k];
    if (p.struct_size != sizeof(bf_tick_part)) return name(k, fail(c, BF_EINVAL, "bad bf_tick_part.struct_size"));
    if (!p.out) return name(k, fail(c, BF_EINVAL, "null bf_touched_out"));
    if (!(rs[k] = live_batch(c, p.handle))) return name(k, fail(c, BF_EINVAL, "unknown resident batch"));
    if (!named.emplace(p.handle, k).second)
      return name(k, fail(c, BF_EINVAL, "parts " + std::to_string(named[p.handle]) + " and " + std::to_string(k) + " name the same resident batch"));
    if (int rc = check_touched(c, rs[k], p.deltas, p.n_deltas, p.n_runs, p.out)) return name(k, rc);
  }
  if (n_parts == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  // after a failure the records and marks of any part may be half updated: every part's next touched tick is full
  auto failed = [&](uint32_t k, int rc) {
    for (Resident* r : rs) { r->need_full = true; r->commit_all = true; }
    return name(k, rc);
  };
  uint32_t first_rejected = BF_COMMIT_NONE;
  std::string rejected_msg;
  auto note_rejected = [&](uint32_t k, uint64_t n) {
    if (!n || first_rejected <= k) return;
    first_rejected = k;
    rejected_deltas(c, n, true);
    rejected_msg = c->err;
  };

  std::vector<uint32_t> group;   // the parts that tick together, ascending
  for (uint32_t k = 0; k < n_parts; ++k) {
    const bf_tick_part& p = parts[k];
    if (!rs[k]->full_due(c, p.n_runs, flags, max_iterations)) { group.push_back(k); continue; }
    const int rc = touched_tick_locked(c, rs[k], p.deltas, p.n_deltas, p.n_runs, flags, max_iterations, p.out, p.counts);
    if (rc == BF_EINVAL && first_rejected > k) {   // the checks passed, so rejected deltas: the others were applied and the pass ran
      first_rejected = k;
      rejected_msg = c->err;
    } else if (rc != BF_OK && rc != BF_EINVAL) {
      return failed(k, rc);
    }
  }

  const uint32_t n = (uint32_t)group.size();
  if (n) {
    if (c->part_tails_cap < n) {   // pinned: a tail per part, then a rejected-delta count per part
      bf::ResultTail* nt = nullptr;
      const cudaError_t e = cudaHostAlloc(&nt, (size_t)n * (sizeof(bf::ResultTail) + 4), cudaHostAllocDefault);
      if (e != cudaSuccess) { cudaGetLastError(); return failed(group[0], fail(c, BF_ENOMEM, std::string("cudaHostAlloc: ") + cudaGetErrorString(e))); }
      if (c->part_tails) cudaFreeHost(c->part_tails);
      c->part_tails = nt; c->part_tails_cap = n;
    }
    uint32_t* h_rejected = reinterpret_cast<uint32_t*>(c->part_tails + c->part_tails_cap);
    if (c->touch.size() < n) c->touch.resize(n);
    std::vector<TouchedTick> ticks;
    ticks.reserve(n);
    for (uint32_t i = 0; i < n; ++i) {
      const bf_tick_part& p = parts[group[i]];
      ticks.push_back(TouchedTick{rs[group[i]], p.n_runs, p.n_deltas, p.out, &c->touch[i]});
      c->part_tails[i] = bf::ResultTail{};
      if (int rc = touched_prepare(c, ticks[i], flags, c->touch[i].events)) return failed(group[i], rc);
    }
    // one upload: delta tables | delta starts | list-mode tables | list-build starts | compaction starts | counters | counts |
    // pageable deltas.  The tables hold device addresses inside it, so it is laid out and allocated first.
    std::vector<uint32_t> listed;   // the ticks with launches beyond the scatter
    for (uint32_t i = 0; i < n; ++i)
      if (ticks[i].bound) listed.push_back(i);
    const uint32_t m = (uint32_t)listed.size();
    size_t at = 0;
    auto take = [&](size_t bytes) { const size_t o = at; at = round_up_sz(at + bytes, 16); return o; };
    const size_t o_dp = take(n * sizeof(bf::DeltaParams)), o_df = take((n + 1) * 4), o_tp = take(m * sizeof(bf::TouchedParams));
    const size_t o_lf = take((m + 1) * 4), o_cf = take((m + 1) * 4), o_rej = take(n * 4), o_cnt = take((size_t)n * 32);
    std::vector<const bf_delta*> in_place(n);
    uint64_t staged = 0, total = 0;
    for (uint32_t i = 0; i < n; ++i) {
      in_place[i] = ticks[i].n_deltas ? deltas_in_place(parts[group[i]].deltas) : nullptr;
      if (!in_place[i]) staged += ticks[i].n_deltas;
      total += ticks[i].n_deltas;
    }
    if (total >= (1ull << 32)) return failed(group[0], fail(c, BF_EINVAL, "more than 2^32 - 1 deltas in one call"));
    const size_t o_d = take(staged * sizeof(bf_delta));
    if (int rc = c->d_call.ensure(c, std::max<size_t>(at, 16))) return failed(group[0], rc);
    uint8_t* d = c->d_call;
    std::vector<uint8_t> image(at, 0);
    auto* dp = reinterpret_cast<bf::DeltaParams*>(image.data() + o_dp);
    auto* df = reinterpret_cast<uint32_t*>(image.data() + o_df);
    auto* tp = reinterpret_cast<bf::TouchedParams*>(image.data() + o_tp);
    auto* lf = reinterpret_cast<uint32_t*>(image.data() + o_lf);
    auto* cf = reinterpret_cast<uint32_t*>(image.data() + o_cf);
    auto* cnt = reinterpret_cast<unsigned long long*>(d + o_cnt);
    auto* rej = reinterpret_cast<uint32_t*>(d + o_rej);
    uint64_t off = 0, soff = 0;
    for (uint32_t i = 0; i < n; ++i) {
      const bf_delta* src = in_place[i];
      if (!src) {
        src = reinterpret_cast<const bf_delta*>(d + o_d) + soff;
        if (ticks[i].n_deltas) memcpy(image.data() + o_d + soff * sizeof(bf_delta), parts[group[i]].deltas, (size_t)ticks[i].n_deltas * sizeof(bf_delta));
        soff += ticks[i].n_deltas;
      }
      dp[i] = delta_params(ticks[i].r, src, ticks[i].n_deltas, rej + i);
      df[i] = (uint32_t)off;
      off += ticks[i].n_deltas;
    }
    df[n] = (uint32_t)off;
    uint32_t lb = 0, cb = 0;
    for (uint32_t j = 0; j < m; ++j) {
      const uint32_t i = listed[j];
      bf::TouchedParams T = ticks[i].T;
      T.C.host_tail = &c->part_tails[i];
      T.C.counts = (flags & BF_EVAL_NO_COUNTS) ? nullptr : cnt + 4 * (size_t)i;
      T.C.rejected = nullptr;   // the counters come back in one copy behind the compaction
      tp[j] = T;
      lf[j] = lb; cf[j] = cb;
      lb += (T.n_marks + 2047) / 2048; cb += (T.bound + 511) / 512;
    }
    lf[m] = lb; cf[m] = cb;
    cudaStream_t s = c->stream;
    auto issue = [&]() -> int {
      BF_CUDA(c, cudaMemcpyAsync(d, image.data(), at, cudaMemcpyHostToDevice, s));
      BF_CUDA(c, bf::launch_apply_deltas_many(reinterpret_cast<bf::DeltaParams*>(d + o_dp), reinterpret_cast<uint32_t*>(d + o_df), n,
                                              (uint32_t)total, s));
      if (m) {
        const auto* dtp = reinterpret_cast<const bf::TouchedParams*>(d + o_tp);
        BF_CUDA(c, bf::launch_touched_list_many(dtp, reinterpret_cast<uint32_t*>(d + o_lf), m, lb, s));
        for (uint32_t j = 0; j < m; ++j)
          if (int rc = mark_commit_due(c, ticks[listed[j]])) return rc;
        for (uint32_t j = 0; j < m; ++j)
          if (int rc = touched_pass(c, ticks[listed[j]], flags, max_iterations, cnt + 4 * (size_t)listed[j])) return rc;
        BF_CUDA(c, bf::launch_touched_compact_many(dtp, reinterpret_cast<uint32_t*>(d + o_cf), m, cb, s));
      }
      c->stats.kernel_launches += (total ? 1 : 0) + (m ? 4 : 0);
      BF_CUDA(c, cudaMemcpyAsync(h_rejected, rej, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
      return BF_OK;
    };
    const int rc = issue();
    const cudaError_t es = cudaStreamSynchronize(s);
    if (rc != BF_OK) return failed(group[0], rc);
    if (es != cudaSuccess) return failed(group[0], cuda_fail(c, es, "cudaStreamSynchronize"));
    for (uint32_t i = 0; i < n; ++i) {
      const uint32_t k = group[i];
      const TouchedTick& t = ticks[i];
      const bf::ResultTail& tail = c->part_tails[i];
      touched_end(c, t, flags, tail, parts[k].counts);
      c->last_touched_events = tail.events;
      // pageable lists: downloaded now that their lengths are known
      bf_touched_out* out = t.out;
      const uint32_t nl = std::min(out->n_listed, out->runs_cap);
      const uint64_t ne = std::min<uint64_t>(tail.events, out->events ? out->events_cap : 0);
      cudaError_t e = cudaSuccess;
      if (nl && !t.posted_lists) {
        e = cudaMemcpyAsync(out->runs, t.ts->runs, (size_t)nl * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out->head, t.ts->head, (size_t)nl * 4, cudaMemcpyDeviceToHost, s);
      }
      if (e == cudaSuccess && ne && !t.posted_events) e = cudaMemcpyAsync(out->events, t.ts->events, (size_t)ne * 2, cudaMemcpyDeviceToHost, s);
      if (e != cudaSuccess) { cudaStreamSynchronize(s); return failed(k, cuda_fail(c, e, "cudaMemcpyAsync")); }
      note_rejected(k, h_rejected[i]);
    }
    if (const int rc2 = bf::end_call(c, cudaSuccess, "cudaMemcpyAsync")) return failed(group[0], rc2);
  }
  Resident* last = rs[n_parts - 1];   // the evaluated snapshot is the last part's, as after the per-part calls
  c->snap = {true, parts[n_parts - 1].n_runs, last->L, last->d_state, last->d_result};
  if (first_rejected == BF_COMMIT_NONE) return BF_OK;
  if (bad_part) *bad_part = first_rejected;
  c->err = "parts[" + std::to_string(first_rejected) + "]: " + rejected_msg;
  return BF_EINVAL;
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

// The locks of two distinct ctxs, taken in address order so that two calls over the same pair never wait on each other.
static std::pair<std::unique_lock<std::mutex>, std::unique_lock<std::mutex>> lock_pair(bf_ctx* a, bf_ctx* b) {
  if (std::less<bf_ctx*>()(b, a)) std::swap(a, b);
  std::unique_lock<std::mutex> first(a->mu);
  std::unique_lock<std::mutex> second(b->mu);
  return {std::move(first), std::move(second)};
}

// The staged runs of a cross-ctx transfer, as offsets from the start of the staging (GatherParams), the same in both ctxs'
// scratch: the unfit word, reasons, identity indices, marks, state records, result records, then each side area the source has.
struct RunStaging {
  size_t reason = 16, ident, mark, state, result, timers, sched_in, runctl, bytes;
  RunStaging(uint32_t n, const bf_layout& F, const RunAreas& A) {
    auto next = [](size_t o, size_t b) { return round_up_sz(o + b, 16); };
    ident = next(reason, n * 4ull);
    mark = next(ident, n * 4ull);
    state = next(mark, n * 4ull);
    result = next(state, (size_t)n * F.state_stride);
    timers = next(result, (size_t)n * F.result_stride);
    sched_in = next(timers, (size_t)n * A.timer_k * 8);
    runctl = next(sched_in, A.d_sched_in ? n * sizeof(bf_sched_run) : 0);
    bytes = next(runctl, A.d_runctl ? n * sizeof(bf_run_ctl) : 0);
  }
  // the staged runs at `base` as a source view: an ExtentBatch of layout F over the slots of the ctx holding them
  bf::ExtentBatch view(uint8_t* base, const bf::ExtentBatch& src, const RunAreas& A, uint32_t n, const bf::Slot* slots,
                       uint32_t n_slots) const {
    bf::ExtentBatch B = src;
    B.state = base + state; B.result = base + result; B.mark = reinterpret_cast<uint32_t*>(base + mark);
    B.areas = {A.timer_k ? reinterpret_cast<unsigned long long*>(base + timers) : nullptr, A.timer_k,
               A.d_sched_in ? reinterpret_cast<bf_sched_run*>(base + sched_in) : nullptr, nullptr, src.areas.sched_stride,
               A.d_runctl ? reinterpret_cast<bf_run_ctl*>(base + runctl) : nullptr};
    B.slots = slots; B.n_slots = n_slots;
    B.prev_runs = 0; B.eval_runs = n; B.full_epoch = 0;
    return B;
  }
};

// The packed topology records of `slots` of ctx c (live), each at a 16-byte boundary in order, into out: one H2D copy of the
// moves, one move_records launch into c->d_call, one D2H copy, enqueued on the ctx stream; the caller synchronises it.
static int pack_records(bf_ctx* c, const std::vector<uint32_t>& slots, std::vector<uint8_t>& out) {
  std::vector<unsigned long long> moves(4 * slots.size());
  size_t off = 0;
  for (size_t i = 0; i < slots.size(); ++i) {
    const TopoMeta& m = c->meta[slots[i]];
    moves[4 * i] = m.offset; moves[4 * i + 1] = off; moves[4 * i + 2] = m.bytes; moves[4 * i + 3] = 0;
    off += round_up_sz(m.bytes, 16);
  }
  BF_CUDA(c, cudaSetDevice(c->device));
  const unsigned long long* d_moves = nullptr;
  uint8_t* packed = nullptr;
  CallStage st;
  st.up(d_moves, moves.data(), moves.size());
  st.out(packed, off);
  if (int rc = st.send(c, "bf_resident_transfer_ctx (slot map)")) return rc;
  out.resize(off);
  BF_CUDA(c, bf::launch_move_records(c->arena, packed, d_moves, (uint32_t)slots.size(), c->stream));
  BF_CUDA(c, cudaMemcpyAsync(out.data(), packed, off, cudaMemcpyDeviceToHost, c->stream));
  c->stats.kernel_launches += 1;
  return BF_OK;
}

// Live runs move to a batch of another ctx (resident.cu): bf_resident_transfer with the source's runs gathered into a staging
// area, copied to the destination's scratch and re-laid there from it.  Every check, the slot map's records, the gather, the
// copy, the fit launch and its synchronisation come before anything is written, so a refused or failed call changes nothing;
// then the transfer launch on the destination, the retire launch on the source, and one synchronisation of each.
int bf_resident_transfer_ctx(bf_ctx* sc, uint32_t hs, bf_ctx* dc, uint32_t hd, bf_ctx_transfer* t) {
  if (!sc || !dc) return BF_EINVAL;
  if (sc == dc) {
    std::lock_guard<std::mutex> g(sc->mu);
    return fail(sc, BF_EINVAL, "a transfer within one ctx is bf_resident_transfer");
  }
  auto locks = lock_pair(sc, dc);
  if (!t || t->struct_size != sizeof(bf_ctx_transfer)) return fail(sc, BF_EINVAL, "null bf_ctx_transfer or bad struct_size");
  t->unfit = BF_EXTENT_NO_RUN;
  t->unfit_reason = BF_UNFIT_NONE;
  t->why = bf_extent{};
  Resident* src = live_batch(sc, hs);
  if (!src) return fail(sc, BF_EINVAL, "unknown resident batch (source)");
  Resident* dst = live_batch(dc, hd);
  if (!dst) return fail(sc, BF_EINVAL, "unknown resident batch (destination)");
  const uint32_t N = t->src_n_runs, D = t->dst_n_runs, n = t->n, n_map = t->n_slot_map;
  if (N > src->cap) return fail(sc, BF_EINVAL, "src_n_runs exceeds the source batch");
  if ((uint64_t)D + n > dst->cap) return fail(sc, BF_EINVAL, "dst_n_runs + n exceeds the destination batch (reshape it first)");
  if (n && !t->runs) return fail(sc, BF_EINVAL, "null runs");
  if (n_map && !t->slot_map) return fail(sc, BF_EINVAL, "null slot_map with a non-zero n_slot_map");
  std::vector<uint8_t> gone(N, 0);
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t q = t->runs[i];
    if (q >= N) return fail(sc, BF_EINVAL, "runs[" + std::to_string(i) + "] is not below src_n_runs");
    if (gone[q]) return fail(sc, BF_EINVAL, "runs[" + std::to_string(i) + "] is moved twice");
    gone[q] = 1;
  }
  if (n == 0) { t->n_moves = 0; return BF_OK; }
  if (src->areas.d_sched_in && !dst->areas.d_sched_in)
    return fail(sc, BF_EINVAL, "the source batch has limiter inputs and the destination has no area for them (bf_resident_sched)");
  // the map as the gather reads it: an entry of a source slot that is not live becomes kSlotDead; every other used entry must
  // name a live destination slot holding the same packed record.  The records of the used entries are packed on each device
  // and come back in one copy per ctx.
  std::vector<uint32_t> dmap(t->slot_map, t->slot_map + n_map), used_s, used_d;
  for (uint32_t s = 0; s < n_map; ++s) {
    if (dmap[s] == BF_SLOT_NONE) continue;
    uint32_t bs = 0, bd = 0;
    if (bf_topology_record(sc, s, nullptr, &bs) != BF_OK) { dmap[s] = bf::kSlotDead; continue; }
    const std::string at = "slot_map[" + std::to_string(s) + "] = " + std::to_string(dmap[s]) + ": ";
    if (bf_topology_record(dc, dmap[s], nullptr, &bd) != BF_OK) return fail(sc, BF_EINVAL, at + "not a live slot of the destination ctx");
    if (bs != bd) return fail(sc, BF_EINVAL, at + "its topology record differs from the source slot's");
    used_s.push_back(s); used_d.push_back(dmap[s]);
  }
  if (!used_s.empty()) {
    std::vector<uint8_t> rec_s, rec_d;
    int rc = pack_records(sc, used_s, rec_s);
    if (rc == BF_OK) { rc = pack_records(dc, used_d, rec_d); if (rc != BF_OK) fail(sc, rc, dc->err); }
    const cudaError_t e1 = cudaStreamSynchronize(sc->stream), e2 = cudaStreamSynchronize(dc->stream);
    if (rc != BF_OK) return rc;
    if (e1 != cudaSuccess || e2 != cudaSuccess) return cuda_fail(sc, e1 != cudaSuccess ? e1 : e2, "bf_resident_transfer_ctx (slot map)");
    size_t o = 0;
    for (size_t i = 0; i < used_s.size(); ++i) {
      const uint32_t b = sc->meta[used_s[i]].bytes;
      if (memcmp(rec_s.data() + o, rec_d.data() + o, b) != 0)
        return fail(sc, BF_EINVAL, "slot_map[" + std::to_string(used_s[i]) + "] = " + std::to_string(used_d[i]) +
                                       ": its topology record differs from the source slot's");
      o += round_up_sz(b, 16);
    }
  }
  const uint32_t m = N - n;
  std::vector<uint32_t> to;
  const uint32_t n_moves = retire_moves(gone, m, n, to);
  const bf_layout F = src->L;
  const RunStaging stg(n, F, src->areas);
  // the source: runs, map and moves up, the gather into the staging behind them, an event behind the gather
  BF_CUDA(sc, cudaSetDevice(sc->device));
  bf::GatherParams G{};
  bf::RetireParams Q{};   // the source's compaction, once the destination took the runs
  const uint32_t head[4] = {BF_EXTENT_NO_RUN, 0u, 0u, 0u};
  uint8_t* s_rest = nullptr;
  CallStage st;
  st.up(G.runs, t->runs, n);
  if (n_map) st.up(G.slot_map, dmap.data(), n_map);
  st.up(Q.to, to.data(), n);
  st.up(G.unfit, head, 4);
  st.out(s_rest, stg.bytes - stg.reason);   // the sections follow one another: the staging starts at G.unfit
  if (int rc = st.send(sc, "bf_resident_transfer_ctx")) return rc;
  uint8_t* s_base = reinterpret_cast<uint8_t*>(G.unfit);
  G.src = extent_batch(sc, src, dst->L);
  G.n = n; G.n_slot_map = n_map;
  const bf::ExtentBatch sv = stg.view(s_base, G.src, src->areas, n, nullptr, 0);
  G.reason = reinterpret_cast<uint32_t*>(s_base + stg.reason); G.ident = reinterpret_cast<uint32_t*>(s_base + stg.ident);
  G.mark = const_cast<uint32_t*>(sv.mark); G.state = const_cast<uint8_t*>(sv.state); G.result = const_cast<uint8_t*>(sv.result);
  G.areas = sv.areas;
  cudaEvent_t gathered = nullptr;
  BF_CUDA(sc, cudaEventCreateWithFlags(&gathered, cudaEventDisableTiming));
  std::unique_ptr<CUevent_st, cudaError_t (*)(cudaEvent_t)> ev_owner(gathered, cudaEventDestroy);
  BF_CUDA(sc, bf::launch_gather(G, sc->stream));
  BF_CUDA(sc, cudaEventRecord(gathered, sc->stream));
  sc->stats.kernel_launches += 1;
  // the destination: the staging copied in, the fit launch over it, its verdict down
  BF_CUDA(sc, cudaSetDevice(dc->device));
  if (int rc = bf::sync_slots(dc, dc->stream)) { cudaStreamSynchronize(sc->stream); return fail(sc, rc, dc->err); }
  bf::TransferParams P{};
  uint8_t* d_base = nullptr;
  CallStage dt;
  dt.out(d_base, stg.bytes);
  dt.out(P.extent, n);
  if (int rc = dt.send(dc, "bf_resident_transfer_ctx")) { cudaStreamSynchronize(sc->stream); return fail(sc, rc, dc->err); }
  P.src = stg.view(d_base, G.src, src->areas, n, dc->slots_dev, (uint32_t)dc->slots_host.size());
  P.runs = reinterpret_cast<uint32_t*>(d_base + stg.ident);
  P.unfit = reinterpret_cast<uint32_t*>(d_base);
  P.dst_state = dst->d_state; P.dst_result = dst->d_result; P.dst_mark = dst->d_mark; P.mark_value = dst->mark_must_list();
  P.dst_areas = dst->areas_view();
  P.n = n; P.dst_first = D; P.T = dst->L;
  cudaStream_t ds = dc->stream;
  cudaError_t e = cudaStreamWaitEvent(ds, gathered, 0);
  if (e == cudaSuccess) e = cudaMemcpyPeerAsync(d_base, dc->device, s_base, sc->device, stg.bytes, ds);
  if (e == cudaSuccess) e = bf::launch_transfer_fit(P, ds);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&dc->pinned->word, P.unfit, 4, cudaMemcpyDeviceToHost, ds);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ds);
  const cudaError_t es = cudaStreamSynchronize(sc->stream);   // the gather went through before the copy; nothing else is queued
  if (e == cudaSuccess) e = es;
  if (e != cudaSuccess) return cuda_fail(sc, e, "bf_resident_transfer_ctx (gather, copy and fit)");
  dc->stats.kernel_launches += 1;
  const uint32_t unfit = dc->pinned->word;
  if (unfit != BF_EXTENT_NO_RUN) {   // the refused run's extent and verdict, read on this path only
    uint32_t x[4] = {}, why = 0;
    BF_CUDA(sc, cudaMemcpy(x, P.extent + unfit, sizeof x, cudaMemcpyDeviceToHost));
    BF_CUDA(sc, cudaMemcpy(&why, d_base + stg.reason + 4ull * unfit, 4, cudaMemcpyDeviceToHost));
    t->unfit = unfit;
    t->unfit_reason = why ? why : (uint32_t)BF_UNFIT_LAYOUT;
    t->why.struct_size = sizeof(bf_extent); t->why.n_runs = N;
    t->why.steps_max = std::max(1u, x[0]); t->why.child_nibbles = x[1]; t->why.fields = x[2];
    t->why.widest_run = x[0] ? t->runs[unfit] : BF_EXTENT_NO_RUN;
    if (why) {
      static const char* const kWhy[] = {"", "", "is not mapped", "is at or past n_slot_map", "is not live in the source ctx"};
      return fail(sc, BF_EINVAL, "runs[" + std::to_string(unfit) + "] (run " + std::to_string(t->runs[unfit]) + "): its topology slot " +
                                     kWhy[why]);
    }
    return fail(sc, BF_EINVAL, "runs[" + std::to_string(unfit) + "] (run " + std::to_string(t->runs[unfit]) +
                                   ") does not fit the destination layout: it needs steps_max " + std::to_string(x[0]) +
                                   ", child_nibbles " + std::to_string(x[1]) + ", fields " + std::to_string(x[2]) + ", " +
                                   std::to_string(x[3] & 0x7FFFFFFFu) + " timer slot(s) of the destination's " +
                                   std::to_string(P.dst_areas.timer_k) +
                                   ((x[3] >> 31) ? ", and a run-control area (bf_resident_runctl) for its stop or deadlines" : ""));
  }
  bool src_baseline = src->prev_valid;
  for (uint32_t i = 0; i < n && src_baseline; ++i) src_baseline = t->runs[i] < src->prev_runs;
  src->state_changed(sc);   // as after an upload, both batches
  dst->state_changed(dc);
  const cudaError_t e_dst = bf::launch_transfer(P, ds);
  Q.state = src->d_state; Q.result = src->d_result; Q.mark = src->d_mark; Q.mark_value = src->mark_must_list();
  Q.m = m; Q.n = n; Q.state_stride = F.state_stride; Q.result_stride = F.result_stride; Q.areas = src->areas_view();
  // the staging holds the runs: the source compacts at once, unless the transfer could not be launched (then the runs stay)
  e = e_dst == cudaSuccess ? cudaSetDevice(sc->device) : cudaSuccess;
  if (e == cudaSuccess && e_dst == cudaSuccess) e = bf::launch_retire(Q, sc->stream);
  const int r_src = src->sync_in_place(sc, e, "bf_resident_transfer_ctx (retire)");
  const int r_dst = dst->sync_in_place(dc, e_dst, "bf_resident_transfer_ctx (transfer)");
  sc->stats.kernel_launches += e_dst == cudaSuccess ? 1 : 0;
  dc->stats.kernel_launches += 1;
  if (r_src != BF_OK || r_dst != BF_OK) {   // either side may be half written: neither keeps a baseline
    src->records_unknown(); dst->records_unknown();
    return r_src != BF_OK ? r_src : fail(sc, r_dst, dc->err);
  }
  dst->received(D, n, src_baseline);
  src->compact_to(m, N, to);
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
// The limiter parameters of one part: the call's S, over runs [0, n_runs) of batch r
static bf::SchedParams sched_part_params(const bf::SchedParams& S, const Resident* r, uint32_t n_runs) {
  const bf_layout& L = r->L;
  bf::SchedParams P = S;
  const bf::RunAreasView A = r->areas_view();
  P.state = r->d_state; P.result = r->d_result; P.runs = A.sched_in; P.records = A.sched_rec; P.n_runs = n_runs;
  P.words = L.words; P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.off_child = L.off_child;
  P.child_nibbles = L.child_nibbles; P.result_stride = L.result_stride; P.off_ready = L.off_ready; P.stride = A.sched_stride;
  return P;
}

// The checks of one schedule over parts of ctx c (the caller holds its lock): rs receives each part's batch.
static int check_schedule(bf_ctx* c, const bf_sched_tables* t, uint32_t now, const bf_resident_sched_part* parts, uint32_t n_parts,
                          const bf_sched_out* totals, std::vector<Resident*>& rs) {
  if (!t || t->struct_size != sizeof(bf_sched_tables)) return fail(c, BF_EINVAL, "bad bf_sched_tables.struct_size");
  if ((t->n_stories && !t->story_limit) || (t->n_queues && (!t->queue_limit || !t->queue_aging_s)))
    return fail(c, BF_EINVAL, "null limit table");
  if (!totals || totals->struct_size != sizeof(bf_sched_out)) return fail(c, BF_EINVAL, "bad bf_sched_out.struct_size");
  if (now == BF_SCHED_NONE) return fail(c, BF_EINVAL, "now must be below BF_SCHED_NONE");
  if (n_parts && !parts) return fail(c, BF_EINVAL, "null parts");
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
  return BF_OK;
}

static int resident_schedule_locked(bf_ctx* c, const bf_sched_tables* t, uint32_t now, bf_resident_sched_part* parts, uint32_t n_parts,
                                    bf_sched_out* totals) {
  std::vector<Resident*> rs(n_parts);
  if (int rc = check_schedule(c, t, now, parts, n_parts, totals, rs)) return rc;
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  if (int rc = bf::sync_slots(c, s)) return rc;   // topology puts and drops since the ticks count as they stand now
  // tables | totals | per part: run events | CTA listed runs and events | two totals | staged lists
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
  struct Plan {
    bf::ResSchedParams R;
    OutList<uint32_t> runs;
    OutList<bf_sched_header> heads;
    OutList<uint16_t> events;
  };
  std::vector<Plan> plan;
  plan.reserve(n_parts);   // the staged lists' pointers are taken in place
  for (uint32_t i = 0; i < n_parts; ++i) {
    const bf_resident_sched_part& p = parts[i];
    const uint32_t runs_cap = std::min(p.runs_cap, p.n_runs);
    plan.push_back(Plan{{}, {p.runs, runs_cap}, {p.heads, runs_cap},
                        {p.events, std::min<uint64_t>(p.events_cap, (uint64_t)p.n_runs * rs[i]->L.words * 32)}});
    Plan& q = plan.back();
    q.runs.pair(q.heads);
    const size_t grid = ((size_t)p.n_runs + 255) / 256;
    st.out(q.R.run_events, p.n_runs); st.out(q.R.cta, 2 * grid); st.out(q.R.totals, 2);
    q.runs.stage(st); q.heads.stage(st); q.events.stage(st);
  }
  if (int rc = st.send(c, "bf_resident_schedule")) return rc;
  S.n_stories = t->n_stories; S.n_queues = t->n_queues; S.global_limit = t->global_limit; S.global_base = t->global_running_base;
  S.n_slots = (uint32_t)c->slots_host.size(); S.slots = c->slots_dev; S.now = now;
  auto part_params = [&](uint32_t i) { return sched_part_params(S, rs[i], parts[i].n_runs); };
  std::vector<unsigned long long> part_tot((size_t)n_parts * 2, 0ull);
  uint64_t launches = 1;
  auto body = [&]() -> cudaError_t {
    cudaError_t e = bf::launch_schedule(S, (uint32_t)c->sm_count, s, bf::kSchedInit);
    for (uint32_t i = 0; i < n_parts && e == cudaSuccess; ++i)
      if (parts[i].n_runs) { e = bf::launch_schedule(part_params(i), (uint32_t)c->sm_count, s, bf::kSchedCount); ++launches; }
    for (uint32_t i = 0; i < n_parts && e == cudaSuccess; ++i) {
      const Plan& q = plan[i];
      bf::ResSchedParams R = q.R;
      R.S = part_params(i);
      R.runs = q.runs.dev; R.heads = q.heads.dev; R.events = q.events.dev;
      R.runs_cap = (uint32_t)q.runs.cap; R.events_cap = q.events.cap;
      R.base_runs = rs[i]->areas.sched_base_runs;
      if (parts[i].n_runs) {
        e = bf::launch_resident_schedule(R, s);
        launches += 3;
        if (e == cudaSuccess && rs[i]->areas.d_due) {   // the runs whose record changed become commit-due
          e = bf::launch_due_mark_sched(rs[i]->areas.d_due, R.run_events, parts[i].n_runs, s);
          launches += 1;
        }
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
    for (Resident* r : rs) { r->areas.sched_base_runs = 0; r->commit_all = true; }
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
    BF_CUDA(c, q.runs.copy(p.n_listed));
    BF_CUDA(c, q.heads.copy(p.n_listed));
    BF_CUDA(c, q.events.copy(p.n_events));
  }
  return BF_OK;
}

int bf_resident_schedule(bf_ctx* c, const bf_sched_tables* t, uint32_t now, bf_resident_sched_part* parts, uint32_t n_parts,
                         bf_sched_out* totals) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  return resident_schedule_locked(c, t, now, parts, n_parts, totals);
}

// Phase 1 of bf_resident_schedule_ctxs on ctx c (its lock held, its parts checked): the totals' start without bases and the
// count launches of its parts, then the D2H copies of the four totals into c->span_totals (pinned): story_running [ns] |
// queue_running [nq] | queue_max_priority [nq] | global_running [1].  Enqueued on the ctx stream; the caller synchronises.
static int span_count(bf_ctx* c, const bf_sched_tables* t, uint32_t now, const std::vector<bf_resident_sched_part>& parts,
                      const std::vector<Resident*>& rs) {
  const size_t ns = t->n_stories, nq = t->n_queues, words = ns + 2 * nq + 1;
  BF_CUDA(c, cudaSetDevice(c->device));
  if (c->span_totals_cap < words) {
    uint32_t* nt = nullptr;
    const cudaError_t e = cudaHostAlloc(reinterpret_cast<void**>(&nt), words * 4, cudaHostAllocDefault);
    if (e != cudaSuccess) { cudaGetLastError(); return fail(c, BF_ENOMEM, std::string("cudaHostAlloc: ") + cudaGetErrorString(e)); }
    if (c->span_totals) cudaFreeHost(c->span_totals);
    c->span_totals = nt; c->span_totals_cap = words;
  }
  cudaStream_t s = c->stream;
  if (int rc = bf::sync_slots(c, s)) return rc;
  bf::SchedParams S{};
  CallStage st;
  st.up(S.queue_aging, t->queue_aging_s, nq);
  st.out(S.story_running, ns); st.out(S.queue_running, nq); st.out(S.queue_maxprio, nq); st.out(S.global_running, 1);
  if (int rc = st.send(c, "bf_resident_schedule_ctxs")) return rc;
  S.n_stories = t->n_stories; S.n_queues = t->n_queues;
  S.n_slots = (uint32_t)c->slots_host.size(); S.slots = c->slots_dev; S.now = now;
  cudaError_t e = bf::launch_schedule(S, (uint32_t)c->sm_count, s, bf::kSchedInit);
  c->stats.kernel_launches += 1;
  for (size_t i = 0; i < parts.size() && e == cudaSuccess; ++i)
    if (parts[i].n_runs) {
      e = bf::launch_schedule(sched_part_params(S, rs[i], parts[i].n_runs), (uint32_t)c->sm_count, s, bf::kSchedCount);
      c->stats.kernel_launches += 1;
    }
  uint32_t* h = c->span_totals;
  if (e == cudaSuccess && ns) e = cudaMemcpyAsync(h, S.story_running, ns * 4, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess && nq) e = cudaMemcpyAsync(h + ns, S.queue_running, nq * 4, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess && nq) e = cudaMemcpyAsync(h + ns + nq, S.queue_maxprio, nq * 4, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(h + ns + 2 * nq, S.global_running, 4, cudaMemcpyDeviceToHost, s);
  return e == cudaSuccess ? BF_OK : cuda_fail(c, e, "bf_resident_schedule_ctxs (count)");
}

// One schedule over resident batches of several ctxs: every check on every ctx first; phase 1 counts each ctx's parts alone;
// the host gives each ctx the table bases plus the other ctxs' counts; phase 2 is bf_resident_schedule on each ctx with those.
int bf_resident_schedule_ctxs(const bf_sched_tables* t, uint32_t now, bf_ctx_sched_part* parts, uint32_t n_parts, bf_sched_out* totals) {
  if (!parts || n_parts == 0) return BF_EINVAL;
  bf_ctx* c0 = parts[0].ctx;
  for (uint32_t i = 0; i < n_parts; ++i) {
    const bf_ctx_sched_part& p = parts[i];
    if (p.struct_size != sizeof(bf_ctx_sched_part) || p.reserved || !p.ctx || !p.part) {
      if (c0) { std::lock_guard<std::mutex> g(c0->mu); fail(c0, BF_EINVAL, "part " + std::to_string(i) + ": bad struct_size, reserved, ctx or part"); }
      return BF_EINVAL;
    }
  }
  // the distinct ctxs in order of first appearance, each with its parts (copies, in call order)
  std::vector<bf_ctx*> ctxs;
  std::vector<std::vector<uint32_t>> of;
  for (uint32_t i = 0; i < n_parts; ++i) {
    const size_t k = std::find(ctxs.begin(), ctxs.end(), parts[i].ctx) - ctxs.begin();
    if (k == ctxs.size()) { ctxs.push_back(parts[i].ctx); of.emplace_back(); }
    of[k].push_back(i);
  }
  std::vector<bf_ctx*> order = ctxs;
  std::sort(order.begin(), order.end(), std::less<bf_ctx*>());
  std::vector<std::unique_lock<std::mutex>> locks;
  for (bf_ctx* c : order) locks.emplace_back(c->mu);
  const size_t K = ctxs.size();
  auto report = [&](size_t k, int code) {   // the first part's ctx carries every refusal's text too
    if (k) ctxs[0]->err = ctxs[k]->err;
    return code;
  };
  std::vector<std::vector<bf_resident_sched_part>> ps(K);
  std::vector<std::vector<Resident*>> rs(K);
  for (size_t k = 0; k < K; ++k) {
    for (uint32_t i : of[k]) ps[k].push_back(*parts[i].part);
    rs[k].resize(ps[k].size());
    if (int rc = check_schedule(ctxs[k], t, now, ps[k].data(), (uint32_t)ps[k].size(), totals, rs[k])) return report(k, rc);
  }
  // phase 1: each ctx's own counts
  int rc = BF_OK;
  size_t started = 0, bad = 0;
  for (; started < K && rc == BF_OK; ++started)
    if ((rc = span_count(ctxs[started], t, now, ps[started], rs[started])) != BF_OK) bad = started;
  for (size_t k = 0; k < started; ++k) {
    const cudaError_t e = cudaStreamSynchronize(ctxs[k]->stream);
    if (rc == BF_OK && e != cudaSuccess) { rc = cuda_fail(ctxs[k], e, "bf_resident_schedule_ctxs (count)"); bad = k; }
  }
  if (rc != BF_OK) return report(bad, rc);
  // the bases of ctx k: the tables' plus every other ctx's counts
  const size_t ns = t->n_stories, nq = t->n_queues;
  std::vector<uint32_t> story_base(ns), queue_base(nq);
  std::vector<int32_t> maxprio_base(nq);
  auto failed = [&](int code) {   // as after a failed bf_resident_schedule, every part of every ctx
    for (auto& v : rs)
      for (Resident* r : v) { r->areas.sched_base_runs = 0; r->commit_all = true; r->scheduled = -1; }
    return code;
  };
  for (size_t k = 0; k < K; ++k) {
    bf_sched_tables tk = *t;
    uint32_t global_base = t->global_running_base;
    for (size_t s = 0; s < ns; ++s) story_base[s] = t->story_running_base ? t->story_running_base[s] : 0u;
    for (size_t q = 0; q < nq; ++q) {
      queue_base[q] = t->queue_running_base ? t->queue_running_base[q] : 0u;
      maxprio_base[q] = t->queue_max_priority_base ? t->queue_max_priority_base[q] : INT32_MIN;
    }
    for (size_t j = 0; j < K; ++j) {
      if (j == k) continue;
      const uint32_t* h = ctxs[j]->span_totals;
      for (size_t s = 0; s < ns; ++s) story_base[s] += h[s];
      for (size_t q = 0; q < nq; ++q) {
        queue_base[q] += h[ns + q];
        maxprio_base[q] = std::max(maxprio_base[q], static_cast<int32_t>(h[ns + nq + q]));
      }
      global_base += h[ns + 2 * nq];
    }
    tk.story_running_base = story_base.data(); tk.queue_running_base = queue_base.data();
    tk.queue_max_priority_base = maxprio_base.data(); tk.global_running_base = global_base;
    // every ctx ends with the same totals: the last one hands them to the caller
    bf_sched_out none{};
    none.struct_size = sizeof(bf_sched_out);
    bf_sched_out* out = k + 1 == K ? totals : &none;
    if (int rk = resident_schedule_locked(ctxs[k], &tk, now, ps[k].data(), (uint32_t)ps[k].size(), out)) return report(k, failed(rk));
    for (size_t i = 0; i < of[k].size(); ++i) {
      bf_resident_sched_part& p = *parts[of[k][i]].part;
      p.n_listed = ps[k][i].n_listed; p.full = ps[k][i].full; p.n_events = ps[k][i].n_events;
    }
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
// With `arm` the same launches take the arms too (resident.cu): the timing table is copied up first when a timing changed, and
// the counts copied back carry the arms' two words.  With `journal` the check launch also counts each run's items and a scan
// launch follows it; the totals come back with the offender, so staged items and runs are copied before the second
// synchronisation.  With `rewritten` (bf_resident_commit_rewrites, journaled) rewrite_runs runs before the check launch: the
// staged planes are taken with the call's other sections, so the apply after a growth still finds them.  With `scope`
// (bf_resident_commit_touched) the same checks and staging feed the list-mode builds of the launches: over the list of due runs
// that the count, scan and list launches build in front of them, or, when the call is full, over [0, n_runs) with every due bit
// set first.  bf_resident_commit, _timed, _journal, _rewrites and _touched are this one call.
static int resident_commit(bf_ctx* c, uint32_t h, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n, bf_commit_out* out,
                           bf_commit_arm* arm, bf_commit_journal* journal, bool journaled, uint32_t* rewritten = nullptr,
                           bool rewrites = false, bf_commit_scope* scope = nullptr) {
  auto [g, r] = lock_resident(c, h);
  if (scope) {   // bf_resident_commit_touched: the form is picked by arm, journal and the scope's flags
    if (scope->struct_size != sizeof(bf_commit_scope)) return fail(c, BF_EINVAL, "bad bf_commit_scope.struct_size");
    scope->full = scope->n_considered = 0;
    if (scope->flags & ~BF_COMMIT_SCOPE_REWRITES) return fail(c, BF_EINVAL, "bf_commit_scope.flags takes BF_COMMIT_SCOPE_REWRITES only");
    if (rewrites && !journal) return fail(c, BF_EINVAL, "BF_COMMIT_SCOPE_REWRITES needs a journal");
  }
  if (rewrites) {
    if (!rewritten) return fail(c, BF_EINVAL, "null n_rewritten");
    *rewritten = 0;
  }
  if (journaled) {
    if (!journal || journal->struct_size != sizeof(bf_commit_journal)) return fail(c, BF_EINVAL, "null bf_commit_journal or bad struct_size");
    if ((journal->items_cap && !journal->items) || (journal->runs_cap && !journal->runs))
      return fail(c, BF_EINVAL, "null items / runs with a non-zero cap");
    journal->n_items = 0;
    journal->n_runs_listed = 0;
  }
  if (!out || out->struct_size != sizeof(bf_commit_out)) return fail(c, BF_EINVAL, "null bf_commit_out or bad struct_size");
  *out = bf_commit_out{};
  out->struct_size = sizeof(bf_commit_out);
  out->bad_run = out->bad_step = BF_COMMIT_NONE;
  auto refuse = [&](uint32_t run, uint32_t step, const std::string& msg, int code = BF_EINVAL) {
    out->bad_run = run; out->bad_step = step;
    return fail(c, code, msg);
  };
  if (arm) {
    if (arm->struct_size != sizeof(bf_commit_arm)) return fail(c, BF_EINVAL, "bad bf_commit_arm struct_size");
    arm->n_armed = 0;
    arm->next_deadline = BF_TIMER_NONE;
  }
  if (!r) return BF_EINVAL;
  if (scope && !r->areas.d_due) return refuse(BF_COMMIT_NONE, BF_COMMIT_NONE, "the batch has no commit-due area (bf_resident_commit_marks)");
  if (arm && !r->areas.timer_k) return refuse(BF_COMMIT_NONE, BF_COMMIT_NONE, "the batch has no timer area (bf_resident_timers) to arm");
  if (arm && arm->now == BF_TIMER_NONE) return refuse(BF_COMMIT_NONE, BF_COMMIT_NONE, "now must not be BF_TIMER_NONE");
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
  // the five counts, then the arms' count and deadline, then the steps written from the stages
  const uint32_t zero_counts[8] = {0u, 0u, 0u, 0u, 0u, 0u, BF_TIMER_NONE, 0u};
  const uint32_t n_counts = rewrites ? 8u : arm ? 7u : 5u;
  if (arm)
    if (int rc = bf::sync_timings(c, s, P.arm)) return rc;
  CallStage st;
  st.up(P.offender, &no_offender, 1);
  st.up(P.counts, zero_counts, n_counts);
  st.up(P.entries, sorted.data(), n);
  // a touched commit: full, or the run list of its due bits and entries (groups of 32 due words)
  const uint32_t form = (arm ? 1u : 0u) | (journaled ? 2u : 0u) | (rewrites ? 4u : 0u);
  const bool full = scope && (r->commit_all || r->commit_form != form || (arm && r->commit_timings != c->timing_changes));
  const bool by_list = scope && !full;
  const unsigned long long all_runs = n_runs;
  const unsigned long long* n_up = nullptr;
  bf::DueListParams D{};
  if (scope && full) st.up(n_up, &all_runs, 1);
  if (by_list) {
    D.n = (uint32_t)((RunAreas::due_words(n_runs) + 31) / 32); D.warps_per_block = 8;
    st.out(D.group_runs, D.n);
    st.out(D.cta, (D.n + 7) / 8);
    st.out(D.total, 1);
    st.out(D.list, n_runs);
  }
  const uint32_t grid = (n_runs - 1u) / 8u + 1u;
  // pinned items / runs are written in place; the others are staged once their numbers are known
  OutList<bf_commit_write> items(journaled ? journal->items : nullptr, journaled ? journal->items_cap : 0, true);
  OutList<uint32_t> listed(journaled ? journal->runs : nullptr, journaled ? std::min(journal->runs_cap, n_runs) : 0);
  if (journaled) {
    st.out(P.run_items, n_runs);
    st.out(P.cta, 2 * (size_t)grid);
    st.out(P.total, 2);
  }
  bf::RewriteParams W{};
  PassStage ps;
  if (rewrites) {   // the shared stage of bf_resident_status per warp for the joins
    if (int rc = plan_pass_stage(c, L, ps)) return rc;
    st.out(W.rw_runs, n_runs);
    st.out(W.rw_planes, (size_t)n_runs * 4u * L.words);
  }
  if (int rc = st.send(c, "bf_resident_commit (check)")) return rc;
  const size_t sent = st.size;
  if (P.arm.tim) {
    P.arm.timers = r->areas.d_timers; P.arm.timer_k = r->areas.timer_k; P.arm.now = arm->now;
    P.arm.decision = L.off_decision != BF_OFF_NONE; P.arm.out = P.counts + 5;
  }
  P.state = r->d_state; P.result = r->d_result; P.sched_rec = A.sched_rec;
  P.slots = c->slots_dev; P.n_slots = (uint32_t)c->slots_host.size();
  P.n_entries = n; P.n_runs = n_runs;
  P.words = L.words; P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.result_stride = L.result_stride;
  P.off_ready = L.off_ready; P.off_skip = L.off_skip; P.off_fail = L.off_fail; P.sched_stride = A.sched_stride;
  P.mark = r->d_mark; P.mark_value = r->mark_touched();
  // the list-mode parameters of a touched commit, as the sections stand (after a growth too)
  const uint32_t list_ctas = (uint32_t)c->sm_count * 4u;
  auto list_params = [&] {
    bf::CommitListParams LP{};
    LP.P = P; LP.list = by_list ? D.list : nullptr; LP.n_list = by_list ? D.total : n_up; LP.due = r->areas.d_due;
    return LP;
  };
  const bool was_all = r->commit_all;
  r->commit_all = true;   // until the call went through or was refused: a failed commit leaves every run due
  cudaError_t e = cudaSuccess;
  if (by_list) {
    D.due = r->areas.d_due; D.entries = P.entries; D.n_entries = n; D.n_runs = n_runs;
    if (e == cudaSuccess) e = bf::launch_due_list(D, s);
  }
  if (rewrites) {
    W.state = r->d_state; W.result = r->d_result; W.slots = c->slots_dev; W.n_slots = P.n_slots; W.runctl = A.runctl;
    W.n_runs = n_runs; W.warps_per_block = ps.wpb;
    W.words = L.words; W.state_stride = L.state_stride; W.off_phase = L.off_phase; W.off_decision = L.off_decision;
    W.off_child = L.off_child; W.topo_bytes = ps.topo; W.result_stride = L.result_stride;
    if (e == cudaSuccess)
      e = scope ? bf::launch_rewrites_list(W, by_list ? D.list : nullptr, by_list ? D.total : n_up, (uint32_t)c->sm_count * 2u,
                                           ps.smem(), s)
                : bf::launch_rewrites(W, ps.smem(), s);
    P.rw_runs = W.rw_runs; P.rw_planes = W.rw_planes; P.rewritten = P.counts + 7;
  }
  uint32_t* host = c->pinned->commit;
  unsigned long long* totals = c->pinned->list_totals;
  if (e == cudaSuccess) e = scope ? bf::launch_commit_list(list_params(), false, n_runs, list_ctas, s) : bf::launch_commit(P, false, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(host, P.offender, 8, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess && journaled) e = cudaMemcpyAsync(totals, P.total, 16, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess && by_list) e = cudaMemcpyAsync(totals + 2, D.total, 8, cudaMemcpyDeviceToHost, s);
  if (int rc = bf::end_call(c, e, "bf_resident_commit (check)")) return rc;
  c->stats.kernel_launches += (journaled ? 2 : 1) + (rewrites ? 1 : 0) + (by_list ? 3 : 0);
  if (scope) { scope->full = full ? 1u : 0u; scope->n_considered = full ? n_runs : (uint32_t)totals[2]; }
  uint64_t key;
  memcpy(&key, host, 8);
  if (key != ~0ull) {
    r->commit_all = was_all;   // refused: nothing written, no due bit cleared
    const uint32_t run = (uint32_t)(key >> 32), step = (uint32_t)(key >> 8) & 0xFFFFFFu, why = (uint32_t)key & 0xFFu;
    const std::string at = "run " + std::to_string(run) + " step " + std::to_string(step) + ": ";
    if (why == bf::kCommitOverflow)
      return refuse(run, step, at + "the run would hold more than " + std::to_string(r->areas.timer_k) + " armed timers", BF_ENOMEM);
    return refuse(run, step, at + (why == bf::kCommitNotLaunched ? "an entry names a step the tick did not launch"
                                   : why == bf::kCommitNotStop   ? "a BF_COMMIT_PHASE entry names a step that is not a stop step"
                                   : why == bf::kCommitNoPhase   ? "a launched stop step has no BF_COMMIT_PHASE entry"
                                                                 : "a timing that writes needs decision planes (BF_F_DECISION)"));
  }
  const uint64_t n_items = journaled ? totals[0] : 0;
  const uint32_t n_listed = journaled ? (uint32_t)totals[1] : 0;
  if (items.staged || listed.staged) {
    items.stage_at(st, n_items);
    listed.stage_at(st, n_listed);
    if (int rc = st.grow(c, sent, "bf_resident_commit")) return rc;
    if (P.arm.tim) P.arm.out = P.counts + 5;   // the arms' words behind the counts, where grow() may have moved them
    if (rewrites) { P.rw_runs = W.rw_runs; P.rw_planes = W.rw_planes; P.rewritten = P.counts + 7; }
  }
  P.items = items.dev; P.items_cap = items.cap;
  P.runs = listed.dev; P.runs_cap = (uint32_t)listed.cap;
  e = cudaSuccess;
  if (scope && full) e = cudaMemsetAsync(r->areas.d_due, 0xFF, r->areas.d_due.cap * 4, s);   // the runs at or past n_runs stay due
  if (e == cudaSuccess) e = scope ? bf::launch_commit_list(list_params(), true, n_runs, list_ctas, s) : bf::launch_commit(P, true, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(host, P.counts, 4 * n_counts, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = items.copy_async(n_items, s);
  if (e == cudaSuccess) e = listed.copy_async(n_listed, s);
  if (int rc = r->sync_in_place(c, e, "bf_resident_commit")) { r->state_changed(c); return rc; }
  c->stats.kernel_launches += 1;
  uint32_t k[8];
  memcpy(k, host, 4 * n_counts);
  out->n_runs_written = k[0]; out->n_skipped = k[1]; out->n_launched = k[2]; out->n_queued = k[3]; out->n_failed = k[4];
  if (arm) { arm->n_armed = k[5]; arm->next_deadline = k[6]; }
  if (journaled) { journal->n_items = n_items; journal->n_runs_listed = n_listed; }
  if (rewrites) *rewritten = k[7];
  if (k[0]) {   // as a delta: the written runs are touched, and the tick a schedule or a commit needs is over
    r->state_changed(c);
    r->pending += k[0];
  }
  r->commit_all = scope ? false : was_all;
  if (scope) { r->commit_form = form; r->commit_timings = c->timing_changes; }
  return BF_OK;
}

int bf_resident_commit_marks(bf_ctx* c, uint32_t h) {
  auto [g, r] = lock_resident(c, h);
  if (!r) return BF_EINVAL;
  BF_CUDA(c, cudaSetDevice(c->device));
  if (!r->areas.d_due) {
    const cudaError_t e = r->areas.d_due.alloc(RunAreas::due_words(r->cap));
    if (e != cudaSuccess) return fail(c, BF_ENOMEM, std::string("commit-due bits: ") + cudaGetErrorString(e));
  }
  r->commit_all = true;
  cudaError_t e = cudaMemsetAsync(r->areas.d_due, 0xFF, r->areas.d_due.cap * 4, c->stream);
  return bf::end_call(c, e, "bf_resident_commit_marks");
}

int bf_resident_commit_touched(bf_ctx* c, uint32_t h, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n, bf_commit_out* out,
                               bf_commit_arm* arm, bf_commit_journal* journal, uint32_t* n_rewritten, bf_commit_scope* scope) {
  if (!scope) {
    if (!c) return BF_EINVAL;
    std::lock_guard<std::mutex> g(c->mu);
    return fail(c, BF_EINVAL, "null bf_commit_scope");
  }
  const bool rewrites = (scope->flags & BF_COMMIT_SCOPE_REWRITES) != 0;
  return resident_commit(c, h, n_runs, entries, n, out, arm, journal, journal != nullptr, n_rewritten, rewrites, scope);
}

int bf_resident_commit_rewrites(bf_ctx* c, uint32_t h, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n,
                                bf_commit_out* out, bf_commit_arm* arm, bf_commit_journal* journal, uint32_t* n_rewritten) {
  return resident_commit(c, h, n_runs, entries, n, out, arm, journal, true, n_rewritten, true);
}

int bf_resident_commit_journal(bf_ctx* c, uint32_t h, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n, bf_commit_out* out,
                               bf_commit_arm* arm, bf_commit_journal* journal) {
  return resident_commit(c, h, n_runs, entries, n, out, arm, journal, true);
}

int bf_resident_commit_timed(bf_ctx* c, uint32_t h, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n, bf_commit_out* out,
                             bf_commit_arm* arm) {
  return resident_commit(c, h, n_runs, entries, n, out, arm, nullptr, false);
}

int bf_resident_commit(bf_ctx* c, uint32_t h, uint32_t n_runs, const bf_commit_entry* entries, uint32_t n, bf_commit_out* out) {
  return resident_commit(c, h, n_runs, entries, n, out, nullptr, nullptr, false);
}

// ---- run status (resident.cu) ---------------------------------------------------------------------------------------------------
// Read-only: the count, scan and list launches over the listed runs, the D2H copy of the event total, one synchronisation.  Pinned
// lists and outputs are used in place; staged records are copied with the total, staged events after the synchronisation, once
// their number is known (a second, blocking copy).
int bf_resident_status(bf_ctx* c, uint32_t h, uint32_t n_runs, const uint32_t* runs, uint32_t n, bf_status_out* out) {
  auto [g, r] = lock_resident(c, h);
  if (!out || out->struct_size != sizeof(bf_status_out)) return fail(c, BF_EINVAL, "null bf_status_out or bad struct_size");
  if (!r) return BF_EINVAL;
  const bf_layout& L = r->L;
  if (int rc = check_run_list(c, r, n_runs, runs, n)) return rc;
  if (n && !out->records) return fail(c, BF_EINVAL, "null records");
  if (out->events_cap && !out->events) return fail(c, BF_EINVAL, "null events with a non-zero events_cap");
  PassStage ps;
  if (int rc = plan_pass_stage(c, L, ps)) return rc;
  out->n_events = 0;
  if (n == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  if (int rc = bf::sync_slots(c, s)) return rc;
  const uint32_t grid = (n - 1u) / ps.wpb + 1u;
  // the list is at most n * 32 * words long (a run on a topology past steps_max but within the words is live): a larger
  // events_cap stages no more
  OutList<bf_status_rec> records(out->records, n);
  OutList<uint16_t> events(out->events, std::min<uint64_t>(out->events_cap, (uint64_t)n * 32u * L.words));
  bf::StatusParams P{};
  P.runs = runs ? static_cast<const uint32_t*>(bf::pinned_dev(runs)) : nullptr;
  CallStage st;
  if (runs && !P.runs) st.up(P.runs, runs, n);
  st.out(P.run_events, n);
  st.out(P.cta, grid);
  st.out(P.total, 1);
  records.stage(st);
  events.stage(st);
  if (int rc = st.send(c, "bf_resident_status")) return rc;
  P.records = records.dev; P.events = events.dev; P.events_cap = events.cap;
  P.state = r->d_state; P.slots = c->slots_dev; P.n_slots = (uint32_t)c->slots_host.size();
  P.runctl = r->areas_view().runctl;
  P.n = n; P.warps_per_block = ps.wpb;
  P.words = L.words; P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.off_decision = L.off_decision;
  P.off_child = L.off_child; P.topo_bytes = ps.topo;
  unsigned long long* totals = c->pinned->list_totals;
  cudaError_t e = bf::launch_status(P, ps.smem(), s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(totals, P.total, 8, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = records.copy_async(n, s);
  if (int rc = bf::end_call(c, e, "bf_resident_status")) return rc;
  c->stats.kernel_launches += 3;
  BF_CUDA(c, events.copy(totals[0]));
  out->n_events = totals[0];
  return BF_OK;
}

// ---- resyncs (resident.cu) ------------------------------------------------------------------------------------------------------
// Every check first, so a refused call changes nothing.  The caller's records go to the call's scratch in one H2D copy straight from
// the caller's buffer (not through CallStage's host image: they are the bulk of the call); then the count, scan and list launches,
// the D2H copy of the totals and one synchronisation.  Pinned drifted / items buffers are written in place, others copied after it.
int bf_resident_resync(bf_ctx* c, uint32_t h, bf_resync* q) {
  auto [g, r] = lock_resident(c, h);
  if (!q || q->struct_size != sizeof(bf_resync)) return fail(c, BF_EINVAL, "null bf_resync or bad struct_size");
  q->bad_run = BF_RESYNC_NONE;
  if (!r) return BF_EINVAL;
  const bf_layout& L = r->L;
  const uint32_t n = q->n, *runs = q->runs;
  if (int rc = check_run_list(c, r, q->n_runs, runs, n)) return rc;
  if (n && !q->records) return fail(c, BF_EINVAL, "null records");
  if ((q->drifted_cap && !q->drifted) || (q->items_cap && !q->items)) return fail(c, BF_EINVAL, "null drifted / items with a non-zero cap");
  if (q->flags & ~BF_RESYNC_CHECK) return fail(c, BF_EINVAL, "unknown flags");
  if (q->fields & ~(uint32_t)BF_RESYNC_ALL_FIELDS) return fail(c, BF_EINVAL, "unknown fields");
  const uint8_t* recs = static_cast<const uint8_t*>(q->records);
  for (uint32_t i = 0; i < n; ++i) {   // a run may hold only a slot a put has returned (alive or dropped since)
    uint32_t slot;
    memcpy(&slot, recs + (size_t)i * L.state_stride, 4);
    if (slot >= c->slots_host.size()) {
      q->bad_run = runs ? runs[i] : i;
      return fail(c, BF_EINVAL, "record of run " + std::to_string(q->bad_run) + " names a slot no put has returned");
    }
  }
  uint32_t fields = q->fields;   // a field the layout does not place is neither compared nor written
  if (L.off_cond == BF_OFF_NONE) fields &= ~BF_RESYNC_FIELD(BF_DELTA_COND);
  if (L.off_decision == BF_OFF_NONE) fields &= ~BF_RESYNC_FIELD(BF_DELTA_DECISION);
  if (L.off_child == BF_OFF_NONE) fields &= ~BF_RESYNC_FIELD(BF_DELTA_CHILD);
  PassStage ps;
  if (int rc = plan_pass_stage(c, L, ps)) return rc;
  q->n_drifted = q->n_written = 0;
  q->n_items = 0;
  if (n == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  if (int rc = bf::sync_slots(c, s)) return rc;
  const bool check = q->flags & BF_RESYNC_CHECK;
  const uint32_t grid = (n - 1u) / ps.wpb + 1u;
  // a run has at most one item per code, nibble and registered bit of the layout, and its flags byte: a larger cap stages no more
  const uint64_t per_run = 3ull * L.words * 32u + L.child_nibbles + 65u;
  OutList<uint32_t> drifted_list(q->drifted, std::min(q->drifted_cap, n));
  OutList<bf_drift> items_list(q->items, std::min<uint64_t>(q->items_cap, (uint64_t)n * per_run), true);
  bf::ResyncParams P{};
  P.runs = runs ? static_cast<const uint32_t*>(bf::pinned_dev(runs)) : nullptr;
  uint8_t* d_records;
  CallStage st;
  if (runs && !P.runs) st.up(P.runs, runs, n);
  st.out(d_records, (size_t)n * L.state_stride);
  st.out(P.run_items, n);
  st.out(P.cta, 2 * (size_t)grid);
  st.out(P.total, 2);
  drifted_list.stage(st);
  items_list.stage(st);
  if (int rc = st.send(c, "bf_resident_resync")) return rc;
  BF_CUDA(c, cudaMemcpyAsync(d_records, recs, (size_t)n * L.state_stride, cudaMemcpyHostToDevice, s));
  P.records = d_records;
  P.state = r->d_state; P.slots = c->slots_dev; P.n_slots = (uint32_t)c->slots_host.size();
  P.runctl = r->areas.d_runctl; P.areas = r->areas_view();
  P.mark = r->d_mark; P.mark_touched = r->mark_touched(); P.mark_must_list = r->mark_must_list();
  P.n = n; P.warps_per_block = ps.wpb;
  P.words = L.words; P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.off_cond = L.off_cond;
  P.off_decision = L.off_decision; P.off_child = L.off_child; P.child_nibbles = L.child_nibbles; P.topo_bytes = ps.topo;
  P.fields = fields; P.check = check;
  P.drifted = drifted_list.dev; P.drifted_cap = (uint32_t)drifted_list.cap;
  P.items = items_list.dev; P.items_cap = items_list.cap;
  unsigned long long* totals = c->pinned->list_totals;
  cudaError_t e = bf::launch_resync(P, ps.smem(), s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(totals, P.total, 16, cudaMemcpyDeviceToHost, s);
  if (check) {
    if (int rc = bf::end_call(c, e, "bf_resident_resync")) return rc;
  } else if (int rc = r->sync_in_place(c, e, "bf_resident_resync")) {
    r->state_changed(c);
    return rc;
  }
  c->stats.kernel_launches += 3;
  const uint64_t items = totals[0];
  const uint32_t drifted = (uint32_t)totals[1];
  if (!check && drifted) {   // as a commit that wrote: the evaluated snapshot and the tick end (before any copy can fail)
    r->state_changed(c);
    r->pending += drifted;
  }
  BF_CUDA(c, drifted_list.copy(drifted));
  BF_CUDA(c, items_list.copy(items));
  q->n_items = items;
  q->n_drifted = drifted;
  q->n_written = check ? 0 : drifted;
  return BF_OK;
}

// ---- side-area resyncs (resident.cu) ---------------------------------------------------------------------------------------------
// Every check first, on the host, so a refused call changes nothing.  Each selected area's rows go to the call's scratch in one H2D
// copy straight from the caller's array; then the count, scan and list launches, the D2H copy of the totals and one synchronisation.
// Pinned drifted / items buffers are written in place, others copied after it.
int bf_resident_resync_areas(bf_ctx* c, uint32_t h, bf_resync_areas* q) {
  auto [g, r] = lock_resident(c, h);
  if (!q || q->struct_size != sizeof(bf_resync_areas)) return fail(c, BF_EINVAL, "null bf_resync_areas or bad struct_size");
  q->bad_run = BF_RESYNC_NONE;
  if (!r) return BF_EINVAL;
  const bf_layout& L = r->L;
  const uint32_t n = q->n, *runs = q->runs, sel = q->areas;
  if (int rc = check_run_list(c, r, q->n_runs, runs, n)) return rc;
  if (q->flags & ~BF_RESYNC_CHECK) return fail(c, BF_EINVAL, "unknown flags");
  if (sel & ~BF_RESYNC_ALL_AREAS) return fail(c, BF_EINVAL, "unknown areas");
  const bool t_sel = sel & BF_RESYNC_AREA_TIMERS, s_sel = sel & BF_RESYNC_AREA_SCHED, c_sel = sel & BF_RESYNC_AREA_RUNCTL;
  if ((t_sel && !r->areas.timer_k) || (s_sel && !r->areas.d_sched_in) || (c_sel && !r->areas.d_runctl))
    return fail(c, BF_EINVAL, "a selected area the batch has no area for");
  if (n && ((t_sel && !q->timers) || (s_sel && !q->sched) || (c_sel && !q->runctl)))
    return fail(c, BF_EINVAL, "null array of a selected area");
  if ((q->drifted_cap && !q->drifted) || (q->items_cap && !q->items)) return fail(c, BF_EINVAL, "null drifted / items with a non-zero cap");
  const uint32_t K = r->areas.timer_k;
  auto refuse = [&](uint32_t i, const std::string& why) {
    q->bad_run = runs ? runs[i] : i;
    return fail(c, BF_EINVAL, "run " + std::to_string(q->bad_run) + ": " + why);
  };
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t run = runs ? runs[i] : i;
    if (t_sel) {   // canonical: armed slots first, strictly ascending by step; empty slots all NONE and zero
      const bf_timer_slot* row = q->timers + (size_t)i * K;
      bool empty_seen = false;
      for (uint32_t k = 0; k < K; ++k) {
        const bf_timer_slot& t = row[k];
        if (t.deadline == BF_TIMER_NONE) {
          if (t.step || t.code || t.reserved) return refuse(i, "an empty timer slot with non-zero bytes");
          empty_seen = true;
          continue;
        }
        if (empty_seen) return refuse(i, "an armed timer slot after an empty one");
        if (k && t.step <= row[k - 1].step) return refuse(i, "timer slots not strictly ascending by step");
        if (t.step >= L.steps_max || t.code > 3 || t.reserved) return refuse(i, "a timer slot's step, code or reserved byte");
        if (t.code != BF_DEC_PENDING && L.off_decision == BF_OFF_NONE) return refuse(i, "a non-PENDING timer code without decision planes");
      }
    }
    if (s_sel) {
      const bf_sched_put& s = q->sched[i];
      if (s.run != run || s.reserved[0] || s.reserved[1]) return refuse(i, "a limiter-input row's run or reserved words");
    }
    if (c_sel) {
      const bf_run_ctl& k = q->runctl[i];
      bool zero = k.saved_flags == 0;
      for (uint8_t b : k.reserved) zero = zero && b == 0;
      if (k.stop > BF_STOP_HOST || !zero) return refuse(i, "a run-control row's stop, saved_flags or reserved bytes");
    }
  }
  q->n_drifted = q->n_written = 0;
  q->n_items = 0;
  if (n == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  const bool check = q->flags & BF_RESYNC_CHECK;
  bf::ResyncAreasParams P{};
  P.warps_per_block = 8;
  const uint32_t grid = (n - 1u) / P.warps_per_block + 1u;
  // a run has at most two items per slot pair, five inputs and three run-control fields: a larger cap stages no more
  const uint64_t per_run = 2ull * K + 8u;
  OutList<uint32_t> drifted_list(q->drifted, std::min(q->drifted_cap, n));
  OutList<bf_drift> items_list(q->items, std::min<uint64_t>(q->items_cap, (uint64_t)n * per_run), true);
  P.runs = runs ? static_cast<const uint32_t*>(bf::pinned_dev(runs)) : nullptr;
  CallStage st;
  if (runs && !P.runs) st.up(P.runs, runs, n);
  if (t_sel) st.out(P.timers, (size_t)n * K);
  if (s_sel) st.out(P.sched, n);
  if (c_sel) st.out(P.runctl, n);
  st.out(P.run_items, n);
  st.out(P.cta, 2 * (size_t)grid);
  st.out(P.total, 4);
  drifted_list.stage(st);
  items_list.stage(st);
  if (int rc = st.send(c, "bf_resident_resync_areas")) return rc;
  auto up = [&](const void* dst, const void* src, size_t bytes) {
    return bytes ? cudaMemcpyAsync(const_cast<void*>(dst), src, bytes, cudaMemcpyHostToDevice, s) : cudaSuccess;
  };
  if (t_sel) BF_CUDA(c, up(P.timers, q->timers, (size_t)n * K * sizeof(bf_timer_slot)));
  if (s_sel) BF_CUDA(c, up(P.sched, q->sched, (size_t)n * sizeof(bf_sched_put)));
  if (c_sel) BF_CUDA(c, up(P.runctl, q->runctl, (size_t)n * sizeof(bf_run_ctl)));
  P.state = r->d_state; P.areas = r->areas_view();
  P.mark = r->d_mark; P.mark_touched = r->mark_touched();
  P.n = n;
  P.words = L.words; P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.off_decision = L.off_decision;
  P.sel = sel; P.fired_now = q->fired_now; P.check = check;
  P.drifted = drifted_list.dev; P.drifted_cap = (uint32_t)drifted_list.cap;
  P.items = items_list.dev; P.items_cap = items_list.cap;
  unsigned long long* totals = c->pinned->list_totals;
  cudaError_t e = bf::launch_resync_areas(P, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(totals, P.total, 32, cudaMemcpyDeviceToHost, s);
  if (check) {
    if (int rc = bf::end_call(c, e, "bf_resident_resync_areas")) return rc;
  } else if (int rc = r->sync_in_place(c, e, "bf_resident_resync_areas")) {
    r->state_changed(c);
    return rc;
  }
  c->stats.kernel_launches += 3;
  const uint64_t items = totals[0];
  const uint32_t drifted = (uint32_t)totals[1], written = check ? 0u : (uint32_t)totals[2], stopped = check ? 0u : (uint32_t)totals[3];
  if (stopped) {   // as bf_resident_runctl_put with a stop: the evaluated snapshot and the tick end (before any copy can fail)
    r->state_changed(c);
    r->pending += stopped;
  }
  BF_CUDA(c, drifted_list.copy(drifted));
  BF_CUDA(c, items_list.copy(items));
  q->n_items = items;
  q->n_drifted = drifted;
  q->n_written = written;
  return BF_OK;
}
