// abi.cu — the C ABI of include/bobrafrontier.h: context, batch evaluation, limiters.
//
// Host side of the boundary.  Plans the launch shape of a pass (run_pass) and drives H2D -> kernels -> D2H for the
// host-buffer entry points.  The topology arena is topology.cu, resident batches resident_abi.cu, device groups group.cu.
#include <stdlib.h>
#include <string.h>

#include <new>

#include "ctx.h"

using bf::cuda_fail; using bf::fail; using bf::round_up; using bf::round_up_sz;

// ---- host helpers of a pass, shared with resident_abi.cu (ctx.h) ----------------------------
namespace bf {

int check_layout(bf_ctx* c, const bf_layout& L) {
  if (L.steps_max == 0 || L.steps_max > BF_MAX_STEPS) return fail(c, BF_EINVAL, "layout.steps_max out of range");
  if (L.words != (L.steps_max + 31) / 32) return fail(c, BF_EINVAL, "layout.words != ceil(steps_max/32)");
  if (L.state_stride % 16 || L.result_stride % 16 || L.state_stride == 0 || L.result_stride == 0)
    return fail(c, BF_EINVAL, "strides must be non-zero multiples of 16");
  if (L.off_phase == BF_OFF_NONE || L.off_ready == BF_OFF_NONE || L.off_skip == BF_OFF_NONE)
    return fail(c, BF_EINVAL, "phase / ready / skip fields are mandatory");
  const uint32_t W = L.words;
  // 64-bit sums: a caller-supplied offset near 2^32 must not wrap past the bound
  auto in_state = [&](uint32_t off, uint32_t len) { return off == BF_OFF_NONE || (off % 4 == 0 && off >= 16 && (uint64_t)off + len <= L.state_stride); };
  auto in_res = [&](uint32_t off, uint32_t len) { return off == BF_OFF_NONE || (off % 4 == 0 && off >= 16 && (uint64_t)off + len <= L.result_stride); };
  if (L.child_nibbles > 0xFFFFu) return fail(c, BF_EINVAL, "layout.child_nibbles exceeds 65535");
  if (L.state_stride > (1u << 20) || L.result_stride > (1u << 20)) return fail(c, BF_EINVAL, "record stride exceeds 1 MiB");
  if (!in_state(L.off_phase, W * 16) || !in_state(L.off_cond, W * 8) || !in_state(L.off_decision, W * 8) ||
      !in_state(L.off_child, (L.child_nibbles + 1) / 2))
    return fail(c, BF_EINVAL, "state field outside the record");
  if (!in_res(L.off_ready, W * 4) || !in_res(L.off_skip, W * 4) || !in_res(L.off_fail, W * 4) ||
      !in_res(L.off_needs_cond, W * 4) || !in_res(L.off_skip_dep, W * 4) || !in_res(L.off_phase_out, W * 16))
    return fail(c, BF_EINVAL, "result field outside the record");
  return BF_OK;
}

uint32_t result_tail_of(const bf_layout& L) {
  uint32_t tail = (uint32_t)sizeof(bf_result_header);
  auto upd = [&](uint32_t off, uint32_t len) { if (off != BF_OFF_NONE && off + len > tail) tail = off + len; };
  upd(L.off_ready, L.words * 4); upd(L.off_skip, L.words * 4); upd(L.off_fail, L.words * 4);
  upd(L.off_needs_cond, L.words * 4); upd(L.off_skip_dep, L.words * 4); upd(L.off_phase_out, L.words * 16);
  return tail;
}

}  // namespace bf

// ---- one pass on device buffers: the plan of its launch shape, then its launches --------------
namespace {

constexpr uint32_t kSmemBudget = 227u * 1024u;   // shared memory a CTA may use
constexpr uint32_t kMinGroups = 8;               // the fewest slot groups per CTA that make a useful packed-lanes ring

bf::Knobs read_knobs() {
  auto is = [](const char* name, const char* value) { const char* e = getenv(name); return e && !strcmp(e, value); };
  auto num = [](const char* name) { const char* e = getenv(name); return e ? atoi(e) : 0; };
  bf::Knobs k;
  k.general = is("BF_KERNEL", "general"); k.blocked = is("BF_ASSIGN", "blocked");
  k.warps = num("BF_WARPS"); k.groups = num("BF_GROUPS"); k.stages = num("BF_STAGES");
  k.blocks_per_sm = num("BF_BLOCKS_PER_SM"); k.wq = num("BF_WQ"); k.pack_ctas = num("BF_PACK_CTAS");
  return k;
}

// the kernels of a pass, in the order of bf_stats.last_kernel for a pass over a whole batch
enum class Kernel : uint32_t { general, pack, two_tier };

// The launch shape of one pass, complete before anything is launched.
struct PassPlan {
  Kernel kernel = Kernel::general;
  // packed lanes: lanes per run (R = 32 / wq runs per warp trip), warps and slot groups per CTA, per-warp scratch bytes,
  // shared memory, grid
  uint32_t wq = 32, wq_log2 = 5, warps = 0, groups = 0, work = 0, smem = 0, grid = 0;
  // the general kernel, alone or as the second tier: ring stages, warps per CTA, build (occ2), per-warp scratch bytes,
  // shared memory, grid
  uint32_t g_stages = 0, g_wpb = 0, g_occ2 = 0, g_work = 0, g_smem = 0, g_grid = 0;
  // what the packed-lanes kernel takes on when it runs alone over a non-empty batch: the BF_EVAL_COUNTS_SET totals, a
  // compact tick's head words, a start under the previous pass (BF_EVAL_PIPELINED)
  bool counts_in_kernel = false, fused_heads = false, pipelined = false;
};

// Packed lanes (frontier_pack.cu, a group of R = 32 / Wq runs per warp trip) for single-pass batches whose records
// leave room for at least kMinGroups slot groups per SM; the one-run-per-warp kernel (frontier_kernel.cu) for the
// device fixpoint, for S > 512 and when every live topology has `parallel` steps.  Mixed batches: the packed kernel
// defers the runs whose topology has parallel steps to a device list that the general kernel then takes (second
// launch; exits at once when the list is empty).  BF_KERNEL=general forces the general kernel (A/B timing).
// Leaves pp.kernel general when the packed-lanes kernel does not take the pass.
void plan_pack(const bf_ctx* c, const bf_batch& b, const bf::Knobs& k, uint32_t stage_bytes, PassPlan& pp) {
  const bf_layout& L = b.layout;
  if ((b.flags & BF_EVAL_FIXPOINT) || L.words > 16 || c->n_with_parallel == c->n_alive || k.general) return;
  uint32_t wq = 1, lg = 0;
  while (wq < L.words) { wq <<= 1; lg++; }
  while (wq < (uint32_t)k.wq && wq < 32) { wq <<= 1; lg++; }   // fewer runs per group (lanes per run rounded up further)
  const uint32_t R = 32u / wq, max_warps = bf::frontier_pack_max_warps();
  // experiment knob (tools/build_variant.sh with -DPACK_MIN_BLOCKS=k -DPACK_MAX_WARPS=24/k): k packed-lanes CTAs per SM, each
  // with 1/k of the shared memory
  const uint32_t ctas_per_sm = k.pack_ctas >= 1 && k.pack_ctas <= 4 ? (uint32_t)k.pack_ctas : 1u;
  const uint32_t group_bytes = R * stage_bytes;
  // per-warp scratch (frontier_pack.cu): status pairs 512 B | fix-up words | walk table R x 16, in units of 256 bytes.  The
  // reservation is still that of the status-byte layout before it (R x st_stride bytes of status, st_stride = 256 at wq = 8,
  // 32 wq + 16 otherwise), 512 - 1024 bytes per warp more than the kernel reads: a smaller one moves slot groups and shared
  // memory of every launch shape, a change to be measured for itself (warps per CTA measured flat from 20 to 28, DESIGN §5).
  const uint32_t st_stride = wq == 8 ? 256u : 32u * wq + 16u;
  const uint32_t work = round_up(R * st_stride + 128u + 16u * R, 256);
  auto groups_for = [&](uint32_t warps) -> uint32_t {   // slot groups that fit beside `warps` scratch areas
    const uint32_t fixed = 128u + 768u + 256u + warps * work;   // 768: mbarriers + armed words of up to 64 groups; 256: scratch alignment
    const uint32_t cta_budget = kSmemBudget / ctas_per_sm - (ctas_per_sm > 1 ? 1024u : 0u);   // (the per-CTA reservation of the driver)
    const uint32_t n = fixed < cta_budget ? (cta_budget - fixed) / group_bytes : 0;
    return n > 64 ? 64 : n;
  };
  uint32_t nw = k.warps ? std::min((uint32_t)k.warps, max_warps) : max_warps;
  while (nw > 1 && groups_for(nw) < nw) --nw;               // never more warps than slot groups
  uint32_t ng = std::min(groups_for(nw), 32u * nw);   // never more slot groups than threads: thread i sets up slot group i (frontier_pack.cu)
  if ((uint32_t)k.groups >= nw && (uint32_t)k.groups <= ng) ng = (uint32_t)k.groups;
  if (ng < kMinGroups || ng < nw) return;   // records too large for a useful ring: one run per warp instead
  // a small batch gives a CTA only a few groups: no more warps and slot groups than it will use, so that the CTAs of
  // consecutive (pipelined) passes fit an SM side by side instead of waiting for each other's shared memory
  const uint32_t n_groups = (b.n_runs + R - 1) / R;
  const uint32_t slots_sm = (uint32_t)c->sm_count * ctas_per_sm;
  const uint32_t grid = slots_sm < n_groups ? slots_sm : (n_groups ? n_groups : 1);
  const uint32_t t_max = n_groups ? (n_groups + grid - 1) / grid : 1;
  pp.kernel = c->n_with_parallel != 0 ? Kernel::two_tier : Kernel::pack;
  pp.wq = wq; pp.wq_log2 = lg; pp.work = work; pp.grid = grid;
  pp.warps = std::min(nw, t_max); pp.groups = std::min(ng, t_max);
  pp.smem = 128u + round_up(pp.groups * 12u, 128) + pp.groups * group_bytes + 256u + pp.warps * work;
}

// The general kernel's shape (alone, or the second tier of a two-tier pass), planned once per layout, largest record,
// variant and knobs and cached on the ctx: as many resident warps per SM as registers / shared memory allow — the pass is
// latency/issue bound before it is HBM bound — then ring depth: >= 2 stages keep the next trip's TMA copies in flight
// under the current evaluation.  P: the pass's parameters as far as the choice of build reads them (no run list yet).
int plan_general(bf_ctx* c, const bf_batch& b, const bf::Knobs& k, const bf::KParams& P, uint32_t rec_bytes, bool run_list,
                 PassPlan& pp) {
  const bf_layout& L = b.layout;
  const bool two_tier = pp.kernel == Kernel::two_tier;
  const uint32_t work = round_up(4 * L.words, 16) + 32 * L.words + 16;  // fix-up mask words + status bytes + PAD guard
  const uint32_t variant = (b.flags & BF_EVAL_FIXPOINT) | (P.any_parallel << 8) | ((two_tier ? 1u : 0u) << 9) | (L.fields << 16);
  bf_ctx::Plan& pl = c->plan[run_list ? 1 : 0];
  if (pl.wpb == 0 || pl.key_stride != L.state_stride || pl.key_words != L.words || pl.key_rec != rec_bytes ||
      pl.key_variant != variant || !(pl.key_knobs == k)) {
    bf_ctx::Plan best{};
    uint32_t best_score = 0;
    for (uint32_t st = 1; st <= 4; ++st) {
      if (k.stages && (uint32_t)k.stages != st) continue;
      for (uint32_t wpb = 24; wpb >= 1; wpb = (wpb > 4 ? wpb - 4 : wpb - 1)) {   // 24 / 20: the 80-register build (frontier_kernel.cu)
        if (k.warps && !two_tier && (uint32_t)k.warps != wpb) continue;
        if (wpb > 16 && (two_tier || run_list)) continue;   // the run-list builds are the 16-warp build only
        const uint32_t smem = 128 + wpb * (st * P.stage_bytes + work + 64);
        if (smem > kSmemBudget) continue;
        uint32_t occ2 = 0;
        int ctas = bf::frontier_max_blocks_per_sm(P, wpb * 32, smem, &occ2);
        if (ctas < 1) continue;
        if (ctas > 2) ctas = 2;   // the builds are compiled for one or two resident CTAs; many small CTAs measured slower
        if (k.blocks_per_sm >= 1 && k.blocks_per_sm < ctas) ctas = k.blocks_per_sm;
        const uint32_t warps_sm = (uint32_t)ctas * wpb;
        const uint32_t depth = st >= 3 ? 2 : st - 1;           // 0, 1, 2, 2
        const uint32_t score = warps_sm * 16 + depth * 24 + (wpb >= 8 ? 2 : 0) + (4 - st);
        if (score > best_score) {
          best_score = score;
          best.stages = st; best.wpb = wpb; best.per_sm = (uint32_t)ctas; best.occ2 = occ2; best.smem = smem;
        }
      }
    }
    if (best.wpb == 0) return fail(c, BF_ETOPO, "topology record + run state do not fit shared memory");
    best.key_stride = L.state_stride; best.key_words = L.words; best.key_rec = rec_bytes; best.key_variant = variant;
    best.key_knobs = k;
    pl = best;
  }
  // a run list (a touched tick, or the runs the packed-lanes kernel deferred) takes the 16-warp run-list build, one CTA per SM
  const bool listed = two_tier || run_list;
  const uint32_t blocks = (b.n_runs + pl.wpb - 1) / pl.wpb;
  pp.g_stages = pl.stages; pp.g_wpb = pl.wpb; pp.g_occ2 = listed ? 0 : pl.occ2; pp.g_work = work; pp.g_smem = pl.smem;
  pp.g_grid = std::min((uint32_t)c->sm_count * (listed ? 1u : pl.per_sm), blocks ? blocks : 1u);
  return BF_OK;
}

}  // namespace

namespace bf {

// One pass on device buffers: its plan, then its launches.
// run_list (touched ticks): the pass takes the runs run_list[0 .. *run_list_count) (b.n_runs bounds the count) and writes
// each run's record at its own index.  heads (compact ticks): where the pass may leave the head words itself.
int run_pass(bf_ctx* c, const bf_batch& b, const uint8_t* d_state, uint8_t* d_result, bf_expansion* d_exp,
             unsigned long long* d_counts, cudaStream_t stream, const uint32_t* run_list, const uint32_t* run_list_count,
             FusedHeads* heads) {
  const bf_layout& L = b.layout;
  if (int rc = sync_slots(c, stream)) return rc;
  if (c->n_alive == 0) return fail(c, BF_ETOPO, "no topology has been uploaded");
  // the largest record a run of this batch can stage: topologies wider than the layout are rejected by the kernels
  uint32_t batch_rec_bytes = largest_record(c, L.words);
  if (batch_rec_bytes == 0) batch_rec_bytes = 64;   // no topology fits the layout: every run will be marked dead
  const Knobs k = read_knobs();

  KParams P{};
  P.state = d_state; P.result = d_result; P.slots = c->slots_dev; P.ff_mask = c->ff_dev;
  P.counts = (b.flags & BF_EVAL_NO_COUNTS) ? nullptr : d_counts;
  P.n_slots = (uint32_t)c->slots_host.size();
  P.n_runs = b.n_runs; P.flags = b.flags; P.max_iter = b.max_iterations;
  P.any_parallel = c->n_with_parallel != 0;
  P.words = L.words;
  P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.off_cond = L.off_cond;
  P.off_decision = L.off_decision; P.off_child = L.off_child;
  P.result_stride = L.result_stride; P.off_ready = L.off_ready; P.off_skip = L.off_skip; P.off_fail = L.off_fail;
  P.off_needs_cond = L.off_needs_cond; P.off_skip_dep = L.off_skip_dep; P.off_phase_out = L.off_phase_out;
  P.result_tail = result_tail_of(L);
  P.run_blocked = k.blocked;
  P.topo_buf_bytes = round_up(batch_rec_bytes, 16);
  P.stage_bytes = L.state_stride + P.topo_buf_bytes;
  const bool want_exp = (b.flags & BF_EVAL_EXPANSION) && d_exp != nullptr;

  // ---- the plan ----
  PassPlan pp;
  plan_pack(c, b, k, P.stage_bytes, pp);
  if (pp.kernel != Kernel::pack)
    if (int rc = plan_general(c, b, k, P, batch_rec_bytes, run_list != nullptr, pp)) return rc;
  const bool alone = pp.kernel == Kernel::pack && b.n_runs != 0;
  // BF_EVAL_COUNTS_SET: the packed-lanes kernel alone publishes the totals itself (last CTA out); every other shape of a pass
  // (two tiers, the general kernel, expansion counts, an empty batch) zeroes the block first and adds as usual
  const bool counts_set = (b.flags & BF_EVAL_COUNTS_SET) && P.counts != nullptr;
  pp.counts_in_kernel = counts_set && alone && !want_exp;
  pp.fused_heads = heads && alone && !run_list;
  // BF_EVAL_PIPELINED applies to a pass that is the packed-lanes kernel alone and touches the counts only behind its wait
  pp.pipelined = alone && !want_exp && (pp.counts_in_kernel || P.counts == nullptr);

  // ---- the launches ----
  if (want_exp) {
    if (int rc = c->d_exp_counts.ensure(c, b.n_runs)) return rc;
    if (int rc = c->d_offsets.ensure(c, b.n_runs)) return rc;
    if (int rc = c->d_block_sums.ensure(c, (size_t)(b.n_runs + 1023) / 1024 + 1)) return rc;
    P.exp_counts = c->d_exp_counts;
  }
  if (counts_set && !pp.counts_in_kernel) BF_CUDA(c, cudaMemsetAsync(P.counts, 0, sizeof(bf_counts), stream));
  P.acc = pp.counts_in_kernel ? c->d_acc + 8 * (size_t)(c->acc_seq++ % bf_ctx::kAccSlots) : nullptr;
  if (pp.fused_heads) { P.head = heads->head; P.head_sums = heads->sums; }
  if (heads) heads->done = pp.fused_heads;
  if (!pp.pipelined) P.flags &= ~BF_EVAL_PIPELINED;
  P.run_list = run_list; P.run_list_count = run_list_count;
  const bool pack = pp.kernel != Kernel::general;
  if (pack) {
    P.wq = pp.wq; P.wq_log2 = pp.wq_log2; P.warps_per_block = pp.warps; P.slot_groups = pp.groups; P.stages = 1;
    P.work_bytes = pp.work;
  } else {
    P.wq = 32u; P.wq_log2 = 5u; P.warps_per_block = pp.g_wpb; P.stages = pp.g_stages; P.occ2 = pp.g_occ2;
    P.work_bytes = pp.g_work;
  }
  if (pp.kernel == Kernel::two_tier) {
    if (int rc = c->d_defer.ensure(c, (size_t)b.n_runs + 1)) return rc;
    P.defer_count = c->d_defer;
    P.defer_list = c->d_defer + 1;
  }
  if (b.n_runs) {
    if (pp.kernel == Kernel::two_tier) BF_CUDA(c, cudaMemsetAsync(c->d_defer, 0, sizeof(uint32_t), stream));
    if (pack) BF_CUDA(c, launch_frontier_pack(P, pp.grid, pp.smem, stream));
    else BF_CUDA(c, launch_frontier(P, pp.g_grid, pp.g_smem, stream));
    c->stats.kernel_launches += 1;
    if (pp.kernel == Kernel::two_tier) {  // second tier: the general kernel over the deferred runs
      KParams P2 = P;
      P2.defer_list = nullptr; P2.defer_count = nullptr;
      P2.run_list = c->d_defer + 1; P2.run_list_count = c->d_defer;
      P2.work_bytes = pp.g_work; P2.stages = pp.g_stages; P2.warps_per_block = pp.g_wpb; P2.occ2 = pp.g_occ2; P2.wq = 32; P2.wq_log2 = 5;
      BF_CUDA(c, launch_frontier(P2, pp.g_grid, pp.g_smem, stream));
      c->stats.kernel_launches += 1;
    }
    if (want_exp) {
      uint32_t nl = 0;
      BF_CUDA(c, launch_expansion(P, c->d_block_sums, c->d_offsets, d_exp, b.expansion_cap, stream, &nl));
      c->stats.kernel_launches += nl;
    }
  }
  c->stats.last_kernel = (uint32_t)pp.kernel + (run_list ? 3u : 0u); c->stats.last_runs_per_trip = 32u / pp.wq;
  c->stats.last_grid = pack ? pp.grid : pp.g_grid; c->stats.last_block = (pack ? pp.warps : pp.g_wpb) * 32;
  c->stats.last_smem_bytes = pack ? pp.smem : pp.g_smem; c->stats.last_stages = pack ? pp.groups : pp.g_stages;
  return BF_OK;
}

// the device address of a buffer in pinned host memory (bf_alloc_pinned, cudaHostAlloc / cudaHostRegister), else nullptr
void* pinned_dev(const void* p) {
  cudaPointerAttributes at{};
  if (p && cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer) return at.devicePointer;
  cudaGetLastError();   // an unregistered host pointer is not an error here
  return nullptr;
}

// ---- compact results: masks -> heads + 16-bit events on the device, then two small D2H copies ----
// Enqueue on `s` (after the passes that wrote d_result): compaction kernels, D2H of the head words and of a first slice of the
// event list sized from the previous list (+ 3 % + slack; none when the kernel posts the list).  The exact length arrives after
// the sync, with the counts, in the pinned tail the last kernel writes; compact_finish then fetches the rest.

// what every compaction takes from the layout and the ctx: the result fields it reads, and the pinned tail its last kernel
// writes with the counts and the rejected-delta counter (the kernel reads and clears it) when asked for them
CompactParams compact_params(bf_ctx* c, const bf_layout& L, uint32_t n_runs, bool want_counts, bool want_rejected) {
  CompactParams P{};
  P.n_runs = n_runs; P.words = L.words; P.result_stride = L.result_stride; P.result_tail = result_tail_of(L);
  P.off_ready = L.off_ready; P.off_skip = L.off_skip;
  P.off_fail = L.off_fail; P.off_needs_cond = L.off_needs_cond; P.off_skip_dep = L.off_skip_dep;
  P.host_tail = &c->pinned->tail; P.counts = want_counts ? c->d_counts.p : nullptr; P.rejected = want_rejected ? c->d_rejected.p : nullptr;
  return P;
}

int events_first(bf_ctx* c, uint16_t* events, uint64_t prev, uint64_t slack, uint64_t cap, bool posted, cudaStream_t s, uint64_t& first) {
  const uint64_t n = posted ? 0 : std::min(prev + prev / 32 + slack, cap);
  first = posted ? cap : n;   // posted: the whole list is in the caller's buffer after the synchronise
  if (n) BF_CUDA(c, cudaMemcpyAsync(events, c->d_events, (size_t)n * sizeof(uint16_t), cudaMemcpyDeviceToHost, s));
  return BF_OK;
}

// head words + the scratch block of a compaction (zeroed once; the kernels leave it clean): before the pass, so that a fused
// pass can write into them
int compact_prepare(bf_ctx* c, uint32_t n_runs, cudaStream_t s) {
  if (int rc = c->d_head.ensure(c, n_runs ? n_runs : 1)) return rc;
  const size_t cap_before = c->d_cblock.cap;
  if (int rc = c->d_cblock.ensure(c, 2 * ((size_t)(n_runs + 511) / 512 + 1) + 2)) return rc;
  if (c->d_cblock.cap != cap_before) c->cblock_clean = false;
  if (!c->cblock_clean) {
    BF_CUDA(c, cudaMemsetAsync(c->d_cblock, 0, c->d_cblock.cap * sizeof(unsigned long long), s));
    c->cblock_clean = true;
  }
  return BF_OK;
}
unsigned long long* cblock_sums(bf_ctx* c, uint32_t which) { return c->d_cblock + 2 + (size_t)which * ((c->d_cblock.cap - 2) / 2); }

int compact_enqueue(bf_ctx* c, const bf_layout& L, const uint8_t* d_result, const uint8_t* d_prev, uint32_t n_runs, bf_compact_out* out,
                    cudaStream_t s, uint64_t& first_slice, bool with_rejected, bool heads_done) {
  const uint64_t cap = out->events ? out->events_cap : 0;
  if (int rc = compact_prepare(c, n_runs, s)) return rc;
  if (int rc = c->d_events.ensure(c, cap ? (size_t)cap : 1)) return rc;
  CompactParams P = compact_params(c, L, n_runs, true, with_rejected);
  P.result = d_result; P.prev_result = d_prev; P.head = c->d_head; P.cap = cap;
  P.block_sums = cblock_sums(c, c->cblock_flip); P.zero_sums = cblock_sums(c, c->cblock_flip ^ 1u); P.total = c->d_cblock;
  P.zero_len = (uint32_t)((c->d_cblock.cap - 2) / 2);
  P.heads_done = heads_done ? 1u : 0u;
  c->cblock_flip ^= 1u;   // the next compaction (and a pass fused with it) uses the buffer this one leaves zeroed
  // a head buffer in pinned host memory (bf_alloc_pinned, cudaHostAlloc / cudaHostRegister) gets the head words posted by the
  // kernel itself; any other buffer gets them by a download
  if (out->head && n_runs && !getenv("BF_NO_ZC_HEADS")) P.host_head = static_cast<uint32_t*>(pinned_dev(out->head));
  // the event list likewise: posted by the emit kernel, no download
  uint16_t* p_events = cap && !getenv("BF_NO_ZC_EVENTS") ? static_cast<uint16_t*>(pinned_dev(out->events)) : nullptr;
  P.events = p_events ? p_events : c->d_events;
  if (n_runs == 0) BF_CUDA(c, cudaStreamSynchronize(s));   // the empty case stores to the pinned block from the host
  c->cblock_clean = false;   // until the call has gone through (pass_end sets it again after the sync)
  BF_CUDA(c, bf::launch_compact(P, s));
  c->stats.kernel_launches += n_runs ? (heads_done ? 1 : 2) : 0;
  if (int rc = events_first(c, out->events, c->last_events, 4096, cap, p_events != nullptr, s, first_slice)) return rc;
  if (out->head && n_runs && !P.host_head) BF_CUDA(c, cudaMemcpyAsync(out->head, c->d_head, (size_t)n_runs * 4, cudaMemcpyDeviceToHost, s));
  return BF_OK;
}
// after the stream has been synchronised: fetch what the first slice missed; the length sizes the next first slice (prev)
int compact_finish(bf_ctx* c, bf_compact_out* out, uint64_t first_slice, uint64_t& prev) {
  const ResultTail& tail = c->pinned->tail;
  const uint64_t cap = out->events ? out->events_cap : 0;
  const uint64_t have = tail.events < cap ? tail.events : cap;
  if (have > first_slice)
    BF_CUDA(c, cudaMemcpy(out->events + first_slice, c->d_events + first_slice, (size_t)(have - first_slice) * sizeof(uint16_t),
                          cudaMemcpyDeviceToHost));
  out->n_events = tail.events;
  out->n_listed = (uint32_t)tail.listed;
  prev = tail.events;
  return BF_OK;
}

// ---- the chunked pipeline of a pass between host buffers and the device: bf_eval, bf_eval_compact, each shard of bf_group_eval,
// and the full resident ticks (resident_abi.cu), which keep their state on the device and so upload nothing ----
// Large batches are cut into chunks of runs (runs are independent) so that the upload of chunk k+1, the pass of chunk k and the
// download of chunk k-1 overlap on three streams: PCIe is full duplex and the pass itself is ~5x faster than either copy, so the
// call costs about max(H2D, D2H) instead of their sum.

// The chunk count of a call that moves `bytes` through the pipeline: one below 2 MiB, else bytes / per_chunk rounded, at least
// at_least; BF_E2E_CHUNKS overrides it there (tools/e2e_sweep.py sweeps it).  Several chunks need the copy streams and events,
// created on first use.
int plan_chunks(bf_ctx* c, size_t bytes, size_t per_chunk, uint32_t at_least, uint32_t& chunks) {
  chunks = 1;
  if (bytes >= (2u << 20)) {
    chunks = std::max((uint32_t)((bytes + per_chunk / 2) / per_chunk), at_least);
    if (const char* e = getenv("BF_E2E_CHUNKS")) chunks = (uint32_t)atoi(e);
    chunks = std::clamp(chunks, 1u, bf_ctx::kMaxChunks);
  }
  if (chunks == 1 || c->pipe_ready) return BF_OK;
  if (!c->s_in) BF_CUDA(c, cudaStreamCreateWithFlags(&c->s_in, cudaStreamNonBlocking));
  if (!c->s_out) BF_CUDA(c, cudaStreamCreateWithFlags(&c->s_out, cudaStreamNonBlocking));
  for (uint32_t k = 0; k < bf_ctx::kMaxChunks; ++k) {
    if (!c->ev_in[k]) BF_CUDA(c, cudaEventCreateWithFlags(&c->ev_in[k], cudaEventDisableTiming));
    if (!c->ev_k[k]) BF_CUDA(c, cudaEventCreateWithFlags(&c->ev_k[k], cudaEventDisableTiming));
  }
  c->pipe_ready = true;
  return BF_OK;
}

// The pass over db.n_runs runs as `chunks` passes on c->stream that add into c->d_counts.  h_state (optional): the host records,
// each chunk's uploaded in front of its pass; h_result (optional): where each chunk's result records are downloaded behind its
// pass.  The copies run on s_in / s_out when there are several chunks.  taper: chunk sizes shrink linearly (weights c, c-1, .., 1):
// big early copies overlap best, a small last chunk leaves a short un-overlapped tail (kernel + download of that chunk).
int chunked_pass(bf_ctx* c, bf_batch db, uint32_t chunks, bool taper, uint8_t* d_state, uint8_t* d_result, const uint8_t* h_state,
                 uint8_t* h_result, bf_expansion* d_exp, FusedHeads* heads) {
  const bf_layout& L = db.layout;
  const size_t n = db.n_runs;
  const bool piped = chunks > 1;
  cudaStream_t s = c->stream, s_in = piped ? c->s_in : s, s_out = piped ? c->s_out : s;
  for (uint32_t k = 0; k < chunks; ++k) {
    size_t lo = n * k / chunks, hi = n * (k + 1) / chunks;
    if (taper && piped) {
      const uint64_t tot = (uint64_t)chunks * (chunks + 1) / 2;
      auto cum = [&](uint32_t kk) { return (uint64_t)kk * chunks - (uint64_t)kk * (kk - 1) / 2; };  // sum of the first kk weights
      lo = (size_t)(n * cum(k) / tot);
      hi = (size_t)(n * cum(k + 1) / tot);
    }
    const size_t so = lo * L.state_stride, ro = lo * L.result_stride;
    if (h_state) {
      if (hi > lo) BF_CUDA(c, cudaMemcpyAsync(d_state + so, h_state + so, (hi - lo) * L.state_stride, cudaMemcpyHostToDevice, s_in));
      if (piped) {
        BF_CUDA(c, cudaEventRecord(c->ev_in[k], s_in));
        BF_CUDA(c, cudaStreamWaitEvent(s, c->ev_in[k], 0));
      }
    }
    db.n_runs = (uint32_t)(hi - lo);
    if (int rc = run_pass(c, db, d_state + so, d_result + ro, d_exp, c->d_counts, s, nullptr, nullptr, heads)) return rc;
    if (piped) {
      BF_CUDA(c, cudaEventRecord(c->ev_k[k], s));
      BF_CUDA(c, cudaStreamWaitEvent(s_out, c->ev_k[k], 0));
    }
    if (hi > lo && h_result)
      BF_CUDA(c, cudaMemcpyAsync(h_result + ro, d_result + ro, (hi - lo) * L.result_stride, cudaMemcpyDeviceToHost, s_out));
  }
  return BF_OK;
}

// behind the chunks: the compaction of the records, whose last kernel posts the counts in the pinned tail, or the counts alone
int pass_results(bf_ctx* c, const bf_layout& L, const uint8_t* d_result, const uint8_t* d_prev, uint32_t n_runs, bf_compact_out* co,
                 uint64_t& first_slice, bool with_rejected, bool heads_done) {
  if (co) return compact_enqueue(c, L, d_result, d_prev, n_runs, co, c->stream, first_slice, with_rejected, heads_done);
  BF_CUDA(c, cudaMemcpyAsync(c->pinned->tail.counts, c->d_counts, sizeof(bf_counts), cudaMemcpyDeviceToHost, c->stream));
  return BF_OK;
}

// The end of a pipelined call whose enqueueing returned rc: never return while a copy that touches the caller's buffers is still in
// flight (the first error wins).  A failed call leaves the self-cleaning scratch in an unknown state, to be zeroed before its next
// use; a compaction that went through has left its scratch zeroed.
int pass_end(bf_ctx* c, int rc, uint32_t chunks, bool uploaded, bool compacted) {
  cudaError_t es = cudaStreamSynchronize(c->stream);
  if (chunks > 1) {
    const cudaError_t ei = uploaded ? cudaStreamSynchronize(c->s_in) : cudaSuccess, eo = cudaStreamSynchronize(c->s_out);
    if (es == cudaSuccess) es = ei != cudaSuccess ? ei : eo;
  }
  if (rc == BF_OK && es != cudaSuccess) rc = cuda_fail(c, es, "cudaStreamSynchronize");
  if (rc != BF_OK) {
    c->cblock_clean = false; c->rejected_clean = false;
    return rc;
  }
  if (compacted) c->cblock_clean = true;
  c->stats.last_eval_chunks = chunks;
  return BF_OK;
}

// A pass went through: its records are what bf_schedule reads, and its counts and event list go to the caller.  prev: the
// event count that sizes the first slice of the next list of this kind (compact_finish).
int publish_pass(bf_ctx* c, uint32_t n_runs, const bf_layout& L, const uint8_t* d_state, const uint8_t* d_result, bf_counts* counts,
                 bf_compact_out* co, uint64_t first_slice, uint64_t& prev) {
  c->snap = {true, n_runs, L, d_state, d_result};
  if (counts) *counts = c->pinned->counts();
  return co ? compact_finish(c, co, first_slice, prev) : BF_OK;
}

}  // namespace bf

// =============================================================================== C ABI
extern "C" {

uint32_t bf_abi_version(void) { return BF_ABI_VERSION; }

const char* bf_strerror(int status) {
  switch (status) {
    case BF_OK: return "ok";
    case BF_EINVAL: return "invalid argument";
    case BF_ENOMEM: return "out of memory";
    case BF_ECUDA: return "CUDA error";
    case BF_ENCCL: return "collective error";
    case BF_ETOPO: return "topology rejected";
    case BF_ENODEV: return "no usable device";
    default: return "unknown status";
  }
}

const char* bf_last_error(const bf_ctx* ctx) { return ctx ? ctx->err.c_str() : "null ctx"; }

int bf_create(bf_ctx** out, const bf_config* cfg) {
  if (!out) return BF_EINVAL;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return BF_ENODEV; }
  const int dev = cfg ? cfg->device : 0;
  if (dev < 0 || dev >= ndev) return BF_ENODEV;
  cudaDeviceProp prop{};
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return BF_ECUDA;
  if (prop.major != 9 || prop.minor != 0) return BF_ENODEV;  // built for sm_90a only: the cubin loads on compute capability 9.0 alone
  bf_ctx* c = new (std::nothrow) bf_ctx();
  if (!c) return BF_ENOMEM;
  c->device = dev;
  c->sm_count = prop.multiProcessorCount;
  if (cfg && (cfg->flags & 0xFFu) && (int)(cfg->flags & 0xFFu) < c->sm_count) c->sm_count -= (int)(cfg->flags & 0xFFu);   // BF_CFG_RESERVE_SMS
  c->stats.sm_count = (uint32_t)prop.multiProcessorCount;
  if (cudaSetDevice(dev) != cudaSuccess || cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
      c->d_counts.alloc(sizeof(bf_counts) / 8) != cudaSuccess ||
      c->d_acc.alloc(bf_ctx::kAccSlots * 8) != cudaSuccess || cudaMemset(c->d_acc, 0, bf_ctx::kAccSlots * 64) != cudaSuccess ||
      cudaHostAlloc(&c->pinned, sizeof *c->pinned, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    bf_destroy(c);  // releases whatever was created
    return BF_ECUDA;
  }
  if (cfg && cfg->arena_bytes) {
    std::lock_guard<std::mutex> g(c->mu);
    if (bf::grow_arena(c, (size_t)cfg->arena_bytes) != BF_OK) { bf_destroy(c); return BF_ENOMEM; }
  }
  if (cfg && cfg->max_topologies) { c->meta.reserve(cfg->max_topologies); c->slots_host.reserve(cfg->max_topologies); c->ff_host.reserve((size_t)cfg->max_topologies * bf::FF_STRIDE); }
  *out = c;
  return BF_OK;
}

void bf_destroy(bf_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) { cudaStreamSynchronize(c->stream); cudaStreamDestroy(c->stream); }
  if (c->s_in) cudaStreamDestroy(c->s_in);
  if (c->s_out) cudaStreamDestroy(c->s_out);
  for (uint32_t k = 0; k < bf_ctx::kMaxChunks; ++k) {
    if (c->ev_in[k]) cudaEventDestroy(c->ev_in[k]);
    if (c->ev_k[k]) cudaEventDestroy(c->ev_k[k]);
  }
  cudaFreeHost(c->pinned);
  if (c->part_tails) cudaFreeHost(c->part_tails);
  if (c->span_totals) cudaFreeHost(c->span_totals);
  delete c;   // the device buffers of the ctx and of its resident batches free themselves
}

int bf_layout_init(bf_layout* out, uint32_t steps_max, uint32_t child_nibbles, uint32_t fields) {
  if (!out || steps_max == 0 || steps_max > BF_MAX_STEPS) return BF_EINVAL;
  bf_layout L{};
  L.steps_max = steps_max;
  L.words = (steps_max + 31) / 32;
  L.fields = fields;
  L.child_nibbles = (fields & BF_F_CHILD) ? child_nibbles : 0;
  uint32_t off = sizeof(bf_run_header);
  L.off_phase = off; off += L.words * 16;
  L.off_cond = BF_OFF_NONE; L.off_decision = BF_OFF_NONE; L.off_child = BF_OFF_NONE;
  if (fields & BF_F_COND) { L.off_cond = off; off += L.words * 8; }
  if (fields & BF_F_DECISION) { L.off_decision = off; off += L.words * 8; }
  if (fields & BF_F_CHILD) { L.off_child = off; off += round_up((L.child_nibbles + 1) / 2, 4); }
  L.state_stride = round_up(off, 16);
  off = sizeof(bf_result_header);
  L.off_ready = off; off += L.words * 4;
  L.off_skip = off; off += L.words * 4;
  L.off_fail = L.off_needs_cond = L.off_skip_dep = L.off_phase_out = BF_OFF_NONE;
  if (fields & BF_F_OUT_FAIL) { L.off_fail = off; off += L.words * 4; }
  if (fields & BF_F_OUT_NEEDS_COND) { L.off_needs_cond = off; off += L.words * 4; }
  if (fields & BF_F_OUT_SKIP_DEP) { L.off_skip_dep = off; off += L.words * 4; }
  if (fields & BF_F_OUT_PHASE) { L.off_phase_out = off; off += L.words * 16; }
  L.result_stride = round_up(off, 16);
  *out = L;
  return BF_OK;
}

int bf_eval_device(bf_ctx* c, const bf_batch* b, void* stream) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  if (!b || b->struct_size != sizeof(bf_batch)) return fail(c, BF_EINVAL, "bad bf_batch.struct_size");
  if (int rc = bf::check_layout(c, b->layout)) return rc;
  if (b->n_runs && (!b->state || !b->result)) return fail(c, BF_EINVAL, "null state/result");
  BF_CUDA(c, cudaSetDevice(c->device));
  return bf::run_pass(c, *b, static_cast<const uint8_t*>(b->state), static_cast<uint8_t*>(b->result), b->expansion,
                  reinterpret_cast<unsigned long long*>(b->counts), static_cast<cudaStream_t>(stream));
}

}  // extern "C"

namespace bf {

int eval_host(bf_ctx* c, const bf_batch* b, bf_compact_out* co) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  if (!b || b->struct_size != sizeof(bf_batch)) return fail(c, BF_EINVAL, "bad bf_batch.struct_size");
  if (co && co->struct_size != sizeof(bf_compact_out)) return fail(c, BF_EINVAL, "bad bf_compact_out.struct_size");
  if (co && co->events_cap && !co->events) return fail(c, BF_EINVAL, "null events with a non-zero events_cap");
  if (int rc = bf::check_layout(c, b->layout)) return rc;
  if (b->n_runs && (!b->state || (!b->result && !co))) return fail(c, BF_EINVAL, "null state/result");
  c->snap.valid = false;
  const bf_layout& L = b->layout;
  const size_t sbytes = (size_t)b->n_runs * L.state_stride, rbytes = (size_t)b->n_runs * L.result_stride;
  if (b->flags & BF_EVAL_VALIDATE) {
    const uint8_t* st = static_cast<const uint8_t*>(b->state);
    for (uint32_t r = 0; r < b->n_runs; ++r) {
      const bf_run_header* h = reinterpret_cast<const bf_run_header*>(st + (size_t)r * L.state_stride);
      if (h->topo_slot >= c->meta.size() || !c->meta[h->topo_slot].alive)
        return fail(c, BF_ETOPO, "run " + std::to_string(r) + ": unknown topology slot");
      const TopoMeta& m = c->meta[h->topo_slot];
      if (m.S > L.steps_max) return fail(c, BF_EINVAL, "run " + std::to_string(r) + ": topology larger than layout.steps_max");
      if (L.off_child != BF_OFF_NONE && m.child_nibbles > L.child_nibbles)
        return fail(c, BF_EINVAL, "run " + std::to_string(r) + ": child area too small");
      const uint32_t* ph = reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(h) + L.off_phase);
      for (uint32_t w = 0; w < (m.S + 31) / 32; ++w)
        if (ph[w] & ph[L.words + w] & ph[2 * L.words + w] & ph[3 * L.words + w])
          return fail(c, BF_EINVAL, "run " + std::to_string(r) + ": reserved phase code 15");
    }
  }
  BF_CUDA(c, cudaSetDevice(c->device));
  if (int rc = c->d_state.ensure(c, sbytes)) return rc;
  if (int rc = c->d_result.ensure(c, rbytes)) return rc;
  const bool want_exp = (b->flags & BF_EVAL_EXPANSION) && b->expansion && b->expansion_cap;
  if (want_exp)
    if (int rc = c->d_exp.ensure(c, (size_t)b->expansion_cap)) return rc;
  // ~5.5 MB of state and results per chunk, at least two; expansion needs a batch-wide scan and stays on one stream
  uint32_t chunks = 1;
  if (int rc = bf::plan_chunks(c, want_exp ? 0 : sbytes + rbytes, 11u << 19, 2, chunks)) return rc;
  const char* shape_env = getenv("BF_E2E_SHAPE");
  const bool taper = shape_env && !strcmp(shape_env, "taper");
  uint64_t first_slice = 0;
  auto body = [&]() -> int {
    BF_CUDA(c, cudaMemsetAsync(c->d_counts, 0, sizeof(bf_counts), c->stream));
    bf_batch db = *b;
    db.flags &= ~(uint32_t)(BF_EVAL_COUNTS_SET | BF_EVAL_PIPELINED);   // bf_eval_device only: the chunks here add into one block
    if (!want_exp) db.flags &= ~BF_EVAL_EXPANSION;
    if (int rc = bf::chunked_pass(c, db, chunks, taper, c->d_state, c->d_result, static_cast<const uint8_t*>(b->state),
                                  co ? nullptr : static_cast<uint8_t*>(b->result), want_exp ? c->d_exp.p : nullptr, nullptr))
      return rc;
    return bf::pass_results(c, L, c->d_result, nullptr, b->n_runs, co, first_slice, false, false);
  };
  if (int rc = bf::pass_end(c, body(), chunks, true, co != nullptr)) return rc;
  if (want_exp) {
    const uint64_t n = std::min<uint64_t>(c->pinned->counts().expansion, b->expansion_cap);
    if (n) BF_CUDA(c, cudaMemcpy(b->expansion, c->d_exp, (size_t)n * sizeof(bf_expansion), cudaMemcpyDeviceToHost));
  }
  return bf::publish_pass(c, b->n_runs, L, c->d_state, c->d_result, b->counts, co, first_slice, c->last_events);
}

}  // namespace bf

extern "C" {

int bf_eval(bf_ctx* c, const bf_batch* b) { return bf::eval_host(c, b, nullptr); }
int bf_eval_compact(bf_ctx* c, const bf_batch* b, bf_compact_out* out) {
  if (!out) return c ? fail(c, BF_EINVAL, "null bf_compact_out") : BF_EINVAL;
  return bf::eval_host(c, b, out);
}

// ---- limiters (rows a9 / f4) ----------------------------------------------------------------------------
static int fill_sched_params(bf_ctx* c, const bf_batch* b, const bf_sched_tables* t, bf::SchedParams& P) {
  if (!b || b->struct_size != sizeof(bf_batch)) return fail(c, BF_EINVAL, "bad bf_batch.struct_size");
  if (!t || t->struct_size != sizeof(bf_sched_tables)) return fail(c, BF_EINVAL, "bad bf_sched_tables.struct_size");
  if (int rc = bf::check_layout(c, b->layout)) return rc;
  if ((t->n_stories && !t->story_limit) || (t->n_queues && (!t->queue_limit || !t->queue_aging_s)))
    return fail(c, BF_EINVAL, "null limit table");
  const bf_layout& L = b->layout;
  P.n_stories = t->n_stories; P.n_queues = t->n_queues; P.global_limit = t->global_limit; P.global_base = t->global_running_base;
  P.n_slots = (uint32_t)c->slots_host.size(); P.n_runs = b->n_runs;
  P.words = L.words; P.state_stride = L.state_stride; P.off_phase = L.off_phase; P.off_child = L.off_child;
  P.child_nibbles = L.child_nibbles;
  P.result_stride = L.result_stride; P.off_ready = L.off_ready; P.stride = BF_SCHED_STRIDE(L.words);
  P.slots = c->slots_dev;
  P.now = BF_SCHED_NONE;   // runs[r].queued_elapsed_s is the elapsed time itself
  return BF_OK;
}

int bf_schedule_device(bf_ctx* c, const bf_batch* b, const bf_sched_run* runs, const bf_sched_tables* t, bf_sched_out* out,
                       void* stream) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  bf::SchedParams P{};
  if (int rc = fill_sched_params(c, b, t, P)) return rc;
  if (!out || out->struct_size != sizeof(bf_sched_out)) return fail(c, BF_EINVAL, "bad bf_sched_out.struct_size");
  if (b->n_runs && (!b->state || !b->result || !runs || !out->records)) return fail(c, BF_EINVAL, "null state/result/runs/records");
  if (!out->story_running || !out->queue_running || !out->queue_max_priority || !out->global_running)
    return fail(c, BF_EINVAL, "device path: the totals arrays are the reduction scratch and must be given");
  BF_CUDA(c, cudaSetDevice(c->device));
  if (int rc = bf::sync_slots(c, static_cast<cudaStream_t>(stream))) return rc;
  P.slots = c->slots_dev;
  P.state = static_cast<const uint8_t*>(b->state); P.result = static_cast<const uint8_t*>(b->result);
  P.runs = runs; P.records = static_cast<uint8_t*>(out->records);
  P.story_running = out->story_running; P.queue_running = out->queue_running; P.queue_maxprio = out->queue_max_priority;
  P.global_running = out->global_running;
  P.story_limit = t->story_limit; P.queue_limit = t->queue_limit; P.queue_aging = t->queue_aging_s;
  P.story_base = t->story_running_base; P.queue_base = t->queue_running_base; P.queue_maxprio_base = t->queue_max_priority_base;
  BF_CUDA(c, bf::launch_schedule(P, (uint32_t)c->sm_count, static_cast<cudaStream_t>(stream)));
  c->stats.kernel_launches += 3;
  return BF_OK;
}

}  // extern "C"

namespace bf {

int schedule_host(bf_ctx* c, const bf_batch* b, const bf_sched_run* runs, const bf_sched_tables* t, bf_sched_out* out,
                  sched_between_fn between, void* user, bool with_bases) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  bf::SchedParams P{};
  if (int rc = fill_sched_params(c, b, t, P)) return rc;
  if (!out || out->struct_size != sizeof(bf_sched_out)) return fail(c, BF_EINVAL, "bad bf_sched_out.struct_size");
  if (b->n_runs && (!runs || !out->records)) return fail(c, BF_EINVAL, "null runs/records");
  if (!c->snap.matches(b->n_runs, b->layout))
    return fail(c, BF_EINVAL, "bf_schedule must follow bf_eval / bf_resident_eval of the same batch (n_runs and layout) on this ctx");
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  // topology puts and drops since the pass: the reduction reads the slot table as it is now (a dropped slot counts nothing; a
  // stale device table could point at moved arena records, or hold fewer slots than n_slots)
  if (int rc = bf::sync_slots(c, s)) return rc;
  P.slots = c->slots_dev;
  // one device allocation: runs | records | story_running | queue_running | queue_maxprio | global | limits | bases
  const size_t n = b->n_runs, ns = t->n_stories, nq = t->n_queues;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off = round_up_sz(off + bytes, 16); return o; };
  const size_t o_runs = take(n * sizeof(bf_sched_run)), o_rec = take(n * (size_t)P.stride), o_sr = take(ns * 4), o_qr = take(nq * 4),
               o_mp = take(nq * 4), o_gl = take(4), o_sl = take(ns * 4), o_ql = take(nq * 4), o_qa = take(nq * 4), o_sb = take(ns * 4),
               o_qb = take(nq * 4), o_pb = take(nq * 4);
  if (int rc = c->d_sched.ensure(c, off ? off : 16)) return rc;
  uint8_t* d = c->d_sched;
  auto up = [&](size_t o, const void* src, size_t bytes) -> cudaError_t {
    return (src && bytes) ? cudaMemcpyAsync(d + o, src, bytes, cudaMemcpyHostToDevice, s) : cudaSuccess;
  };
  BF_CUDA(c, up(o_runs, runs, n * sizeof(bf_sched_run)));
  BF_CUDA(c, up(o_sl, t->story_limit, ns * 4));
  BF_CUDA(c, up(o_ql, t->queue_limit, nq * 4));
  BF_CUDA(c, up(o_qa, t->queue_aging_s, nq * 4));
  if (with_bases) {   // a sharded schedule adds the running bases on one shard only (the totals are summed across shards)
    BF_CUDA(c, up(o_sb, t->story_running_base, ns * 4));
    BF_CUDA(c, up(o_qb, t->queue_running_base, nq * 4));
  }
  BF_CUDA(c, up(o_pb, t->queue_max_priority_base, nq * 4));
  P.state = c->snap.state; P.result = c->snap.result;
  P.runs = reinterpret_cast<const bf_sched_run*>(d + o_runs); P.records = d + o_rec;
  P.story_running = reinterpret_cast<uint32_t*>(d + o_sr); P.queue_running = reinterpret_cast<uint32_t*>(d + o_qr);
  P.queue_maxprio = reinterpret_cast<int32_t*>(d + o_mp); P.global_running = reinterpret_cast<uint32_t*>(d + o_gl);
  P.story_limit = reinterpret_cast<const int32_t*>(d + o_sl); P.queue_limit = reinterpret_cast<const int32_t*>(d + o_ql);
  P.queue_aging = reinterpret_cast<const int32_t*>(d + o_qa);
  P.story_base = (with_bases && t->story_running_base) ? reinterpret_cast<const uint32_t*>(d + o_sb) : nullptr;
  P.queue_base = (with_bases && t->queue_running_base) ? reinterpret_cast<const uint32_t*>(d + o_qb) : nullptr;
  P.queue_maxprio_base = t->queue_max_priority_base ? reinterpret_cast<const int32_t*>(d + o_pb) : nullptr;
  if (!with_bases) P.global_base = 0;
  cudaError_t e = bf::launch_schedule(P, (uint32_t)c->sm_count, s, bf::kSchedTotals);
  if (e == cudaSuccess && between) {
    const SchedTotals tot{P.story_running, P.queue_running, P.queue_maxprio, P.global_running, (uint32_t)ns, (uint32_t)nq};
    if (int rc = between(user, tot, s)) { cudaStreamSynchronize(s); return rc; }
  }
  if (e == cudaSuccess) e = bf::launch_schedule(P, (uint32_t)c->sm_count, s, bf::kSchedApply);
  c->stats.kernel_launches += 3;
  auto down = [&](void* dst, size_t o, size_t bytes) -> cudaError_t {
    return (dst && bytes) ? cudaMemcpyAsync(dst, d + o, bytes, cudaMemcpyDeviceToHost, s) : cudaSuccess;
  };
  if (e == cudaSuccess) e = down(out->records, o_rec, n * (size_t)P.stride);
  if (e == cudaSuccess) e = down(out->story_running, o_sr, ns * 4);
  if (e == cudaSuccess) e = down(out->queue_running, o_qr, nq * 4);
  if (e == cudaSuccess) e = down(out->queue_max_priority, o_mp, nq * 4);
  if (e == cudaSuccess) e = down(out->global_running, o_gl, 4);
  const cudaError_t es = cudaStreamSynchronize(s);  // never return with copies into the caller's buffers in flight
  if (e != cudaSuccess) return cuda_fail(c, e, "bf_schedule");
  if (es != cudaSuccess) return cuda_fail(c, es, "cudaStreamSynchronize");
  return BF_OK;
}

}  // namespace bf

extern "C" {

int bf_schedule(bf_ctx* c, const bf_batch* b, const bf_sched_run* runs, const bf_sched_tables* t, bf_sched_out* out) {
  return bf::schedule_host(c, b, runs, t, out, nullptr, nullptr, true);
}

int bf_alloc_pinned(bf_ctx* c, size_t bytes, void** out) {
  if (!c || !out) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaError_t e = cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault);
  if (e != cudaSuccess) return fail(c, BF_ENOMEM, std::string("cudaHostAlloc: ") + cudaGetErrorString(e));
  return BF_OK;
}

int bf_free_pinned(bf_ctx* c, void* p) {
  if (!c) return BF_EINVAL;
  if (!p) return BF_OK;
  std::lock_guard<std::mutex> g(c->mu);
  BF_CUDA(c, cudaFreeHost(p));
  return BF_OK;
}

int bf_get_stats(const bf_ctx* c, bf_stats* out) {
  if (!c || !out) return BF_EINVAL;
  *out = c->stats;
  out->arena_used_bytes = c->arena_used;
  out->arena_compactions = (uint32_t)c->arena_compactions;
  out->arena_cap_bytes = c->arena.cap;
  out->n_topologies = c->n_alive;
  out->sm_count = (uint32_t)c->sm_count;
  return BF_OK;
}

}  // extern "C"
