// abi.cu — the C ABI of include/bobrafrontier.h: context, topology arena, batch evaluation.
//
// Host side of the boundary.  Packs Story topologies into the device record format
// (device_record.h), validates what validateRuntimeDependencyGraph validates
// (internal/controller/runs/dag.go:3076-3146), plans shared memory for the frontier
// kernel and drives H2D -> kernels -> D2H for the host-buffer entry point.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <new>
#include <thread>

#include "ctx.h"

using bf::cuda_fail; using bf::fail; using bf::round_up; using bf::round_up_sz;

namespace {

// ---- record building -----------------------------------------------------------------------
// BF_TOPO_FORMAT=csr keeps every topology in CSR form, =ell16 keeps the fixed-width rows at u16 entries (A/B timing and
// the parity tests of those paths); read per upload.  0 = default (best format), 1 = CSR only, 2 = no byte entries
static int forced_format() {
  const char* e = getenv("BF_TOPO_FORMAT");
  if (e && !strcmp(e, "csr")) return 1;
  if (e && !strcmp(e, "ell16")) return 2;
  return 0;
}

struct RecPlan {
  uint32_t off_col, off_planes, off_par, off_allow, rec_bytes, W, child_nibbles, ell, max_deg;
  uint32_t ff[bf::FF_STRIDE];   // the topology's row of the fail-fast mask table
  std::vector<uint32_t> child_first, allow_off;
};

int plan_record(const bf_topology& t, RecPlan& p, std::string& why, bool host_kahn = true, int forced = 0) {
  if (t.n_steps == 0 || t.n_steps > BF_MAX_STEPS) { why = "n_steps out of range (1..1024)"; return BF_ETOPO; }
  if (t.n_edges > BF_MAX_EDGES) { why = "n_edges exceeds 65535"; return BF_ETOPO; }
  if (!t.row_ptr || !t.step_flags || (t.n_edges && !t.col_idx)) { why = "null topology array"; return BF_EINVAL; }
  if (t.n_parallel > BF_MAX_PARALLEL) { why = "more than 64 parallel steps"; return BF_ETOPO; }
  if (t.n_parallel && !t.parallel) { why = "null parallel descs"; return BF_EINVAL; }
  const uint32_t S = t.n_steps, E = t.n_edges;
  if (t.row_ptr[0] != 0 || t.row_ptr[S] != E) { why = "row_ptr[0] != 0 or row_ptr[S] != E"; return BF_ETOPO; }
  for (uint32_t i = 0; i < S; ++i)
    if (t.row_ptr[i + 1] < t.row_ptr[i]) { why = "row_ptr not monotone"; return BF_ETOPO; }
  for (uint32_t e = 0; e < E; ++e)
    if (t.col_idx[e] >= S) { why = "unknown step dependency (col_idx >= S)"; return BF_ETOPO; }  // dag.go:3087-3098
  // acyclicity (Kahn), dag.go:3100-3145.  indegree[i] = number of deps of i.
  if (host_kahn) {
    std::vector<uint32_t> indeg(S), head(S + 1, 0), out(E), stack;
    for (uint32_t i = 0; i < S; ++i) indeg[i] = t.row_ptr[i + 1] - t.row_ptr[i];
    for (uint32_t e = 0; e < E; ++e) head[t.col_idx[e] + 1]++;
    for (uint32_t i = 0; i < S; ++i) head[i + 1] += head[i];
    std::vector<uint32_t> fill(head.begin(), head.end() - 1);
    for (uint32_t i = 0; i < S; ++i)
      for (uint32_t e = t.row_ptr[i]; e < t.row_ptr[i + 1]; ++e) out[fill[t.col_idx[e]]++] = i;
    for (uint32_t i = 0; i < S; ++i)
      if (indeg[i] == 0) stack.push_back(i);
    uint32_t visited = 0;
    while (!stack.empty()) {
      const uint32_t u = stack.back();
      stack.pop_back();
      ++visited;
      for (uint32_t x = head[u]; x < head[u + 1]; ++x)
        if (--indeg[out[x]] == 0) stack.push_back(out[x]);
    }
    if (visited != S) { why = "dependency cycle detected"; return BF_ETOPO; }
  }
  uint32_t prev_step = 0;
  p.child_first.assign(t.n_parallel, 0);
  p.allow_off.assign(t.n_parallel, 0);
  uint32_t nib = 0, allow_words = 0;
  for (uint32_t q = 0; q < t.n_parallel; ++q) {
    const bf_parallel_desc& d = t.parallel[q];
    if (d.step >= S) { why = "parallel desc step out of range"; return BF_ETOPO; }
    if ((t.step_flags[d.step] & BF_SF_TYPE_MASK) != BF_STEP_PARALLEL) { why = "parallel desc on a non-parallel step"; return BF_ETOPO; }
    if (q && d.step <= prev_step) { why = "parallel descs must ascend by step"; return BF_ETOPO; }
    if (t.branch_allow_bits && (uint64_t)d.allow_first + d.branches > t.n_branch_allow_bits) { why = "branch_allow_bits too short"; return BF_EINVAL; }
    prev_step = d.step;
    nib = round_up(nib, 8);
    p.child_first[q] = nib;
    nib += d.branches;
    allow_words += (d.branches + 31) / 32 + (d.branches == 0 ? 1 : 0);
  }
  if (nib > 0xFFFF) { why = "too many parallel branches"; return BF_ETOPO; }
  p.child_nibbles = round_up(nib, 8);
  p.W = (S + 31) / 32;
  memset(p.ff, 0, sizeof p.ff);
  if (p.W <= bf::FF_STRIDE) {
    bool main_only = true;
    for (uint32_t i = 0; i < S && main_only; ++i) {
      main_only = ((t.step_flags[i] & BF_SF_GROUP_MASK) >> BF_SF_GROUP_SHIFT) == BF_GROUP_MAIN;
      if (!(t.step_flags[i] & BF_SF_ALLOW_FAILURE)) p.ff[i >> 5] |= 1u << (i & 31u);
    }
    if (!main_only) memset(p.ff, 0, sizeof p.ff);
  }
  uint32_t off = sizeof(bf::TopoHeader);
  // Row format (device_record.h): fixed-width rows of K = 2 / 4 entries (no row_ptr; unused entries = PAD) when no step
  // has more than K needs and the block is not larger than the CSR block it replaces, else CSR.
  uint32_t md = 0;
  for (uint32_t i = 0; i < S; ++i) { const uint32_t d = t.row_ptr[i + 1] - t.row_ptr[i]; if (d > md) md = d; }
  p.max_deg = md;
  // + 4 zero entries: the branch-free walk fetches col[e0..e0+3] whatever the row length (e0 = E for trailing
  // rows without deps), so the last rows read past E; zero padding keeps every fetched index a valid step index
  // and the walk needs no clamp
  const uint32_t csr_bytes = round_up(2 * (S + 1), 16) + round_up(2 * E + 8, 16);
  const uint32_t K = md <= 2 ? 2u : (md <= 4 ? 4u : 0u);
  p.ell = 0;
  p.W = (S + 31) / 32;
  const uint32_t ell_rows = 32 * p.W;   // a row for every step of every word, so the walk fetches without a bounds test
  if (K && forced != 1) {
    // byte entries (device_record.h): every step index of a topology of at most 256 steps fits a byte
    if (ell_rows <= 256 && forced != 2 && K * ell_rows + 4 * p.W <= csr_bytes) p.ell = K | bf::ELL_BYTE;
    // 10-bit entries: topologies of more than 512 steps (never staged by the packed-lanes kernel) with rows of up to 4 needs
    else if (K == 4 && p.W > 16 && forced != 2 && 5 * ell_rows + 4 * p.W <= csr_bytes) p.ell = 4 | bf::ELL_PACK10;
    // (no u16 rows at 8 words: their PAD index 256 has no status byte — the packed kernel keeps a run's status bytes on a
    //  256-byte stride there; such a topology has byte entries unless BF_TOPO_FORMAT forbids them, then CSR)
    else if (2 * K * ell_rows <= csr_bytes && ell_rows != 256) p.ell = K;
  }
  if (p.ell) {
    p.off_col = off;
    off += bf::ell_row_bytes(p.ell) * ell_rows;
  } else {
    off += round_up(2 * (S + 1), 16);
    p.off_col = off;
    off += round_up(2 * E + 8, 16);
  }
  p.off_planes = off;
  off += round_up(bf::plane_count(p.ell) * p.W * 4, 16);
  p.off_par = off;
  off += t.n_parallel * (uint32_t)sizeof(bf::ParDesc);
  p.off_allow = off;
  uint32_t aw = 0;
  for (uint32_t q = 0; q < t.n_parallel; ++q) {
    p.allow_off[q] = p.off_allow + aw * 4;
    aw += (t.parallel[q].branches + 31) / 32 + (t.parallel[q].branches == 0 ? 1 : 0);
  }
  off += allow_words * 4;
  p.rec_bytes = round_up(off, 16);
  return BF_OK;
}

void build_record(const bf_topology& t, const RecPlan& p, uint8_t* rec) {
  memset(rec, 0, p.rec_bytes);
  const uint32_t S = t.n_steps, E = t.n_edges, W = p.W;
  bf::TopoHeader h{};
  h.S = (uint16_t)S; h.W = (uint16_t)W; h.P = (uint16_t)t.n_parallel;
  h.max_deg = (uint16_t)(p.max_deg > 0xFFFF ? 0xFFFF : p.max_deg);
  h.child_nibbles = (uint16_t)p.child_nibbles;
  h.off_col = (uint16_t)p.off_col; h.ell = (uint16_t)p.ell; h.off_planes = p.off_planes; h.off_par = p.off_par; h.rec_bytes = p.rec_bytes;
  if (bf::ell_has_nodep(p.ell)) {
    // byte / 10-bit entries: a short row repeats its first entry, a row without needs holds its own index and is flagged
    // NODEP (as are the rows past S); the planes are zeroed above and filled below
    uint8_t* col = rec + p.off_col;
    uint32_t* lo = reinterpret_cast<uint32_t*>(col);
    uint32_t* nodep = reinterpret_cast<uint32_t*>(rec + p.off_planes) + bf::PL_NODEP * W;
    const uint32_t K = bf::ell_k(p.ell);
    for (uint32_t i = 0; i < 32 * W; ++i) {
      const uint32_t e0 = i < S ? t.row_ptr[i] : 0, n = i < S ? t.row_ptr[i + 1] - e0 : 0;
      if (n == 0) nodep[i >> 5] |= 1u << (i & 31u);
      uint32_t x[4] = {0, 0, 0, 0};
      for (uint32_t k = 0; k < K; ++k) x[k] = n == 0 ? i : t.col_idx[e0 + (k < n ? k : 0)];
      if (p.ell & bf::ELL_PACK10) {
        lo[i] = x[0] | (x[1] << 10) | (x[2] << 20) | (x[3] << 30);
        col[128 * W + i] = (uint8_t)(x[3] >> 2);
      } else {
        for (uint32_t k = 0; k < K; ++k) col[i * K + k] = (uint8_t)x[k];
      }
    }
  } else if (p.ell) {
    uint16_t* col = reinterpret_cast<uint16_t*>(rec + p.off_col);
    const uint16_t pad = (uint16_t)(32 * W);  // the status byte just past the last step word: always "satisfied"
    for (uint32_t i = 0; i < S; ++i) {
      const uint32_t e0 = t.row_ptr[i], n = t.row_ptr[i + 1] - e0;
      for (uint32_t k = 0; k < p.ell; ++k) col[i * p.ell + k] = k < n ? t.col_idx[e0 + k] : pad;
    }
    for (uint32_t x = S * p.ell; x < 32 * W * p.ell; ++x) col[x] = pad;
  } else {
    uint16_t* rp = reinterpret_cast<uint16_t*>(rec + sizeof(bf::TopoHeader));
    for (uint32_t i = 0; i <= S; ++i) rp[i] = (uint16_t)t.row_ptr[i];
    if (E) memcpy(rec + p.off_col, t.col_idx, 2 * (size_t)E);
  }
  uint32_t* planes = reinterpret_cast<uint32_t*>(rec + p.off_planes);
  uint32_t nm = 0, nc = 0, nf = 0;
  for (uint32_t i = 0; i < S; ++i) {
    const uint8_t f = t.step_flags[i];
    const uint32_t w = i >> 5, b = 1u << (i & 31u);
    if (f & 1u) planes[bf::PL_T0 * W + w] |= b;
    if (f & 2u) planes[bf::PL_T1 * W + w] |= b;
    if (f & 4u) planes[bf::PL_T2 * W + w] |= b;
    if (f & BF_SF_ALLOW_FAILURE) planes[bf::PL_AF * W + w] |= b;
    if (f & BF_SF_ON_TIMEOUT_SKIP) planes[bf::PL_TS * W + w] |= b;
    if (f & BF_SF_HAS_IF) planes[bf::PL_HASIF * W + w] |= b;
    const uint32_t g = (f & BF_SF_GROUP_MASK) >> BF_SF_GROUP_SHIFT;
    if (g == BF_GROUP_COMPENSATION) { planes[bf::PL_G1 * W + w] |= b; nc++; }
    else if (g == BF_GROUP_MAIN) nm++;
    else { planes[bf::PL_G2 * W + w] |= b; nf++; }  // 2 (and the unused code 3) count as finally
  }
  h.n_main = (uint16_t)nm; h.n_comp = (uint16_t)nc; h.n_final = (uint16_t)nf;
  bf::ParDesc* pd = reinterpret_cast<bf::ParDesc*>(rec + p.off_par);
  for (uint32_t q = 0; q < t.n_parallel; ++q) {
    pd[q].step = t.parallel[q].step;
    pd[q].branches = t.parallel[q].branches;
    pd[q].child_first = p.child_first[q];
    pd[q].allow_off = p.allow_off[q];
    pd[q].reserved = 0;
    uint32_t* aw = reinterpret_cast<uint32_t*>(rec + p.allow_off[q]);
    if (t.branch_allow_bits)
      for (uint32_t b = 0; b < t.parallel[q].branches; ++b) {
        const uint32_t src = t.parallel[q].allow_first + b;
        if ((t.branch_allow_bits[src >> 3] >> (src & 7u)) & 1u) aw[b >> 5] |= 1u << (b & 31u);
      }
  }
  memcpy(rec, &h, sizeof h);
}

int grow_arena(bf_ctx* c, size_t need_total) {
  if (need_total <= c->arena.cap) return BF_OK;
  size_t ncap = c->arena.cap ? c->arena.cap : (size_t)64 << 20;
  while (ncap < need_total) ncap *= 2;
  DevBuf<uint8_t> na;
  cudaError_t e = na.alloc(ncap);
  if (e != cudaSuccess) {  // retry exact
    e = na.alloc(round_up_sz(need_total, (size_t)1 << 20));
    if (e != cudaSuccess) return fail(c, BF_ENOMEM, std::string("arena cudaMalloc: ") + cudaGetErrorString(e));
  }
  if (c->arena && c->arena_used) {
    e = cudaMemcpy(na, c->arena, c->arena_used, cudaMemcpyDeviceToDevice);
    if (e != cudaSuccess) return cuda_fail(c, e, "arena copy");
  }
  c->arena = std::move(na);
  for (size_t s = 0; s < c->meta.size(); ++s)
    if (c->meta[s].alive) c->slots_host[s].addr = (uint64_t)(uintptr_t)(c->arena + c->meta[s].offset);
  c->slots_dirty = true;
  return BF_OK;
}

// The arena is a bump allocator; a long-lived operator puts one topology per Story generation and drops the old one, so
// dead records pile up below arena_used.  When they outweigh the live ones the live records are re-packed into a fresh
// arena (one warp per record on the device), the slot table follows, and the freed space is reusable again.
int compact_arena(bf_ctx* c, size_t incoming) {
  std::vector<uint32_t> live;
  size_t live_bytes = 0;
  for (uint32_t s = 0; s < c->meta.size(); ++s)
    if (c->meta[s].alive) { live.push_back(s); live_bytes += round_up_sz(c->meta[s].bytes, 16); }
  size_t ncap = (size_t)64 << 20;
  while (ncap < live_bytes + incoming) ncap *= 2;
  DevBuf<uint8_t> na;
  cudaError_t e = na.alloc(ncap);
  if (e != cudaSuccess) return BF_OK;   // no room for a second arena right now: keep appending
  std::vector<unsigned long long> moves(4 * live.size());
  size_t off = 0;
  for (size_t i = 0; i < live.size(); ++i) {
    const TopoMeta& m = c->meta[live[i]];
    moves[4 * i] = m.offset; moves[4 * i + 1] = off; moves[4 * i + 2] = m.bytes; moves[4 * i + 3] = 0;
    off += round_up_sz(m.bytes, 16);
  }
  void* d_moves = nullptr;
  if (!live.empty()) {
    e = cudaMalloc(&d_moves, moves.size() * sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_moves, moves.data(), moves.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = bf::launch_move_records(c->arena, na, d_moves, (uint32_t)live.size(), c->stream);
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();   // nothing may still read the old arena when it is freed
  cudaFree(d_moves);
  if (e != cudaSuccess) return cuda_fail(c, e, "arena compaction");
  c->arena = std::move(na); c->arena_used = off; c->arena_dead = 0;
  for (size_t i = 0; i < live.size(); ++i) {
    TopoMeta& m = c->meta[live[i]];
    m.offset = (size_t)moves[4 * i + 1];
    c->slots_host[live[i]].addr = (uint64_t)(uintptr_t)(c->arena + m.offset);
  }
  c->slots_dirty = true;
  c->rec_max_dirty = true;
  c->arena_compactions++;
  c->stats.kernel_launches += live.empty() ? 0 : 1;
  return BF_OK;
}

int put_many_locked(bf_ctx* c, const bf_topology* topos, uint32_t count, uint32_t* slots_out, bool host_kahn = true) {
  std::vector<RecPlan> plans(count);
  size_t total = 0;
  std::string why;
  const int forced = forced_format();
  // validation (Kahn) and record building are per topology: spread a bulk upload over the host cores
  const uint32_t n_thr = count >= 512 ? std::min<uint32_t>(16, std::max(1u, std::thread::hardware_concurrency())) : 1;
  auto parallel_for = [&](auto&& fn) {
    if (n_thr == 1) { fn(0u, count); return; }
    std::vector<std::thread> th;
    for (uint32_t t = 0; t < n_thr; ++t)
      th.emplace_back([&, t] { fn((uint32_t)((uint64_t)count * t / n_thr), (uint32_t)((uint64_t)count * (t + 1) / n_thr)); });
    for (auto& x : th) x.join();
  };
  std::vector<int> rcs(count, BF_OK);
  std::mutex why_mu;
  uint32_t first_bad = count;
  parallel_for([&](uint32_t lo, uint32_t hi) {
    std::string w;
    for (uint32_t i = lo; i < hi; ++i) {
      rcs[i] = plan_record(topos[i], plans[i], w, host_kahn, forced);
      if (rcs[i] != BF_OK) {
        std::lock_guard<std::mutex> g(why_mu);
        if (i < first_bad) { first_bad = i; why = w; }
        return;
      }
    }
  });
  if (first_bad < count) return fail(c, rcs[first_bad], "topology " + std::to_string(first_bad) + ": " + why);
  for (uint32_t i = 0; i < count; ++i) total += plans[i].rec_bytes;
  if (c->arena_dead > ((size_t)1 << 20) && c->arena_dead * 2 > c->arena_used)
    if (int rc = compact_arena(c, total)) return rc;
  const size_t base = round_up_sz(c->arena_used, 16);
  if (int rc = grow_arena(c, base + total)) return rc;
  std::vector<uint8_t> staging;
  try { staging.resize(total); } catch (const std::bad_alloc&) { return fail(c, BF_ENOMEM, "host staging allocation failed"); }
  std::vector<size_t> rec_off(count);
  size_t off = 0;
  for (uint32_t i = 0; i < count; ++i) { rec_off[i] = off; off += plans[i].rec_bytes; }
  parallel_for([&](uint32_t lo, uint32_t hi) {
    for (uint32_t i = lo; i < hi; ++i) build_record(topos[i], plans[i], staging.data() + rec_off[i]);
  });
  if (total) BF_CUDA(c, cudaMemcpy(c->arena + base, staging.data(), total, cudaMemcpyHostToDevice));
  off = 0;
  for (uint32_t i = 0; i < count; ++i) {
    uint32_t slot;
    if (!c->free_slots.empty()) { slot = c->free_slots.back(); c->free_slots.pop_back(); c->slot_changes++; }
    else {
      slot = (uint32_t)c->meta.size();
      c->meta.emplace_back();
      c->slots_host.push_back(bf::Slot{0, 0, 0});
      c->ff_host.resize(c->ff_host.size() + bf::FF_STRIDE, 0u);
    }
    TopoMeta& m = c->meta[slot];
    m.alive = true; m.S = topos[i].n_steps; m.E = topos[i].n_edges; m.P = topos[i].n_parallel;
    m.bytes = plans[i].rec_bytes; m.offset = base + off; m.child_first = plans[i].child_first;
    m.child_nibbles = plans[i].child_nibbles;
    m.par_step.resize(m.P); m.par_branches.resize(m.P);
    for (uint32_t q = 0; q < m.P; ++q) { m.par_step[q] = topos[i].parallel[q].step; m.par_branches[q] = topos[i].parallel[q].branches; }
    c->slots_host[slot] = bf::Slot{(uint64_t)(uintptr_t)(c->arena + m.offset), m.bytes,
                                   m.S | (m.P << 16) | (bf::slot_row_bytes(plans[i].ell) << 24)};
    memcpy(&c->ff_host[(size_t)slot * bf::FF_STRIDE], plans[i].ff, sizeof plans[i].ff);
    if (m.bytes > c->max_rec_bytes) c->max_rec_bytes = m.bytes;
    if (m.bytes > c->max_rec_by_w[plans[i].W]) c->max_rec_by_w[plans[i].W] = m.bytes;
    off += plans[i].rec_bytes;
    slots_out[i] = slot;
    c->n_alive++;
    if (m.P) c->n_with_parallel++;
  }
  c->arena_used = base + total;
  c->slots_dirty = true;
  return BF_OK;
}

}  // namespace

// ---- host helpers of a pass, shared with resident_abi.cu (ctx.h) ----------------------------
namespace bf {

// copy / compute streams and events of the chunked pipelines (bf_eval, bf_resident_tick); created on first use
int ensure_pipe(bf_ctx* c) {
  if (c->pipe_ready) return BF_OK;
  if (!c->s_in) BF_CUDA(c, cudaStreamCreateWithFlags(&c->s_in, cudaStreamNonBlocking));
  if (!c->s_out) BF_CUDA(c, cudaStreamCreateWithFlags(&c->s_out, cudaStreamNonBlocking));
  for (uint32_t k = 0; k < bf_ctx::kMaxChunks; ++k) {
    if (!c->ev_in[k]) BF_CUDA(c, cudaEventCreateWithFlags(&c->ev_in[k], cudaEventDisableTiming));
    if (!c->ev_k[k]) BF_CUDA(c, cudaEventCreateWithFlags(&c->ev_k[k], cudaEventDisableTiming));
  }
  c->pipe_ready = true;
  return BF_OK;
}

int sync_slots(bf_ctx* c, cudaStream_t stream) {
  if (!c->slots_dirty) return BF_OK;
  const size_t n = c->slots_host.size();
  if (n > c->slots_dev.cap) {
    size_t ncap = c->slots_dev.cap ? c->slots_dev.cap : 1024;
    while (ncap < n) ncap *= 2;
    DevBuf<bf::Slot> np;
    DevBuf<uint32_t> nf;
    if (cudaError_t e = np.alloc(ncap)) return cuda_fail(c, e, "cudaMalloc slot table");
    if (cudaError_t e = nf.alloc(ncap * bf::FF_STRIDE)) return cuda_fail(c, e, "cudaMalloc fail-fast masks");
    c->slots_dev = std::move(np);
    c->ff_dev = std::move(nf);
  }
  if (n) BF_CUDA(c, cudaMemcpyAsync(c->slots_dev, c->slots_host.data(), n * sizeof(bf::Slot), cudaMemcpyHostToDevice, stream));
  if (n) BF_CUDA(c, cudaMemcpyAsync(c->ff_dev, c->ff_host.data(), n * bf::FF_STRIDE * sizeof(uint32_t), cudaMemcpyHostToDevice, stream));
  BF_CUDA(c, cudaStreamSynchronize(stream));
  c->slots_dirty = false;
  return BF_OK;
}

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

// shared-memory plan + launch of one pass on device buffers
// run_list (touched ticks): the pass takes the runs run_list[0 .. *run_list_count) (b.n_runs bounds the count) and writes
// each run's record at its own index
int run_pass(bf_ctx* c, const bf_batch& b, const uint8_t* d_state, uint8_t* d_result, bf_expansion* d_exp,
             unsigned long long* d_counts, cudaStream_t stream, const uint32_t* run_list, const uint32_t* run_list_count) {
  const bf_layout& L = b.layout;
  if (int rc = sync_slots(c, stream)) return rc;
  if (c->rec_max_dirty) {  // drops since the last plan: the largest live record per word count
    c->max_rec_bytes = 0;
    memset(c->max_rec_by_w, 0, sizeof c->max_rec_by_w);
    for (const TopoMeta& m : c->meta)
      if (m.alive) {
        const uint32_t w = (m.S + 31) / 32;
        if (m.bytes > c->max_rec_bytes) c->max_rec_bytes = m.bytes;
        if (m.bytes > c->max_rec_by_w[w]) c->max_rec_by_w[w] = m.bytes;
      }
    c->rec_max_dirty = false;
  }
  if (c->max_rec_bytes == 0) return fail(c, BF_ETOPO, "no topology has been uploaded");
  // the largest record a run of this batch can stage: topologies wider than the layout are rejected by the kernels
  uint32_t batch_rec_bytes = 0;
  for (uint32_t w = 1; w <= L.words && w <= 32; ++w)
    if (c->max_rec_by_w[w] > batch_rec_bytes) batch_rec_bytes = c->max_rec_by_w[w];
  if (batch_rec_bytes == 0) batch_rec_bytes = 64;   // no topology fits the layout: every run will be marked dead

  bf::KParams P{};
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

  P.run_blocked = 0;
  if (const char* e = getenv("BF_ASSIGN")) P.run_blocked = !strcmp(e, "blocked");
  const bool want_exp = (b.flags & BF_EVAL_EXPANSION) && d_exp != nullptr;
  if (want_exp) {
    if (int rc = c->d_exp_counts.ensure(c, b.n_runs)) return rc;
    if (int rc = c->d_offsets.ensure(c, b.n_runs)) return rc;
    if (int rc = c->d_block_sums.ensure(c, (size_t)(b.n_runs + 1023) / 1024 + 1)) return rc;
    P.exp_counts = c->d_exp_counts;
  }

  // ---- kernel choice ----
  // Packed lanes (frontier_pack.cu, a group of R = 32 / Wq runs per warp trip) for single-pass batches whose records
  // leave room for at least kMinGroups slot groups per SM; the one-run-per-warp kernel (frontier_kernel.cu) for the
  // device fixpoint, for S > 512 and when every live topology has `parallel` steps.  Mixed batches: the packed kernel
  // defers the runs whose topology has parallel steps to a device list that the general kernel then takes (second
  // launch; exits at once when the list is empty).  BF_KERNEL=general forces the general kernel (A/B timing).
  const uint32_t budget = 227u * 1024u;
  // experiment knob (tools/build_variant.sh with -DPACK_MIN_BLOCKS=k -DPACK_MAX_WARPS=24/k): k packed-lanes CTAs per SM, each
  // with 1/k of the shared memory
  uint32_t pack_ctas_per_sm = 1;
  if (const char* e = getenv("BF_PACK_CTAS")) { const uint32_t v = (uint32_t)atoi(e); if (v >= 1 && v <= 4) pack_ctas_per_sm = v; }
  const uint32_t work_general = round_up(4 * L.words, 16) + 32 * L.words + 16;  // fix-up mask words + status bytes + PAD guard
  P.topo_buf_bytes = round_up(batch_rec_bytes, 16);
  P.stage_bytes = L.state_stride + P.topo_buf_bytes;
  bool pack = !(b.flags & BF_EVAL_FIXPOINT) && L.words <= 16 && c->n_with_parallel != c->n_alive;
  if (const char* env_k = getenv("BF_KERNEL")) pack = pack && strcmp(env_k, "general") != 0;
  uint32_t wq = 1, lg = 0;
  while (wq < L.words) { wq <<= 1; lg++; }
  if (const char* e = getenv("BF_WQ")) {   // experiment knob: fewer runs per group (lanes per run rounded up further)
    const uint32_t v = (uint32_t)atoi(e);
    while (wq < v && wq < 32) { wq <<= 1; lg++; }
  }
  const uint32_t R = 32u / wq;
  constexpr uint32_t kMinGroups = 8;
  uint32_t nw = bf::frontier_pack_max_warps(), ng = 0, pack_smem = 0;
  if (pack) {
    if (const char* e = getenv("BF_WARPS")) nw = (uint32_t)atoi(e);
    if (nw < 1) nw = 1;
    if (nw > bf::frontier_pack_max_warps()) nw = bf::frontier_pack_max_warps();
    const uint32_t group_bytes = R * P.stage_bytes;
    // per-warp scratch (frontier_pack.cu): status bytes R x st_stride | fix-up words | walk table R x 16, in units of 256 bytes
    const uint32_t st_stride = wq == 8 ? 256u : 32u * wq + 16u;
    const uint32_t work = round_up(R * st_stride + 128u + 16u * R, 256);
    auto groups_for = [&](uint32_t warps) -> uint32_t {   // slot groups that fit beside `warps` scratch areas
      const uint32_t fixed = 128u + 768u + 256u + warps * work;   // 768: mbarriers + armed words of up to 64 groups; 256: scratch alignment
      const uint32_t cta_budget = budget / pack_ctas_per_sm - (pack_ctas_per_sm > 1 ? 1024u : 0u);   // (the per-CTA reservation of the driver)
      const uint32_t n = fixed < cta_budget ? (cta_budget - fixed) / group_bytes : 0;
      return n > 64 ? 64 : n;
    };
    while (nw > 1 && groups_for(nw) < nw) --nw;               // never more warps than slot groups
    ng = groups_for(nw);
    if (ng > 32u * nw) ng = 32u * nw;   // never more slot groups than threads: thread i sets up slot group i (frontier_pack.cu)
    if (const char* e = getenv("BF_GROUPS")) { const uint32_t v = (uint32_t)atoi(e); if (v >= nw && v <= ng) ng = v; }
    if (ng < kMinGroups || ng < nw) pack = false;   // records too large for a useful ring: one run per warp instead
    else {
      // a small batch gives a CTA only a few groups: no more warps and slot groups than it will use, so that the CTAs of
      // consecutive (pipelined) passes fit an SM side by side instead of waiting for each other's shared memory
      const uint32_t n_groups = (b.n_runs + R - 1) / R;
      const uint32_t slots_sm = (uint32_t)c->sm_count * pack_ctas_per_sm;
      const uint32_t ctas = slots_sm < n_groups ? slots_sm : (n_groups ? n_groups : 1);
      const uint32_t t_max = n_groups ? (n_groups + ctas - 1) / ctas : 1;
      if (nw > t_max) nw = t_max;
      if (ng > t_max) ng = t_max;
      pack_smem = 128u + round_up(ng * 12u, 128) + ng * group_bytes + 256u + nw * work;
    }
    P.work_bytes = work;
  }
  const bool two_tier = pack && c->n_with_parallel != 0;

  // ---- shared-memory plan of the general kernel (also the second tier of a mixed batch) ----
  uint32_t g_st = 0, g_wpb = 0, g_occ2 = 0;
  int g_per_sm = 1;
  if (!pack || two_tier) {
    bf::KParams PG = P;
    PG.work_bytes = work_general;
    const uint32_t variant = (b.flags & BF_EVAL_FIXPOINT) | (P.any_parallel << 8) | ((two_tier ? 1u : 0u) << 9) | (L.fields << 16);
    bf_ctx::Plan& pl = c->plan[run_list ? 1 : 0];
    // the shape knobs are read on every pass and are part of the plan key: a changed knob re-plans on the same ctx
    const char* env_st = getenv("BF_STAGES");
    const char* env_w = getenv("BF_WARPS");
    const char* env_b = getenv("BF_BLOCKS_PER_SM");
    const int knobs[3] = {env_st ? atoi(env_st) : 0, env_w ? atoi(env_w) : 0, env_b ? atoi(env_b) : 0};
    if (pl.wpb == 0 || pl.key_stride != L.state_stride || pl.key_words != L.words ||
        pl.key_rec != batch_rec_bytes || pl.key_variant != variant ||
        memcmp(pl.key_knobs, knobs, sizeof knobs) != 0) {
      // Plan: as many resident warps per SM as registers / shared memory allow — the pass is latency/issue bound
      // before it is HBM bound — then ring depth: >= 2 stages keep the next trip's TMA copies in flight under the
      // current evaluation.
      uint32_t best_st = 0, best_wpb = 0, best_score = 0, best_occ2 = 0;
      int best_ctas = 1;
      for (uint32_t st = 1; st <= 4; ++st) {
        if (env_st && (uint32_t)atoi(env_st) != st) continue;
        for (uint32_t wpb = 24; wpb >= 1; wpb = (wpb > 4 ? wpb - 4 : wpb - 1)) {   // 24 / 20: the 80-register build (frontier_kernel.cu)
          if (env_w && !pack && (uint32_t)atoi(env_w) != wpb) continue;
          if (wpb > 16 && (two_tier || run_list)) continue;   // the run-list builds are the 16-warp build only
          const uint32_t smem_try = 128 + wpb * (st * P.stage_bytes + work_general + 64);
          if (smem_try > budget) continue;
          uint32_t occ2 = 0;
          int ctas = bf::frontier_max_blocks_per_sm(PG, wpb * 32, smem_try, &occ2);
          if (ctas < 1) continue;
          if (ctas > 2) ctas = 2;   // the builds are compiled for one or two resident CTAs; many small CTAs measured slower
          if (env_b && atoi(env_b) >= 1 && atoi(env_b) < ctas) ctas = atoi(env_b);
          const uint32_t warps_sm = (uint32_t)ctas * wpb;
          const uint32_t depth = st >= 3 ? 2 : st - 1;           // 0, 1, 2, 2
          const uint32_t score = warps_sm * 16 + depth * 24 + (wpb >= 8 ? 2 : 0) + (4 - st);
          if (score > best_score) { best_score = score; best_st = st; best_wpb = wpb; best_ctas = ctas; best_occ2 = occ2; }
        }
      }
      if (best_wpb == 0) return fail(c, BF_ETOPO, "topology record + run state do not fit shared memory");
      pl.stages = best_st; pl.wpb = best_wpb; pl.per_sm = (uint32_t)best_ctas; pl.occ2 = best_occ2;
      pl.key_stride = L.state_stride; pl.key_words = L.words; pl.key_rec = batch_rec_bytes;
      pl.key_variant = variant;
      memcpy(pl.key_knobs, knobs, sizeof knobs);
    }
    g_st = pl.stages; g_wpb = pl.wpb; g_occ2 = pl.occ2; g_per_sm = (int)pl.per_sm;
  }
  const uint32_t g_smem = 128 + g_wpb * (g_st * P.stage_bytes + work_general + 64);

  // BF_EVAL_COUNTS_SET: the packed-lanes kernel alone publishes the totals itself (last CTA out); every other shape of a pass
  // (two tiers, the general kernel, expansion counts, an empty batch) zeroes the block first and adds as usual
  const bool counts_set = (b.flags & BF_EVAL_COUNTS_SET) && P.counts != nullptr;
  const bool counts_in_kernel = counts_set && pack && !two_tier && !want_exp && b.n_runs != 0;
  if (counts_set && !counts_in_kernel) BF_CUDA(c, cudaMemsetAsync(P.counts, 0, sizeof(bf_counts), stream));
  P.acc = counts_in_kernel ? c->d_acc + 8 * (size_t)(c->acc_seq++ % bf_ctx::kAccSlots) : nullptr;
  c->fused_done = false;
  if (c->fuse_head && pack && !two_tier && !run_list && b.n_runs != 0) {   // a compact tick: the packed-lanes pass leaves heads + block totals itself
    P.head = c->fuse_head; P.head_sums = c->fuse_sums;
    c->fused_done = true;
  }
  // BF_EVAL_PIPELINED applies to a pass that is the packed-lanes kernel alone and touches the counts only behind its wait
  if (!(pack && !two_tier && !want_exp && b.n_runs != 0 && (counts_in_kernel || P.counts == nullptr))) P.flags &= ~BF_EVAL_PIPELINED;

  uint32_t grid = 0, smem = 0;
  if (pack) {
    P.wq = wq; P.wq_log2 = lg; P.warps_per_block = nw; P.slot_groups = ng; P.stages = 1;
    P.run_list = run_list; P.run_list_count = run_list_count;
    if (two_tier) {
      if (int rc = c->d_defer.ensure(c, (size_t)b.n_runs + 1)) return rc;
      P.defer_count = c->d_defer;
      P.defer_list = c->d_defer + 1;
    }
    const uint32_t n_groups = (b.n_runs + R - 1) / R;
    grid = (uint32_t)c->sm_count * pack_ctas_per_sm < n_groups ? (uint32_t)c->sm_count * pack_ctas_per_sm : (n_groups ? n_groups : 1);
    smem = pack_smem;
    if (b.n_runs) {
      if (two_tier) BF_CUDA(c, cudaMemsetAsync(c->d_defer, 0, sizeof(uint32_t), stream));
      BF_CUDA(c, bf::launch_frontier_pack(P, grid, smem, stream));
      c->stats.kernel_launches += 1;
      if (two_tier) {  // second tier: the general kernel over the deferred runs
        bf::KParams P2 = P;
        P2.defer_list = nullptr; P2.defer_count = nullptr;
        P2.run_list = c->d_defer + 1; P2.run_list_count = c->d_defer;
        P2.work_bytes = work_general; P2.stages = g_st; P2.warps_per_block = g_wpb; P2.occ2 = 0; P2.wq = 32; P2.wq_log2 = 5;
        uint32_t grid2 = (uint32_t)c->sm_count;
        const uint32_t nb2 = (b.n_runs + g_wpb - 1) / g_wpb;
        if (grid2 > nb2) grid2 = nb2 ? nb2 : 1;
        BF_CUDA(c, bf::launch_frontier(P2, grid2, g_smem, stream));
        c->stats.kernel_launches += 1;
      }
    }
  } else {
    P.wq = 32u; P.wq_log2 = 5u; P.work_bytes = work_general;
    P.stages = g_st; P.warps_per_block = g_wpb; P.occ2 = g_occ2;
    grid = (uint32_t)c->sm_count * (uint32_t)g_per_sm;
    if (run_list) {   // the 16-warp run-list build, one CTA per SM
      P.run_list = run_list; P.run_list_count = run_list_count; P.occ2 = 0;
      grid = (uint32_t)c->sm_count;
    }
    const uint32_t need_blocks = (b.n_runs + g_wpb - 1) / g_wpb;
    if (grid > need_blocks) grid = need_blocks ? need_blocks : 1;
    smem = g_smem;
    if (b.n_runs) {
      BF_CUDA(c, bf::launch_frontier(P, grid, smem, stream));
      c->stats.kernel_launches += 1;
    }
  }
  if (b.n_runs && want_exp) {
    uint32_t nl = 0;
    BF_CUDA(c, bf::launch_expansion(P, c->d_block_sums, c->d_offsets, d_exp, b.expansion_cap, stream, &nl));
    c->stats.kernel_launches += nl;
  }
  c->stats.last_kernel = (pack ? (two_tier ? 2u : 1u) : 0u) + (run_list ? 3u : 0u); c->stats.last_runs_per_trip = pack ? R : 1u;
  c->stats.last_grid = grid; c->stats.last_block = (pack ? nw : g_wpb) * 32; c->stats.last_smem_bytes = smem;
  c->stats.last_stages = pack ? ng : g_st;
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
// Enqueue on `s` (after the passes that wrote d_result): compaction kernels, D2H of the head words and of a first slice of
// the event list sized from the previous pass (the exact length is only known after the sync; it arrives, with the counts,
// in the pinned tail block the last kernel writes itself).
uint32_t result_tail_of(const bf_layout& L) {
  uint32_t tail = (uint32_t)sizeof(bf_result_header);
  auto upd = [&](uint32_t off, uint32_t len) { if (off != BF_OFF_NONE && off + len > tail) tail = off + len; };
  upd(L.off_ready, L.words * 4); upd(L.off_skip, L.words * 4); upd(L.off_fail, L.words * 4);
  upd(L.off_needs_cond, L.words * 4); upd(L.off_skip_dep, L.words * 4); upd(L.off_phase_out, L.words * 16);
  return tail;
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
                    cudaStream_t s, uint64_t* first_slice, bool with_rejected, bool heads_done) {
  const uint64_t cap = out->events ? out->events_cap : 0;
  if (int rc = compact_prepare(c, n_runs, s)) return rc;
  if (int rc = c->d_events.ensure(c, cap ? (size_t)cap : 1)) return rc;
  bf::CompactParams P{};
  P.result = d_result; P.prev_result = d_prev; P.head = c->d_head; P.events = c->d_events; P.cap = cap;
  P.block_sums = cblock_sums(c, c->cblock_flip); P.zero_sums = cblock_sums(c, c->cblock_flip ^ 1u); P.total = c->d_cblock;
  P.zero_len = (uint32_t)((c->d_cblock.cap - 2) / 2);
  P.heads_done = heads_done ? 1u : 0u;
  c->cblock_flip ^= 1u;   // the next compaction (and a pass fused with it) uses the buffer this one leaves zeroed
  P.n_runs = n_runs; P.words = L.words; P.result_stride = L.result_stride; P.result_tail = result_tail_of(L);
  P.off_ready = L.off_ready; P.off_skip = L.off_skip;
  P.off_fail = L.off_fail; P.off_needs_cond = L.off_needs_cond; P.off_skip_dep = L.off_skip_dep;
  // the small results (event total, counts, rejected deltas, listed runs) are written to the pinned block by the last kernel
  // itself: no latency-bound small D2H copies
  unsigned long long* tail = reinterpret_cast<unsigned long long*>(c->h_counts + 2);   // 7 x u64 in the pinned block
  P.host_tail = tail; P.counts = c->d_counts; P.rejected = with_rejected ? c->d_rejected.p : nullptr;
  // a head buffer in pinned host memory (bf_alloc_pinned, cudaHostAlloc / cudaHostRegister) gets the head words posted by the
  // kernel itself; any other buffer gets them by a download
  P.host_head = nullptr;
  if (out->head && n_runs && !getenv("BF_NO_ZC_HEADS")) P.host_head = static_cast<uint32_t*>(pinned_dev(out->head));
  bool events_posted = false;
  if (out->events && cap && !getenv("BF_NO_ZC_EVENTS")) {   // the event list likewise: posted by the emit kernel, no download
    if (void* d = pinned_dev(out->events)) {
      P.events = static_cast<uint16_t*>(d);
      events_posted = true;
    }
  }
  if (n_runs == 0) BF_CUDA(c, cudaStreamSynchronize(s));   // the empty case stores to the pinned block from the host
  c->cblock_clean = false;   // until the call has gone through (resident_tick_locked / eval_host set it again after the sync)
  BF_CUDA(c, bf::launch_compact(P, s));
  c->stats.kernel_launches += n_runs ? (heads_done ? 1 : 2) : 0;
  uint64_t guess = c->last_events + c->last_events / 32 + 4096;   // the previous tick's list + 3 %: one copy in the steady state
  if (guess > cap) guess = cap;
  if (events_posted) guess = 0;
  if (guess) BF_CUDA(c, cudaMemcpyAsync(out->events, c->d_events, (size_t)guess * sizeof(uint16_t), cudaMemcpyDeviceToHost, s));
  if (out->head && n_runs && !P.host_head) BF_CUDA(c, cudaMemcpyAsync(out->head, c->d_head, (size_t)n_runs * 4, cudaMemcpyDeviceToHost, s));
  *first_slice = events_posted ? cap : guess;   // posted: the whole list is in the caller's buffer after the synchronise
  return BF_OK;
}
// after the stream has been synchronised: fetch what the first slice missed
int compact_finish(bf_ctx* c, bf_compact_out* out, uint64_t first_slice) {
  const unsigned long long* tail = reinterpret_cast<const unsigned long long*>(c->h_counts + 2);
  const uint64_t total = tail[0];
  const uint64_t cap = out->events ? out->events_cap : 0;
  const uint64_t have = total < cap ? total : cap;
  if (have > first_slice)
    BF_CUDA(c, cudaMemcpy(out->events + first_slice, c->d_events + first_slice, (size_t)(have - first_slice) * sizeof(uint16_t),
                          cudaMemcpyDeviceToHost));
  out->n_events = total;
  out->n_listed = (uint32_t)tail[6];
  c->last_events = total;
  return BF_OK;
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
      cudaHostAlloc(reinterpret_cast<void**>(&c->h_counts), 5 * sizeof(bf_counts), cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    bf_destroy(c);  // releases whatever was created
    return BF_ECUDA;
  }
  if (cfg && cfg->arena_bytes) {
    std::lock_guard<std::mutex> g(c->mu);
    if (grow_arena(c, (size_t)cfg->arena_bytes) != BF_OK) { bf_destroy(c); return BF_ENOMEM; }
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
  cudaFreeHost(c->h_counts);
  delete c;   // the device buffers of the ctx and of its resident batches free themselves
}

int bf_topology_put_many(bf_ctx* c, const bf_topology* topos, uint32_t count, uint32_t* slots_out) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  if ((!topos || !slots_out) && count) return fail(c, BF_EINVAL, "null topos/slots_out");
  BF_CUDA(c, cudaSetDevice(c->device));
  return put_many_locked(c, topos, count, slots_out);
}

int bf_topology_put(bf_ctx* c, const bf_topology* topo, uint32_t* slot_out) { return bf_topology_put_many(c, topo, 1, slot_out); }

static int check_locked(bf_ctx* c, const uint32_t* slots, uint32_t count, uint32_t* status_out) {
  if (count == 0) return BF_OK;
  if (int rc = bf::sync_slots(c, c->stream)) return rc;
  uint32_t* d_ids = nullptr;
  uint32_t* d_status = nullptr;
  BF_CUDA(c, cudaMalloc(&d_ids, (size_t)count * 4));
  if (cudaMalloc(&d_status, (size_t)count * 4) != cudaSuccess) { cudaFree(d_ids); return fail(c, BF_ENOMEM, "cudaMalloc status"); }
  cudaError_t e = cudaMemcpyAsync(d_ids, slots, (size_t)count * 4, cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) e = bf::launch_validate(c->slots_dev, d_ids, count, (uint32_t)c->slots_host.size(), d_status, c->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(status_out, d_status, (size_t)count * 4, cudaMemcpyDeviceToHost, c->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  cudaFree(d_ids);
  cudaFree(d_status);
  if (e != cudaSuccess) return cuda_fail(c, e, "device validation");
  c->stats.kernel_launches += 1;
  return BF_OK;
}

int bf_topology_check(bf_ctx* c, const uint32_t* slots, uint32_t count, uint32_t* status_out) {
  if (!c || (count && (!slots || !status_out))) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  BF_CUDA(c, cudaSetDevice(c->device));
  return check_locked(c, slots, count, status_out);
}

int bf_topology_closure(bf_ctx* c, const uint32_t* slots, const uint32_t* steps, uint32_t count, uint32_t words, uint32_t* masks_out) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  if (count && (!slots || !steps || !masks_out)) return fail(c, BF_EINVAL, "null argument");
  if (words == 0 || words > BF_MAX_STEPS / 32) return fail(c, BF_EINVAL, "words out of range (1..32)");
  for (uint32_t i = 0; i < count; ++i) {
    if (slots[i] >= c->meta.size() || !c->meta[slots[i]].alive) return fail(c, BF_ETOPO, "query " + std::to_string(i) + ": unknown topology slot");
    const TopoMeta& m = c->meta[slots[i]];
    if (steps[i] >= m.S) return fail(c, BF_EINVAL, "query " + std::to_string(i) + ": step index out of range");  // "step %q not found", :541
    if ((m.S + 31) / 32 > words) return fail(c, BF_EINVAL, "query " + std::to_string(i) + ": mask too narrow for the topology");
  }
  if (count == 0) return BF_OK;
  BF_CUDA(c, cudaSetDevice(c->device));
  if (int rc = bf::sync_slots(c, c->stream)) return rc;
  uint32_t* d = nullptr;
  const size_t q_bytes = (size_t)count * 4, m_bytes = (size_t)count * words * 4;
  BF_CUDA(c, cudaMalloc(&d, 2 * q_bytes + m_bytes));
  cudaError_t e = cudaMemcpyAsync(d, slots, q_bytes, cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d + count, steps, q_bytes, cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) e = bf::launch_closure(c->slots_dev, d, d + count, count, (uint32_t)c->slots_host.size(), words, d + 2 * (size_t)count, c->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(masks_out, d + 2 * (size_t)count, m_bytes, cudaMemcpyDeviceToHost, c->stream);
  const cudaError_t es = cudaStreamSynchronize(c->stream);
  cudaFree(d);
  c->stats.kernel_launches += 1;
  if (e != cudaSuccess) return cuda_fail(c, e, "bf_topology_closure");
  if (es != cudaSuccess) return cuda_fail(c, es, "cudaStreamSynchronize");
  return BF_OK;
}

static int drop_locked(bf_ctx* c, uint32_t slot);

int bf_topology_put_many_checked_on_device(bf_ctx* c, const bf_topology* topos, uint32_t count, uint32_t* slots_out,
                                           uint32_t* status_out) {
  if (!c || (count && (!topos || !slots_out || !status_out))) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  BF_CUDA(c, cudaSetDevice(c->device));
  if (int rc = put_many_locked(c, topos, count, slots_out, /*host_kahn=*/false)) return rc;
  if (int rc = check_locked(c, slots_out, count, status_out)) return rc;
  for (uint32_t i = 0; i < count; ++i)
    if (status_out[i] & 1u) {  // "dependency cycle detected", dag.go:3145
      drop_locked(c, slots_out[i]);
      slots_out[i] = 0xFFFFFFFFu;
    }
  return BF_OK;
}

static int drop_locked(bf_ctx* c, uint32_t slot) {
  if (slot >= c->meta.size() || !c->meta[slot].alive) return fail(c, BF_ETOPO, "drop of an unknown slot");
  c->meta[slot].alive = false;
  c->slot_changes++;
  if (c->meta[slot].P) c->n_with_parallel--;
  c->slots_host[slot] = bf::Slot{0, 0, 0};
  memset(&c->ff_host[(size_t)slot * bf::FF_STRIDE], 0, bf::FF_STRIDE * sizeof(uint32_t));
  c->free_slots.push_back(slot);
  c->n_alive--;
  c->slots_dirty = true;
  c->rec_max_dirty = true;
  c->arena_dead += round_up_sz(c->meta[slot].bytes, 16);
  if (c->n_alive == 0) {  // nothing left: the bump allocator starts over
    c->arena_used = 0;
    c->arena_dead = 0;
  }
  return BF_OK;
}

int bf_topology_drop(bf_ctx* c, uint32_t slot) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  return drop_locked(c, slot);
}

int bf_topology_child_first(const bf_ctx* c, uint32_t slot, uint32_t* out, uint32_t cap) {
  if (!c || slot >= c->meta.size() || !c->meta[slot].alive) return BF_ETOPO;
  const TopoMeta& m = c->meta[slot];
  for (uint32_t q = 0; q < m.P && q < cap; ++q) out[q] = m.child_first[q];
  return (int)m.P;
}

int bf_topology_record(const bf_ctx* c, uint32_t slot, uint64_t* dev_addr, uint32_t* bytes) {
  if (!c || slot >= c->meta.size() || !c->meta[slot].alive) return BF_ETOPO;
  if (dev_addr) *dev_addr = c->slots_host[slot].addr;
  if (bytes) *bytes = c->meta[slot].bytes;
  return BF_OK;
}

int bf_topology_record_build(const bf_topology* topo, void* out, uint32_t cap, uint32_t* bytes_out) {
  if (!topo) return BF_EINVAL;
  RecPlan p;
  std::string why;
  if (int rc = plan_record(*topo, p, why, true, forced_format())) return rc;
  if (bytes_out) *bytes_out = p.rec_bytes;
  if (!out || cap < p.rec_bytes) return BF_ENOMEM;
  build_record(*topo, p, static_cast<uint8_t*>(out));
  return BF_OK;
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

static int eval_host(bf_ctx* c, const bf_batch* b, bf_compact_out* co) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  if (!b || b->struct_size != sizeof(bf_batch)) return fail(c, BF_EINVAL, "bad bf_batch.struct_size");
  if (co && co->struct_size != sizeof(bf_compact_out)) return fail(c, BF_EINVAL, "bad bf_compact_out.struct_size");
  if (co && co->events_cap && !co->events) return fail(c, BF_EINVAL, "null events with a non-zero events_cap");
  if (int rc = bf::check_layout(c, b->layout)) return rc;
  if (b->n_runs && (!b->state || (!b->result && !co))) return fail(c, BF_EINVAL, "null state/result");
  c->last_eval_valid = false;
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
  cudaStream_t s = c->stream;
  // Large batches are cut into chunks of runs (runs are independent) so that the upload of chunk k+1, the
  // kernel of chunk k and the download of chunk k-1 overlap: PCIe is full duplex and the pass itself is ~5x
  // faster than either copy, so the call costs about max(H2D, D2H) instead of their sum.  Expansion needs a
  // batch-wide scan and stays on the single-stream path.
  uint32_t chunks = 1;
  if (!want_exp && sbytes + rbytes >= (2u << 20)) {
    // ~5.5 MB per chunk, at least two (tools/e2e_sweep.py sweeps the chunk count through BF_E2E_CHUNKS)
    chunks = (uint32_t)((sbytes + rbytes + (11u << 18)) / (11u << 19));
    if (chunks < 2) chunks = 2;
    if (const char* e = getenv("BF_E2E_CHUNKS")) chunks = (uint32_t)atoi(e);
    if (chunks > bf_ctx::kMaxChunks) chunks = bf_ctx::kMaxChunks;
    if (chunks < 1) chunks = 1;
  }
  if (chunks > 1)
    if (int rc = bf::ensure_pipe(c)) return rc;
  const char* shape_env = getenv("BF_E2E_SHAPE");
  const bool taper = shape_env && !strcmp(shape_env, "taper");
  bf_counts hc{};
  uint64_t first_slice = 0;
  auto body = [&]() -> int {
    BF_CUDA(c, cudaMemsetAsync(c->d_counts, 0, sizeof(bf_counts), s));
    bf_batch db = *b;
    db.flags &= ~(uint32_t)(BF_EVAL_COUNTS_SET | BF_EVAL_PIPELINED);   // bf_eval_device only: the chunks here add into one block
    if (!want_exp) db.flags &= ~BF_EVAL_EXPANSION;
    const uint8_t* hs = static_cast<const uint8_t*>(b->state);
    uint8_t* hr = static_cast<uint8_t*>(b->result);
    for (uint32_t k = 0; k < chunks; ++k) {
      // chunk sizes shrink linearly (weights c, c-1, .., 1) when BF_E2E_SHAPE=taper: big early copies overlap best,
      // a small last chunk leaves a short un-overlapped tail (kernel + download of that chunk)
      size_t lo = (size_t)b->n_runs * k / chunks, hi = (size_t)b->n_runs * (k + 1) / chunks;
      if (taper && chunks > 1) {
        const uint64_t tot = (uint64_t)chunks * (chunks + 1) / 2;
        auto cum = [&](uint32_t kk) { return (uint64_t)kk * chunks - (uint64_t)kk * (kk - 1) / 2; };  // sum of the first kk weights
        lo = (size_t)((uint64_t)b->n_runs * cum(k) / tot);
        hi = (size_t)((uint64_t)b->n_runs * cum(k + 1) / tot);
      }
      const size_t so = lo * L.state_stride, ro = lo * L.result_stride;
      const size_t sb = (hi - lo) * L.state_stride, rb = (hi - lo) * L.result_stride;
      const bool piped = chunks > 1;
      if (sb) BF_CUDA(c, cudaMemcpyAsync(c->d_state + so, hs + so, sb, cudaMemcpyHostToDevice, piped ? c->s_in : s));
      if (piped) {
        BF_CUDA(c, cudaEventRecord(c->ev_in[k], c->s_in));
        BF_CUDA(c, cudaStreamWaitEvent(s, c->ev_in[k], 0));
      }
      db.n_runs = (uint32_t)(hi - lo);
      if (int rc = bf::run_pass(c, db, c->d_state + so, c->d_result + ro, want_exp ? c->d_exp.p : nullptr, c->d_counts, s)) return rc;
      if (piped) {
        BF_CUDA(c, cudaEventRecord(c->ev_k[k], s));
        BF_CUDA(c, cudaStreamWaitEvent(c->s_out, c->ev_k[k], 0));
      }
      if (rb && !co) BF_CUDA(c, cudaMemcpyAsync(hr + ro, c->d_result + ro, rb, cudaMemcpyDeviceToHost, piped ? c->s_out : s));
    }
    if (co) {   // counts travel with the compaction's tail block
      if (int rc = bf::compact_enqueue(c, L, c->d_result, nullptr, b->n_runs, co, s, &first_slice, false)) return rc;
    } else {
      BF_CUDA(c, cudaMemcpyAsync(c->h_counts, c->d_counts, sizeof hc, cudaMemcpyDeviceToHost, s));
    }
    return BF_OK;
  };
  const int body_rc = body();
  // never return while a copy that touches the caller's buffers is still in flight
  cudaError_t e_sync = cudaStreamSynchronize(s);
  if (chunks > 1) {
    const cudaError_t e1 = cudaStreamSynchronize(c->s_in), e2 = cudaStreamSynchronize(c->s_out);
    if (e_sync == cudaSuccess) e_sync = e1 != cudaSuccess ? e1 : e2;
  }
  if (body_rc != BF_OK || e_sync != cudaSuccess) c->cblock_clean = false;   // (the compaction scratch may hold a partial pass)
  if (body_rc != BF_OK) return body_rc;
  if (e_sync != cudaSuccess) return cuda_fail(c, e_sync, "cudaStreamSynchronize");
  hc = *c->h_counts;
  if (co) { memcpy(&hc, reinterpret_cast<const unsigned long long*>(c->h_counts + 2) + 1, sizeof hc); c->cblock_clean = true; }
  c->stats.last_eval_chunks = chunks;
  c->last_eval_valid = true; c->last_eval_runs = b->n_runs; c->last_eval_layout = L;
  c->last_state = c->d_state; c->last_result = c->d_result;
  if (want_exp) {
    const uint64_t n = hc.expansion < b->expansion_cap ? hc.expansion : b->expansion_cap;
    if (n) BF_CUDA(c, cudaMemcpy(b->expansion, c->d_exp, (size_t)n * sizeof(bf_expansion), cudaMemcpyDeviceToHost));
  }
  if (b->counts) *b->counts = hc;
  if (co) return bf::compact_finish(c, co, first_slice);
  return BF_OK;
}

int bf_eval(bf_ctx* c, const bf_batch* b) { return eval_host(c, b, nullptr); }
int bf_eval_compact(bf_ctx* c, const bf_batch* b, bf_compact_out* out) {
  if (!out) return c ? fail(c, BF_EINVAL, "null bf_compact_out") : BF_EINVAL;
  return eval_host(c, b, out);
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

// totals hook of a sharded schedule: called between the counting and the truncation kernels with the device totals
struct SchedTotals { uint32_t* story_running; uint32_t* queue_running; int32_t* queue_maxprio; uint32_t* global_running; uint32_t ns, nq; };
typedef int (*sched_between_fn)(void* user, const SchedTotals& t, cudaStream_t s);

static int schedule_host(bf_ctx* c, const bf_batch* b, const bf_sched_run* runs, const bf_sched_tables* t, bf_sched_out* out,
                         sched_between_fn between, void* user, bool with_bases) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  bf::SchedParams P{};
  if (int rc = fill_sched_params(c, b, t, P)) return rc;
  if (!out || out->struct_size != sizeof(bf_sched_out)) return fail(c, BF_EINVAL, "bad bf_sched_out.struct_size");
  if (b->n_runs && (!runs || !out->records)) return fail(c, BF_EINVAL, "null runs/records");
  if (!c->last_eval_valid || c->last_eval_runs != b->n_runs || memcmp(&c->last_eval_layout, &b->layout, sizeof(bf_layout)) != 0)
    return fail(c, BF_EINVAL, "bf_schedule must follow bf_eval / bf_resident_eval of the same batch (n_runs and layout) on this ctx");
  BF_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
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
  P.state = c->last_state; P.result = c->last_result;
  P.runs = reinterpret_cast<const bf_sched_run*>(d + o_runs); P.records = d + o_rec;
  P.story_running = reinterpret_cast<uint32_t*>(d + o_sr); P.queue_running = reinterpret_cast<uint32_t*>(d + o_qr);
  P.queue_maxprio = reinterpret_cast<int32_t*>(d + o_mp); P.global_running = reinterpret_cast<uint32_t*>(d + o_gl);
  P.story_limit = reinterpret_cast<const int32_t*>(d + o_sl); P.queue_limit = reinterpret_cast<const int32_t*>(d + o_ql);
  P.queue_aging = reinterpret_cast<const int32_t*>(d + o_qa);
  P.story_base = (with_bases && t->story_running_base) ? reinterpret_cast<const uint32_t*>(d + o_sb) : nullptr;
  P.queue_base = (with_bases && t->queue_running_base) ? reinterpret_cast<const uint32_t*>(d + o_qb) : nullptr;
  P.queue_maxprio_base = t->queue_max_priority_base ? reinterpret_cast<const int32_t*>(d + o_pb) : nullptr;
  if (!with_bases) P.global_base = 0;
  cudaError_t e = bf::launch_schedule(P, (uint32_t)c->sm_count, s, 1);
  if (e == cudaSuccess && between) {
    const SchedTotals tot{P.story_running, P.queue_running, P.queue_maxprio, P.global_running, (uint32_t)ns, (uint32_t)nq};
    if (int rc = between(user, tot, s)) { cudaStreamSynchronize(s); return rc; }
  }
  if (e == cudaSuccess) e = bf::launch_schedule(P, (uint32_t)c->sm_count, s, 2);
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

int bf_schedule(bf_ctx* c, const bf_batch* b, const bf_sched_run* runs, const bf_sched_tables* t, bf_sched_out* out) {
  return schedule_host(c, b, runs, t, out, nullptr, nullptr, true);
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

// =============================================================================== device groups (row e)
// One process, G devices: a ctx per device, an NCCL communicator over them (libnccl.so.2 via dlopen, so the library
// loads on hosts without NCCL and single-device users never touch it), one worker thread per shard for the duration
// of a call.  The data path has no collective; the one exchange of a pass is the all-gather of the 32-byte counts.
#include <dlfcn.h>
#include <nccl.h>

#include <thread>

namespace {

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool load(std::string& why) {
    if (lib) return true;
    const char* names[] = {getenv("BF_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      if (!n || !*n) continue;
      lib = dlopen(n, RTLD_NOW | RTLD_LOCAL);
      if (lib) break;
    }
    if (!lib) { why = std::string("cannot load libnccl.so.2: ") + (dlerror() ? dlerror() : "?"); return false; }
    CommInitAll = reinterpret_cast<decltype(CommInitAll)>(dlsym(lib, "ncclCommInitAll"));
    CommDestroy = reinterpret_cast<decltype(CommDestroy)>(dlsym(lib, "ncclCommDestroy"));
    AllGather = reinterpret_cast<decltype(AllGather)>(dlsym(lib, "ncclAllGather"));
    AllReduce = reinterpret_cast<decltype(AllReduce)>(dlsym(lib, "ncclAllReduce"));
    GetErrorString = reinterpret_cast<decltype(GetErrorString)>(dlsym(lib, "ncclGetErrorString"));
    if (!CommInitAll || !CommDestroy || !AllGather || !AllReduce || !GetErrorString) { why = "libnccl lacks a required symbol"; return false; }
    return true;
  }
};
NcclApi g_nccl;
std::mutex g_nccl_mu;

}  // namespace

struct bf_group {
  std::vector<bf_ctx*> ctx;
  std::vector<int> dev;
  std::vector<ncclComm_t> comm;
  std::vector<unsigned long long*> d_gather;   // per device: [G][4] gathered counts
  std::vector<bf_counts*> h_gather;            // pinned landing zones
  bool have_nccl = false;
  std::mutex mu;                               // one group call at a time
  std::string err;
  // last bf_group_eval (what bf_group_schedule refers to)
  bool last_valid = false;
  uint32_t last_runs = 0;
};

namespace {
int gfail(bf_group* g, int code, const std::string& msg) {
  if (g) g->err = msg;
  return code;
}
void shard_range(uint32_t n, uint32_t G, uint32_t k, uint32_t* first, uint32_t* count) {
  const uint32_t per = (n + G - 1) / G;
  const uint32_t lo = (uint64_t)k * per < n ? k * per : n;
  const uint32_t hi = (uint64_t)lo + per < n ? lo + per : n;
  *first = lo;
  *count = hi - lo;
}
}  // namespace

extern "C" {

int bf_group_create(bf_group** out, const int32_t* devices, uint32_t n_devices, const bf_config* cfg) {
  if (!out) return BF_EINVAL;
  *out = nullptr;
  if (!devices || n_devices == 0 || n_devices > 64) return BF_EINVAL;
  for (uint32_t i = 0; i < n_devices; ++i)
    for (uint32_t j = 0; j < i; ++j)
      if (devices[i] == devices[j]) return BF_EINVAL;
  bf_group* g = new (std::nothrow) bf_group();
  if (!g) return BF_ENOMEM;
  int rc = BF_OK;
  for (uint32_t i = 0; i < n_devices && rc == BF_OK; ++i) {
    bf_config c1{};
    if (cfg) c1 = *cfg;
    c1.struct_size = sizeof(bf_config);
    c1.device = devices[i];
    bf_ctx* c = nullptr;
    rc = bf_create(&c, &c1);
    if (rc == BF_OK) { g->ctx.push_back(c); g->dev.push_back(devices[i]); }
  }
  if (rc != BF_OK) { bf_group_destroy(g); return rc; }
  // the communicator: required for G > 1, optional (counts of one shard are their own gather) for G == 1
  std::string why;
  {
    std::lock_guard<std::mutex> lk(g_nccl_mu);
    g->have_nccl = g_nccl.load(why);
  }
  if (g->have_nccl) {
    g->comm.assign(n_devices, nullptr);
    const ncclResult_t r = g_nccl.CommInitAll(g->comm.data(), (int)n_devices, g->dev.data());
    if (r != ncclSuccess) {
      why = std::string("ncclCommInitAll: ") + g_nccl.GetErrorString(r);
      g->comm.clear();
      g->have_nccl = false;
    }
  }
  if (!g->have_nccl && n_devices > 1) {
    // no way to report text through a destroyed group: leave it in the first ctx-less form
    fprintf(stderr, "bobrafrontier: bf_group_create: %s\n", why.c_str());
    bf_group_destroy(g);
    return BF_ENCCL;
  }
  for (uint32_t i = 0; i < n_devices; ++i) {
    cudaSetDevice(g->dev[i]);
    unsigned long long* d = nullptr;
    bf_counts* h = nullptr;
    if (cudaMalloc(&d, (size_t)n_devices * sizeof(bf_counts)) != cudaSuccess ||
        cudaHostAlloc(reinterpret_cast<void**>(&h), (size_t)n_devices * sizeof(bf_counts), cudaHostAllocDefault) != cudaSuccess) {
      cudaFree(d);
      bf_group_destroy(g);
      return BF_ENOMEM;
    }
    g->d_gather.push_back(d);
    g->h_gather.push_back(h);
  }
  *out = g;
  return BF_OK;
}

void bf_group_destroy(bf_group* g) {
  if (!g) return;
  for (size_t i = 0; i < g->comm.size(); ++i)
    if (g->comm[i]) { cudaSetDevice(g->dev[i]); g_nccl.CommDestroy(g->comm[i]); }
  for (size_t i = 0; i < g->d_gather.size(); ++i) { cudaSetDevice(g->dev[i]); cudaFree(g->d_gather[i]); cudaFreeHost(g->h_gather[i]); }
  for (bf_ctx* c : g->ctx) bf_destroy(c);
  delete g;
}

uint32_t bf_group_size(const bf_group* g) { return g ? (uint32_t)g->ctx.size() : 0; }
bf_ctx* bf_group_ctx(bf_group* g, uint32_t shard) { return g && shard < g->ctx.size() ? g->ctx[shard] : nullptr; }
const char* bf_group_last_error(const bf_group* g) { return g ? g->err.c_str() : "null group"; }

int bf_group_shard_range(const bf_group* g, uint32_t n_runs, uint32_t shard, uint32_t* first, uint32_t* count) {
  if (!g || shard >= g->ctx.size() || !first || !count) return BF_EINVAL;
  shard_range(n_runs, (uint32_t)g->ctx.size(), shard, first, count);
  return BF_OK;
}

int bf_group_topology_put_many(bf_group* g, const bf_topology* topos, uint32_t count, uint32_t* slots_out) {
  if (!g || (count && (!topos || !slots_out))) return BF_EINVAL;
  std::lock_guard<std::mutex> lk(g->mu);
  std::vector<uint32_t> other(count);
  for (size_t k = 0; k < g->ctx.size(); ++k) {
    const int rc = bf_topology_put_many(g->ctx[k], topos, count, k == 0 ? slots_out : other.data());
    if (rc != BF_OK) return gfail(g, rc, "shard " + std::to_string(k) + ": " + bf_last_error(g->ctx[k]));
    if (k && memcmp(other.data(), slots_out, (size_t)count * 4) != 0)
      return gfail(g, BF_ETOPO, "shard " + std::to_string(k) + " assigned different slots: replicated uploads must precede per-shard ones");
  }
  return BF_OK;
}

int bf_group_eval(bf_group* g, const bf_batch* b, bf_counts* shard_counts) {
  if (!g) return BF_EINVAL;
  std::lock_guard<std::mutex> lk(g->mu);
  g->last_valid = false;
  if (!b || b->struct_size != sizeof(bf_batch)) return gfail(g, BF_EINVAL, "bad bf_batch.struct_size");
  if (b->flags & BF_EVAL_EXPANSION) return gfail(g, BF_EINVAL, "expansion lists are per shard: use bf_eval on bf_group_ctx");
  if (b->n_runs && (!b->state || !b->result)) return gfail(g, BF_EINVAL, "null state/result");
  const uint32_t G = (uint32_t)g->ctx.size();
  std::vector<int> rcs(G, BF_OK);
  std::vector<std::string> errs(G);
  std::vector<bf_counts> local(G);
  auto work = [&](uint32_t k) {
    bf_ctx* c = g->ctx[k];
    uint32_t first, count;
    shard_range(b->n_runs, G, k, &first, &count);
    cudaSetDevice(g->dev[k]);
    memset(&local[k], 0, sizeof(bf_counts));
    if (count) {
      bf_batch sb = *b;
      sb.n_runs = count;
      sb.state = static_cast<const uint8_t*>(b->state) + (size_t)first * b->layout.state_stride;
      sb.result = static_cast<uint8_t*>(b->result) + (size_t)first * b->layout.result_stride;
      sb.counts = &local[k];
      rcs[k] = eval_host(c, &sb, nullptr);
      if (rcs[k] != BF_OK) errs[k] = bf_last_error(c);
    } else {
      cudaMemsetAsync(c->d_counts, 0, sizeof(bf_counts), c->stream);   // an empty shard contributes zeros
    }
    // the pass's one exchange: all-gather of the counts blocks left on the devices (every shard takes part, also after a
    // local failure, so that nobody waits for a missing rank)
    if (g->have_nccl) {
      const ncclResult_t r = g_nccl.AllGather(c->d_counts, g->d_gather[k], 4, ncclUint64, g->comm[k], c->stream);
      if (r != ncclSuccess && rcs[k] == BF_OK) { rcs[k] = BF_ENCCL; errs[k] = std::string("ncclAllGather: ") + g_nccl.GetErrorString(r); }
      cudaMemcpyAsync(g->h_gather[k], g->d_gather[k], (size_t)G * sizeof(bf_counts), cudaMemcpyDeviceToHost, c->stream);
      const cudaError_t e = cudaStreamSynchronize(c->stream);
      if (e != cudaSuccess && rcs[k] == BF_OK) { rcs[k] = BF_ENCCL; errs[k] = std::string("count all-gather: ") + cudaGetErrorString(e); }
    } else {
      g->h_gather[k][0] = local[k];   // G == 1 without NCCL
    }
  };
  if (G == 1) work(0);
  else {
    std::vector<std::thread> th;
    for (uint32_t k = 0; k < G; ++k) th.emplace_back(work, k);
    for (auto& t : th) t.join();
  }
  for (uint32_t k = 0; k < G; ++k)
    if (rcs[k] != BF_OK) return gfail(g, rcs[k], "shard " + std::to_string(k) + ": " + errs[k]);
  // every shard holds the same gathered table; cross-check shard 0's against the locally returned counts
  bf_counts tot{};
  for (uint32_t k = 0; k < G; ++k) {
    const bf_counts& gk = g->h_gather[0][k];
    if (memcmp(&gk, &local[k], sizeof(bf_counts)) != 0) return gfail(g, BF_ENCCL, "gathered counts of shard " + std::to_string(k) + " differ from its own");
    if (shard_counts) shard_counts[k] = gk;
    tot.ready += gk.ready; tot.skip += gk.skip; tot.expansion += gk.expansion; tot.evals += gk.evals;
  }
  if (b->counts) *b->counts = tot;
  g->last_valid = true;
  g->last_runs = b->n_runs;
  return BF_OK;
}

int bf_group_schedule(bf_group* g, const bf_batch* b, const bf_sched_run* runs, const bf_sched_tables* t, bf_sched_out* out) {
  if (!g) return BF_EINVAL;
  std::lock_guard<std::mutex> lk(g->mu);
  if (!b || b->struct_size != sizeof(bf_batch)) return gfail(g, BF_EINVAL, "bad bf_batch.struct_size");
  if (!t || t->struct_size != sizeof(bf_sched_tables) || !out || out->struct_size != sizeof(bf_sched_out))
    return gfail(g, BF_EINVAL, "bad bf_sched_tables / bf_sched_out struct_size");
  if (!g->last_valid || g->last_runs != b->n_runs) return gfail(g, BF_EINVAL, "bf_group_schedule must follow bf_group_eval of the same batch");
  if (b->n_runs && (!runs || !out->records)) return gfail(g, BF_EINVAL, "null runs/records");
  const uint32_t G = (uint32_t)g->ctx.size();
  if (G > 1 && !g->have_nccl) return gfail(g, BF_ENCCL, "no communicator");
  const uint32_t stride = BF_SCHED_STRIDE(b->layout.words);
  std::vector<int> rcs(G, BF_OK);
  std::vector<std::string> errs(G);
  struct Hook { bf_group* g; uint32_t k; };
  auto between = [](void* user, const SchedTotals& tt, cudaStream_t s) -> int {
    Hook* h = static_cast<Hook*>(user);
    bf_group* gg = h->g;
    if (gg->ctx.size() == 1 || !gg->have_nccl) return BF_OK;
    ncclComm_t cm = gg->comm[h->k];
    ncclResult_t r = ncclSuccess;
    if (tt.ns) r = g_nccl.AllReduce(tt.story_running, tt.story_running, tt.ns, ncclUint32, ncclSum, cm, s);
    if (r == ncclSuccess && tt.nq) r = g_nccl.AllReduce(tt.queue_running, tt.queue_running, tt.nq, ncclUint32, ncclSum, cm, s);
    if (r == ncclSuccess && tt.nq) r = g_nccl.AllReduce(tt.queue_maxprio, tt.queue_maxprio, tt.nq, ncclInt32, ncclMax, cm, s);
    if (r == ncclSuccess) r = g_nccl.AllReduce(tt.global_running, tt.global_running, 1, ncclUint32, ncclSum, cm, s);
    if (r != ncclSuccess) { gg->ctx[h->k]->err = std::string("ncclAllReduce: ") + g_nccl.GetErrorString(r); return BF_ENCCL; }
    return BF_OK;
  };
  auto work = [&](uint32_t k) {
    uint32_t first, count;
    shard_range(b->n_runs, G, k, &first, &count);
    cudaSetDevice(g->dev[k]);
    bf_batch sb = *b;
    sb.n_runs = count;
    bf_sched_out so = *out;
    so.records = static_cast<uint8_t*>(out->records) + (size_t)first * stride;
    if (k) { so.story_running = nullptr; so.queue_running = nullptr; so.queue_max_priority = nullptr; so.global_running = nullptr; }
    Hook h{g, k};
    if (count == 0) {   // an empty shard still takes part in the reductions, with zero contributions
      bf_ctx* c = g->ctx[k];
      c->last_eval_valid = true; c->last_eval_runs = 0; c->last_eval_layout = b->layout;
    }
    rcs[k] = schedule_host(g->ctx[k], &sb, runs ? runs + first : nullptr, t, &so, between, &h, k == 0);
    if (rcs[k] != BF_OK) errs[k] = bf_last_error(g->ctx[k]);
  };
  if (G == 1) work(0);
  else {
    std::vector<std::thread> th;
    for (uint32_t k = 0; k < G; ++k) th.emplace_back(work, k);
    for (auto& tt : th) tt.join();
  }
  for (uint32_t k = 0; k < G; ++k)
    if (rcs[k] != BF_OK) return gfail(g, rcs[k], "shard " + std::to_string(k) + ": " + errs[k]);
  return BF_OK;
}

}  // extern "C"
