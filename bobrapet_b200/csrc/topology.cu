// topology.cu — the topology arena of the C ABI (include/bobrafrontier.h): the bf_topology_* entry points.
//
// Packs Story topologies into the device record format (device_record.h), validates what validateRuntimeDependencyGraph
// validates (internal/controller/runs/dag.go:3076-3146), and keeps the records in one device arena behind a slot table.
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
  uint32_t ff[bf::FF_STRIDE];   // the topology's row of the cut table: fail-fast mask, then dependency floors
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
  bool main_only = p.W <= bf::FF_WORDS;
  for (uint32_t i = 0; i < S && main_only; ++i) {
    main_only = ((t.step_flags[i] & BF_SF_GROUP_MASK) >> BF_SF_GROUP_SHIFT) == BF_GROUP_MAIN;
    if (!(t.step_flags[i] & BF_SF_ALLOW_FAILURE)) p.ff[i >> 5] |= 1u << (i & 31u);
  }
  if (!main_only) memset(p.ff, 0, sizeof p.ff);
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
    // (no u16 rows at 8 words: such a topology has byte entries unless BF_TOPO_FORMAT forbids them, then CSR.  The packed
    //  kernel's status words read PAD = 256 as satisfied too, the zero pair behind a run's words; the rule keeps these
    //  topologies' record format.)
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
  // dependency floors (device_record.h): a step without needs is NODEP in byte-entry rows (never walked), walked otherwise
  for (uint32_t w = 0; main_only && w < p.W; ++w) {
    uint32_t fl = bf::FF_FLOOR_NONE;
    for (uint32_t i = 32 * w; i < S && i < 32 * w + 32 && fl != 0; ++i) {
      if (t.row_ptr[i + 1] == t.row_ptr[i]) { if (!bf::ell_has_nodep(p.ell)) fl = 0; continue; }
      for (uint32_t e = t.row_ptr[i]; e < t.row_ptr[i + 1]; ++e) fl = std::min(fl, (uint32_t)t.col_idx[e] + 1u);
    }
    p.ff[bf::FF_WORDS + w] = fl;
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
  DevBuf<unsigned long long> d_moves;
  if (!live.empty()) {
    e = d_moves.alloc(moves.size());
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_moves, moves.data(), moves.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = bf::launch_move_records(c->arena, na, d_moves, (uint32_t)live.size(), c->stream);
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();   // nothing may still read the old arena when it is freed
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
  if (int rc = bf::grow_arena(c, base + total)) return rc;
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

// ---- arena helpers shared with the other translation units (ctx.h) ----------------------------
namespace bf {

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

// the largest live record among the topologies of at most w words (ceil(S/32)), 0 when there is none; drops and arena
// compactions since the last call recompute the maxima first
uint32_t largest_record(bf_ctx* c, uint32_t w) {
  if (c->rec_max_dirty) {
    memset(c->max_rec_by_w, 0, sizeof c->max_rec_by_w);
    for (const TopoMeta& m : c->meta)
      if (m.alive) {
        const uint32_t mw = (m.S + 31) / 32;
        if (m.bytes > c->max_rec_by_w[mw]) c->max_rec_by_w[mw] = m.bytes;
      }
    c->rec_max_dirty = false;
  }
  uint32_t bytes = 0;
  for (uint32_t k = 1; k <= w && k <= 32; ++k)
    if (c->max_rec_by_w[k] > bytes) bytes = c->max_rec_by_w[k];
  return bytes;
}

}  // namespace bf

static int check_locked(bf_ctx* c, const uint32_t* slots, uint32_t count, uint32_t* status_out) {
  if (count == 0) return BF_OK;
  if (int rc = bf::sync_slots(c, c->stream)) return rc;
  DevBuf<uint32_t> d_ids, d_status;
  BF_CUDA(c, d_ids.alloc(count));
  if (d_status.alloc(count) != cudaSuccess) return fail(c, BF_ENOMEM, "cudaMalloc status");
  cudaError_t e = cudaMemcpyAsync(d_ids, slots, (size_t)count * 4, cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) e = bf::launch_validate(c->slots_dev, d_ids, count, (uint32_t)c->slots_host.size(), d_status, c->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(status_out, d_status, (size_t)count * 4, cudaMemcpyDeviceToHost, c->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  if (e != cudaSuccess) return cuda_fail(c, e, "device validation");
  c->stats.kernel_launches += 1;
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

// =============================================================================== C ABI
extern "C" {

int bf_topology_put_many(bf_ctx* c, const bf_topology* topos, uint32_t count, uint32_t* slots_out) {
  if (!c) return BF_EINVAL;
  std::lock_guard<std::mutex> g(c->mu);
  if ((!topos || !slots_out) && count) return fail(c, BF_EINVAL, "null topos/slots_out");
  BF_CUDA(c, cudaSetDevice(c->device));
  return put_many_locked(c, topos, count, slots_out);
}

int bf_topology_put(bf_ctx* c, const bf_topology* topo, uint32_t* slot_out) { return bf_topology_put_many(c, topo, 1, slot_out); }

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
  DevBuf<uint32_t> d;   // slots | steps | masks
  const size_t q_bytes = (size_t)count * 4, m_bytes = (size_t)count * words * 4;
  BF_CUDA(c, d.alloc((size_t)count * (2 + words)));
  cudaError_t e = cudaMemcpyAsync(d, slots, q_bytes, cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d + count, steps, q_bytes, cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) e = bf::launch_closure(c->slots_dev, d, d + count, count, (uint32_t)c->slots_host.size(), words, d + 2 * (size_t)count, c->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(masks_out, d + 2 * (size_t)count, m_bytes, cudaMemcpyDeviceToHost, c->stream);
  const cudaError_t es = cudaStreamSynchronize(c->stream);
  c->stats.kernel_launches += 1;
  if (e != cudaSuccess) return cuda_fail(c, e, "bf_topology_closure");
  if (es != cudaSuccess) return cuda_fail(c, es, "cudaStreamSynchronize");
  return BF_OK;
}

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

}  // extern "C"
