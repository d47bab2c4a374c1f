// host_mirror.cc — C++ host-side mirror of the reference's Story / StoryRun objects for the frontier path
// (include/bobrafrontier_host.h).  Pure host code: name -> index maps, the template-reference scanner of
// buildDependencyGraphs, CSR packing, in-place bit-plane updates of the state records, result decoding.
#include <assert.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/bobrafrontier_host.h"
#include "retire_moves.h"

namespace {

inline uint32_t round_up(uint32_t v, uint32_t a) { return (v + a - 1) / a * a; }
inline bool name_char(char c) {  // [a-zA-Z0-9_\-], the character class of dag.go:3029
  return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '_' || c == '-';
}
inline bool is_space(char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\f' || c == '\v'; }

// One left-to-right pass equivalent to regexp.FindAllStringSubmatch with the pattern of dag.go:3028-3030:
//   steps\.(NAME)\.  |  steps\s*\[\s*['"](NAME)['"]\s*\]  |  \(index\s+\.steps\s+["'](NAME)["']\)
// (leftmost match, alternatives tried in order, matches do not overlap).
void scan_step_refs(const std::string& e, std::vector<std::string>& out) {
  const size_t n = e.size();
  size_t i = 0;
  auto name_at = [&](size_t p, size_t& end) {  // greedy NAME+ starting at p
    size_t q = p;
    while (q < n && name_char(e[q])) ++q;
    end = q;
    return q > p;
  };
  while (i < n) {
    size_t adv = 0;
    if (e.compare(i, 5, "steps") == 0) {
      size_t p = i + 5, q;
      // alternative 1: steps.NAME.
      if (p < n && e[p] == '.' && name_at(p + 1, q) && q < n && e[q] == '.') {
        out.emplace_back(e, p + 1, q - p - 1);
        adv = q + 1 - i;
      } else {
        // alternative 2: steps\s*[\s*'NAME'\s*]
        size_t r = p;
        while (r < n && is_space(e[r])) ++r;
        if (r < n && e[r] == '[') {
          ++r;
          while (r < n && is_space(e[r])) ++r;
          if (r < n && (e[r] == '\'' || e[r] == '"')) {
            size_t s0 = r + 1, s1;
            if (name_at(s0, s1) && s1 < n && (e[s1] == '\'' || e[s1] == '"')) {
              size_t t = s1 + 1;
              while (t < n && is_space(e[t])) ++t;
              if (t < n && e[t] == ']') {
                out.emplace_back(e, s0, s1 - s0);
                adv = t + 1 - i;
              }
            }
          }
        }
      }
    } else if (e.compare(i, 6, "(index") == 0) {
      // alternative 3: (index\s+.steps\s+"NAME")
      size_t r = i + 6, r0 = r;
      while (r < n && is_space(e[r])) ++r;
      if (r > r0 && e.compare(r, 6, ".steps") == 0) {
        size_t u = r + 6, u0 = u;
        while (u < n && is_space(e[u])) ++u;
        if (u > u0 && u < n && (e[u] == '"' || e[u] == '\'')) {
          size_t s0 = u + 1, s1;
          if (name_at(s0, s1) && s1 + 1 < n && (e[s1] == '"' || e[s1] == '\'') && e[s1 + 1] == ')') {
            out.emplace_back(e, s0, s1 - s0);
            adv = s1 + 2 - i;
          }
        }
      }
    }
    i += adv ? adv : 1;
  }
}

std::string sanitize(const std::string& name) {  // step_executor.go:1652-1670
  std::string s = name;
  for (char& c : s)
    if (!((c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c == '_')) c = '_';
  return s;
}

const char* kPhaseNames[14] = {"",       "Pending", "Running",    "Succeeded", "Failed",  "Finished", "Canceled",
                               "Compensated", "Paused",  "Blocked", "Scheduling", "Timeout", "Aborted", "Skipped"};
const char* kQueuedPrefixes[4] = {"Queued due to story concurrency limit", "Queued due to queue concurrency limit",
                                  "Queued due to global concurrency limit", "Queued due to higher-priority work"};

int phase_code_of(const char* phase, const char* message) {
  if (!phase || !*phase) return BF_PHASE_NONE;
  for (int c = 1; c <= 13; ++c)
    if (!strcmp(phase, kPhaseNames[c])) {
      if (c == BF_PHASE_PENDING && message)
        for (const char* p : kQueuedPrefixes)
          if (!strncmp(message, p, strlen(p))) return BF_PHASE_PENDING_QUEUED;  // dag.go:2035-2051
      return c;
    }
  return -1;
}

struct StepDef {
  std::string name;
  int group, type;
  bool allow, toskip, has_if, has_with;
  std::string if_expr, with_raw;
  std::vector<std::string> needs;
  std::vector<std::pair<std::string, bool>> branches;
  int timing_code = -1;   // bfh_story_set_step_timing: BF_DEC_* and delay, or -1: none
  uint32_t timing_delay = 0;
};

inline void set_code(uint8_t* base, uint32_t W, int nbits, uint32_t i, int v) {
  uint32_t* w = reinterpret_cast<uint32_t*>(base);
  const uint32_t m = 1u << (i & 31u);
  for (int b = 0; b < nbits; ++b) {
    uint32_t& x = w[(uint32_t)b * W + (i >> 5)];
    x = ((v >> b) & 1) ? (x | m) : (x & ~m);
  }
}
inline int get_code(const uint8_t* base, uint32_t W, int nbits, uint32_t i) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(base);
  int v = 0;
  for (int b = 0; b < nbits; ++b) v |= (int)((w[(uint32_t)b * W + (i >> 5)] >> (i & 31u)) & 1u) << b;
  return v;
}

// (run, field, index) of a pending delta: the key of bfh_batch::delta_at
inline uint64_t delta_key(uint32_t run, uint32_t field, uint32_t index) { return ((uint64_t)run << 32) | ((uint64_t)field << 16) | index; }

// A batch's state and result arrays, zeroed: pinned when a ctx is given and can pin them, else plain host memory.  The
// destructor frees them; reshape and retire allocate the new arrays first and swap them in once nothing can fail.
struct HostRecords {
  bf_ctx* ctx = nullptr;
  uint8_t* state = nullptr;
  uint8_t* result = nullptr;
  bool pinned = false;

  HostRecords() = default;
  HostRecords(const HostRecords&) = delete;
  HostRecords& operator=(const HostRecords&) = delete;
  ~HostRecords() {
    if (pinned) { bf_free_pinned(ctx, state); bf_free_pinned(ctx, result); }
    else { free(state); free(result); }
  }
  bool alloc(bf_ctx* c, size_t sb, size_t rb) {
    void *ps = nullptr, *pr = nullptr;
    const bool pin = c && bf_alloc_pinned(c, sb, &ps) == BF_OK && bf_alloc_pinned(c, rb, &pr) == BF_OK;
    if (!pin) {
      if (c && ps) bf_free_pinned(c, ps);
      ps = malloc(sb); pr = malloc(rb);
      if (!ps || !pr) { free(ps); free(pr); return false; }
    }
    ctx = c; pinned = pin;
    state = static_cast<uint8_t*>(ps); result = static_cast<uint8_t*>(pr);
    memset(ps, 0, sb); memset(pr, 0, rb);
    return true;
  }
  void swap(HostRecords& o) {
    std::swap(ctx, o.ctx); std::swap(state, o.state); std::swap(result, o.result); std::swap(pinned, o.pinned);
  }
};

}  // namespace

struct bfh_story {
  std::vector<StepDef> defs;           // insertion order
  int continue_on_failure = -1;
  bool realtime = false;
  bool finalized = false;
  std::string err;
  // packed form (index space = allStorySteps)
  std::vector<uint32_t> order;         // index -> def handle
  std::vector<uint32_t> index_of_def;  // def handle -> index
  std::unordered_map<std::string, uint32_t> index;
  std::vector<uint32_t> row_ptr;
  std::vector<uint16_t> col_idx;
  std::vector<uint8_t> flags;
  std::vector<bf_parallel_desc> par;
  std::vector<uint8_t> allow_bits;
  std::vector<uint32_t> child_first;
  uint32_t child_nibbles = 0;
};

struct bfh_batch {
  bf_ctx* ctx = nullptr;
  bf_layout L{};
  uint32_t cap = 0, n = 0;
  HostRecords rec;
  std::vector<const bfh_story*> story_of_run;
  std::string err;
  // resident mode (row f2): the device holds the records, setters log coalesced deltas, eval sends only those
  bool resident = false;
  uint32_t handle = 0;
  uint32_t uploaded = 0;                             // runs [0, uploaded) exist on the device
  uint32_t evaluated = 0;                            // the result records of runs [0, evaluated) hold the last eval's results
  std::unordered_map<uint64_t, uint32_t> delta_at;   // (run, field, index) -> position in `deltas`
  std::vector<bf_delta> deltas;
  uint64_t delta_bytes_sent = 0, full_bytes_sent = 0;

  void log_delta(uint32_t run, uint32_t field, uint32_t index, uint32_t code) {
    if (!resident || run >= uploaded) return;        // a run not yet on the device travels as a full record
    const uint64_t key = delta_key(run, field, index);
    auto it = delta_at.find(key);
    if (it != delta_at.end()) { deltas[it->second].code = (uint8_t)code; return; }   // the last value of a tick wins
    delta_at[key] = (uint32_t)deltas.size();
    bf_delta d;
    d.run = run; d.index = (uint16_t)index; d.field = (uint8_t)field; d.code = (uint8_t)code;
    deltas.push_back(d);
  }
};

// Rewrite the pending deltas in order: fn edits a delta in place and returns whether it stays.  delta_at follows.
template <typename Fn>
static void rewrite_deltas(bfh_batch* b, Fn fn) {
  if (b->deltas.empty()) return;
  size_t keep = 0;
  for (size_t k = 0; k < b->deltas.size(); ++k) {
    bf_delta d = b->deltas[k];
    if (fn(d)) b->deltas[keep++] = d;
  }
  b->deltas.resize(keep);
  b->delta_at.clear();
  for (size_t i = 0; i < keep; ++i) b->delta_at[delta_key(b->deltas[i].run, b->deltas[i].field, b->deltas[i].index)] = (uint32_t)i;
}

// Resident mode: the runs not yet on the device go up as full records
static int flush_uploads(bfh_batch* b) {
  if (b->uploaded >= b->n) return BF_OK;
  const int rc = bf_resident_upload(b->ctx, b->handle, b->uploaded, b->n - b->uploaded, b->rec.state + (size_t)b->uploaded * b->L.state_stride);
  if (rc == BF_OK) { b->full_bytes_sent += (uint64_t)(b->n - b->uploaded) * b->L.state_stride; b->uploaded = b->n; }
  return rc;
}

extern "C" {

// ------------------------------------------------------------------------------------------ Story
bfh_story* bfh_story_new(void) { return new (std::nothrow) bfh_story(); }
void bfh_story_free(bfh_story* s) { delete s; }
const char* bfh_story_error(const bfh_story* s) { return s ? s->err.c_str() : "null story"; }

int bfh_story_add_step(bfh_story* s, const char* name, int group, int type, int allow_failure, int on_timeout_skip,
                       const char* if_expr, const char* with_raw) {
  if (!s || !name || group < 0 || group > 2 || type < 0 || type > 7) return BF_EINVAL;
  if (s->finalized) { s->err = "story already finalized"; return BF_EINVAL; }
  StepDef d;
  d.name = name; d.group = group; d.type = type; d.allow = allow_failure != 0; d.toskip = on_timeout_skip != 0;
  d.has_if = if_expr != nullptr; d.has_with = with_raw != nullptr;
  if (if_expr) d.if_expr = if_expr;
  if (with_raw) d.with_raw = with_raw;
  s->defs.push_back(std::move(d));
  return (int)s->defs.size() - 1;
}
int bfh_step_add_need(bfh_story* s, int step, const char* dep) {
  if (!s || !dep || step < 0 || (size_t)step >= s->defs.size() || s->finalized) return BF_EINVAL;
  s->defs[step].needs.emplace_back(dep);
  return BF_OK;
}
int bfh_step_add_branch(bfh_story* s, int step, const char* bname, int allow) {
  if (!s || !bname || step < 0 || (size_t)step >= s->defs.size() || s->finalized) return BF_EINVAL;
  s->defs[step].branches.emplace_back(bname, allow != 0);
  return BF_OK;
}
int bfh_story_set_policy(bfh_story* s, int cont, int realtime) {
  if (!s) return BF_EINVAL;
  s->continue_on_failure = cont;
  s->realtime = realtime != 0;
  return BF_OK;
}

int bfh_story_set_step_timing(bfh_story* s, int step, int code, uint32_t delay) {
  if (!s || step < 0 || (size_t)step >= s->defs.size()) return BF_EINVAL;
  const int ty = s->defs[step].type;
  const bool ok = code < 0 || (ty == BF_STEP_SLEEP ? code == BF_DEC_SUCCEED || code == BF_DEC_FAIL
                             : ty == BF_STEP_GATE  ? code == BF_DEC_TIMED_OUT || code == BF_DEC_FAIL
                             : ty == BF_STEP_WAIT  ? code == BF_DEC_TIMED_OUT || code == BF_DEC_PENDING || code == BF_DEC_FAIL
                                                   : false);
  if (!ok) { s->err = "step " + s->defs[step].name + ": its type does not take timing code " + std::to_string(code); return BF_EINVAL; }
  s->defs[step].timing_code = code;
  s->defs[step].timing_delay = code < 0 ? 0u : delay;
  return BF_OK;
}

int bfh_story_finalize(bfh_story* s) {
  if (!s) return BF_EINVAL;
  if (s->finalized) return BF_OK;
  const uint32_t n = (uint32_t)s->defs.size();
  if (n == 0 || n > BF_MAX_STEPS) { s->err = "step count out of range (1..1024)"; return BF_ETOPO; }
  // allStorySteps order: main ++ compensations ++ finally (dag.go:3270-3280)
  s->order.clear();
  for (int g = 0; g < 3; ++g)
    for (uint32_t h = 0; h < n; ++h)
      if (s->defs[h].group == g) s->order.push_back(h);
  s->index_of_def.assign(n, 0);
  s->index.clear();
  for (uint32_t i = 0; i < n; ++i) {
    s->index_of_def[s->order[i]] = i;
    if (!s->index.emplace(s->defs[s->order[i]].name, i).second) { s->err = "duplicate step name " + s->defs[s->order[i]].name; return BF_ETOPO; }
  }
  // buildDependencyGraphs is called on the evaluated group's list (dag.go:1700): alias maps are per group
  std::vector<std::vector<uint32_t>> rows(n);
  std::vector<std::string> unknown;
  for (int g = 0; g < 3; ++g) {
    std::unordered_map<std::string, std::string> alias_to_real;  // dag.go:3033-3039
    for (uint32_t i = 0; i < n; ++i) {
      const StepDef& d = s->defs[s->order[i]];
      if (d.group != g) continue;
      const std::string a = sanitize(d.name);
      if (a != d.name) alias_to_real[a] = d.name;
    }
    for (uint32_t i = 0; i < n; ++i) {
      const StepDef& d = s->defs[s->order[i]];
      if (d.group != g) continue;
      std::vector<std::string> deps = d.needs;  // 1. explicit needs (dag.go:3051)
      std::vector<std::string> refs;
      if (d.has_if) scan_step_refs(d.if_expr, refs);  // 2. `if` (dag.go:3056)
      if (d.has_with && (d.type == BF_STEP_ENGRAM || d.type == BF_STEP_EXECUTE_STORY)) scan_step_refs(d.with_raw, refs);  // 3. :3061-3070
      for (std::string& r : refs) {
        auto it = alias_to_real.find(r);
        deps.push_back(it == alias_to_real.end() ? r : it->second);
      }
      for (const std::string& dep : deps) {
        auto it = s->index.find(dep);
        if (it == s->index.end()) unknown.push_back(d.name + "->" + dep);
        else rows[i].push_back(it->second);
      }
      std::sort(rows[i].begin(), rows[i].end());
      rows[i].erase(std::unique(rows[i].begin(), rows[i].end()), rows[i].end());
    }
  }
  if (!unknown.empty()) {  // dag.go:3087-3098
    std::sort(unknown.begin(), unknown.end());
    s->err = "unknown step dependencies: ";
    for (size_t k = 0; k < unknown.size(); ++k) s->err += (k ? ", " : "") + unknown[k];
    return BF_ETOPO;
  }
  s->row_ptr.assign(n + 1, 0);
  s->col_idx.clear();
  s->flags.assign(n, 0);
  s->par.clear(); s->allow_bits.clear(); s->child_first.clear();
  std::vector<bool> bits;
  uint32_t nib = 0;
  for (uint32_t i = 0; i < n; ++i) {
    const StepDef& d = s->defs[s->order[i]];
    s->row_ptr[i + 1] = s->row_ptr[i] + (uint32_t)rows[i].size();
    for (uint32_t c : rows[i]) s->col_idx.push_back((uint16_t)c);
    uint8_t f = (uint8_t)d.type;
    if (d.allow) f |= BF_SF_ALLOW_FAILURE;
    if (d.toskip && (d.type == BF_STEP_GATE || d.type == BF_STEP_WAIT)) f |= BF_SF_ON_TIMEOUT_SKIP;
    if (d.has_if && !d.if_expr.empty()) f |= BF_SF_HAS_IF;
    f |= (uint8_t)(d.group << BF_SF_GROUP_SHIFT);
    s->flags[i] = f;
    if (d.type == BF_STEP_PARALLEL) {
      if (s->par.size() >= BF_MAX_PARALLEL) { s->err = "more than 64 parallel steps"; return BF_ETOPO; }
      bf_parallel_desc pd;
      pd.step = (uint16_t)i; pd.branches = (uint16_t)d.branches.size(); pd.allow_first = (uint32_t)bits.size();
      for (auto& b : d.branches) bits.push_back(b.second);
      s->par.push_back(pd);
      nib = round_up(nib, 8);
      s->child_first.push_back(nib);
      nib += pd.branches;
    }
  }
  if (s->col_idx.size() > BF_MAX_EDGES) { s->err = "too many edges"; return BF_ETOPO; }
  s->child_nibbles = round_up(nib, 8);
  s->allow_bits.assign((bits.size() + 7) / 8, 0);
  for (size_t k = 0; k < bits.size(); ++k)
    if (bits[k]) s->allow_bits[k >> 3] |= (uint8_t)(1u << (k & 7));
  s->finalized = true;
  return BF_OK;
}

int bfh_story_dims(const bfh_story* s, uint32_t* S, uint32_t* E, uint32_t* P) {
  if (!s || !s->finalized) return BF_EINVAL;
  if (S) *S = (uint32_t)s->flags.size();
  if (E) *E = (uint32_t)s->col_idx.size();
  if (P) *P = (uint32_t)s->par.size();
  return BF_OK;
}
int bfh_story_csr(const bfh_story* s, uint32_t* rp, uint16_t* ci, uint8_t* fl) {
  if (!s || !s->finalized) return BF_EINVAL;
  if (rp) memcpy(rp, s->row_ptr.data(), s->row_ptr.size() * 4);
  if (ci && !s->col_idx.empty()) memcpy(ci, s->col_idx.data(), s->col_idx.size() * 2);
  if (fl) memcpy(fl, s->flags.data(), s->flags.size());
  return BF_OK;
}
int bfh_story_upload(bfh_story* s, bf_ctx* ctx, uint32_t* slot_out) {
  if (!s || !ctx || !slot_out) return BF_EINVAL;
  if (!s->finalized)
    if (int rc = bfh_story_finalize(s)) return rc;
  bf_topology t{};
  t.n_steps = (uint32_t)s->flags.size(); t.n_edges = (uint32_t)s->col_idx.size();
  t.row_ptr = s->row_ptr.data(); t.col_idx = s->col_idx.data(); t.step_flags = s->flags.data();
  t.parallel = s->par.data(); t.n_parallel = (uint32_t)s->par.size();
  t.branch_allow_bits = s->allow_bits.empty() ? nullptr : s->allow_bits.data();
  t.n_branch_allow_bits = (uint32_t)s->allow_bits.size() * 8;
  int rc = bf_topology_put(ctx, &t, slot_out);
  std::vector<bf_step_timing> tim;
  for (uint32_t i = 0; rc == BF_OK && i < t.n_steps; ++i) {
    const StepDef& d = s->defs[s->order[i]];
    if (d.timing_code >= 0) tim.push_back(bf_step_timing{(uint16_t)i, (uint8_t)d.timing_code, 0, d.timing_delay});
  }
  if (!tim.empty() && (rc = bf_topology_timings(ctx, *slot_out, tim.data(), (uint32_t)tim.size())) != BF_OK) {
    const std::string why = bf_last_error(ctx);
    bf_topology_drop(ctx, *slot_out);
    s->err = why;
    return rc;
  }
  if (rc != BF_OK) s->err = bf_last_error(ctx);
  return rc;
}
int bfh_story_step_index(const bfh_story* s, const char* name) {
  if (!s || !s->finalized || !name) return -1;
  auto it = s->index.find(name);
  return it == s->index.end() ? -1 : (int)it->second;
}
const char* bfh_story_step_name(const bfh_story* s, uint32_t idx) {
  if (!s || !s->finalized || idx >= s->order.size()) return nullptr;
  return s->defs[s->order[idx]].name.c_str();
}
uint32_t bfh_story_run_flags(const bfh_story* s) {
  if (!s) return 0;
  uint32_t f = 0;
  if (s->continue_on_failure != 1) f |= BF_RF_FAIL_FAST;  // shouldFailFast, dag.go:3504-3511
  if (s->realtime) f |= BF_RF_REALTIME;
  return f;
}
int bfh_scan_step_refs(const char* expression, char* out, size_t cap) {
  if (!expression) return BF_EINVAL;
  std::vector<std::string> refs;
  scan_step_refs(expression, refs);
  std::string j;
  for (auto& r : refs) { j += r; j += '\n'; }
  if (out && cap) { strncpy(out, j.c_str(), cap - 1); out[cap - 1] = 0; }
  return (int)refs.size();
}

// ------------------------------------------------------------------------------------------ Batch
bfh_batch* bfh_batch_new(bf_ctx* ctx, uint32_t steps_max, uint32_t child_nibbles, uint32_t fields, uint32_t capacity) {
  bfh_batch* b = new (std::nothrow) bfh_batch();
  if (!b) return nullptr;
  b->ctx = ctx;
  if (bf_layout_init(&b->L, steps_max, child_nibbles, fields) != BF_OK || capacity == 0) { delete b; return nullptr; }
  b->cap = capacity;
  if (!b->rec.alloc(ctx, (size_t)capacity * b->L.state_stride, (size_t)capacity * b->L.result_stride)) {
    delete b;
    return nullptr;
  }
  return b;
}
void bfh_batch_free(bfh_batch* b) {
  if (!b) return;
  if (b->resident) bf_resident_destroy(b->ctx, b->handle);
  delete b;
}
const char* bfh_batch_error(const bfh_batch* b) { return b ? b->err.c_str() : "null batch"; }
const bf_layout* bfh_batch_layout(const bfh_batch* b) { return b ? &b->L : nullptr; }
uint32_t bfh_batch_size(const bfh_batch* b) { return b ? b->n : 0; }
const void* bfh_batch_state(const bfh_batch* b) { return b ? b->rec.state : nullptr; }
const void* bfh_batch_result(const bfh_batch* b) { return b ? b->rec.result : nullptr; }

int bfh_batch_add_run(bfh_batch* b, const bfh_story* story, uint32_t slot) {
  if (!b || !story || !story->finalized) return BF_EINVAL;
  if (b->n >= b->cap) { b->err = "batch full"; return BF_ENOMEM; }
  if (story->flags.size() > b->L.steps_max) { b->err = "story larger than the batch layout"; return BF_EINVAL; }
  if (b->L.off_child != BF_OFF_NONE && story->child_nibbles > b->L.child_nibbles) { b->err = "child area too small"; return BF_EINVAL; }
  uint8_t* rec = b->rec.state + (size_t)b->n * b->L.state_stride;
  memset(rec, 0, b->L.state_stride);
  bf_run_header* h = reinterpret_cast<bf_run_header*>(rec);
  h->topo_slot = slot;
  h->run_flags = (uint8_t)bfh_story_run_flags(story);
  b->story_of_run.push_back(story);
  return (int)b->n++;
}
int bfh_batch_remove_last_run(bfh_batch* b) {
  if (!b || b->n == 0) return BF_EINVAL;
  b->story_of_run.pop_back();
  --b->n;
  if (b->uploaded > b->n) b->uploaded = b->n;  // the slot's next occupant is uploaded as a full record
  if (b->evaluated > b->n) b->evaluated = b->n;   // and has not been evaluated
  // pending deltas of the removed run must not land on the slot's next occupant (whose full record is uploaded first)
  if (b->resident) rewrite_deltas(b, [gone = b->n](bf_delta& d) { return d.run != gone; });
  return BF_OK;
}

#define RUN_CHECK(b, run, step)                                                                                   \
  if (!(b) || (run) >= (b)->n) return BF_EINVAL;                                                                 \
  const bfh_story* st = (b)->story_of_run[run];                                                                  \
  if ((step) >= st->flags.size()) return BF_EINVAL;                                                              \
  uint8_t* rec = (b)->rec.state + (size_t)(run) * (b)->L.state_stride;

int bfh_run_set_phase_code(bfh_batch* b, uint32_t run, uint32_t step, int code) {
  RUN_CHECK(b, run, step)
  if (code < 0 || code > 14) return BF_EINVAL;
  set_code(rec + b->L.off_phase, b->L.words, 4, step, code);
  b->log_delta(run, BF_DELTA_PHASE, step, (uint32_t)code);
  return BF_OK;
}
int bfh_run_set_phase(bfh_batch* b, uint32_t run, uint32_t step, const char* phase, const char* message) {
  const int c = phase_code_of(phase, message);
  if (c < 0) return BF_EINVAL;
  return bfh_run_set_phase_code(b, run, step, c);
}
int bfh_run_set_cond(bfh_batch* b, uint32_t run, uint32_t step, int code) {
  RUN_CHECK(b, run, step)
  if (b->L.off_cond == BF_OFF_NONE || code < 0 || code > 3) return BF_EINVAL;
  set_code(rec + b->L.off_cond, b->L.words, 2, step, code);
  b->log_delta(run, BF_DELTA_COND, step, (uint32_t)code);
  return BF_OK;
}
int bfh_run_set_decision(bfh_batch* b, uint32_t run, uint32_t step, int code) {
  RUN_CHECK(b, run, step)
  if (b->L.off_decision == BF_OFF_NONE || code < 0 || code > 3) return BF_EINVAL;
  set_code(rec + b->L.off_decision, b->L.words, 2, step, code);
  b->log_delta(run, BF_DELTA_DECISION, step, (uint32_t)code);
  return BF_OK;
}
int bfh_run_set_gate(bfh_batch* b, uint32_t run, uint32_t step, const char* gate_state, int timed_out) {
  int d = BF_DEC_PENDING;  // dag.go:1489-1533: Approved > Rejected > (pending: timeout check)
  if (gate_state && !strcmp(gate_state, "Approved")) d = BF_DEC_SUCCEED;
  else if (gate_state && !strcmp(gate_state, "Rejected")) d = BF_DEC_FAIL;
  else if (timed_out) d = BF_DEC_TIMED_OUT;
  return bfh_run_set_decision(b, run, step, d);
}
int bfh_run_set_run_flags(bfh_batch* b, uint32_t run, int topology_terminated, int host_group) {
  if (!b || run >= b->n) return BF_EINVAL;
  bf_run_header* h = reinterpret_cast<bf_run_header*>(b->rec.state + (size_t)run * b->L.state_stride);
  uint8_t f = (uint8_t)bfh_story_run_flags(b->story_of_run[run]);
  if (topology_terminated) f |= BF_RF_TOPOLOGY_TERMINATED;
  if (host_group >= 0) f |= (uint8_t)(BF_RF_HOST_GROUP | ((host_group & 3) << BF_RF_HOST_GROUP_SHIFT));
  h->run_flags = f;
  b->log_delta(run, BF_DELTA_RUN_FLAGS, 0, f);
  return BF_OK;
}
int bfh_run_register_children(bfh_batch* b, uint32_t run, uint32_t q, int on) {
  if (!b || run >= b->n || q >= b->story_of_run[run]->par.size()) return BF_EINVAL;
  bf_run_header* h = reinterpret_cast<bf_run_header*>(b->rec.state + (size_t)run * b->L.state_stride);
  if (on) h->children_registered |= 1ull << q; else h->children_registered &= ~(1ull << q);
  b->log_delta(run, BF_DELTA_REGISTERED, q, on ? 1u : 0u);
  return BF_OK;
}
int bfh_run_set_child_phase(bfh_batch* b, uint32_t run, uint32_t q, uint32_t branch, const char* phase) {
  if (!b || run >= b->n || b->L.off_child == BF_OFF_NONE) return BF_EINVAL;
  const bfh_story* st = b->story_of_run[run];
  if (q >= st->par.size() || branch >= st->par[q].branches) return BF_EINVAL;
  const int c = phase_code_of(phase, nullptr);
  if (c < 0) return BF_EINVAL;
  uint8_t* ch = b->rec.state + (size_t)run * b->L.state_stride + b->L.off_child;
  const uint32_t i = st->child_first[q] + branch;
  const uint8_t sh = (uint8_t)((i & 1u) * 4u);
  ch[i >> 1] = (uint8_t)((ch[i >> 1] & ~(0xFu << sh)) | ((unsigned)c << sh));
  b->log_delta(run, BF_DELTA_CHILD, i, (uint32_t)c);
  return BF_OK;
}

// The device writes the commit (bf_resident_commit_journal) and the mirror applies the PHASE and REGISTERED items of its journal,
// so that the commit's rules live only in the kernel.  An item whose (run, field, index) a pending delta covers is skipped: the
// next eval applies that delta after the commit, on the device too.  The journal is sized from the last results: a run lists at
// most its ready, skip and fail steps and its ready parallel steps' descs.  With rewrites (bfh_batch_commit_rewrites) a run whose
// result carries BF_SUM_PHASE_CHANGED may list a PHASE item for any step of its Story instead.
static int mirror_commit(bfh_batch* b, const bf_commit_entry* entries, uint32_t n, bf_commit_out* out, uint32_t* n_rewritten,
                         bool rewrites, const char* what) {
  if (!b) return BF_EINVAL;
  if (!b->resident) { b->err = std::string(what) + " needs resident mode"; return BF_EINVAL; }
  const bf_layout& L = b->L;
  const uint32_t runs = b->evaluated;
  uint64_t cap = 0;
  for (uint32_t r = 0; r < runs; ++r) {
    const uint8_t* res = b->rec.result + (size_t)r * L.result_stride;
    auto word = [&](uint32_t off, uint32_t w) { return off == BF_OFF_NONE ? 0u : reinterpret_cast<const uint32_t*>(res + off)[w]; };
    const bool rewriting = rewrites && (reinterpret_cast<const bf_result_header*>(res)->summary & BF_SUM_PHASE_CHANGED);
    if (rewriting) cap += 32ull * L.words;
    else
      for (uint32_t w = 0; w < L.words; ++w) cap += (uint64_t)__builtin_popcount(word(L.off_ready, w) | word(L.off_skip, w) | word(L.off_fail, w));
    for (const bf_parallel_desc& d : b->story_of_run[r]->par) cap += (word(L.off_ready, d.step >> 5) >> (d.step & 31u)) & 1u;
  }
  std::vector<bf_commit_write> items(cap);
  bf_commit_out o{};
  o.struct_size = sizeof o;
  bf_commit_journal j{};
  j.struct_size = sizeof j;
  j.items = items.data(); j.items_cap = cap;
  uint32_t nrw = 0;
  const int rc = rewrites ? bf_resident_commit_rewrites(b->ctx, b->handle, runs, entries, n, &o, nullptr, &j, &nrw)
                          : bf_resident_commit_journal(b->ctx, b->handle, runs, entries, n, &o, nullptr, &j);
  if (out) *out = o;
  if (n_rewritten) *n_rewritten = nrw;
  if (rc != BF_OK) { b->err = bf_last_error(b->ctx); return rc; }
  // cap bounds the journal: the commit reads the result records this mirror holds (the last eval's), the mirror's batch has no
  // limiter area (launched = ready, nothing queued) and the call arms nothing, so every PHASE item is a ready, skip or fail step
  // (any step of a rewriting run) and every REGISTERED item the desc of a ready parallel step
  assert(j.n_items <= cap);
  for (uint64_t i = 0; i < std::min<uint64_t>(j.n_items, cap); ++i) {
    const bf_commit_write& w = items[i];
    if (b->delta_at.count(delta_key(w.run, w.field, w.index))) continue;
    uint8_t* rec = b->rec.state + (size_t)w.run * L.state_stride;
    if (w.field == BF_DELTA_PHASE) set_code(rec + L.off_phase, L.words, 4, w.index, (int)w.after);
    else if (w.field == BF_DELTA_REGISTERED) reinterpret_cast<bf_run_header*>(rec)->children_registered |= 1ull << w.index;
  }
  return BF_OK;
}

int bfh_batch_commit(bfh_batch* b, const bf_commit_entry* entries, uint32_t n, bf_commit_out* out) {
  return mirror_commit(b, entries, n, out, nullptr, false, "bfh_batch_commit");
}

int bfh_batch_commit_rewrites(bfh_batch* b, const bf_commit_entry* entries, uint32_t n, bf_commit_out* out, uint32_t* n_rewritten) {
  return mirror_commit(b, entries, n, out, n_rewritten, true, "bfh_batch_commit_rewrites");
}

int bfh_batch_eval(bfh_batch* b, uint32_t eval_flags, bf_counts* counts) {
  if (!b) return BF_EINVAL;
  if (!b->ctx) { b->err = "batch was created without a device context"; return BF_ENODEV; }
  if (b->resident) {
    // new runs as full records, everything else as the tick's coalesced deltas, then one pass over the device copy
    int rc = flush_uploads(b);
    if (rc == BF_OK && !b->deltas.empty()) {
      rc = bf_resident_apply(b->ctx, b->handle, b->deltas.data(), (uint32_t)b->deltas.size());
      b->delta_bytes_sent += b->deltas.size() * sizeof(bf_delta);
    }
    b->deltas.clear();
    b->delta_at.clear();
    if (rc == BF_OK) rc = bf_resident_eval(b->ctx, b->handle, b->n, eval_flags & ~(uint32_t)BF_EVAL_EXPANSION, 0, b->rec.result, counts);
    if (rc != BF_OK) b->err = bf_last_error(b->ctx);
    b->evaluated = rc == BF_OK ? b->n : 0;
    return rc;
  }
  bf_batch bb{};
  bb.struct_size = sizeof(bf_batch);
  bb.n_runs = b->n; bb.flags = eval_flags; bb.layout = b->L;
  bb.state = b->rec.state; bb.result = b->rec.result; bb.counts = counts;
  const int rc = bf_eval(b->ctx, &bb);
  if (rc != BF_OK) b->err = bf_last_error(b->ctx);
  b->evaluated = rc == BF_OK ? b->n : 0;
  return rc;
}

int bfh_story_migration_map(const bfh_story* os, const bfh_story* ns, uint16_t* map, uint32_t cap) {
  if (!os || !ns || !os->finalized || !ns->finalized || (cap && !map)) return BF_EINVAL;
  const uint32_t S = (uint32_t)os->order.size();
  for (uint32_t i = 0; i < S && i < cap; ++i) {
    auto it = ns->index.find(os->defs[os->order[i]].name);
    map[i] = it == ns->index.end() ? (uint16_t)BF_MIGRATE_GONE : (uint16_t)it->second;
  }
  return (int)S;
}

int bfh_batch_migrate(bfh_batch* b, const bfh_story* os, const bfh_story* ns, uint32_t old_slot, uint32_t new_slot) {
  if (!b || !os || !ns || !os->finalized || !ns->finalized) return BF_EINVAL;
  const bf_layout& L = b->L;
  const uint32_t So = (uint32_t)os->flags.size(), W = L.words;
  if (old_slot == new_slot) { b->err = "migration from a slot to itself"; return BF_EINVAL; }
  if (ns->flags.size() > L.steps_max || (L.off_child != BF_OFF_NONE && ns->child_nibbles > L.child_nibbles)) {
    b->err = "the new story does not fit the batch layout";
    return BF_EINVAL;
  }
  std::vector<uint16_t> map(So);
  bfh_story_migration_map(os, ns, map.data(), So);
  std::vector<uint16_t> inv((size_t)W * 32, (uint16_t)BF_MIGRATE_GONE);
  for (uint32_t i = 0; i < So; ++i)
    if (map[i] != BF_MIGRATE_GONE) inv[map[i]] = (uint16_t)i;
  std::vector<int> desc_to(os->par.size(), -1);   // old parallel desc -> new desc, or -1
  for (size_t p = 0; p < os->par.size(); ++p) {
    const uint16_t j = map[os->par[p].step];
    if (j == BF_MIGRATE_GONE) continue;
    for (size_t q = 0; q < ns->par.size(); ++q)
      if (ns->par[q].step == j) {
        if (ns->par[q].branches != os->par[p].branches) {
          b->err = "parallel step " + os->defs[os->order[os->par[p].step]].name + " changes its branch count: re-pack its runs";
          return BF_EINVAL;
        }
        desc_to[p] = (int)q;
      }
  }
  std::vector<uint8_t> moved(b->n, 0);
  uint32_t n_moved = 0, n_on_device = 0;
  for (uint32_t r = 0; r < b->n; ++r) {
    if (reinterpret_cast<const bf_run_header*>(b->rec.state + (size_t)r * L.state_stride)->topo_slot != old_slot) continue;
    if (b->story_of_run[r] != os) { b->err = "run " + std::to_string(r) + " holds old_slot but is not a run of old_story"; return BF_EINVAL; }
    moved[r] = 1;
    ++n_moved;
    if (r < b->uploaded) ++n_on_device;
  }
  if (b->resident && b->uploaded) {   // the device first: it validates what the mirror cannot (live slots), and fails without changes
    bf_migration m{};
    m.struct_size = sizeof m; m.old_slot = old_slot; m.new_slot = new_slot; m.n_runs = b->uploaded;
    m.step_map = map.data(); m.n_old_steps = So;
    const int rc = bf_resident_migrate(b->ctx, b->handle, &m);
    if (rc != BF_OK) { b->err = bf_last_error(b->ctx); return rc; }
    if (m.migrated != n_on_device) {
      // the device copy had diverged from the mirror (its records were changed behind the mirror's back) and has now moved
      // runs the mirror did not: the mirror stays as it was, and the next bfh_batch_eval re-sends every record in full
      b->uploaded = 0;
      b->deltas.clear();
      b->delta_at.clear();
      b->err = "the device moved " + std::to_string(m.migrated) + " runs, the mirror holds " + std::to_string(n_on_device) +
               " on the old slot: the mirror is unchanged and its records will be uploaded in full";
      return BF_EINVAL;
    }
  }
  // re-pack the mirror's records: codes by step name, child phases and registered bits by parallel desc
  std::vector<uint8_t> old(L.state_stride);
  for (uint32_t r = 0; r < b->n; ++r) {
    if (!moved[r]) continue;
    uint8_t* rec = b->rec.state + (size_t)r * L.state_stride;
    memcpy(old.data(), rec, L.state_stride);
    for (uint32_t j = 0; j < W * 32; ++j) {
      const uint32_t o = inv[j];
      set_code(rec + L.off_phase, W, 4, j, o == BF_MIGRATE_GONE ? 0 : get_code(old.data() + L.off_phase, W, 4, o));
      if (L.off_cond != BF_OFF_NONE) set_code(rec + L.off_cond, W, 2, j, o == BF_MIGRATE_GONE ? 0 : get_code(old.data() + L.off_cond, W, 2, o));
      if (L.off_decision != BF_OFF_NONE)
        set_code(rec + L.off_decision, W, 2, j, o == BF_MIGRATE_GONE ? 0 : get_code(old.data() + L.off_decision, W, 2, o));
    }
    bf_run_header* h = reinterpret_cast<bf_run_header*>(rec);
    const uint64_t reg_old = h->children_registered;
    uint64_t reg = 0;
    if (L.off_child != BF_OFF_NONE)
      for (uint32_t i = 0; i < L.child_nibbles; ++i) rec[L.off_child + (i >> 1)] &= (uint8_t)~(0xFu << ((i & 1u) * 4u));
    for (size_t p = 0; p < os->par.size(); ++p) {
      if (desc_to[p] < 0) continue;
      const uint32_t q = (uint32_t)desc_to[p];
      if ((reg_old >> p) & 1u) reg |= 1ull << q;
      if (L.off_child == BF_OFF_NONE) continue;
      for (uint32_t br = 0; br < os->par[p].branches; ++br) {
        const uint32_t si = os->child_first[p] + br, di = ns->child_first[q] + br;
        const uint32_t v = (old[L.off_child + (si >> 1)] >> ((si & 1u) * 4u)) & 0xFu;
        rec[L.off_child + (di >> 1)] |= (uint8_t)(v << ((di & 1u) * 4u));
      }
    }
    h->children_registered = reg;
    h->topo_slot = new_slot;
    b->story_of_run[r] = ns;
  }
  // pending deltas of the moved runs follow their step / desc, or are dropped with a removed step
  rewrite_deltas(b, [&](bf_delta& d) {
    if (d.run >= b->n || !moved[d.run]) return true;
    if (d.field == BF_DELTA_PHASE || d.field == BF_DELTA_COND || d.field == BF_DELTA_DECISION) {
      if (d.index >= So || map[d.index] == BF_MIGRATE_GONE) return false;
      d.index = map[d.index];
    } else if (d.field == BF_DELTA_REGISTERED) {
      if (d.index >= desc_to.size() || desc_to[d.index] < 0) return false;
      d.index = (uint16_t)desc_to[d.index];
    } else if (d.field == BF_DELTA_CHILD) {
      for (size_t p = 0; p < os->par.size(); ++p)
        if (desc_to[p] >= 0 && d.index >= os->child_first[p] && d.index < os->child_first[p] + os->par[p].branches) {
          d.index = (uint16_t)(ns->child_first[desc_to[p]] + (d.index - os->child_first[p]));
          return true;
        }
      return false;
    }
    return true;
  });
  return (int)n_moved;
}

// Reset set of a redrive from `start` (resolveRedriveFromStepSet, storyrun_controller.go:535-558): start plus every step of its
// group reachable through the dependents edges, by a queue over the story's rows reversed.  mask: ceil(S/32) words.
static void redrive_closure(const bfh_story* s, uint32_t start, std::vector<uint32_t>& mask) {
  const uint32_t S = (uint32_t)s->flags.size();
  std::vector<std::vector<uint32_t>> dependents(S);
  for (uint32_t i = 0; i < S; ++i)
    for (uint32_t e = s->row_ptr[i]; e < s->row_ptr[i + 1]; ++e) dependents[s->col_idx[e]].push_back(i);
  auto group = [&](uint32_t i) { return (s->flags[i] & BF_SF_GROUP_MASK) >> BF_SF_GROUP_SHIFT; };
  mask.assign((S + 31) / 32, 0u);
  mask[start >> 5] |= 1u << (start & 31u);
  std::vector<uint32_t> queue{start};
  for (size_t k = 0; k < queue.size(); ++k)
    for (uint32_t i : dependents[queue[k]])
      if (group(i) == group(start) && !((mask[i >> 5] >> (i & 31u)) & 1u)) {
        mask[i >> 5] |= 1u << (i & 31u);
        queue.push_back(i);
      }
}

int bfh_batch_redrive(bfh_batch* b, const uint32_t* runs, const int32_t* steps, uint32_t n) {
  if (!b || (n && (!runs || !steps))) return BF_EINVAL;
  const bf_layout& L = b->L;
  const uint32_t W = L.words;
  for (uint32_t i = 0; i < n; ++i) {
    if (runs[i] >= b->n) { b->err = "request " + std::to_string(i) + ": run out of range"; return BF_EINVAL; }
    if (steps[i] < -1 || (steps[i] >= 0 && (uint32_t)steps[i] >= b->story_of_run[runs[i]]->flags.size())) {
      b->err = "request " + std::to_string(i) + ": step not found in the run's story";
      return BF_EINVAL;
    }
  }
  bool resync = false;
  if (b->resident) {   // the device first: it fails without changes, and then the mirror stays as it was too
    std::vector<bf_redrive> req;
    for (uint32_t i = 0; i < n; ++i) {
      if (runs[i] >= b->uploaded) continue;   // not on the device yet: it travels as a full record
      bf_redrive q{};
      q.run = runs[i];
      q.slot = reinterpret_cast<const bf_run_header*>(b->rec.state + (size_t)runs[i] * L.state_stride)->topo_slot;
      q.step = steps[i] < 0 ? BF_REDRIVE_ALL : (uint32_t)steps[i];
      req.push_back(q);
    }
    if (!req.empty()) {
      std::vector<uint8_t> status(req.size());
      uint32_t applied = 0;
      const int rc = bf_resident_redrive(b->ctx, b->handle, req.data(), (uint32_t)req.size(), status.data(), &applied);
      if (rc != BF_OK) { b->err = bf_last_error(b->ctx); return rc; }
      resync = applied != req.size();   // a device record held another slot: it diverged from the mirror
    }
  }
  // reset the mirror's records; reset[(run, field, index)] marks the pending deltas the reset supersedes
  std::map<std::pair<const bfh_story*, int32_t>, std::vector<uint32_t>> closures;
  std::unordered_map<uint64_t, bool> superseded;
  std::vector<uint8_t> reset_runs(b->n, 0);
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t run = runs[i];
    const bfh_story* st = b->story_of_run[run];
    const uint32_t S = (uint32_t)st->flags.size();
    std::vector<uint32_t>& m = closures[{st, steps[i]}];
    if (m.empty()) {
      if (steps[i] < 0) {
        m.assign((S + 31) / 32, 0u);
        for (uint32_t j = 0; j < S; ++j) m[j >> 5] |= 1u << (j & 31u);
      } else {
        redrive_closure(st, (uint32_t)steps[i], m);
      }
    }
    uint8_t* rec = b->rec.state + (size_t)run * L.state_stride;
    auto in = [&](uint32_t j) { return ((m[j >> 5] >> (j & 31u)) & 1u) != 0; };
    for (uint32_t j = 0; j < S; ++j) {
      if (!in(j)) continue;
      set_code(rec + L.off_phase, W, 4, j, 0);
      superseded[delta_key(run, BF_DELTA_PHASE, j)] = true;
      if (L.off_decision != BF_OFF_NONE) { set_code(rec + L.off_decision, W, 2, j, BF_DEC_PENDING); superseded[delta_key(run, BF_DELTA_DECISION, j)] = true; }
      if (L.off_cond != BF_OFF_NONE) {
        set_code(rec + L.off_cond, W, 2, j, (st->flags[j] & BF_SF_HAS_IF) ? BF_COND_HOLD : BF_COND_PASS);
        superseded[delta_key(run, BF_DELTA_COND, j)] = true;
      }
    }
    bf_run_header* h = reinterpret_cast<bf_run_header*>(rec);
    for (size_t p = 0; p < st->par.size(); ++p) {
      if (!in(st->par[p].step)) continue;
      h->children_registered &= ~(1ull << p);
      superseded[delta_key(run, BF_DELTA_REGISTERED, (uint32_t)p)] = true;
      if (L.off_child == BF_OFF_NONE) continue;
      for (uint32_t br = 0; br < st->par[p].branches; ++br) {
        const uint32_t c = st->child_first[p] + br;
        rec[L.off_child + (c >> 1)] &= (uint8_t)~(0xFu << ((c & 1u) * 4u));
        superseded[delta_key(run, BF_DELTA_CHILD, c)] = true;
      }
    }
    h->run_flags &= (uint8_t)~BF_RF_TOPOLOGY_TERMINATED;
    reset_runs[run] = 1;
  }
  if (resync) {   // the mirror's records are the truth: the next bfh_batch_eval sends them all in full
    b->uploaded = 0;
    b->deltas.clear();
    b->delta_at.clear();
  } else {
    rewrite_deltas(b, [&](bf_delta& d) {
      if (superseded.count(delta_key(d.run, d.field, d.index))) return false;
      if (d.field == BF_DELTA_RUN_FLAGS && d.run < b->n && reset_runs[d.run]) d.code &= (uint8_t)~BF_RF_TOPOLOGY_TERMINATED;
      return true;
    });
  }
  return BF_OK;
}

// Plane field of a record re-laid from `from_off` (Wo words per plane) to `to_off` (Wn words per plane, zeroed): each plane
// keeps its low min(Wn, Wo) words, the words above them stay 0; a field either layout lacks stays 0 / is dropped.
static void relay_planes(uint8_t* dst, const uint8_t* src, uint32_t to_off, uint32_t from_off, uint32_t planes, uint32_t Wn, uint32_t Wo) {
  if (to_off == BF_OFF_NONE || from_off == BF_OFF_NONE) return;
  const size_t w = std::min(Wn, Wo);
  for (uint32_t p = 0; p < planes; ++p) memcpy(dst + to_off + (size_t)p * Wn * 4, src + from_off + (size_t)p * Wo * 4, w * 4);
}

static uint32_t child_area_bytes(const bf_layout& L) { return L.off_child == BF_OFF_NONE ? 0u : ((L.child_nibbles + 1) / 2 + 3) / 4 * 4; }

// Run r's state and result records in `from` (layout F) re-laid to run q of `to` (layout T), as bf_resident_reshape, _narrow and
// _transfer re-lay the device's: the whole destination records written, the headers kept, each plane and mask its low words,
// the child area its low bytes, everything else zero.
static void relay_record(const HostRecords& from, uint32_t r, const bf_layout& F, HostRecords& to, uint32_t q, const bf_layout& T) {
  const uint32_t Wn = T.words, Wo = F.words;
  const uint8_t* s = from.state + (size_t)r * F.state_stride;
  uint8_t* d = to.state + (size_t)q * T.state_stride;
  memset(d, 0, T.state_stride);
  memcpy(d, s, sizeof(bf_run_header));
  relay_planes(d, s, T.off_phase, F.off_phase, 4, Wn, Wo);
  relay_planes(d, s, T.off_cond, F.off_cond, 2, Wn, Wo);
  relay_planes(d, s, T.off_decision, F.off_decision, 2, Wn, Wo);
  if (F.off_child != BF_OFF_NONE && T.off_child != BF_OFF_NONE)
    memcpy(d + T.off_child, s + F.off_child, std::min(child_area_bytes(F), child_area_bytes(T)));
  s = from.result + (size_t)r * F.result_stride;
  d = to.result + (size_t)q * T.result_stride;
  memset(d, 0, T.result_stride);
  memcpy(d, s, sizeof(bf_result_header));
  relay_planes(d, s, T.off_ready, F.off_ready, 1, Wn, Wo);
  relay_planes(d, s, T.off_skip, F.off_skip, 1, Wn, Wo);
  relay_planes(d, s, T.off_fail, F.off_fail, 1, Wn, Wo);
  relay_planes(d, s, T.off_needs_cond, F.off_needs_cond, 1, Wn, Wo);
  relay_planes(d, s, T.off_skip_dep, F.off_skip_dep, 1, Wn, Wo);
  relay_planes(d, s, T.off_phase_out, F.off_phase_out, 4, Wn, Wo);
}

// every record of the mirror re-laid from F to T into nr, at the same index
static void relay_records(const bfh_batch* b, HostRecords& nr, const bf_layout& F, const bf_layout& T) {
  for (uint32_t r = 0; r < b->cap; ++r) relay_record(b->rec, r, F, nr, r, T);
}

int bfh_batch_reshape(bfh_batch* b, uint32_t steps_max, uint32_t child_nibbles, uint32_t fields, uint32_t capacity) {
  if (!b) return BF_EINVAL;
  bf_layout T;
  if (bf_layout_init(&T, steps_max, child_nibbles, fields) != BF_OK) { b->err = "steps_max out of range"; return BF_EINVAL; }
  const bf_layout F = b->L;
  if (capacity < b->cap || T.steps_max < F.steps_max || (F.fields & ~T.fields) ||
      (F.off_child != BF_OFF_NONE && T.child_nibbles < F.child_nibbles)) {
    b->err = "a reshape only grows the batch (capacity, steps_max, fields, child_nibbles)";
    return BF_EINVAL;
  }
  HostRecords nr;
  if (!nr.alloc(b->ctx, (size_t)capacity * T.state_stride, (size_t)capacity * T.result_stride)) {
    b->err = "out of host memory";
    return BF_ENOMEM;
  }
  if (b->resident) {   // the device first: it fails without changes, and then the mirror stays as it was too
    const int rc = bf_resident_reshape(b->ctx, b->handle, &T, capacity);
    if (rc != BF_OK) { b->err = bf_last_error(b->ctx); return rc; }
  }
  relay_records(b, nr, F, T);
  b->rec.swap(nr);
  b->L = T; b->cap = capacity;
  return BF_OK;
}

// steps needed by plane word w holding v: one past its highest set bit
static uint32_t word_extent(uint32_t w, uint32_t v) { return v ? 32u * w + 32u - (uint32_t)__builtin_clz(v) : 0u; }

// the input fields (BF_F_COND, _DECISION, _CHILD) layout T has a place for
static uint32_t placed(const bf_layout& T) {
  return (T.off_cond != BF_OFF_NONE ? BF_F_COND : 0u) | (T.off_decision != BF_OFF_NONE ? BF_F_DECISION : 0u) |
         (T.off_child != BF_OFF_NONE ? BF_F_CHILD : 0u);
}

struct RunExtent {
  uint32_t steps = 0, child = 0, fields = 0;   // steps_max and child_nibbles it needs, the input fields holding a non-default code
};

// The extent of bf_resident_extent over run r of a mirror alone, against a target layout T: the code planes and child nibbles of
// its record (any r < cap), its Story (r < n), and the result planes T keeps when the last eval evaluated it (r < evaluated).
static RunExtent run_extent(const bfh_batch* b, uint32_t r, const bf_layout& T) {
  const bf_layout& F = b->L;
  const uint32_t W = F.words;
  RunExtent e;
  auto planes = [&](const uint8_t* rec, uint32_t off, uint32_t n, uint32_t field) {
    if (off == BF_OFF_NONE) return;
    const uint32_t* p = reinterpret_cast<const uint32_t*>(rec + off);
    for (uint32_t k = 0; k < n * W; ++k)
      if (p[k]) { e.steps = std::max(e.steps, word_extent(k % W, p[k])); e.fields |= field; }
  };
  const uint8_t* rec = b->rec.state + (size_t)r * F.state_stride;
  planes(rec, F.off_phase, 4, 0);
  planes(rec, F.off_cond, 2, BF_F_COND);
  planes(rec, F.off_decision, 2, BF_F_DECISION);
  for (uint32_t i = 0; F.off_child != BF_OFF_NONE && i < F.child_nibbles; ++i)
    if ((rec[F.off_child + i / 2] >> ((i & 1u) * 4u)) & 0xFu) { e.child = std::max(e.child, i + 1); e.fields |= BF_F_CHILD; }
  if (r >= b->n) return e;
  e.steps = std::max(e.steps, (uint32_t)b->story_of_run[r]->flags.size());
  e.child = std::max(e.child, b->story_of_run[r]->child_nibbles);
  if (r >= b->evaluated) return e;   // a run added since the last eval has no results yet
  const uint8_t* res = b->rec.result + (size_t)r * F.result_stride;
  auto kept = [](uint32_t to, uint32_t from) { return to != BF_OFF_NONE ? from : BF_OFF_NONE; };
  planes(res, F.off_ready, 1, 0);
  planes(res, F.off_skip, 1, 0);
  planes(res, kept(T.off_fail, F.off_fail), 1, 0);
  planes(res, kept(T.off_needs_cond, F.off_needs_cond), 1, 0);
  planes(res, kept(T.off_skip_dep, F.off_skip_dep), 1, 0);
  planes(res, kept(T.off_phase_out, F.off_phase_out), 4, 0);
  return e;
}

// whether a pending delta still has its place in layout T
static bool delta_fits(const bf_delta& d, const bf_layout& T) {
  return d.field == BF_DELTA_PHASE      ? d.index < T.steps_max
         : d.field == BF_DELTA_COND     ? T.off_cond != BF_OFF_NONE && d.index < T.steps_max
         : d.field == BF_DELTA_DECISION ? T.off_decision != BF_OFF_NONE && d.index < T.steps_max
         : d.field == BF_DELTA_CHILD    ? T.off_child != BF_OFF_NONE && d.index < T.child_nibbles
                                        : true;
}

int bfh_batch_narrow(bfh_batch* b, uint32_t steps_max, uint32_t child_nibbles, uint32_t fields) {
  if (!b) return BF_EINVAL;
  bf_layout T;
  if (bf_layout_init(&T, steps_max, child_nibbles, fields) != BF_OK) { b->err = "steps_max out of range"; return BF_EINVAL; }
  const bf_layout F = b->L;
  if (T.steps_max > F.steps_max || (T.fields & ~F.fields) ||
      (F.off_child != BF_OFF_NONE && T.off_child != BF_OFF_NONE && T.child_nibbles > F.child_nibbles)) {
    b->err = "a narrow only shrinks the layout (steps_max, fields, child_nibbles)";
    return BF_EINVAL;
  }
  if (memcmp(&F, &T, sizeof T) == 0) return BF_OK;
  RunExtent x;   // the extent of bf_resident_narrow: every record of the mirror, the runs' Stories, the evaluated results
  for (uint32_t r = 0; r < b->cap; ++r) {
    const RunExtent e = run_extent(b, r, T);
    x.steps = std::max(x.steps, e.steps); x.child = std::max(x.child, e.child); x.fields |= e.fields;
  }
  if (x.steps > T.steps_max) { b->err = "the batch needs steps_max " + std::to_string(x.steps); return BF_EINVAL; }
  if (T.off_child != BF_OFF_NONE && x.child > T.child_nibbles) { b->err = "the batch needs child_nibbles " + std::to_string(x.child); return BF_EINVAL; }
  if (x.fields & ~placed(T)) { b->err = "the new layout drops an input field holding a non-default code"; return BF_EINVAL; }
  for (const bf_delta& d : b->deltas)   // a pending delta must still have its place: none is dropped
    if (!delta_fits(d, T)) { b->err = "a pending delta of run " + std::to_string(d.run) + " lies outside the new layout"; return BF_EINVAL; }
  HostRecords nr;
  if (!nr.alloc(b->ctx, (size_t)b->cap * T.state_stride, (size_t)b->cap * T.result_stride)) {
    b->err = "out of host memory";
    return BF_ENOMEM;
  }
  if (b->resident) {   // every run on the device first, then the device: it fails without changes, and so does the mirror
    int rc = flush_uploads(b);
    if (rc == BF_OK) {
      bf_extent e{};
      e.struct_size = sizeof e; e.n_runs = b->n;
      rc = bf_resident_narrow(b->ctx, b->handle, &T, &e);
    }
    if (rc != BF_OK) { b->err = bf_last_error(b->ctx); return rc; }
  }
  relay_records(b, nr, F, T);
  b->rec.swap(nr);
  b->L = T;
  return BF_OK;
}

// The mirror compacted once the n runs marked in `gone` have left it (retired or transferred) and the device has agreed, as
// bf_resident_retire compacts the device's records: the live runs of [m, N) move into the freed indices by the move rule of
// retire_moves.h and [m, N) is zeroed; the pending deltas of leaving runs go, those of moved runs apply at the new index (no two
// keys meet: a target has left); the moves go out to moves_from / moves_to.  -> the number of moves
static int compact_runs(bfh_batch* b, const std::vector<uint8_t>& gone, uint32_t n, uint32_t* moves_from, uint32_t* moves_to) {
  const uint32_t N = b->n, m = N - n;
  std::vector<uint32_t> to;
  const uint32_t n_moves = bf::retire_moves(gone, m, n, to);
  const size_t ss = b->L.state_stride, rs = b->L.result_stride;
  for (uint32_t i = 0; i < n; ++i) {
    if (to[i] == bf::kRetireNoMove) continue;
    memcpy(b->rec.state + to[i] * ss, b->rec.state + (m + i) * ss, ss);
    memcpy(b->rec.result + to[i] * rs, b->rec.result + (m + i) * rs, rs);
    b->story_of_run[to[i]] = b->story_of_run[m + i];
  }
  memset(b->rec.state + (size_t)m * ss, 0, (size_t)n * ss);
  memset(b->rec.result + (size_t)m * rs, 0, (size_t)n * rs);
  b->story_of_run.resize(m);
  rewrite_deltas(b, [&](bf_delta& d) {
    if (d.run < N && gone[d.run]) return false;
    if (d.run >= m) d.run = to[d.run - m];
    return true;
  });
  b->n = m;
  if (b->uploaded > m) b->uploaded = m;
  // a run moved from at or above `evaluated` takes its unevaluated record below it
  for (uint32_t i = 0; i < n; ++i)
    if (to[i] != bf::kRetireNoMove && m + i >= b->evaluated) b->evaluated = std::min(b->evaluated, to[i]);
  if (b->evaluated > m) b->evaluated = m;
  bf::write_moves(to, m, moves_from, moves_to);
  return (int)n_moves;
}

int bfh_batch_retire(bfh_batch* b, const uint32_t* runs, uint32_t n, uint32_t capacity, uint32_t* moves_from, uint32_t* moves_to) {
  if (!b) return BF_EINVAL;
  const uint32_t N = b->n;
  if (n && !runs) { b->err = "null runs"; return BF_EINVAL; }
  std::vector<uint8_t> gone(N, 0);
  for (uint32_t i = 0; i < n; ++i) {
    if (runs[i] >= N || gone[runs[i]]) { b->err = "runs[" + std::to_string(i) + "] is out of range or retired twice"; return BF_EINVAL; }
    gone[runs[i]] = 1;
  }
  const uint32_t m = N - n, cap = capacity ? capacity : b->cap;
  if (cap < m || cap > b->cap) { b->err = "capacity must be 0 or within [size - n, the current capacity]"; return BF_EINVAL; }
  if (n == 0 && cap == b->cap) return 0;
  const bf_layout& L = b->L;
  HostRecords nr;
  if (cap != b->cap && !nr.alloc(b->ctx, (size_t)cap * L.state_stride, (size_t)cap * L.result_stride)) {
    b->err = "out of host memory";
    return BF_ENOMEM;
  }
  if (b->resident) {   // every run on the device first, then the device: it fails without changes, and so does the mirror
    int rc = flush_uploads(b);
    if (rc == BF_OK) {
      bf_retire rt{};
      rt.struct_size = sizeof rt; rt.n_runs = N; rt.runs = runs; rt.n = n; rt.capacity = capacity;
      rc = bf_resident_retire(b->ctx, b->handle, &rt);
    }
    if (rc != BF_OK) { b->err = bf_last_error(b->ctx); return rc; }
  }
  const int n_moves = compact_runs(b, gone, n, moves_from, moves_to);
  if (nr.state) {
    memcpy(nr.state, b->rec.state, (size_t)m * L.state_stride);
    memcpy(nr.result, b->rec.result, (size_t)m * L.result_stride);
    b->rec.swap(nr);
    b->cap = cap;
  }
  return n_moves;
}

int bfh_batch_transfer(bfh_batch* src, bfh_batch* dst, const uint32_t* runs, uint32_t n, uint32_t* moves_from, uint32_t* moves_to) {
  if (!src || !dst) return BF_EINVAL;
  auto refuse = [&](const std::string& why) { src->err = why; dst->err = why; return BF_EINVAL; };
  if (src == dst) return refuse("a transfer from a batch to itself");
  if (src->ctx != dst->ctx || src->resident != dst->resident) return refuse("both batches must be of one ctx and in the same mode");
  const uint32_t N = src->n, D = dst->n;
  if (n && !runs) return refuse("null runs");
  if ((uint64_t)D + n > dst->cap) return refuse("the destination batch is full (reshape it first)");
  std::vector<uint8_t> gone(N, 0);
  for (uint32_t i = 0; i < n; ++i) {
    if (runs[i] >= N || gone[runs[i]]) return refuse("runs[" + std::to_string(i) + "] is out of range or moved twice");
    gone[runs[i]] = 1;
  }
  if (n == 0) return 0;
  // each run must fit the destination layout by bf_resident_narrow's test applied to it alone
  const bf_layout F = src->L, T = dst->L;
  for (uint32_t i = 0; i < n; ++i) {
    const RunExtent e = run_extent(src, runs[i], T);
    if (e.steps > T.steps_max || (T.off_child != BF_OFF_NONE && e.child > T.child_nibbles) || (e.fields & ~placed(T)))
      return refuse("runs[" + std::to_string(i) + "] (run " + std::to_string(runs[i]) + ") does not fit the destination layout");
  }
  for (const bf_delta& d : src->deltas)   // a pending delta of a moved run must still have its place: none is dropped
    if (d.run < N && gone[d.run] && !delta_fits(d, T))
      return refuse("a pending delta of run " + std::to_string(d.run) + " lies outside the destination layout");
  if (src->resident) {   // every run of both batches on the device first, then the device: it fails without changes, and so do the mirrors
    int rc = flush_uploads(src);
    if (rc == BF_OK) rc = flush_uploads(dst);
    if (rc == BF_OK) {
      bf_transfer t{};
      t.struct_size = sizeof t; t.src_n_runs = N; t.dst_n_runs = D; t.runs = runs; t.n = n;
      rc = bf_resident_transfer(src->ctx, src->handle, dst->handle, &t);
    }
    if (rc != BF_OK) { src->err = dst->err = bf_last_error(src->ctx); return rc; }
  }
  // arrivals: re-laid at the destination layout, in the order of runs[]
  for (uint32_t i = 0; i < n; ++i) {
    relay_record(src->rec, runs[i], F, dst->rec, D + i, T);
    dst->story_of_run.push_back(src->story_of_run[runs[i]]);
  }
  // pending deltas of moved runs go to the destination's log under their new index (no key meets one there: every index from
  // D on was free); an arrival is on the device in resident mode, and its evaluated results travelled with it
  std::vector<uint32_t> arrival(N, UINT32_MAX);
  for (uint32_t i = 0; i < n; ++i) arrival[runs[i]] = D + i;
  for (const bf_delta& d0 : src->deltas) {
    if (d0.run >= N || !gone[d0.run]) continue;
    bf_delta d = d0;
    d.run = arrival[d0.run];
    dst->delta_at[delta_key(d.run, d.field, d.index)] = (uint32_t)dst->deltas.size();
    dst->deltas.push_back(d);
  }
  const bool all_evaluated = dst->evaluated == D && std::all_of(runs, runs + n, [&](uint32_t r) { return r < src->evaluated; });
  dst->n = D + n;
  if (dst->resident) dst->uploaded = dst->n;
  if (all_evaluated) dst->evaluated = dst->n;
  return compact_runs(src, gone, n, moves_from, moves_to);   // after the arrivals, which read the source's records
}

int bfh_batch_set_resident(bfh_batch* b, int on) {
  if (!b) return BF_EINVAL;
  if (!b->ctx) { b->err = "batch was created without a device context"; return BF_ENODEV; }
  if ((on != 0) == b->resident) return BF_OK;
  if (on) {
    const int rc = bf_resident_create(b->ctx, &b->L, b->cap, &b->handle);
    if (rc != BF_OK) { b->err = bf_last_error(b->ctx); return rc; }
    b->resident = true; b->uploaded = 0;
  } else {
    bf_resident_destroy(b->ctx, b->handle);
    b->resident = false; b->uploaded = 0;
    b->deltas.clear(); b->delta_at.clear();
  }
  return BF_OK;
}
int bfh_batch_traffic(const bfh_batch* b, uint64_t* full_record_bytes, uint64_t* delta_bytes, uint32_t* pending_deltas) {
  if (!b) return BF_EINVAL;
  if (full_record_bytes) *full_record_bytes = b->full_bytes_sent;
  if (delta_bytes) *delta_bytes = b->delta_bytes_sent;
  if (pending_deltas) *pending_deltas = (uint32_t)b->deltas.size();
  return BF_OK;
}

uint32_t bfh_run_summary(const bfh_batch* b, uint32_t run) {
  if (!b || run >= b->n) return 0xFFFFFFFFu;
  return reinterpret_cast<const bf_result_header*>(b->rec.result + (size_t)run * b->L.result_stride)->summary;
}
static int mask_list(const bfh_batch* b, uint32_t run, uint32_t off, uint32_t* out, uint32_t cap) {
  if (!b || run >= b->n || off == BF_OFF_NONE) return BF_EINVAL;
  const uint32_t* m = reinterpret_cast<const uint32_t*>(b->rec.result + (size_t)run * b->L.result_stride + off);
  const uint32_t S = (uint32_t)b->story_of_run[run]->flags.size();
  int n = 0;
  for (uint32_t i = 0; i < S; ++i)
    if ((m[i >> 5] >> (i & 31u)) & 1u) {
      if (out && (uint32_t)n < cap) out[n] = i;
      ++n;
    }
  return n;
}
int bfh_run_ready(const bfh_batch* b, uint32_t run, uint32_t* out, uint32_t cap) { return mask_list(b, run, b ? b->L.off_ready : 0, out, cap); }
int bfh_run_skipped(const bfh_batch* b, uint32_t run, uint32_t* out, uint32_t cap) { return mask_list(b, run, b ? b->L.off_skip : 0, out, cap); }
int bfh_run_failed(const bfh_batch* b, uint32_t run, uint32_t* out, uint32_t cap) { return mask_list(b, run, b ? b->L.off_fail : BF_OFF_NONE, out, cap); }
int bfh_run_needs_cond(const bfh_batch* b, uint32_t run, uint32_t* out, uint32_t cap) { return mask_list(b, run, b ? b->L.off_needs_cond : BF_OFF_NONE, out, cap); }
int bfh_run_phase_out(const bfh_batch* b, uint32_t run, uint32_t step) {
  if (!b || run >= b->n || b->L.off_phase_out == BF_OFF_NONE || step >= b->story_of_run[run]->flags.size()) return -1;
  return get_code(b->rec.result + (size_t)run * b->L.result_stride + b->L.off_phase_out, b->L.words, 4, step);
}
int bfh_run_skip_reason(const bfh_batch* b, uint32_t run, uint32_t step, char* out, size_t cap) {
  if (!b || run >= b->n || !out || !cap) return BF_EINVAL;
  const bfh_story* st = b->story_of_run[run];
  if (step >= st->flags.size()) return BF_EINVAL;
  const uint8_t* rrec = b->rec.result + (size_t)run * b->L.result_stride;
  std::string msg = "Skipped due to 'if' condition";  // dag.go:2831
  bool by_dep = false;
  if (b->L.off_skip_dep != BF_OFF_NONE)
    by_dep = (reinterpret_cast<const uint32_t*>(rrec + b->L.off_skip_dep)[step >> 5] >> (step & 31u)) & 1u;
  if (by_dep) {
    msg = "Skipped due to failed dependency: ";  // dag.go:2737; the named dep = first failed one in CSR order
    const uint8_t* ph = b->L.off_phase_out != BF_OFF_NONE ? rrec + b->L.off_phase_out
                                                         : b->rec.state + (size_t)run * b->L.state_stride + b->L.off_phase;
    for (uint32_t e = st->row_ptr[step]; e < st->row_ptr[step + 1]; ++e) {
      const uint32_t d = st->col_idx[e];
      const int p = get_code(ph, b->L.words, 4, d);
      const bool term = (BF_LUT_TERMINAL >> p) & 1u;
      const bool compl_ = ((BF_LUT_COMPLETED0 >> p) & 1u) || (term && (st->flags[d] & BF_SF_ALLOW_FAILURE));
      // a dep set Failed earlier in this same pass (dag.go:2745) counts even with allowFailure: `completed` is stale
      const bool failed_now = b->L.off_fail != BF_OFF_NONE && d < step &&
                              ((reinterpret_cast<const uint32_t*>(rrec + b->L.off_fail)[d >> 5] >> (d & 31u)) & 1u);
      if ((term && !compl_) || failed_now) { msg += st->defs[st->order[d]].name; break; }
    }
  }
  strncpy(out, msg.c_str(), cap - 1);
  out[cap - 1] = 0;
  return BF_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------ limiters (rows a9 / f4)
namespace {
std::string normalize_queue(const char* name) {  // scheduling.go:21-27: TrimSpace + ToLower
  std::string q = name ? name : "";
  size_t a = 0, b = q.size();
  while (a < b && is_space(q[a])) ++a;
  while (b > a && is_space(q[b - 1])) --b;
  q = q.substr(a, b - a);
  for (char& c : q) if (c >= 'A' && c <= 'Z') c = (char)(c - 'A' + 'a');
  return q;
}
int phase_code_plain(const char* phase) { return phase_code_of(phase ? phase : "", ""); }
}  // namespace

struct bfh_sched {
  bfh_batch* batch = nullptr;
  std::string err;
  int32_t global_limit = 0;
  uint32_t global_base = 0;
  std::vector<std::string> queue_names;
  std::unordered_map<std::string, uint32_t> queue_key;
  std::vector<int32_t> queue_limit, queue_default_prio, queue_aging;
  std::vector<uint32_t> queue_base;
  std::unordered_map<std::string, uint32_t> story_key;   // "namespace/name"
  std::vector<int32_t> story_limit;
  std::vector<uint32_t> story_base;
  std::vector<bf_sched_run> runs;
  // results
  std::vector<uint8_t> records;
  std::vector<uint32_t> story_running, queue_running;
  std::vector<int32_t> queue_maxprio;
  uint32_t global_running = 0;
  bool applied = false;

  uint32_t queue_of(const std::string& normalized) {  // "" -> default (queueLabelValue, scheduling.go:29-35)
    const std::string n = normalized.empty() ? "default" : normalized;
    auto it = queue_key.find(n);
    if (it != queue_key.end()) return it->second;
    const uint32_t k = (uint32_t)queue_names.size();
    queue_key[n] = k;
    queue_names.push_back(n);
    queue_limit.push_back(0); queue_default_prio.push_back(0); queue_aging.push_back(0); queue_base.push_back(0);
    return k;
  }
  uint32_t story_of(const char* ns, const char* name) {
    const std::string k = std::string(ns ? ns : "") + "/" + (name ? name : "");
    auto it = story_key.find(k);
    if (it != story_key.end()) return it->second;
    const uint32_t id = (uint32_t)story_limit.size();
    story_key[k] = id;
    story_limit.push_back(0); story_base.push_back(0);
    return id;
  }
};

extern "C" {

bfh_sched* bfh_sched_new(bfh_batch* batch) {
  if (!batch) return nullptr;
  bfh_sched* s = new (std::nothrow) bfh_sched();
  if (!s) return nullptr;
  s->batch = batch;
  // the default scheduling config: queue "default" ages every 60 s (internal/config/controller_config.go:731-739)
  const uint32_t k = s->queue_of("default");
  s->queue_aging[k] = 60;
  return s;
}
void bfh_sched_free(bfh_sched* s) { delete s; }
const char* bfh_sched_error(const bfh_sched* s) { return s ? s->err.c_str() : "null sched"; }

int bfh_sched_set_global(bfh_sched* s, int32_t limit, uint32_t base) {
  if (!s) return BF_EINVAL;
  s->global_limit = limit; s->global_base = base;
  return BF_OK;
}
int bfh_sched_set_queue(bfh_sched* s, const char* name, int32_t concurrency, int32_t default_priority, int32_t aging, uint32_t base) {
  if (!s) return BF_EINVAL;
  const uint32_t k = s->queue_of(normalize_queue(name));
  s->queue_limit[k] = concurrency; s->queue_default_prio[k] = default_priority; s->queue_aging[k] = aging; s->queue_base[k] = base;
  return (int)k;
}
int bfh_sched_set_story_base(bfh_sched* s, const char* ns, const char* name, uint32_t base) {
  if (!s) return BF_EINVAL;
  const uint32_t k = s->story_of(ns, name);
  s->story_base[k] = base;
  return (int)k;
}
int bfh_sched_set_run(bfh_sched* s, uint32_t run, const char* ns, const char* name, int32_t story_concurrency, const char* policy_queue,
                      int has_priority, int32_t policy_priority, const char* run_phase, int64_t queued_since_ns, int64_t now_ns) {
  if (!s || run >= s->batch->n) { if (s) s->err = "run index out of range"; return BF_EINVAL; }
  if (s->runs.size() < s->batch->n) s->runs.resize(s->batch->n);
  // resolveSchedulingDecision, scheduling.go:130-163 (no fallback decision on this path: dag.go:1805 passes nil)
  const std::string sq = normalize_queue(policy_queue);
  const uint32_t qk = s->queue_of(sq);
  int32_t prio;
  if (has_priority) prio = policy_priority;
  else prio = s->queue_default_prio[qk];  // both remaining cases read queueDefaultPriority of the decided queue
  const uint32_t sk = s->story_of(ns, name);
  s->story_limit[sk] = story_concurrency > 0 ? story_concurrency : 0;  // storyConcurrencyLimit, dag.go:1863-1868
  bf_sched_run& r = s->runs[run];
  memset(&r, 0, sizeof r);
  r.story_key = sk; r.queue_key = qk; r.priority = prio;
  r.run_phase = (uint32_t)phase_code_plain(run_phase);
  if (queued_since_ns < 0) r.queued_elapsed_s = BF_SCHED_NONE;
  else {
    const int64_t el_ns = now_ns - queued_since_ns;  // elapsed <= 0 -> base priority (dag.go:1952-1955)
    const int64_t el = el_ns <= 0 ? 0 : el_ns / 1000000000ll;  // int32(elapsed.Seconds())
    r.queued_elapsed_s = el > 0x7FFFFFFF ? 0x7FFFFFFFu : (uint32_t)el;
  }
  s->applied = false;
  return BF_OK;
}
const bf_sched_run* bfh_sched_runs(const bfh_sched* s) { return s && !s->runs.empty() ? s->runs.data() : nullptr; }
int bfh_sched_tables(const bfh_sched* s, bf_sched_tables* t) {
  if (!s || !t) return BF_EINVAL;
  memset(t, 0, sizeof *t);
  t->struct_size = sizeof *t;
  t->n_stories = (uint32_t)s->story_limit.size(); t->n_queues = (uint32_t)s->queue_limit.size();
  t->global_limit = s->global_limit; t->global_running_base = s->global_base;
  t->story_limit = s->story_limit.data(); t->story_running_base = s->story_base.data();
  t->queue_limit = s->queue_limit.data(); t->queue_aging_s = s->queue_aging.data(); t->queue_running_base = s->queue_base.data();
  return BF_OK;
}
const char* bfh_sched_queue_name(const bfh_sched* s, uint32_t k) { return s && k < s->queue_names.size() ? s->queue_names[k].c_str() : ""; }

int bfh_sched_apply(bfh_sched* s) {
  if (!s) return BF_EINVAL;
  bfh_batch* b = s->batch;
  if (!b->ctx) { s->err = "batch was created without a device context"; return BF_ENODEV; }
  if (s->runs.size() != b->n) { s->err = "bfh_sched_set_run was not called for every run of the batch"; return BF_EINVAL; }
  bf_sched_tables t;
  bfh_sched_tables(s, &t);
  const uint32_t stride = BF_SCHED_STRIDE(b->L.words);
  s->records.assign((size_t)b->n * stride, 0);
  s->story_running.assign(t.n_stories, 0); s->queue_running.assign(t.n_queues, 0); s->queue_maxprio.assign(t.n_queues, 0);
  bf_sched_out out{};
  out.struct_size = sizeof out;
  out.records = s->records.data();
  out.story_running = s->story_running.data(); out.queue_running = s->queue_running.data();
  out.queue_max_priority = s->queue_maxprio.data(); out.global_running = &s->global_running;
  bf_batch bb{};
  bb.struct_size = sizeof(bf_batch);
  bb.n_runs = b->n; bb.layout = b->L;
  const int rc = bf_schedule(b->ctx, &bb, s->runs.data(), &t, &out);
  if (rc != BF_OK) { s->err = bf_last_error(b->ctx); return rc; }
  s->applied = true;
  return BF_OK;
}

int bfh_sched_steps(const bfh_sched* s, uint32_t run, int which, uint32_t* out, uint32_t cap) {
  if (!s || !s->applied || run >= s->batch->n || which < 0 || which > 2) return BF_EINVAL;
  const uint32_t W = s->batch->L.words, stride = BF_SCHED_STRIDE(W);
  const uint32_t* m = reinterpret_cast<const uint32_t*>(s->records.data() + (size_t)run * stride + 16) + (size_t)which * W;
  const uint32_t S = (uint32_t)s->batch->story_of_run[run]->flags.size();
  int n = 0;
  for (uint32_t i = 0; i < S; ++i)
    if ((m[i >> 5] >> (i & 31u)) & 1u) {
      if (out && (uint32_t)n < cap) out[n] = i;
      ++n;
    }
  return n;
}

int bfh_sched_format_message(int reason, uint32_t running, int32_t limit, char* out, size_t cap) {
  if (!out || !cap) return BF_EINVAL;
  const char* prefix;
  switch (reason) {
    case 0: prefix = "Queued due to story concurrency limit"; break;        // dag.go:104, 1797
    case BF_QUEUED_GLOBAL: prefix = "Queued due to global concurrency limit"; break;  // :106, 1850
    case BF_QUEUED_QUEUE: prefix = "Queued due to queue concurrency limit"; break;    // :105, 1852
    case BF_QUEUED_PRIORITY: snprintf(out, cap, "Queued due to higher-priority work"); return BF_OK;  // :107, 1944
    case BF_QUEUED_OTHER: snprintf(out, cap, "Queued due to scheduling limits"); return BF_OK;        // :1854
    default: out[0] = 0; return BF_OK;
  }
  snprintf(out, cap, "%s (%u running, limit %d)", prefix, running, limit);
  return BF_OK;
}

int bfh_sched_message(const bfh_sched* s, uint32_t run, int which, char* out, size_t cap) {
  if (!s || !s->applied || run >= s->batch->n || !out || !cap || (which != 1 && which != 2)) return BF_EINVAL;
  const uint32_t stride = BF_SCHED_STRIDE(s->batch->L.words);
  const bf_sched_header* h = reinterpret_cast<const bf_sched_header*>(s->records.data() + (size_t)run * stride);
  const bf_sched_run& r = s->runs[run];
  out[0] = 0;
  if (which == 1) {
    if (h->n_queued_story) return bfh_sched_format_message(0, s->story_running[r.story_key], s->story_limit[r.story_key], out, cap);
    return BF_OK;
  }
  if (!h->n_queued_sched) return BF_OK;
  if (h->sched_reason == BF_QUEUED_GLOBAL) return bfh_sched_format_message(BF_QUEUED_GLOBAL, s->global_running, s->global_limit, out, cap);
  if (h->sched_reason == BF_QUEUED_QUEUE) return bfh_sched_format_message(BF_QUEUED_QUEUE, s->queue_running[r.queue_key], s->queue_limit[r.queue_key], out, cap);
  return bfh_sched_format_message((int)h->sched_reason, 0, 0, out, cap);
}

}  // extern "C"
