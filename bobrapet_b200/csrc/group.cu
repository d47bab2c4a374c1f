// group.cu — device groups of the C ABI (include/bobrafrontier.h, row e): the bf_group_* entry points.
//
// One process, G devices: a ctx per device, an NCCL communicator over them (libnccl.so.2 via dlopen, so the library
// loads on hosts without NCCL and single-device users never touch it), one worker thread per shard for the duration
// of a call.  The data path has no collective; the one exchange of a pass is the all-gather of the 32-byte counts.
#include <dlfcn.h>
#include <nccl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <new>
#include <thread>

#include "ctx.h"

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
      rcs[k] = bf::eval_host(c, &sb, nullptr);
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
  auto between = [](void* user, const bf::SchedTotals& tt, cudaStream_t s) -> int {
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
    if (count == 0) g->ctx[k]->snap = {true, 0, b->layout, nullptr, nullptr};   // an empty shard still takes part in the reductions
    rcs[k] = bf::schedule_host(g->ctx[k], &sb, runs ? runs + first : nullptr, t, &so, between, &h, k == 0);
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
