/*
 * gtnb_capi.cu -- the C-ABI entry points of include/gtn_b200.h: context,
 * memory helpers, host-side packing (levelisation) of generic graphs, the
 * host half of the frame-synchronous composition, and thin wrappers that
 * launch the sm_90a kernels in k_*.cu.
 *
 * No CPU fallback lives here: every compute entry point ends in a kernel
 * launch on the context's stream.
 */
#include <algorithm>
#include <thread>
#include <cmath>
#include <cstring>
#include <limits>
#include <mutex>
#include <queue>
#include <set>
#include <utility>

#include "gtnb_internal.h"

using namespace gtnb;

namespace {
thread_local std::string tlsError;
}

namespace gtnb {

int fail(gtnb_ctx* ctx, int code, const std::string& msg) {
  if (ctx)
    ctx->err = msg;
  else
    tlsError = msg;
  return code;
}

int stage_begin(gtnb_ctx* ctx) {
  if (!ctx->stage_ev) GTNB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->stage_ev, cudaEventDisableTiming));
  if (ctx->stage_pending) GTNB_CUDA(ctx, cudaEventSynchronize(ctx->stage_ev));
  ctx->stage_pending = false;
  ctx->stage_used = 0;
  return GTNB_OK;
}

int stage_upload(gtnb_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes) {
  if (bytes == 0) return GTNB_OK;
  const size_t need = ctx->stage_used + ((bytes + 255) & ~(size_t)255);
  if (need > ctx->stage_bytes) {
    // copies already issued from the old buffer must finish before it is released
    GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    size_t nb = std::max(need * 2, (size_t)1 << 20);
    unsigned char* fresh = nullptr;
    GTNB_CUDA(ctx, cudaMallocHost((void**)&fresh, nb));
    if (ctx->stage) cudaFreeHost(ctx->stage);
    ctx->stage = fresh;
    ctx->stage_bytes = nb;
    ctx->stage_used = 0;
  }
  unsigned char* p = ctx->stage + ctx->stage_used;
  std::memcpy(p, src_host, bytes);
  ctx->stage_used += (bytes + 255) & ~(size_t)255;
  GTNB_CUDA(ctx, cudaMemcpyAsync(dst_dev, p, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return GTNB_OK;
}

int stage_reserve(gtnb_ctx* ctx, size_t bytes) {
  const size_t need = ctx->stage_used + bytes;
  if (need <= ctx->stage_bytes) return GTNB_OK;
  GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // copies already issued from the old buffer
  size_t nb = std::max(need * 2, (size_t)1 << 20);
  unsigned char* fresh = nullptr;
  GTNB_CUDA(ctx, cudaMallocHost((void**)&fresh, nb));
  if (ctx->stage_used) std::memcpy(fresh, ctx->stage, ctx->stage_used);
  if (ctx->stage) cudaFreeHost(ctx->stage);
  ctx->stage = fresh;
  ctx->stage_bytes = nb;
  return GTNB_OK;
}

int stage_place(gtnb_ctx* ctx, const void* src_host, size_t bytes, void** where) {
  const size_t sz = (bytes + 255) & ~(size_t)255;
  if (ctx->stage_used + sz > ctx->stage_bytes)
    return fail(ctx, GTNB_ERR_LOGIC, "stage_place: stage_reserve the pass first (placed addresses must stay valid)");
  unsigned char* p = ctx->stage + ctx->stage_used;
  if (bytes) std::memcpy(p, src_host, bytes);
  ctx->stage_used += sz;
  *where = p;
  return GTNB_OK;
}

int stage_end(gtnb_ctx* ctx) {
  GTNB_CUDA(ctx, cudaEventRecord(ctx->stage_ev, ctx->stream));
  ctx->stage_pending = true;
  return GTNB_OK;
}

int readback_reserve(gtnb_ctx* ctx, size_t bytes) {
  if (bytes <= ctx->readback_bytes) return GTNB_OK;
  if (ctx->readback) cudaFreeHost(ctx->readback);
  ctx->readback = nullptr;
  ctx->readback_bytes = 0;
  GTNB_CUDA(ctx, cudaMallocHost((void**)&ctx->readback, bytes * 2));
  ctx->readback_bytes = bytes * 2;
  return GTNB_OK;
}

int cuda_fail(gtnb_ctx* ctx, cudaError_t e, const char* what, const char* file, int line) {
  char buf[512];
  snprintf(buf, sizeof(buf), "[gtn_b200] CUDA error %d (%s) in %s at %s:%d",
           (int)e, cudaGetErrorString(e), what, file, line);
  return fail(ctx, GTNB_ERR_RUNTIME, buf);
}

int ensure_side_streams(gtnb_ctx* ctx, int n_streams, int n_events) {
  if (!ctx->copy_stream) {
    GTNB_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
    GTNB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
    GTNB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
  }
  while ((int)ctx->side_streams.size() < n_streams) {
    cudaStream_t s;
    GTNB_CUDA(ctx, cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    ctx->side_streams.push_back(s);
  }
  while ((int)ctx->side_events.size() < n_events) {
    cudaEvent_t e;
    GTNB_CUDA(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    ctx->side_events.push_back(e);
  }
  return GTNB_OK;
}

int ensure_max_smem(gtnb_ctx* ctx, const void* kernel) {
  static std::mutex mu;
  static std::set<std::pair<int, const void*>> done;
  std::lock_guard<std::mutex> l(mu);
  const auto key = std::make_pair(ctx->device, kernel);
  if (done.count(key)) return GTNB_OK;
  GTNB_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynamicSmem));
  done.insert(key);
  return GTNB_OK;
}

} // namespace gtnb

extern "C" {

int gtnb_version(void) {
  return GTNB_VERSION;
}

int gtnb_ctx_create(int device, void* cuda_stream, gtnb_ctx** out) {
  if (!out) return fail(nullptr, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctx_create: out is NULL");
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) {
    return fail(nullptr, GTNB_ERR_RUNTIME,
                std::string("[gtn_b200] no usable CUDA device (there is no CPU fallback): ") +
                    cudaGetErrorString(e));
  }
  if (device < 0 || device >= n)
    return fail(nullptr, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctx_create: bad device index");
  gtnb_ctx* ctx = new gtnb_ctx();
  ctx->device = device;
  if ((e = cudaSetDevice(device)) != cudaSuccess) {
    int rc = cuda_fail(nullptr, e, "cudaSetDevice", __FILE__, __LINE__);
    delete ctx;
    return rc;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) {
    ctx->sm_count = prop.multiProcessorCount;
    ctx->total_mem = prop.totalGlobalMem;
  }
  if (cuda_stream) {
    ctx->stream = (cudaStream_t)cuda_stream;
  } else {
    if ((e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess) {
      int rc = cuda_fail(nullptr, e, "cudaStreamCreate", __FILE__, __LINE__);
      delete ctx;
      return rc;
    }
    ctx->own_stream = true;
  }
  cudaEventCreate(&ctx->ev0);
  cudaEventCreate(&ctx->ev1);
  // keep freed blocks cached in the stream-ordered pool
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t thr = UINT64_MAX;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  *out = ctx;
  return GTNB_OK;
}

void gtnb_ctx_destroy(gtnb_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->flush_buf) cudaFree(ctx->flush_buf);
  if (ctx->arena) cudaFree(ctx->arena);
  if (ctx->stage) cudaFreeHost(ctx->stage);
  if (ctx->readback) cudaFreeHost(ctx->readback);
  if (ctx->stage_ev) cudaEventDestroy(ctx->stage_ev);
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  for (auto s : ctx->side_streams) cudaStreamDestroy(s);
  for (auto e : ctx->side_events) cudaEventDestroy(e);
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
  if (ctx->ev0) cudaEventDestroy(ctx->ev0);
  if (ctx->ev1) cudaEventDestroy(ctx->ev1);
  for (auto& pe : ctx->prof) {
    cudaEventDestroy(pe.a);
    cudaEventDestroy(pe.b);
  }
  for (auto e : ctx->ev_pool) cudaEventDestroy(e);
  if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

const char* gtnb_last_error(const gtnb_ctx* ctx) {
  return ctx ? ctx->err.c_str() : tlsError.c_str();
}

int gtnb_ctx_synchronize(gtnb_ctx* ctx) {
  GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return GTNB_OK;
}

void* gtnb_ctx_stream(gtnb_ctx* ctx) {
  return (void*)ctx->stream;
}

int gtnb_ctx_device(const gtnb_ctx* ctx) {
  return ctx ? ctx->device : -1;
}

int64_t gtnb_ctx_launch_count(const gtnb_ctx* ctx) {
  return ctx->launches;
}

int gtnb_device_alloc(gtnb_ctx* ctx, size_t bytes, void** out) {
  // stream-ordered: cudaMalloc / cudaFree synchronise the whole device and would serialise the
  // per-thread streams of the gtn:: C++ layer
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  GTNB_CUDA(ctx, cudaMallocAsync(out, bytes ? bytes : 16, ctx->stream));
  return GTNB_OK;
}
int gtnb_device_free(gtnb_ctx* ctx, void* p) {
  GTNB_CUDA(ctx, cudaFreeAsync(p, ctx->stream));
  return GTNB_OK;
}
int gtnb_host_alloc(gtnb_ctx* ctx, size_t bytes, void** out) {
  GTNB_CUDA(ctx, cudaMallocHost(out, bytes ? bytes : 16));
  return GTNB_OK;
}
int gtnb_host_free(gtnb_ctx* ctx, void* p) {
  GTNB_CUDA(ctx, cudaFreeHost(p));
  return GTNB_OK;
}
int gtnb_memcpy_h2d(gtnb_ctx* ctx, void* dst, const void* src, size_t bytes) {
  GTNB_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return GTNB_OK;
}
int gtnb_memcpy_d2h(gtnb_ctx* ctx, void* dst, const void* src, size_t bytes) {
  GTNB_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  return GTNB_OK;
}
int gtnb_memset(gtnb_ctx* ctx, void* dst, int value, size_t bytes) {
  GTNB_CUDA(ctx, cudaMemsetAsync(dst, value, bytes, ctx->stream));
  return GTNB_OK;
}
int gtnb_timer_start(gtnb_ctx* ctx) {
  GTNB_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
  return GTNB_OK;
}
int gtnb_timer_stop(gtnb_ctx* ctx, float* ms) {
  GTNB_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
  GTNB_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
  GTNB_CUDA(ctx, cudaEventElapsedTime(ms, ctx->ev0, ctx->ev1));
  return GTNB_OK;
}
int gtnb_ctx_set_flag(gtnb_ctx* ctx, const char* name, int value) {
  if (ctx && name && std::string(name) == "staged") {
    ctx->use_staged = value != 0;
    return GTNB_OK;
  }
  if (ctx && name && std::string(name) == "implicit") {
    ctx->use_implicit = value != 0;
    return GTNB_OK;
  }
  if (ctx && name && std::string(name) == "exact_ties") {
    ctx->exact_ties = value != 0;
    return GTNB_OK;
  }
  if (ctx && name && std::string(name) == "bidir") {
    ctx->use_bidir = value < 0 ? kBidirDefault : value != 0; // -1: back to the default
    return GTNB_OK;
  }
  if (ctx && name && std::string(name) == "bidir_mode") {
    if (value < -1 || value > 1) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctx_set_flag: bidir_mode is -1 (default), 0 or 1");
    ctx->bidir_mode = value;
    return GTNB_OK;
  }
  if (ctx && name && std::string(name) == "sparse_cluster") {
    if (value != 0 && value != 1 && value != 2 && value != 4 && value != 8)
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctx_set_flag: sparse_cluster is 0 (default), 1, 2, 4 or 8");
    ctx->sparse_cluster = value;
    return GTNB_OK;
  }
  return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctx_set_flag: unknown flag");
}

int gtnb_profile_enable(gtnb_ctx* ctx, int on) {
  ctx->profiling = on != 0;
  return GTNB_OK;
}

const char* gtnb_profile_read(gtnb_ctx* ctx) {
  // "name count total_ms\n" per kernel name, in first-launch order; clears the log
  cudaStreamSynchronize(ctx->stream);
  std::vector<std::string> names;
  std::vector<int> counts;
  std::vector<double> ms;
  for (auto& pe : ctx->prof) {
    float t = 0.f;
    cudaEventElapsedTime(&t, pe.a, pe.b);
    size_t i = 0;
    for (; i < names.size(); i++)
      if (names[i] == pe.name) break;
    if (i == names.size()) {
      names.push_back(pe.name);
      counts.push_back(0);
      ms.push_back(0.0);
    }
    counts[i]++;
    ms[i] += t;
    ctx->ev_pool.push_back(pe.a);
    ctx->ev_pool.push_back(pe.b);
  }
  ctx->prof.clear();
  ctx->prof_text.clear();
  char buf[256];
  for (size_t i = 0; i < names.size(); i++) {
    snprintf(buf, sizeof(buf), "%s %d %.6f\n", names[i].c_str(), counts[i], ms[i]);
    ctx->prof_text += buf;
  }
  return ctx->prof_text.c_str();
}

int gtnb_flush_l2(gtnb_ctx* ctx) {
  if (!ctx->flush_buf) {
    ctx->flush_bytes = (size_t)256 << 20; // over 5x the 50 MB L2 of an H100
    GTNB_CUDA(ctx, cudaMalloc(&ctx->flush_buf, ctx->flush_bytes));
  }
  GTNB_CUDA(ctx, cudaMemsetAsync(ctx->flush_buf, 0, ctx->flush_bytes, ctx->stream));
  return GTNB_OK;
}

} // extern "C"

/* ------------------------------------------------------------------ */
/* host-side adjacency helpers                                         */
/* ------------------------------------------------------------------ */

namespace {

struct Adj {
  std::vector<int32_t> in_ptr, in_arcs, out_ptr, out_arcs, start, accept;
};

} // namespace

int gtnb::validate_view(gtnb_ctx* ctx, const gtnb_graph_view& v) {
  if (v.num_nodes < 0 || v.num_arcs < 0)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "graph view: negative size");
  if (v.num_nodes > 0 && !v.node_flags)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "graph view: node_flags is NULL");
  if (v.num_arcs > 0 && (!v.arc_src || !v.arc_dst || !v.arc_ilabel || !v.arc_olabel))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "graph view: arc arrays are NULL");
  for (int a = 0; a < v.num_arcs; a++) {
    if (v.arc_src[a] < 0 || v.arc_src[a] >= v.num_nodes || v.arc_dst[a] < 0 ||
        v.arc_dst[a] >= v.num_nodes)
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "graph view: arc endpoint out of range");
  }
  return GTNB_OK;
}

namespace {

void build_adj(const gtnb_graph_view& v, Adj& adj) {
  int N = v.num_nodes, A = v.num_arcs;
  if (v.in_ptr && v.in_arcs) {
    adj.in_ptr.assign(v.in_ptr, v.in_ptr + N + 1);
    adj.in_arcs.assign(v.in_arcs, v.in_arcs + A);
  } else {
    adj.in_ptr.assign(N + 1, 0);
    for (int a = 0; a < A; a++) adj.in_ptr[v.arc_dst[a] + 1]++;
    for (int n = 0; n < N; n++) adj.in_ptr[n + 1] += adj.in_ptr[n];
    adj.in_arcs.resize(A);
    std::vector<int32_t> pos(adj.in_ptr.begin(), adj.in_ptr.end() - 1);
    for (int a = 0; a < A; a++) adj.in_arcs[pos[v.arc_dst[a]]++] = a;
  }
  if (v.out_ptr && v.out_arcs) {
    adj.out_ptr.assign(v.out_ptr, v.out_ptr + N + 1);
    adj.out_arcs.assign(v.out_arcs, v.out_arcs + A);
  } else {
    adj.out_ptr.assign(N + 1, 0);
    for (int a = 0; a < A; a++) adj.out_ptr[v.arc_src[a] + 1]++;
    for (int n = 0; n < N; n++) adj.out_ptr[n + 1] += adj.out_ptr[n];
    adj.out_arcs.resize(A);
    std::vector<int32_t> pos(adj.out_ptr.begin(), adj.out_ptr.end() - 1);
    for (int a = 0; a < A; a++) adj.out_arcs[pos[v.arc_src[a]]++] = a;
  }
  if (v.start) {
    adj.start.assign(v.start, v.start + v.num_start);
  } else {
    for (int n = 0; n < N; n++)
      if (v.node_flags[n] & 1) adj.start.push_back(n);
  }
  if (v.accept) {
    adj.accept.assign(v.accept, v.accept + v.num_accept);
  } else {
    for (int n = 0; n < N; n++)
      if (v.node_flags[n] & 2) adj.accept.push_back(n);
  }
}

/* One graph levelised for the device (see GraphMeta for the layout). */
struct PackedGraph {
  int N = 0, A = 0, L = 0, LB = 0, status = GTNB_OK;
  bool level_local = true;
  int max_lvl_nodes = 0, max_lvl_arcs = 0;
  std::vector<int32_t> lvl_node_ptr, lvl_arc_ptr, src, acc, node_orig, arc_orig, relax_rank;
  std::vector<int32_t> blvl_ptr, bnodes;
  std::vector<uint32_t> row_ptr;
  std::vector<float> w;
};

/*
 * Forward schedule = the reference's Kahn sweep (shortest.cpp:92-100,118-145),
 * backward schedule = its reverse sweep (shortest.cpp:45-60,62-80).
 */
void pack_one(const gtnb_graph_view& v, const Adj& adj, PackedGraph& p) {
  const int N = v.num_nodes, A = v.num_arcs;
  std::vector<int32_t> deg(N), level(N, 0), pop(N, -1), rank(A, -1);
  for (int n = 0; n < N; n++) deg[n] = adj.in_ptr[n + 1] - adj.in_ptr[n];
  std::vector<int32_t> order;
  order.reserve(N);
  size_t qh = 0;
  for (int n : adj.start)
    if (deg[n] == 0 && pop[n] < 0) {
      // a node listed twice in start() would be pushed twice by the
      // reference; Graph::addNode never does that.
      pop[n] = (int)order.size();
      order.push_back(n);
    }
  int counter = 0;
  while (qh < order.size()) {
    int n = order[qh++];
    for (int k = adj.out_ptr[n]; k < adj.out_ptr[n + 1]; k++) {
      int a = adj.out_arcs[k];
      int dn = v.arc_dst[a];
      rank[a] = counter++;
      level[dn] = std::max(level[dn], level[n] + 1);
      if (--deg[dn] == 0) {
        pop[dn] = (int)order.size();
        order.push_back(dn);
      }
    }
  }
  for (int n : adj.accept)
    if (deg[n] > 0) p.status = GTNB_ERR_INVALID_ARGUMENT;

  // device node order: (level, pop order); then never-scheduled accept nodes
  std::vector<int32_t> sched(order);
  std::stable_sort(sched.begin(), sched.end(), [&](int a, int b) { return level[a] < level[b]; });
  std::vector<int32_t> new_id(N, -1);
  p.node_orig.clear();
  for (int n : sched) {
    new_id[n] = (int)p.node_orig.size();
    p.node_orig.push_back(n);
  }
  int n_sched = (int)p.node_orig.size();
  p.L = 0;
  for (int n : sched) p.L = std::max(p.L, level[n] + 1);
  p.lvl_node_ptr.assign(p.L + 1, 0);
  for (int n : sched) p.lvl_node_ptr[level[n] + 1]++;
  for (int l = 0; l < p.L; l++) p.lvl_node_ptr[l + 1] += p.lvl_node_ptr[l];
  if (p.status == GTNB_OK) {
    for (int n : adj.accept)
      if (pop[n] < 0 && new_id[n] < 0) { // deg == 0, never scheduled: score stays 0.0f
        new_id[n] = (int)p.node_orig.size();
        p.node_orig.push_back(n);
      }
  }
  p.N = (int)p.node_orig.size();

  p.row_ptr.assign(p.N + 1, 0);
  p.src.clear();
  p.w.clear();
  p.arc_orig.clear();
  p.relax_rank.clear();
  for (int i = 0; i < p.N; i++) {
    int n = p.node_orig[i];
    uint32_t flags = ((v.node_flags[n] & 1) ? kStartBit : 0) | ((v.node_flags[n] & 2) ? kAcceptBit : 0);
    p.row_ptr[i] = (uint32_t)p.src.size() | flags;
    if (i < n_sched) {
      for (int k = adj.in_ptr[n]; k < adj.in_ptr[n + 1]; k++) {
        int a = adj.in_arcs[k];
        int s = v.arc_src[a];
        p.src.push_back(new_id[s]);
        p.w.push_back(v.weights ? v.weights[a] : 0.0f);
        p.arc_orig.push_back(a);
        p.relax_rank.push_back(rank[a]);
        if (level[s] != level[n] - 1) p.level_local = false;
      }
    }
  }
  p.A = (int)p.src.size();
  p.row_ptr[p.N] = (uint32_t)p.A;
  p.lvl_arc_ptr.assign(p.L + 1, 0);
  for (int l = 0; l <= p.L; l++) p.lvl_arc_ptr[l] = (int)(p.row_ptr[p.lvl_node_ptr[l]] & kRowMask);
  for (int l = 0; l < p.L; l++) {
    p.max_lvl_nodes = std::max(p.max_lvl_nodes, p.lvl_node_ptr[l + 1] - p.lvl_node_ptr[l]);
    p.max_lvl_arcs = std::max(p.max_lvl_arcs, p.lvl_arc_ptr[l + 1] - p.lvl_arc_ptr[l]);
  }
  p.acc.clear();
  if (p.status == GTNB_OK)
    for (int n : adj.accept) p.acc.push_back(new_id[n]);

  // backward schedule
  p.blvl_ptr.assign(1, 0);
  p.bnodes.clear();
  p.LB = 0;
  if (p.status == GTNB_OK) {
    std::vector<int32_t> od(N), bl(N, 0), border;
    for (int n = 0; n < N; n++) od[n] = adj.out_ptr[n + 1] - adj.out_ptr[n];
    std::vector<uint8_t> seen(N, 0);
    for (int n : adj.accept)
      if (od[n] == 0 && !seen[n]) {
        seen[n] = 1;
        border.push_back(n);
      }
    size_t h = 0;
    while (h < border.size()) {
      int n = border[h++];
      for (int k = adj.in_ptr[n]; k < adj.in_ptr[n + 1]; k++) {
        int un = v.arc_src[adj.in_arcs[k]];
        bl[un] = std::max(bl[un], bl[n] + 1);
        if (--od[un] == 0) border.push_back(un);
      }
    }
    // only nodes that own device in-arcs do any work
    std::vector<int32_t> work;
    for (int n : border)
      if (new_id[n] >= 0 && new_id[n] < n_sched) work.push_back(n);
    std::stable_sort(work.begin(), work.end(), [&](int a, int b) { return bl[a] < bl[b]; });
    int cur = -1;
    for (int n : work) {
      while (cur < bl[n]) {
        cur++;
        if (cur > 0) p.blvl_ptr.push_back((int)p.bnodes.size());
      }
      p.bnodes.push_back(new_id[n]);
    }
    p.LB = work.empty() ? 0 : cur + 1;
    p.blvl_ptr.push_back((int)p.bnodes.size());
    if (work.empty()) p.blvl_ptr.assign(1, 0);
  }
}

void free_lattice_device(gtnb_ctx* ctx, gtnb_lattice* lat) {
  dev_free(ctx, lat->meta);
  dev_free(ctx, lat->lvl_node_ptr);
  dev_free(ctx, lat->lvl_arc_ptr);
  dev_free(ctx, lat->row_ptr);
  dev_free(ctx, lat->arcs);
  dev_free(ctx, lat->acc_nodes);
  dev_free(ctx, lat->gi);
  dev_free(ctx, lat->node_orig);
  dev_free(ctx, lat->arc_orig);
  dev_free(ctx, lat->relax_rank);
  dev_free(ctx, lat->blvl_ptr);
  dev_free(ctx, lat->bnodes);
  dev_free(ctx, lat->scores);
  dev_free(ctx, lat->out_scores);
  dev_free(ctx, lat->best_accept);
  dev_free(ctx, lat->node_grad);
  dev_free(ctx, lat->arc_grad);
  dev_free(ctx, lat->back_ptr);
  dev_free(ctx, lat->sg_flags);
  dev_free(ctx, lat->sg_in_ptr);
  dev_free(ctx, lat->sg_in_src);
  dev_free(ctx, lat->sg_in_label);
  dev_free(ctx, lat->sg_in_arc);
  dev_free(ctx, lat->sg_in_w);
  dev_free(ctx, lat->sg_ilabel);
  dev_free(ctx, lat->sg_olabel);
  dev_free(ctx, lat->sg_out_pos);
  dev_free(ctx, lat->sg_start_rank);
  dev_free(ctx, lat->alive);
}

template <typename T>
int upload_slabs(
    gtnb_ctx* ctx, T* dst, const std::vector<long long>& bases,
    const std::vector<const std::vector<T>*>& parts) {
  // gather into one staging vector so a single copy moves the whole batch
  long long total = 0;
  for (size_t i = 0; i < parts.size(); i++)
    total = std::max(total, bases[i] + (long long)parts[i]->size());
  if (total == 0) return GTNB_OK;
  std::vector<T> stage((size_t)total);
  for (size_t i = 0; i < parts.size(); i++)
    if (!parts[i]->empty())
      std::memcpy(stage.data() + bases[i], parts[i]->data(), sizeof(T) * parts[i]->size());
  return upload(ctx, dst, stage.data(), total);
}

} // namespace


namespace gtnb {

/*
 * Size and allocate a composed lattice batch (level == frame).  Capacities are
 * upper bounds ((T+1) * N nodes, T * A arcs per utterance) so no device->host
 * round trip is needed before the kernels run; the exact counts are written
 * into the device-side GraphMeta by compose_scan_kernel.
 */
int composed_alloc(
    gtnb_ctx* ctx, int B, const SgDims* dims, int n_graphs, int linear_first, const int32_t* T,
    int C, const float* emissions_dev, int64_t emissions_stride, std::vector<long long>& sgn,
    std::vector<long long>& sga, gtnb_lattice** out, bool implicit_only) {
  *out = nullptr;
  int maxN = 0, maxA = 0, maxIn = 0, maxOut = 0;
  bool arc = false;
  for (int g = 0; g < n_graphs; g++) {
    maxN = std::max(maxN, dims[g].N);
    maxA = std::max(maxA, dims[g].A);
    maxIn = std::max(maxIn, dims[g].max_in);
    maxOut = std::max(maxOut, dims[g].max_out);
    arc |= !dims[g].uniform;
  }
  gtnb_lattice* lat = new gtnb_lattice();
  lat->arc_labels = implicit_only && arc;
  lat->max_in_deg = maxIn;
  lat->max_out_deg = maxOut;
  lat->B = B;
  lat->composed = true;
  lat->linear_first = linear_first != 0;
  lat->shared_graph = n_graphs == 1;
  lat->level_local = true;
  lat->sizes_known = false;
  lat->C = C;
  lat->emissions = emissions_dev;
  lat->emissions_stride = emissions_stride;
  lat->max_lvl_nodes = maxN;
  lat->max_lvl_arcs = maxA;
  lat->alive_words = (maxN + 31) / 32;
  lat->meta_h.resize(B);

  sgn.assign(n_graphs, 0);
  sga.assign(n_graphs, 0);
  long long tsn = 0, tsa = 0;
  for (int g = 0; g < n_graphs; g++) {
    sgn[g] = tsn;
    sga[g] = tsa;
    tsn += align_up(dims[g].N + 1, kAlign);
    tsa += align_up(std::max(dims[g].A, 1), kAlign);
  }
  lat->tot_sgN = tsn;
  lat->tot_sgA = tsa;

  long long tn = 0, ta = 0, tl = 0, tc = 0, gg_off = 0;
  int maxT = 0;
  const int fixed_pitch = (implicit_only && maxN <= kImplicitFixedPitch) ? kImplicitFixedPitch : 0;
  lat->score_pitch = fixed_pitch;
  for (int b = 0; b < B; b++) {
    if (T[b] < 0) {
      delete lat;
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_compose_linear: negative T");
    }
    const int g = n_graphs == 1 ? 0 : b;
    const SgDims& s = dims[g];
    GraphMeta& m = lat->meta_h[b];
    std::memset(&m, 0, sizeof(m));
    long long capN = align_up((long long)(T[b] + 1) * s.N + 1, kAlign);
    long long capA = align_up(std::max<long long>((long long)T[b] * s.A, 1), kAlign);
    if (implicit_only) {
      // implicit lattice (k_implicit.cu): only dense per-frame node scores, rows padded to 16 bytes
      // (graphs of up to 224 nodes: rows of 224, the fixed pitch of k_bidir.cu's FX kernels; the two sweeps of
      // k_implicit.cu use the first align_up(N) * (T + 1) floats of the same slab)
      capN = (long long)(T[b] + 1) * (fixed_pitch ? fixed_pitch : align_up(s.N, kAlign)) + kAlign;
      capA = kAlign;
    }
    if (!implicit_only && (capA >= (1ll << 30) || capN >= (1ll << 30))) {
      delete lat;
      return fail(ctx, GTNB_ERR_UNSUPPORTED,
                  "gtnb_compose_linear: lattice too large to materialise (use the factored path)");
    }
    m.node_base = tn;
    m.arc_base = ta;
    m.lvl_base = tl;
    m.acc_base = tc;
    m.sg_node_base = sgn[g];
    m.sg_arc_base = sga[g];
    m.emis_off = (long long)b * emissions_stride;
    m.grad_graph_off = gg_off;
    if (n_graphs != 1) gg_off += s.A;
    m.L = T[b] + 1;
    m.n_accept = s.n_acc; // provisional: the graph's accept count, compose_scan_kernel rewrites it
    m.LB = -1;
    m.status = GTNB_OK;
    m.T = T[b];
    m.sg_N = s.N;
    m.sg_A = s.A;
    m.sg_all_valid = s.all_valid;
    m.sg_uniform = s.uniform;
    m.cap_N = (int)std::min<long long>(capN, 0x7fffffff);
    m.cap_A = (int)capA;
    m.cap_L = (int)align_up(T[b] + 2, kAlign);
    tn += capN;
    ta += capA;
    tl += m.cap_L;
    tc += align_up(std::max<long long>(s.n_acc, 1), kAlign);
    maxT = std::max(maxT, T[b]);
  }
  lat->tot_N = tn;
  lat->tot_A = ta;
  lat->tot_L = tl;
  lat->tot_acc = tc;
  lat->max_T = maxT;

  size_t need = (size_t)(tn * 8 + ta * 20 + tl * 8) + (size_t)B * (maxT + 1) * lat->alive_words * 4;
  if (implicit_only) need = (size_t)tn * 4;
  // the device's capacity, cached at context creation: cudaMemGetInfo is a driver round trip of tens
  // of microseconds, and this runs once per criterion call, ahead of the first kernel launch
  if (ctx->total_mem && need > ctx->total_mem) {
    delete lat;
    return fail(ctx, GTNB_ERR_UNSUPPORTED,
                "gtnb_compose_linear: materialised lattice would not fit in HBM (use the factored path)");
  }
  int rc = GTNB_OK;
#define TRYA(x)               \
  do {                        \
    if ((rc = (x))) goto bad; \
  } while (0)
  TRYA(dev_alloc(ctx, &lat->meta, B));
  if (!implicit_only) {
    TRYA(dev_alloc(ctx, &lat->lvl_node_ptr, tl));
    TRYA(dev_alloc(ctx, &lat->lvl_arc_ptr, tl));
    TRYA(dev_alloc(ctx, &lat->row_ptr, tn));
    TRYA(dev_alloc(ctx, &lat->arcs, ta));
    TRYA(dev_alloc(ctx, &lat->gi, ta));
  }
  TRYA(dev_alloc(ctx, &lat->acc_nodes, tc));
  TRYA(dev_alloc(ctx, &lat->scores, tn));
  TRYA(dev_alloc(ctx, &lat->out_scores, B));
  TRYA(dev_alloc(ctx, &lat->best_accept, B));
  TRYA(dev_alloc(ctx, &lat->sg_flags, tsn));
  TRYA(dev_alloc(ctx, &lat->sg_in_ptr, tsn));
  TRYA(dev_alloc(ctx, &lat->sg_in_src, tsa));
  TRYA(dev_alloc(ctx, &lat->sg_in_label, tsa));
  TRYA(dev_alloc(ctx, &lat->sg_in_arc, tsa));
  TRYA(dev_alloc(ctx, &lat->sg_in_w, tsa));
  TRYA(dev_alloc(ctx, &lat->sg_ilabel, tsa));
  TRYA(dev_alloc(ctx, &lat->sg_olabel, tsa));
  if (!implicit_only) TRYA(dev_alloc(ctx, &lat->alive, (long long)B * (maxT + 1) * lat->alive_words));
#undef TRYA
  *out = lat;
  return GTNB_OK;
bad:
  free_lattice_device(ctx, lat);
  delete lat;
  return rc;
}

} // namespace gtnb

extern "C" {

/* ------------------------------------------------------------------ */
/* gtnb_pack                                                           */
/* ------------------------------------------------------------------ */

int gtnb_pack(gtnb_ctx* ctx, int B, const gtnb_graph_view* graphs, gtnb_lattice** out) {
  if (!ctx || !out || B < 0 || (B > 0 && !graphs))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_pack: bad arguments");
  *out = nullptr;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  std::vector<PackedGraph> P(B);
  for (int b = 0; b < B; b++) {
    int rc = validate_view(ctx, graphs[b]);
    if (rc) return rc;
    if (graphs[b].num_arcs >= (1 << 30))
      return fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_pack: more than 2^30 arcs in one graph");
    Adj adj;
    build_adj(graphs[b], adj);
    pack_one(graphs[b], adj, P[b]);
  }
  gtnb_lattice* lat = new gtnb_lattice();
  lat->B = B;
  lat->composed = false;
  lat->level_local = true;
  lat->sizes_known = true;
  lat->meta_h.resize(B);
  std::vector<long long> nb(B), ab(B), lb(B), cb(B), blb(B), bnb(B);
  long long tn = 0, ta = 0, tl = 0, tc = 0, tbl = 0, tbn = 0;
  for (int b = 0; b < B; b++) {
    PackedGraph& p = P[b];
    GraphMeta& m = lat->meta_h[b];
    std::memset(&m, 0, sizeof(m));
    nb[b] = tn;
    ab[b] = ta;
    lb[b] = tl;
    cb[b] = tc;
    blb[b] = tbl;
    bnb[b] = tbn;
    m.node_base = tn;
    m.arc_base = ta;
    m.lvl_base = tl;
    m.acc_base = tc;
    m.blvl_base = tbl;
    m.bnode_base = tbn;
    m.L = p.L;
    m.N = p.N;
    m.A = p.A;
    m.n_accept = (int)p.acc.size();
    m.LB = p.LB;
    m.status = p.status;
    m.cap_N = (int)align_up(p.N + 1, kAlign);
    m.cap_A = (int)align_up(std::max(p.A, 1), kAlign);
    m.cap_L = (int)align_up(p.L + 1, kAlign);
    tn += m.cap_N;
    ta += m.cap_A;
    tl += m.cap_L;
    tc += align_up(std::max<long long>(p.acc.size(), 1), kAlign);
    tbl += align_up((long long)p.blvl_ptr.size(), kAlign);
    tbn += align_up(std::max<long long>(p.bnodes.size(), 1), kAlign);
    lat->level_local = lat->level_local && p.level_local;
    lat->max_lvl_nodes = std::max(lat->max_lvl_nodes, p.max_lvl_nodes);
    lat->max_lvl_arcs = std::max(lat->max_lvl_arcs, p.max_lvl_arcs);
  }
  lat->tot_N = tn;
  lat->tot_A = ta;
  lat->tot_L = tl;
  lat->tot_acc = tc;
  lat->tot_bl = tbl;
  lat->tot_bn = tbn;

  int rc = GTNB_OK;
#define TRY(x)              \
  do {                      \
    if ((rc = (x))) goto bad; \
  } while (0)
  {
    TRY(dev_alloc(ctx, &lat->meta, B));
    TRY(dev_alloc(ctx, &lat->lvl_node_ptr, tl));
    TRY(dev_alloc(ctx, &lat->lvl_arc_ptr, tl));
    TRY(dev_alloc(ctx, &lat->row_ptr, tn));
    TRY(dev_alloc(ctx, &lat->arcs, ta));
    TRY(dev_alloc(ctx, &lat->acc_nodes, tc));
    TRY(dev_alloc(ctx, &lat->arc_orig, ta));
    TRY(dev_alloc(ctx, &lat->relax_rank, ta));
    TRY(dev_alloc(ctx, &lat->blvl_ptr, tbl));
    TRY(dev_alloc(ctx, &lat->bnodes, tbn));
    TRY(dev_alloc(ctx, &lat->scores, tn));
    TRY(dev_alloc(ctx, &lat->out_scores, B));
    TRY(dev_alloc(ctx, &lat->best_accept, B));
    TRY(upload(ctx, lat->meta, lat->meta_h.data(), B));
    std::vector<const std::vector<int32_t>*> pi(B);
    std::vector<const std::vector<uint32_t>*> pu(B);
    std::vector<const std::vector<float>*> pf(B);
    for (int b = 0; b < B; b++) pi[b] = &P[b].lvl_node_ptr;
    TRY(upload_slabs(ctx, lat->lvl_node_ptr, lb, pi));
    for (int b = 0; b < B; b++) pi[b] = &P[b].lvl_arc_ptr;
    TRY(upload_slabs(ctx, lat->lvl_arc_ptr, lb, pi));
    for (int b = 0; b < B; b++) pu[b] = &P[b].row_ptr;
    TRY(upload_slabs(ctx, lat->row_ptr, nb, pu));
    {
      std::vector<std::vector<int2>> inter(B);
      std::vector<const std::vector<int2>*> pa(B);
      for (int b = 0; b < B; b++) {
        inter[b].resize(P[b].src.size());
        for (size_t a = 0; a < P[b].src.size(); a++) {
          int wb;
          std::memcpy(&wb, &P[b].w[a], 4);
          inter[b][a] = make_int2(P[b].src[a], wb);
        }
        pa[b] = &inter[b];
      }
      TRY(upload_slabs(ctx, lat->arcs, ab, pa));
    }
    for (int b = 0; b < B; b++) pi[b] = &P[b].acc;
    TRY(upload_slabs(ctx, lat->acc_nodes, cb, pi));
    for (int b = 0; b < B; b++) pi[b] = &P[b].arc_orig;
    TRY(upload_slabs(ctx, lat->arc_orig, ab, pi));
    for (int b = 0; b < B; b++) pi[b] = &P[b].relax_rank;
    TRY(upload_slabs(ctx, lat->relax_rank, ab, pi));
    for (int b = 0; b < B; b++) pi[b] = &P[b].blvl_ptr;
    TRY(upload_slabs(ctx, lat->blvl_ptr, blb, pi));
    for (int b = 0; b < B; b++) pi[b] = &P[b].bnodes;
    TRY(upload_slabs(ctx, lat->bnodes, bnb, pi));
  }
  lat->h_node_orig.resize(B);
  lat->h_arc_orig.resize(B);
  lat->h_ilabel.resize(B);
  lat->h_olabel.resize(B);
  lat->h_arcs_orig_count.resize(B);
  for (int b = 0; b < B; b++) {
    lat->h_node_orig[b] = std::move(P[b].node_orig);
    lat->h_arc_orig[b] = std::move(P[b].arc_orig);
    lat->h_ilabel[b].assign(graphs[b].arc_ilabel, graphs[b].arc_ilabel + graphs[b].num_arcs);
    lat->h_olabel[b].assign(graphs[b].arc_olabel, graphs[b].arc_olabel + graphs[b].num_arcs);
    lat->h_arcs_orig_count[b] = graphs[b].num_arcs;
  }
  *out = lat;
  return GTNB_OK;
bad:
  free_lattice_device(ctx, lat);
  delete lat;
  return rc;
#undef TRY
}

void gtnb_lattice_destroy(gtnb_ctx* ctx, gtnb_lattice* lat) {
  if (!lat) return;
  if (ctx) {
    cudaSetDevice(ctx->device);
    free_lattice_device(ctx, lat);
  }
  delete lat;
}

int gtnb_lattice_batch(const gtnb_lattice* lat) {
  return lat ? lat->B : 0;
}

static int fetch_sizes(gtnb_ctx* ctx, gtnb_lattice* lat) {
  if (lat->sizes_known) return GTNB_OK;
  GTNB_CUDA(ctx, cudaMemcpyAsync(lat->meta_h.data(), lat->meta, sizeof(GraphMeta) * lat->B,
                                 cudaMemcpyDeviceToHost, ctx->stream));
  GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  lat->sizes_known = true;
  return GTNB_OK;
}

int gtnb_lattice_sizes(gtnb_ctx* ctx, gtnb_lattice* lat, int32_t* num_nodes, int32_t* num_arcs) {
  if (!ctx || !lat) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_lattice_sizes: NULL");
  int rc = fetch_sizes(ctx, lat);
  if (rc) return rc;
  for (int b = 0; b < lat->B; b++) {
    if (num_nodes) num_nodes[b] = lat->meta_h[b].N;
    if (num_arcs) num_arcs[b] = lat->meta_h[b].A;
  }
  return GTNB_OK;
}

/* exact_ties: a composed lattice's rows are put in the reference's relaxation order (k_order.cu) before the first
 * call that hands out arc ids or per-arc values -- download, arc gradients in or out, a Viterbi path -- so that every
 * such call sees one numbering whatever ran before it.  forward and backward work in either order (the sort
 * carries arc_grad), so a lattice whose arcs never cross the ABI is never sorted.  Runs at most once. */
static int settle_order(gtnb_ctx* ctx, gtnb_lattice* lat) {
  if (!lat->order_pending) return GTNB_OK;
  int rc = launch_relax_order(ctx, lat);
  if (rc) return rc;
  lat->order_pending = false;
  return GTNB_OK;
}

int gtnb_lattice_download(
    gtnb_ctx* ctx, gtnb_lattice* lat, int b, uint8_t* node_flags, int32_t* arc_src,
    int32_t* arc_dst, int32_t* arc_ilabel, int32_t* arc_olabel, float* weights,
    int32_t* gi_graph, int32_t* gi_linear) {
  if (!ctx || !lat || b < 0 || b >= lat->B)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_lattice_download: bad arguments");
  int rc = fetch_sizes(ctx, lat);
  if (rc) return rc;
  if ((rc = settle_order(ctx, lat))) return rc;
  const GraphMeta& m = lat->meta_h[b];
  std::vector<uint32_t> rp(m.N + 1);
  std::vector<int32_t> src(std::max(m.A, 1)), gg(std::max(m.A, 1), -1), gl(std::max(m.A, 1), -1);
  std::vector<float> w(std::max(m.A, 1));
  std::vector<int2> arcs_h(std::max(m.A, 1)), gi_h(std::max(m.A, 1));
  GTNB_CUDA(ctx, cudaMemcpyAsync(rp.data(), lat->row_ptr + m.node_base, sizeof(uint32_t) * (m.N + 1),
                                 cudaMemcpyDeviceToHost, ctx->stream));
  if (m.A > 0) {
    GTNB_CUDA(ctx, cudaMemcpyAsync(arcs_h.data(), lat->arcs + m.arc_base, sizeof(int2) * m.A,
                                   cudaMemcpyDeviceToHost, ctx->stream));
    if (lat->gi)
      GTNB_CUDA(ctx, cudaMemcpyAsync(gi_h.data(), lat->gi + m.arc_base, sizeof(int2) * m.A,
                                     cudaMemcpyDeviceToHost, ctx->stream));
  }
  std::vector<int32_t> il, ol;
  if (lat->composed && (arc_ilabel || arc_olabel)) {
    il.resize(std::max(m.sg_A, 1));
    ol.resize(std::max(m.sg_A, 1));
    GTNB_CUDA(ctx, cudaMemcpyAsync(il.data(), lat->sg_ilabel + m.sg_arc_base, sizeof(int32_t) * m.sg_A,
                                   cudaMemcpyDeviceToHost, ctx->stream));
    GTNB_CUDA(ctx, cudaMemcpyAsync(ol.data(), lat->sg_olabel + m.sg_arc_base, sizeof(int32_t) * m.sg_A,
                                   cudaMemcpyDeviceToHost, ctx->stream));
  }
  GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int a = 0; a < m.A; a++) {
    src[a] = arcs_h[a].x;
    std::memcpy(&w[a], &arcs_h[a].y, 4);
    if (lat->gi) {
      gg[a] = gi_h[a].x;
      gl[a] = gi_h[a].y;
    }
  }
  if (lat->composed) {
    // device numbering IS the Graph numbering of a composed lattice
    for (int n = 0; n < m.N; n++) {
      if (node_flags) node_flags[n] = ((rp[n] & kStartBit) ? 1 : 0) | ((rp[n] & kAcceptBit) ? 2 : 0);
      for (uint32_t a = rp[n] & kRowMask; a < (rp[n + 1] & kRowMask); a++) {
        if (arc_src) arc_src[a] = src[a];
        if (arc_dst) arc_dst[a] = n;
        if (weights) weights[a] = w[a];
        int c = gl[a] % lat->C;
        if (arc_ilabel) arc_ilabel[a] = lat->linear_first ? c : il[gg[a]];
        if (arc_olabel) arc_olabel[a] = lat->linear_first ? ol[gg[a]] : c;
        if (gi_graph) gi_graph[a] = gg[a];
        if (gi_linear) gi_linear[a] = gl[a];
      }
    }
  } else {
    const auto& no = lat->h_node_orig[b];
    const auto& ao = lat->h_arc_orig[b];
    for (int n = 0; n < m.N; n++) {
      if (node_flags) node_flags[no[n]] = ((rp[n] & kStartBit) ? 1 : 0) | ((rp[n] & kAcceptBit) ? 2 : 0);
      for (uint32_t a = rp[n] & kRowMask; a < (rp[n + 1] & kRowMask); a++) {
        int oa = ao[a];
        if (arc_src) arc_src[oa] = no[src[a]];
        if (arc_dst) arc_dst[oa] = no[n];
        if (weights) weights[oa] = w[a];
        if (arc_ilabel) arc_ilabel[oa] = lat->h_ilabel[b][oa];
        if (arc_olabel) arc_olabel[oa] = lat->h_olabel[b][oa];
        if (gi_graph) gi_graph[oa] = -1;
        if (gi_linear) gi_linear[oa] = -1;
      }
    }
  }
  return GTNB_OK;
}

/* ------------------------------------------------------------------ */
/* forward / backward / path                                           */
/* ------------------------------------------------------------------ */

static int first_bad_status(gtnb_ctx* ctx, gtnb_lattice* lat, int32_t* status_host) {
  int bad = GTNB_OK;
  for (int b = 0; b < lat->B; b++) {
    int s = lat->meta_h[b].status;
    if (status_host) status_host[b] = s;
    if (s != GTNB_OK && bad == GTNB_OK) bad = s;
  }
  if (bad != GTNB_OK)
    return fail(ctx, bad, "Graph has a cycle, self-loop or is disconnected!"); // shortest.cpp:150
  return GTNB_OK;
}

int gtnb_forward(gtnb_ctx* ctx, gtnb_lattice* lat, int tropical, float* scores_host, int32_t* status_host) {
  if (!ctx || !lat) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_forward: NULL");
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  int bad = first_bad_status(ctx, lat, status_host);
  int rc = launch_forward(ctx, lat, tropical ? MODE_TROPICAL : MODE_LOG);
  if (rc) return rc;
  lat->forward_done = true;
  lat->forward_mode = tropical ? MODE_TROPICAL : MODE_LOG;
  if (scores_host) {
    GTNB_CUDA(ctx, cudaMemcpyAsync(scores_host, lat->out_scores, sizeof(float) * lat->B,
                                   cudaMemcpyDeviceToHost, ctx->stream));
    GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return bad;
}

int gtnb_backward(gtnb_ctx* ctx, gtnb_lattice* lat, int tropical, const float* deltas_host) {
  if (!ctx || !lat) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_backward: NULL");
  if (!lat->forward_done || lat->forward_mode != (tropical ? MODE_TROPICAL : MODE_LOG))
    return fail(ctx, GTNB_ERR_LOGIC, "gtnb_backward: no matching gtnb_forward on this lattice");
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  float* deltas_dev = nullptr;
  int rc;
  if (deltas_host) {
    if ((rc = dev_alloc(ctx, &deltas_dev, lat->B))) return rc;
    if ((rc = upload(ctx, deltas_dev, deltas_host, lat->B))) return rc;
  }
  if (!lat->arc_grad && (rc = dev_alloc(ctx, &lat->arc_grad, lat->tot_A))) return rc;
  rc = launch_backward(ctx, lat, tropical, deltas_dev);
  dev_free(ctx, deltas_dev);
  return rc;
}

const float* gtnb_lattice_arc_grads_dev(gtnb_ctx* ctx, gtnb_lattice* lat) {
  if (!ctx || !lat) {
    fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_lattice_arc_grads_dev: NULL");
    return nullptr;
  }
  if (cudaSetDevice(ctx->device) != cudaSuccess || settle_order(ctx, lat)) return nullptr;
  return lat->arc_grad;
}

int gtnb_lattice_arc_grads(gtnb_ctx* ctx, gtnb_lattice* lat, int b, float* out_host) {
  if (!ctx || !lat || b < 0 || b >= lat->B || !out_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_lattice_arc_grads: bad arguments");
  if (!lat->arc_grad) return fail(ctx, GTNB_ERR_LOGIC, "gtnb_lattice_arc_grads: no backward yet");
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  int rc = fetch_sizes(ctx, lat);
  if (rc) return rc;
  if ((rc = settle_order(ctx, lat))) return rc;
  const GraphMeta& m = lat->meta_h[b];
  if (lat->composed) {
    GTNB_CUDA(ctx, cudaMemcpyAsync(out_host, lat->arc_grad + m.arc_base, sizeof(float) * m.A,
                                   cudaMemcpyDeviceToHost, ctx->stream));
    GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GTNB_OK;
  }
  std::vector<float> tmp(std::max(m.A, 1));
  GTNB_CUDA(ctx, cudaMemcpyAsync(tmp.data(), lat->arc_grad + m.arc_base, sizeof(float) * m.A,
                                 cudaMemcpyDeviceToHost, ctx->stream));
  GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  int A0 = lat->h_arcs_orig_count[b];
  for (int a = 0; a < A0; a++) out_host[a] = 0.0f; // arcs the sweep never reaches keep 0 (shortest.cpp:44)
  for (int a = 0; a < m.A; a++) out_host[lat->h_arc_orig[b][a]] = tmp[a];
  return GTNB_OK;
}

int gtnb_lattice_set_arc_grads(gtnb_ctx* ctx, gtnb_lattice* lat, int b, const float* grads_host) {
  if (!ctx || !lat || b < 0 || b >= lat->B || !grads_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_lattice_set_arc_grads: bad arguments");
  if (!lat->composed)
    return fail(ctx, GTNB_ERR_LOGIC, "gtnb_lattice_set_arc_grads: only for composed lattices");
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  int rc = fetch_sizes(ctx, lat);
  if (rc) return rc;
  if (!lat->arc_grad && (rc = dev_alloc(ctx, &lat->arc_grad, lat->tot_A))) return rc;
  if ((rc = settle_order(ctx, lat))) return rc;
  const GraphMeta& m = lat->meta_h[b];
  GTNB_CUDA(ctx, cudaMemcpyAsync(lat->arc_grad + m.arc_base, grads_host, sizeof(float) * m.A,
                                 cudaMemcpyHostToDevice, ctx->stream));
  return GTNB_OK;
}

int gtnb_viterbi_path(
    gtnb_ctx* ctx, gtnb_lattice* lat, int max_len, int32_t* path_arcs_host,
    int32_t* path_ilabels_host, int32_t* path_olabels_host, float* path_weights_host,
    int32_t* path_len_host, int32_t* status_host) {
  if (!ctx || !lat || max_len < 0 || !path_len_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_viterbi_path: bad arguments");
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  int bad = first_bad_status(ctx, lat, status_host);
  int rc;
  if (!lat->back_ptr && (rc = dev_alloc(ctx, &lat->back_ptr, lat->tot_N))) return rc;
  if ((rc = settle_order(ctx, lat))) return rc;
  if ((rc = launch_forward(ctx, lat, MODE_PATH))) return rc;
  lat->forward_done = false; // scores now hold the path recursion, not shortestDistance
  int B = lat->B;
  int32_t *path_dev = nullptr, *len_dev = nullptr;
  long long tot = (long long)B * std::max(max_len, 1);
  if ((rc = dev_alloc(ctx, &path_dev, tot))) return rc;
  if ((rc = dev_alloc(ctx, &len_dev, B))) return rc;
  if ((rc = launch_traceback(ctx, lat, max_len, path_dev, len_dev))) return rc;
  std::vector<int32_t> path((size_t)tot);
  GTNB_CUDA(ctx, cudaMemcpyAsync(path.data(), path_dev, sizeof(int32_t) * tot, cudaMemcpyDeviceToHost, ctx->stream));
  GTNB_CUDA(ctx, cudaMemcpyAsync(path_len_host, len_dev, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, ctx->stream));
  std::vector<int32_t> gg, gl;
  bool want_labels = path_ilabels_host || path_olabels_host;
  std::vector<int32_t> sil, sol;
  if (lat->composed && want_labels) {
    sil.resize((size_t)std::max<long long>(lat->tot_sgA, 1));
    sol.resize(sil.size());
    GTNB_CUDA(ctx, cudaMemcpyAsync(sil.data(), lat->sg_ilabel, sizeof(int32_t) * lat->tot_sgA, cudaMemcpyDeviceToHost, ctx->stream));
    GTNB_CUDA(ctx, cudaMemcpyAsync(sol.data(), lat->sg_olabel, sizeof(int32_t) * lat->tot_sgA, cudaMemcpyDeviceToHost, ctx->stream));
  }
  GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  // composed lattices: labels come from the provenance arrays (gathered on device by traceback
  // into the upper half of path_dev would be nicer; the paths are tiny so do it here)
  std::vector<int32_t> prov_g, prov_l;
  if ((lat->composed && want_labels) || path_weights_host) {
    // fetch provenance / weights for just the path arcs
    prov_g.resize(path.size());
    prov_l.resize(path.size());
    int32_t *pg = nullptr, *pl = nullptr;
    float* pw = nullptr;
    if ((rc = dev_alloc(ctx, &pg, tot))) return rc;
    if ((rc = dev_alloc(ctx, &pl, tot))) return rc;
    if (path_weights_host && (rc = dev_alloc(ctx, &pw, tot))) return rc;
    if ((rc = launch_gather_prov(ctx, lat, max_len, path_dev, len_dev, pg, pl, pw))) return rc;
    if (lat->gi) {
      GTNB_CUDA(ctx, cudaMemcpyAsync(prov_g.data(), pg, sizeof(int32_t) * tot, cudaMemcpyDeviceToHost, ctx->stream));
      GTNB_CUDA(ctx, cudaMemcpyAsync(prov_l.data(), pl, sizeof(int32_t) * tot, cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (pw)
      GTNB_CUDA(ctx, cudaMemcpyAsync(path_weights_host, pw, sizeof(float) * tot, cudaMemcpyDeviceToHost, ctx->stream));
    GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    dev_free(ctx, pg);
    dev_free(ctx, pl);
    dev_free(ctx, pw);
  }
  for (int b = 0; b < B; b++) {
    int len = path_len_host[b];
    const GraphMeta& m = lat->meta_h[b];
    for (int i = 0; i < std::min(len, max_len); i++) {
      size_t k = (size_t)b * max_len + i;
      int a = path[k];
      if (lat->composed) {
        if (path_arcs_host) path_arcs_host[k] = a;
        if (want_labels) {
          int c = prov_l[k] % lat->C;
          int ga = prov_g[k] + (int)m.sg_arc_base;
          if (path_ilabels_host) path_ilabels_host[k] = lat->linear_first ? c : sil[ga];
          if (path_olabels_host) path_olabels_host[k] = lat->linear_first ? sol[ga] : c;
        }
      } else {
        int oa = lat->h_arc_orig[b][a];
        if (path_arcs_host) path_arcs_host[k] = oa;
        if (path_ilabels_host) path_ilabels_host[k] = lat->h_ilabel[b][oa];
        if (path_olabels_host) path_olabels_host[k] = lat->h_olabel[b][oa];
      }
    }
  }
  dev_free(ctx, path_dev);
  dev_free(ctx, len_dev);
  return bad;
}

/* ------------------------------------------------------------------ */
/* frame-synchronous composition: host half                            */
/* ------------------------------------------------------------------ */

int gtnb_compose_linear(
    gtnb_ctx* ctx, int B, const gtnb_graph_view* graphs, int n_graphs, int linear_first,
    const int32_t* T, int C, const float* emissions_dev, int64_t emissions_stride,
    gtnb_lattice** out) {
  return gtnb::compose_linear_impl(ctx, B, graphs, n_graphs, linear_first, T, C, emissions_dev,
                                   emissions_stride, false, out);
}

} // extern "C"

/* implicit_only: upload the graph operands' tables and allocate the dense score rows, but build no
 * lattice (the criteria's implicit sweeps, k_implicit.cu); GTNB_ERR_UNSUPPORTED when the operands
 * do not qualify for them */
int gtnb::compose_linear_impl(
    gtnb_ctx* ctx, int B, const gtnb_graph_view* graphs, int n_graphs, int linear_first,
    const int32_t* T, int C, const float* emissions_dev, int64_t emissions_stride, bool implicit_only,
    gtnb_lattice** out, bool arc_labels, const float* arc_weights_dev) {
  if (!ctx || !out || B < 0 || !graphs || !T || C <= 0 || (n_graphs != B && n_graphs != 1))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_compose_linear: bad arguments");
  *out = nullptr;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));

  // canonical in-arc tables of the small graphs
  struct SG {
    int N = 0, A = 0;
    std::vector<uint8_t> flags;
    std::vector<int32_t> in_ptr, in_src, in_label, in_arc, il, ol, acc;
    std::vector<int32_t> in_out_pos, start_rank; // exact_ties only (k_order.cu)
    std::vector<float> in_w;
  };
  std::vector<SG> sg(n_graphs);
  int maxN = 0, maxA = 0;
  const bool exact_ties = ctx->exact_ties;
  // one graph's tables; independent of the others, so a large batch is spread over host threads (the list
  // forms of the gtn:: layer hand in B graphs at once)
  auto build_one = [&](int g) -> int {
    const gtnb_graph_view& v = graphs[g];
    if (validate_view(nullptr, v)) return GTNB_ERR_INVALID_ARGUMENT;
    Adj adj;
    build_adj(v, adj);
    SG& s = sg[g];
    s.N = v.num_nodes;
    s.A = v.num_arcs;
    s.flags.assign(v.node_flags, v.node_flags + s.N);
    s.il.assign(v.arc_ilabel, v.arc_ilabel + s.A);
    s.ol.assign(v.arc_olabel, v.arc_olabel + s.A);
    s.acc = adj.accept;
    // position of every arc in its source's out list: the order the
    // reference's matchers enumerate a state's arcs in (compose.cpp:211-374)
    std::vector<int32_t> out_pos(s.A, 0);
    for (int n = 0; n < s.N; n++)
      for (int k = adj.out_ptr[n]; k < adj.out_ptr[n + 1]; k++) out_pos[adj.out_arcs[k]] = k - adj.out_ptr[n];
    s.in_ptr.assign(s.N + 1, 0);
    for (int d = 0; d < s.N; d++) {
      std::vector<int32_t> arcs(adj.in_arcs.begin() + adj.in_ptr[d], adj.in_arcs.begin() + adj.in_ptr[d + 1]);
      std::stable_sort(arcs.begin(), arcs.end(), [&](int a, int b) {
        if (v.arc_src[a] != v.arc_src[b]) return v.arc_src[a] < v.arc_src[b];
        return out_pos[a] < out_pos[b];
      });
      for (int a : arcs) {
        // the label matched against the emissions' labels
        int lab = linear_first ? v.arc_ilabel[a] : v.arc_olabel[a];
        if (lab == GTNB_EPSILON)
          return GTNB_ERR_UNSUPPORTED;
        if (arc_labels && !(lab >= 0 && lab < C)) continue; // never matches: no entry, gradient 0
        s.in_src.push_back(v.arc_src[a]);
        s.in_label.push_back((lab >= 0 && lab < C) ? lab : -1);
        s.in_arc.push_back(a);
        s.in_w.push_back(v.weights ? v.weights[a] : 0.0f);
        if (exact_ties) s.in_out_pos.push_back(out_pos[a]);
      }
      s.in_ptr[d + 1] = (int)s.in_src.size();
    }
    if (arc_labels) {
      // the tables hold the entries kept; the by-arc-id label copies (read for Viterbi paths only, which
      // the loss never asks for) are cut to the same slab size
      s.A = (int)s.in_src.size();
      s.il.resize(s.A);
      s.ol.resize(s.A);
    }
    if (exact_ties) {
      s.start_rank.assign(s.N, -1);
      for (size_t k = 0; k < adj.start.size(); k++) s.start_rank[adj.start[k]] = (int32_t)k;
    }
      return GTNB_OK;
  };
  {
    std::vector<int> rcs(n_graphs, GTNB_OK);
    const int nthr = n_graphs >= 32 ? (int)std::min<unsigned>(16, std::max(1u, std::thread::hardware_concurrency())) : 1;
    if (nthr > 1) {
      std::vector<std::thread> pool;
      for (int t = 0; t < nthr; t++)
        pool.emplace_back([&, t] {
          for (int g = t; g < n_graphs; g += nthr) rcs[g] = build_one(g);
        });
      for (auto& th : pool) th.join();
    } else {
      for (int g = 0; g < n_graphs; g++) rcs[g] = build_one(g);
    }
    for (int g = 0; g < n_graphs; g++) {
      if (rcs[g] == GTNB_ERR_UNSUPPORTED)
        return fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_compose_linear: epsilon on the matched side (use the host compose)");
      if (rcs[g]) return validate_view(ctx, graphs[g]) ? GTNB_ERR_INVALID_ARGUMENT : rcs[g]; // (sets the message)
      maxN = std::max(maxN, sg[g].N);
      maxA = std::max(maxA, sg[g].A);
    }
  }

  std::vector<SgDims> dims(n_graphs);
  for (int g = 0; g < n_graphs; g++) {
    const SG& s = sg[g];
    int all_valid = 1, uniform = 1, max_in = 0;
    for (int lab : s.in_label) all_valid &= lab >= 0;
    std::vector<int> outdeg(s.N, 0);
    for (int d = 0; d < s.N; d++) {
      max_in = std::max(max_in, s.in_ptr[d + 1] - s.in_ptr[d]);
      for (int k = s.in_ptr[d]; k < s.in_ptr[d + 1]; k++) {
        uniform &= s.in_label[k] == s.in_label[s.in_ptr[d]];
        outdeg[s.in_src[k]]++;
      }
    }
    int max_out = 0;
    for (int n = 0; n < s.N; n++) max_out = std::max(max_out, outdeg[n]);
    dims[g] = SgDims{s.N, s.A, (int)s.acc.size(), all_valid, uniform, max_in, max_out};
  }
  if (implicit_only && !implicit_dims_supported(dims.data(), n_graphs, arc_labels ? C : 0))
    return fail(ctx, GTNB_ERR_UNSUPPORTED, "graph operand does not qualify for the implicit sweeps");
  std::vector<long long> sgn, sga;
  gtnb_lattice* lat = nullptr;
  int rc = composed_alloc(ctx, B, dims.data(), n_graphs, linear_first, T, C, emissions_dev,
                          emissions_stride, sgn, sga, &lat, implicit_only);
  if (rc) return rc;
  if (arc_labels && n_graphs != 1) { // arc-gradient slabs in Graph arc numbering, whatever was left out
    long long off = 0;
    for (int b = 0; b < B; b++) {
      lat->meta_h[b].grad_graph_off = off;
      off += graphs[b].num_arcs;
    }
  }
  const long long tc = lat->tot_acc;
#define TRY(x)              \
  do {                      \
    if ((rc = (x))) goto bad; \
  } while (0)
  {
    TRY(upload(ctx, lat->meta, lat->meta_h.data(), B));
    std::vector<const std::vector<int32_t>*> pi(n_graphs);
    std::vector<const std::vector<uint8_t>*> pb(n_graphs);
    std::vector<const std::vector<float>*> pf(n_graphs);
    for (int g = 0; g < n_graphs; g++) pb[g] = &sg[g].flags;
    TRY(upload_slabs(ctx, lat->sg_flags, sgn, pb));
    for (int g = 0; g < n_graphs; g++) pi[g] = &sg[g].in_ptr;
    TRY(upload_slabs(ctx, lat->sg_in_ptr, sgn, pi));
    for (int g = 0; g < n_graphs; g++) pi[g] = &sg[g].in_src;
    TRY(upload_slabs(ctx, lat->sg_in_src, sga, pi));
    for (int g = 0; g < n_graphs; g++) pi[g] = &sg[g].in_label;
    TRY(upload_slabs(ctx, lat->sg_in_label, sga, pi));
    for (int g = 0; g < n_graphs; g++) pi[g] = &sg[g].in_arc;
    TRY(upload_slabs(ctx, lat->sg_in_arc, sga, pi));
    for (int g = 0; g < n_graphs; g++) pf[g] = &sg[g].in_w;
    TRY(upload_slabs(ctx, lat->sg_in_w, sga, pf));
    if (arc_weights_dev) {
      // entry k of graph g reads arc_weights_dev[first arc of g + in_arc[k]]; padding keeps its 0
      std::vector<int32_t> widx((size_t)lat->tot_sgA, -1);
      long long first = 0;
      for (int g = 0; g < n_graphs; g++) {
        for (size_t k = 0; k < sg[g].in_arc.size(); k++) widx[sga[g] + k] = (int32_t)(first + sg[g].in_arc[k]);
        first += graphs[g].num_arcs;
      }
      int32_t* widx_dev = nullptr;
      TRY(dev_alloc(ctx, &widx_dev, lat->tot_sgA));
      rc = upload(ctx, widx_dev, widx.data(), lat->tot_sgA);
      if (!rc) rc = launch_gather(ctx, lat->sg_in_w, widx_dev, arc_weights_dev, lat->tot_sgA);
      dev_free(ctx, widx_dev);
      if (rc) goto bad;
    }
    for (int g = 0; g < n_graphs; g++) pi[g] = &sg[g].il;
    TRY(upload_slabs(ctx, lat->sg_ilabel, sga, pi));
    for (int g = 0; g < n_graphs; g++) pi[g] = &sg[g].ol;
    TRY(upload_slabs(ctx, lat->sg_olabel, sga, pi));
    if (ctx->exact_ties) {
      TRY(dev_alloc(ctx, &lat->sg_out_pos, lat->tot_sgA));
      TRY(dev_alloc(ctx, &lat->sg_start_rank, lat->tot_sgN));
      for (int g = 0; g < n_graphs; g++) pi[g] = &sg[g].in_out_pos;
      TRY(upload_slabs(ctx, lat->sg_out_pos, sga, pi));
      for (int g = 0; g < n_graphs; g++) pi[g] = &sg[g].start_rank;
      TRY(upload_slabs(ctx, lat->sg_start_rank, sgn, pi));
    }
    // accept lists in g.accept() order: the kernel turns them into lattice nodes
    std::vector<int32_t> acc_stage((size_t)tc, 0);
    std::vector<int32_t> nacc(B);
    for (int b = 0; b < B; b++) {
      const SG& s = sg[n_graphs == 1 ? 0 : b];
      std::copy(s.acc.begin(), s.acc.end(), acc_stage.begin() + lat->meta_h[b].acc_base);
    }
    TRY(upload(ctx, lat->meta, lat->meta_h.data(), B));
    TRY(upload(ctx, lat->acc_nodes, acc_stage.data(), tc));
    if (!implicit_only) TRY(launch_compose(ctx, lat));
    // exact_ties: rows and accept list in the reference's relaxation / creation order (k_order.cu)
    // ... lazily: only Viterbi paths depend on it, and the sort is the most expensive compose kernel, so it
    // runs before the first gtnb_viterbi_path unless arc ids were handed out first (download / backward)
    lat->order_pending = !implicit_only && ctx->exact_ties;
  }
  *out = lat;
  return GTNB_OK;
bad:
  free_lattice_device(ctx, lat);
  delete lat;
  return rc;
#undef TRY
}

extern "C" {

int gtnb_compose_grad(
    gtnb_ctx* ctx, gtnb_lattice* lat, float* grad_graph_dev, float* grad_emissions_dev,
    int64_t grad_stride) {
  if (!ctx || !lat) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_compose_grad: NULL");
  if (!lat->composed) return fail(ctx, GTNB_ERR_LOGIC, "gtnb_compose_grad: lattice was not composed on the device");
  if (!lat->arc_grad) return fail(ctx, GTNB_ERR_LOGIC, "gtnb_compose_grad: no backward yet");
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  return launch_compose_grad(ctx, lat, grad_graph_dev, grad_emissions_dev, grad_stride);
}

int gtnb_linear_forward(
    gtnb_ctx* ctx, int B, const int32_t* T, int C, const float* emissions_dev,
    int64_t emissions_stride, int tropical, float* scores_dev, float* grad_emissions_dev,
    int64_t grad_stride, const float* deltas_dev, float delta_all) {
  if (!ctx || B < 0 || !T || C <= 0 || !emissions_dev || !scores_dev)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_linear_forward: bad arguments");
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  int32_t* T_dev = nullptr;
  int rc;
  if ((rc = dev_alloc(ctx, &T_dev, B))) return rc;
  if ((rc = upload(ctx, T_dev, T, B))) return rc;
  int maxT = 0;
  for (int b = 0; b < B; b++) maxT = std::max(maxT, T[b]);
  rc = launch_linear_forward(ctx, B, T_dev, maxT, C, emissions_dev, emissions_stride, tropical,
                             scores_dev, grad_emissions_dev, grad_stride, deltas_dev, delta_all);
  dev_free(ctx, T_dev);
  return rc;
}

} // extern "C"
