/*
 * gtnb_criteria.cu -- whole-minibatch criteria: what the reference does with
 * parallelMap(fwd) + parallelMap(bwd) (benchmarks/ctc.cpp:150-165) as ONE call
 * that only enqueues device work: no per-utterance host objects, one pinned
 * staging upload, one small read-back.
 */
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <limits>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "gtnb_internal.h"
#include "gtnb_product.h"

using namespace gtnb;

/* return a nonzero status; what the call holds is released by its CallScope */
#define GTNB_TRY(x)                       \
  do {                                    \
    if (const int rc__ = (x)) return rc__; \
  } while (0)

namespace {
/* GTNB_TIMES=1: wall-clock microseconds between the host-side phases of one gtnb_ctc_loss call (stderr) */
struct PhaseClock {
  bool on;
  std::chrono::steady_clock::time_point t;
  std::string line;
  PhaseClock() : on(std::getenv("GTNB_TIMES") != nullptr), t(std::chrono::steady_clock::now()) {}
  void mark(const char* what) {
    if (!on) return;
    const auto n = std::chrono::steady_clock::now();
    line += std::string(what) + " " + std::to_string(std::chrono::duration_cast<std::chrono::nanoseconds>(n - t).count() / 1000.0) + "  ";
    t = n;
  }
  ~PhaseClock() {
    if (on) std::fprintf(stderr, "[gtnb_ctc_loss us] %s\n", line.c_str());
  }
};

/*
 * A user buffer the call writes: the user's own storage when it is on the device and may be written in place, else
 * scratch that copy_out copies into it once the work is enqueued.  user NULL: scratch only.
 */
struct OutBuf {
  float* user = nullptr;
  int on_device = 0;
  float* dev = nullptr;
  int copy_out(gtnb_ctx* ctx, long long n) const {
    if (user && dev != user && n > 0)
      GTNB_CUDA(ctx, cudaMemcpyAsync(user, dev, sizeof(float) * n,
                                     on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, ctx->stream));
    return GTNB_OK;
  }
};

/*
 * The device resources of one criterion call.  It opens the context's arena, hands out scratch, owns the lattices
 * of the call and remembers the caller's stream.  When it ends, on every return path, it puts ctx->stream back;
 * if the call did not get as far as synchronising its stream (an error mid-way) it waits for the side streams,
 * since nothing may still run there when the buffers go; then it frees the scratch, destroys the lattices and
 * closes the arena.
 */
class CallScope {
 public:
  explicit CallScope(gtnb_ctx* ctx) : ctx_(ctx), stream_(ctx->stream) {
    scratch_.reserve(16); // (one host allocation: the call's enqueue time is part of the step)
    arena_begin(ctx);
  }
  ~CallScope() {
    release();
    arena_end(ctx_);
  }
  CallScope(const CallScope&) = delete;
  CallScope& operator=(const CallScope&) = delete;

  gtnb_ctx* ctx() const { return ctx_; }

  template <typename T>
  int alloc(T** p, long long n) {
    GTNB_TRY(dev_alloc(ctx_, p, n));
    scratch_.push_back(*p);
    return GTNB_OK;
  }
  /* the user's buffer when `alias`, else n elements of scratch */
  template <typename T>
  int borrow(const T* user, bool alias, long long n, T** dev) {
    if (!alias) return alloc(dev, n);
    *dev = const_cast<T*>(user);
    return GTNB_OK;
  }
  /* a user buffer the kernels read: aliased when it is on the device, else scratch filled on the call's stream */
  template <typename T>
  int input(const T* user, int on_device, long long n, T** dev) {
    GTNB_TRY(borrow(user, on_device != 0, n, dev));
    if (!on_device)
      GTNB_CUDA(ctx_, cudaMemcpyAsync(*dev, user, sizeof(T) * n, cudaMemcpyHostToDevice, ctx_->stream));
    return GTNB_OK;
  }
  /* alias = false: scratch even for a device buffer (the kernels need more room than the user's n elements) */
  int output(float* user, int on_device, long long n, OutBuf* out, bool alias = true) {
    *out = OutBuf{user, on_device, nullptr};
    return borrow(user, user && on_device && alias, n, &out->dev);
  }
  /* a slot for a lattice of the call, destroyed with the scope */
  gtnb_lattice*& lattice() {
    lattices_.push_back(nullptr);
    return lattices_.back();
  }
  /* waits for the call's stream, which every route joins its side streams into before its read-back */
  int sync() {
    GTNB_CUDA(ctx_, cudaStreamSynchronize(ctx_->stream));
    synced_ = true;
    return GTNB_OK;
  }
  /* the exact route's retry: everything of the first attempt released, the arena opened afresh */
  void reopen() {
    release();
    arena_end(ctx_);
    arena_begin(ctx_);
  }

 private:
  void release() {
    ctx_->stream = stream_;
    if (!synced_) {
      if (ctx_->copy_stream) cudaStreamSynchronize(ctx_->copy_stream);
      for (cudaStream_t s : ctx_->side_streams) cudaStreamSynchronize(s);
    }
    for (gtnb_lattice* lat : lattices_) gtnb_lattice_destroy(ctx_, lat);
    lattices_.clear();
    for (void* p : scratch_) dev_free(ctx_, p);
    scratch_.clear();
    synced_ = false;
  }

  gtnb_ctx* ctx_;
  cudaStream_t stream_;
  std::vector<void*> scratch_;
  std::deque<gtnb_lattice*> lattices_; // (a deque: the slots handed out stay where they are)
  bool synced_ = false;
};

/* launches inside the block go to stream s; the previous stream is back when it ends */
struct OnStream {
  OnStream(gtnb_ctx* ctx, cudaStream_t s) : ctx_(ctx), prev_(ctx->stream) { ctx->stream = s; }
  ~OnStream() { ctx_->stream = prev_; }
  OnStream(const OnStream&) = delete;
  OnStream& operator=(const OnStream&) = delete;
  gtnb_ctx* ctx_;
  cudaStream_t prev_;
};

/* work enqueued on `side` from here on runs after everything already on the call's stream */
int fork_to(gtnb_ctx* ctx, cudaStream_t side) {
  GTNB_CUDA(ctx, cudaEventRecord(ctx->ev_fork, ctx->stream));
  GTNB_CUDA(ctx, cudaStreamWaitEvent(side, ctx->ev_fork, 0));
  return GTNB_OK;
}

/* the call's stream waits for everything enqueued on `side` so far */
int join_from(gtnb_ctx* ctx, cudaStream_t side) {
  GTNB_CUDA(ctx, cudaEventRecord(ctx->ev_join, side));
  GTNB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
  return GTNB_OK;
}

/* n floats of a user buffer that a host-side route reads: copied out of the device on the call's stream */
int read_to_host(gtnb_ctx* ctx, float* dst, const float* src, int on_device, long long n) {
  if (!on_device) {
    std::memcpy(dst, src, sizeof(float) * n);
    return GTNB_OK;
  }
  GTNB_CUDA(ctx, cudaMemcpyAsync(dst, src, sizeof(float) * n, cudaMemcpyDeviceToHost, ctx->stream));
  GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return GTNB_OK;
}

/*
 * The read-back of a criterion: [den | num | status] in one pinned block, then losses = den - num
 * (subtract, functions.cpp:52).  *needs_exact: some status word is set, a sweep met a non-finite weight.
 */
int read_losses(CallScope& scope, int B, const float* den, const float* num, const int32_t* status, long long n_status,
                float* losses, bool* needs_exact) {
  gtnb_ctx* ctx = scope.ctx();
  GTNB_TRY(readback_reserve(ctx, sizeof(float) * (2ll * B + n_status)));
  float* d = reinterpret_cast<float*>(ctx->readback);
  float* n = d + B;
  int32_t* st = reinterpret_cast<int32_t*>(n + B);
  GTNB_CUDA(ctx, cudaMemcpyAsync(d, den, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
  GTNB_CUDA(ctx, cudaMemcpyAsync(n, num, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
  if (n_status)
    GTNB_CUDA(ctx, cudaMemcpyAsync(st, status, sizeof(int32_t) * n_status, cudaMemcpyDeviceToHost, ctx->stream));
  GTNB_TRY(scope.sync());
  for (int b = 0; b < B; b++) losses[b] = d[b] - n[b];
  for (long long k = 0; k < n_status; k++) *needs_exact |= st[k] != 0;
  return GTNB_OK;
}

/*
 * attempt(fast, &needs_exact) once; when the fast route met a non-finite value, again on the exact route (the
 * materialised lattices reproduce the reference's inf / NaN propagation arc by arc, shortest.cpp:62-80; the
 * implicit sweeps cannot tell a missing node from one whose score is -inf).
 */
template <class Attempt>
int with_exact_retry(CallScope& scope, bool fast, Attempt&& attempt) {
  bool needs_exact = false;
  int rc = attempt(fast, &needs_exact);
  if (rc == GTNB_OK && needs_exact) {
    scope.reopen();
    rc = attempt(false, &needs_exact);
  }
  return rc;
}

/*
 * The targets of a batch, checked: target_lens[b] >= 0, targets set when some target is non-empty, T_b (input_lens[b],
 * else T) in [0, T].  Labels are classified, not checked: in_range[b] says whether every label of utterance b lies in
 * [0, C).
 */
struct Targets {
  int B = 0;
  long long tot_t = 0;
  int maxT = 0;
  const int32_t* labels = nullptr; // the caller's targets, concatenated
  std::vector<int32_t> meta; // [offsets | lens | T]
  std::vector<int> skips; // consecutive labels that differ: the CTC graph's skip arcs
  std::vector<char> in_range;
  const int32_t* off() const { return meta.data(); }
  const int32_t* lens() const { return meta.data() + B; }
  const int32_t* T() const { return meta.data() + 2ll * B; }
  const int32_t* labels_of(int b) const { return labels + off()[b]; }
  /* [targets | offsets | lens | T]: what the device builders read, in ONE copy (each small copy costs microseconds
   * of stream latency) */
  std::vector<int32_t> packed() const {
    std::vector<int32_t> p((size_t)(tot_t + 3ll * B));
    if (tot_t) std::memcpy(p.data(), labels, sizeof(int32_t) * tot_t);
    std::memcpy(p.data() + tot_t, meta.data(), sizeof(int32_t) * 3 * B);
    return p;
  }
};

int parse_targets(gtnb_ctx* ctx, const char* fn, int B, int T, int C, const int32_t* input_lens,
                  const int32_t* targets, const int32_t* target_lens, Targets* t) {
  t->B = B;
  t->labels = targets;
  t->meta.resize(3 * (size_t)B);
  t->skips.resize(B);
  t->in_range.resize(B);
  int32_t* off = t->meta.data();
  long long tot_t = 0;
  for (int b = 0; b < B; b++) {
    const int U = target_lens[b];
    if (U < 0) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, std::string(fn) + ": negative target length");
    if (U > 0 && !targets) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, std::string(fn) + ": targets is NULL");
    const int32_t* y = targets + tot_t;
    off[b] = (int32_t)tot_t;
    off[B + b] = U;
    tot_t += U;
    int skips = 0;
    int valid = U == 0 || (unsigned)y[0] < (unsigned)C; // (an int: a bool keeps the loop from vectorising)
    for (int u = 1; u < U; u++) { // one pass: skip arcs exist where consecutive labels differ; labels in [0, C)
      skips += y[u] != y[u - 1];
      valid &= (unsigned)y[u] < (unsigned)C;
    }
    t->skips[b] = skips;
    t->in_range[b] = valid;
    const int Tb = input_lens ? input_lens[b] : T;
    if (Tb < 0 || Tb > T) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, std::string(fn) + ": input_lens outside [0, T]");
    off[2ll * B + b] = Tb;
    t->maxT = std::max(t->maxT, Tb);
  }
  t->tot_t = tot_t;
  return GTNB_OK;
}

/* a graph built on the host, ilabel = olabel, kept alive while the lattices built from its view are */
struct HostGraph {
  std::vector<uint8_t> flags;
  std::vector<int32_t> src, dst, label;
  std::vector<float> w; // empty: every weight 0
  void arc(int s, int d, int l, float weight) {
    src.push_back(s);
    dst.push_back(d);
    label.push_back(l);
    w.push_back(weight);
  }
  gtnb_graph_view view() const {
    gtnb_graph_view v;
    std::memset(&v, 0, sizeof(v));
    v.num_nodes = (int)flags.size();
    v.num_arcs = (int)src.size();
    v.node_flags = flags.data();
    v.arc_src = src.data();
    v.arc_dst = dst.data();
    v.arc_ilabel = v.arc_olabel = label.data();
    v.weights = w.empty() ? nullptr : w.data();
    return v;
  }
};

/*
 * The numerator graph of CTC for U labels: 2U+1 nodes; arcs = self loops + step arcs + skip arcs
 * (benchmarks/ctc.cpp:40-58), skip arcs exist where consecutive labels differ (`skips` of them).  all_valid: every
 * label and the blank lie in [0, C).
 */
SgDims ctc_num_dims(int U, int skips, int all_valid) {
  const int L = 2 * U + 1;
  return SgDims{L, L + (L - 1) + skips, L >= 2 ? 2 : 1, all_valid, /*uniform=*/1, /*max_in=*/3, /*max_out=*/3};
}

/*
 * One attempt.  allow_implicit: sweep the frames without building the lattice (k_implicit.cu)
 * when the target graphs qualify; *needs_exact is set when that sweep met a non-finite weight,
 * in which case the outputs are not to be used and the caller repeats the call materialised.
 * dtype: the element type of emissions and grads (GTNB_BF16 / GTNB_F16: both on the device).  16-bit buffers go to
 * k_bidir.cu as they are when the batch takes it; otherwise the emissions are widened into float32 scratch, the
 * float32 route runs on that, and its gradient is rounded into grads.
 */
int ctc_loss_run(
    CallScope& scope, int B, int T, int C, const void* emissions_in, int emissions_on_device,
    const int32_t* input_lens, const int32_t* targets, const int32_t* target_lens, int blank,
    float* losses_host, void* grads_in, int grads_on_device, bool allow_implicit, bool* needs_exact,
    int dtype = GTNB_F32) {
  gtnb_ctx* ctx = scope.ctx();
  const bool half = dtype != GTNB_F32;
  // float32: the caller's buffers; 16-bit: none yet (the route decides below)
  const float* emissions = half ? nullptr : static_cast<const float*>(emissions_in);
  float* grads = half ? nullptr : static_cast<float*>(grads_in);
  *needs_exact = false;
  PhaseClock pc;
  const long long per = (long long)T * C;

  // host: only sizes
  Targets t;
  GTNB_TRY(parse_targets(ctx, "gtnb_ctc_loss", B, T, C, input_lens, targets, target_lens, &t));
  std::vector<SgDims> dims(B);
  for (int b = 0; b < B; b++)
    dims[b] = ctc_num_dims(target_lens[b], t.skips[b], blank >= 0 && blank < C && t.in_range[b]);
  const long long tot_t = t.tot_t;
  const int maxT = t.maxT;
  pc.mark("sizes");

  const bool implicit = allow_implicit && implicit_dims_supported(dims.data(), B);
  // Host buffers: cut the batch into K sub-batches whose H2D copy, kernels and D2H copy run on
  // their own streams, so that the two PCIe directions and the (latency-bound) sweeps overlap.
  // Device buffers: K = 1, and the normaliser (k_linear.cu) runs beside the forward sweep.
  int K = 1; // sub-batches (implicit path with host buffers)
  if (implicit && (!emissions_on_device || (grads && !grads_on_device))) {
    const long long bytes = (long long)sizeof(float) * per * B;
    K = (int)std::min<long long>(std::max<long long>(bytes / (4ll << 20), 1), 16);
    K = std::min(K, B);
  }
  GTNB_TRY(ensure_side_streams(ctx, K, K + 2));
  std::vector<int> chunk_lo(K + 1);
  for (int k = 0; k <= K; k++) chunk_lo[k] = (int)((long long)B * k / K);
  float *e_dev = nullptr, *z_dev = nullptr, *deltas_dev = nullptr;
  float* row_scratch = nullptr; // k_linear.cu's per-frame scores, allocated once for all sub-batches
  float* zparts_dev = nullptr; // k_bidir.cu: forwardScore(emissions) as two partial sums per utterance
  float* boff_dev = nullptr; // k_bidir.cu: per-block score offsets of the two CTAs of every utterance
  float* bidir_scores_dev = nullptr; // k_bidir.cu: the lattices' scores, inside the read-back block
  int32_t* small_dev = nullptr; // [targets | offsets | lens | T]
  int32_t* status_dev = nullptr;
  OutBuf g;
  // host emissions: the copy runs on a second stream while this one builds the target graphs and the
  // lattice structure (k_ctc.cu, compose alive / count / scan need no emissions)
  if (!half) GTNB_TRY(scope.borrow(emissions, emissions_on_device != 0, per * B, &e_dev));
  if (grads) {
    GTNB_TRY(scope.output(grads, grads_on_device, per * B, &g));
    // with full-length utterances the normaliser's gradient overwrites every element
    if (input_lens) GTNB_CUDA(ctx, cudaMemsetAsync(g.dev, 0, sizeof(float) * per * B, ctx->stream));
  }
  GTNB_TRY(scope.alloc(&z_dev, B));
  GTNB_TRY(scope.alloc(&deltas_dev, B));
  GTNB_TRY(scope.alloc(&small_dev, tot_t + 3ll * B));
  std::vector<long long> sgn, sga;
  gtnb_lattice*& lat = scope.lattice();
  GTNB_TRY(composed_alloc(ctx, B, dims.data(), B, 0, t.T(), C, e_dev, per, sgn, sga, &lat, implicit));
  bool native = false; // 16-bit buffers read and written by k_bidir.cu in place
  if (half) {
    native = implicit && ctx->use_bidir && bidir_supported(lat, emissions_in, per, grads_in, per, dtype);
    if (native) {
      // the kernel reads elements of dtype through lat->emissions (only k_bidir.cu runs on this route; e_dev stays
      // NULL, nothing reads float32 emissions)
      lat->emissions = static_cast<const float*>(emissions_in);
      if (grads_in && input_lens) GTNB_CUDA(ctx, cudaMemsetAsync(grads_in, 0, 2ull * per * B, ctx->stream));
    } else {
      float* wide = nullptr;
      GTNB_TRY(scope.alloc(&wide, per * B));
      GTNB_TRY(launch_widen(ctx, emissions_in, dtype, wide, per * B));
      lat->emissions = e_dev = wide;
      if (grads_in) {
        GTNB_TRY(scope.alloc(&g.dev, per * B));
        if (input_lens) GTNB_CUDA(ctx, cudaMemsetAsync(g.dev, 0, sizeof(float) * per * B, ctx->stream));
        grads = g.dev;
      }
    }
  }
  pc.mark("alloc+meta");
  // the whole criterion in one launch per sub-batch (k_bidir.cu) when the batch qualifies
  // (native: true, the 16-bit envelope lies inside the float32 one and the buffers' alignment was checked above)
  const bool bidir = implicit && ctx->use_bidir && bidir_supported(lat, e_dev, per, g.dev, per);
  // PAIR kernels (graphs from the targets, one launch): everything small goes through MAPPED pinned memory --
  // the kernel reads the descriptors and targets in place and writes its results straight into the read-back
  // block; no upload, no memset, no download on the path (those enqueues were a large share of the host work)
  const bool direct = implicit && ctx->use_bidir && ctx->bidir_mode != 0 &&
                      bidir_supported(lat, e_dev, per, g.dev, per) && bidir_takes_targets(lat, blank);
  if (bidir && direct) {
    const long long zpb = 2ll * B * bidir_zparts();
    GTNB_TRY(readback_reserve(ctx, (zpb + 2ll * B) * sizeof(float)));
    zparts_dev = reinterpret_cast<float*>(ctx->readback);
    bidir_scores_dev = zparts_dev + zpb;
    status_dev = reinterpret_cast<int32_t*>(zparts_dev + zpb + B);
    std::memset(status_dev, 0, sizeof(int32_t) * B);
    GTNB_TRY(scope.alloc(&boff_dev, 8ll * B * bidir_blocks(maxT)));
  } else if (bidir) {
    // one block for everything that is read back: [partial sums of forwardScore(e) | lattice scores | status]
    const long long zpb = 2ll * B * bidir_zparts();
    GTNB_TRY(scope.alloc(&zparts_dev, zpb + 2ll * B));
    bidir_scores_dev = zparts_dev + zpb;
    status_dev = reinterpret_cast<int32_t*>(zparts_dev + zpb + B);
    GTNB_TRY(scope.alloc(&boff_dev, 8ll * B * bidir_blocks(maxT)));
    GTNB_CUDA(ctx, cudaMemsetAsync(status_dev, 0, sizeof(int32_t) * B, ctx->stream));
  } else if (implicit) {
    GTNB_TRY(scope.alloc(&row_scratch, (long long)B * std::max(maxT, 1)));
    GTNB_TRY(scope.alloc(&status_dev, B));
    GTNB_CUDA(ctx, cudaMemsetAsync(status_dev, 0, sizeof(int32_t) * B, ctx->stream));
  }

  // one pinned staging pass for everything the kernels need from the host
  const GraphMeta* meta_mapped = nullptr;
  const int32_t* small_mapped = nullptr;
  GTNB_TRY(stage_begin(ctx));
  if (bidir && direct) {
    // the kernel needs the descriptors (with the target offsets) and the labels, nothing else
    void *m = nullptr, *tg = nullptr;
    for (int b = 0; b < B; b++) lat->meta_h[b].tgt_off = t.off()[b];
    GTNB_TRY(stage_reserve(ctx, sizeof(GraphMeta) * B + sizeof(int32_t) * (size_t)tot_t + 1024));
    GTNB_TRY(stage_place(ctx, lat->meta_h.data(), sizeof(GraphMeta) * B, &m));
    GTNB_TRY(stage_place(ctx, targets, sizeof(int32_t) * (size_t)tot_t, &tg));
    meta_mapped = static_cast<const GraphMeta*>(m);
    small_mapped = static_cast<const int32_t*>(tg);
  } else {
    const std::vector<int32_t> small_h = t.packed();
    GTNB_TRY(stage_upload(ctx, lat->meta, lat->meta_h.data(), sizeof(GraphMeta) * B));
    GTNB_TRY(stage_upload(ctx, small_dev, small_h.data(), sizeof(int32_t) * small_h.size()));
  }
  if (!bidir) {
    std::vector<float> minus1(B, -1.0f); // subtract's gradFunc, functions.cpp:53-58
    GTNB_TRY(stage_upload(ctx, deltas_dev, minus1.data(), sizeof(float) * B));
  }
  if (!(bidir && direct)) GTNB_TRY(stage_end(ctx)); // (direct: no copy was issued from the staging buffer; the call synchronises before it returns)
  pc.mark("staging");
  cudaEvent_t h2d_event = nullptr;
  if (!emissions_on_device) {
    // enqueued AFTER the small staged upload: the copy engine serves one direction in
    // submission order, and the graphs must not queue behind 65 MB of emissions
    GTNB_TRY(fork_to(ctx, ctx->copy_stream)); // orders the copy after the allocation
    for (int k = 0; k < K; k++) {
      const long long lo = (long long)chunk_lo[k] * per, n = (long long)(chunk_lo[k + 1] - chunk_lo[k]) * per;
      GTNB_CUDA(ctx, cudaMemcpyAsync(e_dev + lo, emissions + lo, sizeof(float) * n, cudaMemcpyHostToDevice,
                                     ctx->copy_stream));
      GTNB_CUDA(ctx, cudaEventRecord(ctx->side_events[k], ctx->copy_stream));
    }
    GTNB_CUDA(ctx, cudaEventRecord(ctx->ev_join, ctx->copy_stream));
    h2d_event = ctx->ev_join;
  }

  // ctcGraph -> intersect(ctc, emissions) -> forwardScore -> backward(-1) -> compose gradFunc
  // (k_bidir.cu's PAIR kernels take the CTC target graphs from the targets themselves: no tables to build)
  if (!(bidir && direct))
    GTNB_TRY(launch_ctc_build(ctx, lat, small_dev, small_dev + tot_t, small_dev + tot_t + B, blank));
  const int32_t* bidir_targets = direct ? small_mapped : small_dev;
  if (implicit) {
    // everything below only needs what is already enqueued on the main stream (graphs, staging,
    // the memset of the gradients) plus its own slice of the emissions
    cudaEvent_t ev_setup = ctx->side_events[K], ev_lin = ctx->side_events[K + 1];
    const int32_t* T_dev = small_dev + tot_t + 2ll * B;
    GTNB_CUDA(ctx, cudaEventRecord(ev_setup, ctx->stream));
    if (native) {
      GTNB_TRY(launch_bidir_ctc(ctx, lat, status_dev, zparts_dev, boff_dev, grads_in, per, 0, -1, bidir_scores_dev,
                                blank, bidir_targets, bidir_targets + tot_t, direct ? meta_mapped : nullptr, dtype));
    } else if (bidir && K == 1 && !h2d_event && !(grads && !grads_on_device)) {
      GTNB_TRY(launch_bidir_ctc(ctx, lat, status_dev, zparts_dev, boff_dev, g.dev, per, 0, -1, bidir_scores_dev,
                                blank, bidir_targets, bidir_targets + tot_t, direct ? meta_mapped : nullptr));
    } else if (!bidir && K == 1 && !h2d_event && !(grads && !grads_on_device)) {
      // forwardScore(emissions) and its +1 gradient beside the forward sweep
      GTNB_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ev_setup, 0));
      {
        OnStream side(ctx, ctx->copy_stream);
        GTNB_TRY(launch_linear_forward(ctx, B, T_dev, maxT, C, e_dev, per, 0, z_dev, g.dev, per, nullptr, 1.0f,
                                       input_lens ? 0 : 1, row_scratch));
      }
      GTNB_CUDA(ctx, cudaEventRecord(ev_lin, ctx->copy_stream));
      GTNB_TRY(launch_implicit_forward(ctx, lat, status_dev));
      GTNB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ev_lin, 0));
      if (grads) GTNB_TRY(launch_implicit_backward(ctx, lat, deltas_dev, g.dev, per));
    } else {
      for (int k = 0; k < K; k++) {
        const int b0 = chunk_lo[k], nb = chunk_lo[k + 1] - chunk_lo[k];
        cudaStream_t cs = ctx->side_streams[k];
        GTNB_CUDA(ctx, cudaStreamWaitEvent(cs, ev_setup, 0));
        if (h2d_event) GTNB_CUDA(ctx, cudaStreamWaitEvent(cs, ctx->side_events[k], 0));
        {
          OnStream side(ctx, cs);
          if (bidir) {
            GTNB_TRY(launch_bidir_ctc(ctx, lat, status_dev, zparts_dev, boff_dev, g.dev, per, b0, nb, bidir_scores_dev,
                                      blank, bidir_targets, bidir_targets + tot_t, direct ? meta_mapped : nullptr));
          } else {
            GTNB_TRY(launch_linear_forward(ctx, nb, T_dev + b0, maxT, C, e_dev + (long long)b0 * per, per, 0,
                                           z_dev + b0, g.dev ? g.dev + (long long)b0 * per : nullptr, per, nullptr,
                                           1.0f, input_lens ? 0 : 1,
                                           row_scratch + (long long)b0 * std::max(maxT, 1)));
            GTNB_TRY(launch_implicit_forward(ctx, lat, status_dev, b0, nb));
            if (grads) GTNB_TRY(launch_implicit_backward(ctx, lat, deltas_dev, g.dev, per, b0, nb));
          }
        }
        if (grads && !grads_on_device)
          GTNB_CUDA(ctx, cudaMemcpyAsync(grads + (long long)b0 * per, g.dev + (long long)b0 * per,
                                         sizeof(float) * per * nb, cudaMemcpyDeviceToHost, cs));
        GTNB_CUDA(ctx, cudaEventRecord(ctx->side_events[k], cs));
        GTNB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->side_events[k], 0));
      }
    }
  } else {
    GTNB_TRY(launch_compose(ctx, lat, h2d_event));
    // forwardScore(emissions) and its +1 gradient
    GTNB_TRY(launch_linear_forward(ctx, B, small_dev + tot_t + 2ll * B, maxT, C, e_dev, per, 0, z_dev, g.dev,
                                   per, nullptr, 1.0f, input_lens ? 0 : 1));
    GTNB_TRY(launch_forward(ctx, lat, MODE_LOG));
    lat->forward_done = true;
    lat->forward_mode = MODE_LOG;
  }
  if (grads && !implicit) {
    // shortestDistanceGrad and compose's gradFunc fused when the lattice qualifies
    const int rc = launch_backward_fused(ctx, lat, deltas_dev, g.dev, per);
    if (rc == GTNB_ERR_UNSUPPORTED) {
      if (!lat->arc_grad) GTNB_TRY(dev_alloc(ctx, &lat->arc_grad, lat->tot_A));
      GTNB_TRY(launch_backward(ctx, lat, 0, deltas_dev));
      GTNB_TRY(launch_compose_grad(ctx, lat, nullptr, g.dev, per));
    } else {
      GTNB_TRY(rc);
    }
    GTNB_TRY(g.copy_out(ctx, per * B));
  }
  // 16-bit, widened: the float32 gradient rounded into the caller's buffer
  if (half && !native && grads_in) GTNB_TRY(launch_narrow(ctx, g.dev, grads_in, dtype, per * B));
  pc.mark("launches");
  const int zp = bidir ? 2 * bidir_zparts() : 1; // partial sums of forwardScore(emissions) per utterance
  GTNB_TRY(readback_reserve(ctx, (zp + 2) * sizeof(float) * B));
  float* z = reinterpret_cast<float*>(ctx->readback);
  float* s = z + (long long)zp * B;
  int32_t* st = reinterpret_cast<int32_t*>(s + B);
  if (bidir && direct) {
    // the kernel wrote straight into this block
  } else if (bidir) { // one copy: the block is laid out like the host buffer
    GTNB_CUDA(ctx, cudaMemcpyAsync(z, zparts_dev, sizeof(float) * (zp + 2) * B, cudaMemcpyDeviceToHost, ctx->stream));
  } else {
    GTNB_CUDA(ctx, cudaMemcpyAsync(z, z_dev, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    GTNB_CUDA(ctx, cudaMemcpyAsync(s, lat->out_scores, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    if (implicit)
      GTNB_CUDA(ctx, cudaMemcpyAsync(st, status_dev, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, ctx->stream));
  }
  pc.mark("readback enqueue");
  GTNB_TRY(scope.sync());
  pc.mark("sync");
  for (int b = 0; b < B; b++) { // subtract, functions.cpp:52
    float zb = 0.0f;
    for (int k = 0; k < zp; k++) zb += z[(long long)zp * b + k];
    losses_host[b] = zb - s[b];
  }
  if (implicit)
    for (int b = 0; b < B; b++)
      if (st[b]) *needs_exact = true;
  return GTNB_OK;
}

} // namespace

extern "C" int gtnb_ctc_loss(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
    const int32_t* input_lens, const int32_t* targets, const int32_t* target_lens, int blank,
    float* losses_host, float* grads, int grads_on_device) {
  if (!ctx || B < 0 || T < 0 || C <= 0 || !emissions || !target_lens || !losses_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctc_loss: bad arguments");
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  CallScope scope(ctx);
  return with_exact_retry(scope, ctx->use_implicit, [&](bool implicit, bool* needs_exact) {
    return ctc_loss_run(scope, B, T, C, emissions, emissions_on_device, input_lens, targets, target_lens, blank,
                        losses_host, grads, grads_on_device, implicit, needs_exact);
  });
}

extern "C" int gtnb_ctc_loss_ex(
    gtnb_ctx* ctx, int B, int T, int C, const void* emissions_dev, int dtype, const int32_t* input_lens,
    const int32_t* targets, const int32_t* target_lens, int blank, float* losses_host, void* grads_dev) {
  if (dtype != GTNB_F32 && dtype != GTNB_BF16 && dtype != GTNB_F16)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctc_loss_ex: unknown dtype");
  if (dtype == GTNB_F32)
    return gtnb_ctc_loss(ctx, B, T, C, static_cast<const float*>(emissions_dev), 1, input_lens, targets, target_lens,
                         blank, losses_host, static_cast<float*>(grads_dev), 1);
  if (!ctx || B < 0 || T < 0 || C <= 0 || !emissions_dev || !target_lens || !losses_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctc_loss_ex: bad arguments");
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  CallScope scope(ctx);
  return with_exact_retry(scope, ctx->use_implicit, [&](bool implicit, bool* needs_exact) {
    return ctc_loss_run(scope, B, T, C, emissions_dev, 1, input_lens, targets, target_lens, blank, losses_host,
                        grads_dev, 1, implicit, needs_exact, dtype);
  });
}

namespace {

/*
 * The context's arena pointed at a caller's block for one asynchronous call (base NULL: sizing only, nothing is
 * launched).  dev_alloc fails once the block is full instead of allocating; the context's own arena is back when the
 * scope ends.
 */
class BorrowedArena {
 public:
  BorrowedArena(gtnb_ctx* ctx, void* base, size_t bytes) : ctx_(ctx), arena_(ctx->arena), cap_(ctx->arena_cap) {
    ctx->arena = static_cast<unsigned char*>(base);
    ctx->arena_cap = bytes;
    ctx->arena_borrowed = true;
    arena_begin(ctx);
  }
  ~BorrowedArena() {
    ctx_->arena_on = false;
    ctx_->arena_borrowed = false;
    ctx_->arena = arena_;
    ctx_->arena_cap = cap_;
  }
  BorrowedArena(const BorrowedArena&) = delete;
  BorrowedArena& operator=(const BorrowedArena&) = delete;
  size_t need() const { return ctx_->arena_need; }

 private:
  gtnb_ctx* ctx_;
  unsigned char* arena_;
  size_t cap_;
};

/*
 * Every asynchronous call is one run(bool launch) after its argument checks: the call's scratch taken from the arena
 * and, when launch, its work enqueued.  async_workspace sizes it: the bytes run(false) takes from an unbounded arena,
 * 0 for an empty batch.
 */
template <class Run>
int async_workspace(gtnb_ctx* ctx, int B, size_t* bytes, Run&& run) {
  *bytes = 0;
  if (B == 0) return GTNB_OK;
  BorrowedArena arena(ctx, nullptr, std::numeric_limits<size_t>::max());
  GTNB_TRY(run(false));
  *bytes = arena.need();
  return GTNB_OK;
}

/*
 * async_enqueue runs it on the caller's stream (NULL is the default stream, like any stream handle) with its scratch
 * in the caller's workspace.  A non-NULL workspace must be 256-byte aligned; a NULL one has 0 bytes, so the first
 * scratch a call takes from it fails with "workspace too small".
 */
template <class Run>
int async_enqueue(gtnb_ctx* ctx, const std::string& fn, int B, void* cuda_stream, void* workspace, size_t bytes,
                  Run&& run) {
  if ((uintptr_t)workspace & 255) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": workspace not 256-byte aligned");
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  BorrowedArena arena(ctx, workspace, workspace ? bytes : 0);
  OnStream on(ctx, static_cast<cudaStream_t>(cuda_stream));
  return run(true);
}

/* an output buffer to a sizing run, which tests it for presence only */
alignas(16) float stand_in[4];

struct CtcAsyncArgs {
  int B, T, C, S, dtype;
  const void* emissions;
  const int32_t *input_lens, *targets, *target_lens;
  int blank;
  float* losses;
  int32_t* status;
  void* grads;
};

/*
 * gtnb_ctc_loss_async's run.  The route is ctc_loss_run's for a batch at the bounds (every utterance U = S, T_b = T,
 * S - 1 skip arcs), decided from the bounds, the dtype, the buffers' alignment and the context's flags; the prepare kernel
 * then writes every utterance's own descriptor over the bound-uniform slabs.  Sizing passes NULL buffers: a 16-bit
 * batch is then sized for the widened route, which needs more scratch than reading the buffers in place.
 */
int ctc_async_run(gtnb_ctx* ctx, const CtcAsyncArgs& a, bool launch) {
  const int B = a.B, T = a.T, C = a.C, S = a.S;
  const bool half = a.dtype != GTNB_F32;
  const long long per = (long long)T * C;
  if (!ctx->use_implicit)
    return fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_ctc_loss_async: the \"implicit\" flag is off (materialised route)");
  if (a.blank < 0 || a.blank >= C) return fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_ctc_loss_async: blank outside [0, C)");
  const std::vector<SgDims> dims(B, ctc_num_dims(S, std::max(S - 1, 0), /*all_valid=*/1));
  if (!implicit_dims_supported(dims.data(), B))
    return fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_ctc_loss_async: bounds outside the implicit sweeps");
  const std::vector<int32_t> Tv(B, T);
  std::vector<long long> sgn, sga;
  gtnb_lattice* lat_raw = nullptr;
  GTNB_TRY(composed_alloc(ctx, B, dims.data(), B, 0, Tv.data(), C, static_cast<const float*>(a.emissions), per, sgn,
                          sga, &lat_raw, true));
  const std::unique_ptr<gtnb_lattice> lat(lat_raw); // (its device buffers lie in the arena: nothing to free)
  int32_t *small = nullptr, *valid = nullptr, *kstatus = nullptr;
  float* deltas = nullptr;
  GTNB_TRY(dev_alloc(ctx, &small, 3ll * B));
  GTNB_TRY(dev_alloc(ctx, &valid, B));
  GTNB_TRY(dev_alloc(ctx, &kstatus, B));
  GTNB_TRY(dev_alloc(ctx, &deltas, B));
  // 16-bit buffers in place when k_bidir.cu takes them, else widened into float32 scratch (ctc_loss_run's rule)
  const bool native = half && a.emissions && ctx->use_bidir &&
                      bidir_supported(lat.get(), a.emissions, per, a.grads, per, a.dtype);
  const float* e = static_cast<const float*>(a.emissions);
  float* g = static_cast<float*>(a.grads);
  if (half && !native) {
    float* wide = nullptr;
    GTNB_TRY(dev_alloc(ctx, &wide, per * B));
    lat->emissions = e = wide;
    if (a.grads) GTNB_TRY(dev_alloc(ctx, &g, per * B));
  }
  const bool bidir = ctx->use_bidir && (native || bidir_supported(lat.get(), e, per, g, per));
  const bool direct = bidir && ctx->bidir_mode != 0 && bidir_takes_targets(lat.get(), a.blank);
  // [partial sums of forwardScore(e) | lattice scores] and the block offsets of k_bidir.cu, or the normaliser's
  // scores and per-frame rows of the sweeps; sizing takes both, since the alignment of the buffers decides
  float *z = nullptr, *s = nullptr, *boff = nullptr, *rows = nullptr;
  const int zp = bidir ? 2 * bidir_zparts() : 1;
  if (bidir || !launch) {
    GTNB_TRY(dev_alloc(ctx, &z, 2ll * bidir_zparts() * B + B));
    s = z + (long long)zp * B;
    GTNB_TRY(dev_alloc(ctx, &boff, 8ll * B * bidir_blocks(T)));
  }
  if (!bidir || !launch) {
    GTNB_TRY(dev_alloc(ctx, &z, B));
    GTNB_TRY(dev_alloc(ctx, &rows, (long long)B * std::max(T, 1)));
    s = lat->out_scores;
  }
  if (!launch) return GTNB_OK;

  // the gradient the kernels write: the caller's (float32, or 16-bit in place) or the float32 scratch of the widened
  // route, which launch_narrow rounds into the caller's at the end
  void* gk = native ? a.grads : static_cast<void*>(g);
  const long long row_words = native ? per / 2 : per;
  if (gk && a.input_lens) GTNB_CUDA(ctx, cudaMemsetAsync(gk, 0, 4ull * row_words * B, ctx->stream));
  if (half && !native) GTNB_TRY(launch_widen(ctx, a.emissions, a.dtype, const_cast<float*>(e), per * B));
  GTNB_TRY(launch_ctc_async_prepare(ctx, B, S, T, C, lat->meta_h[0], lat->meta_h[B > 1 ? 1 : 0], a.input_lens,
                                    a.targets, a.target_lens, lat->meta, small, deltas, valid, kstatus));
  if (!direct) GTNB_TRY(launch_ctc_build(ctx, lat.get(), a.targets, small, small + B, a.blank));
  if (bidir) {
    GTNB_TRY(launch_bidir_ctc(ctx, lat.get(), kstatus, z, boff, gk, per, 0, -1, s, a.blank, a.targets, small, nullptr,
                              native ? a.dtype : GTNB_F32));
  } else {
    GTNB_TRY(launch_linear_forward(ctx, B, small + 2ll * B, T, C, e, per, 0, z, g, per, nullptr, 1.0f,
                                   a.input_lens ? 0 : 1, rows));
    GTNB_TRY(launch_implicit_forward(ctx, lat.get(), kstatus));
    if (g) GTNB_TRY(launch_implicit_backward(ctx, lat.get(), deltas, g, per));
  }
  GTNB_TRY(launch_ctc_async_finalize(ctx, B, zp, z, s, kstatus, valid, a.losses, a.status, gk, row_words));
  if (half && !native && a.grads) GTNB_TRY(launch_narrow(ctx, g, a.grads, a.dtype, per * B));
  return GTNB_OK;
}

bool ctc_async_dtype(int dtype) { return dtype == GTNB_F32 || dtype == GTNB_BF16 || dtype == GTNB_F16; }

} // namespace

extern "C" int gtnb_ctc_loss_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int S, int dtype, int with_grad,
                                             size_t* bytes) {
  if (!ctx || B < 0 || T < 0 || C <= 0 || S < 0 || !bytes)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctc_loss_async_workspace: bad arguments");
  if (!ctc_async_dtype(dtype)) return fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_ctc_loss_async_workspace: unknown dtype");
  const CtcAsyncArgs a{B, T, C, S, dtype, nullptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr,
                       with_grad ? stand_in : nullptr};
  return async_workspace(ctx, B, bytes, [&](bool launch) { return ctc_async_run(ctx, a, launch); });
}

extern "C" int gtnb_ctc_loss_async(
    gtnb_ctx* ctx, void* cuda_stream, int B, int T, int C, int S, const void* emissions_dev, int dtype,
    const int32_t* input_lens_dev, const int32_t* targets_dev, const int32_t* target_lens_dev, int blank,
    float* losses_dev, int32_t* status_dev, void* grads_dev, void* workspace_dev, size_t workspace_bytes) {
  if (!ctx || B < 0 || T < 0 || C <= 0 || S < 0 || !emissions_dev || (S > 0 && !targets_dev) || !target_lens_dev ||
      !losses_dev)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctc_loss_async: bad arguments");
  if (!ctc_async_dtype(dtype)) return fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_ctc_loss_async: unknown dtype");
  const CtcAsyncArgs a{B, T, C, S, dtype, emissions_dev, input_lens_dev, targets_dev, target_lens_dev, blank,
                       losses_dev, status_dev, grads_dev};
  return async_enqueue(ctx, "gtnb_ctc_loss_async", B, cuda_stream, workspace_dev, workspace_bytes,
                       [&](bool launch) { return ctc_async_run(ctx, a, launch); });
}

namespace {

/* the transition weights of a dense kind: ASG [s | W] (C + C*C), BIGRAM W (C*C) */
long long dense_trans_count(bool bigram, int C) { return (bigram ? 0 : (long long)C) + (long long)C * C; }

/*
 * The body of gtnb_viterbi_dense and gtnb_viterbi_dense_ex: viterbiPath / viterbiScore of the lattice of every
 * utterance through the factored kernel (k_dense.cu); the T*C*C lattice is never materialised.  Host transitions
 * and input_lens go up in one staged copy; device transitions are read where they are.  Outputs on the device are
 * written in place and the call returns once the work is enqueued; host outputs are copied back and waited for.
 * empty_score: the score of an utterance with T_b = 0.  dtype: the element type behind emissions (GTNB_BF16 / GTNB_F16:
 * a device buffer of that type, which the kernel reads in place).
 * (the device scratch of a call comes from the context's call-scoped arena, as in gtnb_ctc_loss: no stream-ordered
 * allocations on the path after the first call of a shape)
 */
int viterbi_dense_run(gtnb_ctx* ctx, const char* fn, int B, int T, int C, const float* emissions,
                      int emissions_on_device, const int32_t* input_lens, bool bigram, const float* trans_w,
                      int trans_on_device, int32_t* paths, float* scores, int outputs_on_device, float empty_score,
                      int dtype = GTNB_F32) {
  if (!ctx || B < 0 || T < 0 || C <= 0 || !emissions || !trans_w)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, std::string(fn) + ": bad arguments");
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  if (input_lens)
    for (int b = 0; b < B; b++)
      if (input_lens[b] < 0 || input_lens[b] > T)
        return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, std::string(fn) + ": input_lens out of range");
  const long long per = (long long)T * C;
  const long long n_trans = dense_trans_count(bigram, C);
  CallScope scope(ctx);
  float *e_dev = nullptr, *tr_dev = nullptr, *sc_dev = nullptr;
  int32_t *T_dev = nullptr, *paths_dev = nullptr;
  uint8_t* bp = nullptr;
  GTNB_TRY(scope.input(emissions, emissions_on_device, per * B, &e_dev));
  GTNB_TRY(scope.borrow(trans_w, trans_on_device != 0, n_trans, &tr_dev));
  GTNB_TRY(scope.borrow(scores, scores && outputs_on_device, B, &sc_dev));
  GTNB_TRY(scope.borrow(paths, paths && outputs_on_device, (long long)B * std::max(T, 1), &paths_dev));
  GTNB_TRY(scope.alloc(&bp, (long long)B * std::max(T, 1) * dense_bp_pitch(C)));
  if (input_lens) GTNB_TRY(scope.alloc(&T_dev, B));
  GTNB_TRY(stage_begin(ctx));
  if (!trans_on_device) GTNB_TRY(stage_upload(ctx, tr_dev, trans_w, sizeof(float) * n_trans));
  if (input_lens) GTNB_TRY(stage_upload(ctx, T_dev, input_lens, sizeof(int32_t) * B));
  GTNB_TRY(stage_end(ctx));
  GTNB_TRY(launch_viterbi_dense(ctx, B, T, C, bigram, T_dev, e_dev, per, tr_dev, empty_score, bp, paths_dev, sc_dev,
                                dtype));
  if (outputs_on_device) return GTNB_OK;
  if (paths && T > 0)
    GTNB_CUDA(ctx, cudaMemcpyAsync(paths, paths_dev, sizeof(int32_t) * (size_t)B * T, cudaMemcpyDeviceToHost,
                                   ctx->stream));
  if (scores)
    GTNB_CUDA(ctx, cudaMemcpyAsync(scores, sc_dev, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
  return scope.sync();
}

} // namespace

/*
 * viterbiPath(compose(linearGraph(T, C; e_b), transitions)) for a whole minibatch, with the
 * dense transitions graph of test/criterion_test.cpp:244-254 / :316-326: the ASG kind of
 * gtnb_viterbi_dense_ex with host transitions and host outputs, except that T_b = 0 scores 0.
 */
extern "C" int gtnb_viterbi_dense(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
    const int32_t* input_lens, const float* trans_w_host, int32_t* paths_host, float* scores_host) {
  return viterbi_dense_run(ctx, "gtnb_viterbi_dense", B, T, C, emissions, emissions_on_device, input_lens, false,
                           trans_w_host, 0, paths_host, scores_host, 0, 0.0f);
}

extern "C" int gtnb_viterbi_dense_ex(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    int kind, const float* trans_w, int trans_on_device, int32_t* paths, float* scores, int outputs_on_device) {
  if (kind != GTNB_DENSE_ASG && kind != GTNB_DENSE_BIGRAM)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_viterbi_dense_ex: unknown graph kind");
  // T_b = 0: linearGraph(0, C) is one start node that does not accept (creations.cpp:20-33): no path, score -inf
  return viterbi_dense_run(ctx, "gtnb_viterbi_dense_ex", B, T, C, emissions, emissions_on_device, input_lens,
                           kind == GTNB_DENSE_BIGRAM, trans_w, trans_on_device, paths, scores, outputs_on_device,
                           -std::numeric_limits<float>::infinity());
}

extern "C" int gtnb_viterbi_dense_typed(
    gtnb_ctx* ctx, int B, int T, int C, const void* emissions_dev, int dtype, const int32_t* input_lens, int kind,
    const float* trans_w_dev, int32_t* paths_dev, float* scores_dev) {
  if (dtype != GTNB_F32 && dtype != GTNB_BF16 && dtype != GTNB_F16)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_viterbi_dense_typed: unknown dtype");
  if (kind != GTNB_DENSE_ASG && kind != GTNB_DENSE_BIGRAM)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_viterbi_dense_typed: unknown graph kind");
  // (16-bit emissions travel in the float pointer; the kernel reads them as dtype)
  return viterbi_dense_run(ctx, "gtnb_viterbi_dense_typed", B, T, C, static_cast<const float*>(emissions_dev), 1,
                           input_lens, kind == GTNB_DENSE_BIGRAM, trans_w_dev, 1, paths_dev, scores_dev, 1,
                           -std::numeric_limits<float>::infinity(), dtype);
}

namespace {

/* the arguments of gtnb_ngram_ctc_loss, gtnb_asg_loss_ex and (host buffers, blank unused) gtnb_asg_loss */
struct TransitionArgs {
  int B, T, C;
  const float* emissions;
  int emissions_on_device;
  const int32_t* input_lens;
  const float* trans_w;
  int trans_on_device;
  const int32_t* targets;
  const int32_t* target_lens;
  int blank;
  float* losses_host;
  float* grads;
  int grads_on_device;
  float* trans_grad;
  int trans_grad_on_device;
  // the element type behind emissions and grads: GTNB_F32, or (the _typed entry points) GTNB_BF16 / GTNB_F16 for
  // device buffers of that type carried in these pointers, which only trellis_loss_fast and widened read
  int dtype = GTNB_F32;
};

/* n floats on the call's stream, outside its arena: they outlive the scope's reopen() of an exact retry inside a
 * route (asg_loss's), which hands the arena out afresh */
struct StreamFloats {
  gtnb_ctx* ctx;
  float* p = nullptr;
  int alloc(long long n) {
    GTNB_CUDA(ctx, cudaMallocAsync((void**)&p, sizeof(float) * (size_t)std::max(n, 1ll), ctx->stream));
    return GTNB_OK;
  }
  ~StreamFloats() {
    if (p) cudaFreeAsync(p, ctx->stream);
  }
};

/*
 * A route that reads float32 emissions, run for a (a.dtype 16-bit: the emissions widened once into float32 by
 * launch_widen, the route run on them with its gradient in float32, which launch_narrow then rounds into a.grads and
 * the call waits for).  A float32 a goes to the route as it is.
 */
template <class Route>
int widened(CallScope& scope, const TransitionArgs& a, Route&& route) {
  if (a.dtype == GTNB_F32) return route(a);
  gtnb_ctx* ctx = scope.ctx();
  const long long n = (long long)a.B * a.T * a.C;
  TransitionArgs w = a;
  StreamFloats e{ctx}, g{ctx};
  GTNB_TRY(e.alloc(n));
  GTNB_TRY(launch_widen(ctx, a.emissions, a.dtype, e.p, n));
  w.emissions = e.p;
  w.dtype = GTNB_F32;
  if (a.grads) {
    GTNB_TRY(g.alloc(n));
    w.grads = g.p;
  }
  GTNB_TRY(route(w));
  if (!a.grads) return GTNB_OK;
  GTNB_TRY(launch_narrow(ctx, w.grads, a.grads, a.dtype, n));
  return scope.sync();
}

/*
 * gtnb_ngram_ctc_loss, gtnb_asg_loss_ex and gtnb_graph_loss after their argument checks: attempt(scope, fast,
 * &needs_exact) through with_exact_retry.  An empty batch gives a zero transition gradient (n_trans floats).
 * T_b = 0: linearGraph(0, C) is one start node that does not accept (creations.cpp:20-33), so both scores are
 * -inf and the reference's loss is -inf - -inf = NaN (no gradient).
 */
template <class Attempt>
int run_criterion(gtnb_ctx* ctx, int B, const int32_t* Tb, float* losses, float* trans_grad, int trans_grad_on_device,
                  long long n_trans, bool fast, Attempt&& attempt) {
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  if (B == 0) {
    if (trans_grad && trans_grad_on_device) {
      GTNB_CUDA(ctx, cudaMemsetAsync(trans_grad, 0, sizeof(float) * n_trans, ctx->stream));
      GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    } else if (trans_grad) {
      std::memset(trans_grad, 0, sizeof(float) * n_trans);
    }
    return GTNB_OK;
  }
  CallScope scope(ctx);
  GTNB_TRY(with_exact_retry(scope, fast, [&](bool f, bool* needs_exact) { return attempt(scope, f, needs_exact); }));
  for (int b = 0; b < B; b++)
    if (Tb[b] == 0) losses[b] = std::numeric_limits<float>::quiet_NaN();
  return GTNB_OK;
}

/*
 * ASG criterion for a whole minibatch (test/criterion_test.cpp:244-305, examples/asg.cpp:59-81):
 *   loss_b = forwardScore(compose(e_b, transitions))
 *          - forwardScore(compose(compose(fal_b, transitions), e_b))
 * with the dense transitions graph shared by the batch; gradients w.r.t. the emissions and
 * (accumulated over the batch, graph.cpp:96-100) the transitions.  The denominator lattice
 * is materialised on the device (C + (T-1) C^2 arcs per utterance); compose(fal_b,
 * transitions) is a 2U-arc chain built on the host from the target (pure construction).
 * input_lens (nullable: T for every utterance): e_b is linearGraph(T_b, C) on the first T_b rows; the rows of
 * grads beyond T_b are zeroed.  Host transitions and transition gradient.
 */
struct AsgGraphs {
  HostGraph trans; // criterion_test.cpp:244-254
  std::vector<HostGraph> chains; // compose(fal_b, transitions)
  std::vector<gtnb_graph_view> chain_views;
  std::vector<int32_t> map; // transitions arc of every chain arc
};

/*
 * The dense transition graph G of the trellis criteria from host weights, and the trans_w slot of every arc (map,
 * nullable).  ASG (criterion_test.cpp:244-254, w = [s | W]): node 0 starts, nodes 1..C accept, arc i = 0 -> i+1 of
 * weight s[i], arc C + i*C + j = j+1 -> i+1 of weight W[i][j] (arc k reads w[k]).  BIGRAM (benchmarks/ctc.cpp
 * transitionsGraph with a label-determined destination, w = W): C nodes, all start and accept, arc j*C + i = j -> i
 * of weight W[i][j].  The arc into state i carries label i.
 */
void dense_graph(bool bigram, int C, const float* w, HostGraph* G, std::vector<int32_t>* map) {
  const long long n = dense_trans_count(bigram, C);
  G->src.resize(n);
  G->dst.resize(n);
  G->label.resize(n);
  G->w.resize(n);
  if (map) map->resize(n);
  if (bigram) {
    G->flags.assign(C, 3);
    for (int j = 0; j < C; j++)
      for (int i = 0; i < C; i++) {
        const long long k = (long long)j * C + i;
        G->src[k] = j;
        G->dst[k] = i;
        G->label[k] = i;
        G->w[k] = w[(long long)i * C + j];
        if (map) (*map)[k] = i * C + j;
      }
    return;
  }
  G->flags.assign(C + 1, 2);
  G->flags[0] = 1;
  G->w.assign(w, w + n);
  for (int i = 0; i < C; i++) {
    G->src[i] = 0;
    G->dst[i] = i + 1;
    G->label[i] = i;
  }
  for (int i = 0; i < C; i++)
    for (int j = 0; j < C; j++) {
      const int a = C + i * C + j;
      G->src[a] = j + 1;
      G->dst[a] = i + 1;
      G->label[a] = i;
    }
  if (map)
    for (long long k = 0; k < n; k++) (*map)[k] = (int32_t)k;
}

void build_asg_graphs(int C, const float* trans_w_host, const Targets& t, AsgGraphs* g) {
  dense_graph(false, C, trans_w_host, &g->trans, nullptr);
  // compose(fal_b, transitions): node l = "l labels consumed"; arcs: 0->1, then per node a
  // self loop and the step to the next label, in the reference's creation order
  g->chains.resize(t.B);
  g->chain_views.resize(t.B);
  for (int b = 0; b < t.B; b++) {
    const int U = t.lens()[b];
    const int32_t* y = t.labels_of(b);
    HostGraph& f = g->chains[b];
    f.flags.assign(U + 1, 0);
    f.flags[0] |= 1;
    if (U > 0) f.flags[U] |= 2;
    auto add = [&](int s, int d, int lab, int tarc) {
      f.arc(s, d, lab, trans_w_host[tarc]);
      g->map.push_back(tarc);
    };
    if (U > 0) add(0, 1, y[0], y[0]);
    for (int l = 1; l <= U; l++) {
      add(l, l, y[l - 1], C + y[l - 1] * C + y[l - 1]);
      if (l < U) add(l, l + 1, y[l], C + y[l] * C + y[l - 1]);
    }
    g->chain_views[b] = f.view();
  }
}

/* One attempt (see ctc_loss_run); implicit sweeps (k_implicit.cu) when allow_implicit and the graphs qualify. */
int asg_loss_run(CallScope& scope, const TransitionArgs& a, const Targets& t, const AsgGraphs& gr, bool allow_implicit,
                 bool* needs_exact) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = a.B, C = a.C;
  const long long per = (long long)a.T * C, nTrans = C + (long long)C * C, nFt = (long long)gr.map.size();
  const bool want = a.grads || a.trans_grad;
  const gtnb_graph_view tview = gr.trans.view();
  float *e_dev = nullptr, *ft_grad = nullptr, *minus1 = nullptr;
  int32_t *ft_map_dev = nullptr, *status = nullptr;
  OutBuf g, tg;
  gtnb_lattice*& den = scope.lattice();
  gtnb_lattice*& num = scope.lattice();
  GTNB_TRY(scope.input(a.emissions, a.emissions_on_device, per * B, &e_dev));
  if (want) {
    GTNB_TRY(scope.output(a.grads, a.grads_on_device, per * B, &g));
    GTNB_CUDA(ctx, cudaMemsetAsync(g.dev, 0, sizeof(float) * per * B, ctx->stream));
    GTNB_TRY(scope.output(a.trans_grad, 0, nTrans, &tg));
    GTNB_CUDA(ctx, cudaMemsetAsync(tg.dev, 0, sizeof(float) * nTrans, ctx->stream));
    GTNB_TRY(scope.alloc(&ft_grad, std::max<long long>(nFt, 1)));
    GTNB_CUDA(ctx, cudaMemsetAsync(ft_grad, 0, sizeof(float) * std::max<long long>(nFt, 1), ctx->stream));
    GTNB_TRY(scope.alloc(&ft_map_dev, std::max<long long>(nFt, 1)));
    GTNB_TRY(scope.alloc(&minus1, B));
  }
  // implicit sweeps (k_implicit.cu): neither lattice is built; the dense transitions graph takes
  // the G-lanes-per-node kernels, the forced-alignment chains the one-node-per-thread kernels
  bool implicit = allow_implicit;
  if (implicit) {
    int rc = compose_linear_impl(ctx, B, &tview, 1, 1, t.T(), C, e_dev, per, true, &den);
    if (!rc) rc = compose_linear_impl(ctx, B, gr.chain_views.data(), B, 0, t.T(), C, e_dev, per, true, &num);
    if (rc == GTNB_ERR_UNSUPPORTED) {
      gtnb_lattice_destroy(ctx, den);
      den = nullptr;
      implicit = false;
    } else {
      GTNB_TRY(rc);
    }
  }
  if (implicit) {
    GTNB_TRY(ensure_side_streams(ctx, 0, 0));
    GTNB_TRY(scope.alloc(&status, 2ll * B));
    GTNB_CUDA(ctx, cudaMemsetAsync(status, 0, sizeof(int32_t) * 2 * B, ctx->stream));
    // the numerator's sweeps (forced-alignment chains: small) run on the second stream beside the
    // denominator's (dense transitions: wide); they share nothing but the emission gradient, which both
    // accumulate with red.global.add
    GTNB_TRY(fork_to(ctx, ctx->copy_stream));
    GTNB_TRY(launch_implicit_forward(ctx, den, status));
    OnStream side(ctx, ctx->copy_stream);
    GTNB_TRY(launch_implicit_forward(ctx, num, status + B));
  } else {
    GTNB_TRY(gtnb_compose_linear(ctx, B, &tview, 1, 1, t.T(), C, e_dev, per, &den));
    GTNB_TRY(gtnb_compose_linear(ctx, B, gr.chain_views.data(), B, 0, t.T(), C, e_dev, per, &num));
    GTNB_TRY(gtnb_forward(ctx, den, 0, nullptr, nullptr));
    GTNB_TRY(gtnb_forward(ctx, num, 0, nullptr, nullptr));
  }
  if (want) {
    std::vector<float> m1(B, -1.0f);
    if (implicit) {
      GTNB_TRY(stage_begin(ctx));
      GTNB_TRY(stage_upload(ctx, minus1, m1.data(), sizeof(float) * B));
      GTNB_TRY(stage_end(ctx));
      // +1 / -1: subtract's gradFunc (functions.cpp:53-58); graph-side gradients straight into
      // the transitions' (shared by the batch) and the forced-alignment chains' slabs
      GTNB_TRY(fork_to(ctx, ctx->copy_stream)); // the staged -1 seeds
      GTNB_TRY(launch_implicit_backward(ctx, den, nullptr, g.dev, per, 0, -1, tg.dev));
      {
        OnStream side(ctx, ctx->copy_stream);
        GTNB_TRY(launch_implicit_backward(ctx, num, minus1, g.dev, per, 0, -1, ft_grad));
      }
      GTNB_TRY(join_from(ctx, ctx->copy_stream));
    } else {
      GTNB_TRY(gtnb_backward(ctx, den, 0, nullptr)); // +1 (subtract's gradFunc, functions.cpp:53-58)
      GTNB_TRY(gtnb_backward(ctx, num, 0, m1.data())); // -1
      GTNB_TRY(gtnb_compose_grad(ctx, den, tg.dev, g.dev, per));
      GTNB_TRY(gtnb_compose_grad(ctx, num, ft_grad, g.dev, per));
    }
    if (nFt) {
      GTNB_TRY(stage_begin(ctx));
      GTNB_TRY(stage_upload(ctx, ft_map_dev, gr.map.data(), sizeof(int32_t) * nFt));
      GTNB_TRY(stage_end(ctx));
      GTNB_TRY(launch_scatter_add(ctx, tg.dev, ft_map_dev, ft_grad, nFt));
    }
    GTNB_TRY(g.copy_out(ctx, per * B));
    GTNB_TRY(tg.copy_out(ctx, nTrans));
  } else if (implicit) { // loss only: the numerator's forward sweep is still on the second stream
    GTNB_TRY(join_from(ctx, ctx->copy_stream));
  }
  return read_losses(scope, B, den->out_scores, num->out_scores, status, implicit ? 2ll * B : 0, a.losses_host,
                     needs_exact);
}

/* a.targets checked into t; a non-finite weight met by the implicit sweeps repeats the call materialised */
int asg_loss(CallScope& scope, const TransitionArgs& a, const Targets& t) {
  AsgGraphs gr;
  build_asg_graphs(a.C, a.trans_w, t, &gr);
  return with_exact_retry(scope, scope.ctx()->use_implicit, [&](bool implicit, bool* needs_exact) {
    return asg_loss_run(scope, a, t, gr, implicit, needs_exact);
  });
}

} // namespace

extern "C" int gtnb_asg_loss(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
    const float* trans_w_host, const int32_t* targets, const int32_t* target_lens,
    float* losses_host, float* grads, int grads_on_device, float* trans_grad_host) {
  const TransitionArgs a{B, T, C, emissions, emissions_on_device, nullptr, trans_w_host, 0, targets, target_lens,
                         -1, losses_host, grads, grads_on_device, trans_grad_host, 0};
  if (!ctx || B < 0 || T < 0 || C <= 0 || !emissions || !trans_w_host || !target_lens || !losses_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss: bad arguments");
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  Targets t;
  GTNB_TRY(parse_targets(ctx, "gtnb_asg_loss", B, T, C, nullptr, targets, target_lens, &t));
  for (int b = 0; b < B; b++)
    if (!t.in_range[b]) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss: label out of range");
  CallScope scope(ctx);
  return asg_loss(scope, a, t);
}

namespace {

/*
 * The trellis criteria: CTC with a learned bigram transition graph G (gtnb_ngram_ctc_loss) and ASG with per-utterance
 * frame counts and device-resident transitions (gtnb_asg_loss_ex), on their device route (k_ngram.cu).  The
 * numerator graphs are built on the device from the targets and the transitions and swept by k_implicit.cu on the
 * second stream; the dense trellis of the denominator runs on the context's stream.  Both add their emission
 * gradients into the zero-filled rows with red.add; the numerator's arc gradients are scattered into the transition
 * gradient after the streams join.  *needs_exact: a non-finite weight was met.
 */
struct TrellisCriterion {
  long long n_trans; // floats of trans_w and trans_grad
  long long alpha_floats; // of the denominator's alpha buffer
  // n-gram: the numerator's start arcs carry sigma_i = logsumexp_j W[i][j] (launch_ngram_sigma), whose gradient C
  // extra slots after W's collect and launch_ngram_fold folds into W's; the gradient is then never built in place
  bool fold;
  decltype(&launch_ngram_den_forward) den_forward;
  decltype(&launch_ngram_den_backward) den_backward;
  float* alpha = nullptr;
  int dtype = GTNB_F32; // the element type of the emissions the sweeps read (GTNB_F32 / GTNB_BF16 / GTNB_F16)

  /*
   * The interface of trellis_loss_fast's denominators: n_sigma (the folded start weights, 0 without a fold), alloc
   * (scratch), stage (uploads in the call's one staging pass), sigma (the folded start weights from the transitions
   * on the device), forward / backward (the sweeps; the backward adds into the zero-filled emission rows and the
   * transition gradient), fold (the sigma slots of the gradient into the transitions').
   */
  long long n_sigma(int C) const { return fold ? C : 0; }
  int alloc(CallScope& scope, int /*B*/, int /*T*/) { return scope.alloc(&alpha, alpha_floats); }
  int stage(CallScope&) { return GTNB_OK; }
  int sigma(gtnb_ctx* ctx, int C, const float* w, float* sig) { return launch_ngram_sigma(ctx, C, w, sig); }
  int forward(gtnb_ctx* ctx, int B, int T, int C, const int32_t* lens, const float* e, long long per, const float* w,
              float* den, int32_t* status) {
    return den_forward(ctx, B, T, C, lens, e, per, w, alpha, den, status, dtype);
  }
  int backward(gtnb_ctx* ctx, int B, int T, int C, const int32_t* lens, const float* e, long long per, const float* w,
               const float* den, float* grad, float* wgrad) {
    return den_backward(ctx, B, T, C, lens, e, per, w, alpha, den, grad, per, wgrad, dtype);
  }
  int fold_grad(gtnb_ctx* ctx, int C, const float* w, const float* sig, float* wgrad) {
    return launch_ngram_fold(ctx, C, w, sig, wgrad);
  }
};

/*
 * The numerator of gtnb_ngram_ctc_loss / gtnb_asg_loss_ex: graphs built on the device from the targets
 * (launch_ngram_num_build / launch_asg_num_build) straight into the small-graph tables of an implicit lattice.
 * The interface of trellis_loss_fast's numerators: alloc (scratch and, where it can, the lattice), stage (uploads in
 * the call's one staging pass), build (on the call's stream once the transitions and sigma are there), T_dev (the
 * frame counts), map (the transition slot of every numerator arc, tot_A of them), scatter (the arc gradient's
 * other destinations).
 */
struct TargetsNumerator {
  using Build = int (*)(gtnb_ctx*, gtnb_lattice*, const int32_t*, const int32_t*, const int32_t*, int, const float*,
                        const float*, int32_t*);
  const Targets& t;
  const std::vector<SgDims>& dims;
  int C;
  Build build_kernel;
  int blank;
  long long tot_A = 0;
  std::vector<int32_t> small_h;
  int32_t *small_dev = nullptr, *map = nullptr;

  bool wants_arc_grads() const { return false; }
  int alloc(CallScope& scope, const float* e_dev, long long per, gtnb_lattice** lat) {
    std::vector<long long> sgn, sga;
    tot_A = 0;
    for (int b = 0; b < t.B; b++) tot_A += dims[b].A;
    small_h = t.packed();
    GTNB_TRY(scope.alloc(&small_dev, (long long)small_h.size()));
    GTNB_TRY(scope.alloc(&map, tot_A));
    return composed_alloc(scope.ctx(), t.B, dims.data(), t.B, 0, t.T(), C, e_dev, per, sgn, sga, lat, true);
  }
  int stage(CallScope& scope, gtnb_lattice* lat) {
    GTNB_TRY(stage_upload(scope.ctx(), lat->meta, lat->meta_h.data(), sizeof(GraphMeta) * t.B));
    return stage_upload(scope.ctx(), small_dev, small_h.data(), sizeof(int32_t) * small_h.size());
  }
  const int32_t* T_dev() const { return small_dev + t.tot_t + 2ll * t.B; }
  int build(CallScope& scope, gtnb_lattice*& lat, const float* w_dev, const float* sigma) {
    return build_kernel(scope.ctx(), lat, small_dev, small_dev + t.tot_t, small_dev + t.tot_t + t.B, blank, w_dev,
                        sigma, map);
  }
  int scatter(CallScope&, const float*) { return GTNB_OK; }
};

/*
 * 16-bit a (a.dtype, the native route; the denominator k reads the same type): both sweeps read the caller's emissions
 * in place, add their gradients into float32 scratch as for float32, and narrow_kernel rounds that into a.grads once
 * the streams have joined.
 */
template <class Numerator, class Denominator>
int trellis_loss_fast(CallScope& scope, Denominator& k, const TransitionArgs& a, Numerator& num, bool* needs_exact) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = a.B, T = a.T, C = a.C;
  const long long per = (long long)T * C;
  const long long n_sigma = k.n_sigma(C);
  const bool want = a.grads || a.trans_grad || num.wants_arc_grads();
  const bool half = a.dtype != GTNB_F32;
  float *e_dev = nullptr, *w_dev = nullptr, *sigma = nullptr, *den = nullptr;
  float *ggrad = nullptr, *minus1 = nullptr;
  int32_t* status = nullptr;
  OutBuf g, tg;
  std::vector<float> m1(B, -1.0f);
  gtnb_lattice*& lat = scope.lattice();

  GTNB_TRY(ensure_side_streams(ctx, 0, 0));
  GTNB_TRY(scope.input(a.emissions, a.emissions_on_device, per * B, &e_dev));
  GTNB_TRY(scope.borrow(a.trans_w, a.trans_on_device != 0, k.n_trans, &w_dev)); // (host: staged below)
  GTNB_TRY(scope.alloc(&status, 2ll * B));
  if (n_sigma) GTNB_TRY(scope.alloc(&sigma, n_sigma));
  GTNB_TRY(k.alloc(scope, B, T));
  GTNB_TRY(scope.alloc(&den, B));
  GTNB_TRY(num.alloc(scope, e_dev, per, &lat));
  if (half) lat->dtype = a.dtype; // (16-bit: the targets' numerators only, whose alloc makes the lattice)
  const long long tot_A = num.tot_A;
  if (want) {
    const long long n_grad = k.n_trans + n_sigma; // [d/dtrans | d/dsigma]
    GTNB_TRY(scope.output(half ? nullptr : a.grads, a.grads_on_device, per * B, &g));
    GTNB_TRY(scope.output(a.trans_grad, a.trans_grad_on_device, n_grad, &tg, /*alias=*/!n_sigma));
    GTNB_TRY(scope.alloc(&ggrad, tot_A));
    GTNB_TRY(scope.alloc(&minus1, B));
    GTNB_CUDA(ctx, cudaMemsetAsync(g.dev, 0, sizeof(float) * per * B, ctx->stream));
    GTNB_CUDA(ctx, cudaMemsetAsync(tg.dev, 0, sizeof(float) * n_grad, ctx->stream));
    if (tot_A) GTNB_CUDA(ctx, cudaMemsetAsync(ggrad, 0, sizeof(float) * tot_A, ctx->stream));
  }
  GTNB_CUDA(ctx, cudaMemsetAsync(status, 0, sizeof(int32_t) * 2 * B, ctx->stream));
  // one pinned staging pass: the numerator's (descriptors, [targets | offsets | lens | T] or the product maps), the
  // transitions from the host, the -1 seeds
  GTNB_TRY(stage_begin(ctx));
  GTNB_TRY(num.stage(scope, lat));
  GTNB_TRY(k.stage(scope));
  if (!a.trans_on_device) GTNB_TRY(stage_upload(ctx, w_dev, a.trans_w, sizeof(float) * k.n_trans));
  if (want) GTNB_TRY(stage_upload(ctx, minus1, m1.data(), sizeof(float) * B));
  GTNB_TRY(stage_end(ctx));

  if (n_sigma) GTNB_TRY(k.sigma(ctx, C, w_dev, sigma));
  GTNB_TRY(num.build(scope, lat, w_dev, sigma));
  // the numerator (a few in-arcs per node) on the second stream beside the denominator (C^2 per frame)
  GTNB_TRY(fork_to(ctx, ctx->copy_stream));
  {
    OnStream side(ctx, ctx->copy_stream);
    GTNB_TRY(launch_implicit_forward(ctx, lat, status + B));
    if (want) GTNB_TRY(launch_implicit_backward(ctx, lat, minus1, g.dev, per, 0, -1, ggrad));
  }
  const int32_t* T_dev = num.T_dev();
  GTNB_TRY(k.forward(ctx, B, T, C, T_dev, e_dev, per, w_dev, den, status));
  if (want) GTNB_TRY(k.backward(ctx, B, T, C, T_dev, e_dev, per, w_dev, den, g.dev, tg.dev));
  GTNB_TRY(join_from(ctx, ctx->copy_stream));
  if (want) {
    GTNB_TRY(launch_scatter_add(ctx, tg.dev, num.map, ggrad, tot_A)); // numerator arcs -> transition (and sigma) slots
    if (n_sigma) GTNB_TRY(k.fold_grad(ctx, C, w_dev, sigma, tg.dev));
    GTNB_TRY(num.scatter(scope, ggrad));
    GTNB_TRY(g.copy_out(ctx, per * B));
    if (half && a.grads) GTNB_TRY(launch_narrow(ctx, g.dev, a.grads, a.dtype, per * B));
    GTNB_TRY(tg.copy_out(ctx, k.n_trans));
  }
  return read_losses(scope, B, den, lat->out_scores, status, 2ll * B, a.losses_host, needs_exact);
}

/*
 * The materialised route of the trellis criteria, graph by graph as the reference composes them: the denominator
 * compose(E_b, G) (G from dense_graph, one for the batch, gmap its arcs' transition slots) and the numerator
 * compose(P_b, E_b) with the host-built products P_b (pmap: the transition slot of every arc, in batch order).
 * arc_of (nullable): the slot of arc_grads (tot_arcs floats) of every numerator arc.  Reproduces the reference's
 * inf / NaN propagation arc by arc; the path for non-finite weights.
 */
int transitions_loss_materialised(CallScope& scope, const TransitionArgs& a, const int32_t* Tb, const HostGraph& G,
                                  const std::vector<int32_t>& gmap, long long n_trans,
                                  const std::vector<gtnb_graph_view>& pviews, const std::vector<int32_t>& pmap,
                                  const std::vector<int32_t>* arc_of, const OutBuf* arc_grads, long long tot_arcs) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = a.B, T = a.T, C = a.C;
  const long long per = (long long)T * C, nG = (long long)gmap.size(), nP = (long long)pmap.size();
  const bool want = a.grads || a.trans_grad || arc_grads;
  const gtnb_graph_view gview = G.view();
  float *e_dev = nullptr, *ft_grad = nullptr, *gg_grad = nullptr;
  int32_t *ft_map_dev = nullptr, *gg_map_dev = nullptr, *arc_of_dev = nullptr;
  OutBuf g, tg;
  gtnb_lattice*& den = scope.lattice();
  gtnb_lattice*& num = scope.lattice();
  GTNB_TRY(scope.input(a.emissions, a.emissions_on_device, per * B, &e_dev));
  GTNB_TRY(gtnb_compose_linear(ctx, B, &gview, 1, 1, Tb, C, e_dev, per, &den));
  GTNB_TRY(gtnb_compose_linear(ctx, B, pviews.data(), B, 0, Tb, C, e_dev, per, &num));
  GTNB_TRY(gtnb_forward(ctx, den, 0, nullptr, nullptr));
  GTNB_TRY(gtnb_forward(ctx, num, 0, nullptr, nullptr));
  if (want) {
    GTNB_TRY(scope.output(a.grads, a.grads_on_device, per * B, &g));
    GTNB_CUDA(ctx, cudaMemsetAsync(g.dev, 0, sizeof(float) * per * B, ctx->stream));
    GTNB_TRY(scope.output(a.trans_grad, a.trans_grad_on_device, n_trans, &tg, /*alias=*/false));
    GTNB_TRY(scope.alloc(&gg_grad, nG));
    GTNB_TRY(scope.alloc(&ft_grad, std::max<long long>(nP, 1)));
    GTNB_TRY(scope.alloc(&gg_map_dev, nG));
    GTNB_TRY(scope.alloc(&ft_map_dev, std::max<long long>(nP, 1)));
    if (arc_of) GTNB_TRY(scope.alloc(&arc_of_dev, std::max<long long>(nP, 1)));
    GTNB_CUDA(ctx, cudaMemsetAsync(tg.dev, 0, sizeof(float) * n_trans, ctx->stream));
    GTNB_CUDA(ctx, cudaMemsetAsync(gg_grad, 0, sizeof(float) * nG, ctx->stream));
    GTNB_CUDA(ctx, cudaMemsetAsync(ft_grad, 0, sizeof(float) * std::max<long long>(nP, 1), ctx->stream));
    if (arc_grads && tot_arcs) GTNB_CUDA(ctx, cudaMemsetAsync(arc_grads->dev, 0, sizeof(float) * tot_arcs, ctx->stream));
    std::vector<float> m1(B, -1.0f);
    GTNB_TRY(gtnb_backward(ctx, den, 0, nullptr)); // +1 / -1: subtract's gradFunc (functions.cpp:53-58)
    GTNB_TRY(gtnb_backward(ctx, num, 0, m1.data()));
    GTNB_TRY(gtnb_compose_grad(ctx, den, gg_grad, g.dev, per));
    GTNB_TRY(gtnb_compose_grad(ctx, num, ft_grad, g.dev, per));
    GTNB_TRY(stage_begin(ctx));
    GTNB_TRY(stage_upload(ctx, gg_map_dev, gmap.data(), sizeof(int32_t) * nG));
    if (nP) GTNB_TRY(stage_upload(ctx, ft_map_dev, pmap.data(), sizeof(int32_t) * nP));
    if (arc_of && nP) GTNB_TRY(stage_upload(ctx, arc_of_dev, arc_of->data(), sizeof(int32_t) * nP));
    GTNB_TRY(stage_end(ctx));
    GTNB_TRY(launch_scatter_add(ctx, tg.dev, gg_map_dev, gg_grad, nG));
    GTNB_TRY(launch_scatter_add(ctx, tg.dev, ft_map_dev, ft_grad, nP));
    if (arc_grads && arc_of) GTNB_TRY(launch_scatter_add(ctx, arc_grads->dev, arc_of_dev, ft_grad, nP));
    GTNB_TRY(g.copy_out(ctx, per * B));
    GTNB_TRY(tg.copy_out(ctx, n_trans));
    if (arc_grads) GTNB_TRY(arc_grads->copy_out(ctx, tot_arcs));
  }
  bool unused = false;
  return read_losses(scope, B, den->out_scores, num->out_scores, nullptr, 0, a.losses_host, &unused);
}

/*
 * n-gram CTC through materialised lattices: intersect(E_b, G) and intersect(P_b, E_b), where P_b = intersect(ctc_b,
 * G) is built on the host WITHOUT the fold (C start states (0, s), then (l, label(l))).
 */
int ngram_ctc_loss_exact(CallScope& scope, const TransitionArgs& a, const Targets& t) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = a.B, C = a.C;
  const long long CC = (long long)C * C;
  std::vector<float> W(CC);
  GTNB_TRY(read_to_host(ctx, W.data(), a.trans_w, a.trans_on_device, CC));
  HostGraph G;
  std::vector<int32_t> gmap;
  dense_graph(true, C, W.data(), &G, &gmap);
  std::vector<HostGraph> pg(B);
  std::vector<gtnb_graph_view> pviews(B);
  std::vector<int32_t> pmap;
  for (int b = 0; b < B; b++) {
    const int L = 2 * t.lens()[b] + 1;
    const int32_t* y = t.labels_of(b);
    auto lab = [&](int l) { return (l & 1) ? y[(l - 1) / 2] : a.blank; };
    // node of CTC node l: (0, blank) for l = 0, C + l - 1 otherwise; nodes [0, C) are the start states (0, s)
    auto node = [&](int l) { return l == 0 ? a.blank : C + l - 1; };
    HostGraph& p = pg[b];
    p.flags.assign(C + L - 1, 0);
    for (int s = 0; s < C; s++) p.flags[s] = 1 | (L == 1 ? 2 : 0);
    for (int l = std::max(1, L - 2); l < L; l++) p.flags[node(l)] |= 2;
    auto arc = [&](int ls, int l) { // every arc of ctc_b (ls -> l) times the matching arcs of G
      const int i = lab(l);
      if (ls == 0) {
        for (int s = 0; s < C; s++) {
          p.arc(s, node(l), i, W[(long long)i * C + s]);
          pmap.push_back(i * C + s);
        }
      } else {
        p.arc(node(ls), node(l), i, W[(long long)i * C + lab(ls)]);
        pmap.push_back(i * C + lab(ls));
      }
    };
    for (int l = 0; l < L; l++) {
      arc(l, l);
      if (l > 0) arc(l - 1, l);
      if ((l & 1) && l > 1 && lab(l) != lab(l - 2)) arc(l - 2, l);
    }
    pviews[b] = p.view();
  }
  return transitions_loss_materialised(scope, a, t.T(), G, gmap, CC, pviews, pmap, nullptr, nullptr, 0);
}

/*
 * ASG's route for C > 128, a non-finite weight or used emission, or the implicit path switched off: gtnb_asg_loss's
 * machinery with the same T_b (the implicit sweeps, else the materialised lattices).  Device-resident transitions
 * and their gradient go through host copies on this route only.
 */
int asg_loss_generic(CallScope& scope, const TransitionArgs& a, const Targets& t) {
  gtnb_ctx* ctx = scope.ctx();
  const long long nTrans = a.C + (long long)a.C * a.C;
  std::vector<float> tw, tg;
  TransitionArgs h = a;
  if (a.trans_on_device) {
    tw.resize(nTrans);
    GTNB_TRY(read_to_host(ctx, tw.data(), a.trans_w, 1, nTrans));
    h.trans_w = tw.data();
    h.trans_on_device = 0;
  }
  if (a.trans_grad && a.trans_grad_on_device) {
    tg.resize(nTrans);
    h.trans_grad = tg.data();
    h.trans_grad_on_device = 0;
  }
  GTNB_TRY(asg_loss(scope, h, t));
  if (!tg.empty()) {
    GTNB_CUDA(ctx, cudaMemcpyAsync(a.trans_grad, tg.data(), sizeof(float) * nTrans, cudaMemcpyHostToDevice,
                                   ctx->stream));
    GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return GTNB_OK;
}

} // namespace

/*
 * CTC with a learned bigram transition graph G (benchmarks/ctc.cpp:107-134, k_ngram.cu):
 *   loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(ctc_b, G), E_b))
 * G: C nodes, all start and accept, arc j -> i with label i and weight W[i*C + j].
 */
namespace {

/* the folded numerator graph of n-gram CTC: the start node S + CTC's graph; arcs = CTC's + the two S arcs (one if
 * U = 0) */
SgDims ngram_num_dims(int U, int skips) {
  SgDims d = ctc_num_dims(U, skips, /*all_valid=*/1);
  d.A += std::min(d.N, 2);
  d.N += 1;
  return d;
}

/* gtnb_ngram_ctc_loss and gtnb_ngram_ctc_loss_typed: a.dtype's emissions on the native route, or widened */
int ngram_ctc_loss_call(gtnb_ctx* ctx, const TransitionArgs& a) {
  const int B = a.B, T = a.T, C = a.C;
  if (!ctx || B < 0 || T < 0 || C <= 0 || !a.emissions || !a.trans_w || !a.target_lens || !a.losses_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss: bad arguments");
  if (a.blank < 0 || a.blank >= C)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss: blank outside [0, C)");
  if (C > kNgramMaxLabels)
    return fail(ctx, GTNB_ERR_UNSUPPORTED,
                "gtnb_ngram_ctc_loss: C = " + std::to_string(C) + " labels; the trellis kernels hold W on chip for C <= " +
                    std::to_string(kNgramMaxLabels));
  Targets t;
  GTNB_TRY(parse_targets(ctx, "gtnb_ngram_ctc_loss", B, T, C, a.input_lens, a.targets, a.target_lens, &t));
  std::vector<SgDims> dims(B);
  for (int b = 0; b < B; b++) {
    if (!t.in_range[b]) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss: label outside [0, C)");
    dims[b] = ngram_num_dims(a.target_lens[b], t.skips[b]);
  }
  TrellisCriterion ngram{(long long)C * C, (long long)B * (T + 1) * C, /*fold=*/true, launch_ngram_den_forward,
                               launch_ngram_den_backward};
  ngram.dtype = a.dtype;
  const bool fast = implicit_dims_supported(dims.data(), B) && ctx->use_implicit;
  return run_criterion(ctx, B, t.T(), a.losses_host, a.trans_grad, a.trans_grad_on_device, (long long)C * C, fast,
                       [&](CallScope& scope, bool f, bool* needs_exact) {
                         if (!f)
                           return widened(scope, a, [&](const TransitionArgs& w) {
                             return ngram_ctc_loss_exact(scope, w, t);
                           });
                         TargetsNumerator num{t, dims, C, launch_ngram_num_build, a.blank};
                         return trellis_loss_fast(scope, ngram, a, num, needs_exact);
                       });
}

bool known_dtype(int dtype) { return dtype == GTNB_F32 || dtype == GTNB_BF16 || dtype == GTNB_F16; }

} // namespace

/*
 * CTC with a learned bigram transition graph G (benchmarks/ctc.cpp:107-134, k_ngram.cu):
 *   loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(ctc_b, G), E_b))
 * G: C nodes, all start and accept, arc j -> i with label i and weight W[i*C + j].
 */
extern "C" int gtnb_ngram_ctc_loss(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const float* trans_w, int trans_on_device, const int32_t* targets, const int32_t* target_lens, int blank,
    float* losses_host, float* grads, int grads_on_device, float* trans_grad, int trans_grad_on_device) {
  return ngram_ctc_loss_call(ctx, TransitionArgs{B, T, C, emissions, emissions_on_device, input_lens, trans_w,
                                                 trans_on_device, targets, target_lens, blank, losses_host, grads,
                                                 grads_on_device, trans_grad, trans_grad_on_device});
}

extern "C" int gtnb_ngram_ctc_loss_typed(
    gtnb_ctx* ctx, int B, int T, int C, const void* emissions_dev, int dtype, const int32_t* input_lens,
    const float* trans_w_dev, const int32_t* targets, const int32_t* target_lens, int blank, float* losses_host,
    void* grads_dev, float* trans_grad_dev) {
  if (!known_dtype(dtype)) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss_typed: unknown dtype");
  return ngram_ctc_loss_call(ctx, TransitionArgs{B, T, C, static_cast<const float*>(emissions_dev), 1, input_lens,
                                                 trans_w_dev, 1, targets, target_lens, blank, losses_host,
                                                 static_cast<float*>(grads_dev), 1, trans_grad_dev, 1, dtype});
}

namespace {
int asg_num_build(gtnb_ctx* ctx, gtnb_lattice* lat, const int32_t* targets_dev, const int32_t* tgt_off_dev,
                  const int32_t* tgt_len_dev, int /*blank*/, const float* trans_w, const float* /*sigma*/,
                  int32_t* map) {
  return launch_asg_num_build(ctx, lat, targets_dev, tgt_off_dev, tgt_len_dev, trans_w, map);
}
} // namespace

/*
 * ASG with per-utterance frame counts and device-resident transitions (gtnb_asg_loss_ex):
 *   loss_b = forwardScore(compose(E_b, transitions)) - forwardScore(compose(compose(fal_b, transitions), E_b))
 * with E_b = linearGraph(T_b, C) on the first T_b rows.  For C <= 128 the denominator is k_ngram.cu's dense trellis
 * in its start mode and the numerator graphs are built on the device; otherwise (and for non-finite weights) the
 * call goes through gtnb_asg_loss's machinery with the same T_b.
 */
namespace {

/* the numerator graph of ASG, compose(fal_b, transitions): U+1 nodes, 2U arcs (none when U = 0), node U accepts */
SgDims asg_num_dims(int U) {
  return SgDims{U + 1, 2 * U, U > 0 ? 1 : 0, /*all_valid=*/1, /*uniform=*/1, /*max_in=*/2, /*max_out=*/2};
}

/* gtnb_asg_loss_ex and gtnb_asg_loss_typed: a.dtype's emissions on the native route, or widened */
int asg_loss_ex_call(gtnb_ctx* ctx, const TransitionArgs& a) {
  const int B = a.B, T = a.T, C = a.C;
  if (!ctx || B < 0 || T < 0 || C <= 0 || !a.emissions || !a.trans_w || !a.target_lens || !a.losses_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss_ex: bad arguments");
  const long long nTrans = C + (long long)C * C;
  Targets t;
  GTNB_TRY(parse_targets(ctx, "gtnb_asg_loss_ex", B, T, C, a.input_lens, a.targets, a.target_lens, &t));
  std::vector<SgDims> dims(B);
  for (int b = 0; b < B; b++) {
    if (!t.in_range[b]) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss_ex: label outside [0, C)");
    dims[b] = asg_num_dims(a.target_lens[b]);
  }
  TrellisCriterion asg{nTrans, asg_alpha_floats(B, T, C), /*fold=*/false, launch_asg_den_forward,
                             launch_asg_den_backward};
  asg.dtype = a.dtype;
  // (a non-finite weight: gtnb_asg_loss's sweeps raise the same status bit and end in the materialised lattices)
  const bool fast = C <= kNgramMaxLabels && ctx->use_implicit && implicit_dims_supported(dims.data(), B);
  return run_criterion(ctx, B, t.T(), a.losses_host, a.trans_grad, a.trans_grad_on_device, nTrans, fast,
                       [&](CallScope& scope, bool f, bool* needs_exact) {
                         if (!f)
                           return widened(scope, a, [&](const TransitionArgs& w) {
                             return asg_loss_generic(scope, w, t);
                           });
                         TargetsNumerator num{t, dims, C, asg_num_build, -1};
                         return trellis_loss_fast(scope, asg, a, num, needs_exact);
                       });
}

} // namespace

/*
 * ASG with per-utterance frame counts and device-resident transitions (gtnb_asg_loss_ex):
 *   loss_b = forwardScore(compose(E_b, transitions)) - forwardScore(compose(compose(fal_b, transitions), E_b))
 * with E_b = linearGraph(T_b, C) on the first T_b rows.  For C <= 128 the denominator is k_ngram.cu's dense trellis
 * in its start mode and the numerator graphs are built on the device; otherwise (and for non-finite weights) the
 * call goes through gtnb_asg_loss's machinery with the same T_b.
 */
extern "C" int gtnb_asg_loss_ex(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const float* trans_w, int trans_on_device, const int32_t* targets, const int32_t* target_lens,
    float* losses_host, float* grads, int grads_on_device, float* trans_grad, int trans_grad_on_device) {
  return asg_loss_ex_call(ctx, TransitionArgs{B, T, C, emissions, emissions_on_device, input_lens, trans_w,
                                              trans_on_device, targets, target_lens, -1, losses_host, grads,
                                              grads_on_device, trans_grad, trans_grad_on_device});
}

extern "C" int gtnb_asg_loss_typed(
    gtnb_ctx* ctx, int B, int T, int C, const void* emissions_dev, int dtype, const int32_t* input_lens,
    const float* trans_w_dev, const int32_t* targets, const int32_t* target_lens, float* losses_host,
    void* grads_dev, float* trans_grad_dev) {
  if (!known_dtype(dtype)) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss_typed: unknown dtype");
  return asg_loss_ex_call(ctx, TransitionArgs{B, T, C, static_cast<const float*>(emissions_dev), 1, input_lens,
                                              trans_w_dev, 1, targets, target_lens, -1, losses_host,
                                              static_cast<float*>(grads_dev), 1, trans_grad_dev, 1, dtype});
}

namespace {

struct TrellisAsyncArgs {
  int B, T, C, S, dtype;
  const void* emissions;
  const int32_t* input_lens;
  const float* trans_w;
  const int32_t *targets, *target_lens;
  int blank; // (n-gram only)
  float* losses;
  int32_t* status;
  void* grads;
  float* trans_grad;
};

/*
 * The run of gtnb_ngram_ctc_loss_async / gtnb_asg_loss_async (asg).  The route is trellis_loss_fast's for a batch at
 * the bounds (every utterance U = S, T_b = T, and for n-gram S - 1 skip arcs): the numerator graphs built on the
 * device from the padded targets and swept by k_implicit.cu on the side stream, the dense trellis of k_ngram.cu on the
 * call's stream.  Where it differs: the prepare kernel writes the descriptors and [offsets | lens | T] the host would
 * have staged; the gate kernel, once both forward sweeps are done, keeps a flagged utterance out of the denominator's
 * backward; the numerator's arc gradients are scattered utterance by utterance, flagged ones left out; the losses and
 * status are formed on the device.  Sizing passes NULL buffers (want: trans_grad set) and takes the largest scratch.
 */
int trellis_async_run(gtnb_ctx* ctx, bool asg, const TrellisAsyncArgs& a, bool launch) {
  const char* fn = asg ? "gtnb_asg_loss_async" : "gtnb_ngram_ctc_loss_async";
  const int B = a.B, T = a.T, C = a.C, S = a.S;
  const bool half = a.dtype != GTNB_F32;
  const long long per = (long long)T * C;
  if (C > kNgramMaxLabels)
    return fail(ctx, GTNB_ERR_UNSUPPORTED, std::string(fn) + ": C = " + std::to_string(C) +
                                               " labels; the trellis kernels hold the transitions on chip for C <= " +
                                               std::to_string(kNgramMaxLabels));
  if (!ctx->use_implicit)
    return fail(ctx, GTNB_ERR_UNSUPPORTED, std::string(fn) + ": the \"implicit\" flag is off (materialised route)");
  if (!asg && (a.blank < 0 || a.blank >= C))
    return fail(ctx, GTNB_ERR_UNSUPPORTED, std::string(fn) + ": blank outside [0, C)");
  const SgDims bound = asg ? asg_num_dims(S) : ngram_num_dims(S, std::max(S - 1, 0));
  const std::vector<SgDims> dims(B, bound);
  if (!implicit_dims_supported(dims.data(), B))
    return fail(ctx, GTNB_ERR_UNSUPPORTED, std::string(fn) + ": bounds outside the implicit sweeps");
  const long long n_trans = (asg ? C : 0) + (long long)C * C;
  const long long n_sigma = asg ? 0 : C;
  const long long tot_A = (long long)B * bound.A;
  const bool want = a.grads || a.trans_grad;
  const std::vector<int32_t> Tv(B, T);
  std::vector<long long> sgn, sga;
  gtnb_lattice* lat_raw = nullptr;
  GTNB_TRY(composed_alloc(ctx, B, dims.data(), B, 0, Tv.data(), C, static_cast<const float*>(a.emissions), per, sgn,
                          sga, &lat_raw, true));
  const std::unique_ptr<gtnb_lattice> lat(lat_raw); // (its device buffers lie in the arena: nothing to free)
  if (half) lat->dtype = a.dtype; // 16-bit emissions read in place by both sweeps, as the _typed calls do
  int32_t *small = nullptr, *valid = nullptr, *kstatus = nullptr, *T_bwd = nullptr, *map = nullptr;
  float *deltas = nullptr, *sigma = nullptr, *alpha = nullptr, *den = nullptr, *ggrad = nullptr, *tg = nullptr;
  float* g = half ? nullptr : static_cast<float*>(a.grads);
  GTNB_TRY(dev_alloc(ctx, &small, 3ll * B));
  GTNB_TRY(dev_alloc(ctx, &valid, B));
  GTNB_TRY(dev_alloc(ctx, &kstatus, 2ll * B));
  GTNB_TRY(dev_alloc(ctx, &T_bwd, B));
  GTNB_TRY(dev_alloc(ctx, &deltas, B));
  GTNB_TRY(dev_alloc(ctx, &map, tot_A));
  if (n_sigma) GTNB_TRY(dev_alloc(ctx, &sigma, n_sigma));
  GTNB_TRY(dev_alloc(ctx, &alpha, asg ? asg_alpha_floats(B, T, C) : (long long)B * (T + 1) * C));
  GTNB_TRY(dev_alloc(ctx, &den, B));
  if (want) {
    GTNB_TRY(dev_alloc(ctx, &ggrad, tot_A));
    // [d/dtrans | d/dsigma]: the caller's buffer when it has the room (ASG, no sigma slots), else scratch that is
    // copied out at the end (sizing takes the scratch: it cannot tell whether trans_grad will be given)
    if (n_sigma || !a.trans_grad || !launch)
      GTNB_TRY(dev_alloc(ctx, &tg, n_trans + n_sigma));
    else
      tg = a.trans_grad;
    // float32 emission gradient: the caller's, else (16-bit, or transitions only) scratch
    if (!g) GTNB_TRY(dev_alloc(ctx, &g, per * B));
  }
  if (!launch) return GTNB_OK;

  // the side stream and its events exist once a call has run outside capture; a capture must not create them
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  GTNB_CUDA(ctx, cudaStreamIsCapturing(ctx->stream, &cap));
  if (cap != cudaStreamCaptureStatusNone && (!ctx->copy_stream || ctx->side_events.empty()))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT,
                std::string(fn) + ": call it once outside stream capture first (it creates its side stream then)");
  GTNB_TRY(ensure_side_streams(ctx, 0, 1));
  const float* e = static_cast<const float*>(a.emissions); // (a.dtype's elements: the kernels read them as such)
  const int32_t* T_fwd = small + 2ll * B;
  if (want) {
    GTNB_CUDA(ctx, cudaMemsetAsync(g, 0, sizeof(float) * per * B, ctx->stream));
    GTNB_CUDA(ctx, cudaMemsetAsync(tg, 0, sizeof(float) * (n_trans + n_sigma), ctx->stream));
    GTNB_CUDA(ctx, cudaMemsetAsync(ggrad, 0, sizeof(float) * tot_A, ctx->stream));
  }
  GTNB_TRY(launch_trellis_async_prepare(ctx, asg, B, S, T, C, lat->meta_h[0], lat->meta_h[B > 1 ? 1 : 0],
                                        a.input_lens, a.targets, a.target_lens, lat->meta, small, deltas, valid,
                                        kstatus));
  if (asg) {
    GTNB_TRY(launch_asg_num_build(ctx, lat.get(), a.targets, small, small + B, a.trans_w, map));
  } else {
    GTNB_TRY(launch_ngram_sigma(ctx, C, a.trans_w, sigma));
    GTNB_TRY(launch_ngram_num_build(ctx, lat.get(), a.targets, small, small + B, a.blank, a.trans_w, sigma, map));
  }
  // the numerator (a few in-arcs per node) on the side stream beside the denominator (C^2 per frame)
  cudaEvent_t num_forward_done = ctx->side_events[0];
  GTNB_TRY(fork_to(ctx, ctx->copy_stream));
  {
    OnStream side(ctx, ctx->copy_stream);
    GTNB_TRY(launch_implicit_forward(ctx, lat.get(), kstatus + B));
    GTNB_CUDA(ctx, cudaEventRecord(num_forward_done, ctx->copy_stream));
    if (want) GTNB_TRY(launch_implicit_backward(ctx, lat.get(), deltas, g, per, 0, -1, ggrad));
  }
  if (asg)
    GTNB_TRY(launch_asg_den_forward(ctx, B, T, C, T_fwd, e, per, a.trans_w, alpha, den, kstatus, a.dtype));
  else
    GTNB_TRY(launch_ngram_den_forward(ctx, B, T, C, T_fwd, e, per, a.trans_w, alpha, den, kstatus, a.dtype));
  GTNB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, num_forward_done, 0));
  GTNB_TRY(launch_trellis_async_gate(ctx, B, T_fwd, valid, kstatus, T_bwd, den));
  if (want) {
    if (asg)
      GTNB_TRY(launch_asg_den_backward(ctx, B, T, C, T_bwd, e, per, a.trans_w, alpha, den, g, per, tg, a.dtype));
    else
      GTNB_TRY(launch_ngram_den_backward(ctx, B, T, C, T_bwd, e, per, a.trans_w, alpha, den, g, per, tg, a.dtype));
  }
  GTNB_TRY(join_from(ctx, ctx->copy_stream));
  if (want) {
    GTNB_TRY(launch_trellis_async_scatter(ctx, B, lat->meta, kstatus, map, ggrad, tg));
    if (n_sigma) GTNB_TRY(launch_ngram_fold(ctx, C, a.trans_w, sigma, tg));
  }
  // losses = den - num in float32 as read_losses forms them; a flagged utterance's emission-gradient row zeroed
  GTNB_TRY(launch_ctc_async_finalize(ctx, B, 1, den, lat->out_scores, kstatus, valid, a.losses, a.status,
                                     a.grads ? g : nullptr, per));
  if (half && a.grads) GTNB_TRY(launch_narrow(ctx, g, a.grads, a.dtype, per * B));
  if (a.trans_grad && tg != a.trans_grad) // (n-gram: ngram_fold_kernel reads the sigma slots right after W's)
    GTNB_CUDA(ctx, cudaMemcpyAsync(a.trans_grad, tg, sizeof(float) * n_trans, cudaMemcpyDeviceToDevice,
                                   ctx->stream));
  return GTNB_OK;
}

int trellis_async_workspace(gtnb_ctx* ctx, bool asg, int B, int T, int C, int S, int dtype, int with_grad,
                            size_t* bytes) {
  const char* fn = asg ? "gtnb_asg_loss_async_workspace" : "gtnb_ngram_ctc_loss_async_workspace";
  if (!ctx || B < 0 || T < 0 || C <= 0 || S < 0 || !bytes)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, std::string(fn) + ": bad arguments");
  if (!known_dtype(dtype)) return fail(ctx, GTNB_ERR_UNSUPPORTED, std::string(fn) + ": unknown dtype");
  // (grads NULL sizes the float32 scratch gradient)
  const TrellisAsyncArgs a{B, T, C, S, dtype, nullptr, nullptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr,
                           nullptr, with_grad ? stand_in : nullptr};
  return async_workspace(ctx, B, bytes, [&](bool launch) { return trellis_async_run(ctx, asg, a, launch); });
}

int trellis_async_call(gtnb_ctx* ctx, bool asg, void* cuda_stream, const TrellisAsyncArgs& a, void* workspace_dev,
                       size_t workspace_bytes) {
  const char* fn = asg ? "gtnb_asg_loss_async" : "gtnb_ngram_ctc_loss_async";
  if (!ctx || a.B < 0 || a.T < 0 || a.C <= 0 || a.S < 0 || !a.emissions || !a.trans_w ||
      (a.S > 0 && !a.targets) || !a.target_lens || !a.losses)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, std::string(fn) + ": bad arguments");
  if (!known_dtype(a.dtype)) return fail(ctx, GTNB_ERR_UNSUPPORTED, std::string(fn) + ": unknown dtype");
  if (a.B == 0 && a.trans_grad) {
    const long long n_trans = (asg ? a.C : 0) + (long long)a.C * a.C;
    GTNB_CUDA(ctx, cudaMemsetAsync(a.trans_grad, 0, sizeof(float) * n_trans, static_cast<cudaStream_t>(cuda_stream)));
  }
  return async_enqueue(ctx, fn, a.B, cuda_stream, workspace_dev, workspace_bytes,
                       [&](bool launch) { return trellis_async_run(ctx, asg, a, launch); });
}

} // namespace

extern "C" int gtnb_ngram_ctc_loss_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int S, int dtype,
                                                   int with_grad, size_t* bytes) {
  return trellis_async_workspace(ctx, false, B, T, C, S, dtype, with_grad, bytes);
}

extern "C" int gtnb_ngram_ctc_loss_async(
    gtnb_ctx* ctx, void* cuda_stream, int B, int T, int C, int S, const void* emissions_dev, int dtype,
    const int32_t* input_lens_dev, const float* trans_w_dev, const int32_t* targets_dev,
    const int32_t* target_lens_dev, int blank, float* losses_dev, int32_t* status_dev, void* grads_dev,
    float* trans_grad_dev, void* workspace_dev, size_t workspace_bytes) {
  return trellis_async_call(ctx, false, cuda_stream,
                            TrellisAsyncArgs{B, T, C, S, dtype, emissions_dev, input_lens_dev, trans_w_dev, targets_dev,
                                             target_lens_dev, blank, losses_dev, status_dev, grads_dev, trans_grad_dev},
                            workspace_dev, workspace_bytes);
}

extern "C" int gtnb_asg_loss_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int S, int dtype, int with_grad,
                                             size_t* bytes) {
  return trellis_async_workspace(ctx, true, B, T, C, S, dtype, with_grad, bytes);
}

extern "C" int gtnb_asg_loss_async(
    gtnb_ctx* ctx, void* cuda_stream, int B, int T, int C, int S, const void* emissions_dev, int dtype,
    const int32_t* input_lens_dev, const float* trans_w_dev, const int32_t* targets_dev,
    const int32_t* target_lens_dev, float* losses_dev, int32_t* status_dev, void* grads_dev, float* trans_grad_dev,
    void* workspace_dev, size_t workspace_bytes) {
  return trellis_async_call(ctx, true, cuda_stream,
                            TrellisAsyncArgs{B, T, C, S, dtype, emissions_dev, input_lens_dev, trans_w_dev, targets_dev,
                                             target_lens_dev, 0, losses_dev, status_dev, grads_dev, trans_grad_dev},
                            workspace_dev, workspace_bytes);
}

/*
 * Forced alignment without a host synchronisation: viterbiPath / viterbiScore of each loss's own numerator, from
 * padded device targets, under gtnb_*_loss_async's contract.  The lattices are those of the synchronous aligners:
 *   CTC         intersect(ctcGraph(y_b), E_b)                 (gtnb_graph_viterbi on CTC graphs)
 *   n-gram CTC  intersect(intersect(ctc_b, G), E_b)           (gtnb_graph_transitions_viterbi, BIGRAM)
 *   ASG         compose(compose(fal_b, transitions), E_b)     (gtnb_graph_transitions_viterbi, ASG)
 * One route for the three, on the call's stream: the prepare kernel's descriptors, the numerator built by the loss's
 * build kernel (n-gram: its folded start arcs weigh tau_l = max_j W[l][j], the tropical sigma), the tropical forward of
 * k_implicit.cu, its trace, and align_async_finalize_kernel, which maps the status and each traced arc to its target
 * position.  16-bit emissions are widened once into the workspace: the tropical kernels are float32 only.
 */
namespace {

struct AlignAsyncArgs {
  int B, T, C, S, dtype;
  const void* emissions;
  const int32_t* input_lens;
  const float* trans_w; // n-gram W [C*C], ASG [C + C*C]; NULL for CTC
  const int32_t *targets, *target_lens;
  int blank; // (not ASG)
  int32_t *paths, *tokens;
  float* scores;
  int32_t* status;
};

const char* align_async_name(AlignCriterion kind) {
  return kind == AlignCriterion::Ctc     ? "gtnb_ctc_align_async"
         : kind == AlignCriterion::Ngram ? "gtnb_ngram_ctc_align_async"
                                         : "gtnb_asg_align_async";
}

/*
 * The run of the three.  Sized from the bounds (every utterance U = S, T_b = T, CTC with S - 1 skips), as the losses'
 * asynchronous calls are; sizing passes NULL buffers and takes the arcs row of the token mapping whether or not tokens
 * will be asked for.
 */
int align_async_run(gtnb_ctx* ctx, AlignCriterion kind, const AlignAsyncArgs& a, bool launch) {
  const std::string fn = align_async_name(kind);
  const int B = a.B, T = a.T, C = a.C, S = a.S;
  const bool half = a.dtype != GTNB_F32;
  const long long per = (long long)T * C;
  if (!ctx->use_implicit)
    return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": the \"implicit\" flag is off (materialised route)");
  if (kind != AlignCriterion::Asg && (a.blank < 0 || a.blank >= C))
    return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": blank outside [0, C)");
  const int skips = std::max(S - 1, 0);
  const SgDims bound = kind == AlignCriterion::Ctc     ? ctc_num_dims(S, skips, /*all_valid=*/1)
                       : kind == AlignCriterion::Ngram ? ngram_num_dims(S, skips)
                                                       : asg_num_dims(S);
  const std::vector<SgDims> dims(B, bound);
  if (!implicit_dims_supported(dims.data(), B))
    return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": bounds outside the implicit sweeps (use the graph aligners)");
  const std::vector<int32_t> Tv(B, T);
  std::vector<long long> sgn, sga;
  gtnb_lattice* lat_raw = nullptr;
  GTNB_TRY(composed_alloc(ctx, B, dims.data(), B, 0, Tv.data(), C, static_cast<const float*>(a.emissions), per, sgn,
                          sga, &lat_raw, true));
  const std::unique_ptr<gtnb_lattice> lat(lat_raw); // (its device buffers lie in the arena: nothing to free)
  if (!implicit_trace_supported(lat.get()))
    return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": bounds outside the trace's shared memory (use the graph aligners)");
  int32_t *small = nullptr, *valid = nullptr, *kstatus = nullptr, *map = nullptr, *arcs = nullptr;
  float *deltas = nullptr, *tau = nullptr;
  GTNB_TRY(dev_alloc(ctx, &small, 3ll * B));
  GTNB_TRY(dev_alloc(ctx, &valid, B));
  GTNB_TRY(dev_alloc(ctx, &kstatus, kind == AlignCriterion::Ctc ? B : 2ll * B)); // (the trellis prepare zeroes 2B)
  GTNB_TRY(dev_alloc(ctx, &deltas, B)); // (written by the prepare kernel, read by no sweep here)
  if (kind != AlignCriterion::Ctc) GTNB_TRY(dev_alloc(ctx, &map, (long long)B * bound.A));
  if (kind == AlignCriterion::Ngram) GTNB_TRY(dev_alloc(ctx, &tau, C));
  if (a.tokens || !launch) GTNB_TRY(dev_alloc(ctx, &arcs, (long long)B * T));
  float* wide = nullptr;
  if (half) {
    GTNB_TRY(dev_alloc(ctx, &wide, per * B));
    lat->emissions = wide;
  }
  if (!launch) return GTNB_OK;

  if (half) GTNB_TRY(launch_widen(ctx, a.emissions, a.dtype, wide, per * B));
  const GraphMeta& m0 = lat->meta_h[0];
  const GraphMeta& m1 = lat->meta_h[B > 1 ? 1 : 0];
  if (kind == AlignCriterion::Ctc) {
    GTNB_TRY(launch_ctc_async_prepare(ctx, B, S, T, C, m0, m1, a.input_lens, a.targets, a.target_lens, lat->meta,
                                      small, deltas, valid, kstatus));
    GTNB_TRY(launch_ctc_build(ctx, lat.get(), a.targets, small, small + B, a.blank));
  } else {
    const bool asg = kind == AlignCriterion::Asg;
    GTNB_TRY(launch_trellis_async_prepare(ctx, asg, B, S, T, C, m0, m1, a.input_lens, a.targets, a.target_lens,
                                          lat->meta, small, deltas, valid, kstatus));
    if (asg) {
      GTNB_TRY(launch_asg_num_build(ctx, lat.get(), a.targets, small, small + B, a.trans_w, map));
    } else {
      GTNB_TRY(launch_ngram_tau(ctx, C, a.trans_w, tau));
      GTNB_TRY(launch_ngram_num_build(ctx, lat.get(), a.targets, small, small + B, a.blank, a.trans_w, tau, map));
    }
  }
  GTNB_TRY(launch_implicit_forward(ctx, lat.get(), kstatus, 0, -1, /*tropical=*/true));
  GTNB_TRY(launch_implicit_trace(ctx, lat.get(), kstatus, a.paths, arcs, a.scores, T));
  return launch_align_async_finalize(ctx, kind, B, T, lat->meta, lat->sg_in_ptr, kstatus, valid, arcs, a.paths,
                                     a.tokens, a.scores, a.status);
}

int align_async_workspace(gtnb_ctx* ctx, AlignCriterion kind, int B, int T, int C, int S, int dtype, size_t* bytes) {
  const std::string fn = std::string(align_async_name(kind)) + "_workspace";
  if (!ctx || B < 0 || T < 0 || C <= 0 || S < 0 || !bytes)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  if (!known_dtype(dtype)) return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": unknown dtype");
  // (blank 0: sizing does not depend on it)
  const AlignAsyncArgs a{B, T, C, S, dtype, nullptr, nullptr, nullptr, nullptr, nullptr, 0,
                         nullptr, nullptr, nullptr, nullptr};
  return async_workspace(ctx, B, bytes, [&](bool launch) { return align_async_run(ctx, kind, a, launch); });
}

int align_async_call(gtnb_ctx* ctx, AlignCriterion kind, void* cuda_stream, const AlignAsyncArgs& a,
                     void* workspace_dev, size_t workspace_bytes) {
  const std::string fn = align_async_name(kind);
  if (!ctx || a.B < 0 || a.T < 0 || a.C <= 0 || a.S < 0 || !a.emissions ||
      (kind != AlignCriterion::Ctc && !a.trans_w) || (a.S > 0 && !a.targets) || !a.target_lens || !a.scores)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  if (!known_dtype(a.dtype)) return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": unknown dtype");
  return async_enqueue(ctx, fn, a.B, cuda_stream, workspace_dev, workspace_bytes,
                       [&](bool launch) { return align_async_run(ctx, kind, a, launch); });
}

} // namespace

extern "C" int gtnb_ctc_align_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int S, int dtype, size_t* bytes) {
  return align_async_workspace(ctx, AlignCriterion::Ctc, B, T, C, S, dtype, bytes);
}

extern "C" int gtnb_ctc_align_async(
    gtnb_ctx* ctx, void* cuda_stream, int B, int T, int C, int S, const void* emissions_dev, int dtype,
    const int32_t* input_lens_dev, const int32_t* targets_dev, const int32_t* target_lens_dev, int blank,
    int32_t* paths_dev, int32_t* tokens_dev, float* scores_dev, int32_t* status_dev, void* workspace_dev,
    size_t workspace_bytes) {
  return align_async_call(ctx, AlignCriterion::Ctc, cuda_stream,
                          AlignAsyncArgs{B, T, C, S, dtype, emissions_dev, input_lens_dev, nullptr, targets_dev,
                                         target_lens_dev, blank, paths_dev, tokens_dev, scores_dev, status_dev},
                          workspace_dev, workspace_bytes);
}

extern "C" int gtnb_ngram_ctc_align_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int S, int dtype,
                                                    size_t* bytes) {
  return align_async_workspace(ctx, AlignCriterion::Ngram, B, T, C, S, dtype, bytes);
}

extern "C" int gtnb_ngram_ctc_align_async(
    gtnb_ctx* ctx, void* cuda_stream, int B, int T, int C, int S, const void* emissions_dev, int dtype,
    const int32_t* input_lens_dev, const float* trans_w_dev, const int32_t* targets_dev,
    const int32_t* target_lens_dev, int blank, int32_t* paths_dev, int32_t* tokens_dev, float* scores_dev,
    int32_t* status_dev, void* workspace_dev, size_t workspace_bytes) {
  return align_async_call(ctx, AlignCriterion::Ngram, cuda_stream,
                          AlignAsyncArgs{B, T, C, S, dtype, emissions_dev, input_lens_dev, trans_w_dev, targets_dev,
                                         target_lens_dev, blank, paths_dev, tokens_dev, scores_dev, status_dev},
                          workspace_dev, workspace_bytes);
}

extern "C" int gtnb_asg_align_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int S, int dtype, size_t* bytes) {
  return align_async_workspace(ctx, AlignCriterion::Asg, B, T, C, S, dtype, bytes);
}

extern "C" int gtnb_asg_align_async(
    gtnb_ctx* ctx, void* cuda_stream, int B, int T, int C, int S, const void* emissions_dev, int dtype,
    const int32_t* input_lens_dev, const float* trans_w_dev, const int32_t* targets_dev,
    const int32_t* target_lens_dev, int32_t* paths_dev, int32_t* tokens_dev, float* scores_dev, int32_t* status_dev,
    void* workspace_dev, size_t workspace_bytes) {
  return align_async_call(ctx, AlignCriterion::Asg, cuda_stream,
                          AlignAsyncArgs{B, T, C, S, dtype, emissions_dev, input_lens_dev, trans_w_dev, targets_dev,
                                         target_lens_dev, 0, paths_dev, tokens_dev, scores_dev, status_dev},
                          workspace_dev, workspace_bytes);
}

/*
 * Loss over user-supplied target graphs (the criterion of the reference's pytorch_loss.py and of its word
 * decomposition examples):
 *   loss_b = forwardScore(E_b) - forwardScore(intersect(A_b, E_b))
 * E_b: linearGraph(T_b, C) on the first T_b rows of emissions_b; A_b: graph b, matched on its olabels.
 * The implicit sweeps of k_implicit.cu run intersect(A_b, E_b) without building it (the arc-label instantiations
 * when some graph is not label-uniform), with forwardScore(E_b) (k_linear.cu) beside the forward sweep.  Graphs that
 * do not fit the implicit layout, C above the arc-label limit, the implicit flag off, or a non-finite value met by
 * a sweep take the materialised lattices (gtnb_compose_linear, forward, backward, compose_grad), the normaliser's
 * included.
 */
namespace {

/*
 * The batch of user target graphs every graph entry point takes, as parse_graphs checks it.  The arcs are numbered
 * through the batch, graph after graph (first_arc).  Host arc weights are spliced into the copied views; device arc
 * weights (arc_weights_dev) are used where they lie, and the views keep the caller's weights pointer.
 */
struct GraphBatch {
  int B = 0, T = 0, C = 0;
  std::vector<int32_t> Tb;
  std::vector<gtnb_graph_view> views;
  std::vector<long long> first_arc; // every view's first arc in the batch's numbering
  long long tot_arcs = 0;
  const float* arc_weights_dev = nullptr;

  /* the views with host weights, for the routes that run on the host: device weights are read back into *host_w */
  int host_views(gtnb_ctx* ctx, std::vector<float>* host_w, std::vector<gtnb_graph_view>* out) const {
    *out = views;
    if (!arc_weights_dev) return GTNB_OK;
    host_w->resize((size_t)std::max(tot_arcs, 1ll));
    if (tot_arcs) GTNB_TRY(read_to_host(ctx, host_w->data(), arc_weights_dev, 1, tot_arcs));
    for (int b = 0; b < B; b++) (*out)[b].weights = host_w->data() + first_arc[b];
    return GTNB_OK;
  }
};

/*
 * The argument check the graph entry points share, then own_checks() (the entry point's own), then the graphs: T_b =
 * input_lens[b] (or T) in [0, T], well-formed views, no epsilon arc, fewer than 2^31 arcs in all.  args_ok: the
 * entry point's own pointer arguments are present.
 */
template <class Checks>
int parse_graphs(gtnb_ctx* ctx, const char* fn, int B, int T, int C, const float* emissions,
                 const gtnb_graph_view* graphs, bool args_ok, const int32_t* input_lens, const float* arc_weights,
                 int arc_weights_on_device, GraphBatch* gb, Checks&& own_checks) {
  if (!ctx || B < 0 || T < 0 || C <= 0 || !args_ok || (B > 0 && (!emissions || !graphs)))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, std::string(fn) + ": bad arguments");
  GTNB_TRY(own_checks());
  gb->B = B, gb->T = T, gb->C = C;
  gb->Tb.resize(B);
  gb->views.assign(graphs, graphs + B);
  gb->first_arc.resize(B);
  gb->arc_weights_dev = arc_weights_on_device ? arc_weights : nullptr;
  for (int b = 0; b < B; b++) {
    gtnb_graph_view& v = gb->views[b];
    gb->Tb[b] = input_lens ? input_lens[b] : T;
    if (gb->Tb[b] < 0 || gb->Tb[b] > T)
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, std::string(fn) + ": input_lens outside [0, T]");
    if (validate_view(ctx, v)) return GTNB_ERR_INVALID_ARGUMENT;
    for (int k = 0; k < v.num_arcs; k++)
      if (v.arc_olabel[k] == GTNB_EPSILON)
        return fail(ctx, GTNB_ERR_UNSUPPORTED,
                    std::string(fn) + ": graph " + std::to_string(b) +
                        " has epsilon arcs; remove them first (remove(g, epsilon))");
    gb->first_arc[b] = gb->tot_arcs;
    if (arc_weights && !arc_weights_on_device) v.weights = arc_weights + gb->tot_arcs;
    gb->tot_arcs += v.num_arcs;
  }
  if (gb->tot_arcs >= (1ll << 31)) return fail(ctx, GTNB_ERR_UNSUPPORTED, std::string(fn) + ": more than 2^31 arcs");
  return GTNB_OK;
}

int no_own_checks() { return GTNB_OK; }

/* rc of building the implicit sweeps: GTNB_ERR_UNSUPPORTED (the graphs do not fit the implicit layout) turns
 * *implicit off, so that the caller materialises */
int implicit_or_materialise(int rc, bool* implicit) {
  if (rc != GTNB_ERR_UNSUPPORTED) return rc;
  *implicit = false;
  return GTNB_OK;
}

struct GraphLossArgs {
  const float* emissions;
  int emissions_on_device;
  float* losses_host;
  float* grads;
  int grads_on_device;
  float* arc_grads;
  int arc_grads_on_device;
};

/* one attempt; implicit: try the sweeps first (the materialised lattices when the graphs do not qualify).
 * *needs_exact: a sweep met a non-finite weight or emission, the outputs are not to be used. */
int graph_loss_once(CallScope& scope, const GraphLossArgs& a, const GraphBatch& gb, bool implicit,
                    bool* needs_exact) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = gb.B, T = gb.T, C = gb.C;
  const std::vector<int32_t>& Tb = gb.Tb;
  const long long per = (long long)T * C, tot_arcs = gb.tot_arcs;
  const bool want = a.grads || a.arc_grads;
  const int maxT = *std::max_element(Tb.begin(), Tb.end());
  float *e_dev = nullptr, *den = nullptr, *minus1 = nullptr;
  int32_t *T_dev = nullptr, *status = nullptr;
  OutBuf g, ag;
  gtnb_lattice*& lat = scope.lattice();
  gtnb_lattice*& dlat = scope.lattice();
  const float* den_scores = nullptr;
  std::vector<float> m1(B, -1.0f); // subtract's gradFunc, functions.cpp:53-58
  // materialised route: forwardScore(E_b) as the reference computes it, non-finite emissions included (its sweep
  // turns a node whose in-scores are all NaN into -inf), from the lattice of one start-and-accept node with a
  // self-loop per label: compose(free, E_b) is E_b arc for arc
  HostGraph free_graph;
  free_graph.flags.assign(1, 3);
  free_graph.src.assign(C, 0);
  free_graph.dst = free_graph.src;
  free_graph.label.resize(C);
  for (int c = 0; c < C; c++) free_graph.label[c] = c;
  const gtnb_graph_view free_view = free_graph.view();

  GTNB_TRY(ensure_side_streams(ctx, 0, 0));
  GTNB_TRY(scope.input(a.emissions, a.emissions_on_device, per * B, &e_dev));
  GTNB_TRY(scope.alloc(&den, B));
  GTNB_TRY(scope.alloc(&T_dev, B));
  GTNB_TRY(scope.alloc(&status, B));
  GTNB_TRY(scope.alloc(&minus1, B));
  if (want) {
    // (the emission gradient is also the scratch of a call that only wants the arc gradients)
    GTNB_TRY(scope.output(a.grads, a.grads_on_device, per * B, &g));
    GTNB_CUDA(ctx, cudaMemsetAsync(g.dev, 0, sizeof(float) * per * B, ctx->stream));
    if (a.arc_grads) {
      GTNB_TRY(scope.output(a.arc_grads, a.arc_grads_on_device, tot_arcs, &ag));
      if (tot_arcs) GTNB_CUDA(ctx, cudaMemsetAsync(ag.dev, 0, sizeof(float) * tot_arcs, ctx->stream));
    }
  }
  GTNB_CUDA(ctx, cudaMemsetAsync(status, 0, sizeof(int32_t) * B, ctx->stream));
  GTNB_TRY(stage_begin(ctx));
  GTNB_TRY(stage_upload(ctx, T_dev, Tb.data(), sizeof(int32_t) * B));
  GTNB_TRY(stage_upload(ctx, minus1, m1.data(), sizeof(float) * B));
  GTNB_TRY(stage_end(ctx));

  if (implicit)
    GTNB_TRY(implicit_or_materialise(compose_linear_impl(ctx, B, gb.views.data(), B, 0, Tb.data(), C, e_dev, per,
                                                         true, &lat, true, gb.arc_weights_dev),
                                     &implicit));
  if (implicit) {
    // forwardScore(E_b) and its +1 gradient on the second stream, beside the forward sweep
    GTNB_TRY(fork_to(ctx, ctx->copy_stream));
    {
      OnStream side(ctx, ctx->copy_stream);
      GTNB_TRY(launch_linear_forward(ctx, B, T_dev, maxT, C, e_dev, per, 0, den, want ? g.dev : nullptr, per,
                                     nullptr, 1.0f, 0));
    }
    GTNB_TRY(launch_implicit_forward(ctx, lat, status));
    GTNB_TRY(join_from(ctx, ctx->copy_stream));
    if (want) GTNB_TRY(launch_implicit_backward(ctx, lat, minus1, g.dev, per, 0, -1, ag.dev));
    den_scores = den;
  } else {
    GTNB_TRY(compose_linear_impl(ctx, B, gb.views.data(), B, 0, Tb.data(), C, e_dev, per, false, &lat, false,
                                 gb.arc_weights_dev));
    GTNB_TRY(compose_linear_impl(ctx, B, &free_view, 1, 0, Tb.data(), C, e_dev, per, false, &dlat));
    GTNB_TRY(gtnb_forward(ctx, dlat, 0, nullptr, nullptr));
    GTNB_TRY(gtnb_forward(ctx, lat, 0, nullptr, nullptr));
    if (want) {
      GTNB_TRY(gtnb_backward(ctx, dlat, 0, nullptr)); // +1
      GTNB_TRY(gtnb_compose_grad(ctx, dlat, nullptr, g.dev, per));
      GTNB_TRY(gtnb_backward(ctx, lat, 0, m1.data()));
      GTNB_TRY(gtnb_compose_grad(ctx, lat, ag.dev, g.dev, per));
    }
    den_scores = dlat->out_scores;
  }
  GTNB_TRY(g.copy_out(ctx, per * B));
  GTNB_TRY(ag.copy_out(ctx, tot_arcs));
  // (the materialised route leaves the status words 0)
  return read_losses(scope, B, den_scores, lat->out_scores, status, B, a.losses_host, needs_exact);
}

} // namespace

extern "C" int gtnb_graph_loss(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const gtnb_graph_view* graphs, const float* arc_weights, int arc_weights_on_device, float* losses_host,
    float* grads, int grads_on_device, float* arc_grads, int arc_grads_on_device) {
  GraphBatch gb;
  GTNB_TRY(parse_graphs(ctx, "gtnb_graph_loss", B, T, C, emissions, graphs, B == 0 || losses_host, input_lens,
                        arc_weights, arc_weights_on_device, &gb, no_own_checks));
  const GraphLossArgs a{emissions, emissions_on_device, losses_host, grads, grads_on_device, arc_grads,
                        arc_grads_on_device};
  // (graphs that are not label-uniform need C <= k_implicit.cu's kArcMaxLabels: compose_linear_impl checks)
  return run_criterion(ctx, B, gb.Tb.data(), losses_host, nullptr, 0, 0, ctx->use_implicit,
                       [&](CallScope& scope, bool implicit, bool* needs_exact) {
                         return graph_loss_once(scope, a, gb, implicit, needs_exact);
                       });
}

/*
 * Loss over user-supplied target graphs with a learned dense transition graph G (the ASG and CTC alignment graphs of
 * the reference's examples/learned_decompositions.cpp and examples/priors.cpp, completed with "the standard emissions
 * and transitions graph"):
 *   ASG:    loss_b = forwardScore(compose(E_b, G)) - forwardScore(compose(compose(A_b, G), E_b))
 *   BIGRAM: loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(A_b, G), E_b))
 * G and trans_w as in gtnb_asg_loss_ex / gtnb_ngram_ctc_loss; E_b, A_b and the arc weights as in gtnb_graph_loss.
 * The numerators are the products of gtnb_product.h, built on the host once per call; their weights are folded on
 * the device from the transitions where they lie (launch_product_fold).  The device route sweeps them with
 * k_implicit.cu beside k_ngram.cu's dense trellis (trellis_loss_fast); a non-finite value, the implicit flag off or
 * a product that does not fit the implicit layout take the materialised lattices.
 */
namespace {

/* the checks of the entry points that take a dense transition graph kind */
int check_dense_kind(gtnb_ctx* ctx, const char* fn, int kind, int C) {
  if (kind != GTNB_DENSE_ASG && kind != GTNB_DENSE_BIGRAM)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, std::string(fn) + ": unknown graph kind");
  if (C > kNgramMaxLabels)
    return fail(ctx, GTNB_ERR_UNSUPPORTED,
                std::string(fn) + ": C = " + std::to_string(C) +
                    " labels; the product builder and the trellis kernels take C <= " +
                    std::to_string(kNgramMaxLabels));
  return GTNB_OK;
}

/* the device route's numerators, build(view, &p) for every graph of the batch, and whether the implicit sweeps take
 * them all (the dense kinds' products are label-uniform, so C bears only on gtnb_sparse_transitions_loss's) */
template <class Build>
bool device_products(const GraphBatch& gb, Build&& build, std::vector<ProductGraph>* prods) {
  prods->resize(gb.B);
  std::vector<SgDims> dims(gb.B);
  for (int b = 0; b < gb.B; b++) {
    ProductGraph& p = (*prods)[b];
    build(gb.views[b], &p);
    dims[b] = SgDims{(int)p.flags.size(), (int)p.src.size(), p.n_acc, /*all_valid=*/1, p.uniform ? 1 : 0, p.max_in,
                     p.max_out};
  }
  return implicit_dims_supported(dims.data(), gb.B, gb.C);
}

/* trellis_loss_fast's numerator for the user graphs: the (folded) products, weighted by launch_product_fold */
struct GraphNumerator {
  const GraphBatch& gb;
  const std::vector<ProductGraph>& prods;
  int n_w; // slots of Wx before sigma: the transition count
  float* arc_grads;
  int arc_grads_on_device;
  bool arc_labels = false; // some product is not label-uniform: k_implicit.cu's arc-label instantiations
  long long tot_A = 0;
  std::vector<gtnb_graph_view> pviews;
  std::vector<int32_t> tidx_h, arc_of_h;
  std::vector<float> w_A_h;
  int32_t *map = nullptr, *arc_of = nullptr, *Tb_dev = nullptr;
  float *w_A = nullptr, *fw = nullptr;
  const float* e_dev = nullptr;
  long long per = 0;
  OutBuf ag;

  bool wants_arc_grads() const { return arc_grads != nullptr; }
  int alloc(CallScope& scope, const float* e, long long stride, gtnb_lattice**) {
    const int B = gb.B;
    const long long tot_arcs = gb.tot_arcs;
    e_dev = e;
    per = stride;
    pviews.resize(B);
    for (int b = 0; b < B; b++) {
      pviews[b] = prods[b].view();
      tidx_h.insert(tidx_h.end(), prods[b].tidx.begin(), prods[b].tidx.end());
      for (int32_t k : prods[b].arc_of) arc_of_h.push_back((int32_t)(gb.first_arc[b] + k));
      arc_labels |= !prods[b].uniform;
    }
    tot_A = (long long)tidx_h.size();
    GTNB_TRY(scope.alloc(&Tb_dev, B));
    GTNB_TRY(scope.alloc(&map, tot_A));
    GTNB_TRY(scope.alloc(&arc_of, tot_A));
    GTNB_TRY(scope.alloc(&fw, tot_A));
    if (!gb.arc_weights_dev) {
      w_A_h.assign(tot_arcs, 0.0f);
      for (int b = 0; b < B; b++) {
        const gtnb_graph_view& v = gb.views[b];
        if (v.weights) std::copy(v.weights, v.weights + v.num_arcs, w_A_h.begin() + gb.first_arc[b]);
      }
      GTNB_TRY(scope.alloc(&w_A, tot_arcs));
    }
    if (arc_grads) {
      GTNB_TRY(scope.output(arc_grads, arc_grads_on_device, tot_arcs, &ag));
      if (tot_arcs) GTNB_CUDA(scope.ctx(), cudaMemsetAsync(ag.dev, 0, sizeof(float) * tot_arcs, scope.ctx()->stream));
    }
    return GTNB_OK;
  }
  int stage(CallScope& scope, gtnb_lattice*) {
    gtnb_ctx* ctx = scope.ctx();
    GTNB_TRY(stage_upload(ctx, Tb_dev, gb.Tb.data(), sizeof(int32_t) * gb.Tb.size()));
    if (tot_A) {
      GTNB_TRY(stage_upload(ctx, map, tidx_h.data(), sizeof(int32_t) * tot_A));
      GTNB_TRY(stage_upload(ctx, arc_of, arc_of_h.data(), sizeof(int32_t) * tot_A));
    }
    if (!gb.arc_weights_dev && gb.tot_arcs)
      GTNB_TRY(stage_upload(ctx, w_A, w_A_h.data(), sizeof(float) * gb.tot_arcs));
    return GTNB_OK;
  }
  const int32_t* T_dev() const { return Tb_dev; }
  int build(CallScope& scope, gtnb_lattice*& lat, const float* w_dev, const float* sigma) {
    gtnb_ctx* ctx = scope.ctx();
    GTNB_TRY(launch_product_fold(ctx, tot_A, gb.arc_weights_dev ? gb.arc_weights_dev : w_A, arc_of, w_dev, n_w, sigma,
                                 map, fw));
    // the dense kinds' products are label-uniform: the plain instantiations, with the folded weights gathered into
    // the tables
    return compose_linear_impl(ctx, (int)pviews.size(), pviews.data(), (int)pviews.size(), 0, gb.Tb.data(), gb.C,
                               e_dev, per, true, &lat, arc_labels, fw);
  }
  int scatter(CallScope& scope, const float* ggrad) {
    if (!arc_grads) return GTNB_OK;
    GTNB_TRY(launch_scatter_add(scope.ctx(), ag.dev, arc_of, ggrad, tot_A));
    return ag.copy_out(scope.ctx(), gb.tot_arcs);
  }
};

/*
 * The materialised route of gtnb_graph_transitions_loss and gtnb_sparse_transitions_loss: make_G(W, &G, &gmap)
 * builds G from the n_trans host weights W, gmap holding the trans_w slot of each of G's arcs; unfold(view, &p)
 * builds the unfolded products, which are weighted on the host.  built (nullable): the device route's products,
 * taken as they are where folding changes nothing (ASG).
 */
template <class MakeG, class Unfold>
int transitions_exact(CallScope& scope, const TransitionArgs& a, const GraphBatch& gb, long long n_trans,
                      MakeG&& make_G, Unfold&& unfold, const std::vector<ProductGraph>* built, float* arc_grads,
                      int arc_grads_on_device) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = gb.B;
  std::vector<float> W(std::max(n_trans, 1ll)), host_w;
  if (n_trans) GTNB_TRY(read_to_host(ctx, W.data(), a.trans_w, a.trans_on_device, n_trans));
  std::vector<gtnb_graph_view> views;
  GTNB_TRY(gb.host_views(ctx, &host_w, &views));
  HostGraph G;
  std::vector<int32_t> gmap;
  make_G(W.data(), &G, &gmap);
  std::vector<ProductGraph> unfolded(built ? 0 : B);
  const std::vector<ProductGraph>& prods = built ? *built : unfolded;
  std::vector<std::vector<float>> pw(B);
  std::vector<gtnb_graph_view> pviews(B);
  std::vector<int32_t> pmap, arc_of;
  for (int b = 0; b < B; b++) {
    if (!built) unfold(views[b], &unfolded[b]);
    product_weights(prods[b], views[b].weights, W.data(), &pw[b]);
    pviews[b] = prods[b].view();
    pviews[b].weights = pw[b].data();
    pmap.insert(pmap.end(), prods[b].tidx.begin(), prods[b].tidx.end());
    for (int32_t k : prods[b].arc_of) arc_of.push_back((int32_t)(gb.first_arc[b] + k));
  }
  OutBuf ag;
  if (arc_grads) GTNB_TRY(scope.output(arc_grads, arc_grads_on_device, gb.tot_arcs, &ag));
  return transitions_loss_materialised(scope, a, gb.Tb.data(), G, gmap, n_trans, pviews, pmap, &arc_of,
                                       arc_grads ? &ag : nullptr, gb.tot_arcs);
}

} // namespace

extern "C" int gtnb_graph_transitions_loss(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const gtnb_graph_view* graphs, const float* arc_weights, int arc_weights_on_device, int kind,
    const float* trans_w, int trans_on_device, float* losses_host, float* grads, int grads_on_device,
    float* arc_grads, int arc_grads_on_device, float* trans_grad, int trans_grad_on_device) {
  const char* fn = "gtnb_graph_transitions_loss";
  GraphBatch gb;
  GTNB_TRY(parse_graphs(ctx, fn, B, T, C, emissions, graphs, trans_w && (B == 0 || losses_host), input_lens,
                        arc_weights, arc_weights_on_device, &gb, [&] { return check_dense_kind(ctx, fn, kind, C); }));
  const bool bigram = kind == GTNB_DENSE_BIGRAM;
  const TransitionArgs a{B, T, C, emissions, emissions_on_device, input_lens, trans_w, trans_on_device, nullptr,
                         nullptr, -1, losses_host, grads, grads_on_device, trans_grad, trans_grad_on_device};
  const long long n_trans = dense_trans_count(bigram, C);
  // the device route's numerators (BIGRAM: folded), whose shapes decide whether it can be taken
  std::vector<ProductGraph> prods;
  const bool fits = device_products(
      gb, [&](const gtnb_graph_view& v, ProductGraph* p) { build_product(v, C, bigram, /*fold=*/true, p); }, &prods);
  TrellisCriterion k = bigram ? TrellisCriterion{n_trans, (long long)B * (T + 1) * C, /*fold=*/true,
                                                       launch_ngram_den_forward, launch_ngram_den_backward}
                                    : TrellisCriterion{n_trans, asg_alpha_floats(B, T, C), /*fold=*/false,
                                                       launch_asg_den_forward, launch_asg_den_backward};
  return run_criterion(ctx, B, gb.Tb.data(), losses_host, trans_grad, trans_grad_on_device, n_trans,
                       ctx->use_implicit && fits, [&](CallScope& scope, bool f, bool* needs_exact) {
                         if (!f)
                           return transitions_exact(
                               scope, a, gb, n_trans,
                               [&](const float* W, HostGraph* G, std::vector<int32_t>* gmap) {
                                 dense_graph(bigram, C, W, G, gmap);
                               },
                               [&](const gtnb_graph_view& v, ProductGraph* p) {
                                 build_product(v, C, bigram, /*fold=*/false, p);
                               },
                               bigram ? nullptr : &prods, arc_grads, arc_grads_on_device);
                         GraphNumerator num{gb, prods, (int)n_trans, arc_grads, arc_grads_on_device};
                         return trellis_loss_fast(scope, k, a, num, needs_exact);
                       });
}

/*
 * Loss over user-supplied target graphs with a learned transition graph G of any shape (an epsilon-free acceptor:
 * n-gram graphs of any order, pruned token LMs, HMM topologies; the intersect(emissions, transitions) pattern of the
 * reference's benchmarks/ctc.cpp and examples):
 *   loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(A_b, G), E_b))
 * with E_b, A_b and the arc weights of gtnb_graph_transitions_loss and G's weights in trans_w by arc id.  The device
 * route sweeps the denominator with k_sparse.cu over G's tables and the folded products of gtnb_product.h with
 * k_implicit.cu (trellis_loss_fast); a non-finite value, the implicit flag off, or a G or product outside the
 * kernels' layout take the materialised lattices with the unfolded products.
 */
namespace {

/* G's tables and start groups (gtnb_product.h) in one device buffer: pack() them, then alloc() the buffer from a call's
 * scratch and stage() it, or place() them at a buffer of packed.size() words the caller owns (gtnb_transitions) */
struct SparseDevTables {
  std::vector<int32_t> packed;
  std::vector<size_t> at;
  int S = 0, A = 0;
  int32_t* tab = nullptr;
  SparseDev dev{};
  const int32_t *grp_ptr = nullptr, *grp_arc = nullptr;

  void pack(const SparseTables& t) {
    S = t.S, A = t.A;
    packed.assign(t.flags.begin(), t.flags.end());
    at.clear();
    for (const std::vector<int32_t>* v : {&t.in_ptr, &t.in_src, &t.in_lab, &t.in_arc, &t.out_ptr, &t.out_dst,
                                          &t.out_lab, &t.out_arc, &t.grp_ptr, &t.grp_arc}) {
      at.push_back(packed.size());
      packed.insert(packed.end(), v->begin(), v->end());
    }
  }
  void place(int32_t* buf) {
    tab = buf;
    dev = SparseDev{S, A, sparse_den_lanes(S, A), tab, tab + at[0], tab + at[1], tab + at[2], tab + at[3],
                    tab + at[4], tab + at[5], tab + at[6], tab + at[7]};
    grp_ptr = tab + at[8];
    grp_arc = tab + at[9];
  }
  int alloc(CallScope& scope, const SparseTables& t) {
    pack(t);
    int32_t* buf = nullptr;
    GTNB_TRY(scope.alloc(&buf, (long long)packed.size()));
    place(buf);
    return GTNB_OK;
  }
  int stage(CallScope& scope) { return stage_upload(scope.ctx(), tab, packed.data(), sizeof(int32_t) * packed.size()); }
};

/*
 * Which of k_sparse.cu's kernels sweep an epsilon-free G = t: true when some do, with sp->N = 1 for the one-CTA
 * kernels and sp = the plan of a thread-block cluster otherwise.  The "sparse_cluster" flag decides: 0 the one-CTA
 * kernels or nothing; 1 the cluster kernels for a G outside the one-CTA envelope; 2, 4, 8 a cluster of that size
 * wherever it fits, the rule of 1 elsewhere.
 */
bool sparse_route(const gtnb_ctx* ctx, const SparseTables& t, int C, SparseSplit* sp) {
  const int flag = ctx->sparse_cluster;
  if (flag > 1 && sparse_cluster_plan(t, C, flag, sp)) return true;
  sp->N = 1;
  if (sparse_den_supported(t.S, t.A, C)) return true;
  return flag != 0 && sparse_cluster_plan(t, C, 0, sp) != 0;
}

/* G's arcs with a label in [0, C), weighted from the host weights W; gmap (nullable) gets each one's arc id */
void sparse_host_graph(const gtnb_graph_view& Gv, const SparseTables& t, int C, const float* W, HostGraph* G,
                       std::vector<int32_t>* gmap) {
  G->flags = t.flags;
  for (int g = 0; g < Gv.num_arcs; g++)
    if (Gv.arc_olabel[g] >= 0 && Gv.arc_olabel[g] < C) {
      G->arc(Gv.arc_src[g], Gv.arc_dst[g], Gv.arc_olabel[g], W[g]);
      if (gmap) gmap->push_back(g);
    }
}

/* trellis_loss_fast's denominator for a G of any shape: G's tables and start groups in one device buffer */
struct SparseDenominator {
  const SparseTables& t;
  long long n_trans; // G's arcs, labels outside [0, C) included
  SparseSplit split; // sparse_route's: N = 1 the one-CTA sweeps, else a cluster's
  SparseDevTables tabs;
  float* alpha = nullptr;
  double* offs = nullptr;

  int groups() const { return (int)t.grp_ptr.size() - 1; }
  long long n_sigma(int) const { return groups(); }
  int alloc(CallScope& scope, int B, int T) {
    GTNB_TRY(tabs.alloc(scope, t));
    GTNB_TRY(scope.alloc(&alpha, (long long)B * (T + 1) * t.S));
    return scope.alloc(&offs, (long long)B * (T + 1));
  }
  int stage(CallScope& scope) { return tabs.stage(scope); }
  int sigma(gtnb_ctx* ctx, int, const float* w, float* sig) {
    return launch_sparse_sigma(ctx, groups(), tabs.grp_ptr, tabs.grp_arc, w, sig);
  }
  int forward(gtnb_ctx* ctx, int B, int T, int C, const int32_t* lens, const float* e, long long per, const float* w,
              float* den, int32_t* status) {
    return launch_sparse_den_forward(ctx, tabs.dev, split, B, T, C, lens, e, per, w, alpha, offs, den, status);
  }
  int backward(gtnb_ctx* ctx, int B, int T, int C, const int32_t* lens, const float* e, long long per, const float* w,
               const float*, float* grad, float* wgrad) {
    return launch_sparse_den_backward(ctx, tabs.dev, split, B, T, C, lens, e, per, w, alpha, offs, grad, per, wgrad);
  }
  int fold_grad(gtnb_ctx* ctx, int, const float* w, const float* sig, float* wgrad) {
    return launch_sparse_fold(ctx, groups(), tabs.grp_ptr, tabs.grp_arc, (int)n_trans, w, sig, wgrad);
  }
};

/* the checks of gtnb_sparse_transitions_loss's transition graph; epsilon (the backoff entry points): epsilon arcs,
 * GTNB_EPSILON on both sides, are G's own */
int check_transition_graph(gtnb_ctx* ctx, const std::string& fn, const gtnb_graph_view& Gv, bool epsilon = false) {
  if (validate_view(ctx, Gv)) return GTNB_ERR_INVALID_ARGUMENT;
  if (Gv.num_nodes < 1) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the transition graph has no nodes");
  for (int g = 0; g < Gv.num_arcs; g++) {
    if (!epsilon && (Gv.arc_ilabel[g] == GTNB_EPSILON || Gv.arc_olabel[g] == GTNB_EPSILON))
      return fail(ctx, GTNB_ERR_UNSUPPORTED,
                  fn + ": the transition graph has epsilon arcs; remove them first (remove(g, epsilon))");
    if (Gv.arc_ilabel[g] != Gv.arc_olabel[g])
      return fail(ctx, GTNB_ERR_UNSUPPORTED,
                  fn + ": the transition graph is a transducer; make it an acceptor first (projectInput / "
                       "projectOutput)");
  }
  return GTNB_OK;
}

/* gtnb_sparse_transitions_loss after its checks, t = sparse_tables(Gv); also gtnb_backoff_transitions_loss's route for
 * an epsilon-free G */
int sparse_transitions_loss_run(gtnb_ctx* ctx, const TransitionArgs& a, const GraphBatch& gb, const gtnb_graph_view& Gv,
                                const SparseTables& t, float* arc_grads, int arc_grads_on_device) {
  const int B = a.B, C = a.C;
  const long long n_trans = Gv.num_arcs;
  // the device route's numerators (folded), whose shapes decide, with G's, whether it can be taken
  std::vector<ProductGraph> prods;
  SparseSplit split{};
  const bool fast = ctx->use_implicit && sparse_route(ctx, t, C, &split) &&
                    device_products(
                        gb,
                        [&](const gtnb_graph_view& v, ProductGraph* p) {
                          build_sparse_product(v, Gv, t, C, /*fold=*/true, p);
                        },
                        &prods);
  return run_criterion(ctx, B, gb.Tb.data(), a.losses_host, a.trans_grad, a.trans_grad_on_device, n_trans, fast,
                       [&](CallScope& scope, bool f, bool* needs_exact) {
                         if (!f)
                           return transitions_exact(
                               scope, a, gb, n_trans,
                               [&](const float* W, HostGraph* G, std::vector<int32_t>* gmap) {
                                 sparse_host_graph(Gv, t, C, W, G, gmap);
                               },
                               [&](const gtnb_graph_view& v, ProductGraph* p) {
                                 build_sparse_product(v, Gv, t, C, /*fold=*/false, p);
                               },
                               nullptr, arc_grads, arc_grads_on_device);
                         SparseDenominator den{t, n_trans, split};
                         GraphNumerator num{gb, prods, (int)n_trans, arc_grads, arc_grads_on_device};
                         return trellis_loss_fast(scope, den, a, num, needs_exact);
                       });
}

} // namespace

extern "C" int gtnb_sparse_transitions_loss(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const gtnb_graph_view* graphs, const float* arc_weights, int arc_weights_on_device,
    const gtnb_graph_view* transitions, const float* trans_w, int trans_on_device, float* losses_host, float* grads,
    int grads_on_device, float* arc_grads, int arc_grads_on_device, float* trans_grad, int trans_grad_on_device) {
  const std::string fn = "gtnb_sparse_transitions_loss";
  GraphBatch gb;
  GTNB_TRY(parse_graphs(ctx, fn.c_str(), B, T, C, emissions, graphs,
                        transitions && (B == 0 || (losses_host && trans_w)), input_lens, arc_weights,
                        arc_weights_on_device, &gb, [&] { return check_transition_graph(ctx, fn, *transitions); }));
  const TransitionArgs a{B, T, C, emissions, emissions_on_device, input_lens, trans_w, trans_on_device, nullptr,
                         nullptr, -1, losses_host, grads, grads_on_device, trans_grad, trans_grad_on_device};
  SparseTables t;
  sparse_tables(*transitions, C, &t);
  return sparse_transitions_loss_run(ctx, a, gb, *transitions, t, arc_grads, arc_grads_on_device);
}

/*
 * Viterbi alignment over user-supplied target graphs: viterbiPath / viterbiScore of compose(A_b, E_b), with E_b, A_b,
 * the arc weights, the olabel matching and the epsilon rule of gtnb_graph_loss.  The device route sweeps
 * intersect(A_b, E_b) in the tropical semiring without building it and traces the path back from the saved score
 * rows (k_implicit.cu).  An utterance whose trace met a tie (with exact_ties on) or whose sweep met a non-finite
 * value is re-run alone on the materialised route, which breaks ties as the reference does; the whole batch takes
 * that route when the graphs do not fit the implicit layout or the implicit flag is off.
 */
namespace {

struct GraphViterbiArgs {
  const float* emissions;
  int emissions_on_device;
  int32_t* paths;
  int32_t* arcs;
  float* scores;
  int outputs_on_device;
};

/* the device buffers of a graph Viterbi call: the emissions, the outputs (the user's own when they are on the
 * device) and one zeroed status word per utterance */
struct ViterbiBufs {
  float *e_dev = nullptr, *s_dev = nullptr;
  int32_t *p_dev = nullptr, *a_dev = nullptr, *status = nullptr;
};

/* 0, 1, ... as long as the largest view's arc list: the arc ids a view's ilabels are replaced with */
std::vector<int32_t> arc_ids(const std::vector<gtnb_graph_view>& views) {
  int max_arcs = 0;
  for (const gtnb_graph_view& v : views) max_arcs = std::max(max_arcs, v.num_arcs);
  std::vector<int32_t> ids(std::max(max_arcs, 1));
  for (int k = 0; k < max_arcs; k++) ids[k] = k;
  return ids;
}

/*
 * The materialised route for the utterances `which`: gtnb_compose_linear (the lattice is put in the reference's
 * relaxation order while exact_ties is on, k_order.cu), gtnb_forward(tropical) for the score and gtnb_viterbi_path.
 * views: one per utterance, with host weights.  A_b is matched on its olabels, so its ilabels play no part in the
 * composition: they are replaced by the arc ids, which the path's ilabels then carry back.  linear_first
 * (gtnb_viterbi_sparse): views holds one graph G shared by the batch, matched on its ilabels, and the lattice is
 * compose(E_b, G) -- the reference's intersect(E_b, G) -- with G's olabels replaced by the arc ids instead.  The rows
 * are written into the device outputs v.p_dev / v.a_dev (nullable) and v.s_dev.  arc_map (nullable): per utterance,
 * the arc the caller reports for each arc of views[b] (gtnb_graph_transitions_viterbi: views[b] is compose(A_b, G),
 * the map its gradInfo into A_b).  The utterances run in groups whose lattices fit the device memory together (a
 * tie-heavy batch does not materialise every lattice at once); one that does not fit alone is
 * GTNB_ERR_UNSUPPORTED, from gtnb_compose_linear.
 */
int graph_viterbi_exact(CallScope& scope, const GraphBatch& gb, const std::vector<gtnb_graph_view>& views,
                        const ViterbiBufs& v, const std::vector<int>& which,
                        const std::vector<std::vector<int32_t>>* arc_map = nullptr, bool linear_first = false) {
  gtnb_ctx* ctx = scope.ctx();
  const int T = gb.T, C = gb.C, ml = std::max(T, 1);
  const long long per = (long long)T * C;
  const std::vector<int32_t> ids = arc_ids(views);
  // the utterances with frames (T_b = 0 accepts nothing) and their emission rows, contiguous
  std::vector<int> sub;
  for (int b : which)
    if (gb.Tb[b] > 0) sub.push_back(b);
  const int n = (int)sub.size();
  std::vector<float> sc(std::max(n, 1), -std::numeric_limits<float>::infinity());
  std::vector<int32_t> parc((size_t)std::max(n, 1) * ml, -1), plab(parc.size(), -1), plen(std::max(n, 1), -1);
  const float* e_sub = v.e_dev;
  if (n > 0 && n < gb.B) {
    float* e_copy = nullptr;
    GTNB_TRY(scope.alloc(&e_copy, per * n));
    for (int k = 0; k < n; k++)
      GTNB_CUDA(ctx, cudaMemcpyAsync(e_copy + per * k, v.e_dev + per * sub[k], sizeof(float) * per,
                                     cudaMemcpyDeviceToDevice, ctx->stream));
    e_sub = e_copy;
  }
  // the groups' budget: half of the device memory still free (this call's own buffers, e.g. the decode's
  // back-pointers, already count as used), the rest left to gtnb_forward and gtnb_viterbi_path
  size_t free_b = 0, total_b = 0;
  GTNB_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
  const unsigned long long budget = std::min<unsigned long long>(free_b, ctx->total_mem ? ctx->total_mem : free_b) / 2;
  for (int k0 = 0, k1 = 0; k0 < n; k0 = k1) {
    // the group [k0, k1): the bytes gtnb_compose_linear asks for its lattice (gtnb_capi.cu: every graph's node, arc
    // and level slabs, then one alive bit per frame and node of the largest graph), within the budget
    unsigned long long slabs = 0;
    long long maxN = 0, maxT = 0;
    for (; k1 < n; k1++) {
      const gtnb_graph_view& g = views[linear_first ? 0 : sub[k1]];
      const long long Tb = gb.Tb[sub[k1]], N = g.num_nodes;
      const unsigned long long s = 8ull * align_up((Tb + 1) * N + 1, kAlign) +
                                   20ull * align_up(std::max(Tb * g.num_arcs, 1ll), kAlign) +
                                   8ull * align_up(Tb + 2, kAlign);
      const long long mN = std::max(maxN, N), mT = std::max(maxT, Tb);
      const unsigned long long need = slabs + s + 4ull * (k1 - k0 + 1) * (mT + 1) * ((mN + 31) / 32);
      if (k1 > k0 && need > budget) break;
      slabs += s;
      maxN = mN;
      maxT = mT;
    }
    const int m = k1 - k0;
    std::vector<gtnb_graph_view> sv(linear_first ? 1 : m);
    std::vector<int32_t> sT(m);
    for (int k = 0; k < m; k++) {
      if (k < (int)sv.size()) {
        sv[k] = views[linear_first ? 0 : sub[k0 + k]];
        (linear_first ? sv[k].arc_olabel : sv[k].arc_ilabel) = ids.data();
      }
      sT[k] = gb.Tb[sub[k0 + k]];
    }
    gtnb_lattice*& lat = scope.lattice();
    GTNB_TRY(gtnb_compose_linear(ctx, m, sv.data(), (int)sv.size(), linear_first ? 1 : 0, sT.data(), C,
                                 e_sub + per * k0, per, &lat));
    GTNB_TRY(gtnb_forward(ctx, lat, 1, sc.data() + k0, nullptr));
    // the arc ids are the path's ilabels (A_b) or olabels (G, linear_first)
    int32_t* ia = (linear_first ? plab : parc).data() + (size_t)k0 * ml;
    int32_t* oa = (linear_first ? parc : plab).data() + (size_t)k0 * ml;
    GTNB_TRY(gtnb_viterbi_path(ctx, lat, ml, nullptr, ia, oa, nullptr, plen.data() + k0, nullptr));
    gtnb_lattice_destroy(ctx, lat); // (gtnb_viterbi_path has synchronised)
    lat = nullptr;
  }
  // the rows of every utterance in `which` (T_b = 0: score -inf, no path), staged on the host and copied from
  // pageable memory (each copy has left the host buffer when it returns)
  const size_t nw = which.size();
  std::vector<int32_t> prow(nw * ml), arow(nw * ml);
  std::vector<float> srow(nw);
  size_t k = 0;
  for (size_t j = 0; j < nw; j++) {
    const int b = which[j];
    const bool run = k < sub.size() && sub[k] == b;
    const int len = run ? plen[k] : -1;
    for (int t = 0; t < T; t++) {
      prow[j * ml + t] = t < len ? plab[k * ml + t] : -1;
      arow[j * ml + t] = t >= len ? -1 : arc_map ? (*arc_map)[b][parc[k * ml + t]] : parc[k * ml + t];
    }
    srow[j] = run ? sc[k] : -std::numeric_limits<float>::infinity();
    if (v.p_dev && T > 0)
      GTNB_CUDA(ctx, cudaMemcpyAsync(v.p_dev + (long long)b * T, &prow[j * ml], sizeof(int32_t) * T,
                                     cudaMemcpyHostToDevice, ctx->stream));
    if (v.a_dev && T > 0)
      GTNB_CUDA(ctx, cudaMemcpyAsync(v.a_dev + (long long)b * T, &arow[j * ml], sizeof(int32_t) * T,
                                     cudaMemcpyHostToDevice, ctx->stream));
    GTNB_CUDA(ctx, cudaMemcpyAsync(v.s_dev + b, &srow[j], sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    k += run;
  }
  return scope.sync();
}

int viterbi_open(CallScope& scope, const GraphViterbiArgs& a, const GraphBatch& gb, ViterbiBufs* v) {
  gtnb_ctx* ctx = scope.ctx();
  const long long nrow = (long long)gb.B * gb.T;
  const bool dev_out = a.outputs_on_device != 0;
  GTNB_TRY(scope.input(a.emissions, a.emissions_on_device, (long long)gb.T * gb.C * gb.B, &v->e_dev));
  GTNB_TRY(scope.borrow(a.scores, a.scores && dev_out, gb.B, &v->s_dev));
  if (a.paths) GTNB_TRY(scope.borrow(a.paths, dev_out, nrow, &v->p_dev));
  if (a.arcs) GTNB_TRY(scope.borrow(a.arcs, dev_out, nrow, &v->a_dev));
  GTNB_TRY(scope.alloc(&v->status, gb.B));
  GTNB_CUDA(ctx, cudaMemsetAsync(v->status, 0, sizeof(int32_t) * gb.B, ctx->stream));
  return GTNB_OK;
}

/*
 * The tail both graph Viterbi calls share.  implicit: the device route has written every row, and one status word
 * per utterance decides which re-run alone on the exact route: bit 1 a non-finite value, bit 2 a tie on the traced
 * path while exact_ties is on.  Otherwise every utterance takes the exact route.  exact(which) writes the rows of
 * `which`; then host outputs are copied out.
 */
template <typename Exact>
int viterbi_finish(CallScope& scope, const GraphViterbiArgs& a, const GraphBatch& gb, bool implicit,
                   const ViterbiBufs& v, Exact&& exact) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = gb.B;
  const long long nrow = (long long)B * gb.T;
  std::vector<int> which;
  if (implicit) {
    GTNB_TRY(readback_reserve(ctx, sizeof(int32_t) * B));
    int32_t* st = reinterpret_cast<int32_t*>(ctx->readback);
    GTNB_CUDA(ctx, cudaMemcpyAsync(st, v.status, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, ctx->stream));
    GTNB_TRY(scope.sync());
    for (int b = 0; b < B; b++)
      if (gb.Tb[b] > 0 && ((st[b] & 1) || ((st[b] & 2) && ctx->exact_ties))) which.push_back(b);
  } else {
    for (int b = 0; b < B; b++) which.push_back(b);
  }
  if (!which.empty()) GTNB_TRY(exact(which));
  if (!a.outputs_on_device) {
    if (a.scores)
      GTNB_CUDA(ctx, cudaMemcpyAsync(a.scores, v.s_dev, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    if (a.paths && nrow)
      GTNB_CUDA(ctx, cudaMemcpyAsync(a.paths, v.p_dev, sizeof(int32_t) * nrow, cudaMemcpyDeviceToHost, ctx->stream));
    if (a.arcs && nrow)
      GTNB_CUDA(ctx, cudaMemcpyAsync(a.arcs, v.a_dev, sizeof(int32_t) * nrow, cudaMemcpyDeviceToHost, ctx->stream));
  }
  return scope.sync();
}

int graph_viterbi_run(CallScope& scope, const GraphViterbiArgs& a, const GraphBatch& gb) {
  gtnb_ctx* ctx = scope.ctx();
  ViterbiBufs v;
  GTNB_TRY(viterbi_open(scope, a, gb, &v));
  bool implicit = ctx->use_implicit;
  gtnb_lattice*& lat = scope.lattice();
  if (implicit) {
    GTNB_TRY(implicit_or_materialise(compose_linear_impl(ctx, gb.B, gb.views.data(), gb.B, 0, gb.Tb.data(), gb.C,
                                                         v.e_dev, (long long)gb.T * gb.C, true, &lat, true,
                                                         gb.arc_weights_dev),
                                     &implicit));
    implicit = implicit && implicit_trace_supported(lat);
  }
  if (implicit) {
    GTNB_TRY(launch_implicit_forward(ctx, lat, v.status, 0, -1, /*tropical=*/true));
    GTNB_TRY(launch_implicit_trace(ctx, lat, v.status, v.p_dev, v.a_dev, v.s_dev, gb.T));
  }
  return viterbi_finish(scope, a, gb, implicit, v, [&](const std::vector<int>& which) {
    std::vector<float> host_w;
    std::vector<gtnb_graph_view> views;
    GTNB_TRY(gb.host_views(ctx, &host_w, &views));
    return graph_viterbi_exact(scope, gb, views, v, which);
  });
}

} // namespace

extern "C" int gtnb_graph_viterbi(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const gtnb_graph_view* graphs, const float* arc_weights, int arc_weights_on_device, int32_t* paths, int32_t* arcs,
    float* scores, int outputs_on_device) {
  GraphBatch gb;
  GTNB_TRY(parse_graphs(ctx, "gtnb_graph_viterbi", B, T, C, emissions, graphs, true, input_lens, arc_weights,
                        arc_weights_on_device, &gb, no_own_checks));
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  CallScope scope(ctx);
  return graph_viterbi_run(scope, GraphViterbiArgs{emissions, emissions_on_device, paths, arcs, scores,
                                                   outputs_on_device},
                           gb);
}

/*
 * Viterbi alignment over user-supplied target graphs with learned transitions: viterbiPath / viterbiScore of the
 * numerators of gtnb_graph_transitions_loss, compose(compose(A_b, G), E_b) for ASG and
 * intersect(intersect(A_b, G), E_b) for BIGRAM.  The device route sweeps the loss's products (gtnb_product.h, BIGRAM
 * folded) in the tropical semiring, with weights folded on the device from the transitions where they lie; BIGRAM's
 * folded start arcs read tau_l = max_j W[l][j] there instead of sigma_l.  The trace reports product arcs, which
 * launch_product_arc_map takes back to A_b's.  The exact route composes A_b with G in the reference's own numbering
 * (gtnb_compose_graphs) and runs graph_viterbi_exact on the result, so ties break as the reference breaks them.
 */
namespace {

/* the exact route for the utterances `which`: compose(A'_b, G) on the device in the reference's numbering, G (gv,
 * host weights) the second operand, then graph_viterbi_exact through the composed graphs' gradInfo into A_b */
int graph_transitions_viterbi_exact(CallScope& scope, const char* fn, const GraphBatch& gb, const gtnb_graph_view& gv,
                                    const ViterbiBufs& vb, const std::vector<int>& which) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = gb.B;
  std::vector<float> host_w;
  std::vector<gtnb_graph_view> views;
  GTNB_TRY(gb.host_views(ctx, &host_w, &views));
  // A'_b: A_b with its ilabels replaced by the arc ids (A_b is matched on its olabels, so the composition is the
  // same); the pairs that can accept anything
  const std::vector<int32_t> ids = arc_ids(views);
  std::vector<int> pairs;
  std::vector<gtnb_graph_view> first;
  for (int b : which) {
    if (gb.Tb[b] == 0 || views[b].num_nodes == 0) continue;
    gtnb_graph_view v = views[b];
    v.arc_ilabel = ids.data();
    pairs.push_back(b);
    first.push_back(v);
  }
  const int n = (int)pairs.size();
  // the composed graphs on the host, in the reference's numbering; arc_map[b]: the A_b arc of each of their arcs
  struct Composed {
    std::vector<uint8_t> flags;
    std::vector<int32_t> src, dst, il, ol;
    std::vector<float> w;
  };
  std::vector<Composed> cg(n);
  std::vector<std::vector<int32_t>> arc_map(B);
  std::vector<gtnb_graph_view> cviews(B);
  for (auto& v : cviews) std::memset(&v, 0, sizeof(v)); // (utterances without a pair: the empty graph)
  if (n > 0) {
    std::vector<int32_t> kind(n, 0); // the reference's unsorted matcher
    gtnb_composed* res = nullptr;
    GTNB_TRY(gtnb_compose_graphs(ctx, n, first.data(), n, &gv, 1, kind.data(), &res));
    int rc = GTNB_OK;
    for (int k = 0; k < n && rc == GTNB_OK; k++) {
      int32_t N = 0, A = 0;
      rc = gtnb_composed_sizes(res, k, &N, &A);
      if (rc != GTNB_OK) {
        rc = fail(ctx, rc, std::string(fn) + ": sizes of a composed graph");
        break;
      }
      Composed& c = cg[k];
      c.flags.resize(std::max(N, 1));
      for (auto* x : {&c.src, &c.dst, &c.il, &c.ol}) x->resize(std::max(A, 1));
      c.w.resize(std::max(A, 1));
      std::vector<int32_t>& m = arc_map[pairs[k]];
      m.resize(std::max(A, 1));
      rc = gtnb_composed_download(ctx, res, k, c.flags.data(), c.src.data(), c.dst.data(), c.il.data(), c.ol.data(),
                                  c.w.data(), m.data(), nullptr);
      gtnb_graph_view& v = cviews[pairs[k]];
      v.num_nodes = N;
      v.num_arcs = A;
      v.node_flags = c.flags.data();
      v.arc_src = c.src.data();
      v.arc_dst = c.dst.data();
      v.arc_ilabel = c.il.data();
      v.arc_olabel = c.ol.data();
      v.weights = c.w.data();
    }
    gtnb_composed_destroy(ctx, res);
    GTNB_TRY(rc);
  }
  return graph_viterbi_exact(scope, gb, cviews, vb, which, &arc_map);
}

/* the weights of the folded start arcs of a dense kind's products: BIGRAM's tau_l = max_j W[l][j], none for ASG */
struct DenseTau {
  bool bigram;
  int C;
  float* tau = nullptr;
  int alloc(CallScope& scope) { return bigram ? scope.alloc(&tau, C) : GTNB_OK; }
  int stage(CallScope&) { return GTNB_OK; }
  int launch(gtnb_ctx* ctx, const float* w) { return bigram ? launch_ngram_tau(ctx, C, w, tau) : GTNB_OK; }
};

/* ... and of a G of any shape: tau_k = max over G's start group k (gtnb_product.h) */
struct SparseTau {
  const SparseTables& t;
  std::vector<int32_t> packed;
  int32_t* tab = nullptr;
  float* tau = nullptr;
  int groups() const { return (int)t.grp_ptr.size() - 1; }
  int alloc(CallScope& scope) {
    packed = t.grp_ptr;
    packed.insert(packed.end(), t.grp_arc.begin(), t.grp_arc.end());
    GTNB_TRY(scope.alloc(&tab, (long long)packed.size()));
    return scope.alloc(&tau, std::max(groups(), 1));
  }
  int stage(CallScope& scope) { return stage_upload(scope.ctx(), tab, packed.data(), sizeof(int32_t) * packed.size()); }
  int launch(gtnb_ctx* ctx, const float* w) {
    return launch_sparse_tau(ctx, groups(), tab, tab + t.grp_ptr.size(), w, tau);
  }
};

/*
 * The Viterbi alignment of the transitions losses' numerators.  prods: the device route's (folded) products, taken
 * when `fast`; tau: the weights of their folded start arcs, slots n_trans... of Wx; make_G(W, &G): G from the
 * n_trans host weights, for the exact route.
 */
template <class Tau, class MakeG>
int transitions_viterbi_run(CallScope& scope, const char* fn, const GraphViterbiArgs& a, const GraphBatch& gb,
                            const std::vector<ProductGraph>& prods, bool fast, long long n_trans, const float* trans_w,
                            int trans_on_device, Tau& tau, MakeG&& make_G) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = gb.B, T = gb.T, C = gb.C;
  ViterbiBufs v;
  GTNB_TRY(viterbi_open(scope, a, gb, &v));
  bool implicit = ctx->use_implicit && fast;
  GraphNumerator num{gb, prods, (int)n_trans, nullptr, 0};
  gtnb_lattice*& lat = scope.lattice();
  if (implicit) {
    GTNB_TRY(num.alloc(scope, v.e_dev, (long long)T * C, nullptr));
    float* w_dev = nullptr;
    long long* off = nullptr;
    GTNB_TRY(scope.borrow(trans_w, trans_on_device != 0, std::max(n_trans, 1ll), &w_dev));
    GTNB_TRY(tau.alloc(scope));
    // off: every utterance's first product arc, then its first A arc (launch_product_arc_map)
    std::vector<long long> off_h(2 * (size_t)B, 0);
    for (int b = 0; b < B; b++) {
      if (b > 0) off_h[b] = off_h[b - 1] + (long long)prods[b - 1].src.size();
      off_h[B + b] = gb.first_arc[b];
    }
    if (v.a_dev) GTNB_TRY(scope.alloc(&off, 2ll * B));
    GTNB_TRY(stage_begin(ctx));
    GTNB_TRY(num.stage(scope, nullptr));
    GTNB_TRY(tau.stage(scope));
    if (!trans_on_device) GTNB_TRY(stage_upload(ctx, w_dev, trans_w, sizeof(float) * n_trans));
    if (off) GTNB_TRY(stage_upload(ctx, off, off_h.data(), sizeof(long long) * 2 * B));
    GTNB_TRY(stage_end(ctx));
    GTNB_TRY(tau.launch(ctx, w_dev));
    GTNB_TRY(implicit_or_materialise(num.build(scope, lat, w_dev, tau.tau), &implicit));
    implicit = implicit && implicit_trace_supported(lat);
    if (implicit) {
      GTNB_TRY(launch_implicit_forward(ctx, lat, v.status, 0, -1, /*tropical=*/true));
      GTNB_TRY(launch_implicit_trace(ctx, lat, v.status, v.p_dev, v.a_dev, v.s_dev, T));
      if (v.a_dev) GTNB_TRY(launch_product_arc_map(ctx, B, T, off, num.arc_of, v.a_dev));
    }
  }
  return viterbi_finish(scope, a, gb, implicit, v, [&](const std::vector<int>& which) {
    std::vector<float> W(std::max(n_trans, 1ll));
    if (n_trans) GTNB_TRY(read_to_host(ctx, W.data(), trans_w, trans_on_device, n_trans));
    HostGraph G;
    make_G(W.data(), &G);
    return graph_transitions_viterbi_exact(scope, fn, gb, G.view(), v, which);
  });
}

int graph_transitions_viterbi_run(CallScope& scope, const GraphViterbiArgs& a, const GraphBatch& gb, bool bigram,
                                  const float* trans_w, int trans_on_device) {
  const int C = gb.C;
  // the loss's numerators (BIGRAM folded), whose shapes decide whether the device route can be taken
  std::vector<ProductGraph> prods;
  const bool fits = device_products(
      gb, [&](const gtnb_graph_view& view, ProductGraph* p) { build_product(view, C, bigram, /*fold=*/true, p); },
      &prods);
  DenseTau tau{bigram, C};
  return transitions_viterbi_run(scope, "gtnb_graph_transitions_viterbi", a, gb, prods, fits,
                                 dense_trans_count(bigram, C), trans_w, trans_on_device, tau,
                                 [&](const float* W, HostGraph* G) { dense_graph(bigram, C, W, G, nullptr); });
}

} // namespace

extern "C" int gtnb_graph_transitions_viterbi(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const gtnb_graph_view* graphs, const float* arc_weights, int arc_weights_on_device, int kind,
    const float* trans_w, int trans_on_device, int32_t* paths, int32_t* arcs, float* scores, int outputs_on_device) {
  const char* fn = "gtnb_graph_transitions_viterbi";
  GraphBatch gb;
  GTNB_TRY(parse_graphs(ctx, fn, B, T, C, emissions, graphs, trans_w != nullptr, input_lens, arc_weights,
                        arc_weights_on_device, &gb, [&] { return check_dense_kind(ctx, fn, kind, C); }));
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  CallScope scope(ctx);
  return graph_transitions_viterbi_run(scope,
                                       GraphViterbiArgs{emissions, emissions_on_device, paths, arcs, scores,
                                                        outputs_on_device},
                                       gb, kind == GTNB_DENSE_BIGRAM, trans_w, trans_on_device);
}

/*
 * Viterbi decoding and alignment with a learned transition graph G of any shape (gtnb_sparse_transitions_loss's G):
 *   gtnb_viterbi_sparse:              viterbiPath / viterbiScore of intersect(E_b, G), the decode;
 *   gtnb_sparse_transitions_viterbi:  ... of intersect(intersect(A_b, G), E_b), the loss's numerator.
 * The decode's device route sweeps G's tables in the tropical semiring (k_sparse.cu) and traces the path back from
 * 16-bit back-pointers; its exact route composes E_b with G, G's olabels replaced by its arc ids, so that the path's
 * olabels carry the arcs back.  The alignment is graph_transitions_viterbi's sequence with the loss's folded sparse
 * products, whose folded start arcs weigh tau_k = max over G's start group k.  Both take their exact route per
 * utterance on a non-finite value or a tie (exact_ties on), and for the whole batch outside the kernels' layout or
 * with the implicit flag off; only the exact routes read trans_w to the host.
 */
namespace {

int viterbi_sparse_run(CallScope& scope, const GraphViterbiArgs& a, const GraphBatch& gb, const gtnb_graph_view& Gv,
                       const float* trans_w, int trans_on_device) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = gb.B, T = gb.T, C = gb.C;
  const long long n_trans = Gv.num_arcs;
  ViterbiBufs v;
  GTNB_TRY(viterbi_open(scope, a, gb, &v));
  SparseTables t;
  sparse_tables(Gv, C, &t);
  SparseSplit split{};
  const bool implicit = ctx->use_implicit && sparse_route(ctx, t, C, &split);
  if (implicit) {
    SparseDevTables tabs;
    GTNB_TRY(tabs.alloc(scope, t));
    float* w_dev = nullptr;
    int32_t *T_dev = nullptr, *head = nullptr;
    uint16_t* bp = nullptr;
    GTNB_TRY(scope.borrow(trans_w, trans_on_device != 0, std::max(n_trans, 1ll), &w_dev));
    GTNB_TRY(scope.alloc(&T_dev, B));
    GTNB_TRY(scope.alloc(&head, B));
    GTNB_TRY(scope.alloc(&bp, std::max((long long)B * T * t.S, 1ll)));
    GTNB_TRY(stage_begin(ctx));
    GTNB_TRY(tabs.stage(scope));
    GTNB_TRY(stage_upload(ctx, T_dev, gb.Tb.data(), sizeof(int32_t) * B));
    if (!trans_on_device) GTNB_TRY(stage_upload(ctx, w_dev, trans_w, sizeof(float) * n_trans));
    GTNB_TRY(stage_end(ctx));
    GTNB_TRY(launch_sparse_viterbi(ctx, tabs.dev, split, B, T, C, T_dev, v.e_dev, (long long)T * C, w_dev, bp, head,
                                   v.s_dev, v.p_dev, v.a_dev, v.status));
  }
  return viterbi_finish(scope, a, gb, implicit, v, [&](const std::vector<int>& which) {
    std::vector<float> W(std::max(n_trans, 1ll));
    if (n_trans) GTNB_TRY(read_to_host(ctx, W.data(), trans_w, trans_on_device, n_trans));
    gtnb_graph_view g = Gv;
    g.weights = W.data();
    return graph_viterbi_exact(scope, gb, {g}, v, which, nullptr, /*linear_first=*/true);
  });
}

} // namespace

extern "C" int gtnb_viterbi_sparse(gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
                                   const int32_t* input_lens, const gtnb_graph_view* transitions, const float* trans_w,
                                   int trans_on_device, int32_t* paths, int32_t* arcs, float* scores,
                                   int outputs_on_device) {
  const std::string fn = "gtnb_viterbi_sparse";
  if (!ctx || B < 0 || T < 0 || C <= 0 || !transitions || (B > 0 && (!emissions || !trans_w)))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  GTNB_TRY(check_transition_graph(ctx, fn, *transitions));
  GraphBatch gb; // the batch without target graphs: its lengths
  gb.B = B, gb.T = T, gb.C = C;
  gb.Tb.resize(B);
  for (int b = 0; b < B; b++) {
    gb.Tb[b] = input_lens ? input_lens[b] : T;
    if (gb.Tb[b] < 0 || gb.Tb[b] > T) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": input_lens outside [0, T]");
  }
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  CallScope scope(ctx);
  return viterbi_sparse_run(scope, GraphViterbiArgs{emissions, emissions_on_device, paths, arcs, scores,
                                                    outputs_on_device},
                            gb, *transitions, trans_w, trans_on_device);
}

extern "C" int gtnb_sparse_transitions_viterbi(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const gtnb_graph_view* graphs, const float* arc_weights, int arc_weights_on_device,
    const gtnb_graph_view* transitions, const float* trans_w, int trans_on_device, int32_t* paths, int32_t* arcs,
    float* scores, int outputs_on_device) {
  const std::string fn = "gtnb_sparse_transitions_viterbi";
  GraphBatch gb;
  GTNB_TRY(parse_graphs(ctx, fn.c_str(), B, T, C, emissions, graphs, transitions && (B == 0 || trans_w), input_lens,
                        arc_weights, arc_weights_on_device, &gb,
                        [&] { return check_transition_graph(ctx, fn, *transitions); }));
  if (B == 0) return GTNB_OK;
  const gtnb_graph_view& Gv = *transitions;
  SparseTables t;
  sparse_tables(Gv, C, &t);
  // the loss's numerators (folded), whose shapes decide, with G's, whether the device route can be taken
  std::vector<ProductGraph> prods;
  SparseSplit split{}; // (the alignment sweeps the products alone: only whether G has a device route matters)
  const bool fast = ctx->use_implicit && sparse_route(ctx, t, C, &split) &&
                    device_products(
                        gb,
                        [&](const gtnb_graph_view& v, ProductGraph* p) {
                          build_sparse_product(v, Gv, t, C, /*fold=*/true, p);
                        },
                        &prods);
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  CallScope scope(ctx);
  SparseTau tau{t};
  return transitions_viterbi_run(
      scope, fn.c_str(), GraphViterbiArgs{emissions, emissions_on_device, paths, arcs, scores, outputs_on_device}, gb, prods, fast,
      Gv.num_arcs, trans_w, trans_on_device, tau,
      [&](const float* W, HostGraph* G) { sparse_host_graph(Gv, t, C, W, G, nullptr); });
}

/*
 * Loss and Viterbi decoding with a backoff transition graph G: the formulas of gtnb_sparse_transitions_loss and
 * gtnb_viterbi_sparse with epsilon arcs in G (ilabel == olabel == GTNB_EPSILON), the backoff arcs of a pruned n-gram
 * LM.  An epsilon arc moves G without consuming a frame, at any frame 0 .. T_b, and weighs its trans_w alone
 * (compose.cpp:139-205).  An epsilon-free G takes the sparse entry points' own routes.  Otherwise the device route
 * sweeps the denominator over G's tables and the numerators P_b = A_b o G (gtnb_product.h, unfolded, with G's
 * epsilon arcs) over their own tables, one CTA each, with k_sparse.cu's sparse_eps_* kernels, and the decode sweeps G
 * in the tropical semiring.  The exact route composes E_b with G, and P_b with E_b, in the reference's numbering
 * (gtnb_compose_graphs, which composes epsilon arcs), then runs gtnb_forward / gtnb_backward / gtnb_viterbi_path, one
 * utterance at a time.
 */
namespace {

/* acceptors with epsilon arcs (SparseTables with its epsilon tables) in one device buffer for the sparse_eps_*
 * kernels: add() every graph, its arc ids shifted by arc_base and its score rows at `rows`, then alloc(), stage(); or
 * place() them at buffers the caller owns (packed.size() words and desc.size() descriptors; gtnb_transitions) */
struct EpsDevTables {
  std::vector<int32_t> packed;
  std::vector<std::vector<size_t>> at; // per graph: where each of its tables starts in packed
  std::vector<SparseEpsDev> desc;
  int32_t* tab = nullptr;
  SparseEpsDev* dev = nullptr;
  int max_S = 1, max_AE = 0;

  void add(const SparseTables& t, int32_t arc_base, long long rows) {
    std::vector<size_t> o{packed.size()};
    packed.insert(packed.end(), t.flags.begin(), t.flags.end());
    auto put = [&](const std::vector<int32_t>& v, int32_t shift) {
      o.push_back(packed.size());
      for (int32_t x : v) packed.push_back(x + shift);
    };
    for (auto* v : {&t.in_ptr, &t.in_src, &t.in_lab}) put(*v, 0);
    put(t.in_arc, arc_base);
    for (auto* v : {&t.out_ptr, &t.out_dst, &t.out_lab}) put(*v, 0);
    put(t.out_arc, arc_base);
    put(t.eps_in_ptr, 0);
    put(t.eps_in_src, 0);
    put(t.eps_in_arc, arc_base);
    put(t.eps_out_ptr, 0);
    put(t.eps_out_dst, 0);
    put(t.eps_out_arc, arc_base);
    for (auto* v : {&t.fwd_ptr, &t.fwd_node, &t.bwd_ptr, &t.bwd_node, &t.lanes}) put(*v, 0);
    at.push_back(o);
    SparseEpsDev d{};
    d.g.S = t.S;
    d.g.A = t.A;
    d.g.lanes = sparse_den_lanes(t.S, t.A);
    d.E = t.E;
    d.L = t.L;
    d.rows = rows;
    desc.push_back(d);
    max_S = std::max(max_S, t.S);
    max_AE = std::max(max_AE, t.A + t.E);
  }
  int alloc(CallScope& scope) {
    int32_t* t = nullptr;
    SparseEpsDev* d = nullptr;
    GTNB_TRY(scope.alloc(&t, (long long)packed.size()));
    GTNB_TRY(scope.alloc(&d, (long long)desc.size()));
    place(t, d);
    return GTNB_OK;
  }
  /* desc's pointers into tab_buf; dev = dev_buf, which then takes desc */
  void place(int32_t* tab_buf, SparseEpsDev* dev_buf) {
    tab = tab_buf;
    dev = dev_buf;
    for (size_t i = 0; i < desc.size(); i++) {
      const int32_t* p[20];
      for (int j = 0; j < 20; j++) p[j] = tab + at[i][j];
      SparseEpsDev& d = desc[i];
      d.g.flags = p[0];
      d.g.in_ptr = p[1], d.g.in_src = p[2], d.g.in_lab = p[3], d.g.in_arc = p[4];
      d.g.out_ptr = p[5], d.g.out_dst = p[6], d.g.out_lab = p[7], d.g.out_arc = p[8];
      d.eps_in_ptr = p[9], d.eps_in_src = p[10], d.eps_in_arc = p[11];
      d.eps_out_ptr = p[12], d.eps_out_dst = p[13], d.eps_out_arc = p[14];
      d.fwd_ptr = p[15], d.fwd_node = p[16], d.bwd_ptr = p[17], d.bwd_node = p[18], d.lanes = p[19];
    }
  }
  int stage(CallScope& scope) {
    GTNB_TRY(stage_upload(scope.ctx(), tab, packed.data(), sizeof(int32_t) * packed.size()));
    return stage_upload(scope.ctx(), dev, desc.data(), sizeof(SparseEpsDev) * desc.size());
  }
};

bool eps_fits(const SparseTables& t, int C) { return sparse_eps_supported(t.S, t.A, t.E, t.L, t.max_in_all, C); }

/*
 * sparse_route for a G with epsilon arcs (t with its epsilon tables): true when k_sparse.cu has kernels for its
 * denominator, with sp->N = 1 for the one-CTA sparse_eps_* kernels and sp = the plan of a thread-block cluster (the
 * sparse_cl_eps_* kernels) otherwise.  The "sparse_cluster" flag decides as there: 0 the one-CTA kernels or nothing;
 * 1 a cluster for a G outside the one-CTA envelope; 2, 4, 8 a cluster of that size wherever it fits, the rule of 1
 * elsewhere.  The numerators keep the one-CTA kernels and their envelope (backoff_products).
 */
bool backoff_route(const gtnb_ctx* ctx, const SparseTables& t, int C, SparseSplit* sp) {
  const int flag = ctx->sparse_cluster;
  if (flag > 1 && sparse_cluster_plan(t, C, flag, sp)) return true;
  sp->N = 1;
  if (eps_fits(t, C)) return true;
  return flag != 0 && sparse_cluster_plan(t, C, 0, sp) != 0;
}

/* the checks of the backoff entry points' G, and its tables (with the epsilon tables) into t: a cycle of epsilon arcs
 * has no finite closure (the reference's forwardScore and viterbi throw "Graph has a cycle", shortest.cpp:150, 230) */
int check_backoff_graph(gtnb_ctx* ctx, const std::string& fn, const gtnb_graph_view& Gv, int C, SparseTables* t) {
  GTNB_TRY(check_transition_graph(ctx, fn, Gv, /*epsilon=*/true));
  sparse_tables(Gv, C, t);
  sparse_eps_tables(Gv, t);
  if (t->cycle.empty()) return GTNB_OK;
  std::string path;
  for (int32_t v : t->cycle) path += std::to_string(v) + " -> ";
  return fail(ctx, GTNB_ERR_INVALID_ARGUMENT,
              fn + ": the transition graph has a cycle of epsilon arcs: " + path + std::to_string(t->cycle[0]));
}

/* the device route's numerators P_b = A_b o G (unfolded, with G's epsilon arcs) into prods and their tables into
 * ptabs, for the whole batch; false, at the first that does not fit the backoff envelope */
bool backoff_products(const GraphBatch& gb, const gtnb_graph_view& Gv, const SparseTables& t, int C,
                      std::vector<ProductGraph>* prods, std::vector<SparseTables>* ptabs) {
  prods->resize(gb.B);
  ptabs->resize(gb.B);
  for (int b = 0; b < gb.B; b++) {
    build_sparse_product(gb.views[b], Gv, t, C, /*fold=*/false, &(*prods)[b]);
    const gtnb_graph_view pv = (*prods)[b].view();
    sparse_tables(pv, C, &(*ptabs)[b]);
    sparse_eps_tables(pv, &(*ptabs)[b]);
    if (!eps_fits((*ptabs)[b], C)) return false;
  }
  return true;
}

/* the numerators' device tables, one graph per CTA with its rows ((T_b + 1) * S_b entries) after the previous
 * utterance's, and the product arcs' A arc (arc_of, -1 for G's epsilon arcs) and G arc (tidx) in the batch's
 * numbering; -> the rows of the batch */
long long backoff_numerators(const GraphBatch& gb, const std::vector<ProductGraph>& prods,
                             const std::vector<SparseTables>& ptabs, EpsDevTables* num_t,
                             std::vector<int32_t>* arc_of, std::vector<int32_t>* tidx) {
  long long rows = 0;
  for (int b = 0; b < gb.B; b++) {
    num_t->add(ptabs[b], (int32_t)tidx->size(), rows);
    rows += (long long)(gb.Tb[b] + 1) * ptabs[b].S;
    for (int32_t k : prods[b].arc_of) arc_of->push_back(k < 0 ? -1 : (int32_t)(gb.first_arc[b] + k));
    tidx->insert(tidx->end(), prods[b].tidx.begin(), prods[b].tidx.end());
  }
  return rows;
}

/* the batch's host arc weights in its numbering into w_A (an arc without weights: 0) when they are not on the device;
 * -> whether there are any to upload */
bool host_arc_weights(const GraphBatch& gb, std::vector<float>* w_A) {
  if (gb.arc_weights_dev) return false;
  w_A->assign((size_t)std::max(gb.tot_arcs, 1ll), 0.0f);
  for (int b = 0; b < gb.B; b++) {
    const gtnb_graph_view& v = gb.views[b];
    if (v.weights) std::copy(v.weights, v.weights + v.num_arcs, w_A->begin() + gb.first_arc[b]);
  }
  return true;
}

/* the device route of gtnb_backoff_transitions_loss: ptabs[b] the tables of prods[b] (P_b = A_b o G, unfolded);
 * split: backoff_route's, a cluster's plan for the denominator when split.N > 1 */
int backoff_loss_fast(CallScope& scope, const TransitionArgs& a, const GraphBatch& gb, long long n_trans,
                      const SparseTables& t, const SparseSplit& split, const std::vector<ProductGraph>& prods,
                      const std::vector<SparseTables>& ptabs, float* arc_grads, int arc_grads_on_device,
                      bool* needs_exact) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = a.B, T = a.T, C = a.C;
  const long long per = (long long)T * C, tot_arcs = gb.tot_arcs;
  const bool want = a.grads || a.trans_grad || arc_grads;
  EpsDevTables den_t, num_t;
  den_t.add(t, 0, 0);
  std::vector<int32_t> arc_of_h, tidx_h;
  const long long rows = backoff_numerators(gb, prods, ptabs, &num_t, &arc_of_h, &tidx_h);
  const long long tot_P = (long long)tidx_h.size();
  std::vector<float> w_A_h;
  std::vector<int32_t> cut_h;
  if (split.N > 1) sparse_eps_cluster_cuts(t, split, &cut_h);
  float *e_dev = nullptr, *w_dev = nullptr, *den = nullptr, *num = nullptr, *alpha_d = nullptr, *alpha_n = nullptr;
  float *fw = nullptr, *w_A = nullptr, *pgrad = nullptr;
  double *offs_d = nullptr, *offs_n = nullptr;
  int32_t *status = nullptr, *T_dev = nullptr, *arc_of = nullptr, *tidx = nullptr, *cut = nullptr;
  OutBuf g, tg, ag;
  GTNB_TRY(ensure_side_streams(ctx, 0, 0));
  GTNB_TRY(scope.input(a.emissions, a.emissions_on_device, per * B, &e_dev));
  GTNB_TRY(scope.borrow(a.trans_w, a.trans_on_device != 0, n_trans, &w_dev)); // (host: staged below)
  GTNB_TRY(scope.alloc(&status, 2ll * B));
  GTNB_TRY(scope.alloc(&den, B));
  GTNB_TRY(scope.alloc(&num, B));
  GTNB_TRY(scope.alloc(&T_dev, B));
  GTNB_TRY(scope.alloc(&offs_d, (long long)B * (T + 1)));
  GTNB_TRY(scope.alloc(&offs_n, (long long)B * (T + 1)));
  GTNB_TRY(scope.alloc(&alpha_d, (long long)B * (T + 1) * t.S));
  GTNB_TRY(scope.alloc(&alpha_n, rows));
  GTNB_TRY(scope.alloc(&fw, tot_P));
  GTNB_TRY(scope.alloc(&arc_of, tot_P));
  GTNB_TRY(scope.alloc(&tidx, tot_P));
  GTNB_TRY(den_t.alloc(scope));
  GTNB_TRY(num_t.alloc(scope));
  if (!cut_h.empty()) GTNB_TRY(scope.alloc(&cut, (long long)cut_h.size()));
  if (host_arc_weights(gb, &w_A_h)) GTNB_TRY(scope.alloc(&w_A, (long long)w_A_h.size()));
  if (want) {
    GTNB_TRY(scope.output(a.grads, a.grads_on_device, per * B, &g));
    GTNB_TRY(scope.output(a.trans_grad, a.trans_grad_on_device, n_trans, &tg));
    GTNB_TRY(scope.output(arc_grads, arc_grads_on_device, tot_arcs, &ag));
    GTNB_TRY(scope.alloc(&pgrad, tot_P));
    GTNB_CUDA(ctx, cudaMemsetAsync(g.dev, 0, sizeof(float) * per * B, ctx->stream));
    if (n_trans) GTNB_CUDA(ctx, cudaMemsetAsync(tg.dev, 0, sizeof(float) * n_trans, ctx->stream));
    if (tot_arcs) GTNB_CUDA(ctx, cudaMemsetAsync(ag.dev, 0, sizeof(float) * tot_arcs, ctx->stream));
    if (tot_P) GTNB_CUDA(ctx, cudaMemsetAsync(pgrad, 0, sizeof(float) * tot_P, ctx->stream));
  }
  GTNB_CUDA(ctx, cudaMemsetAsync(status, 0, sizeof(int32_t) * 2 * B, ctx->stream));
  GTNB_TRY(stage_begin(ctx));
  GTNB_TRY(den_t.stage(scope));
  GTNB_TRY(num_t.stage(scope));
  if (cut) GTNB_TRY(stage_upload(ctx, cut, cut_h.data(), sizeof(int32_t) * cut_h.size()));
  GTNB_TRY(stage_upload(ctx, T_dev, gb.Tb.data(), sizeof(int32_t) * B));
  if (tot_P) {
    GTNB_TRY(stage_upload(ctx, arc_of, arc_of_h.data(), sizeof(int32_t) * tot_P));
    GTNB_TRY(stage_upload(ctx, tidx, tidx_h.data(), sizeof(int32_t) * tot_P));
  }
  if (!a.trans_on_device && n_trans) GTNB_TRY(stage_upload(ctx, w_dev, a.trans_w, sizeof(float) * n_trans));
  if (w_A) GTNB_TRY(stage_upload(ctx, w_A, w_A_h.data(), sizeof(float) * w_A_h.size()));
  GTNB_TRY(stage_end(ctx));
  GTNB_TRY(launch_sparse_eps_gather(ctx, tot_P, gb.arc_weights_dev ? gb.arc_weights_dev : w_A, arc_of, w_dev, tidx, fw));
  // the numerators (small, one graph per CTA) on the second stream beside the denominator (G for every CTA); both
  // add into the zero-filled emission rows with red.add
  GTNB_TRY(fork_to(ctx, ctx->copy_stream));
  {
    OnStream side(ctx, ctx->copy_stream);
    const SparseSplit one{1}; // the numerators: one CTA each
    GTNB_TRY(launch_sparse_eps_forward(ctx, num_t.dev, one, nullptr, 1, num_t.max_S, B, T, C, T_dev, e_dev, per, fw,
                                       alpha_n, offs_n, num, status + B));
    if (want)
      GTNB_TRY(launch_sparse_eps_backward(ctx, num_t.dev, one, nullptr, 1, num_t.max_S, num_t.max_AE, B, T, C, T_dev,
                                          e_dev, per, fw, alpha_n, offs_n, -1.0f, g.dev, per, pgrad));
  }
  GTNB_TRY(launch_sparse_eps_forward(ctx, den_t.dev, split, cut, 0, t.S, B, T, C, T_dev, e_dev, per, w_dev, alpha_d,
                                     offs_d, den, status));
  if (want)
    GTNB_TRY(launch_sparse_eps_backward(ctx, den_t.dev, split, cut, 0, t.S, t.A + t.E, B, T, C, T_dev, e_dev, per, w_dev,
                                        alpha_d, offs_d, 1.0f, g.dev, per, tg.dev));
  GTNB_TRY(join_from(ctx, ctx->copy_stream));
  if (want) {
    GTNB_TRY(launch_sparse_eps_scatter(ctx, tot_P, pgrad, arc_of, tidx, tg.dev, arc_grads ? ag.dev : nullptr));
    GTNB_TRY(g.copy_out(ctx, per * B));
    GTNB_TRY(tg.copy_out(ctx, n_trans));
    GTNB_TRY(ag.copy_out(ctx, tot_arcs));
  }
  return read_losses(scope, B, den, num, status, 2ll * B, a.losses_host, needs_exact);
}

/* the composed graph of one pair, downloaded: gi1 / gi2 the arcs of the two operands behind each arc (-1: none) */
struct ComposedHost {
  std::vector<uint8_t> flags;
  std::vector<int32_t> src, dst, il, ol, gi1, gi2;
  std::vector<float> w;
  int N = 0, A = 0;
  gtnb_graph_view view() const {
    gtnb_graph_view v;
    std::memset(&v, 0, sizeof(v));
    v.num_nodes = N;
    v.num_arcs = A;
    v.node_flags = flags.data();
    v.arc_src = src.data();
    v.arc_dst = dst.data();
    v.arc_ilabel = il.data();
    v.arc_olabel = ol.data();
    v.weights = w.data();
    return v;
  }
};

/* compose(first, second) in the reference's numbering; kind: the matcher (gtnb_compose_graphs) */
int compose_host(gtnb_ctx* ctx, const gtnb_graph_view& first, const gtnb_graph_view& second, int32_t kind,
                 ComposedHost* c) {
  gtnb_composed* res = nullptr;
  GTNB_TRY(gtnb_compose_graphs(ctx, 1, &first, 1, &second, 1, &kind, &res));
  int rc = gtnb_composed_sizes(res, 0, &c->N, &c->A);
  if (rc == GTNB_OK) {
    c->flags.resize(std::max(c->N, 1));
    for (auto* v : {&c->src, &c->dst, &c->il, &c->ol, &c->gi1, &c->gi2}) v->resize(std::max(c->A, 1));
    c->w.resize(std::max(c->A, 1));
    rc = gtnb_composed_download(ctx, res, 0, c->flags.data(), c->src.data(), c->dst.data(), c->il.data(), c->ol.data(),
                                c->w.data(), c->gi1.data(), c->gi2.data());
  }
  gtnb_composed_destroy(ctx, res);
  return rc;
}

/* E_b = linearGraph(T_b, C) on host rows e ([T_b][C]): arc t * C + c goes t -> t + 1 with label c.  The reference's
 * linearGraph is marked arc-sorted (creations.cpp:30-31), so it composes with the sorted matcher on its side. */
void linear_host(int Tb, int C, const float* e, HostGraph* E) {
  E->flags.assign(Tb + 1, 0);
  E->flags[0] |= 1;
  E->flags[Tb] |= 2;
  for (int t = 0; t < Tb; t++)
    for (int c = 0; c < C; c++) E->arc(t, t + 1, c, e[(long long)t * C + c]);
}

/* n floats from the host into a user buffer on the device or the host */
int write_user(gtnb_ctx* ctx, float* user, int on_device, const float* host, long long n) {
  if (!user || n <= 0) return GTNB_OK;
  if (!on_device) {
    std::memcpy(user, host, sizeof(float) * n);
    return GTNB_OK;
  }
  GTNB_CUDA(ctx, cudaMemcpyAsync(user, host, sizeof(float) * n, cudaMemcpyHostToDevice, ctx->stream));
  GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return GTNB_OK;
}

/*
 * The exact route of gtnb_backoff_transitions_loss, one utterance at a time: the denominator compose(E_b, G) and the
 * numerator compose(P_b, E_b) (P_b unfolded, weighted on the host) in the reference's numbering, packed into one
 * lattice, gtnb_forward and gtnb_backward with +1 / -1, and the arc gradients taken back through the compositions'
 * gradInfo.  Reproduces the reference's inf / NaN propagation arc by arc.
 */
int backoff_loss_exact(CallScope& scope, const TransitionArgs& a, const GraphBatch& gb, const gtnb_graph_view& Gv,
                       const SparseTables& t, float* arc_grads, int arc_grads_on_device) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = a.B, T = a.T, C = a.C;
  const long long per = (long long)T * C, n_trans = Gv.num_arcs, tot_arcs = gb.tot_arcs;
  const bool want = a.grads || a.trans_grad || arc_grads;
  std::vector<float> W(std::max(n_trans, 1ll)), host_w, e((size_t)std::max(per * B, 1ll));
  if (n_trans) GTNB_TRY(read_to_host(ctx, W.data(), a.trans_w, a.trans_on_device, n_trans));
  if (per * B) GTNB_TRY(read_to_host(ctx, e.data(), a.emissions, a.emissions_on_device, per * B));
  std::vector<gtnb_graph_view> views;
  GTNB_TRY(gb.host_views(ctx, &host_w, &views));
  gtnb_graph_view G = Gv;
  G.weights = W.data();
  std::vector<float> gh(want ? (size_t)std::max(per * B, 1ll) : 0, 0.0f), agh((size_t)std::max(tot_arcs, 1ll), 0.0f);
  std::vector<double> tgd((size_t)std::max(n_trans, 1ll), 0.0);
  for (int b = 0; b < B; b++) {
    const int Tb = gb.Tb[b];
    if (Tb == 0) continue; // (NaN, no gradient: run_criterion)
    HostGraph E;
    linear_host(Tb, C, e.data() + per * b, &E);
    const gtnb_graph_view Ev = E.view();
    ProductGraph p;
    build_sparse_product(views[b], Gv, t, C, /*fold=*/false, &p);
    std::vector<float> pw;
    product_weights(p, views[b].weights, W.data(), &pw);
    gtnb_graph_view pv = p.view();
    pv.weights = pw.data();
    ComposedHost cg[2];
    GTNB_TRY(compose_host(ctx, Ev, G, /*first sorted=*/1, &cg[0]));
    GTNB_TRY(compose_host(ctx, pv, Ev, /*second sorted=*/2, &cg[1]));
    // an empty composition (nothing reachable) scores -inf and has no gradient
    float sc[2] = {-std::numeric_limits<float>::infinity(), -std::numeric_limits<float>::infinity()};
    std::vector<gtnb_graph_view> lv;
    std::vector<int> which;
    for (int k = 0; k < 2; k++)
      if (cg[k].N > 0) {
        lv.push_back(cg[k].view());
        which.push_back(k);
      }
    if (!lv.empty()) {
      gtnb_lattice*& lat = scope.lattice();
      GTNB_TRY(gtnb_pack(ctx, (int)lv.size(), lv.data(), &lat));
      float s[2];
      GTNB_TRY(gtnb_forward(ctx, lat, 0, s, nullptr));
      for (size_t i = 0; i < which.size(); i++) sc[which[i]] = s[i];
      if (want) {
        float deltas[2];
        for (size_t i = 0; i < which.size(); i++) deltas[i] = which[i] == 0 ? 1.0f : -1.0f; // subtract's gradFunc
        GTNB_TRY(gtnb_backward(ctx, lat, 0, deltas));
        for (size_t i = 0; i < which.size(); i++) {
          const ComposedHost& c = cg[which[i]];
          std::vector<float> ga((size_t)std::max(c.A, 1));
          GTNB_TRY(gtnb_lattice_arc_grads(ctx, lat, (int)i, ga.data()));
          for (int k = 0; k < c.A; k++) {
            const float v = ga[k];
            // E_b is the first operand of the denominator and the second of the numerator
            const int ea = which[i] == 0 ? c.gi1[k] : c.gi2[k], oa = which[i] == 0 ? c.gi2[k] : c.gi1[k];
            if (ea >= 0) gh[per * b + ea] += v;
            if (oa < 0) continue;
            if (which[i] == 0) {
              tgd[oa] += v;
            } else {
              tgd[p.tidx[oa]] += v;
              if (p.arc_of[oa] >= 0) agh[gb.first_arc[b] + p.arc_of[oa]] += v;
            }
          }
        }
      }
      gtnb_lattice_destroy(ctx, lat);
      lat = nullptr;
    }
    a.losses_host[b] = sc[0] - sc[1];
  }
  if (!want) return GTNB_OK;
  std::vector<float> tgh(tgd.begin(), tgd.end());
  GTNB_TRY(write_user(ctx, a.grads, a.grads_on_device, gh.data(), per * B));
  GTNB_TRY(write_user(ctx, a.trans_grad, a.trans_grad_on_device, tgh.data(), n_trans));
  return write_user(ctx, arc_grads, arc_grads_on_device, agh.data(), tot_arcs);
}

int backoff_loss_run(gtnb_ctx* ctx, const TransitionArgs& a, const GraphBatch& gb, const gtnb_graph_view& Gv,
                     const SparseTables& t, float* arc_grads, int arc_grads_on_device) {
  const int B = a.B, C = a.C;
  const long long n_trans = Gv.num_arcs;
  // the device route's numerators and their tables, whose shapes decide, with G's, whether it can be taken
  std::vector<ProductGraph> prods;
  std::vector<SparseTables> ptabs;
  SparseSplit split{};
  const bool fast =
      ctx->use_implicit && backoff_route(ctx, t, C, &split) && backoff_products(gb, Gv, t, C, &prods, &ptabs);
  return run_criterion(ctx, B, gb.Tb.data(), a.losses_host, a.trans_grad, a.trans_grad_on_device, n_trans, fast,
                       [&](CallScope& scope, bool f, bool* needs_exact) {
                         if (!f) return backoff_loss_exact(scope, a, gb, Gv, t, arc_grads, arc_grads_on_device);
                         return backoff_loss_fast(scope, a, gb, n_trans, t, split, prods, ptabs, arc_grads,
                                                  arc_grads_on_device, needs_exact);
                       });
}

/*
 * The exact Viterbi route of the backoff entry points for the utterances `which`, one at a time: compose(b, E_b, &c)
 * composes utterance b's lattice c (E_b = linearGraph(T_b, C) on its rows) in the reference's numbering, then
 * gtnb_forward(tropical) and gtnb_viterbi_path run on it.  The path's arcs with an epsilon ilabel are G's epsilon
 * arcs, which use no frame and are not reported; of the others, the ilabel is the label and the olabel the reported
 * arc, or the other way round when arc_in.
 */
template <class Compose>
int eps_viterbi_exact(CallScope& scope, const GraphBatch& gb, const ViterbiBufs& v, const std::vector<int>& which,
                      bool arc_in, Compose&& compose) {
  gtnb_ctx* ctx = scope.ctx();
  const int T = gb.T, C = gb.C;
  const long long per = (long long)T * C;
  std::vector<float> e((size_t)std::max(per, 1ll));
  std::vector<int32_t> prow(std::max(T, 1)), arow(std::max(T, 1));
  for (int b : which) {
    const int Tb = gb.Tb[b];
    std::fill(prow.begin(), prow.end(), -1);
    std::fill(arow.begin(), arow.end(), -1);
    float score = -std::numeric_limits<float>::infinity();
    if (Tb > 0) {
      GTNB_TRY(read_to_host(ctx, e.data(), v.e_dev + per * b, 1, (long long)Tb * C));
      HostGraph E;
      linear_host(Tb, C, e.data(), &E);
      ComposedHost c;
      GTNB_TRY(compose(b, E.view(), &c));
      if (c.N > 0) {
        const gtnb_graph_view cv = c.view();
        gtnb_lattice*& lat = scope.lattice();
        GTNB_TRY(gtnb_pack(ctx, 1, &cv, &lat));
        float s = 0.0f;
        GTNB_TRY(gtnb_forward(ctx, lat, 1, &s, nullptr));
        const int ml = std::max(c.N, 1);
        std::vector<int32_t> pa(ml), il(ml), ol(ml);
        int32_t len = -1;
        GTNB_TRY(gtnb_viterbi_path(ctx, lat, ml, pa.data(), il.data(), ol.data(), nullptr, &len, nullptr));
        gtnb_lattice_destroy(ctx, lat);
        lat = nullptr;
        if (len >= 0) {
          score = s;
          for (int k = 0, f = 0; k < len; k++)
            if (il[k] != GTNB_EPSILON && f < T) {
              prow[f] = arc_in ? ol[k] : il[k];
              arow[f++] = arc_in ? il[k] : ol[k];
            }
        }
      }
    }
    if (v.p_dev && T > 0)
      GTNB_CUDA(ctx, cudaMemcpyAsync(v.p_dev + (long long)b * T, prow.data(), sizeof(int32_t) * T,
                                     cudaMemcpyHostToDevice, ctx->stream));
    if (v.a_dev && T > 0)
      GTNB_CUDA(ctx, cudaMemcpyAsync(v.a_dev + (long long)b * T, arow.data(), sizeof(int32_t) * T,
                                     cudaMemcpyHostToDevice, ctx->stream));
    GTNB_CUDA(ctx, cudaMemcpyAsync(v.s_dev + b, &score, sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    GTNB_TRY(scope.sync()); // (the rows are reused by the next utterance)
  }
  return GTNB_OK;
}

/* the exact route of gtnb_viterbi_backoff: compose(E_b, G'), G' = G with its arc ids as olabels (host weights W) */
int backoff_viterbi_exact(CallScope& scope, const GraphBatch& gb, const gtnb_graph_view& Gv, const float* W,
                          const ViterbiBufs& v, const std::vector<int>& which) {
  std::vector<int32_t> ids(std::max(Gv.num_arcs, 1));
  for (int k = 0; k < Gv.num_arcs; k++) ids[k] = k;
  gtnb_graph_view G = Gv;
  G.arc_olabel = ids.data();
  G.weights = W;
  return eps_viterbi_exact(scope, gb, v, which, /*arc_in=*/false,
                           [&](int, const gtnb_graph_view& E, ComposedHost* c) {
                             return compose_host(scope.ctx(), E, G, /*first sorted=*/1, c);
                           });
}

int backoff_viterbi_run(CallScope& scope, const GraphViterbiArgs& a, const GraphBatch& gb, const gtnb_graph_view& Gv,
                        const SparseTables& t, const float* trans_w, int trans_on_device) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = gb.B, T = gb.T, C = gb.C;
  const long long n_trans = Gv.num_arcs;
  ViterbiBufs v;
  GTNB_TRY(viterbi_open(scope, a, gb, &v));
  SparseSplit split{};
  const bool implicit = ctx->use_implicit && backoff_route(ctx, t, C, &split);
  if (implicit) {
    EpsDevTables tabs;
    tabs.add(t, 0, 0);
    GTNB_TRY(tabs.alloc(scope));
    std::vector<int32_t> cut_h;
    if (split.N > 1) sparse_eps_cluster_cuts(t, split, &cut_h);
    float* w_dev = nullptr;
    int32_t *T_dev = nullptr, *head = nullptr, *cut = nullptr;
    uint16_t* bp = nullptr;
    GTNB_TRY(scope.borrow(trans_w, trans_on_device != 0, std::max(n_trans, 1ll), &w_dev));
    GTNB_TRY(scope.alloc(&T_dev, B));
    GTNB_TRY(scope.alloc(&head, B));
    GTNB_TRY(scope.alloc(&bp, (long long)B * (T + 1) * t.S));
    if (!cut_h.empty()) GTNB_TRY(scope.alloc(&cut, (long long)cut_h.size()));
    GTNB_TRY(stage_begin(ctx));
    GTNB_TRY(tabs.stage(scope));
    if (cut) GTNB_TRY(stage_upload(ctx, cut, cut_h.data(), sizeof(int32_t) * cut_h.size()));
    GTNB_TRY(stage_upload(ctx, T_dev, gb.Tb.data(), sizeof(int32_t) * B));
    if (!trans_on_device && n_trans) GTNB_TRY(stage_upload(ctx, w_dev, trans_w, sizeof(float) * n_trans));
    GTNB_TRY(stage_end(ctx));
    GTNB_TRY(launch_sparse_eps_viterbi(ctx, tabs.dev, split, cut, t.S, B, T, C, T_dev, v.e_dev, (long long)T * C, w_dev,
                                       bp, head, v.s_dev, v.p_dev, v.a_dev, v.status));
  }
  return viterbi_finish(scope, a, gb, implicit, v, [&](const std::vector<int>& which) {
    std::vector<float> W(std::max(n_trans, 1ll));
    if (n_trans) GTNB_TRY(read_to_host(ctx, W.data(), trans_w, trans_on_device, n_trans));
    return backoff_viterbi_exact(scope, gb, Gv, W.data(), v, which);
  });
}

/*
 * The exact route of gtnb_backoff_transitions_viterbi: compose(compose(A'_b, G), E_b), A'_b = A_b with its arc ids
 * as ilabels (its olabels are matched, so the composition is the same) and G with its epsilon arcs and host weights
 * W, in the reference's numbering: the unsorted matcher for the first (graph_transitions_viterbi_exact's), E_b's side
 * sorted for the second (backoff_loss_exact's).  The path's ilabels are A_b's arcs and its olabels the labels.
 */
int backoff_align_exact(CallScope& scope, const GraphBatch& gb, const gtnb_graph_view& Gv, const float* W,
                        const ViterbiBufs& v, const std::vector<int>& which) {
  gtnb_ctx* ctx = scope.ctx();
  std::vector<float> host_w;
  std::vector<gtnb_graph_view> views;
  GTNB_TRY(gb.host_views(ctx, &host_w, &views));
  const std::vector<int32_t> ids = arc_ids(views);
  gtnb_graph_view G = Gv;
  G.weights = W;
  return eps_viterbi_exact(scope, gb, v, which, /*arc_in=*/true,
                           [&](int b, const gtnb_graph_view& E, ComposedHost* c) {
                             if (views[b].num_nodes == 0) return GTNB_OK; // (c->N = 0: no path)
                             gtnb_graph_view a = views[b];
                             a.arc_ilabel = ids.data();
                             ComposedHost num;
                             GTNB_TRY(compose_host(ctx, a, G, /*unsorted=*/0, &num));
                             if (num.N == 0) return GTNB_OK;
                             return compose_host(ctx, num.view(), E, /*second sorted=*/2, c);
                           });
}

/*
 * gtnb_backoff_transitions_viterbi for a G with epsilon arcs (t its tables).  The device route reuses the loss's
 * numerators and their tables (backoff_products, backoff_numerators): their weights are gathered on the device, and
 * sparse_eps_align_* sweep them one CTA each and trace the paths back to A_b's arcs.  viterbi_finish re-runs an
 * utterance on backoff_align_exact on a non-finite value or a tie (exact_ties on); the whole batch takes that route
 * outside the envelope or with the implicit flag off.  Only that route reads trans_w to the host.
 */
int backoff_align_run(CallScope& scope, const GraphViterbiArgs& a, const GraphBatch& gb, const gtnb_graph_view& Gv,
                      const SparseTables& t, const std::vector<ProductGraph>& prods,
                      const std::vector<SparseTables>& ptabs, bool fast, const float* trans_w, int trans_on_device) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = gb.B, T = gb.T, C = gb.C;
  const long long n_trans = Gv.num_arcs;
  ViterbiBufs v;
  GTNB_TRY(viterbi_open(scope, a, gb, &v));
  const bool implicit = ctx->use_implicit && fast;
  if (implicit) {
    EpsDevTables num_t;
    std::vector<int32_t> arc_of_h, tidx_h, a_first_h(B);
    const long long rows = backoff_numerators(gb, prods, ptabs, &num_t, &arc_of_h, &tidx_h);
    const long long tot_P = (long long)tidx_h.size();
    for (int b = 0; b < B; b++) a_first_h[b] = (int32_t)gb.first_arc[b];
    std::vector<float> w_A_h;
    float *w_dev = nullptr, *fw = nullptr, *w_A = nullptr;
    int32_t *T_dev = nullptr, *head = nullptr, *arc_of = nullptr, *tidx = nullptr, *a_first = nullptr;
    uint16_t* bp = nullptr;
    GTNB_TRY(scope.borrow(trans_w, trans_on_device != 0, std::max(n_trans, 1ll), &w_dev));
    GTNB_TRY(scope.alloc(&T_dev, B));
    GTNB_TRY(scope.alloc(&head, B));
    GTNB_TRY(scope.alloc(&a_first, B));
    GTNB_TRY(scope.alloc(&bp, std::max(rows, 1ll)));
    GTNB_TRY(scope.alloc(&fw, std::max(tot_P, 1ll)));
    GTNB_TRY(scope.alloc(&arc_of, std::max(tot_P, 1ll)));
    GTNB_TRY(scope.alloc(&tidx, std::max(tot_P, 1ll)));
    GTNB_TRY(num_t.alloc(scope));
    if (host_arc_weights(gb, &w_A_h)) GTNB_TRY(scope.alloc(&w_A, (long long)w_A_h.size()));
    GTNB_TRY(stage_begin(ctx));
    GTNB_TRY(num_t.stage(scope));
    GTNB_TRY(stage_upload(ctx, T_dev, gb.Tb.data(), sizeof(int32_t) * B));
    GTNB_TRY(stage_upload(ctx, a_first, a_first_h.data(), sizeof(int32_t) * B));
    if (tot_P) {
      GTNB_TRY(stage_upload(ctx, arc_of, arc_of_h.data(), sizeof(int32_t) * tot_P));
      GTNB_TRY(stage_upload(ctx, tidx, tidx_h.data(), sizeof(int32_t) * tot_P));
    }
    if (!trans_on_device && n_trans) GTNB_TRY(stage_upload(ctx, w_dev, trans_w, sizeof(float) * n_trans));
    if (w_A) GTNB_TRY(stage_upload(ctx, w_A, w_A_h.data(), sizeof(float) * w_A_h.size()));
    GTNB_TRY(stage_end(ctx));
    GTNB_TRY(launch_sparse_eps_gather(ctx, tot_P, gb.arc_weights_dev ? gb.arc_weights_dev : w_A, arc_of, w_dev, tidx,
                                      fw));
    GTNB_TRY(launch_sparse_eps_align(ctx, num_t.dev, num_t.max_S, B, T, C, T_dev, v.e_dev, (long long)T * C, fw, bp,
                                     head, v.s_dev, arc_of, a_first, v.p_dev, v.a_dev, v.status));
  }
  return viterbi_finish(scope, a, gb, implicit, v, [&](const std::vector<int>& which) {
    std::vector<float> W(std::max(n_trans, 1ll));
    if (n_trans) GTNB_TRY(read_to_host(ctx, W.data(), trans_w, trans_on_device, n_trans));
    return backoff_align_exact(scope, gb, Gv, W.data(), v, which);
  });
}

} // namespace

extern "C" int gtnb_backoff_transitions_loss(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const gtnb_graph_view* graphs, const float* arc_weights, int arc_weights_on_device,
    const gtnb_graph_view* transitions, const float* trans_w, int trans_on_device, float* losses_host, float* grads,
    int grads_on_device, float* arc_grads, int arc_grads_on_device, float* trans_grad, int trans_grad_on_device) {
  const std::string fn = "gtnb_backoff_transitions_loss";
  GraphBatch gb;
  SparseTables t;
  GTNB_TRY(parse_graphs(ctx, fn.c_str(), B, T, C, emissions, graphs,
                        transitions && (B == 0 || (losses_host && trans_w)), input_lens, arc_weights,
                        arc_weights_on_device, &gb, [&] { return check_backoff_graph(ctx, fn, *transitions, C, &t); }));
  const TransitionArgs a{B, T, C, emissions, emissions_on_device, input_lens, trans_w, trans_on_device, nullptr,
                         nullptr, -1, losses_host, grads, grads_on_device, trans_grad, trans_grad_on_device};
  if (t.E == 0) return sparse_transitions_loss_run(ctx, a, gb, *transitions, t, arc_grads, arc_grads_on_device);
  return backoff_loss_run(ctx, a, gb, *transitions, t, arc_grads, arc_grads_on_device);
}

extern "C" int gtnb_viterbi_backoff(gtnb_ctx* ctx, int B, int T, int C, const float* emissions,
                                    int emissions_on_device, const int32_t* input_lens,
                                    const gtnb_graph_view* transitions, const float* trans_w, int trans_on_device,
                                    int32_t* paths, int32_t* arcs, float* scores, int outputs_on_device) {
  const std::string fn = "gtnb_viterbi_backoff";
  if (!ctx || B < 0 || T < 0 || C <= 0 || !transitions || (B > 0 && (!emissions || !trans_w)))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  SparseTables t;
  GTNB_TRY(check_backoff_graph(ctx, fn, *transitions, C, &t));
  GraphBatch gb; // the batch without target graphs: its lengths
  gb.B = B, gb.T = T, gb.C = C;
  gb.Tb.resize(B);
  for (int b = 0; b < B; b++) {
    gb.Tb[b] = input_lens ? input_lens[b] : T;
    if (gb.Tb[b] < 0 || gb.Tb[b] > T) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": input_lens outside [0, T]");
  }
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  CallScope scope(ctx);
  const GraphViterbiArgs a{emissions, emissions_on_device, paths, arcs, scores, outputs_on_device};
  if (t.E == 0) return viterbi_sparse_run(scope, a, gb, *transitions, trans_w, trans_on_device);
  return backoff_viterbi_run(scope, a, gb, *transitions, t, trans_w, trans_on_device);
}

extern "C" int gtnb_backoff_transitions_viterbi(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const gtnb_graph_view* graphs, const float* arc_weights, int arc_weights_on_device,
    const gtnb_graph_view* transitions, const float* trans_w, int trans_on_device, int32_t* paths, int32_t* arcs,
    float* scores, int outputs_on_device) {
  const std::string fn = "gtnb_backoff_transitions_viterbi";
  GraphBatch gb;
  SparseTables t;
  GTNB_TRY(parse_graphs(ctx, fn.c_str(), B, T, C, emissions, graphs, transitions && (B == 0 || trans_w), input_lens,
                        arc_weights, arc_weights_on_device, &gb,
                        [&] { return check_backoff_graph(ctx, fn, *transitions, C, &t); }));
  if (B == 0) return GTNB_OK;
  if (t.E == 0)
    return gtnb_sparse_transitions_viterbi(ctx, B, T, C, emissions, emissions_on_device, input_lens, graphs,
                                           arc_weights, arc_weights_on_device, transitions, trans_w, trans_on_device,
                                           paths, arcs, scores, outputs_on_device);
  // the loss's numerators, whose shapes decide, with G's, whether the device route can be taken
  std::vector<ProductGraph> prods;
  std::vector<SparseTables> ptabs;
  SparseSplit split{}; // (the alignment sweeps the numerators alone: only whether G has a device route matters)
  const bool fast = ctx->use_implicit && backoff_route(ctx, t, C, &split) &&
                    backoff_products(gb, *transitions, t, C, &prods, &ptabs);
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  CallScope scope(ctx);
  return backoff_align_run(scope, GraphViterbiArgs{emissions, emissions_on_device, paths, arcs, scores,
                                                   outputs_on_device},
                           gb, *transitions, t, prods, ptabs, fast, trans_w, trans_on_device);
}

/*
 * Decoding without a host synchronisation, under gtnb_ctc_loss_async's contract.
 *   gtnb_viterbi_transitions_async: gtnb_viterbi_sparse / gtnb_viterbi_backoff on a G prepared once
 *     (gtnb_transitions): its tables, epsilon descriptor and cluster cuts live in device memory the handle owns, so a
 *     call uploads nothing.  The route is the synchronous decoders' device route: the prepare kernel, the tropical
 *     sweep and trace of k_sparse.cu (one CTA or a cluster per utterance, with or without epsilon arcs) and the
 *     finalize kernel, which maps the kernel status where the synchronous decoders read it back and re-run.
 *   gtnb_viterbi_dense_async: gtnb_viterbi_dense_typed with device lengths: the prepare kernel, k_dense.cu's decode
 *     and the finalize kernel (the dense kernel raises no status: only invalid lengths are flagged).
 * Back-pointers are sized from the bounds.
 */
struct gtnb_transitions {
  int device = 0, C = 0, S = 0;
  long long n_arcs = 0; // G's arcs: the length of trans_w
  bool eps = false; // G has epsilon arcs: the sparse_eps_* kernels over eps_dev (else the sparse_* kernels over dev)
  SparseSplit split{}; // sparse_route's / backoff_route's: N = 1 one CTA per utterance, else a cluster's plan
  void* mem = nullptr; // every device buffer below
  SparseDev dev{};
  SparseEpsDev* eps_dev = nullptr;
  int32_t* cut = nullptr; // sparse_eps_cluster_cuts (eps and split.N > 1), else NULL
  ~gtnb_transitions() {
    if (mem) cudaFree(mem);
  }
};


extern "C" int gtnb_transitions_create(gtnb_ctx* ctx, const gtnb_graph_view* Gv, int C, int backoff,
                                       gtnb_transitions** out) {
  const std::string fn = "gtnb_transitions_create";
  if (out) *out = nullptr;
  if (!ctx || !Gv || C <= 0 || !out || (backoff != 0 && backoff != 1))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  const std::string sync = backoff ? "gtnb_viterbi_backoff" : "gtnb_viterbi_sparse";
  SparseTables t;
  if (backoff) {
    GTNB_TRY(check_backoff_graph(ctx, fn, *Gv, C, &t));
  } else {
    GTNB_TRY(check_transition_graph(ctx, fn, *Gv));
    sparse_tables(*Gv, C, &t);
  }
  if (!ctx->use_implicit)
    return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": the \"implicit\" flag is off (materialised route): decode with " + sync);
  std::unique_ptr<gtnb_transitions> h(new gtnb_transitions);
  h->device = ctx->device;
  h->C = C;
  h->S = t.S;
  h->n_arcs = Gv->num_arcs;
  h->eps = t.E > 0;
  const bool fits = h->eps ? backoff_route(ctx, t, C, &h->split) : sparse_route(ctx, t, C, &h->split);
  if (!fits)
    return fail(ctx, GTNB_ERR_UNSUPPORTED,
                fn + ": the transition graph is outside the device decoders' envelope: decode with " + sync);
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  // one allocation, 256-byte granules: the packed tables, then (epsilon arcs) the descriptor and the cuts
  std::vector<const void*> src;
  std::vector<size_t> bytes;
  std::vector<void*> dst;
  SparseDevTables st;
  EpsDevTables et;
  std::vector<int32_t> cut_h;
  if (h->eps) {
    et.add(t, 0, 0);
    if (h->split.N > 1) sparse_eps_cluster_cuts(t, h->split, &cut_h);
    bytes = {sizeof(int32_t) * et.packed.size(), sizeof(SparseEpsDev), sizeof(int32_t) * cut_h.size()};
  } else {
    st.pack(t);
    bytes = {sizeof(int32_t) * st.packed.size()};
  }
  size_t total = 0;
  for (size_t n : bytes) total += (n + 255) & ~(size_t)255;
  GTNB_CUDA(ctx, cudaMalloc(&h->mem, total));
  for (size_t i = 0, at = 0; i < bytes.size(); at += (bytes[i] + 255) & ~(size_t)255, i++)
    dst.push_back(static_cast<unsigned char*>(h->mem) + at);
  if (h->eps) {
    et.place(static_cast<int32_t*>(dst[0]), static_cast<SparseEpsDev*>(dst[1]));
    src = {et.packed.data(), et.desc.data(), cut_h.data()};
    h->eps_dev = et.dev;
    if (!cut_h.empty()) h->cut = static_cast<int32_t*>(dst[2]);
  } else {
    st.place(static_cast<int32_t*>(dst[0]));
    src = {st.packed.data()};
    h->dev = st.dev;
  }
  for (size_t i = 0; i < bytes.size(); i++)
    if (bytes[i]) GTNB_CUDA(ctx, cudaMemcpy(dst[i], src[i], bytes[i], cudaMemcpyHostToDevice));
  GTNB_CUDA(ctx, cudaDeviceSynchronize()); // (set-up: the tables are on the device before any stream reads them)
  *out = h.release();
  return GTNB_OK;
}

extern "C" void gtnb_transitions_destroy(gtnb_ctx* ctx, gtnb_transitions* G) {
  if (!G) return;
  if (ctx) cudaSetDevice(G->device);
  delete G; // (cudaFree waits for the device: no launch still reads the tables)
}

namespace {

struct DecodeAsyncArgs {
  int B, T;
  const void* emissions;
  int dtype; // (dense only)
  const int32_t* input_lens;
  const float* trans_w;
  int32_t *paths, *arcs;
  float* scores;
  int32_t* status;
};

/* gtnb_viterbi_transitions_async's run */
int transitions_async_run(gtnb_ctx* ctx, const gtnb_transitions* G, const DecodeAsyncArgs& a, bool launch) {
  const int B = a.B, T = a.T, C = G->C, S = G->S;
  int32_t *lens = nullptr, *valid = nullptr, *kstatus = nullptr, *head = nullptr;
  uint16_t* bp = nullptr;
  GTNB_TRY(dev_alloc(ctx, &lens, B));
  GTNB_TRY(dev_alloc(ctx, &valid, B));
  GTNB_TRY(dev_alloc(ctx, &kstatus, B));
  GTNB_TRY(dev_alloc(ctx, &head, B));
  // (the synchronous decoders' sizes at T_b = T)
  GTNB_TRY(dev_alloc(ctx, &bp, G->eps ? (long long)B * (T + 1) * S : std::max((long long)B * T * S, 1ll)));
  if (!launch) return GTNB_OK;
  const float* e = static_cast<const float*>(a.emissions);
  GTNB_TRY(launch_decode_async_prepare(ctx, B, T, a.input_lens, lens, valid, kstatus));
  if (G->eps)
    GTNB_TRY(launch_sparse_eps_viterbi(ctx, G->eps_dev, G->split, G->cut, S, B, T, C, lens, e, (long long)T * C,
                                       a.trans_w, bp, head, a.scores, a.paths, a.arcs, kstatus));
  else
    GTNB_TRY(launch_sparse_viterbi(ctx, G->dev, G->split, B, T, C, lens, e, (long long)T * C, a.trans_w, bp, head,
                                   a.scores, a.paths, a.arcs, kstatus));
  return launch_decode_async_finalize(ctx, B, T, lens, kstatus, valid, a.paths, a.arcs, a.scores, a.status);
}

/* gtnb_viterbi_dense_async's run; sizing takes the paths row whether or not paths will be given */
int dense_async_run(gtnb_ctx* ctx, int C, bool bigram, const DecodeAsyncArgs& a, bool launch) {
  const int B = a.B, T = a.T;
  if (!viterbi_dense_supported(C))
    return fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_viterbi_dense_async: the transitions tile does not fit shared memory "
                                           "(C <= 224)");
  int32_t *lens = nullptr, *valid = nullptr, *kstatus = nullptr, *paths = a.paths;
  uint8_t* bp = nullptr;
  GTNB_TRY(dev_alloc(ctx, &lens, B));
  GTNB_TRY(dev_alloc(ctx, &valid, B));
  GTNB_TRY(dev_alloc(ctx, &kstatus, B));
  GTNB_TRY(dev_alloc(ctx, &bp, (long long)B * std::max(T, 1) * dense_bp_pitch(C)));
  if (!paths || !launch) GTNB_TRY(dev_alloc(ctx, &paths, (long long)B * std::max(T, 1)));
  if (!launch) return GTNB_OK;
  GTNB_TRY(launch_decode_async_prepare(ctx, B, T, a.input_lens, lens, valid, kstatus));
  GTNB_TRY(launch_viterbi_dense(ctx, B, T, C, bigram, lens, a.emissions, (long long)T * C, a.trans_w,
                                -std::numeric_limits<float>::infinity(), bp, paths, a.scores, a.dtype));
  return launch_decode_async_finalize(ctx, B, T, lens, kstatus, valid, a.paths, nullptr, a.scores, a.status);
}

} // namespace

extern "C" int gtnb_viterbi_transitions_async_workspace(gtnb_ctx* ctx, const gtnb_transitions* G, int B, int T,
                                                        size_t* bytes) {
  const char* fn = "gtnb_viterbi_transitions_async_workspace";
  if (!ctx || !G || B < 0 || T < 0 || !bytes) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, std::string(fn) + ": bad arguments");
  if (G->device != ctx->device)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, std::string(fn) + ": the transition graph was made on another device");
  const DecodeAsyncArgs a{B, T, nullptr, GTNB_F32, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  return async_workspace(ctx, B, bytes, [&](bool launch) { return transitions_async_run(ctx, G, a, launch); });
}

extern "C" int gtnb_viterbi_transitions_async(
    gtnb_ctx* ctx, void* cuda_stream, const gtnb_transitions* G, int B, int T, const float* emissions_dev,
    const int32_t* input_lens_dev, const float* trans_w_dev, int32_t* paths_dev, int32_t* arcs_dev, float* scores_dev,
    int32_t* status_dev, void* workspace_dev, size_t workspace_bytes) {
  const std::string fn = "gtnb_viterbi_transitions_async";
  if (!ctx || !G || B < 0 || T < 0 || (B > 0 && (!emissions_dev || !trans_w_dev || !paths_dev || !scores_dev)))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  if (G->device != ctx->device)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the transition graph was made on another device");
  const DecodeAsyncArgs a{B, T, emissions_dev, GTNB_F32, input_lens_dev, trans_w_dev, paths_dev, arcs_dev, scores_dev,
                          status_dev};
  return async_enqueue(ctx, fn, B, cuda_stream, workspace_dev, workspace_bytes,
                       [&](bool launch) { return transitions_async_run(ctx, G, a, launch); });
}

extern "C" int gtnb_viterbi_dense_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int dtype, int kind,
                                                  size_t* bytes) {
  const std::string fn = "gtnb_viterbi_dense_async_workspace";
  if (!ctx || B < 0 || T < 0 || C <= 0 || !bytes || (kind != GTNB_DENSE_ASG && kind != GTNB_DENSE_BIGRAM))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  if (!known_dtype(dtype)) return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": unknown dtype");
  const DecodeAsyncArgs a{B, T, nullptr, dtype, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  return async_workspace(ctx, B, bytes,
                         [&](bool launch) { return dense_async_run(ctx, C, kind == GTNB_DENSE_BIGRAM, a, launch); });
}

extern "C" int gtnb_viterbi_dense_async(
    gtnb_ctx* ctx, void* cuda_stream, int B, int T, int C, const void* emissions_dev, int dtype,
    const int32_t* input_lens_dev, int kind, const float* trans_w_dev, int32_t* paths_dev, float* scores_dev,
    int32_t* status_dev, void* workspace_dev, size_t workspace_bytes) {
  const std::string fn = "gtnb_viterbi_dense_async";
  if (!ctx || B < 0 || T < 0 || C <= 0 || (kind != GTNB_DENSE_ASG && kind != GTNB_DENSE_BIGRAM) ||
      (B > 0 && (!emissions_dev || !trans_w_dev || !scores_dev)))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  if (!known_dtype(dtype)) return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": unknown dtype");
  const DecodeAsyncArgs a{B, T, emissions_dev, dtype, input_lens_dev, trans_w_dev, paths_dev, nullptr, scores_dev,
                          status_dev};
  return async_enqueue(ctx, fn, B, cuda_stream, workspace_dev, workspace_bytes,
                       [&](bool launch) { return dense_async_run(ctx, C, kind == GTNB_DENSE_BIGRAM, a, launch); });
}

namespace {

/* gtnb_edit_distance_async's run: the move words of the alignment (when asked for) taken from the arena and, when
 * launch, the one kernel enqueued */
int edit_async_run(gtnb_ctx* ctx, int B, const int32_t* hyp, int N, const int32_t* hyp_lens, const int32_t* ref,
                   int M, const int32_t* ref_lens, int word_sep, int32_t* distance, int32_t* ops, int32_t* units,
                   int32_t* status, int32_t* hyp_align, int32_t* ref_align, bool with_alignment, bool launch) {
  uint32_t* moves = nullptr;
  if (with_alignment) GTNB_TRY(dev_alloc(ctx, &moves, edit_distance_move_words(B, N, M, word_sep)));
  if (!launch) return GTNB_OK;
  return launch_edit_distance(ctx, B, hyp, N, hyp_lens, ref, M, ref_lens, word_sep, distance, ops, units, status,
                              hyp_align, ref_align, moves);
}

/* k_edit.cu holds at most 4096 rows (8 warps of 32 lanes of 16 rows) and both sequences in shared memory */
int edit_async_bounds(gtnb_ctx* ctx, const std::string& fn, int N, int M) {
  if (N > 4096 || M > 4096)
    return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": N and M are limited to 4096 units on the device");
  return GTNB_OK;
}

} // namespace

extern "C" int gtnb_edit_distance_async_workspace(gtnb_ctx* ctx, int B, int N, int M, int word_sep,
                                                  int with_alignment, size_t* bytes) {
  const std::string fn = "gtnb_edit_distance_async_workspace";
  if (!ctx || B < 0 || N < 0 || M < 0 || !bytes) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  GTNB_TRY(edit_async_bounds(ctx, fn, N, M));
  return async_workspace(ctx, B, bytes, [&](bool launch) {
    return edit_async_run(ctx, B, nullptr, N, nullptr, nullptr, M, nullptr, word_sep, nullptr, nullptr, nullptr,
                          nullptr, nullptr, nullptr, with_alignment != 0, launch);
  });
}

extern "C" int gtnb_edit_distance_async(
    gtnb_ctx* ctx, void* cuda_stream, int B, const int32_t* hyp_dev, int N, const int32_t* hyp_lengths_dev,
    const int32_t* ref_dev, int M, const int32_t* ref_lengths_dev, int word_sep, int32_t* distance_dev,
    int32_t* ops_dev, int32_t* units_dev, int32_t* status_dev, int32_t* hyp_align_dev, int32_t* ref_align_dev,
    void* workspace_dev, size_t workspace_bytes) {
  const std::string fn = "gtnb_edit_distance_async";
  if (!ctx || B < 0 || N < 0 || M < 0 ||
      (B > 0 && (!hyp_lengths_dev || !ref_lengths_dev || (N > 0 && !hyp_dev) || (M > 0 && !ref_dev) ||
                 !distance_dev || !ops_dev || !units_dev || !status_dev)))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  GTNB_TRY(edit_async_bounds(ctx, fn, N, M));
  return async_enqueue(ctx, fn, B, cuda_stream, workspace_dev, workspace_bytes, [&](bool launch) {
    return edit_async_run(ctx, B, hyp_dev, N, hyp_lengths_dev, ref_dev, M, ref_lengths_dev, word_sep, distance_dev,
                          ops_dev, units_dev, status_dev, hyp_align_dev, ref_align_dev,
                          hyp_align_dev || ref_align_dev, launch);
  });
}

/*
 * The LM of gtnb_beam_decode_lm_async, prepared once: the graph's resolved table, weight [S][C + 1] float32 and
 * destination [S][C + 1] int32 in one device allocation.  Column C holds the end weights.
 */
struct gtnb_lm {
  int device = 0, C = 0, S = 0, start = 0;
  void* mem = nullptr;
  float* w = nullptr;
  int32_t* d = nullptr;
  ~gtnb_lm() {
    if (mem) cudaFree(mem);
  }
};

namespace {

struct BeamAsyncArgs {
  int B, T, C, dtype;
  const void* emissions;
  const int32_t* input_lens;
  int kind;
  const float* trans_w;
  int blank, beam, nbest;
  int32_t *tokens, *lengths;
  float* scores;
  int32_t* status;
};

/* the bounds k_beam.cu covers, and the kind-specific arguments */
int beam_async_check(gtnb_ctx* ctx, const std::string& fn, const BeamAsyncArgs& a) {
  if (a.kind != GTNB_DENSE_CTC && a.kind != GTNB_DENSE_BIGRAM && a.kind != GTNB_DENSE_ASG)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": unknown kind");
  if (!known_dtype(a.dtype)) return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": unknown dtype");
  if (!beam_decode_supported(a.C, a.beam, a.nbest))
    return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": needs 1 <= beam <= 64, 1 <= nbest <= beam and C <= 256");
  if (a.kind != GTNB_DENSE_ASG && (a.blank < 0 || a.blank >= a.C))
    return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": blank outside [0, C)");
  return GTNB_OK;
}

/* gtnb_beam_decode_async's run: the back-pointers and (with transitions) the transposed weights, the start weights
 * and the row flags taken from the arena and, when launch, the weights kernel and the search under policy f enqueued
 * (the same scratch for every policy) */
template <class F>
int beam_async_run(gtnb_ctx* ctx, const BeamAsyncArgs& a, bool launch, const F& f) {
  uint16_t* bp = nullptr;
  float *wt = nullptr, *wfirst = nullptr;
  int32_t* wbad = nullptr;
  GTNB_TRY(dev_alloc(ctx, &bp, (long long)a.B * std::max(a.T, 1) * a.beam));
  if (a.kind != GTNB_DENSE_CTC) {
    GTNB_TRY(dev_alloc(ctx, &wt, (long long)a.C * a.C));
    GTNB_TRY(dev_alloc(ctx, &wfirst, a.C));
    GTNB_TRY(dev_alloc(ctx, &wbad, a.C));
  }
  if (!launch) return GTNB_OK;
  if (a.kind != GTNB_DENSE_CTC) GTNB_TRY(launch_beam_weights(ctx, a.C, a.kind, a.trans_w, wt, wfirst, wbad));
  return launch_beam_decode(ctx, a.B, a.T, a.C, a.emissions, a.dtype, a.input_lens, a.kind, wt,
                            a.kind == GTNB_DENSE_ASG ? a.trans_w : wfirst, wbad, a.blank, a.beam, a.nbest, bp,
                            a.tokens, a.lengths, a.scores, a.status, f);
}

} // namespace

extern "C" int gtnb_beam_decode_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int dtype, int kind, int beam,
                                                int nbest, size_t* bytes) {
  const std::string fn = "gtnb_beam_decode_async_workspace";
  if (!ctx || B < 0 || T < 0 || C <= 0 || !bytes) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  const BeamAsyncArgs a{B, T, C, dtype, nullptr, nullptr, kind, nullptr, 0, beam, nbest,
                        nullptr, nullptr, nullptr, nullptr};
  GTNB_TRY(beam_async_check(ctx, fn, a));
  return async_workspace(ctx, B, bytes, [&](bool launch) { return beam_async_run(ctx, a, launch, BeamNoLm()); });
}

extern "C" int gtnb_beam_decode_async(
    gtnb_ctx* ctx, void* cuda_stream, int B, int T, int C, const void* emissions_dev, int dtype,
    const int32_t* input_lens_dev, int kind, const float* trans_w_dev, int blank, int beam, int nbest,
    int32_t* tokens_dev, int32_t* lengths_dev, float* scores_dev, int32_t* status_dev, void* workspace_dev,
    size_t workspace_bytes) {
  const std::string fn = "gtnb_beam_decode_async";
  if (!ctx || B < 0 || T < 0 || C <= 0 ||
      (B > 0 && ((T > 0 && !emissions_dev) || !tokens_dev || !lengths_dev || !scores_dev)) ||
      (kind == GTNB_DENSE_CTC) != (trans_w_dev == nullptr))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  const BeamAsyncArgs a{B, T, C, dtype, emissions_dev, input_lens_dev, kind, trans_w_dev, blank, beam, nbest,
                        tokens_dev, lengths_dev, scores_dev, status_dev};
  GTNB_TRY(beam_async_check(ctx, fn, a));
  return async_enqueue(ctx, fn, B, cuda_stream, workspace_dev, workspace_bytes,
                       [&](bool launch) { return beam_async_run(ctx, a, launch, BeamNoLm()); });
}

namespace {

constexpr long long kLmMaxEntries = 1ll << 25;

/*
 * The graph checks of a backoff LM over the labels [0, L] (gtnb_lm_create: L = C; gtnb_lexicon_create's word LM:
 * L = V), label L being end of sentence: one start node, an acceptor, no NaN or +inf weight, labels in [0, L] or
 * epsilon, at most one arc per (node, label) and one epsilon arc per node, no cycle of epsilon arcs.  A graph of more
 * than max_nodes nodes is GTNB_ERR_UNSUPPORTED (too_big).  Out: the start node, each node's epsilon (backoff) arc or -1
 * and backoff depth (the number of epsilon arcs to a node without one), the emitting arcs sorted by (source, label),
 * and whether any arc is labelled L.
 */
struct LmGraph {
  int start = -1;
  std::vector<int32_t> eps, arcs;
  std::vector<int> depth;
  bool has_end = false;
};

int lm_check(gtnb_ctx* ctx, const std::string& fn, const gtnb_graph_view& G, int L, long long max_nodes,
             const char* too_big, LmGraph* g) {
  if (validate_view(ctx, G)) return GTNB_ERR_INVALID_ARGUMENT;
  const int S = G.num_nodes;
  if (S < 1) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the LM has no nodes");
  if (S > max_nodes) return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + too_big);
  g->start = -1;
  for (int s = 0; s < S; s++)
    if (G.node_flags[s] & 1) {
      if (g->start >= 0) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the LM has more than one start node");
      g->start = s;
    }
  if (g->start < 0) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the LM has no start node");
  g->eps.assign(S, -1);
  g->arcs.clear();
  g->has_end = false;
  for (int a = 0; a < G.num_arcs; a++) {
    const int s = G.arc_src[a], l = G.arc_ilabel[a];
    const float x = G.weights ? G.weights[a] : 0.0f;
    if (l != G.arc_olabel[a]) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the LM is not an acceptor");
    if (x != x || x == std::numeric_limits<float>::infinity())
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the LM has a NaN or +inf weight");
    if (l == GTNB_EPSILON) {
      if (g->eps[s] >= 0) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": a node has two epsilon arcs");
      g->eps[s] = a;
      continue;
    }
    if (l < 0 || l > L)
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": an LM label outside [0, " + std::to_string(L) + "]");
    g->arcs.push_back(a);
    g->has_end |= l == L;
  }
  std::stable_sort(g->arcs.begin(), g->arcs.end(), [&](int32_t a, int32_t b) {
    return G.arc_src[a] != G.arc_src[b] ? G.arc_src[a] < G.arc_src[b] : G.arc_ilabel[a] < G.arc_ilabel[b];
  });
  for (size_t i = 1; i < g->arcs.size(); i++) {
    const int a = g->arcs[i - 1], b = g->arcs[i];
    if (G.arc_src[a] == G.arc_src[b] && G.arc_ilabel[a] == G.arc_ilabel[b])
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": a node has two arcs with one label");
  }
  // backoff depth (more than S epsilon arcs in a row means a cycle)
  std::vector<int>& depth = g->depth;
  const std::vector<int32_t>& eps = g->eps;
  depth.assign(S, -1);
  for (int s = 0; s < S; s++) {
    int v = s, k = 0;
    while (depth[v] < 0 && eps[v] >= 0 && k <= S) {
      v = G.arc_dst[eps[v]];
      k++;
    }
    if (k > S) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the LM has a cycle of epsilon arcs");
    int base = depth[v] < 0 ? 0 : depth[v];
    for (int u = s; u != v; u = G.arc_dst[eps[u]]) depth[u] = base + k--;
    if (depth[v] < 0) depth[v] = 0;
  }
  return GTNB_OK;
}

/* the nodes of a checked LM in order of backoff depth: a backoff destination comes before the nodes that back off
 * to it */
std::vector<int> lm_depth_order(const LmGraph& g) {
  std::vector<int> order(g.depth.size());
  for (size_t s = 0; s < order.size(); s++) order[s] = (int)s;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return g.depth[a] < g.depth[b]; });
  return order;
}

/*
 * gtnb_lm_create's resolution: w(s, c) is s's arc labelled c, else s's epsilon (backoff) arc's weight plus the
 * resolution of c from its destination, else -inf.  Nodes are resolved in order of backoff depth, so a backoff
 * destination's row is complete before the rows that back off to it.  Without any arc labelled C, every end weight
 * (column C) is 0.
 */
int lm_resolve(gtnb_ctx* ctx, const std::string& fn, const gtnb_graph_view& G, int C, int* start,
               std::vector<float>* w, std::vector<int32_t>* d) {
  LmGraph g;
  GTNB_TRY(lm_check(ctx, fn, G, C, kLmMaxEntries / (C + 1), ": S * (C + 1) > 2^25 table entries", &g));
  *start = g.start;
  const int S = G.num_nodes;
  const long long n = (long long)S * (C + 1);
  const float ninf = -std::numeric_limits<float>::infinity();
  std::vector<int32_t> arc(n, -1);
  for (int a : g.arcs) arc[(long long)G.arc_src[a] * (C + 1) + G.arc_ilabel[a]] = a;
  w->assign(n, ninf);
  d->assign(n, 0);
  for (int s : lm_depth_order(g)) {
    const long long row = (long long)s * (C + 1);
    const int e = g.eps[s];
    const long long brow = e >= 0 ? (long long)G.arc_dst[e] * (C + 1) : -1;
    const float be = e >= 0 ? (G.weights ? G.weights[e] : 0.0f) : 0.0f;
    for (int c = 0; c <= C; c++) {
      const int a = arc[row + c];
      if (a >= 0) {
        (*w)[row + c] = G.weights ? G.weights[a] : 0.0f;
        (*d)[row + c] = G.arc_dst[a];
      } else if (e >= 0) {
        (*w)[row + c] = be + (*w)[brow + c];
        (*d)[row + c] = (*d)[brow + c];
      }
    }
    if (!g.has_end) (*w)[row + C] = 0.0f;
  }
  return GTNB_OK;
}

} // namespace

extern "C" int gtnb_lm_create(gtnb_ctx* ctx, const gtnb_graph_view* lm, int C, gtnb_lm** out) {
  const std::string fn = "gtnb_lm_create";
  if (out) *out = nullptr;
  if (!ctx || !lm || C <= 0 || !out) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  if (C > 256) return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": C > 256");
  std::unique_ptr<gtnb_lm> h(new gtnb_lm);
  std::vector<float> w;
  std::vector<int32_t> d;
  GTNB_TRY(lm_resolve(ctx, fn, *lm, C, &h->start, &w, &d));
  h->device = ctx->device;
  h->C = C;
  h->S = lm->num_nodes;
  const size_t wb = (sizeof(float) * w.size() + 255) & ~(size_t)255;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  GTNB_CUDA(ctx, cudaMalloc(&h->mem, wb + sizeof(int32_t) * d.size()));
  h->w = static_cast<float*>(h->mem);
  h->d = reinterpret_cast<int32_t*>(static_cast<unsigned char*>(h->mem) + wb);
  GTNB_CUDA(ctx, cudaMemcpy(h->w, w.data(), sizeof(float) * w.size(), cudaMemcpyHostToDevice));
  GTNB_CUDA(ctx, cudaMemcpy(h->d, d.data(), sizeof(int32_t) * d.size(), cudaMemcpyHostToDevice));
  GTNB_CUDA(ctx, cudaDeviceSynchronize()); // (set-up: the table is on the device before any stream reads it)
  *out = h.release();
  return GTNB_OK;
}

extern "C" void gtnb_lm_destroy(gtnb_ctx* ctx, gtnb_lm* lm) {
  if (!lm) return;
  if (ctx) cudaSetDevice(lm->device);
  delete lm; // (cudaFree waits for the device: no launch still reads the table)
}

namespace {

int beam_lm_check(gtnb_ctx* ctx, const std::string& fn, const BeamAsyncArgs& a, int token_beam) {
  GTNB_TRY(beam_async_check(ctx, fn, a));
  if (token_beam < 1 || token_beam > a.C) return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": token_beam outside [1, C]");
  return GTNB_OK;
}

} // namespace

extern "C" int gtnb_beam_decode_lm_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int dtype, int kind, int beam,
                                                   int nbest, int token_beam, size_t* bytes) {
  const std::string fn = "gtnb_beam_decode_lm_async_workspace";
  if (!ctx || B < 0 || T < 0 || C <= 0 || !bytes) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  const BeamAsyncArgs a{B, T, C, dtype, nullptr, nullptr, kind, nullptr, 0, beam, nbest,
                        nullptr, nullptr, nullptr, nullptr};
  GTNB_TRY(beam_lm_check(ctx, fn, a, token_beam));
  const BeamLm f{token_beam, nullptr, nullptr, 0, 0.0f, 0.0f, nullptr, nullptr};
  return async_workspace(ctx, B, bytes, [&](bool launch) { return beam_async_run(ctx, a, launch, f); });
}

extern "C" int gtnb_beam_decode_lm_async(
    gtnb_ctx* ctx, void* cuda_stream, int B, int T, int C, const void* emissions_dev, int dtype,
    const int32_t* input_lens_dev, int kind, const float* trans_w_dev, int blank, int beam, int nbest,
    const gtnb_lm* lm, float lm_weight, float token_bonus, int token_beam, int32_t* tokens_dev, int32_t* lengths_dev,
    float* scores_dev, float* am_scores_dev, float* lm_scores_dev, int32_t* status_dev, void* workspace_dev,
    size_t workspace_bytes) {
  const std::string fn = "gtnb_beam_decode_lm_async";
  if (!ctx || B < 0 || T < 0 || C <= 0 ||
      (B > 0 && ((T > 0 && !emissions_dev) || !tokens_dev || !lengths_dev || !scores_dev)) ||
      (kind == GTNB_DENSE_CTC) != (trans_w_dev == nullptr))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  if (!(lm_weight >= 0.0f && std::isfinite(lm_weight)) || !std::isfinite(token_bonus))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": lm_weight must be finite and >= 0, token_bonus finite");
  if (lm && lm->device != ctx->device)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the LM was made on another device");
  if (lm && lm->C != C) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the LM was made for another C");
  const BeamAsyncArgs a{B, T, C, dtype, emissions_dev, input_lens_dev, kind, trans_w_dev, blank, beam, nbest,
                        tokens_dev, lengths_dev, scores_dev, status_dev};
  GTNB_TRY(beam_lm_check(ctx, fn, a, token_beam));
  const BeamLm f{token_beam, lm ? lm->w : nullptr, lm ? lm->d : nullptr, lm ? lm->start : 0,
                 lm_weight, token_bonus, am_scores_dev, lm_scores_dev};
  return async_enqueue(ctx, fn, B, cuda_stream, workspace_dev, workspace_bytes,
                       [&](bool launch) { return beam_async_run(ctx, a, launch, f); });
}

/*
 * The lexicon of gtnb_beam_decode_lexicon_async, prepared once, in one device allocation:
 *   the token classes [C]; the trie, numbered breadth first so that each node's children are consecutive in token
 *   order (the root is 0, its children 1, 2, ...): child masks [nodes][MW], first child, word id and smear [nodes];
 *   the word LM: an open-addressing hash of its emitting arcs [H][2] (key node << 32 | word, all ones in an empty
 *   slot; value destination << 32 | weight bits; H a power of two >= 2 * arcs, linear probing from the key times
 *   hmul's top hbits bits), and each node's backoff weight, backoff destination and resolved end weight [S].
 */
struct gtnb_lexicon {
  int device = 0, C = 0, V = 0, nodes = 0, S = 0, start = 0, hbits = 0, max_depth = 0;
  unsigned long long hmul = 0;
  std::vector<int32_t> cls;
  std::vector<uint8_t> spelled; // [C] the token appears in a spelling
  void* mem = nullptr;
  int32_t *d_cls = nullptr, *d_first = nullptr, *d_word = nullptr, *d_bod = nullptr;
  unsigned long long* d_hash = nullptr;
  uint32_t* d_mask = nullptr;
  float *d_smear = nullptr, *d_bow = nullptr, *d_endw = nullptr;
  ~gtnb_lexicon() {
    if (mem) cudaFree(mem);
  }
};

namespace {

constexpr int kLexMaxV = 1 << 20;
constexpr int kLexMaxNodes = 1 << 24;
constexpr long long kLexMaxLmArcs = 1ll << 26;
constexpr unsigned long long kLexHashMul = 0x9e3779b97f4a7c15ull;

/* the word LM's emitting arcs in the order lm_check sorted them, with a row start per node */
struct WordLm {
  const gtnb_graph_view* G = nullptr;
  LmGraph g;
  std::vector<long long> row; // [S + 1] into g.arcs
  float weight(int a) const { return G->weights ? G->weights[a] : 0.0f; }
  /* the arc of s labelled x, or -1 */
  int arc(int s, int x) const {
    long long lo = row[s], hi = row[s + 1];
    while (lo < hi) {
      const long long mid = (lo + hi) / 2;
      const int l = G->arc_ilabel[g.arcs[mid]];
      if (l == x) return g.arcs[mid];
      if (l < x)
        lo = mid + 1;
      else
        hi = mid;
    }
    return -1;
  }
  /* w(s, x) in float32, backoff weights added innermost first (gtnb_lm_create's order) */
  float resolve(int s, int x) const {
    std::vector<int> chain;
    int v = s, a;
    while ((a = arc(v, x)) < 0) {
      const int e = g.eps[v];
      if (e < 0) return -std::numeric_limits<float>::infinity();
      chain.push_back(e);
      v = G->arc_dst[e];
    }
    float w = weight(a);
    for (size_t i = chain.size(); i-- > 0;) w = weight(chain[i]) + w;
    return w;
  }
};

} // namespace

extern "C" int gtnb_lexicon_create(gtnb_ctx* ctx, int C, const int32_t* token_class, int V, int num_spellings,
                                   const int32_t* spelling_offsets, const int32_t* spelling_tokens,
                                   const int32_t* spelling_words, const gtnb_graph_view* word_lm,
                                   gtnb_lexicon** out) {
  const std::string fn = "gtnb_lexicon_create";
  if (out) *out = nullptr;
  if (!ctx || C <= 0 || V <= 0 || num_spellings < 0 || !token_class || !out ||
      (num_spellings > 0 && (!spelling_offsets || !spelling_tokens || !spelling_words)))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  if (C > 256) return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": C > 256");
  if (V > kLexMaxV) return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": V > 2^20 words");
  std::unique_ptr<gtnb_lexicon> h(new gtnb_lexicon);
  h->C = C;
  h->V = V;
  h->cls.assign(token_class, token_class + C);
  h->spelled.assign(C, 0);
  for (int c = 0; c < C; c++)
    if (token_class[c] < 0 || token_class[c] > 2)
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": a token class outside {0, 1, 2}");
  // the trie, first with children in insertion order
  std::vector<std::vector<std::pair<int, int>>> kids(1);
  std::vector<int32_t> wid(1, -1);
  if (num_spellings > 0 && spelling_offsets[0] != 0)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": spelling_offsets[0] != 0");
  for (int i = 0; i < num_spellings; i++) {
    const int o0 = spelling_offsets[i], o1 = spelling_offsets[i + 1], w = spelling_words[i];
    if (o1 <= o0) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": an empty spelling");
    if (w < 0 || w >= V) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": a word id outside [0, V)");
    int n = 0;
    for (int p = o0; p < o1; p++) {
      const int c = spelling_tokens[p];
      if (c < 0 || c >= C) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": a spelling token outside [0, C)");
      if (token_class[c] == 1) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": a separator in a spelling");
      if (token_class[c] == 2 && p > o0)
        return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": a word-start token after a spelling's first position");
      h->spelled[c] = 1;
      int next = -1;
      for (const auto& k : kids[n])
        if (k.first == c) next = k.second;
      if (next < 0) {
        if ((int)kids.size() >= kLexMaxNodes)
          return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": the trie has more than 2^24 nodes");
        next = (int)kids.size();
        kids[n].push_back({c, next});
        kids.emplace_back();
        wid.push_back(-1);
      }
      n = next;
    }
    if (wid[n] >= 0 && wid[n] != w)
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": two words share a spelling");
    wid[n] = w;
  }
  // the word LM
  WordLm lm;
  if (word_lm) {
    if ((long long)word_lm->num_arcs > kLexMaxLmArcs)
      return fail(ctx, GTNB_ERR_UNSUPPORTED, fn + ": the word LM has more than 2^26 arcs");
    lm.G = word_lm;
    GTNB_TRY(lm_check(ctx, fn, *word_lm, V, kLexMaxLmArcs, ": the word LM has more than 2^26 nodes", &lm.g));
    const int S = word_lm->num_nodes;
    lm.row.assign(S + 1, 0);
    for (int a : lm.g.arcs) lm.row[word_lm->arc_src[a] + 1]++;
    for (int s = 0; s < S; s++) lm.row[s + 1] += lm.row[s];
    h->S = S;
    h->start = lm.g.start;
    for (int d : lm.g.depth) h->max_depth = std::max(h->max_depth, d);
  }
  // breadth-first numbering, each node's children in token order
  const int nodes = (int)kids.size(), MW = (C + 31) / 32;
  std::vector<int> bfs(1, 0), id(nodes, 0);
  for (size_t q = 0; q < bfs.size(); q++) {
    auto& k = kids[bfs[q]];
    std::sort(k.begin(), k.end());
    for (const auto& x : k) {
      id[x.second] = (int)bfs.size();
      bfs.push_back(x.second);
    }
  }
  std::vector<uint32_t> mask((size_t)nodes * MW, 0u);
  std::vector<int32_t> first(nodes, 0), word(nodes, -1);
  std::vector<float> smear(nodes, -std::numeric_limits<float>::infinity());
  for (int q = 0; q < nodes; q++) {
    const int n = bfs[q];
    word[q] = wid[n];
    first[q] = kids[n].empty() ? 0 : id[kids[n][0].second];
    for (const auto& x : kids[n]) mask[(size_t)q * MW + (x.first >> 5)] |= 1u << (x.first & 31);
  }
  // smear: the largest finite w(start, word) at or below each node (0 when none is, at the root, without an LM)
  if (word_lm) {
    for (int q = nodes - 1; q > 0; q--) {
      float best = word[q] >= 0 ? lm.resolve(lm.g.start, word[q]) : -std::numeric_limits<float>::infinity();
      const int n = bfs[q];
      for (size_t i = 0; i < kids[n].size(); i++) best = std::max(best, smear[first[q] + i]);
      smear[q] = best;
    }
  }
  for (int q = 0; q < nodes; q++)
    if (q == 0 || !(smear[q] > -std::numeric_limits<float>::infinity())) smear[q] = 0.0f;
  // the word LM's arc hash, backoff arrays and end weights
  std::vector<unsigned long long> hash;
  std::vector<int32_t> bod;
  std::vector<float> bow, endw;
  if (word_lm) {
    const int S = h->S;
    long long n_emit = 0;
    for (int a : lm.g.arcs) n_emit += word_lm->arc_ilabel[a] < V;
    int hb = 1;
    while ((1ll << hb) < 2 * n_emit) hb++;
    h->hbits = hb;
    h->hmul = kLexHashMul;
    const long long H = 1ll << hb;
    hash.assign(2 * H, 0ull);
    for (long long i = 0; i < H; i++) hash[2 * i] = ~0ull;
    for (int a : lm.g.arcs) {
      const int x = word_lm->arc_ilabel[a];
      if (x >= V) continue;
      const unsigned long long key = ((unsigned long long)(unsigned)word_lm->arc_src[a] << 32) | (unsigned)x;
      long long i = (long long)((key * h->hmul) >> (64 - hb));
      while (hash[2 * i] != ~0ull) i = (i + 1) & (H - 1);
      const float wt = lm.weight(a);
      uint32_t bits;
      std::memcpy(&bits, &wt, 4);
      hash[2 * i] = key;
      hash[2 * i + 1] = ((unsigned long long)(unsigned)word_lm->arc_dst[a] << 32) | bits;
    }
    bod.assign(S, -1);
    bow.assign(S, 0.0f);
    endw.assign(S, -std::numeric_limits<float>::infinity());
    for (int s = 0; s < S; s++)
      if (lm.g.eps[s] >= 0) {
        bod[s] = word_lm->arc_dst[lm.g.eps[s]];
        bow[s] = lm.weight(lm.g.eps[s]);
      }
    for (int s : lm_depth_order(lm.g)) {
      const int a = lm.arc(s, V);
      if (!lm.g.has_end)
        endw[s] = 0.0f;
      else if (a >= 0)
        endw[s] = lm.weight(a);
      else if (bod[s] >= 0)
        endw[s] = bow[s] + endw[bod[s]];
    }
  }
  // one device allocation: each array at a 256-byte boundary
  auto r256 = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t b_cls = r256(4ull * C), b_mask = r256(4ull * nodes * MW), b_node = r256(4ull * nodes),
               b_hash = r256(8ull * hash.size()), b_s = r256(4ull * bod.size());
  const size_t total = b_cls + b_mask + 3 * b_node + b_hash + 3 * b_s;
  h->device = ctx->device;
  h->nodes = nodes;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  GTNB_CUDA(ctx, cudaMalloc(&h->mem, total));
  unsigned char* m = static_cast<unsigned char*>(h->mem);
  auto put = [&](auto** dst, const void* src, size_t bytes, size_t span) -> int {
    *dst = reinterpret_cast<std::remove_pointer_t<decltype(dst)>>(m);
    m += span;
    if (bytes) GTNB_CUDA(ctx, cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice));
    return GTNB_OK;
  };
  GTNB_TRY(put(&h->d_cls, h->cls.data(), 4ull * C, b_cls));
  GTNB_TRY(put(&h->d_mask, mask.data(), 4ull * mask.size(), b_mask));
  GTNB_TRY(put(&h->d_first, first.data(), 4ull * nodes, b_node));
  GTNB_TRY(put(&h->d_word, word.data(), 4ull * nodes, b_node));
  GTNB_TRY(put(&h->d_smear, smear.data(), 4ull * nodes, b_node));
  if (word_lm) {
    GTNB_TRY(put(&h->d_hash, hash.data(), 8ull * hash.size(), b_hash));
    GTNB_TRY(put(&h->d_bow, bow.data(), 4ull * bow.size(), b_s));
    GTNB_TRY(put(&h->d_bod, bod.data(), 4ull * bod.size(), b_s));
    GTNB_TRY(put(&h->d_endw, endw.data(), 4ull * endw.size(), b_s));
  }
  GTNB_CUDA(ctx, cudaDeviceSynchronize()); // (set-up: the lexicon is on the device before any stream reads it)
  *out = h.release();
  return GTNB_OK;
}

extern "C" void gtnb_lexicon_destroy(gtnb_ctx* ctx, gtnb_lexicon* lex) {
  if (!lex) return;
  if (ctx) cudaSetDevice(lex->device);
  delete lex; // (cudaFree waits for the device: no launch still reads the lexicon)
}

extern "C" int gtnb_beam_decode_lexicon_async(
    gtnb_ctx* ctx, void* cuda_stream, int B, int T, int C, const void* emissions_dev, int dtype,
    const int32_t* input_lens_dev, int kind, const float* trans_w_dev, int blank, int beam, int nbest,
    const gtnb_lexicon* lexicon, float lm_weight, float word_bonus, int token_beam, int32_t* tokens_dev,
    int32_t* lengths_dev, float* scores_dev, float* am_scores_dev, float* lm_scores_dev, int32_t* words_dev,
    int32_t* word_counts_dev, int32_t* status_dev, void* workspace_dev, size_t workspace_bytes) {
  const std::string fn = "gtnb_beam_decode_lexicon_async";
  if (!ctx || B < 0 || T < 0 || C <= 0 || !lexicon ||
      (B > 0 && ((T > 0 && !emissions_dev) || !tokens_dev || !lengths_dev || !scores_dev)) ||
      (kind == GTNB_DENSE_CTC) != (trans_w_dev == nullptr))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": bad arguments");
  if (!(lm_weight >= 0.0f && std::isfinite(lm_weight)) || !std::isfinite(word_bonus))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": lm_weight must be finite and >= 0, word_bonus finite");
  if (lexicon->device != ctx->device)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the lexicon was made on another device");
  if (lexicon->C != C) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the lexicon was made for another C");
  const BeamAsyncArgs a{B, T, C, dtype, emissions_dev, input_lens_dev, kind, trans_w_dev, blank, beam, nbest,
                        tokens_dev, lengths_dev, scores_dev, status_dev};
  GTNB_TRY(beam_lm_check(ctx, fn, a, token_beam));
  if (kind != GTNB_DENSE_ASG && (lexicon->spelled[blank] || lexicon->cls[blank] == 1))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, fn + ": the lexicon spells with the blank or makes it a separator");
  const BeamLex f{{token_beam, nullptr, nullptr, lexicon->start, lm_weight, word_bonus, am_scores_dev, lm_scores_dev},
                 lexicon->d_cls,
                 (C + 31) / 32,
                 lexicon->d_mask,
                 lexicon->d_first,
                 lexicon->d_word,
                 lexicon->d_smear,
                 lexicon->d_hash,
                 lexicon->hmul,
                 lexicon->hbits,
                 lexicon->d_bow,
                 lexicon->d_bod,
                 lexicon->d_endw,
                 words_dev,
                 word_counts_dev};
  return async_enqueue(ctx, fn, B, cuda_stream, workspace_dev, workspace_bytes,
                       [&](bool launch) { return beam_async_run(ctx, a, launch, f); });
}
