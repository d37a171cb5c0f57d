/*
 * gtnb_criteria.cu -- whole-minibatch criteria: what the reference does with
 * parallelMap(fwd) + parallelMap(bwd) (benchmarks/ctc.cpp:150-165) as ONE call
 * that only enqueues device work: no per-utterance host objects, one pinned
 * staging upload, one small read-back.
 */
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <limits>
#include <string>
#include <vector>

#include "gtnb_internal.h"

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
 * One attempt.  allow_implicit: sweep the frames without building the lattice (k_implicit.cu)
 * when the target graphs qualify; *needs_exact is set when that sweep met a non-finite weight,
 * in which case the outputs are not to be used and the caller repeats the call materialised.
 */
int ctc_loss_run(
    CallScope& scope, int B, int T, int C, const float* emissions, int emissions_on_device,
    const int32_t* input_lens, const int32_t* targets, const int32_t* target_lens, int blank,
    float* losses_host, float* grads, int grads_on_device, bool allow_implicit, bool* needs_exact) {
  gtnb_ctx* ctx = scope.ctx();
  *needs_exact = false;
  PhaseClock pc;
  const long long per = (long long)T * C;

  // host: only sizes.  Graph b has 2U+1 nodes; arcs = self loops + step arcs + skip arcs
  // (benchmarks/ctc.cpp:40-58), skip arcs exist where consecutive labels differ.
  Targets t;
  GTNB_TRY(parse_targets(ctx, "gtnb_ctc_loss", B, T, C, input_lens, targets, target_lens, &t));
  std::vector<SgDims> dims(B);
  for (int b = 0; b < B; b++) {
    const int L = 2 * target_lens[b] + 1;
    const int all_valid = blank >= 0 && blank < C && t.in_range[b];
    dims[b] = SgDims{L, L + (L - 1) + t.skips[b], L >= 2 ? 2 : 1, all_valid, /*uniform=*/1, /*max_in=*/3, /*max_out=*/3};
  }
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
  GTNB_TRY(scope.borrow(emissions, emissions_on_device != 0, per * B, &e_dev));
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
  pc.mark("alloc+meta");
  // the whole criterion in one launch per sub-batch (k_bidir.cu) when the batch qualifies
  const bool bidir =
      implicit && ctx->use_bidir && ctx->use_banded == 0 && bidir_supported(lat, e_dev, per, g.dev, per);
  // PAIR / QUAD kernels (graphs from the targets, one launch): everything small goes through MAPPED pinned memory --
  // the kernel reads the descriptors and targets in place and writes its results straight into the read-back
  // block; no upload, no memset, no download on the path (those enqueues were a large share of the host work)
  const bool direct = implicit && ctx->use_bidir && ctx->use_banded == 0 && ctx->bidir_mode != 0 &&
                      bidir_supported(lat, e_dev, per, g.dev, per) && bidir_takes_targets(lat, 1, blank);
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
  // (k_bidir.cu's PAIR / QUAD kernels take the CTC target graphs from the targets themselves: no tables to build)
  if (!(bidir && direct))
    GTNB_TRY(launch_ctc_build(ctx, lat, small_dev, small_dev + tot_t, small_dev + tot_t + B, blank));
  const int32_t* bidir_targets = direct ? small_mapped : small_dev;
  if (implicit) {
    // the sweeps: k_implicit.cu, or (experimental flag) the temporally blocked ones of k_banded.cu
    const bool banded = ctx->use_banded != 0 && banded_supported(ctx, lat);
    auto sweep_forward = [&](int b0, int nb) {
      return banded ? launch_banded_forward(ctx, lat, status_dev, b0, nb)
                    : launch_implicit_forward(ctx, lat, status_dev, b0, nb);
    };
    auto sweep_backward = [&](int b0, int nb) {
      return banded ? launch_banded_backward(ctx, lat, deltas_dev, g.dev, per, b0, nb)
                    : launch_implicit_backward(ctx, lat, deltas_dev, g.dev, per, b0, nb);
    };
    // everything below only needs what is already enqueued on the main stream (graphs, staging,
    // the memset of the gradients) plus its own slice of the emissions
    cudaEvent_t ev_setup = ctx->side_events[K], ev_lin = ctx->side_events[K + 1];
    const int32_t* T_dev = small_dev + tot_t + 2ll * B;
    GTNB_CUDA(ctx, cudaEventRecord(ev_setup, ctx->stream));
    if (bidir && K == 1 && !h2d_event && !(grads && !grads_on_device)) {
      GTNB_TRY(launch_bidir_ctc(ctx, lat, status_dev, zparts_dev, boff_dev, g.dev, per, 0, -1, /*zero_w=*/1,
                                bidir_scores_dev, blank, bidir_targets, bidir_targets + tot_t,
                                direct ? meta_mapped : nullptr));
    } else if (!bidir && K == 1 && !h2d_event && !(grads && !grads_on_device)) {
      // forwardScore(emissions) and its +1 gradient beside the forward sweep
      GTNB_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ev_setup, 0));
      {
        OnStream side(ctx, ctx->copy_stream);
        GTNB_TRY(launch_linear_forward(ctx, B, T_dev, maxT, C, e_dev, per, 0, z_dev, g.dev, per, nullptr, 1.0f,
                                       input_lens ? 0 : 1, row_scratch));
      }
      GTNB_CUDA(ctx, cudaEventRecord(ev_lin, ctx->copy_stream));
      GTNB_TRY(sweep_forward(0, -1));
      GTNB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ev_lin, 0));
      if (grads) GTNB_TRY(sweep_backward(0, -1));
    } else {
      for (int k = 0; k < K; k++) {
        const int b0 = chunk_lo[k], nb = chunk_lo[k + 1] - chunk_lo[k];
        cudaStream_t cs = ctx->side_streams[k];
        GTNB_CUDA(ctx, cudaStreamWaitEvent(cs, ev_setup, 0));
        if (h2d_event) GTNB_CUDA(ctx, cudaStreamWaitEvent(cs, ctx->side_events[k], 0));
        {
          OnStream side(ctx, cs);
          if (bidir) {
            GTNB_TRY(launch_bidir_ctc(ctx, lat, status_dev, zparts_dev, boff_dev, g.dev, per, b0, nb, /*zero_w=*/1,
                                      bidir_scores_dev, blank, bidir_targets, bidir_targets + tot_t,
                                      direct ? meta_mapped : nullptr));
          } else {
            GTNB_TRY(launch_linear_forward(ctx, nb, T_dev + b0, maxT, C, e_dev + (long long)b0 * per, per, 0,
                                           z_dev + b0, g.dev ? g.dev + (long long)b0 * per : nullptr, per, nullptr,
                                           1.0f, input_lens ? 0 : 1,
                                           row_scratch + (long long)b0 * std::max(maxT, 1)));
            GTNB_TRY(sweep_forward(b0, nb));
            if (grads) GTNB_TRY(sweep_backward(b0, nb));
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

/*
 * viterbiPath(compose(linearGraph(T, C; e_b), transitions)) for a whole minibatch, with the
 * dense transitions graph of test/criterion_test.cpp:244-254 / :316-326, through the
 * factored kernel (k_dense.cu): the T*C*C lattice is never materialised.
 * (the device scratch of a call comes from the context's call-scoped arena, as in gtnb_ctc_loss: no stream-ordered
 * allocations on the path after the first call of a shape)
 */
extern "C" int gtnb_viterbi_dense(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
    const int32_t* input_lens, const float* trans_w_host, int32_t* paths_host, float* scores_host) {
  if (!ctx || B < 0 || T < 0 || C <= 0 || !emissions || !trans_w_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_viterbi_dense: bad arguments");
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  if (input_lens)
    for (int b = 0; b < B; b++)
      if (input_lens[b] < 0 || input_lens[b] > T)
        return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_viterbi_dense: input_lens out of range");
  const long long per = (long long)T * C;
  CallScope scope(ctx);
  float *e_dev = nullptr, *tr_dev = nullptr, *sc_dev = nullptr;
  int32_t *T_dev = nullptr, *paths_dev = nullptr;
  uint8_t* bp = nullptr;
  GTNB_TRY(scope.input(emissions, emissions_on_device, per * B, &e_dev));
  GTNB_TRY(scope.alloc(&tr_dev, (long long)C + (long long)C * C));
  GTNB_TRY(scope.alloc(&sc_dev, B));
  GTNB_TRY(scope.alloc(&paths_dev, (long long)B * std::max(T, 1)));
  GTNB_TRY(scope.alloc(&bp, (long long)B * std::max(T, 1) * C));
  if (input_lens) GTNB_TRY(scope.alloc(&T_dev, B));
  GTNB_TRY(stage_begin(ctx));
  GTNB_TRY(stage_upload(ctx, tr_dev, trans_w_host, sizeof(float) * ((size_t)C + (size_t)C * C)));
  if (input_lens) GTNB_TRY(stage_upload(ctx, T_dev, input_lens, sizeof(int32_t) * B));
  GTNB_TRY(stage_end(ctx));
  GTNB_TRY(launch_viterbi_dense(ctx, B, T, C, T_dev, e_dev, per, tr_dev, bp, paths_dev, sc_dev));
  if (paths_host && T > 0)
    GTNB_CUDA(ctx, cudaMemcpyAsync(paths_host, paths_dev, sizeof(int32_t) * (size_t)B * T, cudaMemcpyDeviceToHost,
                                   ctx->stream));
  if (scores_host)
    GTNB_CUDA(ctx, cudaMemcpyAsync(scores_host, sc_dev, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
  return scope.sync();
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
};

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

void build_asg_graphs(int C, const float* trans_w_host, const Targets& t, AsgGraphs* g) {
  const int nTrans = C + C * C;
  HostGraph& tr = g->trans;
  tr.flags.assign(C + 1, 2);
  tr.flags[0] = 1;
  tr.src.resize(nTrans);
  tr.dst.resize(nTrans);
  tr.label.resize(nTrans);
  tr.w.assign(trans_w_host, trans_w_host + nTrans);
  for (int i = 0; i < C; i++) {
    tr.src[i] = 0;
    tr.dst[i] = i + 1;
    tr.label[i] = i;
  }
  for (int i = 0; i < C; i++)
    for (int j = 0; j < C; j++) {
      const int a = C + i * C + j;
      tr.src[a] = j + 1;
      tr.dst[a] = i + 1;
      tr.label[a] = i;
    }
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
  decltype(&launch_ngram_num_build) num_build;
  decltype(&launch_ngram_den_forward) den_forward;
  decltype(&launch_ngram_den_backward) den_backward;
};

int trellis_loss_fast(CallScope& scope, const TrellisCriterion& k, const TransitionArgs& a, const Targets& t,
                      const std::vector<SgDims>& dims, bool* needs_exact) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = a.B, T = a.T, C = a.C;
  const long long per = (long long)T * C, tot_t = t.tot_t;
  const bool want = a.grads || a.trans_grad;
  long long tot_A = 0;
  for (int b = 0; b < B; b++) tot_A += dims[b].A;
  float *e_dev = nullptr, *w_dev = nullptr, *sigma = nullptr, *alpha = nullptr, *den = nullptr;
  float *ggrad = nullptr, *minus1 = nullptr;
  int32_t *small_dev = nullptr, *status = nullptr, *map = nullptr;
  OutBuf g, tg;
  std::vector<long long> sgn, sga;
  std::vector<float> m1(B, -1.0f);
  gtnb_lattice*& lat = scope.lattice();

  GTNB_TRY(ensure_side_streams(ctx, 0, 0));
  GTNB_TRY(scope.input(a.emissions, a.emissions_on_device, per * B, &e_dev));
  GTNB_TRY(scope.borrow(a.trans_w, a.trans_on_device != 0, k.n_trans, &w_dev)); // (host: staged below)
  const std::vector<int32_t> small_h = t.packed();
  GTNB_TRY(scope.alloc(&small_dev, (long long)small_h.size()));
  GTNB_TRY(scope.alloc(&status, 2ll * B));
  if (k.fold) GTNB_TRY(scope.alloc(&sigma, C));
  GTNB_TRY(scope.alloc(&alpha, k.alpha_floats));
  GTNB_TRY(scope.alloc(&den, B));
  GTNB_TRY(scope.alloc(&map, tot_A));
  GTNB_TRY(composed_alloc(ctx, B, dims.data(), B, 0, t.T(), C, e_dev, per, sgn, sga, &lat, true));
  if (want) {
    const long long n_grad = k.n_trans + (k.fold ? C : 0); // [d/dtrans | d/dsigma]
    GTNB_TRY(scope.output(a.grads, a.grads_on_device, per * B, &g));
    GTNB_TRY(scope.output(a.trans_grad, a.trans_grad_on_device, n_grad, &tg, /*alias=*/!k.fold));
    GTNB_TRY(scope.alloc(&ggrad, tot_A));
    GTNB_TRY(scope.alloc(&minus1, B));
    GTNB_CUDA(ctx, cudaMemsetAsync(g.dev, 0, sizeof(float) * per * B, ctx->stream));
    GTNB_CUDA(ctx, cudaMemsetAsync(tg.dev, 0, sizeof(float) * n_grad, ctx->stream));
    if (tot_A) GTNB_CUDA(ctx, cudaMemsetAsync(ggrad, 0, sizeof(float) * tot_A, ctx->stream));
  }
  GTNB_CUDA(ctx, cudaMemsetAsync(status, 0, sizeof(int32_t) * 2 * B, ctx->stream));
  // one pinned staging pass: descriptors, [targets | offsets | lens | T], the transitions from the host, the -1 seeds
  GTNB_TRY(stage_begin(ctx));
  GTNB_TRY(stage_upload(ctx, lat->meta, lat->meta_h.data(), sizeof(GraphMeta) * B));
  GTNB_TRY(stage_upload(ctx, small_dev, small_h.data(), sizeof(int32_t) * small_h.size()));
  if (!a.trans_on_device) GTNB_TRY(stage_upload(ctx, w_dev, a.trans_w, sizeof(float) * k.n_trans));
  if (want) GTNB_TRY(stage_upload(ctx, minus1, m1.data(), sizeof(float) * B));
  GTNB_TRY(stage_end(ctx));

  if (k.fold) GTNB_TRY(launch_ngram_sigma(ctx, C, w_dev, sigma));
  GTNB_TRY(k.num_build(ctx, lat, small_dev, small_dev + tot_t, small_dev + tot_t + B, a.blank, w_dev, sigma, map));
  // the numerator (a few in-arcs per node) on the second stream beside the denominator (C^2 per frame)
  GTNB_TRY(fork_to(ctx, ctx->copy_stream));
  {
    OnStream side(ctx, ctx->copy_stream);
    GTNB_TRY(launch_implicit_forward(ctx, lat, status + B));
    if (want) GTNB_TRY(launch_implicit_backward(ctx, lat, minus1, g.dev, per, 0, -1, ggrad));
  }
  const int32_t* T_dev = small_dev + tot_t + 2ll * B;
  GTNB_TRY(k.den_forward(ctx, B, T, C, T_dev, e_dev, per, w_dev, alpha, den, status));
  if (want) GTNB_TRY(k.den_backward(ctx, B, T, C, T_dev, e_dev, per, w_dev, alpha, den, g.dev, per, tg.dev));
  GTNB_TRY(join_from(ctx, ctx->copy_stream));
  if (want) {
    GTNB_TRY(launch_scatter_add(ctx, tg.dev, map, ggrad, tot_A)); // numerator arcs -> transition (and sigma) slots
    if (k.fold) GTNB_TRY(launch_ngram_fold(ctx, C, w_dev, sigma, tg.dev));
    GTNB_TRY(g.copy_out(ctx, per * B));
    GTNB_TRY(tg.copy_out(ctx, k.n_trans));
  }
  return read_losses(scope, B, den, lat->out_scores, status, 2ll * B, a.losses_host, needs_exact);
}

/*
 * n-gram CTC through materialised lattices, graph by graph as the reference composes them: intersect(E_b, G) and
 * intersect(P_b, E_b), where P_b = intersect(ctc_b, G) is built on the host WITHOUT the fold (C start states
 * (0, s), then (l, label(l))).  Reproduces the reference's inf / NaN propagation arc by arc; the path for
 * non-finite weights.
 */
int ngram_ctc_loss_exact(CallScope& scope, const TransitionArgs& a, const Targets& t) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = a.B, T = a.T, C = a.C;
  const long long per = (long long)T * C, CC = (long long)C * C;
  const bool want = a.grads || a.trans_grad;
  std::vector<float> W(CC);
  GTNB_TRY(read_to_host(ctx, W.data(), a.trans_w, a.trans_on_device, CC));
  // G (benchmarks/ctc.cpp transitionsGraph with a label-determined destination): arc j*C + i = j -> i
  HostGraph G;
  G.flags.assign(C, 3);
  G.src.resize(CC);
  G.dst.resize(CC);
  G.label.resize(CC);
  G.w.resize(CC);
  std::vector<int32_t> gmap(CC);
  for (int j = 0; j < C; j++)
    for (int i = 0; i < C; i++) {
      const long long k = (long long)j * C + i;
      G.src[k] = j;
      G.dst[k] = i;
      G.label[k] = i;
      G.w[k] = W[(long long)i * C + j];
      gmap[k] = i * C + j;
    }
  const gtnb_graph_view gview = G.view();
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
  const long long nP = (long long)pmap.size();
  float *e_dev = nullptr, *ft_grad = nullptr, *gg_grad = nullptr;
  int32_t *ft_map_dev = nullptr, *gg_map_dev = nullptr;
  OutBuf g, tg;
  gtnb_lattice*& den = scope.lattice();
  gtnb_lattice*& num = scope.lattice();
  GTNB_TRY(scope.input(a.emissions, a.emissions_on_device, per * B, &e_dev));
  GTNB_TRY(gtnb_compose_linear(ctx, B, &gview, 1, 1, t.T(), C, e_dev, per, &den));
  GTNB_TRY(gtnb_compose_linear(ctx, B, pviews.data(), B, 0, t.T(), C, e_dev, per, &num));
  GTNB_TRY(gtnb_forward(ctx, den, 0, nullptr, nullptr));
  GTNB_TRY(gtnb_forward(ctx, num, 0, nullptr, nullptr));
  if (want) {
    GTNB_TRY(scope.output(a.grads, a.grads_on_device, per * B, &g));
    GTNB_CUDA(ctx, cudaMemsetAsync(g.dev, 0, sizeof(float) * per * B, ctx->stream));
    GTNB_TRY(scope.output(a.trans_grad, a.trans_grad_on_device, CC, &tg, /*alias=*/false));
    GTNB_TRY(scope.alloc(&gg_grad, CC));
    GTNB_TRY(scope.alloc(&ft_grad, std::max<long long>(nP, 1)));
    GTNB_TRY(scope.alloc(&gg_map_dev, CC));
    GTNB_TRY(scope.alloc(&ft_map_dev, std::max<long long>(nP, 1)));
    GTNB_CUDA(ctx, cudaMemsetAsync(tg.dev, 0, sizeof(float) * CC, ctx->stream));
    GTNB_CUDA(ctx, cudaMemsetAsync(gg_grad, 0, sizeof(float) * CC, ctx->stream));
    GTNB_CUDA(ctx, cudaMemsetAsync(ft_grad, 0, sizeof(float) * std::max<long long>(nP, 1), ctx->stream));
    std::vector<float> m1(B, -1.0f);
    GTNB_TRY(gtnb_backward(ctx, den, 0, nullptr)); // +1 / -1: subtract's gradFunc (functions.cpp:53-58)
    GTNB_TRY(gtnb_backward(ctx, num, 0, m1.data()));
    GTNB_TRY(gtnb_compose_grad(ctx, den, gg_grad, g.dev, per));
    GTNB_TRY(gtnb_compose_grad(ctx, num, ft_grad, g.dev, per));
    GTNB_TRY(stage_begin(ctx));
    GTNB_TRY(stage_upload(ctx, gg_map_dev, gmap.data(), sizeof(int32_t) * CC));
    if (nP) GTNB_TRY(stage_upload(ctx, ft_map_dev, pmap.data(), sizeof(int32_t) * nP));
    GTNB_TRY(stage_end(ctx));
    GTNB_TRY(launch_scatter_add(ctx, tg.dev, gg_map_dev, gg_grad, CC));
    GTNB_TRY(launch_scatter_add(ctx, tg.dev, ft_map_dev, ft_grad, nP));
    GTNB_TRY(g.copy_out(ctx, per * B));
    GTNB_TRY(tg.copy_out(ctx, CC));
  }
  bool unused = false;
  return read_losses(scope, B, den->out_scores, num->out_scores, nullptr, 0, a.losses_host, &unused);
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
extern "C" int gtnb_ngram_ctc_loss(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const float* trans_w, int trans_on_device, const int32_t* targets, const int32_t* target_lens, int blank,
    float* losses_host, float* grads, int grads_on_device, float* trans_grad, int trans_grad_on_device) {
  const TransitionArgs a{B, T, C, emissions, emissions_on_device, input_lens, trans_w, trans_on_device, targets,
                         target_lens, blank, losses_host, grads, grads_on_device, trans_grad, trans_grad_on_device};
  if (!ctx || B < 0 || T < 0 || C <= 0 || !emissions || !trans_w || !target_lens || !losses_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss: bad arguments");
  if (blank < 0 || blank >= C)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss: blank outside [0, C)");
  if (C > kNgramMaxLabels)
    return fail(ctx, GTNB_ERR_UNSUPPORTED,
                "gtnb_ngram_ctc_loss: C = " + std::to_string(C) + " labels; the trellis kernels hold W on chip for C <= " +
                    std::to_string(kNgramMaxLabels));
  Targets t;
  GTNB_TRY(parse_targets(ctx, "gtnb_ngram_ctc_loss", B, T, C, input_lens, targets, target_lens, &t));
  std::vector<SgDims> dims(B);
  for (int b = 0; b < B; b++) {
    if (!t.in_range[b]) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss: label outside [0, C)");
    // folded numerator graph: S + 2U+1 CTC nodes; arcs = self loops + steps + skips + the two S arcs (one if U = 0)
    const int L = 2 * target_lens[b] + 1;
    dims[b] = SgDims{L + 1, L + (L - 1) + t.skips[b] + std::min(L, 2), L >= 2 ? 2 : 1, /*all_valid=*/1,
                     /*uniform=*/1, /*max_in=*/3, /*max_out=*/3};
  }
  const TrellisCriterion ngram{(long long)C * C, (long long)B * (T + 1) * C, /*fold=*/true, launch_ngram_num_build,
                               launch_ngram_den_forward, launch_ngram_den_backward};
  const bool fast = implicit_dims_supported(dims.data(), B) && ctx->use_implicit;
  return run_criterion(ctx, B, t.T(), losses_host, trans_grad, trans_grad_on_device, (long long)C * C, fast,
                       [&](CallScope& scope, bool f, bool* needs_exact) {
                         return f ? trellis_loss_fast(scope, ngram, a, t, dims, needs_exact)
                                  : ngram_ctc_loss_exact(scope, a, t);
                       });
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
extern "C" int gtnb_asg_loss_ex(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const float* trans_w, int trans_on_device, const int32_t* targets, const int32_t* target_lens,
    float* losses_host, float* grads, int grads_on_device, float* trans_grad, int trans_grad_on_device) {
  const TransitionArgs a{B, T, C, emissions, emissions_on_device, input_lens, trans_w, trans_on_device, targets,
                         target_lens, -1, losses_host, grads, grads_on_device, trans_grad, trans_grad_on_device};
  if (!ctx || B < 0 || T < 0 || C <= 0 || !emissions || !trans_w || !target_lens || !losses_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss_ex: bad arguments");
  const long long nTrans = C + (long long)C * C;
  Targets t;
  GTNB_TRY(parse_targets(ctx, "gtnb_asg_loss_ex", B, T, C, input_lens, targets, target_lens, &t));
  std::vector<SgDims> dims(B);
  for (int b = 0; b < B; b++) {
    if (!t.in_range[b]) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss_ex: label outside [0, C)");
    // compose(fal_b, transitions): U+1 nodes, 2U arcs (none when U = 0), node U accepts
    const int U = target_lens[b];
    dims[b] = SgDims{U + 1, 2 * U, U > 0 ? 1 : 0, /*all_valid=*/1, /*uniform=*/1, /*max_in=*/2, /*max_out=*/2};
  }
  const TrellisCriterion asg{nTrans, asg_alpha_floats(B, T, C), /*fold=*/false, asg_num_build, launch_asg_den_forward,
                             launch_asg_den_backward};
  // (a non-finite weight: gtnb_asg_loss's sweeps raise the same status bit and end in the materialised lattices)
  const bool fast = C <= kNgramMaxLabels && ctx->use_implicit && implicit_dims_supported(dims.data(), B);
  return run_criterion(ctx, B, t.T(), losses_host, trans_grad, trans_grad_on_device, nTrans, fast,
                       [&](CallScope& scope, bool f, bool* needs_exact) {
                         return f ? trellis_loss_fast(scope, asg, a, t, dims, needs_exact)
                                  : asg_loss_generic(scope, a, t);
                       });
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

struct GraphLossArgs {
  int B, T, C;
  const float* emissions;
  int emissions_on_device;
  const gtnb_graph_view* graphs;
  const float* arc_weights;
  int arc_weights_on_device;
  float* losses_host;
  float* grads;
  int grads_on_device;
  float* arc_grads;
  int arc_grads_on_device;
};

/* one attempt; implicit: try the sweeps first (the materialised lattices when the graphs do not qualify).
 * *needs_exact: a sweep met a non-finite weight or emission, the outputs are not to be used. */
int graph_loss_once(CallScope& scope, const GraphLossArgs& a, const std::vector<gtnb_graph_view>& views,
                    const std::vector<int32_t>& Tb, long long tot_arcs, bool implicit, bool* needs_exact) {
  gtnb_ctx* ctx = scope.ctx();
  const int B = a.B, T = a.T, C = a.C;
  const long long per = (long long)T * C;
  const bool want = a.grads || a.arc_grads;
  const int maxT = *std::max_element(Tb.begin(), Tb.end());
  float *e_dev = nullptr, *den = nullptr, *minus1 = nullptr;
  int32_t *T_dev = nullptr, *status = nullptr;
  OutBuf g, ag;
  gtnb_lattice*& lat = scope.lattice();
  gtnb_lattice*& dlat = scope.lattice();
  const float* aw_dev = a.arc_weights_on_device ? a.arc_weights : nullptr;
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

  if (implicit) {
    const int rc = compose_linear_impl(ctx, B, views.data(), B, 0, Tb.data(), C, e_dev, per, true, &lat, true, aw_dev);
    if (rc == GTNB_ERR_UNSUPPORTED) // does not fit the implicit layout: materialise
      implicit = false;
    else
      GTNB_TRY(rc);
  }
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
    GTNB_TRY(compose_linear_impl(ctx, B, views.data(), B, 0, Tb.data(), C, e_dev, per, false, &lat, false, aw_dev));
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
  const GraphLossArgs a{B, T, C, emissions, emissions_on_device, graphs, arc_weights, arc_weights_on_device,
                        losses_host, grads, grads_on_device, arc_grads, arc_grads_on_device};
  if (!ctx || B < 0 || T < 0 || C <= 0 || (B > 0 && (!emissions || !graphs || !losses_host)))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_graph_loss: bad arguments");
  std::vector<int32_t> Tb(B);
  std::vector<gtnb_graph_view> views(graphs, graphs + B);
  long long tot_arcs = 0;
  for (int b = 0; b < B; b++) {
    Tb[b] = input_lens ? input_lens[b] : T;
    if (Tb[b] < 0 || Tb[b] > T) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_graph_loss: input_lens outside [0, T]");
    if (validate_view(ctx, views[b])) return GTNB_ERR_INVALID_ARGUMENT;
    for (int k = 0; k < views[b].num_arcs; k++)
      if (views[b].arc_olabel[k] == GTNB_EPSILON)
        return fail(ctx, GTNB_ERR_UNSUPPORTED,
                    "gtnb_graph_loss: graph " + std::to_string(b) +
                        " has epsilon arcs; remove them first (remove(g, epsilon))");
    if (arc_weights && !arc_weights_on_device) views[b].weights = arc_weights + tot_arcs;
    tot_arcs += views[b].num_arcs;
  }
  if (tot_arcs >= (1ll << 31)) return fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_graph_loss: more than 2^31 arcs");
  // (graphs that are not label-uniform need C <= k_implicit.cu's kArcMaxLabels: compose_linear_impl checks)
  return run_criterion(ctx, B, Tb.data(), losses_host, nullptr, 0, 0, ctx->use_implicit,
                       [&](CallScope& scope, bool implicit, bool* needs_exact) {
                         return graph_loss_once(scope, a, views, Tb, tot_arcs, implicit, needs_exact);
                       });
}
