/*
 * gtnb_criteria.cu -- whole-minibatch criteria: what the reference does with
 * parallelMap(fwd) + parallelMap(bwd) (benchmarks/ctc.cpp:150-165) as ONE call
 * that only enqueues device work: no per-utterance host objects, one pinned
 * staging upload, one small read-back.
 */
#include <algorithm>
#include <cstdlib>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <string>
#include <vector>

#include "gtnb_internal.h"

using namespace gtnb;

/*
 * One attempt.  allow_implicit: sweep the frames without building the lattice (k_implicit.cu)
 * when the target graphs qualify; *needs_exact is set when that sweep met a non-finite weight,
 * in which case the outputs are not to be used and the caller repeats the call materialised.
 */
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
} // namespace

static int ctc_loss_run(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
    const int32_t* input_lens, const int32_t* targets, const int32_t* target_lens, int blank,
    float* losses_host, float* grads, int grads_on_device, bool allow_implicit, bool* needs_exact) {
  *needs_exact = false;
  if (!ctx || B < 0 || T < 0 || C <= 0 || !emissions || !target_lens || !losses_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctc_loss: bad arguments");
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  PhaseClock pc;
  bool direct = false; // the PAIR / QUAD kernels of k_bidir.cu on mapped pinned memory (see below)
  const GraphMeta* meta_mapped = nullptr;
  const int32_t* small_mapped = nullptr;
  const long long per = (long long)T * C;
  int rc = GTNB_OK;
  float* e_dev = nullptr;
  float* g_dev = nullptr;
  float* z_dev = nullptr;
  float* deltas_dev = nullptr;
  int32_t* small_dev = nullptr; // [targets | offsets | lens | T]
  int32_t* status_dev = nullptr;
  float* row_scratch = nullptr; // k_linear.cu's per-frame scores, allocated once for all sub-batches
  float* zparts_dev = nullptr; // k_bidir.cu: forwardScore(emissions) as two partial sums per utterance
  float* boff_dev = nullptr; // k_bidir.cu: per-block score offsets of the two CTAs of every utterance
  float* bidir_scores_dev = nullptr; // k_bidir.cu: the lattices' scores, inside the read-back block
  bool implicit = false;
  bool bidir = false;
  int zp = 1;
  int K = 1; // sub-batches (implicit path with host buffers)
  std::vector<int> chunk_lo;
  cudaStream_t main_stream = ctx->stream;
  gtnb_lattice* lat = nullptr;
  cudaEvent_t h2d_event = nullptr;
  std::vector<long long> sgn, sga;

  // host: only sizes.  Graph b has 2U+1 nodes; arcs = self loops + step arcs + skip arcs
  // (benchmarks/ctc.cpp:40-58), skip arcs exist where consecutive labels differ.
  std::vector<SgDims> dims(B);
  std::vector<int32_t> Tb(B), off(B);
  long long tot_t = 0;
  for (int b = 0; b < B; b++) {
    const int U = target_lens[b];
    if (U < 0) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctc_loss: negative target length");
    if (U > 0 && !targets) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctc_loss: targets is NULL");
    off[b] = (int32_t)tot_t;
    const int32_t* tg = targets + tot_t;
    int skips = 0;
    int all_valid = blank >= 0 && blank < C;
    if (U > 0) all_valid &= (unsigned)tg[0] < (unsigned)C;
    for (int u = 1; u < U; u++) { // one pass: skip arcs exist where consecutive labels differ; labels in [0, C)
      skips += tg[u] != tg[u - 1];
      all_valid &= (unsigned)tg[u] < (unsigned)C;
    }
    const int L = 2 * U + 1;
    dims[b] = SgDims{L, L + (L - 1) + skips, L >= 2 ? 2 : 1, all_valid, /*uniform=*/1, /*max_in=*/3, /*max_out=*/3};
    tot_t += U;
    Tb[b] = input_lens ? input_lens[b] : T;
    if (Tb[b] < 0 || Tb[b] > T)
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ctc_loss: input_lens out of range");
  }
  int maxT = 0;
  for (int b = 0; b < B; b++) maxT = std::max(maxT, Tb[b]);
  pc.mark("sizes");

#define TRY(x)                 \
  do {                         \
    if ((rc = (x))) goto done; \
  } while (0)
#define TRYCUDA(call)                                      \
  do {                                                     \
    cudaError_t e__ = (call);                              \
    if (e__ != cudaSuccess) {                              \
      rc = cuda_fail(ctx, e__, #call, __FILE__, __LINE__); \
      goto done;                                           \
    }                                                      \
  } while (0)

  implicit = allow_implicit && implicit_dims_supported(dims.data(), B);
  // Host buffers: cut the batch into K sub-batches whose H2D copy, kernels and D2H copy run on
  // their own streams, so that the two PCIe directions and the (latency-bound) sweeps overlap.
  // Device buffers: K = 1, and the normaliser (k_linear.cu) runs beside the forward sweep.
  if (implicit && (!emissions_on_device || (grads && !grads_on_device))) {
    const long long bytes = (long long)sizeof(float) * per * B;
    K = (int)std::min<long long>(std::max<long long>(bytes / (4ll << 20), 1), 16);
    K = std::min(K, B);
  }
  TRY(ensure_side_streams(ctx, K, K + 2));
  chunk_lo.resize(K + 1);
  for (int k = 0; k <= K; k++) chunk_lo[k] = (int)((long long)B * k / K);
  if (emissions_on_device) {
    e_dev = const_cast<float*>(emissions);
  } else {
    // the copy runs on a second stream while this one builds the target graphs and the
    // lattice structure (k_ctc.cu, compose alive / count / scan need no emissions)
    TRY(dev_alloc(ctx, &e_dev, per * B));
  }
  if (grads) {
    if (grads_on_device)
      g_dev = grads;
    else
      TRY(dev_alloc(ctx, &g_dev, per * B));
    // with full-length utterances the normaliser's gradient overwrites every element
    if (input_lens) TRYCUDA(cudaMemsetAsync(g_dev, 0, sizeof(float) * per * B, ctx->stream));
  }
  TRY(dev_alloc(ctx, &z_dev, B));
  TRY(dev_alloc(ctx, &deltas_dev, B));
  TRY(dev_alloc(ctx, &small_dev, tot_t + 3ll * B));
  TRY(composed_alloc(ctx, B, dims.data(), B, 0, Tb.data(), C, e_dev, per, sgn, sga, &lat, implicit));
  pc.mark("alloc+meta");
  // the whole criterion in one launch per sub-batch (k_bidir.cu) when the batch qualifies
  bidir = implicit && ctx->use_bidir && ctx->use_banded == 0 && bidir_supported(lat, e_dev, per, g_dev, per);
  // PAIR / QUAD kernels (graphs from the targets, one launch): everything small goes through MAPPED pinned memory --
  // the kernel reads the descriptors and targets in place and writes its results straight into the read-back
  // block; no upload, no memset, no download on the path (those enqueues were a large share of the host work)
  direct = implicit && ctx->use_bidir && ctx->use_banded == 0 && ctx->bidir_mode != 0 &&
           bidir_supported(lat, e_dev, per, g_dev, per) && bidir_takes_targets(lat, 1, blank);
  if (bidir && direct) {
    const long long zpb = 2ll * B * bidir_zparts();
    TRY(readback_reserve(ctx, (zpb + 2ll * B) * sizeof(float)));
    zparts_dev = reinterpret_cast<float*>(ctx->readback);
    bidir_scores_dev = zparts_dev + zpb;
    status_dev = reinterpret_cast<int32_t*>(zparts_dev + zpb + B);
    std::memset(status_dev, 0, sizeof(int32_t) * B);
    TRY(dev_alloc(ctx, &boff_dev, 8ll * B * bidir_blocks(maxT)));
  } else if (bidir) {
    // one block for everything that is read back: [partial sums of forwardScore(e) | lattice scores | status]
    const long long zpb = 2ll * B * bidir_zparts();
    TRY(dev_alloc(ctx, &zparts_dev, zpb + 2ll * B));
    bidir_scores_dev = zparts_dev + zpb;
    status_dev = reinterpret_cast<int32_t*>(zparts_dev + zpb + B);
    TRY(dev_alloc(ctx, &boff_dev, 8ll * B * bidir_blocks(maxT)));
    TRYCUDA(cudaMemsetAsync(status_dev, 0, sizeof(int32_t) * B, ctx->stream));
  } else if (implicit) {
    TRY(dev_alloc(ctx, &row_scratch, (long long)B * std::max(maxT, 1)));
    TRY(dev_alloc(ctx, &status_dev, B));
    TRYCUDA(cudaMemsetAsync(status_dev, 0, sizeof(int32_t) * B, ctx->stream));
  }

  // one pinned staging pass for everything the kernels need from the host
  TRY(stage_begin(ctx));
  {
    // [targets | offsets | lens | T] in ONE copy (each small copy costs microseconds of stream latency)
    std::vector<int32_t> small_h;
    if (!(bidir && direct)) {
      small_h.resize((size_t)(tot_t + 3ll * B));
      if (tot_t) std::memcpy(small_h.data(), targets, sizeof(int32_t) * tot_t);
      std::memcpy(small_h.data() + tot_t, off.data(), sizeof(int32_t) * B);
      std::memcpy(small_h.data() + tot_t + B, target_lens, sizeof(int32_t) * B);
      std::memcpy(small_h.data() + tot_t + 2ll * B, Tb.data(), sizeof(int32_t) * B);
    }
    if (bidir && direct) {
      // the kernel needs the descriptors (with the target offsets) and the labels, nothing else
      void *m = nullptr, *t = nullptr;
      for (int b = 0; b < B; b++) lat->meta_h[b].tgt_off = off[b];
      TRY(stage_reserve(ctx, sizeof(GraphMeta) * B + sizeof(int32_t) * (size_t)tot_t + 1024));
      TRY(stage_place(ctx, lat->meta_h.data(), sizeof(GraphMeta) * B, &m));
      TRY(stage_place(ctx, targets, sizeof(int32_t) * (size_t)tot_t, &t));
      meta_mapped = static_cast<const GraphMeta*>(m);
      small_mapped = static_cast<const int32_t*>(t);
    } else {
      TRY(stage_upload(ctx, lat->meta, lat->meta_h.data(), sizeof(GraphMeta) * B));
      TRY(stage_upload(ctx, small_dev, small_h.data(), sizeof(int32_t) * small_h.size()));
    }
  }
  if (!bidir) {
    std::vector<float> minus1(B, -1.0f); // subtract's gradFunc, functions.cpp:53-58
    TRY(stage_upload(ctx, deltas_dev, minus1.data(), sizeof(float) * B));
  }
  if (!(bidir && direct)) TRY(stage_end(ctx)); // (direct: no copy was issued from the staging buffer; the call synchronises before it returns)
  pc.mark("staging");
  if (!emissions_on_device) {
    // enqueued AFTER the small staged upload: the copy engine serves one direction in
    // submission order, and the graphs must not queue behind 65 MB of emissions
    TRYCUDA(cudaEventRecord(ctx->ev_fork, ctx->stream)); // orders the copy after the allocation
    TRYCUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_fork, 0));
    for (int k = 0; k < K; k++) {
      const long long lo = (long long)chunk_lo[k] * per, n = (long long)(chunk_lo[k + 1] - chunk_lo[k]) * per;
      TRYCUDA(cudaMemcpyAsync(e_dev + lo, emissions + lo, sizeof(float) * n, cudaMemcpyHostToDevice,
                              ctx->copy_stream));
      TRYCUDA(cudaEventRecord(ctx->side_events[k], ctx->copy_stream));
    }
    TRYCUDA(cudaEventRecord(ctx->ev_join, ctx->copy_stream));
    h2d_event = ctx->ev_join;
  }

  // ctcGraph -> intersect(ctc, emissions) -> forwardScore -> backward(-1) -> compose gradFunc
  // (k_bidir.cu's PAIR / QUAD kernels take the CTC target graphs from the targets themselves: no tables to build)
  if (!(bidir && direct))
    TRY(launch_ctc_build(ctx, lat, small_dev, small_dev + tot_t, small_dev + tot_t + B, blank));
  if (implicit) {
    // the sweeps: k_implicit.cu, or (experimental flag) the temporally blocked ones of k_banded.cu
    const bool banded = ctx->use_banded != 0 && banded_supported(ctx, lat);
    auto sweep_forward = [&](int b0, int nb) {
      return banded ? launch_banded_forward(ctx, lat, status_dev, b0, nb)
                    : launch_implicit_forward(ctx, lat, status_dev, b0, nb);
    };
    auto sweep_backward = [&](int b0, int nb) {
      return banded ? launch_banded_backward(ctx, lat, deltas_dev, g_dev, per, b0, nb)
                    : launch_implicit_backward(ctx, lat, deltas_dev, g_dev, per, b0, nb);
    };
    // everything below only needs what is already enqueued on the main stream (graphs, staging,
    // the memset of the gradients) plus its own slice of the emissions
    cudaEvent_t ev_setup = ctx->side_events[K], ev_lin = ctx->side_events[K + 1];
    const int32_t* T_dev = small_dev + tot_t + 2ll * B;
    TRYCUDA(cudaEventRecord(ev_setup, main_stream));
    if (bidir && K == 1 && !h2d_event && !(grads && !grads_on_device)) {
      TRY(launch_bidir_ctc(ctx, lat, status_dev, zparts_dev, boff_dev, g_dev, per, 0, -1, /*zero_w=*/1, bidir_scores_dev, blank, direct ? small_mapped : small_dev,
                               (direct ? small_mapped : small_dev) + tot_t, direct ? meta_mapped : nullptr));
    } else if (bidir) {
      for (int k = 0; k < K && !rc; k++) {
        const int b0 = chunk_lo[k], nb = chunk_lo[k + 1] - chunk_lo[k];
        cudaStream_t cs = ctx->side_streams[k];
        TRYCUDA(cudaStreamWaitEvent(cs, ev_setup, 0));
        if (h2d_event) TRYCUDA(cudaStreamWaitEvent(cs, ctx->side_events[k], 0));
        ctx->stream = cs;
        rc = launch_bidir_ctc(ctx, lat, status_dev, zparts_dev, boff_dev, g_dev, per, b0, nb, /*zero_w=*/1, bidir_scores_dev, blank, direct ? small_mapped : small_dev,
                               (direct ? small_mapped : small_dev) + tot_t, direct ? meta_mapped : nullptr);
        ctx->stream = main_stream;
        if (rc) goto done;
        if (grads && !grads_on_device)
          TRYCUDA(cudaMemcpyAsync(grads + (long long)b0 * per, g_dev + (long long)b0 * per,
                                  sizeof(float) * per * nb, cudaMemcpyDeviceToHost, cs));
        TRYCUDA(cudaEventRecord(ctx->side_events[k], cs));
        TRYCUDA(cudaStreamWaitEvent(main_stream, ctx->side_events[k], 0));
      }
    } else if (K == 1 && !h2d_event && !(grads && !grads_on_device)) {
      // forwardScore(emissions) and its +1 gradient beside the forward sweep
      TRYCUDA(cudaStreamWaitEvent(ctx->copy_stream, ev_setup, 0));
      ctx->stream = ctx->copy_stream;
      rc = launch_linear_forward(ctx, B, T_dev, maxT, C, e_dev, per, 0, z_dev, g_dev, per, nullptr, 1.0f,
                                 input_lens ? 0 : 1, row_scratch);
      ctx->stream = main_stream;
      if (rc) goto done;
      TRYCUDA(cudaEventRecord(ev_lin, ctx->copy_stream));
      TRY(sweep_forward(0, -1));
      TRYCUDA(cudaStreamWaitEvent(main_stream, ev_lin, 0));
      if (grads) TRY(sweep_backward(0, -1));
    } else {
      for (int k = 0; k < K && !rc; k++) {
        const int b0 = chunk_lo[k], nb = chunk_lo[k + 1] - chunk_lo[k];
        cudaStream_t cs = ctx->side_streams[k];
        TRYCUDA(cudaStreamWaitEvent(cs, ev_setup, 0));
        if (h2d_event) TRYCUDA(cudaStreamWaitEvent(cs, ctx->side_events[k], 0));
        ctx->stream = cs;
        rc = launch_linear_forward(ctx, nb, T_dev + b0, maxT, C, e_dev + (long long)b0 * per, per, 0,
                                   z_dev + b0, g_dev ? g_dev + (long long)b0 * per : nullptr, per, nullptr,
                                   1.0f, input_lens ? 0 : 1, row_scratch + (long long)b0 * std::max(maxT, 1));
        if (!rc) rc = sweep_forward(b0, nb);
        if (!rc && grads) rc = sweep_backward(b0, nb);
        ctx->stream = main_stream;
        if (rc) goto done;
        if (grads && !grads_on_device)
          TRYCUDA(cudaMemcpyAsync(grads + (long long)b0 * per, g_dev + (long long)b0 * per,
                                  sizeof(float) * per * nb, cudaMemcpyDeviceToHost, cs));
        TRYCUDA(cudaEventRecord(ctx->side_events[k], cs));
        TRYCUDA(cudaStreamWaitEvent(main_stream, ctx->side_events[k], 0));
      }
    }
  } else {
    TRY(launch_compose(ctx, lat, h2d_event));
    // forwardScore(emissions) and its +1 gradient
    TRY(launch_linear_forward(ctx, B, small_dev + tot_t + 2ll * B, maxT, C, e_dev, per, 0, z_dev, g_dev,
                              per, nullptr, 1.0f, input_lens ? 0 : 1));
    TRY(launch_forward(ctx, lat, MODE_LOG));
    lat->forward_done = true;
    lat->forward_mode = MODE_LOG;
  }
  if (grads && !implicit) {
    // shortestDistanceGrad and compose's gradFunc fused when the lattice qualifies
    rc = launch_backward_fused(ctx, lat, deltas_dev, g_dev, per);
    if (rc == GTNB_ERR_UNSUPPORTED) {
      if (!lat->arc_grad) TRY(dev_alloc(ctx, &lat->arc_grad, lat->tot_A));
      TRY(launch_backward(ctx, lat, 0, deltas_dev));
      TRY(launch_compose_grad(ctx, lat, nullptr, g_dev, per));
    } else if (rc) {
      goto done;
    }
    if (!grads_on_device)
      TRYCUDA(cudaMemcpyAsync(grads, g_dev, sizeof(float) * per * B, cudaMemcpyDeviceToHost, ctx->stream));
  }
  pc.mark("launches");
  zp = bidir ? 2 * bidir_zparts() : 1; // partial sums of forwardScore(emissions) per utterance
  TRY(readback_reserve(ctx, (zp + 2) * sizeof(float) * B));
  {
    float* z = reinterpret_cast<float*>(ctx->readback);
    float* s = z + (long long)zp * B;
    int32_t* st = reinterpret_cast<int32_t*>(s + B);
    if (bidir && direct) {
      // the kernel wrote straight into this block
    } else if (bidir) { // one copy: the block is laid out like the host buffer
      TRYCUDA(cudaMemcpyAsync(z, zparts_dev, sizeof(float) * (zp + 2) * B, cudaMemcpyDeviceToHost, ctx->stream));
    } else {
      TRYCUDA(cudaMemcpyAsync(z, z_dev, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
      TRYCUDA(cudaMemcpyAsync(s, lat->out_scores, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
      if (implicit)
        TRYCUDA(cudaMemcpyAsync(st, status_dev, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, ctx->stream));
    }
    pc.mark("readback enqueue");
    TRYCUDA(cudaStreamSynchronize(ctx->stream));
    pc.mark("sync");
    for (int b = 0; b < B; b++) { // subtract, functions.cpp:52
      float zb = 0.0f;
      for (int k = 0; k < zp; k++) zb += z[(long long)zp * b + k];
      losses_host[b] = zb - s[b];
    }
    if (implicit)
      for (int b = 0; b < B; b++)
        if (st[b]) *needs_exact = true;
  }

done:
  ctx->stream = main_stream;
  if (rc && implicit) {
    // an error mid-way: nothing may still be running on the side streams when the buffers go
    cudaStreamSynchronize(ctx->copy_stream);
    for (int k = 0; k < K && k < (int)ctx->side_streams.size(); k++) cudaStreamSynchronize(ctx->side_streams[k]);
  }
  if (!bidir) dev_free(ctx, status_dev); // (bidir: part of the zparts block)
  dev_free(ctx, row_scratch);
  if (!direct) dev_free(ctx, zparts_dev);
  dev_free(ctx, boff_dev);
  if (lat) gtnb_lattice_destroy(ctx, lat);
  if (!emissions_on_device) dev_free(ctx, e_dev);
  if (grads && !grads_on_device) dev_free(ctx, g_dev);
  dev_free(ctx, z_dev);
  dev_free(ctx, deltas_dev);
  dev_free(ctx, small_dev);
  return rc;
#undef TRY
#undef TRYCUDA
}

extern "C" int gtnb_ctc_loss(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
    const int32_t* input_lens, const int32_t* targets, const int32_t* target_lens, int blank,
    float* losses_host, float* grads, int grads_on_device) {
  bool needs_exact = false;
  if (ctx) arena_begin(ctx);
  int rc = ctc_loss_run(ctx, B, T, C, emissions, emissions_on_device, input_lens, targets, target_lens, blank,
                        losses_host, grads, grads_on_device, ctx && ctx->use_implicit, &needs_exact);
  if (ctx) arena_end(ctx);
  if (rc == GTNB_OK && needs_exact)
    // a non-finite emission: the materialised lattice reproduces the reference's inf / NaN
    // propagation arc by arc (shortest.cpp:62-80), the implicit sweep cannot tell a missing
    // node from one whose score is -inf
    rc = ctc_loss_run(ctx, B, T, C, emissions, emissions_on_device, input_lens, targets, target_lens, blank,
                      losses_host, grads, grads_on_device, false, &needs_exact);
  return rc;
}

/*
 * viterbiPath(compose(linearGraph(T, C; e_b), transitions)) for a whole minibatch, with the
 * dense transitions graph of test/criterion_test.cpp:244-254 / :316-326, through the
 * factored kernel (k_dense.cu): the T*C*C lattice is never materialised.
 */
static int viterbi_dense_run(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
    const int32_t* input_lens, const float* trans_w_host, int32_t* paths_host, float* scores_host) {
  if (!ctx || B < 0 || T < 0 || C <= 0 || !emissions || !trans_w_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_viterbi_dense: bad arguments");
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  const long long per = (long long)T * C;
  int rc = GTNB_OK;
  float *e_dev = nullptr, *tr_dev = nullptr, *sc_dev = nullptr;
  int32_t *T_dev = nullptr, *paths_dev = nullptr;
  uint8_t* bp = nullptr;
#define TRY(x)                 \
  do {                         \
    if ((rc = (x))) goto done; \
  } while (0)
#define TRYCUDA(call)                                      \
  do {                                                     \
    cudaError_t e__ = (call);                              \
    if (e__ != cudaSuccess) {                              \
      rc = cuda_fail(ctx, e__, #call, __FILE__, __LINE__); \
      goto done;                                           \
    }                                                      \
  } while (0)
  if (input_lens)
    for (int b = 0; b < B; b++)
      if (input_lens[b] < 0 || input_lens[b] > T)
        return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_viterbi_dense: input_lens out of range");
  if (emissions_on_device) {
    e_dev = const_cast<float*>(emissions);
  } else {
    TRY(dev_alloc(ctx, &e_dev, per * B));
    TRYCUDA(cudaMemcpyAsync(e_dev, emissions, sizeof(float) * per * B, cudaMemcpyHostToDevice, ctx->stream));
  }
  TRY(dev_alloc(ctx, &tr_dev, (long long)C + (long long)C * C));
  TRY(dev_alloc(ctx, &sc_dev, B));
  TRY(dev_alloc(ctx, &paths_dev, (long long)B * std::max(T, 1)));
  TRY(dev_alloc(ctx, &bp, (long long)B * std::max(T, 1) * C));
  if (input_lens) TRY(dev_alloc(ctx, &T_dev, B));
  TRY(stage_begin(ctx));
  TRY(stage_upload(ctx, tr_dev, trans_w_host, sizeof(float) * ((size_t)C + (size_t)C * C)));
  if (input_lens) TRY(stage_upload(ctx, T_dev, input_lens, sizeof(int32_t) * B));
  TRY(stage_end(ctx));
  TRY(launch_viterbi_dense(ctx, B, T, C, T_dev, e_dev, per, tr_dev, bp, paths_dev, sc_dev));
  if (paths_host && T > 0)
    TRYCUDA(cudaMemcpyAsync(paths_host, paths_dev, sizeof(int32_t) * (size_t)B * T, cudaMemcpyDeviceToHost, ctx->stream));
  if (scores_host)
    TRYCUDA(cudaMemcpyAsync(scores_host, sc_dev, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
  TRYCUDA(cudaStreamSynchronize(ctx->stream));
done:
  if (!emissions_on_device) dev_free(ctx, e_dev);
  dev_free(ctx, tr_dev);
  dev_free(ctx, sc_dev);
  dev_free(ctx, paths_dev);
  dev_free(ctx, bp);
  dev_free(ctx, T_dev);
  return rc;
#undef TRY
#undef TRYCUDA
}

/* (the device scratch of a call comes from the context's call-scoped arena, as in gtnb_ctc_loss: no stream-ordered
 * allocations on the path after the first call of a shape) */
extern "C" int gtnb_viterbi_dense(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
    const int32_t* input_lens, const float* trans_w_host, int32_t* paths_host, float* scores_host) {
  if (ctx) arena_begin(ctx);
  const int rc = viterbi_dense_run(ctx, B, T, C, emissions, emissions_on_device, input_lens, trans_w_host, paths_host,
                                   scores_host);
  if (ctx) arena_end(ctx);
  return rc;
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
 * grads beyond T_b are zeroed.
 */
static int asg_loss_call(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
    const int32_t* input_lens, const float* trans_w_host, const int32_t* targets, const int32_t* target_lens,
    float* losses_host, float* grads, int grads_on_device, float* trans_grad_host);

static int asg_loss_run(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
    const int32_t* input_lens, const float* trans_w_host, const int32_t* targets, const int32_t* target_lens,
    float* losses_host, float* grads, int grads_on_device, float* trans_grad_host) {
  if (!ctx || B < 0 || T < 0 || C <= 0 || !emissions || !trans_w_host || !target_lens || !losses_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss: bad arguments");
  if (B == 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  const long long per = (long long)T * C;
  const int nTrans = C + C * C;
  const bool want = grads || trans_grad_host;
  int rc = GTNB_OK;
  float *e_dev = nullptr, *g_dev = nullptr, *tg_dev = nullptr, *ft_grad = nullptr, *minus1 = nullptr;
  int32_t* ft_map_dev = nullptr;
  int32_t* status_dev = nullptr;
  bool implicit = false, needs_exact = false;
  gtnb_lattice *den = nullptr, *num = nullptr;
  cudaStream_t asg_main = ctx->stream;

  // transitions graph view (criterion_test.cpp:244-254)
  std::vector<uint8_t> tflags(C + 1, 2);
  tflags[0] = 1;
  std::vector<int32_t> tsrc(nTrans), tdst(nTrans), tlab(nTrans);
  for (int i = 0; i < C; i++) {
    tsrc[i] = 0;
    tdst[i] = i + 1;
    tlab[i] = i;
  }
  for (int i = 0; i < C; i++)
    for (int j = 0; j < C; j++) {
      const int a = C + i * C + j;
      tsrc[a] = j + 1;
      tdst[a] = i + 1;
      tlab[a] = i;
    }
  gtnb_graph_view tview;
  std::memset(&tview, 0, sizeof(tview));
  tview.num_nodes = C + 1;
  tview.num_arcs = nTrans;
  tview.node_flags = tflags.data();
  tview.arc_src = tsrc.data();
  tview.arc_dst = tdst.data();
  tview.arc_ilabel = tview.arc_olabel = tlab.data();
  tview.weights = trans_w_host;

  // compose(fal_b, transitions): node l = "l labels consumed"; arcs: 0->1, then per node a
  // self loop and the step to the next label, in the reference's creation order
  struct Ft {
    std::vector<uint8_t> flags;
    std::vector<int32_t> src, dst, lab, map;
    std::vector<float> w;
  };
  std::vector<Ft> ft(B);
  std::vector<gtnb_graph_view> fviews(B);
  std::vector<int32_t> ft_map;
  std::vector<int32_t> Tb(B, T);
  if (input_lens) std::copy(input_lens, input_lens + B, Tb.begin());
  long long toff = 0;
  for (int b = 0; b < B; b++) {
    const int U = target_lens[b];
    if (U < 0) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss: negative target length");
    const int32_t* y = targets + toff;
    toff += U;
    for (int u = 0; u < U; u++)
      if (y[u] < 0 || y[u] >= C) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss: label out of range");
    Ft& f = ft[b];
    f.flags.assign(U + 1, 0);
    f.flags[0] |= 1;
    if (U > 0) f.flags[U] |= 2;
    auto add = [&](int s, int d, int lab, int tarc) {
      f.src.push_back(s);
      f.dst.push_back(d);
      f.lab.push_back(lab);
      f.w.push_back(trans_w_host[tarc]);
      f.map.push_back(tarc);
    };
    if (U > 0) add(0, 1, y[0], y[0]);
    for (int l = 1; l <= U; l++) {
      add(l, l, y[l - 1], C + y[l - 1] * C + y[l - 1]);
      if (l < U) add(l, l + 1, y[l], C + y[l] * C + y[l - 1]);
    }
    gtnb_graph_view& v = fviews[b];
    std::memset(&v, 0, sizeof(v));
    v.num_nodes = U + 1;
    v.num_arcs = (int)f.src.size();
    v.node_flags = f.flags.data();
    v.arc_src = f.src.data();
    v.arc_dst = f.dst.data();
    v.arc_ilabel = v.arc_olabel = f.lab.data();
    v.weights = f.w.data();
    ft_map.insert(ft_map.end(), f.map.begin(), f.map.end());
  }
  const long long nFt = (long long)ft_map.size();

#define TRY(x)                 \
  do {                         \
    if ((rc = (x))) goto done; \
  } while (0)
#define TRYCUDA(call)                                      \
  do {                                                     \
    cudaError_t e__ = (call);                              \
    if (e__ != cudaSuccess) {                              \
      rc = cuda_fail(ctx, e__, #call, __FILE__, __LINE__); \
      goto done;                                           \
    }                                                      \
  } while (0)
  if (emissions_on_device) {
    e_dev = const_cast<float*>(emissions);
  } else {
    TRY(dev_alloc(ctx, &e_dev, per * B));
    TRYCUDA(cudaMemcpyAsync(e_dev, emissions, sizeof(float) * per * B, cudaMemcpyHostToDevice, ctx->stream));
  }
  if (want) {
    if (grads && grads_on_device)
      g_dev = grads;
    else
      TRY(dev_alloc(ctx, &g_dev, per * B));
    TRYCUDA(cudaMemsetAsync(g_dev, 0, sizeof(float) * per * B, ctx->stream));
    TRY(dev_alloc(ctx, &tg_dev, nTrans));
    TRYCUDA(cudaMemsetAsync(tg_dev, 0, sizeof(float) * nTrans, ctx->stream));
    TRY(dev_alloc(ctx, &ft_grad, std::max<long long>(nFt, 1)));
    TRYCUDA(cudaMemsetAsync(ft_grad, 0, sizeof(float) * std::max<long long>(nFt, 1), ctx->stream));
    TRY(dev_alloc(ctx, &ft_map_dev, std::max<long long>(nFt, 1)));
    TRY(dev_alloc(ctx, &minus1, B));
  }
  // implicit sweeps (k_implicit.cu): neither lattice is built; the dense transitions graph takes
  // the G-lanes-per-node kernels, the forced-alignment chains the one-node-per-thread kernels
  implicit = ctx->use_implicit;
  if (implicit) {
    rc = compose_linear_impl(ctx, B, &tview, 1, 1, Tb.data(), C, e_dev, per, true, &den);
    if (!rc) rc = compose_linear_impl(ctx, B, fviews.data(), B, 0, Tb.data(), C, e_dev, per, true, &num);
    if (rc == GTNB_ERR_UNSUPPORTED) {
      if (den) gtnb_lattice_destroy(ctx, den);
      den = nullptr;
      implicit = false;
      rc = GTNB_OK;
    } else if (rc) {
      goto done;
    }
  }
  if (implicit) {
    TRY(ensure_side_streams(ctx, 0, 0));
    TRY(dev_alloc(ctx, &status_dev, 2ll * B));
    TRYCUDA(cudaMemsetAsync(status_dev, 0, sizeof(int32_t) * 2 * B, ctx->stream));
    // the numerator's sweeps (forced-alignment chains: small) run on the second stream beside the
    // denominator's (dense transitions: wide); they share nothing but the emission gradient, which both
    // accumulate with red.global.add
    TRYCUDA(cudaEventRecord(ctx->ev_fork, ctx->stream));
    TRYCUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_fork, 0));
    TRY(launch_implicit_forward(ctx, den, status_dev));
    ctx->stream = ctx->copy_stream;
    rc = launch_implicit_forward(ctx, num, status_dev + B);
    ctx->stream = asg_main;
    if (rc) goto done;
  } else {
    TRY(gtnb_compose_linear(ctx, B, &tview, 1, 1, Tb.data(), C, e_dev, per, &den));
    TRY(gtnb_compose_linear(ctx, B, fviews.data(), B, 0, Tb.data(), C, e_dev, per, &num));
    TRY(gtnb_forward(ctx, den, 0, nullptr, nullptr));
    TRY(gtnb_forward(ctx, num, 0, nullptr, nullptr));
  }
  if (want) {
    std::vector<float> m1(B, -1.0f);
    if (implicit) {
      TRY(stage_begin(ctx));
      TRY(stage_upload(ctx, minus1, m1.data(), sizeof(float) * B));
      TRY(stage_end(ctx));
      // +1 / -1: subtract's gradFunc (functions.cpp:53-58); graph-side gradients straight into
      // the transitions' (shared by the batch) and the forced-alignment chains' slabs
      TRYCUDA(cudaEventRecord(ctx->ev_fork, ctx->stream)); // the staged -1 seeds
      TRYCUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_fork, 0));
      TRY(launch_implicit_backward(ctx, den, nullptr, g_dev, per, 0, -1, tg_dev));
      ctx->stream = ctx->copy_stream;
      rc = launch_implicit_backward(ctx, num, minus1, g_dev, per, 0, -1, ft_grad);
      ctx->stream = asg_main;
      if (rc) goto done;
    } else {
      TRY(gtnb_backward(ctx, den, 0, nullptr)); // +1 (subtract's gradFunc, functions.cpp:53-58)
      TRY(gtnb_backward(ctx, num, 0, m1.data())); // -1
      TRY(gtnb_compose_grad(ctx, den, tg_dev, g_dev, per));
      TRY(gtnb_compose_grad(ctx, num, ft_grad, g_dev, per));
    }
    if (implicit) { // join the numerator's stream
      TRYCUDA(cudaEventRecord(ctx->ev_join, ctx->copy_stream));
      TRYCUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    }
    if (nFt) {
      TRY(stage_begin(ctx));
      TRY(stage_upload(ctx, ft_map_dev, ft_map.data(), sizeof(int32_t) * nFt));
      TRY(stage_end(ctx));
      TRY(launch_scatter_add(ctx, tg_dev, ft_map_dev, ft_grad, nFt));
    }
    if (grads && !grads_on_device)
      TRYCUDA(cudaMemcpyAsync(grads, g_dev, sizeof(float) * per * B, cudaMemcpyDeviceToHost, ctx->stream));
    if (trans_grad_host)
      TRYCUDA(cudaMemcpyAsync(trans_grad_host, tg_dev, sizeof(float) * nTrans, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (implicit && !want) { // loss only: the numerator's forward sweep is still on the second stream
    TRYCUDA(cudaEventRecord(ctx->ev_join, ctx->copy_stream));
    TRYCUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
  }
  TRY(readback_reserve(ctx, 4 * sizeof(float) * B));
  {
    float* d = reinterpret_cast<float*>(ctx->readback);
    float* n = d + B;
    int32_t* st = reinterpret_cast<int32_t*>(n + B);
    TRYCUDA(cudaMemcpyAsync(d, den->out_scores, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaMemcpyAsync(n, num->out_scores, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    if (implicit)
      TRYCUDA(cudaMemcpyAsync(st, status_dev, sizeof(int32_t) * 2 * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaStreamSynchronize(ctx->stream));
    for (int b = 0; b < B; b++) losses_host[b] = d[b] - n[b];
    if (implicit)
      for (int b = 0; b < 2 * B; b++) needs_exact |= st[b] != 0;
  }
done:
  dev_free(ctx, status_dev);
  if (den) gtnb_lattice_destroy(ctx, den);
  if (num) gtnb_lattice_destroy(ctx, num);
  if (!emissions_on_device) dev_free(ctx, e_dev);
  if (!(grads && grads_on_device)) dev_free(ctx, g_dev);
  dev_free(ctx, tg_dev);
  dev_free(ctx, ft_grad);
  dev_free(ctx, ft_map_dev);
  dev_free(ctx, minus1);
  if (rc == GTNB_OK && needs_exact) {
    // a non-finite weight: repeat through the materialised lattices, which reproduce the
    // reference's inf / NaN propagation arc by arc
    ctx->use_implicit = false;
    rc = asg_loss_call(ctx, B, T, C, emissions, emissions_on_device, input_lens, trans_w_host, targets, target_lens,
                       losses_host, grads, grads_on_device, trans_grad_host);
    ctx->use_implicit = true;
  }
  return rc;
#undef TRY
#undef TRYCUDA
}

static int asg_loss_call(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
    const int32_t* input_lens, const float* trans_w_host, const int32_t* targets, const int32_t* target_lens,
    float* losses_host, float* grads, int grads_on_device, float* trans_grad_host) {
  if (ctx) arena_begin(ctx);
  const int rc = asg_loss_run(ctx, B, T, C, emissions, emissions_on_device, input_lens, trans_w_host, targets,
                              target_lens, losses_host, grads, grads_on_device, trans_grad_host);
  if (ctx) arena_end(ctx);
  return rc;
}

extern "C" int gtnb_asg_loss(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device,
    const float* trans_w_host, const int32_t* targets, const int32_t* target_lens,
    float* losses_host, float* grads, int grads_on_device, float* trans_grad_host) {
  return asg_loss_call(ctx, B, T, C, emissions, emissions_on_device, nullptr, trans_w_host, targets, target_lens,
                       losses_host, grads, grads_on_device, trans_grad_host);
}

/*
 * CTC with a learned bigram transition graph G (benchmarks/ctc.cpp:107-134, k_ngram.cu):
 *   loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(ctc_b, G), E_b))
 * G: C nodes, all start and accept, arc j -> i with label i and weight W[i*C + j].
 */
namespace {

struct NgramArgs {
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

#define TRY(x)                 \
  do {                         \
    if ((rc = (x))) goto done; \
  } while (0)
#define TRYCUDA(call)                                      \
  do {                                                     \
    cudaError_t e__ = (call);                              \
    if (e__ != cudaSuccess) {                              \
      rc = cuda_fail(ctx, e__, #call, __FILE__, __LINE__); \
      goto done;                                           \
    }                                                      \
  } while (0)

/* the gradients' destinations: emission rows zeroed (every row is written), W's gradient copied out */
int ngram_copy_out(gtnb_ctx* ctx, const NgramArgs& a, const float* tg_dev) {
  if (a.trans_grad)
    GTNB_CUDA(ctx, cudaMemcpyAsync(a.trans_grad, tg_dev, sizeof(float) * a.C * a.C,
                                   a.trans_grad_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                                   ctx->stream));
  return GTNB_OK;
}

/*
 * Materialised lattices, graph by graph as the reference composes them: intersect(E_b, G) and
 * intersect(P_b, E_b), where P_b = intersect(ctc_b, G) is built on the host WITHOUT the fold (C start states
 * (0, s), then (l, label(l))).  Reproduces the reference's inf / NaN propagation arc by arc; the path for
 * non-finite weights.
 */
int ngram_ctc_loss_exact(gtnb_ctx* ctx, const NgramArgs& a, const std::vector<int32_t>& Tb) {
  const int B = a.B, T = a.T, C = a.C;
  const long long per = (long long)T * C, CC = (long long)C * C;
  const bool want = a.grads || a.trans_grad;
  int rc = GTNB_OK;
  float *e_dev = nullptr, *g_dev = nullptr, *tg_dev = nullptr, *ft_grad = nullptr, *gg_grad = nullptr;
  int32_t *ft_map_dev = nullptr, *gg_map_dev = nullptr;
  gtnb_lattice *den = nullptr, *num = nullptr;
  std::vector<float> W(CC);
  // G (benchmarks/ctc.cpp transitionsGraph with a label-determined destination): arc j*C + i = j -> i
  std::vector<uint8_t> gflags(C, 3);
  std::vector<int32_t> gsrc(CC), gdst(CC), glab(CC), gmap(CC);
  std::vector<float> gw(CC);
  struct P {
    std::vector<uint8_t> flags;
    std::vector<int32_t> src, dst, lab;
    std::vector<float> w;
  };
  std::vector<P> pg(B);
  std::vector<gtnb_graph_view> pviews(B);
  std::vector<int32_t> pmap;
  gtnb_graph_view gview;
  std::memset(&gview, 0, sizeof(gview));

  if (a.trans_on_device)
    GTNB_CUDA(ctx, cudaMemcpy(W.data(), a.trans_w, sizeof(float) * CC, cudaMemcpyDeviceToHost));
  else
    std::memcpy(W.data(), a.trans_w, sizeof(float) * CC);
  for (int j = 0; j < C; j++)
    for (int i = 0; i < C; i++) {
      const long long k = (long long)j * C + i;
      gsrc[k] = j;
      gdst[k] = i;
      glab[k] = i;
      gw[k] = W[(long long)i * C + j];
      gmap[k] = i * C + j;
    }
  gview.num_nodes = C;
  gview.num_arcs = (int)CC;
  gview.node_flags = gflags.data();
  gview.arc_src = gsrc.data();
  gview.arc_dst = gdst.data();
  gview.arc_ilabel = gview.arc_olabel = glab.data();
  gview.weights = gw.data();
  {
    long long toff = 0;
    for (int b = 0; b < B; b++) {
      const int U = a.target_lens[b], L = 2 * U + 1;
      const int32_t* y = a.targets + toff;
      toff += U;
      auto lab = [&](int l) { return (l & 1) ? y[(l - 1) / 2] : a.blank; };
      // node of CTC node l: (0, blank) for l = 0, C + l - 1 otherwise; nodes [0, C) are the start states (0, s)
      auto node = [&](int l) { return l == 0 ? a.blank : C + l - 1; };
      P& p = pg[b];
      p.flags.assign(C + L - 1, 0);
      for (int s = 0; s < C; s++) p.flags[s] = 1 | (L == 1 ? 2 : 0);
      for (int l = std::max(1, L - 2); l < L; l++) p.flags[node(l)] |= 2;
      auto arc = [&](int ls, int l) { // every arc of ctc_b (ls -> l) times the matching arcs of G
        const int i = lab(l);
        if (ls == 0) {
          for (int s = 0; s < C; s++) {
            p.src.push_back(s), p.dst.push_back(node(l)), p.lab.push_back(i);
            p.w.push_back(W[(long long)i * C + s]), pmap.push_back(i * C + s);
          }
        } else {
          p.src.push_back(node(ls)), p.dst.push_back(node(l)), p.lab.push_back(i);
          p.w.push_back(W[(long long)i * C + lab(ls)]), pmap.push_back(i * C + lab(ls));
        }
      };
      for (int l = 0; l < L; l++) {
        arc(l, l);
        if (l > 0) arc(l - 1, l);
        if ((l & 1) && l > 1 && lab(l) != lab(l - 2)) arc(l - 2, l);
      }
      gtnb_graph_view& v = pviews[b];
      std::memset(&v, 0, sizeof(v));
      v.num_nodes = (int)p.flags.size();
      v.num_arcs = (int)p.src.size();
      v.node_flags = p.flags.data();
      v.arc_src = p.src.data();
      v.arc_dst = p.dst.data();
      v.arc_ilabel = v.arc_olabel = p.lab.data();
      v.weights = p.w.data();
    }
  }
  {
    const long long nP = (long long)pmap.size();
    if (a.emissions_on_device) {
      e_dev = const_cast<float*>(a.emissions);
    } else {
      TRY(dev_alloc(ctx, &e_dev, per * B));
      TRYCUDA(cudaMemcpyAsync(e_dev, a.emissions, sizeof(float) * per * B, cudaMemcpyHostToDevice, ctx->stream));
    }
    TRY(gtnb_compose_linear(ctx, B, &gview, 1, 1, Tb.data(), C, e_dev, per, &den));
    TRY(gtnb_compose_linear(ctx, B, pviews.data(), B, 0, Tb.data(), C, e_dev, per, &num));
    TRY(gtnb_forward(ctx, den, 0, nullptr, nullptr));
    TRY(gtnb_forward(ctx, num, 0, nullptr, nullptr));
    if (want) {
      if (a.grads && a.grads_on_device)
        g_dev = a.grads;
      else
        TRY(dev_alloc(ctx, &g_dev, per * B));
      TRYCUDA(cudaMemsetAsync(g_dev, 0, sizeof(float) * per * B, ctx->stream));
      TRY(dev_alloc(ctx, &tg_dev, CC));
      TRY(dev_alloc(ctx, &gg_grad, CC));
      TRY(dev_alloc(ctx, &ft_grad, std::max<long long>(nP, 1)));
      TRY(dev_alloc(ctx, &gg_map_dev, CC));
      TRY(dev_alloc(ctx, &ft_map_dev, std::max<long long>(nP, 1)));
      TRYCUDA(cudaMemsetAsync(tg_dev, 0, sizeof(float) * CC, ctx->stream));
      TRYCUDA(cudaMemsetAsync(gg_grad, 0, sizeof(float) * CC, ctx->stream));
      TRYCUDA(cudaMemsetAsync(ft_grad, 0, sizeof(float) * std::max<long long>(nP, 1), ctx->stream));
      std::vector<float> m1(B, -1.0f);
      TRY(gtnb_backward(ctx, den, 0, nullptr)); // +1 / -1: subtract's gradFunc (functions.cpp:53-58)
      TRY(gtnb_backward(ctx, num, 0, m1.data()));
      TRY(gtnb_compose_grad(ctx, den, gg_grad, g_dev, per));
      TRY(gtnb_compose_grad(ctx, num, ft_grad, g_dev, per));
      TRY(stage_begin(ctx));
      TRY(stage_upload(ctx, gg_map_dev, gmap.data(), sizeof(int32_t) * CC));
      if (nP) TRY(stage_upload(ctx, ft_map_dev, pmap.data(), sizeof(int32_t) * nP));
      TRY(stage_end(ctx));
      TRY(launch_scatter_add(ctx, tg_dev, gg_map_dev, gg_grad, CC));
      TRY(launch_scatter_add(ctx, tg_dev, ft_map_dev, ft_grad, nP));
      if (a.grads && !a.grads_on_device)
        TRYCUDA(cudaMemcpyAsync(a.grads, g_dev, sizeof(float) * per * B, cudaMemcpyDeviceToHost, ctx->stream));
      TRY(ngram_copy_out(ctx, a, tg_dev));
    }
    TRY(readback_reserve(ctx, 2 * sizeof(float) * B));
    float* d = reinterpret_cast<float*>(ctx->readback);
    float* n = d + B;
    TRYCUDA(cudaMemcpyAsync(d, den->out_scores, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaMemcpyAsync(n, num->out_scores, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaStreamSynchronize(ctx->stream));
    for (int b = 0; b < B; b++) a.losses_host[b] = d[b] - n[b];
  }
done:
  if (den) gtnb_lattice_destroy(ctx, den);
  if (num) gtnb_lattice_destroy(ctx, num);
  if (!a.emissions_on_device) dev_free(ctx, e_dev);
  if (!(a.grads && a.grads_on_device)) dev_free(ctx, g_dev);
  dev_free(ctx, tg_dev);
  dev_free(ctx, gg_grad);
  dev_free(ctx, ft_grad);
  dev_free(ctx, gg_map_dev);
  dev_free(ctx, ft_map_dev);
  return rc;
}

/*
 * The device path (k_ngram.cu): the folded numerator graphs built on the device from the targets and W, swept by
 * k_implicit.cu on the second stream; the dense trellis of the denominator on the context's stream.  Both add
 * their emission gradients into the zero-filled rows with red.add.  *needs_exact: a non-finite weight was met.
 */
int ngram_ctc_loss_fast(gtnb_ctx* ctx, const NgramArgs& a, const std::vector<int32_t>& Tb,
                        const std::vector<SgDims>& dims, const std::vector<int32_t>& off, bool* needs_exact) {
  const int B = a.B, T = a.T, C = a.C;
  const long long per = (long long)T * C, CC = (long long)C * C;
  const bool want = a.grads || a.trans_grad;
  long long tot_t = 0, tot_A = 0;
  for (int b = 0; b < B; b++) {
    tot_t += a.target_lens[b];
    tot_A += dims[b].A;
  }
  int rc = GTNB_OK;
  float *e_dev = nullptr, *g_dev = nullptr, *w_dev = nullptr, *tg_dev = nullptr, *sigma = nullptr;
  float *alpha = nullptr, *den = nullptr, *ggrad = nullptr, *minus1 = nullptr;
  int32_t *small_dev = nullptr, *status = nullptr, *map = nullptr;
  gtnb_lattice* lat = nullptr;
  cudaStream_t main_stream = ctx->stream;
  std::vector<long long> sgn, sga;
  std::vector<int32_t> small_h((size_t)(tot_t + 3ll * B));
  std::vector<float> m1(B, -1.0f);
  if (tot_t) std::memcpy(small_h.data(), a.targets, sizeof(int32_t) * tot_t);
  std::memcpy(small_h.data() + tot_t, off.data(), sizeof(int32_t) * B);
  std::memcpy(small_h.data() + tot_t + B, a.target_lens, sizeof(int32_t) * B);
  std::memcpy(small_h.data() + tot_t + 2ll * B, Tb.data(), sizeof(int32_t) * B);

  TRY(ensure_side_streams(ctx, 0, 0));
  if (a.emissions_on_device) {
    e_dev = const_cast<float*>(a.emissions);
  } else {
    TRY(dev_alloc(ctx, &e_dev, per * B));
    TRYCUDA(cudaMemcpyAsync(e_dev, a.emissions, sizeof(float) * per * B, cudaMemcpyHostToDevice, ctx->stream));
  }
  if (a.trans_on_device)
    w_dev = const_cast<float*>(a.trans_w);
  else
    TRY(dev_alloc(ctx, &w_dev, CC));
  TRY(dev_alloc(ctx, &small_dev, (long long)small_h.size()));
  TRY(dev_alloc(ctx, &status, 2ll * B));
  TRY(dev_alloc(ctx, &sigma, C));
  TRY(dev_alloc(ctx, &alpha, (long long)B * (T + 1) * C));
  TRY(dev_alloc(ctx, &den, B));
  TRY(dev_alloc(ctx, &map, tot_A));
  TRY(composed_alloc(ctx, B, dims.data(), B, 0, Tb.data(), C, e_dev, per, sgn, sga, &lat, true));
  if (want) {
    if (a.grads && a.grads_on_device)
      g_dev = a.grads;
    else
      TRY(dev_alloc(ctx, &g_dev, per * B));
    TRY(dev_alloc(ctx, &tg_dev, CC + C)); // [d/dW | d/dsigma]
    TRY(dev_alloc(ctx, &ggrad, tot_A));
    TRY(dev_alloc(ctx, &minus1, B));
    TRYCUDA(cudaMemsetAsync(g_dev, 0, sizeof(float) * per * B, ctx->stream));
    TRYCUDA(cudaMemsetAsync(tg_dev, 0, sizeof(float) * (CC + C), ctx->stream));
    TRYCUDA(cudaMemsetAsync(ggrad, 0, sizeof(float) * tot_A, ctx->stream));
  }
  TRYCUDA(cudaMemsetAsync(status, 0, sizeof(int32_t) * 2 * B, ctx->stream));
  // one pinned staging pass: descriptors, [targets | offsets | lens | T], W from the host, the -1 seeds
  TRY(stage_begin(ctx));
  TRY(stage_upload(ctx, lat->meta, lat->meta_h.data(), sizeof(GraphMeta) * B));
  TRY(stage_upload(ctx, small_dev, small_h.data(), sizeof(int32_t) * small_h.size()));
  if (!a.trans_on_device) TRY(stage_upload(ctx, w_dev, a.trans_w, sizeof(float) * CC));
  if (want) TRY(stage_upload(ctx, minus1, m1.data(), sizeof(float) * B));
  TRY(stage_end(ctx));

  TRY(launch_ngram_sigma(ctx, C, w_dev, sigma));
  TRY(launch_ngram_num_build(ctx, lat, small_dev, small_dev + tot_t, small_dev + tot_t + B, a.blank, w_dev, sigma,
                             map));
  // the numerator (2U+2 nodes, <= 3 in-arcs) on the second stream beside the denominator (C^2 per frame)
  TRYCUDA(cudaEventRecord(ctx->ev_fork, ctx->stream));
  TRYCUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_fork, 0));
  ctx->stream = ctx->copy_stream;
  rc = launch_implicit_forward(ctx, lat, status + B);
  if (!rc && want) rc = launch_implicit_backward(ctx, lat, minus1, g_dev, per, 0, -1, ggrad);
  ctx->stream = main_stream;
  if (rc) goto done;
  TRY(launch_ngram_den_forward(ctx, B, T, C, small_dev + tot_t + 2ll * B, e_dev, per, w_dev, alpha, den, status));
  if (want)
    TRY(launch_ngram_den_backward(ctx, B, T, C, small_dev + tot_t + 2ll * B, e_dev, per, w_dev, alpha, den, g_dev,
                                  per, tg_dev));
  TRYCUDA(cudaEventRecord(ctx->ev_join, ctx->copy_stream));
  TRYCUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
  if (want) {
    TRY(launch_scatter_add(ctx, tg_dev, map, ggrad, tot_A)); // numerator arcs -> W entries and sigma slots
    TRY(launch_ngram_fold(ctx, C, w_dev, sigma, tg_dev));
    if (a.grads && !a.grads_on_device)
      TRYCUDA(cudaMemcpyAsync(a.grads, g_dev, sizeof(float) * per * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRY(ngram_copy_out(ctx, a, tg_dev));
  }
  TRY(readback_reserve(ctx, 4 * sizeof(float) * B));
  {
    float* d = reinterpret_cast<float*>(ctx->readback);
    float* n = d + B;
    int32_t* st = reinterpret_cast<int32_t*>(n + B);
    TRYCUDA(cudaMemcpyAsync(d, den, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaMemcpyAsync(n, lat->out_scores, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaMemcpyAsync(st, status, sizeof(int32_t) * 2 * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaStreamSynchronize(ctx->stream));
    for (int b = 0; b < B; b++) a.losses_host[b] = d[b] - n[b];
    for (int b = 0; b < 2 * B; b++) *needs_exact |= st[b] != 0;
  }
done:
  ctx->stream = main_stream;
  if (rc) cudaStreamSynchronize(ctx->copy_stream); // nothing may still run on the second stream when the buffers go
  if (lat) gtnb_lattice_destroy(ctx, lat);
  if (!a.emissions_on_device) dev_free(ctx, e_dev);
  if (!(a.grads && a.grads_on_device)) dev_free(ctx, g_dev);
  if (!a.trans_on_device) dev_free(ctx, w_dev);
  dev_free(ctx, small_dev);
  dev_free(ctx, status);
  dev_free(ctx, sigma);
  dev_free(ctx, alpha);
  dev_free(ctx, den);
  dev_free(ctx, map);
  dev_free(ctx, tg_dev);
  dev_free(ctx, ggrad);
  dev_free(ctx, minus1);
  return rc;
}

#undef TRY
#undef TRYCUDA

int ngram_ctc_loss_run(gtnb_ctx* ctx, const NgramArgs& a) {
  const int B = a.B, T = a.T, C = a.C;
  if (!ctx || B < 0 || T < 0 || C <= 0 || !a.emissions || !a.trans_w || !a.target_lens || !a.losses_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss: bad arguments");
  if (a.blank < 0 || a.blank >= C)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss: blank outside [0, C)");
  if (C > kNgramMaxLabels)
    return fail(ctx, GTNB_ERR_UNSUPPORTED,
                "gtnb_ngram_ctc_loss: C = " + std::to_string(C) + " labels; the trellis kernels hold W on chip for C <= " +
                    std::to_string(kNgramMaxLabels));
  std::vector<int32_t> Tb(B), off(B);
  std::vector<SgDims> dims(B);
  long long tot_t = 0;
  for (int b = 0; b < B; b++) {
    const int U = a.target_lens[b];
    if (U < 0) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss: negative target length");
    if (U > 0 && !a.targets) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss: targets is NULL");
    const int32_t* y = a.targets + tot_t;
    int skips = 0;
    for (int u = 0; u < U; u++) {
      if (y[u] < 0 || y[u] >= C) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss: label outside [0, C)");
      if (u > 0) skips += y[u] != y[u - 1];
    }
    off[b] = (int32_t)tot_t;
    tot_t += U;
    Tb[b] = a.input_lens ? a.input_lens[b] : T;
    if (Tb[b] < 0 || Tb[b] > T)
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_ngram_ctc_loss: input_lens outside [0, T]");
    // folded numerator graph: S + 2U+1 CTC nodes; arcs = self loops + steps + skips + the two S arcs (one if U = 0)
    const int L = 2 * U + 1;
    dims[b] = SgDims{L + 1, L + (L - 1) + skips + std::min(L, 2), L >= 2 ? 2 : 1, /*all_valid=*/1, /*uniform=*/1,
                     /*max_in=*/3, /*max_out=*/3};
  }
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  if (B == 0) { // an empty batch: the transition gradient is 0
    if (a.trans_grad) {
      if (a.trans_grad_on_device) {
        GTNB_CUDA(ctx, cudaMemsetAsync(a.trans_grad, 0, sizeof(float) * C * C, ctx->stream));
        GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
      } else {
        std::memset(a.trans_grad, 0, sizeof(float) * C * C);
      }
    }
    return GTNB_OK;
  }
  bool needs_exact = false;
  int rc = (implicit_dims_supported(dims.data(), B) && ctx->use_implicit)
               ? ngram_ctc_loss_fast(ctx, a, Tb, dims, off, &needs_exact)
               : ngram_ctc_loss_exact(ctx, a, Tb);
  if (rc == GTNB_OK && needs_exact) {
    // a non-finite weight: the materialised lattices reproduce the reference's inf / NaN propagation
    arena_end(ctx);
    arena_begin(ctx);
    rc = ngram_ctc_loss_exact(ctx, a, Tb);
  }
  // T_b = 0: linearGraph(0, C) is one start node that does not accept (creations.cpp:20-33), so both
  // intersections are empty and the reference's loss is -inf - -inf = NaN (no gradient)
  for (int b = 0; b < B && rc == GTNB_OK; b++)
    if (Tb[b] == 0) a.losses_host[b] = std::numeric_limits<float>::quiet_NaN();
  return rc;
}

} // namespace

extern "C" int gtnb_ngram_ctc_loss(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const float* trans_w, int trans_on_device, const int32_t* targets, const int32_t* target_lens, int blank,
    float* losses_host, float* grads, int grads_on_device, float* trans_grad, int trans_grad_on_device) {
  const NgramArgs a{B, T, C, emissions, emissions_on_device, input_lens, trans_w, trans_on_device, targets,
                    target_lens, blank, losses_host, grads, grads_on_device, trans_grad, trans_grad_on_device};
  if (ctx) arena_begin(ctx);
  const int rc = ngram_ctc_loss_run(ctx, a);
  if (ctx) arena_end(ctx);
  return rc;
}

/*
 * ASG with per-utterance frame counts and device-resident transitions (gtnb_asg_loss_ex):
 *   loss_b = forwardScore(compose(E_b, transitions)) - forwardScore(compose(compose(fal_b, transitions), E_b))
 * with E_b = linearGraph(T_b, C) on the first T_b rows.  For C <= 128 the denominator is k_ngram.cu's dense trellis
 * in its start mode and the numerator graphs are built on the device; otherwise (and for non-finite weights) the
 * call goes through asg_loss_run with the same T_b.
 */
namespace {

struct AsgArgs {
  int B, T, C;
  const float* emissions;
  int emissions_on_device;
  const int32_t* input_lens;
  const float* trans_w;
  int trans_on_device;
  const int32_t* targets;
  const int32_t* target_lens;
  float* losses_host;
  float* grads;
  int grads_on_device;
  float* trans_grad;
  int trans_grad_on_device;
};

#define TRY(x)                 \
  do {                         \
    if ((rc = (x))) goto done; \
  } while (0)
#define TRYCUDA(call)                                      \
  do {                                                     \
    cudaError_t e__ = (call);                              \
    if (e__ != cudaSuccess) {                              \
      rc = cuda_fail(ctx, e__, #call, __FILE__, __LINE__); \
      goto done;                                           \
    }                                                      \
  } while (0)

/*
 * The device path: the numerator graphs (U+1 nodes, two in-arcs each) built on the device from the targets and
 * trans_w and swept by k_implicit.cu on the second stream; the denominator's dense trellis in start mode on the
 * context's stream.  Both add their emission gradients into the zero-filled rows with red.add; the numerator's
 * arc gradients are scattered into trans_grad after the streams join.  *needs_exact: a non-finite weight.
 */
int asg_loss_ex_fast(gtnb_ctx* ctx, const AsgArgs& a, const std::vector<int32_t>& Tb, const std::vector<SgDims>& dims,
                     const std::vector<int32_t>& off, bool* needs_exact) {
  const int B = a.B, T = a.T, C = a.C;
  const long long per = (long long)T * C, nTrans = C + (long long)C * C;
  const bool want = a.grads || a.trans_grad;
  long long tot_t = 0, tot_A = 0;
  for (int b = 0; b < B; b++) {
    tot_t += a.target_lens[b];
    tot_A += dims[b].A;
  }
  int rc = GTNB_OK;
  float *e_dev = nullptr, *g_dev = nullptr, *w_dev = nullptr, *tg_dev = nullptr;
  float *alpha = nullptr, *den = nullptr, *ggrad = nullptr, *minus1 = nullptr;
  int32_t *small_dev = nullptr, *status = nullptr, *map = nullptr;
  gtnb_lattice* lat = nullptr;
  cudaStream_t main_stream = ctx->stream;
  std::vector<long long> sgn, sga;
  std::vector<int32_t> small_h((size_t)(tot_t + 3ll * B));
  std::vector<float> m1(B, -1.0f);
  if (tot_t) std::memcpy(small_h.data(), a.targets, sizeof(int32_t) * tot_t);
  std::memcpy(small_h.data() + tot_t, off.data(), sizeof(int32_t) * B);
  std::memcpy(small_h.data() + tot_t + B, a.target_lens, sizeof(int32_t) * B);
  std::memcpy(small_h.data() + tot_t + 2ll * B, Tb.data(), sizeof(int32_t) * B);

  TRY(ensure_side_streams(ctx, 0, 0));
  if (a.emissions_on_device) {
    e_dev = const_cast<float*>(a.emissions);
  } else {
    TRY(dev_alloc(ctx, &e_dev, per * B));
    TRYCUDA(cudaMemcpyAsync(e_dev, a.emissions, sizeof(float) * per * B, cudaMemcpyHostToDevice, ctx->stream));
  }
  if (a.trans_on_device)
    w_dev = const_cast<float*>(a.trans_w);
  else
    TRY(dev_alloc(ctx, &w_dev, nTrans));
  TRY(dev_alloc(ctx, &small_dev, (long long)small_h.size()));
  TRY(dev_alloc(ctx, &status, 2ll * B));
  TRY(dev_alloc(ctx, &alpha, asg_alpha_floats(B, T, C))); // rows and per-frame offsets
  TRY(dev_alloc(ctx, &den, B));
  TRY(dev_alloc(ctx, &map, tot_A));
  TRY(composed_alloc(ctx, B, dims.data(), B, 0, Tb.data(), C, e_dev, per, sgn, sga, &lat, true));
  if (want) {
    if (a.grads && a.grads_on_device)
      g_dev = a.grads;
    else
      TRY(dev_alloc(ctx, &g_dev, per * B));
    if (a.trans_grad && a.trans_grad_on_device)
      tg_dev = a.trans_grad;
    else
      TRY(dev_alloc(ctx, &tg_dev, nTrans));
    TRY(dev_alloc(ctx, &ggrad, tot_A));
    TRY(dev_alloc(ctx, &minus1, B));
    TRYCUDA(cudaMemsetAsync(g_dev, 0, sizeof(float) * per * B, ctx->stream));
    TRYCUDA(cudaMemsetAsync(tg_dev, 0, sizeof(float) * nTrans, ctx->stream));
    if (tot_A) TRYCUDA(cudaMemsetAsync(ggrad, 0, sizeof(float) * tot_A, ctx->stream));
  }
  TRYCUDA(cudaMemsetAsync(status, 0, sizeof(int32_t) * 2 * B, ctx->stream));
  // one pinned staging pass: descriptors, [targets | offsets | lens | T], trans_w from the host, the -1 seeds
  TRY(stage_begin(ctx));
  TRY(stage_upload(ctx, lat->meta, lat->meta_h.data(), sizeof(GraphMeta) * B));
  TRY(stage_upload(ctx, small_dev, small_h.data(), sizeof(int32_t) * small_h.size()));
  if (!a.trans_on_device) TRY(stage_upload(ctx, w_dev, a.trans_w, sizeof(float) * nTrans));
  if (want) TRY(stage_upload(ctx, minus1, m1.data(), sizeof(float) * B));
  TRY(stage_end(ctx));

  TRY(launch_asg_num_build(ctx, lat, small_dev, small_dev + tot_t, small_dev + tot_t + B, w_dev, map));
  // the numerator (U+1 nodes, <= 2 in-arcs) on the second stream beside the denominator (C^2 per frame)
  TRYCUDA(cudaEventRecord(ctx->ev_fork, ctx->stream));
  TRYCUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_fork, 0));
  ctx->stream = ctx->copy_stream;
  rc = launch_implicit_forward(ctx, lat, status + B);
  if (!rc && want) rc = launch_implicit_backward(ctx, lat, minus1, g_dev, per, 0, -1, ggrad);
  ctx->stream = main_stream;
  if (rc) goto done;
  TRY(launch_asg_den_forward(ctx, B, T, C, small_dev + tot_t + 2ll * B, e_dev, per, w_dev, alpha, den, status));
  if (want)
    TRY(launch_asg_den_backward(ctx, B, T, C, small_dev + tot_t + 2ll * B, e_dev, per, w_dev, alpha, den, g_dev, per,
                                tg_dev));
  TRYCUDA(cudaEventRecord(ctx->ev_join, ctx->copy_stream));
  TRYCUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
  if (want) {
    TRY(launch_scatter_add(ctx, tg_dev, map, ggrad, tot_A)); // numerator arcs -> start weights and matrix entries
    if (a.grads && !a.grads_on_device)
      TRYCUDA(cudaMemcpyAsync(a.grads, g_dev, sizeof(float) * per * B, cudaMemcpyDeviceToHost, ctx->stream));
    if (a.trans_grad && !a.trans_grad_on_device)
      TRYCUDA(cudaMemcpyAsync(a.trans_grad, tg_dev, sizeof(float) * nTrans, cudaMemcpyDeviceToHost, ctx->stream));
  }
  TRY(readback_reserve(ctx, 4 * sizeof(float) * B));
  {
    float* d = reinterpret_cast<float*>(ctx->readback);
    float* n = d + B;
    int32_t* st = reinterpret_cast<int32_t*>(n + B);
    TRYCUDA(cudaMemcpyAsync(d, den, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaMemcpyAsync(n, lat->out_scores, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaMemcpyAsync(st, status, sizeof(int32_t) * 2 * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaStreamSynchronize(ctx->stream));
    for (int b = 0; b < B; b++) a.losses_host[b] = d[b] - n[b];
    for (int b = 0; b < 2 * B; b++) *needs_exact |= st[b] != 0;
  }
done:
  ctx->stream = main_stream;
  if (rc) cudaStreamSynchronize(ctx->copy_stream); // nothing may still run on the second stream when the buffers go
  if (lat) gtnb_lattice_destroy(ctx, lat);
  if (!a.emissions_on_device) dev_free(ctx, e_dev);
  if (!(a.grads && a.grads_on_device)) dev_free(ctx, g_dev);
  if (!a.trans_on_device) dev_free(ctx, w_dev);
  if (!(a.trans_grad && a.trans_grad_on_device)) dev_free(ctx, tg_dev);
  dev_free(ctx, small_dev);
  dev_free(ctx, status);
  dev_free(ctx, alpha);
  dev_free(ctx, den);
  dev_free(ctx, map);
  dev_free(ctx, ggrad);
  dev_free(ctx, minus1);
  return rc;
}

/*
 * Every other case -- C > 128, a non-finite weight or used emission, or the implicit path switched off -- through
 * asg_loss_run with the same T_b (the implicit sweeps, else the materialised lattices).  Device-resident
 * transitions and their gradient go through host copies on this route only.
 */
int asg_loss_ex_generic(gtnb_ctx* ctx, const AsgArgs& a, const std::vector<int32_t>& Tb) {
  const long long nTrans = a.C + (long long)a.C * a.C;
  std::vector<float> tw, tg;
  const float* tw_host = a.trans_w;
  if (a.trans_on_device) {
    tw.resize(nTrans);
    GTNB_CUDA(ctx, cudaMemcpy(tw.data(), a.trans_w, sizeof(float) * nTrans, cudaMemcpyDeviceToHost));
    tw_host = tw.data();
  }
  float* tg_host = a.trans_grad;
  if (a.trans_grad && a.trans_grad_on_device) {
    tg.resize(nTrans);
    tg_host = tg.data();
  }
  const int rc = asg_loss_run(ctx, a.B, a.T, a.C, a.emissions, a.emissions_on_device, Tb.data(), tw_host, a.targets,
                              a.target_lens, a.losses_host, a.grads, a.grads_on_device, tg_host);
  if (rc == GTNB_OK && a.trans_grad && a.trans_grad_on_device)
    GTNB_CUDA(ctx, cudaMemcpy(a.trans_grad, tg.data(), sizeof(float) * nTrans, cudaMemcpyHostToDevice));
  return rc;
}

#undef TRY
#undef TRYCUDA

int asg_loss_ex_run(gtnb_ctx* ctx, const AsgArgs& a) {
  const int B = a.B, T = a.T, C = a.C;
  if (!ctx || B < 0 || T < 0 || C <= 0 || !a.emissions || !a.trans_w || !a.target_lens || !a.losses_host)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss_ex: bad arguments");
  const long long nTrans = C + (long long)C * C;
  std::vector<int32_t> Tb(B), off(B);
  std::vector<SgDims> dims(B);
  long long tot_t = 0;
  for (int b = 0; b < B; b++) {
    const int U = a.target_lens[b];
    if (U < 0) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss_ex: negative target length");
    if (U > 0 && !a.targets) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss_ex: targets is NULL");
    const int32_t* y = a.targets + tot_t;
    for (int u = 0; u < U; u++)
      if (y[u] < 0 || y[u] >= C) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss_ex: label outside [0, C)");
    off[b] = (int32_t)tot_t;
    tot_t += U;
    Tb[b] = a.input_lens ? a.input_lens[b] : T;
    if (Tb[b] < 0 || Tb[b] > T)
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_asg_loss_ex: input_lens outside [0, T]");
    // compose(fal_b, transitions): U+1 nodes, 2U arcs (none when U = 0), node U accepts
    dims[b] = SgDims{U + 1, 2 * U, U > 0 ? 1 : 0, /*all_valid=*/1, /*uniform=*/1, /*max_in=*/2, /*max_out=*/2};
  }
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  if (B == 0) { // an empty batch: the transition gradient is 0
    if (a.trans_grad) {
      if (a.trans_grad_on_device) {
        GTNB_CUDA(ctx, cudaMemsetAsync(a.trans_grad, 0, sizeof(float) * nTrans, ctx->stream));
        GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
      } else {
        std::memset(a.trans_grad, 0, sizeof(float) * nTrans);
      }
    }
    return GTNB_OK;
  }
  bool needs_exact = false;
  const bool fast = C <= kNgramMaxLabels && ctx->use_implicit && implicit_dims_supported(dims.data(), B);
  int rc = fast ? asg_loss_ex_fast(ctx, a, Tb, dims, off, &needs_exact) : asg_loss_ex_generic(ctx, a, Tb);
  if (rc == GTNB_OK && needs_exact) {
    // a non-finite weight: asg_loss_run's sweeps raise the same status bit and end in the materialised lattices,
    // which reproduce the reference's inf / NaN propagation
    arena_end(ctx);
    arena_begin(ctx);
    rc = asg_loss_ex_generic(ctx, a, Tb);
  }
  // T_b = 0: linearGraph(0, C) is one start node that does not accept (creations.cpp:20-33), so both
  // compositions are empty and the reference's loss is -inf - -inf = NaN (no gradient)
  for (int b = 0; b < B && rc == GTNB_OK; b++)
    if (Tb[b] == 0) a.losses_host[b] = std::numeric_limits<float>::quiet_NaN();
  return rc;
}

} // namespace

extern "C" int gtnb_asg_loss_ex(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const float* trans_w, int trans_on_device, const int32_t* targets, const int32_t* target_lens,
    float* losses_host, float* grads, int grads_on_device, float* trans_grad, int trans_grad_on_device) {
  const AsgArgs a{B, T, C, emissions, emissions_on_device, input_lens, trans_w, trans_on_device, targets,
                  target_lens, losses_host, grads, grads_on_device, trans_grad, trans_grad_on_device};
  if (ctx) arena_begin(ctx);
  const int rc = asg_loss_ex_run(ctx, a);
  if (ctx) arena_end(ctx);
  return rc;
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
  const int32_t* input_lens;
  const gtnb_graph_view* graphs;
  const float* arc_weights;
  int arc_weights_on_device;
  float* losses_host;
  float* grads;
  int grads_on_device;
  float* arc_grads;
  int arc_grads_on_device;
};

#define TRY(x)                 \
  do {                         \
    if ((rc = (x))) goto done; \
  } while (0)
#define TRYCUDA(call)                                      \
  do {                                                     \
    cudaError_t e__ = (call);                              \
    if (e__ != cudaSuccess) {                              \
      rc = cuda_fail(ctx, e__, #call, __FILE__, __LINE__); \
      goto done;                                           \
    }                                                      \
  } while (0)

/* one attempt; implicit: try the sweeps first (the materialised lattices when the graphs do not qualify).
 * *needs_exact: a sweep met a non-finite weight or emission, the outputs are not to be used. */
int graph_loss_once(gtnb_ctx* ctx, const GraphLossArgs& a, const std::vector<gtnb_graph_view>& views,
                    const std::vector<int32_t>& Tb, long long tot_arcs, bool implicit, bool* needs_exact) {
  const int B = a.B, T = a.T, C = a.C;
  const long long per = (long long)T * C;
  const bool want = a.grads || a.arc_grads;
  int maxT = 0;
  for (int b = 0; b < B; b++) maxT = std::max(maxT, Tb[b]);
  int rc = GTNB_OK;
  float *e_dev = nullptr, *g_dev = nullptr, *ag_dev = nullptr, *den = nullptr, *minus1 = nullptr;
  int32_t *T_dev = nullptr, *status = nullptr;
  gtnb_lattice *lat = nullptr, *dlat = nullptr;
  cudaStream_t main_stream = ctx->stream;
  const float* aw_dev = a.arc_weights_on_device ? a.arc_weights : nullptr;
  const float* den_scores = nullptr;
  std::vector<float> m1(B, -1.0f); // subtract's gradFunc, functions.cpp:53-58
  // materialised route: forwardScore(E_b) as the reference computes it, non-finite emissions included (its sweep
  // turns a node whose in-scores are all NaN into -inf), from the lattice of one start-and-accept node with a
  // self-loop per label: compose(free, E_b) is E_b arc for arc
  std::vector<uint8_t> free_flags(1, 3);
  std::vector<int32_t> free_src(C, 0), free_lab(C);
  for (int c = 0; c < C; c++) free_lab[c] = c;
  gtnb_graph_view free_view;
  std::memset(&free_view, 0, sizeof(free_view));
  free_view.num_nodes = 1;
  free_view.num_arcs = C;
  free_view.node_flags = free_flags.data();
  free_view.arc_src = free_view.arc_dst = free_src.data();
  free_view.arc_ilabel = free_view.arc_olabel = free_lab.data();

  TRY(ensure_side_streams(ctx, 0, 0));
  if (a.emissions_on_device) {
    e_dev = const_cast<float*>(a.emissions);
  } else {
    TRY(dev_alloc(ctx, &e_dev, per * B));
    TRYCUDA(cudaMemcpyAsync(e_dev, a.emissions, sizeof(float) * per * B, cudaMemcpyHostToDevice, ctx->stream));
  }
  TRY(dev_alloc(ctx, &den, B));
  TRY(dev_alloc(ctx, &T_dev, B));
  TRY(dev_alloc(ctx, &status, B));
  TRY(dev_alloc(ctx, &minus1, B));
  if (want) {
    if (a.grads && a.grads_on_device)
      g_dev = a.grads;
    else
      TRY(dev_alloc(ctx, &g_dev, per * B)); // also the scratch of a call that only wants the arc gradients
    TRYCUDA(cudaMemsetAsync(g_dev, 0, sizeof(float) * per * B, ctx->stream));
    if (a.arc_grads) {
      if (a.arc_grads_on_device)
        ag_dev = a.arc_grads;
      else
        TRY(dev_alloc(ctx, &ag_dev, tot_arcs));
      if (tot_arcs) TRYCUDA(cudaMemsetAsync(ag_dev, 0, sizeof(float) * tot_arcs, ctx->stream));
    }
  }
  TRYCUDA(cudaMemsetAsync(status, 0, sizeof(int32_t) * B, ctx->stream));
  TRY(stage_begin(ctx));
  TRY(stage_upload(ctx, T_dev, Tb.data(), sizeof(int32_t) * B));
  TRY(stage_upload(ctx, minus1, m1.data(), sizeof(float) * B));
  TRY(stage_end(ctx));

  if (implicit) {
    rc = compose_linear_impl(ctx, B, views.data(), B, 0, Tb.data(), C, e_dev, per, true, &lat, true, aw_dev);
    if (rc == GTNB_ERR_UNSUPPORTED) { // does not fit the implicit layout: materialise
      implicit = false;
      rc = GTNB_OK;
    } else if (rc) {
      goto done;
    }
  }
  if (implicit) {
    // forwardScore(E_b) and its +1 gradient on the second stream, beside the forward sweep
    TRYCUDA(cudaEventRecord(ctx->ev_fork, ctx->stream));
    TRYCUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_fork, 0));
    ctx->stream = ctx->copy_stream;
    rc = launch_linear_forward(ctx, B, T_dev, maxT, C, e_dev, per, 0, den, want ? g_dev : nullptr, per, nullptr,
                               1.0f, 0);
    ctx->stream = main_stream;
    if (rc) goto done;
    TRYCUDA(cudaEventRecord(ctx->ev_join, ctx->copy_stream));
    TRY(launch_implicit_forward(ctx, lat, status));
    TRYCUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
    if (want) TRY(launch_implicit_backward(ctx, lat, minus1, g_dev, per, 0, -1, ag_dev));
    den_scores = den;
  } else {
    TRY(compose_linear_impl(ctx, B, views.data(), B, 0, Tb.data(), C, e_dev, per, false, &lat, false, aw_dev));
    TRY(compose_linear_impl(ctx, B, &free_view, 1, 0, Tb.data(), C, e_dev, per, false, &dlat));
    TRY(gtnb_forward(ctx, dlat, 0, nullptr, nullptr));
    TRY(gtnb_forward(ctx, lat, 0, nullptr, nullptr));
    if (want) {
      TRY(gtnb_backward(ctx, dlat, 0, nullptr)); // +1
      TRY(gtnb_compose_grad(ctx, dlat, nullptr, g_dev, per));
      TRY(gtnb_backward(ctx, lat, 0, m1.data()));
      TRY(gtnb_compose_grad(ctx, lat, ag_dev, g_dev, per));
    }
    den_scores = dlat->out_scores;
  }
  if (a.grads && !a.grads_on_device)
    TRYCUDA(cudaMemcpyAsync(a.grads, g_dev, sizeof(float) * per * B, cudaMemcpyDeviceToHost, ctx->stream));
  if (a.arc_grads && !a.arc_grads_on_device && tot_arcs)
    TRYCUDA(cudaMemcpyAsync(a.arc_grads, ag_dev, sizeof(float) * tot_arcs, cudaMemcpyDeviceToHost, ctx->stream));
  TRY(readback_reserve(ctx, 3 * sizeof(float) * B));
  {
    float* d = reinterpret_cast<float*>(ctx->readback);
    float* n = d + B;
    int32_t* st = reinterpret_cast<int32_t*>(n + B);
    TRYCUDA(cudaMemcpyAsync(d, den_scores, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaMemcpyAsync(n, lat->out_scores, sizeof(float) * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaMemcpyAsync(st, status, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, ctx->stream));
    TRYCUDA(cudaStreamSynchronize(ctx->stream));
    for (int b = 0; b < B; b++) a.losses_host[b] = d[b] - n[b];
    if (implicit)
      for (int b = 0; b < B; b++) *needs_exact |= st[b] != 0;
  }
done:
  ctx->stream = main_stream;
  if (rc) cudaStreamSynchronize(ctx->copy_stream); // nothing may still run on the second stream when the buffers go
  if (lat) gtnb_lattice_destroy(ctx, lat);
  if (dlat) gtnb_lattice_destroy(ctx, dlat);
  if (!a.emissions_on_device) dev_free(ctx, e_dev);
  if (!(a.grads && a.grads_on_device)) dev_free(ctx, g_dev);
  if (!(a.arc_grads && a.arc_grads_on_device)) dev_free(ctx, ag_dev);
  dev_free(ctx, den);
  dev_free(ctx, T_dev);
  dev_free(ctx, status);
  dev_free(ctx, minus1);
  return rc;
}

#undef TRY
#undef TRYCUDA

int graph_loss_run(gtnb_ctx* ctx, const GraphLossArgs& a) {
  const int B = a.B, T = a.T, C = a.C;
  if (!ctx || B < 0 || T < 0 || C <= 0 || (B > 0 && (!a.emissions || !a.graphs || !a.losses_host)))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_graph_loss: bad arguments");
  std::vector<int32_t> Tb(B);
  std::vector<gtnb_graph_view> views(a.graphs, a.graphs + B);
  long long tot_arcs = 0;
  for (int b = 0; b < B; b++) {
    Tb[b] = a.input_lens ? a.input_lens[b] : T;
    if (Tb[b] < 0 || Tb[b] > T) return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_graph_loss: input_lens outside [0, T]");
    if (validate_view(ctx, views[b])) return GTNB_ERR_INVALID_ARGUMENT;
    for (int k = 0; k < views[b].num_arcs; k++)
      if (views[b].arc_olabel[k] == GTNB_EPSILON)
        return fail(ctx, GTNB_ERR_UNSUPPORTED,
                    "gtnb_graph_loss: graph " + std::to_string(b) +
                        " has epsilon arcs; remove them first (remove(g, epsilon))");
    if (a.arc_weights && !a.arc_weights_on_device) views[b].weights = a.arc_weights + tot_arcs;
    tot_arcs += views[b].num_arcs;
  }
  if (tot_arcs >= (1ll << 31)) return fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_graph_loss: more than 2^31 arcs");
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  if (B == 0) return GTNB_OK;
  // (graphs that are not label-uniform need C <= k_implicit.cu's kArcMaxLabels: compose_linear_impl checks)
  const bool implicit = ctx->use_implicit;
  bool needs_exact = false;
  int rc = graph_loss_once(ctx, a, views, Tb, tot_arcs, implicit, &needs_exact);
  if (rc == GTNB_OK && needs_exact) {
    // a non-finite weight or emission: the materialised lattices reproduce the reference's inf / NaN
    // propagation arc by arc
    arena_end(ctx);
    arena_begin(ctx);
    rc = graph_loss_once(ctx, a, views, Tb, tot_arcs, false, &needs_exact);
  }
  // T_b = 0: linearGraph(0, C) accepts nothing, so both scores are -inf and the loss is NaN (no gradient)
  for (int b = 0; b < B && rc == GTNB_OK; b++)
    if (Tb[b] == 0) a.losses_host[b] = std::numeric_limits<float>::quiet_NaN();
  return rc;
}

} // namespace

extern "C" int gtnb_graph_loss(
    gtnb_ctx* ctx, int B, int T, int C, const float* emissions, int emissions_on_device, const int32_t* input_lens,
    const gtnb_graph_view* graphs, const float* arc_weights, int arc_weights_on_device, float* losses_host,
    float* grads, int grads_on_device, float* arc_grads, int arc_grads_on_device) {
  const GraphLossArgs a{B, T, C, emissions, emissions_on_device, input_lens, graphs, arc_weights,
                        arc_weights_on_device, losses_host, grads, grads_on_device, arc_grads, arc_grads_on_device};
  if (ctx) arena_begin(ctx);
  const int rc = graph_loss_run(ctx, a);
  if (ctx) arena_end(ctx);
  return rc;
}
