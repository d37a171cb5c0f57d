/*
 * gtn_b200.h -- C ABI of the H100-native gtn hot path.
 *
 * One shared library (gtn_b200/lib/libgtn_b200.so, sm_90a CUDA inside)
 * exporting plain-C entry points: opaque handles, plain pointers and sizes,
 * int status returns, no exceptions, no torch / STL types.  This is the seam a
 * gtn maintainer binds instead of the CPU implementations of
 *
 *   gtn::compose / gtn::intersect     reference gtn/functions.cpp:225-251
 *                                       -> detail::compose, functions/compose.cpp:377-522
 *   gtn::forwardScore / viterbiScore  functions.cpp:320-326 -> detail::shortestDistance,
 *                                       functions/shortest.cpp:86-188 (+ grad :33-82)
 *   gtn::viterbiPath                  functions.cpp:328-330 -> detail::shortestPath,
 *                                       functions/shortest.cpp:190-272
 *   compose gradFunc                  functions/compose.cpp:496-518
 *   gtn::linearGraph + setWeights     creations.cpp:20-33, graph.cpp:179-181
 *   parallelMap(fwd) / parallelMap(bwd)  benchmarks/ctc.cpp:150-165 (the batch seam)
 *
 * The reference has no FFI layer of its own (SURVEY.md section 8(b)); the C++
 * mirror of its public headers (gtn_b200/csrc/gtn/) and the pybind11 module
 * sit on top of exactly these functions -- see INTEGRATION.md.
 *
 * Conventions
 *  - every function returns GTNB_OK or a negative-free positive error code;
 *    gtnb_last_error(ctx) gives the message.  The C++ shim maps
 *    GTNB_ERR_INVALID_ARGUMENT -> std::invalid_argument,
 *    GTNB_ERR_LOGIC -> std::logic_error, others -> std::runtime_error, which
 *    is what the reference throws (shortest.cpp:150,230; graph.cpp:71-94).
 *  - all device work is enqueued on the context's stream; functions that
 *    return host results synchronise that stream, the others do not.
 *  - "dev" pointers are device memory on the context's device, "host"
 *    pointers are host memory (pinned or pageable).
 *  - there is NO CPU fallback: every compute entry point launches sm_90a
 *    kernels and fails with GTNB_ERR_RUNTIME when no CUDA device is usable.
 */
#ifndef GTN_B200_H
#define GTN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GTNB_VERSION 100

#define GTNB_OK 0
#define GTNB_ERR_INVALID_ARGUMENT 2 /* std::invalid_argument */
#define GTNB_ERR_LOGIC 3 /* std::logic_error */
#define GTNB_ERR_RUNTIME 4 /* std::runtime_error, incl. CUDA failures */
#define GTNB_ERR_UNSUPPORTED 5 /* shape outside what the device path covers */

#define GTNB_EPSILON (-1) /* gtn::epsilon, graph.h:21 */

typedef struct gtnb_ctx gtnb_ctx;
/* A packed batch of B device-resident graphs (levelised CSR-by-destination). */
typedef struct gtnb_lattice gtnb_lattice;

/*
 * Host view of one gtn::Graph (graph.h:56-465), borrowed for the call only.
 * Arrays are indexed by arc id / node id exactly as Graph numbers them.
 * in_ptr/in_arcs and out_ptr/out_arcs are the per-node arc lists in the
 * Graph's current order (i.e. after any arcSort, graph.cpp:162-177); pass NULL
 * for "insertion order".  accept/start give g.accept()/g.start() order; NULL
 * means ascending node id.
 */
typedef struct gtnb_graph_view {
  int32_t num_nodes;
  int32_t num_arcs;
  const uint8_t* node_flags; /* bit0 = start, bit1 = accept */
  const int32_t* arc_src;
  const int32_t* arc_dst;
  const int32_t* arc_ilabel;
  const int32_t* arc_olabel;
  const float* weights; /* NULL = all 0 */
  const int32_t* in_ptr; /* [num_nodes+1] or NULL */
  const int32_t* in_arcs; /* [num_arcs] */
  const int32_t* out_ptr;
  const int32_t* out_arcs;
  const int32_t* start; /* [num_start] or NULL */
  int32_t num_start;
  const int32_t* accept; /* [num_accept] or NULL */
  int32_t num_accept;
} gtnb_graph_view;

/* ---- context ------------------------------------------------------- */

/* cuda_stream: a cudaStream_t to enqueue on, or NULL for a private stream. */
int gtnb_ctx_create(int device, void* cuda_stream, gtnb_ctx** out);
void gtnb_ctx_destroy(gtnb_ctx* ctx);
/* ctx may be NULL: returns the calling thread's last creation error. */
const char* gtnb_last_error(const gtnb_ctx* ctx);
int gtnb_ctx_synchronize(gtnb_ctx* ctx);
void* gtnb_ctx_stream(gtnb_ctx* ctx);
/* the CUDA device ordinal the context was created on */
int gtnb_ctx_device(const gtnb_ctx* ctx);
int gtnb_version(void);
/* number of kernels this context has launched so far (bench bookkeeping) */
int64_t gtnb_ctx_launch_count(const gtnb_ctx* ctx);

/*
 * Tuning / testing switches.  "staged" (default 1): use the TMA-staged persistent
 * kernels for composed lattices; 0 forces the generic any-DAG kernels (libm-precise),
 * which is how the tests cross-check the two families.  "implicit" (default 1): the
 * criteria (gtnb_ctc_loss) sweep the frames of intersect(target graph, emissions) without
 * materialising the lattice; 0 makes them build it and run the lattice kernels.
 * "bidir_mode" (default -1): the node warps of gtnb_ctc_loss's one-launch kernel (k_bidir.cu) at
 * C = 64 / 128: -1 or 1 the PAIR kernels (a label and a blank node per thread), 0 one node per
 * thread; any other value is rejected.  "exact_ties" (default 0, EXPERIMENTAL; set before gtnb_compose_linear): gtnb_viterbi_path
 * on a composed lattice breaks exact score ties like the reference's shortestPath (k_order.cu).
 * "sparse_cluster" (default 0): the route of gtnb_sparse_transitions_loss, gtnb_viterbi_sparse and
 * gtnb_sparse_transitions_viterbi for a transition graph G beyond one CTA's shared memory (over 4096 nodes or 32768
 * arcs).  0: the materialised route.  1: G is swept by one thread-block cluster of 2, 4 or 8 CTAs per utterance
 * (k_sparse.cu's sparse_cl_* kernels) when it has at most 16384 nodes, 262144 arcs labelled in [0, C), in-degree
 * 32766, C <= 1024, and the cluster's shared memory holds it (the score rows in every CTA, an arc-gradient
 * accumulator split over the CTAs: e.g. 4096 nodes with 262144 arcs, or 16384 nodes with 131072 arcs); a smaller G
 * keeps the one-CTA kernels.  2, 4, 8 (testing and measurement): additionally every G that fits a cluster of that
 * size takes it; results are bit-identical apart from the order of the gradient sums.  Other values are rejected.
 * The flag governs gtnb_backoff_transitions_loss, gtnb_viterbi_backoff and gtnb_backoff_transitions_viterbi the same
 * way for a backoff G (with epsilon arcs) beyond their one-CTA envelope: at 1 its denominator is swept by a cluster
 * (k_sparse.cu's sparse_cl_eps_* kernels) when it has at most 16384 nodes, 262144 emitting plus epsilon arcs, 32
 * levels, a combined in-degree below 32766, C <= 1024, and the cluster's shared memory holds it (e.g. a backoff
 * 4-gram of 8563 states / 65 793 arcs at C = 64 takes 2 CTAs); the numerators keep their one-CTA envelope.
 */
int gtnb_ctx_set_flag(gtnb_ctx* ctx, const char* name, int value);

/* device / pinned memory helpers so callers need no CUDA runtime of their own.
 * gtnb_device_alloc / _free are stream-ordered on the context's stream (cudaMallocAsync):
 * the memory is valid for work enqueued on that stream; synchronise before using it elsewhere. */
int gtnb_device_alloc(gtnb_ctx* ctx, size_t bytes, void** out);
int gtnb_device_free(gtnb_ctx* ctx, void* p);
int gtnb_host_alloc(gtnb_ctx* ctx, size_t bytes, void** out); /* pinned */
int gtnb_host_free(gtnb_ctx* ctx, void* p);
int gtnb_memcpy_h2d(gtnb_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes);
int gtnb_memcpy_d2h(gtnb_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes);
int gtnb_memset(gtnb_ctx* ctx, void* dst_dev, int value, size_t bytes);
/* CUDA-event timing on the context's stream */
int gtnb_timer_start(gtnb_ctx* ctx);
int gtnb_timer_stop(gtnb_ctx* ctx, float* ms); /* synchronises */
/*
 * Per-kernel CUDA-event timing on the context's stream.  gtnb_profile_read
 * synchronises, returns "name launches total_ms\n" lines (one per kernel name,
 * valid until the next call) and clears the log.
 */
int gtnb_profile_enable(gtnb_ctx* ctx, int on);
const char* gtnb_profile_read(gtnb_ctx* ctx);
/* write `bytes` of scratch to evict L2 between timed iterations */
int gtnb_flush_l2(gtnb_ctx* ctx);

/* ---- building device graphs ---------------------------------------- */

/*
 * Generic path: levelise B arbitrary host graphs (Kahn order exactly as
 * shortest.cpp:92-145 walks them) and upload them as one packed batch.
 * Structural errors the reference reports lazily ("Graph has a cycle,
 * self-loop or is disconnected!", shortest.cpp:149-152) are recorded per graph
 * and raised by gtnb_forward / gtnb_viterbi_path.
 */
int gtnb_pack(gtnb_ctx* ctx, int B, const gtnb_graph_view* graphs, gtnb_lattice** out);

/*
 * Frame-synchronous device composition (detail::compose, compose.cpp:377-522,
 * for the case one operand is a gtn::linearGraph): lattice_b =
 *   linear_first ? compose(linear(T_b, C; emissions_b), graphs_b)
 *                : compose(graphs_b, linear(T_b, C; emissions_b)).
 * graphs: n_graphs == B, or == 1 to share one graph across the batch (ASG
 * transitions).  The matched side of each graph must be epsilon-free
 * (GTNB_ERR_UNSUPPORTED otherwise; the host compose handles those).
 * emissions_dev: utterance b's row-major [T_b][C] matrix starts at
 * emissions_dev + b * emissions_stride.  The lattice keeps this pointer: it
 * must stay valid until the lattice is destroyed (weights are read again by
 * nothing, but compose_grad writes through grad pointers you pass then).
 * Arc weight = w_graph + e[t][label]  (compose.cpp:435), provenance kept per
 * arc for gtnb_compose_grad (gradInfo, compose.cpp:445).
 */
int gtnb_compose_linear(
    gtnb_ctx* ctx,
    int B,
    const gtnb_graph_view* graphs,
    int n_graphs,
    int linear_first,
    const int32_t* T, /* host [B] */
    int C,
    const float* emissions_dev,
    int64_t emissions_stride,
    gtnb_lattice** out);

/*
 * General composition on the device (k_gcompose.cu): replaces detail::compose (compose.cpp:377-522) for
 * operand pairs that are NOT frame-synchronous -- epsilon arcs on the matched side (compose.cpp:146-208,
 * 461-488), cyclic graphs, neither operand a chain (intersect(ctc, transitions) of timeNgramCtc,
 * benchmarks/ctc.cpp:118-123).  n_pairs pairs in one call, one CTA each; n_first / n_second are n_pairs, or 1
 * for an operand shared by every pair (parallel_map.h:77-89).  match_kind[b] is the matcher functions.cpp:225-251
 * would pick: 0 unsorted, 1 only the first operand sorted on the matched label, 2 only the second, 3 both.
 * The composed graphs keep the reference's node ids, arc ids and per-node arc order exactly.
 * GTNB_ERR_UNSUPPORTED when the product state space does not fit (>= 2^27 states per pair, or scratch larger
 * than half of the device memory).
 */
typedef struct gtnb_composed gtnb_composed;
int gtnb_compose_graphs(
    gtnb_ctx* ctx,
    int n_pairs,
    const gtnb_graph_view* first,
    int n_first,
    const gtnb_graph_view* second,
    int n_second,
    const int32_t* match_kind,
    gtnb_composed** out);
int gtnb_composed_sizes(const gtnb_composed* c, int pair, int32_t* num_nodes, int32_t* num_arcs);
/* any pointer may be NULL; gi_first / gi_second: compose.cpp:445's gradInfo (-1 on the epsilon side, :201-205) */
int gtnb_composed_download(
    gtnb_ctx* ctx,
    gtnb_composed* c,
    int pair,
    uint8_t* node_flags,
    int32_t* arc_src,
    int32_t* arc_dst,
    int32_t* arc_ilabel,
    int32_t* arc_olabel,
    float* weights,
    int32_t* gi_first,
    int32_t* gi_second);
void gtnb_composed_destroy(gtnb_ctx* ctx, gtnb_composed* c);

void gtnb_lattice_destroy(gtnb_ctx* ctx, gtnb_lattice* lat);
int gtnb_lattice_batch(const gtnb_lattice* lat);
/* per-graph node / arc counts (synchronises) */
int gtnb_lattice_sizes(gtnb_ctx* ctx, gtnb_lattice* lat, int32_t* num_nodes, int32_t* num_arcs);
/*
 * Materialise graph b on the host in Graph numbering (any pointer may be
 * NULL).  gi_graph / gi_linear are the compose provenance (-1 if none).
 */
int gtnb_lattice_download(
    gtnb_ctx* ctx,
    gtnb_lattice* lat,
    int b,
    uint8_t* node_flags,
    int32_t* arc_src,
    int32_t* arc_dst,
    int32_t* arc_ilabel,
    int32_t* arc_olabel,
    float* weights,
    int32_t* gi_graph,
    int32_t* gi_linear);

/* ---- the dynamic programs ------------------------------------------ */

/*
 * detail::shortestDistance over every graph of the batch (log semiring, or
 * tropical when `tropical`).  scores_host [B] (NULL = keep on device only).
 * Node scores stay in the lattice for the backward pass.
 * status_host [B] (nullable): per-graph GTNB_OK / GTNB_ERR_INVALID_ARGUMENT;
 * the call itself returns the first non-OK status.
 */
int gtnb_forward(gtnb_ctx* ctx, gtnb_lattice* lat, int tropical, float* scores_host, int32_t* status_host);

/*
 * shortestDistanceGrad (shortest.cpp:33-82): arc gradients of the last
 * gtnb_forward, scaled per graph by deltas_host[b] (NULL = 1).  Results stay
 * on the device; read them with gtnb_lattice_arc_grads or push them to the
 * compose operands with gtnb_compose_grad.
 */
int gtnb_backward(gtnb_ctx* ctx, gtnb_lattice* lat, int tropical, const float* deltas_host);

/* copy graph b's arc gradients (Graph arc numbering) to the host */
int gtnb_lattice_arc_grads(gtnb_ctx* ctx, gtnb_lattice* lat, int b, float* out_host);
/*
 * Overwrite graph b's arc gradients from the host (composed lattices; Graph arc
 * numbering == device numbering there).  Lets compose's gradFunc run on the device
 * when the deltas were produced or accumulated on the host (autograd.h:37).
 */
int gtnb_lattice_set_arc_grads(gtnb_ctx* ctx, gtnb_lattice* lat, int b, const float* grads_host);
/* device pointer to all arc gradients (device arc order, the order gtnb_lattice_download
 * returns) -- advanced use.  NULL on error (gtnb_last_error) or before any backward. */
const float* gtnb_lattice_arc_grads_dev(gtnb_ctx* ctx, gtnb_lattice* lat);

/*
 * compose gradFunc (compose.cpp:496-518) for a lattice made by
 * gtnb_compose_linear: scatter-add the arc gradients to
 *   grad_graph_dev   [sum of graph arc counts] (one slab per graph, in batch
 *                    order; a single slab when the graph is shared), nullable
 *   grad_emissions_dev  utterance b at + b * grad_stride, [T_b][C], nullable
 * Both are accumulated into (addGrad semantics, graph.cpp:91-129); zero them
 * first for a fresh gradient.
 */
int gtnb_compose_grad(
    gtnb_ctx* ctx,
    gtnb_lattice* lat,
    float* grad_graph_dev,
    float* grad_emissions_dev,
    int64_t grad_stride);

/*
 * detail::shortestPath.  For each graph writes the best path's arcs (Graph
 * arc numbering, start -> end) into path_arcs_host + b * max_len and its
 * length into path_len_host[b] (-1: no accepting path).  ilabels/olabels of
 * those arcs go to path_ilabels_host / path_olabels_host (nullable).
 */
int gtnb_viterbi_path(
    gtnb_ctx* ctx,
    gtnb_lattice* lat,
    int max_len,
    int32_t* path_arcs_host,
    int32_t* path_ilabels_host,
    int32_t* path_olabels_host,
    float* path_weights_host, /* nullable: weights of the path's arcs */
    int32_t* path_len_host,
    int32_t* status_host);

/*
 * forwardScore of the emissions chain itself, forwardScore(linearGraph(T,C))
 * (the CTC normaliser, benchmarks/ctc.cpp:157): scores_dev[b] (device, [B]);
 * when grad_emissions_dev != NULL also accumulates delta_b * d score_b / d e
 * into it (delta = deltas_dev[b], or `delta_all` when deltas_dev == NULL).
 */
int gtnb_linear_forward(
    gtnb_ctx* ctx,
    int B,
    const int32_t* T, /* host [B] */
    int C,
    const float* emissions_dev,
    int64_t emissions_stride,
    int tropical,
    float* scores_dev,
    float* grad_emissions_dev,
    int64_t grad_stride,
    const float* deltas_dev,
    float delta_all);

/* ---- batched criteria: parallelMap(fwd)+parallelMap(bwd) in one call ---- */

/*
 * benchmarks/ctc.cpp:150-165 for a whole minibatch:
 *   loss_b = forwardScore(e_b) - forwardScore(intersect(ctcGraph(target_b), e_b))
 * and, when grads != NULL, d loss_b / d e_b.
 * emissions / grads: [B][T][C] row-major, on the device when *_on_device,
 * else host (copied in / out inside the call on the context's stream).
 * targets: concatenated labels, target_lens[B]; losses_host [B].
 * input_lens (nullable) gives per-utterance frame counts <= T.
 */
int gtnb_ctc_loss(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens,
    const int32_t* targets,
    const int32_t* target_lens,
    int blank,
    float* losses_host,
    float* grads,
    int grads_on_device);

#define GTNB_F32 0 /* float32 elements (the dtype of the *_ex / *_typed entry points) */
#define GTNB_BF16 1 /* bfloat16 elements */
#define GTNB_F16 2 /* IEEE half-precision elements */

/*
 * gtnb_ctc_loss on device buffers of a chosen element type: emissions_dev and grads_dev (nullable) are [B][T][C] of
 * dtype (GTNB_F32, GTNB_BF16 or GTNB_F16), both on the device; losses_host [B] stays float32.  Targets, lengths,
 * blank, infeasible targets, non-finite values and the zeroed rows t >= input_lens[b] follow gtnb_ctc_loss.
 * The result is gtnb_ctc_loss's on the emissions widened to float32 (exact): the same losses, bit for bit, and its
 * float32 gradient rounded to dtype (to nearest, ties to even).  Internally the arithmetic is float32 throughout:
 * the one-launch kernel (k_bidir.cu) reads and writes the 16-bit buffers in place when the batch takes it, C % 8 == 0
 * and both buffers are 16-byte aligned; any other batch is widened into float32 scratch once, run as gtnb_ctc_loss
 * runs it, and its gradient rounded into grads_dev.  GTNB_F32 is gtnb_ctc_loss with both buffers on the device.
 * An unknown dtype is GTNB_ERR_INVALID_ARGUMENT.
 */
int gtnb_ctc_loss_ex(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const void* emissions_dev,
    int dtype,
    const int32_t* input_lens, /* host, nullable */
    const int32_t* targets,
    const int32_t* target_lens,
    int blank,
    float* losses_host,
    void* grads_dev); /* nullable */

/*
 * gtnb_ctc_loss_ex with every per-utterance input and output in device memory, for a training step that must not wait
 * on the host (and may be captured into a CUDA graph).  The call enqueues its work on cuda_stream (NULL: the CUDA
 * default stream, not the context's) and returns: no host synchronisation, no read of device data on the host, no allocation and no
 * staging through host memory.  It issues kernel launches and, with input_lens, one memset of the gradient, all of
 * which stream capture accepts; one context per device serves every stream.  Its scratch memory is workspace_dev
 * (256-byte aligned, at least gtnb_ctc_loss_async_workspace's bytes for the same bounds and dtype; smaller is
 * GTNB_ERR_INVALID_ARGUMENT).
 *
 * targets_dev is [B][S] int32, row b holding target_lens_dev[b] labels; input_lens_dev is [B] (NULL: T each).
 * The call is sized from the bounds, never from the labels: every utterance as if U = S, T_b = T, with S - 1 skip
 * arcs.  The routes follow gtnb_ctc_loss_ex's: the one-launch kernel (k_bidir.cu) when the bounds and buffers take it
 * (16-bit buffers read in place when C % 8 == 0 and both are 16-byte aligned, else widened into the workspace), else
 * the two implicit sweeps.  Bounds outside both, the "implicit" flag at 0, blank outside [0, C) and an unknown dtype
 * are GTNB_ERR_UNSUPPORTED: use the synchronous call.
 *
 * losses_dev [B] float32 and status_dev [B] (nullable) are written on the device:
 *   0  the loss is gtnb_ctc_loss_ex's on the same data, bit for bit;
 *   1  a sweep met a non-finite value.  The synchronous call then repeats the batch on the exact materialised route,
 *      which needs the host; this call cannot, and writes a NaN loss and a zero gradient for the utterance;
 *   2  invalid input: target_lens_dev[b] outside [0, S], input_lens_dev[b] outside [0, T] or a label outside [0, C)
 *      (the synchronous call's GTNB_ERR_INVALID_ARGUMENT, per utterance here): a NaN loss and a zero gradient, and
 *      the utterance is swept as empty, so that no kernel indexes with its lengths or labels.
 * Other utterances are unaffected by a flagged one.  grads_dev (nullable) is [B][T][C] of dtype; rows
 * t >= input_lens_dev[b] are zero.
 */
int gtnb_ctc_loss_async(
    gtnb_ctx* ctx,
    void* cuda_stream,
    int B,
    int T,
    int C,
    int S,
    const void* emissions_dev, /* [B][T][C] of dtype */
    int dtype,
    const int32_t* input_lens_dev, /* [B] or NULL */
    const int32_t* targets_dev, /* [B][S] */
    const int32_t* target_lens_dev, /* [B] */
    int blank,
    float* losses_dev, /* [B] */
    int32_t* status_dev, /* [B] or NULL */
    void* grads_dev, /* [B][T][C] of dtype, or NULL */
    void* workspace_dev,
    size_t workspace_bytes);

/*
 * *bytes: the workspace gtnb_ctc_loss_async needs for these bounds, dtype and with_grad (any alignment of the
 * caller's buffers; host work only).  GTNB_ERR_UNSUPPORTED when the bounds are outside the asynchronous routes.
 */
int gtnb_ctc_loss_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int S, int dtype, int with_grad, size_t* bytes);

/*
 * ASG criterion for a whole minibatch (test/criterion_test.cpp:244-305, examples/asg.cpp:59-81,
 * BASELINE.json configs[2]):
 *   loss_b = forwardScore(compose(e_b, transitions))
 *          - forwardScore(compose(compose(fal_b, transitions), e_b))
 * transitions: the dense graph described at gtnb_viterbi_dense, weights trans_w_host
 * [C + C*C], shared by the batch.  grads (nullable): d loss_b / d e_b, [B][T][C];
 * trans_grad_host (nullable): sum over the batch of d loss_b / d transitions, [C + C*C]
 * (the reference accumulates it under grad_lock, graph.cpp:96-100).
 */
int gtnb_asg_loss(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const float* trans_w_host,
    const int32_t* targets,
    const int32_t* target_lens,
    float* losses_host,
    float* grads,
    int grads_on_device,
    float* trans_grad_host);

/*
 * ASG on a padded minibatch with the transitions anywhere (the loss of gtnb_asg_loss):
 *   loss_b = forwardScore(compose(E_b, transitions)) - forwardScore(compose(compose(fal_b, transitions), E_b))
 * E_b: linearGraph(T_b, C) on the first T_b = input_lens[b] (or T) rows of emissions_b.
 * trans_w [C + C*C] in gtnb_asg_loss's layout (the C start weights, then the C x C matrix, row = destination
 * label) and trans_grad (nullable, [C + C*C]: the batch sum of d loss_b / d trans_w) live on the device when
 * *_on_device, else on the host; likewise emissions and grads (nullable, [B][T][C]: d loss_b / d e_b).  EVERY
 * row of grads is written: rows t >= T_b are set to 0.  T_b = 0 gives NaN (linearGraph(0, C) accepts nothing);
 * an infeasible target (T_b < U) or U = 0 gives +inf and the denominator's gradient alone.  B = 0 zeroes
 * trans_grad.  Labels outside [0, C), negative lengths or T_b > T are GTNB_ERR_INVALID_ARGUMENT.
 * For C <= 128 the transitions never leave the device: the denominator is a dense on-chip trellis and the
 * numerator graphs are built on the device.  Larger alphabets and non-finite weights take the route of
 * gtnb_asg_loss (with T_b), which reads the transitions on the host.
 */
int gtnb_asg_loss_ex(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* nullable */
    const float* trans_w,
    int trans_on_device,
    const int32_t* targets,
    const int32_t* target_lens,
    float* losses_host,
    float* grads, /* nullable */
    int grads_on_device,
    float* trans_grad, /* nullable */
    int trans_grad_on_device);

/*
 * CTC with a learned bigram transition graph for a whole minibatch (benchmarks/ctc.cpp:107-134, timeNgramCtc):
 *   loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(ctc_b, G), E_b))
 * E_b: linearGraph(T_b, C) on the first T_b = input_lens[b] (or T) rows of emissions_b; ctc_b: the CTC graph of
 * target_b with `blank` (as gtnb_ctc_loss); G: C nodes, every node start and accept, arc j -> i with label i and
 * weight trans_w[i*C + j] (row = destination label, column = source label, ASG's layout), so G's state is the
 * previous frame's label, blank included.
 * trans_w [C*C] and trans_grad (nullable, [C*C]: the batch sum of d loss_b / d trans_w, as Graph::addGrad
 * accumulates it) live on the device when *_on_device, else on the host; likewise emissions and grads
 * (nullable, [B][T][C]: d loss_b / d e_b).  Unlike gtnb_ctc_loss, EVERY row of grads is written: rows t >= T_b
 * are set to 0, so the caller needs no memset.  An infeasible target (T_b too short) gives +inf and the
 * denominator's gradient alone.  Needs C <= 128 (GTNB_ERR_UNSUPPORTED above: W is held on chip); labels outside
 * [0, C), negative lengths or T_b > T are GTNB_ERR_INVALID_ARGUMENT.
 */
int gtnb_ngram_ctc_loss(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* nullable */
    const float* trans_w,
    int trans_on_device,
    const int32_t* targets,
    const int32_t* target_lens,
    int blank,
    float* losses_host,
    float* grads, /* nullable */
    int grads_on_device,
    float* trans_grad, /* nullable */
    int trans_grad_on_device);

/*
 * gtnb_ngram_ctc_loss and gtnb_asg_loss_ex on device buffers of a chosen element type: emissions_dev and grads_dev
 * (nullable) are [B][T][C] of dtype (GTNB_F32, GTNB_BF16 or GTNB_F16), all buffers live on the device, and
 * trans_w_dev, trans_grad_dev (nullable) and losses_host stay float32.  Targets, lengths, blank, infeasible targets,
 * T_b = 0, non-finite values, the zeroed rows t >= T_b and every argument check follow the float32 call.
 * The result is that call's on the emissions widened to float32 (exact): the same losses and transition gradient,
 * bit for bit, and its float32 emission gradient rounded to dtype (to nearest, ties to even).  The arithmetic is
 * float32 throughout.  A batch that the float32 call sends to the dense trellis (k_ngram.cu) and the device-built
 * numerators (k_implicit.cu) -- C <= 128, the "implicit" flag on, numerator graphs inside the implicit layout, every
 * weight and used emission finite -- is read in place by those kernels, whose gradient is rounded into grads_dev
 * once.  Any other batch (ASG with C > 128, the flag off, the exact retry after a non-finite value) is widened into
 * float32 scratch once, run as the float32 call runs it, and its gradient rounded into grads_dev.  GTNB_F32 is the
 * float32 call with every buffer on the device; an unknown dtype is GTNB_ERR_INVALID_ARGUMENT.
 */
int gtnb_ngram_ctc_loss_typed(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const void* emissions_dev,
    int dtype,
    const int32_t* input_lens, /* host, nullable */
    const float* trans_w_dev,
    const int32_t* targets,
    const int32_t* target_lens,
    int blank,
    float* losses_host,
    void* grads_dev, /* nullable */
    float* trans_grad_dev); /* nullable */

int gtnb_asg_loss_typed(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const void* emissions_dev,
    int dtype,
    const int32_t* input_lens, /* host, nullable */
    const float* trans_w_dev,
    const int32_t* targets,
    const int32_t* target_lens,
    float* losses_host,
    void* grads_dev, /* nullable */
    float* trans_grad_dev); /* nullable */

/*
 * gtnb_ngram_ctc_loss_typed and gtnb_asg_loss_typed with every per-utterance input and output in device memory, for a
 * training step with learned transitions that must not wait on the host (and may be captured into a CUDA graph).
 * The contract is gtnb_ctc_loss_async's: the call enqueues its work on cuda_stream (NULL: the CUDA default stream) and
 * returns, without a host synchronisation, a read of device data on the host, an allocation or a staging copy.  It
 * issues kernel launches, memsets and event records / waits between cuda_stream and the context's side stream, and
 * for n-gram CTC one device-to-device copy of the transition gradient out of the workspace.  The side stream and its event are created by the first call
 * made outside stream capture; a call under capture before that is GTNB_ERR_INVALID_ARGUMENT.  Scratch memory is
 * workspace_dev (256-byte aligned, at least the matching *_async_workspace's bytes for the same bounds and dtype;
 * smaller is GTNB_ERR_INVALID_ARGUMENT).
 *
 * targets_dev is [B][S] int32, row b holding target_lens_dev[b] labels; input_lens_dev is [B] (NULL: T each).  The
 * call is sized from the bounds, never from the labels: every utterance as if U = S and T_b = T (n-gram CTC: with
 * S - 1 skip arcs).  The route is the synchronous calls' device route: the numerator graphs built on the device and
 * swept by the implicit kernels beside the dense trellis of the denominator; emissions of dtype (GTNB_F32, GTNB_BF16,
 * GTNB_F16) read in place.  C > 128, the "implicit" flag at 0, bounds outside the implicit sweeps, blank outside
 * [0, C) (n-gram) and an unknown dtype are GTNB_ERR_UNSUPPORTED: use the synchronous call.
 *
 * trans_w_dev: float32 on the device, n-gram W [C*C] (row = destination label), ASG [C + C*C] (start weights, then
 * the matrix).  losses_dev [B] float32 and status_dev [B] (nullable) are written on the device:
 *   0  the loss is the synchronous call's on the same data, bit for bit (NaN for T_b = 0, as there);
 *   1  the denominator's or the numerator's sweep met a non-finite value (the synchronous call repeats the batch on
 *      the exact materialised route, which needs the host): a NaN loss and a zero emission-gradient row;
 *   2  invalid input: target_lens_dev[b] outside [0, S], input_lens_dev[b] outside [0, T] or a label outside
 *      [0, C): a NaN loss and a zero row, and the utterance is swept as empty.
 * A flagged utterance (1 or 2) adds nothing to trans_grad_dev, which sums over the batch: the other utterances'
 * gradient is what the synchronous call gives on the batch without it.  A non-finite transition weight flags every
 * utterance, T_b = 0 and 1 included (the denominator checks all of trans_w_dev whatever T_b), and trans_grad_dev is
 * then all zeros.
 * grads_dev (nullable): [B][T][C] of dtype, rows t >= input_lens_dev[b] zero.  trans_grad_dev (nullable): float32, the
 * size of trans_w_dev.  The gradients add with atomics, so they vary from run to run as the synchronous call's do.
 */
int gtnb_ngram_ctc_loss_async(
    gtnb_ctx* ctx,
    void* cuda_stream,
    int B,
    int T,
    int C,
    int S,
    const void* emissions_dev, /* [B][T][C] of dtype */
    int dtype,
    const int32_t* input_lens_dev, /* [B] or NULL */
    const float* trans_w_dev, /* [C*C] */
    const int32_t* targets_dev, /* [B][S] */
    const int32_t* target_lens_dev, /* [B] */
    int blank,
    float* losses_dev, /* [B] */
    int32_t* status_dev, /* [B] or NULL */
    void* grads_dev, /* [B][T][C] of dtype, or NULL */
    float* trans_grad_dev, /* [C*C] or NULL */
    void* workspace_dev,
    size_t workspace_bytes);

/* gtnb_ngram_ctc_loss_async without a blank, on ASG's transitions */
int gtnb_asg_loss_async(
    gtnb_ctx* ctx,
    void* cuda_stream,
    int B,
    int T,
    int C,
    int S,
    const void* emissions_dev, /* [B][T][C] of dtype */
    int dtype,
    const int32_t* input_lens_dev, /* [B] or NULL */
    const float* trans_w_dev, /* [C + C*C] */
    const int32_t* targets_dev, /* [B][S] */
    const int32_t* target_lens_dev, /* [B] */
    float* losses_dev, /* [B] */
    int32_t* status_dev, /* [B] or NULL */
    void* grads_dev, /* [B][T][C] of dtype, or NULL */
    float* trans_grad_dev, /* [C + C*C] or NULL */
    void* workspace_dev,
    size_t workspace_bytes);

/*
 * *bytes: the workspace gtnb_ngram_ctc_loss_async / gtnb_asg_loss_async need for these bounds and dtype (with_grad:
 * either gradient will be asked for; host work only).  GTNB_ERR_UNSUPPORTED when the call would be.
 */
int gtnb_ngram_ctc_loss_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int S, int dtype, int with_grad,
                                        size_t* bytes);
int gtnb_asg_loss_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int S, int dtype, int with_grad, size_t* bytes);

/*
 * Forced alignment without a host synchronisation: viterbiPath / viterbiScore of the numerator of gtnb_ctc_loss_async,
 * gtnb_ngram_ctc_loss_async or gtnb_asg_loss_async, which tells which frames each target token occupies:
 *   gtnb_ctc_align_async        intersect(ctcGraph(y_b), E_b)              (gtnb_graph_viterbi on CTC graphs)
 *   gtnb_ngram_ctc_align_async  intersect(intersect(ctc_b, G), E_b)        (gtnb_graph_transitions_viterbi, BIGRAM)
 *   gtnb_asg_align_async        compose(compose(fal_b, transitions), E_b)  (gtnb_graph_transitions_viterbi, ASG)
 * The contract is gtnb_ctc_loss_async's: the call enqueues kernel launches on cuda_stream (NULL: the CUDA default
 * stream) and returns, without a host synchronisation, a read of device data on the host, an allocation or a staging
 * copy; it may be captured into a CUDA graph.  Scratch memory is workspace_dev (256-byte aligned, at least the matching
 * *_align_async_workspace's bytes for the same bounds and dtype; smaller is GTNB_ERR_INVALID_ARGUMENT).  The call is
 * sized from the bounds (every utterance as if U = S and T_b = T), never from the labels.  Emissions of dtype
 * GTNB_BF16 / GTNB_F16 are widened to float32 in the workspace: the results are the float32 call's on the widened
 * emissions.  The "implicit" flag at 0, bounds outside the implicit sweeps or the trace, blank outside [0, C) and an
 * unknown dtype are GTNB_ERR_UNSUPPORTED: use gtnb_graph_viterbi / gtnb_graph_transitions_viterbi.  There is no
 * bound on C beyond the sweeps' own (n-gram and ASG alignment do not hold a dense trellis).
 *
 * targets_dev [B][S] int32, row b holding target_lens_dev[b] labels; input_lens_dev [B] (NULL: T each); trans_w_dev
 * float32 on the device, n-gram W [C*C] (row = destination label), ASG [C + C*C].  Outputs, written on the device:
 *   paths_dev [B][T] (nullable)   the label of every frame of the best path;
 *   tokens_dev [B][T] (nullable)  the target position u in [0, U_b) each frame is aligned to, -1 for a blank frame
 *                                 (CTC, n-gram CTC; every ASG frame in [0, T_b) has one);
 *                                 both -1 beyond T_b and wherever no path accepts;
 *   scores_dev [B]                viterbiScore: -inf for T_b = 0 or a target with no path;
 *   status_dev [B] (nullable)     0  paths, tokens and score are the synchronous aligner's, ties included;
 *                                 1  the sweep met a non-finite value (the synchronous aligner takes its exact route):
 *                                    a NaN score and -1 rows;
 *                                 2  invalid input: target_lens_dev[b] outside [0, S], input_lens_dev[b] outside
 *                                    [0, T] or a label outside [0, C): a NaN score and -1 rows;
 *                                 3  a tie on the traced path: the score is the synchronous aligner's and the path
 *                                    an optimal one, which may break the tie differently (exact_ties off).
 * A flagged utterance never affects the others.
 */
int gtnb_ctc_align_async(
    gtnb_ctx* ctx,
    void* cuda_stream,
    int B,
    int T,
    int C,
    int S,
    const void* emissions_dev, /* [B][T][C] of dtype */
    int dtype,
    const int32_t* input_lens_dev, /* [B] or NULL */
    const int32_t* targets_dev, /* [B][S] */
    const int32_t* target_lens_dev, /* [B] */
    int blank,
    int32_t* paths_dev, /* [B][T] or NULL */
    int32_t* tokens_dev, /* [B][T] or NULL */
    float* scores_dev, /* [B] */
    int32_t* status_dev, /* [B] or NULL */
    void* workspace_dev,
    size_t workspace_bytes);

int gtnb_ngram_ctc_align_async(
    gtnb_ctx* ctx,
    void* cuda_stream,
    int B,
    int T,
    int C,
    int S,
    const void* emissions_dev, /* [B][T][C] of dtype */
    int dtype,
    const int32_t* input_lens_dev, /* [B] or NULL */
    const float* trans_w_dev, /* [C*C] */
    const int32_t* targets_dev, /* [B][S] */
    const int32_t* target_lens_dev, /* [B] */
    int blank,
    int32_t* paths_dev, /* [B][T] or NULL */
    int32_t* tokens_dev, /* [B][T] or NULL */
    float* scores_dev, /* [B] */
    int32_t* status_dev, /* [B] or NULL */
    void* workspace_dev,
    size_t workspace_bytes);

int gtnb_asg_align_async(
    gtnb_ctx* ctx,
    void* cuda_stream,
    int B,
    int T,
    int C,
    int S,
    const void* emissions_dev, /* [B][T][C] of dtype */
    int dtype,
    const int32_t* input_lens_dev, /* [B] or NULL */
    const float* trans_w_dev, /* [C + C*C] */
    const int32_t* targets_dev, /* [B][S] */
    const int32_t* target_lens_dev, /* [B] */
    int32_t* paths_dev, /* [B][T] or NULL */
    int32_t* tokens_dev, /* [B][T] or NULL */
    float* scores_dev, /* [B] */
    int32_t* status_dev, /* [B] or NULL */
    void* workspace_dev,
    size_t workspace_bytes);

/* *bytes: the workspace the matching *_align_async call needs for these bounds and dtype (host work only) */
int gtnb_ctc_align_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int S, int dtype, size_t* bytes);
int gtnb_ngram_ctc_align_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int S, int dtype, size_t* bytes);
int gtnb_asg_align_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int S, int dtype, size_t* bytes);

/*
 * Loss over one user-supplied target graph per utterance (the criterion of the reference's pytorch_loss.py and of
 * its word-decomposition examples):
 *   loss_b = forwardScore(E_b) - forwardScore(intersect(A_b, E_b))
 * E_b: linearGraph(T_b, C) on the first T_b = input_lens[b] (or T) rows of emissions_b ([B][T][C]); A_b =
 * graphs[b], a host view as gtnb_pack takes it, matched on its olabels (= ilabels for an acceptor).  Arcs labelled
 * outside [0, C) never match (gradient 0); an epsilon arc is GTNB_ERR_UNSUPPORTED (remove(g, epsilon) first).
 * arc_weights (nullable, [sum_b A_b] in batch order, on the device when arc_weights_on_device) replace the views'
 * weights.  grads (nullable, d loss_b / d e_b, [B][T][C]): EVERY row is written, 0 beyond T_b.  arc_grads
 * (nullable, [sum_b A_b]: d loss_b / d A_b's arc weights, Graph arc numbering) is written, not accumulated.
 * T_b = 0 gives NaN (linearGraph(0, C) accepts nothing); a graph with no accepting path of T_b arcs, or an empty
 * graph, gives +inf and the denominator's gradient alone.  T_b > T, negative lengths or a malformed view are
 * GTNB_ERR_INVALID_ARGUMENT.  B = 0 is a no-op.
 * The frames are swept without building intersect(A_b, E_b) when the graphs fit k_implicit.cu's layout (graphs
 * whose nodes have in-arcs of different labels: C <= 1024); otherwise, with the "implicit" flag off, or when a
 * non-finite weight or emission is met, the lattices are materialised.
 */
int gtnb_graph_loss(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* nullable */
    const gtnb_graph_view* graphs,
    const float* arc_weights, /* nullable */
    int arc_weights_on_device,
    float* losses_host,
    float* grads, /* nullable */
    int grads_on_device,
    float* arc_grads, /* nullable */
    int arc_grads_on_device);

/*
 * viterbiPath + viterbiScore of compose(linearGraph(T, C; e_b), transitions) for a whole
 * minibatch (test/criterion_test.cpp:308-345, BASELINE.json configs[3]) WITHOUT
 * materialising the T*C*C lattice (32.75 M arcs per utterance at T=2000, C=128).
 * transitions is the dense graph of criterion_test.cpp:316-326: node 0 start, nodes 1..C
 * accept, arcs 0 -> i+1 (label i, weight trans_w[i]) and j+1 -> i+1 (label i, weight
 * trans_w[C + i*C + j]).  paths_host [B][T]: the best path's labels (-1 where there is no
 * accepting path / beyond input_lens[b]); scores_host [B]: viterbiScore.  Paths are
 * bit-identical to the reference's, ties included.  Needs C <= 224 (GTNB_ERR_UNSUPPORTED
 * above: the C x C weights are held in shared memory).  The ASG kind of gtnb_viterbi_dense_ex
 * with host transitions and host outputs, with one known deviation from the reference kept
 * for compatibility: an utterance with input_lens[b] = 0 scores 0 here, -inf there.
 */
int gtnb_viterbi_dense(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens,
    const float* trans_w_host,
    int32_t* paths_host,
    float* scores_host);

/* graph kinds of gtnb_viterbi_dense_ex */
#define GTNB_DENSE_ASG 0 /* trans_w [C + C*C]: start weights, then W; gtnb_asg_loss_ex's layout */
#define GTNB_DENSE_BIGRAM 1 /* trans_w [C*C]: W alone, every state starts; gtnb_ngram_ctc_loss's layout */
#define GTNB_DENSE_CTC 2 /* no transitions (trans_w NULL): gtnb_ctc_loss's criterion; gtnb_beam_decode_async only */

/*
 * Batched Viterbi decoding with the learned transitions of gtnb_asg_loss_ex (kind GTNB_DENSE_ASG) or
 * gtnb_ngram_ctc_loss (kind GTNB_DENSE_BIGRAM), without materialising the T*C*C lattice:
 *   ASG:    viterbiPath / viterbiScore of compose(E_b, transitions), transitions as at gtnb_viterbi_dense;
 *   BIGRAM: viterbiPath / viterbiScore of intersect(E_b, G), G as at gtnb_ngram_ctc_loss (C nodes, every node
 *           start and accept, arc j -> i with label i and weight trans_w[i*C + j]).
 * E_b: linearGraph(T_b, C) on the first T_b = input_lens[b] (or T) rows of emissions_b ([B][T][C]); rows t >= T_b
 * are never read.  trans_w lives on the device when trans_on_device (read in place on the context's stream, never
 * copied to the host), else on the host; likewise emissions.  paths ([B][T], nullable): the labels of the best
 * path, -1 beyond T_b and where there is no accepting path; EVERY entry is written.  scores ([B], nullable):
 * viterbiScore, -inf without an accepting path.  Both live on the device when outputs_on_device: the call then
 * returns once the work is enqueued on the context's stream; host outputs are complete when it returns.
 * Ties go to the reference's choice (the smallest predecessor state, then the first best final state), so paths
 * and scores equal the reference's for finite emissions and finite or -inf weights (-inf forbids a transition).
 * NaN is never chosen as a maximum, so a NaN acts like -inf; the reference propagates it instead.
 * T_b = 0 gives score -inf and an all -1 path (linearGraph(0, C) accepts nothing).  Needs 1 <= C <= 224
 * (GTNB_ERR_UNSUPPORTED above); an unknown kind, input_lens outside [0, T] or a NULL ctx, emissions or trans_w is
 * GTNB_ERR_INVALID_ARGUMENT.  B = 0 is a no-op.
 */
int gtnb_viterbi_dense_ex(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* host, nullable */
    int kind,
    const float* trans_w,
    int trans_on_device,
    int32_t* paths, /* nullable */
    float* scores, /* nullable */
    int outputs_on_device);

/*
 * gtnb_viterbi_dense_ex on device buffers with emissions of a chosen element type: emissions_dev [B][T][C] of dtype
 * (GTNB_F32, GTNB_BF16 or GTNB_F16); trans_w_dev, paths_dev (nullable) and scores_dev (nullable) on the device, the
 * call returning once the work is enqueued.  The factored kernel (k_dense.cu) reads the 16-bit emissions in place and
 * widens each on load, so paths and scores are == gtnb_viterbi_dense_ex's on the emissions widened to float32, ties
 * included, for every batch.  GTNB_F32 is gtnb_viterbi_dense_ex with every buffer on the device; an unknown dtype is
 * GTNB_ERR_INVALID_ARGUMENT.
 */
int gtnb_viterbi_dense_typed(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const void* emissions_dev,
    int dtype,
    const int32_t* input_lens, /* host, nullable */
    int kind,
    const float* trans_w_dev,
    int32_t* paths_dev, /* nullable */
    float* scores_dev); /* nullable */

/*
 * Loss over one user-supplied target graph per utterance with a learned dense transition graph G (the word
 * decomposition and prior graphs of the reference's examples/learned_decompositions.cpp and examples/priors.cpp,
 * completed with the standard emissions and transitions graph):
 *   GTNB_DENSE_ASG:    loss_b = forwardScore(compose(E_b, G)) - forwardScore(compose(compose(A_b, G), E_b)),
 *                      G and trans_w ([C + C*C]) as at gtnb_asg_loss_ex / gtnb_viterbi_dense;
 *   GTNB_DENSE_BIGRAM: loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(A_b, G), E_b)),
 *                      G and trans_w ([C*C]) as at gtnb_ngram_ctc_loss.
 * E_b, graphs, arc_weights and the epsilon rule are those of gtnb_graph_loss: A_b is matched on its olabels, arcs
 * labelled outside [0, C) never match (gradient 0), an epsilon arc is GTNB_ERR_UNSUPPORTED.  Outputs: losses_host
 * [B]; grads (nullable, [B][T][C], d loss_b / d e_b), EVERY row written, 0 beyond T_b; arc_grads (nullable,
 * [sum_b A_b], d loss_b / d A_b's arc weights in Graph arc numbering) and trans_grad (nullable, the batch sum of
 * d loss_b / d trans_w), written, not accumulated.  Every buffer lives on the device or the host according to its
 * own *_on_device flag.  T_b = 0 gives NaN; a graph with no accepting path of T_b arcs, no start node or no arcs
 * gives +inf and the denominator's gradient alone.  B = 0 zeroes trans_grad.  T_b > T, negative lengths, an
 * unknown kind or a malformed view are GTNB_ERR_INVALID_ARGUMENT; C > 128 is GTNB_ERR_UNSUPPORTED.
 * The numerator compose(A_b, G) is built on the host from the graph's structure only; its weights are folded on
 * the device from the transitions where they lie, which on this route never visit the host.  It is swept without
 * building the lattice beside the dense trellis of the denominator.  Non-finite values, the "implicit" flag off, or
 * products too wide for the implicit layout (e.g. wildcard states at large C) take the materialised lattices.
 */
int gtnb_graph_transitions_loss(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* nullable */
    const gtnb_graph_view* graphs,
    const float* arc_weights, /* nullable */
    int arc_weights_on_device,
    int kind,
    const float* trans_w,
    int trans_on_device,
    float* losses_host,
    float* grads, /* nullable */
    int grads_on_device,
    float* arc_grads, /* nullable */
    int arc_grads_on_device,
    float* trans_grad, /* nullable */
    int trans_grad_on_device);

/*
 * Loss over one user-supplied target graph per utterance with a learned transition graph G of any shape (n-gram
 * graphs of any order, pruned or sparse token LMs, HMM topologies):
 *   loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(A_b, G), E_b)).
 * transitions: G's structure, an epsilon-free acceptor (ilabel == olabel on every arc) with any start and accept
 * sets, cycles and node count; its own weights are ignored.  trans_w: [G.num_arcs] weights in G's arc numbering.
 * E_b, graphs, arc_weights, the outputs and their *_on_device flags are those of gtnb_graph_transitions_loss;
 * trans_grad is [G.num_arcs], the batch sum, written, not accumulated.  An arc of A_b or G labelled outside [0, C)
 * never matches (gradient 0).  T_b = 0 gives NaN; no accepting path of T_b arcs through A_b and G gives +inf and the
 * denominator's gradient alone; a G that accepts nothing in T_b frames gives NaN.  B = 0 zeroes trans_grad.
 * Epsilon arcs in A_b or G, or a G that is a transducer, are GTNB_ERR_UNSUPPORTED (remove(g, epsilon), projectInput
 * / projectOutput first); malformed views, a G without nodes, bad lengths or a NULL trans_w with B > 0 are
 * GTNB_ERR_INVALID_ARGUMENT.
 * Device route (the transitions never visit the host): the denominator is swept over G's tables without building
 * the lattice (k_sparse.cu) when G fits the kernels' envelope -- at most 4096 nodes, 32768 arcs labelled in [0, C),
 * C <= 1024 -- and the numerators are the products of gtnb_product.h, built on the host from structure only, with
 * G's start copies folded into one start node, weighted on the device and swept by the implicit kernels.  A G or a
 * product outside that layout, a non-finite value, or the "implicit" flag off take the materialised lattices.
 * With the "sparse_cluster" flag at 1 a larger G (gtnb_ctx_set_flag: up to 16384 nodes / 262144 arcs, the full trigram
 * at C = 64) stays on the device route, swept by a thread-block cluster per utterance; its scratch grows with G's
 * node count S: 4 * B * (T + 1) * S bytes of score rows (1 GB at B = 128, T = 500, S = 4096), and a failed
 * allocation is GTNB_ERR_RUNTIME as on every route.
 */
int gtnb_sparse_transitions_loss(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* nullable */
    const gtnb_graph_view* graphs,
    const float* arc_weights, /* nullable */
    int arc_weights_on_device,
    const gtnb_graph_view* transitions,
    const float* trans_w,
    int trans_on_device,
    float* losses_host,
    float* grads, /* nullable */
    int grads_on_device,
    float* arc_grads, /* nullable */
    int arc_grads_on_device,
    float* trans_grad, /* nullable */
    int trans_grad_on_device);

/*
 * Batched Viterbi alignment over one user-supplied target graph per utterance: viterbiPath and viterbiScore of
 * compose(A_b, E_b), the best path through the user's own graph (a forced alignment with any topology; CTC graphs
 * give CTC forced alignment).  E_b, graphs, arc_weights, the olabel matching, labels outside [0, C) and the epsilon
 * rule are exactly those of gtnb_graph_loss.  The lattice is frame synchronous, so a path has exactly T_b arcs, one
 * per frame: paths ([B][T], nullable) gets the matched label of the arc taken at frame t, arcs ([B][T], nullable)
 * that arc's id in A_b (Graph arc numbering), both -1 beyond T_b and in every slot when there is no accepting path;
 * EVERY entry is written.  scores ([B], nullable): viterbiScore, -inf without an accepting path (T_b = 0 included:
 * linearGraph(0, C) accepts nothing; so do infeasible and empty graphs).  Outputs live on the device when
 * outputs_on_device, else on the host; emissions and arc_weights each where their own flag says.
 * Paths and scores equal the reference's, ties included: the frames are swept in the tropical semiring without
 * building the lattice and the path is traced back from the saved scores; an utterance whose traced path meets a
 * tie, or whose sweep meets a non-finite value, is re-run alone on the materialised lattice (gtnb_compose_linear,
 * gtnb_forward, gtnb_viterbi_path), as is the whole batch when the graphs do not fit the sweep's layout or the
 * "implicit" flag is off.  With "exact_ties" off a tie keeps the device route's path, which is then one of the
 * optimal paths.  The call reads back one status word per utterance to decide the route, so unlike
 * gtnb_viterbi_dense_ex it returns only once every output is complete, on the device ones too.
 * Malformed views, input_lens outside [0, T] or negative are GTNB_ERR_INVALID_ARGUMENT; an epsilon arc is
 * GTNB_ERR_UNSUPPORTED.  B = 0 is a no-op.
 */
int gtnb_graph_viterbi(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* host, nullable */
    const gtnb_graph_view* graphs,
    const float* arc_weights, /* nullable */
    int arc_weights_on_device,
    int32_t* paths, /* [B][T] nullable: matched label of the arc taken at frame t */
    int32_t* arcs, /* [B][T] nullable: that arc's id in A_b (Graph arc numbering) */
    float* scores, /* [B] nullable: viterbiScore */
    int outputs_on_device);

/*
 * Batched Viterbi alignment over one user-supplied target graph per utterance with a learned dense transition graph
 * G: viterbiPath and viterbiScore of the numerators of gtnb_graph_transitions_loss,
 *   GTNB_DENSE_ASG:    compose(compose(A_b, G), E_b),
 *   GTNB_DENSE_BIGRAM: intersect(intersect(A_b, G), E_b),
 * the decomposition and frame-level alignment a model trained with that loss picks.  G, trans_w's layouts, E_b,
 * graphs, arc_weights, the olabel matching, labels outside [0, C) and the epsilon rule are exactly those of
 * gtnb_graph_transitions_loss.  Outputs are those of gtnb_graph_viterbi: paths ([B][T], nullable) gets the label of
 * the arc taken at frame t, arcs ([B][T], nullable) that arc's id in A_b (Graph arc numbering), both -1 beyond T_b
 * and in every slot when there is no accepting path; EVERY entry is written.  scores ([B], nullable): viterbiScore,
 * -inf without an accepting path (T_b = 0, an empty graph, a graph with no start node and an infeasible graph
 * included).  Outputs live on the device when outputs_on_device, else on the host; emissions, arc_weights and
 * trans_w each where their own flag says.
 * Paths, arcs and scores equal the reference's, ties included.  The device route sweeps the loss's products in the
 * tropical semiring (BIGRAM's folded start arcs weigh tau_l = max_j W[l][j]) with the transitions on the device and
 * traces the path back; an utterance whose traced path meets a tie (with "exact_ties" on), or whose sweep meets a
 * non-finite value, is re-run alone on compose(A_b, G) built in the reference's numbering (gtnb_compose_graphs,
 * then gtnb_compose_linear, gtnb_forward, gtnb_viterbi_path), as is the whole batch when the products do not fit
 * the sweep's layout or the "implicit" flag is off; only that route reads the transitions to the host.  The call
 * reads back one status word per utterance, so it returns only once every output is complete, device ones too.
 * C > 128 and an epsilon arc are GTNB_ERR_UNSUPPORTED, as is a pair too large for gtnb_compose_graphs on the exact
 * route; an unknown kind, T_b > T, negative lengths or a malformed view are GTNB_ERR_INVALID_ARGUMENT.  B = 0 is a
 * no-op.
 */
int gtnb_graph_transitions_viterbi(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* host, nullable */
    const gtnb_graph_view* graphs,
    const float* arc_weights, /* nullable */
    int arc_weights_on_device,
    int kind, /* GTNB_DENSE_ASG | GTNB_DENSE_BIGRAM */
    const float* trans_w,
    int trans_on_device,
    int32_t* paths, /* [B][T] nullable: label of the arc taken at frame t */
    int32_t* arcs, /* [B][T] nullable: that frame's arc id in A_b (Graph arc numbering) */
    float* scores, /* [B] nullable: viterbiScore */
    int outputs_on_device);

/*
 * Batched Viterbi decoding with a learned transition graph G of any shape: viterbiPath and viterbiScore of
 * intersect(E_b, G), E_b = linearGraph(T_b, C) on the first T_b rows of utterance b -- the best label sequence under
 * the G a model trained with gtnb_sparse_transitions_loss learned (an n-gram graph of any order, a pruned token LM,
 * an HMM topology).  transitions and trans_w are exactly those of gtnb_sparse_transitions_loss: G's structure, an
 * epsilon-free acceptor whose own weights are ignored, and [G.num_arcs] weights in G's arc numbering; a G arc
 * labelled outside [0, C) never matches.  paths ([B][T], nullable) gets the label of frame t, arcs ([B][T], nullable)
 * the G arc taken at frame t (Graph arc numbering: the state sequence of an HMM topology), both -1 beyond T_b and in
 * every slot when there is no accepting path; EVERY entry is written.  scores ([B], nullable): viterbiScore, -inf
 * without an accepting path (T_b = 0 included: linearGraph(0, C) accepts nothing).  Outputs live on the device when
 * outputs_on_device, else on the host; emissions and trans_w each where their own flag says.  collapse the paths for
 * transcripts.
 * Paths, arcs and scores equal the reference's, ties included.  The device route sweeps G's tables frame by frame in
 * the tropical semiring without building the T_b * |G| lattice (k_sparse.cu) when G fits the kernels' envelope -- at
 * most 4096 nodes, 32768 arcs labelled in [0, C), C <= 1024 -- keeping a 16-bit back-pointer per frame and node
 * (2 * B * T * S bytes of scratch), and traces the path back.  An utterance whose traced path meets a tie (with
 * "exact_ties" on), or whose sweep meets a NaN or +inf (-inf only forbids an arc), is re-run on the materialised
 * lattice (gtnb_compose_linear with E_b first, gtnb_forward, gtnb_viterbi_path), as is the whole batch outside the
 * envelope or with the "implicit" flag off; only that route reads trans_w to the host, and it runs the utterances in
 * groups that fit the device memory.  With "exact_ties" off a tie keeps the device route's path, one of the optimal
 * paths.  The call reads back one status word per utterance, so it returns only once every output is complete,
 * device ones too.  With the "sparse_cluster" flag at 1 a larger G (gtnb_ctx_set_flag: up to 16384 nodes / 262144
 * arcs) keeps the device route, swept by a thread-block cluster per utterance with the same back-pointers (0.5 GB of
 * them at B = 128, T = 500, S = 4096) and the same retry rules.
 * Epsilon arcs or a transducer G, and a lattice too large to materialise for one utterance on the exact route, are
 * GTNB_ERR_UNSUPPORTED; a malformed view, a G without nodes, a NULL trans_w with B > 0 and input_lens outside [0, T]
 * are GTNB_ERR_INVALID_ARGUMENT.  B = 0 is a no-op.
 */
int gtnb_viterbi_sparse(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* host, nullable */
    const gtnb_graph_view* transitions, /* G: structure only, its own weights ignored */
    const float* trans_w, /* [G.num_arcs], G's arc numbering */
    int trans_on_device,
    int32_t* paths, /* [B][T] nullable: label of frame t */
    int32_t* arcs, /* [B][T] nullable: the G arc taken at frame t (Graph arc numbering) */
    float* scores, /* [B] nullable: viterbiScore */
    int outputs_on_device);

/*
 * Batched Viterbi alignment over one user-supplied target graph per utterance with a learned transition graph G of
 * any shape: viterbiPath and viterbiScore of intersect(intersect(A_b, G), E_b), the numerator of
 * gtnb_sparse_transitions_loss -- the decomposition and frame-level alignment a model trained with that loss picks.
 * E_b, graphs, arc_weights, transitions, trans_w, labels outside [0, C) and the epsilon rule are those of
 * gtnb_sparse_transitions_loss; the outputs, the routing and their rules are those of gtnb_graph_transitions_viterbi
 * (arcs: A_b's arc ids).  The device route sweeps the loss's folded products in the tropical semiring, G's start
 * copies folded into one start node whose arcs weigh tau_k = max over a group of G's start arcs, with trans_w on the
 * device; the exact route composes A_b with G in the reference's numbering (gtnb_compose_graphs).  The device route
 * is taken when G fits gtnb_viterbi_sparse's envelope ("sparse_cluster" at 1: its cluster envelope) and every product
 * the implicit sweeps' layout.
 * Epsilon arcs in A_b or G, a transducer G and a pair too large for the exact route are GTNB_ERR_UNSUPPORTED;
 * malformed views, a G without nodes, a NULL trans_w with B > 0 and bad lengths are GTNB_ERR_INVALID_ARGUMENT.
 * B = 0 is a no-op.
 */
int gtnb_sparse_transitions_viterbi(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* host, nullable */
    const gtnb_graph_view* graphs,
    const float* arc_weights, /* nullable */
    int arc_weights_on_device,
    const gtnb_graph_view* transitions, /* G: structure only, its own weights ignored */
    const float* trans_w, /* [G.num_arcs], G's arc numbering */
    int trans_on_device,
    int32_t* paths, /* [B][T] nullable: label of the arc taken at frame t */
    int32_t* arcs, /* [B][T] nullable: that frame's arc id in A_b (Graph arc numbering) */
    float* scores, /* [B] nullable: viterbiScore */
    int outputs_on_device);

/*
 * Loss with a backoff transition graph G: gtnb_sparse_transitions_loss with epsilon arcs allowed in G, the backoff
 * arcs of a pruned n-gram token LM (each history state has arcs for the labels seen after it and one epsilon arc to
 * its shorter history), composed natively instead of removed:
 *   loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(A_b, G), E_b)).
 * An epsilon arc of G has ilabel == olabel == GTNB_EPSILON.  It moves G without consuming a frame, at any frame
 * 0 .. T_b (leaving a start node at frame 0 and reaching an accept node at frame T_b included), weighs trans_w[arc]
 * alone, and gets its gradient in trans_grad (none in the emission gradient).  The score sums over every path, the
 * backoff paths included, as the reference's does.  Arguments, outputs and every other rule are those of
 * gtnb_sparse_transitions_loss, and an epsilon-free G gives exactly its results.  A cycle of epsilon arcs in G is
 * GTNB_ERR_INVALID_ARGUMENT (the message names it); epsilon arcs in A_b, an arc with epsilon on one side only and a
 * transducer G are GTNB_ERR_UNSUPPORTED.
 * Device route (k_sparse.cu's backoff sweeps): G's epsilon arcs are put in topological levels, and every frame's
 * scores are closed over them one level per CTA barrier.  The denominator sweeps G's tables; the numerators
 * A_b o G (built on the host from structure only, with G's epsilon arcs) sweep their own tables, one CTA each, with
 * weights gathered on the device.  The envelope, for G and for every numerator: at most 4096 nodes, 32768 emitting
 * plus epsilon arcs, 32 levels (the longest chain of epsilon arcs; a backoff n-gram of order n has n - 1), C <= 1024.
 * Outside it, with a non-finite value or with the "implicit" flag off, the exact route composes E_b with G and the
 * numerators with E_b (gtnb_compose_graphs) and runs the materialised lattices utterance by utterance.
 * With the "sparse_cluster" flag at 1 a larger G (gtnb_ctx_set_flag: up to 16384 nodes / 262144 emitting plus epsilon
 * arcs) keeps the device route, its denominator swept by a thread-block cluster per utterance; the scratch grows with
 * G's nodes S: alpha is 4 * B * (T + 1) * S bytes (2.2 GB for a backoff 4-gram of 8563 states at B = 128, T = 500).
 */
int gtnb_backoff_transitions_loss(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* nullable */
    const gtnb_graph_view* graphs,
    const float* arc_weights, /* nullable */
    int arc_weights_on_device,
    const gtnb_graph_view* transitions, /* G: structure only, epsilon arcs allowed; its own weights ignored */
    const float* trans_w, /* [G.num_arcs], G's arc numbering */
    int trans_on_device,
    float* losses_host,
    float* grads, /* nullable */
    int grads_on_device,
    float* arc_grads, /* nullable */
    int arc_grads_on_device,
    float* trans_grad, /* nullable */
    int trans_grad_on_device);

/*
 * Batched Viterbi decoding with a backoff transition graph G: gtnb_viterbi_sparse with epsilon arcs allowed in G
 * (gtnb_backoff_transitions_loss's G and epsilon rule), viterbiPath / viterbiScore of intersect(E_b, G).  An epsilon
 * arc uses no frame and is not reported: paths[b][t] / arcs[b][t] are the label and the emitting G arc taken at
 * frame t.  Scores are bit-exact, and paths, arcs and scores equal the reference's, ties included.  Outputs, routing
 * and their rules are gtnb_viterbi_sparse's, and an epsilon-free G gives exactly its results.  The device route
 * sweeps G's tables in the tropical semiring with the epsilon closure after every frame and keeps a 16-bit
 * back-pointer per frame and node (2 * B * (T + 1) * S bytes of scratch), which indexes the node's emitting in-arcs
 * from the frame before, then its epsilon in-arcs from the same frame; the trace follows epsilon back-pointers
 * inside a frame.  Its envelope is gtnb_backoff_transitions_loss's.  An utterance with a tie on its traced path
 * ("exact_ties" on) or a NaN or +inf is re-run on compose(E_b, G) (gtnb_compose_graphs, gtnb_forward,
 * gtnb_viterbi_path), as is the whole batch outside the envelope or with the "implicit" flag off.
 * With the "sparse_cluster" flag at 1 a larger G (up to 16384 nodes / 262144 emitting plus epsilon arcs) keeps the
 * device route, swept by a thread-block cluster per utterance with the same back-pointers (1.1 GB for a backoff 4-gram
 * of 8563 states at B = 128, T = 500).
 * Error rules are gtnb_backoff_transitions_loss's for G and gtnb_viterbi_sparse's otherwise.
 */
int gtnb_viterbi_backoff(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* host, nullable */
    const gtnb_graph_view* transitions, /* G: structure only, epsilon arcs allowed; its own weights ignored */
    const float* trans_w, /* [G.num_arcs], G's arc numbering */
    int trans_on_device,
    int32_t* paths, /* [B][T] nullable: label of frame t */
    int32_t* arcs, /* [B][T] nullable: the emitting G arc taken at frame t (Graph arc numbering) */
    float* scores, /* [B] nullable: viterbiScore */
    int outputs_on_device);

/*
 * Batched Viterbi alignment over one user-supplied target graph per utterance with a backoff transition graph G:
 * viterbiPath and viterbiScore of intersect(intersect(A_b, G), E_b), the numerator of gtnb_backoff_transitions_loss --
 * the decomposition and frame-level alignment a model trained with that loss picks, under the LM it was trained with.
 * paths[b][t] is the label of the emitting arc taken at frame t and arcs[b][t] that arc's id in A_b; an epsilon arc of
 * G uses no frame and is not reported, at frame 0 and after frame T_b included.  Every other output rule is
 * gtnb_sparse_transitions_viterbi's (-1 beyond T_b and for an utterance without an accepting path, score -inf, every
 * entry written), and an epsilon-free G gives exactly its results.  Error rules for G are
 * gtnb_backoff_transitions_loss's, all others gtnb_sparse_transitions_viterbi's.
 * Device route: the loss's numerators A_b o G (built on the host from structure only, with G's epsilon arcs) are
 * swept in the tropical semiring one CTA each, with the epsilon closure after every frame and bit-exact scores, and
 * keep a 16-bit back-pointer per frame and node (2 * sum over b of (T_b + 1) * S_b bytes of scratch, S_b the
 * numerator's nodes); the trace reports A_b's arcs.  Its envelope is gtnb_backoff_transitions_loss's, for every
 * numerator.  An utterance with a tie on its traced path ("exact_ties" on) or a NaN or +inf is re-run on
 * compose(compose(A_b, G), E_b) (gtnb_compose_graphs, gtnb_forward, gtnb_viterbi_path), as is the whole batch outside
 * the envelope or with the "implicit" flag off; only that route reads trans_w to the host.  With the "sparse_cluster"
 * flag at 1 a G beyond the one-CTA envelope (up to gtnb_viterbi_backoff's cluster envelope) keeps the device route:
 * the alignment sweeps the numerators alone, so only the gate changes.
 */
int gtnb_backoff_transitions_viterbi(
    gtnb_ctx* ctx,
    int B,
    int T,
    int C,
    const float* emissions,
    int emissions_on_device,
    const int32_t* input_lens, /* host, nullable */
    const gtnb_graph_view* graphs,
    const float* arc_weights, /* nullable */
    int arc_weights_on_device,
    const gtnb_graph_view* transitions, /* G: structure only, epsilon arcs allowed; its own weights ignored */
    const float* trans_w, /* [G.num_arcs], G's arc numbering */
    int trans_on_device,
    int32_t* paths, /* [B][T] nullable: label of the emitting arc taken at frame t */
    int32_t* arcs, /* [B][T] nullable: that frame's arc id in A_b (Graph arc numbering) */
    float* scores, /* [B] nullable: viterbiScore */
    int outputs_on_device);

/*
 * A transition graph prepared once for decoding without a host synchronisation (gtnb_viterbi_transitions_async): G's
 * tables packed and uploaded into device memory the handle owns, with the route chosen for them.
 * gtnb_transitions_create checks G as the synchronous decoder it stands for does: backoff 0 as gtnb_viterbi_sparse
 * (epsilon arcs refused), backoff 1 as gtnb_viterbi_backoff (epsilon arcs allowed, a cycle of them refused; an
 * epsilon-free G then takes gtnb_viterbi_sparse's tables).  The route is picked from ctx's flags at creation, as the
 * synchronous decoders pick it per call: "sparse_cluster" (1, or a forced 2 / 4 / 8) lets a G beyond one CTA take a
 * thread-block cluster.  A G outside every device route, or the "implicit" flag at 0, is GTNB_ERR_UNSUPPORTED: decode
 * with gtnb_viterbi_sparse / gtnb_viterbi_backoff instead.  The handle records its device, C, G's arc count (the
 * length of trans_w) and node count; it holds no weights, which stay a per-call argument since they are learned.
 * create allocates, uploads and synchronises: it is a set-up call and may not be captured into a CUDA graph.  A
 * captured graph that decodes with a handle must not be replayed after gtnb_transitions_destroy (which frees the
 * tables; ctx must be a context of the handle's device).
 */
typedef struct gtnb_transitions gtnb_transitions;
int gtnb_transitions_create(gtnb_ctx* ctx, const gtnb_graph_view* G, int C, int backoff, gtnb_transitions** out);
void gtnb_transitions_destroy(gtnb_ctx* ctx, gtnb_transitions* G);

/*
 * Viterbi decoding with a prepared transition graph, without a host synchronisation: viterbiPath / viterbiScore of
 * intersect(E_b, G), the decode of gtnb_viterbi_sparse (G made with backoff 0) or gtnb_viterbi_backoff (backoff 1).
 * The contract is gtnb_ctc_loss_async's: the call enqueues kernel launches on cuda_stream (NULL: the CUDA default
 * stream) and returns, without a host synchronisation, a read of device data on the host, an allocation or a staging
 * copy; it may be captured into a CUDA graph.  Scratch memory is workspace_dev (256-byte aligned, at least
 * gtnb_viterbi_transitions_async_workspace's bytes for the same handle and bounds; smaller is
 * GTNB_ERR_INVALID_ARGUMENT).  It holds 16-bit back-pointers sized from the bounds: 2 * B * T * S bytes, or
 * 2 * B * (T + 1) * S with epsilon arcs.  A handle made on another device is GTNB_ERR_INVALID_ARGUMENT.  Emissions
 * are float32 only, as the synchronous decoders take them (dtype is not a parameter).
 *
 * emissions_dev [B][T][C] float32; input_lens_dev [B] (NULL: T each); trans_w_dev [G arcs] float32.  Outputs, written
 * on the device:
 *   paths_dev [B][T]            the label of every frame of the best path;
 *   arcs_dev [B][T] (nullable)  the emitting G arc taken at every frame (an epsilon arc uses no frame);
 *                               both -1 beyond T_b and wherever no path accepts;
 *   scores_dev [B]              viterbiScore: -inf for T_b = 0 or no accepting path;
 *   status_dev [B] (nullable)   0  the synchronous decoder's result on the same data, bit for bit (exact_ties on);
 *                               1  a NaN or +inf weight or used emission (the synchronous decoder re-runs such an
 *                                  utterance on its exact route): a NaN score and -1 rows;
 *                               2  input_lens_dev[b] outside [0, T]: a NaN score and -1 rows;
 *                               3  a tie on the path or between best accept states: the score is the synchronous
 *                                  decoder's and the path an optimal one, the synchronous decoder's with exact_ties
 *                                  off.
 * A flagged utterance never affects the others.  A -inf weight only forbids its arc.
 */
int gtnb_viterbi_transitions_async_workspace(gtnb_ctx* ctx, const gtnb_transitions* G, int B, int T, size_t* bytes);
int gtnb_viterbi_transitions_async(
    gtnb_ctx* ctx,
    void* cuda_stream,
    const gtnb_transitions* G,
    int B,
    int T,
    const float* emissions_dev, /* [B][T][C] */
    const int32_t* input_lens_dev, /* [B] or NULL */
    const float* trans_w_dev, /* [G arcs] */
    int32_t* paths_dev, /* [B][T] */
    int32_t* arcs_dev, /* [B][T] or NULL */
    float* scores_dev, /* [B] */
    int32_t* status_dev, /* [B] or NULL */
    void* workspace_dev,
    size_t workspace_bytes);

/*
 * gtnb_viterbi_dense_typed without a host synchronisation, under gtnb_viterbi_transitions_async's contract: the
 * factored dense-trellis decode of kind GTNB_DENSE_ASG / GTNB_DENSE_BIGRAM with device lengths.  Emissions of dtype
 * GTNB_F32, GTNB_BF16 or GTNB_F16 are read in place.  paths_dev [B][T] (nullable: the paths then go to the workspace),
 * scores_dev [B] (-inf for T_b = 0).  status_dev [B] (nullable): 0 the synchronous call's result, ties broken as the
 * reference breaks them and NaN read as -inf, as there; 2 input_lens_dev[b] outside [0, T], with a NaN score and -1
 * rows.  The kernel's bounds (C <= 224 for the transition tile) and an unknown dtype are GTNB_ERR_UNSUPPORTED, as in
 * the other asynchronous calls; an unknown kind is GTNB_ERR_INVALID_ARGUMENT.
 */
int gtnb_viterbi_dense_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int dtype, int kind, size_t* bytes);
int gtnb_viterbi_dense_async(
    gtnb_ctx* ctx,
    void* cuda_stream,
    int B,
    int T,
    int C,
    const void* emissions_dev, /* [B][T][C] of dtype */
    int dtype,
    const int32_t* input_lens_dev, /* [B] or NULL */
    int kind, /* GTNB_DENSE_ASG | GTNB_DENSE_BIGRAM */
    const float* trans_w_dev, /* ASG [C + C*C], BIGRAM [C*C] */
    int32_t* paths_dev, /* [B][T] or NULL */
    float* scores_dev, /* [B] */
    int32_t* status_dev, /* [B] or NULL */
    void* workspace_dev,
    size_t workspace_bytes);

/*
 * Batched Levenshtein distance between padded hypotheses and references, under gtnb_ctc_loss_async's contract: the
 * call enqueues kernel launches on cuda_stream (NULL: the CUDA default stream) and nothing else -- no memset, no copy,
 * no host wait -- so it may be captured into a CUDA graph.
 * Pair b compares hyp_dev[b][0 .. hyp_lengths_dev[b]) ([B][N]) against ref_dev[b][0 .. ref_lengths_dev[b]) ([B][M]).
 * word_sep < 0: a unit is a token.  word_sep >= 0: a unit is a word, a maximal run of tokens other than word_sep
 * (leading, trailing and repeated separators make no empty word); two words are equal when their token spans are.
 * The distance is the unit-cost edit distance, -viterbiScore(compose(x, compose(edits, y))) of the reference's
 * examples/edit_distance.cpp over the units.  With i hypothesis units and j reference units,
 *   D[i][j] = min(D[i-1][j-1] + (h_i != r_j), D[i-1][j] + 1 (an insertion), D[i][j-1] + 1 (a deletion)),
 * and every cell picks one predecessor, preferring the diagonal, then a deletion, then an insertion.  The counts and
 * the alignment are those of the chain of chosen predecessors from the last cell: an optimal path of the reference's
 * lattice, not necessarily the one its viterbiPath returns.
 * Outputs: distance_dev [B]; ops_dev [B][3] substitutions, insertions, deletions (summing to the distance);
 * units_dev [B][2] hypothesis and reference units (the reference count is the error rate's denominator); status_dev
 * [B] 0, or 2 for a length outside [0, N] or [0, M], which gets -1 in every scalar and -1 rows (other pairs are
 * unaffected).  hyp_align_dev [B][N] (nullable): per hypothesis unit the index of the reference unit it is aligned
 * to, -1 for an insertion; ref_align_dev [B][M] (nullable): per reference unit the hypothesis unit, -1 for a deletion;
 * both -1 beyond the unit counts.  Indices count units: words in word mode.
 * N, M <= 4096 (GTNB_ERR_UNSUPPORTED above).  Scratch memory is workspace_dev (256-byte aligned, at least
 * gtnb_edit_distance_async_workspace's bytes for the same bounds; smaller is GTNB_ERR_INVALID_ARGUMENT).  Without an
 * alignment pointer it is 0 bytes and workspace_dev may be NULL.  With one it holds the 2-bit move of every grid
 * cell: with rows = min(n, m) and cols = max(n, m), where n = N and m = M in token mode and n = (N + 1) / 2 and
 * m = (M + 1) / 2 in word mode, K the least of 1, 2, 4, 8, 16 with 32 K >= rows (else 16) and W = ceil(rows / 32K),
 *   bytes = 256-byte roundup(4 * (B * W * (cols + 31) * 32 + 16)),
 * which is B * 2 bits * 512 W * (cols + 31): about 2 bits per cell per pair at the bounds.  B = 0 is a no-op.
 */
int gtnb_edit_distance_async_workspace(gtnb_ctx* ctx, int B, int N, int M, int word_sep, int with_alignment,
                                       size_t* bytes);
int gtnb_edit_distance_async(
    gtnb_ctx* ctx,
    void* cuda_stream,
    int B,
    const int32_t* hyp_dev, /* [B][N] */
    int N,
    const int32_t* hyp_lengths_dev, /* [B] */
    const int32_t* ref_dev, /* [B][M] */
    int M,
    const int32_t* ref_lengths_dev, /* [B] */
    int word_sep,
    int32_t* distance_dev, /* [B] */
    int32_t* ops_dev, /* [B][3]: substitutions, insertions, deletions */
    int32_t* units_dev, /* [B][2]: hypothesis, reference */
    int32_t* status_dev, /* [B] */
    int32_t* hyp_align_dev, /* [B][N] or NULL */
    int32_t* ref_align_dev, /* [B][M] or NULL */
    void* workspace_dev,
    size_t workspace_bytes);

/*
 * Batched prefix beam search over transcripts, scored by the training criterion, under gtnb_ctc_loss_async's contract:
 * the call enqueues kernel launches on cuda_stream (NULL: the CUDA default stream) and nothing else -- no memset, no
 * copy, no allocation, no host wait -- so it may be captured into a CUDA graph.
 *
 * Kinds and scores.  For utterance b with T_b = input_lens_dev[b] (NULL: T) frames of emissions_dev [B][T][C], the
 * score of a transcript y (tokens in [0, C), no blanks) is the log-semiring numerator of the matching loss, the value
 * its loss_b is denominator_b - numerator_b of:
 *   GTNB_DENSE_CTC     forwardScore(intersect(ctcGraph(y), E_b)) of gtnb_ctc_loss (trans_w_dev NULL).  A beam
 *                      carries p_blank and p_label, the two numerator states after the last frame; repeating the
 *                      last token needs a blank in between; the empty prefix starts with weight 0.
 *   GTNB_DENSE_BIGRAM  forwardScore(intersect(intersect(ctc_y, G), E_b)) of gtnb_ngram_ctc_loss, trans_w_dev [C*C] in
 *                      its layout.  G's state is the previous frame's label, so every move weighs W[dst][src] with src
 *                      blank or the last token, and the two states track G exactly.  Frame 0 enters label i from G's
 *                      C start states with sigma_i = logsumexp_j W[i][j].
 *   GTNB_DENSE_ASG     forwardScore(compose(compose(A_y, G), E_b)) of gtnb_asg_loss_ex, trans_w_dev [C + C*C] in its
 *                      layout.  One state per prefix, whose last frame's label is the last token: a frame stays
 *                      (W[last][last]) or appends any token c, c == last included, which makes a repeated token as
 *                      A_y does (W[c][last]); frame 0 appends c with the start weight of c.  blank is unused.
 * Every kind's accepting states weigh 0, so a transcript's end weight is 0.
 *
 * Search.  Frame-synchronous prefix beam search with K = beam beams.  At every frame the candidates are each beam
 * kept (blank / repeat / stay) and each beam extended by each non-blank token (every token for ASG).  An extension
 * whose transcript is already a live beam is merged into it (log-add), never kept twice: two live beams never hold
 * the same transcript.  All C tokens are considered: no per-frame token pruning, no LM weight, no insertion bonus.
 * Candidates are ranked by score descending; among equal scores kept beams come before extensions, then the lower
 * previous slot wins, then the lower token.  A candidate of score -inf is not kept.  The N = nbest hypotheses are the
 * top N live beams after frame T_b - 1, in the same order.  Scores are lower bounds: a returned score sums only the
 * alignments that survived the beam, so score <= numerator(y), with equality when no prefix was ever pruned.
 *
 * Outputs, written on the device:
 *   tokens_dev [B][N][T]   each hypothesis's transcript, followed by -1;
 *   lengths_dev [B][N]     its length;
 *   scores_dev [B][N]      its score (float32);
 *   status_dev [B]         (nullable) 0 a result;
 *                          1 a NaN or +inf in an emission of a row t < T_b, or (T_b >= 1, kinds with transitions)
 *                            anywhere in trans_w_dev: NaN scores, -1 lengths and rows.  A -inf value only forbids its
 *                            move;
 *                          2 input_lens_dev[b] outside [0, T]: NaN scores, -1 lengths and rows;
 *                          3 a tie decided the beam (equal scores at the K-th / (K+1)-th boundary of a frame) or the
 *                            N-best order (equal scores between consecutive hypotheses, or the N-th and (N+1)-th
 *                            beam): the results stand, chosen by the tie rule.
 * Unused hypotheses (fewer live transcripts than N) get score -inf, length -1 and -1 rows.  T_b = 0 gives one
 * hypothesis, the empty transcript with score 0 (the empty sum over no frames).  For CTC that is the numerator of
 * the empty target in gtnb_ctc_loss, whose loss there is 0.  gtnb_ngram_ctc_loss and gtnb_asg_loss_ex give NaN at
 * T_b = 0 instead (their linearGraph(0, C) accepts nothing): the decoder does not follow them.  A flagged utterance
 * never affects the others.  Results do not vary from run to run.
 *
 * Bounds: 1 <= beam <= 64, 1 <= nbest <= beam, 1 <= C <= 256 for every kind; emissions of dtype GTNB_F32, GTNB_BF16
 * or GTNB_F16 are read in place and widened on load.  Beyond them, or an unknown dtype: GTNB_ERR_UNSUPPORTED.  A NULL
 * pointer where B > 0 needs one, trans_w_dev given for GTNB_DENSE_CTC or missing for the other kinds, an unknown kind
 * or negative sizes: GTNB_ERR_INVALID_ARGUMENT.  blank outside [0, C) for CTC or BIGRAM: GTNB_ERR_UNSUPPORTED, as
 * gtnb_ctc_align_async treats it.  B = 0 is a no-op.
 *
 * Scratch memory is workspace_dev (256-byte aligned, at least gtnb_beam_decode_async_workspace's bytes for the same
 * bounds; smaller is GTNB_ERR_INVALID_ARGUMENT).  With r(x) = x rounded up to a multiple of 256,
 *   bytes = r(2 * (B * max(T, 1) * beam + 16))                                  (16-bit back-pointers)
 *         + (kind != GTNB_DENSE_CTC ? r(4 * (C*C + 16)) + 2 * r(4 * (C + 16)) : 0)   (transposed W, sigma, flags).
 *
 * Out of scope: beam search with a gtnb_transitions graph (sparse or backoff G: a prefix's state there is a
 * distribution over G's nodes, not two numbers), and lexicons and word-level search.  LM shallow fusion, an
 * insertion bonus and per-frame token pruning are gtnb_beam_decode_lm_async's.
 */
int gtnb_beam_decode_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int dtype, int kind, int beam, int nbest,
                                     size_t* bytes);
int gtnb_beam_decode_async(
    gtnb_ctx* ctx,
    void* cuda_stream,
    int B,
    int T,
    int C,
    const void* emissions_dev, /* [B][T][C] of dtype */
    int dtype,
    const int32_t* input_lens_dev, /* [B] or NULL */
    int kind, /* GTNB_DENSE_CTC | GTNB_DENSE_BIGRAM | GTNB_DENSE_ASG */
    const float* trans_w_dev, /* NULL, BIGRAM [C*C], ASG [C + C*C] */
    int blank,
    int beam,
    int nbest,
    int32_t* tokens_dev, /* [B][nbest][T] */
    int32_t* lengths_dev, /* [B][nbest] */
    float* scores_dev, /* [B][nbest] */
    int32_t* status_dev, /* [B] or NULL */
    void* workspace_dev,
    size_t workspace_bytes);

/*
 * A token n-gram LM prepared once for gtnb_beam_decode_lm_async.  lm is a gtn graph over the tokens that must be
 *   - an acceptor (ilabel == olabel), labelled in [0, C] or GTNB_EPSILON; label C is end of sentence;
 *   - with exactly one start node (node flags other than start are ignored);
 *   - with at most one arc per (node, label) and at most one epsilon arc per node, and no cycle of epsilon arcs;
 *   - free of NaN and +inf weights (a -inf weight is allowed and forbids its arc).
 * Anything else is GTNB_ERR_INVALID_ARGUMENT.  Epsilon arcs are backoff (failure) arcs, as in ARPA: one is taken only
 * when the node has no arc for the token, unlike the log-semiring sum over epsilon paths of
 * gtnb_backoff_transitions_loss.  From node s, token c resolves to
 *   - the arc of s labelled c, if s has one;
 *   - otherwise the weight of s's epsilon arc plus the resolution of c from that arc's destination;
 *   - -inf if neither exists.
 * LM(y) is the sum of the resolved weights along y from the start node, plus the end weight of the node reached: the
 * resolved weight of label C, or 0 for every node when the graph has no arc labelled C at all.  For an epsilon-free
 * LM, LM(y) is forwardScore(compose(linear(y [+ C]), lm)).
 * The handle holds the resolved table on the device, weight [S][C + 1] float32 and destination [S][C + 1] int32, built
 * on the host in order of backoff depth and uploaded once.  Unlike gtnb_transitions it bakes the weights in:
 * resolution sums backoff weights into the table, and a fusion LM is not trained.  Bounds: S * (C + 1) <= 2^25
 * entries (256 MB) and C <= 256, else GTNB_ERR_UNSUPPORTED.  create allocates, uploads and synchronises: it is a
 * set-up call and may not be captured.  A captured graph that decodes with the LM must not be replayed after
 * gtnb_lm_destroy (ctx must be a context of the handle's device).
 */
typedef struct gtnb_lm gtnb_lm;
int gtnb_lm_create(gtnb_ctx* ctx, const gtnb_graph_view* lm, int C, gtnb_lm** out);
void gtnb_lm_destroy(gtnb_ctx* ctx, gtnb_lm* lm);

/*
 * gtnb_beam_decode_async with LM shallow fusion, an insertion bonus and per-frame token pruning, under its contract:
 * the same parameters, kinds (CTC, BIGRAM, ASG), dtypes, tie rule, status codes, bounds and workspace formula
 * (gtnb_beam_decode_lm_async_workspace returns gtnb_beam_decode_async_workspace's bytes); it only launches kernels
 * and may be captured.  The LM acts on the transcript only, so it is independent of the kind.
 *
 * Each beam also carries its LM node and lmacc, the unweighted sum (float32) of its resolved LM weights.
 *   - Ranking key: logsumexp(p_blank, p_label) + (lm_weight * lmacc + token_bonus * len), in that float32 order.  An
 *     extension by c from node s adds the resolved w(s, c) to lmacc; a -inf weight forbids the move for any
 *     lm_weight.  A merged extension has the same transcript, hence the same node and lmacc: only the acoustic states
 *     log-add.
 *   - After frame T_b - 1 each live beam adds its end weight; a beam whose end weight is -inf is dropped.  The N-best
 *     are the top N live beams by the final fused score, ties to the earlier beam (the tie rule's order); status 3
 *     also covers equal final scores between consecutive hypotheses.
 *   - token_beam = P in [1, C]: at each frame extensions use only the P tokens of highest emission (blank excluded
 *     for CTC and BIGRAM); kept moves (blank, repeat, stay) are never pruned.  Equal emissions at the P-th boundary go
 *     to the lower token and, when finite, flag status 3.  P = C means no pruning.  When r's last token was pruned at
 *     a frame, the extension (par[r], last[r]) is simply absent.  Scores stay lower bounds.
 *   - lm NULL: every resolved weight and end weight is 0.
 * Outputs: scores_dev [B][N] am + lm_weight * lm + token_bonus * len (float32, the order above);
 * am_scores_dev [B][N] (nullable) the acoustic lower bound, as gtnb_beam_decode_async returns it; lm_scores_dev
 * [B][N] (nullable) LM(y).  Each is -inf for unused hypotheses and NaN for status 1 and 2.  T_b = 0 gives the empty
 * transcript with am 0 and lm the start node's end weight, or no hypothesis when that is -inf.
 * Errors: lm_weight negative or not finite, token_bonus not finite, or an LM made on another device or for another C:
 * GTNB_ERR_INVALID_ARGUMENT.  token_beam outside [1, C]: GTNB_ERR_UNSUPPORTED, like the other bounds.
 * With lm NULL, token_bonus 0 and token_beam = C, tokens, lengths, scores and status are == gtnb_beam_decode_async's.
 *
 * Out of scope: C > 256 (which pruning makes possible later: the candidates are K * P, not K * C).  Lexicons,
 * word-level search and word LMs beyond the dense table are gtnb_beam_decode_lexicon_async's.
 */
int gtnb_beam_decode_lm_async_workspace(gtnb_ctx* ctx, int B, int T, int C, int dtype, int kind, int beam, int nbest,
                                        int token_beam, size_t* bytes);
int gtnb_beam_decode_lm_async(
    gtnb_ctx* ctx,
    void* cuda_stream,
    int B,
    int T,
    int C,
    const void* emissions_dev, /* [B][T][C] of dtype */
    int dtype,
    const int32_t* input_lens_dev, /* [B] or NULL */
    int kind, /* GTNB_DENSE_CTC | GTNB_DENSE_BIGRAM | GTNB_DENSE_ASG */
    const float* trans_w_dev, /* NULL, BIGRAM [C*C], ASG [C + C*C] */
    int blank,
    int beam,
    int nbest,
    const gtnb_lm* lm, /* or NULL */
    float lm_weight,
    float token_bonus,
    int token_beam,
    int32_t* tokens_dev, /* [B][nbest][T] */
    int32_t* lengths_dev, /* [B][nbest] */
    float* scores_dev, /* [B][nbest] */
    float* am_scores_dev, /* [B][nbest] or NULL */
    float* lm_scores_dev, /* [B][nbest] or NULL */
    int32_t* status_dev, /* [B] or NULL */
    void* workspace_dev,
    size_t workspace_bytes);

/*
 * A lexicon with an optional word n-gram LM, prepared once for gtnb_beam_decode_lexicon_async.
 *   - token_class[c], c in [0, C): 0 an in-word token; 1 a separator (such as wav2letter's "|"), which ends the current
 *     word and belongs to no spelling; 2 a word-start token (such as a SentencePiece piece with a leading space), which
 *     ends the current word and begins a new spelling.
 *   - num_spellings spellings: spelling i is spelling_tokens[spelling_offsets[i] .. spelling_offsets[i + 1]), a
 *     non-empty token sequence, and spells word spelling_words[i] in [0, V).  A word may have several spellings; two
 *     words may not share one (no homophones).  A separator may not appear in a spelling, a word-start token only at
 *     its position 0.
 *   - word_lm (nullable): gtnb_lm_create's graph contract over the labels [0, V], label V being end of sentence: an
 *     acceptor with one start node, at most one arc per (node, label), at most one epsilon (backoff) arc per node, no
 *     cycle of epsilon arcs, no NaN or +inf weight.  w(s, x) is the arc of s labelled x if there is one, else s's
 *     backoff weight plus w(backoff destination, x), added innermost first as gtnb_lm_create's table adds them, else
 *     -inf.  A node's end weight is w(s, V), or 0 for every node when the graph has no arc labelled V.  NULL: every
 *     weight is 0.
 *   - Lookahead: smear(n) is the largest finite w(start, word) over the words spelled at or below trie node n; 0 when
 *     none is finite, at the root, and without a word LM (flashlight's max-unigram smearing).  It only steers the
 *     search: returned scores never include it.
 * Breaking any of these rules, a token outside [0, C) or an empty spelling is GTNB_ERR_INVALID_ARGUMENT.
 * Bounds: C <= 256, V <= 2^20 words, a trie of at most 2^24 nodes (the root and one per distinct spelling prefix), a
 * word LM of at most 2^26 arcs and 2^26 nodes; beyond them GTNB_ERR_UNSUPPORTED.
 * Device bytes, each term rounded up to 256: 4C (classes) + 4 * nodes * ceil(C / 32) (child masks) + 3 * 4 * nodes
 * (first child, word id, smear) and, with a word LM of S nodes and A arcs of labels below V, 16H (an open-addressing
 * hash of those arcs, H the least power of two >= max(2, 2A)) + 3 * 4S (backoff weight and destination, end weight).
 * create allocates, uploads and synchronises: it is a set-up call and may not be captured.  A captured graph that
 * decodes with the lexicon must not be replayed after gtnb_lexicon_destroy (ctx must be a context of its device).
 */
typedef struct gtnb_lexicon gtnb_lexicon;
int gtnb_lexicon_create(gtnb_ctx* ctx, int C, const int32_t* token_class /* [C] */, int V, int num_spellings,
                        const int32_t* spelling_offsets /* [num_spellings + 1] */, const int32_t* spelling_tokens,
                        const int32_t* spelling_words /* [num_spellings] */,
                        const gtnb_graph_view* word_lm /* or NULL */, gtnb_lexicon** out);
void gtnb_lexicon_destroy(gtnb_ctx* ctx, gtnb_lexicon* lexicon);

/*
 * Lexicon-constrained prefix beam search with a word LM: gtnb_beam_decode_lm_async under its contract (parameters,
 * kinds CTC, BIGRAM and ASG, dtypes, tie rule, status codes, token_beam P, bounds, workspace: size it with
 * gtnb_beam_decode_lm_async_workspace), with lexicon in place of the LM and word_bonus in place of token_bonus.  It
 * only launches kernels and may be captured.
 *
 * Each beam also carries a trie node (the root: no pending word), a word-LM node, lmacc (the float32 sum of its
 * completed words' w) and its word count, all functions of the transcript, so a merged extension stays exact.
 *   - Extending a beam at trie node n by token c: an in-word c moves to n's child labelled c, and is forbidden
 *     without one.  A separator changes nothing at the root; at a word end it completes the word and returns to the
 *     root; anywhere else it is forbidden.  A word-start c, at the root or at a word end (completing that word first),
 *     moves to the root's child labelled c; it is forbidden without that child or when n is neither.  Completing word
 *     x adds w(LM node, x) to lmacc, moves the LM node and adds 1 to the word count; a -inf weight forbids the move.
 *     Kept moves (blank, repeat, stay) change none of this.
 *   - Ranking key: am + (lm_weight * (lmacc + smear(n)) + word_bonus * words), each operation rounded to float32 in
 *     that order.
 *   - After frame T_b - 1 each beam at a word end completes its word; a beam still inside a word is dropped.  Each
 *     survivor adds its LM node's end weight (dropped at -inf) and the N-best are ranked by
 *     am + (lm_weight * lm + word_bonus * words), ties to the earlier beam.  T_b = 0 gives the empty transcript, with
 *     no words and lm the start node's end weight (no hypothesis when that is -inf).
 * Outputs: as gtnb_beam_decode_lm_async (scores, am_scores, lm_scores: lm = the word LM's score of the words,
 * end weight included), plus words_dev [B][N][T] (nullable): each hypothesis's word ids followed by -1, read off its
 * tokens by walking the trie; word_counts_dev [B][N] (nullable), -1 for unused hypotheses and status 1 and 2.
 * Hypotheses are distinct token transcripts: two of them may spell the same words (with and without a leading
 * separator, say).
 * Errors: lm_weight negative or not finite, word_bonus not finite, lexicon NULL or made on another device or for
 * another C, or (CTC, BIGRAM) a lexicon that spells with the blank or makes it a separator:
 * GTNB_ERR_INVALID_ARGUMENT.  token_beam outside [1, C]: GTNB_ERR_UNSUPPORTED.
 * Identity: with the identity lexicon (every non-blank token, every token for ASG, a word-start token spelling itself
 * as the word of the same id), no word LM, word_bonus 0 and token_beam = C, tokens, lengths, scores and status are
 * == gtnb_beam_decode_async's.
 *
 * Out of scope: unknown words, a separator score, homophones, lookahead beyond max-unigram smearing, a token LM with
 * the lexicon, C > 256, and merging hypotheses by state instead of by transcript.
 */
int gtnb_beam_decode_lexicon_async(
    gtnb_ctx* ctx,
    void* cuda_stream,
    int B,
    int T,
    int C,
    const void* emissions_dev, /* [B][T][C] of dtype */
    int dtype,
    const int32_t* input_lens_dev, /* [B] or NULL */
    int kind, /* GTNB_DENSE_CTC | GTNB_DENSE_BIGRAM | GTNB_DENSE_ASG */
    const float* trans_w_dev, /* NULL, BIGRAM [C*C], ASG [C + C*C] */
    int blank,
    int beam,
    int nbest,
    const gtnb_lexicon* lexicon,
    float lm_weight,
    float word_bonus,
    int token_beam,
    int32_t* tokens_dev, /* [B][nbest][T] */
    int32_t* lengths_dev, /* [B][nbest] */
    float* scores_dev, /* [B][nbest] */
    float* am_scores_dev, /* [B][nbest] or NULL */
    float* lm_scores_dev, /* [B][nbest] or NULL */
    int32_t* words_dev, /* [B][nbest][T] or NULL */
    int32_t* word_counts_dev, /* [B][nbest] or NULL */
    int32_t* status_dev, /* [B] or NULL */
    void* workspace_dev,
    size_t workspace_bytes);

#ifdef __cplusplus
}
#endif
#endif /* GTN_B200_H */
