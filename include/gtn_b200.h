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
/* device pointer to all arc gradients (device arc order) -- advanced use */
const float* gtnb_lattice_arc_grads_dev(const gtnb_lattice* lat);

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

#ifdef __cplusplus
}
#endif
#endif /* GTN_B200_H */
