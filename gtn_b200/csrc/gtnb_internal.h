/*
 * Internal declarations shared by the C-ABI translation units.
 * Nothing here is visible through include/gtn_b200.h.
 */
#pragma once

#ifdef GTNB_HOST_EMU
#error "GTNB_HOST_EMU is for tests/emu only (kernel sources compiled by g++ for the CPU test suite): the product library is never built with it, and this header is not part of that build"
#endif

#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "gtn_b200.h"

#include "gtnb_meta.h" // GraphMeta + layout constants: plain data, shared with the host-side kernel emulation (tests/emu)

/* dynamic shared memory of the CTA (the host-side emulation defines its own) */
#define GTNB_DYNAMIC_SMEM(type, name) extern __shared__ __align__(16) type name[]
#define GTNB_DYNAMIC_SMEM_128(type, name) extern __shared__ __align__(128) type name[]
#define GTNB_STATIC_SMEM(type, name, count) __shared__ type name[count]
#define GTNB_STATIC_SMEM_2D(type, name, d0, d1) __shared__ type name[d0][d1]

// k_bidir.cu is gtnb_ctc_loss's default path (gtnb_ctx_set_flag("bidir", 0): the two sweeps of k_implicit.cu):
// on an H100 0.36 ms in one launch against 0.26 + 0.31 ms (+ k_linear.cu beside them), and closer to float64
constexpr bool kBidirDefault = true;

struct gtnb_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  std::string err;
  int64_t launches = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  void* flush_buf = nullptr;
  size_t flush_bytes = 0;
  int sm_count = 132; // H100 SXM; replaced by the device's own count at context creation
  size_t total_mem = 0; // device memory, read once at context creation
  // pinned staging: every small host->device upload of one API call is packed here and
  // copied asynchronously (pageable copies would stall the stream each time)
  unsigned char* stage = nullptr;
  size_t stage_bytes = 0, stage_used = 0;
  cudaEvent_t stage_ev = nullptr;
  bool stage_pending = false;
  // second stream + events: overlap the host->device copy of the emissions with the
  // composition passes that only need the target graphs
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  // chunk streams / events: a host-buffer criterion call is cut into sub-batches whose
  // H2D copy, kernels and D2H copy overlap each other (gtnb_criteria.cu)
  std::vector<cudaStream_t> side_streams;
  std::vector<cudaEvent_t> side_events;
  // pinned read-back buffer for small device->host results
  unsigned char* readback = nullptr;
  size_t readback_bytes = 0;
  // optional per-kernel CUDA-event timing (gtnb_profile_*)
  struct ProfEntry {
    const char* name;
    cudaEvent_t a, b;
  };
  bool use_staged = true; // gtnb_ctx_set_flag("staged", 0) forces the generic kernels
  bool use_implicit = true; // gtnb_ctx_set_flag("implicit", 0): criteria materialise the lattice
  int bidir_mode = -1; // k_bidir.cu on CTC graphs ("bidir_mode" flag): 0 one node per thread; 1 and -1 (default) the PAIR kernels, ahead of every other node-warp variant measured on an H100 with and without a gradient (profiles/h100_bidir_pair_saves.json)
  bool use_bidir = kBidirDefault; // gtnb_ctx_set_flag("bidir", 0): the CTC criterion takes the two sweeps of k_implicit.cu instead of the bidirectional kernel (k_bidir.cu)
  bool exact_ties = true; // gtnb_ctx_set_flag("exact_ties", 0) turns it off: composed lattices are put in the reference's relaxation order so that viterbiPath breaks exact ties like shortest.cpp:212-218 (k_order.cu)
  int sparse_cluster = 0; // gtnb_ctx_set_flag("sparse_cluster", v): 0 a G outside the one-CTA envelope of k_sparse.cu takes the materialised route; 1 it takes the cluster kernels where sparse_cluster_plan has a plan; 2, 4, 8 additionally every G that fits a cluster of that size takes it (testing and measurement); the backoff entry points read it the same way for a G with epsilon arcs (backoff_route, sparse_cl_eps_* kernels)
  // Call-scoped device arena (the criteria): while arena_on, dev_alloc bumps a pointer inside one cached
  // allocation instead of ~25 stream-ordered allocations per call (each a microsecond or two of host time
  // ahead of the first launch); everything allocated in the scope is released together when it ends.
  unsigned char* arena = nullptr;
  size_t arena_cap = 0, arena_off = 0, arena_need = 0;
  bool arena_on = false;
  // the arena is a caller's workspace (the *_async calls): dev_alloc fails instead of allocating once it is full
  bool arena_borrowed = false;
  bool profiling = false;
  std::vector<ProfEntry> prof;
  std::vector<cudaEvent_t> ev_pool;
  std::string prof_text;
};

// rows of the saved scores of an implicit lattice whose graphs have at most this many nodes (k_bidir.cu's FX kernels)
constexpr int kImplicitFixedPitch = 224;

struct gtnb_lattice {
  int B = 0;
  bool composed = false;
  bool linear_first = false;
  bool shared_graph = false;
  bool level_local = false; // every arc goes level l-1 -> l
  bool forward_done = false;
  bool sizes_known = false;
  int score_pitch = 0; // implicit lattices: floats per saved-score row when every row has the same (0: the graph's node count rounded up to 4)
  bool order_pending = false; // exact_ties: rows still in compose order; sorted before arc ids or per-arc values first cross the ABI
  int forward_mode = -1;
  int C = 0;
  int max_lvl_nodes = 0, max_lvl_arcs = 0; // upper bounds over the batch
  int max_in_deg = 0, max_out_deg = 0; // of the graph operands (composed lattices)
  bool arc_labels = false; // some graph operand is not label-uniform: k_implicit.cu's arc-label kernels
  int max_T = 0;
  long long tot_N = 0, tot_A = 0, tot_L = 0, tot_acc = 0, tot_bl = 0, tot_bn = 0;
  long long tot_sgN = 0, tot_sgA = 0;

  std::vector<gtnb::GraphMeta> meta_h;
  gtnb::GraphMeta* meta = nullptr;

  // lattice proper
  int32_t* lvl_node_ptr = nullptr;
  int32_t* lvl_arc_ptr = nullptr;
  uint32_t* row_ptr = nullptr;
  int2* arcs = nullptr; // per arc {x = source node, y = bits of the fp32 weight}
  int32_t* acc_nodes = nullptr;
  // provenance of composed arcs (gradInfo)
  int2* gi = nullptr; // per arc {x = arc of the graph operand, y = arc of the linear operand}
  // packed graphs: mapping back to Graph numbering + backward schedule
  int32_t* node_orig = nullptr;
  int32_t* arc_orig = nullptr;
  int32_t* relax_rank = nullptr;
  int32_t* blvl_ptr = nullptr;
  int32_t* bnodes = nullptr;
  // saved state
  float* scores = nullptr;
  float* out_scores = nullptr; // [B]
  int32_t* best_accept = nullptr; // [B] tropical: best accept node
  float* node_grad = nullptr;
  float* arc_grad = nullptr;
  int32_t* back_ptr = nullptr;
  // compose operands kept on the device
  const float* emissions = nullptr;
  int64_t emissions_stride = 0;
  // the element type behind `emissions` (GTNB_F32 / GTNB_BF16 / GTNB_F16).  A 16-bit lattice is read only by
  // k_implicit.cu's one-node / several-nodes-per-thread log-semiring sweeps; every other mode refuses it
  int dtype = GTNB_F32;
  uint8_t* sg_flags = nullptr; // per small-graph node
  int32_t* sg_in_ptr = nullptr; // [sgN + 1] per graph
  int32_t* sg_in_src = nullptr; // per in-entry (sgA)
  int32_t* sg_in_label = nullptr; // matched label, -1 = can never match
  int32_t* sg_in_arc = nullptr; // Graph arc id
  float* sg_in_w = nullptr;
  int32_t* sg_ilabel = nullptr; // by arc id
  int32_t* sg_olabel = nullptr;
  // exact_ties only (else NULL): per in-entry the arc's position in its source's out list; per node its index in g.start()
  int32_t* sg_out_pos = nullptr;
  int32_t* sg_start_rank = nullptr;
  uint32_t* alive = nullptr; // [B][max_T+1][W] bitmasks
  int alive_words = 0;

  // host copies needed to answer queries on packed graphs
  std::vector<std::vector<int32_t>> h_node_orig, h_arc_orig, h_ilabel, h_olabel;
  std::vector<int32_t> h_arcs_orig_count; // Graph's own arc count (>= device A)
};

namespace gtnb {

struct SgDims {
  int N, A, n_acc;
  int all_valid = 0;
  int uniform = 0;
  int max_in = 0, max_out = 0; // largest in- / out-degree of a node
};
int composed_alloc(
    gtnb_ctx* ctx, int B, const SgDims* dims, int n_graphs, int linear_first, const int32_t* T,
    int C, const float* emissions_dev, int64_t emissions_stride, std::vector<long long>& sgn,
    std::vector<long long>& sga, gtnb_lattice** out, bool implicit_only = false);
int stage_begin(gtnb_ctx* ctx);
int stage_upload(gtnb_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes);
int stage_end(gtnb_ctx* ctx);
/* copies into the pinned staging buffer WITHOUT an upload and returns the address: pinned memory is mapped into the
 * device's address space (unified addressing), a kernel may read it in place */
int stage_reserve(gtnb_ctx* ctx, size_t bytes); // room for everything the pass will place (256-byte granules)
int stage_place(gtnb_ctx* ctx, const void* src_host, size_t bytes, void** where);
int readback_reserve(gtnb_ctx* ctx, size_t bytes);
int launch_ctc_build(
    gtnb_ctx* ctx, gtnb_lattice* lat, const int32_t* targets_dev, const int32_t* tgt_off_dev,
    const int32_t* tgt_len_dev, int blank);
/* gtnb_ctc_loss_async's device-side set-up and epilogue (k_ctc.cu): m0 / m1 are the host descriptors of utterances 0
 * and 1 (or 0 again) of the bound-uniform layout; small [3B] = [offsets | lens | T]; valid / kstatus [B] */
int launch_ctc_async_prepare(
    gtnb_ctx* ctx, int B, int S, int T, int C, const GraphMeta& m0, const GraphMeta& m1, const int32_t* input_lens,
    const int32_t* targets, const int32_t* target_lens, GraphMeta* meta, int32_t* small, float* deltas,
    int32_t* valid, int32_t* kstatus);
/* losses / status [B] from the sweeps' partial sums z (zp per utterance), scores s and flags; grad (nullable):
 * row_words 32-bit words per utterance, zeroed for a flagged one */
int launch_ctc_async_finalize(
    gtnb_ctx* ctx, int B, int zp, const float* z, const float* s, const int32_t* kstatus, const int32_t* valid,
    float* losses, int32_t* status, void* grad, long long row_words);
/* the same set-up for gtnb_ngram_ctc_loss_async / gtnb_asg_loss_async (asg): their numerators' descriptors, kstatus
 * [2B] (denominator, numerator) zeroed */
int launch_trellis_async_prepare(
    gtnb_ctx* ctx, bool asg, int B, int S, int T, int C, const GraphMeta& m0, const GraphMeta& m1,
    const int32_t* input_lens, const int32_t* targets, const int32_t* target_lens, GraphMeta* meta, int32_t* small,
    float* deltas, int32_t* valid, int32_t* kstatus);
/* after both forward sweeps: kstatus[b] |= kstatus[B + b] | !valid[b]; T_bwd[b] = flagged ? 0 : T_fwd[b];
 * den[b] = NaN where T_fwd[b] = 0 */
int launch_trellis_async_gate(gtnb_ctx* ctx, int B, const int32_t* T_fwd, const int32_t* valid, int32_t* kstatus,
                              int32_t* T_bwd, float* den);
/* dst[map[o + a]] += src[o + a], a < meta[b].sg_A, o = meta[b].grad_graph_off, for every b with kstatus[b] == 0 */
int launch_trellis_async_scatter(gtnb_ctx* ctx, int B, const GraphMeta* meta, const int32_t* kstatus,
                                 const int32_t* map, const float* src, float* dst);
/* the numerator an asynchronous alignment traces (gtnb_ctc_align_async, gtnb_ngram_ctc_align_async,
 * gtnb_asg_align_async) */
enum class AlignCriterion { Ctc, Ngram, Asg };
/* after launch_implicit_trace: status [B] (nullable) 0 / 1 (kstatus bit 1) / 2 (!valid) / 3 (kstatus bit 2, a tie);
 * a NaN score and -1 rows of paths and tokens for 1 and 2; tokens [B][T_out] (nullable): the target position of each
 * traced arc (arcs [B][T_out], read only when tokens is set), -1 for a blank or no arc */
int launch_align_async_finalize(gtnb_ctx* ctx, AlignCriterion kind, int B, int T_out, const GraphMeta* meta,
                                const int32_t* sg_in_ptr, const int32_t* kstatus, const int32_t* valid,
                                const int32_t* arcs, int32_t* paths, int32_t* tokens, float* scores, int32_t* status);
/* the asynchronous decoders' set-up (gtnb_viterbi_transitions_async, gtnb_viterbi_dense_async): lens / valid / kstatus
 * [B], lens[b] = T_b or 0 where input_lens[b] (NULL: T) lies outside [0, T], valid[b] whether it lies inside, kstatus
 * zeroed */
int launch_decode_async_prepare(gtnb_ctx* ctx, int B, int T, const int32_t* input_lens, int32_t* lens,
                                int32_t* valid, int32_t* kstatus);
/* after the sweep and trace: status [B] (nullable) 0 / 1 (kstatus bit 1) / 2 (!valid) / 3 (kstatus bit 2), kstatus
 * ignored where lens[b] = 0; a NaN score and -1 rows of paths and arcs ([B][T_out], nullable) for 1 and 2 */
int launch_decode_async_finalize(gtnb_ctx* ctx, int B, int T_out, const int32_t* lens, const int32_t* kstatus,
                                 const int32_t* valid, int32_t* paths, int32_t* arcs, float* scores,
                                 int32_t* status);
/* gtnb_edit_distance_async (k_edit.cu): the 32-bit move words its alignment needs for B pairs at these bounds, and
 * the one launch (moves NULL: no alignment; hyp_align / ref_align each nullable) */
long long edit_distance_move_words(int B, int N, int M, int word_sep);
int launch_edit_distance(gtnb_ctx* ctx, int B, const int32_t* hyp, int N, const int32_t* hyp_lens,
                         const int32_t* ref, int M, const int32_t* ref_lens, int word_sep, int32_t* distance,
                         int32_t* ops, int32_t* units, int32_t* status, int32_t* hyp_align, int32_t* ref_align,
                         uint32_t* moves);

/* gtnb_beam_decode_async (k_beam.cu): the bounds it covers, the transposed transitions / start weights / row flags of
 * a call, and the search under policy F (gtnb_meta.h: BeamNoLm, BeamLm or BeamLex; wt, wfirst, wbad unused for
 * GTNB_DENSE_CTC) */
bool beam_decode_supported(int C, int beam, int nbest);
int launch_beam_weights(gtnb_ctx* ctx, int C, int kind, const float* trans_w, float* wt, float* wfirst, int32_t* wbad);
template <class F>
int launch_beam_decode(gtnb_ctx* ctx, int B, int T, int C, const void* emissions, int dtype,
                       const int32_t* input_lens, int kind, const float* wt, const float* wfirst, const int32_t* wbad,
                       int blank, int K, int N, uint16_t* bp, int32_t* tokens, int32_t* lengths, float* scores,
                       int32_t* status, const F& f);
/* the streaming decoder (gtnb_beam_decode_chunk_async): a row's state block in 32-bit words under the BeamLm or the
 * BeamLex policy, and one chunk of the search under policy F (BeamLm, BeamLex); T is T_max */
long long beam_state_row_words(bool lexicon, int K, int C);
template <class F>
int launch_beam_chunk(gtnb_ctx* ctx, int B, int T, int C, const void* emissions, int dtype, int kind,
                      const float* wt, const float* wfirst, const int32_t* wbad, int blank, int K, int N, uint16_t* bp,
                      int32_t* tokens, int32_t* lengths, float* scores, int32_t* status, const F& f,
                      const BeamChunk& r);

int launch_scatter_add(gtnb_ctx* ctx, float* dst, const int32_t* idx, const float* src, long long n);
int launch_gather(gtnb_ctx* ctx, float* dst, const int32_t* idx, const float* src, long long n);
int launch_sub(gtnb_ctx* ctx, const float* a, const float* b, float* out, int n);

int fail(gtnb_ctx* ctx, int code, const std::string& msg);
int cuda_fail(gtnb_ctx* ctx, cudaError_t e, const char* what, const char* file, int line);

#define GTNB_CUDA(ctx, call)                                              \
  do {                                                                    \
    cudaError_t e__ = (call);                                             \
    if (e__ != cudaSuccess)                                               \
      return ::gtnb::cuda_fail((ctx), e__, #call, __FILE__, __LINE__);    \
  } while (0)

#define GTNB_CHECK_LAUNCH(ctx)                                            \
  do {                                                                    \
    (ctx)->launches++;                                                    \
    cudaError_t e__ = cudaGetLastError();                                 \
    if (e__ != cudaSuccess)                                               \
      return ::gtnb::cuda_fail((ctx), e__, "kernel launch", __FILE__, __LINE__); \
  } while (0)

inline cudaEvent_t prof_event(gtnb_ctx* ctx) {
  cudaEvent_t e;
  if (!ctx->ev_pool.empty()) {
    e = ctx->ev_pool.back();
    ctx->ev_pool.pop_back();
  } else {
    cudaEventCreate(&e);
  }
  return e;
}
inline void prof_begin(gtnb_ctx* ctx, const char* name) {
  if (!ctx->profiling) return;
  gtnb_ctx::ProfEntry pe{name, prof_event(ctx), prof_event(ctx)};
  cudaEventRecord(pe.a, ctx->stream);
  ctx->prof.push_back(pe);
}
inline void prof_end(gtnb_ctx* ctx) {
  if (!ctx->profiling || ctx->prof.empty()) return;
  cudaEventRecord(ctx->prof.back().b, ctx->stream);
}

/* Launch a kernel on the context's stream, count it, time it when profiling. */
#define GTNB_LAUNCH(ctx, name, ...)  \
  do {                               \
    ::gtnb::prof_begin((ctx), name); \
    __VA_ARGS__;                     \
    ::gtnb::prof_end((ctx));         \
    GTNB_CHECK_LAUNCH(ctx);          \
  } while (0)

/* Opt a kernel in to the full dynamic shared-memory window, once per (device, kernel).  The
 * attribute is process-wide: setting it per launch to that launch's size races between the
 * per-thread contexts of the gtn:: layer (one thread lowers it under another's launch). */
int ensure_max_smem(gtnb_ctx* ctx, const void* kernel);

template <typename T>
int dev_alloc(gtnb_ctx* ctx, T** p, long long n) {
  *p = nullptr;
  if (n <= 0) n = 1;
  // +16 elements of slack: staged copies round their windows up to 16 bytes
  const size_t bytes = sizeof(T) * (size_t)(n + 16);
  if (ctx->arena_on) {
    const size_t sz = (bytes + 255) & ~(size_t)255;
    ctx->arena_need += sz;
    if (ctx->arena_off + sz <= ctx->arena_cap) {
      *p = reinterpret_cast<T*>(ctx->arena + ctx->arena_off);
      ctx->arena_off += sz;
      return GTNB_OK;
    }
    if (ctx->arena_borrowed)
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT,
                  "workspace too small for these bounds (the call's *_async_workspace gives the size)");
  }
  GTNB_CUDA(ctx, cudaMallocAsync((void**)p, bytes, ctx->stream));
  return GTNB_OK;
}

template <typename T>
void dev_free(gtnb_ctx* ctx, T*& p) {
  const unsigned char* q = reinterpret_cast<const unsigned char*>(p);
  if (p && !(ctx->arena && q >= ctx->arena && q < ctx->arena + ctx->arena_cap)) cudaFreeAsync((void*)p, ctx->stream);
  p = nullptr;
}

/* the arena scope of one criterion call: begin before the first dev_alloc, end after the last dev_free (and
 * after the stream was synchronised, which every criterion does to return its losses) */
inline void arena_begin(gtnb_ctx* ctx) {
  ctx->arena_on = true;
  ctx->arena_off = 0;
  ctx->arena_need = 0;
}
inline void arena_end(gtnb_ctx* ctx) {
  ctx->arena_on = false;
  if (ctx->arena_need > ctx->arena_cap) { // grow for the next call of this shape
    if (ctx->arena) cudaFreeAsync(ctx->arena, ctx->stream);
    ctx->arena = nullptr;
    ctx->arena_cap = 0;
    const size_t want = ctx->arena_need + (ctx->arena_need >> 3);
    void* fresh = nullptr;
    if (cudaMallocAsync(&fresh, want, ctx->stream) == cudaSuccess) {
      ctx->arena = static_cast<unsigned char*>(fresh);
      ctx->arena_cap = want;
    } else {
      cudaGetLastError(); // no arena: the plain allocations keep working
    }
  }
}

// Upload through pinned staging is overkill for the small metadata here;
// pageable cudaMemcpyAsync is synchronous wrt the host and safe.
template <typename T>
int upload(gtnb_ctx* ctx, T* dst, const T* src, long long n) {
  if (n <= 0) return GTNB_OK;
  GTNB_CUDA(ctx, cudaMemcpyAsync(dst, src, sizeof(T) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  return GTNB_OK;
}

inline long long align_up(long long v, long long a) {
  return (v + a - 1) / a * a;
}

// kernels (k_shortest.cu)
int launch_forward(gtnb_ctx* ctx, gtnb_lattice* lat, int mode);
int launch_backward(gtnb_ctx* ctx, gtnb_lattice* lat, int tropical, const float* deltas_dev);
int launch_traceback(gtnb_ctx* ctx, gtnb_lattice* lat, int max_len, int32_t* path_dev, int32_t* len_dev);
int launch_gather_prov(gtnb_ctx* ctx, gtnb_lattice* lat, int max_len, const int32_t* path_dev, const int32_t* len_dev, int32_t* prov_graph, int32_t* prov_linear, float* path_w);
// kernels (k_staged.cu): TMA-staged persistent kernels for level-local lattices
bool staged_supported(const gtnb_lattice* lat);
int launch_forward_staged(gtnb_ctx* ctx, gtnb_lattice* lat, int mode);
int launch_backward_staged(gtnb_ctx* ctx, gtnb_lattice* lat, int tropical, const float* deltas_dev);
int launch_backward_fused(
    gtnb_ctx* ctx, gtnb_lattice* lat, const float* deltas_dev, float* grad_emis, int64_t grad_stride);
// kernels (k_dense.cu): factored dense-trellis Viterbi
bool implicit_supported(const gtnb_lattice* lat);
bool implicit_dims_supported(const SgDims* dims, int n_graphs, int arc_C = 0);
/* tropical: max instead of logadd (viterbiScore); the saved score rows then feed launch_implicit_trace */
int launch_implicit_forward(gtnb_ctx* ctx, gtnb_lattice* lat, int32_t* status_dev, int b0 = 0, int nb = -1,
                            bool tropical = false);
/* viterbiPath from a tropical launch_implicit_forward's score rows: paths / arcs (nullable, [B][T_out]) get the matched
 * label and the graph arc of every frame, -1 beyond T_b and without an accepting path; scores_out [B]; status bit 2
 * marks a tie on the traced path, bit 1 a score of +inf / NaN */
bool implicit_trace_supported(const gtnb_lattice* lat);
int launch_implicit_trace(gtnb_ctx* ctx, gtnb_lattice* lat, int32_t* status_dev, int32_t* paths, int32_t* arcs,
                          float* scores_out, int T_out);
/* k_bidir.cu: the CTC criterion in one launch (two-CTA clusters meeting in the middle), normaliser included */
/* dtype (GTNB_F32 / GTNB_BF16 / GTNB_F16): the element type of the emissions and the gradient, which launch_bidir_ctc
 * reads and writes as they are (lat->emissions then points at elements of that type); 16-bit types need C % 8 == 0 */
bool bidir_supported(const gtnb_lattice* lat, const void* emissions, int64_t stride, const void* grad, int64_t grad_stride,
                     int dtype = GTNB_F32);
int bidir_blocks(int max_T);
int bidir_zparts(); // partial sums of forwardScore(emissions) per CTA
int launch_bidir_ctc(
    gtnb_ctx* ctx, gtnb_lattice* lat, int32_t* status_dev, float* zparts_dev, float* boff_dev, void* grad_emis,
    int64_t grad_stride, int b0 = 0, int nb = -1, float* out_scores_dev = nullptr,
    int ctc_blank = -1, const int32_t* targets_dev = nullptr, const int32_t* tgt_off_dev = nullptr,
    const GraphMeta* meta_src = nullptr, // meta_src: the descriptors somewhere else than lat->meta (mapped host memory)
    int dtype = GTNB_F32);
// ctc_blank >= 0 + the targets: CTC target graphs, taken from the targets themselves (PAIR kernels)
bool bidir_takes_targets(const gtnb_lattice* lat, int ctc_blank);
/* k_order.cu (experimental): a composed lattice's rows and accept list in the order the reference's shortestPath relaxes / creates them */
int launch_relax_order(gtnb_ctx* ctx, gtnb_lattice* lat);
int launch_implicit_backward(
    gtnb_ctx* ctx, gtnb_lattice* lat, const float* deltas_dev, float* grad_emis, int64_t grad_stride,
    int b0 = 0, int nb = -1, float* grad_graph = nullptr);
/* arc_labels (gtnb_graph_loss): arcs whose label is outside [0, C) are left out of the tables, graphs that are not
 * label-uniform may take the implicit sweeps, and graph b's arc-gradient slab starts at the sum of the earlier
 * graphs' num_arcs.  arc_weights_dev (nullable): [sum num_arcs] device weights that replace the views' weights. */
int compose_linear_impl(
    gtnb_ctx* ctx, int B, const gtnb_graph_view* graphs, int n_graphs, int linear_first, const int32_t* T,
    int C, const float* emissions_dev, int64_t emissions_stride, bool implicit_only, gtnb_lattice** out,
    bool arc_labels = false, const float* arc_weights_dev = nullptr);
int validate_view(gtnb_ctx* ctx, const gtnb_graph_view& v);
int ensure_side_streams(gtnb_ctx* ctx, int n_streams, int n_events);
// kernel (k_dense.cu): factored dense-trellis Viterbi.  bigram: trans_dev is n-gram CTC's [C*C] W (every state
// starts), else ASG's [C + C*C]; bp holds [B][T_max][dense_bp_pitch(C)] bytes; 1 <= C <= 224
int dense_bp_pitch(int C);
// whether launch_viterbi_dense takes C: the transition tile fits shared memory (C <= 224)
bool viterbi_dense_supported(int C);
// emis: elements of dtype (GTNB_F32 / GTNB_BF16 / GTNB_F16), read as they are
int launch_viterbi_dense(
    gtnb_ctx* ctx, int B, int T_max, int C, bool bigram, const int32_t* T_dev, const void* emis, int64_t stride,
    const float* trans_dev, float empty_score, uint8_t* bp, int32_t* paths, float* scores, int dtype = GTNB_F32);
// kernels (k_ngram.cu): CTC with a learned bigram transition graph
constexpr int kNgramMaxLabels = 128;
int launch_ngram_sigma(gtnb_ctx* ctx, int C, const float* W, float* sigma);
int launch_ngram_num_build(
    gtnb_ctx* ctx, gtnb_lattice* lat, const int32_t* targets_dev, const int32_t* tgt_off_dev,
    const int32_t* tgt_len_dev, int blank, const float* W, const float* sigma, int32_t* map);
// the dense trellis (launch_*_den_*): emis holds elements of dtype (GTNB_F32 / GTNB_BF16 / GTNB_F16), read as they
// are; grad stays float32
int launch_ngram_den_forward(
    gtnb_ctx* ctx, int B, int T, int C, const int32_t* lens_dev, const void* emis, long long stride,
    const float* W, float* alpha, float* den, int32_t* status, int dtype = GTNB_F32);
int launch_ngram_den_backward(
    gtnb_ctx* ctx, int B, int T, int C, const int32_t* lens_dev, const void* emis, long long stride,
    const float* W, const float* alpha, const float* den, float* grad, long long grad_stride, float* wgrad,
    int dtype = GTNB_F32);
int launch_ngram_fold(gtnb_ctx* ctx, int C, const float* W, const float* sigma, float* wgrad);
// out[k] = w_A[arc_of[k]] + Wx[tidx[k]], Wx = [W (nW floats) | sigma]: the weights of gtnb_product.h's products
int launch_product_fold(gtnb_ctx* ctx, long long n, const float* w_A, const int32_t* arc_of, const float* W, int nW,
                        const float* sigma, const int32_t* tidx, float* out);
// tau_i = max_j W[i][j] (NaN-propagating): the tropical sigma of BIGRAM's folded start arcs
int launch_ngram_tau(gtnb_ctx* ctx, int C, const float* W, float* tau);
// arcs [B][T_out], product arc ids (-1 none) -> A arc ids: arc_of[off[b] + a] - off[B + b]
int launch_product_arc_map(gtnb_ctx* ctx, int B, int T_out, const long long* off, const int32_t* arc_of,
                           int32_t* arcs);
// the same trellis in ASG's start mode (trans_w, trans_grad: [C + C*C], start weights first) and ASG's
// forced-alignment numerator graphs built on the device
long long asg_alpha_floats(int B, int T, int C); // floats of the alpha buffer of launch_asg_den_*
int launch_asg_den_forward(
    gtnb_ctx* ctx, int B, int T, int C, const int32_t* lens_dev, const void* emis, long long stride,
    const float* trans_w, float* alpha, float* den, int32_t* status, int dtype = GTNB_F32);
int launch_asg_den_backward(
    gtnb_ctx* ctx, int B, int T, int C, const int32_t* lens_dev, const void* emis, long long stride,
    const float* trans_w, const float* alpha, const float* den, float* grad, long long grad_stride,
    float* trans_grad, int dtype = GTNB_F32);
int launch_asg_num_build(
    gtnb_ctx* ctx, gtnb_lattice* lat, const int32_t* targets_dev, const int32_t* tgt_off_dev,
    const int32_t* tgt_len_dev, const float* trans_w, int32_t* map);
// kernels (k_sparse.cu): the denominator of gtnb_sparse_transitions_loss over a G of any shape (SparseDev, gtnb_meta.h).
// The envelope, one predicate: 1 <= S <= kSparseMaxStates nodes, A <= kSparseMaxArcs arcs with a label in [0, C),
// 1 <= C <= kSparseMaxLabels.  alpha: [B][(T+1)*S] floats; offs: [B][T+1] doubles (slot 0: Z).
bool sparse_den_supported(int S, int A, int C);
// sp: sparse_route's split.  sp.N = 1 sweeps each utterance with one CTA (G inside sparse_den_supported); otherwise a
// thread-block cluster of sp.N CTAs per utterance does, for a G inside sparse_cluster_plan (gtnb_product.h: S <= 16384,
// A <= 262144, in-degree <= 32766, C <= 1024, and the shared memory of the plan's splits within 227 KB).  Same buffers
// and outputs either way: rows / offsets / scores / back-pointers bit-identical.  The scratch grows with S: alpha
// 4 * B * (T + 1) * S bytes, bp 2 * B * T * S bytes.
int launch_sparse_den_forward(gtnb_ctx* ctx, const SparseDev& g, const SparseSplit& sp, int B, int T, int C,
                              const int32_t* lens, const float* emis, long long stride, const float* w, float* alpha,
                              double* offs, float* den, int32_t* status);
int launch_sparse_den_backward(gtnb_ctx* ctx, const SparseDev& g, const SparseSplit& sp, int B, int T, int C,
                               const int32_t* lens, const float* emis, long long stride, const float* w,
                               const float* alpha, const double* offs, float* grad, long long grad_stride,
                               float* wgrad);
// gtnb_viterbi_sparse over the same tables: the tropical sweep (bp: [B][T][S] back-pointers, head: [B] best accept
// nodes, score: [B]) and the traceback into paths / arcs ([B][T], nullable); status bit 1 non-finite, bit 2 a tie
int launch_sparse_viterbi(gtnb_ctx* ctx, const SparseDev& g, const SparseSplit& sp, int B, int T, int C,
                          const int32_t* lens, const float* emis, long long stride, const float* w, uint16_t* bp,
                          int32_t* head, float* score, int32_t* paths, int32_t* arcs, int32_t* status);
// tau_k = max (NaN kept) over start group k: the folded start arcs of gtnb_sparse_transitions_viterbi
int launch_sparse_tau(gtnb_ctx* ctx, int K, const int32_t* grp_ptr, const int32_t* grp_arc, const float* w,
                      float* tau);
// sigma_k = logsumexp of start group k's weights, and its gradient (wgrad[nG + k]) folded back by softmax
int launch_sparse_sigma(gtnb_ctx* ctx, int K, const int32_t* grp_ptr, const int32_t* grp_arc, const float* w,
                        float* sigma);
int launch_sparse_fold(gtnb_ctx* ctx, int K, const int32_t* grp_ptr, const int32_t* grp_arc, int nG, const float* w,
                       const float* sigma, float* wgrad);
// The backoff sweeps over acceptors with epsilon arcs (SparseEpsDev, gtnb_meta.h): gs[0] for every CTA, or gs[b] for
// CTA b when per_cta (then alpha rows at gs[b].rows, and max_S / max_AE the largest S / A + E of the batch).  The
// envelope: S <= kSparseMaxStates, A + E <= kSparseMaxArcs, L <= kSparseMaxLevels, in-degree below kBpStart, C <=
// kSparseMaxLabels (sparse_eps_supported).  The backward adds sgn times the gradients.  The decode's bp: [B][T + 1][S].
// sp: backoff_route's split; the numerators pass sp.N = 1.  sp.N > 1 sweeps the denominator (gs[0] = G, max_S its
// S, per_cta off, sgn = 1) by a thread-block cluster of sp.N CTAs per utterance, for a G outside sparse_eps_supported
// and inside sparse_cluster_plan (S <= 16384, A + E <= 262144, L <= kSparseMaxLevels, in-degree below kBpStart,
// C <= 1024, and the shared memory of the plan's splits within 227 KB); cut: sparse_eps_cluster_cuts on the device
// (unused when sp.N = 1).  Same outputs either way, bit-identical but for the order of the gradient adds.
int launch_sparse_eps_forward(gtnb_ctx* ctx, const SparseEpsDev* gs, const SparseSplit& sp, const int32_t* cut,
                              int per_cta, int max_S, int B, int T, int C, const int32_t* lens, const float* emis,
                              long long stride, const float* w, float* alpha, double* offs, float* den,
                              int32_t* status);
int launch_sparse_eps_backward(gtnb_ctx* ctx, const SparseEpsDev* gs, const SparseSplit& sp, const int32_t* cut,
                               int per_cta, int max_S, int max_AE, int B, int T, int C, const int32_t* lens,
                               const float* emis, long long stride, const float* w, const float* alpha,
                               const double* offs, float sgn, float* grad, long long grad_stride, float* wgrad);
int launch_sparse_eps_viterbi(gtnb_ctx* ctx, const SparseEpsDev* gs, const SparseSplit& sp, const int32_t* cut, int S,
                              int B, int T, int C, const int32_t* lens, const float* emis, long long stride,
                              const float* w, uint16_t* bp, int32_t* head, float* score, int32_t* paths, int32_t* arcs,
                              int32_t* status);
// gtnb_backoff_transitions_viterbi over the numerators gs[b] (per CTA, max_S their largest S): the decode's sweep with
// bp at gs[b].rows ((T_b + 1) * S_b per utterance), then the trace, which reports arcs[b][t] = arc_of[product arc] -
// a_first[b] (A_b's own arc ids; a_first: [B] each utterance's first A arc in arc_of's numbering)
int launch_sparse_eps_align(gtnb_ctx* ctx, const SparseEpsDev* gs, int max_S, int B, int T, int C,
                            const int32_t* lens, const float* emis, long long stride, const float* w, uint16_t* bp,
                            int32_t* head, float* score, const int32_t* arc_of, const int32_t* a_first,
                            int32_t* paths, int32_t* arcs, int32_t* status);
// out[k] = w_A[arc_of[k]] + W[tidx[k]], W[tidx[k]] alone where arc_of[k] < 0 (G's epsilon arcs in the numerators)
int launch_sparse_eps_gather(gtnb_ctx* ctx, long long n, const float* w_A, const int32_t* arc_of, const float* W,
                             const int32_t* tidx, float* out);
// tgrad[tidx[k]] += pg[k], and agrad[arc_of[k]] += pg[k] where arc_of[k] >= 0 (agrad nullable)
int launch_sparse_eps_scatter(gtnb_ctx* ctx, long long n, const float* pg, const int32_t* arc_of, const int32_t* tidx,
                              float* tgrad, float* agrad);
// kernels (k_compose.cu)
int launch_compose(gtnb_ctx* ctx, gtnb_lattice* lat, cudaEvent_t emissions_ready = nullptr);
int launch_compose_grad(gtnb_ctx* ctx, gtnb_lattice* lat, float* grad_graph, float* grad_emis, int64_t grad_stride);
// kernels (k_cast.cu): n elements between 16-bit storage (GTNB_BF16 / GTNB_F16) and float32, rounding to nearest even
int launch_widen(gtnb_ctx* ctx, const void* src, int dtype, float* dst, long long n);
int launch_narrow(gtnb_ctx* ctx, const float* src, void* dst, int dtype, long long n);
// kernels (k_linear.cu)
int launch_linear_forward(
    gtnb_ctx* ctx, int B, const int32_t* T_dev, int maxT, int C, const float* emis, int64_t stride,
    int tropical, float* scores, float* grad, int64_t grad_stride, const float* deltas, float delta_all,
    int overwrite = 0, float* scratch = nullptr);


} // namespace gtnb
