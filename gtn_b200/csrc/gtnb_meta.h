/*
 * gtnb_meta.h -- the per-graph descriptor the kernels read (one GraphMeta per graph of a packed
 * batch, in HBM).  Plain data, no CUDA types: also included by the host-side kernel emulation of
 * tests/emu.
 */
#pragma once

#include <cstdint>

namespace gtnb {

constexpr uint32_t kRowMask = 0x3FFFFFFFu; // low 30 bits of a row_ptr entry
constexpr uint32_t kStartBit = 0x40000000u; // node is a start node
constexpr uint32_t kAcceptBit = 0x80000000u; // node is an accept node
constexpr int kAlign = 4; // elements; keeps every per-graph slab 16-byte aligned
constexpr int kMaxDynamicSmem = 227 * 1024; // a CTA's opt-in dynamic shared memory on sm_90 (ensure_max_smem)

/*
 * G's tables as k_sparse.cu's denominator sweeps read them (gtnb_product.h's SparseTables on the device): S nodes,
 * A arcs with a label in [0, C); in-arcs by destination, out-arcs by source; *_arc is G's arc id, which indexes the
 * transition weights and their gradient.  lanes: threads per node (a power of two <= 32).
 */
struct SparseDev {
  int S, A, lanes;
  const int32_t* flags; // bit 0 start, bit 1 accept
  const int32_t *in_ptr, *in_src, *in_lab, *in_arc;
  const int32_t *out_ptr, *out_dst, *out_lab, *out_arc;
};
/* the envelope of k_sparse.cu's kernels: rows and arc gradients of G held in shared memory (sparse_den_supported) */
constexpr int kSparseMaxStates = 4096;
constexpr int kSparseMaxArcs = 32768;
constexpr int kSparseMaxLabels = 1024;
/* SparseDev::lanes: a power of two <= 32 with about four arcs per thread at G's mean degree */
inline int sparse_den_lanes(int S, int A) {
  int lanes = 1;
  while (lanes < 32 && 4ll * lanes * (S > 1 ? S : 1) < (long long)A) lanes *= 2;
  return lanes;
}

/* the CTA of k_sparse.cu's sweeps */
constexpr int kSparseThreads = 512;
constexpr int kSparseWarps = kSparseThreads / 32;

/*
 * A G too large for one CTA is swept by a thread-block cluster of N CTAs per utterance (k_sparse.cu's sparse_cl_*
 * kernels): rank r computes the nodes [in[r], in[r + 1]) of the forward and the tropical sweep and the nodes
 * [out[r], out[r + 1]) of the backward sweep (sparse_cluster_splits, gtnb_product.h: contiguous ranges with balanced
 * arc counts).  Every CTA keeps the whole [2][S] score rows; the backward's arc-gradient accumulator holds the rank's
 * own out-arcs only, which is what lifts the arc limit.
 */
constexpr int kSparseClusterMax = 8; // CTAs per cluster: the portable maximum
struct SparseSplit {
  int N; // 2, 4 or 8
  int own_out; // the most out-arcs a rank owns: the backward's accumulators
  int32_t in[kSparseClusterMax + 1], out[kSparseClusterMax + 1];
};
/* the cluster kernels' bounds on G; inside them sparse_cluster_plan (gtnb_product.h) decides from the shared memory
 * the actual splits need (the full trigram at C = 64, 4096 nodes / 262 144 arcs, takes N = 8: 162 KB) */
constexpr int kSparseClusterMaxStates = 16384;
constexpr int kSparseClusterMaxArcs = 262144;
constexpr long long kSparseClusterSmemBytes = 227 * 1024; // a CTA's opt-in dynamic shared memory on sm_90
/* kBpNone = 0xFFFF must not be a position | tie flag: the last position of an in-list is at most 0x7FFD */
constexpr int kSparseClusterMaxInDegree = 32766;
/* floats of dynamic shared memory of the cluster sweeps: rows [2][S], emission rows [2][C], the per-warp row maxima
 * of every rank [2][N * kSparseWarps]; the backward adds the emission gradient [2][C] and own_arcs accumulators */
inline long long sparse_cl_fwd_smem_floats(int S, int C, int N) {
  return 2ll * S + 2ll * C + 2ll * N * kSparseWarps;
}
inline long long sparse_cl_bwd_smem_floats(int S, int C, int N, int own_arcs) {
  return 2ll * S + 4ll * C + own_arcs + 2ll * N * kSparseWarps;
}

/*
 * An acceptor with epsilon arcs as k_sparse.cu's backoff sweeps read it (gtnb_product.h's SparseTables with its
 * epsilon tables): g holds the emitting arcs, then come the E epsilon arcs (by destination and by source; *_arc
 * indexes the weights and their gradient like g's) in L topological levels.  Forward level l is the nodes
 * fwd_node[fwd_ptr[l] .. fwd_ptr[l + 1]), whose epsilon in-arcs leave nodes of earlier levels only; backward level l
 * (bwd_*) likewise over the epsilon out-arcs.  lanes[l] / lanes[L + l]: threads per node of forward / backward level
 * l.  rows: the first float of this graph's score rows when every CTA reads its own graph (the numerators).
 */
struct SparseEpsDev {
  SparseDev g;
  int E, L;
  const int32_t *eps_in_ptr, *eps_in_src, *eps_in_arc;
  const int32_t *eps_out_ptr, *eps_out_dst, *eps_out_arc;
  const int32_t *fwd_ptr, *fwd_node, *bwd_ptr, *bwd_node, *lanes;
  long long rows;
};
/* the envelope's level bound: each level costs one CTA barrier per frame (a backoff n-gram of order n has n - 1) */
constexpr int kSparseMaxLevels = 32;
/* the backoff decode's back-pointer of a start node at frame 0; a node's in-list (emitting then epsilon in-arcs) is
 * below it, so both fit the 15 position bits */
constexpr int kBpStart = 0x7FFE;
/* the envelope of the backoff sweeps, for G and for every numerator: S nodes, A emitting and E epsilon arcs, L levels,
 * max_in the largest in-degree counting both kinds of arc */
inline bool sparse_eps_supported(int S, int A, int E, int L, int max_in, int C) {
  return S >= 1 && S <= kSparseMaxStates && (long long)A + E <= kSparseMaxArcs && L <= kSparseMaxLevels &&
         max_in < kBpStart && C >= 1 && C <= kSparseMaxLabels;
}

/* semiring / output of the shortest-distance kernels */
enum { MODE_LOG = 0, MODE_TROPICAL = 1, MODE_PATH = 2 };

/*
 * Per-graph descriptor, one per batch entry, resident in HBM.  All bases are
 * ELEMENT offsets into the batch-wide arrays of gtnb_lattice.
 *
 * Layout of graph b (device numbering):
 *   nodes  [0, N)   sorted by level; level l = [lvl_node_ptr[l], lvl_node_ptr[l+1])
 *                   nodes [lvl_node_ptr[L], N) are never scheduled by the
 *                   reference's Kahn sweep but are accept nodes with no
 *                   in-arcs: their score is the vector's initial 0.0f
 *                   (shortest.cpp:89).
 *   arcs   [0, A)   CSR by destination: in-arcs of node n are
 *                   [row_ptr[n] & kRowMask, row_ptr[n+1] & kRowMask) in the
 *                   reference's g.in(n) order; the top two bits of row_ptr[n]
 *                   carry the start / accept flags of node n.
 */
struct GraphMeta {
  long long node_base; // row_ptr, scores, node_grad, back_ptr, node_orig
  long long arc_base; // src, w, gi_*, arc_grad, arc_orig, relax_rank
  long long lvl_base; // lvl_node_ptr, lvl_arc_ptr  (L+1 entries)
  long long acc_base; // accept_nodes
  long long blvl_base; // backward level ptr (LB+1 entries), packed graphs only
  long long bnode_base; // backward node list
  long long sg_node_base; // small-graph (compose operand) slabs
  long long sg_arc_base;
  long long emis_off; // utterance's first emission, in floats
  long long grad_graph_off; // this graph's slab in gtnb_compose_grad's grad_graph_dev
  int L; // number of forward levels
  int N; // number of device nodes
  int A; // number of device arcs
  int n_accept;
  int LB; // number of backward levels (packed graphs), -1 = reverse forward levels
  int status; // GTNB_OK or GTNB_ERR_INVALID_ARGUMENT
  int T; // frames (composed lattices)
  int sg_N; // small-graph node / arc counts (composed lattices)
  int sg_A;
  int sg_all_valid; // every arc label of the graph operand can match an emission label
  int sg_uniform; // all in-arcs of a graph node carry the same matched label
  int cap_N; // slab capacities
  int cap_A;
  int cap_L;
  int tgt_off; // gtnb_ctc_loss: first label of this utterance in the concatenated targets (k_bidir.cu PAIR)
  int pad_;
};

/*
 * The policies of k_beam.cu's beam search, as the entry points fill them (their device code is in k_beam.cu):
 * BeamNoLm for gtnb_beam_decode_async, BeamLm for gtnb_beam_decode_lm_async, BeamLex for
 * gtnb_beam_decode_lexicon_async.  on: the policy prunes tokens and ranks by a fused score.  The outputs a policy
 * lacks are static NULLs, so that code writing every output compiles the missing ones away.
 */
struct BeamNoLm {
  static constexpr bool on = false;
  static constexpr int P = 0; // (unused: every token)
  static constexpr float *am = nullptr, *lm = nullptr;
  static constexpr int32_t *words = nullptr, *counts = nullptr;
};
struct BeamLm {
  static constexpr bool on = true;
  int P; // token_beam: tokens per frame, P = C: all of them
  const float* lmw; // [S][C + 1] resolved LM weights (column C: end weights); NULL: no LM, every weight 0
  const int32_t* lmd; // [S][C + 1] destination nodes
  int start; // the LM's start node
  float lw, tb; // lm_weight, token_bonus
  float *am, *lm; // [B][N] nullable: acoustic and LM scores of the hypotheses
  static constexpr int32_t *words = nullptr, *counts = nullptr;
};
/* BeamLex: BeamLm's P, start (the word LM's start node), lw, tb (word_bonus), am and lm; lmw and lmd are NULL */
struct BeamLex : BeamLm {
  const int32_t* cls; // [C] token classes: 0 in-word, 1 separator, 2 word-start
  int MW; // ceil(C / 32)
  const uint32_t* mask; // [nodes][MW] trie child masks (bit c: a child labelled c)
  const int32_t* first; // [nodes] index of the first child (children numbered in token order)
  const int32_t* word; // [nodes] word id spelled at the node, or -1
  const float* smear; // [nodes] lookahead of the node
  const unsigned long long* hash; // [H][2] word LM emitting arcs: key node << 32 | word (all ones: empty), value
                                  // destination << 32 | weight bits; NULL: no word LM, every weight 0
  unsigned long long hmul; // multiplier of the arc hash (0: every key probes from slot 0)
  int hbits; // log2 H
  const float* bow; // [S] backoff weight of each LM node
  const int32_t* bod; // [S] backoff destination, or -1
  const float* endw; // [S] resolved end weights
  int32_t *words, *counts; // [B][N][T] / [B][N] nullable: word ids and word counts of the hypotheses
};

/*
 * One chunk call of the streaming beam decoder (gtnb_beam_decode_chunk_async), for k_beam.cu's beam_chunk_kernel:
 * each row resumes its saved search, runs its frames of the chunk and saves it again (k_beam.cu's beam_state_words
 * gives a row's block).
 */
struct BeamChunk {
  static constexpr bool on = true;
  int Tc; // frames per row of the chunk's emissions [B][Tc][C]
  uint32_t* state; // [B][words] the rows' state blocks
  long long words;
  const int32_t* lens; // [B] frames of each row, nullable: Tc
  const int32_t* control; // [B] GTNB_BEAM_RESET | GTNB_BEAM_END, nullable: 0
  int32_t* best_tokens; // [B][T_max] nullable (with the two below): each row's best beam after its frames
  int32_t* best_lengths; // [B]
  float* best_scores; // [B]
};

} // namespace gtnb
