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

} // namespace gtnb
