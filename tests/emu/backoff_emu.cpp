/*
 * tests/emu/backoff_emu.cpp -- TEST INFRASTRUCTURE for gtnb_backoff_transitions_loss and gtnb_viterbi_backoff: the
 * shipped host builders (gtn_b200/csrc/gtnb_product.h: G's tables with its epsilon levels, the products with G's
 * epsilon arcs) and the SOURCE of k_sparse.cu's backoff kernels (sparse_eps_*), run on the CPU through
 * tests/emu/simt_emu.h.  Only the launch geometry and the packing of the tables into SparseEpsDev are restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_sparse.cu"
#include "../../gtn_b200/csrc/gtnb_product.h"

#include <cstring>
#include <deque>
#include <vector>

namespace {

gtnb_graph_view view_of(int N, int nA, const uint8_t* flags, const int32_t* src, const int32_t* dst,
                        const int32_t* label, const float* w) {
  gtnb_graph_view v{};
  v.num_nodes = N;
  v.num_arcs = nA;
  v.node_flags = flags;
  v.arc_src = src;
  v.arc_dst = dst;
  v.arc_ilabel = v.arc_olabel = label;
  v.weights = w;
  return v;
}

gtnb::SparseTables eps_tables_of(const gtnb_graph_view& G, int C) {
  gtnb::SparseTables t;
  gtnb::sparse_tables(G, C, &t);
  gtnb::sparse_eps_tables(G, &t);
  return t;
}

/* the host copy of what EpsDevTables (gtnb_criteria.cu) uploads: the tables, arc ids shifted by arc_base */
struct HostEps {
  std::deque<std::vector<int32_t>> keep;
  const int32_t* hold(const std::vector<int32_t>& v, int32_t shift = 0) {
    keep.emplace_back(v);
    for (int32_t& x : keep.back()) x += shift;
    keep.back().push_back(0); // (never empty)
    return keep.back().data();
  }
  gtnb::SparseEpsDev add(const gtnb::SparseTables& t, int32_t arc_base, long long rows, int lanes) {
    gtnb::SparseEpsDev d{};
    d.g.S = t.S;
    d.g.A = t.A;
    d.g.lanes = lanes ? lanes : gtnb::sparse_den_lanes(t.S, t.A);
    d.g.flags = hold(std::vector<int32_t>(t.flags.begin(), t.flags.end()));
    d.g.in_ptr = hold(t.in_ptr), d.g.in_src = hold(t.in_src), d.g.in_lab = hold(t.in_lab);
    d.g.in_arc = hold(t.in_arc, arc_base);
    d.g.out_ptr = hold(t.out_ptr), d.g.out_dst = hold(t.out_dst), d.g.out_lab = hold(t.out_lab);
    d.g.out_arc = hold(t.out_arc, arc_base);
    d.E = t.E;
    d.L = t.L;
    d.eps_in_ptr = hold(t.eps_in_ptr), d.eps_in_src = hold(t.eps_in_src), d.eps_in_arc = hold(t.eps_in_arc, arc_base);
    d.eps_out_ptr = hold(t.eps_out_ptr), d.eps_out_dst = hold(t.eps_out_dst);
    d.eps_out_arc = hold(t.eps_out_arc, arc_base);
    d.fwd_ptr = hold(t.fwd_ptr), d.fwd_node = hold(t.fwd_node), d.bwd_ptr = hold(t.bwd_ptr);
    d.bwd_node = hold(t.bwd_node), d.lanes = hold(t.lanes);
    d.rows = rows;
    return d;
  }
};

} // namespace

extern "C" {

/*
 * G's epsilon tables (sparse_eps_tables).  info: [E, L, cycle length, emitting arcs A, largest combined in-degree].
 * Call with the arrays NULL for the sizes, then with room for cycle [cycle length], fwd_ptr / bwd_ptr [L + 1],
 * fwd_node / bwd_node [fwd_ptr[L]] and lanes [2L].
 */
int emu_backoff_tables(int S, int nG, const uint8_t* flags, const int32_t* src, const int32_t* dst,
                       const int32_t* label, int C, int32_t* info, int32_t* cycle, int32_t* fwd_ptr,
                       int32_t* fwd_node, int32_t* bwd_ptr, int32_t* bwd_node, int32_t* lanes) {
  const gtnb::SparseTables t = eps_tables_of(view_of(S, nG, flags, src, dst, label, nullptr), C);
  info[0] = t.E, info[1] = t.L, info[2] = (int32_t)t.cycle.size(), info[3] = t.A, info[4] = t.max_in_all;
  if (!cycle) return 0;
  std::copy(t.cycle.begin(), t.cycle.end(), cycle);
  std::copy(t.fwd_ptr.begin(), t.fwd_ptr.end(), fwd_ptr);
  std::copy(t.fwd_node.begin(), t.fwd_node.end(), fwd_node);
  std::copy(t.bwd_ptr.begin(), t.bwd_ptr.end(), bwd_ptr);
  std::copy(t.bwd_node.begin(), t.bwd_node.end(), bwd_node);
  std::copy(t.lanes.begin(), t.lanes.end(), lanes);
  return 0;
}

/*
 * intersect(A, G) from gtnb_product.h's builder, unfolded, with G's epsilon arcs (label -1, arc_of -1).  Call once
 * with the out arrays NULL for the sizes (*n_nodes, *n_arcs), then again with room for them.
 */
int emu_backoff_product(int N, int nA, const uint8_t* a_flags, const int32_t* a_src, const int32_t* a_dst,
                        const int32_t* a_label, int S, int nG, const uint8_t* g_flags, const int32_t* g_src,
                        const int32_t* g_dst, const int32_t* g_label, int C, int* n_nodes, int* n_arcs,
                        uint8_t* flags, int32_t* src, int32_t* dst, int32_t* label, int32_t* arc_of, int32_t* tidx) {
  const gtnb_graph_view A = view_of(N, nA, a_flags, a_src, a_dst, a_label, nullptr);
  const gtnb_graph_view G = view_of(S, nG, g_flags, g_src, g_dst, g_label, nullptr);
  const gtnb::SparseTables t = eps_tables_of(G, C);
  gtnb::ProductGraph p;
  gtnb::build_sparse_product(A, G, t, C, /*fold=*/false, &p);
  *n_nodes = (int)p.flags.size();
  *n_arcs = (int)p.src.size();
  if (!flags) return 0;
  std::memcpy(flags, p.flags.data(), p.flags.size());
  const size_t bytes = p.src.size() * sizeof(int32_t);
  std::memcpy(src, p.src.data(), bytes);
  std::memcpy(dst, p.dst.data(), bytes);
  std::memcpy(label, p.label.data(), bytes);
  std::memcpy(arc_of, p.arc_of.data(), bytes);
  std::memcpy(tidx, p.tidx.data(), bytes);
  return 0;
}

/*
 * The log-semiring sweeps as backoff_loss_fast launches them.  n_graphs = 1: one graph for every utterance (the
 * denominator, per_cta off); n_graphs = B: graph b for utterance b (the numerators, per-CTA tables, score rows packed
 * by (T_b + 1) * S_b).  Graph g has S[g] nodes and nA[g] arcs, its arrays concatenated with the others' (labels -1:
 * epsilon arcs); w: the weights of all arcs in that order.  Out: den[B], grad [B][T][C] and wgrad (zero on entry:
 * sgn times the gradients added), status[B] (zeroed here).  Returns 0, 1 outside the envelope, 77 when the host
 * refused the threads.
 */
int emu_backoff_sweep(int B, int T, int C, const float* emissions, const int32_t* lens, int n_graphs,
                      const int32_t* S, const int32_t* nA, const uint8_t* flags, const int32_t* src,
                      const int32_t* dst, const int32_t* label, const float* w, float sgn, int threads, float* den,
                      float* grad, float* wgrad, int32_t* status) {
  using namespace gtnb;
  HostEps h;
  std::vector<SparseEpsDev> desc;
  long long rows = 0, node0 = 0, arc0 = 0;
  int max_S = 1, max_AE = 0;
  for (int g = 0; g < n_graphs; g++) {
    const gtnb_graph_view v = view_of(S[g], nA[g], flags + node0, src + arc0, dst + arc0, label + arc0, nullptr);
    const SparseTables t = eps_tables_of(v, C);
    if (!t.cycle.empty() || !sparse_eps_supported(t.S, t.A, t.E, t.L, t.max_in_all, C)) return 1;
    desc.push_back(h.add(t, (int32_t)arc0, rows, 0));
    rows += (long long)((n_graphs == 1 ? T : lens[g]) + 1) * S[g] * (n_graphs == 1 ? B : 1);
    max_S = std::max(max_S, t.S);
    max_AE = std::max(max_AE, t.A + t.E);
    node0 += S[g];
    arc0 += nA[g];
  }
  const int per_cta = n_graphs == 1 ? 0 : 1;
  std::vector<float> alpha((size_t)rows + 16, 0.0f);
  std::vector<double> offs((size_t)B * (T + 1) + 16, 0.0);
  for (int b = 0; b < B; b++) status[b] = 0;
  emu::launch(B, threads, sizeof(float) * sparse_fwd_smem_floats(max_S, C), [&] {
    sparse_eps_forward_kernel(desc.data(), per_cta, T, C, lens, emissions, (long long)T * C, w, alpha.data(),
                              offs.data(), den, status);
  });
  emu::launch(B, threads, sizeof(float) * sparse_bwd_smem_floats(max_S, max_AE, C), [&] {
    sparse_eps_backward_kernel(desc.data(), per_cta, T, C, lens, emissions, (long long)T * C, w, alpha.data(),
                               offs.data(), sgn, grad, (long long)T * C, wgrad);
  });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

/*
 * The decode's device route as backoff_viterbi_run launches it: the tropical sweep with the epsilon closure, then the
 * traceback.  G (S nodes, nG arcs, labels -1: epsilon arcs), w [nG]; lanes: threads per node of the emitting update
 * (0: sparse_den_lanes).  Out: paths, arcs [B][T], scores [B], status [B] (zeroed here).
 */
int emu_backoff_viterbi(int B, int T, int C, const float* emissions, const int32_t* lens, int S, int nG,
                        const uint8_t* g_flags, const int32_t* g_src, const int32_t* g_dst, const int32_t* g_label,
                        const float* w, int lanes, int32_t* paths, int32_t* arcs, float* scores, int32_t* status) {
  using namespace gtnb;
  const SparseTables t = eps_tables_of(view_of(S, nG, g_flags, g_src, g_dst, g_label, nullptr), C);
  if (!t.cycle.empty() || !sparse_eps_supported(t.S, t.A, t.E, t.L, t.max_in_all, C)) return 1;
  HostEps h;
  const SparseEpsDev d = h.add(t, 0, 0, lanes);
  std::vector<uint16_t> bp((size_t)B * (T + 1) * S + 1, 0);
  std::vector<int32_t> head(B + 1, 0);
  for (int b = 0; b < B; b++) status[b] = 0;
  emu::launch(B, kSparseThreads, sizeof(float) * sparse_vit_smem_floats(S, C), [&] {
    sparse_eps_viterbi_kernel(&d, T, C, lens, emissions, (long long)T * C, w, bp.data(), head.data(), scores, status);
  });
  emu::launch((B * 32 + 255) / 256, 256, 0, [&] {
    sparse_eps_trace_kernel(&d, B, T, lens, bp.data(), head.data(), paths, arcs, status);
  });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

/* sparse_eps_gather_kernel and sparse_eps_scatter_kernel over n product arcs, as backoff_loss_fast launches them */
int emu_backoff_gather_scatter(long long n, const float* w_A, const int32_t* arc_of, const float* W,
                               const int32_t* tidx, float* out, const float* pg, float* tgrad, float* agrad) {
  using namespace gtnb;
  if (n > 0) {
    const unsigned blocks = (unsigned)((n + 255) / 256);
    emu::launch(blocks, 256, 0, [&] { sparse_eps_gather_kernel(n, w_A, arc_of, W, tidx, out); });
    emu::launch(blocks, 256, 0, [&] { sparse_eps_scatter_kernel(n, pg, arc_of, tidx, tgrad, agrad); });
  }
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

} // extern "C"
