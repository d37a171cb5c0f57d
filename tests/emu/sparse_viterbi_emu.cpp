/*
 * tests/emu/sparse_viterbi_emu.cpp -- TEST INFRASTRUCTURE for gtnb_viterbi_sparse and gtnb_sparse_transitions_viterbi:
 * the shipped host builder of G's tables (gtn_b200/csrc/gtnb_product.h) and the SOURCE of k_sparse.cu's tropical
 * sweep, traceback and tau kernels, run on the CPU through tests/emu/simt_emu.h.  Only the launch geometry and the
 * packing of the tables into SparseDev are restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_sparse.cu"
#include "../../gtn_b200/csrc/gtnb_product.h"

#include <vector>

namespace {

gtnb::SparseTables tables_of(int S, int nG, const uint8_t* flags, const int32_t* src, const int32_t* dst,
                             const int32_t* label, int C) {
  gtnb_graph_view G{};
  G.num_nodes = S;
  G.num_arcs = nG;
  G.node_flags = flags;
  G.arc_src = src;
  G.arc_dst = dst;
  G.arc_ilabel = G.arc_olabel = label;
  gtnb::SparseTables t;
  gtnb::sparse_tables(G, C, &t);
  return t;
}

} // namespace

extern "C" {

/*
 * The decode's device route as viterbi_sparse_run launches it: the tropical sweep, then the traceback.  emissions
 * [B][T][C], lens[B], G (S nodes, nG arcs), w [nG].  lanes: threads per node (0: sparse_den_lanes).  Out: paths,
 * arcs [B][T], scores [B], status [B] (zeroed here).  Returns 0, 1 outside the envelope, 77 when the host refused the
 * threads.
 */
int emu_sparse_viterbi(int B, int T, int C, const float* emissions, const int32_t* lens, int S, int nG,
                       const uint8_t* g_flags, const int32_t* g_src, const int32_t* g_dst, const int32_t* g_label,
                       const float* w, int lanes, int32_t* paths, int32_t* arcs, float* scores, int32_t* status) {
  using namespace gtnb;
  const SparseTables t = tables_of(S, nG, g_flags, g_src, g_dst, g_label, C);
  if (S < 1 || S > kSparseMaxStates || t.A > kSparseMaxArcs || C > kSparseMaxLabels) return 1;
  std::vector<int32_t> flags(t.flags.begin(), t.flags.end());
  const SparseDev dev{t.S, t.A, lanes ? lanes : sparse_den_lanes(t.S, t.A), flags.data(), t.in_ptr.data(),
                      t.in_src.data(), t.in_lab.data(), t.in_arc.data(), t.out_ptr.data(), t.out_dst.data(),
                      t.out_lab.data(), t.out_arc.data()};
  std::vector<uint16_t> bp((size_t)B * T * S + 1, 0);
  std::vector<int32_t> head(B + 1, 0);
  for (int b = 0; b < B; b++) status[b] = 0;
  emu::launch(B, kSparseThreads, sizeof(float) * sparse_vit_smem_floats(S, C), [&] {
    sparse_viterbi_forward_kernel(dev, T, C, lens, emissions, (long long)T * C, w, bp.data(), head.data(), scores,
                                  status);
  });
  emu::launch((B * 32 + 255) / 256, 256, 0, [&] {
    sparse_viterbi_trace_kernel(dev, B, T, lens, bp.data(), head.data(), paths, arcs, status);
  });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

/* sparse_tau_kernel over G's start groups, as launch_sparse_tau launches it; *K gets the group count */
int emu_sparse_tau(int S, int nG, const uint8_t* g_flags, const int32_t* g_src, const int32_t* g_dst,
                   const int32_t* g_label, int C, const float* w, float* tau, int* K) {
  using namespace gtnb;
  const SparseTables t = tables_of(S, nG, g_flags, g_src, g_dst, g_label, C);
  *K = (int)t.grp_ptr.size() - 1;
  if (*K > 0)
    emu::launch((*K * 32 + 255) / 256, 256, 0, [&] {
      sparse_tau_kernel(*K, t.grp_ptr.data(), t.grp_arc.data(), w, tau);
    });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

} // extern "C"
