/*
 * tests/emu/backoff_cluster_emu.cpp -- TEST INFRASTRUCTURE for the backoff cluster sweeps of k_sparse.cu
 * (sparse_cl_eps_*): the shipped host builders of G's tables with its epsilon levels, of the cluster plan and of the
 * per-level rank cuts (gtn_b200/csrc/gtnb_product.h), and the SOURCE of the cluster kernels and of the one-CTA
 * sparse_eps_* kernels they must reproduce, run on the CPU through tests/emu/simt_emu.h and simt_emu_dsmem.h.  Only
 * the launch geometry and the packing of the tables into SparseEpsDev are restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_sparse.cu"
#include "../../gtn_b200/csrc/gtnb_product.h"

#include <cstring>
#include <deque>
#include <vector>

namespace {

/* G's tables with its epsilon tables, and the SparseEpsDev that EpsDevTables (gtnb_criteria.cu) uploads for them */
struct Tables {
  gtnb::SparseTables t;
  std::deque<std::vector<int32_t>> keep;
  gtnb::SparseEpsDev dev{};

  const int32_t* hold(const std::vector<int32_t>& v) {
    keep.emplace_back(v);
    keep.back().push_back(0); // (never empty)
    return keep.back().data();
  }
};

void tables_of(int S, int nG, const uint8_t* flags, const int32_t* src, const int32_t* dst, const int32_t* label, int C,
               Tables* x) {
  gtnb_graph_view G{};
  G.num_nodes = S;
  G.num_arcs = nG;
  G.node_flags = flags;
  G.arc_src = src;
  G.arc_dst = dst;
  G.arc_ilabel = G.arc_olabel = label;
  gtnb::sparse_tables(G, C, &x->t);
  gtnb::sparse_eps_tables(G, &x->t);
  const gtnb::SparseTables& t = x->t;
  gtnb::SparseEpsDev& d = x->dev;
  d.g.S = t.S;
  d.g.A = t.A;
  d.g.lanes = gtnb::sparse_den_lanes(t.S, t.A);
  d.g.flags = x->hold(std::vector<int32_t>(t.flags.begin(), t.flags.end()));
  d.g.in_ptr = x->hold(t.in_ptr), d.g.in_src = x->hold(t.in_src), d.g.in_lab = x->hold(t.in_lab);
  d.g.in_arc = x->hold(t.in_arc);
  d.g.out_ptr = x->hold(t.out_ptr), d.g.out_dst = x->hold(t.out_dst), d.g.out_lab = x->hold(t.out_lab);
  d.g.out_arc = x->hold(t.out_arc);
  d.E = t.E;
  d.L = t.L;
  d.eps_in_ptr = x->hold(t.eps_in_ptr), d.eps_in_src = x->hold(t.eps_in_src), d.eps_in_arc = x->hold(t.eps_in_arc);
  d.eps_out_ptr = x->hold(t.eps_out_ptr), d.eps_out_dst = x->hold(t.eps_out_dst);
  d.eps_out_arc = x->hold(t.eps_out_arc);
  d.fwd_ptr = x->hold(t.fwd_ptr), d.fwd_node = x->hold(t.fwd_node), d.bwd_ptr = x->hold(t.bwd_ptr);
  d.bwd_node = x->hold(t.bwd_node), d.lanes = x->hold(t.lanes);
}

} // namespace

extern "C" {

/*
 * sparse_cluster_plan for G with its epsilon arcs (force: 0 the smallest N that fits, else that N alone) -> N or 0.
 * Out, when N > 0: the splits in_split / out_split [N + 1], the arcs (emitting + epsilon) every rank owns in_arcs /
 * out_arcs [N], the cuts (sparse_eps_cluster_cuts, [2][L][N + 1]).  Always info [6]: E, L, own_out, the backward's
 * shared-memory bytes under the plan (0 without one), largest combined in-degree, emitting arcs A.
 */
int emu_bc_plan(int S, int nG, const uint8_t* g_flags, const int32_t* g_src, const int32_t* g_dst,
                const int32_t* g_label, int C, int force, int32_t* in_split, int32_t* out_split, int32_t* in_arcs,
                int32_t* out_arcs, int32_t* cut, int64_t* info) {
  Tables x;
  tables_of(S, nG, g_flags, g_src, g_dst, g_label, C, &x);
  const gtnb::SparseTables& t = x.t;
  gtnb::SparseSplit sp{};
  const int N = gtnb::sparse_cluster_plan(t, C, force, &sp);
  info[0] = t.E, info[1] = t.L, info[2] = N ? sp.own_out : 0, info[4] = t.max_in_all, info[5] = t.A;
  info[3] = N ? (int64_t)sizeof(float) * gtnb::sparse_cl_bwd_smem_floats(t.S, C, N, sp.own_out) : 0;
  if (!N) return 0;
  for (int r = 0; r < N; r++) {
    in_arcs[r] = t.in_ptr[sp.in[r + 1]] - t.in_ptr[sp.in[r]] + t.eps_in_ptr[sp.in[r + 1]] - t.eps_in_ptr[sp.in[r]];
    out_arcs[r] =
        t.out_ptr[sp.out[r + 1]] - t.out_ptr[sp.out[r]] + t.eps_out_ptr[sp.out[r + 1]] - t.eps_out_ptr[sp.out[r]];
  }
  std::memcpy(in_split, sp.in, sizeof(int32_t) * (N + 1));
  std::memcpy(out_split, sp.out, sizeof(int32_t) * (N + 1));
  std::vector<int32_t> c;
  gtnb::sparse_eps_cluster_cuts(t, sp, &c);
  std::copy(c.begin(), c.end(), cut);
  return N;
}

/*
 * The denominator's two sweeps over G for every utterance: N = 1 the one-CTA sparse_eps_* kernels (per_cta off,
 * kSparseThreads threads), N in {2, 4, 8} the cluster kernels with sparse_cluster_plan's splits for that N and
 * `threads` threads per CTA.  emissions [B][T][C], lens [B], w [nG].  Out: alpha [B][(T + 1) * S], offs [B][T + 1]
 * (slot 0: Z), den [B], grad [B][T][C] and wgrad [nG] (zero on entry: added into), status [B] (zeroed here).
 * Returns 0, 1 when G has no route for N, 77 when the host refused the threads.
 */
int emu_bc_den(int B, int T, int C, const float* emissions, const int32_t* lens, int S, int nG, const uint8_t* g_flags,
               const int32_t* g_src, const int32_t* g_dst, const int32_t* g_label, const float* w, int N, int threads,
               float* alpha, double* offs, float* den, float* grad, float* wgrad, int32_t* status) {
  using namespace gtnb;
  Tables x;
  tables_of(S, nG, g_flags, g_src, g_dst, g_label, C, &x);
  const SparseTables& t = x.t;
  const long long per = (long long)T * C;
  for (int b = 0; b < B; b++) status[b] = 0;
  if (N == 1) {
    if (!sparse_eps_supported(t.S, t.A, t.E, t.L, t.max_in_all, C)) return 1;
    emu::launch(B, kSparseThreads, sizeof(float) * sparse_fwd_smem_floats(S, C), [&] {
      sparse_eps_forward_kernel(&x.dev, 0, T, C, lens, emissions, per, w, alpha, offs, den, status);
    });
    emu::launch(B, kSparseThreads, sizeof(float) * sparse_bwd_smem_floats(S, t.A + t.E, C), [&] {
      sparse_eps_backward_kernel(&x.dev, 0, T, C, lens, emissions, per, w, alpha, offs, 1.0f, grad, per, wgrad);
    });
  } else {
    SparseSplit sp{};
    if (sparse_cluster_plan(t, C, N, &sp) != N) return 1;
    std::vector<int32_t> cut;
    sparse_eps_cluster_cuts(t, sp, &cut);
    cut.push_back(0);
    emu::launch_clusters_dsmem(B * N, N, threads, sizeof(float) * sparse_cl_fwd_smem_floats(S, C, N), [&] {
      sparse_cl_eps_forward_kernel(&x.dev, sp, cut.data(), T, C, lens, emissions, per, w, alpha, offs, den, status);
    });
    emu::launch_clusters_dsmem(B * N, N, threads, sizeof(float) * sparse_cl_bwd_smem_floats(S, C, N, sp.own_out), [&] {
      sparse_cl_eps_backward_kernel(&x.dev, sp, cut.data(), T, C, lens, emissions, per, w, alpha, offs, grad, per,
                                    wgrad);
    });
  }
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

/*
 * The decode's tropical sweep (N as above) and the traceback, as backoff_viterbi_run launches them.  Out: bp
 * [B][T + 1][S], head [B], scores [B], paths and arcs [B][T], status [B] (zeroed here).  Returns as emu_bc_den.
 */
int emu_bc_viterbi(int B, int T, int C, const float* emissions, const int32_t* lens, int S, int nG,
                   const uint8_t* g_flags, const int32_t* g_src, const int32_t* g_dst, const int32_t* g_label,
                   const float* w, int N, int threads, uint16_t* bp, int32_t* head, float* scores, int32_t* paths,
                   int32_t* arcs, int32_t* status) {
  using namespace gtnb;
  Tables x;
  tables_of(S, nG, g_flags, g_src, g_dst, g_label, C, &x);
  const SparseTables& t = x.t;
  const long long per = (long long)T * C;
  const size_t smem = sizeof(float) * sparse_vit_smem_floats(S, C);
  for (int b = 0; b < B; b++) status[b] = 0;
  if (N == 1) {
    if (!sparse_eps_supported(t.S, t.A, t.E, t.L, t.max_in_all, C)) return 1;
    emu::launch(B, kSparseThreads, smem, [&] {
      sparse_eps_viterbi_kernel(&x.dev, T, C, lens, emissions, per, w, bp, head, scores, status);
    });
  } else {
    SparseSplit sp{};
    if (sparse_cluster_plan(t, C, N, &sp) != N) return 1;
    std::vector<int32_t> cut;
    sparse_eps_cluster_cuts(t, sp, &cut);
    cut.push_back(0);
    emu::launch_clusters_dsmem(B * N, N, threads, smem, [&] {
      sparse_cl_eps_viterbi_kernel(&x.dev, sp, cut.data(), T, C, lens, emissions, per, w, bp, head, scores, status);
    });
  }
  emu::launch((B * 32 + 255) / 256, 256, 0, [&] {
    sparse_eps_trace_kernel(&x.dev, B, T, lens, bp, head, paths, arcs, status);
  });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

} // extern "C"
