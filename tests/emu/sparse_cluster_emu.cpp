/*
 * tests/emu/sparse_cluster_emu.cpp -- TEST INFRASTRUCTURE for the cluster sweeps of k_sparse.cu (sparse_cl_*): the
 * shipped host builders of G's tables, of the cluster splits and of the cluster plan (gtn_b200/csrc/gtnb_product.h),
 * and the SOURCE of the cluster kernels and of the one-CTA kernels they must reproduce, run on the CPU through
 * tests/emu/simt_emu.h and simt_emu_dsmem.h (a cluster's CTAs run concurrently; remote shared-memory stores go to the
 * peer CTA's emulated shared memory).  Only the launch geometry and the packing of the tables into SparseDev are
 * restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_sparse.cu"
#include "../../gtn_b200/csrc/gtnb_product.h"

#include <cstring>
#include <vector>

namespace {

struct Tables {
  gtnb::SparseTables t;
  std::vector<int32_t> flags;
  gtnb::SparseDev dev;
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
  const gtnb::SparseTables& t = x->t;
  x->flags.assign(t.flags.begin(), t.flags.end());
  x->dev = gtnb::SparseDev{t.S, t.A, gtnb::sparse_den_lanes(t.S, t.A), x->flags.data(), t.in_ptr.data(),
                           t.in_src.data(), t.in_lab.data(), t.in_arc.data(), t.out_ptr.data(), t.out_dst.data(),
                           t.out_lab.data(), t.out_arc.data()};
}

} // namespace

extern "C" {

/*
 * sparse_cluster_plan for G (force: 0 the smallest N that fits, else that N alone) -> N or 0.  Out, when N > 0: the
 * splits in_split / out_split [N + 1] and the arcs every rank owns in_arcs / out_arcs [N]; always max_deg[2], G's
 * largest in- and out-degree.
 */
int emu_cluster_plan(int S, int nG, const uint8_t* g_flags, const int32_t* g_src, const int32_t* g_dst,
                     const int32_t* g_label, int C, int force, int32_t* in_split, int32_t* out_split, int32_t* in_arcs,
                     int32_t* out_arcs, int32_t* max_deg) {
  Tables x;
  tables_of(S, nG, g_flags, g_src, g_dst, g_label, C, &x);
  max_deg[0] = x.t.max_in;
  max_deg[1] = x.t.max_out;
  gtnb::SparseSplit sp{};
  const int N = gtnb::sparse_cluster_plan(x.t, C, force, &sp);
  for (int r = 0; r < N; r++) {
    in_arcs[r] = x.t.in_ptr[sp.in[r + 1]] - x.t.in_ptr[sp.in[r]];
    out_arcs[r] = x.t.out_ptr[sp.out[r + 1]] - x.t.out_ptr[sp.out[r]];
  }
  if (N) {
    std::memcpy(in_split, sp.in, sizeof(int32_t) * (N + 1));
    std::memcpy(out_split, sp.out, sizeof(int32_t) * (N + 1));
  }
  return N;
}

/*
 * The denominator's two sweeps over G for every utterance: N = 1 the one-CTA kernels (kSparseThreads threads), N in
 * {2, 4, 8} the cluster kernels with sparse_cluster_plan's splits for that N and `threads` threads per CTA.  emissions
 * [B][T][C], lens [B], w [nG].  Out: alpha [B][(T + 1) * S], offs [B][T + 1] (slot 0: Z), den [B], grad [B][T][C] and
 * wgrad [nG] (zero on entry: added into), status [B] (zeroed here).  Returns 0, 1 when G has no plan for N, 77 when
 * the host refused the threads.
 */
int emu_cluster_den(int B, int T, int C, const float* emissions, const int32_t* lens, int S, int nG,
                    const uint8_t* g_flags, const int32_t* g_src, const int32_t* g_dst, const int32_t* g_label,
                    const float* w, int N, int threads, float* alpha, double* offs, float* den, float* grad,
                    float* wgrad, int32_t* status) {
  using namespace gtnb;
  Tables x;
  tables_of(S, nG, g_flags, g_src, g_dst, g_label, C, &x);
  const long long per = (long long)T * C;
  for (int b = 0; b < B; b++) status[b] = 0;
  if (N == 1) {
    emu::launch(B, kSparseThreads, sizeof(float) * sparse_fwd_smem_floats(S, C), [&] {
      sparse_den_forward_kernel(x.dev, T, C, lens, emissions, per, w, alpha, offs, den, status);
    });
    emu::launch(B, kSparseThreads, sizeof(float) * sparse_bwd_smem_floats(S, x.t.A, C), [&] {
      sparse_den_backward_kernel(x.dev, T, C, lens, emissions, per, w, alpha, offs, grad, per, wgrad);
    });
  } else {
    SparseSplit sp{};
    if (sparse_cluster_plan(x.t, C, N, &sp) != N) return 1;
    emu::launch_clusters_dsmem(B * N, N, threads, sizeof(float) * sparse_cl_fwd_smem_floats(S, C, N), [&] {
      sparse_cl_den_forward_kernel(x.dev, sp, T, C, lens, emissions, per, w, alpha, offs, den, status);
    });
    emu::launch_clusters_dsmem(B * N, N, threads, sizeof(float) * sparse_cl_bwd_smem_floats(S, C, N, sp.own_out), [&] {
      sparse_cl_den_backward_kernel(x.dev, sp, T, C, lens, emissions, per, w, alpha, offs, grad, per, wgrad);
    });
  }
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

/*
 * The decode's tropical sweep (N as above) and the traceback.  Out: bp [B][T][S], head [B], scores [B], paths and
 * arcs [B][T], status [B] (zeroed here).  Returns as emu_cluster_den.
 */
int emu_cluster_viterbi(int B, int T, int C, const float* emissions, const int32_t* lens, int S, int nG,
                        const uint8_t* g_flags, const int32_t* g_src, const int32_t* g_dst, const int32_t* g_label,
                        const float* w, int N, int threads, uint16_t* bp, int32_t* head, float* scores, int32_t* paths,
                        int32_t* arcs, int32_t* status) {
  using namespace gtnb;
  Tables x;
  tables_of(S, nG, g_flags, g_src, g_dst, g_label, C, &x);
  const long long per = (long long)T * C;
  const size_t smem = sizeof(float) * sparse_vit_smem_floats(S, C);
  for (int b = 0; b < B; b++) status[b] = 0;
  if (N == 1) {
    emu::launch(B, kSparseThreads, smem, [&] {
      sparse_viterbi_forward_kernel(x.dev, T, C, lens, emissions, per, w, bp, head, scores, status);
    });
  } else {
    SparseSplit sp{};
    if (sparse_cluster_plan(x.t, C, N, &sp) != N) return 1;
    emu::launch_clusters_dsmem(B * N, N, threads, smem, [&] {
      sparse_cl_viterbi_forward_kernel(x.dev, sp, T, C, lens, emissions, per, w, bp, head, scores, status);
    });
  }
  emu::launch((B * 32 + 255) / 256, 256, 0, [&] {
    sparse_viterbi_trace_kernel(x.dev, B, T, lens, bp, head, paths, arcs, status);
  });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

} // extern "C"
