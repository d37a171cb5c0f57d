/*
 * tests/emu/sparse_emu.cpp -- TEST INFRASTRUCTURE for gtnb_sparse_transitions_loss: the shipped host builders of G's
 * tables and of the numerator products (gtn_b200/csrc/gtnb_product.h), and the SOURCE of k_sparse.cu's kernels (the
 * denominator's forward and backward sweeps, sigma and its fold), run on the CPU (the kernels through
 * tests/emu/simt_emu.h).  Only the launch geometry and the packing of the tables into SparseDev are restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_sparse.cu"
#include "../../gtn_b200/csrc/gtnb_product.h"

#include <cstring>
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

} // namespace

extern "C" {

/*
 * intersect(A, G) from gtnb_product.h's builder (fold or not) and its weights from Wx = [trans_w | sigma]. Call once
 * with out arrays NULL to get the sizes (*n_nodes, *n_arcs, *n_groups), then again with room for them.  Out: flags,
 * src, dst, label, arc_of, tidx, weights; *uniform.
 */
int emu_sparse_product(int N, int nA, const uint8_t* a_flags, const int32_t* a_src, const int32_t* a_dst,
                       const int32_t* a_label, const float* a_w, int S, int nG, const uint8_t* g_flags,
                       const int32_t* g_src, const int32_t* g_dst, const int32_t* g_label, int C, int fold,
                       const float* Wx, int* n_nodes, int* n_arcs, int* n_groups, int* uniform, uint8_t* flags,
                       int32_t* src, int32_t* dst, int32_t* label, int32_t* arc_of, int32_t* tidx, float* weights) {
  const gtnb_graph_view A = view_of(N, nA, a_flags, a_src, a_dst, a_label, a_w);
  const gtnb_graph_view G = view_of(S, nG, g_flags, g_src, g_dst, g_label, nullptr);
  gtnb::SparseTables t;
  gtnb::sparse_tables(G, C, &t);
  gtnb::ProductGraph p;
  gtnb::build_sparse_product(A, G, t, C, fold != 0, &p);
  *n_nodes = (int)p.flags.size();
  *n_arcs = (int)p.src.size();
  *n_groups = (int)t.grp_ptr.size() - 1;
  *uniform = p.uniform ? 1 : 0;
  if (!flags) return 0;
  std::vector<float> pw;
  gtnb::product_weights(p, a_w, Wx, &pw);
  std::memcpy(flags, p.flags.data(), p.flags.size());
  const size_t bytes = p.src.size() * sizeof(int32_t);
  std::memcpy(src, p.src.data(), bytes);
  std::memcpy(dst, p.dst.data(), bytes);
  std::memcpy(label, p.label.data(), bytes);
  std::memcpy(arc_of, p.arc_of.data(), bytes);
  std::memcpy(tidx, p.tidx.data(), bytes);
  std::memcpy(weights, pw.data(), pw.size() * sizeof(float));
  return 0;
}

/*
 * The denominator as trellis_loss_fast runs it on the device route: sigma of G's start groups, then
 * forwardScore(intersect(E_b, G)) for every utterance and its gradients.  emissions [B][T][C], lens[B], G (S nodes,
 * nG arcs), w [nG].  Out: den[B] (float), grad [B][T][C] (zero on entry: added into), wgrad [nG + groups] (zero on
 * entry; the sigma slots are folded into G's by sparse_fold_kernel when fold_grad is set, after the caller added its
 * own there), sigma [groups], status[B].  threads: CTA size (kSparseThreads on the device).  Returns 0, 1 outside the
 * kernels' envelope, 77 when the host refused the threads.
 */
int emu_sparse_den(int B, int T, int C, const float* emissions, const int32_t* lens, int S, int nG,
                   const uint8_t* g_flags, const int32_t* g_src, const int32_t* g_dst, const int32_t* g_label,
                   const float* w, int threads, float* den, float* grad, float* wgrad, float* sigma,
                   int32_t* status) {
  using namespace gtnb;
  const gtnb_graph_view G = view_of(S, nG, g_flags, g_src, g_dst, g_label, nullptr);
  SparseTables t;
  sparse_tables(G, C, &t);
  if (S < 1 || S > kSparseMaxStates || t.A > kSparseMaxArcs || C > kSparseMaxLabels) return 1;
  std::vector<int32_t> flags(t.flags.begin(), t.flags.end());
  const SparseDev dev{t.S, t.A, sparse_den_lanes(t.S, t.A), flags.data(), t.in_ptr.data(), t.in_src.data(),
                      t.in_lab.data(), t.in_arc.data(), t.out_ptr.data(), t.out_dst.data(), t.out_lab.data(),
                      t.out_arc.data()};
  const int K = (int)t.grp_ptr.size() - 1;
  std::vector<float> alpha((size_t)B * (T + 1) * S + 16, 0.0f);
  std::vector<double> offs((size_t)B * (T + 1) + 16, 0.0);
  for (int b = 0; b < B; b++) status[b] = 0;
  if (K > 0)
    emu::launch((K * 32 + 255) / 256, 256, 0, [&] { sparse_sigma_kernel(K, t.grp_ptr.data(), t.grp_arc.data(), w, sigma); });
  emu::launch(B, threads, sizeof(float) * sparse_fwd_smem_floats(S, C), [&] {
    sparse_den_forward_kernel(dev, T, C, lens, emissions, (long long)T * C, w, alpha.data(), offs.data(), den, status);
  });
  emu::launch(B, threads, sizeof(float) * sparse_bwd_smem_floats(S, t.A, C), [&] {
    sparse_den_backward_kernel(dev, T, C, lens, emissions, (long long)T * C, w, alpha.data(), offs.data(), grad,
                               (long long)T * C, wgrad);
  });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

/* sparse_fold_kernel: wgrad[a] += wgrad[nG + k] * exp(w_a - sigma_k) over G's start groups */
int emu_sparse_fold(int S, int nG, const uint8_t* g_flags, const int32_t* g_src, const int32_t* g_dst,
                    const int32_t* g_label, int C, const float* w, const float* sigma, float* wgrad) {
  using namespace gtnb;
  const gtnb_graph_view G = view_of(S, nG, g_flags, g_src, g_dst, g_label, nullptr);
  SparseTables t;
  sparse_tables(G, C, &t);
  const int K = (int)t.grp_ptr.size() - 1;
  if (K > 0)
    emu::launch((K + 255) / 256, 256, 0, [&] {
      sparse_fold_kernel(K, t.grp_ptr.data(), t.grp_arc.data(), nG, w, sigma, wgrad);
    });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

} // extern "C"
