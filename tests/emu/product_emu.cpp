/*
 * tests/emu/product_emu.cpp -- TEST INFRASTRUCTURE for gtnb_graph_transitions_loss: the shipped host builder of its
 * numerator products (gtn_b200/csrc/gtnb_product.h) and the SOURCE of k_ngram.cu's product_fold_kernel, run on the
 * CPU (the kernel through tests/emu/simt_emu.h).  Only the launch geometry is restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_implicit.cu"
#include "../../gtn_b200/csrc/k_ngram.cu"
#include "../../gtn_b200/csrc/gtnb_product.h"

#include <cstring>
#include <vector>

extern "C" {

/*
 * The product of graph A (N nodes, nA arcs; weights w, nullable) with G of the given kind (0 ASG, 1 BIGRAM), folded
 * or not, and its weights from Wx.  Call once with out arrays NULL to get the sizes (*n_nodes, *n_arcs), then again
 * with room for them.  Out: flags, src, dst, label, arc_of, tidx, weights.
 */
int emu_build_product(int N, int nA, const uint8_t* flags_in, const int32_t* src_in, const int32_t* dst_in,
                      const int32_t* olabel, const float* w, int C, int bigram, int fold, const float* Wx,
                      int* n_nodes, int* n_arcs, uint8_t* flags, int32_t* src, int32_t* dst, int32_t* label,
                      int32_t* arc_of, int32_t* tidx, float* weights) {
  gtnb_graph_view v{};
  v.num_nodes = N;
  v.num_arcs = nA;
  v.node_flags = flags_in;
  v.arc_src = src_in;
  v.arc_dst = dst_in;
  v.arc_ilabel = v.arc_olabel = olabel;
  v.weights = w;
  gtnb::ProductGraph p;
  gtnb::build_product(v, C, bigram != 0, fold != 0, &p);
  *n_nodes = (int)p.flags.size();
  *n_arcs = (int)p.src.size();
  if (!flags) return 0;
  std::vector<float> pw;
  gtnb::product_weights(p, w, Wx, &pw);
  std::memcpy(flags, p.flags.data(), p.flags.size());
  const size_t A = p.src.size() * sizeof(int32_t);
  std::memcpy(src, p.src.data(), A);
  std::memcpy(dst, p.dst.data(), A);
  std::memcpy(label, p.label.data(), A);
  std::memcpy(arc_of, p.arc_of.data(), A);
  std::memcpy(tidx, p.tidx.data(), A);
  std::memcpy(weights, pw.data(), pw.size() * sizeof(float));
  return 0;
}

/* product_fold_kernel over n arcs, as launch_product_fold launches it */
int emu_product_fold(long long n, const float* w_A, const int32_t* arc_of, const float* W, int nW, const float* sigma,
                     const int32_t* tidx, float* out) {
  if (n > 0)
    emu::launch((int)((n + 255) / 256), 256, 0, [&] { gtnb::product_fold_kernel(n, w_A, arc_of, W, nW, sigma, tidx, out); });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

} // extern "C"
