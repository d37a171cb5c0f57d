/*
 * tests/emu/plan_emu.cpp -- TEST INFRASTRUCTURE: the launch plans of the five planned kernel families, called on the
 * CPU exactly as their launchers call them, with each outcome returned as plain integers.
 *
 *   bidir     bidir_plan<E> and bidir_shape_supported (k_bidir.cu)
 *   dense     dense_lanes, dense_smem_bytes, viterbi_dense_supported and viterbi_dense_kernel_for<E> (k_dense.cu)
 *   n-gram    ngram_den_shape and ngram_den_{forward,backward}_kernel_for<START, E> (k_ngram.cu)
 *   implicit  wide_lanes, implicit_elem_mode and implicit_{forward,backward}_kernel_for (k_implicit.cu)
 *   staged    plan, fused_layout and sd_{forward,backward}_staged_kernel_for (k_staged.cu)
 *
 * Nothing is decided here.  What the driver adds is, per family, the table of the instantiations the family compiles
 * (every template argument tuple its *_kernel_for / plan names), so that an outcome names a real kernel: each export
 * returns the index of the table entry the plan's pointer equals, -1 when it equals none (a kernel missing from the
 * table), -2 for a null pointer.  tests/test_plan_coverage.py walks the plans' input domains through these exports.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_dense.cu"
#include "../../gtn_b200/csrc/k_implicit.cu"
#include "../../gtn_b200/csrc/k_ngram.cu"
#include "../../gtn_b200/csrc/k_bidir.cu"
#include "../../gtn_b200/csrc/k_staged.cu"

#include <vector>

using namespace gtnb;

namespace {

using bidir::bidir_ctc_kernel;

template <class K>
const void* vp(K k) {
  return reinterpret_cast<const void*>(k);
}

int index_of(const std::vector<const void*>& table, const void* k) {
  if (!k) return -2;
  for (size_t i = 0; i < table.size(); i++)
    if (table[i] == k) return (int)i;
  return -1;
}

/* element sizes 4, 2 (bf16) and 3 (standing for fp16) in table order: float, bf16_t, f16_t */
int elem_slot(int esize) {
  return esize == 4 ? 0 : (esize == 2 ? 1 : 2);
}

/* bidir_ctc_kernel<NQ, FX, MODE, E>: (NQ, FX, MODE) in {(1,0,0), (2,0,0), (1,1,0), (2,1,0), (1,1,1), (2,1,1)} */
template <class E>
void bidir_rows(std::vector<const void*>& t) {
  t.push_back(vp(bidir_ctc_kernel<1, false, 0, E>));
  t.push_back(vp(bidir_ctc_kernel<2, false, 0, E>));
  t.push_back(vp(bidir_ctc_kernel<1, true, 0, E>));
  t.push_back(vp(bidir_ctc_kernel<2, true, 0, E>));
  t.push_back(vp(bidir_ctc_kernel<1, true, 1, E>));
  t.push_back(vp(bidir_ctc_kernel<2, true, 1, E>));
}
const std::vector<const void*>& bidir_table() {
  static const std::vector<const void*> t = [] {
    std::vector<const void*> v;
    bidir_rows<float>(v);
    bidir_rows<bf16_t>(v);
    bidir_rows<f16_t>(v);
    return v;
  }();
  return t;
}

/* viterbi_dense_kernel<G, BIGRAM, E>: G in {1, 2, 4, 8, 16, 32}, BIGRAM in {false, true} */
template <class E>
void dense_rows(std::vector<const void*>& t) {
  t.push_back(vp(viterbi_dense_kernel<1, false, E>));
  t.push_back(vp(viterbi_dense_kernel<1, true, E>));
  t.push_back(vp(viterbi_dense_kernel<2, false, E>));
  t.push_back(vp(viterbi_dense_kernel<2, true, E>));
  t.push_back(vp(viterbi_dense_kernel<4, false, E>));
  t.push_back(vp(viterbi_dense_kernel<4, true, E>));
  t.push_back(vp(viterbi_dense_kernel<8, false, E>));
  t.push_back(vp(viterbi_dense_kernel<8, true, E>));
  t.push_back(vp(viterbi_dense_kernel<16, false, E>));
  t.push_back(vp(viterbi_dense_kernel<16, true, E>));
  t.push_back(vp(viterbi_dense_kernel<32, false, E>));
  t.push_back(vp(viterbi_dense_kernel<32, true, E>));
}
const std::vector<const void*>& dense_table() {
  static const std::vector<const void*> t = [] {
    std::vector<const void*> v;
    dense_rows<float>(v);
    dense_rows<bf16_t>(v);
    dense_rows<f16_t>(v);
    return v;
  }();
  return t;
}

/* ngram_den_{forward,backward}_kernel<K, START, E>: K in {16, 32}, START in {false, true} */
template <class E>
void ngram_rows(std::vector<const void*>& t, bool backward) {
  if (backward) {
    t.push_back(vp(ngram_den_backward_kernel<16, false, E>));
    t.push_back(vp(ngram_den_backward_kernel<16, true, E>));
    t.push_back(vp(ngram_den_backward_kernel<32, false, E>));
    t.push_back(vp(ngram_den_backward_kernel<32, true, E>));
  } else {
    t.push_back(vp(ngram_den_forward_kernel<16, false, E>));
    t.push_back(vp(ngram_den_forward_kernel<16, true, E>));
    t.push_back(vp(ngram_den_forward_kernel<32, false, E>));
    t.push_back(vp(ngram_den_forward_kernel<32, true, E>));
  }
}
const std::vector<const void*>& ngram_table(bool backward) {
  static const std::vector<const void*> f = [] {
    std::vector<const void*> v;
    ngram_rows<float>(v, false);
    ngram_rows<bf16_t>(v, false);
    ngram_rows<f16_t>(v, false);
    return v;
  }();
  static const std::vector<const void*> b = [] {
    std::vector<const void*> v;
    ngram_rows<float>(v, true);
    ngram_rows<bf16_t>(v, true);
    ngram_rows<f16_t>(v, true);
    return v;
  }();
  return backward ? b : f;
}

/* forward: implicit_forward_kernel<ARC, TROP> and implicit_forward_wide_kernel<G, ARC, TROP> (G in 1..32) over float,
 * then implicit_forward_kernel<false, false, E> for bf16_t, f16_t; rows (ARC, TROP) major, then G = 0, 1, ..., 32 */
template <bool ARC, bool TROP>
void imp_fwd_rows(std::vector<const void*>& t) {
  t.push_back(vp(implicit_forward_kernel<ARC, TROP>));
  t.push_back(vp(implicit_forward_wide_kernel<1, ARC, TROP>));
  t.push_back(vp(implicit_forward_wide_kernel<2, ARC, TROP>));
  t.push_back(vp(implicit_forward_wide_kernel<4, ARC, TROP>));
  t.push_back(vp(implicit_forward_wide_kernel<8, ARC, TROP>));
  t.push_back(vp(implicit_forward_wide_kernel<16, ARC, TROP>));
  t.push_back(vp(implicit_forward_wide_kernel<32, ARC, TROP>));
}
/* backward: implicit_backward_kernel<GG, ARC> and implicit_backward_wide_kernel<G, GG, ARC> over float, rows (ARC, GG)
 * major, then implicit_backward_kernel<GG, false, E> for bf16_t, f16_t */
template <bool ARC, bool GG>
void imp_bwd_rows(std::vector<const void*>& t) {
  t.push_back(vp(implicit_backward_kernel<GG, ARC>));
  t.push_back(vp(implicit_backward_wide_kernel<1, GG, ARC>));
  t.push_back(vp(implicit_backward_wide_kernel<2, GG, ARC>));
  t.push_back(vp(implicit_backward_wide_kernel<4, GG, ARC>));
  t.push_back(vp(implicit_backward_wide_kernel<8, GG, ARC>));
  t.push_back(vp(implicit_backward_wide_kernel<16, GG, ARC>));
  t.push_back(vp(implicit_backward_wide_kernel<32, GG, ARC>));
}
const std::vector<const void*>& implicit_table(bool backward) {
  static const std::vector<const void*> f = [] {
    std::vector<const void*> v;
    imp_fwd_rows<false, false>(v);
    imp_fwd_rows<false, true>(v);
    imp_fwd_rows<true, false>(v);
    imp_fwd_rows<true, true>(v);
    v.push_back(vp(implicit_forward_kernel<false, false, bf16_t>));
    v.push_back(vp(implicit_forward_kernel<false, false, f16_t>));
    return v;
  }();
  static const std::vector<const void*> b = [] {
    std::vector<const void*> v;
    imp_bwd_rows<false, false>(v);
    imp_bwd_rows<false, true>(v);
    imp_bwd_rows<true, false>(v);
    imp_bwd_rows<true, true>(v);
    v.push_back(vp(implicit_backward_kernel<false, false, bf16_t>));
    v.push_back(vp(implicit_backward_kernel<true, false, bf16_t>));
    v.push_back(vp(implicit_backward_kernel<false, false, f16_t>));
    v.push_back(vp(implicit_backward_kernel<true, false, f16_t>));
    return v;
  }();
  return backward ? b : f;
}

/* sd_forward_staged<MODE, G>: MODE in {LOG, TROPICAL, PATH} major, G in {1, 4, 16, 32};
 * sd_backward_staged<TROPICAL, G>: TROPICAL in {false, true} major, G likewise */
template <int MODE>
void staged_fwd_rows(std::vector<const void*>& t) {
  t.push_back(vp(sd_forward_staged<MODE, 1>));
  t.push_back(vp(sd_forward_staged<MODE, 4>));
  t.push_back(vp(sd_forward_staged<MODE, 16>));
  t.push_back(vp(sd_forward_staged<MODE, 32>));
}
template <bool TROPICAL>
void staged_bwd_rows(std::vector<const void*>& t) {
  t.push_back(vp(sd_backward_staged<TROPICAL, 1>));
  t.push_back(vp(sd_backward_staged<TROPICAL, 4>));
  t.push_back(vp(sd_backward_staged<TROPICAL, 16>));
  t.push_back(vp(sd_backward_staged<TROPICAL, 32>));
}
const std::vector<const void*>& staged_table(bool backward) {
  static const std::vector<const void*> f = [] {
    std::vector<const void*> v;
    staged_fwd_rows<MODE_LOG>(v);
    staged_fwd_rows<MODE_TROPICAL>(v);
    staged_fwd_rows<MODE_PATH>(v);
    return v;
  }();
  static const std::vector<const void*> b = [] {
    std::vector<const void*> v;
    staged_bwd_rows<false>(v);
    staged_bwd_rows<true>(v);
    return v;
  }();
  return backward ? b : f;
}

template <class E>
void bidir_outcome(int C, int max_nodes, bool fixed_pitch, bool pair_ok, int32_t* out) {
  const BidirPlan p = bidir_plan<E>(C, max_nodes, fixed_pitch, pair_ok);
  out[1] = p.kernel == bidir_ctc_kernel<2, true, 1, E> || p.kernel == bidir_ctc_kernel<2, true, 0, E> ||
                   p.kernel == bidir_ctc_kernel<2, false, 0, E>
               ? 2
               : 1;
  out[2] = p.fx;
  out[3] = p.pair;
  out[4] = p.nwn;
  out[5] = (int32_t)p.block;
  out[6] = p.lay.total;
  out[7] = index_of(bidir_table(), vp(p.kernel));
}

template <class E>
void dense_outcome(int C, bool bigram, int32_t* out) {
  const int G = dense_lanes(C);
  out[1] = G;
  out[2] = (int32_t)dense_smem_bytes(C);
  out[3] = index_of(dense_table(), vp(viterbi_dense_kernel_for<E>(G, bigram)));
}

template <class E>
void ngram_outcome(int K, bool start, int32_t* out) {
  if (start) {
    out[3] = index_of(ngram_table(false), vp(ngram_den_forward_kernel_for<true, E>(K)));
    out[4] = index_of(ngram_table(true), vp(ngram_den_backward_kernel_for<true, E>(K)));
  } else {
    out[3] = index_of(ngram_table(false), vp(ngram_den_forward_kernel_for<false, E>(K)));
    out[4] = index_of(ngram_table(true), vp(ngram_den_backward_kernel_for<false, E>(K)));
  }
}

template <class E>
void implicit_outcome(int Gf, int Gb, bool arc, bool trop, bool grad_graph, int32_t* out) {
  const void* f = arc ? (trop ? vp(implicit_forward_kernel_for<true, true, E>(Gf))
                              : vp(implicit_forward_kernel_for<true, false, E>(Gf)))
                      : (trop ? vp(implicit_forward_kernel_for<false, true, E>(Gf))
                              : vp(implicit_forward_kernel_for<false, false, E>(Gf)));
  const void* b = arc ? vp(implicit_backward_kernel_for<true, E>(Gb, grad_graph))
                      : vp(implicit_backward_kernel_for<false, E>(Gb, grad_graph));
  out[4] = index_of(implicit_table(false), f);
  out[5] = index_of(implicit_table(true), b);
}

} // namespace

extern "C" {

/* table sizes: family 0 bidir, 1 dense, 2 n-gram forward, 3 n-gram backward, 4 implicit forward, 5 implicit backward,
 * 6 staged forward, 7 staged backward */
int emu_plan_table_size(int family) {
  switch (family) {
    case 0: return (int)bidir_table().size();
    case 1: return (int)dense_table().size();
    case 2: return (int)ngram_table(false).size();
    case 3: return (int)ngram_table(true).size();
    case 4: return (int)implicit_table(false).size();
    case 5: return (int)implicit_table(true).size();
    case 6: return (int)staged_table(false).size();
    case 7: return (int)staged_table(true).size();
    default: return -1;
  }
}

/* out[8]: supported (bidir_shape_supported), NQ, FX, PAIR, nwn, block, lay.total, table index.  esize 4: float, 2: bf16,
 * 3: fp16 (its elements are 2 bytes too; 3 only selects the table's fp16 rows) */
void emu_bidir_plan(int C, int max_nodes, int max_in_deg, int max_out_deg, int fixed_pitch, int pair_ok, int esize,
                    int32_t* out) {
  out[0] = bidir_shape_supported(C, max_nodes, max_in_deg, max_out_deg, esize == 4 ? 4 : 2);
  switch (elem_slot(esize)) {
    case 0: bidir_outcome<float>(C, max_nodes, fixed_pitch != 0, pair_ok != 0, out); break;
    case 1: bidir_outcome<bf16_t>(C, max_nodes, fixed_pitch != 0, pair_ok != 0, out); break;
    default: bidir_outcome<f16_t>(C, max_nodes, fixed_pitch != 0, pair_ok != 0, out); break;
  }
}

/* out[4]: viterbi_dense_supported, G (dense_lanes), dense_smem_bytes, table index */
void emu_dense_plan(int C, int bigram, int esize, int32_t* out) {
  out[0] = viterbi_dense_supported(C);
  switch (elem_slot(esize)) {
    case 0: dense_outcome<float>(C, bigram != 0, out); break;
    case 1: dense_outcome<bf16_t>(C, bigram != 0, out); break;
    default: dense_outcome<f16_t>(C, bigram != 0, out); break;
  }
}

/* out[5]: K, lanes, threads (ngram_den_shape), forward and backward table indices; start: ASG's START mode */
void emu_ngram_plan(int C, int start, int esize, int32_t* out) {
  int K, lanes, threads;
  ngram_den_shape(C, &K, &lanes, &threads);
  out[0] = K;
  out[1] = lanes;
  out[2] = threads;
  switch (elem_slot(esize)) {
    case 0: ngram_outcome<float>(K, start != 0, out); break;
    case 1: ngram_outcome<bf16_t>(K, start != 0, out); break;
    default: ngram_outcome<f16_t>(K, start != 0, out); break;
  }
}

/* out[6]: forward G, backward G (wide_lanes), implicit_elem_mode of each (0: GTNB_OK), forward and backward table
 * indices.  dtype: GTNB_F32 / GTNB_BF16 / GTNB_F16 */
void emu_implicit_plan(int max_in, int max_out, int max_nodes, int C, int arc, int tropical, int grad_graph, int dtype,
                       int32_t* out) {
  const int Gf = wide_lanes(max_in, max_out, max_nodes, C, false, arc != 0);
  const int Gb = wide_lanes(max_in, max_out, max_nodes, C, true, arc != 0);
  out[0] = Gf;
  out[1] = Gb;
  out[2] = implicit_elem_mode(dtype, Gf, arc != 0, tropical != 0);
  out[3] = implicit_elem_mode(dtype, Gb, arc != 0, false);
  if (dtype == GTNB_BF16)
    implicit_outcome<bf16_t>(Gf, Gb, arc != 0, tropical != 0, grad_graph != 0, out);
  else if (dtype == GTNB_F16)
    implicit_outcome<f16_t>(Gf, Gb, arc != 0, tropical != 0, grad_graph != 0, out);
  else
    implicit_outcome<float>(Gf, Gb, arc != 0, tropical != 0, grad_graph != 0, out);
}

/* B graphs' L, sg_A, sg_N; out[10]: ok, G, max_L, ls (log2 stages), forward and backward layout totals,
 * fused_layout's verdict and total, and the table indices of the log forward and backward for G */
void emu_staged_plan(int B, const int32_t* L, const int32_t* sg_A, const int32_t* sg_N, int max_lvl_nodes,
                     int max_lvl_arcs, int32_t* out) {
  std::vector<GraphMeta> meta(B > 0 ? B : 1);
  for (int b = 0; b < B; b++) {
    meta[b] = GraphMeta{};
    meta[b].L = L[b];
    meta[b].sg_A = sg_A[b];
    meta[b].sg_N = sg_N[b];
  }
  const StagedPlan p = plan(meta.data(), B, max_lvl_nodes, max_lvl_arcs);
  for (int i = 0; i < 10; i++) out[i] = 0;
  out[0] = p.ok;
  if (!p.ok) return;
  out[1] = p.G;
  out[2] = p.max_L;
  out[3] = p.fwd.log2_stages;
  out[4] = p.fwd.total;
  out[5] = p.bwd.total;
  Layout lay = p.bwd;
  out[6] = fused_layout(lay, max_lvl_nodes, max_lvl_arcs);
  out[7] = lay.total;
  out[8] = index_of(staged_table(false), vp(sd_forward_staged_kernel_for(MODE_LOG, p.G)));
  out[9] = index_of(staged_table(true), vp(sd_backward_staged_kernel_for(false, p.G)));
}

} // extern "C"
