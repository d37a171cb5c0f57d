/*
 * tests/emu/trellis_half_emu.cpp -- TEST INFRASTRUCTURE: the native route of gtnb_ngram_ctc_loss_typed /
 * gtnb_asg_loss_typed and gtnb_viterbi_dense_typed, from the SOURCE of gtn_b200/csrc/k_ngram.cu (the numerator graphs,
 * the dense trellis), k_implicit.cu (the numerator's sweeps) and k_dense.cu (the factored Viterbi) on the CPU through
 * tests/emu/simt_emu.h, for any element type of the emissions: float, bf16_t or f16_t.  As on the device, the
 * gradients stay float32 (the caller rounds them once).  ngram_emu.cpp / asg_emu.cpp / dense_emu.cpp run the float32
 * kernels the same way; only the launch geometry and the table slabs are restated here.  Also exports k_implicit.cu's
 * host check of which modes a 16-bit lattice may take.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_dense.cu"
#include "../../gtn_b200/csrc/k_implicit.cu"
#include "../../gtn_b200/csrc/k_ngram.cu"

#include <vector>

using gtnb::GraphMeta;

namespace {

/*
 * The trellis criterion as trellis_loss_fast runs it: asg = 0 n-gram CTC (W [C*C], the folded numerator), 1 ASG
 * (trans_w [C + C*C], start mode).  Outputs: den[B], num[B], status[2B], grad [B][T][C] (zero on entry), trans_grad
 * (the denominator's plus the scattered numerator's, n-gram before the sigma fold), arc_grad [sum A] and
 * node_scores [sum (T+1) * pitch] of the numerator.
 */
template <class E>
int run_trellis(int asg, int B, int T, int C, const E* emissions, const int32_t* input_lens, const float* W,
                const int32_t* targets, const int32_t* target_lens, int blank, float* den, float* num,
                int32_t* status, float* grad, float* trans_grad, float* arc_grad, float* node_scores) {
  using namespace gtnb;
  if (C < 1 || C > kNgramMaxC) return 1;
  const long long nTrans = (asg ? C : 0) + (long long)C * C;
  std::vector<GraphMeta> meta(B);
  std::vector<int32_t> tgt_off(B), Tb(B);
  long long nodes = 0, arcs = 0, scores_len = 0, acc = 0, toff = 0, gg = 0;
  int maxN = 0, maxA = 0;
  for (int b = 0; b < B; b++) {
    const int U = target_lens[b];
    const int N = asg ? U + 1 : 2 * U + 2;
    const int A = asg ? 2 * U : 3 * N; // (n-gram: a bound; the build gives the count)
    GraphMeta& m = meta[b];
    std::memset(&m, 0, sizeof(m));
    m.sg_node_base = nodes;
    m.sg_arc_base = arcs;
    m.acc_base = acc;
    m.grad_graph_off = gg;
    m.emis_off = (long long)b * T * C;
    m.node_base = scores_len;
    m.T = Tb[b] = input_lens ? input_lens[b] : T;
    m.sg_N = N;
    m.sg_A = A;
    tgt_off[b] = (int32_t)toff;
    toff += U;
    nodes += N + 1;
    arcs += std::max(A, 1);
    gg += A;
    acc += asg ? 1 : 2;
    scores_len += (long long)(T + 1) * ((N + 3) & ~3);
    maxN = std::max(maxN, N);
  }
  std::vector<uint8_t> flags(nodes, 0);
  std::vector<int32_t> in_ptr(nodes, 0), in_src(arcs, 0), in_label(arcs, 0), in_arc(arcs, 0), il(arcs, 0),
      ol(arcs, 0), acc_nodes(acc, 0), map(std::max(gg, 1ll), 0);
  std::vector<float> in_w(arcs, 0.0f), sigma(C), ggrad(std::max(gg, 1ll), 0.0f), tg(nTrans + C, 0.0f);
  std::vector<float> alpha((size_t)(asg ? asg_alpha_floats(B, T, C) : (long long)B * (T + 1) * C), 0.0f);
  std::vector<float> minus1(B, -1.0f);
  for (int b = 0; b < 2 * B; b++) status[b] = 0;

  if (asg) {
    emu::launch(B, 256, 0, [&] {
      asg_num_build_kernel(meta.data(), targets, tgt_off.data(), target_lens, C, W, flags.data(), in_ptr.data(),
                           in_src.data(), in_label.data(), in_arc.data(), in_w.data(), il.data(), ol.data(),
                           acc_nodes.data(), map.data());
    });
  } else {
    emu::launch((C * 32 + 255) / 256, 256, 0, [&] { ngram_sigma_kernel(C, W, sigma.data()); });
    emu::launch(B, 256, 0, [&] {
      ngram_num_build_kernel(meta.data(), targets, tgt_off.data(), target_lens, blank, C, W, sigma.data(),
                             flags.data(), in_ptr.data(), in_src.data(), in_label.data(), in_arc.data(), in_w.data(),
                             il.data(), ol.data(), acc_nodes.data(), map.data());
    });
    for (int b = 0; b < B; b++) meta[b].sg_A = in_ptr[meta[b].sg_node_base + meta[b].sg_N];
  }
  for (int b = 0; b < B; b++) maxA = std::max(maxA, meta[b].sg_A);
  std::vector<float> scores((size_t)scores_len + 16, 0.0f);
  const ImpLayout lf = make_imp_layout(maxN, maxA, false);
  emu::launch(B, kImpThreads, lf.total, [&] {
    implicit_forward_kernel<false, false, E>(meta.data(), flags.data(), in_ptr.data(), in_src.data(), in_label.data(),
                                             in_w.data(), emissions, scores.data(), num, status + B, C, lf);
  });
  const ImpLayout lb = make_imp_layout(maxN, maxA, true);
  emu::launch(B, kImpThreads, lb.total, [&] {
    implicit_backward_kernel<true, false, E>(meta.data(), flags.data(), in_ptr.data(), in_src.data(), in_label.data(),
                                             in_w.data(), in_arc.data(), ggrad.data(), emissions, scores.data(), num,
                                             minus1.data(), grad, (long long)T * C, C, lb);
  });
  int K, lanes, threads;
  ngram_den_shape(C, &K, &lanes, &threads);
#define RUN(KK, START)                                                                                          \
  do {                                                                                                          \
    emu::launch(B, threads, 0, [&] {                                                                            \
      ngram_den_forward_kernel<KK, START, E>(T, C, lanes, Tb.data(), emissions, (long long)T * C, W,            \
                                             alpha.data(), den, status);                                        \
    });                                                                                                         \
    emu::launch(B, threads, 0, [&] {                                                                            \
      ngram_den_backward_kernel<KK, START, E>(T, C, lanes, Tb.data(), emissions, (long long)T * C, W,           \
                                              alpha.data(), den, grad, (long long)T * C, tg.data());            \
    });                                                                                                         \
  } while (0)
  if (K == 16 && asg)
    RUN(16, true);
  else if (K == 16)
    RUN(16, false);
  else if (asg)
    RUN(32, true);
  else
    RUN(32, false);
#undef RUN
  for (long long a = 0; a < gg; a++) tg[map[a]] += ggrad[a];
  for (long long k = 0; k < nTrans; k++) trans_grad[k] = tg[k];
  for (long long a = 0; a < gg; a++) arc_grad[a] = ggrad[a];
  for (long long k = 0; k < scores_len; k++) node_scores[k] = scores[k];
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

/* launch_viterbi_dense's geometry for any C <= 224 */
template <class E>
int run_dense(int B, int T, int C, const E* emissions, const int32_t* lens, int bigram, const float* trans,
              int32_t* paths, float* scores) {
  using namespace gtnb;
  if (C < 1 || C > 224) return 1;
  int G = 1;
  while (G < 32 && C * (G * 2) <= kDenseThreads) G *= 2;
  const size_t smem = sizeof(float) * ((size_t)C * (C + 32 / G) + 2 * (size_t)C);
  std::vector<uint8_t> bp((size_t)B * std::max(T, 1) * dense_bp_pitch(C), 0);
  const float empty = -std::numeric_limits<float>::infinity();
#define RUN(G_)                                                                                                 \
  emu::launch(B, kDenseThreads, smem, [&] {                                                                     \
    if (bigram)                                                                                                 \
      viterbi_dense_kernel<G_, true, E>(T, C, lens, emissions, (long long)T * C, trans, bp.data(), paths, scores, \
                                        empty);                                                                 \
    else                                                                                                        \
      viterbi_dense_kernel<G_, false, E>(T, C, lens, emissions, (long long)T * C, trans, bp.data(), paths,      \
                                         scores, empty);                                                        \
  })
  switch (G) {
    case 1: RUN(1); break;
    case 2: RUN(2); break;
    case 4: RUN(4); break;
    case 8: RUN(8); break;
    case 16: RUN(16); break;
    default: RUN(32); break;
  }
#undef RUN
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

} // namespace

extern "C" {

/* run_trellis for emissions of element type dtype (GTNB_F32, GTNB_BF16, GTNB_F16) */
int emu_trellis_typed(int asg, int B, int T, int C, const void* emissions, int dtype, const int32_t* input_lens,
                      const float* W, const int32_t* targets, const int32_t* target_lens, int blank, float* den,
                      float* num, int32_t* status, float* grad, float* trans_grad, float* arc_grad,
                      float* node_scores) {
  using gtnb::bf16_t;
  using gtnb::f16_t;
  if (dtype == GTNB_BF16)
    return run_trellis(asg, B, T, C, static_cast<const bf16_t*>(emissions), input_lens, W, targets, target_lens, blank,
                       den, num, status, grad, trans_grad, arc_grad, node_scores);
  if (dtype == GTNB_F16)
    return run_trellis(asg, B, T, C, static_cast<const f16_t*>(emissions), input_lens, W, targets, target_lens, blank,
                       den, num, status, grad, trans_grad, arc_grad, node_scores);
  return run_trellis(asg, B, T, C, static_cast<const float*>(emissions), input_lens, W, targets, target_lens, blank,
                     den, num, status, grad, trans_grad, arc_grad, node_scores);
}

/* viterbi_dense_kernel for emissions of element type dtype; bigram: the kind (GTNB_DENSE_BIGRAM) */
int emu_viterbi_dense_typed(int B, int T, int C, const void* emissions, int dtype, const int32_t* lens, int bigram,
                            const float* trans, int32_t* paths, float* scores) {
  using gtnb::bf16_t;
  using gtnb::f16_t;
  if (dtype == GTNB_BF16)
    return run_dense(B, T, C, static_cast<const bf16_t*>(emissions), lens, bigram, trans, paths, scores);
  if (dtype == GTNB_F16)
    return run_dense(B, T, C, static_cast<const f16_t*>(emissions), lens, bigram, trans, paths, scores);
  return run_dense(B, T, C, static_cast<const float*>(emissions), lens, bigram, trans, paths, scores);
}

/* k_implicit.cu's host check: may a lattice of element type dtype take the mode (lanes G, arc-label, tropical)? */
int emu_implicit_elem_mode(int dtype, int G, int arc, int tropical) {
  return gtnb::implicit_elem_mode(dtype, G, arc != 0, tropical != 0);
}
/* k_implicit.cu's choice of lanes per node for a graph operand (0: the kernels that have 16-bit instantiations) */
int emu_wide_lanes(int max_in, int max_out, int maxN, int C, int backward) {
  return gtnb::wide_lanes(max_in, max_out, maxN, C, backward != 0);
}

} // extern "C"
