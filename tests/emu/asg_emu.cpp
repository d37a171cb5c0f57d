/*
 * tests/emu/asg_emu.cpp -- TEST INFRASTRUCTURE: the device side of gtnb_asg_loss_ex as asg_loss_ex_fast runs it,
 * from the SOURCE of gtn_b200/csrc/k_ngram.cu (ASG's numerator graphs, the dense trellis in its start mode) and
 * k_implicit.cu (the numerator's sweeps), on the CPU through tests/emu/simt_emu.h.  Only the launch geometry, the
 * table slabs and the scatter of the numerator's arc gradients (launch_scatter_add: dst[map[a]] += src[a]) are
 * restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_implicit.cu"
#include "../../gtn_b200/csrc/k_ngram.cu"

#include <vector>

using gtnb::GraphMeta;

extern "C" {

/*
 * emissions [B][T][C], input_lens[B] (nullable), trans_w [C + C*C], targets concatenated, target_lens[B].
 * Out: losses[B] (den - num), grad [B][T][C] (zero on entry), trans_grad [C + C*C], status[2B] (denominator,
 * numerator).  Returns 0, 1 for C above the kernels' limit, 77 when the host refused the threads.
 */
int emu_asg(int B, int T, int C, const float* emissions, const int32_t* input_lens, const float* trans_w,
            const int32_t* targets, const int32_t* target_lens, float* losses, float* grad, float* trans_grad,
            int32_t* status) {
  using namespace gtnb;
  if (C < 1 || C > kNgramMaxC) return 1;
  const long long nTrans = C + (long long)C * C;
  std::vector<GraphMeta> meta(B);
  std::vector<int32_t> tgt_off(B), Tb(B);
  long long nodes = 0, arcs = 0, scores_len = 0, acc = 0, toff = 0, gg = 0;
  int maxN = 0, maxA = 0;
  for (int b = 0; b < B; b++) {
    const int U = target_lens[b], N = U + 1, A = 2 * U;
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
    acc += 1;
    scores_len += (long long)(T + 1) * ((N + 3) & ~3);
    maxN = std::max(maxN, N);
    maxA = std::max(maxA, A);
  }
  std::vector<uint8_t> flags(nodes, 0);
  std::vector<int32_t> in_ptr(nodes, 0), in_src(arcs, 0), in_label(arcs, 0), in_arc(arcs, 0), il(arcs, 0),
      ol(arcs, 0), acc_nodes(acc, 0), map(std::max(gg, 1ll), 0);
  std::vector<float> in_w(arcs, 0.0f), ggrad(std::max(gg, 1ll), 0.0f), tg(nTrans, 0.0f);
  std::vector<float> alpha((size_t)asg_alpha_floats(B, T, C), 0.0f), den(B), num(B), minus1(B, -1.0f);
  for (int b = 0; b < 2 * B; b++) status[b] = 0;

  emu::launch(B, 256, 0, [&] {
    asg_num_build_kernel(meta.data(), targets, tgt_off.data(), target_lens, C, trans_w, flags.data(), in_ptr.data(),
                         in_src.data(), in_label.data(), in_arc.data(), in_w.data(), il.data(), ol.data(),
                         acc_nodes.data(), map.data());
  });
  std::vector<float> scores((size_t)scores_len + 16, 0.0f);
  const ImpLayout lf = make_imp_layout(maxN, maxA, false);
  emu::launch(B, kImpThreads, lf.total, [&] {
    implicit_forward_kernel(meta.data(), flags.data(), in_ptr.data(), in_src.data(), in_label.data(), in_w.data(),
                            emissions, scores.data(), num.data(), status + B, C, lf);
  });
  const ImpLayout lb = make_imp_layout(maxN, maxA, true);
  emu::launch(B, kImpThreads, lb.total, [&] {
    implicit_backward_kernel<true>(meta.data(), flags.data(), in_ptr.data(), in_src.data(), in_label.data(),
                                   in_w.data(), in_arc.data(), ggrad.data(), emissions, scores.data(), num.data(),
                                   minus1.data(), grad, (long long)T * C, C, lb);
  });
  int K, lanes, threads;
  ngram_den_shape(C, &K, &lanes, &threads);
#define RUN(KK)                                                                                                 \
  do {                                                                                                          \
    emu::launch(B, threads, 0, [&] {                                                                            \
      ngram_den_forward_kernel<KK, true>(T, C, lanes, Tb.data(), emissions, (long long)T * C, trans_w,         \
                                         alpha.data(), den.data(), status);                                     \
    });                                                                                                         \
    emu::launch(B, threads, 0, [&] {                                                                            \
      ngram_den_backward_kernel<KK, true>(T, C, lanes, Tb.data(), emissions, (long long)T * C, trans_w,        \
                                          alpha.data(), den.data(), grad, (long long)T * C, tg.data());         \
    });                                                                                                         \
  } while (0)
  if (K == 16)
    RUN(16);
  else
    RUN(32);
#undef RUN
  for (long long a = 0; a < gg; a++) tg[map[a]] += ggrad[a];
  for (int b = 0; b < B; b++) losses[b] = den[b] - num[b];
  for (long long k = 0; k < nTrans; k++) trans_grad[k] = tg[k];
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

} // extern "C"
