/*
 * tests/emu/align_async_emu.cpp -- TEST INFRASTRUCTURE: runs the SOURCE of the whole device route of
 * gtnb_ctc_align_async / gtnb_ngram_ctc_align_async / gtnb_asg_align_async on the CPU through tests/emu/simt_emu.h:
 * k_ctc.cu's prepare kernel, the numerator build kernels (k_ctc.cu's ctc_build_kernel; k_ngram.cu's ngram_tau_kernel
 * then ngram_num_build_kernel, or asg_num_build_kernel), k_implicit.cu's tropical forward and implicit_trace_kernel,
 * and k_ctc.cu's align_async_finalize_kernel.  Only the launch geometry (apart from the traceback's staged block,
 * trace_layout's) and the bound-sized slabs are restated here; the bound-uniform descriptors of utterances 0 and 1 come
 * from the caller.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_ctc.cu"
#include "../../gtn_b200/csrc/k_implicit.cu"
#include "../../gtn_b200/csrc/k_ngram.cu"

#include <vector>

using gtnb::GraphMeta;

extern "C" {

/*
 * kind: 0 CTC, 1 n-gram CTC, 2 ASG.  m01: composed_alloc's descriptors of utterances 0 and 1 at the bounds; N, A: the
 * bound numerator's nodes and in-entries.  emissions [B][T][C] float32; trans_w: n-gram W [C*C], ASG [C + C*C] (NULL
 * for CTC); targets [B][S]; input_lens nullable.  Outputs paths / tokens [B][T], scores [B], status [B].
 */
int emu_align_async(int kind, int B, int T, int C, int S, int N, int A, const GraphMeta* m01,
                    const float* emissions, const float* trans_w, const int32_t* input_lens, const int32_t* targets,
                    const int32_t* target_lens, int blank, int32_t* paths, int32_t* tokens, float* scores,
                    int32_t* status) {
  using namespace gtnb;
  std::vector<GraphMeta> meta(B);
  std::vector<int32_t> small(3 * B), valid(B), kstatus(2 * B);
  std::vector<float> deltas(B);
  // the slabs at composed_alloc's strides (m1 - m0), plus slack
  const long long dn = m01[1].sg_node_base - m01[0].sg_node_base, da = m01[1].sg_arc_base - m01[0].sg_arc_base;
  const long long dsc = m01[1].node_base - m01[0].node_base, dacc = m01[1].acc_base - m01[0].acc_base;
  const long long nN = (long long)B * std::max(dn, (long long)N + 1) + 16;
  const long long nA = (long long)B * std::max(da, (long long)std::max(A, 1)) + 16;
  std::vector<uint8_t> flags(nN, 0);
  std::vector<int32_t> in_ptr(nN, 0), in_src(nA, 0), in_label(nA, 0), in_arc(nA, 0), ilabel(nA), olabel(nA),
      map(nA, 0), acc((long long)B * std::max(dacc, 4ll) + 16, 0), arcs((long long)B * T + 1, -7);
  std::vector<float> in_w(nA, 0.0f), tau(C > 0 ? C : 1);
  std::vector<float> sc((long long)B * std::max(dsc, (long long)m01[0].cap_N) + 16, 0.0f), out((size_t)B + 1);
  emu::launch((B + 7) / 8, 256, 0, [&] {
    if (kind == 0)
      ctc_async_prepare_kernel<AsyncGraph::Ctc>(B, S, T, C, m01[0], m01[1], input_lens, targets, target_lens,
                                                meta.data(), small.data(), deltas.data(), valid.data(),
                                                kstatus.data());
    else if (kind == 1)
      ctc_async_prepare_kernel<AsyncGraph::Ngram>(B, S, T, C, m01[0], m01[1], input_lens, targets, target_lens,
                                                  meta.data(), small.data(), deltas.data(), valid.data(),
                                                  kstatus.data());
    else
      ctc_async_prepare_kernel<AsyncGraph::Asg>(B, S, T, C, m01[0], m01[1], input_lens, targets, target_lens,
                                                meta.data(), small.data(), deltas.data(), valid.data(),
                                                kstatus.data());
  });
  const int32_t* off = small.data();
  const int32_t* lens = small.data() + B;
  if (kind == 1) emu::launch((C * 32 + 255) / 256, 256, 0, [&] { ngram_tau_kernel(C, trans_w, tau.data()); });
  emu::launch(B, 256, 0, [&] {
    if (kind == 0)
      ctc_build_kernel(meta.data(), targets, off, lens, blank, C, flags.data(), in_ptr.data(), in_src.data(),
                       in_label.data(), in_arc.data(), in_w.data(), ilabel.data(), olabel.data(), acc.data());
    else if (kind == 1)
      ngram_num_build_kernel(meta.data(), targets, off, lens, blank, C, trans_w, tau.data(), flags.data(),
                             in_ptr.data(), in_src.data(), in_label.data(), in_arc.data(), in_w.data(), ilabel.data(),
                             olabel.data(), acc.data(), map.data());
    else
      asg_num_build_kernel(meta.data(), targets, off, lens, C, trans_w, flags.data(), in_ptr.data(), in_src.data(),
                           in_label.data(), in_arc.data(), in_w.data(), ilabel.data(), olabel.data(), acc.data(),
                           map.data());
  });
  // launch_implicit_forward's pick for these numerators (in-degree <= 3: one CTA per utterance, tropical)
  const ImpLayout lf = make_imp_layout(N, A, false, false, C, false);
  emu::launch(B, kImpThreads, lf.total, [&] {
    implicit_forward_kernel<false, true>(meta.data(), flags.data(), in_ptr.data(), in_src.data(), in_label.data(),
                                         in_w.data(), emissions, sc.data(), out.data(), kstatus.data(), C, lf);
  });
  const TraceLayout lt = trace_layout(N, A, C);
  int32_t* arc_out = tokens ? arcs.data() : nullptr;
  emu::launch(B, kImpThreads, lt.total, [&] {
    implicit_trace_kernel(meta.data(), flags.data(), in_ptr.data(), in_src.data(), in_label.data(), in_w.data(),
                          in_arc.data(), emissions, sc.data(), kstatus.data(), paths, arc_out, scores, T, C, lt);
  });
  emu::launch(B, 256, 0, [&] {
    if (kind == 0)
      align_async_finalize_kernel<AsyncGraph::Ctc>(T, meta.data(), in_ptr.data(), kstatus.data(), valid.data(),
                                                   arc_out, paths, tokens, scores, status);
    else if (kind == 1)
      align_async_finalize_kernel<AsyncGraph::Ngram>(T, meta.data(), in_ptr.data(), kstatus.data(), valid.data(),
                                                     arc_out, paths, tokens, scores, status);
    else
      align_async_finalize_kernel<AsyncGraph::Asg>(T, meta.data(), in_ptr.data(), kstatus.data(), valid.data(),
                                                   arc_out, paths, tokens, scores, status);
  });
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

} // extern "C"
