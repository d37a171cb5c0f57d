/*
 * tests/emu/bidir_emu.cpp -- TEST INFRASTRUCTURE: runs the SOURCE of gtn_b200/csrc/k_bidir.cu (the
 * criterion's bidirectional meet-in-the-middle kernel: two-CTA clusters, TMA-staged emission / score
 * blocks, helper warps) on the CPU through tests/emu/simt_emu.h, fed by k_ctc.cu's ctc_build_kernel
 * exactly as gtnb_ctc_loss feeds it.  The kernel and its geometry are bidir_plan's, as for launch_bidir_ctc; only
 * the device tables are restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_ctc.cu"
#include "../../gtn_b200/csrc/k_bidir.cu"

#include <vector>

using gtnb::GraphMeta;

extern "C" {

/*
 * targets concatenated, target_lens[B]; emissions [B][T][C]; input_lens[B] or NULL.
 * out_scores[B] = forwardScore(intersect(ctc_b, e_b)); znorm[B] = forwardScore(e_b);
 * grad [B][T][C] (NULL: loss only) = d(znorm - out) / d e; status[B].
 * bidir_mode: as gtnb_ctx_set_flag's -- 0 the one-node-per-thread kernel, otherwise launch_bidir_ctc's choice.
 */
int emu_bidir_ctc(
    int B, int T, int C, const float* emissions, const int32_t* input_lens, const int32_t* targets,
    const int32_t* target_lens, int blank, int bidir_mode, float* out_scores, float* znorm, float* grad, int32_t* status) {
  using namespace gtnb;
  std::vector<GraphMeta> meta(B);
  std::vector<int32_t> tgt_off(B);
  long long nodes = 0, arcs = 0, scores_len = 0, acc = 0, toff = 0;
  int maxN = 0;
  for (int b = 0; b < B; b++) maxN = std::max(maxN, 2 * target_lens[b] + 1);
  // saved-score rows of the fixed pitch where the graphs fit it, as gtnb_compose_linear allocates them
  const BidirPlan p = bidir_plan<float>(C, maxN, maxN <= bidir::kFixedPitch, bidir_mode != 0);
  for (int b = 0; b < B; b++) {
    const int L = 2 * target_lens[b] + 1;
    GraphMeta& m = meta[b];
    std::memset(&m, 0, sizeof(m));
    m.sg_node_base = nodes;
    m.sg_arc_base = arcs;
    m.acc_base = acc;
    m.emis_off = (long long)b * T * C;
    m.node_base = scores_len;
    m.T = input_lens ? input_lens[b] : T;
    m.sg_N = L;
    tgt_off[b] = (int32_t)toff;
    toff += target_lens[b];
    nodes += L + 1;
    arcs += 3 * L;
    acc += 2;
    scores_len += (long long)(T + 1) * (p.fx ? bidir::kFixedPitch : ((L + 3) & ~3));
  }
  std::vector<uint8_t> flags(nodes, 0);
  std::vector<int32_t> in_ptr(nodes, 0), in_src(arcs, 0), in_label(arcs, 0), in_arc(arcs, 0), il(arcs, 0),
      ol(arcs, 0), acc_nodes(acc, 0);
  std::vector<float> in_w(arcs, 0.0f);
  emu::launch(B, 256, 0, [&] {
    ctc_build_kernel(meta.data(), targets, tgt_off.data(), target_lens, blank, C, flags.data(), in_ptr.data(),
                     in_src.data(), in_label.data(), in_arc.data(), in_w.data(), il.data(), ol.data(),
                     acc_nodes.data());
  });
  for (int b = 0; b < B; b++) meta[b].sg_A = in_ptr[meta[b].sg_node_base + meta[b].sg_N];
  // the bulk copies need 16-byte aligned sources: the vectors' data() is (malloc), T * C * 4 % 16 == 0 is
  // the caller's business (C % 4 == 0)
  std::vector<float> saved((size_t)scores_len + 16, 0.0f);
  std::vector<float> zparts(2 * (size_t)B * bidir::kHelpers, 0.0f);
  const int nblk_cap = std::max(1, (T + bidir::kBlk - 1) / bidir::kBlk);
  std::vector<float> boff((size_t)B * 2 * nblk_cap * 4 + 16, 0.0f);
  for (int b = 0; b < B; b++) status[b] = 0;
  bidir::Params P;
  P.meta = meta.data();
  P.sg_flags = flags.data();
  P.sg_in_ptr = in_ptr.data();
  P.sg_in_src = in_src.data();
  P.sg_in_label = in_label.data();
  P.sg_in_w = in_w.data();
  P.emissions = emissions;
  P.saved = saved.data();
  P.boff = boff.data();
  P.nblk_cap = nblk_cap;
  P.out_scores = out_scores;
  P.zparts = zparts.data();
  P.status = status;
  P.grad = grad;
  P.grad_stride = (long long)T * C;
  P.C = C;
  P.ctc_blank = blank;
  P.targets = targets;
  for (int b = 0; b < B; b++) meta[b].tgt_off = tgt_off[b];
  P.nwn = p.nwn;
  P.lay = p.lay;
  emu::launch_clusters(2 * B, 2, p.block, P.lay.total, [&] { p.kernel(P); });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  for (int b = 0; b < B; b++) {
    znorm[b] = 0.0f;
    for (int k = 0; k < 2 * bidir::kHelpers; k++) znorm[b] += zparts[2 * bidir::kHelpers * b + k];
  }
  return 0;
}

} // extern "C"
