/*
 * tests/emu/bidir_half_emu.cpp -- TEST INFRASTRUCTURE: tests/emu/bidir_emu.cpp's run of the SOURCE of
 * gtn_b200/csrc/k_bidir.cu on the CPU (tests/emu/simt_emu.h, fed by k_ctc.cu's ctc_build_kernel exactly as
 * gtnb_ctc_loss feeds it), for any element type of the emissions and the gradient: float, bf16_t or fp16 --
 * gtnb_ctc_loss_ex's native route.  Also exports gtnb_ptx.h's emulated 16-bit conversions.  Only the launch
 * geometry and the device tables are restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_ctc.cu"
#include "../../gtn_b200/csrc/k_bidir.cu"

#include <vector>

using gtnb::GraphMeta;

namespace {

/* bidir_emu.cpp's emu_bidir_ctc with emissions and gradient of element type E (float, bf16_t, f16_t) */
template <class E>
int run_bidir_ctc(
    int B, int T, int C, const E* emissions, const int32_t* input_lens, const int32_t* targets,
    const int32_t* target_lens, int blank, int bidir_mode, float* out_scores, float* znorm, E* grad, int32_t* status) {
  using namespace gtnb;
  std::vector<GraphMeta> meta(B);
  std::vector<int32_t> tgt_off(B);
  long long nodes = 0, arcs = 0, scores_len = 0, acc = 0, toff = 0;
  int maxN = 0;
  const bool fx = C == 64 || C == 128; // launch_bidir_ctc's rule: fixed row pitch for the FX kernels
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
    scores_len += (long long)(T + 1) * (fx ? bidir::kFixedPitch : ((L + 3) & ~3));
    maxN = std::max(maxN, L);
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
  // the bulk copies need 16-byte aligned sources: the vectors' data() is (malloc), T * C * sizeof(E) % 16 == 0 is
  // the caller's business (C % 4 == 0; 16-bit elements: C % 8 == 0)
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
  // launch_bidir_ctc's rule: the PAIR kernels (two nodes per thread) for gtnb_ctc_loss's own graphs
  const bool pair = fx && bidir_mode != 0 && maxN <= 2 * 32 * bidir::kMaxPairWarps - 1;
  P.ctc_blank = blank;
  P.targets = targets;
  for (int b = 0; b < B; b++) meta[b].tgt_off = tgt_off[b];
  P.nwn = pair ? std::max(1, ((maxN + 1) / 2 + 31) / 32) : std::max(1, (maxN + 31) / 32);
  P.lay = bidir::make_layout(C, fx ? bidir::kFixedPitch : ((maxN + 3) & ~3), (int)sizeof(E));
  const unsigned block = 32 * (P.nwn + 1 + bidir::kHelpers);
  emu::launch_clusters(2 * B, 2, block, P.lay.total, [&] {
    if (pair)
      C == 64 ? bidir::bidir_ctc_kernel<1, true, 1, E>(P) : bidir::bidir_ctc_kernel<2, true, 1, E>(P);
    else if (fx && C == 64)
      bidir::bidir_ctc_kernel<1, true, 0, E>(P);
    else if (fx)
      bidir::bidir_ctc_kernel<2, true, 0, E>(P);
    else if (C <= 64)
      bidir::bidir_ctc_kernel<1, false, 0, E>(P);
    else
      bidir::bidir_ctc_kernel<2, false, 0, E>(P);
  });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  for (int b = 0; b < B; b++) {
    znorm[b] = 0.0f;
    for (int k = 0; k < 2 * bidir::kHelpers; k++) znorm[b] += zparts[2 * bidir::kHelpers * b + k];
  }
  return 0;
}

} // namespace

extern "C" {

/*
 * targets concatenated, target_lens[B]; emissions and grad (NULL: loss only) [B][T][C] of element type dtype (GTNB_F32,
 * GTNB_BF16, GTNB_F16, as gtnb_ctc_loss_ex); input_lens[B] or NULL.  out_scores[B] = forwardScore(intersect(ctc_b,
 * e_b)); znorm[B] = forwardScore(e_b); grad = d(znorm - out) / d e; status[B].  bidir_mode: as gtnb_ctx_set_flag's --
 * 0 the one-node-per-thread kernel, otherwise launch_bidir_ctc's choice.
 */
int emu_bidir_ctc_ex(
    int B, int T, int C, const void* emissions, int dtype, const int32_t* input_lens, const int32_t* targets,
    const int32_t* target_lens, int blank, int bidir_mode, float* out_scores, float* znorm, void* grad, int32_t* status) {
  using gtnb::bf16_t;
  using gtnb::f16_t;
  if (dtype == GTNB_BF16)
    return run_bidir_ctc<bf16_t>(B, T, C, static_cast<const bf16_t*>(emissions), input_lens, targets, target_lens, blank,
                                 bidir_mode, out_scores, znorm, static_cast<bf16_t*>(grad), status);
  if (dtype == GTNB_F16)
    return run_bidir_ctc<f16_t>(B, T, C, static_cast<const f16_t*>(emissions), input_lens, targets, target_lens, blank,
                                bidir_mode, out_scores, znorm, static_cast<f16_t*>(grad), status);
  return run_bidir_ctc<float>(B, T, C, static_cast<const float*>(emissions), input_lens, targets, target_lens, blank,
                              bidir_mode, out_scores, znorm, static_cast<float*>(grad), status);
}

/* gtnb_ptx.h's emulated conversions over n elements: float32 -> 16-bit bits (round to nearest even) and back */
void emu_f32_to_16(const float* src, uint16_t* dst, int dtype, long long n) {
  for (long long i = 0; i < n; i++)
    dst[i] = (uint16_t)(dtype == GTNB_BF16 ? gtnb::f32_bf16_bits(src[i]) : gtnb::f32_f16_bits(src[i]));
}
void emu_16_to_f32(const uint16_t* src, float* dst, int dtype, long long n) {
  for (long long i = 0; i < n; i++) dst[i] = dtype == GTNB_BF16 ? gtnb::bf16_bits_f32(src[i]) : gtnb::f16_bits_f32(src[i]);
}
/* the emulated packed store stg_elem4 of four floats */
void emu_stg_elem4(const float* src, uint16_t* dst, int dtype) {
  const float4 v = make_float4(src[0], src[1], src[2], src[3]);
  if (dtype == GTNB_BF16)
    gtnb::stg_elem4(reinterpret_cast<gtnb::bf16_t*>(dst), v);
  else
    gtnb::stg_elem4(reinterpret_cast<gtnb::f16_t*>(dst), v);
}

} // extern "C"
