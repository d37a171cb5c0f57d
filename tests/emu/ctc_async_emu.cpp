/*
 * tests/emu/ctc_async_emu.cpp -- TEST INFRASTRUCTURE: runs the SOURCE of gtn_b200/csrc/k_ctc.cu's
 * gtnb_ctc_loss_async kernels (ctc_async_prepare_kernel, ctc_async_finalize_kernel) on the CPU through
 * tests/emu/simt_emu.h, alone and around k_bidir.cu's kernel on the padded, bound-uniform layout the asynchronous
 * call gives it.  Only the launch geometry and the buffers are restated here; the descriptors of utterances 0 and 1
 * (m0, m1) come from the caller.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_ctc.cu"
#include "../../gtn_b200/csrc/k_bidir.cu"

#include <vector>

using gtnb::GraphMeta;

namespace {
void prepare(int B, int S, int T, int C, const GraphMeta* m01, const int32_t* input_lens, const int32_t* targets,
             const int32_t* target_lens, GraphMeta* meta, int32_t* small, float* deltas, int32_t* valid,
             int32_t* kstatus) {
  using namespace gtnb;
  for (int bx = 0; bx < (B + 7) / 8; bx++)
    emu::launch(1, 256, 0, [&] {
      blockIdx.x = bx;
      ctc_async_prepare_kernel(B, S, T, C, m01[0], m01[1], input_lens, targets, target_lens, meta, small, deltas,
                               valid, kstatus);
    });
}

void finalize(int B, int zp, const float* z, const float* s, const int32_t* kstatus, const int32_t* valid,
              float* losses, int32_t* status, void* grad, long long row_words) {
  using namespace gtnb;
  emu::launch(B, 256, 0, [&] {
    ctc_async_finalize_kernel(zp, z, s, kstatus, valid, losses, status, static_cast<uint32_t*>(grad), row_words);
  });
}
} // namespace

extern "C" {

int emu_ctc_async_prepare(int B, int S, int T, int C, const GraphMeta* m01, const int32_t* input_lens,
                          const int32_t* targets, const int32_t* target_lens, GraphMeta* meta, int32_t* small,
                          float* deltas, int32_t* valid, int32_t* kstatus) {
  prepare(B, S, T, C, m01, input_lens, targets, target_lens, meta, small, deltas, valid, kstatus);
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

int emu_ctc_async_finalize(int B, int zp, const float* z, const float* s, const int32_t* kstatus,
                           const int32_t* valid, float* losses, int32_t* status, float* grad, long long row_words) {
  finalize(B, zp, z, s, kstatus, valid, losses, status, grad, row_words);
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

/*
 * The one-launch route of gtnb_ctc_loss_async: prepare, ctc_build_kernel unless the PAIR kernels run, the
 * bidirectional kernel and finalize, on the slabs of m01's layout (score rows (T + 1) * pitch + 4 floats, graph slabs
 * sgn / sga entries per utterance).  targets [B][S]; losses, status [B]; grad [B][T][C] (NULL: loss only).
 */
int emu_ctc_async_bidir(int B, int T, int C, int S, const GraphMeta* m01, long long sgn, long long sga,
                        const float* emissions, const int32_t* input_lens, const int32_t* targets,
                        const int32_t* target_lens, int blank, int bidir_mode, float* losses, int32_t* status,
                        float* grad) {
  using namespace gtnb;
  const int maxN = 2 * S + 1;
  const long long step = B > 1 ? m01[1].node_base - m01[0].node_base : m01[0].cap_N;
  std::vector<GraphMeta> meta(B);
  std::vector<int32_t> small(3 * (size_t)B), valid(B), kstatus(B);
  std::vector<float> deltas(B);
  prepare(B, S, T, C, m01, input_lens, targets, target_lens, meta.data(), small.data(), deltas.data(), valid.data(),
          kstatus.data());
  std::vector<uint8_t> flags((size_t)B * sgn, 0);
  std::vector<int32_t> in_ptr((size_t)B * sgn, 0), in_src((size_t)B * sga, 0), in_label((size_t)B * sga, 0),
      in_arc((size_t)B * sga, 0), il((size_t)B * sga, 0), ol((size_t)B * sga, 0), acc_nodes(4 * (size_t)B, 0);
  std::vector<float> in_w((size_t)B * sga, 0.0f);
  // launch_bidir_ctc's rules: fixed row pitch for C = 64, 128 on the fixed-pitch layout; PAIR kernels below 224 nodes
  const bool fx = (C == 64 || C == 128) && maxN <= bidir::kFixedPitch;
  const bool pair = fx && bidir_mode != 0 && maxN <= 2 * 32 * bidir::kMaxPairWarps - 1;
  if (!pair)
    emu::launch(B, 256, 0, [&] {
      ctc_build_kernel(meta.data(), targets, small.data(), small.data() + B, blank, C, flags.data(), in_ptr.data(),
                       in_src.data(), in_label.data(), in_arc.data(), in_w.data(), il.data(), ol.data(),
                       acc_nodes.data());
    });
  std::vector<float> saved((size_t)B * step + 16, 0.0f);
  const int zp = 2 * bidir::kHelpers;
  std::vector<float> zs((size_t)zp * B + B, 0.0f);
  const int nblk_cap = std::max(1, (T + bidir::kBlk - 1) / bidir::kBlk);
  std::vector<float> boff((size_t)B * 2 * nblk_cap * 4 + 16, 0.0f);
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
  P.out_scores = zs.data() + (size_t)zp * B;
  P.zparts = zs.data();
  P.status = kstatus.data();
  P.grad = grad;
  P.grad_stride = (long long)T * C;
  P.C = C;
  P.ctc_blank = blank;
  P.targets = targets;
  P.nwn = pair ? std::max(1, ((maxN + 1) / 2 + 31) / 32) : std::max(1, (maxN + 31) / 32);
  P.lay = bidir::make_layout(C, fx ? bidir::kFixedPitch : ((maxN + 3) & ~3));
  const unsigned block = 32 * (P.nwn + 1 + bidir::kHelpers);
  emu::launch_clusters(2 * B, 2, block, P.lay.total, [&] {
    if (pair)
      C == 64 ? bidir::bidir_ctc_kernel<1, true, 1>(P) : bidir::bidir_ctc_kernel<2, true, 1>(P);
    else if (fx && C == 64)
      bidir::bidir_ctc_kernel<1, true, 0>(P);
    else if (fx)
      bidir::bidir_ctc_kernel<2, true, 0>(P);
    else if (C <= 64)
      bidir::bidir_ctc_kernel<1, false, 0>(P);
    else
      bidir::bidir_ctc_kernel<2, false, 0>(P);
  });
  finalize(B, zp, zs.data(), zs.data() + (size_t)zp * B, kstatus.data(), valid.data(), losses, status, grad,
           (long long)T * C);
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

} // extern "C"
