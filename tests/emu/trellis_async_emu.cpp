/*
 * tests/emu/trellis_async_emu.cpp -- TEST INFRASTRUCTURE: runs the SOURCE of the kernels gtnb_ngram_ctc_loss_async
 * and gtnb_asg_loss_async add (gtn_b200/csrc/k_ctc.cu: the prepare kernel's n-gram and ASG instantiations,
 * trellis_async_gate_kernel, trellis_async_scatter_kernel; ctc_async_finalize_kernel, which they reuse) and the
 * numerator build kernels of k_ngram.cu they feed, on the CPU through tests/emu/simt_emu.h.  Only the launch
 * geometry is restated here; the descriptors and buffers come from the caller.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_ctc.cu"
#include "../../gtn_b200/csrc/k_ngram.cu"

#include <vector>

using gtnb::GraphMeta;

extern "C" {

/* asg: the ASG instantiation, else n-gram; m01: the bound-uniform descriptors of utterances 0 and 1; kstatus [2B] */
int emu_trellis_async_prepare(int asg, int B, int S, int T, int C, const GraphMeta* m01, const int32_t* input_lens,
                              const int32_t* targets, const int32_t* target_lens, GraphMeta* meta, int32_t* small,
                              float* deltas, int32_t* valid, int32_t* kstatus) {
  using namespace gtnb;
  for (int bx = 0; bx < (B + 7) / 8; bx++)
    emu::launch(1, 256, 0, [&] {
      blockIdx.x = bx;
      if (asg)
        ctc_async_prepare_kernel<AsyncGraph::Asg>(B, S, T, C, m01[0], m01[1], input_lens, targets, target_lens, meta,
                                                  small, deltas, valid, kstatus);
      else
        ctc_async_prepare_kernel<AsyncGraph::Ngram>(B, S, T, C, m01[0], m01[1], input_lens, targets, target_lens,
                                                    meta, small, deltas, valid, kstatus);
    });
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

/*
 * ngram_num_build_kernel (asg = 0: after ngram_sigma_kernel on W) or asg_num_build_kernel (W = ASG's [C + C*C]) for B
 * utterances described by meta, the targets at targets + tgt_off[b], into the caller's tables.
 */
int emu_trellis_num_build(int asg, int B, int C, int blank, const GraphMeta* meta, const int32_t* targets,
                          const int32_t* tgt_off, const int32_t* tgt_len, const float* W, uint8_t* flags,
                          int32_t* in_ptr, int32_t* in_src, int32_t* in_label, int32_t* in_arc, float* in_w,
                          int32_t* ilabel, int32_t* olabel, int32_t* acc_nodes, int32_t* map) {
  using namespace gtnb;
  std::vector<float> sigma(C > 0 ? C : 1);
  if (!asg) emu::launch((C * 32 + 255) / 256, 256, 0, [&] { ngram_sigma_kernel(C, W, sigma.data()); });
  emu::launch(B, 256, 0, [&] {
    if (asg)
      asg_num_build_kernel(meta, targets, tgt_off, tgt_len, C, W, flags, in_ptr, in_src, in_label, in_arc, in_w,
                           ilabel, olabel, acc_nodes, map);
    else
      ngram_num_build_kernel(meta, targets, tgt_off, tgt_len, blank, C, W, sigma.data(), flags, in_ptr, in_src,
                             in_label, in_arc, in_w, ilabel, olabel, acc_nodes, map);
  });
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

int emu_trellis_async_gate(int B, const int32_t* T_fwd, const int32_t* valid, int32_t* kstatus, int32_t* T_bwd,
                           float* den) {
  using namespace gtnb;
  emu::launch((B + 255) / 256, 256, 0, [&] { trellis_async_gate_kernel(B, T_fwd, valid, kstatus, T_bwd, den); });
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

int emu_trellis_async_scatter(int B, const GraphMeta* meta, const int32_t* kstatus, const int32_t* map,
                              const float* src, float* dst) {
  using namespace gtnb;
  emu::launch(B, 256, 0, [&] { trellis_async_scatter_kernel(meta, kstatus, map, src, dst); });
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

/* ctc_async_finalize_kernel as the trellis calls launch it: zp = 1, z = den, s = num */
int emu_trellis_async_finalize(int B, const float* den, const float* num, const int32_t* kstatus,
                               const int32_t* valid, float* losses, int32_t* status, float* grad,
                               long long row_words) {
  using namespace gtnb;
  emu::launch(B, 256, 0, [&] {
    ctc_async_finalize_kernel(1, den, num, kstatus, valid, losses, status, reinterpret_cast<uint32_t*>(grad),
                              row_words);
  });
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

} // extern "C"
