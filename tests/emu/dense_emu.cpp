/*
 * tests/emu/dense_emu.cpp -- TEST INFRASTRUCTURE: the SOURCE of gtn_b200/csrc/k_dense.cu (factored
 * dense-trellis Viterbi, BASELINE config 4) on the CPU through tests/emu/simt_emu.h.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_dense.cu"

#include <vector>

extern "C" {

/* emissions [B][T][C], lens (nullable), trans: [C] start arcs then [C][C] (w(j -> i) at C + i*C + j);
 * paths [B][T], scores [B].  Returns 0, or 1 for an unsupported C. */
int emu_viterbi_dense(int B, int T, int C, const float* emissions, const int32_t* lens, const float* trans,
                      int32_t* paths, float* scores) {
  using namespace gtnb;
  if (!viterbi_dense_supported(C) || (C % 4) != 0) return 1;
  std::vector<uint8_t> bp((size_t)B * std::max(T, 1) * dense_bp_pitch(C), 0);
  const auto kernel = viterbi_dense_kernel_for<float>(dense_lanes(C), false);
  emu::launch(B, kDenseThreads, dense_smem_bytes(C), [&] {
    kernel(T, C, lens, emissions, (long long)T * C, trans, bp.data(), paths, scores, 0.0f);
  });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

} // extern "C"
