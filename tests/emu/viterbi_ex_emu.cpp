/*
 * tests/emu/viterbi_ex_emu.cpp -- TEST INFRASTRUCTURE: the SOURCE of gtn_b200/csrc/k_dense.cu as
 * gtnb_viterbi_dense_ex launches it (both graph kinds, any C, T_b = 0 scores -inf) on the CPU through
 * tests/emu/simt_emu.h.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_dense.cu"

#include <vector>

extern "C" {

/* emissions [B][T][C], lens (nullable), kind 0 (ASG: trans [C] start arcs then [C][C]) or 1 (BIGRAM: trans [C][C],
 * every state starts), w(j -> i) at [i*C + j] of the C x C part; paths [B][T], scores [B].  Returns 0, or 1 for a C
 * the tile does not allow. */
int emu_viterbi_dense_ex(int B, int T, int C, const float* emissions, const int32_t* lens, int kind,
                         const float* trans, int32_t* paths, float* scores) {
  using namespace gtnb;
  if (!viterbi_dense_supported(C)) return 1;
  std::vector<uint8_t> bp((size_t)B * std::max(T, 1) * dense_bp_pitch(C), 0);
  const auto kernel = viterbi_dense_kernel_for<float>(dense_lanes(C), kind == 1);
  emu::launch(B, kDenseThreads, dense_smem_bytes(C), [&] {
    kernel(T, C, lens, emissions, (long long)T * C, trans, bp.data(), paths, scores, -__builtin_inff());
  });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

} // extern "C"
