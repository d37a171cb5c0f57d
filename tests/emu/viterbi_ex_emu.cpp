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
  int G = 1;
  while (G < 32 && C * (G * 2) <= kDenseThreads) G *= 2;
  const size_t smem = sizeof(float) * ((size_t)C * (C + 32 / G) + 2 * (size_t)C);
  if (C < 1 || C > 256 || smem > 227 * 1024) return 1;
  std::vector<uint8_t> bp((size_t)B * std::max(T, 1) * dense_bp_pitch(C), 0);
  const float empty = -__builtin_inff();
#define RUN(G_, K_)                                                                                          \
  emu::launch(B, kDenseThreads, smem, [&] {                                                                  \
    viterbi_dense_kernel<G_, K_>(T, C, lens, emissions, (long long)T * C, trans, bp.data(), paths, scores,  \
                                 empty);                                                                     \
  })
#define RUN_KIND(G_) \
  if (kind == 1)     \
    RUN(G_, true);   \
  else               \
    RUN(G_, false)
  switch (G) {
    case 1: RUN_KIND(1); break;
    case 2: RUN_KIND(2); break;
    case 4: RUN_KIND(4); break;
    case 8: RUN_KIND(8); break;
    case 16: RUN_KIND(16); break;
    default: RUN_KIND(32); break;
  }
#undef RUN_KIND
#undef RUN
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

} // extern "C"
