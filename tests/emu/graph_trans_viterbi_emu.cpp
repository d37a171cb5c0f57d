/*
 * tests/emu/graph_trans_viterbi_emu.cpp -- TEST INFRASTRUCTURE for gtnb_graph_transitions_viterbi: the SOURCE of
 * k_ngram.cu's ngram_tau_kernel and product_arc_map_kernel, run on the CPU through tests/emu/simt_emu.h.  Only the
 * launch geometry is restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_implicit.cu"
#include "../../gtn_b200/csrc/k_ngram.cu"

extern "C" {

/* ngram_tau_kernel over W [C][C], as launch_ngram_tau launches it */
int emu_ngram_tau(int C, const float* W, float* tau) {
  emu::launch((C * 32 + 255) / 256, 256, 0, [&] { gtnb::ngram_tau_kernel(C, W, tau); });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

/* product_arc_map_kernel over arcs [B][T_out], as launch_product_arc_map launches it */
int emu_product_arc_map(int B, int T_out, const long long* off, const int32_t* arc_of, int32_t* arcs) {
  const long long n = (long long)B * T_out;
  if (n > 0)
    emu::launch((int)((n + 255) / 256), 256, 0,
                [&] { gtnb::product_arc_map_kernel(n, T_out, off, arc_of, arcs); });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

} // extern "C"
