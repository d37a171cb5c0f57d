/*
 * tests/emu/beam_emu.cpp -- TEST INFRASTRUCTURE for gtnb_beam_decode_async: the SOURCE of k_beam.cu's
 * beam_weights_kernel and beam_decode_kernel run on the CPU through tests/emu/simt_emu.h at launch_beam_decode's
 * geometry, with the shipped transcript hash or a degenerate one that makes every transcript collide (so the exact
 * compare through the back-pointers decides every re-created parent).
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_beam.cu"

#include <vector>

namespace {

/* every transcript hashes to 0 */
struct CollideHash {
  static uint64_t combine(uint64_t, int32_t) { return 0; }
};

template <class E, class H>
void run(int B, int T, int C, const void* emissions, const int32_t* input_lens, int kind, const float* wt,
         const float* wfirst, const int32_t* wbad, int blank, int K, int N, uint16_t* bp, int32_t* tokens,
         int32_t* lengths, float* scores, int32_t* status) {
  emu::launch(B, gtnb::kBeamThreads, gtnb::beam_smem_bytes(K, C), [&] {
    gtnb::beam_decode_kernel<E, H>(static_cast<const E*>(emissions), T, C, input_lens, kind, wt, wfirst, wbad, blank,
                                   K, N, bp, tokens, lengths, scores, status);
  });
}

template <class H>
void dispatch(int dtype, int B, int T, int C, const void* emissions, const int32_t* input_lens, int kind,
              const float* wt, const float* wfirst, const int32_t* wbad, int blank, int K, int N, uint16_t* bp,
              int32_t* tokens, int32_t* lengths, float* scores, int32_t* status) {
  if (dtype == GTNB_BF16)
    run<gtnb::bf16_t, H>(B, T, C, emissions, input_lens, kind, wt, wfirst, wbad, blank, K, N, bp, tokens, lengths,
                         scores, status);
  else if (dtype == GTNB_F16)
    run<gtnb::f16_t, H>(B, T, C, emissions, input_lens, kind, wt, wfirst, wbad, blank, K, N, bp, tokens, lengths,
                        scores, status);
  else
    run<float, H>(B, T, C, emissions, input_lens, kind, wt, wfirst, wbad, blank, K, N, bp, tokens, lengths, scores,
                  status);
}

} // namespace

extern "C" {

/*
 * One call: the weights kernel (kinds with transitions), then the search.  emissions [B][T][C] of dtype (16-bit
 * types as their bits), input_lens nullable, trans_w as the C ABI takes it (NULL for GTNB_DENSE_CTC).  collide: the
 * degenerate hash.  Returns 0, or 77 when the host refused the threads.
 */
int emu_beam(int B, int T, int C, const void* emissions, int dtype, const int32_t* input_lens, int kind,
             const float* trans_w, int blank, int K, int N, int collide, int32_t* tokens, int32_t* lengths,
             float* scores, int32_t* status) {
  std::vector<float> wt((size_t)C * C, 0.0f), sigma(C, 0.0f);
  std::vector<int32_t> wbad(C, 0);
  if (kind != GTNB_DENSE_CTC)
    emu::launch(C, gtnb::kBeamThreads, 0, [&] {
      gtnb::beam_weights_kernel(C, kind, trans_w, wt.data(), sigma.data(), wbad.data());
    });
  const float* wfirst = kind == GTNB_DENSE_ASG ? trans_w : sigma.data();
  std::vector<uint16_t> bp((size_t)B * (T > 0 ? T : 1) * K, 0xffffu);
  if (collide)
    dispatch<CollideHash>(dtype, B, T, C, emissions, input_lens, kind, wt.data(), wfirst, wbad.data(), blank, K, N,
                          bp.data(), tokens, lengths, scores, status);
  else
    dispatch<gtnb::BeamHash>(dtype, B, T, C, emissions, input_lens, kind, wt.data(), wfirst, wbad.data(), blank, K,
                             N, bp.data(), tokens, lengths, scores, status);
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

} // extern "C"
