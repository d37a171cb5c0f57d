/*
 * tests/emu/beam_emu.cpp -- TEST INFRASTRUCTURE for gtnb_beam_decode_async, gtnb_beam_decode_lm_async and
 * gtnb_beam_decode_lexicon_async: the SOURCE of k_beam.cu's beam_weights_kernel and beam_decode_kernel under each
 * policy run on the CPU through tests/emu/simt_emu.h at launch_beam_decode's geometry, with the shipped transcript
 * hash or a degenerate one that makes every transcript collide (so the exact compare through the back-pointers
 * decides every re-created parent).  The LM comes as its resolved table, the lexicon as the device arrays of
 * gtnb_lexicon_create.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_beam.cu"

#include <vector>

namespace {

/* every transcript hashes to 0 */
struct CollideHash {
  static uint64_t combine(uint64_t, int32_t) { return 0; }
};

template <class E, class H, class F>
void run(int B, int T, int C, const void* emissions, const int32_t* input_lens, int kind, const float* wt,
         const float* wfirst, const int32_t* wbad, int blank, int K, int N, uint16_t* bp, int32_t* tokens,
         int32_t* lengths, float* scores, int32_t* status, const F& f) {
  emu::launch(B, gtnb::kBeamThreads, gtnb::beam_smem_bytes<F>(K, C), [&] {
    gtnb::beam_decode_kernel<E, H, F>(static_cast<const E*>(emissions), T, C, input_lens, kind, wt, wfirst, wbad,
                                      blank, K, N, bp, tokens, lengths, scores, status, f);
  });
}

/* One call: the weights kernel (kinds with transitions), then the search under policy f, of dtype and hash collide */
template <class F>
int search(int B, int T, int C, const void* emissions, int dtype, const int32_t* input_lens, int kind,
           const float* trans_w, int blank, int K, int N, int collide, int32_t* tokens, int32_t* lengths,
           float* scores, int32_t* status, const F& f) {
  std::vector<float> wt((size_t)C * C, 0.0f), sigma(C, 0.0f);
  std::vector<int32_t> wbad(C, 0);
  if (kind != GTNB_DENSE_CTC)
    emu::launch(C, gtnb::kBeamThreads, 0, [&] {
      gtnb::beam_weights_kernel(C, kind, trans_w, wt.data(), sigma.data(), wbad.data());
    });
  const float* wfirst = kind == GTNB_DENSE_ASG ? trans_w : sigma.data();
  std::vector<uint16_t> bp((size_t)B * (T > 0 ? T : 1) * K, 0xffffu);
  const auto go = [&](auto hash, auto elem) {
    run<decltype(elem), decltype(hash)>(B, T, C, emissions, input_lens, kind, wt.data(), wfirst, wbad.data(), blank,
                                        K, N, bp.data(), tokens, lengths, scores, status, f);
  };
  const auto by_dtype = [&](auto hash) {
    if (dtype == GTNB_BF16)
      go(hash, gtnb::bf16_t());
    else if (dtype == GTNB_F16)
      go(hash, gtnb::f16_t());
    else
      go(hash, 0.0f);
  };
  if (collide)
    by_dtype(CollideHash());
  else
    by_dtype(gtnb::BeamHash());
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

} // namespace

extern "C" {

/*
 * emissions [B][T][C] of dtype (16-bit types as their bits), input_lens nullable, trans_w as the C ABI takes it (NULL
 * for GTNB_DENSE_CTC).  collide: the degenerate hash.  Each returns 0, or 77 when the host refused the threads.
 */
int emu_beam(int B, int T, int C, const void* emissions, int dtype, const int32_t* input_lens, int kind,
             const float* trans_w, int blank, int K, int N, int collide, int32_t* tokens, int32_t* lengths,
             float* scores, int32_t* status) {
  return search(B, T, C, emissions, dtype, input_lens, kind, trans_w, blank, K, N, collide, tokens, lengths, scores,
                status, gtnb::BeamNoLm());
}

/* the fused search: lmw / lmd the resolved table [S][C + 1] (lmw NULL: no LM), start its start node; P = token_beam */
int emu_beam_lm(int B, int T, int C, const void* emissions, int dtype, const int32_t* input_lens, int kind,
                const float* trans_w, int blank, int K, int N, const float* lmw, const int32_t* lmd, int start,
                float lm_weight, float token_bonus, int P, int collide, int32_t* tokens, int32_t* lengths,
                float* scores, float* am, float* lm, int32_t* status) {
  return search(B, T, C, emissions, dtype, input_lens, kind, trans_w, blank, K, N, collide, tokens, lengths, scores,
                status, gtnb::BeamLm{P, lmw, lmd, start, lm_weight, token_bonus, am, lm});
}

/*
 * The lexicon search.  The lexicon: cls [C], mask [nodes][ceil(C / 32)], first / word / smear [nodes]; the word LM
 * (hash NULL: none): hash [2^hbits][2] (key, value), hmul, bow / bod / endw [S], start.
 */
int emu_beam_lexicon(int B, int T, int C, const void* emissions, int dtype, const int32_t* input_lens, int kind,
                     const float* trans_w, int blank, int K, int N, const int32_t* cls, const uint32_t* mask,
                     const int32_t* first, const int32_t* word, const float* smear, const unsigned long long* hash,
                     unsigned long long hmul, int hbits, const float* bow, const int32_t* bod, const float* endw,
                     int start, float lm_weight, float word_bonus, int P, int collide, int32_t* tokens,
                     int32_t* lengths, float* scores, float* am, float* lm, int32_t* words, int32_t* counts,
                     int32_t* status) {
  const gtnb::BeamLex f{{P, nullptr, nullptr, start, lm_weight, word_bonus, am, lm},
                        cls,
                        (C + 31) / 32,
                        mask,
                        first,
                        word,
                        smear,
                        hash,
                        hmul,
                        hbits,
                        bow,
                        bod,
                        endw,
                        words,
                        counts};
  return search(B, T, C, emissions, dtype, input_lens, kind, trans_w, blank, K, N, collide, tokens, lengths, scores,
                status, f);
}

} // extern "C"
