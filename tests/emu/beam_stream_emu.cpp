/*
 * tests/emu/beam_stream_emu.cpp -- TEST INFRASTRUCTURE for gtnb_beam_decode_chunk_async: the SOURCE of k_beam.cu's
 * beam_weights_kernel and beam_chunk_kernel under the BeamLm and BeamLex policies run on the CPU through
 * tests/emu/simt_emu.h at launch_beam_chunk's geometry, with the shipped transcript hash or one under which every
 * transcript collides.  The caller keeps the decoder's state between calls: the rows' state blocks [B][words] (zero:
 * every row fresh) and the back-pointers [B][T_max][K], as gtnb_beam_state_create allocates them.  The weights kernel
 * runs at every call (the state's copy is made once; its values are the same).
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_beam.cu"

#include <vector>

namespace {

/* every transcript hashes to 0 */
struct CollideHash {
  static uint64_t combine(uint64_t, int32_t) { return 0; }
};

template <class F>
int chunk(int B, int T, int C, const void* emissions, int dtype, int kind, const float* trans_w, int blank, int K,
          int N, int collide, uint16_t* bp, int32_t* tokens, int32_t* lengths, float* scores, int32_t* status,
          const F& f, const gtnb::BeamChunk& r) {
  std::vector<float> wt((size_t)C * C, 0.0f), sigma(C, 0.0f);
  std::vector<int32_t> wbad(C, 0);
  if (kind != GTNB_DENSE_CTC)
    emu::launch(C, gtnb::kBeamThreads, 0, [&] {
      gtnb::beam_weights_kernel(C, kind, trans_w, wt.data(), sigma.data(), wbad.data());
    });
  const float* wfirst = kind == GTNB_DENSE_ASG ? trans_w : sigma.data();
  const auto go = [&](auto hash, auto elem) {
    using E = decltype(elem);
    emu::launch(B, gtnb::kBeamThreads, gtnb::beam_smem_bytes<F>(K, C), [&] {
      gtnb::beam_chunk_kernel<E, decltype(hash), F>(static_cast<const E*>(emissions), T, C, kind, wt.data(), wfirst,
                                                    wbad.data(), blank, K, N, bp, tokens, lengths, scores, status, f,
                                                    r);
    });
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

/* 32-bit words of a row's state block (k_beam.cu's beam_state_words) */
long long emu_beam_state_words(int lexicon, int K, int C) {
  return lexicon ? gtnb::beam_state_words<gtnb::BeamLex>(K, C) : gtnb::beam_state_words<gtnb::BeamLm>(K, C);
}

/*
 * One chunk under BeamLm: emissions [B][Tc][C] of dtype (16-bit types as their bits), lens / control nullable; lmw /
 * lmd the LM's resolved table [S][C + 1] (lmw NULL: no LM), start its start node; P = token_beam.  The final outputs
 * are [B][N][T] / [B][N] with T = T_max, best [B][T] / [B] / [B] (all NULL: no trace).  Returns 0, or 77 when the
 * host refused the threads.
 */
int emu_beam_chunk_lm(int B, int T, int C, int Tc, const void* emissions, int dtype, const int32_t* lens,
                      const int32_t* control, int kind, const float* trans_w, int blank, int K, int N,
                      const float* lmw, const int32_t* lmd, int start, float lm_weight, float token_bonus, int P,
                      int collide, uint32_t* state, uint16_t* bp, int32_t* tokens, int32_t* lengths, float* scores,
                      float* am, float* lm, int32_t* status, int32_t* best_tokens, int32_t* best_lengths,
                      float* best_scores) {
  const gtnb::BeamChunk r{Tc,   state,   emu_beam_state_words(0, K, C), lens, control, best_tokens, best_lengths,
                          best_scores};
  return chunk(B, T, C, emissions, dtype, kind, trans_w, blank, K, N, collide, bp, tokens, lengths, scores, status,
               gtnb::BeamLm{P, lmw, lmd, start, lm_weight, token_bonus, am, lm}, r);
}

/* One chunk under BeamLex: the lexicon and word LM as tests/emu/beam_emu.cpp's emu_beam_lexicon takes them */
int emu_beam_chunk_lexicon(int B, int T, int C, int Tc, const void* emissions, int dtype, const int32_t* lens,
                           const int32_t* control, int kind, const float* trans_w, int blank, int K, int N,
                           const int32_t* cls, const uint32_t* mask, const int32_t* first, const int32_t* word,
                           const float* smear, const unsigned long long* hash, unsigned long long hmul, int hbits,
                           const float* bow, const int32_t* bod, const float* endw, int start, float lm_weight,
                           float word_bonus, int P, int collide, uint32_t* state, uint16_t* bp, int32_t* tokens,
                           int32_t* lengths, float* scores, float* am, float* lm, int32_t* words, int32_t* counts,
                           int32_t* status, int32_t* best_tokens, int32_t* best_lengths, float* best_scores) {
  const gtnb::BeamChunk r{Tc,   state,   emu_beam_state_words(1, K, C), lens, control, best_tokens, best_lengths,
                          best_scores};
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
  return chunk(B, T, C, emissions, dtype, kind, trans_w, blank, K, N, collide, bp, tokens, lengths, scores, status, f,
               r);
}

} // extern "C"
