/*
 * k_beam.cu -- batched frame-synchronous prefix beam search over transcripts for CTC, n-gram CTC and ASG
 * (gtnb_beam_decode_async).
 *
 * A beam is a transcript (a prefix) with the log-semiring numerator states of the matching loss after the current
 * frame: CTC and n-gram CTC keep two (p_blank: the last frame was a blank, p_label: it was the last token), ASG one
 * (p_label).  At every frame each live beam is kept (blank / repeat / stay) and extended by every token; an extension
 * whose transcript is already a live beam is log-added into that beam's kept candidate; the best K candidates survive.
 * One CTA of 256 threads per utterance:
 * - State.  Scores, length, last token, the beam's parent slot and two 64-bit hashes (of the transcript, and of the
 *   transcript minus its last token) per slot, double-buffered in shared memory.
 * - Merges.  par[r] is the live slot holding r's transcript minus its last token, or -1: extension (par[r], last[r])
 *   is r's transcript, and no other extension is.  par stays exact from frame to frame through the kept slots; only a
 *   prefix re-created by an extension while its child was live is looked up by hash, and every hash match is
 *   confirmed by comparing the two transcripts token by token through the back-pointers.  The hash is a template
 *   parameter, so the emulation can make every hash collide.
 * - Selection.  The K + K*C candidates' order-preserving 32-bit keys sit in shared memory; a radix select of 8-bit
 *   digits (histograms in shared memory, warp 0 picks the digit) finds the K-th key, stopping at the first digit
 *   whose bin holds exactly the candidates still needed.  Equal keys at the boundary are taken in candidate order
 *   (kept beams, then by slot, then by token) by one warp and flag the utterance; the K winners are then ranked by
 *   (score, candidate order) into the new slots.
 * - Back-pointers.  16 bits per frame and slot in the workspace (previous slot, extension bit, token); the N-best
 *   transcripts are traced back from them, one thread per hypothesis.
 * - Weights.  The C x C transitions are read through the L2 in a transposed copy (WT[src][dst], one row per beam
 *   and frame, coalesced over the tokens), made once per call by beam_weights_kernel with the n-gram start weights
 *   sigma_i = logsumexp_j W[i][j] and a per-row NaN / +inf flag.  The emission row of frame t + 1 is loaded while
 *   frame t is searched.
 * - Fusion and pruning (gtnb_beam_decode_lm_async).  beam_decode_kernel's policy F: BeamLm, or BeamNoLm for
 *   gtnb_beam_decode_async, which compiles to the code without them.  Each slot also carries its LM
 *   node and lmacc (the unweighted sum of its resolved LM weights), double-buffered; candidates are ranked by the
 *   fused key am + (lm_weight * lmacc + token_bonus * len).  With token_beam P < C the P best tokens of each frame
 *   are selected first (a rank count per token; ties to the lower token), and extension (s, p) takes candidate
 *   L + s*P + p, token ptok[p].  The LM row of a beam is read through the L2 like WT's; destination nodes, and the
 *   acoustic score of an extension (recomputed), only for the winners and the merges.  After the last frame each beam
 *   adds its end weight and the live ones are ranked again by the final fused score.
 * - Lexicon and word LM (gtnb_beam_decode_lexicon_async).  Policy BeamLex: each slot also carries its trie node, word
 *   count, child mask, first child, smear and, at a word end, the completion's word-LM weight and destination, looked
 *   up once by the thread that writes the slot; admission is a bit test in shared memory and the key is
 *   am + (lm_weight * (lmacc + smear) + word_bonus * words).  After the last frame a beam completes its pending word
 *   (dropped inside one), adds its end weight, and the word ids are read off the traced tokens by walking the trie.
 */
#include <cstdint>

#include "gtnb_ptx.h"

namespace gtnb {

constexpr int kBeamThreads = 256;
constexpr int kBeamMaxK = 64;
constexpr int kBeamMaxC = 256;

/* the transcript hash, a filter only: a match is confirmed by an exact compare of the transcripts */
struct BeamHash {
  __device__ static uint64_t combine(uint64_t h, int32_t tok) {
    h ^= (uint64_t)(uint32_t)tok + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    return h * 0xff51afd7ed558ccdull;
  }
};

/* dynamic shared memory of one CTA: two hash arrays [2][K] of 8 bytes, then 4-byte words (control block, histogram,
 * two emission rows, the two start-weight rows, the double-buffered state, the candidates' scratch and keys) */
inline long long beam_smem_bytes(int K, int C) {
  return 32ll * K + 4ll * (16 + 256 + 4ll * C + 18ll * K + K + (long long)K * C);
}

/* beam_lm_smem_bytes: beam_smem_bytes plus the LM node and lmacc per slot ([2][K] each), the frame's tokens and
 * token -> position map ([C] each) and 8 words of per-warp counts */
inline long long beam_lm_smem_bytes(int K, int C) {
  return beam_smem_bytes(K, C) + 4ll * (4ll * K + 2ll * C + 8);
}

/* beam_lex_smem_bytes: beam_lm_smem_bytes plus the lexicon state per slot (trie node, word count, word id, completion
 * weight and LM destination, first child, smear: [2][K] each; the child mask [2][K][MW]), the root's mask [MW], the
 * smear of the root's children [C] and the token classes [C]; MW = ceil(C / 32) */
inline long long beam_lex_smem_bytes(int K, int C) {
  const long long MW = (C + 31) / 32;
  return beam_lm_smem_bytes(K, C) + 4ll * (14ll * K + 2ll * K * MW + MW + 2ll * C);
}

/* the policy of beam_decode_kernel: BeamNoLm for gtnb_beam_decode_async, BeamLm for gtnb_beam_decode_lm_async,
 * BeamLex for gtnb_beam_decode_lexicon_async */
struct BeamNoLm {
  static constexpr bool on = false;
  static constexpr bool lex = false;
  static constexpr int P = 0; // (unused: every token)
};
struct BeamLm {
  static constexpr bool on = true;
  static constexpr bool lex = false;
  int P; // token_beam: tokens per frame, P = C: all of them
  const float* lmw; // [S][C + 1] resolved LM weights (column C: end weights); NULL: no LM, every weight 0
  const int32_t* lmd; // [S][C + 1] destination nodes
  int start; // the LM's start node
  float lw, tb; // lm_weight, token_bonus
  float *am, *lm; // [B][N] nullable: acoustic and LM scores of the hypotheses
};
/* BeamLex: BeamLm's P, start (the word LM's start node), lw, tb (word_bonus), am and lm; lmw and lmd are NULL */
struct BeamLex : BeamLm {
  static constexpr bool lex = true;
  const int32_t* cls; // [C] token classes: 0 in-word, 1 separator, 2 word-start
  int MW; // ceil(C / 32)
  const uint32_t* mask; // [nodes][MW] trie child masks (bit c: a child labelled c)
  const int32_t* first; // [nodes] index of the first child (children numbered in token order)
  const int32_t* word; // [nodes] word id spelled at the node, or -1
  const float* smear; // [nodes] lookahead of the node
  const unsigned long long* hash; // [H][2] word LM emitting arcs: key node << 32 | word (all ones: empty), value
                                  // destination << 32 | weight bits
  unsigned long long hmul; // multiplier of the arc hash (0: every key probes from slot 0)
  int hbits; // log2 H
  const float* bow; // [S] backoff weight of each LM node
  const int32_t* bod; // [S] backoff destination, or -1
  const float* endw; // [S] resolved end weights
  int32_t *words, *counts; // [B][N][T] / [B][N] nullable: word ids and word counts of the hypotheses
};

/* the fused ranking key, in this float32 order (no contraction): am + (lw * lmacc + tb * len) */
__device__ __forceinline__ float beam_mul_rn(float a, float b) {
#ifdef GTNB_HOST_EMU
  return a * b;
#else
  return __fmul_rn(a, b);
#endif
}
__device__ __forceinline__ float beam_fuse(const BeamLm& f, float am, float lmacc, int len) {
  return __fadd_rn(am, __fadd_rn(beam_mul_rn(f.lw, lmacc), beam_mul_rn(f.tb, (float)len)));
}

/* BeamLex's ranking key, in this float32 order (no contraction): am + (lw * (lmacc + smear) + tb * words) */
__device__ __forceinline__ float beam_lex_fuse(const BeamLm& f, float am, float lmacc, float sm, int words) {
  return __fadd_rn(am, __fadd_rn(beam_mul_rn(f.lw, __fadd_rn(lmacc, sm)), beam_mul_rn(f.tb, (float)words)));
}

/* the rank of child c among the children in mask m (the children below it) */
__device__ __forceinline__ int lex_rank(const uint32_t* m, int c) {
  int r = __popc(m[c >> 5] & ((1u << (c & 31)) - 1u));
  for (int w = 0; w < (c >> 5); w++) r += __popc(m[w]);
  return r;
}
__device__ __forceinline__ bool lex_has(const uint32_t* m, int c) { return (m[c >> 5] >> (c & 31)) & 1u; }

/* the trie move of a slot at node n (word id wd or -1, first child fc, child mask m) by token c of class k; rm and
 * rfc: the root's mask and first child.  -> the node reached, or -1 when forbidden; done: the move completes n's
 * word first */
__device__ __forceinline__ int lex_move(int k, int c, int n, int wd, int fc, const uint32_t* m, const uint32_t* rm,
                                        int rfc, bool& done) {
  done = false;
  if (k == 0) return lex_has(m, c) ? fc + lex_rank(m, c) : -1;
  if (n != 0 && wd < 0) return -1;
  done = n != 0;
  if (k == 1) return 0;
  return lex_has(rm, c) ? rfc + lex_rank(rm, c) : -1;
}

/* w(s, x) of the word LM: the arc of s labelled x, else s's backoff weight plus w(backoff destination, x), added
 * innermost first as gtnb_lm_create's table adds them; -inf (dst -1) when neither exists */
__device__ float lex_resolve(const BeamLex& f, int s, int x, int& dst) {
  dst = -1;
  if (!f.hash) {
    dst = 0;
    return 0.0f;
  }
  const unsigned H = 1u << f.hbits;
  int v = s, hops = 0;
  float w = 0.0f;
  for (;;) {
    const unsigned long long key = ((unsigned long long)(unsigned)v << 32) | (unsigned)x;
    unsigned i = (unsigned)((key * f.hmul) >> (64 - f.hbits));
    unsigned long long k;
    while ((k = __ldg(f.hash + 2 * i)) != key && k != ~0ull) i = (i + 1) & (H - 1);
    if (k == key) {
      const unsigned long long e = __ldg(f.hash + 2 * i + 1);
      w = __int_as_float((int)(unsigned)e);
      dst = (int)(e >> 32);
      break;
    }
    const int nb = __ldg(f.bod + v);
    if (nb < 0) return neg_inf();
    v = nb;
    hops++;
  }
  for (int h = hops - 1; h >= 0; h--) {
    int u = s;
    for (int j = 0; j < h; j++) u = __ldg(f.bod + u);
    w = __fadd_rn(__ldg(f.bow + u), w);
  }
  return w;
}

/* control block words */
enum { kBcL = 0, kBcNwin, kBcPre, kBcShift, kBcNeed, kBcTie, kBcDone, kBcBad, kBcTieAny };

/* an order-preserving key of a score: larger is better, 0 for -inf and NaN (no candidate) */
__device__ __forceinline__ uint32_t beam_key(float v) {
  if (!(v > neg_inf())) return 0u;
  const uint32_t u = (uint32_t)__float_as_int(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float beam_key_float(uint32_t k) {
  if (k == 0u) return neg_inf();
  return __int_as_float((int)((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k));
}
__device__ __forceinline__ float beam_lse2(float a, float b) {
  const float mx = fmaxf(a, b), mn = fminf(a, b);
  if (mx == neg_inf()) return mx;
  return mx + flog1p(fexp(mn - mx));
}

/* the acoustic score of extending a beam (p_blank pb, p_label pl, their logsumexp tot, last token l) by token c */
__device__ __forceinline__ float beam_ext_am(int kind, int blank, int C, const float* er, const float* wp,
                                             const float* __restrict__ wt, float pb, float pl, float tot, int l, int c) {
  float v = neg_inf();
  if (kind == GTNB_DENSE_ASG || c != blank) {
    if (kind == GTNB_DENSE_CTC) {
      v = (c == l ? pb : tot) + er[c];
    } else {
      const float from_pl = l >= 0 && (kind == GTNB_DENSE_ASG || c != l) ? pl + __ldg(wt + (long long)l * C + c)
                                                                           : neg_inf();
      v = beam_lse2(pb + wp[c], from_pl) + er[c];
    }
  }
  return v;
}

/* one token back along the back-pointers from (t, s): the token, with (t, s) moved to before it */
__device__ __forceinline__ int beam_back(const uint16_t* bpu, int K, int& t, int& s) {
  for (;;) {
    const uint32_t e = bpu[(long long)t * K + s];
    t--;
    s = (int)(e >> 9);
    if (e & 256u) return (int)(e & 255u);
  }
}

/* the transcript of slot m at frame t equals the transcript of slot n at frame t without its last token; m holds
 * len tokens */
__device__ bool beam_same(const uint16_t* bpu, int K, int t, int m, int n, int len) {
  int ta = t, sa = m, tb = t, sb = n;
  beam_back(bpu, K, tb, sb);
  for (int r = 0; r < len; r++) {
    if (ta == tb && sa == sb) return true;
    if (beam_back(bpu, K, ta, sa) != beam_back(bpu, K, tb, sb)) return false;
  }
  return true;
}

/*
 * WT[j][i] = W[i][j] ([C][C], row = source label), wbad[i] = a NaN or +inf in W's row i (or ASG's start weight i);
 * BIGRAM: wfirst[i] = sigma_i = logsumexp_j W[i][j].  One block of 256 threads per row i.
 */
__global__ void __launch_bounds__(kBeamThreads) beam_weights_kernel(int C, int kind, const float* __restrict__ trans_w,
                                                                    float* __restrict__ wt, float* __restrict__ wfirst,
                                                                    int32_t* __restrict__ wbad) {
  GTNB_STATIC_SMEM(float, part, kBeamThreads / 32);
  const int i = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* row = trans_w + (kind == GTNB_DENSE_ASG ? C : 0) + (long long)i * C;
  bool bad = false;
  float mx = neg_inf();
  for (int j = tid; j < C; j += kBeamThreads) {
    const float v = row[j];
    wt[(long long)j * C + i] = v;
    bad |= v != v || v == CUDART_INF_F;
    mx = fmaxf(mx, v);
  }
  if (tid == 0 && kind == GTNB_DENSE_ASG) bad |= trans_w[i] != trans_w[i] || trans_w[i] == CUDART_INF_F;
  bad = __syncthreads_or(bad);
  if (kind != GTNB_DENSE_BIGRAM) {
    if (tid == 0) wbad[i] = bad;
    return;
  }
  mx = warp_max(mx);
  if (lane == 0) part[warp] = mx;
  __syncthreads();
  mx = part[0];
  for (int w = 1; w < kBeamThreads / 32; w++) mx = fmaxf(mx, part[w]);
  __syncthreads();
  float s = 0.0f;
  if (mx != neg_inf())
    for (int j = tid; j < C; j += kBeamThreads) s += expf(row[j] - mx);
  s = warp_sum(s);
  if (lane == 0) part[warp] = s;
  __syncthreads();
  if (tid == 0) {
    float tot = 0.0f;
    for (int w = 0; w < kBeamThreads / 32; w++) tot += part[w];
    wfirst[i] = mx == neg_inf() ? mx : mx + logf(tot);
    wbad[i] = bad;
  }
}

/* status 1 or 2: NaN scores, -1 lengths and rows */
__device__ void beam_flag(int b, int T, int N, int code, int32_t* tokens, int32_t* lengths, float* scores,
                          int32_t* status) {
  const int tid = threadIdx.x;
  for (long long p = tid; p < (long long)N * T; p += kBeamThreads) tokens[(long long)b * N * T + p] = -1;
  for (int n = tid; n < N; n += kBeamThreads) {
    scores[(long long)b * N + n] = CUDART_NAN_F;
    lengths[(long long)b * N + n] = -1;
  }
  if (tid == 0 && status) status[b] = code;
}

/* BeamLm: the am and lm scores of a flagged utterance (status 1 or 2), NaN like its scores */
__device__ void beam_flag_lm(int b, int N, const BeamLm& f) {
  for (int n = threadIdx.x; n < N; n += kBeamThreads) {
    if (f.am) f.am[(long long)b * N + n] = CUDART_NAN_F;
    if (f.lm) f.lm[(long long)b * N + n] = CUDART_NAN_F;
  }
}

/*
 * BeamLm, after frame T_b - 1: every live slot adds its end weight (a beam whose end weight is -inf is dropped) and
 * the N-best are the top live beams by the final fused score, ties to the lower slot (the search's own order).
 * fin / lmf ([K]) hold each slot's final fused score and LM score, rank ([K]) rank -> slot.
 */
__device__ void beam_finish_lm(int b, int T, int Tb, int C, int K, int N, const uint16_t* bpu, int cur, int* ctl,
                               const float* stot, const int* slen, const int* snode, const float* slm, float* fin,
                               float* lmf, int* rank, int32_t* tokens, int32_t* lengths, float* scores,
                               int32_t* status, const BeamLm& f) {
  const int tid = threadIdx.x;
  const int L = ctl[kBcL];
  if (tid < L) {
    const int m = cur * K + tid;
    const float we = f.lmw ? __ldg(f.lmw + (long long)snode[m] * (C + 1) + C) : 0.0f;
    const float lm = slm[m] + we;
    fin[tid] = we == neg_inf() ? neg_inf() : beam_fuse(f, stot[m], lm, slen[m]);
    lmf[tid] = lm;
  }
  __syncthreads();
  int live = 0;
  for (int i = 0; i < L; i++) live += fin[i] > neg_inf();
  if (tid < L && fin[tid] > neg_inf()) {
    int r = 0;
    for (int i = 0; i < L; i++) r += fin[i] > fin[tid] || (fin[i] == fin[tid] && i < tid);
    rank[r] = tid;
  }
  __syncthreads();
  int32_t* out = tokens + (long long)b * N * T;
  for (int n = tid; n < N; n += kBeamThreads) {
    const int m = n < live ? rank[n] : -1;
    const int len = m >= 0 ? slen[cur * K + m] : -1;
    const long long o = (long long)b * N + n;
    scores[o] = m >= 0 ? fin[m] : neg_inf();
    if (f.am) f.am[o] = m >= 0 ? stot[cur * K + m] : neg_inf();
    if (f.lm) f.lm[o] = m >= 0 ? lmf[m] : neg_inf();
    lengths[o] = len;
    int tt = Tb - 1, s = m;
    for (int p = len - 1; p >= 0; p--) out[(long long)n * T + p] = beam_back(bpu, K, tt, s);
  }
  for (long long p = tid; p < (long long)N * T; p += kBeamThreads) {
    const int n = (int)(p / T);
    if (p - (long long)n * T >= (n < live ? slen[cur * K + rank[n]] : 0)) out[p] = -1;
  }
  if (tid == 0) {
    bool tied = ctl[kBcTieAny] != 0;
    for (int n = 0; n + 1 < live && n < N; n++) tied |= fin[rank[n]] == fin[rank[n + 1]];
    if (status) status[b] = tied ? 3 : 0;
  }
}

/* BeamLex: beam_flag_lm, and -1 word rows and counts */
__device__ void beam_flag_lex(int b, int T, int N, const BeamLex& f) {
  beam_flag_lm(b, N, f);
  for (long long p = threadIdx.x; p < (long long)N * T; p += kBeamThreads)
    if (f.words) f.words[(long long)b * N * T + p] = -1;
  for (int n = threadIdx.x; n < N; n += kBeamThreads)
    if (f.counts) f.counts[(long long)b * N + n] = -1;
}

/*
 * BeamLex, after frame T_b - 1: every live slot at a word end completes its word, a slot inside a word is dropped;
 * each adds its end weight (dropped at -inf) and the N-best are the top live beams by am + (lw * lm + tb * words),
 * ties to the lower slot.  Each hypothesis's words are read off its traced tokens by walking the trie.  fin / lmf /
 * nwd ([K]) hold each slot's final fused score, LM score and word count, rank ([K]) rank -> slot.
 */
__device__ void beam_finish_lex(int b, int T, int Tb, int K, int N, const uint16_t* bpu, int cur, int* ctl,
                                const float* stot, const int* slen, const int* snode, const float* slm,
                                const int* strie, const int* swn, const int* swd, const float* scw, const int* scd,
                                const int* tcls, float* fin, float* lmf, int* nwd, int* rank, int32_t* tokens,
                                int32_t* lengths, float* scores, int32_t* status, const BeamLex& f) {
  const int tid = threadIdx.x;
  const int L = ctl[kBcL];
  if (tid < L) {
    const int m = cur * K + tid;
    float lm = slm[m];
    int node = snode[m], nw = swn[m];
    bool ok = true;
    if (strie[m] != 0) {
      ok = swd[m] >= 0 && scw[m] > neg_inf();
      lm = __fadd_rn(lm, scw[m]);
      node = scd[m];
      nw++;
    }
    const float we = ok ? (f.endw ? __ldg(f.endw + node) : 0.0f) : neg_inf();
    lm = __fadd_rn(lm, we);
    fin[tid] = we == neg_inf() ? neg_inf() : beam_fuse(f, stot[m], lm, nw);
    lmf[tid] = lm;
    nwd[tid] = nw;
  }
  __syncthreads();
  int live = 0;
  for (int i = 0; i < L; i++) live += fin[i] > neg_inf();
  if (tid < L && fin[tid] > neg_inf()) {
    int r = 0;
    for (int i = 0; i < L; i++) r += fin[i] > fin[tid] || (fin[i] == fin[tid] && i < tid);
    rank[r] = tid;
  }
  __syncthreads();
  int32_t* out = tokens + (long long)b * N * T;
  int32_t* wout = f.words ? f.words + (long long)b * N * T : nullptr;
  for (int n = tid; n < N; n += kBeamThreads) {
    const int m = n < live ? rank[n] : -1;
    const int len = m >= 0 ? slen[cur * K + m] : -1;
    const long long o = (long long)b * N + n;
    scores[o] = m >= 0 ? fin[m] : neg_inf();
    if (f.am) f.am[o] = m >= 0 ? stot[cur * K + m] : neg_inf();
    if (f.lm) f.lm[o] = m >= 0 ? lmf[m] : neg_inf();
    if (f.counts) f.counts[o] = m >= 0 ? nwd[m] : -1;
    lengths[o] = len;
    int tt = Tb - 1, s = m;
    for (int p = len - 1; p >= 0; p--) out[(long long)n * T + p] = beam_back(bpu, K, tt, s);
    if (wout && len > 0) { // (the transcript was admitted: every move exists)
      int node = 0, k = 0;
      for (int p = 0; p < len; p++) {
        const int c = out[(long long)n * T + p], cl = tcls[c];
        if (cl != 0 && node != 0) wout[(long long)n * T + k++] = __ldg(f.word + node);
        if (cl == 1) {
          node = 0;
        } else {
          const int from = cl == 0 ? node : 0;
          node = __ldg(f.first + from) + lex_rank(f.mask + (long long)from * f.MW, c);
        }
      }
      if (node != 0) wout[(long long)n * T + k++] = __ldg(f.word + node);
    }
  }
  __syncthreads();
  for (long long p = tid; p < (long long)N * T; p += kBeamThreads) {
    const int n = (int)(p / T);
    const int r = n < live ? rank[n] : -1;
    if (p - (long long)n * T >= (r >= 0 ? slen[cur * K + r] : 0)) out[p] = -1;
    if (wout && p - (long long)n * T >= (r >= 0 ? nwd[r] : 0)) wout[p] = -1;
  }
  if (tid == 0) {
    bool tied = ctl[kBcTieAny] != 0;
    for (int n = 0; n + 1 < live && n < N; n++) tied |= fin[rank[n]] == fin[rank[n + 1]];
    if (status) status[b] = tied ? 3 : 0;
  }
}

/*
 * One CTA of kBeamThreads per utterance b.  emissions [B][T][C] of E; input_lens [B] (nullable: T); kind
 * GTNB_DENSE_CTC / _BIGRAM / _ASG; wt [C][C] (transposed W), wfirst [C] (BIGRAM sigma, ASG start weights) and wbad
 * [C] from beam_weights_kernel (unused for CTC); blank (CTC, BIGRAM); K beams, N hypotheses.  bp: [B][T][K] back-
 * pointers (scratch).  Out: tokens [B][N][T], lengths [B][N], scores [B][N], status [B] (nullable).  F: BeamNoLm, or
 * BeamLm with the LM, its weights, token_beam and the am / lm outputs.
 */
template <class E, class Hash, class F = BeamNoLm>
__global__ void __launch_bounds__(kBeamThreads) beam_decode_kernel(
    const E* __restrict__ emissions, int T, int C, const int32_t* __restrict__ input_lens, int kind,
    const float* __restrict__ wt, const float* __restrict__ wfirst, const int32_t* __restrict__ wbad, int blank, int K,
    int N, uint16_t* bp, int32_t* __restrict__ tokens, int32_t* __restrict__ lengths, float* __restrict__ scores,
    int32_t* __restrict__ status, const F fz = F()) {
  GTNB_DYNAMIC_SMEM(uint64_t, hsm);
  uint64_t* hh = hsm; // [2][K] hash of the transcript
  uint64_t* hq = hsm + 2 * K; // [2][K] hash of the transcript minus its last token
  int* ctl = reinterpret_cast<int*>(hsm + 4 * K);
  int* hist = ctl + 16;
  float* erow = reinterpret_cast<float*>(hist + 256); // [2][C]
  float* w0 = erow + 2 * C; // weight of a token entered from p_blank at frame 0 (BIGRAM sigma, ASG start)
  float* wb = w0 + C; // ... at frames >= 1 (BIGRAM W[c][blank])
  float* spb = wb + C; // [2][K] p_blank
  float* spl = spb + 2 * K; // [2][K] p_label
  float* stot = spl + 2 * K; // [2][K] logsumexp(p_blank, p_label)
  int* slen = reinterpret_cast<int*>(stot + 2 * K); // [2][K]
  int* slast = slen + 2 * K; // [2][K] last token, -1 for the empty transcript
  int* spar = slast + 2 * K; // [2][K] the slot holding the transcript minus its last token, or -1
  float* kpb = reinterpret_cast<float*>(spar + 2 * K); // [K] kept candidates' states
  float* kpl = kpb + K;
  int* kslot = reinterpret_cast<int*>(kpl + K); // [K] old slot -> its kept beam's new slot, or -1
  int* src = kslot + K; // [K] new slot -> candidate
  int* widx = src + K; // [K] winners: candidate
  uint32_t* wkey = reinterpret_cast<uint32_t*>(widx + K); // [K] winners: key
  uint32_t* keys = wkey + K; // [K + K*P]: kept beams r at r, extension (s, p) at L + s*P + p
  // (BeamLm only)
  int* snode = reinterpret_cast<int*>(keys + K + K * C); // [2][K] LM node
  float* slm = reinterpret_cast<float*>(snode + 2 * K); // [2][K] lmacc
  int* ptok = reinterpret_cast<int*>(slm + 2 * K); // [P] the frame's tokens, ascending
  int* ppos = ptok + C; // [C] token -> its position in ptok, or -1
  int* wcnt = ppos + C; // [8] selected tokens per warp
  // (BeamLex only)
  const int MW = (C + 31) / 32;
  int* strie = wcnt + 8; // [2][K] trie node (the root is 0, its children 1, 2, ... in token order)
  int* swn = strie + 2 * K; // [2][K] word count
  int* swd = swn + 2 * K; // [2][K] word id of the trie node, or -1
  float* scw = reinterpret_cast<float*>(swd + 2 * K); // [2][K] completion weight w(LM node, word id), word ends
  int* scd = reinterpret_cast<int*>(scw + 2 * K); // [2][K] ... and its LM destination
  int* sfc = scd + 2 * K; // [2][K] first child
  float* ssm = reinterpret_cast<float*>(sfc + 2 * K); // [2][K] smear
  uint32_t* smask = reinterpret_cast<uint32_t*>(ssm + 2 * K); // [2][K][MW] child mask
  uint32_t* rmask = smask + 2 * K * MW; // [MW] the root's child mask
  float* rsm = reinterpret_cast<float*>(rmask + MW); // [C] smear of the root's child labelled c
  int* tcls = reinterpret_cast<int*>(rsm + C); // [C] token classes
  const int P = F::on ? fz.P : C;

  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int Tb = input_lens ? input_lens[b] : T;
  if (!(Tb >= 0 && Tb <= T)) {
    beam_flag(b, T, N, 2, tokens, lengths, scores, status);
    if constexpr (F::lex)
      beam_flag_lex(b, T, N, fz);
    else if constexpr (F::on)
      beam_flag_lm(b, N, fz);
    return;
  }
  const E* em = emissions + (long long)b * T * C;
  uint16_t* bpu = bp + (long long)b * T * K;
  if (tid < 16) ctl[tid] = 0;
  for (int i = tid; i < 256; i += kBeamThreads) hist[i] = 0;
  if (tid == 0) {
    ctl[kBcL] = 1;
    spb[0] = 0.0f;
    spl[0] = neg_inf();
    stot[0] = 0.0f;
    slen[0] = 0;
    slast[0] = -1;
    spar[0] = -1;
    hh[0] = hq[0] = 0;
    if constexpr (F::on) {
      snode[0] = fz.lmw ? fz.start : 0;
      slm[0] = 0.0f;
    }
  }
  if constexpr (F::on) {
    if (tid < C) { // (every frame's selection when P < C)
      ptok[tid] = tid;
      ppos[tid] = tid;
    }
  }
  if constexpr (F::lex) {
    if (tid == 0) {
      snode[0] = fz.start;
      strie[0] = swn[0] = scd[0] = 0;
      swd[0] = -1;
      scw[0] = ssm[0] = 0.0f;
      sfc[0] = __ldg(fz.first);
    }
    if (tid < MW) smask[tid] = rmask[tid] = __ldg(fz.mask + tid);
    if (tid < C) {
      tcls[tid] = __ldg(fz.cls + tid);
      rsm[tid] = lex_has(fz.mask, tid) ? __ldg(fz.smear + 1 + lex_rank(fz.mask, tid)) : 0.0f;
    }
  }
  __syncthreads();
  if (tid < C) {
    w0[tid] = kind == GTNB_DENSE_CTC ? 0.0f : wfirst[tid];
    wb[tid] = kind == GTNB_DENSE_BIGRAM ? wt[(long long)blank * C + tid] : 0.0f;
    if (Tb > 0) {
      const float v = ldg_elem(em + tid);
      erow[tid] = v;
      if (v != v || v == CUDART_INF_F || (kind != GTNB_DENSE_CTC && wbad[tid])) ctl[kBcBad] = 1;
    }
  }
  __syncthreads();

  int cur = 0;
  for (int t = 0; t < Tb; t++) {
    if (ctl[kBcBad]) break;
    const int L = ctl[kBcL];
    const float* er = erow + (t & 1) * C;
    const bool pf = t + 1 < Tb && tid < C;
    const float ahead = pf ? ldg_elem(em + (long long)(t + 1) * C + tid) : 0.0f;
    const float* wp = t == 0 ? w0 : wb;
    const float *pb0 = spb + cur * K, *pl0 = spl + cur * K, *tot0 = stot + cur * K;
    const int *len0 = slen + cur * K, *last0 = slast + cur * K, *par0 = spar + cur * K;
    const int* node0 = snode + cur * K;
    const float* lm0 = slm + cur * K;
    const int *trie0 = strie + cur * K, *wn0 = swn + cur * K, *wd0 = swd + cur * K, *cd0 = scd + cur * K;
    const int* fc0 = sfc + cur * K;
    const float *cw0 = scw + cur * K, *sm0 = ssm + cur * K;
    const uint32_t* mask0 = smask + cur * K * MW;

    if constexpr (F::on) {
      // token pruning: the P best tokens of the frame (blank excluded for CTC and BIGRAM), ties to the lower token;
      // a tie at the boundary between finite emissions flags the utterance
      if (P < C) {
        bool sel = false;
        if (tid < C && (kind == GTNB_DENSE_ASG || tid != blank)) {
          const float v = er[tid];
          int gt = 0, eq = 0;
          for (int j = 0; j < C; j++) {
            const float x = er[j];
            const bool ok = kind == GTNB_DENSE_ASG || j != blank;
            gt += ok && x > v;
            eq += ok && x == v && j < tid;
          }
          sel = gt + eq < P;
          if (gt + eq == P && eq > 0 && v > neg_inf()) ctl[kBcTieAny] = 1;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, sel);
        if (lane == 0) wcnt[warp] = __popc(bal);
        __syncthreads();
        if (tid < C) {
          int pos = __popc(bal & ((1u << lane) - 1u));
          for (int w = 0; w < warp; w++) pos += wcnt[w];
          ppos[tid] = sel ? pos : -1;
          if (sel) ptok[pos] = tid;
        }
        __syncthreads();
      }
    }

    // candidates: kept beams, then every extension
    if (tid < L) {
      const float pb = pb0[tid], pl = pl0[tid];
      const int l = last0[tid];
      float nb, nl = neg_inf();
      if (kind == GTNB_DENSE_CTC) {
        nb = tot0[tid] + er[blank];
        if (l >= 0) nl = pl + er[l];
      } else {
        const float* wl = wt + (long long)(l < 0 ? 0 : l) * C;
        nb = kind == GTNB_DENSE_ASG ? neg_inf()
                                    : beam_lse2(pb + wp[blank], l >= 0 ? pl + __ldg(wl + blank) : neg_inf()) + er[blank];
        if (l >= 0) nl = pl + __ldg(wl + l) + er[l];
      }
      kpb[tid] = nb;
      kpl[tid] = nl;
      float v = beam_lse2(nb, nl);
      if constexpr (F::lex)
        v = beam_lex_fuse(fz, v, lm0[tid], sm0[tid], wn0[tid]);
      else if constexpr (F::on)
        v = beam_fuse(fz, v, lm0[tid], len0[tid]);
      keys[tid] = beam_key(v);
      kslot[tid] = -1;
    }
    if (tid == 0) ctl[kBcNwin] = ctl[kBcDone] = 0;
    const int next = L * P;
    {
      int s = tid / P, p = tid - s * P;
      for (int q = tid; q < next; q += kBeamThreads) {
        const int c = F::on ? ptok[p] : p;
        float v = neg_inf();
        if constexpr (!F::on) {
          if (kind == GTNB_DENSE_ASG || c != blank) {
            const float pb = pb0[s], pl = pl0[s];
            const int l = last0[s];
            if (kind == GTNB_DENSE_CTC) {
              v = (c == l ? pb : tot0[s]) + er[c];
            } else {
              const float from_pl = l >= 0 && (kind == GTNB_DENSE_ASG || c != l) ? pl + __ldg(wt + (long long)l * C + c)
                                                                                   : neg_inf();
              v = beam_lse2(pb + wp[c], from_pl) + er[c];
            }
          }
        } else if constexpr (F::lex) {
          v = beam_ext_am(kind, blank, C, er, wp, wt, pb0[s], pl0[s], tot0[s], last0[s], c);
          if (v > neg_inf()) { // (admission is a bit test; an in-word child's smear is one row per beam, via the L2)
            bool done;
            const int k = tcls[c];
            const int ch = lex_move(k, c, trie0[s], wd0[s], fc0[s], mask0 + s * MW, rmask, 1, done);
            if (ch < 0 || (done && !(cw0[s] > neg_inf()))) {
              v = neg_inf();
            } else {
              const float sm = k == 0 ? __ldg(fz.smear + ch) : k == 2 ? rsm[c] : 0.0f;
              v = beam_lex_fuse(fz, v, done ? __fadd_rn(lm0[s], cw0[s]) : lm0[s], sm, wn0[s] + (int)done);
            }
          }
        } else {
          v = beam_ext_am(kind, blank, C, er, wp, wt, pb0[s], pl0[s], tot0[s], last0[s], c);
          if (v > neg_inf() && fz.lmw) {
            const float w = __ldg(fz.lmw + (long long)node0[s] * (C + 1) + c); // (one row per beam, via the L2)
            v = w == neg_inf() ? w : beam_fuse(fz, v, lm0[s] + w, len0[s] + 1);
          } else if (v > neg_inf()) {
            v = beam_fuse(fz, v, lm0[s], len0[s] + 1);
          }
        }
        keys[L + q] = beam_key(v);
        p += kBeamThreads;
        while (p >= P) {
          p -= P;
          s++;
        }
      }
    }
    __syncthreads();

    // merge: extension (par[r], last[r]) is r's transcript (absent when last[r] was pruned at this frame)
    if (tid < L && par0[tid] >= 0 && (!F::on || ppos[last0[tid]] >= 0)) {
      const int q = L + par0[tid] * P + (F::on ? ppos[last0[tid]] : last0[tid]);
      float v = beam_key_float(keys[q]);
      if constexpr (F::on) { // (the key holds the fused score: the acoustic one again)
        const int s = par0[tid];
        v = keys[q] ? beam_ext_am(kind, blank, C, er, wp, wt, pb0[s], pl0[s], tot0[s], last0[s], last0[tid])
                    : neg_inf();
      }
      keys[q] = 0u;
      kpl[tid] = beam_lse2(kpl[tid], v);
      v = beam_lse2(kpb[tid], kpl[tid]);
      if constexpr (F::lex)
        v = beam_lex_fuse(fz, v, lm0[tid], sm0[tid], wn0[tid]);
      else if constexpr (F::on)
        v = beam_fuse(fz, v, lm0[tid], len0[tid]);
      keys[tid] = beam_key(v);
    }
    __syncthreads();
    // radix select of the K-th key among the nonzero keys
    const int ncand = L + next;
    uint32_t pre = 0u;
    int sh = 0, need = K;
    bool tie = false;
    for (int pass = 0; pass < 4; pass++) {
      const int d_sh = 24 - 8 * pass;
      // runs of one digit are added at once: most candidates share the few top digits, and same-address shared
      // atomics serialise
      int run_bin = 0, run = 0;
      for (int j = tid; j < ncand; j += kBeamThreads) {
        const uint32_t k = keys[j];
        if (k && (pass == 0 || (k >> (d_sh + 8)) == pre)) {
          const int bin = (int)((k >> d_sh) & 255u);
          if (bin != run_bin && run) {
            atomicAdd(&hist[run_bin], run);
            run = 0;
          }
          run_bin = bin;
          run++;
        }
      }
      if (run) atomicAdd(&hist[run_bin], run);
      __syncthreads();
      if (warp == 0) {
        int cnt[8], sum = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) {
          const int bin = 255 - 8 * lane - i; // lane 0 holds the highest bins
          cnt[i] = hist[bin];
          hist[bin] = 0;
          sum += cnt[i];
        }
        int inc = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int y = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= o) inc += y;
        }
        const int total = __shfl_sync(0xffffffffu, inc, 31);
        if (pass == 0 && total <= need) {
          if (lane == 0) { // every candidate wins
            ctl[kBcPre] = 0;
            ctl[kBcShift] = 0;
            ctl[kBcTie] = 0;
            ctl[kBcDone] = 1;
          }
        } else if (inc - sum < need && inc >= need) {
          int above = inc - sum, d = -1, eq = 0;
#pragma unroll
          for (int i = 0; i < 8; i++) { // (unrolled: cnt stays in registers)
            if (d < 0 && above + cnt[i] >= need) {
              d = 255 - 8 * lane - i;
              eq = cnt[i];
            }
            if (d < 0) above += cnt[i];
          }
          const int left = need - above;
          ctl[kBcPre] = (int)((pre << 8) | (uint32_t)d);
          ctl[kBcShift] = d_sh;
          ctl[kBcNeed] = left;
          ctl[kBcTie] = pass == 3 && eq > left;
          ctl[kBcDone] = eq == left || pass == 3;
        }
      }
      __syncthreads();
      pre = (uint32_t)ctl[kBcPre];
      sh = ctl[kBcShift];
      need = ctl[kBcNeed];
      tie = ctl[kBcTie] != 0;
      // (warp 0 rewrites ctl only after the next pass's first barrier)
      if (ctl[kBcDone]) break;
    }

    // the winners: keys above the boundary, and at it all of them or (a tie) the first `need` in candidate order
    for (int j = tid; j < ncand; j += kBeamThreads) {
      const uint32_t k = keys[j];
      if (k && ((k >> sh) > pre || (!tie && (k >> sh) == pre))) {
        const int w = atomicAdd(&ctl[kBcNwin], 1);
        widx[w] = j;
        wkey[w] = k;
      }
    }
    __syncthreads();
    if (tie) {
      if (warp == 0) {
        const int base = ctl[kBcNwin];
        const unsigned below = (1u << lane) - 1u;
        int taken = 0;
        for (int j0 = 0; j0 < ncand && taken < need; j0 += 32) {
          const int j = j0 + lane;
          const uint32_t k = j < ncand ? keys[j] : 0u;
          const bool m = k && (k >> sh) == pre;
          const unsigned bal = __ballot_sync(0xffffffffu, m);
          const int rank = taken + __popc(bal & below);
          if (m && rank < need) {
            widx[base + rank] = j;
            wkey[base + rank] = k;
          }
          taken += __popc(bal);
        }
        if (lane == 0) {
          ctl[kBcNwin] = base + need;
          ctl[kBcTieAny] = 1;
        }
      }
      __syncthreads();
    }
    const int nw = ctl[kBcNwin];

    // rank the winners into the new slots (score descending, then candidate order)
    const int nx = cur ^ 1;
    if (tid < nw) {
      const uint32_t k = wkey[tid];
      const int j = widx[tid];
      int n = 0;
      for (int i = 0; i < nw; i++) {
        const uint32_t ki = wkey[i];
        n += ki > k || (ki == k && widx[i] < j);
      }
      uint32_t code;
      float am = 0.0f; // (BeamLm: the acoustic score; the key holds the fused one)
      if (j < L) {
        spb[nx * K + n] = kpb[j];
        spl[nx * K + n] = kpl[j];
        slen[nx * K + n] = len0[j];
        slast[nx * K + n] = last0[j];
        hh[nx * K + n] = hh[cur * K + j];
        hq[nx * K + n] = hq[cur * K + j];
        if constexpr (F::on) {
          am = beam_lse2(kpb[j], kpl[j]);
          snode[nx * K + n] = node0[j];
          slm[nx * K + n] = lm0[j];
        }
        if constexpr (F::lex) {
          const int o = nx * K + n;
          strie[o] = trie0[j];
          swn[o] = wn0[j];
          swd[o] = wd0[j];
          scw[o] = cw0[j];
          scd[o] = cd0[j];
          sfc[o] = fc0[j];
          ssm[o] = sm0[j];
          for (int w = 0; w < MW; w++) smask[o * MW + w] = mask0[j * MW + w];
        }
        kslot[j] = n;
        code = (uint32_t)j << 9;
      } else {
        const int s = (j - L) / P, p = j - L - s * P;
        const int c = F::on ? ptok[p] : p;
        if constexpr (F::lex) {
          // the new slot's trie node and LM state; on a word end, the completion's weight and destination are looked
          // up here, once, so that no LM lookup sits on the per-candidate path
          am = beam_ext_am(kind, blank, C, er, wp, wt, pb0[s], pl0[s], tot0[s], last0[s], c);
          bool done;
          const int ch = lex_move(tcls[c], c, trie0[s], wd0[s], fc0[s], mask0 + s * MW, rmask, 1, done);
          const int o = nx * K + n;
          const int ln = done ? cd0[s] : node0[s];
          snode[o] = ln;
          slm[o] = done ? __fadd_rn(lm0[s], cw0[s]) : lm0[s];
          swn[o] = wn0[s] + (int)done;
          strie[o] = ch;
          const int wd = __ldg(fz.word + ch);
          swd[o] = wd;
          sfc[o] = __ldg(fz.first + ch);
          ssm[o] = __ldg(fz.smear + ch);
          for (int w = 0; w < MW; w++) smask[o * MW + w] = __ldg(fz.mask + (long long)ch * MW + w);
          int d = 0;
          scw[o] = wd >= 0 ? lex_resolve(fz, ln, wd, d) : 0.0f;
          scd[o] = d;
        } else if constexpr (F::on) {
          am = beam_ext_am(kind, blank, C, er, wp, wt, pb0[s], pl0[s], tot0[s], last0[s], c);
          const long long at = (long long)node0[s] * (C + 1) + c;
          snode[nx * K + n] = fz.lmw ? __ldg(fz.lmd + at) : 0;
          slm[nx * K + n] = fz.lmw ? lm0[s] + __ldg(fz.lmw + at) : lm0[s];
        }
        spb[nx * K + n] = neg_inf();
        spl[nx * K + n] = F::on ? am : beam_key_float(k);
        slen[nx * K + n] = len0[s] + 1;
        slast[nx * K + n] = c;
        hh[nx * K + n] = Hash::combine(hh[cur * K + s], c);
        hq[nx * K + n] = hh[cur * K + s];
        code = ((uint32_t)s << 9) | 256u | (uint32_t)c;
      }
      stot[nx * K + n] = F::on ? am : beam_key_float(k);
      src[n] = j;
      bpu[(long long)t * K + n] = (uint16_t)code;
    }
    __syncthreads();

    // parents in the new frame; a kept beam whose parent was not live looks for it among the new extensions
    if (tid < nw) {
      const int j = src[tid];
      int par = -1;
      if (j >= L) {
        par = kslot[(j - L) / P];
      } else if (par0[j] >= 0) {
        par = kslot[par0[j]];
      } else if (len0[j] >= 2) {
        const uint64_t want = hq[nx * K + tid];
        for (int m = 0; m < nw && par < 0; m++)
          if (src[m] >= L && slen[nx * K + m] == len0[j] - 1 && hh[nx * K + m] == want &&
              beam_same(bpu, K, t, m, tid, len0[j] - 1))
            par = m;
      }
      spar[nx * K + tid] = par;
    }
    if (pf) {
      erow[((t + 1) & 1) * C + tid] = ahead;
      if (ahead != ahead || ahead == CUDART_INF_F) ctl[kBcBad] = 1;
    }
    if (tid == 0) ctl[kBcL] = nw;
    cur = nx;
    __syncthreads();
  }

  if (ctl[kBcBad]) {
    beam_flag(b, T, N, 1, tokens, lengths, scores, status);
    if constexpr (F::lex)
      beam_flag_lex(b, T, N, fz);
    else if constexpr (F::on)
      beam_flag_lm(b, N, fz);
    return;
  }
  if constexpr (F::lex) {
    beam_finish_lex(b, T, Tb, K, N, bpu, cur, ctl, stot, slen, snode, slm, strie, swn, swd, scw, scd, tcls, kpb, kpl,
                    widx, src, tokens, lengths, scores, status, fz);
    return;
  } else if constexpr (F::on) {
    beam_finish_lm(b, T, Tb, C, K, N, bpu, cur, ctl, stot, slen, snode, slm, kpb, kpl, src, tokens, lengths, scores,
                   status, fz);
    return;
  }
  const int L = ctl[kBcL];
  int32_t* out = tokens + (long long)b * N * T;
  for (int n = tid; n < N; n += kBeamThreads) {
    const int len = n < L ? slen[cur * K + n] : -1;
    scores[(long long)b * N + n] = n < L ? stot[cur * K + n] : neg_inf();
    lengths[(long long)b * N + n] = len;
    int tt = Tb - 1, s = n;
    for (int p = len - 1; p >= 0; p--) out[(long long)n * T + p] = beam_back(bpu, K, tt, s);
  }
  for (long long p = tid; p < (long long)N * T; p += kBeamThreads) {
    const int n = (int)(p / T);
    if (p - (long long)n * T >= (n < L ? slen[cur * K + n] : 0)) out[p] = -1;
  }
  if (tid == 0) {
    bool tied = ctl[kBcTieAny] != 0;
    for (int n = 0; n + 1 < L && n < N; n++) tied |= stot[cur * K + n] == stot[cur * K + n + 1];
    if (status) status[b] = tied ? 3 : 0;
  }
}

#ifndef GTNB_HOST_EMU

bool beam_decode_supported(int C, int beam, int nbest) {
  return C >= 1 && C <= kBeamMaxC && beam >= 1 && beam <= kBeamMaxK && nbest >= 1 && nbest <= beam;
}

int launch_beam_weights(gtnb_ctx* ctx, int C, int kind, const float* trans_w, float* wt, float* wfirst,
                        int32_t* wbad) {
  GTNB_LAUNCH(ctx, "beam_weights",
              beam_weights_kernel<<<C, kBeamThreads, 0, ctx->stream>>>(C, kind, trans_w, wt, wfirst, wbad));
  return GTNB_OK;
}

int launch_beam_decode(gtnb_ctx* ctx, int B, int T, int C, const void* emissions, int dtype,
                       const int32_t* input_lens, int kind, const float* wt, const float* wfirst, const int32_t* wbad,
                       int blank, int K, int N, uint16_t* bp, int32_t* tokens, int32_t* lengths, float* scores,
                       int32_t* status) {
  if (B <= 0) return GTNB_OK;
  const long long smem = beam_smem_bytes(K, C);
#define GTNB_BEAM_LAUNCH(E_)                                                                                  \
  {                                                                                                           \
    if (smem > 48 * 1024) {                                                                                   \
      const int rc__ = ensure_max_smem(ctx, (const void*)beam_decode_kernel<E_, BeamHash, BeamNoLm>);                   \
      if (rc__) return rc__;                                                                                  \
    }                                                                                                         \
    GTNB_LAUNCH(ctx, "beam_decode",                                                                           \
                beam_decode_kernel<E_, BeamHash, BeamNoLm><<<B, kBeamThreads, smem, ctx->stream>>>(                     \
                    static_cast<const E_*>(emissions), T, C, input_lens, kind, wt, wfirst, wbad, blank, K, N, bp, \
                    tokens, lengths, scores, status));                                                        \
  }
  if (dtype == GTNB_BF16)
    GTNB_BEAM_LAUNCH(bf16_t)
  else if (dtype == GTNB_F16)
    GTNB_BEAM_LAUNCH(f16_t)
  else
    GTNB_BEAM_LAUNCH(float)
#undef GTNB_BEAM_LAUNCH
  return GTNB_OK;
}

int launch_beam_decode_lm(gtnb_ctx* ctx, int B, int T, int C, const void* emissions, int dtype,
                          const int32_t* input_lens, int kind, const float* wt, const float* wfirst, const int32_t* wbad,
                          int blank, int K, int N, uint16_t* bp, int32_t* tokens, int32_t* lengths, float* scores,
                          int32_t* status, const BeamLmLaunch& lm) {
  if (B <= 0) return GTNB_OK;
  const long long smem = beam_lm_smem_bytes(K, C);
  const BeamLm f{lm.P, lm.lmw, lm.lmd, lm.start, lm.lm_weight, lm.token_bonus, lm.am_scores, lm.lm_scores};
#define GTNB_BEAM_LM_LAUNCH(E_)                                                                               \
  {                                                                                                           \
    if (smem > 48 * 1024) {                                                                                   \
      const int rc__ = ensure_max_smem(ctx, (const void*)beam_decode_kernel<E_, BeamHash, BeamLm>);           \
      if (rc__) return rc__;                                                                                  \
    }                                                                                                         \
    GTNB_LAUNCH(ctx, "beam_decode_lm",                                                                        \
                beam_decode_kernel<E_, BeamHash, BeamLm><<<B, kBeamThreads, smem, ctx->stream>>>(             \
                    static_cast<const E_*>(emissions), T, C, input_lens, kind, wt, wfirst, wbad, blank, K, N, bp, \
                    tokens, lengths, scores, status, f));                                                     \
  }
  if (dtype == GTNB_BF16)
    GTNB_BEAM_LM_LAUNCH(bf16_t)
  else if (dtype == GTNB_F16)
    GTNB_BEAM_LM_LAUNCH(f16_t)
  else
    GTNB_BEAM_LM_LAUNCH(float)
#undef GTNB_BEAM_LM_LAUNCH
  return GTNB_OK;
}

int launch_beam_decode_lex(gtnb_ctx* ctx, int B, int T, int C, const void* emissions, int dtype,
                           const int32_t* input_lens, int kind, const float* wt, const float* wfirst,
                           const int32_t* wbad, int blank, int K, int N, uint16_t* bp, int32_t* tokens,
                           int32_t* lengths, float* scores, int32_t* status, const BeamLexLaunch& x) {
  if (B <= 0) return GTNB_OK;
  const long long smem = beam_lex_smem_bytes(K, C);
  BeamLex f;
  static_cast<BeamLm&>(f) = BeamLm{x.P, nullptr, nullptr, x.start, x.lm_weight, x.word_bonus, x.am_scores,
                                   x.lm_scores};
  f.cls = x.cls;
  f.MW = (C + 31) / 32;
  f.mask = x.mask;
  f.first = x.first;
  f.word = x.word;
  f.smear = x.smear;
  f.hash = x.hash;
  f.hmul = x.hmul;
  f.hbits = x.hbits;
  f.bow = x.bow;
  f.bod = x.bod;
  f.endw = x.endw;
  f.words = x.words;
  f.counts = x.counts;
#define GTNB_BEAM_LEX_LAUNCH(E_)                                                                              \
  {                                                                                                           \
    if (smem > 48 * 1024) {                                                                                   \
      const int rc__ = ensure_max_smem(ctx, (const void*)beam_decode_kernel<E_, BeamHash, BeamLex>);          \
      if (rc__) return rc__;                                                                                  \
    }                                                                                                         \
    GTNB_LAUNCH(ctx, "beam_decode_lexicon",                                                                   \
                beam_decode_kernel<E_, BeamHash, BeamLex><<<B, kBeamThreads, smem, ctx->stream>>>(            \
                    static_cast<const E_*>(emissions), T, C, input_lens, kind, wt, wfirst, wbad, blank, K, N, bp, \
                    tokens, lengths, scores, status, f));                                                     \
  }
  if (dtype == GTNB_BF16)
    GTNB_BEAM_LEX_LAUNCH(bf16_t)
  else if (dtype == GTNB_F16)
    GTNB_BEAM_LEX_LAUNCH(f16_t)
  else
    GTNB_BEAM_LEX_LAUNCH(float)
#undef GTNB_BEAM_LEX_LAUNCH
  return GTNB_OK;
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
