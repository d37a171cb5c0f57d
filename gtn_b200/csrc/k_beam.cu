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
 * - Policies.  beam_decode_kernel's policy F (gtnb_meta.h) is BeamNoLm for gtnb_beam_decode_async, BeamLm or BeamLex;
 *   BeamSlots<F> holds its per-slot state and the operations the frame loop and the epilogue call (BeamNoLm's are
 *   empty, its key the acoustic score), BeamSmem<F> carves the shared memory for the kernel and sizes it for the
 *   host, and beam_finish ranks every policy's final scores the same way.
 * - Fusion and pruning (gtnb_beam_decode_lm_async).  Policy BeamLm: each slot also carries its LM
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
 * - Streaming (gtnb_beam_decode_chunk_async).  beam_chunk_kernel runs the same body, beam_search, under BeamChunk:
 *   a row's live slots and control words are restored from its state block in global memory (or, at its first frame,
 *   the one-shot init runs), its chunk's frames run at their absolute frame numbers, and the state is saved again;
 *   on END the one-shot epilogue runs at the frames consumed.  The arrays saved are the ones BeamSmem<F>::each lists.
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

/* the same for beam s of the state arrays, read only past the blank test (BeamNoLm's form: the fused policies read
 * the slot anyway, and each form is the one that keeps its kernel's registers down) */
__device__ __forceinline__ float beam_ext_am(int kind, int blank, int C, const float* er, const float* wp,
                                             const float* __restrict__ wt, const float* pb, const float* pl,
                                             const float* tot, const int* last, int s, int c) {
  if (kind != GTNB_DENSE_ASG && c == blank) return neg_inf();
  return beam_ext_am(kind, blank, C, er, wp, wt, pb[s], pl[s], tot[s], last[s], c);
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

/* carves a CTA's dynamic shared memory front to back; on the host a NULL base only counts the bytes (int: at most
 * kMaxDynamicSmem) */
struct BeamCarve {
  char* base;
  int bytes = 0;
  template <class T>
  __host__ __device__ T* take(int n) {
#ifdef __CUDA_ARCH__
    T* p = reinterpret_cast<T*>(base + bytes);
#else
    T* p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
#endif
    bytes += (int)sizeof(T) * n;
    return p;
  }
};

/* a state array as 32-bit words, for the streaming decoder's save and restore */
template <class T>
__host__ __device__ uint32_t* beam_words(T* p) {
  return reinterpret_cast<uint32_t*>(p);
}

/*
 * A policy's per-slot state in shared memory ([2][K] arrays, indexed by buffer * K + slot) and the operations
 * beam_decode_kernel calls: each (visits every per-slot array as (32-bit words, words per slot): what a streaming
 * decoder saves between chunks), init (the root slot when root, and the tables the frames read), key (of a kept or merged candidate whose
 * acoustic score is am), ext_key (of extension (m, c) whose acoustic score is am, -inf when the policy forbids it),
 * keep (slot o carries slot m), extend (slot o is extension (m, c)), final (the final score of slot m, after the last
 * frame), hyp (a hypothesis's own outputs, m -1 for none) and words (the lexicon's word read-off).
 */
template <class F>
struct BeamSlots;

/* BeamNoLm: no state; the key is the acoustic score */
template <>
struct BeamSlots<BeamNoLm> {
  __host__ __device__ void carve(BeamCarve&, int, int) {}
  template <class Op>
  __host__ __device__ void each(Op&&) const {}
  __device__ void init(const BeamNoLm&, int, int, bool) const {}
  __device__ float key(const BeamNoLm&, float am, int, int) const { return am; }
  __device__ float ext_key(const BeamNoLm&, float am, int, int, int, int) const { return am; }
  __device__ void keep(int, int) const {}
  __device__ void extend(const BeamNoLm&, int, int, int, int) const {}
  __device__ float final(const BeamNoLm&, int, float am, int, int) const { return am; }
  __device__ void hyp(const BeamNoLm&, long long, int, float) const {}
  __device__ void words(const BeamNoLm&, int, int, int, int, const int*, const int*, int, const int32_t*) const {}
};

/* BeamLm: the LM node and lmacc (the unweighted sum of the slot's resolved LM weights); the key is
 * am + (lw * lmacc + tb * len) */
template <>
struct BeamSlots<BeamLm> {
  int* node;
  float* lm;
  __host__ __device__ void carve(BeamCarve& m, int K, int) {
    node = m.take<int>(2 * K);
    lm = m.take<float>(2 * K);
  }
  template <class Op>
  __host__ __device__ void each(Op&& op) const {
    op(beam_words(node), 1);
    op(beam_words(lm), 1);
  }
  __device__ void init(const BeamLm& f, int tid, int, bool root) const {
    if (root && tid == 0) {
      node[0] = f.lmw ? f.start : 0;
      lm[0] = 0.0f;
    }
  }
  __device__ float key(const BeamLm& f, float am, int m, int len) const { return beam_fuse(f, am, lm[m], len); }
  __device__ float ext_key(const BeamLm& f, float v, int m, int c, int len, int C) const {
    if (v > neg_inf() && f.lmw) {
      const float w = __ldg(f.lmw + (long long)node[m] * (C + 1) + c); // (one row per beam, via the L2)
      v = w == neg_inf() ? w : beam_fuse(f, v, lm[m] + w, len + 1);
    } else if (v > neg_inf()) {
      v = beam_fuse(f, v, lm[m], len + 1);
    }
    return v;
  }
  __device__ void keep(int o, int m) const {
    node[o] = node[m];
    lm[o] = lm[m];
  }
  __device__ void extend(const BeamLm& f, int o, int m, int c, int C) const {
    const long long at = (long long)node[m] * (C + 1) + c;
    node[o] = f.lmw ? __ldg(f.lmd + at) : 0;
    lm[o] = f.lmw ? lm[m] + __ldg(f.lmw + at) : lm[m];
  }
  /* adds the end weight to lmacc (a beam whose end weight is -inf is dropped) */
  __device__ float final(const BeamLm& f, int m, float am, int len, int C) const {
    const float we = f.lmw ? __ldg(f.lmw + (long long)node[m] * (C + 1) + C) : 0.0f;
    lm[m] = lm[m] + we;
    return we == neg_inf() ? neg_inf() : beam_fuse(f, am, lm[m], len);
  }
  __device__ void hyp(const BeamLm& f, long long o, int m, float am) const {
    if (f.am) f.am[o] = am;
    if (f.lm) f.lm[o] = m >= 0 ? lm[m] : neg_inf();
  }
  __device__ void words(const BeamLm&, int, int, int, int, const int*, const int*, int, const int32_t*) const {}
};

/* BeamLex: the word LM's node and lmacc, and the trie node, word count, word id of the trie node (or -1), at a word
 * end the completion's weight w(LM node, word id) and LM destination, first child, smear and child mask [2][K][MW]
 * of each slot; the root's child mask [MW], the smear of the root's child labelled c [C] and the token classes [C].
 * The key is am + (lw * (lmacc + smear) + tb * words) */
template <>
struct BeamSlots<BeamLex> {
  int* node;
  float* lm;
  int *trie, *wn, *wd; // (the root is trie node 0, its children 1, 2, ... in token order)
  float* cw;
  int *cd, *fc;
  float* sm;
  uint32_t *mask, *rmask;
  float* rsm;
  int* cls;
  int MW;
  __host__ __device__ void carve(BeamCarve& m, int K, int C) {
    MW = (C + 31) / 32;
    node = m.take<int>(2 * K);
    lm = m.take<float>(2 * K);
    trie = m.take<int>(2 * K);
    wn = m.take<int>(2 * K);
    wd = m.take<int>(2 * K);
    cw = m.take<float>(2 * K);
    cd = m.take<int>(2 * K);
    fc = m.take<int>(2 * K);
    sm = m.take<float>(2 * K);
    mask = m.take<uint32_t>(2 * K * MW);
    rmask = m.take<uint32_t>(MW);
    rsm = m.take<float>(C);
    cls = m.take<int>(C);
  }
  template <class Op>
  __host__ __device__ void each(Op&& op) const {
    op(beam_words(node), 1);
    op(beam_words(lm), 1);
    op(beam_words(trie), 1);
    op(beam_words(wn), 1);
    op(beam_words(wd), 1);
    op(beam_words(cw), 1);
    op(beam_words(cd), 1);
    op(beam_words(fc), 1);
    op(beam_words(sm), 1);
    op(mask, MW);
  }
  __device__ void init(const BeamLex& f, int tid, int C, bool root) const {
    if (root && tid == 0) {
      node[0] = f.start;
      lm[0] = 0.0f;
      trie[0] = wn[0] = cd[0] = 0;
      wd[0] = -1;
      cw[0] = sm[0] = 0.0f;
      fc[0] = __ldg(f.first);
    }
    if (tid < MW) {
      const uint32_t v = __ldg(f.mask + tid);
      rmask[tid] = v;
      if (root) mask[tid] = v;
    }
    if (tid < C) {
      cls[tid] = __ldg(f.cls + tid);
      rsm[tid] = lex_has(f.mask, tid) ? __ldg(f.smear + 1 + lex_rank(f.mask, tid)) : 0.0f;
    }
  }
  __device__ float key(const BeamLex& f, float am, int m, int) const {
    return beam_lex_fuse(f, am, lm[m], sm[m], wn[m]);
  }
  /* admission is a bit test; an in-word child's smear is one row per beam, via the L2 */
  __device__ float ext_key(const BeamLex& f, float v, int m, int c, int, int) const {
    if (v > neg_inf()) {
      bool done;
      const int k = cls[c];
      const int ch = lex_move(k, c, trie[m], wd[m], fc[m], mask + m * MW, rmask, 1, done);
      if (ch < 0 || (done && !(cw[m] > neg_inf()))) {
        v = neg_inf();
      } else {
        const float s = k == 0 ? __ldg(f.smear + ch) : k == 2 ? rsm[c] : 0.0f;
        v = beam_lex_fuse(f, v, done ? __fadd_rn(lm[m], cw[m]) : lm[m], s, wn[m] + (int)done);
      }
    }
    return v;
  }
  __device__ void keep(int o, int m) const {
    node[o] = node[m];
    lm[o] = lm[m];
    trie[o] = trie[m];
    wn[o] = wn[m];
    wd[o] = wd[m];
    cw[o] = cw[m];
    cd[o] = cd[m];
    fc[o] = fc[m];
    sm[o] = sm[m];
    for (int w = 0; w < MW; w++) mask[o * MW + w] = mask[m * MW + w];
  }
  /* the new slot's trie node and LM state; on a word end, the completion's weight and destination are looked up
   * here, once, so that no LM lookup sits on the per-candidate path */
  __device__ void extend(const BeamLex& f, int o, int m, int c, int) const {
    bool done;
    const int ch = lex_move(cls[c], c, trie[m], wd[m], fc[m], mask + m * MW, rmask, 1, done);
    const int ln = done ? cd[m] : node[m];
    node[o] = ln;
    lm[o] = done ? __fadd_rn(lm[m], cw[m]) : lm[m];
    wn[o] = wn[m] + (int)done;
    trie[o] = ch;
    const int w = __ldg(f.word + ch);
    wd[o] = w;
    fc[o] = __ldg(f.first + ch);
    sm[o] = __ldg(f.smear + ch);
    for (int i = 0; i < MW; i++) mask[o * MW + i] = __ldg(f.mask + (long long)ch * MW + i);
    int d = 0;
    cw[o] = w >= 0 ? lex_resolve(f, ln, w, d) : 0.0f;
    cd[o] = d;
  }
  /* completes the pending word at a word end (a slot inside a word is dropped), then adds the end weight (dropped at
   * -inf) */
  __device__ float final(const BeamLex& f, int m, float am, int, int) const {
    float l = lm[m];
    int n = node[m], nw = wn[m];
    bool ok = true;
    if (trie[m] != 0) {
      ok = wd[m] >= 0 && cw[m] > neg_inf();
      l = __fadd_rn(l, cw[m]);
      n = cd[m];
      nw++;
    }
    const float we = ok ? (f.endw ? __ldg(f.endw + n) : 0.0f) : neg_inf();
    l = __fadd_rn(l, we);
    lm[m] = l;
    wn[m] = nw;
    return we == neg_inf() ? neg_inf() : beam_fuse(f, am, l, nw);
  }
  __device__ void hyp(const BeamLex& f, long long o, int m, float am) const {
    if (f.am) f.am[o] = am;
    if (f.lm) f.lm[o] = m >= 0 ? lm[m] : neg_inf();
    if (f.counts) f.counts[o] = m >= 0 ? wn[m] : -1;
  }
  /* each hypothesis's word ids, read off its traced tokens (out, of this thread's hypotheses) by walking the trie,
   * then -1; slot m0 + rank[n] holds hypothesis n < live, len its token count */
  __device__ void words(const BeamLex& f, int b, int T, int N, int live, const int* rank, const int* len, int m0,
                        const int32_t* out) const {
    if (!f.words) return;
    int32_t* wout = f.words + (long long)b * N * T;
    for (int n = threadIdx.x; n < live && n < N; n += kBeamThreads) {
      const int m = m0 + rank[n]; // (the transcript was admitted: every move exists)
      int node = 0, k = 0;
      for (int p = 0; p < len[m]; p++) {
        const int c = out[(long long)n * T + p], cl = cls[c];
        if (cl != 0 && node != 0) wout[(long long)n * T + k++] = __ldg(f.word + node);
        if (cl == 1) {
          node = 0;
        } else {
          const int from = cl == 0 ? node : 0;
          node = __ldg(f.first + from) + lex_rank(f.mask + (long long)from * MW, c);
        }
      }
      if (node != 0) wout[(long long)n * T + k++] = __ldg(f.word + node);
    }
    for (long long p = threadIdx.x; p < (long long)N * T; p += kBeamThreads) {
      const int n = (int)(p / T);
      if (p - (long long)n * T >= (n < live ? wn[m0 + rank[n]] : 0)) wout[p] = -1;
    }
  }
};

/*
 * The dynamic shared memory of one CTA, one carve for the kernel and for the host's size: two hash arrays [2][K] of
 * 8 bytes, then 4-byte words (control block, histogram, two emission rows, the two start-weight rows, the double-
 * buffered state, the candidates' scratch and keys); with token pruning (F::on) the frame's tokens and token ->
 * position map and per-warp counts; then the policy's BeamSlots.
 */
template <class F>
struct BeamSmem {
  uint64_t *hh, *hq; // [2][K] hash of the transcript, and of the transcript minus its last token
  int *ctl, *hist; // [16] control block, [256] histogram
  float* erow; // [2][C]
  float *w0, *wb; // [C] weight of a token entered from p_blank at frame 0 (BIGRAM sigma, ASG start), at frames >= 1
                  // (BIGRAM W[c][blank])
  float *spb, *spl, *stot; // [2][K] p_blank, p_label, logsumexp(p_blank, p_label)
  int *slen, *slast, *spar; // [2][K] length, last token (-1: the empty transcript), the slot holding the transcript
                            // minus its last token (or -1)
  float *kpb, *kpl; // [K] kept candidates' states
  int *kslot, *src, *widx; // [K] old slot -> its kept beam's new slot (or -1); new slot -> candidate; winners:
                           // candidate
  uint32_t *wkey, *keys; // [K] winners: key; [K + K*P]: kept beams r at r, extension (s, p) at L + s*P + p
  int *ptok, *ppos, *wcnt; // (F::on) [P] the frame's tokens, ascending; [C] token -> position in ptok, or -1; [8]
                           // selected tokens per warp
  BeamSlots<F> x;
  int bytes;
  __host__ __device__ BeamSmem(char* base, int K, int C) {
    BeamCarve m{base};
    hh = m.take<uint64_t>(2 * K);
    hq = m.take<uint64_t>(2 * K);
    ctl = m.take<int>(16);
    hist = m.take<int>(256);
    erow = m.take<float>(2 * C);
    w0 = m.take<float>(C);
    wb = m.take<float>(C);
    spb = m.take<float>(2 * K);
    spl = m.take<float>(2 * K);
    stot = m.take<float>(2 * K);
    slen = m.take<int>(2 * K);
    slast = m.take<int>(2 * K);
    spar = m.take<int>(2 * K);
    kpb = m.take<float>(K);
    kpl = m.take<float>(K);
    kslot = m.take<int>(K);
    src = m.take<int>(K);
    widx = m.take<int>(K);
    wkey = m.take<uint32_t>(K);
    keys = m.take<uint32_t>(K + K * C);
    ptok = ppos = wcnt = nullptr;
    if (F::on) {
      ptok = m.take<int>(C);
      ppos = m.take<int>(C);
      wcnt = m.take<int>(8);
    }
    x.carve(m, K, C);
    bytes = m.bytes;
  }
  /* every per-slot array of the search, the policy's last: a streaming decoder's state between chunks */
  template <class Op>
  __host__ __device__ void each(Op&& op) const {
    op(beam_words(hh), 2);
    op(beam_words(hq), 2);
    op(beam_words(spb), 1);
    op(beam_words(spl), 1);
    op(beam_words(stot), 1);
    op(beam_words(slen), 1);
    op(beam_words(slast), 1);
    op(beam_words(spar), 1);
    x.each(op);
  }
};

/*
 * The streaming decoder's state block of a row (32-bit words): a header, then each array BeamSmem<F>::each visits, as
 * [K][words per slot] (its live slots, the first kBcL, are what a resumed search reads).  Header: frames consumed since
 * the utterance began, the sticky invalid flag (status 2), and the control words kBcL, kBcTieAny and kBcBad.
 */
enum { kStT = 0, kStInv, kStL, kStTie, kStBad, kStHeader = 8 };
template <class F>
__host__ __device__ long long beam_state_words(int K, int C) {
  long long w = kStHeader;
  BeamSmem<F>(nullptr, K, C).each([&](uint32_t*, int per) { w += (long long)K * per; });
  return w;
}

/* status 1 or 2: NaN scores, -1 lengths and rows in every output of the policy */
template <class F>
__device__ void beam_flag(int b, int T, int N, int code, int32_t* tokens, int32_t* lengths, float* scores,
                          int32_t* status, const F& f) {
  const int tid = threadIdx.x;
  for (long long p = tid; p < (long long)N * T; p += kBeamThreads) {
    tokens[(long long)b * N * T + p] = -1;
    if (f.words) f.words[(long long)b * N * T + p] = -1;
  }
  for (int n = tid; n < N; n += kBeamThreads) {
    const long long o = (long long)b * N + n;
    scores[o] = CUDART_NAN_F;
    lengths[o] = -1;
    if (f.am) f.am[o] = CUDART_NAN_F;
    if (f.lm) f.lm[o] = CUDART_NAN_F;
    if (f.counts) f.counts[o] = -1;
  }
  if (tid == 0 && status) status[b] = code;
}

/*
 * After frame T_b - 1: each live slot's final score from the policy (dropped at -inf), and the N-best are the top
 * live beams by it, ties to the lower slot (the search's own order).  fin ([K]) holds each slot's final score, rank
 * ([K]) rank -> slot.  For BeamNoLm this is the slots' own order, exactly: they are ranked by (key, candidate order)
 * and the key is order-preserving on stot, so ranking by stot with ties to the lower slot is the identity, no slot is
 * dropped, and the tie check compares what the search compared.
 */
template <class F>
__device__ void beam_finish(int b, int T, int Tb, int C, int K, int N, const uint16_t* bpu, int cur, const int* ctl,
                            const float* stot, const int* slen, const BeamSlots<F>& x, float* fin, int* rank,
                            int32_t* tokens, int32_t* lengths, float* scores, int32_t* status, const F& f) {
  const int tid = threadIdx.x;
  const int L = ctl[kBcL];
  const int m0 = cur * K;
  if (tid < L) fin[tid] = x.final(f, m0 + tid, stot[m0 + tid], slen[m0 + tid], C);
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
    const int r = n < live ? rank[n] : -1;
    const int len = r >= 0 ? slen[m0 + r] : -1;
    const long long o = (long long)b * N + n;
    scores[o] = r >= 0 ? fin[r] : neg_inf();
    x.hyp(f, o, r >= 0 ? m0 + r : -1, r >= 0 ? stot[m0 + r] : neg_inf());
    lengths[o] = len;
    int tt = Tb - 1, s = r;
    for (int p = len - 1; p >= 0; p--) out[(long long)n * T + p] = beam_back(bpu, K, tt, s);
  }
  for (long long p = tid; p < (long long)N * T; p += kBeamThreads) {
    const int n = (int)(p / T);
    if (p - (long long)n * T >= (n < live ? slen[m0 + rank[n]] : 0)) out[p] = -1;
  }
  x.words(f, b, T, N, live, rank, slen, m0, out);
  if (tid == 0) {
    bool tied = ctl[kBcTieAny] != 0;
    for (int n = 0; n + 1 < live && n < N; n++) tied |= fin[rank[n]] == fin[rank[n + 1]];
    if (status) status[b] = tied ? 3 : 0;
  }
}

/* the one-shot search: every row from frame 0 to its input length, nothing kept */
struct BeamOnce {
  static constexpr bool on = false;
};

/*
 * The search of utterance b, one CTA of kBeamThreads (beam_decode_kernel, beam_chunk_kernel).  emissions [B][T][C]
 * of E; input_lens [B] (nullable: T); kind GTNB_DENSE_CTC / _BIGRAM / _ASG; wt [C][C] (transposed W), wfirst [C]
 * (BIGRAM sigma, ASG start weights) and wbad [C] from beam_weights_kernel (unused for CTC); blank (CTC, BIGRAM); K
 * beams, N hypotheses.  bp: [B][T][K] back-pointers (scratch).  Out: tokens [B][N][T], lengths [B][N], scores [B][N],
 * status [B] (nullable), and the policy's own outputs.  F: the policy (BeamNoLm, BeamLm, BeamLex).
 * R: BeamOnce, or BeamChunk (gtnb_meta.h): a chunk of a streaming decoder.  Then T is T_max, emissions are [B][Tc][C]
 * and input_lens is unused: the row's saved state is restored (or, at its first frame, the search starts as the
 * one-shot one does), its chunk_lens[b] frames run at their absolute frame numbers, and the state is saved again, or
 * on END the one-shot epilogue runs at the frames consumed and the row restarts.
 */
template <class E, class Hash, class F, class R>
__device__ __forceinline__ void beam_search(const E* __restrict__ emissions, int T, int C,
                                            const int32_t* __restrict__ input_lens, int kind,
                                            const float* __restrict__ wt, const float* __restrict__ wfirst,
                                            const int32_t* __restrict__ wbad, int blank, int K, int N, uint16_t* bp,
                                            int32_t* __restrict__ tokens, int32_t* __restrict__ lengths,
                                            float* __restrict__ scores, int32_t* __restrict__ status, const F& fz,
                                            const R& rz) {
  GTNB_DYNAMIC_SMEM(uint64_t, hsm);
  const BeamSmem<F> sm(reinterpret_cast<char*>(hsm), K, C);
  uint64_t *hh = sm.hh, *hq = sm.hq;
  int *ctl = sm.ctl, *hist = sm.hist;
  float *erow = sm.erow, *w0 = sm.w0, *wb = sm.wb, *spb = sm.spb, *spl = sm.spl, *stot = sm.stot;
  int *slen = sm.slen, *slast = sm.slast, *spar = sm.spar;
  float *kpb = sm.kpb, *kpl = sm.kpl;
  int *kslot = sm.kslot, *src = sm.src, *widx = sm.widx;
  uint32_t *wkey = sm.wkey, *keys = sm.keys;
  int *ptok = sm.ptok, *ppos = sm.ppos, *wcnt = sm.wcnt;
  const BeamSlots<F>& xs = sm.x;
  const int P = F::on ? fz.P : C;

  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // frames [t0, Tb) run; em: frame t0's row
  int t0 = 0, Tb;
  bool fresh = true, end = false, inv = false;
  uint32_t* st = nullptr;
  if constexpr (R::on) {
    st = rz.state + (long long)b * rz.words;
    const int bits = rz.control ? rz.control[b] : 0;
    const int n = rz.lens ? rz.lens[b] : rz.Tc;
    if (n == 0 && bits == 0) return; // (the row is left as it is)
    const bool reset = (bits & GTNB_BEAM_RESET) != 0;
    end = (bits & GTNB_BEAM_END) != 0;
    t0 = reset ? 0 : (int)st[kStT];
    inv = !reset && st[kStInv] != 0;
    if (!(n >= 0 && n <= rz.Tc) || n > T - t0) inv = true;
    Tb = inv ? t0 : t0 + n;
    fresh = t0 == 0;
  } else {
    Tb = input_lens ? input_lens[b] : T;
    if (!(Tb >= 0 && Tb <= T)) {
      beam_flag(b, T, N, 2, tokens, lengths, scores, status, fz);
      return;
    }
  }
  int Te = T; // frames per row of emissions
  if constexpr (R::on) Te = rz.Tc;
  const E* em = emissions + (long long)b * Te * C;
  uint16_t* bpu = bp + (long long)b * T * K;
  if (tid < 16) {
    int v = 0;
    if constexpr (R::on)
      if (!fresh) v = tid == kBcL ? st[kStL] : tid == kBcTieAny ? st[kStTie] : tid == kBcBad ? st[kStBad] : 0;
    ctl[tid] = v;
  }
  for (int i = tid; i < 256; i += kBeamThreads) hist[i] = 0;
  if constexpr (R::on) {
    if (!fresh) { // the live slots into buffer 0
      const int L = (int)st[kStL];
      long long off = kStHeader;
      sm.each([&](uint32_t* a, int per) {
        for (int i = tid; i < L * per; i += kBeamThreads) a[i] = st[off + i];
        off += (long long)K * per;
      });
    }
  }
  if (fresh && tid == 0) {
    ctl[kBcL] = 1;
    spb[0] = 0.0f;
    spl[0] = neg_inf();
    stot[0] = 0.0f;
    slen[0] = 0;
    slast[0] = -1;
    spar[0] = -1;
    hh[0] = hq[0] = 0;
  }
  if constexpr (F::on) {
    if (tid < C) { // (every frame's selection when P < C)
      ptok[tid] = tid;
      ppos[tid] = tid;
    }
  }
  xs.init(fz, tid, C, fresh);
  __syncthreads();
  if (tid < C) {
    w0[tid] = kind == GTNB_DENSE_CTC ? 0.0f : wfirst[tid];
    wb[tid] = kind == GTNB_DENSE_BIGRAM ? wt[(long long)blank * C + tid] : 0.0f;
    if (Tb > t0) {
      const float v = ldg_elem(em + tid);
      erow[tid] = v;
      if (v != v || v == CUDART_INF_F || (kind != GTNB_DENSE_CTC && t0 == 0 && wbad[tid])) ctl[kBcBad] = 1;
    }
  }
  __syncthreads();

  int cur = 0;
  for (int t = t0; t < Tb; t++) {
    if (ctl[kBcBad]) break;
    const int L = ctl[kBcL];
    const float* er = erow + ((t - t0) & 1) * C;
    const bool pf = t + 1 < Tb && tid < C;
    const float ahead = pf ? ldg_elem(em + (long long)(t + 1 - t0) * C + tid) : 0.0f;
    const float* wp = t == 0 ? w0 : wb;
    const float *pb0 = spb + cur * K, *pl0 = spl + cur * K, *tot0 = stot + cur * K;
    const int *len0 = slen + cur * K, *last0 = slast + cur * K, *par0 = spar + cur * K;

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
      keys[tid] = beam_key(xs.key(fz, beam_lse2(nb, nl), cur * K + tid, len0[tid]));
      kslot[tid] = -1;
    }
    if (tid == 0) ctl[kBcNwin] = ctl[kBcDone] = 0;
    const int next = L * P;
    {
      int s = tid / P, p = tid - s * P;
      for (int q = tid; q < next; q += kBeamThreads) {
        const int c = F::on ? ptok[p] : p;
        const float am = F::on ? beam_ext_am(kind, blank, C, er, wp, wt, pb0[s], pl0[s], tot0[s], last0[s], c)
                               : beam_ext_am(kind, blank, C, er, wp, wt, pb0, pl0, tot0, last0, s, c);
        keys[L + q] = beam_key(xs.ext_key(fz, am, cur * K + s, c, len0[s], C));
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
      const int s = par0[tid];
      // (BeamNoLm: the key is the acoustic score; otherwise it holds the fused one: the acoustic one again)
      const float v = !F::on ? beam_key_float(keys[q])
                      : keys[q] ? beam_ext_am(kind, blank, C, er, wp, wt, pb0[s], pl0[s], tot0[s], last0[s], last0[tid])
                                : neg_inf();
      keys[q] = 0u;
      kpl[tid] = beam_lse2(kpl[tid], v);
      keys[tid] = beam_key(xs.key(fz, beam_lse2(kpb[tid], kpl[tid]), cur * K + tid, len0[tid]));
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
      float am; // (BeamNoLm: the key; otherwise it holds the fused score: the acoustic one again)
      if (j < L) {
        spb[nx * K + n] = kpb[j];
        spl[nx * K + n] = kpl[j];
        slen[nx * K + n] = len0[j];
        slast[nx * K + n] = last0[j];
        hh[nx * K + n] = hh[cur * K + j];
        hq[nx * K + n] = hq[cur * K + j];
        am = F::on ? beam_lse2(kpb[j], kpl[j]) : beam_key_float(k);
        xs.keep(nx * K + n, cur * K + j);
        kslot[j] = n;
        code = (uint32_t)j << 9;
      } else {
        const int s = (j - L) / P, p = j - L - s * P;
        const int c = F::on ? ptok[p] : p;
        am = F::on ? beam_ext_am(kind, blank, C, er, wp, wt, pb0[s], pl0[s], tot0[s], last0[s], c)
                   : beam_key_float(k);
        xs.extend(fz, nx * K + n, cur * K + s, c, C);
        spb[nx * K + n] = neg_inf();
        spl[nx * K + n] = am;
        slen[nx * K + n] = len0[s] + 1;
        slast[nx * K + n] = c;
        hh[nx * K + n] = Hash::combine(hh[cur * K + s], c);
        hq[nx * K + n] = hh[cur * K + s];
        code = ((uint32_t)s << 9) | 256u | (uint32_t)c;
      }
      stot[nx * K + n] = am;
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
      erow[((t + 1 - t0) & 1) * C + tid] = ahead;
      if (ahead != ahead || ahead == CUDART_INF_F) ctl[kBcBad] = 1;
    }
    if (tid == 0) ctl[kBcL] = nw;
    cur = nx;
    __syncthreads();
  }

  if constexpr (R::on) {
    const int L = ctl[kBcL];
    const bool bad = ctl[kBcBad] != 0;
    if (rz.best_tokens) { // slot 0: the best key, in the search's tie order
      const int m0 = cur * K;
      const int len = inv || bad || L == 0 ? -1 : slen[m0];
      int32_t* out = rz.best_tokens + (long long)b * T;
      if (tid == 0) {
        rz.best_lengths[b] = len;
        rz.best_scores[b] = inv || bad ? CUDART_NAN_F : L == 0 ? neg_inf() : xs.key(fz, stot[m0], m0, len);
        int tt = Tb - 1, s = 0;
        for (int p = len - 1; p >= 0; p--) out[p] = beam_back(bpu, K, tt, s);
      }
      for (int p = tid; p < T; p += kBeamThreads)
        if (p >= len) out[p] = -1;
      __syncthreads(); // (the epilogue's final scores change the policy's state)
    }
    if (end) {
      if (inv || bad)
        beam_flag(b, T, N, inv ? 2 : 1, tokens, lengths, scores, status, fz);
      else
        beam_finish(b, T, Tb, C, K, N, bpu, cur, ctl, stot, slen, xs, kpb, src, tokens, lengths, scores, status,
                    fz);
      if (tid == 0) st[kStT] = st[kStInv] = 0;
      return;
    }
    long long off = kStHeader;
    sm.each([&](uint32_t* a, int per) {
      for (int i = tid; i < L * per; i += kBeamThreads) st[off + i] = a[(long long)cur * K * per + i];
      off += (long long)K * per;
    });
    if (tid == 0) {
      st[kStT] = (uint32_t)Tb;
      st[kStInv] = inv;
      st[kStL] = (uint32_t)L;
      st[kStTie] = (uint32_t)ctl[kBcTieAny];
      st[kStBad] = bad;
    }
  } else {
    if (ctl[kBcBad]) {
      beam_flag(b, T, N, 1, tokens, lengths, scores, status, fz);
      return;
    }
    beam_finish(b, T, Tb, C, K, N, bpu, cur, ctl, stot, slen, xs, kpb, src, tokens, lengths, scores, status, fz);
  }
}

/* the one-shot search (gtnb_beam_decode_async, _lm_async, _lexicon_async) */
template <class E, class Hash, class F = BeamNoLm>
__global__ void __launch_bounds__(kBeamThreads) beam_decode_kernel(
    const E* __restrict__ emissions, int T, int C, const int32_t* __restrict__ input_lens, int kind,
    const float* __restrict__ wt, const float* __restrict__ wfirst, const int32_t* __restrict__ wbad, int blank, int K,
    int N, uint16_t* bp, int32_t* __restrict__ tokens, int32_t* __restrict__ lengths, float* __restrict__ scores,
    int32_t* __restrict__ status, const F fz = F()) {
  beam_search<E, Hash, F>(emissions, T, C, input_lens, kind, wt, wfirst, wbad, blank, K, N, bp, tokens, lengths,
                          scores, status, fz, BeamOnce());
}

/* one chunk of the streaming decoder (gtnb_beam_decode_chunk_async): T = T_max, emissions [B][rz.Tc][C] */
template <class E, class Hash, class F>
__global__ void __launch_bounds__(kBeamThreads) beam_chunk_kernel(
    const E* __restrict__ emissions, int T, int C, int kind, const float* __restrict__ wt,
    const float* __restrict__ wfirst, const int32_t* __restrict__ wbad, int blank, int K, int N, uint16_t* bp,
    int32_t* __restrict__ tokens, int32_t* __restrict__ lengths, float* __restrict__ scores,
    int32_t* __restrict__ status, const F fz, const BeamChunk rz) {
  beam_search<E, Hash, F>(emissions, T, C, nullptr, kind, wt, wfirst, wbad, blank, K, N, bp, tokens, lengths, scores,
                          status, fz, rz);
}

/* the dynamic shared memory of beam_decode_kernel<E, Hash, F> at K beams and C tokens; the by-policy names are the
 * same carve, for callers that size one policy's launch (the per-policy emulation drivers) */
template <class F = BeamNoLm>
long long beam_smem_bytes(int K, int C) {
  return BeamSmem<F>(nullptr, K, C).bytes;
}
inline long long beam_lm_smem_bytes(int K, int C) { return beam_smem_bytes<BeamLm>(K, C); }
inline long long beam_lex_smem_bytes(int K, int C) { return beam_smem_bytes<BeamLex>(K, C); }

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

template <class F>
int launch_beam_decode(gtnb_ctx* ctx, int B, int T, int C, const void* emissions, int dtype,
                       const int32_t* input_lens, int kind, const float* wt, const float* wfirst, const int32_t* wbad,
                       int blank, int K, int N, uint16_t* bp, int32_t* tokens, int32_t* lengths, float* scores,
                       int32_t* status, const F& f) {
  if (B <= 0) return GTNB_OK;
  const long long smem = beam_smem_bytes<F>(K, C);
  // (the names the per-kernel profile reports)
  const char* name = std::is_same_v<F, BeamLex> ? "beam_decode_lexicon" : F::on ? "beam_decode_lm" : "beam_decode";
  const auto run = [&](const auto* e) {
    using E = std::remove_const_t<std::remove_pointer_t<decltype(e)>>;
    if (smem > 48 * 1024)
      if (const int rc = ensure_max_smem(ctx, (const void*)beam_decode_kernel<E, BeamHash, F>)) return rc;
    GTNB_LAUNCH(ctx, name,
                beam_decode_kernel<E, BeamHash, F><<<B, kBeamThreads, smem, ctx->stream>>>(
                    e, T, C, input_lens, kind, wt, wfirst, wbad, blank, K, N, bp, tokens, lengths, scores, status, f));
    return (int)GTNB_OK;
  };
  if (dtype == GTNB_BF16) return run(static_cast<const bf16_t*>(emissions));
  if (dtype == GTNB_F16) return run(static_cast<const f16_t*>(emissions));
  return run(static_cast<const float*>(emissions));
}
#define GTNB_BEAM_POLICY(F_)                                                                                     \
  template int launch_beam_decode<F_>(gtnb_ctx*, int, int, int, const void*, int, const int32_t*, int,          \
                                      const float*, const float*, const int32_t*, int, int, int, uint16_t*,       \
                                      int32_t*, int32_t*, float*, int32_t*, const F_&);
GTNB_BEAM_POLICY(BeamNoLm)
GTNB_BEAM_POLICY(BeamLm)
GTNB_BEAM_POLICY(BeamLex)
#undef GTNB_BEAM_POLICY

long long beam_state_row_words(bool lexicon, int K, int C) {
  return lexicon ? beam_state_words<BeamLex>(K, C) : beam_state_words<BeamLm>(K, C);
}

template <class F>
int launch_beam_chunk(gtnb_ctx* ctx, int B, int T, int C, const void* emissions, int dtype, int kind,
                      const float* wt, const float* wfirst, const int32_t* wbad, int blank, int K, int N, uint16_t* bp,
                      int32_t* tokens, int32_t* lengths, float* scores, int32_t* status, const F& f,
                      const BeamChunk& r) {
  if (B <= 0) return GTNB_OK;
  const long long smem = beam_smem_bytes<F>(K, C);
  const char* name = std::is_same_v<F, BeamLex> ? "beam_chunk_lexicon" : "beam_chunk_lm";
  const auto run = [&](const auto* e) {
    using E = std::remove_const_t<std::remove_pointer_t<decltype(e)>>;
    if (smem > 48 * 1024)
      if (const int rc = ensure_max_smem(ctx, (const void*)beam_chunk_kernel<E, BeamHash, F>)) return rc;
    GTNB_LAUNCH(ctx, name,
                beam_chunk_kernel<E, BeamHash, F><<<B, kBeamThreads, smem, ctx->stream>>>(
                    e, T, C, kind, wt, wfirst, wbad, blank, K, N, bp, tokens, lengths, scores, status, f, r));
    return (int)GTNB_OK;
  };
  if (dtype == GTNB_BF16) return run(static_cast<const bf16_t*>(emissions));
  if (dtype == GTNB_F16) return run(static_cast<const f16_t*>(emissions));
  return run(static_cast<const float*>(emissions));
}
#define GTNB_BEAM_CHUNK_POLICY(F_)                                                                              \
  template int launch_beam_chunk<F_>(gtnb_ctx*, int, int, int, const void*, int, int, const float*, const float*, \
                                     const int32_t*, int, int, int, uint16_t*, int32_t*, int32_t*, float*,        \
                                     int32_t*, const F_&, const BeamChunk&);
GTNB_BEAM_CHUNK_POLICY(BeamLm)
GTNB_BEAM_CHUNK_POLICY(BeamLex)
#undef GTNB_BEAM_CHUNK_POLICY

#endif // GTNB_HOST_EMU

} // namespace gtnb
