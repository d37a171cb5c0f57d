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

/*
 * One CTA of kBeamThreads per utterance b.  emissions [B][T][C] of E; input_lens [B] (nullable: T); kind
 * GTNB_DENSE_CTC / _BIGRAM / _ASG; wt [C][C] (transposed W), wfirst [C] (BIGRAM sigma, ASG start weights) and wbad
 * [C] from beam_weights_kernel (unused for CTC); blank (CTC, BIGRAM); K beams, N hypotheses.  bp: [B][T][K] back-
 * pointers (scratch).  Out: tokens [B][N][T], lengths [B][N], scores [B][N], status [B] (nullable).
 */
template <class E, class Hash>
__global__ void __launch_bounds__(kBeamThreads) beam_decode_kernel(
    const E* __restrict__ emissions, int T, int C, const int32_t* __restrict__ input_lens, int kind,
    const float* __restrict__ wt, const float* __restrict__ wfirst, const int32_t* __restrict__ wbad, int blank, int K,
    int N, uint16_t* bp, int32_t* __restrict__ tokens, int32_t* __restrict__ lengths, float* __restrict__ scores,
    int32_t* __restrict__ status) {
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
  uint32_t* keys = wkey + K; // [K + K*C]: kept beams r at r, extension (s, c) at L + s*C + c

  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int Tb = input_lens ? input_lens[b] : T;
  if (!(Tb >= 0 && Tb <= T)) {
    beam_flag(b, T, N, 2, tokens, lengths, scores, status);
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
      keys[tid] = beam_key(beam_lse2(nb, nl));
      kslot[tid] = -1;
    }
    if (tid == 0) ctl[kBcNwin] = ctl[kBcDone] = 0;
    const int next = L * C;
    {
      int s = tid / C, c = tid - s * C;
      for (int q = tid; q < next; q += kBeamThreads) {
        float v = neg_inf();
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
        keys[L + q] = beam_key(v);
        c += kBeamThreads;
        while (c >= C) {
          c -= C;
          s++;
        }
      }
    }
    __syncthreads();

    // merge: extension (par[r], last[r]) is r's transcript
    if (tid < L && par0[tid] >= 0) {
      const int q = L + par0[tid] * C + last0[tid];
      const float v = beam_key_float(keys[q]);
      keys[q] = 0u;
      kpl[tid] = beam_lse2(kpl[tid], v);
      keys[tid] = beam_key(beam_lse2(kpb[tid], kpl[tid]));
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
      if (j < L) {
        spb[nx * K + n] = kpb[j];
        spl[nx * K + n] = kpl[j];
        slen[nx * K + n] = len0[j];
        slast[nx * K + n] = last0[j];
        hh[nx * K + n] = hh[cur * K + j];
        hq[nx * K + n] = hq[cur * K + j];
        kslot[j] = n;
        code = (uint32_t)j << 9;
      } else {
        const int s = (j - L) / C, c = j - L - s * C;
        spb[nx * K + n] = neg_inf();
        spl[nx * K + n] = beam_key_float(k);
        slen[nx * K + n] = len0[s] + 1;
        slast[nx * K + n] = c;
        hh[nx * K + n] = Hash::combine(hh[cur * K + s], c);
        hq[nx * K + n] = hh[cur * K + s];
        code = ((uint32_t)s << 9) | 256u | (uint32_t)c;
      }
      stot[nx * K + n] = beam_key_float(k);
      src[n] = j;
      bpu[(long long)t * K + n] = (uint16_t)code;
    }
    __syncthreads();

    // parents in the new frame; a kept beam whose parent was not live looks for it among the new extensions
    if (tid < nw) {
      const int j = src[tid];
      int par = -1;
      if (j >= L) {
        par = kslot[(j - L) / C];
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
      const int rc__ = ensure_max_smem(ctx, (const void*)beam_decode_kernel<E_, BeamHash>);                   \
      if (rc__) return rc__;                                                                                  \
    }                                                                                                         \
    GTNB_LAUNCH(ctx, "beam_decode",                                                                           \
                beam_decode_kernel<E_, BeamHash><<<B, kBeamThreads, smem, ctx->stream>>>(                     \
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

#endif // GTNB_HOST_EMU

} // namespace gtnb
