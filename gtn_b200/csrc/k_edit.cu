/*
 * k_edit.cu -- batched Levenshtein distance between padded hypotheses and references (gtnb_edit_distance_async).
 *
 * The reference scores a transcript as -viterbiScore(compose(x, compose(edits, y))) with `edits` a one-state
 * transducer of substitution, insertion and deletion arcs (examples/edit_distance.cpp).  That composed graph is an
 * (n+1) x (m+1) grid with three arc kinds, so its tropical shortest distance is the textbook recurrence
 *   D[i][j] = min(D[i-1][j-1] + (h_i != r_j), D[i-1][j] + 1 (insertion), D[i][j-1] + 1 (deletion)),
 * run here without materialising the grid.  One CTA per pair:
 * - Units.  Token mode: the tokens.  Word mode (word_sep >= 0): the CTA splits hypothesis and reference, as one
 *   concatenation with a forced boundary between them, into maximal runs of non-separators (ballots and prefix sums),
 *   hashes every word, and gives it the index of the first word with an equal span as its id: a hash filter, then an
 *   exact span compare.  The recurrence then compares ints.
 * - Frame.  The shorter sequence forms the rows, the longer the columns (swap: the rows are the reference, which
 *   turns insertions into vertical and deletions into horizontal moves; the tie rule is applied in the caller's terms).
 * - Wavefront.  Lane s of the CTA owns rows s*K+1 .. s*K+K in registers and processes column j at its warp's step
 *   j - 1 + lane: the strip's bottom cell reaches the next lane through __shfl_up_sync, with no barrier on the chain.
 *   Warp w + 1 receives warp w's bottom row through a shared-memory ring with produced / consumed counters.
 * - Tie rule.  Every cell prefers the diagonal, then a deletion, then an insertion; the substitution and insertion
 *   counts (16 bits each in one int) travel with D along the chosen predecessor, so no backtrace is needed for them.
 * - Alignment (moves != NULL).  Each lane stores its strip's K 2-bit moves per column as one 32-bit word at
 *   [pair][warp][step][lane], so a warp's store at one step is one coalesced 128-byte line; thread 0 traces back.
 */
#include <cstdint>

#include "gtnb_ptx.h"

namespace gtnb {

constexpr int kEditMaxWarps = 8; // 8 warps x 32 lanes x 16 rows: 4096 rows
constexpr int kEditMaxK = 16; // rows per lane: 16 two-bit moves fill the lane's 32-bit move word
constexpr int kEditRing = 64; // columns in flight between two warps (a power of two)
// ints of the kernel's control block at the start of its shared memory (ring, counts, progress, result), kept even
constexpr int kEditCtlInts = 2 * kEditMaxWarps * kEditRing + 5 * kEditMaxWarps + 2;

/* the word hash, a filter only: equal hashes are confirmed by an exact compare of the spans */
struct EditHash {
  __device__ static uint64_t combine(uint64_t h, int32_t tok) {
    h ^= (uint64_t)(uint32_t)tok + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    return h * 0xff51afd7ed558ccdull;
  }
};

/* launch geometry of one call, from the bounds alone: K rows per lane, warps per CTA, the column bound, dynamic
 * shared memory, and the 32-bit move words of one pair (warps x (cols + 31) steps x 32 lanes) */
struct EditPlan {
  int K, warps, cols;
  long long smem_bytes, pair_move_words;
};

inline EditPlan edit_plan(int N, int M, int word_sep) {
  // a word takes at least one token and one separator after it, except the last
  const int un = word_sep >= 0 ? (N + 1) / 2 : N, um = word_sep >= 0 ? (M + 1) / 2 : M;
  const int rows = un < um ? un : um;
  EditPlan p{};
  p.cols = un > um ? un : um;
  p.K = 1;
  while (p.K < kEditMaxK && 32 * p.K < rows) p.K *= 2;
  p.warps = rows > 32 * p.K ? (rows + 32 * p.K - 1) / (32 * p.K) : 1;
  const long long cap = (long long)un + um;
  // control block, tokens; word mode: word start, end, id, then the 8-byte-aligned hashes
  p.smem_bytes = 4ll * (kEditCtlInts + N + M);
  if (word_sep >= 0) p.smem_bytes = (p.smem_bytes + 12 * cap + 7) / 8 * 8 + 8 * cap;
  p.pair_move_words = (long long)p.warps * (p.cols + 31) * 32;
  return p;
}

/* the packed counts (substitutions | insertions << 16) of the frame's first column (row i) and first row (column j) */
__device__ __forceinline__ int edit_first_col(int i, bool swap) { return swap ? 0 : i << 16; }
__device__ __forceinline__ int edit_first_row(int j, bool swap) { return swap ? j << 16 : 0; }

/*
 * One CTA of 32 * warps threads per pair b.  hyp [B][N], ref [B][M] with lengths hyp_lens / ref_lens [B];
 * word_sep < 0: token units.  Out: distance [B], ops [B][3] (substitutions, insertions, deletions), units [B][2]
 * (hypothesis, reference), status [B] (0, or 2 for a length outside [0, N] / [0, M]: -1 everywhere);
 * hyp_align [B][N], ref_align [B][M] (each nullable, read only with moves): the aligned unit's index or -1, -1 beyond
 * the unit counts.  moves (nullable): [B][pair_move_words] scratch.  cols: the plan's column bound.
 */
template <int K, class Hash>
__global__ void __launch_bounds__(32 * kEditMaxWarps) edit_distance_kernel(
    const int32_t* __restrict__ hyp, int N, const int32_t* __restrict__ hyp_lens, const int32_t* __restrict__ ref,
    int M, const int32_t* __restrict__ ref_lens, int word_sep, int cols, int32_t* __restrict__ distance,
    int32_t* __restrict__ ops, int32_t* __restrict__ units, int32_t* __restrict__ status,
    int32_t* __restrict__ hyp_align, int32_t* __restrict__ ref_align, uint32_t* __restrict__ moves) {
  // all shared memory is dynamic, so that the kernel may opt in to the whole window: the control block, then the data
  GTNB_DYNAMIC_SMEM(int, ctl);
  int* ring = ctl; // warp w's bottom row: {D, counts} by column
  int* cnt = ring + 2 * kEditMaxWarps * kEditRing; // word mode: per-warp counts of starts, ends, hypothesis starts
  int* produced = cnt + 3 * kEditMaxWarps; // columns warp w has put in its ring
  int* consumed = produced + kEditMaxWarps; // columns warp w has taken from warp w - 1's ring
  int* res = consumed + kEditMaxWarps; // D and the packed counts of the last cell
  int* smem = ctl + kEditCtlInts;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nthreads = blockDim.x, nwarps = nthreads >> 5;
  const int nh = hyp_lens[b], nr = ref_lens[b];
  const long long hrow = (long long)b * N, rrow = (long long)b * M;
  if (!(nh >= 0 && nh <= N && nr >= 0 && nr <= M)) {
    if (tid == 0) {
      distance[b] = -1;
      ops[3ll * b] = ops[3ll * b + 1] = ops[3ll * b + 2] = -1;
      units[2ll * b] = units[2ll * b + 1] = -1;
      status[b] = 2;
    }
    if (moves && hyp_align)
      for (int i = tid; i < N; i += nthreads) hyp_align[hrow + i] = -1;
    if (moves && ref_align)
      for (int i = tid; i < M; i += nthreads) ref_align[rrow + i] = -1;
    return;
  }
  int* tok = smem; // hypothesis tokens, then reference tokens
  const int total = nh + nr;
  for (int p = tid; p < total; p += nthreads) tok[p] = p < nh ? hyp[hrow + p] : ref[rrow + p - nh];
  if (tid < kEditMaxWarps) produced[tid] = consumed[tid] = 0;
  __syncthreads();

  const int* unit = tok; // hypothesis units, then reference units
  int hu = nh, ru = nr;
  if (word_sep >= 0) {
    const long long cap = (long long)((N + 1) / 2) + (M + 1) / 2;
    int* wstart = tok + N + M;
    int* wend = wstart + cap;
    int* wid = wend + cap;
    uint64_t* whash = reinterpret_cast<uint64_t*>(smem + ((N + M + 3 * cap + 1) & ~1ll)); // (kEditCtlInts even)
    const unsigned below = (1u << lane) - 1;
    int words = 0, hwords = 0, ends = 0;
    for (int base = 0; base < total; base += nthreads) {
      const int p = base + tid;
      bool s = false, e = false;
      if (p < total && tok[p] != word_sep) {
        s = p == 0 || p == nh || tok[p - 1] == word_sep;
        e = p == nh - 1 || p == total - 1 || tok[p + 1] == word_sep;
      }
      const unsigned bs = __ballot_sync(0xffffffffu, s), be = __ballot_sync(0xffffffffu, e);
      const unsigned bh = __ballot_sync(0xffffffffu, s && p < nh);
      if (lane == 0) {
        cnt[warp] = __popc(bs);
        cnt[kEditMaxWarps + warp] = __popc(be);
        cnt[2 * kEditMaxWarps + warp] = __popc(bh);
      }
      __syncthreads();
      int os = words, oe = ends;
      for (int w = 0; w < nwarps; w++) {
        if (w < warp) {
          os += cnt[w];
          oe += cnt[kEditMaxWarps + w];
        }
        words += cnt[w];
        ends += cnt[kEditMaxWarps + w];
        hwords += cnt[2 * kEditMaxWarps + w];
      }
      if (s) wstart[os + __popc(bs & below)] = p;
      if (e) wend[oe + __popc(be & below)] = p + 1;
      __syncthreads();
    }
    for (int q = tid; q < words; q += nthreads) {
      uint64_t h = (uint64_t)(wend[q] - wstart[q]);
      for (int t = wstart[q]; t < wend[q]; t++) h = Hash::combine(h, tok[t]);
      whash[q] = h;
    }
    __syncthreads();
    for (int q = tid; q < words; q += nthreads) {
      const uint64_t h = whash[q];
      const int s0 = wstart[q], len = wend[q] - s0;
      int id = q;
      for (int o = 0; o < q && id == q; o++) {
        if (whash[o] != h || wend[o] - wstart[o] != len) continue;
        int t = 0;
        while (t < len && tok[wstart[o] + t] == tok[s0 + t]) t++;
        if (t == len) id = o;
      }
      wid[q] = id;
    }
    __syncthreads();
    unit = wid;
    hu = hwords;
    ru = words - hwords;
  }

  const bool swap = hu > ru;
  const int R = swap ? ru : hu, L = swap ? hu : ru;
  const int* rowU = swap ? unit + hu : unit;
  const int* colU = swap ? unit : unit + hu;
  if (tid == 0 && R == 0) {
    res[0] = L;
    res[1] = edit_first_row(L, swap);
  }
  const int active = (R + 32 * K - 1) / (32 * K);
  if (warp < active) {
    const int i0 = (warp * 32 + lane) * K; // rows i0 + 1 .. i0 + K
    int D[K], P[K], U[K];
#pragma unroll
    for (int r = 0; r < K; r++) {
      const int i = i0 + r + 1;
      U[r] = i <= R ? rowU[i - 1] : 0;
      D[r] = i;
      P[r] = edit_first_col(i, swap);
    }
    int prevD = i0, prevP = edit_first_col(i0, swap); // the cell above the strip, one column back
    int botD = D[K - 1], botP = P[K - 1];
    const bool last = warp == active - 1;
    const int own = (R - 1) / K; // the lane (of the CTA) whose strip holds row R
    volatile int* vprod = produced;
    volatile int* vcons = consumed;
    int seen = 0, room = kEditRing;
    uint32_t* mv_out = moves ? moves + ((long long)b * nwarps + warp) * (cols + 31) * 32 + lane : nullptr;
    for (int t = 0; t < L + 31; t++) {
      const int j = t - lane + 1;
      const bool act = j >= 1 && j <= L;
      int upD = __shfl_up_sync(0xffffffffu, botD, 1), upP = __shfl_up_sync(0xffffffffu, botP, 1);
      if (lane == 0 && act) {
        if (warp == 0) {
          upD = j;
          upP = edit_first_row(j, swap);
        } else {
          while (seen < j) {
            seen = vprod[warp - 1];
            if (seen < j) __nanosleep(20);
          }
          __threadfence_block();
          const volatile int* slot = ring + 2 * ((warp - 1) * kEditRing + (j & (kEditRing - 1)));
          upD = slot[0];
          upP = slot[1];
          __threadfence_block();
          vcons[warp] = j;
        }
      }
      if (act) {
        const int c = colU[j - 1];
        int dgD = prevD, dgP = prevP, abD = upD, abP = upP;
        uint32_t mv = 0;
#pragma unroll
        for (int r = 0; r < K; r++) {
          const int lfD = D[r], lfP = P[r];
          const int mis = U[r] != c;
          const int delD = swap ? abD : lfD, delP = swap ? abP : lfP;
          const int insD = swap ? lfD : abD, insP = swap ? lfP : abP;
          int bD = dgD + mis, bP = dgP + mis;
          uint32_t code = 0;
          if (delD + 1 < bD) {
            bD = delD + 1;
            bP = delP;
            code = 1;
          }
          if (insD + 1 < bD) {
            bD = insD + 1;
            bP = insP + 0x10000;
            code = 2;
          }
          mv |= code << (2 * r);
          dgD = lfD;
          dgP = lfP;
          D[r] = abD = bD;
          P[r] = abP = bP;
        }
        prevD = upD;
        prevP = upP;
        if (mv_out) mv_out[32ll * t] = mv;
        if (j == L && warp * 32 + lane == own) {
#pragma unroll
          for (int r = 0; r < K; r++)
            if (i0 + r + 1 == R) {
              res[0] = D[r];
              res[1] = P[r];
            }
        }
      }
      botD = D[K - 1];
      botP = P[K - 1];
      if (lane == 31 && act && !last) {
        while (room < j) {
          room = vcons[warp + 1] + kEditRing;
          if (room < j) __nanosleep(20);
        }
        __threadfence_block();
        volatile int* slot = ring + 2 * (warp * kEditRing + (j & (kEditRing - 1)));
        slot[0] = botD;
        slot[1] = botP;
        __threadfence_block();
        vprod[warp] = j;
      }
    }
  }
  __syncthreads();
  if (tid == 0) {
    const int d = res[0], p = res[1];
    distance[b] = d;
    ops[3ll * b] = p & 0xffff;
    ops[3ll * b + 1] = p >> 16;
    ops[3ll * b + 2] = d - (p & 0xffff) - (p >> 16);
    units[2ll * b] = hu;
    units[2ll * b + 1] = ru;
    status[b] = 0;
  }
  if (!moves) return;
  if (hyp_align)
    for (int i = hu + tid; i < N; i += nthreads) hyp_align[hrow + i] = -1;
  if (ref_align)
    for (int i = ru + tid; i < M; i += nthreads) ref_align[rrow + i] = -1;
  if (tid != 0) return;
  int i = R, j = L;
  while (i > 0 || j > 0) {
    int code; // 0 diagonal, 1 deletion, 2 insertion
    if (i == 0) {
      code = swap ? 2 : 1;
    } else if (j == 0) {
      code = swap ? 1 : 2;
    } else {
      const int s = (i - 1) / K, w = s >> 5, l = s & 31;
      const uint32_t word = moves[(((long long)b * nwarps + w) * (cols + 31) + (j - 1 + l)) * 32 + l];
      code = (word >> (2 * ((i - 1) % K))) & 3;
    }
    const int hi = swap ? j - 1 : i - 1, ri = swap ? i - 1 : j - 1;
    if (code == 0) {
      if (hyp_align) hyp_align[hrow + hi] = ri;
      if (ref_align) ref_align[rrow + ri] = hi;
      i--;
      j--;
    } else if (code == 1) {
      if (ref_align) ref_align[rrow + ri] = -1;
      if (swap) i--;
      else j--;
    } else {
      if (hyp_align) hyp_align[hrow + hi] = -1;
      if (swap) j--;
      else i--;
    }
  }
}

#ifndef GTNB_HOST_EMU

long long edit_distance_move_words(int B, int N, int M, int word_sep) {
  return (long long)B * edit_plan(N, M, word_sep).pair_move_words;
}

int launch_edit_distance(gtnb_ctx* ctx, int B, const int32_t* hyp, int N, const int32_t* hyp_lens,
                         const int32_t* ref, int M, const int32_t* ref_lens, int word_sep, int32_t* distance,
                         int32_t* ops, int32_t* units, int32_t* status, int32_t* hyp_align, int32_t* ref_align,
                         uint32_t* moves) {
  if (B <= 0) return GTNB_OK;
  const EditPlan p = edit_plan(N, M, word_sep);
#define GTNB_EDIT_LAUNCH(K_)                                                                                    \
  case K_: {                                                                                                    \
    if (p.smem_bytes > 48 * 1024) {                                                                             \
      const int rc__ = ensure_max_smem(ctx, (const void*)edit_distance_kernel<K_, EditHash>);                   \
      if (rc__) return rc__;                                                                                    \
    }                                                                                                           \
    GTNB_LAUNCH(ctx, "edit_distance",                                                                           \
                edit_distance_kernel<K_, EditHash><<<B, 32 * p.warps, p.smem_bytes, ctx->stream>>>(             \
                    hyp, N, hyp_lens, ref, M, ref_lens, word_sep, p.cols, distance, ops, units, status,        \
                    hyp_align, ref_align, moves));                                                              \
    break;                                                                                                      \
  }
  switch (p.K) {
    GTNB_EDIT_LAUNCH(1)
    GTNB_EDIT_LAUNCH(2)
    GTNB_EDIT_LAUNCH(4)
    GTNB_EDIT_LAUNCH(8)
    GTNB_EDIT_LAUNCH(16)
    default: return fail(ctx, GTNB_ERR_LOGIC, "launch_edit_distance: no kernel for this strip height");
  }
#undef GTNB_EDIT_LAUNCH
  return GTNB_OK;
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
