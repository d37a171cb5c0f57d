/*
 * k_dense.cu -- factored dense-trellis Viterbi: viterbiPath / viterbiScore of
 * compose(emissions, transitions) (test/criterion_test.cpp:328-344, SURVEY.md config 4)
 * WITHOUT materialising the lattice.  At T=2000, C=128 the composed graph has
 * 32.75 M arcs per utterance (16.8 G for B=512): it cannot exist in HBM, so the
 * lattice stays factored, w(t, j->i) = e[t][i] + trans[j->i], and only the [T][C]
 * back-pointers (1 byte each) and the rolling [C] score vector are stored.
 *
 * Two graph kinds, a compile-time flag (they differ only in the first frame and the weight offset):
 *   - ASG (BIGRAM = false): the transitions graph of criterion_test.cpp:316-326, one start node with C start
 *     arcs (trans[0..C)) and the C x C matrix after them (trans[C + i*C + j] = w(j -> i)).  Frame 0 has the
 *     start node as its single predecessor: fl(0 + fl(e[0][i] + trans[i])).
 *   - BIGRAM: n-gram CTC's G (gtnb_ngram_ctc_loss), C nodes, every node start and accept, arc j -> i with
 *     label i and weight trans[i*C + j]; the lattice is intersect(E, G).  Frame 0 has the C start states of G
 *     (score 0 each) as predecessors: max_j fl(0 + fl(e[0][i] + W[i][j])), i.e. the recursion of the later
 *     frames run on a zero score vector.
 *
 * Exactness (the path must be bit-identical to the reference's):
 *   - the reference's arc weight is first.weight + second.weight = fl(e + trans)
 *     (compose.cpp:435) and the relaxation is fl(score[src] + w) (shortest.cpp:213):
 *     both adds are kept as separate __fadd_rn, in that association;
 *   - ties: shortestPath keeps the FIRST relaxation that reaches the maximum
 *     (strict '>', shortest.cpp:214).  For these lattices the reference pops the
 *     frame-t nodes in ascending state order, so the smallest predecessor j wins;
 *     the best accept node is the first maximum in ascending state order (:226-237).
 *   - -inf weights forbid arcs: a state all of whose candidates are -inf keeps -inf, and when every final
 *     state is -inf there is no accepting path (score -inf, path all -1).  A NaN candidate never compares
 *     greater, so it acts like -inf; the reference propagates NaN instead, and no parity is claimed for NaN.
 *
 * One CTA per utterance; the C x C transition tile lives in shared memory for the
 * whole utterance (padded so that the G lanes sharing an output state hit distinct
 * banks); G = 256 / C lanes split the predecessor range of one state and combine with
 * warp shuffles; the traceback runs on one warp with 8 back-pointer rows in flight.
 * Back-pointer rows are dense_bp_pitch(C) bytes apart (C rounded up to a multiple of 4), so the
 * traceback reads every row as whole 32-bit words for any C.
 * The emissions may be float32, bfloat16 or fp16 (template parameter E, gtnb_viterbi_dense_typed): every element is
 * widened to float32 on load, so the 16-bit kernels relax exactly the float32 kernels' candidates.
 */
#include "gtnb_ptx.h"

namespace gtnb {

/* bytes between two back-pointer rows: C rounded up to whole 32-bit words */
int dense_bp_pitch(int C) {
  return (C + 3) & ~3;
}

namespace {

constexpr int kDenseThreads = 256;

template <int G, bool BIGRAM = false, class E = float> // E: the element type of the emissions (float, bf16_t, f16_t)
__global__ void __launch_bounds__(kDenseThreads) viterbi_dense_kernel(
    int T_max,
    int C,
    const int32_t* __restrict__ T_arr, // nullable
    const E* __restrict__ emis,
    long long stride,
    const float* __restrict__ trans, // ASG: [C] start arcs, then [C][C]; BIGRAM: [C][C]; w(j -> i) at [i*C + j]
    uint8_t* __restrict__ bp, // [B][T_max][pitch]
    int32_t* __restrict__ paths, // [B][T_max]: the path, then -1
    float* __restrict__ scores,
    float empty_score = 0.0f) { // viterbiScore of an utterance with T_b = 0 (gtnb_viterbi_dense's 0 by default)
  GTNB_DYNAMIC_SMEM(unsigned char, smem_raw);
  const int P = C + 32 / G; // padded row stride of the transition tile
  const int pitch = (C + 3) & ~3; // dense_bp_pitch(C)
  float* s_tr = reinterpret_cast<float*>(smem_raw); // s_tr[j * P + i] = w(j -> i)
  float* s_sc = s_tr + (size_t)C * P; // [2][C]
  const int b = blockIdx.x;
  const int T = T_arr ? T_arr[b] : T_max;
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  constexpr int SPW = 32 / G; // states per warp
  const int sub = lane / SPW; // which slice of the predecessors
  const E* e = emis + (long long)b * stride;
  uint8_t* mybp = bp + (long long)b * T_max * pitch;
  const float* W = BIGRAM ? trans : trans + C;

  for (int k = tid; k < C * C; k += kDenseThreads) {
    const int i = k / C, j = k % C;
    s_tr[j * P + i] = W[k];
  }
  for (int i = tid; i < C; i += kDenseThreads) {
    if (BIGRAM) {
      s_sc[C + i] = 0.0f; // the start states of G, read as frame -1 by the loop below
    } else if (T > 0) {
      // frame 0: single predecessor, the start node (score 0): fl(0 + fl(e + w_start))
      s_sc[i] = __fadd_rn(0.0f, __fadd_rn(ld_elem(e + i), trans[i]));
      mybp[i] = 0;
    }
  }
  __syncthreads();

  const int n_pass = (C + kDenseThreads / G - 1) / (kDenseThreads / G);
  for (int t = BIGRAM ? 0 : 1; t < T; t++) {
    const float* prev = s_sc + ((t - 1) & 1) * C;
    float* cur = s_sc + (t & 1) * C;
    uint8_t* bprow = mybp + (long long)t * pitch;
    for (int p = 0; p < n_pass; p++) {
      const int i = p * (kDenseThreads / G) + warp * SPW + (lane % SPW);
      const bool live = i < C;
      const float et = live ? ldg_elem(e + (long long)t * C + i) : 0.0f;
      float best = -CUDART_INF_F;
      int bj = 0x7fffffff;
      if (live) {
        const float* col = s_tr + i;
        // strict '>' in ascending j: the smallest j of a slice wins ties.  G <= 2 (C > 64): four predecessors at a
        // time, their shared-memory loads issued ahead of the adds (ptxas interleaves them otherwise, 1.1 ms at
        // configs[3]); G >= 4: the plain unrolled loop, which measured faster there
        if (G <= 2) {
          int j = sub;
          for (; j + 3 * G < C; j += 4 * G) {
            float w[4], q[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
              w[u] = col[(j + u * G) * P];
              q[u] = prev[j + u * G];
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
              const float v = __fadd_rn(q[u], __fadd_rn(et, w[u]));
              if (v > best) {
                best = v;
                bj = j + u * G;
              }
            }
          }
          for (; j < C; j += G) {
            const float v = __fadd_rn(prev[j], __fadd_rn(et, col[j * P]));
            if (v > best) {
              best = v;
              bj = j;
            }
          }
        } else {
#pragma unroll 4
          for (int j = sub; j < C; j += G) {
            const float v = __fadd_rn(prev[j], __fadd_rn(et, col[j * P]));
            if (v > best) {
              best = v;
              bj = j;
            }
          }
        }
      }
      if (G > 1) {
#pragma unroll
        for (int o = SPW; o < 32; o <<= 1) {
          const float ob = __shfl_xor_sync(0xffffffffu, best, o);
          const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
          if (ob > best || (ob == best && oj < bj)) {
            best = ob;
            bj = oj;
          }
        }
      }
      if (live && sub == 0) {
        cur[i] = best;
        bprow[i] = (uint8_t)(bj == 0x7fffffff ? 0 : bj);
      }
    }
    __syncthreads();
  }

  // best accept node: first maximum in ascending state order; then the traceback
  if (warp == 0) {
    int32_t* out = paths + (long long)b * T_max;
    for (int t = T + lane; t < T_max; t += 32) out[t] = -1; // beyond T_b
    if (T == 0) {
      if (lane == 0) scores[b] = empty_score;
      return;
    }
    const float* fin = s_sc + ((T - 1) & 1) * C;
    float best = -CUDART_INF_F;
    int bi = 0x7fffffff;
    for (int i = lane; i < C; i += 32) {
      if (fin[i] > best) {
        best = fin[i];
        bi = i;
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) {
        best = ob;
        bi = oi;
      }
    }
    if (lane == 0) scores[b] = best;
    if (bi == 0x7fffffff) { // every path is -inf: no accepting path (shortest.cpp:233)
      for (int t = lane; t < T; t += 32) out[t] = -1;
      return;
    }
    // make this CTA's back-pointer stores visible to its own loads
    __threadfence_block();
    int state = bi;
    const int words = pitch / 4; // <= 64
    for (int t0 = T - 1; t0 >= 0; t0 -= 8) {
      // rows t0, t0-1, ..., t0-7 in flight; lane holds bytes [4*lane, 4*lane+4) (+128)
      uint32_t lo[8], hi[8];
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const int t = t0 - k;
        lo[k] = hi[k] = 0;
        if (t >= 1) {
          const uint32_t* row = reinterpret_cast<const uint32_t*>(mybp) + (long long)t * words;
          if (lane < words) lo[k] = __ldcg(row + lane);
          if (lane + 32 < words) hi[k] = __ldcg(row + lane + 32);
        }
      }
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const int t = t0 - k;
        if (t < 0) break;
        if (lane == 0) out[t] = state;
        if (t >= 1) {
          const int w = state >> 2;
          const uint32_t word = (w < 32) ? __shfl_sync(0xffffffffu, lo[k], w) : __shfl_sync(0xffffffffu, hi[k], w - 32);
          state = (int)((word >> (8 * (state & 3))) & 0xffu);
        }
      }
    }
  }
}

} // namespace

#ifndef GTNB_HOST_EMU

namespace {

/* lanes per state: G = 256 / C rounded down to a power of two, at most 32 */
int dense_lanes(int C) {
  int G = 1;
  while (G < 32 && C * (G * 2) <= kDenseThreads) G *= 2;
  return G;
}

/* the transition tile and the two score rows */
size_t dense_smem_bytes(int C) {
  return sizeof(float) * ((size_t)C * (C + 32 / dense_lanes(C)) + 2 * (size_t)C);
}

template <class E>
int viterbi_dense_typed(
    gtnb_ctx* ctx, int B, int T_max, int C, bool bigram, const int32_t* T_dev, const E* emis, int64_t stride,
    const float* trans_dev, float empty_score, uint8_t* bp, int32_t* paths, float* scores) {
  const int G = dense_lanes(C);
  const size_t smem = dense_smem_bytes(C);
  if (smem > (size_t)kMaxDynamicSmem)
    return fail(ctx, GTNB_ERR_UNSUPPORTED,
                "gtnb_viterbi_dense: the transitions tile does not fit shared memory (C <= 224)");
#define LAUNCH_DENSE(G_, K_)                                                                        \
  do {                                                                                              \
    int rc__ = ensure_max_smem(ctx, (const void*)viterbi_dense_kernel<G_, K_, E>);                  \
    if (rc__) return rc__;                                                                          \
    GTNB_LAUNCH(ctx, K_ ? "viterbi_dense_bigram" : "viterbi_dense",                                 \
                viterbi_dense_kernel<G_, K_, E><<<B, kDenseThreads, smem, ctx->stream>>>(           \
                    T_max, C, T_dev, emis, (long long)stride, trans_dev, bp, paths, scores, empty_score)); \
  } while (0)
#define LAUNCH_KIND(G_)            \
  do {                             \
    if (bigram)                    \
      LAUNCH_DENSE(G_, true);      \
    else                           \
      LAUNCH_DENSE(G_, false);     \
  } while (0)
  switch (G) {
    case 1: LAUNCH_KIND(1); break;
    case 2: LAUNCH_KIND(2); break;
    case 4: LAUNCH_KIND(4); break;
    case 8: LAUNCH_KIND(8); break;
    case 16: LAUNCH_KIND(16); break;
    default: LAUNCH_KIND(32); break;
  }
#undef LAUNCH_KIND
#undef LAUNCH_DENSE
  return GTNB_OK;
}

} // namespace

bool viterbi_dense_supported(int C) {
  return C >= 1 && C <= 256 && dense_smem_bytes(C) <= (size_t)kMaxDynamicSmem;
}

int launch_viterbi_dense(
    gtnb_ctx* ctx, int B, int T_max, int C, bool bigram, const int32_t* T_dev, const void* emis, int64_t stride,
    const float* trans_dev, float empty_score, uint8_t* bp, int32_t* paths, float* scores, int dtype) {
  if (B == 0) return GTNB_OK;
  if (C < 1 || C > 256)
    return fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_viterbi_dense: needs 1 <= C <= 256");
  switch (dtype) {
    case GTNB_F32:
      return viterbi_dense_typed(ctx, B, T_max, C, bigram, T_dev, static_cast<const float*>(emis), stride, trans_dev,
                                 empty_score, bp, paths, scores);
    case GTNB_BF16:
      return viterbi_dense_typed(ctx, B, T_max, C, bigram, T_dev, static_cast<const bf16_t*>(emis), stride, trans_dev,
                                 empty_score, bp, paths, scores);
    case GTNB_F16:
      return viterbi_dense_typed(ctx, B, T_max, C, bigram, T_dev, static_cast<const f16_t*>(emis), stride, trans_dev,
                                 empty_score, bp, paths, scores);
    default: return fail(ctx, GTNB_ERR_LOGIC, "launch_viterbi_dense: unknown element type");
  }
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
