/*
 * k_implicit.cu -- forwardScore(intersect(g, emissions)) and its backward WITHOUT
 * materialising the lattice ("implicit lattice": SURVEY.md section 8(d), B_io formulation).
 *
 * compose(g, linearGraph(T, C)) is frame synchronous: composed node (u, t) exists iff graph
 * node u can be reached from a start node in exactly t arcs and can reach an accept node in
 * exactly T - t arcs (compose.cpp:64-104 findReachable + the forward BFS :400-470); its
 * in-arcs are the graph's in-arcs (i -> u, label c, weight w) whose source (i, t-1) exists,
 * with weight fl(w + emissions[t-1][c]) (compose.cpp:435).  So instead of building the
 * lattice and sweeping it, one CTA per utterance keeps the graph operand in shared memory /
 * registers and sweeps the frames directly:
 *
 *   forward  S_t[u] = logadd_{(i->u)} ( S_{t-1}[i] + fl(w + e[t-1][c]) ),  S_0 = 0 on start
 *            nodes, -inf elsewhere (shortest.cpp:102-136).  Nodes the reference prunes are
 *            either unreachable (their score is -inf and contributes exp(-inf) = 0 to every
 *            sum, exactly like an absent arc) or cannot reach an accept node (they never feed
 *            a surviving node), so the surviving nodes get the reference's scores.
 *   backward shortestDistanceGrad (shortest.cpp:33-82) + compose's gradFunc
 *            (compose.cpp:496-518) on the same implicit structure: a node with score -inf
 *            does not exist (no gradient), a node that cannot reach an accept node receives
 *            exactly 0.  Per level the only value on the serial chain is the node gradient:
 *            the arc factors exp(S_{t-1}[i] + w' - S_t[u]) do not depend on it and are
 *            computed one level ahead, in the shadow of the barrier.
 *
 * HBM traffic per utterance: emissions read once per pass (4TC each), dense per-frame node
 * scores written by forward and read by backward (4(T+1)pitch each), emission gradients
 * accumulated with one red.global per (node, frame).  No row_ptr / arc / gradInfo arrays.
 *
 * Valid only when every weight is finite (then "score == -inf" <=> "node does not exist");
 * both kernels raise a per-utterance status bit on a non-finite emission or arc weight and
 * the caller re-runs the batch through the materialised path, which reproduces the
 * reference's NaN / inf propagation arc by arc.  Requires: no epsilon labels, all labels in
 * [0, C), all in-arcs of a graph node carry the same label (CTC, forced alignment, ASG).
 *
 * Arc-label mode (template flag ARC, gtnb_graph_loss on graphs where some node's in-arcs carry
 * different labels: a wildcard state, hand-built graphs): every in-arc reads its own emission
 * e[t-1][label(a)] from the frame's emission row staged in shared memory (any C up to
 * kArcMaxLabels), and the backward sums the arc posteriors of a frame per label in a C-float
 * shared row that is flushed to global memory once per frame.  Only the several-nodes-per-thread
 * path and the wide kernels have this mode; with ARC = false they compile to what they were.
 *
 * Tropical mode (template flag TROP, gtnb_graph_viterbi): the forward kernels take the max instead of the logadd,
 * and implicit_trace_kernel walks the best path back from the saved score rows (with TROP = false the forward
 * kernels compile to what they were).
 *
 * Element type (template parameter E, lat->dtype): the one-node / several-nodes-per-thread log-semiring kernels of
 * label-uniform graphs -- the mode the trellis criteria's numerators take -- also read bfloat16 / fp16 emissions,
 * widened to float32 where a frame uses them (the prefetch rings hold the 16 bits); the emission gradient stays
 * float32.  Every other mode has float32 instantiations only and refuses a 16-bit lattice (implicit_elem_mode).
 */
#include <algorithm>

#include "gtnb_ptx.h"

namespace gtnb {

namespace {

constexpr int kImpThreads = 256;
constexpr int kPf = 8; // frames of register prefetch (emissions, saved scores)
/* (Alternatives that were slower at B=256 on an earlier GPU target, not re-measured on the H100: a 2-deep
 * register ring behind prefetch.global.L1 issued 8 frames ahead; prefetching the three source scores
 * of every arc into registers instead of staging the row in shared memory.) */
// Fast path (graph operand with <= kImpThreads nodes, in/out degree <= 3): one node per thread,
// branch-free.  Score rows and arc-gradient buffers have compile-time strides so that the two
// halves of each double buffer differ by an immediate offset; absent arcs point at a dummy
// slot (score -inf / gradient 0) instead of being predicated off.
constexpr int kFastRow = kImpThreads + 8; // floats per score row
constexpr int kRowDummy = kImpThreads + 4; // holds -inf in both rows
constexpr int kFastCur = 3 * kImpThreads + 8; // floats per arc-gradient buffer
constexpr int kCurDummy = 3 * kImpThreads + 4; // holds 0 in both buffers

struct ImpLayout {
  int pitch; // floats per score row in shared memory (max over the batch, multiple of 4)
  int tabN, tabA; // table capacities
  int off_S, off_inptr, off_src, off_w, off_lab, off_flags, off_red;
  int off_outptr, off_outent, off_cursor, off_cur, off_ng, off_accg; // backward only
  int off_sw, off_act, off_erow, off_rows3; // wide kernels
  int total;
  int off_alab, off_earc, off_ge; // arc-label mode: per-entry labels, [2][C] emission rows, [C] emission gradients
};

// arc-label mode: the emission row of a frame is staged by every thread in steps of kImpThreads,
// kArcRows values per thread (held in registers while the frame before is swept)
constexpr int kArcRows = 4;
constexpr int kArcMaxLabels = kArcRows * kImpThreads;

ImpLayout make_imp_layout(int maxN, int maxA, bool backward, bool wide = false, int C = 0, bool arc = false) {
  ImpLayout o;
  o.pitch = (maxN + 3) & ~3;
  o.tabN = maxN + 1;
  o.tabA = std::max(maxA, 1);
  int off = 0;
  auto take = [&](int bytes) {
    int at = off;
    off += (bytes + 15) & ~15;
    return at;
  };
  o.off_S = take(4 * 2 * std::max(o.pitch, kFastRow));
  o.off_inptr = take(4 * (o.tabN + 1));
  o.off_src = take(4 * o.tabA);
  o.off_w = take(4 * o.tabA);
  o.off_lab = take(4 * o.tabN);
  o.off_flags = take(o.tabN);
  o.off_red = take(4 * 16);
  o.off_outptr = o.off_outent = o.off_cursor = o.off_cur = o.off_ng = o.off_accg = 0;
  o.off_sw = o.off_act = o.off_erow = o.off_rows3 = 0;
  if (backward) {
    o.off_outptr = take(4 * (o.tabN + 1));
    o.off_outent = take(4 * o.tabA);
    o.off_cursor = take(4 * o.tabN);
    o.off_cur = take(4 * 2 * std::max(o.tabA, kFastCur));
    o.off_ng = take(4 * o.pitch);
    o.off_accg = take(4 * o.tabA);
  }
  if (wide) {
    o.off_sw = take(8 * o.tabA);
    o.off_act = take(4 * 2 * o.tabN);
    o.off_erow = take(4 * 2 * std::max(C, 4));
    o.off_rows3 = take(4 * 3 * o.pitch);
  }
  o.off_alab = o.off_earc = o.off_ge = 0;
  if (arc) {
    o.off_alab = take(4 * o.tabA);
    o.off_earc = wide ? o.off_erow : take(4 * 2 * std::max(C, 4));
    if (backward) o.off_ge = take(4 * std::max(C, 4));
  }
  o.total = off;
  return o;
}

__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < kImpThreads / 32; w++) r = fmaxf(r, red[w]);
  return r;
}
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < kImpThreads / 32; w++) r += red[w];
  return r;
}

/* the graph operand's in-arc tables -> shared memory; returns "some weight is not finite" */
__device__ __forceinline__ bool load_tables(
    const GraphMeta& m, const uint8_t* __restrict__ sg_flags, const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ sg_in_src, const int32_t* __restrict__ sg_in_label,
    const float* __restrict__ sg_in_w, int* t_inptr, int* t_src, float* t_w, int* t_lab,
    unsigned char* t_flags) {
  const int tid = threadIdx.x, N1 = m.sg_N, A1 = m.sg_A;
  const int32_t* ip = sg_in_ptr + m.sg_node_base;
  const int32_t* is = sg_in_src + m.sg_arc_base;
  const int32_t* il = sg_in_label + m.sg_arc_base;
  const float* iw = sg_in_w + m.sg_arc_base;
  const uint8_t* fl = sg_flags + m.sg_node_base;
  bool bad = false;
  for (int i = tid; i <= N1; i += kImpThreads) t_inptr[i] = ip[i];
  for (int e = tid; e < A1; e += kImpThreads) {
    t_src[e] = is[e];
    const float w = iw[e];
    t_w[e] = w;
    bad |= !is_finite(w);
  }
  __syncthreads();
  for (int i = tid; i < N1; i += kImpThreads) {
    t_lab[i] = (t_inptr[i] < t_inptr[i + 1]) ? il[t_inptr[i]] : -1;
    t_flags[i] = fl[i];
  }
  __syncthreads();
  return bad;
}

/* one node, any in-degree: the reference's two passes (shortest.cpp:121-136, :102-114) */
__device__ __noinline__ float imp_fwd_node_any(
    int e0, int e1, float e, const int* t_src, const float* t_w, const float* prev) {
  float mx = neg_inf();
#pragma unroll 1
  for (int a = e0; a < e1; a++) mx = fmaxf(mx, prev[t_src[a]] + (t_w[a] + e));
  if (mx == CUDART_INF_F || mx == -CUDART_INF_F) return mx;
  float sum = -1.0f;
#pragma unroll 1
  for (int a = e0; a < e1; a++) sum += fexp((prev[t_src[a]] + (t_w[a] + e)) - mx);
  return mx + flog1p(sum);
}

/* arc-label mode: the same two passes, every in-arc with its own label's emission */
__device__ __noinline__ float imp_fwd_node_arc(
    int e0, int e1, const float* erow, const int* t_alab, const int* t_src, const float* t_w, const float* prev) {
  float mx = neg_inf();
#pragma unroll 1
  for (int a = e0; a < e1; a++) mx = fmaxf(mx, prev[t_src[a]] + (t_w[a] + erow[t_alab[a]]));
  if (mx == CUDART_INF_F || mx == -CUDART_INF_F) return mx;
  float sum = -1.0f;
#pragma unroll 1
  for (int a = e0; a < e1; a++) sum += fexp((prev[t_src[a]] + (t_w[a] + erow[t_alab[a]])) - mx);
  return mx + flog1p(sum);
}

/* tropical (max) semiring: the first pass alone -- the best in-arc value fl(S[src] + fl(w + e)) */
__device__ __noinline__ float imp_fwd_node_max(
    int e0, int e1, float e, const int* t_src, const float* t_w, const float* prev) {
  float mx = neg_inf();
#pragma unroll 1
  for (int a = e0; a < e1; a++) mx = fmaxf(mx, prev[t_src[a]] + (t_w[a] + e));
  return mx;
}
__device__ __noinline__ float imp_fwd_node_arc_max(
    int e0, int e1, const float* erow, const int* t_alab, const int* t_src, const float* t_w, const float* prev) {
  float mx = neg_inf();
#pragma unroll 1
  for (int a = e0; a < e1; a++) mx = fmaxf(mx, prev[t_src[a]] + (t_w[a] + erow[t_alab[a]]));
  return mx;
}

/* the fast path's combine of three in-arc values: logadd, or max in the tropical semiring */
template <bool TROP>
__device__ __forceinline__ float combine3(float v0, float v1, float v2) {
  return TROP ? fmaxf(fmaxf(v0, v1), v2) : lse3(v0, v1, v2);
}

/* arc-label mode: the per-entry matched labels of the graph operand -> shared memory */
__device__ __forceinline__ void load_arc_labels(const GraphMeta& m, const int32_t* __restrict__ sg_in_label,
                                                int* t_alab) {
  const int32_t* il = sg_in_label + m.sg_arc_base;
  for (int e = threadIdx.x; e < m.sg_A; e += kImpThreads) t_alab[e] = il[e];
  __syncthreads();
}

/* arc-label mode: emission row `row` (C elements) -> shared memory; returns "some value is not finite" */
template <class E>
__device__ __forceinline__ bool stage_erow(const E* row, float* dst, int C) {
  bool bad = false;
  for (int c = threadIdx.x; c < C; c += kImpThreads) {
    const float v = ldg_elem(row + c);
    dst[c] = v;
    bad |= !is_finite(v);
  }
  return bad;
}

/* arc-label mode: one frame's per-label sums of the arc posteriors -> the emission gradient, and the
 * row zeroed for the next frame (each thread flushes and zeroes the same labels) */
__device__ __forceinline__ void flush_erow_grad(float* GE, float* gr, int C, float delta) {
  for (int c = threadIdx.x; c < C; c += kImpThreads) {
    const float v = GE[c];
    GE[c] = 0.0f;
    if (v != 0.0f) atomicAdd(gr + c, v * delta);
  }
}

/* ------------------------------------------------------------------ */
/* forward                                                             */
/* ------------------------------------------------------------------ */

/* TROP: the tropical semiring (viterbiScore, gtnb_graph_viterbi): every logadd becomes a max, the score rows are
 * saved as before for implicit_trace_kernel.  E: the element type of the emissions (float, or bf16_t / f16_t, widened
 * on load; only <false, false> is built for those) */
template <bool ARC = false, bool TROP = false, class E = float>
__global__ void __launch_bounds__(kImpThreads) implicit_forward_kernel(
    const GraphMeta* __restrict__ meta,
    const uint8_t* __restrict__ sg_flags,
    const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ sg_in_src,
    const int32_t* __restrict__ sg_in_label,
    const float* __restrict__ sg_in_w,
    const E* __restrict__ emissions,
    float* __restrict__ scores,
    float* __restrict__ out_scores,
    int32_t* __restrict__ status,
    int C,
    const ImpLayout lay) {
  GTNB_DYNAMIC_SMEM(unsigned char, smem);
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x;
  const int N1 = m.sg_N, T = m.T;
  const int pitch = (N1 + 3) & ~3;
  float* S = reinterpret_cast<float*>(smem + lay.off_S);
  int* t_inptr = reinterpret_cast<int*>(smem + lay.off_inptr);
  int* t_src = reinterpret_cast<int*>(smem + lay.off_src);
  float* t_w = reinterpret_cast<float*>(smem + lay.off_w);
  int* t_lab = reinterpret_cast<int*>(smem + lay.off_lab);
  unsigned char* t_flags = smem + lay.off_flags;
  float* red = reinterpret_cast<float*>(smem + lay.off_red);

  bool bad = load_tables(m, sg_flags, sg_in_ptr, sg_in_src, sg_in_label, sg_in_w, t_inptr, t_src, t_w,
                         t_lab, t_flags);
  int* t_alab = reinterpret_cast<int*>(smem + lay.off_alab); // ARC only
  float* E_s = reinterpret_cast<float*>(smem + lay.off_earc); // ARC only: [2][C], frame t-1 at (t-1) & 1
  if (ARC) load_arc_labels(m, sg_in_label, t_alab);
  float* sc = scores + m.node_base;
  const E* em = emissions + m.emis_off;
  // fast path: one node per thread, every node with at most three in-arcs (block-uniform)
  int my_deg = 0;
  if (tid < N1) my_deg = t_inptr[tid + 1] - t_inptr[tid];
  const bool fast = !ARC && (N1 <= kImpThreads) && !__syncthreads_or(my_deg > 3);
  float* S0 = S;
  float* S1 = S + (fast ? kFastRow : lay.pitch);
  // frame 0: start nodes carry the implicit 0 (shortest.cpp:129-135), nothing else exists
  if (fast) {
    const float v = (tid < N1 && (t_flags[tid] & 1)) ? 0.0f : neg_inf();
    S0[tid] = v;
    if (tid < N1) sc[tid] = v;
    if (tid == 0) S0[kRowDummy] = S1[kRowDummy] = neg_inf();
  } else {
    for (int i = tid; i < N1; i += kImpThreads) {
      const float v = (t_flags[i] & 1) ? 0.0f : neg_inf();
      S0[i] = v;
      sc[i] = v;
    }
    if (ARC && T > 0) bad |= stage_erow(em, E_s, C);
  }
  __syncthreads();

  if (fast) {
    const bool act = tid < N1;
    const int deg = my_deg;
    const bool has = deg > 0;
    int i0 = kRowDummy, i1 = kRowDummy, i2 = kRowDummy;
    float w0 = 0.0f, w1 = 0.0f, w2 = 0.0f;
    if (has) {
      const int e0 = t_inptr[tid];
      i0 = t_src[e0];
      w0 = t_w[e0];
      if (deg > 1) {
        i1 = t_src[e0 + 1];
        w1 = t_w[e0 + 1];
      }
      if (deg > 2) {
        i2 = t_src[e0 + 2];
        w2 = t_w[e0 + 2];
      }
    }
    const E* eml = em + (has ? t_lab[tid] : 0);
    // Emissions of the node's label reach the thread through two register blocks: pf[] holds
    // frames f0 .. f0+kPf-1 (complete), nx[] frames f0+kPf .. f0+2kPf-1, in flight since the
    // previous block boundary.  At a block boundary nx[] is copied to pf[] and the kPf loads of
    // the block after next are issued into nx[], all together.  ptxas tracks every one of these
    // loads on ONE scoreboard and waits for it once per block, so a load issued one frame before
    // that wait (the former one-load-per-frame ring) stalled every block for a full memory
    // latency, and that single wait held the largest share of the kernel's stall samples.
    // (Where the refill sits matters to ptxas: at the END of the block here -- all loads on one
    // scoreboard, waited 7 frames later; at the top it spreads them over the scoreboards the
    // LDS / MUFU results use.  The backward sweep needs it at the top.  Checked in SASS.)
    // (16-bit elements travel through the ring as their bits and are widened where a step uses them)
    ring_t<E> pf[kPf], nx[kPf];
#pragma unroll
    for (int j = 0; j < kPf; j++) pf[j] = (has && j < T) ? ldg_ring(eml + (long long)j * C) : ring_t<E>(0);
#pragma unroll
    for (int j = 0; j < kPf; j++)
      nx[j] = (has && kPf + j < T) ? ldg_ring(eml + (long long)(kPf + j) * C) : ring_t<E>(0);
    const E* epf = eml + (long long)(2 * kPf) * C; // first frame of the next refill
    float* grow = sc + pitch + tid; // this node's score in frame f + 1
    float chk = 0.0f; // becomes NaN when a used emission is not finite
    int f0 = 0;
#define GTNB_FWD_STEP(j)                                                 \
  {                                                                      \
    const float e = has ? ring_f32<E>(pf[j]) : 0.0f; /* idle threads load node 0's */ \
    const float* P = ((j)&1) ? S1 : S0;                                  \
    float* Q = ((j)&1) ? S0 : S1;                                        \
    const float sv = combine3<TROP>(P[i0] + (w0 + e), P[i1] + (w1 + e), P[i2] + (w2 + e)); \
    chk = fmaf(e, 0.0f, chk);                                            \
    Q[tid] = sv;                                                         \
    bar_named<1>(nact);                                                     \
    if (act) *grow = sv; /* after the barrier: nothing waits for it */   \
    grow += pitch;                                                       \
  }
#define GTNB_FWD_REFILL(GUARDED)                                         \
  {                                                                      \
    _Pragma("unroll") for (int j = 0; j < kPf; j++) pf[j] = nx[j];       \
    _Pragma("unroll") for (int j = 0; j < kPf; j++) {                    \
      if (GUARDED)                                                       \
        ldg_if(has && f0 + 2 * kPf + j < T, nx[j], epf + (long long)j * C); \
      else                                                               \
        ldg_keep(nx[j], epf + (long long)j * C);                         \
    }                                                                    \
    epf += (long long)kPf * C;                                           \
  }
    // threads of the warps that hold nodes: the frame loop synchronises them alone on named barrier 1, so that
    // warps without a graph node leave it instead of issuing its instruction stream for nothing (CTC at
    // U=100: 201 nodes = 7 of the 8 warps)
    const int nact = (N1 + 31) & ~31;
    if (tid < nact) {
      for (; f0 + 3 * kPf <= T; f0 += kPf) {
#pragma unroll
        for (int j = 0; j < kPf; j++) GTNB_FWD_STEP(j)
        GTNB_FWD_REFILL(false)
      }
      for (; f0 < T; f0 += kPf) {
#pragma unroll
        for (int j = 0; j < kPf; j++) {
          if (f0 + j >= T) break;
          GTNB_FWD_STEP(j)
        }
        GTNB_FWD_REFILL(true)
      }
    }
#undef GTNB_FWD_REFILL
#undef GTNB_FWD_STEP
    bad |= !(chk == 0.0f);
    __syncthreads(); // the idle warps meet the others again (S rows are read below)
  } else {
    // ---- any graph: several nodes per thread, tables in shared memory
    float* prev = S0;
    float* cur = S1;
    for (int t = 1; t <= T; t++) {
      const E* er = em + (long long)(t - 1) * C;
      float* srow = sc + (long long)t * pitch;
      if (ARC) {
        // frame t-1's row was staged before the last barrier; frame t's goes to the other half
        const float* Ecur = E_s + ((t - 1) & 1) * C;
        for (int i = tid; i < N1; i += kImpThreads) {
          const int e0 = t_inptr[i], e1 = t_inptr[i + 1];
          float sv = neg_inf();
          if (e1 > e0)
            sv = TROP ? imp_fwd_node_arc_max(e0, e1, Ecur, t_alab, t_src, t_w, prev)
                      : imp_fwd_node_arc(e0, e1, Ecur, t_alab, t_src, t_w, prev);
          cur[i] = sv;
          srow[i] = sv;
        }
        if (t < T) bad |= stage_erow(er + C, E_s + (t & 1) * C, C);
      } else {
        for (int i = tid; i < N1; i += kImpThreads) {
          const int e0 = t_inptr[i], e1 = t_inptr[i + 1];
          float sv = neg_inf();
          if (e1 > e0) {
            const float e = ldg_elem(er + t_lab[i]);
            bad |= !is_finite(e);
            sv = TROP ? imp_fwd_node_max(e0, e1, e, t_src, t_w, prev) : imp_fwd_node_any(e0, e1, e, t_src, t_w, prev);
          }
          cur[i] = sv;
          srow[i] = sv;
        }
      }
      float* tmp = prev;
      prev = cur;
      cur = tmp;
      __syncthreads();
    }
  }

  // accept nodes of the last frame (shortest.cpp:147-159)
  const float* Sf = (T & 1) ? S1 : S0;
  float mx = neg_inf();
  for (int i = tid; i < N1; i += kImpThreads)
    if (t_flags[i] & 2) mx = fmaxf(mx, Sf[i]);
  mx = block_max(mx, red);
  float out = mx;
  if (!TROP && mx != CUDART_INF_F && mx != -CUDART_INF_F) {
    float sum = 0.0f;
    for (int i = tid; i < N1; i += kImpThreads)
      if (t_flags[i] & 2) sum += expf(Sf[i] - mx);
    sum = block_sum(sum, red);
    out = mx + log1pf(sum - 1.0f);
  }
  if (tid == 0) out_scores[blockIdx.x] = out;
  if (bad) atomicOr(&status[blockIdx.x], 1);
}

/* out-arc lists of the graph operand (in-entries grouped by source, ascending): the node
 * gradients are gathered through them, fixed order, no floating-point atomics */
__device__ __forceinline__ void build_out_lists(
    int N1, int A1, const int* t_src, int* t_outptr, int* t_outent, int* t_cursor) {
  const int tid = threadIdx.x;
  for (int i = tid; i <= N1; i += kImpThreads) t_outptr[i] = 0;
  __syncthreads();
  for (int e = tid; e < A1; e += kImpThreads) atomicAdd(&t_outptr[t_src[e] + 1], 1);
  __syncthreads();
  if (tid == 0)
    for (int u = 0; u < N1; u++) t_outptr[u + 1] += t_outptr[u];
  __syncthreads();
  for (int u = tid; u < N1; u += kImpThreads) t_cursor[u] = t_outptr[u];
  __syncthreads();
  for (int e = tid; e < A1; e += kImpThreads) t_outent[atomicAdd(&t_cursor[t_src[e]], 1)] = e;
  __syncthreads();
  for (int u = tid; u < N1; u += kImpThreads) {
    const int q0 = t_outptr[u], q1 = t_outptr[u + 1];
    for (int q = q0 + 1; q < q1; q++) {
      const int v = t_outent[q];
      int p = q - 1;
      while (p >= q0 && t_outent[p] > v) {
        t_outent[p + 1] = t_outent[p];
        p--;
      }
      t_outent[p + 1] = v;
    }
  }
  __syncthreads();
}

/* ------------------------------------------------------------------ */
/* backward                                                            */
/* ------------------------------------------------------------------ */

/* E: as in implicit_forward_kernel (only <*, false> is built for 16-bit types); the emission gradient stays float32 */
template <bool GRAPH_GRAD, bool ARC = false, class E = float>
__global__ void __launch_bounds__(kImpThreads) implicit_backward_kernel(
    const GraphMeta* __restrict__ meta,
    const uint8_t* __restrict__ sg_flags,
    const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ sg_in_src,
    const int32_t* __restrict__ sg_in_label,
    const float* __restrict__ sg_in_w,
    const int32_t* __restrict__ sg_in_arc,
    float* __restrict__ grad_graph,
    const E* __restrict__ emissions,
    const float* __restrict__ scores,
    const float* __restrict__ out_scores,
    const float* __restrict__ deltas,
    float* __restrict__ grad_emis,
    long long grad_stride,
    int C,
    const ImpLayout lay) {
  GTNB_DYNAMIC_SMEM(unsigned char, smem);
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x;
  const int N1 = m.sg_N, A1 = m.sg_A, T = m.T;
  const int pitch = (N1 + 3) & ~3;
  float* S = reinterpret_cast<float*>(smem + lay.off_S); // [2][pitch]: rows of saved scores
  int* t_inptr = reinterpret_cast<int*>(smem + lay.off_inptr);
  int* t_src = reinterpret_cast<int*>(smem + lay.off_src);
  float* t_w = reinterpret_cast<float*>(smem + lay.off_w);
  int* t_lab = reinterpret_cast<int*>(smem + lay.off_lab);
  unsigned char* t_flags = smem + lay.off_flags;
  float* red = reinterpret_cast<float*>(smem + lay.off_red);
  int* t_outptr = reinterpret_cast<int*>(smem + lay.off_outptr);
  int* t_outent = reinterpret_cast<int*>(smem + lay.off_outent);
  int* t_cursor = reinterpret_cast<int*>(smem + lay.off_cursor);
  float* CUR = reinterpret_cast<float*>(smem + lay.off_cur); // [2][tabA]: arc gradients of a level
  float* NG = reinterpret_cast<float*>(smem + lay.off_ng); // node gradients (general path)
  float* ACCG = reinterpret_cast<float*>(smem + lay.off_accg); // graph-arc gradients (general path)
  const int32_t* in_arc = sg_in_arc + m.sg_arc_base;
  float* ggr = GRAPH_GRAD ? grad_graph + m.grad_graph_off : nullptr;

  load_tables(m, sg_flags, sg_in_ptr, sg_in_src, sg_in_label, sg_in_w, t_inptr, t_src, t_w, t_lab, t_flags);
  int* t_alab = reinterpret_cast<int*>(smem + lay.off_alab); // ARC only
  float* E_s = reinterpret_cast<float*>(smem + lay.off_earc); // ARC only: frame t-1's emission row
  float* GE = reinterpret_cast<float*>(smem + lay.off_ge); // ARC only: frame t-1's emission gradient per label
  if (ARC) load_arc_labels(m, sg_in_label, t_alab);

  build_out_lists(N1, A1, t_src, t_outptr, t_outent, t_cursor);

  const float out = out_scores[blockIdx.x];
  if (!is_finite(out) || T < 1) return; // no accepting path (empty lattice): no gradient
  const float delta = deltas ? deltas[blockIdx.x] : 1.0f;
  const float* sc = scores + m.node_base;
  const E* em = emissions + m.emis_off;
  float* gem = grad_emis + (long long)blockIdx.x * grad_stride;
  // seeds: nodeGrad[accept] = exp(score - maxA) / exp(out - maxA) (shortest.cpp:49-60)
  float mxa = neg_inf();
  for (int i = tid; i < N1; i += kImpThreads)
    if (t_flags[i] & 2) mxa = fmaxf(mxa, sc[(long long)T * pitch + i]);
  mxa = block_max(mxa, red);
  const float denom = expf(out - mxa);

  int my_deg = 0, my_od = 0;
  if (tid < N1) {
    my_deg = t_inptr[tid + 1] - t_inptr[tid];
    my_od = t_outptr[tid + 1] - t_outptr[tid];
  }
  const bool fast = !ARC && (N1 <= kImpThreads) && !__syncthreads_or(my_deg > 3 || my_od > 3);
  float* Sa = S;
  float* Sb = S + (fast ? kFastRow : lay.pitch);
  float* CURa = CUR;
  float* CURb = CUR + (fast ? kFastCur : lay.tabA);

  if (fast) {
    const bool act = tid < N1;
    const int deg = my_deg, od = my_od;
    const bool has = deg > 0;
    int i0 = kRowDummy, i1 = kRowDummy, i2 = kRowDummy; // sources of the in-arcs
    int a0 = kCurDummy, a1 = kCurDummy, a2 = kCurDummy; // in-entries (arc-gradient slots)
    int q0 = kCurDummy, q1 = kCurDummy, q2 = kCurDummy; // out-arcs (in-entries of the successors)
    float w0 = 0.0f, w1 = 0.0f, w2 = 0.0f;
    if (has) {
      const int e0 = t_inptr[tid];
      i0 = t_src[e0];
      w0 = t_w[e0];
      a0 = e0;
      if (deg > 1) {
        i1 = t_src[e0 + 1];
        w1 = t_w[e0 + 1];
        a1 = e0 + 1;
      }
      if (deg > 2) {
        i2 = t_src[e0 + 2];
        w2 = t_w[e0 + 2];
        a2 = e0 + 2;
      }
    }
    if (od > 0) q0 = t_outent[t_outptr[tid]];
    if (od > 1) q1 = t_outent[t_outptr[tid] + 1];
    if (od > 2) q2 = t_outent[t_outptr[tid] + 2];
    const E* eml = em + (has ? t_lab[tid] : 0);
    const float* scu = sc + (act ? tid : 0);

    // iteration i handles level t = T - i and prepares level t - 1, for which it needs frame
    // f = t - 2 = T - 2 - i of the saved scores and of the emissions.  Two register blocks as in
    // the forward sweep: a block of kPf iterations copies nxs/nxe (loaded during the previous
    // block) to ps/pe and issues all loads of the next block.
    float ps[kPf], nxs[kPf];
    ring_t<E> pe[kPf], nxe[kPf]; // (16-bit elements as their bits, as in the forward sweep)
#pragma unroll
    for (int j = 0; j < kPf; j++) {
      const int f = T - 2 - j;
      nxs[j] = (act && f >= 0) ? __ldg(scu + (long long)f * pitch) : neg_inf();
      nxe[j] = (has && f >= 0) ? ldg_ring(eml + (long long)f * C) : ring_t<E>(0);
    }
    // first frame of the next refill; only dereferenced while >= row 0
    const float* spf = scu + (long long)(T - 2 - kPf) * pitch;
    const E* epf = eml + (long long)(T - 2 - kPf) * C;
    // prologue: the arc factors of level T need row T-1 in shared memory
    float s_own = act ? __ldg(scu + (long long)T * pitch) : neg_inf(); // S_T[u]
    float s_nxt = act ? __ldg(scu + (long long)(T - 1) * pitch) : neg_inf(); // S_{T-1}[u]
    Sb[tid] = s_nxt;
    if (tid == 0) {
      Sa[kRowDummy] = Sb[kRowDummy] = neg_inf();
      CURa[kCurDummy] = CURb[kCurDummy] = 0.0f;
    }
    float g = (act && (t_flags[tid] & 2)) ? expf(s_own - mxa) / denom : 0.0f;
    __syncthreads();
    float E0, E1, E2;
    {
      const float e = has ? ldg_elem(eml + (long long)(T - 1) * C) : 0.0f;
      const float se = (s_own == -CUDART_INF_F) ? CUDART_INF_F : s_own;
      E0 = fexp(Sb[i0] + (w0 + e) - se);
      E1 = fexp(Sb[i1] + (w1 + e) - se);
      E2 = fexp(Sb[i2] + (w2 + e) - se);
    }
    float* gl = gem + (long long)(T - 1) * C + (has ? t_lab[tid] : 0); // emission gradient of level t
    float ga0 = 0.0f, ga1 = 0.0f, ga2 = 0.0f; // gradients of the node's in-arcs of the graph operand
    int i0_ = 0;
    // buffers alternate with the iteration parity: iteration i writes row buffer (i & 1 ? Sb : Sa)
    // and arc-gradient buffer (i & 1 ? CURb : CURa) before its barrier and reads them after it
#define GTNB_BWD_STEP(j)                                                              \
  {                                                                                   \
    float* Cw = ((j)&1) ? CURb : CURa;                                                \
    float* Sw = ((j)&1) ? Sb : Sa;                                                    \
    const float c0 = g * E0, c1 = g * E1, c2 = g * E2;                                \
    Cw[a0] = c0;                                                                      \
    Cw[a1] = c1;                                                                      \
    Cw[a2] = c2;                                                                      \
    const float acc = (c0 + c1) + c2;                                                 \
    if (GRAPH_GRAD) {                                                                 \
      ga0 += c0;                                                                      \
      ga1 += c1;                                                                      \
      ga2 += c2;                                                                      \
    }                                                                                 \
    const float s_f = ps[j]; /* S_{t-2}[u] */                                         \
    const float e_f = has ? ring_f32<E>(pe[j]) : 0.0f; /* e[t-2][label] */            \
    Sw[tid] = s_f;                                                                    \
    bar_named<1>(nact);                                                                  \
    g = (Cw[q0] + Cw[q1]) + Cw[q2]; /* node gradient of level t-1: the serial chain */ \
    /* the emission gradient of level t leaves after the barrier, in the shadow of the gather \
       (ptxas turns the predicated red into a branch: before the barrier it delayed every   \
       warp's arrival) */                                                             \
    red_if(acc != 0.0f, gl, acc * delta);                                             \
    gl -= C;                                                                          \
    s_own = s_nxt;                                                                    \
    s_nxt = s_f;                                                                      \
    { /* arc factors of level t-1; a node that does not exist (score -inf) gets exp(-inf) */ \
      const float se = (s_own == -CUDART_INF_F) ? CUDART_INF_F : s_own;               \
      E0 = fexp(Sw[i0] + (w0 + e_f) - se);                                            \
      E1 = fexp(Sw[i1] + (w1 + e_f) - se);                                            \
      E2 = fexp(Sw[i2] + (w2 + e_f) - se);                                            \
    }                                                                                 \
  }
#define GTNB_BWD_REFILL(GUARDED)                                                      \
  {                                                                                   \
    _Pragma("unroll") for (int j = 0; j < kPf; j++) {                                 \
      ps[j] = nxs[j];                                                                 \
      pe[j] = nxe[j];                                                                 \
    }                                                                                 \
    _Pragma("unroll") for (int j = 0; j < kPf; j++) {                                 \
      if (GUARDED) {                                                                  \
        const bool inb = T - 2 - (i0_ + kPf + j) >= 0;                                \
        ldg_if(act && inb, nxs[j], spf - (long long)j * pitch);                       \
        ldg_if(has && inb, nxe[j], epf - (long long)j * C);                           \
      } else {                                                                        \
        ldg_keep(nxs[j], spf - (long long)j * pitch);                                 \
        ldg_keep(nxe[j], epf - (long long)j * C);                                     \
      }                                                                               \
    }                                                                                 \
    spf -= (long long)kPf * pitch;                                                    \
    epf -= (long long)kPf * C;                                                        \
  }
    const int nact = (N1 + 31) & ~31; // threads of the warps that hold nodes (see the forward kernel)
    if (tid < nact) {
      for (; i0_ + 2 * kPf + 1 <= T; i0_ += kPf) {
        GTNB_BWD_REFILL(false)
#pragma unroll
        for (int j = 0; j < kPf; j++) GTNB_BWD_STEP(j)
      }
      for (; i0_ < T; i0_ += kPf) {
        GTNB_BWD_REFILL(true)
#pragma unroll
        for (int j = 0; j < kPf; j++) {
          if (i0_ + j >= T) break;
          GTNB_BWD_STEP(j)
        }
      }
    }
#undef GTNB_BWD_REFILL
#undef GTNB_BWD_STEP
    if (GRAPH_GRAD && has) {
      // compose gradFunc, graph side (compose.cpp:500-506): the arc's gradient over all frames
      const int e0 = t_inptr[tid];
      atomicAdd(&ggr[in_arc[e0]], ga0 * delta);
      if (deg > 1) atomicAdd(&ggr[in_arc[e0 + 1]], ga1 * delta);
      if (deg > 2) atomicAdd(&ggr[in_arc[e0 + 2]], ga2 * delta);
    }
  } else {
    // ---- general path: several nodes per thread, two barriers per level
    if (GRAPH_GRAD)
      for (int a = tid; a < A1; a += kImpThreads) ACCG[a] = 0.0f;
    if (ARC)
      for (int c = tid; c < C; c += kImpThreads) GE[c] = 0.0f;
    for (int i = tid; i < N1; i += kImpThreads) {
      const float sT = sc[(long long)T * pitch + i];
      Sa[i] = sT;
      NG[i] = (t_flags[i] & 2) ? expf(sT - mxa) / denom : 0.0f;
    }
    float* Sown = Sa; // row t
    float* Sprev = Sb; // row t-1
    for (int t = T; t >= 1; t--) {
      const E* er = em + (long long)(t - 1) * C;
      float* gr = gem + (long long)(t - 1) * C;
      for (int i = tid; i < N1; i += kImpThreads) Sprev[i] = sc[(long long)(t - 1) * pitch + i];
      if (ARC) stage_erow(er, E_s, C);
      __syncthreads();
      if (ARC) {
        for (int i = tid; i < N1; i += kImpThreads) {
          const int e0 = t_inptr[i], e1 = t_inptr[i + 1];
          if (e1 == e0) continue;
          const float gi = NG[i], sn = Sown[i];
          const bool ex = sn > -CUDART_INF_F;
#pragma unroll 1
          for (int a = e0; a < e1; a++) {
            const int lab = t_alab[a];
            const float c = ex ? gi * fexp(Sprev[t_src[a]] + (t_w[a] + E_s[lab]) - sn) : 0.0f;
            CURa[a] = c;
            if (GRAPH_GRAD) ACCG[a] += c; // entry a belongs to this thread only
            if (c != 0.0f) atomicAdd(&GE[lab], c); // shared: one global add per label and frame below
          }
        }
      } else {
        for (int i = tid; i < N1; i += kImpThreads) {
          const int e0 = t_inptr[i], e1 = t_inptr[i + 1];
          if (e1 == e0) continue;
          const float gi = NG[i], sn = Sown[i];
          const bool ex = sn > -CUDART_INF_F;
          const float e = ldg_elem(er + t_lab[i]);
          float acc = 0.0f;
#pragma unroll 1
          for (int a = e0; a < e1; a++) {
            const float c = ex ? gi * fexp(Sprev[t_src[a]] + (t_w[a] + e) - sn) : 0.0f;
            CURa[a] = c;
            acc += c;
            if (GRAPH_GRAD) ACCG[a] += c; // entry a belongs to this thread only
          }
          if (acc != 0.0f) atomicAdd(gr + t_lab[i], acc * delta);
        }
      }
      __syncthreads();
      if (ARC) flush_erow_grad(GE, gr, C, delta);
      for (int u = tid; u < N1; u += kImpThreads) {
        float gn = 0.0f;
#pragma unroll 1
        for (int q = t_outptr[u]; q < t_outptr[u + 1]; q++) gn += CURa[t_outent[q]];
        NG[u] = gn;
      }
      float* ts = Sown;
      Sown = Sprev;
      Sprev = ts;
      // the next iteration's first barrier orders NG / Sprev writes before their reads
    }
    if (GRAPH_GRAD) {
      __syncthreads();
      for (int a = tid; a < A1; a += kImpThreads)
        if (ACCG[a] != 0.0f) atomicAdd(&ggr[in_arc[a]], ACCG[a] * delta);
    }
  }
}


/* ------------------------------------------------------------------ */
/* wide graphs (in-/out-degree > 3, e.g. the dense ASG transitions):   */
/* G lanes per node, each holding up to kWideCap arcs in registers     */
/* ------------------------------------------------------------------ */

constexpr int kWideCap = 20;

/* packed {source, weight bits} per in-entry; compact lists of the nodes that have in-arcs
 * (t_act[0..n), n at t_act[N1]) and, for the backward, out-arcs (t_acto likewise) */
__device__ __forceinline__ void build_wide_tables(
    int N1, int A1, const int* t_inptr, const int* t_src, const float* t_w, const int* t_outptr, int2* t_sw,
    int* t_act, int* t_acto) {
  const int tid = threadIdx.x;
  for (int a = tid; a < A1; a += kImpThreads) t_sw[a] = make_int2(t_src[a], __float_as_int(t_w[a]));
  if (tid == 0) {
    int n = 0;
    for (int u = 0; u < N1; u++)
      if (t_inptr[u + 1] > t_inptr[u]) t_act[n++] = u;
    t_act[N1] = n;
  }
  if (tid == 32 && t_outptr) {
    int n = 0;
    for (int u = 0; u < N1; u++)
      if (t_outptr[u + 1] > t_outptr[u]) t_acto[n++] = u;
    t_acto[N1] = n;
  }
  __syncthreads();
}

template <int G>
__device__ __forceinline__ unsigned group_mask() {
  return (G >= 32) ? 0xffffffffu : (((1u << G) - 1u) << ((threadIdx.x & 31) & ~(G - 1)));
}

template <int G, bool ARC = false, bool TROP = false>
__global__ void __launch_bounds__(kImpThreads) implicit_forward_wide_kernel(
    const GraphMeta* __restrict__ meta,
    const uint8_t* __restrict__ sg_flags,
    const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ sg_in_src,
    const int32_t* __restrict__ sg_in_label,
    const float* __restrict__ sg_in_w,
    const float* __restrict__ emissions,
    float* __restrict__ scores,
    float* __restrict__ out_scores,
    int32_t* __restrict__ status,
    int C,
    const ImpLayout lay) {
  GTNB_DYNAMIC_SMEM(unsigned char, smem);
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x;
  const int N1 = m.sg_N, A1 = m.sg_A, T = m.T;
  const int pitch = (N1 + 3) & ~3;
  float* S = reinterpret_cast<float*>(smem + lay.off_S);
  int* t_inptr = reinterpret_cast<int*>(smem + lay.off_inptr);
  int* t_src = reinterpret_cast<int*>(smem + lay.off_src);
  float* t_w = reinterpret_cast<float*>(smem + lay.off_w);
  int* t_lab = reinterpret_cast<int*>(smem + lay.off_lab);
  unsigned char* t_flags = smem + lay.off_flags;
  float* red = reinterpret_cast<float*>(smem + lay.off_red);
  int2* t_sw = reinterpret_cast<int2*>(smem + lay.off_sw);
  int* t_act = reinterpret_cast<int*>(smem + lay.off_act);
  float* E_s = reinterpret_cast<float*>(smem + lay.off_erow); // [2][C]: emission rows, one frame ahead

  bool bad = load_tables(m, sg_flags, sg_in_ptr, sg_in_src, sg_in_label, sg_in_w, t_inptr, t_src, t_w,
                         t_lab, t_flags);
  int* t_alab = reinterpret_cast<int*>(smem + lay.off_alab); // ARC only
  if (ARC) load_arc_labels(m, sg_in_label, t_alab);
  build_wide_tables(N1, A1, t_inptr, t_src, t_w, nullptr, t_sw, t_act, nullptr);
  float* sc = scores + m.node_base;
  const float* em = emissions + m.emis_off;
  float* prev = S;
  float* cur = S + lay.pitch;
  for (int i = tid; i < N1; i += kImpThreads) {
    const float v = (t_flags[i] & 1) ? 0.0f : neg_inf();
    prev[i] = v;
    sc[i] = v;
  }
  if (ARC) {
    if (T > 0) bad |= stage_erow(em, E_s, C);
  } else if (T > 0 && tid < C) {
    const float e0v = __ldg(em + tid);
    E_s[tid] = e0v;
    bad |= !is_finite(e0v);
  }
  __syncthreads();

  constexpr int kSlots = kImpThreads / G;
  const int sub = tid % G, slot0 = tid / G;
  const unsigned gmask = group_mask<G>();
  const int n_act = t_act[N1];
  const int rounds = (n_act + kSlots - 1) / kSlots;
  for (int t = 1; t <= T; t++) {
    const float* Ecur = E_s + ((t - 1) & 1) * C;
    float* Enext = E_s + (t & 1) * C;
    const bool ld = (t < T) && tid < C; // next frame's emissions: in flight during this level
    float enext = 0.0f;
    if (!ARC && ld) enext = __ldg(em + (long long)t * C + tid);
    float en[kArcRows]; // ARC: the next frame's row, kArcRows values per thread
    if (ARC) {
#pragma unroll
      for (int k = 0; k < kArcRows; k++) {
        const int c = tid + k * kImpThreads;
        en[k] = (t < T && c < C) ? __ldg(em + (long long)t * C + c) : 0.0f;
      }
    }
    float* srow = sc + (long long)t * pitch;
    for (int r = 0; r < rounds; r++) {
      const int slot = r * kSlots + slot0;
      const bool on = slot < n_act;
      const int u = on ? t_act[slot] : 0;
      const int e0 = on ? t_inptr[u] : 0, e1 = on ? t_inptr[u + 1] : 0;
      const float e = (!ARC && on) ? Ecur[t_lab[u]] : 0.0f;
      float v[kWideCap];
      float mx = neg_inf();
#pragma unroll
      for (int k = 0; k < kWideCap; k++) {
        const int a = e0 + sub + k * G;
        v[k] = neg_inf();
        if (a < e1) {
          const int2 sw = t_sw[a];
          v[k] = prev[sw.x] + (__int_as_float(sw.y) + (ARC ? Ecur[t_alab[a]] : e));
        }
        mx = fmaxf(mx, v[k]);
      }
#pragma unroll
      for (int o = G / 2; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(gmask, mx, o));
      float sv = mx;
      if (!TROP) {
        float sum = 0.0f;
#pragma unroll
        for (int k = 0; k < kWideCap; k++) sum += fexp(v[k] - mx);
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(gmask, sum, o);
        const float lg = lg2(sum);
        sv = (fabsf(mx) == CUDART_INF_F) ? mx : fmaf(lg, 0.6931471805599453f, mx);
      }
      if (on && sub == 0) {
        cur[u] = sv;
        srow[u] = sv;
      }
    }
    // a node without in-arcs does not exist past frame 0
    for (int i = tid; i < N1; i += kImpThreads)
      if (t_inptr[i + 1] == t_inptr[i]) {
        cur[i] = neg_inf();
        srow[i] = neg_inf();
      }
    if (!ARC && ld) {
      Enext[tid] = enext;
      bad |= !is_finite(enext);
    }
    if (ARC) {
#pragma unroll
      for (int k = 0; k < kArcRows; k++) {
        const int c = tid + k * kImpThreads;
        if (t < T && c < C) {
          Enext[c] = en[k];
          bad |= !is_finite(en[k]);
        }
      }
    }
    float* tmp = prev;
    prev = cur;
    cur = tmp;
    __syncthreads();
  }

  // accept nodes of the last frame (shortest.cpp:147-159); `prev` is the last row written
  const float* Sf = prev;
  float mx = neg_inf();
  for (int i = tid; i < N1; i += kImpThreads)
    if (t_flags[i] & 2) mx = fmaxf(mx, Sf[i]);
  mx = block_max(mx, red);
  float out = mx;
  if (!TROP && mx != CUDART_INF_F && mx != -CUDART_INF_F) {
    float sum = 0.0f;
    for (int i = tid; i < N1; i += kImpThreads)
      if (t_flags[i] & 2) sum += expf(Sf[i] - mx);
    sum = block_sum(sum, red);
    out = mx + log1pf(sum - 1.0f);
  }
  if (tid == 0) out_scores[blockIdx.x] = out;
  if (bad) atomicOr(&status[blockIdx.x], 1);
}

template <int G, bool GRAPH_GRAD, bool ARC = false>
__global__ void __launch_bounds__(kImpThreads) implicit_backward_wide_kernel(
    const GraphMeta* __restrict__ meta,
    const uint8_t* __restrict__ sg_flags,
    const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ sg_in_src,
    const int32_t* __restrict__ sg_in_label,
    const float* __restrict__ sg_in_w,
    const int32_t* __restrict__ sg_in_arc,
    float* __restrict__ grad_graph,
    const float* __restrict__ emissions,
    const float* __restrict__ scores,
    const float* __restrict__ out_scores,
    const float* __restrict__ deltas,
    float* __restrict__ grad_emis,
    long long grad_stride,
    int C,
    const ImpLayout lay) {
  GTNB_DYNAMIC_SMEM(unsigned char, smem);
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x;
  const int N1 = m.sg_N, A1 = m.sg_A, T = m.T;
  const int pitch = (N1 + 3) & ~3;
  int* t_inptr = reinterpret_cast<int*>(smem + lay.off_inptr);
  int* t_src = reinterpret_cast<int*>(smem + lay.off_src);
  float* t_w = reinterpret_cast<float*>(smem + lay.off_w);
  int* t_lab = reinterpret_cast<int*>(smem + lay.off_lab);
  unsigned char* t_flags = smem + lay.off_flags;
  float* red = reinterpret_cast<float*>(smem + lay.off_red);
  int* t_outptr = reinterpret_cast<int*>(smem + lay.off_outptr);
  int* t_outent = reinterpret_cast<int*>(smem + lay.off_outent);
  int* t_cursor = reinterpret_cast<int*>(smem + lay.off_cursor);
  float* CUR = reinterpret_cast<float*>(smem + lay.off_cur);
  float* NG = reinterpret_cast<float*>(smem + lay.off_ng);
  float* ACCG = reinterpret_cast<float*>(smem + lay.off_accg);
  int2* t_sw = reinterpret_cast<int2*>(smem + lay.off_sw);
  int* t_act = reinterpret_cast<int*>(smem + lay.off_act);
  int* t_acto = t_act + lay.tabN;
  float* E_s = reinterpret_cast<float*>(smem + lay.off_erow);
  float* R3 = reinterpret_cast<float*>(smem + lay.off_rows3); // three score rows: t, t-1, staging
  const int32_t* in_arc = sg_in_arc + m.sg_arc_base;
  float* ggr = GRAPH_GRAD ? grad_graph + m.grad_graph_off : nullptr;

  load_tables(m, sg_flags, sg_in_ptr, sg_in_src, sg_in_label, sg_in_w, t_inptr, t_src, t_w, t_lab, t_flags);
  int* t_alab = reinterpret_cast<int*>(smem + lay.off_alab); // ARC only
  float* GE = reinterpret_cast<float*>(smem + lay.off_ge); // ARC only: frame t-1's emission gradient per label
  if (ARC) load_arc_labels(m, sg_in_label, t_alab);
  build_out_lists(N1, A1, t_src, t_outptr, t_outent, t_cursor);
  build_wide_tables(N1, A1, t_inptr, t_src, t_w, t_outptr, t_sw, t_act, t_acto);

  const float out = out_scores[blockIdx.x];
  if (!is_finite(out) || T < 1) return; // no accepting path (empty lattice): no gradient
  const float delta = deltas ? deltas[blockIdx.x] : 1.0f;
  const float* sc = scores + m.node_base;
  const float* em = emissions + m.emis_off;
  float* gem = grad_emis + (long long)blockIdx.x * grad_stride;

  float mxa = neg_inf();
  for (int i = tid; i < N1; i += kImpThreads)
    if (t_flags[i] & 2) mxa = fmaxf(mxa, sc[(long long)T * pitch + i]);
  mxa = block_max(mxa, red);
  const float denom = expf(out - mxa);

  float* own = R3; // row t
  float* prv = R3 + lay.pitch; // row t-1
  float* nxt = R3 + 2 * lay.pitch; // row t-2, staged during level t
  for (int i = tid; i < N1; i += kImpThreads) {
    const float sT = sc[(long long)T * pitch + i];
    own[i] = sT;
    prv[i] = sc[(long long)(T - 1) * pitch + i];
    NG[i] = (t_flags[i] & 2) ? expf(sT - mxa) / denom : 0.0f; // shortest.cpp:49-60
  }
  if (GRAPH_GRAD)
    for (int a = tid; a < A1; a += kImpThreads) ACCG[a] = 0.0f;
  if (ARC) {
    stage_erow(em + (long long)(T - 1) * C, E_s + ((T - 1) & 1) * C, C);
    for (int c = tid; c < C; c += kImpThreads) GE[c] = 0.0f;
  } else if (tid < C) {
    E_s[((T - 1) & 1) * C + tid] = __ldg(em + (long long)(T - 1) * C + tid);
  }
  __syncthreads();

  constexpr int kSlots = kImpThreads / G;
  const int sub = tid % G, slot0 = tid / G;
  const unsigned gmask = group_mask<G>();
  const int n_act = t_act[N1], n_acto = t_acto[N1];
  const int rounds = (n_act + kSlots - 1) / kSlots, rounds_o = (n_acto + kSlots - 1) / kSlots;
  for (int t = T; t >= 1; t--) {
    const float* Ecur = E_s + ((t - 1) & 1) * C; // frame t-1
    float* Enext = E_s + (t & 1) * C; // frame t-2 (same parity as t)
    const bool more = t >= 2;
    float snext = neg_inf(), enext = 0.0f; // in flight during this level
    if (more && tid < N1) snext = __ldg(sc + (long long)(t - 2) * pitch + tid);
    if (!ARC && more && tid < C) enext = __ldg(em + (long long)(t - 2) * C + tid);
    float en[kArcRows]; // ARC: frame t-2's row, kArcRows values per thread
    if (ARC) {
#pragma unroll
      for (int k = 0; k < kArcRows; k++) {
        const int c = tid + k * kImpThreads;
        en[k] = (more && c < C) ? __ldg(em + (long long)(t - 2) * C + c) : 0.0f;
      }
    }
    float* gr = gem + (long long)(t - 1) * C;
    // phase 1: arc gradients of level t (shortest.cpp:62-80), emission gradient per node (ARC: per label)
    for (int r = 0; r < rounds; r++) {
      const int slot = r * kSlots + slot0;
      const bool on = slot < n_act;
      const int u = on ? t_act[slot] : 0;
      const int e0 = on ? t_inptr[u] : 0, e1 = on ? t_inptr[u + 1] : 0;
      const int lab = on ? t_lab[u] : 0;
      const float e = (!ARC && on) ? Ecur[lab] : 0.0f;
      const float g = NG[u], sn = own[u];
      const float se = (sn == -CUDART_INF_F) ? CUDART_INF_F : sn; // missing node: factors exp(-inf)
      float acc = 0.0f;
#pragma unroll
      for (int k = 0; k < kWideCap; k++) {
        const int a = e0 + sub + k * G;
        if (a < e1) {
          const int2 sw = t_sw[a];
          const int alab = ARC ? t_alab[a] : 0;
          const float c = g * fexp(prv[sw.x] + (__int_as_float(sw.y) + (ARC ? Ecur[alab] : e)) - se);
          CUR[a] = c;
          acc += c;
          if (GRAPH_GRAD) ACCG[a] += c; // entry a belongs to this lane only
          if (ARC && c != 0.0f) atomicAdd(&GE[alab], c); // shared: one global add per label and frame below
        }
      }
      if (!ARC) {
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(gmask, acc, o);
        if (on && sub == 0 && acc != 0.0f) atomicAdd(gr + lab, acc * delta);
      }
    }
    __syncthreads();
    if (ARC) flush_erow_grad(GE, gr, C, delta);
    // phase 2: node gradients of frame t-1, gathered over the out-arcs
    for (int r = 0; r < rounds_o; r++) {
      const int slot = r * kSlots + slot0;
      const bool on = slot < n_acto;
      const int u = on ? t_acto[slot] : 0;
      const int o0 = on ? t_outptr[u] : 0, o1 = on ? t_outptr[u + 1] : 0;
      float sum = 0.0f;
#pragma unroll
      for (int k = 0; k < kWideCap; k++) {
        const int q = o0 + sub + k * G;
        if (q < o1) sum += CUR[t_outent[q]];
      }
#pragma unroll
      for (int o = G / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(gmask, sum, o);
      if (on && sub == 0) NG[u] = sum;
    }
    for (int i = tid; i < N1; i += kImpThreads)
      if (t_outptr[i + 1] == t_outptr[i]) NG[i] = 0.0f;
    if (tid < N1) nxt[tid] = snext;
    if (!ARC && more && tid < C) Enext[tid] = enext;
    if (ARC) {
#pragma unroll
      for (int k = 0; k < kArcRows; k++) {
        const int c = tid + k * kImpThreads;
        if (more && c < C) Enext[c] = en[k];
      }
    }
    float* tmp = own;
    own = prv;
    prv = nxt;
    nxt = tmp;
    __syncthreads();
  }
  if (GRAPH_GRAD)
    for (int a = tid; a < A1; a += kImpThreads)
      if (ACCG[a] != 0.0f) atomicAdd(&ggr[in_arc[a]], ACCG[a] * delta);
}

/* ------------------------------------------------------------------ */
/* Viterbi traceback of a tropical forward sweep (any variant above)   */
/* ------------------------------------------------------------------ */

constexpr int kTrMaxFrames = 16; // frames of score and emission rows per staged block
constexpr int kTrSmemTarget = 96 * 1024; // the block shrinks until the CTA fits two per SM
constexpr int kTrTie = 2; // status bit beside the non-finite bit 1: a tie on the traced path
constexpr int kTrLoads = 8; // staging loads in flight per thread

struct TraceLayout {
  int K; // frames per staged block
  int pitch; // floats per staged score row (max over the batch, multiple of 4)
  int off_inptr, off_src, off_w, off_lab, off_arc, off_red, off_buf;
  int total;
};

TraceLayout make_trace_layout(int maxN, int maxA, int C, int K) {
  TraceLayout o;
  o.K = K;
  o.pitch = (maxN + 3) & ~3;
  const int A = std::max(maxA, 1);
  int off = 0;
  auto take = [&](long long bytes) {
    int at = off;
    off += (int)((bytes + 15) & ~15ll);
    return at;
  };
  o.off_inptr = take(4ll * (maxN + 2));
  o.off_src = take(4ll * A);
  o.off_w = take(4ll * A);
  o.off_lab = take(4ll * A);
  o.off_arc = take(4ll * A);
  o.off_red = take(4 * 16);
  o.off_buf = take(4ll * 2 * K * (o.pitch + C)); // two blocks: K score rows, then K emission rows
  o.total = off;
  return o;
}

/*
 * viterbiPath of intersect(A_b, E_b) from the score rows a TROP forward saved, without back-pointers: at node v of
 * frame t every in-arc's candidate fl(S_{t-1}[src] + fl(w + e[t-1][label])) is recomputed exactly as the forward
 * computed it, and the in-arc whose candidate == S_t[v] is taken.  One CTA per utterance; warp 0 walks a block of
 * K frames held in shared memory while the other warps stage the next block with independent loads, so the
 * dependent chain of T_b steps pays shared-memory latency, not a global load per frame.
 * Outputs: paths / arcs (nullable, [B][T_out]): the matched label and the graph arc of the in-arc taken at every
 * frame, -1 beyond T_b and everywhere without an accepting path; out_scores [B]: viterbiScore (-inf for T_b = 0:
 * linearGraph(0, C) accepts nothing).  Status: kTrTie when two accept nodes share the best score at frame T_b or two
 * candidates reach the maximum at a node of the path (the reference breaks such ties by its own arc order, which the
 * caller reproduces on the materialised route); bit 1 for a score of +inf / NaN.  Only nodes of the traced path are
 * visited, and every predecessor of one lies on an accepting path, so nodes the reference prunes play no part.
 */
__global__ void __launch_bounds__(kImpThreads) implicit_trace_kernel(
    const GraphMeta* __restrict__ meta,
    const uint8_t* __restrict__ sg_flags,
    const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ sg_in_src,
    const int32_t* __restrict__ sg_in_label,
    const float* __restrict__ sg_in_w,
    const int32_t* __restrict__ sg_in_arc,
    const float* __restrict__ emissions,
    const float* __restrict__ scores,
    int32_t* __restrict__ status,
    int32_t* __restrict__ paths,
    int32_t* __restrict__ arcs,
    float* __restrict__ out_scores,
    int T_out,
    int C,
    const TraceLayout lay) {
  GTNB_DYNAMIC_SMEM(unsigned char, smem);
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31;
  const int N1 = m.sg_N, A1 = m.sg_A, T = m.T, K = lay.K;
  const int pitch = (N1 + 3) & ~3;
  int* t_inptr = reinterpret_cast<int*>(smem + lay.off_inptr);
  int* t_src = reinterpret_cast<int*>(smem + lay.off_src);
  float* t_w = reinterpret_cast<float*>(smem + lay.off_w);
  int* t_lab = reinterpret_cast<int*>(smem + lay.off_lab);
  int* t_arc = reinterpret_cast<int*>(smem + lay.off_arc);
  float* red = reinterpret_cast<float*>(smem + lay.off_red);
  float* buf = reinterpret_cast<float*>(smem + lay.off_buf);
  const int bstride = K * (lay.pitch + C);
  const float* sc = scores + m.node_base;
  const float* em = emissions + m.emis_off;
  int32_t* po = paths ? paths + (long long)blockIdx.x * T_out : nullptr;
  int32_t* ao = arcs ? arcs + (long long)blockIdx.x * T_out : nullptr;

  for (int i = tid; i <= N1; i += kImpThreads) t_inptr[i] = sg_in_ptr[m.sg_node_base + i];
  for (int a = tid; a < A1; a += kImpThreads) {
    t_src[a] = sg_in_src[m.sg_arc_base + a];
    t_w[a] = sg_in_w[m.sg_arc_base + a];
    t_lab[a] = sg_in_label[m.sg_arc_base + a];
    t_arc[a] = sg_in_arc[m.sg_arc_base + a];
  }
  // the best accept node of frame T_b (shortest.cpp:147-159), the first of them, and how many share its score
  const float* sT = sc + (long long)T * pitch;
  const uint8_t* fl = sg_flags + m.sg_node_base;
  float mx = neg_inf();
  for (int i = tid; i < N1; i += kImpThreads)
    if (fl[i] & 2) mx = fmaxf(mx, sT[i]);
  mx = block_max(mx, red); // (its barriers also order the table writes above)
  float first = neg_inf(), n_best = 0.0f; // -(node id), exact in a float
  for (int i = tid; i < N1; i += kImpThreads)
    if ((fl[i] & 2) && sT[i] == mx) {
      first = fmaxf(first, -(float)i);
      n_best += 1.0f;
    }
  first = block_max(first, red);
  n_best = block_sum(n_best, red);
  const bool found = T > 0 && is_finite(mx);
  if (tid == 0) {
    out_scores[blockIdx.x] = T > 0 ? mx : neg_inf();
    const int st = ((T > 0 && mx != -CUDART_INF_F && !found) ? 1 : 0) | ((found && n_best > 1.0f) ? kTrTie : 0);
    if (st) atomicOr(&status[blockIdx.x], st);
  }
  for (int t = (found ? T : 0) + tid; t < T_out; t += kImpThreads) {
    if (po) po[t] = -1;
    if (ao) ao[t] = -1;
  }
  if (!found) return;

  // n rows of `width` floats (the first `valid` read, the rest 0) -> shared memory, kTrLoads independent loads in
  // flight per thread: one load at a time would make the staging warps, not the walk, set the pace
  auto copy_rows = [&](float* dst, int dpitch, const float* src, int spitch, int width, int valid, int n, int first,
                       int nthr) {
    const int total = n * width;
    for (int base = tid - first; base < total; base += kTrLoads * nthr) {
      float v[kTrLoads];
#pragma unroll
      for (int u = 0; u < kTrLoads; u++) {
        const int idx = base + u * nthr, k = idx / width, i = idx - k * width;
        v[u] = (idx < total && i < valid) ? __ldg(src + (long long)k * spitch + i) : 0.0f;
      }
#pragma unroll
      for (int u = 0; u < kTrLoads; u++) {
        const int idx = base + u * nthr, k = idx / width, i = idx - k * width;
        if (idx < total) dst[k * dpitch + i] = v[u];
      }
    }
  };
  // block j holds frames [max(0, T - (j+1)K), T - jK) in buffer j & 1
  auto stage = [&](int j, int first, int nthr) {
    const int fhi = T - j * K, flo = max(0, fhi - K), n = fhi - flo;
    float* ds = buf + (j & 1) * bstride;
    copy_rows(ds, lay.pitch, sc + (long long)flo * pitch, pitch, pitch, N1, n, first, nthr);
    copy_rows(ds + K * lay.pitch, C, em + (long long)flo * C, C, C, C, n, first, nthr);
  };
  const int nblk = (T + K - 1) / K;
  stage(0, 0, kImpThreads);
  __syncthreads();
  const int v = (int)-first;
  float s = mx;
  int e0 = t_inptr[v], e1 = t_inptr[v + 1]; // the in-entries of v, fetched one step ahead by the lane that picks v
  bool tie = false, lost = false;
  for (int j = 0; j < nblk; j++) {
    if (tid < 32) {
      const int fhi = T - j * K, flo = max(0, fhi - K);
      const float* blk = buf + (j & 1) * bstride;
      for (int f = fhi - 1; f >= flo; f--) {
        const float* Srow = blk + (f - flo) * lay.pitch;
        const float* Erow = blk + K * lay.pitch + (f - flo) * C;
        int pick = -1, hits = 0, n0 = e0, n1 = e0;
        float ns = s;
        for (int base = e0; base < e1; base += 32) {
          const int a = base + lane;
          int p0 = 0, p1 = 0;
          float sp = neg_inf();
          bool hit = false;
          if (a < e1) {
            const int src = t_src[a];
            sp = Srow[src];
            p0 = t_inptr[src];
            p1 = t_inptr[src + 1];
            hit = sp + (t_w[a] + Erow[t_lab[a]]) == s; // the forward's association, bit for bit
          }
          const unsigned mk = __ballot_sync(0xffffffffu, hit);
          hits += __popc(mk);
          if (pick < 0 && mk) {
            const int l = __popc((mk & (0u - mk)) - 1u); // the lowest hit lane
            pick = base + l;
            ns = __shfl_sync(0xffffffffu, sp, l);
            n0 = __shfl_sync(0xffffffffu, p0, l);
            n1 = __shfl_sync(0xffffffffu, p1, l);
          }
        }
        tie |= hits > 1;
        lost |= hits == 0; // (cannot happen with finite values; the caller re-runs the utterance if it does)
        if (lane == 0) {
          if (po) po[f] = pick < 0 ? -1 : t_lab[pick];
          if (ao) ao[f] = pick < 0 ? -1 : t_arc[pick];
        }
        s = ns;
        e0 = n0;
        e1 = n1;
      }
    } else if (j + 1 < nblk) {
      stage(j + 1, 32, kImpThreads - 32);
    }
    __syncthreads();
  }
  if (tid == 0 && (tie || lost)) atomicOr(&status[blockIdx.x], (tie ? kTrTie : 0) | (lost ? 1 : 0));
}

} // namespace

namespace {

/* 0: one node per thread / several nodes per thread (implicit_*_kernel decides per CTA);
 * otherwise the lanes per node of the wide kernels (arc-label mode: C up to kArcMaxLabels) */
int wide_lanes(int max_in, int max_out, int maxN, int C, bool backward, bool arc = false) {
  const int deg = backward ? std::max(max_in, max_out) : max_in;
  if (deg <= 3 || maxN > kImpThreads || C > (arc ? kArcMaxLabels : kImpThreads)) return 0;
  int G = 1;
  while (G < 32 && (deg + G - 1) / G > kWideCap) G *= 2;
  if ((deg + G - 1) / G > kWideCap) return 0;
  return G;
}

} // namespace

/* GTNB_OK when a lattice of element type dtype may take the mode (G: wide_lanes; arc-label; tropical), else
 * GTNB_ERR_LOGIC: 16-bit emissions have instantiations of the one-node / several-nodes-per-thread log-semiring sweeps
 * of label-uniform graphs only (the trellis criteria's numerators), and no other kernel may read them as float32 */
int implicit_elem_mode(int dtype, int G, bool arc, bool tropical) {
  if (dtype == GTNB_F32) return GTNB_OK;
  return (dtype == GTNB_BF16 || dtype == GTNB_F16) && G == 0 && !arc && !tropical ? GTNB_OK : GTNB_ERR_LOGIC;
}

#ifndef GTNB_HOST_EMU

/* arc_C > 0 (gtnb_graph_loss, labels in [0, arc_C)): graphs that are not label-uniform are accepted
 * and take the arc-label kernels, which need C <= kArcMaxLabels and the larger layout */
bool implicit_dims_supported(const SgDims* dims, int n_graphs, int arc_C) {
  int maxN = 0, maxA = 0;
  bool arc = false;
  for (int g = 0; g < n_graphs; g++) {
    if (!dims[g].all_valid) return false;
    if (!dims[g].uniform) {
      if (arc_C <= 0) return false;
      arc = true;
    }
    maxN = std::max(maxN, dims[g].N);
    maxA = std::max(maxA, dims[g].A);
  }
  if (arc && arc_C > kArcMaxLabels) return false;
  return make_imp_layout(maxN, maxA, true, true, arc ? arc_C : kImpThreads, arc).total <= 200 * 1024;
}

/* true when every graph of the batch can take the implicit path */
bool implicit_supported(const gtnb_lattice* lat) {
  if (!lat->composed) return false;
  for (int b = 0; b < lat->B; b++)
    if (!lat->meta_h[b].sg_uniform || !lat->meta_h[b].sg_all_valid) return false;
  const ImpLayout lay = make_imp_layout(lat->max_lvl_nodes, lat->max_lvl_arcs, true, true, kImpThreads);
  return lay.total <= 200 * 1024;
}

// E: the element type the kernel reads lat->emissions as
#define GTNB_FWD_ARGS(E)                                                                          \
  lat->meta + b0, lat->sg_flags, lat->sg_in_ptr, lat->sg_in_src, lat->sg_in_label, lat->sg_in_w, \
      reinterpret_cast<const E*>(lat->emissions), lat->scores, lat->out_scores + b0, status_dev + b0, lat->C, lay
#define GTNB_BWD_ARGS(E)                                                                          \
  lat->meta + b0, lat->sg_flags, lat->sg_in_ptr, lat->sg_in_src, lat->sg_in_label, lat->sg_in_w, \
      lat->sg_in_arc, grad_graph, reinterpret_cast<const E*>(lat->emissions), lat->scores,       \
      lat->out_scores + b0, deltas_dev ? deltas_dev + b0 : nullptr,                               \
      grad_emis + (long long)b0 * grad_stride, (long long)grad_stride, lat->C, lay

namespace {

/* the launch of one mode; the arc-label instantiations carry their own names in the profile log */
template <bool ARC, bool TROP>
int implicit_forward_mode(gtnb_ctx* ctx, gtnb_lattice* lat, int32_t* status_dev, int b0, int nb) {
  const int G = wide_lanes(lat->max_in_deg, lat->max_out_deg, lat->max_lvl_nodes, lat->C, false, ARC);
  const ImpLayout lay = make_imp_layout(lat->max_lvl_nodes, lat->max_lvl_arcs, false, G > 0, lat->C, ARC);
  const char* name = ARC ? (TROP ? "implicit_forward_arc_max" : "implicit_forward_arc")
                         : (TROP ? "implicit_forward_max" : "implicit_forward");
  if (implicit_elem_mode(lat->dtype, G, ARC, TROP))
    return fail(ctx, GTNB_ERR_LOGIC, "launch_implicit_forward: no instantiation for 16-bit emissions in this mode");
#define GTNB_LAUNCH_FWD_E(K, E)                                                                  \
  do {                                                                                           \
    if (lay.total > 48 * 1024) {                                                                 \
      int rc = ensure_max_smem(ctx, (const void*)K);                                             \
      if (rc) return rc;                                                                         \
    }                                                                                            \
    GTNB_LAUNCH(ctx, name, K<<<nb, kImpThreads, lay.total, ctx->stream>>>(GTNB_FWD_ARGS(E)));    \
  } while (0)
#define GTNB_LAUNCH_FWD(K) GTNB_LAUNCH_FWD_E(K, float)
  switch (G) {
    case 0:
      if constexpr (!ARC && !TROP) {
        if (lat->dtype == GTNB_BF16) {
          GTNB_LAUNCH_FWD_E((implicit_forward_kernel<false, false, bf16_t>), bf16_t);
          break;
        }
        if (lat->dtype == GTNB_F16) {
          GTNB_LAUNCH_FWD_E((implicit_forward_kernel<false, false, f16_t>), f16_t);
          break;
        }
      }
      GTNB_LAUNCH_FWD((implicit_forward_kernel<ARC, TROP>));
      break;
    case 1: GTNB_LAUNCH_FWD((implicit_forward_wide_kernel<1, ARC, TROP>)); break;
    case 2: GTNB_LAUNCH_FWD((implicit_forward_wide_kernel<2, ARC, TROP>)); break;
    case 4: GTNB_LAUNCH_FWD((implicit_forward_wide_kernel<4, ARC, TROP>)); break;
    case 8: GTNB_LAUNCH_FWD((implicit_forward_wide_kernel<8, ARC, TROP>)); break;
    case 16: GTNB_LAUNCH_FWD((implicit_forward_wide_kernel<16, ARC, TROP>)); break;
    default: GTNB_LAUNCH_FWD((implicit_forward_wide_kernel<32, ARC, TROP>)); break;
  }
#undef GTNB_LAUNCH_FWD
#undef GTNB_LAUNCH_FWD_E
  return GTNB_OK;
}

template <bool ARC>
int implicit_backward_mode(
    gtnb_ctx* ctx, gtnb_lattice* lat, const float* deltas_dev, float* grad_emis, int64_t grad_stride,
    int b0, int nb, float* grad_graph) {
  const int G = wide_lanes(lat->max_in_deg, lat->max_out_deg, lat->max_lvl_nodes, lat->C, true, ARC);
  const ImpLayout lay = make_imp_layout(lat->max_lvl_nodes, lat->max_lvl_arcs, true, G > 0, lat->C, ARC);
  const char* name = ARC ? "implicit_backward_arc" : "implicit_backward";
  if (implicit_elem_mode(lat->dtype, G, ARC, false))
    return fail(ctx, GTNB_ERR_LOGIC, "launch_implicit_backward: no instantiation for 16-bit emissions in this mode");
#define GTNB_LAUNCH_BWD_E(K, E)                                                                  \
  do {                                                                                           \
    if (lay.total > 48 * 1024) {                                                                 \
      int rc = ensure_max_smem(ctx, (const void*)K);                                             \
      if (rc) return rc;                                                                         \
    }                                                                                            \
    GTNB_LAUNCH(ctx, name, K<<<nb, kImpThreads, lay.total, ctx->stream>>>(GTNB_BWD_ARGS(E)));    \
  } while (0)
#define GTNB_LAUNCH_BWD(K) GTNB_LAUNCH_BWD_E(K, float)
/* the one-node / several-nodes-per-thread kernel for lat->dtype */
#define GTNB_LAUNCH_BWD_0(GRAPH_GRAD_)                                                           \
  do {                                                                                           \
    if constexpr (!ARC) {                                                                        \
      if (lat->dtype == GTNB_BF16) {                                                             \
        GTNB_LAUNCH_BWD_E((implicit_backward_kernel<GRAPH_GRAD_, false, bf16_t>), bf16_t);       \
        break;                                                                                   \
      }                                                                                          \
      if (lat->dtype == GTNB_F16) {                                                              \
        GTNB_LAUNCH_BWD_E((implicit_backward_kernel<GRAPH_GRAD_, false, f16_t>), f16_t);         \
        break;                                                                                   \
      }                                                                                          \
    }                                                                                            \
    GTNB_LAUNCH_BWD((implicit_backward_kernel<GRAPH_GRAD_, ARC>));                               \
  } while (0)
#define GTNB_LAUNCH_BWD_G(GG)                                               \
  do {                                                                      \
    if (grad_graph)                                                         \
      GTNB_LAUNCH_BWD((implicit_backward_wide_kernel<GG, true, ARC>));      \
    else                                                                    \
      GTNB_LAUNCH_BWD((implicit_backward_wide_kernel<GG, false, ARC>));     \
  } while (0)
  switch (G) {
    case 0:
      if (grad_graph)
        GTNB_LAUNCH_BWD_0(true);
      else
        GTNB_LAUNCH_BWD_0(false);
      break;
    case 1: GTNB_LAUNCH_BWD_G(1); break;
    case 2: GTNB_LAUNCH_BWD_G(2); break;
    case 4: GTNB_LAUNCH_BWD_G(4); break;
    case 8: GTNB_LAUNCH_BWD_G(8); break;
    case 16: GTNB_LAUNCH_BWD_G(16); break;
    default: GTNB_LAUNCH_BWD_G(32); break;
  }
#undef GTNB_LAUNCH_BWD_0
#undef GTNB_LAUNCH_BWD_G
#undef GTNB_LAUNCH_BWD
#undef GTNB_LAUNCH_BWD_E
  return GTNB_OK;
}

} // namespace

/* utterances [b0, b0 + nb) of the batch (nb < 0: all): one CTA each, on ctx->stream */
int launch_implicit_forward(gtnb_ctx* ctx, gtnb_lattice* lat, int32_t* status_dev, int b0, int nb, bool tropical) {
  if (nb < 0) nb = lat->B - b0;
  if (nb <= 0) return GTNB_OK;
  if (tropical)
    return lat->arc_labels ? implicit_forward_mode<true, true>(ctx, lat, status_dev, b0, nb)
                           : implicit_forward_mode<false, true>(ctx, lat, status_dev, b0, nb);
  return lat->arc_labels ? implicit_forward_mode<true, false>(ctx, lat, status_dev, b0, nb)
                         : implicit_forward_mode<false, false>(ctx, lat, status_dev, b0, nb);
}

namespace {
/* the staged block of the traceback: kTrMaxFrames frames, halved until the CTA fits two per SM */
TraceLayout trace_layout(const gtnb_lattice* lat) {
  TraceLayout lay = make_trace_layout(lat->max_lvl_nodes, lat->max_lvl_arcs, lat->C, kTrMaxFrames);
  while (lay.K > 1 && lay.total > kTrSmemTarget)
    lay = make_trace_layout(lat->max_lvl_nodes, lat->max_lvl_arcs, lat->C, lay.K / 2);
  return lay;
}
} // namespace

bool implicit_trace_supported(const gtnb_lattice* lat) {
  return trace_layout(lat).total <= kMaxDynamicSmem;
}

int launch_implicit_trace(gtnb_ctx* ctx, gtnb_lattice* lat, int32_t* status_dev, int32_t* paths, int32_t* arcs,
                          float* scores_out, int T_out) {
  if (lat->B <= 0) return GTNB_OK;
  if (lat->dtype != GTNB_F32)
    return fail(ctx, GTNB_ERR_LOGIC, "launch_implicit_trace: no instantiation for 16-bit emissions");
  const TraceLayout lay = trace_layout(lat);
  if (lay.total > kMaxDynamicSmem) return fail(ctx, GTNB_ERR_UNSUPPORTED, "implicit_trace: graphs too large");
  if (lay.total > 48 * 1024) {
    int rc = ensure_max_smem(ctx, (const void*)implicit_trace_kernel);
    if (rc) return rc;
  }
  GTNB_LAUNCH(ctx, "implicit_trace",
              implicit_trace_kernel<<<lat->B, kImpThreads, lay.total, ctx->stream>>>(
                  lat->meta, lat->sg_flags, lat->sg_in_ptr, lat->sg_in_src, lat->sg_in_label, lat->sg_in_w,
                  lat->sg_in_arc, lat->emissions, lat->scores, status_dev, paths, arcs, scores_out, T_out, lat->C,
                  lay));
  return GTNB_OK;
}

/* grad_graph (may be NULL): gradients w.r.t. the graph operands' arc weights, slab of graph b at
 * meta[b].grad_graph_off (0 for a graph shared by the batch), accumulated with atomics */
int launch_implicit_backward(
    gtnb_ctx* ctx, gtnb_lattice* lat, const float* deltas_dev, float* grad_emis, int64_t grad_stride,
    int b0, int nb, float* grad_graph) {
  if (nb < 0) nb = lat->B - b0;
  if (nb <= 0) return GTNB_OK;
  return lat->arc_labels
             ? implicit_backward_mode<true>(ctx, lat, deltas_dev, grad_emis, grad_stride, b0, nb, grad_graph)
             : implicit_backward_mode<false>(ctx, lat, deltas_dev, grad_emis, grad_stride, b0, nb, grad_graph);
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
