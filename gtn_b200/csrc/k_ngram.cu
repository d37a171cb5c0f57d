/*
 * k_ngram.cu -- CTC with a learned bigram transition graph (gtnb_ngram_ctc_loss, the timeNgramCtc workload of
 * benchmarks/ctc.cpp:107-134) without building either lattice.
 *
 * G is the label-determined bigram graph: C nodes, every node start and accept, arc j -> i with label i and
 * weight W[i*C + j] (row = destination, column = source, ASG's layout).  Its state is the previous frame's label.
 *
 * Denominator, forwardScore(intersect(E, G)): a dense C-state trellis
 *     alpha_0 = 0,   alpha_t[i] = e[t-1][i] + logsumexp_j (alpha_{t-1}[j] + W[i][j]),   Z = logsumexp_i alpha_T[i]
 * (the C start states of G carry 0 at frame 0, so the first frame needs no special case).  One CTA per
 * utterance, W resident in registers for the whole utterance: the forward kernel holds K entries of one ROW
 * per thread (lanes_per_row threads per row, a shuffle reduction merges them), the backward kernel K entries
 * of one COLUMN (beta_{t-1}[j] = logsumexp_i (W[i][j] + e[t-1][i] + beta_t[i])).  The backward kernel also
 * sums the pair posteriors exp(alpha_{t-1}[j] + W[i][j] + e[t-1][i] + beta_t[i] - Z) over the frames in
 * registers and flushes them with one atomic per W entry per CTA.  Log semiring, exact per-thread maxima,
 * exp / log on the SFU (ex2.approx / lg2.approx): every sum has a term equal to 1, so nothing underflows to
 * zero whatever the spread of W or the emissions.
 *
 * Numerator, forwardScore(intersect(intersect(ctc, G), E)): every in-arc of CTC node l >= 1 carries label(l), so
 * the product is the CTC graph with arc weights W[label(dst)][label(src)], plus the C start states (0, s) of
 * which only (0, blank) survives frame 0.  Folding those into one start node S gives S -> ctc 0 (weight
 * sigma_blank) and S -> ctc 1 (sigma_y1), sigma_i = logsumexp_j W[i][j], d sigma_i / d W[i][j] =
 * softmax_j(W[i][:]).  ngram_num_build_kernel writes that graph (2U+2 nodes, <= 3 in-arcs each) into the
 * small-graph tables of an implicit lattice, plus an arc -> W-index map (C*C + i for the S arcs, which carry
 * sigma_i); the sweeps are k_implicit.cu's, and ngram_fold_kernel applies the sigma chain rule.
 *
 * Valid only for finite weights: the denominator's forward kernel raises a status bit on any non-finite W
 * entry or used emission, and the caller repeats the call through the materialised lattices.
 *
 * ASG (gtnb_asg_loss_ex) runs the same trellis in its START mode: the first frame starts from ASG's start weights,
 * alpha_1 = e[0] + s, and the rows are kept relative to per-frame offsets accumulated in double (see the forward
 * kernel).  Its numerator, compose(fal_b, transitions), is a U+1-node chain that asg_num_build_kernel writes into the
 * same small-graph tables for k_implicit.cu's sweeps; it needs no fold.
 *
 * Both trellis kernels take the element type E of the emissions as a template parameter (float, or bf16_t / f16_t for
 * gtnb_ngram_ctc_loss_typed / gtnb_asg_loss_typed): each element is widened to float32 exactly (prefetched as its
 * bits and widened where the frame uses it), the is_finite checks see the widened value, and everything after the
 * load is the float32 kernel's own.  The emission gradient stays float32; E = float compiles to the float32 kernels
 * as they were.
 */
#include <algorithm>

#include "gtnb_ptx.h"

namespace gtnb {

constexpr int kNgramMaxC = 128; // labels the trellis kernels hold on chip (K * lanes_per_row <= 128)
#ifndef GTNB_HOST_EMU
static_assert(kNgramMaxC == kNgramMaxLabels, "gtnb_internal.h states the same limit");
#endif
constexpr int kNgramMaxThreads = 512;

/* entries of W per thread and lanes per row (power of two) for an alphabet of C labels */
inline void ngram_den_shape(int C, int* K, int* lanes, int* threads) {
  *K = C <= 64 ? 16 : 32;
  int l = 1;
  while (l * *K < C) l *= 2;
  *lanes = l;
  *threads = (C * l + 31) & ~31;
}

/*
 * The start mode's alpha buffer (asg_den_* launchers): the alpha rows [B][(T+1)*C], then, 8-byte aligned, the
 * per-frame offsets [B][T+1] as doubles (slot 0: Z).
 */
long long asg_alpha_floats(int B, int T, int C) {
  return ((long long)B * (T + 1) * C + 1) / 2 * 2 + 2ll * B * (T + 1);
}

namespace {

/* (m, s) = logsumexp as max + sum of exp(x - max), merged over the `lanes` lanes of a row / column */
__device__ __forceinline__ void ng_merge(float& m, float& s, int lanes) {
  for (int o = 1; o < lanes; o <<= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const float os = __shfl_xor_sync(0xffffffffu, s, o);
    const float M = fmaxf(m, om);
    const float Mm = M == neg_inf() ? 0.0f : M; // all -inf: s stays 0
    s = s * exp_fast(m - Mm) + os * exp_fast(om - Mm);
    m = M;
  }
}

__device__ __forceinline__ double* asg_offsets(float* alpha, int B, int T, int C, int b) {
  return reinterpret_cast<double*>(alpha + ((long long)B * (T + 1) * C + 1) / 2 * 2) + (long long)b * (T + 1);
}

/*
 * alpha rows of every utterance to alpha[b][(T+1)*C], Z to den[b]; status[b] |= 1 on a non-finite weight.
 * START (ASG's denominator, forwardScore(compose(E, transitions))): W is ASG's [C + C*C] -- the start weights s,
 * then the C x C matrix -- and the first frame starts from them, alpha_1[i] = e[0][i] + s[i]; the recursion
 * through the matrix begins at t = 2.  Without START, alpha_0 = 0 and W is the C x C matrix alone.
 * START also keeps every row relative to an offset, alpha_t = row_t + c_t with c_t = c_{t-1} + row_{t-1}[0]
 * accumulated in double (asg_offsets; c_1 = 0): the stored rows stay within a frame's spread of scores, so the
 * backward kernel's posteriors exp(alpha + beta - Z) do not cancel fp32 scores that grow with t.
 */
template <int K, bool START = false, class E = float>
__global__ void __launch_bounds__(kNgramMaxThreads) ngram_den_forward_kernel(
    int T, int C, int lanes, const int32_t* __restrict__ lens, const E* __restrict__ emis, long long stride,
    const float* __restrict__ W, float* __restrict__ alpha, float* __restrict__ den, int32_t* __restrict__ status) {
  GTNB_STATIC_SMEM_2D(float, A, 2, kNgramMaxC);
  const int b = blockIdx.x, tid = threadIdx.x;
  const int Tb = lens[b];
  const int i = tid / lanes, q = tid % lanes;
  const bool row = i < C;
  const bool lead = row && q == 0;
  const E* em = emis + (long long)b * stride;
  const float* Wm = START ? W + C : W;
  float* al = alpha + (long long)b * (T + 1) * C;
  double* cs = START ? asg_offsets(alpha, gridDim.x, T, C, b) : nullptr;
  double c = 0.0; // START: the offset of the row in A[(t - 1) & 1]
  bool bad = false;
  float w[K]; // W[i][q + lanes * k]: interleaved columns, so the lanes of a row read distinct banks
#pragma unroll
  for (int k = 0; k < K; k++) {
    const int j = q + lanes * k;
    const bool on = row && j < C;
    w[k] = on ? __ldg(Wm + i * C + j) : neg_inf();
    if (on) bad |= !is_finite(w[k]);
  }
  float s_i = 0.0f;
  if (START && lead) {
    s_i = __ldg(W + i);
    bad |= !is_finite(s_i);
  }
  for (int j = tid; j < kNgramMaxC; j += blockDim.x) A[0][j] = A[1][j] = 0.0f; // alpha_0 = 0; padding stays 0
  for (int j = tid; j < C; j += blockDim.x) al[j] = 0.0f;
  __syncthreads();
  // the next frame's emission, one frame ahead; a 16-bit one stays in its bits until the frame uses it, so the
  // load is not waited for before the frame's barrier
  ring_t<E> e_nx = (lead && Tb > 0) ? ldg_ring(em + i) : ring_t<E>(0);
  if (START && Tb > 0) { // alpha_1 = e[0] + s
    const float e = ring_f32<E>(e_nx);
    if (lead && Tb > 1) e_nx = ldg_ring(em + C + i);
    bad |= !is_finite(e);
    if (lead) {
      const float v = e + s_i;
      A[1][i] = v;
      al[C + i] = v;
    }
    if (tid == 0) cs[1] = 0.0;
    __syncthreads();
  }
  for (int t = START ? 2 : 1; t <= Tb; t++) {
    const float e = ring_f32<E>(e_nx);
    if (lead && t < Tb) e_nx = ldg_ring(em + (long long)t * C + i);
    bad |= !is_finite(e);
    const float* P = A[(t - 1) & 1];
    float x[K];
    float m = neg_inf();
#pragma unroll
    for (int k = 0; k < K; k++) {
      x[k] = P[q + lanes * k] + w[k];
      m = fmaxf(m, x[k]);
    }
    const float mm = m == neg_inf() ? 0.0f : m;
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < K; k++) s += exp_fast(x[k] - mm);
    ng_merge(m, s, lanes);
    if (lead) {
      float v = e + (m + log_fast(s));
      if (START) v -= P[0];
      A[t & 1][i] = v;
      al[(long long)t * C + i] = v;
    }
    if (START) {
      c += (double)P[0];
      if (tid == 0) cs[t] = c;
    }
    __syncthreads();
  }
  bad = __syncthreads_or(bad);
  if (tid < 32) {
    const float* F = A[Tb & 1];
    float m = neg_inf();
    for (int j = tid; j < C; j += 32) m = fmaxf(m, F[j]);
    m = warp_max(m);
    float s = 0.0f;
    for (int j = tid; j < C; j += 32) s += expf(F[j] - m);
    s = warp_sum(s);
    if (tid == 0) {
      if (START) {
        const double Z = c + (double)(m + logf(s));
        cs[0] = Z;
        den[b] = (float)Z;
      } else {
        den[b] = m + logf(s);
      }
      if (bad) atomicOr(&status[b], 1);
    }
  }
}

/*
 * d Z / d e added into grad (rows t < T_b), d Z / d W added into wgrad[C*C] (one atomic per entry per CTA).
 * START: W and wgrad are ASG's [C + C*C]; the pair posteriors on the matrix run over t >= 2 only, and the
 * frame-1 node posteriors exp(alpha_1[i] + beta_1[i] - Z) are the start weights' gradient.  As in the forward
 * kernel, beta_t = row_t + d_t with d_{t-1} = d_t + G[0] in double (d_T = 0), and a posterior's exponent is
 * row + row' + (float)(c + d - Z).
 */
template <int K, bool START = false, class E = float>
__global__ void __launch_bounds__(kNgramMaxThreads) ngram_den_backward_kernel(
    int T, int C, int lanes, const int32_t* __restrict__ lens, const E* __restrict__ emis, long long stride,
    const float* __restrict__ W, const float* __restrict__ alpha, const float* __restrict__ den,
    float* __restrict__ grad, long long grad_stride, float* __restrict__ wgrad) {
  GTNB_STATIC_SMEM_2D(float, Bt, 2, kNgramMaxC); // beta_t, beta_{t-1}
  GTNB_STATIC_SMEM(float, G, kNgramMaxC); // e[t-1][i] + beta_t[i]; padding 0
  const int b = blockIdx.x, tid = threadIdx.x;
  const int Tb = lens[b];
  const float Z = den[b];
  if (!is_finite(Z) || Tb < 1) return; // (non-finite: the caller repeats the call materialised)
  const int j = tid / lanes, q = tid % lanes;
  const bool col = j < C;
  const bool lead = col && q == 0;
  const E* em = emis + (long long)b * stride;
  const float* al = alpha + (long long)b * (T + 1) * C;
  float* gr = grad + (long long)b * grad_stride;
  const float* Wm = START ? W + C : W;
  const double* cs = START ? asg_offsets(const_cast<float*>(alpha), gridDim.x, T, C, b) : nullptr;
  const double Zd = START ? cs[0] : 0.0;
  double d = 0.0, c_t = START ? cs[Tb] : 0.0, c_nx = (START && Tb > 1) ? cs[Tb - 1] : 0.0;
  float w[K], acc[K]; // W[q + lanes * k][j] and its pair posteriors
#pragma unroll
  for (int k = 0; k < K; k++) {
    const int i = q + lanes * k;
    w[k] = (col && i < C) ? __ldg(Wm + i * C + j) : neg_inf();
    acc[k] = 0.0f;
  }
  for (int i = tid; i < kNgramMaxC; i += blockDim.x) {
    Bt[Tb & 1][i] = 0.0f; // every node accepts: beta_T = 0
    G[i] = 0.0f;
  }
  // one frame of prefetch: alpha_t and e[t-1] of the rows this thread turns into G, alpha_{t-1} of its column
  const bool rowt = tid < C;
  float a_nx = rowt ? al[(long long)Tb * C + tid] : 0.0f;
  // the emission prefetch as in the forward kernel, but for ASG's start mode at K = 32: there the extra live register
  // of the 16 bits would spill 4 bytes more than the float32 kernel, so the element is widened where it is loaded
  constexpr bool kBits = !(START && K == 32);
  using Pf = std::conditional_t<kBits, ring_t<E>, float>;
  auto load_e = [&](long long k) -> Pf {
    if constexpr (kBits)
      return ldg_ring(em + k);
    else
      return ldg_elem(em + k);
  };
  auto use_e = [](Pf v) -> float {
    if constexpr (kBits)
      return ring_f32<E>(v);
    else
      return v;
  };
  Pf e_nx = rowt ? load_e((long long)(Tb - 1) * C + tid) : Pf(0);
  float aj_nx = col ? al[(long long)(Tb - 1) * C + j] : 0.0f;
  __syncthreads();
  for (int t = Tb; t >= 1; t--) {
    const float a_t = a_nx, e_t = use_e(e_nx), aj = aj_nx;
    const double c_prev = c_nx; // START: c_{t-1}
    if (t > 1) {
      if (rowt) {
        a_nx = al[(long long)(t - 1) * C + tid];
        e_nx = load_e((long long)(t - 2) * C + tid);
      }
      if (col) aj_nx = al[(long long)(t - 2) * C + j];
      if (START && t > 2) c_nx = cs[t - 2];
    }
    if (rowt) {
      const float bt = Bt[t & 1][tid];
      G[tid] = e_t + bt;
      const float p = exp_fast(START ? (a_t + bt) + (float)(c_t + d - Zd) : a_t + bt - Z); // node posterior
      atomicAdd(gr + (long long)(t - 1) * C + tid, p);
      if (START && t == 1) atomicAdd(wgrad + tid, p); // d Z / d s
    }
    if (START && t == 1) break; // (uniform) frame 1 has no transition through the matrix
    __syncthreads();
    float x[K];
    float m = neg_inf();
#pragma unroll
    for (int k = 0; k < K; k++) {
      x[k] = w[k] + G[q + lanes * k];
      m = fmaxf(m, x[k]);
    }
    const float mm = m == neg_inf() ? 0.0f : m;
    float s = 0.0f;
    const float f = exp_fast(START ? (mm + aj) + (float)(c_prev + d - Zd) : (mm + aj) - Z); // pair = exp(x - mm) * f
#pragma unroll
    for (int k = 0; k < K; k++) {
      const float p = exp_fast(x[k] - mm);
      s += p;
      acc[k] = fmaf(p, f, acc[k]);
    }
    ng_merge(m, s, lanes);
    if (START) {
      const float g0 = G[0];
      if (lead) Bt[(t - 1) & 1][j] = (m + log_fast(s)) - g0;
      d += (double)g0;
      c_t = c_prev;
    } else if (lead) {
      Bt[(t - 1) & 1][j] = m + log_fast(s);
    }
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < K; k++) {
    const int i = q + lanes * k;
    if (col && i < C && acc[k] != 0.0f) atomicAdd(wgrad + (START ? C : 0) + i * C + j, acc[k]);
  }
}

/* sigma_i = logsumexp_j W[i][j], one warp per row */
__global__ void __launch_bounds__(256) ngram_sigma_kernel(int C, const float* __restrict__ W, float* __restrict__ sigma) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (i >= C) return; // whole warps
  float m = neg_inf();
  for (int j = lane; j < C; j += 32) m = fmaxf(m, W[i * C + j]);
  m = warp_max(m);
  float s = 0.0f;
  for (int j = lane; j < C; j += 32) s += expf(W[i * C + j] - m);
  s = warp_sum(s);
  if (lane == 0) sigma[i] = m + logf(s);
}

/*
 * tau_i = max_j W[i][j], one warp per row: the tropical sigma, the weight of BIGRAM's folded start arcs on
 * gtnb_graph_transitions_viterbi's device route.  A NaN anywhere in the row gives tau_i = NaN, so the weights the
 * sweep loads carry it and flag the utterance for the exact route.
 */
__global__ void __launch_bounds__(256) ngram_tau_kernel(int C, const float* __restrict__ W, float* __restrict__ tau) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (i >= C) return; // whole warps
  float m = neg_inf();
  for (int j = lane; j < C; j += 32) m = max_nan(m, __ldg(W + i * C + j));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max_nan(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) tau[i] = m;
}

/*
 * The traced arcs of gtnb_graph_transitions_viterbi from product arc ids to A_b's arc ids, in place: row b of
 * arcs ([B][T_out]) holds product arcs of utterance b (-1: no arc), arc_of its A arcs in the batch's numbering;
 * off[b] = b's first product arc, off[B + b] = b's first A arc.  One thread per entry.
 */
__global__ void __launch_bounds__(256) product_arc_map_kernel(
    long long n, int T_out, const long long* __restrict__ off, const int32_t* __restrict__ arc_of,
    int32_t* __restrict__ arcs) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int a = arcs[k];
  if (a < 0) return;
  const int b = (int)(k / T_out);
  arcs[k] = __ldg(arc_of + __ldg(off + b) + a) - (int32_t)__ldg(off + (n / T_out) + b);
}

/* wgrad[i][j] += wgrad[C*C + i] * softmax_j(W[i][:]): the S arcs' gradient through sigma_i */
__global__ void __launch_bounds__(256) ngram_fold_kernel(
    int C, const float* __restrict__ W, const float* __restrict__ sigma, float* __restrict__ wgrad) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= C * C) return;
  const int i = a / C;
  const float g = wgrad[C * C + i];
  if (g != 0.0f) wgrad[a] += g * expf(W[a] - sigma[i]);
}

/*
 * The arc weights of the numerator products of gtnb_graph_transitions_loss (gtnb_product.h):
 * out[k] = w_A[arc_of[k]] + Wx[tidx[k]], Wx = [W (nW floats) | sigma]; sigma is read for tidx >= nW only (BIGRAM's
 * folded start arcs).  One thread per product arc.
 */
__global__ void __launch_bounds__(256) product_fold_kernel(
    long long n, const float* __restrict__ w_A, const int32_t* __restrict__ arc_of, const float* __restrict__ W,
    int nW, const float* __restrict__ sigma, const int32_t* __restrict__ tidx, float* __restrict__ out) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int t = __ldg(tidx + k);
  const float wx = t < nW ? __ldg(W + t) : __ldg(sigma + (t - nW));
  out[k] = __ldg(w_A + __ldg(arc_of + k)) + wx;
}

/*
 * The folded numerator graph of utterance b in the small-graph tables (k_ctc.cu's ctc_build_kernel with
 * weights): node 0 = S (start), node n >= 1 = CTC node l = n - 1 (benchmarks/ctc.cpp:40-58, accept = last two);
 * in-arcs of node n in the order skip, step, self, then the S arc for l <= 1.  The in-entry index is the arc
 * id, and map[grad_graph_off + arc] its W index (C*C + i for an S arc of weight sigma_i).
 */
__global__ void __launch_bounds__(256) ngram_num_build_kernel(
    const GraphMeta* __restrict__ meta, const int32_t* __restrict__ targets, const int32_t* __restrict__ tgt_off,
    const int32_t* __restrict__ tgt_len, int blank, int C, const float* __restrict__ W,
    const float* __restrict__ sigma, uint8_t* __restrict__ sg_flags, int32_t* __restrict__ sg_in_ptr,
    int32_t* __restrict__ sg_in_src, int32_t* __restrict__ sg_in_label, int32_t* __restrict__ sg_in_arc,
    float* __restrict__ sg_in_w, int32_t* __restrict__ sg_ilabel, int32_t* __restrict__ sg_olabel,
    int32_t* __restrict__ acc_nodes, int32_t* __restrict__ map) {
  GTNB_STATIC_SMEM(int, scan, 256);
  GTNB_STATIC_SMEM(int, carry_box, 1);
  int& carry = carry_box[0];
  const int b = blockIdx.x;
  const GraphMeta m = meta[b];
  const int tid = threadIdx.x;
  const int U = tgt_len[b];
  const int L = 2 * U + 1, N = L + 1;
  const int32_t* tg = targets + tgt_off[b];
  uint8_t* fl = sg_flags + m.sg_node_base;
  int32_t* ip = sg_in_ptr + m.sg_node_base;
  int32_t* is = sg_in_src + m.sg_arc_base;
  int32_t* il = sg_in_label + m.sg_arc_base;
  int32_t* ia = sg_in_arc + m.sg_arc_base;
  float* iw = sg_in_w + m.sg_arc_base;
  int32_t* lab_i = sg_ilabel + m.sg_arc_base;
  int32_t* lab_o = sg_olabel + m.sg_arc_base;
  int32_t* mp = map + m.grad_graph_off;
  auto lab = [&](int l) { return (l & 1) ? tg[(l - 1) / 2] : blank; };
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int n0 = 0; n0 < N; n0 += 256) {
    const int n = n0 + tid, l = n - 1;
    int label = blank, narcs = 0;
    bool skip = false;
    if (n < N && n > 0) {
      label = lab(l);
      skip = (l & 1) && l > 1 && label != tg[(l - 1) / 2 - 1];
      narcs = 1 + (l > 0 ? 1 : 0) + (skip ? 1 : 0) + (l <= 1 ? 1 : 0);
    }
    scan[tid] = narcs;
    __syncthreads();
    for (int o = 1; o < 256; o <<= 1) {
      const int v = tid >= o ? scan[tid - o] : 0;
      __syncthreads();
      scan[tid] += v;
      __syncthreads();
    }
    const int base = carry + scan[tid] - narcs;
    if (n < N) {
      const bool acc = (L >= 2) ? (l == L - 1 || l == L - 2) : (l == 0);
      fl[n] = (uint8_t)((n == 0 ? 1 : 0) | (acc ? 2 : 0));
      ip[n] = base;
      int e = base;
      auto put = [&](int src, float wt, int widx) {
        is[e] = src;
        ia[e] = e;
        il[e] = label;
        iw[e] = wt;
        lab_i[e] = label;
        lab_o[e] = label;
        mp[e] = widx;
        e++;
      };
      if (n > 0) {
        if (skip) put(n - 2, __ldg(W + label * C + lab(l - 2)), label * C + lab(l - 2));
        if (l > 0) put(n - 1, __ldg(W + label * C + lab(l - 1)), label * C + lab(l - 1));
        put(n, __ldg(W + label * C + label), label * C + label);
        if (l <= 1) put(0, sigma[label], C * C + label);
      }
    }
    __syncthreads();
    if (tid == 255) carry += scan[255];
    __syncthreads();
  }
  if (tid == 0) {
    ip[N] = carry;
    int32_t* acc = acc_nodes + m.acc_base;
    if (L >= 2) {
      acc[0] = L - 1; // device nodes of CTC nodes L - 2, L - 1
      acc[1] = L;
    } else {
      acc[0] = 1;
    }
  }
}

/*
 * compose(fal_b, transitions) of ASG's numerator (test/criterion_test.cpp:244-305) in the small-graph tables:
 * U+1 nodes, node l = "l labels consumed", start 0, accept U (none when U = 0).  Arcs in the reference's creation
 * order: 0 -> 1 (weight s[y0]), then per node l >= 1 a self loop (W[y_{l-1}][y_{l-1}]) and the step l -> l+1
 * (W[y_l][y_{l-1}]).  So node n >= 1 has exactly two in-arcs, both labelled y_{n-1}: arc 2n-2 from n-1, arc
 * 2n-1 its self loop; the in-entry index is the arc id, and map[grad_graph_off + arc] its index in trans_w.
 */
__global__ void __launch_bounds__(256) asg_num_build_kernel(
    const GraphMeta* __restrict__ meta, const int32_t* __restrict__ targets, const int32_t* __restrict__ tgt_off,
    const int32_t* __restrict__ tgt_len, int C, const float* __restrict__ trans_w, uint8_t* __restrict__ sg_flags,
    int32_t* __restrict__ sg_in_ptr, int32_t* __restrict__ sg_in_src, int32_t* __restrict__ sg_in_label,
    int32_t* __restrict__ sg_in_arc, float* __restrict__ sg_in_w, int32_t* __restrict__ sg_ilabel,
    int32_t* __restrict__ sg_olabel, int32_t* __restrict__ acc_nodes, int32_t* __restrict__ map) {
  const int b = blockIdx.x;
  const GraphMeta m = meta[b];
  const int U = tgt_len[b], N = U + 1;
  const int32_t* y = targets + tgt_off[b];
  uint8_t* fl = sg_flags + m.sg_node_base;
  int32_t* ip = sg_in_ptr + m.sg_node_base;
  int32_t* is = sg_in_src + m.sg_arc_base;
  int32_t* il = sg_in_label + m.sg_arc_base;
  int32_t* ia = sg_in_arc + m.sg_arc_base;
  float* iw = sg_in_w + m.sg_arc_base;
  int32_t* lab_i = sg_ilabel + m.sg_arc_base;
  int32_t* lab_o = sg_olabel + m.sg_arc_base;
  int32_t* mp = map + m.grad_graph_off;
  for (int n = threadIdx.x; n <= N; n += blockDim.x) {
    if (n == N) {
      ip[N] = 2 * U;
      continue;
    }
    fl[n] = (uint8_t)((n == 0 ? 1 : 0) | (U > 0 && n == U ? 2 : 0));
    ip[n] = n == 0 ? 0 : 2 * (n - 1);
    if (n == 0) continue;
    const int label = y[n - 1], e = 2 * (n - 1);
    const int widx[2] = {n == 1 ? label : C + label * C + y[n - 2], C + label * C + label};
#pragma unroll
    for (int k = 0; k < 2; k++) {
      is[e + k] = n - 1 + k;
      ia[e + k] = e + k;
      il[e + k] = label;
      iw[e + k] = __ldg(trans_w + widx[k]);
      lab_i[e + k] = label;
      lab_o[e + k] = label;
      mp[e + k] = widx[k];
    }
  }
  if (threadIdx.x == 0 && U > 0) acc_nodes[m.acc_base] = U;
}

} // namespace

#ifndef GTNB_HOST_EMU

int launch_ngram_sigma(gtnb_ctx* ctx, int C, const float* W, float* sigma) {
  GTNB_LAUNCH(ctx, "ngram_sigma", ngram_sigma_kernel<<<(C * 32 + 255) / 256, 256, 0, ctx->stream>>>(C, W, sigma));
  return GTNB_OK;
}

int launch_ngram_num_build(
    gtnb_ctx* ctx, gtnb_lattice* lat, const int32_t* targets_dev, const int32_t* tgt_off_dev,
    const int32_t* tgt_len_dev, int blank, const float* W, const float* sigma, int32_t* map) {
  if (lat->B == 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "ngram_num_build", ngram_num_build_kernel<<<lat->B, 256, 0, ctx->stream>>>(
      lat->meta, targets_dev, tgt_off_dev, tgt_len_dev, blank, lat->C, W, sigma, lat->sg_flags, lat->sg_in_ptr,
      lat->sg_in_src, lat->sg_in_label, lat->sg_in_arc, lat->sg_in_w, lat->sg_ilabel, lat->sg_olabel,
      lat->acc_nodes, map));
  return GTNB_OK;
}

namespace {

template <bool START, class E>
int den_forward(gtnb_ctx* ctx, const char* name, int B, int T, int C, const int32_t* lens_dev, const E* emis,
                long long stride, const float* W, float* alpha, float* den, int32_t* status) {
  if (B == 0) return GTNB_OK;
  int K, lanes, threads;
  ngram_den_shape(C, &K, &lanes, &threads);
  if (K == 16)
    GTNB_LAUNCH(ctx, name, ngram_den_forward_kernel<16, START, E><<<B, threads, 0, ctx->stream>>>(
        T, C, lanes, lens_dev, emis, stride, W, alpha, den, status));
  else
    GTNB_LAUNCH(ctx, name, ngram_den_forward_kernel<32, START, E><<<B, threads, 0, ctx->stream>>>(
        T, C, lanes, lens_dev, emis, stride, W, alpha, den, status));
  return GTNB_OK;
}

template <bool START, class E>
int den_backward(gtnb_ctx* ctx, const char* name, int B, int T, int C, const int32_t* lens_dev, const E* emis,
                 long long stride, const float* W, const float* alpha, const float* den, float* grad,
                 long long grad_stride, float* wgrad) {
  if (B == 0) return GTNB_OK;
  int K, lanes, threads;
  ngram_den_shape(C, &K, &lanes, &threads);
  if (K == 16)
    GTNB_LAUNCH(ctx, name, ngram_den_backward_kernel<16, START, E><<<B, threads, 0, ctx->stream>>>(
        T, C, lanes, lens_dev, emis, stride, W, alpha, den, grad, grad_stride, wgrad));
  else
    GTNB_LAUNCH(ctx, name, ngram_den_backward_kernel<32, START, E><<<B, threads, 0, ctx->stream>>>(
        T, C, lanes, lens_dev, emis, stride, W, alpha, den, grad, grad_stride, wgrad));
  return GTNB_OK;
}

/* f(typed emissions) for the element type dtype names (GTNB_F32 / GTNB_BF16 / GTNB_F16) */
template <class F>
int with_elem(gtnb_ctx* ctx, int dtype, const void* emis, F&& f) {
  switch (dtype) {
    case GTNB_F32: return f(static_cast<const float*>(emis));
    case GTNB_BF16: return f(static_cast<const bf16_t*>(emis));
    case GTNB_F16: return f(static_cast<const f16_t*>(emis));
    default: return fail(ctx, GTNB_ERR_LOGIC, "k_ngram.cu: unknown element type");
  }
}

} // namespace

int launch_ngram_den_forward(
    gtnb_ctx* ctx, int B, int T, int C, const int32_t* lens_dev, const void* emis, long long stride,
    const float* W, float* alpha, float* den, int32_t* status, int dtype) {
  return with_elem(ctx, dtype, emis, [&](auto e) {
    return den_forward<false>(ctx, "ngram_den_forward", B, T, C, lens_dev, e, stride, W, alpha, den, status);
  });
}

int launch_ngram_den_backward(
    gtnb_ctx* ctx, int B, int T, int C, const int32_t* lens_dev, const void* emis, long long stride,
    const float* W, const float* alpha, const float* den, float* grad, long long grad_stride, float* wgrad,
    int dtype) {
  return with_elem(ctx, dtype, emis, [&](auto e) {
    return den_backward<false>(ctx, "ngram_den_backward", B, T, C, lens_dev, e, stride, W, alpha, den, grad,
                               grad_stride, wgrad);
  });
}

int launch_asg_den_forward(
    gtnb_ctx* ctx, int B, int T, int C, const int32_t* lens_dev, const void* emis, long long stride,
    const float* trans_w, float* alpha, float* den, int32_t* status, int dtype) {
  return with_elem(ctx, dtype, emis, [&](auto e) {
    return den_forward<true>(ctx, "asg_den_forward", B, T, C, lens_dev, e, stride, trans_w, alpha, den, status);
  });
}

int launch_asg_den_backward(
    gtnb_ctx* ctx, int B, int T, int C, const int32_t* lens_dev, const void* emis, long long stride,
    const float* trans_w, const float* alpha, const float* den, float* grad, long long grad_stride,
    float* trans_grad, int dtype) {
  return with_elem(ctx, dtype, emis, [&](auto e) {
    return den_backward<true>(ctx, "asg_den_backward", B, T, C, lens_dev, e, stride, trans_w, alpha, den, grad,
                              grad_stride, trans_grad);
  });
}

int launch_asg_num_build(
    gtnb_ctx* ctx, gtnb_lattice* lat, const int32_t* targets_dev, const int32_t* tgt_off_dev,
    const int32_t* tgt_len_dev, const float* trans_w, int32_t* map) {
  if (lat->B == 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "asg_num_build", asg_num_build_kernel<<<lat->B, 256, 0, ctx->stream>>>(
      lat->meta, targets_dev, tgt_off_dev, tgt_len_dev, lat->C, trans_w, lat->sg_flags, lat->sg_in_ptr,
      lat->sg_in_src, lat->sg_in_label, lat->sg_in_arc, lat->sg_in_w, lat->sg_ilabel, lat->sg_olabel,
      lat->acc_nodes, map));
  return GTNB_OK;
}

int launch_ngram_fold(gtnb_ctx* ctx, int C, const float* W, const float* sigma, float* wgrad) {
  GTNB_LAUNCH(ctx, "ngram_fold", ngram_fold_kernel<<<(C * C + 255) / 256, 256, 0, ctx->stream>>>(C, W, sigma, wgrad));
  return GTNB_OK;
}

int launch_product_fold(gtnb_ctx* ctx, long long n, const float* w_A, const int32_t* arc_of, const float* W, int nW,
                        const float* sigma, const int32_t* tidx, float* out) {
  if (n == 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "product_fold", product_fold_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(
      n, w_A, arc_of, W, nW, sigma, tidx, out));
  return GTNB_OK;
}

int launch_ngram_tau(gtnb_ctx* ctx, int C, const float* W, float* tau) {
  GTNB_LAUNCH(ctx, "ngram_tau", ngram_tau_kernel<<<(C * 32 + 255) / 256, 256, 0, ctx->stream>>>(C, W, tau));
  return GTNB_OK;
}

int launch_product_arc_map(gtnb_ctx* ctx, int B, int T_out, const long long* off, const int32_t* arc_of,
                           int32_t* arcs) {
  const long long n = (long long)B * T_out;
  if (n == 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "product_arc_map", product_arc_map_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(
      n, T_out, off, arc_of, arcs));
  return GTNB_OK;
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
