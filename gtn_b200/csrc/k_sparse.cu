/*
 * k_sparse.cu -- the denominator of gtnb_sparse_transitions_loss, forwardScore(intersect(E_b, G)) and its gradients,
 * for a transition graph G of any shape (an epsilon-free acceptor: n-gram graphs of any order, pruned token LMs,
 * HMM topologies), without building the T_b * |G| lattice.
 *
 * The product state at frame t is a G node, so the sweeps are
 *     alpha_0[v] = 0 on G's start nodes (-inf elsewhere),
 *     alpha_t[v] = logsumexp over in-arcs a: u -> v of (alpha_{t-1}[u] + w_a + e[t-1][label_a]),
 *     Z = logsumexp of alpha_{T_b} over G's accept nodes,
 *     beta_{T_b}[u] = 0 on accept nodes, beta_t[u] = logsumexp over out-arcs a: u -> v of (w_a + e[t][label_a] +
 *     beta_{t+1}[v]),
 * and the posterior of arc a at frame t, exp(alpha_t[u] + w_a + e[t][label_a] + beta_{t+1}[v] - Z), is added into the
 * emission gradient (row t, column label_a) and into the arc's weight gradient (summed over frames and utterances).
 *
 * Layout: one CTA per utterance.  The two score rows of the sweep ([2][S] floats), the emission row of the frame
 * ([2][C], double-buffered so that the next row loads during the sweep) and, in the backward kernel, the per-CTA
 * accumulators of the arc gradient ([A] floats) and of the frame's emission gradient ([2][C]) live in shared memory.
 * G's tables (CSR by destination for the forward, by source for the backward) are read through the read-only path
 * from L2, where one copy serves every CTA: at the envelope (S = 4096, A = 32768) they are 400 KB, too large to sit
 * in shared memory beside the rows, and the frames read them in the same order, so the L1 keeps the hot part.  A node
 * is handled by `lanes` threads (a power of two, chosen from G's mean degree) that stride over its arcs with an online
 * logsumexp and merge with shuffles; the loop over nodes has the same trip count in every warp.  Each thread owns the
 * same arcs at every frame, so the arc accumulators take plain adds and go to global memory once per CTA.
 *
 * Scores are kept relative to per-frame offsets accumulated in double (DESIGN.md, "ASG on padded batches"): row t is
 * stored as alpha_t - c_t with c_t = c_{t-1} + max(row_{t-1}) (the maximum of every warp is left in shared memory and
 * merged after the frame's barrier), and likewise beta_t - d_t.  A posterior's exponent is row + row' + (float)(c_t +
 * d_{t+1} - Z), so fp32 scores that grow with t never cancel.  exp / log on the SFU (ex2.approx / lg2.approx).
 *
 * Valid only for finite weights: the forward kernel raises status bit 1 on any non-finite weight or used emission,
 * and the caller repeats the call on the materialised route.
 *
 * A G beyond that CTA's shared memory (S > 4096 or A > 32768) is swept by one thread-block cluster per utterance
 * (the sparse_cl_* kernels below, behind the "sparse_cluster" context flag): the rows whole in every CTA, the nodes
 * and the arc accumulators split over the ranks, results exchanged through distributed shared memory.
 *
 * The decoder gtnb_viterbi_sparse sweeps the same tables in the tropical semiring (sparse_viterbi_forward_kernel):
 * S_t[v] = max over in-arcs a: u -> v of fl(S_{t-1}[u] + fl(w_a + e[t-1][label_a])), the reference's association
 * (compose.cpp:435, then shortest.cpp:213), with absolute scores so that the score is bit-exact.  Per (frame, node) it
 * keeps a 16-bit back-pointer in HBM, the winning in-arc's position in the node's in-list plus a tie flag, and
 * sparse_viterbi_trace_kernel walks them back from the best accept node.
 *
 * The backoff entry points (gtnb_backoff_transitions_loss, gtnb_viterbi_backoff) take a G with epsilon arcs, and
 * their numerators A_b o G have them too.  The sparse_eps_* kernels are the kernels above with an epsilon closure
 * after every frame's emitting update (one CTA barrier per topological level of the epsilon subgraph) and per-CTA
 * tables, so that one launch sweeps B different numerators; an epsilon-free G keeps the kernels above.  The
 * alignment gtnb_backoff_transitions_viterbi runs the decode's tropical sweep and trace over those per-CTA
 * numerators (sparse_eps_align_*), reporting A_b's arcs.  A backoff G beyond one CTA has its denominator swept by a
 * thread-block cluster (sparse_cl_eps_*), the closure's levels cut over the ranks.
 */
#include <algorithm>
#include <utility>

#include "gtnb_ptx.h"

namespace gtnb {

/* floats of dynamic shared memory of the two sweeps */
inline int sparse_fwd_smem_floats(int S, int C) {
  return 2 * S + 2 * C + 2 * kSparseWarps;
}
inline int sparse_bwd_smem_floats(int S, int A, int C) {
  return 2 * S + 4 * C + A + 2 * kSparseWarps;
}
inline int sparse_vit_smem_floats(int S, int C) {
  return 2 * S + 2 * C;
}
/* a back-pointer: the in-list position (in-degree <= kSparseMaxArcs) and the tie flag; kBpNone on a -inf node */
constexpr int kBpTie = 0x8000;
constexpr uint16_t kBpNone = 0xFFFF;

namespace {

/* the per-lane (m, s) of an online logsumexp: s = sum of exp(x - m) over the terms seen; -inf and NaN terms skipped */
__device__ __forceinline__ void lse_add(float& m, float& s, float x) {
  if (x > m) {
    s = s * exp_fast(m - x) + 1.0f;
    m = x;
  } else if (x > neg_inf()) {
    s += exp_fast(x - m);
  }
}

/* (m, s) merged over the `lanes` consecutive lanes of a node; every lane of the group gets the result */
__device__ __forceinline__ void lse_merge(float& m, float& s, int lanes) {
  for (int o = 1; o < lanes; o <<= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const float os = __shfl_xor_sync(0xffffffffu, s, o);
    const float M = fmaxf(m, om);
    const float Mm = M == neg_inf() ? 0.0f : M; // all -inf: s stays 0
    s = s * exp_fast(m - Mm) + os * exp_fast(om - Mm);
    m = M;
  }
}

/* the maximum of the previous frame's row from the per-warp maxima; 0 when the row is all -inf */
__device__ __forceinline__ float row_offset(const float* red) {
  float M = neg_inf();
#pragma unroll
  for (int i = 0; i < kSparseWarps; i++) M = fmaxf(M, red[i]);
  return M == neg_inf() ? 0.0f : M;
}

/*
 * alpha rows of utterance b to alpha[b][(T+1)*S] (relative to the offsets), the offsets c_t to offs[b][t] for t >= 1
 * and Z to offs[b][0] (double) and den[b] (float); status[b] |= 1 on a non-finite weight or used emission.
 */
__global__ void __launch_bounds__(kSparseThreads) sparse_den_forward_kernel(
    SparseDev g, int T, int C, const int32_t* __restrict__ lens, const float* __restrict__ emis, long long stride,
    const float* __restrict__ w, float* __restrict__ alpha, double* __restrict__ offs, float* __restrict__ den,
    int32_t* __restrict__ status) {
  GTNB_DYNAMIC_SMEM(float, sm);
  const int S = g.S, lanes = g.lanes;
  float* rows = sm; // [2][S]
  float* E = sm + 2 * S; // [2][C]
  float* red = E + 2 * C; // [2][kSparseWarps]
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
  const int Tb = lens[b];
  const float* em = emis + (long long)b * stride;
  float* al = alpha + (long long)b * (T + 1) * S;
  double* of = offs + (long long)b * (T + 1);
  bool bad = false;
  float mx = neg_inf();
  for (int v = tid; v < S; v += nt) {
    const float a0 = (__ldg(g.flags + v) & 1) ? 0.0f : neg_inf();
    rows[v] = a0;
    al[v] = a0;
    mx = fmaxf(mx, a0);
  }
  mx = warp_max(mx);
  if (tid % 32 == 0) red[tid / 32] = mx;
  if (Tb > 0)
    for (int c = tid; c < C; c += nt) E[C + c] = __ldg(em + c); // row 0 in E[1]: frame t reads E[t & 1]
  __syncthreads();
  double c_off = 0.0;
  for (int t = 1; t <= Tb; t++) {
    const float* P = rows + ((t - 1) & 1) * S;
    float* Q = rows + (t & 1) * S;
    const float* Er = E + (t & 1) * C;
    if (t < Tb)
      for (int c = tid; c < C; c += nt) E[((t + 1) & 1) * C + c] = __ldg(em + (long long)t * C + c);
    const float Mp = row_offset(red + ((t - 1) & 1) * kSparseWarps);
    mx = neg_inf();
    for (int v0 = 0; v0 < S; v0 += groups) { // (the same trip count in every warp: the merge shuffles)
      const int v = v0 + grp;
      float m = neg_inf(), s = 0.0f;
      if (v < S) {
        const int k1 = __ldg(g.in_ptr + v + 1);
        for (int k = __ldg(g.in_ptr + v) + q; k < k1; k += lanes) {
          const float wk = __ldg(w + __ldg(g.in_arc + k));
          const float ek = Er[__ldg(g.in_lab + k)];
          bad |= !(is_finite(wk) && is_finite(ek));
          lse_add(m, s, P[__ldg(g.in_src + k)] + (wk + ek));
        }
      }
      lse_merge(m, s, lanes);
      if (v < S) {
        const float val = m == neg_inf() ? neg_inf() : (m + log_fast(s)) - Mp;
        if (q == 0) {
          Q[v] = val;
          al[(long long)t * S + v] = val;
        }
        mx = fmaxf(mx, val);
      }
    }
    mx = warp_max(mx);
    if (tid % 32 == 0) red[(t & 1) * kSparseWarps + tid / 32] = mx;
    c_off += (double)Mp;
    if (tid == 0) of[t] = c_off;
    __syncthreads();
  }
  bad = __syncthreads_or(bad);
  if (tid < 32) {
    const float* F = rows + (Tb & 1) * S;
    float m = neg_inf();
    for (int v = tid; v < S; v += 32)
      if (__ldg(g.flags + v) & 2) m = fmaxf(m, F[v]);
    m = warp_max(m);
    float s = 0.0f;
    if (m != neg_inf())
      for (int v = tid; v < S; v += 32)
        if (__ldg(g.flags + v) & 2) s += expf(F[v] - m);
    s = warp_sum(s);
    if (tid == 0) {
      const double Z = m == neg_inf() ? (double)neg_inf() : c_off + (double)(m + logf(s));
      of[0] = Z;
      den[b] = (float)Z;
      if (bad) atomicOr(&status[b], 1);
    }
  }
}

/*
 * d Z / d e added into grad (rows t < T_b; one red.add per label and frame per CTA) and d Z / d w added into
 * wgrad[G's arc id] (one per arc per CTA).  Nothing when Z is not finite (no accepting path: the reference's gradient
 * of a -inf score is 0 on the paths that do not exist) or T_b = 0.
 */
__global__ void __launch_bounds__(kSparseThreads) sparse_den_backward_kernel(
    SparseDev g, int T, int C, const int32_t* __restrict__ lens, const float* __restrict__ emis, long long stride,
    const float* __restrict__ w, const float* __restrict__ alpha, const double* __restrict__ offs,
    float* __restrict__ grad, long long grad_stride, float* __restrict__ wgrad) {
  GTNB_DYNAMIC_SMEM(float, sm);
  const int S = g.S, A = g.A, lanes = g.lanes;
  float* rows = sm; // [2][S] beta rows
  float* E = sm + 2 * S; // [2][C] emission rows
  float* Eg = E + 2 * C; // [2][C] the frame's emission gradient
  float* acc = Eg + 2 * C; // [A] arc gradient, by out-table position
  float* red = acc + A; // [2][kSparseWarps]
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
  const int Tb = lens[b];
  const double* of = offs + (long long)b * (T + 1);
  const double Z = of[0];
  if (Tb < 1 || !(fabs(Z) < (double)CUDART_INF_F)) return;
  const float* em = emis + (long long)b * stride;
  const float* al = alpha + (long long)b * (T + 1) * S;
  float* gr = grad + (long long)b * grad_stride;
  float mx = neg_inf();
  for (int v = tid; v < S; v += nt) {
    const float b0 = (__ldg(g.flags + v) & 2) ? 0.0f : neg_inf();
    rows[(Tb & 1) * S + v] = b0;
    mx = fmaxf(mx, b0);
  }
  mx = warp_max(mx);
  if (tid % 32 == 0) red[(Tb & 1) * kSparseWarps + tid / 32] = mx;
  for (int k = tid; k < A; k += nt) acc[k] = 0.0f;
  for (int c = tid; c < 2 * C; c += nt) Eg[c] = 0.0f;
  for (int c = tid; c < C; c += nt) E[((Tb - 1) & 1) * C + c] = __ldg(em + (long long)(Tb - 1) * C + c);
  __syncthreads();
  double d = 0.0; // d_{t+1}
  for (int t = Tb - 1; t >= 0; t--) {
    const float* Nx = rows + ((t + 1) & 1) * S;
    float* Cur = rows + (t & 1) * S;
    const float* Er = E + (t & 1) * C;
    float* Eg_t = Eg + (t & 1) * C;
    float* Eg_prev = Eg + ((t + 1) & 1) * C; // frame t + 1's, complete since the barrier
    for (int c = tid; c < C; c += nt) {
      if (t > 0) E[((t + 1) & 1) * C + c] = __ldg(em + (long long)(t - 1) * C + c);
      if (t + 1 < Tb) {
        const float v = Eg_prev[c];
        if (v != 0.0f) atomicAdd(gr + (long long)(t + 1) * C + c, v);
        Eg_prev[c] = 0.0f;
      }
    }
    const float Mb = row_offset(red + ((t + 1) & 1) * kSparseWarps);
    const double c_t = t > 0 ? of[t] : 0.0;
    const float fo = (float)(c_t + d - Z);
    mx = neg_inf();
    for (int u0 = 0; u0 < S; u0 += groups) {
      const int u = u0 + grp;
      float m = neg_inf(), s = 0.0f;
      if (u < S) {
        const float au = al[(long long)t * S + u] + fo; // alpha_t[u] + c_t + d_{t+1} - Z, in the exponent's terms
        const int k1 = __ldg(g.out_ptr + u + 1);
        for (int k = __ldg(g.out_ptr + u) + q; k < k1; k += lanes) {
          const int lab = __ldg(g.out_lab + k);
          const float x = Nx[__ldg(g.out_dst + k)] + (__ldg(w + __ldg(g.out_arc + k)) + Er[lab]);
          lse_add(m, s, x);
          const float p = exp_fast(au + x);
          if (p != 0.0f) {
            acc[k] += p;
            atomicAdd(Eg_t + lab, p);
          }
        }
      }
      lse_merge(m, s, lanes);
      if (u < S) {
        const float val = m == neg_inf() ? neg_inf() : (m + log_fast(s)) - Mb;
        if (q == 0) Cur[u] = val;
        mx = fmaxf(mx, val);
      }
    }
    mx = warp_max(mx);
    if (tid % 32 == 0) red[(t & 1) * kSparseWarps + tid / 32] = mx;
    d += (double)Mb;
    __syncthreads();
  }
  for (int c = tid; c < C; c += nt) { // frame 0's emission gradient
    const float v = Eg[c];
    if (v != 0.0f) atomicAdd(gr + c, v);
  }
  for (int k = tid; k < A; k += nt)
    if (acc[k] != 0.0f) atomicAdd(wgrad + __ldg(g.out_arc + k), acc[k]);
}

/* sigma_k = logsumexp of the weights of start group k (gtnb_product.h), one warp per group */
__global__ void __launch_bounds__(256) sparse_sigma_kernel(int K, const int32_t* __restrict__ grp_ptr,
                                                           const int32_t* __restrict__ grp_arc,
                                                           const float* __restrict__ w, float* __restrict__ sigma) {
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (k >= K) return; // whole warps
  const int a0 = __ldg(grp_ptr + k), a1 = __ldg(grp_ptr + k + 1);
  float m = neg_inf();
  for (int j = a0 + lane; j < a1; j += 32) m = fmaxf(m, __ldg(w + __ldg(grp_arc + j)));
  m = warp_max(m);
  float s = 0.0f;
  if (m != neg_inf())
    for (int j = a0 + lane; j < a1; j += 32) s += expf(__ldg(w + __ldg(grp_arc + j)) - m);
  s = warp_sum(s);
  if (lane == 0) sigma[k] = m == neg_inf() ? m : m + logf(s);
}

/* wgrad[a] += wgrad[nG + k] * exp(w_a - sigma_k) for every arc a of start group k: the folded start arcs' gradient
 * through sigma (every arc is in one group at most: no race), one thread per group */
__global__ void __launch_bounds__(256) sparse_fold_kernel(int K, const int32_t* __restrict__ grp_ptr,
                                                          const int32_t* __restrict__ grp_arc, int nG,
                                                          const float* __restrict__ w,
                                                          const float* __restrict__ sigma, float* __restrict__ wgrad) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const float gk = wgrad[nG + k];
  if (gk == 0.0f) return;
  const float sk = sigma[k];
  for (int j = __ldg(grp_ptr + k); j < __ldg(grp_ptr + k + 1); j++) {
    const int a = __ldg(grp_arc + j);
    wgrad[a] += gk * expf(__ldg(w + a) - sk);
  }
}

/* a max and its argmax merged over the `lanes` consecutive lanes of a group: the lowest index among equal maxima,
 * tie = 1 when more than one candidate reaches a finite max; every lane of the group gets the result */
__device__ __forceinline__ void argmax_merge(float& m, int& k, int& tie, int lanes) {
  for (int o = 1; o < lanes; o <<= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const int ok = __shfl_xor_sync(0xffffffffu, k, o);
    const int ot = __shfl_xor_sync(0xffffffffu, tie, o);
    if (om > m) {
      m = om;
      k = ok;
      tie = ot;
    } else if (om == m && m != neg_inf()) {
      k = min(k, ok);
      tie = 1;
    }
  }
}

/* one candidate of a lane's running (m, k, tie): strict >, so the first of equal candidates stays; -inf and NaN
 * candidates never win */
__device__ __forceinline__ void argmax_add(float& m, int& k, int& tie, float x, int j) {
  if (x > m) {
    m = x;
    k = j;
    tie = 0;
  } else if (x == m && x != neg_inf()) {
    tie = 1;
  }
}

/*
 * The tropical sweep of gtnb_viterbi_sparse over intersect(E_b, G) for utterance b = blockIdx.x, in the layout of
 * sparse_den_forward_kernel (rows and emission rows in shared memory, G's tables from L2, `lanes` threads per node).
 * bp[b][t-1][v] (t = 1 .. T_b): the in-list position of the in-arc that reaches S_t[v], | kBpTie when another in-arc
 * reaches it too; kBpNone where S_t[v] = -inf (on no path).  Then the best accept node of frame T_b, the first in
 * node order, to head[b] (-1 when no accept node is finite, T_b = 0 included) and its score to score[b].
 * status[b] |= 1 on a NaN or +inf weight or used emission (-inf only forbids the arc), |= 2 when two accept nodes
 * reach the best score.
 */
__global__ void __launch_bounds__(kSparseThreads) sparse_viterbi_forward_kernel(
    SparseDev g, int T, int C, const int32_t* __restrict__ lens, const float* __restrict__ emis, long long stride,
    const float* __restrict__ w, uint16_t* __restrict__ bp, int32_t* __restrict__ head, float* __restrict__ score,
    int32_t* __restrict__ status) {
  GTNB_DYNAMIC_SMEM(float, sm);
  const int S = g.S, lanes = g.lanes;
  float* rows = sm; // [2][S]
  float* E = sm + 2 * S; // [2][C]
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
  const int Tb = lens[b];
  const float* em = emis + (long long)b * stride;
  uint16_t* bpb = bp + (long long)b * T * S;
  bool bad = false;
  for (int v = tid; v < S; v += nt) rows[v] = (__ldg(g.flags + v) & 1) ? 0.0f : neg_inf();
  if (Tb > 0)
    for (int c = tid; c < C; c += nt) E[C + c] = __ldg(em + c); // row 0 in E[1]: frame t reads E[t & 1]
  __syncthreads();
  for (int t = 1; t <= Tb; t++) {
    const float* P = rows + ((t - 1) & 1) * S;
    float* Q = rows + (t & 1) * S;
    const float* Er = E + (t & 1) * C;
    uint16_t* bpt = bpb + (long long)(t - 1) * S;
    if (t < Tb)
      for (int c = tid; c < C; c += nt) E[((t + 1) & 1) * C + c] = __ldg(em + (long long)t * C + c);
    for (int v0 = 0; v0 < S; v0 += groups) { // (the same trip count in every warp: the merge shuffles)
      const int v = v0 + grp;
      float m = neg_inf();
      int k = 0x7fffffff, tie = 0, k0 = 0;
      if (v < S) {
        k0 = __ldg(g.in_ptr + v);
        const int k1 = __ldg(g.in_ptr + v + 1);
        for (int j = k0 + q; j < k1; j += lanes) {
          const float wk = __ldg(w + __ldg(g.in_arc + j));
          const float ek = Er[__ldg(g.in_lab + j)];
          bad |= !(wk < CUDART_INF_F && ek < CUDART_INF_F);
          argmax_add(m, k, tie, P[__ldg(g.in_src + j)] + (wk + ek), j);
        }
      }
      argmax_merge(m, k, tie, lanes);
      if (v < S && q == 0) {
        Q[v] = m;
        bpt[v] = m == neg_inf() ? kBpNone : (uint16_t)((k - k0) | (tie ? kBpTie : 0));
      }
    }
    __syncthreads();
  }
  bad = __syncthreads_or(bad);
  if (tid < 32) {
    const float* F = rows + (Tb & 1) * S;
    float m = neg_inf();
    int k = 0x7fffffff, tie = 0;
    if (Tb > 0)
      for (int v = tid; v < S; v += 32)
        if (__ldg(g.flags + v) & 2) argmax_add(m, k, tie, F[v], v);
    argmax_merge(m, k, tie, 32);
    if (tid == 0) {
      head[b] = m == neg_inf() ? -1 : k;
      score[b] = m;
      const int st = (bad ? 1 : 0) | (tie ? 2 : 0);
      if (st) atomicOr(&status[b], st);
    }
  }
}

/*
 * The traceback of gtnb_viterbi_sparse, one warp per utterance: paths[b][t] = the label and arcs[b][t] = G's arc id
 * of the arc the best path takes at frame t (both nullable), walked back from head[b] through bp; -1 beyond T_b and
 * in the whole row without a path.  status[b] |= 2 when a node of the path carries the tie flag.
 */
__global__ void __launch_bounds__(256) sparse_viterbi_trace_kernel(
    SparseDev g, int B, int T, const int32_t* __restrict__ lens, const uint16_t* __restrict__ bp,
    const int32_t* __restrict__ head, int32_t* __restrict__ paths, int32_t* __restrict__ arcs,
    int32_t* __restrict__ status) {
  const int b = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (b >= B) return; // whole warps
  const int h = head[b];
  const int n = h < 0 ? 0 : lens[b]; // the path's frames
  int32_t* pr = paths ? paths + (long long)b * T : nullptr;
  int32_t* ar = arcs ? arcs + (long long)b * T : nullptr;
  for (int t = n + lane; t < T; t += 32) {
    if (pr) pr[t] = -1;
    if (ar) ar[t] = -1;
  }
  if (lane != 0 || n == 0) return;
  const uint16_t* bpb = bp + (long long)b * T * g.S;
  int v = h, tie = 0;
  for (int t = n; t >= 1; t--) {
    const int e = __ldg(bpb + (long long)(t - 1) * g.S + v);
    const int k = __ldg(g.in_ptr + v) + (e & (kBpTie - 1));
    tie |= e & kBpTie;
    if (pr) pr[t - 1] = __ldg(g.in_lab + k);
    if (ar) ar[t - 1] = __ldg(g.in_arc + k);
    v = __ldg(g.in_src + k);
  }
  if (tie) atomicOr(&status[b], 2);
}

/* tau_k = the max of the weights of start group k (gtnb_product.h), NaN kept: the tropical counterpart of sigma, the
 * weight of gtnb_sparse_transitions_viterbi's folded start arcs; one warp per group */
__global__ void __launch_bounds__(256) sparse_tau_kernel(int K, const int32_t* __restrict__ grp_ptr,
                                                         const int32_t* __restrict__ grp_arc,
                                                         const float* __restrict__ w, float* __restrict__ tau) {
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
  if (k >= K) return; // whole warps
  const int a0 = __ldg(grp_ptr + k), a1 = __ldg(grp_ptr + k + 1);
  float m = neg_inf();
  for (int j = a0 + lane; j < a1; j += 32) m = max_nan(m, __ldg(w + __ldg(grp_arc + j)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max_nan(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) tau[k] = m;
}

/*
 * The cluster sweeps: the three sweeps above for a G that one CTA's shared memory cannot hold, one thread-block
 * cluster of N = sp.N CTAs per utterance (b = blockIdx.x / N).  Every CTA keeps the whole [2][S] rows; rank r
 * computes the new row for its own nodes only (sp.in for the forward and the tropical sweep, sp.out for the backward),
 * with the `lanes` threads, arc order and merges of the one-CTA kernels, and stores each result into the row of every
 * CTA of the cluster through distributed shared memory.  The per-warp row maxima go the same way ([2][N *
 * kSparseWarps]; a maximum does not depend on how the row is cut), so rows, offsets, Z, scores and back-pointers are
 * bit-identical to the one-CTA kernels'.  One barrier.cluster per frame replaces the CTA barrier: after it the frame's
 * row is complete in every CTA and nobody reads the row before it any more, which is the row the next frame
 * overwrites.  The backward keeps accumulators for its own out-arcs only (about A / N) and its own emission-gradient
 * rows, so only the order of the adds into grad and wgrad differs.  Global outputs are written by a node's owner, the
 * per-utterance ones by rank 0.
 */

/* v into the float at p of every CTA of the cluster, this one included */
__device__ __forceinline__ void cluster_store(float* p, int N, float v) {
  const uint32_t a = smem_u32(p);
  for (int r = 0; r < N; r++) sts_cluster_f32(a, r, v);
}

/* row_offset over the n per-warp maxima of every rank, by whole warps */
__device__ __forceinline__ float cluster_row_offset(const float* red, int n) {
  float M = neg_inf();
  for (int i = threadIdx.x % 32; i < n; i += 32) M = fmaxf(M, red[i]);
  M = warp_max(M);
  return M == neg_inf() ? 0.0f : M;
}

/* a sweep's first row, R[v] = 0 where flags[v] has `bit` and -inf elsewhere: the same in every CTA, so each fills
 * its own copy (also to out, nullable) and leaves the row's maximum in red[par] ([2][n], the rest -inf) */
__device__ __forceinline__ void cluster_first_row(const SparseDev& g, int bit, float* R, float* out, float* red, int n,
                                                  int par) {
  const int tid = threadIdx.x, nt = blockDim.x;
  float mx = neg_inf();
  for (int v = tid; v < g.S; v += nt) {
    const float a0 = (__ldg(g.flags + v) & bit) ? 0.0f : neg_inf();
    R[v] = a0;
    if (out) out[v] = a0;
    mx = fmaxf(mx, a0);
  }
  for (int i = tid; i < 2 * n; i += nt) red[i] = neg_inf();
  __syncthreads();
  mx = warp_max(mx);
  if (tid % 32 == 0) red[par * n + tid / 32] = mx;
}

/* sparse_den_forward_kernel by a cluster: the same outputs */
__global__ void __launch_bounds__(kSparseThreads) sparse_cl_den_forward_kernel(
    SparseDev g, SparseSplit sp, int T, int C, const int32_t* __restrict__ lens, const float* __restrict__ emis,
    long long stride, const float* __restrict__ w, float* __restrict__ alpha, double* __restrict__ offs,
    float* __restrict__ den, int32_t* __restrict__ status) {
  GTNB_DYNAMIC_SMEM(float, sm);
  const int S = g.S, lanes = g.lanes, N = sp.N, nred = N * kSparseWarps;
  float* rows = sm; // [2][S]
  float* E = sm + 2 * S; // [2][C]
  float* red = E + 2 * C; // [2][nred]
  const int rank = (int)cluster_rank(), b = blockIdx.x / N, tid = threadIdx.x, nt = blockDim.x;
  const int n0 = sp.in[rank], n1 = sp.in[rank + 1]; // this CTA's nodes
  const int groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
  const int Tb = lens[b];
  const float* em = emis + (long long)b * stride;
  float* al = alpha + (long long)b * (T + 1) * S;
  double* of = offs + (long long)b * (T + 1);
  bool bad = false;
  cluster_first_row(g, 1, rows, rank == 0 ? al : nullptr, red, nred, 0);
  if (Tb > 0)
    for (int c = tid; c < C; c += nt) E[C + c] = __ldg(em + c); // row 0 in E[1]: frame t reads E[t & 1]
  cluster_sync_all(); // every CTA's first row is in place before a peer stores into its shared memory
  double c_off = 0.0;
  for (int t = 1; t <= Tb; t++) {
    const float* P = rows + ((t - 1) & 1) * S;
    float* Q = rows + (t & 1) * S;
    const float* Er = E + (t & 1) * C;
    if (t < Tb)
      for (int c = tid; c < C; c += nt) E[((t + 1) & 1) * C + c] = __ldg(em + (long long)t * C + c);
    const float Mp = cluster_row_offset(red + ((t - 1) & 1) * nred, nred);
    float mx = neg_inf();
    for (int v0 = n0; v0 < n1; v0 += groups) { // (the same trip count in every warp: the merge shuffles)
      const int v = v0 + grp;
      float m = neg_inf(), s = 0.0f;
      if (v < n1) {
        const int k1 = __ldg(g.in_ptr + v + 1);
        for (int k = __ldg(g.in_ptr + v) + q; k < k1; k += lanes) {
          const float wk = __ldg(w + __ldg(g.in_arc + k));
          const float ek = Er[__ldg(g.in_lab + k)];
          bad |= !(is_finite(wk) && is_finite(ek));
          lse_add(m, s, P[__ldg(g.in_src + k)] + (wk + ek));
        }
      }
      lse_merge(m, s, lanes);
      if (v < n1) {
        const float val = m == neg_inf() ? neg_inf() : (m + log_fast(s)) - Mp;
        if (q == 0) {
          cluster_store(Q + v, N, val);
          al[(long long)t * S + v] = val;
        }
        mx = fmaxf(mx, val);
      }
    }
    mx = warp_max(mx);
    if (tid % 32 == 0) cluster_store(red + (t & 1) * nred + rank * kSparseWarps + tid / 32, N, mx);
    cluster_arrive_only();
    c_off += (double)Mp;
    if (rank == 0 && tid == 0) of[t] = c_off;
    cluster_wait_only();
  }
  bad = __syncthreads_or(bad);
  if (bad && tid == 0) atomicOr(&status[b], 1);
  if (rank == 0 && tid < 32) {
    const float* F = rows + (Tb & 1) * S;
    float m = neg_inf();
    for (int v = tid; v < S; v += 32)
      if (__ldg(g.flags + v) & 2) m = fmaxf(m, F[v]);
    m = warp_max(m);
    float s = 0.0f;
    if (m != neg_inf())
      for (int v = tid; v < S; v += 32)
        if (__ldg(g.flags + v) & 2) s += expf(F[v] - m);
    s = warp_sum(s);
    if (tid == 0) {
      const double Z = m == neg_inf() ? (double)neg_inf() : c_off + (double)(m + logf(s));
      of[0] = Z;
      den[b] = (float)Z;
    }
  }
}

/* sparse_den_backward_kernel by a cluster: rank r adds the posteriors of its own nodes' out-arcs */
__global__ void __launch_bounds__(kSparseThreads) sparse_cl_den_backward_kernel(
    SparseDev g, SparseSplit sp, int T, int C, const int32_t* __restrict__ lens, const float* __restrict__ emis,
    long long stride, const float* __restrict__ w, const float* __restrict__ alpha, const double* __restrict__ offs,
    float* __restrict__ grad, long long grad_stride, float* __restrict__ wgrad) {
  GTNB_DYNAMIC_SMEM(float, sm);
  const int S = g.S, lanes = g.lanes, N = sp.N, nred = N * kSparseWarps;
  float* rows = sm; // [2][S] beta rows
  float* E = sm + 2 * S; // [2][C] emission rows
  float* Eg = E + 2 * C; // [2][C] the frame's emission gradient, this CTA's share
  float* red = Eg + 2 * C; // [2][nred]
  float* acc = red + 2 * nred; // [own out-arcs] arc gradient, by out-table position - ka
  const int rank = (int)cluster_rank(), b = blockIdx.x / N, tid = threadIdx.x, nt = blockDim.x;
  const int n0 = sp.out[rank], n1 = sp.out[rank + 1]; // this CTA's nodes
  const int ka = __ldg(g.out_ptr + n0), kn = __ldg(g.out_ptr + n1) - ka; // and their out-arcs
  const int groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
  const int Tb = lens[b];
  const double* of = offs + (long long)b * (T + 1);
  const double Z = of[0];
  if (Tb < 1 || !(fabs(Z) < (double)CUDART_INF_F)) return; // (the whole cluster)
  const float* em = emis + (long long)b * stride;
  const float* al = alpha + (long long)b * (T + 1) * S;
  float* gr = grad + (long long)b * grad_stride;
  cluster_first_row(g, 2, rows + (Tb & 1) * S, nullptr, red, nred, Tb & 1);
  for (int k = tid; k < kn; k += nt) acc[k] = 0.0f;
  for (int c = tid; c < 2 * C; c += nt) Eg[c] = 0.0f;
  for (int c = tid; c < C; c += nt) E[((Tb - 1) & 1) * C + c] = __ldg(em + (long long)(Tb - 1) * C + c);
  cluster_sync_all();
  double d = 0.0; // d_{t+1}
  for (int t = Tb - 1; t >= 0; t--) {
    const float* Nx = rows + ((t + 1) & 1) * S;
    float* Cur = rows + (t & 1) * S;
    const float* Er = E + (t & 1) * C;
    float* Eg_t = Eg + (t & 1) * C;
    float* Eg_prev = Eg + ((t + 1) & 1) * C; // frame t + 1's, complete since the barrier
    for (int c = tid; c < C; c += nt) {
      if (t > 0) E[((t + 1) & 1) * C + c] = __ldg(em + (long long)(t - 1) * C + c);
      if (t + 1 < Tb) {
        const float v = Eg_prev[c];
        if (v != 0.0f) atomicAdd(gr + (long long)(t + 1) * C + c, v);
        Eg_prev[c] = 0.0f;
      }
    }
    const float Mb = cluster_row_offset(red + ((t + 1) & 1) * nred, nred);
    const double c_t = t > 0 ? of[t] : 0.0;
    const float fo = (float)(c_t + d - Z);
    float mx = neg_inf();
    for (int u0 = n0; u0 < n1; u0 += groups) {
      const int u = u0 + grp;
      float m = neg_inf(), s = 0.0f;
      if (u < n1) {
        const float au = al[(long long)t * S + u] + fo; // alpha_t[u] + c_t + d_{t+1} - Z, in the exponent's terms
        const int k1 = __ldg(g.out_ptr + u + 1);
        for (int k = __ldg(g.out_ptr + u) + q; k < k1; k += lanes) {
          const int lab = __ldg(g.out_lab + k);
          const float x = Nx[__ldg(g.out_dst + k)] + (__ldg(w + __ldg(g.out_arc + k)) + Er[lab]);
          lse_add(m, s, x);
          const float p = exp_fast(au + x);
          if (p != 0.0f) {
            acc[k - ka] += p;
            atomicAdd(Eg_t + lab, p);
          }
        }
      }
      lse_merge(m, s, lanes);
      if (u < n1) {
        const float val = m == neg_inf() ? neg_inf() : (m + log_fast(s)) - Mb;
        if (q == 0) cluster_store(Cur + u, N, val);
        mx = fmaxf(mx, val);
      }
    }
    mx = warp_max(mx);
    if (tid % 32 == 0) cluster_store(red + (t & 1) * nred + rank * kSparseWarps + tid / 32, N, mx);
    cluster_arrive_only();
    d += (double)Mb;
    cluster_wait_only();
  }
  for (int c = tid; c < C; c += nt) { // frame 0's emission gradient
    const float v = Eg[c];
    if (v != 0.0f) atomicAdd(gr + c, v);
  }
  for (int k = tid; k < kn; k += nt)
    if (acc[k] != 0.0f) atomicAdd(wgrad + __ldg(g.out_arc + ka + k), acc[k]);
}

/* sparse_viterbi_forward_kernel by a cluster: the same back-pointers, head, score and status */
__global__ void __launch_bounds__(kSparseThreads) sparse_cl_viterbi_forward_kernel(
    SparseDev g, SparseSplit sp, int T, int C, const int32_t* __restrict__ lens, const float* __restrict__ emis,
    long long stride, const float* __restrict__ w, uint16_t* __restrict__ bp, int32_t* __restrict__ head,
    float* __restrict__ score, int32_t* __restrict__ status) {
  GTNB_DYNAMIC_SMEM(float, sm);
  const int S = g.S, lanes = g.lanes, N = sp.N;
  float* rows = sm; // [2][S]
  float* E = sm + 2 * S; // [2][C]
  const int rank = (int)cluster_rank(), b = blockIdx.x / N, tid = threadIdx.x, nt = blockDim.x;
  const int n0 = sp.in[rank], n1 = sp.in[rank + 1]; // this CTA's nodes
  const int groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
  const int Tb = lens[b];
  const float* em = emis + (long long)b * stride;
  uint16_t* bpb = bp + (long long)b * T * S;
  bool bad = false;
  for (int v = tid; v < S; v += nt) rows[v] = (__ldg(g.flags + v) & 1) ? 0.0f : neg_inf();
  if (Tb > 0)
    for (int c = tid; c < C; c += nt) E[C + c] = __ldg(em + c); // row 0 in E[1]: frame t reads E[t & 1]
  cluster_sync_all();
  for (int t = 1; t <= Tb; t++) {
    const float* P = rows + ((t - 1) & 1) * S;
    float* Q = rows + (t & 1) * S;
    const float* Er = E + (t & 1) * C;
    uint16_t* bpt = bpb + (long long)(t - 1) * S;
    if (t < Tb)
      for (int c = tid; c < C; c += nt) E[((t + 1) & 1) * C + c] = __ldg(em + (long long)t * C + c);
    for (int v0 = n0; v0 < n1; v0 += groups) { // (the same trip count in every warp: the merge shuffles)
      const int v = v0 + grp;
      float m = neg_inf();
      int k = 0x7fffffff, tie = 0, k0 = 0;
      if (v < n1) {
        k0 = __ldg(g.in_ptr + v);
        const int k1 = __ldg(g.in_ptr + v + 1);
        for (int j = k0 + q; j < k1; j += lanes) {
          const float wk = __ldg(w + __ldg(g.in_arc + j));
          const float ek = Er[__ldg(g.in_lab + j)];
          bad |= !(wk < CUDART_INF_F && ek < CUDART_INF_F);
          argmax_add(m, k, tie, P[__ldg(g.in_src + j)] + (wk + ek), j);
        }
      }
      argmax_merge(m, k, tie, lanes);
      if (v < n1 && q == 0) {
        cluster_store(Q + v, N, m);
        bpt[v] = m == neg_inf() ? kBpNone : (uint16_t)((k - k0) | (tie ? kBpTie : 0));
      }
    }
    cluster_sync_all();
  }
  bad = __syncthreads_or(bad);
  if (bad && tid == 0) atomicOr(&status[b], 1);
  if (rank == 0 && tid < 32) {
    const float* F = rows + (Tb & 1) * S;
    float m = neg_inf();
    int k = 0x7fffffff, tie = 0;
    if (Tb > 0)
      for (int v = tid; v < S; v += 32)
        if (__ldg(g.flags + v) & 2) argmax_add(m, k, tie, F[v], v);
    argmax_merge(m, k, tie, 32);
    if (tid == 0) {
      head[b] = m == neg_inf() ? -1 : k;
      score[b] = m;
      if (tie) atomicOr(&status[b], 2);
    }
  }
}

/*
 * The backoff sweeps: the kernels above over an acceptor with epsilon arcs (SparseEpsDev, gtnb_meta.h), one CTA per
 * utterance.  An epsilon arc consumes no frame, so every frame's row, frame 0's and frame T_b's included, is closed
 * over the epsilon arcs after its emitting update, one topological level at a time with one CTA barrier per level.
 * The CTA's graph is gs[b] when per_cta (the numerators: every utterance its own product A_b o G, its score rows at
 * gs[b].rows) and gs[0] otherwise (the denominator, G for the whole batch).
 */

/*
 * The team that closes a row over the epsilon levels.  OneCta: the CTA closes every node of a level, and a CTA barrier
 * ends the level.  Cluster: rank `rank` of a cluster of N CTAs (the sparse_cl_eps_* kernels below) closes its run of
 * each level, cut[(d * L + l) * (N + 1) + rank .. + 1] (d = 0 forward, 1 backward), stores each result into every
 * CTA through distributed shared memory, and a barrier.cluster ends the level.  The closure helpers are written once
 * over the team, so a node is closed by the same threads over the same arcs in the same order either way.
 */
struct OneCta {
  /* the level table of each direction, and this CTA's nodes [n0, n1) of level l in it */
  __device__ __forceinline__ const int32_t* fwd_levels(const SparseEpsDev& x) const { return x.fwd_ptr; }
  __device__ __forceinline__ const int32_t* bwd_levels(const SparseEpsDev& x) const { return x.bwd_ptr; }
  __device__ __forceinline__ void level(const int32_t* lv, int l, int& n0, int& n1) const {
    n0 = __ldg(lv + l), n1 = __ldg(lv + l + 1);
  }
  __device__ __forceinline__ bool owns(int, int, int) const { return true; } // node v of this CTA's [n0, n1)
  __device__ __forceinline__ void put(float* p, float v) const { *p = v; }
  __device__ __forceinline__ void sync() const { __syncthreads(); }
};

struct Cluster {
  const int32_t* cut; // [2][L][N + 1] (sparse_eps_cluster_cuts, gtnb_product.h)
  int N, rank;
  __device__ __forceinline__ const int32_t* fwd_levels(const SparseEpsDev&) const { return cut; }
  __device__ __forceinline__ const int32_t* bwd_levels(const SparseEpsDev& x) const { return cut + x.L * (N + 1); }
  __device__ __forceinline__ void level(const int32_t* lv, int l, int& n0, int& n1) const {
    n0 = __ldg(lv + l * (N + 1) + rank), n1 = __ldg(lv + l * (N + 1) + rank + 1);
  }
  __device__ __forceinline__ bool owns(int v, int n0, int n1) const { return v >= n0 && v < n1; }
  __device__ __forceinline__ void put(float* p, float v) const { cluster_store(p, N, v); }
  __device__ __forceinline__ void sync() const { cluster_sync_all(); }
};

/* the closure of row R over the forward levels, R[v] = logadd(R[v], logsumexp over v's epsilon in-arcs u -> v of
 * R[u] + w): rows relative to one offset stay so.  bad |= a non-finite epsilon weight.  Ends on the team's barrier. */
template <class Team>
__device__ __forceinline__ void eps_close_fwd(Team team, const SparseEpsDev& x, const float* __restrict__ w, float* R,
                                              bool& bad) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const int32_t* lv = team.fwd_levels(x);
  for (int l = 0; l < x.L; l++) {
    const int lanes = __ldg(x.lanes + l), groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
    int n0, n1;
    team.level(lv, l, n0, n1);
    for (int i0 = n0; i0 < n1; i0 += groups) { // (the same trip count in every warp: the merge shuffles)
      const int i = i0 + grp;
      float m = neg_inf(), s = 0.0f;
      int v = 0;
      if (i < n1) {
        v = __ldg(x.fwd_node + i);
        const int k1 = __ldg(x.eps_in_ptr + v + 1);
        for (int k = __ldg(x.eps_in_ptr + v) + q; k < k1; k += lanes) {
          const float wk = __ldg(w + __ldg(x.eps_in_arc + k));
          bad |= !is_finite(wk);
          lse_add(m, s, R[__ldg(x.eps_in_src + k)] + wk);
        }
      }
      lse_merge(m, s, lanes);
      if (i < n1 && q == 0 && m != neg_inf()) {
        lse_add(m, s, R[v]);
        team.put(R + v, m + log_fast(s));
      }
    }
    team.sync();
  }
}

/* the closure of a beta row R over the backward levels, R[u] = logadd(R[u], logsumexp over u's epsilon out-arcs
 * u -> v of w + R[v]), and the posterior exp(al[u] + fo + w + R[v]) of each epsilon arc added into acc[k - ea] (k: its
 * position in the epsilon out-table; ea: the team's first; fo = c_t + d_t - Z, R relative to d_t).  Ends on the
 * team's barrier. */
template <class Team>
__device__ __forceinline__ void eps_close_bwd(Team team, const SparseEpsDev& x, const float* __restrict__ w, float* R,
                                              const float* __restrict__ al, float fo, float* acc, int ea) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const int32_t* lv = team.bwd_levels(x);
  for (int l = 0; l < x.L; l++) {
    const int lanes = __ldg(x.lanes + x.L + l), groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
    int n0, n1;
    team.level(lv, l, n0, n1);
    for (int i0 = n0; i0 < n1; i0 += groups) {
      const int i = i0 + grp;
      float m = neg_inf(), s = 0.0f;
      int u = 0;
      if (i < n1) {
        u = __ldg(x.bwd_node + i);
        const float au = al[u] + fo;
        const int k1 = __ldg(x.eps_out_ptr + u + 1);
        for (int k = __ldg(x.eps_out_ptr + u) + q; k < k1; k += lanes) {
          const float xk = __ldg(w + __ldg(x.eps_out_arc + k)) + R[__ldg(x.eps_out_dst + k)];
          lse_add(m, s, xk);
          const float p = exp_fast(au + xk);
          if (p != 0.0f) acc[k - ea] += p;
        }
      }
      lse_merge(m, s, lanes);
      if (i < n1 && q == 0 && m != neg_inf()) {
        lse_add(m, s, R[u]);
        team.put(R + u, m + log_fast(s));
      }
    }
    team.sync();
  }
}

/* the tropical closure of row R over the forward levels: an epsilon arc u -> v wins over v's score when fl(R[u] + w)
 * is larger; bp[v] then gets its position in v's combined in-list (the ne emitting in-arcs first), and the tie flag
 * when another candidate, of either kind, reaches the same finite maximum.  bad |= a NaN or +inf epsilon weight. */
template <class Team>
__device__ __forceinline__ void eps_close_trop(Team team, const SparseEpsDev& x, const float* __restrict__ w, float* R,
                                               uint16_t* bp, bool& bad) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const int32_t* lv = team.fwd_levels(x);
  for (int l = 0; l < x.L; l++) {
    const int lanes = __ldg(x.lanes + l), groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
    int n0, n1;
    team.level(lv, l, n0, n1);
    for (int i0 = n0; i0 < n1; i0 += groups) {
      const int i = i0 + grp;
      float m = neg_inf();
      int k = 0x7fffffff, tie = 0, v = 0, k0 = 0;
      if (i < n1) {
        v = __ldg(x.fwd_node + i);
        k0 = __ldg(x.eps_in_ptr + v);
        const int k1 = __ldg(x.eps_in_ptr + v + 1);
        for (int j = k0 + q; j < k1; j += lanes) {
          const float wk = __ldg(w + __ldg(x.eps_in_arc + j));
          bad |= !(wk < CUDART_INF_F);
          argmax_add(m, k, tie, R[__ldg(x.eps_in_src + j)] + wk, j);
        }
      }
      argmax_merge(m, k, tie, lanes);
      if (i < n1 && q == 0) {
        const float cur = R[v];
        if (m > cur) {
          const int ne = __ldg(x.g.in_ptr + v + 1) - __ldg(x.g.in_ptr + v);
          team.put(R + v, m);
          bp[v] = (uint16_t)((ne + k - k0) | (tie ? kBpTie : 0));
        } else if (m == cur && m != neg_inf()) {
          bp[v] |= kBpTie;
        }
      }
    }
    team.sync();
  }
}

/* the maximum of a closed row R, whole in every CTA of the team, into red[nt / 32] (merged after the CTA barrier that
 * follows, by row_offset in one CTA and cluster_row_offset in a cluster); R[v] to out[v] (nullable) for this CTA's
 * nodes [n0, n1) */
template <class Team>
__device__ __forceinline__ void row_max(Team team, const float* R, int S, int n0, int n1, float* out, float* red) {
  float mx = neg_inf();
  for (int v = threadIdx.x; v < S; v += blockDim.x) {
    const float r = R[v];
    if (out && team.owns(v, n0, n1)) out[v] = r;
    mx = fmaxf(mx, r);
  }
  mx = warp_max(mx);
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = mx;
}

/*
 * sparse_den_forward_kernel with the epsilon closure: alpha rows (after the closure) to alpha + the CTA's row base,
 * c_t to offs[b][t], Z to offs[b][0] and den[b]; status[b] |= 1 on a non-finite weight or used emission.
 */
__global__ void __launch_bounds__(kSparseThreads) sparse_eps_forward_kernel(
    const SparseEpsDev* __restrict__ gs, int per_cta, int T, int C, const int32_t* __restrict__ lens,
    const float* __restrict__ emis, long long stride, const float* __restrict__ w, float* __restrict__ alpha,
    double* __restrict__ offs, float* __restrict__ den, int32_t* __restrict__ status) {
  GTNB_DYNAMIC_SMEM(float, sm);
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const SparseEpsDev x = gs[per_cta ? b : 0];
  const SparseDev& g = x.g;
  const int S = g.S, lanes = g.lanes;
  float* rows = sm; // [2][S]
  float* E = sm + 2 * S; // [2][C]
  float* red = E + 2 * C; // [2][kSparseWarps]
  const int groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
  const int Tb = lens[b];
  const float* em = emis + (long long)b * stride;
  float* al = alpha + (per_cta ? x.rows : (long long)b * (T + 1) * S);
  double* of = offs + (long long)b * (T + 1);
  bool bad = false;
  for (int v = tid; v < S; v += nt) rows[v] = (__ldg(g.flags + v) & 1) ? 0.0f : neg_inf();
  if (Tb > 0)
    for (int c = tid; c < C; c += nt) E[C + c] = __ldg(em + c); // row 0 in E[1]: frame t reads E[t & 1]
  __syncthreads();
  eps_close_fwd(OneCta(), x, w, rows, bad);
  row_max(OneCta(), rows, S, 0, S, al, red);
  __syncthreads();
  double c_off = 0.0;
  for (int t = 1; t <= Tb; t++) {
    const float* P = rows + ((t - 1) & 1) * S;
    float* Q = rows + (t & 1) * S;
    const float* Er = E + (t & 1) * C;
    if (t < Tb)
      for (int c = tid; c < C; c += nt) E[((t + 1) & 1) * C + c] = __ldg(em + (long long)t * C + c);
    const float Mp = row_offset(red + ((t - 1) & 1) * kSparseWarps);
    for (int v0 = 0; v0 < S; v0 += groups) {
      const int v = v0 + grp;
      float m = neg_inf(), s = 0.0f;
      if (v < S) {
        const int k1 = __ldg(g.in_ptr + v + 1);
        for (int k = __ldg(g.in_ptr + v) + q; k < k1; k += lanes) {
          const float wk = __ldg(w + __ldg(g.in_arc + k));
          const float ek = Er[__ldg(g.in_lab + k)];
          bad |= !(is_finite(wk) && is_finite(ek));
          lse_add(m, s, P[__ldg(g.in_src + k)] + (wk + ek));
        }
      }
      lse_merge(m, s, lanes);
      if (v < S && q == 0) Q[v] = m == neg_inf() ? neg_inf() : (m + log_fast(s)) - Mp;
    }
    __syncthreads();
    eps_close_fwd(OneCta(), x, w, Q, bad);
    row_max(OneCta(), Q, S, 0, S, al + (long long)t * S, red + (t & 1) * kSparseWarps);
    c_off += (double)Mp;
    if (tid == 0) of[t] = c_off;
    __syncthreads();
  }
  bad = __syncthreads_or(bad);
  if (tid < 32) {
    const float* F = rows + (Tb & 1) * S;
    float m = neg_inf();
    for (int v = tid; v < S; v += 32)
      if (__ldg(g.flags + v) & 2) m = fmaxf(m, F[v]);
    m = warp_max(m);
    float s = 0.0f;
    if (m != neg_inf())
      for (int v = tid; v < S; v += 32)
        if (__ldg(g.flags + v) & 2) s += expf(F[v] - m);
    s = warp_sum(s);
    if (tid == 0) {
      const double Z = m == neg_inf() ? (double)neg_inf() : c_off + (double)(m + logf(s));
      of[0] = Z;
      den[b] = (float)Z;
      if (bad) atomicOr(&status[b], 1);
    }
  }
}

/*
 * sparse_den_backward_kernel with the epsilon closure: sgn * d Z / d e added into grad and sgn * d Z / d w into
 * wgrad (the numerators: sgn = -1), an epsilon arc's posterior exp(alpha_t[u] + w + beta_t[v] - Z) into wgrad alone.
 */
__global__ void __launch_bounds__(kSparseThreads) sparse_eps_backward_kernel(
    const SparseEpsDev* __restrict__ gs, int per_cta, int T, int C, const int32_t* __restrict__ lens,
    const float* __restrict__ emis, long long stride, const float* __restrict__ w, const float* __restrict__ alpha,
    const double* __restrict__ offs, float sgn, float* __restrict__ grad, long long grad_stride,
    float* __restrict__ wgrad) {
  GTNB_DYNAMIC_SMEM(float, sm);
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const SparseEpsDev x = gs[per_cta ? b : 0];
  const SparseDev& g = x.g;
  const int S = g.S, A = g.A, lanes = g.lanes;
  float* rows = sm; // [2][S] beta rows
  float* E = sm + 2 * S; // [2][C] emission rows
  float* Eg = E + 2 * C; // [2][C] the frame's emission gradient
  float* acc = Eg + 2 * C; // [A + E] arc gradient, by out-table position, then by epsilon out-table position
  float* red = acc + A + x.E; // [2][kSparseWarps]
  const int groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
  const int Tb = lens[b];
  const double* of = offs + (long long)b * (T + 1);
  const double Z = of[0];
  if (Tb < 1 || !(fabs(Z) < (double)CUDART_INF_F)) return;
  const float* em = emis + (long long)b * stride;
  const float* al = alpha + (per_cta ? x.rows : (long long)b * (T + 1) * S);
  float* gr = grad + (long long)b * grad_stride;
  for (int v = tid; v < S; v += nt) rows[(Tb & 1) * S + v] = (__ldg(g.flags + v) & 2) ? 0.0f : neg_inf();
  for (int k = tid; k < A + x.E; k += nt) acc[k] = 0.0f;
  for (int c = tid; c < 2 * C; c += nt) Eg[c] = 0.0f;
  for (int c = tid; c < C; c += nt) E[((Tb - 1) & 1) * C + c] = __ldg(em + (long long)(Tb - 1) * C + c);
  __syncthreads();
  eps_close_bwd(OneCta(), x, w, rows + (Tb & 1) * S, al + (long long)Tb * S, (float)(of[Tb] - Z), acc + A, 0);
  row_max(OneCta(), rows + (Tb & 1) * S, S, 0, S, nullptr, red + (Tb & 1) * kSparseWarps);
  __syncthreads();
  double d = 0.0; // d_{t+1}
  for (int t = Tb - 1; t >= 0; t--) {
    const float* Nx = rows + ((t + 1) & 1) * S;
    float* Cur = rows + (t & 1) * S;
    const float* Er = E + (t & 1) * C;
    float* Eg_t = Eg + (t & 1) * C;
    float* Eg_prev = Eg + ((t + 1) & 1) * C; // frame t + 1's, complete since the barrier
    for (int c = tid; c < C; c += nt) {
      if (t > 0) E[((t + 1) & 1) * C + c] = __ldg(em + (long long)(t - 1) * C + c);
      if (t + 1 < Tb) {
        const float v = Eg_prev[c];
        if (v != 0.0f) atomicAdd(gr + (long long)(t + 1) * C + c, sgn * v);
        Eg_prev[c] = 0.0f;
      }
    }
    const float Mb = row_offset(red + ((t + 1) & 1) * kSparseWarps);
    const double c_t = t > 0 ? of[t] : 0.0;
    const float fo = (float)(c_t + d - Z);
    for (int u0 = 0; u0 < S; u0 += groups) {
      const int u = u0 + grp;
      float m = neg_inf(), s = 0.0f;
      if (u < S) {
        const float au = al[(long long)t * S + u] + fo;
        const int k1 = __ldg(g.out_ptr + u + 1);
        for (int k = __ldg(g.out_ptr + u) + q; k < k1; k += lanes) {
          const int lab = __ldg(g.out_lab + k);
          const float xk = Nx[__ldg(g.out_dst + k)] + (__ldg(w + __ldg(g.out_arc + k)) + Er[lab]);
          lse_add(m, s, xk);
          const float p = exp_fast(au + xk);
          if (p != 0.0f) {
            acc[k] += p;
            atomicAdd(Eg_t + lab, p);
          }
        }
      }
      lse_merge(m, s, lanes);
      if (u < S && q == 0) Cur[u] = m == neg_inf() ? neg_inf() : (m + log_fast(s)) - Mb;
    }
    __syncthreads();
    eps_close_bwd(OneCta(), x, w, Cur, al + (long long)t * S, (float)(c_t + (d + (double)Mb) - Z), acc + A, 0);
    row_max(OneCta(), Cur, S, 0, S, nullptr, red + (t & 1) * kSparseWarps);
    d += (double)Mb;
    __syncthreads();
  }
  for (int c = tid; c < C; c += nt) { // frame 0's emission gradient
    const float v = Eg[c];
    if (v != 0.0f) atomicAdd(gr + c, sgn * v);
  }
  for (int k = tid; k < A; k += nt)
    if (acc[k] != 0.0f) atomicAdd(wgrad + __ldg(g.out_arc + k), sgn * acc[k]);
  for (int k = tid; k < x.E; k += nt)
    if (acc[A + k] != 0.0f) atomicAdd(wgrad + __ldg(x.eps_out_arc + k), sgn * acc[A + k]);
}

/*
 * sparse_viterbi_forward_kernel with the epsilon closure over graph x = gs[gi] for utterance b = blockIdx.x.  bpb[t][v]
 * (t = 0 .. T_b; bpb = bp + rows_at(b, x), the utterance's back-pointers): the position of the arc that reaches S_t[v] in v's combined in-list
 * (its emitting in-arcs from frame t - 1, then its epsilon in-arcs from frame t), kBpStart for a start node at frame 0
 * that no epsilon arc improves, | kBpTie on a tie; kBpNone where S_t[v] = -inf.
 */
template <class Rows>
__device__ __forceinline__ void eps_viterbi_sweep(const SparseEpsDev* __restrict__ gs, int gi, int C,
                                                  const int32_t* __restrict__ lens,
                                                  const float* __restrict__ emis, long long stride,
                                                  const float* __restrict__ w, uint16_t* __restrict__ bp,
                                                  Rows rows_at, int32_t* __restrict__ head,
                                                  float* __restrict__ score, int32_t* __restrict__ status) {
  GTNB_DYNAMIC_SMEM(float, sm);
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const SparseEpsDev x = gs[gi];
  const SparseDev& g = x.g;
  const int S = g.S, lanes = g.lanes;
  float* rows = sm; // [2][S]
  float* E = sm + 2 * S; // [2][C]
  const int groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
  const int Tb = lens[b];
  const float* em = emis + (long long)b * stride;
  uint16_t* bpb = bp + rows_at(b, x);
  bool bad = false;
  for (int v = tid; v < S; v += nt) {
    const bool st = __ldg(g.flags + v) & 1;
    rows[v] = st ? 0.0f : neg_inf();
    bpb[v] = st ? (uint16_t)kBpStart : kBpNone;
  }
  if (Tb > 0)
    for (int c = tid; c < C; c += nt) E[C + c] = __ldg(em + c); // row 0 in E[1]: frame t reads E[t & 1]
  __syncthreads();
  eps_close_trop(OneCta(), x, w, rows, bpb, bad);
  for (int t = 1; t <= Tb; t++) {
    const float* P = rows + ((t - 1) & 1) * S;
    float* Q = rows + (t & 1) * S;
    const float* Er = E + (t & 1) * C;
    uint16_t* bpt = bpb + (long long)t * S;
    if (t < Tb)
      for (int c = tid; c < C; c += nt) E[((t + 1) & 1) * C + c] = __ldg(em + (long long)t * C + c);
    for (int v0 = 0; v0 < S; v0 += groups) {
      const int v = v0 + grp;
      float m = neg_inf();
      int k = 0x7fffffff, tie = 0, k0 = 0;
      if (v < S) {
        k0 = __ldg(g.in_ptr + v);
        const int k1 = __ldg(g.in_ptr + v + 1);
        for (int j = k0 + q; j < k1; j += lanes) {
          const float wk = __ldg(w + __ldg(g.in_arc + j));
          const float ek = Er[__ldg(g.in_lab + j)];
          bad |= !(wk < CUDART_INF_F && ek < CUDART_INF_F);
          argmax_add(m, k, tie, P[__ldg(g.in_src + j)] + (wk + ek), j);
        }
      }
      argmax_merge(m, k, tie, lanes);
      if (v < S && q == 0) {
        Q[v] = m;
        bpt[v] = m == neg_inf() ? kBpNone : (uint16_t)((k - k0) | (tie ? kBpTie : 0));
      }
    }
    __syncthreads();
    eps_close_trop(OneCta(), x, w, Q, bpt, bad); // (its last barrier ends the frame)
  }
  bad = __syncthreads_or(bad);
  if (tid < 32) {
    const float* F = rows + (Tb & 1) * S;
    float m = neg_inf();
    int k = 0x7fffffff, tie = 0;
    if (Tb > 0)
      for (int v = tid; v < S; v += 32)
        if (__ldg(g.flags + v) & 2) argmax_add(m, k, tie, F[v], v);
    argmax_merge(m, k, tie, 32);
    if (tid == 0) {
      head[b] = m == neg_inf() ? -1 : k;
      score[b] = m;
      const int st = (bad ? 1 : 0) | (tie ? 2 : 0);
      if (st) atomicOr(&status[b], st);
    }
  }
}

/* the decode's sweep, G = gs[0] for every utterance; bp: [B][T + 1][S] */
__global__ void __launch_bounds__(kSparseThreads) sparse_eps_viterbi_kernel(
    const SparseEpsDev* __restrict__ gs, int T, int C, const int32_t* __restrict__ lens,
    const float* __restrict__ emis, long long stride, const float* __restrict__ w, uint16_t* __restrict__ bp,
    int32_t* __restrict__ head, float* __restrict__ score, int32_t* __restrict__ status) {
  eps_viterbi_sweep(gs, 0, C, lens, emis, stride, w, bp,
                    [&](int b, const SparseEpsDev& x) { return (long long)b * (T + 1) * x.g.S; }, head, score,
                    status);
}

/* the alignment's sweep (gtnb_backoff_transitions_viterbi), every CTA its own numerator gs[b] = P_b: its
 * back-pointers at bp + gs[b].rows, (T_b + 1) * S_b of them, the layout of the loss's score rows */
__global__ void __launch_bounds__(kSparseThreads) sparse_eps_align_kernel(
    const SparseEpsDev* __restrict__ gs, int C, const int32_t* __restrict__ lens, const float* __restrict__ emis,
    long long stride, const float* __restrict__ w, uint16_t* __restrict__ bp, int32_t* __restrict__ head,
    float* __restrict__ score, int32_t* __restrict__ status) {
  eps_viterbi_sweep(gs, blockIdx.x, C, lens, emis, stride, w, bp, [](int, const SparseEpsDev& x) { return x.rows; },
                    head, score, status);
}

/*
 * The traceback of eps_viterbi_sweep for utterance b over graph x, its back-pointers at bp + rows_at(S), by lane 0 of
 * its warp (the other lanes only write the row's tail): inside a frame it follows epsilon back-pointers (they use no frame and are not reported), and an emitting
 * one writes paths[b][t - 1] = its label / arcs[b][t - 1] = arc(its arc id) and steps to frame t - 1; it ends at
 * frame 0 on kBpStart.  -1 beyond T_b and in the whole row without a path.  status[b] |= 2 when a node of the path
 * carries the tie flag.
 */
template <class Rows, class Arc>
__device__ __forceinline__ void eps_trace(const SparseEpsDev& x, int b, int T, const int32_t* __restrict__ lens,
                                          const uint16_t* __restrict__ bp, Rows rows_at,
                                          const int32_t* __restrict__ head, int32_t* __restrict__ paths,
                                          int32_t* __restrict__ arcs, int32_t* __restrict__ status, Arc arc) {
  const int lane = threadIdx.x % 32;
  const int h = head[b];
  const int n = h < 0 ? 0 : lens[b];
  int32_t* pr = paths ? paths + (long long)b * T : nullptr;
  int32_t* ar = arcs ? arcs + (long long)b * T : nullptr;
  for (int t = n + lane; t < T; t += 32) {
    if (pr) pr[t] = -1;
    if (ar) ar[t] = -1;
  }
  if (lane != 0 || n == 0) return;
  const int S = x.g.S;
  const uint16_t* bpb = bp + rows_at(S);
  int v = h, tie = 0, t = n;
  for (;;) {
    const int e = __ldg(bpb + (long long)t * S + v);
    if (e == kBpNone) break; // (not on a path from a finite head)
    const int pos = e & (kBpTie - 1);
    tie |= e & kBpTie;
    if (t == 0 && pos == kBpStart) break;
    const int k0 = __ldg(x.g.in_ptr + v), ne = __ldg(x.g.in_ptr + v + 1) - k0;
    if (pos >= ne) { // an epsilon arc inside frame t
      v = __ldg(x.eps_in_src + __ldg(x.eps_in_ptr + v) + pos - ne);
      continue;
    }
    const int k = k0 + pos;
    if (pr) pr[t - 1] = __ldg(x.g.in_lab + k);
    if (ar) ar[t - 1] = arc(__ldg(x.g.in_arc + k));
    v = __ldg(x.g.in_src + k);
    t--;
  }
  if (tie) atomicOr(&status[b], 2);
}

/* the decode's traceback, one warp per utterance: G's arc ids */
__global__ void __launch_bounds__(256) sparse_eps_trace_kernel(
    const SparseEpsDev* __restrict__ gs, int B, int T, const int32_t* __restrict__ lens,
    const uint16_t* __restrict__ bp, const int32_t* __restrict__ head, int32_t* __restrict__ paths,
    int32_t* __restrict__ arcs, int32_t* __restrict__ status) {
  const int b = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
  if (b >= B) return; // whole warps
  const SparseEpsDev x = gs[0];
  eps_trace(x, b, T, lens, bp, [&](int S) { return (long long)b * (T + 1) * S; }, head, paths, arcs, status,
            [](int a) { return a; });
}

/* the alignment's traceback, one warp per utterance over its numerator gs[b]: the product arc's A arc, arc_of (the
 * loss's table, the batch's numbering) less a_first[b], utterance b's first A arc, so A_b's own numbering */
__global__ void __launch_bounds__(256) sparse_eps_align_trace_kernel(
    const SparseEpsDev* __restrict__ gs, int B, int T, const int32_t* __restrict__ lens,
    const uint16_t* __restrict__ bp, const int32_t* __restrict__ head, const int32_t* __restrict__ arc_of,
    const int32_t* __restrict__ a_first, int32_t* __restrict__ paths, int32_t* __restrict__ arcs,
    int32_t* __restrict__ status) {
  const int b = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
  if (b >= B) return; // whole warps
  const SparseEpsDev x = gs[b];
  eps_trace(x, b, T, lens, bp, [&](int) { return x.rows; }, head, paths, arcs, status,
            [&](int a) { return __ldg(arc_of + a) - __ldg(a_first + b); });
}

/*
 * The backoff cluster sweeps: the denominator's sparse_eps_* sweeps (G = gs[0] for every utterance) for a G that one
 * CTA's shared memory cannot hold, one thread-block cluster of N = sp.N CTAs per utterance, the layout of the
 * sparse_cl_* kernels with the closure of the sparse_eps_* ones.  A rank closes the nodes of each level that it owns
 * in the emitting update (sp.in in the forward and the tropical sweep, sp.out in the backward): a level lists its
 * nodes in ascending id, so they are one contiguous run of it, cut[(d * L + l) * (N + 1) + rank] .. [... + rank + 1]
 * (d = 0 forward, 1 backward; sparse_eps_cluster_cuts, gtnb_product.h), and one barrier.cluster per level replaces
 * the CTA barrier.  A level reads only nodes of earlier levels and its own node, so no store lands in an entry a peer
 * reads before the barrier.  A node keeps its owner through the frame, so its alpha entry, its back-pointer and its
 * later tie flag are written by one CTA.  After the last level every CTA holds the whole closed row and takes its
 * maximum itself (a maximum does not depend on the order) behind a CTA barrier.  Per frame: 1 + L cluster barriers
 * and one CTA barrier, against the one-CTA kernels' 2 + L CTA barriers; rows, offsets, Z, back-pointers, head, score
 * and status are theirs bit for bit.  The backward's accumulators hold the rank's own emitting and epsilon out-arcs,
 * flushed with red.add, so only the order of the adds into grad and wgrad differs.  The launch bounds ask for two
 * CTAs per SM: ptxas then allots 64 registers (63 in the backward) and spills nothing (without the minimum it chose
 * 40 / 64 and spilled).
 */

/* sparse_eps_forward_kernel (per_cta off) by a cluster: the same alpha rows, offsets, Z, den and status */
__global__ void __launch_bounds__(kSparseThreads, 2) sparse_cl_eps_forward_kernel(
    const SparseEpsDev* __restrict__ gs, SparseSplit sp, const int32_t* __restrict__ cut, int T, int C,
    const int32_t* __restrict__ lens, const float* __restrict__ emis, long long stride, const float* __restrict__ w,
    float* __restrict__ alpha, double* __restrict__ offs, float* __restrict__ den, int32_t* __restrict__ status) {
  GTNB_DYNAMIC_SMEM(float, sm);
  const SparseEpsDev x = gs[0];
  const SparseDev& g = x.g;
  const int S = g.S, lanes = g.lanes, N = sp.N;
  float* rows = sm; // [2][S]
  float* E = sm + 2 * S; // [2][C]
  float* red = E + 2 * C; // [2][kSparseWarps]: this CTA's per-warp maxima of the closed rows
  const int rank = (int)cluster_rank(), b = blockIdx.x / N, tid = threadIdx.x, nt = blockDim.x;
  const int n0 = sp.in[rank], n1 = sp.in[rank + 1]; // this CTA's nodes
  const Cluster team{cut, N, rank}; // the closure's
  const int groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
  const int Tb = lens[b];
  const float* em = emis + (long long)b * stride;
  float* al = alpha + (long long)b * (T + 1) * S;
  double* of = offs + (long long)b * (T + 1);
  bool bad = false;
  for (int v = tid; v < S; v += nt) rows[v] = (__ldg(g.flags + v) & 1) ? 0.0f : neg_inf();
  if (Tb > 0)
    for (int c = tid; c < C; c += nt) E[C + c] = __ldg(em + c); // row 0 in E[1]: frame t reads E[t & 1]
  cluster_sync_all(); // every CTA's first row is in place before a peer stores into its shared memory
  eps_close_fwd(team, x, w, rows, bad);
  row_max(team, rows, S, n0, n1, al, red);
  __syncthreads();
  double c_off = 0.0;
  for (int t = 1; t <= Tb; t++) {
    const float* P = rows + ((t - 1) & 1) * S;
    float* Q = rows + (t & 1) * S;
    const float* Er = E + (t & 1) * C;
    if (t < Tb)
      for (int c = tid; c < C; c += nt) E[((t + 1) & 1) * C + c] = __ldg(em + (long long)t * C + c);
    const float Mp = cluster_row_offset(red + ((t - 1) & 1) * kSparseWarps, nt / 32);
    for (int v0 = n0; v0 < n1; v0 += groups) { // (the same trip count in every warp: the merge shuffles)
      const int v = v0 + grp;
      float m = neg_inf(), s = 0.0f;
      if (v < n1) {
        const int k1 = __ldg(g.in_ptr + v + 1);
        for (int k = __ldg(g.in_ptr + v) + q; k < k1; k += lanes) {
          const float wk = __ldg(w + __ldg(g.in_arc + k));
          const float ek = Er[__ldg(g.in_lab + k)];
          bad |= !(is_finite(wk) && is_finite(ek));
          lse_add(m, s, P[__ldg(g.in_src + k)] + (wk + ek));
        }
      }
      lse_merge(m, s, lanes);
      if (v < n1 && q == 0) cluster_store(Q + v, N, m == neg_inf() ? neg_inf() : (m + log_fast(s)) - Mp);
    }
    cluster_sync_all();
    eps_close_fwd(team, x, w, Q, bad); // (its last barrier: the closed row is whole in every CTA)
    row_max(team, Q, S, n0, n1, al + (long long)t * S, red + (t & 1) * kSparseWarps);
    c_off += (double)Mp;
    if (rank == 0 && tid == 0) of[t] = c_off;
    __syncthreads();
  }
  bad = __syncthreads_or(bad);
  if (bad && tid == 0) atomicOr(&status[b], 1);
  if (rank == 0 && tid < 32) {
    const float* F = rows + (Tb & 1) * S;
    float m = neg_inf();
    for (int v = tid; v < S; v += 32)
      if (__ldg(g.flags + v) & 2) m = fmaxf(m, F[v]);
    m = warp_max(m);
    float s = 0.0f;
    if (m != neg_inf())
      for (int v = tid; v < S; v += 32)
        if (__ldg(g.flags + v) & 2) s += expf(F[v] - m);
    s = warp_sum(s);
    if (tid == 0) {
      const double Z = m == neg_inf() ? (double)neg_inf() : c_off + (double)(m + logf(s));
      of[0] = Z;
      den[b] = (float)Z;
    }
  }
}

/* sparse_eps_backward_kernel (per_cta off, sgn = 1) by a cluster: rank r adds the posteriors of its own nodes'
 * emitting and epsilon out-arcs */
__global__ void __launch_bounds__(kSparseThreads, 2) sparse_cl_eps_backward_kernel(
    const SparseEpsDev* __restrict__ gs, SparseSplit sp, const int32_t* __restrict__ cut, int T, int C,
    const int32_t* __restrict__ lens, const float* __restrict__ emis, long long stride, const float* __restrict__ w,
    const float* __restrict__ alpha, const double* __restrict__ offs, float* __restrict__ grad, long long grad_stride,
    float* __restrict__ wgrad) {
  GTNB_DYNAMIC_SMEM(float, sm);
  const SparseEpsDev x = gs[0];
  const SparseDev& g = x.g;
  const int S = g.S, lanes = g.lanes, N = sp.N;
  float* rows = sm; // [2][S] beta rows
  float* E = sm + 2 * S; // [2][C] emission rows
  float* Eg = E + 2 * C; // [2][C] the frame's emission gradient, this CTA's share
  float* red = Eg + 2 * C; // [2][kSparseWarps]
  float* acc = red + 2 * kSparseWarps; // own emitting out-arcs (by out-table position - ka), then own epsilon ones
  const int rank = (int)cluster_rank(), b = blockIdx.x / N, tid = threadIdx.x, nt = blockDim.x;
  const int n0 = sp.out[rank], n1 = sp.out[rank + 1]; // this CTA's nodes
  const int ka = __ldg(g.out_ptr + n0), kn = __ldg(g.out_ptr + n1) - ka; // their emitting out-arcs
  const int ea = __ldg(x.eps_out_ptr + n0), en = __ldg(x.eps_out_ptr + n1) - ea; // and epsilon out-arcs
  const Cluster team{cut, N, rank}; // the closure's
  const int groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
  const int Tb = lens[b];
  const double* of = offs + (long long)b * (T + 1);
  const double Z = of[0];
  if (Tb < 1 || !(fabs(Z) < (double)CUDART_INF_F)) return; // (the whole cluster: its ranks share b)
  const float* em = emis + (long long)b * stride;
  const float* al = alpha + (long long)b * (T + 1) * S;
  float* gr = grad + (long long)b * grad_stride;
  for (int v = tid; v < S; v += nt) rows[(Tb & 1) * S + v] = (__ldg(g.flags + v) & 2) ? 0.0f : neg_inf();
  for (int k = tid; k < kn + en; k += nt) acc[k] = 0.0f;
  for (int c = tid; c < 2 * C; c += nt) Eg[c] = 0.0f;
  for (int c = tid; c < C; c += nt) E[((Tb - 1) & 1) * C + c] = __ldg(em + (long long)(Tb - 1) * C + c);
  cluster_sync_all();
  eps_close_bwd(team, x, w, rows + (Tb & 1) * S, al + (long long)Tb * S, (float)(of[Tb] - Z), acc + kn, ea);
  row_max(team, rows + (Tb & 1) * S, S, 0, 0, nullptr, red + (Tb & 1) * kSparseWarps);
  __syncthreads();
  double d = 0.0; // d_{t+1}
  for (int t = Tb - 1; t >= 0; t--) {
    const float* Nx = rows + ((t + 1) & 1) * S;
    float* Cur = rows + (t & 1) * S;
    const float* Er = E + (t & 1) * C;
    float* Eg_t = Eg + (t & 1) * C;
    float* Eg_prev = Eg + ((t + 1) & 1) * C; // frame t + 1's, complete since the barrier
    for (int c = tid; c < C; c += nt) {
      if (t > 0) E[((t + 1) & 1) * C + c] = __ldg(em + (long long)(t - 1) * C + c);
      if (t + 1 < Tb) {
        const float v = Eg_prev[c];
        if (v != 0.0f) atomicAdd(gr + (long long)(t + 1) * C + c, v);
        Eg_prev[c] = 0.0f;
      }
    }
    const float Mb = cluster_row_offset(red + ((t + 1) & 1) * kSparseWarps, nt / 32);
    const double c_t = t > 0 ? of[t] : 0.0;
    const float fo = (float)(c_t + d - Z);
    for (int u0 = n0; u0 < n1; u0 += groups) {
      const int u = u0 + grp;
      float m = neg_inf(), s = 0.0f;
      if (u < n1) {
        const float au = al[(long long)t * S + u] + fo;
        const int k1 = __ldg(g.out_ptr + u + 1);
        for (int k = __ldg(g.out_ptr + u) + q; k < k1; k += lanes) {
          const int lab = __ldg(g.out_lab + k);
          const float xk = Nx[__ldg(g.out_dst + k)] + (__ldg(w + __ldg(g.out_arc + k)) + Er[lab]);
          lse_add(m, s, xk);
          const float p = exp_fast(au + xk);
          if (p != 0.0f) {
            acc[k - ka] += p;
            atomicAdd(Eg_t + lab, p);
          }
        }
      }
      lse_merge(m, s, lanes);
      if (u < n1 && q == 0) cluster_store(Cur + u, N, m == neg_inf() ? neg_inf() : (m + log_fast(s)) - Mb);
    }
    cluster_sync_all();
    eps_close_bwd(team, x, w, Cur, al + (long long)t * S, (float)(c_t + (d + (double)Mb) - Z), acc + kn, ea);
    row_max(team, Cur, S, 0, 0, nullptr, red + (t & 1) * kSparseWarps);
    d += (double)Mb;
    __syncthreads();
  }
  for (int c = tid; c < C; c += nt) { // frame 0's emission gradient
    const float v = Eg[c];
    if (v != 0.0f) atomicAdd(gr + c, v);
  }
  for (int k = tid; k < kn; k += nt)
    if (acc[k] != 0.0f) atomicAdd(wgrad + __ldg(g.out_arc + ka + k), acc[k]);
  for (int k = tid; k < en; k += nt)
    if (acc[kn + k] != 0.0f) atomicAdd(wgrad + __ldg(x.eps_out_arc + ea + k), acc[kn + k]);
}

/* sparse_eps_viterbi_kernel by a cluster: the same back-pointers ([B][T + 1][S]), head, score and status */
__global__ void __launch_bounds__(kSparseThreads, 2) sparse_cl_eps_viterbi_kernel(
    const SparseEpsDev* __restrict__ gs, SparseSplit sp, const int32_t* __restrict__ cut, int T, int C,
    const int32_t* __restrict__ lens, const float* __restrict__ emis, long long stride, const float* __restrict__ w,
    uint16_t* __restrict__ bp, int32_t* __restrict__ head, float* __restrict__ score, int32_t* __restrict__ status) {
  GTNB_DYNAMIC_SMEM(float, sm);
  const SparseEpsDev x = gs[0];
  const SparseDev& g = x.g;
  const int S = g.S, lanes = g.lanes, N = sp.N;
  float* rows = sm; // [2][S]
  float* E = sm + 2 * S; // [2][C]
  const int rank = (int)cluster_rank(), b = blockIdx.x / N, tid = threadIdx.x, nt = blockDim.x;
  const int n0 = sp.in[rank], n1 = sp.in[rank + 1]; // this CTA's nodes
  const Cluster team{cut, N, rank}; // the closure's
  const int groups = nt / lanes, grp = tid / lanes, q = tid % lanes;
  const int Tb = lens[b];
  const float* em = emis + (long long)b * stride;
  uint16_t* bpb = bp + (long long)b * (T + 1) * S;
  bool bad = false;
  for (int v = tid; v < S; v += nt) {
    const bool st = __ldg(g.flags + v) & 1;
    rows[v] = st ? 0.0f : neg_inf();
    if (v >= n0 && v < n1) bpb[v] = st ? (uint16_t)kBpStart : kBpNone;
  }
  if (Tb > 0)
    for (int c = tid; c < C; c += nt) E[C + c] = __ldg(em + c); // row 0 in E[1]: frame t reads E[t & 1]
  cluster_sync_all();
  eps_close_trop(team, x, w, rows, bpb, bad);
  for (int t = 1; t <= Tb; t++) {
    const float* P = rows + ((t - 1) & 1) * S;
    float* Q = rows + (t & 1) * S;
    const float* Er = E + (t & 1) * C;
    uint16_t* bpt = bpb + (long long)t * S;
    if (t < Tb)
      for (int c = tid; c < C; c += nt) E[((t + 1) & 1) * C + c] = __ldg(em + (long long)t * C + c);
    for (int v0 = n0; v0 < n1; v0 += groups) {
      const int v = v0 + grp;
      float m = neg_inf();
      int k = 0x7fffffff, tie = 0, k0 = 0;
      if (v < n1) {
        k0 = __ldg(g.in_ptr + v);
        const int k1 = __ldg(g.in_ptr + v + 1);
        for (int j = k0 + q; j < k1; j += lanes) {
          const float wk = __ldg(w + __ldg(g.in_arc + j));
          const float ek = Er[__ldg(g.in_lab + j)];
          bad |= !(wk < CUDART_INF_F && ek < CUDART_INF_F);
          argmax_add(m, k, tie, P[__ldg(g.in_src + j)] + (wk + ek), j);
        }
      }
      argmax_merge(m, k, tie, lanes);
      if (v < n1 && q == 0) {
        cluster_store(Q + v, N, m);
        bpt[v] = m == neg_inf() ? kBpNone : (uint16_t)((k - k0) | (tie ? kBpTie : 0));
      }
    }
    cluster_sync_all();
    eps_close_trop(team, x, w, Q, bpt, bad); // (its last barrier ends the frame)
  }
  bad = __syncthreads_or(bad);
  if (bad && tid == 0) atomicOr(&status[b], 1);
  if (rank == 0 && tid < 32) {
    const float* F = rows + (Tb & 1) * S;
    float m = neg_inf();
    int k = 0x7fffffff, tie = 0;
    if (Tb > 0)
      for (int v = tid; v < S; v += 32)
        if (__ldg(g.flags + v) & 2) argmax_add(m, k, tie, F[v], v);
    argmax_merge(m, k, tie, 32);
    if (tid == 0) {
      head[b] = m == neg_inf() ? -1 : k;
      score[b] = m;
      if (tie) atomicOr(&status[b], 2);
    }
  }
}

/* the numerators' weights, gathered: w[k] = fl(w_A[arc_of[k]] + W[tidx[k]]), W[tidx[k]] alone for an epsilon arc
 * (arc_of -1); w_A NULL: every A weight 0 */
__global__ void __launch_bounds__(256) sparse_eps_gather_kernel(long long n, const float* __restrict__ w_A,
                                                                const int32_t* __restrict__ arc_of,
                                                                const float* __restrict__ W,
                                                                const int32_t* __restrict__ tidx,
                                                                float* __restrict__ out) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int a = __ldg(arc_of + k);
  const float wg = __ldg(W + __ldg(tidx + k));
  out[k] = a < 0 ? wg : (w_A ? __ldg(w_A + a) : 0.0f) + wg;
}

/* the numerators' arc gradients (already signed) into the transition gradient (tidx) and, where an A arc is behind
 * the product arc, into the arc gradient (arc_of >= 0; nullable) */
__global__ void __launch_bounds__(256) sparse_eps_scatter_kernel(long long n, const float* __restrict__ pg,
                                                                 const int32_t* __restrict__ arc_of,
                                                                 const int32_t* __restrict__ tidx,
                                                                 float* __restrict__ tgrad, float* __restrict__ agrad) {
  const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (k >= n) return;
  const float v = pg[k];
  if (v == 0.0f) return;
  atomicAdd(tgrad + __ldg(tidx + k), v);
  const int a = __ldg(arc_of + k);
  if (agrad && a >= 0) atomicAdd(agrad + a, v);
}

} // namespace

#ifndef GTNB_HOST_EMU

bool sparse_den_supported(int S, int A, int C) {
  return S >= 1 && S <= kSparseMaxStates && A <= kSparseMaxArcs && C >= 1 && C <= kSparseMaxLabels;
}

namespace {

/* kernel on B CTAs of kSparseThreads threads with `floats` floats of dynamic shared memory */
template <class... P, class... A>
int launch_ctas(gtnb_ctx* ctx, const char* name, void (*kernel)(P...), int B, long long floats, A&&... args) {
  if (const int rc = ensure_max_smem(ctx, (const void*)kernel)) return rc;
  GTNB_LAUNCH(ctx, name,
              kernel<<<B, kSparseThreads, sizeof(float) * floats, ctx->stream>>>(std::forward<A>(args)...));
  return GTNB_OK;
}

/* kernel on B clusters of N such CTAs */
template <class... P, class... A>
int launch_clusters(gtnb_ctx* ctx, const char* name, void (*kernel)(P...), int B, int N, long long floats,
                    A&&... args) {
  if (const int rc = ensure_max_smem(ctx, (const void*)kernel)) return rc;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(B * N), 1, 1);
  cfg.blockDim = dim3(kSparseThreads, 1, 1);
  cfg.dynamicSmemBytes = sizeof(float) * floats;
  cfg.stream = ctx->stream;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = (unsigned)N;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  GTNB_LAUNCH(ctx, name, GTNB_CUDA(ctx, cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...)));
  return GTNB_OK;
}

/* one warp per utterance */
unsigned trace_blocks(int B) {
  return (unsigned)(((long long)B * 32 + 255) / 256);
}

} // namespace

int launch_sparse_den_forward(gtnb_ctx* ctx, const SparseDev& g, const SparseSplit& sp, int B, int T, int C,
                              const int32_t* lens, const float* emis, long long stride, const float* w, float* alpha,
                              double* offs, float* den, int32_t* status) {
  if (B == 0) return GTNB_OK;
  if (sp.N == 1)
    return launch_ctas(ctx, "sparse_den_forward", sparse_den_forward_kernel, B, sparse_fwd_smem_floats(g.S, C), g, T,
                       C, lens, emis, stride, w, alpha, offs, den, status);
  return launch_clusters(ctx, "sparse_cl_den_forward", sparse_cl_den_forward_kernel, B, sp.N,
                         sparse_cl_fwd_smem_floats(g.S, C, sp.N), g, sp, T, C, lens, emis, stride, w, alpha, offs,
                         den, status);
}

int launch_sparse_den_backward(gtnb_ctx* ctx, const SparseDev& g, const SparseSplit& sp, int B, int T, int C,
                               const int32_t* lens, const float* emis, long long stride, const float* w,
                               const float* alpha, const double* offs, float* grad, long long grad_stride,
                               float* wgrad) {
  if (B == 0) return GTNB_OK;
  if (sp.N == 1)
    return launch_ctas(ctx, "sparse_den_backward", sparse_den_backward_kernel, B,
                       sparse_bwd_smem_floats(g.S, g.A, C), g, T, C, lens, emis, stride, w, alpha, offs, grad,
                       grad_stride, wgrad);
  return launch_clusters(ctx, "sparse_cl_den_backward", sparse_cl_den_backward_kernel, B, sp.N,
                         sparse_cl_bwd_smem_floats(g.S, C, sp.N, sp.own_out), g, sp, T, C, lens, emis, stride, w,
                         alpha, offs, grad, grad_stride, wgrad);
}

int launch_sparse_sigma(gtnb_ctx* ctx, int K, const int32_t* grp_ptr, const int32_t* grp_arc, const float* w,
                        float* sigma) {
  if (K == 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "sparse_sigma", sparse_sigma_kernel<<<(unsigned)(((long long)K * 32 + 255) / 256), 256, 0,
                                                         ctx->stream>>>(K, grp_ptr, grp_arc, w, sigma));
  return GTNB_OK;
}

int launch_sparse_fold(gtnb_ctx* ctx, int K, const int32_t* grp_ptr, const int32_t* grp_arc, int nG, const float* w,
                       const float* sigma, float* wgrad) {
  if (K == 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "sparse_fold", sparse_fold_kernel<<<(unsigned)((K + 255) / 256), 256, 0, ctx->stream>>>(
      K, grp_ptr, grp_arc, nG, w, sigma, wgrad));
  return GTNB_OK;
}

int launch_sparse_viterbi(gtnb_ctx* ctx, const SparseDev& g, const SparseSplit& sp, int B, int T, int C,
                          const int32_t* lens, const float* emis, long long stride, const float* w, uint16_t* bp,
                          int32_t* head, float* score, int32_t* paths, int32_t* arcs, int32_t* status) {
  if (B == 0) return GTNB_OK;
  const long long floats = sparse_vit_smem_floats(g.S, C);
  if (const int rc = sp.N == 1 ? launch_ctas(ctx, "sparse_viterbi_forward", sparse_viterbi_forward_kernel, B, floats, g,
                                             T, C, lens, emis, stride, w, bp, head, score, status)
                               : launch_clusters(ctx, "sparse_cl_viterbi_forward", sparse_cl_viterbi_forward_kernel, B,
                                                 sp.N, floats, g, sp, T, C, lens, emis, stride, w, bp, head, score,
                                                 status))
    return rc;
  GTNB_LAUNCH(ctx, "sparse_viterbi_trace", sparse_viterbi_trace_kernel<<<trace_blocks(B), 256, 0, ctx->stream>>>(
      g, B, T, lens, bp, head, paths, arcs, status));
  return GTNB_OK;
}

int launch_sparse_tau(gtnb_ctx* ctx, int K, const int32_t* grp_ptr, const int32_t* grp_arc, const float* w,
                      float* tau) {
  if (K == 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "sparse_tau", sparse_tau_kernel<<<(unsigned)(((long long)K * 32 + 255) / 256), 256, 0,
                                                     ctx->stream>>>(K, grp_ptr, grp_arc, w, tau));
  return GTNB_OK;
}

int launch_sparse_eps_forward(gtnb_ctx* ctx, const SparseEpsDev* gs, const SparseSplit& sp, const int32_t* cut,
                              int per_cta, int max_S, int B, int T, int C, const int32_t* lens, const float* emis,
                              long long stride, const float* w, float* alpha, double* offs, float* den,
                              int32_t* status) {
  if (B == 0) return GTNB_OK;
  if (sp.N > 1 && per_cta)
    return fail(ctx, GTNB_ERR_LOGIC, "launch_sparse_eps_forward: a cluster sweeps the denominator alone (per_cta 0)");
  if (sp.N == 1)
    return launch_ctas(ctx, "sparse_eps_forward", sparse_eps_forward_kernel, B, sparse_fwd_smem_floats(max_S, C), gs,
                       per_cta, T, C, lens, emis, stride, w, alpha, offs, den, status);
  return launch_clusters(ctx, "sparse_cl_eps_forward", sparse_cl_eps_forward_kernel, B, sp.N,
                         sparse_cl_fwd_smem_floats(max_S, C, sp.N), gs, sp, cut, T, C, lens, emis, stride, w, alpha,
                         offs, den, status);
}

int launch_sparse_eps_backward(gtnb_ctx* ctx, const SparseEpsDev* gs, const SparseSplit& sp, const int32_t* cut,
                               int per_cta, int max_S, int max_AE, int B, int T, int C, const int32_t* lens,
                               const float* emis, long long stride, const float* w, const float* alpha,
                               const double* offs, float sgn, float* grad, long long grad_stride, float* wgrad) {
  if (B == 0) return GTNB_OK;
  if (sp.N > 1 && (per_cta || sgn != 1.0f))
    return fail(ctx, GTNB_ERR_LOGIC,
                "launch_sparse_eps_backward: a cluster sweeps the denominator alone (per_cta 0, sgn 1)");
  if (sp.N == 1)
    return launch_ctas(ctx, "sparse_eps_backward", sparse_eps_backward_kernel, B,
                       sparse_bwd_smem_floats(max_S, max_AE, C), gs, per_cta, T, C, lens, emis, stride, w, alpha,
                       offs, sgn, grad, grad_stride, wgrad);
  return launch_clusters(ctx, "sparse_cl_eps_backward", sparse_cl_eps_backward_kernel, B, sp.N,
                         sparse_cl_bwd_smem_floats(max_S, C, sp.N, sp.own_out), gs, sp, cut, T, C, lens, emis, stride,
                         w, alpha, offs, grad, grad_stride, wgrad);
}

int launch_sparse_eps_viterbi(gtnb_ctx* ctx, const SparseEpsDev* gs, const SparseSplit& sp, const int32_t* cut, int S,
                              int B, int T, int C, const int32_t* lens, const float* emis, long long stride,
                              const float* w, uint16_t* bp, int32_t* head, float* score, int32_t* paths, int32_t* arcs,
                              int32_t* status) {
  if (B == 0) return GTNB_OK;
  const long long floats = sparse_vit_smem_floats(S, C);
  if (const int rc = sp.N == 1 ? launch_ctas(ctx, "sparse_eps_viterbi", sparse_eps_viterbi_kernel, B, floats, gs, T, C,
                                             lens, emis, stride, w, bp, head, score, status)
                               : launch_clusters(ctx, "sparse_cl_eps_viterbi", sparse_cl_eps_viterbi_kernel, B, sp.N,
                                                 floats, gs, sp, cut, T, C, lens, emis, stride, w, bp, head, score,
                                                 status))
    return rc;
  GTNB_LAUNCH(ctx, "sparse_eps_trace", sparse_eps_trace_kernel<<<trace_blocks(B), 256, 0, ctx->stream>>>(
      gs, B, T, lens, bp, head, paths, arcs, status));
  return GTNB_OK;
}

int launch_sparse_eps_align(gtnb_ctx* ctx, const SparseEpsDev* gs, int max_S, int B, int T, int C,
                            const int32_t* lens, const float* emis, long long stride, const float* w, uint16_t* bp,
                            int32_t* head, float* score, const int32_t* arc_of, const int32_t* a_first,
                            int32_t* paths, int32_t* arcs, int32_t* status) {
  if (B == 0) return GTNB_OK;
  if (const int rc = launch_ctas(ctx, "sparse_eps_align", sparse_eps_align_kernel, B, sparse_vit_smem_floats(max_S, C),
                                 gs, C, lens, emis, stride, w, bp, head, score, status))
    return rc;
  GTNB_LAUNCH(ctx, "sparse_eps_align_trace", sparse_eps_align_trace_kernel<<<trace_blocks(B), 256, 0, ctx->stream>>>(
      gs, B, T, lens, bp, head, arc_of, a_first, paths, arcs, status));
  return GTNB_OK;
}

int launch_sparse_eps_gather(gtnb_ctx* ctx, long long n, const float* w_A, const int32_t* arc_of, const float* W,
                             const int32_t* tidx, float* out) {
  if (n == 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "sparse_eps_gather", sparse_eps_gather_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(
      n, w_A, arc_of, W, tidx, out));
  return GTNB_OK;
}

int launch_sparse_eps_scatter(gtnb_ctx* ctx, long long n, const float* pg, const int32_t* arc_of, const int32_t* tidx,
                              float* tgrad, float* agrad) {
  if (n == 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "sparse_eps_scatter", sparse_eps_scatter_kernel<<<(unsigned)((n + 255) / 256), 256, 0,
                                                                     ctx->stream>>>(n, pg, arc_of, tidx, tgrad, agrad));
  return GTNB_OK;
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
