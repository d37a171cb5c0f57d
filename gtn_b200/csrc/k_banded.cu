/*
 * k_banded.cu -- EXPERIMENTAL (gtnb_ctx_set_flag("banded", K); off by default; parity tested
 * against the oracle by tests/test_gpu_parity.py, no performance claim).
 *
 * The criterion sweeps of k_implicit.cu for graph operands whose in-arcs all come from the node
 * itself or one of its two predecessors in node order (u <- u, u-1, u-2): the CTC target graph
 * (benchmarks/ctc.cpp:40-58) and forced-alignment graphs.  k_implicit.cu is bound by its
 * per-frame dependence chain: three LDS, one CTA-wide barrier and the skew of seven warps every
 * frame (barrier and short-scoreboard waits lead its stall samples).  With one-sided dependencies a warp can advance K frames on its own if it carries 2K
 * halo lanes on the side the dependencies come from:
 *
 *   forward  lane l of warp q holds node q*(32-2K) + l - 2K.  Neighbour scores are warp shuffles
 *            (shfl.up 1, 2).  The 2K low lanes recompute the previous warp's last nodes; they go
 *            stale two lanes per frame, so after K frames exactly the halo is stale.  Then the
 *            own lanes publish their scores to a shared-memory row, ONE barrier, the halo lanes
 *            re-read.  Every own lane stores its score to HBM each frame, as k_implicit.cu does
 *            ([T+1][pitch] rows: the two forward kernels and the two backward kernels are
 *            interchangeable).
 *   backward lane l of warp q holds node q*(30-2K) + l - 2: lanes 0, 1 only supply saved scores to
 *            lanes 2, 3 (the arc factors need S_{t-1}[u-1], S_{t-1}[u-2]); the 2K high lanes are
 *            the halo of the node-gradient recursion, whose dependencies come from u+1, u+2
 *            (shfl.down 1, 2 of the arc gradients).  Emission gradients leave from own lanes only.
 *
 * The lane arithmetic (who holds which node, which lanes are valid after j frames, what is
 * published and re-read) is pinned by the lane-exact numpy model scripts/banded_model.py.
 * Same arithmetic per node as k_implicit.cu's fast path (lse3 on the SFU, arc factors
 * exp(S_{t-1}[src] + fl(w + e) - S_t[u])), arcs taken in offset order 0, 1, 2.
 * Not applicable (status bit 2 -> the caller repeats the call through the other kernels): an
 * in-arc from outside the band, two in-arcs from the same source, in-degree > 3.
 */
#include <algorithm>

#include "gtnb_ptx.h"

namespace gtnb {

namespace {

constexpr int kBandPf = 8; // frames per register prefetch block (see k_implicit.cu)
constexpr int kBandMaxThreads = 512; // 16 warps: leaves 128 registers per thread

/* CTA-wide max / sum for any number of warps <= 32; `red` holds 32 floats */
__device__ __forceinline__ float b_block_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); w++) r = fmaxf(r, red[w]);
  return r;
}
__device__ __forceinline__ float b_block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); w++) r += red[w];
  return r;
}

/* the node's in-arcs in band form: w[d] = weight of the arc (n - d) -> n, -inf when absent */
struct BandNode {
  float w0, w1, w2;
  int label;
  bool has; // has in-arcs
  unsigned char flags; // bit 0 start, bit 1 accept
};

__device__ __forceinline__ BandNode load_band_node(
    const GraphMeta& m, bool ok, int n, const uint8_t* __restrict__ sg_flags,
    const int32_t* __restrict__ sg_in_ptr, const int32_t* __restrict__ sg_in_src,
    const int32_t* __restrict__ sg_in_label, const float* __restrict__ sg_in_w, bool& bad,
    bool& unsupported) {
  BandNode b;
  b.w0 = b.w1 = b.w2 = neg_inf();
  b.label = 0;
  b.has = false;
  b.flags = 0;
  if (!ok) return b;
  const int32_t* ip = sg_in_ptr + m.sg_node_base;
  const int e0 = ip[n], e1 = ip[n + 1];
  b.flags = sg_flags[m.sg_node_base + n];
  b.has = e1 > e0;
  if (b.has) b.label = sg_in_label[m.sg_arc_base + e0];
  unsigned seen = 0;
  for (int a = e0; a < e1; a++) {
    const int d = n - sg_in_src[m.sg_arc_base + a];
    const float w = sg_in_w[m.sg_arc_base + a];
    bad |= !is_finite(w);
    if (d < 0 || d > 2 || ((seen >> d) & 1u)) {
      unsupported = true;
      continue;
    }
    seen |= 1u << d;
    if (d == 0) b.w0 = w;
    if (d == 1) b.w1 = w;
    if (d == 2) b.w2 = w;
  }
  return b;
}

/* ------------------------------------------------------------------ */
/* forward                                                             */
/* ------------------------------------------------------------------ */

template <int K>
__global__ void __launch_bounds__(kBandMaxThreads, 1) banded_forward_kernel(
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
    int row_pitch) {
  static_assert(kBandPf % K == 0, "a prefetch block is a whole number of barrier intervals");
  constexpr int H = 2 * K, OWN = 32 - H;
  GTNB_DYNAMIC_SMEM(float, b_smem);
  float* row0 = b_smem; // exchange rows: scores of all nodes at a block boundary
  float* row1 = b_smem + row_pitch;
  float* red = b_smem + 2 * row_pitch;
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N1 = m.sg_N, T = m.T;
  const int pitch = (N1 + 3) & ~3;
  const int n = warp * OWN + lane - H;
  const bool ok = n >= 0 && n < N1;
  const bool own = ok && lane >= H;
  bool bad = false, unsupported = false;
  const BandNode bn = load_band_node(m, ok, n, sg_flags, sg_in_ptr, sg_in_src, sg_in_label, sg_in_w, bad,
                                     unsupported);
  const float w0 = bn.w0, w1 = bn.w1, w2 = bn.w2;
  const bool has = bn.has;
  float* sc = scores + m.node_base;
  const float* eml = emissions + m.emis_off + bn.label;

  // frame 0: start nodes carry the implicit 0 (shortest.cpp:129-135)
  float s = (ok && (bn.flags & 1)) ? 0.0f : neg_inf();
  if (own) {
    sc[n] = s;
    row0[n] = s;
  }
  const float* fin = row0; // the row that holds the latest published frame
  __syncthreads();

  float pf[kBandPf], nx[kBandPf];
#pragma unroll
  for (int j = 0; j < kBandPf; j++) pf[j] = (has && j < T) ? __ldg(eml + (long long)j * C) : 0.0f;
#pragma unroll
  for (int j = 0; j < kBandPf; j++)
    nx[j] = (has && kBandPf + j < T) ? __ldg(eml + (long long)(kBandPf + j) * C) : 0.0f;
  const float* epf = eml + (long long)(2 * kBandPf) * C;
  float* grow = sc + pitch + (ok ? n : 0); // this node's score in frame f + 1
  float chk = 0.0f;
  int f0 = 0;

#define GTNB_BAND_FWD_FRAME(idx)                                                      \
  {                                                                                   \
    const float e = has ? pf[idx] : 0.0f;                                             \
    const float s1 = __shfl_up_sync(0xffffffffu, s, 1);                               \
    const float s2 = __shfl_up_sync(0xffffffffu, s, 2);                               \
    s = lse3(s + (w0 + e), s1 + (w1 + e), s2 + (w2 + e));                           \
    chk = fmaf(e, 0.0f, chk);                                                         \
    if (own) *grow = s;                                                               \
    grow += pitch;                                                                    \
  }
#define GTNB_BAND_FWD_REFILL(GUARDED)                                                 \
  {                                                                                   \
    _Pragma("unroll") for (int j = 0; j < kBandPf; j++) pf[j] = nx[j];                \
    _Pragma("unroll") for (int j = 0; j < kBandPf; j++) {                             \
      if (GUARDED)                                                                    \
        ldg_if(has && f0 + 2 * kBandPf + j < T, nx[j], epf + (long long)j * C);     \
      else                                                                            \
        ldg_keep(nx[j], epf + (long long)j * C);                                    \
    }                                                                                 \
    epf += (long long)kBandPf * C;                                                    \
  }
  // main part: whole prefetch blocks, kBandPf / K barrier intervals each
  float* rd = row0;
  float* wr = row1;
  for (; f0 + 3 * kBandPf <= T; f0 += kBandPf) {
#pragma unroll
    for (int kb = 0; kb < kBandPf / K; kb++) {
      if (lane < H) s = ok ? rd[n] : neg_inf(); // the halo re-reads the neighbour warp's nodes
#pragma unroll
      for (int j = 0; j < K; j++) GTNB_BAND_FWD_FRAME(kb * K + j)
      if (own) wr[n] = s;
      __syncthreads();
      fin = wr;
      float* t = rd;
      rd = wr;
      wr = t;
    }
    GTNB_BAND_FWD_REFILL(false)
  }
  for (; f0 < T; f0 += kBandPf) {
#pragma unroll
    for (int kb = 0; kb < kBandPf / K; kb++) {
      if (f0 + kb * K >= T) break; // uniform over the CTA
      if (lane < H) s = ok ? rd[n] : neg_inf();
#pragma unroll
      for (int j = 0; j < K; j++) {
        if (f0 + kb * K + j < T) GTNB_BAND_FWD_FRAME(kb * K + j)
      }
      if (own) wr[n] = s;
      __syncthreads();
      fin = wr;
      float* t = rd;
      rd = wr;
      wr = t;
    }
    GTNB_BAND_FWD_REFILL(true)
  }
#undef GTNB_BAND_FWD_REFILL
#undef GTNB_BAND_FWD_FRAME
  bad |= !(chk == 0.0f);

  // accept nodes of the last frame (shortest.cpp:147-159); every node is owned by one lane
  const bool acc = own && (bn.flags & 2);
  const float sT = acc ? fin[n] : neg_inf();
  const float mx = b_block_max(sT, red);
  float out = mx;
  if (mx != CUDART_INF_F && mx != -CUDART_INF_F) {
    const float sum = b_block_sum(acc ? expf(sT - mx) : 0.0f, red);
    out = mx + log1pf(sum - 1.0f);
  }
  if (tid == 0) out_scores[blockIdx.x] = out;
  if (bad) atomicOr(&status[blockIdx.x], 1);
  if (unsupported) atomicOr(&status[blockIdx.x], 2);
}

/* ------------------------------------------------------------------ */
/* backward                                                            */
/* ------------------------------------------------------------------ */

template <int K>
__global__ void __launch_bounds__(kBandMaxThreads, 1) banded_backward_kernel(
    const GraphMeta* __restrict__ meta,
    const uint8_t* __restrict__ sg_flags,
    const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ sg_in_src,
    const int32_t* __restrict__ sg_in_label,
    const float* __restrict__ sg_in_w,
    const float* __restrict__ emissions,
    const float* __restrict__ scores,
    const float* __restrict__ out_scores,
    const float* __restrict__ deltas,
    float* __restrict__ grad_emis,
    long long grad_stride,
    int C,
    int row_pitch) {
  static_assert(kBandPf % K == 0, "a prefetch block is a whole number of barrier intervals");
  constexpr int H = 2 * K, OWN = 30 - H;
  GTNB_DYNAMIC_SMEM(float, b_smem);
  float* row0 = b_smem; // exchange rows: node gradients at a block boundary
  float* row1 = b_smem + row_pitch;
  float* red = b_smem + 2 * row_pitch;
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N1 = m.sg_N, T = m.T;
  const int pitch = (N1 + 3) & ~3;
  const int n = warp * OWN + lane - 2;
  const bool ok = n >= 0 && n < N1;
  const bool own = ok && lane >= 2 && lane < 32 - H;
  bool bad = false, unsupported = false; // already reported by the forward sweep
  const BandNode bn = load_band_node(m, ok, n, sg_flags, sg_in_ptr, sg_in_src, sg_in_label, sg_in_w, bad,
                                     unsupported);
  const float w0 = bn.w0, w1 = bn.w1, w2 = bn.w2;
  const bool has = bn.has;

  const float out = out_scores[blockIdx.x];
  if (!is_finite(out) || T < 1) return; // no accepting path: no gradient (uniform over the CTA)
  const float delta = deltas ? deltas[blockIdx.x] : 1.0f;
  const float* scu = scores + m.node_base + (ok ? n : 0);
  const float* eml = emissions + m.emis_off + bn.label;
  float* gl = grad_emis + (long long)blockIdx.x * grad_stride + (long long)(T - 1) * C + bn.label;

  // seeds: nodeGrad[accept] = exp(score - maxA) / exp(out - maxA) (shortest.cpp:49-60)
  float s_t = ok ? __ldg(scu + (long long)T * pitch) : neg_inf(); // S_T[n]
  const bool acc = ok && (bn.flags & 2);
  const float mxa = b_block_max((own && acc) ? s_t : neg_inf(), red);
  const float denom = expf(out - mxa);
  float G = acc ? expf(s_t - mxa) / denom : 0.0f; // every lane seeds its own node, halo included

  // level t = T - i needs S_{t-1}[n] and e[t-1][label]: frame T - 1 - i
  float ps[kBandPf], pe[kBandPf], nxs[kBandPf], nxe[kBandPf];
#pragma unroll
  for (int j = 0; j < kBandPf; j++) {
    const int f = T - 1 - j;
    nxs[j] = (ok && f >= 0) ? __ldg(scu + (long long)f * pitch) : neg_inf();
    nxe[j] = (has && f >= 0) ? __ldg(eml + (long long)f * C) : 0.0f;
  }
  const float* spf = scu + (long long)(T - 1 - kBandPf) * pitch; // only dereferenced while >= row 0
  const float* epf = eml + (long long)(T - 1 - kBandPf) * C;
  int i0 = 0;

#define GTNB_BAND_BWD_LEVEL(idx)                                                      \
  {                                                                                   \
    const float s_p = ps[idx]; /* S_{t-1}[n] */                                       \
    const float e = has ? pe[idx] : 0.0f; /* e[t-1][label] */                         \
    const float sp1 = __shfl_up_sync(0xffffffffu, s_p, 1);                            \
    const float sp2 = __shfl_up_sync(0xffffffffu, s_p, 2);                            \
    /* a node that does not exist (score -inf) gets exp(-inf) = 0 on all its arcs */  \
    const float se = (s_t == -CUDART_INF_F) ? CUDART_INF_F : s_t;                     \
    const float c0 = G * fexp(s_p + (w0 + e) - se);                                 \
    const float c1 = G * fexp(sp1 + (w1 + e) - se);                                 \
    const float c2 = G * fexp(sp2 + (w2 + e) - se);                                 \
    const float acc_e = (c0 + c1) + c2;                                               \
    G = (c0 + __shfl_down_sync(0xffffffffu, c1, 1)) + __shfl_down_sync(0xffffffffu, c2, 2); \
    red_if(own && acc_e != 0.0f, gl, acc_e * delta);                                \
    gl -= C;                                                                          \
    s_t = s_p;                                                                        \
  }
#define GTNB_BAND_BWD_REFILL(GUARDED)                                                 \
  {                                                                                   \
    _Pragma("unroll") for (int j = 0; j < kBandPf; j++) {                             \
      ps[j] = nxs[j];                                                                 \
      pe[j] = nxe[j];                                                                 \
    }                                                                                 \
    _Pragma("unroll") for (int j = 0; j < kBandPf; j++) {                             \
      if (GUARDED) {                                                                  \
        const bool inb = T - 1 - (i0 + kBandPf + j) >= 0;                             \
        ldg_if(ok && inb, nxs[j], spf - (long long)j * pitch);                      \
        ldg_if(has && inb, nxe[j], epf - (long long)j * C);                         \
      } else {                                                                        \
        ldg_keep(nxs[j], spf - (long long)j * pitch);                               \
        ldg_keep(nxe[j], epf - (long long)j * C);                                   \
      }                                                                               \
    }                                                                                 \
    spf -= (long long)kBandPf * pitch;                                                \
    epf -= (long long)kBandPf * C;                                                    \
  }
  float* wr = row0;
  float* nw = row1;
  // main part: the refill of the block after this one reads frames down to T-1-(i0+2*kBandPf-1)
  for (; i0 + 2 * kBandPf <= T; i0 += kBandPf) {
    GTNB_BAND_BWD_REFILL(false)
#pragma unroll
    for (int kb = 0; kb < kBandPf / K; kb++) {
#pragma unroll
      for (int j = 0; j < K; j++) GTNB_BAND_BWD_LEVEL(kb * K + j)
      if (own) wr[n] = G;
      __syncthreads();
      if (lane >= 32 - H) G = ok ? wr[n] : 0.0f; // the halo re-reads the next warp's nodes
      float* t = wr;
      wr = nw;
      nw = t;
    }
  }
  for (; i0 < T; i0 += kBandPf) {
    GTNB_BAND_BWD_REFILL(true)
#pragma unroll
    for (int kb = 0; kb < kBandPf / K; kb++) {
      if (i0 + kb * K >= T) break; // uniform over the CTA
#pragma unroll
      for (int j = 0; j < K; j++) {
        if (i0 + kb * K + j < T) GTNB_BAND_BWD_LEVEL(kb * K + j)
      }
      if (own) wr[n] = G;
      __syncthreads();
      if (lane >= 32 - H) G = ok ? wr[n] : 0.0f;
      float* t = wr;
      wr = nw;
      nw = t;
    }
  }
#undef GTNB_BAND_BWD_REFILL
#undef GTNB_BAND_BWD_LEVEL
}

} // namespace

#ifndef GTNB_HOST_EMU

namespace {
/* frames per barrier: the value of gtnb_ctx_set_flag("banded", K), K in {1, 2, 4, 8} (else 4) */
int band_k(const gtnb_ctx* ctx) {
  const int k = ctx->use_banded;
  return (k == 1 || k == 2 || k == 4 || k == 8) ? k : 4;
}
} // namespace

/* true when the banded sweeps can take this batch (checked on the host: sizes; the band shape
 * itself is checked by the forward kernel, status bit 2) */
bool banded_supported(const gtnb_ctx* ctx, const gtnb_lattice* lat) {
  if (!lat->composed || lat->max_in_deg > 3) return false;
  const int own_b = 30 - 2 * band_k(ctx); // the backward sweep has fewer own lanes per warp
  const int warps = (lat->max_lvl_nodes + own_b - 1) / own_b;
  return warps >= 1 && 32 * warps <= kBandMaxThreads;
}

int launch_banded_forward(gtnb_ctx* ctx, gtnb_lattice* lat, int32_t* status_dev, int b0, int nb) {
  if (nb < 0) nb = lat->B - b0;
  if (nb <= 0) return GTNB_OK;
  const int K = band_k(ctx);
  const int own = 32 - 2 * K;
  const int warps = std::max(1, (lat->max_lvl_nodes + own - 1) / own);
  const int row_pitch = (warps * own + 3) & ~3;
  const size_t smem = sizeof(float) * (2 * (size_t)row_pitch + 32);
#define GTNB_BAND_FWD(KK)                                                                              \
  GTNB_LAUNCH(ctx, "banded_forward",                                                                   \
              banded_forward_kernel<KK><<<nb, 32 * warps, smem, ctx->stream>>>(                        \
                  lat->meta + b0, lat->sg_flags, lat->sg_in_ptr, lat->sg_in_src, lat->sg_in_label,     \
                  lat->sg_in_w, lat->emissions, lat->scores, lat->out_scores + b0, status_dev + b0,    \
                  lat->C, row_pitch))
  switch (K) {
    case 1: GTNB_BAND_FWD(1); break;
    case 2: GTNB_BAND_FWD(2); break;
    case 8: GTNB_BAND_FWD(8); break;
    default: GTNB_BAND_FWD(4); break;
  }
#undef GTNB_BAND_FWD
  return GTNB_OK;
}

int launch_banded_backward(
    gtnb_ctx* ctx, gtnb_lattice* lat, const float* deltas_dev, float* grad_emis, int64_t grad_stride, int b0,
    int nb) {
  if (nb < 0) nb = lat->B - b0;
  if (nb <= 0) return GTNB_OK;
  const int K = band_k(ctx);
  const int own = 30 - 2 * K;
  const int warps = std::max(1, (lat->max_lvl_nodes + own - 1) / own);
  const int row_pitch = (warps * own + 3) & ~3;
  const size_t smem = sizeof(float) * (2 * (size_t)row_pitch + 32);
#define GTNB_BAND_BWD(KK)                                                                              \
  GTNB_LAUNCH(ctx, "banded_backward",                                                                  \
              banded_backward_kernel<KK><<<nb, 32 * warps, smem, ctx->stream>>>(                       \
                  lat->meta + b0, lat->sg_flags, lat->sg_in_ptr, lat->sg_in_src, lat->sg_in_label,     \
                  lat->sg_in_w, lat->emissions, lat->scores, lat->out_scores + b0,                     \
                  deltas_dev ? deltas_dev + b0 : nullptr, grad_emis + (long long)b0 * grad_stride,     \
                  (long long)grad_stride, lat->C, row_pitch))
  switch (K) {
    case 1: GTNB_BAND_BWD(1); break;
    case 2: GTNB_BAND_BWD(2); break;
    case 8: GTNB_BAND_BWD(8); break;
    default: GTNB_BAND_BWD(4); break;
  }
#undef GTNB_BAND_BWD
  return GTNB_OK;
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
