/*
 * k_linear.cu -- forwardScore / viterbiScore of the emissions chain itself,
 * i.e. detail::shortestDistance (shortest.cpp:86-188) on gtn::linearGraph(T, C)
 * (creations.cpp:20-33), and its gradient (shortest.cpp:33-82).
 *
 * On a chain the recursion factorises: score = sum_t lse_c e[t][c] (log) or
 * sum_t max_c e[t][c] (tropical), and d score / d e[t][c] = softmax_c / first-
 * argmax indicator.  Rows are independent, so this is one warp per frame row,
 * fully coalesced, followed by a fixed-order per-utterance reduction.
 */
#include <cstdint>

#include "gtnb_ptx.h"

namespace gtnb {

namespace {

constexpr int kRowWarps = 8;

template <bool TROPICAL>
__global__ void __launch_bounds__(32 * kRowWarps) linear_rows_kernel(
    const int32_t* __restrict__ T,
    int maxT,
    int C,
    const float* __restrict__ emis,
    long long stride,
    float* __restrict__ row_score, // [B][maxT]
    float* __restrict__ grad,
    long long grad_stride,
    const float* __restrict__ deltas,
    float delta_all,
    int overwrite) {
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * kRowWarps + warp;
  if (t >= T[b]) return;
  const float* e = emis + (long long)b * stride + (long long)t * C;
  float mx = -CUDART_INF_F;
  int arg = 0x7fffffff;
  for (int c = lane; c < C; c += 32) {
    const float v = e[c];
    if (v > mx) {
      mx = v;
      arg = c;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (om > mx || (om == mx && oa < arg)) { // first maximum wins (shortest.cpp:124)
      mx = om;
      arg = oa;
    }
  }
  float score = mx;
  float sum = 0.0f;
  const bool finite = (mx != CUDART_INF_F && mx != -CUDART_INF_F);
  if (!TROPICAL && finite) {
    for (int c = lane; c < C; c += 32) sum += expf(e[c] - mx);
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    score = mx + log1pf(sum - 1.0f);
  }
  if (lane == 0) row_score[(long long)b * maxT + t] = score;
  if (grad) {
    const float delta = deltas ? deltas[b] : delta_all;
    float* g = grad + (long long)b * grad_stride + (long long)t * C;
    if (TROPICAL) {
      for (int c = lane; c < C; c += 32) {
        const float v = (c == arg) ? delta : 0.0f;
        g[c] = overwrite ? v : g[c] + v;
      }
    } else {
      // g = exp(e - mx) / exp(lse - mx)   (shortest.cpp:71-72 on a chain)
      const float denom = expf(score - mx);
      for (int c = lane; c < C; c += 32) {
        const float v = expf(e[c] - mx) / denom * delta;
        g[c] = overwrite ? v : g[c] + v;
      }
    }
  }
}

/*
 * Vector variant for C = 4 * LPR with LPR a power of two <= 32 and 16-byte aligned rows: LPR
 * lanes read one row as float4 (32 / LPR rows per warp pass) and every warp runs kVecIter
 * passes with all of their loads issued up front -- the scalar kernel above keeps one 8-byte
 * load per thread in flight and stays far below the HBM rate this streaming pass
 * should run at (it shares the SMs with the latency-bound forward sweep of the lattice).
 * Same per-element formulas as the scalar kernel; only the association of the row sum differs.
 */
constexpr int kVecIter = 4;

template <bool TROPICAL, int LPR>
__global__ void __launch_bounds__(32 * kRowWarps) linear_rows_vec_kernel(
    const int32_t* __restrict__ T,
    int maxT,
    int C,
    const float* __restrict__ emis,
    long long stride,
    float* __restrict__ row_score,
    float* __restrict__ grad,
    long long grad_stride,
    const float* __restrict__ deltas,
    float delta_all,
    int overwrite) {
  constexpr int RPW = 32 / LPR;
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sub = lane % LPR, r = lane / LPR;
  const int Tb = T[b];
  const int t0 = (blockIdx.x * kRowWarps + warp) * (RPW * kVecIter) + r;
  if (t0 - r >= Tb) return; // warp-uniform
  const float* eb = emis + (long long)b * stride;
  const float ninf = -CUDART_INF_F;
  float4 v[kVecIter];
#pragma unroll
  for (int i = 0; i < kVecIter; i++) {
    const int t = t0 + i * RPW;
    v[i] = (t < Tb) ? __ldg(reinterpret_cast<const float4*>(eb + (long long)t * C) + sub)
                    : make_float4(ninf, ninf, ninf, ninf);
  }
  const float delta = grad ? (deltas ? deltas[b] : delta_all) : 0.0f;
#pragma unroll
  for (int i = 0; i < kVecIter; i++) {
    const int t = t0 + i * RPW;
    const bool ok = t < Tb;
    const float x[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
    float mx = x[0];
    int arg = 4 * sub;
#pragma unroll
    for (int k = 1; k < 4; k++)
      if (x[k] > mx) { // first maximum wins (shortest.cpp:124)
        mx = x[k];
        arg = 4 * sub + k;
      }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, mx, o);
      const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
      if (om > mx || (om == mx && oa < arg)) {
        mx = om;
        arg = oa;
      }
    }
    float score = mx;
    const bool finite = (mx != CUDART_INF_F && mx != -CUDART_INF_F);
    if (!TROPICAL) {
      float sum = 0.0f;
      if (finite) sum = (expf(x[0] - mx) + expf(x[1] - mx)) + (expf(x[2] - mx) + expf(x[3] - mx));
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      if (finite) score = mx + log1pf(sum - 1.0f);
    }
    if (ok && sub == 0) row_score[(long long)b * maxT + t] = score;
    if (grad && ok) {
      float4* g = reinterpret_cast<float4*>(grad + (long long)b * grad_stride + (long long)t * C) + sub;
      float4 out;
      if (TROPICAL) {
        out.x = (arg == 4 * sub + 0) ? delta : 0.0f;
        out.y = (arg == 4 * sub + 1) ? delta : 0.0f;
        out.z = (arg == 4 * sub + 2) ? delta : 0.0f;
        out.w = (arg == 4 * sub + 3) ? delta : 0.0f;
      } else {
        // g = exp(e - mx) / exp(lse - mx)   (shortest.cpp:71-72 on a chain)
        const float denom = expf(score - mx);
        out.x = expf(x[0] - mx) / denom * delta;
        out.y = expf(x[1] - mx) / denom * delta;
        out.z = expf(x[2] - mx) / denom * delta;
        out.w = expf(x[3] - mx) / denom * delta;
      }
      if (!overwrite) {
        const float4 old = *g;
        out.x += old.x;
        out.y += old.y;
        out.z += old.z;
        out.w += old.w;
      }
      *g = out;
    }
  }
}

#ifndef GTNB_HOST_EMU

template <bool TROPICAL, int LPR>
int launch_rows_vec(
    gtnb_ctx* ctx, int B, const int32_t* T_dev, int maxT, int C, const float* emis, long long stride,
    float* row_score, float* grad, long long grad_stride, const float* deltas, float delta_all,
    int overwrite) {
  const int rows_per_block = kRowWarps * (32 / LPR) * kVecIter;
  dim3 grid((maxT + rows_per_block - 1) / rows_per_block, B);
  GTNB_LAUNCH(ctx, "linear_rows", linear_rows_vec_kernel<TROPICAL, LPR><<<grid, 32 * kRowWarps, 0, ctx->stream>>>(
      T_dev, maxT, C, emis, stride, row_score, grad, grad_stride, deltas, delta_all, overwrite));
  return GTNB_OK;
}

constexpr int kNotVectorisable = -1;

/* launches the vector kernel when the shapes allow it; kNotVectorisable otherwise */
template <bool TROPICAL>
int try_rows_vec(
    gtnb_ctx* ctx, int B, const int32_t* T_dev, int maxT, int C, const float* emis, long long stride,
    float* row_score, float* grad, long long grad_stride, const float* deltas, float delta_all,
    int overwrite) {
  auto aligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if ((C & 3) || (stride & 3) || !aligned(emis)) return kNotVectorisable;
  if (grad && ((grad_stride & 3) || !aligned(grad))) return kNotVectorisable;
#define GTNB_ROWS_VEC(L)                                                                             \
  case 4 * L:                                                                                        \
    return launch_rows_vec<TROPICAL, L>(ctx, B, T_dev, maxT, C, emis, stride, row_score, grad,       \
                                        grad_stride, deltas, delta_all, overwrite);
  switch (C) {
    GTNB_ROWS_VEC(1)
    GTNB_ROWS_VEC(2)
    GTNB_ROWS_VEC(4)
    GTNB_ROWS_VEC(8)
    GTNB_ROWS_VEC(16)
    GTNB_ROWS_VEC(32)
    default:
      return kNotVectorisable;
  }
#undef GTNB_ROWS_VEC
}

#endif // GTNB_HOST_EMU

__global__ void __launch_bounds__(256) linear_reduce_kernel(
    const int32_t* __restrict__ T, int maxT, const float* __restrict__ row_score,
    float* __restrict__ scores) {
  GTNB_STATIC_SMEM(double, part, 256);
  const int b = blockIdx.x;
  const int Tb = T[b];
  double s = 0.0;
  for (int t = threadIdx.x; t < Tb; t += 256) s += (double)row_score[(long long)b * maxT + t];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) part[threadIdx.x] += part[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) scores[b] = (float)part[0];
}

} // namespace

#ifndef GTNB_HOST_EMU

int launch_linear_forward(
    gtnb_ctx* ctx, int B, const int32_t* T_dev, int maxT, int C, const float* emis, int64_t stride,
    int tropical, float* scores, float* grad, int64_t grad_stride, const float* deltas,
    float delta_all, int overwrite, float* scratch) {
  if (B == 0) return GTNB_OK;
  // per-frame logsumexp, B * maxT floats: the caller's scratch (no allocation on this stream) or ours
  float* row_score = scratch;
  if (!scratch) {
    int rc = dev_alloc(ctx, &row_score, (long long)B * std::max(maxT, 1));
    if (rc) return rc;
  }
  if (maxT > 0) {
    dim3 grid((maxT + kRowWarps - 1) / kRowWarps, B);
    const int vec = tropical ? try_rows_vec<true>(ctx, B, T_dev, maxT, C, emis, stride, row_score, grad,
                                                   grad_stride, deltas, delta_all, overwrite)
                              : try_rows_vec<false>(ctx, B, T_dev, maxT, C, emis, stride, row_score, grad,
                                                    grad_stride, deltas, delta_all, overwrite);
    if (vec != kNotVectorisable) {
      if (vec != GTNB_OK) return vec;
    } else if (tropical)
      GTNB_LAUNCH(ctx, "linear_rows", linear_rows_kernel<true><<<grid, 32 * kRowWarps, 0, ctx->stream>>>(
          T_dev, maxT, C, emis, stride, row_score, grad, grad_stride, deltas, delta_all, overwrite));
    else
      GTNB_LAUNCH(ctx, "linear_rows", linear_rows_kernel<false><<<grid, 32 * kRowWarps, 0, ctx->stream>>>(
          T_dev, maxT, C, emis, stride, row_score, grad, grad_stride, deltas, delta_all, overwrite));
  }
  GTNB_LAUNCH(ctx, "linear_reduce", linear_reduce_kernel<<<B, 256, 0, ctx->stream>>>(T_dev, maxT, row_score, scores));
  if (!scratch) dev_free(ctx, row_score);
  return GTNB_OK;
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
