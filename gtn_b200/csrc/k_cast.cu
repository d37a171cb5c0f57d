/*
 * k_cast.cu -- elementwise conversions between 16-bit storage (bfloat16, IEEE half) and float32 for the routes of
 * gtnb_ctc_loss_ex that read float32: widen the emissions once into scratch, round the float32 gradient into the
 * caller's buffer.  Widening is exact; narrowing rounds to nearest, ties to even (cvt.rn), as torch's .to() does.
 */
#include <algorithm>

#include "gtnb_ptx.h"

namespace gtnb {

namespace {

constexpr int kCastThreads = 256;

template <class E>
__global__ void __launch_bounds__(kCastThreads) widen_kernel(const E* __restrict__ src, float* __restrict__ dst,
                                                             long long n) {
  for (long long i = (long long)blockIdx.x * kCastThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kCastThreads)
    dst[i] = ldg_elem(src + i);
}

template <class E>
__global__ void __launch_bounds__(kCastThreads) narrow_kernel(const float* __restrict__ src, E* __restrict__ dst,
                                                              long long n) {
  for (long long i = (long long)blockIdx.x * kCastThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kCastThreads)
    stg_elem(dst + i, src[i]);
}

int cast_grid(gtnb_ctx* ctx, long long n) {
  return (int)std::min<long long>((n + kCastThreads - 1) / kCastThreads, 16ll * ctx->sm_count);
}

} // namespace

int launch_widen(gtnb_ctx* ctx, const void* src, int dtype, float* dst, long long n) {
  if (n <= 0) return GTNB_OK;
  const int grid = cast_grid(ctx, n);
  if (dtype == GTNB_BF16)
    GTNB_LAUNCH(ctx, "widen", (widen_kernel<bf16_t><<<grid, kCastThreads, 0, ctx->stream>>>(
                                  static_cast<const bf16_t*>(src), dst, n)));
  else if (dtype == GTNB_F16)
    GTNB_LAUNCH(ctx, "widen", (widen_kernel<f16_t><<<grid, kCastThreads, 0, ctx->stream>>>(
                                  static_cast<const f16_t*>(src), dst, n)));
  else
    return fail(ctx, GTNB_ERR_LOGIC, "launch_widen: not a 16-bit type");
  return GTNB_OK;
}

int launch_narrow(gtnb_ctx* ctx, const float* src, void* dst, int dtype, long long n) {
  if (n <= 0) return GTNB_OK;
  const int grid = cast_grid(ctx, n);
  if (dtype == GTNB_BF16)
    GTNB_LAUNCH(ctx, "narrow", (narrow_kernel<bf16_t><<<grid, kCastThreads, 0, ctx->stream>>>(
                                   src, static_cast<bf16_t*>(dst), n)));
  else if (dtype == GTNB_F16)
    GTNB_LAUNCH(ctx, "narrow", (narrow_kernel<f16_t><<<grid, kCastThreads, 0, ctx->stream>>>(
                                   src, static_cast<f16_t*>(dst), n)));
  else
    return fail(ctx, GTNB_ERR_LOGIC, "launch_narrow: not a 16-bit type");
  return GTNB_OK;
}

} // namespace gtnb
