/*
 * gtnb_ptx.h -- the device primitives of the kernel files: inline PTX, SFU math, shared-window loads and stores,
 * mbarrier / bulk-copy / barrier wrappers and full-warp reductions.  Every primitive whose PTX the host emulation
 * of tests/emu cannot run has its PTX body and its emulator body side by side here, under one
 * `#ifdef GTNB_HOST_EMU`: this header is the one place where the emulated build swaps code.
 *
 * It also does the include switch of the kernel files: under GTNB_HOST_EMU (g++, CPU test suite) the SIMT
 * emulator tests/emu/simt_emu.h and the plain-data headers, otherwise the CUDA runtime and gtnb_internal.h.
 */
#pragma once

#ifdef GTNB_HOST_EMU
#include "gtn_b200.h"
#include "gtnb_meta.h"
#include "simt_emu.h"
#else
#include <cuda_runtime.h>
#include <math_constants.h>

#include "gtnb_internal.h"
#endif

namespace gtnb {

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

__device__ __forceinline__ float neg_inf() {
  return -CUDART_INF_F;
}
__device__ __forceinline__ bool is_finite(float x) {
  return fabsf(x) < CUDART_INF_F;
}

/* the two floats of a 64-bit shared-memory load (the emulator has no CUDA vector types beyond int2 / float4) */
struct f32x2 {
  float x, y;
};

/* full-warp butterfly reductions: every lane gets the result */
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

#ifdef GTNB_HOST_EMU
/* ---- the emulator's restatement of the PTX below (tests/emu/simt_emu.h): shared-window addresses are offsets
 * into the CTA's emulated shared memory; mbarriers, bulk copies and barriers are emu:: objects ---- */

__device__ __forceinline__ float ex2(float x) {
  return exp2f(x);
}
__device__ __forceinline__ float lg2(float x) {
  return log2f(x);
}
__device__ __forceinline__ float rcp_approx(float x) {
  return 1.0f / x;
}
__device__ __forceinline__ float exp_fast(float x) {
  return expf(x);
}
__device__ __forceinline__ float log_fast(float x) {
  return logf(x);
}

__device__ __forceinline__ void ldg_if(bool p, float& dst, const float* src) {
  if (p) dst = *src;
}
__device__ __forceinline__ void ldg_keep(float& dst, const float* src) {
  dst = *src;
}
__device__ __forceinline__ void red_if(bool p, float* dst, float v) {
  if (p) atomicAdd(dst, v);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return emu::shared_window(p);
}
__device__ __forceinline__ float lds_f32(uint32_t addr) {
  return *emu::shared_ptr<float>(addr);
}
__device__ __forceinline__ void sts_f32(uint32_t addr, float v) {
  *emu::shared_ptr<float>(addr) = v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  return *emu::shared_ptr<uint32_t>(addr);
}
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
  *emu::shared_ptr<uint32_t>(addr) = v;
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t addr) {
  return *emu::shared_ptr<uint16_t>(addr);
}
__device__ __forceinline__ void sts_u16(uint32_t addr, uint32_t v) {
  *emu::shared_ptr<uint16_t>(addr) = (uint16_t)v;
}
__device__ __forceinline__ int lds_s8(uint32_t addr) {
  return *emu::shared_ptr<int8_t>(addr);
}
__device__ __forceinline__ void sts_s8(uint32_t addr, int v) {
  *emu::shared_ptr<int8_t>(addr) = (int8_t)v;
}
__device__ __forceinline__ int2 lds_v2_u32(uint32_t addr) {
  return *emu::shared_ptr<int2>(addr);
}
__device__ __forceinline__ f32x2 lds_v2_f32(uint32_t addr) {
  return *emu::shared_ptr<f32x2>(addr);
}
__device__ __forceinline__ void sts_v2_f32(uint32_t addr, float a, float b) {
  *emu::shared_ptr<f32x2>(addr) = f32x2{a, b};
}
__device__ __forceinline__ float4 lds_v4_f32(uint32_t addr) {
  return *emu::shared_ptr<float4>(addr);
}
__device__ __forceinline__ void red_shared_add(uint32_t addr, float v) {
  atomicAdd(emu::shared_ptr<float>(addr), v);
}
__device__ __forceinline__ void smem_max_s32(uint32_t addr, int v) {
  atomicMax(emu::shared_ptr<int32_t>(addr), v);
}
__device__ __forceinline__ void stg_f32(float* p, float v) {
  *p = v;
}
__device__ __forceinline__ void stg_v2_f32(float* p, float a, float b) {
  p[0] = a;
  p[1] = b;
}
__device__ __forceinline__ void stg_v4_f32(float* p, float4 v) {
  *reinterpret_cast<float4*>(p) = v;
}

__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
  emu::mbar_init(bar, count);
}
__device__ __forceinline__ void mbar_init_fence() {}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  emu::mbar_expect_tx(bar, bytes);
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  emu::mbar_arrive(bar);
}
__device__ __forceinline__ void mbar_arrive_n(uint32_t bar, int n) {
  emu::mbar_arrive_n(bar, n);
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  emu::mbar_wait(bar, parity);
}
__device__ __forceinline__ void mbar_wait_sleep(uint32_t bar, uint32_t parity) {
  emu::mbar_wait(bar, parity);
}
__device__ __forceinline__ void mbar_wait_suspend(uint32_t bar, uint32_t parity) {
  emu::mbar_wait(bar, parity);
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  emu::bulk_g2s(dst, src, bytes, bar);
}
__device__ __forceinline__ void fence_proxy_async() {}

__device__ __forceinline__ void bar_named(int id, int nthreads) {
  emu::named_barrier(id, nthreads);
}
template <int ID>
__device__ __forceinline__ void bar_named(int nthreads) {
  emu::named_barrier(ID, nthreads);
}
template <int ID, int N>
__device__ __forceinline__ void bar_named() {
  emu::named_barrier(ID, N);
}
__device__ __forceinline__ void cluster_sync_all() {
  emu::cluster_sync();
}
__device__ __forceinline__ void cluster_arrive_only() {
  emu::cluster_arrive();
}
__device__ __forceinline__ void cluster_wait_only() {
  emu::cluster_wait();
}
__device__ __forceinline__ unsigned cluster_rank() {
  return emu::cluster_ctarank();
}

__device__ __forceinline__ unsigned lanemask_lt() {
  return (1u << (threadIdx.x & 31)) - 1u;
}
__device__ __forceinline__ long long globaltimer() {
  return 0;
}

#else

/* ---- SFU ---- */

/* one MUFU each: 2^x and log2(x), flush-to-zero, relative error ~1e-6 */
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
/* CUDA's __expf / __logf: not ftz, so each is a range test and two scaling multiplies around the MUFU -- a
 * different function from ex2 / lg2 on denormals, kept apart so that their users compile as before */
__device__ __forceinline__ float exp_fast(float x) {
  return __expf(x);
}
__device__ __forceinline__ float log_fast(float x) {
  return __logf(x);
}

/* ---- global loads and stores ---- */

/* Predicated read-only load straight into its destination register.  With a plain
 * `if (p) x = __ldg(q)` in an unrolled frame loop ptxas gathers the prefetches of a block at its end,
 * into temporaries, and copies them to the loop-carried registers at the back edge -- a full-latency
 * stall every block. */
__device__ __forceinline__ void ldg_if(bool p, float& dst, const float* src) {
  asm volatile(
      "{\n"
      ".reg .pred q;\n"
      "setp.ne.s32 q, %2, 0;\n"
      "@q ld.global.nc.f32 %0, [%1];\n"
      "}\n"
      : "+f"(dst)
      : "l"(src), "r"((int)p));
}
/* Unpredicated variant for the steady part of a frame loop (address always valid): a strong
 * (relaxed, CTA scope) load, which ptxas must keep on its side of the bar.sync it was written
 * on, writing the loop-carried ring register directly. */
__device__ __forceinline__ void ldg_keep(float& dst, const float* src) {
  asm volatile("ld.relaxed.cta.global.f32 %0, [%1];" : "=f"(dst) : "l"(src) : "memory");
}
/* predicated red.global.add.f32 (no branch, no reconvergence point in the frame loop) */
__device__ __forceinline__ void red_if(bool p, float* dst, float v) {
  asm volatile(
      "{\n"
      ".reg .pred q;\n"
      "setp.ne.s32 q, %2, 0;\n"
      "@q red.global.add.f32 [%0], %1;\n"
      "}\n" ::"l"(dst),
      "f"(v), "r"((int)p)
      : "memory");
}
__device__ __forceinline__ void stg_f32(float* p, float v) {
  asm volatile("st.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ void stg_v2_f32(float* p, float a, float b) {
  asm volatile("st.global.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void stg_v4_f32(float* p, float4 v) {
  asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

/* ---- shared memory through 32-bit shared-window addresses: keeps per-level address arithmetic in 32-bit
 * integer ops instead of 64-bit generic pointers ---- */

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_f32(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_u16(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ int lds_s8(uint32_t addr) {
  int v;
  asm volatile("ld.shared.s8 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_s8(uint32_t addr, int v) {
  asm volatile("st.shared.u8 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ int2 lds_v2_u32(uint32_t addr) {
  int2 v;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
  return v;
}
__device__ __forceinline__ f32x2 lds_v2_f32(uint32_t addr) {
  f32x2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_v2_f32(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ float4 lds_v4_f32(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void red_shared_add(uint32_t addr, float v) {
  asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void smem_max_s32(uint32_t addr, int v) { // native ATOMS.MAX.S32
  asm volatile("red.shared.max.s32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

/* ---- mbarriers and TMA 1-D bulk copies ---- */

__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
/* makes the mbarrier.init of the elected thread visible to the async proxy */
__device__ __forceinline__ void mbar_init_fence() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
/* n arrivals at once (a warp arriving on behalf of warps that sit a phase out) */
__device__ __forceinline__ void mbar_arrive_n(uint32_t bar, int n) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(n) : "memory");
}
/* spin until the phase of parity `parity` has completed */
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
/* for a waiter that is a whole pipeline stage early: sleep between polls instead of burning the
 * issue slots the other warps need */
__device__ __forceinline__ void mbar_wait_sleep(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  for (;;) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    __nanosleep(64);
  }
}
/* the same, but the try_wait suspends the thread in hardware for up to the hinted time (ns) and wakes it
 * when the phase completes -- no issue slots spent polling */
__device__ __forceinline__ void mbar_wait_suspend(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(20000u)
        : "memory");
  } while (!done);
}
/* TMA 1-D bulk copy global -> shared, completion on an mbarrier */
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}
/* orders generic-proxy accesses (global stores of another CTA, this CTA's reads / writes of a
 * shared-memory stage) before the async-proxy copies issued next */
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async;" ::: "memory");
}

/* ---- barriers ---- */

/* bar.sync id, nthreads: the first `nthreads` threads of the CTA (a multiple of 32); __syncthreads() is
 * barrier 0.  The three forms emit the same barrier and differ only in which operands are immediates.  That
 * still changes ptxas's register allocation and scheduling around the barrier, so each kernel keeps the form
 * it was measured with. */
__device__ __forceinline__ void bar_named(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
/* the barrier id an immediate */
template <int ID>
__device__ __forceinline__ void bar_named(int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"n"(ID), "r"(nthreads) : "memory");
}
/* the barrier id and the thread count immediates */
template <int ID, int N>
__device__ __forceinline__ void bar_named() {
  asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(N) : "memory");
}
/* barrier.cluster: arrive has release, wait has acquire semantics at cluster scope */
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
/* the split form, for a warp that arrives early and waits later */
__device__ __forceinline__ void cluster_arrive_only() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_wait_only() {
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned cluster_rank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

/* ---- special registers ---- */

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}
__device__ __forceinline__ long long globaltimer() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

#endif // GTNB_HOST_EMU

/* natural-log exp / log1p on the SFU */
__device__ __forceinline__ float fexp(float x) {
  return ex2(x * kLog2e);
}
__device__ __forceinline__ float flog1p(float x) {
  // x = sum(exp(s - max)) - 1 >= 0; the series near 0 keeps the relative accuracy log1p is used for
  const float y = lg2(1.0f + x);
  return (x < 1e-3f) ? x * (1.0f - 0.5f * x) : y * kLn2;
}

/* logsumexp of three scores, natural log, branch-free: absent arcs carry -inf and add exp(-inf) = 0 in arc
 * order (shortest.cpp:102-114); an all--inf (or +inf) maximum is returned as is.  The sum is >= 1 (the maximum
 * contributes exp(0)), where lg2.approx has an absolute error <= 2^-22: far below one ulp of any score this
 * recursion produces after a few frames. */
__device__ __forceinline__ float lse3(float v0, float v1, float v2) {
  const float mx = fmaxf(fmaxf(v0, v1), v2);
  const float sum = (fexp(v0 - mx) + fexp(v1 - mx)) + fexp(v2 - mx);
  const float r = fmaf(lg2(sum), kLn2, mx);
  return (fabsf(mx) == CUDART_INF_F) ? mx : r;
}

} // namespace gtnb
