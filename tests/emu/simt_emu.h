/*
 * tests/emu/simt_emu.h -- TEST INFRASTRUCTURE: a minimal SIMT emulator, so that the source of a CUDA
 * kernel (not a restatement of it) can be compiled with g++ and run on the CPU in the `-m "not gpu"`
 * suite.  One std::thread per CUDA thread, one CTA at a time; __syncthreads() is a std::barrier over
 * the CTA, warp shuffles exchange through a per-warp slot array between two phases of a per-warp
 * barrier.  It checks index arithmetic, barrier placement (a misplaced barrier deadlocks or trips the
 * result), shuffle semantics and tails; it does not model the memory system or timing.
 *
 * A kernel file opts in by including gtn_b200/csrc/gtnb_ptx.h, which holds the emulated form of every
 * inline-PTX helper next to its PTX, and by `#ifndef GTNB_HOST_EMU` around its launchers.
 */
#pragma once

#include <array>
#include <atomic>
#include <barrier>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <system_error>
#include <thread>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
#define __launch_bounds__(...)
#define __align__(x) alignas(x)
#define CUDART_INF_F (__builtin_inff())
#define CUDART_NAN_F (__builtin_nanf(""))

namespace emu {

struct Dim3 {
  unsigned x = 1, y = 1, z = 1;
};

struct Cta {
  Cta(unsigned nthreads, size_t smem_bytes)
      : bar(nthreads), smem(smem_bytes + 256), slots((nthreads + 31) / 32) {
    for (unsigned w = 0; w < (nthreads + 31) / 32; w++) {
      const unsigned lanes = std::min(32u, nthreads - 32 * w);
      warp_bar.emplace_back(new std::barrier<>(lanes));
    }
  }
  float* dynamic_smem() {
    auto p = reinterpret_cast<uintptr_t>(smem.data());
    return reinterpret_cast<float*>((p + 127) & ~uintptr_t(127));
  }
  std::barrier<>& named(int id, int nthreads) {
    std::lock_guard<std::mutex> l(named_lock);
    auto& b = named_bars[id];
    if (!b) b.reset(new std::barrier<>(nthreads));
    return *b;
  }
  std::barrier<> bar;
  std::vector<std::unique_ptr<std::barrier<>>> warp_bar;
  std::vector<unsigned char> smem;
  std::vector<std::array<uint32_t, 32>> slots;
  void* static_smem(int key, size_t bytes) {
    std::lock_guard<std::mutex> l(named_lock);
    auto& v = statics[key];
    if (v.empty()) v.assign(bytes + 16, 0);
    return v.data();
  }
  std::map<int, std::vector<unsigned char>> statics; // static __shared__ arrays, by source line
  /* mbarrier objects by shared-window address: arrival count per phase, pending arrivals, outstanding
   * transaction bytes, phase parity (mbarrier.init / arrive / arrive.expect_tx / complete_tx /
   * try_wait.parity) */
  struct MBar {
    int count = 0, pending = 0, phase = 0;
    long long tx = 0;
  };
  std::mutex mbar_lock;
  std::map<uint32_t, MBar> mbars;
  std::mutex named_lock;
  std::map<int, std::unique_ptr<std::barrier<>>> named_bars; // bar.sync id, n (n fixed per id)
  std::atomic<int> vote{0};
};

inline thread_local Cta* g_cta = nullptr;

/* a thread-block cluster: its CTAs run concurrently and share one barrier (barrier.cluster) */
struct Cluster {
  explicit Cluster(unsigned nthreads) : bar(nthreads) {}
  std::barrier<> bar;
};
inline thread_local Cluster* g_cluster = nullptr;
inline thread_local unsigned g_cluster_rank = 0;

} // namespace emu

inline thread_local emu::Dim3 threadIdx, blockIdx, blockDim, gridDim;

namespace emu {

/* set when the host refused to create the threads of a CTA: the drivers return kEmuNoThreads and the
 * tests skip instead of failing (a sandbox with a low thread limit must not turn the suite red) */
inline std::atomic<bool> g_launch_failed{false};
constexpr int kEmuNoThreads = 77;

/* run `body()` once per thread of a grid x block launch, CTAs one after the other */
template <class F>
void launch(unsigned grid, unsigned block, size_t smem_bytes, F&& body) {
  for (unsigned b = 0; b < grid && !g_launch_failed.load(); b++) {
    Cta cta(block, smem_bytes);
    std::vector<std::thread> threads;
    threads.reserve(block);
    // the threads park on `go` until all of them exist: if the host refuses one, none runs the body
    std::atomic<int> go{0}; // 0 wait, 1 run, -1 abandon
    // GTNB_EMU_MAX_THREADS=n simulates a host that refuses the (n+1)-th thread (tests/test_dense_emulation.py)
    const char* cap = std::getenv("GTNB_EMU_MAX_THREADS");
    for (unsigned t = 0; t < block; t++) {
      try {
        if (cap && t >= (unsigned)std::atoi(cap)) throw std::system_error(std::make_error_code(std::errc::resource_unavailable_try_again));
        threads.emplace_back([&, t] {
          while (go.load(std::memory_order_acquire) == 0) std::this_thread::yield();
          if (go.load() < 0) return;
          g_cta = &cta;
          threadIdx = Dim3{t, 0, 0};
          blockIdx = Dim3{b, 0, 0};
          blockDim = Dim3{block, 1, 1};
          gridDim = Dim3{grid, 1, 1};
          body();
          // an exited thread no longer takes part in barriers
          cta.bar.arrive_and_drop();
          cta.warp_bar[t / 32]->arrive_and_drop();
        });
      } catch (const std::system_error&) {
        g_launch_failed.store(true);
        break;
      }
    }
    go.store(g_launch_failed.load() ? -1 : 1, std::memory_order_release);
    for (auto& th : threads) th.join();
  }
}

/* the same for a launch with cluster dimension `csize`: the CTAs of one cluster run concurrently
 * (csize * block host threads), clusters one after the other */
template <class F>
void launch_clusters(unsigned grid, unsigned csize, unsigned block, size_t smem_bytes, F&& body) {
  for (unsigned b0 = 0; b0 < grid && !g_launch_failed.load(); b0 += csize) {
    std::vector<std::unique_ptr<Cta>> ctas;
    for (unsigned k = 0; k < csize; k++) ctas.emplace_back(new Cta(block, smem_bytes));
    Cluster cluster(csize * block);
    std::vector<std::thread> threads;
    threads.reserve(csize * block);
    std::atomic<int> go{0};
    for (unsigned k = 0; k < csize && !g_launch_failed.load(); k++)
      for (unsigned t = 0; t < block; t++) {
        try {
          threads.emplace_back([&, k, t] {
            while (go.load(std::memory_order_acquire) == 0) std::this_thread::yield();
            if (go.load() < 0) return;
            Cta& cta = *ctas[k];
            g_cta = &cta;
            g_cluster = &cluster;
            g_cluster_rank = k;
            threadIdx = Dim3{t, 0, 0};
            blockIdx = Dim3{b0 + k, 0, 0};
            blockDim = Dim3{block, 1, 1};
            gridDim = Dim3{grid, 1, 1};
            body();
            cta.bar.arrive_and_drop();
            cta.warp_bar[t / 32]->arrive_and_drop();
            g_cluster = nullptr;
          });
        } catch (const std::system_error&) {
          g_launch_failed.store(true);
          break;
        }
      }
    go.store(g_launch_failed.load() ? -1 : 1, std::memory_order_release);
    for (auto& th : threads) th.join();
  }
}
/* barrier.cluster.arrive + barrier.cluster.wait: every thread of the cluster exactly once per phase */
inline void cluster_sync() {
  g_cluster->bar.arrive_and_wait();
}
/* the split form: arrive now (non-blocking), wait later */
inline thread_local std::barrier<>::arrival_token* g_cluster_token = nullptr;
inline void cluster_arrive() {
  g_cluster_token = new std::barrier<>::arrival_token(g_cluster->bar.arrive());
}
inline void cluster_wait() {
  g_cluster->bar.wait(std::move(*g_cluster_token));
  delete g_cluster_token;
  g_cluster_token = nullptr;
}
inline unsigned cluster_ctarank() {
  return g_cluster_rank;
}

inline uint32_t exchange(uint32_t v, int src_lane) {
  Cta& c = *g_cta;
  const unsigned w = threadIdx.x / 32, l = threadIdx.x % 32;
  c.slots[w][l] = v;
  c.warp_bar[w]->arrive_and_wait();
  const uint32_t r = c.slots[w][src_lane];
  c.warp_bar[w]->arrive_and_wait();
  return r;
}
template <class T>
T shfl(T v, int src_lane) {
  static_assert(sizeof(T) == 4, "32-bit shuffles only");
  uint32_t bits;
  std::memcpy(&bits, &v, 4);
  bits = exchange(bits, src_lane);
  std::memcpy(&v, &bits, 4);
  return v;
}

/* 32-bit shared-window addresses (cvta.to.shared): offsets into the CTA's dynamic shared memory, biased so
 * that 0 is never a valid address */
constexpr uint32_t kWindowBias = 1024;
inline uint32_t shared_window(const void* p) {
  return (uint32_t)(reinterpret_cast<const unsigned char*>(p) -
                    reinterpret_cast<const unsigned char*>(g_cta->dynamic_smem())) + kWindowBias;
}
template <class T>
T* shared_ptr(uint32_t addr) {
  return reinterpret_cast<T*>(reinterpret_cast<unsigned char*>(g_cta->dynamic_smem()) + (addr - kWindowBias));
}
inline void mbar_complete_locked(Cta::MBar& b) {
  if (b.pending == 0 && b.tx == 0) {
    b.phase ^= 1;
    b.pending = b.count;
  }
}
inline void mbar_init(uint32_t bar, int count) {
  std::lock_guard<std::mutex> l(g_cta->mbar_lock);
  Cta::MBar& b = g_cta->mbars[bar];
  b.count = b.pending = count;
  b.phase = 0;
  b.tx = 0;
}
inline void mbar_arrive(uint32_t bar) {
  std::lock_guard<std::mutex> l(g_cta->mbar_lock);
  Cta::MBar& b = g_cta->mbars[bar];
  b.pending--;
  mbar_complete_locked(b);
}
inline void mbar_arrive_n(uint32_t bar, int n) { // mbarrier.arrive with a count
  std::lock_guard<std::mutex> l(g_cta->mbar_lock);
  Cta::MBar& b = g_cta->mbars[bar];
  b.pending -= n;
  mbar_complete_locked(b);
}
inline void mbar_expect_tx(uint32_t bar, uint32_t bytes) { // mbarrier.arrive.expect_tx
  std::lock_guard<std::mutex> l(g_cta->mbar_lock);
  Cta::MBar& b = g_cta->mbars[bar];
  b.tx += bytes;
  b.pending--;
  mbar_complete_locked(b);
}
inline void mbar_wait(uint32_t bar, uint32_t parity) { // try_wait.parity in a loop
  for (;;) {
    {
      std::lock_guard<std::mutex> l(g_cta->mbar_lock);
      if ((uint32_t)g_cta->mbars[bar].phase != parity) return; // the phase with that parity has completed
    }
    std::this_thread::yield();
  }
}
/* cp.async.bulk global -> shared with mbarrier complete_tx: the copy, then the transaction bytes */
inline void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  std::memcpy(shared_ptr<unsigned char>(dst), src, bytes);
  std::lock_guard<std::mutex> l(g_cta->mbar_lock);
  Cta::MBar& b = g_cta->mbars[bar];
  b.tx -= bytes;
  mbar_complete_locked(b);
}

/* bar.sync id, nthreads: the first nthreads threads of the CTA (the same count at every use) */
inline void named_barrier(int id, int nthreads) {
  g_cta->named(id, nthreads).arrive_and_wait();
}

} // namespace emu

inline void __syncthreads() {
  emu::g_cta->bar.arrive_and_wait();
}
inline int __syncthreads_or(int pred) {
  emu::Cta& c = *emu::g_cta;
  if (pred) c.vote.store(1);
  c.bar.arrive_and_wait();
  const int r = c.vote.load();
  c.bar.arrive_and_wait();
  if (threadIdx.x == 0) c.vote.store(0);
  c.bar.arrive_and_wait();
  return r;
}
template <class T>
T __shfl_up_sync(unsigned, T v, int d) {
  const int l = threadIdx.x % 32;
  return emu::shfl(v, l >= d ? l - d : l);
}
template <class T>
T __shfl_down_sync(unsigned, T v, int d) {
  const int l = threadIdx.x % 32;
  return emu::shfl(v, l + d < 32 ? l + d : l);
}
template <class T>
T __shfl_xor_sync(unsigned, T v, int m) {
  const int l = threadIdx.x % 32;
  return emu::shfl(v, l ^ m);
}
template <class T>
T __shfl_sync(unsigned, T v, int src_lane) {
  return emu::shfl(v, src_lane & 31);
}
template <class T>
T __ldcg(const T* p) {
  return *p;
}
inline void __threadfence_block() {
  std::atomic_thread_fence(std::memory_order_seq_cst);
}
inline void __syncwarp(unsigned = 0xffffffffu) {
  emu::g_cta->warp_bar[threadIdx.x / 32]->arrive_and_wait();
}
inline void __nanosleep(unsigned) {
  std::this_thread::yield();
}
inline float __fadd_rn(float a, float b) {
  return a + b;
}
template <class T>
T __ldg(const T* p) {
  return *p;
}
inline int atomicOr(int32_t* p, int v) {
  return std::atomic_ref<int32_t>(*p).fetch_or(v);
}
inline float atomicAdd(float* p, float v) {
  return std::atomic_ref<float>(*p).fetch_add(v);
}
inline int min(int a, int b) {
  return a < b ? a : b;
}
inline int max(int a, int b) {
  return a > b ? a : b;
}
inline unsigned atomicOr(uint32_t* p, uint32_t v) {
  return std::atomic_ref<uint32_t>(*p).fetch_or(v);
}
inline int __float2int_rn(float x) { // cvt.rni.s32.f32: saturating
  if (!(x > -2147483648.0f)) return -2147483647 - 1;
  if (x >= 2147483648.0f) return 2147483647;
  return (int)lrintf(x);
}
inline int __reduce_max_sync(unsigned, int v) { // redux.sync.max.s32 over the full warp
  for (int o = 16; o > 0; o >>= 1) {
    const int w = emu::shfl(v, (int)((threadIdx.x % 32) ^ o));
    v = w > v ? w : v;
  }
  return v;
}
inline unsigned __ballot_sync(unsigned, int pred) {
  unsigned r = 0;
  for (int i = 0; i < 32; i++) r |= (emu::shfl(pred ? 1u : 0u, i) & 1u) << i;
  return r;
}
inline int __popc(unsigned x) {
  return __builtin_popcount(x);
}
inline int __syncthreads_and(int pred) {
  emu::Cta& c = *emu::g_cta;
  if (!pred) c.vote.store(1);
  c.bar.arrive_and_wait();
  const int r = !c.vote.load();
  c.bar.arrive_and_wait();
  if (threadIdx.x == 0) c.vote.store(0);
  c.bar.arrive_and_wait();
  return r;
}
inline int atomicAdd(int* p, int v) {
  return std::atomic_ref<int>(*p).fetch_add(v);
}
inline int atomicExch(int* p, int v) {
  return std::atomic_ref<int>(*p).exchange(v);
}
inline void __threadfence() {
  std::atomic_thread_fence(std::memory_order_seq_cst);
}
inline int atomicMax(int* p, int v) {
  std::atomic_ref<int> a(*p);
  int cur = a.load();
  while (cur < v && !a.compare_exchange_weak(cur, v)) {
  }
  return cur;
}
struct int2 {
  int x, y;
};
struct alignas(16) float4 {
  float x, y, z, w;
};
inline float4 make_float4(float x, float y, float z, float w) {
  return float4{x, y, z, w};
}
inline int2 make_int2(int x, int y) {
  return int2{x, y};
}
inline int __float_as_int(float f) {
  int i;
  std::memcpy(&i, &f, 4);
  return i;
}
inline float __int_as_float(int i) {
  float f;
  std::memcpy(&f, &i, 4);
  return f;
}

/* a static __shared__ array of the running CTA (one per source line) */
#define GTNB_STATIC_SMEM(type, name, count) \
  type* name = reinterpret_cast<type*>(emu::g_cta->static_smem(__LINE__, sizeof(type) * (count)))

#define GTNB_STATIC_SMEM_2D(type, name, d0, d1) \
  type(*name)[d1] = reinterpret_cast<type(*)[d1]>(emu::g_cta->static_smem(__LINE__, sizeof(type) * (d0) * (d1)))

/* dynamic shared memory of the running CTA, 128-byte aligned */
#define GTNB_DYNAMIC_SMEM(type, name) type* name = reinterpret_cast<type*>(emu::g_cta->dynamic_smem())
#define GTNB_DYNAMIC_SMEM_128(type, name) GTNB_DYNAMIC_SMEM(type, name)
