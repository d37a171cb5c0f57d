/*
 * k_gcompose.cu -- composition of two arbitrary graphs on the device: epsilon arcs on the matched side,
 * cyclic operands, neither operand a chain (SURVEY.md 8(f) rank 2; the frame-synchronous case is
 * k_compose.cu).  Target workload: intersect(ctc, transitions) of timeNgramCtc (benchmarks/ctc.cpp:107-134),
 * lexicon / n-gram operands, batched over the B pairs of a list call.
 *
 * What detail::compose does (compose.cpp:377-522), restated for one CTA per pair of graphs:
 *
 *   1. findReachable (compose.cpp:64-104): the product states (n1, n2) from which an accepting pair can be
 *      reached, by a backward search over label-matched in-arc pairs (epsilon:epsilon pairs included, as the
 *      matcher yields them) plus the epsilon in-arcs of either side alone (:146-208 mirrored backward).
 *      Here: a frontier search over a bitmap in global memory, atomicOr + an append-only queue.  The order
 *      of discovery is irrelevant for a set.
 *   2. the forward construction (compose.cpp:389-489): a FIFO search from the start pairs; a popped pair
 *      enumerates its label-matched out-arc pairs in the MATCHER's order (:211-374), then the first operand's
 *      epsilon-output arcs, then the second operand's epsilon-input arcs (the epsMatched / accept filter of
 *      :461-488), keeps the arcs whose destination pair is co-reachable, and numbers a destination pair the
 *      first time it is seen.  A FIFO search is level-synchronous, so the reference's numbering can be
 *      reproduced EXACTLY in parallel: per level, every candidate arc gets its global index k by a prefix sum
 *      over the frontier in queue order (that index IS the reference's arc id), every undiscovered destination
 *      keeps the smallest k that reaches it (atomicMax on -2 - k), and the winners are numbered by a second
 *      prefix sum in k order.  Node ids, arc ids, arc order inside a node and gradInfo (compose.cpp:445,
 *      201-205) therefore equal the reference's, not merely up to isomorphism -- which keeps downstream
 *      float sums (in-arc order, shortest.cpp:121-128) and Viterbi ties (:212-218) identical too.
 *   3. gcompose_fill_kernel: one thread per output node re-enumerates its arcs and writes them at the offsets
 *      of step 2 (the arc storage is allocated between the two kernels, once the totals are known).
 *
 * One thread enumerates one product state; the nested / binary-search matching below is the three matchers
 * of the reference collapsed into "for each arc of the query list, in list order, the arcs of the searched
 * list with the same label, in list order" -- which is what all three produce (the sorted ones find the run
 * by binary search, :282-374).
 */
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "gtnb_gcompose.h"
#include "gtnb_ptx.h"

namespace gtnb {

namespace gc {

#ifdef GTNB_HOST_EMU
constexpr int kThreads = 128; // (the emulation runs one std::thread per CUDA thread: keep the CTA small; same code paths)
#else
constexpr int kThreads = 1024; // one CTA per pair: every warp it can get to hide the latency of the dependent global loads
#endif
constexpr int kEps = -1; // gtn::epsilon (graph.h:21)
constexpr int kCache = 4; // destinations of a light state kept in registers between the passes of the ordered search

/* reach[] and ids[] are updated with atomics (performed in L2): every read goes to L2 as well (ld.global.cg),
 * a line cached in L1 before the update would be stale */
__device__ __forceinline__ bool reach_get(const uint32_t* reach, long long p) {
  return (__ldcg(&reach[p >> 5]) >> (p & 31)) & 1u;
}
__device__ __forceinline__ int32_t id_get(const int32_t* ids, long long p) {
  return __ldcg(&ids[p]);
}

/* arcs of the list `s` (ns arc ids, sorted by label) whose label is >= v: first position */
__device__ __forceinline__ int lower_bound_label(const int32_t* s, int ns, const int32_t* label, int v) {
  int lo = 0, hi = ns;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (label[s[mid]] < v)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

/*
 * The matcher: calls f(i, j) for the arc pairs (i of g1, j of g2) of the lists of (n1, n2) -- in-arc lists if
 * `in`, else out-arc lists -- with olabel1(i) == ilabel2(j), in the reference's order (compose.cpp:211-374):
 *   kind 0  nothing sorted: for i in list1: for j in list2
 *   kind 1  g1's list sorted on the matched label: for j in list2: the run of list1 with that label
 *   kind 2  g2's list sorted: for i in list1: the run of list2
 *   kind 3  both sorted: the LONGER list is searched (g1's if it is strictly longer, :341-345)
 */
template <class F>
__device__ __forceinline__ void for_matches(const GView& g1, const GView& g2, int n1, int n2, bool in, int kind, F f) {
  const int32_t* l = in ? g1.in_arcs + g1.in_ptr[n1] : g1.out_arcs + g1.out_ptr[n1];
  const int nl = in ? g1.in_ptr[n1 + 1] - g1.in_ptr[n1] : g1.out_ptr[n1 + 1] - g1.out_ptr[n1];
  const int32_t* r = in ? g2.in_arcs + g2.in_ptr[n2] : g2.out_arcs + g2.out_ptr[n2];
  const int nr = in ? g2.in_ptr[n2 + 1] - g2.in_ptr[n2] : g2.out_ptr[n2 + 1] - g2.out_ptr[n2];
  if (kind == 0) {
    for (int a = 0; a < nl; a++) {
      const int i = l[a], lab = g1.ol[i];
      for (int b = 0; b < nr; b++)
        if (g2.il[r[b]] == lab) f(i, r[b]);
    }
    return;
  }
  const bool search1 = kind == 3 ? nl > nr : kind == 1;
  if (search1) {
    for (int b = 0; b < nr; b++) {
      const int j = r[b], lab = g2.il[j];
      for (int a = lower_bound_label(l, nl, g1.ol, lab); a < nl && g1.ol[l[a]] == lab; a++) f(l[a], j);
    }
  } else {
    for (int a = 0; a < nl; a++) {
      const int i = l[a], lab = g1.ol[i];
      for (int b = lower_bound_label(r, nr, g2.il, lab); b < nr && g2.il[r[b]] == lab; b++) f(i, r[b]);
    }
  }
}

/*
 * The same pairs for the co-reachability search, where the order does not matter: ONE WARP per product state,
 * the pairs spread over its lanes (a thread walking them alone issues one dependent atomic after the other:
 * 90 in-arc pairs per state for ctc x bigram).  Sorted kinds: every lane takes one arc of the query
 * list and finds its run in the searched list, a warp prefix sum lays the runs end to end, and the lanes stride
 * over that flat index space.  Unsorted: the nl x nr rectangle, flat.
 */
template <class F>
__device__ __forceinline__ void warp_matches(const GView& g1, const GView& g2, int n1, int n2, bool in, int kind, F f) {
  // f(has, i, j) is called by ALL 32 lanes for every chunk of 32 flat positions (has: this lane holds a pair), in
  // flat order -- which is the reference's enumeration order -- so that f may use warp collectives
  const int lane = threadIdx.x & 31;
  const int32_t* l = in ? g1.in_arcs + g1.in_ptr[n1] : g1.out_arcs + g1.out_ptr[n1];
  const int nl = in ? g1.in_ptr[n1 + 1] - g1.in_ptr[n1] : g1.out_ptr[n1 + 1] - g1.out_ptr[n1];
  const int32_t* r = in ? g2.in_arcs + g2.in_ptr[n2] : g2.out_arcs + g2.out_ptr[n2];
  const int nr = in ? g2.in_ptr[n2 + 1] - g2.in_ptr[n2] : g2.out_ptr[n2 + 1] - g2.out_ptr[n2];
  if (kind == 0) {
    const long long tot = (long long)nl * nr;
    for (long long t0 = 0; t0 < tot; t0 += 32) {
      const long long t = t0 + lane;
      int i = -1, j = -1;
      bool has = false;
      if (t < tot) {
        i = l[t / nr];
        j = r[t % nr];
        has = g1.ol[i] == g2.il[j];
      }
      f(has, i, j);
    }
    return;
  }
  const bool search1 = kind == 3 ? nl > nr : kind == 1;
  const int32_t* q = search1 ? r : l; // query list
  const int nq = search1 ? nr : nl;
  const int32_t* sl = search1 ? l : r; // searched list, sorted on its label
  const int ns = search1 ? nl : nr;
  const int32_t* qlab = search1 ? g2.il : g1.ol;
  const int32_t* slab = search1 ? g1.ol : g2.il;
  for (int base = 0; base < nq; base += 32) {
    int qa = -1, lo = 0, len = 0;
    if (base + lane < nq) {
      qa = q[base + lane];
      const int lab = qlab[qa];
      lo = lower_bound_label(sl, ns, slab, lab);
      len = lower_bound_label(sl, ns, slab, lab + 1) - lo;
    }
    int incl = len; // inclusive prefix sum of the run lengths over the warp
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    const int tot = __shfl_sync(0xffffffffu, incl, 31);
    for (int t0 = 0; t0 < tot; t0 += 32) {
      const int t = t0 + lane;
      // owner of flat index t: the first lane whose inclusive sum exceeds it (every lane takes part in the shuffles)
      int own = 0;
#pragma unroll
      for (int step = 16; step > 0; step >>= 1) {
        const int probe = __shfl_sync(0xffffffffu, incl, min(own + step - 1, 31));
        if (own + step <= 32 && probe <= t) own += step;
      }
      own = min(own, 31);
      const int o_incl = __shfl_sync(0xffffffffu, incl, own);
      const int o_len = __shfl_sync(0xffffffffu, len, own);
      const int o_lo = __shfl_sync(0xffffffffu, lo, own);
      const int o_qa = __shfl_sync(0xffffffffu, qa, own);
      int sa = -1;
      if (t < tot) sa = sl[o_lo + (t - (o_incl - o_len))];
      f(t < tot, search1 ? sa : o_qa, search1 ? o_qa : sa);
    }
  }
}

/*
 * The out-arcs of the product state (n1, n2), in the reference's order (compose.cpp:437-488): f(i, j, d1, d2)
 * with j == -1 for an epsilon-output arc of g1 taken alone, i == -1 for an epsilon-input arc of g2 taken alone.
 * Only arcs whose destination is co-reachable.
 */
template <class F>
__device__ __forceinline__ void for_out_arcs(const PairDev& P, int n1, int n2, F f) {
  const GView& g1 = P.g1;
  const GView& g2 = P.g2;
  const long long N1 = g1.N;
  bool eps_matched = false;
  for_matches(g1, g2, n1, n2, false, P.kind, [&](int i, int j) {
    if (g1.ol[i] == kEps) { // epsilon:epsilon is not an arc of the product (:441-444)
      eps_matched = true;
      return;
    }
    const int d1 = g1.dst[i], d2 = g2.dst[j];
    if (reach_get(P.reach, d1 + N1 * d2)) f(i, j, d1, d2);
  });
  const bool acc1 = g1.flags[n1] & 2, acc2 = g2.flags[n2] & 2;
  if (!eps_matched || acc2 || !acc1) {
    const int32_t* l = g1.out_arcs + g1.out_ptr[n1];
    const int nl = g1.out_ptr[n1 + 1] - g1.out_ptr[n1];
    for (int a = 0; a < nl; a++) {
      const int i = l[a];
      if (g1.ol[i] != kEps) continue;
      const int d1 = g1.dst[i];
      if (reach_get(P.reach, d1 + N1 * n2)) f(i, -1, d1, n2);
    }
  }
  if (!eps_matched || acc1) {
    const int32_t* r = g2.out_arcs + g2.out_ptr[n2];
    const int nr = g2.out_ptr[n2 + 1] - g2.out_ptr[n2];
    for (int b = 0; b < nr; b++) {
      const int j = r[b];
      if (g2.il[j] != kEps) continue;
      const int d2 = g2.dst[j];
      if (reach_get(P.reach, n1 + N1 * d2)) f(-1, j, n1, d2);
    }
  }
}

/*
 * The same by ONE WARP, for product states with long arc lists (a lexicon's root against a language-model state:
 * 2000 x 200 arcs to match -- milliseconds for a single thread): f(valid, i, j, d1, d2, ord) is called by all 32
 * lanes per chunk of the flat enumeration, ord = the arc's position among the state's arcs in the reference's order
 * (ballot prefix counts).  Returns the number of arcs (in every lane).
 */
template <class F>
__device__ __forceinline__ int warp_out_arcs(const PairDev& P, int n1, int n2, F f) {
  const GView& g1 = P.g1;
  const GView& g2 = P.g2;
  const long long N1 = g1.N;
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  int base = 0;
  bool eps_matched = false;
  warp_matches(g1, g2, n1, n2, false, P.kind, [&](bool has, int i, int j) {
    const bool eps = has && g1.ol[i] == kEps;
    int d1 = 0, d2 = 0;
    bool valid = false;
    if (has && !eps) {
      d1 = g1.dst[i];
      d2 = g2.dst[j];
      valid = reach_get(P.reach, d1 + N1 * d2);
    }
    eps_matched = eps_matched || __ballot_sync(0xffffffffu, eps) != 0u;
    const unsigned m = __ballot_sync(0xffffffffu, valid);
    f(valid, i, j, d1, d2, base + __popc(m & lt));
    base += __popc(m);
  });
  const bool acc1 = g1.flags[n1] & 2, acc2 = g2.flags[n2] & 2;
  if (!eps_matched || acc2 || !acc1) {
    const int32_t* l = g1.out_arcs + g1.out_ptr[n1];
    const int nl = g1.out_ptr[n1 + 1] - g1.out_ptr[n1];
    for (int a0 = 0; a0 < nl; a0 += 32) {
      int i = -1, d1 = 0;
      bool valid = false;
      if (a0 + lane < nl) {
        i = l[a0 + lane];
        if (g1.ol[i] == kEps) {
          d1 = g1.dst[i];
          valid = reach_get(P.reach, d1 + N1 * n2);
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, valid);
      f(valid, i, -1, d1, n2, base + __popc(m & lt));
      base += __popc(m);
    }
  }
  if (!eps_matched || acc1) {
    const int32_t* r = g2.out_arcs + g2.out_ptr[n2];
    const int nr = g2.out_ptr[n2 + 1] - g2.out_ptr[n2];
    for (int b0 = 0; b0 < nr; b0 += 32) {
      int j = -1, d2 = 0;
      bool valid = false;
      if (b0 + lane < nr) {
        j = r[b0 + lane];
        if (g2.il[j] == kEps) {
          d2 = g2.dst[j];
          valid = reach_get(P.reach, n1 + N1 * d2);
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, valid);
      f(valid, -1, j, n1, d2, base + __popc(m & lt));
      base += __popc(m);
    }
  }
  return base;
}

/* a state goes to a warp when one thread would have to walk a long list: the whole d1 x d2 rectangle when nothing
 * is sorted, the query list (one binary search per arc) otherwise */
#ifdef GTNB_HOST_EMU
constexpr int kHeavyPairs = 12, kHeavyQuery = 4; // (small test graphs must reach the warp path too)
#else
constexpr int kHeavyPairs = 96, kHeavyQuery = 32;
#endif
__device__ __forceinline__ bool heavy_state(const GView& g1, const GView& g2, int n1, int n2, int kind) {
  const long long d1 = g1.out_ptr[n1 + 1] - g1.out_ptr[n1], d2 = g2.out_ptr[n2 + 1] - g2.out_ptr[n2];
  if (kind == 0) return d1 * d2 > kHeavyPairs;
  const bool search1 = kind == 3 ? d1 > d2 : kind == 1;
  return (search1 ? d2 : d1) > kHeavyQuery || d1 + d2 > 8 * kHeavyQuery; // (the epsilon scans walk both lists)
}

/* exclusive prefix sum over the CTA (kThreads threads); returns this thread's prefix, *total the sum */
__device__ __forceinline__ int block_scan(int v, int* warp_sums, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  int base = 0, tot = 0;
  for (int w = 0; w < kThreads / 32; w++) {
    const int s = warp_sums[w];
    if (w < warp) base += s;
    tot += s;
  }
  __syncthreads();
  *total = tot;
  return base + x - v;
}

/*
 * Step 1 with SEVERAL CTAs per pair (a cooperative launch: they must all be resident), for product state spaces
 * large enough that one SM's 32 warps are the bottleneck (lexicon x LM).  The search is a set
 * computation, so the CTAs simply share the frontier of every wave: warp w of CTA c takes the states
 * head + c * W + w, + G * W, ...; new states are appended behind the wave's end through one of three rotating
 * counters (the one of wave k is read after the barrier that ends wave k and reset during wave k + 1, when nobody
 * uses it), and a software barrier over the pair's G CTAs separates the waves.
 * sync[0..2]: the counters, sync[3]: arrivals, sync[4]: generation, sync[5]: end of the initial frontier.
 */
__device__ __forceinline__ void pair_barrier(int32_t* sync, int G) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const int gen = atomicAdd(&sync[4], 0);
    if (atomicAdd(&sync[3], 1) == G - 1) {
      atomicExch(&sync[3], 0);
      __threadfence();
      atomicAdd(&sync[4], 1);
    } else {
      while (atomicAdd(&sync[4], 0) == gen) {
      }
    }
    __threadfence();
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads) gcompose_reach_kernel(const PairDev* __restrict__ pairs, int G) {
  const PairDev P = pairs[blockIdx.x / G];
  const int c = blockIdx.x % G;
  const GView& g1 = P.g1;
  const GView& g2 = P.g2;
  const long long N1 = g1.N;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int W = kThreads / 32;
  int32_t* queue = P.queue;
  int32_t* sync = P.sync;
  // the accepting pairs: CTA 0 (the lists are short)
  if (c == 0) {
    for (long long k = tid; k < (long long)g1.n_accept * g2.n_accept; k += kThreads) {
      const int f = g1.accept[k / g2.n_accept], s = g2.accept[k % g2.n_accept];
      const long long p = f + N1 * s;
      const uint32_t bit = 1u << (p & 31);
      if (!(atomicOr(&P.reach[p >> 5], bit) & bit)) queue[atomicAdd(&sync[5], 1)] = (int32_t)p;
    }
  }
  pair_barrier(sync, G);
  int head = 0, tail = atomicAdd(&sync[5], 0);
  for (int wave = 0; head < tail; wave++) {
    int32_t* cnt = &sync[wave % 3];
    if (c == 0 && tid == 0) atomicExch(&sync[(wave + 1) % 3], 0);
    auto mark = [&](int u1, int u2) {
      const long long p = u1 + N1 * u2;
      const uint32_t bit = 1u << (p & 31);
      if (__ldcg(&P.reach[p >> 5]) & bit) return;
      if (!(atomicOr(&P.reach[p >> 5], bit) & bit)) queue[tail + atomicAdd(cnt, 1)] = (int32_t)p;
    };
    for (int at = head + c * W + warp; at < tail; at += G * W) {
      const int p = __ldcg(&queue[at]);
      const int n1 = (int)(p % N1), n2 = (int)(p / N1);
      warp_matches(g1, g2, n1, n2, true, P.kind, [&](bool has, int i, int j) {
        if (has) mark(g1.src[i], g2.src[j]);
      });
      for (int a = g1.in_ptr[n1] + lane; a < g1.in_ptr[n1 + 1]; a += 32) {
        const int i = g1.in_arcs[a];
        if (g1.ol[i] == kEps) mark(g1.src[i], n2);
      }
      for (int b = g2.in_ptr[n2] + lane; b < g2.in_ptr[n2 + 1]; b += 32) {
        const int j = g2.in_arcs[b];
        if (g2.il[j] == kEps) mark(n1, g2.src[j]);
      }
    }
    pair_barrier(sync, G);
    head = tail;
    tail += atomicAdd(cnt, 0);
  }
}

/* steps 1 and 2: one CTA per pair.  Needs P.reach zeroed and P.ids filled with kUndiscovered. */
__global__ void __launch_bounds__(kThreads) gcompose_search_kernel(const PairDev* __restrict__ pairs) {
  GTNB_STATIC_SMEM(int, warp_sums, kThreads / 32);
  GTNB_STATIC_SMEM(int, q_tail, 1);
  GTNB_STATIC_SMEM(int, n_heavy, 1);
  GTNB_STATIC_SMEM(int, h_list, kThreads); // slots (thread ids) of the chunk's heavy states
  GTNB_STATIC_SMEM(int, h_val, kThreads); // per slot: arc count, then first arc id
  GTNB_STATIC_SMEM(int, h_wins, kThreads); // per slot: winners, then first new node id
  const PairDev P = pairs[blockIdx.x];
  const GView& g1 = P.g1;
  const GView& g2 = P.g2;
  const long long N1 = g1.N;
  const int tid = threadIdx.x;
  int32_t* queue = P.queue;

  const long long t_start = globaltimer();
  const int lane = tid & 31, warp = tid >> 5;
  // ---- 1. co-reachability (compose.cpp:64-104), unless gcompose_reach_kernel has been there
  if (tid == 0) *q_tail = 0;
  __syncthreads();
  if (!P.reach_done) {
  for (long long k = tid; k < (long long)g1.n_accept * g2.n_accept; k += kThreads) {
    const int f = g1.accept[k / g2.n_accept], s = g2.accept[k % g2.n_accept];
    const long long p = f + N1 * s;
    const uint32_t bit = 1u << (p & 31);
    if (!(atomicOr(&P.reach[p >> 5], bit) & bit)) queue[atomicAdd(q_tail, 1)] = (int32_t)p;
  }
  __syncthreads();
  auto mark = [&](int u1, int u2) {
    const long long p = u1 + N1 * u2;
    const uint32_t bit = 1u << (p & 31);
    if (__ldcg(&P.reach[p >> 5]) & bit) return; // most hits are repeats: an L2 read instead of an atomic
    if (!(atomicOr(&P.reach[p >> 5], bit) & bit)) queue[atomicAdd(q_tail, 1)] = (int32_t)p;
  };
  for (int head = 0;;) {
    const int tail = *q_tail;
    __syncthreads(); // everybody has read the tail before anybody moves it
    if (head == tail) break;
    for (int at = head + warp; at < tail; at += kThreads / 32) { // one warp per product state
      const int p = queue[at];
      const int n1 = (int)(p % N1), n2 = (int)(p / N1);
      warp_matches(g1, g2, n1, n2, true, P.kind, [&](bool has, int i, int j) {
        if (has) mark(g1.src[i], g2.src[j]);
      });
      for (int a = g1.in_ptr[n1] + lane; a < g1.in_ptr[n1 + 1]; a += 32) {
        const int i = g1.in_arcs[a];
        if (g1.ol[i] == kEps) mark(g1.src[i], n2);
      }
      for (int b = g2.in_ptr[n2] + lane; b < g2.in_ptr[n2 + 1]; b += 32) {
        const int j = g2.in_arcs[b];
        if (g2.il[j] == kEps) mark(n1, g2.src[j]);
      }
    }
    head = tail;
    __syncthreads();
  }
  } // !reach_done

  const long long t_reach = globaltimer();
  // ---- 2. forward construction in the reference's order (compose.cpp:389-489)
  // start pairs, in (g1.start() x g2.start()) order: serial, the lists are short
  if (tid == 0) {
    int n = 0;
    for (int a = 0; a < g1.n_start; a++)
      for (int b = 0; b < g2.n_start; b++) {
        const long long p = g1.start[a] + N1 * g2.start[b];
        if (reach_get(P.reach, p) && id_get(P.ids, p) < 0) {
          P.ids[p] = n;
          queue[n++] = (int32_t)p;
        }
      }
    *q_tail = n;
  }
  __syncthreads();
  int lo = 0, hi = *q_tail; // the current level: node ids [lo, hi)
  int next_id = hi, arc_base = 0;
  while (lo < hi) {
    for (int c0 = lo; c0 < hi; c0 += kThreads) {
      const int id = c0 + tid;
      const bool on = id < hi;
      int n1 = 0, n2 = 0;
      bool heavy = false;
      if (on) {
        const int p = queue[id];
        n1 = (int)(p % N1);
        n2 = (int)(p / N1);
        heavy = heavy_state(g1, g2, n1, n2, P.kind);
      }
      // states with long arc lists are enumerated by whole warps (h_list: their slots in this chunk)
      if (tid == 0) *n_heavy = 0;
      __syncthreads();
      if (heavy) h_list[atomicAdd(n_heavy, 1)] = tid;
      __syncthreads();
      const int nh = *n_heavy;
      auto state_of = [&](int slot, int& m1, int& m2) {
        const int p = queue[c0 + slot];
        m1 = (int)(p % N1);
        m2 = (int)(p / N1);
      };
      // (a) the arcs of every state of the chunk: counts -> the reference's arc ids
      // (a light state's first kCache destinations are kept in registers: the three passes below then need no
      // second walk through its arc lists -- every state of a CTC-like lattice qualifies)
      int cnt = 0;
      int cand[kCache];
#pragma unroll
      for (int q = 0; q < kCache; q++) cand[q] = 0;
      if (on && !heavy)
        for_out_arcs(P, n1, n2, [&](int, int, int d1, int d2) {
          const int v = (int)(d1 + N1 * d2);
#pragma unroll
          for (int q = 0; q < kCache; q++)
            if (cnt == q) cand[q] = v;
          cnt++;
        });
      const bool cached = !heavy && cnt <= kCache;
      for (int h = warp; h < nh; h += kThreads / 32) {
        int m1, m2;
        state_of(h_list[h], m1, m2);
        const int c = warp_out_arcs(P, m1, m2, [&](bool, int, int, int, int, int) {});
        if (lane == 0) h_val[h_list[h]] = c;
      }
      if (nh) __syncthreads();
      if (heavy) cnt = h_val[tid];
      int total;
      const int off = arc_base + block_scan(cnt, warp_sums, &total);
      if (on) P.arc_off[id] = off;
      if (heavy) h_val[tid] = off;
      arc_base += total;
      if (nh) __syncthreads();
      // (b) every undiscovered destination keeps the smallest arc id that reaches it
      if (on && cached) {
#pragma unroll
        for (int q = 0; q < kCache; q++)
          if (q < cnt && id_get(P.ids, cand[q]) < 0) atomicMax(&P.ids[cand[q]], -2 - (off + q));
      } else if (on && !heavy) {
        int k = off;
        for_out_arcs(P, n1, n2, [&](int, int, int d1, int d2) {
          const long long p = d1 + N1 * d2;
          if (id_get(P.ids, p) < 0) atomicMax(&P.ids[p], -2 - k);
          k++;
        });
      }
      for (int h = warp; h < nh; h += kThreads / 32) {
        int m1, m2;
        state_of(h_list[h], m1, m2);
        const int o = h_val[h_list[h]];
        warp_out_arcs(P, m1, m2, [&](bool valid, int, int, int d1, int d2, int ord) {
          if (!valid) return;
          const long long p = d1 + N1 * d2;
          if (id_get(P.ids, p) < 0) atomicMax(&P.ids[p], -2 - (o + ord));
        });
      }
      __syncthreads();
      // (c) the winners, numbered in arc-id order
      int wins = 0;
      if (on && cached) {
#pragma unroll
        for (int q = 0; q < kCache; q++) wins += q < cnt && id_get(P.ids, cand[q]) == -2 - (off + q);
      } else if (on && !heavy) {
        int k = off;
        for_out_arcs(P, n1, n2, [&](int, int, int d1, int d2) {
          wins += id_get(P.ids, d1 + N1 * d2) == -2 - k;
          k++;
        });
      }
      for (int h = warp; h < nh; h += kThreads / 32) {
        int m1, m2;
        state_of(h_list[h], m1, m2);
        const int o = h_val[h_list[h]];
        int w = 0;
        warp_out_arcs(P, m1, m2, [&](bool valid, int, int, int d1, int d2, int ord) {
          const bool win = valid && id_get(P.ids, d1 + N1 * d2) == -2 - (o + ord);
          w += __popc(__ballot_sync(0xffffffffu, win));
        });
        if (lane == 0) h_wins[h_list[h]] = w;
      }
      if (nh) __syncthreads();
      if (heavy) wins = h_wins[tid];
      const int wbase = next_id + block_scan(wins, warp_sums, &total);
      if (heavy) h_wins[tid] = wbase;
      if (on && cached && wins) {
        int w = wbase;
#pragma unroll
        for (int q = 0; q < kCache; q++)
          if (q < cnt && id_get(P.ids, cand[q]) == -2 - (off + q)) {
            P.ids[cand[q]] = w;
            queue[w] = cand[q];
            w++;
          }
      } else if (on && !heavy && wins) {
        int k = off, w = wbase;
        for_out_arcs(P, n1, n2, [&](int, int, int d1, int d2) {
          const long long p = d1 + N1 * d2;
          if (id_get(P.ids, p) == -2 - k) {
            P.ids[p] = w;
            queue[w] = (int32_t)p;
            w++;
          }
          k++;
        });
      }
      if (nh) __syncthreads();
      for (int h = warp; h < nh; h += kThreads / 32) {
        int m1, m2;
        state_of(h_list[h], m1, m2);
        const int o = h_val[h_list[h]];
        int w = h_wins[h_list[h]];
        const unsigned lt = (1u << lane) - 1u;
        warp_out_arcs(P, m1, m2, [&](bool valid, int, int, int d1, int d2, int ord) {
          const long long p = d1 + N1 * d2;
          const bool win = valid && id_get(P.ids, p) == -2 - (o + ord);
          const unsigned wm = __ballot_sync(0xffffffffu, win);
          if (win) {
            const int nid = w + __popc(wm & lt);
            P.ids[p] = nid;
            queue[nid] = (int32_t)p;
          }
          w += __popc(wm);
        });
      }
      next_id += total;
      __syncthreads();
    }
    lo = hi;
    hi = next_id;
  }
  if (tid == 0) {
    P.arc_off[next_id] = arc_base;
    P.counts[0] = next_id;
    P.counts[1] = arc_base;
    P.counts[2] = (int32_t)((t_reach - t_start) / 1000); // microseconds of the two phases (GTNB_GC_TIMES=1 prints them)
    P.counts[3] = (int32_t)((globaltimer() - t_reach) / 1000);
  }
}

/* step 3: one thread per output node; grid = pairs x blocks_per_pair (ceil(max nodes / kThreads)) */
__global__ void __launch_bounds__(kThreads) gcompose_fill_kernel(const PairDev* __restrict__ pairs, int blocks_per_pair) {
  const PairDev P = pairs[blockIdx.x / blocks_per_pair];
  const int id = (blockIdx.x % blocks_per_pair) * kThreads + threadIdx.x;
  if (id >= P.counts[0]) return;
  const GView& g1 = P.g1;
  const GView& g2 = P.g2;
  const long long N1 = g1.N;
  const int p = P.queue[id];
  const int n1 = (int)(p % N1), n2 = (int)(p / N1);
  P.out_flags[id] = (uint8_t)(((g1.flags[n1] & g2.flags[n2]) & 1) | ((g1.flags[n1] & g2.flags[n2]) & 2));
  int k = P.arc_off[id];
  for_out_arcs(P, n1, n2, [&](int i, int j, int d1, int d2) {
    P.out_src[k] = id;
    P.out_dst[k] = id_get(P.ids, d1 + N1 * d2);
    P.out_il[k] = i >= 0 ? g1.il[i] : kEps;
    P.out_ol[k] = j >= 0 ? g2.ol[j] : kEps;
    // compose.cpp:435 adds the two weights; an epsilon arc carries its own (:201-205)
    P.out_w[k] = i >= 0 && j >= 0 ? g1.w[i] + g2.w[j] : (i >= 0 ? g1.w[i] : g2.w[j]);
    P.out_gi1[k] = i;
    P.out_gi2[k] = j;
    k++;
  });
}

} // namespace gc

#ifndef GTNB_HOST_EMU

namespace {

int launch_gcompose_search(gtnb_ctx* ctx, const gc::PairDev* pairs_dev, int n_pairs) {
  GTNB_LAUNCH(ctx, "gcompose_search", gc::gcompose_search_kernel<<<n_pairs, gc::kThreads, 0, ctx->stream>>>(pairs_dev));
  return GTNB_OK;
}

int launch_gcompose_fill(gtnb_ctx* ctx, const gc::PairDev* pairs_dev, int n_pairs, int max_nodes) {
  const int bpp = (max_nodes + gc::kThreads - 1) / gc::kThreads;
  GTNB_LAUNCH(ctx, "gcompose_fill",
              gc::gcompose_fill_kernel<<<(unsigned)((long long)bpp * n_pairs), gc::kThreads, 0, ctx->stream>>>(pairs_dev, bpp));
  return GTNB_OK;
}

/* one operand graph in the three staging buffers (int32 / float / byte); offsets in elements */
struct Staged {
  long long flags, src, dst, il, ol, w, in_ptr, in_arcs, out_ptr, out_arcs, start, accept;
  int N, A, n_start, n_accept;
};

int stage_graph(gtnb_ctx* ctx, const gtnb_graph_view& v, std::vector<int32_t>& si, std::vector<float>& sf,
                std::vector<uint8_t>& sb, Staged& o) {
  if (v.num_nodes < 0 || v.num_arcs < 0 || (v.num_nodes && !v.node_flags) ||
      (v.num_arcs && (!v.arc_src || !v.arc_dst || !v.arc_ilabel || !v.arc_olabel)))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_compose_graphs: incomplete graph view");
  const int N = v.num_nodes, A = v.num_arcs;
  o.N = N;
  o.A = A;
  for (int a = 0; a < A; a++)
    if (v.arc_src[a] < 0 || v.arc_src[a] >= N || v.arc_dst[a] < 0 || v.arc_dst[a] >= N)
      return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_compose_graphs: arc endpoint out of range");
  auto put = [&](const int32_t* p, long long n) {
    const long long at = (long long)si.size();
    si.insert(si.end(), p, p + n);
    return at;
  };
  o.flags = (long long)sb.size();
  sb.insert(sb.end(), v.node_flags, v.node_flags + N);
  sb.resize((sb.size() + 3) & ~(size_t)3);
  o.src = put(v.arc_src, A);
  o.dst = put(v.arc_dst, A);
  o.il = put(v.arc_ilabel, A);
  o.ol = put(v.arc_olabel, A);
  o.w = (long long)sf.size();
  if (v.weights)
    sf.insert(sf.end(), v.weights, v.weights + A);
  else
    sf.resize(sf.size() + A, 0.0f);
  // g.in(n) / g.out(n): the caller's lists (the Graph's current order), else insertion order
  auto lists = [&](const int32_t* ptr, const int32_t* arcs, const int32_t* key, long long& optr, long long& oarcs) {
    if (ptr && (arcs || A == 0)) {
      optr = put(ptr, N + 1);
      oarcs = put(arcs, A);
      return;
    }
    std::vector<int32_t> p(N + 1, 0), l(A);
    for (int a = 0; a < A; a++) p[key[a] + 1]++;
    for (int n = 0; n < N; n++) p[n + 1] += p[n];
    std::vector<int32_t> at(p.begin(), p.end() - 1);
    for (int a = 0; a < A; a++) l[at[key[a]]++] = a;
    optr = put(p.data(), N + 1);
    oarcs = put(l.data(), A);
  };
  lists(v.in_ptr, v.in_arcs, v.arc_dst, o.in_ptr, o.in_arcs);
  lists(v.out_ptr, v.out_arcs, v.arc_src, o.out_ptr, o.out_arcs);
  auto marked = [&](const int32_t* given, int n_given, uint8_t bit, long long& at, int& n) {
    if (given) {
      at = put(given, n_given);
      n = n_given;
      return;
    }
    std::vector<int32_t> l;
    for (int u = 0; u < N; u++)
      if (v.node_flags[u] & bit) l.push_back(u);
    at = put(l.data(), (long long)l.size());
    n = (int)l.size();
  };
  marked(v.start, v.num_start, 1, o.start, o.n_start);
  marked(v.accept, v.num_accept, 2, o.accept, o.n_accept);
  return GTNB_OK;
}

} // namespace

#endif

} // namespace gtnb

#ifndef GTNB_HOST_EMU

/* the result of gtnb_compose_graphs: the composed graphs, on the device until downloaded */
struct gtnb_composed {
  int n_pairs = 0;
  std::vector<int32_t> nodes, arcs; // per pair
  std::vector<long long> node_off, arc_off; // into the slabs below
  uint8_t* flags = nullptr;
  int32_t* ints = nullptr; // [6][total arcs]: src, dst, ilabel, olabel, gradInfo first, second
  float* w = nullptr;
  long long tot_nodes = 0, tot_arcs = 0;
};

extern "C" {

int gtnb_compose_graphs(
    gtnb_ctx* ctx, int n_pairs, const gtnb_graph_view* first, int n_first, const gtnb_graph_view* second, int n_second,
    const int32_t* match_kind, gtnb_composed** out) {
  using namespace gtnb;
  if (!ctx || !out || n_pairs < 0 || (n_pairs && (!first || !second || !match_kind)) ||
      (n_first != 1 && n_first != n_pairs) || (n_second != 1 && n_second != n_pairs))
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_compose_graphs: bad arguments");
  *out = nullptr;
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  auto res = new gtnb_composed();
  res->n_pairs = n_pairs;
  res->nodes.assign(n_pairs, 0);
  res->arcs.assign(n_pairs, 0);
  res->node_off.assign(n_pairs + 1, 0);
  res->arc_off.assign(n_pairs + 1, 0);
  if (n_pairs == 0) {
    *out = res;
    return GTNB_OK;
  }
  int rc = GTNB_OK;
  std::vector<int32_t> si;
  std::vector<float> sf;
  std::vector<uint8_t> sb;
  std::vector<Staged> g1(n_first), g2(n_second);
  for (int g = 0; g < n_first && !rc; g++) rc = stage_graph(ctx, first[g], si, sf, sb, g1[g]);
  for (int g = 0; g < n_second && !rc; g++) rc = stage_graph(ctx, second[g], si, sf, sb, g2[g]);
  // scratch per pair: reach bitmap, ids, queue, arc offsets, counts
  std::vector<long long> S(n_pairs), reach_at(n_pairs), ids_at(n_pairs), queue_at(n_pairs), aoff_at(n_pairs);
  long long words = 0, ints = 0;
  for (int b = 0; b < n_pairs && !rc; b++) {
    const Staged &a = g1[n_first == 1 ? 0 : b], &c = g2[n_second == 1 ? 0 : b];
    if (match_kind[b] < 0 || match_kind[b] > 3) rc = fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_compose_graphs: match_kind");
    S[b] = (long long)a.N * c.N;
    if (S[b] >= (1ll << 27))
      rc = fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_compose_graphs: more than 2^27 product states");
    reach_at[b] = words;
    words += (S[b] + 31) / 32 + 4;
    ids_at[b] = ints;
    ints += S[b] + 4;
    queue_at[b] = ints;
    ints += S[b] + 4;
    aoff_at[b] = ints;
    ints += S[b] + 4;
  }
  const size_t need = (size_t)(words + ints + (long long)si.size() + (long long)sf.size()) * 4 + sb.size();
  if (!rc && ctx->total_mem && need > ctx->total_mem / 2)
    rc = fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_compose_graphs: scratch larger than half of the device memory");
  int32_t *si_dev = nullptr, *ints_dev = nullptr, *counts_dev = nullptr, *sync_dev = nullptr;
  float* sf_dev = nullptr;
  uint8_t* sb_dev = nullptr;
  uint32_t* words_dev = nullptr;
  gc::PairDev* pairs_dev = nullptr;
  std::vector<gc::PairDev> pairs(n_pairs);
  std::vector<int32_t> counts(4 * (size_t)n_pairs);
#define TRY(x)               \
  do {                       \
    if (!rc) rc = (x);       \
  } while (0)
  TRY(dev_alloc(ctx, &si_dev, (long long)si.size()));
  TRY(dev_alloc(ctx, &sf_dev, (long long)sf.size()));
  TRY(dev_alloc(ctx, &sb_dev, (long long)sb.size()));
  TRY(dev_alloc(ctx, &words_dev, words));
  TRY(dev_alloc(ctx, &ints_dev, ints));
  TRY(dev_alloc(ctx, &counts_dev, 4ll * n_pairs));
  TRY(dev_alloc(ctx, &sync_dev, 8ll * n_pairs));
  TRY(dev_alloc(ctx, &pairs_dev, n_pairs));
  TRY(upload(ctx, si_dev, si.data(), (long long)si.size()));
  TRY(upload(ctx, sf_dev, sf.data(), (long long)sf.size()));
  TRY(upload(ctx, sb_dev, sb.data(), (long long)sb.size()));
  if (!rc) {
    auto view = [&](const Staged& s) {
      gc::GView v;
      v.N = s.N;
      v.A = s.A;
      v.flags = sb_dev + s.flags;
      v.src = si_dev + s.src;
      v.dst = si_dev + s.dst;
      v.il = si_dev + s.il;
      v.ol = si_dev + s.ol;
      v.w = sf_dev + s.w;
      v.in_ptr = si_dev + s.in_ptr;
      v.in_arcs = si_dev + s.in_arcs;
      v.out_ptr = si_dev + s.out_ptr;
      v.out_arcs = si_dev + s.out_arcs;
      v.start = si_dev + s.start;
      v.n_start = s.n_start;
      v.accept = si_dev + s.accept;
      v.n_accept = s.n_accept;
      return v;
    };
    for (int b = 0; b < n_pairs; b++) {
      gc::PairDev& P = pairs[b];
      std::memset(&P, 0, sizeof(P));
      P.g1 = view(g1[n_first == 1 ? 0 : b]);
      P.g2 = view(g2[n_second == 1 ? 0 : b]);
      P.kind = match_kind[b];
      P.reach = words_dev + reach_at[b];
      P.ids = ints_dev + ids_at[b];
      P.queue = ints_dev + queue_at[b];
      P.arc_off = ints_dev + aoff_at[b];
      P.counts = counts_dev + 4 * b;
      P.sync = sync_dev + 8 * b;
    }
    cudaError_t e = cudaMemsetAsync(words_dev, 0, sizeof(uint32_t) * (size_t)words, ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(ints_dev, 0x80, sizeof(int32_t) * (size_t)ints, ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(counts_dev, 0, sizeof(int32_t) * 4 * (size_t)n_pairs, ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(sync_dev, 0, sizeof(int32_t) * 8 * (size_t)n_pairs, ctx->stream);
    if (e != cudaSuccess) rc = cuda_fail(ctx, e, "cudaMemsetAsync", __FILE__, __LINE__);
  }
  // large product state spaces: the co-reachability search on several SMs per pair (cooperative launch)
  int G = 1;
  if (!rc) {
    long long maxS = 0;
    for (int b = 0; b < n_pairs; b++) maxS = std::max(maxS, S[b]);
    int sms = 0, per_sm = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gc::gcompose_reach_kernel, gc::kThreads, 0);
    const long long room = (long long)sms * per_sm / n_pairs;
    if (maxS >= 65536 && room >= 2) G = (int)std::min<long long>(std::min<long long>(room, 64), maxS / 16384);
    if (G < 2) G = 1;
    for (int b = 0; b < n_pairs; b++) pairs[b].reach_done = G > 1 ? 1 : 0;
  }
  TRY(upload(ctx, pairs_dev, pairs.data(), n_pairs));
  if (!rc && G > 1) {
    const gc::PairDev* pd = pairs_dev;
    void* args[] = {(void*)&pd, (void*)&G};
    prof_begin(ctx, "gcompose_reach");
    cudaError_t e = cudaLaunchCooperativeKernel((const void*)gc::gcompose_reach_kernel, dim3((unsigned)(n_pairs * G)),
                                                dim3(gc::kThreads), args, 0, ctx->stream);
    prof_end(ctx);
    if (e != cudaSuccess) { // not co-resident right now: the single-CTA search does step 1 itself
      cudaGetLastError();
      G = 1;
      for (int b = 0; b < n_pairs; b++) pairs[b].reach_done = 0;
      TRY(upload(ctx, pairs_dev, pairs.data(), n_pairs));
    } else {
      ctx->launches++;
    }
  }
  TRY(launch_gcompose_search(ctx, pairs_dev, n_pairs));
  if (!rc) {
    cudaError_t e = cudaMemcpyAsync(counts.data(), counts_dev, sizeof(int32_t) * counts.size(), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) rc = cuda_fail(ctx, e, "read-back of the composed sizes", __FILE__, __LINE__);
  }
  int max_nodes = 0;
  if (!rc) {
    for (int b = 0; b < n_pairs; b++) {
      res->nodes[b] = counts[4 * b];
      res->arcs[b] = counts[4 * b + 1];
      res->node_off[b + 1] = res->node_off[b] + ((counts[4 * b] + 3) & ~3);
      res->arc_off[b + 1] = res->arc_off[b] + ((counts[4 * b + 1] + 3) & ~3);
      max_nodes = std::max(max_nodes, counts[4 * b]);
      if (b == 0 && std::getenv("GTNB_GC_TIMES"))
        std::fprintf(stderr, "[gtnb_compose_graphs] pair 0: %d nodes, %d arcs, co-reachability %d us, forward %d us\n",
                     counts[0], counts[1], counts[2], counts[3]);
    }
    res->tot_nodes = res->node_off[n_pairs];
    res->tot_arcs = res->arc_off[n_pairs];
  }
  TRY(dev_alloc(ctx, &res->flags, res->tot_nodes));
  TRY(dev_alloc(ctx, &res->ints, 6 * res->tot_arcs));
  TRY(dev_alloc(ctx, &res->w, res->tot_arcs));
  if (!rc && max_nodes > 0) {
    for (int b = 0; b < n_pairs; b++) {
      gc::PairDev& P = pairs[b];
      P.out_flags = res->flags + res->node_off[b];
      int32_t* base = res->ints + res->arc_off[b];
      P.out_src = base;
      P.out_dst = base + res->tot_arcs;
      P.out_il = base + 2 * res->tot_arcs;
      P.out_ol = base + 3 * res->tot_arcs;
      P.out_gi1 = base + 4 * res->tot_arcs;
      P.out_gi2 = base + 5 * res->tot_arcs;
      P.out_w = res->w + res->arc_off[b];
    }
    TRY(upload(ctx, pairs_dev, pairs.data(), n_pairs));
    TRY(launch_gcompose_fill(ctx, pairs_dev, n_pairs, max_nodes));
  }
#undef TRY
  // the scratch goes back (stream-ordered: after the kernels above)
  dev_free(ctx, si_dev);
  dev_free(ctx, sf_dev);
  dev_free(ctx, sb_dev);
  dev_free(ctx, words_dev);
  dev_free(ctx, ints_dev);
  dev_free(ctx, counts_dev);
  dev_free(ctx, sync_dev);
  dev_free(ctx, pairs_dev);
  if (rc) {
    gtnb_composed_destroy(ctx, res);
    return rc;
  }
  *out = res;
  return GTNB_OK;
}

int gtnb_composed_sizes(const gtnb_composed* c, int pair, int32_t* num_nodes, int32_t* num_arcs) {
  if (!c || pair < 0 || pair >= c->n_pairs) return GTNB_ERR_INVALID_ARGUMENT;
  if (num_nodes) *num_nodes = c->nodes[pair];
  if (num_arcs) *num_arcs = c->arcs[pair];
  return GTNB_OK;
}

int gtnb_composed_download(
    gtnb_ctx* ctx, gtnb_composed* c, int pair, uint8_t* node_flags, int32_t* arc_src, int32_t* arc_dst,
    int32_t* arc_ilabel, int32_t* arc_olabel, float* weights, int32_t* gi_first, int32_t* gi_second) {
  using namespace gtnb;
  if (!ctx || !c || pair < 0 || pair >= c->n_pairs)
    return fail(ctx, GTNB_ERR_INVALID_ARGUMENT, "gtnb_composed_download: bad arguments");
  GTNB_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t N = (size_t)c->nodes[pair], A = (size_t)c->arcs[pair];
  if (node_flags && N)
    GTNB_CUDA(ctx, cudaMemcpyAsync(node_flags, c->flags + c->node_off[pair], N, cudaMemcpyDeviceToHost, ctx->stream));
  int32_t* outs[6] = {arc_src, arc_dst, arc_ilabel, arc_olabel, gi_first, gi_second};
  for (int k = 0; k < 6; k++)
    if (outs[k] && A)
      GTNB_CUDA(ctx, cudaMemcpyAsync(outs[k], c->ints + c->arc_off[pair] + k * c->tot_arcs, sizeof(int32_t) * A,
                                     cudaMemcpyDeviceToHost, ctx->stream));
  if (weights && A)
    GTNB_CUDA(ctx, cudaMemcpyAsync(weights, c->w + c->arc_off[pair], sizeof(float) * A, cudaMemcpyDeviceToHost, ctx->stream));
  GTNB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return GTNB_OK;
}

void gtnb_composed_destroy(gtnb_ctx* ctx, gtnb_composed* c) {
  using namespace gtnb;
  if (!c) return;
  if (ctx) {
    cudaSetDevice(ctx->device);
    dev_free(ctx, c->flags);
    dev_free(ctx, c->ints);
    dev_free(ctx, c->w);
  }
  delete c;
}

} // extern "C"

#endif // GTNB_HOST_EMU
