/*
 * k_staged.cu -- the hot kernels: shortest-distance forward / backward over
 * frame-synchronous ("level-local") lattices, one persistent warp-specialised
 * CTA per utterance.
 *
 *   producer warp   walks the levels ahead of the math: for level l it issues
 *                   cp.async.bulk (TMA 1-D bulk copies, SASS UBLKCP) of the
 *                   level's row_ptr window and arc-record window ({src, weight}
 *                   pairs; backward also the saved node scores) from HBM into a
 *                   ring of shared-memory stages, completion tracked by mbarrier
 *                   transaction counts.
 *   consumer warps  wait on the stage's "full" mbarrier, evaluate every node of
 *                   the level from shared memory (frontier scores live in a
 *                   shared double buffer), write node scores / arc gradients back
 *                   coalesced, and hand the stage back through an "empty"
 *                   mbarrier.  G lanes cooperate on one destination node and
 *                   reduce max / sum(exp) with warp shuffles (G = 1 for CTC-like
 *                   lattices with <= 4 in-arcs per node: fully unrolled).
 *
 * Reference semantics: shortestDistance (shortest.cpp:86-188), its gradient
 * (shortest.cpp:33-82) and shortestPath's relaxation (shortest.cpp:190-238);
 * k_shortest.cu holds the generic (any-DAG, libm-precise) versions these are
 * tested against.  The log-semiring math here uses ex2.approx / lg2.approx
 * (relative error ~1e-6, far inside the 1e-4 bar); the tropical semiring and
 * the path recursion are exact (adds and compares only).
 *
 * Windows: level l's nodes are [lo, hi), its in-arcs [alo, ahi).  Bulk copies
 * need 16-byte aligned addresses and sizes, so a stage holds the supersets
 * [lo & ~3, align4(hi + 1)) of row_ptr / scores and [alo & ~1, align2(ahi)) of
 * the 8-byte arc records; per-graph slabs start on 4-element boundaries and
 * every array has 16 elements of slack, so the extra elements are always mapped.
 */
#include <algorithm>

#include "gtnb_ptx.h"

namespace gtnb {

namespace {

// consumer warps per CTA.  The level time is set by the instruction stream of ONE warp
// (its issue-to-issue latency per instruction), so one node per thread and as
// few instructions per level as possible beats fewer, fatter warps.
constexpr int consumer_warps(int /*G*/) {
  return 8;
}
constexpr int kMaxLevelsInSmem = 6144;
constexpr int kMaxStages = 8;

/* Shared-memory carve-up, computed on the host and passed by value. */
struct Layout {
  int win_nodes; // elements per row_ptr / score window
  int win_arcs; // arc records per window
  int off_lvln, off_lvla, off_bufs, off_stage; // byte offsets
  int stage_bytes;
  int st_arcs, st_psc; // byte offsets inside a stage (row_ptr at 0)
  int total;
  int log2_stages;
  int off_tab; // graph-operand tables of the fused criterion backward (0 = none)
  int tab_nodes, tab_arcs;
};

Layout make_layout(int max_lvl_nodes, int max_lvl_arcs, int L, int log2_stages, int n_bufs, bool with_scores) {
  Layout o;
  o.log2_stages = log2_stages;
  o.win_nodes = ((max_lvl_nodes + 1 + 3 + 3) / 4) * 4 + 4;
  o.win_arcs = ((max_lvl_arcs + 1 + 1) / 2) * 2 + 2;
  int lvl_cap = ((L + 1 + 3) / 4) * 4;
  int off = 2 * 8 * kMaxStages; // full[], empty[]
  o.off_lvln = off;
  off += 4 * lvl_cap;
  o.off_lvla = off;
  off += 4 * lvl_cap;
  o.off_bufs = off;
  off += 4 * n_bufs * o.win_nodes;
  off = (off + 127) / 128 * 128;
  o.off_stage = off;
  o.st_arcs = (4 * o.win_nodes + 15) / 16 * 16;
  o.st_psc = o.st_arcs + 8 * o.win_arcs;
  o.stage_bytes = o.st_psc + (with_scores ? 4 * o.win_nodes : 0);
  o.stage_bytes = (o.stage_bytes + 127) / 128 * 128;
  o.total = off + o.stage_bytes * (1 << log2_stages);
  o.off_tab = 0;
  o.tab_nodes = o.tab_arcs = 0;
  return o;
}


/* ---- per-node evaluation, one thread per node (G == 1) ---------------- */

/* any in-degree, start nodes included: the reference's loop verbatim (shortest.cpp:121-136) */
template <int MODE>
__device__ __noinline__ float fwd_node_any(uint32_t r0raw, int r0, int r1, const int2* st_arc, const float* prev) {
  const bool is_start = (r0raw & kStartBit) != 0;
  float mx = -CUDART_INF_F;
#pragma unroll 1
  for (int a = r0; a < r1; a++) {
    const int2 rec = st_arc[a];
    mx = fmaxf(mx, prev[rec.x] + __int_as_float(rec.y));
  }
  if (is_start) mx = fmaxf(mx, 0.0f);
  if (MODE != MODE_LOG || mx == CUDART_INF_F || mx == -CUDART_INF_F) return mx;
  float sum = -1.0f;
#pragma unroll 1
  for (int a = r0; a < r1; a++) {
    const int2 rec = st_arc[a];
    sum += fexp((prev[rec.x] + __int_as_float(rec.y)) - mx);
  }
  if (is_start) sum += fexp(0.0f - mx);
  return mx + flog1p(sum);
}

/* the common row: <= 3 in-arcs, not a start node (every CTC / forced-alignment lattice row
 * past frame 0): fully unrolled, absent arcs contribute exp(-inf) = 0 in arc order.
 * R = shared address of row_ptr[node 0 of the level], A = shared address arc record 0 would
 * have, P = shared address score of node 0 would have (both may lie before the window). */
template <int MODE>
__device__ __forceinline__ float fwd_node(
    int i, uint32_t R, uint32_t A, uint32_t P, const int2* st_arc, const float* prev) {
  const uint32_t r0raw = lds_u32(R + 4u * i);
  const uint32_t r1raw = lds_u32(R + 4u * i + 4u);
  const int r0 = (int)(r0raw & kRowMask);
  const int deg = (int)(r1raw & kRowMask) - r0;
  if (deg > 3 || (r0raw & kStartBit)) return fwd_node_any<MODE>(r0raw, r0, r0 + deg, st_arc, prev);
  const uint32_t a = A + 8u * r0;
  float v0 = -CUDART_INF_F, v1 = -CUDART_INF_F, v2 = -CUDART_INF_F;
  if (deg > 0) {
    const int2 rec = lds_v2_u32(a);
    v0 = lds_f32(P + 4u * rec.x) + __int_as_float(rec.y);
  }
  if (deg > 1) {
    const int2 rec = lds_v2_u32(a + 8u);
    v1 = lds_f32(P + 4u * rec.x) + __int_as_float(rec.y);
  }
  if (deg > 2) {
    const int2 rec = lds_v2_u32(a + 16u);
    v2 = lds_f32(P + 4u * rec.x) + __int_as_float(rec.y);
  }
  const float mx = fmaxf(fmaxf(v0, v1), v2);
  if (MODE != MODE_LOG || mx == CUDART_INF_F || mx == -CUDART_INF_F) return mx;
  float sum = -1.0f;
  sum += fexp(v0 - mx);
  sum += fexp(v1 - mx);
  sum += fexp(v2 - mx);
  return mx + flog1p(sum);
}

/* ------------------------------------------------------------------ */
/* forward                                                             */
/* ------------------------------------------------------------------ */

template <int MODE, int G>
__global__ void __launch_bounds__(32 * consumer_warps(G) + 32) sd_forward_staged(
    const GraphMeta* __restrict__ meta,
    const int32_t* __restrict__ lvl_node_ptr,
    const int32_t* __restrict__ lvl_arc_ptr,
    const uint32_t* __restrict__ row_ptr,
    const int2* __restrict__ arcs,
    const int32_t* __restrict__ acc_nodes,
    float* __restrict__ scores,
    int32_t* __restrict__ back_ptr,
    float* __restrict__ out_scores,
    int32_t* __restrict__ best_accept,
    const Layout lay) {
  GTNB_DYNAMIC_SMEM_128(unsigned char, smem);
  constexpr int kConsumers = 32 * consumer_warps(G);
  constexpr int kStagedThreads = kConsumers + 32;
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x;
  const int S = 1 << lay.log2_stages;
  const uint32_t sbase = smem_u32(smem);
  int* s_lvln = reinterpret_cast<int*>(smem + lay.off_lvln);
  int* s_lvla = reinterpret_cast<int*>(smem + lay.off_lvla);
  float* s_sc = reinterpret_cast<float*>(smem + lay.off_bufs);

  const int L = m.L;
  for (int i = tid; i <= L; i += kStagedThreads) {
    s_lvln[i] = lvl_node_ptr[m.lvl_base + i];
    s_lvla[i] = lvl_arc_ptr[m.lvl_base + i];
  }
  if (tid == 0) {
    for (int s = 0; s < S; s++) {
      mbar_init(sbase + 8 * s, 1);
      mbar_init(sbase + 8 * (kMaxStages + s), 1);
    }
    mbar_init_fence();
  }
  __syncthreads();

  if (tid >= kConsumers) {
    // ===== producer =====
    if (tid == kConsumers) {
      const uint32_t* rp = row_ptr + m.node_base;
      const int2* ga = arcs + m.arc_base;
      int s = 0;
      uint32_t par = 0; // wraps & 1: the slot's previous use is empty-phase (wraps - 1)
#pragma unroll 1
      for (int l = 0; l < L; l++) {
        if (l >= S) mbar_wait_sleep(sbase + 8 * (kMaxStages + s), par ^ 1);
        const uint32_t st = sbase + lay.off_stage + s * lay.stage_bytes;
        const uint32_t fb = sbase + 8 * s;
        const int lo = s_lvln[l], hi = s_lvln[l + 1];
        const int alo = s_lvla[l], ahi = s_lvla[l + 1];
        const int n0 = lo & ~3, n1 = (hi + 1 + 3) & ~3;
        const int a0 = alo & ~1, a1 = (ahi + 1) & ~1;
        const uint32_t nb = (uint32_t)(n1 - n0) * 4u, ab = (uint32_t)(a1 - a0) * 8u;
        mbar_expect_tx(fb, nb + ab);
        bulk_g2s(st, rp + n0, nb, fb);
        if (ab) bulk_g2s(st + lay.st_arcs, ga + a0, ab, fb);
        if (++s == S) {
          s = 0;
          par ^= 1;
        }
      }
    }
    return;
  }

  // ===== consumers =====
  float* sc = scores + m.node_base;
  int32_t* bp = (MODE == MODE_PATH) ? back_ptr + m.node_base : nullptr;
  const int sub = tid % G;
  const int slot = tid / G;
  // lanes cooperating on one node; shuffles stay inside the group so that groups may diverge
  const unsigned gmask = (G >= 32) ? 0xffffffffu : (((1u << G) - 1u) << ((tid & 31) & ~(G - 1)));
  int s = 0;
  uint32_t par = 0;
  int lo = s_lvln[0];
  int prev_lo = 0;
  for (int l = 0; l < L; l++) {
    const int hi = s_lvln[l + 1];
    const int a0 = s_lvla[l] & ~1;
    const unsigned char* st = smem + lay.off_stage + s * lay.stage_bytes;
    const uint32_t* st_rp = reinterpret_cast<const uint32_t*>(st) + (lo & 3);
    const int2* st_arc = reinterpret_cast<const int2*>(st + lay.st_arcs) - a0;
    const float* prev = s_sc + ((l & 1) ^ 1) * lay.win_nodes - prev_lo;
    float* cur = s_sc + (l & 1) * lay.win_nodes;
    const int cnt = hi - lo;
    mbar_wait(sbase + 8 * s, par);
    if (G == 1 && MODE != MODE_PATH) {
      // one thread per node
      const uint32_t stb = sbase + lay.off_stage + s * lay.stage_bytes;
      const uint32_t R = stb + 4u * (lo & 3);
      const uint32_t A = stb + lay.st_arcs - 8u * a0;
      const uint32_t bufs = sbase + lay.off_bufs;
      const uint32_t P = bufs + 4u * (((l & 1) ^ 1) * lay.win_nodes - prev_lo);
      const uint32_t Cw = bufs + 4u * ((l & 1) * lay.win_nodes);
      for (int i = tid; i < cnt; i += kConsumers) {
        const float sv = fwd_node<MODE>(i, R, A, P, st_arc, prev);
        sts_f32(Cw + 4u * i, sv);
        sc[lo + i] = sv;
      }
    } else
    for (int i0 = 0; i0 < cnt; i0 += kConsumers / G) {
      const int i = i0 + slot;
      const bool live = i < cnt;
      uint32_t r0raw = 0;
      int r0 = 0, r1 = 0;
      if (live) {
        r0raw = st_rp[i];
        r0 = (int)(r0raw & kRowMask);
        r1 = (int)(st_rp[i + 1] & kRowMask);
      }
      const bool is_start = (r0raw & kStartBit) != 0;
      const int deg = r1 - r0;
      if (MODE == MODE_PATH) {
        // strictly-greater relaxations in arc order; a start node begins at 0 (shortest.cpp:202-218)
        float best = -CUDART_INF_F;
        int barc = 0x7fffffff;
        for (int a = r0 + sub; a < r1; a += G) {
          const int2 rec = st_arc[a];
          const float v = prev[rec.x] + __int_as_float(rec.y);
          if (v > best) {
            best = v;
            barc = a;
          }
        }
        if (G > 1) {
#pragma unroll
          for (int o = G / 2; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(gmask, best, o);
            const int oa = __shfl_xor_sync(gmask, barc, o);
            if (ob > best || (ob == best && oa < barc)) {
              best = ob;
              barc = oa;
            }
          }
        }
        if (is_start && !(best > 0.0f)) {
          best = 0.0f;
          barc = 0x7fffffff;
        }
        if (live && sub == 0) {
          cur[i] = best;
          sc[lo + i] = best;
          bp[lo + i] = (barc == 0x7fffffff) ? -1 : barc;
        }
      } else {
        float mx = -CUDART_INF_F;
#pragma unroll 1
        for (int a = r0 + sub; a < r1; a += G) {
          const int2 rec = st_arc[a];
          mx = fmaxf(mx, prev[rec.x] + __int_as_float(rec.y));
        }
        if (G > 1) {
#pragma unroll
          for (int o = G / 2; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(gmask, mx, o));
        }
        if (is_start) mx = fmaxf(mx, 0.0f);
        float score = mx;
        if (MODE == MODE_LOG && mx != CUDART_INF_F && mx != -CUDART_INF_F) {
          float sum = (sub == 0) ? -1.0f : 0.0f;
#pragma unroll 1
          for (int a = r0 + sub; a < r1; a += G) {
            const int2 rec = st_arc[a];
            sum += fexp((prev[rec.x] + __int_as_float(rec.y)) - mx);
          }
          if (G > 1) {
#pragma unroll
            for (int o = G / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(gmask, sum, o);
          }
          if (is_start) sum += fexp(0.0f - mx);
          score = mx + flog1p(sum);
        }
        if (live && sub == 0) {
          cur[i] = score;
          sc[lo + i] = score;
        }
      }
    }
    bar_named<1, kConsumers>();
    if (tid == 0) mbar_arrive(sbase + 8 * (kMaxStages + s));
    if (++s == S) {
      s = 0;
      par ^= 1;
    }
    prev_lo = lo;
    lo = hi;
  }

  // accept nodes (all in the last level): shortest.cpp:147-159 / :226-237
  if (tid == 0) {
    const int32_t* acc = acc_nodes + m.acc_base;
    float mx = -CUDART_INF_F;
    int best = -1;
    for (int k = 0; k < m.n_accept; k++) {
      const float v = __ldcg(&sc[acc[k]]);
      if (v > mx) {
        mx = v;
        best = acc[k];
      }
    }
    float out;
    if (MODE == MODE_LOG) {
      if (m.n_accept == 0) {
        out = -CUDART_INF_F;
      } else if (mx == CUDART_INF_F || mx == -CUDART_INF_F) {
        out = mx;
      } else {
        float sum = -1.0f;
        for (int k = 0; k < m.n_accept; k++) sum += expf(__ldcg(&sc[acc[k]]) - mx);
        out = mx + log1pf(sum);
      }
    } else {
      out = (m.n_accept == 0) ? -CUDART_INF_F : mx;
    }
    out_scores[blockIdx.x] = out;
    best_accept[blockIdx.x] = best;
  }
}

/* ------------------------------------------------------------------ */
/* backward                                                            */
/* ------------------------------------------------------------------ */


/* any row, reference formula verbatim (shortest.cpp:62-80), libm-precise */
__device__ __noinline__ void bwd_node_any(
    uint32_t r0raw, int r0, int r1, float g, float sn, float delta, const int2* st_arc,
    const float* st_psc, float* ng_prev, float* ag) {
  float mx = -CUDART_INF_F;
#pragma unroll 1
  for (int a = r0; a < r1; a++) {
    const int2 rec = st_arc[a];
    mx = fmaxf(mx, st_psc[rec.x] + __int_as_float(rec.y));
  }
  if (r0raw & kStartBit) mx = fmaxf(mx, 0.0f);
  const float denom = expf(sn - mx);
#pragma unroll 1
  for (int a = r0; a < r1; a++) {
    const int2 rec = st_arc[a];
    const float cur = g * expf(st_psc[rec.x] + __int_as_float(rec.y) - mx) / denom;
    atomicAdd(&ng_prev[rec.x], cur);
    ag[a] = cur * delta;
  }
}

/* the common row: <= 3 in-arcs, finite score.  g * exp(v - max) / exp(score - max)
 * == g * exp(v - score) then, one SFU op per arc.  R / A / P as in fwd_node (P = saved
 * scores of the level below), NGc / OWN = this level's node gradients / scores, NGp = the
 * node-gradient accumulator of the level below (address node 0 of that level would have). */
__device__ __forceinline__ void bwd_node(
    int i, uint32_t R, uint32_t A, uint32_t P, uint32_t NGc, uint32_t OWN, uint32_t NGp,
    float delta, float* ag, const int2* st_arc, const float* st_psc, float* ng_prev) {
  const uint32_t r0raw = lds_u32(R + 4u * i);
  const uint32_t r1raw = lds_u32(R + 4u * i + 4u);
  const int r0 = (int)(r0raw & kRowMask);
  const int deg = (int)(r1raw & kRowMask) - r0;
  const float g = lds_f32(NGc + 4u * i);
  const float sn = lds_f32(OWN + 4u * i);
  if (deg > 3 || (r0raw & kStartBit) || !(fabsf(sn) < CUDART_INF_F)) {
    bwd_node_any(r0raw, r0, r0 + deg, g, sn, delta, st_arc, st_psc, ng_prev, ag);
    return;
  }
  const uint32_t a = A + 8u * r0;
#pragma unroll
  for (int j = 0; j < 3; j++) {
    if (j < deg) {
      const int2 rec = lds_v2_u32(a + 8u * j);
      const float cur = g * fexp(lds_f32(P + 4u * rec.x) + __int_as_float(rec.y) - sn);
      red_shared_add(NGp + 4u * rec.x, cur);
      ag[r0 + j] = cur * delta;
    }
  }
}

/* one arc of the log-semiring gradient (shortest.cpp:71-75) */
__device__ __forceinline__ float arc_grad_log(float g, float v, float sn, float mx, bool exact) {
  // g * exp(v - max) / exp(score - max) == g * exp(v - score) whenever the score is finite;
  // the exact form reproduces the reference's NaNs for +-inf scores (autograd_test.cpp:340-386)
  return exact ? g * expf(v - mx) / expf(sn - mx) : g * fexp(v - sn);
}

template <bool TROPICAL, int G>
__global__ void __launch_bounds__(32 * consumer_warps(G) + 32) sd_backward_staged(
    const GraphMeta* __restrict__ meta,
    const int32_t* __restrict__ lvl_node_ptr,
    const int32_t* __restrict__ lvl_arc_ptr,
    const uint32_t* __restrict__ row_ptr,
    const int2* __restrict__ arcs,
    const int32_t* __restrict__ acc_nodes,
    const float* __restrict__ scores,
    const float* __restrict__ out_scores,
    const int32_t* __restrict__ best_accept,
    const float* __restrict__ deltas,
    float* __restrict__ arc_grad,
    const Layout lay) {
  GTNB_DYNAMIC_SMEM_128(unsigned char, smem);
  constexpr int kConsumers = 32 * consumer_warps(G);
  constexpr int kStagedThreads = kConsumers + 32;
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x;
  const int S = 1 << lay.log2_stages;
  const uint32_t sbase = smem_u32(smem);
  int* s_lvln = reinterpret_cast<int*>(smem + lay.off_lvln);
  int* s_lvla = reinterpret_cast<int*>(smem + lay.off_lvla);
  // buffers: 3 node-gradient buffers + 1 score window for the top level
  float* s_ng = reinterpret_cast<float*>(smem + lay.off_bufs);
  float* s_top = s_ng + 3 * lay.win_nodes;

  const int L = m.L;
  for (int i = tid; i <= L; i += kStagedThreads) {
    s_lvln[i] = lvl_node_ptr[m.lvl_base + i];
    s_lvla[i] = lvl_arc_ptr[m.lvl_base + i];
  }
  if (tid == 0) {
    for (int s = 0; s < S; s++) {
      mbar_init(sbase + 8 * s, 1);
      mbar_init(sbase + 8 * (kMaxStages + s), 1);
    }
    mbar_init_fence();
  }
  __syncthreads();

  const float* gsc = scores + m.node_base;
  const int iters = L - 1; // levels L-1 .. 1 own in-arcs

  if (tid >= kConsumers) {
    // ===== producer: iteration k handles level l = L-1-k; its stage carries the
    // row_ptr / arc windows of level l and the saved scores of level l-1 =====
    if (tid == kConsumers) {
      const uint32_t* rp = row_ptr + m.node_base;
      const int2* ga = arcs + m.arc_base;
      int s = 0;
      uint32_t par = 0;
#pragma unroll 1
      for (int k = 0; k < iters; k++) {
        const int l = L - 1 - k;
        if (k >= S) mbar_wait_sleep(sbase + 8 * (kMaxStages + s), par ^ 1);
        const uint32_t st = sbase + lay.off_stage + s * lay.stage_bytes;
        const uint32_t fb = sbase + 8 * s;
        const int plo = s_lvln[l - 1], lo = s_lvln[l], hi = s_lvln[l + 1];
        const int alo = s_lvla[l], ahi = s_lvla[l + 1];
        const int n0 = lo & ~3, n1 = (hi + 1 + 3) & ~3;
        const int a0 = alo & ~1, a1 = (ahi + 1) & ~1;
        const int p0 = plo & ~3, p1 = (lo + 3) & ~3;
        const uint32_t nb = (uint32_t)(n1 - n0) * 4u, ab = (uint32_t)(a1 - a0) * 8u;
        const uint32_t pb = (uint32_t)(p1 - p0) * 4u;
        mbar_expect_tx(fb, nb + ab + pb);
        bulk_g2s(st, rp + n0, nb, fb);
        if (ab) bulk_g2s(st + lay.st_arcs, ga + a0, ab, fb);
        if (pb) bulk_g2s(st + lay.st_psc, gsc + p0, pb, fb);
        if (++s == S) {
          s = 0;
          par ^= 1;
        }
      }
    }
    return;
  }

  // ===== consumers =====
  float* ag = arc_grad + m.arc_base;
  const float delta = deltas ? deltas[blockIdx.x] : 1.0f;
  const int sub = tid % G;
  const int slot = tid / G;
  // lanes cooperating on one node; shuffles stay inside the group so that groups may diverge
  const unsigned gmask = (G >= 32) ? 0xffffffffu : (((1u << G) - 1u) << ((tid & 31) & ~(G - 1)));

  // top level: its own scores, and the accept seeds (shortest.cpp:49-60)
  {
    const int lo = L > 0 ? s_lvln[L - 1] : 0, hi = L > 0 ? s_lvln[L] : 0;
    for (int i = tid; i < hi - lo; i += kConsumers) s_top[i] = gsc[lo + i];
    for (int i = tid; i < 3 * lay.win_nodes; i += kConsumers) s_ng[i] = 0.0f;
    bar_named<1, kConsumers>();
    if (tid == 0 && L > 0) {
      const int32_t* acc = acc_nodes + m.acc_base;
      if (TROPICAL) {
        const int best = best_accept[blockIdx.x];
        if (best >= 0) s_ng[best - lo] += 1.0f;
      } else {
        float mx = -CUDART_INF_F;
        for (int k = 0; k < m.n_accept; k++) mx = fmaxf(mx, s_top[acc[k] - lo]);
        const float denom = expf(out_scores[blockIdx.x] - mx);
        for (int k = 0; k < m.n_accept; k++) s_ng[acc[k] - lo] += expf(s_top[acc[k] - lo] - mx) / denom;
      }
    }
    bar_named<1, kConsumers>();
  }

  int s = 0;
  uint32_t par = 0;
  int b_cur = 0; // node-gradient buffer roles rotate: cur -> zero -> prev -> cur
  const float* own = s_top; // scores of the level being processed
  for (int k = 0; k < iters; k++) {
    const int l = L - 1 - k;
    const int plo = s_lvln[l - 1], lo = s_lvln[l], hi = s_lvln[l + 1];
    const int a0 = s_lvla[l] & ~1;
    const unsigned char* st = smem + lay.off_stage + s * lay.stage_bytes;
    const uint32_t* st_rp = reinterpret_cast<const uint32_t*>(st) + (lo & 3);
    const int2* st_arc = reinterpret_cast<const int2*>(st + lay.st_arcs) - a0;
    const float* st_psc = reinterpret_cast<const float*>(st + lay.st_psc) + (plo & 3) - plo;
    const int b_prev = b_cur == 2 ? 0 : b_cur + 1;
    const int b_zero = b_prev == 2 ? 0 : b_prev + 1;
    const float* ng_cur = s_ng + b_cur * lay.win_nodes;
    float* ng_prev = s_ng + b_prev * lay.win_nodes - plo;
    float* ng_zero = s_ng + b_zero * lay.win_nodes;
    const int cnt = hi - lo;
    mbar_wait(sbase + 8 * s, par);
    if (G == 1 && !TROPICAL) {
      const uint32_t stb = sbase + lay.off_stage + s * lay.stage_bytes;
      const uint32_t R = stb + 4u * (lo & 3);
      const uint32_t A = stb + lay.st_arcs - 8u * a0;
      const uint32_t P = stb + lay.st_psc + 4u * ((plo & 3) - plo);
      const uint32_t bufs = sbase + lay.off_bufs;
      const uint32_t NGc = bufs + 4u * (b_cur * lay.win_nodes);
      const uint32_t NGp = bufs + 4u * (b_prev * lay.win_nodes - plo);
      const uint32_t OWN = smem_u32(own);
      for (int i = tid; i < cnt; i += kConsumers)
        bwd_node(i, R, A, P, NGc, OWN, NGp, delta, ag, st_arc, st_psc, ng_prev);
    } else
    for (int i0 = 0; i0 < cnt; i0 += kConsumers / G) {
      const int i = i0 + slot;
      const bool live = i < cnt;
      uint32_t r0raw = 0;
      int r0 = 0, r1 = 0;
      float g = 0.0f, sn = 0.0f;
      if (live) {
        r0raw = st_rp[i];
        r0 = (int)(r0raw & kRowMask);
        r1 = (int)(st_rp[i + 1] & kRowMask);
        g = ng_cur[i];
        sn = own[i];
      }
      if (TROPICAL) {
        // the arc the forward pass cached as its first maximum (shortest.cpp:124-127,131-134)
        float mx = -CUDART_INF_F;
        int arg = 0x7fffffff;
        for (int a = r0 + sub; a < r1; a += G) {
          const int2 rec = st_arc[a];
          const float v = st_psc[rec.x] + __int_as_float(rec.y);
          if (v > mx) {
            mx = v;
            arg = a;
          }
        }
        if (G > 1) {
#pragma unroll
          for (int o = G / 2; o > 0; o >>= 1) {
            const float om = __shfl_xor_sync(gmask, mx, o);
            const int oa = __shfl_xor_sync(gmask, arg, o);
            if (om > mx || (om == mx && oa < arg)) {
              mx = om;
              arg = oa;
            }
          }
        }
        const bool start_wins = (r0raw & kStartBit) && 0.0f > mx;
        for (int a = r0 + sub; a < r1; a += G) {
          const bool hit = (a == arg) && !start_wins;
          ag[a] = (hit ? g : 0.0f) * delta;
          if (hit) atomicAdd(&ng_prev[st_arc[a].x], g);
        }
      } else {
        const bool exact = !(fabsf(sn) < CUDART_INF_F); // +-inf / NaN score: reference formula verbatim
        float mx = 0.0f;
        if (exact) {
          mx = -CUDART_INF_F;
#pragma unroll 1
          for (int a = r0; a < r1; a++) {
            const int2 rec = st_arc[a];
            mx = fmaxf(mx, st_psc[rec.x] + __int_as_float(rec.y));
          }
          if (r0raw & kStartBit) mx = fmaxf(mx, 0.0f);
        }
        if (false) {
        } else {
#pragma unroll 1
          for (int a = r0 + sub; a < r1; a += G) {
            const int2 rec = st_arc[a];
            const float cur = arc_grad_log(g, st_psc[rec.x] + __int_as_float(rec.y), sn, mx, exact);
            atomicAdd(&ng_prev[rec.x], cur);
            ag[a] = cur * delta;
          }
        }
      }
    }
    for (int i = tid; i < lay.win_nodes; i += kConsumers) ng_zero[i] = 0.0f;
    bar_named<1, kConsumers>();
    // the previous iteration's stage held this level's own scores: free it now,
    // and keep this iteration's score window (level l-1) as the next "own"
    if (tid == 0 && k > 0) mbar_arrive(sbase + 8 * (kMaxStages + (s == 0 ? S - 1 : s - 1)));
    own = reinterpret_cast<const float*>(st + lay.st_psc) + (plo & 3);
    b_cur = b_prev;
    if (++s == S) {
      s = 0;
      par ^= 1;
    }
  }
}


/* ------------------------------------------------------------------ */
/* criterion backward: shortestDistanceGrad + compose gradFunc fused   */
/* ------------------------------------------------------------------ */


/* rows the unrolled steady path does not cover (non-finite score, > 3 in-arcs): reference
 * formula verbatim (shortest.cpp:62-80); arc gradients go to the shared arc buffer */
__device__ __noinline__ float fused_row_any(float g, float sn, int e0, int e1, uint32_t Ae, uint32_t P, uint32_t CUR) {
  const bool exact = !(fabsf(sn) < CUDART_INF_F);
  float mx = 0.0f, acc = 0.0f;
  if (exact) {
    mx = -CUDART_INF_F;
#pragma unroll 1
    for (int e = e0; e < e1; e++) {
      const int2 rec = lds_v2_u32(Ae + 8u * e);
      mx = fmaxf(mx, lds_f32(P + 4u * rec.x) + __int_as_float(rec.y));
    }
  }
#pragma unroll 1
  for (int e = e0; e < e1; e++) {
    const int2 rec = lds_v2_u32(Ae + 8u * e);
    const float cur = arc_grad_log(g, lds_f32(P + 4u * rec.x) + __int_as_float(rec.y), sn, mx, exact);
    sts_f32(CUR + 4u * e, cur);
    acc += cur;
  }
  return acc;
}

/* one level of the fused backward outside the fast path: (a) steady but the graph has more
 * nodes than consumer threads -- same two phases, several nodes per thread; (b) not steady
 * (the cone at both ends of the lattice) -- zero the accumulator, scatter with shared atomics,
 * emission gradients through the per-arc provenance */
__device__ __noinline__ void fused_level_slow(
    bool steady, int tid, int N1, int cnt, int alo, int win_nodes, uint32_t R, uint32_t A, uint32_t P,
    uint32_t NGc, uint32_t NGp, uint32_t NGp0, uint32_t OWN, uint32_t CUR, float delta, float* gem,
    float* gem_l, const int2* ggi, const int* t_inptr, const int* t_label, const int* t_outptr,
    const int* t_outent) {
  constexpr int kConsumers = 32 * consumer_warps(1);
  if (steady) {
    const uint32_t Ae = A + 8u * alo;
    for (int i = tid; i < N1; i += kConsumers) {
      const int e0 = t_inptr[i], e1 = t_inptr[i + 1];
      const float acc = fused_row_any(lds_f32(NGc + 4u * i), lds_f32(OWN + 4u * i), e0, e1, Ae, P, CUR);
      if (e1 > e0) atomicAdd(&gem_l[t_label[i]], acc * delta);
    }
    bar_named<1, kConsumers>();
    for (int u = tid; u < N1; u += kConsumers) {
      float sum = 0.0f;
#pragma unroll 1
      for (int q = t_outptr[u]; q < t_outptr[u + 1]; q++) sum += lds_f32(CUR + 4u * t_outent[q]);
      sts_f32(NGp0 + 4u * u, sum);
    }
    bar_named<1, kConsumers>();
    return;
  }
  for (int i = tid; i < win_nodes; i += kConsumers) sts_f32(NGp0 + 4u * i, 0.0f);
  bar_named<1, kConsumers>();
  for (int i = tid; i < cnt; i += kConsumers) {
    const uint32_t r0raw = lds_u32(R + 4u * i);
    const int r0 = (int)(r0raw & kRowMask);
    const int r1 = (int)(lds_u32(R + 4u * i + 4u) & kRowMask);
    const float g = lds_f32(NGc + 4u * i);
    const float sn = lds_f32(OWN + 4u * i);
    const bool exact = !(fabsf(sn) < CUDART_INF_F) || (r0raw & kStartBit);
    float mx = 0.0f;
    if (exact) {
      mx = -CUDART_INF_F;
#pragma unroll 1
      for (int a = r0; a < r1; a++) {
        const int2 rec = lds_v2_u32(A + 8u * a);
        mx = fmaxf(mx, lds_f32(P + 4u * rec.x) + __int_as_float(rec.y));
      }
      if (r0raw & kStartBit) mx = fmaxf(mx, 0.0f);
    }
#pragma unroll 1
    for (int a = r0; a < r1; a++) {
      const int2 rec = lds_v2_u32(A + 8u * a);
      const float v = lds_f32(P + 4u * rec.x) + __int_as_float(rec.y);
      const float cur = arc_grad_log(g, v, sn, mx, exact);
      red_shared_add(NGp + 4u * rec.x, cur);
      atomicAdd(&gem[ggi[a].y], cur * delta);
    }
  }
  bar_named<1, kConsumers>();
}

/*
 * gtnb_ctc_loss only needs d loss / d emissions, never the lattice's own arc gradients.
 * This kernel is sd_backward_staged<false, 1> with compose's gradFunc (compose.cpp:496-518)
 * folded in: the arc gradients of a node are summed in registers and leave the SM as ONE
 * red.global per node, aimed at the emission the node's in-arcs came from; arc_grad is
 * never written and compose_grad_kernel never runs.
 *
 * It also removes the float shared-memory atomics of the generic kernel (fp32 atomicAdd
 * on shared memory is a CAS loop on sm_90a: SASS ATOMS.CAST.SPIN): in the steady state
 * of a frame-synchronous lattice (every graph node alive in frames l and l-1, every
 * label matchable) level l IS the graph operand, arc k of the level is in-entry k of the
 * graph, so the per-source sums are gathered through the graph's out-arc lists kept in
 * shared memory: phase 1 (thread per destination) writes the arc gradients to a shared
 * arc buffer, phase 2 (thread per source) sums its out-arcs.  Frames outside the steady
 * state (the cone at both ends of a CTC lattice) take the generic atomics path.
 */
__global__ void __launch_bounds__(32 * consumer_warps(1) + 32) sd_backward_fused(
    const GraphMeta* __restrict__ meta,
    const int32_t* __restrict__ lvl_node_ptr,
    const int32_t* __restrict__ lvl_arc_ptr,
    const uint32_t* __restrict__ row_ptr,
    const int2* __restrict__ arcs,
    const int2* __restrict__ gi,
    const int32_t* __restrict__ acc_nodes,
    const float* __restrict__ scores,
    const float* __restrict__ out_scores,
    const float* __restrict__ deltas,
    const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ sg_in_src,
    const int32_t* __restrict__ sg_in_label,
    float* __restrict__ grad_emis,
    long long grad_stride,
    int C,
    const Layout lay) {
  GTNB_DYNAMIC_SMEM_128(unsigned char, smem);
  constexpr int kConsumers = 32 * consumer_warps(1);
  constexpr int kStagedThreads = kConsumers + 32;
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x;
  const int S = 1 << lay.log2_stages;
  const uint32_t sbase = smem_u32(smem);
  int* s_lvln = reinterpret_cast<int*>(smem + lay.off_lvln);
  int* s_lvla = reinterpret_cast<int*>(smem + lay.off_lvla);
  float* s_ng = reinterpret_cast<float*>(smem + lay.off_bufs); // [0], [1]: node gradients (ping-pong)
  float* s_top = s_ng + 3 * lay.win_nodes;
  // graph-operand tables
  int* t_inptr = reinterpret_cast<int*>(smem + lay.off_tab); // [N1 + 1]
  int* t_label = t_inptr + lay.tab_nodes + 1; // [N1]   matched label of the node's in-arcs
  int* t_outptr = t_label + lay.tab_nodes; // [N1 + 1]
  int* t_outent = t_outptr + lay.tab_nodes + 1; // [A1]   in-entries grouped by source node
  float* s_cur = reinterpret_cast<float*>(t_outent + lay.tab_arcs); // [A1]   arc gradients of the level

  const int L = m.L;
  for (int i = tid; i <= L; i += kStagedThreads) {
    s_lvln[i] = lvl_node_ptr[m.lvl_base + i];
    s_lvla[i] = lvl_arc_ptr[m.lvl_base + i];
  }
  if (tid == 0) {
    for (int s = 0; s < S; s++) {
      mbar_init(sbase + 8 * s, 1);
      mbar_init(sbase + 8 * (kMaxStages + s), consumer_warps(1)); // every consumer warp releases
    }
    mbar_init_fence();
  }
  __syncthreads();

  const float* gsc = scores + m.node_base;
  const int iters = L - 1;

  if (tid >= kConsumers) {
    if (tid == kConsumers) {
      const uint32_t* rp = row_ptr + m.node_base;
      const int2* ga = arcs + m.arc_base;
      int s = 0;
      uint32_t par = 0;
#pragma unroll 1
      for (int k = 0; k < iters; k++) {
        const int l = L - 1 - k;
        if (k >= S) mbar_wait_sleep(sbase + 8 * (kMaxStages + s), par ^ 1);
        const uint32_t st = sbase + lay.off_stage + s * lay.stage_bytes;
        const uint32_t fb = sbase + 8 * s;
        const int plo = s_lvln[l - 1], lo = s_lvln[l], hi = s_lvln[l + 1];
        const int alo = s_lvla[l], ahi = s_lvla[l + 1];
        const int n0 = lo & ~3, n1 = (hi + 1 + 3) & ~3;
        const int a0 = alo & ~1, a1 = (ahi + 1) & ~1;
        const int p0 = plo & ~3, p1 = (lo + 3) & ~3;
        const uint32_t nb = (uint32_t)(n1 - n0) * 4u, ab = (uint32_t)(a1 - a0) * 8u;
        const uint32_t pb = (uint32_t)(p1 - p0) * 4u;
        mbar_expect_tx(fb, nb + ab + pb);
        bulk_g2s(st, rp + n0, nb, fb);
        if (ab) bulk_g2s(st + lay.st_arcs, ga + a0, ab, fb);
        if (pb) bulk_g2s(st + lay.st_psc, gsc + p0, pb, fb);
        if (++s == S) {
          s = 0;
          par ^= 1;
        }
      }
    }
    return;
  }

  // ===== consumers =====
  const float delta = deltas ? deltas[blockIdx.x] : 1.0f;
  float* gem = grad_emis + (long long)blockIdx.x * grad_stride;
  const int2* ggi = gi + m.arc_base;
  const int N1 = m.sg_N, A1 = m.sg_A;
  const bool steady_ok = m.sg_all_valid != 0;

  // graph tables: in-arc pointers, the (uniform) label of each node's in-arcs, out-arc lists
  {
    const int32_t* ip = sg_in_ptr + m.sg_node_base;
    const int32_t* is = sg_in_src + m.sg_arc_base;
    const int32_t* il = sg_in_label + m.sg_arc_base;
    int* t_src = reinterpret_cast<int*>(s_cur); // borrowed until the tables are built
    for (int i = tid; i <= N1; i += kConsumers) t_inptr[i] = ip[i];
    for (int e = tid; e < A1; e += kConsumers) t_src[e] = is[e];
    bar_named<1, kConsumers>();
    for (int u = tid; u < N1; u += kConsumers) {
      t_label[u] = (t_inptr[u] < t_inptr[u + 1]) ? il[t_inptr[u]] : 0;
      int c = 0;
      for (int e = 0; e < A1; e++) c += (t_src[e] == u);
      t_outptr[u + 1] = c;
    }
    bar_named<1, kConsumers>();
    if (tid == 0) {
      t_outptr[0] = 0;
      for (int u = 0; u < N1; u++) t_outptr[u + 1] += t_outptr[u];
    }
    bar_named<1, kConsumers>();
    for (int u = tid; u < N1; u += kConsumers) {
      int pos = t_outptr[u];
      for (int e = 0; e < A1; e++)
        if (t_src[e] == u) t_outent[pos++] = e;
    }
    bar_named<1, kConsumers>();
  }

  // top level: its own scores, and the accept seeds (shortest.cpp:49-60)
  {
    const int lo = L > 0 ? s_lvln[L - 1] : 0, hi = L > 0 ? s_lvln[L] : 0;
    for (int i = tid; i < hi - lo; i += kConsumers) s_top[i] = gsc[lo + i];
    for (int i = tid; i < 2 * lay.win_nodes; i += kConsumers) s_ng[i] = 0.0f;
    bar_named<1, kConsumers>();
    if (tid == 0 && L > 0) {
      const int32_t* acc = acc_nodes + m.acc_base;
      float mx = -CUDART_INF_F;
      for (int k = 0; k < m.n_accept; k++) mx = fmaxf(mx, s_top[acc[k] - lo]);
      const float denom = expf(out_scores[blockIdx.x] - mx);
      for (int k = 0; k < m.n_accept; k++) s_ng[acc[k] - lo] += expf(s_top[acc[k] - lo] - mx) / denom;
    }
    bar_named<1, kConsumers>();
  }

  // per-thread constants of "my" graph node (thread u <-> node u while N1 <= kConsumers)
  const bool one_to_one = N1 <= kConsumers;
  int my_e0 = 0, my_e1 = 0, my_lab = 0, my_o0 = 0, my_o1 = 0;
  if (tid < N1) {
    my_e0 = t_inptr[tid];
    my_e1 = t_inptr[tid + 1];
    my_lab = t_label[tid];
    my_o0 = t_outptr[tid];
    my_o1 = t_outptr[tid + 1];
  }
  const int my_oe0 = (my_o1 - my_o0 > 0) ? t_outent[my_o0] : 0;
  const int my_oe1 = (my_o1 - my_o0 > 1) ? t_outent[my_o0 + 1] : 0;
  const int my_oe2 = (my_o1 - my_o0 > 2) ? t_outent[my_o0 + 2] : 0;
  float g_reg = 0.0f;
  bool g_in_reg = false;

  int s = 0;
  uint32_t par = 0;
  int b_cur = 0;
  const float* own = s_top;
  auto is_steady = [&](int l) {
    return steady_ok && l >= 1 && (s_lvln[l + 1] - s_lvln[l]) == N1 && (s_lvln[l] - s_lvln[l - 1]) == N1;
  };
  for (int k = 0; k < iters; k++) {
    const int l = L - 1 - k;
    const int plo = s_lvln[l - 1], lo = s_lvln[l], hi = s_lvln[l + 1];
    const int alo = s_lvla[l];
    const int a0 = alo & ~1;
    const unsigned char* st = smem + lay.off_stage + s * lay.stage_bytes;
    const int2* st_arc = reinterpret_cast<const int2*>(st + lay.st_arcs) - a0;
    const float* st_psc = reinterpret_cast<const float*>(st + lay.st_psc) + (plo & 3) - plo;
    const int b_prev = b_cur ^ 1;
    const int cnt = hi - lo;
    const uint32_t stb = sbase + lay.off_stage + s * lay.stage_bytes;
    const uint32_t R = stb + 4u * (lo & 3);
    const uint32_t A = stb + lay.st_arcs - 8u * a0;
    const uint32_t P = stb + lay.st_psc + 4u * ((plo & 3) - plo);
    const uint32_t bufs = sbase + lay.off_bufs;
    const uint32_t NGc = bufs + 4u * (b_cur * lay.win_nodes);
    const uint32_t NGp = bufs + 4u * (b_prev * lay.win_nodes - plo);
    const uint32_t NGp0 = bufs + 4u * (b_prev * lay.win_nodes);
    const uint32_t OWN = smem_u32(own);
    const bool steady = is_steady(l);
    const bool next_steady = (k + 1 < iters) && is_steady(l - 1);
    float* gem_l = gem + (long long)(l - 1) * C;
    // arc-gradient buffer of this level (double-buffered so that the gather of level l can
    // still be running in other warps while level l-1 is being written)
    const uint32_t CUR = smem_u32(s_cur) + 4u * ((k & 1) * lay.tab_arcs);
    mbar_wait(sbase + 8 * s, par);
    if (steady && one_to_one) {
      const uint32_t Ae = A + 8u * alo; // arc record of in-entry 0
      if (tid < N1) {
        // phase 1: destination node `tid`; arc e of the level == in-entry e of the graph
        const float g = g_in_reg ? g_reg : lds_f32(NGc + 4u * tid);
        const float sn = lds_f32(OWN + 4u * tid);
        const int deg = my_e1 - my_e0;
        float acc = 0.0f;
        if (!(fabsf(sn) < CUDART_INF_F) || deg > 3) {
          acc = fused_row_any(g, sn, my_e0, my_e1, Ae, P, CUR);
        } else {
          const uint32_t ae = Ae + 8u * my_e0, ce = CUR + 4u * my_e0;
          if (deg > 0) {
            const int2 rec = lds_v2_u32(ae);
            const float cur = g * fexp(lds_f32(P + 4u * rec.x) + __int_as_float(rec.y) - sn);
            sts_f32(ce, cur);
            acc += cur;
          }
          if (deg > 1) {
            const int2 rec = lds_v2_u32(ae + 8u);
            const float cur = g * fexp(lds_f32(P + 4u * rec.x) + __int_as_float(rec.y) - sn);
            sts_f32(ce + 4u, cur);
            acc += cur;
          }
          if (deg > 2) {
            const int2 rec = lds_v2_u32(ae + 16u);
            const float cur = g * fexp(lds_f32(P + 4u * rec.x) + __int_as_float(rec.y) - sn);
            sts_f32(ce + 8u, cur);
            acc += cur;
          }
        }
        if (deg > 0) atomicAdd(&gem_l[my_lab], acc * delta);
      }
      bar_named<1, kConsumers>();
      if (tid < N1) {
        // phase 2: source node `tid` gathers its out-arcs (no atomics, fixed order)
        float sum = 0.0f;
        const int od = my_o1 - my_o0;
        if (od > 0) sum += lds_f32(CUR + 4u * my_oe0);
        if (od > 1) sum += lds_f32(CUR + 4u * my_oe1);
        if (od > 2) sum += lds_f32(CUR + 4u * my_oe2);
#pragma unroll 1
        for (int q = my_o0 + 3; q < my_o1; q++) sum += lds_f32(CUR + 4u * t_outent[q]);
        g_reg = sum;
        g_in_reg = true;
        if (!next_steady) sts_f32(NGp0 + 4u * tid, sum);
      }
      if (!next_steady) bar_named<1, kConsumers>();
    } else {
      g_in_reg = false;
      fused_level_slow(
          steady, tid, N1, cnt, alo, lay.win_nodes, R, A, P, NGc, NGp, NGp0, OWN, CUR, delta, gem, gem_l,
          ggi, t_inptr, t_label, t_outptr, t_outent);
    }
    // the previous iteration's stage held this level's own scores: every warp is done with it
    __syncwarp();
    if ((tid & 31) == 0 && k > 0) mbar_arrive(sbase + 8 * (kMaxStages + (s == 0 ? S - 1 : s - 1)));
    own = reinterpret_cast<const float*>(st + lay.st_psc) + (plo & 3);
    b_cur = b_prev;
    if (++s == S) {
      s = 0;
      par ^= 1;
    }
  }
}

struct StagedPlan {
  bool ok;
  int G, max_L;
  Layout fwd, bwd;
};

/* the B graphs' descriptors; max_lvl_nodes / max_lvl_arcs: bounds on a level's nodes and arcs over the batch */
StagedPlan plan(const GraphMeta* meta, int B, int max_lvl_nodes, int max_lvl_arcs) {
  StagedPlan p;
  p.ok = false;
  int max_L = 0;
  long long sumA = 0, sumN = 0;
  for (int b = 0; b < B; b++) {
    max_L = std::max(max_L, meta[b].L);
    sumA += meta[b].sg_A;
    sumN += meta[b].sg_N;
  }
  if (max_L + 1 > kMaxLevelsInSmem) return p;
  p.max_L = max_L;
  const double deg = sumN ? (double)sumA / (double)sumN : 0.0;
  p.G = deg <= 4.0 ? 1 : (deg <= 16.0 ? 4 : (deg <= 48.0 ? 16 : 32));
  const int budget = 200 * 1024;
  for (int ls = 3; ls >= 1; ls--) {
    Layout f = make_layout(max_lvl_nodes, max_lvl_arcs, max_L, ls, 2, false);
    Layout bw = make_layout(max_lvl_nodes, max_lvl_arcs, max_L, ls, 4, true);
    // keep two CTAs per SM resident when the graph is small enough
    const int cap = (bw.total <= 100 * 1024 || ls == 1) ? budget : 100 * 1024;
    if (bw.total <= cap && f.total <= cap) {
      p.ok = true;
      p.fwd = f;
      p.bwd = bw;
      return p;
    }
  }
  return p;
}

/* sd_backward_fused's layout: the backward's, then the graph operands' tables; false when it exceeds the budget */
bool fused_layout(Layout& lay, int max_lvl_nodes, int max_lvl_arcs) {
  lay.tab_nodes = max_lvl_nodes;
  lay.tab_arcs = max_lvl_arcs;
  lay.off_tab = (lay.total + 15) / 16 * 16;
  lay.total = lay.off_tab + 4 * (3 * lay.tab_nodes + 2 + 3 * lay.tab_arcs) + 16;
  return lay.total <= 200 * 1024;
}

using StagedForward = void (*)(const GraphMeta*, const int32_t*, const int32_t*, const uint32_t*, const int2*,
                               const int32_t*, float*, int32_t*, float*, int32_t*, const Layout);
using StagedBackward = void (*)(const GraphMeta*, const int32_t*, const int32_t*, const uint32_t*, const int2*,
                                const int32_t*, const float*, const float*, const int32_t*, const float*, float*,
                                const Layout);

/* the instantiations for mode (MODE_*) and G lanes per node (StagedPlan::G) */
template <int MODE>
StagedForward sd_forward_staged_for(int G) {
  return G == 1 ? sd_forward_staged<MODE, 1>
                : G == 4 ? sd_forward_staged<MODE, 4> : G == 16 ? sd_forward_staged<MODE, 16> : sd_forward_staged<MODE, 32>;
}
StagedForward sd_forward_staged_kernel_for(int mode, int G) {
  return mode == MODE_LOG ? sd_forward_staged_for<MODE_LOG>(G)
                          : mode == MODE_TROPICAL ? sd_forward_staged_for<MODE_TROPICAL>(G) : sd_forward_staged_for<MODE_PATH>(G);
}
template <bool TROPICAL>
StagedBackward sd_backward_staged_for(int G) {
  return G == 1 ? sd_backward_staged<TROPICAL, 1>
                : G == 4 ? sd_backward_staged<TROPICAL, 4>
                         : G == 16 ? sd_backward_staged<TROPICAL, 16> : sd_backward_staged<TROPICAL, 32>;
}
StagedBackward sd_backward_staged_kernel_for(bool tropical, int G) {
  return tropical ? sd_backward_staged_for<true>(G) : sd_backward_staged_for<false>(G);
}

#ifndef GTNB_HOST_EMU

StagedPlan plan(const gtnb_lattice* lat) {
  if (!lat->composed || !lat->level_local) return StagedPlan{};
  return plan(lat->meta_h.data(), lat->B, lat->max_lvl_nodes, lat->max_lvl_arcs);
}

template <typename K>
int set_smem(gtnb_ctx* ctx, K kernel, int bytes) {
  if (bytes > kMaxDynamicSmem) return GTNB_ERR_UNSUPPORTED;
  return ensure_max_smem(ctx, (const void*)kernel);
}

#endif // GTNB_HOST_EMU

} // namespace

#ifndef GTNB_HOST_EMU

bool staged_supported(const gtnb_lattice* lat) {
  return plan(lat).ok;
}

int launch_forward_staged(gtnb_ctx* ctx, gtnb_lattice* lat, int mode) {
  const StagedPlan p = plan(lat);
  if (!p.ok) return GTNB_ERR_UNSUPPORTED;
  const StagedForward kernel = sd_forward_staged_kernel_for(mode, p.G);
  int rc = set_smem(ctx, kernel, p.fwd.total);
  if (rc) return rc;
  GTNB_LAUNCH(ctx, "sd_forward",
              kernel<<<lat->B, 32 * consumer_warps(p.G) + 32, p.fwd.total, ctx->stream>>>(
                  lat->meta, lat->lvl_node_ptr, lat->lvl_arc_ptr, lat->row_ptr, lat->arcs, lat->acc_nodes,
                  lat->scores, lat->back_ptr, lat->out_scores, lat->best_accept, p.fwd));
  return GTNB_OK;
}

/* shortestDistanceGrad + compose gradFunc in one kernel (log semiring, emission gradients
 * only).  GTNB_ERR_UNSUPPORTED when the lattice does not qualify: the caller then runs
 * launch_backward + launch_compose_grad. */
int launch_backward_fused(
    gtnb_ctx* ctx, gtnb_lattice* lat, const float* deltas_dev, float* grad_emis, int64_t grad_stride) {
  StagedPlan p = plan(lat);
  if (!ctx->use_staged || !p.ok || p.G != 1 || !lat->gi) return GTNB_ERR_UNSUPPORTED;
  for (int b = 0; b < lat->B; b++)
    if (!lat->meta_h[b].sg_uniform) return GTNB_ERR_UNSUPPORTED;
  Layout lay = p.bwd;
  if (!fused_layout(lay, lat->max_lvl_nodes, lat->max_lvl_arcs)) return GTNB_ERR_UNSUPPORTED;
  int rc = set_smem(ctx, sd_backward_fused, lay.total);
  if (rc) return rc;
  GTNB_LAUNCH(ctx, "sd_backward_fused",
              sd_backward_fused<<<lat->B, 32 * consumer_warps(1) + 32, lay.total, ctx->stream>>>(
                  lat->meta, lat->lvl_node_ptr, lat->lvl_arc_ptr, lat->row_ptr, lat->arcs, lat->gi,
                  lat->acc_nodes, lat->scores, lat->out_scores, deltas_dev, lat->sg_in_ptr,
                  lat->sg_in_src, lat->sg_in_label, grad_emis, (long long)grad_stride, lat->C, lay));
  return GTNB_OK;
}

int launch_backward_staged(gtnb_ctx* ctx, gtnb_lattice* lat, int tropical, const float* deltas_dev) {
  const StagedPlan p = plan(lat);
  if (!p.ok) return GTNB_ERR_UNSUPPORTED;
  const StagedBackward kernel = sd_backward_staged_kernel_for(tropical != 0, p.G);
  int rc = set_smem(ctx, kernel, p.bwd.total);
  if (rc) return rc;
  GTNB_LAUNCH(ctx, "sd_backward",
              kernel<<<lat->B, 32 * consumer_warps(p.G) + 32, p.bwd.total, ctx->stream>>>(
                  lat->meta, lat->lvl_node_ptr, lat->lvl_arc_ptr, lat->row_ptr, lat->arcs, lat->acc_nodes,
                  lat->scores, lat->out_scores, lat->best_accept, deltas_dev, lat->arc_grad, p.bwd));
  return GTNB_OK;
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
