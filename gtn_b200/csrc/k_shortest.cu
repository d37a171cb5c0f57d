/*
 * k_shortest.cu -- shortest-distance dynamic programs over a packed batch of
 * levelised CSR-by-destination graphs; one persistent CTA per graph walks its
 * levels, so the T-serial dependency never leaves the SM.
 *
 *   sd_forward_*   detail::shortestDistance   (shortest.cpp:86-188)
 *                  detail::shortestPath's relaxation (shortest.cpp:190-238) in MODE_PATH
 *   sd_backward_*  shortestDistanceGrad       (shortest.cpp:33-82)
 *   traceback      back-pointer chase         (shortest.cpp:240-245)
 *
 * Two families:
 *   *_generic  any DAG; node scores gathered from HBM/L2 (ld.global.cg).
 *   *_staged   "level-local" graphs (every arc goes level l-1 -> l: all composed
 *              lattices): the arc block of each level is staged into shared
 *              memory by cp.async.bulk (TMA 1-D bulk copy, mbarrier-tracked,
 *              multi-stage ring) and the frontier scores live in shared memory.
 *
 * Arithmetic mirrors the reference: fp32, max taken in in-arc order with strict
 * '>' (first maximum wins), log-sum-exp as max + log1p(sum(exp(s-max)) - 1) with
 * the running sum started at -1 (shortest.cpp:102-114).  score + weight is a
 * single fp32 add (no FMA can be contracted into it: there is no multiply).
 */
#include <cstdlib>

#include "gtnb_ptx.h"

namespace gtnb {

namespace {

constexpr int kThreads = 256;

/* getScore (shortest.cpp:102-114) given max and sum already reduced */
__device__ __forceinline__ float finish_score(int count, float mx, float sum_m1, bool tropical) {
  if (count == 0) return neg_inf();
  if (tropical || mx == CUDART_INF_F || mx == -CUDART_INF_F) return mx;
  return mx + log1pf(sum_m1);
}

/* ------------------------------------------------------------------ */
/* generic forward                                                     */
/* ------------------------------------------------------------------ */

template <int MODE>
__global__ void __launch_bounds__(kThreads) sd_forward_generic(
    const GraphMeta* __restrict__ meta,
    const int32_t* __restrict__ lvl_node_ptr,
    const uint32_t* __restrict__ row_ptr,
    const int2* __restrict__ arcs,
    const int32_t* __restrict__ relax_rank, // MODE_PATH only, nullable
    const int32_t* __restrict__ acc_nodes,
    float* __restrict__ scores,
    int32_t* __restrict__ back_ptr, // MODE_PATH only
    float* __restrict__ out_scores,
    int32_t* __restrict__ best_accept) {
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x;
  if (m.status != GTNB_OK) {
    if (tid == 0) {
      out_scores[blockIdx.x] = CUDART_NAN_F;
      best_accept[blockIdx.x] = -1;
    }
    return;
  }
  const int32_t* lp = lvl_node_ptr + m.lvl_base;
  const uint32_t* rp = row_ptr + m.node_base;
  const int2* ar = arcs + m.arc_base;
  const int32_t* rr = relax_rank ? relax_rank + m.arc_base : nullptr;
  float* sc = scores + m.node_base;
  int32_t* bp = (MODE == MODE_PATH) ? back_ptr + m.node_base : nullptr;

  // nodes the Kahn sweep never reaches keep the vector's initial value:
  // 0.0f in shortestDistance (shortest.cpp:89), -inf in shortestPath (:196)
  const int n_sched = m.L > 0 ? lp[m.L] : 0;
  for (int n = n_sched + tid; n < m.N; n += kThreads) {
    sc[n] = (MODE == MODE_PATH) ? neg_inf() : 0.0f;
    if (MODE == MODE_PATH) bp[n] = -1;
  }

  for (int l = 0; l < m.L; l++) {
    const int lo = lp[l], hi = lp[l + 1];
    for (int n = lo + tid; n < hi; n += kThreads) {
      const uint32_t r0raw = rp[n];
      const int r0 = (int)(r0raw & kRowMask);
      const int r1 = (int)(rp[n + 1] & kRowMask);
      const bool is_start = (r0raw & kStartBit) != 0;
      if (MODE == MODE_PATH) {
        // shortestPath: start nodes begin at 0 with no back-pointer and every
        // relaxation needs a strictly greater score (shortest.cpp:202-218);
        // candidates arrive in the order the reference relaxes them.
        float best = is_start ? 0.0f : neg_inf();
        int barc = -1, brank = -1;
        for (int a = r0; a < r1; a++) {
          const float v = __ldcg(&sc[ar[a].x]) + __int_as_float(ar[a].y);
          const int rk = rr ? rr[a] : a;
          if (v > best || (v == best && barc >= 0 && rk < brank)) {
            best = v;
            barc = a;
            brank = rk;
          }
        }
        sc[n] = best;
        bp[n] = barc;
      } else {
        float mx = neg_inf();
        for (int a = r0; a < r1; a++) {
          const float v = __ldcg(&sc[ar[a].x]) + __int_as_float(ar[a].y);
          if (v > mx) mx = v;
        }
        if (is_start && 0.0f > mx) mx = 0.0f;
        const int count = (r1 - r0) + (is_start ? 1 : 0);
        float sum = -1.0f;
        if (MODE == MODE_LOG && count > 0 && mx != CUDART_INF_F && mx != -CUDART_INF_F) {
          for (int a = r0; a < r1; a++) sum += expf((__ldcg(&sc[ar[a].x]) + __int_as_float(ar[a].y)) - mx);
          if (is_start) sum += expf(0.0f - mx);
        }
        sc[n] = finish_score(count, mx, sum, MODE != MODE_LOG);
      }
    }
    __syncthreads();
  }
  if (m.L == 0) __syncthreads();

  // reduce over the accept nodes in g.accept() order (shortest.cpp:147-159 / :226-237)
  if (tid == 0) {
    const int32_t* acc = acc_nodes + m.acc_base;
    float mx = neg_inf();
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
      float sum = -1.0f;
      if (m.n_accept > 0 && mx != CUDART_INF_F && mx != -CUDART_INF_F)
        for (int k = 0; k < m.n_accept; k++) sum += expf(__ldcg(&sc[acc[k]]) - mx);
      out = finish_score(m.n_accept, mx, sum, false);
    } else {
      out = (m.n_accept == 0) ? neg_inf() : mx;
    }
    out_scores[blockIdx.x] = out;
    best_accept[blockIdx.x] = best;
  }
}

/* ------------------------------------------------------------------ */
/* generic backward                                                    */
/* ------------------------------------------------------------------ */

template <bool TROPICAL>
__global__ void __launch_bounds__(kThreads) sd_backward_generic(
    const GraphMeta* __restrict__ meta,
    const int32_t* __restrict__ lvl_node_ptr,
    const int32_t* __restrict__ blvl_ptr, // nullable
    const int32_t* __restrict__ bnodes,
    const uint32_t* __restrict__ row_ptr,
    const int2* __restrict__ arcs,
    const int32_t* __restrict__ acc_nodes,
    const float* __restrict__ scores,
    const float* __restrict__ out_scores,
    const int32_t* __restrict__ best_accept,
    const float* __restrict__ deltas, // nullable
    float* __restrict__ node_grad,
    float* __restrict__ arc_grad) {
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x;
  if (m.status != GTNB_OK) return;
  const uint32_t* rp = row_ptr + m.node_base;
  const int2* ar = arcs + m.arc_base;
  const float* sc = scores + m.node_base;
  float* ng = node_grad + m.node_base;
  float* ag = arc_grad + m.arc_base;
  const float delta = deltas ? deltas[blockIdx.x] : 1.0f;

  for (int n = tid; n < m.N; n += kThreads) ng[n] = 0.0f;
  for (int a = tid; a < m.A; a += kThreads) ag[a] = 0.0f;
  __syncthreads();

  // seed the accept nodes (shortest.cpp:49-60)
  if (tid == 0) {
    const int32_t* acc = acc_nodes + m.acc_base;
    if (TROPICAL) {
      const int best = best_accept[blockIdx.x];
      if (best >= 0) ng[best] += 1.0f;
    } else {
      float mx = neg_inf();
      for (int k = 0; k < m.n_accept; k++) {
        const float v = sc[acc[k]];
        if (v > mx) mx = v;
      }
      const float denom = expf(out_scores[blockIdx.x] - mx);
      for (int k = 0; k < m.n_accept; k++) ng[acc[k]] += expf(sc[acc[k]] - mx) / denom;
    }
  }
  __syncthreads();

  const bool listed = (m.LB >= 0);
  const int nlev = listed ? m.LB : m.L;
  const int32_t* lp = lvl_node_ptr + m.lvl_base;
  const int32_t* blp = listed ? blvl_ptr + m.blvl_base : nullptr;
  const int32_t* bn = listed ? bnodes + m.bnode_base : nullptr;
  for (int k = 0; k < nlev; k++) {
    int lo, hi;
    if (listed) {
      lo = blp[k];
      hi = blp[k + 1];
    } else {
      lo = lp[m.L - 1 - k];
      hi = lp[m.L - k];
    }
    for (int i = lo + tid; i < hi; i += kThreads) {
      const int n = listed ? bn[i] : i;
      const uint32_t r0raw = rp[n];
      const int r0 = (int)(r0raw & kRowMask);
      const int r1 = (int)(rp[n + 1] & kRowMask);
      if (r1 == r0) continue;
      // the node's gradient is complete: every successor sits in an earlier
      // backward level.  Read it through L2 (peer threads added to it).
      const float g = __ldcg(&ng[n]);
      if (TROPICAL) {
        // first maximum in in-arc order == maxArcIdxCache[n] (shortest.cpp:124-127,131-134)
        float mx = neg_inf();
        int arg = -1;
        for (int a = r0; a < r1; a++) {
          const float v = sc[ar[a].x] + __int_as_float(ar[a].y);
          if (v > mx) {
            mx = v;
            arg = a;
          }
        }
        if ((r0raw & kStartBit) && 0.0f > mx) arg = -1;
        if (arg >= 0) {
          atomicAdd(&ng[ar[arg].x], g);
          ag[arg] = g * delta;
        }
      } else {
        float mx = neg_inf();
        for (int a = r0; a < r1; a++) {
          const float v = sc[ar[a].x] + __int_as_float(ar[a].y);
          if (v > mx) mx = v;
        }
        if ((r0raw & kStartBit) && 0.0f > mx) mx = 0.0f;
        const float denom = expf(sc[n] - mx);
        for (int a = r0; a < r1; a++) {
          const float cur = g * expf(sc[ar[a].x] + __int_as_float(ar[a].y) - mx) / denom;
          atomicAdd(&ng[ar[a].x], cur);
          ag[a] = cur * delta;
        }
      }
    }
    __syncthreads();
  }
}

/* ------------------------------------------------------------------ */
/* traceback (shortest.cpp:240-245) and label provenance               */
/* ------------------------------------------------------------------ */

__global__ void traceback_kernel(
    const GraphMeta* __restrict__ meta,
    const int2* __restrict__ arcs,
    const int32_t* __restrict__ back_ptr,
    const int32_t* __restrict__ best_accept,
    int B,
    int max_len,
    int32_t* __restrict__ path,
    int32_t* __restrict__ path_len) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const GraphMeta m = meta[b];
  if (m.status != GTNB_OK) {
    path_len[b] = -1;
    return;
  }
  const int2* ar = arcs + m.arc_base;
  const int32_t* bp = back_ptr + m.node_base;
  int32_t* p = path + (long long)b * max_len;
  int n = best_accept[b];
  if (n < 0) {
    path_len[b] = -1;
    return;
  }
  int len = 0;
  while (n != -1 && bp[n] != -1) {
    const int a = bp[n];
    if (len < max_len) p[len] = a;
    len++;
    n = ar[a].x;
  }
  const int k = len < max_len ? len : max_len;
  for (int i = 0; i < k / 2; i++) {
    const int t = p[i];
    p[i] = p[k - 1 - i];
    p[k - 1 - i] = t;
  }
  path_len[b] = len;
}

__global__ void gather_prov_kernel(
    const GraphMeta* __restrict__ meta,
    const int2* __restrict__ gi, // nullable
    const int2* __restrict__ arcs,
    int max_len,
    const int32_t* __restrict__ path,
    const int32_t* __restrict__ path_len,
    int32_t* __restrict__ pg,
    int32_t* __restrict__ pl,
    float* __restrict__ pw) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int len = path_len[b] < max_len ? path_len[b] : max_len;
  if (i >= len) return;
  const long long k = (long long)b * max_len + i;
  const long long a = meta[b].arc_base + path[k];
  if (gi) {
    pg[k] = gi[a].x;
    pl[k] = gi[a].y;
  }
  if (pw) pw[k] = __int_as_float(arcs[a].y);
}

} // namespace

#ifndef GTNB_HOST_EMU

static bool use_staged(const gtnb_ctx* ctx, const gtnb_lattice* lat) {
  return ctx->use_staged && staged_supported(lat);
}

/* the generic kernels log under their own names ("sd_forward_generic", "sd_backward_generic"), so a launch profile
 * tells them from the staged kernels ("sd_forward", "sd_backward") */
int launch_forward(gtnb_ctx* ctx, gtnb_lattice* lat, int mode) {
  if (lat->B == 0) return GTNB_OK;
  if (use_staged(ctx, lat)) return launch_forward_staged(ctx, lat, mode);
  dim3 grid(lat->B), block(kThreads);
#define ARGS                                                                           \
  lat->meta, lat->lvl_node_ptr, lat->row_ptr, lat->arcs,                        \
      (mode == MODE_PATH ? lat->relax_rank : nullptr), lat->acc_nodes, lat->scores,    \
      lat->back_ptr, lat->out_scores, lat->best_accept
  if (mode == MODE_LOG)
    GTNB_LAUNCH(ctx, "sd_forward_generic", sd_forward_generic<MODE_LOG><<<grid, block, 0, ctx->stream>>>(ARGS));
  else if (mode == MODE_TROPICAL)
    GTNB_LAUNCH(ctx, "sd_forward_generic", sd_forward_generic<MODE_TROPICAL><<<grid, block, 0, ctx->stream>>>(ARGS));
  else
    GTNB_LAUNCH(ctx, "sd_forward_generic", sd_forward_generic<MODE_PATH><<<grid, block, 0, ctx->stream>>>(ARGS));
#undef ARGS
  return GTNB_OK;
}

int launch_backward(gtnb_ctx* ctx, gtnb_lattice* lat, int tropical, const float* deltas_dev) {
  if (lat->B == 0) return GTNB_OK;
  if (use_staged(ctx, lat)) return launch_backward_staged(ctx, lat, tropical, deltas_dev);
  if (!lat->node_grad) {
    int rc = dev_alloc(ctx, &lat->node_grad, lat->tot_N);
    if (rc) return rc;
  }
  dim3 grid(lat->B), block(kThreads);
#define ARGS                                                                              \
  lat->meta, lat->lvl_node_ptr, lat->blvl_ptr, lat->bnodes, lat->row_ptr, lat->arcs,      \
      lat->acc_nodes, lat->scores, lat->out_scores, lat->best_accept, deltas_dev, \
      lat->node_grad, lat->arc_grad
  if (tropical)
    GTNB_LAUNCH(ctx, "sd_backward_generic", sd_backward_generic<true><<<grid, block, 0, ctx->stream>>>(ARGS));
  else
    GTNB_LAUNCH(ctx, "sd_backward_generic", sd_backward_generic<false><<<grid, block, 0, ctx->stream>>>(ARGS));
#undef ARGS
  return GTNB_OK;
}

int launch_traceback(gtnb_ctx* ctx, gtnb_lattice* lat, int max_len, int32_t* path_dev, int32_t* len_dev) {
  if (lat->B == 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "traceback", traceback_kernel<<<(lat->B + 63) / 64, 64, 0, ctx->stream>>>(
      lat->meta, lat->arcs, lat->back_ptr, lat->best_accept, lat->B, max_len, path_dev, len_dev));
  return GTNB_OK;
}

int launch_gather_prov(
    gtnb_ctx* ctx, gtnb_lattice* lat, int max_len, const int32_t* path_dev,
    const int32_t* len_dev, int32_t* pg, int32_t* pl, float* pw) {
  if (lat->B == 0 || max_len == 0) return GTNB_OK;
  dim3 grid((max_len + 127) / 128, lat->B);
  GTNB_LAUNCH(ctx, "gather_prov", gather_prov_kernel<<<grid, 128, 0, ctx->stream>>>(
      lat->meta, lat->gi, lat->arcs, max_len, path_dev, len_dev, pg, pl, pw));
  return GTNB_OK;
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
