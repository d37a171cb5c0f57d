/*
 * k_compose.cu -- frame-synchronous composition on the device.
 *
 * Replaces detail::compose (compose.cpp:377-522) for the case where one operand
 * is a gtn::linearGraph (the emissions chain, creations.cpp:20-33): a product
 * state is (graph node, frame), every arc advances one frame, and the
 * reference's two passes become
 *
 *   findReachable (compose.cpp:64-104)   -> backward "can reach accept" bitmask
 *                                           per frame                (k1)
 *   forward BFS   (compose.cpp:389-489)  -> forward "reached from start"
 *                                           bitmask per frame        (k1)
 *   node / arc creation                  -> per-frame counts (k2), prefix sums
 *                                           (k3), CSR emission (k4)
 *
 * and the result is written straight into HBM as the levelised CSR-by-
 * destination batch the shortest-distance kernels consume (level == frame).
 * Node numbering: frame-major, then graph node id; arcs are numbered in CSR
 * order (grouped by destination; within a destination by (source node,
 * position in the source's out-arc list)).  The reference leaves compose's
 * numbering unspecified (its tests only check isomorphism,
 * test/functions_test.cpp:137-227).
 *
 *   compose_grad_kernel = compose's gradFunc (compose.cpp:496-518).
 */
#include <algorithm>

#include "gtnb_ptx.h"

namespace gtnb {

namespace {

constexpr int kWarpsPerBlock = 8;
constexpr int kMaxWords = 256; // graphs of up to 8192 nodes

/* ---- k1: per-frame alive sets ------------------------------------- */

__global__ void __launch_bounds__(256) compose_alive_kernel(
    const GraphMeta* __restrict__ meta,
    const uint8_t* __restrict__ sg_flags,
    const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ sg_in_src,
    const int32_t* __restrict__ sg_in_label,
    uint32_t* __restrict__ alive,
    int W,
    int maxT) {
  GTNB_STATIC_SMEM(uint32_t, cur, kMaxWords);
  GTNB_STATIC_SMEM(uint32_t, nxt, kMaxWords);
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x;
  const int N1 = m.sg_N, T = m.T;
  const int Wg = (N1 + 31) / 32;
  const uint8_t* fl = sg_flags + m.sg_node_base;
  const int32_t* ip = sg_in_ptr + m.sg_node_base;
  const int32_t* is = sg_in_src + m.sg_arc_base;
  const int32_t* il = sg_in_label + m.sg_arc_base;
  uint32_t* al = alive + (size_t)blockIdx.x * (maxT + 1) * W;

  // ---- forward reachability: fw[0] = start nodes
  for (int c = tid; c < W; c += blockDim.x) cur[c] = 0;
  __syncthreads();
  for (int n = tid; n < N1; n += blockDim.x)
    if (fl[n] & 1) atomicOr(&cur[n >> 5], 1u << (n & 31));
  __syncthreads();
  for (int c = tid; c < W; c += blockDim.x) al[c] = cur[c];
  int t = 0;
  for (; t < T; t++) {
    for (int c = tid; c < W; c += blockDim.x) nxt[c] = 0;
    __syncthreads();
    for (int d = tid; d < N1; d += blockDim.x) {
      bool hit = false;
      for (int e = ip[d]; e < ip[d + 1] && !hit; e++) {
        const int s = is[e];
        hit = il[e] >= 0 && ((cur[s >> 5] >> (s & 31)) & 1u);
      }
      if (hit) atomicOr(&nxt[d >> 5], 1u << (d & 31));
    }
    __syncthreads();
    int same = 1;
    for (int c = tid; c < Wg; c += blockDim.x) same &= (nxt[c] == cur[c]);
    same = __syncthreads_and(same);
    if (same) break; // fixed point: every later frame has the same set
    for (int c = tid; c < W; c += blockDim.x) {
      cur[c] = nxt[c];
      al[(size_t)(t + 1) * W + c] = nxt[c];
    }
    __syncthreads();
  }
  if (t < T) {
    for (int i = tid; i < (T - t) * W; i += blockDim.x) {
      const int tt = t + 1 + i / W, c = i % W;
      al[(size_t)tt * W + c] = cur[c];
    }
  }
  __syncthreads();

  // ---- backward co-reachability: bw[T] = accept nodes; alive = fw & bw
  for (int c = tid; c < W; c += blockDim.x) cur[c] = 0;
  __syncthreads();
  for (int n = tid; n < N1; n += blockDim.x)
    if (fl[n] & 2) atomicOr(&cur[n >> 5], 1u << (n & 31));
  __syncthreads();
  for (int c = tid; c < W; c += blockDim.x) al[(size_t)T * W + c] &= cur[c];
  t = T;
  for (; t > 0; t--) {
    for (int c = tid; c < W; c += blockDim.x) nxt[c] = 0;
    __syncthreads();
    for (int d = tid; d < N1; d += blockDim.x) {
      if ((cur[d >> 5] >> (d & 31)) & 1u) {
        for (int e = ip[d]; e < ip[d + 1]; e++)
          if (il[e] >= 0) atomicOr(&nxt[is[e] >> 5], 1u << (is[e] & 31));
      }
    }
    __syncthreads();
    int same = 1;
    for (int c = tid; c < Wg; c += blockDim.x) same &= (nxt[c] == cur[c]);
    same = __syncthreads_and(same);
    if (same) break;
    for (int c = tid; c < W; c += blockDim.x) {
      cur[c] = nxt[c];
      al[(size_t)(t - 1) * W + c] &= nxt[c];
    }
    __syncthreads();
  }
  if (t > 0) {
    for (int i = tid; i < t * W; i += blockDim.x) {
      const int tt = i / W, c = i % W;
      al[(size_t)tt * W + c] &= cur[c];
    }
  }
}

/* ---- k2: per-frame node / arc counts -------------------------------- */

__global__ void __launch_bounds__(32 * kWarpsPerBlock) compose_count_kernel(
    const GraphMeta* __restrict__ meta,
    const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ sg_in_src,
    const int32_t* __restrict__ sg_in_label,
    const uint32_t* __restrict__ alive,
    int W,
    int maxT,
    int32_t* __restrict__ lvl_node_ptr,
    int32_t* __restrict__ lvl_arc_ptr) {
  const int b = blockIdx.y;
  const GraphMeta m = meta[b];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * kWarpsPerBlock + warp;
  if (t > m.T) return;
  const int Wg = (m.sg_N + 31) / 32;
  const int32_t* ip = sg_in_ptr + m.sg_node_base;
  const int32_t* is = sg_in_src + m.sg_arc_base;
  const int32_t* il = sg_in_label + m.sg_arc_base;
  const uint32_t* at = alive + ((size_t)b * (maxT + 1) + t) * W;
  const uint32_t* ap = at - W;
  int nodes = 0, arcs = 0;
  // steady state: every graph node alive in this frame and the one before, every label
  // matchable -> the level is the whole graph: nothing to count
  if (t > 0 && m.sg_all_valid) {
    int ct = 0, cp = 0;
    for (int c = lane; c < Wg; c += 32) {
      ct += __popc(at[c]);
      cp += __popc(ap[c]);
    }
    for (int o = 16; o > 0; o >>= 1) {
      ct += __shfl_xor_sync(0xffffffffu, ct, o);
      cp += __shfl_xor_sync(0xffffffffu, cp, o);
    }
    if (ct == m.sg_N && cp == m.sg_N) {
      if (lane == 0) {
        lvl_node_ptr[m.lvl_base + t] = m.sg_N;
        lvl_arc_ptr[m.lvl_base + t] = m.sg_A;
      }
      return;
    }
  }
  for (int c = 0; c < Wg; c++) {
    const uint32_t word = at[c];
    nodes += __popc(word);
    if (t > 0 && ((word >> lane) & 1u)) {
      const int d = c * 32 + lane;
      for (int e = ip[d]; e < ip[d + 1]; e++) {
        const int s = is[e];
        arcs += (il[e] >= 0 && ((ap[s >> 5] >> (s & 31)) & 1u)) ? 1 : 0;
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) arcs += __shfl_xor_sync(0xffffffffu, arcs, o);
  if (lane == 0) {
    lvl_node_ptr[m.lvl_base + t] = nodes;
    lvl_arc_ptr[m.lvl_base + t] = arcs;
  }
}

/* ---- k3: exclusive scans over the frames + accept list -------------- */

__global__ void __launch_bounds__(1024) compose_scan_kernel(
    GraphMeta* __restrict__ meta,
    const uint8_t* __restrict__ sg_flags,
    const uint32_t* __restrict__ alive,
    int W,
    int maxT,
    int32_t* __restrict__ lvl_node_ptr,
    int32_t* __restrict__ lvl_arc_ptr,
    int32_t* __restrict__ acc_nodes) {
  GTNB_STATIC_SMEM(int, sn, 1024);
  GTNB_STATIC_SMEM(int, sa, 1024);
  const int b = blockIdx.x;
  const GraphMeta m = meta[b];
  const int tid = threadIdx.x;
  const int L = m.T + 1;
  int32_t* np = lvl_node_ptr + m.lvl_base;
  int32_t* apn = lvl_arc_ptr + m.lvl_base;
  const int per = (L + 1023) / 1024;
  const int lo = min(tid * per, L), hi = min(lo + per, L);
  int tn = 0, ta = 0;
  for (int i = lo; i < hi; i++) {
    tn += np[i];
    ta += apn[i];
  }
  sn[tid] = tn;
  sa[tid] = ta;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    int vn = 0, va = 0;
    if (tid >= o) {
      vn = sn[tid - o];
      va = sa[tid - o];
    }
    __syncthreads();
    sn[tid] += vn;
    sa[tid] += va;
    __syncthreads();
  }
  int bn = sn[tid] - tn, ba = sa[tid] - ta; // exclusive prefix of this thread's chunk
  // arcs of level l are the in-arcs of its nodes: lvl_arc_ptr[l] = #arcs into levels < l
  for (int i = lo; i < hi; i++) {
    const int cn = np[i], ca = apn[i];
    np[i] = bn;
    apn[i] = ba;
    bn += cn;
    ba += ca;
  }
  const int totN = sn[1023], totA = sa[1023];
  __syncthreads();
  if (tid == 0) {
    np[L] = totN;
    apn[L] = totA;
    // accept nodes of the lattice: (accept node a of the graph, frame T), in
    // g.accept() order of the graph -- its accept list was staged in acc_nodes.
    int32_t* acc = acc_nodes + m.acc_base;
    const uint32_t* aT = alive + ((size_t)b * (maxT + 1) + m.T) * W;
    const int baseT = np[m.T];
    int k = 0;
    for (int i = 0; i < m.n_accept; i++) {
      const int a = acc[i];
      if ((aT[a >> 5] >> (a & 31)) & 1u) {
        int rank = 0;
        for (int c = 0; c < (a >> 5); c++) rank += __popc(aT[c]);
        rank += __popc(aT[a >> 5] & ((1u << (a & 31)) - 1u));
        acc[k++] = baseT + rank;
      }
    }
    meta[b].N = totN;
    meta[b].A = totA;
    meta[b].n_accept = k;
  }
}

/* ---- k4: emit the CSR ------------------------------------------------ */

__global__ void __launch_bounds__(32 * kWarpsPerBlock) compose_emit_kernel(
    const GraphMeta* __restrict__ meta,
    const uint8_t* __restrict__ sg_flags,
    const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ sg_in_src,
    const int32_t* __restrict__ sg_in_label,
    const int32_t* __restrict__ sg_in_arc,
    const float* __restrict__ sg_in_w,
    const uint32_t* __restrict__ alive,
    int W,
    int maxT,
    int C,
    const float* __restrict__ emissions,
    const int32_t* __restrict__ lvl_node_ptr,
    const int32_t* __restrict__ lvl_arc_ptr,
    uint32_t* __restrict__ row_ptr,
    int2* __restrict__ arcs,
    int2* __restrict__ gi) {
  GTNB_STATIC_SMEM_2D(int, pre, kWarpsPerBlock, kMaxWords); // popcount prefix of alive[t-1]
  const int b = blockIdx.y;
  const GraphMeta m = meta[b];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * kWarpsPerBlock + warp;
  if (t > m.T) return;
  const int Wg = (m.sg_N + 31) / 32;
  const uint8_t* fl = sg_flags + m.sg_node_base;
  const int32_t* ip = sg_in_ptr + m.sg_node_base;
  const int32_t* is = sg_in_src + m.sg_arc_base;
  const int32_t* il = sg_in_label + m.sg_arc_base;
  const int32_t* ia = sg_in_arc + m.sg_arc_base;
  const float* iw = sg_in_w + m.sg_arc_base;
  const uint32_t* at = alive + ((size_t)b * (maxT + 1) + t) * W;
  const uint32_t* ap = at - W;
  const int32_t* np = lvl_node_ptr + m.lvl_base;
  const int32_t* apn = lvl_arc_ptr + m.lvl_base;
  uint32_t* rp = row_ptr + m.node_base;
  int2* ao = arcs + m.arc_base;
  int2* go = gi + m.arc_base;
  const float* em = emissions + m.emis_off + (long long)(t - 1) * C;

  const int nb = np[t];
  const int ab = apn[t];
  const int pb = t > 0 ? np[t - 1] : 0;
  // steady state (see compose_count_kernel): the level is the whole graph in its canonical
  // in-arc order; lattice arc k of the level is graph in-entry k, node d has rank d
  if (t > 0 && m.sg_all_valid && np[t + 1] - nb == m.sg_N && nb - pb == m.sg_N) {
    for (int d = lane; d < m.sg_N; d += 32) {
      uint32_t flags = 0;
      if (t == m.T && (fl[d] & 2)) flags |= kAcceptBit;
      rp[nb + d] = (uint32_t)(ab + ip[d]) | flags;
    }
    // four independent entries per lane in flight: all loads first, then the stores
    for (int e0 = lane; e0 < m.sg_A; e0 += 128) {
      int lab[4], srcn[4], arcid[4];
      float wv[4];
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int e = e0 + 32 * k;
        const bool ok = e < m.sg_A;
        lab[k] = ok ? il[e] : 0;
        srcn[k] = ok ? is[e] : 0;
        arcid[k] = ok ? ia[e] : 0;
        wv[k] = ok ? iw[e] : 0.0f;
      }
      float ev[4];
#pragma unroll
      for (int k = 0; k < 4; k++) ev[k] = em[lab[k]];
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int e = e0 + 32 * k;
        if (e < m.sg_A) {
          ao[ab + e] = make_int2(pb + srcn[k], __float_as_int(wv[k] + ev[k]));
          go[ab + e] = make_int2(arcid[k], (t - 1) * C + lab[k]);
        }
      }
    }
    if (t == m.T && lane == 0) rp[np[m.T + 1]] = (uint32_t)apn[m.T + 1];
    return;
  }
  if (t > 0) {
    int run = 0;
    for (int c0 = 0; c0 < Wg; c0 += 32) {
      const int c = c0 + lane;
      const int cnt = c < Wg ? __popc(ap[c]) : 0;
      int inc = cnt;
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
      }
      if (c < Wg) pre[warp][c] = run + inc - cnt;
      run += __shfl_sync(0xffffffffu, inc, 31);
    }
    __syncwarp();
  }
  int run_nodes = 0, run_arcs = 0;
  for (int c = 0; c < Wg; c++) {
    const uint32_t word = at[c];
    const bool live = (word >> lane) & 1u;
    const int d = c * 32 + lane;
    int deg = 0;
    if (live && t > 0) {
      for (int e = ip[d]; e < ip[d + 1]; e++) {
        const int s = is[e];
        deg += (il[e] >= 0 && ((ap[s >> 5] >> (s & 31)) & 1u)) ? 1 : 0;
      }
    }
    int inc = deg;
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += v;
    }
    const int tot = __shfl_sync(0xffffffffu, inc, 31);
    if (live) {
      const int node = nb + run_nodes + __popc(word & lanemask_lt());
      int pos = ab + run_arcs + inc - deg;
      uint32_t flags = 0;
      if (t == 0 && (fl[d] & 1)) flags |= kStartBit;
      if (t == m.T && (fl[d] & 2)) flags |= kAcceptBit;
      rp[node] = (uint32_t)pos | flags;
      if (t > 0) {
        for (int e = ip[d]; e < ip[d + 1]; e++) {
          const int s = is[e];
          const int lab = il[e];
          if (lab >= 0 && ((ap[s >> 5] >> (s & 31)) & 1u)) {
            // weight = first.weight(i) + second.weight(j), compose.cpp:435
            ao[pos] = make_int2(pb + pre[warp][s >> 5] + __popc(ap[s >> 5] & ((1u << (s & 31)) - 1u)),
                                __float_as_int(iw[e] + em[lab]));
            go[pos] = make_int2(ia[e], (t - 1) * C + lab);
            pos++;
          }
        }
      }
    }
    run_nodes += __popc(word);
    run_arcs += tot;
  }
  if (t == m.T && lane == 0) rp[np[m.T + 1]] = (uint32_t)apn[m.T + 1];
}

/* ---- compose gradFunc (compose.cpp:496-518) -------------------------- */

__global__ void __launch_bounds__(256) compose_grad_kernel(
    const GraphMeta* __restrict__ meta,
    const uint32_t* __restrict__ row_ptr,
    const float* __restrict__ arc_grad,
    const int2* __restrict__ gi,
    float* __restrict__ grad_graph,
    float* __restrict__ grad_emis,
    long long grad_stride) {
  // one thread per lattice node: its in-arcs are contiguous and (in every CTC / ASG lattice)
  // share the emission they came from, so their gradients are summed in registers and leave
  // as ONE atomic per node instead of one per arc
  const int b = blockIdx.y;
  const GraphMeta m = meta[b];
  const uint32_t* rp = row_ptr + m.node_base;
  const float* ag = arc_grad + m.arc_base;
  const int2* gp = gi + m.arc_base;
  float* g1 = grad_graph ? grad_graph + m.grad_graph_off : nullptr;
  float* g2 = grad_emis ? grad_emis + (long long)b * grad_stride : nullptr;
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < m.N; n += gridDim.x * blockDim.x) {
    const int r0 = (int)(rp[n] & kRowMask), r1 = (int)(rp[n + 1] & kRowMask);
    if (r1 == r0) continue;
    int key = -1;
    float acc = 0.0f;
    for (int a = r0; a < r1; a++) {
      const float g = ag[a];
      const int2 p = gp[a];
      if (g1) atomicAdd(&g1[p.x], g);
      if (g2) {
        if (p.y == key) {
          acc += g;
        } else {
          if (key >= 0) atomicAdd(&g2[key], acc);
          key = p.y;
          acc = g;
        }
      }
    }
    if (g2 && key >= 0) atomicAdd(&g2[key], acc);
  }
}

} // namespace

#ifndef GTNB_HOST_EMU

int launch_compose(gtnb_ctx* ctx, gtnb_lattice* lat, cudaEvent_t emissions_ready) {
  if (lat->B == 0) return GTNB_OK;
  const int W = lat->alive_words;
  if (W > kMaxWords)
    return fail(ctx, GTNB_ERR_UNSUPPORTED, "gtnb_compose_linear: graph has more than 8192 nodes");
  const int maxT = lat->max_T;
  GTNB_LAUNCH(ctx, "compose_alive", compose_alive_kernel<<<lat->B, 256, 0, ctx->stream>>>(
      lat->meta, lat->sg_flags, lat->sg_in_ptr, lat->sg_in_src, lat->sg_in_label, lat->alive, W, maxT));
  dim3 grid((maxT + 1 + kWarpsPerBlock - 1) / kWarpsPerBlock, lat->B);
  GTNB_LAUNCH(ctx, "compose_count", compose_count_kernel<<<grid, 32 * kWarpsPerBlock, 0, ctx->stream>>>(
      lat->meta, lat->sg_in_ptr, lat->sg_in_src, lat->sg_in_label, lat->alive, W, maxT,
      lat->lvl_node_ptr, lat->lvl_arc_ptr));
  GTNB_LAUNCH(ctx, "compose_scan", compose_scan_kernel<<<lat->B, 1024, 0, ctx->stream>>>(
      lat->meta, lat->sg_flags, lat->alive, W, maxT, lat->lvl_node_ptr, lat->lvl_arc_ptr,
      lat->acc_nodes));
  // the structure passes above never touch the emissions: a host->device copy of them may
  // still be in flight on another stream up to here
  if (emissions_ready) GTNB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, emissions_ready, 0));
  GTNB_LAUNCH(ctx, "compose_emit", compose_emit_kernel<<<grid, 32 * kWarpsPerBlock, 0, ctx->stream>>>(
      lat->meta, lat->sg_flags, lat->sg_in_ptr, lat->sg_in_src, lat->sg_in_label, lat->sg_in_arc,
      lat->sg_in_w, lat->alive, W, maxT, lat->C, lat->emissions, lat->lvl_node_ptr,
      lat->lvl_arc_ptr, lat->row_ptr, lat->arcs, lat->gi));
  return GTNB_OK;
}

int launch_compose_grad(
    gtnb_ctx* ctx, gtnb_lattice* lat, float* grad_graph, float* grad_emis, int64_t grad_stride) {
  if (lat->B == 0) return GTNB_OK;
  int capN = 1;
  for (int b = 0; b < lat->B; b++) capN = std::max(capN, lat->meta_h[b].cap_N);
  int gx = std::min((capN + 255) / 256, 4096);
  dim3 grid(gx, lat->B);
  GTNB_LAUNCH(ctx, "compose_grad", compose_grad_kernel<<<grid, 256, 0, ctx->stream>>>(
      lat->meta, lat->row_ptr, lat->arc_grad, lat->gi, grad_graph, grad_emis,
      (long long)grad_stride));
  return GTNB_OK;
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
