/*
 * k_order.cu -- the reference's tie-breaking order on a device-composed lattice (on by default;
 * gtnb_ctx_set_flag("exact_ties", 0) before gtnb_compose_linear skips it).  GPU-validated in round 2
 * (tests/test_gpu_parity.py::test_viterbi_exact_ties_vs_oracle,
 * tests/test_gpu_config_parity.py::test_forced_alignment_config4_vs_reference).  The sort is deferred until a
 * lattice's arc ids or per-arc values first cross the ABI (gtnb_capi.cu, settle_order) and carries arc_grad with the
 * arcs, so the answers do not depend on the order of calls: tests/test_gpu_lattice_call_order.py (every measured
 * call after every call history, against the reference) and
 * tests/test_compose_emulation.py::test_exact_ties_sort_carries_arc_grads (gradients follow their arcs through
 * lattice_sort_rows_kernel).
 *
 * detail::shortestPath (shortest.cpp:190-245) keeps, for every node, the FIRST-RELAXED predecessor
 * among those that reach the maximum, and the first strictly greatest accept node in g.accept()
 * order.  On compose(g, linearGraph) both orders are structural:
 *
 *   discovery  compose's BFS (compose.cpp:389-470) creates the product states of frame t+1 while it
 *              explores those of frame t in creation order, their matched arcs in matcher order; a
 *              state is created by the first arc that reaches it.  g.accept() of the composed graph
 *              is the creation order of its accepting states.
 *   relaxation shortestPath pops frame t's states in the order they became ready; state (v, t+1)
 *              becomes ready when the LAST of its in-arcs has been relaxed.
 *
 * With pos_D / pos_P the position of a frame-t state in the two orders and o(e) the position of
 * graph arc e in its source's out-arc list (the matcher enumerates a state's arcs in that order when
 * the graph operand is the query side: unsorted and singly-sorted matchers always, the doubly-sorted
 * one while out-degree <= C, compose.cpp:211-374):
 *
 *   key_D(v) = min over in-arcs e: u -> v of  pos_D[u] * K + o(e)      pos_D'[v] = rank of key_D
 *   key_P(v) = max over in-arcs e: u -> v of  pos_P[u] * K + o(e)      pos_P'[v] = rank of key_P
 *
 * and the relaxation rank of lattice arc (u, t) -> (v, t+1) is pos_P[u] * K + o(e).  Every lattice row's
 * arcs (and their provenance) are then sorted by that rank, so that "first maximum in in-arc order" --
 * what every MODE_PATH kernel, staged or generic, already implements -- IS the reference's rule, and the
 * lattice's accept list is put in the composed graph's accept order.
 * One CTA per utterance walks the frames; the ranks of a frame come from a presence bitmap of its keys
 * (distinct integers below N * K) and a prefix sum of the popcounts.
 */
#include <algorithm>

#include "gtnb_ptx.h"

namespace gtnb {

namespace {

constexpr int kOrderThreads = 256;
constexpr int kNoKey = 0x7fffffff;

__device__ __forceinline__ bool bit_of(const uint32_t* words, int n) {
  return (words[n >> 5] >> (n & 31)) & 1u;
}

/* number of set bits below position n */
__device__ __forceinline__ int rank_of(const uint32_t* words, int n) {
  int r = 0;
  for (int c = 0; c < (n >> 5); c++) r += __popc(words[c]);
  return r + __popc(words[n >> 5] & ((1u << (n & 31)) - 1u));
}

__global__ void __launch_bounds__(kOrderThreads) lattice_relax_order_kernel(
    const GraphMeta* __restrict__ meta,
    const uint8_t* __restrict__ sg_flags,
    const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ sg_in_src,
    const int32_t* __restrict__ sg_in_label,
    const int32_t* __restrict__ sg_out_pos, // per in-entry: position of the arc in its source's out list
    const int32_t* __restrict__ sg_start_rank, // per graph node: index in g.start(), -1 if not a start node
    const uint32_t* __restrict__ alive,
    int W,
    int maxT,
    int K, // > every out-arc position
    const int32_t* __restrict__ lvl_node_ptr,
    const uint32_t* __restrict__ row_ptr,
    int32_t* __restrict__ relax_rank, // out, per lattice arc
    int32_t* __restrict__ acc_nodes) { // in / out: reordered to the composed graph's accept order
  GTNB_DYNAMIC_SMEM(int, o_smem);
  const GraphMeta m = meta[blockIdx.x];
  const int tid = threadIdx.x;
  const int N1 = m.sg_N, T = m.T;
  int* posD = o_smem; // positions of the current frame's states
  int* posP = o_smem + N1;
  int* keyD = o_smem + 2 * N1; // keys of the next frame's states
  int* keyP = o_smem + 3 * N1;
  const int32_t* ip = sg_in_ptr + m.sg_node_base;
  const int32_t* is = sg_in_src + m.sg_arc_base;
  const int32_t* il = sg_in_label + m.sg_arc_base;
  const int32_t* op = sg_out_pos + m.sg_arc_base;
  const int32_t* sr = sg_start_rank + m.sg_node_base;
  const uint8_t* fl = sg_flags + m.sg_node_base;
  const uint32_t* al = alive + (size_t)blockIdx.x * (maxT + 1) * W;
  const int32_t* lp = lvl_node_ptr + m.lvl_base;
  const uint32_t* rp = row_ptr + m.node_base;
  int32_t* rr = relax_rank + m.arc_base;

  // frame 0: the start states, in g.start() order, are both created and popped in that order
  for (int u = tid; u < N1; u += kOrderThreads) keyD[u] = (bit_of(al, u) && sr[u] >= 0) ? sr[u] : kNoKey;
  __syncthreads();
  for (int u = tid; u < N1; u += kOrderThreads) {
    int r = -1;
    if (keyD[u] != kNoKey) {
      r = 0;
      for (int w = 0; w < N1; w++) r += keyD[w] < keyD[u];
    }
    posD[u] = r;
    posP[u] = r;
  }
  __syncthreads();

  // Ranks by counting: the keys of a frame are distinct integers below N1 * K (two states never share an arc),
  // so a presence bitmap + a prefix sum of its popcounts gives every rank in O(1) -- the all-pairs count this
  // replaces was quadratic in the states of a frame (N1 = 401 for forced alignment at U = 200).
  const int WB = (N1 * K + 31) >> 5;
  uint32_t* bmD = reinterpret_cast<uint32_t*>(o_smem + 4 * N1);
  uint32_t* bmP = bmD + WB;
  int* pfD = reinterpret_cast<int*>(bmP + WB);
  int* pfP = pfD + WB;
  const int lane = tid & 31, warp = tid >> 5;
  for (int t = 0; t < T; t++) {
    const uint32_t* at = al + (size_t)t * W; // frame t
    const uint32_t* an = at + W; // frame t + 1
    for (int w = tid; w < 2 * WB; w += kOrderThreads) bmD[w] = 0u; // (bmP follows bmD)
    __syncthreads();
    for (int v = tid; v < N1; v += kOrderThreads) {
      int kd = kNoKey, kp = -1;
      if (bit_of(an, v)) {
        // the row of lattice node (v, t+1): its arcs are the in-entries of v whose source is alive in
        // frame t, in in-entry order (compose_emit_kernel)
        int pos = (int)(rp[lp[t + 1] + rank_of(an, v)] & kRowMask);
        for (int e = ip[v]; e < ip[v + 1]; e++) {
          const int u = is[e];
          if (il[e] >= 0 && bit_of(at, u)) {
            kd = min(kd, posD[u] * K + op[e]);
            const int rk = posP[u] * K + op[e];
            kp = max(kp, rk);
            rr[pos++] = rk;
          }
        }
      }
      keyD[v] = kd;
      keyP[v] = kp;
      if (kd != kNoKey) {
        atomicOr(&bmD[kd >> 5], 1u << (kd & 31));
        atomicOr(&bmP[kp >> 5], 1u << (kp & 31));
      }
    }
    __syncthreads();
    if (warp < 2) { // warp 0: prefix popcounts of bmD, warp 1: of bmP
      const uint32_t* bm = warp ? bmP : bmD;
      int* pf = warp ? pfP : pfD;
      int run = 0;
      for (int w0 = 0; w0 < WB; w0 += 32) {
        const int c = w0 + lane < WB ? __popc(bm[w0 + lane]) : 0;
        int x = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int y = __shfl_up_sync(0xffffffffu, x, o);
          if (lane >= o) x += y;
        }
        if (w0 + lane < WB) pf[w0 + lane] = run + x - c;
        run += __shfl_sync(0xffffffffu, x, 31);
      }
    }
    __syncthreads();
    for (int v = tid; v < N1; v += kOrderThreads) {
      int rd = -1, rq = -1;
      const int kd = keyD[v], kp = keyP[v];
      if (kd != kNoKey) { // states that are not alive carry kNoKey
        rd = pfD[kd >> 5] + __popc(bmD[kd >> 5] & ((1u << (kd & 31)) - 1u));
        rq = pfP[kp >> 5] + __popc(bmP[kp >> 5] & ((1u << (kp & 31)) - 1u));
      }
      posD[v] = rd;
      posP[v] = rq;
    }
    __syncthreads();
  }

  // g.accept() of the composed graph: its accepting states in creation order
  if (tid == 0) {
    const uint32_t* aT = al + (size_t)T * W;
    int32_t* acc = acc_nodes + m.acc_base;
    for (int u = 0; u < N1; u++) {
      if (!(bit_of(aT, u) && (fl[u] & 2))) continue;
      int before = 0; // accepting states created earlier
      for (int w = 0; w < N1; w++) before += bit_of(aT, w) && (fl[w] & 2) && posD[w] < posD[u];
      acc[before] = lp[T] + rank_of(aT, u);
    }
  }
}

/* sort the arcs of every lattice row by relaxation rank (rows are a handful of arcs: insertion sort,
 * one thread per lattice node); the provenance and, when a backward pass has run, the arc gradient move
 * with the arc */
__global__ void __launch_bounds__(256) lattice_sort_rows_kernel(
    const GraphMeta* __restrict__ meta,
    const uint32_t* __restrict__ row_ptr,
    int32_t* __restrict__ relax_rank,
    int2* __restrict__ arcs,
    int2* __restrict__ gi,
    float* __restrict__ arc_grad = nullptr) { // nullable: no backward pass has run yet
  const int b = blockIdx.y;
  const GraphMeta m = meta[b];
  const uint32_t* rp = row_ptr + m.node_base;
  int32_t* rr = relax_rank + m.arc_base;
  int2* ar = arcs + m.arc_base;
  int2* gp = gi + m.arc_base;
  float* ag = arc_grad ? arc_grad + m.arc_base : nullptr;
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < m.N; n += gridDim.x * blockDim.x) {
    const int r0 = (int)(rp[n] & kRowMask), r1 = (int)(rp[n + 1] & kRowMask);
    for (int a = r0 + 1; a < r1; a++) {
      const int key = rr[a];
      const int2 av = ar[a], gv = gp[a];
      const float dv = ag ? ag[a] : 0.0f;
      int p = a - 1;
      while (p >= r0 && rr[p] > key) {
        rr[p + 1] = rr[p];
        ar[p + 1] = ar[p];
        gp[p + 1] = gp[p];
        if (ag) ag[p + 1] = ag[p];
        p--;
      }
      rr[p + 1] = key;
      ar[p + 1] = av;
      gp[p + 1] = gv;
      if (ag) ag[p + 1] = dv;
    }
  }
}

} // namespace

#ifndef GTNB_HOST_EMU

/* put a composed lattice in the reference's relaxation order (rows) and accept order, carrying the arc
 * gradients of a backward pass that ran before it; needs the tables the "exact_ties" flag makes
 * gtnb_compose_linear upload */
int launch_relax_order(gtnb_ctx* ctx, gtnb_lattice* lat) {
  if (lat->B == 0) return GTNB_OK;
  if (!lat->sg_out_pos || !lat->sg_start_rank || !lat->alive || !lat->gi)
    return fail(ctx, GTNB_ERR_LOGIC, "exact_ties: the lattice was composed without the flag");
  // positions / keys (4 N) + two key bitmaps and their prefix popcounts (4 ceil(N K / 32)), K = max out-degree + 1
  const size_t smem = sizeof(int) * (4 * (size_t)std::max(lat->max_lvl_nodes, 1) +
                                     4 * (((size_t)std::max(lat->max_lvl_nodes, 1) * (lat->max_out_deg + 1) + 31) / 32));
  if (smem > (size_t)kMaxDynamicSmem)
    return fail(ctx, GTNB_ERR_UNSUPPORTED, "exact_ties: graph operand too large");
  if (smem > 48 * 1024) {
    int rc = ensure_max_smem(ctx, (const void*)lattice_relax_order_kernel);
    if (rc) return rc;
  }
  int32_t* rank = nullptr; // per lattice arc, only needed until the rows are sorted
  int rc = dev_alloc(ctx, &rank, lat->tot_A);
  if (rc) return rc;
  GTNB_LAUNCH(ctx, "relax_order",
              lattice_relax_order_kernel<<<lat->B, kOrderThreads, smem, ctx->stream>>>(
                  lat->meta, lat->sg_flags, lat->sg_in_ptr, lat->sg_in_src, lat->sg_in_label, lat->sg_out_pos,
                  lat->sg_start_rank, lat->alive, lat->alive_words, lat->max_T, lat->max_out_deg + 1,
                  lat->lvl_node_ptr, lat->row_ptr, rank, lat->acc_nodes));
  int capN = 1;
  for (int b = 0; b < lat->B; b++) capN = std::max(capN, lat->meta_h[b].cap_N);
  dim3 grid(std::min((capN + 255) / 256, 4096), lat->B);
  GTNB_LAUNCH(ctx, "sort_rows",
              lattice_sort_rows_kernel<<<grid, 256, 0, ctx->stream>>>(lat->meta, lat->row_ptr, rank, lat->arcs, lat->gi,
                                                                       lat->arc_grad));
  dev_free(ctx, rank);
  return GTNB_OK;
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
