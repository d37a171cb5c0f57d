/*
 * k_ctc.cu -- build the CTC target graphs of a minibatch directly in HBM.
 *
 * The reference builds one Graph per utterance on the host inside the timed
 * loop (ctcGraph, benchmarks/ctc.cpp:40-58: 2U+1 nodes; per node a self-loop,
 * a step arc from l-1, and for odd l a skip arc from l-2 unless the label
 * repeats; accept = last two nodes; arcSort()).  Here one CTA per utterance
 * writes the same graph straight into the small-graph tables compose reads
 * (in-arc lists ordered by (source, position in the source's out list), arc ids
 * in the reference's creation order), so no per-utterance host work is left.
 */
#include <algorithm>

#include "gtnb_ptx.h"

namespace gtnb {

namespace {

__global__ void __launch_bounds__(256) ctc_build_kernel(
    const GraphMeta* __restrict__ meta,
    const int32_t* __restrict__ targets,
    const int32_t* __restrict__ tgt_off,
    const int32_t* __restrict__ tgt_len,
    int blank,
    int C,
    uint8_t* __restrict__ sg_flags,
    int32_t* __restrict__ sg_in_ptr,
    int32_t* __restrict__ sg_in_src,
    int32_t* __restrict__ sg_in_label,
    int32_t* __restrict__ sg_in_arc,
    float* __restrict__ sg_in_w,
    int32_t* __restrict__ sg_ilabel,
    int32_t* __restrict__ sg_olabel,
    int32_t* __restrict__ acc_nodes) {
  GTNB_STATIC_SMEM(int, scan, 256);
  GTNB_STATIC_SMEM(int, carry_box, 1);
  int& carry = carry_box[0];
  const int b = blockIdx.x;
  const GraphMeta m = meta[b];
  const int tid = threadIdx.x;
  const int U = tgt_len[b];
  const int L = 2 * U + 1;
  const int32_t* tg = targets + tgt_off[b];
  uint8_t* fl = sg_flags + m.sg_node_base;
  int32_t* ip = sg_in_ptr + m.sg_node_base;
  int32_t* is = sg_in_src + m.sg_arc_base;
  int32_t* il = sg_in_label + m.sg_arc_base;
  int32_t* ia = sg_in_arc + m.sg_arc_base;
  float* iw = sg_in_w + m.sg_arc_base;
  int32_t* lab_i = sg_ilabel + m.sg_arc_base;
  int32_t* lab_o = sg_olabel + m.sg_arc_base;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int l0 = 0; l0 < L; l0 += 256) {
    const int l = l0 + tid;
    int label = blank, narcs = 0;
    bool skip = false;
    if (l < L) {
      const int idx = (l - 1) / 2;
      label = (l & 1) ? tg[idx] : blank;
      skip = (l & 1) && l > 1 && label != tg[idx - 1];
      narcs = 1 + (l > 0 ? 1 : 0) + (skip ? 1 : 0);
    }
    scan[tid] = narcs;
    __syncthreads();
    for (int o = 1; o < 256; o <<= 1) {
      const int v = tid >= o ? scan[tid - o] : 0;
      __syncthreads();
      scan[tid] += v;
      __syncthreads();
    }
    const int base = carry + scan[tid] - narcs;
    if (l < L) {
      fl[l] = (uint8_t)((l == 0 ? 1 : 0) | ((l == L - 1 || l == L - 2) ? 2 : 0));
      ip[l] = base;
      const int mlab = (label >= 0 && label < C) ? label : -1;
      const int self_id = base, step_id = base + 1, skip_id = base + 2;
      int e = base;
      if (skip) {
        is[e] = l - 2;
        ia[e] = skip_id;
        il[e] = mlab;
        iw[e] = 0.0f;
        e++;
      }
      if (l > 0) {
        is[e] = l - 1;
        ia[e] = step_id;
        il[e] = mlab;
        iw[e] = 0.0f;
        e++;
      }
      is[e] = l;
      ia[e] = self_id;
      il[e] = mlab;
      iw[e] = 0.0f;
      for (int k = 0; k < narcs; k++) {
        lab_i[base + k] = label;
        lab_o[base + k] = label;
      }
    }
    __syncthreads();
    if (tid == 255) carry += scan[255];
    __syncthreads();
  }
  if (tid == 0) {
    ip[L] = carry;
    int32_t* acc = acc_nodes + m.acc_base;
    if (L >= 2) {
      acc[0] = L - 2;
      acc[1] = L - 1;
    } else {
      acc[0] = 0;
    }
  }
}

/*
 * gtnb_ctc_loss_async, before the sweeps: the descriptors and the small arrays of the batch, built on the device from
 * the caller's padded targets.  One warp per utterance.  The slabs were laid out on the host at the bounds (U = S,
 * T_b = T for every utterance), so they sit at a constant stride: every base of utterance b is m0's plus b times the
 * step to m1 (m1 = m0 when B = 1).  The per-utterance fields are what composed_alloc and parse_targets give for the
 * utterance's own target: T = T_b, L = T_b + 1, sg_N = 2U + 1, sg_A = 3U + 1 + skips, n_accept, tgt_off = b * S.
 * small = [offsets | lens | T] (Targets::meta, with row b of the padded targets at b * S); deltas = -1 (subtract's
 * gradFunc, read by the implicit backward).  An utterance with U outside [0, S], T_b outside [0, T] or a label
 * outside [0, C) gets valid = 0 and is swept as U = 0, T_b = 0, so that no kernel indexes with its lengths or labels;
 * the finalize kernel reports it.  kstatus, the sweeps' non-finite flags, starts at 0.
 */
__global__ void __launch_bounds__(256) ctc_async_prepare_kernel(
    int B, int S, int T, int C, const GraphMeta m0, const GraphMeta m1,
    const int32_t* __restrict__ input_lens, // nullable: T each
    const int32_t* __restrict__ targets, // [B][S]
    const int32_t* __restrict__ target_lens,
    GraphMeta* __restrict__ meta, int32_t* __restrict__ small, float* __restrict__ deltas,
    int32_t* __restrict__ valid, int32_t* __restrict__ kstatus) {
  const int b = blockIdx.x * 8 + (int)(threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= B) return;
  int U = target_lens[b];
  int Tb = input_lens ? input_lens[b] : T;
  int ok = U >= 0 && U <= S && Tb >= 0 && Tb <= T;
  int skips = 0;
  if (ok) {
    const int32_t* y = targets + (long long)b * S;
    for (int u0 = 0; u0 < U; u0 += 32) { // (U is the warp's own: every lane runs the same trips)
      const int u = u0 + lane;
      const int32_t v = u < U ? y[u] : 0;
      ok &= __ballot_sync(0xffffffffu, u < U && (unsigned)v >= (unsigned)C) == 0u;
      skips += __popc(__ballot_sync(0xffffffffu, u > 0 && u < U && v != y[u - 1]));
    }
  }
  if (lane != 0) return;
  if (!ok) {
    U = 0;
    Tb = 0;
    skips = 0;
  }
  const int L = 2 * U + 1;
  GraphMeta m = m0;
  m.node_base += b * (m1.node_base - m0.node_base);
  m.arc_base += b * (m1.arc_base - m0.arc_base);
  m.lvl_base += b * (m1.lvl_base - m0.lvl_base);
  m.acc_base += b * (m1.acc_base - m0.acc_base);
  m.sg_node_base += b * (m1.sg_node_base - m0.sg_node_base);
  m.sg_arc_base += b * (m1.sg_arc_base - m0.sg_arc_base);
  m.emis_off += b * (m1.emis_off - m0.emis_off);
  m.grad_graph_off += b * (m1.grad_graph_off - m0.grad_graph_off);
  m.L = Tb + 1;
  m.n_accept = L >= 2 ? 2 : 1;
  m.T = Tb;
  m.sg_N = L;
  m.sg_A = L + (L - 1) + skips;
  m.tgt_off = b * S;
  meta[b] = m;
  small[b] = b * S;
  small[B + b] = U;
  small[2 * B + b] = Tb;
  deltas[b] = -1.0f;
  valid[b] = ok;
  kstatus[b] = 0;
}

/*
 * gtnb_ctc_loss_async, after the sweeps: losses[b] = sum_k z[zp * b + k] - s[b], added in the order of the host loop
 * of ctc_loss_run, so the float32 loss is the synchronous call's.  status[b]: 2 for an utterance the prepare kernel
 * refused, 1 where a sweep met a non-finite value (kstatus), else 0.  A flagged utterance gets a NaN loss and, when
 * grad is set, a zero gradient (row_words 32-bit words per utterance).  One CTA per utterance.
 */
__global__ void __launch_bounds__(256) ctc_async_finalize_kernel(
    int zp, const float* __restrict__ z, const float* __restrict__ s, const int32_t* __restrict__ kstatus,
    const int32_t* __restrict__ valid, float* __restrict__ losses, int32_t* __restrict__ status,
    uint32_t* __restrict__ grad, long long row_words) {
  const int b = blockIdx.x;
  const int st = !valid[b] ? 2 : kstatus[b] != 0 ? 1 : 0;
  if (threadIdx.x == 0) {
    float zb = 0.0f;
    for (int k = 0; k < zp; k++) zb += z[(long long)zp * b + k];
    losses[b] = st ? CUDART_NAN_F : zb - s[b];
    if (status) status[b] = st;
  }
  if (st && grad)
    for (long long i = threadIdx.x; i < row_words; i += blockDim.x) grad[b * row_words + i] = 0u;
}

} // namespace

#ifndef GTNB_HOST_EMU

int launch_ctc_async_prepare(
    gtnb_ctx* ctx, int B, int S, int T, int C, const GraphMeta& m0, const GraphMeta& m1, const int32_t* input_lens,
    const int32_t* targets, const int32_t* target_lens, GraphMeta* meta, int32_t* small, float* deltas,
    int32_t* valid, int32_t* kstatus) {
  if (B <= 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "ctc_async_prepare", ctc_async_prepare_kernel<<<(B + 7) / 8, 256, 0, ctx->stream>>>(
      B, S, T, C, m0, m1, input_lens, targets, target_lens, meta, small, deltas, valid, kstatus));
  return GTNB_OK;
}

int launch_ctc_async_finalize(
    gtnb_ctx* ctx, int B, int zp, const float* z, const float* s, const int32_t* kstatus, const int32_t* valid,
    float* losses, int32_t* status, void* grad, long long row_words) {
  if (B <= 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "ctc_async_finalize", ctc_async_finalize_kernel<<<B, 256, 0, ctx->stream>>>(
      zp, z, s, kstatus, valid, losses, status, static_cast<uint32_t*>(grad), row_words));
  return GTNB_OK;
}

int launch_ctc_build(
    gtnb_ctx* ctx, gtnb_lattice* lat, const int32_t* targets_dev, const int32_t* tgt_off_dev,
    const int32_t* tgt_len_dev, int blank) {
  if (lat->B == 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "ctc_build", ctc_build_kernel<<<lat->B, 256, 0, ctx->stream>>>(
      lat->meta, targets_dev, tgt_off_dev, tgt_len_dev, blank, lat->C, lat->sg_flags, lat->sg_in_ptr,
      lat->sg_in_src, lat->sg_in_label, lat->sg_in_arc, lat->sg_in_w, lat->sg_ilabel,
      lat->sg_olabel, lat->acc_nodes));
  return GTNB_OK;
}

#endif // GTNB_HOST_EMU

} // namespace gtnb

#ifndef GTNB_HOST_EMU
namespace gtnb {
namespace {
__global__ void scatter_add_kernel(float* __restrict__ dst, const int32_t* __restrict__ idx,
                                   const float* __restrict__ src, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    atomicAdd(&dst[idx[i]], src[i]);
}
__global__ void gather_kernel(float* __restrict__ dst, const int32_t* __restrict__ idx,
                              const float* __restrict__ src, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    if (idx[i] >= 0) dst[i] = src[idx[i]];
}
__global__ void sub_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] - b[i];
}
} // namespace

/* dst[idx[i]] += src[i]: the gradFunc of the host-composed (forced alignment x transitions)
 * graph (compose.cpp:496-518) applied on the device */
int launch_scatter_add(gtnb_ctx* ctx, float* dst, const int32_t* idx, const float* src, long long n) {
  if (n <= 0) return GTNB_OK;
  int blocks = (int)std::min<long long>((n + 255) / 256, 1024);
  GTNB_LAUNCH(ctx, "scatter_add", scatter_add_kernel<<<blocks, 256, 0, ctx->stream>>>(dst, idx, src, n));
  return GTNB_OK;
}

/* dst[i] = src[idx[i]] where idx[i] >= 0: device-resident arc weights into a graph operand's in-arc table */
int launch_gather(gtnb_ctx* ctx, float* dst, const int32_t* idx, const float* src, long long n) {
  if (n <= 0) return GTNB_OK;
  int blocks = (int)std::min<long long>((n + 255) / 256, 1024);
  GTNB_LAUNCH(ctx, "gather", gather_kernel<<<blocks, 256, 0, ctx->stream>>>(dst, idx, src, n));
  return GTNB_OK;
}

int launch_sub(gtnb_ctx* ctx, const float* a, const float* b, float* out, int n) {
  if (n <= 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "sub", sub_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(a, b, out, n));
  return GTNB_OK;
}
} // namespace gtnb
#endif // GTNB_HOST_EMU
