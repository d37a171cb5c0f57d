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

/* the numerator graph an asynchronous call's prepare kernel describes (gtnb_ctc_loss_async, gtnb_ngram_ctc_loss_async,
 * gtnb_asg_loss_async) */
enum class AsyncGraph { Ctc, Ngram, Asg };

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
 * G = Ngram / Asg (gtnb_ngram_ctc_loss_async, gtnb_asg_loss_async): the same, for the numerators the build kernels of
 * k_ngram.cu write (the dims of ngram_ctc_loss_call / asg_loss_ex_call): n-gram sg_N = 2U + 2, sg_A = L + (L - 1) +
 * skips + min(L, 2); ASG sg_N = U + 1, sg_A = 2U, n_accept = (U > 0).  kstatus is [2B] there (denominator, numerator),
 * both halves set to 0.
 */
template <AsyncGraph G = AsyncGraph::Ctc>
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
  m.T = Tb;
  if constexpr (G == AsyncGraph::Ctc) {
    m.n_accept = L >= 2 ? 2 : 1;
    m.sg_N = L;
    m.sg_A = L + (L - 1) + skips;
  } else if constexpr (G == AsyncGraph::Ngram) {
    m.n_accept = L >= 2 ? 2 : 1;
    m.sg_N = L + 1;
    m.sg_A = L + (L - 1) + skips + (L < 2 ? L : 2);
  } else {
    m.n_accept = U > 0 ? 1 : 0;
    m.sg_N = U + 1;
    m.sg_A = 2 * U;
  }
  m.tgt_off = b * S;
  meta[b] = m;
  small[b] = b * S;
  small[B + b] = U;
  small[2 * B + b] = Tb;
  deltas[b] = -1.0f;
  valid[b] = ok;
  kstatus[b] = 0;
  if constexpr (G != AsyncGraph::Ctc) kstatus[B + b] = 0;
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

/*
 * gtnb_ngram_ctc_loss_async / gtnb_asg_loss_async, after both forward sweeps (the numerator's on the side stream waited
 * for): kstatus[b] |= kstatus[B + b] | !valid[b], the flag of utterance b from then on, and T_bwd[b] = T_b, or 0 for a
 * flagged utterance, so that the denominator's backward kernel (which returns for T_b < 1) adds nothing for it to the
 * shared transition gradient.  An utterance with T_b = 0 gets den[b] = NaN: its loss is NaN, as the synchronous call
 * gives it (run_criterion), where the trellis would score the empty linear graph log C.  One thread per utterance.
 */
__global__ void __launch_bounds__(256) trellis_async_gate_kernel(
    int B, const int32_t* __restrict__ T_fwd, const int32_t* __restrict__ valid, int32_t* __restrict__ kstatus,
    int32_t* __restrict__ T_bwd, float* __restrict__ den) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int flagged = (kstatus[b] | kstatus[B + b]) != 0 || !valid[b];
  const int Tb = T_fwd[b];
  kstatus[b] = flagged;
  T_bwd[b] = flagged ? 0 : Tb;
  if (Tb == 0) den[b] = CUDART_NAN_F;
}

/*
 * The numerator's arc gradients into the transition gradient, utterance by utterance: dst[map[o + a]] += src[o + a]
 * for a < meta[b].sg_A, o = meta[b].grad_graph_off, for every utterance whose kstatus (the gate's) is 0.  Only the
 * arcs the build kernel wrote are read: the slabs are laid out at the bounds, and the tail of a slab past the
 * utterance's own arcs holds whatever the workspace held.  One CTA per utterance.
 */
__global__ void __launch_bounds__(256) trellis_async_scatter_kernel(
    const GraphMeta* __restrict__ meta, const int32_t* __restrict__ kstatus, const int32_t* __restrict__ map,
    const float* __restrict__ src, float* __restrict__ dst) {
  const int b = blockIdx.x;
  if (kstatus[b]) return;
  const long long o = meta[b].grad_graph_off;
  const int n = meta[b].sg_A;
  for (int a = threadIdx.x; a < n; a += blockDim.x) atomicAdd(dst + map[o + a], src[o + a]);
}

/*
 * gtnb_ctc_align_async / gtnb_ngram_ctc_align_async / gtnb_asg_align_async, after the tropical forward and the trace
 * (k_implicit.cu), which wrote the score, the path's labels and its arcs, and raised kstatus bit 1 (a non-finite
 * value) or bit 2 (kTrTie: a tie on the traced path).  status[b]: 2 for an utterance the prepare kernel refused,
 * 1 for bit 1, 3 for bit 2, else 0.  Status 1 and 2 give a NaN score and -1 rows.  tokens[b][t]: the target position
 * of the arc traced at frame t, found from the numbering of the build kernel G names:
 *   Ctc    arc ids in ctcGraph's creation order, the arcs of node l in [in_ptr[l], in_ptr[l+1]); position (l - 1) / 2
 *          for odd l, -1 (blank) for even l;
 *   Ngram  the in-entry index is the arc id, node n is CTC node l = n - 1, then as Ctc;
 *   Asg    arc a enters node a / 2 + 1: position a / 2.
 * An arc of -1 (beyond T_b, no accepting path) gives -1.  paths, tokens, status nullable.  One CTA per utterance.
 */
template <AsyncGraph G>
__global__ void __launch_bounds__(256) align_async_finalize_kernel(
    int T_out, const GraphMeta* __restrict__ meta, const int32_t* __restrict__ sg_in_ptr,
    const int32_t* __restrict__ kstatus, const int32_t* __restrict__ valid, const int32_t* __restrict__ arcs,
    int32_t* __restrict__ paths, int32_t* __restrict__ tokens, float* __restrict__ scores,
    int32_t* __restrict__ status) {
  const int b = blockIdx.x;
  const int ks = kstatus[b];
  const int st = !valid[b] ? 2 : (ks & 1) ? 1 : (ks & 2) ? 3 : 0;
  const bool flagged = st == 1 || st == 2;
  if (threadIdx.x == 0) {
    if (flagged) scores[b] = CUDART_NAN_F;
    if (status) status[b] = st;
  }
  const GraphMeta m = meta[b];
  const int32_t* ip = sg_in_ptr + m.sg_node_base;
  const long long row = (long long)b * T_out;
  for (int t = threadIdx.x; t < T_out; t += blockDim.x) {
    if (flagged && paths) paths[row + t] = -1;
    if (!tokens) continue;
    const int a = flagged ? -1 : arcs[row + t];
    int u = -1;
    if (a >= 0) {
      if constexpr (G == AsyncGraph::Asg) {
        u = a / 2;
      } else {
        int lo = 0, hi = m.sg_N - 1; // the last node n with in_ptr[n] <= a: the one whose in-entries hold a
        while (lo < hi) {
          const int mid = (lo + hi + 1) / 2;
          if (ip[mid] <= a)
            lo = mid;
          else
            hi = mid - 1;
        }
        const int l = G == AsyncGraph::Ngram ? lo - 1 : lo;
        u = (l & 1) ? (l - 1) / 2 : -1;
      }
    }
    tokens[row + t] = u;
  }
}

/*
 * gtnb_viterbi_transitions_async / gtnb_viterbi_dense_async, before the sweep: lens[b] = T_b (input_lens[b], or T when
 * input_lens is NULL), valid[b] = whether T_b lies in [0, T].  An invalid utterance is swept with lens[b] = 0, so no
 * kernel indexes with its length.  kstatus[b] = 0.  One thread per utterance.
 */
__global__ void __launch_bounds__(256) decode_async_prepare_kernel(int B, int T, const int32_t* __restrict__ input_lens,
                                                                   int32_t* __restrict__ lens,
                                                                   int32_t* __restrict__ valid,
                                                                   int32_t* __restrict__ kstatus) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int Tb = input_lens ? input_lens[b] : T;
  const int ok = Tb >= 0 && Tb <= T;
  lens[b] = ok ? Tb : 0;
  valid[b] = ok;
  kstatus[b] = 0;
}

/*
 * The asynchronous decoders, after the sweep and its trace: status[b] = 2 for an utterance the prepare kernel refused,
 * else, for T_b > 0, 1 for kstatus bit 1 (a non-finite value), 3 for bit 2 (a tie), else 0.  T_b = 0 is 0 whatever
 * the kernel raised: no frame is decoded, and the synchronous decoders ignore the status there too.  Status 1 and 2
 * give a NaN score and -1 rows of paths and arcs (both nullable, [B][T_out]).  status nullable.  One CTA per
 * utterance.
 */
__global__ void __launch_bounds__(256) decode_async_finalize_kernel(
    int T_out, const int32_t* __restrict__ lens, const int32_t* __restrict__ kstatus,
    const int32_t* __restrict__ valid, int32_t* __restrict__ paths, int32_t* __restrict__ arcs,
    float* __restrict__ scores, int32_t* __restrict__ status) {
  const int b = blockIdx.x;
  const int ks = lens[b] > 0 ? kstatus[b] : 0;
  const int st = !valid[b] ? 2 : (ks & 1) ? 1 : (ks & 2) ? 3 : 0;
  if (threadIdx.x == 0) {
    if (st == 1 || st == 2) scores[b] = CUDART_NAN_F;
    if (status) status[b] = st;
  }
  if (st != 1 && st != 2) return;
  const long long row = (long long)b * T_out;
  for (int t = threadIdx.x; t < T_out; t += blockDim.x) {
    if (paths) paths[row + t] = -1;
    if (arcs) arcs[row + t] = -1;
  }
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

int launch_trellis_async_prepare(
    gtnb_ctx* ctx, bool asg, int B, int S, int T, int C, const GraphMeta& m0, const GraphMeta& m1,
    const int32_t* input_lens, const int32_t* targets, const int32_t* target_lens, GraphMeta* meta, int32_t* small,
    float* deltas, int32_t* valid, int32_t* kstatus) {
  if (B <= 0) return GTNB_OK;
  if (asg)
    GTNB_LAUNCH(ctx, "trellis_async_prepare", ctc_async_prepare_kernel<AsyncGraph::Asg><<<(B + 7) / 8, 256, 0,
                ctx->stream>>>(B, S, T, C, m0, m1, input_lens, targets, target_lens, meta, small, deltas, valid,
                               kstatus));
  else
    GTNB_LAUNCH(ctx, "trellis_async_prepare", ctc_async_prepare_kernel<AsyncGraph::Ngram><<<(B + 7) / 8, 256, 0,
                ctx->stream>>>(B, S, T, C, m0, m1, input_lens, targets, target_lens, meta, small, deltas, valid,
                               kstatus));
  return GTNB_OK;
}

int launch_trellis_async_gate(gtnb_ctx* ctx, int B, const int32_t* T_fwd, const int32_t* valid, int32_t* kstatus,
                              int32_t* T_bwd, float* den) {
  if (B <= 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "trellis_async_gate", trellis_async_gate_kernel<<<(B + 255) / 256, 256, 0, ctx->stream>>>(
      B, T_fwd, valid, kstatus, T_bwd, den));
  return GTNB_OK;
}

int launch_trellis_async_scatter(gtnb_ctx* ctx, int B, const GraphMeta* meta, const int32_t* kstatus,
                                 const int32_t* map, const float* src, float* dst) {
  if (B <= 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "trellis_async_scatter", trellis_async_scatter_kernel<<<B, 256, 0, ctx->stream>>>(
      meta, kstatus, map, src, dst));
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

int launch_align_async_finalize(gtnb_ctx* ctx, AlignCriterion kind, int B, int T_out, const GraphMeta* meta,
                                const int32_t* sg_in_ptr, const int32_t* kstatus, const int32_t* valid,
                                const int32_t* arcs, int32_t* paths, int32_t* tokens, float* scores,
                                int32_t* status) {
  if (B <= 0) return GTNB_OK;
#define GTNB_ALIGN_FINALIZE(G_)                                                                                   \
  GTNB_LAUNCH(ctx, "align_async_finalize", align_async_finalize_kernel<G_><<<B, 256, 0, ctx->stream>>>(           \
      T_out, meta, sg_in_ptr, kstatus, valid, arcs, paths, tokens, scores, status))
  switch (kind) {
    case AlignCriterion::Ctc: GTNB_ALIGN_FINALIZE(AsyncGraph::Ctc); break;
    case AlignCriterion::Ngram: GTNB_ALIGN_FINALIZE(AsyncGraph::Ngram); break;
    case AlignCriterion::Asg: GTNB_ALIGN_FINALIZE(AsyncGraph::Asg); break;
  }
#undef GTNB_ALIGN_FINALIZE
  return GTNB_OK;
}

int launch_decode_async_prepare(gtnb_ctx* ctx, int B, int T, const int32_t* input_lens, int32_t* lens,
                                int32_t* valid, int32_t* kstatus) {
  if (B <= 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "decode_async_prepare", decode_async_prepare_kernel<<<(B + 255) / 256, 256, 0, ctx->stream>>>(
      B, T, input_lens, lens, valid, kstatus));
  return GTNB_OK;
}

int launch_decode_async_finalize(gtnb_ctx* ctx, int B, int T_out, const int32_t* lens, const int32_t* kstatus,
                                 const int32_t* valid, int32_t* paths, int32_t* arcs, float* scores,
                                 int32_t* status) {
  if (B <= 0) return GTNB_OK;
  GTNB_LAUNCH(ctx, "decode_async_finalize", decode_async_finalize_kernel<<<B, 256, 0, ctx->stream>>>(
      T_out, lens, kstatus, valid, paths, arcs, scores, status));
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
