/*
 * k_bidir.cu -- the criterion's hot kernel since round 2: forwardScore(intersect(g, emissions)), its
 * backward, forwardScore(emissions) and its backward -- everything gtnb_ctc_loss needs after the
 * target graphs exist -- in ONE launch, with the serial dependence over T cut in half.
 *
 * The implicit-lattice sweeps of k_implicit.cu run the frames twice in a row (alpha front to back,
 * then shortestDistanceGrad back to front: 2T dependent steps per utterance, and at B = 256 the step
 * time IS that chain's latency).  Here each utterance gets a thread-block cluster of two CTAs that run
 * at the same time and meet in the middle:
 *
 *   CTA A (cluster rank 0)  alpha_s[u] = logsumexp over in-arcs (i -> u, w) of alpha_{s-1}[i] + w + e[s-1][label(u)]
 *                           for levels s = 1 .. T   (shortest.cpp:102-136 on the implicit lattice)
 *   CTA B (cluster rank 1)  beta_s[u]  = logsumexp over out-arcs (u -> v, w) of w + e[s][label(v)] + beta_{s+1}[v]
 *                           for levels s = T .. 1   (beta_T = 0 on accept nodes)
 *
 * With M = T/2 rounded up to a multiple of 8 (B starts later: it gets the shorter first phase), A saves alpha_1..alpha_M and B saves beta_T..beta_{M+1}
 * (phase 1, T/2 dependent steps each, concurrently); one barrier.cluster later A continues through
 * levels M+1..T reading B's saved beta, B through levels M..1 reading A's saved alpha (phase 2), and the
 * node posterior gamma_s[u] = exp(alpha_s[u] + beta_s[u] - Z) is formed ON THE FLY, off the serial
 * chain.  That posterior is exactly what shortestDistanceGrad + compose's gradFunc deliver to the
 * emissions (shortest.cpp:33-82, compose.cpp:496-518): the arc gradients into lattice node (u, s) sum
 * to its node gradient, and all of them land on emission (s-1, label(u)).  Z = logsumexp_u(alpha + beta)
 * at the meeting level equals forwardScore of the lattice.  The dependent chain is T steps instead of
 * 2T, and HBM traffic does not grow: each half of the saved scores is written once and read once.
 *
 * Inside a CTA (warp-specialised):
 *   node warps    the recursion.  Two variants (launch_bidir_ctc picks):
 *                 - PAIR (gtnb_ctc_loss at C = 64 / 128): the graphs are CTC target graphs, taken from
 *                   the targets themselves (no ctc_build launch); thread t owns label 2t-1 AND blank 2t, keeps
 *                   their scores in registers, reads its neighbour pair with one LDS.64 (A) / one LDS (B), writes
 *                   one STS.64 (A) / STS (B) and saves the label's score alone (one STG); the blank's two-term
 *                   logsumexp costs 2 MUFU, the label's 3 (max + lg2(1 +
 *                   two terms)), the blank's posterior is never formed (complement label).  <= 4 warps, 26 / 31
 *                   SASS instructions per PAIR and level (the one-node-per-thread kernels: 2 x 19 / 2 x 24).
 *                 - one node per thread (any graph in the envelope; <= 7 warps): per level 3 LDS of the neighbours'
 *                   scores (absent arcs read a slot that holds a large negative finite number, so there is no
 *                   -inf / NaN special casing on the chain), one STS, one named barrier.
 *                 Scores are kept in log2 units (emissions are multiplied by log2(e) on the way in), which removes
 *                 the multiply from every exp and log, and are RENORMALISED every 8 levels by an integer (see
 *                 publish_block_max): the posteriors come out closer to a float64 evaluation than the
 *                 reference's own fp32 gradient (DESIGN.md "Tolerances").
 *   producer warp cp.async.bulk (TMA 1-D bulk copies, mbarrier complete_tx) of 8 emission frames at a time into
 *                 a 4-stage ring and, in phase 2, of the partner's 8 saved score rows (+ that block's offset)
 *                 into a 2-stage ring.
 *   helper warps  (4) own two rows of a block each: row logsumexp of the emissions (forwardScore(emissions) and
 *                 its softmax gradient, k_linear.cu's job before) with LDS.128 and half-warp shuffles, the
 *                 posteriors summed by label -- the node threads write theirs into 4 slots per label of a
 *                 separate block, so a label's mass is one LDS.128; labels on 5..16 nodes sit behind the slots and
 *                 are summed by the row's 16 lanes together; the label with the MOST nodes (CTC: blank) stores
 *                 nothing: its mass is the level's mass minus everybody else's; no floating-point atomics
 *                 anywhere -- and the finished gradient row leaves as one 16-byte store per lane.
 *
 * What bounds it: at the benchmark's shape (B = 256, T = 1000, C = 64, U = 100) node-warp variants whose chains
 * differ widely (7 warps and a barrier, 4 warps and a barrier, and a since-removed one of 1 warp and no barrier,
 * DESIGN.md) all took about the same time; what they share is the saved-score traffic, 229 MB written in phase 1
 * and read back in phase 2 at the fixed pitch, about two thirds of everything the kernel moves (counted from the
 * shapes).  Saving the PAIR kernels' label scores alone (the blank's are read only at the meeting level) halved that
 * traffic and cut the kernel from 0.376 to 0.315 ms (medians, H100 80GB HBM3 at a 400 W limit, DESIGN.md).  How the rest of a level's time splits has not
 * been measured; the dependent chain of a level, several CTAs deep on an SM, is the likeliest bound
 * (scripts/ubench/chain*.cu time its pieces).
 *
 * Numerics: gamma's exponent is evaluated as ((x - Zh) + y) - zsub with x the larger of alpha/beta: both
 * subtractions are exact or nearly so (Sterbenz), so the posterior carries only the rounding error the
 * recursions themselves accumulated -- and those run on renormalised scores (|score| < ~100, ulp 8e-6
 * instead of 5e-4).  tests/test_gpu_config_parity.py holds the gradient to at least as close to a float64
 * evaluation as the reference's own fp32 gradient is (DESIGN.md "Tolerances").
 *
 * Valid when every weight is finite (|x| < 1e29): otherwise a status bit is raised and the caller repeats
 * the batch through the materialised path, which reproduces the reference's inf / NaN propagation arc by
 * arc.  Requires: <= 224 graph nodes, in- and out-degree <= 3, one label per node, every arc weight 0 (the CTC
 * target graphs of gtnb_ctc_loss, its only caller), C a multiple of 4 and <= 128, 16-byte aligned emissions.
 * Anything else takes k_implicit.cu.
 *
 * Element type E (gtnb_ctc_loss_ex): the emissions and the gradient are float32, bfloat16 or fp16; only the edges
 * change -- the TMA copies move kBlk * C * sizeof(E) bytes, the node warps widen their emission with one LDS.U16
 * (bf16: a shift, fp16: a conversion), the helper warps load four labels as 8 bytes and store four rounded gradients
 * as 8 bytes.  Scores, renormalisation, logsumexps, Z and posteriors stay float32, so a 16-bit call returns exactly
 * the float32 kernel's result on the widened emissions, its gradient rounded to E.  16-bit needs C % 8 == 0.
 */
#include <algorithm>

#include "gtnb_ptx.h"

namespace gtnb {

namespace bidir {

constexpr int kMaxNodes = 256; // table capacity
constexpr int kMaxNodeWarps = 7; // graph nodes per utterance: at most 224, one per thread (4 CTAs of 12 warps per SM at 40 registers)
constexpr int kMaxPairWarps = 4; // PAIR kernels: two nodes per thread, (U + 1) <= 112 pairs
constexpr int kRowF = 264; // floats per chain row in shared memory
constexpr int kDummy = 256; // slot of every chain row that holds kNeg (absent arcs point here)
constexpr int kBlk = 8; // frames per block (one TMA copy, one helper pass, one renormalisation)
constexpr int kSE = 4; // emission stages (kSE, kSO, kSG are powers of two: stage = v & (k - 1), parity = (v / k) & 1)
constexpr int kSO = 2; // stages of the partner's saved scores
constexpr int kSG = 2; // posterior blocks between the node warps and the helper warps
constexpr int kHelpers = 4; // helper warps
// (Tried and dropped: gathering the nodes with <= 2 neighbours -- every CTC blank -- in warps of their own that take a
// two-score logsumexp with half the SFU work.  Slower for the loss-only sweep at config 2 on an earlier GPU target (not
// re-measured on the H100): strided saves / stage reads and a branch per level cost more than the SFU cycles saved.)
constexpr int kSlots = 4; // posterior slots per label in a row of the helpers' block (one LDS.128)
constexpr int kMaxHeavy = 4; // labels carried by more than kSlots nodes that get the cooperative sum
constexpr float kNeg = -1.0e30f; // "this node does not exist" (finite: absorbs every later add)
constexpr float kHuge = 1.0e29f; // inputs at or above this magnitude take the exact (materialised) path
constexpr int kIntMin = -2147483647 - 1;
// FX kernels (C == 64 or 128): the saved-score rows in HBM, the rows of their shared-memory stages and the
// overflow area of a posterior row all have this many floats, whatever the utterance's node count -- which makes
// every per-level address of the node warps base + compile-time constant (no pointer arithmetic on the chain)
constexpr int kFixedPitch = 32 * kMaxNodeWarps;
// PAIR kernels: floats per saved LABEL row (one per pair, <= 112 pairs); see pair_role for the block layout
constexpr int kHalfPitch = kFixedPitch / 2;

struct Layout {
  int off_ring, off_e, off_o, off_g, off_od, off_seg, off_perm, off_nlab, off_hlist, off_red, off_redi,
      off_bar;
  int e_stage_bytes, o_stage_bytes, g_block_bytes;
  int pg; // floats per row of a posterior block: kSlots per label, then the overflow positions
  int total;
};

inline Layout make_layout(int C, int max_pitch, int esize = 4) { // esize: bytes per emission element
  Layout L;
  int off = 0;
  auto take = [&](int bytes) {
    int at = off;
    off += (bytes + 127) & ~127;
    return at;
  };
  L.off_ring = take(2 * kRowF * 4);
  L.e_stage_bytes = kBlk * C * esize;
  L.off_e = take(kSE * L.e_stage_bytes);
  L.o_stage_bytes = kBlk * max_pitch * 4;
  // the out-arc scratch of CTA B's set-up (cnt[256] + dst[768] + w[768]) aliases the score stages
  L.off_o = take(std::max(kSO * L.o_stage_bytes, (kMaxNodes + 6 * kMaxNodes) * 4));
  L.pg = kSlots * C + max_pitch;
  L.g_block_bytes = kBlk * L.pg * 4;
  L.off_g = take(kSG * L.g_block_bytes);
  L.off_od = take(kSO * 16);
  L.off_seg = take(C * 4);
  L.off_perm = take(kMaxNodes * 2); // u16: byte offset of a node's posterior word in a row
  L.off_nlab = take(kMaxNodes); // s8: a node's label (-1: no in-arcs)
  L.off_hlist = take((kMaxHeavy + 1) * 4 + kMaxHeavy * 12);
  L.off_red = take(32 * 4);
  L.off_redi = take(8 * 4);
  L.off_bar = take((2 * kSE + 2 * kSO + 2 * kSG + 1) * 8);
  L.total = off;
  return L;
}

struct Params {
  const GraphMeta* meta;
  const uint8_t* sg_flags;
  const int32_t* sg_in_ptr;
  const int32_t* sg_in_src;
  const int32_t* sg_in_label;
  const float* sg_in_w;
  const void* emissions; // [B][T][C] of the kernel's element type E
  float* saved; // [node_base + f * pitch + u]: alpha_{f+1} for f < M (written by A), beta_{f+1} for f >= M (by B)
                // (PAIR kernels: label scores only, see pair_role)
  float* boff; // [utterance][2][nblk_cap][4]: the score offset in effect for the rows of each block, per CTA
  float* out_scores; // [B] forwardScore of the lattice (natural log)
  float* zparts; // [2B * kHelpers] forwardScore(emissions): the part each helper warp of the pair of CTAs summed
  int32_t* status; // [B] bit 0: a weight was not finite
  void* grad; // [B][grad_stride] of E, or NULL (loss only)
  long long grad_stride;
  int C;
  int nwn; // node warps in the launch (ceil(max nodes / 32))
  int nblk_cap;
  int ctc_blank; // PAIR kernels: the graphs are CTC target graphs with this blank label ...
  const int32_t* targets; // ... taken from the targets themselves: concatenated labels,
  // at GraphMeta::tgt_off of utterance b (the kernel never reads ctc_build_kernel's tables)
  Layout lay;
};

__device__ __forceinline__ bool finite_ok(float x) {
  return fabsf(x) < kHuge;
}

/* logsumexp of three scores in log2 units; absent arcs carry kNeg: ex2(kNeg - m) = 0, and three absent arcs give
 * kNeg + lg2(3) = kNeg (absorbed).  max + lg2(1 + 2^(x1 - max) + 2^(x2 - max)) over the two scores that are not
 * the maximum: 3 MUFU instead of 4 -- the SFU was the busiest pipe of these kernels when profiled on an earlier GPU
 * target (not re-measured on the H100), the ALU that sorts the three was not */
__device__ __forceinline__ float lse3_log2(float a, float b, float c) {
  const float lo = fminf(a, b), hi = fmaxf(a, b);
  const float m = fmaxf(hi, c), x1 = fminf(hi, c);
  return m + lg2(1.0f + (ex2(x1 - m) + ex2(lo - m)));
}

/* logsumexp of two scores */
__device__ __forceinline__ float lse2_log2(float a, float b) { // max + lg2(1 + 2^-|a - b|): 2 MUFU
  return fmaxf(a, b) + lg2(1.0f + ex2(-fabsf(a - b)));
}

struct NodeState {
  uint32_t so0, so1, so2; // byte offsets of the three neighbours in a chain row
  uint32_t u4; // this node's byte offset in a row
  uint32_t pc, qc; // chain rows: read / write (swapped every level)
  uint32_t ea; // this node's emission in the current stage row
  uint32_t oa; // this node's slot in the current stage row of the partner's scores
  uint32_t ga; // where this node's posterior of the current level goes (its label's slot in the helpers' block)
  float* gs; // where this node's score of the current level is saved (phase 1)
  float adj; // renormalisation: subtracted from every score at the first level of a block (an integer)
  float D; // sum of the adjustments so far: true score = kept score + D (exact: integers below 2^24)
  float Zh, zsub; // phase 2: posterior = ex2(((own - Zh) + other) - zsub)
  float Zl, Dc; // Z = Dc + Zh + Zl (log2 units); Dc: both CTAs' offsets at the meeting level (an integer)
  uint32_t redi; // the word (of an 8-byte aligned pair) the current block's maximum is published into
};

/* What is the same for every node thread of the CTA (kept in uniform registers / the constant bank, not in
 * per-thread registers: the node warps run at 40 registers).  Threads of the last node warp beyond the
 * utterance's nodes CLONE the last node -- same addresses, same values, harmless duplicate stores -- so
 * that the level code needs no "is this thread a node" state at all; `act` only matters where a thread's
 * value enters a reduction. */
struct NodeUni {
  int c4, p4, g4, pitch; // bytes per emission row / score-stage row / posterior row; floats per saved row
  int nact; // threads of the node warps of this CTA
};

/*
 * Renormalisation.  fp32 scores of a T = 1000 utterance reach several thousand, where one ulp is 5e-4:
 * the posteriors exp(alpha + beta - Z) of an un-normalised recursion carry that as a RELATIVE error
 * (the reference's own fp32 gradient is 2e-3 off the exact one there).  Here every block of 8 levels
 * ends with the integer part of the largest kept score being published (one F2I, one REDUX.MAX, one STS
 * by lane 0 -- no extra barrier: the level's own barrier orders it), and the next block's first level
 * subtracts it from every score.  Integers subtract exactly and their sum D stays exact in fp32, so the
 * kept scores stay within a few hundred of zero (ulp ~ 3e-5) and nothing is lost: true = kept + D.
 */
template <class S>
__device__ __forceinline__ void publish_block_max(S& st, float stored) {
  const int iv = __float2int_rn(fmaxf(stored, -2.0e9f));
  const int wm = __reduce_max_sync(0xffffffffu, iv);
  // two words, used alternately: the one the NEXT block will publish into is reset here (every thread
  // has read it at the start of this block, many barriers ago)
  if ((threadIdx.x & 31) == 0) smem_max_s32(st.redi, wm);
  if (threadIdx.x == 0) sts_u32(st.redi ^ 4u, (uint32_t)kIntMin);
}
/* at the start of the next block: the adjustment every node thread applies (same value in all of them) */
template <class S>
__device__ __forceinline__ void fetch_block_adjust(S& st) {
  const int mx = (int)lds_u32(st.redi);
  st.redi ^= 4u;
  // nothing alive (or nothing published yet): no adjustment
  const float off = (mx <= -2000000000) ? 0.0f : (float)mx;
  st.adj = off;
  st.D += off;
}

/* strides of the per-level accesses: compile-time constants in the FX kernels */
template <int NQ, bool FX, class E>
struct Strd {
  __device__ __forceinline__ static int c4(const NodeUni& un) { return FX ? 64 * (int)sizeof(E) * NQ : un.c4; }
  __device__ __forceinline__ static int p4(const NodeUni& un) { return FX ? 4 * kFixedPitch : un.p4; }
  __device__ __forceinline__ static int g4(const NodeUni& un) {
    return FX ? 4 * (kSlots * 64 * NQ + kFixedPitch) : un.g4;
  }
  __device__ __forceinline__ static int pitch(const NodeUni& un) { return FX ? kFixedPitch : un.pitch; }
};

/* one level.  DIR 0: CTA A (alpha), 1: CTA B (beta).  PH 1: save the score; 2: posterior in place.
 * r: the level's row within the block, counted in the CTA's own direction from the row st.ea / st.oa / st.ga /
 * st.gs point at (a constant after unrolling: with FX every address is register + immediate).
 * last: the block's last level (publishes the maximum for the renormalisation) */
template <int DIR, int PH, int NQ, bool FX, class E>
__device__ __forceinline__ void node_step(NodeState& st, const NodeUni& un, int r, bool last) {
  using SD = Strd<NQ, FX, E>;
  const int rr = DIR ? -r : r;
  const float x = lds_elem<E>(st.ea + (uint32_t)(rr * SD::c4(un)));
  // every arc weight of the graph is 0 (ctc_build_kernel's CTC graphs): no adds
  const float v = lse3_log2(lds_f32(st.pc + st.so0), lds_f32(st.pc + st.so1), lds_f32(st.pc + st.so2));
  // A: alpha_s = v + e[s-1][label(u)].  B: beta_s = v; what the predecessors read is beta_s + e[s-1][label(u)]
  const float val = DIR == 0 ? v + fmaf(x, kLog2e, -st.adj) : v - st.adj;
  const float stored = DIR == 0 ? val : fmaf(x, kLog2e, val);
  st.adj = 0.0f;
  sts_f32(st.qc + st.u4, stored);
  if (PH == 2) {
    // the posterior, written into the node's slot of the helpers' block
    sts_f32(st.ga + (uint32_t)(rr * SD::g4(un)),
            ex2(((val - st.Zh) + lds_f32(st.oa + (uint32_t)(rr * SD::p4(un)))) - st.zsub));
  }
  if (last) publish_block_max(st, stored);
  bar_named(1, un.nact);
  if (PH == 1) stg_f32(st.gs + rr * SD::pitch(un), val); // after the barrier: nothing waits for it
  const uint32_t t = st.pc;
  st.pc = st.qc;
  st.qc = t;
}

/* n levels from the rows st.ea / st.oa / st.ga / st.gs point at; st.gs moves on, the others are set per block */
template <int DIR, int PH, int NQ, bool FX, class E>
__device__ __forceinline__ void node_rows(NodeState& st, const NodeUni& un, int n) {
  // (a rolled loop with the last level peeled was slower on an earlier GPU target; not re-measured on the H100)
  if (n == kBlk) {
#pragma unroll
    for (int r = 0; r < kBlk; r++) node_step<DIR, PH, NQ, FX, E>(st, un, r, r == kBlk - 1);
  } else {
#pragma unroll 1
    for (int r = 0; r < n; r++) node_step<DIR, PH, NQ, FX, E>(st, un, r, r == n - 1);
  }
  if (PH == 1) st.gs += (DIR ? -n : n) * Strd<NQ, FX, E>::pitch(un);
}

/* reduction over the node threads of the CTA (named barrier 1): max, then sum */
__device__ __forceinline__ float node_reduce_max(float v, uint32_t red, int warp, int nwarps, int nact) {
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) sts_f32(red + 4u * warp, v);
  bar_named(1, nact);
  float r = lds_f32(red);
  for (int w = 1; w < nwarps; w++) r = fmaxf(r, lds_f32(red + 4u * w));
  bar_named(1, nact);
  return r;
}
__device__ __forceinline__ float node_reduce_sum(float v, uint32_t red, int warp, int nwarps, int nact) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sts_f32(red + 4u * warp, v);
  bar_named(1, nact);
  float r = lds_f32(red);
  for (int w = 1; w < nwarps; w++) r += lds_f32(red + 4u * w);
  bar_named(1, nact);
  return r;
}

/*
 * The first level of phase 2: the partner's row of the same level is there, so
 *   Z = logsumexp_u(alpha_s[u] + beta_s[u])   (log2 units; + both CTAs' offsets)
 * is reduced over the node threads -- as the pair (Zh, Zl) = (max of the rounded sums, lg2 of the sum of
 * 2^(exact sum - Zh)): the rounding error of every alpha + beta is carried into Zl by a TwoSum -- and the
 * level's posterior follows.  An utterance without any accepting path (Z = kNeg-like) gets Zh = +1e30,
 * which makes every posterior ex2(-huge) = 0.  `doth`: the partner's offset for this block.
 */
template <int DIR, int NQ, bool FX, class E>
__device__ __forceinline__ void node_first_phase2(
    NodeState& st, const NodeUni& un, bool act, uint32_t red, int warp, int nwarps, float doth, bool last,
    float* z_out, uint32_t feas_a, uint32_t spare) {
  using SD = Strd<NQ, FX, E>;
  const float x = lds_elem<E>(st.ea);
  st.ea += DIR ? -SD::c4(un) : SD::c4(un);
  const float v = lse3_log2(lds_f32(st.pc + st.so0), lds_f32(st.pc + st.so1), lds_f32(st.pc + st.so2));
  const float val = DIR == 0 ? v + fmaf(x, kLog2e, -st.adj) : v - st.adj;
  const float stored = DIR == 0 ? val : fmaf(x, kLog2e, val);
  st.adj = 0.0f;
  sts_f32(st.qc + st.u4, stored);
  const float o = lds_f32(st.oa);
  // TwoSum (Knuth): hi + lo == val + o exactly
  const float hi = val + o;
  const float bb = hi - val;
  const float lo = (val - (hi - bb)) + (o - bb);
  const float hv = act ? hi : 2.0f * kNeg; // the clones of the last node stay out of the reductions
  const float m = node_reduce_max(hv, red, warp, nwarps, un.nact);
  const float term = (act && m > 1.5f * kNeg) ? ex2((hi - m) + lo) : 0.0f;
  const float S = node_reduce_sum(term, red, warp, nwarps, un.nact);
  const bool feasible = m > kNeg * 0.5f && S > 0.0f;
  st.Zh = feasible ? m : 1.0e30f;
  st.Zl = feasible ? lg2(S) : 0.0f;
  st.Dc = st.D + doth;
  st.zsub = st.Zl;
  // the posterior mass of a level (1, or 0 without an accepting path): the helper warps take the mass on the
  // label with the most nodes as this minus the other labels' (visible to them through g_full)
  if (threadIdx.x == 0) sts_f32(feas_a, feasible ? 1.0f : 0.0f);
  if (z_out && threadIdx.x == 0)
    *z_out = feasible ? (float)(((double)st.Dc + ((double)m + (double)st.Zl)) * 0.6931471805599453) : -CUDART_INF_F;
  sts_f32(st.ga, ex2(((val - st.Zh) + o) - st.zsub));
  st.oa += DIR ? -SD::p4(un) : SD::p4(un);
  if (st.ga != spare) st.ga += DIR ? -SD::g4(un) : SD::g4(un); // (loss only: the one posterior goes to the spare word)
  if (last) publish_block_max(st, stored);
  bar_named(1, un.nact);
  const uint32_t t = st.pc;
  st.pc = st.qc;
  st.qc = t;
}

/* everything the node warps' phase loops need that is not per-thread state */
struct NodeCtx {
  const uint8_t* fl;
  float* saved;
  float* boff_own;
  float* out_score;
  uint32_t bars, e_base, o_base, g_base, od_base, perm_a, red_a, spare, lab4, feas_a, blank4;
  int e_stage_bytes, o_stage_bytes, g_block_bytes, pg, C, T, pitch, nblk, n_ph1, n_ph2, nw_act, N1;
  bool want_g;
};

/* barrier addresses (all in one array): */
__device__ __forceinline__ uint32_t bar_e_full(uint32_t bars, int s) {
  return bars + 8u * (uint32_t)s;
}
__device__ __forceinline__ uint32_t bar_e_empty(uint32_t bars, int s) {
  return bars + 8u * (uint32_t)(kSE + s);
}
__device__ __forceinline__ uint32_t bar_o_full(uint32_t bars, int s) {
  return bars + 8u * (uint32_t)(2 * kSE + s);
}
__device__ __forceinline__ uint32_t bar_o_empty(uint32_t bars, int s) {
  return bars + 8u * (uint32_t)(2 * kSE + kSO + s);
}
__device__ __forceinline__ uint32_t bar_g_full(uint32_t bars, int s) {
  return bars + 8u * (uint32_t)(2 * kSE + 2 * kSO + s);
}
__device__ __forceinline__ uint32_t bar_g_empty(uint32_t bars, int s) {
  return bars + 8u * (uint32_t)(2 * kSE + 2 * kSO + kSG + s);
}
__device__ __forceinline__ uint32_t bar_tbl_ready(uint32_t bars) {
  return bars + 8u * (uint32_t)(2 * kSE + 2 * kSO + 2 * kSG);
}

/*
 * The node warps of one CTA, both phases.  DIR 0: CTA A walks the blocks 0, 1, .. (rows ascending);
 * DIR 1: CTA B walks nblk-1, nblk-2, .. (rows descending).  Everything that depends only on the
 * direction is folded into per-thread base addresses up front, so that a block costs its levels plus a
 * few dozen instructions.
 */
template <int DIR, int NQ, bool FX, class E>
__device__ __forceinline__ void node_role(NodeState& st, const NodeCtx& cx, bool act, int nid) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  NodeUni un;
  un.c4 = (int)sizeof(E) * cx.C;
  un.p4 = 4 * cx.pitch;
  un.g4 = 4 * cx.pg;
  un.pitch = cx.pitch;
  un.nact = 32 * cx.nw_act;
  const int nact = un.nact;
  // the helper warps read the emission blocks of ONE phase (2 when there is a gradient, else 1); for the
  // other blocks node warp 0 arrives on the stage's "empty" barrier on their behalf
  const int arr1 = (warp == 0 && cx.want_g) ? 1 + kHelpers : 1;
  const int arr2 = (warp == 0 && !cx.want_g) ? 1 + kHelpers : 1;
  // first row of a FULL block in this direction
  const uint32_t e_row0 = cx.e_base + cx.lab4 + (DIR ? (uint32_t)((kBlk - 1) * cx.C * (int)sizeof(E)) : 0u);
  int v = 0; // blocks visited
  if (DIR == 0) {
    // level 0: start nodes carry the implicit 0 (shortest.cpp:129-135)
    if (cx.fl[nid] & 1) sts_f32(st.pc + st.u4, 0.0f);
    bar_named(1, nact);
    st.gs = cx.saved + nid;
    for (; v < cx.n_ph1; v++) {
      const int s = v & (kSE - 1);
      mbar_wait(bar_e_full(cx.bars, s), (v / kSE) & 1);
      st.ea = e_row0 + (uint32_t)(s * cx.e_stage_bytes);
      if (v > 0) fetch_block_adjust(st);
      if (tid == 0) stg_f32(cx.boff_own + 4 * v, st.D);
      node_rows<0, 1, NQ, FX, E>(st, un, kBlk); // A's phase-1 blocks are always full
      __syncwarp();
      if (lane == 0) mbar_arrive_n(bar_e_empty(cx.bars, s), arr1);
    }
  } else if (cx.T > 0) {
    // level T: accept nodes carry 0; what the predecessors read is beta_T + e[T-1][label]
    const int j0 = cx.nblk - 1, n0 = min(kBlk, cx.T - kBlk * j0);
    mbar_wait(bar_e_full(cx.bars, 0), 0);
    st.ea = cx.e_base + (uint32_t)((n0 - 1) * cx.C * (int)sizeof(E)) + cx.lab4;
    if (tid == 0) stg_f32(cx.boff_own + 4 * j0, 0.0f);
    {
      const float e2 = lds_elem<E>(st.ea) * kLog2e;
      st.ea -= un.c4;
      const float val = (cx.fl[nid] & 2) ? 0.0f : kNeg;
      sts_f32(st.pc + st.u4, val + e2); // written to the row the first step READS
      st.gs = cx.saved + (long long)(cx.T - 1) * cx.pitch + nid;
      if (n0 == 1) publish_block_max(st, val + e2);
      bar_named(1, nact);
      stg_f32(st.gs, val);
      st.gs -= un.pitch;
    }
    node_rows<1, 1, NQ, FX, E>(st, un, n0 - 1);
    __syncwarp();
    if (lane == 0) mbar_arrive_n(bar_e_empty(cx.bars, 0), arr1);
    for (v = 1; v < cx.n_ph1; v++) {
      const int s = v & (kSE - 1);
      mbar_wait(bar_e_full(cx.bars, s), (v / kSE) & 1);
      st.ea = e_row0 + (uint32_t)(s * cx.e_stage_bytes);
      fetch_block_adjust(st);
      if (tid == 0) stg_f32(cx.boff_own + 4 * (cx.nblk - 1 - v), st.D);
      node_rows<1, 1, NQ, FX, E>(st, un, kBlk);
      __syncwarp();
      if (lane == 0) mbar_arrive_n(bar_e_empty(cx.bars, s), arr1);
    }
  }
  cluster_sync_all();
  // ---- phase 2
  if (cx.n_ph2 <= 0) return;
  // first row of a full block in stage / block 0
  const uint32_t o_row0 = cx.o_base + 4u * (uint32_t)nid + (DIR ? (uint32_t)((kBlk - 1) * cx.pitch * 4) : 0u);
  uint32_t g_row0 = cx.spare;
  int g_stride = 0;
  if (cx.want_g) {
    mbar_wait(bar_tbl_ready(cx.bars), 0); // the helper warps' tables
    g_row0 = cx.g_base + lds_u16(cx.perm_a + 2u * (uint32_t)nid) + (DIR ? (uint32_t)((kBlk - 1) * cx.pg * 4) : 0u);
    g_stride = cx.g_block_bytes;
  } else {
    // loss only: the posterior of the one level goes to the spare word
  }
  for (int v2 = 0; v2 < cx.n_ph2; v2++, v++) {
    const int s = v & (kSE - 1), so = v2 & (kSO - 1), sg = v2 & (kSG - 1);
    // B's phase-2 blocks are full; A's last one may not be, and A's rows start at 0 either way
    const int nfr = DIR ? kBlk : min(kBlk, cx.T - kBlk * v);
    mbar_wait(bar_e_full(cx.bars, s), (v / kSE) & 1);
    mbar_wait(bar_o_full(cx.bars, so), (v2 / kSO) & 1);
    if (v2 >= kSG) mbar_wait(bar_g_empty(cx.bars, sg), ((v2 / kSG) - 1) & 1);
    st.ea = e_row0 + (uint32_t)(s * cx.e_stage_bytes);
    st.oa = o_row0 + (uint32_t)(so * cx.o_stage_bytes);
    st.ga = g_row0 + (uint32_t)(sg * g_stride);
    if (v > 0) fetch_block_adjust(st);
    const float doth = lds_f32(cx.od_base + 16u * so);
    if (v2 == 0) {
      node_first_phase2<DIR, NQ, FX, E>(st, un, act, cx.red_a, warp, cx.nw_act, doth, nfr == 1,
                                         DIR == 0 ? cx.out_score : nullptr, cx.feas_a, cx.spare);
      if (cx.want_g) node_rows<DIR, 2, NQ, FX, E>(st, un, nfr - 1);
    } else {
      // offsets moved since the meeting level: all integers, the differences are exact
      st.zsub = st.Zl - ((st.D + doth) - st.Dc);
      node_rows<DIR, 2, NQ, FX, E>(st, un, nfr);
    }
    __syncwarp();
    if (lane == 0) {
      mbar_arrive_n(bar_e_empty(cx.bars, s), arr2);
      mbar_arrive(bar_o_empty(cx.bars, so));
      mbar_arrive(bar_g_full(cx.bars, sg));
    }
  }
}

/* ------------------------------------------------------------------ */
/* node warps, CTC pair mode                                           */
/* ------------------------------------------------------------------ */

/*
 * gtnb_ctc_loss only ever hands this kernel the graphs ctc_build_kernel made (benchmarks/ctc.cpp:40-58): node 2t is
 * the t-th blank (self loop, arc from label 2t-1), node 2t-1 the t-th label (self loop, arc from blank 2t-2, skip
 * arc from label 2t-3 unless the label repeats).  The PAIR kernels give thread t BOTH nodes (2t-1, 2t):
 *   - half the node warps (4 instead of 7 at U = 100) and half the barrier arrivals per level;
 *   - the thread's own scores stay in registers; what it needs from its neighbour is ONE LDS.64 (A: the pair
 *     t-1) or one LDS (B: the label of pair t+1) instead of six loads, its two results go to the chain row as
 *     one STS.64 (B: one STS, the label's), and only the label's is saved (one STG);
 *   - the blank's logsumexp has two terms: max + lg2(1 + 2^-|a-b|), 2 MUFU instead of 4;
 *   - the blank's posterior is never formed: blank is the complement label of the helper warps.
 * 28 / 34 SASS instructions per PAIR and level instead of 2 x 19 / 2 x 24, 6 / 7 MUFU instead of 8 / 10.
 * Row layouts: slot(node n) = n + 3 in the chain rows (pair t-1 of thread 0 and the label beyond the last pair read
 * the row's kNeg).  Saved scores: the partner reads a blank score only at the meeting level (Z); every other level
 * it reads the label's alone (blank is the complement label), so the saved rows hold LABEL scores only, kHalfPitch
 * floats per row, pair t at float t: block j of n rows starts at float j * kBlk * kFixedPitch as it always did, its
 * label rows take the first n * kHalfPitch floats, and -- in the block of the meeting level only -- the meeting
 * row's blank scores follow them.  Half the saved-score traffic of full rows, in HBM both ways.
 */
/* start / accept flags of node n of a CTC target graph with N1 = 2U + 1 nodes (benchmarks/ctc.cpp:43-44): the PAIR
 * kernels take the graph from the target itself and never read ctc_build_kernel's tables */
/* does label node n (odd) have the skip in-arc from label n - 2: not for the first label, not for a repeat (:51-54) */
__device__ __forceinline__ bool ctc_skip(const int32_t* tg, int n, int N1) {
  return n >= 3 && n < N1 && tg[(n - 1) / 2] != tg[(n - 3) / 2];
}
__device__ __forceinline__ int ctc_flags(int n, int N1) {
  return (n == 0 ? 1 : 0) | ((n == N1 - 1 || n == N1 - 2) ? 2 : 0);
}

struct PairState {
  float al, ab; // what the neighbours read of this thread's label / blank node (A: alpha, B: beta + emission)
  uint32_t t8; // 8 * pair index
  uint32_t pc, qc; // chain rows: read / write
  uint32_t ea_l, ea_b; // emissions of the label / of blank in the current stage, first row of the block
  uint32_t oa; // the partner's score of this thread's label node, first row of the block
  uint32_t ga; // where the label's posterior goes
  float* gs; // where the label's score is saved (phase 1), first row of the block
  float lastb; // phase 1: the saved blank score of the block's last level (stored only at the meeting level)
  float adj, D, Zh, zsub, Zl, Dc;
  uint32_t redi;
  bool skip; // A: label 2t-1 has the skip in-arc; B: label 2t+1 has it (= this thread's label has the skip out-arc)
};

template <int DIR, int PH, int NQ, class E>
__device__ __forceinline__ void pair_step(PairState& ps, const NodeUni& un, int r, bool last) {
  using SD = Strd<NQ, true, E>;
  const int rr = DIR ? -r : r;
  const float xl = lds_elem<E>(ps.ea_l + (uint32_t)(rr * SD::c4(un)));
  const float xb = lds_elem<E>(ps.ea_b + (uint32_t)(rr * SD::c4(un)));
  float vl, vb;
  if (DIR == 0) {
    const f32x2 pv = lds_v2_f32(ps.pc + ps.t8); // pair t-1: (label 2t-3, blank 2t-2)
    vb = lse2_log2(ps.ab, ps.al);
    vl = lse3_log2(ps.al, pv.y, ps.skip ? pv.x : kNeg);
  } else {
    const float nl = lds_f32(ps.pc + ps.t8 + 16u); // label 2t+1
    vb = lse2_log2(ps.ab, nl);
    vl = lse3_log2(ps.al, ps.ab, ps.skip ? nl : kNeg);
  }
  const float val_l = DIR == 0 ? vl + fmaf(xl, kLog2e, -ps.adj) : vl - ps.adj;
  const float val_b = DIR == 0 ? vb + fmaf(xb, kLog2e, -ps.adj) : vb - ps.adj;
  ps.al = DIR == 0 ? val_l : fmaf(xl, kLog2e, val_l);
  ps.ab = DIR == 0 ? val_b : fmaf(xb, kLog2e, val_b);
  ps.adj = 0.0f;
  if (DIR == 0)
    sts_v2_f32(ps.qc + ps.t8 + 8u, ps.al, ps.ab);
  else
    sts_f32(ps.qc + ps.t8 + 8u, ps.al); // only the label is read by a neighbour
  if (PH == 2)
    sts_f32(ps.ga + (uint32_t)(rr * SD::g4(un)),
        ex2(((val_l - ps.Zh) + lds_f32(ps.oa + (uint32_t)(rr * 4 * kHalfPitch))) - ps.zsub));
  if (last) publish_block_max(ps, fmaxf(ps.al, ps.ab));
  bar_named(1, un.nact);
  if (PH == 1) {
    stg_f32(ps.gs + rr * kHalfPitch, val_l);
    if (last) ps.lastb = val_b;
  }
  const uint32_t t = ps.pc;
  ps.pc = ps.qc;
  ps.qc = t;
}

template <int DIR, int PH, int NQ, class E>
__device__ __forceinline__ void pair_rows(PairState& ps, const NodeUni& un, int n) {
  if (n == kBlk) {
#pragma unroll
    for (int r = 0; r < kBlk; r++) pair_step<DIR, PH, NQ, E>(ps, un, r, r == kBlk - 1);
  } else {
#pragma unroll 1
    for (int r = 0; r < n; r++) pair_step<DIR, PH, NQ, E>(ps, un, r, r == n - 1);
  }
}

/* the first level of phase 2 (see node_first_phase2): Z over BOTH nodes of every pair; ob: the partner's blank
 * score of this pair at this level */
template <int DIR, int NQ, class E>
__device__ __forceinline__ void pair_first_phase2(
    PairState& ps, const NodeUni& un, bool act_l, bool act_b, uint32_t red, int warp, int nwarps, float doth, bool last,
    float* z_out, uint32_t feas_a, bool want_g, uint32_t ob) {
  using SD = Strd<NQ, true, E>;
  const float xl = lds_elem<E>(ps.ea_l), xb = lds_elem<E>(ps.ea_b);
  ps.ea_l += DIR ? -SD::c4(un) : SD::c4(un);
  ps.ea_b += DIR ? -SD::c4(un) : SD::c4(un);
  float vl, vb;
  if (DIR == 0) {
    const f32x2 pv = lds_v2_f32(ps.pc + ps.t8);
    vb = lse2_log2(ps.ab, ps.al);
    vl = lse3_log2(ps.al, pv.y, ps.skip ? pv.x : kNeg);
  } else {
    const float nl = lds_f32(ps.pc + ps.t8 + 16u);
    vb = lse2_log2(ps.ab, nl);
    vl = lse3_log2(ps.al, ps.ab, ps.skip ? nl : kNeg);
  }
  const float val_l = DIR == 0 ? vl + fmaf(xl, kLog2e, -ps.adj) : vl - ps.adj;
  const float val_b = DIR == 0 ? vb + fmaf(xb, kLog2e, -ps.adj) : vb - ps.adj;
  ps.al = DIR == 0 ? val_l : fmaf(xl, kLog2e, val_l);
  ps.ab = DIR == 0 ? val_b : fmaf(xb, kLog2e, val_b);
  ps.adj = 0.0f;
  if (DIR == 0)
    sts_v2_f32(ps.qc + ps.t8 + 8u, ps.al, ps.ab);
  else
    sts_f32(ps.qc + ps.t8 + 8u, ps.al);
  const f32x2 o = {lds_f32(ps.oa), lds_f32(ob)}; // the partner's scores of (label, blank)
  // TwoSum (Knuth) of both: hi + lo == val + o exactly
  const float hl = val_l + o.x, bl = hl - val_l, ll = (val_l - (hl - bl)) + (o.x - bl);
  const float hb = val_b + o.y, bb = hb - val_b, lb = (val_b - (hb - bb)) + (o.y - bb);
  const float m = node_reduce_max(fmaxf(act_l ? hl : 2.0f * kNeg, act_b ? hb : 2.0f * kNeg), red, warp, nwarps, un.nact);
  const bool live = m > 1.5f * kNeg;
  const float term = (act_l && live ? ex2((hl - m) + ll) : 0.0f) + (act_b && live ? ex2((hb - m) + lb) : 0.0f);
  const float S = node_reduce_sum(term, red, warp, nwarps, un.nact);
  const bool feasible = m > kNeg * 0.5f && S > 0.0f;
  ps.Zh = feasible ? m : 1.0e30f;
  ps.Zl = feasible ? lg2(S) : 0.0f;
  ps.Dc = ps.D + doth;
  ps.zsub = ps.Zl;
  if (threadIdx.x == 0) sts_f32(feas_a, feasible ? 1.0f : 0.0f);
  if (z_out && threadIdx.x == 0)
    *z_out = feasible ? (float)(((double)ps.Dc + ((double)m + (double)ps.Zl)) * 0.6931471805599453) : -CUDART_INF_F;
  if (want_g) {
    sts_f32(ps.ga, ex2(((val_l - ps.Zh) + o.x) - ps.zsub));
    ps.ga += DIR ? -SD::g4(un) : SD::g4(un);
  }
  ps.oa += DIR ? -4 * kHalfPitch : 4 * kHalfPitch;
  if (last) publish_block_max(ps, fmaxf(ps.al, ps.ab));
  bar_named(1, un.nact);
  const uint32_t t = ps.pc;
  ps.pc = ps.qc;
  ps.qc = t;
}

/* the pair warps of one CTA, both phases: node_role's protocol (stages, barriers, offsets) on pairs */
template <int DIR, int NQ, class E>
__device__ __forceinline__ void pair_role(PairState& ps, const NodeCtx& cx, int tp, bool act, bool has_label) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  NodeUni un;
  un.c4 = (int)sizeof(E) * cx.C;
  un.p4 = 4 * cx.pitch;
  un.g4 = 4 * cx.pg;
  un.pitch = cx.pitch;
  un.nact = 32 * cx.nw_act;
  const int nact = un.nact;
  const int arr1 = (warp == 0 && cx.want_g) ? 1 + kHelpers : 1;
  const int arr2 = (warp == 0 && !cx.want_g) ? 1 + kHelpers : 1;
  const uint32_t dir_off = DIR ? (uint32_t)((kBlk - 1) * cx.C * (int)sizeof(E)) : 0u;
  const uint32_t e_row0_l = cx.e_base + cx.lab4 + dir_off; // cx.lab4: this thread's label
  const uint32_t e_row0_b = cx.e_base + cx.blank4 + dir_off;
  const bool act_l = act && has_label;
  // saved scores (see the layout above): this pair's label in row 0 of block j.  The meeting level is the last one of
  // the CTA's last phase-1 block (A: the last row of a full block; B: row 0); its blank scores go behind that block's
  // n label rows
  auto label_at = [&](int j) { return cx.saved + (long long)j * (kBlk * kFixedPitch) + tp; };
  int v = 0;
  if (DIR == 0) {
    // level 0: start nodes carry the implicit 0 (shortest.cpp:129-135)
    ps.al = (has_label && (ctc_flags(2 * tp - 1, cx.N1) & 1)) ? 0.0f : kNeg;
    ps.ab = (ctc_flags(2 * tp, cx.N1) & 1) ? 0.0f : kNeg;
    sts_v2_f32(ps.pc + ps.t8 + 8u, ps.al, ps.ab);
    bar_named(1, nact);
    for (; v < cx.n_ph1; v++) {
      const int s = v & (kSE - 1);
      mbar_wait(bar_e_full(cx.bars, s), (v / kSE) & 1);
      ps.ea_l = e_row0_l + (uint32_t)(s * cx.e_stage_bytes);
      ps.ea_b = e_row0_b + (uint32_t)(s * cx.e_stage_bytes);
      ps.gs = label_at(v);
      if (v > 0) fetch_block_adjust(ps);
      if (tid == 0) stg_f32(cx.boff_own + 4 * v, ps.D);
      pair_rows<0, 1, NQ, E>(ps, un, kBlk);
      if (v == cx.n_ph1 - 1) stg_f32(label_at(v) + kBlk * kHalfPitch, ps.lastb);
      __syncwarp();
      if (lane == 0) mbar_arrive_n(bar_e_empty(cx.bars, s), arr1);
    }
  } else if (cx.T > 0) {
    // level T: accept nodes carry 0; what the predecessors read is beta_T + e[T-1][label]
    const int j0 = cx.nblk - 1, n0 = min(kBlk, cx.T - kBlk * j0);
    mbar_wait(bar_e_full(cx.bars, 0), 0);
    ps.ea_l = cx.e_base + (uint32_t)((n0 - 1) * cx.C * (int)sizeof(E)) + cx.lab4;
    ps.ea_b = cx.e_base + (uint32_t)((n0 - 1) * cx.C * (int)sizeof(E)) + cx.blank4;
    if (tid == 0) stg_f32(cx.boff_own + 4 * j0, 0.0f);
    {
      const float el = lds_elem<E>(ps.ea_l) * kLog2e, eb = lds_elem<E>(ps.ea_b) * kLog2e;
      ps.ea_l -= un.c4;
      ps.ea_b -= un.c4;
      const float val_l = (has_label && (ctc_flags(2 * tp - 1, cx.N1) & 2)) ? 0.0f : kNeg;
      const float val_b = (ctc_flags(2 * tp, cx.N1) & 2) ? 0.0f : kNeg;
      ps.al = val_l + el;
      ps.ab = val_b + eb;
      sts_f32(ps.pc + ps.t8 + 8u, ps.al); // written to the row the first step READS
      ps.gs = label_at(j0) + (n0 - 1) * kHalfPitch;
      ps.lastb = val_b;
      if (n0 == 1) publish_block_max(ps, fmaxf(ps.al, ps.ab));
      bar_named(1, nact);
      stg_f32(ps.gs, val_l);
      ps.gs -= kHalfPitch;
    }
    pair_rows<1, 1, NQ, E>(ps, un, n0 - 1);
    if (cx.n_ph1 == 1) stg_f32(label_at(j0) + n0 * kHalfPitch, ps.lastb);
    __syncwarp();
    if (lane == 0) mbar_arrive_n(bar_e_empty(cx.bars, 0), arr1);
    for (v = 1; v < cx.n_ph1; v++) {
      const int s = v & (kSE - 1);
      mbar_wait(bar_e_full(cx.bars, s), (v / kSE) & 1);
      ps.ea_l = e_row0_l + (uint32_t)(s * cx.e_stage_bytes);
      ps.ea_b = e_row0_b + (uint32_t)(s * cx.e_stage_bytes);
      ps.gs = label_at(cx.nblk - 1 - v) + (kBlk - 1) * kHalfPitch;
      fetch_block_adjust(ps);
      if (tid == 0) stg_f32(cx.boff_own + 4 * (cx.nblk - 1 - v), ps.D);
      pair_rows<1, 1, NQ, E>(ps, un, kBlk);
      if (v == cx.n_ph1 - 1) stg_f32(label_at(cx.nblk - 1 - v) + kBlk * kHalfPitch, ps.lastb);
      __syncwarp();
      if (lane == 0) mbar_arrive_n(bar_e_empty(cx.bars, s), arr1);
    }
  }
  cluster_sync_all();
  // ---- phase 2
  if (cx.n_ph2 <= 0) return;
  const uint32_t o_row0 = cx.o_base + 4u * (uint32_t)tp + (DIR ? (uint32_t)((kBlk - 1) * kHalfPitch * 4) : 0u);
  uint32_t g_row0 = 0;
  int g_stride = 0;
  if (cx.want_g) {
    mbar_wait(bar_tbl_ready(cx.bars), 0); // the helper warps' tables
    // the label's slot; a thread without a label node (pair 0) stores into the row's last word, which nobody reads
    const uint32_t slot = has_label ? lds_u16(cx.perm_a + 2u * (uint32_t)(2 * tp - 1)) : 4u * (uint32_t)(cx.pg - 1);
    g_row0 = cx.g_base + slot + (DIR ? (uint32_t)((kBlk - 1) * cx.pg * 4) : 0u);
    g_stride = cx.g_block_bytes;
  }
  for (int v2 = 0; v2 < cx.n_ph2; v2++, v++) {
    const int s = v & (kSE - 1), so = v2 & (kSO - 1), sg = v2 & (kSG - 1);
    const int nfr = DIR ? kBlk : min(kBlk, cx.T - kBlk * v);
    mbar_wait(bar_e_full(cx.bars, s), (v / kSE) & 1);
    mbar_wait(bar_o_full(cx.bars, so), (v2 / kSO) & 1);
    if (v2 >= kSG) mbar_wait(bar_g_empty(cx.bars, sg), ((v2 / kSG) - 1) & 1);
    ps.ea_l = e_row0_l + (uint32_t)(s * cx.e_stage_bytes);
    ps.ea_b = e_row0_b + (uint32_t)(s * cx.e_stage_bytes);
    ps.oa = o_row0 + (uint32_t)(so * cx.o_stage_bytes);
    ps.ga = g_row0 + (uint32_t)(sg * g_stride);
    if (v > 0) fetch_block_adjust(ps);
    const float doth = lds_f32(cx.od_base + 16u * so);
    if (v2 == 0) {
      // the meeting row's blank scores follow the block's nfr label rows (B reads row kBlk - 1, A row 0)
      const uint32_t ob = ps.oa + (uint32_t)((DIR ? 1 : nfr) * kHalfPitch * 4);
      pair_first_phase2<DIR, NQ, E>(ps, un, act_l, act, cx.red_a, warp, cx.nw_act, doth, nfr == 1,
                                 DIR == 0 ? cx.out_score : nullptr, cx.feas_a, cx.want_g, ob);
      if (cx.want_g) pair_rows<DIR, 2, NQ, E>(ps, un, nfr - 1);
    } else {
      ps.zsub = ps.Zl - ((ps.D + doth) - ps.Dc);
      pair_rows<DIR, 2, NQ, E>(ps, un, nfr);
    }
    __syncwarp();
    if (lane == 0) {
      mbar_arrive_n(bar_e_empty(cx.bars, s), arr2);
      mbar_arrive(bar_o_empty(cx.bars, so));
      mbar_arrive(bar_g_full(cx.bars, sg));
    }
  }
}

/* ------------------------------------------------------------------ */
/* helper warps                                                        */
/* ------------------------------------------------------------------ */

/*
 * Every helper warp owns two rows of a block: lanes 0..15 the row 2 * hw, lanes 16..31 the row
 * 2 * hw + 1; lane l16 of a half holds the labels 4 * (l16 + 16 i) .. + 3 (one float4 of the emission
 * row per i), so a row's maximum and sum are four shuffles inside the half-warp and the helper warps
 * never talk to each other.  The posteriors of a row sit in the block as kSlots floats per label -- the
 * node threads write theirs into their label's next free slot, unused slots stay 0 -- so the mass on a
 * label is one LDS.128 and three adds, and the four gradients of a lane leave as one 16-byte store.
 * Labels carried by more than kSlots nodes (CTC: blank) live behind the slots, contiguously, and are
 * summed by the 16 lanes of the row together.
 *
 * seg[c] = overflow start (10 bits) | number of nodes (10 bits) | (cooperative slot + 1, or 15 = summed by
 * the owning lane alone) << 20, the last two only when the label has more than kSlots nodes.
 */
struct HelperState {
  int hw, lane, r, l16;
  int C;
  uint32_t seg;
  float zacc; // lanes 0 and 16: sum of their rows' logsumexp
  bool bad;
};

__device__ __forceinline__ uint32_t seg_pack(int start, int len, int slot1) {
  return (uint32_t)start | ((uint32_t)len << 10) | ((uint32_t)slot1 << 20);
}
__device__ __forceinline__ float half_max(float v) { // over the 16 lanes of a half-warp
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float half_sum(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

/* per-lane constants of the helper warps (NQ float4 chunks of the row per lane) */
template <int NQ>
struct HelperConst {
  uint32_t eoff[NQ]; // byte offset of the chunk in an emission stage (0xffffffff: beyond C)
  uint32_t goff[NQ]; // byte offset of the chunk's first slot in a posterior block
  uint32_t hsel[NQ]; // 4 bits per label of the chunk: 0 = slots, h + 1 = cooperative sum h, 15 = own loop
  uint32_t hoff[kMaxHeavy]; // byte offset of the cooperative label's overflow positions in this lane's row
  int hlen[kMaxHeavy];
  uint32_t ovf; // byte offset of the row's overflow area
};

template <int NQ, bool WANT_G, class E>
__device__ __forceinline__ void helper_block(
    HelperState& hs, const HelperConst<NQ>& k, int nfr, uint32_t estage, uint32_t e_empty_bar, uint32_t gblock,
    uint32_t g_empty_bar, int nheavy, bool has_comp, uint32_t feas_a, E* gout) {
  const bool row_on = hs.r < nfr;
  float4 x[NQ];
  float mx = -3.0e38f;
#pragma unroll
  for (int i = 0; i < NQ; i++) {
    const bool ok = row_on && k.eoff[i] != 0xffffffffu;
    x[i] = ok ? lds_elem4<E>(estage + k.eoff[i]) : make_float4(-3.0e38f, -3.0e38f, -3.0e38f, -3.0e38f);
    const float hi = fmaxf(fmaxf(x[i].x, x[i].y), fmaxf(x[i].z, x[i].w));
    const float lo = fminf(fminf(x[i].x, x[i].y), fminf(x[i].z, x[i].w));
    const float nan_probe = (x[i].x + x[i].y) + (x[i].z + x[i].w); // fmaxf / fminf drop NaNs, a sum keeps them
    if (ok) hs.bad |= !(hi < kHuge && lo > -kHuge && nan_probe == nan_probe);
    mx = fmaxf(mx, hi);
  }
  __syncwarp();
  if (hs.lane == 0) mbar_arrive(e_empty_bar); // the emission rows are in registers
  mx = half_max(mx);
  const float mxs = mx * kLog2e;
  float sm = 0.0f;
#pragma unroll
  for (int i = 0; i < NQ; i++) { // invalid entries: ex2(-huge) = 0
    x[i].x = ex2(fmaf(x[i].x, kLog2e, -mxs));
    x[i].y = ex2(fmaf(x[i].y, kLog2e, -mxs));
    x[i].z = ex2(fmaf(x[i].z, kLog2e, -mxs));
    x[i].w = ex2(fmaf(x[i].w, kLog2e, -mxs));
    sm += (x[i].x + x[i].y) + (x[i].z + x[i].w);
  }
  sm = half_sum(sm);
  if (row_on && hs.l16 == 0) hs.zacc += mx + lg2(sm) * kLn2; // logsumexp of the row
  if (WANT_G) {
    const float inv = 1.0f / sm;
    float hsum[kMaxHeavy];
#pragma unroll
    for (int h = 0; h < kMaxHeavy; h++) {
      hsum[h] = 0.0f;
      if (h < nheavy) {
        float a0 = 0.0f, a1 = 0.0f;
        if (row_on) {
          const uint32_t a = gblock + k.hoff[h];
          int q = hs.l16;
          for (; q + 16 < k.hlen[h]; q += 32) {
            a0 += lds_f32(a + 4u * q);
            a1 += lds_f32(a + 4u * (q + 16));
          }
          if (q < k.hlen[h]) a0 += lds_f32(a + 4u * q);
        }
        hsum[h] = half_sum(a0 + a1);
      }
    }
    float o[4 * NQ];
    float part = 0.0f; // this lane's labels' mass, the complement label aside
#pragma unroll
    for (int i = 0; i < NQ; i++) {
#pragma unroll
      for (int j = 0; j < 4; j++) o[4 * i + j] = 0.0f;
      if (row_on && k.eoff[i] != 0xffffffffu) {
        const uint32_t a = gblock + k.goff[i];
        const float4 g0 = lds_v4_f32(a), g1 = lds_v4_f32(a + 16), g2 = lds_v4_f32(a + 32), g3 = lds_v4_f32(a + 48);
        o[4 * i + 0] = (g0.x + g0.y) + (g0.z + g0.w);
        o[4 * i + 1] = (g1.x + g1.y) + (g1.z + g1.w);
        o[4 * i + 2] = (g2.x + g2.y) + (g2.z + g2.w);
        o[4 * i + 3] = (g3.x + g3.y) + (g3.z + g3.w);
        if (k.hsel[i]) { // some label of the chunk has more than kSlots nodes
#pragma unroll
          for (int j = 0; j < 4; j++) {
            const int s1 = (k.hsel[i] >> (4 * j)) & 15;
            if (s1 == 15) { // beyond the cooperative slots: this lane sums the label's positions itself
              const uint32_t w = lds_u32(hs.seg + 4u * (uint32_t)(k.eoff[i] / (uint32_t)sizeof(E) - hs.r * hs.C + j));
              const int len = (w >> 10) & 1023;
              const uint32_t p = gblock + k.ovf + (w & 1023u) * 4u;
              float acc = 0.0f;
              for (int q = 0; q < len; q++) acc += lds_f32(p + 4u * q);
              o[4 * i + j] = acc;
            } else if (s1 == 14) { // the complement label: nothing was stored for it
              o[4 * i + j] = 0.0f;
            } else if (s1) {
#pragma unroll
              for (int h = 0; h < kMaxHeavy; h++)
                if (h == s1 - 1) o[4 * i + j] = hsum[h];
            }
          }
        }
        part += (o[4 * i + 0] + o[4 * i + 1]) + (o[4 * i + 2] + o[4 * i + 3]);
      }
    }
    if (has_comp) { // mass on the label with the most nodes = the level's mass - everybody else's
      const float cm = lds_f32(feas_a) - half_sum(part);
#pragma unroll
      for (int i = 0; i < NQ; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
          if (((k.hsel[i] >> (4 * j)) & 15) == 14) o[4 * i + j] = cm;
    }
#pragma unroll
    for (int i = 0; i < NQ; i++) {
      if (row_on && k.eoff[i] != 0xffffffffu) {
        // d(forwardScore(e) - forwardScore(lattice)) / d e[f][c] = softmax - posterior mass on label c
        stg_elem4(gout + k.eoff[i] / (uint32_t)sizeof(E),
                  make_float4(fmaf(x[i].x, inv, -o[4 * i + 0]), fmaf(x[i].y, inv, -o[4 * i + 1]),
                              fmaf(x[i].z, inv, -o[4 * i + 2]), fmaf(x[i].w, inv, -o[4 * i + 3])));
      }
    }
    __syncwarp();
    if (hs.lane == 0) mbar_arrive(g_empty_bar); // this warp is done with the posterior block
  }
}

/*
 * The same for the common case, with everything that can be decided once decided once: the emission row is
 * exactly NQ float4 chunks per lane (C == 64 * NQ), the block is full, and every label with more than kSlots
 * nodes (CTC: blank, plus the odd label that occurs five times or more) has a cooperative slot.  htab: per
 * cooperative label {label, overflow start in floats, nodes} in shared memory.  About a third of the generic
 * version's instructions.
 */
template <int NQ, class E>
__device__ __forceinline__ void helper_block_fast(
    HelperState& hs, uint32_t ea, uint32_t e_empty_bar, uint32_t ga, uint32_t ovf_row, uint32_t htab, int nheavy,
    bool has_comp, int comp_rel, uint32_t feas_a, uint32_t g_empty_bar, E* gout) {
  float4 x[NQ];
#pragma unroll
  for (int i = 0; i < NQ; i++) x[i] = lds_elem4<E>(ea + 64u * (uint32_t)sizeof(E) * i); // chunk i: labels 64 i + 4 l16 .. + 3
  __syncwarp();
  if (hs.lane == 0) mbar_arrive(e_empty_bar); // the emission rows are in registers
  float mx = fmaxf(fmaxf(x[0].x, x[0].y), fmaxf(x[0].z, x[0].w));
  float lo = fminf(fminf(x[0].x, x[0].y), fminf(x[0].z, x[0].w));
#pragma unroll
  for (int i = 1; i < NQ; i++) {
    mx = fmaxf(mx, fmaxf(fmaxf(x[i].x, x[i].y), fmaxf(x[i].z, x[i].w)));
    lo = fminf(lo, fminf(fminf(x[i].x, x[i].y), fminf(x[i].z, x[i].w)));
  }
  mx = half_max(mx);
  const float mxs = mx * kLog2e;
  float sm = 0.0f;
#pragma unroll
  for (int i = 0; i < NQ; i++) {
    x[i].x = ex2(fmaf(x[i].x, kLog2e, -mxs));
    x[i].y = ex2(fmaf(x[i].y, kLog2e, -mxs));
    x[i].z = ex2(fmaf(x[i].z, kLog2e, -mxs));
    x[i].w = ex2(fmaf(x[i].w, kLog2e, -mxs));
    sm += (x[i].x + x[i].y) + (x[i].z + x[i].w);
  }
  sm = half_sum(sm);
  // a NaN or +inf emission makes the sum NaN, a -inf / huge one trips the range checks
  hs.bad |= !(lo > -kHuge && mx < kHuge && sm < 3.0e38f);
  if (hs.l16 == 0) hs.zacc += mx + lg2(sm) * kLn2; // logsumexp of the row
  const float inv = rcp_approx(sm);
  float o[4 * NQ];
#pragma unroll
  for (int i = 0; i < NQ; i++) {
    const uint32_t a = ga + 1024u * i; // 64 labels * kSlots floats further on
    const float4 g0 = lds_v4_f32(a), g1 = lds_v4_f32(a + 16), g2 = lds_v4_f32(a + 32), g3 = lds_v4_f32(a + 48);
    o[4 * i + 0] = (g0.x + g0.y) + (g0.z + g0.w);
    o[4 * i + 1] = (g1.x + g1.y) + (g1.z + g1.w);
    o[4 * i + 2] = (g2.x + g2.y) + (g2.z + g2.w);
    o[4 * i + 3] = (g3.x + g3.y) + (g3.z + g3.w);
  }
  // the labels carried by many nodes: the row's 16 lanes sum their positions together
  // (htab: label | first overflow position << 8 | nodes << 18)
#pragma unroll 1
  for (int h = 0; h < nheavy; h++) {
    const uint32_t w = lds_u32(htab + 4u * h);
    const int hlen = (int)(w >> 18);
    const uint32_t hq = ovf_row + 4u * ((w >> 8) & 1023u) + 4u * hs.l16;
    float a0 = hs.l16 < hlen ? lds_f32(hq) : 0.0f;
    for (int q0 = 16; q0 < hlen; q0 += 16) // (rare: a label on more than 16 nodes that is not the complement label)
      if (q0 + hs.l16 < hlen) a0 += lds_f32(hq + 4u * q0);
    const float hsum = half_sum(a0);
    const int rel = (int)(w & 255u) - 4 * hs.l16; // which of this lane's labels (64 i + 4 l16 + j  ->  64 i + j), if any
#pragma unroll
    for (int i = 0; i < NQ; i++) {
#pragma unroll
      for (int j = 0; j < 4; j++) o[4 * i + j] = rel == 64 * i + j ? hsum : o[4 * i + j];
    }
  }
  if (has_comp) {
    // the label with the most nodes (CTC: blank, half of all nodes): its nodes stored nothing; its mass is the
    // level's mass (1, or 0 for an utterance without an accepting path) minus everybody else's
    float part = 0.0f;
#pragma unroll
    for (int i = 0; i < NQ; i++) part += (o[4 * i + 0] + o[4 * i + 1]) + (o[4 * i + 2] + o[4 * i + 3]);
    const float cm = lds_f32(feas_a) - half_sum(part);
#pragma unroll
    for (int i = 0; i < NQ; i++) {
#pragma unroll
      for (int j = 0; j < 4; j++) o[4 * i + j] = comp_rel == 64 * i + j ? cm : o[4 * i + j];
    }
  }
  // d(forwardScore(e) - forwardScore(lattice)) / d e[f][c] = softmax - posterior mass on label c
#pragma unroll
  for (int i = 0; i < NQ; i++) {
    const float4 gr = make_float4(fmaf(x[i].x, inv, -o[4 * i + 0]), fmaf(x[i].y, inv, -o[4 * i + 1]),
                                  fmaf(x[i].z, inv, -o[4 * i + 2]), fmaf(x[i].w, inv, -o[4 * i + 3]));
    stg_elem4(gout + 64 * i, gr);
  }
  __syncwarp();
  if (hs.lane == 0) mbar_arrive(g_empty_bar); // this warp is done with the posterior block
}

/* ------------------------------------------------------------------ */
/* the kernel                                                          */
/* ------------------------------------------------------------------ */

/* MODE 0: one node per thread (any graph in the envelope); 1: PAIR (CTC graphs, two nodes per thread) */
/* E: the element type of the emissions and of the gradient (float, bf16_t or f16_t); everything in between is float32 */
template <int NQ, bool FX, int MODE, class E = float>
__global__ void __launch_bounds__(32 * ((MODE == 1 ? kMaxPairWarps : kMaxNodeWarps) + 1 + kHelpers), 4)
    bidir_ctc_kernel(const Params P) {
  constexpr bool PAIR = MODE == 1;
  GTNB_DYNAMIC_SMEM_128(unsigned char, smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.x >> 1;
  const int dir = (int)cluster_rank(); // 0: CTA A (alpha), 1: CTA B (beta)
  const GraphMeta m = P.meta[b];
  const int N1 = m.sg_N, T = m.T, C = P.C;
  const int pitch = FX ? kFixedPitch : ((N1 + 3) & ~3); // floats per saved-score row (HBM and stages)
  const bool want_g = P.grad != nullptr;
  const Layout& L = P.lay;
  float* ring = reinterpret_cast<float*>(smem + L.off_ring);
  const uint32_t bars = smem_u32(smem + L.off_bar);
  const uint32_t e_base = smem_u32(smem + L.off_e), o_base = smem_u32(smem + L.off_o);
  const uint32_t od_base = smem_u32(smem + L.off_od);
  const uint32_t seg_a = smem_u32(smem + L.off_seg), perm_a = smem_u32(smem + L.off_perm);
  const uint32_t nlab_a = smem_u32(smem + L.off_nlab), hlist_a = smem_u32(smem + L.off_hlist);
  const uint32_t red_a = smem_u32(smem + L.off_red), redi_a = smem_u32(smem + L.off_redi);
  auto e_full = [&](int s) { return bars + 8u * (uint32_t)s; };
  auto e_empty = [&](int s) { return bars + 8u * (uint32_t)(kSE + s); };
  auto o_full = [&](int s) { return bars + 8u * (uint32_t)(2 * kSE + s); };
  auto o_empty = [&](int s) { return bars + 8u * (uint32_t)(2 * kSE + kSO + s); };
  auto g_full = [&](int s) { return bars + 8u * (uint32_t)(2 * kSE + 2 * kSO + s); };
  auto g_empty = [&](int s) { return bars + 8u * (uint32_t)(2 * kSE + 2 * kSO + kSG + s); };
  const uint32_t tbl_ready = bars + 8u * (uint32_t)(2 * kSE + 2 * kSO + 2 * kSG);
  const uint32_t g_base = smem_u32(smem + L.off_g);

  const int n_pairs = (N1 + 1) >> 1; // PAIR: U + 1
  const int nw_act = PAIR ? (n_pairs + 31) >> 5 : (N1 + 31) >> 5; // node warps of THIS utterance
  const int nact = 32 * nw_act;
  const int nblk = (T + kBlk - 1) / kBlk;
  // levels 1..M: alpha saved, posterior by B; M+1..T: beta saved, posterior by A.  T/2 rounded UP to a block: CTA B
  // starts later (it gathers the out-arc tables first), so it gets the shorter first phase and A does not sit at
  // the cluster barrier waiting for it
  const int M = min(((T / 2 + kBlk - 1) / kBlk) * kBlk, (max(T - 1, 0) / kBlk) * kBlk); // (B keeps >= 1 level)
  const int jb = M / kBlk; // blocks [0, jb) belong to B's phase 2, [jb, nblk) to A's
  // blocks this CTA walks, in its own order: A 0, 1, ..; B nblk-1, nblk-2, ..
  const int n_ph1 = dir == 0 ? jb : nblk - jb;
  int n_ph2 = dir == 0 ? nblk - jb : jb;
  // loss only: A needs one more level (for Z), B nothing more
  if (!want_g) n_ph2 = dir == 0 ? (T > 0 ? 1 : 0) : 0;
  const int n_visit = n_ph1 + n_ph2;
  auto block_of = [&](int v) { return dir == 0 ? v : nblk - 1 - v; };
  auto rows_of = [&](int j) { return min(kBlk, T - kBlk * j); };
  float* boff_own = P.boff + ((long long)(2 * b + dir) * P.nblk_cap) * 4;
  const float* boff_oth = P.boff + ((long long)(2 * b + (1 - dir)) * P.nblk_cap) * 4;

  if (tid == 0) {
    for (int s = 0; s < kSE; s++) {
      mbar_init(e_full(s), 1);
      mbar_init(e_empty(s), nw_act + kHelpers);
    }
    for (int s = 0; s < kSO; s++) {
      mbar_init(o_full(s), 1);
      mbar_init(o_empty(s), nw_act);
    }
    for (int s = 0; s < kSG; s++) {
      mbar_init(g_full(s), nw_act);
      mbar_init(g_empty(s), kHelpers);
    }
    mbar_init(tbl_ready, kHelpers);
    mbar_init_fence();
  }
  // chain rows: everything kNeg (the dummy slot stays that way for good)
  for (int i = tid; i < 2 * kRowF; i += blockDim.x) ring[i] = kNeg;
  // posterior blocks: all zero -- the slots no node writes to must read as 0 for good
  if (want_g)
    for (int i = tid; i < kSG * (L.g_block_bytes >> 2); i += blockDim.x) sts_f32(g_base + 4u * i, 0.0f);
  if (tid < 2) sts_u32(redi_a + 4u * tid, (uint32_t)kIntMin);

  const uint8_t* fl = P.sg_flags + m.sg_node_base;
  const int32_t* ip = P.sg_in_ptr + m.sg_node_base;
  const int32_t* is = P.sg_in_src + m.sg_arc_base;
  const int32_t* il = P.sg_in_label + m.sg_arc_base;
  const float* iw = P.sg_in_w + m.sg_arc_base;
  const E* em = static_cast<const E*>(P.emissions) + m.emis_off;
  float* saved = P.saved + m.node_base;

  // B: the out-arcs of every node, gathered from the in-arc tables (scratch aliases the score stages)
  int* o_cnt = reinterpret_cast<int*>(smem + L.off_o);
  int* o_dst = o_cnt + kMaxNodes;
  float* o_w = reinterpret_cast<float*>(o_dst + 3 * kMaxNodes);
  if (dir == 1)
    for (int i = tid; i < kMaxNodes; i += blockDim.x) o_cnt[i] = 0;
  __syncthreads();
  bool bad = false;
  int my_lab = 0, my_deg = 0;
  const int32_t* tg = MODE != 0 ? P.targets + m.tgt_off : nullptr; // this utterance's labels
  if (MODE != 0) {
    // CTC target graph: node n carries blank (even n) or label (n - 1) / 2 (odd n)
    if (tid < N1) sts_s8(nlab_a + (uint32_t)tid, (tid & 1) ? tg[(tid - 1) >> 1] : P.ctc_blank);
  } else if (tid < N1) {
    const int e0 = ip[tid];
    my_deg = ip[tid + 1] - e0;
    if (my_deg > 0) my_lab = il[e0];
    // node labels for the helper warps' tables
    sts_s8(nlab_a + (uint32_t)tid, my_deg > 0 ? my_lab : -1);
    if (dir == 1)
      for (int k = 0; k < my_deg; k++) {
        const int s = is[e0 + k];
        const int slot = atomicAdd(&o_cnt[s], 1);
        if (slot < 3) {
          o_dst[3 * s + slot] = tid;
          o_w[3 * s + slot] = iw[e0 + k];
        }
      }
  }
  __syncthreads();

  if (PAIR && warp < P.nwn) {
    /* ============================ node warps, two nodes per thread ============================ */
    const bool act = tid < n_pairs;
    const int tp = min(tid, n_pairs - 1); // threads beyond the last pair clone it
    const bool has_label = tp >= 1;
    PairState ps;
    ps.t8 = 8u * (uint32_t)tp;
    const int lnode = 2 * tp - 1;
    // A: does this thread's label have the skip in-arc; B: does the NEXT label (= this label's skip out-arc)
    const int sk_node = dir == 0 ? lnode : lnode + 2;
    ps.skip = ctc_skip(tg, sk_node, N1);
    const int labn = has_label ? tg[tp - 1] : P.ctc_blank;
    __syncthreads(); // (S1) all roles
    if (warp >= nw_act) {
      cluster_sync_all();
      return;
    }
    ps.pc = smem_u32(ring);
    ps.qc = smem_u32(ring + kRowF);
    ps.gs = nullptr;
    ps.al = ps.ab = kNeg;
    ps.Zh = ps.zsub = ps.Zl = ps.Dc = 0.0f;
    ps.adj = ps.D = 0.0f;
    ps.ea_l = ps.ea_b = ps.oa = ps.ga = 0;
    ps.redi = redi_a;
    NodeCtx cx;
    cx.fl = fl;
    cx.saved = saved;
    cx.boff_own = boff_own;
    cx.out_score = P.out_scores + b;
    cx.bars = bars;
    cx.e_base = e_base;
    cx.o_base = o_base;
    cx.g_base = g_base;
    cx.od_base = od_base;
    cx.perm_a = perm_a;
    cx.red_a = red_a;
    cx.spare = 0;
    cx.lab4 = (uint32_t)sizeof(E) * (uint32_t)labn;
    cx.blank4 = (uint32_t)sizeof(E) * (uint32_t)P.ctc_blank;
    cx.feas_a = hlist_a + 96u;
    cx.e_stage_bytes = L.e_stage_bytes;
    cx.o_stage_bytes = L.o_stage_bytes;
    cx.g_block_bytes = L.g_block_bytes;
    cx.pg = L.pg;
    cx.C = C;
    cx.T = T;
    cx.N1 = N1;
    cx.pitch = pitch;
    cx.nblk = nblk;
    cx.n_ph1 = n_ph1;
    cx.n_ph2 = n_ph2;
    cx.nw_act = nw_act;
    cx.want_g = want_g;
    if (dir == 0)
      pair_role<0, NQ, E>(ps, cx, tp, act, has_label);
    else
      pair_role<1, NQ, E>(ps, cx, tp, act, has_label);
    if (T == 0 && dir == 0 && tid == 0) {
      int n = 0;
      for (int i = 0; i < N1; i++) n += (ctc_flags(i, N1) & 3) == 3;
      P.out_scores[b] = n ? logf((float)n) : -CUDART_INF_F;
    }
    return;
  }
  if (MODE == 0 && warp < P.nwn) {
    /* ============================ node warps ============================ */
    NodeState st;
    const bool act = tid < N1;
    const int nid = min(tid, N1 - 1); // threads beyond the last node clone it (NodeUni)
    st.u4 = 4u * (uint32_t)nid;
    int nb_[3] = {kDummy, kDummy, kDummy};
    float wb_[3] = {0.0f, 0.0f, 0.0f};
    const int e0n = ip[nid], degn = ip[nid + 1] - e0n;
    const int labn = degn > 0 ? il[e0n] : 0;
    if (dir == 0) {
      for (int k = 0; k < degn && k < 3; k++) {
        nb_[k] = is[e0n + k];
        wb_[k] = iw[e0n + k];
      }
    } else {
      const int od = min(o_cnt[nid], 3);
      for (int k = 0; k < od; k++) {
        nb_[k] = o_dst[3 * nid + k];
        wb_[k] = o_w[3 * nid + k];
      }
      // the atomics filled the slots in arbitrary order: sort by (node, weight) so that the sum of
      // the three exponentials is evaluated in a fixed order
#define GTNB_CSWAP(a, b)                                                          \
  if (nb_[a] > nb_[b] || (nb_[a] == nb_[b] && wb_[a] > wb_[b])) {                \
    const int tn = nb_[a];                                                        \
    nb_[a] = nb_[b];                                                              \
    nb_[b] = tn;                                                                  \
    const float tw = wb_[a];                                                      \
    wb_[a] = wb_[b];                                                              \
    wb_[b] = tw;                                                                  \
  }
      GTNB_CSWAP(0, 1) GTNB_CSWAP(1, 2) GTNB_CSWAP(0, 1)
#undef GTNB_CSWAP
    }
    bad |= !finite_ok(wb_[0]) || !finite_ok(wb_[1]) || !finite_ok(wb_[2]);
    st.so0 = 4u * (uint32_t)nb_[0];
    st.so1 = 4u * (uint32_t)nb_[1];
    st.so2 = 4u * (uint32_t)nb_[2];
    // the scratch is about to be overwritten by the score stages: everybody is done reading it
    __syncthreads(); // (S1) all roles
    if (warp >= nw_act) { // node warp without a node of this utterance
      cluster_sync_all();
      return;
    }
    st.pc = smem_u32(ring);
    st.qc = smem_u32(ring + kRowF);
    const uint32_t spare = smem_u32(ring) + 4u * (kDummy + 1); // a word of the chain row nobody reads
    st.gs = nullptr;
    st.Zh = st.zsub = st.Zl = st.Dc = 0.0f;
    st.adj = st.D = 0.0f;
    st.ea = st.oa = 0;
    st.ga = spare;
    st.redi = redi_a;
    const uint32_t lab4 = (uint32_t)sizeof(E) * (uint32_t)labn;

    NodeCtx cx;
    cx.fl = fl;
    cx.saved = saved;
    cx.boff_own = boff_own;
    cx.out_score = P.out_scores + b;
    cx.bars = bars;
    cx.e_base = e_base;
    cx.o_base = o_base;
    cx.g_base = g_base;
    cx.od_base = od_base;
    cx.perm_a = perm_a;
    cx.red_a = red_a;
    cx.spare = spare;
    cx.lab4 = lab4;
    cx.blank4 = 0;
    cx.feas_a = hlist_a + 96u;
    cx.e_stage_bytes = L.e_stage_bytes;
    cx.o_stage_bytes = L.o_stage_bytes;
    cx.g_block_bytes = L.g_block_bytes;
    cx.pg = L.pg;
    cx.C = C;
    cx.T = T;
    cx.N1 = N1;
    cx.pitch = pitch;
    cx.nblk = nblk;
    cx.n_ph1 = n_ph1;
    cx.n_ph2 = n_ph2;
    cx.nw_act = nw_act;
    cx.want_g = want_g;
    if (dir == 0)
      node_role<0, NQ, FX, E>(st, cx, act, nid);
    else
      node_role<1, NQ, FX, E>(st, cx, act, nid);
    if (bad) *(volatile int32_t*)&P.status[b] = 1; // (every writer stores the same 1: no atomic needed)
    if (T == 0 && dir == 0 && tid == 0) {
      // no frames: the lattice is the graph's start-and-accept nodes, each with score 0
      int n = 0;
      for (int i = 0; i < N1; i++) n += (fl[i] & 3) == 3;
      P.out_scores[b] = n ? logf((float)n) : -CUDART_INF_F;
    }
    return;
  }

  __syncthreads(); // (S1)

  if (warp > P.nwn + kHelpers) { // (no launch has warps beyond the helpers; without this test ptxas schedules every kernel differently)
    cluster_sync_all();
    return;
  }
  if (warp == P.nwn) {
    /* ============================ producer warp: TMA bulk copies ============================ */
    // Emission blocks all the way, and in phase 2 the partner's saved scores (with the block's offset).
    // The emission copies run ahead of the math across the phase boundary, so the warp must not be what
    // the others' cluster barrier waits for: it ARRIVES right away and WAITS only before the first copy
    // that reads what the partner wrote.
    cluster_arrive_only();
    bool waited = false;
    for (int v = 0; v < n_visit; v++) {
      const int s = v % kSE, j = block_of(v);
      if (lane == 0) {
        if (v >= kSE) mbar_wait_suspend(e_empty(s), ((v / kSE) - 1) & 1);
        const uint32_t bytes = (uint32_t)(rows_of(j) * C * (int)sizeof(E));
        mbar_expect_tx(e_full(s), bytes);
        bulk_g2s(e_base + (uint32_t)(s * L.e_stage_bytes), em + (long long)j * kBlk * C, bytes, e_full(s));
      }
      if (v >= n_ph1) {
        const int v2 = v - n_ph1, so = v2 % kSO;
        if (!waited) {
          __syncwarp();
          cluster_wait_only();
          // the partner's saved scores were written with ordinary stores; the bulk copies read them
          // through the async proxy
          fence_proxy_async();
          waited = true;
        }
        if (lane == 0) {
          if (v2 >= kSO) mbar_wait_suspend(o_empty(so), ((v2 / kSO) - 1) & 1);
          // PAIR: the label rows, plus the meeting row's blank scores behind them in the first block
          const uint32_t bytes = PAIR ? (uint32_t)((rows_of(j) + (v2 == 0)) * kHalfPitch * 4) : (uint32_t)(rows_of(j) * pitch * 4);
          mbar_expect_tx(o_full(so), bytes + 16u);
          bulk_g2s(o_base + (uint32_t)(so * L.o_stage_bytes), saved + (long long)j * kBlk * pitch, bytes, o_full(so));
          bulk_g2s(od_base + 16u * so, boff_oth + 4 * j, 16u, o_full(so));
        }
      }
    }
    __syncwarp();
    if (!waited) cluster_wait_only();
    return;
  }

  /* ============================ helper warps ============================ */
  HelperState hs;
  hs.hw = warp - P.nwn - 1;
  hs.lane = lane;
  hs.r = 2 * hs.hw + (lane >> 4);
  hs.l16 = lane & 15;
  hs.C = C;
  hs.seg = seg_a;
  hs.zacc = 0.0f;
  hs.bad = false;
  const int ht = hs.hw * 32 + lane; // index among the helper threads
  int nheavy = 0;
  if (want_g) {
    // Positions in a posterior row.  A label carried by n <= kSlots nodes: its nodes (ascending ids) take the
    // slots kSlots * c + 0 .. n-1.  A label carried by more: its nodes take consecutive overflow positions
    // behind the slots.  Nodes without in-arcs (they exist at level 0 only) go behind everything.
    for (int c = ht; c < C; c += 32 * kHelpers) {
      int n = 0;
      for (int u = 0; u < N1; u++) n += lds_s8(nlab_a + (uint32_t)u) == c;
      sts_u32(seg_a + 4u * c, (uint32_t)n);
    }
    bar_named(2, 32 * kHelpers);
    if (ht == 0) {
      // the label with the most nodes, when it has more than kSlots (CTC: blank): the complement label
      int comp = -1, cn = kSlots;
      for (int c = 0; c < C; c++) {
        const int n = (int)lds_u32(seg_a + 4u * c);
        if (n > cn) {
          cn = n;
          comp = c;
        }
      }
      if (MODE != 0) comp = P.ctc_blank; // the pair threads never form a blank posterior, whatever U is
      sts_u32(hlist_a + 100u, (uint32_t)comp);
      int nh = 0, at = 0;
      for (int c = 0; c < C; c++) {
        const int n = (int)lds_u32(seg_a + 4u * c);
        if (c == comp) {
          sts_u32(seg_a + 4u * c, seg_pack(0, n, 14));
        } else if (n > kSlots) {
          int slot1 = 15;
          if (nh < kMaxHeavy) {
            sts_u32(hlist_a + 4u * nh, (uint32_t)c);
            slot1 = ++nh;
          }
          sts_u32(seg_a + 4u * c, seg_pack(at, n, slot1));
          at += n;
        } else {
          sts_u32(seg_a + 4u * c, seg_pack(0, n, 0));
        }
      }
      sts_u32(hlist_a + 4u * kMaxHeavy, (uint32_t)nh);
      for (int u = 0; u < N1; u++)
        if (lds_s8(nlab_a + (uint32_t)u) < 0) sts_u16(perm_a + 2u * u, 4u * (uint32_t)(kSlots * C + at++));
    }
    bar_named(2, 32 * kHelpers);
    nheavy = (int)lds_u32(hlist_a + 4u * kMaxHeavy);
    for (int c = ht; c < C; c += 32 * kHelpers) {
      const uint32_t w = lds_u32(seg_a + 4u * c);
      const uint32_t s1 = w >> 20;
      // the complement label's nodes all store into the row's last word, which nobody reads (with >= 5 of them
      // out of the overflow area it is never an overflow position)
      uint32_t at = s1 == 14u ? (uint32_t)(L.pg - 1) : s1 ? (uint32_t)(kSlots * C) + (w & 1023u) : (uint32_t)(kSlots * c);
      for (int u = 0; u < N1; u++)
        if (lds_s8(nlab_a + (uint32_t)u) == c) sts_u16(perm_a + 2u * u, 4u * (s1 == 14u ? at : at++));
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(tbl_ready);
    bar_named(2, 32 * kHelpers); // seg is complete before anybody reads other threads' entries below
  }
  HelperConst<NQ> hk;
#pragma unroll
  for (int i = 0; i < NQ; i++) {
    const int c = 4 * (hs.l16 + 16 * i);
    hk.eoff[i] = c < C ? (uint32_t)(hs.r * C + c) * (uint32_t)sizeof(E) : 0xffffffffu;
    hk.goff[i] = (uint32_t)(hs.r * L.pg + kSlots * c) * 4u;
    hk.hsel[i] = 0;
    if (want_g && c < C)
      for (int j = 0; j < 4; j++) hk.hsel[i] |= ((lds_u32(seg_a + 4u * (c + j)) >> 20) & 15u) << (4 * j);
  }
  hk.ovf = (uint32_t)(hs.r * L.pg + kSlots * C) * 4u;
#pragma unroll
  for (int h = 0; h < kMaxHeavy; h++) {
    hk.hoff[h] = 0;
    hk.hlen[h] = 0;
    if (want_g && h < nheavy) {
      const uint32_t w = lds_u32(seg_a + 4u * lds_u32(hlist_a + 4u * h));
      hk.hoff[h] = hk.ovf + (w & 1023u) * 4u;
      hk.hlen[h] = (int)((w >> 10) & 1023u);
    }
  }
  int v = 0;
  if (!want_g) {
    for (; v < n_ph1; v++) {
      const int s = v % kSE;
      mbar_wait_suspend(e_full(s), (v / kSE) & 1);
      helper_block<NQ, false, E>(hs, hk, rows_of(block_of(v)), e_base + (uint32_t)(s * L.e_stage_bytes), e_empty(s), 0, 0,
                              0, false, 0, nullptr);
    }
  }
  cluster_sync_all();
  if (want_g) {
    v = n_ph1;
    // the common shape takes helper_block_fast (warp-uniform, in fact CTA-uniform, decision)
    int n15 = 0;
    for (int c = 0; c < C; c++) n15 += ((lds_u32(seg_a + 4u * c) >> 20) & 15u) == 15u;
    const bool fast = C == 64 * NQ && n15 == 0;
    // label | overflow start << 8 | nodes << 18 of the cooperative labels, for helper_block_fast
    const uint32_t htab = hlist_a + 4u * (kMaxHeavy + 1);
    if (lane < nheavy) { // (every helper warp writes the same values)
      const uint32_t hc = lds_u32(hlist_a + 4u * lane), w = lds_u32(seg_a + 4u * hc);
      sts_u32(htab + 4u * lane, hc | ((w & 1023u) << 8) | (((w >> 10) & 1023u) << 18));
    }
    __syncwarp();
    const int comp = (int)lds_u32(hlist_a + 100u);
    const bool has_comp = comp >= 0;
    const int comp_rel = has_comp ? comp - 4 * hs.l16 : -1000;
    const uint32_t feas_a = hlist_a + 96u;
    const uint32_t f_e = (uint32_t)(hs.r * C + 4 * hs.l16) * (uint32_t)sizeof(E), f_g = (uint32_t)(hs.r * L.pg + kSlots * 4 * hs.l16) * 4u;
    E* const grad = static_cast<E*>(P.grad);
    E* const f_out = grad + (long long)b * P.grad_stride + hs.r * C + 4 * hs.l16;
    for (int v2 = 0; v2 < n_ph2; v2++, v++) {
      const int s = v % kSE, sg = v2 % kSG, j = block_of(v);
      // the node warps arrive on g_full after they are through the block: its emission stage was
      // complete long before that (they waited for it), so one wait covers both
      mbar_wait_suspend(g_full(sg), (v2 / kSG) & 1);
      if (fast && rows_of(j) == kBlk) {
        const uint32_t gb = g_base + (uint32_t)(sg * L.g_block_bytes);
        helper_block_fast<NQ, E>(hs, e_base + (uint32_t)(s * L.e_stage_bytes) + f_e, e_empty(s), gb + f_g, gb + hk.ovf, htab,
                              nheavy, has_comp, comp_rel, feas_a, g_empty(sg), f_out + (long long)j * kBlk * C);
        continue;
      }
      helper_block<NQ, true, E>(hs, hk, rows_of(j), e_base + (uint32_t)(s * L.e_stage_bytes), e_empty(s),
                             g_base + (uint32_t)(sg * L.g_block_bytes), g_empty(sg), nheavy, has_comp, feas_a,
                             grad + (long long)b * P.grad_stride + (long long)j * kBlk * C);
    }
  }
  // forwardScore(emissions): the rows this warp summed
  float z = hs.l16 == 0 ? hs.zacc : 0.0f;
  z += __shfl_xor_sync(0xffffffffu, z, 16);
  if (lane == 0) P.zparts[(2 * b + dir) * kHelpers + hs.hw] = z;
  if (hs.bad) *(volatile int32_t*)&P.status[b] = 1;
}

} // namespace bidir

/* launch_bidir_ctc's kernel and geometry */
struct BidirPlan {
  void (*kernel)(const bidir::Params);
  bool fx; // compile-time strides over saved-score rows of the fixed pitch
  bool pair; // the PAIR kernels (two nodes per thread), which read the CTC graphs from the targets themselves
  int nwn; // node warps
  bidir::Layout lay;
  unsigned block; // threads per CTA
};

/*
 * For C labels, levels of at most max_nodes nodes, saved-score rows of the fixed pitch (fixed_pitch: gtnb_compose_linear,
 * implicit lattices) or of each graph's node count rounded up to 4, and emissions and gradient of type E.  pair_ok: the
 * graphs are ctc_build_kernel's (gtnb_ctc_loss) with the targets at hand, and gtnb_ctx_set_flag("bidir_mode", 0) does
 * not ask for one node per thread.
 */
template <class E>
BidirPlan bidir_plan(int C, int max_nodes, bool fixed_pitch, bool pair_ok) {
  BidirPlan p;
  // FX: the benchmark's shapes (C == 64 or 128)
  p.fx = (C == 64 || C == 128) && fixed_pitch;
  p.pair = p.fx && pair_ok && max_nodes <= 2 * 32 * bidir::kMaxPairWarps - 1;
  // NQ: float4 chunks of an emission row per helper lane
  if (p.pair)
    p.kernel = C == 64 ? bidir::bidir_ctc_kernel<1, true, 1, E> : bidir::bidir_ctc_kernel<2, true, 1, E>;
  else if (p.fx)
    p.kernel = C == 64 ? bidir::bidir_ctc_kernel<1, true, 0, E> : bidir::bidir_ctc_kernel<2, true, 0, E>;
  else
    p.kernel = C <= 64 ? bidir::bidir_ctc_kernel<1, false, 0, E> : bidir::bidir_ctc_kernel<2, false, 0, E>;
  p.nwn = std::max(1, ((p.pair ? (max_nodes + 1) / 2 : max_nodes) + 31) / 32);
  p.lay = bidir::make_layout(C, p.fx ? bidir::kFixedPitch : ((max_nodes + 3) & ~3), (int)sizeof(E));
  p.block = 32 * (p.nwn + 1 + bidir::kHelpers);
  return p;
}

#ifndef GTNB_HOST_EMU

static_assert(bidir::kFixedPitch == kImplicitFixedPitch, "gtnb_compose_linear allocates the rows");

/* true when every utterance of the batch qualifies for the bidirectional kernel with emissions and gradients of
 * type dtype (GTNB_F32 / GTNB_BF16 / GTNB_F16).  16-bit elements need C % 8 == 0: every TMA row copy and every 8-byte
 * access of the helper warps then stays a multiple of 16 / 8 bytes */
bool bidir_supported(const gtnb_lattice* lat, const void* emissions, int64_t stride, const void* grad, int64_t grad_stride,
                     int dtype) {
  if (!lat->composed || lat->C % 4 != 0 || lat->C > 128 || lat->C < 4) return false;
  if (dtype != GTNB_F32 && lat->C % 8 != 0) return false;
  if (lat->max_lvl_nodes > 32 * bidir::kMaxNodeWarps || lat->max_in_deg > 3 || lat->max_out_deg > 3) return false;
  if (((uintptr_t)emissions & 15) || (stride & 3)) return false;
  if (grad && (((uintptr_t)grad & 15) || (grad_stride & 3))) return false;
  for (int b = 0; b < lat->B; b++)
    if (!lat->meta_h[b].sg_uniform || !lat->meta_h[b].sg_all_valid || lat->meta_h[b].sg_N < 1) return false;
  // the saved-score rows: the graph's node count rounded up to 4, or the fixed pitch of the FX kernels
  if (lat->score_pitch != 0 && lat->score_pitch != bidir::kFixedPitch) return false;
  return true;
}

/* true when launch_bidir_ctc would run its PAIR kernels, which read the CTC target graphs from the targets
 * themselves: the caller (gtnb_ctc_loss) then skips ctc_build_kernel altogether */
bool bidir_takes_targets(const gtnb_lattice* lat, int ctc_blank) {
  return bidir_plan<float>(lat->C, lat->max_lvl_nodes, lat->score_pitch == bidir::kFixedPitch,
                           ctc_blank >= 0 && ctc_blank < lat->C)
      .pair;
}

/* blocks of 8 frames per utterance: boff_dev holds B * 2 * bidir_blocks(max T) * 4 floats */
int bidir_blocks(int max_T) {
  return std::max(1, (max_T + bidir::kBlk - 1) / bidir::kBlk);
}

/* utterances [b0, b0 + nb): one cluster of two CTAs each, on ctx->stream.  zparts_dev: [2 * B * bidir_zparts()] */
int bidir_zparts() {
  return bidir::kHelpers;
}
int launch_bidir_ctc(
    gtnb_ctx* ctx, gtnb_lattice* lat, int32_t* status_dev, float* zparts_dev, float* boff_dev, void* grad_emis,
    int64_t grad_stride, int b0, int nb, float* out_scores_dev, int ctc_blank, const int32_t* targets_dev,
    const int32_t* tgt_off_dev, const GraphMeta* meta_src, int dtype) {
  const int esize = dtype == GTNB_F32 ? 4 : 2;
  if (nb < 0) nb = lat->B - b0;
  if (nb <= 0) return GTNB_OK;
  bidir::Params P;
  P.meta = (meta_src ? meta_src : lat->meta) + b0;
  P.sg_flags = lat->sg_flags;
  P.sg_in_ptr = lat->sg_in_ptr;
  P.sg_in_src = lat->sg_in_src;
  P.sg_in_label = lat->sg_in_label;
  P.sg_in_w = lat->sg_in_w;
  P.emissions = lat->emissions;
  P.saved = lat->scores;
  P.nblk_cap = bidir_blocks(lat->max_T);
  P.boff = boff_dev + (long long)b0 * 2 * P.nblk_cap * 4;
  P.out_scores = (out_scores_dev ? out_scores_dev : lat->out_scores) + b0;
  P.zparts = zparts_dev + 2ll * b0 * bidir::kHelpers;
  P.status = status_dev + b0;
  P.grad = grad_emis ? static_cast<char*>(grad_emis) + (long long)b0 * grad_stride * esize : nullptr;
  P.grad_stride = grad_stride;
  P.C = lat->C;
  (void)tgt_off_dev; // (the offsets travel in the descriptors: GraphMeta::tgt_off)
  P.targets = targets_dev;
  P.ctc_blank = ctc_blank;
  const bool fixed = lat->score_pitch == bidir::kFixedPitch;
  const bool pair_ok = targets_dev && ctc_blank >= 0 && ctc_blank < lat->C && ctx->bidir_mode != 0;
  const BidirPlan p = dtype == GTNB_BF16  ? bidir_plan<bf16_t>(lat->C, lat->max_lvl_nodes, fixed, pair_ok)
                      : dtype == GTNB_F16 ? bidir_plan<f16_t>(lat->C, lat->max_lvl_nodes, fixed, pair_ok)
                                          : bidir_plan<float>(lat->C, lat->max_lvl_nodes, fixed, pair_ok);
  P.nwn = p.nwn;
  P.lay = p.lay;
  if (P.lay.total > 48 * 1024) {
    int rc = ensure_max_smem(ctx, (const void*)p.kernel);
    if (rc) return rc;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(2 * nb, 1, 1);
  cfg.blockDim = dim3(p.block, 1, 1);
  cfg.dynamicSmemBytes = P.lay.total;
  cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  GTNB_LAUNCH(ctx, "bidir_ctc", GTNB_CUDA(ctx, cudaLaunchKernelEx(&cfg, p.kernel, P)));
  return GTNB_OK;
}

#endif // GTNB_HOST_EMU

} // namespace gtnb
