/*
 * gtnb_product.h -- host-only: the product of a user target graph A with a dense transition graph G, the numerator
 * graph of gtnb_graph_transitions_loss.  Plain C++ (no CUDA), so the CPU emulation harness builds the same code.
 *
 * G is label-deterministic: every arc into a G state carries that state's label.  A state of compose(A, G) (ASG) or
 * intersect(A, G) (BIGRAM) is therefore (A node v, previous label l), and one O(N + A) pass with per-node label
 * bitmasks builds it:
 *  - node v gets one copy (v, l) per distinct in-label l in [0, C);
 *  - ASG: one more copy per start node u, (u, G's node 0), the only start states; it does not accept (G's node 0
 *    does not);  BIGRAM unfolded: a start node u has all C copies (u, j), every one a start state;
 *  - arc a: u -> v with olabel l gives one arc from every copy of u to (v, l), of weight w_a + s[l] from an ASG
 *    start copy and w_a + W[l][g] from (u, g) (the reference's adds in its association, compose.cpp:435);
 *  - copies of accept nodes accept (except ASG's start copies).
 * BIGRAM folded (the device route): the C start states collapse into one start node S with one arc S -> (v, l) per
 * out-arc of a start node, weight w_a + sigma_l, sigma_l = logsumexp_j W[l][j] (k_ngram.cu's fold for CTC); a start
 * node with in-arcs keeps its in-label copies for frames >= 1.
 * Arcs labelled outside [0, C) never match and give no product arc.  Every product arc records arc_of (the A arc it
 * came from) and tidx (the slot of Wx it reads): Wx = trans_w ([C + C*C]) for ASG, [W | sigma] ([C*C + C]) for
 * BIGRAM.  Its weight is w_A[arc_of] + Wx[tidx].
 */
#pragma once

#include <algorithm>
#include <cstdint>
#include <vector>

#include "gtn_b200.h"

namespace gtnb {

struct ProductGraph {
  std::vector<uint8_t> flags; // bit 0 start, bit 1 accept
  std::vector<int32_t> src, dst, label;
  std::vector<int32_t> arc_of; // A arc of every product arc
  std::vector<int32_t> tidx; // slot of Wx of every product arc
  int n_acc = 0, max_in = 0, max_out = 0;

  gtnb_graph_view view() const {
    gtnb_graph_view v{};
    v.num_nodes = (int)flags.size();
    v.num_arcs = (int)src.size();
    v.node_flags = flags.data();
    v.arc_src = src.data();
    v.arc_dst = dst.data();
    v.arc_ilabel = v.arc_olabel = label.data();
    return v;
  }
};

/* A's epsilon arcs are the caller's to reject; C <= 128 (four mask words per node) */
inline void build_product(const gtnb_graph_view& A, int C, bool bigram, bool fold, ProductGraph* p) {
  const int N = A.num_nodes, nA = A.num_arcs;
  auto lab_of = [&](int a) { return A.arc_olabel[a]; };
  auto valid = [&](int l) { return l >= 0 && l < C; };
  auto is_start = [&](int v) { return (A.node_flags[v] & 1) != 0; };
  std::vector<uint32_t> mask(4 * (size_t)N, 0u);
  for (int a = 0; a < nA; a++)
    if (valid(lab_of(a))) mask[4 * (size_t)A.arc_dst[a] + (lab_of(a) >> 5)] |= 1u << (lab_of(a) & 31);
  // node layout per A node v: [ASG start copy] [in-label copies, ascending]; BIGRAM unfolded start node: C copies
  const bool all_copies = bigram && !fold;
  std::vector<int32_t> base(N + 1, 0), rank(4 * (size_t)N, 0); // rank[w]: copies before mask word w
  int next = (bigram && fold) ? 1 : 0; // node 0 = S
  for (int v = 0; v < N; v++) {
    base[v] = next;
    if (all_copies && is_start(v)) {
      next += C;
      continue;
    }
    if (!bigram && is_start(v)) next++;
    for (int w = 0; w < 4; w++) {
      rank[4 * (size_t)v + w] = next - base[v];
      next += __builtin_popcount(mask[4 * (size_t)v + w]);
    }
  }
  base[N] = next;
  auto copy = [&](int v, int l) { // node of (v, l), l an in-label of v (or any label of an unfolded start node)
    if (all_copies && is_start(v)) return base[v] + l;
    const uint32_t below = mask[4 * (size_t)v + (l >> 5)] & ((1u << (l & 31)) - 1u);
    return base[v] + rank[4 * (size_t)v + (l >> 5)] + __builtin_popcount(below);
  };
  p->flags.assign(std::max(next, 1), 0); // (an empty product keeps one node that neither starts nor accepts)
  if (bigram && fold) p->flags[0] = 1;
  for (int v = 0; v < N; v++) {
    const bool acc = (A.node_flags[v] & 2) != 0;
    const bool start_copy = !bigram && is_start(v);
    for (int n = base[v]; n < base[v + 1]; n++) {
      const bool sc = start_copy && n == base[v];
      p->flags[n] = (uint8_t)((sc || (all_copies && is_start(v)) ? 1 : 0) | (acc && !sc ? 2 : 0));
    }
  }
  p->src.clear();
  p->dst.clear();
  p->label.clear();
  p->arc_of.clear();
  p->tidx.clear();
  const int nW = bigram ? C * C : C + C * C; // Wx: where W ends (BIGRAM: sigma follows)
  auto put = [&](int s, int d, int l, int a, int t) {
    p->src.push_back(s);
    p->dst.push_back(d);
    p->label.push_back(l);
    p->arc_of.push_back(a);
    p->tidx.push_back(t);
  };
  for (int a = 0; a < nA; a++) {
    const int l = lab_of(a);
    if (!valid(l)) continue;
    const int u = A.arc_src[a], d = copy(A.arc_dst[a], l);
    const int wrow = bigram ? l * C : C + l * C; // W[l][.] in Wx
    if (all_copies && is_start(u)) {
      for (int g = 0; g < C; g++) put(base[u] + g, d, l, a, wrow + g);
      continue;
    }
    if (is_start(u)) {
      if (bigram)
        put(0, d, l, a, nW + l); // S -> (v, l), weight w_a + sigma_l
      else
        put(base[u], d, l, a, l); // ASG start copy: w_a + s[l]
    }
    for (int w = 0; w < 4; w++)
      for (uint32_t m = mask[4 * (size_t)u + w]; m; m &= m - 1) {
        const int g = 32 * w + __builtin_ctz(m);
        put(copy(u, g), d, l, a, wrow + g);
      }
  }
  std::vector<int32_t> indeg(p->flags.size(), 0), outdeg(p->flags.size(), 0);
  for (size_t k = 0; k < p->src.size(); k++) {
    indeg[p->dst[k]]++;
    outdeg[p->src[k]]++;
  }
  p->max_in = *std::max_element(indeg.begin(), indeg.end());
  p->max_out = *std::max_element(outdeg.begin(), outdeg.end());
  p->n_acc = (int)std::count_if(p->flags.begin(), p->flags.end(), [](uint8_t f) { return (f & 2) != 0; });
}

/* the product's arc weights: w[k] = w_A[arc_of[k]] + Wx[tidx[k]] (w_A NULL: every A weight 0) */
inline void product_weights(const ProductGraph& p, const float* w_A, const float* Wx, std::vector<float>* w) {
  w->resize(p.src.size());
  for (size_t k = 0; k < p.src.size(); k++) (*w)[k] = (w_A ? w_A[p.arc_of[k]] : 0.0f) + Wx[p.tidx[k]];
}

} // namespace gtnb
