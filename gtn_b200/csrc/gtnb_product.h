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
#include <unordered_map>
#include <vector>

#include "gtn_b200.h"
#include "gtnb_meta.h"

namespace gtnb {

struct ProductGraph {
  std::vector<uint8_t> flags; // bit 0 start, bit 1 accept
  std::vector<int32_t> src, dst, label;
  std::vector<int32_t> arc_of; // A arc of every product arc
  std::vector<int32_t> tidx; // slot of Wx of every product arc
  int n_acc = 0, max_in = 0, max_out = 0;
  bool uniform = true; // every node's in-arcs carry one label (build_sparse_product: not always)

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

/*
 * G of gtnb_sparse_transitions_loss: an epsilon-free acceptor of any shape, weights in trans_w by G's arc id.  Arcs
 * labelled outside [0, C) never match and are left out of every table.
 *  - in_* (by destination) and out_* (by source, ascending label within a source): the denominator's sweeps
 *    (k_sparse.cu) and the product builder;
 *  - the start groups of the fold: the arcs out of start nodes, grouped by (destination, label).  Group k has the
 *    arcs grp_arc[grp_ptr[k] .. grp_ptr[k + 1]); sigma_k = logsumexp of their weights is the weight of the folded
 *    start arcs into that destination with that label.
 */
struct SparseTables {
  int S = 0, A = 0, max_in = 0, max_out = 0;
  std::vector<uint8_t> flags;
  std::vector<int32_t> in_ptr, in_src, in_lab, in_arc;
  std::vector<int32_t> out_ptr, out_dst, out_lab, out_arc;
  std::vector<int32_t> grp_ptr, grp_arc, grp_dst, grp_lab;
  // G's epsilon arcs (sparse_eps_tables; empty for an epsilon-free G), kept apart from the emitting lists above
  int E = 0, L = 0; // epsilon arcs, topological levels
  std::vector<int32_t> eps_in_ptr, eps_in_src, eps_in_arc; // by destination ([S + 1] pointers)
  std::vector<int32_t> eps_out_ptr, eps_out_dst, eps_out_arc; // by source
  std::vector<int32_t> fwd_ptr, fwd_node, bwd_ptr, bwd_node; // [L + 1] pointers: the levels' nodes
  std::vector<int32_t> lanes; // [2L]: threads per node of every forward, then every backward level
  int max_in_all = 0; // the largest in-degree counting both kinds of arc
  std::vector<int32_t> cycle; // the nodes of an epsilon cycle, in arc order, when G has one (then no levels)
};

inline void sparse_tables(const gtnb_graph_view& G, int C, SparseTables* t) {
  const int S = G.num_nodes;
  t->S = S;
  t->flags.assign(G.node_flags, G.node_flags + S);
  std::vector<int32_t> kept;
  for (int g = 0; g < G.num_arcs; g++)
    if (G.arc_olabel[g] >= 0 && G.arc_olabel[g] < C) kept.push_back(g);
  t->A = (int)kept.size();
  auto csr = [&](const int32_t* key, std::vector<int32_t>& order, std::vector<int32_t>& ptr) {
    ptr.assign(S + 1, 0);
    for (int g : kept) ptr[key[g] + 1]++;
    for (int v = 0; v < S; v++) ptr[v + 1] += ptr[v];
    order = kept; // stable: arc id order within a node
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return key[x] < key[y]; });
  };
  std::vector<int32_t> in_order, out_order;
  csr(G.arc_dst, in_order, t->in_ptr);
  csr(G.arc_src, out_order, t->out_ptr);
  for (int u = 0; u < S; u++) // out lists by ascending label (equal_range in build_sparse_product)
    std::stable_sort(out_order.begin() + t->out_ptr[u], out_order.begin() + t->out_ptr[u + 1],
                     [&](int x, int y) { return G.arc_olabel[x] < G.arc_olabel[y]; });
  t->in_src.resize(t->A);
  t->in_lab.resize(t->A);
  t->in_arc = in_order;
  t->out_dst.resize(t->A);
  t->out_lab.resize(t->A);
  t->out_arc = out_order;
  for (int k = 0; k < t->A; k++) {
    t->in_src[k] = G.arc_src[in_order[k]];
    t->in_lab[k] = G.arc_olabel[in_order[k]];
    t->out_dst[k] = G.arc_dst[out_order[k]];
    t->out_lab[k] = G.arc_olabel[out_order[k]];
  }
  t->max_in = t->max_out = 0;
  for (int v = 0; v < S; v++) {
    t->max_in = std::max(t->max_in, t->in_ptr[v + 1] - t->in_ptr[v]);
    t->max_out = std::max(t->max_out, t->out_ptr[v + 1] - t->out_ptr[v]);
  }
  std::unordered_map<long long, int> group;
  std::vector<std::vector<int32_t>> members;
  for (int g : kept) {
    if (!(G.node_flags[G.arc_src[g]] & 1)) continue;
    const long long key = (long long)G.arc_dst[g] * C + G.arc_olabel[g];
    auto it = group.find(key);
    if (it == group.end()) {
      it = group.emplace(key, (int)members.size()).first;
      members.emplace_back();
      t->grp_dst.push_back(G.arc_dst[g]);
      t->grp_lab.push_back(G.arc_olabel[g]);
    }
    members[it->second].push_back(g);
  }
  t->grp_ptr.assign(1, 0);
  t->grp_arc.clear();
  for (const auto& m : members) {
    t->grp_arc.insert(t->grp_arc.end(), m.begin(), m.end());
    t->grp_ptr.push_back((int32_t)t->grp_arc.size());
  }
}

/* N contiguous node ranges with balanced arc counts from a CSR pointer array ptr[S + 1] (plus a second one, eps,
 * when not null: a node's emitting and epsilon arcs counted together): rank r gets the nodes [split[r], split[r + 1]),
 * split[r] the first node at or after arc r * A / N, so that no rank holds more than A / N + the largest degree arcs.
 * A rank may own no node (a hub's list spans several shares). */
inline void sparse_cluster_splits(const std::vector<int32_t>& ptr, int N, int32_t* split,
                                  const std::vector<int32_t>* eps = nullptr) {
  std::vector<int32_t> sum;
  if (eps) {
    sum.resize(ptr.size());
    for (size_t v = 0; v < ptr.size(); v++) sum[v] = ptr[v] + (*eps)[v];
  }
  const std::vector<int32_t>& p = eps ? sum : ptr;
  const int S = (int)p.size() - 1;
  const long long A = p[S];
  split[0] = 0;
  for (int r = 1; r < N; r++)
    split[r] = (int32_t)(std::lower_bound(p.begin(), p.begin() + S, (int32_t)((A * r + N - 1) / N)) - p.begin());
  split[N] = S;
}

/*
 * The cluster size of k_sparse.cu's sparse_cl_* kernels for G = t: the smallest N in {2, 4, 8} (or `force` alone when
 * it is not 0) whose forward and backward sweeps fit the 227 KB of shared memory a CTA can opt in to, with the splits
 * that N gets; 0 when none does or G is outside the kernels' bounds (gtnb_meta.h: S <= 16384 nodes, A <= 262 144
 * arcs, in-degree <= 32 766, C <= 1024).  With C = 64 that is e.g. S = 4096 up to the whole 262 144 arcs (N = 8), or
 * S = 16 384 with 131 072 arcs (N = 8, 194 KB).  *sp gets N and the splits.
 * A G with epsilon arcs (t.E > 0, sparse_eps_tables; the sparse_cl_eps_* kernels) counts them beside the emitting
 * ones: A + E <= 262 144, the splits balance both kinds, own_out holds a rank's emitting and epsilon out-arcs (the
 * backward's accumulators), and L <= kSparseMaxLevels, the combined in-degree below kBpStart.  The backoff 4-gram of
 * 8563 states / 57 231 + 8562 arcs at C = 64 takes N = 2 (about 200 KB).
 */
inline int sparse_cluster_plan(const SparseTables& t, int C, int force, SparseSplit* sp) {
  const bool eps = t.E > 0;
  if (t.S < 1 || t.S > kSparseClusterMaxStates || (long long)t.A + t.E > kSparseClusterMaxArcs || C < 1 ||
      C > kSparseMaxLabels ||
      (eps ? t.L > kSparseMaxLevels || t.max_in_all >= kBpStart : t.max_in > kSparseClusterMaxInDegree))
    return 0;
  for (int N = 2; N <= kSparseClusterMax; N *= 2) {
    if (force && N != force) continue;
    sp->N = N;
    sparse_cluster_splits(t.in_ptr, N, sp->in, eps ? &t.eps_in_ptr : nullptr);
    sparse_cluster_splits(t.out_ptr, N, sp->out, eps ? &t.eps_out_ptr : nullptr);
    sp->own_out = 0;
    for (int r = 0; r < N; r++)
      sp->own_out = std::max(sp->own_out, t.out_ptr[sp->out[r + 1]] - t.out_ptr[sp->out[r]] +
                                              (eps ? t.eps_out_ptr[sp->out[r + 1]] - t.eps_out_ptr[sp->out[r]] : 0));
    const long long floats =
        std::max(sparse_cl_fwd_smem_floats(t.S, C, N), sparse_cl_bwd_smem_floats(t.S, C, N, sp->own_out));
    if (floats * (long long)sizeof(float) <= kSparseClusterSmemBytes) return N;
  }
  return 0;
}

/*
 * The epsilon arcs of G (olabel GTNB_EPSILON; the backoff entry points: ilabel too) into t, after sparse_tables.  An
 * epsilon arc moves G without consuming a frame, so a frame's scores are closed over them in topological order.
 * Kahn's algorithm gives every node a forward level, 0 without epsilon in-arcs, else 1 + the largest level of their
 * sources; levels 1 .. L are t->fwd_* (level l at index l - 1), and a level only reads nodes finished in earlier
 * ones.  The backward levels mirror them over the epsilon out-arcs (0 without any, else 1 + the largest level of
 * their destinations), so that a node's departures are complete before it reads them.  Both number L, the longest
 * epsilon path: a backoff n-gram of order n has n - 1.  A cycle of epsilon arcs leaves t->cycle set (its nodes in
 * arc order) and no levels.
 */
inline void sparse_eps_tables(const gtnb_graph_view& G, SparseTables* t) {
  const int S = t->S;
  std::vector<int32_t> eps;
  for (int g = 0; g < G.num_arcs; g++)
    if (G.arc_olabel[g] == GTNB_EPSILON) eps.push_back(g);
  t->E = (int)eps.size();
  auto csr = [&](const int32_t* key, const int32_t* other, std::vector<int32_t>& ptr, std::vector<int32_t>& nb,
                 std::vector<int32_t>& arc) {
    ptr.assign(S + 1, 0);
    for (int g : eps) ptr[key[g] + 1]++;
    for (int v = 0; v < S; v++) ptr[v + 1] += ptr[v];
    arc = eps;
    std::stable_sort(arc.begin(), arc.end(), [&](int x, int y) { return key[x] < key[y]; });
    nb.resize(arc.size());
    for (size_t k = 0; k < arc.size(); k++) nb[k] = other[arc[k]];
  };
  csr(G.arc_dst, G.arc_src, t->eps_in_ptr, t->eps_in_src, t->eps_in_arc);
  csr(G.arc_src, G.arc_dst, t->eps_out_ptr, t->eps_out_dst, t->eps_out_arc);
  t->max_in_all = 0;
  for (int v = 0; v < S; v++)
    t->max_in_all = std::max(t->max_in_all, t->in_ptr[v + 1] - t->in_ptr[v] + t->eps_in_ptr[v + 1] - t->eps_in_ptr[v]);
  // Kahn over the epsilon subgraph: order holds the nodes in a topological order, lf their forward levels
  std::vector<int32_t> indeg(S), lf(S, 0), order;
  for (int v = 0; v < S; v++) {
    indeg[v] = t->eps_in_ptr[v + 1] - t->eps_in_ptr[v];
    if (!indeg[v]) order.push_back(v);
  }
  for (size_t i = 0; i < order.size(); i++) {
    const int u = order[i];
    for (int k = t->eps_out_ptr[u]; k < t->eps_out_ptr[u + 1]; k++) {
      const int v = t->eps_out_dst[k];
      lf[v] = std::max(lf[v], lf[u] + 1);
      if (--indeg[v] == 0) order.push_back(v);
    }
  }
  t->cycle.clear();
  if ((int)order.size() < S) {
    // every node left has an epsilon in-arc from another node left: walk them back until a node repeats
    int v = 0;
    while (!indeg[v]) v++;
    std::vector<int32_t> seen(S, -1), walk;
    while (seen[v] < 0) {
      seen[v] = (int32_t)walk.size();
      walk.push_back(v);
      for (int k = t->eps_in_ptr[v]; k < t->eps_in_ptr[v + 1]; k++)
        if (indeg[t->eps_in_src[k]]) {
          v = t->eps_in_src[k];
          break;
        }
    }
    t->cycle.assign(walk.begin() + seen[v], walk.end());
    std::reverse(t->cycle.begin(), t->cycle.end());
    t->L = 0;
    return;
  }
  std::vector<int32_t> lb(S, 0);
  for (int i = S - 1; i >= 0; i--) {
    const int u = order[i];
    for (int k = t->eps_out_ptr[u]; k < t->eps_out_ptr[u + 1]; k++) lb[u] = std::max(lb[u], lb[t->eps_out_dst[k]] + 1);
  }
  t->L = S ? std::max(*std::max_element(lf.begin(), lf.end()), 0) : 0;
  auto levels = [&](const std::vector<int32_t>& lev, const std::vector<int32_t>& ptr_of, std::vector<int32_t>& ptr,
                    std::vector<int32_t>& node) {
    ptr.assign(t->L + 1, 0);
    for (int v = 0; v < S; v++)
      if (lev[v]) ptr[lev[v]]++;
    for (int l = 0; l < t->L; l++) ptr[l + 1] += ptr[l];
    node.assign(ptr[t->L], 0);
    std::vector<int32_t> fill(ptr.begin(), ptr.end() - 1);
    for (int v = 0; v < S; v++)
      if (lev[v]) node[fill[lev[v] - 1]++] = v;
    for (int l = 0; l < t->L; l++) { // about four arcs per thread at the level's mean degree
      long long arcs = 0;
      for (int i = ptr[l]; i < ptr[l + 1]; i++) arcs += ptr_of[node[i] + 1] - ptr_of[node[i]];
      t->lanes.push_back(sparse_den_lanes(ptr[l + 1] - ptr[l], (int)arcs));
    }
  };
  t->lanes.clear();
  levels(lf, t->eps_in_ptr, t->fwd_ptr, t->fwd_node);
  levels(lb, t->eps_out_ptr, t->bwd_ptr, t->bwd_node);
}

/*
 * Each rank's share of each epsilon level under the cluster plan sp (sparse_cluster_plan) of G = t: the nodes of a
 * level that the rank owns in the emitting update, sp.in forward and sp.out backward, so that a node keeps one owner
 * through the frame.  A level lists its nodes in ascending id, so the share is one contiguous run of it:
 * cut[(d * L + l) * (N + 1) + r] .. [... + r + 1] into fwd_node (d = 0) or bwd_node (d = 1), found with lower_bound.
 */
inline void sparse_eps_cluster_cuts(const SparseTables& t, const SparseSplit& sp, std::vector<int32_t>* cut) {
  const int N = sp.N;
  cut->assign((size_t)2 * t.L * (N + 1), 0);
  for (int d = 0; d < 2; d++) {
    const std::vector<int32_t>& ptr = d ? t.bwd_ptr : t.fwd_ptr;
    const std::vector<int32_t>& node = d ? t.bwd_node : t.fwd_node;
    const int32_t* split = d ? sp.out : sp.in;
    for (int l = 0; l < t.L; l++)
      for (int r = 0; r <= N; r++)
        (*cut)[(size_t)(d * t.L + l) * (N + 1) + r] =
            (int32_t)(std::lower_bound(node.begin() + ptr[l], node.begin() + ptr[l + 1], split[r]) - node.begin());
  }
}

/*
 * The numerator of gtnb_sparse_transitions_loss, intersect(A, G), from structure only: the (A node, G node) pairs
 * reachable from the start pairs, trimmed to those that reach an accept pair (A and G both accept).  An A arc u -> v
 * and a G arc p -> q with the same label in [0, C) give the arc (u, p) -> (v, q); arc_of is the A arc, tidx the G arc.
 * Unfolded (the exact route): every (A start, G start) pair is a start state.  Folded (the device route): those start
 * copies collapse into one start node S (node 0), with one arc S -> (v, q) per out-arc a: u -> v of an A start node u
 * and per start group k of G with a's label and destination q; its tidx is nG + k (nG = G's arc count), so Wx =
 * [trans_w | sigma] and its weight is w_a + sigma_k.  The pairs with both nodes start are then ordinary states,
 * reached through in-arcs only.  An empty product keeps one node that neither starts nor accepts.
 * When t has epsilon tables (sparse_eps_tables; the backoff entry points, unfolded only), G's epsilon arc p -> q
 * gives (u, p) -> (u, q) for every A node u, labelled GTNB_EPSILON, with arc_of -1 and tidx the G arc.
 */
inline void build_sparse_product(const gtnb_graph_view& A, const gtnb_graph_view& G, const SparseTables& t, int C,
                                 bool fold, ProductGraph* p) {
  const int N = A.num_nodes, nA = A.num_arcs, nG = G.num_arcs;
  const long long S = t.S;
  std::vector<int32_t> a_ptr(N + 1, 0), a_out;
  for (int a = 0; a < nA; a++)
    if (A.arc_olabel[a] >= 0 && A.arc_olabel[a] < C) a_ptr[A.arc_src[a] + 1]++;
  for (int u = 0; u < N; u++) a_ptr[u + 1] += a_ptr[u];
  a_out.resize(a_ptr[N]);
  {
    std::vector<int32_t> fill(a_ptr.begin(), a_ptr.end() - 1);
    for (int a = 0; a < nA; a++)
      if (A.arc_olabel[a] >= 0 && A.arc_olabel[a] < C) a_out[fill[A.arc_src[a]]++] = a;
  }
  std::unordered_map<long long, int32_t> id;
  std::vector<long long> state; // u * S + p of every state; the folded S is -1
  std::vector<int32_t> src, dst, lab, arc_of, tidx;
  auto node = [&](int u, int q) {
    const long long key = (long long)u * S + q;
    auto it = id.find(key);
    if (it != id.end()) return it->second;
    const int32_t n = (int32_t)state.size();
    id.emplace(key, n);
    state.push_back(key);
    return n;
  };
  auto put = [&](int s, int d, int l, int a, int g) {
    src.push_back(s);
    dst.push_back(d);
    lab.push_back(l);
    arc_of.push_back(a);
    tidx.push_back(g);
  };
  const bool a_start_acc = [&] {
    for (int u = 0; u < N; u++)
      if ((A.node_flags[u] & 3) == 3) return true;
    return false;
  }();
  bool g_start_acc = false;
  for (int q = 0; q < t.S; q++) g_start_acc |= (t.flags[q] & 3) == 3;
  if (fold) {
    state.push_back(-1); // S
    std::vector<std::vector<int32_t>> by_label(C);
    for (size_t k = 0; k + 1 < t.grp_ptr.size(); k++) by_label[t.grp_lab[k]].push_back((int32_t)k);
    for (int u = 0; u < N; u++) {
      if (!(A.node_flags[u] & 1)) continue;
      for (int e = a_ptr[u]; e < a_ptr[u + 1]; e++) {
        const int a = a_out[e], l = A.arc_olabel[a];
        for (int32_t k : by_label[l]) put(0, node(A.arc_dst[a], t.grp_dst[k]), l, a, nG + k);
      }
    }
  } else {
    for (int u = 0; u < N; u++)
      if (A.node_flags[u] & 1)
        for (int q = 0; q < t.S; q++)
          if (t.flags[q] & 1) node(u, q);
  }
  // breadth-first over the states found so far; every new state is appended, so one pass reaches them all
  for (size_t n = fold ? 1 : 0; n < state.size(); n++) {
    const int u = (int)(state[n] / S), q = (int)(state[n] % S);
    const int32_t* ol = t.out_lab.data();
    for (int e = a_ptr[u]; e < a_ptr[u + 1]; e++) {
      const int a = a_out[e], l = A.arc_olabel[a];
      const int32_t* lo = std::lower_bound(ol + t.out_ptr[q], ol + t.out_ptr[q + 1], l);
      for (const int32_t* it = lo; it != ol + t.out_ptr[q + 1] && *it == l; it++) {
        const int k = (int)(it - ol);
        put((int)n, node(A.arc_dst[a], t.out_dst[k]), l, a, t.out_arc[k]);
      }
    }
    // G's epsilon arcs (sparse_eps_tables): A stays, G moves, (u, q) -> (u, q'); no A arc, so arc_of is -1
    if (!t.eps_out_ptr.empty())
      for (int k = t.eps_out_ptr[q]; k < t.eps_out_ptr[q + 1]; k++)
        put((int)n, node(u, t.eps_out_dst[k]), GTNB_EPSILON, -1, t.eps_out_arc[k]);
  }
  const int M = (int)state.size();
  auto accepts = [&](int n) {
    if (state[n] < 0) return a_start_acc && g_start_acc;
    return (A.node_flags[state[n] / S] & 2) && (t.flags[state[n] % S] & 2);
  };
  auto starts = [&](int n) {
    if (fold) return n == 0;
    return (A.node_flags[state[n] / S] & 1) && (t.flags[state[n] % S] & 1);
  };
  // trim: keep the states from which an accept state is reachable
  std::vector<int32_t> in_ptr(M + 1, 0), in_src(src.size());
  for (int32_t d : dst) in_ptr[d + 1]++;
  for (int n = 0; n < M; n++) in_ptr[n + 1] += in_ptr[n];
  {
    std::vector<int32_t> fill(in_ptr.begin(), in_ptr.end() - 1);
    for (size_t k = 0; k < src.size(); k++) in_src[fill[dst[k]]++] = src[k];
  }
  std::vector<char> live(M, 0);
  std::vector<int32_t> stack;
  for (int n = 0; n < M; n++)
    if (accepts(n)) {
      live[n] = 1;
      stack.push_back(n);
    }
  while (!stack.empty()) {
    const int n = stack.back();
    stack.pop_back();
    for (int k = in_ptr[n]; k < in_ptr[n + 1]; k++)
      if (!live[in_src[k]]) {
        live[in_src[k]] = 1;
        stack.push_back(in_src[k]);
      }
  }
  std::vector<int32_t> renum(M, -1);
  int kept = 0;
  for (int n = 0; n < M; n++)
    if (live[n]) renum[n] = kept++;
  p->flags.assign(std::max(kept, 1), 0);
  for (int n = 0; n < M; n++)
    if (live[n]) p->flags[renum[n]] = (uint8_t)((starts(n) ? 1 : 0) | (accepts(n) ? 2 : 0));
  p->src.clear();
  p->dst.clear();
  p->label.clear();
  p->arc_of.clear();
  p->tidx.clear();
  for (size_t k = 0; k < src.size(); k++) {
    if (!live[src[k]] || !live[dst[k]]) continue;
    p->src.push_back(renum[src[k]]);
    p->dst.push_back(renum[dst[k]]);
    p->label.push_back(lab[k]);
    p->arc_of.push_back(arc_of[k]);
    p->tidx.push_back(tidx[k]);
  }
  const size_t P = p->flags.size();
  std::vector<int32_t> indeg(P, 0), outdeg(P, 0), in_label(P, -1);
  p->uniform = true;
  for (size_t k = 0; k < p->src.size(); k++) {
    indeg[p->dst[k]]++;
    outdeg[p->src[k]]++;
    if (p->label[k] == GTNB_EPSILON) continue;
    int32_t& il = in_label[p->dst[k]];
    if (il >= 0 && il != p->label[k]) p->uniform = false;
    il = p->label[k];
  }
  p->max_in = *std::max_element(indeg.begin(), indeg.end());
  p->max_out = *std::max_element(outdeg.begin(), outdeg.end());
  p->n_acc = (int)std::count_if(p->flags.begin(), p->flags.end(), [](uint8_t f) { return (f & 2) != 0; });
}

/* the product's arc weights: w[k] = w_A[arc_of[k]] + Wx[tidx[k]] (w_A NULL: every A weight 0); Wx[tidx[k]] alone
 * for an epsilon arc of G (arc_of -1), compose's weight for an arc of one side (compose.cpp:201-205) */
inline void product_weights(const ProductGraph& p, const float* w_A, const float* Wx, std::vector<float>* w) {
  w->resize(p.src.size());
  for (size_t k = 0; k < p.src.size(); k++)
    (*w)[k] = p.arc_of[k] < 0 ? Wx[p.tidx[k]] : (w_A ? w_A[p.arc_of[k]] : 0.0f) + Wx[p.tidx[k]];
}

} // namespace gtnb
