"""Test infrastructure for gtnb_viterbi_sparse and gtnb_sparse_transitions_viterbi (a learned transition graph G of
any shape, sparse_trans_oracle's):

    decode: viterbiPath / viterbiScore of intersect(E_b, G)
    align:  viterbiPath / viterbiScore of intersect(intersect(A_b, G), E_b)

with E_b = linearGraph(T_b, C) on the first T_b rows of utterance b, each utterance run alone.

- ``ref_sparse_viterbi``: the live reference (oracle/_ref) for the decode.  G is matched on its ilabels, so its
  olabels play no part in the intersection; they are replaced by the arc ids (G'), which intersect copies onto the
  lattice's arcs and viterbiPath onto the path's: the path's ilabels are then the labels and its olabels G's arcs.
- ``ref_sparse_trans_viterbi``: the live reference for the alignment, A_b's ilabels replaced by its arc ids as in
  graph_trans_viterbi_oracle.
- ``decode_outcome``: a float32 restatement of the decode's device route, S_t[v] = max over in-arcs of
  fl(S_{t-1}[u] + fl(w_a + e[t-1][label_a])) over G's arcs labelled in [0, C): the score, whether the traceback meets
  a tie (graph_trans_viterbi_oracle.device_route_outcome's rule) and the path it takes where there is none.
- ``golden_batches``: the committed fixture tests/golden/sparse_viterbi_golden.npz
  (tests/golden/make_sparse_viterbi_golden.py).
"""
import os

import numpy as np

from oracle import pyoracle as po
from tests import graph_oracle as go


def ref_sparse_viterbi(emissions, G, trans_w, input_lens=None):
    """-> (paths [B, T] int32, scores [B] float32, arcs [B, T] int32: G's arcs), -1 beyond T_b and without an
    accepting path"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    paths = np.full((B, T), -1, np.int32)
    arcs = np.full((B, T), -1, np.int32)
    scores = np.full(B, -np.inf, np.float32)
    g = dict(G)
    g["w"] = np.asarray(trans_w, np.float32).ravel()
    g["olabel"] = np.arange(len(g["src"]), dtype=np.int32)
    rg = go.ref_graph(g)
    for b in range(B):
        Tb = T if input_lens is None else int(input_lens[b])
        if Tb == 0:  # linearGraph(0, C) accepts nothing
            continue
        lat = po.ref_op("intersect", po.RefGraph.linear(Tb, C, e[b, :Tb].ravel()), rg)
        scores[b] = po.ref_op("viterbi_score", lat).item()
        p = po.ref_op("viterbi_path", lat).arrays()
        n = len(p["src"])
        assert n in (0, Tb) and np.array_equal(p["src"], np.arange(n)), (n, Tb)
        paths[b, :n] = p["ilabel"]
        arcs[b, :n] = p["olabel"]
    return paths, scores, arcs


def ref_sparse_trans_viterbi(emissions, graphs, G, trans_w, input_lens=None, weights=None):
    """-> (paths [B, T] int32, scores [B] float32, arcs [B, T] int32: A_b's arcs), -1 beyond T_b and without an
    accepting path"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    gd = dict(G)
    gd["w"] = np.asarray(trans_w, np.float32).ravel()
    rg = go.ref_graph(gd)
    paths = np.full((B, T), -1, np.int32)
    arcs = np.full((B, T), -1, np.int32)
    scores = np.full(B, -np.inf, np.float32)
    off = 0
    for b in range(B):
        g = dict(graphs[b])
        A = len(g["src"])
        if weights is not None:
            g["w"] = np.asarray(weights[off:off + A], np.float32)
        off += A
        Tb = T if input_lens is None else int(input_lens[b])
        if Tb == 0 or len(g["flags"]) == 0:
            continue
        g["ilabel"] = np.arange(A, dtype=np.int32)
        num = po.ref_op("intersect", go.ref_graph(g), rg)
        lat = po.ref_op("intersect", num, po.RefGraph.linear(Tb, C, e[b, :Tb].ravel()))
        scores[b] = po.ref_op("viterbi_score", lat).item()
        p = po.ref_op("viterbi_path", lat).arrays()
        n = len(p["src"])
        assert n in (0, Tb) and np.array_equal(p["src"], np.arange(n)), (n, Tb)
        arcs[b, :n] = p["ilabel"]
        paths[b, :n] = p["olabel"]
    return paths, scores, arcs


def kept(G, trans_w, C):
    """G with its weights, restricted to the arcs labelled in [0, C) (the others never match); and their arc ids"""
    lab = np.asarray(G["olabel"])
    ids = np.flatnonzero((lab >= 0) & (lab < C))
    w = np.asarray(trans_w, np.float32).ravel()
    g = {"flags": np.asarray(G["flags"], np.uint8), "src": np.asarray(G["src"])[ids],
         "dst": np.asarray(G["dst"])[ids], "olabel": lab[ids], "w": w[ids]}
    return g, ids


def _by_destination(g):
    """g's arcs sorted by destination (stable: arc id order within a node) -> (order, segment starts, their nodes)"""
    order = np.argsort(g["dst"], kind="stable")
    dst = g["dst"][order]
    starts = np.flatnonzero(np.r_[True, dst[1:] != dst[:-1]]) if len(dst) else np.zeros(0, np.int64)
    return order, starts, dst[starts]


def tropical_rows(e, g):
    """[T + 1, N] float32 rows S_t[v] = max over in-arcs of fl(S_{t-1}[u] + fl(w_a + e[t-1][label_a])) over e [T, C]
    (graph_viterbi_oracle.tropical_scores' recursion, by segment maxima: fast enough for whole benchmark batches)"""
    T, N = e.shape[0], len(g["flags"])
    order, starts, nodes = _by_destination(g)
    src, lab, w = g["src"][order], g["olabel"][order], np.asarray(g["w"], np.float32)[order]
    S = np.full((T + 1, N), -np.inf, np.float32)
    S[0, (g["flags"] & 1) != 0] = 0.0
    for t in range(1, T + 1):
        if len(src):
            S[t, nodes] = np.maximum.reduceat(S[t - 1, src] + (w + e[t - 1, lab]), starts)
    return S


def decode_outcome(e, G, trans_w, C):
    """(score, tie, labels, arcs) of the decode's device route over e [T_b, C]: the best accept node's score; whether
    the traceback meets a tie -- two accept nodes at that score, or a node of the path reached at its score by two
    in-arcs (graph_trans_viterbi_oracle.device_route_outcome's rule; before the first tie the path is unique); and,
    without a tie, the path (labels and G's arc ids per frame; None with a tie or without a path)"""
    g, ids = kept(G, trans_w, C)
    T = e.shape[0]
    S = tropical_rows(e, g)
    acc = np.flatnonzero((g["flags"] & 2) != 0)
    if T == 0 or len(acc) == 0 or not np.isfinite(S[T, acc]).any():
        return np.float32(-np.inf), False, None, None
    score = S[T, acc].max()
    if np.count_nonzero(S[T, acc] == score) > 1:
        return score, True, None, None
    order, starts, nodes = _by_destination(g)
    seg = dict(zip(nodes.tolist(), zip(starts.tolist(), np.r_[starts[1:], len(order)].tolist())))
    v = int(acc[np.argmax(S[T, acc])])
    labels, arcs = np.zeros(T, np.int32), np.zeros(T, np.int32)
    for t in range(T, 0, -1):
        i0, i1 = seg[v]
        ins = order[i0:i1]
        cand = S[t - 1, g["src"][ins]] + (g["w"][ins] + e[t - 1, g["olabel"][ins]])
        hit = np.flatnonzero(cand == S[t, v])
        if len(hit) != 1:
            return score, True, None, None
        k = ins[hit[0]]
        labels[t - 1], arcs[t - 1] = g["olabel"][k], ids[k]
        v = int(g["src"][k])
    return score, False, labels, arcs


def path_value(e, G, trans_w, arcs):
    """the value of a decode path (G's arc ids, one per frame of e [T_b, C]) in the device route's association"""
    w = np.asarray(trans_w, np.float32).ravel()
    s = np.float32(0.0)
    for t, a in enumerate(arcs):
        s = np.float32(s + np.float32(w[a] + e[t, G["olabel"][a]]))
    return s


def is_path(G, arcs):
    """whether G's arcs form a path from a start node to an accept node"""
    f, src, dst = np.asarray(G["flags"]), np.asarray(G["src"]), np.asarray(G["dst"])
    if len(arcs) == 0:
        return False
    ok = bool(f[src[arcs[0]]] & 1) and bool(f[dst[arcs[-1]]] & 2)
    return ok and all(dst[arcs[t]] == src[arcs[t + 1]] for t in range(len(arcs) - 1))


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sparse_viterbi_golden.npz")
NAMES = ("a", "b", "c")


def golden_batches():
    """-> [(name, emissions, lens, G, trans_w, graphs, decode (paths, scores, arcs), align (paths, scores, arcs))]"""
    z = np.load(GOLDEN)
    out = []
    for name in NAMES:
        graphs, n0, a0 = [], 0, 0
        for n, a in zip(z[name + "_n_nodes"], z[name + "_n_arcs"]):
            g = {"flags": z[name + "_flags"][n0:n0 + n]}
            for k in ("src", "dst", "ilabel", "olabel", "w"):
                g[k] = z[name + "_" + k][a0:a0 + a]
            graphs.append(g)
            n0, a0 = n0 + n, a0 + a
        G = go.make(z[name + "_G_flags"], z[name + "_G_src"], z[name + "_G_dst"], z[name + "_G_label"])
        res = [tuple(z["%s_%s_%s" % (name, op, k)] for k in ("paths", "scores", "arcs")) for op in ("dec", "ali")]
        out.append((name, z[name + "_e"], z[name + "_lens"], G, z[name + "_trans_w"], graphs, res[0], res[1]))
    return out
