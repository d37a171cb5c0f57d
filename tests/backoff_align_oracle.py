"""Test infrastructure for gtnb_backoff_transitions_viterbi (a transition graph G with epsilon arcs, backoff_oracle's):

    align: viterbiPath / viterbiScore of intersect(intersect(A_b, G), E_b), the numerator of
           gtnb_backoff_transitions_loss

with E_b = linearGraph(T_b, C) on the first T_b rows of utterance b, each utterance run alone.

- ``ref_backoff_trans_viterbi``: the live reference (oracle/_ref), sparse_viterbi_oracle.ref_sparse_trans_viterbi
  with the path's epsilon arcs dropped: A_b's ilabels are replaced by its arc ids, so the path's arcs with an epsilon
  ilabel are G's epsilon arcs, which use no frame; T_b arcs remain.
- ``ref_backoff_trans_forward``: forwardScore of the same numerator (a max over paths is at most their logsumexp).
- ``product``: P_b = A_b o G restated in numpy (unfolded: node (u, p) for every pair, an emitting arc for every A arc
  and G arc of the same label in [0, C), an epsilon arc (u, p) -> (u, q) for every A node u and G epsilon arc
  p -> q), with the A arc (arc_of, -1 on epsilon arcs) and the G arc (tidx) behind each arc.
- ``restate_align``: a float32 restatement of the alignment's device route, the decode's per-CTA sweep over P_b
  (backoff_oracle.restate_decode) with the weights fl(w_A + w_G) and w_G on epsilon arcs: the score, the tie flag and,
  without a tie, the labels and A_b's arcs.
- ``golden_batches``: the committed fixture tests/golden/backoff_align_golden.npz
  (tests/golden/make_backoff_align_golden.py).
"""
import os

import numpy as np

from oracle import pyoracle as po
from tests import backoff_oracle as bo
from tests import graph_oracle as go

EPS = bo.EPS


def _numerator(g, G, trans_w, weights):
    """the reference's intersect(A'_b, G) for target graph g (A'_b: ilabels replaced by the arc ids)"""
    gd = dict(G)
    gd["w"] = np.asarray(trans_w, np.float32).ravel()
    a = dict(g)
    if weights is not None:
        a["w"] = np.asarray(weights, np.float32)
    a["ilabel"] = np.arange(len(a["src"]), dtype=np.int32)
    return po.ref_op("intersect", go.ref_graph(a), go.ref_graph(gd))


def _split(graphs, weights):
    """per utterance: its slice of the batch's arc weights (None: the graphs' own)"""
    off = np.cumsum([0] + [len(g["src"]) for g in graphs])
    return [None if weights is None else np.asarray(weights, np.float32)[off[b]:off[b + 1]]
            for b in range(len(graphs))]


def ref_backoff_trans_viterbi(emissions, graphs, G, trans_w, input_lens=None, weights=None, eps_used=None):
    """-> (paths [B, T] int32, scores [B] float32, arcs [B, T] int32: A_b's arcs), -1 beyond T_b and without an
    accepting path; eps_used (a list, optional) gets the number of epsilon arcs on every utterance's path"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    paths = np.full((B, T), -1, np.int32)
    arcs = np.full((B, T), -1, np.int32)
    scores = np.full(B, -np.inf, np.float32)
    for b, wb in enumerate(_split(graphs, weights)):
        Tb = T if input_lens is None else int(input_lens[b])
        if Tb == 0 or len(graphs[b]["flags"]) == 0:
            if eps_used is not None:
                eps_used.append(0)
            continue
        num = _numerator(graphs[b], G, trans_w, wb)
        lat = po.ref_op("intersect", num, po.RefGraph.linear(Tb, C, e[b, :Tb].ravel()))
        scores[b] = po.ref_op("viterbi_score", lat).item()
        p = po.ref_op("viterbi_path", lat).arrays()
        emit = p["ilabel"] != EPS
        n = int(emit.sum())
        assert n in (0, Tb), (n, Tb)
        if eps_used is not None:
            eps_used.append(len(emit) - n)
        arcs[b, :n] = p["ilabel"][emit]
        paths[b, :n] = p["olabel"][emit]
    return paths, scores, arcs


def ref_backoff_trans_forward(emissions, graphs, G, trans_w, input_lens=None, weights=None):
    """-> forwardScore [B] float32 of every numerator (-inf for T_b = 0 and an empty graph)"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    out = np.full(B, -np.inf, np.float32)
    for b, wb in enumerate(_split(graphs, weights)):
        Tb = T if input_lens is None else int(input_lens[b])
        if Tb == 0 or len(graphs[b]["flags"]) == 0:
            continue
        lat = po.ref_op("intersect", _numerator(graphs[b], G, trans_w, wb),
                        po.RefGraph.linear(Tb, C, e[b, :Tb].ravel()))
        out[b] = po.ref_op("forward_score", lat).item()
    return out


def product(g, G, C):
    """-> (P in graph_oracle's layout, epsilon arcs labelled -1; arc_of; tidx)"""
    NA, NG = len(g["flags"]), len(G["flags"])
    node = lambda u, p: u * NG + p
    fa, fg = np.asarray(g["flags"]), np.asarray(G["flags"])
    flags = np.zeros(NA * NG, np.uint8)
    for u in range(NA):
        for p in range(NG):
            flags[node(u, p)] = (fa[u] & fg[p] & 1) | (fa[u] & fg[p] & 2)
    src, dst, lab, arc_of, tidx = [], [], [], [], []
    for a in range(len(g["src"])):
        la = int(g["olabel"][a])
        if not 0 <= la < C:
            continue
        for k in np.flatnonzero(np.asarray(G["olabel"]) == la):
            src.append(node(g["src"][a], G["src"][k])), dst.append(node(g["dst"][a], G["dst"][k]))
            lab.append(la), arc_of.append(a), tidx.append(k)
    for k in np.flatnonzero(np.asarray(G["olabel"]) == EPS):
        for u in range(NA):
            src.append(node(u, G["src"][k])), dst.append(node(u, G["dst"][k]))
            lab.append(EPS), arc_of.append(-1), tidx.append(k)
    P = go.make(flags, np.asarray(src, np.int64), np.asarray(dst, np.int64), np.asarray(lab, np.int64))
    return P, np.asarray(arc_of, np.int32), np.asarray(tidx, np.int32)


def restate_align(e, g, G, trans_w, C, w_A=None):
    """(score, tie, labels, A_b's arcs) of the alignment's device route over e [T_b, C] for target graph g (w_A: its
    arc weights, None: g["w"] or 0)"""
    P, arc_of, tidx = product(g, G, C)
    if w_A is None:
        w_A = g.get("w", np.zeros(len(g["src"]), np.float32))
    w_A = np.asarray(w_A, np.float32)
    tw = np.asarray(trans_w, np.float32)
    wP = np.where(arc_of < 0, tw[tidx], w_A[np.maximum(arc_of, 0)] + tw[tidx]).astype(np.float32)
    score, tie, labels, parcs = bo.restate_decode(e, P, wP, C)
    return score, tie, labels, None if parcs is None else arc_of[parcs]


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "backoff_align_golden.npz")
NAMES = ("bigram", "trigram", "random")


def golden_batches():
    """-> [(name, emissions, lens, G, trans_w, graphs, (paths, scores, arcs))]"""
    z = np.load(GOLDEN)
    out = []
    for name in NAMES:
        lens = z[name + "_lens"]
        G = go.make(z[name + "_G_flags"], z[name + "_G_src"], z[name + "_G_dst"], z[name + "_G_label"])
        graphs = []
        for b in range(len(lens)):
            g = go.make(z["%s_A%d_flags" % (name, b)], z["%s_A%d_src" % (name, b)], z["%s_A%d_dst" % (name, b)],
                        z["%s_A%d_label" % (name, b)])
            g["w"] = z["%s_A%d_w" % (name, b)]
            graphs.append(g)
        res = tuple(z["%s_%s" % (name, k)] for k in ("paths", "scores", "arcs"))
        out.append((name, z[name + "_e"], lens, G, z[name + "_trans_w"], graphs, res))
    return out
