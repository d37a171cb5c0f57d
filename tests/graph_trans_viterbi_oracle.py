"""Test infrastructure for gtnb_graph_transitions_viterbi: viterbiPath / viterbiScore of the numerators of
gtnb_graph_transitions_loss,

    ASG:    compose(compose(A_b, G), E_b)
    BIGRAM: intersect(intersect(A_b, G), E_b)

with E_b = linearGraph(T_b, C) on the first T_b rows of utterance b, each utterance run alone.

- ``ref_graph_trans_viterbi``: the live reference (oracle/_ref), with G from ``graph_trans_oracle.dense_graph``.  A_b is
  matched on its olabels, so its ilabels play no part in either composition; they are replaced by the arc ids, which
  both compositions copy onto their arcs and viterbiPath onto the path's: the path's ilabels are then A_b's arcs and
  its olabels the matched labels.
- ``tropical_product``: the device route's graph in plain numpy, the product of A_b and G with BIGRAM's start states
  folded through tau_l = max_j W[l][j] and every arc's weight fl(w_a + W[.]), the A arc of every product arc beside it.
  ``device_route_outcome`` runs graph_viterbi_oracle's float32 tropical recursion over it: the score the device
  route returns, and whether its traceback meets a tie.
"""
import numpy as np

from oracle import pyoracle as po
from tests import graph_oracle as go
from tests import graph_trans_oracle as gto
from tests import graph_viterbi_oracle as gv

ASG, BIGRAM = gto.ASG, gto.BIGRAM


def ref_graph_trans_viterbi(emissions, graphs, kind, trans_w, input_lens=None, weights=None):
    """-> (paths [B, T] int32, scores [B] float32, arcs [B, T] int32), -1 beyond T_b and without an accepting path"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    op = "compose" if kind == ASG else "intersect"
    gd, _ = gto.dense_graph(kind, C, trans_w)
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
        if Tb == 0 or len(g["flags"]) == 0:  # linearGraph(0, C) accepts nothing; nor does an empty graph
            continue
        g["ilabel"] = np.arange(A, dtype=np.int32)
        num = po.ref_op(op, go.ref_graph(g), go.ref_graph(gd))
        lat = po.ref_op(op, num, po.RefGraph.linear(Tb, C, e[b, :Tb].ravel()))
        scores[b] = po.ref_op("viterbi_score", lat).item()
        p = po.ref_op("viterbi_path", lat).arrays()
        n = len(p["src"])
        assert n in (0, Tb) and np.array_equal(p["src"], np.arange(n)), (n, Tb)
        arcs[b, :n] = p["ilabel"]
        paths[b, :n] = p["olabel"]
    return paths, scores, arcs


def tropical_product(g, C, kind, trans_w):
    """(product graph dict with flags / src / dst / olabel / w, A arc of every product arc).  A state is (A node v,
    previous label l); ASG adds one start copy per start node (start weights s[l]); BIGRAM folds its C start states
    into one start node S whose arcs S -> (v, l) weigh w_a + tau_l."""
    tw = np.asarray(trans_w, np.float32).ravel()
    flags_a = np.asarray(g["flags"])
    src_a, dst_a, lab_a = (np.asarray(g[k]) for k in ("src", "dst", "olabel"))
    w_a = np.asarray(g["w"], np.float32) if "w" in g else np.zeros(len(src_a), np.float32)
    N = len(flags_a)
    ok = (lab_a >= 0) & (lab_a < C)
    in_labels = [sorted(set(lab_a[ok & (dst_a == v)].tolist())) for v in range(N)]
    node, flags = {}, []

    def add(key, f):
        node[key] = len(flags)
        flags.append(f)

    if kind == BIGRAM:
        add("S", 1)
    for v in range(N):
        acc = 2 if flags_a[v] & 2 else 0
        if kind == ASG and flags_a[v] & 1:
            add((v, "s"), 1)
        for l in in_labels[v]:
            add((v, l), acc)
    W = tw.reshape(C, C) if kind == BIGRAM else tw[C:].reshape(C, C)
    tau = W.max(axis=1) if kind == BIGRAM else None
    src, dst, lab, w, arc_of = [], [], [], [], []
    for a in np.flatnonzero(ok):
        u, v, l = int(src_a[a]), int(dst_a[a]), int(lab_a[a])
        froms = []
        if flags_a[u] & 1:
            froms.append(("S", tau[l]) if kind == BIGRAM else ((u, "s"), tw[l]))
        froms += [((u, j), W[l, j]) for j in in_labels[u]]
        for key, wx in froms:
            src.append(node[key]), dst.append(node[(v, l)]), lab.append(l), arc_of.append(a)
            w.append(np.float32(w_a[a] + np.float32(wx)))
    i32 = lambda x: np.asarray(x, np.int32)
    p = {"flags": np.asarray(flags, np.uint8), "src": i32(src), "dst": i32(dst), "olabel": i32(lab),
         "w": np.asarray(w, np.float32)}
    return p, i32(arc_of)


def path_value(e, g, kind, trans_w, labels, arcs):
    """the value of a path (A_b's arcs and their labels, one per frame of e [T_b, C]) in the device route's
    association: frame 0 reads s[l] (ASG) or tau_l (BIGRAM), frame t > 0 W[l][label of frame t - 1]"""
    tw = np.asarray(trans_w, np.float32).ravel()
    C = e.shape[1]
    W = tw.reshape(C, C) if kind == BIGRAM else tw[C:].reshape(C, C)
    w_a = np.asarray(g["w"], np.float32)
    s = np.float32(0.0)
    for t, (l, a) in enumerate(zip(labels, arcs)):
        wx = (W[l].max() if kind == BIGRAM else tw[l]) if t == 0 else W[l, labels[t - 1]]
        s = np.float32(s + np.float32(np.float32(w_a[a] + wx) + e[t, l]))
    return s


def device_route_outcome(e, p, C):
    """(score, tie) of the device route on a product p from tropical_product over e [T_b, C]: the best accept node's
    score of the float32 recursion, and whether the traceback meets a tie -- two accept nodes at that score, or a node
    of the path reached at its score by two in-arcs (graph_viterbi_oracle.trace_ties's rule, walked without the
    device's path: before the first tie the path is unique)"""
    T = e.shape[0]
    S = gv.tropical_scores(e, p, C)
    acc = np.flatnonzero((p["flags"] & 2) != 0)
    if T == 0 or len(acc) == 0 or not np.isfinite(S[T, acc]).any():
        return np.float32(-np.inf), False
    best = S[T, acc].max()
    if np.count_nonzero(S[T, acc] == best) > 1:
        return best, True
    v = int(acc[np.argmax(S[T, acc])])
    for t in range(T, 0, -1):
        ins = np.flatnonzero(p["dst"] == v)
        cand = S[t - 1, p["src"][ins]] + (p["w"][ins] + e[t - 1, p["olabel"][ins]])
        hit = np.flatnonzero(cand == S[t, v])
        if len(hit) != 1:
            return best, True
        v = int(p["src"][ins[hit[0]]])
    return best, False
