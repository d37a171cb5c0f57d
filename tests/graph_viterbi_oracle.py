"""Test infrastructure for gtnb_graph_viterbi: viterbiPath / viterbiScore of compose(A_b, E_b) with E_b =
linearGraph(T_b, C) on the first T_b rows of utterance b, each utterance run alone.

- ``ref_graph_viterbi``: the live reference (oracle/_ref).  A_b is matched on its olabels, so its ilabels play no part
  in the composition; they are replaced by the arc ids, which compose copies onto the lattice's arcs and viterbiPath
  onto the path's: the path's ilabels are then A_b's arcs and its olabels the matched labels.
- ``tropical_scores``: a float32 restatement of the frame-synchronous tropical recursion, S_t[v] = max over in-arcs of
  fl(S_{t-1}[src] + fl(w + e[t-1][label])), and ``path_score``: a path's value in the same association.
"""
import numpy as np

from oracle import pyoracle as po
from tests import graph_oracle as go


def ref_graph_viterbi(emissions, graphs, input_lens=None, weights=None, olabel_sorted=False):
    """-> (paths [B, T] int32, scores [B] float32, arcs [B, T] int32), -1 beyond T_b and without an accepting path.
    olabel_sorted: arcSort the graphs on their olabels first (compose then takes the reference's sorted matcher)."""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
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
        rg = go.ref_graph(g)
        if olabel_sorted:
            rg.arc_sort(olabel=True)
        lat = po.ref_op("compose", rg, po.RefGraph.linear(Tb, C, e[b, :Tb].ravel()))
        scores[b] = po.ref_op("viterbi_score", lat).item()
        p = po.ref_op("viterbi_path", lat).arrays()
        n = len(p["src"])
        assert n in (0, Tb) and np.array_equal(p["src"], np.arange(n)), (n, Tb)
        arcs[b, :n] = p["ilabel"]
        paths[b, :n] = p["olabel"]
    return paths, scores, arcs


def tropical_scores(e, g, C):
    """[T + 1, N] float32 node scores of the frame-synchronous tropical recursion over e [T, C]"""
    T, N = e.shape[0], len(g["flags"])
    S = np.full((T + 1, N), -np.inf, np.float32)
    S[0, (g["flags"] & 1) != 0] = 0.0
    lab = g["olabel"]
    ok = (lab >= 0) & (lab < C)
    src, dst, w = g["src"][ok], g["dst"][ok], g["w"][ok].astype(np.float32)
    for t in range(1, T + 1):
        cand = S[t - 1, src] + (w + e[t - 1, lab[ok]])
        np.maximum.at(S[t], dst, cand)
    return S


def path_score(e, g, arcs):
    """the value of a path (arc ids of g, one per frame) in the recursion's association"""
    s = np.float32(0.0)
    for t, a in enumerate(arcs):
        s = np.float32(s + np.float32(np.float32(g["w"][a]) + e[t, g["olabel"][a]]))
    return s


def trace_ties(e, g, C, arcs):
    """whether a best path (arc ids of g, one per frame of e [T_b, C]) meets a tie: two accept nodes at the best score
    of frame T_b, or a node of the path reached at its score by two in-arcs -- the device route's tie rule"""
    T = e.shape[0]
    if T == 0 or len(arcs) == 0 or arcs[0] < 0:
        return False
    S = tropical_scores(e, g, C)
    acc = (g["flags"] & 2) != 0
    if np.count_nonzero(S[T, acc] == S[T, acc].max()) > 1:
        return True
    lab = g["olabel"]
    ok = (lab >= 0) & (lab < C)
    for t in range(1, T + 1):
        v = g["dst"][arcs[t - 1]]
        ins = np.flatnonzero(ok & (g["dst"] == v))
        cand = S[t - 1, g["src"][ins]] + (g["w"][ins].astype(np.float32) + e[t - 1, lab[ins]])
        if np.count_nonzero(cand == S[t, v]) > 1:
            return True
    return False
