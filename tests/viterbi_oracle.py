"""Test infrastructure for gtnb_viterbi_dense_ex's bigram kind: viterbiPath / viterbiScore of

    intersect(linearGraph(T, C; e), G)

with n-gram CTC's bigram graph G (benchmarks/ctc.cpp:107-134): C nodes, every node start and accept, for j, for i:
arc j -> i with label i and weight W[i*C + j], then arcSort().  Two independent evaluations, graph by graph:

- ``ref_viterbi_bigram``: the live reference (oracle/_ref) through its own Graph API.
- ``oracle_viterbi_bigram``: the C restatement (oracle/gtn_oracle.c), literally intersect / shortestPath /
  shortestDistance.

linearGraph(0, C) is one start node that does not accept (creations.cpp:20-33): T = 0 has no accepting path, score
-inf.  Paths are the ilabels of the best path, -1 where there is none.
"""
import numpy as np

from oracle import pyoracle as po
from tests.ngram_oracle import bigram_arrays


def ref_viterbi_bigram(emissions, W):
    """the live reference, one utterance: -> (path [T], score)"""
    e = np.ascontiguousarray(emissions, np.float32)
    T, C = e.shape
    gf, gs, gd, gl, gw = bigram_arrays(W)
    G = po.RefGraph.from_arrays(gf, gs, gd, gl, gl, gw, calc_grad=False)
    G.arc_sort()
    E = po.RefGraph.linear(T, C, e.ravel() if T else None, calc_grad=False)
    lattice = po.ref_op("intersect", E, G)
    path = po.ref_op("viterbi_path", lattice)
    score = po.ref_op("viterbi_score", lattice).item()
    labels = path.arrays()["ilabel"] if path.num_arcs else np.zeros(0, np.int32)
    out = np.full(T, -1, np.int32)
    out[:len(labels)] = labels
    return out, np.float32(score)


def oracle_viterbi_bigram(emissions, W):
    """the C restatement, one utterance: -> (path [T], score)"""
    e = np.ascontiguousarray(emissions, np.float32)
    T, C = e.shape
    gf, gs, gd, gl, gw = bigram_arrays(W)
    G = po.Graph.from_arrays(gf, gs, gd, gl, gl, gw)
    G.arc_sort()
    E = po.Graph.linear(T, C, e.ravel()) if T else po.Graph.from_arrays([1], [], [], [], [])
    lattice = po.intersect(E, G)
    out = np.full(T, -1, np.int32)
    arcs = po.shortest_path(lattice)
    if arcs is not None:
        out[:len(arcs)] = lattice.arrays()["ilabel"][arcs]
    score, _, _, _ = po.shortest_distance(lattice, tropical=True)
    return out, np.float32(score)


def batch(fn, emissions, W, input_lens=None):
    """fn on every utterance's first T_b rows -> (paths [B, T], -1 beyond; scores [B])"""
    e = np.asarray(emissions, np.float32)
    B, T, _ = e.shape
    paths = np.full((B, T), -1, np.int32)
    scores = np.zeros(B, np.float32)
    for b in range(B):
        Tb = T if input_lens is None else int(input_lens[b])
        paths[b, :Tb], scores[b] = fn(e[b, :Tb], W)
    return paths, scores
