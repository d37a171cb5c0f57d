"""Regenerate tests/golden/graph_trans_viterbi_golden.npz from the REAL reference (oracle/_ref/libgtn_ref.so): what
gtnb_graph_transitions_viterbi computes, viterbiPath and viterbiScore of compose(compose(A_b, G), E_b) (ASG) and
intersect(intersect(A_b, G), E_b) (BIGRAM), every utterance run alone on its first T_b rows, A_b matched on its olabels
(tests/graph_trans_viterbi_oracle.py).

Graph batches (the same graphs for both kinds):
  `a` (T=10 C=7, uniform emissions and transitions): a CTC graph, a CTC graph with a wildcard state at each end, a
      random cyclic graph with several start and accept nodes, start nodes with in-arcs and labels >= C, an infeasible
      chain, an empty graph; T_b in {10, 8, 10, 1, 10}.
  `b` (T=8 C=12, uniform emissions, transitions with every 7th entry -inf): a word-piece decomposition graph built with
      the reference's own union / closure / compose / remove, the same with wildcards, a CTC graph with T_b = 0, a
      random cyclic graph; T_b in {8, 8, 0, 5}.
  `c` (T=9 C=4, integer emissions, weights and transitions, tie-heavy): a CTC graph, a wildcard graph, two parallel
      equal arcs into a node with two parallel equal self-loops, a random cyclic graph; T_b in {9, 9, 9, 7}.

Keys, per batch: `*_e` emissions [B, T, C]; `*_lens` (T_b); `*_n_nodes`, `*_n_arcs` per graph and the concatenated
`*_flags`, `*_src`, `*_dst`, `*_ilabel`, `*_olabel`, `*_w`.  Per batch and kind (`asg`, `bigram`): `*_<kind>_trans_w`
and the reference's `*_<kind>_paths` (labels) and `*_<kind>_arcs` (A_b's arc ids) [B, T], -1 beyond T_b and without an
accepting path, and `*_<kind>_scores` [B] (-inf without one).

Run where the reference sources are (it needs oracle/_ref, compiled by `make -C oracle ref`):
    python tests/golden/make_graph_trans_viterbi_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import graph_oracle as go  # noqa: E402
from tests import graph_trans_viterbi_oracle as gtv  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
KEYS = ("flags", "src", "dst", "ilabel", "olabel", "w")
KINDS = {"asg": gtv.ASG, "bigram": gtv.BIGRAM}


def cases():
    """(name, T, C, graphs, input_lens, tie-heavy, -inf transitions), seeded"""
    rng = np.random.default_rng(2027)
    a = [go.ctc_graph([1, 3, 3, 2]), go.with_wildcards(go.ctc_graph([4, 5]), 7, w_loop=-0.4),
         go.random_graph(rng, 9, 30, 7, n_start=3, n_accept=3, label_hi=9),
         go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3]), go.make([], [], [], [])]
    pieces = [(i,) for i in range(5)] + [(0, 1), (1, 2), (3, 4), (2, 3, 4), (4, 4)]
    dec = go.from_ref(go.decomposition_graph(go.REF_OPS, [0, 1, 2, 3, 4, 4], pieces))
    b = [dec, go.with_wildcards(dec, 12, w_loop=-0.2), go.ctc_graph([6, 7]),
         go.random_graph(rng, 7, 25, 12, n_start=2, n_accept=2, label_hi=14)]
    for g in a + b:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    c = [go.ctc_graph([1, 2, 2]), go.with_wildcards(go.ctc_graph([3]), 4, w_loop=0.0),
         go.make([1, 2], [0, 0, 1, 1], [1, 1, 1, 1], [1, 1, 2, 2]),
         go.random_graph(rng, 6, 24, 4, n_start=2, n_accept=2)]
    for g in c:
        g["w"] = rng.integers(-1, 1, len(g["src"])).astype(np.float32)
    c[2]["w"][:] = 0.0
    return [("a", 10, 7, a, [10, 8, 10, 1, 10], False, False), ("b", 8, 12, b, [8, 8, 0, 5], False, True),
            ("c", 9, 4, c, [9, 9, 9, 7], True, False)]


def main():
    out = {}
    for name, T, C, graphs, lens, ties, neginf in cases():
        rng = np.random.default_rng(sum(map(ord, name)) + 47)
        e = (rng.integers(0, 2, (len(graphs), T, C)) if ties else rng.uniform(-3, 3, (len(graphs), T, C)))
        e = e.astype(np.float32)
        out.update({name + "_e": e, name + "_lens": np.asarray(lens, np.int32),
                    name + "_n_nodes": np.asarray([len(g["flags"]) for g in graphs], np.int32),
                    name + "_n_arcs": np.asarray([len(g["src"]) for g in graphs], np.int32)})
        for k in KEYS:
            out[name + "_" + k] = np.concatenate([np.asarray(g[k]) for g in graphs]).astype(
                np.uint8 if k == "flags" else np.float32 if k == "w" else np.int32)
        for kind, k in KINDS.items():
            n = (C + C * C) if k == gtv.ASG else C * C
            tw = (rng.integers(-1, 1, n) if ties else rng.uniform(-1, 1, n)).astype(np.float32)
            if neginf:
                tw[::7] = -np.inf
            paths, scores, arcs = gtv.ref_graph_trans_viterbi(e, graphs, k, tw, lens)
            p = "%s_%s_" % (name, kind)
            out.update({p + "trans_w": tw, p + "paths": paths, p + "scores": scores, p + "arcs": arcs})
    np.savez_compressed(os.path.join(HERE, "graph_trans_viterbi_golden.npz"), **out)


if __name__ == "__main__":
    main()
