"""Regenerate tests/golden/graph_viterbi_golden.npz from the REAL reference (oracle/_ref/libgtn_ref.so): what
gtnb_graph_viterbi computes, viterbiPath and viterbiScore of compose(A_b, E_b), every utterance run alone on its first
T_b rows, A_b matched on its olabels (tests/graph_viterbi_oracle.py).

Graph batches:
  `a` (T=10 C=7, uniform emissions): a CTC graph, a CTC graph with a wildcard state at each end, a random cyclic graph
      with several start and accept nodes and labels >= C, an infeasible chain, an empty graph; T_b in
      {10, 8, 10, 1, 10}.
  `b` (T=8 C=12, uniform emissions): a word-piece decomposition graph built with the reference's own union / closure /
      compose / remove, the same with wildcards, a CTC graph with T_b = 0, a random cyclic graph; T_b in {8, 8, 0, 5}.
  `c` (T=9 C=4, integer emissions and weights, tie-heavy): a CTC graph, a wildcard graph, two parallel equal arcs into
      a node with two parallel equal self-loops, a random cyclic graph; T_b in {9, 9, 9, 7}.

Keys, per batch: `*_e` emissions [B, T, C]; `*_lens` (T_b); `*_n_nodes`, `*_n_arcs` per graph and the concatenated
`*_flags`, `*_src`, `*_dst`, `*_ilabel`, `*_olabel`, `*_w`; the reference's `*_paths` (matched labels) and `*_arcs`
(A_b's arc ids) [B, T], -1 beyond T_b and without an accepting path, and `*_scores` [B] (-inf without one).

Run where the reference sources are (it needs oracle/_ref, compiled by `make -C oracle ref`):
    python tests/golden/make_graph_viterbi_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import graph_oracle as go  # noqa: E402
from tests import graph_viterbi_oracle as gv  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
KEYS = ("flags", "src", "dst", "ilabel", "olabel", "w")


def cases():
    """(name, T, C, graphs, input_lens, tie-heavy), seeded"""
    rng = np.random.default_rng(2026)
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
    return [("a", 10, 7, a, [10, 8, 10, 1, 10], False), ("b", 8, 12, b, [8, 8, 0, 5], False),
            ("c", 9, 4, c, [9, 9, 9, 7], True)]


def main():
    out = {}
    for name, T, C, graphs, lens, ties in cases():
        rng = np.random.default_rng(sum(map(ord, name)) + 43)
        e = (rng.integers(0, 2, (len(graphs), T, C)) if ties else rng.uniform(-3, 3, (len(graphs), T, C)))
        e = e.astype(np.float32)
        out.update({name + "_e": e, name + "_lens": np.asarray(lens, np.int32),
                    name + "_n_nodes": np.asarray([len(g["flags"]) for g in graphs], np.int32),
                    name + "_n_arcs": np.asarray([len(g["src"]) for g in graphs], np.int32)})
        for k in KEYS:
            out[name + "_" + k] = np.concatenate([np.asarray(g[k]) for g in graphs]).astype(
                np.uint8 if k == "flags" else np.float32 if k == "w" else np.int32)
        paths, scores, arcs = gv.ref_graph_viterbi(e, graphs, lens)
        out.update({name + "_paths": paths, name + "_scores": scores, name + "_arcs": arcs})
    np.savez_compressed(os.path.join(HERE, "graph_viterbi_golden.npz"), **out)


if __name__ == "__main__":
    main()
