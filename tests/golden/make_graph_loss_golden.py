"""Regenerate tests/golden/graph_loss_golden.npz from the REAL reference (oracle/_ref/libgtn_ref.so): the loss of
gtnb_graph_loss, forwardScore(E_b) - forwardScore(intersect(A_b, E_b)), every utterance run alone on its first T_b
rows, A_b matched on its olabels.

Cases, one batch each:
  `a` (T=10 C=7): a CTC graph, a CTC graph with a wildcard state at each end (not label-uniform), a random graph
      with cycles, self-loops, several start and accept nodes and labels >= C, an infeasible chain; T_b in
      {10, 8, 10, 1}.
  `b` (T=8 C=12): a word-piece alignment graph built with the reference's own union / closure / compose / remove, the
      same with wildcards, a CTC graph with T_b = 0, an empty graph.

Keys, per batch: `*_e` emissions [B, T, C]; `*_lens` (T_b); `*_n_nodes`, `*_n_arcs` per graph and the concatenated
`*_flags`, `*_src`, `*_dst`, `*_ilabel`, `*_olabel`, `*_w`; the reference's `*_losses` (NaN for T_b = 0, +inf without
an accepting path), `*_grads` (zero beyond T_b) and `*_arc_grads` (batch order, Graph arc numbering).

Run where the reference sources are (it needs oracle/_ref, compiled by `make -C oracle ref`):
    python tests/golden/make_graph_loss_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import graph_oracle as go  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
KEYS = ("flags", "src", "dst", "ilabel", "olabel", "w")


def cases():
    """(name, T, C, graphs, input_lens), seeded"""
    rng = np.random.default_rng(2024)
    a = [go.ctc_graph([1, 3, 3, 2]), go.with_wildcards(go.ctc_graph([4, 5]), 7, w_loop=-0.4),
         go.random_graph(rng, 9, 30, 7, n_start=2, n_accept=3, label_hi=9),
         go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3])]
    pieces = [(i,) for i in range(5)] + [(0, 1), (1, 2), (3, 4), (2, 3, 4), (4, 4)]
    dec = go.from_ref(go.decomposition_graph(go.REF_OPS, [0, 1, 2, 3, 4, 4], pieces))
    b = [dec, go.with_wildcards(dec, 12, w_loop=-0.2), go.ctc_graph([6, 7]), go.make([], [], [], [])]
    for g in a + b:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    return [("a", 10, 7, a, [10, 8, 10, 1]), ("b", 8, 12, b, [8, 8, 0, 5])]


def main():
    out = {}
    for name, T, C, graphs, lens in cases():
        rng = np.random.default_rng(sum(map(ord, name)) + 31)
        e = rng.uniform(-3, 3, (len(graphs), T, C)).astype(np.float32)
        lo, gr, ag = go.ref_graph_loss(e, graphs, lens)
        out.update({name + "_e": e, name + "_lens": np.asarray(lens, np.int32),
                    name + "_n_nodes": np.asarray([len(g["flags"]) for g in graphs], np.int32),
                    name + "_n_arcs": np.asarray([len(g["src"]) for g in graphs], np.int32),
                    name + "_losses": lo, name + "_grads": gr, name + "_arc_grads": ag})
        for k in KEYS:
            out[name + "_" + k] = np.concatenate([g[k] for g in graphs])
    np.savez_compressed(os.path.join(HERE, "graph_loss_golden.npz"), **out)


if __name__ == "__main__":
    main()
