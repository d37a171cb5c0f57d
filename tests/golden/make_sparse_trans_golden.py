"""Regenerate tests/golden/sparse_trans_golden.npz from the REAL reference (oracle/_ref/libgtn_ref.so): the loss of
gtnb_sparse_transitions_loss, every utterance run alone on its first T_b rows, A_b matched on its olabels
(tests/sparse_trans_oracle.py):
    forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(A_b, G), E_b)),   trans_w [G's arcs]

Batches:
  `a` (T=8 C=5): G is the trigram graph at C = 5 (25 nodes, 125 arcs); a CTC graph, a random cyclic graph with
      several start and accept nodes, start nodes with in-arcs and labels >= C, an infeasible chain, a CTC graph;
      T_b in {8, 6, 8, 1}.
  `b` (T=8 C=12): G is a random sparse cyclic graph with 3 start and 3 accept nodes, two unreachable nodes and labels
      >= C; a word-piece decomposition graph built with the reference's own union / closure / compose / remove, a CTC
      graph with T_b = 0, a random cyclic graph; T_b in {8, 0, 5}.
  `c` (T=6 C=12): G is the dense bigram graph at C = 12 with -inf weights (a third of them); the decomposition graph and a
      random graph.

Keys, per batch: `*_e` emissions [B, T, C]; `*_lens` (T_b); `*_n_nodes`, `*_n_arcs` per graph and the concatenated
`*_flags`, `*_src`, `*_dst`, `*_ilabel`, `*_olabel`, `*_w`; G as `*_G_flags`, `*_G_src`, `*_G_dst`, `*_G_label`;
`*_trans_w`; the reference's `*_losses` (NaN for T_b = 0, +inf without an accepting path), `*_grads` (zero beyond
T_b), `*_arc_grads` (batch order, Graph arc numbering) and `*_trans_grad` (the batch sum, G's arc numbering).

Run where the reference sources are (it needs oracle/_ref, compiled by `make -C oracle ref`):
    python tests/golden/make_sparse_trans_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import graph_oracle as go  # noqa: E402
from tests import sparse_trans_oracle as st  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
KEYS = ("flags", "src", "dst", "ilabel", "olabel", "w")


def cases():
    """(name, T, C, graphs, input_lens, G, -inf transitions), seeded"""
    rng = np.random.default_rng(2026)
    a = [go.ctc_graph([1, 3, 3, 2]), go.random_graph(rng, 9, 30, 5, n_start=3, n_accept=3, label_hi=7),
         go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3]), go.ctc_graph([4])]
    pieces = [(i,) for i in range(5)] + [(0, 1), (1, 2), (3, 4), (2, 3, 4), (4, 4)]
    dec = go.from_ref(go.decomposition_graph(go.REF_OPS, [0, 1, 2, 3, 4, 4], pieces))
    b = [dec, go.ctc_graph([6, 7]), go.random_graph(rng, 7, 25, 12, n_start=2, n_accept=2, label_hi=14)]
    c = [dict(dec), go.random_graph(rng, 6, 20, 12, n_start=2, n_accept=2)]
    for g in a + b + c:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    Ga = st.trigram_graph(5)
    Gb = st.sparse_graph(rng, 12, 70, 12, label_hi=14)
    Gc = st.bigram_graph(12)
    return [("a", 8, 5, a, [8, 6, 8, 1], Ga, False), ("b", 8, 12, b, [8, 0, 5], Gb, False),
            ("c", 6, 12, c, [6, 6], Gc, True)]


def main():
    out = {}
    for name, T, C, graphs, lens, G, neg_inf in cases():
        rng = np.random.default_rng(sum(map(ord, name)) + 43)
        e = rng.uniform(-3, 3, (len(graphs), T, C)).astype(np.float32)
        tw = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
        if neg_inf:
            tw[rng.random(len(tw)) < 1 / 3] = -np.inf
        out.update({name + "_e": e, name + "_lens": np.asarray(lens, np.int32),
                    name + "_n_nodes": np.asarray([len(g["flags"]) for g in graphs], np.int32),
                    name + "_n_arcs": np.asarray([len(g["src"]) for g in graphs], np.int32),
                    name + "_G_flags": G["flags"], name + "_G_src": G["src"], name + "_G_dst": G["dst"],
                    name + "_G_label": G["olabel"], name + "_trans_w": tw})
        for k in KEYS:
            out[name + "_" + k] = np.concatenate([g[k] for g in graphs])
        lo, gr, ag, tg = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
        out.update({name + "_losses": lo, name + "_grads": gr, name + "_arc_grads": ag, name + "_trans_grad": tg})
    np.savez_compressed(os.path.join(HERE, "sparse_trans_golden.npz"), **out)


if __name__ == "__main__":
    main()
