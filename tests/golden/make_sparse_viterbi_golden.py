"""Regenerate tests/golden/sparse_viterbi_golden.npz from the REAL reference (oracle/_ref/libgtn_ref.so): what
gtnb_viterbi_sparse and gtnb_sparse_transitions_viterbi compute, viterbiPath and viterbiScore of intersect(E_b, G)
(decode) and of intersect(intersect(A_b, G), E_b) (align), every utterance run alone on its first T_b rows
(tests/sparse_viterbi_oracle.py).

Batches (G, trans_w in G's arc order, emissions, lengths, target graphs A_b):
  `a` (T=9 C=7): a random sparse cyclic G (10 nodes, 45 arcs, several start and accept nodes, 2 unreachable nodes,
      labels up to 8 >= C), every 9th weight -inf; a CTC graph, a CTC graph with wildcard states, a random cyclic graph,
      an infeasible chain, an empty graph; T_b in {9, 0, 1, 6, 9}.
  `b` (T=8 C=4, tie-heavy): the trigram G with zero weights, 0 / 1 emissions and integer arc weights; a CTC graph, a
      random graph, two parallel equal arcs into a node with two parallel equal self-loops, a CTC graph;
      T_b in {8, 8, 5, 1}.
  `c` (T=10 C=30): the trigram G at C = 30 (900 states, 27 000 arcs) with uniform weights; three CTC graphs;
      T_b in {10, 7, 10}.

Keys, per batch: `*_e` [B, T, C]; `*_lens`; G as `*_G_flags`, `*_G_src`, `*_G_dst`, `*_G_label`; `*_trans_w`; the
target graphs as `*_n_nodes`, `*_n_arcs` and the concatenated `*_flags`, `*_src`, `*_dst`, `*_ilabel`, `*_olabel`,
`*_w`; the reference's decode `*_dec_paths` (labels), `*_dec_arcs` (G's arcs) [B, T] and `*_dec_scores` [B], and
alignment `*_ali_paths`, `*_ali_arcs` (A_b's arcs) and `*_ali_scores`; -1 beyond T_b and without an accepting path,
-inf scores without one.

Run where the reference sources are (it needs oracle/_ref, compiled by `make -C oracle ref`):
    python tests/golden/make_sparse_viterbi_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import graph_oracle as go  # noqa: E402
from tests import sparse_trans_oracle as st  # noqa: E402
from tests import sparse_viterbi_oracle as sv  # noqa: E402

KEYS = ("flags", "src", "dst", "ilabel", "olabel", "w")


def cases():
    """(name, T, C, G, trans_w, graphs, input_lens, tie-heavy), seeded"""
    rng = np.random.default_rng(2031)
    G_a = st.sparse_graph(rng, 10, 45, 7, n_start=3, n_accept=3, label_hi=9)
    w_a = rng.uniform(-1, 1, len(G_a["src"])).astype(np.float32)
    w_a[::9] = -np.inf
    a = [go.ctc_graph([1, 3, 3, 2]), go.with_wildcards(go.ctc_graph([4, 5]), 7, w_loop=-0.4),
         go.random_graph(rng, 9, 30, 7, n_start=3, n_accept=3, label_hi=9),
         go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3]), go.make([], [], [], [])]
    for g in a:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    G_b = st.trigram_graph(4)
    b = [go.ctc_graph([1, 2, 2]), go.random_graph(rng, 6, 24, 4, n_start=2, n_accept=2),
         go.make([1, 2], [0, 0, 1, 1], [1, 1, 1, 1], [1, 1, 2, 2]), go.ctc_graph([3])]
    for g in b:
        g["w"] = rng.integers(-1, 1, len(g["src"])).astype(np.float32)
    b[2]["w"][:] = 0.0
    G_c = st.trigram_graph(30)
    w_c = rng.uniform(-1, 1, len(G_c["src"])).astype(np.float32)
    c = [go.ctc_graph(rng.integers(1, 30, 3)) for _ in range(3)]
    for g in c:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    return [("a", 9, 7, G_a, w_a, a, [9, 0, 1, 6, 9], False),
            ("b", 8, 4, G_b, np.zeros(len(G_b["src"]), np.float32), b, [8, 8, 5, 1], True),
            ("c", 10, 30, G_c, w_c, c, [10, 7, 10], False)]


def main():
    out = {}
    for name, T, C, G, tw, graphs, lens, ties in cases():
        rng = np.random.default_rng(sum(map(ord, name)) + 53)
        e = (rng.integers(0, 2, (len(graphs), T, C)) if ties else rng.uniform(-3, 3, (len(graphs), T, C)))
        e = e.astype(np.float32)
        for b, n in enumerate(lens):
            e[b, n:] = np.nan
        out.update({name + "_e": e, name + "_lens": np.asarray(lens, np.int32), name + "_trans_w": tw,
                    name + "_G_flags": G["flags"], name + "_G_src": G["src"], name + "_G_dst": G["dst"],
                    name + "_G_label": G["olabel"],
                    name + "_n_nodes": np.asarray([len(g["flags"]) for g in graphs], np.int32),
                    name + "_n_arcs": np.asarray([len(g["src"]) for g in graphs], np.int32)})
        for k in KEYS:
            out[name + "_" + k] = np.concatenate([np.asarray(g[k]) for g in graphs]).astype(
                np.uint8 if k == "flags" else np.float32 if k == "w" else np.int32)
        for op, res in (("dec", sv.ref_sparse_viterbi(e, G, tw, lens)),
                        ("ali", sv.ref_sparse_trans_viterbi(e, graphs, G, tw, lens))):
            for k, x in zip(("paths", "scores", "arcs"), res):
                out["%s_%s_%s" % (name, op, k)] = x
    np.savez_compressed(sv.GOLDEN, **out)


if __name__ == "__main__":
    main()
