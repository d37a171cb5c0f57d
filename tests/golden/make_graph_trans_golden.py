"""Regenerate tests/golden/graph_trans_golden.npz from the REAL reference (oracle/_ref/libgtn_ref.so): the loss of
gtnb_graph_transitions_loss for both transition kinds, every utterance run alone on its first T_b rows, A_b matched on
its olabels (tests/graph_trans_oracle.py):
    asg:    forwardScore(compose(E_b, G)) - forwardScore(compose(compose(A_b, G), E_b)),   trans_w [C + C*C]
    bigram: forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(A_b, G), E_b)),   trans_w [C*C]

Graph batches, each run with both kinds:
  `a` (T=10 C=7): a CTC graph, a CTC graph with a wildcard state at each end, a random cyclic graph with several start
      and accept nodes, start nodes with in-arcs and labels >= C, an infeasible chain; T_b in {10, 8, 10, 1}.
  `b` (T=8 C=12): a word-piece decomposition graph built with the reference's own union / closure / compose / remove,
      the same with wildcards, a CTC graph with T_b = 0, a random cyclic graph; T_b in {8, 8, 0, 5}.
  `c` (T=6 C=12): the decomposition graph and a random graph with -inf transition weights (a third of W, and one
      start weight for asg).

Keys, per batch: `*_e` emissions [B, T, C]; `*_lens` (T_b); `*_n_nodes`, `*_n_arcs` per graph and the concatenated
`*_flags`, `*_src`, `*_dst`, `*_ilabel`, `*_olabel`, `*_w`; per batch and kind (`*_asg_*`, `*_bigram_*`): `trans_w`,
the reference's `losses` (NaN for T_b = 0, +inf without an accepting path), `grads` (zero beyond T_b), `arc_grads`
(batch order, Graph arc numbering) and `trans_grad` (the batch sum).

Run where the reference sources are (it needs oracle/_ref, compiled by `make -C oracle ref`):
    python tests/golden/make_graph_trans_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import graph_oracle as go  # noqa: E402
from tests import graph_trans_oracle as gt  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
KEYS = ("flags", "src", "dst", "ilabel", "olabel", "w")
KINDS = (("asg", gt.ASG), ("bigram", gt.BIGRAM))


def cases():
    """(name, T, C, graphs, input_lens, -inf transitions), seeded"""
    rng = np.random.default_rng(2025)
    a = [go.ctc_graph([1, 3, 3, 2]), go.with_wildcards(go.ctc_graph([4, 5]), 7, w_loop=-0.4),
         go.random_graph(rng, 9, 30, 7, n_start=3, n_accept=3, label_hi=9),
         go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3])]
    pieces = [(i,) for i in range(5)] + [(0, 1), (1, 2), (3, 4), (2, 3, 4), (4, 4)]
    dec = go.from_ref(go.decomposition_graph(go.REF_OPS, [0, 1, 2, 3, 4, 4], pieces))
    b = [dec, go.with_wildcards(dec, 12, w_loop=-0.2), go.ctc_graph([6, 7]),
         go.random_graph(rng, 7, 25, 12, n_start=2, n_accept=2, label_hi=14)]
    c = [dict(dec), go.random_graph(rng, 6, 20, 12, n_start=2, n_accept=2)]
    for g in a + b + c:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    return [("a", 10, 7, a, [10, 8, 10, 1], False), ("b", 8, 12, b, [8, 8, 0, 5], False),
            ("c", 6, 12, c, [6, 6], True)]


def transitions(rng, C, kind, neg_inf):
    tw = rng.uniform(-1, 1, (C + C * C) if kind == gt.ASG else C * C).astype(np.float32)
    if neg_inf:
        W = tw[-C * C:]
        W[rng.random(C * C) < 1 / 3] = -np.inf
        if kind == gt.ASG:
            tw[2] = -np.inf
    return tw


def main():
    out = {}
    for name, T, C, graphs, lens, neg_inf in cases():
        rng = np.random.default_rng(sum(map(ord, name)) + 41)
        e = rng.uniform(-3, 3, (len(graphs), T, C)).astype(np.float32)
        out.update({name + "_e": e, name + "_lens": np.asarray(lens, np.int32),
                    name + "_n_nodes": np.asarray([len(g["flags"]) for g in graphs], np.int32),
                    name + "_n_arcs": np.asarray([len(g["src"]) for g in graphs], np.int32)})
        for k in KEYS:
            out[name + "_" + k] = np.concatenate([g[k] for g in graphs])
        for kname, kind in KINDS:
            tw = transitions(rng, C, kind, neg_inf)
            lo, gr, ag, tg = gt.ref_graph_trans_loss(e, graphs, kind, tw, lens)
            p = "%s_%s_" % (name, kname)
            out.update({p + "trans_w": tw, p + "losses": lo, p + "grads": gr, p + "arc_grads": ag,
                        p + "trans_grad": tg})
    np.savez_compressed(os.path.join(HERE, "graph_trans_golden.npz"), **out)


if __name__ == "__main__":
    main()
