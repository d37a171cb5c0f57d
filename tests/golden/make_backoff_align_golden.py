"""Regenerate tests/golden/backoff_align_golden.npz from the REAL reference (oracle/_ref/libgtn_ref.so): what
gtnb_backoff_transitions_viterbi computes for a transition graph G with epsilon arcs, every utterance run alone on its
first T_b rows (tests/backoff_align_oracle.py).

Batches (T=9 C=6, five utterances: a CTC graph, a random cyclic graph with labels >= C, a CTC graph, a random graph,
a CTC graph whose target cannot be read in 2 frames; T_b in {9, 0, 1, 6, 2}), for the G kinds of
make_backoff_golden.py:
  `bigram`:  a backoff bigram counted from a random corpus (one level of epsilon arcs)
  `trigram`: a pruned backoff trigram (two levels)
  `random`:  a random G with 14 epsilon arcs forming no cycle, several start and accept nodes, epsilon arcs into
             start nodes

Keys, per batch: `*_e` [B, T, C]; `*_lens`; G as `*_G_flags`, `*_G_src`, `*_G_dst`, `*_G_label` (-1: epsilon);
`*_trans_w`; target graph b as `*_A<b>_flags`, `*_A<b>_src`, `*_A<b>_dst`, `*_A<b>_label`, `*_A<b>_w`; the
alignment's `*_paths`, `*_arcs` (A_b's arcs) and `*_scores`.

Run where the reference sources are (it needs oracle/_ref, compiled by `make -C oracle ref`):
    python tests/golden/make_backoff_align_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import backoff_align_oracle as ba  # noqa: E402
from tests import backoff_oracle as bo  # noqa: E402
from tests import graph_oracle as go  # noqa: E402


def cases():
    """(name, G, trans_w, graphs, emissions, input_lens), seeded"""
    T, C = 9, 6
    for k, name in enumerate(ba.NAMES):
        rng = np.random.default_rng(200 + k)
        if name == "random":
            G, tw = bo.eps_graph(rng, 10, 45, C, 14, label_hi=C + 1)
        else:
            G, tw = bo.backoff_ngram(rng, C, 2 if name == "bigram" else 3, n_tokens=800, min_count=2)
        graphs = [go.ctc_graph([1, 2]), go.random_graph(rng, 5, 16, C, n_start=2, n_accept=2, label_hi=C + 2),
                  go.ctc_graph([3]), go.random_graph(rng, 4, 10, C, n_start=1, n_accept=2),
                  go.ctc_graph([1, 2, 3])]
        for g in graphs:
            g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
        lens = np.asarray([T, 0, 1, 6, 2], np.int32)
        e = rng.uniform(-2, 2, (len(graphs), T, C)).astype(np.float32)
        yield name, G, tw, graphs, e, lens


def main():
    out = {}
    for name, G, tw, graphs, e, lens in cases():
        paths, scores, arcs = ba.ref_backoff_trans_viterbi(e, graphs, G, tw, lens)
        out.update({name + "_e": e, name + "_lens": lens, name + "_G_flags": G["flags"], name + "_G_src": G["src"],
                    name + "_G_dst": G["dst"], name + "_G_label": G["olabel"], name + "_trans_w": tw,
                    name + "_paths": paths, name + "_arcs": arcs, name + "_scores": scores})
        for b, g in enumerate(graphs):
            for k in ("flags", "src", "dst", "w"):
                out["%s_A%d_%s" % (name, b, k)] = g[k]
            out["%s_A%d_label" % (name, b)] = g["olabel"]
    np.savez_compressed(ba.GOLDEN, **out)


if __name__ == "__main__":
    main()
