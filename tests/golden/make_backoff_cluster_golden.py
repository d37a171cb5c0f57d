"""Regenerate tests/golden/backoff_cluster_golden.npz from the REAL reference (oracle/_ref/libgtn_ref.so): a backoff
transition graph G beyond the one-CTA envelope of k_sparse.cu's backoff sweeps (the backoff 4-gram at C = 64 counted
from 60 000 tokens: 8563 states, 57 231 emitting and 8562 epsilon arcs, 3 levels; the cluster kernels take it with
N = 2) at small T, so that the CPU suite holds the restatements and the emulated cluster kernels to the reference at
a size only the cluster route can take.

G, its weights, the emissions and the two target graphs are seeded (``case()``) and not stored; the file holds what
the reference computed:
  `Z` [B]                  forwardScore(intersect(E_b, G))
  `grad` [B, T, C]         its emission gradient (zero beyond T_b)
  `wgrad_idx`, `wgrad_val` its gradient in G's weights, summed over the batch, where it is not zero
  `paths`, `arcs` [B, T], `scores` [B]    viterbiPath / viterbiScore of intersect(E_b, G) (labels, G's emitting arcs)
  `align_paths`, `align_arcs` [2, T], `align_scores` [2]
                           the alignment of the first two utterances within the two target graphs: viterbiPath /
                           viterbiScore of intersect(intersect(A_b, G), E_b) (labels, A_b's arcs)

Run where the reference sources are (it needs oracle/_ref, compiled by `make -C oracle ref`):
    python tests/golden/make_backoff_cluster_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import backoff_oracle as bo  # noqa: E402
from tests import graph_oracle as go  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "backoff_cluster_golden.npz")


def case():
    """-> (emissions [3, 6, 64], lens, G, trans_w, two target graphs), seeded"""
    G, w = bo.backoff_ngram(np.random.default_rng(1), 64, 4, n_tokens=60000)
    rng = np.random.default_rng(8563)
    C, T = 64, 6
    e = rng.uniform(-3, 3, (3, T, C)).astype(np.float32)
    graphs = [go.ctc_graph(rng.integers(1, C, 2)), go.ctc_graph(rng.integers(1, C, 3))]
    for g in graphs:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    return e, np.asarray([6, 5, 3], np.int32), G, w, graphs


def main():
    from oracle import pyoracle as po
    from tests import backoff_align_oracle as ba
    e, lens, G, w, graphs = case()
    B, T, C = e.shape
    gd = dict(G)
    gd["w"] = w
    Z, grad, wgrad = np.zeros(B, np.float32), np.zeros_like(e), np.zeros(len(w), np.float64)
    for b in range(B):
        n = int(lens[b])
        rg = go.ref_graph(gd)
        E = po.RefGraph.linear(n, C, e[b, :n].ravel())
        den = po.ref_op("forward_score", po.ref_op("intersect", E, rg))
        po.ref_backward(den)
        Z[b] = den.item()
        grad[b, :n] = E.grad().weights().reshape(n, C)
        wgrad += rg.grad().weights()
    paths, scores, arcs = bo.ref_backoff_viterbi(e, G, w, lens)
    ap, asc, aa = ba.ref_backoff_trans_viterbi(e[:2], graphs, G, w, lens[:2])
    idx = np.flatnonzero(wgrad).astype(np.int32)
    np.savez_compressed(GOLDEN, Z=Z, grad=grad, wgrad_idx=idx, wgrad_val=wgrad[idx].astype(np.float32), paths=paths,
                        scores=scores, arcs=arcs, align_paths=ap, align_scores=asc, align_arcs=aa)


if __name__ == "__main__":
    main()
