"""Regenerate tests/golden/sparse_cluster_golden.npz from the REAL reference (oracle/_ref/libgtn_ref.so): a transition
graph G beyond the one-CTA envelope of k_sparse.cu (5000 nodes, 40 000 arcs, C = 32; the cluster kernels' smallest
case) at small T, so that the CPU suite holds the restatements the cluster kernels are tested against
(test_sparse_trans_emulation.den64, sparse_viterbi_oracle.decode_outcome) to the reference at that size.

G, its weights and the emissions are seeded (``case()``) and not stored; the file holds what the reference computed:
  `Z` [B]                 forwardScore(intersect(E_b, G))
  `grad` [B, T, C]        its emission gradient (zero beyond T_b)
  `wgrad_idx`, `wgrad_val` its gradient in G's weights, summed over the batch, where it is not zero
  `paths`, `arcs` [B, T], `scores` [B]   viterbiPath / viterbiScore of intersect(E_b, G) (labels, G's arcs)

Run where the reference sources are (it needs oracle/_ref, compiled by `make -C oracle ref`):
    python tests/golden/make_sparse_cluster_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import sparse_trans_oracle as st  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "sparse_cluster_golden.npz")


def case():
    """-> (emissions [3, 4, 32], lens, G, trans_w), seeded"""
    rng = np.random.default_rng(5040)
    C, T = 32, 4
    G = st.sparse_graph(rng, 5000, 40000, C, n_start=40, n_accept=400, n_unreachable=0)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = rng.uniform(-3, 3, (3, T, C)).astype(np.float32)
    return e, np.asarray([4, 3, 1], np.int32), G, w


def main():
    from oracle import pyoracle as po
    from tests import graph_oracle as go
    from tests import sparse_viterbi_oracle as sv
    e, lens, G, w = case()
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
    paths, scores, arcs = sv.ref_sparse_viterbi(e, G, w, lens)
    idx = np.flatnonzero(wgrad).astype(np.int32)
    np.savez_compressed(GOLDEN, Z=Z, grad=grad, wgrad_idx=idx, wgrad_val=wgrad[idx].astype(np.float32), paths=paths,
                        scores=scores, arcs=arcs)


if __name__ == "__main__":
    main()
