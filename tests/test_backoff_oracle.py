"""The backoff fixture (tests/golden/backoff_golden.npz) against the live reference, its cases against their
description, and the float32 / float64 restatements of tests/backoff_oracle.py against the reference."""
import os

import numpy as np

from tests import backoff_oracle as bo
from tests import graph_oracle as go
from tests import sparse_trans_oracle as st
from tests import util
from tests.golden import make_backoff_golden as mk
from tests.test_graph_trans_oracle import need_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "backoff_golden.npz")


def load(z, name):
    G = go.make(z[name + "_G_flags"], z[name + "_G_src"], z[name + "_G_dst"], z[name + "_G_label"])
    graphs = [go.make(z["%s_A%d_flags" % (name, b)], z["%s_A%d_src" % (name, b)], z["%s_A%d_dst" % (name, b)],
                      z["%s_A%d_label" % (name, b)]) for b in range(len(z[name + "_lens"]))]
    return G, graphs


def test_golden_matches_live_reference(oracle):
    need_ref(oracle)
    z = np.load(GOLDEN)
    for name in mk.NAMES:
        G, graphs = load(z, name)
        e, lens, tw = z[name + "_e"], z[name + "_lens"], z[name + "_trans_w"]
        lo, gr, ag, tg = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
        assert util.close(lo, z[name + "_losses"]) and util.close(gr, z[name + "_grads"])
        assert util.close(ag, z[name + "_arc_grads"]) and util.close(tg, z[name + "_trans_grad"])
        paths, scores, arcs = bo.ref_backoff_viterbi(e, G, tw, lens)
        assert np.array_equal(scores, z[name + "_scores"]) and np.array_equal(paths, z[name + "_paths"])
        assert np.array_equal(arcs, z[name + "_arcs"])


def test_golden_cases_are_what_the_docstring_says():
    z = np.load(GOLDEN)
    levels = {}
    for name in mk.NAMES:
        G, _ = load(z, name)
        f, _ = bo.closure_levels(G)
        levels[name] = int(f.max())
        assert np.isnan(z[name + "_losses"][1]) and np.isneginf(z[name + "_scores"][1])
    assert levels["bigram"] == 1 and levels["trigram"] == 2 and (z["random_G_label"] == -1).sum() == 14


def test_restatements_match_the_reference(oracle):
    """restate_loss (float64) and restate_decode (float32, bit-exact scores) against the reference on the fixture"""
    need_ref(oracle)
    z = np.load(GOLDEN)
    for name in mk.NAMES:
        G, _ = load(z, name)
        e, lens, tw = z[name + "_e"], z[name + "_lens"], z[name + "_trans_w"]
        Z, _, _ = bo.restate_loss(e, lens, G, tw, e.shape[2])
        paths, scores, arcs = bo.ref_backoff_viterbi(e, G, tw, lens)
        for b in range(len(lens)):
            if lens[b] == 0:
                continue
            po = oracle
            gd = dict(G)
            gd["w"] = tw
            want = po.ref_op("forward_score", po.ref_op("intersect", po.RefGraph.linear(
                int(lens[b]), e.shape[2], e[b, :lens[b]].ravel()), go.ref_graph(gd))).item()
            assert util.close(np.float32(Z[b]), np.float32(want)), (name, b, Z[b], want)
            score, tie, labels, path_arcs = bo.restate_decode(e[b, :lens[b]], G, tw, e.shape[2])
            assert score == scores[b], (name, b, score, scores[b])
            if not tie:
                assert np.array_equal(labels, paths[b, :lens[b]]) and np.array_equal(path_arcs, arcs[b, :lens[b]])
