"""CPU checks for gtnb_graph_transitions_viterbi's reference outputs: the committed golden fixture
(tests/golden/graph_trans_viterbi_golden.npz, tests/golden/make_graph_trans_viterbi_golden.py) against the live
reference through tests/graph_trans_viterbi_oracle.py; its cases are what its docstring says; and, without the
reference, its scores equal the float32 tropical recursion over the device route's graph (the product with BIGRAM's
start states folded through tau) bit for bit, and every stored path is a path of A_b of T_b arcs whose value in that
association is the score."""
import os

import numpy as np
import pytest

from tests import graph_oracle as go
from tests import graph_trans_viterbi_oracle as gtv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "graph_trans_viterbi_golden.npz")
KINDS = {"asg": gtv.ASG, "bigram": gtv.BIGRAM}


def golden_batches():
    """-> [(name, kind name, emissions, graphs, lens, trans_w, (paths, scores, arcs))] of the committed fixture"""
    z = np.load(GOLDEN)
    out = []
    for name in ("a", "b", "c"):
        graphs, n0, a0 = [], 0, 0
        for n, a in zip(z[name + "_n_nodes"], z[name + "_n_arcs"]):
            g = {"flags": z[name + "_flags"][n0:n0 + n]}
            for k in ("src", "dst", "ilabel", "olabel", "w"):
                g[k] = z[name + "_" + k][a0:a0 + a]
            graphs.append(g)
            n0, a0 = n0 + n, a0 + a
        for kind in KINDS:
            p = "%s_%s_" % (name, kind)
            out.append((name, kind, z[name + "_e"], graphs, z[name + "_lens"], z[p + "trans_w"],
                        (z[p + "paths"], z[p + "scores"], z[p + "arcs"])))
    return out


def need_ref(oracle):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref/libgtn_ref.so is missing")


@pytest.mark.parametrize("case", range(6))
def test_golden_matches_live_reference(oracle, case):
    need_ref(oracle)
    name, kind, e, graphs, lens, tw, want = golden_batches()[case]
    got = gtv.ref_graph_trans_viterbi(e, graphs, KINDS[kind], tw, lens)
    for x, y in zip(got, want):
        assert np.array_equal(x, y), (name, kind, x, y)


@pytest.mark.parametrize("case", range(6))
def test_golden_scores_are_the_float32_recursion_over_the_device_routes_graph(case):
    name, kind, e, graphs, lens, tw, (paths, scores, arcs) = golden_batches()[case]
    C = e.shape[2]
    k = KINDS[kind]
    for b, g in enumerate(graphs):
        Tb = int(lens[b])
        p, _ = gtv.tropical_product(g, C, k, tw)
        s, _ = gtv.device_route_outcome(e[b, :Tb], p, C)
        assert s.tobytes() == scores[b].tobytes(), (name, kind, b, s, scores[b])
        assert (paths[b, Tb:] == -1).all() and (arcs[b, Tb:] == -1).all()
        if not np.isfinite(scores[b]):
            assert (paths[b] == -1).all() and (arcs[b] == -1).all()
            continue
        a = arcs[b, :Tb]
        assert np.array_equal(g["olabel"][a], paths[b, :Tb])
        assert g["flags"][g["src"][a[0]]] & 1 and g["flags"][g["dst"][a[-1]]] & 2
        assert np.array_equal(g["dst"][a[:-1]], g["src"][a[1:]])
        assert gtv.path_value(e[b, :Tb], g, k, tw, paths[b, :Tb], a) == scores[b]


def test_golden_cases_are_what_the_docstring_says():
    batches = {(n, k): (e, g, lens, tw, want) for n, k, e, g, lens, tw, want in golden_batches()}
    for kind in KINDS:
        e, a, lens, tw, (_, s, _) = batches["a", kind]
        assert lens.min() == 1 and (a[2]["olabel"] >= 7).any() and len(a[4]["flags"]) == 0
        starts = np.flatnonzero(a[2]["flags"] & 1)
        assert len(starts) >= 2 and np.isin(a[2]["dst"], starts).any()  # start nodes with in-arcs
        assert np.isneginf(s[[3, 4]]).all() and np.isfinite(s[:3]).all()
        e, b, lens, tw, (_, s, _) = batches["b", kind]
        assert lens.min() == 0 and go.non_uniform_nodes(b[1], 12) > 0  # wildcards
        assert np.isneginf(tw).any() and np.isfinite(s[:2]).all()
        e, c, lens, tw, (_, s, _) = batches["c", kind]
        assert np.array_equal(e, np.round(e)) and np.array_equal(tw, np.round(tw)) and np.isfinite(s).all()
        assert not np.isneginf(batches["a", kind][3]).any()
