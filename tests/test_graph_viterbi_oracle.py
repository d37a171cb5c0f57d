"""CPU checks for gtnb_graph_viterbi: the committed golden fixture (tests/golden/graph_viterbi_golden.npz,
tests/golden/make_graph_viterbi_golden.py) against the live reference; the live reference's viterbiPath / viterbiScore of compose(A, E), as
tests/graph_viterbi_oracle.py reads them (arc ids carried through the ilabels), against a float32 restatement of the
frame-synchronous tropical recursion -- scores bit for bit, and every path a path of A with T_b arcs from a start node
to an accept node whose value is the score -- on CTC, wildcard and random cyclic graphs with several start and accept
nodes, labels >= C, T_b in {0, 1}, infeasible graphs, parallel equal arcs and tie-heavy integer emissions; and the
C-ABI symbol."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import graph_oracle as go
from tests import graph_viterbi_oracle as gv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "graph_viterbi_golden.npz")


def golden_batches():
    """-> [(name, emissions, graphs, lens, (paths, scores, arcs))] of the committed fixture"""
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
        out.append((name, z[name + "_e"], graphs, z[name + "_lens"],
                    (z[name + "_paths"], z[name + "_scores"], z[name + "_arcs"])))
    return out


def need_ref(oracle):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref/libgtn_ref.so is missing")


def cases(C, seed, ties):
    rng = np.random.default_rng(seed)
    graphs = [go.ctc_graph(rng.integers(1, C, 3)),
              go.with_wildcards(go.ctc_graph(rng.integers(1, C, 2)), C, w_loop=0.0 if ties else -0.2),
              go.random_graph(rng, 7, 30, C, n_start=3, n_accept=3, label_hi=C + 2),
              go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3]),  # accepts 3 frames only: infeasible at T_b != 3
              go.make([1, 2], [0, 0, 1, 1], [1, 1, 1, 1], [1, 1, 2, 2])]  # parallel equal arcs and self-loops
    T = 9
    lens = np.asarray([T, 1, T - 2, 0, T], np.int32)
    if ties:
        e = rng.integers(0, 2, (len(graphs), T, C)).astype(np.float32)
        for g in graphs:
            g["w"] = rng.integers(-1, 1, len(g["src"])).astype(np.float32) if len(g["src"]) > 4 else g["w"] * 0
    else:
        e = rng.uniform(-3, 3, (len(graphs), T, C)).astype(np.float32)
        for g in graphs:
            g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    return e, graphs, lens


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("C", [4, 11])
def test_reference_paths_are_best_paths_of_the_graph(oracle, C, ties):
    need_ref(oracle)
    e, graphs, lens = cases(C, 3 + C, ties)
    paths, scores, arcs = gv.ref_graph_viterbi(e, graphs, lens)
    for b, g in enumerate(graphs):
        Tb = int(lens[b])
        assert (paths[b, Tb:] == -1).all() and (arcs[b, Tb:] == -1).all()
        S = gv.tropical_scores(e[b, :Tb], g, C)
        acc = (g["flags"] & 2) != 0
        best = np.float32(S[Tb, acc].max(initial=-np.inf)) if Tb > 0 else np.float32(-np.inf)
        assert scores[b].tobytes() == best.tobytes(), (b, scores[b], best)
        if not np.isfinite(best):
            assert (paths[b] == -1).all() and (arcs[b] == -1).all()
            continue
        a = arcs[b, :Tb]
        assert g["flags"][g["src"][a[0]]] & 1 and g["flags"][g["dst"][a[-1]]] & 2
        assert np.array_equal(g["dst"][a[:-1]], g["src"][a[1:]])
        assert np.array_equal(g["olabel"][a], paths[b, :Tb])
        assert gv.path_score(e[b], g, a).tobytes() == best.tobytes()


@pytest.mark.parametrize("i", [0, 1, 2])
def test_golden_matches_live_reference(oracle, i):
    need_ref(oracle)
    name, e, graphs, lens, (p, s, a) = golden_batches()[i]
    pr, sr, ar = gv.ref_graph_viterbi(e, graphs, lens)
    assert np.array_equal(pr, p) and np.array_equal(ar, a) and np.array_equal(sr.view(np.int32), s.view(np.int32))


def test_golden_cases_are_what_the_docstring_says():
    (_, ea, a, la, (_, sa, _)), (_, eb, b, lb, (_, sb, _)), (_, ec, c, lc, (_, sc, ac)) = golden_batches()
    assert (a[2]["olabel"] >= 7).any() and (b[3]["olabel"] >= 12).any()
    assert np.count_nonzero(a[2]["flags"] & 1) >= 2 and np.count_nonzero(a[2]["flags"] & 2) >= 2
    assert list(la) == [10, 8, 10, 1, 10] and list(lb) == [8, 8, 0, 5]
    assert np.isneginf(sa[3]) and np.isneginf(sa[4]) and len(a[4]["flags"]) == 0 and np.isneginf(sb[2])
    assert go.non_uniform_nodes(a[1], 7) >= 2 and go.non_uniform_nodes(b[1], 12) >= 2
    # tie-heavy: integer values, and the parallel equal arcs tie on the reference's path
    assert np.array_equal(ec, np.round(ec)) and np.array_equal(c[3]["w"], np.round(c[3]["w"]))
    assert np.array_equal(c[2]["src"], [0, 0, 1, 1]) and np.array_equal(c[2]["olabel"], [1, 1, 2, 2])
    assert gv.trace_ties(ec[2, :lc[2]], c[2], 4, ac[2, :lc[2]])


def test_tie_cases_have_ties():
    """the tie-heavy inputs above do tie: some node of frame T_b is reached by two in-arcs at the maximum"""
    e, graphs, lens = cases(4, 7, True)
    g, Tb = graphs[4], int(lens[4])
    S = gv.tropical_scores(e[4, :Tb], g, 4)
    assert np.isfinite(S[Tb, 1])
    cand = [S[Tb - 1, g["src"][a]] + (g["w"][a] + e[4, Tb - 1, g["olabel"][a]]) for a in (2, 3)]
    assert cand[0] == cand[1] == S[Tb, 1]


def test_symbol_declared_and_exported():
    from gtn_b200 import capi
    assert "gtnb_graph_viterbi" in [s[0] for s in capi.SYMBOLS]
    with open(os.path.join(ROOT, "include", "gtn_b200.h")) as f:
        assert "int gtnb_graph_viterbi(" in f.read()
    so = os.path.join(ROOT, "gtn_b200", "lib", "libgtn_b200.so")
    if not os.path.exists(so):
        pytest.skip("the library is not built")
    assert hasattr(C.CDLL(so), "gtnb_graph_viterbi")
