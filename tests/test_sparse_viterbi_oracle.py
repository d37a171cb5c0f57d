"""CPU checks for gtnb_viterbi_sparse and gtnb_sparse_transitions_viterbi: the committed golden fixture
(tests/golden/sparse_viterbi_golden.npz, tests/golden/make_sparse_viterbi_golden.py) against the live reference through
tests/sparse_viterbi_oracle.py, decode and alignment; and, without the reference, the fixture against the decode's
float32 restatement: scores bit-equal, the restatement's path == the reference's wherever it finds no tie (the
first-accept-node rule and the association), ties where the batch is tie-heavy, every stored decode path a path of G
whose value is the score; every stored alignment path a path of A_b carrying its labels; the C-ABI symbols."""
import os

import numpy as np
import pytest

from tests import sparse_viterbi_oracle as sv
from tests.test_graph_trans_oracle import need_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("case", range(len(sv.NAMES)))
def test_golden_matches_live_reference(oracle, case):
    need_ref(oracle)
    name, e, lens, G, tw, graphs, dec, ali = sv.golden_batches()[case]
    for got, want in ((sv.ref_sparse_viterbi(e, G, tw, lens), dec),
                      (sv.ref_sparse_trans_viterbi(e, graphs, G, tw, lens), ali)):
        for x, y in zip(got, want):
            assert np.array_equal(x, y), (name, x, y)


@pytest.mark.parametrize("case", range(len(sv.NAMES)))
def test_golden_decode_is_the_restatement(case):
    name, e, lens, G, tw, graphs, (paths, scores, arcs), _ = sv.golden_batches()[case]
    C = e.shape[2]
    n_ties = 0
    for b in range(e.shape[0]):
        n = int(lens[b])
        score, tie, labels, path_arcs = sv.decode_outcome(e[b, :n], G, tw, C)
        assert scores[b].tobytes() == np.float32(score).tobytes(), (name, b, scores[b], score)
        n_ties += tie
        if not np.isfinite(score):
            assert (paths[b] == -1).all() and (arcs[b] == -1).all()
            continue
        assert (paths[b, n:] == -1).all() and (arcs[b, n:] == -1).all()
        assert sv.is_path(G, arcs[b, :n]) and np.array_equal(paths[b, :n], G["olabel"][arcs[b, :n]])
        assert sv.path_value(e[b, :n], G, tw, arcs[b, :n]) == scores[b]
        if not tie:
            assert np.array_equal(paths[b, :n], labels) and np.array_equal(arcs[b, :n], path_arcs), (name, b)
    assert (n_ties > 0) == (name == "b")


def test_golden_alignment_paths_are_paths_of_the_targets():
    for name, e, lens, G, tw, graphs, _, (paths, scores, arcs) in sv.golden_batches():
        for b, g in enumerate(graphs):
            n = int(lens[b])
            if not np.isfinite(scores[b]):
                assert (paths[b] == -1).all() and (arcs[b] == -1).all()
                continue
            a = arcs[b, :n]
            assert sv.is_path(g, a) and np.array_equal(paths[b, :n], g["olabel"][a]), (name, b)
            assert (paths[b, n:] == -1).all()


def test_golden_cases_are_what_the_docstring_says():
    batches = {x[0]: x for x in sv.golden_batches()}
    _, e, lens, G, tw, graphs, dec, ali = batches["a"]
    assert list(lens) == [9, 0, 1, 6, 9] and e.shape[2] == 7 and (G["olabel"] >= 7).any()
    assert np.isneginf(tw).any() and np.isneginf(dec[1][1]) and np.isneginf(ali[1][[1, 3, 4]]).all()
    assert np.isfinite(dec[1][[0, 2, 3, 4]]).all()
    _, e, lens, G, tw, graphs, dec, ali = batches["b"]
    assert len(G["flags"]) == 16 and not tw.any() and set(np.unique(e[np.isfinite(e)])) <= {0.0, 1.0}
    _, e, lens, G, tw, graphs, dec, ali = batches["c"]
    assert len(G["flags"]) == 900 and len(G["src"]) == 27000 and np.isfinite(dec[1]).all()


def test_symbols_declared_and_exported():
    from gtn_b200 import capi
    names = {name for name, _, _ in capi.SYMBOLS}
    assert {"gtnb_viterbi_sparse", "gtnb_sparse_transitions_viterbi"} <= names
    with open(os.path.join(ROOT, "include", "gtn_b200.h")) as f:
        text = f.read()
    assert "int gtnb_viterbi_sparse(" in text and "int gtnb_sparse_transitions_viterbi(" in text
