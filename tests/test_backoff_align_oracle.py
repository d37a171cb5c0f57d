"""The backoff alignment fixture (tests/golden/backoff_align_golden.npz) against the live reference, its cases against
their description, and the float32 restatement of the alignment's device route (tests/backoff_align_oracle.py)
against the fixture: scores bitwise, paths where it finds no tie."""
import numpy as np

from tests import backoff_align_oracle as ba
from tests import backoff_oracle as bo
from tests.test_graph_trans_oracle import need_ref


def test_golden_matches_live_reference(oracle):
    need_ref(oracle)
    for name, e, lens, G, tw, graphs, want in ba.golden_batches():
        got = ba.ref_backoff_trans_viterbi(e, graphs, G, tw, lens)
        for x, y in zip(got, want):
            assert np.array_equal(x, y), name


def test_golden_cases_are_what_the_docstring_says(oracle):
    """T_b = 0 and an utterance too short for its target (no accepting path) score -inf with -1 rows; the G kinds have
    the levels they are named for; epsilon arcs into start nodes; at least one traced path uses epsilon arcs"""
    need_ref(oracle)
    n_eps = 0
    for name, e, lens, G, tw, graphs, (paths, scores, arcs) in ba.golden_batches():
        assert lens[1] == 0 and np.isneginf(scores[1]) and (paths[1] == -1).all() and (arcs[1] == -1).all()
        assert lens[4] == 2 and np.isneginf(scores[4]) and (paths[4] == -1).all()
        assert np.isfinite(scores[0]) and np.isfinite(scores[2])
        f, _ = bo.closure_levels(G)
        assert int(f.max()) == {"bigram": 1, "trigram": 2}.get(name, int(f.max()))
        if name == "random":
            eps = G["olabel"] == bo.EPS
            assert eps.sum() == 14 and (G["flags"][G["dst"][eps]] & 1).any()
        used = []
        ba.ref_backoff_trans_viterbi(e, graphs, G, tw, lens, eps_used=used)
        n_eps += sum(used)
    assert n_eps > 0


def test_restatement_matches_the_golden():
    """restate_align over the product restated in numpy: scores bitwise, labels and A_b's arcs where no tie"""
    for name, e, lens, G, tw, graphs, (paths, scores, arcs) in ba.golden_batches():
        for b in range(len(lens)):
            n = int(lens[b])
            score, tie, labels, parcs = ba.restate_align(e[b, :n], graphs[b], G, tw, e.shape[2])
            assert np.array_equal(np.float32(score), scores[b]), (name, b, score, scores[b])
            if np.isfinite(score) and not tie:
                assert np.array_equal(labels, paths[b, :n]) and np.array_equal(parcs, arcs[b, :n]), (name, b)
