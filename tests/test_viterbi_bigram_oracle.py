"""CPU checks of the test infrastructure for gtnb_viterbi_dense_ex's bigram kind (tests/viterbi_oracle.py): the C
oracle's evaluation against the committed golden fixture (tests/golden/viterbi_bigram_golden.npz, from the live
reference) and against the live reference on tie-heavy random cases; and the new C-ABI symbol."""
import os

import numpy as np
import pytest

from tests import viterbi_oracle as vo

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize("name", ["ties", "inf", "wide"])
def test_golden_matches_oracle(oracle, name):
    g = np.load(os.path.join(HERE, "golden", "viterbi_bigram_golden.npz"))
    e, W, lens = g[name + "_e"], g[name + "_W"], g[name + "_lens"]
    assert 0 in lens and 1 in lens
    for b in range(len(lens)):
        path, score = vo.oracle_viterbi_bigram(e[b, :lens[b]], W)
        assert np.array_equal(path, g[name + "_paths"][b, :lens[b]]), (name, b)
        assert (g[name + "_paths"][b, lens[b]:] == -1).all()
        assert np.float32(score) == g[name + "_scores"][b], (name, b, score)
    assert g[name + "_scores"][list(lens).index(0)] == -np.inf  # linearGraph(0, C) accepts nothing


def test_oracle_matches_live_reference_on_ties(oracle):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref/libgtn_ref.so is not built")
    rng = np.random.default_rng(2024)
    for k in range(120):
        C, T = int(rng.integers(2, 8)), int(rng.integers(0, 8))
        e = rng.integers(-1, 2, (1, T, C)).astype(np.float32)
        W = rng.integers(-1, 2, C * C).astype(np.float32)
        if k % 3 == 0:
            W[rng.random(C * C) < 0.3] = -np.inf
        pr, sr = vo.ref_viterbi_bigram(e[0], W)
        path, score = vo.oracle_viterbi_bigram(e[0], W)
        assert np.array_equal(path, pr) and score == sr, (C, T, path, pr, score, sr)


def test_symbol_declared_and_exported():
    from gtn_b200 import capi
    assert "gtnb_viterbi_dense_ex" in [s[0] for s in capi.SYMBOLS]
    header = open(os.path.join(HERE, "..", "include", "gtn_b200.h")).read()
    assert "int gtnb_viterbi_dense_ex(" in header
    assert "#define GTNB_DENSE_ASG 0" in header and "#define GTNB_DENSE_BIGRAM 1" in header
    assert (capi.DENSE_ASG, capi.DENSE_BIGRAM) == (0, 1)
    so = capi.LIB_PATH
    if not os.path.exists(so):
        pytest.skip("the library is not built")
    import ctypes
    assert hasattr(ctypes.CDLL(so), "gtnb_viterbi_dense_ex")
