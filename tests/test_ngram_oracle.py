"""CPU checks of the test infrastructure for gtnb_ngram_ctc_loss (tests/ngram_oracle.py): the committed golden
fixture (tests/golden/ngram_golden.npz, from the live reference) against the C oracle; the oracle against the live
reference on random cases; the float64 referee against the oracle; and the new C-ABI symbol."""
import os

import numpy as np
import pytest

from tests import ngram_oracle as no
from tests import util

HERE = os.path.dirname(os.path.abspath(__file__))


def _split(cat, lens):
    out, o = [], 0
    for n in lens:
        out.append(cat[o:o + n])
        o += n
    return out


def _same(a, b, rtol=1e-5, atol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.allclose(a, b, rtol=rtol, atol=atol, equal_nan=True)


@pytest.mark.parametrize("name", ["a", "b"])
def test_golden_matches_oracle(oracle, name):
    g = np.load(os.path.join(HERE, "golden", "ngram_golden.npz"))
    e, W, blank = g[name + "_e"], g[name + "_w"], int(g[name + "_blank"])
    targets, lens = _split(g[name + "_targets"], g[name + "_target_lens"]), g[name + "_lens"]
    tg = np.zeros_like(W)
    for b in range(len(targets)):
        lo, go, to = no.oracle_ngram_ctc(e[b, :lens[b]], W, targets[b], blank)
        assert _same(lo, g[name + "_losses"][b])
        assert _same(go, g[name + "_grads"][b, :lens[b]])
        tg += to
    assert _same(tg, g[name + "_trans_grad"], atol=1e-4)


def _random_case(rng, C):
    T = int(rng.integers(0, 12))
    blank = int(rng.integers(0, C))
    kind = rng.integers(0, 4)
    U = 0 if kind == 0 else int(rng.integers(1, 6))
    labels = [c for c in range(C) if c != blank] or [blank]
    tg = [int(x) for x in rng.choice(labels, U)]
    if kind == 1 and U > 1:
        tg = [tg[0]] * U  # repeats: no skip arc
    e = rng.uniform(-5, 5, (T, C)).astype(np.float32)
    W = rng.uniform(-3, 3, C * C).astype(np.float32)
    return e, W, tg, blank


@pytest.mark.parametrize("C", [4, 8, 28, 64])
def test_oracle_matches_live_reference(oracle, C):
    po = oracle
    if not po.have_ref():
        pytest.skip("oracle/_ref/libgtn_ref.so is not built")
    rng = np.random.default_rng(C)
    for _ in range(6):
        e, W, tg, blank = _random_case(rng, C)
        lr, gr, tr = no.ref_ngram_ctc(e, W, tg, blank)
        lo, go, to = no.oracle_ngram_ctc(e, W, tg, blank)
        assert _same(lo, lr) or (np.isnan(lo) and np.isnan(lr)), (e.shape, tg, lo, lr)
        assert _same(go, gr) and _same(to, tr, atol=1e-4)


@pytest.mark.parametrize("C", [4, 8, 28, 64])
def test_f64_referee_matches_oracle(oracle, C):
    rng = np.random.default_rng(100 + C)
    for _ in range(6):
        e, W, tg, blank = _random_case(rng, C)
        l64, g64, t64 = no.ngram_ctc_f64(e, W, tg, blank)
        lo, go, to = no.oracle_ngram_ctc(e, W, tg, blank)
        assert util.close(l64, lo, rtol=1e-5, atol=1e-4)
        assert np.abs(g64 - go).max(initial=0) < 1e-5
        assert np.abs(t64 - to).max() < 1e-4


def test_symbol_declared_and_exported():
    from gtn_b200 import capi
    names = [s[0] for s in capi.SYMBOLS]
    assert "gtnb_ngram_ctc_loss" in names
    header = open(os.path.join(HERE, "..", "include", "gtn_b200.h")).read()
    assert "int gtnb_ngram_ctc_loss(" in header
    so = capi.LIB_PATH
    if not os.path.exists(so):
        pytest.skip("the library is not built")
    import ctypes
    assert hasattr(ctypes.CDLL(so), "gtnb_ngram_ctc_loss")
