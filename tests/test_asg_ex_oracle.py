"""CPU checks of the test infrastructure for gtnb_asg_loss_ex (tests/asg_oracle.py): the committed golden fixture
(tests/golden/asg_ex_golden.npz, from the live reference) against the C oracle; the oracle and the float64 referee
against the live reference on random padded cases; and the new C-ABI symbol."""
import os

import numpy as np
import pytest

from tests import asg_oracle as ao
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
    return (np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isposinf(a), np.isposinf(b))
            and np.allclose(a, b, rtol=rtol, atol=atol, equal_nan=True))


@pytest.mark.parametrize("name", ["a", "b"])
def test_golden_matches_oracle(oracle, name):
    g = np.load(os.path.join(HERE, "golden", "asg_ex_golden.npz"))
    e, tw, lens = g[name + "_e"], g[name + "_tw"], g[name + "_lens"]
    targets = _split(g[name + "_targets"], g[name + "_target_lens"])
    lo, go, to = ao.oracle_asg_batch(e, tw, targets, lens)
    assert _same(lo, g[name + "_losses"])
    assert _same(go, g[name + "_grads"])
    assert _same(to, g[name + "_trans_grad"], atol=1e-4)
    l64, g64, t64 = ao.asg_f64_batch(e, tw, targets, lens)
    assert _same(l64, g[name + "_losses"], atol=1e-4)
    assert np.abs(g64 - g[name + "_grads"]).max() < 1e-5 and np.abs(t64 - g[name + "_trans_grad"]).max() < 1e-4


def _random_case(rng, C):
    B, T = 4, int(rng.integers(1, 12))
    targets = [[int(x) for x in rng.integers(0, C, int(rng.integers(0, 6)))] for _ in range(B)]
    lens = rng.integers(0, T + 1, B).astype(np.int32)
    e = rng.uniform(-5, 5, (B, T, C)).astype(np.float32)
    tw = rng.uniform(-3, 3, C + C * C).astype(np.float32)
    return e, tw, targets, lens


@pytest.mark.parametrize("C", [4, 8, 28])
def test_oracle_and_f64_match_live_reference(oracle, C):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref/libgtn_ref.so is not built")
    rng = np.random.default_rng(C + 50)
    for _ in range(4):
        e, tw, targets, lens = _random_case(rng, C)
        lr, gr, tr = ao.ref_asg_batch(e, tw, targets, lens)
        lo, go, to = ao.oracle_asg_batch(e, tw, targets, lens)
        l64, g64, t64 = ao.asg_f64_batch(e, tw, targets, lens)
        assert _same(lo, lr) and _same(go, gr) and _same(to, tr, atol=1e-4), (lens, targets)
        assert _same(l64, lr, atol=1e-4), (l64, lr)
        assert np.abs(g64 - gr).max() < 1e-5 and np.abs(t64 - tr).max() < 1e-4


def test_f64_referee_edge_cases():
    rng = np.random.default_rng(3)
    e = rng.uniform(-3, 3, (4, 5)).astype(np.float32)
    tw = rng.uniform(-2, 2, 5 + 25).astype(np.float32)
    l, g, t = ao.asg_f64(e[:0], tw, [1, 2])
    assert np.isnan(l) and g.shape == (0, 5) and not t.any()
    l, g, t = ao.asg_f64(e, tw, [])
    assert np.isposinf(l) and util.close(g.sum(), 4.0) and util.close(t.sum(), 4.0)  # one path posterior per frame
    l, g, t = ao.asg_f64(e, tw, [1, 2, 3, 4, 0])
    assert np.isposinf(l) and util.close(g.sum(), 4.0)


def test_symbol_declared_and_exported():
    from gtn_b200 import capi
    assert "gtnb_asg_loss_ex" in [s[0] for s in capi.SYMBOLS]
    header = open(os.path.join(HERE, "..", "include", "gtn_b200.h")).read()
    assert "int gtnb_asg_loss_ex(" in header
    so = capi.LIB_PATH
    if not os.path.exists(so):
        pytest.skip("the library is not built")
    import ctypes
    assert hasattr(ctypes.CDLL(so), "gtnb_asg_loss_ex")
