"""CPU checks for gtnb_graph_loss's test infrastructure: the committed golden fixture
(tests/golden/graph_loss_golden.npz, tests/golden/make_graph_loss_golden.py) against the live reference through
tests/graph_oracle.py and against the arc-label kernels' emulation, and the C-ABI symbol."""
import ctypes
import os

import numpy as np
import pytest

from tests import graph_oracle as go
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "graph_loss_golden.npz")


def graphs_of(z, name):
    out, n0, a0 = [], 0, 0
    for n, a in zip(z[name + "_n_nodes"], z[name + "_n_arcs"]):
        g = {"flags": z[name + "_flags"][n0:n0 + n]}
        for k in ("src", "dst", "ilabel", "olabel", "w"):
            g[k] = z[name + "_" + k][a0:a0 + a]
        out.append(g)
        n0, a0 = n0 + n, a0 + a
    return out


@pytest.mark.parametrize("name", ["a", "b"])
def test_golden_matches_live_reference(oracle, name):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref/libgtn_ref.so is missing")
    z = np.load(GOLDEN)
    lo, gr, ag = go.ref_graph_loss(z[name + "_e"], graphs_of(z, name), z[name + "_lens"])
    assert util.close(lo, z[name + "_losses"])
    assert np.array_equal(gr, z[name + "_grads"]) and np.array_equal(ag, z[name + "_arc_grads"])


def test_golden_cases_are_what_the_docstring_says():
    z = np.load(GOLDEN)
    C = {"a": 7, "b": 12}
    a, b = graphs_of(z, "a"), graphs_of(z, "b")
    assert go.non_uniform_nodes(a[1], C["a"]) > 0 and go.non_uniform_nodes(b[1], C["b"]) > 0
    assert (a[2]["olabel"] >= C["a"]).any()
    assert np.isnan(z["b_losses"][2]) and np.isposinf(z["b_losses"][3]) and np.isposinf(z["a_losses"][3])
    assert not z["b_grads"][2].any()


@pytest.mark.parametrize("name", ["a", "b"])
def test_golden_matches_the_arc_label_kernels(name):
    """numerator score and gradients of the emulated kernels = the fixture's, with the normaliser in float64"""
    from tests import emu_build
    from tests import test_graph_loss_emulation as te
    lib = ctypes.CDLL(emu_build.build("graph", ["k_implicit.cu"]))
    lib.emu_graph_arc.restype = ctypes.c_int
    z = np.load(GOLDEN)
    e, lens, graphs = z[name + "_e"], z[name + "_lens"], graphs_of(z, name)
    s, g, ag, st, _ = te.run_arc(lib, e, graphs, lens)
    assert not st.any()
    B, T, C = e.shape
    den, dg = np.zeros(B), np.zeros((B, T, C))
    for b in range(B):
        x = e[b, :lens[b]].astype(np.float64)
        m = x.max(1, keepdims=True)
        den[b] = np.sum(np.log(np.exp(x - m).sum(1)) + m[:, 0])
        dg[b, :lens[b]] = np.exp(x - m) / np.exp(x - m).sum(1, keepdims=True)
    live = lens > 0
    assert util.close((den - s)[live], z[name + "_losses"][live])
    assert util.grad_close((dg - g)[live], z[name + "_grads"][live], 50.0)
    assert util.grad_close(-ag, z[name + "_arc_grads"], 50.0)


def test_symbol_declared_and_exported():
    from gtn_b200 import capi
    assert "gtnb_graph_loss" in [s[0] for s in capi.SYMBOLS]
    with open(os.path.join(ROOT, "include", "gtn_b200.h")) as f:
        assert "int gtnb_graph_loss(" in f.read()
    so = os.path.join(ROOT, "gtn_b200", "lib", "libgtn_b200.so")
    if not os.path.exists(so):
        pytest.skip("the library is not built")
    assert hasattr(ctypes.CDLL(so), "gtnb_graph_loss")
