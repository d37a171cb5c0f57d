"""k_implicit.cu's arc-label instantiations (gtnb_graph_loss) run from their source through the SIMT emulator
(tests/emu/graph_emu.cpp), against the live reference (oracle/_ref): forwardScore(compose(A_b, E_b)), its emission
gradient and its arc-weight gradient, utterance by utterance on its own T_b rows."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_build
from tests import graph_oracle as go
from tests import util

_f32p = C.POINTER(C.c_float)
_i32p = C.POINTER(C.c_int32)
_i64p = C.POINTER(C.c_int64)
_u8p = C.POINTER(C.c_uint8)


@pytest.fixture(scope="module")
def ref(oracle):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref/libgtn_ref.so is missing (built by `make -C oracle ref` where the reference is)")
    oracle.libref()
    return oracle


@pytest.fixture(scope="module")
def lib():
    L = C.CDLL(emu_build.build("graph", ["k_implicit.cu"]))
    L.emu_graph_arc.restype = C.c_int
    return L


@pytest.fixture(scope="module")
def lib_node():
    L = C.CDLL(emu_build.build("implicit", ["k_ctc.cu", "k_implicit.cu"]))
    L.emu_implicit_general.restype = C.c_int
    return L


def _p(a, t):
    return a.ctypes.data_as(t)


def _pack(graphs, C_):
    flags, ptr, src, lab, arc, w, nn, base = [], [], [], [], [], [], [], []
    off = 0
    for g in graphs:
        p, s, l, a, ww = go.tables(g, C_)
        flags.append(g["flags"]), ptr.append(p), src.append(s), lab.append(l), arc.append(a), w.append(ww)
        nn.append(len(g["flags"]))
        base.append(off)
        off += len(g["src"])
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0), dt)  # noqa: E731
    return (np.asarray(nn, np.int32), cat(flags, np.uint8), cat(ptr, np.int32), cat(src, np.int32),
            cat(lab, np.int32), cat(arc, np.int32), cat(w, np.float32), np.asarray(base, np.int64), off)


def run_arc(lib, e, graphs, lens, force_narrow=False):
    """-> (scores [B], grads [B,T,C], arc_grads [sum A_b], status [B], lanes) with deltas = +1"""
    B, T, C_ = e.shape
    nn, fl, ptr, src, lab, arc, w, base, n_arcs = _pack(graphs, C_)
    lens = np.ascontiguousarray(lens, np.int32)
    e = np.ascontiguousarray(e, np.float32)
    out, st = np.zeros(B, np.float32), np.zeros(B, np.int32)
    grad, ag = np.zeros_like(e), np.zeros(max(n_arcs, 1), np.float32)
    deltas = np.ones(B, np.float32)
    G = lib.emu_graph_arc(B, T, C_, _p(e, _f32p), _p(lens, _i32p), _p(nn, _i32p), _p(fl, _u8p), _p(ptr, _i32p),
                          _p(src, _i32p), _p(lab, _i32p), _p(arc, _i32p), _p(w, _f32p), _p(base, _i64p),
                          _p(deltas, _f32p), int(force_narrow), _p(out, _f32p), _p(grad, _f32p), _p(ag, _f32p),
                          _p(st, _i32p))
    emu_build.check(0 if G >= 0 else -G)
    return out, grad, ag[:n_arcs], st, G


def ref_numerator(e, graphs, lens):
    """forwardScore(compose(A_b, E_b)) and its gradients from the reference, utterance by utterance"""
    from oracle import pyoracle as po
    B, T, C_ = e.shape
    scores, grads, ags = np.zeros(B, np.float32), np.zeros_like(e), []
    for b, g in enumerate(graphs):
        Tb = int(lens[b])
        E = po.RefGraph.linear(Tb, C_, e[b, :Tb].ravel())
        A = go.ref_graph(g)
        s = po.ref_op("forward_score", po.ref_op("compose", A, E))
        po.ref_backward(s)
        scores[b] = s.item()
        if Tb:
            grads[b, :Tb] = E.grad().weights().reshape(Tb, C_)
        ags.append(A.grad().weights() if len(g["src"]) else np.zeros(0, np.float32))
    return scores, grads, np.concatenate(ags)


def check(lib, e, graphs, lens, force_narrow=False, expect_lanes=None):
    s, g, ag, st, G = run_arc(lib, e, graphs, lens, force_narrow)
    assert not st.any()
    rs, rg, rag = ref_numerator(e, graphs, lens)
    live = np.asarray(lens) > 0  # T_b = 0: the criterion's NaN; the kernels write no gradient
    assert util.close(s[live], rs[live]), (s, rs)
    mag = float(np.max(np.abs(rs[live & np.isfinite(rs)]), initial=1.0))
    assert util.grad_close(g, rg, mag), float(np.abs(g - rg).max())
    assert util.grad_close(ag, rag, mag), float(np.abs(ag - rag).max())
    assert not g[~live].any()
    if expect_lanes is not None:
        assert (G > 0) == expect_lanes, G
    return s, g, ag


def emissions(B, T, C_, seed):
    return np.random.default_rng(seed).uniform(-3, 3, (B, T, C_)).astype(np.float32)


def test_ctc_graphs_match_reference_and_node_labelled_mode(ref, lib, lib_node):
    B, T, C_ = 3, 24, 10
    rng = np.random.default_rng(1)
    graphs = [go.ctc_graph(rng.integers(1, C_, U), 0, w=None) for U in (4, 7, 1)]
    for g in graphs:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    e, lens = emissions(B, T, C_, 2), [24, 17, 9]
    s, g, ag = check(lib, e, graphs, lens)
    # the node-labelled instantiations on the same tables
    nn, fl, ptr, src, lab, arc, w, base, n_arcs = _pack(graphs, C_)
    ln = np.ascontiguousarray(lens, np.int32)
    out, st = np.zeros(B, np.float32), np.zeros(B, np.int32)
    grad, gg = np.zeros_like(e), np.zeros(n_arcs, np.float32)
    deltas = np.ones(B, np.float32)
    rc = lib_node.emu_implicit_general(
        B, T, C_, _p(e, _f32p), _p(ln, _i32p), _p(nn, _i32p), _p(fl, _u8p), _p(ptr, _i32p), _p(src, _i32p),
        _p(lab, _i32p), _p(arc, _i32p), _p(w, _f32p), _p(deltas, _f32p), _p(out, _f32p), _p(grad, _f32p),
        _p(gg, _f32p), _p(st, _i32p))
    emu_build.check(0 if rc >= 0 else -rc)
    assert util.close(s, out)
    assert util.grad_close(g, grad, float(np.abs(out).max()))
    assert util.grad_close(ag, gg, float(np.abs(out).max()))


def _small_inventory():
    return [(i,) for i in range(6)] + [(0, 1), (1, 2), (2, 3), (3, 4, 5), (0, 0), (5, 1, 2)]


def test_word_decomposition_graphs(ref, lib):
    pieces = _small_inventory()
    C_ = len(pieces) + 1
    rng = np.random.default_rng(3)
    graphs = []
    for U in (7, 5):
        letters = [int(x) for x in rng.integers(0, 6, U)]
        g = go.from_ref(go.decomposition_graph(go.REF_OPS, letters, pieces))
        g["w"] = rng.uniform(-0.5, 0.5, len(g["src"])).astype(np.float32)
        graphs.append(g)
    e = emissions(2, 16, C_, 4)
    check(lib, e, graphs, [16, 12])


def test_wildcard_graphs_are_not_label_uniform(ref, lib):
    C_ = 9
    rng = np.random.default_rng(5)
    graphs = [go.with_wildcards(go.ctc_graph(rng.integers(1, C_, U)), C_, w_loop=-0.3) for U in (3, 2)]
    for g in graphs:
        assert go.non_uniform_nodes(g, C_) >= 2
    e = emissions(2, 20, C_, 6)
    check(lib, e, graphs, [20, 13], expect_lanes=True)
    check(lib, e, graphs, [20, 13], force_narrow=True)


def test_random_graphs_cycles_hubs_and_many_nodes(ref, lib):
    C_ = 7
    rng = np.random.default_rng(7)
    hub = go.random_graph(rng, 12, 40, C_, n_start=3, n_accept=2)
    # a node with more in-arcs than a wide lane holds (kWideCap = 20), self-loops among them
    extra = 30
    hub = go.make(hub["flags"], np.concatenate([hub["src"], rng.integers(0, 12, extra)]),
                  np.concatenate([hub["dst"], np.full(extra, 5)]), np.concatenate([hub["ilabel"], rng.integers(0, C_, extra)]),
                  w=np.concatenate([hub["w"], rng.uniform(-1, 1, extra)]))
    big = go.random_graph(rng, 300, 700, C_, n_start=4, n_accept=5)  # more nodes than threads
    e = emissions(2, 9, C_, 8)
    check(lib, e, [hub, big], [9, 8])
    check(lib, e[:1], [hub], [9], expect_lanes=True)


def test_labels_outside_the_alphabet_never_match(ref, lib):
    C_ = 5
    rng = np.random.default_rng(9)
    g = go.random_graph(rng, 8, 30, C_, label_hi=C_ + 3)
    assert (g["olabel"] >= C_).any()
    e = emissions(1, 7, C_, 10)
    _, _, ag = check(lib, e, [g], [7])
    assert not ag[g["olabel"] >= C_].any()


def test_edge_lengths_infeasible_and_empty_graphs(ref, lib):
    C_ = 6
    chain = go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3])  # accepts only length 3
    wild = go.with_wildcards(go.ctc_graph([2, 3]), C_)
    empty = go.make([], [], [], [])
    e = emissions(4, 6, C_, 12)
    s, g, ag, st, _ = run_arc(lib, e, [wild, wild, chain, empty], [0, 1, 5, 6])
    assert not st.any()
    assert np.isneginf(s[2]) and np.isneginf(s[3])  # no accepting path of T_b arcs / no graph at all
    Aw = len(wild["src"])
    assert not g[[0, 2, 3]].any() and not ag[:Aw].any() and not ag[2 * Aw:].any()
    check(lib, e[:2], [wild, chain], [1, 3])


def test_alphabet_above_256(ref, lib):
    C_ = 300
    rng = np.random.default_rng(13)
    g = go.with_wildcards(go.ctc_graph(rng.integers(1, C_, 3)), C_, w_loop=-0.1)
    e = emissions(1, 6, C_, 14)
    check(lib, e, [g], [6], force_narrow=True)
    check(lib, e, [g], [6])


def test_non_finite_emission_raises_the_status_bit(lib):
    C_ = 5
    g = go.with_wildcards(go.ctc_graph([1, 2]), C_)
    e = emissions(1, 6, C_, 15)
    e[0, 3, 4] = np.inf
    _, _, _, st, _ = run_arc(lib, e, [g], [6])
    assert st[0] != 0
