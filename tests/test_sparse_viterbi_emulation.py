"""k_sparse.cu's decoder kernels (the tropical sweep and traceback of gtnb_viterbi_sparse, and sparse_tau of
gtnb_sparse_transitions_viterbi) run from their source through the SIMT emulator (tests/emu/sparse_viterbi_emu.cpp)
against the float32 restatement of tests/sparse_viterbi_oracle.py: scores bit-equal; paths and G's arcs == wherever
the tie bit is not raised; the tie bit raised exactly where the restatement finds a tie on the traced path; the
non-finite bit exactly for NaN / +inf in a used weight or emission, and not for -inf.  Ragged T_b with 0 and 1, NaN
padding rows, C not a multiple of 4, labels >= C, unreachable nodes, the trigram, lanes 1 ... 32, G at the envelope's
edge, tie-heavy integer inputs; tau against numpy with NaN in every lane position and all -inf groups."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_build
from tests import graph_oracle as go
from tests import sparse_trans_oracle as st
from tests import sparse_viterbi_oracle as sv
from tests.test_sparse_trans_oracle import _p, graph_args, start_groups

f32p, i32p, u8p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)


def load():
    """tests/emu/sparse_viterbi_emu.cpp built and declared"""
    lib = C.CDLL(emu_build.build("sparse_viterbi", ["k_sparse.cu", "gtnb_product.h"]))
    lib.emu_sparse_viterbi.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, C.c_int, C.c_int, u8p, i32p, i32p, i32p,
                                       f32p, C.c_int, i32p, i32p, f32p, i32p]
    lib.emu_sparse_tau.argtypes = [C.c_int, C.c_int, u8p, i32p, i32p, i32p, C.c_int, f32p, f32p,
                                   C.POINTER(C.c_int)]
    return lib


@pytest.fixture(scope="module")
def emu():
    return load()


def run(emu, e, lens, G, w, lanes=0):
    B, T, Cn = e.shape
    _, ga = graph_args(G)
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    w = np.ascontiguousarray(w, np.float32)
    paths = np.full((B, T), -7, np.int32)
    arcs = np.full((B, T), -7, np.int32)
    scores = np.full(B, np.nan, np.float32)
    status = np.zeros(B, np.int32)
    rc = emu.emu_sparse_viterbi(B, T, Cn, _p(e, f32p), _p(lens, i32p), len(G["flags"]), len(G["src"]), *ga,
                                _p(w, f32p), lanes, _p(paths, i32p), _p(arcs, i32p), _p(scores, f32p),
                                _p(status, i32p))
    emu_build.check(rc)
    return paths, arcs, scores, status


def check(emu, e, lens, G, w, lanes=0):
    """the kernels against the restatement; -> the number of utterances whose trace met a tie"""
    paths, arcs, scores, status = run(emu, e, lens, G, w, lanes)
    Cn = e.shape[2]
    assert not (status & 1).any()
    n_ties = 0
    for b in range(e.shape[0]):
        n = int(lens[b])
        score, tie, labels, path_arcs = sv.decode_outcome(e[b, :n], G, w, Cn)
        assert np.array_equal(scores[b], score), (b, scores[b], score)
        assert bool(status[b] & 2) == tie, (b, status[b], tie)
        n_ties += tie
        if not np.isfinite(score):
            assert (paths[b] == -1).all() and (arcs[b] == -1).all()
            continue
        assert (paths[b, n:] == -1).all() and (arcs[b, n:] == -1).all()
        assert sv.is_path(G, arcs[b, :n]) and np.array_equal(paths[b, :n], G["olabel"][arcs[b, :n]])
        assert sv.path_value(e[b, :n], G, w, arcs[b, :n]) == score
        if not tie:
            assert np.array_equal(paths[b, :n], labels) and np.array_equal(arcs[b, :n], path_arcs)
    return n_ties


def test_random_sparse_graph_ragged(emu):
    """several start and accept nodes, unreachable nodes, labels >= C, C = 7, T_b in {0, 1}, NaN padding"""
    rng = np.random.default_rng(1)
    Cn, T = 7, 9
    G = st.sparse_graph(rng, 10, 45, Cn, label_hi=9)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = rng.uniform(-3, 3, (5, T, Cn)).astype(np.float32)
    lens = np.asarray([9, 0, 1, 6, 9], np.int32)
    e[3, 6:] = np.nan
    assert check(emu, e, lens, G, w) == 0


def test_trigram(emu):
    rng = np.random.default_rng(2)
    Cn, T = 5, 12
    G = st.trigram_graph(Cn)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = rng.uniform(-3, 3, (2, T, Cn)).astype(np.float32)
    check(emu, e, np.asarray([12, 7], np.int32), G, w)


@pytest.mark.parametrize("lanes", [1, 2, 4, 8, 16, 32])
def test_every_lane_count(emu, lanes):
    """the per-node argmax merged over 1 ... 32 lanes: nodes with up to 40 in-arcs"""
    rng = np.random.default_rng(3)
    Cn, T = 6, 7
    G = st.sparse_graph(rng, 6, 200, Cn, n_unreachable=0)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = rng.uniform(-3, 3, (3, T, Cn)).astype(np.float32)
    check(emu, e, np.asarray([7, 4, 1], np.int32), G, w, lanes)


def test_envelope_edge(emu):
    """4096 nodes, 32768 arcs; one node more is outside the envelope"""
    rng = np.random.default_rng(4)
    Cn, T, S, A = 64, 3, 4096, 32768
    G = st.sparse_graph(rng, S, A, Cn, n_start=64, n_accept=512, n_unreachable=0)
    w = rng.uniform(-1, 1, A).astype(np.float32)
    e = rng.uniform(-3, 3, (1, T, Cn)).astype(np.float32)
    check(emu, e, np.asarray([T], np.int32), G, w)
    G2 = st.sparse_graph(rng, S + 1, 8, Cn, n_unreachable=0)
    _, ga = graph_args(G2)
    out = np.zeros(64, np.int32)
    rc = emu.emu_sparse_viterbi(1, T, Cn, _p(e, f32p), _p(np.asarray([T], np.int32), i32p), S + 1, 8, *ga,
                                _p(np.zeros(8, np.float32), f32p), 0, _p(out, i32p), _p(out, i32p),
                                _p(np.zeros(4, np.float32), f32p), _p(out, i32p))
    assert rc == 1


@pytest.mark.parametrize("graph", ["trigram", "sparse"])
def test_tie_heavy_integer_inputs(emu, graph):
    """zero weights and 0 / 1 emissions: the tie bit exactly where the restatement meets a tie on the traced path"""
    rng = np.random.default_rng(5)
    Cn, T = 4, 6
    G = st.trigram_graph(Cn) if graph == "trigram" else st.sparse_graph(rng, 8, 40, Cn)
    w = np.zeros(len(G["src"]), np.float32)
    if graph == "sparse":
        w[:] = rng.integers(-1, 2, len(w))
    e = rng.integers(0, 2, (6, T, Cn)).astype(np.float32)
    assert check(emu, e, np.asarray([6, 5, 6, 1, 3, 6], np.int32), G, w) > 0


def test_neginf_forbids_without_the_status_bit(emu):
    rng = np.random.default_rng(6)
    Cn, T = 5, 8
    G = st.sparse_graph(rng, 9, 50, Cn)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    w[::3] = -np.inf
    e = rng.uniform(-3, 3, (3, T, Cn)).astype(np.float32)
    e[1, 2, 0] = -np.inf
    check(emu, e, np.asarray([8, 8, 5], np.int32), G, w)


@pytest.mark.parametrize("value", [np.nan, np.inf])
def test_nan_and_inf_raise_the_status_bit(emu, value):
    rng = np.random.default_rng(7)
    Cn, T = 4, 5
    G = st.trigram_graph(Cn)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = rng.uniform(-3, 3, (3, T, Cn)).astype(np.float32)
    e[1, 2, 3] = value  # a used emission
    e[2, 4:] = value  # padding beyond T_b: unused
    lens = np.asarray([T, T, 4], np.int32)
    assert list(run(emu, e, lens, G, w)[3] & 1) == [0, 1, 0]
    w2 = w.copy()
    w2[11] = value
    assert (run(emu, np.nan_to_num(e, nan=0.0, posinf=0.0), lens, G, w2)[3] & 1).all()
    # an arc labelled outside [0, C) is never used
    G3 = go.make(G["flags"], np.r_[G["src"], 0], np.r_[G["dst"], 1], np.r_[G["olabel"], Cn + 3])
    w3 = np.r_[w, np.float32(value)].astype(np.float32)
    assert not (run(emu, np.nan_to_num(e, nan=0.0, posinf=0.0), lens, G3, w3)[3] & 1).any()


def tau(emu, G, w, Cn):
    _, ga = graph_args(G)
    w = np.ascontiguousarray(w, np.float32)
    out = np.full(len(G["src"]) + 1, 7.0, np.float32)
    K = C.c_int()
    emu_build.check(emu.emu_sparse_tau(len(G["flags"]), len(G["src"]), *ga, Cn, _p(w, f32p), _p(out, f32p),
                                       C.byref(K)))
    return out[:K.value]


def test_tau_matches_numpy(emu):
    rng = np.random.default_rng(8)
    Cn = 6
    G = st.sparse_graph(rng, 9, 300, Cn, n_start=5, label_hi=8)
    w = rng.uniform(-4, 4, len(G["src"])).astype(np.float32)
    groups = start_groups(G, Cn)
    assert max(len(m) for m in groups) > 1
    assert np.array_equal(tau(emu, G, w, Cn), np.asarray([w[m].max() for m in groups], np.float32))
    w[groups[0]] = -np.inf  # an all -inf group stays -inf
    assert tau(emu, G, w, Cn)[0] == -np.inf


def test_tau_keeps_nan_in_every_lane_position(emu):
    Cn = 3
    n = 40  # one start group of 40 arcs: positions 0 ... 39 cover every lane, some lanes twice
    G = go.make([1, 2], np.zeros(n, np.int32), np.ones(n, np.int32), np.full(n, 2, np.int32))
    w = np.random.default_rng(9).uniform(-1, 1, n).astype(np.float32)
    for j in range(n):
        wj = w.copy()
        wj[j] = np.nan
        assert np.isnan(tau(emu, G, wj, Cn)).all(), j
