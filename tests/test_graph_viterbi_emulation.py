"""gtnb_graph_viterbi's device route -- k_implicit.cu's tropical forward instantiations and implicit_trace_kernel --
run from their source through the SIMT emulator (tests/emu/graph_viterbi_emu.cpp), against the live reference
(oracle/_ref, tests/graph_viterbi_oracle.py): every forward variant (the fast one-node-per-thread path, several nodes
per thread, the wide kernels with G = 1 .. 32 lanes per node, the arc-label instantiations); scores bit-equal to the
reference's; paths and arcs == wherever the tie bit is not raised, and the tie bit raised exactly where the traced
path meets a tie; the non-finite bit on NaN / inf emissions and weights."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_build
from tests import graph_oracle as go
from tests import graph_viterbi_oracle as gv
from tests.test_graph_loss_emulation import _pack

_f32p = C.POINTER(C.c_float)
_i32p = C.POINTER(C.c_int32)
_u8p = C.POINTER(C.c_uint8)


@pytest.fixture(scope="module")
def ref(oracle):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref/libgtn_ref.so is missing (built by `make -C oracle ref` where the reference is)")
    oracle.libref()
    return oracle


@pytest.fixture(scope="module")
def lib():
    L = C.CDLL(emu_build.build("graph_viterbi", ["k_implicit.cu"]))
    L.emu_graph_viterbi.restype = C.c_int
    return L


def _p(a, t):
    return a.ctypes.data_as(t)


def run(lib, e, graphs, lens, arc, lanes=-1, frames=0):
    """-> (paths [B,T], scores [B], arcs [B,T], status [B], lanes of the forward)"""
    B, T, C_ = e.shape
    nn, fl, ptr, src, lab, ids, w, _, _ = _pack(graphs, C_)
    lens = np.ascontiguousarray(lens, np.int32)
    e = np.ascontiguousarray(e, np.float32)
    paths, arcs = np.full((B, max(T, 1)), -7, np.int32), np.full((B, max(T, 1)), -7, np.int32)
    scores, st = np.full(B, np.nan, np.float32), np.zeros(B, np.int32)
    G = lib.emu_graph_viterbi(B, T, C_, _p(e, _f32p), _p(lens, _i32p), _p(nn, _i32p), _p(fl, _u8p), _p(ptr, _i32p),
                              _p(src, _i32p), _p(lab, _i32p), _p(ids, _i32p), _p(w, _f32p), int(arc), int(lanes),
                              int(frames), _p(paths, _i32p), _p(arcs, _i32p), _p(scores, _f32p), _p(st, _i32p))
    emu_build.check(0 if G >= 0 else -G)
    return paths[:, :T], scores, arcs[:, :T], st, G


def check(lib, e, graphs, lens, arc, lanes=-1, frames=0, expect_ties=None):
    p, s, a, st, G = run(lib, e, graphs, lens, arc, lanes, frames)
    pr, sr, ar = gv.ref_graph_viterbi(e, graphs, lens)
    assert not (st & 1).any(), st
    assert np.array_equal(s.view(np.int32), sr.view(np.int32)), (s, sr)
    C_ = e.shape[2]
    for b, g in enumerate(graphs):
        Tb = int(lens[b])
        assert (p[b, Tb:] == -1).all() and (a[b, Tb:] == -1).all()
        tie = gv.trace_ties(e[b, :Tb], g, C_, a[b, :Tb])
        assert bool(st[b] & 2) == tie, (b, st[b], tie)
        if not tie:
            assert np.array_equal(p[b], pr[b]) and np.array_equal(a[b], ar[b]), b
        else:  # one of the optimal paths, the reference's own choice left to the exact route
            assert gv.path_score(e[b], g, a[b, :Tb]).tobytes() == s[b].tobytes()
            assert np.array_equal(g["olabel"][a[b, :Tb]], p[b, :Tb])
    if expect_ties is not None:
        assert bool((st & 2).any()) == expect_ties, st
    return G


def emissions(B, T, C_, seed, ties=False):
    rng = np.random.default_rng(seed)
    return (rng.integers(0, 2, (B, T, C_)) if ties else rng.uniform(-3, 3, (B, T, C_))).astype(np.float32)


def ctc_batch(C_, seed, ties=False):
    rng = np.random.default_rng(seed)
    graphs = [go.ctc_graph(rng.integers(1, C_, U)) for U in (4, 7, 1, 3)]
    for g in graphs:
        g["w"] = (rng.integers(-1, 1, len(g["src"])) if ties else rng.uniform(-1, 1, len(g["src"]))).astype(np.float32)
    return graphs, emissions(4, 20, C_, seed + 1, ties), np.asarray([20, 13, 1, 0], np.int32)


@pytest.mark.parametrize("ties", [False, True])
def test_fast_path_ctc_graphs(ref, lib, ties):
    """CTC graphs (in-degree <= 3, label-uniform): one node per thread; T_b in {0, 1}; frames staged 3 at a time"""
    graphs, e, lens = ctc_batch(8, 1 + ties, ties)
    assert check(lib, e, graphs, lens, arc=False, lanes=0, frames=3, expect_ties=True if ties else None) == 0


def test_several_nodes_per_thread(ref, lib):
    """more nodes than threads, in-degree > 3 at some node: the general path of the same kernel"""
    C_ = 7
    rng = np.random.default_rng(3)
    big = go.ctc_graph(rng.integers(1, C_, 140))  # 281 nodes
    big["w"] = rng.uniform(-1, 1, len(big["src"])).astype(np.float32)
    hub = go.ctc_graph([1, 2, 3])
    hub = go.make(hub["flags"], np.concatenate([hub["src"], [0, 1, 2, 3]]), np.concatenate([hub["dst"], [4] * 4]),
                  np.concatenate([hub["ilabel"], [0] * 4]), w=rng.uniform(-1, 1, len(hub["src"]) + 4))  # 4: a blank
    e = emissions(2, 12, C_, 4)
    check(lib, e, [big, hub], np.asarray([12, 9], np.int32), arc=False, lanes=0, frames=5)


@pytest.mark.parametrize("G", [1, 2, 4, 8, 16, 32])
def test_wide_kernels(ref, lib, G):
    """label-uniform nodes with many in-arcs (every node into the hub), each lane count"""
    C_ = 6
    rng = np.random.default_rng(10 + G)
    N = 16  # the hub's N + 1 in-arcs fit one lane's kWideCap = 20 registers at G = 1
    src = list(range(N)) + list(range(N - 1))
    dst = [N - 1] * N + list(range(1, N))
    lab = [3] * N + [int(x) for x in rng.integers(0, C_, N - 1)]
    # a node's in-arcs share the label of its first in-arc: label-uniform
    first = {}
    for a, d in enumerate(dst):
        lab[a] = first.setdefault(d, lab[a])
    flags = np.zeros(N, np.uint8)
    flags[0] |= 1
    flags[[N - 1, N - 2]] |= 2
    g = go.make(flags, src, dst, lab, w=rng.uniform(-1, 1, len(src)))
    e = emissions(1, 10, C_, 20 + G)
    check(lib, e, [g], np.asarray([10], np.int32), arc=False, lanes=G, frames=4)


@pytest.mark.parametrize("lanes", [-1, 0])
def test_arc_label_mode_wildcards_and_random_graphs(ref, lib, lanes):
    """not label-uniform: wildcard states (the wide arc-label kernels at lanes = -1) and random cyclic graphs with
    several start and accept nodes and labels >= C"""
    C_ = 9
    rng = np.random.default_rng(30)
    graphs = [go.with_wildcards(go.ctc_graph(rng.integers(1, C_, 3)), C_, w_loop=-0.3),
              go.random_graph(rng, 10, 40, C_, n_start=3, n_accept=3, label_hi=C_ + 2)]
    for g in graphs:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    e = emissions(2, 14, C_, 31)
    G = check(lib, e, graphs, np.asarray([14, 11], np.int32), arc=True, lanes=lanes, frames=4)
    assert (G > 0) == (lanes == -1)


def test_ties_raise_the_tie_bit(ref, lib):
    """parallel equal arcs tie on every frame; the untied utterance beside them raises nothing"""
    C_ = 4
    par = go.make([1, 2], [0, 0, 1, 1], [1, 1, 1, 1], [1, 1, 2, 2])
    rng = np.random.default_rng(40)
    plain = go.ctc_graph([1, 2])
    plain["w"] = rng.uniform(-1, 1, len(plain["src"])).astype(np.float32)
    e = emissions(2, 8, C_, 41)
    for lanes in (0, -1):  # (node 1's in-arcs carry labels 1 and 2: the arc-label instantiations)
        p, s, a, st, _ = run(lib, e, [par, plain], [8, 8], arc=True, lanes=lanes)
        assert st[0] == 2 and st[1] == 0, st
        check(lib, e, [par, plain], np.asarray([8, 8], np.int32), arc=True, lanes=lanes)


@pytest.mark.parametrize("arc", [True, False])
@pytest.mark.parametrize("where", ["emission_nan", "emission_inf", "w_inf", "w_nan"])
def test_non_finite_values_raise_the_status_bit(lib, where, arc):
    """utterance 1 holds the non-finite value (an emission of a label its graph matches, or an arc weight), utterance
    0 none"""
    C_ = 5
    g = go.with_wildcards(go.ctc_graph([1, 2]), C_) if arc else go.ctc_graph([1, 2])
    h = go.ctc_graph([3, 4])
    e = emissions(2, 6, C_, 50)
    if where == "emission_nan":
        e[1, 3, 4] = np.nan
    elif where == "emission_inf":
        e[1, 2, 3] = np.inf
    elif where == "w_inf":
        h["w"][2] = np.inf
    else:
        h["w"][1] = np.nan
    _, _, _, st, _ = run(lib, e, [g, h], [6, 6], arc=arc)
    assert st[1] & 1 and not st[0] & 1, st
