"""CPU checks for gtnb_graph_transitions_viterbi:
- the source of its two kernels through the SIMT emulator: tau_l = max_j W[l][j] against numpy for C in {1, 4, 29, 128},
  NaN propagating and all -inf rows kept; the map from traced product arcs to A_b's arcs;
- the device route end to end, every step from its source (the shipped builder's folded products, tau, the fold
  kernel, k_implicit.cu's tropical forward and traceback, the arc map), against the live reference: scores bit-equal,
  paths and arcs == wherever the tie bit is not raised, the tie bit raised exactly where the float32 restatement finds
  a tie on the traced path and the non-finite bit exactly where a weight or emission is not finite;
- the device route's graph against the live reference: the product the shipped builder (gtnb_product.h) makes, with
  BIGRAM's folded start arcs weighted by tau, swept in float32 by tests/graph_trans_viterbi_oracle.py's restatement,
  gives the reference's viterbiScore bit for bit (the tau argument of DESIGN.md), and a path's value in the device
  route's association equals that score;
- the C-ABI symbol is declared and exported."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import emu_build
from tests import graph_oracle as go
from tests import graph_trans_viterbi_oracle as gtv
from tests.test_graph_trans_oracle import build_product, need_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32p, i32p, i64p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_longlong)


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("graph_trans_viterbi", ["k_ngram.cu", "k_implicit.cu"]))
    lib.emu_ngram_tau.argtypes = [C.c_int, f32p, f32p]
    lib.emu_product_arc_map.argtypes = [C.c_int, C.c_int, i64p, i32p, i32p]
    return lib


@pytest.fixture(scope="module")
def product_emu():
    lib = C.CDLL(emu_build.build("product", ["k_ngram.cu", "k_implicit.cu", "gtnb_product.h"]))
    u8p = C.POINTER(C.c_uint8)
    lib.emu_build_product.argtypes = [C.c_int, C.c_int, u8p, i32p, i32p, i32p, f32p, C.c_int, C.c_int, C.c_int, f32p,
                                      i32p, i32p, u8p, i32p, i32p, i32p, i32p, i32p, f32p]
    return lib


def _p(a, t):
    return a.ctypes.data_as(t)


@pytest.mark.parametrize("C_", [1, 4, 29, 128])
def test_tau_matches_numpy(emu, C_):
    rng = np.random.default_rng(C_)
    W = rng.uniform(-4, 4, (C_, C_)).astype(np.float32)
    if C_ > 1:
        W[0, C_ - 1] = np.nan  # NaN in the last lane's column: propagates through the warp reduction
        W[C_ - 1, :] = -np.inf  # a forbidden row stays -inf
        W[C_ // 2, 0] = np.inf
    tau = np.full(C_, 7.0, np.float32)
    emu_build.check(emu.emu_ngram_tau(C_, _p(W, f32p), _p(tau, f32p)))
    want = np.max(W, axis=1)  # np.max propagates NaN
    assert np.array_equal(tau, want, equal_nan=True), (tau, want)
    if C_ > 1:
        assert np.isnan(tau[0]) and np.isneginf(tau[C_ - 1]) and np.isposinf(tau[C_ // 2])


def test_tau_nan_in_every_position(emu):
    C_ = 40
    for j in range(C_):
        W = np.zeros((C_, C_), np.float32)
        W[3, j] = np.nan
        tau = np.zeros(C_, np.float32)
        emu_build.check(emu.emu_ngram_tau(C_, _p(W, f32p), _p(tau, f32p)))
        assert np.isnan(tau[3]) and not np.isnan(np.delete(tau, 3)).any(), j


def test_arc_map(emu):
    rng = np.random.default_rng(2)
    B, T = 5, 37
    n_prod = rng.integers(0, 60, B)
    n_a = rng.integers(1, 20, B)
    off = np.zeros(2 * B, np.int64)
    off[1:B] = np.cumsum(n_prod)[:-1]
    off[B + 1:] = np.cumsum(n_a)[:-1]
    arc_of = np.concatenate([off[B + b] + rng.integers(0, n_a[b], n_prod[b]) for b in range(B)]).astype(np.int32)
    arcs = np.full((B, T), -1, np.int32)
    for b in range(B):
        if n_prod[b]:
            k = int(rng.integers(0, T + 1))
            arcs[b, :k] = rng.integers(0, n_prod[b], k)
    want = arcs.copy()
    for b in range(B):
        ok = want[b] >= 0
        want[b, ok] = arc_of[off[b] + want[b, ok]] - off[B + b]
    emu_build.check(emu.emu_product_arc_map(B, T, _p(off, i64p), _p(arc_of, i32p), _p(arcs, i32p)))
    assert np.array_equal(arcs, want)


def _cases(rng, C_):
    yield go.random_graph(rng, 7, 24, C_, n_start=2, n_accept=2, label_hi=C_ + 2)
    yield go.with_wildcards(go.ctc_graph(rng.integers(1, C_, 2)), C_, w_loop=-0.2)
    yield go.ctc_graph(rng.integers(1, C_, 3))


@pytest.mark.parametrize("kind", [gtv.ASG, gtv.BIGRAM])
@pytest.mark.parametrize("C_", [3, 6])
def test_device_route_graph_gives_the_reference_score(oracle, product_emu, kind, C_):
    need_ref(oracle)
    rng = np.random.default_rng(10 * C_ + kind)
    n = 0
    for rep in range(4):
        for g in _cases(rng, C_):
            g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
            tw = rng.uniform(-1, 1, (C_ + C_ * C_) if kind == gtv.ASG else C_ * C_).astype(np.float32)
            T = int(rng.integers(1, 9))
            e = rng.uniform(-3, 3, (1, T, C_)).astype(np.float32)
            paths, scores, arcs = gtv.ref_graph_trans_viterbi(e, [g], kind, tw)
            # Wx of the shipped builder: [trans_w] for ASG, [W | tau] for BIGRAM
            Wx = tw if kind == gtv.ASG else np.concatenate([tw, tw.reshape(C_, C_).max(axis=1)]).astype(np.float32)
            p, _, _ = build_product(product_emu, g, C_, kind, True, Wx)
            s, _ = gtv.device_route_outcome(e[0], p, C_)
            r, _ = gtv.device_route_outcome(e[0], gtv.tropical_product(g, C_, kind, tw)[0], C_)
            assert s == scores[0] or (np.isneginf(s) and np.isneginf(scores[0])), (s, scores[0])
            assert r == s or (np.isneginf(r) and np.isneginf(s))
            if np.isfinite(scores[0]):
                n += 1
                assert gtv.path_value(e[0], g, kind, tw, paths[0], arcs[0]) == scores[0]
    assert n > 4


def test_symbol_declared_and_exported():
    from gtn_b200 import capi
    assert any(name == "gtnb_graph_transitions_viterbi" for name, _, _ in capi.SYMBOLS)
    with open(os.path.join(ROOT, "include", "gtn_b200.h")) as f:
        assert "int gtnb_graph_transitions_viterbi(" in f.read()


@pytest.fixture(scope="module")
def trace_lib():
    L = C.CDLL(emu_build.build("graph_viterbi", ["k_implicit.cu"]))
    L.emu_graph_viterbi.restype = C.c_int
    return L


def device_route(emu, product_emu, trace_lib, e, graphs, lens, kind, tw):
    """the device route, every step from its source: the shipped builder's folded products, ngram_tau_kernel (BIGRAM),
    product_fold_kernel for their weights, the tropical forward and implicit_trace_kernel (k_implicit.cu, through
    tests/emu/graph_viterbi_emu.cpp), then product_arc_map_kernel -> (paths, scores, arcs, status, products)"""
    from tests.test_graph_viterbi_emulation import run as run_trace
    B, T, C_ = e.shape
    tw = np.ascontiguousarray(tw, np.float32)
    tau = np.zeros(max(C_, 1), np.float32)
    if kind == gtv.BIGRAM:
        emu_build.check(emu.emu_ngram_tau(C_, _p(tw, f32p), _p(tau, f32p)))
    nW = C_ * C_ if kind == gtv.BIGRAM else C_ + C_ * C_
    Wx = np.concatenate([tw, tau[:C_]]) if kind == gtv.BIGRAM else tw
    prods, arc_of, tidx, w_A = [], [], [], []
    off = np.zeros(2 * B, np.int64)
    for b, g in enumerate(graphs):
        p, ao, ti = build_product(product_emu, g, C_, kind, True, Wx)
        if b + 1 < B:
            off[b + 1] = off[b] + len(ao)
            off[B + b + 1] = off[B + b] + len(g["src"])
        prods.append(p)
        arc_of.append(ao + off[B + b])
        tidx.append(ti)
        w_A.append(np.asarray(g["w"], np.float32))
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0), dt)  # noqa: E731
    arc_of, tidx, w_A = cat(arc_of, np.int32), cat(tidx, np.int32), cat(w_A, np.float32)
    fw = np.zeros(max(len(arc_of), 1), np.float32)
    emu_build.check(product_emu.emu_product_fold(len(arc_of), _p(w_A, f32p), _p(arc_of, i32p), _p(tw, f32p), nW,
                                                 _p(tau, f32p), _p(tidx, i32p), _p(fw, f32p)))
    for b, p in enumerate(prods):
        w = fw[off[b]:off[b] + len(p["src"])]
        assert w.tobytes() == p["w"].tobytes()  # the fold kernel gives the host builder's weights
        p["w"] = w.copy()
    paths, scores, parcs, st, _ = run_trace(trace_lib, e, prods, lens, arc=False)
    arcs = np.ascontiguousarray(parcs, np.int32)
    emu_build.check(emu.emu_product_arc_map(B, T, _p(off, i64p), _p(arc_of, i32p), _p(arcs, i32p)))
    return paths, scores, arcs, st, prods


def check_device_route(emu, product_emu, trace_lib, e, graphs, lens, kind, tw):
    """scores bit-equal to the live reference's; paths and arcs == wherever the tie bit is not raised, one of the
    optimal paths where it is; the tie bit raised exactly where the float32 restatement finds a tie on the traced path;
    the non-finite bit exactly where a weight or an emission of the utterance is not finite -> (ties, non-finite)"""
    p, s, a, st, prods = device_route(emu, product_emu, trace_lib, e, graphs, lens, kind, tw)
    pr, sr, ar = gtv.ref_graph_trans_viterbi(e, graphs, kind, tw, lens)
    C_ = e.shape[2]
    n_tie = n_bad = 0
    for b, g in enumerate(graphs):
        Tb = int(lens[b])
        if Tb == 0:
            assert np.isneginf(s[b]) and (p[b] == -1).all() and (a[b] == -1).all()
            continue
        bad = not (np.isfinite(prods[b]["w"]).all() and np.isfinite(e[b, :Tb]).all())
        assert bool(st[b] & 1) == bad, (b, st[b])
        if bad:  # the exact route's
            n_bad += 1
            continue
        want_score, tie = gtv.device_route_outcome(e[b, :Tb], prods[b], C_)
        assert s[b].tobytes() == sr[b].tobytes() == want_score.tobytes(), (b, s[b], sr[b])
        assert bool(st[b] & 2) == tie, (b, st[b], tie)
        assert (p[b, Tb:] == -1).all() and (a[b, Tb:] == -1).all()
        if not tie:
            assert np.array_equal(p[b], pr[b]) and np.array_equal(a[b], ar[b]), b
        else:
            n_tie += 1
            assert gtv.path_value(e[b, :Tb], g, kind, tw, p[b, :Tb], a[b, :Tb]) == s[b]
            assert np.array_equal(g["olabel"][a[b, :Tb]], p[b, :Tb])
    return n_tie, n_bad


@pytest.mark.parametrize("case", range(6))
def test_device_route_end_to_end_on_the_golden_graphs(oracle, emu, product_emu, trace_lib, case):
    need_ref(oracle)
    from tests.test_graph_trans_viterbi_oracle import golden_batches
    name, kind, e, graphs, lens, tw, _ = golden_batches()[case]
    k = gtv.ASG if kind == "asg" else gtv.BIGRAM
    keep = [i for i, g in enumerate(graphs) if len(g["flags"])]  # (the empty graph's product accepts nothing)
    graphs, lens, e = [graphs[i] for i in keep], np.ascontiguousarray(lens[keep]), np.ascontiguousarray(e[keep])
    n_tie, n_bad = check_device_route(emu, product_emu, trace_lib, e, graphs, lens, k, tw)
    assert (n_bad > 0) == (name == "b")  # batch b's -inf transitions reach every utterance with frames
    if name == "c":
        assert n_tie > 0


@pytest.mark.parametrize("kind", [gtv.ASG, gtv.BIGRAM])
@pytest.mark.parametrize("ties", [False, True])
def test_device_route_end_to_end_random(oracle, emu, product_emu, trace_lib, kind, ties):
    need_ref(oracle)
    rng = np.random.default_rng(100 + 2 * kind + ties)
    C_, T = 5, 9
    graphs = [g for _ in range(2) for g in _cases(rng, C_)]
    for g in graphs:
        g["w"] = (rng.integers(-1, 1, len(g["src"])) if ties else rng.uniform(-1, 1, len(g["src"]))).astype(np.float32)
    lens = rng.integers(1, T + 1, len(graphs)).astype(np.int32)
    e = (rng.integers(0, 2, (len(graphs), T, C_)) if ties else rng.uniform(-3, 3, (len(graphs), T, C_)))
    tw = rng.integers(-1, 1, (C_ + C_ * C_) if kind == gtv.ASG else C_ * C_) if ties else \
        rng.uniform(-1, 1, (C_ + C_ * C_) if kind == gtv.ASG else C_ * C_)
    n_tie, n_bad = check_device_route(emu, product_emu, trace_lib, e.astype(np.float32), graphs, lens, kind,
                                      tw.astype(np.float32))
    assert n_bad == 0 and (n_tie > 0) == ties
