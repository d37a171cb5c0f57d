"""k_sparse.cu's alignment kernels (sparse_eps_align_kernel, sparse_eps_align_trace_kernel) run from their source
through the SIMT emulator (tests/emu/backoff_align_emu.cpp) over per-utterance numerators P_b = A_b o G
(backoff_align_oracle.product) against the float32 restatement (backoff_align_oracle.restate_align): numerators of
different sizes in one launch, scores bitwise, the tie bit where the restatement finds a tie, A_b's arcs and labels
elsewhere; an epsilon arc on the path and one after the last frame; a tie on an epsilon candidate; no accepting path;
the non-finite status bit."""
import ctypes as C

import numpy as np
import pytest

from tests import backoff_align_oracle as ba
from tests import backoff_oracle as bo
from tests import emu_build
from tests import graph_oracle as go
from tests.test_sparse_trans_oracle import _p

f32p, i32p, u8p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)
EPS = bo.EPS


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("backoff_align", ["k_sparse.cu", "gtnb_product.h"]))
    lib.emu_backoff_align.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, i32p, i32p, u8p, i32p, i32p, i32p, f32p,
                                      i32p, i32p, i32p, i32p, f32p, i32p]
    return lib


def align(emu, e, lens, graphs, G, tw):
    """the device route over the numpy numerators, weights gathered as sparse_eps_gather does
    -> (paths, arcs, scores, status)"""
    B, T, Cn = e.shape
    prods = [ba.product(g, G, Cn) for g in graphs]
    first = np.cumsum([0] + [len(g["src"]) for g in graphs])
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs) if len(xs) else np.zeros(0), dt)
    flags = cat([P["flags"] for P, _, _ in prods], np.uint8)
    src, dst, lab = (cat([P[k] for P, _, _ in prods], np.int32) for k in ("src", "dst", "olabel"))
    arc_of = cat([np.where(ao < 0, -1, ao + first[b]) for b, (_, ao, _) in enumerate(prods)], np.int32)
    w_A = np.concatenate([g["w"] for g in graphs]).astype(np.float32)
    tidx = cat([ti for _, _, ti in prods], np.int32)
    w = np.where(arc_of < 0, tw[tidx], w_A[np.maximum(arc_of, 0)] + tw[tidx]).astype(np.float32)
    S = np.asarray([len(P["flags"]) for P, _, _ in prods], np.int32)
    nA = np.asarray([len(P["src"]) for P, _, _ in prods], np.int32)
    a_first = np.ascontiguousarray(first[:B], np.int32)
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    paths, arcs = np.full((B, T), -7, np.int32), np.full((B, T), -7, np.int32)
    scores, status = np.full(B, np.nan, np.float32), np.zeros(B, np.int32)
    emu_build.check(emu.emu_backoff_align(B, T, Cn, _p(e, f32p), _p(lens, i32p), _p(S, i32p), _p(nA, i32p),
                                          _p(flags, u8p), _p(src, i32p), _p(dst, i32p), _p(lab, i32p), _p(w, f32p),
                                          _p(arc_of, i32p), _p(a_first, i32p), _p(paths, i32p), _p(arcs, i32p),
                                          _p(scores, f32p), _p(status, i32p)))
    return paths, arcs, scores, status


def check(emu, e, lens, graphs, G, tw):
    """-> the number of utterances with the tie bit"""
    paths, arcs, scores, status = align(emu, e, lens, graphs, G, tw)
    assert not (status & 1).any()
    n_ties = 0
    for b, g in enumerate(graphs):
        n = int(lens[b])
        score, tie, labels, a_arcs = ba.restate_align(e[b, :n], g, G, tw, e.shape[2])
        assert np.array_equal(scores[b], np.float32(score)), (b, scores[b], score)
        assert bool(status[b] & 2) == tie, (b, status[b], tie)
        n_ties += tie
        if not np.isfinite(score):
            assert (paths[b] == -1).all() and (arcs[b] == -1).all()
            continue
        assert (paths[b, n:] == -1).all() and (arcs[b, n:] == -1).all()
        assert np.array_equal(paths[b, :n], g["olabel"][arcs[b, :n]])
        if not tie:
            assert np.array_equal(paths[b, :n], labels) and np.array_equal(arcs[b, :n], a_arcs)
    return n_ties


@pytest.mark.parametrize("kind", ["bigram", "trigram", "random"])
def test_numerators_of_different_sizes(emu, kind):
    """CTC graphs of 1 .. 3 labels and random graphs (labels >= C, several start and accept nodes), ragged T_b with 0
    and 1: numerators of different S_b in one launch"""
    rng = np.random.default_rng({"bigram": 41, "trigram": 42, "random": 43}[kind])
    Cn, T = 6, 8
    if kind == "random":
        G, tw = bo.eps_graph(rng, 8, 30, Cn, 10, label_hi=Cn + 1)
    else:
        G, tw = bo.backoff_ngram(rng, Cn, 2 if kind == "bigram" else 3, n_tokens=600, min_count=2)
    graphs = [go.ctc_graph(rng.integers(1, Cn, k)) for k in (1, 3, 2)] + \
             [go.random_graph(rng, 5, 14, Cn, n_start=2, n_accept=2, label_hi=Cn + 2)]
    for g in graphs:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    e = rng.uniform(-2, 2, (len(graphs), T, Cn)).astype(np.float32)
    lens = np.asarray([T, 5, 0, 1], np.int32)
    for b in range(len(lens)):
        e[b, lens[b]:] = np.nan
    assert len({len(g["flags"]) for g in graphs}) > 1
    check(emu, e, lens, graphs, G, tw)


def test_epsilon_arcs_on_the_path_and_after_the_last_frame(emu):
    """G: 0 -a-> 1, 1 -eps-> 2, 2 -b-> 3, 3 -eps-> 4, 4 accepts alone, so that every path crosses an epsilon arc
    between its frames and ends on one after the last frame; the trace reports A_b's two arcs only"""
    Cn = 3
    G = go.make([1, 0, 0, 0, 2], [0, 1, 2, 3], [1, 2, 3, 4], [1, EPS, 2, EPS])
    tw = np.asarray([0.5, -0.25, 0.25, -0.5], np.float32)
    g = go.make([1, 0, 2], [0, 1], [1, 2], [1, 2])
    g["w"] = np.asarray([0.125, 0.375], np.float32)
    e = np.random.default_rng(5).uniform(-1, 1, (1, 2, Cn)).astype(np.float32)
    paths, arcs, scores, status = align(emu, e, np.asarray([2], np.int32), [g], G, tw)
    assert list(paths[0]) == [1, 2] and list(arcs[0]) == [0, 1] and not status[0]
    check(emu, e, np.asarray([2], np.int32), [g], G, tw)


def test_tie_on_an_epsilon_candidate(emu):
    """an epsilon arc that reaches a product node with exactly the score of its emitting in-arc raises the tie bit;
    a strictly better one is followed inside the frame"""
    Cn = 2
    # G: 0 -a-> 1, 0 -a-> 2, 2 -eps-> 1, 1 -a-> 0; 0 starts, 1 accepts (backoff_emulation's tie case)
    G = go.make([1, 2, 0], [0, 0, 2, 1], [1, 2, 1, 0], [0, 0, EPS, 0])
    g = go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [0, 0, 0])
    g["w"] = np.zeros(3, np.float32)
    e = np.zeros((2, 3, Cn), np.float32)
    e[:, :, 0] = 1.0
    lens = np.asarray([3, 3], np.int32)
    for tw, tie in ((np.zeros(4, np.float32), True), (np.asarray([0, 0, 1, 0], np.float32), False)):
        status = align(emu, e, lens, [g, g], G, tw)[3]
        assert bool(status[0] & 2) == tie and bool(status[1] & 2) == tie
        assert check(emu, e, lens, [g, g], G, tw) == (2 if tie else 0)


def test_no_accepting_path(emu):
    """a target longer than the frames, a graph without a start node and T_b = 0: score -inf, rows of -1"""
    rng = np.random.default_rng(6)
    Cn, T = 5, 3
    G, tw = bo.backoff_ngram(rng, Cn, 3, n_tokens=500, min_count=2)
    graphs = [go.make([1, 0, 0, 0, 0, 2], [0, 1, 2, 3, 4], [1, 2, 3, 4, 5], [1, 2, 3, 4, 1]),
              go.make([0, 2], [0], [1], [1]), go.ctc_graph([1])]
    e = rng.uniform(-1, 1, (3, T, Cn)).astype(np.float32)
    paths, arcs, scores, status = align(emu, e, np.asarray([T, T, 0], np.int32), graphs, G, tw)
    assert np.isneginf(scores).all() and (paths == -1).all() and (arcs == -1).all() and not status.any()


def test_nonfinite_status_bit(emu):
    """a NaN or +inf product weight raises bit 1; -inf only forbids the arc"""
    rng = np.random.default_rng(7)
    Cn, T = 5, 5
    G, tw0 = bo.backoff_ngram(rng, Cn, 3, n_tokens=400, min_count=2)
    eps = np.flatnonzero(G["olabel"] == EPS)
    graphs = [go.ctc_graph([1, 2]), go.ctc_graph([3])]
    e = rng.uniform(-1, 1, (2, T, Cn)).astype(np.float32)
    lens = np.asarray([T, T], np.int32)
    for v, bit in ((np.nan, 1), (np.inf, 1), (-np.inf, 0)):
        tw = tw0.copy()
        tw[eps] = v
        assert bool((align(emu, e, lens, graphs, G, tw)[3] & 1).all()) == bool(bit)
    assert not (align(emu, e, lens, graphs, G, tw0)[3] & 1).any()
