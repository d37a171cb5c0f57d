"""k_sparse.cu's backoff kernels (sparse_eps_*) and gtnb_product.h's epsilon tables, run from their source through the
SIMT emulator (tests/emu/backoff_emu.cpp), against the restatements of tests/backoff_oracle.py and, for the product
builder, the live reference: the level builder and the cycle it reports; the log-semiring sweeps over G (one graph for
every CTA) and over per-utterance numerators (per-CTA tables, the numerator's sign); the gather and scatter of the
numerators' weights and gradients; the tropical sweep and trace, an epsilon arc tying an emitting arc included; the
level bound at the envelope's edge; the non-finite status bit."""
import ctypes as C

import numpy as np
import pytest

from tests import backoff_oracle as bo
from tests import emu_build
from tests import graph_oracle as go
from tests import util
from tests.test_graph_trans_oracle import need_ref
from tests.test_sparse_trans_oracle import _p, graph_args

f32p, i32p, u8p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)
ip = C.POINTER(C.c_int)
EPS = bo.EPS


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("backoff", ["k_sparse.cu", "gtnb_product.h"]))
    lib.emu_backoff_tables.argtypes = [C.c_int, C.c_int, u8p, i32p, i32p, i32p, C.c_int, i32p, i32p, i32p, i32p, i32p,
                                       i32p, i32p]
    lib.emu_backoff_product.argtypes = [C.c_int, C.c_int, u8p, i32p, i32p, i32p, C.c_int, C.c_int, u8p, i32p, i32p,
                                        i32p, C.c_int, ip, ip, u8p, i32p, i32p, i32p, i32p, i32p]
    lib.emu_backoff_sweep.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, C.c_int, i32p, i32p, u8p, i32p, i32p,
                                      i32p, f32p, C.c_float, C.c_int, f32p, f32p, f32p, i32p]
    lib.emu_backoff_viterbi.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, C.c_int, C.c_int, u8p, i32p, i32p,
                                        i32p, f32p, C.c_int, i32p, i32p, f32p, i32p]
    lib.emu_backoff_gather_scatter.argtypes = [C.c_longlong, f32p, i32p, f32p, i32p, f32p, f32p, f32p, f32p]
    return lib


def tables(emu, G, Cn):
    """-> (info [E, L, cycle length, A, max in-degree], cycle, fwd_ptr, fwd_node, bwd_ptr, bwd_node, lanes)"""
    _, ga = graph_args(G)
    info = np.zeros(5, np.int32)
    emu.emu_backoff_tables(len(G["flags"]), len(G["src"]), *ga, Cn, _p(info, i32p), None, None, None, None, None, None)
    L = int(info[1])
    cyc = np.zeros(max(int(info[2]), 1), np.int32)
    fp, bp = np.zeros(L + 1, np.int32), np.zeros(L + 1, np.int32)
    fn, bn = np.zeros(len(G["flags"]) + 1, np.int32), np.zeros(len(G["flags"]) + 1, np.int32)
    lanes = np.zeros(2 * L + 1, np.int32)
    emu.emu_backoff_tables(len(G["flags"]), len(G["src"]), *ga, Cn, _p(info, i32p), _p(cyc, i32p), _p(fp, i32p),
                           _p(fn, i32p), _p(bp, i32p), _p(bn, i32p), _p(lanes, i32p))
    return info, cyc[:info[2]], fp, fn[:fp[-1]], bp, bn[:bp[-1]], lanes[:2 * L]


def product(emu, g, G, Cn):
    """-> (P graph_oracle layout with epsilon arcs labelled -1, arc_of, tidx) through the shipped builder"""
    _, aa = graph_args(g)
    _, ga = graph_args(G)
    nn, na = C.c_int(), C.c_int()
    args = (len(g["flags"]), len(g["src"]), *aa, len(G["flags"]), len(G["src"]), *ga, Cn, C.byref(nn), C.byref(na))
    emu.emu_backoff_product(*args, None, None, None, None, None, None)
    fl = np.zeros(nn.value, np.uint8)
    s, d, lab, ao, ti = (np.zeros(max(na.value, 1), np.int32) for _ in range(5))
    emu.emu_backoff_product(*args, _p(fl, u8p), _p(s, i32p), _p(d, i32p), _p(lab, i32p), _p(ao, i32p), _p(ti, i32p))
    n = na.value
    return go.make(fl, s[:n], d[:n], lab[:n]), ao[:n], ti[:n]


def sweep(emu, e, lens, graphs, ws, sgn=1.0, threads=512):
    """emu_backoff_sweep over one graph for every utterance (len(graphs) == 1) or graph b for utterance b
    -> (Z [B], grad [B, T, C], wgrad per graph, status)"""
    B, T, Cn = e.shape
    cat = lambda k, dt: np.ascontiguousarray(np.concatenate([g[k] for g in graphs]), dt)
    flags, src, dst, lab = cat("flags", np.uint8), cat("src", np.int32), cat("dst", np.int32), cat("olabel", np.int32)
    S = np.asarray([len(g["flags"]) for g in graphs], np.int32)
    nA = np.asarray([len(g["src"]) for g in graphs], np.int32)
    w = np.ascontiguousarray(np.concatenate(ws), np.float32)
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    den = np.zeros(B, np.float32)
    grad = np.zeros_like(e)
    wgrad = np.zeros(max(len(w), 1), np.float32)
    status = np.zeros(B, np.int32)
    rc = emu.emu_backoff_sweep(B, T, Cn, _p(e, f32p), _p(lens, i32p), len(graphs), _p(S, i32p), _p(nA, i32p),
                               _p(flags, u8p), _p(src, i32p), _p(dst, i32p), _p(lab, i32p), _p(w, f32p), sgn, threads,
                               _p(den, f32p), _p(grad, f32p), _p(wgrad, f32p), _p(status, i32p))
    emu_build.check(rc)
    return den, grad, np.split(wgrad[:len(w)], np.cumsum(nA)[:-1]), status


def decode(emu, e, lens, G, w, lanes=0):
    B, T, Cn = e.shape
    _, ga = graph_args(G)
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    w = np.ascontiguousarray(w, np.float32)
    paths, arcs = np.full((B, T), -7, np.int32), np.full((B, T), -7, np.int32)
    scores, status = np.full(B, np.nan, np.float32), np.zeros(B, np.int32)
    rc = emu.emu_backoff_viterbi(B, T, Cn, _p(e, f32p), _p(lens, i32p), len(G["flags"]), len(G["src"]), *ga,
                                 _p(w, f32p), lanes, _p(paths, i32p), _p(arcs, i32p), _p(scores, f32p),
                                 _p(status, i32p))
    emu_build.check(rc)
    return paths, arcs, scores, status


def check_sweep(got, e, lens, G, w, Cn, sgn=1.0):
    Z, grad, wgrad = bo.restate_loss(e, lens, G, w, Cn)
    den, g, wg, status = got
    assert not status.any()
    assert util.close(den, Z.astype(np.float32)), (den, Z)
    mag = float(np.max(np.abs(Z[np.isfinite(Z)]), initial=1.0)) + 5.0 * e.shape[1]
    assert util.grad_close(g, sgn * grad, mag), float(np.abs(g - sgn * grad).max())
    assert util.grad_close(wg, sgn * wgrad, mag * len(lens)), float(np.abs(wg - sgn * wgrad).max())


def test_levels_and_cycle(emu):
    """the forward and backward levels of a backoff trigram (two levels), of a bigram (one) and of a random epsilon
    DAG against the restatement; an epsilon cycle is reported as its nodes in arc order, with no levels"""
    rng = np.random.default_rng(3)
    for G, Cn, L in ((bo.backoff_ngram(rng, 6, 3)[0], 6, 2), (bo.backoff_ngram(rng, 6, 2)[0], 6, 1),
                     (bo.eps_graph(rng, 12, 30, 5, 15)[0], 5, None)):
        info, cyc, fp, fn, bp, bn, lanes = tables(emu, G, Cn)
        f, b = bo.closure_levels(G)
        assert info[0] == (G["olabel"] == EPS).sum() and info[2] == 0
        assert info[1] == f.max() == b.max() and (L is None or info[1] == L)
        for l in range(info[1]):
            assert sorted(fn[fp[l]:fp[l + 1]]) == sorted(np.flatnonzero(f == l + 1))
            assert sorted(bn[bp[l]:bp[l + 1]]) == sorted(np.flatnonzero(b == l + 1))
        assert ((lanes >= 1) & (lanes <= 32) & ((lanes & (lanes - 1)) == 0)).all()
    G, _ = bo.eps_cycle_graph()
    info, cyc, *_ = tables(emu, G, 3)
    assert info[2] == 3 and info[1] == 0
    assert list(np.roll(cyc, -int(np.argmin(cyc)))) == [1, 2, 3]


@pytest.mark.parametrize("case", ["bigram", "trigram", "random"])
def test_denominator_sweep(emu, case):
    """one G for every CTA: Z, the emission gradient and the arc gradient (epsilon arcs' included) against the
    float64 restatement; ragged T_b with 0 and 1, NaN padding, epsilon arcs out of start and into accept nodes"""
    rng = np.random.default_rng({"bigram": 1, "trigram": 2, "random": 3}[case])
    Cn, T, B = 6, 7, 5
    if case == "random":
        G, w = bo.eps_graph(rng, 10, 40, Cn, 12, label_hi=Cn + 1)
    else:
        G, w = bo.backoff_ngram(rng, Cn, 2 if case == "bigram" else 3, n_tokens=600, min_count=2)
    e = rng.uniform(-2, 2, (B, T, Cn)).astype(np.float32)
    lens = np.asarray([T, 0, 1, 4, T], np.int32)
    for b in range(B):
        e[b, lens[b]:] = np.nan
    check_sweep(sweep(emu, e, lens, [G], [w]), e, lens, G, w, Cn)


def test_numerators_per_cta(emu):
    """every CTA its own numerator P_b = A_b o G (the shipped builder with G's epsilon arcs), the numerator's sign,
    then the gather of its weights and the scatter of its gradients into trans_grad and arc_grads"""
    rng = np.random.default_rng(4)
    Cn, T, B = 6, 8, 4
    G, tw = bo.backoff_ngram(rng, Cn, 3, n_tokens=600, min_count=2)
    graphs = [go.ctc_graph(rng.integers(1, Cn, int(rng.integers(1, 3)))) for _ in range(B)]
    for g in graphs:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    prods = [product(emu, g, G, Cn) for g in graphs]
    assert all((P["olabel"] == EPS).any() for P, _, _ in prods)
    # the gather: fl(w_A + w_G), w_G alone on an epsilon arc
    first = np.cumsum([0] + [len(g["src"]) for g in graphs])
    arc_of = np.concatenate([np.where(ao < 0, -1, ao + first[b]) for b, (_, ao, _) in enumerate(prods)]).astype(np.int32)
    tidx = np.concatenate([ti for _, _, ti in prods]).astype(np.int32)
    w_A = np.concatenate([g["w"] for g in graphs]).astype(np.float32)
    n = len(tidx)
    fw, pg = np.zeros(n, np.float32), rng.uniform(-1, 1, n).astype(np.float32)
    tg, ag = np.zeros(len(tw), np.float32), np.zeros(len(w_A), np.float32)
    emu_build.check(emu.emu_backoff_gather_scatter(n, _p(w_A, f32p), _p(arc_of, i32p), _p(tw, f32p), _p(tidx, i32p),
                                                   _p(fw, f32p), _p(pg, f32p), _p(tg, f32p), _p(ag, f32p)))
    want = np.where(arc_of < 0, tw[tidx], w_A[np.maximum(arc_of, 0)] + tw[tidx]).astype(np.float32)
    assert np.array_equal(fw, want)
    tg_want, ag_want = np.zeros(len(tw)), np.zeros(len(w_A))
    np.add.at(tg_want, tidx, pg)
    np.add.at(ag_want, arc_of[arc_of >= 0], pg[arc_of >= 0])
    assert np.allclose(tg, tg_want, atol=1e-5) and np.allclose(ag, ag_want, atol=1e-5)
    # the sweeps with per-CTA tables
    e = rng.uniform(-2, 2, (B, T, Cn)).astype(np.float32)
    lens = np.asarray([T, 5, 0, 3], np.int32)
    ws = np.split(fw, np.cumsum([len(P["src"]) for P, _, _ in prods])[:-1])
    den, g, wg, status = sweep(emu, e, lens, [P for P, _, _ in prods], ws, sgn=-1.0)
    assert not status.any()
    for b, (P, _, _) in enumerate(prods):
        Z, grad, wgrad = bo.restate_loss(e[b:b + 1], lens[b:b + 1], P, ws[b], Cn)
        assert util.close(den[b], np.float32(Z[0])), (b, den[b], Z[0])
        mag = abs(float(Z[0])) if np.isfinite(Z[0]) else 1.0
        assert util.grad_close(g[b], -grad[0], mag + 5.0 * T)
        assert util.grad_close(wg[b], -wgrad, mag + 5.0 * T)


def test_product_matches_reference_intersection(oracle, emu):
    """forwardScore(compose(P_b, E_b)) of the built product with G's epsilon arcs = the reference's
    forwardScore(intersect(intersect(A_b, G), E_b)); the product's gradients mapped back through arc_of / tidx = the
    reference's A_b and G gradients"""
    need_ref(oracle)
    po = oracle
    rng = np.random.default_rng(5)
    Cn, T = 5, 6
    for G, tw in (bo.backoff_ngram(rng, Cn, 3, n_tokens=500, min_count=2),
                  bo.eps_graph(rng, 8, 30, Cn, 10, label_hi=Cn + 1)):
        gd = dict(G)
        gd["w"] = tw
        for g in (go.ctc_graph([1, 2, 1]), go.random_graph(rng, 5, 14, Cn, n_start=2, n_accept=2)):
            g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
            P, arc_of, tidx = product(emu, g, G, Cn)
            P["w"] = np.where(arc_of < 0, tw[tidx], g["w"][np.maximum(arc_of, 0)] + tw[tidx]).astype(np.float32)
            e = rng.uniform(-2, 2, (T, Cn)).astype(np.float32)
            rp = go.ref_graph(P)
            s = po.ref_op("forward_score", po.ref_op("compose", rp, po.RefGraph.linear(T, Cn, e.ravel())))
            po.ref_backward(s)
            A, RG = go.ref_graph(g), go.ref_graph(gd)
            want = po.ref_op("forward_score", po.ref_op("intersect", po.ref_op("intersect", A, RG),
                                                         po.RefGraph.linear(T, Cn, e.ravel())))
            po.ref_backward(want)
            assert util.close(s.item(), want.item()), (s.item(), want.item())
            if not np.isfinite(want.item()):
                continue
            pg = rp.grad().weights().astype(np.float64)
            ag = np.bincount(arc_of[arc_of >= 0], pg[arc_of >= 0], minlength=len(g["src"]))
            tg = np.zeros(len(tw))
            np.add.at(tg, tidx, pg)
            mag = abs(want.item()) + 5.0 * T
            assert util.grad_close(ag, A.grad().weights(), mag)
            assert util.grad_close(tg, RG.grad().weights(), mag)


def check_decode(emu, e, lens, G, w, lanes=0):
    paths, arcs, scores, status = decode(emu, e, lens, G, w, lanes)
    Cn = e.shape[2]
    assert not (status & 1).any()
    n_ties = 0
    for b in range(e.shape[0]):
        n = int(lens[b])
        score, tie, labels, path_arcs = bo.restate_decode(e[b, :n], G, w, Cn)
        assert np.array_equal(scores[b], score), (b, scores[b], score)
        assert bool(status[b] & 2) == tie, (b, status[b], tie)
        n_ties += tie
        if not np.isfinite(score):
            assert (paths[b] == -1).all() and (arcs[b] == -1).all()
            continue
        assert (paths[b, n:] == -1).all() and (arcs[b, n:] == -1).all()
        assert np.array_equal(paths[b, :n], G["olabel"][arcs[b, :n]])
        if not tie:
            assert np.array_equal(paths[b, :n], labels) and np.array_equal(arcs[b, :n], path_arcs)
    return n_ties


@pytest.mark.parametrize("lanes", [0, 1, 4, 32])
def test_decode(emu, lanes):
    """the tropical sweep with the epsilon closure and the trace through epsilon back-pointers: scores bit-equal to
    the float32 restatement, the tie bit where it finds a tie, its path elsewhere"""
    rng = np.random.default_rng(6 + lanes)
    Cn, T, B = 6, 9, 5
    e = rng.uniform(-2, 2, (B, T, Cn)).astype(np.float32)
    lens = np.asarray([T, 0, 1, 5, T], np.int32)
    for G, w in (bo.backoff_ngram(rng, Cn, 3, n_tokens=600, min_count=2),
                 bo.eps_graph(rng, 10, 40, Cn, 12, label_hi=Cn + 1)):
        check_decode(emu, e, lens, G, w, lanes)


def test_decode_epsilon_ties_emitting(emu):
    """an epsilon arc that reaches a node with exactly the score of its emitting in-arc raises the tie bit; one that
    is strictly better is followed inside the frame, and the frame reports the emitting arc before it"""
    Cn = 2
    # 0 -a-> 1, 0 -a-> 2, 2 -eps-> 1, 1 -a-> 0; 0 starts, 1 accepts
    G = go.make([1, 2, 0], [0, 0, 2, 1], [1, 2, 1, 0], [0, 0, EPS, 0])
    e = np.zeros((2, 3, Cn), np.float32)
    e[:, :, 0] = 1.0
    lens = np.asarray([3, 1], np.int32)
    for w, tie in ((np.asarray([0, 0, 0, 0], np.float32), True), (np.asarray([0, 0, 1, 0], np.float32), False)):
        paths, arcs, scores, status = decode(emu, e, lens, G, w)
        assert bool(status[0] & 2) == tie and bool(status[1] & 2) == tie
        if not tie:
            assert list(arcs[1, :1]) == [1] and scores[1] == 2.0 and list(arcs[0]) == [1, 3, 1]
        check_decode(emu, e, lens, G, w)


def test_level_bound_at_the_envelope_edge(emu):
    """a chain of 32 epsilon arcs (32 levels) is swept; 33 is outside the envelope"""
    rng = np.random.default_rng(7)
    Cn, T = 3, 4
    for n_eps, inside in ((32, True), (33, False)):
        N = n_eps + 1
        src = list(range(n_eps)) + list(range(N))
        dst = list(range(1, N)) + list(range(N))
        lab = [EPS] * n_eps + list(rng.integers(0, Cn, N))
        flags = np.zeros(N, np.uint8)
        flags[0] = 1
        flags[-1] = 2
        G = go.make(flags, src, dst, lab)
        w = rng.uniform(-1, 0, len(src)).astype(np.float32)
        e = rng.uniform(-1, 1, (2, T, Cn)).astype(np.float32)
        lens = np.asarray([T, 2], np.int32)
        info = tables(emu, G, Cn)[0]
        assert info[1] == n_eps
        if inside:
            check_sweep(sweep(emu, e, lens, [G], [w]), e, lens, G, w, Cn)
            check_decode(emu, e, lens, G, w)
        else:
            with pytest.raises(AssertionError):
                sweep(emu, e, lens, [G], [w])


def test_nonfinite_status_bit(emu):
    """a NaN or infinite epsilon weight raises the status bit of the log sweep; the decode raises it for NaN and +inf
    and not for -inf, which only forbids the arc"""
    rng = np.random.default_rng(8)
    Cn, T = 5, 5
    G, w0 = bo.backoff_ngram(rng, Cn, 3, n_tokens=400, min_count=2)
    eps = np.flatnonzero(G["olabel"] == EPS)
    e = rng.uniform(-1, 1, (2, T, Cn)).astype(np.float32)
    lens = np.asarray([T, T], np.int32)
    for v, log_bit, vit_bit in ((np.nan, 1, 1), (np.inf, 1, 1), (-np.inf, 1, 0)):
        w = w0.copy()
        w[eps] = v
        assert (sweep(emu, e, lens, [G], [w])[3] & 1).all() == bool(log_bit)
        assert bool((decode(emu, e, lens, G, w)[3] & 1).all()) == bool(vit_bit)
    assert not sweep(emu, e, lens, [G], [w0])[3].any()
