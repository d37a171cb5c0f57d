"""The cluster sweeps of k_sparse.cu (sparse_cl_den_forward / backward, sparse_cl_viterbi_forward: one thread-block
cluster per utterance for a transition graph G too large for one CTA) run from their source through the SIMT emulator
(tests/emu/sparse_cluster_emu.cpp), with N = 2 and 4 CTAs of 64 threads, against the one-CTA kernels run in the same
emulator on the same inputs: alpha rows, offsets, Z, back-pointers, head, score, paths, arcs and status ==; the
gradients within util.close (only the order of the adds differs); and against the float64 / float32 restatements.
Node counts that are not a multiple of N, a rank without nodes, a hub whose in-list spans a rank's whole share, an
unreachable node, T_b in {0, 1}, ties, NaN raising the status bit, T = 300 with emissions near -20.  Then the host
side: the split builder's balance and sparse_cluster_plan's envelope, and the golden fixture of a 5000-node G."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_build
from tests import graph_oracle as go
from tests import sparse_trans_oracle as st
from tests import sparse_viterbi_oracle as sv
from tests import util
from tests.golden import make_sparse_cluster_golden as mk
from tests.test_sparse_trans_emulation import den64
from tests.test_sparse_trans_oracle import _p, graph_args

f32p, f64p, i32p, u8p, u16p = (C.POINTER(t) for t in (C.c_float, C.c_double, C.c_int32, C.c_uint8, C.c_uint16))
THREADS = 64  # per CTA of a cluster: N * 64 host threads


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("sparse_cluster", ["k_sparse.cu", "gtnb_product.h"]))
    graph = [C.c_int, C.c_int, u8p, i32p, i32p, i32p]
    lib.emu_cluster_plan.argtypes = graph + [C.c_int, C.c_int, i32p, i32p, i32p, i32p, i32p]
    run = [C.c_int, C.c_int, C.c_int, f32p, i32p] + graph + [f32p, C.c_int, C.c_int]
    lib.emu_cluster_den.argtypes = run + [f32p, f64p, f32p, f32p, f32p, i32p]
    lib.emu_cluster_viterbi.argtypes = run + [u16p, i32p, f32p, i32p, i32p, i32p]
    return lib


def _inputs(e, lens, G, w):
    _, ga = graph_args(G)
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    w = np.ascontiguousarray(w, np.float32)
    B, T, Cn = e.shape
    return [B, T, Cn, _p(e, f32p), _p(lens, i32p), len(G["flags"]), len(G["src"]), *ga, _p(w, f32p)], (e, lens, w)


def den(emu, e, lens, G, w, N):
    """-> alpha [B, T + 1, S], offs [B, T + 1], den [B], grad, wgrad, status"""
    args, keep = _inputs(e, lens, G, w)
    B, T, Cn = e.shape
    S = len(G["flags"])
    out = (np.zeros((B, T + 1, S), np.float32), np.zeros((B, T + 1), np.float64), np.zeros(B, np.float32),
           np.zeros((B, T, Cn), np.float32), np.zeros(len(w), np.float32), np.zeros(B, np.int32))
    emu_build.check(emu.emu_cluster_den(*args, N, THREADS, *(_p(a, t) for a, t in zip(out, (f32p, f64p, f32p, f32p,
                                                                                            f32p, i32p)))))
    return out


def viterbi(emu, e, lens, G, w, N):
    """-> bp [B, T, S], head, scores, paths, arcs, status"""
    args, keep = _inputs(e, lens, G, w)
    B, T, _ = e.shape
    out = (np.zeros((B, T, len(G["flags"])), np.uint16), np.zeros(B, np.int32), np.zeros(B, np.float32),
           np.zeros((B, T), np.int32), np.zeros((B, T), np.int32), np.zeros(B, np.int32))
    emu_build.check(emu.emu_cluster_viterbi(*args, N, THREADS, *(_p(a, t) for a, t in zip(out, (u16p, i32p, f32p, i32p,
                                                                                                i32p, i32p)))))
    return out


def same_den(emu, e, lens, G, w, N, rows=True):
    """the cluster kernels == the one-CTA kernels (rows only up to T_b: beyond it neither writes); -> the cluster's"""
    one, cl = den(emu, e, lens, G, w, 1), den(emu, e, lens, G, w, N)
    for b, n in enumerate(lens):
        assert np.array_equal(one[0][b, :n + 1], cl[0][b, :n + 1]), b
        assert np.array_equal(one[1][b, :n + 1], cl[1][b, :n + 1]), b
    assert np.array_equal(one[2], cl[2]) and np.array_equal(one[5], cl[5])
    assert util.close(cl[3], one[3]) and util.close(cl[4], one[4])
    return cl


def same_viterbi(emu, e, lens, G, w, N):
    one, cl = viterbi(emu, e, lens, G, w, 1), viterbi(emu, e, lens, G, w, N)
    for b, n in enumerate(lens):
        assert np.array_equal(one[0][b, :n], cl[0][b, :n]), b
    for x, y in zip(one[1:], cl[1:]):
        assert np.array_equal(x, y)
    return cl


def check(emu, e, lens, G, w, N):
    """both sweeps against the one-CTA kernels and against the restatements"""
    _, _, Z, grad, wgrad, status = same_den(emu, e, lens, G, w, N)
    assert not status.any()
    Z64, ge, gw = den64(e, lens, G, w)
    fin = np.isfinite(Z64)
    assert np.array_equal(np.isfinite(Z), fin)
    assert np.allclose(Z[fin], Z64[fin], rtol=1e-5, atol=1e-4)
    assert np.allclose(grad, ge, rtol=1e-4, atol=2e-5) and np.allclose(wgrad, gw, rtol=1e-4, atol=2e-5 * e[0].size)
    _, _, scores, paths, arcs, vstatus = same_viterbi(emu, e, lens, G, w, N)
    ties = 0
    for b, n in enumerate(lens):
        score, tie, labels, path_arcs = sv.decode_outcome(e[b, :n], G, w, e.shape[2])
        assert np.array_equal(scores[b], score) and bool(vstatus[b] & 2) == tie and not vstatus[b] & 1
        ties += tie
        if np.isfinite(score) and not tie:
            assert np.array_equal(paths[b, :n], labels) and np.array_equal(arcs[b, :n], path_arcs)
        assert (paths[b, n:] == -1).all()
    return ties


@pytest.mark.parametrize("N", [2, 4])
def test_ragged_batch_with_unreachable_nodes(emu, N):
    """13 nodes (not a multiple of N), two of them unreachable, labels >= C, T_b in {0, 1}, NaN in the padding"""
    rng = np.random.default_rng(10 + N)
    Cn, T = 7, 9
    G = st.sparse_graph(rng, 11, 50, Cn, label_hi=9)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = rng.uniform(-3, 3, (5, T, Cn)).astype(np.float32)
    lens = np.asarray([9, 0, 1, 6, 9], np.int32)
    e[3, 6:] = np.nan
    assert check(emu, e, lens, G, w, N) == 0


@pytest.mark.parametrize("N", [2, 4])
def test_trigram_has_several_lanes_per_node(emu, N):
    rng = np.random.default_rng(20 + N)
    Cn, T = 5, 10
    G = st.trigram_graph(Cn)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = rng.uniform(-3, 3, (2, T, Cn)).astype(np.float32)
    check(emu, e, np.asarray([T, 7], np.int32), G, w, N)


def hub_graph(rng, Cn):
    """node 3 takes 60 of the 90 arcs: with N = 4 its in-list is the whole share of a rank and more, so the next
    rank owns no node of the forward sweep; node 5 sends 40 arcs, the same for the backward"""
    S = 9
    src = np.r_[rng.integers(0, S, 60), np.full(30, 5), rng.integers(0, S, 10)]
    dst = np.r_[np.full(60, 3), rng.integers(0, S, 30), np.full(10, 5)]
    flags = np.zeros(S, np.uint8)
    flags[[0, 3]] |= 1
    flags[[3, 5, 7]] |= 2
    return go.make(flags, src, dst, rng.integers(0, Cn, 100))


def test_hub_and_a_rank_without_nodes(emu):
    rng = np.random.default_rng(30)
    Cn, T = 6, 8
    G = hub_graph(rng, Cn)
    args, keep = _inputs(np.zeros((1, 1, Cn)), [1], G, np.zeros(100))
    sp = [np.zeros(9, np.int32) for _ in range(4)] + [np.zeros(2, np.int32)]
    assert emu.emu_cluster_plan(*args[5:11], Cn, 4, *(_p(a, i32p) for a in sp)) == 4
    assert 0 in np.diff(sp[0][:5]) and 0 in np.diff(sp[1][:5])  # a rank without nodes, in either sweep
    w = rng.uniform(-1, 1, 100).astype(np.float32)
    e = rng.uniform(-3, 3, (3, T, Cn)).astype(np.float32)
    check(emu, e, np.asarray([T, 5, 2], np.int32), G, w, 4)
    check(emu, e, np.asarray([T, 5, 2], np.int32), G, w, 2)


@pytest.mark.parametrize("N", [2, 4])
def test_ties_raise_the_tie_bit_as_the_one_cta_kernel_does(emu, N):
    rng = np.random.default_rng(40)
    Cn, T = 4, 6
    G = st.trigram_graph(Cn)
    e = rng.integers(0, 2, (5, T, Cn)).astype(np.float32)
    assert check(emu, e, np.asarray([6, 5, 6, 1, 3], np.int32), G, np.zeros(len(G["src"]), np.float32), N) > 0


def test_nan_raises_the_status_bit_in_whichever_rank_meets_it(emu):
    rng = np.random.default_rng(50)
    Cn, T = 5, 6
    G = st.sparse_graph(rng, 12, 60, Cn, n_unreachable=0)
    e = rng.uniform(-3, 3, (3, T, Cn)).astype(np.float32)
    lens = np.asarray([T, T, 4], np.int32)
    e[2, 4:] = np.nan  # padding: unused
    for arc in (0, len(G["src"]) - 1):  # an arc of the first and of the last rank's nodes
        w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
        w[np.argsort(G["dst"], kind="stable")[arc]] = np.nan
        for N in (2, 4):
            assert (den(emu, e, lens, G, w, N)[5] == 1).all() and (den(emu, e, lens, G, w, 1)[5] == 1).all()
            assert (same_viterbi(emu, e, lens, G, w, N)[5] & 1).all()
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e[1, 2, :] = np.nan
    assert list(den(emu, e, lens, G, w, 4)[5]) == [0, 1, 0]
    assert list(viterbi(emu, e, lens, G, w, 4)[5] & 1) == [0, 1, 0]


def test_offsets_over_300_frames_near_minus_20(emu):
    """alpha falls by about 20 a frame: the rows stay relative to the offsets, which the ranks agree on bit for bit"""
    rng = np.random.default_rng(60)
    Cn, T = 4, 300
    G = st.sparse_graph(rng, 10, 40, Cn, n_unreachable=0)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = (rng.uniform(-1, 1, (1, T, Cn)) - 20.0).astype(np.float32)
    lens = np.asarray([T], np.int32)
    alpha, offs, Z, grad, wgrad, status = same_den(emu, e, lens, G, w, 2)
    Z64, ge, gw = den64(e, lens, G, w)
    assert Z64[0] < -5000 and abs(Z[0] - Z64[0]) <= 1e-6 * abs(Z64[0])
    assert np.abs(alpha[0][np.isfinite(alpha[0])]).max() < 100 and offs[0, T] < -5000
    assert np.allclose(grad, ge, rtol=1e-3, atol=1e-4) and np.allclose(wgrad, gw, rtol=1e-3, atol=1e-2)


def plan(emu, G, Cn, force=0):
    """-> (N, in split, out split, in arcs, out arcs per rank, (max in-degree, max out-degree))"""
    args, keep = _inputs(np.zeros((1, 1, Cn)), [1], G, np.zeros(len(G["src"])))
    sp = [np.zeros(9, np.int32) for _ in range(4)] + [np.zeros(2, np.int32)]
    N = emu.emu_cluster_plan(*args[5:11], Cn, force, *(_p(a, i32p) for a in sp))
    return (N, sp[0][:N + 1], sp[1][:N + 1], sp[2][:N], sp[3][:N], sp[4])


def test_splits_are_balanced(emu):
    rng = np.random.default_rng(70)
    for G, Cn in ((st.sparse_graph(rng, 3000, 20000, 16, n_unreachable=0), 16), (hub_graph(rng, 6), 6),
                  (st.trigram_graph(12), 12)):
        for force in (2, 4, 8):
            N, si, so, ai, ao, deg = plan(emu, G, Cn, force)
            assert N == force and si[0] == so[0] == 0 and si[N] == so[N] == len(G["flags"])
            assert (np.diff(si) >= 0).all() and (np.diff(so) >= 0).all()
            A = int((G["olabel"] < Cn).sum())
            assert ai.sum() == ao.sum() == A
            assert ai.max() <= A / N + deg[0] and ao.max() <= A / N + deg[1]


def test_plan_envelope(emu):
    rng = np.random.default_rng(80)
    assert plan(emu, st.trigram_graph(64), 64)[0] == 8  # 4096 nodes, 262 144 arcs
    assert plan(emu, st.sparse_graph(rng, 16384, 131072, 64, n_unreachable=0), 64)[0] == 8
    edge = st.sparse_graph(rng, 4096, 32768, 64, n_unreachable=0)  # the one-CTA envelope's edge: a cluster of 2 would do
    assert plan(emu, edge, 64)[0] == 2
    assert plan(emu, st.sparse_graph(rng, 5000, 40000, 32, n_unreachable=0), 32)[0] == 2
    assert plan(emu, st.sparse_graph(rng, 16385, 20000, 64, n_unreachable=0), 64)[0] == 0  # nodes over the bound
    assert plan(emu, st.sparse_graph(rng, 40, 262145, 64, n_unreachable=0), 64)[0] == 0  # arcs over the bound
    assert plan(emu, st.sparse_graph(rng, 16384, 262144, 64, n_unreachable=0), 64)[0] == 0  # no N fits 227 KB
    assert plan(emu, st.sparse_graph(rng, 50, 200, 1025, n_unreachable=0), 1025)[0] == 0  # C over the bound
    for deg, want in ((32766, 2), (32767, 0)):  # position | tie flag must stay below kBpNone
        hub = go.make([3, 0], np.zeros(deg, np.int32), np.ones(deg, np.int32), np.zeros(deg, np.int32))
        assert plan(emu, hub, 4)[0] == want


def test_golden_5000_node_graph(emu):
    """the reference's values for a G beyond the one-CTA envelope: the restatements and the emulated cluster kernels"""
    e, lens, G, w = mk.case()
    z = np.load(mk.GOLDEN)
    assert plan(emu, G, e.shape[2])[0] == 2
    want_w = np.zeros(len(w), np.float32)
    want_w[z["wgrad_idx"]] = z["wgrad_val"]
    Z64, ge, gw = den64(e, lens, G, w)
    _, _, Z, grad, wgrad, status = den(emu, e, lens, G, w, 2)
    assert not status.any()
    for got in ((Z64, ge, gw), (Z, grad, wgrad)):
        assert np.allclose(got[0], z["Z"], rtol=1e-5) and util.grad_close(got[1], z["grad"], 50.0)
        assert util.grad_close(got[2], want_w, 50.0)
    _, _, scores, paths, arcs, vstatus = viterbi(emu, e, lens, G, w, 2)
    assert not vstatus.any()
    assert np.array_equal(scores, z["scores"]) and np.array_equal(paths, z["paths"]) and np.array_equal(arcs, z["arcs"])
    for b, n in enumerate(lens):
        score, tie, labels, path_arcs = sv.decode_outcome(e[b, :n], G, w, e.shape[2])
        assert score == z["scores"][b] and not tie and np.array_equal(path_arcs, z["arcs"][b, :n])
