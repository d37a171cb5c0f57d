"""k_sparse.cu (the denominator of gtnb_sparse_transitions_loss over a G of any shape) run from its source through the
SIMT emulator (tests/emu/sparse_emu.cpp) against a float64 forward-backward over G's arcs: forwardScore(intersect(E_b,
G)), the emission gradient and the arc-weight gradient; ragged lengths, T_b in {0, 1}, C not a multiple of 4, unreachable
nodes and labels >= C, the trigram graph, G at the envelope's edge (4096 nodes, 32768 arcs), several lanes per node;
sigma of G's start groups and its fold against numpy."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_build
from tests import sparse_trans_oracle as st
from tests.test_sparse_trans_oracle import _p, emu, graph_args, sigma_of, start_groups  # noqa: F401

f32p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
THREADS = 512  # kSparseThreads


def den64(e, lens, G, w):
    """float64 forward-backward of intersect(E_b, G) -> (Z [B], emission gradient [B, T, C], arc gradient [nG])"""
    B, T, Cn = e.shape
    S = len(G["flags"])
    keep = (G["olabel"] >= 0) & (G["olabel"] < Cn)
    src, dst, lab = G["src"][keep], G["dst"][keep], G["olabel"][keep]
    ids = np.flatnonzero(keep)
    ww = w[keep].astype(np.float64)
    start, acc = (G["flags"] & 1) != 0, (G["flags"] & 2) != 0

    def seg_lse(x, seg):
        m = np.full(S, -np.inf)
        np.maximum.at(m, seg, x)
        mm = np.where(np.isfinite(m), m, 0.0)
        s = np.zeros(S)
        np.add.at(s, seg, np.exp(x - mm[seg]))
        with np.errstate(divide="ignore"):
            return np.where(s > 0, mm + np.log(s), -np.inf)

    Z = np.zeros(B)
    ge = np.zeros((B, T, Cn))
    gw = np.zeros(len(w))
    for b in range(B):
        Tb = int(lens[b])
        eb = e[b].astype(np.float64)
        al = [np.where(start, 0.0, -np.inf)]
        for t in range(Tb):
            al.append(seg_lse(al[-1][src] + ww + eb[t, lab], dst))
        fin = al[Tb][acc]
        Z[b] = -np.inf if not np.isfinite(fin).any() else np.logaddexp.reduce(fin)
        if Tb == 0 or not np.isfinite(Z[b]):
            continue
        be = np.where(acc, 0.0, -np.inf)
        for t in range(Tb - 1, -1, -1):
            x = ww + eb[t, lab] + be[dst]
            p = np.exp(al[t][src] + x - Z[b])
            np.add.at(ge[b, t], lab, p)
            np.add.at(gw, ids, p)
            be = seg_lse(x, src)
    return Z, ge, gw


def run_den(emu, e, lens, G, w):
    B, T, Cn = e.shape
    ka, ga = graph_args(G)
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    w = np.ascontiguousarray(w, np.float32)
    K = len(start_groups(G, Cn))
    den = np.zeros(B, np.float32)
    grad = np.zeros((B, T, Cn), np.float32)
    wgrad = np.zeros(len(w) + K, np.float32)
    sigma = np.zeros(max(K, 1), np.float32)
    status = np.zeros(B, np.int32)
    rc = emu.emu_sparse_den(B, T, Cn, _p(e, f32p), _p(lens, i32p), len(G["flags"]), len(G["src"]), *ga, _p(w, f32p),
                            THREADS, _p(den, f32p), _p(grad, f32p), _p(wgrad, f32p), _p(sigma, f32p),
                            _p(status, i32p))
    emu_build.check(rc)
    return den, grad, wgrad[:len(w)], sigma[:K], status


def check_den(emu, e, lens, G, w):
    den, grad, wgrad, _, status = run_den(emu, e, lens, G, w)
    Z, ge, gw = den64(e, lens, G, w)
    assert not status.any()
    fin = np.isfinite(Z)
    assert np.array_equal(np.isfinite(den), fin)
    assert np.allclose(den[fin], Z[fin], rtol=1e-5, atol=1e-4), np.abs(den[fin] - Z[fin]).max()
    assert np.allclose(grad, ge, rtol=1e-4, atol=2e-5), np.abs(grad - ge).max()
    assert np.allclose(wgrad, gw, rtol=1e-4, atol=2e-5 * len(lens) * e.shape[1]), np.abs(wgrad - gw).max()
    return Z


def test_random_sparse_graph_ragged(emu):
    """several start and accept nodes, unreachable nodes, labels >= C, C = 7 (not a multiple of 4), T_b in {0, 1}"""
    rng = np.random.default_rng(1)
    Cn, T = 7, 9
    G = st.sparse_graph(rng, 10, 45, Cn, label_hi=9)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = rng.uniform(-3, 3, (5, T, Cn)).astype(np.float32)
    lens = np.asarray([9, 0, 1, 6, 9], np.int32)
    e[3, 6:] = np.nan
    Z = check_den(emu, e, lens, G, w)
    assert np.isfinite(Z[[0, 3, 4]]).all()


def test_trigram(emu):
    """the trigram at C = 5: every node starts and accepts, C in-arcs per node (lanes > 1)"""
    rng = np.random.default_rng(2)
    Cn, T = 5, 12
    G = st.trigram_graph(Cn)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = rng.uniform(-3, 3, (2, T, Cn)).astype(np.float32)
    check_den(emu, e, np.asarray([12, 7], np.int32), G, w)


def test_long_utterance_offsets(emu):
    """scores that grow with t (T = 300, emissions far from 0): the per-frame offsets keep the posteriors exact"""
    rng = np.random.default_rng(3)
    Cn, T = 6, 300
    G = st.sparse_graph(rng, 8, 40, Cn, n_unreachable=0)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = (rng.uniform(-3, 3, (1, T, Cn)) - 20.0).astype(np.float32)
    check_den(emu, e, np.asarray([T], np.int32), G, w)


def test_envelope_edge(emu):
    """G at the envelope's edge: 4096 nodes, 32768 arcs (8 per node: lanes = 2)"""
    rng = np.random.default_rng(4)
    Cn, T, S, A = 64, 3, 4096, 32768
    G = st.sparse_graph(rng, S, A, Cn, n_start=64, n_accept=512, n_unreachable=0)
    assert len(G["flags"]) == S and len(G["src"]) == A
    w = rng.uniform(-1, 1, A).astype(np.float32)
    e = rng.uniform(-3, 3, (1, T, Cn)).astype(np.float32)
    check_den(emu, e, np.asarray([T], np.int32), G, w)
    # one node too many: outside the envelope
    G2 = st.sparse_graph(rng, S + 1, 8, Cn, n_unreachable=0)
    ka, ga = graph_args(G2)
    w2 = np.zeros(8, np.float32)
    out = np.zeros(3 * T * Cn + 64, np.float32)
    st_ = np.zeros(1, np.int32)
    rc = emu.emu_sparse_den(1, T, Cn, _p(e, f32p), _p(np.asarray([T], np.int32), i32p), S + 1, 8, *ga, _p(w2, f32p),
                            THREADS, _p(out, f32p), _p(out, f32p), _p(out, f32p), _p(out, f32p), _p(st_, i32p))
    assert rc == 1


def test_non_finite_raises_the_status_bit(emu):
    rng = np.random.default_rng(5)
    Cn, T = 4, 5
    G = st.trigram_graph(Cn)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = rng.uniform(-3, 3, (2, T, Cn)).astype(np.float32)
    w2 = w.copy()
    w2[7] = -np.inf
    assert run_den(emu, e, np.asarray([T, T], np.int32), G, w2)[4].all()
    e2 = e.copy()
    e2[1, 2, 3] = np.nan
    st_ = run_den(emu, e2, np.asarray([T, T], np.int32), G, w)[4]
    assert list(st_) == [0, 1]


def test_sigma_and_fold(emu):
    """sigma_k = logsumexp over start group k, and the fold wgrad[a] += wgrad[nG + k] * softmax, against numpy"""
    rng = np.random.default_rng(6)
    Cn = 6
    G = st.sparse_graph(rng, 9, 60, Cn, n_start=4, label_hi=8)
    w = rng.uniform(-2, 2, len(G["src"])).astype(np.float32)
    groups = start_groups(G, Cn)
    assert groups and max(len(m) for m in groups) > 1
    e = rng.uniform(-3, 3, (1, 3, Cn)).astype(np.float32)
    sigma = run_den(emu, e, np.asarray([3], np.int32), G, w)[3]
    assert np.allclose(sigma, sigma_of(w, groups), rtol=1e-6, atol=1e-6)
    nG, K = len(w), len(groups)
    wgrad = np.zeros(nG + K, np.float32)
    wgrad[:nG] = rng.uniform(-1, 1, nG)
    wgrad[nG:] = rng.uniform(-1, 1, K)
    want = wgrad[:nG].astype(np.float64)
    for k, m in enumerate(groups):
        want[m] += wgrad[nG + k] * np.exp(w[m].astype(np.float64) - sigma[k])
    ka, ga = graph_args(G)
    emu_build.check(emu.emu_sparse_fold(len(G["flags"]), nG, *ga, Cn, _p(w, f32p), _p(sigma, f32p), _p(wgrad, f32p)))
    assert np.allclose(wgrad[:nG], want, rtol=1e-5, atol=1e-6)
