"""The golden fixture of the backoff cluster route (tests/golden/make_backoff_cluster_golden.py: the reference's values
for a backoff 4-gram of 8563 states at C = 64, beyond the one-CTA envelope, so only the cluster kernels can sweep it on
the device) against the float64 loss restatement (backoff_oracle.restate_loss), a float32 restatement of the decode's
scores, the emulated cluster kernels (tests/emu/backoff_cluster_emu.cpp, N = 2), and, for the alignment, the float32
decode restatement (backoff_oracle.restate_decode) over the numerators built by the shipped product builder."""
import ctypes as C

import numpy as np
import pytest

from tests import backoff_oracle as bo
from tests import emu_build
from tests import util
from tests.golden import make_backoff_cluster_golden as mk
from tests.test_backoff_cluster_emulation import den, emu, plan, viterbi  # noqa: F401  (emu: the fixture)
from tests.test_backoff_emulation import product

EPS = bo.EPS
u8p, i32p = C.POINTER(C.c_uint8), C.POINTER(C.c_int32)


@pytest.fixture(scope="module")
def case():
    return mk.case() + (np.load(mk.GOLDEN),)


@pytest.fixture(scope="module")
def backoff_emu():
    lib = C.CDLL(emu_build.build("backoff", ["k_sparse.cu", "gtnb_product.h"]))
    ip = C.POINTER(C.c_int)
    lib.emu_backoff_product.argtypes = [C.c_int, C.c_int, u8p, i32p, i32p, i32p, C.c_int, C.c_int, u8p, i32p, i32p,
                                        i32p, C.c_int, ip, ip, u8p, i32p, i32p, i32p, i32p, i32p]
    return lib


def dense_wgrad(z, n):
    w = np.zeros(n, np.float32)
    w[z["wgrad_idx"]] = z["wgrad_val"]
    return w


def restate_scores(e, G, w, C):
    """float32 restatement of the decode's score for one utterance (e: its T_b rows): S_t[v] = max over emitting
    in-arcs of fl(S_{t-1}[u] + fl(w + e)), then, level by level, max with fl(S_t[u] + w) over epsilon in-arcs; the
    best accept node's score (-inf without one)"""
    src, dst, lab = G["src"], G["dst"], G["olabel"]
    w = np.asarray(w, np.float32)
    emit = np.flatnonzero((lab >= 0) & (lab < C))
    eps = np.flatnonzero(lab == EPS)
    f, _ = bo.closure_levels(G)
    by_level = [eps[f[dst[eps]] == l] for l in range(1, int(f.max()) + 1)]
    N = len(G["flags"])

    def close(S):
        for ks in by_level:
            m = np.full(N, -np.inf, np.float32)
            np.maximum.at(m, dst[ks], (S[src[ks]] + w[ks]).astype(np.float32))
            S = np.maximum(S, m)
        return S

    S = close(np.where(G["flags"] & 1, 0.0, -np.inf).astype(np.float32))
    for t in range(e.shape[0]):
        m = np.full(N, -np.inf, np.float32)
        np.maximum.at(m, dst[emit], (S[src[emit]] + (w[emit] + e[t, lab[emit]]).astype(np.float32)).astype(np.float32))
        S = close(m)
    acc = (G["flags"] & 2) != 0
    return np.float32(S[acc].max()) if e.shape[0] and acc.any() else np.float32(-np.inf)


def test_fixture_is_beyond_one_cta(emu, case):  # noqa: F811
    e, lens, G, w, graphs, z = case
    assert len(G["flags"]) > 4096 and len(G["src"]) > 32768  # emitting plus epsilon arcs
    assert plan(emu, G, e.shape[2])[0] == 2


def test_float64_loss_restatement_matches_the_reference(case):
    e, lens, G, w, graphs, z = case
    Z64, ge, gw = bo.restate_loss(e, lens, G, w, e.shape[2])
    assert np.allclose(Z64, z["Z"], rtol=1e-5)
    assert util.grad_close(ge, z["grad"], 50.0) and util.grad_close(gw, dense_wgrad(z, len(w)), 50.0)


def test_float32_decode_scores_match_the_reference(case):
    e, lens, G, w, graphs, z = case
    for b, n in enumerate(lens):
        assert restate_scores(e[b, :n], G, w, e.shape[2]) == z["scores"][b], b


def test_emulated_cluster_kernels_match_the_reference(emu, case):  # noqa: F811
    e, lens, G, w, graphs, z = case
    _, _, Z, grad, wgrad, status = den(emu, e, lens, G, w, 2)
    assert not status.any()
    assert np.allclose(Z, z["Z"], rtol=1e-5)
    assert util.grad_close(grad, z["grad"], 50.0) and util.grad_close(wgrad, dense_wgrad(z, len(w)), 50.0)
    _, _, scores, paths, arcs, vstatus = viterbi(emu, e, lens, G, w, 2)
    assert not vstatus.any()
    assert np.array_equal(scores, z["scores"]) and np.array_equal(paths, z["paths"]) and np.array_equal(arcs, z["arcs"])


def test_alignment_restatement_matches_the_reference(backoff_emu, case):
    """the alignment sweeps the numerators A_b o G (one CTA each): restated over the shipped builder's numerators"""
    e, lens, G, w, graphs, z = case
    Cn = e.shape[2]
    for b, g in enumerate(graphs):
        n = int(lens[b])
        P, arc_of, tidx = product(backoff_emu, g, G, Cn)
        assert len(P["flags"]) < 4096  # (the numerator fits one CTA)
        wP = np.where(arc_of < 0, w[tidx], g["w"][np.maximum(arc_of, 0)] + w[tidx]).astype(np.float32)
        score, tie, labels, parcs = bo.restate_decode(e[b, :n], P, wP, Cn)
        assert np.float32(score) == z["align_scores"][b] and not tie
        assert np.array_equal(arc_of[parcs], z["align_arcs"][b, :n]) and np.array_equal(labels, z["align_paths"][b, :n])
