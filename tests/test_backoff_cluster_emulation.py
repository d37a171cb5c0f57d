"""The backoff cluster sweeps of k_sparse.cu (sparse_cl_eps_forward / backward / viterbi: one thread-block cluster per
utterance for a backoff transition graph G too large for one CTA, the epsilon closure's levels cut over the ranks) run
from their source through the SIMT emulator (tests/emu/backoff_cluster_emu.cpp), with N = 2 and 4 CTAs of 64
threads, against the one-CTA sparse_eps_* kernels run in the same emulator on the same inputs: alpha rows, offsets,
Z, back-pointers, head, score, paths, arcs and status ==; the gradients within util.close (only the order of the adds
differs); and against the float64 loss and float32 decode restatements of tests/backoff_oracle.py.  Then the host
side: the per-level rank cuts, the balance of the splits and the envelope of sparse_cluster_plan for an epsilon G."""
import ctypes as C

import numpy as np
import pytest

from tests import backoff_oracle as bo
from tests import emu_build
from tests import graph_oracle as go
from tests import sparse_trans_oracle as st
from tests import util
from tests.test_sparse_trans_oracle import _p, graph_args

f32p, f64p, i32p, i64p, u8p, u16p = (C.POINTER(t) for t in (C.c_float, C.c_double, C.c_int32, C.c_int64, C.c_uint8,
                                                             C.c_uint16))
THREADS = 64  # per CTA of a cluster: N * 64 host threads
EPS = bo.EPS


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("backoff_cluster", ["k_sparse.cu", "gtnb_product.h"]))
    graph = [C.c_int, C.c_int, u8p, i32p, i32p, i32p]
    lib.emu_bc_plan.argtypes = graph + [C.c_int, C.c_int, i32p, i32p, i32p, i32p, i32p, i64p]
    run = [C.c_int, C.c_int, C.c_int, f32p, i32p] + graph + [f32p, C.c_int, C.c_int]
    lib.emu_bc_den.argtypes = run + [f32p, f64p, f32p, f32p, f32p, i32p]
    lib.emu_bc_viterbi.argtypes = run + [u16p, i32p, f32p, i32p, i32p, i32p]
    return lib


def _inputs(e, lens, G, w):
    _, ga = graph_args(G)
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    w = np.ascontiguousarray(w, np.float32)
    B, T, Cn = e.shape
    return [B, T, Cn, _p(e, f32p), _p(lens, i32p), len(G["flags"]), len(G["src"]), *ga, _p(w, f32p)], (e, lens, w, ga)


def den(emu, e, lens, G, w, N):
    """-> alpha [B, T + 1, S], offs [B, T + 1], den [B], grad, wgrad, status"""
    args, keep = _inputs(e, lens, G, w)
    B, T, Cn = e.shape
    S = len(G["flags"])
    out = (np.zeros((B, T + 1, S), np.float32), np.zeros((B, T + 1), np.float64), np.zeros(B, np.float32),
           np.zeros((B, T, Cn), np.float32), np.zeros(len(w), np.float32), np.zeros(B, np.int32))
    emu_build.check(emu.emu_bc_den(*args, N, THREADS, *(_p(a, t) for a, t in zip(out, (f32p, f64p, f32p, f32p, f32p,
                                                                                       i32p)))))
    return out


def viterbi(emu, e, lens, G, w, N):
    """-> bp [B, T + 1, S], head, scores, paths, arcs, status"""
    args, keep = _inputs(e, lens, G, w)
    B, T, _ = e.shape
    out = (np.zeros((B, T + 1, len(G["flags"])), np.uint16), np.zeros(B, np.int32), np.zeros(B, np.float32),
           np.zeros((B, T), np.int32), np.zeros((B, T), np.int32), np.zeros(B, np.int32))
    emu_build.check(emu.emu_bc_viterbi(*args, N, THREADS, *(_p(a, t) for a, t in zip(out, (u16p, i32p, f32p, i32p, i32p,
                                                                                           i32p)))))
    return out


def same_den(emu, e, lens, G, w, N):
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
        assert np.array_equal(one[0][b, :n + 1], cl[0][b, :n + 1]), b
    for x, y in zip(one[1:], cl[1:]):
        assert np.array_equal(x, y)
    return cl


def check(emu, e, lens, G, w, N):
    """both sweeps against the one-CTA kernels and against the restatements; -> the number of tied utterances"""
    Cn = e.shape[2]
    _, _, Z, grad, wgrad, status = same_den(emu, e, lens, G, w, N)
    assert not status.any()
    Z64, ge, gw = bo.restate_loss(e, lens, G, w, Cn)
    fin = np.isfinite(Z64)
    used = lens > 0  # (T_b = 0: the restatement leaves Z at -inf, the kernels close frame 0; the loss is NaN there)
    assert np.array_equal(np.isfinite(Z)[used], fin[used])
    assert np.allclose(Z[fin], Z64[fin], rtol=1e-5, atol=1e-4)
    mag = float(np.max(np.abs(Z64[fin]), initial=1.0)) + 5.0 * e.shape[1]
    assert util.grad_close(grad, ge, mag), float(np.abs(grad - ge).max())
    assert util.grad_close(wgrad, gw, mag * len(lens)), float(np.abs(wgrad - gw).max())
    _, _, scores, paths, arcs, vstatus = same_viterbi(emu, e, lens, G, w, N)
    ties = 0
    for b, n in enumerate(lens):
        score, tie, labels, path_arcs = bo.restate_decode(e[b, :n], G, w, Cn)
        assert np.array_equal(scores[b], np.float32(score)) and bool(vstatus[b] & 2) == tie and not vstatus[b] & 1
        ties += tie
        if np.isfinite(score) and not tie:
            assert np.array_equal(paths[b, :n], labels) and np.array_equal(arcs[b, :n], path_arcs)
        assert (paths[b, n:] == -1).all()
    return ties


def plan(emu, G, Cn, force=0):
    """-> (N, in split, out split, in arcs, out arcs per rank, cuts [2][L][N + 1], info [E, L, own_out, bwd bytes,
    max in-degree, A])"""
    args, keep = _inputs(np.zeros((1, 1, Cn)), [1], G, np.zeros(len(G["src"])))
    sp = [np.zeros(9, np.int32) for _ in range(4)]
    cut = np.zeros(2 * 33 * 9, np.int32)
    info = np.zeros(6, np.int64)
    N = emu.emu_bc_plan(*args[5:11], Cn, force, *(_p(a, i32p) for a in sp), _p(cut, i32p), _p(info, i64p))
    L = int(info[1])
    return N, sp[0][:N + 1], sp[1][:N + 1], sp[2][:N], sp[3][:N], cut[:2 * L * (N + 1)].reshape(2, L, N + 1), info


@pytest.mark.parametrize("N", [2, 4])
@pytest.mark.parametrize("order", [3, 4, 5])
def test_backoff_ngram(emu, N, order):
    """backoff n-grams of orders 3-5 (2-4 levels), ragged T_b with 0 and 1, NaN in the padding"""
    rng = np.random.default_rng(100 + 10 * order + N)
    Cn, T = 5, 7
    G, w = bo.backoff_ngram(rng, Cn, order, n_tokens=400, min_count=2)
    e = rng.uniform(-3, 3, (4, T, Cn)).astype(np.float32)
    lens = np.asarray([T, 0, 1, 5], np.int32)
    e[3, 5:] = np.nan
    check(emu, e, lens, G, w, N)


@pytest.mark.parametrize("N", [2, 4])
def test_pruned_trigram_at_small_c(emu, N):
    rng = np.random.default_rng(200 + N)
    Cn, T = 6, 6
    G, w = bo.backoff_lm(rng, C=Cn, n_bigram_arcs=3, n_trigram=12, n_trigram_arcs=2)
    e = rng.uniform(-3, 3, (3, T, Cn)).astype(np.float32)
    check(emu, e, np.asarray([T, 4, 2], np.int32), G, w, N)


@pytest.mark.parametrize("N", [2, 4])
def test_random_epsilon_dag_with_epsilon_arcs_into_start_nodes(emu, N):
    """several start and accept nodes, epsilon arcs into start nodes: the frame-0 closure improves a start node"""
    Cn, T = 5, 6
    for seed in range(300 + N, 400):  # the first seed whose G has an epsilon arc into a start node
        rng = np.random.default_rng(seed)
        G, w = bo.eps_graph(rng, 14, 45, Cn, 16, n_start=3, n_accept=3, eps_into_start=True)
        start = np.flatnonzero(G["flags"] & 1)
        eps = np.flatnonzero(G["olabel"] == EPS)
        if np.isin(G["dst"][eps], start).any():
            break
    assert np.isin(G["dst"][eps], start).any()
    e = rng.uniform(-3, 3, (3, T, Cn)).astype(np.float32)
    check(emu, e, np.asarray([T, 3, 0], np.int32), G, w, N)


def test_ranks_and_levels_without_nodes(emu):
    """a level without a node in some rank, and a rank that owns no node at all (a hub's in-list spans its share)"""
    rng = np.random.default_rng(400)
    Cn, T = 4, 5
    S = 10
    src = np.r_[rng.integers(0, S, 60), rng.integers(0, S, 12), [1, 2, 8]]
    dst = np.r_[np.full(60, 3), rng.integers(0, S, 12), [2, 9, 9]]
    lab = np.r_[rng.integers(0, Cn, 72), [EPS] * 3]
    flags = np.zeros(S, np.uint8)
    flags[[0, 1]] |= 1
    flags[[3, 9, 5]] |= 2
    G = go.make(flags, src, dst, lab)
    w = rng.uniform(-1, 1, len(src)).astype(np.float32)
    N, si, so, ai, ao, cut, info = plan(emu, G, Cn, 4)
    assert N == 4 and 0 in np.diff(si)  # a rank without nodes in the forward sweep
    fwd_sizes = np.diff(cut[0], axis=1)
    assert (fwd_sizes == 0).any()  # a level with no node in some rank
    e = rng.uniform(-3, 3, (2, T, Cn)).astype(np.float32)
    check(emu, e, np.asarray([T, 3], np.int32), G, w, 4)
    check(emu, e, np.asarray([T, 3], np.int32), G, w, 2)


@pytest.mark.parametrize("N", [2, 4])
def test_neg_inf_weights(emu, N):
    rng = np.random.default_rng(500 + N)
    Cn, T = 5, 6
    G, w = bo.backoff_ngram(rng, Cn, 3, n_tokens=400, min_count=2, n_neg_inf=6)
    e = rng.uniform(-3, 3, (3, T, Cn)).astype(np.float32)
    lens = np.asarray([T, 4, 2], np.int32)
    # the log sweeps raise the status bit on a -inf weight (the loss then retries on the exact route), as one CTA does
    assert (same_den(emu, e, lens, G, w, N)[5] == 1).all()
    _, _, scores, paths, arcs, vstatus = same_viterbi(emu, e, lens, G, w, N)
    for b, n in enumerate(lens):  # the decode forbids the arc
        score, tie, labels, path_arcs = bo.restate_decode(e[b, :n], G, w, Cn)
        assert scores[b] == np.float32(score) and not vstatus[b] & 1 and not tie
        assert np.array_equal(arcs[b, :n], path_arcs) and np.isfinite(w[arcs[b, :n]]).all()


@pytest.mark.parametrize("N", [2, 4])
def test_integer_emissions_tie_as_the_one_cta_kernel_does(emu, N):
    """integer emissions and weights: emitting candidates tie, and an epsilon candidate equals the emitting maximum"""
    rng = np.random.default_rng(600 + N)
    Cn, T = 4, 6
    G, w = bo.backoff_ngram(rng, Cn, 3, n_tokens=300, min_count=2)
    w = np.round(w).astype(np.float32)
    e = rng.integers(-2, 1, (5, T, Cn)).astype(np.float32)
    assert check(emu, e, np.asarray([6, 5, 6, 1, 3], np.int32), G, w, N) > 0
    # an epsilon arc that ties the emitting maximum at its destination: both kernels flag it the same way
    _, _, _, _, _, vs = same_viterbi(emu, e, np.asarray([6, 5, 6, 1, 3], np.int32), G, np.zeros_like(w), N)
    assert (vs & 2).any()


def test_nan_raises_the_status_bit_in_whichever_rank_meets_it(emu):
    rng = np.random.default_rng(700)
    Cn, T = 5, 6
    G, w0 = bo.backoff_ngram(rng, Cn, 4, n_tokens=400, min_count=2)
    e = rng.uniform(-3, 3, (3, T, Cn)).astype(np.float32)
    lens = np.asarray([T, T, 4], np.int32)
    eps = np.flatnonzero(G["olabel"] == EPS)
    emit = np.flatnonzero(G["olabel"] != EPS)
    for arc in (emit[0], emit[-1], eps[0], eps[-1]):
        w = w0.copy()
        w[arc] = np.nan
        for N in (2, 4):
            assert (den(emu, e, lens, G, w, N)[5] & 1).any() and np.array_equal(den(emu, e, lens, G, w, N)[5],
                                                                                 den(emu, e, lens, G, w, 1)[5])
            same_viterbi(emu, e, lens, G, w, N)


def test_cuts_partition_every_level(emu):
    rng = np.random.default_rng(800)
    for G, Cn in ((bo.backoff_ngram(rng, 6, 5, n_tokens=800, min_count=2)[0], 6),
                  (bo.eps_graph(rng, 40, 150, 7, 50)[0], 7), (bo.backoff_lm(rng, 8, 3, 30, 2)[0], 8)):
        f, b = bo.closure_levels(G)
        E = int((G["olabel"] == EPS).sum())
        for force in (2, 4, 8):
            N, si, so, ai, ao, cut, info = plan(emu, G, Cn, force)
            assert N == force and info[0] == E and info[1] == f.max()
            A = int(((G["olabel"] >= 0) & (G["olabel"] < Cn)).sum())
            assert ai.sum() == ao.sum() == A + E and info[2] == ao.max()
            for d, (split, lev) in enumerate(((si, f), (so, b))):
                for l in range(int(info[1])):
                    nodes = np.flatnonzero(lev == l + 1)  # ascending: the level's list
                    got = [np.arange(cut[d, l, r], cut[d, l, r + 1]) for r in range(N)]
                    assert np.array_equal(np.concatenate(got) - cut[d, l, 0], np.arange(len(nodes)))
                    for r in range(N):  # the share of rank r is the level's nodes in its own range
                        owned = nodes[(nodes >= split[r]) & (nodes < split[r + 1])]
                        assert len(owned) == cut[d, l, r + 1] - cut[d, l, r]
            # own epsilon out-arcs: contiguous slices of the epsilon out-table that sum to E
            eps_src = np.sort(G["src"][G["olabel"] == EPS])
            own = [((eps_src >= so[r]) & (eps_src < so[r + 1])).sum() for r in range(N)]
            assert sum(own) == E
            assert info[3] <= 227 * 1024


def test_epsilon_free_graph_keeps_its_plan(emu):
    """E = 0: the plan is the epsilon-free planner's (tests/test_sparse_cluster_emulation.py holds that one)"""
    rng = np.random.default_rng(900)
    G = st.sparse_graph(rng, 3000, 20000, 16, n_unreachable=0)
    for force in (0, 2, 4, 8):
        N, si, so, ai, ao, cut, info = plan(emu, G, 16, force)
        assert info[0] == 0 and N == (force or 2)
        for split, key in ((si, "dst"), (so, "src")):
            ptr = np.r_[0, np.cumsum(np.bincount(G[key], minlength=3000))]
            want = [0] + [int(np.searchsorted(ptr[:3000], (ptr[-1] * r + N - 1) // N)) for r in range(1, N)] + [3000]
            assert list(split) == want


def _lm_like(S, n_emit, n_eps, Cn, chain=0):
    """S nodes, n_emit emitting arcs spread over the nodes and n_eps epsilon arcs shaped like backoff arcs, node i to
    node (i - 1) // 8 (a few levels); chain > 0: instead a chain of epsilon arcs 0 -> 1 -> .. -> chain (chain levels)"""
    src = np.arange(n_emit) % S
    dst = (np.arange(n_emit) * 7 + 1) % S
    lab = np.arange(n_emit) % Cn
    es = np.arange(chain) if chain else np.arange(1, n_eps + 1)
    ed = es + 1 if chain else (es - 1) // 8
    flags = np.full(S, 2, np.uint8)
    flags[0] = 3
    return go.make(flags, np.r_[src, es], np.r_[dst, ed], np.r_[lab, np.full(len(es), EPS)])


def test_plan_envelope(emu):
    """0 just past each bound: S = 16 385, A + E = 262 145, L = 33, C = 1025; the 4-gram-sized G takes N = 2"""
    assert plan(emu, _lm_like(16384, 20000, 100, 64), 64)[0] > 0
    assert plan(emu, _lm_like(16385, 20000, 100, 64), 64)[0] == 0
    assert plan(emu, _lm_like(4096, 262144 - 1000, 1000, 64), 64)[0] == 8
    assert plan(emu, _lm_like(4096, 262145 - 1000, 1000, 64), 64)[0] == 0
    deep = _lm_like(5000, 20000, 0, 64, chain=32)
    assert plan(emu, deep, 64)[6][1] == 32 and plan(emu, deep, 64)[0] > 0
    deeper = _lm_like(5000, 20000, 0, 64, chain=33)
    assert plan(emu, deeper, 64)[6][1] == 33 and plan(emu, deeper, 64)[0] == 0
    assert plan(emu, _lm_like(5000, 20000, 100, 1024), 1024)[0] > 0
    assert plan(emu, _lm_like(5000, 20000, 100, 1025), 1025)[0] == 0
    # sized like the backoff 4-gram at C = 64 (8563 states, 57 231 + 8562 arcs): two CTAs, about 200 KB
    N, *_, info = plan(emu, _lm_like(8563, 57231, 8562, 64), 64)
    assert N == 2 and 190 * 1024 < info[3] <= 227 * 1024


@pytest.mark.parametrize("name", ["fourgram_c64", "fivegram_c64", "trigram_c128"])
def test_plans_of_real_backoff_lms(emu, name):
    """sparse_cluster_plan on the backoff LMs that DESIGN.md quotes (backoff_ngram, seed 1): cluster size and the
    backward's shared memory"""
    C, order, tokens, min_count, N, kb = {"fourgram_c64": (64, 4, 60000, 3, 2, 196.7),
                                          "fivegram_c64": (64, 5, 150000, 5, 4, 219.9),
                                          "trigram_c128": (128, 3, 200000, 3, 4, 207.9)}[name]
    G, _ = bo.backoff_ngram(np.random.default_rng(1), C, order, n_tokens=tokens, min_count=min_count)
    assert len(G["flags"]) > 4096
    got, *_, info = plan(emu, G, C)
    assert got == N and info[1] == order - 1 and round(info[3] / 1024, 1) == kb
