"""The device route of the asynchronous decoders from kernel source on the CPU, through the SIMT emulator of tests/emu
(tests/emu/decode_async_emu.cpp): k_ctc.cu's decode_async_prepare_kernel and decode_async_finalize_kernel alone, and
around k_sparse.cu's tropical sweep and trace as gtnb_viterbi_transitions_async chains them.

- prepare: every invalid length (negative, above T, INT_MIN, INT_MAX) sanitised to 0 with valid 0; NULL lengths give T;
  the kernel status zeroed;
- finalize: every kernel status bit alone and combined, with T_b = 0 and T_b > 0, valid and invalid: status 0 / 1 /
  2 / 3, NaN scores and -1 rows for 1 and 2 only, other rows untouched;
- the whole route on ragged lengths against the existing sparse Viterbi emulation (status 0 and 3: ==) and the live
  reference (status 0: ==): tie-heavy integer emissions flagged 3 exactly where the sweep reports a tie, NaN / +inf
  flagged 1 alone, -inf weights not flagged, an invalid length flagged 2 alone.
"""
import ctypes as C

import numpy as np
import pytest

from tests import emu_build
from tests import sparse_trans_oracle as st
from tests import sparse_viterbi_oracle as sv
from tests import test_sparse_viterbi_emulation as sve
from tests.test_sparse_trans_oracle import graph_args

f32p, i32p, u8p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("decode_async", ["k_ctc.cu", "k_sparse.cu", "gtnb_product.h"]))
    lib.emu_decode_prepare.argtypes = [C.c_int, C.c_int, i32p, i32p, i32p, i32p]
    lib.emu_decode_finalize.argtypes = [C.c_int, C.c_int, i32p, i32p, i32p, i32p, i32p, f32p, i32p]
    lib.emu_decode_route.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, C.c_int, C.c_int, u8p, i32p, i32p, i32p,
                                     f32p, i32p, i32p, f32p, i32p]
    return lib


@pytest.fixture(scope="module")
def sparse_emu():
    return sve.load()


def prepare(emu, B, T, il):
    lens, valid, ks = (np.full(B, -7, np.int32) for _ in range(3))
    ks[:] = 5
    emu_build.check(emu.emu_decode_prepare(B, T, _p(il, i32p), _p(lens, i32p), _p(valid, i32p), _p(ks, i32p)))
    return lens, valid, ks


def test_prepare_every_invalid_length(emu):
    T = 9
    il = np.asarray([0, 1, T, T + 1, -1, np.iinfo(np.int32).min, np.iinfo(np.int32).max, 4], np.int32)
    lens, valid, ks = prepare(emu, len(il), T, il)
    ok = (il >= 0) & (il <= T)
    assert np.array_equal(valid, ok.astype(np.int32))
    assert np.array_equal(lens, np.where(ok, il, 0))
    assert (ks == 0).all()
    lens, valid, ks = prepare(emu, 300, T, None)  # NULL: T for every utterance, over more than one CTA
    assert (lens == T).all() and (valid == 1).all() and (ks == 0).all()


def test_finalize_every_status_combination(emu):
    T = 5
    rows = [(tb, v, k) for tb in (0, 3) for v in (0, 1) for k in (0, 1, 2, 3)]
    B = len(rows)
    lens = np.asarray([r[0] for r in rows], np.int32)
    valid = np.asarray([r[1] for r in rows], np.int32)
    ks = np.asarray([r[2] for r in rows], np.int32)
    paths = np.arange(B * T, dtype=np.int32).reshape(B, T)
    arcs = paths + 1000
    scores = np.arange(B, dtype=np.float32) - 2.5
    status = np.full(B, -7, np.int32)
    p0, a0, s0 = paths.copy(), arcs.copy(), scores.copy()
    emu_build.check(emu.emu_decode_finalize(B, T, _p(lens, i32p), _p(ks, i32p), _p(valid, i32p), _p(paths, i32p),
                                            _p(arcs, i32p), _p(scores, f32p), _p(status, i32p)))
    for b, (tb, v, k) in enumerate(rows):
        want = 2 if not v else 0 if tb == 0 else 1 if k & 1 else 3 if k & 2 else 0
        assert status[b] == want, (b, rows[b], status[b])
        if want in (1, 2):
            assert np.isnan(scores[b]) and (paths[b] == -1).all() and (arcs[b] == -1).all()
        else:
            assert scores[b] == s0[b] and np.array_equal(paths[b], p0[b]) and np.array_equal(arcs[b], a0[b])
    # nullable rows and status
    emu_build.check(emu.emu_decode_finalize(B, T, _p(lens, i32p), _p(ks, i32p), _p(valid, i32p), None, None,
                                            _p(scores, f32p), None))


def route(emu, e, il, G, w):
    B, T, Cn = e.shape
    _, ga = graph_args(G)
    e = np.ascontiguousarray(e, np.float32)
    w = np.ascontiguousarray(w, np.float32)
    il = None if il is None else np.ascontiguousarray(il, np.int32)
    paths = np.full((B, T), -7, np.int32)
    arcs = np.full((B, T), -7, np.int32)
    scores = np.full(B, 7.0, np.float32)
    status = np.full(B, -7, np.int32)
    emu_build.check(emu.emu_decode_route(B, T, Cn, _p(e, f32p), _p(il, i32p), len(G["flags"]), len(G["src"]), *ga,
                                         _p(w, f32p), _p(paths, i32p), _p(arcs, i32p), _p(scores, f32p),
                                         _p(status, i32p)))
    return paths, arcs, scores, status


def against_sync(emu, sparse_emu, e, lens, G, w):
    """the route against the synchronous decoder's device route on the same inputs -> status"""
    p, a, s, status = route(emu, e, lens, G, w)
    sp, sa, ss, sst = sve.run(sparse_emu, e, lens, G, w)
    for b in range(e.shape[0]):
        if lens[b] == 0:
            assert status[b] == 0 and s[b] == -np.inf and (p[b] == -1).all()
            continue
        want = 1 if sst[b] & 1 else 3 if sst[b] & 2 else 0
        assert status[b] == want, (b, status[b], sst[b])
        if want == 1:
            assert np.isnan(s[b]) and (p[b] == -1).all() and (a[b] == -1).all()
        else:
            assert np.array_equal(s[b], ss[b]) and np.array_equal(p[b], sp[b]) and np.array_equal(a[b], sa[b])
    return p, a, s, status


def ragged(rng, B, T):
    lens = rng.integers(0, T + 1, B).astype(np.int32)
    lens[0], lens[1], lens[2] = T, 0, 1
    return lens


def test_route_random_graph_ragged(emu, sparse_emu):
    rng = np.random.default_rng(1)
    C = 13
    G = st.sparse_graph(rng, 11, 60, C, n_start=3, n_accept=3, label_hi=C + 2)
    e = rng.uniform(-3, 3, (9, 14, C)).astype(np.float32)
    lens = ragged(rng, 9, 14)
    for b in range(9):
        e[b, lens[b]:] = np.nan  # padding is never read
    _, _, _, status = against_sync(emu, sparse_emu, e, lens, G, rng.uniform(-1, 1, len(G["src"])).astype(np.float32))
    assert (status == 0).all()


def test_route_against_the_reference(emu, oracle):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref/libgtn_ref.so is missing")
    oracle.libref()
    rng = np.random.default_rng(2)
    C = 9
    G = st.sparse_graph(rng, 8, 40, C, n_start=2, n_accept=3, label_hi=C + 1)
    e = rng.uniform(-3, 3, (6, 10, C)).astype(np.float32)
    lens = np.asarray([10, 0, 1, 7, 10, 4], np.int32)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    p, a, s, status = route(emu, e, lens, G, w)
    pr, sr, ar = sv.ref_sparse_viterbi(e, G, w, lens)
    assert (status == 0).all()
    assert np.array_equal(s, sr) and np.array_equal(p, pr) and np.array_equal(a, ar)


def test_route_ties_are_flagged_3(emu, sparse_emu):
    rng = np.random.default_rng(3)
    C = 5
    G = st.trigram_graph(C)
    e = rng.integers(0, 2, (8, 12, C)).astype(np.float32)
    lens = ragged(rng, 8, 12)
    _, _, _, status = against_sync(emu, sparse_emu, e, lens, G, np.zeros(len(G["src"]), np.float32))
    assert (status == 3).any()


def test_route_nonfinite_and_bad_lengths_flagged_alone(emu, sparse_emu):
    rng = np.random.default_rng(4)
    C, B, T = 6, 8, 10
    G = st.sparse_graph(rng, 9, 50, C, n_start=2, n_accept=3)
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    w[::5] = -np.inf  # forbids arcs, raises nothing
    lens = np.full(B, T, np.int32)
    clean = route(emu, e, lens, G, w)
    assert (clean[3] == 0).all()
    e2, l2 = e.copy(), lens.copy()
    e2[1, 3, :] = np.nan
    e2[2, 0, :] = np.inf
    l2[3], l2[4] = -3, T + 1
    p, a, s, status = route(emu, e2, l2, G, w)
    assert list(status[1:5]) == [1, 1, 2, 2]
    for b in (1, 2, 3, 4):
        assert np.isnan(s[b]) and (p[b] == -1).all() and (a[b] == -1).all()
    for b in (0, 5, 6, 7):
        assert status[b] == 0 and s[b] == clean[2][b] and np.array_equal(p[b], clean[0][b])
        assert np.array_equal(a[b], clean[1][b])
