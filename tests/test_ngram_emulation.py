"""The SOURCE of gtn_b200/csrc/k_ngram.cu (CTC with a learned bigram transition graph: the dense-trellis
denominator, the folded numerator graphs, the sigma fold) with k_implicit.cu's sweeps, run on the CPU through
the SIMT emulator of tests/emu, against the C oracle (no fold) and the float64 referee.

The shapes cover both kernel shapes (K = 16 entries per thread for C <= 64, 32 above), lanes per row 1 to 4,
partial warps (C = 28: 56 threads), T in {0, 1, small}, ragged input_lens, U = 0, repeated labels, an
infeasible target and blank != 0."""
import ctypes as C
import math

import numpy as np
import pytest

from tests import emu_build
from tests import ngram_oracle as no

f32p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("ngram", ["k_ngram.cu", "k_implicit.cu"]))
    lib.emu_ngram_ctc.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, f32p, i32p, i32p, C.c_int, f32p, f32p, f32p,
                                  i32p]
    return lib


def run(emu, e, W, targets, blank, lens=None):
    B, T, Cn = e.shape
    cat = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32) for t in targets] + [np.zeros(0, np.int32)]),
                               np.int32)
    tl = np.asarray([len(t) for t in targets], np.int32)
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    losses = np.zeros(B, np.float32)
    grads = np.zeros_like(e)
    tg = np.zeros(Cn * Cn, np.float32)
    status = np.zeros(2 * B, np.int32)
    rc = emu.emu_ngram_ctc(B, T, Cn, e.ctypes.data_as(f32p), None if il is None else il.ctypes.data_as(i32p),
                           W.ctypes.data_as(f32p), cat.ctypes.data_as(i32p), tl.ctypes.data_as(i32p), blank,
                           losses.ctypes.data_as(f32p), grads.ctypes.data_as(f32p), tg.ctypes.data_as(f32p),
                           status.ctypes.data_as(i32p))
    emu_build.check(rc)
    return losses, grads, tg, status


def random_targets(rng, B, Cn, blank, max_u):
    labels = [c for c in range(Cn) if c != blank]
    return [list(rng.choice(labels, size=int(rng.integers(0, max_u + 1)))) for _ in range(B)]


CASES = [  # B, T, C, blank, max U
    (3, 1, 4, 0, 1),
    (3, 6, 4, 3, 2),
    (3, 9, 8, 5, 3),
    (2, 7, 28, 0, 3),
    (2, 5, 64, 7, 2),
    (2, 4, 100, 1, 2),
    (1, 3, 128, 0, 1),
]


@pytest.mark.parametrize("shape", CASES)
def test_ngram_kernels_match_oracle(emu, oracle, shape):
    B, T, Cn, blank, max_u = shape
    rng = np.random.default_rng(Cn * 31 + T)
    e = rng.uniform(-4, 4, (B, T, Cn)).astype(np.float32)
    W = rng.uniform(-3, 3, Cn * Cn).astype(np.float32)
    targets = random_targets(rng, B, Cn, blank, max_u)
    lens = np.array([T - (b % 3) for b in range(B)], np.int32).clip(0, T)
    losses, grads, tg, status = run(emu, e, W, targets, blank, lens)
    assert not status.any()
    want_tg = np.zeros(Cn * Cn)
    for b in range(B):
        Tb = int(lens[b])
        lo, go, tgo = no.oracle_ngram_ctc(e[b, :Tb], W, targets[b], blank)
        lf, gf, tgf = no.ngram_ctc_f64(e[b, :Tb], W, targets[b], blank)
        want_tg += tgf
        if Tb > 0:  # (T_b = 0 is decided on the host: NaN, as the reference)
            assert math.isclose(losses[b], lo, rel_tol=1e-5, abs_tol=1e-4) or (np.isinf(lo) and np.isinf(losses[b])), \
                (b, losses[b], lo)
        assert np.abs(grads[b, :Tb] - gf).max(initial=0) < 2e-5, b
        assert np.abs(grads[b, :Tb] - go).max(initial=0) < 2e-5, b
        assert not grads[b, Tb:].any()
    assert np.abs(tg - want_tg).max() < 1e-4 * max(1.0, np.abs(want_tg).max())


def test_ngram_edge_cases_match_oracle(emu, oracle):
    """U = 0, T_b = 0, repeated labels (no skip arc), an infeasible target, blank != 0, in one batch"""
    Cn, T, blank = 6, 5, 2
    rng = np.random.default_rng(7)
    targets = [[], [1, 1, 1], [3, 3], [4, 1, 5, 0], [1], [5, 4, 3, 1, 0, 1]]
    lens = np.array([5, 5, 0, 5, 1, 5], np.int32)  # [3,3] at T_b = 0; 6 labels in 5 frames: infeasible
    B = len(targets)
    e = rng.uniform(-4, 4, (B, T, Cn)).astype(np.float32)
    W = rng.uniform(-3, 3, Cn * Cn).astype(np.float32)
    losses, grads, tg, status = run(emu, e, W, targets, blank, lens)
    assert not status.any()
    want_tg = np.zeros(Cn * Cn)
    for b in range(B):
        Tb = int(lens[b])
        lo, go, _ = no.oracle_ngram_ctc(e[b, :Tb], W, targets[b], blank)
        _, gf, tgf = no.ngram_ctc_f64(e[b, :Tb], W, targets[b], blank)
        want_tg += tgf
        if Tb > 0:
            assert (np.isinf(lo) and np.isinf(losses[b])) or math.isclose(losses[b], lo, rel_tol=1e-5, abs_tol=1e-4)
        assert np.abs(grads[b, :Tb] - gf).max(initial=0) < 2e-5
    assert np.isinf(losses[5])  # the infeasible target: +inf, and the denominator's gradient alone
    assert np.abs(tg - want_tg).max() < 1e-4


def test_ngram_peaky_emissions_and_wide_w(emu, oracle):
    """log-softmax emissions with one dominant label per frame and W spread over ~60 nats: the log-domain
    trellis has no underflow to lose (every sum has a term equal to 1)"""
    B, T, Cn, blank = 2, 12, 16, 0
    rng = np.random.default_rng(3)
    logits = rng.normal(0, 1, (B, T, Cn))
    logits[np.arange(B)[:, None], np.arange(T)[None, :], rng.integers(0, Cn, (B, T))] += 40.0
    e = (logits - np.log(np.exp(logits - logits.max(-1, keepdims=True)).sum(-1, keepdims=True))
         - logits.max(-1, keepdims=True)).astype(np.float32)
    W = rng.uniform(-30, 30, Cn * Cn).astype(np.float32)
    targets = [[3, 5, 5], [1, 2]]
    losses, grads, tg, status = run(emu, e, W, targets, blank)
    want_tg = np.zeros(Cn * Cn)
    for b in range(B):
        lf, gf, tgf = no.ngram_ctc_f64(e[b], W, targets[b], blank)
        want_tg += tgf
        assert math.isclose(losses[b], lf, rel_tol=1e-5, abs_tol=1e-3), (losses[b], lf)
        assert np.abs(grads[b] - gf).max() < 1e-4
    assert np.abs(tg - want_tg).max() < 1e-4 * max(1.0, np.abs(want_tg).max())


def test_ngram_non_finite_weight_raises_status(emu):
    Cn, T = 4, 3
    e = np.zeros((2, T, Cn), np.float32)
    W = np.zeros(Cn * Cn, np.float32)
    W[5] = np.inf
    _, _, _, status = run(emu, e, W, [[1], [2]], 0)
    assert status[:2].all()
    W[5] = 0.0
    e[1, 2, 3] = np.nan
    _, _, _, status = run(emu, e, W, [[1], [2]], 0)
    assert not status[0] and status[1]
