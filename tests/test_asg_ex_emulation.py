"""The SOURCE of gtn_b200/csrc/k_ngram.cu in ASG's start mode (the dense-trellis denominator starting from the
start weights, the forced-alignment numerator graphs built on the device) with k_implicit.cu's sweeps, run on the
CPU through the SIMT emulator of tests/emu, against the float64 referee and the C oracle (tests/asg_oracle.py).

Every batch mixes T_b in {0, 1, U-1, U, T} with one U = 0 utterance; C in {4, 28, 64, 128} covers both kernel
shapes (K = 16 entries per thread up to C = 64, 32 above), lanes per row 1 to 4 and a partial warp (C = 28)."""
import ctypes as C
import math

import numpy as np
import pytest

from tests import asg_oracle as ao
from tests import emu_build

f32p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("asg", ["k_ngram.cu", "k_implicit.cu"]))
    lib.emu_asg.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, f32p, i32p, i32p, f32p, f32p, f32p, i32p]
    return lib


def run(emu, e, tw, targets, lens=None):
    B, T, Cn = e.shape
    cat = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32) for t in targets] + [np.zeros(0, np.int32)]),
                               np.int32)
    tl = np.asarray([len(t) for t in targets], np.int32)
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    losses = np.zeros(B, np.float32)
    grads = np.zeros_like(e)
    tg = np.zeros(Cn + Cn * Cn, np.float32)
    status = np.zeros(2 * B, np.int32)
    rc = emu.emu_asg(B, T, Cn, e.ctypes.data_as(f32p), None if il is None else il.ctypes.data_as(i32p),
                     tw.ctypes.data_as(f32p), cat.ctypes.data_as(i32p), tl.ctypes.data_as(i32p),
                     losses.ctypes.data_as(f32p), grads.ctypes.data_as(f32p), tg.ctypes.data_as(f32p),
                     status.ctypes.data_as(i32p))
    emu_build.check(rc)
    return losses, grads, tg, status


def log_softmax_peaky(rng, B, T, Cn, peak=40.0):
    """log-softmax emissions with one label per frame 40 nats above the rest"""
    logits = rng.normal(0, 1, (B, T, Cn))
    logits[np.arange(B)[:, None], np.arange(T)[None, :], rng.integers(0, Cn, (B, T))] += peak
    m = logits.max(-1, keepdims=True)
    return (logits - m - np.log(np.exp(logits - m).sum(-1, keepdims=True))).astype(np.float32)


def batch(rng, T, Cn, U):
    """targets of U labels (one of them U = 0) and T_b in {0, 1, U-1, U, T}"""
    targets = [list(rng.integers(0, Cn, U)) for _ in range(5)] + [[]]
    lens = np.array([0, 1, max(U - 1, 0), U, T, T], np.int32)
    return targets, lens


def check(losses, grads, tg, e, tw, targets, lens, gtol):
    l64, g64, t64 = ao.asg_f64_batch(e, tw, targets, lens)
    lo, go, _ = ao.oracle_asg_batch(e, tw, targets, lens)
    for b in range(len(targets)):
        Tb = int(lens[b])
        if Tb > 0:  # (T_b = 0 is decided on the host: NaN, as the reference)
            if np.isinf(l64[b]):
                assert np.isposinf(losses[b]) and np.isposinf(lo[b]), (b, losses[b])
            else:
                assert math.isclose(losses[b], l64[b], rel_tol=1e-5, abs_tol=1e-4), (b, losses[b], l64[b])
                assert math.isclose(losses[b], lo[b], rel_tol=1e-5, abs_tol=1e-4), (b, losses[b], lo[b])
        assert np.abs(grads[b, :Tb] - g64[b, :Tb]).max(initial=0) < gtol, (b, np.abs(grads[b, :Tb] - g64[b, :Tb]).max())
        assert np.abs(grads[b, :Tb] - go[b, :Tb]).max(initial=0) < gtol, b
        assert not grads[b, Tb:].any()
    assert np.abs(tg - t64).max() < 1e-4 * max(1.0, np.abs(t64).max()), np.abs(tg - t64).max()


@pytest.mark.parametrize("Cn,T,U", [(4, 7, 3), (28, 9, 4), (64, 7, 3), (128, 5, 2)])
def test_asg_start_mode_kernels_match_f64(emu, oracle, Cn, T, U):
    rng = np.random.default_rng(Cn * 7 + T)
    targets, lens = batch(rng, T, Cn, U)
    B = len(targets)
    e = rng.uniform(-4, 4, (B, T, Cn)).astype(np.float32)
    tw = rng.uniform(-3, 3, Cn + Cn * Cn).astype(np.float32)
    losses, grads, tg, status = run(emu, e, tw, targets, lens)
    assert not status.any()
    check(losses, grads, tg, e, tw, targets, lens, 2e-5)


@pytest.mark.parametrize("Cn,T,U", [(4, 8, 3), (28, 8, 3), (64, 6, 3), (128, 4, 2)])
def test_asg_peaky_emissions_and_wide_transitions(emu, oracle, Cn, T, U):
    """log-softmax emissions with a 40-nat peak, start weights and matrix spread over 60 nats: every sum of the
    log-domain trellis has a term equal to 1, so nothing underflows"""
    rng = np.random.default_rng(Cn + 1000 * T)
    targets, lens = batch(rng, T, Cn, U)
    e = log_softmax_peaky(rng, len(targets), T, Cn)
    tw = rng.uniform(-30, 30, Cn + Cn * Cn).astype(np.float32)
    losses, grads, tg, status = run(emu, e, tw, targets, lens)
    assert not status.any()
    check(losses, grads, tg, e, tw, targets, lens, 1e-4)


def test_asg_all_full_length_without_input_lens(emu, oracle):
    rng = np.random.default_rng(5)
    B, T, Cn = 3, 6, 8
    targets = [[1, 2, 3], [4, 4], [7]]
    e = rng.uniform(-4, 4, (B, T, Cn)).astype(np.float32)
    tw = rng.uniform(-3, 3, Cn + Cn * Cn).astype(np.float32)
    losses, grads, tg, status = run(emu, e, tw, targets)
    assert not status.any()
    check(losses, grads, tg, e, tw, targets, np.full(B, T, np.int32), 2e-5)


@pytest.mark.parametrize("where", ["start", "matrix", "emission"])
def test_asg_non_finite_weight_raises_status(emu, where):
    Cn, T = 4, 3
    e = np.zeros((2, T, Cn), np.float32)
    tw = np.zeros(Cn + Cn * Cn, np.float32)
    if where == "start":
        tw[3] = np.inf
    elif where == "matrix":
        tw[Cn + 5] = np.nan
    else:
        e[1, 2, 3] = np.nan
    _, _, _, status = run(emu, e, tw, [[1], [2]])
    if where == "emission":
        assert not status[0] and status[1]
    else:
        assert status[:2].all()
