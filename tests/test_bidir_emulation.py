"""The SOURCE of gtn_b200/csrc/k_bidir.cu -- the criterion's bidirectional meet-in-the-middle kernel (two-CTA
clusters: alpha from the front, beta from the back, posteriors formed on the fly; TMA-staged blocks; helper
warps doing the emissions' logsumexp and the per-label sums) -- compiled with g++ against the SIMT emulator
of tests/emu/simt_emu.h (both CTAs of a cluster run concurrently) and compared with the oracle and the
float64 referee.

What this pins without a GPU: the block / phase bookkeeping (partial first and last blocks, the phase
boundary, T < 16 where one CTA has no second phase, T = 0 / 1), the mbarrier pipelines, the helper warps'
lane mapping for C = 4 .. 128, heavy labels (blank and long runs of one label), ragged input lengths,
loss-only calls, the non-finite status bit.  Speed and the compiled code are the GPU tests' business."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_build, util

f32p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build('bidir', ['k_bidir.cu', 'k_ctc.cu']))
    lib.emu_bidir_ctc.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, i32p, i32p, C.c_int, C.c_int, f32p, f32p, f32p, i32p]
    return lib


def run(lib, e, targets, lens=None, blank=0, want_grad=True, bidir_mode=-1):
    B, T, Cn = e.shape
    e = np.ascontiguousarray(e, np.float32)
    tl = np.asarray([len(t) for t in targets], np.int32)
    cat = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32) for t in targets] + [np.zeros(0, np.int32)]), np.int32)
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    out = np.zeros(B, np.float32)
    zn = np.zeros(B, np.float32)
    grad = np.zeros((B, T, Cn), np.float32) if want_grad else None
    status = np.zeros(B, np.int32)
    rc = lib.emu_bidir_ctc(B, T, Cn, e.ctypes.data_as(f32p), None if il is None else il.ctypes.data_as(i32p),
                           cat.ctypes.data_as(i32p), tl.ctypes.data_as(i32p), blank, bidir_mode, out.ctypes.data_as(f32p),
                           zn.ctypes.data_as(f32p), None if grad is None else grad.ctypes.data_as(f32p),
                           status.ctypes.data_as(i32p))
    emu_build.check(rc)
    return zn - out, grad, status


@pytest.mark.parametrize("shape", [
    (3, 40, 8, 5),     # T/2 rounds to 16: both phases in both CTAs
    (2, 9, 4, 3),      # T < 16: M = 0, CTA B has no second phase
    (2, 16, 12, 2),    # M = 8 exactly; C = 12 -> 2 labels per helper lane, some lanes beyond C
    (1, 100, 28, 10),  # BASELINE configs[0]
    (2, 37, 64, 7),    # C = 64: the benchmark's helper mapping, partial first / last blocks
    (1, 23, 128, 4),   # C = 128: 16 labels per helper lane
    (2, 1, 8, 0),      # T = 1, empty targets
    (2, 33, 8, 16),    # T = 2U + 1: a single feasible alignment per utterance
    (2, 8, 8, 2),      # T = 8: one block, everything in CTA B's first phase
    (2, 12, 64, 0),    # PAIR kernels on an empty target (one pair: the blank alone)
    (2, 20, 64, 1),    # ... and on a single label
    (1, 232, 64, 111), # ... and on the longest target they take (223 nodes: 112 pairs)
    (1, 24, 8, 3),     # T = 24: M = 16, the halves differ by a block
])
def test_bidir_kernel_source_matches_oracle(emu, oracle, shape):
    from oracle import f64
    B, T, Cn, U = shape
    e, targets = util.bench_inputs(B, T, Cn, U, seed=77 + T)
    # bidir_mode: -1 gtnb_ctc_loss's choice (C = 64 / 128: the PAIR kernels, two nodes per thread), 0 the
    # one-node-per-thread kernel on the same graphs
    for bidir_mode in ((-1,) if Cn not in (64, 128) else (-1, 0)):
        check_one(emu, oracle, f64, e, targets, B, T, bidir_mode)


def check_one(emu, oracle, f64, e, targets, B, T, bidir_mode):
    loss, grad, status = run(emu, e, targets, bidir_mode=bidir_mode)
    assert not status.any()
    for b in range(B):
        lo, go = oracle.ctc_loss(e[b], targets[b], 0, True)
        l64, g64 = f64.ctc_f64(e[b], targets[b])
        assert util.close(loss[b], lo), (b, loss[b], lo)
        assert abs(loss[b] - l64) <= 2e-6 * abs(l64) + 1e-5
        ref_err = np.abs(go - g64).max()
        my_err = np.abs(grad[b] - g64).max()
        assert my_err <= 2.0 * ref_err + 2e-6, (b, my_err, ref_err)
        assert util.grad_close(grad[b], go, 5.0 * T), b


@pytest.mark.parametrize("Cn", [8, 64])  # 64: the PAIR kernels (gtnb_ctc_loss's default)
def test_bidir_ragged_lengths_repeats_and_infeasible(emu, oracle, Cn):
    """input_lens < T (rows beyond stay untouched), long runs of one label (a second heavy label next to
    blank), blank != 0, and a target too long for its T (no accepting path: +inf loss, gradient = softmax)."""
    B, T = 5, 48
    rng = np.random.default_rng(5)
    e = rng.uniform(-5, 5, (B, T, Cn)).astype(np.float32)
    targets = [rng.integers(0, Cn - 1, 6), np.full(14, 3), rng.integers(0, Cn - 1, 9), np.full(30, 2),
               rng.integers(0, Cn - 1, 1)]
    lens = np.array([48, 45, 17, 40, 2], np.int32)
    blank = Cn - 1
    loss, grad, status = run(emu, e, targets, lens=lens, blank=blank)
    assert not status.any()
    for b in range(B):
        lo, go = oracle.ctc_loss(e[b, :lens[b]], targets[b], blank, True)
        assert util.close(loss[b], lo), (b, loss[b], lo)
        assert not grad[b, lens[b]:].any()
        if np.isfinite(lo):
            assert util.grad_close(grad[b, :lens[b]], go, 5.0 * T), b
        else:
            sm = np.exp(e[b, :lens[b]] - np.log(np.exp(e[b, :lens[b]].astype(np.float64)).sum(1, keepdims=True)))
            assert np.allclose(grad[b, :lens[b]], sm, atol=1e-6)


def test_bidir_loss_only_and_non_finite(emu, oracle):
    # C = 8: the one-node-per-thread kernel; C = 64 / 128: the PAIR kernels, which loss-only calls take too
    for Cn in (8, 64, 128):
        B, T, U = 3, 50, 6
        e, targets = util.bench_inputs(B, T, Cn, U, seed=9)
        loss, grad, status = run(emu, e, targets, want_grad=False)
        assert grad is None and not status.any()
        for b in range(B):
            lo, _ = oracle.ctc_loss(e[b], targets[b], 0, False)
            assert util.close(loss[b], lo), (Cn, b, loss[b], lo)
        e[1, 20, 3] = -np.inf
        e[2, 40, 0] = np.nan
        _, _, status = run(emu, e, targets)
        assert status[0] == 0 and status[1] == 1 and status[2] == 1, Cn


def test_bidir_benchmark_graph(emu, oracle):
    """One utterance with the benchmark's target length (U = 100: 201 nodes, 7 node warps, blank on 101 of
    them) at a T that keeps the emulation short."""
    from oracle import f64
    e, targets = util.bench_inputs(1, 260, 64, 100, seed=3)
    loss, grad, status = run(emu, e, targets)
    lo, go = oracle.ctc_loss(e[0], targets[0], 0, True)
    _, g64 = f64.ctc_f64(e[0], targets[0])
    assert not status.any() and util.close(loss[0], lo)
    assert np.abs(grad[0] - g64).max() <= 2.0 * np.abs(go - g64).max() + 2e-6
    assert np.abs(grad[0].sum(axis=1)).max() < 1e-3
