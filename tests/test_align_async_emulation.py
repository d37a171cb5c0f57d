"""The whole device route of the asynchronous forced alignments (gtnb_ctc_align_async, gtnb_ngram_ctc_align_async,
gtnb_asg_align_async) from kernel source on the CPU, through the SIMT emulator of tests/emu: the prepare kernel, the
numerator build (n-gram: tau, then the build with tau in place of sigma), k_implicit.cu's tropical forward and trace,
and align_async_finalize_kernel.  Against the live reference (oracle/_ref) and a float32 restatement
(tests/align_async_oracle.py):

- scores bit-equal to the reference's wherever the status is 0 or 3;
- paths and tokens == the reference's wherever the status is 0, the tokens derived from the reference's arcs;
- status 3 exactly where the restatement finds a tie on the traced path, and then an optimal, valid path;
- status 2 for each invalid length or label, status 1 for inf / NaN emissions and NaN transitions, with a NaN score and
  -1 rows, and the other utterances unaffected;
- ragged lengths, T_b in {0, 1}, U = 0, an infeasible target, repeats, blank != 0, C in {4, 29, 64, 128, 256}, and
  tie-heavy integer emissions.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import align_async_oracle as ao
from tests import emu_build
from tests import test_ctc_async_emulation as ca
from tests import test_trellis_async_emulation as ta

f32p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
CTC, NGRAM, ASG = ao.CTC, ao.NGRAM, ao.ASG


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("align_async", ["k_ctc.cu", "k_implicit.cu", "k_ngram.cu"]))
    lib.emu_align_async.argtypes = [C.c_int] * 7 + [C.POINTER(ca.GraphMeta), f32p, f32p, i32p, i32p, i32p, C.c_int,
                                                    i32p, i32p, f32p, i32p]
    return lib


@pytest.fixture(scope="module")
def ref():
    if not po.have_ref():
        pytest.skip("oracle/_ref/libgtn_ref.so is missing")


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def bound(kind, B, T, C_, S):
    """(m01, N, A): composed_alloc's descriptors of utterances 0 and 1 at the bounds, and the bound numerator's size"""
    if kind == CTC:
        N, A = ca.bound_dims(S)
        return ca.m01(B, T, C_, S), N, A
    N, A, _ = ta.dims(kind == ASG, S, max(S - 1, 0))
    return ta.m01(kind == ASG, B, T, C_, S), N, A


def run(lib, kind, e, W, targets, lens, il, blank):
    B, T, C_ = e.shape
    S = targets.shape[1]
    m01, N, A = bound(kind, B, T, C_, S)
    paths = np.full((B, T), -7, np.int32)
    tokens = np.full((B, T), -7, np.int32)
    scores = np.full(B, 7.0, np.float32)
    status = np.full(B, -7, np.int32)
    e = np.ascontiguousarray(e, np.float32)
    W = None if W is None else np.ascontiguousarray(W, np.float32)
    emu_build.check(lib.emu_align_async(kind, B, T, C_, S, N, A, m01, _p(e, f32p), _p(W, f32p),
                                        _p(il, i32p), _p(np.ascontiguousarray(targets, np.int32), i32p),
                                        _p(np.ascontiguousarray(lens, np.int32), i32p), blank, _p(paths, i32p),
                                        _p(tokens, i32p), _p(scores, f32p), _p(status, i32p)))
    return paths, tokens, scores, status


def transitions(kind, C_, rng, integer=False):
    if kind == CTC:
        return None
    n = C_ * C_ + (C_ if kind == ASG else 0)
    return (rng.integers(-2, 1, n) if integer else rng.normal(0, 1, n)).astype(np.float32)


def batch(kind, B, T, C_, S, blank, rng, integer=False):
    """ragged targets without the blank label (ctc_graph and ctcGraph agree there), with repeats, U = 0, T_b = 0 and 1,
    and one target too long for its frames"""
    labels = np.array([c for c in range(C_) if kind == ASG or c != blank], np.int32)
    targets = labels[rng.integers(0, len(labels), (B, S))]
    lens = rng.integers(0, S + 1, B).astype(np.int32)
    il = rng.integers(0, T + 1, B).astype(np.int32)
    if B >= 6 and S >= 3:
        lens[0], il[0] = S, T
        targets[1, 1] = targets[1, 0]  # a repeat
        lens[1] = max(lens[1], 2)
        lens[2] = 0  # U = 0
        il[3] = 0  # T_b = 0
        il[4], lens[4] = 1, 1  # T_b = 1
        lens[5], il[5] = S, 1 if kind == ASG else 2  # infeasible: more labels than frames allow
        targets[5, :] = targets[5, 0]  # (CTC: repeats need blanks between them)
    if integer:
        e = rng.integers(-3, 1, (B, T, C_)).astype(np.float32)
    else:
        e = rng.normal(0, 2, (B, T, C_)).astype(np.float32)
    return e, targets, lens, il


def check_against_reference(kind, e, W, targets, lens, il, blank, out):
    paths, tokens, scores, status = out
    B, T, _ = e.shape
    rp, rt, rs = ao.reference(kind, e, W, targets, lens, il, blank)
    counts = {0: 0, 3: 0}
    for b in range(B):
        Tb = T if il is None else int(il[b])
        y = targets[b, :lens[b]]
        assert status[b] in (0, 3), (b, status[b])
        assert scores[b] == rs[b] or (np.isneginf(scores[b]) and np.isneginf(rs[b])), (b, scores[b], rs[b])
        want_score, want_tie = ao.restated(kind, e[b, :Tb], W, y, blank)
        assert scores[b] == want_score or (np.isneginf(scores[b]) and np.isneginf(want_score)), b
        assert (status[b] == 3) == bool(want_tie), (b, status[b], want_tie)
        counts[int(status[b])] += 1
        if status[b] == 0:
            assert np.array_equal(paths[b], rp[b]), b
            assert np.array_equal(tokens[b], rt[b]), b
        else:  # an optimal, valid path; its value is the score
            assert ao.valid_path(kind, paths[b, :Tb], tokens[b, :Tb], y, blank), b
            assert ao.path_value(kind, e[b, :Tb], W, paths[b, :Tb]) == scores[b], b
            assert (paths[b, Tb:] == -1).all() and (tokens[b, Tb:] == -1).all()
        if not np.isfinite(scores[b]):
            assert (paths[b] == -1).all() and (tokens[b] == -1).all(), b
    return counts


@pytest.mark.parametrize("kind", [CTC, NGRAM, ASG])
@pytest.mark.parametrize("C_,blank", [(4, 0), (29, 3), (64, 0), (128, 127), (256, 5)])
def test_route_matches_reference(emu, ref, kind, C_, blank):
    rng = np.random.default_rng(1000 * kind + C_)
    B, T, S = 8, 14, 5
    e, targets, lens, il = batch(kind, B, T, C_, S, blank, rng)
    W = transitions(kind, C_, rng)
    out = run(emu, kind, e, W, targets, lens, il, blank)
    check_against_reference(kind, e, W, targets, lens, il, blank, out)
    assert np.isneginf(out[2][3]) and (out[0][3] == -1).all()  # T_b = 0
    assert np.isneginf(out[2][5])  # the infeasible target
    # without input lengths: T_b = T
    out = run(emu, kind, e, W, targets, lens, None, blank)
    check_against_reference(kind, e, W, targets, lens, None, blank, out)


@pytest.mark.parametrize("kind", [CTC, NGRAM, ASG])
def test_ties_on_integer_emissions(emu, ref, kind):
    rng = np.random.default_rng(77 + kind)
    B, T, C_, S = 12, 12, 4, 4
    e, targets, lens, il = batch(kind, B, T, C_, S, 0, rng, integer=True)
    lens[6:], il[6:] = S, T  # full-length utterances: many optimal paths
    W = transitions(kind, C_, rng, integer=True)
    counts = check_against_reference(kind, e, W, targets, lens, il, 0, run(emu, kind, e, W, targets, lens, il, 0))
    assert counts[3] > 0, counts  # the restatement's ties are what raised them


@pytest.mark.parametrize("kind", [CTC, NGRAM, ASG])
def test_invalid_and_non_finite_utterances_are_flagged_alone(emu, ref, kind):
    rng = np.random.default_rng(5 + kind)
    B, T, C_, S, blank = 10, 10, 6, 3, 0
    e, targets, lens, il = batch(kind, B, T, C_, S, blank, rng)
    targets[:] = rng.integers(1, C_, (B, S))
    lens[:], il[:] = S, T
    W = transitions(kind, C_, rng)
    lens[1] = -1  # U < 0
    lens[2] = S + 1  # U > S
    il[3] = T + 1  # T_b > T
    il[4] = -1  # T_b < 0
    targets[5, 1] = C_  # a label >= C
    targets[6, 0] = -2  # a negative label
    e[7, 2, :] = np.inf  # non-finite emissions in a used frame
    e[8, 4, targets[8, 0]] = np.nan  # (a label of the numerator: the sweep reads only those)
    out = run(emu, kind, e, W, targets, lens, il, blank)
    paths, tokens, scores, status = out
    assert status.tolist()[1:9] == [2] * 6 + [1, 1], status
    for b in range(1, 9):
        assert np.isnan(scores[b]) and (paths[b] == -1).all() and (tokens[b] == -1).all(), b
    # the rest equal a run of the batch without the flagged ones
    keep = [0, 9]
    alone = run(emu, kind, e[keep], W, targets[keep], lens[keep], il[keep], blank)
    for k, b in enumerate(keep):
        assert status[b] == alone[3][k] and scores[b] == alone[2][k], b
        assert np.array_equal(paths[b], alone[0][k]) and np.array_equal(tokens[b], alone[1][k]), b
    if kind != CTC:  # a NaN transition weight that utterance 0's path must take: its first arc's
        W2 = W.copy()
        y0 = int(targets[0, 0])
        if kind == ASG:
            W2[y0] = np.nan
        else:
            W2[y0 * C_:(y0 + 1) * C_] = np.nan  # tau_y0 is NaN
        out = run(emu, kind, e[[0]], W2, targets[[0]], lens[[0]], il[[0]], blank)
        assert out[3][0] == 1 and np.isnan(out[2][0]) and (out[0][0] == -1).all(), out
