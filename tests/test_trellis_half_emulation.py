"""16-bit emissions in k_ngram.cu's dense trellis, k_implicit.cu's numerator sweeps and k_dense.cu's Viterbi (the native
route of gtnb_ngram_ctc_loss_typed, gtnb_asg_loss_typed and gtnb_viterbi_dense_typed), from SOURCE on the SIMT emulator.

The contract: with bfloat16 or fp16 emissions the kernels return what their float32 instantiations return on the same
emissions widened to float32.  Widening is exact and the arithmetic after the load is the float32 kernels' own, so the
sweeps' scores -- Z of both sweeps, the numerator's node scores, the status bits, Viterbi paths and scores -- are
compared with ==.  So are the transition and numerator arc gradients, which each CTA adds once per entry (the emulator
runs one CTA at a time).  The emission gradient is the one value several threads of a CTA add into (nodes of one label,
the denominator's row, with atomics in both instantiations): it is == where the order cannot matter (at most one
numerator node per label, ASG with distinct labels) and otherwise within float32 reassociation.

Also: k_implicit.cu's host check that a 16-bit lattice in a mode without a 16-bit instantiation is refused."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import emu_build, util

f32p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
F32, BF16, F16 = 0, 1, 2
TORCH = {BF16: torch.bfloat16, F16: torch.float16}
OK, ERR_LOGIC = 0, 3


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("trellis_half", ["k_ngram.cu", "k_implicit.cu", "k_dense.cu"]))
    lib.emu_trellis_typed.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, i32p, f32p, i32p, i32p,
                                      C.c_int, f32p, f32p, i32p, f32p, f32p, f32p, f32p]
    lib.emu_viterbi_dense_typed.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, i32p, C.c_int, f32p, i32p,
                                            f32p]
    return lib


def bits(t):
    """the 16-bit patterns of a bfloat16 / float16 tensor as uint16 numpy"""
    return t.contiguous().view(torch.int16).numpy().view(np.uint16)


def run_trellis(lib, asg, e, dtype, W, targets, lens=None, blank=0):
    """e: float32 [B, T, C] for F32, else uint16 bit patterns -> dict of every output of the native route"""
    B, T, Cn = e.shape
    e = np.ascontiguousarray(e)
    tl = np.asarray([len(t) for t in targets], np.int32)
    cat = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32) for t in targets] + [np.zeros(0, np.int32)]),
                               np.int32)
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    N = [(u + 1) if asg else (2 * u + 2) for u in tl]
    A = sum((2 * u) if asg else 3 * n for u, n in zip(tl, N))
    out = dict(den=np.zeros(B, np.float32), num=np.zeros(B, np.float32), status=np.zeros(2 * B, np.int32),
               grad=np.zeros((B, T, Cn), np.float32), tg=np.zeros(W.size, np.float32),
               arc=np.zeros(max(A, 1), np.float32),
               scores=np.zeros(sum((T + 1) * ((n + 3) & ~3) for n in N), np.float32))
    rc = lib.emu_trellis_typed(asg, B, T, Cn, e.ctypes.data, dtype, None if il is None else il.ctypes.data_as(i32p),
                               np.ascontiguousarray(W, np.float32).ctypes.data_as(f32p), cat.ctypes.data_as(i32p),
                               tl.ctypes.data_as(i32p), blank, *[out[k].ctypes.data_as(i32p if k == "status" else f32p)
                                                                for k in ("den", "num", "status", "grad", "tg", "arc",
                                                                          "scores")])
    emu_build.check(rc)
    return out


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def check_trellis(lib, asg, e32, dtype, W, targets, grad_exact=False, **kw):
    """the kernels on e32 rounded to dtype against the float32 kernels on those widened back"""
    th = torch.from_numpy(e32).to(TORCH[dtype])
    h = run_trellis(lib, asg, bits(th), dtype, W, targets, **kw)
    f = run_trellis(lib, asg, th.float().numpy(), F32, W, targets, **kw)
    assert np.array_equal(h["status"], f["status"])
    for k in ("den", "num", "scores", "tg", "arc"):
        assert same_bits(h[k], f[k]), k
    if grad_exact:
        assert same_bits(h["grad"], f["grad"])
    else:
        fin = np.isfinite(f["grad"])
        assert np.array_equal(fin, np.isfinite(h["grad"]))
        assert np.allclose(h["grad"][fin], f["grad"][fin], rtol=1e-5, atol=1e-6)
    return f


def inputs(B, T, Cn, U, seed, asg):
    e, targets = util.bench_inputs(B, T, Cn, U, seed=seed)
    rng = np.random.default_rng(seed)
    W = rng.uniform(-2, 2, (Cn + Cn * Cn) if asg else Cn * Cn).astype(np.float32)
    return e, targets, W


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("asg", [0, 1])
@pytest.mark.parametrize("Cn", [64, 128, 30])  # K = 16, K = 32, C not a multiple of 8
def test_trellis_half_equals_float32_on_widened_emissions(emu, dtype, asg, Cn):
    e, targets, W = inputs(2, 21, Cn, 4, 11 + Cn, asg)
    lens = np.array([21, 13], np.int32)
    f = check_trellis(emu, asg, e, dtype, W, targets, lens=lens, blank=0 if asg else Cn - 1)
    assert not f["status"].any() and np.isfinite(f["den"]).all()
    for b in range(2):
        assert not f["grad"][b, lens[b]:].any()


@pytest.mark.parametrize("dtype", [BF16, F16])
def test_asg_distinct_labels_gradient_is_bitwise(emu, dtype):
    """one numerator node per label and frame: the emission gradient has at most two addends per element, so the
    order of the atomics cannot change it and it is == too"""
    B, T, Cn = 2, 17, 64
    rng = np.random.default_rng(3)
    e = rng.uniform(-4, 4, (B, T, Cn)).astype(np.float32)
    W = rng.uniform(-2, 2, Cn + Cn * Cn).astype(np.float32)
    targets = [rng.permutation(Cn)[:5].astype(np.int32), rng.permutation(Cn)[:3].astype(np.int32)]
    check_trellis(emu, 1, e, dtype, W, targets, grad_exact=True)


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("asg", [0, 1])
def test_trellis_half_edges(emu, dtype, asg):
    """T_b in {0, 1}, U = 0, an infeasible target (+inf loss), blank != 0, long runs of one label"""
    B, T, Cn = 5, 12, 32
    rng = np.random.default_rng(7)
    e = rng.uniform(-5, 5, (B, T, Cn)).astype(np.float32)
    W = rng.uniform(-2, 2, (Cn + Cn * Cn) if asg else Cn * Cn).astype(np.float32)
    targets = [rng.integers(0, Cn - 1, 3), np.zeros(0, np.int32), rng.integers(0, Cn - 1, 14), np.full(4, 2),
               rng.integers(0, Cn - 1, 2)]
    lens = np.array([0, 1, 12, 12, 1], np.int32)
    f = check_trellis(emu, asg, e, dtype, W, targets, lens=lens, blank=5)
    assert np.isinf(f["den"][2] - f["num"][2])  # 14 labels do not fit 12 frames


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("asg", [0, 1])
@pytest.mark.parametrize("bad", [np.inf, np.nan])
def test_trellis_half_status_bit(emu, dtype, asg, bad):
    """an inf or NaN emission raises the status bits exactly as in float32 (the caller then takes the exact retry)"""
    e, targets, W = inputs(3, 15, 64, 3, 5, asg)
    e[1, 6, 0] = bad
    th = torch.from_numpy(e).to(TORCH[dtype])
    h = run_trellis(emu, asg, bits(th), dtype, W, targets)
    f = run_trellis(emu, asg, th.float().numpy(), F32, W, targets)
    assert np.array_equal(h["status"], f["status"])
    assert h["status"][1] != 0 and h["status"][0] == 0 and h["status"][2] == 0


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("bigram", [0, 1])
@pytest.mark.parametrize("Cn", [128, 30, 8])  # G = 2 (four predecessors at a time), an odd pitch, G = 32
def test_viterbi_dense_half_ties(emu, dtype, bigram, Cn):
    """integer-valued emissions and weights (exact in bf16 up to 256) make ties common: paths and scores =="""
    B, T = 3, 40
    rng = np.random.default_rng(Cn + bigram)
    e = rng.integers(-4, 5, (B, T, Cn)).astype(np.float32)
    W = rng.integers(-3, 1, (Cn * Cn) if bigram else (Cn + Cn * Cn)).astype(np.float32)
    lens = np.array([40, 17, 0], np.int32)
    res = {}
    th = torch.from_numpy(e).to(TORCH[dtype])
    assert np.array_equal(th.float().numpy(), e)
    for dt, arr in ((dtype, bits(th)), (F32, e)):
        paths = np.zeros((B, T), np.int32)
        scores = np.zeros(B, np.float32)
        rc = emu.emu_viterbi_dense_typed(B, T, Cn, np.ascontiguousarray(arr).ctypes.data, dt, lens.ctypes.data_as(i32p),
                                         bigram, W.ctypes.data_as(f32p), paths.ctypes.data_as(i32p),
                                         scores.ctypes.data_as(f32p))
        emu_build.check(rc)
        res[dt] = (paths, scores)
    assert np.array_equal(res[dtype][0], res[F32][0])
    assert same_bits(res[dtype][1], res[F32][1])
    assert (res[F32][0][2] == -1).all() and np.isneginf(res[F32][1][2])


def test_16bit_lattice_refused_outside_its_modes(emu):
    """launch_implicit_forward / _backward / _trace refuse a 16-bit lattice in a mode without a 16-bit instantiation
    (GTNB_ERR_LOGIC) instead of reading 16-bit elements as float32"""
    m = emu.emu_implicit_elem_mode
    for dt in (BF16, F16):
        assert m(dt, 0, 0, 0) == OK  # the trellis numerators' mode
        assert m(dt, 0, 1, 0) == ERR_LOGIC  # arc-label
        assert m(dt, 0, 0, 1) == ERR_LOGIC  # tropical
        assert m(dt, 0, 1, 1) == ERR_LOGIC
        G = emu.emu_wide_lanes(64, 64, 65, 64, 0)  # the dense ASG transitions graph as an implicit operand: wide
        assert G > 0 and m(dt, G, 0, 0) == ERR_LOGIC
        assert emu.emu_wide_lanes(3, 3, 102, 64, 1) == 0  # an n-gram CTC numerator (<= 3 in- / out-arcs)
    for G, arc, trop in ((0, 0, 0), (4, 1, 1), (32, 0, 1)):
        assert m(F32, G, arc, trop) == OK
    assert m(7, 0, 0, 0) == ERR_LOGIC
