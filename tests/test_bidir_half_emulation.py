"""16-bit emissions and gradients in k_bidir.cu (gtnb_ctc_loss_ex's native route), from SOURCE on the SIMT emulator.

The contract: with bfloat16 or fp16 emissions the kernel returns exactly what its float32 instantiation returns on the
same emissions widened to float32 -- losses bit-identical, gradients bit-identical to the float32 gradient rounded to
the type (to nearest, ties to even: what torch's .to() does).  Widening is exact and the arithmetic between the
typed load and the typed store is the float32 kernel's own, so nothing here needs a tolerance.

Also: the host forms of gtnb_ptx.h's conversions against torch's CPU conversions on NaN, infinities, subnormals,
ties and the largest finite values."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import emu_build, util

f32p, i32p, u16p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint16)
F32, BF16, F16 = 0, 1, 2
TORCH = {BF16: torch.bfloat16, F16: torch.float16}


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build('bidir_half', ['k_bidir.cu', 'k_ctc.cu']))
    lib.emu_bidir_ctc_ex.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, i32p, i32p, i32p, C.c_int, C.c_int,
                                     f32p, f32p, C.c_void_p, i32p]
    lib.emu_f32_to_16.argtypes = [f32p, u16p, C.c_int, C.c_longlong]
    lib.emu_16_to_f32.argtypes = [u16p, f32p, C.c_int, C.c_longlong]
    lib.emu_stg_elem4.argtypes = [f32p, u16p, C.c_int]
    return lib


def bits(t):
    """the 16-bit patterns of a bfloat16 / float16 tensor as uint16 numpy"""
    return t.contiguous().view(torch.int16).numpy().view(np.uint16)


def run(lib, e, dtype, targets, lens=None, blank=0, want_grad=True, bidir_mode=-1):
    """e: float32 [B, T, C] for F32, else uint16 bit patterns -> (losses, grad (float32 or uint16), status)"""
    B, T, Cn = e.shape
    e = np.ascontiguousarray(e)
    tl = np.asarray([len(t) for t in targets], np.int32)
    cat = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32) for t in targets] + [np.zeros(0, np.int32)]), np.int32)
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    out = np.zeros(B, np.float32)
    zn = np.zeros(B, np.float32)
    grad = np.zeros((B, T, Cn), e.dtype) if want_grad else None
    status = np.zeros(B, np.int32)
    rc = lib.emu_bidir_ctc_ex(B, T, Cn, e.ctypes.data, dtype, None if il is None else il.ctypes.data_as(i32p),
                              cat.ctypes.data_as(i32p), tl.ctypes.data_as(i32p), blank, bidir_mode,
                              out.ctypes.data_as(f32p), zn.ctypes.data_as(f32p), None if grad is None else grad.ctypes.data,
                              status.ctypes.data_as(i32p))
    emu_build.check(rc)
    return zn - out, grad, status


def check_contract(lib, e32, dtype, targets, **kw):
    """e32: float32 emissions; the kernel runs on them rounded to dtype, the float32 kernel on those widened back"""
    th = torch.from_numpy(e32).to(TORCH[dtype])
    loss_h, grad_h, st_h = run(lib, bits(th), dtype, targets, **kw)
    loss_f, grad_f, st_f = run(lib, th.float().numpy(), F32, targets, **kw)
    assert np.array_equal(st_h, st_f)
    assert np.array_equal(loss_h.view(np.uint32), loss_f.view(np.uint32)), (loss_h, loss_f)
    if grad_f is None:
        assert grad_h is None
    else:
        assert np.array_equal(grad_h, bits(torch.from_numpy(grad_f).to(TORCH[dtype])))
    return loss_f, grad_f, st_f


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("shape,bidir_mode", [
    ((2, 37, 64, 7), -1),   # C = 64: the PAIR kernel, partial first / last blocks
    ((2, 37, 64, 7), 0),    # ... one node per thread, FX
    ((1, 23, 128, 4), -1),  # C = 128: the PAIR kernel, two chunks per helper lane
    ((1, 23, 128, 4), 0),
    ((2, 40, 32, 5), -1),   # C = 32: not FX, the generic helper block
    ((2, 9, 8, 3), -1),     # C = 8, T < 16: CTA B has no second phase
])
def test_half_kernel_equals_float32_kernel_on_widened_emissions(emu, dtype, shape, bidir_mode):
    B, T, Cn, U = shape
    e, targets = util.bench_inputs(B, T, Cn, U, seed=31 + T)
    _, _, status = check_contract(emu, e, dtype, targets, bidir_mode=bidir_mode)
    assert not status.any()


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("Cn", [16, 64])  # 64: the PAIR kernel
def test_half_ragged_lengths_repeats_and_infeasible(emu, oracle, dtype, Cn):
    """input_lens < T (padding rows stay untouched by the kernel), long runs of one label, blank != 0, and a target
    too long for its T (no accepting path: +inf loss)"""
    B, T = 5, 48
    rng = np.random.default_rng(5)
    e = rng.uniform(-5, 5, (B, T, Cn)).astype(np.float32)
    targets = [rng.integers(0, Cn - 1, 6), np.full(14, 3), rng.integers(0, Cn - 1, 9), np.full(30, 2),
               rng.integers(0, Cn - 1, 1)]
    lens = np.array([48, 45, 17, 40, 2], np.int32)
    loss, grad, status = check_contract(emu, e, dtype, targets, lens=lens, blank=Cn - 1)
    assert not status.any()
    assert np.isinf(loss[3]) and np.isfinite(loss[[0, 1, 2, 4]]).all()
    for b in range(B):
        assert not grad[b, lens[b]:].any()


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("Cn", [8, 64, 128])
def test_half_loss_only(emu, dtype, Cn):
    e, targets = util.bench_inputs(3, 50, Cn, 6, seed=9)
    _, grad, status = check_contract(emu, e, dtype, targets, want_grad=False)
    assert grad is None and not status.any()


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("Cn", [8, 64])
def test_half_non_finite_raises_the_status_bit(emu, dtype, Cn):
    """a -inf or NaN emission raises the utterance's status bit exactly as in the float32 kernel (the caller then
    repeats the batch on the exact route)"""
    B, T, U = 3, 50, 6
    e, targets = util.bench_inputs(B, T, Cn, U, seed=9)
    e[1, 20, 3] = -np.inf
    e[2, 40, 0] = np.nan
    th = torch.from_numpy(e).to(TORCH[dtype])
    _, _, st_h = run(emu, bits(th), dtype, targets)
    _, _, st_f = run(emu, th.float().numpy(), F32, targets)
    assert list(st_h) == [0, 1, 1] and np.array_equal(st_h, st_f)


def special_values():
    """NaN, +-inf, zeros, float32 and 16-bit subnormals, ties at both types' rounding points, the largest finite
    values and the overflow thresholds, plus random bit patterns"""
    f = np.float32
    v = [np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0, -1.0, 1e-45, -1e-45, 1.17549435e-38, 1.1754942e-38,
         np.finfo(f).max, -np.finfo(f).max, 65504.0, 65519.996, 65520.0, -65520.0, 65536.0, 3.3895314e38, 3.3961776e38,
         2.0 ** -24, 2.0 ** -25, 2.0 ** -25 * 1.0000001, 3 * 2.0 ** -25, 2.0 ** -14, 2.0 ** -14 * (1 - 2.0 ** -11),
         6.0e-8, 5.96e-8, 1e-7, 3.0517578e-05, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -11,
         1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -11 + 2.0 ** -20, 2049.0, 2051.0, 257.0, 259.0]
    rng = np.random.default_rng(0)
    rnd = rng.integers(0, 2 ** 32, 20000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    ties = (rng.integers(0, 2 ** 16, 4000, dtype=np.uint32) << 16 | 0x8000).view(np.float32)  # bf16 ties
    ties16 = ((rng.integers(0x33000000 >> 13, 0x47800000 >> 13, 4000, dtype=np.uint32) << 13) | 0x1000).view(np.float32)
    return np.concatenate([np.asarray(v, f), rnd, ties, ties16, -ties16])


@pytest.mark.parametrize("dtype", [BF16, F16])
def test_host_conversions_match_torch(emu, dtype):
    x = special_values()
    got = np.zeros(x.size, np.uint16)
    emu.emu_f32_to_16(x.ctypes.data_as(f32p), got.ctypes.data_as(u16p), dtype, x.size)
    want = bits(torch.from_numpy(x).to(TORCH[dtype]))
    nan = np.isnan(x)
    assert np.array_equal(got[~nan], want[~nan]), np.flatnonzero(got[~nan] != want[~nan])[:10]
    # NaN stays NaN (torch canonicalises the payload, the conversion here keeps the sign and quiets it)
    back = np.zeros(x.size, np.float32)
    emu.emu_16_to_f32(got.ctypes.data_as(u16p), back.ctypes.data_as(f32p), dtype, x.size)
    assert np.isnan(back[nan]).all()
    # widening is exact: every 16-bit pattern comes back as torch widens it
    allp = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    wide = np.zeros(allp.size, np.float32)
    emu.emu_16_to_f32(allp.ctypes.data_as(u16p), wide.ctypes.data_as(f32p), dtype, allp.size)
    ref = torch.from_numpy(allp.view(np.int16)).view(TORCH[dtype]).float().numpy()
    fin = ~np.isnan(ref)
    assert np.array_equal(wide[fin].view(np.uint32), ref[fin].view(np.uint32))
    assert np.isnan(wide[~fin]).all()
    # the packed store of four floats rounds each exactly as the scalar conversion does, first element lowest
    for k in range(0, 64, 4):
        out = np.zeros(4, np.uint16)
        emu.emu_stg_elem4(x[k:k + 4].ctypes.data_as(f32p), out.ctypes.data_as(u16p), dtype)
        assert np.array_equal(out, got[k:k + 4])
