"""gtnb_ctc_loss_ex with bfloat16 / fp16 emissions and gradients, and torch ctc_loss on 16-bit tensors, on the GPU.

The contract: the losses are gtnb_ctc_loss's on the emissions widened to float32, bit for bit, and the gradient is
that call's float32 gradient rounded to the dtype (what torch's .to() does), on every route -- k_bidir.cu reading
the 16-bit buffers in place, and the widened route (C > 128, C % 8 != 0, misaligned buffers, other flags, the exact
retry after a non-finite value).  So every comparison here is ==, with NaN equal to NaN."""
import numpy as np
import pytest
import torch

from gtn_b200 import capi
from tests import util

pytestmark = pytest.mark.gpu
F32, BF16, F16 = capi.F32, capi.BF16, capi.F16
TORCH = {BF16: torch.bfloat16, F16: torch.float16}
DTYPES = [BF16, F16]


@pytest.fixture(scope="module")
def hctx():
    c = capi.Ctx(0)
    yield c
    c.close()


def call_ex(ctx, e, dtype, targets, blank=0, lens=None, want_grad=True, grad=None):
    """gtnb_ctc_loss_ex on the device tensor e -> (losses, grad tensor or None); grad starts as NaN everywhere so
    that rows the call must write (or zero) show up"""
    B, T, Cn = e.shape
    cat, tl = capi._cat_targets(targets)
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    losses = np.zeros(B, np.float32)
    if want_grad and grad is None:
        grad = torch.full_like(e, float("nan"))
    torch.cuda.synchronize()
    ctx._check(capi.lib().gtnb_ctc_loss_ex(
        ctx.h, B, T, Cn, e.data_ptr(), dtype, None if il is None else il.ctypes.data_as(capi._i32p),
        cat.ctypes.data_as(capi._i32p), tl.ctypes.data_as(capi._i32p), blank, losses.ctypes.data_as(capi._f32p),
        grad.data_ptr() if want_grad else None))
    return losses, grad if want_grad else None


def call_f32(ctx, e32, targets, blank=0, lens=None, want_grad=True):
    """gtnb_ctc_loss on device float32 buffers"""
    B, T, Cn = e32.shape
    cat, tl = capi._cat_targets(targets)
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    losses = np.zeros(B, np.float32)
    grad = torch.full_like(e32, float("nan")) if want_grad else None
    torch.cuda.synchronize()
    ctx._check(capi.lib().gtnb_ctc_loss(
        ctx.h, B, T, Cn, e32.data_ptr(), 1, None if il is None else il.ctypes.data_as(capi._i32p),
        cat.ctypes.data_as(capi._i32p), tl.ctypes.data_as(capi._i32p), blank, losses.ctypes.data_as(capi._f32p),
        grad.data_ptr() if want_grad else None, 1))
    return losses, grad


def same(a, b):
    """== with NaN equal to NaN (float32 numpy arrays or tensors of one dtype)"""
    a = torch.as_tensor(a).cpu()
    b = torch.as_tensor(b).cpu()
    assert a.dtype == b.dtype and a.shape == b.shape
    return bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def half_inputs(B, T, Cn, U, dtype, seed=1234):
    e, tg = util.bench_inputs(B, T, Cn, U, seed)
    return torch.from_numpy(e).cuda().to(TORCH[dtype]), tg


def check_contract(ctx, eh, dtype, targets, **kw):
    """eh: a 16-bit device tensor; returns (losses, float32 grad) of the float32 call on eh.float()"""
    lh, gh = call_ex(ctx, eh, dtype, targets, **kw)
    lf, gf = call_f32(ctx, eh.float().contiguous(), targets, blank=kw.get("blank", 0), lens=kw.get("lens"),
                      want_grad=kw.get("want_grad", True))
    assert same(lh, lf), (lh, lf)
    if gf is not None:
        assert gh.dtype == eh.dtype and same(gh, gf.to(eh.dtype))
    return lf, gf


def reset_flags(ctx):
    ctx.set_flag("bidir_mode", -1)
    ctx.set_flag("bidir", -1)
    ctx.set_flag("implicit", 1)


def kernels_of(ctx, fn):
    """fn() with the context's launch profile on -> the names of the kernels it launched"""
    ctx.profile(True)
    ctx.profile_read()
    fn()
    names = set(ctx.profile_read())
    ctx.profile(False)
    return names


@pytest.mark.parametrize("dtype", DTYPES)
def test_benchmark_shape_native(hctx, dtype):
    """B=256 T=1000 C=64 U=100: the PAIR kernel on the 16-bit buffers, no conversion kernel"""
    eh, tg = half_inputs(256, 1000, 64, 100, dtype)
    names = kernels_of(hctx, lambda: check_contract(hctx, eh, dtype, tg))
    assert "bidir_ctc" in names and "widen" not in names and "narrow" not in names, names
    # loss only
    check_contract(hctx, eh[:16], dtype, tg[:16], want_grad=False)


@pytest.mark.parametrize("dtype", DTYPES)
def test_c128_native(hctx, dtype):
    eh, tg = half_inputs(16, 300, 128, 40, dtype, seed=5)
    names = kernels_of(hctx, lambda: check_contract(hctx, eh, dtype, tg))
    assert "bidir_ctc" in names and "widen" not in names, names


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Cn", [64, 32])
def test_ragged_lengths_zero_the_padding(hctx, dtype, Cn):
    B, T = 12, 200
    eh, tg = half_inputs(B, T, Cn, 20, dtype, seed=11)
    lens = np.random.default_rng(3).integers(0, T + 1, B).astype(np.int32)
    lens[0], lens[1] = T, 5  # full length; shorter than the target (infeasible: +inf)
    check_contract(hctx, eh, dtype, tg, lens=lens)
    _, gh = call_ex(hctx, eh, dtype, tg, lens=lens)
    for b in range(B):
        assert not gh[b, lens[b]:].float().abs().sum().item() and not torch.isnan(gh[b, lens[b]:]).any()


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_bidir_mode_and_route_flag(hctx, dtype):
    """bidir_mode -1 / 1 (PAIR), 0 (one node per thread); bidir 0 (two sweeps of k_implicit.cu) and implicit 0
    (materialised), which read the widened copy"""
    eh, tg = half_inputs(8, 120, 64, 12, dtype, seed=21)
    try:
        for flag, val, native in (("bidir_mode", -1, True), ("bidir_mode", 1, True), ("bidir_mode", 0, True),
                                  ("bidir", 0, False), ("implicit", 0, False)):
            hctx.set_flag(flag, val)
            names = kernels_of(hctx, lambda: check_contract(hctx, eh, dtype, tg))
            assert ("widen" in names) != native and ("bidir_ctc" in names) == native, (flag, val, names)
            reset_flags(hctx)
    finally:
        reset_flags(hctx)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Cn", [256, 60])
def test_widened_route_wide_and_odd_alphabets(hctx, dtype, Cn):
    """C = 256 (beyond k_bidir.cu) and C = 60 (k_bidir.cu in float32, but not a multiple of 8)"""
    eh, tg = half_inputs(6, 90, Cn, 10, dtype, seed=Cn)
    names = kernels_of(hctx, lambda: check_contract(hctx, eh, dtype, tg))
    assert "widen" in names and "narrow" in names, names


@pytest.mark.parametrize("dtype", DTYPES)
def test_widened_route_misaligned_buffers(hctx, dtype):
    B, T, Cn = 4, 64, 64
    eh, tg = half_inputs(B, T, Cn, 8, dtype, seed=8)
    n = B * T * Cn
    buf = torch.empty(n + 8, dtype=eh.dtype, device="cuda")
    em = buf[1:1 + n].view(B, T, Cn)  # 2 bytes past a 16-byte boundary
    em.copy_(eh)
    names = kernels_of(hctx, lambda: check_contract(hctx, em, dtype, tg))
    assert "widen" in names, names
    # an aligned emission buffer with a misaligned gradient
    gbuf = torch.full((n + 8,), float("nan"), dtype=eh.dtype, device="cuda")
    lh, gh = call_ex(hctx, eh, dtype, tg, grad=gbuf[1:1 + n].view(B, T, Cn))
    lf, gf = call_f32(hctx, eh.float(), tg)
    assert same(lh, lf) and same(gh, gf.to(eh.dtype))
    assert torch.isnan(gbuf[0]) and torch.isnan(gbuf[n + 1:]).all()  # nothing outside the view


@pytest.mark.parametrize("dtype", DTYPES)
def test_non_finite_takes_the_exact_retry(hctx, dtype):
    """an inf emission raises the kernel's status bit; the batch is repeated on the materialised route, widened"""
    eh, tg = half_inputs(4, 80, 64, 8, dtype, seed=2)
    eh[1, 30, 5] = float("inf")
    eh[2, 10, 0] = float("-inf")
    lf, _ = check_contract(hctx, eh, dtype, tg)
    assert np.isfinite(lf[[0, 3]]).all() and not np.isfinite(lf[1])


def test_f32_through_ex_is_gtnb_ctc_loss(hctx):
    e, tg = util.bench_inputs(8, 150, 64, 15, seed=4)
    e32 = torch.from_numpy(e).cuda()
    lh, gh = call_ex(hctx, e32, F32, tg)
    lf, gf = call_f32(hctx, e32, tg)
    assert same(lh, lf) and same(gh, gf)
    lens = np.array([150, 20, 3, 149, 100, 0, 77, 150], np.int32)
    lh, gh = call_ex(hctx, e32, F32, tg, lens=lens)
    lf, gf = call_f32(hctx, e32, tg, lens=lens)
    assert same(lh, lf) and same(gh, gf)


def test_unknown_dtype_is_invalid_argument(hctx):
    e = torch.zeros(1, 4, 8, device="cuda")
    with pytest.raises(capi.GtnbError) as ei:
        call_ex(hctx, e, 3, [[1]])
    assert ei.value.code == capi.ERR_INVALID_ARGUMENT


def test_reference_parity_on_widened_bf16(oracle):
    """losses within 1e-4 relative of the reference on bf16 emissions widened to float32 (guards the widening)"""
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing"
    from gtn_b200.torch_loss import ctc_loss
    e, tg = util.bench_inputs(2, 200, 64, 20, seed=17)
    eh = torch.from_numpy(e).cuda().to(torch.bfloat16)
    got = ctc_loss(eh, tg, reduction="none").cpu().numpy()
    lr, _, _ = oracle.ref_ctc_batch(eh.float().cpu().numpy(), tg, want_grad=False)
    assert util.close(got, lr), (got, lr)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_torch_ctc_loss_half(dt):
    from gtn_b200.torch_loss import ctc_loss
    B, T, Cn = 8, 120, 64
    e, tg = util.bench_inputs(B, T, Cn, 12, seed=6)
    base = torch.from_numpy(e).cuda().to(dt)
    # the float32 call on the widened emissions
    x32 = base.float().requires_grad_(True)
    l32 = ctc_loss(x32, tg, reduction="none")
    l32.sum().backward()
    g32 = x32.grad
    # reduction "none": float32 losses, a gradient of the input dtype equal to the rounded float32 gradient
    x = base.clone().requires_grad_(True)
    lo = ctc_loss(x, tg, reduction="none")
    assert lo.dtype == torch.float32 and same(lo.detach(), l32.detach())
    lo.sum().backward()
    assert x.grad.dtype == dt and same(x.grad, g32.to(dt))
    # "mean": fp32_grad.to(dtype) * (1 / B), evaluated by torch in that dtype
    y = base.clone().requires_grad_(True)
    m = ctc_loss(y, tg)
    assert m.dtype == torch.float32 and same(m.detach(), l32.detach().mean())
    m.backward()
    assert y.grad.dtype == dt and same(y.grad, g32.to(dt) * (1 / B))


def test_torch_autocast_training_step():
    """a small model under torch.autocast(bfloat16) feeds its logits straight in and trains one step"""
    from gtn_b200.torch_loss import ctc_loss
    torch.manual_seed(0)
    B, T, F, Cn = 4, 60, 32, 32
    model = torch.nn.Sequential(torch.nn.Linear(F, 64), torch.nn.ReLU(), torch.nn.Linear(64, Cn)).cuda()
    opt = torch.optim.SGD(model.parameters(), lr=0.1)
    feats = torch.randn(B, T, F, device="cuda")
    tg = [np.random.default_rng(b).integers(1, Cn, 8).astype(np.int32) for b in range(B)]
    before = [p.detach().clone() for p in model.parameters()]
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits = model(feats)
        assert logits.dtype == torch.bfloat16
        loss = ctc_loss(logits, tg)
    assert loss.dtype == torch.float32 and torch.isfinite(loss)
    opt.zero_grad()
    loss.backward()
    for p, q in zip(model.parameters(), before):
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().sum() > 0
    opt.step()
    assert any(not torch.equal(p.detach(), q) for p, q in zip(model.parameters(), before))
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert torch.isfinite(ctc_loss(model(feats), tg))
