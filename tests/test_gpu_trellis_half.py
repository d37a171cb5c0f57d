"""gtnb_ngram_ctc_loss_typed, gtnb_asg_loss_typed and gtnb_viterbi_dense_typed with bfloat16 / fp16 emissions, and the
torch criteria and decoders on 16-bit tensors, on the GPU.

The contract: the result is the float32 call's on the emissions widened to float32, on every route -- the dense trellis
and the numerator sweeps reading the 16-bit buffers in place, and the widened route (ASG with C > 128, the "implicit"
flag off, the exact retry after a non-finite value).  Losses, Viterbi paths and scores are compared with ==.  The
gradients are sums that the float32 call itself accumulates with atomics (the two streams into one emission row, every
CTA into the transition gradient), in an order that varies from run to run, so two float32 calls already differ in
their last bits: the transition gradient is held to float32 reassociation and the emission gradient to the float32
gradient rounded to the dtype, within one unit in the last place of the dtype where a rounding boundary lies between
two orders of the same sum."""
import numpy as np
import pytest
import torch

from gtn_b200 import capi
from tests import util

pytestmark = pytest.mark.gpu
F32, BF16, F16 = capi.F32, capi.BF16, capi.F16
TORCH = {BF16: torch.bfloat16, F16: torch.float16}
DTYPES = [BF16, F16]
ASG, NGRAM = "asg", "ngram"


@pytest.fixture(scope="module")
def hctx():
    c = capi.Ctx(0)
    yield c
    c.close()


def n_trans(kind, Cn):
    return Cn * Cn if kind == NGRAM else Cn + Cn * Cn


def trans(kind, Cn, seed=3):
    rng = np.random.default_rng(seed)
    return torch.from_numpy(rng.uniform(-1, 1, n_trans(kind, Cn)).astype(np.float32)).cuda()


def call(ctx, kind, e, dtype, w, targets, blank=0, lens=None, want_grad=True):
    """the _typed call on device tensors (dtype F32 included) -> (losses, grad or None, trans_grad or None); grad starts
    as NaN everywhere so that rows the call must write (or zero) show up"""
    B, T, Cn = e.shape
    cat, tl = capi._cat_targets(targets)
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    losses = np.zeros(B, np.float32)
    grad = torch.full_like(e, float("nan")) if want_grad else None
    tg = torch.full((w.numel(),), float("nan"), device=e.device) if want_grad else None
    il_p = None if il is None else il.ctypes.data_as(capi._i32p)
    args = [cat.ctypes.data_as(capi._i32p), tl.ctypes.data_as(capi._i32p)]
    torch.cuda.synchronize()
    if kind == NGRAM:
        ctx._check(capi.lib().gtnb_ngram_ctc_loss_typed(
            ctx.h, B, T, Cn, e.data_ptr(), dtype, il_p, w.data_ptr(), *args, blank, losses.ctypes.data_as(capi._f32p),
            grad.data_ptr() if want_grad else None, tg.data_ptr() if want_grad else None))
    else:
        ctx._check(capi.lib().gtnb_asg_loss_typed(
            ctx.h, B, T, Cn, e.data_ptr(), dtype, il_p, w.data_ptr(), *args, losses.ctypes.data_as(capi._f32p),
            grad.data_ptr() if want_grad else None, tg.data_ptr() if want_grad else None))
    return losses, grad, tg


def call_f32(ctx, kind, e32, w, targets, blank=0, lens=None, want_grad=True):
    """the existing float32 entry point on device buffers"""
    B, T, Cn = e32.shape
    cat, tl = capi._cat_targets(targets)
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    losses = np.zeros(B, np.float32)
    grad = torch.full_like(e32, float("nan")) if want_grad else None
    tg = torch.full((w.numel(),), float("nan"), device=e32.device) if want_grad else None
    il_p = None if il is None else il.ctypes.data_as(capi._i32p)
    g_p, t_p = (grad.data_ptr(), tg.data_ptr()) if want_grad else (None, None)
    torch.cuda.synchronize()
    if kind == NGRAM:
        ctx._check(capi.lib().gtnb_ngram_ctc_loss(
            ctx.h, B, T, Cn, e32.data_ptr(), 1, il_p, w.data_ptr(), 1, cat.ctypes.data_as(capi._i32p),
            tl.ctypes.data_as(capi._i32p), blank, losses.ctypes.data_as(capi._f32p), g_p, 1, t_p, 1))
    else:
        ctx._check(capi.lib().gtnb_asg_loss_ex(
            ctx.h, B, T, Cn, e32.data_ptr(), 1, il_p, w.data_ptr(), 1, cat.ctypes.data_as(capi._i32p),
            tl.ctypes.data_as(capi._i32p), losses.ctypes.data_as(capi._f32p), g_p, 1, t_p, 1))
    return losses, grad, tg


def same(a, b):
    """== with NaN equal to NaN"""
    a = torch.as_tensor(a).cpu()
    b = torch.as_tensor(b).cpu()
    assert a.dtype == b.dtype and a.shape == b.shape
    return bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def rounded_close(gh, gf):
    """gh (16-bit) == gf (float32) rounded to gh's dtype, but for elements within one unit in the last place of the
    dtype (the float32 sums differ in their last bits between orders of the atomics)"""
    want = gf.to(gh.dtype)
    assert torch.equal(torch.isnan(gh), torch.isnan(want))
    ok = ~torch.isnan(want)
    a, b = gh[ok].float(), want[ok].float()
    ulp = (2.0 ** -7 if gh.dtype == torch.bfloat16 else 2.0 ** -10) * b.abs() + 2.0 ** -24
    assert bool(((a - b).abs() <= ulp).all()), float((a - b).abs().max())
    if a.numel():
        assert float((a == b).float().mean()) > 0.99


def check_contract(ctx, kind, eh, dtype, w, targets, **kw):
    """eh: a 16-bit device tensor; returns what the float32 call gives on eh.float()"""
    lh, gh, th = call(ctx, kind, eh, dtype, w, targets, **kw)
    lf, gf, tf = call_f32(ctx, kind, eh.float().contiguous(), w, targets, **kw)
    assert same(lh, lf), (lh, lf)
    if gf is not None:
        assert gh.dtype == eh.dtype
        rounded_close(gh, gf)
        fin = torch.isfinite(tf)
        assert torch.equal(fin, torch.isfinite(th))
        if fin.any():
            assert torch.allclose(th[fin], tf[fin], rtol=1e-5, atol=1e-5 * max(1.0, float(tf[fin].abs().max())))
    return lf, gf, tf


def inputs(B, T, Cn, U, dtype, seed=1234):
    e, tg = util.bench_inputs(B, T, Cn, U, seed)
    return torch.from_numpy(e).cuda().to(TORCH[dtype]), tg


def launches(ctx, fn):
    """fn() with the context's launch profile on -> {kernel name: launches}"""
    ctx.profile(True)
    ctx.profile_read()
    fn()
    names = {k: n for k, (n, _) in ctx.profile_read().items()}
    ctx.profile(False)
    return names


def reset_flags(ctx):
    ctx.set_flag("implicit", 1)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", [NGRAM, ASG])
@pytest.mark.parametrize("Cn", [64, 128])
def test_benchmark_shapes_native(hctx, dtype, kind, Cn):
    """B=128 T=500 U=50: the native route reads the 16-bit emissions in place (no widen_kernel) and rounds the
    gradient once (one narrow_kernel)"""
    eh, tg = inputs(128, 500, Cn, 50, dtype)
    w = trans(kind, Cn)
    names = launches(hctx, lambda: call(hctx, kind, eh, dtype, w, tg))
    assert "widen" not in names and names.get("narrow") == 1, names
    den = "ngram_den_forward" if kind == NGRAM else "asg_den_forward"
    assert den in names and "implicit_forward" in names and "implicit_backward" in names
    assert "narrow" not in launches(hctx, lambda: call(hctx, kind, eh, dtype, w, tg, want_grad=False))
    lf, _, _ = check_contract(hctx, kind, eh, dtype, w, tg)
    assert np.isfinite(lf).all()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", [NGRAM, ASG])
def test_ragged_lengths_zero_the_padding(hctx, dtype, kind):
    B, T, Cn = 6, 120, 64
    eh, tg = inputs(B, T, Cn, 12, dtype, seed=5)
    w = trans(kind, Cn)
    lens = np.array([120, 97, 40, 120, 31, 64], np.int32)
    _, gh, _ = call(hctx, kind, eh, dtype, w, tg, lens=lens)
    for b in range(B):
        assert not gh[b, lens[b]:].any()
    check_contract(hctx, kind, eh, dtype, w, tg, lens=lens)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", [NGRAM, ASG])
def test_edges(hctx, dtype, kind):
    """T_b = 0 (NaN), U = 0 (+inf for ASG, whose numerator then has no accepting node), an infeasible target (+inf),
    blank != 0"""
    B, T, Cn = 4, 30, 32
    rng = np.random.default_rng(9)
    eh = torch.from_numpy(rng.uniform(-4, 4, (B, T, Cn)).astype(np.float32)).cuda().to(TORCH[dtype])
    tg = [rng.integers(0, Cn, 5), np.zeros(0, np.int32), rng.integers(0, Cn, 40), rng.integers(0, Cn, 3)]
    lens = np.array([0, 30, 30, 12], np.int32)
    lf, _, _ = check_contract(hctx, kind, eh, dtype, trans(kind, Cn), tg, lens=lens, blank=7)
    assert np.isnan(lf[0]) and np.isposinf(lf[2]) and np.isfinite(lf[3])
    assert np.isposinf(lf[1]) if kind == ASG else np.isfinite(lf[1])


@pytest.mark.parametrize("dtype", DTYPES)
def test_asg_c160_takes_the_widened_route(hctx, dtype):
    eh, tg = inputs(4, 60, 160, 8, dtype, seed=2)
    w = trans(ASG, 160)
    names = launches(hctx, lambda: call(hctx, ASG, eh, dtype, w, tg))
    assert "widen" in names and names.get("narrow") == 1
    check_contract(hctx, ASG, eh, dtype, w, tg, lens=np.array([60, 50, 33, 60], np.int32))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", [NGRAM, ASG])
def test_implicit_off_takes_the_widened_route(hctx, dtype, kind):
    eh, tg = inputs(4, 60, 32, 6, dtype, seed=4)
    w = trans(kind, 32)
    hctx.set_flag("implicit", 0)
    try:
        names = launches(hctx, lambda: call(hctx, kind, eh, dtype, w, tg))
        assert "widen" in names and "ngram_den_forward" not in names and "asg_den_forward" not in names
        check_contract(hctx, kind, eh, dtype, w, tg)
    finally:
        reset_flags(hctx)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", [NGRAM, ASG])
@pytest.mark.parametrize("where", ["emission_inf", "trans_ninf", "trans_nan"])
def test_non_finite_takes_the_exact_retry(hctx, dtype, kind, where):
    B, T, Cn = 3, 40, 16
    eh, tg = inputs(B, T, Cn, 4, dtype, seed=8)
    w = trans(kind, Cn)
    if where == "emission_inf":
        eh[1, 10, 3] = float("inf")
    else:
        w[(Cn if kind == ASG else 0) + 2 * Cn + 1] = float("-inf") if where == "trans_ninf" else float("nan")
    names = launches(hctx, lambda: call(hctx, kind, eh, dtype, w, tg))
    assert "widen" in names  # the first attempt's status bit sends the batch to the widened exact route
    check_contract(hctx, kind, eh, dtype, w, tg)


@pytest.mark.parametrize("kind", [NGRAM, ASG])
def test_f32_through_typed_is_the_float32_call(hctx, kind):
    e, tg = inputs(8, 80, 64, 9, BF16)
    e = e.float().contiguous()
    w = trans(kind, 64)
    lt, gt, tt = call(hctx, kind, e, F32, w, tg, lens=np.arange(73, 81, dtype=np.int32))
    lf, gf, tf = call_f32(hctx, kind, e, w, tg, lens=np.arange(73, 81, dtype=np.int32))
    assert same(lt, lf) and torch.allclose(gt, gf, rtol=1e-5, atol=1e-6) and torch.allclose(tt, tf, rtol=1e-5, atol=1e-5)
    assert "widen" not in launches(hctx, lambda: call(hctx, kind, e, F32, w, tg))


@pytest.mark.parametrize("kind", [NGRAM, ASG])
def test_unknown_dtype_is_invalid_argument(hctx, kind):
    e, tg = inputs(1, 10, 8, 2, BF16)
    with pytest.raises(capi.GtnbError) as ei:
        call(hctx, kind, e, 3, trans(kind, 8), tg)
    assert ei.value.code == capi.ERR_INVALID_ARGUMENT
    paths = torch.empty((1, 10), dtype=torch.int32, device="cuda")
    with pytest.raises(capi.GtnbError) as ei:
        hctx._check(capi.lib().gtnb_viterbi_dense_typed(hctx.h, 1, 10, 8, e.data_ptr(), 7, None, capi.DENSE_ASG,
                                                        trans(ASG, 8).data_ptr(), paths.data_ptr(), None))
    assert ei.value.code == capi.ERR_INVALID_ARGUMENT


def viterbi(ctx, e, dtype, w, kind, lens=None):
    B, T, Cn = e.shape
    paths = torch.full((B, T), -7, dtype=torch.int32, device="cuda")
    scores = torch.full((B,), 7.0, device="cuda")
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    il_p = None if il is None else il.ctypes.data_as(capi._i32p)
    torch.cuda.synchronize()
    if dtype is None:
        ctx._check(capi.lib().gtnb_viterbi_dense_ex(ctx.h, B, T, Cn, e.data_ptr(), 1, il_p, kind, w.data_ptr(), 1,
                                                    paths.data_ptr(), scores.data_ptr(), 1))
    else:
        ctx._check(capi.lib().gtnb_viterbi_dense_typed(ctx.h, B, T, Cn, e.data_ptr(), dtype, il_p, kind, w.data_ptr(),
                                                       paths.data_ptr(), scores.data_ptr()))
    torch.cuda.synchronize()
    return paths.cpu(), scores.cpu()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", [capi.DENSE_ASG, capi.DENSE_BIGRAM])
def test_viterbi_typed(hctx, dtype, kind):
    """B=512 T=2000 C=128, then ragged lengths with integer-valued emissions (ties): paths and scores =="""
    Cn = 128
    w = trans(ASG if kind == capi.DENSE_ASG else NGRAM, Cn)
    eh, _ = inputs(512, 2000, Cn, 1, dtype, seed=21)
    ph, sh = viterbi(hctx, eh, dtype, w, kind)
    pf, sf = viterbi(hctx, eh.float().contiguous(), None, w, kind)
    assert torch.equal(ph, pf) and same(sh, sf)
    rng = np.random.default_rng(kind)
    ei = torch.from_numpy(rng.integers(-4, 5, (16, 300, Cn)).astype(np.float32)).cuda()
    wi = torch.from_numpy(rng.integers(-3, 1, w.numel()).astype(np.float32)).cuda()
    lens = rng.integers(0, 301, 16).astype(np.int32)
    lens[0] = 0
    ph, sh = viterbi(hctx, ei.to(TORCH[dtype]), dtype, wi, kind, lens)
    pf, sf = viterbi(hctx, ei, None, wi, kind, lens)
    assert torch.equal(ph, pf) and same(sh, sf)
    pt, st = viterbi(hctx, ei, F32, wi, kind, lens)
    assert torch.equal(pt, pf) and same(st, sf)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("kind", [NGRAM, ASG])
@pytest.mark.parametrize("reduction", ["mean", "none"])
def test_torch_losses_half(dt, kind, reduction):
    from gtn_b200.torch_loss import asg_loss, ngram_ctc_loss
    B, T, Cn = 6, 90, 32
    e, tg = util.bench_inputs(B, T, Cn, 8, seed=13)
    w0 = trans(kind, Cn)
    lens = [90, 80, 70, 90, 55, 90]
    res = {}
    for name, x0 in (("half", torch.from_numpy(e).cuda().to(dt)), ("f32", torch.from_numpy(e).cuda().to(dt).float())):
        x = x0.clone().requires_grad_(True)
        w = w0.clone().requires_grad_(reduction == "mean")
        if kind == NGRAM:
            loss = ngram_ctc_loss(x, w, tg, input_lengths=lens, reduction=reduction)
        else:
            loss = asg_loss(x, w, tg, input_lengths=lens, reduction=reduction)
        assert loss.dtype == torch.float32
        up = torch.linspace(0.5, 2.0, B, device="cuda") if reduction == "none" else None  # non-uniform
        (loss if up is None else (loss * up).sum()).backward()
        assert x.grad.dtype == x0.dtype
        res[name] = (loss.detach(), x.grad, w.grad)
    assert same(res["half"][0], res["f32"][0])
    # the 16-bit step rounds the float32 gradient once, then scales it: compare with the float32 step rounded
    gh, gf = res["half"][1].float(), res["f32"][1]
    assert torch.allclose(gh, gf, rtol=2.0 ** -6 if dt == torch.bfloat16 else 2.0 ** -9, atol=1e-6)
    if reduction == "mean":
        assert torch.allclose(res["half"][2], res["f32"][2], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_torch_asg_without_input_lengths(dt):
    """asg_loss on 16-bit emissions without input_lengths == asg_loss(e.float(), input_lengths=[T] * B), with
    transitions on the CPU getting their gradient there"""
    from gtn_b200.torch_loss import asg_loss
    B, T, Cn = 4, 50, 16
    e, tg = util.bench_inputs(B, T, Cn, 5, seed=23)
    w0 = trans(ASG, Cn).cpu()
    x = torch.from_numpy(e).cuda().to(dt).requires_grad_(True)
    w = w0.clone().requires_grad_(True)
    lh = asg_loss(x, w, tg, reduction="none")
    lh.sum().backward()
    assert w.grad.device.type == "cpu" and x.grad.dtype == dt
    xf = x.detach().float().requires_grad_(True)
    wf = w0.clone().cuda().requires_grad_(True)
    lf = asg_loss(xf, wf, tg, reduction="none", input_lengths=[T] * B)
    lf.sum().backward()
    assert same(lh.detach(), lf.detach())
    rounded_close(x.grad, xf.grad)
    assert torch.allclose(w.grad, wf.grad.cpu(), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_torch_decoders_half(dt):
    from gtn_b200.torch_loss import asg_viterbi, ngram_ctc_viterbi
    e, _ = util.bench_inputs(8, 120, 64, 1, seed=29)
    eh = torch.from_numpy(e).cuda().to(dt)
    for fn, kind in ((asg_viterbi, ASG), (ngram_ctc_viterbi, NGRAM)):
        w = trans(kind, 64)
        ph, sh = fn(eh, w, input_lengths=[120, 100, 0, 1, 120, 77, 64, 5])
        pf, sf = fn(eh.float(), w, input_lengths=[120, 100, 0, 1, 120, 77, 64, 5])
        assert torch.equal(ph, pf) and same(sh, sf)


@pytest.mark.parametrize("kind", [NGRAM, ASG])
def test_torch_autocast_training_step(kind):
    """a bf16 autocast model's logits go straight into the loss (no .float()), with learned transitions"""
    from gtn_b200.torch_loss import asg_loss, ngram_ctc_loss
    torch.manual_seed(0)
    B, T, D, Cn = 4, 60, 32, 24
    model = torch.nn.Linear(D, Cn).cuda()
    w = torch.nn.Parameter(torch.zeros(n_trans(kind, Cn), device="cuda"))
    opt = torch.optim.SGD(list(model.parameters()) + [w], lr=0.1)
    x = torch.randn(B, T, D, device="cuda")
    tg = [np.random.default_rng(b).integers(1, Cn, 6) for b in range(B)]
    losses = []
    for _ in range(3):
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits = model(x)
            assert logits.dtype == torch.bfloat16
            loss = (ngram_ctc_loss(logits, w, tg) if kind == NGRAM else asg_loss(logits, w, tg))
        loss.backward()
        assert model.weight.grad.dtype == torch.float32 and w.grad is not None and torch.isfinite(w.grad).all()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < losses[0]


@pytest.mark.parametrize("kind", [NGRAM, ASG])
def test_reference_parity_on_widened_bf16(oracle, kind):
    """losses within 1e-4 relative of the reference on bf16 emissions widened to float32 (guards the widening)"""
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing"
    from gtn_b200.torch_loss import asg_loss, ngram_ctc_loss
    from tests import asg_oracle as ao
    from tests import ngram_oracle as no
    B, T, Cn = 2, 40, 16
    e, tg = util.bench_inputs(B, T, Cn, 5, seed=17)
    eh = torch.from_numpy(e).cuda().to(torch.bfloat16)
    w = trans(kind, Cn)
    lens = np.array([40, 33], np.int32)
    e64 = eh.float().cpu().numpy()
    if kind == NGRAM:
        got = ngram_ctc_loss(eh, w, tg, input_lengths=lens, reduction="none").cpu().numpy()
        lr, _, _ = no.ref_ngram_ctc_batch(e64, w.cpu().numpy().reshape(Cn, Cn), tg, 0, lens)
    else:
        got = asg_loss(eh, w, tg, input_lengths=lens, reduction="none").cpu().numpy()
        lr, _, _ = ao.ref_asg_batch(e64, w.cpu().numpy(), tg, lens)
    assert util.close(got, lr), (got, lr)
