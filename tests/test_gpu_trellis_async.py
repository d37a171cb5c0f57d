"""gtnb_ngram_ctc_loss_async, gtnb_asg_loss_async and torch ngram_ctc_loss / asg_loss on tensor targets, on the GPU.

The contract: on inputs the synchronous call (gtnb_*_typed, list targets) takes without its exact retry, the losses
are == to it and the status is 0.  Both calls add their gradients with atomics whose order varies from run to run,
so the emission and transition gradients are held to the synchronous call's own run-to-run spread; the transition
gradient may also differ by the regrouping of the float32 sums of the numerator's arc gradients, which the
asynchronous call adds utterance by utterance (`within`).  A non-finite value gives status 1 and an invalid length or label status 2: a NaN loss, a
zero emission-gradient row and no share of the transition gradient, for that utterance only.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from gtn_b200 import capi
from gtn_b200 import torch_loss as tl_mod

pytestmark = pytest.mark.gpu

DT = {torch.float32: capi.F32, torch.bfloat16: capi.BF16, torch.float16: capi.F16}
KINDS = ["ngram", "asg"]


@pytest.fixture(scope="module")
def ctx():
    c = capi.Ctx(0)
    yield c
    c.close()


def n_trans(kind, C_):
    return C_ * C_ if kind == "ngram" else C_ + C_ * C_


def transitions(kind, C_, seed=0):
    g = torch.Generator().manual_seed(seed + 100)
    return torch.empty(n_trans(kind, C_)).normal_(0, 1, generator=g).cuda()


def batch(B, T, C_, S, seed=0, ragged=False):
    """utterance 0 has U = S labels without a repeat, the bounds the asynchronous call is sized for, so both calls
    sweep layouts of the same shape"""
    g = torch.Generator().manual_seed(seed)
    e = torch.empty(B, T, C_).uniform_(-5, 5, generator=g)
    tg = torch.randint(1, C_, (B, S), generator=g).int()
    if S > 1:
        while bool((tg[0, 1:] == tg[0, :-1]).any()):
            tg[0] = torch.randint(1, C_, (S,), generator=g).int()
    lens = torch.full((B,), S, dtype=torch.int32)
    il = None
    if ragged:
        lens = torch.randint(0, S + 1, (B,), generator=g).int()
        lens[0] = S
        il = torch.randint(max(1, T // 2), T + 1, (B,), generator=g).int()
        il[0] = T
    return e, tg, lens, il


def lists(tg, lens):
    return [tg[b, :int(lens[b])].numpy().astype(np.int32) for b in range(tg.shape[0])]


def sync_call(ctx, kind, e, W, tg, lens, il, blank=0):
    """gtnb_ngram_ctc_loss_typed / gtnb_asg_loss_typed on device buffers and host list targets -> (losses, grad, tg)"""
    B, T, C_ = e.shape
    cat = np.ascontiguousarray(np.concatenate(lists(tg, lens)) if int(lens.sum()) else np.zeros(1), np.int32)
    ln = np.ascontiguousarray(lens.numpy(), np.int32)
    iln = None if il is None else np.ascontiguousarray(il.numpy(), np.int32)
    losses = np.zeros(B, np.float32)
    grad = torch.empty_like(e)
    tgrad = torch.empty(W.numel(), device="cuda")
    il_p = capi._p(iln, capi._i32p)
    if kind == "ngram":
        rc = capi.lib().gtnb_ngram_ctc_loss_typed(
            ctx.h, B, T, C_, e.data_ptr(), DT[e.dtype], il_p, W.data_ptr(), cat.ctypes.data_as(capi._i32p),
            ln.ctypes.data_as(capi._i32p), blank, losses.ctypes.data_as(capi._f32p), grad.data_ptr(), tgrad.data_ptr())
    else:
        rc = capi.lib().gtnb_asg_loss_typed(
            ctx.h, B, T, C_, e.data_ptr(), DT[e.dtype], il_p, W.data_ptr(), cat.ctypes.data_as(capi._i32p),
            ln.ctypes.data_as(capi._i32p), losses.ctypes.data_as(capi._f32p), grad.data_ptr(), tgrad.data_ptr())
    ctx._check(rc)
    torch.cuda.synchronize()
    return losses, grad, tgrad


def workspace(ctx, kind, B, T, C_, S, dtype, with_grad=1, dt=None):
    n = C.c_size_t()
    fn = capi.lib().gtnb_ngram_ctc_loss_async_workspace if kind == "ngram" else capi.lib().gtnb_asg_loss_async_workspace
    rc = fn(ctx.h, B, T, C_, S, DT[dtype] if dt is None else dt, with_grad, C.byref(n))
    return rc, n.value


def launch(ctx, kind, e, W, tg, lens, il, blank, losses, status, grad, tgrad, ws, nb):
    B, T, C_ = e.shape
    S = tg.shape[1]
    common = (ctx.h, torch.cuda.current_stream().cuda_stream, B, T, C_, S, e.data_ptr(), DT[e.dtype],
              None if il is None else il.data_ptr(), W.data_ptr(), tg.data_ptr(), lens.data_ptr())
    outs = (losses.data_ptr(), None if status is None else status.data_ptr(), None if grad is None else grad.data_ptr(),
            None if tgrad is None else tgrad.data_ptr(), ws, nb)
    if kind == "ngram":
        return capi.lib().gtnb_ngram_ctc_loss_async(*common, blank, *outs)
    return capi.lib().gtnb_asg_loss_async(*common, *outs)


def async_call(ctx, kind, e, W, tg, lens, il, blank=0, want_grad=True, ws_bytes=None, ws_offset=0):
    """-> (rc, losses, status, grad, tgrad) with the device buffers read back after a synchronise"""
    B, T, C_ = e.shape
    rc, need = workspace(ctx, kind, B, T, C_, tg.shape[1], e.dtype, int(want_grad))
    if rc:
        return rc, None, None, None, None
    nb = need if ws_bytes is None else ws_bytes
    ws = torch.empty(nb + 512, dtype=torch.uint8, device="cuda")
    tgd, lensd = tg.cuda().contiguous(), lens.cuda().contiguous()
    ild = None if il is None else il.cuda().contiguous()
    losses = torch.full((B,), -7.0, device="cuda")
    status = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    grad = torch.full_like(e, 3.0) if want_grad else None
    tgrad = torch.full((W.numel(),), 3.0, device="cuda") if want_grad else None
    rc = launch(ctx, kind, e, W, tgd, lensd, ild, blank, losses, status, grad, tgrad, ws.data_ptr() + ws_offset, nb)
    torch.cuda.synchronize()
    return rc, losses.cpu().numpy(), status.cpu().numpy(), grad, tgrad


def same(a, b):
    """== with NaN equal to NaN (a T_b = 0 utterance's loss is NaN in both calls)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(((a == b) | (np.isnan(a) & np.isnan(b))).all())


def spread(ctx, kind, e, W, tg, lens, il, gs, ts, runs=4):
    """the largest difference between (gs, ts) and further synchronous runs"""
    sg = st = 0.0
    for _ in range(runs):
        _, g2, t2 = sync_call(ctx, kind, e, W, tg, lens, il)
        sg = max(sg, (gs.float() - g2.float()).abs().max().item())
        st = max(st, (ts - t2).abs().max().item())
    return sg, st


def within(ga, gs, sg, tga, tgs, st):
    """the gradients of the asynchronous call against the synchronous call's run-to-run spread (sg, st).

    Emission gradient: both calls add the same terms with the same kernels, only in another atomic order, so the
    asynchronous result is one more draw of that order: at most twice the measured spread, with a floor of two
    float32 ulps of the largest entry where the runs happened to agree.

    Transition gradient: the spread plus 8 float32 ulps of the largest entry.  The synchronous call's own spread is
    about one ulp, since few of its sums change order from run to run.  The asynchronous call adds the numerator's
    arc gradients utterance by utterance instead of in one flat pass, which regroups the float32 sums of every entry;
    on the H100 that moved entries by up to 2.7 ulps of the largest one.  The 8 ulps allow for that regrouping, a
    tolerance beyond the spread itself (DESIGN.md, the trellis criteria's asynchronous calls, "Tests")."""
    eps = torch.finfo(torch.float32).eps
    dg = (ga.float() - gs.float()).abs().max().item()
    dt = (tga - tgs).abs().max().item()
    assert dg <= max(2 * sg, 2 * eps * gs.float().abs().max().item()), (dg, sg)
    assert dt <= st + 8 * eps * tgs.abs().max().item(), (dt, st, tgs.abs().max().item())


def check_contract(ctx, kind, e, W, tg, lens, il):
    rc, la, sa, ga, tga = async_call(ctx, kind, e, W, tg, lens, il)
    assert rc == 0, capi.lib().gtnb_last_error(ctx.h)
    assert (sa == 0).all(), sa
    ls, gs, tgs = sync_call(ctx, kind, e, W, tg, lens, il)
    assert same(la, ls), (la[:4], ls[:4])
    if il is not None:
        for b in range(e.shape[0]):
            assert (ga[b, int(il[b]):] == 0).all()
    sg, st = spread(ctx, kind, e, W, tg, lens, il, gs, tgs)
    within(ga, gs, sg, tga, tgs, st)
    return la


def routes(ctx, fn):
    ctx.profile(True)
    ctx.profile_read()
    fn()
    names = set(ctx.profile_read())
    ctx.profile(False)
    return names


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("C_", [64, 128])
def test_benchmark_shape(ctx, kind, C_):
    e, tg, lens, il = batch(128, 500, C_, 50, seed=C_)
    check_contract(ctx, kind, e.cuda(), transitions(kind, C_), tg, lens, il)


@pytest.mark.parametrize("kind", KINDS)
def test_ragged_lengths_c30(ctx, kind):
    e, tg, lens, il = batch(16, 200, 30, 25, seed=3, ragged=True)
    check_contract(ctx, kind, e.cuda(), transitions(kind, 30), tg, lens, il)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_half_precision(ctx, kind, dtype):
    e, tg, lens, il = batch(16, 150, 64, 20, seed=7, ragged=True)
    e = e.to(dtype).cuda()
    names = routes(ctx, lambda: check_contract(ctx, kind, e, transitions(kind, 64), tg, lens, il))
    assert "narrow" in names and "widen" not in names


@pytest.mark.parametrize("kind", KINDS)
def test_edge_cases(ctx, kind):
    B, T, C_, S = 6, 60, 64, 20
    e, tg, lens, il = batch(B, T, C_, S, seed=4)
    il = torch.full((B,), T, dtype=torch.int32)
    il[1] = 0  # T_b = 0
    lens[2] = 0  # U = 0
    il[3] = 10  # 20 labels in 10 frames: infeasible
    tg[4, 1] = tg[4, 0]  # a repeat
    lens[5] = S - 6
    padded = tg.clone()
    padded[5, S - 6:] = 999  # padding beyond U_b is never read
    W = transitions(kind, C_)
    ec = e.cuda()
    rc, la, st, ga, tga = async_call(ctx, kind, ec, W, padded, lens, il)
    assert rc == 0
    assert (st[[0, 1, 2, 4, 5]] == 0).all(), st
    assert np.isnan(la[1])  # T_b = 0: NaN, as the synchronous call gives it
    ls, gs, tgs = sync_call(ctx, kind, ec, W, tg, lens, il)
    ok = st == 0
    assert same(la[ok], ls[ok])
    keep = [b for b in range(B) if st[b] == 0]
    if st[3]:  # NaN with status 1, and no share of the transition gradient
        assert st[3] == 1 and np.isnan(la[3]) and (ga[3] == 0).all()
        ls, gs, tgs = sync_call(ctx, kind, ec[keep], W, tg[keep], lens[keep], il[keep])
        assert same(la[keep], ls)
    else:  # +inf with status 0
        assert la[3] == np.inf
    sg, stt = spread(ctx, kind, ec[keep], W, tg[keep], lens[keep], il[keep], gs if st[3] else gs[keep], tgs)
    within(ga[keep], gs if st[3] else gs[keep], sg, tga, tgs, stt)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("bad", [float("inf"), float("nan")])
def test_non_finite_emission(ctx, kind, bad):
    e, tg, lens, il = batch(4, 80, 64, 10, seed=8)
    W = transitions(kind, 64)
    clean = e.clone().cuda()
    e[2, 7, 3] = bad
    rc, la, st, ga, tga = async_call(ctx, kind, e.cuda(), W, tg, lens, il)
    assert rc == 0 and st.tolist() == [0, 0, 1, 0]
    assert np.isnan(la[2]) and (ga[2] == 0).all()
    keep = [0, 1, 3]
    ls, gs, tgs = sync_call(ctx, kind, clean[keep], W, tg[keep], lens[keep], None)
    assert same(la[keep], ls)
    sg, stt = spread(ctx, kind, clean[keep], W, tg[keep], lens[keep], None, gs, tgs)
    within(ga[keep], gs, sg, tga, tgs, stt)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("where", ["first", "last"])
def test_non_finite_transition_weight(ctx, kind, where):
    """every utterance flagged, T_b = 0 and T_b = 1 included: each CTA of the denominator's forward loads and checks
    the whole of trans_w before its first frame (ASG: the start weights and the matrix), whatever its T_b"""
    e, tg, lens, il = batch(6, 40, 32, 6, seed=9, ragged=True)
    il[1], il[2] = 0, 1  # T_b = 0, T_b = 1 (ASG's frame 1 reads only the start weights)
    lens[2] = 1
    W = transitions(kind, 32)
    W[0 if where == "first" else W.numel() - 7] = float("nan")  # ASG: a start weight, else the matrix
    rc, la, st, ga, tga = async_call(ctx, kind, e.cuda(), W, tg, lens, il)
    assert rc == 0 and (st == 1).all(), st
    assert np.isnan(la).all() and (ga == 0).all() and (tga == 0).all()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", ["negative_U", "U_over_S", "T_over_T", "negative_T", "label_C", "negative_label"])
def test_invalid_inputs(ctx, kind, case):
    B, T, C_, S = 5, 60, 64, 12
    e, tg, lens, _ = batch(B, T, C_, S, seed=9)
    il = torch.full((B,), T, dtype=torch.int32)
    tg_bad, lens_bad, il_bad = tg.clone(), lens.clone(), il.clone()
    if case == "negative_U":
        lens_bad[1] = -1
    elif case == "U_over_S":
        lens_bad[1] = S + 1
    elif case == "T_over_T":
        il_bad[1] = T + 1
    elif case == "negative_T":
        il_bad[1] = -3
    elif case == "label_C":
        tg_bad[1, 4] = C_
    else:
        tg_bad[1, 0] = -2
    ec, W = e.cuda(), transitions(kind, C_)
    rc, la, st, ga, tga = async_call(ctx, kind, ec, W, tg_bad, lens_bad, il_bad)
    assert rc == 0 and st.tolist() == [0, 2, 0, 0, 0]
    assert np.isnan(la[1]) and (ga[1] == 0).all()
    keep = [0, 2, 3, 4]
    ls, gs, tgs = sync_call(ctx, kind, ec[keep], W, tg[keep], lens[keep], il[keep])
    assert same(la[keep], ls)
    sg, stt = spread(ctx, kind, ec[keep], W, tg[keep], lens[keep], il[keep], gs, tgs)
    within(ga[keep], gs, sg, tga, tgs, stt)


@pytest.mark.parametrize("kind", KINDS)
def test_unsupported_and_bad_workspace(ctx, kind):
    B, T, C_, S = 4, 64, 64, 10
    e, tg, lens, il = batch(B, T, C_, S, seed=10)
    ec, W = e.cuda(), transitions(kind, C_)
    assert workspace(ctx, kind, B, T, 129, S, torch.float32)[0] == capi.ERR_UNSUPPORTED
    e129 = torch.zeros(B, T, 129, device="cuda")
    assert async_call(ctx, kind, e129, transitions(kind, 129), tg, lens, il)[0] == capi.ERR_UNSUPPORTED
    assert workspace(ctx, kind, B, T, C_, S, torch.float32, dt=7)[0] == capi.ERR_UNSUPPORTED
    if kind == "ngram":
        assert async_call(ctx, kind, ec, W, tg, lens, il, blank=C_)[0] == capi.ERR_UNSUPPORTED
    ctx.set_flag("implicit", 0)
    try:
        assert async_call(ctx, kind, ec, W, tg, lens, il)[0] == capi.ERR_UNSUPPORTED
    finally:
        ctx.set_flag("implicit", 1)
    _, need = workspace(ctx, kind, B, T, C_, S, torch.float32)
    assert async_call(ctx, kind, ec, W, tg, lens, il, ws_bytes=need // 2)[0] == capi.ERR_INVALID_ARGUMENT
    assert async_call(ctx, kind, ec, W, tg, lens, il, ws_offset=16)[0] == capi.ERR_INVALID_ARGUMENT


@pytest.mark.parametrize("kind", KINDS)
def test_launch_profile_and_no_staging_copy(ctx, kind):
    B, T, C_, S = 8, 100, 64, 12
    e, tg, lens, il = batch(B, T, C_, S, seed=12, ragged=True)
    ec, W = e.cuda(), transitions(kind, C_)
    async_call(ctx, kind, ec, W, tg, lens, il)  # warm-up: side stream, kernels
    rc, need = workspace(ctx, kind, B, T, C_, S, torch.float32)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    tgd, lensd, ild = tg.cuda(), lens.cuda(), il.cuda()
    losses = torch.empty(B, device="cuda")
    grad = torch.empty_like(ec)
    tgrad = torch.empty(W.numel(), device="cuda")
    torch.cuda.synchronize()
    ctx.profile(True)
    ctx.profile_read()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        assert launch(ctx, kind, ec, W, tgd, lensd, ild, 0, losses, None, grad, tgrad, ws.data_ptr(), need) == 0
        torch.cuda.synchronize()
    names = set(ctx.profile_read())
    ctx.profile(False)
    den = "ngram_den" if kind == "ngram" else "asg_den"
    build = "ngram_num_build" if kind == "ngram" else "asg_num_build"
    for k in ("trellis_async_prepare", build, "implicit_forward", "implicit_backward", den + "_forward",
              den + "_backward", "trellis_async_gate", "trellis_async_scatter", "ctc_async_finalize"):
        assert k in names, (k, names)
    assert ("ngram_sigma" in names) == ("ngram_fold" in names) == (kind == "ngram")
    copies = [ev.name for ev in prof.events() if "Memcpy" in ev.name]
    assert not any("HtoD" in n or "DtoH" in n for n in copies), copies


# ---- torch -------------------------------------------------------------------------------------------------------

def loss_fn(kind, x, W, tg, **kw):
    if kind == "ngram":
        return tl_mod.ngram_ctc_loss(x, W, tg, **kw)
    return tl_mod.asg_loss(x, W, tg, **kw)


def torch_inputs(kind, B=8, T=100, C_=64, S=15, seed=11):
    e, tg, lens, il = batch(B, T, C_, S, seed=seed, ragged=True)
    return e.cuda(), transitions(kind, C_, seed), tg.cuda(), lens.cuda(), il.cuda(), lists(tg, lens), il


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("reduction", ["mean", "none"])
def test_torch_reductions_match_list_targets(ctx, kind, reduction):
    e, W0, tg, lens, il, tl_list, il_host = torch_inputs(kind)
    outs = []
    for tensor_targets in (True, False):
        x = e.clone().requires_grad_(True)
        W = W0.clone().requires_grad_(True)
        if tensor_targets:
            loss = loss_fn(kind, x, W, tg, reduction=reduction, input_lengths=il, target_lengths=lens)
        else:
            loss = loss_fn(kind, x, W, tl_list, reduction=reduction, input_lengths=il_host)
        (loss if reduction == "mean" else loss.sum()).backward()
        outs.append((loss.detach(), x.grad, W.grad))
    assert outs[0][0].is_cuda and same(outs[0][0].cpu().numpy(), outs[1][0].cpu().numpy())
    # the gradients: within the synchronous call's spread, as through the C ABI
    assert torch.allclose(outs[0][1], outs[1][1], rtol=1e-4, atol=1e-6)
    assert torch.allclose(outs[0][2], outs[1][2], rtol=1e-4, atol=1e-5)
    if reduction == "none":  # a non-uniform upstream gradient: NaN transition gradient, no host assert
        x = e.clone().requires_grad_(True)
        W = W0.clone().requires_grad_(True)
        loss = loss_fn(kind, x, W, tg, reduction="none", input_lengths=il, target_lengths=lens)
        (loss * torch.linspace(0.5, 2.0, loss.shape[0], device="cuda")).sum().backward()
        assert torch.isnan(W.grad).all() and torch.isfinite(x.grad).all()


@pytest.mark.parametrize("kind", KINDS)
def test_torch_no_host_wait(kind):
    e, W0, tg, lens, il, _, _ = torch_inputs(kind, B=32, T=300)
    x = e.clone().requires_grad_(True)
    W = W0.clone().requires_grad_(True)
    loss_fn(kind, x, W, tg, input_lengths=il, target_lengths=lens).backward()  # warm-up
    torch.cuda.synchronize()
    done = torch.cuda.Event()
    torch.cuda._sleep(100_000_000)  # tens of milliseconds of GPU time
    loss = loss_fn(kind, x, W, tg, input_lengths=il, target_lengths=lens)
    done.record()
    assert not done.query(), "forward waited for the device"
    loss.backward()
    done.record()
    assert not done.query(), "backward waited for the device"
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = loss_fn(kind, x, W, tg, input_lengths=il, target_lengths=lens, reduction="none")
        loss.sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    # (an empty ASG target has no accepting state: +inf, as the list-target call gives it)
    assert (torch.isfinite(loss) | ((lens == 0) & (kind == "asg"))).all().item()


@pytest.mark.parametrize("kind", KINDS)
def test_torch_cuda_graph_training_step(kind):
    torch.manual_seed(0)
    B, T, F, C_, S = 8, 50, 32, 64, 10
    model = torch.nn.Linear(F, C_).cuda()
    trans = torch.nn.Parameter(0.1 * torch.randn(n_trans(kind, C_), device="cuda"))
    params = list(model.parameters()) + [trans]
    opt = torch.optim.SGD(params, lr=0.05)
    sx = torch.randn(B, T, F, device="cuda")
    stg = torch.randint(1, C_, (B, S), device="cuda", dtype=torch.int32)
    stl = torch.full((B,), S, device="cuda", dtype=torch.int32)
    sil = torch.full((B,), T, device="cuda", dtype=torch.int32)

    def step(m, w, o, x, tg, tl_, il):
        o.zero_grad(set_to_none=False)
        loss = loss_fn(kind, m(x), w, tg, input_lengths=il, target_lengths=tl_)
        loss.backward()
        o.step()
        return loss.detach()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step(model, trans, opt, sx, stg, stl, sil)
    torch.cuda.current_stream().wait_stream(side)
    start = trans.detach().clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_loss = step(model, trans, opt, sx, stg, stl, sil)
    # the eager reference: the same step run from the parameters the replay starts from, so that every replay is
    # compared with eager steps from identical parameters and no divergence carries over from the earlier steps
    ref = copy.deepcopy(model)
    ref_w = torch.nn.Parameter(trans.detach().clone())
    ref_params = list(ref.parameters()) + [ref_w]
    ref_opt = torch.optim.SGD(ref_params, lr=0.05)
    gen = torch.Generator(device="cuda").manual_seed(1)
    for _ in range(4):
        x = torch.randn(B, T, F, device="cuda", generator=gen)
        tg = torch.randint(1, C_, (B, S), device="cuda", dtype=torch.int32, generator=gen)
        tl_ = torch.randint(1, S + 1, (B,), device="cuda", dtype=torch.int32, generator=gen)
        il = torch.randint(T // 2, T + 1, (B,), device="cuda", dtype=torch.int32, generator=gen)
        sx.copy_(x)
        stg.copy_(tg)
        stl.copy_(tl_)
        sil.copy_(il)
        before = [p.detach().clone() for p in params]
        graph.replay()
        captured = [p.detach().clone() for p in params]
        eager = []
        for _ in range(3):  # three eager draws of the step: their spread is the atomics' run-to-run spread
            with torch.no_grad():
                for q, b in zip(ref_params, before):
                    q.copy_(b)
            loss = step(ref, ref_w, ref_opt, x, tg, tl_, il)
            # the forward (model, trellis, numerator sweeps, mean) has no atomics: the loss is == every time
            assert torch.equal(static_loss, loss), (static_loss, loss)
            eager.append([q.detach().clone() for q in ref_params])
        # the update: the captured one within twice the eager draws' largest pairwise distance, parameter by
        # parameter (the largest difference over every element, which varies little from draw to draw), with a floor
        # of two float32 ulps where the three draws agree
        for k, c in enumerate(captured):
            pair = max((eager[i][k] - eager[j][k]).abs().max().item() for i, j in ((0, 1), (0, 2), (1, 2)))
            floor = 2 * torch.finfo(torch.float32).eps * c.abs().max().item()
            d = (c - eager[0][k]).abs().max().item()
            assert d <= max(2 * pair, floor), (k, d, pair, floor)
    assert torch.isfinite(trans).all() and not torch.equal(trans.detach(), start)  # the replays trained it


@pytest.mark.parametrize("kind", KINDS)
def test_torch_autocast_bf16_step(kind):
    torch.manual_seed(2)
    B, T, F, C_, S = 8, 60, 32, 64, 10
    model = torch.nn.Linear(F, C_).cuda()
    W = torch.nn.Parameter(0.1 * torch.randn(n_trans(kind, C_), device="cuda"))
    x = torch.randn(B, T, F, device="cuda")
    tg = torch.randint(1, C_, (B, S), device="cuda", dtype=torch.int32)
    lens = torch.full((B,), S, device="cuda", dtype=torch.int32)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits = model(x)
        assert logits.dtype == torch.bfloat16
        loss = loss_fn(kind, logits, W, tg, target_lengths=lens, reduction="none")
        il = torch.full((B,), T, dtype=torch.int32)
        ref = loss_fn(kind, logits.detach(), W.detach(), lists(tg.cpu(), lens.cpu()), reduction="none",
                      input_lengths=il)
    assert torch.equal(loss.detach(), ref)
    loss.mean().backward()
    assert model.weight.grad is not None and torch.isfinite(model.weight.grad).all() and torch.isfinite(W.grad).all()


@pytest.mark.parametrize("kind", KINDS)
def test_torch_c129_falls_back_outside_capture_and_raises_under_capture(kind):
    B, T, C_, S = 2, 40, 129, 4
    e = torch.randn(B, T, C_, device="cuda")
    W = transitions(kind, C_)
    tg = torch.randint(1, C_, (B, S), device="cuda", dtype=torch.int32)
    lens = torch.tensor([3, 4], device="cuda", dtype=torch.int32)
    lst = [tg[0, :3].cpu().numpy(), tg[1, :4].cpu().numpy()]
    if kind == "asg":
        got = loss_fn(kind, e, W, tg, target_lengths=lens, reduction="none")
        want = loss_fn(kind, e, W, lst, reduction="none")
        assert torch.equal(got, want)
    else:  # the synchronous n-gram call has no route for C > 128 either: its error, raised outside capture too
        with pytest.raises(RuntimeError):
            loss_fn(kind, e, W, lst, reduction="none")
        with pytest.raises(RuntimeError):
            loss_fn(kind, e, W, tg, target_lengths=lens, reduction="none")
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="cannot be captured"):
        with torch.cuda.graph(graph):
            loss_fn(kind, e, W, tg, target_lengths=lens, reduction="none")
