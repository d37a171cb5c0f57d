"""gtnb_ctc_loss_async and torch ctc_loss on tensor targets, on the GPU.

The contract: on inputs the synchronous call (gtnb_ctc_loss_ex, list targets) takes without its exact retry, the
losses are == to it; the gradient is == on the one-launch route (no floating-point atomics) and, on the sweeps route,
within the synchronous call's own run-to-run spread (== wherever two synchronous calls agree).  Non-finite emissions
give status 1, invalid lengths or labels status 2: a NaN loss and a zero gradient for that utterance only.
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


@pytest.fixture(scope="module")
def ctx():
    c = capi.Ctx(0)
    yield c
    c.close()


def batch(B, T, C_, S, seed=0, ragged=False, blank=0):
    g = torch.Generator().manual_seed(seed)
    e = torch.empty(B, T, C_).uniform_(-5, 5, generator=g)
    labels = [l for l in range(C_) if l != blank]
    tg = torch.tensor(labels)[torch.randint(0, len(labels), (B, S), generator=g)].int()
    lens = torch.full((B,), S, dtype=torch.int32)
    il = None
    if S > 1:  # utterance 0 without repeats: S - 1 skip arcs, the bounds of gtnb_ctc_loss_async
        while bool((tg[0, 1:] == tg[0, :-1]).any()):
            tg[0] = torch.tensor(labels)[torch.randint(0, len(labels), (S,), generator=g)].int()
    if ragged:
        lens = torch.randint(0, S + 1, (B,), generator=g).int()
        lens[0] = S
        il = torch.randint(max(1, T // 2), T + 1, (B,), generator=g).int()
        il[0] = T
    return e, tg, lens, il


def lists(tg, lens):
    return [tg[b, :int(lens[b])].numpy().astype(np.int32) for b in range(tg.shape[0])]


def sync_call(ctx, e, tg, lens, il, blank):
    """gtnb_ctc_loss_ex on device emissions (any dtype) and host list targets -> (losses, grad)"""
    B, T, C_ = e.shape
    cat = np.ascontiguousarray(np.concatenate(lists(tg, lens)) if int(lens.sum()) else np.zeros(1), np.int32)
    ln = np.ascontiguousarray(lens.numpy(), np.int32)
    iln = None if il is None else np.ascontiguousarray(il.numpy(), np.int32)
    losses = np.zeros(B, np.float32)
    grad = torch.empty_like(e)
    ctx._check(capi.lib().gtnb_ctc_loss_ex(
        ctx.h, B, T, C_, e.data_ptr(), DT[e.dtype], capi._p(iln, capi._i32p), cat.ctypes.data_as(capi._i32p),
        ln.ctypes.data_as(capi._i32p), blank, losses.ctypes.data_as(capi._f32p), grad.data_ptr()))
    torch.cuda.synchronize()
    return losses, grad


def workspace(ctx, B, T, C_, S, dtype, with_grad=1):
    n = C.c_size_t()
    rc = capi.lib().gtnb_ctc_loss_async_workspace(ctx.h, B, T, C_, S, DT[dtype], with_grad, C.byref(n))
    return rc, n.value


def async_call(ctx, e, tg, lens, il, blank, want_grad=True, ws_bytes=None, ws_offset=0):
    """-> (rc, losses, status, grad) with the device buffers read back after a synchronise"""
    B, T, C_ = e.shape
    S = tg.shape[1]
    rc, need = workspace(ctx, B, T, C_, S, e.dtype, int(want_grad))
    if rc:
        return rc, None, None, None
    nb = need if ws_bytes is None else ws_bytes
    ws = torch.empty(nb + 512, dtype=torch.uint8, device="cuda")
    tgd, lensd = tg.cuda().contiguous(), lens.cuda().contiguous()
    ild = None if il is None else il.cuda().contiguous()
    losses = torch.full((B,), -7.0, device="cuda")
    status = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    grad = torch.full_like(e, 3.0) if want_grad else None
    rc = capi.lib().gtnb_ctc_loss_async(
        ctx.h, torch.cuda.current_stream().cuda_stream, B, T, C_, S, e.data_ptr(), DT[e.dtype],
        None if ild is None else ild.data_ptr(), tgd.data_ptr(), lensd.data_ptr(), blank, losses.data_ptr(),
        status.data_ptr(), None if grad is None else grad.data_ptr(), ws.data_ptr() + ws_offset, nb)
    torch.cuda.synchronize()
    return rc, losses.cpu().numpy(), status.cpu().numpy(), grad


def same(a, b):
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


def routes(ctx, fn):
    ctx.profile(True)
    ctx.profile_read()
    fn()
    names = set(ctx.profile_read())
    ctx.profile(False)
    return names


def sync_spread(ctx, e, tg, lens, il, blank, gs, runs):
    """the largest difference between gs and further synchronous runs, and where they all agree with gs"""
    spread, agree = 0.0, torch.ones_like(gs, dtype=torch.bool)
    for _ in range(runs):
        _, g2 = sync_call(ctx, e, tg, lens, il, blank)
        spread = max(spread, (gs.float() - g2.float()).abs().max().item())
        agree &= gs == g2
    return spread, agree


def check_contract(ctx, e, tg, lens, il, blank=0, sweeps=False):
    """sweeps: the batch sees the same layout bounds in both calls (an utterance with U = S and U - 1 skip arcs)"""
    rc, la, st, ga = async_call(ctx, e, tg, lens, il, blank)
    assert rc == 0, capi.lib().gtnb_last_error(ctx.h)
    assert (st == 0).all(), st
    ls, gs = sync_call(ctx, e, tg, lens, il, blank)
    assert same(la, ls), (la[:4], ls[:4])
    if il is not None:
        for b in range(e.shape[0]):
            assert (ga[b, int(il[b]):] == 0).all()
    diff = (ga.float() - gs.float()).abs()
    if sweeps:
        spread, agree = sync_spread(ctx, e, tg, lens, il, blank, gs, 1)
        assert diff.max().item() <= spread, (diff.max().item(), spread, int((diff > 0).sum()))
        assert torch.equal(ga[agree], gs[agree]), int((ga[agree] != gs[agree]).sum())
    elif not torch.equal(ga, gs):
        # a difference the one-launch route may show only where the synchronous call differs from itself run to run
        spread, _ = sync_spread(ctx, e, tg, lens, il, blank, gs, 3)
        assert diff.max().item() <= spread, (diff.max().item(), spread, int((diff > 0).sum()))
    return la, st


@pytest.mark.parametrize("C_", [64, 128])
def test_benchmark_shape(ctx, C_):
    e, tg, lens, il = batch(256, 1000, C_, 100, seed=C_)
    e = e.cuda()
    names = routes(ctx, lambda: check_contract(ctx, e, tg, lens, il))
    assert "bidir_ctc" in names and "ctc_async_prepare" in names and "ctc_async_finalize" in names
    assert "ctc_build" not in names  # the PAIR kernels read the padded targets themselves


def test_ragged_lengths_zero_padding_rows(ctx):
    e, tg, lens, il = batch(16, 200, 64, 30, seed=3, ragged=True)
    tg[1, int(lens[1]):] = 999  # padding beyond U_b is never read
    check_contract(ctx, e.cuda(), tg, lens, il)


def test_empty_input_empty_target_infeasible_and_blank(ctx):
    blank = 5
    e, tg, lens, il = batch(6, 60, 64, 20, seed=4, blank=blank)
    il = torch.full((6,), 60, dtype=torch.int32)
    il[1] = 0  # T_b = 0
    lens[2] = 0  # U = 0
    il[3] = 10  # 20 labels in 10 frames: infeasible
    tg[4, 1] = tg[4, 0]  # a repeat
    rc, la, st, _ = async_call(ctx, e.cuda(), tg, lens, il, blank)
    assert rc == 0
    ls, _ = sync_call(ctx, e.cuda(), tg, lens, il, blank)
    ok = st == 0
    assert ok[[0, 1, 2, 4, 5]].all()
    assert same(la[ok], ls[ok])
    if st[3]:
        assert np.isnan(la[3]) and st[3] == 1


@pytest.mark.parametrize("C_,B,T,S,sweeps", [(60, 8, 120, 20, False), (256, 8, 100, 20, True),
                                             (1024, 4, 50, 10, True)])
def test_other_label_counts(ctx, C_, B, T, S, sweeps):
    e, tg, lens, il = batch(B, T, C_, S, seed=C_, ragged=True)
    e = e.cuda()
    names = routes(ctx, lambda: check_contract(ctx, e, tg, lens, il, sweeps=sweeps))
    if sweeps:
        assert "implicit_forward" in names and "bidir_ctc" not in names
    else:
        assert "bidir_ctc" in names and "ctc_build" in names


@pytest.mark.parametrize("S", [111, 112])
def test_either_side_of_the_pair_bound(ctx, S):
    e, tg, lens, il = batch(8, 300, 64, S, seed=S)
    e = e.cuda()
    names = routes(ctx, lambda: check_contract(ctx, e, tg, lens, il))
    assert ("ctc_build" in names) == (S == 112)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("C_", [64, 256])
def test_half_precision(ctx, dtype, C_):
    e, tg, lens, il = batch(8, 150, C_, 20, seed=7, ragged=True)
    e = e.to(dtype).cuda()
    names = routes(ctx, lambda: check_contract(ctx, e, tg, lens, il, sweeps=C_ > 128))
    if C_ == 64:
        assert "bidir_ctc" in names and "widen" not in names and "narrow" not in names
    else:
        assert "widen" in names and "narrow" in names and "implicit_forward" in names


@pytest.mark.parametrize("bad", [float("inf"), float("nan")])
def test_non_finite_emission(ctx, bad):
    e, tg, lens, il = batch(4, 80, 64, 10, seed=8)
    clean = e.clone().cuda()
    e[2, 7, 3] = bad
    rc, la, st, ga = async_call(ctx, e.cuda(), tg, lens, il, 0)
    assert rc == 0 and st.tolist() == [0, 0, 1, 0]
    assert np.isnan(la[2]) and (ga[2] == 0).all()
    ls, gs = sync_call(ctx, clean, tg, lens, il, 0)  # utterances are independent on this route
    keep = [0, 1, 3]
    assert same(la[keep], ls[keep]) and torch.equal(ga[keep], gs[keep])


@pytest.mark.parametrize("case", ["negative_U", "U_over_S", "T_over_T", "negative_T", "label_C", "negative_label"])
def test_invalid_inputs(ctx, case):
    B, T, C_, S = 5, 60, 64, 12
    e, tg, lens, il = batch(B, T, C_, S, seed=9)
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
    ec = e.cuda()
    rc, la, st, ga = async_call(ctx, ec, tg_bad, lens_bad, il_bad, 0)
    assert rc == 0 and st.tolist() == [0, 2, 0, 0, 0]
    assert np.isnan(la[1]) and (ga[1] == 0).all()
    _, la2, st2, ga2 = async_call(ctx, ec, tg, lens, il, 0)
    keep = [0, 2, 3, 4]
    assert (st2 == 0).all() and same(la[keep], la2[keep]) and torch.equal(ga[keep], ga2[keep])


def test_misaligned_views_and_unsupported(ctx):
    B, T, C_, S = 4, 64, 64, 10
    e, tg, lens, il = batch(B, T, C_, S, seed=10)
    # a view one element off 16-byte alignment: bf16 is widened, float32 takes the sweeps
    for dtype, sweeps in ((torch.bfloat16, False), (torch.float32, True)):
        base = torch.empty(B * T * C_ + 1, dtype=dtype, device="cuda")
        view = base[1:].view(B, T, C_)
        view.copy_(e.to(dtype))
        names = routes(ctx, lambda: check_contract(ctx, view, tg, lens, il, sweeps=sweeps))
        assert ("widen" in names) == (dtype == torch.bfloat16)
    ec = e.cuda()
    # bounds outside both routes
    big = torch.randint(1, C_, (B, 4000), dtype=torch.int32)
    assert workspace(ctx, B, T, C_, 4000, torch.float32)[0] == capi.ERR_UNSUPPORTED
    assert async_call(ctx, ec, big, lens, il, 0)[0] == capi.ERR_UNSUPPORTED
    n = C.c_size_t()
    assert capi.lib().gtnb_ctc_loss_async_workspace(ctx.h, B, T, C_, S, 7, 1, C.byref(n)) == capi.ERR_UNSUPPORTED
    assert async_call(ctx, ec, tg, lens, il, C_)[0] == capi.ERR_UNSUPPORTED  # blank outside [0, C)
    ctx.set_flag("implicit", 0)
    try:
        assert async_call(ctx, ec, tg, lens, il, 0)[0] == capi.ERR_UNSUPPORTED
    finally:
        ctx.set_flag("implicit", 1)
    # a workspace too small or misaligned
    _, need = workspace(ctx, B, T, C_, S, torch.float32)
    assert async_call(ctx, ec, tg, lens, il, 0, ws_bytes=need // 2)[0] == capi.ERR_INVALID_ARGUMENT
    assert async_call(ctx, ec, tg, lens, il, 0, ws_offset=16)[0] == capi.ERR_INVALID_ARGUMENT


# ---- torch -------------------------------------------------------------------------------------------------------

def torch_inputs(B=8, T=100, C_=64, S=15, seed=11):
    e, tg, lens, il = batch(B, T, C_, S, seed=seed, ragged=True)
    return e.cuda(), tg.cuda(), lens.cuda(), il.cuda(), lists(tg, lens), il


@pytest.mark.parametrize("reduction", ["mean", "none"])
def test_torch_reductions_match_list_targets(reduction):
    e, tg, lens, il, tl_list, il_host = torch_inputs()
    w = torch.linspace(0.5, 2.0, e.shape[0], device="cuda")
    outs = []
    for tensor_targets in (True, False):
        x = e.clone().requires_grad_(True)
        if tensor_targets:
            loss = tl_mod.ctc_loss(x, tg, reduction=reduction, input_lengths=il, target_lengths=lens)
        else:
            loss = tl_mod.ctc_loss(x, tl_list, reduction=reduction, input_lengths=il_host)
        (loss if reduction == "mean" else (loss * w).sum()).backward()
        outs.append((loss.detach(), x.grad))
    assert outs[0][0].is_cuda and torch.equal(outs[0][0], outs[1][0])
    assert torch.equal(outs[0][1], outs[1][1])


def test_torch_no_host_wait():
    e, tg, lens, il, _, _ = torch_inputs(B=32, T=300)
    x = e.clone().requires_grad_(True)
    tl_mod.ctc_loss(x, tg, input_lengths=il, target_lengths=lens).backward()  # warm-up: context, kernels, cache
    torch.cuda.synchronize()
    done = torch.cuda.Event()
    torch.cuda._sleep(100_000_000)  # tens of milliseconds of GPU time
    loss = tl_mod.ctc_loss(x, tg, input_lengths=il, target_lengths=lens)
    done.record()
    assert not done.query(), "forward waited for the device"
    loss.backward()
    done.record()
    assert not done.query(), "backward waited for the device"
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = tl_mod.ctc_loss(x, tg, input_lengths=il, target_lengths=lens)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.isfinite(loss).item()


def test_torch_cuda_graph_training_step():
    torch.manual_seed(0)
    B, T, F, C_, S = 8, 50, 32, 64, 10
    model = torch.nn.Linear(F, C_).cuda()
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    sx = torch.randn(B, T, F, device="cuda")
    stg = torch.randint(1, C_, (B, S), device="cuda", dtype=torch.int32)
    stl = torch.full((B,), S, device="cuda", dtype=torch.int32)
    sil = torch.full((B,), T, device="cuda", dtype=torch.int32)

    def step(m, o, x, tg, tl_, il):
        o.zero_grad(set_to_none=False)
        loss = tl_mod.ctc_loss(m(x), tg, input_lengths=il, target_lengths=tl_)
        loss.backward()
        o.step()
        return loss.detach()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step(model, opt, sx, stg, stl, sil)
    torch.cuda.current_stream().wait_stream(side)
    ref = copy.deepcopy(model)
    ref_opt = torch.optim.SGD(ref.parameters(), lr=0.05)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_loss = step(model, opt, sx, stg, stl, sil)
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
        graph.replay()
        want = step(ref, ref_opt, x, tg, tl_, il)
        assert torch.equal(static_loss, want)
        for p, q in zip(model.parameters(), ref.parameters()):
            assert torch.equal(p, q)


def test_torch_autocast_bf16_step():
    torch.manual_seed(2)
    B, T, F, C_, S = 8, 60, 32, 64, 10
    model = torch.nn.Linear(F, C_).cuda()
    x = torch.randn(B, T, F, device="cuda")
    tg = torch.randint(1, C_, (B, S), device="cuda", dtype=torch.int32)
    lens = torch.full((B,), S, device="cuda", dtype=torch.int32)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits = model(x)
        assert logits.dtype == torch.bfloat16
        loss = tl_mod.ctc_loss(logits, tg, target_lengths=lens, reduction="none")
        ref = tl_mod.ctc_loss(logits.detach(), lists(tg.cpu(), lens.cpu()), reduction="none")
    assert torch.equal(loss.detach(), ref)
    loss.mean().backward()
    assert model.weight.grad is not None and torch.isfinite(model.weight.grad).all()


def test_torch_unsupported_bounds_fall_back_outside_capture():
    e, _, _, _, _, _ = torch_inputs(B=2, T=40, C_=64)
    tg = torch.randint(1, 64, (2, 4000), device="cuda", dtype=torch.int32)
    lens = torch.tensor([3, 5], device="cuda", dtype=torch.int32)
    got = tl_mod.ctc_loss(e, tg, target_lengths=lens, reduction="none")
    want = tl_mod.ctc_loss(e, [tg[0, :3].cpu().numpy(), tg[1, :5].cpu().numpy()], reduction="none")
    assert torch.equal(got, want)
