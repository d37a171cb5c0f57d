"""gtnb_beam_decode_async and torch ctc_beam_decode / ngram_ctc_beam_decode / asg_beam_decode on the GPU:

- the loss calls as referee: each hypothesis fed back as a target into ctc_loss / ngram_ctc_loss / asg_loss
  (reduction="none") gives score_k + loss_k = the denominator for every k where the beam is exhaustive, and
  score_k <= denominator - loss_k at the benchmark's shapes (the lower-bound property); hypotheses are distinct,
  sorted, blank-free and in range;
- against the float64 restatement (tests/beam_oracle.py) at B = 32, T = 200, C = 64, K = 16, N = 4, on every
  utterance whose decision margin exceeds 1e-3;
- T_b = 0 (the empty transcript, score 0: ctc_loss's numerator there, where ngram_ctc_loss gives NaN); bf16 / fp16
  emissions;
- two runs bit-identical; bounds, bad arguments and a short workspace; a launch profile of the two kernels without a
  copy or a memset; sync-debug mode "error"; a captured ngram_ctc_beam_decode + edit_distance step replayed == eager.
"""
import ctypes as C_
import os
import sys

import numpy as np
import pytest
import torch

from gtn_b200 import capi
from gtn_b200 import torch_loss as tl
from tests import beam_oracle as bo

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import bench_beam_decode as bbd  # noqa: E402  (the benchmark's seeded workloads)

L = capi.lib
KINDS = (capi.DENSE_CTC, capi.DENSE_BIGRAM, capi.DENSE_ASG)


@pytest.fixture(scope="module")
def ctx():
    c = capi.Ctx(0)
    yield c
    c.close()


def decode(kind, e, w, beam, nbest, il=None):
    if kind == capi.DENSE_CTC:
        return tl.ctc_beam_decode(e, beam, nbest, il)
    if kind == capi.DENSE_BIGRAM:
        return tl.ngram_ctc_beam_decode(e, w, beam, nbest, il)
    return tl.asg_beam_decode(e, w, beam, nbest, il)


def denominator(kind, e, w):
    """float64 forwardScore of the denominator graph per utterance (all T frames)"""
    e = e.double()
    B, T, Cn = e.shape
    if kind == capi.DENSE_CTC:
        return torch.logsumexp(e, -1).sum(-1)
    wd = w.double()
    W = (wd[Cn:] if kind == capi.DENSE_ASG else wd).view(Cn, Cn)
    first = wd[:Cn] if kind == capi.DENSE_ASG else torch.logsumexp(W, 1)
    a = first + e[:, 0]
    for t in range(1, T):
        a = torch.logsumexp(a[:, None, :] + W[None], -1) + e[:, t]
    return torch.logsumexp(a, -1)


def losses_of(kind, e, w, out):
    """loss of every live hypothesis as a target, [B, N] float64 (NaN where unused)"""
    B, N, T = out.tokens.shape
    live = out.lengths >= 0
    ee = e.repeat_interleave(N, 0)
    tg = out.tokens.reshape(B * N, T).clamp(min=0)
    tlen = out.lengths.reshape(-1).clamp(min=0)
    if kind == capi.DENSE_CTC:
        ls = tl.ctc_loss(ee.float(), tg, 0, "none", None, tlen)
    elif kind == capi.DENSE_BIGRAM:
        ls = tl.ngram_ctc_loss(ee.float(), w, tg, None, 0, "none", False, tlen)
    else:
        ls = tl.asg_loss(ee.float(), w, tg, "none", False, None, tlen)
    ls = ls.double().view(B, N)
    return torch.where(live, ls, torch.full_like(ls, float("nan")))


def hypotheses_well_formed(kind, out, Cn, blank=0):
    tok, ln, sc = out.tokens.cpu().numpy(), out.lengths.cpu().numpy(), out.scores.cpu().numpy()
    for b in range(tok.shape[0]):
        seen = set()
        for n in range(tok.shape[1]):
            if ln[b, n] < 0:
                assert np.isneginf(sc[b, n:]).all() and (ln[b, n:] == -1).all()
                break
            y = tuple(tok[b, n, :ln[b, n]])
            assert (tok[b, n, ln[b, n]:] == -1).all()
            assert all(0 <= c < Cn for c in y) and (kind == capi.DENSE_ASG or blank not in y)
            assert y not in seen
            seen.add(y)
            if n:
                assert sc[b, n] <= sc[b, n - 1]


@pytest.mark.parametrize("kind", KINDS)
def test_loss_calls_referee_exhaustive(kind):
    rng = np.random.default_rng(kind)
    Cn = 2 if kind == capi.DENSE_ASG else 3
    B, T, N = 8, 5, 16
    e, w = bbd.inputs(rng, kind, B, T, Cn)
    out = decode(kind, e, w, 64, N)
    assert (out.status.cpu() != 1).all() and (out.status.cpu() != 2).all()
    hypotheses_well_formed(kind, out, Cn)
    den = denominator(kind, e, w)
    tot = out.scores.double() + losses_of(kind, e, w, out)
    live = out.lengths >= 0
    for b in range(B):
        v = tot[b][live[b]]
        assert torch.allclose(v, den[b].expand_as(v), rtol=1e-4, atol=1e-4), (b, v, den[b])


@pytest.mark.parametrize("kind", KINDS)
def test_lower_bound_at_benchmark_shapes(kind):
    B, T, Cn = (64, 1000, 64) if kind == capi.DENSE_CTC else (32, 500, 64)
    e, w = bbd.inputs(np.random.default_rng(10 + kind), kind, B, T, Cn)
    out = decode(kind, e, w, 16, 8)
    hypotheses_well_formed(kind, out, Cn)
    num = denominator(kind, e, w)[:, None] - losses_of(kind, e, w, out)
    live = out.lengths >= 0
    sc = out.scores.double()
    assert (sc[live] <= num[live] + 1e-4 * num[live].abs()).all()


@pytest.mark.parametrize("kind", KINDS)
def test_against_restatement(kind):
    B, T, Cn, K, N = 32, 200, 64, 16, 4
    e, w = bbd.inputs(np.random.default_rng(20 + kind), kind, B, T, Cn)
    # at a 10x log-probability scale: over 200 frames, unit-scale rows put candidates within 1e-3 of the boundary
    e, w = e * 10, None if w is None else w * 10
    il = torch.as_tensor(np.random.default_rng(3).integers(T // 2, T + 1, B).astype(np.int32)).cuda()
    out = decode(kind, e, w, K, N, il)
    want = bo.batch(e.cpu().numpy(), kind, None if w is None else w.cpu().numpy(), il.cpu().numpy(), 0, K, N)
    ok = want["margin"] > 1e-3
    assert ok.mean() >= 0.75, want["margin"]
    got = {k: getattr(out, k).cpu().numpy() for k in ("tokens", "lengths", "scores", "status")}
    for b in np.nonzero(ok)[0]:
        for k in ("tokens", "lengths", "status"):
            assert np.array_equal(got[k][b], want[k][b]), (k, b)
        fin = np.isfinite(want["scores"][b])
        assert np.allclose(got["scores"][b][fin], want["scores"][b][fin], rtol=1e-4), b


def test_empty_utterance_and_half_emissions():
    rng = np.random.default_rng(4)
    B, T, Cn = 16, 120, 32
    e, _ = bbd.inputs(rng, capi.DENSE_CTC, B, T, Cn)
    il = torch.full((B,), T, dtype=torch.int32, device="cuda")
    il[3] = 0
    out = tl.ctc_beam_decode(e, 8, 4, il)
    assert out.status[3] == 0 and out.scores[3, 0] == 0 and out.lengths[3, 0] == 0
    assert (out.tokens[3] == -1).all() and torch.isinf(out.scores[3, 1:]).all()
    # ctc_loss of the empty target at T_b = 0 is 0: the decoder's score is its numerator there
    loss = tl.ctc_loss(e, torch.ones((B, 2), dtype=torch.int32, device="cuda"), 0, "none", il,
                       torch.zeros(B, dtype=torch.int32, device="cuda"))
    assert loss[3] == 0
    # n-gram CTC gives NaN at T_b = 0 (its E accepts nothing); the decoder still returns the empty transcript
    w = torch.zeros(Cn * Cn, device="cuda")
    loss = tl.ngram_ctc_loss(e, w, torch.ones((B, 2), dtype=torch.int32, device="cuda"), il, 0, "none", False,
                             torch.zeros(B, dtype=torch.int32, device="cuda"))
    assert torch.isnan(loss[3])
    out = tl.ngram_ctc_beam_decode(e, w, 8, 4, il)
    assert out.status[3] == 0 and out.scores[3, 0] == 0 and out.lengths[3, 0] == 0
    for dt in (torch.bfloat16, torch.float16):
        h = e.to(dt)
        a = tl.ctc_beam_decode(h, 8, 4, il)
        b = tl.ctc_beam_decode(h.float(), 8, 4, il)
        for x, y in zip(a, b):
            assert torch.equal(x, y), dt


def test_two_runs_bit_identical_and_status():
    for kind in KINDS:
        e, w = bbd.inputs(np.random.default_rng(30 + kind), kind, 64, 300, 48)
        e[1, 7, 3] = float("nan")
        il = torch.full((64,), 300, dtype=torch.int32, device="cuda")
        il[2] = 301
        a = decode(kind, e, w, 32, 8, il)
        b = decode(kind, e, w, 32, 8, il)
        for x, y in zip(a, b):  # (bit patterns: the flagged rows hold NaN)
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), kind
        st = a.status.cpu().numpy()
        assert st[1] == 1 and st[2] == 2 and set(st[3:]) <= {0, 3}
        assert torch.isnan(a.scores[1]).all() and (a.tokens[2] == -1).all()


def test_error_codes(ctx):
    n = C_.c_size_t()
    W = L().gtnb_beam_decode_async_workspace
    assert W(ctx.h, 4, 10, 64, 0, capi.DENSE_CTC, 65, 1, C_.byref(n)) == capi.ERR_UNSUPPORTED
    assert W(ctx.h, 4, 10, 64, 0, capi.DENSE_CTC, 8, 9, C_.byref(n)) == capi.ERR_UNSUPPORTED
    assert W(ctx.h, 4, 10, 64, 0, capi.DENSE_CTC, 8, 0, C_.byref(n)) == capi.ERR_UNSUPPORTED
    assert W(ctx.h, 4, 10, 257, 0, capi.DENSE_ASG, 8, 1, C_.byref(n)) == capi.ERR_UNSUPPORTED
    assert W(ctx.h, 4, 10, 64, 7, capi.DENSE_CTC, 8, 1, C_.byref(n)) == capi.ERR_UNSUPPORTED
    assert W(ctx.h, 4, 10, 64, 0, 9, 8, 1, C_.byref(n)) == capi.ERR_INVALID_ARGUMENT
    assert W(ctx.h, 0, 10, 256, 0, capi.DENSE_BIGRAM, 64, 64, C_.byref(n)) == 0 and n.value == 0
    B, T, Cn = 4, 10, 64
    assert W(ctx.h, B, T, Cn, 0, capi.DENSE_BIGRAM, 8, 2, C_.byref(n)) == 0
    r = lambda x: (x + 255) // 256 * 256  # noqa: E731
    assert n.value == r(2 * (B * T * 8 + 16)) + r(4 * (Cn * Cn + 16)) + 2 * r(4 * (Cn + 16))
    e = torch.zeros((B, T, Cn), device="cuda")
    w = torch.zeros(Cn * Cn, device="cuda")
    tok = torch.empty((B, 2, T), dtype=torch.int32, device="cuda")
    ln = torch.empty((B, 2), dtype=torch.int32, device="cuda")
    sc = torch.empty((B, 2), device="cuda")
    ws = torch.empty(n.value + 256, dtype=torch.uint8, device="cuda")

    def go(kind=capi.DENSE_BIGRAM, wp=w.data_ptr(), blank=0, nbytes=n.value, off=0, tp=tok.data_ptr()):
        return L().gtnb_beam_decode_async(ctx.h, None, B, T, Cn, e.data_ptr(), 0, None, kind, wp, blank, 8, 2, tp,
                                          ln.data_ptr(), sc.data_ptr(), None, ws.data_ptr() + off, nbytes)
    assert go() == 0
    assert go(nbytes=n.value - 256) == capi.ERR_INVALID_ARGUMENT
    assert go(off=16) == capi.ERR_INVALID_ARGUMENT
    assert go(wp=None) == capi.ERR_INVALID_ARGUMENT
    assert go(kind=capi.DENSE_CTC) == capi.ERR_INVALID_ARGUMENT
    assert go(tp=None) == capi.ERR_INVALID_ARGUMENT
    assert go(blank=Cn) == capi.ERR_UNSUPPORTED
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError):
        tl.ctc_beam_decode(e, 65)
    with pytest.raises(RuntimeError):
        tl.ctc_beam_decode(torch.zeros((2, 3, 300), device="cuda"))


def test_launch_profile(ctx):
    B, T, Cn = 8, 50, 64
    e = torch.randn((B, T, Cn), device="cuda")
    w = torch.randn(Cn + Cn * Cn, device="cuda")
    n = C_.c_size_t()
    ctx._check(L().gtnb_beam_decode_async_workspace(ctx.h, B, T, Cn, 0, capi.DENSE_ASG, 16, 4, C_.byref(n)))
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    out = [torch.empty(s, dtype=dt, device="cuda") for s, dt in
           (((B, 4, T), torch.int32), ((B, 4), torch.int32), ((B, 4), torch.float32), ((B,), torch.int32))]

    def go():
        return L().gtnb_beam_decode_async(ctx.h, None, B, T, Cn, e.data_ptr(), 0, None, capi.DENSE_ASG, w.data_ptr(),
                                          0, 16, 4, *[o.data_ptr() for o in out], ws.data_ptr(), n.value)
    assert go() == 0
    torch.cuda.synchronize()
    ctx.profile(True)
    ctx.profile_read()
    before = ctx.launches
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        assert go() == 0
        torch.cuda.synchronize()
    got = ctx.profile_read()
    ctx.profile(False)
    assert set(got) == {"beam_weights", "beam_decode"} and ctx.launches - before == 2, got
    copies = [ev.name for ev in prof.events() if "Memcpy" in ev.name or "Memset" in ev.name]
    assert not copies, copies


def test_no_wait_sync_debug_and_captured_step():
    rng = np.random.default_rng(8)
    B, T, Cn = 32, 300, 40
    e, w = bbd.inputs(rng, capi.DENSE_BIGRAM, B, T, Cn)
    il = torch.as_tensor(rng.integers(T // 2, T + 1, B).astype(np.int32)).cuda()
    r = torch.as_tensor(rng.integers(1, Cn, (B, 120)).astype(np.int32)).cuda()
    rl = torch.as_tensor(rng.integers(0, 121, B).astype(np.int32)).cuda()

    def step():
        out = tl.ngram_ctc_beam_decode(e, w, 16, 4, il)
        return out, tl.edit_distance(out.tokens[:, 0], out.lengths[:, 0], r, rl)
    step()
    torch.cuda.synchronize()
    done = torch.cuda.Event()
    torch.cuda._sleep(100_000_000)
    step()
    done.record()
    assert not done.query(), "the call waited for the device"
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            cap = step()
    torch.cuda.current_stream().wait_stream(s)
    for seed in (1, 2):
        rr = np.random.default_rng(seed)
        e.copy_(bbd.inputs(rr, capi.DENSE_BIGRAM, B, T, Cn)[0])
        g.replay()
        eager = step()
        torch.cuda.synchronize()
        for c, w_ in zip(cap, eager):
            for x, y in zip(c, w_):
                assert (x is None and y is None) or torch.equal(x, y), seed
        assert (eager[1].status == 0).all()
    del g
