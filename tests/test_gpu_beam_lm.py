"""gtnb_lm_create / gtnb_beam_decode_lm_async and torch LanguageModel / ctc_lm_beam_decode / ngram_ctc_lm_beam_decode /
asg_lm_beam_decode on the GPU:

- against the float64 restatement (tests/beam_lm_oracle.py) at B = 32, T = 200, C = 64, K = 16, N = 4 with the
  benchmark's backoff trigram (backoff_lm), on every utterance whose decision margin exceeds 1e-3; this also holds
  gtnb_lm_create's resolved table to the walk over arcs and backoff arcs;
- scores == am + lm_weight * lm + token_bonus * length, recomputed in float32;
- with no LM, no bonus and token_beam = C, == ctc_beam_decode, ngram_ctc_beam_decode and asg_beam_decode;
- two runs bit-identical; error codes, an LM from another C included; a launch profile without a copy or a memset;
  sync-debug mode "error"; a captured ctc_lm_beam_decode + edit_distance step replayed == eager;
- a seeded quality check: the token error rate with fusion is lower than without.
"""
import ctypes as C_
import os
import sys

import numpy as np
import pytest
import torch

from gtn_b200 import capi
from gtn_b200 import torch_loss as tl
from tests import backoff_oracle as bko
from tests import beam_lm_oracle as blo

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import bench_beam_decode as bbd  # noqa: E402  (the beam benchmark's seeded emissions)
import bench_beam_lm as bbl  # noqa: E402  (the LM benchmark's graphs and quality workload)

L = capi.lib
KINDS = (capi.DENSE_CTC, capi.DENSE_BIGRAM, capi.DENSE_ASG)


@pytest.fixture(scope="module")
def ctx():
    c = capi.Ctx(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def trigram():
    """backoff_lm(C = 64): its graph, weights, restatement and LanguageModel"""
    G, w = bko.backoff_lm(np.random.default_rng(64), C=64)
    return G, w, blo.LM(G, w, 64), tl.LanguageModel(bbl.gtn_graph(G, w), 64)


def plain(kind, e, w, K, N, il=None):
    if kind == capi.DENSE_CTC:
        return tl.ctc_beam_decode(e, K, N, il)
    if kind == capi.DENSE_BIGRAM:
        return tl.ngram_ctc_beam_decode(e, w, K, N, il)
    return tl.asg_beam_decode(e, w, K, N, il)


@pytest.mark.parametrize("kind", KINDS)
def test_against_restatement(kind, trigram):
    _, _, lm_r, lm = trigram
    B, T, Cn, K, N = 32, 200, 64, 16, 4
    e, w = bbd.inputs(np.random.default_rng(40 + kind), kind, B, T, Cn)
    e, w = e * 10, None if w is None else w * 10  # (well separated decisions, as in test_gpu_beam_decode)
    il = torch.as_tensor(np.random.default_rng(4).integers(T // 2, T + 1, B).astype(np.int32)).cuda()
    alpha, beta, P = 0.5, 1.0, (16 if kind == capi.DENSE_ASG else None)
    out = bbl.decode_lm(kind, e, w, lm, K, N, alpha, beta, P, il)
    want = blo.batch(e.cpu().numpy(), kind, None if w is None else w.cpu().numpy(), il.cpu().numpy(), 0, K, N,
                     lm_r, alpha, beta, P)
    ok = want["margin"] > 1e-3
    # (ASG's stay and repeat tie by construction, and their near-ties under the LM put more utterances within 1e-3)
    assert ok.mean() >= (0.5 if kind == capi.DENSE_ASG else 0.75), want["margin"]
    got = {k: getattr(out, k).cpu().numpy() for k in ("tokens", "lengths", "scores", "am_scores", "lm_scores",
                                                       "status")}
    for b in np.nonzero(ok)[0]:
        for k in ("tokens", "lengths", "status"):
            assert np.array_equal(got[k][b], want[k][b]), (k, b)
        for k, kw in (("scores", "scores"), ("am_scores", "am"), ("lm_scores", "lm")):
            fin = np.isfinite(want[kw][b])
            assert np.array_equal(np.isfinite(got[k][b]), fin), (k, b)
            assert np.allclose(got[k][b][fin], want[kw][b][fin], rtol=1e-4, atol=1e-4), (k, b)


@pytest.mark.parametrize("kind", KINDS)
def test_scores_are_the_fused_sum_and_no_lm_is_beam_decode(kind, trigram):
    lm = trigram[3]
    e, w = bbd.inputs(np.random.default_rng(50 + kind), kind, 64, 300, 64)
    for lw, tb, P in ((0.7, -0.3, None), (2.0, 1.5, 8)):
        out = bbl.decode_lm(kind, e, w, lm, 16, 4, lw, tb, P)
        live = out.lengths >= 0
        want = out.am_scores + (lw * out.lm_scores + tb * out.lengths.float())
        assert live[:, 0].all() and torch.equal(out.scores[live], want[live])
        assert torch.isneginf(out.scores[~live]).all() and torch.isneginf(out.am_scores[~live]).all()
    a = plain(kind, e, w, 16, 4)
    b = bbl.decode_lm(kind, e, w, None, 16, 4, 1.0, 0.0, None)
    for k in ("tokens", "lengths", "scores", "status"):
        assert torch.equal(getattr(a, k), getattr(b, k)), (kind, k)
    assert torch.equal(b.am_scores, b.scores) and (b.lm_scores[b.lengths >= 0] == 0).all()


def test_two_runs_bit_identical_and_status(trigram):
    lm = trigram[3]
    for kind in KINDS:
        e, w = bbd.inputs(np.random.default_rng(60 + kind), kind, 64, 300, 64)
        e[1, 7, 3] = float("nan")
        il = torch.full((64,), 300, dtype=torch.int32, device="cuda")
        il[2], il[3] = 301, 0
        a = bbl.decode_lm(kind, e, w, lm, 32, 8, 0.5, 1.0, 12, il)
        b = bbl.decode_lm(kind, e, w, lm, 32, 8, 0.5, 1.0, 12, il)
        for x, y in zip(a, b):  # (bit patterns: the flagged rows hold NaN)
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), kind
        st = a.status.cpu().numpy()
        assert st[1] == 1 and st[2] == 2 and set(st[4:]) <= {0, 3}
        for x in (a.scores, a.am_scores, a.lm_scores):
            assert torch.isnan(x[1]).all() and torch.isnan(x[2]).all()
        assert a.lengths[3, 0] == 0 and a.am_scores[3, 0] == 0 and a.lm_scores[3, 0] == 0  # (no eos arcs: end 0)


def test_lm_checks_and_error_codes(ctx):
    C = 8
    G, w = bko.backoff_ngram(np.random.default_rng(3), C, 3)

    def create(G, w, C=C):
        v, keep = capi.make_view(G["flags"], G["src"], G["dst"], G["ilabel"], G["olabel"], w)
        h = C_.c_void_p()
        rc = L().gtnb_lm_create(ctx.h, C_.byref(v), C, C_.byref(h))
        return rc, h

    rc, h = create(G, w)
    assert rc == 0
    bad = []
    g = dict(G, olabel=G["olabel"].copy())
    g["olabel"][0] = (g["olabel"][0] + 1) % C
    bad.append((g, w))  # a transducer
    g = dict(G, flags=G["flags"].copy())
    g["flags"][1] |= 1
    bad.append((g, w))  # two start nodes
    g = dict(G, flags=G["flags"] & 2)
    bad.append((g, w))  # no start node
    g = dict(G, ilabel=G["ilabel"].copy(), olabel=G["olabel"].copy())
    g["ilabel"][0] = g["olabel"][0] = C + 1
    bad.append((g, w))  # a label beyond C
    a = int(np.flatnonzero(G["ilabel"] >= 0)[1])
    g = {k: np.concatenate([v, v[[a]]]) if k != "flags" else v for k, v in G.items()}
    bad.append((g, np.concatenate([w, w[[a]]])))  # two arcs with one label
    e0 = int(np.flatnonzero(G["ilabel"] < 0)[0])
    g = {k: np.concatenate([v, v[[e0]]]) if k != "flags" else v for k, v in G.items()}
    bad.append((g, np.concatenate([w, w[[e0]]])))  # two epsilon arcs
    for x in (np.nan, np.inf):
        w2 = w.copy()
        w2[0] = x
        bad.append((G, w2))
    s = int(G["src"][e0])  # a state that backs off: an epsilon arc from the root into it closes a cycle
    g = dict(flags=G["flags"], src=np.append(G["src"], 0), dst=np.append(G["dst"], s), ilabel=np.append(G["ilabel"], -1),
             olabel=np.append(G["olabel"], -1))
    bad.append((g, np.append(w, np.float32(-1.0))))
    for g, ww in bad:
        rc2, h2 = create(g, ww)
        assert rc2 == capi.ERR_INVALID_ARGUMENT and not h2.value
    w2 = w.copy()
    w2[0] = -np.inf  # a forbidden arc is no error
    rc2, h2 = create(G, w2)
    assert rc2 == 0
    L().gtnb_lm_destroy(ctx.h, h2)
    assert create(G, w, 257)[0] == capi.ERR_UNSUPPORTED
    big = dict(flags=np.full((1 << 25) // 9 + 1, 0, np.uint8), src=np.zeros(0, np.int32), dst=np.zeros(0, np.int32),
               ilabel=np.zeros(0, np.int32), olabel=np.zeros(0, np.int32))
    big["flags"][0] = 1
    assert create(big, np.zeros(0, np.float32))[0] == capi.ERR_UNSUPPORTED
    # the call
    n = C_.c_size_t()
    W = L().gtnb_beam_decode_lm_async_workspace
    assert W(ctx.h, 4, 10, C, 0, capi.DENSE_CTC, 8, 2, 0, C_.byref(n)) == capi.ERR_UNSUPPORTED
    assert W(ctx.h, 4, 10, C, 0, capi.DENSE_CTC, 8, 2, C + 1, C_.byref(n)) == capi.ERR_UNSUPPORTED
    assert W(ctx.h, 4, 10, C, 0, capi.DENSE_CTC, 65, 2, C, C_.byref(n)) == capi.ERR_UNSUPPORTED
    m = C_.c_size_t()
    for kind in KINDS:
        assert W(ctx.h, 4, 10, C, 0, kind, 8, 2, 3, C_.byref(n)) == 0
        assert L().gtnb_beam_decode_async_workspace(ctx.h, 4, 10, C, 0, kind, 8, 2, C_.byref(m)) == 0
        assert n.value == m.value
    B, T = 4, 10
    assert W(ctx.h, B, T, C, 0, capi.DENSE_CTC, 8, 2, C, C_.byref(n)) == 0
    e = torch.zeros((B, T, C), device="cuda")
    out = [torch.empty(s, dtype=dt, device="cuda") for s, dt in
           (((B, 2, T), torch.int32), ((B, 2), torch.int32), ((B, 2), torch.float32), ((B, 2), torch.float32),
            ((B, 2), torch.float32), ((B,), torch.int32))]
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    rc16, h16 = create(G, w, 16)
    assert rc16 == 0

    def go(lm=h, lw=1.0, tb=0.0, P=C, nbytes=n.value):
        return L().gtnb_beam_decode_lm_async(ctx.h, None, B, T, C, e.data_ptr(), 0, None, capi.DENSE_CTC, None, 0, 8,
                                             2, lm, lw, tb, P, *[o.data_ptr() for o in out], ws.data_ptr(), nbytes)
    assert go() == 0 and go(lm=None) == 0
    assert go(lw=-0.5) == capi.ERR_INVALID_ARGUMENT
    assert go(lw=float("inf")) == capi.ERR_INVALID_ARGUMENT
    assert go(lw=float("nan")) == capi.ERR_INVALID_ARGUMENT
    assert go(tb=float("nan")) == capi.ERR_INVALID_ARGUMENT
    assert go(tb=float("-inf")) == capi.ERR_INVALID_ARGUMENT
    assert go(lm=h16) == capi.ERR_INVALID_ARGUMENT  # an LM made for another C
    assert go(P=0) == capi.ERR_UNSUPPORTED and go(P=C + 1) == capi.ERR_UNSUPPORTED
    assert go(nbytes=n.value - 256) == capi.ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    L().gtnb_lm_destroy(ctx.h, h)
    L().gtnb_lm_destroy(ctx.h, h16)
    with pytest.raises(RuntimeError):
        tl.LanguageModel(bbl.gtn_graph(bad[1][0], w), C)
    lm16 = tl.LanguageModel(bbl.gtn_graph(G, w), 16)
    with pytest.raises(RuntimeError):
        tl.ctc_lm_beam_decode(e, lm16)


def test_launch_profile(ctx, trigram):
    lm = trigram[3]
    B, T, Cn = 8, 50, 64
    e = torch.randn((B, T, Cn), device="cuda")
    w = torch.randn(Cn + Cn * Cn, device="cuda")
    n = C_.c_size_t()
    ctx._check(L().gtnb_beam_decode_lm_async_workspace(ctx.h, B, T, Cn, 0, capi.DENSE_ASG, 16, 4, 16, C_.byref(n)))
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    out = [torch.empty(s, dtype=dt, device="cuda") for s, dt in
           (((B, 4, T), torch.int32), ((B, 4), torch.int32), ((B, 4), torch.float32), ((B, 4), torch.float32),
            ((B, 4), torch.float32), ((B,), torch.int32))]

    def go():
        return L().gtnb_beam_decode_lm_async(ctx.h, None, B, T, Cn, e.data_ptr(), 0, None, capi.DENSE_ASG,
                                             w.data_ptr(), 0, 16, 4, lm.h, 0.5, 1.0, 16,
                                             *[o.data_ptr() for o in out], ws.data_ptr(), n.value)
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
    assert set(got) == {"beam_weights", "beam_decode_lm"} and ctx.launches - before == 2, got
    copies = [ev.name for ev in prof.events() if "Memcpy" in ev.name or "Memset" in ev.name]
    assert not copies, copies


def test_no_wait_sync_debug_and_captured_step(trigram):
    lm = trigram[3]
    rng = np.random.default_rng(9)
    B, T, Cn = 32, 300, 64
    e, _ = bbd.inputs(rng, capi.DENSE_CTC, B, T, Cn)
    il = torch.as_tensor(rng.integers(T // 2, T + 1, B).astype(np.int32)).cuda()
    r = torch.as_tensor(rng.integers(1, Cn, (B, 120)).astype(np.int32)).cuda()
    rl = torch.as_tensor(rng.integers(0, 121, B).astype(np.int32)).cuda()

    def step():
        out = tl.ctc_lm_beam_decode(e, lm, 0.5, 1.0, 16, 4, 16, il)
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
        e.copy_(bbd.inputs(np.random.default_rng(seed), capi.DENSE_CTC, B, T, Cn)[0])
        g.replay()
        eager = step()
        torch.cuda.synchronize()
        for c, w_ in zip(cap, eager):
            for x, y in zip(c, w_):
                assert (x is None and y is None) or torch.equal(x, y), seed
        assert (eager[1].status == 0).all()
    del g
    small = bbl.gtn_graph(*bko.backoff_ngram(np.random.default_rng(1), 8, 2))
    with pytest.raises(RuntimeError):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            tl.LanguageModel(small, 8)


def test_fusion_lowers_the_token_error_rate():
    G, w, _, e, refs = bbl.quality_workload()
    lm = tl.LanguageModel(bbl.gtn_graph(G, w), e.shape[2])
    ed = torch.as_tensor(e).cuda()
    without = bbl.ter(*tl.ctc_lm_beam_decode(ed, None, 1.0, 0.0, 8)[:2], refs)
    fused = bbl.ter(*tl.ctc_lm_beam_decode(ed, lm, 1.0, 0.0, 8)[:2], refs)
    assert fused < 0.75 * without, (fused, without)
