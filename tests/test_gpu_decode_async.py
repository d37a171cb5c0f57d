"""gtnb_transitions_create / gtnb_viterbi_transitions_async, gtnb_viterbi_dense_async and torch TransitionGraph /
transitions_decode / asg_decode / ngram_ctc_decode, on the GPU.

The contract: with the synchronous decoders' "exact_ties" flag off, every utterance of status 0 or 3 has ==
paths, arcs and scores; with it on (their default), every status-0 utterance is ==.  The synchronous decoders are
themselves held to the reference; one sample here goes to the reference directly.  A bad length or a non-finite
emission is flagged alone, the other rows unchanged."""
import ctypes as C_
import os
import sys

import numpy as np
import pytest
import torch

from gtn_b200 import capi
from gtn_b200 import torch_loss as tl
from tests import backoff_oracle as bo
from tests import sparse_trans_oracle as st
from tests import sparse_viterbi_oracle as sv
from tests import util

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import bench_sparse_transitions as bst  # noqa: E402  (the benchmark's 2000-state token LM)

L = capi.lib


@pytest.fixture(scope="module")
def ctx():
    c = capi.Ctx(0)
    yield c
    c.close()


def view_of(G):
    return capi.make_view(G["flags"], G["src"], G["dst"], G["olabel"], G["olabel"])


class Handle:
    def __init__(self, ctx, G, C, backoff=False):
        self.ctx = ctx
        v, keep = view_of(G)
        h = C_.c_void_p()
        self.rc = L().gtnb_transitions_create(ctx.h, C_.byref(v), C, int(backoff), C_.byref(h))
        self.h = h

    def __del__(self):
        if self.h.value:
            L().gtnb_transitions_destroy(self.ctx.h, self.h)


def workspace(ctx, h, B, T):
    n = C_.c_size_t()
    ctx._check(L().gtnb_viterbi_transitions_async_workspace(ctx.h, h.h, B, T, C_.byref(n)))
    return n.value


def decode(ctx, h, e, w, lens=None, ws=None, arcs=True):
    """gtnb_viterbi_transitions_async on the current stream -> (paths, scores, arcs, status) as numpy"""
    B, T, _ = e.shape
    ed = torch.as_tensor(e).cuda()
    wd = torch.as_tensor(w).cuda() if len(w) else torch.zeros(1, device="cuda")
    ld = None if lens is None else torch.as_tensor(lens, dtype=torch.int32).cuda()
    n = workspace(ctx, h, B, T)
    wsd = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda") if ws is None else ws
    p = torch.full((B, T), -7, dtype=torch.int32, device="cuda")
    a = torch.full((B, T), -7, dtype=torch.int32, device="cuda")
    s = torch.full((B,), 7.0, device="cuda")
    st_ = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    ctx._check(L().gtnb_viterbi_transitions_async(
        ctx.h, torch.cuda.current_stream().cuda_stream, h.h, B, T, ed.data_ptr(), None if ld is None else ld.data_ptr(),
        wd.data_ptr(), p.data_ptr(), a.data_ptr() if arcs else None, s.data_ptr(), st_.data_ptr(), wsd.data_ptr(), n))
    torch.cuda.synchronize()
    return p.cpu().numpy(), s.cpu().numpy(), a.cpu().numpy(), st_.cpu().numpy()


def sync_decode(ctx, G, e, w, lens, backoff, exact_ties):
    v = view_of(G)
    f = ctx.viterbi_backoff_dev if backoff else ctx.viterbi_sparse_dev
    ctx.set_flag("exact_ties", exact_ties)
    try:
        return f(e, v, w, input_lens=lens)
    finally:
        ctx.set_flag("exact_ties", 1)


def parity(ctx, G, C, e, w, lens, backoff=False, cluster=0):
    ctx.set_flag("sparse_cluster", cluster)
    try:
        h = Handle(ctx, G, C, backoff)
        ctx._check(h.rc)
        p, s, a, status = decode(ctx, h, e, w, lens)
        off = sync_decode(ctx, G, e, w, lens, backoff, 0)
        on = sync_decode(ctx, G, e, w, lens, backoff, 1)
    finally:
        ctx.set_flag("sparse_cluster", 0)
    assert set(np.unique(status)) <= {0, 3}, status
    for b in range(len(status)):
        (pr, sr, ar) = off
        assert np.array_equal(s[b], sr[b], equal_nan=True) and np.array_equal(p[b], pr[b]) and \
            np.array_equal(a[b], ar[b]), b
        if status[b] == 0:
            (pr, sr, ar) = on
            assert np.array_equal(s[b], sr[b], equal_nan=True) and np.array_equal(p[b], pr[b]) and \
                np.array_equal(a[b], ar[b]), b
    return status


def ragged(rng, B, T):
    lens = rng.integers(T // 2, T + 1, B).astype(np.int32)
    lens[0], lens[-1] = T, 0
    return lens


@pytest.mark.parametrize("case", ["trigram30", "lm2000", "backoff_trigram64", "cluster_trigram64"])
def test_parity_with_the_synchronous_decoders(ctx, case):
    rng = np.random.default_rng(7)
    backoff, cluster = False, 0
    if case == "trigram30":
        C, B, T, G = 30, 128, 200, st.trigram_graph(30)
    elif case == "lm2000":
        C, B, T = 64, 128, 500
        G = bst.sparse_lm(rng, 2000, C, 16)
    elif case == "backoff_trigram64":
        C, B, T, G, backoff = 64, 128, 500, bo.backoff_lm(rng)[0], True
    else:
        C, B, T, G, cluster = 64, 4, 50, st.trigram_graph(64), 1
    e, _ = util.bench_inputs(B, T, C, 10)
    w = rng.uniform(-2, 0, len(G["src"])).astype(np.float32)
    status = parity(ctx, G, C, e, w, ragged(rng, B, T), backoff, cluster)
    assert (status == 0).sum() > B // 2


@pytest.mark.parametrize("split", [2, 4, 8])
@pytest.mark.parametrize("backoff", [False, True])
def test_forced_cluster_splits(ctx, split, backoff):
    rng = np.random.default_rng(split)
    C = 16
    G = bo.backoff_ngram(rng, C, 3)[0] if backoff else st.sparse_graph(rng, 200, 3000, C, n_start=3, n_accept=20)
    e = rng.uniform(-3, 3, (8, 40, C)).astype(np.float32)
    w = rng.uniform(-1, 0, len(G["src"])).astype(np.float32)
    parity(ctx, G, C, e, w, ragged(rng, 8, 40), backoff, split)


def test_ties_are_flagged_3_and_match_exact_ties_off(ctx):
    rng = np.random.default_rng(3)
    C, B, T = 30, 16, 40
    G = st.trigram_graph(C)
    e = rng.integers(0, 2, (B, T, C)).astype(np.float32)
    w = np.zeros(len(G["src"]), np.float32)
    status = parity(ctx, G, C, e, w, ragged(rng, B, T))
    assert (status == 3).any()


def test_reference_sample(ctx, oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing"
    oracle.libref()
    rng = np.random.default_rng(11)
    C = 28
    G = st.sparse_graph(rng, 12, 70, C, n_start=3, n_accept=3, label_hi=C + 2)
    e = rng.uniform(-3, 3, (6, 15, C)).astype(np.float32)
    lens = np.asarray([15, 9, 0, 15, 12, 1], np.int32)
    w = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    h = Handle(ctx, G, C)
    ctx._check(h.rc)
    p, s, a, status = decode(ctx, h, e, w, lens)
    pr, sr, ar = sv.ref_sparse_viterbi(e, G, w, lens)
    assert (status == 0).all(), status
    assert np.array_equal(s, sr) and np.array_equal(p, pr) and np.array_equal(a, ar)


@pytest.mark.parametrize("backoff", [False, True])
def test_bad_inputs_are_flagged_alone(ctx, backoff):
    rng = np.random.default_rng(5)
    C, B, T = 30, 8, 30
    G = bo.backoff_ngram(rng, C, 3)[0] if backoff else st.trigram_graph(C)
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    w = rng.uniform(-1, 0, len(G["src"])).astype(np.float32)
    w[::7] = -np.inf  # -inf only forbids an arc: no flag
    lens = np.full(B, T, np.int32)
    h = Handle(ctx, G, C, backoff)
    ctx._check(h.rc)
    clean = decode(ctx, h, e, w, lens)
    assert (clean[3] == 0).all() or set(np.unique(clean[3])) <= {0, 3}
    bad_e, bad_l = e.copy(), lens.copy()
    bad_l[1], bad_l[2] = -1, T + 1
    bad_e[3, 5, :] = np.nan
    bad_e[4, 2, 0] = np.inf
    got = decode(ctx, h, bad_e, w, bad_l)
    assert list(got[3][1:5]) == [2, 2, 1, 1]
    for b in (1, 2, 3, 4):
        assert np.isnan(got[1][b]) and (got[0][b] == -1).all() and (got[2][b] == -1).all()
    for b in (0, 5, 6, 7):
        assert got[3][b] == clean[3][b] and np.array_equal(got[0][b], clean[0][b]) and got[1][b] == clean[1][b]
        assert np.array_equal(got[2][b], clean[2][b])


def test_errors(ctx):
    rng = np.random.default_rng(0)
    C, B, T = 30, 4, 20
    G = st.trigram_graph(C)
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    w = rng.uniform(-1, 0, len(G["src"])).astype(np.float32)
    h = Handle(ctx, G, C)
    ctx._check(h.rc)
    n = workspace(ctx, h, B, T)
    big = torch.empty(n + 512, dtype=torch.uint8, device="cuda")
    ed, wd = torch.as_tensor(e).cuda(), torch.as_tensor(w).cuda()
    out = [torch.empty((B, T), dtype=torch.int32, device="cuda"), torch.empty(B, device="cuda")]

    def call(ws, nbytes, BB=B):
        return L().gtnb_viterbi_transitions_async(ctx.h, None, h.h, BB, T, ed.data_ptr(), None, wd.data_ptr(),
                                                  out[0].data_ptr(), None, out[1].data_ptr(), None, ws, nbytes)
    assert call(big.data_ptr(), n) == 0
    assert call(big.data_ptr(), n - 256) == capi.ERR_INVALID_ARGUMENT  # too small
    assert call(big.data_ptr() + 16, n) == capi.ERR_INVALID_ARGUMENT  # misaligned
    assert call(None, n) == capi.ERR_INVALID_ARGUMENT
    assert call(None, 0, 0) == 0  # B = 0
    torch.cuda.synchronize()
    # G outside the device envelope, the implicit flag off, epsilon arcs without backoff
    big_G = Handle(ctx, st.trigram_graph(64), 64)
    assert big_G.rc == capi.ERR_UNSUPPORTED and "gtnb_viterbi_sparse" in L().gtnb_last_error(ctx.h).decode()
    ctx.set_flag("implicit", 0)
    try:
        assert Handle(ctx, G, C).rc == capi.ERR_UNSUPPORTED
    finally:
        ctx.set_flag("implicit", 1)
    assert Handle(ctx, bo.backoff_ngram(rng, C, 2)[0], C).rc == capi.ERR_UNSUPPORTED
    assert Handle(ctx, bo.eps_cycle_graph()[0], 4, True).rc == capi.ERR_INVALID_ARGUMENT
    # dense: unknown dtype, C beyond the tile, unknown kind
    nb = C_.c_size_t()
    assert L().gtnb_viterbi_dense_async_workspace(ctx.h, B, T, 8, 7, capi.DENSE_ASG, C_.byref(nb)) == \
        capi.ERR_UNSUPPORTED
    assert L().gtnb_viterbi_dense_async_workspace(ctx.h, B, T, 240, capi.F32, capi.DENSE_ASG, C_.byref(nb)) == \
        capi.ERR_UNSUPPORTED
    assert L().gtnb_viterbi_dense_async_workspace(ctx.h, B, T, 8, capi.F32, 9, C_.byref(nb)) == \
        capi.ERR_INVALID_ARGUMENT


def test_handle_from_another_device(ctx):
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU visible")
    c1 = capi.Ctx(1)
    try:
        G = st.trigram_graph(8)
        h = Handle(c1, G, 8)
        c1._check(h.rc)
        n = C_.c_size_t()
        assert L().gtnb_viterbi_transitions_async_workspace(ctx.h, h.h, 1, 1, C_.byref(n)) == \
            capi.ERR_INVALID_ARGUMENT
        del h
    finally:
        c1.close()


def test_launch_profile_and_no_copy(ctx):
    rng = np.random.default_rng(2)
    C, B, T = 30, 8, 50
    for G, backoff, names in ((st.trigram_graph(C), False, {"sparse_viterbi_forward", "sparse_viterbi_trace"}),
                              (bo.backoff_ngram(rng, C, 3)[0], True, {"sparse_eps_viterbi", "sparse_eps_trace"})):
        h = Handle(ctx, G, C, backoff)
        ctx._check(h.rc)
        e = torch.as_tensor(rng.uniform(-3, 3, (B, T, C)).astype(np.float32)).cuda()
        w = torch.as_tensor(rng.uniform(-1, 0, len(G["src"])).astype(np.float32)).cuda()
        lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
        n = workspace(ctx, h, B, T)
        ws = torch.empty(n, dtype=torch.uint8, device="cuda")
        out = [torch.empty((B, T), dtype=torch.int32, device="cuda"), torch.empty((B, T), dtype=torch.int32,
                                                                                  device="cuda"),
               torch.empty(B, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda")]

        def call():
            return L().gtnb_viterbi_transitions_async(
                ctx.h, None, h.h, B, T, e.data_ptr(), lens.data_ptr(), w.data_ptr(), *[o.data_ptr() for o in out],
                ws.data_ptr(), n)
        assert call() == 0  # warm-up
        torch.cuda.synchronize()
        ctx.profile(True)
        ctx.profile_read()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            assert call() == 0
            torch.cuda.synchronize()
        got = set(ctx.profile_read())
        ctx.profile(False)
        assert got == names | {"decode_async_prepare", "decode_async_finalize"}, got
        copies = [ev.name for ev in prof.events() if "Memcpy" in ev.name or "Memset" in ev.name]
        assert not copies, copies


# ---- dense -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("kind", ["asg", "bigram"])
def test_dense_parity(C, dtype, kind):
    g = torch.Generator().manual_seed(C)
    B, T = 32, 120
    e = torch.log_softmax(torch.empty(B, T, C).normal_(0, 3, generator=g), -1).cuda().to(dtype)
    n = C * C + (C if kind == "asg" else 0)
    w = torch.empty(n).normal_(0, 1, generator=g).cuda()
    il = torch.randint(0, T + 1, (B,), generator=g).int()
    il[0] = T
    il[1] = 0
    sync, asyn = (tl.asg_viterbi, tl.asg_decode) if kind == "asg" else (tl.ngram_ctc_viterbi, tl.ngram_ctc_decode)
    pw, sw = sync(e, w, il)
    p, s, status = asyn(e, w, il.cuda())
    assert (status == 0).all()
    assert torch.equal(p, pw) and torch.equal(s, sw)
    bad = il.clone()
    bad[2], bad[3] = -1, T + 1
    p2, s2, st2 = asyn(e, w, bad.cuda())
    assert st2[2].item() == 2 and st2[3].item() == 2 and torch.isnan(s2[2:4]).all() and (p2[2:4] == -1).all()
    keep = [b for b in range(B) if b not in (2, 3)]
    assert torch.equal(p2[keep], p[keep]) and torch.equal(s2[keep], s[keep]) and (st2[keep] == 0).all()


def test_dense_c_abi_matches_torch(ctx):
    g = torch.Generator().manual_seed(0)
    B, T, C = 8, 50, 64
    e = torch.empty(B, T, C).normal_(0, 3, generator=g).cuda()
    w = torch.empty(C * C).normal_(0, 1, generator=g).cuda()
    n = C_.c_size_t()
    ctx._check(L().gtnb_viterbi_dense_async_workspace(ctx.h, B, T, C, capi.F32, capi.DENSE_BIGRAM, C_.byref(n)))
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    s = torch.empty(B, device="cuda")
    st_ = torch.empty(B, dtype=torch.int32, device="cuda")
    ctx._check(L().gtnb_viterbi_dense_async(ctx.h, None, B, T, C, e.data_ptr(), capi.F32, None, capi.DENSE_BIGRAM,
                                            w.data_ptr(), None, s.data_ptr(), st_.data_ptr(), ws.data_ptr(), n.value))
    torch.cuda.synchronize()
    _, sw, stw = tl.ngram_ctc_decode(e, w)
    assert torch.equal(s, sw) and torch.equal(st_, stw)


# ---- torch -------------------------------------------------------------------------------------------------------

def _gtn_graph(G):
    from gtn_b200 import gtn
    h = gtn.Graph()
    for f in G["flags"]:
        h.add_node(bool(f & 1), bool(f & 2))
    for a in range(len(G["src"])):
        h.add_arc(int(G["src"][a]), int(G["dst"][a]), int(G["olabel"][a]), int(G["olabel"][a]), 0.0)
    return h


def test_torch_transitions_decode(ctx):
    rng = np.random.default_rng(9)
    C, B, T = 30, 32, 80
    G = st.trigram_graph(C)
    tg = tl.TransitionGraph(_gtn_graph(G), C)
    e = torch.as_tensor(rng.uniform(-3, 3, (B, T, C)).astype(np.float32)).cuda()
    w = torch.as_tensor(rng.uniform(-1, 0, len(G["src"])).astype(np.float32)).cuda()
    il = torch.as_tensor(ragged(rng, B, T)).cuda()
    p, s, a, status = tl.transitions_decode(e, w, tg, il)
    h = Handle(ctx, G, C)
    ctx._check(h.rc)
    want = decode(ctx, h, e.cpu().numpy(), w.cpu().numpy(), il.cpu().numpy())
    for x, y in zip((p, s, a, status), want):
        assert np.array_equal(x.cpu().numpy(), y)
    # the synchronous torch decoder on every status-0 utterance
    pw, sw, aw = tl.sparse_viterbi(e, w, _gtn_graph(G), il)
    ok = status == 0
    assert torch.equal(p[ok], pw[ok]) and torch.equal(s[ok], sw[ok]) and torch.equal(a[ok], aw[ok])
    # no host wait, no synchronisation
    torch.cuda.synchronize()
    done = torch.cuda.Event()
    torch.cuda._sleep(100_000_000)
    tl.transitions_decode(e, w, tg, il)
    tl.asg_decode(e, torch.zeros(C + C * C, device="cuda"), il)
    done.record()
    assert not done.query(), "the call waited for the device"
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = tl.transitions_decode(e, w, tg, il)
        tl.collapse(out[0], 0)
        tl.ngram_ctc_decode(e, torch.zeros(C * C, device="cuda"), il)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_torch_captured_decode_replays_as_eager():
    rng = np.random.default_rng(4)
    C, B, T = 30, 16, 60
    G = st.trigram_graph(C)
    tg = tl.TransitionGraph(_gtn_graph(G), C)
    w = torch.as_tensor(rng.uniform(-1, 0, len(G["src"])).astype(np.float32)).cuda()
    wd = torch.empty(C + C * C).normal_().cuda()
    se = torch.as_tensor(rng.uniform(-3, 3, (B, T, C)).astype(np.float32)).cuda()
    sil = torch.as_tensor(ragged(rng, B, T)).cuda()
    tl.transitions_decode(se, w, tg, sil)  # warm-up: the shared-memory opt-in
    tl.asg_decode(se, wd, sil)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            p, sc, a, status = tl.transitions_decode(se, w, tg, sil)
            lab, n = tl.collapse(p, 0)
            pd, sd, std = tl.asg_decode(se, wd, sil)
            with pytest.raises(RuntimeError, match="before capturing"):
                tl.TransitionGraph(_gtn_graph(G), C)
    torch.cuda.current_stream().wait_stream(s)
    for seed in (1, 2):
        r = np.random.default_rng(seed)
        se.copy_(torch.as_tensor(r.uniform(-3, 3, (B, T, C)).astype(np.float32)))
        sil.copy_(torch.as_tensor(ragged(r, B, T)))
        g.replay()
        want = tl.transitions_decode(se, w, tg, sil)
        wl, wn = tl.collapse(want[0], 0)
        wd_out = tl.asg_decode(se, wd, sil)
        torch.cuda.synchronize()
        assert all(torch.equal(x, y) for x, y in zip((p, sc, a, status, lab, n), want + (wl, wn))), seed
        assert all(torch.equal(x, y) for x, y in zip((pd, sd, std), wd_out)), seed
    del g
