"""gtnb_ctc_align_async, gtnb_ngram_ctc_align_async, gtnb_asg_align_async and torch ctc_align / ngram_ctc_align /
asg_align / align_spans, on the GPU.

The contract: for every utterance with status 0, paths, tokens and the score are == to the synchronous aligners
(gtnb_graph_viterbi on CTC graphs; gtnb_graph_transitions_viterbi on CTC graphs with BIGRAM and on force-align chains
with ASG), which are themselves held to the reference; tokens are derived from the synchronous call's arcs.  A status 3
utterance has the synchronous score and an optimal, valid path.  For CTC with exact_ties at 0 the two calls trace
in-arc tables of the same order, so every output is == on every utterance.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gtn_b200 import capi
from gtn_b200 import torch_loss as tl
from oracle import pyoracle as po
from tests import align_async_oracle as ao

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = {torch.float32: capi.F32, torch.bfloat16: capi.BF16, torch.float16: capi.F16}
CTC, NGRAM, ASG = ao.CTC, ao.NGRAM, ao.ASG
NAMES = {CTC: "ctc", NGRAM: "ngram_ctc", ASG: "asg"}


@pytest.fixture(scope="module")
def ctx():
    c = capi.Ctx(0)
    yield c
    c.close()


def transitions(kind, C_, seed=0):
    if kind == CTC:
        return None
    g = torch.Generator().manual_seed(seed + 100)
    n = C_ * C_ + (C_ if kind == ASG else 0)
    return torch.empty(n).normal_(0, 1, generator=g).cuda()


def batch(B, T, C_, S, seed=0, ragged=False, blank=0, repeats=False):
    """log-softmax emissions; targets without the blank label; ragged: U_b and T_b below the bounds"""
    g = torch.Generator().manual_seed(seed)
    e = torch.log_softmax(torch.empty(B, T, C_).normal_(0, 3, generator=g), -1)
    labels = torch.tensor([c for c in range(C_) if c != blank], dtype=torch.int32)
    tg = labels[torch.randint(0, len(labels), (B, S), generator=g)]
    if repeats:
        tg[:, 1::3] = tg[:, 0::3][:, :tg[:, 1::3].shape[1]]
    lens = torch.full((B,), S, dtype=torch.int32)
    il = None
    if ragged:
        lens = torch.randint(0, S + 1, (B,), generator=g).int()
        il = torch.randint(T // 2, T + 1, (B,), generator=g).int()
    return e, tg, lens, il


def workspace(ctx, kind, B, T, C_, S, dt):
    n = C.c_size_t()
    fn = getattr(capi.lib(), "gtnb_%s_align_async_workspace" % NAMES[kind])
    return fn(ctx.h, B, T, C_, S, dt, C.byref(n)), n.value


def launch(ctx, kind, e, W, tg, lens, il, blank, outs, ws, nb):
    B, T, C_ = e.shape
    S = tg.shape[1]
    ptr = lambda x: None if x is None else x.data_ptr()  # noqa: E731
    head = (ctx.h, torch.cuda.current_stream().cuda_stream, B, T, C_, S, e.data_ptr(), DT[e.dtype], ptr(il))
    tail = tuple(ptr(x) for x in outs) + (ws, nb)
    fn = getattr(capi.lib(), "gtnb_%s_align_async" % NAMES[kind])
    if kind == CTC:
        return fn(*head, tg.data_ptr(), lens.data_ptr(), blank, *tail)
    if kind == NGRAM:
        return fn(*head, W.data_ptr(), tg.data_ptr(), lens.data_ptr(), blank, *tail)
    return fn(*head, W.data_ptr(), tg.data_ptr(), lens.data_ptr(), *tail)


def async_call(ctx, kind, e, W, tg, lens, il, blank=0, ws_bytes=None):
    """-> (rc, paths, tokens, scores, status) as numpy after a synchronise"""
    e = e.cuda().contiguous()
    B, T, C_ = e.shape
    rc, need = workspace(ctx, kind, B, T, C_, tg.shape[1], DT[e.dtype])
    if rc:
        return rc, None, None, None, None
    nb = need if ws_bytes is None else ws_bytes
    ws = torch.empty(max(nb, 1), dtype=torch.uint8, device="cuda")
    outs = (torch.full((B, T), -7, dtype=torch.int32, device="cuda"),
            torch.full((B, T), -7, dtype=torch.int32, device="cuda"),
            torch.full((B,), 7.0, device="cuda"), torch.full((B,), -7, dtype=torch.int32, device="cuda"))
    rc = launch(ctx, kind, e, W, tg.cuda().contiguous(), lens.cuda().contiguous(),
                None if il is None else il.cuda().contiguous(), blank, outs, ws.data_ptr(), nb)
    torch.cuda.synchronize()
    return (rc,) + tuple(x.cpu().numpy() for x in outs)


def graphs_of(kind, tg, lens, blank=0):
    return [ao.numerator_graph(kind, tg[b, :int(lens[b])].numpy(), blank) for b in range(tg.shape[0])]


def sync_call(ctx, kind, e, W, tg, lens, il, blank=0):
    """the synchronous aligner on the host-built numerators -> (paths, tokens, scores)"""
    graphs = graphs_of(kind, tg, lens, blank)
    views = [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
    en = e.float().numpy()
    iln = None if il is None else il.numpy()
    if kind == CTC:
        paths, scores, arcs = ctx.graph_viterbi_dev(en, views, iln)
    else:
        paths, scores, arcs = ctx.graph_transitions_viterbi_dev(
            en, views, W.cpu().numpy(), capi.DENSE_ASG if kind == ASG else capi.DENSE_BIGRAM, iln)
    tokens = np.full(paths.shape, -1, np.int32)
    for b, g in enumerate(graphs):
        ok = arcs[b] >= 0
        tokens[b, ok] = ao.positions(kind, g)[arcs[b, ok]]
    return paths, tokens, scores


def same_score(a, b):
    return a == b or (np.isneginf(a) and np.isneginf(b))


def check_parity(kind, e, W, tg, lens, il, out, want, blank=0):
    """status 0: == the synchronous call; status 3: its score, and an optimal valid path.  -> number of status 3"""
    rc, paths, tokens, scores, status = out
    assert rc == 0
    rp, rt, rs = want
    T = e.shape[1]
    en = e.float().numpy()
    Wn = None if W is None else W.cpu().numpy()
    assert set(np.unique(status).tolist()) <= {0, 3}, np.unique(status)
    for b in range(e.shape[0]):
        assert same_score(scores[b], rs[b]), (b, scores[b], rs[b])
        if status[b] == 0:
            assert np.array_equal(paths[b], rp[b]) and np.array_equal(tokens[b], rt[b]), b
        else:
            Tb = T if il is None else int(il[b])
            y = tg[b, :int(lens[b])].numpy()
            assert ao.valid_path(kind, paths[b, :Tb], tokens[b, :Tb], y, blank), b
            assert ao.path_value(kind, en[b, :Tb], Wn, paths[b, :Tb]) == scores[b], b
    return int((status == 3).sum())


# ---- parity with the synchronous aligners ------------------------------------------------------------------------

@pytest.mark.parametrize("B,T,C_,S", [(256, 1000, 64, 100), (256, 1000, 128, 100), (128, 500, 64, 50)])
def test_ctc_parity(ctx, B, T, C_, S):
    e, tg, lens, il = batch(B, T, C_, S, seed=C_ + S)
    out = async_call(ctx, CTC, e, None, tg, lens, il)
    n3 = check_parity(CTC, e, None, tg, lens, il, out, sync_call(ctx, CTC, e, None, tg, lens, il))
    print("ctc B=%d T=%d C=%d U=%d: %d of %d utterances with status 3" % (B, T, C_, S, n3, B))
    # exact_ties off: the synchronous call keeps its device choice too, and both trace in-arcs in the same order
    ctx.set_flag("exact_ties", 0)
    try:
        rp, rt, rs = sync_call(ctx, CTC, e, None, tg, lens, il)
    finally:
        ctx.set_flag("exact_ties", 1)
    assert np.array_equal(out[1], rp) and np.array_equal(out[2], rt) and np.array_equal(out[3], rs)


def test_ctc_parity_ragged(ctx):
    e, tg, lens, il = batch(128, 500, 64, 50, seed=3, ragged=True, blank=5)
    out = async_call(ctx, CTC, e, None, tg, lens, il, blank=5)
    check_parity(CTC, e, None, tg, lens, il, out, sync_call(ctx, CTC, e, None, tg, lens, il, blank=5), blank=5)


@pytest.mark.parametrize("kind", [NGRAM, ASG])
@pytest.mark.parametrize("ragged", [False, True])
def test_transitions_parity(ctx, kind, ragged):
    B, T, C_, S = 128, 500, 64, 50
    e, tg, lens, il = batch(B, T, C_, S, seed=7 + kind, ragged=ragged)
    W = transitions(kind, C_)
    out = async_call(ctx, kind, e, W, tg, lens, il)
    n3 = check_parity(kind, e, W, tg, lens, il, out, sync_call(ctx, kind, e, W, tg, lens, il))
    print("%s ragged=%s: %d of %d utterances with status 3" % (NAMES[kind], ragged, n3, B))


def test_asg_ties_on_repeated_labels(ctx):
    """ASG on targets with repeated labels: the self loop and the step between equal labels weigh the same, so many
    traced paths meet a tie; every one of them is an optimal, valid path"""
    B, T, C_, S = 128, 500, 64, 50
    e, tg, lens, il = batch(B, T, C_, S, seed=21, repeats=True)
    W = transitions(ASG, C_)
    out = async_call(ctx, ASG, e, W, tg, lens, il)
    n3 = check_parity(ASG, e, W, tg, lens, il, out, sync_call(ctx, ASG, e, W, tg, lens, il))
    print("asg with repeated labels: %d of %d utterances with status 3" % (n3, B))
    assert n3 > 0


# ---- the live reference, including C = 256 for n-gram and ASG ----------------------------------------------------

@pytest.mark.parametrize("kind", [CTC, NGRAM, ASG])
@pytest.mark.parametrize("C_", [29, 256])
def test_reference_sample(ctx, kind, C_):
    if not po.have_ref():
        pytest.skip("oracle/_ref/libgtn_ref.so is missing")
    B, T, S = 6, 40, 8
    e, tg, lens, il = batch(B, T, C_, S, seed=C_ + kind, ragged=True)
    W = transitions(kind, C_)
    out = async_call(ctx, kind, e, W, tg, lens, il)
    Wn = None if W is None else W.cpu().numpy()
    want = ao.reference(kind, e.numpy(), Wn, tg.numpy(), lens.numpy(), il.numpy(), 0)
    check_parity(kind, e, W, tg, lens, il, out, want)


# ---- 16-bit emissions and the range of C -------------------------------------------------------------------------

@pytest.mark.parametrize("kind", [CTC, NGRAM, ASG])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_half_precision_is_the_widened_float32_call(ctx, kind, dtype):
    e, tg, lens, il = batch(32, 200, 64, 20, seed=9, ragged=True)
    W = transitions(kind, 64)
    h = e.to(dtype)
    got = async_call(ctx, kind, h, W, tg, lens, il)
    want = async_call(ctx, kind, h.float(), W, tg, lens, il)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("C_", [60, 256, 1024])
def test_ctc_label_range(ctx, C_):
    e, tg, lens, il = batch(16, 150, C_, 20, seed=C_, ragged=True)
    out = async_call(ctx, CTC, e, None, tg, lens, il)
    ctx.set_flag("exact_ties", 0)
    try:
        rp, rt, rs = sync_call(ctx, CTC, e, None, tg, lens, il)
    finally:
        ctx.set_flag("exact_ties", 1)
    assert out[0] == 0 and (out[4] == 0).all()
    assert np.array_equal(out[1], rp) and np.array_equal(out[2], rt) and np.array_equal(out[3], rs)


# ---- edge and bad inputs, each flagged alone ---------------------------------------------------------------------

@pytest.mark.parametrize("kind", [CTC, NGRAM, ASG])
def test_edge_and_bad_inputs_are_flagged_alone(ctx, kind):
    B, T, C_, S = 12, 60, 32, 10
    e, tg, lens, il = batch(B, T, C_, S, seed=40 + kind)
    il = torch.full((B,), T, dtype=torch.int32)
    W = transitions(kind, C_)
    lens[1], il[2], il[3] = 0, 0, 1  # U = 0, T_b = 0, T_b = 1
    lens[4] = -1
    lens[5] = S + 1
    il[6] = T + 1
    tg[7, 3] = C_
    e[8, 5, :] = float("nan")
    e[9, 7, int(tg[9, 0])] = float("inf")
    want_status = {4: 2, 5: 2, 6: 2, 7: 2, 8: 1, 9: 1}
    rc, paths, tokens, scores, status = async_call(ctx, kind, e, W, tg, lens, il)
    assert rc == 0
    for b, st in want_status.items():
        assert status[b] == st and np.isnan(scores[b]) and (paths[b] == -1).all() and (tokens[b] == -1).all(), b
    assert np.isneginf(scores[2]) and (paths[2] == -1).all()
    keep = [b for b in range(B) if b not in want_status]
    alone = async_call(ctx, kind, e[keep], W, tg[keep], lens[keep], il[keep])
    for k, b in enumerate(keep):
        assert status[b] == alone[4][k] and same_score(scores[b], alone[3][k]), b
        assert np.array_equal(paths[b], alone[1][k]) and np.array_equal(tokens[b], alone[2][k]), b
    if kind != CTC:  # a NaN transition weight flags the utterances whose numerator uses it
        W2 = W.clone()
        W2[:] = float("nan")
        out = async_call(ctx, kind, e[keep], W2, tg[keep], lens[keep], il[keep])
        used = np.array([il[b] > 0 and (kind == NGRAM or lens[b] > 0) for b in keep])
        assert (out[4][used] == 1).all() and np.isnan(out[3][used]).all(), out[4]


# ---- errors and the launch profile -------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", [CTC, NGRAM, ASG])
def test_unsupported_and_bad_workspace(ctx, kind):
    B, T, C_, S = 4, 30, 16, 5
    e, tg, lens, il = batch(B, T, C_, S, seed=1)
    W = transitions(kind, C_)
    assert workspace(ctx, kind, B, T, C_, S, 7)[0] == capi.ERR_UNSUPPORTED  # unknown dtype
    assert workspace(ctx, kind, B, T, C_, 20000, capi.F32)[0] == capi.ERR_UNSUPPORTED  # beyond the sweeps
    ctx.set_flag("implicit", 0)
    try:
        assert workspace(ctx, kind, B, T, C_, S, capi.F32)[0] == capi.ERR_UNSUPPORTED
    finally:
        ctx.set_flag("implicit", 1)
    if kind != ASG:
        assert async_call(ctx, kind, e, W, tg, lens, il, blank=C_)[0] == capi.ERR_UNSUPPORTED
    rc, need = workspace(ctx, kind, B, T, C_, S, capi.F32)
    assert rc == 0 and need > 0
    assert async_call(ctx, kind, e, W, tg, lens, il, ws_bytes=need - 256)[0] == capi.ERR_INVALID_ARGUMENT
    assert async_call(ctx, kind, e, W, tg, lens, il)[0] == 0


@pytest.mark.parametrize("kind", [CTC, NGRAM, ASG])
def test_launch_profile_and_no_copy(ctx, kind):
    B, T, C_, S = 8, 100, 64, 12
    e, tg, lens, il = batch(B, T, C_, S, seed=12, ragged=True)
    W = transitions(kind, C_)
    async_call(ctx, kind, e, W, tg, lens, il)  # warm-up
    ec, tgd, lensd, ild = e.cuda(), tg.cuda(), lens.cuda(), il.cuda()
    rc, need = workspace(ctx, kind, B, T, C_, S, capi.F32)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    outs = (torch.empty((B, T), dtype=torch.int32, device="cuda"), torch.empty((B, T), dtype=torch.int32, device="cuda"),
            torch.empty(B, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    ctx.profile(True)
    ctx.profile_read()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        assert launch(ctx, kind, ec, W, tgd, lensd, ild, 0, outs, ws.data_ptr(), need) == 0
        torch.cuda.synchronize()
    names = set(ctx.profile_read())
    ctx.profile(False)
    build = {CTC: {"ctc_async_prepare", "ctc_build"}, NGRAM: {"trellis_async_prepare", "ngram_tau", "ngram_num_build"},
             ASG: {"trellis_async_prepare", "asg_num_build"}}[kind]
    assert names == build | {"implicit_forward_max", "implicit_trace", "align_async_finalize"}, names
    copies = [ev.name for ev in prof.events() if "Memcpy" in ev.name or "Memset" in ev.name]
    assert not copies, copies


# ---- torch -------------------------------------------------------------------------------------------------------

def align_fn(kind, e, W, tg, lens, il=None):
    if kind == CTC:
        return tl.ctc_align(e, tg, lens, il)
    if kind == NGRAM:
        return tl.ngram_ctc_align(e, W, tg, lens, il)
    return tl.asg_align(e, W, tg, lens, il)


@pytest.mark.parametrize("kind", [CTC, NGRAM, ASG])
def test_torch_matches_c_abi_and_does_not_wait(ctx, kind):
    e, tg, lens, il = batch(32, 300, 64, 30, seed=5, ragged=True)
    W = transitions(kind, 64)
    ec, tgd, lensd, ild = e.cuda(), tg.cuda(), lens.cuda(), il.cuda()
    got = align_fn(kind, ec, W, tgd, lensd, ild)
    want = async_call(ctx, kind, e, W, tg, lens, il)
    for a, b in zip(got, want[1:]):
        assert np.array_equal(a.cpu().numpy(), b)
    torch.cuda.synchronize()
    done = torch.cuda.Event()
    torch.cuda._sleep(100_000_000)  # tens of milliseconds of GPU time
    align_fn(kind, ec, W, tgd, lensd, ild)
    done.record()
    assert not done.query(), "the call waited for the device"
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = align_fn(kind, ec, W, tgd, lensd, ild)
        tl.align_spans(out[1], tg.shape[1])
    finally:
        torch.cuda.set_sync_debug_mode("default")


@pytest.mark.parametrize("kind", [CTC, NGRAM, ASG])
def test_torch_autocast_bf16(kind):
    e, tg, lens, il = batch(16, 120, 64, 15, seed=6, ragged=True)
    W = transitions(kind, 64)
    proj = torch.nn.Linear(64, 64).cuda()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits = proj(e.cuda())
        assert logits.dtype == torch.bfloat16
        got = align_fn(kind, logits, W, tg.cuda(), lens.cuda(), il.cuda())
    want = align_fn(kind, logits.float(), W, tg.cuda(), lens.cuda(), il.cuda())
    for a, b in zip(got, want):
        assert torch.equal(a, b)


_CAPTURE = r"""
import sys, torch
sys.path.insert(0, %(root)r)
from gtn_b200 import torch_loss as tl
from tests.test_gpu_align_async import batch, transitions, align_fn
kind = %(kind)d
B, T, C_, S = 32, 200, 128, 100  # the trace's staged rows need more than 48 KB of shared memory at C = 128
W = transitions(kind, C_)
e0, tg0, l0, il0 = batch(4, 20, 8, 3, seed=0)
align_fn(kind, e0.cuda(), transitions(kind, 8), tg0.cuda(), l0.cuda())  # warm-up: a small shape, the context only
torch.cuda.synchronize()
e, tg, lens, il = batch(B, T, C_, S, seed=1, ragged=True)
se, stg, sl, sil = e.cuda(), tg.cuda(), lens.cuda(), il.cuda()
g = torch.cuda.CUDAGraph()
s = torch.cuda.Stream()
s.wait_stream(torch.cuda.current_stream())
with torch.cuda.stream(s):
    with torch.cuda.graph(g):  # the first call at this shape is captured
        out = align_fn(kind, se, W, stg, sl, sil)
torch.cuda.current_stream().wait_stream(s)
for seed in (2, 3):
    e, tg, lens, il = batch(B, T, C_, S, seed=seed, ragged=True)
    se.copy_(e); stg.copy_(tg); sl.copy_(lens); sil.copy_(il)
    g.replay()
    want = align_fn(kind, e.cuda(), W, tg.cuda(), lens.cuda(), il.cuda())
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(out, want)), seed
print("capture ok")
"""


@pytest.mark.parametrize("kind", [CTC, NGRAM, ASG])
def test_torch_captured_alignment_replays_as_eager(kind):
    """in a fresh process, so that the trace kernel's shared-memory opt-in happens for the first time under capture"""
    r = subprocess.run([sys.executable, "-c", _CAPTURE % {"root": ROOT, "kind": kind}], capture_output=True, text=True,
                       cwd=ROOT, timeout=600)
    assert r.returncode == 0 and "capture ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_torch_unsupported_bounds_raise():
    e, tg, lens, _ = batch(2, 10, 8, 3, seed=0)
    tg = torch.zeros((2, 20000), dtype=torch.int32)
    with pytest.raises(RuntimeError, match="graph_viterbi"):
        tl.ctc_align(e.cuda(), tg.cuda(), lens.cuda())
    with pytest.raises(RuntimeError, match="graph_transitions_viterbi"):
        tl.asg_align(e.cuda(), transitions(ASG, 8), tg.cuda(), lens.cuda())


def test_align_spans_matches_a_loop():
    rng = np.random.default_rng(0)
    B, T, S = 9, 50, 7
    tokens = np.full((B, T), -1, np.int32)
    for b in range(B):
        t = 0
        for u in range(int(rng.integers(0, S + 1))):
            t += int(rng.integers(0, 3))  # blank frames
            n = int(rng.integers(1, 4))
            tokens[b, t:t + n] = u
            t += n
    start, end = tl.align_spans(torch.from_numpy(tokens).cuda(), S)
    want_s, want_e = np.full((B, S), -1), np.full((B, S), -1)
    for b in range(B):
        for t in range(T):
            u = tokens[b, t]
            if u >= 0:
                want_s[b, u] = t if want_s[b, u] < 0 else want_s[b, u]
                want_e[b, u] = t + 1
    assert start.dtype == torch.int32 and end.dtype == torch.int32
    assert np.array_equal(start.cpu().numpy(), want_s) and np.array_equal(end.cpu().numpy(), want_e)
