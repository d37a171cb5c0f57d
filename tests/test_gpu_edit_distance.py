"""gtnb_edit_distance_async and torch edit_distance on the GPU, against the restatement (tests/edit_oracle.py):

- the C ABI == the restatement at the benchmark shapes (scripts/bench_edit_distance.py) and at N = M = 4096, in token
  and word mode, with and without alignment (the scalars equal either way);
- a direct reference sample (-viterbiScore(compose(x, compose(edits, y))) through oracle/_ref);
- error codes: bounds above 4096, a too-small or misaligned workspace;
- the launch profile: the one kernel, no copy and no memset;
- torch: the call returns while the device is busy, runs clean under sync-debug "error", a captured
  ngram_ctc_decode -> collapse -> edit_distance step replays == eager, and collapse's output is taken unchanged.
"""
import ctypes as C_
import os
import sys

import numpy as np
import pytest
import torch

from gtn_b200 import capi
from gtn_b200 import torch_loss as tl
from tests import edit_oracle as eo

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import bench_edit_distance as bed  # noqa: E402  (the benchmark's seeded workloads)

L = capi.lib
KEYS = ("distance", "ops", "units", "status", "hyp_align", "ref_align")


@pytest.fixture(scope="module")
def ctx():
    c = capi.Ctx(0)
    yield c
    c.close()


def workspace(ctx, B, N, M, sep, align):
    n = C_.c_size_t()
    ctx._check(L().gtnb_edit_distance_async_workspace(ctx.h, B, N, M, sep, int(align), C_.byref(n)))
    return n.value


def call(ctx, hyp, hl, ref, rl, sep=-1, align=True, ws_bytes=None, ws_offset=0):
    """the C ABI on device copies of numpy inputs -> (rc, dict of numpy outputs)"""
    B, N = hyp.shape
    M = ref.shape[1]
    d = [torch.as_tensor(np.ascontiguousarray(a, np.int32)).cuda() for a in (hyp, hl, ref, rl)]
    out = dict(distance=torch.full((B,), 77, dtype=torch.int32, device="cuda"),
               ops=torch.full((B, 3), 77, dtype=torch.int32, device="cuda"),
               units=torch.full((B, 2), 77, dtype=torch.int32, device="cuda"),
               status=torch.full((B,), 77, dtype=torch.int32, device="cuda"),
               hyp_align=torch.full((B, N), 77, dtype=torch.int32, device="cuda") if align else None,
               ref_align=torch.full((B, M), 77, dtype=torch.int32, device="cuda") if align else None)
    need = workspace(ctx, B, N, M, sep, align)
    n = need if ws_bytes is None else ws_bytes
    ws = torch.empty(max(need, 1) + 512, dtype=torch.uint8, device="cuda")
    wp = ws.data_ptr() + ws_offset if n else None
    rc = L().gtnb_edit_distance_async(
        ctx.h, None, B, d[0].data_ptr(), N, d[1].data_ptr(), d[2].data_ptr(), M, d[3].data_ptr(), sep,
        *[None if out[k] is None else out[k].data_ptr() for k in KEYS], wp, n)
    torch.cuda.synchronize()
    return rc, {k: None if v is None else v.cpu().numpy() for k, v in out.items()}


def check(ctx, hyp, hl, ref, rl, sep=-1, want=None):
    want = want or eo.batch(hyp, hl, ref, rl, sep)
    scalars = None
    for align in (True, False):
        rc, got = call(ctx, hyp, hl, ref, rl, sep, align)
        ctx._check(rc)
        for k in KEYS:
            if got[k] is not None:
                assert np.array_equal(got[k], want[k]), (k, align, np.argwhere(got[k] != want[k])[:5])
        s = [got[k] for k in KEYS[:4]]
        if scalars is not None:
            assert all(np.array_equal(a, b) for a, b in zip(s, scalars))
        scalars = s
    return want


@pytest.mark.parametrize("name", ["token", "word"])
def test_benchmark_shapes(ctx, name):
    h, hl, r, rl, sep = bed.WORKLOADS[name]()
    check(ctx, h, hl, r, rl, -1 if sep is None else sep)


def test_long_pairs(ctx):
    h, hl, r, rl, _ = bed.long_workload(B=6)
    check(ctx, h, hl, r, rl)


@pytest.mark.parametrize("sep", [-1, 0])
def test_bounds_4096(ctx, sep):
    rng = np.random.default_rng(4096 + sep)
    N = M = 4096
    r = rng.integers(0, 6 if sep >= 0 else 128, (4, M)).astype(np.int32)
    h = r.copy()
    h[:, ::37] = rng.integers(0, 6, h[:, ::37].shape)
    if sep >= 0:  # alternating tokens and separators: the most words the bounds allow
        h[0, 1::2] = 0
        r[0, 1::2] = 0
        h[0, 0::2] = np.maximum(h[0, 0::2], 1)
        r[0, 0::2] = np.maximum(r[0, 0::2], 1)
    hl = np.array([N, N, 4000, 1], np.int32)
    rl = np.array([M, 3000, M, M], np.int32)
    check(ctx, h, hl, r, rl, sep)


def test_ragged_invalid_and_empty(ctx):
    rng = np.random.default_rng(5)
    h, hl, r, rl, _ = bed.token_workload(B=16)
    hl[1], rl[2] = -1, r.shape[1] + 1
    hl[3], rl[4] = np.iinfo(np.int32).min, np.iinfo(np.int32).max
    hl[5], rl[6] = 0, 0
    hl[7] = rl[7] = 0
    h[8, :hl[8]] = rng.integers(0, 2, hl[8])
    want = check(ctx, h, hl, r, rl)
    assert list(want["status"][:5]) == [0, 2, 2, 2, 2]


def test_reference_sample(ctx):
    from oracle import pyoracle as po
    if not po.have_ref():
        pytest.skip("oracle/_ref is not built")
    from tests.test_edit_oracle import ref_distance
    h, hl, r, rl, sep = bed.word_workload(B=3, words=12)
    rc, got = call(ctx, h, hl, r, rl, sep, False)
    ctx._check(rc)
    for b in range(3):
        hu, ru = eo.units(h[b, :hl[b]], r[b, :rl[b]], sep)
        assert got["distance"][b] == ref_distance(hu, ru, max(hu + ru) + 1)
    h, hl, r, rl, _ = bed.token_workload(B=2)
    hl[:], rl[:] = 40, 30
    rc, got = call(ctx, h, hl, r, rl, -1, False)
    ctx._check(rc)
    for b in range(2):
        assert got["distance"][b] == ref_distance(list(h[b, :40]), list(r[b, :30]), bed.C_TOK)


def test_errors(ctx):
    n = C_.c_size_t()
    assert L().gtnb_edit_distance_async_workspace(ctx.h, 2, 4097, 10, -1, 0, C_.byref(n)) == capi.ERR_UNSUPPORTED
    assert L().gtnb_edit_distance_async_workspace(ctx.h, 2, 10, 4097, 0, 1, C_.byref(n)) == capi.ERR_UNSUPPORTED
    assert L().gtnb_edit_distance_async_workspace(ctx.h, -1, 10, 10, 0, 1, C_.byref(n)) == capi.ERR_INVALID_ARGUMENT
    buf = torch.zeros(64, dtype=torch.int32, device="cuda")
    t = buf.data_ptr()
    assert L().gtnb_edit_distance_async(ctx.h, None, 2, t, 4097, t, t, 10, t, -1, t, t, t, t, None, None, None,
                                        0) == capi.ERR_UNSUPPORTED
    rng = np.random.default_rng(6)
    h, r = rng.integers(0, 5, (3, 50)), rng.integers(0, 5, (3, 60))
    hl, rl = np.full(3, 50), np.full(3, 60)
    need = workspace(ctx, 3, 50, 60, -1, True)
    assert need > 0 and workspace(ctx, 3, 50, 60, -1, False) == 0
    assert call(ctx, h, hl, r, rl, ws_bytes=need - 256)[0] == capi.ERR_INVALID_ARGUMENT  # too small
    assert call(ctx, h, hl, r, rl, ws_bytes=0)[0] == capi.ERR_INVALID_ARGUMENT
    assert call(ctx, h, hl, r, rl, ws_offset=16)[0] == capi.ERR_INVALID_ARGUMENT  # misaligned
    assert call(ctx, h, hl, r, rl, align=False)[0] == 0  # no alignment: no workspace
    with pytest.raises(RuntimeError, match="4096"):
        t = torch.zeros((1, 5000), dtype=torch.int32, device="cuda")
        tl.edit_distance(t, torch.ones(1, dtype=torch.int64, device="cuda"), t[:, :10],
                         torch.ones(1, dtype=torch.int64, device="cuda"))


def test_launch_profile_and_no_copy(ctx):
    h, hl, r, rl, sep = bed.word_workload(B=8)
    d = [torch.as_tensor(a).cuda() for a in (h, hl, r, rl)]
    B, N = h.shape
    M = r.shape[1]
    need = workspace(ctx, B, N, M, sep, True)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = [torch.empty(s, dtype=torch.int32, device="cuda") for s in ((B,), (B, 3), (B, 2), (B,), (B, N), (B, M))]

    def go():
        return L().gtnb_edit_distance_async(ctx.h, None, B, d[0].data_ptr(), N, d[1].data_ptr(), d[2].data_ptr(), M,
                                            d[3].data_ptr(), sep, *[o.data_ptr() for o in out], ws.data_ptr(), need)
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
    assert set(got) == {"edit_distance"} and ctx.launches - before == 1, got
    copies = [ev.name for ev in prof.events() if "Memcpy" in ev.name or "Memset" in ev.name]
    assert not copies, copies


def test_torch_no_wait_sync_debug_and_collapse():
    h, hl, r, rl, _ = bed.token_workload(B=64)
    hd, rd = torch.as_tensor(h).cuda(), torch.as_tensor(r).cuda()
    hld, rld = torch.as_tensor(hl).cuda().long(), torch.as_tensor(rl).cuda().long()
    res = tl.edit_distance(hd, hld, rd, rld, alignment=True)
    want = eo.batch(h, hl, r, rl)
    assert np.array_equal(res.distance.cpu().numpy(), want["distance"])
    assert np.array_equal(torch.stack([res.substitutions, res.insertions, res.deletions], 1).cpu().numpy(),
                          want["ops"])
    assert np.array_equal(res.hyp_align.cpu().numpy(), want["hyp_align"])
    assert res.ref_units.dtype == torch.int32 and res.status.is_cuda
    # no host wait
    torch.cuda.synchronize()
    done = torch.cuda.Event()
    torch.cuda._sleep(100_000_000)
    tl.edit_distance(hd, hld, rd, rld, alignment=True)
    tl.edit_distance(hd, hld, rd, rld, word_sep=0)
    done.record()
    assert not done.query(), "the call waited for the device"
    torch.cuda.synchronize()
    # collapse's output (int32 labels, int64 lengths) taken unchanged
    paths = torch.as_tensor(np.repeat(h[:, :200], 2, axis=1)).cuda()
    paths[:, ::7] = 0
    torch.cuda.set_sync_debug_mode("error")
    try:
        lab, n = tl.collapse(paths, 0)
        got = tl.edit_distance(lab, n, rd, rld)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert lab.dtype == torch.int32 and n.dtype == torch.int64
    lab_h, n_h = lab.cpu().numpy(), n.cpu().numpy()
    w2 = eo.batch(lab_h, n_h, r, rl)
    assert np.array_equal(got.distance.cpu().numpy(), w2["distance"])
    ok = got.status == 0
    rate = got.distance[ok].sum() / got.ref_units[ok].sum()
    assert abs(float(rate) - w2["distance"].sum() / rl.sum()) < 1e-6


def test_torch_captured_step_replays_as_eager():
    rng = np.random.default_rng(8)
    B, T, Cn = 32, 300, 40
    e = torch.as_tensor(rng.standard_normal((B, T, Cn), dtype=np.float32)).cuda()
    w = torch.as_tensor(rng.uniform(-2, 0, Cn * Cn).astype(np.float32)).cuda()
    il = torch.as_tensor(rng.integers(T // 2, T + 1, B).astype(np.int32)).cuda()
    r = torch.as_tensor(rng.integers(1, Cn, (B, 120)).astype(np.int32)).cuda()
    rl = torch.as_tensor(rng.integers(0, 121, B).astype(np.int32)).cuda()

    def step():
        p, _, _ = tl.ngram_ctc_decode(e, w, il)
        lab, n = tl.collapse(p, 0)
        return tl.edit_distance(lab, n, r, rl, alignment=True), tl.edit_distance(lab, n, r, rl, word_sep=3)
    step()  # warm-up: the contexts exist before capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            cap = step()
    torch.cuda.current_stream().wait_stream(s)
    for seed in (1, 2):
        rr = np.random.default_rng(seed)
        e.copy_(torch.as_tensor(rr.standard_normal((B, T, Cn), dtype=np.float32)))
        rl.copy_(torch.as_tensor(rr.integers(0, 121, B).astype(np.int32)))
        g.replay()
        eager = step()
        torch.cuda.synchronize()
        for c, w_ in zip(cap, eager):
            for x, y in zip(c, w_):
                assert (x is None and y is None) or torch.equal(x, y), seed
    del g
