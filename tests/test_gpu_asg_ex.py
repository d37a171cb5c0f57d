"""gtnb_asg_loss_ex (ASG on a padded minibatch with device-resident transitions) on the GPU, against the live
reference (oracle/_ref, every utterance alone on its first T_b rows), the C oracle and the float64 referee
(tests/asg_oracle.py).  The bar (DESIGN.md "Tolerances"): losses within 1e-4 relative of the reference; emission
and transition gradients at least as close to float64 as the reference's own fp32 gradients are, x2; non-finite
results equal in kind (inf / NaN) to the reference's.  With GTNB_PARITY_DIR set, the observed errors are written to
$GTNB_PARITY_DIR/asg_ex_parity_observed.json."""
import json
import os
import sys

import numpy as np
import pytest

from tests import asg_oracle as ao
from tests import util

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


def inputs(B, T, C, U, seed=1234, w_scale=2.0):
    """emissions U(-5, 5) and targets in [1, C-1] per utterance (seed + b), trans_w U(-w_scale, w_scale) from 4321"""
    e, tg = util.bench_inputs(B, T, C, U, seed)
    tw = np.random.default_rng(4321).uniform(-w_scale, w_scale, C + C * C).astype(np.float32)
    return e, tg, tw


def _err(a, b):
    a, b = np.nan_to_num(np.asarray(a, np.float64)), np.nan_to_num(np.asarray(b, np.float64))
    return float(np.abs(a - b).max(initial=0.0))


def check_bar(got, want_ref, exact):
    """losses, grads, trans_grad of the CUDA path vs the reference's and float64's; returns the observed errors"""
    (l, g, t), (lr, gr, tr), (l64, g64, t64) = got, want_ref, exact
    assert util.close(l, lr), (l, lr)
    stats = {}
    for name, ours, theirs, ex in (("grad", g, gr, g64), ("trans_grad", t, tr, t64)):
        eo, er = _err(ours, ex), _err(theirs, ex)
        assert eo <= 2.0 * er + util.ATOL, (name, eo, er)
        stats[name] = {"ours_vs_f64": eo, "ref_vs_f64": er, "ours_vs_ref": _err(ours, theirs)}
    fin = np.isfinite(lr)
    stats["loss_rel_vs_ref"] = float(np.max(np.abs(l[fin] - lr[fin]) / np.maximum(np.abs(lr[fin]), 1e-30), initial=0.0))
    return stats


def same_kind(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return (np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isposinf(a), np.isposinf(b))
            and np.array_equal(np.isneginf(a), np.isneginf(b)))


def _record(name, stats):
    d = os.environ.get("GTNB_PARITY_DIR")
    if not d:
        return
    os.makedirs(d, exist_ok=True)
    p = os.path.join(d, "asg_ex_parity_observed.json")
    try:
        cur = json.load(open(p))
    except Exception:
        cur = {}
    cur[name] = stats
    json.dump(cur, open(p, "w"), indent=1, sort_keys=True)


def padded(e, lens):
    """the emissions with NaN in every padding row: the call must never read them"""
    p = e.copy()
    for b, Tb in enumerate(lens):
        p[b, Tb:] = np.nan
    return p


@pytest.mark.parametrize("C", [4, 28, 64, 128, 160])
def test_asg_ex_parity_host_and_device_buffers(ctx, ref, C):
    """random input_lens (NaN padding rows), host and device buffers; C = 160 takes the generic route"""
    B, T, U = 6, 30, 6
    e, tg, tw = inputs(B, T, C, U, seed=13 * C)
    rng = np.random.default_rng(C)
    lens = rng.integers(U, T + 1, B).astype(np.int32)
    lens[1], lens[4] = T, U
    tg[2] = np.full(3, tg[2][0])  # repeats
    lr, gr, tr = ao.ref_asg_batch(e, tw, tg, lens)
    exact = ao.asg_f64_batch(e, tw, tg, lens)
    ep = padded(e, lens)
    for dev in (False, True):
        got = (ctx.asg_loss_ex_dev if dev else ctx.asg_loss_ex)(ep, tw, tg, input_lens=lens)
        for b in range(B):
            assert not got[1][b, lens[b]:].any()  # every row is written: exact zeros beyond T_b
        stats = check_bar(got, (lr, gr, tr), exact)
        _record("capi_C%d_%s" % (C, "device" if dev else "host"), stats)
    lo, _, _ = ao.oracle_asg_batch(e, tw, tg, lens)  # the C oracle agrees too
    assert util.close(got[0], lo)


def test_asg_ex_equal_lengths_agrees_with_asg_loss(ctx, ref):
    B, T, C, U = 5, 40, 28, 8
    e, tg, tw = inputs(B, T, C, U, seed=77)
    lr, gr, tr = ao.ref_asg_batch(e, tw, tg)
    exact = ao.asg_f64_batch(e, tw, tg)
    old = ctx.asg_loss(e, tw, tg)
    check_bar(old, (lr, gr, tr), exact)
    for new in (ctx.asg_loss_ex(e, tw, tg), ctx.asg_loss_ex(e, tw, tg, input_lens=np.full(B, T, np.int32)),
                ctx.asg_loss_ex_dev(e, tw, tg)):
        check_bar(new, (lr, gr, tr), exact)
        assert util.close(new[0], old[0], rtol=1e-4, atol=0.0)


@pytest.mark.parametrize("C", [6, 160])
def test_asg_ex_edge_cases(ctx, ref, C):
    """T_b = 0 (NaN: linearGraph(0, C) accepts nothing), an infeasible target and U = 0 (+inf, the denominator's
    gradient alone), T_b = 1, repeated labels; on the device path (C = 6) and the generic route (C = 160)"""
    T = 5
    rng = np.random.default_rng(7)
    tg = [[], [1, 1, 1], [3, 3], [4, 1, 5, 0], [1], [5, 4, 3, 1, 0, 1], [], [2]]
    lens = np.array([5, 5, 0, 5, 1, 5, 0, 3], np.int32)
    B = len(tg)
    e = rng.uniform(-4, 4, (B, T, C)).astype(np.float32)
    tw = rng.uniform(-3, 3, C + C * C).astype(np.float32)
    lr, gr, tr = ao.ref_asg_batch(e, tw, tg, lens)
    assert np.isnan(lr[2]) and np.isnan(lr[6]) and np.isposinf(lr[0]) and np.isposinf(lr[5])
    for got in (ctx.asg_loss_ex(padded(e, lens), tw, tg, input_lens=lens),
                ctx.asg_loss_ex_dev(padded(e, lens), tw, tg, input_lens=lens)):
        check_bar(got, (lr, gr, tr), ao.asg_f64_batch(e, tw, tg, lens))
        assert same_kind(got[0], lr)
        assert not got[1][2].any() and not got[1][6].any()


def test_asg_ex_empty_batch_zeroes_transition_gradient(ctx):
    from gtn_b200 import capi
    C = 8
    e = np.zeros((0, 4, C), np.float32)
    tw = np.ones(C + C * C, np.float32)
    l, g, t = ctx.asg_loss_ex(e, tw, [])
    assert l.shape == (0,) and t.shape == (C + C * C,) and not t.any()
    w_dev, tg_dev = ctx.to_device(tw), ctx.to_device(np.full(C + C * C, 7.0, np.float32))
    try:
        ctx._check(capi.lib().gtnb_asg_loss_ex(ctx.h, 0, 4, C, w_dev.ptr, 1, None, w_dev.ptr, 1, None,
                                               np.zeros(1, np.int32).ctypes.data_as(capi._i32p),
                                               np.zeros(1, np.float32).ctypes.data_as(capi._f32p), None, 1,
                                               tg_dev.ptr, 1))
        assert not tg_dev.download((C + C * C,)).any()
    finally:
        w_dev.free()
        tg_dev.free()


@pytest.mark.parametrize("where", ["start_inf", "start_nan", "w_inf", "w_nan", "emission_nan", "emission_inf"])
def test_asg_ex_non_finite_weights_match_reference_in_kind(ctx, ref, where):
    B, T, C, U = 3, 8, 6, 2
    e, tg, tw = inputs(B, T, C, U, seed=5)
    lens = np.array([8, 6, 7], np.int32)
    if where == "start_inf":
        tw[tg[1][0]] = np.inf
    elif where == "start_nan":
        tw[2] = np.nan
    elif where == "w_inf":
        tw[C + tg[2][1] * C + tg[2][0]] = -np.inf
    elif where == "w_nan":
        tw[C + 7] = np.nan
    elif where == "emission_nan":
        e[1, 3, 2] = np.nan
    else:
        e[0, 2, tg[0][0]] = np.inf
    lr, gr, tr = ao.ref_asg_batch(e, tw, tg, lens)
    for got in (ctx.asg_loss_ex(padded(e, lens), tw, tg, input_lens=lens),
                ctx.asg_loss_ex_dev(padded(e, lens), tw, tg, input_lens=lens)):
        l, g, t = got
        for a, b_ in ((l, lr), (g, gr), (t, tr)):
            assert same_kind(a, b_), where
        fin = np.isfinite(lr)
        assert util.close(l[fin], lr[fin])


def test_asg_ex_bad_arguments(ctx):
    from gtn_b200 import capi
    e = np.zeros((2, 4, 5), np.float32)
    tw = np.zeros(30, np.float32)
    for tg, kw in (([[1], [5]], {}), ([[1], [-1]], {}), ([[1], [2]], {"input_lens": [4, 5]}),
                   ([[1], [2]], {"input_lens": [-1, 2]})):
        with pytest.raises(capi.GtnbInvalidArgument):
            ctx.asg_loss_ex(e, tw, tg, **kw)


def test_asg_ex_at_config(ctx, ref):
    """16 utterances of configs[2]'s shape (B=128 T=500 C=64 U=50) with random lengths: the whole batch on the GPU,
    the first 16 against the reference and float64"""
    B, T, C, U, n = 128, 500, 64, 50, 16
    e, tg, tw = inputs(B, T, C, U)
    lens = np.random.default_rng(11).integers(U, T + 1, B).astype(np.int32)
    got = ctx.asg_loss_ex_dev(padded(e, lens), tw, tg, input_lens=lens)
    part = ctx.asg_loss_ex_dev(padded(e[:n], lens[:n]), tw, tg[:n], input_lens=lens[:n])
    assert np.array_equal(got[0][:n], part[0])  # one CTA per utterance and lattice: the same scores
    assert np.abs(got[1][:n] - part[1]).max() < 1e-6  # (emission gradients: red.add from two streams, any order)
    lr, gr, tr = ao.ref_asg_batch(e[:n], tw, tg[:n], lens[:n])
    stats = check_bar(part, (lr, gr, tr), ao.asg_f64_batch(e[:n], tw, tg[:n], lens[:n]))
    stats["shape"] = "B=%d (first %d checked) T=%d C=%d U=%d, input_lens U(U, T)" % (B, n, T, C, U)
    _record("config_B128_T500_C64_U50_ragged", stats)


@pytest.mark.parametrize("reduction", ["mean", "none"])
def test_torch_asg_loss_input_lengths_matches_truncated_loop(reduction):
    torch = pytest.importorskip("torch")
    from gtn_b200 import torch_loss
    B, T, C, U = 5, 40, 12, 5
    e, tg, tw = inputs(B, T, C, U, seed=99)
    lens = np.array([40, 33, 5, 12, 27], np.int32)
    for il in (torch.tensor(lens), list(lens), torch.tensor(lens).cuda()):
        x = torch.tensor(padded(e, lens), device="cuda", requires_grad=True)
        w = torch.tensor(tw, device="cuda", requires_grad=True)
        loss = torch_loss.asg_loss(x, w, tg, reduction=reduction, input_lengths=il)
        (loss if reduction == "mean" else loss.sum()).backward()
        want_l, want_w, want_x = [], torch.zeros_like(w), torch.zeros_like(x)
        for b in range(B):  # the existing path, one truncated utterance at a time
            xb = torch.tensor(e[b:b + 1, :lens[b]], device="cuda", requires_grad=True)
            wb = torch.tensor(tw, device="cuda", requires_grad=True)
            lb = torch_loss.asg_loss(xb, wb, tg[b:b + 1], reduction="none")
            (lb.sum() / (B if reduction == "mean" else 1)).backward()
            want_l.append(float(lb.detach()))
            want_w += wb.grad
            want_x[b, :lens[b]] = xb.grad[0]
        got_l = loss.detach().cpu().numpy()
        assert util.close(got_l, np.mean(want_l) if reduction == "mean" else np.array(want_l))
        assert not x.grad.isnan().any()  # the NaN padding rows were never read
        # (two fp32 evaluations, each about 1e-5 from float64 at T = 40: DESIGN.md "Tolerances")
        assert np.abs((x.grad - want_x).cpu().numpy()).max() < 5e-5
        assert np.abs((w.grad - want_w).cpu().numpy()).max() < 1e-4 * max(1.0, float(want_w.abs().max()))
        assert w.grad.is_cuda and w.grad.shape == w.shape


@pytest.mark.parametrize("reduction", ["mean", "none"])
def test_torch_ctc_loss_input_lengths_matches_truncated_loop(reduction):
    torch = pytest.importorskip("torch")
    from gtn_b200 import torch_loss
    B, T, C, U = 5, 40, 12, 5
    e, tg = util.bench_inputs(B, T, C, U, 31)
    lens = np.array([40, 33, 11, 12, 27], np.int32)
    for il in (torch.tensor(lens), list(lens)):
        x = torch.tensor(e, device="cuda", requires_grad=True)  # (rows beyond T_b: random scores, not to be read)
        loss = torch_loss.ctc_loss(x, tg, reduction=reduction, input_lengths=il)
        (loss if reduction == "mean" else loss.sum()).backward()
        want_l, want_x = [], torch.zeros_like(x)
        for b in range(B):
            xb = torch.tensor(e[b:b + 1, :lens[b]], device="cuda", requires_grad=True)
            lb = torch_loss.ctc_loss(xb, tg[b:b + 1], reduction="none")
            (lb.sum() / (B if reduction == "mean" else 1)).backward()
            want_l.append(float(lb.detach()))
            want_x[b, :lens[b]] = xb.grad[0]
        got_l = loss.detach().cpu().numpy()
        assert util.close(got_l, np.mean(want_l) if reduction == "mean" else np.array(want_l))
        assert np.abs((x.grad - want_x).cpu().numpy()).max() < 1e-5


def _rank(rank, world, port, total, q):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from gtn_b200 import dist as gd, torch_loss
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world,
                            device_id=torch.device("cuda", rank))
    T, C, U = 30, 10, 4
    first, count = gd.shard(rank, world, total)
    e, tg, tw = inputs(total, T, C, U, seed=11)
    lens = np.arange(total, dtype=np.int32) % 7 + 20
    x = torch.tensor(e[first:first + count], device="cuda", requires_grad=True)
    w = torch.tensor(tw, device="cuda", requires_grad=True)
    torch_loss.asg_loss(x, w, tg[first:first + count], reduction="none",
                        input_lengths=lens[first:first + count]).sum().backward()
    if rank == 0:
        q.put(w.grad.cpu().numpy())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_ranks_nccl_asg_ex_transition_gradient(oracle):
    torch = pytest.importorskip("torch")
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    total, world, port = 7, 2, 29587
    mctx = mp.get_context("spawn")
    q = mctx.Queue()
    procs = [mctx.Process(target=_rank, args=(r, world, port, total, q)) for r in range(world)]
    for p in procs:
        p.start()
    tgrad = q.get(timeout=240)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    T, C, U = 30, 10, 4
    e, tg, tw = inputs(total, T, C, U, seed=11)
    lens = np.arange(total, dtype=np.int32) % 7 + 20
    _, _, want = ao.asg_f64_batch(e, tw, tg, lens)
    assert np.abs(tgrad - want).max() < 1e-3 * max(1.0, np.abs(want).max())
