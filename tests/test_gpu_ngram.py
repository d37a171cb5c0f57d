"""gtnb_ngram_ctc_loss (CTC with a learned bigram transition graph, benchmarks/ctc.cpp:107-134) on the GPU, against
the live reference (oracle/_ref, graph by graph, no fold), the C oracle and the float64 referee
(tests/ngram_oracle.py).  The bar (DESIGN.md "Tolerances"): losses within 1e-4 relative of the reference;
emission and transition gradients at least as close to float64 as the reference's own fp32 gradients are, x2;
non-finite weights equal in kind (inf / NaN) to the reference.  With GTNB_PARITY_DIR set, the observed errors
are written to $GTNB_PARITY_DIR/ngram_parity_observed.json."""
import json
import os
import sys

import numpy as np
import pytest

from tests import ngram_oracle as no
from tests import util

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


def inputs(B, T, C, U, seed=1234, w_scale=2.0):
    """emissions U(-5, 5) and targets in [1, C-1] per utterance (seed + b), W U(-w_scale, w_scale) from seed 4321"""
    e, tg = util.bench_inputs(B, T, C, U, seed)
    W = np.random.default_rng(4321).uniform(-w_scale, w_scale, C * C).astype(np.float32)
    return e, tg, W


def f64_batch(e, W, targets, blank=0, lens=None):
    B, T, C = e.shape
    l64, g64, t64 = np.zeros(B), np.zeros((B, T, C)), np.zeros(C * C)
    for b in range(B):
        Tb = T if lens is None else int(lens[b])
        l64[b], g64[b, :Tb], t = no.ngram_ctc_f64(e[b, :Tb], W, targets[b], blank)
        t64 += t
    return l64, g64, t64


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


def _record(name, stats):
    d = os.environ.get("GTNB_PARITY_DIR")
    if not d:
        return
    os.makedirs(d, exist_ok=True)
    p = os.path.join(d, "ngram_parity_observed.json")
    try:
        cur = json.load(open(p))
    except Exception:
        cur = {}
    cur[name] = stats
    json.dump(cur, open(p, "w"), indent=1, sort_keys=True)


@pytest.mark.parametrize("C", [4, 8, 28, 64, 128])
def test_ngram_capi_parity_host_and_device_buffers(ctx, ref, C):
    B, T, U, blank = 6, 30, 6, 1 if C > 4 else 0
    e, tg, W = inputs(B, T, C, U, seed=17 * C)
    tg = [np.where(t == blank, (blank + 1) % C, t) for t in tg]
    lens = np.array([T, T - 3, 11, T, 1, 19], np.int32)
    tg[1] = tg[1][:0]  # U = 0
    tg[2] = np.full(3, tg[2][0])  # repeats
    lr, gr, tr = no.ref_ngram_ctc_batch(e, W, tg, blank, lens)
    exact = f64_batch(e, W, tg, blank, lens)
    for dev in (False, True):
        if dev:
            got = ctx.ngram_ctc_loss_dev(e, W, tg, blank=blank, input_lens=lens)
        else:
            got = ctx.ngram_ctc_loss(e, W, tg, blank=blank, input_lens=lens)
        for b in range(B):
            assert not got[1][b, lens[b]:].any()  # every row is written: zeros beyond T_b
        stats = check_bar(got, (lr, gr, tr), exact)
    _record("capi_C%d" % C, stats)
    for b in range(B):  # the C oracle (no fold) agrees too
        lo, go, _ = no.oracle_ngram_ctc(e[b, :lens[b]], W, tg[b], blank)
        assert util.close(got[0][b], lo)


def test_ngram_edge_cases(ctx, ref):
    """T_b = 0 (NaN, as the reference: linearGraph(0, C) accepts nothing), U = 0, repeated labels, an infeasible
    target (+inf, the denominator's gradient alone), blank != 0"""
    C, T, blank = 6, 5, 2
    rng = np.random.default_rng(7)
    tg = [[], [1, 1, 1], [3, 3], [4, 1, 5, 0], [1], [5, 4, 3, 1, 0, 1], []]
    lens = np.array([5, 5, 0, 5, 1, 5, 0], np.int32)
    B = len(tg)
    e = rng.uniform(-4, 4, (B, T, C)).astype(np.float32)
    W = rng.uniform(-3, 3, C * C).astype(np.float32)
    lr, gr, tr = no.ref_ngram_ctc_batch(e, W, tg, blank, lens)
    assert np.isnan(lr[2]) and np.isnan(lr[6]) and np.isinf(lr[5])
    got = ctx.ngram_ctc_loss(e, W, tg, blank=blank, input_lens=lens)
    check_bar(got, (lr, gr, tr), f64_batch(e, W, tg, blank, lens))
    assert np.array_equal(np.isnan(got[0]), np.isnan(lr)) and np.array_equal(np.isinf(got[0]), np.isinf(lr))


@pytest.mark.parametrize("where", ["emission_nan", "emission_inf", "w_inf", "w_nan"])
def test_ngram_non_finite_weights_match_reference_in_kind(ctx, ref, where):
    B, T, C, U = 3, 8, 6, 2
    e, tg, W = inputs(B, T, C, U, seed=5)
    if where == "emission_nan":
        e[1, 3, 2] = np.nan
    elif where == "emission_inf":
        e[0, 2, tg[0][0]] = np.inf
    elif where == "w_inf":
        W[tg[2][1] * C + tg[2][0]] = -np.inf
    else:
        W[7] = np.nan
    lr, gr, tr = no.ref_ngram_ctc_batch(e, W, tg)
    for got in (ctx.ngram_ctc_loss(e, W, tg), ctx.ngram_ctc_loss_dev(e, W, tg)):
        l, g, t = got
        for a, b_ in ((l, lr), (g, gr), (t, tr)):
            assert np.array_equal(np.isnan(a), np.isnan(b_)), where
            assert np.array_equal(np.isposinf(a), np.isposinf(b_)) and np.array_equal(np.isneginf(a), np.isneginf(b_))
        fin = np.isfinite(lr)
        assert util.close(l[fin], lr[fin])


def test_ngram_bad_arguments(ctx):
    from gtn_b200 import capi
    e = np.zeros((2, 4, 5), np.float32)
    W = np.zeros(25, np.float32)
    for tg, kw in (([[1], [5]], {}), ([[1], [2]], {"input_lens": [4, 5]}), ([[1], [2]], {"input_lens": [-1, 2]}),
                   ([[1], [2]], {"blank": 5})):
        with pytest.raises(capi.GtnbInvalidArgument):
            ctx.ngram_ctc_loss(e, W, tg, **kw)
    big = np.zeros((1, 2, 129), np.float32)
    with pytest.raises(capi.GtnbError) as ei:
        ctx.ngram_ctc_loss(big, np.zeros(129 * 129, np.float32), [[1]])
    assert ei.value.code == capi.ERR_UNSUPPORTED and "128" in str(ei.value)


def test_ngram_at_config(ctx, ref):
    """16 utterances of the benchmark's shape (configs[2]'s B=128 T=500 C=64 U=50): the whole batch on the GPU, the
    first 16 against the reference and float64"""
    B, T, C, U, n = 128, 500, 64, 50, 16
    e, tg, W = inputs(B, T, C, U)
    got = ctx.ngram_ctc_loss_dev(e, W, tg)
    lr, gr, tr = no.ref_ngram_ctc_batch(e[:n], W, tg[:n])
    exact = f64_batch(e[:n], W, tg[:n])
    # the transition gradient of the first n utterances alone
    part = ctx.ngram_ctc_loss_dev(e[:n], W, tg[:n])
    assert np.array_equal(got[0][:n], part[0])  # one CTA per utterance and lattice: the same scores
    assert np.abs(got[1][:n] - part[1]).max() < 1e-6  # (emission gradients: red.add from two streams, any order)
    stats = check_bar(part, (lr, gr, tr), exact)
    stats["shape"] = "B=%d (first %d checked) T=%d C=%d U=%d" % (B, n, T, C, U)
    _record("config_B128_T500_C64_U50", stats)


def test_torch_ngram_ctc_loss(ref):
    torch = pytest.importorskip("torch")
    from gtn_b200 import torch_loss
    B, T, C, U, blank = 5, 40, 12, 5, 3
    e, tg, W = inputs(B, T, C, U, seed=99)
    tg = [np.where(t == blank, 1, t) for t in tg]
    lens = np.array([40, 33, 40, 12, 27], np.int32)
    lr, gr, tr = no.ref_ngram_ctc_batch(e, W, tg, blank, lens)
    exact = f64_batch(e, W, tg, blank, lens)
    for reduction, il in (("mean", torch.tensor(lens)), ("none", list(lens)), ("mean", torch.tensor(lens).cuda())):
        x = torch.tensor(e, device="cuda", requires_grad=True)
        w = torch.tensor(W.reshape(C, C), device="cuda", requires_grad=True)
        loss = torch_loss.ngram_ctc_loss(x, w, tg, input_lengths=il, blank=blank, reduction=reduction)
        (loss if reduction == "mean" else loss.sum()).backward()
        s = 1.0 / B if reduction == "mean" else 1.0
        ls = loss.detach().cpu().numpy()
        got = (np.full(B, ls) if reduction == "mean" else ls, x.grad.cpu().numpy() / s,
               w.grad.cpu().numpy().ravel() / s)
        if reduction == "mean":
            assert util.close(ls, lr.mean())
            got = (lr, got[1], got[2])
        check_bar(got, (lr, gr, tr), exact)
        assert w.grad.shape == (C, C)


def test_torch_ngram_ctc_loss_moves_nothing_but_the_losses(monkeypatch):
    """Only the B losses visit the host: no Python-side copy of any CUDA tensor during the forward"""
    torch = pytest.importorskip("torch")
    from gtn_b200 import torch_loss
    B, T, C, U = 4, 20, 8, 3
    e, tg, W = inputs(B, T, C, U, seed=3)
    x = torch.tensor(e, device="cuda", requires_grad=True)
    w = torch.tensor(W, device="cuda", requires_grad=True)
    torch.cuda.synchronize()

    def refuse(*a, **k):
        raise AssertionError("a CUDA tensor was moved or read on the host")

    for name in ("cpu", "numpy", "tolist", "item"):
        monkeypatch.setattr(torch.Tensor, name, refuse)
    real_to = torch.Tensor.to

    def to(self, *a, **k):
        assert not self.is_cuda, "a CUDA tensor was moved"
        return real_to(self, *a, **k)

    monkeypatch.setattr(torch.Tensor, "to", to)
    per = torch_loss.ngram_ctc_loss(x, w, tg, reduction="none")
    monkeypatch.undo()
    assert per.is_cuda and per.shape == (B,)
    assert w.is_cuda and w.data_ptr() == w.detach().data_ptr()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        torch_loss.ngram_ctc_loss(x, w, tg, reduction="none")
        torch.cuda.synchronize()
    d2h = [ev for ev in prof.events() if "DtoH" in ev.name or "Device -> Host" in ev.name]
    assert len(d2h) <= 3, [ev.name for ev in d2h]  # the read-back: B denominator and numerator scores, 2B status words


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
    e, tg, W = inputs(total, T, C, U, seed=11)
    x = torch.tensor(e[first:first + count], device="cuda", requires_grad=True)
    w = torch.tensor(W, device="cuda", requires_grad=True)
    torch_loss.ngram_ctc_loss(x, w, tg[first:first + count], reduction="none").sum().backward()
    if rank == 0:
        q.put(w.grad.cpu().numpy())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_ranks_nccl_ngram_transition_gradient(oracle):
    torch = pytest.importorskip("torch")
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    total, world, port = 7, 2, 29583
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
    e, tg, W = inputs(total, T, C, U, seed=11)
    _, _, want = f64_batch(e, W, tg)
    assert np.abs(tgrad - want).max() < 1e-3 * max(1.0, np.abs(want).max())
