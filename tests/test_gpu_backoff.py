"""gtnb_backoff_transitions_loss and gtnb_viterbi_backoff (a transition graph G with epsilon arcs, the backoff arcs of
a pruned n-gram LM) on the GPU against the live reference (tests/backoff_oracle.py), utterance by utterance: both
routes of the loss (k_sparse.cu's backoff sweeps, the exact composition), asserted from the kernel profile, with host
and device buffers; the decode's paths, arcs and scores ==, ties included, with exact_ties on and off; the benchmark's
backoff trigram at C = 64 on the device route; an epsilon-free G == the sparse entry points; the golden fixture; edge
cases, bad input and the torch functions."""
import ctypes as C_
import os

import numpy as np
import pytest

from gtn_b200 import capi
from tests import backoff_oracle as bo
from tests import graph_oracle as go
from tests import sparse_trans_oracle as st
from tests import util
from tests.test_gpu_graph_transitions import _gtn_graph, views_of

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "backoff_golden.npz")
DEVICE = {"sparse_eps_forward", "sparse_eps_gather"}


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


def gview(G):
    return capi.make_view(G["flags"], G["src"], G["dst"], G["olabel"], G["olabel"])


def routed(ctx, run, device=DEVICE):
    """run() with the kernel profile on -> (its result, the route: "device" launches the backoff sweeps and composes
    nothing, "exact" composes and launches no backoff sweep, "both" a retry after the device route)"""
    ctx.profile(True)
    ctx.profile_read()
    try:
        out = run()
        names = set(ctx.profile_read())
    finally:
        ctx.profile(False)
    dev = device <= names
    exact = any(n.startswith("gcompose") or n == "compose_emit" for n in names)
    if dev and not exact:
        return out, "device"
    if exact and not (names & device):
        return out, "exact"
    return out, "both: %s" % sorted(names)


def routed_names(ctx, run):
    """run() with the kernel profile on -> (its result, the names of the kernels it launched)"""
    ctx.profile(True)
    ctx.profile_read()
    try:
        out = run()
        return out, set(ctx.profile_read())
    finally:
        ctx.profile(False)


def check(got, want, T):
    (l, g, ag, tg), (lr, gr, agr, tgr) = got, want
    assert util.close(l, lr), (l, lr)
    mag = float(np.max(np.abs(lr[np.isfinite(lr)]), initial=1.0)) + 5.0 * T
    assert util.grad_close(g, gr, mag), float(np.nanmax(np.abs(g - gr)))
    assert util.grad_close(ag, agr, mag), float(np.nanmax(np.abs(ag - agr)))
    assert util.grad_close(tg, tgr, mag * len(l)), float(np.nanmax(np.abs(tg - tgr)))


def batch(rng, C, B=6, T=12):
    """CTC graphs and random graphs (several start and accept nodes, labels >= C); ragged lengths, NaN padding"""
    graphs = []
    for b in range(B):
        if b % 2 == 0:
            g = go.ctc_graph(rng.integers(1, C, int(rng.integers(1, 4))))
        else:
            g = go.random_graph(rng, 6, 24, C, n_start=2, n_accept=2, label_hi=C + 2)
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
        graphs.append(g)
    lens = rng.integers(T // 2, T + 1, B).astype(np.int32)
    lens[0] = T
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    for b in range(B):
        e[b, lens[b]:] = np.nan
    return e, graphs, lens


def Gs(rng, C):
    return {"bigram": bo.backoff_ngram(rng, C, 2, n_tokens=1500), "trigram": bo.backoff_ngram(rng, C, 3),
            "random": bo.eps_graph(rng, 10, 50, C, 14, label_hi=C + 1)}


@pytest.mark.parametrize("kind", ["bigram", "trigram", "random"])
@pytest.mark.parametrize("implicit", [1, 0])
def test_loss_parity_both_routes_host_and_device(ref, ctx, kind, implicit):
    C = 8
    rng = np.random.default_rng(len(kind) + 7 * implicit)
    G, tw = Gs(rng, C)[kind]
    e, graphs, lens = batch(rng, C)
    aw = np.concatenate([g["w"] for g in graphs]) + 0.125
    want = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
    want_aw = st.ref_sparse_trans_loss(e, graphs, G, tw, lens, weights=aw)
    assert np.isfinite(want[0]).any()
    ctx.set_flag("implicit", implicit)
    try:
        for run, arc_weights, w in ((ctx.backoff_transitions_loss, None, want),
                                    (ctx.backoff_transitions_loss, aw, want_aw),
                                    (ctx.backoff_transitions_loss_dev, None, want),
                                    (ctx.backoff_transitions_loss_dev, aw, want_aw)):
            got, taken = routed(ctx, lambda: run(e, views_of(graphs), gview(G), tw, input_lens=lens,
                                                 arc_weights=arc_weights))
            assert taken == ("device" if implicit else "exact"), taken
            check(got, w, e.shape[1])
            for b in range(len(lens)):
                assert not got[1][b, lens[b]:].any()
    finally:
        ctx.set_flag("implicit", 1)


def test_nonfinite_takes_the_exact_route(ref, ctx):
    """-inf transitions (pruned arcs) move the call to the exact route, which matches the reference"""
    C = 6
    rng = np.random.default_rng(21)
    G, tw = bo.backoff_ngram(rng, C, 3, n_neg_inf=4)
    e, graphs, lens = batch(rng, C, B=4, T=8)
    want = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
    got, taken = routed(ctx, lambda: ctx.backoff_transitions_loss_dev(e, views_of(graphs), gview(G), tw,
                                                                      input_lens=lens))
    assert taken.startswith("both"), taken
    assert util.close(got[0], want[0])
    check(got[:3] + (np.nan_to_num(got[3]),), want[:3] + (np.nan_to_num(want[3]),), e.shape[1])


@pytest.mark.parametrize("exact_ties", [1, 0])
@pytest.mark.parametrize("kind", ["bigram", "trigram", "random", "ties"])
def test_decode_equals_the_reference(ref, ctx, kind, exact_ties):
    """paths, arcs and scores == the reference's; "ties": integer emissions and zero weights, so that paths tie and
    exact_ties decides (off: a tied utterance keeps a best path of the device route, with the same score)"""
    C, T, B = 7, 14, 6
    rng = np.random.default_rng(len(kind) + 3 * exact_ties)
    if kind == "ties":
        G, tw = bo.backoff_ngram(rng, C, 3)
        tw = np.zeros_like(tw)
        e = rng.integers(-1, 2, (B, T, C)).astype(np.float32)
    else:
        G, tw = Gs(rng, C)[kind]
        e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    lens = np.asarray([T, 0, 1, 5, T - 2, T], np.int32)
    want = bo.ref_backoff_viterbi(e, G, tw, lens)
    ctx.set_flag("exact_ties", exact_ties)
    try:
        for run in (ctx.viterbi_backoff, ctx.viterbi_backoff_dev):
            paths, scores, arcs = run(e, gview(G), tw, input_lens=lens)
            assert np.array_equal(scores, want[1]), (scores, want[1])
            if exact_ties or kind != "ties":
                assert np.array_equal(paths, want[0]) and np.array_equal(arcs, want[2])
            for b in range(B):  # every path is a path of G's emitting arcs with its own labels
                n = int(lens[b]) if np.isfinite(scores[b]) else 0
                assert (arcs[b, n:] == -1).all() and np.array_equal(paths[b, :n], G["olabel"][arcs[b, :n]])
        ctx.set_flag("implicit", 0)
        paths, scores, arcs = ctx.viterbi_backoff(e, gview(G), tw, input_lens=lens)
        assert np.array_equal(scores, want[1]) and np.array_equal(paths, want[0]) and np.array_equal(arcs, want[2])
    finally:
        ctx.set_flag("exact_ties", 1)
        ctx.set_flag("implicit", 1)


def test_backoff_trigram_c64_takes_the_device_route(ref, ctx):
    """the benchmark's pruned backoff trigram (2065 states, 17 344 emitting and 2064 epsilon arcs; 189 440 arcs with
    its epsilons removed, beyond the envelope) trains and decodes without building a lattice"""
    C, T, B = 64, 30, 3
    rng = np.random.default_rng(64)
    G, tw = bo.backoff_lm(rng, C)
    assert len(G["flags"]) == 2065 and (G["olabel"] == -1).sum() == 2064
    graphs = [go.ctc_graph(rng.integers(1, C, 5)) for _ in range(B)]
    lens = np.asarray([T, T - 4, T - 9], np.int32)
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    want = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
    got, taken = routed(ctx, lambda: ctx.backoff_transitions_loss_dev(e, views_of(graphs), gview(G), tw,
                                                                      input_lens=lens))
    assert taken == "device", taken
    check(got, want, T)
    wv = bo.ref_backoff_viterbi(e, G, tw, lens)
    ctx.set_flag("exact_ties", 0)  # (a tie would re-run its utterance on the exact route)
    try:
        (paths, scores, arcs), taken = routed(ctx, lambda: ctx.viterbi_backoff_dev(e, gview(G), tw, input_lens=lens),
                                              {"sparse_eps_viterbi", "sparse_eps_trace"})
    finally:
        ctx.set_flag("exact_ties", 1)
    assert taken == "device", taken
    assert np.array_equal(scores, wv[1]) and np.array_equal(paths, wv[0]) and np.array_equal(arcs, wv[2])


def test_epsilon_free_equals_the_sparse_entry_points(ctx):
    """an epsilon-free G takes gtnb_sparse_transitions_loss's and gtnb_viterbi_sparse's own routes (the same kernels):
    losses and decode outputs ==; the gradients, which both accumulate with float atomics in a run-to-run order, agree
    to float32 rounding"""
    C = 10
    rng = np.random.default_rng(9)
    G = st.sparse_graph(rng, 12, 80, C, label_hi=C + 1)
    tw = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e, graphs, lens = batch(rng, C)
    e = np.nan_to_num(e, nan=0.5)
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            a, ra = routed_names(ctx, lambda: ctx.backoff_transitions_loss_dev(e, views_of(graphs), gview(G), tw,
                                                                               input_lens=lens))
            b, rb = routed_names(ctx, lambda: ctx.sparse_transitions_loss_dev(e, views_of(graphs), gview(G), tw,
                                                                              input_lens=lens))
            assert ra == rb and not any(n.startswith("sparse_eps") for n in ra), (ra, rb)
            assert np.array_equal(a[0], b[0], equal_nan=True)
            for x, y in zip(a[1:], b[1:]):
                assert np.allclose(x, y, rtol=1e-5, atol=1e-6), float(np.abs(x - y).max())
            a = ctx.viterbi_backoff(e, gview(G), tw, input_lens=lens)
            b = ctx.viterbi_sparse(e, gview(G), tw, input_lens=lens)
            for x, y in zip(a, b):
                assert np.array_equal(x, y)
        finally:
            ctx.set_flag("implicit", 1)


@pytest.mark.parametrize("name", ["bigram", "trigram", "random"])
def test_golden_both_routes(ctx, name):
    z = np.load(GOLDEN)
    G = go.make(z[name + "_G_flags"], z[name + "_G_src"], z[name + "_G_dst"], z[name + "_G_label"])
    tw, e, lens = z[name + "_trans_w"], z[name + "_e"], z[name + "_lens"]
    graphs = [go.make(z["%s_A%d_flags" % (name, b)], z["%s_A%d_src" % (name, b)], z["%s_A%d_dst" % (name, b)],
                      z["%s_A%d_label" % (name, b)]) for b in range(len(lens))]
    want = (z[name + "_losses"], z[name + "_grads"], z[name + "_arc_grads"], z[name + "_trans_grad"])
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            check(ctx.backoff_transitions_loss(e, views_of(graphs), gview(G), tw, input_lens=lens), want, e.shape[1])
            paths, scores, arcs = ctx.viterbi_backoff(e, gview(G), tw, input_lens=lens)
            assert np.array_equal(scores, z[name + "_scores"]) and np.array_equal(paths, z[name + "_paths"])
            assert np.array_equal(arcs, z[name + "_arcs"])
        finally:
            ctx.set_flag("implicit", 1)


def test_edge_cases(ref, ctx):
    C = 5
    rng = np.random.default_rng(2)
    G, tw = bo.backoff_ngram(rng, C, 3, n_tokens=800)
    for run in (ctx.backoff_transitions_loss, ctx.backoff_transitions_loss_dev):  # B = 0 zeroes the transition gradient
        assert not run(np.zeros((0, 3, C), np.float32), [], gview(G), tw)[3].any()
    e = rng.uniform(-2, 2, (4, 4, C)).astype(np.float32)
    graphs = [go.make([1, 0, 2], [0, 1], [1, 2], [1, 2]), go.make([1, 0, 0, 0, 0, 2], [0, 1, 2, 3, 4],
                                                                  [1, 2, 3, 4, 5], [1, 2, 3, 4, 1]),
              go.make([0, 2], [0], [1], [1]), go.make([], [], [], [])]
    lens = np.asarray([0, 4, 4, 4], np.int32)  # T_b = 0; too short; no start node; no arcs
    want = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            l, g, ag, tg = ctx.backoff_transitions_loss(e, views_of(graphs), gview(G), tw, input_lens=lens)
        finally:
            ctx.set_flag("implicit", 1)
        assert np.isnan(l[0]) and np.isposinf(l[1:]).all()
        assert not g[0].any() and not ag.any() and np.isfinite(g).all() and np.isfinite(tg).all()
        check((l, g, ag, tg), want, 4)
    # epsilon arcs out of a start node at frame 0 and into an accept node at frame T_b
    G2 = go.make([1, 0, 0, 2], [0, 1, 2, 1], [1, 2, 3, 1], [-1, 0, -1, 1])
    tw2 = np.asarray([0.5, -0.25, 0.75, 0.1], np.float32)
    ctc = [go.ctc_graph([0])] * 2
    want = st.ref_sparse_trans_loss(e[:2], ctc, G2, tw2, [3, 1])
    wv = bo.ref_backoff_viterbi(e[:2], G2, tw2, [3, 1])
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            check(ctx.backoff_transitions_loss(e[:2], views_of(ctc), gview(G2), tw2, input_lens=[3, 1]), want, 4)
            got = ctx.viterbi_backoff(e[:2], gview(G2), tw2, input_lens=[3, 1])
            assert all(np.array_equal(x, y) for x, y in zip(got, wv))
        finally:
            ctx.set_flag("implicit", 1)


def test_bad_input(ctx):
    C = 5
    e = np.zeros((1, 4, C), np.float32)
    graphs = views_of([go.ctc_graph([1])])
    G, tw = bo.eps_cycle_graph()
    for call in (lambda: ctx.backoff_transitions_loss(e, graphs, gview(G), tw),
                 lambda: ctx.viterbi_backoff(e, gview(G), tw)):
        with pytest.raises(capi.GtnbInvalidArgument) as ex:
            call()
        assert "cycle of epsilon arcs" in str(ex.value)
    half = go.make([1, 2], [0], [1], [-1], [1])  # epsilon on one side only: a transducer
    for call in (lambda: ctx.backoff_transitions_loss(e, graphs, capi.make_view(
                     half["flags"], half["src"], half["dst"], half["ilabel"], half["olabel"]), np.zeros(1, np.float32)),
                 lambda: ctx.viterbi_backoff(e, capi.make_view(half["flags"], half["src"], half["dst"], half["ilabel"],
                                                               half["olabel"]), np.zeros(1, np.float32))):
        with pytest.raises(capi.GtnbError) as ex:
            call()
        assert ex.value.code == capi.ERR_UNSUPPORTED
    G, tw = bo.backoff_ngram(np.random.default_rng(1), C, 2, n_tokens=300)
    with pytest.raises(capi.GtnbError) as ex:  # epsilon in A_b
        ctx.backoff_transitions_loss(e, views_of([go.make([1, 2], [0], [1], [-1])]), gview(G), tw)
    assert ex.value.code == capi.ERR_UNSUPPORTED
    with pytest.raises(capi.GtnbInvalidArgument):  # T_b > T
        ctx.backoff_transitions_loss(e, graphs, gview(G), tw, input_lens=[5])
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.viterbi_backoff(e, gview(G), tw, input_lens=[5])
    gv, _keep = gview(G)
    arr = (capi.GraphView * 1)(graphs[0][0])
    losses = np.zeros(1, np.float32)
    rc = capi.lib().gtnb_backoff_transitions_loss(ctx.h, 1, 4, C, e.ctypes.data, 0, None, arr, None, 0, C_.byref(gv),
                                                   None, 0, losses.ctypes.data_as(capi._f32p), None, 0, None, 0, None,
                                                   0)
    assert rc == capi.ERR_INVALID_ARGUMENT


@pytest.mark.parametrize("reduction", ["mean", "none"])
def test_torch_functions(ref, reduction):
    torch = pytest.importorskip("torch")
    import gtn_b200.gtn as gtn
    from gtn_b200 import torch_loss
    C = 9
    rng = np.random.default_rng(13)
    G, tw0 = bo.backoff_ngram(rng, C, 3, n_tokens=1200)
    e, graphs, lens = batch(rng, C)
    e = np.nan_to_num(e, nan=7.0)
    B = len(graphs)
    w0 = np.concatenate([g["w"] for g in graphs]) + 0.25
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        x = torch.tensor(e, device="cuda", requires_grad=True)
        tr = torch.tensor(tw0, device="cuda", requires_grad=True)
        w = torch.tensor(w0, device="cuda", requires_grad=True)
        out = torch_loss.backoff_transitions_loss(x, tr, _gtn_graph(gtn, G), [_gtn_graph(gtn, g) for g in graphs],
                                                  input_lengths=torch.tensor(lens), weights=w, reduction=reduction)
        up = 1.5
        (out * (up if reduction == "none" else 1.0)).sum().backward()
        paths, scores, arcs = torch_loss.backoff_viterbi(x.detach(), tr.detach(), _gtn_graph(gtn, G),
                                                         input_lengths=torch.tensor(lens))
    side.synchronize()
    lr, gr, agr, tgr = st.ref_sparse_trans_loss(e, graphs, G, tw0, lens, weights=w0)
    scale = up if reduction == "none" else 1.0 / B
    if reduction == "mean":
        assert util.close(out.item(), lr.mean())
    else:
        assert util.close(out.detach().cpu().numpy(), lr)
    assert util.grad_close(x.grad.cpu().numpy(), gr * scale, 50.0)
    assert util.grad_close(tr.grad.cpu().numpy(), tgr * scale, 50.0 * B)
    assert util.grad_close(w.grad.cpu().numpy(), agr * scale, 50.0)
    wp, ws, wa = bo.ref_backoff_viterbi(e, G, tw0, lens)
    assert np.array_equal(scores.cpu().numpy(), ws) and np.array_equal(paths.cpu().numpy(), wp)
    assert np.array_equal(arcs.cpu().numpy(), wa)
