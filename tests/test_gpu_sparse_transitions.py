"""gtnb_sparse_transitions_loss (user target graphs with a learned transition graph G of any shape) on the GPU against
the live reference (tests/sparse_trans_oracle.py), utterance by utterance on its own T_b rows: both routes (k_sparse.cu's
sweeps over G beside the implicit sweeps of the folded products, materialised lattices), asserted from the kernel
profile; host and device buffers, device arc weights; the golden fixture; the trigram at C = 30; the identities with
gtnb_graph_transitions_loss, gtnb_ngram_ctc_loss and gtnb_asg_loss_ex when G is their dense graph; edge cases, bad
input and torch_loss.sparse_transitions_loss."""
import ctypes as C_

import numpy as np
import pytest

from gtn_b200 import capi
from tests import graph_oracle as go
from tests import graph_trans_oracle as gt
from tests import sparse_trans_oracle as st
from tests import util
from tests.test_gpu_graph_transitions import _gtn_graph, views_of
from tests.test_sparse_trans_oracle import GOLDEN, G_of, graphs_of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


def gview(G):
    return capi.make_view(G["flags"], G["src"], G["dst"], G["olabel"], G["olabel"])


def batch(C, seed, B=6, T=12):
    """CTC graphs and random cyclic graphs (several start and accept nodes, labels >= C); ragged lengths, NaN in the
    padding"""
    rng = np.random.default_rng(seed)
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


def dense_G(rng, C, N=8):
    """a random G in which every path of labels has a match: N nodes, each with one out-arc per label to a random
    node (so a node's in-arcs carry several labels: the products are not label-uniform), 20 more arcs labelled >= C,
    3 start and 3 accept nodes, and two unreachable nodes with arcs among themselves"""
    flags = np.zeros(N + 2, np.uint8)
    flags[rng.choice(N, 3, replace=False)] |= 1
    flags[rng.choice(N, 3, replace=False)] |= 2
    flags[N:] = 2
    src = np.concatenate([np.repeat(np.arange(N), C), rng.integers(0, N, 20), [N, N + 1]])
    dst = np.concatenate([rng.integers(0, N, N * C), rng.integers(0, N, 20), [N + 1, N]])
    lab = np.concatenate([np.tile(np.arange(C), N), rng.integers(C, C + 2, 20), [0, 1]])
    return go.make(flags, src, dst, lab)


def check(got, want, T):
    (l, g, ag, tg), (lr, gr, agr, tgr) = got, want
    assert util.close(l, lr), (l, lr)
    mag = float(np.max(np.abs(lr[np.isfinite(lr)]), initial=1.0)) + 5.0 * T
    assert util.grad_close(g, gr, mag), float(np.nanmax(np.abs(g - gr)))
    assert util.grad_close(ag, agr, mag), float(np.nanmax(np.abs(ag - agr)))
    assert util.grad_close(tg, tgr, mag * len(l)), float(np.nanmax(np.abs(tg - tgr)))


def routed(ctx, run):
    """run() with the kernel profile on -> (its result, the route the call took): the device route launches
    k_sparse.cu's sweeps and the product fold and builds no lattice; the materialised route builds lattices
    (compose_emit) and launches neither.  A call that took both (a retry after the device route) is neither."""
    ctx.profile(True)
    ctx.profile_read()
    try:
        out = run()
        names = set(ctx.profile_read())
    finally:
        ctx.profile(False)
    dev = {"product_fold", "sparse_den_forward"} & names
    if dev == {"product_fold", "sparse_den_forward"} and "compose_emit" not in names:
        return out, "device"
    if not dev and "compose_emit" in names:
        return out, "materialised"
    return out, "both: %s" % sorted(names)


def run_all(ctx, e, graphs, lens, G, tw, want, want_aw, aw, route):
    """host and device buffers, with and without arc weights, each call on the expected route"""
    for run, arc_weights, w in ((ctx.sparse_transitions_loss, None, want), (ctx.sparse_transitions_loss, aw, want_aw),
                                (ctx.sparse_transitions_loss_dev, None, want),
                                (ctx.sparse_transitions_loss_dev, aw, want_aw)):
        got, taken = routed(ctx, lambda: run(e, views_of(graphs), gview(G), tw, input_lens=lens,
                                             arc_weights=arc_weights))
        if route:
            assert taken == route, (taken, route)
        check(got, w, e.shape[1])
        assert not np.isnan(got[1]).any()  # every row written, 0 beyond T_b
        for b in range(len(lens)):
            assert not got[1][b, lens[b]:].any()


@pytest.mark.parametrize("C", [4, 28, 30, 64, 128])
@pytest.mark.parametrize("implicit", [1, 0])
def test_parity_both_routes_host_and_device(ref, ctx, C, implicit):
    rng = np.random.default_rng(C + 17 * implicit)
    e, graphs, lens = batch(C, seed=C + implicit)
    G = dense_G(rng, C)
    tw = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    aw = np.concatenate([g["w"] for g in graphs]) + 0.125
    want = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
    want_aw = st.ref_sparse_trans_loss(e, graphs, G, tw, lens, weights=aw)
    assert np.isfinite(want[0]).any()
    ctx.set_flag("implicit", implicit)
    try:
        run_all(ctx, e, graphs, lens, G, tw, want, want_aw, aw, "device" if implicit else "materialised")
    finally:
        ctx.set_flag("implicit", 1)


@pytest.mark.parametrize("name", ["a", "b", "c"])
@pytest.mark.parametrize("implicit", [1, 0])
def test_golden_both_routes(ctx, name, implicit):
    """the fixture (trigram G; sparse G with unreachable nodes and labels >= C; -inf transitions, which the device
    route hands to the materialised one) on both routes"""
    z = np.load(GOLDEN)
    e, lens, G, tw = z[name + "_e"], z[name + "_lens"], G_of(z, name), z[name + "_trans_w"]
    want = (z[name + "_losses"], z[name + "_grads"], z[name + "_arc_grads"], z[name + "_trans_grad"])
    route = ("materialised" if not implicit else "device" if name != "c" else None)
    ctx.set_flag("implicit", implicit)
    try:
        for run in (ctx.sparse_transitions_loss, ctx.sparse_transitions_loss_dev):
            got, taken = routed(ctx, lambda: run(e, views_of(graphs_of(z, name)), gview(G), tw, input_lens=lens))
            if route:
                assert taken == route, (taken, route)
            else:
                assert taken.startswith("both"), taken  # the status bit moved the call
            if np.isfinite(want[3]).all():
                check(got, want, e.shape[1])
            else:  # -inf transitions: NaN transition gradient slots, as the reference's
                assert util.close(got[0], want[0]) and util.close(got[3], want[3])
                check(got[:3] + (np.nan_to_num(got[3]),), want[:3] + (np.nan_to_num(want[3]),), e.shape[1])
    finally:
        ctx.set_flag("implicit", 1)


def test_trigram_at_c30_takes_the_device_route(ref, ctx):
    """the corrected trigram of timeNgramCtc's alphabet (900 states, 27 000 arcs) with CTC graphs"""
    C, T, B = 30, 24, 3
    rng = np.random.default_rng(30)
    G = st.trigram_graph(C)
    tw = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    graphs = [go.ctc_graph(rng.integers(1, C, 4)) for _ in range(B)]
    lens = np.asarray([T, T - 3, T - 8], np.int32)
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    want = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
    got, taken = routed(ctx, lambda: ctx.sparse_transitions_loss_dev(e, views_of(graphs), gview(G), tw,
                                                                     input_lens=lens))
    assert taken == "device", taken
    check(got, want, T)


def _rel(a, b):
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-30)))


def test_identity_bigram(ctx):
    """G = the dense bigram graph reproduces gtnb_graph_transitions_loss BIGRAM and, on CTC graphs,
    gtnb_ngram_ctc_loss, at the n-gram benchmark shape B=128 T=500 C=64 U=50"""
    B, T, C, U = 128, 500, 64, 50
    e, targets = util.bench_inputs(B, T, C, U)
    W = np.random.default_rng(1).uniform(-0.5, 0.5, C * C).astype(np.float32)
    lens = np.asarray([T - 3 * b for b in range(B)], np.int32)
    graphs = [go.ctc_graph(t, blank=0) for t in targets]
    G, slots = st.bigram_graph(C), st.bigram_slots(C)
    (l, g, ag, tg), taken = routed(ctx, lambda: ctx.sparse_transitions_loss_dev(e, views_of(graphs), gview(G), W[slots],
                                                                                 input_lens=lens))
    assert taken == "device", taken
    tg_w = np.zeros(C * C, np.float64)
    np.add.at(tg_w, slots, tg)
    ld, gd, agd, tgd = ctx.graph_transitions_loss_dev(e, views_of(graphs), W, kind=capi.DENSE_BIGRAM, input_lens=lens)
    ln, gn, tgn = ctx.ngram_ctc_loss_dev(e, W, targets, blank=0, input_lens=lens)
    for lw, gw, tgw in ((ld, gd, tgd), (ln, gn, tgn)):
        assert _rel(l, lw) <= 1e-5, _rel(l, lw)
        assert util.grad_close(g, gw, 5.0 * T), float(np.abs(g - gw).max())
        assert util.grad_close(tg_w, tgw, 5.0 * T * B), float(np.abs(tg_w - tgw).max())
    assert util.grad_close(ag, agd, 5.0 * T), float(np.abs(ag - agd).max())


def test_identity_asg(ctx):
    """G = ASG's graph reproduces gtnb_graph_transitions_loss ASG and, on force-align chains, gtnb_asg_loss_ex, at
    B=128 T=500 C=64 U=50"""
    B, T, C, U = 128, 500, 64, 50
    e, targets = util.bench_inputs(B, T, C, U)
    tw = np.random.default_rng(2).uniform(-0.5, 0.5, C + C * C).astype(np.float32)
    lens = np.asarray([T - 3 * b for b in range(B)], np.int32)
    graphs = [gt.fal_graph(t) for t in targets]
    G = st.asg_graph(C)  # arc k reads trans_w[k]
    (l, g, ag, tg), taken = routed(ctx, lambda: ctx.sparse_transitions_loss_dev(e, views_of(graphs), gview(G), tw,
                                                                                 input_lens=lens))
    assert taken == "device", taken
    ld, gd, agd, tgd = ctx.graph_transitions_loss_dev(e, views_of(graphs), tw, kind=capi.DENSE_ASG, input_lens=lens)
    la, ga, tga = ctx.asg_loss_ex_dev(e, tw, targets, input_lens=lens)
    for lw, gw, tgw in ((ld, gd, tgd), (la, ga, tga)):
        assert _rel(l, lw) <= 1e-5, _rel(l, lw)
        assert util.grad_close(g, gw, 5.0 * T), float(np.abs(g - gw).max())
        assert util.grad_close(tg, tgw, 5.0 * T * B), float(np.abs(tg - tgw).max())
    assert util.grad_close(ag, agd, 5.0 * T), float(np.abs(ag - agd).max())


def test_edge_cases(ref, ctx):
    C = 5
    rng = np.random.default_rng(2)
    G = st.trigram_graph(C)
    tw = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    # B = 0 zeroes the transition gradient
    for run in (ctx.sparse_transitions_loss, ctx.sparse_transitions_loss_dev):
        assert not run(np.zeros((0, 3, C), np.float32), [], gview(G), tw)[3].any()
    e = rng.uniform(-2, 2, (4, 4, C)).astype(np.float32)
    chain = go.make([1, 0, 2], [0, 1], [1, 2], [1, 2])
    graphs = [chain, go.make([1, 0, 0, 0, 0, 2], [0, 1, 2, 3, 4], [1, 2, 3, 4, 5], [1, 2, 3, 4, 1]),
              go.make([0, 2], [0], [1], [1]), go.make([], [], [], [])]
    lens = np.asarray([0, 4, 4, 4], np.int32)  # T_b = 0; too short; no start node; no arcs
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            l, g, ag, tg = ctx.sparse_transitions_loss(e, views_of(graphs), gview(G), tw, input_lens=lens)
        finally:
            ctx.set_flag("implicit", 1)
        assert np.isnan(l[0]) and np.isposinf(l[1:]).all()
        assert not g[0].any() and not ag.any() and np.isfinite(g).all() and np.isfinite(tg).all()
        assert np.allclose(g[1:].sum(axis=2), 1.0, atol=1e-4)  # the denominator's gradient alone
        want = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
        check((l, g, ag, tg), want, 4)
    # a G that accepts nothing in T_b frames: a 3-arc chain against 4 frames, NaN as the reference's
    Gc = go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3])
    twc = np.zeros(3, np.float32)
    ctc = [go.ctc_graph([1, 2])] * 2
    want = st.ref_sparse_trans_loss(e[:2], ctc, Gc, twc, [4, 4])
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            got = ctx.sparse_transitions_loss(e[:2], views_of(ctc), gview(Gc), twc, input_lens=[4, 4])
        finally:
            ctx.set_flag("implicit", 1)
        assert np.isnan(got[0]).all() and np.isnan(want[0]).all()
        assert util.close(got[1], want[1]) and util.close(got[3], want[3])


def test_bad_input(ctx):
    C = 5
    e = np.zeros((1, 4, C), np.float32)
    graphs = views_of([go.ctc_graph([1])])
    eps = go.make([1, 2], [0], [1], [-1])
    with pytest.raises(capi.GtnbError) as ex:
        ctx.sparse_transitions_loss(e, graphs, gview(eps), np.zeros(1, np.float32))
    assert ex.value.code == capi.ERR_UNSUPPORTED and "remove" in str(ex.value)
    trans = go.make([1, 2], [0], [1], [1], [2])
    with pytest.raises(capi.GtnbError) as ex:
        ctx.sparse_transitions_loss(e, graphs, capi.make_view(trans["flags"], trans["src"], trans["dst"],
                                                              trans["ilabel"], trans["olabel"]), np.zeros(1, np.float32))
    assert ex.value.code == capi.ERR_UNSUPPORTED and "project" in str(ex.value)
    bad = go.make([1, 2], [0], [5], [1])  # arc into a node that does not exist
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.sparse_transitions_loss(e, graphs, gview(bad), np.zeros(1, np.float32))
    G = st.trigram_graph(C)
    with pytest.raises(capi.GtnbInvalidArgument):  # T_b > T
        ctx.sparse_transitions_loss(e, graphs, gview(G), np.zeros(C ** 3, np.float32), input_lens=[5])
    ag = go.make([1, 2], [0], [1], [-1])  # epsilon in A_b
    with pytest.raises(capi.GtnbError) as ex:
        ctx.sparse_transitions_loss(e, views_of([ag]), gview(G), np.zeros(C ** 3, np.float32))
    assert ex.value.code == capi.ERR_UNSUPPORTED
    # NULL trans_w with B > 0
    gv, _keep = gview(G)
    arr = (capi.GraphView * 1)(graphs[0][0])
    losses = np.zeros(1, np.float32)
    rc = capi.lib().gtnb_sparse_transitions_loss(ctx.h, 1, 4, C, e.ctypes.data, 0, None, arr, None, 0, C_.byref(gv),
                                                  None, 0, losses.ctypes.data_as(capi._f32p), None, 0, None, 0, None,
                                                  0)
    assert rc == capi.ERR_INVALID_ARGUMENT


@pytest.mark.parametrize("reduction", ["mean", "none"])
@pytest.mark.parametrize("with_weights", [True, False])
def test_torch_sparse_transitions_loss_matches_the_oracle(ref, reduction, with_weights):
    torch = pytest.importorskip("torch")
    import gtn_b200.gtn as gtn
    from gtn_b200 import torch_loss
    C = 12
    rng = np.random.default_rng(11)
    e, graphs, lens = batch(C, seed=11)
    e = np.nan_to_num(e, nan=7.0)
    B = len(graphs)
    G = dense_G(rng, C)
    tw0 = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    w0 = np.concatenate([g["w"] for g in graphs]) + 0.25
    x = torch.tensor(e, device="cuda", requires_grad=True)
    tr = torch.tensor(tw0, device="cuda", requires_grad=True)
    w = torch.tensor(w0, device="cuda", requires_grad=True) if with_weights else None
    out = torch_loss.sparse_transitions_loss(x, tr, _gtn_graph(gtn, G), [_gtn_graph(gtn, g) for g in graphs],
                                             input_lengths=torch.tensor(lens), weights=w, reduction=reduction)
    up = 1.5  # reduction "none": the transition gradient supports a uniform upstream gradient
    (out * (up if reduction == "none" else 1.0)).sum().backward()
    lr, gr, agr, tgr = st.ref_sparse_trans_loss(e, graphs, G, tw0, lens, weights=w0 if with_weights else None)
    fin = np.isfinite(lr)
    scale = up if reduction == "none" else 1.0 / B
    if reduction == "mean":
        assert util.close(out.item(), lr.mean())
    else:
        assert util.close(out.detach().cpu().numpy(), lr)
    assert fin.any()
    assert util.grad_close(x.grad.cpu().numpy(), gr * scale, 50.0)
    assert util.grad_close(tr.grad.cpu().numpy(), tgr * scale, 50.0 * B)
    if with_weights:
        assert util.grad_close(w.grad.cpu().numpy(), agr * scale, 50.0)
