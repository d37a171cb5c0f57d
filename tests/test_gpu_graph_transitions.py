"""gtnb_graph_transitions_loss (user target graphs with learned ASG or bigram transitions) on the GPU against the live
reference (tests/graph_trans_oracle.py), utterance by utterance on its own T_b rows: both kinds, both routes
(implicit sweeps beside the dense trellis, materialised lattices), host and device buffers, device arc weights, the
golden fixture's graph families and -inf transitions; the identities with gtnb_asg_loss_ex (force-align chains) and
gtnb_ngram_ctc_loss (CTC graphs); edge cases and bad input; torch_loss.graph_transitions_loss."""
import numpy as np
import pytest

from gtn_b200 import capi
from tests import graph_oracle as go
from tests import graph_trans_oracle as gt
from tests import util
from tests.test_graph_trans_oracle import GOLDEN, graphs_of

pytestmark = pytest.mark.gpu
KINDS = {"asg": capi.DENSE_ASG, "bigram": capi.DENSE_BIGRAM}


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


def views_of(graphs):
    return [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]


def transitions(rng, C, kind, scale=1.0):
    return rng.uniform(-scale, scale, (C + C * C) if kind == capi.DENSE_ASG else C * C).astype(np.float32)


def batch(C, seed, kinds=("ctc", "wild", "rand")):
    """one graph of each family, cycled to B = 2 * len(kinds); ragged lengths, NaN in the padding"""
    rng = np.random.default_rng(seed)
    graphs = []
    for k in kinds * 2:
        if k == "ctc":
            g = go.ctc_graph(rng.integers(1, C, int(rng.integers(1, 5))))
        elif k == "wild":
            g = go.with_wildcards(go.ctc_graph(rng.integers(1, C, int(rng.integers(1, 3)))), C, w_loop=-0.2)
        else:
            g = go.random_graph(rng, 8, 30, C, n_start=2, n_accept=2, label_hi=C + 2)
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
        graphs.append(g)
    B, T = len(graphs), 12
    lens = rng.integers(T // 2, T + 1, B).astype(np.int32)
    lens[0] = T
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    for b in range(B):
        e[b, lens[b]:] = np.nan
    return e, graphs, lens


def check(got, want, T):
    (l, g, ag, tg), (lr, gr, agr, tgr) = got, want
    assert util.close(l, lr), (l, lr)
    mag = float(np.max(np.abs(lr[np.isfinite(lr)]), initial=1.0)) + 5.0 * T
    assert util.grad_close(g, gr, mag), float(np.nanmax(np.abs(g - gr)))
    assert util.grad_close(ag, agr, mag), float(np.nanmax(np.abs(ag - agr)))
    assert util.grad_close(tg, tgr, mag * len(l)), float(np.nanmax(np.abs(tg - tgr)))


def routed(ctx, run):
    """run() with the kernel profile on -> (its result, the route the call took): the device route launches the
    product fold and the dense trellis and builds no lattice; the materialised route builds lattices (compose_emit)
    and launches neither.  A call that took both (a retry after the device route) is neither."""
    ctx.profile(True)
    ctx.profile_read()
    try:
        out = run()
        names = set(ctx.profile_read())
    finally:
        ctx.profile(False)
    trellis = {"product_fold", "asg_den_forward", "ngram_den_forward"} & names
    if "product_fold" in names and trellis - {"product_fold"} and "compose_emit" not in names:
        return out, "device"
    if not trellis and "compose_emit" in names:
        return out, "materialised"
    return out, "both: %s" % sorted(names)


def check_all_buffers(ctx, e, graphs, lens, k, tw, want, want_aw, aw, route):
    """host and device buffers, with and without arc weights, each call on the expected route"""
    for run, arc_weights, w in ((ctx.graph_transitions_loss, None, want),
                                (ctx.graph_transitions_loss, aw, want_aw),
                                (ctx.graph_transitions_loss_dev, None, want),
                                (ctx.graph_transitions_loss_dev, aw, want_aw)):
        got, taken = routed(ctx, lambda: run(e, views_of(graphs), tw, kind=k, input_lens=lens, arc_weights=arc_weights))
        assert taken == route, (taken, route)
        check(got, w, e.shape[1])
        assert not np.isnan(got[1]).any()  # every row written, 0 beyond T_b
        for b in range(len(lens)):
            assert not got[1][b, lens[b]:].any()


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("C", [4, 28, 29, 64, 128])
@pytest.mark.parametrize("implicit", [1, 0])
def test_parity_both_routes_host_and_device(ref, ctx, kind, C, implicit):
    """CTC graphs and random cyclic graphs (several start and accept nodes, start nodes with in-arcs, labels >= C):
    their products fit the implicit layout at every C, so implicit = 1 takes the device route and implicit = 0 the
    materialised one"""
    k = KINDS[kind]
    e, graphs, lens = batch(C, seed=C + implicit + 7 * k, kinds=("ctc", "rand"))
    assert any((g["flags"][g["dst"]] & 1).any() for g in graphs[1::2])  # start nodes with in-arcs
    tw = transitions(np.random.default_rng(C), C, k)
    aw = np.concatenate([g["w"] for g in graphs]) + 0.125
    want = gt.ref_graph_trans_loss(e, graphs, k, tw, lens)
    want_aw = gt.ref_graph_trans_loss(e, graphs, k, tw, lens, weights=aw)
    ctx.set_flag("implicit", implicit)
    try:
        check_all_buffers(ctx, e, graphs, lens, k, tw, want, want_aw, aw, "device" if implicit else "materialised")
    finally:
        ctx.set_flag("implicit", 1)


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("C,route", [(4, "device"), (128, "materialised")])
def test_wildcard_graphs(ref, ctx, kind, C, route):
    """wildcard states: a wildcard node becomes C copies with C in-arcs each, which fits the implicit layout at small C
    and not at C = 128, where the call takes the materialised lattices with the implicit flag on"""
    k = KINDS[kind]
    e, graphs, lens = batch(C, seed=C + 3 * k, kinds=("wild", "ctc"))
    tw = transitions(np.random.default_rng(C + 1), C, k)
    aw = np.concatenate([g["w"] for g in graphs]) - 0.125
    want = gt.ref_graph_trans_loss(e, graphs, k, tw, lens)
    want_aw = gt.ref_graph_trans_loss(e, graphs, k, tw, lens, weights=aw)
    check_all_buffers(ctx, e, graphs, lens, k, tw, want, want_aw, aw, route)


@pytest.fixture(scope="module")
def decompositions_c128(ref):
    """word-piece decomposition graphs over 127 pieces (C = 128), built with the reference's own ops"""
    pieces = go.inventory(26, 128, seed=7)
    rng = np.random.default_rng(21)
    graphs = []
    for _ in range(3):
        g = go.from_ref(go.decomposition_graph(go.REF_OPS, [int(x) for x in rng.integers(0, 26, 8)], pieces))
        g["w"] = rng.uniform(-0.5, 0.5, len(g["src"])).astype(np.float32)
        graphs.append(g)
    return graphs


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_decompositions_at_c128_on_the_device_route(ctx, decompositions_c128, kind):
    """the benchmark's headline workload at a small size: decomposition graphs at C = 128 on the device route, every
    output against the reference"""
    graphs, C = decompositions_c128, 128
    k = KINDS[kind]
    rng = np.random.default_rng(31)
    T = 24
    lens = np.asarray([24, 17, 20], np.int32)
    e = rng.uniform(-3, 3, (len(graphs), T, C)).astype(np.float32)
    for b in range(len(graphs)):
        e[b, lens[b]:] = np.nan
    tw = transitions(rng, C, k)
    aw = np.concatenate([g["w"] for g in graphs]) + 0.25
    want = gt.ref_graph_trans_loss(e, graphs, k, tw, lens)
    want_aw = gt.ref_graph_trans_loss(e, graphs, k, tw, lens, weights=aw)
    assert np.isfinite(want[0]).all()
    check_all_buffers(ctx, e, graphs, lens, k, tw, want, want_aw, aw, "device")


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("name", ["a", "b", "c"])
@pytest.mark.parametrize("implicit", [1, 0])
def test_golden_fixture(ctx, name, kind, implicit):
    """decomposition, CTC, random cyclic and wildcard graphs, T_b in {0, 1}, infeasible graphs, -inf transitions
    (batch c: the reference's inf / NaN propagation)"""
    z = np.load(GOLDEN)
    p = "%s_%s_" % (name, kind)
    graphs, e, lens = graphs_of(z, name), z[name + "_e"], z[name + "_lens"]
    want = tuple(z[p + s] for s in ("losses", "grads", "arc_grads", "trans_grad"))
    ctx.set_flag("implicit", implicit)
    try:
        for run in (ctx.graph_transitions_loss, ctx.graph_transitions_loss_dev):
            check(run(e, views_of(graphs), z[p + "trans_w"], kind=KINDS[kind], input_lens=lens), want, e.shape[1])
    finally:
        ctx.set_flag("implicit", 1)


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_non_finite_weight_gives_the_references_inf_nan(ref, ctx, kind):
    k = KINDS[kind]
    C = 6
    e, graphs, lens = batch(C, seed=3, kinds=("ctc", "rand"))
    tw = transitions(np.random.default_rng(5), C, k)
    tw[-C * C + 1] = -np.inf
    tw[-C * C + 7] = np.inf
    want = gt.ref_graph_trans_loss(e, graphs, k, tw, lens)
    got = ctx.graph_transitions_loss_dev(e, views_of(graphs), tw, kind=k, input_lens=lens)
    check(got, want, e.shape[1])


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_identity_with_the_target_criteria(ctx, kind):
    """force-align chains (ASG) / CTC graphs (BIGRAM) give gtnb_asg_loss_ex / gtnb_ngram_ctc_loss at the n-gram
    benchmark shape (B=128 T=500 C=64 U=50), 16 utterances"""
    B, T, C, U = 16, 500, 64, 50
    e, targets = util.bench_inputs(B, T, C, U)
    k = KINDS[kind]
    tw = transitions(np.random.default_rng(1), C, k, scale=0.5)
    lens = np.asarray([T - 7 * b for b in range(B)], np.int32)
    if k == capi.DENSE_ASG:
        graphs = [gt.fal_graph(t) for t in targets]
        lw, gw, tgw = ctx.asg_loss_ex_dev(e, tw, targets, input_lens=lens)
    else:
        graphs = [go.ctc_graph(t, blank=0) for t in targets]
        lw, gw, tgw = ctx.ngram_ctc_loss_dev(e, tw, targets, blank=0, input_lens=lens)
    l, g, _, tg = ctx.graph_transitions_loss_dev(e, views_of(graphs), tw, kind=k, input_lens=lens)
    assert util.close(l, lw), np.abs(l - lw).max()
    assert util.grad_close(g, gw, 5.0 * T), float(np.abs(g - gw).max())
    assert util.grad_close(tg, tgw, 5.0 * T * B), float(np.abs(tg - tgw).max())


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_edge_cases(ctx, kind):
    k = KINDS[kind]
    C = 5
    tw = transitions(np.random.default_rng(2), C, k)
    # B = 0 zeroes the transition gradient
    _, _, _, tg = ctx.graph_transitions_loss(np.zeros((0, 3, C), np.float32), [], tw, kind=k)
    assert not tg.any()
    _, _, _, tg = ctx.graph_transitions_loss_dev(np.zeros((0, 3, C), np.float32), [], tw, kind=k)
    assert not tg.any()
    e = np.random.default_rng(3).uniform(-2, 2, (4, 4, C)).astype(np.float32)
    chain = go.make([1, 0, 2], [0, 1], [1, 2], [1, 2])
    graphs = [chain, go.make([1, 0, 0, 0, 0, 2], [0, 1, 2, 3, 4], [1, 2, 3, 4, 5], [1, 2, 3, 4, 1]),
              go.make([0, 2], [0], [1], [1]), go.make([], [], [], [])]
    lens = np.asarray([0, 4, 4, 4], np.int32)  # T_b = 0; too short; no start node; no arcs
    l, g, ag, tg = ctx.graph_transitions_loss(e, views_of(graphs), tw, kind=k, input_lens=lens)
    assert np.isnan(l[0]) and np.isposinf(l[1:]).all()
    assert not g[0].any() and not ag.any() and np.isfinite(g).all() and np.isfinite(tg).all()
    # the denominator's gradient alone: each row of an infeasible utterance is the softmax-like posterior, sum 1
    assert np.allclose(g[1:].sum(axis=2), 1.0, atol=1e-4)


def test_bad_input(ctx):
    C = 5
    e = np.zeros((1, 4, C), np.float32)
    tw = np.zeros(C + C * C, np.float32)
    g = go.ctc_graph([1, 2])
    with pytest.raises(capi.GtnbError) as ei:
        ctx.graph_transitions_loss(e, views_of([go.make([1, 2], [0], [1], [-1])]), tw)
    assert ei.value.code == capi.ERR_UNSUPPORTED and "remove" in str(ei.value)
    for lens in ([5], [-1]):
        with pytest.raises(capi.GtnbInvalidArgument):
            ctx.graph_transitions_loss(e, views_of([g]), tw, input_lens=lens)
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.graph_transitions_loss(e, views_of([go.make([1, 2], [0], [7], [1])]), tw)
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.graph_transitions_loss(e, views_of([g]), tw, kind=2)
    C = 129
    with pytest.raises(capi.GtnbError) as ei:
        ctx.graph_transitions_loss(np.zeros((1, 4, C), np.float32), views_of([g]), np.zeros(C * C, np.float32),
                                   kind=capi.DENSE_BIGRAM)
    assert ei.value.code == capi.ERR_UNSUPPORTED


def _gtn_graph(gtn, g):
    h = gtn.Graph()
    for f in g["flags"]:
        h.add_node(bool(f & 1), bool(f & 2))
    for a in range(len(g["src"])):
        h.add_arc(int(g["src"][a]), int(g["dst"][a]), int(g["ilabel"][a]), int(g["olabel"][a]), float(g["w"][a]))
    return h


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("reduction", ["mean", "none"])
@pytest.mark.parametrize("with_weights", [True, False])
def test_torch_graph_transitions_loss_matches_the_oracle(ref, kind, reduction, with_weights):
    torch = pytest.importorskip("torch")
    import gtn_b200.gtn as gtn
    from gtn_b200 import torch_loss
    k = KINDS[kind]
    C = 12
    e, graphs, lens = batch(C, seed=11, kinds=("wild", "ctc", "rand"))
    e = np.nan_to_num(e, nan=7.0)
    B = len(graphs)
    tw0 = transitions(np.random.default_rng(4), C, k)
    w0 = np.concatenate([g["w"] for g in graphs]) + 0.25
    x = torch.tensor(e, device="cuda", requires_grad=True)
    tr = torch.tensor(tw0, device="cuda", requires_grad=True)
    w = torch.tensor(w0, device="cuda", requires_grad=True) if with_weights else None
    out = torch_loss.graph_transitions_loss(x, tr, [_gtn_graph(gtn, g) for g in graphs], kind=kind,
                                            input_lengths=torch.tensor(lens), weights=w, reduction=reduction)
    up = 1.5  # reduction "none": the transition gradient supports a uniform upstream gradient
    (out * (up if reduction == "none" else 1.0)).sum().backward()
    lr, gr, agr, tgr = gt.ref_graph_trans_loss(e, graphs, k, tw0, lens, weights=w0 if with_weights else None)
    scale = up if reduction == "none" else 1.0 / B
    if reduction == "mean":
        assert util.close(out.item(), lr.mean())
    else:
        assert util.close(out.detach().cpu().numpy(), lr)
    assert util.grad_close(x.grad.cpu().numpy(), gr * scale, 50.0)
    assert util.grad_close(tr.grad.cpu().numpy(), tgr * scale, 50.0 * B)
    if with_weights:
        assert util.grad_close(w.grad.cpu().numpy(), agr * scale, 50.0)
