"""gtnb_graph_viterbi (Viterbi alignment over user-supplied target graphs) on the GPU against the live reference
(tests/graph_viterbi_oracle.py), utterance by utterance on its own T_b rows: paths, arcs and scores ==, on both routes
(tropical sweep + traceback, materialised lattices), host and device buffers, device arc weights; the route each call
took, read from the kernel profile; tie-heavy inputs, which send the tied utterances alone to the materialised route;
an olabel-sorted graph with a node of out-degree > C; non-finite values; edge cases and bad input; CTC graphs against
the reference's CTC forced alignment; and torch_loss.graph_viterbi against the C ABI."""
import numpy as np
import pytest

from gtn_b200 import capi
from tests import graph_oracle as go
from tests import graph_viterbi_oracle as gv
from tests import util

pytestmark = pytest.mark.gpu

COMPOSE = {"compose_count", "compose_emit"}


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


def views_of(graphs, adjacency=None):
    if adjacency is None:
        return [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
    return [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"], *adj)
            for g, adj in zip(graphs, adjacency)]


def batch(C, seed, kinds=("ctc", "wild", "rand"), ties=False, T=18):
    """one graph of each kind, cycled to B = 2 * len(kinds); ragged lengths, NaN in the padding"""
    rng = np.random.default_rng(seed)
    graphs = []
    for k in kinds * 2:
        if k == "ctc":
            g = go.ctc_graph(rng.integers(1, C, int(rng.integers(1, 6))))
        elif k == "wild":
            g = go.with_wildcards(go.ctc_graph(rng.integers(1, C, int(rng.integers(1, 4)))), C, w_loop=-0.2)
        else:
            g = go.random_graph(rng, 10, 40, C, label_hi=C + 2)
        g["w"] = (rng.integers(-1, 1, len(g["src"])) if ties else rng.uniform(-1, 1, len(g["src"]))).astype(np.float32)
        graphs.append(g)
    B = len(graphs)
    lens = rng.integers(T // 2, T + 1, B).astype(np.int32)
    lens[0] = T
    e = (rng.integers(0, 2, (B, T, C)) if ties else rng.uniform(-3, 3, (B, T, C))).astype(np.float32)
    for b in range(B):
        e[b, lens[b]:] = np.nan
    return e, graphs, lens


def routed(ctx, run):
    """run() with the kernel profile on -> (its result, the kernel names it launched)"""
    ctx.profile(True)
    ctx.profile_read()
    try:
        out = run()
        names = set(ctx.profile_read())
    finally:
        ctx.profile(False)
    return out, names


def route_of(names):
    dev = {"implicit_trace"} <= names and bool({"implicit_forward_max", "implicit_forward_arc_max"} & names)
    if dev and not COMPOSE & names:
        return "device"
    if not dev and COMPOSE <= names:
        return "materialised"
    if dev and COMPOSE <= names:
        return "device+exact"
    return "unknown %s" % sorted(names)


def same(got, want):
    (p, s, a), (pr, sr, ar) = got, want
    assert np.array_equal(s, sr, equal_nan=True), (s, sr)
    assert np.array_equal(p, pr), np.argwhere(p != pr)[:5]
    assert np.array_equal(a, ar), np.argwhere(a != ar)[:5]


def check_both_buffers(ctx, e, graphs, lens, route, weights=None, adjacency=None):
    want = gv.ref_graph_viterbi(e, graphs, lens, weights, olabel_sorted=adjacency is not None)
    for f in (ctx.graph_viterbi, ctx.graph_viterbi_dev):
        got, names = routed(ctx, lambda: f(e, views_of(graphs, adjacency), input_lens=lens, arc_weights=weights))
        same(got, want)
        if route is not None:
            assert route_of(names) == route, (route_of(names), route)
    return want


@pytest.mark.parametrize("C", [4, 28, 64, 256, 1024])
@pytest.mark.parametrize("implicit", [1, 0])
def test_parity_both_routes_host_and_device(ref, ctx, C, implicit):
    e, graphs, lens = batch(C, seed=C + implicit)
    ctx.set_flag("implicit", implicit)
    try:
        # wildcard states at C = 1024 have more in-arcs than the wide kernels hold: the route is not asserted there
        check_both_buffers(ctx, e, graphs, lens, None if C == 1024 else ("device" if implicit else "materialised"))
    finally:
        ctx.set_flag("implicit", 1)


@pytest.mark.parametrize("implicit", [1, 0])
def test_golden_fixture(ctx, implicit):
    """the committed fixture's graph families (tests/golden/graph_viterbi_golden.npz), on both routes"""
    from tests.test_graph_viterbi_oracle import golden_batches
    ctx.set_flag("implicit", implicit)
    try:
        for name, e, graphs, lens, want in golden_batches():
            for f in (ctx.graph_viterbi, ctx.graph_viterbi_dev):
                same(f(e, views_of(graphs), input_lens=lens), want)
    finally:
        ctx.set_flag("implicit", 1)


@pytest.mark.parametrize("C", [4, 28])
def test_device_arc_weights(ref, ctx, C):
    e, graphs, lens = batch(C, seed=40 + C)
    w = np.random.default_rng(6).uniform(-2, 2, sum(len(g["src"]) for g in graphs)).astype(np.float32)
    check_both_buffers(ctx, e, graphs, lens, "device", weights=w)


@pytest.fixture(scope="module")
def decompositions(ref):
    """word-piece alignment graphs over 127 pieces (C = 128), built with the reference's own ops, and the same with
    wildcard states"""
    pieces = go.inventory(26, 128, seed=7)
    rng = np.random.default_rng(21)
    graphs = []
    for _ in range(3):
        g = go.from_ref(go.decomposition_graph(go.REF_OPS, [int(x) for x in rng.integers(0, 26, 6)], pieces))
        g["w"] = rng.uniform(-0.5, 0.5, len(g["src"])).astype(np.float32)
        graphs.append(g)
    return graphs


@pytest.mark.parametrize("wild", [False, True])
def test_decomposition_graphs(ctx, decompositions, wild):
    C, T = 128, 24
    graphs = [go.with_wildcards(g, C, w_loop=-0.1) if wild else g for g in decompositions]
    rng = np.random.default_rng(31)
    lens = np.asarray([24, 17, 20], np.int32)
    e = rng.uniform(-3, 3, (len(graphs), T, C)).astype(np.float32)
    for b in range(len(graphs)):
        e[b, lens[b]:] = np.nan
    check_both_buffers(ctx, e, graphs, lens, "device")


@pytest.mark.parametrize("C", [4, 28])
def test_ties_take_the_exact_route_and_match(ref, ctx, C):
    """integer emissions and weights: many utterances tie; they alone re-run on the materialised lattices"""
    e, graphs, lens = batch(C, seed=50 + C, ties=True)
    check_both_buffers(ctx, e, graphs, lens, "device+exact")


def test_a_tie_sends_only_its_utterance_to_the_exact_route(ref, ctx):
    """one utterance ties (two parallel equal self-loops), the others do not: the call takes both routes, and the
    untied utterances alone take the device route"""
    C, T = 6, 10
    rng = np.random.default_rng(60)
    graphs = [go.ctc_graph(rng.integers(1, C, 3)) for _ in range(3)]
    for g in graphs:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    graphs.append(go.make([1, 2], [0, 0, 1, 1], [1, 1, 1, 1], [1, 1, 2, 2]))
    e = rng.uniform(-3, 3, (4, T, C)).astype(np.float32)
    want = gv.ref_graph_viterbi(e, graphs)
    got, names = routed(ctx, lambda: ctx.graph_viterbi(e, views_of(graphs)))
    same(got, want)
    assert route_of(names) == "device+exact", names
    got, names = routed(ctx, lambda: ctx.graph_viterbi(e[:3], views_of(graphs[:3])))
    same(got, tuple(x[:3] for x in want))
    assert route_of(names) == "device", names
    # with exact_ties off the tie keeps the device route's path, one of the optimal ones
    ctx.set_flag("exact_ties", 0)
    try:
        (p, s, a), names = routed(ctx, lambda: ctx.graph_viterbi(e, views_of(graphs)))
    finally:
        ctx.set_flag("exact_ties", 1)
    assert route_of(names) == "device", names
    assert np.array_equal(s, want[1]) and np.array_equal(p[:3], want[0][:3]) and np.array_equal(a[:3], want[2][:3])
    assert gv.path_score(e[3], graphs[3], a[3]) == s[3]


def test_olabel_sorted_graph_with_out_degree_above_c(ref, ctx):
    """an olabel-sorted graph (the reference's sorted matcher) with a node of out-degree > C, tie-heavy emissions"""
    C, T = 3, 8
    rng = np.random.default_rng(70)
    N = 4
    src, dst, lab = [], [], []
    for s in range(N):
        for d in range(N):
            for c in range(C):
                src.append(s), dst.append(d), lab.append(c)
    perm = rng.permutation(len(src))
    g = go.make([1, 0, 0, 2], np.asarray(src)[perm], np.asarray(dst)[perm], np.asarray(lab)[perm],
                w=rng.integers(-1, 1, len(src)))
    rg = go.ref_graph(g)
    rg.arc_sort(olabel=True)
    ip, ia, op, oa = rg.adjacency()
    assert (np.diff(op) > C).any()
    e = rng.integers(0, 2, (2, T, C)).astype(np.float32)
    _, scores, arcs = check_both_buffers(ctx, e, [g, g], None, "device+exact", adjacency=[(ip, ia, op, oa)] * 2)
    assert np.isfinite(scores).all() and (arcs >= 0).all()


@pytest.mark.parametrize("where", ["emission_nan", "emission_inf", "w_neginf", "w_nan"])
def test_non_finite_values(ref, ctx, where):
    C = 9
    e, graphs, lens = batch(C, seed=9, kinds=("wild", "ctc"))
    e = np.nan_to_num(e, nan=0.0)
    if where == "emission_nan":
        e[1, 3, 2] = np.nan
    elif where == "emission_inf":
        e[2, 2, int(graphs[2]["olabel"][1])] = np.inf
    elif where == "w_neginf":
        graphs[3]["w"][1] = -np.inf
    else:
        graphs[0]["w"][3] = np.nan
    check_both_buffers(ctx, e, graphs, lens, None)


def test_edge_cases(ref, ctx):
    C = 6
    wild = go.with_wildcards(go.ctc_graph([2, 3]), C)
    chain = go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3])  # accepts length 3 only
    empty = go.make([], [], [], [])
    graphs = [wild, wild, chain, empty, chain]
    lens = np.asarray([0, 1, 5, 6, 3], np.int32)
    e = np.random.default_rng(8).uniform(-3, 3, (5, 6, C)).astype(np.float32)
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            for f in (ctx.graph_viterbi, ctx.graph_viterbi_dev):
                p, s, a = f(e, views_of(graphs), input_lens=lens)
                assert np.isneginf(s[[0, 2, 3]]).all() and (p[[0, 2, 3]] == -1).all() and (a[[0, 2, 3]] == -1).all()
                same((p, s, a), gv.ref_graph_viterbi(e, graphs, lens))
        finally:
            ctx.set_flag("implicit", 1)
    p, s, a = ctx.graph_viterbi(np.zeros((0, 5, C), np.float32), [])
    assert p.shape == (0, 5) and s.shape == (0,)


def test_bad_input(ctx):
    C = 5
    g = go.ctc_graph([1, 2])
    e = np.zeros((1, 4, C), np.float32)
    eps = go.make([1, 2], [0], [1], [-1])
    with pytest.raises(capi.GtnbError) as ei:
        ctx.graph_viterbi(e, views_of([eps]))
    assert ei.value.code == capi.ERR_UNSUPPORTED and "remove" in str(ei.value)
    for lens in ([5], [-1]):
        with pytest.raises(capi.GtnbInvalidArgument):
            ctx.graph_viterbi(e, views_of([g]), input_lens=lens)
    bad = go.make([1, 2], [0], [7], [1])  # arc endpoint outside the graph
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.graph_viterbi(e, views_of([bad]))


def test_ctc_graphs_agree_with_the_reference_ctc_alignment(ref, ctx):
    B, T, C, U = 16, 1000, 64, 100  # BASELINE.json configs[1] shape
    e, targets = util.bench_inputs(B, T, C, U)
    pr, sr, _ = ref.ref_viterbi_ctc_batch(e, targets, blank=0)
    (p, s, a), names = routed(ctx, lambda: ctx.graph_viterbi(e, views_of([go.ctc_graph(t) for t in targets])))
    assert route_of(names) == "device", names
    assert np.array_equal(s, sr), np.abs(s - sr).max()
    assert np.array_equal(p, pr)


def _gtn_graph(gtn, g):
    h = gtn.Graph()
    for f in g["flags"]:
        h.add_node(bool(f & 1), bool(f & 2))
    for a in range(len(g["src"])):
        h.add_arc(int(g["src"][a]), int(g["dst"][a]), int(g["ilabel"][a]), int(g["olabel"][a]), float(g["w"][a]))
    return h


@pytest.mark.parametrize("with_weights", [False, True])
def test_torch_graph_viterbi_equals_the_c_abi(ref, ctx, with_weights):
    torch = pytest.importorskip("torch")
    import gtn_b200.gtn as gtn
    from gtn_b200 import torch_loss
    C = 12
    e, graphs, lens = batch(C, seed=11, kinds=("wild", "ctc", "rand"))
    w = np.concatenate([g["w"] for g in graphs]) + 0.25 if with_weights else None
    x = torch.tensor(np.nan_to_num(e, nan=7.0), device="cuda")
    p, s, a = torch_loss.graph_viterbi(x, [_gtn_graph(gtn, g) for g in graphs], input_lengths=torch.tensor(lens),
                                       weights=None if w is None else torch.tensor(w, device="cuda"))
    assert p.is_cuda and p.dtype == torch.int32 and s.dtype == torch.float32 and a.shape == p.shape
    got = (p.cpu().numpy(), s.cpu().numpy(), a.cpu().numpy())
    same(got, ctx.graph_viterbi(x.cpu().numpy(), views_of(graphs), input_lens=lens, arc_weights=w))
    same(got, gv.ref_graph_viterbi(x.cpu().numpy(), graphs, lens, w))
    labels, n = torch_loss.collapse(p, blank=0)
    assert labels.shape == p.shape and n.shape == (len(graphs),)
