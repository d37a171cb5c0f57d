"""gtnb_graph_transitions_viterbi (Viterbi alignment over user-supplied target graphs with learned ASG or bigram
transitions) on the GPU against the live reference (tests/graph_trans_viterbi_oracle.py), utterance by utterance on
its own T_b rows: paths, arcs and scores ==, with the route each call took read from the kernel profile.  Both kinds
at C in {4, 28, 29, 64, 128} on both routes; host and device buffers, device arc weights, transitions on the host and
on the device; the golden fixture; decomposition and wildcard graphs; tie-heavy inputs, whose tied utterances alone re-run on the exact
route; the identities with gtnb_graph_viterbi (zero transitions) and gtnb_viterbi_dense_ex (the free graph);
non-finite values; edge cases and bad input; and torch_loss.graph_transitions_viterbi against the C ABI."""
import numpy as np
import pytest

from gtn_b200 import capi
from tests import graph_oracle as go
from tests import graph_trans_viterbi_oracle as gtv

pytestmark = pytest.mark.gpu

KINDS = {"asg": capi.DENSE_ASG, "bigram": capi.DENSE_BIGRAM}
DEVICE = {"implicit_forward_max", "implicit_trace", "product_fold"}
EXACT = {"gcompose_search", "compose_emit"}


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


def views_of(graphs):
    return [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]


def transitions(rng, C, kind, ties=False):
    n = (C + C * C) if kind == capi.DENSE_ASG else C * C
    return (rng.integers(-1, 1, n) if ties else rng.uniform(-1, 1, n)).astype(np.float32)


def batch(C, seed, kinds=("ctc", "wild", "rand"), ties=False, T=14):
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
    """run() with the kernel profile on -> (its result, the route it took)"""
    ctx.profile(True)
    ctx.profile_read()
    try:
        out = run()
        names = set(ctx.profile_read())
    finally:
        ctx.profile(False)
    dev, exact = DEVICE <= names, EXACT <= names
    route = {(True, False): "device", (False, True): "exact", (True, True): "device+exact"}.get((dev, exact))
    return out, route or "unknown %s" % sorted(names)


def same(got, want):
    (p, s, a), (pr, sr, ar) = got, want
    assert np.array_equal(s, sr, equal_nan=True), (s, sr)
    assert np.array_equal(p, pr), np.argwhere(p != pr)[:5]
    assert np.array_equal(a, ar), np.argwhere(a != ar)[:5]


def runs(ctx):
    """host buffers; device buffers with the transitions on the device; device buffers with host transitions"""
    return (ctx.graph_transitions_viterbi, ctx.graph_transitions_viterbi_dev,
            lambda *a, **k: ctx.graph_transitions_viterbi_dev(*a, trans_on_device=False, **k))


def check_all_buffers(ctx, e, graphs, lens, k, tw, route, weights=None):
    want = gtv.ref_graph_trans_viterbi(e, graphs, k, tw, lens, weights)
    for f in runs(ctx):
        got, taken = routed(ctx, lambda: f(e, views_of(graphs), tw, kind=k, input_lens=lens, arc_weights=weights))
        same(got, want)
        if route is not None:
            assert taken == route, (taken, route)
    return want


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("C", [4, 28, 29, 64, 128])
@pytest.mark.parametrize("implicit", [1, 0])
def test_parity_both_routes_host_and_device(ref, ctx, kind, C, implicit):
    """CTC graphs and random cyclic graphs (several start and accept nodes, start nodes with in-arcs, labels >= C)"""
    k = KINDS[kind]
    e, graphs, lens = batch(C, seed=C + implicit + 7 * k, kinds=("ctc", "rand"))
    tw = transitions(np.random.default_rng(C), C, k)
    ctx.set_flag("implicit", implicit)
    try:
        check_all_buffers(ctx, e, graphs, lens, k, tw, "device" if implicit else "exact")
    finally:
        ctx.set_flag("implicit", 1)


@pytest.mark.parametrize("implicit", [1, 0])
def test_golden_fixture(ctx, implicit):
    """the committed fixture (tests/golden/graph_trans_viterbi_golden.npz): decomposition, CTC, random cyclic and
    wildcard graphs, T_b in {0, 1}, infeasible and empty graphs, -inf transitions, tie-heavy integer inputs"""
    from tests.test_graph_trans_viterbi_oracle import golden_batches
    ctx.set_flag("implicit", implicit)
    try:
        for name, kind, e, graphs, lens, tw, want in golden_batches():
            for f in runs(ctx):
                same(f(e, views_of(graphs), tw, kind=KINDS[kind], input_lens=lens), want)
    finally:
        ctx.set_flag("implicit", 1)


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("C", [4, 28])
def test_device_arc_weights(ref, ctx, kind, C):
    k = KINDS[kind]
    e, graphs, lens = batch(C, seed=40 + C + k, kinds=("ctc", "rand"))
    w = np.random.default_rng(6).uniform(-2, 2, sum(len(g["src"]) for g in graphs)).astype(np.float32)
    check_all_buffers(ctx, e, graphs, lens, k, transitions(np.random.default_rng(C + 3), C, k), "device", weights=w)


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("C,route", [(4, "device"), (128, "exact")])
def test_wildcard_graphs(ref, ctx, kind, C, route):
    """a wildcard node becomes C copies with C in-arcs each: the sweep's layout holds it at C = 4, not at C = 128"""
    k = KINDS[kind]
    e, graphs, lens = batch(C, seed=C + 3 * k, kinds=("wild", "ctc"))
    check_all_buffers(ctx, e, graphs, lens, k, transitions(np.random.default_rng(C + 1), C, k), route)


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
def test_decompositions_at_c128(ctx, decompositions_c128, kind):
    graphs, C, T = decompositions_c128, 128, 24
    k = KINDS[kind]
    rng = np.random.default_rng(31)
    lens = np.asarray([24, 17, 20], np.int32)
    e = rng.uniform(-3, 3, (len(graphs), T, C)).astype(np.float32)
    for b in range(len(graphs)):
        e[b, lens[b]:] = np.nan
    _, scores, _ = check_all_buffers(ctx, e, graphs, lens, k, transitions(rng, C, k), "device")
    assert np.isfinite(scores).all()


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("C", [4, 28])
def test_ties_take_the_exact_route_and_match(ref, ctx, kind, C):
    """integer emissions, weights and transitions: many utterances tie; they alone re-run on the exact route.  With
    exact_ties off every utterance keeps the device route's path, which is one of the optimal paths"""
    k = KINDS[kind]
    e, graphs, lens = batch(C, seed=50 + C + k, kinds=("ctc", "rand", "wild"), ties=True)
    tw = transitions(np.random.default_rng(C + 5), C, k, ties=True)
    want = check_all_buffers(ctx, e, graphs, lens, k, tw, "device+exact")
    ctx.set_flag("exact_ties", 0)
    try:
        (p, s, a), taken = routed(ctx, lambda: ctx.graph_transitions_viterbi(e, views_of(graphs), tw, kind=k,
                                                                             input_lens=lens))
    finally:
        ctx.set_flag("exact_ties", 1)
    assert taken == "device", taken
    assert np.array_equal(s, want[1])
    for b in range(len(graphs)):
        n = int(lens[b])
        if np.isfinite(s[b]):
            assert gtv.path_value(e[b, :n], graphs[b], k, tw, p[b, :n], a[b, :n]) == s[b]
            assert np.array_equal(p[b, :n], graphs[b]["olabel"][a[b, :n]])


def test_a_tie_sends_only_its_utterance_to_the_exact_route(ref, ctx):
    """two parallel equal self-loops tie in one utterance; the others take the device route alone"""
    C, T, k = 6, 10, capi.DENSE_ASG
    rng = np.random.default_rng(60)
    graphs = [go.ctc_graph(rng.integers(1, C, 3)) for _ in range(3)]
    for g in graphs:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    graphs.append(go.make([1, 2], [0, 0, 1, 1], [1, 1, 1, 1], [1, 1, 2, 2]))
    e = rng.uniform(-3, 3, (4, T, C)).astype(np.float32)
    tw = transitions(rng, C, k)
    want = gtv.ref_graph_trans_viterbi(e, graphs, k, tw)
    got, taken = routed(ctx, lambda: ctx.graph_transitions_viterbi(e, views_of(graphs), tw, kind=k))
    same(got, want)
    assert taken == "device+exact", taken
    got, taken = routed(ctx, lambda: ctx.graph_transitions_viterbi(e[:3], views_of(graphs[:3]), tw, kind=k))
    same(got, tuple(x[:3] for x in want))
    assert taken == "device", taken


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("C", [4, 28])
def test_zero_transitions_equal_graph_viterbi(ctx, kind, C):
    """fl(w_a + 0) = w_a and the product adds no tie: all-zero transitions give gtnb_graph_viterbi's result"""
    k = KINDS[kind]
    e, graphs, lens = batch(C, seed=80 + C + k, kinds=("ctc", "rand", "wild"))
    tw = np.zeros((C + C * C) if k == capi.DENSE_ASG else C * C, np.float32)
    want = ctx.graph_viterbi(e, views_of(graphs), input_lens=lens)
    assert np.isfinite(want[1]).any()
    for f in runs(ctx):
        same(f(e, views_of(graphs), tw, kind=k, input_lens=lens), want)


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("C", [4, 28])
def test_free_graph_equals_viterbi_dense_ex(ctx, kind, C):
    """one start + accept node with a self-loop of every label: the dense decoder's paths and scores"""
    k = KINDS[kind]
    rng = np.random.default_rng(90 + C + k)
    B, T = 4, 20
    free = go.make([3], [0] * C, [0] * C, list(range(C)))
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    lens = np.asarray([20, 11, 1, 17], np.int32)
    tw = transitions(rng, C, k)
    pd, sd = ctx.viterbi_dense_ex(e, tw, kind=k, input_lens=lens)
    for f in runs(ctx):
        p, s, a = f(e, views_of([free] * B), tw, kind=k, input_lens=lens)
        assert np.array_equal(s, sd), (s, sd)
        assert np.array_equal(p, pd)
        assert np.array_equal(a, p)  # arc l of the free graph carries label l


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("where", ["emission_nan", "emission_inf", "w_nan", "w_neginf", "trans_neginf"])
def test_non_finite_values(ref, ctx, kind, where):
    k = KINDS[kind]
    C = 9
    e, graphs, lens = batch(C, seed=9 + k, kinds=("wild", "ctc"))
    e = np.nan_to_num(e, nan=0.0)
    tw = transitions(np.random.default_rng(19), C, k)
    if where == "emission_nan":
        e[1, 3, 2] = np.nan
    elif where == "emission_inf":
        e[2, 2, int(graphs[2]["olabel"][1])] = np.inf
    elif where == "w_nan":
        graphs[0]["w"][3] = np.nan
    elif where == "w_neginf":
        graphs[3]["w"][1] = -np.inf
    else:
        (tw[C:] if k == capi.DENSE_ASG else tw)[::5] = -np.inf
    check_all_buffers(ctx, e, graphs, lens, k, tw, None)


def test_nan_read_only_by_the_folded_start_arcs(ref, ctx):
    """BIGRAM: a NaN in W[l][j] with j no in-label of any source of an l arc is read by the folded start arcs alone,
    through tau_l: the utterance goes to the exact route and matches"""
    C, T, k = 5, 6, capi.DENSE_BIGRAM
    g = go.make([1, 0, 2], [0, 1, 1, 2], [1, 1, 2, 2], [1, 1, 2, 2])  # labels 1 then 2; in-labels {1}, {1, 2}
    g["w"] = np.asarray([0.5, -0.25, 0.125, 0.0], np.float32)
    tw = transitions(np.random.default_rng(3), C, k)
    tw[1 * C + 4] = np.nan  # W[1][4]: label 1 after label 4, only the start arc 0 -> 1 reads it
    e = np.random.default_rng(4).uniform(-3, 3, (2, T, C)).astype(np.float32)
    want = gtv.ref_graph_trans_viterbi(e, [g, g], k, tw)
    for f in runs(ctx):
        got, taken = routed(ctx, lambda: f(e, views_of([g, g]), tw, kind=k))
        same(got, want)
        assert taken in ("exact", "device+exact"), taken


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_edge_cases(ref, ctx, kind):
    k = KINDS[kind]
    C = 6
    wild = go.with_wildcards(go.ctc_graph([2, 3]), C)
    chain = go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3])  # accepts length 3 only
    empty = go.make([], [], [], [])
    no_start = go.make([0, 2], [0, 1], [1, 1], [1, 2])
    graphs = [wild, wild, chain, empty, chain, no_start]
    lens = np.asarray([0, 1, 5, 6, 3, 4], np.int32)
    e = np.random.default_rng(8).uniform(-3, 3, (6, 6, C)).astype(np.float32)
    tw = transitions(np.random.default_rng(9), C, k)
    want = gtv.ref_graph_trans_viterbi(e, graphs, k, tw, lens)
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            for f in runs(ctx):
                p, s, a = f(e, views_of(graphs), tw, kind=k, input_lens=lens)
                dead = [0, 2, 3, 5]
                assert np.isneginf(s[dead]).all() and (p[dead] == -1).all() and (a[dead] == -1).all()
                same((p, s, a), want)
        finally:
            ctx.set_flag("implicit", 1)
    p, s, a = ctx.graph_transitions_viterbi(np.zeros((0, 5, C), np.float32), [], tw, kind=k)
    assert p.shape == (0, 5) and s.shape == (0,)


def test_bad_input(ctx):
    C = 5
    g = go.ctc_graph([1, 2])
    e = np.zeros((1, 4, C), np.float32)
    tw = np.zeros(C + C * C, np.float32)
    eps = go.make([1, 2], [0], [1], [-1])
    with pytest.raises(capi.GtnbError) as ei:
        ctx.graph_transitions_viterbi(e, views_of([eps]), tw)
    assert ei.value.code == capi.ERR_UNSUPPORTED and "remove" in str(ei.value)
    with pytest.raises(capi.GtnbError) as ei:
        ctx.graph_transitions_viterbi(np.zeros((1, 4, 129), np.float32), views_of([g]),
                                      np.zeros(129 + 129 * 129, np.float32))
    assert ei.value.code == capi.ERR_UNSUPPORTED
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.graph_transitions_viterbi(e, views_of([g]), tw, kind=7)
    for lens in ([5], [-1]):
        with pytest.raises(capi.GtnbInvalidArgument):
            ctx.graph_transitions_viterbi(e, views_of([g]), tw, input_lens=lens)
    bad = go.make([1, 2], [0], [7], [1])  # arc endpoint outside the graph
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.graph_transitions_viterbi(e, views_of([bad]), tw)


def _gtn_graph(gtn, g):
    h = gtn.Graph()
    for f in g["flags"]:
        h.add_node(bool(f & 1), bool(f & 2))
    for a in range(len(g["src"])):
        h.add_arc(int(g["src"][a]), int(g["dst"][a]), int(g["ilabel"][a]), int(g["olabel"][a]), float(g["w"][a]))
    return h


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("with_weights", [False, True])
def test_torch_graph_transitions_viterbi_equals_the_c_abi(ref, ctx, kind, with_weights):
    torch = pytest.importorskip("torch")
    import gtn_b200.gtn as gtn
    from gtn_b200 import torch_loss
    C = 12
    k = KINDS[kind]
    e, graphs, lens = batch(C, seed=11, kinds=("wild", "ctc", "rand"))
    w = np.concatenate([g["w"] for g in graphs]) + 0.25 if with_weights else None
    tw = transitions(np.random.default_rng(12), C, k)
    x = torch.tensor(np.nan_to_num(e, nan=7.0), device="cuda")
    p, s, a = torch_loss.graph_transitions_viterbi(
        x, torch.tensor(tw, device="cuda"), [_gtn_graph(gtn, g) for g in graphs], kind=kind,
        input_lengths=torch.tensor(lens), weights=None if w is None else torch.tensor(w, device="cuda"))
    assert p.is_cuda and p.dtype == torch.int32 and s.dtype == torch.float32 and a.shape == p.shape
    got = (p.cpu().numpy(), s.cpu().numpy(), a.cpu().numpy())
    xe = x.cpu().numpy()
    same(got, ctx.graph_transitions_viterbi(xe, views_of(graphs), tw, kind=k, input_lens=lens, arc_weights=w))
    same(got, gtv.ref_graph_trans_viterbi(xe, graphs, k, tw, lens, w))
    labels, n = torch_loss.collapse(p, blank=0)
    assert labels.shape == p.shape and n.shape == (len(graphs),)
