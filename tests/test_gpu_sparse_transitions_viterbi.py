"""gtnb_sparse_transitions_viterbi (Viterbi alignment over user-supplied target graphs with a learned transition graph
G of any shape) on the GPU against the live reference (tests/sparse_viterbi_oracle.py), utterance by utterance on its
own T_b rows: paths, A_b's arcs and scores ==, with the route each call took read from the kernel profile.  Random
sparse G at C in {4, 28, 30, 64, 128} on both routes; host and device buffers, transitions on the host and on the
device; the trigram at C = 30 on the device route; tie-heavy inputs; non-finite values; the identities with
gtnb_graph_transitions_viterbi (the bigram and ASG graphs) and gtnb_graph_viterbi (the free graph); edge cases and bad
input; and torch_loss.sparse_transitions_viterbi against the C ABI."""
import numpy as np
import pytest

from gtn_b200 import capi
from tests import graph_oracle as go
from tests import sparse_trans_oracle as st
from tests import sparse_viterbi_oracle as sv
from tests.test_gpu_graph_transitions_viterbi import batch, same, views_of
from tests.test_gpu_sparse_viterbi import _gtn_graph, view_of, weights

pytestmark = pytest.mark.gpu

DEVICE = {"implicit_trace", "sparse_tau"}  # (the forward is implicit_forward_max or _arc_max)
EXACT = {"gcompose_search", "compose_emit"}


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


def runs(ctx):
    return (ctx.sparse_transitions_viterbi, ctx.sparse_transitions_viterbi_dev,
            lambda *a, **k: ctx.sparse_transitions_viterbi_dev(*a, trans_on_device=False, **k))


def check_all_buffers(ctx, e, graphs, lens, G, tw, route, arc_weights=None):
    want = sv.ref_sparse_trans_viterbi(e, graphs, G, tw, lens, arc_weights)
    for f in runs(ctx):
        ctx.profile(True)
        ctx.profile_read()
        try:
            got = f(e, views_of(graphs), view_of(G), tw, input_lens=lens, arc_weights=arc_weights)
            names = set(ctx.profile_read())
        finally:
            ctx.profile(False)
        same(got, want)
        if route is not None:
            dev, exact = DEVICE <= names, EXACT <= names
            taken = {(True, False): "device", (False, True): "exact", (True, True): "device+exact"}.get((dev, exact))
            assert taken == route, (taken, route, sorted(names))
    return want


@pytest.mark.parametrize("C", [4, 28, 30, 64, 128])
@pytest.mark.parametrize("implicit", [1, 0])
def test_parity_both_routes_host_and_device(ref, ctx, C, implicit):
    rng = np.random.default_rng(C + 7 * implicit)
    e, graphs, lens = batch(C, seed=C + implicit, kinds=("ctc", "rand"))
    G = st.sparse_graph(rng, 6, 30, C, n_start=2, n_accept=3, label_hi=C + 1)
    ctx.set_flag("implicit", implicit)
    try:
        check_all_buffers(ctx, e, graphs, lens, G, weights(rng, G), "device" if implicit else "exact")
    finally:
        ctx.set_flag("implicit", 1)


def test_trigram_c30_device_route(ref, ctx):
    C = 30
    rng = np.random.default_rng(31)
    e, graphs, lens = batch(C, seed=31, kinds=("ctc",))
    G = st.trigram_graph(C)
    w = rng.uniform(-2, 2, sum(len(g["src"]) for g in graphs)).astype(np.float32)
    _, s, _ = check_all_buffers(ctx, e, graphs, lens, G, weights(rng, G), "device", arc_weights=w)
    assert np.isfinite(s).all()


@pytest.mark.parametrize("C", [4, 28])
def test_ties_take_the_exact_route_and_match(ref, ctx, C):
    """integer emissions and weights, zero transitions: the tied utterances re-run on the exact route (device+exact),
    and the others alone take the device route.  With exact_ties off every utterance keeps the device route's path,
    one of the optimal paths"""
    rng = np.random.default_rng(50 + C)
    e, graphs, lens = batch(C, seed=50 + C, kinds=("ctc", "rand"), ties=True)
    G = st.bigram_graph(C)  # every state starts and accepts: every path of A_b has a product path
    tw = weights(rng, G, ties=True)
    e[0, :lens[0]] = 0.0  # with zero weights, every alignment of the CTC graph scores 0: a tie for certain
    graphs[0]["w"][:] = 0.0
    want = check_all_buffers(ctx, e, graphs, lens, G, tw, "device+exact")
    ctx.set_flag("exact_ties", 0)
    try:
        p, s, a = ctx.sparse_transitions_viterbi(e, views_of(graphs), view_of(G), tw, input_lens=lens)
    finally:
        ctx.set_flag("exact_ties", 1)
    assert np.array_equal(s, want[1])
    for b in range(len(graphs)):
        n = int(lens[b])
        if np.isfinite(s[b]):
            assert np.array_equal(p[b, :n], graphs[b]["olabel"][a[b, :n]])
    # a tie-free subset of the batch: random emissions for the first half, which then take the device route alone
    e2 = np.nan_to_num(e[:2], nan=0.0) + rng.uniform(-0.5, 0.5, e[:2].shape).astype(np.float32)
    tw2 = weights(rng, G)
    for g in graphs[:2]:
        g["w"] = g["w"] + rng.uniform(-0.5, 0.5, len(g["w"])).astype(np.float32)
    check_all_buffers(ctx, e2, graphs[:2], lens[:2], G, tw2, "device")


def test_beyond_the_envelope_takes_the_exact_route(ref, ctx):
    """a G of 4097 states is outside the kernels' envelope: the whole batch takes the exact route, at small B * T"""
    C = 16
    rng = np.random.default_rng(41)
    e, graphs, lens = batch(C, seed=41, kinds=("ctc", "rand"), T=6)
    G = st.sparse_graph(rng, 4097, 12000, C, n_start=64, n_accept=512, n_unreachable=0)
    check_all_buffers(ctx, e, graphs, lens, G, weights(rng, G), "exact")


@pytest.mark.parametrize("where", ["emission_nan", "w_nan", "trans_nan", "trans_neginf"])
def test_non_finite_values(ref, ctx, where):
    C = 9
    rng = np.random.default_rng(9)
    e, graphs, lens = batch(C, seed=9, kinds=("wild", "ctc"))
    e = np.nan_to_num(e, nan=0.0)
    G = st.sparse_graph(rng, 5, 30, C, n_start=2, n_accept=2)
    tw = weights(rng, G)
    if where == "emission_nan":
        e[1, 3, 2] = np.nan
    elif where == "w_nan":
        graphs[0]["w"][3] = np.nan
    elif where == "trans_nan":
        tw[::7] = np.nan
    else:
        tw[::5] = -np.inf
    check_all_buffers(ctx, e, graphs, lens, G, tw, None)


@pytest.mark.parametrize("C", [4, 28])
def test_bigram_and_asg_graphs_equal_graph_transitions_viterbi(ctx, C):
    rng = np.random.default_rng(90 + C)
    e, graphs, lens = batch(C, seed=90 + C, kinds=("ctc", "rand"))
    W = rng.uniform(-1, 1, C * C).astype(np.float32)
    want = ctx.graph_transitions_viterbi(e, views_of(graphs), W, kind=capi.DENSE_BIGRAM, input_lens=lens)
    for f in runs(ctx):
        same(f(e, views_of(graphs), view_of(st.bigram_graph(C)), W[st.bigram_slots(C)], input_lens=lens), want)
    Wa = rng.uniform(-1, 1, C + C * C).astype(np.float32)
    want = ctx.graph_transitions_viterbi(e, views_of(graphs), Wa, kind=capi.DENSE_ASG, input_lens=lens)
    for f in runs(ctx):
        same(f(e, views_of(graphs), view_of(st.asg_graph(C)), Wa, input_lens=lens), want)


def test_free_graph_equals_graph_viterbi(ctx):
    C = 12
    e, graphs, lens = batch(C, seed=7, kinds=("ctc", "rand", "wild"))
    G = go.make([3], [0] * C, [0] * C, list(range(C)))
    want = ctx.graph_viterbi(e, views_of(graphs), input_lens=lens)
    for f in runs(ctx):
        same(f(e, views_of(graphs), view_of(G), np.zeros(C, np.float32), input_lens=lens), want)


def test_edge_cases_and_bad_input(ref, ctx):
    C = 6
    rng = np.random.default_rng(8)
    wild = go.with_wildcards(go.ctc_graph([2, 3]), C)
    chain = go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3])
    empty = go.make([], [], [], [])
    graphs = [wild, wild, chain, empty, chain]
    lens = np.asarray([0, 1, 5, 6, 3], np.int32)
    e = rng.uniform(-3, 3, (5, 6, C)).astype(np.float32)
    G = st.sparse_graph(rng, 5, 30, C, n_start=2, n_accept=2)
    tw = weights(rng, G)
    want = sv.ref_sparse_trans_viterbi(e, graphs, G, tw, lens)
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            for f in runs(ctx):
                same(f(e, views_of(graphs), view_of(G), tw, input_lens=lens), want)
        finally:
            ctx.set_flag("implicit", 1)
    p, s, a = ctx.sparse_transitions_viterbi(np.zeros((0, 5, C), np.float32), [], view_of(G), tw)
    assert p.shape == (0, 5) and s.shape == (0,)
    eps = go.make([1, 2], [0], [1], [-1])
    with pytest.raises(capi.GtnbError) as ei:
        ctx.sparse_transitions_viterbi(e[:1], views_of([chain]), view_of(eps), np.zeros(1, np.float32))
    assert ei.value.code == capi.ERR_UNSUPPORTED
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.sparse_transitions_viterbi(e[:1], views_of([chain]), view_of(G), None)
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.sparse_transitions_viterbi(e[:1], views_of([chain]), view_of(G), tw, input_lens=[7])


def test_torch_sparse_transitions_viterbi_equals_the_c_abi(ref, ctx):
    torch = pytest.importorskip("torch")
    import gtn_b200.gtn as gtn
    from gtn_b200 import torch_loss
    C = 12
    rng = np.random.default_rng(13)
    e, graphs, lens = batch(C, seed=13, kinds=("wild", "ctc", "rand"))
    G = st.sparse_graph(rng, 6, 40, C)
    tw = weights(rng, G)
    x = torch.tensor(np.nan_to_num(e, nan=7.0), device="cuda")
    p, s, a = torch_loss.sparse_transitions_viterbi(
        x, torch.tensor(tw, device="cuda"), _gtn_graph(gtn, G), [_target(gtn, g) for g in graphs],
        input_lengths=torch.tensor(lens))
    assert p.is_cuda and p.dtype == torch.int32 and s.dtype == torch.float32 and a.shape == p.shape
    got = (p.cpu().numpy(), s.cpu().numpy(), a.cpu().numpy())
    xe = x.cpu().numpy()
    same(got, ctx.sparse_transitions_viterbi(xe, views_of(graphs), view_of(G), tw, input_lens=lens))
    same(got, sv.ref_sparse_trans_viterbi(xe, graphs, G, tw, lens))


def _target(gtn, g):
    h = gtn.Graph()
    for f in g["flags"]:
        h.add_node(bool(f & 1), bool(f & 2))
    for a in range(len(g["src"])):
        h.add_arc(int(g["src"][a]), int(g["dst"][a]), int(g["ilabel"][a]), int(g["olabel"][a]), float(g["w"][a]))
    return h
