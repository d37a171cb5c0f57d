"""gtnb_viterbi_sparse (Viterbi decoding with a learned transition graph G of any shape) on the GPU against the live
reference (tests/sparse_viterbi_oracle.py), utterance by utterance on its own T_b rows: paths, G's arcs and scores ==,
with the route each call took read from the kernel profile.  Random sparse cyclic G (several start and accept nodes,
unreachable nodes, labels >= C) at C in {4, 28, 30, 64, 128} on both routes; host and device buffers, transitions on
the host and on the device; the trigram at C = 30 on the device route; G at the envelope's edge and beyond it;
tie-heavy inputs, whose tied utterances alone re-run on the exact route; exact_ties off; non-finite values; the
identities with gtnb_viterbi_dense_ex (the bigram and ASG graphs) and with a per-frame argmax (the free graph);
edge cases and bad input; and torch_loss.sparse_viterbi against the C ABI on a side stream."""
import numpy as np
import pytest

from gtn_b200 import capi
from tests import graph_oracle as go
from tests import sparse_trans_oracle as st
from tests import sparse_viterbi_oracle as sv

pytestmark = pytest.mark.gpu

DEVICE = {"sparse_viterbi_forward", "sparse_viterbi_trace"}
EXACT = {"compose_emit"}


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


def view_of(G):
    return capi.make_view(G["flags"], G["src"], G["dst"], G["olabel"], G["olabel"], None)


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
    return (ctx.viterbi_sparse, ctx.viterbi_sparse_dev,
            lambda *a, **k: ctx.viterbi_sparse_dev(*a, trans_on_device=False, **k))


def check_all_buffers(ctx, e, G, tw, lens, route):
    want = sv.ref_sparse_viterbi(e, G, tw, lens)
    for f in runs(ctx):
        got, taken = routed(ctx, lambda: f(e, view_of(G), tw, input_lens=lens))
        same(got, want)
        if route is not None:
            assert taken == route, (taken, route)
    return want


def inputs(rng, B, T, C, ties=False):
    lens = rng.integers(T // 2, T + 1, B).astype(np.int32)
    lens[0] = T
    e = (rng.integers(0, 2, (B, T, C)) if ties else rng.uniform(-3, 3, (B, T, C))).astype(np.float32)
    for b in range(B):
        e[b, lens[b]:] = np.nan
    return e, lens


def weights(rng, G, ties=False):
    n = len(G["src"])
    return (np.zeros(n) if ties else rng.uniform(-1, 1, n)).astype(np.float32)


@pytest.mark.parametrize("C", [4, 28, 30, 64, 128])
@pytest.mark.parametrize("implicit", [1, 0])
def test_parity_both_routes_host_and_device(ref, ctx, C, implicit):
    rng = np.random.default_rng(C + 100 * implicit)
    G = st.sparse_graph(rng, 12, 70, C, n_start=3, n_accept=3, label_hi=C + 2)
    e, lens = inputs(rng, 6, 15, C)
    ctx.set_flag("implicit", implicit)
    try:
        _, s, _ = check_all_buffers(ctx, e, G, weights(rng, G), lens, "device" if implicit else "exact")
    finally:
        ctx.set_flag("implicit", 1)
    assert np.isfinite(s).any()


def test_trigram_c30_device_route(ref, ctx):
    C = 30
    rng = np.random.default_rng(3)
    G = st.trigram_graph(C)
    e, lens = inputs(rng, 4, 20, C)
    _, s, _ = check_all_buffers(ctx, e, G, weights(rng, G), lens, "device")
    assert np.isfinite(s).all()


def test_envelope_edge_and_beyond(ref, ctx):
    """4096 nodes and 32768 arcs take the device route; 4097 nodes the exact route, at small B * T"""
    rng = np.random.default_rng(4)
    C = 64
    G = st.sparse_graph(rng, 4096, 32768, C, n_start=64, n_accept=512, n_unreachable=0)
    e, lens = inputs(rng, 2, 6, C)
    check_all_buffers(ctx, e, G, weights(rng, G), lens, "device")
    G2 = st.sparse_graph(rng, 4097, 20000, C, n_start=64, n_accept=512, n_unreachable=0)
    check_all_buffers(ctx, e, G2, weights(rng, G2), lens, "exact")


@pytest.mark.parametrize("C", [4, 30])
def test_ties_take_the_exact_route_and_match(ref, ctx, C):
    """zero-initialised transitions and integer emissions: many utterances tie, and they alone re-run on the exact
    route (the restatement predicts which).  With exact_ties off every utterance keeps the device route's path, one
    of the optimal paths"""
    rng = np.random.default_rng(50 + C)
    G = st.trigram_graph(C) if C == 4 else st.sparse_graph(rng, 10, 60, C, n_start=3, n_accept=3)
    tw = weights(rng, G, ties=True)
    e, lens = inputs(rng, 6, 8, C, ties=True)
    assert any(sv.decode_outcome(e[b, :lens[b]], G, tw, C)[1] for b in range(6))
    want = check_all_buffers(ctx, e, G, tw, lens, "device+exact")
    ctx.set_flag("exact_ties", 0)
    try:
        (p, s, a), taken = routed(ctx, lambda: ctx.viterbi_sparse(e, view_of(G), tw, input_lens=lens))
    finally:
        ctx.set_flag("exact_ties", 1)
    assert taken == "device", taken
    assert np.array_equal(s, want[1])
    for b in range(6):
        n = int(lens[b])
        if np.isfinite(s[b]):
            assert sv.is_path(G, a[b, :n])
            assert sv.path_value(e[b, :n], G, tw, a[b, :n]) == s[b]
            assert np.array_equal(p[b, :n], G["olabel"][a[b, :n]])


def test_a_tie_sends_only_its_utterance_to_the_exact_route(ref, ctx):
    """two equal parallel self-loops with label L on a start and accept node: the utterance whose emissions favour L
    ties at every frame; the others, where L is forbidden, take the device route alone"""
    C, T, L = 6, 10, 5
    rng = np.random.default_rng(60)
    g = st.sparse_graph(rng, 9, 50, C - 1, n_start=2, n_accept=2, n_unreachable=0)
    flags = g["flags"].copy()
    flags[0] |= 3
    G = go.make(flags, np.r_[g["src"], 0, 0], np.r_[g["dst"], 0, 0], np.r_[g["olabel"], L, L])
    tw = weights(rng, G)
    tw[-2:] = 0.25
    e, lens = inputs(rng, 4, T, C)
    e = np.nan_to_num(e, nan=0.0)
    e[:3, :, L] = -np.inf
    e[3, :, L] = 20.0
    want = sv.ref_sparse_viterbi(e, G, tw, lens)
    assert [sv.decode_outcome(e[b, :lens[b]], G, tw, C)[1] for b in range(4)] == [False, False, False, True]
    got, taken = routed(ctx, lambda: ctx.viterbi_sparse(e, view_of(G), tw, input_lens=lens))
    same(got, want)
    assert taken == "device+exact", taken
    got, taken = routed(ctx, lambda: ctx.viterbi_sparse(e[:3], view_of(G), tw, input_lens=lens[:3]))
    same(got, tuple(x[:3] for x in want))
    assert taken == "device", taken


def test_neginf_weights_stay_on_the_device_route(ref, ctx):
    C = 8
    rng = np.random.default_rng(70)
    G = st.sparse_graph(rng, 10, 60, C)
    tw = weights(rng, G)
    tw[::4] = -np.inf
    e, lens = inputs(rng, 5, 12, C)
    e[2, 3, 1] = -np.inf
    check_all_buffers(ctx, e, G, tw, lens, "device")


@pytest.mark.parametrize("where", ["emission_nan", "emission_inf", "w_nan", "w_inf"])
def test_nan_and_inf_take_the_exact_route(ref, ctx, where):
    C = 7
    rng = np.random.default_rng(80)
    G = st.sparse_graph(rng, 8, 40, C)
    tw = weights(rng, G)
    e, lens = inputs(rng, 4, 9, C)
    e = np.nan_to_num(e, nan=0.0)
    if where == "emission_nan":
        e[1, 3, :] = np.nan
    elif where == "emission_inf":
        e[2, 2, :] = np.inf
    elif where == "w_nan":
        tw[np.flatnonzero(G["olabel"] < C)[::3]] = np.nan
    else:
        tw[np.flatnonzero(G["olabel"] < C)[::3]] = np.inf
    want = sv.ref_sparse_viterbi(e, G, tw, lens)
    for f in runs(ctx):
        got, taken = routed(ctx, lambda: f(e, view_of(G), tw, input_lens=lens))
        same(got, want)
        assert taken in ("exact", "device+exact"), taken


@pytest.mark.parametrize("C", [4, 28])
def test_bigram_graph_equals_viterbi_dense_ex(ctx, C):
    """bigram_graph(C) with weights permuted by bigram_slots is gtnb_viterbi_dense_ex BIGRAM's G"""
    rng = np.random.default_rng(90 + C)
    W = rng.uniform(-1, 1, C * C).astype(np.float32)
    G = st.bigram_graph(C)
    e, lens = inputs(rng, 5, 16, C)
    e = np.nan_to_num(e, nan=0.0)
    pd, sd = ctx.viterbi_dense_ex(e, W, kind=capi.DENSE_BIGRAM, input_lens=lens)
    for f in runs(ctx):
        p, s, a = f(e, view_of(G), W[st.bigram_slots(C)], input_lens=lens)
        assert np.array_equal(s, sd), (s, sd)
        assert np.array_equal(p, pd)


@pytest.mark.parametrize("C", [4, 28])
def test_asg_graph_equals_viterbi_dense_ex(ctx, C):
    rng = np.random.default_rng(95 + C)
    W = rng.uniform(-1, 1, C + C * C).astype(np.float32)
    G = st.asg_graph(C)
    e, lens = inputs(rng, 5, 16, C)
    e = np.nan_to_num(e, nan=0.0)
    pd, sd = ctx.viterbi_dense_ex(e, W, kind=capi.DENSE_ASG, input_lens=lens)
    for f in runs(ctx):
        p, s, a = f(e, view_of(G), W, input_lens=lens)
        assert np.array_equal(s, sd), (s, sd)
        assert np.array_equal(p, pd)


def test_free_graph_is_a_per_frame_argmax(ctx):
    C, T = 9, 12
    rng = np.random.default_rng(11)
    G = go.make([3], [0] * C, [0] * C, list(range(C)))
    e, lens = inputs(rng, 4, T, C)
    e = np.nan_to_num(e, nan=0.0)
    p, s, a = ctx.viterbi_sparse(e, view_of(G), np.zeros(C, np.float32), input_lens=lens)
    for b in range(4):
        n = int(lens[b])
        assert np.array_equal(p[b, :n], e[b, :n].argmax(axis=1)) and (p[b, n:] == -1).all()
        assert np.array_equal(a[b], p[b])
        want = np.float32(0.0)
        for t in range(n):
            want = np.float32(want + e[b, t].max())
        assert s[b] == want


def test_edge_cases(ref, ctx):
    """T_b in {0, 1}; a G that accepts nothing in T_b frames; a G with no arc labelled in [0, C); B = 0"""
    C = 5
    rng = np.random.default_rng(12)
    chain = go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3])  # accepts length 3 only
    e, _ = inputs(rng, 4, 6, C)
    lens = np.asarray([0, 1, 3, 6], np.int32)
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            for f in runs(ctx):
                p, s, a = f(e, view_of(chain), np.asarray([0.5, -1, 2], np.float32), input_lens=lens)
                assert np.isneginf(s[[0, 1, 3]]).all() and (p[[0, 1, 3]] == -1).all() and (a[[0, 1, 3]] == -1).all()
                same((p, s, a), sv.ref_sparse_viterbi(e, chain, [0.5, -1, 2], lens))
                assert np.array_equal(a[2, :3], [0, 1, 2])
            high = go.make([3], [0], [0], [C + 1])
            p, s, a = ctx.viterbi_sparse(e, view_of(high), np.zeros(1, np.float32), input_lens=lens)
            assert np.isneginf(s).all() and (p == -1).all() and (a == -1).all()
        finally:
            ctx.set_flag("implicit", 1)
    p, s, a = ctx.viterbi_sparse(np.zeros((0, 5, C), np.float32), view_of(chain), np.zeros(3, np.float32))
    assert p.shape == (0, 5) and s.shape == (0,)


def test_bad_input(ctx):
    C = 5
    G = st.sparse_graph(np.random.default_rng(1), 4, 10, C)
    tw = np.zeros(len(G["src"]), np.float32)
    e = np.zeros((2, 4, C), np.float32)
    eps = go.make([1, 2], [0], [1], [-1])
    with pytest.raises(capi.GtnbError) as ei:
        ctx.viterbi_sparse(e, view_of(eps), np.zeros(1, np.float32))
    assert ei.value.code == capi.ERR_UNSUPPORTED and "remove" in str(ei.value)
    transducer = capi.make_view([1, 2], [0], [1], [1], [2], None)
    with pytest.raises(capi.GtnbError) as ei:
        ctx.viterbi_sparse(e, transducer, np.zeros(1, np.float32))
    assert ei.value.code == capi.ERR_UNSUPPORTED
    for lens in ([5, 1], [-1, 1]):
        with pytest.raises(capi.GtnbInvalidArgument):
            ctx.viterbi_sparse(e, view_of(G), tw, input_lens=lens)
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.viterbi_sparse(e, view_of(G), None)
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.viterbi_sparse(e, view_of(go.make([], [], [], [])), np.zeros(0, np.float32))
    bad = go.make([1, 2], [0], [7], [1])  # arc endpoint outside the graph
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.viterbi_sparse(e, view_of(bad), np.zeros(1, np.float32))


def _gtn_graph(gtn, g):
    h = gtn.Graph()
    for f in g["flags"]:
        h.add_node(bool(f & 1), bool(f & 2))
    for a in range(len(g["src"])):
        h.add_arc(int(g["src"][a]), int(g["dst"][a]), int(g["olabel"][a]), int(g["olabel"][a]), 0.0)
    return h


def test_torch_sparse_viterbi_equals_the_c_abi_on_a_side_stream(ref, ctx):
    torch = pytest.importorskip("torch")
    import gtn_b200.gtn as gtn
    from gtn_b200 import torch_loss
    C = 12
    rng = np.random.default_rng(13)
    G = st.sparse_graph(rng, 10, 60, C, label_hi=C + 1)
    tw = weights(rng, G)
    e, lens = inputs(rng, 5, 11, C)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        x = torch.tensor(np.nan_to_num(e, nan=7.0), device="cuda")
        p, s, a = torch_loss.sparse_viterbi(x, torch.tensor(tw, device="cuda"), _gtn_graph(gtn, G),
                                            input_lengths=torch.tensor(lens))
        labels, n = torch_loss.collapse(p, blank=0)
    side.synchronize()
    assert p.is_cuda and p.dtype == torch.int32 and s.dtype == torch.float32 and a.shape == p.shape
    got = (p.cpu().numpy(), s.cpu().numpy(), a.cpu().numpy())
    xe = x.cpu().numpy()
    same(got, ctx.viterbi_sparse(xe, view_of(G), tw, input_lens=lens))
    same(got, sv.ref_sparse_viterbi(xe, G, tw, lens))
    assert labels.shape == p.shape and n.shape == (5,)
