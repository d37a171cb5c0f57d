"""The cluster route of the sparse-transition entry points (gtnb_ctx_set_flag "sparse_cluster": a transition graph G
beyond one CTA's shared memory swept by one thread-block cluster per utterance, k_sparse.cu's sparse_cl_* kernels) on
the GPU against the live reference: gtnb_sparse_transitions_loss, gtnb_viterbi_sparse and
gtnb_sparse_transitions_viterbi for a G of 5000 nodes / 40 000 arcs and for the full trigram at C = 64 (4096 / 262 144),
at small B and T so that the reference can materialise; the route read from the kernel profile; host and device
buffers.  With the flag at 0 a 4097-node G still takes the exact route.  With the flag at 2 / 4 / 8 a G inside the
one-CTA envelope gives the one-CTA kernels' decode and losses ==.  Ties, a non-finite value, ragged lengths with zeros,
B = 0, a bad flag value, and the torch functions with large_transitions=True on a side stream."""
import numpy as np
import pytest

from gtn_b200 import capi
from tests import graph_oracle as go
from tests import sparse_trans_oracle as st
from tests import sparse_viterbi_oracle as sv
from tests import util
from tests.test_gpu_graph_transitions import views_of
from tests.test_gpu_sparse_transitions import check as check_loss
from tests.test_gpu_sparse_viterbi import _gtn_graph, same, view_of

pytestmark = pytest.mark.gpu

CLUSTER_LOSS = {"sparse_cl_den_forward", "sparse_cl_den_backward", "product_fold"}
CLUSTER_DECODE = {"sparse_cl_viterbi_forward", "sparse_viterbi_trace"}
ONE_CTA = {"sparse_den_forward", "sparse_den_backward", "sparse_viterbi_forward"}


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


@pytest.fixture
def flag(ctx):
    """set(v): the "sparse_cluster" flag for the test, back to 0 after it"""
    yield lambda v: ctx.set_flag("sparse_cluster", v)
    ctx.set_flag("sparse_cluster", 0)


def profiled(ctx, run):
    """run() -> (its result, the names of the kernels it launched)"""
    ctx.profile(True)
    ctx.profile_read()
    try:
        out = run()
        return out, set(ctx.profile_read())
    finally:
        ctx.profile(False)


def big_graphs():
    """(name, C, G): 5000 nodes / 40 000 arcs (a cluster of 2), the full trigram at C = 64 (a cluster of 8)"""
    rng = np.random.default_rng(5)
    return [("sparse5000", 32, st.sparse_graph(rng, 5000, 40000, 32, n_start=40, n_accept=2500, n_unreachable=0)),
            ("trigram64", 64, st.trigram_graph(64))]


def walk(rng, G, n):
    """the labels of a random path of n arcs through G from a start node to an accept node"""
    order = np.argsort(G["src"], kind="stable")
    first = np.searchsorted(G["src"][order], np.arange(len(G["flags"]) + 1))
    while True:
        v, labels = int(rng.choice(np.flatnonzero(G["flags"] & 1))), []
        while len(labels) < n and first[v] < first[v + 1]:
            a = order[rng.integers(first[v], first[v + 1])]
            labels.append(int(G["olabel"][a]))
            v = int(G["dst"][a])
        if len(labels) == n and G["flags"][v] & 2:
            return labels


def inputs(rng, B, T, C, G):
    """ragged lengths with a zero; every target graph the chain of a path of T_b arcs through G, so that A_b o G is
    small and accepts whatever G's shape"""
    lens = np.asarray([T, T - 1, 0, T - 2][:B], np.int32)
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    graphs = []
    for n in lens:
        labels = walk(rng, G, max(int(n), 1))
        k = len(labels)
        graphs.append(go.make([1] + [0] * (k - 1) + [2], np.arange(k), np.arange(1, k + 1), labels))
    for g in graphs:
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
    return e, lens, graphs, rng.uniform(-1, 1, len(G["src"])).astype(np.float32)


def test_flag_0_keeps_the_exact_route_beyond_one_cta(ref, ctx):
    rng = np.random.default_rng(1)
    C = 16
    G = st.sparse_graph(rng, 4097, 12000, C, n_start=64, n_accept=512, n_unreachable=0)
    e, lens, graphs, tw = inputs(rng, 2, 5, C, G)
    got, names = profiled(ctx, lambda: ctx.viterbi_sparse(e, view_of(G), tw, input_lens=lens))
    same(got, sv.ref_sparse_viterbi(e, G, tw, lens))
    assert "compose_emit" in names and not names & (CLUSTER_DECODE - {"sparse_viterbi_trace"}) and not names & ONE_CTA
    _, names = profiled(ctx, lambda: ctx.sparse_transitions_loss(e, views_of(graphs), view_of(G), tw, input_lens=lens))
    assert "compose_emit" in names and not names & CLUSTER_LOSS and not names & ONE_CTA


@pytest.mark.parametrize("which", [0, 1])
def test_flag_1_loss_decode_and_alignment_match_the_reference(ref, ctx, flag, which):
    name, C, G = big_graphs()[which]
    rng = np.random.default_rng(10 + which)
    B, T = 4, 5
    e, lens, graphs, tw = inputs(rng, B, T, C, G)
    flag(1)
    want = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
    assert np.isfinite(want[0][[0, 1, 3]]).all()
    for run in (ctx.sparse_transitions_loss, ctx.sparse_transitions_loss_dev):
        got, names = profiled(ctx, lambda: run(e, views_of(graphs), view_of(G), tw, input_lens=lens))
        assert CLUSTER_LOSS <= names and "compose_emit" not in names and not names & ONE_CTA, sorted(names)
        fin = np.isfinite(want[0])
        assert np.allclose(got[0][fin], want[0][fin], rtol=1e-4, atol=0) and np.isnan(got[0][2])
        check_loss(got, want, T)
    want = sv.ref_sparse_viterbi(e, G, tw, lens)
    for run in (ctx.viterbi_sparse, ctx.viterbi_sparse_dev):
        got, names = profiled(ctx, lambda: run(e, view_of(G), tw, input_lens=lens))
        assert CLUSTER_DECODE <= names and "compose_emit" not in names and not names & ONE_CTA, sorted(names)
        same(got, want)
    want = sv.ref_sparse_trans_viterbi(e, graphs, G, tw, lens)
    for run in (ctx.sparse_transitions_viterbi, ctx.sparse_transitions_viterbi_dev):
        got, names = profiled(ctx, lambda: run(e, views_of(graphs), view_of(G), tw, input_lens=lens))
        assert {"implicit_trace", "sparse_tau"} <= names and "compose_emit" not in names, sorted(names)
        same(got, want)


@pytest.mark.parametrize("graph", ["trigram30", "sparse2000"])
def test_forced_cluster_sizes_reproduce_the_one_cta_kernels(ctx, flag, graph):
    rng = np.random.default_rng(20)
    C = 30
    G = st.trigram_graph(C) if graph == "trigram30" else st.sparse_graph(rng, 2000, 32000, C, n_start=20,
                                                                         n_accept=200, n_unreachable=0)
    B, T = 6, 40
    tw = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    lens = np.asarray([T, T - 7, 1, 0, T - 1, T // 2], np.int32)
    graphs = [go.ctc_graph(rng.integers(1, C, 4)) for _ in range(B)]
    dec0, names = profiled(ctx, lambda: ctx.viterbi_sparse(e, view_of(G), tw, input_lens=lens))
    assert "sparse_viterbi_forward" in names
    loss0 = ctx.sparse_transitions_loss_dev(e, views_of(graphs), view_of(G), tw, input_lens=lens)
    for N in (2, 4, 8):
        flag(N)
        dec, names = profiled(ctx, lambda: ctx.viterbi_sparse(e, view_of(G), tw, input_lens=lens))
        assert CLUSTER_DECODE <= names and "sparse_viterbi_forward" not in names
        same(dec, dec0)
        loss, names = profiled(ctx, lambda: ctx.sparse_transitions_loss_dev(e, views_of(graphs), view_of(G), tw,
                                                                            input_lens=lens))
        assert CLUSTER_LOSS <= names and not names & ONE_CTA
        assert np.array_equal(loss[0], loss0[0], equal_nan=True)
        for x, y in zip(loss[1:], loss0[1:]):
            assert util.close(x, y)


def test_ties_and_a_non_finite_value_are_retried_on_the_exact_route(ref, ctx, flag):
    """integer emissions and zero weights on the 5000-node G: tied utterances re-run alone on the exact route, and
    with exact_ties off keep the cluster kernels' path; an utterance with a NaN emission is retried too"""
    _, C, G = big_graphs()[0]
    rng = np.random.default_rng(30)
    B, T = 3, 4
    e = rng.integers(0, 2, (B, T, C)).astype(np.float32)
    lens = np.asarray([T, T, 2], np.int32)
    tw = np.zeros(len(G["src"]), np.float32)
    flag(1)
    want = sv.ref_sparse_viterbi(e, G, tw, lens)
    assert any(sv.decode_outcome(e[b, :lens[b]], G, tw, C)[1] for b in range(B))
    got, names = profiled(ctx, lambda: ctx.viterbi_sparse(e, view_of(G), tw, input_lens=lens))
    same(got, want)
    assert CLUSTER_DECODE <= names and "compose_emit" in names
    ctx.set_flag("exact_ties", 0)
    try:
        (p, s, a), names = profiled(ctx, lambda: ctx.viterbi_sparse(e, view_of(G), tw, input_lens=lens))
    finally:
        ctx.set_flag("exact_ties", 1)
    assert CLUSTER_DECODE <= names and "compose_emit" not in names
    assert np.array_equal(s, want[1])
    for b in range(B):
        assert sv.is_path(G, a[b, :lens[b]]) and sv.path_value(e[b, :lens[b]], G, tw, a[b, :lens[b]]) == s[b]
    e2 = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    tw2 = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e2[1, 1, :] = np.nan
    got, names = profiled(ctx, lambda: ctx.viterbi_sparse(e2, view_of(G), tw2, input_lens=lens))
    same(got, sv.ref_sparse_viterbi(e2, G, tw2, lens))
    assert CLUSTER_DECODE <= names and "compose_emit" in names
    _, _, graphs, _ = inputs(rng, B, T, C, G)
    got, names = profiled(ctx, lambda: ctx.sparse_transitions_loss(e2, views_of(graphs), view_of(G), tw2,
                                                                   input_lens=lens))
    want = st.ref_sparse_trans_loss(e2, graphs, G, tw2, lens)
    assert "sparse_cl_den_forward" in names and "compose_emit" in names
    assert util.close(got[0], want[0])


def test_empty_batch_and_bad_flag_values(ctx, flag):
    _, C, G = big_graphs()[0]
    tw = np.zeros(len(G["src"]), np.float32)
    flag(1)
    p, s, a = ctx.viterbi_sparse(np.zeros((0, 5, C), np.float32), view_of(G), tw)
    assert p.shape == (0, 5) and s.shape == (0,)
    assert not ctx.sparse_transitions_loss(np.zeros((0, 3, C), np.float32), [], view_of(G), tw)[3].any()
    for bad in (-1, 3, 5, 16):
        with pytest.raises(capi.GtnbInvalidArgument):
            ctx.set_flag("sparse_cluster", bad)
    p, s, a = ctx.viterbi_sparse(np.zeros((2, 3, C), np.float32), view_of(G), tw, input_lens=[0, 0])
    assert np.isneginf(s).all() and (p == -1).all()  # (the flag is still 1: a refused value changes nothing)


def test_torch_functions_with_large_transitions_on_a_side_stream(ref, ctx):
    torch = pytest.importorskip("torch")
    import gtn_b200.gtn as gtn
    from gtn_b200 import torch_loss
    _, C, G = big_graphs()[0]
    rng = np.random.default_rng(40)
    B, T = 2, 5
    e, lens, graphs, tw = inputs(rng, B, T, C, G)
    Gg, gg = _gtn_graph(gtn, G), [_gtn_graph(gtn, g) for g in graphs]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        x = torch.tensor(e, device="cuda", requires_grad=True)
        tr = torch.tensor(tw, device="cuda", requires_grad=True)
        il = torch.tensor(lens)
        out = torch_loss.sparse_transitions_loss(x, tr, Gg, gg, input_lengths=il, reduction="mean",
                                                 large_transitions=True)
        out.backward()
        dec = torch_loss.sparse_viterbi(x.detach(), tr.detach(), Gg, input_lengths=il, large_transitions=True)
        ali = torch_loss.sparse_transitions_viterbi(x.detach(), tr.detach(), Gg, gg, input_lengths=il,
                                                    large_transitions=True)
    side.synchronize()
    for g in graphs:
        g["w"] = np.zeros(len(g["src"]), np.float32)  # _gtn_graph builds the graphs with zero weights
    lr, gr, _, tgr = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
    assert util.close(out.item(), lr.mean())
    assert util.grad_close(x.grad.cpu().numpy(), gr / B, 50.0)
    assert util.grad_close(tr.grad.cpu().numpy(), tgr / B, 50.0 * B)
    same(tuple(t.cpu().numpy() for t in dec), sv.ref_sparse_viterbi(e, G, tw, lens))
    same(tuple(t.cpu().numpy() for t in ali), sv.ref_sparse_trans_viterbi(e, graphs, G, tw, lens))
    # without the keyword the same G takes the materialised route and gives the same losses
    with torch.cuda.stream(side):
        plain = torch_loss.sparse_transitions_loss(x.detach(), tr.detach(), Gg, gg, input_lengths=il)
    side.synchronize()
    assert util.close(plain.item(), lr.mean())
