"""The cluster route of the backoff entry points (gtnb_ctx_set_flag "sparse_cluster": a backoff transition graph G
beyond one CTA's shared memory, its denominator swept by one thread-block cluster per utterance, k_sparse.cu's
sparse_cl_eps_* kernels) on the GPU against the live reference: gtnb_backoff_transitions_loss, gtnb_viterbi_backoff
and gtnb_backoff_transitions_viterbi for a backoff 4-gram of 8563 states (57 231 emitting, 8562 epsilon arcs), at
small B and T so that the reference can materialise; the route read from the kernel profile; host and device
buffers.  With the flag at 0 the same G takes the materialised route with the same outputs.  With the flag at 2 / 4 /
8 the benchmark's pruned trigram (inside the one-CTA envelope) gives the one-CTA kernels' losses and decode ==.  Ties,
a non-finite value, ragged lengths with a zero, B = 0, an epsilon-free G, and the torch functions with
large_transitions=True on a side stream."""
import functools

import numpy as np
import pytest

from tests import backoff_align_oracle as ba
from tests import backoff_oracle as bo
from tests import graph_oracle as go
from tests import sparse_trans_oracle as st
from tests import util
from tests.test_gpu_backoff import check, gview
from tests.test_gpu_graph_transitions import _gtn_graph, views_of

pytestmark = pytest.mark.gpu

CLUSTER_LOSS = {"sparse_cl_eps_forward", "sparse_cl_eps_backward", "sparse_eps_forward", "sparse_eps_gather"}
CLUSTER_DECODE = {"sparse_cl_eps_viterbi", "sparse_eps_trace"}
ONE_CTA_DEN = {"sparse_eps_viterbi"}


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


def composes(names):
    return any(n.startswith("gcompose") or n == "compose_emit" for n in names)


@functools.lru_cache(maxsize=None)
def fourgram():
    """the backoff 4-gram at C = 64 counted from 60 000 tokens (seed 1): 8563 states, beyond the one-CTA envelope"""
    G, tw = bo.backoff_ngram(np.random.default_rng(1), 64, 4, n_tokens=60000)
    assert len(G["flags"]) > 4096
    return G, tw


def inputs(rng, B, T, C):
    """ragged lengths with a zero; CTC graphs (even b) and path chains (odd b) of random labels"""
    lens = np.asarray([T, T - 1, 0, T - 2][:B], np.int32)
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    graphs = []
    for b in range(B):
        labels = rng.integers(1, C, 3)
        if b % 2 == 0:
            g = go.ctc_graph(labels)
        else:
            k = max(int(lens[b]), 1)
            lab = rng.integers(0, C, k)
            g = go.make([1] + [0] * (k - 1) + [2], np.arange(k), np.arange(1, k + 1), lab)
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
        graphs.append(g)
    return e, lens, graphs


def test_flag_1_loss_decode_and_alignment_match_the_reference(ref, ctx, flag):
    G, tw = fourgram()
    C, B, T = 64, 4, 10
    rng = np.random.default_rng(2)
    e, lens, graphs = inputs(rng, B, T, C)
    want = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
    assert np.isfinite(want[0][[0, 1, 3]]).all()
    wdec = bo.ref_backoff_viterbi(e, G, tw, lens)
    wali = ba.ref_backoff_trans_viterbi(e, graphs, G, tw, lens)
    # flag 0: the materialised route
    got0, names = profiled(ctx, lambda: ctx.backoff_transitions_loss(e, views_of(graphs), gview(G), tw,
                                                                     input_lens=lens))
    assert composes(names) and not names & CLUSTER_LOSS, sorted(names)
    dec0, names = profiled(ctx, lambda: ctx.viterbi_backoff(e, gview(G), tw, input_lens=lens))
    assert composes(names) and not names & CLUSTER_DECODE, sorted(names)
    flag(1)
    for run in (ctx.backoff_transitions_loss, ctx.backoff_transitions_loss_dev):
        got, names = profiled(ctx, lambda: run(e, views_of(graphs), gview(G), tw, input_lens=lens))
        assert CLUSTER_LOSS <= names and not composes(names), sorted(names)
        fin = np.isfinite(want[0])
        assert np.allclose(got[0][fin], want[0][fin], rtol=1e-4, atol=0) and np.isnan(got[0][2])
        check(got, want, T)
        assert np.allclose(got[0][fin], got0[0][fin], rtol=1e-4, atol=0)
    for run in (ctx.viterbi_backoff, ctx.viterbi_backoff_dev):
        got, names = profiled(ctx, lambda: run(e, gview(G), tw, input_lens=lens))
        assert CLUSTER_DECODE <= names and not composes(names), sorted(names)
        for x, y, z in zip(got, wdec, dec0):
            assert np.array_equal(x, y) and np.array_equal(x, z)
    for run in (ctx.backoff_transitions_viterbi, ctx.backoff_transitions_viterbi_dev):
        got, names = profiled(ctx, lambda: run(e, views_of(graphs), gview(G), tw, input_lens=lens))
        assert "sparse_eps_align" in names and not composes(names), sorted(names)
        for x, y in zip(got, wali):
            assert np.array_equal(x, y)
    flag(0)
    got, names = profiled(ctx, lambda: ctx.backoff_transitions_viterbi(e, views_of(graphs), gview(G), tw,
                                                                       input_lens=lens))
    assert composes(names) and "sparse_eps_align" not in names
    for x, y in zip(got, wali):
        assert np.array_equal(x, y)


def test_forced_cluster_sizes_reproduce_the_one_cta_kernels(ctx, flag):
    """the benchmark's pruned trigram (2065 states, inside the one-CTA envelope) with 2, 4 and 8 CTAs per utterance"""
    rng = np.random.default_rng(64)
    C = 64
    G, tw = bo.backoff_lm(rng, C)
    B, T = 6, 40
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    lens = np.asarray([T, T - 7, 1, 0, T - 1, T // 2], np.int32)
    graphs = [go.ctc_graph(rng.integers(1, C, 4)) for _ in range(B)]
    ctx.set_flag("exact_ties", 0)
    try:
        dec0, names = profiled(ctx, lambda: ctx.viterbi_backoff_dev(e, gview(G), tw, input_lens=lens))
        assert ONE_CTA_DEN <= names
        loss0, names = profiled(ctx, lambda: ctx.backoff_transitions_loss_dev(e, views_of(graphs), gview(G), tw,
                                                                              input_lens=lens))
        assert "sparse_eps_backward" in names and not names & CLUSTER_LOSS - {"sparse_eps_forward", "sparse_eps_gather"}
        for N in (2, 4, 8):
            flag(N)
            dec, names = profiled(ctx, lambda: ctx.viterbi_backoff_dev(e, gview(G), tw, input_lens=lens))
            assert CLUSTER_DECODE <= names and not names & ONE_CTA_DEN
            for x, y in zip(dec, dec0):
                assert np.array_equal(x, y)
            loss, names = profiled(ctx, lambda: ctx.backoff_transitions_loss_dev(e, views_of(graphs), gview(G), tw,
                                                                                 input_lens=lens))
            assert CLUSTER_LOSS <= names
            assert np.array_equal(loss[0], loss0[0], equal_nan=True)
            for x, y in zip(loss[1:], loss0[1:]):
                assert util.close(x, y)
    finally:
        ctx.set_flag("exact_ties", 1)


def test_ties_and_a_non_finite_value_are_retried_on_the_exact_route(ref, ctx, flag):
    """integer emissions and zero weights on the 4-gram: tied utterances re-run alone on the exact route; with
    exact_ties off they keep the cluster's path and score; a NaN emission is retried too"""
    G, _ = fourgram()
    C, B, T = 64, 3, 4
    rng = np.random.default_rng(30)
    e = rng.integers(0, 2, (B, T, C)).astype(np.float32)
    lens = np.asarray([T, T, 2], np.int32)
    tw = np.zeros(len(G["src"]), np.float32)
    flag(1)
    want = bo.ref_backoff_viterbi(e, G, tw, lens)
    got, names = profiled(ctx, lambda: ctx.viterbi_backoff(e, gview(G), tw, input_lens=lens))
    assert CLUSTER_DECODE <= names and composes(names)
    for x, y in zip(got, want):
        assert np.array_equal(x, y)
    ctx.set_flag("exact_ties", 0)
    try:
        (p, s, a), names = profiled(ctx, lambda: ctx.viterbi_backoff(e, gview(G), tw, input_lens=lens))
    finally:
        ctx.set_flag("exact_ties", 1)
    assert CLUSTER_DECODE <= names and not composes(names)
    assert np.array_equal(s, want[1])
    for b in range(B):
        n = int(lens[b])
        assert np.array_equal(p[b, :n], G["olabel"][a[b, :n]])
    tw2 = fourgram()[1]
    e2 = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    e2[1, 1, :] = np.nan
    got, names = profiled(ctx, lambda: ctx.viterbi_backoff(e2, gview(G), tw2, input_lens=lens))
    for x, y in zip(got, bo.ref_backoff_viterbi(e2, G, tw2, lens)):
        assert np.array_equal(x, y)
    assert CLUSTER_DECODE <= names and composes(names)
    _, _, graphs = inputs(rng, B, T, C)
    got, names = profiled(ctx, lambda: ctx.backoff_transitions_loss(e2, views_of(graphs), gview(G), tw2,
                                                                     input_lens=lens))
    want = st.ref_sparse_trans_loss(e2, graphs, G, tw2, lens)
    assert "sparse_cl_eps_forward" in names and composes(names)
    assert util.close(got[0], want[0])


def test_empty_batch_and_zero_lengths(ctx, flag):
    G, tw = fourgram()
    C = 64
    flag(1)
    p, s, a = ctx.viterbi_backoff(np.zeros((0, 5, C), np.float32), gview(G), tw)
    assert p.shape == (0, 5) and s.shape == (0,)
    assert not ctx.backoff_transitions_loss(np.zeros((0, 3, C), np.float32), [], gview(G), tw)[3].any()
    p, s, a = ctx.viterbi_backoff(np.zeros((2, 3, C), np.float32), gview(G), tw, input_lens=[0, 0])
    assert np.isneginf(s).all() and (p == -1).all()


def test_epsilon_free_graph_keeps_the_sparse_cluster_kernels(ctx, flag):
    """an epsilon-free G through the backoff functions with the flag at 1 takes sparse_cl_*, as the sparse ones do"""
    rng = np.random.default_rng(50)
    C = 32
    G = st.sparse_graph(rng, 5000, 40000, C, n_start=40, n_accept=2500, n_unreachable=0)
    tw = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    B, T = 2, 6
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    flag(1)
    got, names = profiled(ctx, lambda: ctx.viterbi_backoff(e, gview(G), tw))
    assert "sparse_cl_viterbi_forward" in names and not names & CLUSTER_DECODE
    want = ctx.viterbi_sparse(e, gview(G), tw)
    for x, y in zip(got, want):
        assert np.array_equal(x, y)


def test_torch_functions_with_large_transitions_on_a_side_stream(ref, ctx):
    torch = pytest.importorskip("torch")
    import gtn_b200.gtn as gtn
    from gtn_b200 import torch_loss
    G, tw = fourgram()
    C, B, T = 64, 2, 6
    rng = np.random.default_rng(40)
    e, lens, graphs = inputs(rng, B, T, C)
    Gg, gg = _gtn_graph(gtn, G), [_gtn_graph(gtn, g) for g in graphs]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        x = torch.tensor(e, device="cuda", requires_grad=True)
        tr = torch.tensor(tw, device="cuda", requires_grad=True)
        il = torch.tensor(lens)
        out = torch_loss.backoff_transitions_loss(x, tr, Gg, gg, input_lengths=il, reduction="mean",
                                                  large_transitions=True)
        out.backward()
        dec = torch_loss.backoff_viterbi(x.detach(), tr.detach(), Gg, input_lengths=il, large_transitions=True)
        ali = torch_loss.backoff_transitions_viterbi(x.detach(), tr.detach(), Gg, gg, input_lengths=il,
                                                     large_transitions=True)
    side.synchronize()  # (_gtn_graph keeps the graphs' own weights, g["w"])
    lr, gr, _, tgr = st.ref_sparse_trans_loss(e, graphs, G, tw, lens)
    assert util.close(out.item(), lr.mean())
    assert util.grad_close(x.grad.cpu().numpy(), gr / B, 50.0)
    assert util.grad_close(tr.grad.cpu().numpy(), tgr / B, 50.0 * B)
    for got, want in ((dec, bo.ref_backoff_viterbi(e, G, tw, lens)), (ali, ba.ref_backoff_trans_viterbi(e, graphs, G, tw,
                                                                                                     lens))):
        for x_, y_ in zip(got, want):
            assert np.array_equal(x_.cpu().numpy(), y_)
