"""gtnb_backoff_transitions_viterbi (the Viterbi alignment of gtnb_backoff_transitions_loss's numerators, G with epsilon
arcs) on the GPU against the live reference (tests/backoff_align_oracle.py): paths, arcs and scores == on both routes
(asserted from the kernel profile), with host and device buffers, with and without arc weights; ties with exact_ties
on and off; the benchmark's backoff trigram at C = 64 on the device route; an epsilon-free G == the sparse entry
point; scores at most the numerator's forwardScore; the golden fixture; edge cases, bad input and the torch
function on a side stream."""
import ctypes as C_

import numpy as np
import pytest

from gtn_b200 import capi
from tests import backoff_align_oracle as ba
from tests import backoff_oracle as bo
from tests import graph_oracle as go
from tests import sparse_trans_oracle as st
from tests.test_gpu_backoff import Gs, batch, gview, routed
from tests.test_gpu_graph_transitions import _gtn_graph, views_of

pytestmark = pytest.mark.gpu

DEVICE = {"sparse_eps_gather", "sparse_eps_align", "sparse_eps_align_trace"}


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


def check_rows(got, want, lens, graphs, exact):
    """scores ==; paths and arcs == when exact, else a path of A_b's emitting arcs with their own labels"""
    paths, scores, arcs = got
    assert np.array_equal(scores, want[1]), (scores, want[1])
    if exact:
        assert np.array_equal(paths, want[0]) and np.array_equal(arcs, want[2])
    for b in range(len(lens)):
        n = int(lens[b]) if np.isfinite(scores[b]) else 0
        assert (arcs[b, n:] == -1).all() and (paths[b, n:] == -1).all()
        assert np.array_equal(paths[b, :n], graphs[b]["olabel"][arcs[b, :n]])


@pytest.mark.parametrize("kind", ["bigram", "trigram", "random"])
@pytest.mark.parametrize("implicit", [1, 0])
def test_align_both_routes_host_and_device(ref, ctx, kind, implicit):
    C = 8
    rng = np.random.default_rng(len(kind) + 11 * implicit)
    G, tw = Gs(rng, C)[kind]
    e, graphs, lens = batch(rng, C)
    aw = np.concatenate([g["w"] for g in graphs]) + 0.125
    want = ba.ref_backoff_trans_viterbi(e, graphs, G, tw, lens)
    want_aw = ba.ref_backoff_trans_viterbi(e, graphs, G, tw, lens, weights=aw)
    assert np.isfinite(want[1]).any()
    ctx.set_flag("implicit", implicit)
    try:
        for run, arc_weights, w in ((ctx.backoff_transitions_viterbi, None, want),
                                    (ctx.backoff_transitions_viterbi, aw, want_aw),
                                    (ctx.backoff_transitions_viterbi_dev, None, want),
                                    (ctx.backoff_transitions_viterbi_dev, aw, want_aw)):
            got, taken = routed(ctx, lambda: run(e, views_of(graphs), gview(G), tw, input_lens=lens,
                                                 arc_weights=arc_weights), DEVICE)
            assert taken == ("device" if implicit else "exact"), taken
            check_rows(got, w, lens, graphs, True)
            fwd = ba.ref_backoff_trans_forward(e, graphs, G, tw, lens, weights=arc_weights)
            fin = np.isfinite(got[1])
            assert (got[1][fin] <= fwd[fin]).all() and np.array_equal(fin, np.isfinite(fwd))
    finally:
        ctx.set_flag("implicit", 1)


@pytest.mark.parametrize("exact_ties", [1, 0])
def test_ties(ref, ctx, exact_ties):
    """integer emissions and zero weights, so that paths tie: exact_ties on gives the reference's paths (the tied
    utterances re-run on the exact route), off an optimal path of the device route with the reference's score"""
    C, T, B = 6, 12, 5
    rng = np.random.default_rng(31 + exact_ties)
    G, tw = bo.backoff_ngram(rng, C, 3)
    tw = np.zeros_like(tw)
    graphs = [go.ctc_graph(rng.integers(1, C, int(rng.integers(1, 4)))) for _ in range(B)]
    e = rng.integers(-1, 2, (B, T, C)).astype(np.float32)
    lens = np.asarray([T, 0, 3, 7, T], np.int32)
    want = ba.ref_backoff_trans_viterbi(e, graphs, G, tw, lens)
    ctx.set_flag("exact_ties", exact_ties)
    try:
        for run in (ctx.backoff_transitions_viterbi, ctx.backoff_transitions_viterbi_dev):
            check_rows(run(e, views_of(graphs), gview(G), tw, input_lens=lens), want, lens, graphs, bool(exact_ties))
    finally:
        ctx.set_flag("exact_ties", 1)


def test_backoff_trigram_c64_takes_the_device_route(ref, ctx):
    """the benchmark's pruned backoff trigram with CTC graphs aligns without building a lattice"""
    C, T, B = 64, 30, 3
    rng = np.random.default_rng(65)
    G, tw = bo.backoff_lm(rng, C)
    graphs = [go.ctc_graph(rng.integers(1, C, 5)) for _ in range(B)]
    lens = np.asarray([T, T - 4, T - 9], np.int32)
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    want = ba.ref_backoff_trans_viterbi(e, graphs, G, tw, lens)
    ctx.set_flag("exact_ties", 0)  # (a tie would re-run its utterance on the exact route)
    try:
        got, taken = routed(ctx, lambda: ctx.backoff_transitions_viterbi_dev(e, views_of(graphs), gview(G), tw,
                                                                             input_lens=lens), DEVICE)
    finally:
        ctx.set_flag("exact_ties", 1)
    assert taken == "device", taken
    check_rows(got, want, lens, graphs, True)


def test_epsilon_free_equals_the_sparse_entry_point(ctx):
    """an epsilon-free G takes gtnb_sparse_transitions_viterbi's own code: outputs =="""
    C = 10
    rng = np.random.default_rng(19)
    G = st.sparse_graph(rng, 12, 80, C, label_hi=C + 1)
    tw = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
    e, graphs, lens = batch(rng, C)
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            a = ctx.backoff_transitions_viterbi(e, views_of(graphs), gview(G), tw, input_lens=lens)
            b = ctx.sparse_transitions_viterbi(e, views_of(graphs), gview(G), tw, input_lens=lens)
            for x, y in zip(a, b):
                assert np.array_equal(x, y)
        finally:
            ctx.set_flag("implicit", 1)


@pytest.mark.parametrize("name", ba.NAMES)
def test_golden_both_routes(ctx, name):
    _, e, lens, G, tw, graphs, want = [x for x in ba.golden_batches() if x[0] == name][0]
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            got = ctx.backoff_transitions_viterbi(e, views_of(graphs), gview(G), tw, input_lens=lens)
            assert all(np.array_equal(x, y) for x, y in zip(got, want))
        finally:
            ctx.set_flag("implicit", 1)


def test_edge_cases(ref, ctx):
    """T_b = 0, a graph too short for its frames, no start node, no arcs; epsilon arcs out of a start node at frame 0
    and into an accept node after the last frame, which are not reported"""
    C = 5
    rng = np.random.default_rng(2)
    G, tw = bo.backoff_ngram(rng, C, 3, n_tokens=800)
    e = rng.uniform(-2, 2, (4, 4, C)).astype(np.float32)
    graphs = [go.make([1, 0, 2], [0, 1], [1, 2], [1, 2]), go.make([1, 0, 0, 0, 0, 2], [0, 1, 2, 3, 4],
                                                                  [1, 2, 3, 4, 5], [1, 2, 3, 4, 1]),
              go.make([0, 2], [0], [1], [1]), go.make([], [], [], [])]
    lens = np.asarray([0, 4, 4, 4], np.int32)
    want = ba.ref_backoff_trans_viterbi(e, graphs, G, tw, lens)
    G2 = go.make([1, 0, 0, 2], [0, 1, 2, 1], [1, 2, 3, 1], [-1, 0, -1, 1])
    tw2 = np.asarray([0.5, -0.25, 0.75, 0.1], np.float32)
    ctc = [go.ctc_graph([0])] * 2
    want2 = ba.ref_backoff_trans_viterbi(e[:2], ctc, G2, tw2, [3, 1])
    assert np.isfinite(want2[1][1])
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        try:
            got = ctx.backoff_transitions_viterbi(e, views_of(graphs), gview(G), tw, input_lens=lens)
            assert np.isneginf(got[1]).all() and (got[0] == -1).all() and (got[2] == -1).all()
            assert all(np.array_equal(x, y) for x, y in zip(got, want))
            got = ctx.backoff_transitions_viterbi(e[:2], views_of(ctc), gview(G2), tw2, input_lens=[3, 1])
            assert all(np.array_equal(x, y) for x, y in zip(got, want2))
        finally:
            ctx.set_flag("implicit", 1)
    e0 = np.zeros((0, 3, C), np.float32)
    for run in (ctx.backoff_transitions_viterbi, ctx.backoff_transitions_viterbi_dev):  # B = 0 is a no-op
        paths, scores, arcs = run(e0, [], gview(G), tw)
        assert paths.shape == (0, 3) and scores.shape == (0,)


def test_bad_input(ctx):
    C = 5
    e = np.zeros((1, 4, C), np.float32)
    graphs = views_of([go.ctc_graph([1])])
    G, tw = bo.eps_cycle_graph()
    with pytest.raises(capi.GtnbInvalidArgument) as ex:
        ctx.backoff_transitions_viterbi(e, graphs, gview(G), tw)
    assert "cycle of epsilon arcs" in str(ex.value)
    half = go.make([1, 2], [0], [1], [-1], [1])  # epsilon on one side only: a transducer
    with pytest.raises(capi.GtnbError) as ex:
        ctx.backoff_transitions_viterbi(e, graphs, capi.make_view(half["flags"], half["src"], half["dst"],
                                                                  half["ilabel"], half["olabel"]),
                                        np.zeros(1, np.float32))
    assert ex.value.code == capi.ERR_UNSUPPORTED
    G, tw = bo.backoff_ngram(np.random.default_rng(1), C, 2, n_tokens=300)
    with pytest.raises(capi.GtnbError) as ex:  # epsilon in A_b
        ctx.backoff_transitions_viterbi(e, views_of([go.make([1, 2], [0], [1], [-1])]), gview(G), tw)
    assert ex.value.code == capi.ERR_UNSUPPORTED
    with pytest.raises(capi.GtnbInvalidArgument):  # T_b > T
        ctx.backoff_transitions_viterbi(e, graphs, gview(G), tw, input_lens=[5])
    gv, _keep = gview(G)
    arr = (capi.GraphView * 1)(graphs[0][0])
    rc = capi.lib().gtnb_backoff_transitions_viterbi(ctx.h, 1, 4, C, e.ctypes.data, 0, None, arr, None, 0,
                                                     C_.byref(gv), None, 0, None, None, None, 0)
    assert rc == capi.ERR_INVALID_ARGUMENT  # no trans_w


def test_torch_function_on_a_side_stream(ref):
    torch = pytest.importorskip("torch")
    import gtn_b200.gtn as gtn
    from gtn_b200 import torch_loss
    C = 9
    rng = np.random.default_rng(17)
    G, tw0 = bo.backoff_ngram(rng, C, 3, n_tokens=1200)
    e, graphs, lens = batch(rng, C)
    e = np.nan_to_num(e, nan=7.0)
    w0 = np.concatenate([g["w"] for g in graphs]) + 0.25
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        x = torch.tensor(e, device="cuda")
        tr = torch.tensor(tw0, device="cuda")
        w = torch.tensor(w0, device="cuda")
        paths, scores, arcs = torch_loss.backoff_transitions_viterbi(
            x, tr, _gtn_graph(gtn, G), [_gtn_graph(gtn, g) for g in graphs], input_lengths=torch.tensor(lens),
            weights=w)
    side.synchronize()
    wp, ws, wa = ba.ref_backoff_trans_viterbi(e, graphs, G, tw0, lens, weights=w0)
    assert np.array_equal(scores.cpu().numpy(), ws) and np.array_equal(paths.cpu().numpy(), wp)
    assert np.array_equal(arcs.cpu().numpy(), wa)
