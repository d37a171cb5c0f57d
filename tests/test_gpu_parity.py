"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle.

Bit-exact for indices / paths, 1e-4 relative (+1e-5 abs, see tests/util.py) for
scores and gradients -- BASELINE.json:north_star.
"""
import os

import numpy as np
import pytest

from tests import util

pytestmark = pytest.mark.gpu


def _oracle_graph(oracle, flags, src, dst, il, ol, w):
    return oracle.Graph.from_arrays(flags, src, dst, il, ol, w)


# ---------------------------------------------------------------------------
# generic graphs through gtnb_pack
# ---------------------------------------------------------------------------

def test_known_answers_forward(ctx, oracle):
    """test/functions_test.cpp:231-389 'Test Forward' known answers."""
    inf = np.inf
    cases = []
    # empty graph -> -inf (:233-236)
    cases.append((np.zeros(0, np.uint8), [], [], [], -inf))
    # two -inf arcs (:297-304) ; inf arc (:306-314) ; single node (:316-320)
    cases.append((np.array([1, 2], np.uint8), [0, 0], [1, 1], [-inf, -inf], -inf))
    cases.append((np.array([1, 2], np.uint8), [0, 0], [1, 1], [inf, 0.0], inf))
    cases.append((np.array([3], np.uint8), [], [], [], 0.0))
    # simple case (:322-334) = 6.8152
    cases.append((np.array([1, 0, 2], np.uint8), [0, 0, 0, 1, 1, 1], [1, 1, 1, 2, 2, 2],
                  [1, 2, 3, 1, 2, 3], 6.8152))
    views = []
    for flags, src, dst, w, _ in cases:
        lab = np.zeros(len(src), np.int32)
        views.append(util.capi.make_view(flags, np.asarray(src, np.int32), np.asarray(dst, np.int32),
                                         lab, lab, np.asarray(w, np.float32)))
    lat = ctx.pack(views)
    got = lat.forward()
    for g, c in zip(got, cases):
        if np.isinf(c[4]):
            assert g == c[4]
        else:
            assert abs(g - c[4]) < 1e-3
    lat.free()


def test_invalid_graphs_raise(ctx):
    """self-loop / cycle / orphan predecessor -> invalid_argument (functions_test.cpp:238-291)."""
    bad = [
        (np.array([3], np.uint8), [0], [0]),
        (np.array([1, 0, 2], np.uint8), [0, 1, 1], [1, 2, 1]),
        (np.array([1, 0, 2], np.uint8), [0, 1, 2], [1, 2, 2]),
        (np.array([1, 0, 2], np.uint8), [0, 1, 2], [1, 2, 0]),
        (np.array([1, 0, 2], np.uint8), [0, 1], [2, 2]),
    ]
    for flags, src, dst in bad:
        lab = np.zeros(len(src), np.int32)
        v = util.capi.make_view(flags, np.asarray(src, np.int32), np.asarray(dst, np.int32), lab, lab,
                                np.zeros(len(src), np.float32))
        lat = ctx.pack([v])
        with pytest.raises(ValueError):
            lat.forward()
        with pytest.raises(ValueError):
            lat.viterbi_path(8)
        lat.free()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_dags_vs_oracle(ctx, oracle, seed):
    rng = np.random.default_rng(seed)
    graphs, views = [], []
    for _ in range(24):
        n = int(rng.integers(2, 40))
        a = int(rng.integers(n, 4 * n))
        flags, src, dst, il, ol, w = util.random_dag(rng, n, a)
        # extra start / accept nodes now and then
        if rng.random() < 0.5:
            flags[int(rng.integers(0, n))] |= 1
        if rng.random() < 0.5:
            flags[int(rng.integers(0, n))] |= 2
        g = _oracle_graph(oracle, flags, src, dst, il, ol, w)
        graphs.append(g)
        views.append(util.view_of(g))
    lat = ctx.pack(views)
    for tropical in (False, True):
        got = lat.forward(tropical=tropical)
        lat.backward(tropical=tropical)
        for b, g in enumerate(graphs):
            s, gr = oracle.forward_score_and_grad(g, tropical)
            assert util.close(got[b], s), (b, got[b], s)
            mine = lat.arc_grads(b, g.num_arcs)
            if tropical:
                assert np.array_equal(mine, gr), (b, mine, gr)
            else:
                assert util.close(mine, gr), (b, np.abs(mine - gr).max())
    lat.free()


@pytest.mark.parametrize("seed", [3, 4])
def test_viterbi_path_ties_vs_oracle(ctx, oracle, seed):
    """Integer weights force ties; the path must be the reference's (first-relaxed wins)."""
    rng = np.random.default_rng(seed)
    graphs, views = [], []
    for _ in range(32):
        n = int(rng.integers(2, 30))
        a = int(rng.integers(n, 5 * n))
        flags, src, dst, il, ol, w = util.random_dag(rng, n, a, int_weights=True)
        g = _oracle_graph(oracle, flags, src, dst, il, ol, w)
        graphs.append(g)
        views.append(util.view_of(g))
    lat = ctx.pack(views)
    out = lat.viterbi_path(64)
    for b, g in enumerate(graphs):
        want = oracle.shortest_path(g)
        assert want is not None
        assert out["lens"][b] == len(want)
        assert np.array_equal(out["arcs"][b, :len(want)], want), (b, out["arcs"][b, :len(want)], want)
    lat.free()


# ---------------------------------------------------------------------------
# frame-synchronous compose + CTC
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("blank_last", [False, True])
def test_compose_ctc_structure_and_scores(ctx, oracle, blank_last):
    rng = np.random.default_rng(7)
    B, T, C, U = 6, 40, 9, 5
    e = rng.uniform(-5, 5, (B, T, C)).astype(np.float32)
    blank = C - 1 if blank_last else 0
    targets = [rng.integers(0 if blank_last else 1, C - 1 if blank_last else C, U) for _ in range(B)]
    targets[1] = np.array([2, 2, 2, 3, 3])  # repeats: no skip arcs
    e_dev = ctx.to_device(e)
    ctcs = [oracle.Graph.ctc(t, blank, True) for t in targets]
    views = [util.view_of(g) for g in ctcs]
    lat = ctx.compose_linear(views, [T] * B, C, e_dev, T * C)
    nn, na = lat.sizes()
    got = lat.forward()
    got_t = lat.forward(tropical=True)
    for b in range(B):
        ref = oracle.intersect(ctcs[b], oracle.Graph.linear(T, C, e[b]))
        assert (nn[b], na[b]) == (ref.num_nodes, ref.num_arcs)
        s, _, _, _ = oracle.shortest_distance(ref, False)
        st, _, _, _ = oracle.shortest_distance(ref, True)
        assert util.close(got[b], s)
        assert got_t[b] == st  # tropical: adds only, same association -> bit exact
        d = lat.download(b)
        # same multiset of (ilabel, olabel, weight) arcs as the reference's lattice
        ra = ref.arrays()
        mine = sorted(zip(d["ilabel"].tolist(), d["olabel"].tolist(), d["w"].tolist()))
        theirs = sorted(zip(ra["ilabel"].tolist(), ra["olabel"].tolist(), ra["w"].tolist()))
        assert mine == theirs
    lat.free()
    e_dev.free()


def test_ctc_loss_and_grad_small(ctx, oracle):
    B, T, C, U = 5, 60, 12, 7
    e, targets = util.bench_inputs(B, T, C, U)
    losses, grads = ctx.ctc_loss(e, targets, blank=0)
    for b in range(B):
        lo, go = oracle.ctc_loss(e[b], targets[b], 0, True)
        assert util.close(losses[b], lo), (losses[b], lo)
        assert util.grad_close(grads[b], go, 5.0 * T), np.abs(grads[b] - go).max()


def test_ctc_reference_known_answers(ctx):
    """test/criterion_test.cpp:84-179: TensorFlow CTC cases (loss + emission gradients)."""
    T, N = 5, 6
    probs3 = np.array([
        0.633766, 0.221185, 0.0917319, 0.0129757, 0.0142857, 0.0260553,
        0.111121, 0.588392, 0.278779, 0.0055756, 0.00569609, 0.010436,
        0.0357786, 0.633813, 0.321418, 0.00249248, 0.00272882, 0.0037688,
        0.0663296, 0.643849, 0.280111, 0.00283995, 0.0035545, 0.00331533,
        0.458235, 0.396634, 0.123377, 0.00648837, 0.00903441, 0.00623107], np.float32)
    grad3 = np.array([
        -0.366234, 0.221185, 0.0917319, 0.0129757, 0.0142857, 0.0260553,
        0.111121, -0.411608, 0.278779, 0.0055756, 0.00569609, 0.010436,
        0.0357786, 0.633813, -0.678582, 0.00249248, 0.00272882, 0.0037688,
        0.0663296, -0.356151, 0.280111, 0.00283995, 0.0035545, 0.00331533,
        -0.541765, 0.396634, 0.123377, 0.00648837, 0.00903441, 0.00623107], np.float32)
    probs4 = np.array([
        0.30176, 0.28562, 0.0831517, 0.0862751, 0.0816851, 0.161508,
        0.24082, 0.397533, 0.0557226, 0.0546814, 0.0557528, 0.19549,
        0.230246, 0.450868, 0.0389607, 0.038309, 0.0391602, 0.202456,
        0.280884, 0.429522, 0.0326593, 0.0339046, 0.0326856, 0.190345,
        0.423286, 0.315517, 0.0338439, 0.0393744, 0.0339315, 0.154046], np.float32)
    grad4 = np.array([
        -0.69824, 0.28562, 0.0831517, 0.0862751, 0.0816851, 0.161508,
        0.24082, -0.602467, 0.0557226, 0.0546814, 0.0557528, 0.19549,
        0.230246, 0.450868, 0.0389607, 0.038309, 0.0391602, -0.797544,
        0.280884, -0.570478, 0.0326593, 0.0339046, 0.0326856, 0.190345,
        -0.576714, 0.315517, 0.0338439, 0.0393744, 0.0339315, 0.154046], np.float32)
    e = np.log(np.stack([probs3, probs4]).reshape(2, T, N))
    losses, grads = ctx.ctc_loss(e, [[0, 1, 2, 1, 0], [0, 1, 1, 0]], blank=N - 1)
    assert abs(losses[0] - 3.34211) < 1e-4
    assert abs(losses[1] - 5.42262) < 1e-4
    assert np.abs(grads[0].ravel() - grad3).max() < 1e-5
    assert np.abs(grads[1].ravel() - grad4).max() < 1e-5


def test_ctc_config1_plumbing(ctx, oracle):
    """BASELINE.json configs[0]: B=1 T=100 C=28 U=10."""
    e, targets = util.bench_inputs(1, 100, 28, 10)
    losses, grads = ctx.ctc_loss(e, targets)
    lo, go = oracle.ctc_loss(e[0], targets[0], 0, True)
    assert util.close(losses[0], lo)
    assert util.grad_close(grads[0], go, 5.0 * 100)


def test_ctc_ragged_and_edge(ctx, oracle):
    """ragged input lengths, empty target, target too long for T (infeasible -> +inf loss)."""
    B, T, C = 4, 30, 6
    rng = np.random.default_rng(11)
    e = rng.uniform(-5, 5, (B, T, C)).astype(np.float32)
    targets = [rng.integers(1, C, 4), np.zeros(0, np.int32), rng.integers(1, C, 3),
               np.array([1, 1, 1, 1, 1, 1, 1, 1])]
    lens = np.array([30, 12, 1, 10], np.int32)
    losses, grads = ctx.ctc_loss(e, targets, input_lens=lens)
    for b in range(B):
        lo, go = oracle.ctc_loss(e[b, :lens[b]], targets[b], 0, True)
        assert util.close(losses[b], lo), (b, losses[b], lo)
        if np.isfinite(lo):
            assert util.grad_close(grads[b, :lens[b]], go, 5.0 * T), b
        assert not grads[b, lens[b]:].any()


def test_ctc_full_size_properties(ctx):
    """BASELINE config 2 shape (a slice of it): size-independent properties at T=1000, C=64.

    sum_c grad[t, c] == 0 for every frame (softmax part sums to 1, occupation
    part sums to 1), and the loss is invariant to adding a per-frame constant.
    """
    B, T, C, U = 8, 1000, 64, 100
    e, targets = util.bench_inputs(B, T, C, U)
    losses, grads = ctx.ctc_loss(e, targets)
    assert np.all(np.isfinite(losses)) and np.all(losses > 0)
    # (the reference's own fp32 row sums drift to 2.9e-3 here: tests/golden/README.md)
    assert np.abs(grads.sum(axis=2)).max() < 1e-2
    shift = np.random.default_rng(5).uniform(-1, 1, (B, T, 1)).astype(np.float32)
    losses2, _ = ctx.ctc_loss(e + shift, targets, want_grad=False)
    assert np.allclose(losses, losses2, rtol=1e-4)


def test_staged_and_generic_kernels_agree(ctx, oracle):
    """The TMA-staged kernels (SFU exp/log) against the generic libm-precise kernels on the
    same composed lattices: log scores/gradients within tolerance, tropical bit-exact."""
    B, T, C, U = 6, 200, 20, 12
    e, targets = util.bench_inputs(B, T, C, U)
    e_dev = ctx.to_device(e)
    views = [util.view_of(oracle.Graph.ctc(t, 0, True)) for t in targets]
    res = {}
    for staged in (1, 0):
        ctx.set_flag("staged", staged)
        lat = ctx.compose_linear(views, [T] * B, C, e_dev, T * C)
        _, na = lat.sizes()
        s_log = lat.forward()
        lat.backward(deltas=np.full(B, -1.0, np.float32))
        g_log = [lat.arc_grads(b, int(na[b])) for b in range(B)]
        s_trop = lat.forward(tropical=True)
        lat.backward(tropical=True)
        g_trop = [lat.arc_grads(b, int(na[b])) for b in range(B)]
        path = lat.viterbi_path(T)
        res[staged] = (s_log, g_log, s_trop, g_trop, path)
        lat.free()
    ctx.set_flag("staged", 1)
    assert util.close(res[1][0], res[0][0])
    assert np.array_equal(res[1][2], res[0][2])
    for b in range(B):
        assert util.grad_close(res[1][1][b], res[0][1][b], 5.0 * T)
        assert np.array_equal(res[1][3][b], res[0][3][b])
    assert np.array_equal(res[1][4]["arcs"], res[0][4]["arcs"])
    assert np.array_equal(res[1][4]["ilabels"], res[0][4]["ilabels"])
    # forced alignment against the oracle (viterbiPath(intersect(ctc, emissions)))
    for b in range(B):
        p, s = oracle.viterbi_ctc(e[b], targets[b], 0, True)
        assert np.array_equal(res[1][4]["ilabels"][b], p), b
        assert res[1][2][b] == s
    e_dev.free()


# ---------------------------------------------------------------------------
# dense-trellis Viterbi (BASELINE.json configs[3]) through the factored kernel
# ---------------------------------------------------------------------------

def test_viterbi_dense_golden_ties(ctx):
    """Integer scores: ties on every frame; paths must equal the reference's (golden fixture)."""
    gold = np.load(util.__file__.replace("util.py", "golden/reference_golden.npz"))
    e, tw = gold["vit_e"], gold["vit_tw"]
    # C = 6 in the fixture is not a multiple of 4: pad states with -inf-like scores that never win
    B, T, C = e.shape
    Cp = 8
    ep = np.full((B, T, Cp), -1e30, np.float32)
    ep[:, :, :C] = e
    twp = np.full(Cp + Cp * Cp, -1e30, np.float32)
    twp[:C] = tw[:C]
    tr = tw[C:].reshape(C, C)
    trp = np.full((Cp, Cp), -1e30, np.float32)
    trp[:C, :C] = tr
    twp[Cp:] = trp.ravel()
    paths, scores = ctx.viterbi_dense(ep, twp)
    assert np.array_equal(paths, gold["vit_paths"])
    assert np.array_equal(scores, gold["vit_scores"])


def test_viterbi_dense_vs_oracle_and_materialised(ctx, oracle):
    """Random float scores, C multiple of 4: the factored kernel, the materialised lattice path
    (gtnb_compose_linear + gtnb_viterbi_path) and the oracle agree bit for bit."""
    rng = np.random.default_rng(21)
    B, T, C = 5, 40, 8
    e = rng.uniform(-5, 5, (B, T, C)).astype(np.float32)
    e[0] = np.round(e[0])  # one utterance with ties
    tw = rng.uniform(-5, 5, C + C * C).astype(np.float32)
    tw_int = np.round(tw)
    for trans in (tw, tw_int):
        paths, scores = ctx.viterbi_dense(e, trans)
        e_dev = ctx.to_device(e)
        view = util.view_of(oracle.Graph.transitions(C, trans))
        lat = ctx.compose_linear([view], [T] * B, C, e_dev, T * C, linear_first=True, B=B)
        out = lat.viterbi_path(T)
        sc = lat.forward(tropical=True)
        for b in range(B):
            p, s = oracle.viterbi_dense(e[b], trans)
            assert np.array_equal(paths[b], p), b
            assert scores[b] == s
            assert np.array_equal(out["ilabels"][b], p), b
            assert sc[b] == s
        lat.free()
        e_dev.free()


def test_viterbi_dense_full_size_properties(ctx):
    """configs[3] shape (T=2000, C=128; a 16-utterance slice of the B=512 batch): the path's own
    score, re-accumulated on the host in the kernel's association, equals the returned
    viterbiScore bit for bit, and no single-frame substitution improves it."""
    B, T, C = 16, 2000, 128
    rng = np.random.default_rng(99)
    e = rng.uniform(-5, 5, (B, T, C)).astype(np.float32)
    tw = rng.uniform(-5, 5, C + C * C).astype(np.float32)
    paths, scores = ctx.viterbi_dense(e, tw)
    tr = tw[C:].reshape(C, C)  # tr[i, j] = w(j -> i)
    for b in range(B):
        p = paths[b]
        assert p.min() >= 0 and p.max() < C
        s = np.float32(0.0) + (e[b, 0, p[0]] + tw[p[0]])
        for t in range(1, T):
            s = np.float32(s + np.float32(e[b, t, p[t]] + tr[p[t], p[t - 1]]))
        assert s == scores[b], (b, s, scores[b])
    # local optimality on one utterance: changing any single interior frame cannot score higher
    b, p = 0, paths[0].astype(np.int64)
    for t in range(1, T - 1, 97):
        alt = e[b, t] + tr[:, p[t - 1]] + tr[p[t + 1], :]
        cur = e[b, t, p[t]] + tr[p[t], p[t - 1]] + tr[p[t + 1], p[t]]
        assert alt.max() <= cur + 1e-3


# ---------------------------------------------------------------------------
# ASG (BASELINE.json configs[2]) through the batched criterion
# ---------------------------------------------------------------------------

def test_asg_golden(ctx):
    """Three utterances sharing one transitions graph (fixture made by the real reference)."""
    gold = np.load(util.__file__.replace("util.py", "golden/reference_golden.npz"))
    e, tw, tg = gold["asg_e"], gold["asg_tw"], gold["asg_targets"]
    losses, grads, tgrad = ctx.asg_loss(e, tw, [t for t in tg])
    assert util.close(losses, gold["asg_loss"])
    assert util.grad_close(grads, gold["asg_grad"], 5.0 * e.shape[1])
    assert util.grad_close(tgrad, gold["asg_tgrad"], 5.0 * e.shape[1])


def test_asg_vs_oracle_medium(ctx, oracle):
    rng = np.random.default_rng(31)
    B, T, C, U = 6, 60, 16, 7
    e = rng.uniform(-5, 5, (B, T, C)).astype(np.float32)
    tw = rng.uniform(-5, 5, C + C * C).astype(np.float32)
    targets = [rng.integers(0, C, U).astype(np.int32) for _ in range(B)]
    targets[2] = np.array([3, 3, 3, 4], np.int32)  # repeats
    losses, grads, tgrad = ctx.asg_loss(e, tw, targets)
    tsum = np.zeros_like(tgrad)
    for b in range(B):
        lo, go, tg = oracle.asg_loss(e[b], tw, targets[b])
        tsum += tg
        assert util.close(losses[b], lo), (b, losses[b], lo)
        assert util.grad_close(grads[b], go, 5.0 * T), b
    assert util.grad_close(tgrad, tsum, 5.0 * T * B)


def test_asg_config3_shape_properties(ctx):
    """configs[2] shape (T=500, C=64, U=50; a 16-utterance slice of B=128): posteriors sum to
    one per frame on both lattices, so every frame's emission gradient sums to 0, and the
    transition gradient sums to 0 too (T-1 dense transitions + 1 start arc on each side)."""
    B, T, C, U = 16, 500, 64, 50
    rng = np.random.default_rng(41)
    e = rng.uniform(-5, 5, (B, T, C)).astype(np.float32)
    tw = rng.uniform(-5, 5, C + C * C).astype(np.float32)
    targets = [rng.integers(0, C, U).astype(np.int32) for _ in range(B)]
    losses, grads, tgrad = ctx.asg_loss(e, tw, targets)
    assert np.all(np.isfinite(losses)) and np.all(losses > 0)
    assert np.abs(grads.sum(axis=2)).max() < 1e-2
    assert abs(tgrad.sum()) < 1e-3 * T * B  # fp32 drift over T frames (see tests/golden/README.md)
    assert abs(tgrad[:C].sum()) < 1e-2 * B


def test_ctc_config2_utterance_vs_reference_and_float64(ctx):
    """One utterance of BASELINE.json configs[1] (T=1000, C=64, U=100) against the golden fixture:
    the reference's own fp32 result and a float64 evaluation of the same lattice.  The CUDA path
    must be at least as close to the float64 truth as the reference is (x2 slack), and within the
    conditioned tolerance of the reference (tests/util.py:grad_close)."""
    gold = np.load(util.__file__.replace("util.py", "golden/reference_golden.npz"))
    e, tg = util.bench_inputs(1, 1000, 64, 100)
    losses, grads = ctx.ctc_loss(e, tg)
    assert util.close(losses[0], gold["c2_loss"][0])
    assert abs(losses[0] - float(gold["c2_loss_f64"])) <= 2e-4 * abs(float(gold["c2_loss_f64"]))
    ref_err = np.abs(gold["c2_grad"][0] - gold["c2_grad_f64"]).max()
    my_err = np.abs(grads[0] - gold["c2_grad_f64"]).max()
    assert my_err <= 2.0 * ref_err + 1e-5, (my_err, ref_err)
    assert util.grad_close(grads[0], gold["c2_grad"][0], 5000.0)


def test_forced_alignment_full_size(ctx, oracle):
    """viterbiPath(intersect(ctc, emissions)) at T=2000, C=128, U=200 (SURVEY.md section 8(d), C4's
    second data point): bit-exact labels against the oracle for 2 utterances, and for 16 more the
    size-independent property that the path collapses (CTC rule) to the target."""
    B, T, C, U = 18, 2000, 128, 200
    e, targets = util.bench_inputs(B, T, C, U, seed=777)
    e_dev = ctx.to_device(e)
    views = [util.view_of(oracle.Graph.ctc(t, 0, True)) for t in targets]
    lat = ctx.compose_linear(views, [T] * B, C, e_dev, T * C)
    out = lat.viterbi_path(T)
    scores = lat.forward(tropical=True)
    for b in range(2):
        p, s = oracle.viterbi_ctc(e[b], targets[b], 0, True)
        assert np.array_equal(out["ilabels"][b], p)
        assert scores[b] == s
    for b in range(B):
        lab = out["ilabels"][b]
        assert out["lens"][b] == T
        keep = np.concatenate([[True], lab[1:] != lab[:-1]])
        collapsed = lab[keep]
        collapsed = collapsed[collapsed != 0]
        assert np.array_equal(collapsed, targets[b]), b
        # the path's score, re-accumulated on the host, is the returned viterbiScore
        s = np.float32(0.0)
        for t in range(T):
            s = np.float32(s + np.float32(0.0 + e[b, t, lab[t]]))
        assert s == scores[b]
    lat.free()
    e_dev.free()


# ---------------------------------------------------------------------------
# implicit-lattice criterion kernels (k_implicit.cu) against the materialised path
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("shape", [(4, 120, 16, 9), (3, 37, 8, 1), (2, 400, 32, 150), (2, 9, 5, 4)])
def test_ctc_implicit_and_materialised_agree(ctx, oracle, shape):
    """gtnb_ctc_loss sweeps the frames without building the lattice; with the flag off it builds
    compose's lattice and runs the generic kernels.  Same losses / gradients, both equal to the
    oracle.  (2, 400, 32, 150): 301 graph nodes > 256 threads (several nodes per thread);
    (2, 9, 5, 4): T == 2U+1, almost every node pruned."""
    B, T, C, U = shape
    e, targets = util.bench_inputs(B, T, C, U, seed=4321)
    lens = np.array([T - (3 * b) % max(T // 2, 1) for b in range(B)], np.int32)
    res = {}
    ctx.set_flag("bidir", 0)  # the two sweeps of k_implicit.cu (k_bidir.cu has its own tests below)
    try:
        for imp in (1, 0):
            ctx.set_flag("implicit", imp)
            ctx.profile(True)
            ctx.profile_read()
            res[imp] = ctx.ctc_loss(e, targets, input_lens=lens)
            names = set(ctx.profile_read())
            ctx.profile(False)
            assert ("implicit_forward" in names) == bool(imp), names
            assert ("compose_emit" in names) == (not imp), names
    finally:
        ctx.set_flag("implicit", 1)
        ctx.set_flag("bidir", -1)
    assert util.close(res[1][0], res[0][0])
    for b in range(B):
        lo, go = oracle.ctc_loss(e[b, :lens[b]], targets[b], 0, True)
        assert util.close(res[1][0][b], lo), (b, res[1][0][b], lo)
        if np.isfinite(lo):
            assert util.grad_close(res[1][1][b, :lens[b]], go, 5.0 * T), b
            assert util.grad_close(res[1][1][b], res[0][1][b], 5.0 * T), b
        assert not res[1][1][b, lens[b]:].any()


def test_ctc_implicit_falls_back_on_non_finite_emissions(ctx):
    """-inf on a label the target uses: the reference propagates inf / NaN arc by arc
    (shortest.cpp:62-80); the implicit sweep detects it and the call is repeated materialised,
    so the result is the materialised path's, bit for bit in the NaN pattern."""
    B, T, C, U = 3, 40, 6, 5
    e, targets = util.bench_inputs(B, T, C, U, seed=99)
    e[1, 7, int(targets[1][2])] = -np.inf
    ctx.profile(True)
    ctx.profile_read()
    l1, g1 = ctx.ctc_loss(e, targets)
    names = set(ctx.profile_read())
    ctx.profile(False)
    assert "implicit_forward" in names and "compose_emit" in names, names
    ctx.set_flag("implicit", 0)
    l0, g0 = ctx.ctc_loss(e, targets)
    ctx.set_flag("implicit", 1)
    assert np.array_equal(np.isnan(l1), np.isnan(l0)) and np.array_equal(np.isnan(g1), np.isnan(g0))
    assert np.allclose(l1[~np.isnan(l1)], l0[~np.isnan(l0)], rtol=1e-5)
    assert np.allclose(np.nan_to_num(g1, posinf=0, neginf=0), np.nan_to_num(g0, posinf=0, neginf=0),
                       rtol=1e-4, atol=1e-5)


def test_ctc_host_buffers_sub_batches_match_device_buffers(ctx):
    """Host buffers above 8 MB are cut into sub-batches of >= 4 MB that run on their own streams (H2D,
    sweeps and D2H overlapping); the result must equal the single-launch device-buffer call."""
    import ctypes as Ct
    from gtn_b200 import capi
    L = capi.lib()
    B, T, C, U = 24, 1000, 192, 60  # 18.4 MB of emissions -> 4 sub-batches
    e, targets = util.bench_inputs(B, T, C, U, seed=2024)
    lens = np.asarray([len(t) for t in targets], np.int32)
    cat = np.ascontiguousarray(np.concatenate(targets), np.int32)
    il = np.array([T - 7 * (b % 5) for b in range(B)], np.int32)
    # device buffers, one launch per kernel
    e_dev = ctx.to_device(e)
    g_dev = ctx.alloc(e.nbytes)
    l_dev = np.zeros(B, np.float32)
    ctx._check(L.gtnb_ctc_loss(ctx.h, B, T, C, e_dev.ptr, 1, il.ctypes.data_as(capi._i32p),
                               cat.ctypes.data_as(capi._i32p), lens.ctypes.data_as(capi._i32p), 0,
                               l_dev.ctypes.data_as(capi._f32p), g_dev.ptr, 1))
    g_from_dev = np.empty_like(e)
    ctx._check(L.gtnb_memcpy_d2h(ctx.h, g_from_dev.ctypes.data, g_dev.ptr, e.nbytes))
    ctx.synchronize()
    # host buffers (pageable numpy arrays): sub-batches
    ctx.profile(True)
    ctx.profile_read()
    l_host, g_host = ctx.ctc_loss(e, targets, input_lens=il)
    prof = ctx.profile_read()
    ctx.profile(False)
    assert prof["implicit_forward"][0] == 4 and prof["implicit_backward"][0] == 4, prof
    assert np.allclose(l_host, l_dev, rtol=1e-6)
    assert np.allclose(g_host, g_from_dev, rtol=1e-5, atol=1e-6)
    for b in range(B):
        assert not g_host[b, il[b]:].any()
    e_dev.free()
    g_dev.free()


@pytest.mark.parametrize("shape", [(5, 48, 12, 6), (3, 30, 64, 4), (2, 7, 5, 7)])
def test_asg_implicit_and_materialised_agree(ctx, oracle, shape):
    """gtnb_asg_loss without building either lattice (the dense transitions graph through the
    G-lanes-per-node sweeps, the forced-alignment chains one node per thread) against the
    materialised lattices and the oracle.  (3, 30, 64, 4): C=64 as in BASELINE configs[2], 65
    in-arcs per node; (2, 7, 5, 7): T == U, a single feasible alignment."""
    B, T, C, U = shape
    rng = np.random.default_rng(100 + T)
    e = rng.uniform(-5, 5, (B, T, C)).astype(np.float32)
    tw = rng.uniform(-5, 5, C + C * C).astype(np.float32)
    targets = [rng.integers(0, C, U).astype(np.int32) for _ in range(B)]
    targets[-1] = np.full(U, 1, np.int32)  # one label repeated
    res = {}
    for imp in (1, 0):
        ctx.set_flag("implicit", imp)
        ctx.profile(True)
        ctx.profile_read()
        res[imp] = ctx.asg_loss(e, tw, targets)
        names = set(ctx.profile_read())
        ctx.profile(False)
        assert ("implicit_forward" in names) == bool(imp), names
        assert ("compose_emit" in names) == (not imp), names
    ctx.set_flag("implicit", 1)
    assert util.close(res[1][0], res[0][0])
    tsum = np.zeros_like(res[1][2])
    for b in range(B):
        lo, go, tg = oracle.asg_loss(e[b], tw, targets[b])
        tsum += tg
        assert util.close(res[1][0][b], lo), (b, res[1][0][b], lo)
        assert util.grad_close(res[1][1][b], go, 5.0 * T), b
        assert util.grad_close(res[1][1][b], res[0][1][b], 5.0 * T), b
    assert util.grad_close(res[1][2], tsum, 5.0 * T * B)
    assert util.grad_close(res[1][2], res[0][2], 5.0 * T * B)


# ---------------------------------------------------------------------------
# the bidirectional meet-in-the-middle kernel (k_bidir.cu): gtnb_ctc_loss's default since round 2
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("shape", [(4, 120, 16, 9), (3, 37, 8, 1), (2, 9, 4, 4), (1, 100, 28, 10), (3, 64, 28, 30),
                                   (2, 300, 128, 111), (2, 1000, 64, 100), (5, 1, 8, 0)])
@pytest.mark.parametrize("want_grad", [True, False])
def test_ctc_bidir_agrees_with_two_sweeps_and_oracle(ctx, oracle, shape, want_grad):
    """gtnb_ctc_loss through k_bidir.cu (one launch: alpha from the front and beta from the back in a
    two-CTA cluster, posteriors on the fly, normaliser fused) against the two sweeps of k_implicit.cu
    (flag "bidir" 0), the oracle and the float64 referee; ragged input lengths; loss only.
    (2, 300, 128, 111): 223 graph nodes = all 7 node warps, C = 128; (5, 1, 8, 0): T = 1, empty targets."""
    from oracle import f64
    B, T, C, U = shape
    e, targets = util.bench_inputs(B, T, C, U, seed=555)
    lens = np.array([T - (5 * b) % max(T // 2, 1) for b in range(B)], np.int32)
    res = {}
    for bidir in (1, 0):
        ctx.set_flag("bidir", bidir)
        ctx.profile(True)
        ctx.profile_read()
        try:
            res[bidir] = ctx.ctc_loss(e, targets, input_lens=lens, want_grad=want_grad)
        finally:
            ctx.set_flag("bidir", -1)
        names = set(ctx.profile_read())
        ctx.profile(False)
        assert ("bidir_ctc" in names) == bool(bidir), names
        assert ("implicit_forward" in names) == (not bidir), names
        assert "compose_emit" not in names, names
    assert util.close(res[1][0], res[0][0])
    for b in range(B):
        lo, go = oracle.ctc_loss(e[b, :lens[b]], targets[b], 0, want_grad)
        assert util.close(res[1][0][b], lo), (b, res[1][0][b], lo)
        if want_grad and np.isfinite(lo):
            _, g64 = f64.ctc_f64(e[b, :lens[b]], targets[b])
            mine = res[1][1][b, :lens[b]]
            oracle_err = np.abs(go - g64).max()
            assert np.abs(mine - g64).max() <= 2.0 * oracle_err + 2e-6, b
            # the distance to the oracle's fp32 gradient is the oracle's own distance to the exact one
            assert np.abs(mine - go).max() <= 1.5 * oracle_err + 1e-5, b
            assert not res[1][1][b, lens[b]:].any()


@pytest.mark.parametrize("shape", [(6, 300, 64, 30), (3, 41, 64, 0), (2, 250, 128, 111), (4, 16, 64, 1)])
def test_ctc_bidir_node_warp_variants_agree(ctx, oracle, shape):
    """k_bidir.cu's two node-warp variants on the same CTC batch (C = 64 / 128): "bidir_mode" 0 one node per
    thread (reads ctc_build's tables), 1 PAIR (label + blank per thread, graphs from the targets, one launch);
    -1 = the default choice; 2 (a removed variant) is refused.  Loss and gradient against the oracle and the
    float64 referee for each; ragged lengths; blank = C - 1 for the second half of the modes."""
    from oracle import f64
    B, T, C, U = shape
    e, targets = util.bench_inputs(B, T, C, U, seed=91)
    lens = np.array([T - (3 * b) % max(T // 2, 1) for b in range(B)], np.int32)
    with pytest.raises(ValueError, match="bidir_mode"):
        ctx.set_flag("bidir_mode", 2)
    for mode in (0, 1, -1):
        ctx.set_flag("bidir_mode", mode)
        ctx.profile(True)
        ctx.profile_read()
        try:
            for want_grad in (True, False):
                before = ctx.launches
                loss, grad = ctx.ctc_loss(e, targets, input_lens=lens, want_grad=want_grad)
                if mode != 0:
                    assert ctx.launches - before == 1, "PAIR: the criterion is one launch"
                for b in range(B):
                    lo, go = oracle.ctc_loss(e[b, :lens[b]], targets[b], 0, want_grad)
                    assert util.close(loss[b], lo), (mode, b, loss[b], lo)
                    if want_grad and np.isfinite(lo):
                        _, g64 = f64.ctc_f64(e[b, :lens[b]], targets[b])
                        oracle_err = np.abs(go - g64).max()
                        assert np.abs(grad[b, :lens[b]] - g64).max() <= 2.0 * oracle_err + 2e-6, (mode, b)
                        assert not grad[b, lens[b]:].any()
        finally:
            ctx.set_flag("bidir_mode", -1)
        names = set(ctx.profile_read())
        ctx.profile(False)
        assert "bidir_ctc" in names and "implicit_forward" not in names, names
        assert ("ctc_build" in names) == (mode == 0), names


def test_ctc_bidir_falls_back_on_non_finite_emissions(ctx):
    """a non-finite emission raises the status bit and the call is repeated materialised, like the
    two-sweep path (C = 8: bidir eligible)."""
    B, T, C, U = 3, 40, 8, 5
    e, targets = util.bench_inputs(B, T, C, U, seed=98)
    e[1, 7, int(targets[1][2])] = -np.inf
    ctx.profile(True)
    ctx.profile_read()
    ctx.set_flag("bidir", 1)
    try:
        l1, g1 = ctx.ctc_loss(e, targets)
    finally:
        ctx.set_flag("bidir", -1)
    names = set(ctx.profile_read())
    ctx.profile(False)
    assert "bidir_ctc" in names and "compose_emit" in names, names
    ctx.set_flag("implicit", 0)
    l0, g0 = ctx.ctc_loss(e, targets)
    ctx.set_flag("implicit", 1)
    assert np.array_equal(np.isnan(l1), np.isnan(l0)) and np.array_equal(np.isnan(g1), np.isnan(g0))
    assert np.allclose(l1[~np.isnan(l1)], l0[~np.isnan(l0)], rtol=1e-5)


def test_ctc_bidir_host_buffers_sub_batches(ctx):
    """host buffers above 8 MB: sub-batches on their own streams, one bidir launch each."""
    B, T, C, U = 40, 1000, 128, 60  # 20.5 MB of emissions -> 4 sub-batches
    e, targets = util.bench_inputs(B, T, C, U, seed=2025)
    il = np.array([T - 7 * (b % 5) for b in range(B)], np.int32)
    ctx.set_flag("bidir", 1)
    try:
        l_dev, g_dev = ctx.ctc_loss_dev(e, targets, input_lens=il)
        ctx.profile(True)
        ctx.profile_read()
        l_host, g_host = ctx.ctc_loss(e, targets, input_lens=il)
    finally:
        ctx.set_flag("bidir", -1)
    prof = ctx.profile_read()
    ctx.profile(False)
    assert prof["bidir_ctc"][0] == 4, prof
    assert np.array_equal(l_host, l_dev)
    assert np.array_equal(g_host, g_dev)


# ---------------------------------------------------------------------------
# exact score ties in viterbiPath on device lattices (k_order.cu): on by default since round 2;
# gtnb_ctx_set_flag("exact_ties", 0) skips the ordering pass.
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("blank_last", [False, True])
def test_viterbi_exact_ties_vs_oracle(ctx, oracle, blank_last):
    """Integer-valued emissions make nearly every lattice
    node a tie; the path through the lattice API must then be the reference's, label for label."""
    B, T, C, U = 6, 40, 6, 7
    rng = np.random.default_rng(5 + blank_last)
    e = rng.integers(-1, 2, (B, T, C)).astype(np.float32)
    blank = C - 1 if blank_last else 0
    labels = [l for l in range(C) if l != blank]
    targets = [rng.choice(labels, U).astype(np.int32) for _ in range(B)]
    lens = [T - 3 * b for b in range(B)]
    e_dev = ctx.to_device(e)
    views = [util.view_of(oracle.Graph.ctc(t, blank, True)) for t in targets]
    lat = ctx.compose_linear(views, lens, C, e_dev, T * C)
    out = lat.viterbi_path(T)
    for b in range(B):
        p, s = oracle.viterbi_ctc(e[b, :lens[b]], targets[b], blank, True)
        assert out["lens"][b] == lens[b]
        assert np.array_equal(out["ilabels"][b][:lens[b]], p), (b, out["ilabels"][b][:lens[b]], p)
    lat.free()
    e_dev.free()
