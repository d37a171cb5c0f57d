"""k_beam.cu's beam_decode_kernel under the BeamLm policy (gtnb_beam_decode_lm_async) from source on the CPU, through
the SIMT emulator of tests/emu (tests/emu/beam_lm_emu.cpp), against the float64 restatement (tests/beam_lm_oracle.py)
for CTC, n-gram CTC and ASG.

Tokens, lengths and status are ==, scores, acoustic and LM scores within 1e-4, on every utterance whose decision
margin exceeds 1e-3.  Cases: K = 1; token_beam P < C, with a tie at the P-th boundary (status 3); P = C; T_b = 0 (with
a finite and a -inf end weight); a forbidden token; a hash under which every transcript collides; bf16 and fp16.  And
with no LM, no bonus and P = C, the results are == tests/emu/beam_emu.cpp's (gtnb_beam_decode_async's kernel).
"""
import ctypes as C_

import numpy as np
import pytest

from tests import backoff_oracle as bko
from tests import beam_lm_oracle as blo
from tests import beam_oracle as bo
from tests import emu_build
from tests import test_beam_emulation as tbe

vp = C_.c_void_p
CTC, BIGRAM, ASG = bo.CTC, bo.BIGRAM, bo.ASG
F32, BF16, F16 = 0, 1, 2


@pytest.fixture(scope="module")
def emu():
    lib = C_.CDLL(emu_build.build("beam_lm", ["k_beam.cu"]))
    lib.emu_beam_lm.argtypes = [C_.c_int, C_.c_int, C_.c_int, vp, C_.c_int, vp, C_.c_int, vp, C_.c_int, C_.c_int,
                                C_.c_int, vp, vp, C_.c_int, C_.c_float, C_.c_float, C_.c_int, C_.c_int, vp, vp, vp, vp,
                                vp, vp]
    return lib


def _p(a):
    return None if a is None else a.ctypes.data


def table(lm):
    """the resolved table of gtnb_lm_create, float32 sums in its order: (weight [S, C + 1], destination [S, C + 1])"""
    S, C = lm.S, lm.C
    w = np.full((S, C + 1), -np.inf, np.float32)
    d = np.zeros((S, C + 1), np.int32)
    depth = np.zeros(S, np.int64)
    for s in range(S):
        v = s
        while v in lm.eps:
            v = int(lm.dst[lm.eps[v]])
            depth[s] += 1
    for s in np.argsort(depth, kind="stable"):
        for c in range(C + 1):
            a = lm.arc.get((int(s), c))
            if a is not None:
                w[s, c], d[s, c] = np.float32(lm.w[a]), lm.dst[a]
            elif int(s) in lm.eps:
                e = lm.eps[int(s)]
                b = int(lm.dst[e])
                w[s, c], d[s, c] = np.float32(lm.w[e]) + w[b, c], d[b, c]
        if not lm.has_end:
            w[s, C] = 0.0
    return w, d


def run(emu, e, kind, trans_w=None, lens=None, blank=0, K=8, N=2, lm=None, alpha=1.0, beta=0.0, P=None,
        collide=False, dtype=F32):
    e = np.ascontiguousarray(e)
    B, T, Cn = e.shape
    tw = None if trans_w is None else np.ascontiguousarray(trans_w, np.float32)
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    lw, ld = table(lm) if lm is not None else (None, None)
    out = dict(tokens=np.full((B, N, T), 77, np.int32), lengths=np.full((B, N), 77, np.int32),
               scores=np.full((B, N), 77, np.float32), am=np.full((B, N), 77, np.float32),
               lm=np.full((B, N), 77, np.float32), status=np.full(B, 77, np.int32))
    emu_build.check(emu.emu_beam_lm(B, T, Cn, _p(e), dtype, _p(il), kind, _p(tw), blank, K, N, _p(lw), _p(ld),
                                    lm.start if lm is not None else 0, alpha, beta, Cn if P is None else P,
                                    int(collide), _p(out["tokens"]), _p(out["lengths"]), _p(out["scores"]),
                                    _p(out["am"]), _p(out["lm"]), _p(out["status"])))
    return out


def compare(got, want, frac=0.3):
    """== where the margin exceeds 1e-3 (at least frac of the utterances qualify)"""
    ok = (want["margin"] > 1e-3) | (want["status"] == 1) | (want["status"] == 2)
    assert ok.mean() >= frac, (ok.mean(), want["margin"])
    for b in np.nonzero(ok)[0]:
        assert got["status"][b] == want["status"][b], (b, got["status"][b], want["status"][b])
        assert np.array_equal(got["tokens"][b], want["tokens"][b]), (b, got["tokens"][b], want["tokens"][b])
        assert np.array_equal(got["lengths"][b], want["lengths"][b]), (b, got["lengths"][b], want["lengths"][b])
        for k in ("scores", "am", "lm"):
            g, w = got[k][b].astype(np.float64), want[k][b]
            fin = np.isfinite(w)
            assert np.array_equal(np.isnan(g), np.isnan(w)) and np.array_equal(g[~fin & ~np.isnan(w)],
                                                                                w[~fin & ~np.isnan(w)]), (k, b, g, w)
            assert np.allclose(g[fin], w[fin], rtol=1e-4, atol=1e-4), (k, b, g, w)
    return ok


def check(emu, e, kind, trans_w=None, lens=None, blank=0, K=8, N=2, lm=None, alpha=1.0, beta=0.0, P=None, frac=0.5,
          **kw):
    got = run(emu, e, kind, trans_w, lens, blank, K, N, lm, alpha, beta, P, **kw)
    want = blo.batch(e, kind, trans_w, lens, blank, K, N, lm, alpha, beta, P)
    ok = compare(got, want, frac)
    return got, want, ok


def with_eos(rng, G, w, C, n_neg_inf=0):
    """G with an end-of-sentence arc (label C) on every node, to itself; n_neg_inf of them weigh -inf"""
    S = len(G["flags"])
    x = np.log(rng.uniform(0.05, 0.5, S)).astype(np.float32)
    if n_neg_inf:
        x[rng.choice(np.arange(1, S), n_neg_inf, replace=False)] = -np.inf
    H = dict(G)
    for k, v in (("src", np.arange(S)), ("dst", np.arange(S)), ("ilabel", np.full(S, C)), ("olabel", np.full(S, C))):
        H[k] = np.concatenate([G[k], v]).astype(np.int32)
    return H, np.concatenate([w, x]).astype(np.float32)


def make_lm(rng, C, eos=True, n_neg_inf=0, n_end_neg_inf=0, order=3):
    G, w = bko.backoff_ngram(rng, C, order, n_tokens=1500, min_count=2, n_neg_inf=n_neg_inf)
    if eos:
        G, w = with_eos(rng, G, w, C, n_end_neg_inf)
    return blo.LM(G, w, C), G, w


def case(rng, kind, B, T, Cn):
    return tbe.case(rng, kind, B, T, Cn)


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
@pytest.mark.parametrize("K,N", [(1, 1), (8, 3)])
def test_random_ragged_fusion(emu, kind, K, N):
    rng = np.random.default_rng(200 + 10 * kind + K)
    B, T, Cn = 10, 30, 8
    e, tw = case(rng, kind, B, T, Cn)
    lens = rng.integers(0, T + 1, B)
    lens[0] = T
    lm = make_lm(rng, Cn, eos=K > 1)[0]
    check(emu, e, kind, tw, lens, blank=0, K=K, N=N, lm=lm, alpha=2.0, beta=1.5)


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
def test_token_pruning(emu, kind):
    rng = np.random.default_rng(300 + kind)
    B, T, Cn = 10, 30, 10
    e, tw = case(rng, kind, B, T, Cn)
    lm = make_lm(rng, Cn)[0]
    got, want, _ = check(emu, e, kind, tw, K=8, N=3, lm=lm, alpha=0.5, beta=-1.0, P=3)
    full = run(emu, e, kind, tw, K=8, N=3, lm=lm, alpha=0.5, beta=-1.0)
    assert not np.array_equal(full["scores"], got["scores"])  # (pruning changed something here)


@pytest.mark.parametrize("kind", [CTC, ASG])
def test_pruning_boundary_tie_flags(emu, kind):
    rng = np.random.default_rng(310 + kind)
    B, T, Cn = 4, 12, 8
    e, tw = case(rng, kind, B, T, Cn)
    e[:, 5, :] = -20.0
    e[:, 5, [2, 4, 6]] = -0.5  # tokens 2, 4 and 6 tie for the 2 places of P = 2
    lm = make_lm(rng, Cn)[0]
    got, want, _ = check(emu, e, kind, tw, K=4, N=2, lm=lm, alpha=0.5, P=2, frac=0.0)
    assert (got["status"] == 3).all() and (want["status"] == 3).all()


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
def test_full_token_beam_and_no_lm_is_beam_decode(emu, kind):
    rng = np.random.default_rng(320 + kind)
    B, T, Cn = 10, 30, 9
    e, tw = case(rng, kind, B, T, Cn)
    lens = rng.integers(0, T + 1, B)
    ref = tbe.run(_beam_emu(), e, kind, tw, lens, K=8, N=4)
    got = run(emu, e, kind, tw, lens, K=8, N=4, lm=None, alpha=1.0, beta=0.0, P=Cn)
    for k in ("tokens", "lengths", "scores", "status"):
        assert np.array_equal(ref[k], got[k]), k
    live = got["lengths"] >= 0
    assert np.array_equal(got["am"][live], got["scores"][live]) and (got["lm"][live] == 0).all()


def _beam_emu():
    lib = C_.CDLL(emu_build.build("beam", ["k_beam.cu"]))
    lib.emu_beam.argtypes = [C_.c_int, C_.c_int, C_.c_int, vp, C_.c_int, vp, C_.c_int, vp, C_.c_int, C_.c_int,
                             C_.c_int, C_.c_int, vp, vp, vp, vp]
    return lib


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
def test_empty_utterance_takes_the_start_end_weight(emu, kind):
    rng = np.random.default_rng(330 + kind)
    Cn = 6
    e, tw = case(rng, kind, 2, 5, Cn)
    lm, G, w = make_lm(rng, Cn)
    got = run(emu, e, kind, tw, [0, 0], K=4, N=2, lm=lm, alpha=2.0, beta=1.0)
    end = lm.end(lm.start)
    assert np.isfinite(end)
    assert (got["lengths"][:, 0] == 0).all() and (got["am"][:, 0] == 0).all()
    assert np.allclose(got["lm"][:, 0], end) and np.allclose(got["scores"][:, 0], 2.0 * end)
    assert (got["lengths"][:, 1] == -1).all() and np.isneginf(got["scores"][:, 1]).all()
    # a -inf end weight at the start node: no hypothesis
    w2 = w.copy()
    start_eos = np.flatnonzero((G["src"] == lm.start) & (G["ilabel"] == Cn))[0]
    w2[start_eos] = -np.inf
    got = run(emu, e, kind, tw, [0, 5], K=4, N=2, lm=blo.LM(G, w2, Cn), alpha=2.0, beta=1.0)
    assert (got["lengths"][0] == -1).all() and np.isneginf(got["scores"][0]).all()
    assert np.isneginf(got["am"][0]).all() and np.isneginf(got["lm"][0]).all()


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
def test_forbidden_tokens_and_end_weights(emu, kind):
    rng = np.random.default_rng(340 + kind)
    B, T, Cn = 10, 25, 6
    e, tw = case(rng, kind, B, T, Cn)
    lm, G, w = make_lm(rng, Cn, n_neg_inf=4, n_end_neg_inf=3)
    w2 = w.copy()
    root = np.flatnonzero((G["src"] == lm.start) & (G["ilabel"] == 2))
    w2[root] = -np.inf  # token 2 is forbidden from the root, whatever the history backs off to it
    lm = blo.LM(G, w2, Cn)
    got, want, _ = check(emu, e, kind, tw, K=8, N=4, lm=lm, alpha=0.5, beta=0.0)
    for b in range(B):
        for n in range(4):
            y = got["tokens"][b, n, :got["lengths"][b, n]]
            if got["lengths"][b, n] >= 0:
                assert np.isfinite(lm.score(y)), (b, n, y)


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
def test_degenerate_hash(emu, kind):
    rng = np.random.default_rng(350 + kind)
    B, T, Cn = 8, 30, 5
    e, tw = case(rng, kind, B, T, Cn)
    lm = make_lm(rng, Cn)[0]
    got, _, _ = check(emu, e, kind, tw, K=16, N=16, lm=lm, alpha=0.5, beta=1.0, P=3, collide=True)
    ref = run(emu, e, kind, tw, K=16, N=16, lm=lm, alpha=0.5, beta=1.0, P=3)
    for k in ref:
        assert np.array_equal(ref[k], got[k]), k


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("kind", [CTC, ASG])
def test_half_emissions_are_the_widened_float32(emu, dtype, kind):
    rng = np.random.default_rng(360 + dtype)
    B, T, Cn = 8, 25, 9
    e = tbe.emissions(rng, B, T, Cn, peak=8.0)
    if dtype == BF16:
        bits = (e.view(np.uint32) >> 16).astype(np.uint16)
        wide = (bits.astype(np.uint32) << 16).view(np.float32)
    else:
        bits = e.astype(np.float16).view(np.uint16)
        wide = bits.view(np.float16).astype(np.float32)
    tw = tbe.weights(rng, kind, Cn)
    lm = make_lm(rng, Cn)[0]
    got = run(emu, bits, kind, tw, K=8, N=3, lm=lm, alpha=0.5, beta=0.5, P=4, dtype=dtype)
    ref = run(emu, wide, kind, tw, K=8, N=3, lm=lm, alpha=0.5, beta=0.5, P=4)
    for k in ref:
        assert np.array_equal(ref[k], got[k]), k
    compare(got, blo.batch(wide, kind, tw, None, 0, 8, 3, lm, 0.5, 0.5, 4))
