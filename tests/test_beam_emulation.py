"""k_beam.cu's beam_weights_kernel and beam_decode_kernel from source on the CPU, through the SIMT emulator of tests/emu
(tests/emu/beam_emu.cpp), against the float64 restatement (tests/beam_oracle.py) for CTC, n-gram CTC and ASG.

Tokens, lengths and status are ==, scores within 1e-4 relative, on every utterance whose decision margin exceeds
1e-3 (and at least 90 % of them qualify).  Also: K = 1; N = K with fewer transcripts than N (the -inf slots); T_b = 0;
all-equal emissions (flagged 3, deterministic); -inf, NaN and +inf emissions and weights and each bad length alone,
with the other utterances unchanged; the degenerate hash (same results, never two live beams with one transcript);
bf16 / fp16 emissions against float32 on the widened values.
"""
import ctypes as C

import numpy as np
import pytest

from tests import beam_oracle as bo
from tests import emu_build

vp = C.c_void_p
CTC, BIGRAM, ASG = bo.CTC, bo.BIGRAM, bo.ASG
F32, BF16, F16 = 0, 1, 2


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("beam", ["k_beam.cu"]))
    lib.emu_beam.argtypes = [C.c_int, C.c_int, C.c_int, vp, C.c_int, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int,
                             C.c_int, vp, vp, vp, vp]
    return lib


def _p(a):
    return None if a is None else a.ctypes.data


def run(emu, e, kind, trans_w=None, lens=None, blank=0, K=8, N=2, collide=False, dtype=F32):
    """e: float32 [B, T, C], or uint16 bits for dtype BF16 / F16"""
    e = np.ascontiguousarray(e)
    B, T, Cn = e.shape
    tw = None if trans_w is None else np.ascontiguousarray(trans_w, np.float32)
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    out = dict(tokens=np.full((B, N, T), 77, np.int32), lengths=np.full((B, N), 77, np.int32),
               scores=np.full((B, N), 77, np.float32), status=np.full(B, 77, np.int32))
    emu_build.check(emu.emu_beam(B, T, Cn, _p(e), dtype, _p(il), kind, _p(tw), blank, K, N, int(collide),
                                 _p(out["tokens"]), _p(out["lengths"]), _p(out["scores"]), _p(out["status"])))
    return out


def weights(rng, kind, Cn, scale=1.0):
    if kind == CTC:
        return None
    return (rng.standard_normal(Cn * Cn + (Cn if kind == ASG else 0)) * scale).astype(np.float32)


def emissions(rng, B, T, Cn, peak=3.0):
    """log-softmax-like rows with a few peaked labels, so that beams and greedy paths differ a little"""
    x = rng.standard_normal((B, T, Cn)) * peak
    x -= np.log(np.exp(x).sum(-1, keepdims=True))
    return x.astype(np.float32)


def case(rng, kind, B, T, Cn):
    """emissions and weights whose decisions are well separated: CTC and n-gram CTC at a 10x log-probability scale,
    ASG on sharper rows (random rows at unit scale put near-equal candidates at the beam's boundary)"""
    if kind == ASG:
        return emissions(rng, B, T, Cn, peak=8.0), weights(rng, kind, Cn)
    return emissions(rng, B, T, Cn, peak=1.0) * 10, weights(rng, kind, Cn, 10.0)


QUALIFIED = [0, 0]  # utterances compared, utterances in the comparisons of this module


def compare(got, want, frac=0.3):
    """== where the margin exceeds 1e-3; at least frac of the utterances qualify here, 90 % over the module"""
    ok = (want["margin"] > 1e-3) | (want["status"] == 1) | (want["status"] == 2)
    assert ok.mean() >= frac, (ok.mean(), want["margin"])
    QUALIFIED[0] += int(ok.sum())
    QUALIFIED[1] += len(ok)
    for b in np.nonzero(ok)[0]:
        assert got["status"][b] == want["status"][b], (b, got["status"][b], want["status"][b])
        assert np.array_equal(got["tokens"][b], want["tokens"][b]), (b, got["tokens"][b], want["tokens"][b])
        assert np.array_equal(got["lengths"][b], want["lengths"][b]), (b, got["lengths"][b], want["lengths"][b])
        g, w = got["scores"][b].astype(np.float64), want["scores"][b]
        fin = np.isfinite(w)
        assert np.array_equal(np.isnan(g), np.isnan(w)) and np.array_equal(g[~fin & ~np.isnan(w)],
                                                                            w[~fin & ~np.isnan(w)]), (b, g, w)
        assert np.allclose(g[fin], w[fin], rtol=1e-4, atol=1e-4), (b, g, w)
    return ok


def check(emu, e, kind, trans_w=None, lens=None, blank=0, K=8, N=2, frac=0.5, **kw):
    got = run(emu, e, kind, trans_w, lens, blank, K, N, **kw)
    want = bo.batch(e, kind, trans_w, lens, blank, K, N)
    compare(got, want, frac)
    return got, want


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
@pytest.mark.parametrize("K,N", [(1, 1), (4, 2), (16, 5)])
def test_random_ragged(emu, kind, K, N):
    rng = np.random.default_rng(100 * kind + K)
    B, T, Cn = 10, 40, 12 if K < 16 else 7
    e, tw = case(rng, kind, B, T, Cn)
    lens = rng.integers(0, T + 1, B)
    lens[0] = T
    check(emu, e, kind, tw, lens, blank=kind == CTC and 3 or 0, K=K, N=N)


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
def test_fewer_transcripts_than_n_and_empty(emu, kind):
    rng = np.random.default_rng(5)
    Cn = 3 if kind != ASG else 2
    e = emissions(rng, 3, 2, Cn)
    got, want = check(emu, e, kind, weights(rng, kind, Cn), [2, 1, 0], K=16, N=16, frac=0.3)
    assert (got["scores"][2, 0] == 0.0 and got["lengths"][2, 0] == 0 and (got["tokens"][2] == -1).all() and
            np.isneginf(got["scores"][2, 1:]).all() and (got["lengths"][2, 1:] == -1).all())
    live = got["lengths"][0] >= 0
    assert live.sum() < 16 and np.isneginf(got["scores"][0][~live]).all()


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
def test_all_equal_is_a_deterministic_tie(emu, kind):
    Cn = 6
    e = np.zeros((2, 12, Cn), np.float32)
    tw = None if kind == CTC else np.zeros(Cn * Cn + (Cn if kind == ASG else 0), np.float32)
    a = run(emu, e, kind, tw, K=8, N=4)
    b = run(emu, e, kind, tw, K=8, N=4)
    assert (a["status"] == 3).all()
    assert (bo.batch(e, kind, tw, None, 0, 8, 4)["status"] == 3).all()
    for k in a:
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
def test_non_finite_and_bad_lengths_flag_alone(emu, kind):
    rng = np.random.default_rng(11 + kind)
    B, T, Cn = 7, 20, 8
    e = emissions(rng, B, T, Cn)
    tw = weights(rng, kind, Cn)
    lens = np.full(B, T)
    e[1, 3, 2] = np.nan
    e[2, 5, 4] = np.inf
    e[3, 2, :] = -np.inf  # every move of the frame forbidden: no hypothesis survives
    e[3, 2, 0] = -np.inf
    e[4, :, 5] = -np.inf  # one label forbidden throughout
    lens[5], lens[6] = -1, T + 1
    e[0, T - 1, 1] = np.nan
    lens[0] = T - 1  # a NaN beyond T_b is never read
    got, want = check(emu, e, kind, tw, lens, K=8, N=3, frac=0.3)
    assert list(got["status"][1:3]) == [1, 1] and list(got["status"][5:]) == [2, 2]
    assert got["status"][0] in (0, 3) and got["status"][4] in (0, 3)
    assert (got["lengths"][3] == -1).all() and np.isneginf(got["scores"][3]).all()
    assert not (got["tokens"][4] == 5).any()
    for b in (1, 2, 5, 6):
        assert np.isnan(got["scores"][b]).all() and (got["lengths"][b] == -1).all() and (got["tokens"][b] == -1).all()
    ref = run(emu, e[[0, 4]], kind, tw, lens[[0, 4]], K=8, N=3)  # the flagged utterances change nothing else
    for k in ref:
        assert np.array_equal(ref[k], got[k][[0, 4]]), k
    if kind != CTC:
        for bad in (np.nan, np.inf):
            tw2 = tw.copy()
            tw2[len(tw2) // 2] = bad
            g2 = run(emu, e[[0, 4]], kind, tw2, [T - 1, 0], K=8, N=3)
            assert list(g2["status"]) == [1, 0] and g2["scores"][1, 0] == 0.0
        tw3 = tw.copy()
        tw3[len(tw3) - 1] = -np.inf  # a forbidden transition is no error
        check(emu, e[[0, 4]], kind, tw3, [T - 1, T], K=8, N=3, frac=0.3)


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
def test_degenerate_hash(emu, kind):
    rng = np.random.default_rng(21 + kind)
    B, T, Cn = 10, 40, 5
    e, tw = case(rng, kind, B, T, Cn)
    got, want = check(emu, e, kind, tw, K=16, N=16, collide=True)
    ref = run(emu, e, kind, tw, K=16, N=16)
    for k in ref:
        assert np.array_equal(ref[k], got[k]), k
    for b in range(B):
        seen = {tuple(got["tokens"][b, n, :got["lengths"][b, n]]) for n in range(16) if got["lengths"][b, n] >= 0}
        assert len(seen) == (got["lengths"][b] >= 0).sum()


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("kind", [CTC, ASG])
def test_half_emissions_are_the_widened_float32(emu, dtype, kind):
    rng = np.random.default_rng(31 + dtype)
    B, T, Cn = 10, 30, 9
    e = emissions(rng, B, T, Cn, peak=8.0)
    if dtype == BF16:
        bits = (e.view(np.uint32) >> 16).astype(np.uint16)
        wide = (bits.astype(np.uint32) << 16).view(np.float32)
    else:
        bits = e.astype(np.float16).view(np.uint16)
        wide = bits.view(np.float16).astype(np.float32)
    tw = weights(rng, kind, Cn)
    got = run(emu, bits, kind, tw, K=8, N=3, dtype=dtype)
    ref = run(emu, wide, kind, tw, K=8, N=3)
    for k in ref:
        assert np.array_equal(ref[k], got[k]), k
    compare(got, bo.batch(wide, kind, tw, None, 0, 8, 3))


def test_margin_filter_keeps_most_utterances():
    """(runs after the comparisons above, in file order) the margin filter left at least 90 % of them compared"""
    if QUALIFIED[1] == 0:
        pytest.skip("no comparison ran in this session")
    assert QUALIFIED[0] >= 0.9 * QUALIFIED[1], QUALIFIED
