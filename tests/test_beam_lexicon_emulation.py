"""k_beam.cu's beam_decode_kernel under the BeamLex policy (gtnb_beam_decode_lexicon_async) from source on the CPU,
through the SIMT emulator of tests/emu (tests/emu/beam_lexicon_emu.cpp), against the float64 restatement
(tests/beam_lexicon_oracle.py) for CTC, n-gram CTC and ASG.

Tokens, words, lengths, word counts and status are ==, scores, acoustic and LM scores within 1e-4, on every utterance
whose decision margin exceeds 1e-3.  Cases: K = 1; N = K with fewer transcripts than N; T_b = 0; status 1 and 2
flagged alone; token_beam P < C; a transcript hash under which everything collides and a word-LM arc hash under which
every key probes from one slot; bf16 and fp16; backoff chains of full depth; a beam dropped at the end inside a word; a
lexicon that forbids every transcript.  The lexicon's device arrays are built here as gtnb_lexicon_create builds them
(device_arrays).
"""
import ctypes as C_

import numpy as np
import pytest

from tests import backoff_oracle as bko
from tests import beam_lexicon_oracle as lxo
from tests import beam_lm_oracle as blo
from tests import beam_oracle as bo
from tests import emu_build
from tests import test_beam_emulation as tbe

vp = C_.c_void_p
CTC, BIGRAM, ASG = bo.CTC, bo.BIGRAM, bo.ASG
F32, BF16, F16 = 0, 1, 2
HMUL = 0x9E3779B97F4A7C15


@pytest.fixture(scope="module")
def emu():
    lib = C_.CDLL(emu_build.build("beam_lexicon", ["k_beam.cu"]))
    lib.emu_beam_lexicon.argtypes = ([C_.c_int] * 3 + [vp, C_.c_int, vp, C_.c_int, vp] + [C_.c_int] * 3 + [vp] * 6 +
                                     [C_.c_ulonglong, C_.c_int, vp, vp, vp, C_.c_int, C_.c_float, C_.c_float,
                                      C_.c_int, C_.c_int] + [vp] * 8)
    return lib


def _p(a):
    return None if a is None else a.ctypes.data


def _resolve32(lm, s, x):
    """w(s, x) in float32, backoff weights added innermost first"""
    chain = []
    while (s, x) not in lm.arc:
        e = lm.eps.get(s)
        if e is None:
            return np.float32(-np.inf)
        chain.append(e)
        s = int(lm.dst[e])
    w = np.float32(lm.w[lm.arc[(s, x)]])
    for e in reversed(chain):
        w = np.float32(np.float32(lm.w[e]) + w)
    return w


def device_arrays(lex, hmul=HMUL):
    """gtnb_lexicon_create's device arrays of a beam_lexicon_oracle.Lexicon (breadth-first trie numbering, children
    in token order; float32 smear and end weights; the word LM's arc hash) as a dict of numpy arrays"""
    C, MW = lex.C, (lex.C + 31) // 32
    order, ident = [0], {0: 0}
    for n in order:
        for c in sorted(lex.kids[n]):
            ident[lex.kids[n][c]] = len(order)
            order.append(lex.kids[n][c])
    nodes = len(order)
    mask = np.zeros((nodes, MW), np.uint32)
    first = np.zeros(nodes, np.int32)
    word = np.full(nodes, -1, np.int32)
    for q, n in enumerate(order):
        word[q] = lex.word[n]
        ks = sorted(lex.kids[n])
        first[q] = ident[lex.kids[n][ks[0]]] if ks else 0
        for c in ks:
            mask[q, c >> 5] |= np.uint32(1 << (c & 31))
    smear = np.full(nodes, -np.inf, np.float32)
    lm = lex.lm
    out = dict(cls=np.asarray(lex.cls, np.int32), mask=mask, first=first, word=word, hash=None, hmul=hmul, hbits=0,
               bow=None, bod=None, endw=None, start=0)
    if lm is not None:
        for q in range(nodes - 1, 0, -1):
            best = _resolve32(lm, lm.start, int(word[q])) if word[q] >= 0 else np.float32(-np.inf)
            for i in range(len(lex.kids[order[q]])):
                best = max(best, smear[first[q] + i])
            smear[q] = best
        arcs = [(s, x, a) for (s, x), a in lm.arc.items() if x < lex.V]
        hb = 1
        while (1 << hb) < 2 * len(arcs):
            hb += 1
        H = 1 << hb
        table = np.zeros((H, 2), np.uint64)
        table[:, 0] = np.uint64(2**64 - 1)
        for s, x, a in arcs:
            key = (s << 32) | x
            i = (key * hmul % (1 << 64)) >> (64 - hb)
            while table[i, 0] != np.uint64(2**64 - 1):
                i = (i + 1) & (H - 1)
            table[i] = [key, (int(lm.dst[a]) << 32) | int(np.float32(lm.w[a]).view(np.uint32))]
        S = lm.S
        bod = np.full(S, -1, np.int32)
        bow = np.zeros(S, np.float32)
        for s, e in lm.eps.items():
            bod[s], bow[s] = lm.dst[e], lm.w[e]
        endw = np.array([_resolve32(lm, s, lex.V) if lm.has_end else 0.0 for s in range(S)], np.float32)
        out.update(hash=table, hbits=hb, bow=bow, bod=bod, endw=endw, start=lm.start)
    smear[0] = 0.0
    smear[~np.isfinite(smear)] = 0.0
    out["smear"] = smear
    return out


def run(emu, e, kind, lex, trans_w=None, lens=None, blank=0, K=8, N=2, lm_weight=1.0, word_bonus=0.0, P=None,
        collide=False, dtype=F32, hmul=HMUL):
    e = np.ascontiguousarray(e)
    B, T, Cn = e.shape
    tw = None if trans_w is None else np.ascontiguousarray(trans_w, np.float32)
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    d = device_arrays(lex, hmul)
    out = dict(tokens=np.full((B, N, T), 77, np.int32), lengths=np.full((B, N), 77, np.int32),
               scores=np.full((B, N), 77, np.float32), am=np.full((B, N), 77, np.float32),
               lm=np.full((B, N), 77, np.float32), words=np.full((B, N, T), 77, np.int32),
               counts=np.full((B, N), 77, np.int32), status=np.full(B, 77, np.int32))
    emu_build.check(emu.emu_beam_lexicon(
        B, T, Cn, _p(e), dtype, _p(il), kind, _p(tw), blank, K, N, _p(d["cls"]), _p(d["mask"]), _p(d["first"]),
        _p(d["word"]), _p(d["smear"]), _p(d["hash"]), d["hmul"], d["hbits"], _p(d["bow"]), _p(d["bod"]),
        _p(d["endw"]), d["start"], lm_weight, word_bonus, Cn if P is None else P, int(collide),
        *[_p(out[k]) for k in ("tokens", "lengths", "scores", "am", "lm", "words", "counts", "status")]))
    return out


def compare(got, want, frac=0.3):
    """== where the margin exceeds 1e-3 (at least frac of the utterances qualify)"""
    ok = (want["margin"] > 1e-3) | (want["status"] == 1) | (want["status"] == 2)
    assert ok.mean() >= frac, (ok.mean(), want["margin"])
    for b in np.nonzero(ok)[0]:
        for k in ("status", "tokens", "lengths", "words", "counts"):
            assert np.array_equal(got[k][b], want[k][b]), (k, b, got[k][b], want[k][b])
        for k in ("scores", "am", "lm"):
            g, w = got[k][b].astype(np.float64), want[k][b]
            fin = np.isfinite(w)
            assert np.array_equal(np.isnan(g), np.isnan(w)) and np.array_equal(g[~fin & ~np.isnan(w)],
                                                                                w[~fin & ~np.isnan(w)]), (k, b, g, w)
            assert np.allclose(g[fin], w[fin], rtol=1e-4, atol=1e-4), (k, b, g, w)
    return ok


def check(emu, e, kind, lex, trans_w=None, lens=None, blank=0, K=8, N=2, lm_weight=1.0, word_bonus=0.0, P=None,
          frac=0.5, **kw):
    got = run(emu, e, kind, lex, trans_w, lens, blank, K, N, lm_weight, word_bonus, P, **kw)
    want = lxo.batch(e, kind, trans_w, lens, blank, K, N, lex, lm_weight, word_bonus, P)
    ok = compare(got, want, frac)
    return got, want, ok


def word_lm(rng, V, order=3, eos=True, n_neg_inf=0, n_tokens=1500):
    """a backoff n-gram word LM over V words (labels [0, V], V end of sentence) -> beam_lm_oracle.LM"""
    G, w = bko.backoff_ngram(rng, V, order, n_tokens=n_tokens, min_count=2, n_neg_inf=n_neg_inf)
    if eos:
        S = len(G["flags"])
        x = np.log(rng.uniform(0.05, 0.5, S)).astype(np.float32)
        G = dict(G)
        for k, v in (("src", np.arange(S)), ("dst", np.arange(S)), ("ilabel", np.full(S, V)),
                     ("olabel", np.full(S, V))):
            G[k] = np.concatenate([G[k], v]).astype(np.int32)
        w = np.concatenate([w, x]).astype(np.float32)
    return blo.LM(G, w, V)


def letters_lexicon(rng, Cn, n_words, lm=True, mode="sep", **kw):
    """separator mode: token Cn - 1 is the separator; word-start mode: tokens Cn - 3 .. Cn - 1 start words"""
    if mode == "sep":
        cls, sp = lxo.random_lexicon(rng, Cn, n_words, sep=Cn - 1, max_len=3, **kw)
    else:
        cls, sp = lxo.random_lexicon(rng, Cn, n_words, word_start=range(Cn - 3, Cn), max_len=3, **kw)
    V = 1 + max(w for _, w in sp)
    return lxo.Lexicon(Cn, cls, sp, V, word_lm(rng, V) if lm else None)


def peaked(rng, kind, B, T, Cn):
    e, tw = tbe.case(rng, kind, B, T, Cn)
    return e * 3, tw


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
@pytest.mark.parametrize("mode", ["sep", "start"])
@pytest.mark.parametrize("K,N", [(1, 1), (8, 3)])
def test_random_ragged(emu, kind, mode, K, N):
    rng = np.random.default_rng(400 + 10 * kind + K + (mode == "sep"))
    B, T, Cn = 8, 20, 8
    e, tw = peaked(rng, kind, B, T, Cn)
    lens = rng.integers(0, T + 1, B)
    lens[0] = T
    lex = letters_lexicon(rng, Cn, 30, mode=mode, extra_spellings=3)
    check(emu, e, kind, lex, tw, lens, K=K, N=N, lm_weight=0.7, word_bonus=1.0, frac=0.3)


@pytest.mark.parametrize("kind", [CTC, ASG])
def test_token_pruning_and_colliding_hashes(emu, kind):
    rng = np.random.default_rng(410 + kind)
    B, T, Cn = 6, 20, 10
    e, tw = peaked(rng, kind, B, T, Cn)
    lex = letters_lexicon(rng, Cn, 40)
    got, _, _ = check(emu, e, kind, lex, tw, K=8, N=4, lm_weight=0.5, word_bonus=0.5, P=4, frac=0.3)
    for kw in (dict(collide=True), dict(hmul=0)):
        other = run(emu, e, kind, lex, tw, K=8, N=4, lm_weight=0.5, word_bonus=0.5, P=4, **kw)
        for k in got:
            assert np.array_equal(got[k].view(np.int32), other[k].view(np.int32)), (kw, k)


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
def test_identity_lexicon_is_beam_decode(emu, kind):
    rng = np.random.default_rng(420 + kind)
    B, T, Cn = 8, 25, 7
    e, tw = tbe.case(rng, kind, B, T, Cn)
    lens = rng.integers(0, T + 1, B)
    cls, sp = lxo.identity(Cn, kind)
    lex = lxo.Lexicon(Cn, cls, sp, Cn)
    ref = tbe.run(_beam_emu(), e, kind, tw, lens, K=8, N=4)
    got = run(emu, e, kind, lex, tw, lens, K=8, N=4)
    for k in ("tokens", "lengths", "scores", "status"):
        assert np.array_equal(ref[k], got[k]), k
    live = got["lengths"] >= 0
    assert np.array_equal(got["counts"][live], got["lengths"][live])
    assert np.array_equal(got["words"], got["tokens"])


def _beam_emu():
    lib = C_.CDLL(emu_build.build("beam", ["k_beam.cu"]))
    lib.emu_beam.argtypes = [C_.c_int, C_.c_int, C_.c_int, vp, C_.c_int, vp, C_.c_int, vp, C_.c_int, C_.c_int,
                             C_.c_int, C_.c_int, vp, vp, vp, vp]
    return lib


def test_fewer_transcripts_than_n_empty_utterance_and_flags(emu):
    rng = np.random.default_rng(430)
    Cn = 5
    # a lexicon of two one-letter words: few transcripts in 3 frames
    cls = [lxo.IN_WORD] * Cn
    cls[4] = lxo.SEPARATOR
    lex = lxo.Lexicon(Cn, cls, [((1,), 0), ((2,), 1)], 2, word_lm(rng, 2, order=2, n_tokens=200))
    e, _ = tbe.case(rng, CTC, 4, 3, Cn)
    e[1, 1, 2] = np.nan
    got, want, _ = check(emu, e, CTC, lex, lens=[3, 3, 4, 0], K=16, N=16, frac=0.0)
    assert got["status"][1] == 1 and got["status"][2] == 2
    for b in (1, 2):
        assert (got["counts"][b] == -1).all() and (got["words"][b] == -1).all() and np.isnan(got["lm"][b]).all()
    assert 0 < (got["lengths"][0] >= 0).sum() < 16
    assert got["lengths"][3, 0] == 0 and got["counts"][3, 0] == 0 and (got["lengths"][3, 1:] == -1).all()
    assert np.isclose(got["lm"][3, 0], lex.lm.end(lex.lm.start))


@pytest.mark.parametrize("kind", [CTC, ASG])
def test_dropped_inside_a_word_and_all_forbidden(emu, kind):
    rng = np.random.default_rng(440 + kind)
    Cn, T = 6, 6
    cls = [lxo.IN_WORD] * Cn
    cls[5] = lxo.SEPARATOR
    # the only word is 1 2 3 4: in 3 frames a beam that began it is still inside it and is dropped at the end, so
    # only separators survive
    lex = lxo.Lexicon(Cn, cls, [((1, 2, 3, 4), 0)], 1)
    e, tw = tbe.case(rng, kind, 3, T, Cn)
    e[:2, :, 1] += 30.0  # (the word's first token is by far the likeliest)
    got, want, _ = check(emu, e, kind, lex, tw, lens=[3, 3, 6], K=8, N=2, frac=0.0)
    live = got["lengths"][:2] >= 0
    assert live.any() and (got["counts"][:2][live] == 0).all()
    assert all(set(got["tokens"][b, n, :got["lengths"][b, n]]) <= {5} for b in range(2) for n in range(2)
               if live[b, n])
    # a lexicon whose single word is forbidden by its LM weight: only transcripts without a word remain
    G = dict(flags=np.array([1], np.uint8), src=np.array([0, 0], np.int32), dst=np.array([0, 0], np.int32),
             ilabel=np.array([0, 1], np.int32), olabel=np.array([0, 1], np.int32))
    lm = blo.LM(G, np.array([-np.inf, -1.0], np.float32), 1)
    lex2 = lxo.Lexicon(Cn, cls, [((1,), 0), ((2,), 0)], 1, lm)
    got, want, _ = check(emu, e, kind, lex2, tw, K=8, N=2, frac=0.0)
    live = got["lengths"] >= 0
    assert (got["counts"][live] == 0).all()


@pytest.mark.parametrize("kind", [CTC, BIGRAM])
def test_full_depth_backoff_chains(emu, kind):
    rng = np.random.default_rng(450 + kind)
    Cn = 8
    cls, sp = lxo.random_lexicon(rng, Cn, 12, sep=Cn - 1, max_len=2)
    V = 12
    # a 5-gram counted from a short corpus: histories back off through every order down to the root
    G, w = bko.backoff_ngram(rng, V, 5, n_tokens=400, min_count=1)
    lm = blo.LM(G, w, V)
    depth = max(_depth(lm, s) for s in range(lm.S))
    assert depth >= 3
    lex = lxo.Lexicon(Cn, cls, sp, V, lm)
    e, tw = peaked(rng, kind, 6, 25, Cn)
    check(emu, e, kind, lex, tw, K=8, N=3, lm_weight=1.0, word_bonus=0.5, frac=0.3)


def _depth(lm, s):
    d = 0
    while s in lm.eps:
        s = int(lm.dst[lm.eps[s]])
        d += 1
    return d


@pytest.mark.parametrize("dtype", [BF16, F16])
def test_half_emissions_are_the_widened_float32(emu, dtype):
    rng = np.random.default_rng(460 + dtype)
    B, T, Cn = 6, 20, 9
    e = tbe.emissions(rng, B, T, Cn, peak=8.0)
    if dtype == BF16:
        bits = (e.view(np.uint32) >> 16).astype(np.uint16)
        wide = (bits.astype(np.uint32) << 16).view(np.float32)
    else:
        bits = e.astype(np.float16).view(np.uint16)
        wide = bits.view(np.float16).astype(np.float32)
    lex = letters_lexicon(rng, Cn, 30, mode="start")
    got = run(emu, bits, CTC, lex, K=8, N=3, lm_weight=0.5, word_bonus=0.5, P=4, dtype=dtype)
    ref = run(emu, wide, CTC, lex, K=8, N=3, lm_weight=0.5, word_bonus=0.5, P=4)
    for k in ref:
        assert np.array_equal(ref[k], got[k]), k
    compare(got, lxo.batch(wide, CTC, None, None, 0, 8, 3, lex, 0.5, 0.5, 4))
