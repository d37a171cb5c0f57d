"""gtnb_lexicon_create / gtnb_beam_decode_lexicon_async and torch Lexicon / ctc_lexicon_beam_decode /
ngram_ctc_lexicon_beam_decode / asg_lexicon_beam_decode on the GPU:

- against the float64 restatement (tests/beam_lexicon_oracle.py) at B = 32, T = 200, C = 32, a seeded lexicon of
  about 2 000 words (letters with a separator; word-start tokens for ASG) with a backoff word trigram, K = 16, N = 4,
  for the three kinds, on every utterance whose decision margin exceeds 1e-3;
- the identity lexicon == ctc_beam_decode, ngram_ctc_beam_decode and asg_beam_decode for every dtype, and with a
  word LM equal to a token LM, lm_scores == the token-LM decoder's for every transcript both return;
- scores == am + (lm_weight * lm + word_bonus * words) recomputed in float32; words == a host segmentation of the
  tokens; two runs bit-identical; error codes; a launch profile without a copy, memset or allocation; sync-debug
  mode; a captured ctc_lexicon_beam_decode + edit_distance on word ids replayed == eager;
- a seeded quality check: the word error rate with the lexicon and word LM is below the one without an LM.
"""
import ctypes as C_
import os
import sys

import numpy as np
import pytest
import torch

from gtn_b200 import capi
from gtn_b200 import torch_loss as tl
from tests import backoff_oracle as bko
from tests import beam_lexicon_oracle as lxo
from tests import beam_lm_oracle as blo

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import bench_beam_decode as bbd  # noqa: E402  (the beam benchmark's seeded emissions)
import bench_beam_lm as bbl  # noqa: E402  (the LM benchmark's graphs)
import bench_beam_lexicon as bbx  # noqa: E402  (the lexicon benchmark's lexicons and quality workload)

L = capi.lib
KINDS = (capi.DENSE_CTC, capi.DENSE_BIGRAM, capi.DENSE_ASG)


@pytest.fixture(scope="module")
def ctx():
    c = capi.Ctx(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def letters():
    """C = 32 letters with "|" as separator, ~2 000 words and a backoff word trigram: (restatement, Lexicon)"""
    rng = np.random.default_rng(32)
    C, sep = 32, 31
    cls, sp = lxo.random_lexicon(rng, C, 2000, sep=sep, min_len=2, max_len=6, extra_spellings=50)
    V = 2000
    G, w = bko.backoff_ngram(rng, V, 3, n_tokens=20000, min_count=2)
    lm = blo.LM(G, w, V)
    return lxo.Lexicon(C, cls, sp, V, lm), tl.Lexicon(sp, C, V, separator=sep, lm=(G, w))


def decode(kind, e, w, lex, K, N, lw=1.0, wb=0.0, P=None, il=None):
    if kind == capi.DENSE_CTC:
        return tl.ctc_lexicon_beam_decode(e, lex, lw, wb, K, N, P, il)
    if kind == capi.DENSE_BIGRAM:
        return tl.ngram_ctc_lexicon_beam_decode(e, w, lex, lw, wb, K, N, P, il)
    return tl.asg_lexicon_beam_decode(e, w, lex, lw, wb, K, N, P, il)


@pytest.fixture(scope="module")
def pieces():
    """C = 32 with word-start tokens 24 .. 31 and no separator, ~2 000 words and a backoff word trigram"""
    rng = np.random.default_rng(33)
    C = 32
    cls, sp = lxo.random_lexicon(rng, C, 2000, word_start=range(24, C), min_len=2, max_len=5, extra_spellings=50)
    V = 2000
    G, w = bko.backoff_ngram(rng, V, 3, n_tokens=20000, min_count=2)
    return lxo.Lexicon(C, cls, sp, V, blo.LM(G, w, V)), tl.Lexicon(sp, C, V, word_start=range(24, C), lm=(G, w))


@pytest.mark.parametrize("kind", KINDS)
def test_against_restatement(kind, letters, pieces):
    # (ASG with a separator ties exactly at every repeated separator: it changes no lexicon state, and ASG's stay and
    # repeat score the same; word-start tokens change the state, as the token LM's tokens do)
    lex_r, lex = pieces if kind == capi.DENSE_ASG else letters
    B, T, Cn, K, N = 32, 200, 32, 16, 4
    e, w = bbx.spelled_inputs(np.random.default_rng(70 + kind), kind, lex_r, B, T)
    e, w = e * 10, None if w is None else w * 10  # (well separated decisions, as in test_gpu_beam_lm)
    il = torch.as_tensor(np.random.default_rng(7).integers(T // 2, T + 1, B).astype(np.int32)).cuda()
    lw, wb = 0.5, 1.0
    out = decode(kind, e, w, lex, K, N, lw, wb, None, il)
    want = lxo.batch(e.cpu().numpy(), kind, None if w is None else w.cpu().numpy(), il.cpu().numpy(), 0, K, N, lex_r,
                     lw, wb)
    ok = want["margin"] > 1e-3
    # (ASG's stay and repeat tie by construction, which puts more utterances within 1e-3)
    assert ok.mean() >= (0.3 if kind == capi.DENSE_ASG else 0.5), want["margin"]
    got = {k: getattr(out, k).cpu().numpy() for k in out._fields}
    for b in np.nonzero(ok)[0]:
        for k, kw in (("tokens", "tokens"), ("lengths", "lengths"), ("status", "status"), ("words", "words"),
                      ("word_counts", "counts")):
            assert np.array_equal(got[k][b], want[kw][b]), (k, b)
        for k, kw in (("scores", "scores"), ("am_scores", "am"), ("lm_scores", "lm")):
            fin = np.isfinite(want[kw][b])
            assert np.array_equal(np.isfinite(got[k][b]), fin), (k, b)
            assert np.allclose(got[k][b][fin], want[kw][b][fin], rtol=1e-4, atol=1e-4), (k, b)
    assert (got["word_counts"][:, 0] > 0).mean() > 0.9


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("kind", KINDS)
def test_identity_lexicon_is_beam_decode(kind, dtype):
    e, w = bbd.inputs(np.random.default_rng(80 + kind), kind, 32, 150, 40)
    e = e.to(dtype)
    cls, sp = lxo.identity(40, kind)
    lex = tl.Lexicon(sp, 40, 40, word_start=range(40))
    a = bbd.decode(kind, e, w, 16, 4)
    b = decode(kind, e, w, lex, 16, 4)
    for k in ("tokens", "lengths", "scores", "status"):
        assert torch.equal(getattr(a, k), getattr(b, k)), (kind, k)
    live = b.lengths >= 0
    assert torch.equal(b.words, b.tokens) and torch.equal(b.word_counts[live], b.lengths[live])


def test_word_lm_equal_to_a_token_lm():
    C = 64
    G, w = bko.backoff_lm(np.random.default_rng(24), C=C)
    cls, sp = lxo.identity(C, capi.DENSE_CTC)
    lex = tl.Lexicon(sp, C, C, word_start=range(C), lm=(G, w))
    lm = tl.LanguageModel(bbl.gtn_graph(G, w), C)
    e, _ = bbd.inputs(np.random.default_rng(3), capi.DENSE_CTC, 32, 20, C)  # (short: the two N-best lists overlap)
    a = tl.ctc_lm_beam_decode(e, lm, 0.5, 0.0, 16, 16)
    b = tl.ctc_lexicon_beam_decode(e, lex, 0.5, 0.0, 16, 16)
    n = 0
    for u in range(32):
        la = {tuple(a.tokens[u, i, :a.lengths[u, i]].tolist()): a.lm_scores[u, i].item() for i in range(16)
              if a.lengths[u, i] >= 0}
        for i in range(16):
            y = tuple(b.tokens[u, i, :b.lengths[u, i]].tolist())
            if b.lengths[u, i] >= 0 and y in la:
                assert b.lm_scores[u, i].item() == la[y], (u, y)
                n += 1
    assert n > 32


@pytest.mark.parametrize("kind", KINDS)
def test_scores_identity_words_and_reruns(kind, letters):
    lex_r, lex = letters
    e, w = bbx.spelled_inputs(np.random.default_rng(90 + kind), kind, lex_r, 48, 200)
    e[1, 7, 3] = float("nan")
    il = torch.full((48,), 200, dtype=torch.int32, device="cuda")
    il[2], il[3] = 201, 0
    for lw, wb, P in ((0.7, -0.3, None), (2.0, 1.5, 8)):
        out = decode(kind, e, w, lex, 16, 4, lw, wb, P, il)
        again = decode(kind, e, w, lex, 16, 4, lw, wb, P, il)
        for x, y in zip(out, again):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32))
        st = out.status.cpu().numpy()
        assert st[1] == 1 and st[2] == 2 and set(st[4:]) <= {0, 3}
        assert (out.word_counts[1:3] == -1).all() and (out.words[1:3] == -1).all()
        live = out.lengths >= 0
        want = out.am_scores + (lw * out.lm_scores + wb * out.word_counts.float())
        assert torch.equal(out.scores[live], want[live])
        tok, ln, wd, wc = (x.cpu().numpy() for x in (out.tokens, out.lengths, out.words, out.word_counts))
        for u in range(48):
            for n in range(4):
                if ln[u, n] >= 0:
                    seg = lex_r.segment(tok[u, n, :ln[u, n]])
                    assert seg is not None and wc[u, n] == len(seg) and list(wd[u, n, :len(seg)]) == seg
                    assert (wd[u, n, len(seg):] == -1).all()


def test_lexicon_checks_and_error_codes(ctx):
    C, V = 8, 5

    def create(cls, sp, V=V, C=C, G=None):
        toks = np.asarray([c for y, _ in sp for c in y], np.int32)
        offs = np.cumsum([0] + [len(y) for y, _ in sp]).astype(np.int32)
        words = np.asarray([x for _, x in sp], np.int32)
        cls = np.asarray(cls, np.int32)
        v = None
        if G is not None:
            v, keep = capi.make_view(G[0]["flags"], G[0]["src"], G[0]["dst"], G[0]["ilabel"], G[0]["olabel"], G[1])
        h = C_.c_void_p()
        rc = L().gtnb_lexicon_create(ctx.h, C, cls.ctypes.data, V, len(sp), offs.ctypes.data,
                                     toks.ctypes.data if len(toks) else None, words.ctypes.data,
                                     None if v is None else C_.byref(v), C_.byref(h))
        return rc, h

    cls = [0] * 7 + [1]
    good = [((1, 2), 0), ((1, 2, 3), 1), ((4,), 2), ((4, 5), 2)]
    rc, h = create(cls, good)
    assert rc == 0
    L().gtnb_lexicon_destroy(ctx.h, h)
    INV, UNS = capi.ERR_INVALID_ARGUMENT, capi.ERR_UNSUPPORTED
    for c2, sp in ((cls, good + [((1, 2), 3)]),  # two words share a spelling
                   (cls, good + [((7,), 3)]),  # a separator in a spelling
                   ([0] * 6 + [2, 1], good + [((1, 6), 3)]),  # a word-start token after position 0
                   (cls, good + [((), 3)]),  # an empty spelling
                   (cls, good + [((8,), 3)]),  # a token outside [0, C)
                   (cls, good + [((1,), 5)]),  # a word outside [0, V)
                   ([0] * 7 + [3], good)):  # a bad class
        assert create(c2, sp)[0] == INV, sp
    assert create([0] * 257, [((1,), 0)], C=257)[0] == UNS
    assert create(cls, good, V=(1 << 20) + 1)[0] == UNS
    G, w = bko.backoff_ngram(np.random.default_rng(3), V, 3)
    assert create(cls, good, G=(G, w))[0] == 0
    g = dict(G, ilabel=G["ilabel"].copy(), olabel=G["olabel"].copy())
    g["ilabel"][0] = g["olabel"][0] = V + 1
    assert create(cls, good, G=(g, w))[0] == INV  # a word LM label beyond V
    # the call
    lex = tl.Lexicon(good, C, V, separator=7, lm=(G, w))
    B, T = 4, 10
    n = C_.c_size_t()
    ctx._check(L().gtnb_beam_decode_lm_async_workspace(ctx.h, B, T, C, 0, capi.DENSE_CTC, 8, 2, C, C_.byref(n)))
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    e = torch.zeros((B, T, C), device="cuda")
    out = [torch.empty(s, dtype=dt, device="cuda") for s, dt in
           (((B, 2, T), torch.int32), ((B, 2), torch.int32), ((B, 2), torch.float32), ((B, 2), torch.float32),
            ((B, 2), torch.float32), ((B, 2, T), torch.int32), ((B, 2), torch.int32), ((B,), torch.int32))]

    def go(lx=lex.h, lw=1.0, wb=0.0, P=C, blank=0, Cn=C):
        return L().gtnb_beam_decode_lexicon_async(ctx.h, None, B, T, Cn, e.data_ptr(), 0, None, capi.DENSE_CTC, None,
                                                  blank, 8, 2, lx, lw, wb, P, *[o.data_ptr() for o in out],
                                                  ws.data_ptr(), n.value)
    assert go() == 0
    assert go(lw=-0.5) == INV and go(lw=float("nan")) == INV and go(lw=float("inf")) == INV
    assert go(wb=float("nan")) == INV and go(wb=float("-inf")) == INV
    assert go(lx=None) == INV
    assert go(Cn=C - 1) == INV  # a lexicon made for another C
    assert go(blank=1) == INV  # the blank is spelled
    assert go(blank=7) == INV  # the blank is the separator
    assert go(P=0) == UNS and go(P=C + 1) == UNS
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError):
        tl.Lexicon(good + [((1, 2), 3)], C, V, separator=7)


def test_launch_profile(ctx, letters):
    lex = letters[1]
    B, T, Cn = 8, 50, 32
    e = torch.randn((B, T, Cn), device="cuda")
    w = torch.randn(Cn + Cn * Cn, device="cuda")
    decode(capi.DENSE_ASG, e, w, lex, 16, 4, 0.5, 1.0, 16)
    torch.cuda.synchronize()
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    n = C_.c_size_t()
    ctx._check(L().gtnb_beam_decode_lm_async_workspace(ctx.h, B, T, Cn, 0, capi.DENSE_ASG, 16, 4, 16, C_.byref(n)))
    assert n.value <= ws.numel()
    out = [torch.empty(s, dtype=dt, device="cuda") for s, dt in
           (((B, 4, T), torch.int32), ((B, 4), torch.int32), ((B, 4), torch.float32), ((B, 4), torch.float32),
            ((B, 4), torch.float32), ((B, 4, T), torch.int32), ((B, 4), torch.int32), ((B,), torch.int32))]

    def go():
        return L().gtnb_beam_decode_lexicon_async(ctx.h, None, B, T, Cn, e.data_ptr(), 0, None, capi.DENSE_ASG,
                                                  w.data_ptr(), 0, 16, 4, lex.h, 0.5, 1.0, 16,
                                                  *[o.data_ptr() for o in out], ws.data_ptr(), n.value)
    assert go() == 0
    torch.cuda.synchronize()
    ctx.profile(True)
    ctx.profile_read()
    before = ctx.launches
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        assert go() == 0
        torch.cuda.synchronize()
    got = ctx.profile_read()
    ctx.profile(False)
    assert set(got) == {"beam_weights", "beam_decode_lexicon"} and ctx.launches - before == 2, got
    copies = [ev.name for ev in prof.events() if "Memcpy" in ev.name or "Memset" in ev.name or "alloc" in ev.name]
    assert not copies, copies


def test_no_wait_sync_debug_and_captured_step(letters):
    lex_r, lex = letters
    rng = np.random.default_rng(9)
    B, T = 32, 200
    e, _ = bbx.spelled_inputs(rng, capi.DENSE_CTC, lex_r, B, T)
    il = torch.as_tensor(rng.integers(T // 2, T + 1, B).astype(np.int32)).cuda()
    r = torch.as_tensor(rng.integers(0, 2000, (B, 40)).astype(np.int32)).cuda()
    rl = torch.as_tensor(rng.integers(0, 41, B).astype(np.int32)).cuda()

    def step():
        out = tl.ctc_lexicon_beam_decode(e, lex, 0.5, 1.0, 16, 4, 16, il)
        return out, tl.edit_distance(out.words[:, 0], out.word_counts[:, 0].clamp(min=0), r, rl)
    step()
    torch.cuda.synchronize()
    done = torch.cuda.Event()
    torch.cuda._sleep(100_000_000)
    step()
    done.record()
    assert not done.query(), "the call waited for the device"
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            cap = step()
    torch.cuda.current_stream().wait_stream(s)
    for seed in (1, 2):
        e.copy_(bbx.spelled_inputs(np.random.default_rng(seed), capi.DENSE_CTC, lex_r, B, T)[0])
        g.replay()
        eager = step()
        torch.cuda.synchronize()
        for c, w_ in zip(cap, eager):
            for x, y in zip(c, w_):
                assert (x is None and y is None) or torch.equal(x, y), seed
    del g
    with pytest.raises(RuntimeError):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            tl.Lexicon([((1,), 0)], 4, 1)


def test_word_lm_lowers_the_word_error_rate():
    q = bbx.quality_workload()
    ed = torch.as_tensor(q["e"]).cuda()
    no_lm = bbx.wer(tl.ctc_lexicon_beam_decode(ed, q["lex_nolm"], 0.0, 0.0, 8), q["refs"])
    fused = bbx.wer(tl.ctc_lexicon_beam_decode(ed, q["lex"], 1.0, 0.0, 8), q["refs"])
    assert fused < no_lm, (fused, no_lm)
