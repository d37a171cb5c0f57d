"""gtnb_beam_decode_chunk_async / torch StreamingBeamDecoder on the GPU.

The streaming decoder's outputs at END are == the shipped one-shot async calls (ctc / ngram_ctc / asg, _lm_ and
_lexicon_beam_decode) on the frames each row consumed, at realistic sizes: CTC B = 64, T = 300, C = 64; n-gram CTC and
ASG at C = 128; no LM, a backoff trigram LM with token pruning, and a lexicon with a word trigram.  Each configuration
is split several ways: one whole chunk, fixed chunks of 1, 7 and 32 frames, random chunk sizes, and a serving
schedule where rows start and end at different steps.  Also: a captured step replayed over every chunk == eager
steps; the call does not wait for the device and runs under sync-debug "error"; the launch profile is one kernel per
chunk call with no copy or memset; create raises under capture; an LM or lexicon for another C is
GTNB_ERR_INVALID_ARGUMENT.
"""
import os
import sys

import numpy as np
import pytest
import torch

from gtn_b200 import capi
from gtn_b200 import torch_loss as tl
from tests import backoff_oracle as bko
from tests import beam_lexicon_oracle as lxo

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import bench_beam_decode as bbd  # noqa: E402  (the beam benchmark's seeded emissions)
import bench_beam_lm as bbl  # noqa: E402  (gtn graphs of LM arrays)

KIND = {capi.DENSE_CTC: "ctc", capi.DENSE_BIGRAM: "ngram_ctc", capi.DENSE_ASG: "asg"}


@pytest.fixture(scope="module")
def lms():
    out = {}
    for C in (64, 128):
        G, w = bko.backoff_lm(np.random.default_rng(C), C=C)
        out[C] = tl.LanguageModel(bbl.gtn_graph(G, w), C)
    return out


@pytest.fixture(scope="module")
def lexicons():
    """C = 64 and 128 letters with the last token as separator, ~2 000 words and a backoff word trigram"""
    out = {}
    for C in (64, 128):
        rng = np.random.default_rng(C + 7)
        cls, sp = lxo.random_lexicon(rng, C, 2000, sep=C - 1, min_len=2, max_len=6, extra_spellings=50)
        G, w = bko.backoff_ngram(rng, 2000, 3, n_tokens=20000, min_count=2)
        out[C] = tl.Lexicon(sp, C, 2000, separator=C - 1, lm=(G, w))
    return out


def oneshot(kind, e, w, lens, cfg):
    """the shipped one-shot call of a configuration"""
    name = KIND[kind]
    if cfg.get("lexicon") is not None:
        fn = getattr(tl, name + "_lexicon_beam_decode")
        args = (e, cfg["lexicon"]) if kind == capi.DENSE_CTC else (e, w, cfg["lexicon"])
        return fn(*args, cfg["lm_weight"], cfg["bonus"], cfg["beam"], cfg["nbest"], cfg["token_beam"], lens)
    fn = getattr(tl, name + "_lm_beam_decode")
    args = (e,) if kind == capi.DENSE_CTC else (e, w)
    return fn(*args, cfg.get("lm"), cfg["lm_weight"], cfg["bonus"], cfg["beam"], cfg["nbest"], cfg["token_beam"], lens)


def decoder(kind, e, w, cfg):
    B, T, C = e.shape
    return tl.StreamingBeamDecoder(B, T, C, KIND[kind], w, lm=cfg.get("lm"), lexicon=cfg.get("lexicon"),
                                   lm_weight=cfg["lm_weight"], bonus=cfg["bonus"], beam=cfg["beam"],
                                   nbest=cfg["nbest"], token_beam=cfg["token_beam"])


def chunks(e, pos, n, Tc):
    """rows' next n[b] frames of e from pos[b], NaN-padded to [B, Tc, C]"""
    B, T, C = e.shape
    ep = torch.cat([e, torch.full((B, 1, C), float("nan"), device=e.device, dtype=e.dtype)], 1)
    j = torch.arange(Tc, device=e.device)
    p, m = torch.as_tensor(pos, device=e.device), torch.as_tensor(n, device=e.device)
    idx = torch.where(j[None] < m[:, None], p[:, None] + j[None], T)
    return ep[torch.arange(B, device=e.device)[:, None], idx]


def run_schedule(dec, e, lens, plan, start=None, reset_first=False):
    """Feed each row its lens[b] frames, step i taking plan(i) frames at most, row b from step start[b]; END on the
    chunk that takes its last frame (reset_first: RESET on step 0).  -> the final results of every row (copied at its
    END step)"""
    B = e.shape[0]
    start = np.zeros(B, np.int64) if start is None else start
    pos = np.zeros(B, np.int64)
    done = np.zeros(B, bool)
    fields = dec.results._fields
    out = {k: torch.empty_like(getattr(dec.results, k)) for k in fields}
    i = 0
    while not done.all():
        Tc = plan(i)
        live = (start <= i) & ~done
        n = np.where(live, np.minimum(Tc, lens - pos), 0)
        end = live & (pos + n == lens)
        dec.step(chunks(e, pos, n, Tc), torch.as_tensor(n.astype(np.int32), device=e.device),
                 end=torch.as_tensor(end, device=e.device),
                 reset=torch.full((B,), i == 0, device=e.device) if reset_first else None)
        if end.any():
            m = torch.as_tensor(end, device=e.device)
            for k in fields:
                out[k][m] = getattr(dec.results, k)[m]
        pos += n
        done |= end
        i += 1
    return out


def assert_equal(got, want):
    for k in want._fields:
        x, y = got[k], getattr(want, k)
        assert x.shape == y.shape and torch.equal(x.view(torch.int32), y.view(torch.int32)), k


CONFIGS = [
    ("ctc_lm", capi.DENSE_CTC, 64, 300, 64, dict(lm="lm", lm_weight=0.5, bonus=0.5, beam=16, nbest=4, token_beam=16)),
    ("ctc_plain", capi.DENSE_CTC, 64, 300, 64, dict(lm_weight=1.0, bonus=0.0, beam=8, nbest=2, token_beam=None)),
    ("bigram_lm", capi.DENSE_BIGRAM, 32, 200, 128, dict(lm="lm", lm_weight=0.5, bonus=0.2, beam=16, nbest=3,
                                                        token_beam=32)),
    ("asg_lm", capi.DENSE_ASG, 32, 200, 128, dict(lm="lm", lm_weight=0.5, bonus=0.2, beam=16, nbest=3,
                                                  token_beam=32)),
    ("ctc_lexicon", capi.DENSE_CTC, 64, 300, 64, dict(lexicon="lex", lm_weight=0.7, bonus=1.0, beam=16, nbest=4,
                                                      token_beam=24)),
    ("asg_lexicon", capi.DENSE_ASG, 32, 200, 128, dict(lexicon="lex", lm_weight=0.7, bonus=1.0, beam=16, nbest=3,
                                                       token_beam=32)),
]


@pytest.mark.parametrize("name,kind,B,T,C,cfg", CONFIGS, ids=list(next(zip(*CONFIGS))))
def test_chunked_equals_oneshot(lms, lexicons, name, kind, B, T, C, cfg):
    cfg = dict(cfg)
    if cfg.get("lm"):
        cfg["lm"] = lms[C]
    if cfg.get("lexicon"):
        cfg["lexicon"] = lexicons[C]
    rng = np.random.default_rng(sum(map(ord, name)))
    e, w = bbd.inputs(rng, kind, B, T, C)
    lens = rng.integers(0, T + 1, B)
    lens[0], lens[1] = T, 0
    want = oneshot(kind, e, w, torch.as_tensor(lens.astype(np.int32), device="cuda"), cfg)
    sizes = rng.integers(0, 40, 10_000)
    plans = [lambda i: T, lambda i: 1, lambda i: 7, lambda i: 32, lambda i: int(sizes[i])]
    for plan in plans:
        dec = decoder(kind, e, w, cfg)
        assert_equal(run_schedule(dec, e, lens, plan), want)
    # serving: rows start at different steps, 16-frame chunks; the same decoder serves a second round of utterances
    dec = decoder(kind, e, w, cfg)
    for r in range(2):
        start = rng.integers(0, 12, B)
        assert_equal(run_schedule(dec, e, lens, lambda i: 16, start), want)


def test_half_emissions_and_reset(lms):
    rng = np.random.default_rng(5)
    B, T, C = 32, 120, 64
    e, _ = bbd.inputs(rng, capi.DENSE_CTC, B, T, C)
    cfg = dict(lm=lms[C], lm_weight=0.5, bonus=0.5, beam=16, nbest=2, token_beam=16)
    lens = rng.integers(0, T + 1, B)
    for dt in (torch.bfloat16, torch.float16):
        eh = e.to(dt)
        want = oneshot(capi.DENSE_CTC, eh, None, torch.as_tensor(lens.astype(np.int32), device="cuda"), cfg)
        dec = decoder(capi.DENSE_CTC, eh, None, cfg)
        # garbage first, discarded by a RESET at the first real chunk
        dec.step(torch.randn(B, 9, C, device="cuda").to(dt))
        assert_equal(run_schedule(dec, eh, lens, lambda i: 10, reset_first=True), want)


def test_captured_step_replays_the_eager_steps(lms):
    rng = np.random.default_rng(6)
    B, T, C, Tc = 64, 256, 64, 16
    e, _ = bbd.inputs(rng, capi.DENSE_CTC, B, T, C)
    cfg = dict(lm=lms[C], lm_weight=0.5, bonus=0.5, beam=16, nbest=2, token_beam=16)
    eager, capd = decoder(capi.DENSE_CTC, e, None, cfg), decoder(capi.DENSE_CTC, e, None, cfg)
    x = torch.zeros(B, Tc, C, device="cuda")
    n = torch.zeros(B, dtype=torch.int32, device="cuda")
    end = torch.zeros(B, dtype=torch.bool, device="cuda")
    lens = rng.integers(T // 2, T + 1, B)
    # warm-up outside capture (a row with no frames and no flag is untouched)
    capd.step(x, n, end=end)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            best = capd.step(x, n, end=end)
    torch.cuda.current_stream().wait_stream(s)
    pos = np.zeros(B, np.int64)
    for i in range(T // Tc):
        k = np.minimum(Tc, lens - pos)
        fin = pos + k == lens
        xc = chunks(e, pos, k, Tc)
        x.copy_(xc)
        n.copy_(torch.as_tensor(k.astype(np.int32)))
        end.copy_(torch.as_tensor(fin & (k > 0)))
        g.replay()
        want = eager.step(xc, n.clone(), end=end.clone())
        torch.cuda.synchronize()
        for a, b in zip(best, want):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), i
        for f in capd.results._fields:
            assert torch.equal(getattr(capd.results, f).view(torch.int32), getattr(eager.results, f).view(torch.int32))
        pos += k
    del g


def test_no_wait_sync_debug_and_launch_profile(lms, lexicons):
    rng = np.random.default_rng(7)
    B, T, C, Tc = 64, 300, 64, 32
    e, _ = bbd.inputs(rng, capi.DENSE_CTC, B, T, C)
    for cfg, prof_name in ((dict(lm=lms[C], lm_weight=0.5, bonus=0.5, beam=16, nbest=2, token_beam=16),
                            "beam_chunk_lm"),
                           (dict(lexicon=lexicons[C], lm_weight=0.5, bonus=0.5, beam=16, nbest=2, token_beam=16),
                            "beam_chunk_lexicon")):
        dec = decoder(capi.DENSE_CTC, e, None, cfg)
        x = e[:, :Tc].contiguous()
        n = torch.full((B,), Tc, dtype=torch.int32, device="cuda")
        dec.step(x, n)
        torch.cuda.synchronize()
        done = torch.cuda.Event()
        torch.cuda._sleep(100_000_000)
        dec.step(x, n)
        done.record()
        assert not done.query(), "the call waited for the device"
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            dec.step(x, n, end=torch.ones(B, dtype=torch.bool, device="cuda"))
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        # the C call alone: one kernel per chunk call, no copy or memset
        ctl = torch.full((B,), capi.BEAM_END, dtype=torch.int32, device="cuda")
        r = dec.results
        lex = cfg.get("lexicon") is not None

        def go(c):
            return capi.lib().gtnb_beam_decode_chunk_async(
                dec._g.h, None, dec.h, Tc, x.data_ptr(), 0, n.data_ptr(), c, r.tokens.data_ptr(),
                r.lengths.data_ptr(), r.scores.data_ptr(), r.am_scores.data_ptr(), r.lm_scores.data_ptr(),
                r.words.data_ptr() if lex else None, r.word_counts.data_ptr() if lex else None, r.status.data_ptr(),
                dec.best_tokens.data_ptr(), dec.best_lengths.data_ptr(), dec.best_scores.data_ptr())
        g = dec._g
        g.profile(True)
        g.profile_read()
        before = g.launches
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            assert go(None) == 0
            assert go(ctl.data_ptr()) == 0
            torch.cuda.synchronize()
        got = g.profile_read()
        g.profile(False)
        assert set(got) == {prof_name} and g.launches - before == 2, got
        copies = [ev.name for ev in prof.events() if "Memcpy" in ev.name or "Memset" in ev.name or "alloc" in ev.name]
        assert not copies, copies


def test_create_raises_under_capture_and_argument_errors(lms, lexicons):
    C = 64
    with pytest.raises(RuntimeError):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            tl.StreamingBeamDecoder(4, 10, C)
    for kw in (dict(lm=lms[128]), dict(lexicon=lexicons[128])):
        with pytest.raises(capi.GtnbError) as ex:
            tl.StreamingBeamDecoder(4, 10, C, **kw)
        assert ex.value.code == capi.ERR_INVALID_ARGUMENT
    with pytest.raises(capi.GtnbError) as ex:
        tl.StreamingBeamDecoder(4, 10, C, lm=lms[C], lexicon=lexicons[C])
    assert ex.value.code == capi.ERR_INVALID_ARGUMENT
    with pytest.raises(capi.GtnbError) as ex:
        tl.StreamingBeamDecoder(4, 10, C, beam=65)
    assert ex.value.code == capi.ERR_UNSUPPORTED
    dec = tl.StreamingBeamDecoder(4, 10, C)
    with pytest.raises(ValueError):
        dec.step(torch.zeros(4, 3, C + 1, device="cuda"))
    # the C call: the best outputs all or none, word outputs without a lexicon
    r = dec.results
    base = [dec._g.h, None, dec.h, 0, None, 0, None, None, r.tokens.data_ptr(), r.lengths.data_ptr(),
            r.scores.data_ptr(), None, None, None, None, None]
    assert capi.lib().gtnb_beam_decode_chunk_async(*base, dec.best_tokens.data_ptr(), None, None) == \
        capi.ERR_INVALID_ARGUMENT
    bad = list(base)
    bad[13] = r.tokens.data_ptr()
    assert capi.lib().gtnb_beam_decode_chunk_async(*bad, None, None, None) == capi.ERR_INVALID_ARGUMENT
    assert capi.lib().gtnb_beam_decode_chunk_async(*base, None, None, None) == 0
    if torch.cuda.device_count() > 1:
        other = capi.Ctx(1)
        assert capi.lib().gtnb_beam_decode_chunk_async(other.h, *base[1:], None, None, None) == \
            capi.ERR_INVALID_ARGUMENT
        other.close()
