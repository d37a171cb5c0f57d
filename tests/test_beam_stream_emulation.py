"""k_beam.cu's beam_chunk_kernel (gtnb_beam_decode_chunk_async) from source on the CPU, through the SIMT emulator of
tests/emu (tests/emu/beam_stream_emu.cpp), against the emulated one-shot kernel (tests/emu/beam_emu.cpp) on the
concatenated frames.

The spec of the streaming decoder is that chunking changes nothing: the outputs a row gets at END are == bit for bit
to the one-shot call on the frames it consumed since its previous END or RESET, padded to T_max with that many
frames, whatever the split.  Each schedule here is driven by a host model of the rows (frames since the last restart,
the sticky invalid flag), and after every step:
- a row with END gets exactly the one-shot outputs (or, flagged invalid, status 2 with NaN scores and -1 rows); every
  other row's final outputs are left unwritten;
- a row with frames or control bits gets its best beam: the one-shot call's top hypothesis at the frames so far,
  exactly, where the final ranking is the key ranking (no LM, an LM without end-of-sentence arcs, or the identity
  lexicon);
- a row with zero frames and no control bits keeps its best outputs.
Chunk padding is NaN, so a frame read outside a row's chunk would flag it.
"""
import ctypes as C_

import numpy as np
import pytest

from tests import beam_lexicon_oracle as lxo
from tests import beam_oracle as bo
from tests import emu_build
from tests import test_beam_emulation as tbe
from tests import test_beam_lexicon_emulation as tlx
from tests import test_beam_lm_emulation as tlm

vp = C_.c_void_p
CTC, BIGRAM, ASG = bo.CTC, bo.BIGRAM, bo.ASG
F32, BF16, F16 = 0, 1, 2
RESET, END = 1, 2
SENT = 77


@pytest.fixture(scope="module")
def libs():
    s = C_.CDLL(emu_build.build("beam_stream", ["k_beam.cu"]))
    s.emu_beam_state_words.restype = C_.c_longlong
    s.emu_beam_state_words.argtypes = [C_.c_int] * 3
    s.emu_beam_chunk_lm.argtypes = ([C_.c_int] * 4 + [vp, C_.c_int, vp, vp, C_.c_int, vp] + [C_.c_int] * 3 +
                                    [vp, vp, C_.c_int, C_.c_float, C_.c_float, C_.c_int, C_.c_int] + [vp] * 11)
    s.emu_beam_chunk_lexicon.argtypes = ([C_.c_int] * 4 + [vp, C_.c_int, vp, vp, C_.c_int, vp] + [C_.c_int] * 3 +
                                         [vp] * 6 + [C_.c_ulonglong, C_.c_int, vp, vp, vp, C_.c_int, C_.c_float,
                                                     C_.c_float, C_.c_int, C_.c_int] + [vp] * 13)
    o = C_.CDLL(emu_build.build("beam", ["k_beam.cu"]))
    o.emu_beam_lm.argtypes = [C_.c_int, C_.c_int, C_.c_int, vp, C_.c_int, vp, C_.c_int, vp, C_.c_int, C_.c_int,
                              C_.c_int, vp, vp, C_.c_int, C_.c_float, C_.c_float, C_.c_int, C_.c_int, vp, vp, vp, vp,
                              vp, vp]
    o.emu_beam_lexicon.argtypes = ([C_.c_int] * 3 + [vp, C_.c_int, vp, C_.c_int, vp] + [C_.c_int] * 3 + [vp] * 6 +
                                   [C_.c_ulonglong, C_.c_int, vp, vp, vp, C_.c_int, C_.c_float, C_.c_float,
                                    C_.c_int, C_.c_int] + [vp] * 8)
    return s, o


def _p(a):
    return None if a is None else a.ctypes.data


def to_dtype(x, dtype):
    """float32 -> the bits the kernels read for dtype (NaN stays NaN)"""
    if dtype == BF16:
        return (np.ascontiguousarray(x, np.float32).view(np.uint32) >> 16).astype(np.uint16)
    if dtype == F16:
        return x.astype(np.float16).view(np.uint16)
    return np.ascontiguousarray(x, np.float32)


class Config:
    """One decoder configuration: policy "lm" (lm a beam_lm_oracle.LM or None) or "lex" (lex a
    beam_lexicon_oracle.Lexicon)"""

    def __init__(self, kind, C, tw=None, K=4, N=3, P=None, blank=0, lm=None, lex=None, alpha=1.0, beta=0.0,
                 collide=False, dtype=F32):
        self.kind, self.C, self.tw, self.K, self.N, self.blank = kind, C, tw, K, N, blank
        self.P = C if P is None else P
        self.lm, self.lex, self.alpha, self.beta, self.collide, self.dtype = lm, lex, alpha, beta, collide, dtype
        self.table = tlm.table(lm) if lm is not None else (None, None)
        self.dev = tlx.device_arrays(lex) if lex is not None else None

    def oneshot(self, libs, e, lens):
        """the one-shot kernel on e [B][T_max][C] (float32) with input lengths lens"""
        o = libs[1]
        bits = to_dtype(e, self.dtype)
        if self.lex is None:
            return tlm.run(o, bits, self.kind, self.tw, lens, self.blank, self.K, self.N, self.lm, self.alpha,
                           self.beta, self.P, collide=self.collide, dtype=self.dtype)
        return tlx.run(o, bits, self.kind, self.lex, self.tw, lens, self.blank, self.K, self.N, self.alpha,
                       self.beta, self.P, collide=self.collide, dtype=self.dtype)


class Stream:
    """the decoder's device state on the host, and one chunk call"""

    def __init__(self, libs, cfg, B, T):
        self.lib, self.cfg, self.B, self.T = libs[0], cfg, B, T
        words = self.lib.emu_beam_state_words(int(cfg.lex is not None), cfg.K, cfg.C)
        self.state = np.zeros((B, words), np.uint32)
        self.bp = np.full((B, T, cfg.K), 0xFFFF, np.uint16)
        self.best = dict(tokens=np.full((B, T), SENT, np.int32), lengths=np.full(B, SENT, np.int32),
                         scores=np.full(B, SENT, np.float32))

    def step(self, e, lens, control, best=True):
        cfg, B, T, N = self.cfg, self.B, self.T, self.cfg.N
        Tc = e.shape[1]
        out = dict(tokens=np.full((B, N, T), SENT, np.int32), lengths=np.full((B, N), SENT, np.int32),
                   scores=np.full((B, N), SENT, np.float32), am=np.full((B, N), SENT, np.float32),
                   lm=np.full((B, N), SENT, np.float32), status=np.full(B, SENT, np.int32))
        bits = to_dtype(e, cfg.dtype)
        ln = None if lens is None else np.ascontiguousarray(lens, np.int32)
        ct = None if control is None else np.ascontiguousarray(control, np.int32)
        tw = None if cfg.tw is None else np.ascontiguousarray(cfg.tw, np.float32)
        bt = [_p(self.best[k]) for k in ("tokens", "lengths", "scores")] if best else [None] * 3
        if cfg.lex is None:
            lw, ld = cfg.table
            rc = self.lib.emu_beam_chunk_lm(
                B, T, cfg.C, Tc, _p(bits), cfg.dtype, _p(ln), _p(ct), cfg.kind, _p(tw), cfg.blank, cfg.K, N, _p(lw),
                _p(ld), cfg.lm.start if cfg.lm is not None else 0, cfg.alpha, cfg.beta, cfg.P, int(cfg.collide),
                _p(self.state), _p(self.bp), *[_p(out[k]) for k in ("tokens", "lengths", "scores", "am", "lm",
                                                                    "status")], *bt)
        else:
            d = cfg.dev
            out.update(words=np.full((B, N, T), SENT, np.int32), counts=np.full((B, N), SENT, np.int32))
            rc = self.lib.emu_beam_chunk_lexicon(
                B, T, cfg.C, Tc, _p(bits), cfg.dtype, _p(ln), _p(ct), cfg.kind, _p(tw), cfg.blank, cfg.K, N,
                _p(d["cls"]), _p(d["mask"]), _p(d["first"]), _p(d["word"]), _p(d["smear"]), _p(d["hash"]), d["hmul"],
                d["hbits"], _p(d["bow"]), _p(d["bod"]), _p(d["endw"]), d["start"], cfg.alpha, cfg.beta, cfg.P,
                int(cfg.collide), _p(self.state), _p(self.bp),
                *[_p(out[k]) for k in ("tokens", "lengths", "scores", "am", "lm", "words", "counts", "status")], *bt)
        emu_build.check(rc)
        return out


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.int32) if a.dtype == np.float32 else a,
                                                 b.view(np.int32) if b.dtype == np.float32 else b)


def drive(libs, cfg, T, events, frames, best="exact"):
    """Run a schedule.  events[b]: the row's chunks, (n, control) each, n frames taken in order from frames[b]
    ([frames, C] float32; n outside [0, Tc] is passed as is and takes no frames); steps run until every row is done.
    best: "exact" (== the one-shot top hypothesis) or None (no trace).  Returns the number of END outputs and best beams checked."""
    B, C = len(events), cfg.C
    st = Stream(libs, cfg, B, T)
    pos = [0] * B
    cur = [[] for _ in range(B)]
    inv = [False] * B
    checked = [0, 0]
    for i in range(max(len(ev) for ev in events)):
        step = [ev[i] if i < len(ev) else (0, 0) for ev in events]
        Tc = max([n for n, _ in step if 0 <= n <= T + 8] + [0]) + int(i % 3 == 1)
        e = np.full((B, Tc, C), np.nan, np.float32)
        lens = np.zeros(B, np.int32)
        ctl = np.zeros(B, np.int32)
        ended = []
        for b, (n, c) in enumerate(step):
            lens[b], ctl[b] = n, c
            if c & RESET:
                cur[b], inv[b] = [], False
            if not 0 <= n <= Tc:
                inv[b] = True
                continue
            e[b, :n] = frames[b][pos[b]:pos[b] + n]
            pos[b] += n
            if len(cur[b]) + n > T:
                inv[b] = True
            if not inv[b]:
                cur[b].extend(e[b, :n])
        prev_best = {k: v.copy() for k, v in st.best.items()}
        got = st.step(e, lens if i % 4 != 3 or not (lens == Tc).all() else None,
                      ctl if ctl.any() or i % 2 else None, best=best is not None)
        # the one-shot call on each row's frames so far
        ref_e = np.zeros((B, T, C), np.float32)
        ref_len = np.zeros(B, np.int32)
        for b in range(B):
            if not inv[b]:
                ref_len[b] = len(cur[b])
                if cur[b]:
                    ref_e[b, :len(cur[b])] = np.asarray(cur[b])
        want = cfg.oneshot(libs, ref_e, ref_len)
        touched = [(n != 0 or c != 0) for n, c in step]
        for b, (n, c) in enumerate(step):
            if c & END:
                checked[0] += 1
                if inv[b]:
                    assert got["status"][b] == 2, (i, b, got["status"][b])
                    assert np.isnan(got["scores"][b]).all() and (got["lengths"][b] == -1).all()
                    assert (got["tokens"][b] == -1).all()
                else:
                    for k in want:
                        if k != "margin":
                            assert same(got[k][b], want[k][b]), (i, b, k, got[k][b], want[k][b])
            else:
                for k in got:
                    assert (got[k][b] == SENT).all(), (i, b, k)
            if best is None:
                continue
            if not touched[b]:
                for k in st.best:
                    assert same(st.best[k][b], prev_best[k][b]), (i, b, k)
                continue
            L = st.best["lengths"][b]
            if inv[b]:
                assert L == -1 and np.isnan(st.best["scores"][b]) and (st.best["tokens"][b] == -1).all()
            elif best == "exact":
                checked[1] += 1
                assert L == want["lengths"][b, 0], (i, b, L, want["lengths"][b])
                assert same(st.best["tokens"][b], want["tokens"][b, 0]), (i, b, st.best["tokens"][b])
                assert same(st.best["scores"][b], want["scores"][b, 0]), (i, b, st.best["scores"][b],
                                                                          want["scores"][b])
        for b, (n, c) in enumerate(step):
            if c & END:
                cur[b], inv[b] = [], False
    return checked


def split(rng, n, zeros=True):
    """n frames in random pieces of 0 .. 5 frames (the last piece takes the rest)"""
    out = []
    while n > 0:
        k = int(rng.integers(0 if zeros else 1, 6))
        out.append(min(k, n))
        n -= out[-1]
    if not out or (zeros and rng.random() < 0.3):
        out.append(0)
    return out


def schedule(rng, B, T, utts=(1, 3), reset=0.0):
    """each row: utts[0] .. utts[1] - 1 utterances of 0 .. T frames, each split at random and ended by END on its last
    piece (with probability reset, a RESET on one piece)"""
    events = []
    for b in range(B):
        ev = []
        for _ in range(int(rng.integers(*utts))):
            n = int(rng.integers(0, T + 1)) if b else T
            pieces = split(rng, n)
            ctl = [0] * len(pieces)
            if rng.random() < reset:
                ctl[int(rng.integers(0, len(pieces)))] |= RESET
            ctl[-1] |= END
            ev.extend(zip(pieces, ctl))
        events.append(ev)
    return events


def frames_for(rng, cfg, B, T, n_extra=40):
    e, _ = tbe.case(rng, cfg.kind, B, 3 * T + n_extra, cfg.C)
    return [e[b] for b in range(B)]


def lm_config(rng, kind, C, which, **kw):
    tw = tbe.weights(rng, kind, C) if kind != CTC else None
    if which == "plain":
        return Config(kind, C, tw, **kw)
    lm = tlm.make_lm(rng, C, eos=which == "lm_eos")[0]
    return Config(kind, C, tw, lm=lm, alpha=0.5, beta=0.75, **kw)


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
@pytest.mark.parametrize("which", ["plain", "lm", "lm_eos"])
def test_random_splits_lm_policy(libs, kind, which):
    rng = np.random.default_rng(900 + 10 * kind + len(which))
    B, T, C = 5, 14, 6
    cfg = lm_config(rng, kind, C, which, K=4, N=3, P=C if which == "plain" else 4)
    events = schedule(rng, B, T, reset=0.3)
    ends, bests = drive(libs, cfg, T, events, frames_for(rng, cfg, B, T), best="exact" if which != "lm_eos" else None)
    assert ends >= B and (which == "lm_eos" or bests > 10)


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
def test_one_frame_chunks_and_one_whole_chunk(libs, kind):
    rng = np.random.default_rng(950 + kind)
    B, T, C = 3, 10, 5
    cfg = lm_config(rng, kind, C, "lm", K=4, N=2)
    frames = frames_for(rng, cfg, B, T)
    ones = [[(1, 0)] * (T - 1) + [(1, END)] for _ in range(B)]
    whole = [[(T, END)] for _ in range(B)]
    for events in (ones, whole):
        drive(libs, cfg, T, events, frames)


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
@pytest.mark.parametrize("mode", ["sep", "start"])
def test_random_splits_lexicon_policy(libs, kind, mode):
    rng = np.random.default_rng(960 + 10 * kind + (mode == "sep"))
    B, T, C = 4, 12, 8
    lex = tlx.letters_lexicon(rng, C, 24, mode=mode, extra_spellings=2)
    tw = tbe.weights(rng, kind, C) if kind != CTC else None
    cfg = Config(kind, C, tw, K=4, N=3, P=6, lex=lex, alpha=0.7, beta=1.0)
    e, _ = tlx.peaked(rng, kind, B, 3 * T + 40, C)
    events = schedule(rng, B, T, reset=0.3)
    ends, _ = drive(libs, cfg, T, events, [e[b] for b in range(B)], best=None)
    assert ends >= B


@pytest.mark.parametrize("kind", [CTC, ASG])
def test_identity_lexicon_best_beam(libs, kind):
    """with the identity lexicon the key ranking is the plain search's, so the best beam is exact there too"""
    rng = np.random.default_rng(970 + kind)
    B, T, C = 4, 12, 6
    cls, sp = lxo.identity(C, kind)
    lex = lxo.Lexicon(C, cls, sp, C)
    tw = tbe.weights(rng, kind, C) if kind != CTC else None
    cfg = Config(kind, C, tw, K=4, N=2, lex=lex)
    ends, bests = drive(libs, cfg, T, schedule(rng, B, T, reset=0.3), frames_for(rng, cfg, B, T))
    assert bests > 10


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("policy", ["lm", "lex"])
def test_half_emissions(libs, dtype, policy):
    rng = np.random.default_rng(980 + dtype + 5 * (policy == "lex"))
    B, T, C = 4, 12, 8
    if policy == "lm":
        cfg = lm_config(rng, BIGRAM, C, "lm", K=4, N=2, P=5, dtype=dtype)
        best = "exact"
    else:
        lex = tlx.letters_lexicon(rng, C, 20)
        cfg = Config(ASG, C, tbe.weights(rng, ASG, C), K=4, N=2, lex=lex, alpha=0.5, beta=0.5, dtype=dtype)
        best = None
    drive(libs, cfg, T, schedule(rng, B, T), frames_for(rng, cfg, B, T), best=best)


@pytest.mark.parametrize("policy", ["lm", "lex"])
def test_colliding_hash(libs, policy):
    rng = np.random.default_rng(990 + (policy == "lex"))
    B, T, C = 4, 14, 5
    if policy == "lm":
        cfg = lm_config(rng, CTC, C, "lm", K=8, N=4, P=3, collide=True)
    else:
        lex = tlx.letters_lexicon(rng, C, 12)
        cfg = Config(CTC, C, None, K=8, N=4, lex=lex, alpha=0.5, beta=0.5, collide=True)
    drive(libs, cfg, T, schedule(rng, B, T, reset=0.2), frames_for(rng, cfg, B, T),
          best="exact" if policy == "lm" else None)


@pytest.mark.parametrize("kind", [CTC, BIGRAM, ASG])
def test_flags_stay_on_their_row(libs, kind):
    """END after 0 frames, RESET | END on one chunk, a row pushed past T_max, an out-of-range chunk length and a NaN in
    a late chunk: each flags its own row only (status 2, or the one-shot call's status 1)"""
    rng = np.random.default_rng(1000 + kind)
    B, T, C = 6, 10, 5
    cfg = lm_config(rng, kind, C, "lm", K=4, N=2)
    frames = frames_for(rng, cfg, B, T)
    frames[4][8] = np.nan  # row 4's ninth frame, in its third chunk
    events = [
        [(0, END), (3, 0), (0, END)],  # END after 0 frames, fresh and after frames
        [(4, 0), (2, RESET | END), (3, END)],  # RESET | END on one chunk
        [(6, 0), (5, 0), (2, END), (2, END)],  # past T_max at the second chunk: status 2 until END, then fresh
        [(3, 0), (-1, 0), (2, END), (9, 0), (3, 0), (1, END)],  # a negative length; then past T_max again
        [(4, 0), (3, 0), (2, END), (1, END)],  # a NaN in the third chunk: status 1
        [(2, 0), (2, 0), (0, 0), (0, RESET), (3, END)],  # RESET with no frames mid-utterance
    ]
    drive(libs, cfg, T, events, frames)
