"""Benchmark of the lexicon beam decoders (gtnb_beam_decode_lexicon_async through torch ctc_lexicon_beam_decode and
asg_lexicon_beam_decode) on an H100: ms until the results are on the device, medians of timed calls, the variants of
each workload alternating call by call, at N = 1, float32:
  letters     C = 29 (blank, 26 letters, apostrophe, "|" separator), CTC B=256 T=1000, lexicons of 20 000 and 200 000
              words, each with a backoff word trigram (synth_word_lm);
  pieces      C = 256 word pieces, 128 of them word-start tokens, CTC B=128 T=500, 20 000 words;
  asg         ASG on the letters, B=128 T=500, 20 000 words;
  big_lm      the 200 000-word letters lexicon with a word LM of 24 M arcs (a third of the arc bound, a 512 MB hash
              far beyond the L2), against the 1.3 M-arc trigram;
at K = 8 and 64, token_beam P = C and P = 16.  Each workload also times the same emissions through
*_beam_decode (no LM) and *_lm_beam_decode with a token backoff trigram (tests/backoff_oracle: backoff_ngram at
C = 29, backoff_lm at C = 256), and the
host time of one lexicon call (enqueue only, no synchronisation).  Emissions are noisy around alignments of random
word sequences of the lexicon (spelled_inputs).

Also the word error rate of the first hypothesis on a seeded quality workload (quality_workload: sentences sampled
from a word trigram, spelled with "|" between words) for: no LM (ctc_beam_decode, its tokens split at "|" and looked
up in the lexicon), the lexicon alone, and the lexicon with the word LM.  The card's name and power limit are read in
the same run.  Prints one JSON line per setting, then the whole record (also written to --out when given).
"""
import argparse
import json
import os
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from gtn_b200 import capi  # noqa: E402
from gtn_b200 import torch_loss as tl  # noqa: E402
from tests import backoff_oracle as bko  # noqa: E402
import bench_beam_lm as bbl  # noqa: E402  (card, timed, the token-LM decoders)


def random_spellings(rng, n_words, letters, min_len=2, max_len=10, word_start=()):
    """n_words distinct random spellings over `letters` (word-start mode: each begins with a word-start token)"""
    ws = np.asarray(list(word_start))
    seen, sp = set(), []
    while len(sp) < n_words:
        n = int(rng.integers(min_len, max_len + 1))
        y = [int(c) for c in rng.choice(letters, n)]
        if len(ws):
            y[0] = int(rng.choice(ws))
        y = tuple(y)
        if y not in seen:
            seen.add(y)
            sp.append((y, len(sp)))
    return sp


def synth_word_lm(rng, V, n_bigram, n_trigram, arcs=20):
    """a backoff word trigram of about V + (n_bigram + n_trigram) * arcs arcs -> (graph dict, weights).  Node 0 is the
    empty history (start) with an arc per word (Zipf-like weights) and an end arc; nodes 1 .. n_bigram are the
    histories of words 0 .. n_bigram - 1, the next n_trigram nodes two-word histories; each has `arcs` word arcs (to
    the history of the word, or the root) and backs off to a shorter history."""
    S = 1 + n_bigram + n_trigram
    uni = -np.log(np.arange(1, V + 1)) - np.log(np.log(V) + 0.58)
    src = [np.zeros(V + 1, np.int64)]
    lab = [np.arange(V + 1)]
    dst = [np.where(np.arange(V + 1) < n_bigram, 1 + np.arange(V + 1), 0)]
    w = [np.concatenate([uni, [np.log(0.05)]])]
    hs = np.arange(1, S)
    for_each = np.repeat(hs, arcs)
    x = np.minimum(rng.zipf(1.3, len(for_each)) - 1, V - 1)
    src.append(for_each)
    lab.append(x)
    dst.append(np.where(x < n_bigram, 1 + x, 0))
    w.append(np.log(rng.uniform(0.01, 0.2, len(for_each))))
    src.append(hs)
    lab.append(np.full(len(hs), -1))
    dst.append(np.where(hs <= n_bigram, 0, 1 + rng.integers(0, n_bigram, len(hs))))
    w.append(np.log(rng.uniform(0.2, 0.6, len(hs))))
    src, lab, dst, w = (np.concatenate(a) for a in (src, lab, dst, w))
    key = src * (V + 2) + lab + 1  # one arc per (node, label)
    _, keep = np.unique(key, return_index=True)
    flags = np.full(S, 2, np.uint8)
    flags[0] = 3
    lab = lab[keep].astype(np.int32)
    return (dict(flags=flags, src=src[keep].astype(np.int32), dst=dst[keep].astype(np.int32), ilabel=lab,
                 olabel=lab), w[keep].astype(np.float32))


def spelled_inputs(rng, kind, lex, B, T, noise=1.0, peak=5.0, n_words=None):
    """(emissions [B, T, C] on the device, transitions or None): random word sequences of lex (anything with C, cls
    and spellings), spelled with a separator between words when cls has one, each token held 1 or 2 frames (blanks
    between them half of the time and always between repeats, for CTC), blank / the last token to the end; emissions
    log_softmax(noise * N(0, 1) + peak at the aligned label)"""
    C, cls, sp = lex.C, list(lex.cls), lex.spellings
    sep = cls.index(1) if 1 in cls else None
    x = rng.standard_normal((B, T, C)).astype(np.float32) * noise
    for b in range(B):
        toks = []
        while len(toks) < (T * 0.45 if kind != capi.DENSE_ASG else T * 0.6):
            if toks and sep is not None:
                toks.append(sep)
            toks.extend(sp[int(rng.integers(len(sp)))][0])
        lab = []
        for i, c in enumerate(toks):
            if kind != capi.DENSE_ASG and ((i and toks[i - 1] == c) or rng.random() < 0.5):
                lab.append(0)
            lab += [c] * int(rng.integers(1, 3))
        lab = lab[:T]
        lab += [0 if kind != capi.DENSE_ASG else lab[-1]] * (T - len(lab))
        x[b, np.arange(T), lab] += peak
    e = torch.log_softmax(torch.as_tensor(x), -1).cuda()
    if kind == capi.DENSE_CTC:
        return e, None
    n = C * C + (C if kind == capi.DENSE_ASG else 0)
    return e, torch.as_tensor((rng.standard_normal(n) * 0.1).astype(np.float32)).cuda()


def letters_classes():
    cls = [0] * 29
    cls[28] = 1
    return cls


def wer(out, refs):
    """word error rate of the first hypotheses (a LexiconBeamDecode) against refs, through edit_distance"""
    return _wer(out.words[:, 0], out.word_counts[:, 0], refs)


def _wer(words, counts, refs):
    B = len(refs)
    M = max(map(len, refs))
    r = torch.full((B, M), -1, dtype=torch.int32, device=words.device)
    for b, y in enumerate(refs):
        r[b, :len(y)] = torch.as_tensor(y, dtype=torch.int32)
    rl = torch.as_tensor([len(y) for y in refs], dtype=torch.int32, device=words.device)
    d = tl.edit_distance(words, counts.clamp(min=0), r, rl)
    return float(d.distance.sum()) / float(rl.sum())


def _resolve(arcs, eps, s, x):
    acc = 0.0
    while (s, x) not in arcs:
        if s not in eps:
            return -np.inf, -1
        acc += eps[s][0]
        s = eps[s][1]
    w, d = arcs[(s, x)]
    return acc + w, d


def quality_workload(seed=1, n_words=300, B=32, U=8, T=160, noise=1.5, peak=2.5):
    """dict(e [B, T, 29] float32, refs (word id lists), spellings, lex (Lexicon with the word LM), lex_nolm,
    sep): a lexicon of n_words letter spellings, a synthetic word trigram, U-word sentences sampled from it (its
    resolved weights renormalised), spelled with "|" between words, emissions noisy around a CTC alignment."""
    rng = np.random.default_rng(seed)
    sp = random_spellings(rng, n_words, np.arange(1, 28), 2, 6)
    G, w = synth_word_lm(rng, n_words, n_words // 2, n_words, arcs=6)
    arcs, eps = {}, {}
    for a in range(len(w)):
        s, x = int(G["src"][a]), int(G["ilabel"][a])
        if x < 0:
            eps[s] = (float(w[a]), int(G["dst"][a]))
        else:
            arcs[(s, x)] = (float(w[a]), int(G["dst"][a]))
    refs = []
    for _ in range(B):
        s, y = 0, []
        for _ in range(U):
            r = np.array([_resolve(arcs, eps, s, x)[0] for x in range(n_words)])
            p = np.exp(r - r.max())
            x = int(rng.choice(n_words, p=p / p.sum()))
            y.append(x)
            s = _resolve(arcs, eps, s, x)[1]
        refs.append(y)
    x = rng.standard_normal((B, T, 29)) * noise
    for b, y in enumerate(refs):
        toks = []
        for i, wd in enumerate(y):
            if i:
                toks.append(28)
            toks.extend(sp[wd][0])
        lab = []
        for i, c in enumerate(toks):
            if (i and toks[i - 1] == c) or rng.random() < 0.5:
                lab.append(0)
            lab += [c] * int(rng.integers(1, 3))
        lab += [0] * (T - len(lab))
        x[b, np.arange(T), lab[:T]] += peak
    e = (x - np.log(np.exp(x).sum(-1, keepdims=True))).astype(np.float32)
    return dict(e=e, refs=refs, spellings=sp, sep=28, lex=tl.Lexicon(sp, 29, n_words, separator=28, lm=(G, w)),
                lex_nolm=tl.Lexicon(sp, 29, n_words, separator=28))


def split_words(tokens, lengths, spellings, sep):
    """ctc_beam_decode's first hypotheses split at the separator and looked up in the lexicon (-2: not a word)"""
    look = {y: w for y, w in spellings}
    tok, ln = tokens[:, 0].cpu().numpy(), lengths[:, 0].cpu().numpy()
    B, T = tok.shape
    words = np.full((B, T), -1, np.int32)
    counts = np.zeros(B, np.int32)
    for b in range(B):
        cur, ws = [], []
        for c in list(tok[b, :max(ln[b], 0)]) + [sep]:
            if c == sep:
                if cur:
                    ws.append(look.get(tuple(cur), -2))
                cur = []
            else:
                cur.append(int(c))
        words[b, :len(ws)] = ws
        counts[b] = len(ws)
    return torch.as_tensor(words).cuda(), torch.as_tensor(counts).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="small workloads (a rehearsal)")
    a = ap.parse_args()
    rec = dict(card=bbl.card(), settings=[])
    print(json.dumps(dict(card=rec["card"])), flush=True)
    rng = np.random.default_rng(0)
    scale = 10 if a.quick else 1
    letters = np.arange(1, 28)
    lexicons = {}

    def make(name, C, cls, sp, V, G=None, ws=()):
        t0 = time.perf_counter()
        sep = cls.index(1) if 1 in cls else None
        lx = tl.Lexicon(sp, C, V, separator=sep, word_start=ws, lm=G)
        ms = (time.perf_counter() - t0) * 1e3
        lexicons[name] = (lx, types.SimpleNamespace(C=C, cls=cls, spellings=sp))
        print(json.dumps(dict(lexicon=name, words=V, lm_arcs=0 if G is None else int(len(G[1])), create_ms=ms)),
              flush=True)

    for V in (20000, 200000):
        V //= scale
        sp = random_spellings(rng, V, letters)
        make("letters_%d" % V, 29, letters_classes(), sp, V, synth_word_lm(rng, V, V // 4, V // 2, 8))
        if V == 200000 // scale:
            n_tri = ((1 << 25) // scale - V) // 20 - V
            make("letters_%d_big_lm" % V, 29, letters_classes(), sp, V, synth_word_lm(rng, V, V, n_tri, 20))
    Vp = 20000 // scale
    ws = list(range(128, 256))
    make("pieces_%d" % Vp, 256, [0] * 128 + [2] * 128,
         random_spellings(rng, Vp, np.arange(1, 128), 1, 4, word_start=ws), Vp,
         synth_word_lm(rng, Vp, Vp // 4, Vp // 2, 8), ws)
    tok_lms = {29: tl.LanguageModel(bbl.gtn_graph(*bko.backoff_ngram(np.random.default_rng(29), 29, 3,
                                                                      n_tokens=20000, min_count=2)), 29),
               256: tl.LanguageModel(bbl.gtn_graph(*bko.backoff_lm(np.random.default_rng(256), C=256)), 256)}
    work = [("letters_%d" % (20000 // scale), capi.DENSE_CTC, 256, 1000),
            ("letters_%d" % (200000 // scale), capi.DENSE_CTC, 256, 1000),
            ("letters_%d_big_lm" % (200000 // scale), capi.DENSE_CTC, 256, 1000),
            ("pieces_%d" % Vp, capi.DENSE_CTC, 128, 500),
            ("letters_%d" % (20000 // scale), capi.DENSE_ASG, 128, 500)]
    if a.quick:
        work = [(n, k, 8, 100) for n, k, _, _ in work]
    for name, kind, B, T in work:
        lx, info = lexicons[name]
        C = info.C
        e, w = spelled_inputs(rng, kind, info, B, T)
        for K in (8, 64):
            def lex_fn(P):
                if kind == capi.DENSE_CTC:
                    return lambda: tl.ctc_lexicon_beam_decode(e, lx, 1.0, 0.5, K, 1, P)
                return lambda: tl.asg_lexicon_beam_decode(e, w, lx, 1.0, 0.5, K, 1, P)
            fns = {"beam": lambda: bbl.bbd.decode(kind, e, w, K, 1),
                   "token_lm": lambda: bbl.decode_lm(kind, e, w, tok_lms[C], K, 1),
                   "lexicon": lex_fn(None), "lexicon_p16": lex_fn(16)}
            for fn in fns.values():
                fn()
            torch.cuda.synchronize()
            host = []
            for _ in range(5):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fns["lexicon"]()
                host.append((time.perf_counter() - t0) * 1e3)
            torch.cuda.synchronize()
            ms = bbl.timed(fns, 3 if a.quick else a.reps)
            s = dict(workload=name, kind={2: "ctc", 0: "asg"}[kind], B=B, T=T, C=C, K=K, N=1, ms=ms,
                     lexicon_host_ms=float(np.median(host)))
            rec["settings"].append(s)
            print(json.dumps(s), flush=True)
    q = quality_workload()
    ed = torch.as_tensor(q["e"]).cuda()
    res = {}
    for K in (8, 16):
        plain = tl.ctc_beam_decode(ed, K, 1)
        res["K%d" % K] = dict(
            no_lm=_wer(*split_words(plain.tokens, plain.lengths, q["spellings"], q["sep"]), q["refs"]),
            lexicon=wer(tl.ctc_lexicon_beam_decode(ed, q["lex_nolm"], 0.0, 0.0, K), q["refs"]),
            lexicon_word_lm=wer(tl.ctc_lexicon_beam_decode(ed, q["lex"], 1.0, 0.0, K), q["refs"]))
    rec["quality_wer"] = res
    print(json.dumps(dict(quality_wer=res)), flush=True)
    print(json.dumps(rec))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
