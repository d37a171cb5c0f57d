"""A float64 restatement of gtnb_beam_decode_lexicon_async (include/gtn_b200.h): tests/beam_lm_oracle.py's fused
prefix beam search, with a lexicon trie and a word LM in place of the token LM.

The search itself is beam_lm_oracle.search: its LM is an object with a start state, resolve(state, token) ->
(weight, next state) and end(state).  Here a state is (trie node, word-LM node) and the weight of a move is the
increase of the ranking key's LM part, lm_weight * (lmacc + smear(node)) + word_bonus * words, so that search's
alpha = 1, beta = 0 ranks by exactly am + (lm_weight * (lmacc + smear) + word_bonus * words) (in float64).  A move
the lexicon forbids, or a completed word of weight -inf, resolves to -inf.  The end weight completes the pending word
(-inf inside a word), takes the smear off and adds the word LM's end weight, so the final key is
am + lm_weight * lm + word_bonus * words.

The word LM is a beam_lm_oracle.LM over the labels [0, V] (label V is end of sentence), resolved by walking it.  The
words of a hypothesis are its segmentation: the trie walk over its tokens, a word completed at every separator or
word-start token that follows a word end, and at the end.
"""
import numpy as np

from tests import beam_lm_oracle as blo

NEG = -np.inf
IN_WORD, SEPARATOR, WORD_START = 0, 1, 2


class Lexicon:
    """classes [C] of IN_WORD / SEPARATOR / WORD_START; spellings: (token tuple, word id) pairs; lm: a
    beam_lm_oracle.LM over [0, V] or None (every weight 0).  The trie's nodes are numbered in insertion order."""

    def __init__(self, C, classes, spellings, V, lm=None):
        self.C, self.V, self.cls, self.lm = C, V, [int(k) for k in classes], lm
        self.spellings = [(tuple(int(c) for c in y), int(w)) for y, w in spellings]
        self.kids, self.word = [{}], [-1]
        for toks, w in spellings:
            n = 0
            for c in toks:
                c = int(c)
                if c not in self.kids[n]:
                    self.kids[n][c] = len(self.kids)
                    self.kids.append({})
                    self.word.append(-1)
                n = self.kids[n][c]
            self.word[n] = int(w)
        # smear: the largest finite w(start, word) at or below each node; 0 when none, at the root, without an LM
        best = [NEG] * len(self.kids)
        if lm is not None:
            for n in range(len(self.kids) - 1, 0, -1):  # (children are created after their parent)
                if self.word[n] >= 0:
                    best[n] = max(best[n], lm.resolve(lm.start, self.word[n])[0])
                for k in self.kids[n].values():
                    best[n] = max(best[n], best[k])
        self.smear = [b if n and b > NEG else 0.0 for n, b in enumerate(best)]

    def move(self, n, c):
        """-> (node reached, whether it completes n's word) or None when forbidden"""
        k = self.cls[c]
        if k == IN_WORD:
            return (self.kids[n][c], False) if c in self.kids[n] else None
        if n != 0 and self.word[n] < 0:
            return None
        if k == SEPARATOR:
            return 0, n != 0
        return (self.kids[0][c], n != 0) if c in self.kids[0] else None

    def segment(self, y):
        """the words of transcript y, or None when the lexicon does not admit it"""
        n, words = 0, []
        for c in y:
            mv = self.move(n, int(c))
            if mv is None:
                return None
            if mv[1]:
                words.append(self.word[n])
            n = mv[0]
        if n != 0:
            if self.word[n] < 0:
                return None
            words.append(self.word[n])
        return words

    def resolve(self, s, w):
        return (0.0, 0) if self.lm is None else self.lm.resolve(s, w)

    def end(self, s):
        return 0.0 if self.lm is None else self.lm.end(s)

    def lm_score(self, words):
        """the word LM's score of a word sequence, end weight included"""
        s, tot = (0 if self.lm is None else self.lm.start), 0.0
        for w in words:
            x, s = self.resolve(s, w)
            if x == NEG:
                return NEG
            tot += x
        return tot + self.end(s)


class _KeyLM:
    """the beam_lm_oracle.search LM interface over (trie node, word-LM node): weights are increments of
    lm_weight * (lmacc + smear) + word_bonus * words"""

    def __init__(self, lex, lm_weight, word_bonus):
        self.lex, self.a, self.b = lex, lm_weight, word_bonus
        self.start = (0, 0 if lex.lm is None else lex.lm.start)

    def _complete(self, n, s):
        """completing n's word from LM node s -> (key increment, LM node), or (-inf, None)"""
        x, s2 = self.lex.resolve(s, self.lex.word[n])
        return (NEG, None) if x == NEG else (self.a * x + self.b, s2)

    def resolve(self, state, c):
        n, s = state
        mv = self.lex.move(n, c)
        if mv is None:
            return NEG, None
        n2, done = mv
        x = 0.0
        if done:
            x, s = self._complete(n, s)
            if x == NEG:
                return NEG, None
        return x + self.a * (self.lex.smear[n2] - self.lex.smear[n]), (n2, s)

    def end(self, state):
        n, s = state
        x = -self.a * self.lex.smear[n]
        if n != 0:
            if self.lex.word[n] < 0:
                return NEG
            d, s = self._complete(n, s)
            if d == NEG:
                return NEG
            x += d
        we = self.lex.end(s)
        return NEG if we == NEG else x + self.a * we


def batch(emissions, kind, trans_w=None, input_lens=None, blank=0, K=16, N=1, lex=None, lm_weight=1.0,
          word_bonus=0.0, P=None):
    """The call's outputs for a batch, as beam_lm_oracle.batch (lm: the word LM's score of the words), plus
    words [B, N, T] int32 (-1 after the last word) and counts [B, N] int32 (-1 for unused hypotheses)"""
    out = blo.batch(emissions, kind, trans_w, input_lens, blank, K, N, _KeyLM(lex, lm_weight, word_bonus), 1.0, 0.0,
                    P)
    B, _, T = out["tokens"].shape
    out["words"] = np.full((B, N, T), -1, np.int32)
    out["counts"] = np.full((B, N), -1, np.int32)
    for b in range(B):
        for n in range(N):
            if out["lengths"][b, n] < 0:
                continue
            w = lex.segment(out["tokens"][b, n, :out["lengths"][b, n]])
            out["words"][b, n, :len(w)] = w
            out["counts"][b, n] = len(w)
            out["lm"][b, n] = lex.lm_score(w)
    return out


def identity(C, kind, blank=0):
    """the identity lexicon: every non-blank token (every token for ASG) a word-start token spelling itself as the
    word of the same id -> (classes, spellings)"""
    toks = [c for c in range(C) if kind == blo.ASG or c != blank]
    cls = [WORD_START] * C
    return cls, [((c,), c) for c in toks]


def random_lexicon(rng, C, n_words, sep=None, word_start=(), blank=0, min_len=1, max_len=5, extra_spellings=0):
    """a seeded lexicon over the letters (the tokens that are neither blank, separator nor word-start): n_words
    distinct random spellings (word-start mode: each begins with a word-start token) and extra_spellings second
    spellings of random words -> (classes, spellings)"""
    ws = list(word_start)
    letters = [c for c in range(C) if c != blank and c != sep and c not in ws]
    cls = [IN_WORD] * C
    if sep is not None:
        cls[sep] = SEPARATOR
    for c in ws:
        cls[c] = WORD_START
    seen, sp = set(), []
    while len(sp) < n_words + extra_spellings:
        n = int(rng.integers(min_len, max_len + 1))
        y = [int(c) for c in rng.choice(letters, n)]
        if ws:
            y = [int(rng.choice(ws))] + y[1:]
        y = tuple(y)
        if y in seen:
            continue
        seen.add(y)
        w = len(sp) if len(sp) < n_words else int(rng.integers(n_words))
        sp.append((y, w))
    return cls, sp
