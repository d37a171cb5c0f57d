"""The lexicon beam-search restatement (tests/beam_lexicon_oracle.py) against the live reference.  On tiny shapes,
where a beam of 64 never prunes, its N-best list is the full ranking of every admitted transcript y by

    numerator(y) + alpha * forwardScore(compose(linear(words(y) + [V]), G)) + beta * |words(y)|,

with scores to 1e-5.  Admission and words(y) are the output labels of compose(linear(y), L), L a lexicon transducer
built here from the classes and spellings.  Cases: separator and word-start mode, spellings that are prefixes of
others, a word with two spellings, a deterministic word LM and the resolved graph of a backoff_ngram word LM with and
without end-of-sentence arcs, -inf arcs and end weights, CTC, n-gram CTC and ASG.  A separate test holds arpa_graph to
the textbook backoff formula on a hand-written ARPA text (it needs no reference)."""
import itertools

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import beam_lexicon_oracle as lxo
from tests import beam_lm_oracle as blo
from tests import beam_oracle as bo
from tests import test_beam_lm_oracle as tlo
from tests import test_beam_oracle as tbo

need_ref = pytest.mark.skipif(not po.have_ref(), reason="oracle/_ref not built (needs the reference sources)")
EPS = -1


def lexicon_transducer(lex):
    """L: input tokens, output words.  Nodes are the trie's plus a final node F; in-word arcs follow the trie, a
    separator or word-start token at a word end outputs its word, and a word end has an epsilon-input arc to F that
    outputs its word.  The root and F accept."""
    n = len(lex.kids)
    F = n
    src, dst, il, ol = [], [], [], []

    def arc(a, b, i, o):
        src.append(a), dst.append(b), il.append(i), ol.append(o)
    for u in range(n):
        for c in range(lex.C):
            mv = lex.move(u, c)
            if mv is not None:
                arc(u, mv[0], c, lex.word[u] if mv[1] else EPS)
        if u and lex.word[u] >= 0:
            arc(u, F, EPS, lex.word[u])
    flags = np.zeros(n + 1, np.uint8)
    flags[0] = 3
    flags[F] = 2
    g = po.RefGraph.from_arrays(flags, src, dst, il, ol, np.zeros(len(src), np.float32), calc_grad=False)
    g.arc_sort()
    return g


def ref_words(L, y):
    """the output labels along compose(linear(y), L)'s path, or None when it has none"""
    C = po.ref_op("compose", tlo.chain(list(y)), L)
    if not np.isfinite(po.ref_op("viterbi_score", C).item()):
        return None
    p = po.ref_op("viterbi_path", C).arrays()
    return [int(o) for o in p["olabel"] if o != EPS]


def ref_word_lm(G, w, words, V):
    return tlo.ref_lm(G, w, list(words), [V])


LEXICONS = {  # (classes, spellings) over C = 5, blank 0
    "sep": ([0, 0, 0, 0, 1], [((1,), 0), ((1, 2), 1), ((2, 3), 2), ((3,), 2)]),
    "start": ([0, 2, 2, 0, 0], [((1,), 0), ((1, 3), 1), ((2, 4), 2), ((2,), 1)]),
}


def word_lm(rng, which, V, eos):
    if which == "det":
        return tlo.deterministic_lm(rng, V, eos)
    return tlo.backoff_resolved(rng, V, eos)


CASES = [("sep", "det", True, 0.5, 0.0), ("sep", "backoff", False, 2.0, -1.0), ("start", "det", False, 1.0, 1.5),
         ("start", "backoff", True, 0.5, 0.5)]


@need_ref
@pytest.mark.parametrize("kind", [bo.CTC, bo.BIGRAM, bo.ASG])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_exhaustive_lexicon_beam_is_the_reference_ranking(kind, case):
    mode, which, eos, alpha, beta = CASES[case]
    cls, sp = LEXICONS[mode]
    C, V, T = 5, 3, 3
    rng = np.random.default_rng(40 * kind + case)
    e = rng.standard_normal((T, C)).astype(np.float32)
    tw = None if kind == bo.CTC else rng.standard_normal(C * C + (C if kind == bo.ASG else 0)).astype(np.float32)
    W, start = bo.split_weights(kind, tw, C)
    G, w = word_lm(rng, which, V, eos)
    lm = blo.LM(G, w, V)
    lex = lxo.Lexicon(C, cls, sp, V, lm)
    L = lexicon_transducer(lex)
    tokens = range(C) if kind == bo.ASG else range(1, C)
    ref = {}
    for n in range(T + 1):
        for y in itertools.product(tokens, repeat=n):
            ws = ref_words(L, y)
            assert (ws is None) == (lex.segment(y) is None) and (ws is None or ws == lex.segment(y)), y
            if ws is None:
                continue
            num = tbo.ref_numerator(e, kind, y, tw) if n or kind != bo.ASG else -np.inf
            lmv = ref_word_lm(G, w, ws, V) if (eos or which == "backoff") else tlo.ref_lm(G, w, ws, [])
            if num > -np.inf and lmv > -np.inf:
                ref[y] = (num + alpha * lmv + beta * len(ws), num, lmv)
    assert 0 < len(ref) <= 64
    out = lxo.batch(e[None], kind, tw, None, 0, 64, 64, lex, alpha, beta)
    got = {}
    for n in range(64):
        ln = out["lengths"][0, n]
        if ln >= 0:
            got[tuple(out["tokens"][0, n, :ln])] = (out["scores"][0, n], out["am"][0, n], out["lm"][0, n])
    assert set(got) == set(ref), (sorted(got), sorted(ref))
    for y, v in got.items():
        for g, x in zip(v, ref[y]):
            assert abs(g - x) <= 1e-5 * max(1.0, abs(x)), (y, v, ref[y])


ARPA = r"""
\data\
ngram 1=5
ngram 2=4
ngram 3=1

\1-grams:
-99 <s> -0.30
-0.60 the -0.25
-0.70 cat -0.20
-0.90 sat
-0.80 </s>

\2-grams:
-0.20 <s> the -0.10
-0.40 the cat -0.15
-0.30 cat sat
-0.50 cat </s>

\3-grams:
-0.05 <s> the cat

\end\
"""


def test_arpa_graph_is_the_backoff_formula():
    from gtn_b200 import torch_loss as tl
    words = ["the", "cat", "sat", "dog"]  # ("dog" is never seen; n-grams outside the vocabulary are dropped)
    G, w = tl.arpa_graph(ARPA.strip().splitlines(), words)
    V = len(words)
    lm = blo.LM(G, w, V)
    ln10 = np.log(10.0)
    p = {}  # the ARPA table: n-gram -> (log10 p, log10 backoff)
    sect = 0
    for line in ARPA.strip().splitlines():
        if line.startswith("\\") and line.endswith("-grams:"):
            sect = int(line[1])
        elif sect and line.strip() and not line.startswith("\\"):
            f = line.split()
            p[tuple(f[1:1 + sect])] = (float(f[0]), float(f[1 + sect]) if len(f) > 1 + sect else 0.0)

    def textbook(h, x):
        """log10 P(x | h) by the backoff formula"""
        if h + (x,) in p:
            return p[h + (x,)][0]
        if not h:
            return -np.inf
        return (p[h][1] if h in p else 0.0) + textbook(h[1:], x)
    names = words + ["</s>"]
    for h in [("<s>",), ("<s>", "the"), ("<s>", "the", "cat"), ("<s>", "cat", "sat")]:
        s = lm.start
        for x in h[1:]:
            s = lm.resolve(s, names.index(x))[1]
        for i, x in enumerate(names):
            want = textbook(h[-2:], x) * ln10
            got = lm.resolve(s, i)[0]
            assert (want == got == -np.inf) or abs(got - want) < 1e-5, (h, x, got, want)
    # a sentence: ln P(the cat sat </s>) from <s>
    want = (textbook(("<s>",), "the") + textbook(("<s>", "the"), "cat") + textbook(("the", "cat"), "sat") +
            textbook(("cat", "sat"), "</s>")) * ln10
    assert abs(lm.score([0, 1, 2]) - want) < 1e-5
