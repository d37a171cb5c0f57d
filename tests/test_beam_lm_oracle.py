"""The fused beam-search restatement (tests/beam_lm_oracle.py) against the live reference.  On the tiny shapes of
test_beam_oracle.py, where a beam of 64 never prunes, its N-best list is the full ranking of every transcript y by

    reference numerator(y) + alpha * LM(y) + beta * |y|,     LM(y) = forwardScore(compose(linear(y [+ C]), lm)),

with scores to 1e-5, for an epsilon-free deterministic LM and for the resolved graph of a backoff_ngram LM, with and
without end-of-sentence arcs, with a -inf arc and a -inf end weight, for CTC, n-gram CTC and ASG.  A separate test
holds the resolved graph (an epsilon-free graph built from the walk over arcs and backoff arcs) to that walk."""
import itertools

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import backoff_oracle as bko
from tests import beam_lm_oracle as blo
from tests import beam_oracle as bo
from tests import test_beam_oracle as tbo

pytestmark = pytest.mark.skipif(not po.have_ref(), reason="oracle/_ref not built (needs the reference sources)")


def chain(y):
    n = len(y)
    flags = [0] * (n + 1)
    flags[0] |= 1
    flags[n] |= 2
    return tbo._graph(flags, list(range(n)), list(range(1, n + 1)), list(y), np.zeros(n))


def ref_lm(G, w, y, eos):
    """forwardScore(compose(linear(y [+ C]), G)), G's nodes all accepting"""
    flags = np.asarray(G["flags"]) | 2
    lm = tbo._graph(flags, G["src"], G["dst"], G["ilabel"], w)
    return po.ref_op("forward_score", po.ref_op("compose", chain(list(y) + eos), lm)).item()


def deterministic_lm(rng, C, eos):
    """3 nodes, an arc per (node, token) to a random node; one token arc weighs -inf; with eos, an arc labelled C
    per node, one of which (not the start's) weighs -inf"""
    S = 3
    src, dst, lab, w = [], [], [], []
    for s in range(S):
        for c in range(C):
            src.append(s), dst.append(int(rng.integers(S))), lab.append(c), w.append(np.log(rng.uniform(0.1, 1.0)))
    w[int(rng.integers(S * C))] = -np.inf
    if eos:
        for s in range(S):
            src.append(s), dst.append(s), lab.append(C), w.append(np.log(rng.uniform(0.1, 1.0)) if s != 2 else -np.inf)
    flags = np.zeros(S, np.uint8)
    flags[0] = 1
    G = dict(flags=flags, src=np.asarray(src, np.int32), dst=np.asarray(dst, np.int32),
             ilabel=np.asarray(lab, np.int32), olabel=np.asarray(lab, np.int32))
    return G, np.asarray(w, np.float32)


def backoff_resolved(rng, C, eos):
    """the resolved graph of a backoff_ngram LM (with eos: an end arc per node, one of them -inf)"""
    while True:  # (a corpus that shows every token: the chain is peaked and may stick to one)
        G, w = bko.backoff_ngram(rng, C, 2, n_tokens=400, min_count=1, n_neg_inf=1)
        if len(G["flags"]) == C + 1:
            break
    if eos:
        S = len(G["flags"])
        x = np.log(rng.uniform(0.1, 0.5, S)).astype(np.float32)
        x[S - 1] = -np.inf
        G = dict(G)
        for k, v in (("src", np.arange(S)), ("dst", np.arange(S)), ("ilabel", np.full(S, C)),
                     ("olabel", np.full(S, C))):
            G[k] = np.concatenate([G[k], v]).astype(np.int32)
        w = np.concatenate([w, x])
    return blo.resolved_graph(blo.LM(G, w, C))


CASES = [  # (lm, eos, alpha, beta)
    ("det", True, 0.5, 0.0), ("det", False, 2.0, -1.0), ("det", True, 0.0, 1.5),
    ("backoff", True, 2.0, 1.5), ("backoff", False, 0.5, -1.0), ("backoff", True, 0.5, 0.0),
]


@pytest.mark.parametrize("kind", [bo.CTC, bo.BIGRAM, bo.ASG])
@pytest.mark.parametrize("T", [2, 5])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_exhaustive_fused_beam_is_the_reference_ranking(kind, T, case):
    which, eos, alpha, beta = CASES[case]
    C = 2 if kind == bo.ASG else 3
    rng = np.random.default_rng(100 * kind + 10 * T + case)
    e = rng.standard_normal((T, C)).astype(np.float32)
    tw = None if kind == bo.CTC else rng.standard_normal(C * C + (C if kind == bo.ASG else 0)).astype(np.float32)
    W, start = bo.split_weights(kind, tw, C)
    if which == "det":
        G, w = deterministic_lm(rng, C, eos)
        end = [C] if eos else []
    else:
        G, w = backoff_resolved(rng, C, eos)
        end = [C]  # (the resolved graph always ends with label C, weight 0 without eos arcs)
    lm = blo.LM(G, w, C)
    tokens = range(C) if kind == bo.ASG else [c for c in range(C) if c != 0]
    ref = {}
    for n in range(T + 1):
        for y in itertools.product(tokens, repeat=n):
            num = tbo.ref_numerator(e, kind, y, tw)
            lmv = ref_lm(G, w, y, end)
            if num > -np.inf and lmv > -np.inf:
                ref[y] = (num + alpha * lmv + beta * len(y), num, lmv)
    assert 0 < len(ref) <= 64
    r = blo.search(e, kind, W, start, 0, 64, 64, lm, alpha, beta)
    got = {y: (sc, am, lmv) for y, sc, am, lmv in r["hyps"]}
    assert set(got) == set(ref), (sorted(got), sorted(ref))
    for y, v in got.items():
        for g, x in zip(v, ref[y]):
            assert abs(g - x) <= 1e-5 * max(1.0, abs(x)), (y, v, ref[y])
    scores = [sc for _, sc, _, _ in r["hyps"]]
    assert scores == sorted(scores, reverse=True)


@pytest.mark.parametrize("eos", [True, False])
def test_resolved_graph_is_the_walk(eos):
    """LM(y) by walking arcs and backoff arcs == the reference's score of y + [C] on the resolved graph"""
    rng = np.random.default_rng(5 + eos)
    C = 4
    G, w = bko.backoff_ngram(rng, C, 3, n_tokens=600, min_count=2, n_neg_inf=2)
    if eos:
        S = len(G["flags"])
        G = dict(G)
        for k, v in (("src", np.arange(S)), ("dst", np.arange(S)), ("ilabel", np.full(S, C)),
                     ("olabel", np.full(S, C))):
            G[k] = np.concatenate([G[k], v]).astype(np.int32)
        w = np.concatenate([w, np.log(rng.uniform(0.1, 0.5, S)).astype(np.float32)])
    lm = blo.LM(G, w, C)
    R, rw = blo.resolved_graph(lm)
    n_inf = 0
    for n in range(4):
        for y in itertools.product(range(C), repeat=n):
            want = lm.score(y)
            got = ref_lm(R, rw, y, [C])
            n_inf += want == -np.inf
            assert (want == got == -np.inf) or abs(want - got) <= 1e-5 * max(1.0, abs(want)), (y, want, got)
    assert n_inf > 0  # (the -inf arcs are reached)
