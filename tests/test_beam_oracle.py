"""The beam-search restatement (tests/beam_oracle.py) against the live reference.  On tiny shapes where a beam of 64
never prunes (C = 3 with T <= 5 for CTC and n-gram CTC, C = 2 with T <= 5 for ASG), its N-best list is the full
ranking of every transcript by the reference's forwardScore of the numerator graph:
  CTC        forwardScore(intersect(ctcGraph(y), E))
  n-gram CTC forwardScore(intersect(intersect(ctc_y, G), E))
  ASG        forwardScore(compose(compose(A_y, G), E))
with scores to 1e-5.  This pins the first-frame weights, ASG's repeated tokens and the end weights."""
import itertools

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import beam_oracle as bo
from tests import ngram_oracle as no

pytestmark = pytest.mark.skipif(not po.have_ref(), reason="oracle/_ref not built (needs the reference sources)")


def _graph(flags, src, dst, lab, w):
    g = po.RefGraph.from_arrays(flags, src, dst, lab, lab, np.asarray(w, np.float32), calc_grad=False)
    g.arc_sort()
    return g


def ref_numerator(e, kind, y, trans_w, blank=0):
    T, C = e.shape
    E = po.RefGraph.linear(T, C, np.ascontiguousarray(e, np.float32).ravel(), calc_grad=False)
    if kind == bo.ASG:
        U = len(y)
        flags = [1 if u == 0 else 0 for u in range(U + 1)]
        flags[U] |= 2
        src, dst, lab = [], [], []
        for u, c in enumerate(y):
            src += [u, u + 1]
            dst += [u + 1, u + 1]
            lab += [c, c]
        A = _graph(flags, src, dst, lab, np.zeros(len(src)))
        tw = np.asarray(trans_w, np.float32)
        gs, gd, gl, gw = [], [], [], []
        for i in range(C):
            gs.append(0), gd.append(i + 1), gl.append(i), gw.append(tw[i])
        for j in range(C):
            for i in range(C):
                gs.append(j + 1), gd.append(i + 1), gl.append(i), gw.append(tw[C + i * C + j])
        G = _graph([1] + [2] * C, gs, gd, gl, gw)
        num = po.ref_op("compose", po.ref_op("compose", A, G), E)
    else:
        fl, s, d, lab = no.ctc_arrays(y, blank)
        ctc = _graph(fl, s, d, lab, np.zeros(len(s)))
        if kind == bo.BIGRAM:
            gf, gs, gd, gl, gw = no.bigram_arrays(trans_w)
            ctc = po.ref_op("intersect", ctc, _graph(gf, gs, gd, gl, gw))
        num = po.ref_op("intersect", ctc, E)
    return po.ref_op("forward_score", num).item()


@pytest.mark.parametrize("kind", [bo.CTC, bo.BIGRAM, bo.ASG])
@pytest.mark.parametrize("T", [1, 2, 3, 5])
def test_exhaustive_beam_is_the_reference_ranking(kind, T):
    C = 2 if kind == bo.ASG else 3
    rng = np.random.default_rng(10 * kind + T)
    e = rng.standard_normal((T, C)).astype(np.float32)
    tw = None if kind == bo.CTC else rng.standard_normal(C * C + (C if kind == bo.ASG else 0)).astype(np.float32)
    W, start = bo.split_weights(kind, tw, C)
    tokens = range(C) if kind == bo.ASG else [c for c in range(C) if c != 0]
    ref = {}
    for n in range(T + 1):
        for y in itertools.product(tokens, repeat=n):
            v = ref_numerator(e, kind, y, tw)
            if v > -np.inf:
                ref[y] = v
    assert len(ref) <= 64
    r = bo.search(e, kind, W, start, 0, 64, 64)
    got = dict(r["hyps"])
    assert set(got) == set(ref), (sorted(got), sorted(ref))
    for y, v in got.items():
        assert abs(v - ref[y]) <= 1e-5 * max(1.0, abs(ref[y])), (y, v, ref[y])
        assert abs(bo.numerator(e, kind, y, W, start) - ref[y]) <= 1e-5 * max(1.0, abs(ref[y]))
    scores = [v for _, v in r["hyps"]]
    assert scores == sorted(scores, reverse=True)
