"""The edit-distance restatement (tests/edit_oracle.py) against the live reference: the distance is
-viterbiScore(compose(x, compose(edits, y))) with `edits` built as in the reference's examples/edit_distance.cpp, in
token and word mode; the restatement's path, recomputed as arcs of that lattice, costs the distance."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import edit_oracle as eo

pytestmark = pytest.mark.skipif(not po.have_ref(), reason="oracle/_ref not built (needs /root/reference)")


def ref_graph(g):
    return po.RefGraph.from_arrays(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"],
                                   calc_grad=False)


def ref_distance(h, r, C):
    x, y, edits = ref_graph(eo.chain_graph(h)), ref_graph(eo.chain_graph(r)), ref_graph(eo.edits_graph(C))
    return -po.ref_op("viterbi_score", po.ref_op("compose", x, po.ref_op("compose", edits, y))).item()


def cases(rng, C):
    out = [([], []), ([], [1, 2]), ([3, 0], []), ([1, 2, 3], [1, 2, 3]), ([0, 0, 0], [1, 1]),
           ([2] * 6, [2] * 4), ([0, 1, 0, 1], [0, 0, 0, 1, 1])]
    for _ in range(40):
        n, m = rng.integers(0, 14, size=2)
        out.append((list(rng.integers(0, C, n)), list(rng.integers(0, C, m))))
    return out


@pytest.mark.parametrize("C", [5, 28])
def test_distance_is_reference_viterbi_score(C):
    rng = np.random.default_rng(C)
    for h, r in cases(rng, C):
        o = eo.edit_distance(h, r)
        assert o["distance"] == ref_distance(h, r, C), (h, r)
        assert o["sub"] + o["ins"] + o["dele"] == o["distance"]
        assert eo.path_cost(h, r) == o["distance"]


def test_reference_example():
    assert ref_distance([0, 1, 0, 1], [0, 0, 0, 1, 1], 5) == 2 == eo.edit_distance([0, 1, 0, 1], [0, 0, 0, 1, 1])[
        "distance"]


def test_word_mode_is_reference_over_word_ids():
    rng = np.random.default_rng(7)
    sep = 0
    seqs = [([0, 0], [0]), ([0, 1, 2, 0, 0, 3, 0], [1, 2, 0, 3]), ([4, 0, 4, 4], [4, 4, 0, 4])]
    for _ in range(30):
        seqs.append((list(rng.integers(0, 4, rng.integers(0, 20))), list(rng.integers(0, 4, rng.integers(0, 20)))))
    for hyp, ref in seqs:
        h, r = eo.units(hyp, ref, sep)
        assert len(h) == len(eo.words(hyp, sep)) and len(r) == len(eo.words(ref, sep))
        C = max([0] + h + r) + 1
        o = eo.edit_distance(hyp, ref, sep)
        assert o["distance"] == ref_distance(h, r, C), (hyp, ref)
        assert eo.path_cost(h, r) == o["distance"]
