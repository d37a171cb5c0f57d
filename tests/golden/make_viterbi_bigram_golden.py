"""Regenerate tests/golden/viterbi_bigram_golden.npz from the REAL reference (oracle/_ref/libgtn_ref.so):
viterbiPath / viterbiScore of intersect(linearGraph(T_b, C), G) with n-gram CTC's bigram graph G
(benchmarks/ctc.cpp:107-134; C nodes, every node start and accept, arc j -> i with label i and weight W[i*C + j],
arcSort()), every utterance on its first T_b rows.

Batches: `ties` (T=7 C=5, integer emissions and weights in {-1, 0, 1}: many equal-score paths), `inf` (T=9 C=6,
about a third of W -inf, one label that no transition reaches), `wide` (T=12 C=29, uniform values).  Every batch has
T_b = 0 (score -inf, no path) and T_b = 1 among its lengths.

Keys, per batch: `*_e` emissions [B, T, C], `*_W` [C*C] (row = destination label), `*_lens` (T_b), and the
reference's `*_paths` [B, T] (labels, -1 beyond the path) and `*_scores` [B].

Run where the reference sources are (it needs oracle/_ref, compiled by `make -C oracle ref`):
    python tests/golden/make_viterbi_bigram_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import viterbi_oracle as vo  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def cases():
    """(name, T, C, input_lens, kind), seeded"""
    return [
        ("ties", 7, 5, [7, 0, 1, 4, 6, 7, 2, 5], "ties"),
        ("inf", 9, 6, [9, 1, 0, 8, 3], "inf"),
        ("wide", 12, 29, [12, 0, 1, 11, 7], "uniform"),
    ]


def inputs(name, T, C, B, kind):
    rng = np.random.default_rng(sum(map(ord, name)) + 29)
    if kind == "uniform":
        return (rng.uniform(-5, 5, (B, T, C)).astype(np.float32),
                rng.uniform(-3, 3, C * C).astype(np.float32))
    e = rng.integers(-1, 2, (B, T, C)).astype(np.float32)
    W = rng.integers(-1, 2, C * C).astype(np.float32)
    if kind == "inf":
        W[rng.random(C * C) < 0.35] = -np.inf
        W.reshape(C, C)[C - 1] = -np.inf
    return e, W


def main():
    out = {}
    for name, T, C, lens, kind in cases():
        e, W = inputs(name, T, C, len(lens), kind)
        paths, scores = vo.batch(vo.ref_viterbi_bigram, e, W, np.asarray(lens, np.int32))
        out.update({name + "_e": e, name + "_W": W, name + "_lens": np.asarray(lens, np.int32),
                    name + "_paths": paths, name + "_scores": scores})
    np.savez_compressed(os.path.join(HERE, "viterbi_bigram_golden.npz"), **out)


if __name__ == "__main__":
    main()
