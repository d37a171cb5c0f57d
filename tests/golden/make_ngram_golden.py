"""Regenerate tests/golden/ngram_golden.npz from the REAL reference (oracle/_ref/libgtn_ref.so): CTC with a learned
bigram transition graph (benchmarks/ctc.cpp:107-134, the graph G of tests/ngram_oracle.py) on small ragged
shapes with blank != 0, graph by graph through the reference's own Graph API.

Run where the reference sources are (it needs oracle/_ref, compiled by `make -C oracle ref`):
    python tests/golden/make_ngram_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import ngram_oracle as no  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def cases():
    """(name, T, C, blank, targets, input_lens), seeded"""
    return [
        ("a", 9, 6, 2, [[1, 3, 3], [], [5, 0, 4, 1]], [9, 7, 9]),
        ("b", 14, 10, 7, [[1, 2, 3, 4], [9, 9], [0]], [14, 5, 11]),
    ]


def main():
    out = {}
    for name, T, C, blank, targets, lens in cases():
        rng = np.random.default_rng(sum(map(ord, name)))
        e = rng.uniform(-5, 5, (len(targets), T, C)).astype(np.float32)
        W = rng.uniform(-2, 2, C * C).astype(np.float32)
        lo, go, to = no.ref_ngram_ctc_batch(e, W, targets, blank, np.asarray(lens))
        out.update({name + "_e": e, name + "_w": W, name + "_blank": np.int32(blank),
                    name + "_targets": np.concatenate([np.asarray(t, np.int32) for t in targets]),
                    name + "_target_lens": np.asarray([len(t) for t in targets], np.int32),
                    name + "_lens": np.asarray(lens, np.int32), name + "_losses": lo, name + "_grads": go,
                    name + "_trans_grad": to})
    np.savez_compressed(os.path.join(HERE, "ngram_golden.npz"), **out)


if __name__ == "__main__":
    main()
