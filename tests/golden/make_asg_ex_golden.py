"""Regenerate tests/golden/asg_ex_golden.npz from the REAL reference (oracle/_ref/libgtn_ref.so): ASG
(test/criterion_test.cpp:244-305) on padded minibatches, every utterance run alone on its first T_b rows, with
T_b = 0, T_b < U, U = 0 and repeated labels among the cases.

Keys, per batch `a` (T=9 C=6) and `b` (T=14 C=10): `*_e` emissions [B, T, C], `*_tw` transitions [C + C*C],
`*_targets` (concatenated) and `*_target_lens`, `*_lens` (T_b), and the reference's `*_losses` (NaN for T_b = 0,
+inf for T_b < U or U = 0), `*_grads` (zero beyond T_b) and `*_trans_grad` (the batch sum).

Run where the reference sources are (it needs oracle/_ref, compiled by `make -C oracle ref`):
    python tests/golden/make_asg_ex_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import asg_oracle as ao  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def cases():
    """(name, T, C, targets, input_lens), seeded"""
    return [
        ("a", 9, 6, [[1, 3, 3], [], [5, 0, 4, 1], [2, 2], [0, 1, 2, 3, 4]], [9, 7, 6, 0, 3]),
        ("b", 14, 10, [[1, 2, 3, 4], [9, 9], [0], [7, 7, 7, 7, 7]], [14, 5, 11, 14]),
    ]


def main():
    out = {}
    for name, T, C, targets, lens in cases():
        rng = np.random.default_rng(sum(map(ord, name)) + 17)
        e = rng.uniform(-5, 5, (len(targets), T, C)).astype(np.float32)
        tw = rng.uniform(-2, 2, C + C * C).astype(np.float32)
        lo, go, to = ao.ref_asg_batch(e, tw, targets, np.asarray(lens))
        out.update({name + "_e": e, name + "_tw": tw,
                    name + "_targets": np.concatenate([np.asarray(t, np.int32) for t in targets]),
                    name + "_target_lens": np.asarray([len(t) for t in targets], np.int32),
                    name + "_lens": np.asarray(lens, np.int32), name + "_losses": lo, name + "_grads": go,
                    name + "_trans_grad": to})
    np.savez_compressed(os.path.join(HERE, "asg_ex_golden.npz"), **out)


if __name__ == "__main__":
    main()
