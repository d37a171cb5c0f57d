"""k_edit.cu's edit_distance_kernel from source on the CPU, through the SIMT emulator of tests/emu
(tests/emu/edit_emu.cpp), compared == against the restatement (tests/edit_oracle.py): distances, counts, unit counts,
status and both alignment rows.

- ragged lengths at the launch geometry, every strip height K and the multi-warp ring at small widths;
- the role swap in both orientations (the shorter sequence forms the rows);
- repeated-token and all-tie inputs, where the tie rule decides the counts and the alignment;
- word mode with leading, trailing and repeated separators and empty word lists, with the shipped hash and with a
  degenerate one under which every word pair collides;
- every invalid length alone, flagged 2 with the other pairs unchanged;
- alignment on, off and one-sided giving the same scalars.
"""
import ctypes as C

import numpy as np
import pytest

from tests import edit_oracle as eo
from tests import emu_build

i32p = C.POINTER(C.c_int32)
IMIN, IMAX = np.iinfo(np.int32).min, np.iinfo(np.int32).max


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("edit", ["k_edit.cu"]))
    lib.emu_edit.argtypes = [C.c_int, i32p, C.c_int, i32p, i32p, C.c_int, i32p, C.c_int, C.c_int, C.c_int, C.c_int,
                             C.c_int, i32p, i32p, i32p, i32p, i32p, i32p]
    lib.emu_edit_plan.argtypes = [C.c_int, C.c_int, C.c_int, i32p]
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(i32p)


def run(emu, hyp, hl, ref, rl, word_sep=-1, K=0, warps=0, collide=False, align=(True, True)):
    hyp, ref = np.ascontiguousarray(hyp, np.int32), np.ascontiguousarray(ref, np.int32)
    hl, rl = np.ascontiguousarray(hl, np.int32), np.ascontiguousarray(rl, np.int32)
    B, N = hyp.shape
    M = ref.shape[1]
    out = dict(distance=np.full(B, 77, np.int32), ops=np.full((B, 3), 77, np.int32),
               units=np.full((B, 2), 77, np.int32), status=np.full(B, 77, np.int32),
               hyp_align=np.full((B, N), 77, np.int32) if align[0] else None,
               ref_align=np.full((B, M), 77, np.int32) if align[1] else None)
    emu_build.check(emu.emu_edit(B, _p(hyp), N, _p(hl), _p(ref), M, _p(rl), word_sep, K, warps, int(collide),
                                 int(align[0] or align[1]), _p(out["distance"]), _p(out["ops"]), _p(out["units"]),
                                 _p(out["status"]), _p(out["hyp_align"]), _p(out["ref_align"])))
    return out


def check(emu, hyp, hl, ref, rl, word_sep=-1, **kw):
    got = run(emu, hyp, hl, ref, rl, word_sep, **kw)
    want = eo.batch(hyp, hl, ref, rl, word_sep)
    for k in ("distance", "ops", "units", "status", "hyp_align", "ref_align"):
        if got[k] is not None:
            assert np.array_equal(got[k], want[k]), (k, got[k], want[k])
    return got


def pairs(rng, B, N, M, C, lo=0):
    """ragged pairs: hypotheses about 30 % edited copies of references (some unrelated), padded with garbage"""
    hyp = rng.integers(-5, 99, (B, N)).astype(np.int32)
    ref = rng.integers(-5, 99, (B, M)).astype(np.int32)
    hl = rng.integers(lo, N + 1, B).astype(np.int32)
    rl = rng.integers(lo, M + 1, B).astype(np.int32)
    for b in range(B):
        r = rng.integers(0, C, rl[b])
        ref[b, :rl[b]] = r
        h = [t for t in r if rng.random() > 0.15]
        h = [t if rng.random() > 0.15 else int(rng.integers(0, C)) for t in h]
        for _ in range(int(rng.integers(0, 4))):
            h.insert(int(rng.integers(0, len(h) + 1)), int(rng.integers(0, C)))
        if b % 4 == 3:
            h = list(rng.integers(0, C, hl[b]))
        hl[b] = min(len(h), N)
        hyp[b, :hl[b]] = h[:hl[b]]
    return hyp, hl, ref, rl


def test_plan_buckets(emu):
    out = (C.c_int32 * 3)()
    for (N, M, sep), want in {(10, 40, -1): (1, 1, 40), (33, 80, -1): (2, 1, 80), (300, 200, -1): (8, 1, 300),
                              (513, 600, -1): (16, 2, 600), (4096, 4096, -1): (16, 8, 4096),
                              (4096, 4096, 0): (16, 4, 2048), (9, 5, 0): (1, 1, 5)}.items():
        emu.emu_edit_plan(N, M, sep, out)
        assert tuple(out) == want, (N, M, sep, tuple(out))


def test_ragged_at_plan_geometry(emu):
    rng = np.random.default_rng(1)
    hyp, hl, ref, rl = pairs(rng, 12, 40, 37, 6)
    hl[0], rl[0] = 0, 0
    hl[1], rl[1] = 0, 5
    hl[2], rl[2] = 7, 0
    check(emu, hyp, hl, ref, rl)


@pytest.mark.parametrize("K,warps,width", [(1, 1, 30), (2, 1, 60), (4, 1, 120), (8, 1, 250), (1, 2, 60), (1, 3, 90),
                                           (2, 3, 180), (16, 1, 300), (16, 2, 530)])
def test_every_bucket_and_the_warp_ring(emu, K, warps, width):
    rng = np.random.default_rng(K * 10 + warps)
    B = 3 if width > 200 else 6
    hyp, hl, ref, rl = pairs(rng, B, width, width + 7, 5, lo=width // 2)
    hl[0], rl[0] = width, width + 7  # the full bound: every strip of every warp carries rows
    check(emu, hyp, hl, ref, rl, K=K, warps=warps)


def test_role_swap_both_orientations(emu):
    rng = np.random.default_rng(3)
    N, M = 50, 50
    hyp = rng.integers(0, 3, (4, N)).astype(np.int32)
    ref = rng.integers(0, 3, (4, M)).astype(np.int32)
    hl = np.array([50, 10, 33, 34], np.int32)
    rl = np.array([10, 50, 34, 33], np.int32)
    got = check(emu, hyp, hl, ref, rl, K=1, warps=2)
    # swapping hypothesis and reference swaps insertions and deletions
    back = check(emu, ref, rl, hyp, hl, K=1, warps=2)
    assert np.array_equal(got["distance"], back["distance"])
    assert np.array_equal(got["ops"][:, 1], back["ops"][:, 2]) and np.array_equal(got["ops"][:, 2], back["ops"][:, 1])


def test_repeated_tokens_and_ties(emu):
    N = M = 40
    rows = [([0] * 40, [0] * 25), ([0] * 25, [0] * 40), ([0, 1] * 20, [1, 0] * 20), ([0] * 20, [1] * 20),
            ([0] * 40, [1] * 13), ([1] * 7, [0, 1] * 20), ([2, 2, 3, 3] * 10, [3, 3, 2, 2] * 10), ([5], [6])]
    hyp = np.zeros((len(rows), N), np.int32)
    ref = np.zeros((len(rows), M), np.int32)
    hl = np.array([len(h) for h, _ in rows], np.int32)
    rl = np.array([len(r) for _, r in rows], np.int32)
    for b, (h, r) in enumerate(rows):
        hyp[b, :len(h)], ref[b, :len(r)] = h, r
    check(emu, hyp, hl, ref, rl)
    check(emu, hyp, hl, ref, rl, K=1, warps=2)


def word_rows(rng, B, N, M):
    """token rows over {0, 1, 2, 3}, separator 0, with fixed rows first"""
    hyp = rng.integers(0, 4, (B, N)).astype(np.int32)
    ref = rng.integers(0, 4, (B, M)).astype(np.int32)
    fixed = [([0, 0, 1, 2, 0, 0, 3, 0], [1, 2, 0, 3]), ([0, 0, 0], [1, 0, 1]), ([0], []), ([], [0, 0]),
             ([1, 1, 0, 1], [1, 0, 1, 1]), ([2, 0, 2, 0, 2], [2, 2, 0, 2]), ([1, 0, 2], [0] * M)]
    hl = rng.integers(0, N + 1, B).astype(np.int32)
    rl = rng.integers(0, M + 1, B).astype(np.int32)
    for b, (h, r) in enumerate(fixed):
        hyp[b, :len(h)], ref[b, :len(r)] = h, r
        hl[b], rl[b] = len(h), len(r)
    return hyp, hl, ref, rl


@pytest.mark.parametrize("collide", [False, True])
def test_word_mode(emu, collide):
    rng = np.random.default_rng(5 + collide)
    hyp, hl, ref, rl = word_rows(rng, 14, 30, 26)
    got = check(emu, hyp, hl, ref, rl, word_sep=0, collide=collide)
    assert tuple(got["units"][3]) == (0, 0) and tuple(got["units"][6]) == (2, 0)
    check(emu, hyp, hl, ref, rl, word_sep=0, collide=collide, K=1, warps=2)
    # a separator other than 0
    hyp2 = np.where(hyp == 0, 3, np.where(hyp == 3, 0, hyp)).astype(np.int32)
    ref2 = np.where(ref == 0, 3, np.where(ref == 3, 0, ref)).astype(np.int32)
    check(emu, hyp2, hl, ref2, rl, word_sep=3, collide=collide)
    # longer rows: the word split runs over several chunks of a four-warp CTA
    hyp, hl, ref, rl = word_rows(rng, 9, 200, 190)
    hl[-1], rl[-1] = 200, 190
    check(emu, hyp, hl, ref, rl, word_sep=0, collide=collide, K=1, warps=4)


def test_every_invalid_length_alone(emu):
    rng = np.random.default_rng(9)
    N, M = 20, 24
    hyp, hl, ref, rl = pairs(rng, 3, N, M, 4)
    want = eo.batch(hyp, hl, ref, rl)
    for side, bound in ((0, N), (1, M)):
        for bad in (-1, bound + 1, IMIN, IMAX):
            h2, r2 = hl.copy(), rl.copy()
            (h2 if side == 0 else r2)[1] = bad
            got = check(emu, hyp, h2, ref, r2)
            assert got["status"][1] == 2 and got["distance"][1] == -1 and (got["ops"][1] == -1).all()
            assert (got["units"][1] == -1).all()
            assert (got["hyp_align"][1] == -1).all() and (got["ref_align"][1] == -1).all()
            for b in (0, 2):
                for k in ("distance", "ops", "units", "status", "hyp_align", "ref_align"):
                    assert np.array_equal(got[k][b], want[k][b]), (side, bad, b, k)
            check(emu, hyp, h2, ref, r2, word_sep=0)


def test_alignment_on_off_same_scalars(emu):
    rng = np.random.default_rng(11)
    hyp, hl, ref, rl = pairs(rng, 8, 45, 40, 5)
    full = check(emu, hyp, hl, ref, rl)
    for align in ((False, False), (True, False), (False, True)):
        got = check(emu, hyp, hl, ref, rl, align=align)
        for k in ("distance", "ops", "units", "status"):
            assert np.array_equal(got[k], full[k]), (align, k)
