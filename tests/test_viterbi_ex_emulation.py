"""The SOURCE of gtn_b200/csrc/k_dense.cu as gtnb_viterbi_dense_ex launches it, run on the CPU through the SIMT
emulator of tests/emu against the C oracle: both graph kinds (ASG: compose(emissions, transitions); BIGRAM:
intersect(emissions, G) with n-gram CTC's bigram graph), C not a multiple of 4, ragged lengths with T_b in {0, 1},
tie-heavy integer inputs and -inf transitions.  Paths compared with ==, scores bit for bit."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_build
from tests import viterbi_oracle as vo

f32p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build('viterbi_ex', ['k_dense.cu']))
    lib.emu_viterbi_dense_ex.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, C.c_int, f32p, i32p, f32p]
    return lib


@pytest.mark.parametrize("shape", [(2, 9, 4), (4, 9, 5), (4, 17, 28), (4, 11, 29), (3, 12, 64), (4, 8, 127),
                                   (3, 10, 128)])
@pytest.mark.parametrize("inputs", ["uniform", "ties", "forbid"])
@pytest.mark.parametrize("kind", ["asg", "bigram"])
def test_viterbi_ex_kernel_source_matches_oracle(emu, oracle, shape, inputs, kind):
    B, T, Cn = shape
    n_trans = Cn * Cn if kind == "bigram" else Cn + Cn * Cn
    rng = np.random.default_rng(Cn + 1000 * ["uniform", "ties", "forbid"].index(inputs))
    if inputs == "uniform":
        e = rng.uniform(-5, 5, (B, T, Cn)).astype(np.float32)
        tw = rng.uniform(-5, 5, n_trans).astype(np.float32)
    else:  # small integers: many equal-score paths, the first-relaxed predecessor must win
        e = rng.integers(-2, 3, (B, T, Cn)).astype(np.float32)
        tw = rng.integers(-1, 2, n_trans).astype(np.float32)
    if inputs == "forbid":  # forbidden transitions, and a label no transition reaches
        tw[rng.random(n_trans) < 0.3] = -np.inf
        tw[-Cn * Cn:].reshape(Cn, Cn)[Cn - 1] = -np.inf
    lens = np.array([T, 1, 0, T - 3][:B], np.int32)
    pad = e.copy()
    for b in range(B):
        pad[b, lens[b]:] = np.nan  # rows beyond T_b are never read
    paths = np.full((B, T), -7, np.int32)
    scores = np.full(B, 7.0, np.float32)
    rc = emu.emu_viterbi_dense_ex(B, T, Cn, pad.ctypes.data_as(f32p), lens.ctypes.data_as(i32p),
                                  int(kind == "bigram"), tw.ctypes.data_as(f32p), paths.ctypes.data_as(i32p),
                                  scores.ctypes.data_as(f32p))
    emu_build.check(rc)
    for b in range(B):
        if kind == "bigram":
            want_path, want_score = vo.oracle_viterbi_bigram(e[b, :lens[b]], tw)
        else:  # (compose with the transitions' non-accepting start node: T_b = 0 gives -inf here too)
            want_path, want_score = oracle.viterbi_dense(e[b, :lens[b]], tw)
        assert np.array_equal(paths[b, :lens[b]], want_path), (b, paths[b, :lens[b]], want_path)
        assert (paths[b, lens[b]:] == -1).all()  # every entry is written
        assert scores[b] == np.float32(want_score), (b, scores[b], want_score)
    if B > 2:
        assert scores[2] == -np.inf  # T_b = 0: linearGraph(0, C) accepts nothing


def test_c_above_the_tile_is_refused(emu):
    e = np.zeros((1, 2, 225), np.float32)
    tw = np.zeros(225 * 225, np.float32)
    paths, scores = np.zeros((1, 2), np.int32), np.zeros(1, np.float32)
    assert emu.emu_viterbi_dense_ex(1, 2, 225, e.ctypes.data_as(f32p), None, 1, tw.ctypes.data_as(f32p),
                                    paths.ctypes.data_as(i32p), scores.ctypes.data_as(f32p)) == 1
