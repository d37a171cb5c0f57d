"""The SOURCE of gtnb_ctc_loss_async's kernels (k_ctc.cu: ctc_async_prepare_kernel, ctc_async_finalize_kernel) on the
CPU through the SIMT emulator of tests/emu.

- The prepare kernel's descriptors and [offsets | lens | T] arrays equal what the host gives for the same batch:
  composed_alloc's slabs at the bounds (U = S, T_b = T, restated below as `bound_meta`), with parse_targets' per-
  utterance fields (T_b, 2U + 1 nodes, arcs with the skip arcs, the target's offset) and Targets::packed's arrays.
- Invalid lengths and labels are flagged and swept as empty.
- The finalize kernel forms the losses like ctc_loss_run's host loop, bit for bit, with NaN and zero rows for flagged
  utterances.
- k_bidir.cu's kernel fed the prepared padded layout equals the packed layout of gtnb_ctc_loss (tests/emu/bidir_emu.cpp).
"""
import ctypes as C

import numpy as np
import pytest

from tests import emu_build

f32p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
FIXED_PITCH = 224  # kImplicitFixedPitch
HELPERS2 = 8  # 2 * bidir_zparts(): the partial sums of forwardScore(e) of the two CTAs


class GraphMeta(C.Structure):  # gtnb_meta.h
    _fields_ = [(n, C.c_longlong) for n in ("node_base", "arc_base", "lvl_base", "acc_base", "blvl_base", "bnode_base",
                                            "sg_node_base", "sg_arc_base", "emis_off", "grad_graph_off")] + \
               [(n, C.c_int) for n in ("L", "N", "A", "n_accept", "LB", "status", "T", "sg_N", "sg_A", "sg_all_valid",
                                       "sg_uniform", "cap_N", "cap_A", "cap_L", "tgt_off", "pad_")]


def align4(v):
    return (v + 3) // 4 * 4


def bound_dims(S):
    L = 2 * S + 1
    return L, L + (L - 1) + max(S - 1, 0)


def bound_meta(B, T, C_, S, b):
    """composed_alloc's descriptor of utterance b (implicit_only) for a batch of B graphs all at the bounds"""
    N, A = bound_dims(S)
    pitch = FIXED_PITCH if N <= FIXED_PITCH else align4(N)
    capN = (T + 1) * pitch + 4
    m = GraphMeta()
    m.node_base, m.arc_base, m.lvl_base, m.acc_base = b * capN, b * 4, b * align4(T + 2), b * 4
    m.sg_node_base, m.sg_arc_base = b * align4(N + 1), b * align4(max(A, 1))
    m.emis_off = b * T * C_
    m.grad_graph_off = b * A if B > 1 else 0
    m.L, m.n_accept, m.LB, m.status, m.T = T + 1, 2 if N >= 2 else 1, -1, 0, T
    m.sg_N, m.sg_A, m.sg_all_valid, m.sg_uniform = N, A, 1, 1
    m.cap_N, m.cap_A, m.cap_L = capN, 4, align4(T + 2)
    return m


def m01(B, T, C_, S):
    return (GraphMeta * 2)(bound_meta(B, T, C_, S, 0), bound_meta(B, T, C_, S, 1 if B > 1 else 0))


def as_dict(m):
    return {n: getattr(m, n) for n, _ in GraphMeta._fields_}


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("ctc_async", ["k_ctc.cu", "k_bidir.cu"]))
    lib.emu_ctc_async_prepare.argtypes = [C.c_int] * 4 + [C.POINTER(GraphMeta), i32p, i32p, i32p,
                                                          C.POINTER(GraphMeta), i32p, f32p, i32p, i32p]
    lib.emu_ctc_async_finalize.argtypes = [C.c_int, C.c_int, f32p, f32p, i32p, i32p, f32p, i32p, f32p, C.c_longlong]
    lib.emu_ctc_async_bidir.argtypes = [C.c_int] * 4 + [C.POINTER(GraphMeta), C.c_longlong, C.c_longlong, f32p, i32p,
                                                        i32p, i32p, C.c_int, C.c_int, f32p, i32p, f32p]
    return lib


@pytest.fixture(scope="module")
def packed():
    lib = C.CDLL(emu_build.build("bidir", ["k_ctc.cu", "k_bidir.cu"]))
    lib.emu_bidir_ctc.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, i32p, i32p, C.c_int, C.c_int, f32p, f32p,
                                  f32p, i32p]
    return lib


def p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def prepare(lib, B, T, C_, S, targets, lens, il):
    meta = (GraphMeta * B)()
    small = np.full(3 * B, -7, np.int32)
    deltas = np.zeros(B, np.float32)
    valid = np.full(B, -7, np.int32)
    kst = np.full(B, -7, np.int32)
    emu_build.check(lib.emu_ctc_async_prepare(B, S, T, C_, m01(B, T, C_, S), p(il, i32p), p(targets, i32p),
                                              p(lens, i32p), meta, p(small, i32p), p(deltas, f32p), p(valid, i32p),
                                              p(kst, i32p)))
    return meta, small, deltas, valid, kst


def parse(targets, lens, il, T, C_):
    """parse_targets on the rows of the padded targets: (U, T_b, skips, valid) per utterance"""
    out = []
    S = targets.shape[1]
    for b in range(len(lens)):
        U = int(lens[b])
        Tb = T if il is None else int(il[b])
        ok = 0 <= U <= S and 0 <= Tb <= T
        y = targets[b, :U] if ok else targets[b, :0]
        ok = ok and bool(((y >= 0) & (y < C_)).all())
        if not ok:
            out.append((0, 0, 0, False))
        else:
            out.append((U, Tb, int((y[1:] != y[:-1]).sum()), True))
    return out


@pytest.mark.parametrize("B,T,C_,S", [(11, 40, 64, 7), (3, 9, 28, 0), (1, 5, 128, 3), (17, 30, 60, 120)])
def test_prepare_matches_the_host_descriptors(emu, B, T, C_, S):
    rng = np.random.default_rng(B * 1000 + S)
    targets = rng.integers(0, C_, (B, S)).astype(np.int32)
    if S > 2:
        targets[0, 1] = targets[0, 0]  # a repeat: no skip arc there
    lens = rng.integers(0, S + 1, B).astype(np.int32)
    lens[0] = S
    il = rng.integers(0, T + 1, B).astype(np.int32)
    for in_lens in (None, il):
        meta, small, deltas, valid, kst = prepare(emu, B, T, C_, S, targets, lens, in_lens)
        for b, (U, Tb, skips, ok) in enumerate(parse(targets, lens, in_lens, T, C_)):
            want = bound_meta(B, T, C_, S, b)
            L = 2 * U + 1
            want.T, want.L, want.sg_N, want.sg_A = Tb, Tb + 1, L, L + (L - 1) + skips
            want.n_accept, want.tgt_off = 2 if L >= 2 else 1, b * S
            assert as_dict(meta[b]) == as_dict(want), b
            assert ok
        # Targets::packed's [offsets | lens | T], the padded rows at b * S
        want_T = np.full(B, T, np.int32) if in_lens is None else in_lens
        assert (small == np.concatenate([np.arange(B, dtype=np.int32) * S, lens, want_T])).all()
        assert (deltas == -1.0).all() and (valid == 1).all() and (kst == 0).all()


def test_prepare_flags_and_sanitises_invalid_utterances(emu):
    B, T, C_, S = 6, 20, 32, 5
    targets = np.tile(np.arange(1, S + 1, dtype=np.int32), (B, 1))
    lens = np.array([S, -1, S + 1, 3, 4, 2], np.int32)  # U < 0, U > S
    il = np.array([T, T, T, T + 1, T, -2], np.int32)  # T_b > T, T_b < 0
    targets[4, 3] = C_  # a label >= C inside the target
    targets[3, 4] = C_ + 5  # beyond U = 3: padding, never read
    meta, small, deltas, valid, kst = prepare(emu, B, T, C_, S, targets, lens, il)
    assert valid.tolist() == [1, 0, 0, 0, 0, 0]
    for b in range(1, B):
        assert (meta[b].T, meta[b].L, meta[b].sg_N, meta[b].sg_A) == (0, 1, 1, 1), b
        assert small[B + b] == 0 and small[2 * B + b] == 0
    # a label >= C alone, with valid lengths
    il2 = np.full(B, T, np.int32)
    lens2 = np.full(B, S, np.int32)
    t2 = np.tile(np.arange(1, S + 1, dtype=np.int32), (B, 1))
    t2[2, S - 1] = C_
    t2[5, 0] = C_ + 100
    _, _, _, valid2, _ = prepare(emu, B, T, C_, S, t2, lens2, il2)
    assert valid2.tolist() == [1, 1, 0, 1, 1, 0]


def test_finalize_matches_the_host_loss_loop(emu):
    rng = np.random.default_rng(5)
    B, T, C_ = 7, 6, 12
    for zp in (1, HELPERS2):
        z = rng.normal(0, 50, zp * B).astype(np.float32)
        s = rng.normal(0, 50, B).astype(np.float32)
        kst = np.array([0, 1, 0, 0, 3, 0, 0], np.int32)
        valid = np.array([1, 1, 0, 1, 1, 1, 0], np.int32)
        grad = rng.normal(0, 1, (B, T, C_)).astype(np.float32)
        g0 = grad.copy()
        losses = np.zeros(B, np.float32)
        status = np.full(B, -1, np.int32)
        emu_build.check(emu.emu_ctc_async_finalize(B, zp, p(z, f32p), p(s, f32p), p(kst, i32p), p(valid, i32p),
                                                   p(losses, f32p), p(status, i32p), p(grad, f32p), T * C_))
        assert status.tolist() == [0, 1, 2, 0, 1, 0, 2]
        for b in range(B):
            if status[b]:
                assert np.isnan(losses[b]) and (grad[b] == 0).all()
                continue
            zb = np.float32(0)
            for k in range(zp):  # ctc_loss_run's loop, in float32
                zb = np.float32(zb + z[zp * b + k])
            assert losses[b].tobytes() == np.float32(zb - s[b]).tobytes()
            assert (grad[b] == g0[b]).all()


@pytest.mark.parametrize("C_,S,mode", [(64, 6, -1), (128, 5, -1), (64, 6, 0), (32, 4, -1)])
def test_bidir_on_the_padded_layout_equals_the_packed_layout(emu, packed, C_, S, mode):
    """PAIR kernels (C = 64, 128), the one-node-per-thread kernels after ctc_build_kernel (bidir_mode 0, C = 32):
    ragged lengths, a repeat, an empty target and an infeasible one, against gtnb_ctc_loss's packed targets"""
    rng = np.random.default_rng(C_ + S + mode)
    B, T = 4, 19
    e = rng.normal(0, 2, (B, T, C_)).astype(np.float32)
    targets = rng.integers(1, C_, (B, S)).astype(np.int32)
    targets[0, 2] = targets[0, 1]
    lens = np.array([S, S - 2, 0, S], np.int32)
    il = np.array([T, T - 5, 7, 3], np.int32)  # utterance 3: S labels in 3 frames, infeasible
    blank = 0
    N, A = bound_dims(S)
    losses = np.zeros(B, np.float32)
    status = np.zeros(B, np.int32)
    grad = np.zeros((B, T, C_), np.float32)
    emu_build.check(emu.emu_ctc_async_bidir(B, T, C_, S, m01(B, T, C_, S), align4(N + 1), align4(A), p(e, f32p),
                                            p(il, i32p), p(targets, i32p), p(lens, i32p), blank, mode,
                                            p(losses, f32p), p(status, i32p), p(grad, f32p)))
    cat = np.concatenate([targets[b, :lens[b]] for b in range(B)]).astype(np.int32)
    out = np.zeros(B, np.float32)
    zn = np.zeros(B, np.float32)
    g2 = np.zeros((B, T, C_), np.float32)
    st2 = np.zeros(B, np.int32)
    emu_build.check(packed.emu_bidir_ctc(B, T, C_, p(e, f32p), p(il, i32p), p(cat, i32p), p(lens, i32p), blank, mode,
                                         p(out, f32p), p(zn, f32p), p(g2, f32p), p(st2, i32p)))
    assert (status == st2).all()
    for b in range(B):
        if st2[b]:
            continue
        assert losses[b].tobytes() == np.float32(zn[b] - out[b]).tobytes(), b
        assert (grad[b] == g2[b]).all(), b
