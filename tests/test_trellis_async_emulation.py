"""The SOURCE of the kernels gtnb_ngram_ctc_loss_async and gtnb_asg_loss_async add (k_ctc.cu: the prepare kernel's
n-gram and ASG instantiations, trellis_async_gate_kernel, trellis_async_scatter_kernel) and of those they reuse
(ctc_async_finalize_kernel; k_ngram.cu's numerator build kernels) on the CPU through the SIMT emulator of tests/emu.

- The prepare kernel's descriptors and [offsets | lens | T] arrays equal what the host gives: composed_alloc's slabs
  at the bounds (every utterance U = S, T_b = T; n-gram with S - 1 skips), restated below as `bound_meta`, with the
  per-utterance fields ngram_ctc_loss_call / asg_loss_ex_call take from parse_targets.  Invalid lengths and labels
  are flagged and swept as empty.
- The build kernels fed the padded, bound-strided layout write the same tables as on gtnb_ngram_ctc_loss's packed
  layout, utterance by utterance.
- The gated scatter adds each unflagged utterance's own arcs and nothing else; the gate combines the two status words
  and zeroes the backward's T_b of a flagged utterance; the finalize loss is read_losses' den - num in float32.
"""
import ctypes as C

import numpy as np
import pytest

from tests import emu_build
from tests.test_ctc_async_emulation import FIXED_PITCH, GraphMeta, align4, as_dict

f32p, i32p, u8p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)


def dims(asg, U, skips):
    """(N, A, n_accept) of the numerator graph of one utterance (ngram_ctc_loss_call / asg_loss_ex_call)"""
    if asg:
        return U + 1, 2 * U, 1 if U > 0 else 0
    L = 2 * U + 1
    return L + 1, L + (L - 1) + skips + min(L, 2), 2 if L >= 2 else 1


def bound_meta(asg, B, T, C_, S, b):
    """composed_alloc's descriptor of utterance b (implicit_only) for a batch of B graphs all at the bounds"""
    N, A, n_acc = dims(asg, S, max(S - 1, 0))
    pitch = FIXED_PITCH if N <= FIXED_PITCH else align4(N)
    capN = (T + 1) * pitch + 4
    m = GraphMeta()
    m.node_base, m.arc_base, m.lvl_base, m.acc_base = b * capN, b * 4, b * align4(T + 2), b * align4(max(n_acc, 1))
    m.sg_node_base, m.sg_arc_base = b * align4(N + 1), b * align4(max(A, 1))
    m.emis_off = b * T * C_
    m.grad_graph_off = b * A if B > 1 else 0
    m.L, m.n_accept, m.LB, m.status, m.T = T + 1, n_acc, -1, 0, T
    m.sg_N, m.sg_A, m.sg_all_valid, m.sg_uniform = N, A, 1, 1
    m.cap_N, m.cap_A, m.cap_L = capN, 4, align4(T + 2)
    return m


def m01(asg, B, T, C_, S):
    return (GraphMeta * 2)(bound_meta(asg, B, T, C_, S, 0), bound_meta(asg, B, T, C_, S, 1 if B > 1 else 0))


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("trellis_async", ["k_ctc.cu", "k_ngram.cu"]))
    lib.emu_trellis_async_prepare.argtypes = [C.c_int] * 5 + [C.POINTER(GraphMeta), i32p, i32p, i32p,
                                                              C.POINTER(GraphMeta), i32p, f32p, i32p, i32p]
    lib.emu_trellis_num_build.argtypes = [C.c_int] * 4 + [C.POINTER(GraphMeta), i32p, i32p, i32p, f32p, u8p, i32p,
                                                          i32p, i32p, i32p, f32p, i32p, i32p, i32p, i32p]
    lib.emu_trellis_async_gate.argtypes = [C.c_int, i32p, i32p, i32p, i32p, f32p]
    lib.emu_trellis_async_scatter.argtypes = [C.c_int, C.POINTER(GraphMeta), i32p, i32p, f32p, f32p]
    lib.emu_trellis_async_finalize.argtypes = [C.c_int, f32p, f32p, i32p, i32p, f32p, i32p, f32p, C.c_longlong]
    return lib


def p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def prepare(lib, asg, B, T, C_, S, targets, lens, il):
    meta = (GraphMeta * B)()
    small = np.full(3 * B, -7, np.int32)
    deltas = np.zeros(B, np.float32)
    valid = np.full(B, -7, np.int32)
    kst = np.full(2 * B, -7, np.int32)
    emu_build.check(lib.emu_trellis_async_prepare(int(asg), B, S, T, C_, m01(asg, B, T, C_, S), p(il, i32p),
                                                  p(targets, i32p), p(lens, i32p), meta, p(small, i32p),
                                                  p(deltas, f32p), p(valid, i32p), p(kst, i32p)))
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
        out.append((U, Tb, int((y[1:] != y[:-1]).sum()), True) if ok else (0, 0, 0, False))
    return out


def batch(B, T, C_, S, seed):
    rng = np.random.default_rng(seed)
    targets = rng.integers(0, C_, (B, S)).astype(np.int32)
    if S > 2:
        targets[0, 1] = targets[0, 0]  # a repeat: one skip arc fewer
        targets[1 % B, :] = targets[1 % B, 0]  # all repeats: no skip arc at all
    lens = rng.integers(0, S + 1, B).astype(np.int32)
    lens[0] = S
    lens[1 % B] = S
    il = rng.integers(0, T + 1, B).astype(np.int32)
    return targets, lens, il


@pytest.mark.parametrize("asg", [False, True])
@pytest.mark.parametrize("B,T,C_,S", [(11, 40, 64, 7), (3, 9, 28, 0), (1, 5, 128, 3), (17, 30, 60, 120)])
def test_prepare_matches_the_host_descriptors(emu, asg, B, T, C_, S):
    targets, lens, il = batch(B, T, C_, S, B * 1000 + S + asg)
    for in_lens in (None, il):
        meta, small, deltas, valid, kst = prepare(emu, asg, B, T, C_, S, targets, lens, in_lens)
        for b, (U, Tb, skips, ok) in enumerate(parse(targets, lens, in_lens, T, C_)):
            assert ok
            want = bound_meta(asg, B, T, C_, S, b)
            want.T, want.L, want.tgt_off = Tb, Tb + 1, b * S
            want.sg_N, want.sg_A, want.n_accept = dims(asg, U, skips)
            assert as_dict(meta[b]) == as_dict(want), b
        want_T = np.full(B, T, np.int32) if in_lens is None else in_lens
        assert (small == np.concatenate([np.arange(B, dtype=np.int32) * S, lens, want_T])).all()
        assert (deltas == -1.0).all() and (valid == 1).all() and (kst == 0).all()


@pytest.mark.parametrize("asg", [False, True])
def test_prepare_flags_and_sanitises_invalid_utterances(emu, asg):
    B, T, C_, S = 7, 20, 32, 5
    targets = np.tile(np.arange(1, S + 1, dtype=np.int32), (B, 1))
    lens = np.array([S, -1, S + 1, 3, 4, 2, S], np.int32)  # U < 0, U > S
    il = np.array([T, T, T, T + 1, T, -2, T], np.int32)  # T_b > T, T_b < 0
    targets[4, 3] = C_  # a label >= C inside the target
    targets[3, 4] = C_ + 5  # beyond U = 3: padding, never read
    targets[6, 0] = -1  # a negative label
    meta, small, deltas, valid, kst = prepare(emu, asg, B, T, C_, S, targets, lens, il)
    assert valid.tolist() == [1, 0, 0, 0, 0, 0, 0]
    empty = dims(asg, 0, 0)
    for b in range(1, B):
        assert (meta[b].T, meta[b].L, meta[b].sg_N, meta[b].sg_A, meta[b].n_accept) == (0, 1) + empty, b
        assert small[B + b] == 0 and small[2 * B + b] == 0
    assert (kst == 0).all()


def packed_meta(asg, Us, skips):
    """gtnb_ngram_ctc_loss / gtnb_asg_loss_ex's packed slabs: each utterance right after the previous one"""
    metas, n, a, acc = [], 0, 0, 0
    for U, s in zip(Us, skips):
        N, A, n_acc = dims(asg, U, s)
        m = GraphMeta()
        m.sg_node_base, m.sg_arc_base, m.acc_base, m.grad_graph_off = n, a, acc, a
        m.sg_N, m.sg_A, m.n_accept = N, A, n_acc
        metas.append(m)
        n, a, acc = n + align4(N + 1), a + align4(max(A, 1)), acc + align4(max(n_acc, 1))
    return metas, n, a, acc


def build(emu, asg, metas, n, a, acc, C_, blank, targets, off, lens, W):
    B = len(metas)
    t = dict(flags=np.full(n + 8, 0xEE, np.uint8), in_ptr=np.full(n + 8, -9, np.int32),
             in_src=np.full(a + 8, -9, np.int32), in_label=np.full(a + 8, -9, np.int32),
             in_arc=np.full(a + 8, -9, np.int32), in_w=np.full(a + 8, -9, np.float32),
             ilabel=np.full(a + 8, -9, np.int32), olabel=np.full(a + 8, -9, np.int32),
             acc=np.full(acc + 8, -9, np.int32), map=np.full(a + 8, -9, np.int32))
    emu_build.check(emu.emu_trellis_num_build(
        int(asg), B, C_, blank, (GraphMeta * B)(*metas), p(targets, i32p), p(off, i32p), p(lens, i32p), p(W, f32p),
        p(t["flags"], u8p), p(t["in_ptr"], i32p), p(t["in_src"], i32p), p(t["in_label"], i32p), p(t["in_arc"], i32p),
        p(t["in_w"], f32p), p(t["ilabel"], i32p), p(t["olabel"], i32p), p(t["acc"], i32p), p(t["map"], i32p)))
    return t


def graph_of(t, m):
    """utterance m's own tables: nodes [0, N], arcs [0, A), its accept nodes"""
    N, A = m.sg_N, m.sg_A
    nodes = {k: t[k][m.sg_node_base:m.sg_node_base + N + (k == "in_ptr")].tolist() for k in ("flags", "in_ptr")}
    arcs = {k: t[k][m.sg_arc_base:m.sg_arc_base + A].tolist()
            for k in ("in_src", "in_label", "in_arc", "in_w", "ilabel", "olabel")}
    arcs["map"] = t["map"][m.grad_graph_off:m.grad_graph_off + A].tolist()
    return nodes, arcs, t["acc"][m.acc_base:m.acc_base + m.n_accept].tolist()


@pytest.mark.parametrize("asg", [False, True])
@pytest.mark.parametrize("C_,S", [(64, 9), (30, 4), (128, 1)])
def test_build_kernels_on_the_padded_layout_equal_the_packed_layout(emu, asg, C_, S):
    B, T, blank = 6, 25, 0
    targets, lens, il = batch(B, T, C_, S, C_ + S + asg)
    lens[2] = 0  # an empty target
    rng = np.random.default_rng(C_ * S)
    W = rng.normal(0, 1, (C_ + C_ * C_) if asg else C_ * C_).astype(np.float32)
    meta, small, _, valid, _ = prepare(emu, asg, B, T, C_, S, targets, lens, il)
    assert (valid == 1).all()
    N, A, n_acc = dims(asg, S, max(S - 1, 0))
    padded = build(emu, asg, list(meta), B * align4(N + 1), B * align4(max(A, 1)), B * align4(max(n_acc, 1)), C_,
                   blank, targets, small[:B].copy(), small[B:2 * B].copy(), W)
    rows = [targets[b, :lens[b]] for b in range(B)]
    cat = np.ascontiguousarray(np.concatenate(rows) if lens.sum() else np.zeros(1), np.int32)
    off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32)
    skips = [int((r[1:] != r[:-1]).sum()) for r in rows]
    pm, n, a, acc = packed_meta(asg, lens.tolist(), skips)
    ref = build(emu, asg, pm, n, a, acc, C_, blank, cat, off, lens, W)
    for b in range(B):
        assert (meta[b].sg_N, meta[b].sg_A, meta[b].n_accept) == (pm[b].sg_N, pm[b].sg_A, pm[b].n_accept), b
        got, want = graph_of(padded, meta[b]), graph_of(ref, pm[b])
        assert got == want, b
        # the arc count the build kernel writes (in_ptr[N]) is the prepared sg_A the scatter reads
        assert got[0]["in_ptr"][-1] == meta[b].sg_A


def test_gated_scatter_reads_only_each_utterances_own_arcs(emu):
    rng = np.random.default_rng(3)
    B, nT, cap = 5, 40, 12  # transition slots, slab of 12 arcs per utterance (the bounds)
    sink = nT  # where a stale map entry of a slab's tail points: must stay 0
    sgA = [12, 7, 0, 3, 9]
    meta = (GraphMeta * B)()
    mp = np.full(B * cap, sink, np.int32)  # the tails: garbage the build kernels never overwrite
    src = np.full(B * cap, 1.0e6, np.float32)
    for b in range(B):
        meta[b].grad_graph_off, meta[b].sg_A = b * cap, sgA[b]
        mp[b * cap:b * cap + sgA[b]] = rng.integers(0, nT, sgA[b])
        src[b * cap:b * cap + sgA[b]] = rng.normal(0, 1, sgA[b]).astype(np.float32)
    kst = np.array([0, 1, 0, 0, 0], np.int32)  # utterance 1 flagged by the gate
    dst = np.zeros(nT + 1, np.float32)
    emu_build.check(emu.emu_trellis_async_scatter(B, meta, p(kst, i32p), p(mp, i32p), p(src, f32p), p(dst, f32p)))
    want = np.zeros(nT + 1, np.float64)
    for b in (0, 2, 3, 4):
        for k in range(b * cap, b * cap + sgA[b]):
            want[mp[k]] += src[k]
    assert dst[sink] == 0.0
    assert np.allclose(dst, want, rtol=1e-6, atol=1e-6)


def test_gate_combines_the_status_words(emu):
    B = 300  # two CTAs of the gate
    rng = np.random.default_rng(4)
    kst = np.zeros(2 * B, np.int32)
    kst[rng.integers(0, B, 30)] = 1  # the denominator's flags
    kst[B + rng.integers(0, B, 30)] = 1  # the numerator's
    valid = (rng.random(B) > 0.1).astype(np.int32)
    T_fwd = rng.integers(0, 50, B).astype(np.int32)
    T_fwd[:5] = 0
    den = rng.normal(0, 10, B).astype(np.float32)
    den0, k0 = den.copy(), kst.copy()
    T_bwd = np.full(B, -7, np.int32)
    emu_build.check(emu.emu_trellis_async_gate(B, p(T_fwd, i32p), p(valid, i32p), p(kst, i32p), p(T_bwd, i32p),
                                               p(den, f32p)))
    flagged = (k0[:B] != 0) | (k0[B:] != 0) | (valid == 0)
    assert (kst[:B] == flagged.astype(np.int32)).all()
    assert (kst[B:] == k0[B:]).all()
    assert (T_bwd == np.where(flagged, 0, T_fwd)).all()
    assert np.isnan(den[T_fwd == 0]).all()
    assert (den[T_fwd != 0] == den0[T_fwd != 0]).all()


def test_finalize_matches_the_host_loss_loop(emu):
    rng = np.random.default_rng(5)
    B, T, C_ = 7, 6, 12
    den = rng.normal(0, 50, B).astype(np.float32)
    num = rng.normal(0, 50, B).astype(np.float32)
    den[5], num[6] = np.nan, -np.inf  # T_b = 0 (the gate's NaN); an infeasible target
    kst = np.array([0, 1, 1, 0, 0, 0, 0], np.int32)  # the gate's combined flags (invalid ones included)
    valid = np.array([1, 1, 0, 1, 1, 1, 1], np.int32)
    grad = rng.normal(0, 1, (B, T, C_)).astype(np.float32)
    g0 = grad.copy()
    losses = np.zeros(B, np.float32)
    status = np.full(B, -1, np.int32)
    emu_build.check(emu.emu_trellis_async_finalize(B, p(den, f32p), p(num, f32p), p(kst, i32p), p(valid, i32p),
                                                   p(losses, f32p), p(status, i32p), p(grad, f32p), T * C_))
    assert status.tolist() == [0, 1, 2, 0, 0, 0, 0]
    for b in range(B):
        if status[b]:
            assert np.isnan(losses[b]) and (grad[b] == 0).all()
            continue
        want = np.float32(den[b] - num[b])  # read_losses: d[b] - n[b] in float32
        assert losses[b].tobytes() == want.tobytes() or (np.isnan(want) and np.isnan(losses[b])), b
        assert (grad[b] == g0[b]).all()
    assert losses[6] == np.inf
