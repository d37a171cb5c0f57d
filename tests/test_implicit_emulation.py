"""The SOURCE of gtn_b200/csrc/k_implicit.cu -- the criterion's implicit-lattice forward / backward sweeps,
the hot kernels of bench.py -- compiled with g++ against the SIMT emulator of tests/emu/simt_emu.h and run
on the CPU (one std::thread per CUDA thread) against the oracle.

What this pins without a GPU: the one-node-per-thread fast path with its register prefetch blocks, guarded
tails and the named barrier the idle warps skip; the several-nodes-per-thread general path (more than 256
graph nodes); ragged input lengths; the non-finite-weight status bit.  The SFU instructions are replaced
by exp2f / log2f, and nothing is said about speed -- the GPU parity tests (tests/test_gpu_parity.py) stay
the authority for the compiled kernels."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import emu_build, util

HERE = os.path.dirname(os.path.abspath(__file__))
f32p, i32p, u8p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build('implicit', ['k_implicit.cu', 'k_ctc.cu']))
    lib.emu_implicit.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, i32p, u8p, i32p, i32p, i32p, f32p, f32p,
                                 f32p, i32p]
    lib.emu_implicit_ctc.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, i32p, i32p, C.c_int, f32p, f32p, i32p,
                                     i32p, i32p, i32p]
    return lib


def ctc_tables(target, blank=0):
    """What k_ctc.cu:ctc_build_kernel writes for one target: CSR by destination, in-arcs of node l in
    the order skip (l-2), step (l-1), self (l); all weights 0."""
    U = len(target)
    L = 2 * U + 1
    flags = np.zeros(L, np.uint8)
    flags[0] |= 1
    flags[L - 1] |= 2
    if L > 1:
        flags[L - 2] |= 2
    ptr, src, lab = [0], [], []
    for l in range(L):
        label = int(target[(l - 1) // 2]) if l % 2 else blank
        if l % 2 and l > 1 and label != int(target[(l - 3) // 2]):
            src.append(l - 2), lab.append(label)
        if l > 0:
            src.append(l - 1), lab.append(label)
        src.append(l), lab.append(label)
        ptr.append(len(src))
    return flags, np.array(ptr, np.int32), np.array(src, np.int32), np.array(lab, np.int32), np.zeros(len(src), np.float32)


def run(lib, e, tables, lens):
    B, T, Cn = e.shape
    e = np.ascontiguousarray(e, np.float32)
    nn = np.array([len(t[0]) for t in tables], np.int32)
    flags = np.ascontiguousarray(np.concatenate([t[0] for t in tables]), np.uint8)
    ptr = np.ascontiguousarray(np.concatenate([t[1] for t in tables]), np.int32)
    src = np.ascontiguousarray(np.concatenate([t[2] for t in tables]), np.int32)
    lab = np.ascontiguousarray(np.concatenate([t[3] for t in tables]), np.int32)
    w = np.ascontiguousarray(np.concatenate([t[4] for t in tables]), np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    out = np.zeros(B, np.float32)
    grad = np.zeros((B, T, Cn), np.float32)
    status = np.zeros(B, np.int32)
    rc = lib.emu_implicit(B, T, Cn, e.ctypes.data_as(f32p), lens.ctypes.data_as(i32p), nn.ctypes.data_as(i32p),
                          flags.ctypes.data_as(u8p), ptr.ctypes.data_as(i32p), src.ctypes.data_as(i32p),
                          lab.ctypes.data_as(i32p), w.ctypes.data_as(f32p), out.ctypes.data_as(f32p),
                          grad.ctypes.data_as(f32p), status.ctypes.data_as(i32p))
    emu_build.check(rc)
    return out, grad, status


def float64_gradient(x, target):
    """d loss / d emissions of the same lattice evaluated in float64 (oracle/f64.py): the referee when two
    fp32 evaluations differ by more than the tolerance -- the oracle's own fp32 gradient is 5e-4 off it at
    T=270, C=8 (tests/golden/README.md has the T=1000 figures)."""
    from oracle import f64
    return f64.ctc_f64(x, target)[1]


def check_against_oracle(oracle, e, targets, lens, out, grad, T):
    for b in range(e.shape[0]):
        Tb = int(lens[b])
        lo, go = oracle.ctc_loss(e[b, :Tb], targets[b], 0, True)
        x = e[b, :Tb].astype(np.float64)
        mx = x.max(1, keepdims=True)
        lse = mx[:, 0] + np.log(np.exp(x - mx).sum(1))
        if not np.isfinite(lo):
            assert not np.isfinite(out[b])
            continue
        assert util.close(float(lse.sum() - np.float64(out[b])), lo), (b, out[b], lo)
        g = np.exp(x - lse[:, None]) + grad[b, :Tb]  # normaliser's softmax + (-1) x lattice posterior
        if not util.grad_close(g, go, 5.0 * T):
            g64 = float64_gradient(x, targets[b])
            assert np.abs(g - g64).max() <= np.abs(go - g64).max(), (b, float(np.abs(g - go).max()))
        assert not grad[b, Tb:].any()


# (B, T, C, U).  Fast path: T below / at / above one and three 8-frame prefetch blocks, one to seven node
# warps (the named barrier), T == 2U+1.  (1, 40, 8, 130): 261 graph nodes > 256 threads -> general path.
SHAPES = [(2, 5, 4, 1), (3, 13, 6, 3), (2, 9, 5, 4), (2, 31, 8, 12), (2, 40, 16, 18), (1, 57, 28, 26), (1, 24, 5, 11),
          (1, 230, 64, 100), (1, 270, 8, 130)]


@pytest.mark.parametrize("shape", SHAPES)
def test_implicit_kernel_source_matches_oracle(emu, oracle, shape):
    B, T, Cn, U = shape
    e, targets = util.bench_inputs(B, T, Cn, U, seed=8642)
    if U > 2:
        for t in targets:
            t[1] = t[0]  # a repeated label: no skip arc
    lens = np.minimum(np.array([max(T - 5 * b, 2 * U) for b in range(B)], np.int32), T)
    out, grad, status = run(emu, e, [ctc_tables(t) for t in targets], lens)
    assert not status.any(), status
    check_against_oracle(oracle, e, targets, lens, out, grad, T)


def test_implicit_kernel_reports_non_finite_emissions(emu):
    B, T, Cn, U = 1, 12, 5, 3
    e, targets = util.bench_inputs(B, T, Cn, U, seed=5)
    e[0, 4, int(targets[0][1])] = -np.inf
    out, grad, status = run(emu, e, [ctc_tables(t) for t in targets], np.array([T], np.int32))
    assert status[0] & 1


@pytest.mark.parametrize("shape", [(3, 21, 7, 4), (2, 40, 16, 18), (1, 30, 64, 100 // 8), (2, 9, 6, 0)])
def test_ctc_build_kernel_then_sweeps(emu, oracle, shape):
    """The criterion's device side end to end: k_ctc.cu's ctc_build_kernel (tables of the target graph,
    benchmarks/ctc.cpp:40-58) feeding the sweeps; graph 0's tables against the restatement above."""
    B, T, Cn, U = shape
    e, targets = util.bench_inputs(B, T, Cn, max(U, 1), seed=97)
    if U == 0:
        targets = [t[:0] for t in targets]  # empty transcript: the single blank node
    elif U > 2:
        targets[0][1] = targets[0][0]
    lens = np.minimum(np.array([max(T - 3 * b, 2 * U + 1) for b in range(B)], np.int32), T)
    e = np.ascontiguousarray(e, np.float32)
    cat = np.ascontiguousarray(np.concatenate(targets) if U else np.zeros(1), np.int32)
    tl = np.array([len(t) for t in targets], np.int32)
    out = np.zeros(B, np.float32)
    grad = np.zeros((B, T, Cn), np.float32)
    status = np.zeros(B, np.int32)
    N0 = 2 * len(targets[0]) + 1
    ptr0 = np.zeros(N0 + 1, np.int32)
    src0 = np.zeros(3 * N0, np.int32)
    lab0 = np.zeros(3 * N0, np.int32)
    rc = emu.emu_implicit_ctc(B, T, Cn, e.ctypes.data_as(f32p), lens.ctypes.data_as(i32p), cat.ctypes.data_as(i32p),
                              tl.ctypes.data_as(i32p), 0, out.ctypes.data_as(f32p), grad.ctypes.data_as(f32p),
                              status.ctypes.data_as(i32p), ptr0.ctypes.data_as(i32p), src0.ctypes.data_as(i32p),
                              lab0.ctypes.data_as(i32p))
    emu_build.check(rc)
    assert not status.any()
    _, ptr, src, lab, _ = ctc_tables(targets[0])
    assert np.array_equal(ptr0, ptr)
    assert np.array_equal(src0[:ptr[-1]], src) and np.array_equal(lab0[:ptr[-1]], lab)
    check_against_oracle(oracle, e, targets, lens, out, grad, T)


def test_kernel_sources_at_the_benchmark_shape_against_the_reference_golden(emu):
    """One utterance of BASELINE config 2 (T=1000, C=64, U=100: 201 graph nodes, 7 node warps) through the
    source of k_ctc.cu + k_implicit.cu against the golden vector generated from the real reference
    (tests/golden/make_golden.py) and its float64 evaluation."""
    gold = np.load(os.path.join(HERE, "golden", "reference_golden.npz"))
    e, tg = util.bench_inputs(1, 1000, 64, 100)
    T, Cn = 1000, 64
    x = e[0].astype(np.float64)
    mx = x.max(1, keepdims=True)
    lse = mx[:, 0] + np.log(np.exp(x - mx).sum(1))
    soft = np.exp(x - lse[:, None])

    cat = np.ascontiguousarray(tg[0], np.int32)
    tl = np.array([len(tg[0])], np.int32)
    lens = np.array([T], np.int32)
    out = np.zeros(1, np.float32)
    grad = np.zeros((1, T, Cn), np.float32)
    status = np.zeros(1, np.int32)
    ee = np.ascontiguousarray(e, np.float32)
    rc = emu.emu_implicit_ctc(1, T, Cn, ee.ctypes.data_as(f32p), lens.ctypes.data_as(i32p), cat.ctypes.data_as(i32p),
                              tl.ctypes.data_as(i32p), 0, out.ctypes.data_as(f32p), grad.ctypes.data_as(f32p),
                              status.ctypes.data_as(i32p), None, None, None)
    emu_build.check(rc)
    assert not status.any()
    loss = float(lse.sum() - np.float64(out[0]))
    assert util.close(loss, gold["c2_loss"][0]), (loss, gold["c2_loss"][0])
    assert abs(loss - float(gold["c2_loss_f64"])) < 1e-3 * abs(loss)
    g = soft + grad[0]
    # two fp32 evaluations of this lattice differ by ~1e-3 (tests/golden/README.md): the float64
    # gradient is the referee, and the kernel must be no further from it than the reference is
    g64 = gold["c2_grad_f64"]  # [T][C]
    assert g64.shape == g.shape
    err_kernel = np.abs(g - g64).max()
    err_reference = np.abs(gold["c2_grad"][0] - g64).max()
    assert util.grad_close(g, gold["c2_grad"][0], 5.0 * T) or err_kernel <= err_reference, err_kernel
    assert np.allclose(-grad[0].sum(1), 1.0, atol=2e-3)


def general_tables(og, Cn):
    """CSR by destination of an oracle graph, in-arcs ordered by (source, arc id) like gtnb_compose_linear."""
    a = og.arrays()
    N = len(a["flags"])
    ptr, src, lab, arc, w = [0], [], [], [], []
    for d in range(N):
        for k in sorted(np.nonzero(a["dst"] == d)[0].tolist(), key=lambda k: (int(a["src"][k]), k)):
            src.append(int(a["src"][k])), lab.append(int(a["ilabel"][k])), arc.append(k), w.append(float(a["w"][k]))
        ptr.append(len(src))
    return (a["flags"].astype(np.uint8), np.array(ptr, np.int32), np.array(src, np.int32), np.array(lab, np.int32),
            np.array(w, np.float32), np.array(arc, np.int32))


@pytest.mark.parametrize("Cn,T", [(6, 9), (20, 7), (40, 5), (64, 4)])
def test_wide_kernels_on_asg_transitions(emu, Cn, T):
    """forwardScore(compose(transitions, emissions)) and its backward for the dense ASG transitions graph
    (start -> c and c' -> c for every pair, test/criterion_test.cpp:244-254): in- / out-degrees above three take
    the G-lanes-per-node kernels, arc gradients of the graph operand included (the ASG denominator of
    BASELINE config 3).  Oracle: its own compose + shortest-distance gradient + compose gradFunc."""
    from oracle import pyoracle as po
    rng = np.random.default_rng(Cn)
    tw = rng.uniform(-2, 2, Cn + Cn * Cn).astype(np.float32)
    B = 2
    e = rng.uniform(-3, 3, (B, T, Cn)).astype(np.float32)
    lens = np.array([T, T - 2], np.int32)
    og = po.Graph.transitions(Cn, tw)
    tab = general_tables(og, Cn)
    A = len(tab[2])
    nn = np.array([len(tab[0])] * B, np.int32)
    catb = lambda k, dt: np.ascontiguousarray(np.concatenate([tab[k]] * B), dt)
    flags, ptr, src, lab, w, arc = catb(0, np.uint8), catb(1, np.int32), catb(2, np.int32), catb(3, np.int32), catb(4, np.float32), catb(5, np.int32)
    out = np.zeros(B, np.float32)
    grad = np.zeros((B, T, Cn), np.float32)
    gg = np.zeros(B * A, np.float32)
    status = np.zeros(B, np.int32)
    deltas = np.array([1.0, -0.5], np.float32)
    ee = np.ascontiguousarray(e)
    emu.emu_implicit_general.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, i32p, u8p, i32p, i32p, i32p, i32p, f32p,
                                         f32p, f32p, f32p, f32p, i32p]
    G = emu.emu_implicit_general(B, T, Cn, ee.ctypes.data_as(f32p), lens.ctypes.data_as(i32p), nn.ctypes.data_as(i32p),
                                 flags.ctypes.data_as(u8p), ptr.ctypes.data_as(i32p), src.ctypes.data_as(i32p),
                                 lab.ctypes.data_as(i32p), arc.ctypes.data_as(i32p), w.ctypes.data_as(f32p),
                                 deltas.ctypes.data_as(f32p), out.ctypes.data_as(f32p), grad.ctypes.data_as(f32p),
                                 gg.ctypes.data_as(f32p), status.ctypes.data_as(i32p))
    if G == -77:
        pytest.skip("the host refused to create the emulator's threads")
    assert G > 0, G  # the wide kernels were used
    assert not status.any()
    for b in range(B):
        Tb = int(lens[b])
        lin = po.Graph.linear(Tb, Cn, e[b, :Tb])
        comp = po.compose(og, lin)
        score, arc_grads = po.forward_score_and_grad(comp, False, float(deltas[b]))
        g1, g2 = po.compose_grad(comp, arc_grads, len(og.arrays()["src"]), Tb * Cn)
        assert util.close(out[b], score), (b, out[b], score)
        assert util.grad_close(grad[b, :Tb].reshape(-1), g2, 5.0 * T), b
        assert not grad[b, Tb:].any()
        mine = np.zeros(A, np.float32)
        mine[:] = gg[b * A:(b + 1) * A]  # indexed by Graph arc id through in_arc
        assert util.grad_close(mine, g1, 5.0 * T), (b, float(np.abs(mine - g1).max()))
