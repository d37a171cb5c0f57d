"""CPU checks for gtnb_graph_transitions_loss: the committed golden fixture (tests/golden/graph_trans_golden.npz,
tests/golden/make_graph_trans_golden.py) against the live reference through tests/graph_trans_oracle.py; the shipped
host builder of the numerator products (gtn_b200/csrc/gtnb_product.h), folded and unfolded, against the reference's
compose(A_b, G) / intersect(A_b, G); the source of the product fold kernel through the SIMT emulator against numpy,
bit for bit; and the C-ABI symbol."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from tests import emu_build
from tests import graph_oracle as go
from tests import graph_trans_oracle as gt
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "graph_trans_golden.npz")
KINDS = {"asg": gt.ASG, "bigram": gt.BIGRAM}
f32p, i32p, u8p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)


def graphs_of(z, name):
    out, n0, a0 = [], 0, 0
    for n, a in zip(z[name + "_n_nodes"], z[name + "_n_arcs"]):
        g = {"flags": z[name + "_flags"][n0:n0 + n]}
        for k in ("src", "dst", "ilabel", "olabel", "w"):
            g[k] = z[name + "_" + k][a0:a0 + a]
        out.append(g)
        n0, a0 = n0 + n, a0 + a
    return out


def need_ref(oracle):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref/libgtn_ref.so is missing")


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("name", ["a", "b", "c"])
def test_golden_matches_live_reference(oracle, name, kind):
    need_ref(oracle)
    z = np.load(GOLDEN)
    p = "%s_%s_" % (name, kind)
    lo, gr, ag, tg = gt.ref_graph_trans_loss(z[name + "_e"], graphs_of(z, name), KINDS[kind], z[p + "trans_w"],
                                             z[name + "_lens"])
    assert util.close(lo, z[p + "losses"])
    assert util.close(gr, z[p + "grads"]) and util.close(ag, z[p + "arc_grads"]) and util.close(tg, z[p + "trans_grad"])


def test_golden_cases_are_what_the_docstring_says():
    z = np.load(GOLDEN)
    a, b = graphs_of(z, "a"), graphs_of(z, "b")
    assert (a[2]["olabel"] >= 7).any() and (b[3]["olabel"] >= 12).any()
    starts = np.flatnonzero(a[2]["flags"] & 1)
    assert len(starts) >= 2 and np.isin(a[2]["dst"], starts).any()  # start nodes with in-arcs
    assert go.non_uniform_nodes(b[1], 12) > 0  # wildcards
    for kind in KINDS:
        assert np.isposinf(z["a_%s_losses" % kind][3]) and np.isnan(z["b_%s_losses" % kind][2])
        assert not z["b_%s_grads" % kind][2].any()
        assert np.isneginf(z["c_%s_trans_w" % kind]).any() and not np.isneginf(z["a_%s_trans_w" % kind]).any()
    assert z["a_lens"].min() == 1 and z["b_lens"].min() == 0


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("product", ["k_ngram.cu", "k_implicit.cu", "gtnb_product.h"]))
    lib.emu_build_product.argtypes = [C.c_int, C.c_int, u8p, i32p, i32p, i32p, f32p, C.c_int, C.c_int, C.c_int, f32p,
                                      i32p, i32p, u8p, i32p, i32p, i32p, i32p, i32p, f32p]
    lib.emu_product_fold.argtypes = [C.c_longlong, f32p, i32p, f32p, C.c_int, f32p, i32p, f32p]
    return lib


def _p(a, t):
    return a.ctypes.data_as(t)


def build_product(emu, g, Cn, kind, fold, Wx):
    """-> product arrays (graph_oracle layout) + arc_of, tidx, through the shipped builder"""
    flags, src, dst = (np.ascontiguousarray(g[k], t) for k, t in (("flags", np.uint8), ("src", np.int32),
                                                                   ("dst", np.int32)))
    ol, w = np.ascontiguousarray(g["olabel"], np.int32), np.ascontiguousarray(g["w"], np.float32)
    Wx = np.ascontiguousarray(Wx, np.float32)
    nn, na = C.c_int(), C.c_int()
    args = [len(flags), len(src), _p(flags, u8p), _p(src, i32p), _p(dst, i32p), _p(ol, i32p), _p(w, f32p), Cn,
            int(kind == gt.BIGRAM), int(fold), _p(Wx, f32p), C.byref(nn), C.byref(na)]
    emu.emu_build_product(*args, *([None] * 7))
    N, A = nn.value, na.value
    out = [np.zeros(N, np.uint8)] + [np.zeros(max(A, 1), np.int32) for _ in range(5)] + [np.zeros(max(A, 1), np.float32)]
    emu.emu_build_product(*args, _p(out[0], u8p), *[_p(o, i32p) for o in out[1:6]], _p(out[6], f32p))
    fl, s, d, lab, arc_of, tidx, pw = out[0], *[o[:A] for o in out[1:]]
    return go.make(fl, s, d, lab, w=pw), arc_of, tidx


PRODUCT_CASES = [(name, kind, fold) for name in ("a", "b") for kind in KINDS
                 for fold in ((False, True) if kind == "bigram" else (False,))]


@pytest.mark.parametrize("name,kind,fold", PRODUCT_CASES)
def test_product_builder_matches_reference_composition(oracle, emu, name, kind, fold):
    """forwardScore(compose(P_b, E_b)) of the built product = the reference's numerator, and the product's arc
    gradients mapped back through arc_of / tidx (and, folded, through sigma) = the reference's A_b and G gradients"""
    need_ref(oracle)
    po = oracle
    z = np.load(GOLDEN)
    e, lens = z[name + "_e"], z[name + "_lens"]
    Cn = e.shape[2]
    k = KINDS[kind]
    tw = z["%s_%s_trans_w" % (name, kind)]
    CC = Cn * Cn
    if k == gt.BIGRAM:
        W = tw.reshape(Cn, Cn).astype(np.float64)
        sigma = (np.log(np.exp(W - W.max(1, keepdims=True)).sum(1)) + W.max(1)).astype(np.float32)
        Wx = np.concatenate([tw, sigma])
    else:
        Wx = tw
    op = "compose" if k == gt.ASG else "intersect"
    gd, slot = gt.dense_graph(k, Cn, tw)
    for b, g in enumerate(graphs_of(z, name)):
        Tb = int(lens[b])
        if Tb == 0:
            continue
        P, arc_of, tidx = build_product(emu, g, Cn, k, fold, Wx)
        E = po.RefGraph.linear(Tb, Cn, e[b, :Tb].ravel())
        rp = go.ref_graph(P)
        s = po.ref_op("forward_score", po.ref_op("compose", rp, E))
        po.ref_backward(s)
        A, G = go.ref_graph(g), go.ref_graph(gd)
        E2 = po.RefGraph.linear(Tb, Cn, e[b, :Tb].ravel())
        want = po.ref_op("forward_score", po.ref_op(op, po.ref_op(op, A, G), E2))
        po.ref_backward(want)
        assert util.close(s.item(), want.item()), (b, s.item(), want.item())
        if not math.isfinite(want.item()):
            continue
        pg = rp.grad().weights().astype(np.float64) if len(P["src"]) else np.zeros(0)
        ag = np.bincount(arc_of, pg, minlength=len(g["src"]))
        tgx = np.zeros(len(Wx))
        np.add.at(tgx, tidx, pg)
        tg = tgx[:len(tw)].copy()
        if k == gt.BIGRAM:  # the folded start arcs: d sigma_l / d W[l][j] = softmax_j(W[l][:])
            tg += (tgx[CC:, None] * np.exp(W - sigma[:, None].astype(np.float64))).ravel()
        tg_ref = np.zeros(len(tw))
        np.add.at(tg_ref, slot, G.grad().weights().astype(np.float64))
        mag = abs(want.item())
        assert util.grad_close(ag, A.grad().weights() if len(g["src"]) else np.zeros(0), mag), b
        assert util.grad_close(tg, tg_ref, mag), (b, np.abs(tg - tg_ref).max())
        assert util.grad_close(E.grad().weights(), E2.grad().weights(), mag), b


def test_product_sizes(emu):
    """one copy per (node, distinct in-label), one arc per (arc, copy of its source); a wildcard node at C labels
    becomes C copies with C in-arcs each"""
    Cn = 5
    wild = go.make([3], [0] * Cn, [0] * Cn, list(range(Cn)))
    for kind, fold, nodes, arcs in ((gt.ASG, False, 1 + Cn, Cn + Cn * Cn), (gt.BIGRAM, False, Cn, Cn * Cn),
                                    (gt.BIGRAM, True, 1 + Cn, Cn + Cn * Cn)):
        Wx = np.zeros(Cn + Cn * Cn, np.float32)
        P, _, _ = build_product(emu, wild, Cn, kind, fold, Wx)
        assert (len(P["flags"]), len(P["src"])) == (nodes, arcs)
    chain = go.make([1, 0, 2], [0, 1, 1], [1, 2, 2], [3, 9, 1])  # label 9 >= C never matches
    P, arc_of, tidx = build_product(emu, chain, Cn, gt.ASG, False, np.arange(Cn + Cn * Cn, dtype=np.float32))
    assert list(P["flags"]) == [1, 0, 2] and list(arc_of) == [0, 2] and list(tidx) == [3, Cn + 1 * Cn + 3]


@pytest.mark.parametrize("n,nW,with_sigma", [(1, 4, False), (257, 30, False), (1000, 12, True), (5000, 16384, True)])
def test_fold_kernel_matches_numpy_bitwise(emu, n, nW, with_sigma):
    rng = np.random.default_rng(n)
    n_arcs = max(n // 3, 1)
    w_A = rng.normal(size=n_arcs).astype(np.float32)
    W = rng.normal(size=nW).astype(np.float32)
    sigma = rng.normal(size=64).astype(np.float32)
    arc_of = rng.integers(0, n_arcs, n).astype(np.int32)
    tidx = rng.integers(0, nW + (64 if with_sigma else 0), n).astype(np.int32)
    out = np.full(n, np.nan, np.float32)
    emu_build.check(emu.emu_product_fold(n, _p(w_A, f32p), _p(arc_of, i32p), _p(W, f32p), nW, _p(sigma, f32p),
                                         _p(tidx, i32p), _p(out, f32p)))
    Wx = np.concatenate([W, sigma])
    want = w_A[arc_of] + Wx[tidx]
    assert np.array_equal(out.view(np.int32), want.view(np.int32))


def test_symbol_declared_and_exported():
    from gtn_b200 import capi
    assert "gtnb_graph_transitions_loss" in [s[0] for s in capi.SYMBOLS]
    with open(os.path.join(ROOT, "include", "gtn_b200.h")) as f:
        assert "int gtnb_graph_transitions_loss(" in f.read()
    so = os.path.join(ROOT, "gtn_b200", "lib", "libgtn_b200.so")
    if not os.path.exists(so):
        pytest.skip("the library is not built")
    assert hasattr(C.CDLL(so), "gtnb_graph_transitions_loss")
