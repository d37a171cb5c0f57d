"""CPU checks for gtnb_sparse_transitions_loss: the committed golden fixture (tests/golden/sparse_trans_golden.npz,
tests/golden/make_sparse_trans_golden.py) against the live reference through tests/sparse_trans_oracle.py; the shipped
host builder of the numerator products (gtn_b200/csrc/gtnb_product.h), folded and unfolded, against the reference's
intersect(intersect(A_b, G), E_b), scores and gradients mapped back through arc_of / tidx (and sigma); the C-ABI
symbol."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from tests import emu_build
from tests import graph_oracle as go
from tests import sparse_trans_oracle as st
from tests import util
from tests.test_graph_trans_oracle import graphs_of, need_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sparse_trans_golden.npz")
f32p, i32p, u8p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)
ip = C.POINTER(C.c_int)


def G_of(z, name):
    return go.make(z[name + "_G_flags"], z[name + "_G_src"], z[name + "_G_dst"], z[name + "_G_label"])


@pytest.mark.parametrize("name", ["a", "b", "c"])
def test_golden_matches_live_reference(oracle, name):
    need_ref(oracle)
    z = np.load(GOLDEN)
    lo, gr, ag, tg = st.ref_sparse_trans_loss(z[name + "_e"], graphs_of(z, name), G_of(z, name),
                                              z[name + "_trans_w"], z[name + "_lens"])
    assert util.close(lo, z[name + "_losses"])
    assert util.close(gr, z[name + "_grads"]) and util.close(ag, z[name + "_arc_grads"])
    assert util.close(tg, z[name + "_trans_grad"])


def test_golden_cases_are_what_the_docstring_says():
    z = np.load(GOLDEN)
    a, Ga, Gb = graphs_of(z, "a"), G_of(z, "a"), G_of(z, "b")
    assert len(Ga["flags"]) == 25 and len(Ga["src"]) == 125 and (Ga["flags"] == 3).all()  # the trigram at C = 5
    assert (Gb["olabel"] >= 12).any() and (Gb["flags"] & 1).sum() >= 2 and (Gb["flags"] & 2).sum() >= 2
    assert (a[1]["olabel"] >= 5).any()
    assert np.isposinf(z["a_losses"][2]) and np.isnan(z["b_losses"][1]) and not z["b_grads"][1].any()
    assert np.isneginf(z["c_trans_w"]).any() and np.isfinite(z["c_losses"]).all()
    assert z["a_lens"].min() == 1 and z["b_lens"].min() == 0


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("sparse", ["k_sparse.cu", "gtnb_product.h"]))
    lib.emu_sparse_product.argtypes = [C.c_int, C.c_int, u8p, i32p, i32p, i32p, f32p, C.c_int, C.c_int, u8p, i32p,
                                       i32p, i32p, C.c_int, C.c_int, f32p, ip, ip, ip, ip, u8p, i32p, i32p, i32p,
                                       i32p, i32p, f32p]
    lib.emu_sparse_den.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, C.c_int, C.c_int, u8p, i32p, i32p, i32p,
                                   f32p, C.c_int, f32p, f32p, f32p, f32p, i32p]
    lib.emu_sparse_fold.argtypes = [C.c_int, C.c_int, u8p, i32p, i32p, i32p, C.c_int, f32p, f32p, f32p]
    return lib


def _p(a, t):
    return a.ctypes.data_as(t)


def graph_args(g):
    arrs = [np.ascontiguousarray(g["flags"], np.uint8)] + \
           [np.ascontiguousarray(g[k], np.int32) for k in ("src", "dst", "olabel")]
    return arrs, [_p(arrs[0], u8p)] + [_p(a, i32p) for a in arrs[1:]]


def start_groups(G, Cn):
    """G's start groups as gtnb_product.h numbers them: arcs out of start nodes with a label in [0, C), grouped by
    (destination, label) in order of first appearance"""
    keys, members = {}, []
    for a in range(len(G["src"])):
        lab = int(G["olabel"][a])
        if 0 <= lab < Cn and G["flags"][G["src"][a]] & 1:
            k = (int(G["dst"][a]), lab)
            if k not in keys:
                keys[k] = len(members)
                members.append([])
            members[keys[k]].append(a)
    return members


def sigma_of(tw, groups):
    out = []
    for m in groups:
        w = tw[m].astype(np.float64)
        mx = w.max()
        out.append(-np.inf if mx == -np.inf else mx + np.log(np.exp(w - mx).sum()))
    return np.asarray(out, np.float32)


def build_product(emu, g, G, Cn, fold, Wx):
    """-> product arrays (graph_oracle layout), arc_of, tidx, uniform, through the shipped builder"""
    ka, aa = graph_args(g)
    kg, ga = graph_args(G)
    w = np.ascontiguousarray(g["w"], np.float32)
    Wx = np.ascontiguousarray(Wx, np.float32)
    nn, na, ng, un = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    args = [len(g["flags"]), len(g["src"]), *aa, _p(w, f32p), len(G["flags"]), len(G["src"]), *ga, Cn, int(fold),
            _p(Wx, f32p), C.byref(nn), C.byref(na), C.byref(ng), C.byref(un)]
    emu.emu_sparse_product(*args, *([None] * 7))
    N, A = nn.value, na.value
    out = [np.zeros(N, np.uint8)] + [np.zeros(max(A, 1), np.int32) for _ in range(5)] + [np.zeros(max(A, 1), np.float32)]
    emu.emu_sparse_product(*args, _p(out[0], u8p), *[_p(o, i32p) for o in out[1:6]], _p(out[6], f32p))
    fl, s, d, lab, arc_of, tidx, pw = out[0], *[o[:A] for o in out[1:]]
    return go.make(fl, s, d, lab, w=pw), arc_of, tidx, bool(un.value)


@pytest.mark.parametrize("name", ["a", "b", "c"])
@pytest.mark.parametrize("fold", [False, True])
def test_product_builder_matches_reference_intersection(oracle, emu, name, fold):
    """forwardScore(compose(P_b, E_b)) of the built product = the reference's numerator
    forwardScore(intersect(intersect(A_b, G), E_b)); the product's arc gradients mapped back through arc_of / tidx
    (and, folded, through sigma by softmax) = the reference's A_b and G gradients"""
    need_ref(oracle)
    po = oracle
    z = np.load(GOLDEN)
    e, lens, G, tw = z[name + "_e"], z[name + "_lens"], G_of(z, name), z[name + "_trans_w"]
    Cn = e.shape[2]
    groups = start_groups(G, Cn)
    sigma = sigma_of(tw, groups)
    Wx = np.concatenate([tw, sigma])
    nG = len(tw)
    gd = dict(G)
    gd["w"] = tw
    for b, g in enumerate(graphs_of(z, name)):
        Tb = int(lens[b])
        if Tb == 0:
            continue
        P, arc_of, tidx, _ = build_product(emu, g, G, Cn, fold, Wx)
        assert fold or (tidx < nG).all()
        E = po.RefGraph.linear(Tb, Cn, e[b, :Tb].ravel())
        rp = go.ref_graph(P)
        s = po.ref_op("forward_score", po.ref_op("compose", rp, E))
        po.ref_backward(s)
        A, RG = go.ref_graph(g), go.ref_graph(gd)
        E2 = po.RefGraph.linear(Tb, Cn, e[b, :Tb].ravel())
        want = po.ref_op("forward_score", po.ref_op("intersect", po.ref_op("intersect", A, RG), E2))
        po.ref_backward(want)
        assert util.close(s.item(), want.item()), (b, s.item(), want.item())
        if not math.isfinite(want.item()) or not np.isfinite(tw).all():
            continue
        pg = rp.grad().weights().astype(np.float64) if len(P["src"]) else np.zeros(0)
        ag = np.bincount(arc_of, pg, minlength=len(g["src"]))
        tgx = np.zeros(len(Wx))
        np.add.at(tgx, tidx, pg)
        tg = tgx[:nG].copy()
        for k, m in enumerate(groups):  # the folded start arcs: d sigma_k / d w_a = softmax over the group
            tg[m] += tgx[nG + k] * np.exp(tw[m].astype(np.float64) - float(sigma[k]))
        mag = abs(want.item())
        assert util.grad_close(ag, A.grad().weights() if len(g["src"]) else np.zeros(0), mag), b
        assert util.grad_close(tg, RG.grad().weights(), mag), (b, np.abs(tg - RG.grad().weights()).max())
        assert util.grad_close(E.grad().weights(), E2.grad().weights(), mag), b


def test_product_sizes(emu):
    """the trigram's start copies: C^2 per A start node unfolded, one S folded; a CTC graph's folded product is
    label-uniform under the trigram and not under a G whose nodes have in-arcs with several labels"""
    Cn = 4
    G = st.trigram_graph(Cn)
    tw = np.zeros(Cn ** 3, np.float32)
    groups = start_groups(G, Cn)
    assert len(groups) == Cn * Cn  # (destination b*C+m, label m): C arcs each
    Wx = np.concatenate([tw, np.zeros(len(groups), np.float32)])
    ctc = go.ctc_graph([1, 2])
    P, _, tidx, uniform = build_product(emu, ctc, G, Cn, False, Wx)
    assert (P["flags"] & 1).sum() == Cn * Cn and uniform  # one per G node: the CTC graph starts at node 0
    P, _, tidx, uniform = build_product(emu, ctc, G, Cn, True, Wx)
    assert list(np.flatnonzero(P["flags"] & 1)) == [0] and uniform and (tidx >= Cn ** 3).any()
    mixed = go.make([3, 3], [0, 1, 0], [1, 1, 0], [1, 2, 3])  # node 1 entered by labels 1 and 2
    P, _, _, uniform = build_product(emu, go.make([3], [0, 0, 0], [0, 0, 0], [1, 2, 3]), mixed, Cn, True,
                                     np.zeros(3 + 4, np.float32))
    assert not uniform


def test_symbol_declared_and_exported():
    from gtn_b200 import capi
    assert "gtnb_sparse_transitions_loss" in [s[0] for s in capi.SYMBOLS]
    with open(os.path.join(ROOT, "include", "gtn_b200.h")) as f:
        assert "int gtnb_sparse_transitions_loss(" in f.read()
    so = os.path.join(ROOT, "gtn_b200", "lib", "libgtn_b200.so")
    if not os.path.exists(so):
        pytest.skip("the library is not built")
    assert hasattr(C.CDLL(so), "gtnb_sparse_transitions_loss")
