"""gtnb_sparse_transitions_viterbi's device route end to end, every step from its source on the CPU: the shipped builder's
folded sparse products (gtnb_product.h, through tests/emu/sparse_emu.cpp), sparse_tau_kernel for the folded start arcs
(tests/emu/sparse_viterbi_emu.cpp), product_fold_kernel with Wx = [trans_w | tau], k_implicit.cu's tropical forward and
implicit_trace_kernel (tests/emu/graph_viterbi_emu.cpp), then product_arc_map_kernel -- as
tests/test_graph_trans_viterbi_emulation.py runs it for the dense kinds.  Against the committed fixture
(tests/golden/sparse_viterbi_golden.npz: random sparse G with -inf weights, the tie-heavy trigram, the trigram at
C = 30) and, on random sparse G and the trigram, tie-free and tie-heavy, against the live reference: scores bit-equal,
paths and arcs == wherever the tie bit is not raised, the tie bit raised exactly where the float32 restatement
(graph_trans_viterbi_oracle.device_route_outcome over the folded product) finds a tie on the traced path, the
non-finite bit exactly where a product weight or emission is not finite."""
import ctypes as C

import numpy as np
import pytest

from tests import emu_build
from tests import graph_oracle as go
from tests import graph_trans_viterbi_oracle as gtv
from tests import sparse_trans_oracle as st
from tests import sparse_viterbi_oracle as sv
from tests.test_graph_trans_oracle import need_ref
from tests.test_graph_trans_viterbi_emulation import product_emu, trace_lib  # noqa: F401  (fixtures)
from tests.test_sparse_trans_oracle import _p, build_product, emu  # noqa: F401  (emu: the sparse builder)
from tests.test_sparse_viterbi_emulation import tau

f32p, i32p, i64p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_longlong)


@pytest.fixture(scope="module")
def kernels():
    """sparse_tau_kernel (sparse_viterbi_emu.cpp) and product_arc_map_kernel (graph_trans_viterbi_emu.cpp)"""
    from tests.test_sparse_viterbi_emulation import load
    vit = load()
    arcmap = C.CDLL(emu_build.build("graph_trans_viterbi", ["k_ngram.cu", "k_implicit.cu"]))
    arcmap.emu_product_arc_map.argtypes = [C.c_int, C.c_int, i64p, i32p, i32p]
    return vit, arcmap


def device_route(emu, product_emu, trace_lib, kernels, e, graphs, lens, G, tw):  # noqa: F811
    """-> (paths, scores, arcs, status, folded products)"""
    from tests.test_graph_viterbi_emulation import run as run_trace
    vit, arcmap = kernels
    B, T, C_ = e.shape
    tw = np.ascontiguousarray(tw, np.float32)
    t = np.ascontiguousarray(tau(vit, G, tw, C_), np.float32)
    Wx = np.concatenate([tw, t])
    prods, arc_of, tidx, w_A, uniform = [], [], [], [], True
    off = np.zeros(2 * B, np.int64)
    for b, g in enumerate(graphs):
        p, ao, ti, un = build_product(emu, g, G, C_, True, Wx)
        if b + 1 < B:
            off[b + 1] = off[b] + len(ao)
            off[B + b + 1] = off[B + b] + len(g["src"])
        prods.append(p)
        arc_of.append(ao + off[B + b])
        tidx.append(ti)
        w_A.append(np.asarray(g["w"], np.float32))
        uniform &= un
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0), dt)  # noqa: E731
    arc_of, tidx, w_A = cat(arc_of, np.int32), cat(tidx, np.int32), cat(w_A, np.float32)
    fw = np.zeros(max(len(arc_of), 1), np.float32)
    tt = np.ascontiguousarray(np.r_[t, np.float32(0)], np.float32)
    emu_build.check(product_emu.emu_product_fold(len(arc_of), _p(w_A, f32p), _p(arc_of, i32p), _p(tw, f32p), len(tw),
                                                 _p(tt, f32p), _p(tidx, i32p), _p(fw, f32p)))
    for b, p in enumerate(prods):
        w = fw[off[b]:off[b] + len(p["src"])]
        assert w.tobytes() == p["w"].tobytes()  # the fold kernel gives the host builder's weights
        p["w"] = w.copy()
    paths, scores, parcs, status, _ = run_trace(trace_lib, e, prods, lens, arc=not uniform)
    arcs = np.ascontiguousarray(parcs, np.int32)
    emu_build.check(arcmap.emu_product_arc_map(B, T, _p(off, i64p), _p(arc_of, i32p), _p(arcs, i32p)))
    return paths, scores, arcs, status, prods


def check(emu, product_emu, trace_lib, kernels, e, graphs, lens, G, tw, want):  # noqa: F811
    """the device route against `want` (the reference's paths, scores, arcs) -> (ties, non-finite)"""
    p, s, a, status, prods = device_route(emu, product_emu, trace_lib, kernels, e, graphs, lens, G, tw)
    pr, sr, ar = want
    C_ = e.shape[2]
    n_tie = n_bad = 0
    for b, g in enumerate(graphs):
        Tb = int(lens[b])
        if Tb == 0:
            assert np.isneginf(s[b]) and (p[b] == -1).all() and (a[b] == -1).all()
            continue
        bad = not (np.isfinite(prods[b]["w"]).all() and np.isfinite(e[b, :Tb]).all())
        assert bool(status[b] & 1) == bad, (b, status[b])
        if bad:  # the exact route's
            n_bad += 1
            continue
        want_score, tie = gtv.device_route_outcome(e[b, :Tb], prods[b], C_)
        assert s[b].tobytes() == sr[b].tobytes() == want_score.tobytes(), (b, s[b], sr[b])
        assert bool(status[b] & 2) == tie, (b, status[b], tie)
        assert (p[b, Tb:] == -1).all() and (a[b, Tb:] == -1).all()
        if not tie:
            assert np.array_equal(p[b], pr[b]) and np.array_equal(a[b], ar[b]), b
        else:
            n_tie += 1
            assert sv.is_path(g, a[b, :Tb]) and np.array_equal(g["olabel"][a[b, :Tb]], p[b, :Tb])
    return n_tie, n_bad


@pytest.mark.parametrize("case", range(len(sv.NAMES)))
def test_device_route_end_to_end_on_the_golden_batches(emu, product_emu, trace_lib, kernels, case):  # noqa: F811
    name, e, lens, G, tw, graphs, _, ali = sv.golden_batches()[case]
    keep = [i for i, g in enumerate(graphs) if len(g["flags"])]  # (the empty graph's product accepts nothing)
    graphs, lens, e = [graphs[i] for i in keep], np.ascontiguousarray(lens[keep]), np.ascontiguousarray(e[keep])
    ali = tuple(x[keep] for x in ali)
    n_tie, n_bad = check(emu, product_emu, trace_lib, kernels, e, graphs, lens, G, tw, ali)
    if name == "b":
        assert n_tie > 0


@pytest.mark.parametrize("graph", ["sparse", "trigram"])
@pytest.mark.parametrize("ties", [False, True])
def test_device_route_end_to_end_random(oracle, emu, product_emu, trace_lib, kernels, graph, ties):  # noqa: F811
    need_ref(oracle)
    rng = np.random.default_rng(200 + 2 * (graph == "trigram") + ties)
    C_, T = 5, 8
    G = st.trigram_graph(C_) if graph == "trigram" else st.sparse_graph(rng, 7, 40, C_, n_start=3, n_accept=3,
                                                                         label_hi=C_ + 1)
    graphs = [go.ctc_graph(rng.integers(1, C_, 2)), go.random_graph(rng, 6, 20, C_, n_start=2, n_accept=2),
              go.with_wildcards(go.ctc_graph([2]), C_), go.ctc_graph(rng.integers(1, C_, 3))]
    for g in graphs:
        g["w"] = (rng.integers(-1, 1, len(g["src"])) if ties else rng.uniform(-1, 1, len(g["src"]))).astype(np.float32)
    tw = (np.zeros(len(G["src"])) if ties else rng.uniform(-1, 1, len(G["src"]))).astype(np.float32)
    lens = rng.integers(1, T + 1, len(graphs)).astype(np.int32)
    e = (rng.integers(0, 2, (len(graphs), T, C_)) if ties else rng.uniform(-3, 3, (len(graphs), T, C_)))
    e = e.astype(np.float32)
    want = sv.ref_sparse_trans_viterbi(e, graphs, G, tw, lens)
    n_tie, n_bad = check(emu, product_emu, trace_lib, kernels, e, graphs, lens, G, tw, want)
    assert n_bad == 0 and (n_tie > 0) == ties
