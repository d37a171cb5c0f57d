"""The SOURCE of gtn_b200/csrc/k_compose.cu (frame-synchronous device composition with a
gtn::linearGraph operand: alive sets, counts, scans, CSR emission, and compose's gradFunc) run on the CPU
through the SIMT emulator of tests/emu against the oracle's compose (which is pinned to the reference's,
tests/test_oracle.py).

The device numbers the lattice frame-major; the reference numbers it in BFS discovery order and leaves
that unspecified (test/functions_test.cpp:137-227 check isomorphism only).  So the comparison is by
provenance: every composed arc is identified by gradInfo = (arc of the graph operand, arc of the
emissions chain) (compose.cpp:445), which is unique; the two lattices must hold the same set of
(provenance, weight) with bit-identical weights, the same node count, and the device lattice must be
consistent with its own CSR (an arc's end points sit in consecutive frames and correspond to the graph
arc's end points)."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import emu_build, util

f32p, i32p, u8p, u32p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint8), C.POINTER(C.c_uint32)


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("compose", ["k_compose.cu", "k_shortest.cu", "k_order.cu", "k_staged.cu"]))
    lib.emu_compose.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, i32p, u8p, i32p, i32p, i32p, i32p, f32p, i32p, i32p,
                                i32p, i32p, u32p, i32p, f32p, i32p, i32p, i32p, i32p, i32p, f32p, f32p, f32p]
    return lib


def tables_of(og, Cn):
    """What gtnb_compose_linear uploads for a graph operand: CSR by destination, in-arcs of a node
    ordered by (source, arc id), matched label = ilabel or -1 when it cannot match an emission."""
    a = og.arrays()
    N = len(a["flags"])
    ptr, src, lab, arc, w = [0], [], [], [], []
    for d in range(N):
        ins = sorted(np.nonzero(a["dst"] == d)[0].tolist(), key=lambda k: (int(a["src"][k]), k))
        for k in ins:
            l = int(a["ilabel"][k])
            src.append(int(a["src"][k])), lab.append(l if 0 <= l < Cn else -1), arc.append(k), w.append(float(a["w"][k]))
        ptr.append(len(src))
    return dict(flags=a["flags"].astype(np.uint8), ptr=np.array(ptr, np.int32), src=np.array(src, np.int32),
                lab=np.array(lab, np.int32), arc=np.array(arc, np.int32), w=np.array(w, np.float32),
                acc=a["accept"].astype(np.int32), g_src=a["src"], g_dst=a["dst"])


def cat(xs, dt):
    xs = [np.asarray(x, dt) for x in xs]
    return np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0, dt), dt)


def run(lib, e, lens, tabs, arc_grads=None):
    B, T, Cn = e.shape
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    nn = np.array([len(t["flags"]) for t in tabs], np.int32)
    capN = [int((lens[b] + 1) * nn[b] + 1) for b in range(B)]
    capA = [max(int(lens[b]) * len(tabs[b]["src"]), 1) for b in range(B)]
    outN, outA, nacc_out = np.zeros(B, np.int32), np.zeros(B, np.int32), np.zeros(B, np.int32)
    row_ptr = np.zeros(sum(capN), np.uint32)
    arc_src, gi_g, gi_e = (np.zeros(sum(capA), np.int32) for _ in range(3))
    arc_w = np.zeros(sum(capA), np.float32)
    lvl = np.zeros(int(sum(lens + 2)), np.int32)
    acc_out = np.zeros(max(sum(len(t["acc"]) for t in tabs), 1), np.int32)
    n_acc = np.array([len(t["acc"]) for t in tabs], np.int32)
    gg = np.zeros(max(sum(len(t["src"]) for t in tabs), 1), np.float32)
    ge = np.zeros((B, T, Cn), np.float32)
    ag = None
    if arc_grads is not None:
        ag = np.zeros(sum(capA), np.float32)
        off = 0
        for b in range(B):
            ag[off:off + len(arc_grads[b])] = arc_grads[b]
            off += capA[b]
    P = lambda a, t: a.ctypes.data_as(t)
    flags, ptr = cat([t["flags"] for t in tabs], np.uint8), cat([t["ptr"] for t in tabs], np.int32)
    src, lab = cat([t["src"] for t in tabs], np.int32), cat([t["lab"] for t in tabs], np.int32)
    arc, w, acc = cat([t["arc"] for t in tabs], np.int32), cat([t["w"] for t in tabs], np.float32), cat([t["acc"] for t in tabs], np.int32)
    rc = lib.emu_compose(B, T, Cn, P(e, f32p), P(lens, i32p), P(nn, i32p), P(flags, u8p), P(ptr, i32p), P(src, i32p),
                         P(lab, i32p), P(arc, i32p), P(w, f32p), P(n_acc, i32p), P(acc, i32p), P(outN, i32p), P(outA, i32p),
                         P(row_ptr, u32p), P(arc_src, i32p), P(arc_w, f32p), P(gi_g, i32p), P(gi_e, i32p), P(lvl, i32p),
                         P(acc_out, i32p), P(nacc_out, i32p), None if ag is None else P(ag, f32p), P(gg, f32p), P(ge, f32p))
    emu_build.check(rc)
    res, no, ao, lo, co, go = [], 0, 0, 0, 0, 0
    for b in range(B):
        N, A = int(outN[b]), int(outA[b])
        res.append(dict(N=N, A=A, row_ptr=row_ptr[no:no + N + 1].copy(), src=arc_src[ao:ao + A].copy(),
                        w=arc_w[ao:ao + A].copy(), gi_g=gi_g[ao:ao + A].copy(), gi_e=gi_e[ao:ao + A].copy(),
                        lvl=lvl[lo:lo + int(lens[b]) + 2].copy(), acc=acc_out[co:co + int(nacc_out[b])].copy(),
                        grad_graph=gg[go:go + len(tabs[b]["src"])].copy(), grad_emis=ge[b].copy()))
        no, ao, lo, co, go = no + capN[b], ao + capA[b], lo + int(lens[b]) + 2, co + len(tabs[b]["acc"]), go + len(tabs[b]["src"])
    return res


def check_lattice(r, tab, og, e_b, Tb, Cn):
    lin = po.Graph.linear(Tb, Cn, e_b[:Tb])
    want = po.compose(og, lin)
    g1, g2 = want.gradinfo()
    wa = want.arrays()
    assert r["N"] == len(wa["flags"]) and r["A"] == len(wa["src"]), (r["N"], len(wa["flags"]), r["A"], len(wa["src"]))
    # same arcs by provenance, bit-identical weights (compose.cpp:435: first.weight + second.weight)
    mine = sorted(zip(r["gi_g"].tolist(), r["gi_e"].tolist(), r["w"].view(np.int32).tolist()))
    ref = sorted(zip(g1.tolist(), g2.tolist(), wa["w"].view(np.int32).tolist()))
    assert mine == ref
    # CSR consistency: level = frame, node identity = (graph node, frame)
    rp = (r["row_ptr"] & 0x3FFFFFFF).astype(np.int64)
    assert rp[0] == 0 and rp[r["N"]] == r["A"] and (np.diff(rp) >= 0).all()
    lvl = r["lvl"]
    assert lvl[0] == 0 and lvl[Tb + 1] == r["N"]
    level_of = np.searchsorted(lvl[1:], np.arange(r["N"]), side="right")
    ident = {}
    for n in range(r["N"]):
        for a in range(rp[n], rp[n + 1]):
            i, j = int(r["gi_g"][a]), int(r["gi_e"][a])
            t = j // Cn + 1
            assert level_of[n] == t and level_of[r["src"][a]] == t - 1
            assert ident.setdefault(n, int(tab["g_dst"][i])) == int(tab["g_dst"][i])
            assert ident.setdefault(int(r["src"][a]), int(tab["g_src"][i])) == int(tab["g_src"][i])
    # start / accept bits
    starts = [n for n in range(r["N"]) if r["row_ptr"][n] & 0x40000000]
    assert all(level_of[n] == 0 for n in starts) and len(starts) == int((wa["flags"] & 1).sum())
    accepts = sorted(n for n in range(r["N"]) if r["row_ptr"][n] & 0x80000000)
    assert accepts == sorted(r["acc"].tolist()) and len(accepts) == int(((wa["flags"] & 2) > 0).sum())
    assert all(level_of[n] == Tb for n in accepts)
    return want


@pytest.mark.parametrize("shape", [(3, 14, 6, 3), (2, 9, 5, 4), (2, 40, 8, 12), (1, 3, 4, 0), (1, 25, 40, 9)])
def test_compose_kernels_ctc_lattices(emu, shape):
    """CTC target graphs x emissions; ragged T (the cone at both ends and the all-alive steady state of
    compose_count / compose_emit both occur), T == 2U+1, an empty transcript."""
    B, T, Cn, U = shape
    e, targets = util.bench_inputs(B, T, Cn, max(U, 1), seed=31)
    if U == 0:
        targets = [t[:0] for t in targets]
    lens = np.minimum(np.array([max(T - 4 * b, 2 * U + 1) for b in range(B)], np.int32), T)
    ogs = [po.Graph.ctc(t, 0, True) for t in targets]
    tabs = [tables_of(g, Cn) for g in ogs]
    rng = np.random.default_rng(5)
    res = run(emu, e, lens, tabs)
    grads = [rng.integers(-3, 4, r["A"]).astype(np.float32) for r in res]
    res = run(emu, e, lens, tabs, arc_grads=grads)
    for b in range(B):
        check_lattice(res[b], tabs[b], ogs[b], e[b], int(lens[b]), Cn)
        # compose's gradFunc (compose.cpp:496-518): scatter-add by provenance
        gg = np.zeros(len(tabs[b]["src"]), np.float32)
        np.add.at(gg, res[b]["gi_g"], grads[b])
        ge = np.zeros(T * Cn, np.float32)
        np.add.at(ge, res[b]["gi_e"], grads[b])
        assert np.array_equal(res[b]["grad_graph"], gg)
        assert np.array_equal(res[b]["grad_emis"].reshape(-1), ge)


@pytest.mark.parametrize("seed", range(6))
def test_compose_kernels_general_graph_operand(emu, seed):
    """Any epsilon-free graph operand: cycles, several start / accept nodes, dead ends, mixed labels per
    node, labels that no emission carries (they can never match, compose.cpp:211-374)."""
    rng = np.random.default_rng(900 + seed)
    Cn, T, B = 5, int(rng.integers(1, 9)), 2
    ogs, tabs = [], []
    for _ in range(B):
        n = int(rng.integers(1, 40 if seed == 5 else 9))
        flags = np.zeros(n, np.uint8)
        flags[rng.integers(0, n, max(1, n // 3))] |= 1
        flags[rng.integers(0, n, max(1, n // 3))] |= 2
        na = int(rng.integers(0, 3 * n + 1))
        src, dst = rng.integers(0, n, na), rng.integers(0, n, na)
        lab = rng.integers(0, Cn + 2, na)  # Cn, Cn+1: no such emission
        w = rng.integers(-3, 4, na).astype(np.float32)
        og = po.Graph.from_arrays(flags, src, dst, lab, lab, w)
        ogs.append(og)
        tabs.append(tables_of(og, Cn))
    e = rng.integers(-4, 5, (B, T, Cn)).astype(np.float32)
    lens = np.array([T, max(T - 1, 0)], np.int32)
    res = run(emu, e, lens, tabs)
    for b in range(B):
        check_lattice(res[b], tabs[b], ogs[b], e[b], int(lens[b]), Cn)


def run_materialised(lib, e, lens, tabs, deltas, viterbi=False):
    B, T, Cn = e.shape
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    deltas = np.ascontiguousarray(deltas, np.float32)
    nn = np.array([len(t["flags"]) for t in tabs], np.int32)
    n_acc = np.array([len(t["acc"]) for t in tabs], np.int32)
    out = np.zeros(B, np.float32)
    gg = np.zeros(max(sum(len(t["src"]) for t in tabs), 1), np.float32)
    ge = np.zeros((B, T, Cn), np.float32)
    vs = np.zeros(B, np.float32)
    vl = np.full((B, max(T, 1)), -9, np.int32)
    P = lambda a, t: a.ctypes.data_as(t)
    flags, ptr = cat([t["flags"] for t in tabs], np.uint8), cat([t["ptr"] for t in tabs], np.int32)
    src, lab = cat([t["src"] for t in tabs], np.int32), cat([t["lab"] for t in tabs], np.int32)
    arc, w, acc = cat([t["arc"] for t in tabs], np.int32), cat([t["w"] for t in tabs], np.float32), cat([t["acc"] for t in tabs], np.int32)
    lib.emu_materialised.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, i32p, u8p, i32p, i32p, i32p, i32p, f32p, i32p,
                                     i32p, f32p, f32p, f32p, f32p, C.c_int, f32p, i32p]
    rc = lib.emu_materialised(B, T, Cn, P(e, f32p), P(lens, i32p), P(nn, i32p), P(flags, u8p), P(ptr, i32p), P(src, i32p),
                              P(lab, i32p), P(arc, i32p), P(w, f32p), P(n_acc, i32p), P(acc, i32p), P(deltas, f32p),
                              P(out, f32p), P(gg, f32p), P(ge, f32p), int(viterbi), P(vs, f32p), P(vl, i32p))
    emu_build.check(rc)
    return out, gg, ge, vs, vl


@pytest.mark.parametrize("shape", [(3, 14, 6, 3), (2, 9, 5, 4), (2, 40, 8, 12), (1, 25, 40, 9)])
def test_materialised_ctc_path_end_to_end(emu, oracle, shape):
    """compose -> sd_forward_generic -> sd_backward_generic -> compose gradFunc (k_compose.cu + k_shortest.cu):
    the CSR formulation of the north star, as gtnb_ctc_loss runs it with the implicit and staged flags off."""
    B, T, Cn, U = shape
    e, targets = util.bench_inputs(B, T, Cn, U, seed=77)
    lens = np.minimum(np.array([max(T - 4 * b, 2 * U + 1) for b in range(B)], np.int32), T)
    ogs = [po.Graph.ctc(t, 0, True) for t in targets]
    tabs = [tables_of(g, Cn) for g in ogs]
    out, gg, ge, _, _ = run_materialised(emu, e, lens, tabs, -np.ones(B, np.float32))
    for b in range(B):
        Tb = int(lens[b])
        lo, go = oracle.ctc_loss(e[b, :Tb], targets[b], 0, True)
        x = e[b, :Tb].astype(np.float64)
        mx = x.max(1, keepdims=True)
        lse = mx[:, 0] + np.log(np.exp(x - mx).sum(1))
        assert util.close(float(lse.sum() - np.float64(out[b])), lo), (b, out[b], lo)
        g = np.exp(x - lse[:, None]) + ge[b, :Tb]
        assert util.grad_close(g, go, 5.0 * T), (b, float(np.abs(g - go).max()))
        assert not ge[b, Tb:].any()
    # the graph-side gradient (compose.cpp:500-506): minus the expected count of each target-graph arc; the
    # arcs into one graph node are used once per frame the node is occupied, so per utterance they sum to -T
    off = 0
    for b in range(B):
        A = len(tabs[b]["src"])
        assert np.isclose(gg[off:off + A].sum(), -float(lens[b]), rtol=1e-4)
        off += A


@pytest.mark.parametrize("ties", [False, True])
def test_materialised_viterbi_path(emu, oracle, ties):
    """viterbiPath(intersect(ctc, emissions)): MODE_PATH forward + traceback + label provenance; the score
    bit for bit, the path with == when nothing ties exactly."""
    B, T, Cn, U = 3, 18, 6, 4
    rng = np.random.default_rng(21 + ties)
    e = (rng.integers(-2, 3, (B, T, Cn)) if ties else rng.uniform(-5, 5, (B, T, Cn))).astype(np.float32)
    targets = [rng.integers(1, Cn, U).astype(np.int32) for _ in range(B)]
    lens = np.array([T, T - 3, T - 7], np.int32)
    ogs = [po.Graph.ctc(t, 0, True) for t in targets]
    tabs = [tables_of(g, Cn) for g in ogs]
    _, _, _, vs, vl = run_materialised(emu, e, lens, tabs, np.ones(B, np.float32), viterbi=True)
    for b in range(B):
        Tb = int(lens[b])
        want_path, want_score = oracle.viterbi_ctc(e[b, :Tb], targets[b], 0, True)
        assert vs[b] == np.float32(want_score)
        got = vl[b, :Tb]
        if not ties:
            assert np.array_equal(got, want_path), (b, got, want_path)
            continue
        # exact ties: the reference keeps the first-RELAXED predecessor, which follows compose's BFS
        # numbering of the product states; the device lattice is numbered frame-major, so an equally
        # optimal alignment may come back (DESIGN.md section 4).  It must be one: a valid CTC
        # alignment of the target with the same total score.
        collapsed = [int(l) for k, l in enumerate(got) if l != 0 and (k == 0 or l != got[k - 1])]
        assert collapsed == targets[b].tolist(), (b, got, targets[b])
        assert np.float32(sum(float(e[b, t, got[t]]) for t in range(Tb))) == np.float32(want_score)


def tables_with_out_pos(og, Cn):
    """tables_of + the two tables the exact-ties option uploads: per in-entry the position of the arc in its
    source's out-arc list (the reference's per-node order, after any arcSort), per node its index in g.start()."""
    a = og.arrays()
    ip, ia, op, oa = og.adjacency()
    N = len(a["flags"])
    out_pos = np.zeros(len(a["src"]), np.int32)
    for n in range(N):
        for k in range(op[n], op[n + 1]):
            out_pos[oa[k]] = k - op[n]
    t = tables_of(og, Cn)
    # in-arcs of a node ordered by (source, position in the source's out list), as gtnb_compose_linear does
    ptr, src, lab, arc, w, opos = [0], [], [], [], [], []
    for d in range(N):
        ins = sorted(np.nonzero(a["dst"] == d)[0].tolist(), key=lambda k: (int(a["src"][k]), int(out_pos[k])))
        for k in ins:
            l = int(a["ilabel"][k])
            src.append(int(a["src"][k])), lab.append(l if 0 <= l < Cn else -1), arc.append(k)
            w.append(float(a["w"][k])), opos.append(int(out_pos[k]))
        ptr.append(len(src))
    t.update(ptr=np.array(ptr, np.int32), src=np.array(src, np.int32), lab=np.array(lab, np.int32),
             arc=np.array(arc, np.int32), w=np.array(w, np.float32), out_pos=np.array(opos, np.int32))
    sr = np.full(N, -1, np.int32)
    for k, s in enumerate(a["start"]):
        sr[s] = k
    t["start_rank"] = sr
    t["max_out"] = int(max([op[n + 1] - op[n] for n in range(N)] + [0]))
    return t


def run_exact(lib, e, lens, tabs, staged=False):
    B, T, Cn = e.shape
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    nn = np.array([len(t["flags"]) for t in tabs], np.int32)
    n_acc = np.array([len(t["acc"]) for t in tabs], np.int32)
    vs = np.zeros(B, np.float32)
    vl = np.full((B, max(T, 1)), -9, np.int32)
    vg = np.full((B, max(T, 1)), -9, np.int32)
    P = lambda a, t: a.ctypes.data_as(t)
    flags, ptr = cat([t["flags"] for t in tabs], np.uint8), cat([t["ptr"] for t in tabs], np.int32)
    src, lab = cat([t["src"] for t in tabs], np.int32), cat([t["lab"] for t in tabs], np.int32)
    arc, w, acc = cat([t["arc"] for t in tabs], np.int32), cat([t["w"] for t in tabs], np.float32), cat([t["acc"] for t in tabs], np.int32)
    opos, sr = cat([t["out_pos"] for t in tabs], np.int32), cat([t["start_rank"] for t in tabs], np.int32)
    lib.emu_viterbi_exact.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, i32p, u8p, i32p, i32p, i32p, i32p, f32p, i32p,
                                      i32p, C.c_int, i32p, i32p, C.c_int, f32p, i32p, i32p]
    rc = lib.emu_viterbi_exact(B, T, Cn, P(e, f32p), P(lens, i32p), P(nn, i32p), P(flags, u8p), P(ptr, i32p), P(src, i32p),
                               P(lab, i32p), P(arc, i32p), P(w, f32p), P(opos, i32p), P(sr, i32p),
                               max(t["max_out"] for t in tabs), P(n_acc, i32p), P(acc, i32p), int(staged), P(vs, f32p),
                               P(vl, i32p), P(vg, i32p))
    emu_build.check(rc)
    return vs, vl, vg


def reference_path(og, e_b, Tb, Cn):
    """The oracle's shortestPath (pinned to the reference's, ties included: tests/test_oracle.py) on its own
    compose: (graph arc ids, emission labels) along the path, and the score."""
    lin = po.Graph.linear(Tb, Cn, e_b[:Tb])
    comp = po.compose(og, lin)
    arcs = po.shortest_path(comp)
    if arcs is None:
        return None, None, None
    g1, g2 = comp.gradinfo()
    w = comp.arrays()["w"]
    score = np.float32(0.0)
    for k in arcs:
        score = np.float32(score + w[k])
    return [int(g1[k]) for k in arcs], [int(g2[k]) % Cn for k in arcs], score


@pytest.mark.parametrize("staged", [False, True])
@pytest.mark.parametrize("blank_last", [False, True])
def test_exact_ties_option_reproduces_the_reference_path_on_ctc_lattices(emu, blank_last, staged):
    """k_order.cu: with every lattice row sorted by the reference's relaxation rank and the accept list in
    creation order, viterbiPath through the device lattice -- generic or TMA-staged path kernel -- returns the
    reference's path on integer-valued emissions (ties at nearly every node), for blank first and blank last
    (where compose's discovery order is not the node order)."""
    B, T, Cn, U = 4, 16, 5, 3
    rng = np.random.default_rng(11 + blank_last)
    e = rng.integers(-1, 2, (B, T, Cn)).astype(np.float32)
    blank = Cn - 1 if blank_last else 0
    labels = [l for l in range(Cn) if l != blank]
    targets = [rng.choice(labels, U).astype(np.int32) for _ in range(B)]
    targets[1][1] = targets[1][0]
    lens = np.array([T, T - 2, T - 5, 2 * U + 1], np.int32)
    ogs = [po.Graph.ctc(t, blank, True) for t in targets]
    tabs = [tables_with_out_pos(g, Cn) for g in ogs]
    vs, vl, vg = run_exact(emu, e, lens, tabs, staged)
    for b in range(B):
        Tb = int(lens[b])
        want_arcs, want_labels, want_score = reference_path(ogs[b], e[b], Tb, Cn)
        assert vg[b, :Tb].tolist() == want_arcs, (b, vg[b, :Tb], want_arcs)
        assert vl[b, :Tb].tolist() == want_labels
        assert vs[b] == want_score


@pytest.mark.parametrize("seed", range(8))
def test_exact_ties_option_on_general_graph_operands(emu, seed):
    """Any epsilon-free graph operand, sorted or not (unsorted / singly / doubly sorted matchers), integer
    weights: same path, arc for arc, as the reference."""
    rng = np.random.default_rng(4000 + seed)
    Cn, T, B = 4, int(rng.integers(2, 8)), 2
    ogs, tabs = [], []
    for _ in range(B):
        n = int(rng.integers(2, 8))
        flags = np.zeros(n, np.uint8)
        flags[rng.integers(0, n, max(1, n // 3))] |= 1
        flags[rng.integers(0, n, max(1, n // 2))] |= 2
        na = int(rng.integers(n, 3 * n + 1))
        src, dst = rng.integers(0, n, na), rng.integers(0, n, na)
        lab = rng.integers(0, Cn, na)
        w = rng.integers(-1, 2, na).astype(np.float32)
        og = po.Graph.from_arrays(flags, src, dst, lab, lab, w)
        if seed % 2:
            og.arc_sort(False)
        ogs.append(og)
        tabs.append(tables_with_out_pos(og, Cn))
    e = rng.integers(-1, 2, (B, T, Cn)).astype(np.float32)
    lens = np.array([T, T - 1], np.int32)
    vs, vl, vg = run_exact(emu, e, lens, tabs)
    for b in range(B):
        Tb = int(lens[b])
        want_arcs, want_labels, want_score = reference_path(ogs[b], e[b], Tb, Cn)
        if want_arcs is None:
            assert not np.isfinite(vs[b]) or (vg[b, :Tb] < 0).all()
            continue
        assert vg[b, :Tb].tolist() == want_arcs, (b, vg[b, :Tb], want_arcs)
        assert vs[b] == want_score


def run_sort_with_grads(lib, e, lens, tabs, grad_in):
    """The exact-ties row sort on a lattice whose arc_grad holds grad_in (compose order, graph after graph) ->
    (arc counts, grad_out, provenance before, provenance after), the last three in that layout"""
    B, T, Cn = e.shape
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    grad_in = np.ascontiguousarray(grad_in, np.float32)
    nn = np.array([len(t["flags"]) for t in tabs], np.int32)
    n_acc = np.array([len(t["acc"]) for t in tabs], np.int32)
    n_arcs = np.zeros(B, np.int32)
    grad_out = np.full(len(grad_in), np.nan, np.float32)
    gi_in, gi_out = np.zeros((len(grad_in), 2), np.int32), np.zeros((len(grad_in), 2), np.int32)
    P = lambda a, t: a.ctypes.data_as(t)
    flags, ptr = cat([t["flags"] for t in tabs], np.uint8), cat([t["ptr"] for t in tabs], np.int32)
    src, lab = cat([t["src"] for t in tabs], np.int32), cat([t["lab"] for t in tabs], np.int32)
    arc, w, acc = cat([t["arc"] for t in tabs], np.int32), cat([t["w"] for t in tabs], np.float32), cat([t["acc"] for t in tabs], np.int32)
    opos, sr = cat([t["out_pos"] for t in tabs], np.int32), cat([t["start_rank"] for t in tabs], np.int32)
    lib.emu_sort_rows_with_grads.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, i32p, u8p, i32p, i32p, i32p, i32p,
                                             f32p, i32p, i32p, C.c_int, i32p, i32p, f32p, f32p, i32p, i32p, i32p]
    rc = lib.emu_sort_rows_with_grads(B, T, Cn, P(e, f32p), P(lens, i32p), P(nn, i32p), P(flags, u8p), P(ptr, i32p),
                                      P(src, i32p), P(lab, i32p), P(arc, i32p), P(w, f32p), P(opos, i32p), P(sr, i32p),
                                      max(t["max_out"] for t in tabs), P(n_acc, i32p), P(acc, i32p), P(grad_in, f32p),
                                      P(grad_out, f32p), P(gi_in, i32p), P(gi_out, i32p), P(n_arcs, i32p))
    emu_build.check(rc)
    A = int(n_arcs.sum())
    return n_arcs, grad_out[:A], gi_in[:A], gi_out[:A]


def sort_operands(kind, seed):
    """tie-heavy emissions and the exact-ties tables of CTC graphs (blank first / last, a repeated label) or of
    general graph operands, sorted or not"""
    rng = np.random.default_rng(6000 + seed)
    if kind == "general":
        Cn, T = 4, int(rng.integers(2, 8))
        ogs = []
        for i in range(3):
            n = int(rng.integers(2, 8))
            flags = np.zeros(n, np.uint8)
            flags[rng.integers(0, n, max(1, n // 3))] |= 1
            flags[rng.integers(0, n, max(1, n // 2))] |= 2
            na = int(rng.integers(n, 3 * n + 1))
            src, dst, lab = rng.integers(0, n, na), rng.integers(0, n, na), rng.integers(0, Cn, na)
            og = po.Graph.from_arrays(flags, src, dst, lab, lab, rng.integers(-1, 2, na).astype(np.float32))
            if i % 2:
                og.arc_sort(False)
            ogs.append(og)
        lens = [T, T - 1, 1]
    else:
        Cn, T, U = 5, 16, 3
        blank = Cn - 1 if kind == "ctc_blank_last" else 0
        labels = [l for l in range(Cn) if l != blank]
        targets = [rng.choice(labels, U).astype(np.int32) for _ in range(3)]
        targets[1][1] = targets[1][0]
        ogs = [po.Graph.ctc(t, blank, True) for t in targets]
        lens = [T, T - 5, 2 * U + 1]
    e = rng.integers(-1, 2, (len(ogs), T, Cn)).astype(np.float32)
    return rng, e, np.array(lens, np.int32), [tables_with_out_pos(g, Cn) for g in ogs]


@pytest.mark.parametrize("kind,seed", [("ctc_blank_first", 0), ("ctc_blank_last", 1), ("general", 2), ("general", 3),
                                       ("general", 4), ("general", 5)])
def test_exact_ties_sort_carries_arc_grads(emu, kind, seed):
    """gtnb_backward may run before the exact-ties sort: lattice_sort_rows_kernel then moves arc_grad with the arcs.
    Looked up by entry and provenance (which names an arc of a composed lattice), every arc's gradient is the one it
    had before the sort.  On the CTC lattices the sort does move arcs, so a gradient left in place is caught."""
    rng, e, lens, tabs = sort_operands(kind, seed)
    cap = max(sum(int(lens[b]) * len(tabs[b]["src"]) for b in range(len(tabs))), 1)  # >= every lattice's arc count
    grad_in = rng.integers(-50, 51, cap).astype(np.float32) / 8
    n_arcs, grad_out, gi_in, gi_out = run_sort_with_grads(emu, e, lens, tabs, grad_in)
    entry = np.repeat(np.arange(len(tabs)), n_arcs).tolist()
    before = [(b, *g) for b, g in zip(entry, gi_in.tolist())]
    after = [(b, *g) for b, g in zip(entry, gi_out.tolist())]
    assert len(set(before)) == len(before) and sorted(after) == sorted(before)
    was = dict(zip(before, grad_in[:len(before)].tolist()))
    assert [was[k] for k in after] == grad_out.tolist()
    if kind != "general":
        assert before != after


def run_staged(lib, e, lens, tabs, deltas, fused, viterbi=False):
    B, T, Cn = e.shape
    e = np.ascontiguousarray(e, np.float32)
    lens = np.ascontiguousarray(lens, np.int32)
    deltas = np.ascontiguousarray(deltas, np.float32)
    nn = np.array([len(t["flags"]) for t in tabs], np.int32)
    n_acc = np.array([len(t["acc"]) for t in tabs], np.int32)
    out = np.zeros(B, np.float32)
    ge = np.zeros((B, T, Cn), np.float32)
    vs = np.zeros(B, np.float32)
    vl = np.full((B, max(T, 1)), -9, np.int32)
    P = lambda a, t: a.ctypes.data_as(t)
    flags, ptr = cat([t["flags"] for t in tabs], np.uint8), cat([t["ptr"] for t in tabs], np.int32)
    src, lab = cat([t["src"] for t in tabs], np.int32), cat([t["lab"] for t in tabs], np.int32)
    arc, w, acc = cat([t["arc"] for t in tabs], np.int32), cat([t["w"] for t in tabs], np.float32), cat([t["acc"] for t in tabs], np.int32)
    lib.emu_materialised_staged.argtypes = [C.c_int, C.c_int, C.c_int, f32p, i32p, i32p, u8p, i32p, i32p, i32p, i32p, f32p,
                                            i32p, i32p, f32p, C.c_int, f32p, f32p, C.c_int, f32p, i32p]
    rc = lib.emu_materialised_staged(B, T, Cn, P(e, f32p), P(lens, i32p), P(nn, i32p), P(flags, u8p), P(ptr, i32p),
                                     P(src, i32p), P(lab, i32p), P(arc, i32p), P(w, f32p), P(n_acc, i32p), P(acc, i32p),
                                     P(deltas, f32p), int(fused), P(out, f32p), P(ge, f32p), int(viterbi), P(vs, f32p),
                                     P(vl, i32p))
    emu_build.check(rc)
    return out, ge, vs, vl


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("shape", [(3, 14, 6, 3), (2, 9, 5, 4), (2, 40, 8, 12), (1, 25, 40, 9), (1, 70, 16, 30)])
def test_tma_staged_kernels_end_to_end(emu, oracle, shape, fused):
    """k_staged.cu -- the warp-specialised persistent kernels of the materialised path (producer warp:
    cp.async.bulk + mbarrier ring; eight consumer warps) -- with the bulk copies and mbarriers emulated:
    sd_forward_staged, then sd_backward_staged + compose's gradFunc, or the fused criterion backward."""
    B, T, Cn, U = shape
    e, targets = util.bench_inputs(B, T, Cn, U, seed=123)
    lens = np.minimum(np.array([max(T - 4 * b, 2 * U + 1) for b in range(B)], np.int32), T)
    ogs = [po.Graph.ctc(t, 0, True) for t in targets]
    tabs = [tables_of(g, Cn) for g in ogs]
    out, ge, _, _ = run_staged(emu, e, lens, tabs, -np.ones(B, np.float32), fused)
    for b in range(B):
        Tb = int(lens[b])
        lo, go = oracle.ctc_loss(e[b, :Tb], targets[b], 0, True)
        x = e[b, :Tb].astype(np.float64)
        mx = x.max(1, keepdims=True)
        lse = mx[:, 0] + np.log(np.exp(x - mx).sum(1))
        assert util.close(float(lse.sum() - np.float64(out[b])), lo), (b, out[b], lo)
        g = np.exp(x - lse[:, None]) + ge[b, :Tb]
        assert util.grad_close(g, go, 5.0 * T), (b, float(np.abs(g - go).max()))
        assert not ge[b, Tb:].any()


def test_tma_staged_viterbi_path(emu, oracle):
    B, T, Cn, U = 3, 18, 6, 4
    rng = np.random.default_rng(8)
    e = rng.uniform(-5, 5, (B, T, Cn)).astype(np.float32)
    targets = [rng.integers(1, Cn, U).astype(np.int32) for _ in range(B)]
    lens = np.array([T, T - 3, T - 7], np.int32)
    tabs = [tables_of(po.Graph.ctc(t, 0, True), Cn) for t in targets]
    _, _, vs, vl = run_staged(emu, e, lens, tabs, np.ones(B, np.float32), False, viterbi=True)
    for b in range(B):
        Tb = int(lens[b])
        want_path, want_score = oracle.viterbi_ctc(e[b, :Tb], targets[b], 0, True)
        assert np.array_equal(vl[b, :Tb], want_path) and vs[b] == np.float32(want_score)
