"""The launch plans' outcomes against the case table of tests/test_gpu_instantiations.py, on the CPU.

(a) walks each plan's input domain through tests/emu/plan_emu.cpp (the plans' own code, unchanged) and collects the
    distinct outcomes, each naming an entry of the driver's instantiation table, and the boundaries between them;
(b) maps every case of tests/instantiation_cases.py to its outcome through the same exports;
(c) asserts that every reachable outcome is covered, that every boundary has a case on each side, and that every
    compiled instantiation is reached by a case or listed below with the reason it is not.

A new instantiation or a moved threshold makes this file fail until a case covers it."""
import ctypes as C
from collections import defaultdict

import numpy as np
import pytest

from tests import emu_build
from tests import instantiation_cases as ic

i32p = C.POINTER(C.c_int32)
KERNELS = ["k_dense.cu", "k_implicit.cu", "k_ngram.cu", "k_bidir.cu", "k_staged.cu"]
HALF = (ic.BF16, ic.F16)

# Instantiations no input can reach, by (family table, index) -> reason.  Indices follow plan_emu.cpp's tables.
# bidir: float rows 0-5, bf16 6-11, fp16 12-17; (NQ, FX, PAIR) = (1,0,0) (2,0,0) (1,1,0) (2,1,0) (1,1,1) (2,1,1)
# implicit forward: float (ARC, TROP) = (0,0) 0-6, (0,1) 7-13, (1,0) 14-20, (1,1) 21-27 over G = 0,1,2,4,8,16,32;
#   bf16 28, fp16 29.  implicit backward: float (ARC, GG) = (0,0) 0-6, (0,1) 7-13, (1,0) 14-20, (1,1) 21-27;
#   bf16 (GG 0, 1) 28-29, fp16 30-31.
NO_GG_HALF = "a 16-bit lattice exists only for the trellis criteria's numerators (gtnb_criteria.cu sets lat->dtype " \
             "there alone), whose backward always accumulates the graph gradient; every other caller widens first"
UNREACHED = {("implicit_bwd", 28): NO_GG_HALF, ("implicit_bwd", 30): NO_GG_HALF}


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build("plan", KERNELS))
    lib.emu_bidir_plan.argtypes = [C.c_int] * 7 + [i32p]
    lib.emu_dense_plan.argtypes = [C.c_int] * 3 + [i32p]
    lib.emu_ngram_plan.argtypes = [C.c_int] * 3 + [i32p]
    lib.emu_implicit_plan.argtypes = [C.c_int] * 8 + [i32p]
    lib.emu_staged_plan.argtypes = [C.c_int, i32p, i32p, i32p, C.c_int, C.c_int, i32p]
    return lib


def bidir(emu, C_, max_nodes, pair_ok, esize, max_in=3, max_out=3, fixed_pitch=None):
    o = np.zeros(8, np.int32)
    fp = int(max_nodes <= 224) if fixed_pitch is None else fixed_pitch
    emu.emu_bidir_plan(C_, max_nodes, max_in, max_out, fp, pair_ok, esize, o.ctypes.data_as(i32p))
    return int(o[7]) if o[0] else None  # None: bidir_shape_supported refuses


def dense(emu, C_, bigram, esize):
    o = np.zeros(4, np.int32)
    emu.emu_dense_plan(C_, bigram, esize, o.ctypes.data_as(i32p))
    return int(o[3]) if o[0] else None


def ngram(emu, C_, start, esize):
    if C_ > 128:  # kNgramMaxC: wider alphabets do not take the trellis kernels
        return None
    o = np.zeros(5, np.int32)
    emu.emu_ngram_plan(C_, start, esize, o.ctypes.data_as(i32p))
    return (int(o[3]), int(o[4]))


def implicit(emu, max_in, max_out, max_nodes, C_, arc, trop, gg, dtype):
    o = np.zeros(6, np.int32)
    emu.emu_implicit_plan(max_in, max_out, max_nodes, C_, arc, trop, gg, dtype, o.ctypes.data_as(i32p))
    return tuple(int(x) for x in o)


def staged(emu, L, sg_A, sg_N, max_lvl_nodes, max_lvl_arcs):
    o = np.zeros(10, np.int32)
    a = [np.ascontiguousarray(x, np.int32) for x in (L, sg_A, sg_N)]
    emu.emu_staged_plan(len(L), *(x.ctypes.data_as(i32p) for x in a), max_lvl_nodes, max_lvl_arcs,
                        o.ctypes.data_as(i32p))
    return dict(ok=int(o[0]), G=int(o[1]), ls=int(o[3]), fused=int(o[6]), fwd=int(o[8]), bwd=int(o[9]))


def staged_key(p):
    return (p["fwd"], p["bwd"], p["ls"], p["fused"]) if p["ok"] else None


def ctc_sizes(U):
    """the staged plan's inputs for one CTC graph of U distinct consecutive labels in U + 8 frames (the cases' shape)"""
    N, A = ic.ctc_graph_size(list(range(1, U + 1)))
    return [U + 9], [A], [N], N, A


# ---- (a) the outcomes and their boundaries --------------------------------------------------------------------------


def walk(values, outcome):
    """outcome over an ordered axis -> ({outcome: (first, last)}, [(last value of one outcome, first of the next)])"""
    spans, bounds, prev = {}, [], (None, None)
    for v in values:
        o = outcome(v)
        lo, _ = spans.get(o, (v, v))
        spans[o] = (lo, v)
        if prev[0] is not None and o != prev[1]:
            bounds.append((prev[0], v))
        prev = (v, o)
    return spans, bounds


def ctc_nodes():
    return range(1, 2 * 200 + 2, 2)  # CTC graphs: 2U + 1 nodes


def bidir_domain(emu):
    """per (esize, pair_ok): outcomes over C (at 41 nodes), and over the node count for the PAIR kernels (C = 64), the FX
    kernels (C = 128, one node per thread asked for) and the others (C = 40)"""
    out = {}
    for esize in (4, 2, 3):
        for pair_ok in (0, 1):
            out[(esize, pair_ok, "C")] = walk(range(1, 257), lambda c: bidir(emu, c, 41, pair_ok, esize))
        for c, pair_ok in ((40, 1), (64, 1), (128, 0)):
            out[(esize, pair_ok, "nodes", c)] = walk(ctc_nodes(), lambda n: bidir(emu, c, n, pair_ok, esize))
    return out


def dense_domain(emu):
    return {(esize, bg): walk(range(1, 257), lambda c: dense(emu, c, bg, esize)) for esize in (4, 2, 3) for bg in (0, 1)}


def ngram_domain(emu):
    """over the trellis kernels' alphabets (n-gram CTC needs a label besides the blank)"""
    return {(esize, st): walk(range(1 + (1 - st), 129), lambda c: ngram(emu, c, st, esize))
            for esize in (4, 2, 3) for st in (0, 1)}


def implicit_domain(emu):
    """wide_lanes over the in-degree (out-degree 3, 8 nodes) and over the node count (in-degree 21), forward and
    backward, label-uniform and not: the G each input takes"""
    out = {}
    for arc in (0, 1):
        out[(arc, "deg")] = walk(range(1, 700), lambda d: implicit(emu, d, 3, 8, 6, arc, 0, 0, ic.F32)[:2])
        out[(arc, "nodes")] = walk(range(2, 400), lambda n: implicit(emu, 21, 3, n, 6, arc, 0, 0, ic.F32)[:2])
    return out


def staged_domain(emu):
    deg = walk(range(16, 16 * 64), lambda a: staged(emu, [6], [a], [16], 16, a)["G"])
    size = walk(range(0, 1500), lambda u: staged_key(staged(emu, *ctc_sizes(u))))
    return deg, size


def test_domains_have_the_expected_shape(emu):
    """the outcome counts per family (a change here is a change of a plan: update the case table with it)"""
    b = bidir_domain(emu)
    bid = set()
    for spans, _ in b.values():
        bid |= {o for o in spans if o is not None}
    assert bid == set(range(18)), sorted(bid)
    d = set()
    for spans, _ in dense_domain(emu).values():
        d |= {o for o in spans if o is not None}
    assert d == set(range(36)), sorted(d)
    n = set()
    for spans, _ in ngram_domain(emu).values():
        n |= {o for o in spans if o is not None}
    assert len(n) == 12, sorted(n)
    deg, size = staged_domain(emu)
    assert set(deg[0]) == {1, 4, 16, 32}
    assert len(size[0]) == 5, size[0]  # ls = 3, 2, 1; fused refused; plan refused


def test_implicit_outcomes_are_instantiations(emu):
    """wide_lanes over in/out-degrees up to 700 and the flag combinations: every outcome names a table entry, and the
    16-bit element types take only G = 0 in the log semiring without arc labels"""
    seen_f, seen_b = set(), set()
    for dtype in (ic.F32, ic.BF16, ic.F16):
        for arc in (0, 1):
            for trop in (0, 1):
                for gg in (0, 1):
                    for deg in list(range(0, 64)) + list(range(64, 700, 7)) + [640, 641]:
                        Gf, Gb, okf, okb, f, b = implicit(emu, deg, 2, 64, 32, arc, trop, gg, dtype)
                        if okf == 0:
                            assert f >= 0, (dtype, arc, trop, deg, Gf)
                            seen_f.add(f)
                        else:
                            assert dtype != ic.F32 and (Gf or arc or trop)
                        if okb == 0:
                            assert b >= 0, (dtype, arc, gg, deg, Gb)
                            seen_b.add(b)
    assert seen_f == set(range(30)) and seen_b == set(range(32)), (sorted(seen_f), sorted(seen_b))


# ---- (b) the cases' outcomes ---------------------------------------------------------------------------------------


def case_outcome(emu, case):
    p = ic.plan_inputs(case)
    if case.family == "bidir":
        return bidir(emu, p["C"], p["max_nodes"], p["pair_ok"], p["esize"], p["max_in"], p["max_out"],
                     p["fixed_pitch"])
    if case.family == "dense":
        return dense(emu, p["C"], p["bigram"], p["esize"])
    if case.family == "ngram":
        return ngram(emu, p["C"], p["start"], p["esize"])
    if case.family == "implicit":
        return implicit(emu, p["max_in"], p["max_out"], p["max_nodes"], p["C"], p["arc"], p["trop"], p["gg"], ic.F32)
    return staged(emu, p["L"], p["sg_A"], p["sg_N"], p["max_lvl_nodes"], p["max_lvl_arcs"])


def reached(emu):
    """{(table, index)} the cases reach"""
    got = set()
    for case in ic.all_cases():
        o = case_outcome(emu, case)
        if o is None:
            continue
        if case.family == "bidir":
            got.add(("bidir", o))
        elif case.family == "dense":
            got.add(("dense", o))
        elif case.family == "ngram":
            got |= {("ngram_fwd", o[0]), ("ngram_bwd", o[1])}
            # the numerator: the implicit log sweeps over the case's own numerator graphs, the backward with the
            # graph gradient (the transitions' gradient flows through it)
            deg, nodes = ic.numerator_dims(case)
            Gf, Gb, okf, okb, f, b = implicit(emu, deg, 3, nodes, case.C, 0, 0, 1, case.dtype)
            assert (Gf, Gb, okf, okb) == (0, 0, 0, 0)
            got |= {("implicit_fwd", f), ("implicit_bwd", b)}
        elif case.family == "implicit":
            got |= {("implicit_fwd", o[4])} | ({("implicit_bwd", o[5])} if case.kind != "viterbi" else set())
        elif o["ok"]:
            got |= {("staged_fwd", o["fwd"]), ("staged_bwd", o["bwd"])}
            if case.graphs is not None:  # the tropical forward, the path and the tropical backward at the same G
                got |= {("staged_fwd", o["fwd"] + 4), ("staged_fwd", o["fwd"] + 8), ("staged_bwd", o["bwd"] + 4)}
    return got


def test_staged_cases_declare_their_route(emu):
    """the route test_gpu_instantiations asserts for each materialised CTC case is the plan's"""
    for case in ic.all_cases():
        if case.family == "staged" and case.expect is not None:
            o = case_outcome(emu, case)
            assert (o["ok"], o["ok"] and o["G"] == 1 and o["fused"]) == (case.expect["staged"],
                                                                            case.expect["fused"]), case.id


# ---- (c) coverage --------------------------------------------------------------------------------------------------

TABLES = {"bidir": 0, "dense": 1, "ngram_fwd": 2, "ngram_bwd": 3, "implicit_fwd": 4, "implicit_bwd": 5,
          "staged_fwd": 6, "staged_bwd": 7}


def test_every_instantiation_is_reached_or_listed(emu):
    got = reached(emu)
    missing = []
    for name, fam in TABLES.items():
        for i in range(emu.emu_plan_table_size(fam)):
            if (name, i) not in got and (name, i) not in UNREACHED:
                missing.append((name, i))
    assert not missing, missing
    stale = [k for k in UNREACHED if k in got]
    assert not stale, stale


def near(cases_vals, a, b):
    return a in cases_vals and b in cases_vals


def test_every_boundary_has_a_case_on_each_side(emu):
    cases = ic.all_cases()
    # bidir over C: per element size, the alphabets of the cases with the default bidir_mode
    for (esize, pair_ok, axis, *rest), (_, bounds) in bidir_domain(emu).items():
        sel = [c for c in cases if c.family == "bidir" and ic.ESIZE[c.dtype] == esize
               and ic.plan_inputs(c)["pair_ok"] == pair_ok]
        if axis == "C":
            vals = {c.C for c in sel if ic.plan_inputs(c)["max_nodes"] == 41}
            # changes between supported alphabets only (C % 4, C % 8 refusals interleave every other value)
            sup = [v for v in range(1, 257) if bidir(emu, v, 41, pair_ok, esize) is not None]
            for lo, hi in zip(sup, sup[1:]):
                if bidir(emu, lo, 41, pair_ok, esize) != bidir(emu, hi, 41, pair_ok, esize):
                    assert near(vals, lo, hi), (esize, pair_ok, lo, hi, sorted(vals))
            assert sup[-1] in vals, (esize, pair_ok, sup[-1])
        else:
            c0 = rest[0]
            if esize != 4 and c0 % 8:
                continue
            vals = {ic.plan_inputs(c)["max_nodes"] for c in sel if c.C == c0}
            for lo, hi in bounds:
                assert near(vals, lo, hi), (esize, pair_ok, c0, lo, hi, sorted(vals))
    for (esize, bg), (_, bounds) in dense_domain(emu).items():
        vals = {c.C for c in cases if c.family == "dense" and ic.ESIZE[c.dtype] == esize and (c.kind == "bigram") == bg}
        for lo, hi in bounds:
            assert near(vals, lo, hi), (esize, bg, lo, hi)
    for (esize, st), (_, bounds) in ngram_domain(emu).items():
        vals = {c.C for c in cases if c.family == "ngram" and ic.ESIZE[c.dtype] == esize and (c.kind == "asg") == st}
        for lo, hi in bounds:
            assert near(vals, lo, hi), (esize, st, lo, hi)
    (_, deg_bounds), (_, size_bounds) = staged_domain(emu)
    degs = [ic.plan_inputs(c) for c in cases if c.family == "staged" and c.graphs is not None]
    degs = {sum(p["sg_A"]) / sum(p["sg_N"]) for p in degs}
    for lo, hi in deg_bounds:  # arcs over 16 nodes: a case within half an arc per node on each side
        x = lo / 16.0
        assert any(x - 0.5 <= d <= x for d in degs) and any(x < d <= x + 0.5 for d in degs), (x, sorted(degs))
    us = {len(c.targets[0]) for c in cases if c.family == "staged" and c.targets is not None}
    for lo, hi in size_bounds:
        assert near(us, lo, hi), (lo, hi, sorted(us))
    for (arc, axis), (_, bounds) in implicit_domain(emu).items():
        sel = [ic.plan_inputs(c) for c in cases if c.family == "implicit"]
        if axis == "deg":
            vals = {p["max_in"] for p in sel if p["arc"] == arc and p["max_nodes"] == 8}
        else:
            vals = {p["max_nodes"] for p in sel if p["arc"] == arc and p["max_in"] == 21}
        for lo, hi in bounds:
            assert near(vals, lo, hi), (arc, axis, lo, hi, sorted(vals))


def test_every_outcome_is_covered(emu):
    """every distinct supported outcome of (a) is some case's outcome"""
    cases = ic.all_cases()
    outs = defaultdict(set)
    for c in cases:
        o = case_outcome(emu, c)
        outs[c.family].add(staged_key(o) if c.family == "staged" else o)
    want_b = set()
    for spans, _ in bidir_domain(emu).values():
        want_b |= {o for o in spans if o is not None}
    assert want_b <= outs["bidir"], sorted(want_b - outs["bidir"])
    want_d = set()
    for spans, _ in dense_domain(emu).values():
        want_d |= set(spans)
    assert want_d <= outs["dense"], want_d - outs["dense"]
    want_n = set()
    for spans, _ in ngram_domain(emu).values():
        want_n |= set(spans)
    want_n.discard(None)
    assert want_n <= outs["ngram"], want_n - outs["ngram"]
    deg, size = staged_domain(emu)
    assert set(size[0]) <= outs["staged"], set(size[0]) - outs["staged"]
    gs = {case_outcome(emu, c)["G"] for c in cases if c.family == "staged"}
    assert set(deg[0]) <= gs, set(deg[0]) - gs
    got = {case_outcome(emu, c)[:2] for c in cases if c.family == "implicit"}
    for spans, _ in implicit_domain(emu).values():
        assert set(spans) <= got, set(spans) - got
