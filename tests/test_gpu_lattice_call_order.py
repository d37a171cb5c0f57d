"""A composed lattice answers the same whatever ran on it before.

With exact_ties on (the default), gtnb_compose_linear leaves each row's in-arcs in compose order and marks the
lattice for k_order.cu's sort into the reference's relaxation order, where "first maximum in row order" is
shortestPath's tie rule (shortest.cpp:190-245).  The sort runs before the first call that hands arc ids or per-arc
values across the ABI (download, arc gradients in or out, a Viterbi path) and carries any arc gradients with it, so
forward and backward may run before it.  The reference is stateless: its answer holds for every call history.  So
each case below runs one measured operation on a freshly composed lattice after each history and compares it with
the reference and with a lattice that saw no history.

Inputs are tie-heavy on purpose: integer emissions in {-1, 0, 1}, CTC graphs with blank first and blank last
(where compose's discovery order is not the node order), repeated labels, ragged lengths with T_b = 1 and an
infeasible utterance, and general graph operands with integer weights, sorted and unsorted.

Arcs are matched by provenance (graph operand arc, emissions arc), which names an arc of compose(g, linear)
uniquely in both libraries.  A tropical gradient is not compared with the reference arc for arc: it marks one of
the tied best paths, so it is checked to be a best path."""
import numpy as np
import pytest

from gtn_b200 import capi
from oracle import pyoracle as po
from tests import util
from tests.test_gpu_gtn_lattice_entries import TS, Batch, needs_ref, total

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lctx():
    """a context of its own: the tests set its flags"""
    c = capi.Ctx(0)
    yield c
    c.close()


# ---------------------------------------------------------------------------------------------
# cases: graph operands, emissions, lengths, and what the reference (the C oracle, pinned to it) says of each entry


def random_graph(rng, Cn):
    n = int(rng.integers(2, 8))
    flags = np.zeros(n, np.uint8)
    flags[rng.integers(0, n, max(1, n // 3))] |= 1
    flags[rng.integers(0, n, max(1, n // 2))] |= 2
    na = int(rng.integers(n, 3 * n + 1))
    src, dst = rng.integers(0, n, na), rng.integers(0, n, na)
    lab = rng.integers(0, Cn, na)
    w = rng.integers(-1, 2, na).astype(np.float32)
    return po.Graph.from_arrays(flags, src, dst, lab, lab, w)


def make_case(name):
    if name == "general":
        rng = np.random.default_rng(4100)
        Cn, T = 4, 7
        lens = [T, T - 1, 2, T - 3, T, 1]
        ogs = []
        # operands with an accepting path at their length, sorted or not, and last one without
        while len(ogs) < len(lens):
            og = random_graph(rng, Cn)
            if len(ogs) % 2:
                og.arc_sort(False)
            lin = po.Graph.linear(lens[len(ogs)], Cn, np.zeros((lens[len(ogs)], Cn), np.float32))
            if (po.shortest_path(po.compose(og, lin)) is None) == (len(ogs) == len(lens) - 1):
                ogs.append(og)
        targets, blank = None, None
    else:
        blank_last = name == "ctc_blank_last"
        rng = np.random.default_rng(17 + blank_last)
        Cn, T = 6, 40
        blank = Cn - 1 if blank_last else 0
        labels = [l for l in range(Cn) if l != blank]
        targets = [rng.choice(labels, U).astype(np.int32) for U in (7, 5, 9, 1, 6, 8)]
        targets[1][1] = targets[1][0]  # a repeat: no skip arc between the two
        targets[2][3:6] = targets[2][2]  # a run of four
        # entry 3: one frame, one label; entry 5: eight labels in five frames, no alignment
        lens = [T, 33, 24, 1, 37, 5]
        ogs = [po.Graph.ctc(t, blank, True) for t in targets]
    B = len(ogs)
    e = rng.integers(-1, 2, (B, T, Cn)).astype(np.float32)
    deltas = np.array([1.5, -0.5, 2.0, 1.0, 0.25, -1.0][:B], np.float32)
    ref = []
    for b in range(B):
        Tb = lens[b]
        comp = po.compose(ogs[b], po.Graph.linear(Tb, Cn, e[b, :Tb]))
        g1, g2 = comp.gradinfo()
        arrs = comp.arrays()
        path = po.shortest_path(comp)
        log_s, log_g = po.forward_score_and_grad(comp, False, float(deltas[b]))
        trop_s = po.shortest_distance(comp, True)[0]
        r = dict(prov=list(zip(g1.tolist(), g2.tolist())), arrs=arrs, path=None if path is None else path.tolist(),
                 log=np.float32(log_s), log_grad=log_g, trop=np.float32(trop_s))
        if targets is not None and path is not None:
            r["ctc_labels"], r["ctc_score"] = po.viterbi_ctc(e[b, :Tb], targets[b], blank, True)
        ref.append(r)
    return dict(ogs=ogs, views=[util.view_of(g) for g in ogs], e=e, lens=lens, T=T, Cn=Cn, B=B, deltas=deltas,
                ref=ref)


CASES = ["ctc_blank_first", "ctc_blank_last", "general"]
_cases = {}


def case_of(name):
    if name not in _cases:
        _cases[name] = make_case(name)
    return _cases[name]


def compose(c, cs, exact_ties=1):
    c.set_flag("exact_ties", exact_ties)
    try:
        e_dev = c.to_device(cs["e"])
        lat = c.compose_linear(cs["views"], cs["lens"], cs["Cn"], e_dev, cs["T"] * cs["Cn"])
    finally:
        c.set_flag("exact_ties", 1)
    return lat


def downloads(lat):
    return [lat.download(b) for b in range(lat.B)]


# ---------------------------------------------------------------------------------------------
# histories: what may run on a freshly composed lattice before the measured operation


def h_forward(tropical):
    return lambda lat, cs: lat.forward(tropical, want_status=True)


def h_backward(tropical, with_deltas):
    def run(lat, cs):
        lat.forward(tropical, want_status=True)
        lat.backward(tropical, cs["deltas"] if with_deltas else None)
    return run


def h_set_arc_grads(lat, cs):
    _, na = lat.sizes()
    lat.set_arc_grads(2, np.arange(int(na[2]), dtype=np.float32) - 3.0)


def h_read_arc_grads(lat, cs):
    h_backward(False, True)(lat, cs)
    _, na = lat.sizes()
    lat.arc_grads(4, int(na[4]))


def h_download_other(lat, cs):
    lat.download(1)


def h_path(lat, cs):
    lat.viterbi_path(cs["T"], want_status=True)


STEPS = {
    "forward_log": h_forward(False),
    "forward_tropical": h_forward(True),
    "backward_log": h_backward(False, False),
    "backward_log_deltas": h_backward(False, True),
    "backward_tropical": h_backward(True, False),
    "backward_tropical_deltas": h_backward(True, True),
    "set_arc_grads": h_set_arc_grads,
    "arc_grads_read": h_read_arc_grads,
    "download_other": h_download_other,
    "viterbi_path": h_path,
}
HISTORIES = [[]] + [[s] for s in STEPS] + [
    ["backward_log", "set_arc_grads"],
    ["set_arc_grads", "backward_tropical_deltas"],
    ["download_other", "backward_log"],
    ["viterbi_path", "backward_log_deltas"],
    ["arc_grads_read", "viterbi_path"],
    ["backward_tropical", "arc_grads_read"],
]
HISTORY_IDS = ["+".join(h) or "nothing" for h in HISTORIES]


def run_history(lat, cs, history):
    for s in history:
        STEPS[s](lat, cs)


# ---------------------------------------------------------------------------------------------
# what must hold after any history


def check_paths(lat, cs):
    """viterbi_path: the reference's path, arc for arc (by provenance), its labels and its score"""
    out, _ = lat.viterbi_path(cs["T"], want_status=True)
    for b, r in enumerate(cs["ref"]):
        if r["path"] is None:
            assert out["lens"][b] == -1, (b, out["lens"][b])
            continue
        n = len(r["path"])
        assert out["lens"][b] == n, (b, out["lens"][b], n)
        d = lat.download(b)
        arcs = out["arcs"][b][:n]
        got = list(zip(d["gi_graph"][arcs].tolist(), d["gi_linear"][arcs].tolist()))
        want = [r["prov"][k] for k in r["path"]]
        assert got == want, (b, got, want)
        assert out["ilabels"][b][:n].tolist() == r["arrs"]["ilabel"][r["path"]].tolist(), b
        assert out["olabels"][b][:n].tolist() == r["arrs"]["olabel"][r["path"]].tolist(), b
        assert out["weights"][b][:n].tolist() == r["arrs"]["w"][r["path"]].tolist(), b
        score = np.float32(0.0)
        for w in out["weights"][b][:n]:
            score = np.float32(score + w)
        assert score == r["trop"], (b, score, r["trop"])
        if "ctc_labels" in r:
            assert out["ilabels"][b][:n].tolist() == r["ctc_labels"].tolist(), b
            assert score == np.float32(r["ctc_score"])


def check_downloads(lat, cs):
    """download returns the arc list a lattice that saw nothing returns"""
    fresh = compose(lat.ctx, cs)
    want = downloads(fresh)
    fresh.free()
    for b, (got, w) in enumerate(zip(downloads(lat), want)):
        for k in w:
            assert np.array_equal(got[k], w[k]), (b, k)


def check_grads(lat, cs):
    """arc gradients, read after a backward pass and paired with a download, are the reference's (log semiring) or
    mark a best path (tropical); the scores are the reference's"""
    s, _ = lat.forward(False, want_status=True)
    lat.backward(False, cs["deltas"])
    _, na = lat.sizes()
    grads = [lat.arc_grads(b, int(na[b])) for b in range(lat.B)]
    d = downloads(lat)
    for b, r in enumerate(cs["ref"]):
        assert util.close(s[b], r["log"]), (b, s[b], r["log"])
        if not np.isfinite(r["log"]):
            continue
        prov = list(zip(d[b]["gi_graph"].tolist(), d[b]["gi_linear"].tolist()))
        assert sorted(prov) == sorted(r["prov"])
        ours = dict(zip(prov, grads[b].tolist()))
        got = np.array([ours[p] for p in r["prov"]], np.float32)
        assert util.grad_close(got, r["log_grad"], abs(r["log"])), (b, float(np.abs(got - r["log_grad"]).max()))
    s, _ = lat.forward(True, want_status=True)
    lat.backward(True, cs["deltas"])
    grads = [lat.arc_grads(b, int(na[b])) for b in range(lat.B)]
    for b, r in enumerate(cs["ref"]):
        assert s[b] == r["trop"], (b, s[b], r["trop"])
        if not np.isfinite(r["trop"]):
            continue
        on = np.nonzero(grads[b])[0]
        assert (grads[b][on] == cs["deltas"][b]).all(), b
        # one arc per frame, chained from a start node to an accept node, scoring the best path
        on = on[np.argsort(d[b]["gi_linear"][on] // cs["Cn"])]
        assert len(on) == cs["lens"][b], (b, len(on))
        assert (d[b]["flags"][d[b]["src"][on[0]]] & 1) and (d[b]["flags"][d[b]["dst"][on[-1]]] & 2), b
        assert (d[b]["src"][on[1:]] == d[b]["dst"][on[:-1]]).all(), b
        assert np.float32(d[b]["w"][on].astype(np.float64).sum()) == r["trop"], b


CHECKS = {"viterbi_path": check_paths, "download": check_downloads, "arc_grads": check_grads}


@pytest.mark.parametrize("measured", list(CHECKS))
@pytest.mark.parametrize("history", HISTORIES, ids=HISTORY_IDS)
@pytest.mark.parametrize("staged", [1, 0])
@pytest.mark.parametrize("case", CASES)
def test_answers_do_not_depend_on_call_order(lctx, case, staged, history, measured):
    cs = case_of(case)
    lctx.set_flag("staged", staged)
    try:
        lat = compose(lctx, cs)
        run_history(lat, cs, history)
        CHECKS[measured](lat, cs)
        lat.free()
    finally:
        lctx.set_flag("staged", 1)


# ---------------------------------------------------------------------------------------------
# controls


@pytest.mark.parametrize("history", [[], ["backward_log"], ["set_arc_grads"], ["arc_grads_read", "viterbi_path"]],
                         ids=["nothing", "backward_log", "set_arc_grads", "arc_grads_read+viterbi_path"])
def test_without_exact_ties_the_lattice_stays_in_compose_order(lctx, history):
    """exact_ties = 0: nothing is sorted; paths, arc lists and scores are those of a lattice that saw nothing"""
    cs = case_of("ctc_blank_last")
    fresh = compose(lctx, cs, exact_ties=0)
    want_dl = downloads(fresh)
    want_path = fresh.viterbi_path(cs["T"], want_status=True)[0]
    fresh.free()
    lat = compose(lctx, cs, exact_ties=0)
    run_history(lat, cs, history)
    path = lat.viterbi_path(cs["T"], want_status=True)[0]
    assert np.array_equal(path["lens"], want_path["lens"])
    for b, n in enumerate(want_path["lens"]):
        for k in ("arcs", "ilabels", "olabels", "weights"):
            assert np.array_equal(path[k][b][:max(n, 0)], want_path[k][b][:max(n, 0)]), (b, k)
    for got, w in zip(downloads(lat), want_dl):
        for k in w:
            assert np.array_equal(got[k], w[k]), k
    lat.free()


def test_sort_runs_once_and_never_on_forward_or_backward(lctx):
    """forward + backward launch what they launch without exact_ties; the first arc-gradient read sorts (two
    launches), later reads and a path do not sort again"""
    cs = case_of("ctc_blank_last")
    counts = []
    for exact in (0, 1):
        lat = compose(lctx, cs, exact_ties=exact)
        before = lctx.launches
        lat.forward(False, want_status=True)
        lat.backward(False, cs["deltas"])
        counts.append(lctx.launches - before)
        if exact:
            _, na = lat.sizes()
            before = lctx.launches
            lat.arc_grads(0, int(na[0]))
            assert lctx.launches - before == 2  # relax_order + sort_rows
            before = lctx.launches
            lat.arc_grads(1, int(na[1]))
            lat.download(2)
            assert lctx.launches == before
            before = lctx.launches
            lat.viterbi_path(cs["T"], want_status=True)
            path_launches = lctx.launches - before
        else:
            before = lctx.launches
            lat.viterbi_path(cs["T"], want_status=True)
            plain_path_launches = lctx.launches - before
        lat.free()
    assert counts[0] == counts[1], counts
    assert path_launches == plain_path_launches


def test_arc_grads_dev_is_in_download_order(lctx):
    """the device pointer to the arc gradients sorts a pending lattice first, like the host read"""
    cs = case_of("ctc_blank_last")
    lat = compose(lctx, cs)
    lat.forward(False, want_status=True)
    lat.backward(False, cs["deltas"])
    ptr = lat.arc_grads_dev()
    assert ptr
    _, na = lat.sizes()
    host = lat.arc_grads(0, int(na[0]))  # entry 0 starts the slab
    dev = np.zeros(int(na[0]), np.float32)
    lctx._check(capi.lib().gtnb_memcpy_d2h(lctx.h, dev.ctypes.data, ptr, dev.nbytes))
    lctx.synchronize()
    assert np.array_equal(dev, host)
    lat.free()


def test_backward_after_a_path_still_needs_a_forward(lctx):
    cs = case_of("ctc_blank_first")
    lat = compose(lctx, cs)
    lat.forward(False, want_status=True)
    lat.viterbi_path(cs["T"], want_status=True)
    with pytest.raises(capi.GtnbError, match="no matching gtnb_forward") as ex:
        lat.backward(False)
    assert ex.value.code == capi.ERR_LOGIC
    lat.free()


# ---------------------------------------------------------------------------------------------
# the gtn API, against the reference compiled into oracle/_ref


@pytest.fixture(scope="module")
def gtn():
    import gtn_b200.gtn as g
    return g


def assert_paths(paths, rpaths):
    for b, (p, r) in enumerate(zip(paths, rpaths)):
        ra = r.arrays()
        assert p.labels_to_list() == ra["ilabel"].tolist(), b
        assert p.labels_to_list(False) == ra["olabel"].tolist(), b
        assert p.weights_to_list() == ra["w"].tolist(), b


@needs_ref
@pytest.mark.parametrize("read_between", [True, False], ids=["read", "unread"])
@pytest.mark.parametrize("op", ["viterbi_score", "forward_score"])
def test_gtn_single_lattice_score_backward_path(gtn, op, read_between):
    """Viterbi training then decoding on one lattice: score -> backward -> viterbi_path"""
    bt = Batch(gtn, integer=True)
    for b in range(len(TS)):
        lat = gtn.intersect(bt.ctcs[b], bt.ems[b])
        rlat = po.ref_op("intersect", bt.rctcs[b], bt.rems[b])
        s, rs = getattr(gtn, op)(lat), po.ref_op(op, rlat)
        if op == "viterbi_score":
            assert s.item() == rs.item(), b
        assert util.close(s.item(), rs.item()), b
        gtn.backward(s)
        po.ref_backward(rs)
        if read_between:
            lat.grad().weights_to_numpy()
        path = gtn.viterbi_path(lat)
        assert_paths([path], [po.ref_op("viterbi_path", rlat)])
        if op == "forward_score":
            go, gr = bt.lattice_grads(b, lat, rlat)
            assert util.grad_close(go, gr, abs(rs.item())), b
            for g, r in ((bt.ems[b], bt.rems[b]), (bt.ctcs[b], bt.rctcs[b])):
                assert util.grad_close(g.grad().weights_to_numpy(), r.grad().weights(), abs(rs.item())), b
        else:
            # a tied best path's one-hot: one label per frame, scoring the Viterbi score
            ge = bt.ems[b].grad().weights_to_numpy().reshape(TS[b], -1)
            assert (ge.sum(1) == 1).all() and set(np.unique(ge)) <= {0.0, 1.0}, b
            assert np.float32((ge * bt.es[b]).sum()) == np.float32(rs.item()), b


@needs_ref
@pytest.mark.parametrize("read_between", [True, False], ids=["read", "unread"])
def test_gtn_list_score_backward_path(gtn, read_between):
    """intersect(list, list) -> forward_score(list) -> backward -> viterbi_path(list)"""
    bt = Batch(gtn, integer=True)
    lats, rlats = bt.lattices()
    scores = gtn.forward_score(lats)
    rscores = [po.ref_op("forward_score", r) for r in rlats]
    for s, r in zip(scores, rscores):
        assert util.close(s.item(), r.item())
    mag = max(abs(r.item()) for r in rscores)
    gtn.backward(total(gtn, scores))
    for r in rscores:
        po.ref_backward(r)
    if read_between:
        for b in range(len(TS)):
            go, gr = bt.lattice_grads(b, lats[b], rlats[b])
            assert util.grad_close(go, gr, mag), b
    assert_paths(gtn.viterbi_path(lats), [po.ref_op("viterbi_path", r) for r in rlats])
    for b in range(len(TS)):
        go, gr = bt.lattice_grads(b, lats[b], rlats[b])
        assert util.grad_close(go, gr, mag), b
        for g, r in ((bt.ems[b], bt.rems[b]), (bt.ctcs[b], bt.rctcs[b])):
            assert util.grad_close(g.grad().weights_to_numpy(), r.grad().weights(), mag), b
