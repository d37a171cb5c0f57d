"""Single-graph and list ops on the entries of a batched lattice, held to the unmodified reference.

gtn.intersect(list, list) over (target graph, emissions) pairs returns B graphs that are entries of ONE device lattice
(gtn/batched.cpp).  Every other op can be handed such an entry: forward_score / viterbi_score / viterbi_path of one
entry, list forms whose entries are a subset, a permutation or contain a duplicate, paths decoded in a batch,
gradients accumulated over several backward passes, an entry differentiated both through its score and through its
path.  Each test runs the same gtn program on gtn_b200.gtn and on the reference compiled into oracle/_ref (where the
list overloads are per-element loops, as in the reference's bindings) and compares scores, paths and gradients.

Composed lattices are numbered frame-major here and in BFS order by the reference, so arc gradients of a lattice are
compared per arc identity: a CTC graph is deterministic (the out-arcs of a state carry distinct labels), so an arc of
intersect(ctc, emissions) is named by (frame, CTC state it leaves, label)."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import util

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not po.have_ref(), reason="oracle/_ref not built (needs /root/reference)")

# ragged batch: entry 0 is neither the longest nor the shortest lattice, so an op that falls back to entry 0, or
# sizes a buffer by the entry it was given, gives a wrong number
TS = [22, 40, 31, 15, 36, 27]
US = [5, 11, 8, 3, 10, 6]
C = 7
B = len(TS)


@pytest.fixture(scope="module")
def gtn():
    import gtn_b200.gtn as g
    return g


def ctc_arrays(target, blank=0):
    """ctcGraph of test/criterion_test.cpp:37-54 as arrays, in its arc creation order."""
    L = len(target)
    S = 2 * L + 1
    flags = np.zeros(S, np.uint8)
    flags[0] |= 1
    flags[S - 1] |= 2
    flags[S - 2] |= 2
    src, dst, lab = [], [], []
    for s in range(S):
        label = target[(s - 1) // 2] if s % 2 else blank
        src.append(s), dst.append(s), lab.append(label)
        if s > 0:
            src.append(s - 1), dst.append(s), lab.append(label)
        if s % 2 and s > 1 and label != target[(s - 1) // 2 - 1]:
            src.append(s - 2), dst.append(s), lab.append(label)
    lab = np.asarray(lab, np.int32)
    return flags, np.asarray(src, np.int32), np.asarray(dst, np.int32), lab, lab.copy(), np.zeros(len(lab), np.float32)


class Batch:
    """The same B (CTC graph, emissions) pairs in gtn_b200.gtn (ctcs, ems) and in the reference (rctcs, rems)."""

    def __init__(self, gtn, seed=7):
        rng = np.random.default_rng(seed)
        self.gtn = gtn
        self.es = [rng.uniform(-5, 5, (T, C)).astype(np.float32) for T in TS]
        self.targets = [rng.integers(1, C, U).astype(np.int32).tolist() for U in US]
        self.arrays = [ctc_arrays(t) for t in self.targets]
        self.ctcs, self.ems, self.rctcs, self.rems = [], [], [], []
        for b in range(B):
            flags, src, dst, il, ol, w = self.arrays[b]
            g = gtn.Graph()
            for f in flags:
                g.add_node(bool(f & 1), bool(f & 2))
            for a in range(len(src)):
                g.add_arc(int(src[a]), int(dst[a]), int(il[a]), int(ol[a]), float(w[a]))
            g.arc_sort()
            em = gtn.linear_graph(TS[b], C)
            em.set_weights(self.es[b].ravel())
            self.ctcs.append(g)
            self.ems.append(em)
            if po.have_ref():
                r = po.RefGraph.from_arrays(*self.arrays[b])
                r.arc_sort()
                self.rctcs.append(r)
                self.rems.append(po.RefGraph.linear(TS[b], C, self.es[b].ravel()))

    def lattices(self):
        lats = self.gtn.intersect(self.ctcs, self.ems)
        assert all(g.is_device_resident() for g in lats)
        rlats = [po.ref_op("intersect", c, e) for c, e in zip(self.rctcs, self.rems)] if self.rctcs else []
        return lats, rlats

    def arc_keys(self, b, flags, src, dst, il):
        """(frame, CTC state left, label) of every arc of entry b's lattice; node 0..N-1 numbering of either library."""
        cf, cs, cd, cl, _, _ = self.arrays[b]
        step = {(int(s), int(l)): int(d) for s, d, l in zip(cs, cd, cl)}
        starts = np.nonzero(flags & 1)[0]
        assert len(starts) == 1
        state = {int(starts[0]): (0, 0)}
        out = {}
        for a in range(len(src)):
            out.setdefault(int(src[a]), []).append(a)
        todo = [int(starts[0])]
        while todo:
            u = todo.pop()
            t, s = state[u]
            for a in out.get(u, []):
                nxt = (t + 1, step[(s, int(il[a]))])
                v = int(dst[a])
                if v not in state:
                    state[v] = nxt
                    todo.append(v)
                assert state[v] == nxt
        return [state[int(src[a])] + (int(il[a]),) for a in range(len(src))]

    def lattice_grads(self, b, lat, rlat):
        """entry b's lattice gradient in both libraries, arcs put in one order by their identity"""
        d = self.gtn.arc_lists(lat)
        ko = self.arc_keys(b, d["flags"], d["src"], d["dst"], d["ilabel"])
        ra = rlat.arrays()
        kr = self.arc_keys(b, ra["flags"], ra["src"], ra["dst"], ra["ilabel"])
        assert sorted(ko) == sorted(kr)
        go = lat.grad().weights_to_numpy()
        gr = rlat.grad().weights()
        return go[sorted(range(len(ko)), key=ko.__getitem__)], gr[sorted(range(len(kr)), key=kr.__getitem__)]


def grad_or_none(g):
    return g.grad().weights_to_numpy() if g.is_grad_available() else None


def ref_grad_or_none(r):
    return r.grad().weights() if r.is_grad_available() else None


def assert_grads(bt, mag, lats=None, rlats=None, entries=range(B), exact=False):
    """emissions, target graphs and (where given) lattice entries carry the reference's gradient, or none where it
    has none"""
    same = np.array_equal if exact else (lambda a, b: util.grad_close(a, b, mag))
    for b in entries:
        pairs = [("ems", bt.ems[b], bt.rems[b]), ("ctcs", bt.ctcs[b], bt.rctcs[b])]
        for what, g, r in pairs:
            go, gr = grad_or_none(g), ref_grad_or_none(r)
            assert (go is None) == (gr is None), (what, b, go is None, gr is None)
            if go is not None:
                assert same(go, gr), (what, b, float(np.abs(go - gr).max()))
        if lats is not None:
            assert lats[b].is_grad_available() == rlats[b].is_grad_available(), ("lattice", b)
            if rlats[b].is_grad_available():
                go, gr = bt.lattice_grads(b, lats[b], rlats[b])
                assert same(go, gr), ("lattice", b, float(np.abs(go - gr).max()))


def total(gtn, scores):
    """one scalar over a list of scalars, so that one backward pass walks every tape once"""
    acc = scores[0]
    for s in scores[1:]:
        acc = gtn.add(acc, s)
    return acc


def ref_total(scores):
    acc = scores[0]
    for s in scores[1:]:
        acc = po.ref_op("add", acc, s)
    return acc


def raises(fn):
    try:
        fn()
    except Exception as ex:  # noqa: BLE001 -- the two libraries raise their own types
        return ex
    return None


# ---------------------------------------------------------------------------------------------
# A. single ops on each entry


@needs_ref
@pytest.mark.parametrize("entry,op", [(4, "forward_score"), (0, "viterbi_score"), (3, "forward_score")])
def test_single_ops_on_each_entry(gtn, entry, op):
    bt = Batch(gtn)
    lats, rlats = bt.lattices()
    mag = 0.0
    for b in range(B):
        for name in ("forward_score", "viterbi_score"):
            got = getattr(gtn, name)(lats[b]).item()
            want = po.ref_op(name, rlats[b]).item()
            mag = max(mag, abs(want))
            if name == "viterbi_score":
                assert got == want, (b, got, want)
            assert util.close(got, want), (name, b, got, want)
    s = getattr(gtn, op)(lats[entry])
    rs = po.ref_op(op, rlats[entry])
    assert util.close(s.item(), rs.item())
    gtn.backward(s)
    po.ref_backward(rs)
    assert_grads(bt, mag, lats, rlats)
    for b in range(B):
        assert bt.ems[b].is_grad_available() == (b == entry)


# ---------------------------------------------------------------------------------------------
# B. list forms that miss the one-batch route


@needs_ref
@pytest.mark.parametrize("order", [[3, 1], [5, 4, 3, 2, 1, 0], [0, 0, 2, 3, 4, 5]], ids=["subset", "reversed", "duplicate"])
@pytest.mark.parametrize("op", ["forward_score", "viterbi_score"])
def test_list_forms_off_the_batch_route(gtn, order, op):
    bt = Batch(gtn)
    lats, rlats = bt.lattices()
    scores = getattr(gtn, op)([lats[b] for b in order])
    rscores = [po.ref_op(op, rlats[b]) for b in order]
    assert len(scores) == len(order)
    for s, r in zip(scores, rscores):
        assert util.close(s.item(), r.item()), (s.item(), r.item())
    mag = max(abs(r.item()) for r in rscores)
    gtn.backward(total(gtn, scores))
    po.ref_backward(ref_total(rscores))
    assert_grads(bt, mag, lats, rlats)


# ---------------------------------------------------------------------------------------------
# C. decoding


@needs_ref
@pytest.mark.parametrize("form", ["list", "single"])
def test_viterbi_paths_of_entries(gtn, form):
    bt = Batch(gtn)
    lats, rlats = bt.lattices()
    paths = gtn.viterbi_path(lats) if form == "list" else [gtn.viterbi_path(g) for g in lats]
    rpaths = [po.ref_op("viterbi_path", r) for r in rlats]
    for b in range(B):
        ra = rpaths[b].arrays()
        assert paths[b].num_arcs() == rpaths[b].num_arcs == TS[b], b
        assert paths[b].labels_to_list() == ra["ilabel"].tolist(), b
        assert paths[b].labels_to_list(False) == ra["olabel"].tolist(), b
        assert paths[b].weights_to_list() == ra["w"].tolist(), b
    gtn.backward(total(gtn, [gtn.viterbi_score(p) for p in paths]))
    po.ref_backward(ref_total([po.ref_op("viterbi_score", p) for p in rpaths]))
    assert_grads(bt, 0.0, lats, rlats, exact=True)
    for b in range(B):
        onehot = np.zeros((TS[b], C), np.float32)
        onehot[np.arange(TS[b]), paths[b].labels_to_list()] = 1.0
        assert np.array_equal(bt.ems[b].grad().weights_to_numpy().reshape(TS[b], C), onehot), b


# ---------------------------------------------------------------------------------------------
# D. accumulation across iterations, without zero_grad


@needs_ref
@pytest.mark.parametrize("read_between", [True, False], ids=["read", "unread"])
def test_gradients_accumulate_across_iterations(gtn, read_between):
    bt = Batch(gtn)

    def iteration():
        lats, rlats = bt.lattices()
        losses = gtn.subtract(gtn.forward_score(bt.ems), gtn.forward_score(lats))
        rlosses = [po.ref_op("subtract", po.ref_op("forward_score", e), po.ref_op("forward_score", r))
                   for e, r in zip(bt.rems, rlats)]
        gtn.backward(losses)
        for r in rlosses:
            po.ref_backward(r)
        for s, r in zip(losses, rlosses):
            assert util.close(s.item(), r.item())
        return max(abs(po.ref_op("forward_score", e).item()) for e in bt.rems)

    mag = iteration()
    if read_between:
        assert_grads(bt, mag)
    iteration()
    assert_grads(bt, 2 * mag)
    for g in bt.ems + bt.ctcs:
        g.zero_grad()
    for r in bt.rems + bt.rctcs:
        r.zero_grad()
    iteration()
    assert_grads(bt, mag)


# ---------------------------------------------------------------------------------------------
# E. both a recorded seed and host deltas on one entry


@needs_ref
@pytest.mark.parametrize("entry", [2, 0])
def test_seed_and_host_deltas_on_one_entry(gtn, entry):
    bt = Batch(gtn)
    lats, rlats = bt.lattices()
    s = gtn.forward_score(lats)
    rs = po.ref_op("forward_score", rlats[entry])
    assert util.close(s[entry].item(), rs.item())
    loss = gtn.add(s[entry], gtn.viterbi_score(gtn.viterbi_path(lats[entry])))
    rloss = po.ref_op("add", rs, po.ref_op("viterbi_score", po.ref_op("viterbi_path", rlats[entry])))
    assert util.close(loss.item(), rloss.item())
    gtn.backward(loss)
    po.ref_backward(rloss)
    assert_grads(bt, abs(rloss.item()), lats, rlats)


# ---------------------------------------------------------------------------------------------
# F. mixed semirings


@needs_ref
@pytest.mark.parametrize("entry", [1, 0])
def test_mixed_semirings_through_single_ops(gtn, entry):
    bt = Batch(gtn)
    lats, rlats = bt.lattices()
    loss = gtn.add(gtn.forward_score(lats[entry]), gtn.viterbi_score(lats[entry]))
    rloss = po.ref_op("add", po.ref_op("forward_score", rlats[entry]), po.ref_op("viterbi_score", rlats[entry]))
    assert util.close(loss.item(), rloss.item())
    gtn.backward(loss)
    po.ref_backward(rloss)
    assert_grads(bt, abs(rloss.item()), lats, rlats)


def test_mixed_semirings_through_list_forms_is_refused(gtn):
    """Both list forms of one batched lattice in one backward pass would need two batched backward sweeps in two
    semirings: an explicit error, never a number."""
    bt = Batch(gtn)
    lats = gtn.intersect(bt.ctcs, bt.ems)
    fs, vs = gtn.forward_score(lats), gtn.viterbi_score(lats)
    with pytest.raises(RuntimeError, match="cannot both be differentiated"):
        gtn.backward(gtn.add(fs[3], vs[3]))


# ---------------------------------------------------------------------------------------------
# G. parked gradients are not clobbered by a later single-entry backward


@needs_ref
@pytest.mark.parametrize("between", ["nothing", "emissions", "everything"])
def test_parked_gradients_survive_single_entry_backward(gtn, between):
    """The list route's lattice-entry gradients stay on the device until read; a later backward of a single op on
    the same lattice relaunches over every entry.  'nothing': the batch has not run its backward yet; 'emissions':
    it has, its lattice-entry gradients are still unread; 'everything': all read."""
    bt = Batch(gtn)
    lats, rlats = bt.lattices()
    s = gtn.forward_score(lats)
    rs = [po.ref_op("forward_score", r) for r in rlats]
    gtn.backward(s)
    for r in rs:
        po.ref_backward(r)
    mag = max(abs(r.item()) for r in rs)
    if between != "nothing":
        for b in range(B):
            bt.ems[b].grad().weights_to_numpy()
            bt.ctcs[b].grad().weights_to_numpy()
            if between == "everything":
                lats[b].grad().weights_to_numpy()
    s0 = gtn.forward_score(lats[0])
    rs0 = po.ref_op("forward_score", rlats[0])
    assert util.close(s0.item(), rs0.item())
    # both backwards run without retain_graph: whatever the reference's cleared tape lets through, and whether it
    # raises, is the expectation
    ours, theirs = raises(lambda: gtn.backward(s0)), raises(lambda: po.ref_backward(rs0))
    assert (ours is None) == (theirs is None), (ours, theirs)
    assert_grads(bt, mag, lats, rlats)


# ---------------------------------------------------------------------------------------------
# H. decoding every entry of a batch is one launch


def test_list_viterbi_path_is_one_packed_launch(gtn):
    bt = Batch(gtn)
    lats = gtn.intersect(bt.ctcs, bt.ems)
    l0 = gtn.device_launch_count()
    one = gtn.viterbi_path(lats[0])
    single = gtn.device_launch_count() - l0
    lats = gtn.intersect(bt.ctcs, bt.ems)
    l0 = gtn.device_launch_count()
    paths = gtn.viterbi_path(lats)
    launches = gtn.device_launch_count() - l0
    # a whole-batch decode for one entry costs what the list costs; decoding per entry would cost B of them
    assert 0 < launches <= single, (launches, single)
    assert len(paths) == B
    assert paths[0].labels_to_list() == one.labels_to_list()
    assert [p.num_arcs() for p in paths] == TS
