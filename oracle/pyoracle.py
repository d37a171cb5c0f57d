"""ctypes access to the CPU oracle -- TEST INFRASTRUCTURE, not product code.

Two libraries:
  * ``liboracle``  = oracle/libgtn_oracle.so, the plain-C restatement
    (oracle/gtn_oracle.c) -- travels everywhere, built by `make -C oracle oracle`.
  * ``libref``     = oracle/_ref/libgtn_ref.so, the UNMODIFIED reference
    compiled from /root/reference plus our C shim (oracle/ref_driver.cpp).
    Built only where /root/reference exists; the prebuilt .so travels to the
    GPU box with the snapshot.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
``--impl reference`` legs may import this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "libgtn_oracle.so")
REF_SO = os.path.join(HERE, "_ref", "libgtn_ref.so")

_f32p = C.POINTER(C.c_float)
_i32p = C.POINTER(C.c_int)
_i64p = C.POINTER(C.c_int64)
_u8p = C.POINTER(C.c_uint8)


def build(ref=True):
    """Compile the oracle (and the reference, when its sources are present)."""
    subprocess.check_call(["make", "-s", "-C", HERE, "oracle"])
    if ref:
        subprocess.check_call(["make", "-s", "-C", HERE, "ref"])


class OGraph(C.Structure):
    _fields_ = [
        ("num_nodes", C.c_int), ("num_arcs", C.c_int),
        ("cap_nodes", C.c_int), ("cap_arcs", C.c_int),
        ("flags", _u8p),
        ("src", _i32p), ("dst", _i32p), ("ilabel", _i32p), ("olabel", _i32p),
        ("w", _f32p),
        ("in_", C.POINTER(_i32p)), ("out", C.POINTER(_i32p)),
        ("nin", _i32p), ("nout", _i32p), ("cin", _i32p), ("cout", _i32p),
        ("start", _i32p), ("num_start", C.c_int), ("cap_start", C.c_int),
        ("accept", _i32p), ("num_accept", C.c_int), ("cap_accept", C.c_int),
        ("ilabel_sorted", C.c_int), ("olabel_sorted", C.c_int),
        ("gi1", _i32p), ("gi2", _i32p),
    ]


_OGP = C.POINTER(OGraph)


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def _i32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.int32)


def _u8(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.uint8)


_lib = None


def liboracle():
    global _lib
    if _lib is None:
        if not os.path.exists(ORACLE_SO):
            build(ref=False)
        L = C.CDLL(ORACLE_SO)
        L.og_new.restype = _OGP
        L.og_from_arrays.restype = _OGP
        L.og_from_arrays.argtypes = [C.c_int, _u8p, C.c_int, _i32p, _i32p, _i32p, _i32p, _f32p]
        L.og_linear.restype = _OGP
        L.og_linear.argtypes = [C.c_int, C.c_int, _f32p]
        L.og_compose.restype = _OGP
        L.og_compose.argtypes = [_OGP, _OGP, C.c_int]
        L.og_free.argtypes = [_OGP]
        L.og_arc_sort.argtypes = [_OGP, C.c_int]
        L.og_get_adj.argtypes = [_OGP, _i32p, _i32p, _i32p, _i32p]
        L.og_ctc_graph.restype = _OGP
        L.og_ctc_graph.argtypes = [_i32p, C.c_int, C.c_int, C.c_int]
        L.og_transitions_graph.restype = _OGP
        L.og_transitions_graph.argtypes = [C.c_int, _f32p]
        L.og_fal_graph.restype = _OGP
        L.og_fal_graph.argtypes = [_i32p, C.c_int]
        L.og_shortest_distance.argtypes = [_OGP, C.c_int, _f32p, _f32p, _f32p, _i64p]
        L.og_shortest_distance_grad.argtypes = [
            _OGP, C.c_int, C.c_float, C.c_float, _f32p, _f32p, _i64p, _f32p]
        L.og_shortest_path.argtypes = [_OGP, _i32p, _i32p]
        L.og_compose_grad.argtypes = [_OGP, _f32p, _f32p, _f32p]
        L.og_ctc_loss.argtypes = [
            C.c_int, C.c_int, _f32p, _i32p, C.c_int, C.c_int, C.c_int, _f32p, _f32p]
        L.og_asg_loss.argtypes = [
            C.c_int, C.c_int, _f32p, _f32p, _i32p, C.c_int, _f32p, _f32p, _f32p]
        L.og_viterbi_dense.argtypes = [C.c_int, C.c_int, _f32p, _f32p, _i32p, _f32p]
        L.og_viterbi_ctc.argtypes = [
            C.c_int, C.c_int, _f32p, _i32p, C.c_int, C.c_int, C.c_int, _i32p, _f32p]
        _lib = L
    return _lib


class OracleError(Exception):
    def __init__(self, code):
        super().__init__("oracle status %d" % code)
        self.code = code


class Graph:
    """Owning handle on an og_graph."""

    def __init__(self, ptr):
        self.ptr = ptr

    def __del__(self):
        try:
            if self.ptr:
                liboracle().og_free(self.ptr)
                self.ptr = None
        except Exception:
            pass

    @staticmethod
    def from_arrays(flags, src, dst, il, ol, w=None):
        flags, src, dst, il, ol, w = _u8(flags), _i32(src), _i32(dst), _i32(il), _i32(ol), _f32(w)
        return Graph(liboracle().og_from_arrays(
            len(flags), _p(flags, _u8p), len(src), _p(src, _i32p), _p(dst, _i32p),
            _p(il, _i32p), _p(ol, _i32p), _p(w, _f32p)))

    @staticmethod
    def linear(T, Cn, w=None):
        w = _f32(w)
        return Graph(liboracle().og_linear(T, Cn, _p(w, _f32p)))

    @staticmethod
    def ctc(target, blank, arc_sort):
        t = _i32(target)
        return Graph(liboracle().og_ctc_graph(_p(t, _i32p), len(t), blank, int(arc_sort)))

    @staticmethod
    def transitions(Cn, w=None):
        w = _f32(w)
        return Graph(liboracle().og_transitions_graph(Cn, _p(w, _f32p)))

    @staticmethod
    def fal(target):
        t = _i32(target)
        return Graph(liboracle().og_fal_graph(_p(t, _i32p), len(t)))

    @property
    def g(self):
        return self.ptr.contents

    @property
    def num_nodes(self):
        return self.g.num_nodes

    @property
    def num_arcs(self):
        return self.g.num_arcs

    def _arr(self, p, n, dt):
        if n == 0:
            return np.zeros(0, dtype=dt)
        return np.ctypeslib.as_array(p, shape=(n,)).astype(dt, copy=True)

    def arrays(self):
        g = self.g
        return dict(
            flags=self._arr(g.flags, g.num_nodes, np.uint8),
            src=self._arr(g.src, g.num_arcs, np.int32),
            dst=self._arr(g.dst, g.num_arcs, np.int32),
            ilabel=self._arr(g.ilabel, g.num_arcs, np.int32),
            olabel=self._arr(g.olabel, g.num_arcs, np.int32),
            w=self._arr(g.w, g.num_arcs, np.float32),
            start=self._arr(g.start, g.num_start, np.int32),
            accept=self._arr(g.accept, g.num_accept, np.int32),
        )

    def gradinfo(self):
        g = self.g
        return self._arr(g.gi1, g.num_arcs, np.int32), self._arr(g.gi2, g.num_arcs, np.int32)

    def adjacency(self):
        n, a = self.num_nodes, self.num_arcs
        ip, ia = np.zeros(n + 1, np.int32), np.zeros(max(a, 1), np.int32)
        op, oa = np.zeros(n + 1, np.int32), np.zeros(max(a, 1), np.int32)
        liboracle().og_get_adj(self.ptr, _p(ip, _i32p), _p(ia, _i32p), _p(op, _i32p), _p(oa, _i32p))
        return ip, ia[:a], op, oa[:a]

    def arc_sort(self, olabel=False):
        liboracle().og_arc_sort(self.ptr, int(olabel))

    def set_sorted(self, ilabel_sorted, olabel_sorted):
        self.g.ilabel_sorted = int(ilabel_sorted)
        self.g.olabel_sorted = int(olabel_sorted)


def compose(a, b):
    return Graph(liboracle().og_compose(a.ptr, b.ptr, 0))


def intersect(a, b):
    return Graph(liboracle().og_compose(a.ptr, b.ptr, 1))


def shortest_distance(g, tropical=False):
    """-> (score, scores[N], max_cache[N+1], arg_cache[N+1])"""
    n = g.num_nodes
    out = C.c_float()
    sc = np.zeros(n + 1, np.float32)
    mc = np.zeros(n + 1, np.float32)
    ac = np.zeros(n + 1, np.int64)
    rc = liboracle().og_shortest_distance(
        g.ptr, int(tropical), C.byref(out), _p(sc, _f32p), _p(mc, _f32p), _p(ac, _i64p))
    if rc:
        raise OracleError(rc)
    return out.value, sc[:n], mc, ac


def shortest_distance_grad(g, tropical, output, delta, scores, max_cache, arg_cache):
    gr = np.zeros(max(g.num_arcs, 1), np.float32)
    sc = np.zeros(g.num_nodes + 1, np.float32)
    sc[:g.num_nodes] = scores
    rc = liboracle().og_shortest_distance_grad(
        g.ptr, int(tropical), float(output), float(delta), _p(sc, _f32p),
        _p(_f32(max_cache), _f32p), _p(np.ascontiguousarray(arg_cache, np.int64), _i64p),
        _p(gr, _f32p))
    if rc:
        raise OracleError(rc)
    return gr[:g.num_arcs]


def forward_score_and_grad(g, tropical=False, delta=1.0):
    s, sc, mc, ac = shortest_distance(g, tropical)
    return s, shortest_distance_grad(g, tropical, s, delta, sc, mc, ac)


def shortest_path(g):
    """-> list of arc ids (start->end), or None when no accepting path."""
    arcs = np.zeros(g.num_nodes + 1, np.int32)
    n = C.c_int()
    rc = liboracle().og_shortest_path(g.ptr, _p(arcs, _i32p), C.byref(n))
    if rc:
        raise OracleError(rc)
    return None if n.value < 0 else arcs[:n.value].copy()


def compose_grad(composed, deltas, n1, n2):
    g1 = np.zeros(max(n1, 1), np.float32)
    g2 = np.zeros(max(n2, 1), np.float32)
    liboracle().og_compose_grad(composed.ptr, _p(_f32(deltas), _f32p), _p(g1, _f32p), _p(g2, _f32p))
    return g1[:n1], g2[:n2]


def ctc_loss(emissions, target, blank=0, arc_sort=True, want_grad=True):
    e = _f32(emissions)
    T, Cn = e.shape
    t = _i32(target)
    loss = C.c_float()
    grad = np.zeros((T, Cn), np.float32) if want_grad else None
    rc = liboracle().og_ctc_loss(
        T, Cn, _p(e, _f32p), _p(t, _i32p), len(t), blank, int(arc_sort),
        C.byref(loss), _p(grad, _f32p))
    if rc:
        raise OracleError(rc)
    return loss.value, grad


def asg_loss(emissions, trans_w, target, want_grad=True):
    e = _f32(emissions)
    T, Cn = e.shape
    tw = _f32(trans_w)
    t = _i32(target)
    loss = C.c_float()
    grad = np.zeros((T, Cn), np.float32) if want_grad else None
    tg = np.zeros(Cn + Cn * Cn, np.float32) if want_grad else None
    rc = liboracle().og_asg_loss(
        T, Cn, _p(e, _f32p), _p(tw, _f32p), _p(t, _i32p), len(t),
        C.byref(loss), _p(grad, _f32p), _p(tg, _f32p))
    if rc:
        raise OracleError(rc)
    return loss.value, grad, tg


def viterbi_dense(emissions, trans_w):
    e = _f32(emissions)
    T, Cn = e.shape
    tw = _f32(trans_w)
    path = np.zeros(T, np.int32)
    score = C.c_float()
    rc = liboracle().og_viterbi_dense(T, Cn, _p(e, _f32p), _p(tw, _f32p), _p(path, _i32p), C.byref(score))
    if rc:
        raise OracleError(rc)
    return path, score.value


def viterbi_ctc(emissions, target, blank=0, arc_sort=True):
    e = _f32(emissions)
    T, Cn = e.shape
    t = _i32(target)
    path = np.zeros(T, np.int32)
    score = C.c_float()
    rc = liboracle().og_viterbi_ctc(
        T, Cn, _p(e, _f32p), _p(t, _i32p), len(t), blank, int(arc_sort),
        _p(path, _i32p), C.byref(score))
    if rc:
        raise OracleError(rc)
    return path, score.value


# ---------------------------------------------------------------------------
# the real reference (oracle/_ref)
# ---------------------------------------------------------------------------

_ref = None


def have_ref():
    return os.path.exists(REF_SO)


def libref():
    global _ref
    if _ref is None:
        R = C.CDLL(REF_SO)
        R.ref_last_error.restype = C.c_char_p
        R.ref_graph_new.argtypes = [C.c_int, _u8p, C.c_int, _i32p, _i32p, _i32p, _i32p, _f32p, C.c_int]
        R.ref_graph_get.argtypes = [C.c_int, _u8p, _i32p, _i32p, _i32p, _i32p, _f32p]
        R.ref_graph_get_adj.argtypes = [C.c_int, _i32p, _i32p, _i32p, _i32p]
        R.ref_graph_set_weights.argtypes = [C.c_int, _f32p]
        R.ref_graph_item.argtypes = [C.c_int, _f32p]
        R.ref_scalar_graph.argtypes = [C.c_float, C.c_int]
        for name in ("ref_ctc_batch", "ref_asg_batch", "ref_viterbi_dense_batch", "ref_viterbi_ctc_batch"):
            getattr(R, name).restype = C.c_double
        R.ref_ctc_batch.argtypes = [
            C.c_int, C.c_int, C.c_int, _f32p, _i32p, _i32p, C.c_int, C.c_int, _f32p, _f32p]
        R.ref_asg_batch.argtypes = [
            C.c_int, C.c_int, C.c_int, _f32p, _f32p, _i32p, _i32p, _f32p, _f32p, _f32p]
        R.ref_viterbi_dense_batch.argtypes = [C.c_int, C.c_int, C.c_int, _f32p, _f32p, _i32p, _f32p]
        R.ref_viterbi_ctc_batch.argtypes = [
            C.c_int, C.c_int, C.c_int, _f32p, _i32p, _i32p, C.c_int, C.c_int, _i32p, _f32p]
        _ref = R
    return _ref


class RefError(Exception):
    def __init__(self, code, msg):
        super().__init__("%s (ref status %d)" % (msg, code))
        self.code = code


def _rc(v):
    if v < 0:
        raise RefError(int(v), libref().ref_last_error().decode())
    return v


class RefGraph:
    """Handle on a gtn::Graph living inside libgtn_ref.so."""

    def __init__(self, h):
        self.h = _rc(h)

    def __del__(self):
        try:
            libref().ref_graph_free(self.h)
        except Exception:
            pass

    @staticmethod
    def from_arrays(flags, src, dst, il, ol, w=None, calc_grad=True):
        flags, src, dst, il, ol, w = _u8(flags), _i32(src), _i32(dst), _i32(il), _i32(ol), _f32(w)
        return RefGraph(libref().ref_graph_new(
            len(flags), _p(flags, _u8p), len(src), _p(src, _i32p), _p(dst, _i32p),
            _p(il, _i32p), _p(ol, _i32p), _p(w, _f32p), int(calc_grad)))

    @staticmethod
    def linear(T, Cn, w=None, calc_grad=True):
        g = RefGraph(libref().ref_linear_graph(T, Cn, int(calc_grad)))
        if w is not None:
            g.set_weights(w)
        return g

    @property
    def num_nodes(self):
        return _rc(libref().ref_graph_num_nodes(self.h))

    @property
    def num_arcs(self):
        return _rc(libref().ref_graph_num_arcs(self.h))

    def set_weights(self, w):
        w = _f32(w).ravel()
        assert w.size == self.num_arcs
        _rc(libref().ref_graph_set_weights(self.h, _p(w, _f32p)))

    def arc_sort(self, olabel=False):
        _rc(libref().ref_graph_arc_sort(self.h, int(olabel)))

    def arrays(self):
        n, a = self.num_nodes, self.num_arcs
        flags = np.zeros(max(n, 1), np.uint8)
        src, dst, il, ol = (np.zeros(max(a, 1), np.int32) for _ in range(4))
        w = np.zeros(max(a, 1), np.float32)
        _rc(libref().ref_graph_get(
            self.h, _p(flags, _u8p), _p(src, _i32p), _p(dst, _i32p), _p(il, _i32p),
            _p(ol, _i32p), _p(w, _f32p)))
        return dict(flags=flags[:n], src=src[:a], dst=dst[:a], ilabel=il[:a], olabel=ol[:a], w=w[:a])

    def adjacency(self):
        n, a = self.num_nodes, self.num_arcs
        ip, ia = np.zeros(n + 1, np.int32), np.zeros(max(a, 1), np.int32)
        op, oa = np.zeros(n + 1, np.int32), np.zeros(max(a, 1), np.int32)
        _rc(libref().ref_graph_get_adj(self.h, _p(ip, _i32p), _p(ia, _i32p), _p(op, _i32p), _p(oa, _i32p)))
        return ip, ia[:a], op, oa[:a]

    def item(self):
        v = C.c_float()
        _rc(libref().ref_graph_item(self.h, C.byref(v)))
        return v.value

    def grad(self):
        return RefGraph(libref().ref_graph_grad(self.h))

    def is_grad_available(self):
        try:
            self.grad()
        except RefError:
            return False
        return True

    def zero_grad(self):
        _rc(libref().ref_graph_zero_grad(self.h))

    def weights(self):
        return self.arrays()["w"]


def ref_op(name, *gs):
    return RefGraph(getattr(libref(), "ref_" + name)(*[g.h for g in gs]))


def ref_backward(g, retain=False):
    _rc(libref().ref_backward(g.h, int(retain)))


def ref_backward_with(g, seed, retain=False):
    _rc(libref().ref_backward_with(g.h, seed.h, int(retain)))


def _handles(gs):
    return (C.c_int * len(gs))(*[g.h for g in gs])


def ref_concat(gs):
    return RefGraph(libref().ref_concat(_handles(gs), len(gs)))


def ref_union(gs):
    return RefGraph(libref().ref_union(_handles(gs), len(gs)))


def ref_closure(g):
    return RefGraph(libref().ref_closure(g.h))


def ref_remove(g, ilabel=-1, olabel=None):
    return RefGraph(libref().ref_remove(g.h, ilabel, ilabel if olabel is None else olabel))


def ref_clone(g, projection=0):
    return RefGraph(libref().ref_clone(g.h, projection))


def ref_equal(a, b):
    return bool(_rc(libref().ref_equal(a.h, b.h)))


def ref_isomorphic(a, b):
    return bool(_rc(libref().ref_isomorphic(a.h, b.h)))


def ref_serialise(g, kind):
    """kind: 0 binary save(), 1 saveTxt(), 2 operator<<, 3 draw()."""
    R = libref()
    R.ref_serialise.restype = C.c_longlong
    R.ref_serialise.argtypes = [C.c_int, C.c_int, C.c_char_p, C.c_longlong]
    n = _rc(R.ref_serialise(g.h, kind, None, 0))
    buf = C.create_string_buffer(max(int(n), 1))
    _rc(R.ref_serialise(g.h, kind, buf, n))
    return buf.raw[:n]


def ref_parse(blob, kind):
    """kind: 0 binary load(), 1 loadTxt()."""
    R = libref()
    R.ref_parse.argtypes = [C.c_int, C.c_char_p, C.c_longlong]
    return RefGraph(R.ref_parse(kind, blob, len(blob)))


def ref_sample(g, seed, max_length=1000):
    R = libref()
    R.ref_sample.argtypes = [C.c_int, C.c_uint, C.c_longlong]
    return RefGraph(R.ref_sample(g.h, seed, max_length))


def ref_rand_equivalent(a, b, seed, num_samples=100):
    R = libref()
    R.ref_rand_equivalent.argtypes = [C.c_int, C.c_int, C.c_uint, C.c_int]
    return bool(_rc(R.ref_rand_equivalent(a.h, b.h, seed, num_samples)))


def _cat_targets(targets):
    lens = np.asarray([len(t) for t in targets], np.int32)
    cat = np.concatenate([np.asarray(t, np.int32) for t in targets]) if len(targets) else np.zeros(0, np.int32)
    return np.ascontiguousarray(cat, np.int32), lens


def ref_ctc_batch(emissions, targets, blank=0, arc_sort=True, want_grad=True):
    """emissions [B,T,C] -> (losses[B], grads[B,T,C] or None, seconds)"""
    e = _f32(emissions)
    B, T, Cn = e.shape
    cat, lens = _cat_targets(targets)
    losses = np.zeros(B, np.float32)
    grads = np.zeros_like(e) if want_grad else None
    sec = _rc(libref().ref_ctc_batch(
        B, T, Cn, _p(e, _f32p), _p(cat, _i32p), _p(lens, _i32p), blank, int(arc_sort),
        _p(losses, _f32p), _p(grads, _f32p)))
    return losses, grads, sec


def ref_asg_batch(emissions, trans_w, targets, want_grad=True):
    e = _f32(emissions)
    B, T, Cn = e.shape
    tw = _f32(trans_w)
    cat, lens = _cat_targets(targets)
    losses = np.zeros(B, np.float32)
    grads = np.zeros_like(e) if want_grad else None
    tg = np.zeros(Cn + Cn * Cn, np.float32) if want_grad else None
    sec = _rc(libref().ref_asg_batch(
        B, T, Cn, _p(e, _f32p), _p(tw, _f32p), _p(cat, _i32p), _p(lens, _i32p),
        _p(losses, _f32p), _p(grads, _f32p), _p(tg, _f32p)))
    return losses, grads, tg, sec


def ref_viterbi_dense_batch(emissions, trans_w):
    e = _f32(emissions)
    B, T, Cn = e.shape
    tw = _f32(trans_w)
    paths = np.zeros((B, T), np.int32)
    scores = np.zeros(B, np.float32)
    sec = _rc(libref().ref_viterbi_dense_batch(
        B, T, Cn, _p(e, _f32p), _p(tw, _f32p), _p(paths, _i32p), _p(scores, _f32p)))
    return paths, scores, sec


def ref_viterbi_ctc_batch(emissions, targets, blank=0, arc_sort=True):
    e = _f32(emissions)
    B, T, Cn = e.shape
    cat, lens = _cat_targets(targets)
    paths = np.zeros((B, T), np.int32)
    scores = np.zeros(B, np.float32)
    sec = _rc(libref().ref_viterbi_ctc_batch(
        B, T, Cn, _p(e, _f32p), _p(cat, _i32p), _p(lens, _i32p), blank, int(arc_sort),
        _p(paths, _i32p), _p(scores, _f32p)))
    return paths, scores, sec
