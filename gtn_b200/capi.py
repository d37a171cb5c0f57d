"""ctypes binding of include/gtn_b200.h (the C-ABI shared library).

This module never computes anything itself: every call goes into
``gtn_b200/lib/libgtn_b200.so`` (hand-written sm_90a CUDA).  If the library is
missing, or no CUDA device is usable, it raises -- there is no CPU fallback.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libgtn_b200.so")

OK = 0
ERR_INVALID_ARGUMENT = 2
ERR_LOGIC = 3
ERR_RUNTIME = 4
ERR_UNSUPPORTED = 5
EPSILON = -1
DENSE_ASG = 0  # gtnb_viterbi_dense_ex graph kinds
DENSE_BIGRAM = 1
DENSE_CTC = 2  # gtnb_beam_decode_async: CTC without transitions
BEAM_RESET = 1  # gtnb_beam_decode_chunk_async's per-row control bits
BEAM_END = 2
F32 = 0  # element types of gtnb_ctc_loss_ex and the *_typed entry points
BF16 = 1
F16 = 2

_f32p = C.POINTER(C.c_float)
_i32p = C.POINTER(C.c_int32)
_u8p = C.POINTER(C.c_uint8)
_vp = C.c_void_p


class GraphView(C.Structure):
    _fields_ = [
        ("num_nodes", C.c_int32), ("num_arcs", C.c_int32),
        ("node_flags", _u8p),
        ("arc_src", _i32p), ("arc_dst", _i32p), ("arc_ilabel", _i32p), ("arc_olabel", _i32p),
        ("weights", _f32p),
        ("in_ptr", _i32p), ("in_arcs", _i32p), ("out_ptr", _i32p), ("out_arcs", _i32p),
        ("start", _i32p), ("num_start", C.c_int32),
        ("accept", _i32p), ("num_accept", C.c_int32),
    ]


# every symbol include/gtn_b200.h declares: (name, restype, argtypes)
SYMBOLS = [
    ("gtnb_version", C.c_int, []),
    ("gtnb_ctx_create", C.c_int, [C.c_int, _vp, C.POINTER(_vp)]),
    ("gtnb_ctx_destroy", None, [_vp]),
    ("gtnb_last_error", C.c_char_p, [_vp]),
    ("gtnb_ctx_synchronize", C.c_int, [_vp]),
    ("gtnb_ctx_stream", _vp, [_vp]),
    ("gtnb_ctx_device", C.c_int, [_vp]),
    ("gtnb_ctx_launch_count", C.c_int64, [_vp]),
    ("gtnb_ctx_set_flag", C.c_int, [_vp, C.c_char_p, C.c_int]),
    ("gtnb_device_alloc", C.c_int, [_vp, C.c_size_t, C.POINTER(_vp)]),
    ("gtnb_device_free", C.c_int, [_vp, _vp]),
    ("gtnb_host_alloc", C.c_int, [_vp, C.c_size_t, C.POINTER(_vp)]),
    ("gtnb_host_free", C.c_int, [_vp, _vp]),
    ("gtnb_memcpy_h2d", C.c_int, [_vp, _vp, _vp, C.c_size_t]),
    ("gtnb_memcpy_d2h", C.c_int, [_vp, _vp, _vp, C.c_size_t]),
    ("gtnb_memset", C.c_int, [_vp, _vp, C.c_int, C.c_size_t]),
    ("gtnb_timer_start", C.c_int, [_vp]),
    ("gtnb_timer_stop", C.c_int, [_vp, _f32p]),
    ("gtnb_flush_l2", C.c_int, [_vp]),
    ("gtnb_profile_enable", C.c_int, [_vp, C.c_int]),
    ("gtnb_profile_read", C.c_char_p, [_vp]),
    ("gtnb_pack", C.c_int, [_vp, C.c_int, C.POINTER(GraphView), C.POINTER(_vp)]),
    ("gtnb_compose_linear", C.c_int,
     [_vp, C.c_int, C.POINTER(GraphView), C.c_int, C.c_int, _i32p, C.c_int, _vp, C.c_int64,
      C.POINTER(_vp)]),
    ("gtnb_compose_graphs", C.c_int,
     [_vp, C.c_int, C.POINTER(GraphView), C.c_int, C.POINTER(GraphView), C.c_int, _i32p, C.POINTER(_vp)]),
    ("gtnb_composed_sizes", C.c_int, [_vp, C.c_int, _i32p, _i32p]),
    ("gtnb_composed_download", C.c_int,
     [_vp, _vp, C.c_int, _u8p, _i32p, _i32p, _i32p, _i32p, _f32p, _i32p, _i32p]),
    ("gtnb_composed_destroy", None, [_vp, _vp]),
    ("gtnb_lattice_destroy", None, [_vp, _vp]),
    ("gtnb_lattice_batch", C.c_int, [_vp]),
    ("gtnb_lattice_sizes", C.c_int, [_vp, _vp, _i32p, _i32p]),
    ("gtnb_lattice_download", C.c_int,
     [_vp, _vp, C.c_int, _u8p, _i32p, _i32p, _i32p, _i32p, _f32p, _i32p, _i32p]),
    ("gtnb_forward", C.c_int, [_vp, _vp, C.c_int, _f32p, _i32p]),
    ("gtnb_backward", C.c_int, [_vp, _vp, C.c_int, _f32p]),
    ("gtnb_lattice_arc_grads", C.c_int, [_vp, _vp, C.c_int, _f32p]),
    ("gtnb_lattice_arc_grads_dev", _vp, [_vp, _vp]),
    ("gtnb_lattice_set_arc_grads", C.c_int, [_vp, _vp, C.c_int, _f32p]),
    ("gtnb_compose_grad", C.c_int, [_vp, _vp, _vp, _vp, C.c_int64]),
    ("gtnb_viterbi_path", C.c_int, [_vp, _vp, C.c_int, _i32p, _i32p, _i32p, _f32p, _i32p, _i32p]),
    ("gtnb_linear_forward", C.c_int,
     [_vp, C.c_int, _i32p, C.c_int, _vp, C.c_int64, C.c_int, _vp, _vp, C.c_int64, _vp, C.c_float]),
    ("gtnb_asg_loss", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _f32p, _i32p, _i32p, _f32p, _vp, C.c_int, _f32p]),
    ("gtnb_viterbi_dense", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, _f32p, _i32p, _f32p]),
    ("gtnb_viterbi_dense_ex", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, C.c_int, _vp, C.c_int, _vp, _vp, C.c_int]),
    ("gtnb_ctc_loss", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, _i32p, _i32p, C.c_int, _f32p, _vp,
      C.c_int]),
    ("gtnb_ctc_loss_ex", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, _i32p, _i32p, C.c_int, _f32p, _vp]),
    ("gtnb_ctc_loss_async", C.c_int,
     [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp, _vp,
      C.c_size_t]),
    ("gtnb_ctc_loss_async_workspace", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    ("gtnb_ngram_ctc_loss_async", C.c_int,
     [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp, _vp,
      _vp, C.c_size_t]),
    ("gtnb_ngram_ctc_loss_async_workspace", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    ("gtnb_asg_loss_async", C.c_int,
     [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
      C.c_size_t]),
    ("gtnb_asg_loss_async_workspace", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    ("gtnb_ctc_align_async", C.c_int,
     [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp, _vp, _vp,
      C.c_size_t]),
    ("gtnb_ngram_ctc_align_async", C.c_int,
     [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp, _vp,
      _vp, C.c_size_t]),
    ("gtnb_asg_align_async", C.c_int,
     [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
      C.c_size_t]),
    ("gtnb_ctc_align_async_workspace", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    ("gtnb_ngram_ctc_align_async_workspace", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    ("gtnb_asg_align_async_workspace", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    ("gtnb_ngram_ctc_loss", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, _vp, C.c_int, _i32p, _i32p, C.c_int, _f32p, _vp,
      C.c_int, _vp, C.c_int]),
    ("gtnb_asg_loss_ex", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, _vp, C.c_int, _i32p, _i32p, _f32p, _vp, C.c_int, _vp,
      C.c_int]),
    ("gtnb_ngram_ctc_loss_typed", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, _vp, _i32p, _i32p, C.c_int, _f32p, _vp, _vp]),
    ("gtnb_asg_loss_typed", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, _vp, _i32p, _i32p, _f32p, _vp, _vp]),
    ("gtnb_viterbi_dense_typed", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, C.c_int, _vp, _vp, _vp]),
    ("gtnb_graph_loss", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, C.POINTER(GraphView), _vp, C.c_int, _f32p, _vp, C.c_int,
      _vp, C.c_int]),
    ("gtnb_graph_transitions_loss", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, C.POINTER(GraphView), _vp, C.c_int, C.c_int, _vp, C.c_int,
      _f32p, _vp, C.c_int, _vp, C.c_int, _vp, C.c_int]),
    ("gtnb_sparse_transitions_loss", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, C.POINTER(GraphView), _vp, C.c_int, C.POINTER(GraphView),
      _vp, C.c_int, _f32p, _vp, C.c_int, _vp, C.c_int, _vp, C.c_int]),
    ("gtnb_graph_viterbi", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, C.POINTER(GraphView), _vp, C.c_int, _vp, _vp, _vp,
      C.c_int]),
    ("gtnb_graph_transitions_viterbi", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, C.POINTER(GraphView), _vp, C.c_int, C.c_int, _vp, C.c_int,
      _vp, _vp, _vp, C.c_int]),
    ("gtnb_viterbi_sparse", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, C.POINTER(GraphView), _vp, C.c_int, _vp, _vp, _vp,
      C.c_int]),
    ("gtnb_sparse_transitions_viterbi", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, C.POINTER(GraphView), _vp, C.c_int, C.POINTER(GraphView),
      _vp, C.c_int, _vp, _vp, _vp, C.c_int]),
    ("gtnb_backoff_transitions_loss", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, C.POINTER(GraphView), _vp, C.c_int, C.POINTER(GraphView),
      _vp, C.c_int, _f32p, _vp, C.c_int, _vp, C.c_int, _vp, C.c_int]),
    ("gtnb_viterbi_backoff", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, C.POINTER(GraphView), _vp, C.c_int, _vp, _vp, _vp,
      C.c_int]),
    ("gtnb_backoff_transitions_viterbi", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _i32p, C.POINTER(GraphView), _vp, C.c_int, C.POINTER(GraphView),
      _vp, C.c_int, _vp, _vp, _vp, C.c_int]),
    ("gtnb_transitions_create", C.c_int, [_vp, C.POINTER(GraphView), C.c_int, C.c_int, C.POINTER(_vp)]),
    ("gtnb_transitions_destroy", None, [_vp, _vp]),
    ("gtnb_viterbi_transitions_async_workspace", C.c_int, [_vp, _vp, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    ("gtnb_viterbi_transitions_async", C.c_int,
     [_vp, _vp, _vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_size_t]),
    ("gtnb_viterbi_dense_async_workspace", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    ("gtnb_viterbi_dense_async", C.c_int,
     [_vp, _vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_size_t]),
    ("gtnb_edit_distance_async_workspace", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    ("gtnb_beam_decode_async_workspace", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    ("gtnb_beam_decode_async", C.c_int,
     [_vp, _vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, C.c_int, _vp, C.c_int, C.c_int, C.c_int, _vp, _vp,
      _vp, _vp, _vp, C.c_size_t]),
    ("gtnb_lm_create", C.c_int, [_vp, C.POINTER(GraphView), C.c_int, C.POINTER(_vp)]),
    ("gtnb_lm_destroy", None, [_vp, _vp]),
    ("gtnb_beam_decode_lm_async_workspace", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    ("gtnb_beam_decode_lm_async", C.c_int,
     [_vp, _vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, C.c_int, _vp, C.c_int, C.c_int, C.c_int, _vp,
      C.c_float, C.c_float, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_size_t]),
    ("gtnb_lexicon_create", C.c_int,
     [_vp, C.c_int, _vp, C.c_int, C.c_int, _vp, _vp, _vp, C.POINTER(GraphView), C.POINTER(_vp)]),
    ("gtnb_lexicon_destroy", None, [_vp, _vp]),
    ("gtnb_beam_decode_lexicon_async", C.c_int,
     [_vp, _vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, C.c_int, _vp, C.c_int, C.c_int, C.c_int, _vp,
      C.c_float, C.c_float, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_size_t]),
    ("gtnb_beam_state_create", C.c_int,
     [_vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp, _vp, C.c_float,
      C.c_float, C.POINTER(_vp)]),
    ("gtnb_beam_state_destroy", None, [_vp, _vp]),
    ("gtnb_beam_decode_chunk_async", C.c_int,
     [_vp, _vp, _vp, C.c_int, _vp, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    ("gtnb_edit_distance_async", C.c_int,
     [_vp, _vp, C.c_int, _vp, C.c_int, _vp, _vp, C.c_int, _vp, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
      C.c_size_t]),
]

_lib = None


def lib():
    """Load the shared library (once) and declare every prototype."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "gtn_b200: %s is missing -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


class GtnbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(msg)
        self.code = code


class GtnbInvalidArgument(GtnbError, ValueError):
    """std::invalid_argument in the reference -> ValueError through pybind11."""


def _raise(code, msg):
    if code == ERR_INVALID_ARGUMENT:
        raise GtnbInvalidArgument(code, msg)
    raise GtnbError(code, msg)


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def make_view(flags, src, dst, ilabel, olabel, weights=None, in_ptr=None, in_arcs=None,
              out_ptr=None, out_arcs=None, start=None, accept=None):
    """Build a GraphView over numpy arrays; returns (view, keepalive list)."""
    keep = []

    def arr(a, dt):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype=dt)
        keep.append(a)
        return a

    flags = arr(flags, np.uint8)
    src, dst = arr(src, np.int32), arr(dst, np.int32)
    ilabel, olabel = arr(ilabel, np.int32), arr(olabel, np.int32)
    weights = arr(weights, np.float32)
    in_ptr, in_arcs = arr(in_ptr, np.int32), arr(in_arcs, np.int32)
    out_ptr, out_arcs = arr(out_ptr, np.int32), arr(out_arcs, np.int32)
    start, accept = arr(start, np.int32), arr(accept, np.int32)
    v = GraphView()
    v.num_nodes = len(flags)
    v.num_arcs = len(src)
    v.node_flags = _p(flags, _u8p)
    v.arc_src, v.arc_dst = _p(src, _i32p), _p(dst, _i32p)
    v.arc_ilabel, v.arc_olabel = _p(ilabel, _i32p), _p(olabel, _i32p)
    v.weights = _p(weights, _f32p)
    v.in_ptr, v.in_arcs = _p(in_ptr, _i32p), _p(in_arcs, _i32p)
    v.out_ptr, v.out_arcs = _p(out_ptr, _i32p), _p(out_arcs, _i32p)
    v.start = _p(start, _i32p)
    v.num_start = 0 if start is None else len(start)
    v.accept = _p(accept, _i32p)
    v.num_accept = 0 if accept is None else len(accept)
    return v, keep


class DeviceBuffer:
    def __init__(self, ctx, nbytes):
        self.ctx = ctx
        self.nbytes = int(nbytes)
        p = _vp()
        ctx._check(lib().gtnb_device_alloc(ctx.h, self.nbytes, C.byref(p)))
        self.ptr = p.value

    def free(self):
        if self.ptr and self.ctx.h:
            lib().gtnb_device_free(self.ctx.h, self.ptr)
        self.ptr = None

    def upload(self, a):
        a = np.ascontiguousarray(a)
        assert a.nbytes <= self.nbytes
        self.ctx._check(lib().gtnb_memcpy_h2d(self.ctx.h, self.ptr, a.ctypes.data, a.nbytes))
        self.ctx.synchronize()
        return self

    def download(self, shape, dtype=np.float32):
        out = np.empty(shape, dtype=dtype)
        assert out.nbytes <= self.nbytes
        self.ctx._check(lib().gtnb_memcpy_d2h(self.ctx.h, out.ctypes.data, self.ptr, out.nbytes))
        self.ctx.synchronize()
        return out

    def zero(self):
        self.ctx._check(lib().gtnb_memset(self.ctx.h, self.ptr, 0, self.nbytes))


class Ctx:
    def __init__(self, device=0, stream=None):
        h = _vp()
        rc = lib().gtnb_ctx_create(device, stream, C.byref(h))
        if rc:
            _raise(rc, lib().gtnb_last_error(None).decode())
        self.h = h.value
        self.device = device

    def close(self):
        if self.h:
            lib().gtnb_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc:
            _raise(rc, lib().gtnb_last_error(self.h).decode())

    def synchronize(self):
        self._check(lib().gtnb_ctx_synchronize(self.h))

    @property
    def launches(self):
        return lib().gtnb_ctx_launch_count(self.h)

    def alloc(self, nbytes):
        return DeviceBuffer(self, nbytes)

    def to_device(self, a):
        a = np.ascontiguousarray(a)
        return DeviceBuffer(self, max(a.nbytes, 16)).upload(a)

    def timer_start(self):
        self._check(lib().gtnb_timer_start(self.h))

    def timer_stop(self):
        ms = C.c_float()
        self._check(lib().gtnb_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def set_flag(self, name, value):
        self._check(lib().gtnb_ctx_set_flag(self.h, name.encode(), int(value)))

    def profile(self, on=True):
        self._check(lib().gtnb_profile_enable(self.h, int(on)))

    def profile_read(self):
        """-> {kernel name: (launches, total_ms)} since the last read."""
        out = {}
        for line in lib().gtnb_profile_read(self.h).decode().splitlines():
            name, n, ms = line.split()
            out[name] = (int(n), float(ms))
        return out

    def flush_l2(self):
        self._check(lib().gtnb_flush_l2(self.h))

    # ---- graph batches -------------------------------------------------
    def pack(self, views):
        arr = (GraphView * max(len(views), 1))(*[v for v, _ in views])
        h = _vp()
        self._check(lib().gtnb_pack(self.h, len(views), arr, C.byref(h)))
        return Lattice(self, h.value, keep=views)

    def compose_linear(self, views, T, Cn, emissions_dev, stride, linear_first=False, B=None):
        B = len(T) if B is None else B
        arr = (GraphView * max(len(views), 1))(*[v for v, _ in views])
        Tn = np.ascontiguousarray(T, dtype=np.int32)
        h = _vp()
        ptr = emissions_dev.ptr if isinstance(emissions_dev, DeviceBuffer) else emissions_dev
        self._check(lib().gtnb_compose_linear(
            self.h, B, arr, len(views), int(linear_first), _p(Tn, _i32p), Cn, ptr, stride,
            C.byref(h)))
        return Lattice(self, h.value, keep=(views, emissions_dev))

    def linear_forward(self, T, Cn, emissions_dev, stride, tropical=False, grad_dev=None,
                       grad_stride=0, delta=1.0):
        B = len(T)
        Tn = np.ascontiguousarray(T, dtype=np.int32)
        scores = self.alloc(4 * max(B, 1))
        self._check(lib().gtnb_linear_forward(
            self.h, B, _p(Tn, _i32p), Cn, emissions_dev.ptr, stride, int(tropical), scores.ptr,
            None if grad_dev is None else grad_dev.ptr, grad_stride, None, float(delta)))
        out = scores.download((B,))
        scores.free()
        return out

    def asg_loss(self, emissions, trans_w, targets, want_grad=True):
        """Host-buffer entry: -> (losses [B], grads [B,T,C] or None, trans_grad [C + C*C] or None)."""
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        tw = np.ascontiguousarray(trans_w, dtype=np.float32)
        cat, lens = _cat_targets(targets)
        losses = np.zeros(B, np.float32)
        grads = np.zeros_like(e) if want_grad else None
        tg = np.zeros(Cn + Cn * Cn, np.float32) if want_grad else None
        self._check(lib().gtnb_asg_loss(
            self.h, B, T, Cn, e.ctypes.data, 0, _p(tw, _f32p), _p(cat, _i32p), _p(lens, _i32p),
            _p(losses, _f32p), None if grads is None else grads.ctypes.data, 0, _p(tg, _f32p)))
        return losses, grads, tg

    def viterbi_dense(self, emissions, trans_w, input_lens=None):
        """Host-buffer entry: emissions [B,T,C], trans_w [C + C*C] -> (paths [B,T], scores [B])."""
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        tw = np.ascontiguousarray(trans_w, dtype=np.float32)
        assert tw.size == Cn + Cn * Cn
        il = None if input_lens is None else np.ascontiguousarray(input_lens, np.int32)
        paths = np.full((B, max(T, 1)), -1, np.int32)
        scores = np.zeros(max(B, 1), np.float32)
        self._check(lib().gtnb_viterbi_dense(
            self.h, B, T, Cn, e.ctypes.data, 0, _p(il, _i32p), _p(tw, _f32p), _p(paths, _i32p),
            _p(scores, _f32p)))
        return paths[:, :T], scores[:B]

    def viterbi_dense_ex(self, emissions, trans_w, kind=DENSE_ASG, input_lens=None):
        """Host-buffer entry of gtnb_viterbi_dense_ex: emissions [B,T,C], trans_w [C + C*C] (DENSE_ASG) or [C*C]
        (DENSE_BIGRAM) -> (paths [B,T] int32, -1 beyond T_b; scores [B])."""
        return self._viterbi_dense_ex(False, emissions, trans_w, kind, input_lens)

    def viterbi_dense_ex_dev(self, emissions, trans_w, kind=DENSE_ASG, input_lens=None):
        """Device-buffer entry: emissions and trans_w uploaded once, gtnb_viterbi_dense_ex on device pointers
        (paths and scores in HBM), downloaded afterwards -> (paths, scores)."""
        return self._viterbi_dense_ex(True, emissions, trans_w, kind, input_lens)

    def _viterbi_dense_ex(self, dev, emissions, trans_w, kind, input_lens):
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        tw = np.ascontiguousarray(trans_w, dtype=np.float32).ravel()
        assert tw.size == (Cn * Cn if kind == DENSE_BIGRAM else Cn + Cn * Cn)
        il = None if input_lens is None else np.ascontiguousarray(input_lens, np.int32)
        paths = np.full((max(B, 1), max(T, 1)), -7, np.int32)  # every entry is written
        scores = np.full(max(B, 1), np.nan, np.float32)
        with _Placed(self, dev) as p:
            self._check(lib().gtnb_viterbi_dense_ex(
                self.h, B, T, Cn, p.inp(e), p.flag, _p(il, _i32p), int(kind), p.inp(tw), p.flag, p.out(paths),
                p.out(scores), p.flag))
        return paths.ravel()[:B * T].reshape(B, T), scores[:B]

    def ctc_loss(self, emissions, targets, blank=0, want_grad=True, input_lens=None):
        """Host-buffer entry point: emissions [B,T,C] float32 numpy -> (losses, grads)."""
        return self._ctc_loss(False, emissions, targets, blank, want_grad, input_lens)

    def ctc_loss_dev(self, emissions, targets, blank=0, input_lens=None):
        """Device-buffer entry point: uploads once, runs gtnb_ctc_loss on device pointers (emissions
        in HBM in, gradients in HBM out), downloads the gradients afterwards -> (losses, grads)."""
        return self._ctc_loss(True, emissions, targets, blank, True, input_lens)

    def _ctc_loss(self, dev, emissions, targets, blank, want_grad, input_lens):
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        cat, lens = _cat_targets(targets)
        il = None if input_lens is None else np.ascontiguousarray(input_lens, np.int32)
        losses = np.zeros(B, np.float32)
        grads = np.zeros_like(e) if want_grad else None
        with _Placed(self, dev) as p:
            self._check(lib().gtnb_ctc_loss(
                self.h, B, T, Cn, p.inp(e), p.flag, _p(il, _i32p), _p(cat, _i32p), _p(lens, _i32p),
                blank, _p(losses, _f32p), p.out(grads), p.flag))
        return losses, grads


    def ngram_ctc_loss(self, emissions, trans_w, targets, blank=0, want_grad=True, input_lens=None):
        """Host-buffer entry of gtnb_ngram_ctc_loss: emissions [B,T,C], trans_w [C*C] (row = destination label)
        -> (losses [B], grads [B,T,C] or None, trans_grad [C*C] or None)."""
        return self._ngram_ctc_loss(False, emissions, trans_w, targets, blank, want_grad, input_lens)

    def ngram_ctc_loss_dev(self, emissions, trans_w, targets, blank=0, input_lens=None):
        """Device-buffer entry: emissions and W uploaded once, gtnb_ngram_ctc_loss on device pointers (gradients
        in HBM), downloaded afterwards -> (losses, grads, trans_grad)."""
        return self._ngram_ctc_loss(True, emissions, trans_w, targets, blank, True, input_lens)

    def _ngram_ctc_loss(self, dev, emissions, trans_w, targets, blank, want_grad, input_lens):
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        tw = np.ascontiguousarray(trans_w, dtype=np.float32).ravel()
        assert tw.size == Cn * Cn
        cat, lens = _cat_targets(targets)
        il = None if input_lens is None else np.ascontiguousarray(input_lens, np.int32)
        losses = np.zeros(B, np.float32)
        grads = np.full_like(e, np.nan) if want_grad else None  # every row is written
        tg = np.zeros(Cn * Cn, np.float32) if want_grad else None
        with _Placed(self, dev) as p:
            self._check(lib().gtnb_ngram_ctc_loss(
                self.h, B, T, Cn, p.inp(e), p.flag, _p(il, _i32p), p.inp(tw), p.flag, _p(cat, _i32p),
                _p(lens, _i32p), int(blank), _p(losses, _f32p), p.out(grads), p.flag, p.out(tg), p.flag))
        return losses, grads, tg

    def asg_loss_ex(self, emissions, trans_w, targets, want_grad=True, input_lens=None):
        """Host-buffer entry of gtnb_asg_loss_ex: emissions [B,T,C], trans_w [C + C*C] (start weights, then the
        C x C matrix, row = destination label), input_lens [B] or None
        -> (losses [B], grads [B,T,C] or None, trans_grad [C + C*C] or None)."""
        return self._asg_loss_ex(False, emissions, trans_w, targets, want_grad, input_lens)

    def asg_loss_ex_dev(self, emissions, trans_w, targets, input_lens=None):
        """Device-buffer entry: emissions and trans_w uploaded once, gtnb_asg_loss_ex on device pointers (gradients
        in HBM), downloaded afterwards -> (losses, grads, trans_grad)."""
        return self._asg_loss_ex(True, emissions, trans_w, targets, True, input_lens)

    def _asg_loss_ex(self, dev, emissions, trans_w, targets, want_grad, input_lens):
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        tw = np.ascontiguousarray(trans_w, dtype=np.float32).ravel()
        assert tw.size == Cn + Cn * Cn
        cat, lens = _cat_targets(targets)
        il = None if input_lens is None else np.ascontiguousarray(input_lens, np.int32)
        losses = np.zeros(B, np.float32)
        grads = np.full_like(e, np.nan) if want_grad else None  # every row is written
        tg = np.zeros(Cn + Cn * Cn, np.float32) if want_grad else None
        with _Placed(self, dev) as p:
            self._check(lib().gtnb_asg_loss_ex(
                self.h, B, T, Cn, p.inp(e), p.flag, _p(il, _i32p), p.inp(tw), p.flag, _p(cat, _i32p),
                _p(lens, _i32p), _p(losses, _f32p), p.out(grads), p.flag, p.out(tg), p.flag))
        return losses, grads, tg

    def graph_loss(self, emissions, views, want_grad=True, input_lens=None, arc_weights=None):
        """Host-buffer entry of gtnb_graph_loss: emissions [B,T,C], views: B (view, keepalive) pairs from make_view,
        arc_weights [sum A_b] or None -> (losses [B], grads [B,T,C] or None, arc_grads [sum A_b] or None)."""
        return self._graph_loss(False, emissions, views, want_grad, input_lens, arc_weights)

    def graph_loss_dev(self, emissions, views, input_lens=None, arc_weights=None):
        """Device-buffer entry: emissions (and arc_weights, when given) uploaded once, gtnb_graph_loss on device
        pointers (gradients in HBM), downloaded afterwards -> (losses, grads, arc_grads)."""
        return self._graph_loss(True, emissions, views, True, input_lens, arc_weights)

    def _graph_loss(self, dev, emissions, views, want_grad, input_lens, arc_weights):
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        arr, n_arcs, aw = _graph_batch(views, B, arc_weights)
        il = None if input_lens is None else np.ascontiguousarray(input_lens, np.int32)
        losses = np.zeros(B, np.float32)
        grads = np.full_like(e, np.nan) if want_grad else None  # every row is written
        ag = np.full(max(n_arcs, 1), np.nan, np.float32) if want_grad else None  # written, not accumulated
        with _Placed(self, dev) as p:
            self._check(lib().gtnb_graph_loss(
                self.h, B, T, Cn, p.inp(e), p.flag, _p(il, _i32p), arr, p.inp(aw), p.flag, _p(losses, _f32p),
                p.out(grads), p.flag, p.out(ag), p.flag))
        return losses, grads, None if ag is None else ag[:n_arcs]

    def graph_viterbi(self, emissions, views, input_lens=None, arc_weights=None):
        """Host-buffer entry of gtnb_graph_viterbi: emissions [B,T,C], views: B (view, keepalive) pairs from make_view,
        arc_weights [sum A_b] or None -> (paths [B,T] int32, scores [B], arcs [B,T] int32)."""
        return self._graph_viterbi(False, emissions, views, input_lens, arc_weights)

    def graph_viterbi_dev(self, emissions, views, input_lens=None, arc_weights=None):
        """Device-buffer entry: emissions (and arc_weights, when given) uploaded once, gtnb_graph_viterbi on device
        pointers (outputs in HBM), downloaded afterwards -> (paths, scores, arcs)."""
        return self._graph_viterbi(True, emissions, views, input_lens, arc_weights)

    def _graph_viterbi(self, dev, emissions, views, input_lens, arc_weights):
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        arr, _, aw = _graph_batch(views, B, arc_weights)
        il = None if input_lens is None else np.ascontiguousarray(input_lens, np.int32)
        out = _viterbi_outputs(B, T)
        with _Placed(self, dev) as p:
            self._check(lib().gtnb_graph_viterbi(
                self.h, B, T, Cn, p.inp(e), p.flag, _p(il, _i32p), arr, p.inp(aw), p.flag, *map(p.out, out),
                p.flag))
        return _viterbi_results(out, B, T)

    def graph_transitions_loss(self, emissions, views, trans_w, kind=DENSE_ASG, want_grad=True, input_lens=None,
                               arc_weights=None):
        """Host-buffer entry of gtnb_graph_transitions_loss: emissions [B,T,C], views: B (view, keepalive) pairs from
        make_view, trans_w [C + C*C] (DENSE_ASG) or [C*C] (DENSE_BIGRAM), arc_weights [sum A_b] or None
        -> (losses [B], grads [B,T,C] or None, arc_grads [sum A_b] or None, trans_grad or None)."""
        return self._graph_transitions_loss(False, emissions, views, trans_w, kind, want_grad, input_lens, arc_weights)

    def graph_transitions_loss_dev(self, emissions, views, trans_w, kind=DENSE_ASG, input_lens=None,
                                   arc_weights=None):
        """Device-buffer entry: emissions, trans_w (and arc_weights, when given) uploaded once,
        gtnb_graph_transitions_loss on device pointers (gradients in HBM), downloaded afterwards
        -> (losses, grads, arc_grads, trans_grad)."""
        return self._graph_transitions_loss(True, emissions, views, trans_w, kind, True, input_lens, arc_weights)

    def _graph_transitions_loss(self, dev, emissions, views, trans_w, kind, want_grad, input_lens, arc_weights):
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        arr, n_arcs, aw = _graph_batch(views, B, arc_weights)
        tw = np.ascontiguousarray(trans_w, dtype=np.float32).ravel()
        il = None if input_lens is None else np.ascontiguousarray(input_lens, np.int32)
        losses = np.zeros(B, np.float32)
        grads = np.full_like(e, np.nan) if want_grad else None  # every row is written
        ag = np.full(max(n_arcs, 1), np.nan, np.float32) if want_grad else None  # written, not accumulated
        tg = np.full(tw.size, np.nan, np.float32) if want_grad else None
        with _Placed(self, dev) as p:
            self._check(lib().gtnb_graph_transitions_loss(
                self.h, B, T, Cn, p.inp(e), p.flag, _p(il, _i32p), arr, p.inp(aw), p.flag, kind, p.inp(tw), p.flag,
                _p(losses, _f32p), p.out(grads), p.flag, p.out(ag), p.flag, p.out(tg), p.flag))
        return losses, grads, None if ag is None else ag[:n_arcs], tg

    def sparse_transitions_loss(self, emissions, views, transitions, trans_w, want_grad=True, input_lens=None,
                                arc_weights=None):
        """Host-buffer entry of gtnb_sparse_transitions_loss: emissions [B,T,C], views: B (view, keepalive) pairs from
        make_view, transitions: G's (view, keepalive) pair (an acceptor; its weights are ignored), trans_w
        [G.num_arcs], arc_weights [sum A_b] or None
        -> (losses [B], grads [B,T,C] or None, arc_grads [sum A_b] or None, trans_grad [G.num_arcs] or None)."""
        return self._sparse_transitions_loss(False, emissions, views, transitions, trans_w, want_grad, input_lens,
                                             arc_weights)

    def sparse_transitions_loss_dev(self, emissions, views, transitions, trans_w, input_lens=None, arc_weights=None):
        """Device-buffer entry: emissions, trans_w (and arc_weights, when given) uploaded once,
        gtnb_sparse_transitions_loss on device pointers (gradients in HBM), downloaded afterwards
        -> (losses, grads, arc_grads, trans_grad)."""
        return self._sparse_transitions_loss(True, emissions, views, transitions, trans_w, True, input_lens,
                                             arc_weights)

    def backoff_transitions_loss(self, emissions, views, transitions, trans_w, want_grad=True, input_lens=None,
                                 arc_weights=None):
        """Host-buffer entry of gtnb_backoff_transitions_loss: sparse_transitions_loss's arguments and results, with
        epsilon arcs (backoff arcs) allowed in the transition graph."""
        return self._sparse_transitions_loss(False, emissions, views, transitions, trans_w, want_grad, input_lens,
                                             arc_weights, "gtnb_backoff_transitions_loss")

    def backoff_transitions_loss_dev(self, emissions, views, transitions, trans_w, input_lens=None, arc_weights=None):
        """Device-buffer entry of gtnb_backoff_transitions_loss, as sparse_transitions_loss_dev
        -> (losses, grads, arc_grads, trans_grad)."""
        return self._sparse_transitions_loss(True, emissions, views, transitions, trans_w, True, input_lens,
                                             arc_weights, "gtnb_backoff_transitions_loss")

    def _sparse_transitions_loss(self, dev, emissions, views, transitions, trans_w, want_grad, input_lens,
                                 arc_weights, fn="gtnb_sparse_transitions_loss"):
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        arr, n_arcs, aw = _graph_batch(views, B, arc_weights)
        gv = transitions[0]
        tw = np.ascontiguousarray(trans_w, dtype=np.float32).ravel()
        assert tw.size == gv.num_arcs
        # an empty G: no host pointer at all, or a device buffer that is never read
        tw_arg = tw if tw.size else np.zeros(1, np.float32) if dev else None
        il = None if input_lens is None else np.ascontiguousarray(input_lens, np.int32)
        losses = np.zeros(B, np.float32)
        grads = np.full_like(e, np.nan) if want_grad else None  # every row is written
        ag = np.full(max(n_arcs, 1), np.nan, np.float32) if want_grad else None  # written, not accumulated
        tg = np.full(max(tw.size, 1), np.nan, np.float32) if want_grad else None
        with _Placed(self, dev) as p:
            self._check(getattr(lib(), fn)(
                self.h, B, T, Cn, p.inp(e), p.flag, _p(il, _i32p), arr, p.inp(aw), p.flag, C.byref(gv), p.inp(tw_arg),
                p.flag, _p(losses, _f32p), p.out(grads), p.flag, p.out(ag), p.flag, p.out(tg), p.flag))
        return (losses, grads, None if ag is None else ag[:n_arcs], None if tg is None else tg[:tw.size])

    def graph_transitions_viterbi(self, emissions, views, trans_w, kind=DENSE_ASG, input_lens=None, arc_weights=None):
        """Host-buffer entry of gtnb_graph_transitions_viterbi: emissions [B,T,C], views: B (view, keepalive) pairs
        from make_view, trans_w [C + C*C] (DENSE_ASG) or [C*C] (DENSE_BIGRAM), arc_weights [sum A_b] or None
        -> (paths [B,T] int32, scores [B], arcs [B,T] int32)."""
        return self._graph_transitions_viterbi(False, emissions, views, trans_w, kind, input_lens, arc_weights, False)

    def graph_transitions_viterbi_dev(self, emissions, views, trans_w, kind=DENSE_ASG, input_lens=None,
                                      arc_weights=None, trans_on_device=True):
        """Device-buffer entry: emissions (and arc_weights, when given; trans_w unless trans_on_device is False)
        uploaded once, gtnb_graph_transitions_viterbi on device pointers (outputs in HBM), downloaded afterwards
        -> (paths, scores, arcs)."""
        return self._graph_transitions_viterbi(True, emissions, views, trans_w, kind, input_lens, arc_weights,
                                               bool(trans_on_device))

    def _graph_transitions_viterbi(self, dev, emissions, views, trans_w, kind, input_lens, arc_weights,
                                   trans_on_device):
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        arr, _, aw = _graph_batch(views, B, arc_weights)
        tw = np.ascontiguousarray(trans_w, dtype=np.float32).ravel()
        il = None if input_lens is None else np.ascontiguousarray(input_lens, np.int32)
        out = _viterbi_outputs(B, T)
        with _Placed(self, dev) as p:
            self._check(lib().gtnb_graph_transitions_viterbi(
                self.h, B, T, Cn, p.inp(e), p.flag, _p(il, _i32p), arr, p.inp(aw), p.flag, kind,
                p.inp(tw, trans_on_device), int(trans_on_device), *map(p.out, out), p.flag))
        return _viterbi_results(out, B, T)

    def viterbi_sparse(self, emissions, transitions, trans_w, input_lens=None):
        """Host-buffer entry of gtnb_viterbi_sparse: emissions [B,T,C], transitions: G's (view, keepalive) pair (an
        acceptor; its weights are ignored), trans_w [G.num_arcs] -> (paths [B,T] int32, scores [B], arcs [B,T] int32:
        G's arc per frame)."""
        return self._viterbi_sparse(False, emissions, transitions, trans_w, input_lens, False)

    def viterbi_sparse_dev(self, emissions, transitions, trans_w, input_lens=None, trans_on_device=True):
        """Device-buffer entry: emissions (and trans_w unless trans_on_device is False) uploaded once,
        gtnb_viterbi_sparse on device pointers (outputs in HBM), downloaded afterwards -> (paths, scores, arcs)."""
        return self._viterbi_sparse(True, emissions, transitions, trans_w, input_lens, bool(trans_on_device))

    def viterbi_backoff(self, emissions, transitions, trans_w, input_lens=None):
        """Host-buffer entry of gtnb_viterbi_backoff: viterbi_sparse's arguments and results, with epsilon arcs
        (backoff arcs) allowed in the transition graph; arcs holds the emitting G arc of every frame."""
        return self._viterbi_sparse(False, emissions, transitions, trans_w, input_lens, False, "gtnb_viterbi_backoff")

    def viterbi_backoff_dev(self, emissions, transitions, trans_w, input_lens=None, trans_on_device=True):
        """Device-buffer entry of gtnb_viterbi_backoff, as viterbi_sparse_dev -> (paths, scores, arcs)."""
        return self._viterbi_sparse(True, emissions, transitions, trans_w, input_lens, bool(trans_on_device),
                                    "gtnb_viterbi_backoff")

    def _viterbi_sparse(self, dev, emissions, transitions, trans_w, input_lens, trans_on_device,
                        fn="gtnb_viterbi_sparse"):
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        gv = transitions[0]
        tw = _sparse_trans_w(gv, trans_w)
        il = None if input_lens is None else np.ascontiguousarray(input_lens, np.int32)
        out = _viterbi_outputs(B, T)
        with _Placed(self, dev) as p:
            self._check(getattr(lib(), fn)(
                self.h, B, T, Cn, p.inp(e), p.flag, _p(il, _i32p), C.byref(gv), p.inp(tw, trans_on_device),
                int(trans_on_device), *map(p.out, out), p.flag))
        return _viterbi_results(out, B, T)

    def sparse_transitions_viterbi(self, emissions, views, transitions, trans_w, input_lens=None, arc_weights=None):
        """Host-buffer entry of gtnb_sparse_transitions_viterbi: emissions [B,T,C], views: B (view, keepalive) pairs
        from make_view, transitions: G's (view, keepalive) pair, trans_w [G.num_arcs], arc_weights [sum A_b] or None
        -> (paths [B,T] int32, scores [B], arcs [B,T] int32: A_b's arc per frame)."""
        return self._sparse_transitions_viterbi(False, emissions, views, transitions, trans_w, input_lens, arc_weights,
                                                False)

    def sparse_transitions_viterbi_dev(self, emissions, views, transitions, trans_w, input_lens=None,
                                       arc_weights=None, trans_on_device=True):
        """Device-buffer entry: emissions (and arc_weights, when given; trans_w unless trans_on_device is False)
        uploaded once, gtnb_sparse_transitions_viterbi on device pointers (outputs in HBM), downloaded afterwards
        -> (paths, scores, arcs)."""
        return self._sparse_transitions_viterbi(True, emissions, views, transitions, trans_w, input_lens, arc_weights,
                                                bool(trans_on_device))

    def backoff_transitions_viterbi(self, emissions, views, transitions, trans_w, input_lens=None, arc_weights=None):
        """Host-buffer entry of gtnb_backoff_transitions_viterbi: sparse_transitions_viterbi's arguments and results,
        with epsilon arcs (backoff arcs) allowed in the transition graph; arcs holds A_b's emitting arc of every
        frame."""
        return self._sparse_transitions_viterbi(False, emissions, views, transitions, trans_w, input_lens, arc_weights,
                                                False, "gtnb_backoff_transitions_viterbi")

    def backoff_transitions_viterbi_dev(self, emissions, views, transitions, trans_w, input_lens=None,
                                        arc_weights=None, trans_on_device=True):
        """Device-buffer entry of gtnb_backoff_transitions_viterbi, as sparse_transitions_viterbi_dev
        -> (paths, scores, arcs)."""
        return self._sparse_transitions_viterbi(True, emissions, views, transitions, trans_w, input_lens, arc_weights,
                                                bool(trans_on_device), "gtnb_backoff_transitions_viterbi")

    def _sparse_transitions_viterbi(self, dev, emissions, views, transitions, trans_w, input_lens, arc_weights,
                                    trans_on_device, fn="gtnb_sparse_transitions_viterbi"):
        e = np.ascontiguousarray(emissions, dtype=np.float32)
        B, T, Cn = e.shape
        arr, _, aw = _graph_batch(views, B, arc_weights)
        gv = transitions[0]
        tw = _sparse_trans_w(gv, trans_w)
        il = None if input_lens is None else np.ascontiguousarray(input_lens, np.int32)
        out = _viterbi_outputs(B, T)
        with _Placed(self, dev) as p:
            self._check(getattr(lib(), fn)(
                self.h, B, T, Cn, p.inp(e), p.flag, _p(il, _i32p), arr, p.inp(aw), p.flag, C.byref(gv),
                p.inp(tw, trans_on_device), int(trans_on_device), *map(p.out, out), p.flag))
        return _viterbi_results(out, B, T)


class Lattice:
    def __init__(self, ctx, h, keep=None):
        self.ctx = ctx
        self.h = h
        self._keep = keep
        self.B = lib().gtnb_lattice_batch(h)

    def free(self):
        if self.h and self.ctx.h:
            lib().gtnb_lattice_destroy(self.ctx.h, self.h)
        self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def sizes(self):
        n = np.zeros(max(self.B, 1), np.int32)
        a = np.zeros(max(self.B, 1), np.int32)
        self.ctx._check(lib().gtnb_lattice_sizes(self.ctx.h, self.h, _p(n, _i32p), _p(a, _i32p)))
        return n[:self.B], a[:self.B]

    def download(self, b):
        nn, na = self.sizes()
        N, A = int(nn[b]), int(na[b])
        flags = np.zeros(max(N, 1), np.uint8)
        src, dst, il, ol, gg, gl = (np.zeros(max(A, 1), np.int32) for _ in range(6))
        w = np.zeros(max(A, 1), np.float32)
        self.ctx._check(lib().gtnb_lattice_download(
            self.ctx.h, self.h, b, _p(flags, _u8p), _p(src, _i32p), _p(dst, _i32p), _p(il, _i32p),
            _p(ol, _i32p), _p(w, _f32p), _p(gg, _i32p), _p(gl, _i32p)))
        return dict(flags=flags[:N], src=src[:A], dst=dst[:A], ilabel=il[:A], olabel=ol[:A],
                    w=w[:A], gi_graph=gg[:A], gi_linear=gl[:A])

    def forward(self, tropical=False, want_status=False):
        scores = np.zeros(max(self.B, 1), np.float32)
        status = np.zeros(max(self.B, 1), np.int32)
        rc = lib().gtnb_forward(self.ctx.h, self.h, int(tropical), _p(scores, _f32p), _p(status, _i32p))
        if want_status:
            if rc not in (OK, ERR_INVALID_ARGUMENT):
                self.ctx._check(rc)
            return scores[:self.B], status[:self.B]
        self.ctx._check(rc)
        return scores[:self.B]

    def backward(self, tropical=False, deltas=None):
        d = None if deltas is None else np.ascontiguousarray(deltas, np.float32)
        self.ctx._check(lib().gtnb_backward(self.ctx.h, self.h, int(tropical), _p(d, _f32p)))

    def arc_grads(self, b, num_arcs):
        out = np.zeros(max(num_arcs, 1), np.float32)
        self.ctx._check(lib().gtnb_lattice_arc_grads(self.ctx.h, self.h, b, _p(out, _f32p)))
        return out[:num_arcs]

    def set_arc_grads(self, b, grads):
        g = np.ascontiguousarray(grads, np.float32)
        self.ctx._check(lib().gtnb_lattice_set_arc_grads(self.ctx.h, self.h, b, _p(g, _f32p)))

    def arc_grads_dev(self):
        """device address of every entry's arc gradients, in download order (0: error or no backward yet)"""
        return lib().gtnb_lattice_arc_grads_dev(self.ctx.h, self.h) or 0

    def compose_grad(self, grad_graph_dev=None, grad_emissions_dev=None, grad_stride=0):
        self.ctx._check(lib().gtnb_compose_grad(
            self.ctx.h, self.h,
            None if grad_graph_dev is None else grad_graph_dev.ptr,
            None if grad_emissions_dev is None else grad_emissions_dev.ptr, grad_stride))

    def viterbi_path(self, max_len, want_status=False):
        B = self.B
        arcs = np.full((max(B, 1), max(max_len, 1)), -1, np.int32)
        il = np.full_like(arcs, -1)
        ol = np.full_like(arcs, -1)
        lens = np.zeros(max(B, 1), np.int32)
        status = np.zeros(max(B, 1), np.int32)
        pw = np.zeros(arcs.shape, np.float32)
        rc = lib().gtnb_viterbi_path(
            self.ctx.h, self.h, max_len, _p(arcs, _i32p), _p(il, _i32p), _p(ol, _i32p),
            _p(pw, _f32p), _p(lens, _i32p), _p(status, _i32p))
        if want_status:
            if rc not in (OK, ERR_INVALID_ARGUMENT):
                self.ctx._check(rc)
        else:
            self.ctx._check(rc)
        out = dict(arcs=arcs[:B], ilabels=il[:B], olabels=ol[:B], lens=lens[:B], weights=pw[:B])
        return (out, status[:B]) if want_status else out


class _Placed:
    """Where the buffers of one call live.  On the host a buffer is passed as a pointer into its numpy array.  On the
    device (dev) it is uploaded and passed as a device pointer; an output is downloaded back into its array when the
    `with` block ends without an error.  Every device buffer is freed when the block ends, on every path."""

    def __init__(self, ctx, dev):
        self.ctx, self.dev, self.flag = ctx, bool(dev), int(bool(dev))
        self._bufs, self._outs = [], []

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc, tb):
        try:
            if exc_type is None:
                for buf, a in self._outs:
                    a[...] = buf.download(a.shape, a.dtype)
        finally:
            for buf in self._bufs:
                buf.free()

    def inp(self, a, dev=None):
        """pointer to a (None: None); dev overrides where this one buffer lives"""
        if a is None:
            return None
        if not (self.dev if dev is None else dev):
            return a.ctypes.data
        buf = self.ctx.to_device(a)
        self._bufs.append(buf)
        return buf.ptr

    def out(self, a):
        """pointer to the output a, which holds its fill (the value of every entry the call fails to write)"""
        ptr = self.inp(a)
        if a is not None and self.dev:
            self._outs.append((self._bufs[-1], a))
        return ptr


def _graph_batch(views, B, arc_weights):
    """-> (GraphView array of the B (view, keepalive) pairs, their arc count, arc_weights as float32 or None)"""
    assert len(views) == B
    arr = (GraphView * max(B, 1))(*[v for v, _ in views])
    n_arcs = sum(v.num_arcs for v, _ in views)
    aw = None if arc_weights is None else np.ascontiguousarray(arc_weights, np.float32).ravel()
    assert aw is None or aw.size == n_arcs
    return arr, n_arcs, aw


def _viterbi_outputs(B, T):
    """paths, arcs and scores of a graph Viterbi call, filled so that an entry left unwritten shows"""
    fill = np.full((max(B, 1), max(T, 1)), -7, np.int32)
    return fill, fill.copy(), np.full(max(B, 1), np.nan, np.float32)


def _viterbi_results(out, B, T):
    """-> (paths [B,T], scores [B], arcs [B,T])"""
    paths, arcs, scores = out
    return paths.ravel()[:B * T].reshape(B, T), scores[:B], arcs.ravel()[:B * T].reshape(B, T)


def _sparse_trans_w(gv, trans_w):
    """trans_w as float32 for a G of gv.num_arcs arcs (None stays None, for the argument checks); an empty G gets a
    one-element buffer that is never read"""
    if trans_w is None:
        return None
    tw = np.ascontiguousarray(trans_w, dtype=np.float32).ravel()
    assert tw.size == gv.num_arcs
    return tw if tw.size else np.zeros(1, np.float32)


def _cat_targets(targets):
    lens = np.asarray([len(t) for t in targets], np.int32)
    cat = np.concatenate([np.asarray(t, np.int32) for t in targets]) if len(targets) else np.zeros(0, np.int32)
    return np.ascontiguousarray(cat, np.int32), lens
