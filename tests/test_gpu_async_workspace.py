"""The workspace rule every asynchronous call shares, call by call: the sized workspace runs; a NULL workspace has 0
bytes, so with B > 0 the call fails with GTNB_ERR_INVALID_ARGUMENT (workspace too small) and with B = 0, where every
query gives 0 bytes, it succeeds; a workspace off 256-byte alignment is GTNB_ERR_INVALID_ARGUMENT."""
import ctypes as C_

import pytest
import torch

from gtn_b200 import capi
from tests import sparse_trans_oracle as st

pytestmark = pytest.mark.gpu

L = capi.lib
T, Cn, S, CG = 20, 16, 5, 8  # CG: the labels of the prepared trigram G


def inputs(B, seed=0):
    """device emissions [B, T, Cn], targets [B, S], target lengths, transitions (ASG's C + C*C) and the trigram G's
    weights of a seeded batch; at least one row, so that B = 0 still passes non-NULL buffers"""
    g = torch.Generator().manual_seed(seed)
    rows = max(B, 1)
    e = torch.randn(rows, T, Cn, generator=g).log_softmax(-1).cuda()
    tg = torch.randint(1, Cn, (rows, S), generator=g, dtype=torch.int32).cuda()
    lens = torch.randint(0, S + 1, (rows,), generator=g, dtype=torch.int32).cuda()
    w = (0.1 * torch.randn(Cn + Cn * Cn, generator=g)).cuda()
    wg = (0.1 * torch.randn(CG * CG * CG, generator=g)).cuda()  # the trigram G's arc weights
    return e, tg, lens, w, wg


def out(*shape, dtype=torch.float32):
    return torch.full(shape, -7, dtype=dtype, device="cuda")


def ptrs(ts):
    return [None if t is None else t.data_ptr() for t in ts]


def calls(ctx, G, B):
    """{name: (sizing query, its arguments, enqueue(workspace, bytes) -> rc, output tensors)} for a batch of B"""
    e, tg, lens, w, wg = inputs(B)
    r = max(B, 1)
    i32 = torch.int32
    h = ctx.h
    loss = [out(r), out(r, dtype=i32), out(r, T, Cn)]
    trellis = loss + [out(Cn + Cn * Cn)]
    align = [out(r, T, dtype=i32), out(r, T, dtype=i32), out(r), out(r, dtype=i32)]
    dense = [out(r, T, dtype=i32), out(r), out(r, dtype=i32)]
    beam = [out(r, 2, T, dtype=i32), out(r, 2, dtype=i32), out(r, 2), out(r, dtype=i32)]
    eg = e[..., :CG].contiguous()
    trans = [out(r, T, dtype=i32), out(r, T, dtype=i32), out(r), out(r, dtype=i32)]
    edit = [out(r, dtype=i32), out(r, 3, dtype=i32), out(r, 2, dtype=i32), out(r, dtype=i32), out(r, S, dtype=i32),
            out(r, S, dtype=i32)]
    hyp, ref_lens = tg.flip(1).contiguous(), lens.flip(0).contiguous()
    a = (B, T, Cn, S, e.data_ptr(), capi.F32, None)
    return {
        "ctc_loss": ("gtnb_ctc_loss_async_workspace", (B, T, Cn, S, capi.F32, 1), lambda ws, n: L().gtnb_ctc_loss_async(
            h, None, *a, tg.data_ptr(), lens.data_ptr(), 0, *ptrs(loss), ws, n), loss),
        "ngram_ctc_loss": ("gtnb_ngram_ctc_loss_async_workspace", (B, T, Cn, S, capi.F32, 1),
                           lambda ws, n: L().gtnb_ngram_ctc_loss_async(
                               h, None, *a, w[Cn:].data_ptr(), tg.data_ptr(), lens.data_ptr(), 0, *ptrs(trellis[:3]),
                               trellis[3][Cn:].data_ptr(), ws, n), trellis),
        "asg_loss": ("gtnb_asg_loss_async_workspace", (B, T, Cn, S, capi.F32, 1), lambda ws, n: L().gtnb_asg_loss_async(
            h, None, *a, w.data_ptr(), tg.data_ptr(), lens.data_ptr(), *ptrs(trellis), ws, n), trellis),
        "ctc_align": ("gtnb_ctc_align_async_workspace", (B, T, Cn, S, capi.F32), lambda ws, n: L().gtnb_ctc_align_async(
            h, None, *a, tg.data_ptr(), lens.data_ptr(), 0, *ptrs(align), ws, n), align),
        "ngram_ctc_align": ("gtnb_ngram_ctc_align_async_workspace", (B, T, Cn, S, capi.F32),
                            lambda ws, n: L().gtnb_ngram_ctc_align_async(
                                h, None, *a, w[Cn:].data_ptr(), tg.data_ptr(), lens.data_ptr(), 0, *ptrs(align), ws, n),
                            align),
        "asg_align": ("gtnb_asg_align_async_workspace", (B, T, Cn, S, capi.F32), lambda ws, n: L().gtnb_asg_align_async(
            h, None, *a, w.data_ptr(), tg.data_ptr(), lens.data_ptr(), *ptrs(align), ws, n), align),
        "viterbi_transitions": ("gtnb_viterbi_transitions_async_workspace", (G, B, T),
                                lambda ws, n: L().gtnb_viterbi_transitions_async(
                                    h, None, G, B, T, eg.data_ptr(), None, wg.data_ptr(), *ptrs(trans), ws, n), trans),
        "viterbi_dense": ("gtnb_viterbi_dense_async_workspace", (B, T, Cn, capi.F32, capi.DENSE_ASG),
                          lambda ws, n: L().gtnb_viterbi_dense_async(
                              h, None, B, T, Cn, e.data_ptr(), capi.F32, None, capi.DENSE_ASG, w.data_ptr(),
                              *ptrs(dense), ws, n), dense),
        "edit_distance": ("gtnb_edit_distance_async_workspace", (B, S, S, -1, 1),
                          lambda ws, n: L().gtnb_edit_distance_async(
                              h, None, B, hyp.data_ptr(), S, lens.data_ptr(), tg.data_ptr(), S, ref_lens.data_ptr(),
                              -1, *ptrs(edit), ws, n), edit),
        "beam_decode": ("gtnb_beam_decode_async_workspace", (B, T, Cn, capi.F32, capi.DENSE_BIGRAM, 4, 2),
                        lambda ws, n: L().gtnb_beam_decode_async(
                            h, None, B, T, Cn, e.data_ptr(), capi.F32, None, capi.DENSE_BIGRAM, w[Cn:].data_ptr(), 0, 4,
                            2, *ptrs(beam), ws, n), beam),
    }


NAMES = ["ctc_loss", "ngram_ctc_loss", "asg_loss", "ctc_align", "ngram_ctc_align", "asg_align", "viterbi_transitions",
         "viterbi_dense", "edit_distance", "beam_decode"]


@pytest.fixture(scope="module")
def G(ctx):
    g = st.trigram_graph(CG)
    view, keep = capi.make_view(g["flags"], g["src"], g["dst"], g["olabel"], g["olabel"])
    h = C_.c_void_p()
    ctx._check(L().gtnb_transitions_create(ctx.h, C_.byref(view), CG, 0, C_.byref(h)))
    yield h
    L().gtnb_transitions_destroy(ctx.h, h)


def size(ctx, sizing, args):
    n = C_.c_size_t()
    ctx._check(getattr(L(), sizing)(ctx.h, *args, C_.byref(n)))
    return n.value


@pytest.mark.parametrize("name", NAMES)
def test_workspace_rule(ctx, G, name):
    sizing, args, enqueue, outs = calls(ctx, G, 4)[name]
    need = size(ctx, sizing, args)
    assert need > 0 and need % 256 == 0
    ws = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    assert enqueue(None, need) == capi.ERR_INVALID_ARGUMENT
    assert enqueue(ws.data_ptr() + 16, need) == capi.ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    assert all((o == -7).all() for o in outs)  # a refused call writes nothing
    assert enqueue(ws.data_ptr(), need) == 0
    torch.cuda.synchronize()
    assert not all((o == -7).all() for o in outs)
    # B = 0: no bytes, and a NULL workspace is enough
    sizing, args, enqueue, outs = calls(ctx, G, 0)[name]
    assert size(ctx, sizing, args) == 0
    assert enqueue(None, 0) == 0
    assert enqueue(ws.data_ptr() + 16, 0) == capi.ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    # (the loss calls zero the transition gradient for B = 0)
    assert all((o == -7).all() for o in outs if o.numel() != Cn + Cn * Cn)
