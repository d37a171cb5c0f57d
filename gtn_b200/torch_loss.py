"""PyTorch criteria on CUDA tensors, end to end on the device (SURVEY.md section 8(f) rank 1).

The reference's example (bindings/python/examples/pytorch_loss.py:19-102) moves the emissions to
the CPU, builds one Graph per utterance inside gtn.parallel_for and copies the gradients back.
Here the [B, T, C] CUDA tensor goes straight into the C ABI (`gtnb_ctc_loss`, device pointers in,
device gradients out) on the tensor's own CUDA stream; only the B losses visit the host.
"""
import ctypes as C
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import capi

_ctx_cache = {}


def _lengths(input_lengths, B):
    """None, or input_lengths (a list or an int tensor on any device) as a contiguous int32 [B] host array"""
    if input_lengths is None:
        return None
    il = np.ascontiguousarray(
        input_lengths.detach().cpu().numpy() if torch.is_tensor(input_lengths) else input_lengths, np.int32)
    assert il.shape == (B,)
    return il


def _ctx_for(device, stream):
    key = (device.index, stream)
    if key not in _ctx_cache:
        _ctx_cache[key] = capi.Ctx(device.index, stream)
    return _ctx_cache[key]


def _clustered(g, large_transitions, call):
    """call() with the "sparse_cluster" flag of the cached context g at 1 when large_transitions: a transition graph
    beyond one CTA's shared memory (over 4096 states or 32 768 arcs) then takes the thread-block-cluster kernels of
    k_sparse.cu instead of the materialised route; the flag is restored after the call"""
    if not large_transitions:
        return call()
    g.set_flag("sparse_cluster", 1)
    try:
        return call()
    finally:
        g.set_flag("sparse_cluster", 0)


def _allreduce_transitions(ctx, tg, allreduce):
    """Sum the transition gradient tg over the ranks when torch.distributed is initialised (the multi-GPU form of
    Graph::addGrad under grad_lock, graph.cpp:96-100); ctx.world is the number of ranks summed over."""
    ctx.world = 1
    if allreduce and torch.distributed.is_available() and torch.distributed.is_initialized():
        torch.distributed.all_reduce(tg, op=torch.distributed.ReduceOp.SUM)
        ctx.world = torch.distributed.get_world_size()


def _transition_backward(ctx, grad_output):
    """(emission gradient, transition gradient) of asg_loss / ngram_ctc_loss times the upstream gradient; the emission
    gradient keeps its dtype (float32, or the 16-bit dtype of the emissions)"""
    grad, tg = ctx.saved_tensors
    if ctx.reduction == "mean":
        # the mean over the GLOBAL batch when the transition gradient was summed over the ranks
        scale = grad_output / ctx.B
        return grad * scale, tg * (scale / ctx.world)
    # reduction "none": the incoming gradient is per utterance; the transition gradient was already summed
    # over the batch inside the kernel, which is only the chain rule's answer for a uniform grad_output (the
    # emission gradient is right for any grad_output, so transitions that need no gradient take any)
    if ctx.needs_input_grad[1]:
        assert bool((grad_output == grad_output.flatten()[0]).all()), \
            "reduction='none' supports a uniform upstream gradient (sum / mean of the losses)"
    # (a 16-bit grad times the float32 [B] upstream gradient promotes to float32: back to the emissions' dtype)
    return (grad * grad_output.view(-1, 1, 1)).to(grad.dtype), tg * grad_output.flatten()[0]


# the element types of the emissions of ctc_loss, asg_loss, ngram_ctc_loss and the dense Viterbi decoders, as the
# C ABI names them (gtnb_ctc_loss_ex, gtnb_*_typed)
_CTC_DTYPES = {torch.float32: capi.F32, torch.bfloat16: capi.BF16, torch.float16: capi.F16}
_EMISSION_DTYPES = _CTC_DTYPES


class CTCLossFunction(torch.autograd.Function):
    """loss_b = forwardScore(e_b) - forwardScore(intersect(ctcGraph(target_b), e_b))  (benchmarks/ctc.cpp:150-158).

    emissions: float32, bfloat16 or float16 CUDA tensor [B, T, C] (unnormalised scores are fine: the normaliser is
    part of the loss); targets: list of 1-D int sequences; input_lengths: None (T frames each), a list or an int
    tensor (any device): e_b is then the first input_lengths[b] frames, and the gradient of the padding frames is 0.
    Returns the mean loss over the batch (reduction="mean") or the [B] vector, as float32 whatever the emissions'
    dtype (under autocast torch's own ctc_loss runs in float32 too).

    Half-precision emissions (bf16 / fp16 logits of a model under torch.autocast) go in as they are, through
    gtnb_ctc_loss_ex: the losses are those of the float32 call on emissions.float(), bit for bit, and the gradient,
    kept for backward and returned in the emissions' dtype, is that call's float32 gradient rounded to the dtype.
    Nothing is upcast outside the call.
    """

    @staticmethod
    def forward(ctx, emissions, targets, blank=0, reduction="mean", input_lengths=None):
        assert emissions.is_cuda and emissions.dim() == 3
        assert emissions.dtype in _CTC_DTYPES, "ctc_loss: emissions must be float32, bfloat16 or float16"
        e = emissions.contiguous()
        B, T, Cn = e.shape
        stream = torch.cuda.current_stream(e.device).cuda_stream
        g = _ctx_for(e.device, stream)
        cat, lens = capi._cat_targets(targets)
        il = _lengths(input_lengths, B)
        losses = np.zeros(B, np.float32)
        grad = torch.empty_like(e)  # (with input_lengths the call zeroes the padding rows)
        il_p = None if il is None else il.ctypes.data_as(capi._i32p)
        if e.dtype == torch.float32:
            g._check(capi.lib().gtnb_ctc_loss(
                g.h, B, T, Cn, e.data_ptr(), 1, il_p,
                cat.ctypes.data_as(capi._i32p),
                lens.ctypes.data_as(capi._i32p), int(blank), losses.ctypes.data_as(capi._f32p),
                grad.data_ptr(), 1))
        else:
            g._check(capi.lib().gtnb_ctc_loss_ex(
                g.h, B, T, Cn, e.data_ptr(), _CTC_DTYPES[e.dtype], il_p, cat.ctypes.data_as(capi._i32p),
                lens.ctypes.data_as(capi._i32p), int(blank), losses.ctypes.data_as(capi._f32p), grad.data_ptr()))
        out = torch.from_numpy(losses).to(e.device)
        ctx.save_for_backward(grad)
        ctx.reduction = reduction
        ctx.B = B
        return out.mean() if reduction == "mean" else out

    @staticmethod
    def backward(ctx, grad_output):
        (grad,) = ctx.saved_tensors
        if ctx.reduction == "mean":
            scale = grad_output / ctx.B
            return grad * scale, None, None, None, None
        # (a 16-bit grad times the float32 [B] upstream gradient promotes to float32: back to the emissions' dtype)
        return (grad * grad_output.view(-1, 1, 1)).to(grad.dtype), None, None, None, None


_async_ctx_cache = {}


def _async_ctx(device, name="ctc_loss"):
    """One context per device for the asynchronous calls (gtnb_ctc_loss_async, gtnb_ngram_ctc_loss_async,
    gtnb_asg_loss_async), which are handed their stream on every call. It is created by the first call outside stream
    capture: creating a context is not something a capture may record."""
    g = _async_ctx_cache.get(device.index)
    if g is None:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("%s: call it once with tensor targets before capturing a CUDA graph (warm-up), "
                               "so that its context exists" % name)
        g = _async_ctx_cache[device.index] = capi.Ctx(device.index)
    return g


def _workspace(g, device, sizing, *args):
    """The workspace of an asynchronous call: sizing (the call's *_async_workspace) asked for the bytes these
    arguments need, taken from torch's allocator on device (under capture, from the graph's pool) -> (uint8 tensor,
    bytes).  A call that needs none gets an empty tensor, whose data_ptr() is NULL.  A nonzero code raises."""
    nbytes = C.c_size_t()
    g._check(sizing(g.h, *args, C.byref(nbytes)))
    return torch.empty(nbytes.value, dtype=torch.uint8, device=device), nbytes.value


def _host_targets(ctx, err, name, routes, reduction, targets, target_lengths, forward):
    """A loss on tensor targets whose sizing query raised err: for GTNB_ERR_UNSUPPORTED (bounds outside the
    asynchronous routes) the list-target call forward(lists) with reduction "none" on the targets copied to the host
    -- a documented synchronisation -- and a RuntimeError under capture; any other error raised as it is."""
    if err.code != capi.ERR_UNSUPPORTED:
        raise err
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("%s: these bounds are outside the asynchronous %s (%s) and cannot be captured"
                           % (name, routes, err)) from None
    rows = targets.cpu().tolist()
    lens = target_lengths.cpu().tolist()
    out = forward([r[:n] for r, n in zip(rows, lens)])
    ctx.reduction = reduction
    return out.mean() if reduction == "mean" else out


class CTCLossAsyncFunction(torch.autograd.Function):
    """ctc_loss on tensor targets: gtnb_ctc_loss_async on the current stream, with no host synchronisation in forward
    or backward, so that the step can be captured in a CUDA graph.

    targets: [B, S] integer tensor on the emissions' device, row b holding target_lengths[b] labels; target_lengths
    and input_lengths (or None): [B] integer tensors on that device.  The losses are float32 device tensors, those of
    the list-target call bit for bit.  An utterance the device call flags gets a NaN loss and a zero gradient: a
    non-finite emission (the list-target call repeats such a batch exactly on the host), or an invalid length or
    label (the list-target call raises for the whole batch).  Bounds outside the asynchronous routes run the
    synchronous call on the targets copied to the host -- a documented synchronisation -- and raise under capture.
    """

    @staticmethod
    def forward(ctx, emissions, targets, blank, reduction, input_lengths, target_lengths):
        e = emissions.contiguous()
        B, T, Cn = e.shape
        S = targets.shape[1]
        tg = targets.to(torch.int32).contiguous()
        tl = target_lengths.to(torch.int32).contiguous()
        il = None if input_lengths is None else input_lengths.to(torch.int32).contiguous()
        dtype = _CTC_DTYPES[e.dtype]
        g = _async_ctx(e.device)
        try:
            ws, nbytes = _workspace(g, e.device, capi.lib().gtnb_ctc_loss_async_workspace, B, T, Cn, S, dtype, 1)
        except capi.GtnbError as err:
            return _host_targets(ctx, err, "ctc_loss", "routes", reduction, tg, tl,
                                 lambda lists: CTCLossFunction.forward(ctx, e, lists, blank, "none", input_lengths))
        losses = torch.empty(B, dtype=torch.float32, device=e.device)
        grad = torch.empty_like(e)
        g._check(capi.lib().gtnb_ctc_loss_async(
            g.h, torch.cuda.current_stream(e.device).cuda_stream, B, T, Cn, S, e.data_ptr(), dtype,
            None if il is None else il.data_ptr(), tg.data_ptr(), tl.data_ptr(), int(blank), losses.data_ptr(), None,
            grad.data_ptr(), ws.data_ptr(), nbytes))
        ctx.save_for_backward(grad)
        ctx.reduction = reduction
        ctx.B = B
        return losses.mean() if reduction == "mean" else losses

    @staticmethod
    def backward(ctx, grad_output):
        return CTCLossFunction.backward(ctx, grad_output)[:1] + (None,) * 5


def ctc_loss(emissions, targets, blank=0, reduction="mean", input_lengths=None, target_lengths=None):
    """CTC loss (CTCLossFunction).  With targets a 2-D integer CUDA tensor on the emissions' device and target_lengths
    given, the call runs on the device without a host synchronisation (CTCLossAsyncFunction)."""
    if torch.is_tensor(targets) and targets.is_cuda and targets.dim() == 2:
        assert not targets.is_floating_point() and targets.device == emissions.device
        assert torch.is_tensor(target_lengths) and target_lengths.device == emissions.device, \
            "ctc_loss: tensor targets need target_lengths on the emissions' device"
        assert input_lengths is None or (torch.is_tensor(input_lengths) and input_lengths.device == emissions.device), \
            "ctc_loss: with tensor targets, input_lengths must be None or a tensor on the emissions' device"
        assert emissions.is_cuda and emissions.dim() == 3 and emissions.dtype in _CTC_DTYPES
        assert targets.shape[0] == emissions.shape[0] and target_lengths.shape == (emissions.shape[0],)
        return CTCLossAsyncFunction.apply(emissions, targets, blank, reduction, input_lengths, target_lengths)
    return CTCLossFunction.apply(emissions, targets, blank, reduction, input_lengths)


class ASGLossFunction(torch.autograd.Function):
    """loss_b = forwardScore(compose(e_b, transitions)) - forwardScore(compose(compose(fal_b, transitions), e_b))
    (examples/asg.cpp:59-81, test/criterion_test.cpp:244-305) with ONE learned transitions graph shared by the
    minibatch -- and by all ranks: with torch.distributed initialised, the transition gradient of the local shard
    is all-reduced (sum) over NCCL, the multi-GPU form of Graph::addGrad under grad_lock (graph.cpp:96-100).

    emissions: float32, bfloat16 or float16 CUDA tensor [B, T, C]; transitions: float32 tensor [C + C*C] (start
    weights, then the C x C matrix, row = destination label) on any device; targets: list of 1-D int sequences.
    The losses are float32 whatever the emissions' dtype.

    input_lengths: None (T frames each), a list or an int tensor (any device).  When given, e_b is the first
    input_lengths[b] frames (the gradient of the padding frames is 0) and the call goes through gtnb_asg_loss_ex
    on device pointers: transitions must then be a float32 CUDA tensor on the emissions' device, and the
    transition gradient stays on the device.

    Half-precision emissions (bf16 / fp16 logits of a model under torch.autocast) go in as they are, through
    gtnb_asg_loss_typed: the losses and the transition gradient are those of the float32 call on emissions.float(),
    bit for bit, and the emission gradient, kept for backward in the emissions' dtype, is that call's float32
    gradient rounded to the dtype.  Without input_lengths that call takes T_b = T, with the transitions copied to the
    emissions' device as float32 and their gradient returned on transitions.device: asg_loss(e, ...) then equals
    asg_loss(e.float(), ..., input_lengths=[T] * B).
    """

    @staticmethod
    def forward(ctx, emissions, transitions, targets, reduction="mean", allreduce=True, input_lengths=None):
        assert emissions.is_cuda and emissions.dim() == 3
        assert emissions.dtype in _EMISSION_DTYPES, "asg_loss: emissions must be float32, bfloat16 or float16"
        e = emissions.contiguous()
        B, T, Cn = e.shape
        half = e.dtype != torch.float32
        assert transitions.numel() == Cn + Cn * Cn
        stream = torch.cuda.current_stream(e.device).cuda_stream
        g = _ctx_for(e.device, stream)
        cat, lens = capi._cat_targets(targets)
        losses = np.zeros(B, np.float32)
        if half:
            assert transitions.dtype == torch.float32, "asg_loss: transitions must be float32"
            il = _lengths(input_lengths, B)
            w = transitions.detach().to(e.device).contiguous()
            grad = torch.empty_like(e)  # every row is written by the call
            tg = torch.empty(Cn + Cn * Cn, dtype=torch.float32, device=e.device)
            g._check(capi.lib().gtnb_asg_loss_typed(
                g.h, B, T, Cn, e.data_ptr(), _EMISSION_DTYPES[e.dtype], None if il is None else il.ctypes.data_as(capi._i32p),
                w.data_ptr(), cat.ctypes.data_as(capi._i32p), lens.ctypes.data_as(capi._i32p),
                losses.ctypes.data_as(capi._f32p), grad.data_ptr(), tg.data_ptr()))
            tg = tg.view_as(transitions)
        elif input_lengths is not None:
            assert transitions.is_cuda and transitions.device == e.device and transitions.dtype == torch.float32
            il = _lengths(input_lengths, B)
            w = transitions.detach().contiguous()
            grad = torch.empty_like(e)  # every row is written by the call
            tg = torch.empty(Cn + Cn * Cn, dtype=torch.float32, device=e.device)
            g._check(capi.lib().gtnb_asg_loss_ex(
                g.h, B, T, Cn, e.data_ptr(), 1, il.ctypes.data_as(capi._i32p), w.data_ptr(), 1,
                cat.ctypes.data_as(capi._i32p), lens.ctypes.data_as(capi._i32p), losses.ctypes.data_as(capi._f32p),
                grad.data_ptr(), 1, tg.data_ptr(), 1))
            tg = tg.view_as(transitions)
        else:
            tw = np.ascontiguousarray(transitions.detach().to("cpu", torch.float32).numpy())
            tgrad = np.zeros(Cn + Cn * Cn, np.float32)
            grad = torch.empty_like(e)
            g._check(capi.lib().gtnb_asg_loss(
                g.h, B, T, Cn, e.data_ptr(), 1, tw.ctypes.data_as(capi._f32p), cat.ctypes.data_as(capi._i32p),
                lens.ctypes.data_as(capi._i32p), losses.ctypes.data_as(capi._f32p), grad.data_ptr(), 1,
                tgrad.ctypes.data_as(capi._f32p)))
            tg = torch.from_numpy(tgrad).to(e.device)
        _allreduce_transitions(ctx, tg, allreduce)
        out = torch.from_numpy(losses).to(e.device)
        ctx.save_for_backward(grad, tg)
        ctx.reduction = reduction
        ctx.B = B
        ctx.tdev = transitions.device
        return out.mean() if reduction == "mean" else out

    @staticmethod
    def backward(ctx, grad_output):
        grad, tg = _transition_backward(ctx, grad_output)
        return grad, tg.to(ctx.tdev), None, None, None, None


def _tensor_targets(name, emissions, targets, input_lengths, target_lengths):
    """True when targets is a 2-D integer CUDA tensor, the asynchronous route's input (its arguments checked)"""
    if not (torch.is_tensor(targets) and targets.is_cuda and targets.dim() == 2):
        return False
    assert not targets.is_floating_point() and targets.device == emissions.device
    assert torch.is_tensor(target_lengths) and target_lengths.device == emissions.device, \
        "%s: tensor targets need target_lengths on the emissions' device" % name
    assert input_lengths is None or (torch.is_tensor(input_lengths) and input_lengths.device == emissions.device), \
        "%s: with tensor targets, input_lengths must be None or a tensor on the emissions' device" % name
    assert emissions.is_cuda and emissions.dim() == 3 and emissions.dtype in _EMISSION_DTYPES
    assert targets.shape[0] == emissions.shape[0] and target_lengths.shape == (emissions.shape[0],)
    return True


class TrellisLossAsyncFunction(torch.autograd.Function):
    """asg_loss and ngram_ctc_loss on tensor targets: gtnb_asg_loss_async / gtnb_ngram_ctc_loss_async on the current
    stream, with no host synchronisation in forward or backward, so that a step that trains the transitions can be
    captured in a CUDA graph.

    targets: [B, S] integer tensor on the emissions' device, row b holding target_lengths[b] labels; target_lengths
    and input_lengths (or None): [B] integer tensors on that device; transitions: float32 CUDA tensor on that device.
    The losses are float32 device tensors, those of the list-target call bit for bit.  An utterance the device call
    flags gets a NaN loss, a zero emission gradient and no share of the transition gradient: a non-finite emission or
    transition weight (the list-target call repeats such a batch exactly on the host), or an invalid length or label
    (the list-target call raises for the whole batch).  Bounds outside the asynchronous route run the synchronous call
    on the targets copied to the host -- a documented synchronisation -- and raise under capture.

    reduction="none": the transition gradient is summed over the batch inside the kernels, the chain rule's answer
    only for a uniform upstream gradient.  The list-target call asserts that on the host; here, where nothing may
    synchronise, a non-uniform upstream gradient gives a NaN transition gradient instead.
    """

    @staticmethod
    def forward(ctx, emissions, transitions, targets, asg, blank, reduction, allreduce, input_lengths, target_lengths):
        name = "asg_loss" if asg else "ngram_ctc_loss"
        e = emissions.contiguous()
        B, T, Cn = e.shape
        S = targets.shape[1]
        assert transitions.is_cuda and transitions.device == e.device and transitions.dtype == torch.float32
        assert transitions.numel() == (Cn + Cn * Cn if asg else Cn * Cn)
        w = transitions.detach().contiguous()
        tgt = targets.to(torch.int32).contiguous()
        tl = target_lengths.to(torch.int32).contiguous()
        il = None if input_lengths is None else input_lengths.to(torch.int32).contiguous()
        dtype = _EMISSION_DTYPES[e.dtype]
        g = _async_ctx(e.device, name)
        lib = capi.lib()
        call = lib.gtnb_asg_loss_async if asg else lib.gtnb_ngram_ctc_loss_async
        sizing = lib.gtnb_asg_loss_async_workspace if asg else lib.gtnb_ngram_ctc_loss_async_workspace
        try:
            ws, nbytes = _workspace(g, e.device, sizing, B, T, Cn, S, dtype, 1)
        except capi.GtnbError as err:
            return _host_targets(ctx, err, name, "route", reduction, tgt, tl, lambda lists: (
                ASGLossFunction.forward(ctx, e, transitions, lists, "none", allreduce, input_lengths) if asg else
                NgramCTCLossFunction.forward(ctx, e, transitions, lists, input_lengths, blank, "none", allreduce)))
        losses = torch.empty(B, dtype=torch.float32, device=e.device)
        grad = torch.empty_like(e)
        tg = torch.empty(transitions.numel(), dtype=torch.float32, device=e.device)
        stream = torch.cuda.current_stream(e.device).cuda_stream
        il_p = None if il is None else il.data_ptr()
        if asg:
            rc = call(g.h, stream, B, T, Cn, S, e.data_ptr(), dtype, il_p, w.data_ptr(), tgt.data_ptr(), tl.data_ptr(),
                      losses.data_ptr(), None, grad.data_ptr(), tg.data_ptr(), ws.data_ptr(), nbytes)
        else:
            rc = call(g.h, stream, B, T, Cn, S, e.data_ptr(), dtype, il_p, w.data_ptr(), tgt.data_ptr(), tl.data_ptr(),
                      int(blank), losses.data_ptr(), None, grad.data_ptr(), tg.data_ptr(), ws.data_ptr(), nbytes)
        g._check(rc)
        tg = tg.view_as(transitions)
        _allreduce_transitions(ctx, tg, allreduce)
        ctx.save_for_backward(grad, tg)
        ctx.reduction = reduction
        ctx.B = B
        return losses.mean() if reduction == "mean" else losses

    @staticmethod
    def backward(ctx, grad_output):
        grad, tg = ctx.saved_tensors
        if ctx.reduction == "mean":
            scale = grad_output / ctx.B
            egrad, tgrad = grad * scale, tg * (scale / ctx.world)
        else:
            # (a 16-bit grad times the float32 [B] upstream gradient promotes to float32: back to the emissions' dtype)
            egrad = (grad * grad_output.view(-1, 1, 1)).to(grad.dtype)
            g0 = grad_output.flatten()[0]
            uniform = (grad_output == g0).all()  # a 0-dim device bool: chosen on the device, no synchronisation
            tgrad = torch.where(uniform, tg * g0, torch.full_like(tg, float("nan")))
        return egrad, tgrad, None, None, None, None, None, None, None


def asg_loss(emissions, transitions, targets, reduction="mean", allreduce=True, input_lengths=None,
             target_lengths=None):
    """ASG loss (ASGLossFunction).  With targets a 2-D integer CUDA tensor on the emissions' device and target_lengths
    given, the call runs on the device without a host synchronisation (TrellisLossAsyncFunction)."""
    if _tensor_targets("asg_loss", emissions, targets, input_lengths, target_lengths):
        return TrellisLossAsyncFunction.apply(emissions, transitions, targets, True, 0, reduction, allreduce,
                                              input_lengths, target_lengths)
    return ASGLossFunction.apply(emissions, transitions, targets, reduction, allreduce, input_lengths)


class NgramCTCLossFunction(torch.autograd.Function):
    """CTC with a learned bigram transition graph G (benchmarks/ctc.cpp:107-134, timeNgramCtc):
        loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(ctc_b, G), E_b))
    G: C nodes, all start and accept, arc j -> i with label i and weight transitions[i, j] (row = destination
    label, column = source label), shared by the minibatch and, with torch.distributed initialised, by all ranks
    (the transition gradient is all-reduced over NCCL, as asg_loss does).

    emissions: float32, bfloat16 or float16 CUDA tensor [B, T, C]; transitions: float32 CUDA tensor of C*C elements
    ([C, C] or flat) on the same device; targets: list of 1-D int sequences; input_lengths: None, a list or an int
    tensor (any device).  Everything runs on the current stream of the emissions' device, device pointers in and
    out: only the B losses (and input_lengths, when given on the GPU) are copied to the host.  The losses are
    float32 whatever the emissions' dtype.

    Half-precision emissions (bf16 / fp16 logits of a model under torch.autocast) go in as they are, through
    gtnb_ngram_ctc_loss_typed: the losses and the transition gradient are those of the float32 call on
    emissions.float(), bit for bit, and the emission gradient, kept for backward in the emissions' dtype, is that
    call's float32 gradient rounded to the dtype.
    """

    @staticmethod
    def forward(ctx, emissions, transitions, targets, input_lengths=None, blank=0, reduction="mean", allreduce=True):
        assert emissions.is_cuda and emissions.dim() == 3
        assert emissions.dtype in _EMISSION_DTYPES, "ngram_ctc_loss: emissions must be float32, bfloat16 or float16"
        e = emissions.contiguous()
        B, T, Cn = e.shape
        assert transitions.is_cuda and transitions.device == e.device and transitions.dtype == torch.float32
        assert transitions.numel() == Cn * Cn
        w = transitions.detach().contiguous()
        stream = torch.cuda.current_stream(e.device).cuda_stream
        g = _ctx_for(e.device, stream)
        cat, lens = capi._cat_targets(targets)
        il = _lengths(input_lengths, B)
        losses = np.zeros(B, np.float32)
        grad = torch.empty_like(e)  # every row is written by the call
        tg = torch.empty(Cn * Cn, dtype=torch.float32, device=e.device)
        il_p = None if il is None else il.ctypes.data_as(capi._i32p)
        if e.dtype == torch.float32:
            g._check(capi.lib().gtnb_ngram_ctc_loss(
                g.h, B, T, Cn, e.data_ptr(), 1, il_p, w.data_ptr(), 1,
                cat.ctypes.data_as(capi._i32p), lens.ctypes.data_as(capi._i32p), int(blank),
                losses.ctypes.data_as(capi._f32p), grad.data_ptr(), 1, tg.data_ptr(), 1))
        else:
            g._check(capi.lib().gtnb_ngram_ctc_loss_typed(
                g.h, B, T, Cn, e.data_ptr(), _EMISSION_DTYPES[e.dtype], il_p, w.data_ptr(), cat.ctypes.data_as(capi._i32p),
                lens.ctypes.data_as(capi._i32p), int(blank), losses.ctypes.data_as(capi._f32p), grad.data_ptr(),
                tg.data_ptr()))
        tg = tg.view_as(transitions)
        _allreduce_transitions(ctx, tg, allreduce)
        out = torch.from_numpy(losses).to(e.device)
        ctx.save_for_backward(grad, tg)
        ctx.reduction = reduction
        ctx.B = B
        return out.mean() if reduction == "mean" else out

    @staticmethod
    def backward(ctx, grad_output):
        grad, tg = _transition_backward(ctx, grad_output)
        return grad, tg, None, None, None, None, None


def ngram_ctc_loss(emissions, transitions, targets, input_lengths=None, blank=0, reduction="mean", allreduce=True,
                   target_lengths=None):
    """n-gram CTC loss (NgramCTCLossFunction).  With targets a 2-D integer CUDA tensor on the emissions' device and
    target_lengths given, the call runs on the device without a host synchronisation (TrellisLossAsyncFunction)."""
    if _tensor_targets("ngram_ctc_loss", emissions, targets, input_lengths, target_lengths):
        return TrellisLossAsyncFunction.apply(emissions, transitions, targets, False, blank, reduction, allreduce,
                                              input_lengths, target_lengths)
    return NgramCTCLossFunction.apply(emissions, transitions, targets, input_lengths, blank, reduction, allreduce)


@torch.no_grad()
def _viterbi_dense(emissions, transitions, input_lengths, kind):
    assert emissions.is_cuda and emissions.dim() == 3
    assert emissions.dtype in _EMISSION_DTYPES, "emissions must be float32, bfloat16 or float16"
    e = emissions.contiguous()
    B, T, Cn = e.shape
    assert transitions.is_cuda and transitions.device == e.device and transitions.dtype == torch.float32
    assert transitions.numel() == (Cn * Cn if kind == capi.DENSE_BIGRAM else Cn + Cn * Cn)
    w = transitions.detach().contiguous()
    current = torch.cuda.current_stream(e.device)
    g = _ctx_for(e.device, current.cuda_stream)
    il = _lengths(input_lengths, B)
    paths = torch.empty((B, T), dtype=torch.int32, device=e.device)  # every entry is written by the call
    scores = torch.empty(B, dtype=torch.float32, device=e.device)
    # the call returns once its work is enqueued on the context's stream, which is the current stream unless that
    # is the legacy default stream (the context then has a stream of its own): order the two both ways
    ctx_stream = torch.cuda.ExternalStream(capi.lib().gtnb_ctx_stream(g.h), device=e.device)
    ctx_stream.wait_stream(current)
    il_p = None if il is None else il.ctypes.data_as(capi._i32p)
    if e.dtype == torch.float32:
        g._check(capi.lib().gtnb_viterbi_dense_ex(
            g.h, B, T, Cn, e.data_ptr(), 1, il_p, kind, w.data_ptr(), 1, paths.data_ptr(), scores.data_ptr(), 1))
    else:  # 16-bit emissions, read in place by the kernel
        g._check(capi.lib().gtnb_viterbi_dense_typed(
            g.h, B, T, Cn, e.data_ptr(), _EMISSION_DTYPES[e.dtype], il_p, kind, w.data_ptr(), paths.data_ptr(),
            scores.data_ptr()))
    current.wait_stream(ctx_stream)
    return paths, scores


def asg_viterbi(emissions, transitions, input_lengths=None):
    """Best path of compose(E_b, transitions) for every utterance, with the transitions asg_loss trains
    (examples/asg.cpp's decoding, test/criterion_test.cpp:328-344), through gtnb_viterbi_dense_ex.

    emissions: float32, bfloat16 or float16 CUDA tensor [B, T, C] (16-bit emissions go through
    gtnb_viterbi_dense_typed: the paths and scores of the float32 call on emissions.float(), ties included);
    transitions: float32 CUDA tensor of C + C*C elements (start weights, then the C x C matrix, row = destination
    label) on the same device; input_lengths: None, a list or an int tensor (any device).  Returns (paths [B, T] int32, the label of every frame, -1 beyond T_b; scores [B], viterbiScore,
    -inf for T_b = 0), both CUDA tensors written on the current stream; only input_lengths visits the host.
    """
    return _viterbi_dense(emissions, transitions, input_lengths, capi.DENSE_ASG)


def ngram_ctc_viterbi(emissions, transitions, input_lengths=None):
    """Best path of intersect(E_b, G) for every utterance, G the bigram transition graph ngram_ctc_loss trains,
    through gtnb_viterbi_dense_ex.  transitions: float32 CUDA tensor of C*C elements ([C, C] or flat, row =
    destination label).  The arguments and results are those of asg_viterbi; collapse(paths, blank) gives the
    transcript.
    """
    return _viterbi_dense(emissions, transitions, input_lengths, capi.DENSE_BIGRAM)


@torch.no_grad()
def collapse(paths, blank=None):
    """Transcripts of frame-level paths: repeats merged, then `blank` dropped when one is given (CTC's rule; with
    blank=None, ASG's).  paths: int tensor [B, T], -1 padding.  Returns (labels [B, T] int32, each row's transcript
    followed by -1, lengths [B] int64), on the paths' device, without a host synchronisation."""
    p = paths.int()
    B, T = p.shape
    keep = p >= 0
    keep[:, 1:] &= p[:, 1:] != p[:, :-1]
    if blank is not None:
        keep &= p != blank
    lengths = keep.sum(dim=1)
    # the kept labels of a row go to the front: slot = number of kept labels before them
    slot = torch.where(keep, keep.cumsum(dim=1) - 1, T)
    out = torch.full((B, T + 1), -1, dtype=torch.int32, device=p.device)
    out.scatter_(1, slot, torch.where(keep, p, -1))
    return out[:, :T].contiguous(), lengths


@torch.no_grad()
def _align_async(name, emissions, transitions, targets, target_lengths, input_lengths, blank, kind):
    """gtnb_{ctc,ngram_ctc,asg}_align_async on the current stream (kind: "ctc", "ngram", "asg")"""
    assert _tensor_targets(name, emissions, targets, input_lengths, target_lengths), \
        "%s: targets must be a 2-D integer CUDA tensor on the emissions' device" % name
    e = emissions.contiguous()
    B, T, Cn = e.shape
    S = targets.shape[1]
    w = None
    if kind != "ctc":
        assert transitions.is_cuda and transitions.device == e.device and transitions.dtype == torch.float32
        assert transitions.numel() == (Cn + Cn * Cn if kind == "asg" else Cn * Cn)
        w = transitions.detach().contiguous()
    tgt = targets.to(torch.int32).contiguous()
    tl = target_lengths.to(torch.int32).contiguous()
    il = None if input_lengths is None else input_lengths.to(torch.int32).contiguous()
    dtype = _EMISSION_DTYPES[e.dtype]
    g = _async_ctx(e.device, name)
    lib = capi.lib()
    call, sizing = {"ctc": (lib.gtnb_ctc_align_async, lib.gtnb_ctc_align_async_workspace),
                    "ngram": (lib.gtnb_ngram_ctc_align_async, lib.gtnb_ngram_ctc_align_async_workspace),
                    "asg": (lib.gtnb_asg_align_async, lib.gtnb_asg_align_async_workspace)}[kind]
    try:
        ws, nbytes = _workspace(g, e.device, sizing, B, T, Cn, S, dtype)
    except capi.GtnbError as err:
        if err.code != capi.ERR_UNSUPPORTED:
            raise
        other = "graph_viterbi" if kind == "ctc" else "graph_transitions_viterbi"
        raise RuntimeError("%s: these bounds are outside the device alignment (%s); align on the host-built graphs "
                           "with %s instead" % (name, err, other)) from None
    paths = torch.empty((B, T), dtype=torch.int32, device=e.device)
    tokens = torch.empty((B, T), dtype=torch.int32, device=e.device)
    scores = torch.empty(B, dtype=torch.float32, device=e.device)
    status = torch.empty(B, dtype=torch.int32, device=e.device)
    stream = torch.cuda.current_stream(e.device).cuda_stream
    il_p = None if il is None else il.data_ptr()
    outs = (paths.data_ptr(), tokens.data_ptr(), scores.data_ptr(), status.data_ptr(), ws.data_ptr(), nbytes)
    if kind == "ctc":
        rc = call(g.h, stream, B, T, Cn, S, e.data_ptr(), dtype, il_p, tgt.data_ptr(), tl.data_ptr(), int(blank), *outs)
    elif kind == "ngram":
        rc = call(g.h, stream, B, T, Cn, S, e.data_ptr(), dtype, il_p, w.data_ptr(), tgt.data_ptr(), tl.data_ptr(),
                  int(blank), *outs)
    else:
        rc = call(g.h, stream, B, T, Cn, S, e.data_ptr(), dtype, il_p, w.data_ptr(), tgt.data_ptr(), tl.data_ptr(),
                  *outs)
    g._check(rc)
    return paths, tokens, scores, status


def ctc_align(emissions, targets, target_lengths, input_lengths=None, blank=0):
    """Forced alignment of CTC: viterbiPath / viterbiScore of intersect(ctcGraph(y_b), E_b), the numerator of ctc_loss,
    through gtnb_ctc_align_async on the current stream, without a host synchronisation (it may be captured in a CUDA
    graph).

    emissions: float32, bfloat16 or float16 CUDA tensor [B, T, C] (16-bit: the results of the float32 call on
    emissions.float()); targets: [B, S] integer tensor on the emissions' device, row b holding target_lengths[b]
    labels; target_lengths and input_lengths (or None): [B] integer tensors on that device.  Returns device tensors
    (paths [B, T] int32, the label of every frame; tokens [B, T] int32, the target position each frame is aligned to,
    -1 for a blank frame; both -1 beyond T_b and where no path accepts; scores [B] float32, -inf for a target with no
    path; status [B] int32: 0 as gtnb_graph_viterbi, 1 a non-finite value, 2 an invalid length or label, both with a
    NaN score and -1 rows, 3 a tie on the path, which is then an optimal path that gtnb_graph_viterbi may break
    differently).  Bounds outside the device route raise a RuntimeError; graph_viterbi on ctc graphs covers them.
    """
    return _align_async("ctc_align", emissions, None, targets, target_lengths, input_lengths, blank, "ctc")


def ngram_ctc_align(emissions, transitions, targets, target_lengths, input_lengths=None, blank=0):
    """Forced alignment of n-gram CTC: viterbiPath / viterbiScore of intersect(intersect(ctc_b, G), E_b), the numerator
    of ngram_ctc_loss, through gtnb_ngram_ctc_align_async.  transitions: float32 CUDA tensor of C*C elements (row =
    destination label) on the emissions' device.  Arguments and results otherwise as ctc_align's; any C the device
    sweeps take, beyond ngram_ctc_loss's 128 labels.  Bounds outside the device route raise a RuntimeError;
    graph_transitions_viterbi (kind "bigram") covers them.
    """
    return _align_async("ngram_ctc_align", emissions, transitions, targets, target_lengths, input_lengths, blank,
                        "ngram")


def asg_align(emissions, transitions, targets, target_lengths, input_lengths=None):
    """Forced alignment of ASG: viterbiPath / viterbiScore of compose(compose(fal_b, transitions), E_b), the numerator
    of asg_loss, through gtnb_asg_align_async.  transitions: float32 CUDA tensor of C + C*C elements (start weights,
    then the matrix) on the emissions' device.  Every frame in [0, T_b) of an accepted path gets a target position.
    Arguments and results otherwise as ctc_align's.  Bounds outside the device route raise a RuntimeError;
    graph_transitions_viterbi (kind "asg") on force-align chains covers them.
    """
    return _align_async("asg_align", emissions, transitions, targets, target_lengths, input_lengths, 0, "asg")


@torch.no_grad()
def align_spans(tokens, S):
    """The frames each target position occupies: tokens [B, T] (ctc_align's, -1 for none) -> (start, end), each
    [B, S] int32, the first frame and one past the last frame of position u, -1 where u is absent.  Elementwise and
    scatter ops on the tokens' device, without a host synchronisation."""
    tok = tokens.long()
    B, T = tok.shape
    present = (tok >= 0) & (tok < S)
    slot = torch.where(present, tok, S)  # absent frames go to an extra column that is dropped
    t = torch.arange(T, device=tok.device).expand(B, T)
    start = torch.full((B, S + 1), T, dtype=torch.long, device=tok.device)
    start.scatter_reduce_(1, slot, torch.where(present, t, T), "amin")
    end = torch.full((B, S + 1), -1, dtype=torch.long, device=tok.device)
    end.scatter_reduce_(1, slot, torch.where(present, t + 1, -1), "amax")
    absent = end[:, :S] < 0
    return (torch.where(absent, -1, start[:, :S]).int(), torch.where(absent, -1, end[:, :S]).int())


class TransitionGraph:
    """A transition graph prepared once for transitions_decode: the tables of G (a gtn_b200.gtn.Graph, the structure of
    sparse_viterbi's or, with backoff=True, backoff_viterbi's transitions_graph) packed and uploaded to `device` (the
    current CUDA device by default) through gtnb_transitions_create, with the route for num_labels labels.
    large_transitions: a G beyond one CTA takes the thread-block-cluster kernels, as in sparse_viterbi.  G's weights are
    not kept: the learned transitions are passed to every transitions_decode call.

    Creating one allocates and synchronises, so it raises while a stream is capturing: build it before capture.  A
    captured CUDA graph that decodes with it reads its tables, and must not be replayed once it is gone: keep it alive
    as long as the captured graph.  A G outside the device decoders' envelope raises a RuntimeError that names the
    synchronous decoder to use instead."""

    def __init__(self, graph, num_labels, device=None, backoff=False, large_transitions=False):
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("TransitionGraph: create it before capturing a CUDA graph (it allocates and "
                               "synchronises)")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.num_labels = int(num_labels)
        self.backoff = bool(backoff)
        view, keep = _graph_view(graph)
        self.num_arcs = view.num_arcs
        self._g = _async_ctx(self.device, "TransitionGraph")
        h = C.c_void_p()
        rc = _clustered(self._g, large_transitions, lambda: capi.lib().gtnb_transitions_create(
            self._g.h, C.byref(view), self.num_labels, int(self.backoff), C.byref(h)))
        del keep
        if rc == capi.ERR_UNSUPPORTED:
            raise RuntimeError("TransitionGraph: %s" % capi.lib().gtnb_last_error(self._g.h).decode())
        self._g._check(rc)
        self.h = h

    def __del__(self):
        h = getattr(self, "h", None)
        if h is not None and h.value:
            capi.lib().gtnb_transitions_destroy(self._g.h, h)
            self.h = None


def _decode_lengths(e, input_lengths):
    """input_lengths as int32 on the emissions' device, without a copy between devices (None stays None)"""
    if input_lengths is None:
        return None
    assert torch.is_tensor(input_lengths) and input_lengths.device == e.device and \
        not input_lengths.is_floating_point(), "input_lengths must be None or an integer tensor on the emissions' device"
    assert input_lengths.shape == (e.shape[0],)
    return input_lengths.to(torch.int32).contiguous()


@torch.no_grad()
def transitions_decode(emissions, transitions, graph, input_lengths=None):
    """Best path of intersect(E_b, G) for every utterance, G a prepared TransitionGraph, through
    gtnb_viterbi_transitions_async on the current stream, without a host synchronisation (it may be captured in a
    CUDA graph; the workspace comes from torch's allocator).

    emissions: float32 CUDA tensor [B, T, C], C = graph.num_labels, on graph's device; transitions: float32 tensor of
    graph.num_arcs elements on that device (G's arc numbering); input_lengths: None or a [B] integer tensor on that
    device.  Returns device tensors (paths [B, T] int32, the label of every frame; scores [B] float32, viterbiScore;
    arcs [B, T] int32, the emitting G arc of every frame; status [B] int32).  Status 0: sparse_viterbi's (or
    backoff_viterbi's) result, bit for bit; 1: a NaN or +inf weight or used emission, 2: a length outside [0, T], both
    with a NaN score and -1 rows; 3: a tie, the score exact and the path an optimal one (the synchronous decoder's
    with the "exact_ties" flag off).  Rows are -1 beyond T_b and where no path accepts (score -inf).
    collapse(paths, blank) turns the paths into transcripts.
    """
    assert isinstance(graph, TransitionGraph)
    assert emissions.is_cuda and emissions.dim() == 3 and emissions.dtype == torch.float32, \
        "emissions must be a float32 CUDA tensor [B, T, C]"
    e = emissions.contiguous()
    B, T, Cn = e.shape
    assert e.device == graph.device and Cn == graph.num_labels
    assert transitions.is_cuda and transitions.device == e.device and transitions.dtype == torch.float32
    assert transitions.numel() == graph.num_arcs
    w = transitions.detach().contiguous() if transitions.numel() else torch.zeros(1, device=e.device)
    il = _decode_lengths(e, input_lengths)
    g = graph._g
    lib = capi.lib()
    ws, nbytes = _workspace(g, e.device, lib.gtnb_viterbi_transitions_async_workspace, graph.h, B, T)
    paths = torch.empty((B, T), dtype=torch.int32, device=e.device)
    arcs = torch.empty((B, T), dtype=torch.int32, device=e.device)
    scores = torch.empty(B, dtype=torch.float32, device=e.device)
    status = torch.empty(B, dtype=torch.int32, device=e.device)
    g._check(lib.gtnb_viterbi_transitions_async(
        g.h, torch.cuda.current_stream(e.device).cuda_stream, graph.h, B, T, e.data_ptr(),
        None if il is None else il.data_ptr(), w.data_ptr(), paths.data_ptr(), arcs.data_ptr(), scores.data_ptr(),
        status.data_ptr(), ws.data_ptr(), nbytes))
    return paths, scores, arcs, status


@torch.no_grad()
def _dense_decode(name, emissions, transitions, input_lengths, kind):
    """gtnb_viterbi_dense_async on the current stream"""
    assert emissions.is_cuda and emissions.dim() == 3
    assert emissions.dtype in _EMISSION_DTYPES, "emissions must be float32, bfloat16 or float16"
    e = emissions.contiguous()
    B, T, Cn = e.shape
    assert transitions.is_cuda and transitions.device == e.device and transitions.dtype == torch.float32
    assert transitions.numel() == (Cn * Cn if kind == capi.DENSE_BIGRAM else Cn + Cn * Cn)
    w = transitions.detach().contiguous()
    il = _decode_lengths(e, input_lengths)
    dtype = _EMISSION_DTYPES[e.dtype]
    g = _async_ctx(e.device, name)
    lib = capi.lib()
    ws, nbytes = _workspace(g, e.device, lib.gtnb_viterbi_dense_async_workspace, B, T, Cn, dtype, kind)
    paths = torch.empty((B, T), dtype=torch.int32, device=e.device)
    scores = torch.empty(B, dtype=torch.float32, device=e.device)
    status = torch.empty(B, dtype=torch.int32, device=e.device)
    g._check(lib.gtnb_viterbi_dense_async(
        g.h, torch.cuda.current_stream(e.device).cuda_stream, B, T, Cn, e.data_ptr(), dtype,
        None if il is None else il.data_ptr(), kind, w.data_ptr(), paths.data_ptr(), scores.data_ptr(),
        status.data_ptr(), ws.data_ptr(), nbytes))
    return paths, scores, status


def asg_decode(emissions, transitions, input_lengths=None):
    """asg_viterbi without a host synchronisation: gtnb_viterbi_dense_async on the current stream (it may be captured
    in a CUDA graph).  emissions and transitions as in asg_viterbi; input_lengths: None or a [B] integer tensor on the
    emissions' device.  Returns device tensors (paths [B, T] int32, scores [B] float32, status [B] int32): status 0 is
    asg_viterbi's result, ties and NaN handling included; status 2 a length outside [0, T], with a NaN score and -1
    rows."""
    return _dense_decode("asg_decode", emissions, transitions, input_lengths, capi.DENSE_ASG)


def ngram_ctc_decode(emissions, transitions, input_lengths=None):
    """ngram_ctc_viterbi without a host synchronisation, as asg_decode is asg_viterbi's: (paths, scores, status) on
    the current stream; collapse(paths, blank) gives the transcripts."""
    return _dense_decode("ngram_ctc_decode", emissions, transitions, input_lengths, capi.DENSE_BIGRAM)


class BeamDecode(NamedTuple):
    """The beam decoders' results, device tensors: tokens [B, N, T] int32 (each transcript followed by -1), lengths
    [B, N] int32, scores [B, N] float32 and status [B] int32"""
    tokens: torch.Tensor
    lengths: torch.Tensor
    scores: torch.Tensor
    status: torch.Tensor


def _beam_inputs(emissions, transitions, input_lengths, kind):
    """The beam decoders' common inputs, checked: (emissions contiguous, transitions contiguous or None for CTC,
    input lengths as _decode_lengths gives them, the dtype code)"""
    assert emissions.is_cuda and emissions.dim() == 3
    assert emissions.dtype in _EMISSION_DTYPES, "emissions must be float32, bfloat16 or float16"
    e = emissions.contiguous()
    Cn = e.shape[2]
    w = None
    if kind != capi.DENSE_CTC:
        assert transitions.is_cuda and transitions.device == e.device and transitions.dtype == torch.float32
        assert transitions.numel() == (Cn * Cn if kind == capi.DENSE_BIGRAM else Cn + Cn * Cn)
        w = transitions.detach().contiguous()
    return e, w, _decode_lengths(e, input_lengths), _EMISSION_DTYPES[e.dtype]


@torch.no_grad()
def _beam_decode(name, emissions, transitions, input_lengths, kind, beam, nbest, blank):
    """gtnb_beam_decode_async on the current stream"""
    e, w, il, dtype = _beam_inputs(emissions, transitions, input_lengths, kind)
    B, T, Cn = e.shape
    g = _async_ctx(e.device, name)
    lib = capi.lib()
    ws, nbytes = _workspace(g, e.device, lib.gtnb_beam_decode_async_workspace, B, T, Cn, dtype, kind, int(beam),
                            int(nbest))
    tokens = torch.empty((B, nbest, T), dtype=torch.int32, device=e.device)
    lengths = torch.empty((B, nbest), dtype=torch.int32, device=e.device)
    scores = torch.empty((B, nbest), dtype=torch.float32, device=e.device)
    status = torch.empty(B, dtype=torch.int32, device=e.device)
    g._check(lib.gtnb_beam_decode_async(
        g.h, torch.cuda.current_stream(e.device).cuda_stream, B, T, Cn, e.data_ptr(), dtype,
        None if il is None else il.data_ptr(), kind, None if w is None else w.data_ptr(), int(blank), int(beam),
        int(nbest), tokens.data_ptr(), lengths.data_ptr(), scores.data_ptr(), status.data_ptr(), ws.data_ptr(), nbytes))
    return BeamDecode(tokens, lengths, scores, status)


def ctc_beam_decode(emissions, beam=16, nbest=1, input_lengths=None, blank=0):
    """Prefix beam search over transcripts scored by ctc_loss's numerator, forwardScore(intersect(ctcGraph(y), E_b)),
    through gtnb_beam_decode_async on the current stream, without a host synchronisation (it may be captured in a
    CUDA graph; the workspace comes from torch's allocator).

    emissions: [B, T, C] float32, bfloat16 or float16 CUDA tensor (read in place); input_lengths: None or a [B]
    integer tensor on its device.  beam K in [1, 64] beams, nbest N in [1, K] hypotheses, C <= 256; beyond, a
    RuntimeError.  Returns a BeamDecode of device tensors: tokens [B, N, T] (each transcript followed by -1), lengths
    [B, N], scores [B, N] (the numerator over the alignments that survived the beam, a lower bound of ctc_loss's
    numerator; -inf and length -1 for unused hypotheses) and status [B]: 0 a result, 1 a NaN or +inf emission, 2 a
    length outside [0, T] (both with NaN scores and -1 rows), 3 a tie decided the beam or the N-best order (the
    results stand, chosen by the tie rule of include/gtn_b200.h).  tokens[:, 0] and lengths[:, 0] go straight into
    edit_distance.
    """
    return _beam_decode("ctc_beam_decode", emissions, None, input_lengths, capi.DENSE_CTC, beam, nbest, blank)


def ngram_ctc_beam_decode(emissions, transitions, beam=16, nbest=1, input_lengths=None, blank=0):
    """ctc_beam_decode scored by ngram_ctc_loss's numerator, forwardScore(intersect(intersect(ctc_y, G), E_b)), with
    the learned bigram transitions [C*C] of ngram_ctc_loss (float32, on the emissions' device).  A NaN or +inf weight
    flags every utterance with T_b >= 1 (status 1)."""
    return _beam_decode("ngram_ctc_beam_decode", emissions, transitions, input_lengths, capi.DENSE_BIGRAM, beam,
                        nbest, blank)


def asg_beam_decode(emissions, transitions, beam=16, nbest=1, input_lengths=None):
    """ctc_beam_decode scored by asg_loss's numerator, forwardScore(compose(compose(A_y, G), E_b)), with asg_loss's
    transitions [C + C*C] (float32, on the emissions' device).  ASG has no blank: a frame stays on the last token or
    appends any token, the last one included (a repeated token).  Staying and repeating score a frame alike, so such
    ties are frequent and flagged with status 3."""
    return _beam_decode("asg_beam_decode", emissions, transitions, input_lengths, capi.DENSE_ASG, beam, nbest, 0)


class LanguageModel:
    """A token n-gram LM prepared once for the fused beam decoders (ctc_lm_beam_decode, ngram_ctc_lm_beam_decode,
    asg_lm_beam_decode): graph, a gtn_b200.gtn.Graph acceptor over the tokens [0, num_labels) with label num_labels
    for end of sentence and epsilon arcs as backoff (failure) arcs, resolved on the host into a dense table and
    uploaded to `device` (the current CUDA device by default) through gtnb_lm_create.  Its weights are baked in.  The
    graph's conditions (one start node, at most one arc per node and label, at most one epsilon arc per node and no
    cycle of them, no NaN or +inf weight) are in include/gtn_b200.h; a graph that breaks one raises a RuntimeError.

    Creating one allocates and synchronises, so it raises while a stream is capturing: build it before capture, and
    keep it alive as long as a captured CUDA graph that decodes with it."""

    def __init__(self, graph, num_labels, device=None):
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("LanguageModel: create it before capturing a CUDA graph (it allocates and "
                               "synchronises)")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.num_labels = int(num_labels)
        view, keep = _graph_view(graph)
        self._g = _async_ctx(self.device, "LanguageModel")
        h = C.c_void_p()
        rc = capi.lib().gtnb_lm_create(self._g.h, C.byref(view), self.num_labels, C.byref(h))
        del keep
        if rc != 0:
            raise RuntimeError("LanguageModel: %s" % capi.lib().gtnb_last_error(self._g.h).decode())
        self.h = h

    def __del__(self):
        h = getattr(self, "h", None)
        if h is not None and h.value:
            capi.lib().gtnb_lm_destroy(self._g.h, h)
            self.h = None


class LMBeamDecode(NamedTuple):
    """The fused beam decoders' results, device tensors: tokens [B, N, T] int32 (each transcript followed by -1),
    lengths [B, N] int32, scores [B, N] float32 (am + lm_weight * lm + token_bonus * length), am_scores [B, N] float32
    (the acoustic lower bound), lm_scores [B, N] float32 (the LM's score of the transcript, end weight included) and
    status [B] int32"""
    tokens: torch.Tensor
    lengths: torch.Tensor
    scores: torch.Tensor
    am_scores: torch.Tensor
    lm_scores: torch.Tensor
    status: torch.Tensor


@torch.no_grad()
def _lm_beam_decode(name, emissions, transitions, lm, lm_weight, token_bonus, beam, nbest, token_beam, input_lengths,
                    kind, blank):
    """gtnb_beam_decode_lm_async on the current stream"""
    e, w, il, dtype = _beam_inputs(emissions, transitions, input_lengths, kind)
    B, T, Cn = e.shape
    assert lm is None or isinstance(lm, LanguageModel)
    P = Cn if token_beam is None else int(token_beam)
    g = _async_ctx(e.device, name)
    lib = capi.lib()
    ws, nbytes = _workspace(g, e.device, lib.gtnb_beam_decode_lm_async_workspace, B, T, Cn, dtype, kind, int(beam),
                            int(nbest), P)
    tokens = torch.empty((B, nbest, T), dtype=torch.int32, device=e.device)
    lengths = torch.empty((B, nbest), dtype=torch.int32, device=e.device)
    scores = torch.empty((B, nbest), dtype=torch.float32, device=e.device)
    am = torch.empty((B, nbest), dtype=torch.float32, device=e.device)
    lms = torch.empty((B, nbest), dtype=torch.float32, device=e.device)
    status = torch.empty(B, dtype=torch.int32, device=e.device)
    g._check(lib.gtnb_beam_decode_lm_async(
        g.h, torch.cuda.current_stream(e.device).cuda_stream, B, T, Cn, e.data_ptr(), dtype,
        None if il is None else il.data_ptr(), kind, None if w is None else w.data_ptr(), int(blank), int(beam),
        int(nbest), None if lm is None else lm.h, float(lm_weight), float(token_bonus), P, tokens.data_ptr(),
        lengths.data_ptr(), scores.data_ptr(), am.data_ptr(), lms.data_ptr(), status.data_ptr(), ws.data_ptr(),
        nbytes))
    return LMBeamDecode(tokens, lengths, scores, am, lms, status)


def ctc_lm_beam_decode(emissions, lm=None, lm_weight=1.0, token_bonus=0.0, beam=16, nbest=1, token_beam=None,
                       input_lengths=None, blank=0):
    """ctc_beam_decode with LM shallow fusion, an insertion bonus and per-frame token pruning, through
    gtnb_beam_decode_lm_async on the current stream, without a host synchronisation (it may be captured in a CUDA
    graph).  Beams are ranked by am + (lm_weight * lmacc + token_bonus * length), lmacc the LanguageModel's resolved
    weights along the prefix; after the last frame each beam adds its end weight and the N-best are ranked by
    scores = am + lm_weight * lm + token_bonus * length.

    lm: a LanguageModel for C = emissions.shape[2] on the emissions' device, or None (no LM).  lm_weight >= 0 and
    token_bonus finite.  token_beam P in [1, C] (None: C, no pruning): each frame extends beams by its P most likely
    tokens only, blank excluded.  Returns an LMBeamDecode of device tensors; status as ctc_beam_decode's, where 3 also
    covers equal emissions at the P-th token boundary and equal final scores.  With lm None, token_bonus 0 and
    token_beam None, tokens, lengths, scores and status are those of ctc_beam_decode.
    """
    return _lm_beam_decode("ctc_lm_beam_decode", emissions, None, lm, lm_weight, token_bonus, beam, nbest, token_beam,
                           input_lengths, capi.DENSE_CTC, blank)


def ngram_ctc_lm_beam_decode(emissions, transitions, lm=None, lm_weight=1.0, token_bonus=0.0, beam=16, nbest=1,
                             token_beam=None, input_lengths=None, blank=0):
    """ctc_lm_beam_decode scored by ngram_ctc_loss's numerator, as ngram_ctc_beam_decode is ctc_beam_decode's"""
    return _lm_beam_decode("ngram_ctc_lm_beam_decode", emissions, transitions, lm, lm_weight, token_bonus, beam, nbest,
                           token_beam, input_lengths, capi.DENSE_BIGRAM, blank)


def asg_lm_beam_decode(emissions, transitions, lm=None, lm_weight=1.0, token_bonus=0.0, beam=16, nbest=1,
                       token_beam=None, input_lengths=None):
    """ctc_lm_beam_decode scored by asg_loss's numerator, as asg_beam_decode is ctc_beam_decode's (every token may be
    selected by token_beam: ASG has no blank)"""
    return _lm_beam_decode("asg_lm_beam_decode", emissions, transitions, lm, lm_weight, token_bonus, beam, nbest,
                           token_beam, input_lengths, capi.DENSE_ASG, 0)


class Lexicon:
    """A lexicon with an optional word n-gram LM, prepared once for the lexicon beam decoders
    (ctc_lexicon_beam_decode, ngram_ctc_lexicon_beam_decode, asg_lexicon_beam_decode) through gtnb_lexicon_create.

    spellings: (tokens, word id) pairs, each a non-empty token sequence in [0, num_labels) spelling a word in
    [0, num_words); a word may have several spellings, two words may not share one.  separator: a token that ends a word
    and is in no spelling (wav2letter's "|"), or None.  word_start: tokens that end the current word and begin a new
    spelling, allowed only at a spelling's position 0 (SentencePiece pieces with a leading space).  Every other token is
    an in-word token.  lm: the word LM, a gtn_b200.gtn.Graph or a (graph dict, weights) pair as arpa_graph returns,
    an acceptor over [0, num_words] with label num_words for end of sentence and epsilon arcs as backoff arcs (the
    conditions of include/gtn_b200.h), or None (every weight 0).  A lexicon or LM that breaks a condition raises a
    RuntimeError.

    Creating one allocates and synchronises, so it raises while a stream is capturing: build it before capture, and
    keep it alive as long as a captured CUDA graph that decodes with it."""

    def __init__(self, spellings, num_labels, num_words, separator=None, word_start=(), lm=None, device=None):
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("Lexicon: create it before capturing a CUDA graph (it allocates and synchronises)")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.num_labels, self.num_words = int(num_labels), int(num_words)
        cls = np.zeros(self.num_labels, np.int32)
        for c in word_start:
            cls[int(c)] = 2
        if separator is not None:
            cls[int(separator)] = 1
        toks, words, offs = [], [], [0]
        for y, w in spellings:
            toks.extend(int(c) for c in y)
            offs.append(len(toks))
            words.append(int(w))
        toks = np.asarray(toks, np.int32)
        offs = np.asarray(offs, np.int32)
        words = np.asarray(words, np.int32)
        view, keep = None, None
        if lm is not None:
            if isinstance(lm, tuple):
                G, w = lm
                view, keep = capi.make_view(G["flags"], G["src"], G["dst"], G["ilabel"], G.get("olabel", G["ilabel"]),
                                            np.asarray(w, np.float32))
            else:
                view, keep = _graph_view(lm)
        self._g = _async_ctx(self.device, "Lexicon")
        h = C.c_void_p()
        rc = capi.lib().gtnb_lexicon_create(self._g.h, self.num_labels, cls.ctypes.data, self.num_words, len(words),
                                            offs.ctypes.data, toks.ctypes.data if len(toks) else None,
                                            words.ctypes.data if len(words) else None,
                                            None if view is None else C.byref(view), C.byref(h))
        del keep
        if rc != 0:
            raise RuntimeError("Lexicon: %s" % capi.lib().gtnb_last_error(self._g.h).decode())
        self.h = h

    def __del__(self):
        h = getattr(self, "h", None)
        if h is not None and h.value:
            capi.lib().gtnb_lexicon_destroy(self._g.h, h)
            self.h = None


class LexiconBeamDecode(NamedTuple):
    """The lexicon beam decoders' results, device tensors: tokens [B, N, T] int32 (each transcript followed by -1),
    lengths [B, N] int32, words [B, N, T] int32 (each hypothesis's word ids followed by -1), word_counts [B, N] int32,
    scores [B, N] float32 (am + lm_weight * lm + word_bonus * word_count), am_scores [B, N] float32 (the acoustic lower
    bound), lm_scores [B, N] float32 (the word LM's score of the words, end weight included) and status [B] int32.
    words[:, 0] and word_counts[:, 0] go straight into edit_distance for a word error rate on the device."""
    tokens: torch.Tensor
    lengths: torch.Tensor
    words: torch.Tensor
    word_counts: torch.Tensor
    scores: torch.Tensor
    am_scores: torch.Tensor
    lm_scores: torch.Tensor
    status: torch.Tensor


@torch.no_grad()
def _lexicon_beam_decode(name, emissions, transitions, lexicon, lm_weight, word_bonus, beam, nbest, token_beam,
                         input_lengths, kind, blank):
    """gtnb_beam_decode_lexicon_async on the current stream"""
    e, w, il, dtype = _beam_inputs(emissions, transitions, input_lengths, kind)
    B, T, Cn = e.shape
    assert isinstance(lexicon, Lexicon)
    P = Cn if token_beam is None else int(token_beam)
    g = _async_ctx(e.device, name)
    lib = capi.lib()
    ws, nbytes = _workspace(g, e.device, lib.gtnb_beam_decode_lm_async_workspace, B, T, Cn, dtype, kind, int(beam),
                            int(nbest), P)
    i32, f32 = dict(dtype=torch.int32, device=e.device), dict(dtype=torch.float32, device=e.device)
    out = LexiconBeamDecode(torch.empty((B, nbest, T), **i32), torch.empty((B, nbest), **i32),
                            torch.empty((B, nbest, T), **i32), torch.empty((B, nbest), **i32),
                            torch.empty((B, nbest), **f32), torch.empty((B, nbest), **f32),
                            torch.empty((B, nbest), **f32), torch.empty(B, **i32))
    g._check(lib.gtnb_beam_decode_lexicon_async(
        g.h, torch.cuda.current_stream(e.device).cuda_stream, B, T, Cn, e.data_ptr(), dtype,
        None if il is None else il.data_ptr(), kind, None if w is None else w.data_ptr(), int(blank), int(beam),
        int(nbest), lexicon.h, float(lm_weight), float(word_bonus), P, out.tokens.data_ptr(), out.lengths.data_ptr(),
        out.scores.data_ptr(), out.am_scores.data_ptr(), out.lm_scores.data_ptr(), out.words.data_ptr(),
        out.word_counts.data_ptr(), out.status.data_ptr(), ws.data_ptr(), nbytes))
    return out


def ctc_lexicon_beam_decode(emissions, lexicon, lm_weight=1.0, word_bonus=0.0, beam=16, nbest=1, token_beam=None,
                            input_lengths=None, blank=0):
    """ctc_lm_beam_decode constrained by a Lexicon and fused with its word LM, through gtnb_beam_decode_lexicon_async
    on the current stream, without a host synchronisation (it may be captured in a CUDA graph).  Transcripts are
    sequences of spelled words (with separators or word-start tokens between them, as the lexicon's token classes
    say); beams are ranked by am + (lm_weight * (lmacc + smear) + word_bonus * words), lmacc the word LM's weights of
    the completed words and smear the best unigram weight of a word the pending prefix can still become.  After the
    last frame a beam completes its pending word (a beam inside a word is dropped), adds the end weight, and the
    N-best are ranked by scores = am + lm_weight * lm + word_bonus * words.

    lexicon: a Lexicon for C = emissions.shape[2] on the emissions' device; it may not spell with the blank or make it
    the separator.  lm_weight >= 0 and word_bonus finite; token_beam P in [1, C] (None: C).  Returns a
    LexiconBeamDecode of device tensors; status as ctc_lm_beam_decode's.  Hypotheses are distinct token transcripts,
    so two of them may spell the same words."""
    return _lexicon_beam_decode("ctc_lexicon_beam_decode", emissions, None, lexicon, lm_weight, word_bonus, beam, nbest,
                                token_beam, input_lengths, capi.DENSE_CTC, blank)


def ngram_ctc_lexicon_beam_decode(emissions, transitions, lexicon, lm_weight=1.0, word_bonus=0.0, beam=16, nbest=1,
                                  token_beam=None, input_lengths=None, blank=0):
    """ctc_lexicon_beam_decode scored by ngram_ctc_loss's numerator, as ngram_ctc_beam_decode is ctc_beam_decode's"""
    return _lexicon_beam_decode("ngram_ctc_lexicon_beam_decode", emissions, transitions, lexicon, lm_weight,
                                word_bonus, beam, nbest, token_beam, input_lengths, capi.DENSE_BIGRAM, blank)


def asg_lexicon_beam_decode(emissions, transitions, lexicon, lm_weight=1.0, word_bonus=0.0, beam=16, nbest=1,
                            token_beam=None, input_lengths=None):
    """ctc_lexicon_beam_decode scored by asg_loss's numerator, as asg_beam_decode is ctc_beam_decode's"""
    return _lexicon_beam_decode("asg_lexicon_beam_decode", emissions, transitions, lexicon, lm_weight, word_bonus,
                                beam, nbest, token_beam, input_lengths, capi.DENSE_ASG, 0)


def arpa_graph(path_or_lines, words):
    """An ARPA n-gram LM as the backoff graph Lexicon takes -> (graph dict of int32 / uint8 numpy arrays flags, src,
    dst, ilabel, olabel; float32 weights).

    words: the vocabulary, a list (word id = position) or a dict word -> id; V = its size.  Nodes are the histories:
    every n-gram of order < the LM's order that the file lists (with "<s>" as a history only), and the empty history.
    The start node is the history "<s>" (the empty history when the file has no "<s>" unigram).  An n-gram
    (h, x) with probability p becomes an arc from node h labelled x (V for "</s>") weighted ln p, to the longest
    suffix of h + x that is a node; an n-gram's backoff weight b becomes an epsilon arc from its node to the node of
    its history minus the oldest word, weighted ln b (ln 1 when the file lists none).  log10 values are converted to natural logs.  n-grams naming a
    word outside the vocabulary (other than "<s>" and "</s>") are dropped, and "<s>" is never a label."""
    if isinstance(path_or_lines, str):
        with open(path_or_lines, encoding="utf-8") as f:
            lines = f.read().splitlines()
    else:
        lines = list(path_or_lines)
    vocab = dict(words) if isinstance(words, dict) else {w: i for i, w in enumerate(words)}
    V = len(vocab)
    ln10 = float(np.log(10.0))
    grams = {}  # tuple of words -> (log10 p, log10 backoff or None)
    order = 0
    for line in lines:
        line = line.strip()
        if not line or line.startswith("\\") or line.startswith("ngram "):
            if line.startswith("\\") and line.endswith("-grams:"):
                order = int(line[1:line.index("-")])
            continue
        if order == 0:
            continue
        parts = line.split()
        if len(parts) < 1 + order:
            continue
        ng = tuple(parts[1:1 + order])
        if any(w not in vocab and w not in ("<s>", "</s>") for w in ng):
            continue
        bo = float(parts[1 + order]) if len(parts) > 1 + order else None
        grams[ng] = (float(parts[0]), bo)
    max_order = max((len(g) for g in grams), default=1)
    hist = {(): 0}
    for g in sorted(grams, key=len):
        if len(g) < max_order and g[-1] != "</s>" and g not in hist:
            hist[g] = len(hist)
    S = len(hist)
    src, dst, lab, w = [], [], [], []

    def node_of(h):
        while h not in hist:
            h = h[1:]
        return hist[h]
    for g, (lp, bo) in grams.items():
        if g[-1] != "<s>":
            h = g[:-1]
            if h in hist:
                x = V if g[-1] == "</s>" else vocab[g[-1]]
                src.append(hist[h]), lab.append(x), w.append(lp * ln10), dst.append(node_of(g))
    for g, s in hist.items():  # (a history without a listed backoff weight backs off with weight 1)
        if g:
            bo = grams.get(g, (0.0, None))[1]
            src.append(s), lab.append(-1), w.append((bo or 0.0) * ln10), dst.append(node_of(g[1:]))
    flags = np.full(S, 2, np.uint8)
    flags[hist.get(("<s>",), 0)] |= 1
    lab = np.asarray(lab, np.int32)
    return (dict(flags=flags, src=np.asarray(src, np.int32), dst=np.asarray(dst, np.int32), ilabel=lab,
                 olabel=lab.copy()), np.asarray(w, np.float32))


class EditDistance(NamedTuple):
    """edit_distance's results, device tensors of [B] int32 (alignments [B, N] / [B, M] int32, or None)"""
    distance: torch.Tensor
    substitutions: torch.Tensor
    insertions: torch.Tensor
    deletions: torch.Tensor
    hyp_units: torch.Tensor
    ref_units: torch.Tensor
    status: torch.Tensor
    hyp_align: Optional[torch.Tensor] = None
    ref_align: Optional[torch.Tensor] = None


def _edit_operand(name, x, dim, device):
    assert torch.is_tensor(x) and x.is_cuda and x.dim() == dim and not x.is_floating_point() and \
        not x.is_complex(), "%s must be an integer CUDA tensor of %d dimension(s)" % (name, dim)
    assert device is None or x.device == device, "%s must be on the hypotheses' device" % name
    return x.to(torch.int32).contiguous()


@torch.no_grad()
def edit_distance(hyp, hyp_lengths, ref, ref_lengths, word_sep=None, alignment=False):
    """Levenshtein distance between every hypothesis hyp[b, :hyp_lengths[b]] and reference ref[b, :ref_lengths[b]],
    through gtnb_edit_distance_async on the current stream, without a host synchronisation (it may be captured in a
    CUDA graph; the workspace comes from torch's allocator).  collapse(paths, blank)'s output is taken as hyp,
    hyp_lengths unchanged.

    hyp [B, N] and ref [B, M]: integer CUDA tensors on one device; the lengths: [B] integer tensors on that device.
    word_sep None: a unit is a token; an int: a unit is a word, a maximal run of tokens other than word_sep (no empty
    words), two words being equal when their token spans are.  The distance is -viterbiScore(compose(x, compose(edits,
    y))) of the reference's edit-distance example over the units, with unit costs.

    Each cell of the recurrence picks one predecessor, preferring the diagonal (a match or a substitution), then a
    deletion (a reference unit missing from the hypothesis), then an insertion (an extra hypothesis unit); the counts
    and the alignment follow that chain of predecessors, an optimal path that need not be the reference's viterbiPath.

    Returns an EditDistance of device tensors: distance, substitutions, insertions, deletions (summing to the
    distance), hyp_units, ref_units and status, all [B] int32, and with alignment=True hyp_align [B, N] (the reference
    unit each hypothesis unit is aligned to, -1 for an insertion) and ref_align [B, M] (the hypothesis unit, -1 for a
    deletion), both -1 beyond the unit counts and counted in units (words in word mode).  Status 0 is a result;
    status 2 a length outside [0, N] or [0, M], with -1 in every output of that pair.  An error rate (WER, or CER at
    token level) is distance[ok].sum() / ref_units[ok].sum() with ok = status == 0.

    N or M above 4096 raises RuntimeError.
    """
    h = _edit_operand("hyp", hyp, 2, None)
    dev = hyp.device
    r = _edit_operand("ref", ref, 2, dev)
    hl = _edit_operand("hyp_lengths", hyp_lengths, 1, dev)
    rl = _edit_operand("ref_lengths", ref_lengths, 1, dev)
    B, N = h.shape
    M = r.shape[1]
    assert r.shape[0] == B and hl.shape == (B,) and rl.shape == (B,), "one hypothesis, reference and length per pair"
    sep = -1 if word_sep is None else int(word_sep)
    assert sep >= -1, "word_sep must be None or a non-negative token"
    g = _async_ctx(dev, "edit_distance")
    lib = capi.lib()
    ws, nbytes = _workspace(g, dev, lib.gtnb_edit_distance_async_workspace, B, N, M, sep, int(bool(alignment)))
    dist, status = (torch.empty(B, dtype=torch.int32, device=dev) for _ in range(2))
    ops, units = torch.empty((B, 3), dtype=torch.int32, device=dev), torch.empty((B, 2), dtype=torch.int32, device=dev)
    ha = torch.empty((B, N), dtype=torch.int32, device=dev) if alignment else None
    ra = torch.empty((B, M), dtype=torch.int32, device=dev) if alignment else None
    g._check(lib.gtnb_edit_distance_async(
        g.h, torch.cuda.current_stream(dev).cuda_stream, B, h.data_ptr(), N, hl.data_ptr(), r.data_ptr(), M,
        rl.data_ptr(), sep, dist.data_ptr(), ops.data_ptr(), units.data_ptr(), status.data_ptr(),
        None if ha is None else ha.data_ptr(), None if ra is None else ra.data_ptr(),
        ws.data_ptr(), nbytes))
    return EditDistance(dist, ops[:, 0], ops[:, 1], ops[:, 2], units[:, 0], units[:, 1], status, ha, ra)


def _graph_view(g):
    """capi view of a gtn_b200.gtn.Graph built on the host, in its own arc-list order"""
    from . import _gtn
    d = _gtn.arc_lists(g)
    return capi.make_view(d["flags"], d["src"], d["dst"], d["ilabel"], d["olabel"], d["weights"], d["in_ptr"],
                          d["in_arcs"], d["out_ptr"], d["out_arcs"], d["start"], d["accept"])


class _GraphCall:
    """One batch of user graphs as the graph criteria and decoders hand it to the C ABI: the emissions (e, B, T, C),
    the context of the current stream (g), input_lengths (il: a pointer or None), the graphs' views (kept alive here)
    and their GraphView array (arr), the arc weights (w: a device pointer or None) and, with arc_grads and weights,
    the buffer the call writes the weights' gradient into (ag) and the utterance of every arc (owner)."""

    def __init__(self, emissions, graphs, weights, input_lengths, arc_grads):
        assert emissions.is_cuda and emissions.dtype == torch.float32 and emissions.dim() == 3
        self.e = e = emissions.contiguous()
        B, T, Cn = e.shape
        self.B, self.T, self.C = B, T, Cn
        if graphs is None:  # a decoder without target graphs
            graphs = []
        else:
            assert len(graphs) == B
        self.views = [_graph_view(g) for g in graphs]
        counts = [v.num_arcs for v, _ in self.views]
        self.n_arcs = sum(counts)
        self.arr = (capi.GraphView * max(B, 1))(*[v for v, _ in self.views])
        self.weights = self.ag = self.owner = None
        if weights is not None:
            assert weights.is_cuda and weights.device == e.device and weights.dtype == torch.float32
            assert weights.numel() == self.n_arcs
            self.weights = weights.detach().contiguous()
            if arc_grads:
                self.ag = torch.empty(max(self.n_arcs, 1), dtype=torch.float32, device=e.device)  # written by the call
                # utterance of every arc, for a per-utterance upstream gradient (reduction "none")
                self.owner = torch.repeat_interleave(torch.arange(B), torch.tensor(counts, dtype=torch.long)).to(
                    e.device)
        self.w = None if self.weights is None else self.weights.data_ptr()
        self.current = torch.cuda.current_stream(e.device)
        self.g = _ctx_for(e.device, self.current.cuda_stream)
        self.lengths = _lengths(input_lengths, B)
        self.il = None if self.lengths is None else self.lengths.ctypes.data_as(capi._i32p)

    def loss_output(self, ctx, losses, reduction, weights):
        """the criterion's output from the B host losses; ctx keeps what _weight_backward needs"""
        # (the arc gradient is computed here, neither an input nor an output: held on ctx)
        ctx.ag = None if self.ag is None else self.ag[:self.n_arcs].view_as(weights)
        ctx.owner = self.owner
        ctx.reduction = reduction
        ctx.B = self.B
        out = torch.from_numpy(losses).to(self.e.device)
        return out.mean() if reduction == "mean" else out

    def viterbi(self, call):
        """(paths, scores, arcs) of call(paths, arcs, scores), a graph Viterbi C call on device pointers"""
        B, T, device = self.B, self.T, self.e.device
        paths = torch.empty((B, T), dtype=torch.int32, device=device)  # every entry is written by the call
        arcs = torch.empty((B, T), dtype=torch.int32, device=device)
        scores = torch.empty(B, dtype=torch.float32, device=device)
        # the context's stream is the current stream unless that is the legacy default stream: order the two both ways
        ctx_stream = torch.cuda.ExternalStream(capi.lib().gtnb_ctx_stream(self.g.h), device=device)
        ctx_stream.wait_stream(self.current)
        self.g._check(call(paths.data_ptr(), arcs.data_ptr(), scores.data_ptr()))
        self.current.wait_stream(ctx_stream)
        return paths, scores, arcs


def _weight_backward(ctx, grad_output):
    """the arc-weight gradient of the graph criteria times the upstream gradient (None without weights)"""
    ag = ctx.ag
    if ag is None:
        return None
    if ctx.reduction == "mean":
        return ag * (grad_output / ctx.B)
    # reduction "none": every graph belongs to one utterance, so its arcs take that utterance's upstream gradient
    return ag * grad_output.reshape(-1)[ctx.owner].view_as(ag)


class GraphLossFunction(torch.autograd.Function):
    """loss_b = forwardScore(E_b) - forwardScore(intersect(A_b, E_b)) with one target graph A_b per utterance
    (bindings/python/examples/pytorch_loss.py, the word-decomposition examples), through gtnb_graph_loss.

    emissions: float32 CUDA tensor [B, T, C]; graphs: B gtn_b200.gtn.Graph built on the host, matched on their
    olabels (epsilon arcs must be removed first); input_lengths: None, a list or an int tensor (any device).
    weights: None (the graphs' own weights, no gradient) or a float32 CUDA tensor of sum_b A_b elements, the arc
    weights of all graphs in batch order and Graph arc numbering, which replace the graphs' weights and receive their
    gradient (gather it from a parameter to learn, e.g., decomposition weights).  Everything runs on the current
    stream of the emissions' device; the emission and weight gradients stay on the device, only the B losses are
    copied to the host.
    """

    @staticmethod
    def forward(ctx, emissions, weights, graphs, input_lengths=None, reduction="mean"):
        c = _GraphCall(emissions, graphs, weights, input_lengths, arc_grads=True)
        losses = np.zeros(c.B, np.float32)
        grad = torch.empty_like(c.e)  # every row is written by the call
        c.g._check(capi.lib().gtnb_graph_loss(
            c.g.h, c.B, c.T, c.C, c.e.data_ptr(), 1, c.il, c.arr, c.w, 1, losses.ctypes.data_as(capi._f32p),
            grad.data_ptr(), 1, None if c.ag is None else c.ag.data_ptr(), 1))
        ctx.save_for_backward(grad)
        return c.loss_output(ctx, losses, reduction, weights)

    @staticmethod
    def backward(ctx, grad_output):
        (grad,) = ctx.saved_tensors
        if ctx.reduction == "mean":
            egrad = grad * (grad_output / ctx.B)
        else:
            egrad = grad * grad_output.reshape(-1).view(-1, 1, 1)
        return egrad, _weight_backward(ctx, grad_output), None, None, None


def graph_loss(emissions, graphs, input_lengths=None, weights=None, reduction="mean"):
    return GraphLossFunction.apply(emissions, weights, graphs, input_lengths, reduction)


def _transitions_forward(ctx, emissions, transitions, weights, graphs, input_lengths, reduction, allreduce, n_tg,
                         call):
    """the forward of graph_transitions_loss and sparse_transitions_loss: call(c, tw, losses, grad, tg) makes the C
    call, with a transition gradient buffer of n_tg floats"""
    c = _GraphCall(emissions, graphs, weights, input_lengths, arc_grads=True)
    assert transitions.is_cuda and transitions.device == c.e.device and transitions.dtype == torch.float32
    tw = transitions.detach().contiguous()
    losses = np.zeros(c.B, np.float32)
    grad = torch.empty_like(c.e)  # every row is written by the call
    tg = torch.empty(n_tg, dtype=torch.float32, device=c.e.device)
    c.g._check(call(c, tw, losses, grad, tg))
    tg = tg[:transitions.numel()].view_as(transitions)
    _allreduce_transitions(ctx, tg, allreduce)
    ctx.save_for_backward(grad, tg)
    return c.loss_output(ctx, losses, reduction, weights)


class GraphTransitionsLossFunction(torch.autograd.Function):
    """graph_loss's user target graphs with asg_loss's or ngram_ctc_loss's learned transitions, through
    gtnb_graph_transitions_loss:
        kind "asg":    loss_b = forwardScore(compose(E_b, G)) - forwardScore(compose(compose(A_b, G), E_b))
        kind "bigram": loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(A_b, G), E_b))
    G: asg_loss's transitions graph (transitions [C + C*C]: start weights, then the C x C matrix, row = destination
    label) or ngram_ctc_loss's bigram graph (transitions [C*C], every state starts and accepts).  The graphs, weights
    and input_lengths are graph_loss's.  transitions: float32 CUDA tensor on the emissions' device.  The emission,
    transition and weight gradients stay on the device; only the B losses are copied to the host.  The transition
    gradient is summed over the ranks as asg_loss does (allreduce).
    """

    @staticmethod
    def forward(ctx, emissions, transitions, weights, graphs, kind="asg", input_lengths=None, reduction="mean",
                allreduce=True):
        assert kind in ("asg", "bigram")
        kid = capi.DENSE_BIGRAM if kind == "bigram" else capi.DENSE_ASG
        Cn = emissions.shape[-1]
        assert transitions.numel() == (Cn * Cn if kid == capi.DENSE_BIGRAM else Cn + Cn * Cn)
        return _transitions_forward(
            ctx, emissions, transitions, weights, graphs, input_lengths, reduction, allreduce, transitions.numel(),
            lambda c, tw, losses, grad, tg: capi.lib().gtnb_graph_transitions_loss(
                c.g.h, c.B, c.T, c.C, c.e.data_ptr(), 1, c.il, c.arr, c.w, 1, kid, tw.data_ptr(), 1,
                losses.ctypes.data_as(capi._f32p), grad.data_ptr(), 1, None if c.ag is None else c.ag.data_ptr(), 1,
                tg.data_ptr(), 1))

    @staticmethod
    def backward(ctx, grad_output):
        egrad, tgrad = _transition_backward(ctx, grad_output)
        return egrad, tgrad, _weight_backward(ctx, grad_output), None, None, None, None, None


def graph_transitions_loss(emissions, transitions, graphs, kind="asg", input_lengths=None, weights=None,
                           reduction="mean", allreduce=True):
    return GraphTransitionsLossFunction.apply(emissions, transitions, weights, graphs, kind, input_lengths, reduction,
                                              allreduce)


class SparseTransitionsLossFunction(GraphTransitionsLossFunction):
    """graph_loss's user target graphs with a learned transition graph G of any shape (an n-gram graph of any order,
    a pruned token LM, an HMM topology), through gtnb_sparse_transitions_loss:
        loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(A_b, G), E_b))
    transitions_graph: G, a gtn_b200.gtn.Graph acceptor without epsilon arcs, whose own weights are ignored;
    transitions: float32 CUDA tensor of G.num_arcs() weights in G's arc numbering, on the emissions' device.  The
    graphs, weights, input_lengths, reduction and allreduce are graph_transitions_loss's; so is the backward.
    large_transitions=True: a G of up to 16 384 states and 262 144 arcs (a full trigram at C = 64) keeps the device
    route, swept by one thread-block cluster per utterance (_clustered); a smaller G is not affected.
    """

    @staticmethod
    def forward(ctx, emissions, transitions, weights, graphs, transitions_graph, input_lengths=None, reduction="mean",
                allreduce=True, large_transitions=False):
        gv = _graph_view(transitions_graph)
        assert transitions.numel() == gv[0].num_arcs
        return _transitions_forward(
            ctx, emissions, transitions, weights, graphs, input_lengths, reduction, allreduce,
            max(transitions.numel(), 1),
            lambda c, tw, losses, grad, tg: _clustered(
                c.g, large_transitions, lambda: capi.lib().gtnb_sparse_transitions_loss(
                    c.g.h, c.B, c.T, c.C, c.e.data_ptr(), 1, c.il, c.arr, c.w, 1, C.byref(gv[0]), tw.data_ptr(), 1,
                    losses.ctypes.data_as(capi._f32p), grad.data_ptr(), 1,
                    None if c.ag is None else c.ag.data_ptr(), 1, tg.data_ptr(), 1)))

    @staticmethod
    def backward(ctx, grad_output):
        return GraphTransitionsLossFunction.backward(ctx, grad_output) + (None,)


def sparse_transitions_loss(emissions, transitions, transitions_graph, graphs, input_lengths=None, weights=None,
                            reduction="mean", allreduce=True, large_transitions=False):
    return SparseTransitionsLossFunction.apply(emissions, transitions, weights, graphs, transitions_graph,
                                               input_lengths, reduction, allreduce, large_transitions)


class BackoffTransitionsLossFunction(GraphTransitionsLossFunction):
    """sparse_transitions_loss with a backoff transition graph, through gtnb_backoff_transitions_loss: G may have
    epsilon arcs (ilabel == olabel == gtn.epsilon), the backoff arcs of a pruned n-gram token LM, which move G without
    consuming a frame and weigh their own transitions entry; the score sums over every path, the backoff paths
    included.  The arguments and the backward are sparse_transitions_loss's; an epsilon-free G gives its results.
    large_transitions=True: a backoff G beyond one CTA (over 4096 states or 32 768 emitting plus epsilon arcs), up to
    16 384 states and 262 144 arcs, keeps the device route, its denominator swept by one thread-block cluster per
    utterance (_clustered); a smaller G is not affected.
    """

    @staticmethod
    def forward(ctx, emissions, transitions, weights, graphs, transitions_graph, input_lengths=None, reduction="mean",
                allreduce=True, large_transitions=False):
        gv = _graph_view(transitions_graph)
        assert transitions.numel() == gv[0].num_arcs
        return _transitions_forward(
            ctx, emissions, transitions, weights, graphs, input_lengths, reduction, allreduce,
            max(transitions.numel(), 1),
            lambda c, tw, losses, grad, tg: _clustered(
                c.g, large_transitions, lambda: capi.lib().gtnb_backoff_transitions_loss(
                    c.g.h, c.B, c.T, c.C, c.e.data_ptr(), 1, c.il, c.arr, c.w, 1, C.byref(gv[0]), tw.data_ptr(), 1,
                    losses.ctypes.data_as(capi._f32p), grad.data_ptr(), 1,
                    None if c.ag is None else c.ag.data_ptr(), 1, tg.data_ptr(), 1)))

    @staticmethod
    def backward(ctx, grad_output):
        return GraphTransitionsLossFunction.backward(ctx, grad_output) + (None,)


def backoff_transitions_loss(emissions, transitions, transitions_graph, graphs, input_lengths=None, weights=None,
                             reduction="mean", allreduce=True, large_transitions=False):
    return BackoffTransitionsLossFunction.apply(emissions, transitions, weights, graphs, transitions_graph,
                                                input_lengths, reduction, allreduce, large_transitions)


@torch.no_grad()
def graph_viterbi(emissions, graphs, input_lengths=None, weights=None):
    """Best path of compose(A_b, E_b) for every utterance, A_b = graphs[b] (viterbiPath / viterbiScore of the lattice
    graph_loss sums over), through gtnb_graph_viterbi: the alignment the model picks within its own target graph, e.g.
    a forced alignment with CTC, word-piece decomposition or hand-built graphs.

    emissions: float32 CUDA tensor [B, T, C]; graphs, input_lengths and weights as in graph_loss (weights: None, or
    a float32 CUDA tensor of sum_b A_b arc weights that replace the graphs' own).  Returns (paths [B, T] int32, the
    matched label of the arc taken at every frame; scores [B] float32, viterbiScore; arcs [B, T] int32, that arc's id
    in graphs[b]), all -1 beyond T_b and where there is no accepting path (score -inf), as CUDA tensors on the
    emissions' device, written on the current stream.  Ties are broken as the reference breaks them.
    collapse(paths, blank) turns the paths into transcripts.
    """
    c = _GraphCall(emissions, graphs, weights, input_lengths, arc_grads=False)
    return c.viterbi(lambda paths, arcs, scores: capi.lib().gtnb_graph_viterbi(
        c.g.h, c.B, c.T, c.C, c.e.data_ptr(), 1, c.il, c.arr, c.w, 1, paths, arcs, scores, 1))


@torch.no_grad()
def graph_transitions_viterbi(emissions, transitions, graphs, kind="asg", input_lengths=None, weights=None):
    """Best path of graph_transitions_loss's numerator for every utterance, through gtnb_graph_transitions_viterbi:
        kind "asg":    viterbiPath / viterbiScore of compose(compose(A_b, G), E_b)
        kind "bigram": viterbiPath / viterbiScore of intersect(intersect(A_b, G), E_b)
    the decomposition and frame-level alignment a model trained with graph_transitions_loss picks within its own
    target graph.  emissions, transitions, graphs, kind, input_lengths and weights as in graph_transitions_loss.
    Returns (paths [B, T] int32, the label of the arc taken at every frame; scores [B] float32, viterbiScore; arcs
    [B, T] int32, that arc's id in graphs[b]), all -1 beyond T_b and where there is no accepting path (score -inf), as
    CUDA tensors on the emissions' device, written on the current stream.  Ties are broken as the reference breaks
    them.  collapse(paths, blank) turns the paths into transcripts.
    """
    assert kind in ("asg", "bigram")
    c = _GraphCall(emissions, graphs, weights, input_lengths, arc_grads=False)
    assert transitions.is_cuda and transitions.device == c.e.device and transitions.dtype == torch.float32
    kid = capi.DENSE_BIGRAM if kind == "bigram" else capi.DENSE_ASG
    assert transitions.numel() == (c.C * c.C if kid == capi.DENSE_BIGRAM else c.C + c.C * c.C)
    tw = transitions.detach().contiguous()
    return c.viterbi(lambda paths, arcs, scores: capi.lib().gtnb_graph_transitions_viterbi(
        c.g.h, c.B, c.T, c.C, c.e.data_ptr(), 1, c.il, c.arr, c.w, 1, kid, tw.data_ptr(), 1, paths, arcs, scores, 1))


def _sparse_transitions(c, transitions, transitions_graph):
    """(G's view pair, trans_w on the device) of the sparse Viterbi calls"""
    assert transitions.is_cuda and transitions.device == c.e.device and transitions.dtype == torch.float32
    gv = _graph_view(transitions_graph)
    assert transitions.numel() == gv[0].num_arcs
    # (an empty G: a one-element buffer that is never read)
    tw = transitions.detach().contiguous() if transitions.numel() else torch.zeros(1, device=c.e.device)
    return gv, tw


@torch.no_grad()
def sparse_viterbi(emissions, transitions, transitions_graph, input_lengths=None, large_transitions=False):
    """Best path of intersect(E_b, G) for every utterance, G the learned transition graph of sparse_transitions_loss
    (an n-gram graph of any order, a pruned token LM, an HMM topology), through gtnb_viterbi_sparse: the decode of a
    model trained with that loss.  emissions, transitions, transitions_graph and input_lengths as in
    sparse_transitions_loss.  Returns (paths [B, T] int32, the label of every frame; scores [B] float32, viterbiScore;
    arcs [B, T] int32, the G arc taken at every frame, i.e. the state sequence), all -1 beyond T_b and where there is
    no accepting path (score -inf), as CUDA tensors on the emissions' device, written on the current stream; only
    input_lengths and one status word per utterance visit the host.  Ties are broken as the reference breaks them.
    collapse(paths, blank) turns the paths into transcripts.  large_transitions as in sparse_transitions_loss.
    """
    c = _GraphCall(emissions, None, None, input_lengths, arc_grads=False)
    gv, tw = _sparse_transitions(c, transitions, transitions_graph)
    return c.viterbi(lambda paths, arcs, scores: _clustered(
        c.g, large_transitions, lambda: capi.lib().gtnb_viterbi_sparse(
            c.g.h, c.B, c.T, c.C, c.e.data_ptr(), 1, c.il, C.byref(gv[0]), tw.data_ptr(), 1, paths, arcs, scores, 1)))


@torch.no_grad()
def backoff_viterbi(emissions, transitions, transitions_graph, input_lengths=None, large_transitions=False):
    """Best path of intersect(E_b, G) for every utterance, G the backoff transition graph of backoff_transitions_loss
    (epsilon arcs allowed), through gtnb_viterbi_backoff: the decode of a model trained with that loss.  The arguments
    and outputs are sparse_viterbi's.  arcs[b, t] is the emitting G arc taken at frame t: an epsilon arc uses no frame
    and is not reported.  Ties are broken as the reference breaks them.  large_transitions as in
    backoff_transitions_loss.
    """
    c = _GraphCall(emissions, None, None, input_lengths, arc_grads=False)
    gv, tw = _sparse_transitions(c, transitions, transitions_graph)
    return c.viterbi(lambda paths, arcs, scores: _clustered(
        c.g, large_transitions, lambda: capi.lib().gtnb_viterbi_backoff(
            c.g.h, c.B, c.T, c.C, c.e.data_ptr(), 1, c.il, C.byref(gv[0]), tw.data_ptr(), 1, paths, arcs, scores, 1)))


@torch.no_grad()
def sparse_transitions_viterbi(emissions, transitions, transitions_graph, graphs, input_lengths=None, weights=None,
                               large_transitions=False):
    """Best path of sparse_transitions_loss's numerator, intersect(intersect(A_b, G), E_b), for every utterance,
    through gtnb_sparse_transitions_viterbi: the decomposition and frame-level alignment a model trained with
    sparse_transitions_loss picks within its own target graph.  The arguments are sparse_transitions_loss's.  Returns
    (paths [B, T] int32, the label of the arc taken at every frame; scores [B] float32, viterbiScore; arcs [B, T]
    int32, that arc's id in graphs[b]), all -1 beyond T_b and where there is no accepting path (score -inf), as CUDA
    tensors on the emissions' device, written on the current stream.  Ties are broken as the reference breaks them.
    large_transitions as in sparse_transitions_loss.
    """
    c = _GraphCall(emissions, graphs, weights, input_lengths, arc_grads=False)
    gv, tw = _sparse_transitions(c, transitions, transitions_graph)
    return c.viterbi(lambda paths, arcs, scores: _clustered(
        c.g, large_transitions, lambda: capi.lib().gtnb_sparse_transitions_viterbi(
            c.g.h, c.B, c.T, c.C, c.e.data_ptr(), 1, c.il, c.arr, c.w, 1, C.byref(gv[0]), tw.data_ptr(), 1, paths,
            arcs, scores, 1)))


@torch.no_grad()
def backoff_transitions_viterbi(emissions, transitions, transitions_graph, graphs, input_lengths=None, weights=None,
                                large_transitions=False):
    """Best path of backoff_transitions_loss's numerator, intersect(intersect(A_b, G), E_b), for every utterance,
    through gtnb_backoff_transitions_viterbi: the decomposition and frame-level alignment a model trained with
    backoff_transitions_loss picks within its own target graph, under the backoff LM it was trained with.  The
    arguments are backoff_transitions_loss's and the outputs sparse_transitions_viterbi's: arcs[b, t] is the arc of
    graphs[b] taken at frame t, and an epsilon arc of G uses no frame and is not reported.  Ties are broken as the
    reference breaks them.  large_transitions as in backoff_transitions_loss.
    """
    c = _GraphCall(emissions, graphs, weights, input_lengths, arc_grads=False)
    gv, tw = _sparse_transitions(c, transitions, transitions_graph)
    return c.viterbi(lambda paths, arcs, scores: _clustered(
        c.g, large_transitions, lambda: capi.lib().gtnb_backoff_transitions_viterbi(
            c.g.h, c.B, c.T, c.C, c.e.data_ptr(), 1, c.il, c.arr, c.w, 1, C.byref(gv[0]), tw.data_ptr(), 1, paths,
            arcs, scores, 1)))
