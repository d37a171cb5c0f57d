"""PyTorch criteria on CUDA tensors, end to end on the device (SURVEY.md section 8(f) rank 1).

The reference's example (bindings/python/examples/pytorch_loss.py:19-102) moves the emissions to
the CPU, builds one Graph per utterance inside gtn.parallel_for and copies the gradients back.
Here the [B, T, C] CUDA tensor goes straight into the C ABI (`gtnb_ctc_loss`, device pointers in,
device gradients out) on the tensor's own CUDA stream; only the B losses visit the host.
"""
import ctypes as C

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


def _allreduce_transitions(ctx, tg, allreduce):
    """Sum the transition gradient tg over the ranks when torch.distributed is initialised (the multi-GPU form of
    Graph::addGrad under grad_lock, graph.cpp:96-100); ctx.world is the number of ranks summed over."""
    ctx.world = 1
    if allreduce and torch.distributed.is_available() and torch.distributed.is_initialized():
        torch.distributed.all_reduce(tg, op=torch.distributed.ReduceOp.SUM)
        ctx.world = torch.distributed.get_world_size()


def _transition_backward(ctx, grad_output):
    """(emission gradient, transition gradient) of asg_loss / ngram_ctc_loss times the upstream gradient"""
    grad, tg = ctx.saved_tensors
    if ctx.reduction == "mean":
        # the mean over the GLOBAL batch when the transition gradient was summed over the ranks
        scale = grad_output / ctx.B
        return grad * scale, tg * (scale / ctx.world)
    # reduction "none": the incoming gradient is per utterance; the transition gradient was already summed
    # over the batch inside the kernel, which is only the chain rule's answer for a uniform grad_output
    assert bool((grad_output == grad_output.flatten()[0]).all()), \
        "reduction='none' supports a uniform upstream gradient (sum / mean of the losses)"
    return grad * grad_output.view(-1, 1, 1), tg * grad_output.flatten()[0]


class CTCLossFunction(torch.autograd.Function):
    """loss_b = forwardScore(e_b) - forwardScore(intersect(ctcGraph(target_b), e_b))  (benchmarks/ctc.cpp:150-158).

    emissions: float32 CUDA tensor [B, T, C] (unnormalised scores are fine: the normaliser is part of the loss);
    targets: list of 1-D int sequences; input_lengths: None (T frames each), a list or an int tensor (any device):
    e_b is then the first input_lengths[b] frames, and the gradient of the padding frames is 0.  Returns the mean
    loss over the batch (reduction="mean") or the [B] vector.
    """

    @staticmethod
    def forward(ctx, emissions, targets, blank=0, reduction="mean", input_lengths=None):
        assert emissions.is_cuda and emissions.dtype == torch.float32 and emissions.dim() == 3
        e = emissions.contiguous()
        B, T, Cn = e.shape
        stream = torch.cuda.current_stream(e.device).cuda_stream
        g = _ctx_for(e.device, stream)
        cat, lens = capi._cat_targets(targets)
        il = _lengths(input_lengths, B)
        losses = np.zeros(B, np.float32)
        grad = torch.empty_like(e)  # (with input_lengths the call zeroes the padding rows)
        g._check(capi.lib().gtnb_ctc_loss(
            g.h, B, T, Cn, e.data_ptr(), 1, None if il is None else il.ctypes.data_as(capi._i32p),
            cat.ctypes.data_as(capi._i32p),
            lens.ctypes.data_as(capi._i32p), int(blank), losses.ctypes.data_as(capi._f32p),
            grad.data_ptr(), 1))
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
        return grad * grad_output.view(-1, 1, 1), None, None, None, None


def ctc_loss(emissions, targets, blank=0, reduction="mean", input_lengths=None):
    return CTCLossFunction.apply(emissions, targets, blank, reduction, input_lengths)


class ASGLossFunction(torch.autograd.Function):
    """loss_b = forwardScore(compose(e_b, transitions)) - forwardScore(compose(compose(fal_b, transitions), e_b))
    (examples/asg.cpp:59-81, test/criterion_test.cpp:244-305) with ONE learned transitions graph shared by the
    minibatch -- and by all ranks: with torch.distributed initialised, the transition gradient of the local shard
    is all-reduced (sum) over NCCL, the multi-GPU form of Graph::addGrad under grad_lock (graph.cpp:96-100).

    emissions: float32 CUDA tensor [B, T, C]; transitions: float32 tensor [C + C*C] (start weights, then the
    C x C matrix, row = destination label) on any device; targets: list of 1-D int sequences.

    input_lengths: None (T frames each), a list or an int tensor (any device).  When given, e_b is the first
    input_lengths[b] frames (the gradient of the padding frames is 0) and the call goes through gtnb_asg_loss_ex
    on device pointers: transitions must then be a float32 CUDA tensor on the emissions' device, and the
    transition gradient stays on the device.
    """

    @staticmethod
    def forward(ctx, emissions, transitions, targets, reduction="mean", allreduce=True, input_lengths=None):
        assert emissions.is_cuda and emissions.dtype == torch.float32 and emissions.dim() == 3
        e = emissions.contiguous()
        B, T, Cn = e.shape
        assert transitions.numel() == Cn + Cn * Cn
        stream = torch.cuda.current_stream(e.device).cuda_stream
        g = _ctx_for(e.device, stream)
        cat, lens = capi._cat_targets(targets)
        losses = np.zeros(B, np.float32)
        if input_lengths is not None:
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


def asg_loss(emissions, transitions, targets, reduction="mean", allreduce=True, input_lengths=None):
    return ASGLossFunction.apply(emissions, transitions, targets, reduction, allreduce, input_lengths)


class NgramCTCLossFunction(torch.autograd.Function):
    """CTC with a learned bigram transition graph G (benchmarks/ctc.cpp:107-134, timeNgramCtc):
        loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(ctc_b, G), E_b))
    G: C nodes, all start and accept, arc j -> i with label i and weight transitions[i, j] (row = destination
    label, column = source label), shared by the minibatch and, with torch.distributed initialised, by all ranks
    (the transition gradient is all-reduced over NCCL, as asg_loss does).

    emissions: float32 CUDA tensor [B, T, C]; transitions: float32 CUDA tensor of C*C elements ([C, C] or flat) on
    the same device; targets: list of 1-D int sequences; input_lengths: None, a list or an int tensor (any
    device).  Everything runs on the current stream of the emissions' device, device pointers in and out: only
    the B losses (and input_lengths, when given on the GPU) are copied to the host.
    """

    @staticmethod
    def forward(ctx, emissions, transitions, targets, input_lengths=None, blank=0, reduction="mean", allreduce=True):
        assert emissions.is_cuda and emissions.dtype == torch.float32 and emissions.dim() == 3
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
        g._check(capi.lib().gtnb_ngram_ctc_loss(
            g.h, B, T, Cn, e.data_ptr(), 1, None if il is None else il.ctypes.data_as(capi._i32p), w.data_ptr(), 1,
            cat.ctypes.data_as(capi._i32p), lens.ctypes.data_as(capi._i32p), int(blank),
            losses.ctypes.data_as(capi._f32p), grad.data_ptr(), 1, tg.data_ptr(), 1))
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


def ngram_ctc_loss(emissions, transitions, targets, input_lengths=None, blank=0, reduction="mean", allreduce=True):
    return NgramCTCLossFunction.apply(emissions, transitions, targets, input_lengths, blank, reduction, allreduce)


def _graph_view(g):
    """capi view of a gtn_b200.gtn.Graph built on the host, in its own arc-list order"""
    from . import _gtn
    d = _gtn.arc_lists(g)
    return capi.make_view(d["flags"], d["src"], d["dst"], d["ilabel"], d["olabel"], d["weights"], d["in_ptr"],
                          d["in_arcs"], d["out_ptr"], d["out_arcs"], d["start"], d["accept"])


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
        assert emissions.is_cuda and emissions.dtype == torch.float32 and emissions.dim() == 3
        e = emissions.contiguous()
        B, T, Cn = e.shape
        assert len(graphs) == B
        views = [_graph_view(g) for g in graphs]
        counts = [v.num_arcs for v, _ in views]
        n_arcs = sum(counts)
        arr = (capi.GraphView * max(B, 1))(*[v for v, _ in views])
        w = ag = None
        if weights is not None:
            assert weights.is_cuda and weights.device == e.device and weights.dtype == torch.float32
            assert weights.numel() == n_arcs
            w = weights.detach().contiguous()
            ag = torch.empty(max(n_arcs, 1), dtype=torch.float32, device=e.device)  # written by the call
        stream = torch.cuda.current_stream(e.device).cuda_stream
        g = _ctx_for(e.device, stream)
        il = _lengths(input_lengths, B)
        losses = np.zeros(B, np.float32)
        grad = torch.empty_like(e)  # every row is written by the call
        g._check(capi.lib().gtnb_graph_loss(
            g.h, B, T, Cn, e.data_ptr(), 1, None if il is None else il.ctypes.data_as(capi._i32p), arr,
            None if w is None else w.data_ptr(), 1, losses.ctypes.data_as(capi._f32p), grad.data_ptr(), 1,
            None if ag is None else ag.data_ptr(), 1))
        out = torch.from_numpy(losses).to(e.device)
        if ag is not None:
            ag = ag[:n_arcs].view_as(weights)
            # utterance of every arc, for a per-utterance upstream gradient (reduction "none")
            ctx.owner = torch.repeat_interleave(torch.arange(B), torch.tensor(counts, dtype=torch.long)).to(e.device)
        ctx.save_for_backward(grad, ag)
        ctx.reduction = reduction
        ctx.B = B
        return out.mean() if reduction == "mean" else out

    @staticmethod
    def backward(ctx, grad_output):
        grad, ag = ctx.saved_tensors
        if ctx.reduction == "mean":
            scale = grad_output / ctx.B
            return grad * scale, None if ag is None else ag * scale, None, None, None
        # reduction "none": every graph belongs to one utterance, so its arcs take that utterance's upstream gradient
        go = grad_output.reshape(-1)
        wg = None if ag is None else ag * go[ctx.owner].view_as(ag)
        return grad * go.view(-1, 1, 1), wg, None, None, None


def graph_loss(emissions, graphs, input_lengths=None, weights=None, reduction="mean"):
    return GraphLossFunction.apply(emissions, weights, graphs, input_lengths, reduction)
