"""Test infrastructure for gtnb_graph_transitions_loss (user target graphs with a learned dense transition graph G):

    ASG:    loss_b = forwardScore(compose(E_b, G)) - forwardScore(compose(compose(A_b, G), E_b))
    BIGRAM: loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(A_b, G), E_b))

- ``ref_graph_trans_loss``: the live reference (oracle/_ref), utterance by utterance, with G built as a reference
  Graph from trans_w (``dense_graph``).  Returns the losses and the emission, transition and arc-weight gradients.
  T_b = 0 is NaN with no gradient (linearGraph(0, C) accepts nothing), as in graph_oracle.ref_graph_loss.
- ``dense_graph``: G as arrays, with the trans_w slot of every arc.
"""
import numpy as np

from oracle import pyoracle as po
from tests import graph_oracle as go

ASG, BIGRAM = 0, 1


def dense_graph(kind, C, trans_w):
    """(graph arrays, slot of trans_w of every arc).  ASG: node 0 starts, nodes 1..C accept, arc 0 -> i+1 (label i,
    s[i]), arc j+1 -> i+1 (label i, W[i][j] = trans_w[C + i*C + j]).  BIGRAM: C nodes, all start and accept, arc
    j -> i (label i, W[i][j] = trans_w[i*C + j])."""
    tw = np.asarray(trans_w, np.float32).ravel()
    src, dst, lab, slot = [], [], [], []
    if kind == ASG:
        flags = [1] + [2] * C
        for i in range(C):
            src.append(0), dst.append(i + 1), lab.append(i), slot.append(i)
        for i in range(C):
            for j in range(C):
                src.append(j + 1), dst.append(i + 1), lab.append(i), slot.append(C + i * C + j)
    else:
        flags = [3] * C
        for j in range(C):
            for i in range(C):
                src.append(j), dst.append(i), lab.append(i), slot.append(i * C + j)
    slot = np.asarray(slot, np.int64)
    return go.make(flags, src, dst, lab, w=tw[slot]), slot


def ref_graph_trans_loss(emissions, graphs, kind, trans_w, input_lens=None, weights=None):
    """-> (losses [B], grads [B, T, C] (zero beyond T_b), arc_grads [sum A_b] in batch order, trans_grad)"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    op = "compose" if kind == ASG else "intersect"
    gd, slot = dense_graph(kind, C, trans_w)
    losses, grads = np.zeros(B, np.float32), np.zeros_like(e)
    tg = np.zeros(np.asarray(trans_w).size, np.float64)
    arc_grads, off = [], 0
    for b in range(B):
        g = dict(graphs[b])
        A = len(g["src"])
        if weights is not None:
            g["w"] = np.asarray(weights[off:off + A], np.float32)
        off += A
        Tb = T if input_lens is None else int(input_lens[b])
        if Tb == 0:
            losses[b] = np.nan
            arc_grads.append(np.zeros(A, np.float32))
            continue
        ag, G = go.ref_graph(g), go.ref_graph(gd)
        E = po.RefGraph.linear(Tb, C, e[b, :Tb].ravel())
        den = po.ref_op("forward_score", po.ref_op(op, E, G))
        num = po.ref_op("forward_score", po.ref_op(op, po.ref_op(op, ag, G), E))
        loss = po.ref_op("subtract", den, num)
        po.ref_backward(loss)
        losses[b] = loss.item()
        grads[b, :Tb] = E.grad().weights().reshape(Tb, C)
        np.add.at(tg, slot, G.grad().weights().astype(np.float64))
        arc_grads.append(ag.grad().weights() if A else np.zeros(0, np.float32))
    ag = np.concatenate(arc_grads) if arc_grads else np.zeros(0, np.float32)
    return losses, grads, ag, tg.astype(np.float32)


def fal_graph(target):
    """ASG's force-align chain of a target (criterion_test.cpp): U+1 nodes, 0 -> 1 and per node a self-loop and the
    step to the next label; node U accepts"""
    U = len(target)
    flags = [1] + [0] * U
    flags[U] |= 2 if U else 0
    src, dst, lab = [], [], []
    for n in range(1, U + 1):
        src.append(n - 1), dst.append(n), lab.append(int(target[n - 1]))
        src.append(n), dst.append(n), lab.append(int(target[n - 1]))
    return go.make(flags, src, dst, lab)
