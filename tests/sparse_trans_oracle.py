"""Test infrastructure for gtnb_sparse_transitions_loss (user target graphs with a learned transition graph G of any
shape):

    loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(A_b, G), E_b))

- ``ref_sparse_trans_loss``: the live reference (oracle/_ref), utterance by utterance, with G built as a reference Graph
  from its structure and trans_w (its weights in arc order).  Returns the losses and the emission, transition and
  arc-weight gradients; T_b = 0 is NaN with no gradient (linearGraph(0, C) accepts nothing), as in
  graph_trans_oracle.ref_graph_trans_loss, of which this is the generalisation to any G.
- G builders: the trigram graph (C^2 nodes, all start and accept; node a*C + b means "the last two labels were a, b";
  arc a*C+b -> b*C+m has label m and weight trans_w[(a*C+b)*C + m]), and random sparse cyclic graphs with several
  start and accept nodes, unreachable nodes and labels >= C.
"""
import numpy as np

from oracle import pyoracle as po
from tests import graph_oracle as go


def ref_sparse_trans_loss(emissions, graphs, G, trans_w, input_lens=None, weights=None):
    """-> (losses [B], grads [B, T, C] (zero beyond T_b), arc_grads [sum A_b] in batch order, trans_grad [G arcs])"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    gd = dict(G)
    gd["w"] = np.asarray(trans_w, np.float32).ravel()
    losses, grads = np.zeros(B, np.float32), np.zeros_like(e)
    tg = np.zeros(len(gd["src"]), np.float64)
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
        ag, rg = go.ref_graph(g), go.ref_graph(gd)
        E = po.RefGraph.linear(Tb, C, e[b, :Tb].ravel())
        den = po.ref_op("forward_score", po.ref_op("intersect", E, rg))
        num = po.ref_op("forward_score", po.ref_op("intersect", po.ref_op("intersect", ag, rg), E))
        loss = po.ref_op("subtract", den, num)
        po.ref_backward(loss)
        losses[b] = loss.item()
        grads[b, :Tb] = E.grad().weights().reshape(Tb, C)
        if len(gd["src"]):
            tg += rg.grad().weights().astype(np.float64)
        arc_grads.append(ag.grad().weights() if A else np.zeros(0, np.float32))
    ag = np.concatenate(arc_grads) if arc_grads else np.zeros(0, np.float32)
    return losses, grads, ag, tg.astype(np.float32)


def trigram_graph(C):
    """the trigram G over C labels: arc (a*C+b)*C + m goes a*C+b -> b*C+m with label m"""
    n = np.arange(C * C * C)
    ab, m = n // C, n % C
    src = ab
    dst = (ab % C) * C + m
    return go.make(np.full(C * C, 3, np.uint8), src, dst, m)


def bigram_graph(C):
    """gtnb_graph_transitions_loss's BIGRAM G as a graph: arc j*C + i goes j -> i with label i (weight W[i][j])"""
    n = np.arange(C * C)
    return go.make(np.full(C, 3, np.uint8), n // C, n % C, n % C)


def bigram_slots(C):
    """trans_w slot (W[i][j] = i*C + j) of every arc of bigram_graph"""
    n = np.arange(C * C)
    return (n % C) * C + n // C


def asg_graph(C):
    """gtnb_asg_loss_ex's G as a graph (graph_trans_oracle.dense_graph(ASG)); arc k reads trans_w[k]"""
    from tests import graph_trans_oracle as gt
    g, _ = gt.dense_graph(gt.ASG, C, np.zeros(C + C * C, np.float32))
    return g


def sparse_graph(rng, N, A, C, n_start=3, n_accept=3, label_hi=None, n_unreachable=2):
    """a random sparse cyclic G: N reachable-ish nodes with A random arcs (labels in [0, label_hi)), several start
    and accept nodes, plus n_unreachable nodes that only have arcs among themselves"""
    g = go.random_graph(rng, N, A, C, n_start=n_start, n_accept=n_accept, label_hi=label_hi)
    if n_unreachable:
        u = np.arange(N, N + n_unreachable)
        flags = np.concatenate([g["flags"], np.full(n_unreachable, 2, np.uint8)])
        src = np.concatenate([g["src"], u, u])
        dst = np.concatenate([g["dst"], u, np.roll(u, 1)])
        lab = np.concatenate([g["olabel"], rng.integers(0, C, 2 * n_unreachable)])
        g = go.make(flags, src, dst, lab)
    return g
