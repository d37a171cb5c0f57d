"""Test infrastructure for gtnb_ngram_ctc_loss (CTC with a learned bigram transition graph G, the timeNgramCtc
workload of benchmarks/ctc.cpp:107-134), three independent evaluations of

    loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(ctc_b, G), E_b))

with G: C nodes, every node start and accept, for j, for i: arc j -> i, label i, weight W[i*C + j], then arcSort().

- ``ref_ngram_ctc``: the live reference (oracle/_ref), graph by graph through its own Graph API, no fold.
- ``oracle_ngram_ctc``: the C restatement (oracle/gtn_oracle.c), literally intersect / forward_score_and_grad /
  compose_grad, no fold.
- ``ngram_ctc_f64``: a float64 referee (alpha / beta recursions; the product's C start states folded into
  sigma_i = logsumexp_j W[i][j], which is exact in real arithmetic), the yardstick of the gradient bar.

Gradients with respect to W are returned in W's layout ([C*C], row = destination label).
"""
import numpy as np

from oracle import f64
from oracle import pyoracle as po


def ctc_arrays(target, blank):
    """ctcGraph(target) of benchmarks/ctc.cpp:40-58 with a blank parameter: (flags, src, dst, labels)."""
    U = len(target)
    L = 2 * U + 1
    flags, src, dst, lab = [], [], [], []
    for l in range(L):
        flags.append((1 if l == 0 else 0) | (2 if l in (L - 1, L - 2) else 0))
        label = int(target[(l - 1) // 2]) if l % 2 else blank
        src.append(l), dst.append(l), lab.append(label)
        if l > 0:
            src.append(l - 1), dst.append(l), lab.append(label)
        if l % 2 and l > 1 and label != int(target[(l - 1) // 2 - 1]):
            src.append(l - 2), dst.append(l), lab.append(label)
    return flags, src, dst, lab


def bigram_arrays(W):
    """G: (flags, src, dst, labels, weights); arc j*C + i is j -> i with weight W[i*C + j]."""
    C = int(round(np.sqrt(np.asarray(W).size)))
    Wm = np.asarray(W, np.float32).reshape(C, C)
    j, i = np.meshgrid(np.arange(C), np.arange(C), indexing="ij")
    return [3] * C, j.ravel(), i.ravel(), i.ravel(), Wm[i.ravel(), j.ravel()]


def _arc_grad_to_w(garc, C):
    """gradient per arc of G (arc j*C + i) -> W's layout (i*C + j)"""
    return np.asarray(garc, np.float32).reshape(C, C).T.ravel().copy()


def ref_ngram_ctc(emissions, W, target, blank=0):
    """The live reference, one utterance: -> (loss, d/d e [T, C], d/d W [C*C])."""
    e = np.ascontiguousarray(emissions, np.float32)
    T, C = e.shape
    fl, s, d, lab = ctc_arrays(target, blank)
    ctc = po.RefGraph.from_arrays(fl, s, d, lab, lab, np.zeros(len(s), np.float32), calc_grad=False)
    ctc.arc_sort()
    gf, gs, gd, gl, gw = bigram_arrays(W)
    G = po.RefGraph.from_arrays(gf, gs, gd, gl, gl, gw)
    G.arc_sort()
    E = po.RefGraph.linear(T, C, e.ravel())
    num = po.ref_op("forward_score", po.ref_op("intersect", po.ref_op("intersect", ctc, G), E))
    den = po.ref_op("forward_score", po.ref_op("intersect", E, G))
    loss = po.ref_op("subtract", den, num)
    po.ref_backward(loss)
    return loss.item(), E.grad().weights().reshape(T, C).copy(), _arc_grad_to_w(G.grad().weights(), C)


def ref_ngram_ctc_batch(emissions, W, targets, blank=0, input_lens=None):
    """-> (losses [B], grads [B, T, C] (zero beyond T_b), trans_grad [C*C] summed over the batch)"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    losses = np.zeros(B, np.float32)
    grads = np.zeros_like(e)
    tg = np.zeros(C * C, np.float32)
    for b in range(B):
        Tb = T if input_lens is None else int(input_lens[b])
        losses[b], grads[b, :Tb], g = ref_ngram_ctc(e[b, :Tb], W, targets[b], blank)
        tg += g
    return losses, grads, tg


def oracle_ngram_ctc(emissions, W, target, blank=0):
    """The C restatement, one utterance, no fold: -> (loss, d/d e [T, C], d/d W [C*C])."""
    e = np.ascontiguousarray(emissions, np.float32)
    T, C = e.shape
    fl, s, d, lab = ctc_arrays(target, blank)
    ctc = po.Graph.from_arrays(fl, s, d, lab, lab, np.zeros(len(s), np.float32))
    ctc.arc_sort()
    gf, gs, gd, gl, gw = bigram_arrays(W)
    G = po.Graph.from_arrays(gf, gs, gd, gl, gl, gw)
    G.arc_sort()
    # (the reference's linearGraph(0, C) is one start node that does not accept, creations.cpp:20-33)
    E = po.Graph.linear(T, C, e.ravel()) if T else po.Graph.from_arrays([1], [], [], [], [])
    P = po.intersect(ctc, G)
    num = po.intersect(P, E)
    den = po.intersect(E, G)
    zn, gnum = po.forward_score_and_grad(num, delta=-1.0)
    zd, gden = po.forward_score_and_grad(den, delta=1.0)
    gP, gE_num = po.compose_grad(num, gnum, P.num_arcs, E.num_arcs)
    _, gG_num = po.compose_grad(P, gP, ctc.num_arcs, G.num_arcs)
    gE_den, gG_den = po.compose_grad(den, gden, E.num_arcs, G.num_arcs)
    with np.errstate(invalid="ignore"):
        loss = np.float32(np.float32(zd) - np.float32(zn))
    ge = (gE_num + gE_den).reshape(T, C)
    return float(loss), ge, _arc_grad_to_w(gG_num + gG_den, C)


def ngram_ctc_f64(emissions, W, target, blank=0):
    """float64 referee, one utterance: -> (loss, d/d e [T, C], d/d W [C*C])."""
    e = np.asarray(emissions, np.float64)
    T, C = e.shape
    Wm = np.asarray(W, np.float64).reshape(C, C)  # Wm[i, j] = w(j -> i)
    tg = np.asarray(target, np.int64)
    U = len(tg)
    L = 2 * U + 1
    if T == 0:  # linearGraph(0, C) accepts nothing: both forward scores are -inf
        return float("nan"), np.zeros((0, C)), np.zeros(C * C)
    NEG = -np.inf
    lse = f64._lse

    # denominator: alpha_0 = 0 on every state of G
    a = np.zeros((T + 1, C))
    for t in range(1, T + 1):
        a[t] = e[t - 1] + lse(a[t - 1][None, :] + Wm, axis=1)
    Zd = lse(a[T])
    bt = np.zeros((T + 1, C))
    xi = np.zeros((C, C))
    for t in range(T, 0, -1):
        g = e[t - 1] + bt[t]
        xi += np.exp(a[t - 1][None, :] + Wm + g[:, None] - Zd)
        bt[t - 1] = lse(Wm + g[:, None], axis=0)
    gd = np.exp(a[1:] + bt[1:] - Zd)

    # numerator: CTC nodes, arc weights W[label(dst)][label(src)]; frame 1 from the folded start (sigma)
    lab = np.full(L, blank, np.int64)
    lab[1::2] = tg
    skip = np.zeros(L, bool)
    if U > 1:
        skip[3::2] = tg[1:] != tg[:-1]
    sig = lse(Wm, axis=1)
    w_self = Wm[lab, lab]
    w_step = np.concatenate(([NEG], Wm[lab[1:], lab[:-1]]))
    w_skip = np.full(L, NEG)
    if L > 2:
        w_skip[2:] = np.where(skip[2:], Wm[lab[2:], lab[:-2]], NEG)
    el = e[:, lab]
    al = np.full((T + 1, L), NEG)
    al[1, 0] = sig[lab[0]] + el[0, 0]
    if L > 1:
        al[1, 1] = sig[lab[1]] + el[0, 1]
    with np.errstate(invalid="ignore"):
        for t in range(2, T + 1):
            p = al[t - 1]
            p1 = np.concatenate(([NEG], p[:-1]))
            p2 = np.concatenate(([NEG, NEG], p[:-2]))[:L]
            al[t] = el[t - 1] + np.logaddexp(np.logaddexp(p + w_self, p1 + w_step), p2 + w_skip)
        acc = [0] if L == 1 else [L - 2, L - 1]
        Zn = lse(al[T, acc])
        be = np.full((T + 1, L), NEG)
        be[T, acc] = 0.0
        for t in range(T, 1, -1):
            q = be[t] + el[t - 1]
            q1 = np.concatenate((q[1:] + w_step[1:], [NEG]))
            q2 = np.concatenate((q[2:] + w_skip[2:], [NEG, NEG]))[:L]
            be[t - 1] = np.logaddexp(np.logaddexp(q + w_self, q1), q2)
    grad = gd.copy()
    gW = xi.copy()
    if np.isfinite(Zn):
        with np.errstate(invalid="ignore"):
            gn = np.nan_to_num(np.exp(al[1:] + be[1:] - Zn), nan=0.0)  # [T, L]
            for l in range(L):
                grad[:, lab[l]] -= gn[:, l]
            soft = np.exp(Wm - sig[:, None])
            for l in range(min(L, 2)):  # the S arcs: d sigma_i / d W[i][:] = softmax
                gW[lab[l]] -= gn[0, l] * soft[lab[l]]
            for t in range(2, T + 1):
                post = lambda src, w: np.nan_to_num(np.exp(src + w + el[t - 1] + be[t] - Zn), nan=0.0)
                np.add.at(gW, (lab, lab), -post(al[t - 1], w_self))
                p1 = np.concatenate(([NEG], al[t - 1][:-1]))
                np.add.at(gW, (lab[1:], lab[:-1]), -post(p1, w_step)[1:])
                if L > 2:
                    p2 = np.concatenate(([NEG, NEG], al[t - 1][:-2]))
                    m = skip[2:]
                    np.add.at(gW, (lab[2:][m], lab[:-2][m]), -post(p2, w_skip)[2:][m])
    return float(Zd - Zn), grad, gW.ravel()
