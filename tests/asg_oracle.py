"""Test infrastructure for gtnb_asg_loss_ex (ASG on a padded minibatch, test/criterion_test.cpp:244-305): three
independent evaluations of

    loss_b = forwardScore(compose(E_b, transitions)) - forwardScore(compose(compose(fal_b, transitions), E_b))

with E_b = linearGraph(T_b, C) on the first T_b rows of utterance b, each run on e[b, :T_b] alone.

- ``ref_asg_batch``: the live reference (oracle/_ref), one utterance at a time.
- ``oracle_asg_batch``: the C restatement (oracle/gtn_oracle.c).
- ``asg_f64_batch``: the float64 referee (oracle/f64.asg_f64), extended to the cases it does not cover, with the
  reference's answers: T_b = 0 is NaN with no gradient (linearGraph(0, C) accepts nothing), U = 0 is +inf with the
  denominator's gradient alone (fal has no accepting node).

trans_w and the transition gradients are ASG's [C + C*C]: start weights, then the matrix, row = destination label.
"""
import numpy as np

from oracle import f64
from oracle import pyoracle as po


def _lens(B, T, input_lens):
    return [T] * B if input_lens is None else [int(x) for x in input_lens]


def ref_asg_batch(emissions, trans_w, targets, input_lens=None):
    """-> (losses [B], grads [B, T, C] (zero beyond T_b), trans_grad [C + C*C] summed over the batch)"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    losses, grads, tg = np.zeros(B, np.float32), np.zeros_like(e), np.zeros(C + C * C, np.float32)
    for b, Tb in enumerate(_lens(B, T, input_lens)):
        lo, go, to, _ = po.ref_asg_batch(e[b:b + 1, :Tb], trans_w, [targets[b]])
        losses[b], grads[b, :Tb] = lo[0], go[0]
        tg += to
    return losses, grads, tg


def oracle_asg_batch(emissions, trans_w, targets, input_lens=None):
    """the C oracle, utterance by utterance on its own rows -> (losses, grads, trans_grad)"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    losses, grads, tg = np.zeros(B, np.float32), np.zeros_like(e), np.zeros(C + C * C, np.float32)
    for b, Tb in enumerate(_lens(B, T, input_lens)):
        losses[b], grads[b, :Tb], t = po.asg_loss(e[b, :Tb], trans_w, targets[b])
        tg += t
    return losses, grads, tg


def asg_f64(emissions, trans_w, target):
    """float64 referee for one utterance, every T and U -> (loss, d/d e [T, C], d/d trans_w [C + C*C])"""
    e = np.asarray(emissions, np.float64)
    T, C = e.shape
    if T == 0:
        return float("nan"), np.zeros((0, C)), np.zeros(C + C * C)
    if len(target) == 0:  # the numerator's score is -inf: the denominator's gradient alone
        _, g, t = _denominator_f64(e, trans_w)
        return float("inf"), g, t
    return f64.asg_f64(e, trans_w, target)


def _denominator_f64(e, trans_w):
    """forwardScore(compose(e, transitions)) and its gradients, float64"""
    T, C = e.shape
    tw = np.asarray(trans_w, np.float64)
    st, tr = tw[:C], tw[C:].reshape(C, C)
    a = np.empty((T, C))
    a[0] = st + e[0]
    for t in range(1, T):
        a[t] = f64._lse(a[t - 1][None, :] + tr, axis=1) + e[t]
    Z = f64._lse(a[T - 1])
    b = np.zeros((T, C))
    for t in range(T - 2, -1, -1):
        b[t] = f64._lse((b[t + 1] + e[t + 1])[:, None] + tr, axis=0)
    g = np.exp(a + b - Z)
    tg = np.zeros(C + C * C)
    tg[:C] = g[0]
    xi = np.zeros((C, C))
    for t in range(1, T):
        xi += np.exp(a[t - 1][None, :] + tr + (e[t] + b[t])[:, None] - Z)
    tg[C:] = xi.ravel()
    return Z, g, tg


def asg_f64_batch(emissions, trans_w, targets, input_lens=None):
    """-> (losses [B], grads [B, T, C], trans_grad [C + C*C]) in float64"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    losses, grads, tg = np.zeros(B), np.zeros((B, T, C)), np.zeros(C + C * C)
    for b, Tb in enumerate(_lens(B, T, input_lens)):
        losses[b], grads[b, :Tb], t = asg_f64(e[b, :Tb], trans_w, targets[b])
        tg += t
    return losses, grads, tg
