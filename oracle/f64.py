"""float64 referee (TEST INFRASTRUCTURE, like everything under oracle/).

The north star asks for 1e-4 relative on scores and gradients, but at T=1000 with unnormalised
emissions the reference's own fp32 gradient is ~2e-3 (max abs) away from an exact evaluation of the same
lattice (fp32 node scores reach ~4800, 1 ulp = 4.9e-4, and every gradient is exp(score differences)).
Two fp32 evaluations cannot agree better than either agrees with the truth, so the tests and bench.py's
in-run parity block judge the CUDA path and the reference against THIS evaluation: plain numpy float64
alpha/beta recursions over the same lattices (benchmarks/ctc.cpp:40-58,150-165 for CTC,
test/criterion_test.cpp:244-305 for ASG).  Independent of oracle/gtn_oracle.c and of the product.
"""
import numpy as np


def _lse(a, axis=None):
    m = np.max(a, axis=axis, keepdims=True)
    m = np.where(np.isfinite(m), m, 0.0)
    with np.errstate(divide="ignore"):
        r = np.log(np.sum(np.exp(a - m), axis=axis, keepdims=True)) + m
    return np.squeeze(r, axis=axis) if axis is not None else float(r.reshape(()))


def ctc_f64(emissions, target, blank=0):
    """loss = forwardScore(e) - forwardScore(intersect(ctc(target), e)) and d loss / d e, float64.
    The CTC graph of benchmarks/ctc.cpp:40-58: 2U+1 nodes, self loop, step arc, skip arc between
    different labels; accept = last two nodes."""
    e = np.asarray(emissions, np.float64)
    T, C = e.shape
    tg = np.asarray(target, np.int64)
    U = len(tg)
    L = 2 * U + 1
    lab = np.full(L, blank, np.int64)
    lab[1::2] = tg
    skip = np.zeros(L, bool)
    if U > 1:
        skip[3::2] = tg[1:] != tg[:-1]
    NEG = -np.inf
    el = e[:, lab]  # [T, L]
    alpha = np.full((T + 1, L), NEG)
    alpha[0, 0] = 0.0
    with np.errstate(invalid="ignore"):
        for t in range(1, T + 1):
            p = alpha[t - 1]
            p1 = np.concatenate(([NEG], p))[:L]
            p2 = np.where(skip, np.concatenate(([NEG, NEG], p))[:L], NEG)
            alpha[t] = np.logaddexp(np.logaddexp(p, p1), p2) + el[t - 1]
        beta = np.full((T + 1, L), NEG)
        beta[T, L - 1] = 0.0
        if L > 1:
            beta[T, L - 2] = 0.0
        skip_out = np.concatenate((skip, [False, False]))[2:]  # node u has a skip arc to u+2
        for t in range(T - 1, -1, -1):
            q = beta[t + 1] + el[t]  # weight of an arc INTO node v at level t+1, plus beta there
            q1 = np.concatenate((q, [NEG]))[1:]
            q2 = np.where(skip_out, np.concatenate((q, [NEG, NEG]))[2:], NEG)
            beta[t] = np.logaddexp(np.logaddexp(q, q1), q2)
    acc = [L - 1] if L == 1 else [L - 2, L - 1]
    Z = _lse(alpha[T, acc])
    norm = _lse(e, axis=1)  # [T]
    loss = float(norm.sum() - Z)
    grad = np.exp(e - norm[:, None])  # softmax: d forwardScore(e) / d e
    if np.isfinite(Z):
        with np.errstate(invalid="ignore"):
            gamma = np.exp(alpha[1:] + beta[1:] - Z)  # [T, L] posterior of node u at level t
        gamma = np.nan_to_num(gamma, nan=0.0)
        occ = np.zeros((T, C))
        for u in range(L):
            occ[:, lab[u]] += gamma[:, u]
        grad = grad - occ
    return loss, grad


def asg_f64(emissions, trans_w, target):
    """ASG loss of test/criterion_test.cpp:244-305 in float64:
    loss = forwardScore(compose(e, trans)) - forwardScore(compose(compose(fal, trans), e)).
    trans_w = [start weights (C)] ++ [C x C, row = destination label, column = source label].
    Returns (loss, d/d e [T,C], d/d trans_w [C + C*C])."""
    e = np.asarray(emissions, np.float64)
    T, C = e.shape
    tw = np.asarray(trans_w, np.float64)
    st, tr = tw[:C], tw[C:].reshape(C, C)  # tr[i, j] = w(j -> i)
    tg = np.asarray(target, np.int64)
    U = len(tg)

    # denominator: full trellis
    a = np.empty((T, C))
    a[0] = st + e[0]
    for t in range(1, T):
        a[t] = _lse(a[t - 1][None, :] + tr, axis=1) + e[t]
    Zd = _lse(a[T - 1])
    b = np.empty((T, C))
    b[T - 1] = 0.0
    for t in range(T - 2, -1, -1):
        b[t] = _lse((b[t + 1] + e[t + 1])[:, None] + tr, axis=0)
    gd = np.exp(a + b - Zd)  # node posteriors [T, C]
    tgd = np.zeros(C + C * C)
    tgd[:C] = gd[0]
    xi = np.zeros((C, C))
    for t in range(1, T):
        xi += np.exp(a[t - 1][None, :] + tr + (e[t] + b[t])[:, None] - Zd)
    tgd[C:] = xi.ravel()

    # numerator: forced alignment chain (U nodes, self loop + step), arcs weighted by trans + e
    NEG = -np.inf
    al = np.full((T, U), NEG)
    al[0, 0] = st[tg[0]] + e[0, tg[0]]
    self_w = tr[tg, tg]
    step_w = np.concatenate(([NEG], tr[tg[1:], tg[:-1]]))
    with np.errstate(invalid="ignore"):
        for t in range(1, T):
            p = al[t - 1]
            p1 = np.concatenate(([NEG], p[:-1]))
            al[t] = np.logaddexp(p + self_w, p1 + step_w) + e[t, tg]
        Zn = al[T - 1, U - 1]
        be = np.full((T, U), NEG)
        be[T - 1, U - 1] = 0.0
        for t in range(T - 2, -1, -1):
            q = be[t + 1] + e[t + 1, tg]
            q1 = np.concatenate((q[1:] + step_w[1:], [NEG]))
            be[t] = np.logaddexp(q + self_w, q1)
        gn = np.nan_to_num(np.exp(al + be - Zn), nan=0.0)
    loss = float(Zd - Zn)
    grad = gd.copy()
    tgn = np.zeros(C + C * C)
    if np.isfinite(Zn):
        for u in range(U):
            grad[:, tg[u]] -= gn[:, u]
        tgn[tg[0]] += gn[0, 0]
        with np.errstate(invalid="ignore"):
            for t in range(1, T):
                s_self = np.nan_to_num(np.exp(al[t - 1] + self_w + e[t, tg] + be[t] - Zn), nan=0.0)
                p1 = np.concatenate(([NEG], al[t - 1][:-1]))
                s_step = np.nan_to_num(np.exp(p1 + step_w + e[t, tg] + be[t] - Zn), nan=0.0)
                np.add.at(tgn, C + tg * C + tg, s_self)
                if U > 1:
                    np.add.at(tgn, C + tg[1:] * C + tg[:-1], s_step[1:])
    return loss, grad, tgd - tgn


def lattice_f64(flags, src, dst, w, tropical=False):
    """forwardScore of a lattice (a DAG) in float64, and its gradient with respect to every arc weight, which is the
    arc's posterior: exp(alpha[src] + w + beta[dst] - Z) in the log semiring; in the tropical semiring 1 on the arcs
    of the best path (first maximum in topological order), 0 elsewhere.  flags: bit 0 start, bit 1 accept.  Nodes are
    taken in a topological order computed here, so the lattice's own node numbering does not matter.
    Returns (score, arc gradient [A], best path as arc ids or None, smallest margin of a decision on that path)."""
    flags = np.asarray(flags)
    src = np.asarray(src, np.int64)
    dst = np.asarray(dst, np.int64)
    w = np.asarray(w, np.float64)
    N, A = len(flags), len(src)
    indeg = np.bincount(dst, minlength=N)
    order, stack = [], [n for n in range(N) if indeg[n] == 0]
    ins = [[] for _ in range(N)]
    outs = [[] for _ in range(N)]
    for a in range(A):
        ins[dst[a]].append(a)
        outs[src[a]].append(a)
    while stack:
        n = stack.pop()
        order.append(n)
        for a in outs[n]:
            indeg[dst[a]] -= 1
            if indeg[dst[a]] == 0:
                stack.append(dst[a])
    assert len(order) == N, "not a DAG"
    NEG = -np.inf
    alpha = np.full(N, NEG)
    best_in = np.full(N, -1)
    margin_in = np.full(N, np.inf)
    for n in order:
        cand = [alpha[src[a]] + w[a] for a in ins[n]]
        if flags[n] & 1:
            cand.append(0.0)
        if not cand:
            continue
        c = np.asarray(cand)
        if tropical:
            k = int(np.argmax(c))
            alpha[n] = c[k]
            if k < len(ins[n]):
                best_in[n] = ins[n][k]
            rest = np.delete(c, k)
            margin_in[n] = c[k] - rest.max() if len(rest) and np.isfinite(c[k]) else np.inf
        else:
            alpha[n] = _lse(c)
    acc = [n for n in range(N) if flags[n] & 2]
    if not acc:
        return -np.inf, np.zeros(A), None, np.inf
    fin = alpha[acc]
    Z = float(np.max(fin)) if tropical else _lse(fin)
    grad = np.zeros(A)
    if not np.isfinite(Z):
        return Z, grad, None, np.inf
    if tropical:
        k = int(np.argmax(fin))
        rest = np.delete(fin, k)
        margin = fin[k] - rest.max() if len(rest) else np.inf
        path, n = [], acc[k]
        while best_in[n] >= 0:
            margin = min(margin, margin_in[n])
            path.append(int(best_in[n]))
            n = src[best_in[n]]
        margin = min(margin, margin_in[n])
        path.reverse()
        grad[path] = 1.0
        return Z, grad, path, margin
    beta = np.full(N, NEG)
    for n in reversed(order):
        cand = [w[a] + beta[dst[a]] for a in outs[n]]
        if flags[n] & 2:
            cand.append(0.0)
        if cand:
            beta[n] = _lse(np.asarray(cand))
    with np.errstate(invalid="ignore"):
        grad = np.nan_to_num(np.exp(alpha[src] + w + beta[dst] - Z), nan=0.0)
    return Z, grad, None, np.inf
