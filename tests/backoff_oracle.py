"""Test infrastructure for gtnb_backoff_transitions_loss and gtnb_viterbi_backoff (a transition graph G with epsilon
arcs, the backoff arcs of a pruned n-gram token LM):

    loss_b = forwardScore(intersect(E_b, G)) - forwardScore(intersect(intersect(A_b, G), E_b))
    decode: viterbiPath / viterbiScore of intersect(E_b, G)

An epsilon arc of G has ilabel == olabel == -1: it moves G without consuming a frame and weighs its trans_w alone.

- ``sparse_trans_oracle.ref_sparse_trans_loss`` is the live reference for the loss: it passes G to the reference
  unchanged, epsilon arcs included.
- ``ref_backoff_viterbi``: the live reference for the decode, G's olabels replaced by its arc ids (G') as in
  sparse_viterbi_oracle; the path's arcs with an epsilon ilabel are G's epsilon arcs, which use no frame and are
  dropped, so the path has T_b arcs left.
- G builders, seeded: ``backoff_ngram`` (a backoff n-gram counted from a random corpus and pruned), ``backoff_lm`` (the
  benchmark's pruned trigram shape), ``eps_graph`` (a random G with epsilon arcs, several start and accept nodes) and
  ``eps_cycle_graph``.  A graph is a dict of numpy arrays (graph_oracle.make); the builders return (G, trans_w).
- ``closure_levels``: the topological levels of G's epsilon subgraph, restated.
"""
import numpy as np

from oracle import pyoracle as po
from tests import graph_oracle as go

EPS = -1


def ref_backoff_viterbi(emissions, G, trans_w, input_lens=None):
    """-> (paths [B, T] int32, scores [B] float32, arcs [B, T] int32: G's emitting arcs), -1 beyond T_b and without an
    accepting path"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    paths = np.full((B, T), -1, np.int32)
    arcs = np.full((B, T), -1, np.int32)
    scores = np.full(B, -np.inf, np.float32)
    g = dict(G)
    g["w"] = np.asarray(trans_w, np.float32).ravel()
    g["olabel"] = np.arange(len(g["src"]), dtype=np.int32)
    rg = go.ref_graph(g)
    for b in range(B):
        Tb = T if input_lens is None else int(input_lens[b])
        if Tb == 0:  # linearGraph(0, C) accepts nothing
            continue
        lat = po.ref_op("intersect", po.RefGraph.linear(Tb, C, e[b, :Tb].ravel()), rg)
        scores[b] = po.ref_op("viterbi_score", lat).item()
        p = po.ref_op("viterbi_path", lat).arrays()
        emit = p["ilabel"] != EPS
        n = int(emit.sum())
        assert n in (0, Tb), (n, Tb)
        paths[b, :n] = p["ilabel"][emit]
        arcs[b, :n] = p["olabel"][emit]
    return paths, scores, arcs


def _finish(flags, src, dst, lab, w):
    G = go.make(flags, src, dst, lab)
    return G, np.asarray(w, np.float32)


def backoff_ngram(rng, C, order, n_tokens=3000, min_count=3, n_neg_inf=0, start_all=False):
    """a backoff n-gram of `order` counted from a random corpus: states are the histories of length < order seen at
    least min_count times (the root, the empty history, always), a state has one arc per label seen after it, to the
    longest kept suffix of (history, label), weighted by its log relative count, and one epsilon arc to its history
    minus the oldest label, weighted log(0.1 .. 0.5).  The root starts; every state accepts (start_all: every state
    starts too).  n_neg_inf emitting arcs get weight -inf."""
    P = rng.dirichlet(np.full(C, 0.3), C)  # a peaked first-order chain, so that histories repeat
    toks = [int(rng.integers(C))]
    for _ in range(n_tokens - 1):
        toks.append(int(rng.choice(C, p=P[toks[-1]])))
    counts = {}
    for i, c in enumerate(toks):
        for k in range(min(order, i + 1)):
            h = tuple(toks[i - k:i])
            counts.setdefault(h, {})
            counts[h][c] = counts[h].get(c, 0) + 1
    states = [()] + sorted(h for h in counts if 0 < len(h) < order and sum(counts[h].values()) >= min_count)
    sid = {h: i for i, h in enumerate(states)}

    def target(h):
        while h not in sid:
            h = h[1:]
        return sid[h]

    src, dst, lab, w = [], [], [], []
    for h in states:
        tot = sum(counts[h].values())
        for c in sorted(counts[h]):
            src.append(sid[h])
            dst.append(target((h + (c,))[-(order - 1):] if order > 1 else ()))
            lab.append(c)
            w.append(np.log(counts[h][c] / tot))
        if h:
            src.append(sid[h])
            dst.append(sid[h[1:]])
            lab.append(EPS)
            w.append(np.log(rng.uniform(0.1, 0.5)))
    w = np.asarray(w, np.float32)
    if n_neg_inf:
        emit = np.flatnonzero(np.asarray(lab) != EPS)
        w[rng.choice(emit, n_neg_inf, replace=False)] = -np.inf
    flags = np.full(len(states), 3 if start_all else 2, np.uint8)
    flags[0] = 3
    return _finish(flags, src, dst, lab, w)


def backoff_lm(rng, C=64, n_bigram_arcs=20, n_trigram=2000, n_trigram_arcs=8):
    """the benchmark's pruned backoff trigram: 1 root + C bigram states + n_trigram trigram states (histories (a, b)
    drawn without replacement); the root has an arc per label, a bigram state n_bigram_arcs, a trigram state
    n_trigram_arcs, each to (b, c) when that trigram state exists, else to (c); every non-root state backs off by
    one epsilon arc.  Log-softmax weights; the root starts, every state accepts."""
    pairs = rng.choice(C * C, n_trigram, replace=False)
    tri = {int(p): 1 + C + i for i, p in enumerate(pairs)}
    S = 1 + C + n_trigram
    src, dst, lab, w = [], [], [], []

    def out(s, labels, hist):
        x = rng.normal(0.0, 1.0, len(labels))
        x = x - np.log(np.exp(x).sum()) - 0.5  # (the backoff keeps the rest of the mass)
        for c, wc in zip(labels, x):
            src.append(s)
            dst.append(tri.get(hist * C + int(c), 1 + int(c)) if hist >= 0 else 1 + int(c))
            lab.append(int(c))
            w.append(wc)

    out(0, np.arange(C), -1)
    for b in range(C):
        out(1 + b, rng.choice(C, n_bigram_arcs, replace=False), b)
    for p, s in tri.items():
        out(s, rng.choice(C, n_trigram_arcs, replace=False), p % C)
    for b in range(C):
        src.append(1 + b), dst.append(0), lab.append(EPS), w.append(np.log(rng.uniform(0.2, 0.5)))
    for p, s in tri.items():
        src.append(s), dst.append(1 + p % C), lab.append(EPS), w.append(np.log(rng.uniform(0.2, 0.5)))
    flags = np.full(S, 2, np.uint8)
    flags[0] = 3
    return _finish(flags, src, dst, lab, w)


def eps_graph(rng, N, A, C, n_eps, n_start=3, n_accept=3, label_hi=None, eps_into_start=True):
    """a random G with n_eps epsilon arcs that form no cycle (from lower to higher positions of a random order),
    several start and accept nodes, labels in [0, label_hi)"""
    g = go.random_graph(rng, N, A, C, n_start=n_start, n_accept=n_accept, label_hi=label_hi)
    order = rng.permutation(N)
    pos = np.empty(N, np.int64)
    pos[order] = np.arange(N)
    es, ed = [], []
    while len(es) < n_eps:
        u, v = rng.integers(0, N, 2)
        if pos[u] < pos[v] and (eps_into_start or not g["flags"][v] & 1):
            es.append(u), ed.append(v)
    src = np.concatenate([g["src"], es])
    dst = np.concatenate([g["dst"], ed])
    lab = np.concatenate([g["olabel"], np.full(n_eps, EPS)])
    return _finish(g["flags"], src, dst, lab, rng.uniform(-1, 1, len(src)))


def eps_cycle_graph():
    """epsilon arcs 1 -> 2 -> 3 -> 1 beside emitting arcs"""
    return _finish([1, 0, 0, 2], [0, 1, 2, 3, 0, 2], [1, 2, 3, 1, 3, 3], [0, EPS, EPS, EPS, 1, 2],
                   np.zeros(6, np.float32))


def closure_levels(G):
    """(forward levels, backward levels) of G's epsilon subgraph: level(v) = 0 without epsilon in-arcs, else 1 + the
    largest level of their sources; backward over the out-arcs.  None when the epsilon arcs have a cycle."""
    N = len(G["flags"])
    eps = np.flatnonzero(G["olabel"] == EPS)
    f = np.zeros(N, np.int64)
    b = np.zeros(N, np.int64)
    for _ in range(N + 1):
        nf = f.copy()
        nb = b.copy()
        for k in eps:
            nf[G["dst"][k]] = max(nf[G["dst"][k]], f[G["src"][k]] + 1)
            nb[G["src"][k]] = max(nb[G["src"][k]], b[G["dst"][k]] + 1)
        if (nf == f).all() and (nb == b).all():
            return f, b
        f, b = nf, nb
    return None


def _eps_order(G):
    """G's epsilon arcs in an order that closes a frame: by the forward level of their destination"""
    f, _ = closure_levels(G)
    eps = np.flatnonzero(G["olabel"] == EPS)
    return eps[np.argsort(f[G["dst"][eps]], kind="stable")]


def restate_loss(e, lens, G, w, C):
    """float64 restatement of one sweep of the device route over G (epsilon arcs closed after every frame, frame 0
    and T_b included): -> (Z [B], grad [B, T, C], wgrad [G arcs])"""
    e = np.asarray(e, np.float64)
    B, T, _ = e.shape
    w = np.asarray(w, np.float64)
    src, dst, lab = G["src"], G["dst"], G["olabel"]
    emit = np.flatnonzero((lab >= 0) & (lab < C))
    order = _eps_order(G)
    N = len(G["flags"])
    start = np.where(G["flags"] & 1, 0.0, -np.inf)
    accept = np.where(G["flags"] & 2, 0.0, -np.inf)
    Z = np.full(B, -np.inf)
    grad = np.zeros_like(e)
    wgrad = np.zeros(len(src))

    def close_f(a):
        for k in order:  # by destination level: every source is final
            a[dst[k]] = np.logaddexp(a[dst[k]], a[src[k]] + w[k])
        return a

    def close_b(b):
        for k in order[::-1]:
            b[src[k]] = np.logaddexp(b[src[k]], b[dst[k]] + w[k])
        return b

    def lse_into(n, idx, x):
        out = np.full(n, -np.inf)
        np.logaddexp.at(out, idx, x)
        return out

    for b in range(B):
        Tb = int(lens[b])
        if Tb == 0:
            continue
        al = [close_f(start.copy())]
        for t in range(Tb):
            al.append(close_f(lse_into(N, dst[emit], al[-1][src[emit]] + w[emit] + e[b, t, lab[emit]])))
        Z[b] = np.logaddexp.reduce(al[Tb] + accept)
        if not np.isfinite(Z[b]):
            continue
        be = close_b(accept.copy())
        for t in range(Tb, -1, -1):
            if t < Tb:
                x = w[emit] + e[b, t, lab[emit]] + be[dst[emit]]
                p = np.exp(al[t][src[emit]] + x - Z[b])
                np.add.at(grad[b, t], lab[emit], p)
                np.add.at(wgrad, emit, p)
                be = close_b(lse_into(N, src[emit], x))
            wgrad[order] += np.exp(al[t][src[order]] + w[order] + be[dst[order]] - Z[b])
    return Z, grad, wgrad


def restate_decode(e, G, w, C):
    """float32 restatement of the decode's device route for one utterance (e: its T_b rows): S_t[v] = max over
    emitting in-arcs of fl(S_{t-1}[u] + fl(w + e)), then over epsilon in-arcs of fl(S_t[u] + w), the levels in order;
    -> (score, tie on the traced path or between best accept nodes, labels, G's emitting arcs) with the lowest in-list
    position among equal candidates (emitting in-arcs by arc id, then epsilon in-arcs by arc id)"""
    e = np.asarray(e, np.float32)
    Tb = e.shape[0]
    w = np.asarray(w, np.float32)
    src, dst, lab = G["src"], G["dst"], G["olabel"]
    N = len(G["flags"])
    f, _ = closure_levels(G)
    ins = [[k for k in range(len(src)) if dst[k] == v and 0 <= lab[k] < C] for v in range(N)]
    eins = [[k for k in range(len(src)) if dst[k] == v and lab[k] == EPS] for v in range(N)]
    by_level = sorted(range(N), key=lambda v: f[v])
    neg = np.float32(-np.inf)
    S = np.where(G["flags"] & 1, np.float32(0), neg).astype(np.float32)
    bps, ties = [], []

    def close(S, bp, tie, frame0):
        for v in by_level:
            if f[v] == 0:
                continue
            cands = [np.float32(S[src[k]] + w[k]) for k in eins[v]]
            m = max(cands, default=neg)
            if not m > neg:
                continue
            if m > S[v]:
                j = cands.index(m)
                tie[v] = cands.count(m) > 1
                S[v], bp[v] = m, ("eps", eins[v][j])
            elif m == S[v]:
                tie[v] = True

    bp = [("start", -1) if G["flags"][v] & 1 else None for v in range(N)]
    tie = [False] * N
    close(S, bp, tie, True)
    bps.append(bp)
    ties.append(tie)
    for t in range(Tb):
        Sn = np.full(N, neg, np.float32)
        bp = [None] * N
        tie = [False] * N
        for v in range(N):
            cands = [np.float32(S[src[k]] + np.float32(w[k] + e[t, lab[k]])) for k in ins[v]]
            m = max(cands, default=neg)
            if m > neg:
                Sn[v], bp[v] = m, ("emit", ins[v][cands.index(m)])
                tie[v] = cands.count(m) > 1
        close(Sn, bp, tie, False)
        S = Sn
        bps.append(bp)
        ties.append(tie)
    acc = [v for v in range(N) if G["flags"][v] & 2]
    vals = [S[v] for v in acc]
    m = max(vals, default=neg)
    if Tb == 0 or not m > neg:
        return neg, False, None, None
    head = acc[vals.index(m)]
    tie_any = vals.count(m) > 1
    labels, arcs = [], []
    v, t = head, Tb
    while True:
        tie_any |= ties[t][v]
        kind, k = bps[t][v]
        if kind == "start":
            break
        v = src[k]
        if kind == "emit":
            labels.append(int(lab[k]))
            arcs.append(int(k))
            t -= 1
    return m, tie_any, np.asarray(labels[::-1], np.int32), np.asarray(arcs[::-1], np.int32)
