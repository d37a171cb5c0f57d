"""A float64 restatement of gtnb_beam_decode_async's prefix beam search (include/gtn_b200.h), for the three kinds.

Each beam is (transcript, p_blank, p_label); the transcripts are tuples, so merges are dictionary lookups and never
depend on a hash.  At every frame the candidates are each beam kept and each beam extended by each non-blank token
(every token for ASG); an extension whose transcript is a live beam is log-added into that beam's kept candidate.
Candidates of score -inf are dropped; the rest are ranked by (score descending, kept before extensions, previous
slot, token) and the first K survive, in that order.

Besides the N-best lists, every utterance reports its smallest decision margin: the smallest nonzero score gap at
any frame's K-th / (K+1)-th boundary and between consecutive N-best entries (and the N-th and (N+1)-th beam).  A gap
of exactly 0 is a tie, decided by the tie rule and flagged (status 3).  ASG makes such ties by construction: staying
on the last token and appending it again score the same frame with the same operations, in float32 as in float64.
Where the margin is large, float32 rounding cannot change a decision.
"""
import numpy as np

CTC, BIGRAM, ASG = 2, 1, 0  # GTNB_DENSE_CTC, GTNB_DENSE_BIGRAM, GTNB_DENSE_ASG
NEG = -np.inf


def _lae(a, b):
    with np.errstate(invalid="ignore"):
        return np.logaddexp(a, b)


def _logsumexp_rows(W):
    m = W.max(axis=1)
    safe = np.where(np.isfinite(m), m, 0.0)
    with np.errstate(divide="ignore"):
        return np.where(m == NEG, NEG, safe + np.log(np.exp(W - safe[:, None]).sum(axis=1)))


def search(e, kind, W=None, start=None, blank=0, K=16, N=1):
    """One utterance: e [T_b, C] (float, the widened emissions), W [C, C] (row = destination label) and, for ASG,
    start [C].  -> dict(hyps: list of (transcript tuple, score) of up to N entries, tie: bool, margin: float)"""
    e = np.asarray(e, np.float64)
    Tb, C = e.shape
    if kind != CTC:
        W = np.asarray(W, np.float64).reshape(C, C)
    sigma = _logsumexp_rows(W) if kind == BIGRAM else None
    beams = [((), 0.0, NEG)]  # slot order
    margin, tie = np.inf, False
    tokens = np.arange(C)
    for t in range(Tb):
        et = e[t]
        index = {y: r for r, (y, _, _) in enumerate(beams)}
        kept = []
        for r, (y, pb, pl) in enumerate(beams):
            l = y[-1] if y else -1
            if kind == CTC:
                nb = _lae(pb, pl) + et[blank]
                nl = pl + et[l] if l >= 0 else NEG
            elif kind == BIGRAM:
                wpb = sigma[blank] if t == 0 else W[blank, blank]
                nb = _lae(pb + wpb, pl + W[blank, l] if l >= 0 else NEG) + et[blank]
                nl = pl + W[l, l] + et[l] if l >= 0 else NEG
            else:
                nb = NEG
                nl = pl + W[l, l] + et[l] if l >= 0 else NEG
            kept.append([nb, nl])
        ext = []  # (score, slot, token)
        for s, (y, pb, pl) in enumerate(beams):
            l = y[-1] if y else -1
            if kind == CTC:
                v = np.where(tokens == l, pb, _lae(pb, pl)) + et
            else:
                wpb = (sigma if t == 0 else W[:, blank]) if kind == BIGRAM else start
                from_pb = pb + np.asarray(wpb, np.float64) if pb > NEG else np.full(C, NEG)
                from_pl = pl + W[:, l] if l >= 0 and pl > NEG else np.full(C, NEG)
                if kind == BIGRAM and l >= 0:
                    from_pl = np.where(tokens == l, NEG, from_pl)
                v = _lae(from_pb, from_pl) + et
            if kind != ASG:
                v = np.where(tokens == blank, NEG, v)
            for c in np.nonzero(v > NEG)[0]:
                r = index.get(y + (int(c),))
                if r is not None:
                    kept[r][1] = _lae(kept[r][1], v[c])
                else:
                    ext.append((float(v[c]), s, int(c)))
        cands = []  # (score, kind, slot, token, transcript, pb, pl)
        for r, (nb, nl) in enumerate(kept):
            sc = _lae(nb, nl)
            if sc > NEG:
                cands.append((sc, 0, r, 0, beams[r][0], nb, nl))
        for sc, s, c in ext:
            cands.append((sc, 1, s, c, beams[s][0] + (c,), NEG, sc))
        cands.sort(key=lambda x: (-x[0], x[1], x[2], x[3]))
        if len(cands) > K:
            gap = cands[K - 1][0] - cands[K][0]
            margin = min(margin, gap) if gap > 0 else margin
            tie |= gap == 0
        beams = [(x[4], x[5], x[6]) for x in cands[:K]]
    scores = [float(_lae(pb, pl)) for _, pb, pl in beams]
    for n in range(min(N, len(beams) - 1)):
        gap = scores[n] - scores[n + 1]
        margin = min(margin, gap) if gap > 0 else margin
        tie |= gap == 0
    return dict(hyps=[(beams[n][0], scores[n]) for n in range(min(N, len(beams)))], tie=tie, margin=margin)


def split_weights(kind, trans_w, C):
    """(W [C, C], start [C] or None) from a flat trans_w in the C ABI's layout"""
    if kind == CTC:
        return None, None
    w = np.asarray(trans_w, np.float64).ravel()
    if kind == ASG:
        return w[C:].reshape(C, C), w[:C]
    return w.reshape(C, C), None


def batch(emissions, kind, trans_w=None, input_lens=None, blank=0, K=16, N=1):
    """The call's outputs for a batch: emissions [B, T, C] (float, widened), trans_w flat or None, input_lens [B] or
    None -> dict(tokens [B, N, T] int32, lengths [B, N] int32, scores [B, N] float64, status [B] int32,
    margin [B] float64)"""
    e = np.asarray(emissions, np.float64)
    B, T, C = e.shape
    W, start = split_weights(kind, trans_w, C)
    tokens = np.full((B, N, T), -1, np.int32)
    lengths = np.full((B, N), -1, np.int32)
    scores = np.full((B, N), NEG)
    status = np.zeros(B, np.int32)
    margin = np.full(B, np.inf)
    for b in range(B):
        Tb = T if input_lens is None else int(input_lens[b])
        if not 0 <= Tb <= T:
            status[b], scores[b] = 2, np.nan
            continue
        used = [e[b, :Tb]]
        if kind != CTC and Tb > 0:
            used.append(np.asarray(trans_w, np.float64))
        if any(np.isnan(u).any() or (u == np.inf).any() for u in used):
            status[b], scores[b] = 1, np.nan
            continue
        r = search(e[b, :Tb], kind, W, start, blank, K, N)
        for n, (y, sc) in enumerate(r["hyps"]):
            tokens[b, n, :len(y)] = y
            lengths[b, n] = len(y)
            scores[b, n] = sc
        status[b] = 3 if r["tie"] else 0
        margin[b] = r["margin"]
    return dict(tokens=tokens, lengths=lengths, scores=scores, status=status, margin=margin)


def numerator(e, kind, y, W=None, start=None, blank=0):
    """float64 forward score of the numerator graph for transcript y (every alignment; the value the beam's score
    bounds from below): e [T_b, C]"""
    e = np.asarray(e, np.float64)
    Tb, C = e.shape
    y = list(y)
    if kind == ASG:
        if not y or Tb < len(y):
            return NEG
        a = np.full(len(y), NEG)
        a[0] = start[y[0]] + e[0, y[0]]
        for t in range(1, Tb):
            stay = a + np.array([W[c, c] for c in y])
            move = np.concatenate([[NEG], a[:-1] + np.array([W[y[u + 1], y[u]] for u in range(len(y) - 1)])])
            a = _lae(stay, move) + e[t, y]
        return float(a[-1])
    lab = [blank] + sum([[c, blank] for c in y], [])
    S = len(lab)
    a = np.full(S, NEG)
    if Tb == 0:
        return NEG

    def w(dst, src):
        return 0.0 if kind == CTC else W[dst, src]
    sigma = _logsumexp_rows(W) if kind == BIGRAM else None
    a[0] = (0.0 if kind == CTC else sigma[lab[0]]) + e[0, lab[0]]
    if S > 1:
        a[1] = (0.0 if kind == CTC else sigma[lab[1]]) + e[0, lab[1]]
    for t in range(1, Tb):
        n = np.full(S, NEG)
        for s in range(S):
            v = a[s] + w(lab[s], lab[s])
            if s >= 1:
                v = _lae(v, a[s - 1] + w(lab[s], lab[s - 1]))
            if s >= 2 and lab[s] != blank and lab[s] != lab[s - 2]:
                v = _lae(v, a[s - 2] + w(lab[s], lab[s - 2]))
            n[s] = v + e[t, lab[s]]
        a = n
    return float(_lae(a[-1], a[-2]) if S > 1 else a[-1])
