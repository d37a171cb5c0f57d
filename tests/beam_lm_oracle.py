"""A float64 restatement of gtnb_beam_decode_lm_async (include/gtn_b200.h): tests/beam_oracle.py's prefix beam search
with a token LM fused into the ranking, an insertion bonus and per-frame token pruning.

The LM is resolved by walking it, not through a dense table: from node s, token c takes the arc of s labelled c, else
s's epsilon (backoff) arc and c again from its destination, adding the backoff weights on the way; -inf when neither
exists.  The end weight of a node is the resolution of label C, or 0 everywhere when the graph has no arc labelled C.

A beam is (transcript, p_blank, p_label, LM node, lmacc).  Candidates are ranked by the fused key
am + (alpha * lmacc + beta * len) and then by the tie rule of beam_oracle (kept before extensions, previous slot,
token).  With token_beam P < C a frame's extensions use only the P eligible tokens of highest emission (blank is not
eligible for CTC and n-gram CTC), ties to the lower token; equal finite emissions at the boundary count as a tie.
After the last frame each beam adds its end weight (dropped at -inf) and the live beams are ranked again by the final
fused score, ties to the earlier beam.  Every utterance reports its smallest nonzero decision margin, as beam_oracle
does, over the fused keys and the final order.
"""
import numpy as np

from tests import beam_oracle as bo

CTC, BIGRAM, ASG = bo.CTC, bo.BIGRAM, bo.ASG
NEG = -np.inf
EPS = -1


class LM:
    """G: a graph dict (tests/graph_oracle.make) over labels [0, C] and EPS; w its arc weights"""

    def __init__(self, G, w, C):
        self.C, self.S = C, len(G["flags"])
        self.w = np.asarray(w, np.float64)
        self.dst = np.asarray(G["dst"])
        self.arc, self.eps = {}, {}
        for a, (s, l) in enumerate(zip(G["src"], G["ilabel"])):
            if l == EPS:
                self.eps[int(s)] = a
            else:
                self.arc[(int(s), int(l))] = a
        self.has_end = any(int(l) == C for l in G["ilabel"])
        self.start = int(np.flatnonzero(np.asarray(G["flags"]) & 1)[0])
        self._memo = {}

    def resolve(self, s, c):
        """-> (weight, destination node) of token c from node s; (-inf, -1) when it is forbidden"""
        r = self._memo.get((s, c))
        if r is None:
            r = self._memo[(s, c)] = self._walk(s, c)
        return r

    def _walk(self, s, c):
        acc = 0.0
        while True:
            a = self.arc.get((s, c))
            if a is not None:
                return acc + self.w[a], int(self.dst[a])
            e = self.eps.get(s)
            if e is None:
                return NEG, -1
            acc += self.w[e]
            s = int(self.dst[e])

    def end(self, s):
        return self.resolve(s, self.C)[0] if self.has_end else 0.0

    def score(self, y):
        """LM(y): the resolved weights along y plus the end weight of the node reached"""
        s, tot = self.start, 0.0
        for c in y:
            x, s = self.resolve(s, int(c))
            if x == NEG:
                return NEG
            tot += x
        return tot + self.end(s)


class NoLM:
    """lm NULL: every weight 0"""
    start = 0

    def resolve(self, s, c):
        return 0.0, 0

    def end(self, s):
        return 0.0

    def score(self, y):
        return 0.0


def pruned_tokens(et, kind, blank, P):
    """(the frame's tokens in ascending order, boundary tie) for token_beam P"""
    C = len(et)
    if P >= C:
        return list(range(C)), False
    elig = [c for c in range(C) if kind == ASG or c != blank]
    order = sorted(elig, key=lambda c: (-et[c], c))
    tie = len(order) > P and et[order[P - 1]] == et[order[P]] and et[order[P]] > NEG
    return sorted(order[:P]), tie


def search(e, kind, W=None, start=None, blank=0, K=16, N=1, lm=None, alpha=1.0, beta=0.0, P=None):
    """One utterance -> dict(hyps: list of (transcript, fused score, am, lm) of up to N entries, tie, margin)"""
    e = np.asarray(e, np.float64)
    Tb, C = e.shape
    lm = NoLM() if lm is None else lm
    P = C if P is None else P
    if kind != CTC:
        W = np.asarray(W, np.float64).reshape(C, C)
    sigma = bo._logsumexp_rows(W) if kind == BIGRAM else None

    def fuse(am, acc, n):
        return am + (alpha * acc + beta * n)

    beams = [((), 0.0, NEG, lm.start, 0.0)]  # (transcript, p_blank, p_label, node, lmacc)
    margin, tie = np.inf, False
    for t in range(Tb):
        et = e[t]
        toks, ptie = pruned_tokens(et, kind, blank, P)
        tie |= ptie
        index = {b[0]: r for r, b in enumerate(beams)}
        kept = []
        for r, (y, pb, pl, _, _) in enumerate(beams):
            l = y[-1] if y else -1
            if kind == CTC:
                nb = bo._lae(pb, pl) + et[blank]
                nl = pl + et[l] if l >= 0 else NEG
            elif kind == BIGRAM:
                wpb = sigma[blank] if t == 0 else W[blank, blank]
                nb = bo._lae(pb + wpb, pl + W[blank, l] if l >= 0 else NEG) + et[blank]
                nl = pl + W[l, l] + et[l] if l >= 0 else NEG
            else:
                nb = NEG
                nl = pl + W[l, l] + et[l] if l >= 0 else NEG
            kept.append([nb, nl])
        ext = []  # (am, slot, token, node, lmacc)
        for s, (y, pb, pl, node, acc) in enumerate(beams):
            l = y[-1] if y else -1
            for c in toks:
                if kind != ASG and c == blank:
                    continue
                if kind == CTC:
                    v = (pb if c == l else bo._lae(pb, pl)) + et[c]
                else:
                    wpb = (sigma[c] if t == 0 else W[c, blank]) if kind == BIGRAM else start[c]
                    from_pb = pb + wpb if pb > NEG else NEG
                    from_pl = pl + W[c, l] if l >= 0 and pl > NEG and (kind == ASG or c != l) else NEG
                    v = bo._lae(from_pb, from_pl) + et[c]
                if not v > NEG:
                    continue
                r = index.get(y + (c,))
                if r is not None:
                    kept[r][1] = bo._lae(kept[r][1], v)
                    continue
                x, nd = lm.resolve(node, c)
                if x == NEG:
                    continue
                ext.append((float(v), s, c, nd, acc + x))
        cands = []  # (key, kind, slot, token, beam)
        for r, (nb, nl) in enumerate(kept):
            am = bo._lae(nb, nl)
            if am > NEG:
                y, _, _, node, acc = beams[r]
                cands.append((fuse(am, acc, len(y)), 0, r, 0, (y, nb, nl, node, acc)))
        for v, s, c, nd, acc in ext:
            y = beams[s][0] + (c,)
            cands.append((fuse(v, acc, len(y)), 1, s, c, (y, NEG, v, nd, acc)))
        cands.sort(key=lambda x: (-x[0], x[1], x[2], x[3]))
        if len(cands) > K:
            gap = cands[K - 1][0] - cands[K][0]
            margin = min(margin, gap) if gap > 0 else margin
            tie |= gap == 0
        beams = [x[4] for x in cands[:K]]
    fin = []  # (final, slot, transcript, am, lm)
    for r, (y, pb, pl, node, acc) in enumerate(beams):
        we = lm.end(node)
        if we == NEG:
            continue
        am = float(bo._lae(pb, pl))
        fin.append((fuse(am, acc + we, len(y)), r, y, am, acc + we))
    fin.sort(key=lambda x: (-x[0], x[1]))
    for n in range(min(N, len(fin) - 1)):
        gap = fin[n][0] - fin[n + 1][0]
        margin = min(margin, gap) if gap > 0 else margin
        tie |= gap == 0
    return dict(hyps=[(f[2], f[0], f[3], f[4]) for f in fin[:N]], tie=tie, margin=margin)


def batch(emissions, kind, trans_w=None, input_lens=None, blank=0, K=16, N=1, lm=None, alpha=1.0, beta=0.0, P=None):
    """The call's outputs for a batch, as beam_oracle.batch, plus am [B, N] and lm [B, N] (float64)"""
    e = np.asarray(emissions, np.float64)
    B, T, C = e.shape
    W, start = bo.split_weights(kind, trans_w, C)
    out = dict(tokens=np.full((B, N, T), -1, np.int32), lengths=np.full((B, N), -1, np.int32),
               scores=np.full((B, N), NEG), am=np.full((B, N), NEG), lm=np.full((B, N), NEG),
               status=np.zeros(B, np.int32), margin=np.full(B, np.inf))
    for b in range(B):
        Tb = T if input_lens is None else int(input_lens[b])
        if not 0 <= Tb <= T:
            out["status"][b] = 2
            for k in ("scores", "am", "lm"):
                out[k][b] = np.nan
            continue
        used = [e[b, :Tb]]
        if kind != CTC and Tb > 0:
            used.append(np.asarray(trans_w, np.float64))
        if any(np.isnan(u).any() or (u == np.inf).any() for u in used):
            out["status"][b] = 1
            for k in ("scores", "am", "lm"):
                out[k][b] = np.nan
            continue
        r = search(e[b, :Tb], kind, W, start, blank, K, N, lm, alpha, beta, P)
        for n, (y, sc, am, lmv) in enumerate(r["hyps"]):
            out["tokens"][b, n, :len(y)] = y
            out["lengths"][b, n] = len(y)
            out["scores"][b, n], out["am"][b, n], out["lm"][b, n] = sc, am, lmv
        out["status"][b] = 3 if r["tie"] else 0
        out["margin"][b] = r["margin"]
    return out


def resolved_graph(lm):
    """The resolved LM as an epsilon-free graph dict and weights: node s has an arc for every token c in [0, C] that
    does not resolve to -inf, to its destination (label C to a new final node); only that node accepts.  Its
    forwardScore(compose(linear(y + [C]), G)) is LM(y) for an LM with eos arcs, and the same with an end weight
    of 0 otherwise."""
    S = lm.S
    src, dst, lab, w = [], [], [], []
    for s in range(S):
        for c in range(lm.C):
            x, d = lm.resolve(s, c)
            if x > NEG:
                src.append(s), dst.append(d), lab.append(c), w.append(x)
        x = lm.end(s)
        if x > NEG:
            src.append(s), dst.append(S), lab.append(lm.C), w.append(x)
    flags = np.zeros(S + 1, np.uint8)
    flags[lm.start] |= 1
    flags[S] = 2
    return dict(flags=flags, src=np.asarray(src, np.int32), dst=np.asarray(dst, np.int32),
                ilabel=np.asarray(lab, np.int32), olabel=np.asarray(lab, np.int32)), np.asarray(w, np.float32)
