"""A numpy restatement of gtnb_edit_distance_async's contract, the referee of its tests.

- units: the tokens (word_sep None or < 0), or the words of the sequence, maximal runs of tokens other than word_sep,
  compared by their exact token spans;
- D[i][j] = min(D[i-1][j-1] + (h_i != r_j), D[i-1][j] + 1 (insertion), D[i][j-1] + 1 (deletion)), D[i][0] = i,
  D[0][j] = j, with i counting hypothesis units and j reference units;
- every cell picks one predecessor, preferring the diagonal, then a deletion, then an insertion; the counts and the
  alignment are those of the chain of chosen predecessors from the last cell back to (0, 0).
"""
import numpy as np

DIAG, DEL, INS = 0, 1, 2


def words(seq, sep):
    """the words of seq as tuples of tokens"""
    out, cur = [], []
    for t in seq:
        if t == sep:
            if cur:
                out.append(tuple(cur))
            cur = []
        else:
            cur.append(int(t))
    if cur:
        out.append(tuple(cur))
    return out


def units(hyp, ref, word_sep=None):
    """(hypothesis units, reference units) as int lists; in word mode, equal words share an id"""
    if word_sep is None or word_sep < 0:
        return [int(t) for t in hyp], [int(t) for t in ref]
    hw, rw = words(hyp, word_sep), words(ref, word_sep)
    ids = {}
    for w in hw + rw:
        ids.setdefault(w, len(ids))
    return [ids[w] for w in hw], [ids[w] for w in rw]


def grid(h, r):
    """D [n+1][m+1] and the chosen move of every cell (DIAG / DEL / INS; -1 at (0, 0)), one row at a time: with
    A[j] = min(D[i-1][j-1] + (h_i != r_j), D[i-1][j] + 1) and A[0] = i, D[i][j] = min over k <= j of A[k] + j - k, a
    running minimum of A[k] - k.  The move is the first of diagonal, deletion, insertion that reaches D[i][j]."""
    n, m = len(h), len(r)
    h, r = np.asarray(h, np.int64), np.asarray(r, np.int64)
    D = np.zeros((n + 1, m + 1), np.int64)
    mv = np.full((n + 1, m + 1), -1, np.int8)
    D[0] = np.arange(m + 1)
    mv[1:, 0] = INS
    mv[0, 1:] = DEL
    k = np.arange(m + 1)
    for i in range(1, n + 1):
        diag = D[i - 1, :-1] + (r != h[i - 1])
        A = np.concatenate(([i], np.minimum(diag, D[i - 1, 1:] + 1)))
        D[i] = np.minimum.accumulate(A - k) + k
        row = np.full(m, INS, np.int8)
        row[D[i, :-1] + 1 == D[i, 1:]] = DEL
        row[diag == D[i, 1:]] = DIAG
        mv[i, 1:] = row
    return D, mv


def path(h, r, mv=None):
    """the chosen path from (n, m) back to (0, 0): a list of (move, i, j) for the cell each move leaves, last first
    (mv: grid(h, r)'s moves, when already computed)"""
    if mv is None:
        mv = grid(h, r)[1]
    i, j, out = len(h), len(r), []
    while i > 0 or j > 0:
        move = int(mv[i, j])
        out.append((move, i, j))
        if move == DIAG:
            i, j = i - 1, j - 1
        elif move == DEL:
            j -= 1
        else:
            i -= 1
    return out


def edit_distance(hyp, ref, word_sep=None):
    """dict: distance, sub, ins, dele, hyp_units, ref_units, hyp_align, ref_align for one pair"""
    h, r = units(hyp, ref, word_sep)
    D, mv = grid(h, r)
    ha, ra = [-1] * len(h), [-1] * len(r)
    sub = ins = dele = 0
    for move, i, j in path(h, r, mv):
        if move == DIAG:
            ha[i - 1], ra[j - 1] = j - 1, i - 1
            sub += h[i - 1] != r[j - 1]
        elif move == DEL:
            dele += 1
        else:
            ins += 1
    return dict(distance=int(D[-1, -1]), sub=sub, ins=ins, dele=dele, hyp_units=len(h), ref_units=len(r),
                hyp_align=ha, ref_align=ra)


def batch(hyp, hyp_lens, ref, ref_lens, word_sep=None):
    """the C ABI's outputs for padded [B][N] / [B][M] int arrays: distance [B], ops [B][3], units [B][2], status [B],
    hyp_align [B][N], ref_align [B][M] (status 2 for a length outside the bounds: -1 everywhere)"""
    hyp, ref = np.asarray(hyp), np.asarray(ref)
    B, N = hyp.shape
    M = ref.shape[1]
    dist = np.full(B, -1, np.int32)
    ops = np.full((B, 3), -1, np.int32)
    un = np.full((B, 2), -1, np.int32)
    status = np.full(B, 2, np.int32)
    ha = np.full((B, N), -1, np.int32)
    ra = np.full((B, M), -1, np.int32)
    for b in range(B):
        nh, nr = int(hyp_lens[b]), int(ref_lens[b])
        if not (0 <= nh <= N and 0 <= nr <= M):
            continue
        o = edit_distance(hyp[b, :nh], ref[b, :nr], word_sep)
        dist[b], status[b] = o["distance"], 0
        ops[b] = (o["sub"], o["ins"], o["dele"])
        un[b] = (o["hyp_units"], o["ref_units"])
        ha[b, :o["hyp_units"]] = o["hyp_align"]
        ra[b, :o["ref_units"]] = o["ref_align"]
    return dict(distance=dist, ops=ops, units=un, status=status, hyp_align=ha, ref_align=ra)


def edits_graph(C):
    """the reference example's one-state edits transducer over C unit ids, as arrays (epsilon = -1)"""
    src, il, ol, w = [], [], [], []
    for i in range(C):
        for j in range(C):
            il.append(i), ol.append(j), w.append(-float(i != j))
        il.append(i), ol.append(-1), w.append(-1.0)
        il.append(-1), ol.append(i), w.append(-1.0)
    n = len(il)
    return dict(flags=np.array([3], np.uint8), src=np.zeros(n, np.int32), dst=np.zeros(n, np.int32),
                ilabel=np.array(il, np.int32), olabel=np.array(ol, np.int32), w=np.array(w, np.float32))


def chain_graph(seq):
    """an acceptor of exactly seq (node 0 start; the last node accepts, node 0 itself for an empty seq)"""
    n = len(seq)
    flags = np.zeros(n + 1, np.uint8)
    flags[0] |= 1
    flags[n] |= 2
    lab = np.asarray(seq, np.int32).reshape(-1)
    return dict(flags=flags, src=np.arange(n, dtype=np.int32), dst=np.arange(1, n + 1, dtype=np.int32),
                ilabel=lab, olabel=lab, w=np.zeros(n, np.float32))


def path_cost(h, r):
    """the restatement's path recomputed as arcs of the reference lattice: the edits arcs it takes, summed as -w"""
    e = edits_graph(max([0] + list(h) + list(r)) + 1)
    C = int(e["ilabel"].max()) + 1
    cost = 0.0
    for move, i, j in path(h, r):
        if move == DIAG:
            k = h[i - 1] * (C + 2) + r[j - 1]
            assert e["ilabel"][k] == h[i - 1] and e["olabel"][k] == r[j - 1]
        elif move == INS:
            k = h[i - 1] * (C + 2) + C
            assert e["ilabel"][k] == h[i - 1] and e["olabel"][k] == -1
        else:
            k = r[j - 1] * (C + 2) + C + 1
            assert e["ilabel"][k] == -1 and e["olabel"][k] == r[j - 1]
        cost -= float(e["w"][k])
    return cost
