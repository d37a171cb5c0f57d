"""Test infrastructure for gtnb_graph_loss (one user-supplied target graph per utterance):

    loss_b = forwardScore(E_b) - forwardScore(intersect(A_b, E_b))

with E_b = linearGraph(T_b, C) on the first T_b rows of utterance b, each utterance run alone.

- ``ref_graph_loss``: the live reference (oracle/_ref), utterance by utterance, with compose(A_b, E_b) (A_b matched on
  its olabels, as the device call matches it).  T_b = 0 is NaN with no gradient: linearGraph(0, C) accepts nothing.
- ``tables``: the in-arc tables the device builder (gtnb_compose_linear's) makes of a graph, for the kernel emulation.
- graph builders: CTC graphs, word-piece decomposition graphs built with a graph library's own union / closure /
  compose / remove (the reference's here, gtn_b200.gtn's on the GPU), the same with a wildcard state at each end,
  and random arc-labelled graphs.  A graph is a dict of numpy arrays: flags, src, dst, ilabel, olabel, w.
"""
import numpy as np

from oracle import pyoracle as po

EPS = -1


def make(flags, src, dst, ilabel, olabel=None, w=None):
    ilabel = np.asarray(ilabel, np.int32)
    return dict(flags=np.asarray(flags, np.uint8), src=np.asarray(src, np.int32), dst=np.asarray(dst, np.int32),
                ilabel=ilabel, olabel=ilabel.copy() if olabel is None else np.asarray(olabel, np.int32),
                w=np.zeros(len(ilabel), np.float32) if w is None else np.asarray(w, np.float32))


def ref_graph(g):
    return po.RefGraph.from_arrays(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"])


def from_ref(rg):
    a = rg.arrays()
    return make(a["flags"], a["src"], a["dst"], a["ilabel"], a["olabel"], a["w"])


def ref_graph_loss(emissions, graphs, input_lens=None, weights=None):
    """-> (losses [B], grads [B, T, C] (zero beyond T_b), arc_grads [sum A_b] in batch order)"""
    e = np.asarray(emissions, np.float32)
    B, T, C = e.shape
    losses, grads = np.zeros(B, np.float32), np.zeros_like(e)
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
        ag = ref_graph(g)
        E = po.RefGraph.linear(Tb, C, e[b, :Tb].ravel())
        num = po.ref_op("forward_score", po.ref_op("compose", ag, E))
        den = po.ref_op("forward_score", E)
        loss = po.ref_op("subtract", den, num)
        po.ref_backward(loss)
        losses[b] = loss.item()
        grads[b, :Tb] = E.grad().weights().reshape(Tb, C)
        arc_grads.append(ag.grad().weights() if A else np.zeros(0, np.float32))
    return losses, grads, (np.concatenate(arc_grads) if arc_grads else np.zeros(0, np.float32))


def tables(g, C):
    """in-arc tables as the device builder makes them: per destination, arcs by (source, position in the source's
    out list); arcs labelled outside [0, C) left out.  -> (in_ptr, in_src, in_label, in_arc, in_w)"""
    N = len(g["flags"])
    order = sorted(range(len(g["src"])), key=lambda a: (int(g["dst"][a]), int(g["src"][a]), a))
    ptr, src, lab, arc, w = [0] * (N + 1), [], [], [], []
    for a in order:
        c = int(g["olabel"][a])
        if 0 <= c < C:
            src.append(int(g["src"][a]))
            lab.append(c)
            arc.append(a)
            w.append(float(g["w"][a]))
            ptr[int(g["dst"][a]) + 1] += 1
    ptr = np.cumsum(ptr).astype(np.int32)
    return (ptr, np.asarray(src, np.int32), np.asarray(lab, np.int32), np.asarray(arc, np.int32),
            np.asarray(w, np.float32))


def non_uniform_nodes(g, C):
    ptr, _, lab, _, _ = tables(g, C)
    return sum(len(set(lab[ptr[n]:ptr[n + 1]].tolist())) > 1 for n in range(len(ptr) - 1))


def ctc_graph(target, blank=0, w=None):
    """benchmarks/ctc.cpp:40-58: 2U+1 nodes, self loops, steps and skips where consecutive labels differ"""
    L = 2 * len(target) + 1
    lab = [blank if i % 2 == 0 else int(target[i // 2]) for i in range(L)]
    flags = np.zeros(L, np.uint8)
    flags[0] |= 1
    flags[L - 1] |= 2
    if L > 1:
        flags[L - 2] |= 2
    src, dst, il = [], [], []
    for i in range(L):
        src.append(i), dst.append(i), il.append(lab[i])
        if i + 1 < L:
            src.append(i), dst.append(i + 1), il.append(lab[i + 1])
        if i + 2 < L and lab[i + 2] != blank and lab[i + 2] != lab[i]:
            src.append(i), dst.append(i + 2), il.append(lab[i + 2])
    g = make(flags, src, dst, il)
    if w is not None:
        g["w"] = np.asarray(w, np.float32)
    return g


def inventory(n_letters=26, C=256, seed=7):
    """word pieces: the letters, then seeded random 2- and 3-letter pieces; C - 1 pieces (label C - 1 is unused
    by the pieces, as a CTC blank would be)"""
    rng = np.random.default_rng(seed)
    pieces = [(i,) for i in range(n_letters)]
    seen = set(pieces)
    while len(pieces) < C - 1:
        p = tuple(int(x) for x in rng.integers(0, n_letters, int(rng.integers(2, 4))))
        if p not in seen:
            seen.add(p)
            pieces.append(p)
    return pieces


def decomposition_graph(ops, letters, pieces):
    """the alignment graph of word_decompositions.py with a graph library's own host ops:
    decomps = remove(project_output(compose(transcript, closure(union(lexicon))))),
    alignments = project_input(remove(compose(closure(union(tokens)), decomps))).
    ops: dict of callables graph(arrays), union(list), closure, compose, remove, project_input, project_output."""
    lex = []
    for i, wp in enumerate(pieces):
        n = len(wp)
        flags = [1] + [0] * (n - 1) + [2]
        lex.append(ops["graph"](make(flags, list(range(n)), list(range(1, n + 1)), list(wp),
                                     [EPS] * (n - 1) + [i])))
    lexicon = ops["closure"](ops["union"](lex))
    U = len(letters)
    transcript = ops["graph"](make([1] + [0] * (U - 1) + [2], list(range(U)), list(range(1, U + 1)), letters))
    decomps = ops["remove"](ops["project_output"](ops["compose"](transcript, lexicon)))
    tokens = [ops["graph"](make([1, 2], [0, 1], [1, 1], [i, i], [i, EPS])) for i in range(len(pieces))]
    return ops["project_input"](ops["remove"](ops["compose"](ops["closure"](ops["union"](tokens)), decomps)))


REF_OPS = dict(
    graph=ref_graph, union=po.ref_union, closure=po.ref_closure,
    compose=lambda a, b: po.ref_op("compose", a, b), remove=po.ref_remove,
    project_input=lambda g: po.ref_clone(g, 1), project_output=lambda g: po.ref_clone(g, 2))


def with_wildcards(g, C, w_loop=0.0):
    """a wildcard state at each end: a new start node with one self-loop per label that leads into the graph (a copy
    of every out-arc of the start nodes), and a new accept node with one self-loop per label entered the way the
    accept nodes are (a copy of every in-arc of the accept nodes), so that the frames before and after the graph
    match anything.  The graph's own start and accept nodes keep their roles."""
    N = len(g["flags"])
    ws, we = N, N + 1
    flags = np.concatenate([g["flags"], np.asarray([1, 2], np.uint8)])
    src, dst, lab, w = list(g["src"]), list(g["dst"]), list(g["olabel"]), list(g["w"])
    A = len(src)
    for c in range(C):
        src.append(ws), dst.append(ws), lab.append(c), w.append(w_loop)
    for a in range(A):
        if g["flags"][g["src"][a]] & 1:
            src.append(ws), dst.append(int(g["dst"][a])), lab.append(int(g["olabel"][a])), w.append(float(g["w"][a]))
    for c in range(C):
        src.append(we), dst.append(we), lab.append(c), w.append(w_loop)
    for a in range(A):
        if g["flags"][g["dst"][a]] & 2:
            src.append(int(g["src"][a])), dst.append(we), lab.append(int(g["olabel"][a])), w.append(float(g["w"][a]))
    return make(flags, src, dst, lab, w=w)


def random_graph(rng, N, A, C, n_start=2, n_accept=2, label_hi=None, w_scale=1.0):
    """random arc-labelled graph with cycles and self-loops, several start and accept nodes; labels in
    [0, label_hi) (label_hi > C: some arcs can never match)"""
    label_hi = C if label_hi is None else label_hi
    flags = np.zeros(N, np.uint8)
    flags[rng.choice(N, min(n_start, N), replace=False)] |= 1
    flags[rng.choice(N, min(n_accept, N), replace=False)] |= 2
    src = rng.integers(0, N, A)
    dst = rng.integers(0, N, A)
    lab = rng.integers(0, label_hi, A)
    w = rng.uniform(-w_scale, w_scale, A).astype(np.float32)
    return make(flags, src, dst, lab, w=w)
