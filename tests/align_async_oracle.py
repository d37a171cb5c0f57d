"""Test infrastructure for the asynchronous forced alignments (gtnb_ctc_align_async, gtnb_ngram_ctc_align_async,
gtnb_asg_align_async): what each utterance's outputs should be, from the live reference and a float32 restatement.

- ``numerator_graph``: the graph whose composition with E_b is aligned, as the synchronous aligners take it: the CTC
  graph of the target (graph_oracle.ctc_graph) for CTC and n-gram CTC, ASG's force-align chain for ASG.
- ``positions``: the target position of every arc of that graph (the node it enters: odd CTC node l -> (l - 1) / 2,
  even -> -1 for blank; chain node n -> n - 1), which turns a path's arcs into tokens.
- ``reference``: paths, scores and tokens from the live reference (oracle/_ref), each utterance alone.
- ``restated``: (score, tie) of the device route's float32 tropical recursion on the device's numerator, and
  ``path_value``: a path's value in the device route's association.
"""
import numpy as np

from tests import graph_oracle as go
from tests import graph_trans_oracle as gto
from tests import graph_trans_viterbi_oracle as gtv
from tests import graph_viterbi_oracle as gv

CTC, NGRAM, ASG = 0, 1, 2


def numerator_graph(kind, y, blank):
    return gto.fal_graph(y) if kind == ASG else go.ctc_graph(y, blank)


def positions(kind, g):
    dst = np.asarray(g["dst"])
    if kind == ASG:
        return (dst - 1).astype(np.int32)
    return np.where(dst % 2 == 1, (dst - 1) // 2, -1).astype(np.int32)


def reference(kind, e, W, targets, lens, il, blank):
    """-> (paths, tokens [B, T] int32, scores [B] float32) of the live reference, utterance by utterance"""
    B, T, C_ = e.shape
    graphs = [numerator_graph(kind, targets[b, :lens[b]], blank) for b in range(B)]
    if kind == CTC:
        paths, scores, arcs = gv.ref_graph_viterbi(e, graphs, il)
    else:
        paths, scores, arcs = gtv.ref_graph_trans_viterbi(e, graphs, gtv.ASG if kind == ASG else gtv.BIGRAM, W, il)
    tokens = np.full((B, T), -1, np.int32)
    for b in range(B):
        pos = positions(kind, graphs[b])
        ok = arcs[b] >= 0
        tokens[b, ok] = pos[arcs[b, ok]]
    return paths, tokens, scores


def restated(kind, e_b, W, y, blank):
    """(score, tie) of the float32 tropical recursion on the device route's numerator of y over e_b [T_b, C]"""
    C_ = e_b.shape[1]
    g = numerator_graph(kind, y, blank)
    if kind == CTC:
        p = dict(g, w=np.zeros(len(g["src"]), np.float32))
    else:
        p, _ = gtv.tropical_product(dict(g, w=np.zeros(len(g["src"]), np.float32)), C_,
                                    gtv.ASG if kind == ASG else gtv.BIGRAM, W)
    return gtv.device_route_outcome(e_b, p, C_)


def path_value(kind, e_b, W, labels):
    """the value of a label path over e_b [T_b, C] in the device route's association: fl(s + fl(w + e)) per frame,
    w = 0 (CTC), tau_l / W[l][l'] (n-gram), s[l] / W[l][l'] (ASG)"""
    C_ = e_b.shape[1]
    tw = None if W is None else np.asarray(W, np.float32).ravel()
    s = np.float32(0.0)
    for t, l in enumerate(labels):
        if kind == CTC:
            w = np.float32(0.0)
        elif kind == NGRAM:
            M = tw.reshape(C_, C_)
            w = M[l].max() if t == 0 else M[l, labels[t - 1]]
        else:
            M = tw[C_:].reshape(C_, C_)
            w = tw[l] if t == 0 else M[l, labels[t - 1]]
        s = np.float32(s + np.float32(np.float32(w) + e_b[t, l]))
    return s


def valid_path(kind, labels, tokens, y, blank):
    """labels / tokens [T_b] follow an accepting path of the numerator of y"""
    U = len(y)
    prev = -1  # the last position met
    seen = []
    for t, (l, u) in enumerate(zip(labels, tokens)):
        if u < 0:
            if kind == ASG or l != blank:
                return False
            continue
        if l != y[u] or u < prev or u > prev + 1 or (kind == ASG and t == 0 and u != 0):
            return False
        after_blank = t > 0 and tokens[t - 1] < 0
        if kind != ASG and u == prev and after_blank:  # blank -> the same label node: no such arc
            return False
        if kind != ASG and u == prev + 1 and prev >= 0 and not after_blank and y[u] == y[prev]:  # no skip arc
            return False
        if u != prev:
            seen.append(u)
        prev = u
    return seen == list(range(U))
