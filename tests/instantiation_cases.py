"""The case table of tests/test_gpu_instantiations.py: small batches chosen on both sides of every boundary of the five
launch plans (bidir_plan, dense_lanes, ngram_den_shape, wide_lanes, staged plan / fused_layout), so that every kernel
instantiation a plan can return runs on the device against a float64 referee.

Plain data and generators, importable without a GPU.  Each case names its family, the public entry point, the dtype,
B / T / C, the per-utterance frame counts and targets (or graphs) and the context flags it sets; plan_inputs(case)
computes the plan's inputs from the case's own data (max_nodes = 2U + 1 over the batch, the graphs' arc and node
counts, ...), and tests/test_plan_coverage.py maps every case to its plan outcome through tests/emu/plan_emu.cpp.

The boundary sits in utterance 0 of a ragged batch; the utterances beside it are smaller (so the batch maxima are
utterance 0's) and carry the edges the entry point allows: T_b = 1, U = 0, repeated labels, an infeasible target.
A column of -inf emissions (a label impossible on every frame) goes to the dense Viterbi decoder only: the loss kernels
raise their status bit on a non-finite emission and repeat the batch on another route, which is tested elsewhere.
Dense Viterbi cases alternate uniform emissions with small integers (exact float32 sums, so ties are exact and the
first predecessor must win).
"""
from dataclasses import dataclass, field

import numpy as np

F32, BF16, F16 = 0, 1, 2  # capi.F32 / BF16 / F16
DTYPES = (F32, BF16, F16)
ESIZE = {F32: 4, BF16: 2, F16: 3}  # plan_emu's element selector (3: fp16, two bytes like bf16)
DTYPE_NAME = {F32: "f32", BF16: "bf16", F16: "f16"}


@dataclass
class Case:
    family: str  # "bidir", "dense", "ngram", "staged", "implicit"
    entry: str  # the public entry point
    dtype: int
    C: int
    T_b: list  # frames per utterance
    targets: list = None  # label sequences (CTC, n-gram CTC, ASG)
    graphs: list = None  # (N, src, dst, labels, weights) per utterance (compose_linear)
    kind: str = ""  # dense / trellis: "asg" or "bigram"
    flags: dict = field(default_factory=dict)  # gtnb_ctx_set_flag before the call
    ties: bool = False  # integer-valued emissions and transitions
    neg_col: int = -1  # a label whose emissions are -inf on every frame
    seed: int = 0
    name: str = ""
    expect: dict = None  # staged CTC cases: whether the staged kernels and the fused backward run

    @property
    def B(self):
        return len(self.T_b)

    @property
    def T(self):
        return max(self.T_b)

    @property
    def id(self):
        return "%s-%s-%s-C%d-%s%s" % (self.family, self.entry, DTYPE_NAME[self.dtype], self.C, self.kind, self.name)


# ---- plan inputs, computed from the case's own data ---------------------------------------------------------------


def ctc_graph_size(target):
    """(nodes, arcs) of the CTC graph of target: 2U + 1 nodes, a self loop each, U step arcs into labels and U into
    blanks, a skip arc between different consecutive labels"""
    U = len(target)
    skips = sum(1 for i in range(1, U) if target[i] != target[i - 1])
    return 2 * U + 1, (2 * U + 1) + 2 * U + skips


def plan_inputs(case):
    """the inputs of the case's plan, as tests/test_plan_coverage.py passes them to plan_emu"""
    if case.family == "bidir":
        max_nodes = max(2 * len(t) + 1 for t in case.targets)
        pair_ok = int(case.flags.get("bidir_mode", -1) != 0)
        # gtnb_compose_linear gives implicit lattices of up to 224 nodes the fixed pitch; CTC graphs have degree <= 3
        return dict(C=case.C, max_nodes=max_nodes, max_in=3, max_out=3, fixed_pitch=int(max_nodes <= 224),
                    pair_ok=pair_ok, esize=ESIZE[case.dtype])
    if case.family == "dense":
        return dict(C=case.C, bigram=int(case.kind == "bigram"), esize=ESIZE[case.dtype])
    if case.family == "ngram":
        return dict(C=case.C, start=int(case.kind == "asg"), esize=ESIZE[case.dtype])
    if case.family == "implicit":
        dims = [graph_dims(g) for g in case.graphs]
        return dict(max_in=max(d[0] for d in dims), max_out=max(d[1] for d in dims),
                    max_nodes=max(g[0] for g in case.graphs), C=case.C, arc=int(not all(d[2] for d in dims)),
                    trop=int(case.kind == "viterbi"), gg=int(case.kind == "loss-gg"))
    if case.family == "staged":
        if case.graphs is not None:
            sizes = [(g[0], len(g[1])) for g in case.graphs]
        else:
            sizes = [ctc_graph_size(t) for t in case.targets]
        # compose_linear: one level per frame plus the first, the operand's node and arc counts as level bounds
        return dict(L=[t + 1 for t in case.T_b], sg_A=[a for _, a in sizes], sg_N=[n for n, _ in sizes],
                    max_lvl_nodes=max(n for n, _ in sizes), max_lvl_arcs=max(a for _, a in sizes))
    raise ValueError(case.family)


def graph_dims(g):
    """(largest in-degree, largest out-degree, label-uniform: every node's in-arcs carry one label) of a graph"""
    N, src, dst, lab, _ = g
    uniform = all(len(set(lab[dst == n].tolist())) <= 1 for n in range(N))
    return int(np.bincount(dst, minlength=N).max()), int(np.bincount(src, minlength=N).max()), uniform


def numerator_dims(case):
    """(largest in-degree, nodes) of the numerator graphs the trellis criteria sweep with k_implicit.cu: n-gram CTC's
    folded CTC graph (2U + 2 nodes: the start S, then ctcGraph's, each with a self loop, a step and a skip arc in),
    ASG's forced-alignment chain (U + 1 nodes: a step arc and a self loop)"""
    if case.kind == "bigram":
        skip = any(t[i] != t[i - 1] for t in case.targets for i in range(1, len(t)))
        return 3 if skip else 2, max(2 * len(t) + 2 for t in case.targets)
    return 2, max(len(t) + 1 for t in case.targets)


# ---- generators ---------------------------------------------------------------------------------------------------


def distinct_target(U, C, rng, blank=0):
    """U labels in [0, C) other than blank, no two consecutive alike (every skip arc present)"""
    labels = [c for c in range(C) if c != blank]
    out = []
    for _ in range(U):
        choices = [c for c in labels if not out or c != out[-1]] or labels
        out.append(int(rng.choice(choices)))
    return out


def label_batch(C, U0, T0, rng, blank=None, companions=True):
    """utterance 0: U0 labels in T0 frames (the boundary); then T_b = 1 with U = 0, repeated labels, and an
    infeasible target (more labels than frames), all smaller than utterance 0"""
    skip = {blank} if blank is not None else set()
    pool = [c for c in range(C) if c not in skip]
    T_b = [T0]
    tg = [distinct_target(U0, C, rng, blank if blank is not None else -1) if pool else []]
    if companions and pool:
        small = max(1, min(U0, 3))
        rep = int(pool[0])
        T_b += [1, min(T0, 2 * small + 3), min(T0, 2)]
        tg += [[], [rep] * small, [pool[-1]] * min(small, 1) + [pool[0]] * 3]
    return T_b, tg


def bidir_cases():
    out = []
    rng = np.random.default_rng(11)
    # (C, U0, flags, name): NQ 1 / 2, FX or not, PAIR or one node per thread; the PAIR bound (U = 111: 223 nodes) and the
    # support bound (U = 112: 225 nodes, not bidirectional)
    shapes = [(8, 20, {}, "nq1"), (56, 20, {}, "nq1-high"), (60, 20, {}, "nq1-high"), (64, 20, {}, "pair-nq1"),
              (64, 20, {"bidir_mode": 0}, "fx-nq1"), (68, 20, {}, "nq2-low"), (72, 20, {}, "nq2-low"),
              (120, 20, {}, "nq2-high"), (124, 20, {}, "nq2-high"), (128, 20, {}, "pair-nq2"),
              (128, 20, {"bidir_mode": 0}, "fx-nq2"), (64, 111, {}, "pair-max"), (64, 112, {}, "over-support"),
              (128, 111, {"bidir_mode": 0}, "fx-max"), (40, 111, {}, "nq1-max"), (40, 112, {}, "over-support"),
              (128, 112, {"bidir_mode": 0}, "over-support"), (16, 1, {}, "u1")]
    # the same alphabet boundaries with one node per thread asked for (bidir_mode 0)
    shapes += [(C, 20, {"bidir_mode": 0}, "mode0") for C in (56, 60, 68, 72, 120, 124)]
    for dtype in DTYPES:
        for C, U0, flags, name in shapes:
            if dtype != F32 and C % 8:
                continue
            T_b, tg = label_batch(C, U0, 2 * U0 + 6, rng, blank=0)
            out.append(Case("bidir", "gtnb_ctc_loss_ex", dtype, C, T_b, targets=tg, flags=dict(flags), seed=C + U0,
                            name=name))
    # 16-bit with C % 4 == 0 but not % 8: the shape rules refuse, the call is widened
    T_b, tg = label_batch(12, 5, 16, rng, blank=0)
    out.append(Case("bidir", "gtnb_ctc_loss_ex", BF16, 12, T_b, targets=tg, seed=12, name="c12-half"))
    return out


# the first and last C of each dense lane count (dense_lanes), and the support limit
DENSE_CS = (1, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 224, 225)


def dense_cases():
    out = []
    for dtype in DTYPES:
        for kind in ("asg", "bigram"):
            for i, C in enumerate(DENSE_CS):
                ties = bool(i % 2)
                T_b = [7, 1, 0, 4]
                out.append(Case("dense", "gtnb_viterbi_dense_typed", dtype, C, T_b, kind=kind, ties=ties,
                                neg_col=C - 1 if C > 1 else -1, seed=C * 7 + (kind == "asg"), name="t%d" % ties))
    return out


# the first and last C of each trellis shape (ngram_den_shape), and the trellis limit 128
NGRAM_CS = (2, 16, 17, 32, 33, 64, 65, 128)


def ngram_cases():
    out = []
    rng = np.random.default_rng(5)
    for dtype in DTYPES:
        for kind in ("bigram", "asg"):
            for C in NGRAM_CS:
                blank = 0 if kind == "bigram" else None
                U0 = min(6, C - 1) if kind == "bigram" else 6
                T_b, tg = label_batch(C, U0, 2 * U0 + 4, rng, blank=blank)
                entry = "gtnb_ngram_ctc_loss_typed" if kind == "bigram" else "gtnb_asg_loss_typed"
                out.append(Case("ngram", entry, dtype, C, T_b, targets=tg, kind=kind, seed=C, name=kind))
    return out


def dense_graph(N, A, C, rng):
    """a DAG of N nodes (start 0, accept N - 1) with A arcs: the chain 0 -> 1 -> ... -> N-1, then arcs between random
    ordered pairs (parallel arcs allowed), random labels and weights"""
    src = list(range(N - 1))
    dst = list(range(1, N))
    while len(src) < A:
        s = int(rng.integers(0, N - 1))
        src.append(s)
        dst.append(int(rng.integers(s + 1, N)))
    lab = rng.integers(0, C, A).astype(np.int32)
    w = rng.uniform(-1, 1, A).astype(np.float32)
    return (N, np.asarray(src, np.int32), np.asarray(dst, np.int32), lab, w)


def staged_cases():
    out = []
    rng = np.random.default_rng(3)
    # the batch's average degree (16 nodes; A0 + 6 arcs) on both sides of 4, 16 and 48 (G = 1 / 4 / 16 / 32):
    # compose_linear + forward / backward / path
    for A0 in (58, 59, 250, 251, 762, 763):
        N, C = 8, 5
        graphs = [dense_graph(N, A0, C, rng), dense_graph(5, 4, C, rng), dense_graph(3, 2, C, rng)]
        T_b = [5, 4, 1]  # the chain graphs need N - 1 frames: utterance 1 has them, utterance 2 does not (infeasible)
        out.append(Case("staged", "gtnb_compose_linear", F32, C, T_b, graphs=graphs, flags={"staged": 1},
                        name="deg%d-%d" % (A0, N)))
    # CTC graphs of U labels through the materialised criterion (implicit 0): the staged layout's three stage counts,
    # the fused backward's 200 KB refusal, and the plan's refusal (the generic kernels)
    # (U0, the staged kernels run, the fused backward runs), with T0 = U0 + 8 frames
    for U0, staged, fused in ((205, 1, 1), (206, 1, 1), (384, 1, 1), (385, 1, 1), (864, 1, 1), (865, 1, 0),
                              (1341, 1, 0), (1342, 0, 0)):
        C = 20
        T_b, tg = label_batch(C, U0, U0 + 8, rng, blank=0)
        out.append(Case("staged", "gtnb_ctc_loss", F32, C, T_b, targets=tg, flags={"implicit": 0, "staged": 1},
                        expect=dict(staged=staged, fused=fused), name="u%d" % U0))
    return out


def hub_graph(N, deg, C, rng, arc=False):
    """N nodes (start 0, accept N - 1), a self loop on every node and the chain 0 -> 1 -> ... -> N-1; the accept node
    gets deg in-arcs in all (its self loop, the chain's and deg - 2 more from the other nodes in turn).  Each node's
    in-arcs carry one label unless arc, where the accept node's extra in-arcs take random labels."""
    node_lab = rng.integers(0, C, N)
    src = list(range(N)) + list(range(N - 1))
    dst = list(range(N)) + list(range(1, N))
    for k in range(deg - 2):
        src.append(k % (N - 1))
        dst.append(N - 1)
    src, dst = np.asarray(src, np.int32), np.asarray(dst, np.int32)
    lab = node_lab[dst].astype(np.int32)
    if arc:
        extra = np.arange(2 * N - 1, len(src))
        lab[extra] = rng.integers(0, C, len(extra))
    w = rng.uniform(-1, 1, len(src)).astype(np.float32)
    return (N, src, dst, lab, w)


# the in-degrees on both sides of each wide_lanes step (kWideCap = 20 in-arcs per lane: 3 | 4, 20 | 21, ..., 640 | 641)
IMPLICIT_DEGS = (3, 4, 20, 21, 40, 41, 80, 81, 160, 161, 320, 321, 640, 641)


def implicit_cases():
    """gtnb_graph_loss (with and without the graphs' arc gradient) and gtnb_graph_viterbi on graphs whose accept node
    has the boundary in-degree, label-uniform and not; and the node-count limit of the wide kernels (256 | 257)"""
    out = []
    rng = np.random.default_rng(17)
    C = 6
    shapes = [(8, d) for d in IMPLICIT_DEGS] + [(256, 21), (257, 21)]
    for arc in (False, True):
        for N, deg in shapes:
            for kind in ("loss", "loss-gg", "viterbi"):
                graphs = [hub_graph(N, deg, C, rng, arc), hub_graph(5, 3, C, rng), hub_graph(3, 3, C, rng)]
                T_b = [N + 2, 1, 4]  # utterance 1: no path of one arc from start to accept (infeasible)
                entry = "gtnb_graph_viterbi" if kind == "viterbi" else "gtnb_graph_loss"
                out.append(Case("implicit", entry, F32, C, T_b, graphs=graphs, kind=kind, seed=N * 1000 + deg,
                                name="-N%d-deg%d%s" % (N, deg, "-arc" if arc else "")))
    return out


def all_cases():
    return bidir_cases() + dense_cases() + ngram_cases() + staged_cases() + implicit_cases()


# ---- data -----------------------------------------------------------------------------------------------------------


def round_to(x, dtype):
    """float32 array rounded to the case's dtype and widened back (exact), round to nearest even"""
    x = np.asarray(x, np.float32)
    if dtype == F32:
        return x
    if dtype == F16:
        return x.astype(np.float16).astype(np.float32)
    b = x.view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) >> 16 << 16
    return b.astype(np.uint32).view(np.float32)


def emissions(case):
    """[B, T, C] float32 holding values exactly representable in the case's dtype"""
    rng = np.random.default_rng(1000 + case.seed)
    shape = (case.B, case.T, case.C)
    if case.ties:
        e = rng.integers(-2, 3, shape).astype(np.float32)
    else:
        e = rng.uniform(-3, 3, shape).astype(np.float32)
    e = round_to(e, case.dtype)
    if case.neg_col >= 0:
        e[:, :, case.neg_col] = -np.inf
    return e


def transitions(case):
    """ASG: [C start weights] ++ [C x C]; bigram: [C x C], row = destination (float32, used as is)"""
    rng = np.random.default_rng(2000 + case.seed)
    n = case.C * case.C + (case.C if case.kind == "asg" else 0)
    if case.ties:
        return rng.integers(-1, 2, n).astype(np.float32)
    return rng.uniform(-1, 1, n).astype(np.float32)
