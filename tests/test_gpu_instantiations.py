"""Every case of tests/instantiation_cases.py on the GPU: first the route, read from the context's launch profile, so
that a fall-back cannot pass for the instantiation under test; then the result against a float64 referee that shares
no code with the kernels (oracle/f64.py, tests/ngram_oracle.py, and a float64 dense Viterbi DP here).

16-bit cases hold values exactly representable in the dtype, so the referee evaluates the widened values.  Scores
are held to util.close, gradients to util.grad_close; Viterbi paths and scores to == wherever every decision of the
referee's best path wins by more than 1e-3 (integer-valued cases are exact in float32, ties included, and always
compared); infeasible targets must give what the reference gives (+inf, the denominator's gradient alone)."""
import numpy as np
import pytest
import torch

from gtn_b200 import capi
from oracle import f64
from tests import instantiation_cases as ic
from tests import util
from tests.ngram_oracle import ngram_ctc_f64

pytestmark = pytest.mark.gpu
TORCH = {ic.F32: torch.float32, ic.BF16: torch.bfloat16, ic.F16: torch.float16}
MARGIN = 1e-3
CASES = ic.all_cases()
# unit roundoff of the 16-bit gradients (bf16: 8 significand bits, fp16: 11): a gradient rounded to nearest is within
# ROUND * |g| of the float32 value, which itself is held to util.grad_close's bar
ROUND = {ic.F32: 0.0, ic.BF16: 2.0 ** -8, ic.F16: 2.0 ** -11}
# kernels of the materialised route: a status-word retry of a fast route would launch them
MATERIALISED = {"compose_emit", "sd_forward", "sd_forward_generic", "sd_backward", "sd_backward_generic",
                "sd_backward_fused"}


def of(family):
    return list(filter(lambda case: case.family == family, CASES))


def case_id(case):
    return case.id


@pytest.fixture(scope="module")
def ictx():
    c = capi.Ctx(0)
    yield c
    c.close()


def run(ctx, case, fn):
    """fn() with the case's flags set and the launch profile on -> (fn's result, the names of the launched kernels)"""
    for k, v in case.flags.items():
        ctx.set_flag(k, v)
    try:
        ctx.profile(True)
        ctx.profile_read()
        out = fn()
        names = set(ctx.profile_read())
    finally:
        ctx.profile(False)
        for k in case.flags:
            ctx.set_flag(k, {"bidir_mode": -1}.get(k, 1))
    return out, names


def device(e, dtype):
    return torch.from_numpy(e).cuda().to(TORCH[dtype]).contiguous()


def grad_ok(case, got, g, mag):
    """util.grad_close's bar, widened by the rounding of a 16-bit gradient"""
    return util.close(got, g, rtol=util.RTOL + ROUND[case.dtype], atol=util.ATOL + 4.0 * util.ulp32(mag))


def check_loss(case, losses, grads, ref):
    """losses [B], grads [B, T, C] (float64 views) against ref(b) -> (loss, grad [T_b, C])"""
    for b in range(case.B):
        Tb = case.T_b[b]
        loss, g = ref(b)
        assert util.close(losses[b], loss), (b, losses[b], loss)
        mag = abs(loss) if np.isfinite(loss) else 0.0
        assert grad_ok(case, grads[b, :Tb], g, mag), b
        assert np.all(grads[b, Tb:] == 0), b


# ---- CTC: bidir_plan ----------------------------------------------------------------------------------------------


def ctc_case(ctx, case):
    e = ic.emissions(case)
    ed = device(e, case.dtype)
    cat, tl = capi._cat_targets(case.targets)
    il = np.asarray(case.T_b, np.int32)
    losses = np.zeros(case.B, np.float32)
    grad = torch.full_like(ed, float("nan"))

    def call():
        torch.cuda.synchronize()
        ctx._check(capi.lib().gtnb_ctc_loss_ex(
            ctx.h, case.B, case.T, case.C, ed.data_ptr(), case.dtype, il.ctypes.data_as(capi._i32p),
            cat.ctypes.data_as(capi._i32p), tl.ctypes.data_as(capi._i32p), 0, losses.ctypes.data_as(capi._f32p),
            grad.data_ptr()))
        torch.cuda.synchronize()

    _, names = run(ctx, case, call)
    return e, losses, grad.float().cpu().numpy().astype(np.float64), names


def check_ctc(case, e, losses, grads):
    check_loss(case, losses, grads, lambda b: f64.ctc_f64(e[b, :case.T_b[b]], case.targets[b]))


@pytest.mark.parametrize("case", of("bidir"), ids=case_id)
def test_ctc_bidir(ictx, case):
    e, losses, grads, names = ctc_case(ictx, case)
    # bidir_shape_supported: at most 224 nodes (every case's C is a multiple of 4, at most 128); a 16-bit batch it
    # refuses is widened to float32 first, and then takes the float32 kernels when the node count allows
    bidir = max(2 * len(t) + 1 for t in case.targets) <= 224
    native = bidir and (case.dtype == ic.F32 or case.C % 8 == 0)
    assert ("bidir_ctc" in names) == bidir, names
    assert ("widen" in names) == (not native and case.dtype != ic.F32), names
    if bidir:  # no status-word retry on the materialised route
        assert not names & MATERIALISED, names
    check_ctc(case, e, losses, grads)


# ---- dense Viterbi: dense_lanes -----------------------------------------------------------------------------------


def dense_f64(e, tw, C, bigram):
    """float64 Viterbi over the dense trellis -> (score, path, smallest margin of a decision on the path); ties go to
    the smallest predecessor and the smallest final state, as the reference's shortestPath breaks them"""
    T = e.shape[0]
    if T == 0:  # linearGraph(0, C) is one start node that does not accept: no path
        return -np.inf, [], np.inf
    W = (tw if bigram else tw[C:]).astype(np.float64).reshape(C, C)  # W[i, j] = w(j -> i)
    e = e.astype(np.float64)
    bp = np.zeros((T, C), np.int64)
    marg = np.full((T, C), np.inf)

    def step(prev, t):
        cand = prev[None, :] + (e[t][:, None] + W)  # [i, j]
        j = np.argmax(cand, axis=1)
        best = cand[np.arange(C), j]
        srt = np.sort(cand, axis=1)
        m = best - srt[:, -2] if C > 1 else np.full(C, np.inf)
        return best, j, np.where(np.isfinite(best), m, np.inf)

    if bigram:
        sc, bp[0], marg[0] = step(np.zeros(C), 0)
    else:
        sc = tw[:C].astype(np.float64) + e[0]
    for t in range(1, T):
        sc, bp[t], marg[t] = step(sc, t)
    k = int(np.argmax(sc))
    if not np.isfinite(sc[k]):
        return sc[k], [-1] * T, np.inf
    srt = np.sort(sc)
    margin = sc[k] - srt[-2] if C > 1 else np.inf
    path = [k]
    for t in range(T - 1, 0, -1):
        margin = min(margin, marg[t][path[-1]])
        path.append(int(bp[t][path[-1]]))
    if bigram:
        margin = min(margin, marg[0][path[-1]])
    return float(sc[k]), path[::-1], margin


@pytest.mark.parametrize("case", of("dense"), ids=case_id)
def test_dense_viterbi(ictx, case):
    e = ic.emissions(case)
    tw = ic.transitions(case)
    ed = device(e, case.dtype)
    wd = torch.from_numpy(tw).cuda()
    il = np.asarray(case.T_b, np.int32)
    paths = torch.full((case.B, case.T), -7, dtype=torch.int32, device="cuda")
    scores = torch.full((case.B,), 7.0, device="cuda")
    kind = capi.DENSE_BIGRAM if case.kind == "bigram" else capi.DENSE_ASG

    def call():
        torch.cuda.synchronize()
        rc = capi.lib().gtnb_viterbi_dense_typed(ictx.h, case.B, case.T, case.C, ed.data_ptr(), case.dtype,
                                                 il.ctypes.data_as(capi._i32p), kind, wd.data_ptr(), paths.data_ptr(),
                                                 scores.data_ptr())
        torch.cuda.synchronize()
        return rc

    rc, names = run(ictx, case, call)
    if case.C > 224:  # the transition tile does not fit shared memory
        assert rc == capi.ERR_UNSUPPORTED and not names, (rc, names)
        return
    assert rc == capi.OK, rc
    assert names == {"viterbi_dense_bigram" if case.kind == "bigram" else "viterbi_dense"}, names
    paths, scores = paths.cpu().numpy(), scores.cpu().numpy()
    compared = 0
    for b in range(case.B):
        Tb = case.T_b[b]
        score, path, margin = dense_f64(e[b, :Tb], tw, case.C, case.kind == "bigram")
        assert np.all(paths[b, Tb:] == -1), b
        if case.ties or margin > MARGIN or not np.isfinite(score):
            assert scores[b] == np.float32(score) if case.ties else util.close(scores[b], score), (b, scores[b], score)
            assert list(paths[b, :Tb]) == path, b
            compared += 1
        else:
            assert util.close(scores[b], score), (b, scores[b], score)
    assert compared > 0, "every utterance was excluded as near-tied"


# ---- n-gram CTC and ASG: ngram_den_shape --------------------------------------------------------------------------


def asg_ref(e, tw, target):
    if len(target) == 0:  # no labels: nothing is accepted; a target longer than T_b has the same (empty) numerator
        target = [0] * (e.shape[0] + 1)
    return f64.asg_f64(e, tw, target)


@pytest.mark.parametrize("case", of("ngram"), ids=case_id)
def test_trellis_loss(ictx, case):
    e = ic.emissions(case)
    tw = ic.transitions(case)
    ed = device(e, case.dtype)
    wd = torch.from_numpy(tw).cuda()
    cat, tl = capi._cat_targets(case.targets)
    il = np.asarray(case.T_b, np.int32)
    losses = np.zeros(case.B, np.float32)
    grad = torch.full_like(ed, float("nan"))  # the emission gradient has the emissions' dtype
    tg = torch.full((tw.size,), float("nan"), device="cuda")
    args = [cat.ctypes.data_as(capi._i32p), tl.ctypes.data_as(capi._i32p)]

    def call():
        torch.cuda.synchronize()
        if case.kind == "bigram":
            ictx._check(capi.lib().gtnb_ngram_ctc_loss_typed(
                ictx.h, case.B, case.T, case.C, ed.data_ptr(), case.dtype, il.ctypes.data_as(capi._i32p),
                wd.data_ptr(), *args, 0, losses.ctypes.data_as(capi._f32p), grad.data_ptr(), tg.data_ptr()))
        else:
            ictx._check(capi.lib().gtnb_asg_loss_typed(
                ictx.h, case.B, case.T, case.C, ed.data_ptr(), case.dtype, il.ctypes.data_as(capi._i32p),
                wd.data_ptr(), *args, losses.ctypes.data_as(capi._f32p), grad.data_ptr(), tg.data_ptr()))
        torch.cuda.synchronize()

    _, names = run(ictx, case, call)
    den = "ngram_den_forward" if case.kind == "bigram" else "asg_den_forward"
    assert den in names and "widen" not in names and not names & MATERIALISED, names
    grads = grad.float().cpu().numpy().astype(np.float64)
    refs = []
    for b in range(case.B):
        eb = e[b, :case.T_b[b]]
        refs.append(ngram_ctc_f64(eb, tw, case.targets[b]) if case.kind == "bigram"
                    else asg_ref(eb, tw, case.targets[b]))
    for b in range(case.B):
        loss, g, _ = refs[b]
        assert util.close(losses[b], loss), (b, losses[b], loss)
        mag = abs(loss) if np.isfinite(loss) else 0.0
        assert grad_ok(case, grads[b, :case.T_b[b]], g, mag), b
        assert np.all(grads[b, case.T_b[b]:] == 0), b
    tref = sum(r[2] for r in refs)
    mag = max(abs(r[0]) for r in refs if np.isfinite(r[0]))
    assert util.grad_close(tg.cpu().numpy(), tref, mag)


# ---- staged sweeps: plan / fused_layout ---------------------------------------------------------------------------


def graph_view(g):
    N, src, dst, lab, w = g
    flags = np.zeros(N, np.uint8)
    flags[0] |= 1
    flags[N - 1] |= 2
    in_arcs = np.argsort(dst, kind="stable").astype(np.int32)
    out_arcs = np.argsort(src, kind="stable").astype(np.int32)
    in_ptr = np.concatenate(([0], np.cumsum(np.bincount(dst, minlength=N)))).astype(np.int32)
    out_ptr = np.concatenate(([0], np.cumsum(np.bincount(src, minlength=N)))).astype(np.int32)
    return capi.make_view(flags, src, dst, lab, lab, w, in_ptr, in_arcs, out_ptr, out_arcs,
                          np.array([0], np.int32), np.array([N - 1], np.int32))


def staged_lattice(ictx, case):
    e = ic.emissions(case)
    e_dev = ictx.to_device(e)
    views = [graph_view(g) for g in case.graphs]
    out = {}

    def call():
        lat = ictx.compose_linear(views, case.T_b, case.C, e_dev, case.T * case.C)
        _, na = lat.sizes()
        out["log"] = lat.forward()
        lat.backward()
        out["grad"] = [lat.arc_grads(b, int(na[b])) for b in range(case.B)]
        out["trop"] = lat.forward(tropical=True)
        lat.backward(tropical=True)
        out["tgrad"] = [lat.arc_grads(b, int(na[b])) for b in range(case.B)]
        out["path"] = lat.viterbi_path(case.T + 1)
        out["lat"] = [lat.download(b) for b in range(case.B)]
        lat.free()

    _, names = run(ictx, case, call)
    return out, names


@pytest.mark.parametrize("case", of("staged"), ids=case_id)
def test_staged(ictx, case):
    if case.graphs is None:  # the materialised CTC criterion
        e, losses, grads, names = ctc_case(ictx, case)
        # (test_plan_coverage holds case.expect to the plan); the generic kernels log as sd_*_generic
        staged = bool(case.expect["staged"])
        assert ("sd_forward" in names) == staged and ("sd_forward_generic" in names) != staged, names
        assert ("sd_backward_fused" in names) == bool(case.expect["fused"]), names
        if not case.expect["fused"]:
            assert ("sd_backward" in names) == staged and ("sd_backward_generic" in names) != staged, names
        assert "bidir_ctc" not in names and "implicit_forward" not in names, names
        check_ctc(case, e, losses, grads)
        return
    out, names = staged_lattice(ictx, case)
    assert {"sd_forward", "sd_backward"} <= names and not names & {"sd_forward_generic", "sd_backward_generic"}, names
    compared = 0
    for b in range(case.B):
        lat = out["lat"][b]
        s, g, _, _ = f64.lattice_f64(lat["flags"], lat["src"], lat["dst"], lat["w"])
        assert util.close(out["log"][b], s), (b, out["log"][b], s)
        assert util.grad_close(out["grad"][b], g, abs(s) if np.isfinite(s) else 0.0), b
        st, _, path, margin = f64.lattice_f64(lat["flags"], lat["src"], lat["dst"], lat["w"], tropical=True)
        assert util.close(out["trop"][b], st), (b, out["trop"][b], st)
        n = int(out["path"]["lens"][b])
        if path is None:  # no accepting path: length -1
            assert n == -1, b
        elif margin > MARGIN:
            assert list(out["path"]["arcs"][b, :n]) == path, b
            # the tropical gradient: 1 on the arcs of the best path, 0 elsewhere
            assert np.array_equal(out["tgrad"][b], np.isin(np.arange(len(lat["src"])), path).astype(np.float32)), b
            compared += 1
    assert compared > 0, "every utterance was excluded as near-tied"


# ---- graph criteria on the implicit sweeps: wide_lanes ------------------------------------------------------------


def compose_f64(g, e, tropical=False):
    """intersect(A, E) of a graph and linearGraph(T_b, C) composed here in float64, frame by frame: node (t, n), arc
    (t, a) from (t, src a) to (t + 1, dst a) of weight w_a + e[t, label a].  Returns (forwardScore or viterbiScore,
    d score / d e [T_b, C], d score / d w [A], best path as arc ids per frame or None, smallest margin on that path)."""
    N, src, dst, lab, w = g
    T, C = e.shape
    e = e.astype(np.float64)
    w = w.astype(np.float64)
    A = len(src)
    ok = (lab >= 0) & (lab < C)
    NEG = -np.inf

    def arcs(t):
        return np.where(ok, w + e[t, np.clip(lab, 0, C - 1)], NEG)

    alpha = np.full((T + 1, N), NEG)
    alpha[0, 0] = 0.0
    choice = np.full((T + 1, N), -1)
    marg = np.full((T + 1, N), np.inf)
    for t in range(T):
        v = alpha[t][src] + arcs(t)
        if tropical:
            for n in range(N):
                ins = np.nonzero(dst == n)[0]
                if len(ins) == 0:
                    continue
                k = ins[int(np.argmax(v[ins]))]
                alpha[t + 1, n] = v[k]
                rest = np.sort(v[ins])
                marg[t + 1, n] = rest[-1] - rest[-2] if len(ins) > 1 and np.isfinite(rest[-1]) else np.inf
                choice[t + 1, n] = k
        else:
            m = np.full(N, NEG)
            np.maximum.at(m, dst, v)
            mm = np.where(np.isfinite(m), m, 0.0)
            acc = np.zeros(N)
            np.add.at(acc, dst, np.exp(v - mm[dst]))
            with np.errstate(divide="ignore"):
                alpha[t + 1] = np.log(acc) + mm
    Z = alpha[T, N - 1]
    ge, gw = np.zeros((T, C)), np.zeros(A)
    if not np.isfinite(Z):
        return Z, ge, gw, None, np.inf
    if tropical:
        path, n, margin = [], N - 1, np.inf
        for t in range(T, 0, -1):
            margin = min(margin, marg[t, n])
            k = choice[t, n]
            path.append(int(k))
            ge[t - 1, lab[k]] += 1.0
            gw[k] += 1.0
            n = src[k]
        return Z, ge, gw, path[::-1], margin
    beta = np.full((T + 1, N), NEG)
    beta[T, N - 1] = 0.0
    for t in range(T - 1, -1, -1):
        v = arcs(t) + beta[t + 1][dst]
        m = np.full(N, NEG)
        np.maximum.at(m, src, v)
        mm = np.where(np.isfinite(m), m, 0.0)
        acc = np.zeros(N)
        np.add.at(acc, src, np.exp(v - mm[src]))
        with np.errstate(divide="ignore"):
            beta[t] = np.log(acc) + mm
        with np.errstate(invalid="ignore"):
            p = np.nan_to_num(np.exp(alpha[t][src] + arcs(t) + beta[t + 1][dst] - Z), nan=0.0)
        np.add.at(ge[t], lab[ok], p[ok])
        gw += p
    return Z, ge, gw, None, np.inf


def graph_loss_f64(g, e):
    """gtnb_graph_loss's loss = forwardScore(E) - forwardScore(intersect(A, E)), d / d e and d / d w"""
    e64 = e.astype(np.float64)
    norm = f64._lse(e64, axis=1)
    Z, ge, gw, _, _ = compose_f64(g, e)
    soft = np.exp(e64 - norm[:, None])
    if not np.isfinite(Z):  # no accepting path: +inf, the denominator's gradient alone
        return np.inf, soft, np.zeros(len(g[1]))
    return float(norm.sum() - Z), soft - ge, -gw


@pytest.mark.parametrize("case", of("implicit"), ids=case_id)
def test_graph_implicit(ictx, case):
    e = ic.emissions(case)
    views = [graph_view(g) for g in case.graphs]
    arr = (capi.GraphView * case.B)(*[v for v, _ in views])
    il = np.asarray(case.T_b, np.int32)
    arc = ic.plan_inputs(case)["arc"]
    n_arcs = sum(len(g[1]) for g in case.graphs)
    if case.kind == "viterbi":
        paths = np.full((case.B, case.T), -7, np.int32)
        arcs = np.full((case.B, case.T), -7, np.int32)
        scores = np.full(case.B, np.nan, np.float32)

        def call():
            ictx._check(capi.lib().gtnb_graph_viterbi(
                ictx.h, case.B, case.T, case.C, e.ctypes.data, 0, il.ctypes.data_as(capi._i32p), arr, None, 0,
                paths.ctypes.data, arcs.ctypes.data, scores.ctypes.data, 0))

        _, names = run(ictx, case, call)
        fwd = "implicit_forward_arc_max" if arc else "implicit_forward_max"
        assert fwd in names and "implicit_trace" in names and not names & MATERIALISED, names
        compared = 0
        for b in range(case.B):
            s, _, _, path, margin = compose_f64(case.graphs[b], e[b, :case.T_b[b]], tropical=True)
            assert util.close(scores[b], s), (b, scores[b], s)
            if path is None:
                assert np.all(arcs[b] == -1), b
            elif margin > MARGIN:
                assert list(arcs[b, :case.T_b[b]]) == path, b
                compared += 1
        assert compared > 0, "every utterance was excluded as near-tied"
        return
    losses = np.zeros(case.B, np.float32)
    grads = np.full(e.shape, np.nan, np.float32)
    ag = np.full(n_arcs, np.nan, np.float32) if case.kind == "loss-gg" else None

    def call():
        ictx._check(capi.lib().gtnb_graph_loss(
            ictx.h, case.B, case.T, case.C, e.ctypes.data, 0, il.ctypes.data_as(capi._i32p), arr, None, 0,
            losses.ctypes.data_as(capi._f32p), grads.ctypes.data, 0, None if ag is None else ag.ctypes.data, 0))

    _, names = run(ictx, case, call)
    fwd, bwd = ("implicit_forward_arc", "implicit_backward_arc") if arc else ("implicit_forward", "implicit_backward")
    assert fwd in names and bwd in names and not names & MATERIALISED, names
    off = 0
    for b in range(case.B):
        g = case.graphs[b]
        loss, ge, gw = graph_loss_f64(g, e[b, :case.T_b[b]])
        mag = abs(loss) if np.isfinite(loss) else 0.0
        assert util.close(losses[b], loss), (b, losses[b], loss)
        assert util.grad_close(grads[b, :case.T_b[b]], ge, mag), b
        assert np.all(grads[b, case.T_b[b]:] == 0), b
        if ag is not None:
            # an arc's gradient sums its T_b per-frame posteriors (all of one sign), each held to grad_close's bar:
            # the relative part adds up to the same relative bar, the absolute part to T_b times it
            atol = case.T_b[b] * (util.ATOL + 4.0 * util.ulp32(mag))
            assert util.close(ag[off:off + len(g[1])], gw, rtol=util.RTOL, atol=atol), b
        off += len(g[1])

