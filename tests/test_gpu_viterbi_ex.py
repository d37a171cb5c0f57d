"""gtnb_viterbi_dense_ex (batched Viterbi decoding with the learned transitions of ASG and n-gram CTC) on the GPU,
and the torch decoders asg_viterbi / ngram_ctc_viterbi / collapse.  Paths and scores are compared with == against
the live reference (oracle/_ref: every utterance alone on its first T_b rows), for both graph kinds:
  ASG:    viterbiPath / viterbiScore of compose(E_b, transitions)  (test/criterion_test.cpp:328-344)
  BIGRAM: viterbiPath / viterbiScore of intersect(E_b, G), G n-gram CTC's bigram graph (benchmarks/ctc.cpp:107-134)
"""
import numpy as np
import pytest

from tests import viterbi_oracle as vo

pytestmark = pytest.mark.gpu

KINDS = ("asg", "bigram")


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


def _kind(kind):
    from gtn_b200 import capi
    return capi.DENSE_BIGRAM if kind == "bigram" else capi.DENSE_ASG


def inputs(B, T, C, kind, seed, ties=False, forbid=False):
    """emissions [B, T, C] and transitions ([C + C*C] for ASG, [C*C] for BIGRAM): U(-5, 5) and U(-3, 3), or
    integers in {-2..2} and {-1, 0, 1} (ties); forbid: about a third of the transitions -inf"""
    rng = np.random.default_rng(seed)
    n = C * C if kind == "bigram" else C + C * C
    if ties:
        e = rng.integers(-2, 3, (B, T, C)).astype(np.float32)
        tw = rng.integers(-1, 2, n).astype(np.float32)
    else:
        e = rng.uniform(-5, 5, (B, T, C)).astype(np.float32)
        tw = rng.uniform(-3, 3, n).astype(np.float32)
    if forbid:
        tw[rng.random(n) < 0.35] = -np.inf
    return e, tw


def padded(e, lens):
    """the emissions with NaN in every padding row: the call must never read them"""
    p = e.copy()
    for b, Tb in enumerate(lens):
        p[b, Tb:] = np.nan
    return p


def reference(ref, kind, e, tw, lens):
    """the live reference, every utterance on its first T_b rows -> (paths [B, T], -1 beyond; scores [B])"""
    B, T, _ = e.shape
    if kind == "bigram":
        return vo.batch(vo.ref_viterbi_bigram, e, tw, lens)
    paths = np.full((B, T), -1, np.int32)
    scores = np.zeros(B, np.float32)
    for b in range(B):
        p, s, _ = ref.ref_viterbi_dense_batch(e[b:b + 1, :lens[b]], tw)
        paths[b, :lens[b]] = p[0]
        scores[b] = s[0]
    return paths, scores


def call(ctx, kind, e, tw, lens, emissions_dev, trans_dev, outputs_dev):
    """gtnb_viterbi_dense_ex with each buffer on the host or the device; outputs prefilled with junk"""
    from gtn_b200 import capi
    B, T, Cn = e.shape
    il = None if lens is None else np.ascontiguousarray(lens, np.int32)
    paths = np.full((B, T), -7, np.int32)
    scores = np.full(B, np.nan, np.float32)
    bufs = []

    def where(a, on_dev):
        if not on_dev:
            return a.ctypes.data
        d = ctx.to_device(a)
        bufs.append(d)
        return d.ptr

    try:
        ep, wp = where(e, emissions_dev), where(tw, trans_dev)
        pp, sp = where(paths, outputs_dev), where(scores, outputs_dev)
        ctx._check(capi.lib().gtnb_viterbi_dense_ex(
            ctx.h, B, T, Cn, ep, int(emissions_dev), None if il is None else il.ctypes.data_as(capi._i32p),
            _kind(kind), wp, int(trans_dev), pp, sp, int(outputs_dev)))
        if outputs_dev:
            paths = bufs[-2].download((B, T), np.int32)
            scores = bufs[-1].download((B,))
    finally:
        for d in bufs:
            d.free()
    return paths, scores


def viterbi_np(e, tw, kind):
    """float32 restatement of the kernel's recursion for a batch of equal lengths (the same adds in the same
    association, first maximum wins) -> (paths [B, T], scores [B])"""
    B, T, Cn = e.shape
    W = tw[-Cn * Cn:].reshape(Cn, Cn)  # W[i, j] = w(j -> i)
    zero = np.float32(0)
    if kind == "bigram":
        s = (zero + (e[:, 0, :, None] + W[None])).max(axis=2)
    else:
        s = zero + (e[:, 0] + tw[:Cn][None])
    bp = np.zeros((B, T, Cn), np.int32)
    for t in range(1, T):
        cand = s[:, None, :] + (e[:, t, :, None] + W[None])  # [b, i, j]
        bp[:, t] = cand.argmax(axis=2)
        s = np.take_along_axis(cand, bp[:, t][:, :, None], axis=2)[:, :, 0]
    paths = np.full((B, T), -1, np.int32)
    best = s.argmax(axis=1)
    scores = s[np.arange(B), best]
    for b in range(B):
        if scores[b] == -np.inf:
            continue
        st = best[b]
        for t in range(T - 1, -1, -1):
            paths[b, t] = st
            st = bp[b, t, st]
    return paths, scores


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("C", [4, 28, 29, 64, 128, 224])
def test_parity_with_reference_every_buffer_placement(ctx, ref, kind, C):
    """ragged lengths with T_b in {0, 1} and NaN padding rows; emissions, transitions and outputs each on the host
    and on the device"""
    B, T = 6, 11
    lens = np.array([T, 1, 0, 7, T - 1, 4], np.int32)
    for ties, forbid in ((False, False), (True, False), (True, True)):
        e, tw = inputs(B, T, C, kind, seed=C + 10 * ties + 20 * forbid, ties=ties, forbid=forbid)
        want_p, want_s = reference(ref, kind, e, tw, lens)
        assert want_s[2] == -np.inf and (want_p[2] == -1).all()  # T_b = 0: linearGraph(0, C) accepts nothing
        ep = padded(e, lens)
        for emissions_dev, trans_dev, outputs_dev in ((0, 0, 0), (1, 1, 1), (0, 1, 0), (1, 0, 1)):
            got_p, got_s = call(ctx, kind, ep, tw, lens, emissions_dev, trans_dev, outputs_dev)
            where = (kind, C, ties, forbid, emissions_dev, trans_dev, outputs_dev)
            assert np.array_equal(got_p, want_p), where
            assert np.array_equal(got_s, want_s), where


@pytest.mark.parametrize("kind", KINDS)
def test_forbidden_transitions_and_no_accepting_path(ctx, ref, kind):
    """-inf weights: a label that nothing reaches is never decoded after frame 0; with every transition between
    labels -inf an utterance longer than one frame has no accepting path (score -inf, path -1), and neither has any
    utterance of the bigram kind, whose first frame takes a transition too"""
    B, T, Cn = 4, 9, 12
    e, tw = inputs(B, T, Cn, kind, seed=5)
    W = tw[-Cn * Cn:].reshape(Cn, Cn)
    W[3] = -np.inf
    lens = np.array([9, 1, 5, 0], np.int32)
    want = reference(ref, kind, e, tw, lens)
    for dev in (False, True):
        got = call(ctx, kind, padded(e, lens), tw, lens, dev, dev, dev)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert not (got[0][:, 1:] == 3).any()
    tw[-Cn * Cn:] = -np.inf
    want = reference(ref, kind, e, tw, lens)
    got = call(ctx, kind, e, tw, lens, 1, 1, 1)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert (got[0][[0, 2, 3]] == -1).all() and (got[1][[0, 2, 3]] == -np.inf).all()
    assert np.isfinite(got[1][1]) == (kind == "asg")  # one frame: ASG takes a start arc alone


@pytest.mark.parametrize("kind", KINDS)
def test_config4_shape(ctx, ref, kind):
    """configs[3] (B=512 T=2000 C=128), the whole batch on the device: the first 16 utterances equal a run of those
    16 alone, a float32 restatement of the recursion, and, for the first 2 (seconds and ~3 GB each), the live
    reference; one utterance is integer valued so that ties occur on most frames"""
    B, T, Cn, n = 512, 2000, 128, 16
    e, tw = inputs(B, T, Cn, kind, seed=314)
    e[1] = np.round(e[1])
    full = call(ctx, kind, e, tw, None, 1, 1, 1)
    part = call(ctx, kind, e[:n], tw, None, 1, 1, 1)
    assert np.array_equal(full[0][:n], part[0]) and np.array_equal(full[1][:n], part[1])
    want = viterbi_np(e[:n], tw, kind)
    assert np.array_equal(part[0], want[0]) and np.array_equal(part[1], want[1])
    rp, rs = reference(ref, kind, e[:2], tw, np.full(2, T, np.int32))
    assert np.array_equal(part[0][:2], rp) and np.array_equal(part[1][:2], rs)


def test_asg_kind_matches_gtnb_viterbi_dense(ctx):
    """host buffers, C % 4 == 0: the old entry point and the ASG kind agree everywhere but at T_b = 0 (0 vs -inf)"""
    for Cn, ties in ((8, True), (64, False), (128, True)):
        B, T = 5, 30
        e, tw = inputs(B, T, Cn, "asg", seed=Cn, ties=ties)
        lens = np.array([30, 0, 1, 17, 29], np.int32)
        old_p, old_s = ctx.viterbi_dense(e, tw, input_lens=lens)
        new_p, new_s = ctx.viterbi_dense_ex(e, tw, input_lens=lens)
        live = lens > 0
        assert np.array_equal(old_p[live], new_p[live]) and np.array_equal(old_s[live], new_s[live])
        assert old_s[1] == 0.0 and new_s[1] == -np.inf and (new_p[1] == -1).all()
        old_p, old_s = ctx.viterbi_dense(e, tw)
        new_p, new_s = ctx.viterbi_dense_ex_dev(e, tw)
        assert np.array_equal(old_p, new_p) and np.array_equal(old_s, new_s)


def test_bad_arguments(ctx):
    from gtn_b200 import capi
    L = capi.lib()
    e = np.zeros((2, 4, 5), np.float32)
    tw = np.zeros(30, np.float32)
    p = np.zeros((2, 4), np.int32)
    s = np.zeros(2, np.float32)

    def run(kind=0, lens=None, emissions=e.ctypes.data, trans=tw.ctypes.data, Cn=5, T=4):
        il = None if lens is None else np.asarray(lens, np.int32)
        return L.gtnb_viterbi_dense_ex(ctx.h, 2, T, Cn, emissions, 0, None if il is None else il.ctypes.data_as(capi._i32p),
                                       kind, trans, 0, p.ctypes.data, s.ctypes.data, 0)

    assert run() == capi.OK
    for kw in ({"kind": 2}, {"kind": -1}, {"lens": [4, 5]}, {"lens": [-1, 2]}, {"emissions": None}, {"trans": None},
               {"Cn": 0}, {"T": -1}):
        assert run(**kw) == capi.ERR_INVALID_ARGUMENT, kw
    big = np.zeros(225 * 225, np.float32)
    eb = np.zeros((2, 4, 225), np.float32)
    assert L.gtnb_viterbi_dense_ex(ctx.h, 2, 4, 225, eb.ctypes.data, 0, None, 1, big.ctypes.data, 0, p.ctypes.data,
                                   s.ctypes.data, 0) == capi.ERR_UNSUPPORTED
    assert L.gtnb_viterbi_dense_ex(ctx.h, 0, 4, 5, e.ctypes.data, 0, None, 0, tw.ctypes.data, 0, None, None,
                                   0) == capi.OK  # B = 0 is a no-op
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.viterbi_dense_ex(e, tw, input_lens=[2, 9])


@pytest.mark.parametrize("kind", KINDS)
def test_torch_decoders_match_capi(kind):
    torch = pytest.importorskip("torch")
    from gtn_b200 import torch_loss
    B, T, Cn = 5, 40, 29
    e, tw = inputs(B, T, Cn, kind, seed=77, ties=True)
    lens = np.array([40, 0, 1, 33, 12], np.int32)
    fn = torch_loss.ngram_ctc_viterbi if kind == "bigram" else torch_loss.asg_viterbi
    from gtn_b200 import capi
    ctx = capi.Ctx(0)
    want_p, want_s = ctx.viterbi_dense_ex(padded(e, lens), tw, _kind(kind), input_lens=lens)
    ctx.close()
    x = torch.tensor(padded(e, lens), device="cuda", requires_grad=True)
    shapes = [(tw.size,)] + ([(Cn, Cn)] if kind == "bigram" else [])
    for shape in shapes:
        w = torch.tensor(tw.reshape(shape), device="cuda", requires_grad=True)
        for il in (torch.tensor(lens), list(lens), torch.tensor(lens).cuda()):
            paths, scores = fn(x, w, il)
            assert paths.is_cuda and paths.dtype == torch.int32 and paths.shape == (B, T)
            assert scores.is_cuda and scores.shape == (B,) and not scores.requires_grad
            assert np.array_equal(paths.cpu().numpy(), want_p) and np.array_equal(scores.cpu().numpy(), want_s)
    full_p, full_s = fn(torch.tensor(e, device="cuda"), torch.tensor(tw, device="cuda"))
    ctx = capi.Ctx(0)
    wp, ws = ctx.viterbi_dense_ex(e, tw, _kind(kind))
    ctx.close()
    assert np.array_equal(full_p.cpu().numpy(), wp) and np.array_equal(full_s.cpu().numpy(), ws)


def _collapse_loop(paths, blank):
    out = []
    for row in paths:
        labels, prev = [], None
        for v in row:
            if v < 0:
                break
            if v != prev and v != blank:
                labels.append(int(v))
            prev = v
        out.append(labels)
    return out


@pytest.mark.parametrize("blank", [None, 0, 3])
def test_collapse_matches_python_loop(blank):
    torch = pytest.importorskip("torch")
    from gtn_b200 import torch_loss
    rng = np.random.default_rng(9)
    B, T = 12, 25
    p = rng.integers(0, 5, (B, T)).astype(np.int32)
    p[:, 10:14] = p[:, 9:10]  # repeats
    for b, Tb in enumerate([25, 0, 1, 7, 25, 3, 12, 25, 2, 18, 24, 25]):
        p[b, Tb:] = -1
    p[7] = 0  # all blank (blank = 0)
    labels, lengths = torch_loss.collapse(torch.tensor(p, device="cuda"), blank=blank)
    assert labels.is_cuda and labels.dtype == torch.int32 and labels.shape == (B, T) and lengths.is_cuda
    want = _collapse_loop(p, blank)
    labels, lengths = labels.cpu().numpy(), lengths.cpu().numpy()
    for b in range(B):
        assert lengths[b] == len(want[b])
        assert labels[b, :lengths[b]].tolist() == want[b] and (labels[b, lengths[b]:] == -1).all()
    e0 = torch.zeros((2, 0), dtype=torch.int32, device="cuda")
    l0, n0 = torch_loss.collapse(e0, blank=blank)
    assert l0.shape == (2, 0) and n0.tolist() == [0, 0]


@pytest.mark.parametrize("kind", KINDS)
def test_torch_decoders_move_nothing_but_the_lengths(kind, monkeypatch):
    """Only input_lengths visits the host: no Python-side copy of a CUDA tensor, and the call copies nothing from
    the device to the host"""
    torch = pytest.importorskip("torch")
    from gtn_b200 import torch_loss
    B, T, Cn = 4, 20, 8
    e, tw = inputs(B, T, Cn, kind, seed=3)
    fn = torch_loss.ngram_ctc_viterbi if kind == "bigram" else torch_loss.asg_viterbi
    x = torch.tensor(e, device="cuda")
    w = torch.tensor(tw, device="cuda")
    lens = [20, 7, 0, 13]
    fn(x, w, lens)  # the context of this stream exists
    torch.cuda.synchronize()

    def refuse(*a, **k):
        raise AssertionError("a CUDA tensor was moved or read on the host")

    for name in ("cpu", "numpy", "tolist", "item"):
        monkeypatch.setattr(torch.Tensor, name, refuse)
    real_to = torch.Tensor.to

    def to(self, *a, **k):
        assert not self.is_cuda, "a CUDA tensor was moved"
        return real_to(self, *a, **k)

    monkeypatch.setattr(torch.Tensor, "to", to)
    paths, scores = fn(x, w, lens)
    labels, n = torch_loss.collapse(paths, blank=0 if kind == "bigram" else None)
    monkeypatch.undo()
    assert paths.is_cuda and scores.is_cuda and labels.is_cuda and n.is_cuda
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        paths, scores = fn(x, w, lens)
        torch_loss.collapse(paths, blank=0)
        torch.cuda.synchronize()
    d2h = [ev for ev in prof.events() if "DtoH" in ev.name or "Device -> Host" in ev.name]
    assert not d2h, [ev.name for ev in d2h]
