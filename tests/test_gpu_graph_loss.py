"""gtnb_graph_loss (one user-supplied target graph per utterance) on the GPU against the live reference
(tests/graph_oracle.py), utterance by utterance on its own T_b rows, on both routes (implicit sweeps, materialised
lattices), host and device buffers; the routing seen in the profile log; non-finite and bad input; CTC graphs
against gtnb_ctc_loss; and torch_loss.graph_loss."""
import numpy as np
import pytest

from gtn_b200 import capi
from tests import graph_oracle as go
from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(oracle):
    assert oracle.have_ref(), "oracle/_ref/libgtn_ref.so is missing: run `make -C oracle ref` where the reference sources are"
    oracle.libref()
    return oracle


def views_of(graphs):
    return [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]


def batch(C, seed, kinds=("ctc", "wild", "rand")):
    """one graph of each kind, cycled to B = 2 * len(kinds); ragged lengths, NaN in the padding"""
    rng = np.random.default_rng(seed)
    graphs = []
    for k in kinds * 2:
        if k == "ctc":
            g = go.ctc_graph(rng.integers(1, C, int(rng.integers(1, 6))))
        elif k == "wild":
            g = go.with_wildcards(go.ctc_graph(rng.integers(1, C, int(rng.integers(1, 4)))), C, w_loop=-0.2)
        else:
            g = go.random_graph(rng, 10, 40, C, label_hi=C + 2)
        g["w"] = rng.uniform(-1, 1, len(g["src"])).astype(np.float32)
        graphs.append(g)
    B, T = len(graphs), 18
    lens = rng.integers(T // 2, T + 1, B).astype(np.int32)
    lens[0] = T
    e = rng.uniform(-3, 3, (B, T, C)).astype(np.float32)
    for b in range(B):
        e[b, lens[b]:] = np.nan
    return e, graphs, lens


def check(got, want, T):
    (l, g, ag), (lr, gr, agr) = got, want
    assert util.close(l, lr), (l, lr)
    mag = float(np.max(np.abs(lr[np.isfinite(lr)]), initial=1.0)) + 5.0 * T
    assert util.grad_close(g, gr, mag), float(np.nanmax(np.abs(g - gr)))
    assert util.grad_close(ag, agr, mag), float(np.nanmax(np.abs(ag - agr)))


@pytest.mark.parametrize("C", [4, 28, 64, 256, 1024])
@pytest.mark.parametrize("implicit", [1, 0])
def test_parity_both_routes_host_and_device(ref, ctx, C, implicit):
    e, graphs, lens = batch(C, seed=C + implicit)
    want = go.ref_graph_loss(e, graphs, lens)
    ctx.set_flag("implicit", implicit)
    try:
        got = ctx.graph_loss(e, views_of(graphs), input_lens=lens)
        check(got, want, e.shape[1])
        assert not np.isnan(got[1]).any()  # every row written, 0 beyond T_b
        for b in range(len(lens)):
            assert not got[1][b, lens[b]:].any()
        got = ctx.graph_loss_dev(e, views_of(graphs), input_lens=lens)
        check(got, want, e.shape[1])
    finally:
        ctx.set_flag("implicit", 1)


@pytest.mark.parametrize("on_device", [0, 1])
def test_arc_weights_override_the_views(ref, ctx, on_device):
    C = 28
    e, graphs, lens = batch(C, seed=5)
    w = np.random.default_rng(6).uniform(-2, 2, sum(len(g["src"]) for g in graphs)).astype(np.float32)
    want = go.ref_graph_loss(e, graphs, lens, weights=w)
    f = ctx.graph_loss_dev if on_device else ctx.graph_loss
    check(f(e, views_of(graphs), input_lens=lens, arc_weights=w), want, e.shape[1])


def test_routing_arc_kernels_only_when_needed(ctx):
    C = 28
    e, graphs, lens = batch(C, seed=7, kinds=("ctc",))
    ctx.profile(True)
    ctx.graph_loss(e, views_of(graphs), input_lens=lens)
    names = ctx.profile_read()
    assert "implicit_forward" in names and "implicit_forward_arc" not in names, names
    e, graphs, lens = batch(C, seed=7, kinds=("ctc", "wild"))
    ctx.graph_loss(e, views_of(graphs), input_lens=lens)
    names = ctx.profile_read()
    assert "implicit_forward_arc" in names and "implicit_backward_arc" in names, names
    assert "implicit_forward" not in names, names
    ctx.profile(False)


def test_edge_cases(ref, ctx):
    C = 6
    wild = go.with_wildcards(go.ctc_graph([2, 3]), C)
    chain = go.make([1, 0, 0, 2], [0, 1, 2], [1, 2, 3], [1, 2, 3])  # accepts length 3 only
    empty = go.make([], [], [], [])
    graphs = [wild, wild, chain, empty]
    lens = np.asarray([0, 1, 5, 6], np.int32)
    e = np.random.default_rng(8).uniform(-3, 3, (4, 6, C)).astype(np.float32)
    for implicit in (1, 0):
        ctx.set_flag("implicit", implicit)
        l, g, ag = ctx.graph_loss(e, views_of(graphs), input_lens=lens)
        ctx.set_flag("implicit", 1)
        assert np.isnan(l[0]) and not g[0].any()
        assert np.isposinf(l[2]) and np.isposinf(l[3])
        lr, gr, agr = go.ref_graph_loss(e[1:3], graphs[1:3], lens[1:3])
        assert util.close(l[1:3], lr)
        assert util.grad_close(g[1:3], gr, 50.0) and util.grad_close(ag[len(wild["src"]):], agr, 50.0)
        # +inf: the denominator's gradient alone (softmax of each frame)
        p = np.exp(e[3] - e[3].max(1, keepdims=True))
        assert util.grad_close(g[3], p / p.sum(1, keepdims=True), 50.0)
    assert ctx.graph_loss(np.zeros((0, 5, C), np.float32), [])[0].shape == (0,)


@pytest.mark.parametrize("where", ["emission_nan", "emission_inf", "w_inf", "w_nan"])
def test_non_finite_emissions_and_weights_match_the_reference_in_kind(ref, ctx, where):
    C = 9
    e, graphs, lens = batch(C, seed=9, kinds=("wild", "ctc"))
    e = np.nan_to_num(e, nan=0.0)
    if where == "emission_nan":
        e[1, 3, 2] = np.nan
    elif where == "emission_inf":
        e[2, 2, int(graphs[2]["olabel"][1])] = np.inf
    elif where == "w_inf":
        graphs[3]["w"][1] = -np.inf
    else:
        graphs[0]["w"][3] = np.nan
    lr, gr, agr = go.ref_graph_loss(e, graphs, lens)
    for got in (ctx.graph_loss(e, views_of(graphs), input_lens=lens),
                ctx.graph_loss_dev(e, views_of(graphs), input_lens=lens)):
        for a, b_ in zip(got, (lr, gr, agr)):
            assert np.array_equal(np.isnan(a), np.isnan(b_)), where
            assert np.array_equal(np.isposinf(a), np.isposinf(b_)) and np.array_equal(np.isneginf(a), np.isneginf(b_))
        fin = np.isfinite(lr)
        assert util.close(got[0][fin], lr[fin])


def test_bad_input(ctx):
    C = 5
    g = go.ctc_graph([1, 2])
    e = np.zeros((1, 4, C), np.float32)
    eps = go.make([1, 2], [0], [1], [-1])
    with pytest.raises(capi.GtnbError) as ei:
        ctx.graph_loss(e, views_of([eps]))
    assert ei.value.code == capi.ERR_UNSUPPORTED and "remove" in str(ei.value)
    for lens in ([5], [-1]):
        with pytest.raises(capi.GtnbInvalidArgument):
            ctx.graph_loss(e, views_of([g]), input_lens=lens)
    bad = go.make([1, 2], [0], [7], [1])  # arc endpoint outside the graph
    with pytest.raises(capi.GtnbInvalidArgument):
        ctx.graph_loss(e, views_of([bad]))


def test_ctc_graphs_agree_with_ctc_loss_at_benchmark_shape(ctx):
    B, T, C, U = 16, 1000, 64, 100  # BASELINE.json configs[1] shape
    e, targets = util.bench_inputs(B, T, C, U)
    lc, gc = ctx.ctc_loss(e, targets, blank=0)
    l, g, _ = ctx.graph_loss(e, views_of([go.ctc_graph(t) for t in targets]))
    assert util.close(l, lc), np.abs(l - lc).max()
    assert util.grad_close(g, gc, 5.0 * T), float(np.abs(g - gc).max())


def _gtn_graph(gtn, g):
    h = gtn.Graph()
    for f in g["flags"]:
        h.add_node(bool(f & 1), bool(f & 2))
    for a in range(len(g["src"])):
        h.add_arc(int(g["src"][a]), int(g["dst"][a]), int(g["ilabel"][a]), int(g["olabel"][a]), float(g["w"][a]))
    return h


def _torch_case(seed=11):
    torch = pytest.importorskip("torch")
    import gtn_b200.gtn as gtn
    C = 12
    e, graphs, lens = batch(C, seed=seed, kinds=("wild", "ctc"))
    e = np.nan_to_num(e, nan=7.0)
    return torch, gtn, e, graphs, lens


@pytest.mark.parametrize("reduction", ["mean", "none"])
def test_torch_graph_loss_matches_a_reference_loop(ref, reduction):
    torch, gtn, e, graphs, lens = _torch_case()
    from gtn_b200 import torch_loss
    B = len(graphs)
    w0 = np.concatenate([g["w"] for g in graphs])
    x = torch.tensor(e, device="cuda", requires_grad=True)
    w = torch.tensor(w0 + 0.25, device="cuda", requires_grad=True)
    out = torch_loss.graph_loss(x, [_gtn_graph(gtn, g) for g in graphs], input_lengths=torch.tensor(lens),
                                weights=w, reduction=reduction)
    up = torch.linspace(0.5, 2.0, B, device="cuda")  # a non-uniform upstream gradient
    (out * (up if reduction == "none" else 1.0)).sum().backward()
    lr, gr, agr = go.ref_graph_loss(e, graphs, lens, weights=w0 + 0.25)
    scale = up.cpu().numpy() if reduction == "none" else np.full(B, 1.0 / B)
    if reduction == "mean":
        assert util.close(out.item(), lr.mean())
    else:
        assert util.close(out.detach().cpu().numpy(), lr)
    gw = np.concatenate([agr[o:o + len(g["src"])] * scale[b] for b, (g, o) in
                         enumerate(zip(graphs, np.cumsum([0] + [len(g["src"]) for g in graphs])))])
    assert util.grad_close(x.grad.cpu().numpy(), gr * scale[:, None, None], 50.0)
    assert util.grad_close(w.grad.cpu().numpy(), gw, 50.0)


def test_torch_graph_loss_without_weights_uses_the_graphs(ref):
    torch, gtn, e, graphs, lens = _torch_case(seed=12)
    from gtn_b200 import torch_loss
    x = torch.tensor(e, device="cuda", requires_grad=True)
    out = torch_loss.graph_loss(x, [_gtn_graph(gtn, g) for g in graphs], input_lengths=list(lens), reduction="none")
    out.sum().backward()
    lr, gr, _ = go.ref_graph_loss(e, graphs, lens)
    assert util.close(out.detach().cpu().numpy(), lr)
    assert util.grad_close(x.grad.cpu().numpy(), gr, 50.0)


def test_torch_graph_loss_moves_nothing_but_the_losses(monkeypatch):
    """Only the B losses visit the host: no Python-side copy of any CUDA tensor during the forward"""
    torch, gtn, e, graphs, lens = _torch_case(seed=13)
    from gtn_b200 import torch_loss
    gg = [_gtn_graph(gtn, g) for g in graphs]
    x = torch.tensor(e, device="cuda", requires_grad=True)
    w = torch.tensor(np.concatenate([g["w"] for g in graphs]), device="cuda", requires_grad=True)
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
    per = torch_loss.graph_loss(x, gg, input_lengths=list(lens), weights=w, reduction="none")
    monkeypatch.undo()
    assert per.is_cuda and per.shape == (len(gg),)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        per = torch_loss.graph_loss(x, gg, input_lengths=list(lens), weights=w, reduction="none")
        per.sum().backward()
        torch.cuda.synchronize()
    d2h = [ev for ev in prof.events() if "DtoH" in ev.name or "Device -> Host" in ev.name]
    assert len(d2h) <= 3, [ev.name for ev in d2h]  # the read-back: B normaliser and numerator scores, B status words
