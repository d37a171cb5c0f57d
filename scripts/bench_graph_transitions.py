"""gtnb_graph_transitions_loss (user target graphs with learned ASG or bigram transitions) on four workloads, in one
run.  One JSON record on stdout (and in --out when given):

  decomp_asg    word-piece decomposition graphs with ASG transitions, B=128 T=500, C = 127 pieces + 1 = 128: a seeded
                inventory of the 26 letters and random 2- and 3-letter pieces, seeded transcripts of ~60 letters, each
                graph built with gtn_b200.gtn's host ops as word_decompositions.py builds it
  ctc_bigram    CTC graphs with bigram transitions at the n-gram shape (B=128 T=500 C=64 U=50), next to
                gtnb_ngram_ctc_loss on the same inputs (what the generic product costs against the built-in graphs)
  fal_asg       ASG force-align chains with ASG transitions at the same shape, next to gtnb_asg_loss_ex
  wildcard_asg  decomposition graphs at C=64 with a wildcard state at each end, ASG transitions; the record says
                which route the products take (a wildcard node becomes C copies with C in-arcs each)

For each: ms per call on the device route and on the materialised route (set_flag("implicit", 0)), every buffer on
the device, from CUDA events with L2 flushed before each call, the median over --rounds rounds of --steps calls; the
kernels of each route (gtnb_profile_*, CUDA events per launch); a lower bound on the host share of a device-route call
(1 - the sum of its kernel times over its wall-clock time: the time the GPU waits for host packing and launches; the
numerator's sweeps overlap the denominator on a second stream, so the sum counts that overlap twice); the largest
relative difference between the two routes' losses and the largest differences between their emission, arc-weight and
transition gradients, with whether they are within tests/util.py's grad_close bar.

--baseline-lib: another build of libgtn_b200.so (e.g. the parent commit's) whose gtnb_ngram_ctc_loss and
gtnb_asg_loss_ex run next to this build's, alternating, with their outputs compared for equality.  The card and its
power limit are read in the same run.

    python scripts/bench_graph_transitions.py [--steps 10] [--warmup 2] [--rounds 5] [--baseline-lib PATH] [--out F]
"""
import argparse
import ctypes as Ct
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gtn_b200.gtn as gtn  # noqa: E402
from gtn_b200 import capi  # noqa: E402
from tests import graph_oracle as go  # noqa: E402
from tests import graph_trans_oracle as gt  # noqa: E402
from tests import util  # noqa: E402


def gtn_graph(d):
    h = gtn.Graph()
    for f in d["flags"]:
        h.add_node(bool(f & 1), bool(f & 2))
    for a in range(len(d["src"])):
        h.add_arc(int(d["src"][a]), int(d["dst"][a]), int(d["ilabel"][a]), int(d["olabel"][a]), float(d["w"][a]))
    return h


GTN_OPS = dict(graph=gtn_graph, union=gtn.union, closure=gtn.closure, compose=gtn.compose, remove=gtn.remove,
               project_input=gtn.project_input, project_output=gtn.project_output)


def as_dict(g):
    d = gtn.arc_lists(g)
    return go.make(d["flags"], d["src"], d["dst"], d["ilabel"], d["olabel"], d["weights"])


def transitions(C, kind):
    """the workloads' seeded transitions: [C + C*C] for ASG, [C*C] for BIGRAM"""
    n = (C + C * C) if kind == capi.DENSE_ASG else C * C
    return np.random.default_rng(5).uniform(-1, 1, n).astype(np.float32)


def decomp_graphs(rng, B, n_labels):
    """B word-piece decomposition graphs of seeded transcripts of ~60 letters over go.inventory(26, n_labels) ->
    (graphs, C = pieces + 1)"""
    pieces = go.inventory(26, n_labels, seed=7)
    gs = []
    for b in range(B):
        letters = [int(x) for x in rng.integers(0, 26, int(rng.integers(55, 66)))]
        g = as_dict(go.decomposition_graph(GTN_OPS, letters, pieces))
        g["w"] = rng.uniform(-0.5, 0.5, len(g["src"])).astype(np.float32)
        gs.append(g)
    return gs, len(pieces) + 1


def workloads():
    """the four workloads of the module docstring, built in turn -> (name, emissions, graphs, kind, input lengths or
    None, targets or None)"""
    B, T = 128, 500
    rng = np.random.default_rng(11)
    dec, C = decomp_graphs(rng, B, 128)
    e = np.random.default_rng(12).uniform(-5, 5, (B, T, C)).astype(np.float32)
    yield "decomp_asg", e, dec, capi.DENSE_ASG, None, None
    B, T, C, U = 128, 500, 64, 50
    e, targets = util.bench_inputs(B, T, C, U)
    lens = np.full(B, T, np.int32)
    yield "ctc_bigram", e, [go.ctc_graph(t, blank=0) for t in targets], capi.DENSE_BIGRAM, lens, targets
    yield "fal_asg", e, [gt.fal_graph(t) for t in targets], capi.DENSE_ASG, lens, targets
    B, T = 128, 500
    dec, C = decomp_graphs(rng, B, 64)
    e = np.random.default_rng(13).uniform(-5, 5, (B, T, C)).astype(np.float32)
    yield "wildcard_asg", e, [go.with_wildcards(g, C, w_loop=-1.0) for g in dec], capi.DENSE_ASG, None, None


class Lib:
    """a build of libgtn_b200.so and a context of it (path None: this build, on ctx)"""

    def __init__(self, path=None, ctx=None):
        vp = Ct.c_void_p
        if path is None:
            self.L, self.h, self.own = capi.lib(), ctx.h, False
            return
        L = Ct.CDLL(path)
        L.gtnb_ctx_create.argtypes = [Ct.c_int, vp, Ct.POINTER(vp)]
        L.gtnb_ctx_destroy.argtypes = [vp]
        for name in ("gtnb_timer_start", "gtnb_flush_l2"):
            getattr(L, name).argtypes = [vp]
        L.gtnb_timer_stop.argtypes = [vp, Ct.POINTER(Ct.c_float)]
        L.gtnb_last_error.restype = Ct.c_char_p
        L.gtnb_last_error.argtypes = [vp]
        L.gtnb_profile_enable.argtypes = [vp, Ct.c_int]
        L.gtnb_profile_read.restype = Ct.c_char_p
        L.gtnb_profile_read.argtypes = [vp]
        for name, _, argtypes in capi.SYMBOLS:
            if name in ("gtnb_ngram_ctc_loss", "gtnb_asg_loss_ex"):
                getattr(L, name).argtypes = argtypes
        h = vp()
        assert L.gtnb_ctx_create(0, None, Ct.byref(h)) == 0
        self.L, self.h, self.own = L, h.value, True

    def check(self, rc):
        if rc:
            raise RuntimeError(self.L.gtnb_last_error(self.h).decode())

    def timed(self, step):
        self.check(self.L.gtnb_flush_l2(self.h))
        self.check(self.L.gtnb_timer_start(self.h))
        t0 = time.perf_counter()
        self.check(step())
        wall = (time.perf_counter() - t0) * 1e3  # (every call synchronises before it returns its losses)
        ms = Ct.c_float()
        self.check(self.L.gtnb_timer_stop(self.h, Ct.byref(ms)))
        return ms.value, wall

    def kernels_ms(self, step, steps):
        self.check(self.L.gtnb_profile_enable(self.h, 1))
        self.L.gtnb_profile_read(self.h)
        for _ in range(steps):
            self.timed(step)
        out = {}
        for line in self.L.gtnb_profile_read(self.h).decode().splitlines():
            name, n, ms = line.split()
            if name != "flush_l2":
                out[name] = out.get(name, 0.0) + float(ms) / steps
        self.check(self.L.gtnb_profile_enable(self.h, 0))
        return out

    def close(self):
        if self.own:
            self.L.gtnb_ctx_destroy(self.h)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--baseline-lib", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = capi.Ctx(0)
    this = Lib(ctx=ctx)
    base = Lib(args.baseline_lib) if args.baseline_lib else None
    L = capi.lib()

    def rounds(libs_steps):
        """{name: (lib, step)} timed in alternating rounds: median over rounds of the mean event ms, and of the wall ms"""
        for lib, step in libs_steps.values():
            for _ in range(args.warmup):
                lib.check(step())
        ev = {k: [] for k in libs_steps}
        wall = {k: [] for k in libs_steps}
        order = list(libs_steps)
        for i in range(args.rounds):
            for k in (order if i % 2 == 0 else order[::-1]):  # (each build goes first in every other round)
                lib, step = libs_steps[k]
                t = [lib.timed(step) for _ in range(args.steps)]
                ev[k].append(float(np.mean([x[0] for x in t])))
                wall[k].append(float(np.mean([x[1] for x in t])))
        return {k: {"ms_per_call_median": float(np.median(ev[k])), "ms_rounds": ev[k],
                    "wall_ms_per_call_median": float(np.median(wall[k]))} for k in libs_steps}

    def workload(e, graphs, kind, lens=None):
        B, T, C = e.shape
        views = [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
        arr = (capi.GraphView * B)(*[v for v, _ in views])
        n_arcs = sum(len(g["src"]) for g in graphs)
        tw = transitions(C, kind)
        il = None if lens is None else np.ascontiguousarray(lens, np.int32)
        bufs = dict(e=ctx.to_device(e), g=ctx.alloc(e.nbytes), ag=ctx.alloc(4 * max(n_arcs, 4)), tw=ctx.to_device(tw),
                    tg=ctx.alloc(tw.nbytes))
        losses = np.zeros(B, np.float32)

        def step():
            return L.gtnb_graph_transitions_loss(
                ctx.h, B, T, C, bufs["e"].ptr, 1, None if il is None else il.ctypes.data_as(capi._i32p), arr, None, 1,
                kind, bufs["tw"].ptr, 1, losses.ctypes.data_as(capi._f32p), bufs["g"].ptr, 1, bufs["ag"].ptr, 1,
                bufs["tg"].ptr, 1)

        rec = {"shape": {"B": B, "T": T, "C": C}, "kind": "asg" if kind == capi.DENSE_ASG else "bigram",
               "graphs": {"nodes_mean": float(np.mean([len(g["flags"]) for g in graphs])),
                          "arcs_mean": float(np.mean([len(g["src"]) for g in graphs]))}}
        def outputs():
            return (losses.copy(), bufs["g"].download(e.shape), bufs["ag"].download((max(n_arcs, 1),))[:n_arcs],
                    bufs["tg"].download(tw.shape))

        r = rounds({"device": (this, step)})["device"]
        kern = this.kernels_ms(step, args.steps)
        dev = outputs()
        # the route taken: the materialised one launches the lattice kernels, the device route the dense trellis
        route = "device" if any(k.startswith(("asg_den", "ngram_den")) for k in kern) else "materialised"
        # (a lower bound: the numerator's sweeps run beside the denominator on a second stream, and the sum counts
        # their overlap twice)
        r.update(kernels_ms_per_call=kern, route_taken=route,
                 host_share_lower_bound=max(0.0, 1.0 - sum(kern.values()) / r["wall_ms_per_call_median"]))
        rec["device_route"] = r
        ctx.set_flag("implicit", 0)
        r = rounds({"exact": (this, step)})["exact"]
        r["kernels_ms_per_call"] = this.kernels_ms(step, args.steps)
        ctx.set_flag("implicit", 1)
        rec["exact_route"] = r
        ex = outputs()
        fin = np.isfinite(dev[0])
        rec["max_rel_loss_diff_between_routes"] = float(np.max(np.abs(ex[0] - dev[0])[fin] / np.abs(ex[0][fin]),
                                                               initial=0.0))
        # the gradients of the two routes.  An emission gradient is one posterior, held to tests/util.py's grad_close
        # (1e-4 relative + 1e-5 + 4 ulp of the largest score).  Both routes take every posterior as exp of a sum of fp32
        # scores of that magnitude, so each term carries a relative error of a few ulp(score); an arc-weight or
        # transition gradient sums many posteriors (frames, copies, utterances) and keeps that relative error, so it
        # is held to 1e-4 + 4 ulp(score) relative (DESIGN.md "Tolerances")
        mag = float(np.max(np.abs(dev[0][fin]), initial=1.0))
        e4 = 4.0 * util.ulp32(mag)
        for key, i in (("grads", 1), ("arc_grads", 2), ("trans_grad", 3)):
            d = np.abs(dev[i].astype(np.float64) - ex[i])
            rec["max_abs_%s_diff_between_routes" % key] = float(np.max(d, initial=0.0))
            rec["max_rel_%s_diff_between_routes" % key] = float(np.max(
                d / np.maximum(np.maximum(np.abs(dev[i]), np.abs(ex[i])), 1e-30), initial=0.0))
            rec["%s_within_bar" % key] = (util.grad_close(dev[i], ex[i], mag) if i == 1 else
                                          util.close(dev[i], ex[i], rtol=util.RTOL + e4, atol=util.ATOL + e4))
        rec["bar_4ulp_of_largest_loss"] = e4
        rec["device_speedup_vs_exact"] = rec["exact_route"]["ms_per_call_median"] / rec["device_route"]["ms_per_call_median"]
        dev_losses = dev[0]
        return rec, bufs, tw, dev_losses

    def target_criterion(name, bufs, tw, targets, lens, graph_losses, rec):
        """gtnb_ngram_ctc_loss / gtnb_asg_loss_ex on the same inputs; with --baseline-lib, the same call of another
        build alternating with this one, outputs compared for equality"""
        B, T, C = rec["shape"]["B"], rec["shape"]["T"], rec["shape"]["C"]
        cat = np.ascontiguousarray(np.concatenate(targets), np.int32)
        tl = np.asarray([len(t) for t in targets], np.int32)
        il = np.ascontiguousarray(lens, np.int32)
        outs = {}

        def make(lib, key):
            losses = np.zeros(B, np.float32)
            g, tg = ctx.alloc(4 * B * T * C), ctx.alloc(tw.nbytes)
            outs[key] = (losses, g, tg)
            fn = getattr(lib.L, name)
            if name == "gtnb_ngram_ctc_loss":
                return lambda: fn(lib.h, B, T, C, bufs["e"].ptr, 1, il.ctypes.data_as(capi._i32p), bufs["tw"].ptr, 1,
                                  cat.ctypes.data_as(capi._i32p), tl.ctypes.data_as(capi._i32p), 0,
                                  losses.ctypes.data_as(capi._f32p), g.ptr, 1, tg.ptr, 1)
            return lambda: fn(lib.h, B, T, C, bufs["e"].ptr, 1, il.ctypes.data_as(capi._i32p), bufs["tw"].ptr, 1,
                              cat.ctypes.data_as(capi._i32p), tl.ctypes.data_as(capi._i32p),
                              losses.ctypes.data_as(capi._f32p), g.ptr, 1, tg.ptr, 1)

        steps = {"this": (this, make(this, "this"))}
        if base:
            steps["baseline"] = (base, make(base, "baseline"))
        r = rounds(steps)
        r["this"]["kernels_ms_per_call"] = this.kernels_ms(steps["this"][1], args.steps)

        def snap(key):
            l, g, tg = outs[key]
            return l.copy(), g.download((B, T, C)), tg.download(tw.shape)

        def diff(x, y):
            return {"losses_equal": bool(np.array_equal(x[0], y[0])),
                    "grads_max_abs_diff": float(np.max(np.abs(x[1] - y[1]))),
                    "trans_grad_max_abs_diff": float(np.max(np.abs(x[2] - y[2])))}

        first = snap("this")
        r["max_rel_loss_diff_vs_graph_transitions"] = float(np.max(np.abs(graph_losses - first[0]) / np.abs(first[0])))
        this.check(steps["this"][1]())
        # the gradients are sums of atomic adds, whose order varies from call to call: the spread of this build
        # against itself is the floor of any comparison
        r["this_vs_this_again"] = diff(first, snap("this"))
        if base:
            r["this_vs_baseline"] = diff(first, snap("baseline"))
        rec[name] = r
        rec["graph_transitions_over_" + name] = rec["device_route"]["ms_per_call_median"] / r["this"]["ms_per_call_median"]
        for _, gg, tt in outs.values():
            gg.free(), tt.free()

    out = {"steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
           "l2": "flushed before every timed call",
           "buffers": "emissions, transitions and every gradient on the device; graphs as host views"}

    criteria = {"ctc_bigram": "gtnb_ngram_ctc_loss", "fal_asg": "gtnb_asg_loss_ex"}
    for name, e, graphs, kind, lens, targets in workloads():
        rec, bufs, tw, gl = workload(e, graphs, kind, lens)
        if name in criteria:  # the same inputs through the built-in target graphs' criterion
            target_criterion(criteria[name], bufs, tw, targets, lens, gl, rec)
        out[name] = rec
        for b in bufs.values():
            b.free()

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    card, plim = [x.strip() for x in (q.split(",") + ["", ""])[:2]]
    out["card"], out["power_limit_w"] = card, plim
    s = json.dumps(out)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(out, indent=1) + "\n")
    if base:
        base.close()
    ctx.close()


if __name__ == "__main__":
    main()
