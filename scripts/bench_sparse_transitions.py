"""gtnb_sparse_transitions_loss (user target graphs with a learned transition graph G of any shape) on four workloads,
in one run.  One JSON record on stdout (and in --out when given):

  trigram_ctc    the trigram G at timeNgramCtc's alphabet (C = 30: 900 states, 27 000 arcs; node a*C + b = "the last
                 two labels were a, b", arc a*C+b -> b*C+m with label m), CTC graphs, B=128 T=200 U=10
  bigram_graph   the dense bigram G given as a graph (64 states, 4096 arcs), CTC graphs at the n-gram shape B=128
                 T=500 C=64 U=50, next to gtnb_graph_transitions_loss BIGRAM and gtnb_ngram_ctc_loss on the same
                 inputs: what the generality costs
  sparse_lm      a random sparse LM-like G at C = 64: 2000 states, each with a blank self-loop and 15 other labels to
                 random states (32 000 arcs), 8 start states, every state accepts; CTC graphs of targets drawn by
                 walking G from a start state, B=128 T=500 U=50
  trigram_c64    the trigram at C = 64 (4096 states, 262 144 arcs: outside the device envelope) with the targets of
                 bigram_graph: the route it takes, or its error

For each: ms per call on the device route and on the materialised route (set_flag("implicit", 0)), every buffer on
the device, from CUDA events with L2 flushed before each call, the median over --rounds rounds of --steps calls; the
kernels of each route (gtnb_profile_*, CUDA events per launch); a lower bound on the host share of a call (1 - the sum
of its kernel times over its wall-clock time; the numerator's sweeps overlap the denominator on a second stream, so the
sum counts that overlap twice); the largest relative difference between the two routes' losses; and the logsumexp
terms per second of the denominator's two sweeps (sum_b T_b * A_G terms each, counted from the shapes) against the
SFU's ex2 rate (132 SMs x 16 per clock at 1980 MHz).  The card and its power limit are read in the same run.

    python scripts/bench_sparse_transitions.py [--steps 5] [--warmup 1] [--rounds 3] [--out F]
"""
import argparse
import ctypes as Ct
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_graph_transitions import Lib  # noqa: E402
from gtn_b200 import capi  # noqa: E402
from tests import graph_oracle as go  # noqa: E402
from tests import sparse_trans_oracle as st  # noqa: E402
from tests import util  # noqa: E402

SFU_EX2_PER_S = 132 * 16 * 1.98e9


def sparse_lm(rng, S, C, per_state):
    """each state: a blank (label 0) self-loop and per_state - 1 other labels to random states; 8 start states"""
    src, dst, lab = [], [], []
    for s in range(S):
        src.append(s), dst.append(s), lab.append(0)
        for m in rng.choice(np.arange(1, C), per_state - 1, replace=False):
            src.append(s), dst.append(int(rng.integers(0, S))), lab.append(int(m))
    flags = np.full(S, 2, np.uint8)
    flags[rng.choice(S, 8, replace=False)] |= 1
    return go.make(flags, src, dst, lab)


def walk_targets(rng, G, B, U):
    """targets G accepts: U non-blank labels along a random walk from a start state"""
    out = {}
    for a in range(len(G["src"])):
        if G["olabel"][a] != 0:
            out.setdefault(int(G["src"][a]), []).append(a)
    starts = np.flatnonzero(G["flags"] & 1)
    targets = []
    for _ in range(B):
        s, t = int(rng.choice(starts)), []
        for _ in range(U):
            a = int(rng.choice(out[s]))
            t.append(int(G["olabel"][a]))
            s = int(G["dst"][a])
        targets.append(np.asarray(t, np.int32))
    return targets


def workloads():
    rng = np.random.default_rng(21)
    B, T, C, U = 128, 200, 30, 10
    e, targets = util.bench_inputs(B, T, C, U)
    yield "trigram_ctc", e, [go.ctc_graph(t, blank=0) for t in targets], st.trigram_graph(C), True, None
    B, T, C, U = 128, 500, 64, 50
    e, targets = util.bench_inputs(B, T, C, U)
    ctc = [go.ctc_graph(t, blank=0) for t in targets]
    yield "bigram_graph", e, ctc, st.bigram_graph(C), False, targets
    G = sparse_lm(rng, 2000, C, 16)
    lm_targets = walk_targets(rng, G, B, U)
    yield "sparse_lm", e, [go.ctc_graph(t, blank=0) for t in lm_targets], G, True, None
    yield "trigram_c64", e, ctc, st.trigram_graph(C), True, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = capi.Ctx(0)
    this = Lib(ctx=ctx)
    L = capi.lib()

    def timed_rounds(step):
        for _ in range(args.warmup):
            this.check(step())
        ev, wall = [], []
        for _ in range(args.rounds):
            t = [this.timed(step) for _ in range(args.steps)]
            ev.append(float(np.mean([x[0] for x in t])))
            wall.append(float(np.mean([x[1] for x in t])))
        kern = this.kernels_ms(step, args.steps)
        return {"ms_per_call_median": float(np.median(ev)), "ms_rounds": ev,
                "wall_ms_per_call_median": float(np.median(wall)), "kernels_ms_per_call": kern,
                "host_share_lower_bound": max(0.0, 1.0 - sum(kern.values()) / float(np.median(wall)))}

    out = {"steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "l2": "flushed before every timed call",
           "buffers": "emissions, transitions and every gradient on the device; graphs as host views",
           "sfu_ex2_per_s": SFU_EX2_PER_S}
    for name, e, graphs, G, exact, targets in workloads():
        B, T, C = e.shape
        views = [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
        arr = (capi.GraphView * B)(*[v for v, _ in views])
        gv, _keep = capi.make_view(G["flags"], G["src"], G["dst"], G["olabel"], G["olabel"])
        n_arcs = sum(len(g["src"]) for g in graphs)
        tw = np.random.default_rng(5).uniform(-1, 1, len(G["src"])).astype(np.float32)
        bufs = dict(e=ctx.to_device(e), g=ctx.alloc(e.nbytes), ag=ctx.alloc(4 * max(n_arcs, 4)), tw=ctx.to_device(tw),
                    tg=ctx.alloc(tw.nbytes))
        losses = np.zeros(B, np.float32)

        def step():
            return L.gtnb_sparse_transitions_loss(
                ctx.h, B, T, C, bufs["e"].ptr, 1, None, arr, None, 1, Ct.byref(gv), bufs["tw"].ptr, 1,
                losses.ctypes.data_as(capi._f32p), bufs["g"].ptr, 1, bufs["ag"].ptr, 1, bufs["tg"].ptr, 1)

        rec = {"shape": {"B": B, "T": T, "C": C}, "G": {"states": len(G["flags"]), "arcs": len(G["src"])},
               "graphs": {"nodes_mean": float(np.mean([len(g["flags"]) for g in graphs])),
                          "arcs_mean": float(np.mean([len(g["src"]) for g in graphs]))}}
        rc = step()
        if rc:
            rec["error"] = {"code": rc, "message": L.gtnb_last_error(ctx.h).decode()}
            out[name] = rec
            for b in bufs.values():
                b.free()
            print(json.dumps({name: rec}), file=sys.stderr)
            continue
        r = timed_rounds(step)
        kern = r["kernels_ms_per_call"]
        r["route_taken"] = "device" if "sparse_den_forward" in kern else "materialised"
        dev = losses.copy()
        rec["finite_losses"] = int(np.isfinite(dev).sum())
        if "sparse_den_forward" in kern:
            terms = float(B * T * rec["G"]["arcs"])  # sum_b T_b * A_G, every T_b = T
            den_ms = kern["sparse_den_forward"] + kern.get("sparse_den_backward", 0.0)
            r["den_lse_terms_per_s"] = 2 * terms / (den_ms * 1e-3)
            r["den_lse_terms_over_sfu_ex2_rate"] = r["den_lse_terms_per_s"] / SFU_EX2_PER_S
        rec["device_route"] = r
        if exact:
            ctx.set_flag("implicit", 0)
            try:
                rc = step()
                if rc:
                    rec["exact_route"] = {"error": {"code": rc, "message": L.gtnb_last_error(ctx.h).decode()}}
                else:
                    rec["exact_route"] = timed_rounds(step)
                    ex = losses.copy()
                    fin = np.isfinite(dev) & np.isfinite(ex)
                    rec["max_rel_loss_diff_between_routes"] = float(
                        np.max(np.abs(ex[fin] - dev[fin]) / np.abs(ex[fin]), initial=0.0))
                    rec["same_non_finite_losses"] = bool(np.array_equal(np.isfinite(dev), np.isfinite(ex)))
                    rec["device_speedup_vs_exact"] = (rec["exact_route"]["ms_per_call_median"] /
                                                      rec["device_route"]["ms_per_call_median"])
            finally:
                ctx.set_flag("implicit", 1)
        if targets is not None:  # the same inputs through the dense criteria
            cat = np.ascontiguousarray(np.concatenate(targets), np.int32)
            tl = np.asarray([len(t) for t in targets], np.int32)
            W = tw[np.argsort(st.bigram_slots(C))]  # W[i*C + j] = the weight of arc j -> i
            wd = ctx.to_device(W)
            l2 = np.zeros(B, np.float32)
            tg2 = ctx.alloc(W.nbytes)

            def dense():
                return L.gtnb_graph_transitions_loss(
                    ctx.h, B, T, C, bufs["e"].ptr, 1, None, arr, None, 1, capi.DENSE_BIGRAM, wd.ptr, 1,
                    l2.ctypes.data_as(capi._f32p), bufs["g"].ptr, 1, bufs["ag"].ptr, 1, tg2.ptr, 1)

            def ngram():
                return L.gtnb_ngram_ctc_loss(
                    ctx.h, B, T, C, bufs["e"].ptr, 1, None, wd.ptr, 1, cat.ctypes.data_as(capi._i32p),
                    tl.ctypes.data_as(capi._i32p), 0, l2.ctypes.data_as(capi._f32p), bufs["g"].ptr, 1, tg2.ptr, 1)

            for key, fn in (("gtnb_graph_transitions_loss_bigram", dense), ("gtnb_ngram_ctc_loss", ngram)):
                rr = timed_rounds(fn)
                rr["max_rel_loss_diff_vs_sparse"] = float(np.max(np.abs(l2 - dev) / np.abs(l2)))
                rec[key] = rr
                rec["sparse_over_" + key] = rec["device_route"]["ms_per_call_median"] / rr["ms_per_call_median"]
            wd.free(), tg2.free()
        out[name] = rec
        print(json.dumps({name: rec}), file=sys.stderr)
        for b in bufs.values():
            b.free()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    card, plim = [x.strip() for x in (q.split(",") + ["", ""])[:2]]
    out["card"], out["power_limit_w"] = card, plim
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(out, indent=1) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
