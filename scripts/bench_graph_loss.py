"""gtnb_graph_loss (one user-supplied target graph per utterance) on three workloads, in one run.  One JSON record
on stdout, nothing written:

  ctc         BASELINE.json configs[1] (B=256 T=1000 C=64 U=100): the CTC graphs as generic graphs, next to
              gtnb_ctc_loss on the same inputs (what generality costs against the specialised kernel)
  decomp      word-piece alignment graphs (B=128 T=500, C = 255 pieces + 1 = 256): a seeded inventory of the 26
              letters and random 2- and 3-letter pieces, seeded transcripts of ~60 letters, each graph built with
              gtn_b200.gtn's host ops as word_decompositions.py builds it; label-uniform, so the node-labelled kernels
  wildcard    the same graphs with a wildcard state at each end (one self-loop per label): not label-uniform, so
              the arc-label kernels

For each: the implicit route and the materialised one (set_flag("implicit", 0)), every buffer on the device, ms per
step from CUDA events with L2 flushed between steps; the kernels of the implicit route (CUDA events per launch); the
graphs' node / arc / non-uniform-node counts; and the reference (oracle/_ref, tests/graph_oracle.py) on the first
--cpu-sample utterances, its wall-clock time and the largest loss difference.  The card and its power limit are read
in the same run.

    python scripts/bench_graph_loss.py [--steps 10] [--warmup 2] [--cpu-sample 2]
"""
import argparse
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cpu-sample", type=int, default=2)
    args = ap.parse_args()
    ctx = capi.Ctx(0)
    L = capi.lib()

    def region(step, profile=False):
        for _ in range(args.warmup):
            step()
        if profile:
            ctx.profile(True)
            ctx.profile_read()
        ts, pr = [], {}
        for _ in range(args.steps):
            ctx.flush_l2()
            ctx.timer_start()
            step()
            ts.append(ctx.timer_stop())
            if profile:
                for k, (cnt, ms_) in ctx.profile_read().items():
                    c0, m0 = pr.get(k, (0, 0.0))
                    pr[k] = (c0 + cnt, m0 + ms_)
        if profile:
            ctx.profile(False)
        return float(np.mean(ts)), float(np.median(ts)), {k: v[1] / args.steps for k, v in pr.items() if k != "flush_l2"}

    def workload(e, graphs, extra=None):
        B, T, C = e.shape
        views = [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
        arr = (capi.GraphView * B)(*[v for v, _ in views])
        n_arcs = sum(len(g["src"]) for g in graphs)
        e_dev, g_dev, ag_dev = ctx.to_device(e), ctx.alloc(e.nbytes), ctx.alloc(4 * max(n_arcs, 4))
        losses = np.zeros(B, np.float32)

        def step():
            ctx._check(L.gtnb_graph_loss(ctx.h, B, T, C, e_dev.ptr, 1, None, arr, None, 1,
                                         losses.ctypes.data_as(capi._f32p), g_dev.ptr, 1, ag_dev.ptr, 1))

        rec = {"shape": {"B": B, "T": T, "C": C},
               "graphs": {"nodes_mean": float(np.mean([len(g["flags"]) for g in graphs])),
                          "nodes_max": int(max(len(g["flags"]) for g in graphs)),
                          "arcs_mean": float(np.mean([len(g["src"]) for g in graphs])),
                          "arcs_max": int(max(len(g["src"]) for g in graphs)),
                          "non_uniform_nodes_mean": float(np.mean([go.non_uniform_nodes(g, C) for g in graphs]))}}
        ms, med, kern = region(step, True)
        imp_losses = losses.copy()
        rec["implicit"] = {"ms_per_step": ms, "ms_per_step_median": med, "utt_per_s": B / (ms * 1e-3),
                           "kernels_ms_per_step": kern}
        ctx.set_flag("implicit", 0)
        ms, med, kern = region(step, True)
        ctx.set_flag("implicit", 1)
        rec["materialised"] = {"ms_per_step": ms, "ms_per_step_median": med, "utt_per_s": B / (ms * 1e-3),
                               "kernels_ms_per_step": kern,
                               "max_rel_loss_vs_implicit": float(np.max(np.abs(losses - imp_losses) / np.abs(losses)))}
        rec["implicit_speedup_vs_materialised"] = rec["materialised"]["ms_per_step"] / rec["implicit"]["ms_per_step"]
        if extra:
            extra(rec, e_dev, g_dev, imp_losses)
        n = min(args.cpu_sample, B)
        t0 = time.time()
        lr, _, _ = go.ref_graph_loss(e[:n], graphs[:n])
        rec["reference_cpu"] = {"utterances": n, "s_per_utterance": (time.time() - t0) / n,
                                "max_rel_loss_diff": float(np.max(np.abs(imp_losses[:n] - lr) / np.abs(lr)))}
        for buf in (e_dev, g_dev, ag_dev):
            buf.free()
        return rec

    out = {"steps": args.steps, "warmup": args.warmup, "l2": "flushed between timed steps",
           "buffers": "emissions, emission gradients and arc gradients on the device; graphs as host views"}

    # 1. CTC graphs as generic graphs vs gtnb_ctc_loss
    B, T, C, U = 256, 1000, 64, 100
    e, targets = util.bench_inputs(B, T, C, U)
    graphs = [go.ctc_graph(t) for t in targets]

    def ctc_extra(rec, e_dev, g_dev, imp_losses):
        cat = np.ascontiguousarray(np.concatenate(targets), np.int32)
        lens = np.full(B, U, np.int32)
        losses = np.zeros(B, np.float32)

        def step():
            ctx._check(L.gtnb_ctc_loss(ctx.h, B, T, C, e_dev.ptr, 1, None, cat.ctypes.data_as(capi._i32p),
                                       lens.ctypes.data_as(capi._i32p), 0, losses.ctypes.data_as(capi._f32p),
                                       g_dev.ptr, 1))

        ms, med, kern = region(step, True)
        rec["ctc_loss"] = {"ms_per_step": ms, "ms_per_step_median": med, "kernels_ms_per_step": kern,
                           "max_rel_loss_diff_vs_graph_loss": float(np.max(np.abs(losses - imp_losses) / np.abs(losses)))}
        rec["graph_loss_over_ctc_loss"] = rec["implicit"]["ms_per_step"] / ms

    out["ctc"] = workload(e, graphs, ctc_extra)
    del e, graphs

    # 2. word-piece decompositions; 3. the same with wildcard states
    B, T = 128, 500
    pieces = go.inventory(26, 256, seed=7)
    C = len(pieces) + 1
    rng = np.random.default_rng(11)
    t0 = time.time()
    dec = []
    for b in range(B):
        letters = [int(x) for x in rng.integers(0, 26, int(rng.integers(55, 66)))]
        g = as_dict(go.decomposition_graph(GTN_OPS, letters, pieces))
        g["w"] = rng.uniform(-0.5, 0.5, len(g["src"])).astype(np.float32)
        dec.append(g)
    build_s = time.time() - t0
    e = np.random.default_rng(12).uniform(-5, 5, (B, T, C)).astype(np.float32)
    out["decomp"] = workload(e, dec)
    out["decomp"]["graph_build_s"] = build_s
    out["wildcard"] = workload(e, [go.with_wildcards(g, C, w_loop=-1.0) for g in dec])

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    card, plim = [x.strip() for x in (q.split(",") + ["", ""])[:2]]
    out["card"], out["power_limit_w"] = card, plim
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
