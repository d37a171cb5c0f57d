"""gtnb_graph_viterbi (Viterbi alignment over user-supplied target graphs) on three workloads, in one run.  One JSON
record on stdout, nothing written:

  ctc         BASELINE.json configs[1] (B=256 T=1000 C=64 U=100): CTC graphs, i.e. CTC forced alignment
  decomp      word-piece alignment graphs (B=128 T=500, C = 255 pieces + 1 = 256), built as scripts/bench_graph_loss.py
              builds them (label-uniform: the node-labelled kernels)
  wildcard    the same graphs with a wildcard state at each end (not label-uniform: the arc-label kernels)

For each: ms per call on the device route (tropical sweep + traceback) and on the materialised route
(set_flag("implicit", 0)), every buffer on the device, L2 flushed before every call, the two routes alternating,
median over --rounds rounds; the kernels of the device route (CUDA events per launch, in a profiled pass of its own);
the share of the device-route call spent outside those kernels (host packing of the graph tables, launches, the
status read-back, and the exact route of tied utterances, if any: the kernels cannot start before the host has packed
the tables, so on a call without exact route this bounds the host's share from below, up to the read-back copy); how
many utterances took the exact route on the device-route call, and why (a tie on the traced path or a non-finite
value, counted with the float32 restatement of tests/graph_viterbi_oracle.py; the profile shows whether compose
kernels ran); that both routes' paths, arcs and scores are ==; and the reference
(oracle/_ref) on the first --cpu-sample utterances, its wall-clock time per utterance and whether it agrees.  The card
and its power limit are read in the same run.

    python scripts/bench_graph_viterbi.py [--rounds 10] [--warmup 2] [--cpu-sample 2]
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench_graph_loss as bgl  # noqa: E402  (the workload builders)
from gtn_b200 import capi  # noqa: E402
from tests import graph_oracle as go  # noqa: E402
from tests import graph_viterbi_oracle as gv  # noqa: E402
from tests import util  # noqa: E402

COMPOSE = ("compose_count", "compose_emit")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cpu-sample", type=int, default=2)
    args = ap.parse_args()
    ctx = capi.Ctx(0)
    L = capi.lib()

    def timed(step):
        ctx.flush_l2()
        ctx.timer_start()
        step()
        return ctx.timer_stop()

    def workload(e, graphs):
        B, T, C = e.shape
        views = [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
        arr = (capi.GraphView * B)(*[v for v, _ in views])
        e_dev = ctx.to_device(e)
        bufs = [e_dev, ctx.alloc(4 * B * T), ctx.alloc(4 * B * T), ctx.alloc(4 * B)]
        _, p_dev, a_dev, s_dev = bufs

        def step():
            ctx._check(L.gtnb_graph_viterbi(ctx.h, B, T, C, e_dev.ptr, 1, None, arr, None, 1, p_dev.ptr, a_dev.ptr,
                                            s_dev.ptr, 1))

        def outputs():
            return (p_dev.download((B, T), np.int32), s_dev.download((B,)), a_dev.download((B, T), np.int32))

        def on_route(implicit, fn):
            ctx.set_flag("implicit", implicit)
            try:
                return fn()
            finally:
                ctx.set_flag("implicit", 1)

        rec = {"shape": {"B": B, "T": T, "C": C},
               "graphs": {"nodes_mean": float(np.mean([len(g["flags"]) for g in graphs])),
                          "nodes_max": int(max(len(g["flags"]) for g in graphs)),
                          "arcs_mean": float(np.mean([len(g["src"]) for g in graphs])),
                          "arcs_max": int(max(len(g["src"]) for g in graphs)),
                          "non_uniform_nodes_mean": float(np.mean([go.non_uniform_nodes(g, C) for g in graphs]))}}
        for implicit in (1, 0):
            for _ in range(args.warmup):
                on_route(implicit, step)
        dev, mat = [], []
        for _ in range(args.rounds):  # alternating: drift on the shared machine hits both routes alike
            dev.append(timed(step))
            mat.append(on_route(0, lambda: timed(step)))
        got_dev = outputs()
        on_route(0, step)
        got_mat = outputs()
        # kernels of the device route, in a pass of its own (profiling adds events around every launch)
        ctx.profile(True)
        ctx.profile_read()
        kern = {}
        for _ in range(args.rounds):
            ctx.flush_l2()
            step()
            for k, (cnt, ms_) in ctx.profile_read().items():
                if k != "flush_l2":
                    kern[k] = kern.get(k, 0.0) + ms_ / args.rounds
        ctx.profile(False)
        dev_ms, mat_ms = float(np.median(dev)), float(np.median(mat))
        kern_ms = sum(kern.values())
        exact_kernels = [k for k in COMPOSE if k in kern]
        rec["device"] = {"ms_per_call_median": dev_ms, "ms_per_call_min": float(np.min(dev)),
                         "utt_per_s": B / (dev_ms * 1e-3), "kernels_ms_per_call": kern,
                         "kernels_ms_total": kern_ms, "share_outside_kernels": 1.0 - kern_ms / dev_ms}
        rec["materialised"] = {"ms_per_call_median": mat_ms, "ms_per_call_min": float(np.min(mat)),
                               "utt_per_s": B / (mat_ms * 1e-3)}
        rec["device_speedup_vs_materialised"] = mat_ms / dev_ms
        # which utterances the device route hands to the exact route, and why, from the float32 restatement of the
        # sweep: a tie on the traced path, or a non-finite emission or weight
        ties = sum(gv.trace_ties(e[b], graphs[b], C, got_dev[2][b]) for b in range(B))
        non_finite = sum(not (np.isfinite(e[b]).all() and np.isfinite(graphs[b]["w"]).all()) for b in range(B))
        rec["exact_route"] = {"compose_kernels_launched": bool(exact_kernels), "utterances_tie": int(ties),
                              "utterances_non_finite": int(non_finite)}
        rec["routes_equal"] = {"paths": bool(np.array_equal(got_dev[0], got_mat[0])),
                               "scores": bool(np.array_equal(got_dev[1], got_mat[1])),
                               "arcs": bool(np.array_equal(got_dev[2], got_mat[2]))}
        n = min(args.cpu_sample, B)
        t0 = time.time()
        pr, sr, ar = gv.ref_graph_viterbi(e[:n], graphs[:n])
        rec["reference_cpu"] = {"utterances": n, "s_per_utterance": (time.time() - t0) / n,
                                "equal": bool(np.array_equal(pr, got_dev[0][:n]) and np.array_equal(sr, got_dev[1][:n])
                                              and np.array_equal(ar, got_dev[2][:n]))}
        for buf in bufs:
            buf.free()
        return rec

    out = {"rounds": args.rounds, "warmup": args.warmup, "l2": "flushed before every timed call",
           "buffers": "emissions, paths, arcs and scores on the device; graphs as host views"}

    B, T, C, U = 256, 1000, 64, 100
    e, targets = util.bench_inputs(B, T, C, U)
    out["ctc"] = workload(e, [go.ctc_graph(t) for t in targets])
    del e

    B, T = 128, 500
    pieces = go.inventory(26, 256, seed=7)
    C = len(pieces) + 1
    rng = np.random.default_rng(11)
    dec = []
    for b in range(B):
        letters = [int(x) for x in rng.integers(0, 26, int(rng.integers(55, 66)))]
        g = bgl.as_dict(go.decomposition_graph(bgl.GTN_OPS, letters, pieces))
        g["w"] = rng.uniform(-0.5, 0.5, len(g["src"])).astype(np.float32)
        dec.append(g)
    e = np.random.default_rng(12).uniform(-5, 5, (B, T, C)).astype(np.float32)
    out["decomp"] = workload(e, dec)
    out["wildcard"] = workload(e, [go.with_wildcards(g, C, w_loop=-1.0) for g in dec])

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    card, plim = [x.strip() for x in (q.split(",") + ["", ""])[:2]]
    out["card"], out["power_limit_w"] = card, plim
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
