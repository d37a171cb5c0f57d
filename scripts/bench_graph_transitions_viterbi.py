"""gtnb_graph_transitions_viterbi (Viterbi alignment over user-supplied target graphs with learned ASG or bigram
transitions) on the four workloads of scripts/bench_graph_transitions.py (built by its workloads()), in one run.  One
JSON record on stdout (and in --out when given):

  decomp_asg    word-piece decomposition graphs with ASG transitions, B=128 T=500 C=128
  ctc_bigram    CTC graphs with bigram transitions, B=128 T=500 C=64 U=50
  fal_asg       ASG force-align chains with ASG transitions, same shape
  wildcard_asg  decomposition graphs at C=64 with a wildcard state at each end, ASG transitions

For each: ms per call on the device route (tropical sweep of the products + traceback) and on the materialised route
(set_flag("implicit", 0): compose(A_b, G) in the reference's numbering, then the lattice), every buffer on the device,
L2 flushed before every call, the two routes alternating, median over --rounds rounds; the kernels of the device route
(CUDA events per launch, in a profiled pass of its own); the share of the device-route call spent outside those
kernels, a lower bound on the host's share when no utterance re-ran on the exact route; how many utterances the device
route hands to the exact route, and why (a tie on the traced path or a non-finite value), predicted with the float32
restatement of tests/graph_trans_viterbi_oracle.py, beside whether the exact route ran (its kernels in the profile); whether both routes' paths, arcs and scores are ==; and the
reference (oracle/_ref) on the first --cpu-sample utterances, its wall-clock time per utterance and whether it agrees.
The card and its power limit are read in the same run.

    python scripts/bench_graph_transitions_viterbi.py [--rounds 10] [--warmup 2] [--cpu-sample 2] [--out F]
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
import bench_graph_transitions as bgt  # noqa: E402  (the workload builders)
from gtn_b200 import capi  # noqa: E402
from tests import graph_trans_viterbi_oracle as gtv  # noqa: E402

EXACT = ("gcompose_search", "compose_emit")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cpu-sample", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = capi.Ctx(0)
    L = capi.lib()

    def timed(step):
        ctx.flush_l2()
        ctx.timer_start()
        step()
        return ctx.timer_stop()

    def workload(e, graphs, kind, lens):
        B, T, C = e.shape
        views = [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
        arr = (capi.GraphView * B)(*[v for v, _ in views])
        tw = bgt.transitions(C, kind)
        il = None if lens is None else np.ascontiguousarray(lens, np.int32)
        bufs = [ctx.to_device(e), ctx.to_device(tw), ctx.alloc(4 * B * T), ctx.alloc(4 * B * T), ctx.alloc(4 * B)]
        e_dev, w_dev, p_dev, a_dev, s_dev = bufs

        def step():
            ctx._check(L.gtnb_graph_transitions_viterbi(
                ctx.h, B, T, C, e_dev.ptr, 1, None if il is None else il.ctypes.data_as(capi._i32p), arr, None, 1,
                kind, w_dev.ptr, 1, p_dev.ptr, a_dev.ptr, s_dev.ptr, 1))

        def outputs():
            return (p_dev.download((B, T), np.int32), s_dev.download((B,)), a_dev.download((B, T), np.int32))

        def on_route(implicit, fn):
            ctx.set_flag("implicit", implicit)
            try:
                return fn()
            finally:
                ctx.set_flag("implicit", 1)

        rec = {"shape": {"B": B, "T": T, "C": C}, "kind": "asg" if kind == capi.DENSE_ASG else "bigram",
               "graphs": {"nodes_mean": float(np.mean([len(g["flags"]) for g in graphs])),
                          "arcs_mean": float(np.mean([len(g["src"]) for g in graphs]))}}
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
        device_route = "product_arc_map" in kern
        rec["device"] = {"ms_per_call_median": dev_ms, "ms_per_call_min": float(np.min(dev)),
                         "utt_per_s": B / (dev_ms * 1e-3), "kernels_ms_per_call": kern, "kernels_ms_total": kern_ms,
                         "share_outside_kernels": 1.0 - kern_ms / dev_ms, "took_the_device_route": device_route}
        rec["materialised"] = {"ms_per_call_median": mat_ms, "ms_per_call_min": float(np.min(mat)),
                               "utt_per_s": B / (mat_ms * 1e-3)}
        rec["device_speedup_vs_materialised"] = mat_ms / dev_ms
        # the utterances the device route hands to the exact route, and why, PREDICTED by the float32 restatement of
        # the sweep over the same products (a tie on the traced path, or a non-finite emission or weight; its tie rule
        # is checked against the kernel's status bit in tests/test_graph_trans_viterbi_emulation.py); the call itself
        # reports only whether the exact route ran, which the profile shows
        ties = non_finite = 0
        if device_route:
            tw_h = tw
            for b in range(B):
                n = T if lens is None else int(lens[b])
                p, _ = gtv.tropical_product(graphs[b], C, kind, tw_h)
                if not (np.isfinite(e[b, :n]).all() and np.isfinite(p["w"]).all()):
                    non_finite += 1
                elif gtv.device_route_outcome(e[b, :n], p, C)[1]:
                    ties += 1
        rec["exact_route"] = {"ran": any(k in kern for k in EXACT),
                              "predicted_utterances_tie": int(ties),
                              "predicted_utterances_non_finite": int(non_finite)}
        rec["routes_equal"] = {"paths": bool(np.array_equal(got_dev[0], got_mat[0])),
                               "scores": bool(np.array_equal(got_dev[1], got_mat[1])),
                               "arcs": bool(np.array_equal(got_dev[2], got_mat[2]))}
        n = min(args.cpu_sample, B)
        t0 = time.time()
        pr, sr, ar = gtv.ref_graph_trans_viterbi(e[:n], graphs[:n], kind, tw, None if lens is None else lens[:n])
        rec["reference_cpu"] = {"utterances": n, "s_per_utterance": (time.time() - t0) / n,
                                "equal": bool(np.array_equal(pr, got_dev[0][:n]) and np.array_equal(sr, got_dev[1][:n])
                                              and np.array_equal(ar, got_dev[2][:n]))}
        for buf in bufs:
            buf.free()
        return rec

    out = {"rounds": args.rounds, "warmup": args.warmup, "l2": "flushed before every timed call",
           "buffers": "emissions, transitions, paths, arcs and scores on the device; graphs as host views"}
    for name, e, graphs, kind, lens, _ in bgt.workloads():
        out[name] = workload(e, graphs, kind, lens)
        print(name, json.dumps({k: out[name][k] for k in ("device", "materialised", "exact_route", "routes_equal")}),
              file=sys.stderr, flush=True)

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
