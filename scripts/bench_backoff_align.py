"""gtnb_backoff_transitions_viterbi on scripts/bench_backoff.py's workload: the pruned backoff trigram LM
(tests/backoff_oracle.py's backoff_lm: C = 64, 2065 states, 17 344 emitting arcs and 2064 epsilon arcs, two levels)
with CTC target graphs at B=128 T=500 U=50.  One JSON record on stdout (and in --out when given):

  device          the whole batch on the device route, exact_ties on and off: ms per call, the kernels (CUDA events
                  per launch, in a profiled pass of its own) and the call's time outside them (host packing of the
                  numerators, staging, the status read-back)
  first_<b-large> both routes on the first --b-large utterances (the materialised route composes A_b with G, then
                  with E_b, one utterance at a time), alternating, and their outputs compared (paths, arcs, scores ==)

Per call: ms (L2 flushed before every call, median over --rounds).  The card and its power limit are read in the same
run.

    python scripts/bench_backoff_align.py [--rounds 5] [--warmup 1] [--b-large 4] [--out F]
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
from gtn_b200 import capi  # noqa: E402
from tests import backoff_oracle as bo  # noqa: E402
from tests import graph_oracle as go  # noqa: E402
from tests import util  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--b-large", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = capi.Ctx(0)
    L = capi.lib()

    def timed(step):
        ctx.flush_l2()
        ctx.timer_start()
        step()
        return ctx.timer_stop()

    def kernels(step):
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
        return kern

    def on_route(implicit, fn):
        ctx.set_flag("implicit", implicit)
        try:
            return fn()
        finally:
            ctx.set_flag("implicit", 1)

    def call(e, graphs, G, tw):
        """(alignment step, outputs) on device buffers"""
        B, T, C = e.shape
        gv = capi.make_view(G["flags"], G["src"], G["dst"], G["olabel"], G["olabel"], None)
        views = [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
        arr = (capi.GraphView * B)(*[v for v, _ in views])
        e_dev, w_dev = ctx.to_device(e), ctx.to_device(tw)
        p_dev, a_dev, s_dev = ctx.alloc(4 * B * T), ctx.alloc(4 * B * T), ctx.alloc(4 * B)
        keep = (gv, views, arr, e_dev, w_dev, p_dev, a_dev, s_dev)

        def align():
            ctx._check(L.gtnb_backoff_transitions_viterbi(ctx.h, B, T, C, e_dev.ptr, 1, None, arr, None, 1,
                                                          Ct.byref(gv[0]), w_dev.ptr, 1, p_dev.ptr, a_dev.ptr,
                                                          s_dev.ptr, 1))

        def outputs():
            return p_dev.download((B, T), np.int32), s_dev.download((B,)), a_dev.download((B, T), np.int32)

        return align, outputs, keep

    def ms_list(step, implicit):
        for _ in range(args.warmup):
            on_route(implicit, step)
        return [on_route(implicit, lambda: timed(step)) for _ in range(args.rounds)]

    rng = np.random.default_rng(64)
    G, tw = bo.backoff_lm(rng, 64)
    B, T, C, U = 128, 500, 64, 50
    e, targets = util.bench_inputs(B, T, C, U)
    graphs = [go.ctc_graph(t, blank=0) for t in targets]
    out = {"rounds": args.rounds, "warmup": args.warmup, "l2": "flushed before every timed call",
           "buffers": "emissions, transitions and outputs on the device; graphs as host views",
           "shape": {"B": B, "T": T, "C": C, "U": U},
           "G": {"states": len(G["flags"]), "emitting_arcs": int((G["olabel"] >= 0).sum()),
                 "epsilon_arcs": int((G["olabel"] == -1).sum()), "levels": int(bo.closure_levels(G)[0].max())}}

    # the whole batch on the device route
    align, outputs, keep = call(e, graphs, G, tw)
    rec = {}
    for ties in (1, 0):
        ctx.set_flag("exact_ties", ties)
        try:
            ms = ms_list(align, 1)
            kern = kernels(align)
        finally:
            ctx.set_flag("exact_ties", 1)
        med = float(np.median(ms))
        k_ms = float(sum(kern.values()))
        rec["exact_ties_on" if ties else "exact_ties_off"] = {
            "ms_per_call_median": med, "ms_per_call_min": float(np.min(ms)), "utt_per_s": B / (med * 1e-3),
            "kernels_ms_per_call": kern, "kernels_ms_sum": k_ms, "outside_kernels_ms": med - k_ms,
            "host_share": (med - k_ms) / med, "exact_route_ran": any(k.startswith("gcompose") for k in kern)}
    align()
    paths, scores, arcs = outputs()
    rec["finite_scores"] = int(np.isfinite(scores).sum())
    out["device"] = rec
    print("device", json.dumps(rec), file=sys.stderr, flush=True)

    # both routes on the first b_large utterances
    nb = args.b_large
    align_s, outputs_s, keep_s = call(e[:nb], graphs[:nb], G, tw)
    dev, mat = [], []
    for _ in range(args.warmup):
        align_s()
        on_route(0, align_s)
    for _ in range(args.rounds):
        dev.append(timed(align_s))
        mat.append(on_route(0, lambda: timed(align_s)))
    align_s()
    got_dev = outputs_s()
    on_route(0, align_s)
    got_mat = outputs_s()
    out["first_%d" % nb] = {
        "device_ms_median": float(np.median(dev)), "materialised_ms_median": float(np.median(mat)),
        "device_speedup_vs_materialised": float(np.median(mat) / np.median(dev)),
        "routes_equal": {k: bool(np.array_equal(x, y)) for k, x, y in zip(("paths", "scores", "arcs"), got_dev,
                                                                         got_mat)},
        "device_equals_full_batch_rows": bool(np.array_equal(got_dev[1], scores[:nb]))}
    print("first_%d" % nb, json.dumps(out["first_%d" % nb]), file=sys.stderr, flush=True)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    card, plim = [x.strip() for x in (q.split(",") + ["", ""])[:2]]
    out["card"], out["power_limit_w"] = card, plim
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(out, indent=1) + "\n")
    for k in (keep, keep_s):
        for buf in k[3:]:
            buf.free()
    ctx.close()


if __name__ == "__main__":
    main()
