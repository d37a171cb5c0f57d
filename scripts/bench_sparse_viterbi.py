"""gtnb_viterbi_sparse (decode: best path of intersect(E_b, G)) and gtnb_sparse_transitions_viterbi (align: best path
of intersect(intersect(A_b, G), E_b)) on the workloads of scripts/bench_sparse_transitions.py (its workloads()), in
one run, plus one tie-heavy variant.  One JSON record on stdout (and in --out when given):

  trigram_ctc       the trigram G at C = 30 (900 states, 27 000 arcs), CTC targets, B=128 T=200
  bigram_graph      the dense bigram given as a graph, C = 64, B=128 T=500 U=50
  sparse_lm         a random 2000-state token LM (32 000 arcs) at C = 64, B=128 T=500
  trigram_c64       the trigram at C = 64 (4096 states, 262 144 arcs: outside the device envelope), first --b-large
                    utterances only: the materialised lattice is T_b * 262 144 arcs per utterance
  trigram_ctc_ties  trigram_ctc with zero transitions (every utterance ties)

For each operation: ms per call on the device route and on the materialised route (set_flag("implicit", 0)), every
buffer on the device, L2 flushed before every call, the routes alternating, median over --rounds rounds; the kernels
of the device route (CUDA events per launch, in a profiled pass of its own); the share of the call outside those
kernels; whether the exact route ran (its kernels in the profile) and, for the decode, how many utterances of the
whole batch it re-runs there and why, predicted with the float32 restatement of tests/sparse_viterbi_oracle.py (a tie
on the traced path, or a non-finite used value), and the call's time with exact_ties off (no re-run for ties);
whether both routes' paths, arcs and scores are ==.  Beside bigram_graph: gtnb_viterbi_dense_ex BIGRAM and gtnb_graph_transitions_viterbi
BIGRAM on the same inputs.  The card and its power limit are read in the same run.

    python scripts/bench_sparse_viterbi.py [--rounds 5] [--warmup 1] [--b-large 8] [--out F]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench_sparse_transitions as bst  # noqa: E402  (the workload builders)
from gtn_b200 import capi  # noqa: E402
from tests import sparse_trans_oracle as st  # noqa: E402
from tests import sparse_viterbi_oracle as sv  # noqa: E402

EXACT = ("compose_emit",)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--b-large", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = capi.Ctx(0)
    L = capi.lib()

    def timed(step):
        ctx.flush_l2()
        ctx.timer_start()
        step()
        return ctx.timer_stop()

    def on_route(implicit, fn):
        ctx.set_flag("implicit", implicit)
        try:
            return fn()
        finally:
            ctx.set_flag("implicit", 1)

    def measure(step, outputs, B):
        """both routes of one call -> record"""
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
        return {"device": {"ms_per_call_median": dev_ms, "ms_per_call_min": float(np.min(dev)),
                           "utt_per_s": B / (dev_ms * 1e-3), "kernels_ms_per_call": kern, "kernels_ms_total": kern_ms,
                           "share_outside_kernels": 1.0 - kern_ms / dev_ms},
                "materialised": {"ms_per_call_median": mat_ms, "ms_per_call_min": float(np.min(mat))},
                "device_speedup_vs_materialised": mat_ms / dev_ms,
                "exact_route_ran_on_the_device_route_call": any(k in kern for k in EXACT),
                "routes_equal": {"paths": bool(np.array_equal(got_dev[0], got_mat[0])),
                                 "scores": bool(np.array_equal(got_dev[1], got_mat[1])),
                                 "arcs": bool(np.array_equal(got_dev[2], got_mat[2]))}}

    def workload(name, e, graphs, G, tw):
        B, T, C = e.shape
        gv = capi.make_view(G["flags"], G["src"], G["dst"], G["olabel"], G["olabel"], None)
        views = [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
        arr = (capi.GraphView * B)(*[v for v, _ in views])
        bufs = [ctx.to_device(e), ctx.to_device(tw), ctx.alloc(4 * B * T), ctx.alloc(4 * B * T), ctx.alloc(4 * B)]
        e_dev, w_dev, p_dev, a_dev, s_dev = bufs

        def outputs():
            return (p_dev.download((B, T), np.int32), s_dev.download((B,)), a_dev.download((B, T), np.int32))

        def decode():
            ctx._check(L.gtnb_viterbi_sparse(ctx.h, B, T, C, e_dev.ptr, 1, None, capi.C.byref(gv[0]), w_dev.ptr, 1,
                                             p_dev.ptr, a_dev.ptr, s_dev.ptr, 1))

        def align():
            ctx._check(L.gtnb_sparse_transitions_viterbi(ctx.h, B, T, C, e_dev.ptr, 1, None, arr, None, 1,
                                                         capi.C.byref(gv[0]), w_dev.ptr, 1, p_dev.ptr, a_dev.ptr,
                                                         s_dev.ptr, 1))

        rec = {"shape": {"B": B, "T": T, "C": C}, "G": {"states": len(G["flags"]), "arcs": len(G["src"])}}
        rec["decode"] = measure(decode, outputs, B)
        # the utterances the decode hands to the exact route, and why, PREDICTED over the whole batch by the float32
        # restatement (its tie rule is held to the kernel's status bit in tests/test_sparse_viterbi_emulation.py)
        _, ids = sv.kept(G, tw, C)
        used = np.zeros(C, bool)
        used[G["olabel"][ids]] = True
        non_finite = [b for b in range(B) if not (np.isfinite(tw[ids]).all() and np.isfinite(e[b][:, used]).all())]
        ties = [b for b in range(B) if b not in non_finite and sv.decode_outcome(e[b], G, tw, C)[1]]
        rec["decode"]["predicted_reruns"] = {"utterances": B, "tie": len(ties), "non_finite": len(non_finite)}
        ctx.set_flag("exact_ties", 0)
        try:
            for _ in range(args.warmup):
                decode()
            rec["decode"]["device_exact_ties_off_ms_median"] = float(np.median([timed(decode)
                                                                               for _ in range(args.rounds)]))
        finally:
            ctx.set_flag("exact_ties", 1)
        rec["align"] = measure(align, outputs, B)
        for buf in bufs:
            buf.free()
        return rec

    def dense_beside(e, graphs, W):
        """gtnb_viterbi_dense_ex BIGRAM and gtnb_graph_transitions_viterbi BIGRAM on the bigram graph's inputs"""
        B, T, C = e.shape
        views = [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
        arr = (capi.GraphView * B)(*[v for v, _ in views])
        bufs = [ctx.to_device(e), ctx.to_device(W), ctx.alloc(4 * B * T), ctx.alloc(4 * B * T), ctx.alloc(4 * B)]
        e_dev, w_dev, p_dev, a_dev, s_dev = bufs
        out = {}
        for name, step in (
                ("viterbi_dense_ex_bigram", lambda: ctx._check(L.gtnb_viterbi_dense_ex(
                    ctx.h, B, T, C, e_dev.ptr, 1, None, capi.DENSE_BIGRAM, w_dev.ptr, 1, p_dev.ptr, s_dev.ptr, 1))),
                ("graph_transitions_viterbi_bigram", lambda: ctx._check(L.gtnb_graph_transitions_viterbi(
                    ctx.h, B, T, C, e_dev.ptr, 1, None, arr, None, 1, capi.DENSE_BIGRAM, w_dev.ptr, 1, p_dev.ptr,
                    a_dev.ptr, s_dev.ptr, 1)))):
            for _ in range(args.warmup):
                step()
            out[name] = {"ms_per_call_median": float(np.median([timed(step) for _ in range(args.rounds)]))}
        for buf in bufs:
            buf.free()
        return out

    out = {"rounds": args.rounds, "warmup": args.warmup, "l2": "flushed before every timed call",
           "buffers": "emissions, transitions, paths, arcs and scores on the device; graphs as host views"}
    rng = np.random.default_rng(5)
    for name, e, graphs, G, _, _ in bst.workloads():
        if name == "trigram_c64":
            e, graphs = e[:args.b_large], graphs[:args.b_large]
        tw = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
        out[name] = workload(name, e, graphs, G, tw)
        if name == "bigram_graph":
            C = e.shape[2]
            W = np.empty(C * C, np.float32)
            W[st.bigram_slots(C)] = tw
            out[name]["beside"] = dense_beside(e, graphs, W)
        if name == "trigram_ctc":
            out[name + "_ties"] = workload(name + "_ties", e, graphs, G, np.zeros(len(G["src"]), np.float32))
        for n in (name, name + "_ties"):
            if n in out:
                print(n, json.dumps({k: {r: out[n][k][r] for r in ("device", "materialised", "routes_equal")}
                                     for k in ("decode", "align")}), file=sys.stderr, flush=True)

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
