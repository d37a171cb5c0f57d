"""The cluster route of the backoff entry points (gtnb_ctx_set_flag "sparse_cluster": the denominator of a backoff
transition graph G beyond one CTA swept by one thread-block cluster per utterance, k_sparse.cu's sparse_cl_eps_*
kernels), measured in one run.  One JSON record on stdout (and in --out when given):

  fourgram_c64, fivegram_c64
                    the backoff 4-gram (C = 64, 60 000 tokens, seed 1) and 5-gram (C = 64, 150 000 tokens, min count
                    5) of tests/backoff_oracle.py's backoff_ngram, beyond the one-CTA envelope, with CTC graphs at
                    B=128 T=500 U=50, flag 1: gtnb_backoff_transitions_loss (with every gradient), gtnb_viterbi_backoff
                    with exact_ties on and off, and gtnb_backoff_transitions_viterbi, ms per call and per kernel.
                    `small` compares the first --b-small utterances at T = --t-small on the cluster route and on the
                    materialised route (implicit 0): time, and whether the outputs agree.
  pruned_trigram    the benchmark's pruned backoff trigram (2065 states, inside the one-CTA envelope) with the flag at
                    0 (one CTA per utterance) and at 2, 4 and 8 (that many CTAs per utterance): loss and decode, ms
                    per call and per kernel, and whether the outputs are == the flag-0 outputs.

Every buffer on the device, L2 flushed before every timed call, one warm-up call per shape and setting, the
settings alternating inside a round, median over --rounds rounds; kernel times from CUDA events per launch in a
profiled pass of its own.  The card and its power limit are read in the same run.

    python scripts/bench_backoff_cluster.py [--rounds 3] [--b-small 2] [--t-small 50] [--out F]
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

DEFAULTS = {"sparse_cluster": 0, "implicit": 1, "exact_ties": 1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--b-small", type=int, default=2)
    ap.add_argument("--t-small", type=int, default=50)
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
        ctx.flush_l2()
        step()
        kern = {k: ms for k, (_, ms) in ctx.profile_read().items() if k != "flush_l2"}
        ctx.profile(False)
        return kern

    def with_settings(settings, step):
        """step() under {flag name: value}, every flag put back to its default afterwards"""
        for k, v in settings.items():
            ctx.set_flag(k, v)
        try:
            return step()
        finally:
            for k in settings:
                ctx.set_flag(k, DEFAULTS[k])

    def compare(variants, step, outputs):
        """variants: {name: settings}; one warm-up each, then rounds in which the variants alternate -> {name: record}
        with the outputs of each compared with the first variant's"""
        names, outs = [], {}
        for n in variants:
            with_settings(variants[n], step)
            names.append(n)
            outs[n] = outputs()
        ms = {n: [] for n in names}
        for _ in range(args.rounds):
            for n in names:
                ms[n].append(with_settings(variants[n], lambda: timed(step)))
        rec = {}
        for n in names:
            rec[n] = {"ms_per_call_median": float(np.median(ms[n])), "ms_rounds": ms[n],
                      "kernels_ms_per_call": with_settings(variants[n], lambda: kernels(step)),
                      "outputs_equal_first_variant": [bool(np.array_equal(x, y, equal_nan=True))
                                                      for x, y in zip(outs[n], outs[names[0]])],
                      "max_rel_diff_vs_first_variant": [
                          float(np.nanmax(np.abs(x.astype(np.float64) - y) / np.maximum(np.abs(y), 1e-6), initial=0.0))
                          for x, y in zip(outs[n], outs[names[0]])]}
        return rec

    def workload(e, graphs, G, tw, variants, decode_variants=None, align=True):
        B, T, C = e.shape
        gv, _keep = capi.make_view(G["flags"], G["src"], G["dst"], G["olabel"], G["olabel"])
        views = [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
        arr = (capi.GraphView * B)(*[v for v, _ in views])
        n_arcs = sum(len(g["src"]) for g in graphs)
        bufs = dict(e=ctx.to_device(e), g=ctx.alloc(e.nbytes), ag=ctx.alloc(4 * max(n_arcs, 4)), tw=ctx.to_device(tw),
                    tg=ctx.alloc(tw.nbytes), p=ctx.alloc(4 * B * T), a=ctx.alloc(4 * B * T), s=ctx.alloc(4 * B))
        losses = np.zeros(B, np.float32)

        def loss():
            ctx._check(L.gtnb_backoff_transitions_loss(
                ctx.h, B, T, C, bufs["e"].ptr, 1, None, arr, None, 1, Ct.byref(gv), bufs["tw"].ptr, 1,
                losses.ctypes.data_as(capi._f32p), bufs["g"].ptr, 1, bufs["ag"].ptr, 1, bufs["tg"].ptr, 1))

        def decode():
            ctx._check(L.gtnb_viterbi_backoff(ctx.h, B, T, C, bufs["e"].ptr, 1, None, Ct.byref(gv), bufs["tw"].ptr, 1,
                                              bufs["p"].ptr, bufs["a"].ptr, bufs["s"].ptr, 1))

        def align_():
            ctx._check(L.gtnb_backoff_transitions_viterbi(ctx.h, B, T, C, bufs["e"].ptr, 1, None, arr, None, 1,
                                                          Ct.byref(gv), bufs["tw"].ptr, 1, bufs["p"].ptr,
                                                          bufs["a"].ptr, bufs["s"].ptr, 1))

        def loss_out():
            return (losses.copy(), bufs["g"].download(e.shape), bufs["tg"].download(tw.shape))

        def path_out():
            return (bufs["p"].download((B, T), np.int32), bufs["s"].download((B,)), bufs["a"].download((B, T), np.int32))

        f, _ = bo.closure_levels(G) if len(G["flags"]) < 3000 else (None, None)
        rec = {"shape": {"B": B, "T": T, "C": C},
               "G": {"states": len(G["flags"]), "emitting_arcs": int((G["olabel"] >= 0).sum()),
                     "epsilon_arcs": int((G["olabel"] == -1).sum())},
               "outputs": {"loss": ["losses", "emission gradient", "transition gradient"],
                           "decode": ["paths", "scores", "arcs"]},
               "loss": compare(variants, loss, loss_out),
               "decode": compare(decode_variants or variants, decode, path_out)}
        if f is not None:
            rec["G"]["levels"] = int(f.max())
        if align:
            rec["align"] = compare(variants, align_, path_out)
        for b in bufs.values():
            b.free()
        return rec

    B, T, C, U = 128, 500, 64, 50
    e, targets = util.bench_inputs(B, T, C, U)
    graphs = [go.ctc_graph(t, blank=0) for t in targets]
    out = {"rounds": args.rounds, "warmup": 1, "l2": "flushed before every timed call",
           "buffers": "emissions, transitions, gradients, paths, arcs and scores on the device; graphs as host views",
           "shape": {"B": B, "T": T, "C": C, "U": U}}
    lms = {"fourgram_c64": bo.backoff_ngram(np.random.default_rng(1), C, 4, n_tokens=60000),
           "fivegram_c64": bo.backoff_ngram(np.random.default_rng(1), C, 5, n_tokens=150000, min_count=5)}
    cl = {"cluster": {"sparse_cluster": 1}}
    for name, (G, tw) in lms.items():
        rec = workload(e, graphs, G, tw, cl, {"cluster_exact_ties_on": {"sparse_cluster": 1},
                                              "cluster_exact_ties_off": {"sparse_cluster": 1, "exact_ties": 0}})
        rec["small"] = workload(np.ascontiguousarray(e[:args.b_small, :args.t_small]), graphs[:args.b_small], G, tw,
                                {"cluster": {"sparse_cluster": 1}, "materialised": {"implicit": 0}})
        out[name] = rec
        print(name, json.dumps(rec), file=sys.stderr, flush=True)
    G, tw = bo.backoff_lm(np.random.default_rng(64), C)
    sizes = {"one_cta": {"sparse_cluster": 0}, "cluster_2": {"sparse_cluster": 2}, "cluster_4": {"sparse_cluster": 4},
             "cluster_8": {"sparse_cluster": 8}}
    out["pruned_trigram"] = workload(e, graphs, G, tw, sizes, {k: dict(v, exact_ties=0) for k, v in sizes.items()},
                                     align=False)
    print("pruned_trigram", json.dumps(out["pruned_trigram"]), file=sys.stderr, flush=True)
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
