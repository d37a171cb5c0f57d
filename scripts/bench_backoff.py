"""gtnb_backoff_transitions_loss and gtnb_viterbi_backoff on a pruned backoff trigram LM (tests/backoff_oracle.py's
backoff_lm: C = 64, 1 root + 64 bigram states + 2000 trigram states, 17 344 emitting arcs and 2064 epsilon arcs, two
levels) with CTC target graphs at B=128 T=500 U=50.  One JSON record on stdout (and in --out when given):

  backoff_trigram   the LM with its epsilon arcs: the loss (with every gradient) and the decode on the device route,
                    the whole batch; the same calls on the materialised route (set_flag("implicit", 0)) for the first
                    --b-large utterances, which compose E_b with G one utterance at a time
  eps_removed       the same LM with its epsilon arcs removed (every state gets the arcs of its backoff chain, weights
                    summed along the chain, parallel arcs kept; remove_epsilons): its arc count, the route gtnb_sparse_transitions_loss
                    takes for it (outside the device envelope of 32 768 arcs: the materialised route) and its time on
                    the first --b-large utterances

Per call: ms (L2 flushed before every call, median over --rounds, routes alternating), the kernels of the device route
(CUDA events per launch, in a profiled pass of its own), and the routes' outputs compared (losses within 1e-4
relative, decode scores and paths ==).  The card and its power limit are read in the same run.

    python scripts/bench_backoff.py [--rounds 5] [--warmup 1] [--b-large 4] [--out F]
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


def remove_epsilons(G, tw):
    """G without its epsilon arcs: state s gets, for every r in its epsilon closure (reached with weight W(s, r), the
    sum along the chain), r's emitting arcs s -> dst with weight W(s, r) + w, parallel arcs kept: the graph a user
    gets from removing the backoff arcs before the sparse entry points (the paths that end on epsilon moves after the
    last frame are gone, so its scores are not the backoff graph's)"""
    eps = {int(G["src"][k]): (int(G["dst"][k]), float(tw[k])) for k in np.flatnonzero(G["olabel"] == -1)}
    out = {}
    for k in np.flatnonzero(G["olabel"] >= 0):
        out.setdefault(int(G["src"][k]), []).append(k)
    src, dst, lab, w = [], [], [], []
    for s in range(len(G["flags"])):
        r, acc = s, 0.0
        while True:
            for k in out.get(r, []):
                src.append(s), dst.append(int(G["dst"][k])), lab.append(int(G["olabel"][k])), w.append(acc + tw[k])
            if r not in eps:
                break
            r, wr = eps[r]
            acc += wr
    return go.make(G["flags"], src, dst, lab), np.asarray(w, np.float32)


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

    def calls(e, graphs, G, tw, fn_loss, fn_dec):
        """(loss step, decode step, outputs) on device buffers"""
        B, T, C = e.shape
        gv = capi.make_view(G["flags"], G["src"], G["dst"], G["olabel"], G["olabel"], None)
        views = [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
        arr = (capi.GraphView * B)(*[v for v, _ in views])
        e_dev, w_dev = ctx.to_device(e), ctx.to_device(tw)
        g_dev, tg_dev, p_dev, a_dev, s_dev = (ctx.alloc(4 * B * T * C), ctx.alloc(4 * len(tw)), ctx.alloc(4 * B * T),
                                              ctx.alloc(4 * B * T), ctx.alloc(4 * B))
        losses = np.zeros(B, np.float32)
        keep = (gv, views, arr, e_dev, w_dev, g_dev, tg_dev, p_dev, a_dev, s_dev)

        def loss():
            ctx._check(getattr(L, fn_loss)(ctx.h, B, T, C, e_dev.ptr, 1, None, arr, None, 1, Ct.byref(gv[0]),
                                           w_dev.ptr, 1, losses.ctypes.data_as(capi._f32p), g_dev.ptr, 1, None, 1,
                                           tg_dev.ptr, 1))

        def dec():
            ctx._check(getattr(L, fn_dec)(ctx.h, B, T, C, e_dev.ptr, 1, None, Ct.byref(gv[0]), w_dev.ptr, 1,
                                          p_dev.ptr, a_dev.ptr, s_dev.ptr, 1))

        def outputs():
            return (losses.copy(), p_dev.download((B, T), np.int32), s_dev.download((B,)),
                    a_dev.download((B, T), np.int32))

        return loss, dec, outputs, keep

    def median_ms(step, implicit):
        for _ in range(args.warmup):
            on_route(implicit, step)
        return [on_route(implicit, lambda: timed(step)) for _ in range(args.rounds)]

    rng = np.random.default_rng(64)
    G, tw = bo.backoff_lm(rng, 64)
    B, T, C, U = 128, 500, 64, 50
    e, targets = util.bench_inputs(B, T, C, U)
    graphs = [go.ctc_graph(t, blank=0) for t in targets]
    out = {"rounds": args.rounds, "warmup": args.warmup, "l2": "flushed before every timed call",
           "buffers": "emissions, transitions, gradients and decode outputs on the device; graphs as host views",
           "shape": {"B": B, "T": T, "C": C, "U": U}}

    # the LM with its epsilon arcs: the device route on the whole batch
    loss, dec, outputs, keep = calls(e, graphs, G, tw, "gtnb_backoff_transitions_loss", "gtnb_viterbi_backoff")
    rec = {"G": {"states": len(G["flags"]), "emitting_arcs": int((G["olabel"] >= 0).sum()),
                 "epsilon_arcs": int((G["olabel"] == -1).sum()), "levels": int(bo.closure_levels(G)[0].max())}}
    for name, step in (("loss", loss), ("decode", dec)):
        ms = median_ms(step, 1)
        kern = kernels(step)
        rec[name] = {"device_ms_per_call_median": float(np.median(ms)), "device_ms_per_call_min": float(np.min(ms)),
                     "utt_per_s": B / (float(np.median(ms)) * 1e-3), "kernels_ms_per_call": kern,
                     "exact_route_ran": any(k.startswith("gcompose") for k in kern)}
    ctx.set_flag("exact_ties", 0)
    try:
        rec["decode"]["device_exact_ties_off_ms_median"] = float(np.median(median_ms(dec, 1)))
    finally:
        ctx.set_flag("exact_ties", 1)
    loss()
    dec()
    full = outputs()
    rec["decode"]["finite_scores"] = int(np.isfinite(full[2]).sum())
    # both routes on the first b_large utterances
    nb = args.b_large
    loss_s, dec_s, outputs_s, keep_s = calls(e[:nb], graphs[:nb], G, tw, "gtnb_backoff_transitions_loss",
                                             "gtnb_viterbi_backoff")
    for name, step in (("loss", loss_s), ("decode", dec_s)):
        dev, mat = [], []
        for _ in range(args.warmup):
            step()
            on_route(0, step)
        for _ in range(args.rounds):
            dev.append(timed(step))
            mat.append(on_route(0, lambda: timed(step)))
        rec[name]["first_%d" % nb] = {"device_ms_median": float(np.median(dev)),
                                      "materialised_ms_median": float(np.median(mat)),
                                      "device_speedup_vs_materialised": float(np.median(mat) / np.median(dev))}
    loss_s()
    dec_s()
    got_dev = outputs_s()
    on_route(0, loss_s)
    on_route(0, dec_s)
    got_mat = outputs_s()
    rec["routes_equal_first_%d" % nb] = {
        "losses_max_rel": float(np.max(np.abs(got_dev[0] - got_mat[0]) / np.maximum(np.abs(got_mat[0]), 1e-30))),
        "paths": bool(np.array_equal(got_dev[1], got_mat[1])), "scores": bool(np.array_equal(got_dev[2], got_mat[2])),
        "arcs": bool(np.array_equal(got_dev[3], got_mat[3]))}
    out["backoff_trigram"] = rec
    print("backoff_trigram", json.dumps(rec), file=sys.stderr, flush=True)

    # the same LM with its epsilon arcs removed, through gtnb_sparse_transitions_loss / gtnb_viterbi_sparse
    Gr, twr = remove_epsilons(G, tw)
    loss_r, dec_r, outputs_r, keep_r = calls(e[:nb], graphs[:nb], Gr, twr, "gtnb_sparse_transitions_loss",
                                             "gtnb_viterbi_sparse")
    kern = kernels(loss_r)
    rec = {"G": {"states": len(Gr["flags"]), "arcs": len(Gr["src"])},
           "route": "device" if "sparse_den_forward" in kern else "materialised"}
    for name, step in (("loss", loss_r), ("decode", dec_r)):
        rec[name] = {"first_%d_ms_median" % nb: float(np.median(median_ms(step, 1)))}
    out["eps_removed"] = rec
    print("eps_removed", json.dumps(rec), file=sys.stderr, flush=True)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    card, plim = [x.strip() for x in (q.split(",") + ["", ""])[:2]]
    out["card"], out["power_limit_w"] = card, plim
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(out, indent=1) + "\n")
    for k in (keep, keep_s, keep_r):
        for buf in k[3:]:
            buf.free()
    ctx.close()


if __name__ == "__main__":
    main()
