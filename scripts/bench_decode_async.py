"""The asynchronous decoders against the synchronous ones on the same inputs, one JSON record on stdout (and in --out):

  sparse_trigram30   gtnb_viterbi_transitions_async vs gtnb_viterbi_sparse, the trigram at C = 30, B=128 T=200
  sparse_lm2000      the same with the 2000-state token LM at C = 64, B=128 T=500, on the inputs of
                     scripts/bench_sparse_viterbi.py, where an utterance ties: the synchronous call with "exact_ties" on
                     re-runs it on the host; also timed with it off
  backoff_trigram64  vs gtnb_viterbi_backoff, the pruned backoff trigram at C = 64, B=128 T=500
  cluster_trigram64  the full trigram at C = 64 on a thread-block cluster ("sparse_cluster" 1), B=128 T=500
  dense_asg / dense_bigram  gtnb_viterbi_dense_async vs gtnb_viterbi_dense_typed, B=512 T=2000 C=128

Per case: ms until the results are on the device (CUDA events on the call's stream, L2 flushed before every call,
the two calls alternating, median of --rounds rounds of --steps calls), the host's wall time per call, and the
kernels' time (CUDA events per launch).  Then a validation step (decode + collapse) captured in a CUDA graph against
the same step run eagerly through the synchronous torch decoder: device time and host time per step.  The card and its
power limit are read in the same run.

    python scripts/bench_decode_async.py [--rounds 5] [--steps 3] [--out F]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import bench_sparse_transitions as bst  # noqa: E402  (the 2000-state token LM)
from gtn_b200 import capi  # noqa: E402
from gtn_b200 import torch_loss as tl  # noqa: E402
from tests import backoff_oracle as bo  # noqa: E402
from tests import sparse_trans_oracle as st  # noqa: E402
from tests import util  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    ctx = capi.Ctx(0)
    L = capi.lib()
    stream = L.gtnb_ctx_stream(ctx.h)

    def timed(call):
        """-> (device ms, host wall ms) of one call, L2 flushed before it"""
        ctx.flush_l2()
        ctx.synchronize()
        ctx.timer_start()
        t0 = time.perf_counter()
        call()
        wall = (time.perf_counter() - t0) * 1e3
        return ctx.timer_stop(), wall

    def rounds(calls):
        """{name: call} alternating -> {name: {ms, wall_ms}} medians over rounds of the per-round means"""
        for c in calls.values():
            c()
        ctx.synchronize()
        acc = {k: ([], []) for k in calls}
        for _ in range(args.rounds):
            for k, c in calls.items():
                t = [timed(c) for _ in range(args.steps)]
                acc[k][0].append(float(np.mean([x[0] for x in t])))
                acc[k][1].append(float(np.mean([x[1] for x in t])))
        return {k: {"ms_median": float(np.median(v[0])), "ms_rounds": v[0], "host_wall_ms_median": float(np.median(v[1]))}
                for k, v in acc.items()}

    def kernels(call):
        ctx.profile(True)
        ctx.profile_read()
        for _ in range(args.steps):
            call()
        ctx.synchronize()
        k = {n: ms / args.steps for n, (cnt, ms) in ctx.profile_read().items()}
        ctx.profile(False)
        return k

    out = {"card": card(), "rounds": args.rounds, "steps": args.steps, "l2": "flushed before every timed call",
           "buffers": "every buffer on the device; the synchronous calls take host lengths", "cases": {}}

    def transitions_case(name, G, e_np, w_np, backoff=False, cluster=0, tie_off=False):
        B, T, C_ = e_np.shape
        e = torch.as_tensor(e_np).cuda()
        w = torch.as_tensor(w_np).cuda()
        lens_h = np.full(B, T, np.int32)
        lens = torch.as_tensor(lens_h).cuda()
        view, keep = capi.make_view(G["flags"], G["src"], G["dst"], G["olabel"], G["olabel"])
        ctx.set_flag("sparse_cluster", cluster)
        h = C.c_void_p()
        ctx._check(L.gtnb_transitions_create(ctx.h, C.byref(view), C_, int(backoff), C.byref(h)))
        n = C.c_size_t()
        ctx._check(L.gtnb_viterbi_transitions_async_workspace(ctx.h, h, B, T, C.byref(n)))
        ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
        p, a = (torch.empty((B, T), dtype=torch.int32, device="cuda") for _ in range(2))
        s = torch.empty(B, device="cuda")
        status = torch.empty(B, dtype=torch.int32, device="cuda")
        ps, as_ = (torch.empty((B, T), dtype=torch.int32, device="cuda") for _ in range(2))
        ss = torch.empty(B, device="cuda")
        sync_fn = L.gtnb_viterbi_backoff if backoff else L.gtnb_viterbi_sparse

        def asyn():
            ctx._check(L.gtnb_viterbi_transitions_async(
                ctx.h, stream, h, B, T, e.data_ptr(), lens.data_ptr(), w.data_ptr(), p.data_ptr(), a.data_ptr(),
                s.data_ptr(), status.data_ptr(), ws.data_ptr(), n.value))

        def sync():
            ctx._check(sync_fn(ctx.h, B, T, C_, e.data_ptr(), 1, lens_h.ctypes.data_as(capi._i32p), C.byref(view),
                               w.data_ptr(), 1, ps.data_ptr(), as_.data_ptr(), ss.data_ptr(), 1))

        def sync_ties_off():
            ctx.set_flag("exact_ties", 0)
            try:
                sync()
            finally:
                ctx.set_flag("exact_ties", 1)
        calls = {"async": asyn, "sync": sync}
        if tie_off:
            calls["sync_exact_ties_off"] = sync_ties_off
        rec = {"B": B, "T": T, "C": C_, "states": len(G["flags"]), "arcs": len(G["src"]), "sparse_cluster": cluster,
               "workspace_bytes": n.value}
        rec.update(rounds(calls))
        rec["async"]["kernels_ms"] = kernels(asyn)
        rec["sync"]["kernels_ms"] = kernels(sync)
        asyn()
        sync()
        ctx.synchronize()
        stv = status.cpu().numpy()
        rec["status_counts"] = {str(k): int((stv == k).sum()) for k in np.unique(stv)}
        ok = torch.as_tensor(stv == 0).cuda()
        rec["status0_equal_to_sync"] = bool(torch.equal(p[ok], ps[ok]) and torch.equal(s[ok], ss[ok]) and
                                            torch.equal(a[ok], as_[ok]))
        L.gtnb_transitions_destroy(ctx.h, h)
        ctx.set_flag("sparse_cluster", 0)
        out["cases"][name] = rec
        print(name, json.dumps({k: rec[k] for k in rec if k.startswith(("async", "sync"))}), file=sys.stderr)

    # the inputs and weights of scripts/bench_sparse_viterbi.py, drawn in its order (the LM's inputs hold a tie)
    rng = np.random.default_rng(5)
    for name, e_np, _, G, _, _ in bst.workloads():
        tw = rng.uniform(-1, 1, len(G["src"])).astype(np.float32)
        if name == "trigram_ctc":
            transitions_case("sparse_trigram30", G, e_np, tw)
        elif name == "sparse_lm":
            transitions_case("sparse_lm2000", G, e_np, tw, tie_off=True)
        elif name == "trigram_c64":
            transitions_case("cluster_trigram64", G, e_np, tw, cluster=1)
            e64 = e_np
    # the pruned backoff trigram of scripts/bench_backoff.py with its own weights
    G, tw = bo.backoff_lm(np.random.default_rng(3), 64)
    transitions_case("backoff_trigram64", G, e64, tw, backoff=True)

    for kind, name in ((capi.DENSE_ASG, "dense_asg"), (capi.DENSE_BIGRAM, "dense_bigram")):
        B, T, C_ = 512, 2000, 128
        g = torch.Generator().manual_seed(0)
        e = torch.log_softmax(torch.empty(B, T, C_).normal_(0, 3, generator=g), -1).cuda()
        w = torch.empty(C_ * C_ + (C_ if kind == capi.DENSE_ASG else 0)).normal_(0, 1, generator=g).cuda()
        lens_h = np.full(B, T, np.int32)
        lens = torch.as_tensor(lens_h).cuda()
        n = C.c_size_t()
        ctx._check(L.gtnb_viterbi_dense_async_workspace(ctx.h, B, T, C_, capi.F32, kind, C.byref(n)))
        ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
        p, ps = (torch.empty((B, T), dtype=torch.int32, device="cuda") for _ in range(2))
        s, ss = (torch.empty(B, device="cuda") for _ in range(2))
        status = torch.empty(B, dtype=torch.int32, device="cuda")

        def asyn():
            ctx._check(L.gtnb_viterbi_dense_async(ctx.h, stream, B, T, C_, e.data_ptr(), capi.F32, lens.data_ptr(),
                                                  kind, w.data_ptr(), p.data_ptr(), s.data_ptr(), status.data_ptr(),
                                                  ws.data_ptr(), n.value))

        def sync():
            ctx._check(L.gtnb_viterbi_dense_typed(ctx.h, B, T, C_, e.data_ptr(), capi.F32,
                                                  lens_h.ctypes.data_as(capi._i32p), kind, w.data_ptr(),
                                                  ps.data_ptr(), ss.data_ptr()))
            ctx.synchronize()  # (the device-buffer call returns once enqueued; the lengths went up through staging)
        rec = {"B": B, "T": T, "C": C_}
        rec.update(rounds({"async": asyn, "sync": sync}))
        rec["async"]["kernels_ms"] = kernels(asyn)
        asyn()
        sync()
        rec["equal_to_sync"] = bool(torch.equal(p, ps) and torch.equal(s, ss))
        out["cases"][name] = rec
        print(name, json.dumps({k: rec[k] for k in ("async", "sync")}), file=sys.stderr)

    # a validation step: decode + collapse, captured against eager with the synchronous torch decoder
    from gtn_b200 import gtn
    G = st.trigram_graph(30)
    gg = gtn.Graph()
    for f in G["flags"]:
        gg.add_node(bool(f & 1), bool(f & 2))
    for k in range(len(G["src"])):
        gg.add_arc(int(G["src"][k]), int(G["dst"][k]), int(G["olabel"][k]), int(G["olabel"][k]), 0.0)
    B, T, C_ = 128, 200, 30
    e_np, _ = util.bench_inputs(B, T, C_, 10)
    se = torch.as_tensor(e_np).cuda()
    sil = torch.as_tensor(np.random.default_rng(2).integers(T // 2, T + 1, B).astype(np.int32)).cuda()
    w = torch.as_tensor(np.random.default_rng(3).uniform(-2, 0, len(G["src"])).astype(np.float32)).cuda()
    tg = tl.TransitionGraph(gg, C_)
    tl.transitions_decode(se, w, tg, sil)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph):
            cp = tl.transitions_decode(se, w, tg, sil)
            cl = tl.collapse(cp[0], 0)
    torch.cuda.current_stream().wait_stream(side)

    def step_eager():
        p_, s_, a_ = tl.sparse_viterbi(se, w, gg, sil)
        return tl.collapse(p_, 0)

    def measure(step):
        for _ in range(2):
            step()
        torch.cuda.synchronize()
        dev, host = [], []
        for _ in range(args.rounds):
            a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a0.record()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                step()
            host.append((time.perf_counter() - t0) * 1e3 / args.steps)
            a1.record()
            torch.cuda.synchronize()
            dev.append(a0.elapsed_time(a1) / args.steps)
        return {"ms_per_step_median": float(np.median(dev)), "host_ms_per_step_median": float(np.median(host))}
    out["validation_step"] = {"workload": "sparse_trigram30 decode + collapse, B=128 T=200",
                              "captured": measure(graph.replay), "eager_sync_decoder": measure(step_eager)}
    print("validation_step", json.dumps(out["validation_step"]), file=sys.stderr)
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
