"""Forced alignment without a host synchronisation (gtnb_ctc_align_async, gtnb_ngram_ctc_align_async,
gtnb_asg_align_async) against the synchronous aligners on host-built numerators (gtnb_graph_viterbi on CTC graphs,
gtnb_graph_transitions_viterbi with BIGRAM on CTC graphs and with ASG on force-align chains).  One JSON record on
stdout, nothing written:

  <workload>.<call>   ms per call on device emissions with device outputs, host clock from the call until its results
                      are on the device and the stream is idle (the synchronous call returns then; the asynchronous one
                      is followed by a stream synchronise).  The two calls alternate, the L2 is flushed (256 MB memset)
                      before each; medians with the 10th and 90th percentiles.  equal: the two calls' scores ==, and
                      paths == on every utterance the asynchronous call gives status 0.
  <workload>.kernels  the asynchronous call's kernels (ms per launch) from a separate profiled pass (gtnb_profile_*,
                      CUDA events around each launch)
  card, power_limit_w read in the same run

    python scripts/bench_align_async.py [--steps 20] [--warmup 3]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from gtn_b200 import capi  # noqa: E402
from tests import align_async_oracle as ao  # noqa: E402

DT = {torch.float32: capi.F32, torch.bfloat16: capi.BF16}
NAMES = {ao.CTC: "ctc", ao.NGRAM: "ngram_ctc", ao.ASG: "asg"}
WORKLOADS = [  # (name, kind, B, T, C, U, dtype)
    ("ctc_configs1", ao.CTC, 256, 1000, 64, 100, torch.float32),
    ("ctc_configs1_bf16", ao.CTC, 256, 1000, 64, 100, torch.bfloat16),
    ("ngram_b128", ao.NGRAM, 128, 500, 64, 50, torch.float32),
    ("asg_b128", ao.ASG, 128, 500, 64, 50, torch.float32),
]


def stats(xs):
    return {"median": float(np.median(xs)), "p10": float(np.percentile(xs, 10)), "p90": float(np.percentile(xs, 90)),
            "n": len(xs)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    return q[0], float(q[1]) if len(q) > 1 else None


def workload(ctx, kind, B, T, Cn, U, dtype, steps, warmup, flush):
    L = capi.lib()
    rng = np.random.default_rng(1234)
    x = rng.normal(0, 3, (B, T, Cn)).astype(np.float32)
    x = x - np.log(np.exp(x).sum(-1, keepdims=True))  # log-softmax
    e = torch.from_numpy(x).to(dtype).cuda()
    ef = e.float().contiguous()  # the synchronous aligners take float32
    W = None
    if kind != ao.CTC:
        W = torch.from_numpy(rng.normal(0, 1, Cn * Cn + (Cn if kind == ao.ASG else 0)).astype(np.float32)).cuda()
    tg = rng.integers(1, Cn, (B, U)).astype(np.int32)
    lens = np.full(B, U, np.int32)
    graphs = [ao.numerator_graph(kind, tg[b], 0) for b in range(B)]
    views = [capi.make_view(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]) for g in graphs]
    arr, _, _ = capi._graph_batch(views, B, None)
    sp = torch.empty((B, T), dtype=torch.int32, device="cuda")
    sa = torch.empty((B, T), dtype=torch.int32, device="cuda")
    ss = torch.empty(B, device="cuda")
    tg_d, lens_d = torch.from_numpy(tg).cuda(), torch.from_numpy(lens).cuda()
    ap = torch.empty((B, T), dtype=torch.int32, device="cuda")
    at = torch.empty((B, T), dtype=torch.int32, device="cuda")
    ascore = torch.empty(B, device="cuda")
    ast = torch.empty(B, dtype=torch.int32, device="cuda")
    n = C.c_size_t()
    ctx._check(getattr(L, "gtnb_%s_align_async_workspace" % NAMES[kind])(ctx.h, B, T, Cn, U, DT[dtype], C.byref(n)))
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def sync_call():
        if kind == ao.CTC:
            rc = L.gtnb_graph_viterbi(ctx.h, B, T, Cn, ef.data_ptr(), 1, None, arr, None, 1, sp.data_ptr(),
                                      sa.data_ptr(), ss.data_ptr(), 1)
        else:
            k = capi.DENSE_ASG if kind == ao.ASG else capi.DENSE_BIGRAM
            rc = L.gtnb_graph_transitions_viterbi(ctx.h, B, T, Cn, ef.data_ptr(), 1, None, arr, None, 1, k,
                                                  W.data_ptr(), 1, sp.data_ptr(), sa.data_ptr(), ss.data_ptr(), 1)
        ctx._check(rc)

    def async_call():
        head = (ctx.h, stream, B, T, Cn, U, e.data_ptr(), DT[dtype], None)
        outs = (ap.data_ptr(), at.data_ptr(), ascore.data_ptr(), ast.data_ptr(), ws.data_ptr(), n.value)
        fn = getattr(L, "gtnb_%s_align_async" % NAMES[kind])
        if kind == ao.CTC:
            ctx._check(fn(*head, tg_d.data_ptr(), lens_d.data_ptr(), 0, *outs))
        elif kind == ao.NGRAM:
            ctx._check(fn(*head, W.data_ptr(), tg_d.data_ptr(), lens_d.data_ptr(), 0, *outs))
        else:
            ctx._check(fn(*head, W.data_ptr(), tg_d.data_ptr(), lens_d.data_ptr(), *outs))
        torch.cuda.current_stream().synchronize()

    times = {"sync": [], "async": []}
    for i in range(warmup + steps):
        for name, fn in (("sync", sync_call), ("async", async_call)):
            flush.zero_()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            dt = (time.perf_counter() - t0) * 1e3
            if i >= warmup:
                times[name].append(dt)
    sync_call()
    async_call()
    torch.cuda.synchronize()
    st = ast.cpu().numpy()
    ok = st == 0
    equal = bool((ascore.cpu() == ss.cpu()).all()) and bool((ap.cpu().numpy()[ok] == sp.cpu().numpy()[ok]).all())
    # the kernel split, in a pass of its own
    ctx.profile(True)
    ctx.profile_read()
    for _ in range(5):
        async_call()
    prof = ctx.profile_read()
    ctx.profile(False)
    kernels = {k: v[1] / v[0] for k, v in prof.items()}
    return {"sync_ms": stats(times["sync"]), "async_ms": stats(times["async"]), "equal": equal,
            "status3": int((st == 3).sum()), "workspace_bytes": n.value, "kernels_ms": kernels}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    name, plimit = card()
    ctx = capi.Ctx(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    out = {"card": name, "power_limit_w": plimit}
    for wname, kind, B, T, Cn, U, dtype in WORKLOADS:
        out[wname] = workload(ctx, kind, B, T, Cn, U, dtype, args.steps, args.warmup, flush)
        out[wname]["shape"] = {"B": B, "T": T, "C": Cn, "U": U, "dtype": str(dtype).replace("torch.", "")}
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
