"""The CTC loss without a host synchronisation (gtnb_ctc_loss_async, torch ctc_loss on tensor targets) against the
synchronous call (gtnb_ctc_loss_ex on list targets).  One JSON record on stdout, nothing written:

  capi.<name>     ms per call on device emissions, host clock from the call until its results are on the device and
                  the stream is idle: the synchronous call returns then; the asynchronous one is followed by a stream
                  synchronise.  Shapes: the flagship B=256 T=1000 U=100 at C = 64 and 128 (one launch) and C = 512,
                  B=128 T=500 U=50 (two sweeps).
  torch.<form>    a training step (an MLP whose forward takes milliseconds, then ctc_loss and backward) with list
                  targets, tensor targets eagerly, and tensor targets captured in a CUDA graph: wall ms per step over
                  a run of steps, and the host ms per step spent inside the loss call and backward (list targets:
                  blocked until the forward pass is done)
  card, power_limit_w   read in the same run

Settings alternate step by step; the L2 is flushed (256 MB memset) before every timed capi call.  Medians with the
10th and 90th percentiles.

    python scripts/bench_ctc_async.py [--steps 30] [--warmup 5]
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
from gtn_b200.torch_loss import ctc_loss  # noqa: E402


def stats(xs):
    return {"median": float(np.median(xs)), "p10": float(np.percentile(xs, 10)), "p90": float(np.percentile(xs, 90)),
            "n": len(xs)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    return q[0], float(q[1]) if len(q) > 1 else None


def capi_calls(ctx, B, T, Cn, U, steps, warmup, flush):
    L = capi.lib()
    rng = np.random.default_rng(1234)
    e = torch.from_numpy(rng.uniform(-5.0, 5.0, (B, T, Cn)).astype(np.float32)).cuda()
    tg = rng.integers(1, Cn, (B, U)).astype(np.int32)
    cat = np.ascontiguousarray(tg.ravel())
    lens = np.full(B, U, np.int32)
    losses_h = np.zeros(B, np.float32)
    grad = torch.empty_like(e)
    tg_d, lens_d = torch.from_numpy(tg).cuda(), torch.from_numpy(lens).cuda()
    losses_d = torch.empty(B, device="cuda")
    n = C.c_size_t()
    ctx._check(L.gtnb_ctc_loss_async_workspace(ctx.h, B, T, Cn, U, capi.F32, 1, C.byref(n)))
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def sync_call():
        ctx._check(L.gtnb_ctc_loss_ex(ctx.h, B, T, Cn, e.data_ptr(), capi.F32, None, cat.ctypes.data_as(capi._i32p),
                                      lens.ctypes.data_as(capi._i32p), 0, losses_h.ctypes.data_as(capi._f32p),
                                      grad.data_ptr()))

    def async_call():
        ctx._check(L.gtnb_ctc_loss_async(ctx.h, stream, B, T, Cn, U, e.data_ptr(), capi.F32, None, tg_d.data_ptr(),
                                         lens_d.data_ptr(), 0, losses_d.data_ptr(), None, grad.data_ptr(),
                                         ws.data_ptr(), n.value))
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
    want = losses_h.copy()
    async_call()
    return {k: stats(v) for k, v in times.items()} | {
        "workspace_bytes": n.value, "losses_equal": bool((losses_d.cpu().numpy() == want).all())}


def torch_steps(steps, warmup, B=64, T=500, F=1024, H=4096, layers=4, Cn=64, U=50):
    torch.manual_seed(0)
    mods = []
    for i in range(layers):
        mods += [torch.nn.Linear(F if i == 0 else H, H), torch.nn.ReLU()]
    model = torch.nn.Sequential(*mods, torch.nn.Linear(H, Cn)).cuda()
    opt = torch.optim.SGD(model.parameters(), lr=1e-4)
    x = torch.randn(B, T, F, device="cuda")
    tg = torch.randint(1, Cn, (B, U), device="cuda", dtype=torch.int32)
    tl = torch.full((B,), U, device="cuda", dtype=torch.int32)
    tg_list = [r.numpy() for r in tg.cpu()]
    inside = [0.0]

    def step(tensor_targets):
        opt.zero_grad(set_to_none=False)
        logits = model(x)
        t0 = time.perf_counter()
        if tensor_targets:
            loss = ctc_loss(logits, tg, target_lengths=tl)
        else:
            loss = ctc_loss(logits, tg_list)
        loss.backward()
        inside[0] += time.perf_counter() - t0
        opt.step()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step(True)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step(True)

    def replay():
        t0 = time.perf_counter()
        graph.replay()
        inside[0] += time.perf_counter() - t0

    forms = {"list_targets": lambda: step(False), "tensor_eager": lambda: step(True), "tensor_graph": replay}
    run = 10
    res = {k: {"wall": [], "host_in_loss": []} for k in forms}
    for i in range(warmup + steps):
        for name, fn in forms.items():
            torch.cuda.synchronize()
            inside[0] = 0.0
            t0 = time.perf_counter()
            for _ in range(run):
                fn()
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3 / run
            if i >= warmup:
                res[name]["wall"].append(wall)
                res[name]["host_in_loss"].append(inside[0] * 1e3 / run)
    # the forward alone, for scale
    fw = []
    for _ in range(10):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            model(x)
        torch.cuda.synchronize()
        fw.append((time.perf_counter() - t0) * 1e3)
    out = {k: {m: stats(v) for m, v in d.items()} for k, d in res.items()}
    out["model"] = {"B": B, "T": T, "F": F, "hidden": H, "layers": layers, "C": Cn, "U": U,
                    "forward_ms": stats(fw), "steps_per_timing": run,
                    "host_in_loss": "graph form: host ms inside graph.replay() for the whole step"}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    name, power = card()
    ctx = capi.Ctx(0)
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    out = {"card": name, "power_limit_w": power, "steps": args.steps, "warmup": args.warmup,
           "l2": "flushed before every timed capi call", "order": "settings alternate step by step", "capi": {}}
    for B, T, Cn, U in ((256, 1000, 64, 100), (256, 1000, 128, 100), (128, 500, 512, 50)):
        out["capi"]["B%d_T%d_C%d_U%d" % (B, T, Cn, U)] = capi_calls(ctx, B, T, Cn, U, args.steps, args.warmup, flush)
    out["torch"] = torch_steps(max(5, args.steps // 3), 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
