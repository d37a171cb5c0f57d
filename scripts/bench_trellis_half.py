"""n-gram CTC and ASG loss + gradients and the dense Viterbi decoders with 16-bit emissions (gtnb_ngram_ctc_loss_typed,
gtnb_asg_loss_typed, gtnb_viterbi_dense_typed) against their float32 calls (gtnb_ngram_ctc_loss, gtnb_asg_loss_ex,
gtnb_viterbi_dense_ex), on device buffers.  The settings alternate step by step in one run, with the L2 flushed before
every timed step.  One JSON record on stdout, nothing written:

  loss.<ngram|asg>.<C>.<f32|bf16|f16>  B=128 T=500 U=50: ms per call (CUDA events around the call) and the time of the
                                       ngram_den_* / asg_den_* and implicit_* kernels (the context's launch profile)
  torch.<ngram|asg>.<upcast|native>    the step a training user runs on bf16 logits at C = 64: loss(logits.float()) +
                                       backward against loss(logits) + backward, ms per step
  viterbi.<asg|bigram>.<f32|bf16|f16>  B=512 T=2000 C=128: ms per call and the viterbi_dense kernel's time
  card, power_limit_w                  read in the same run

    python scripts/bench_trellis_half.py [--steps 30] [--warmup 5] [--C 64 128]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from gtn_b200 import capi  # noqa: E402
from gtn_b200.torch_loss import asg_loss, ngram_ctc_loss  # noqa: E402

NAMES = ["f32", "bf16", "f16"]
DT = {"bf16": (torch.bfloat16, capi.BF16), "f16": (torch.float16, capi.F16)}


def stats(xs):
    return {"mean": float(np.mean(xs)), "median": float(np.median(xs)), "min": float(np.min(xs)),
            "max": float(np.max(xs)), "n": len(xs)}


def alternate(ctx, calls, steps, warmup, kernels):
    """calls: {name: fn}; every step runs each once, L2 flushed before each -> {name: {ms_per_call, <kernel>_ms}}"""
    for _ in range(warmup):
        for f in calls.values():
            f()
    ctx.profile(True)
    ctx.profile_read()
    ms = {n: [] for n in calls}
    kern = {n: {k: [] for k in kernels} for n in calls}
    for _ in range(steps):
        for n, f in calls.items():
            ctx.flush_l2()
            ctx.profile_read()
            ctx.timer_start()
            f()
            ms[n].append(ctx.timer_stop())
            prof = ctx.profile_read()
            for k in kernels:
                kern[n][k].append(prof.get(k, (0, float("nan")))[1])
    ctx.profile(False)
    return {n: dict({"ms_per_call": stats(ms[n])}, **{k + "_ms": stats(v) for k, v in kern[n].items()})
            for n in calls}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--C", type=int, nargs="+", default=[64, 128])
    args = ap.parse_args()
    L = capi.lib()
    ctx = capi.Ctx(0)
    i32p, f32p = capi._i32p, capi._f32p
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")  # 256 MB: more than the 50 MB L2
    out = {"l2": "flushed before every timed step", "order": "settings alternate step by step", "steps": args.steps,
           "warmup": args.warmup, "loss": {"ngram": {}, "asg": {}}, "torch": {}, "viterbi": {}}
    B, T, U = 128, 500, 50
    out["loss_shape"] = {"B": B, "T": T, "U": U}
    for kind in ("ngram", "asg"):
        for C in args.C:
            rng = np.random.default_rng(1234)
            e32 = torch.from_numpy(rng.uniform(-5.0, 5.0, (B, T, C)).astype(np.float32)).cuda()
            tg = [rng.integers(1, C, U).astype(np.int32) for _ in range(B)]
            cat, lens = capi._cat_targets(tg)
            nW = C * C if kind == "ngram" else C + C * C
            w = torch.from_numpy(rng.uniform(-1, 1, nW).astype(np.float32)).cuda()
            tgrad = torch.empty_like(w)
            losses = np.zeros(B, np.float32)
            bufs = {"f32": (e32, torch.empty_like(e32))}
            for n, (dt, _) in DT.items():
                bufs[n] = (e32.to(dt), torch.empty_like(e32, dtype=dt))
            torch.cuda.synchronize()

            def call(n, kind=kind, C=C, bufs=bufs, w=w, tgrad=tgrad, cat=cat, lens=lens, losses=losses):
                em, gr = bufs[n]
                t = (cat.ctypes.data_as(i32p), lens.ctypes.data_as(i32p))
                lp = losses.ctypes.data_as(f32p)
                if kind == "ngram" and n == "f32":
                    ctx._check(L.gtnb_ngram_ctc_loss(ctx.h, B, T, C, em.data_ptr(), 1, None, w.data_ptr(), 1, *t, 0, lp,
                                                     gr.data_ptr(), 1, tgrad.data_ptr(), 1))
                elif kind == "ngram":
                    ctx._check(L.gtnb_ngram_ctc_loss_typed(ctx.h, B, T, C, em.data_ptr(), DT[n][1], None, w.data_ptr(),
                                                           *t, 0, lp, gr.data_ptr(), tgrad.data_ptr()))
                elif n == "f32":
                    ctx._check(L.gtnb_asg_loss_ex(ctx.h, B, T, C, em.data_ptr(), 1, None, w.data_ptr(), 1, *t, lp,
                                                  gr.data_ptr(), 1, tgrad.data_ptr(), 1))
                else:
                    ctx._check(L.gtnb_asg_loss_typed(ctx.h, B, T, C, em.data_ptr(), DT[n][1], None, w.data_ptr(), *t,
                                                     lp, gr.data_ptr(), tgrad.data_ptr()))

            den = "ngram_den" if kind == "ngram" else "asg_den"
            kernels = [den + "_forward", den + "_backward", "implicit_forward", "implicit_backward", "narrow", "widen"]
            res = alternate(ctx, {n: (lambda n=n: call(n)) for n in NAMES}, args.steps, args.warmup, kernels)
            # the losses of bf16 and of float32 on the widened bf16 emissions: == by contract
            call("bf16")
            lb = losses.copy()
            bufs["f32"] = (bufs["bf16"][0].float(), bufs["f32"][1])
            call("f32")
            res["bf16_losses_equal_f32_on_widened"] = bool(np.array_equal(lb, losses))
            out["loss"][kind][str(C)] = res
            del bufs, e32
            torch.cuda.empty_cache()

    # the torch step on bf16 logits, C = 64
    C = 64
    rng = np.random.default_rng(99)
    e32 = torch.from_numpy(rng.uniform(-5.0, 5.0, (B, T, C)).astype(np.float32)).cuda()
    tg = [rng.integers(1, C, U).astype(np.int32) for _ in range(B)]
    for kind, fn, nW in (("ngram", ngram_ctc_loss, C * C), ("asg", asg_loss, C + C * C)):
        leaf = e32.to(torch.bfloat16).requires_grad_(True)
        w = torch.nn.Parameter(torch.from_numpy(rng.uniform(-1, 1, nW).astype(np.float32)).cuda())
        il = [T] * B  # asg_loss's device route for both dtypes
        steps = {"upcast": lambda fn=fn, leaf=leaf, w=w: fn(leaf.float(), w, tg, input_lengths=il).backward(),
                 "native": lambda fn=fn, leaf=leaf, w=w: fn(leaf, w, tg, input_lengths=il).backward()}
        for _ in range(args.warmup):
            for f in steps.values():
                leaf.grad = w.grad = None
                f()
        tms = {k: [] for k in steps}
        for _ in range(args.steps):
            for k, f in steps.items():
                leaf.grad = w.grad = None
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                f()
                b.record()
                b.synchronize()
                tms[k].append(a.elapsed_time(b))
        out["torch"][kind] = {k: {"ms_per_step": stats(v)} for k, v in tms.items()}
        out["torch"][kind]["what"] = ("bf16 leaf [B=%d, T=%d, C=%d], U=%d, learned float32 transitions; upcast: "
                                      "loss(leaf.float(), w, targets).backward(); native: loss(leaf, w, targets)"
                                      ".backward(); reduction mean" % (B, T, C, U))
    del e32
    torch.cuda.empty_cache()

    # Viterbi at B=512 T=2000 C=128
    B, T, C = 512, 2000, 128
    out["viterbi_shape"] = {"B": B, "T": T, "C": C}
    rng = np.random.default_rng(7)
    e32 = torch.from_numpy(rng.uniform(-5.0, 5.0, (B, T, C)).astype(np.float32)).cuda()
    ems = {"f32": e32, "bf16": e32.to(torch.bfloat16), "f16": e32.to(torch.float16)}
    paths = torch.empty((B, T), dtype=torch.int32, device="cuda")
    scores = torch.empty(B, dtype=torch.float32, device="cuda")
    for kname, kind in (("asg", capi.DENSE_ASG), ("bigram", capi.DENSE_BIGRAM)):
        w = torch.from_numpy(rng.uniform(-1, 1, C * C if kind == capi.DENSE_BIGRAM else C + C * C).astype(np.float32))
        w = w.cuda()

        def vcall(n, kind=kind, w=w):
            if n == "f32":
                ctx._check(L.gtnb_viterbi_dense_ex(ctx.h, B, T, C, ems[n].data_ptr(), 1, None, kind, w.data_ptr(), 1,
                                                   paths.data_ptr(), scores.data_ptr(), 1))
            else:
                ctx._check(L.gtnb_viterbi_dense_typed(ctx.h, B, T, C, ems[n].data_ptr(), DT[n][1], None, kind,
                                                      w.data_ptr(), paths.data_ptr(), scores.data_ptr()))

        kn = "viterbi_dense_bigram" if kind == capi.DENSE_BIGRAM else "viterbi_dense"
        out["viterbi"][kname] = alternate(ctx, {n: (lambda n=n: vcall(n)) for n in NAMES}, args.steps, args.warmup,
                                          [kn])
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    card, plim = [x.strip() for x in (q.split(",") + ["", ""])[:2]]
    out["card"], out["power_limit_w"] = card, plim
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
