"""CTC loss + gradient with 16-bit emissions (gtnb_ctc_loss_ex) against float32 (gtnb_ctc_loss), at the flagship shape
B=256 T=1000 U=100 for C = 64 and 128, on device buffers.  The settings alternate step by step in one run, with the L2
flushed before every timed step.  One JSON record on stdout, nothing written:

  capi.<C>.<f32|bf16|f16>   ms per call (CUDA events around the call) and the bidir_ctc kernel's own time (the
                            context's launch profile), mean and median over the steps
  torch.<C>.<upcast|native> the step a training user runs on bf16 logits: ctc_loss(logits.float()) + backward, against
                            ctc_loss(logits) + backward (the gradient reaching the bf16 leaf either way), ms per step
  card, power_limit_w       read in the same run

    python scripts/bench_ctc_half.py [--steps 30] [--warmup 5] [--B 256 --T 1000 --U 100] [--C 64 128]
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
from gtn_b200.torch_loss import ctc_loss  # noqa: E402


def stats(xs):
    return {"mean": float(np.mean(xs)), "median": float(np.median(xs)), "min": float(np.min(xs)), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--B", type=int, default=256)
    ap.add_argument("--T", type=int, default=1000)
    ap.add_argument("--U", type=int, default=100)
    ap.add_argument("--C", type=int, nargs="+", default=[64, 128])
    args = ap.parse_args()
    B, T, U = args.B, args.T, args.U
    L = capi.lib()
    ctx = capi.Ctx(0)
    i32p, f32p = capi._i32p, capi._f32p
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")  # 256 MB: more than the 50 MB L2
    out = {"shape": {"B": B, "T": T, "U": U}, "steps": args.steps, "warmup": args.warmup,
           "l2": "flushed before every timed step", "order": "settings alternate step by step", "capi": {}, "torch": {}}
    for C in args.C:
        rng = np.random.default_rng(1234)
        e = rng.uniform(-5.0, 5.0, (B, T, C)).astype(np.float32)
        tg = [rng.integers(1, C, U).astype(np.int32) for _ in range(B)]
        cat, lens = capi._cat_targets(tg)
        losses = np.zeros(B, np.float32)
        e32 = torch.from_numpy(e).cuda()
        bufs = {"f32": (e32, torch.empty_like(e32))}
        for name, dt in (("bf16", torch.bfloat16), ("f16", torch.float16)):
            eh = e32.to(dt)
            bufs[name] = (eh, torch.empty_like(eh))
        torch.cuda.synchronize()

        def call(name):
            em, gr = bufs[name]
            if name == "f32":
                ctx._check(L.gtnb_ctc_loss(ctx.h, B, T, C, em.data_ptr(), 1, None, cat.ctypes.data_as(i32p),
                                           lens.ctypes.data_as(i32p), 0, losses.ctypes.data_as(f32p), gr.data_ptr(), 1))
            else:
                ctx._check(L.gtnb_ctc_loss_ex(ctx.h, B, T, C, em.data_ptr(), capi.BF16 if name == "bf16" else capi.F16,
                                              None, cat.ctypes.data_as(i32p), lens.ctypes.data_as(i32p), 0,
                                              losses.ctypes.data_as(f32p), gr.data_ptr()))

        names = ["f32", "bf16", "f16"]
        for _ in range(args.warmup):
            for n in names:
                call(n)
        ctx.profile(True)
        ctx.profile_read()
        ms = {n: [] for n in names}
        kern = {n: [] for n in names}
        for _ in range(args.steps):
            for n in names:
                ctx.flush_l2()
                ctx.profile_read()
                ctx.timer_start()
                call(n)
                ms[n].append(ctx.timer_stop())
                kern[n].append(ctx.profile_read().get("bidir_ctc", (0, float("nan")))[1])
        ctx.profile(False)
        out["capi"][str(C)] = {n: {"ms_per_call": stats(ms[n]), "bidir_ctc_kernel_ms": stats(kern[n])} for n in names}
        # losses of the three calls on the same (bf16-representable) emissions: == by contract
        call("bf16")
        lb = losses.copy()
        bufs["f32"] = (bufs["bf16"][0].float(), bufs["f32"][1])
        call("f32")
        out["capi"][str(C)]["bf16_losses_equal_f32_on_widened"] = bool(np.array_equal(lb, losses))
        bufs["f32"] = (e32, bufs["f32"][1])

        # the torch step on bf16 logits
        leaf = e32.to(torch.bfloat16).requires_grad_(True)
        steps = {"upcast": lambda: ctc_loss(leaf.float(), tg).backward(), "native": lambda: ctc_loss(leaf, tg).backward()}
        for _ in range(args.warmup):
            for f in steps.values():
                leaf.grad = None
                f()
        tms = {k: [] for k in steps}
        for _ in range(args.steps):
            for k, f in steps.items():
                leaf.grad = None
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                f()
                b.record()
                b.synchronize()
                tms[k].append(a.elapsed_time(b))
        out["torch"][str(C)] = {k: {"ms_per_step": stats(v)} for k, v in tms.items()}
        out["torch"][str(C)]["what"] = ("bf16 leaf [B, T, C]; upcast: ctc_loss(leaf.float(), targets).backward(); "
                                        "native: ctc_loss(leaf, targets).backward(); reduction mean")
        del bufs, e32, leaf
        torch.cuda.empty_cache()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    card, plim = [x.strip() for x in (q.split(",") + ["", ""])[:2]]
    out["card"], out["power_limit_w"] = card, plim
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
