"""CTC with a learned bigram transition graph (gtnb_ngram_ctc_loss, benchmarks/ctc.cpp:107-134) at BASELINE.json
configs[2]'s shape, B=128 T=500 C=64 U=50, next to the ASG criterion (gtnb_asg_loss, and gtnb_asg_loss_ex with the
transitions on the device) at the same shape, on the same emissions and the same C x C transition matrix, in one
run.  One JSON record on stdout, nothing written:

  ngram.value / asg.value   device-resident buffers, utterances / s (CUDA events, L2 flushed between steps)
  asg_ex.full / .ragged     gtnb_asg_loss_ex, every buffer on the device, with input_lens = T and with input_lens
                            drawn uniformly from [U, T] (seed 5)
  ngram.e2e                 every buffer on the host (pinned emissions and gradients)
  *.kernels_ms_per_step     per-kernel CUDA-event times
  ngram.trellis             the dense-trellis kernels against the bound they hit: 2 B T C^2 MUFU ex2 per step
                            (forward and backward; the pair posterior reuses the backward's), 16 per clock per SM
  ngram.parity, cpu_baseline  the reference (oracle/_ref, graph by graph through its own Graph API,
                            tests/ngram_oracle.py) on the first utterances of the timed batch
  card, power_limit_w       read in the same run

    python scripts/bench_ngram.py [--steps 20] [--warmup 3] [--B 128 --T 500 --C 64 --U 50] [--cpu-sample 4]
"""
import argparse
import ctypes as Ct
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gtn_b200 import capi  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--B", type=int, default=128)
    ap.add_argument("--T", type=int, default=500)
    ap.add_argument("--C", type=int, default=64)
    ap.add_argument("--U", type=int, default=50)
    ap.add_argument("--cpu-sample", type=int, default=4)
    args = ap.parse_args()
    B, T, C, U = args.B, args.T, args.C, args.U

    # ASG's inputs (bench.py --workload asg): transitions U(-5, 5) from seed 7, emissions U(-5, 5) from seed
    # 4321 + b; targets in [1, C-1], blank 0 is not a label
    tw = np.random.default_rng(7).uniform(-5, 5, C + C * C).astype(np.float32)
    W = np.ascontiguousarray(tw[C:])  # row = destination label
    e = np.empty((B, T, C), np.float32)
    tg = []
    for b in range(B):
        rng = np.random.default_rng(4321 + b)
        e[b] = rng.uniform(-5.0, 5.0, (T, C)).astype(np.float32)
        tg.append(rng.integers(1, C, U).astype(np.int32))
    cat = np.ascontiguousarray(np.concatenate(tg), np.int32)
    lens = np.full(B, U, np.int32)

    L = capi.lib()
    ctx = capi.Ctx(0)
    i32p, f32p = capi._i32p, capi._f32p
    e_dev, g_dev = ctx.to_device(e), ctx.alloc(e.nbytes)
    w_dev, wg_dev = ctx.to_device(W), ctx.alloc(W.nbytes)
    tw_dev, twg_dev = ctx.to_device(tw), ctx.alloc(tw.nbytes)
    full_lens = np.full(B, T, np.int32)
    ragged_lens = np.random.default_rng(5).integers(U, T + 1, B).astype(np.int32)
    hp_e, hp_g = Ct.c_void_p(), Ct.c_void_p()
    ctx._check(L.gtnb_host_alloc(ctx.h, e.nbytes, Ct.byref(hp_e)))
    ctx._check(L.gtnb_host_alloc(ctx.h, e.nbytes, Ct.byref(hp_g)))
    Ct.memmove(hp_e.value, e.ctypes.data, e.nbytes)
    losses = np.zeros(B, np.float32)
    wgrad = np.zeros(C * C, np.float32)
    tgrad = np.zeros(C + C * C, np.float32)

    def ngram(dev):
        # device: W and its gradient in HBM (the torch path); host: every buffer on the host
        ctx._check(L.gtnb_ngram_ctc_loss(
            ctx.h, B, T, C, e_dev.ptr if dev else hp_e.value, int(dev), None, w_dev.ptr if dev else W.ctypes.data,
            int(dev), cat.ctypes.data_as(i32p), lens.ctypes.data_as(i32p), 0, losses.ctypes.data_as(f32p),
            g_dev.ptr if dev else hp_g.value, int(dev), wg_dev.ptr if dev else wgrad.ctypes.data, int(dev)))

    def asg():
        ctx._check(L.gtnb_asg_loss(ctx.h, B, T, C, e_dev.ptr, 1, tw.ctypes.data_as(f32p), cat.ctypes.data_as(i32p),
                                   lens.ctypes.data_as(i32p), losses.ctypes.data_as(f32p), g_dev.ptr, 1,
                                   tgrad.ctypes.data_as(f32p)))

    def asg_ex(in_lens):
        # the transitions and their gradient in HBM (the torch path with input_lengths)
        ctx._check(L.gtnb_asg_loss_ex(ctx.h, B, T, C, e_dev.ptr, 1, in_lens.ctypes.data_as(i32p), tw_dev.ptr, 1,
                                      cat.ctypes.data_as(i32p), lens.ctypes.data_as(i32p), losses.ctypes.data_as(f32p),
                                      g_dev.ptr, 1, twg_dev.ptr, 1))

    def region(step, profile):
        for _ in range(args.warmup):
            step()
        if profile:
            ctx.profile(True)
            ctx.profile_read()
        ts, pr = [], {}
        for _ in range(args.steps):
            ctx.flush_l2()
            ctx.timer_start()
            step()
            ts.append(ctx.timer_stop())
            if profile:
                for k, (cnt, ms_) in ctx.profile_read().items():
                    c0, m0 = pr.get(k, (0, 0.0))
                    pr[k] = (c0 + cnt, m0 + ms_)
        if profile:
            ctx.profile(False)
        return float(np.mean(ts)), float(np.median(ts)), {k: v[1] / args.steps for k, v in pr.items() if k != "flush_l2"}

    ms, med, kern = region(lambda: ngram(True), True)
    gpu_losses, gpu_grads = losses.copy(), g_dev.download((B, T, C))
    ems, _, _ = region(lambda: ngram(False), False)
    ams, amed, akern = region(asg, True)
    asg_losses = losses.copy()
    xms, xmed, xkern = region(lambda: asg_ex(full_lens), True)
    ex_losses = losses.copy()
    rms, rmed, rkern = region(lambda: asg_ex(ragged_lens), True)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True).stdout.strip()
    card, plim, mhz = [x.strip() for x in (q.split(",") + ["", "", ""])[:3]]
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tms = kern.get("ngram_den_forward", 0.0) + kern.get("ngram_den_backward", 0.0)
    ops = 2.0 * B * T * C * C
    peak = sms * 16 * float(mhz) * 1e6 if mhz else None
    ach = ops / (tms * 1e-3) if tms else None
    out = {
        "card": card, "power_limit_w": plim, "shape": {"B": B, "T": T, "C": C, "U": U}, "steps": args.steps,
        "warmup": args.warmup, "l2": "flushed between timed steps",
        "ngram": {"value": B / (ms * 1e-3), "unit": "utt/s", "ms_per_step": ms, "ms_per_step_median": med,
                  "e2e": {"value": B / (ems * 1e-3), "unit": "utt/s", "ms_per_step": ems},
                  "kernels_ms_per_step": kern,
                  "trellis": {"kernels": "ngram_den_forward + ngram_den_backward", "ms_per_step": tms, "sfu_ops": ops,
                              "achieved_sfu_ops_per_s": ach, "sfu_peak_per_s": peak, "sm_clock_max_mhz": mhz,
                              "frac": (ach / peak) if (ach and peak) else None}},
        "asg": {"value": B / (ams * 1e-3), "unit": "utt/s", "ms_per_step": ams, "ms_per_step_median": amed,
                "kernels_ms_per_step": akern,
                "note": "implicit_* are k_implicit.cu's wide-path kernels on the dense C x C denominator plus the "
                        "forced-alignment numerator's sweeps"},
        "asg_ex": {"full": {"value": B / (xms * 1e-3), "unit": "utt/s", "ms_per_step": xms, "ms_per_step_median": xmed,
                            "kernels_ms_per_step": xkern, "input_lens": "T for every utterance",
                            "max_rel_loss_vs_asg": float(np.max(np.abs(ex_losses - asg_losses) / np.abs(asg_losses)))},
                   "ragged": {"value": B / (rms * 1e-3), "unit": "utt/s", "ms_per_step": rms,
                              "ms_per_step_median": rmed, "kernels_ms_per_step": rkern,
                              "input_lens": "uniform in [U, T], seed 5, mean %.1f" % float(ragged_lens.mean())},
                   "note": "asg_den_* are k_ngram.cu's trellis kernels in start mode, implicit_* the numerator's "
                           "sweeps on the second stream"}}
    from oracle import pyoracle as po
    if args.cpu_sample > 0 and po.have_ref():
        from tests import ngram_oracle as no
        n = min(args.cpu_sample, B)
        t0 = time.perf_counter()
        lr, gr, _ = no.ref_ngram_ctc_batch(e[:n], W, tg[:n])
        sec = time.perf_counter() - t0
        out["ngram"]["parity"] = {"n": n, "max_rel_loss": float((np.abs(gpu_losses[:n] - lr) / np.abs(lr)).max()),
                                  "max_abs_grad": float(np.abs(gpu_grads[:n] - gr).max())}
        out["ngram"]["cpu_baseline"] = {"value": n / sec, "unit": "utt/s", "seconds": sec,
                                        "kind": "reference, %d utterances one after the other on one thread" % n}
    print(json.dumps(out))
    for buf in (e_dev, g_dev, w_dev, wg_dev, tw_dev, twg_dev):
        buf.free()
    ctx._check(L.gtnb_host_free(ctx.h, hp_e.value))
    ctx._check(L.gtnb_host_free(ctx.h, hp_g.value))
    ctx.close()


if __name__ == "__main__":
    main()
