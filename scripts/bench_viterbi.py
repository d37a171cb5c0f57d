"""Batched Viterbi decoding on the dense trellis (k_dense.cu), three entry points timed in one run, alternating
between them round by round on the same emissions:

  old      gtnb_viterbi_dense: emissions on the device, transitions [C + C*C] on the host (uploaded by every call),
           paths and scores copied back to the host
  asg_ex   gtnb_viterbi_dense_ex, kind GTNB_DENSE_ASG: the same transitions, emissions and outputs on the device
  bigram   gtnb_viterbi_dense_ex, kind GTNB_DENSE_BIGRAM: W = the transitions' C x C part, every buffer on the device

at BASELINE.json configs[3]'s shape (B=512 T=2000 C=128) and at n-gram CTC's shape (B=128 T=500 C=64).  With
--baseline-lib, the gtnb_viterbi_dense of another build of the library (e.g. the parent commit's) joins the
rotation as `old_baseline`, and its outputs are compared with this build's.  One JSON record on stdout, nothing
written:

  <shape>.<leg>.ms_per_step   per round: the mean over --steps calls (CUDA events around each call, L2 flushed
                              between calls); the record keeps every round, their median and their minimum
  <shape>.kernels_ms          per-kernel CUDA-event times of a separate profiled pass
  <shape>.equal               old vs asg_ex paths and scores (==), and old vs old_baseline
  card, power_limit_w         read in the same run

    python scripts/bench_viterbi.py [--steps 10] [--warmup 2] [--rounds 5] [--baseline-lib PATH]
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

SHAPES = {"config4_B512_T2000_C128": (512, 2000, 128), "ngram_B128_T500_C64": (128, 500, 64)}


class Lib:
    """A build of libgtn_b200.so and a context of it: its timer, L2 flush and gtnb_viterbi_dense.  path None: this
    build, on the context ctx."""

    def __init__(self, path=None, ctx=None):
        if path is None:
            self.L, self.h, self.own = capi.lib(), ctx.h, False
            return
        L = Ct.CDLL(path)
        vp = Ct.c_void_p
        L.gtnb_ctx_create.argtypes = [Ct.c_int, vp, Ct.POINTER(vp)]
        L.gtnb_ctx_destroy.argtypes = [vp]
        for name in ("gtnb_timer_start", "gtnb_flush_l2", "gtnb_ctx_synchronize"):
            getattr(L, name).argtypes = [vp]
        L.gtnb_timer_stop.argtypes = [vp, Ct.POINTER(Ct.c_float)]
        L.gtnb_last_error.restype = Ct.c_char_p
        L.gtnb_last_error.argtypes = [vp]
        L.gtnb_viterbi_dense.argtypes = [vp, Ct.c_int, Ct.c_int, Ct.c_int, vp, Ct.c_int, vp, vp, vp, vp]
        L.gtnb_profile_enable.argtypes = [vp, Ct.c_int]
        L.gtnb_profile_read.restype = Ct.c_char_p
        L.gtnb_profile_read.argtypes = [vp]
        h = vp()
        assert L.gtnb_ctx_create(0, None, Ct.byref(h)) == 0
        self.L, self.h, self.own = L, h.value, True

    def check(self, rc):
        if rc:
            raise RuntimeError(self.L.gtnb_last_error(self.h).decode())

    def timed(self, step):
        self.check(self.L.gtnb_flush_l2(self.h))
        self.check(self.L.gtnb_timer_start(self.h))
        self.check(step())
        ms = Ct.c_float()
        self.check(self.L.gtnb_timer_stop(self.h, Ct.byref(ms)))
        return ms.value

    def kernels_ms(self, step, steps):
        """per-kernel CUDA-event milliseconds per call over `steps` calls"""
        self.check(self.L.gtnb_profile_enable(self.h, 1))
        self.L.gtnb_profile_read(self.h)
        for _ in range(steps):
            self.timed(step)
        out = {}
        for line in self.L.gtnb_profile_read(self.h).decode().splitlines():
            name, n, ms = line.split()
            if name != "flush_l2":
                out[name] = float(ms) / steps
        self.check(self.L.gtnb_profile_enable(self.h, 0))
        return out

    def close(self):
        if self.own:
            self.L.gtnb_ctx_destroy(self.h)


def bench_shape(args, ctx, base, B, T, C):
    # emissions U(-5, 5) from seed 99 + b, transitions U(-5, 5) from seed 7
    e = np.empty((B, T, C), np.float32)
    for b in range(B):
        e[b] = np.random.default_rng(99 + b).uniform(-5.0, 5.0, (T, C)).astype(np.float32)
    tw = np.random.default_rng(7).uniform(-5, 5, C + C * C).astype(np.float32)
    W = np.ascontiguousarray(tw[C:])
    e_dev, tw_dev, w_dev = ctx.to_device(e), ctx.to_device(tw), ctx.to_device(W)
    p_dev, s_dev = ctx.alloc(4 * B * T), ctx.alloc(4 * B)
    host = {k: (np.zeros((B, T), np.int32), np.zeros(B, np.float32)) for k in ("old", "old_baseline")}
    this = Lib(ctx=ctx)

    def old(lib, key):
        p, s = host[key]
        return lambda: lib.L.gtnb_viterbi_dense(lib.h, B, T, C, e_dev.ptr, 1, None, tw.ctypes.data_as(capi._f32p),
                                                p.ctypes.data_as(capi._i32p), s.ctypes.data_as(capi._f32p))

    def ex(kind, w):
        return lambda: this.L.gtnb_viterbi_dense_ex(this.h, B, T, C, e_dev.ptr, 1, None, kind, w.ptr, 1, p_dev.ptr,
                                                    s_dev.ptr, 1)

    legs = {"old": (this, old(this, "old")), "asg_ex": (this, ex(capi.DENSE_ASG, tw_dev)),
            "bigram": (this, ex(capi.DENSE_BIGRAM, w_dev))}
    if base is not None:
        legs["old_baseline"] = (base, old(base, "old_baseline"))
    for lib, step in legs.values():
        for _ in range(args.warmup):
            lib.timed(step)
    rounds = {k: [] for k in legs}
    for r in range(args.rounds):
        for k in (list(legs) if r % 2 == 0 else list(legs)[::-1]):
            lib, step = legs[k]
            rounds[k].append(float(np.mean([lib.timed(step) for _ in range(args.steps)])))

    # outputs: the old entry point against asg_ex (==), and against the baseline build
    this.timed(legs["old"][1])
    old_p, old_s = (a.copy() for a in host["old"])
    this.timed(legs["asg_ex"][1])
    equal = {"old_vs_asg_ex": bool(np.array_equal(old_p, p_dev.download((B, T), np.int32))
                                   and np.array_equal(old_s, s_dev.download((B,))))}
    if base is not None:
        base.timed(legs["old_baseline"][1])
        equal["old_vs_old_baseline"] = bool(np.array_equal(old_p, host["old_baseline"][0])
                                            and np.array_equal(old_s, host["old_baseline"][1]))

    # per-kernel times, a separate pass
    kern = {k: lib.kernels_ms(step, args.steps) for k, (lib, step) in legs.items()}

    for buf in (e_dev, tw_dev, w_dev, p_dev, s_dev):
        buf.free()
    out = {k: {"ms_per_step_rounds": v, "ms_per_step_median": float(np.median(v)), "ms_per_step_min": float(min(v))}
           for k, v in rounds.items()}
    out.update({"shape": {"B": B, "T": T, "C": C}, "kernels_ms": kern, "equal": equal})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--baseline-lib", default=None, help="another build of libgtn_b200.so to time next to this one")
    args = ap.parse_args()
    ctx = capi.Ctx(0)
    base = Lib(args.baseline_lib) if args.baseline_lib else None
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    card, plim = [x.strip() for x in (q.split(",") + ["", ""])[:2]]
    out = {"card": card, "power_limit_w": plim, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
           "l2": "flushed between timed calls", "baseline_lib": args.baseline_lib}
    for name, (B, T, C) in SHAPES.items():
        out[name] = bench_shape(args, ctx, base, B, T, C)
    if base is not None:
        base.close()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
