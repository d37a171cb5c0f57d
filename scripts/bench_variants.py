"""gtnb_ctc_loss at a given shape under several context-flag settings: per-kernel CUDA-event times and the
step time (device-resident buffers, L2 flushed between steps), with a gradient / loss comparison against
the first variant.

    python scripts/bench_variants.py [B T C U] > variants.json

The bidir_* variants with an explicit bidir_mode are what the default (bidir_mode -1: the PAIR kernels,
gtnb_internal.h) was chosen from.
"""
import json
import sys

sys.path.insert(0, '.')
import numpy as np

import bench
from gtn_b200 import capi

L = capi.lib()
ctx = capi.Ctx(0)
i32p, f32p = capi._i32p, capi._f32p
B, T, C, U = (int(x) for x in sys.argv[1:5]) if len(sys.argv) >= 5 else (256, 1000, 64, 100)
e, tg = bench.make_inputs(0, B, T, C, U)
lens = np.full(B, U, np.int32)
cat = np.ascontiguousarray(np.concatenate(tg), np.int32)
e_dev = ctx.to_device(e)
g_dev = ctx.alloc(e.nbytes)
losses = np.zeros(B, np.float32)


def step(want_grad=True):
    ctx._check(L.gtnb_ctc_loss(ctx.h, B, T, C, e_dev.ptr, 1, None, cat.ctypes.data_as(i32p), lens.ctypes.data_as(i32p),
                               0, losses.ctypes.data_as(f32p), g_dev.ptr if want_grad else None, 1))


VARIANTS = [("two_sweeps", {"bidir": 0}, True), ("bidir", {"bidir": 1, "bidir_mode": -1}, True),
            ("bidir_loss_only", {"bidir": 1, "bidir_mode": -1}, False), ("two_sweeps_loss_only", {"bidir": 0}, False)]
VARIANTS += [("bidir_%s%s" % (m, "" if wg else "_loss_only"), {"bidir": 1, "bidir_mode": k}, wg)
             for wg in (True, False) for k, m in ((0, "node"), (1, "pair"))]
out = {"shape": [B, T, C, U]}
ref = None
for name, flags, wg in VARIANTS:
    for k, v in flags.items():
        ctx.set_flag(k, v)
    for _ in range(3):
        step(wg)
    res = {}
    if wg:
        g = g_dev.download((B, T, C))
        if ref is None:
            ref = (losses.copy(), g)
        else:
            res["max_rel_loss_diff"] = float((np.abs(losses - ref[0]) / np.abs(ref[0])).max())
            res["max_abs_grad_diff"] = float(np.abs(g - ref[1]).max())
    ctx.profile(True)
    ctx.profile_read()
    ts = []
    for _ in range(30):
        ctx.flush_l2()
        ctx.timer_start()
        step(wg)
        ts.append(ctx.timer_stop())
    pr = ctx.profile_read()
    ctx.profile(False)
    res.update({"ms_mean": float(np.mean(ts)), "ms_median": float(np.median(ts)), "ms_min": float(np.min(ts)),
                "kernels_ms": {k: v[1] / v[0] for k, v in pr.items() if k != "flush_l2"}})
    out[name] = res
    print(name, json.dumps(res), file=sys.stderr, flush=True)
ctx.set_flag("bidir", -1)
ctx.set_flag("bidir_mode", -1)
print(json.dumps(out, indent=1))
