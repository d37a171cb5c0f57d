"""Benchmark of the beam decoders (gtnb_beam_decode_async through torch ctc_beam_decode, ngram_ctc_beam_decode and
asg_beam_decode) on an H100: ms until the results are on the device, medians of timed calls, and the host's wall
time per call, at
  CTC         B=256 T=1000 C=64;
  n-gram, ASG B=128 T=500  C=64 and C=128;
with K in {1, 8, 32, 64}, N in {1, 8} (N <= K), float32 and bf16 emissions.  Against, on the same inputs: the greedy
decoders (argmax + collapse for CTC, ngram_ctc_decode / asg_decode + collapse) and the float64 restatement of
tests/beam_oracle.py per utterance on a sample.  torchaudio's cuda_ctc_decoder is not run: on the CTC workload it
stopped the process with an illegal-address error inside its own decoder.  Also the mean exact numerator gain of the
beam's top transcript over the greedy one, both scored by the loss calls on the same synthetic emissions (not a word
error rate).  The card's name and power limit are read in the same run.  Prints one JSON line per setting, then
the whole record as one JSON line (also written to --out when given).

The emissions are synthetic: log-softmax rows with one favoured label per frame (blank half of the time).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gtn_b200 import capi  # noqa: E402
from gtn_b200 import torch_loss as tl  # noqa: E402


def inputs(rng, kind, B, T, C, device="cuda"):
    """seeded synthetic emissions [B, T, C] (float32, on the device) and transitions (None for CTC)"""
    x = rng.standard_normal((B, T, C)).astype(np.float32) * 2.0
    lab = np.where(rng.random((B, T)) < 0.5, 0, rng.integers(1, C, (B, T)))
    np.put_along_axis(x, lab[..., None], np.take_along_axis(x, lab[..., None], -1) + 5.0, -1)
    e = torch.log_softmax(torch.as_tensor(x), -1).to(device)
    if kind == capi.DENSE_CTC:
        return e, None
    n = C * C + (C if kind == capi.DENSE_ASG else 0)
    return e, torch.as_tensor((rng.standard_normal(n) * 0.5).astype(np.float32)).to(device)


def decode(kind, e, w, K, N):
    if kind == capi.DENSE_CTC:
        return tl.ctc_beam_decode(e, K, N)
    if kind == capi.DENSE_BIGRAM:
        return tl.ngram_ctc_beam_decode(e, w, K, N)
    return tl.asg_beam_decode(e, w, K, N)


def greedy(kind, e, w):
    if kind == capi.DENSE_CTC:
        return tl.collapse(e.argmax(-1).to(torch.int32), 0)
    if kind == capi.DENSE_BIGRAM:
        return tl.collapse(tl.ngram_ctc_decode(e, w)[0], 0)
    return tl.collapse(tl.asg_decode(e, w)[0], None)


def loss(kind, e, w, tokens, lengths):
    tg, tn = tokens.clamp(min=0), lengths.clamp(min=0).to(torch.int32)
    if kind == capi.DENSE_CTC:
        return tl.ctc_loss(e.float(), tg, 0, "none", None, tn)
    if kind == capi.DENSE_BIGRAM:
        return tl.ngram_ctc_loss(e.float(), w, tg, None, 0, "none", False, tn)
    return tl.asg_loss(e.float(), w, tg, "none", False, None, tn)


def timed(fn, reps):
    """(median ms until the results are on the device, median host ms per call)"""
    dev, host = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        dev.append((t2 - t0) * 1e3)
        host.append((t1 - t0) * 1e3)
    return float(np.median(dev)), float(np.median(host))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa: BLE001
        q = "unknown (%s)" % ex
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sample", type=int, default=2, help="utterances per workload for the numpy restatement")
    ap.add_argument("--out", default=None, help="also write the JSON record to this file")
    ap.add_argument("--quick", action="store_true", help="one K and N per workload")
    a = ap.parse_args()
    from tests import beam_oracle as bo
    res = dict(card=card(), torch=torch.__version__, torchaudio_cuda_ctc_decoder="not measured", workloads=[])
    names = {capi.DENSE_CTC: "ctc", capi.DENSE_BIGRAM: "ngram_ctc", capi.DENSE_ASG: "asg"}
    shapes = [(capi.DENSE_CTC, 256, 1000, 64)] + [(k, 128, 500, c) for k in (capi.DENSE_BIGRAM, capi.DENSE_ASG)
                                                  for c in (64, 128)]
    for kind, B, T, C in shapes:
        rng = np.random.default_rng(1000 + kind * 10 + C)
        e32, w = inputs(rng, kind, B, T, C)
        g_tok, g_len = greedy(kind, e32, w)
        g_ms, g_host = timed(lambda: greedy(kind, e32, w), a.reps)
        greedy_loss = loss(kind, e32, w, g_tok, g_len).double()
        row = dict(kind=names[kind], B=B, T=T, C=C, greedy_ms=g_ms, greedy_host_ms=g_host, runs=[])
        for dt in (torch.float32, torch.bfloat16):
            e = e32.to(dt)
            for K in ((8,) if a.quick else (1, 8, 32, 64)):
                for N in ((1,) if a.quick else (1, 8)):
                    if N > K:
                        continue
                    out = decode(kind, e, w, K, N)
                    ms, host = timed(lambda: decode(kind, e, w, K, N), a.reps)
                    r = dict(dtype=str(dt).replace("torch.", ""), K=K, N=N, ms=ms, host_ms=host,
                             status_counts={int(s): int(c) for s, c in zip(*np.unique(out.status.cpu().numpy(),
                                                                                      return_counts=True))})
                    if N == 1 and dt == torch.float32:
                        bl = loss(kind, e32, w, out.tokens[:, 0], out.lengths[:, 0]).double()
                        ok = torch.isfinite(bl) & torch.isfinite(greedy_loss)
                        r["mean_numerator_gain_over_greedy"] = float((greedy_loss[ok] - bl[ok]).mean())
                        r["share_better_than_greedy"] = float((bl[ok] < greedy_loss[ok] - 1e-4).double().mean())
                    if N == 1 and dt == torch.float32 and K == 8 and a.sample:
                        en = e32[:a.sample].cpu().numpy()
                        t0 = time.perf_counter()
                        want = bo.batch(en, kind, None if w is None else w.cpu().numpy(), None, 0, K, N)
                        r["numpy_ms_per_utterance"] = (time.perf_counter() - t0) * 1e3 / a.sample
                        ok = want["margin"] > 1e-3
                        r["numpy_agrees_top1"] = int(sum(
                            np.array_equal(want["tokens"][b], out.tokens[b].cpu().numpy()) for b in np.nonzero(ok)[0]))
                        r["numpy_compared"] = int(ok.sum())
                    row["runs"].append(r)
                    print(json.dumps(dict(kind=row["kind"], C=C, **r)), flush=True)
        res["workloads"].append(row)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
