"""Benchmark of the streaming beam decoder (gtnb_beam_decode_chunk_async through torch StreamingBeamDecoder) on an
H100, against the one-shot call on the same utterances, at N = 1, float32.  Workloads:
  ctc        CTC B=256 T=1000 C=64 (bench_beam_decode's emissions), no LM;
  lm         the same emissions with bench_beam_lm's token backoff trigram (backoff_lm at C = 64), token_beam 16;
  lexicon    CTC B=256 T=1000 on bench_beam_lexicon's 20 000-word letters lexicon (C = 29) with its word trigram;
at K = 8 and 64, in chunks of 1, 8, 32 and 100 frames.  For each: the one-shot call's ms (device, until the results
are on the device), and for the streaming decoder, with and without the best-beam outputs: the whole utterance's ms
over all its chunk calls (CUDA events around the loop), that over the number of calls (ms per chunk call), the host
ms per call (enqueue only), and the same utterance as one captured step replayed per chunk (ms per chunk).  Every
row ends on the last chunk; its results are checked == the one-shot call's.  The card's name and power limit are read
in the same run.  Prints one JSON line per setting, then the whole record (also written to --out when given).
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from gtn_b200 import capi  # noqa: E402
from gtn_b200 import torch_loss as tl  # noqa: E402
from tests import backoff_oracle as bko  # noqa: E402
import bench_beam_decode as bbd  # noqa: E402  (seeded emissions)
import bench_beam_lm as bbl  # noqa: E402  (card, the token LM)
import bench_beam_lexicon as bbx  # noqa: E402  (the letters lexicon and its emissions)


def device_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def stream_run(dec, xs, end):
    """every chunk (frames, lengths) through dec.step, END on the last -> host ms per call"""
    t = 0.0
    for i, (x, n) in enumerate(xs):
        t0 = time.perf_counter()
        dec.step(x, n, end=end if i == len(xs) - 1 else None)
        t += time.perf_counter() - t0
    return t * 1e3 / len(xs)


def captured(dec, xs, end):
    """one step captured on a static chunk buffer, replayed per chunk (the buffers refilled) -> the replay function"""
    x, n = torch.empty_like(xs[0][0]), torch.empty_like(xs[0][1])
    flag = torch.zeros_like(end)
    dec.step(x[:, :0].contiguous(), torch.zeros_like(n))  # (warm-up: no frames, no flag, no change)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            dec.step(x, n, end=flag)
    torch.cuda.current_stream().wait_stream(s)

    def replay():
        for i, (c, k) in enumerate(xs):
            x.copy_(c)
            n.copy_(k)
            flag.fill_(i == len(xs) - 1)
            g.replay()
    return replay, g


def same(r, want):
    return all(torch.equal(getattr(r, k).view(torch.int32), getattr(want, k).view(torch.int32)) for k in want._fields)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="small workloads (a rehearsal)")
    a = ap.parse_args()
    rec = dict(card=bbl.card(), settings=[])
    print(json.dumps(dict(card=rec["card"])), flush=True)
    B, T = (8, 100) if a.quick else (256, 1000)
    rng = np.random.default_rng(0)
    e64, _ = bbd.inputs(np.random.default_rng(1064), capi.DENSE_CTC, B, T, 64)
    lm = tl.LanguageModel(bbl.gtn_graph(*bko.backoff_lm(np.random.default_rng(64), C=64)), 64)
    V = 20000 // (10 if a.quick else 1)
    sp = bbx.random_spellings(rng, V, np.arange(1, 28))
    info = type("Info", (), dict(C=29, cls=bbx.letters_classes(), spellings=sp))
    lex = tl.Lexicon(sp, 29, V, separator=28, lm=bbx.synth_word_lm(rng, V, V // 4, V // 2, 8))
    e29, _ = bbx.spelled_inputs(rng, capi.DENSE_CTC, info, B, T)
    work = [("ctc", e64, dict()), ("lm", e64, dict(lm=lm, lm_weight=0.5, bonus=0.5, token_beam=16)),
            ("lexicon", e29, dict(lexicon=lex, lm_weight=1.0, bonus=0.5))]
    for name, e, kw in work:
        C = e.shape[2]
        for K in (8, 64):
            P = kw.get("token_beam")
            if "lexicon" in kw:
                one = lambda: tl.ctc_lexicon_beam_decode(e, lex, kw["lm_weight"], kw["bonus"], K, 1, P)  # noqa: E731
            else:
                one = lambda: tl.ctc_lm_beam_decode(e, kw.get("lm"), kw.get("lm_weight", 1.0),  # noqa: E731
                                                    kw.get("bonus", 0.0), K, 1, P)
            want = one()
            one_ms = min(device_ms(one) for _ in range(3))
            end = torch.ones(B, dtype=torch.bool, device="cuda")
            for Tc in (1, 8, 32, 100):
                # (the last chunk is padded: its rows take min(Tc, T - t) frames)
                xs = [(torch.nn.functional.pad(e[:, t:t + Tc], (0, 0, 0, Tc - min(Tc, T - t))).contiguous(),
                       torch.full((B,), min(Tc, T - t), dtype=torch.int32, device="cuda")) for t in range(0, T, Tc)]
                s = dict(workload=name, B=B, T=T, C=C, K=K, N=1, chunk=Tc, calls=len(xs), oneshot_ms=one_ms)
                for best in (True, False):
                    dec = tl.StreamingBeamDecoder(B, T, C, lm=kw.get("lm"), lexicon=kw.get("lexicon"),
                                                  lm_weight=kw.get("lm_weight", 1.0), bonus=kw.get("bonus", 0.0),
                                                  beam=K, nbest=1, token_beam=P, best=best)
                    stream_run(dec, xs, end)  # (warm-up)
                    torch.cuda.synchronize()
                    ok = same(dec.results, want)
                    host = []
                    ms = device_ms(lambda: host.append(stream_run(dec, xs, end)))
                    replay, g = captured(dec, xs, end)
                    replay()
                    torch.cuda.synchronize()
                    ok = ok and same(dec.results, want)
                    cap_ms = device_ms(replay)
                    del g
                    tag = "best" if best else "nobest"
                    s.update({"%s_total_ms" % tag: ms, "%s_ms_per_call" % tag: ms / len(xs),
                              "%s_host_ms_per_call" % tag: host[0],
                              "%s_replay_ms_per_chunk" % tag: cap_ms / len(xs),
                              "%s_replay_total_ms" % tag: cap_ms, "%s_equals_oneshot" % tag: ok})
                rec["settings"].append(s)
                print(json.dumps(s), flush=True)
    print(json.dumps(rec))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
