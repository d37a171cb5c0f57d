"""Benchmark of the fused beam decoders (gtnb_beam_decode_lm_async through torch ctc_lm_beam_decode,
ngram_ctc_lm_beam_decode and asg_lm_beam_decode) on an H100: ms until the results are on the device, medians of
timed calls, at
  CTC         B=256 T=1000 C=64, K = 8 and 64;
  n-gram, ASG B=128 T=500  C=64 and C=128, K = 8 and 64;
N = 1, float32.  The variants of each workload run in one session, alternating call by call:
  beam        gtnb_beam_decode_async (ctc_beam_decode, ...), the decoder without fusion;
  lm_none     the fused call with no LM and token_beam = C: the cost of the fused path itself;
  lm          with the benchmark's backoff trigram (tests/backoff_oracle.backoff_lm: 2065 nodes and a 1.1 MB table at C = 64,
              2.2 MB at C = 128);
  lm_p16      the same with token_beam = 16;
  lm_big      an LM at the table bound (big_lm: S * (C + 1) = 2^25 entries, a 256 MB table far beyond the L2,
              against backoff_lm's 1-2 MB one that stays in it).
Also the token error rate with and without fusion on the seeded quality workload (utterances sampled from an n-gram
LM's own chain, emissions noisy around a CTC alignment of them; see quality_workload).  The card's name and power
limit are read in the same run.  Prints one JSON line per setting, then the whole record as one JSON line (also written
to --out when given).
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from gtn_b200 import capi  # noqa: E402
from gtn_b200 import torch_loss as tl  # noqa: E402
from tests import backoff_oracle as bko  # noqa: E402
from tests import beam_lm_oracle as blo  # noqa: E402
import bench_beam_decode as bbd  # noqa: E402  (the beam benchmark's seeded emissions)


def gtn_graph(G, w):
    """a gtn_b200.gtn.Graph of a graph dict (tests/graph_oracle.make) and its weights"""
    from gtn_b200 import gtn
    h = gtn.Graph()
    for f in G["flags"]:
        h.add_node(bool(f & 1), bool(f & 2))
    for a in range(len(G["src"])):
        h.add_arc(int(G["src"][a]), int(G["dst"][a]), int(G["ilabel"][a]), int(G["ilabel"][a]), float(w[a]))
    return h


def big_lm(rng, C, n_arcs=8):
    """an LM at the table bound, S * (C + 1) <= 2^25: a root with an arc per token to its bigram state, C bigram
    states with 20 arcs each, and trigram-like states with n_arcs arcs each to random states; every state but the
    root backs off (epsilon) to a bigram state or the root.  -> (graph dict, weights)"""
    S = (1 << 25) // (C + 1)
    n = C + C * 20 + (S - 1 - C) * n_arcs
    src = np.concatenate([np.zeros(C), np.repeat(np.arange(1, C + 1), 20),
                          np.repeat(np.arange(C + 1, S), n_arcs)]).astype(np.int32)
    lab = np.concatenate([np.arange(C)] + [rng.choice(C, 20, replace=False) for _ in range(C)] +
                         [rng.choice(C, n_arcs, replace=False) for _ in range(S - 1 - C)]).astype(np.int32)
    dst = np.concatenate([1 + np.arange(C), rng.integers(1, S, n - C)]).astype(np.int32)
    x = (rng.standard_normal(n) - 2.5).astype(np.float32)
    eps_src = np.arange(1, S, dtype=np.int32)
    eps_dst = np.where(eps_src <= C, 0, 1 + (eps_src % C)).astype(np.int32)
    flags = np.full(S, 2, np.uint8)
    flags[0] = 3
    G = dict(flags=flags, src=np.concatenate([src, eps_src]), dst=np.concatenate([dst, eps_dst]),
             ilabel=np.concatenate([lab, np.full(S - 1, -1, np.int32)]))
    return G, np.concatenate([x, np.log(rng.uniform(0.2, 0.5, S - 1)).astype(np.float32)])


def lm_from_arrays(G, w, C):
    """a LanguageModel made through gtnb_lm_create straight from arrays (a graph too large to build arc by arc)"""
    import ctypes as C_
    lm = tl.LanguageModel.__new__(tl.LanguageModel)
    lm.device, lm.num_labels = torch.device("cuda", torch.cuda.current_device()), C
    lm._g = tl._async_ctx(lm.device, "LanguageModel")
    v, keep = capi.make_view(G["flags"], G["src"], G["dst"], G["ilabel"], G["ilabel"], w)
    h = C_.c_void_p()
    lm._g._check(capi.lib().gtnb_lm_create(lm._g.h, C_.byref(v), C, C_.byref(h)))
    lm.h = h
    return lm


def decode_lm(kind, e, w, lm, K, N, lm_weight=1.0, token_bonus=0.0, P=None, il=None):
    if kind == capi.DENSE_CTC:
        return tl.ctc_lm_beam_decode(e, lm, lm_weight, token_bonus, K, N, P, il)
    if kind == capi.DENSE_BIGRAM:
        return tl.ngram_ctc_lm_beam_decode(e, w, lm, lm_weight, token_bonus, K, N, P, il)
    return tl.asg_lm_beam_decode(e, w, lm, lm_weight, token_bonus, K, N, P, il)


def sample(rng, lm, C, U, blank=0):
    """a transcript of U tokens drawn from the LM's own chain (its resolved weights renormalised, blank excluded)"""
    s, y = lm.start, []
    for _ in range(U):
        x = np.array([lm.resolve(s, c)[0] for c in range(C)])
        x[blank] = -np.inf
        p = np.exp(x - x.max())
        c = int(rng.choice(C, p=p / p.sum()))
        y.append(c)
        s = lm.resolve(s, c)[1]
    return y


def quality_workload(seed=1, C=32, B=16, U=20, T=60, noise=1.0, peak=3.0):
    """(LM graph dict, its weights, its restatement, emissions [B, T, C] float32, references): a backoff trigram
    counted from a peaked random chain; transcripts sampled from it; each token held 1 or 2 frames, blanks between
    them half of the time (always between repeats), blank to the end; emissions log_softmax(noise * N(0, 1) + peak at
    the aligned label).  Tuned with the restatement: at K = 8 greedy-like decoding without the LM leaves a token error
    rate near 0.5, fusion at lm_weight 1 about half that."""
    rng = np.random.default_rng(seed)
    G, w = bko.backoff_ngram(rng, C, 3, n_tokens=4000, min_count=3)
    lm = blo.LM(G, w, C)
    r2 = np.random.default_rng(seed + 1)
    e = np.zeros((B, T, C), np.float32)
    refs = []
    for b in range(B):
        y = sample(r2, lm, C, U)
        refs.append(y)
        lab = []
        for i, c in enumerate(y):
            if (i and y[i - 1] == c) or r2.random() < 0.5:
                lab.append(0)
            lab += [c] * int(r2.integers(1, 3))
        lab += [0] * (T - len(lab))
        x = r2.standard_normal((T, C)) * noise
        x[np.arange(T), lab[:T]] += peak
        e[b] = x - np.log(np.exp(x).sum(-1, keepdims=True))
    return G, w, lm, e, refs


def ter(tokens, lengths, refs):
    """token error rate of the first hypotheses against refs, through edit_distance on the device"""
    B = len(refs)
    M = max(map(len, refs))
    r = torch.full((B, M), -1, dtype=torch.int32, device=tokens.device)
    for b, y in enumerate(refs):
        r[b, :len(y)] = torch.as_tensor(y, dtype=torch.int32)
    rl = torch.as_tensor([len(y) for y in refs], dtype=torch.int32, device=tokens.device)
    d = tl.edit_distance(tokens[:, 0], lengths[:, 0].clamp(min=0), r, rl)
    return float(d.distance.sum()) / float(rl.sum())


def timed(fns, reps):
    """{name: median ms until the results are on the device}, the variants alternating call by call"""
    t = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            t[k].append((time.perf_counter() - t0) * 1e3)
    return {k: float(np.median(v)) for k, v in t.items()}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="one small workload per kind (a rehearsal)")
    a = ap.parse_args()
    rec = dict(card=card(), settings=[])
    print(json.dumps(dict(card=rec["card"])), flush=True)
    rng = np.random.default_rng(0)
    lms = {}
    for C in (64, 128):
        G, w = bko.backoff_lm(np.random.default_rng(C), C=C)
        lms[(C, "lm")] = tl.LanguageModel(gtn_graph(G, w), C)
        if not a.quick:
            lms[(C, "lm_big")] = lm_from_arrays(*big_lm(np.random.default_rng(C + 1), C), C)
    work = [(capi.DENSE_CTC, 256, 1000, 64), (capi.DENSE_BIGRAM, 128, 500, 64), (capi.DENSE_BIGRAM, 128, 500, 128),
            (capi.DENSE_ASG, 128, 500, 64), (capi.DENSE_ASG, 128, 500, 128)]
    if a.quick:
        work = [(k, 8, 50, 64) for k in (capi.DENSE_CTC, capi.DENSE_BIGRAM, capi.DENSE_ASG)]
    for kind, B, T, C in work:
        e, w = bbd.inputs(rng, kind, B, T, C)
        for K in (8, 64):
            fns = {"beam": lambda: bbd.decode(kind, e, w, K, 1),
                   "lm_none": lambda: decode_lm(kind, e, w, None, K, 1),
                   "lm": lambda: decode_lm(kind, e, w, lms[(C, "lm")], K, 1),
                   "lm_p16": lambda: decode_lm(kind, e, w, lms[(C, "lm")], K, 1, P=16)}
            if (C, "lm_big") in lms:
                fns["lm_big"] = lambda: decode_lm(kind, e, w, lms[(C, "lm_big")], K, 1)
            for fn in fns.values():
                fn()
            # the fused call without an LM ranks exactly as the plain one
            x, y = fns["beam"](), fns["lm_none"]()
            same = all(torch.equal(getattr(x, k), getattr(y, k)) for k in ("tokens", "lengths", "scores", "status"))
            ms = timed(fns, 3 if a.quick else a.reps)
            s = dict(kind={2: "ctc", 1: "ngram_ctc", 0: "asg"}[kind], B=B, T=T, C=C, K=K, N=1, ms=ms,
                     lm_none_equals_beam=same)
            rec["settings"].append(s)
            print(json.dumps(s), flush=True)
    G, w, lm_r, e, refs = quality_workload()
    lm = tl.LanguageModel(gtn_graph(G, w), e.shape[2])
    ed = torch.as_tensor(e).cuda()
    q = {}
    for K in (8, 16):
        q["K%d" % K] = dict(no_lm=ter(*decode_lm(capi.DENSE_CTC, ed, None, None, K, 1)[:2], refs),
                            lm=ter(*decode_lm(capi.DENSE_CTC, ed, None, lm, K, 1)[:2], refs))
    rec["quality_ter"] = q
    print(json.dumps(dict(quality_ter=q)), flush=True)
    print(json.dumps(rec))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
