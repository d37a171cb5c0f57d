"""Batched edit distance on the device (torch edit_distance, gtnb_edit_distance_async) against what a user runs today,
one JSON record on stdout (and in --out).  Three seeded workloads, each with and without alignment:

  token  B=512, references uniform in [200, 500] tokens over C=128, hypotheses with about 10 % random edits
  word   B=512, about 100 words of 1-8 tokens (a 2000-word lexicon over tokens 1..127, separator 0), 10 % word edits
  long   B=64, references of 4000 tokens over C=128, hypotheses with about 10 % edits, at most 4000 tokens

Per workload: ms until the results are on the device (CUDA events on the current stream, median of --reps calls) and
the host's wall time per call.  Against it:
  python   .tolist() and the per-pair numpy DP of tests/edit_oracle.py (distance, counts and alignment), whole batch
  gtn      -viterbi_score(compose(x, compose(edits, y))) through this project's drop-in gtn_b200.gtn, --sample pairs
  ref      the same through the reference library build() compiled into oracle/_ref (skipped where it is absent)
  (the compose routes are not run on the long workload: 48 M arcs per pair)
Then a validation step, ngram_ctc_decode (B=512 T=1000 C=128) -> collapse -> edit_distance against the token
workload's references, captured in a CUDA graph against the same step run eagerly: device and host time per step.
The card and its power limit are read in the same run.

    python scripts/bench_edit_distance.py [--reps 20] [--sample 4] [--out F]
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
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from gtn_b200 import torch_loss as tl  # noqa: E402
from tests import edit_oracle as eo  # noqa: E402

C_TOK = 128


def _edit(rng, ref, C, rate, lo=0):
    """ref with about `rate` of its units substituted, deleted or given an inserted neighbour"""
    out = []
    for t in ref:
        u = rng.random()
        if u < rate / 3:
            out.append(int(rng.integers(lo, C)))
        elif u < 2 * rate / 3:
            continue
        elif u < rate:
            out += [int(t), int(rng.integers(lo, C))]
        else:
            out.append(int(t))
    return out


def _pad(rows, width=None):
    width = width or max(1, max(len(r) for r in rows))
    a = np.full((len(rows), width), -1, np.int32)
    for b, r in enumerate(rows):
        a[b, :len(r)] = r[:width]
    return a, np.array([min(len(r), width) for r in rows], np.int32)


def token_workload(seed=0, B=512):
    rng = np.random.default_rng(seed)
    refs = [list(rng.integers(0, C_TOK, rng.integers(200, 501))) for _ in range(B)]
    hyps = [_edit(rng, r, C_TOK, 0.1) for r in refs]
    (h, hl), (r, rl) = _pad(hyps), _pad(refs)
    return h, hl, r, rl, None


def word_workload(seed=1, B=512, words=100):
    rng = np.random.default_rng(seed)
    lexicon = [tuple(rng.integers(1, C_TOK, rng.integers(1, 9))) for _ in range(2000)]

    def spell(ws):
        out = []
        for w in ws:
            out += list(lexicon[w]) + [0]
        return out[:-1]
    refs = [list(rng.integers(0, len(lexicon), words + rng.integers(-10, 11))) for _ in range(B)]
    hyps = [_edit(rng, r, len(lexicon), 0.1) for r in refs]
    (h, hl), (r, rl) = _pad([spell(w) for w in hyps]), _pad([spell(w) for w in refs])
    return h, hl, r, rl, 0


def long_workload(seed=2, B=64, n=4000):
    rng = np.random.default_rng(seed)
    refs = [list(rng.integers(0, C_TOK, n)) for _ in range(B)]
    hyps = [_edit(rng, r, C_TOK, 0.1) for r in refs]
    (h, hl), (r, rl) = _pad(hyps, n), _pad(refs, n)
    return h, hl, r, rl, None


WORKLOADS = {"token": token_workload, "word": word_workload, "long": long_workload}


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()


def time_device(fn, reps):
    """(median ms until the results are on the device, median host ms per call)"""
    fn()
    torch.cuda.synchronize()
    dev, host = [], []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        t0 = time.perf_counter()
        fn()
        host.append((time.perf_counter() - t0) * 1e3)
        b.record()
        b.synchronize()
        dev.append(a.elapsed_time(b))
    return float(np.median(dev)), float(np.median(host))


def python_route(h, hl, r, rl, sep):
    """what a user runs today: the tensors to lists, then a numpy DP per pair"""
    t0 = time.perf_counter()
    hh, hhl, rr, rrl = h.tolist(), hl.tolist(), r.tolist(), rl.tolist()
    for b in range(len(hh)):
        eo.edit_distance(hh[b][:hhl[b]], rr[b][:rrl[b]], sep)
    return (time.perf_counter() - t0) * 1e3


def compose_route(h, hl, r, rl, sep, n, gtn):
    """-viterbi_score(compose(x, compose(edits, y))) per pair over unit ids through the drop-in gtn module (gtn) or the
    reference (gtn None): (median ms per pair, distances)"""
    from oracle import pyoracle as po
    ms, dist = [], []
    for b in range(n):
        hu, ru = eo.units(h[b, :hl[b]].tolist(), r[b, :rl[b]].tolist(), sep)
        G = [eo.edits_graph(max([C_TOK - 1] + hu + ru) + 1), eo.chain_graph(hu), eo.chain_graph(ru)]
        t0 = time.perf_counter()
        if gtn is None:
            e, x, y = (po.RefGraph.from_arrays(g["flags"], g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"],
                                               calc_grad=False) for g in G)
            d = -po.ref_op("viterbi_score", po.ref_op("compose", x, po.ref_op("compose", e, y))).item()
        else:
            e, x, y = (_gtn_graph(gtn, g) for g in G)
            d = -gtn.viterbi_score(gtn.compose(x, gtn.compose(e, y))).item()
        ms.append((time.perf_counter() - t0) * 1e3)
        dist.append(int(round(d)))
    return float(np.median(ms)), dist


def _gtn_graph(gtn, g):
    G = gtn.Graph(False)
    for f in g["flags"]:
        G.add_node(bool(f & 1), bool(f & 2))
    for s, d, i, o, w in zip(g["src"], g["dst"], g["ilabel"], g["olabel"], g["w"]):
        G.add_arc(int(s), int(d), int(i), int(o), float(w))
    return G


def captured_step(reps):
    rng = np.random.default_rng(3)
    B, T = 512, 1000
    e = torch.as_tensor(rng.standard_normal((B, T, C_TOK), dtype=np.float32)).cuda()
    w = torch.as_tensor(rng.uniform(-2, 0, (C_TOK, C_TOK)).astype(np.float32)).cuda().view(-1)
    il = torch.as_tensor(rng.integers(T // 2, T + 1, B).astype(np.int32)).cuda()
    _, _, r, rl, _ = token_workload()
    r, rl = torch.as_tensor(r).cuda(), torch.as_tensor(rl).cuda()

    def step():
        p, _, _ = tl.ngram_ctc_decode(e, w, il)
        lab, n = tl.collapse(p, 0)
        return tl.edit_distance(lab, n, r, rl)
    eager = step()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            captured = step()
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    same = all(torch.equal(a, b) for a, b in zip(eager[:7], captured[:7]))
    ed, eh = time_device(step, reps)
    cd, ch = time_device(g.replay, reps)
    return {"shape": "ngram_ctc_decode B=512 T=1000 C=128 -> collapse -> edit_distance (token references)",
            "eager_ms": ed, "eager_host_ms": eh, "captured_ms": cd, "captured_host_ms": ch, "replay_equals_eager": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sample", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_edit_distance: no CUDA device")
    from gtn_b200 import gtn
    from oracle import pyoracle as po
    out = {"card": card(), "reps": args.reps, "workloads": {}}
    for name, make in WORKLOADS.items():
        h, hl, r, rl, sep = make()
        hd, hld, rd, rld = (torch.as_tensor(a).cuda() for a in (h, hl, r, rl))
        rec = {"B": int(h.shape[0]), "N": int(h.shape[1]), "M": int(r.shape[1]), "word_sep": sep}
        for align in (False, True):
            ms, host = time_device(lambda: tl.edit_distance(hd, hld, rd, rld, sep, align), args.reps)
            rec["align" if align else "no_align"] = {"ms": ms, "host_ms": host}
        res = tl.edit_distance(hd, hld, rd, rld, sep, True)
        want = eo.batch(h[:16], hl[:16], r[:16], rl[:16], sep)
        rec["first_16_equal_restatement"] = bool(np.array_equal(res.distance[:16].cpu().numpy(), want["distance"]) and
                                                 np.array_equal(res.hyp_align[:16].cpu().numpy(), want["hyp_align"]))
        ok = res.status == 0
        rec["error_rate"] = float(res.distance[ok].sum() / res.ref_units[ok].sum())
        rec["python_ms"] = python_route(hd, hld, rd, rld, sep)
        print(name, json.dumps(rec), file=sys.stderr, flush=True)
        if name == "long":  # a 4001 x 4001 grid of 48 M arcs per pair
            out["workloads"][name] = rec
            rec["gtn_compose_ms_per_pair"] = rec["ref_compose_ms_per_pair"] = "not measured"
            continue
        n = args.sample
        rec["gtn_compose_ms_per_pair"], dg = compose_route(h, hl, r, rl, sep, n, gtn)
        if po.have_ref():
            rec["ref_compose_ms_per_pair"], dr = compose_route(h, hl, r, rl, sep, n, None)
            assert dr == dg
        else:
            rec["ref_compose_ms_per_pair"] = "not measured: oracle/_ref is not built"
        assert dg == res.distance[:n].tolist(), (dg, res.distance[:n].tolist())
        rec["compose_pairs"] = n
        out["workloads"][name] = rec
    out["captured_step"] = captured_step(args.reps)
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
