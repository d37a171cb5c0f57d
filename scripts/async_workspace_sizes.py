"""Every *_async_workspace query over a grid of bounds: one JSON line per query on stdout (the query, its arguments,
its return code and the bytes), nothing written.  Two libraries compared line by line show whether a change moved a
workspace size or an error code of the asynchronous calls.

Grid: B in {1, 7, 64}, T in {1, 50, 400}, C in {29, 64, 128, 200}, S in {0, 1, 30, 120}, every dtype, with_grad,
kind, beam / nbest and alignment flag each query takes; gtnb_viterbi_transitions_async_workspace on one prepared
transition graph without epsilon arcs (the trigram G at C = 29) and one with them (the benchmark's backoff trigram at
C = 64).  Needs a GPU (the contexts and the prepared graphs live on one).

    python scripts/async_workspace_sizes.py [--lib path/to/libgtn_b200.so] > sizes.jsonl
"""
import argparse
import ctypes as C
import itertools
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gtn_b200 import capi  # noqa: E402
from tests import backoff_oracle as bo  # noqa: E402
from tests import sparse_trans_oracle as st  # noqa: E402

BS, TS, CS, SS = (1, 7, 64), (1, 50, 400), (29, 64, 128, 200), (0, 1, 30, 120)
DTYPES = (capi.F32, capi.BF16, capi.F16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="the library to load instead of the package's")
    args = ap.parse_args()
    if args.lib:
        capi.LIB_PATH = os.path.abspath(args.lib)
    L = capi.lib()
    ctx = capi.Ctx(0)

    def query(name, *a):
        n = C.c_size_t(12345)
        rc = getattr(L, name)(ctx.h, *a, C.byref(n))
        print(json.dumps({"fn": name, "args": [x if isinstance(x, int) else str(x) for x in a], "rc": rc,
                          "bytes": n.value}))

    for B, T, Cn, S in itertools.product(BS, TS, CS, SS):
        for dt in DTYPES:
            for g in (0, 1):
                for fn in ("gtnb_ctc_loss_async_workspace", "gtnb_ngram_ctc_loss_async_workspace",
                           "gtnb_asg_loss_async_workspace"):
                    query(fn, B, T, Cn, S, dt, g)
            for fn in ("gtnb_ctc_align_async_workspace", "gtnb_ngram_ctc_align_async_workspace",
                       "gtnb_asg_align_async_workspace"):
                query(fn, B, T, Cn, S, dt)
    for B, T, Cn in itertools.product(BS, TS, CS):
        for dt in DTYPES:
            for kind in (capi.DENSE_ASG, capi.DENSE_BIGRAM):
                query("gtnb_viterbi_dense_async_workspace", B, T, Cn, dt, kind)
            for kind in (capi.DENSE_CTC, capi.DENSE_BIGRAM, capi.DENSE_ASG):
                for beam, nbest in ((1, 1), (8, 4), (64, 64)):
                    query("gtnb_beam_decode_async_workspace", B, T, Cn, dt, kind, beam, nbest)
    # edit distance: N and M from the T and S grids, token and word units, with and without an alignment
    for B, N, M in itertools.product(BS, TS + (4096, 4097), SS):
        for sep in (-1, 0):
            for align in (0, 1):
                query("gtnb_edit_distance_async_workspace", B, N, M, sep, align)
    for label, G, Cn, backoff in (("trigram29", st.trigram_graph(29), 29, 0),
                                  ("backoff_trigram64", bo.backoff_lm(np.random.default_rng(3), 64)[0], 64, 1)):
        view, keep = capi.make_view(G["flags"], G["src"], G["dst"], G["olabel"], G["olabel"])
        h = C.c_void_p()
        ctx._check(L.gtnb_transitions_create(ctx.h, C.byref(view), Cn, backoff, C.byref(h)))
        del keep
        for B, T in itertools.product(BS, TS):
            n = C.c_size_t(12345)
            rc = L.gtnb_viterbi_transitions_async_workspace(ctx.h, h, B, T, C.byref(n))
            print(json.dumps({"fn": "gtnb_viterbi_transitions_async_workspace", "args": [label, B, T], "rc": rc,
                              "bytes": n.value}))
        L.gtnb_transitions_destroy(ctx.h, h)
    ctx.close()


if __name__ == "__main__":
    main()
