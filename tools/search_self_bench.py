#!/usr/bin/env python
"""All-vs-all threshold search over one set, two ways, on the BASELINE config-4 targets (common.config_workload(4): the 50,000
targets, BLOSUM50, gaps 3 / 1, score_size 1, mask_len 150), alternating in one run:
    all    set_sequences(S, S) and search_all: every ordered pair, the diagonal included (2.5e9 pairs)
    self   set_sequences_self(S) and search_self: every unordered pair once (1.25e9 pairs)
The threshold is the one of arm (c) of search_tile_bench.py: the median of the 10th best scores of 32 targets against all
targets (or --thr).  Per call: wall time, total_ms, GCUPS on the triangle's cells (the cells both calls must cover:
sum over pairs i < j of len(i) * len(j)), hits, bytes copied back.  Asserts that the self hits and their mirrors are
exactly the full search's hits without the diagonal, with identical records for the oriented pairs.  Prints the card's name,
power limit and SM clock before and after the run.
    python tools/search_self_bench.py [--reps 1] [--thr 0] [--n 50000] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import common as C  # noqa: E402
from search_bench import _pkg, card  # noqa: E402


def mirror_identical(s, a, lens):
    """self hits + mirrors == full hits without the diagonal, oriented records identical (numpy, keys q * n + r)"""
    n = len(lens)
    order = np.lexsort((np.arange(n), lens))
    rank = np.empty(n, np.int64)
    rank[order] = np.arange(n)
    s_q = np.repeat(np.arange(n, dtype=np.int64), np.diff(s[0]))
    a_q = np.repeat(np.arange(n, dtype=np.int64), np.diff(a[0]))
    s_r, a_r = s[1].astype(np.int64), a[1].astype(np.int64)
    if not (rank[s_q] < rank[s_r]).all():
        return False
    both = np.sort(np.concatenate([s_q * n + s_r, s_r * n + s_q]))
    off = a_q != a_r
    if not np.array_equal(both, np.sort(a_q[off] * n + a_r[off])):
        return False
    ori = off & (rank[a_q] < rank[a_r])
    if not np.array_equal(a_q[ori] * n + a_r[ori], s_q * n + s_r):
        return False
    return all(np.array_equal(a[2][ori][f], s[2][f]) for f in C.CMP_FIELDS)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=1, help="timed calls of each kind, alternating")
    ap.add_argument("--thr", type=int, default=0, help="min_score (0: the 10th best scores of a sample, as search_tile_bench (c))")
    ap.add_argument("--n", type=int, default=50000, help="the first n targets")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    import torch
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    torch.cuda.init()
    emit({"card": card(), "torch_device": torch.cuda.get_device_name(0)})
    L = _pkg()
    W = C.config_workload(4)
    S = W["refs"][: args.n]
    lens = np.array([len(s) for s in S], dtype=np.int64)
    tri_cells = (float(lens.sum()) ** 2 - float((lens.astype(np.float64) ** 2).sum())) / 2
    kw = dict(gap_open=W["gapO"], gap_extend=W["gapE"], mask_len=W["mask_len"], score_size=W["score_size"])
    eng = L.BatchAligner(device=0)
    thr = args.thr
    if thr <= 0:
        eng.set_sequences(S[:32], S)
        thr = int(np.median(eng.search(W["mat"], W["n"], 10, **kw)[1][:, 9]["score1"]))

    def run(arm):
        if arm == "all":
            eng.set_sequences(S, S)
            fn = lambda: eng.search_all(W["mat"], W["n"], thr, **kw)   # noqa: E731
        else:
            eng.set_sequences_self(S)
            fn = lambda: eng.search_self(W["mat"], W["n"], thr, **kw)  # noqa: E731
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        return out, (time.perf_counter() - t0) * 1e3, eng.timing()

    wall = {"all": [], "self": []}
    last = {}
    for rep in range(args.reps):
        for arm in ("all", "self"):
            out, ms, t = run(arm)
            wall[arm].append(ms)
            last[arm] = out
            emit({"arm": arm, "rep": rep, "sequences": len(S), "min_score": thr, "wall_ms": ms, "total_ms": t["total_ms"],
                  "gcups_triangle": tri_cells / ms / 1e6, "hits": int(len(out[1])), "cells_forward": t["cells_forward"],
                  "fill_forward_launches": t["fill_forward_launches"], "leftover_pairs": t["leftover_pairs"],
                  "byte_overflows": t["byte_overflows"], "bytes_to_host": int(40 * len(out[1]) + out[0].nbytes + out[3].nbytes)})
    ok = mirror_identical(last["self"], last["all"], lens)
    med = {a: float(np.median(v)) for a, v in wall.items()}
    emit({"mirror_identical": bool(ok), "all_ms_median": med["all"], "self_ms_median": med["self"],
          "self_over_all": med["self"] / med["all"]})
    emit({"card_after": card()})
    eng.close()
    if args.out:
        with open(args.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")
    assert ok, "self-search hits and their mirrors differ from the full search without the diagonal"
    return 0


if __name__ == "__main__":
    sys.exit(main())
