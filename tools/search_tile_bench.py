#!/usr/bin/env python
"""Searches over grid tiles on the BASELINE config-4 workload (common.config_workload(4): BLOSUM50, score_size 1, mask_len 150),
in one run:

    (a) overhead   the 512-query slice x all 50,000 targets, search(k): untiled against --tile-refs references per tile
                   (12,500: 4 tiles), alternating calls after one warm-up call of each; medians of --reps; the arrays must
                   be identical
    (b) above      config_workload(4, n_queries=10,000, n_targets=220,000), search(k): 2.2e9 pairs, tiled automatically
                   (more than 2^31 - 1 pairs); wall time, GCUPS on the cells of the real pairs, fill launches, leftover pairs
                   (must be 0) and the bytes copied to the host
    (c) all-vs-all the 50,000 targets as queries and references, search_all at --all-thr: 2.5e9 pairs (default: the median
                   of the 10th best scores of 32 targets against all targets, a family-level threshold)
    (d) old path   a 64-query slice x all 50,000 targets forced through the general path (grid_min = 2^31 - 1), the way
                   (b) and (c) ran before grids were tiled

Prints the device's name, power limit and SM clocks first, then one JSON line per arm.

    python tools/search_tile_bench.py [--k 10] [--reps 3] [--tile-refs 12500] [--all-thr 0] [--skip ARMS] [--out FILE]
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


def cells(queries, refs):
    return float(sum(len(q) for q in queries)) * float(sum(len(r) for r in refs))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3, help="timed calls of each kind in (a)")
    ap.add_argument("--tile-refs", type=int, default=12500, help="grid_tile_refs of the tiled calls of (a)")
    ap.add_argument("--all-thr", type=int, default=0, help="min_score of (c) (0: the 10th best scores of a sample)")
    ap.add_argument("--skip", default="", help="arms to leave out, e.g. cd")
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
    refs = W["refs"]
    kw = dict(gap_open=W["gapO"], gap_extend=W["gapE"], mask_len=W["mask_len"], score_size=W["score_size"])
    eng = L.BatchAligner(device=0)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        return out, (time.perf_counter() - t0) * 1e3, eng.timing()

    # (a) tiling overhead on the slice (its calls also warm up the shapes of (b))
    qs = W["queries"][:512]
    eng.set_sequences(qs, refs)
    search = lambda: eng.search(W["mat"], W["n"], args.k, **kw)   # noqa: E731
    arms = {"untiled": 0, "tiled": args.tile_refs}
    wall = {a: [] for a in arms}
    res, tim = {}, {}
    for a, t in arms.items():
        eng.set_option("grid_tile_refs", t)
        res[a] = search()
    for _ in range(args.reps):
        for a, t in arms.items():
            eng.set_option("grid_tile_refs", t)
            res[a], ms, tim[a] = timed(search)
            wall[a].append(ms)
    eng.set_option("grid_tile_refs", 0)
    same = all(np.array_equal(x, y) for x, y in zip(res["untiled"][:3], res["tiled"][:3]))
    med = {a: float(np.median(wall[a])) for a in arms}
    c_a = cells(qs, refs)
    emit({"arm": "a", "queries": len(qs), "targets": len(refs), "k": args.k, "tile_refs": args.tile_refs, "identical": same,
          "untiled_ms_median": med["untiled"], "tiled_ms_median": med["tiled"], "untiled_ms": wall["untiled"], "tiled_ms": wall["tiled"],
          "overhead_pct": 100.0 * (med["tiled"] / med["untiled"] - 1.0), "untiled_gcups": c_a / med["untiled"] / 1e6,
          "fill_forward_launches": {a: tim[a]["fill_forward_launches"] for a in arms},
          "other_launches": {a: tim[a]["other_launches"] for a in arms}})

    if "b" not in args.skip:
        Wb = C.config_workload(4, n_queries=10000, n_targets=220000)
        eng.set_sequences(Wb["queries"], Wb["refs"])
        (hr, h, nh, pool), ms, t = timed(lambda: eng.search(W["mat"], W["n"], args.k, **kw))
        c_b = cells(Wb["queries"], Wb["refs"])
        emit({"arm": "b", "queries": len(Wb["queries"]), "targets": len(Wb["refs"]), "pairs": len(Wb["queries"]) * len(Wb["refs"]),
              "k": args.k, "wall_ms": ms, "total_ms": t["total_ms"], "gcups": c_b / ms / 1e6,
              "fill_forward_launches": t["fill_forward_launches"], "other_launches": t["other_launches"],
              "leftover_pairs": t["leftover_pairs"], "byte_overflows": t["byte_overflows"],
              "bytes_to_host": int(hr.nbytes + h.nbytes + nh.nbytes + pool.nbytes), "hits": int(nh.sum())})
        del Wb, hr, h, nh, pool

    if "c" not in args.skip:
        thr = args.all_thr
        if thr <= 0:
            eng.set_sequences(refs[:32], refs)
            thr = int(np.median(eng.search(W["mat"], W["n"], 10, **kw)[1][:, 9]["score1"]))
        eng.set_sequences(refs, refs)
        (row_off, hr, h, pool), ms, t = timed(lambda: eng.search_all(W["mat"], W["n"], thr, **kw))
        emit({"arm": "c", "sequences": len(refs), "pairs": len(refs) ** 2, "min_score": thr, "wall_ms": ms,
              "total_ms": t["total_ms"], "gcups": cells(refs, refs) / ms / 1e6, "hits": int(len(hr)),
              "fill_forward_launches": t["fill_forward_launches"], "leftover_pairs": t["leftover_pairs"],
              "byte_overflows": t["byte_overflows"], "bytes_to_host": int(40 * len(hr) + row_off.nbytes + pool.nbytes)})
        del row_off, hr, h, pool

    if "d" not in args.skip:
        qd = W["queries"][:64]
        eng.set_sequences(qd, refs)
        eng.set_option("grid_min", 2 ** 31 - 1)
        _, ms, t = timed(lambda: eng.search(W["mat"], W["n"], args.k, **kw))
        eng.set_option("grid_min", -1)
        emit({"arm": "d", "queries": len(qd), "targets": len(refs), "k": args.k, "wall_ms": ms, "gcups": cells(qd, refs) / ms / 1e6,
              "leftover_pairs": t["leftover_pairs"]})
    emit({"card_after": card()})
    eng.close()
    if args.out:
        with open(args.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
