#!/usr/bin/env python
"""Threshold search against top-k search and full-grid alignment on a slice of the BASELINE config-4 workload
(common.config_workload(4): BLOSUM50, score_size 1, mask_len 150), in one run:

    align            every record of the slice x all 50,000 targets
    search           the k best per query (--k, default 10)
    search_all@N     every hit at or above the N-th best score (N = 10, 100, 1,000), the threshold being the median of the
                     N-th best scores of a sample of queries (--sample, taken from outside the slice)

The arms alternate within each of --reps rounds (after one warm-up call of each); for each arm the medians of the wall time
of the call (to host-resident results), the engine's total_ms and resolve_ms are reported, with the hit count and the bytes
the call copies to the host (records 36 B, hits 36 + 4 B, plus the per-query counts).  Prints the device's name, power limit
and SM clock first, then one JSON line per arm.

    python tools/search_all_bench.py [--slice 512] [--k 10] [--reps 3] [--sample 32] [--out FILE]
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import common as C  # noqa: E402


def _pkg():
    spec = importlib.util.spec_from_file_location("ssw_b200_lib", os.path.join(C.PKG, "ssw_lib.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as ex:
        return {"error": str(ex)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--slice", type=int, default=512, help="queries of the slice, of 10,000")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3, help="rounds; every arm runs once per round")
    ap.add_argument("--sample", type=int, default=32, help="queries whose N-th best scores set the thresholds")
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

    # thresholds: the 10th, 100th and 1,000th best scores of a sample of queries from outside the slice
    sample = W["queries"][-args.sample:]
    eng.set_sequences(sample, refs)
    _, hits, n_hits, _ = eng.search(W["mat"], W["n"], 1000, **kw)
    assert (n_hits == 1000).all()
    thr = {n: int(np.median(hits[:, n - 1]["score1"])) for n in (10, 100, 1000)}
    emit({"thresholds": thr, "sample_queries": len(sample)})

    qs = W["queries"][: args.slice]
    eng.set_sequences(qs, refs)
    nq = len(qs)
    keep = {"res": None}

    def do_align():
        res, pool = eng.align(W["mat"], W["n"], W["gapO"], W["gapE"], out=keep["res"], mask_len=W["mask_len"], score_size=W["score_size"])
        keep["res"] = res
        return len(res), res.nbytes + pool.nbytes

    def do_search():
        hr, h, nh, pool = eng.search(W["mat"], W["n"], args.k, **kw)
        return int(nh.sum()), hr.nbytes + h.nbytes + nh.nbytes + pool.nbytes

    def do_all(n):
        def fn():
            row_off, hr, h, pool = eng.search_all(W["mat"], W["n"], thr[n], **kw)
            return len(hr), 40 * len(hr) + 4 * nq + pool.nbytes
        return fn

    arms = [("align", do_align), ("search", do_search)] + [("search_all@%d" % n, do_all(n)) for n in (10, 100, 1000)]
    stats = {name: {"wall": [], "total": [], "resolve": []} for name, _ in arms}
    out = {}
    for name, fn in arms:
        fn()
    for _ in range(args.reps):
        for name, fn in arms:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n, nbytes = fn()
            wall = time.perf_counter() - t0
            t = eng.timing()
            s = stats[name]
            s["wall"].append(wall * 1e3); s["total"].append(t["total_ms"]); s["resolve"].append(t["resolve_ms"])
            out[name] = (n, nbytes, t)
    for name, _ in arms:
        n, nbytes, t = out[name]
        s = stats[name]
        emit({"call": name, "queries": nq, "targets": len(refs), "min_score": thr.get(int(name.split("@")[1])) if "@" in name else None,
              "k": args.k if name == "search" else None, "wall_ms_median": float(np.median(s["wall"])), "wall_ms": s["wall"],
              "total_ms_median": float(np.median(s["total"])), "resolve_ms_median": float(np.median(s["resolve"])),
              "hits" if name != "align" else "records": int(n), "bytes_to_host": int(nbytes),
              "fill_forward_launches": t["fill_forward_launches"], "other_launches": t["other_launches"],
              "byte_overflows": t["byte_overflows"], "leftover_pairs": t["leftover_pairs"]})
    emit({"card_after": card()})
    eng.close()
    if args.out:
        with open(args.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
