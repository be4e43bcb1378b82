#!/usr/bin/env python
"""Top-k search against full-grid alignment on the BASELINE config-4 workload (common.config_workload(4)), in one run:

    (a) align (every record) vs search (k best per query) on the same queries x all 50,000 targets slice: wall time from the
        call to host-resident results, GCUPS, bytes copied back;
    (b) one search over the full 10,000 x 50,000 grid: wall time, GCUPS, and the device memory the engine holds afterwards
        (free-memory drop from before its sequences were made resident: every buffer it allocated, so an upper bound of
        its largest allocation).

Prints the device's name, power limit and SM clocks first, then one JSON line per measurement.

    python tools/search_bench.py [--slice 512] [--k 10] [--reps 3] [--skip-full] [--out FILE]
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
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as ex:
        return {"error": str(ex)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--slice", type=int, default=512, help="queries of (a), of 10,000")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3, help="timed calls of each kind in (a), after one warm-up call")
    ap.add_argument("--skip-full", action="store_true", help="only (a)")
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
    rl = float(sum(len(r) for r in refs))
    kw = dict(mask_len=W["mask_len"], score_size=W["score_size"])

    # (a) the slice: every record vs the k best
    eng = L.BatchAligner(device=0)
    qs = W["queries"][: args.slice]
    eng.set_sequences(qs, refs)
    cells = float(sum(len(q) for q in qs)) * rl
    keep = {"res": None}

    def do_align():
        res, pool = eng.align(W["mat"], W["n"], W["gapO"], W["gapE"], out=keep["res"], **kw)
        keep["res"] = res
        return res.nbytes + pool.nbytes

    def do_search():
        hr, hits, nh, pool = eng.search(W["mat"], W["n"], args.k, gap_open=W["gapO"], gap_extend=W["gapE"], **kw)
        return hr.nbytes + hits.nbytes + nh.nbytes + pool.nbytes

    for name, fn in (("align", do_align), ("search", do_search)):
        fn()
        walls, dev = [], []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            nbytes = fn()
            walls.append(time.perf_counter() - t0)
            dev.append(eng.timing()["total_ms"])
        w = float(np.median(walls))
        emit({"part": "a", "call": name, "queries": len(qs), "targets": len(refs), "k": args.k if name == "search" else None,
              "wall_ms_median": w * 1e3, "wall_ms": [x * 1e3 for x in walls], "device_total_ms": dev, "gcups": cells / w / 1e9,
              "bytes_to_host": int(nbytes), "byte_overflows": eng.timing()["byte_overflows"]})
    eng.close()
    keep["res"] = None

    # (b) the whole grid in one call
    if not args.skip_full:
        torch.cuda.synchronize()
        free0, total = torch.cuda.mem_get_info(0)
        eng = L.BatchAligner(device=0)
        eng.set_sequences(W["queries"], refs)
        cells = float(sum(len(q) for q in W["queries"])) * rl
        t0 = time.perf_counter()
        hr, hits, nh, pool = eng.search(W["mat"], W["n"], args.k, gap_open=W["gapO"], gap_extend=W["gapE"], **kw)
        wall = time.perf_counter() - t0
        free1, _ = torch.cuda.mem_get_info(0)
        t = eng.timing()
        emit({"part": "b", "call": "search", "queries": len(W["queries"]), "targets": len(refs), "k": args.k, "wall_s": wall,
              "gcups": cells / wall / 1e9, "device_total_ms": t["total_ms"], "fill_forward_launches": t["fill_forward_launches"],
              "byte_overflows": t["byte_overflows"], "engine_device_bytes": int(free0 - free1), "device_total_bytes": int(total),
              "bytes_to_host": int(hr.nbytes + hits.nbytes + nh.nbytes + pool.nbytes), "hits": int(nh.sum()),
              "full_grid_records_bytes": 36 * len(W["queries"]) * len(refs)})
        eng.close()
    if args.out:
        with open(args.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
