#!/usr/bin/env python
"""Query codes against the same queries as column profiles (PSSMs, P[i][c] = mat[c][q[i]]: the same records), in one run:

    (a) config 4   the 512-query slice of common.config_workload(4) x all 50,000 targets (BLOSUM50, score size 1):
                   search(k) and align of the full grid
    (b) mixed      tests/test_search_mixed.mixed_workload (--mixed-q queries x --mixed-t targets): search(k)

Each arm alternates the code run and the profile run after one warm-up call of each, --reps times, and reports medians of
the wall time to host-resident results; the arrays of the two runs must be identical.  Prints the device's name, power limit
and SM clocks first, then one JSON line per arm.

    python tools/pssm_search_bench.py [--k 10] [--reps 3] [--mixed-q 2000] [--mixed-t 100000] [--out FILE]
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
from test_search_mixed import mixed_workload  # noqa: E402


def col_profiles(queries, mat, n):
    m = np.asarray(mat, np.int8).reshape(n, n)
    return [np.ascontiguousarray(m[:, np.asarray(q, np.int64)].T) for q in queries]


def same(a, b):
    for x, y in zip(a, b):
        if isinstance(x, np.ndarray) and x.dtype.names:
            for f in x.dtype.names:
                if f != "cigar_off" and not np.array_equal(x[f], y[f]):
                    return False
        elif not np.array_equal(x, y):
            return False
    return True


def alternate(eng, queries, profs, refs, mat, n, call, reps):
    """medians of `reps` alternating (codes, profiles) calls after a warm-up of each; asserts identical arrays"""
    t = {"codes": [], "profiles": []}
    out = {}
    for rep in range(reps + 1):
        for arm in ("codes", "profiles"):
            if arm == "codes":
                eng.set_sequences(queries, refs)
            else:
                eng.set_profiles(profs, refs, n)
            t0 = time.perf_counter()
            out[arm] = call(mat if arm == "codes" else None)
            dt = time.perf_counter() - t0
            if rep:
                t[arm].append(dt * 1e3)
        assert same(out["codes"], out["profiles"]), "profile and code arrays differ"
    med = {k: float(np.median(v)) for k, v in t.items()}
    return {"codes_ms": med["codes"], "profiles_ms": med["profiles"], "change_pct": 100.0 * (med["profiles"] / med["codes"] - 1.0),
            "codes_spread_pct": 100.0 * (max(t["codes"]) - min(t["codes"])) / med["codes"],
            "profiles_spread_pct": 100.0 * (max(t["profiles"]) - min(t["profiles"])) / med["profiles"], "identical": True}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--mixed-q", type=int, default=2000)
    ap.add_argument("--mixed-t", type=int, default=100000)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    emit({"card": card()})
    L = _pkg()
    eng = L.BatchAligner(device=0)
    W = C.config_workload(4, n_queries=512)
    kw = dict(gap_open=W["gapO"], gap_extend=W["gapE"], mask_len=W["mask_len"], score_size=W["score_size"])
    profs = col_profiles(W["queries"], W["mat"], 24)
    emit(dict(arm="config4_search", k=args.k, **alternate(eng, W["queries"], profs, W["refs"], W["mat"], 24,
                                                          lambda m: eng.search(m, 24, args.k, **kw), args.reps)))
    emit(dict(arm="config4_align", **alternate(eng, W["queries"], profs, W["refs"], W["mat"], 24,
                                               lambda m: eng.align(m, 24, **kw), args.reps)))
    M = mixed_workload(args.mixed_q, args.mixed_t)
    kwm = dict(gap_open=M["gapO"], gap_extend=M["gapE"], mask_len=M["mask_len"], score_size=M["score_size"])
    profs = col_profiles(M["queries"], M["mat"], 24)
    emit(dict(arm="mixed_search", k=args.k, n_q=args.mixed_q, n_t=args.mixed_t,
              **alternate(eng, M["queries"], profs, M["refs"], M["mat"], 24, lambda m: eng.search(m, 24, args.k, **kwm), args.reps)))
    emit({"card_after": card()})
    eng.close()
    if args.out:
        with open(args.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
