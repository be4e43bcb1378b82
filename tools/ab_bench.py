#!/usr/bin/env python
"""A/B of two builds of libssw.so through bench.py: step times, their spreads and the records of every shape.

    python tools/ab_bench.py build [--base REV]           # libssw_base.so (REV, default HEAD) next to libssw.so (working tree)
    python tools/ab_bench.py run [--rounds 3] [--out DIR] -- <bench.py arguments>

`build` needs git: it checks REV out into a temporary worktree, builds its library there and copies it into the package
directory as libssw_base.so, then builds the working tree's libssw.so.  `run` needs only the two libraries: it alternates
`bench.py --lib libssw_base.so` and `bench.py --lib libssw.so` (base first in rounds 0, 2, ..., new first in the others, so
that a drift of the device affects both alike), each with --dump-outputs into its own directory, compares every dumped .npy
of every run with the first base run (then deletes the dumps unless --keep-dumps), and prints per shape the median step
time of each build, the spread of each build ((max - min) / median over its runs) and the change of the medians.  The
bench lines and a summary go to DIR (default: a new temporary directory), each bench line as soon as its run ends.
The exit status is 1 unless every record of every run is identical."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "complete-striped-smith-waterman-library_b200")
BUILDS = (("base", "libssw_base.so"), ("new", "libssw.so"))
SHAPES = ("config3", "config2", "config4", "config5")


def build(args):
    wt = tempfile.mkdtemp(prefix="ssw_ab_base_")
    os.rmdir(wt)
    subprocess.run(["git", "-C", ROOT, "worktree", "add", "--detach", wt, args.base], check=True)
    try:
        pkg = os.path.join(wt, os.path.basename(PKG))
        subprocess.run(["make", "-C", pkg, os.path.join(pkg, "libssw.so")], check=True)
        shutil.copy2(os.path.join(pkg, "libssw.so"), os.path.join(PKG, "libssw_base.so"))
    finally:
        subprocess.run(["git", "-C", ROOT, "worktree", "remove", "--force", wt], check=False)
    subprocess.run(["make", "-C", PKG, os.path.join(PKG, "libssw.so")], check=True)
    print("built %s (%s) and %s (working tree)" % (BUILDS[0][1], args.base, BUILDS[1][1]))


def shape_numbers(line):
    """{shape: (ms_per_step, GCUPS)} of one bench line"""
    out = {"config3": (line["ms_per_step"], line["value"])}
    for s in SHAPES[1:]:
        if s in line:
            out[s] = (line[s]["ms_per_step"], line[s]["value"])
    return out


def same_dumps(a, b):
    """names of the .npy files that differ between two dump directories (missing on either side counts)"""
    fa, fb = set(os.listdir(a)), set(os.listdir(b))
    bad = sorted(fa ^ fb)
    for f in sorted(fa & fb):
        x, y = np.load(os.path.join(a, f)), np.load(os.path.join(b, f))
        if x.shape != y.shape or not np.array_equal(x, y, equal_nan=True):
            bad.append(f)
    return bad


def run(args, bench_args):
    for _, lib in BUILDS:
        if not os.path.exists(os.path.join(PKG, lib)):
            raise SystemExit("ab_bench: %s missing (run `ab_bench.py build` first)" % lib)
    out = args.out or tempfile.mkdtemp(prefix="ssw_ab_")
    os.makedirs(out, exist_ok=True)
    runs = []          # (build, round, dump dir, bench line)
    for r in range(args.rounds):
        for name, lib in (BUILDS if r % 2 == 0 else BUILDS[::-1]):
            dump = os.path.join(out, "%s_r%d" % (name, r))
            cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--lib", lib, "--dump-outputs", dump] + bench_args
            print("ab_bench: round %d, %s: %s" % (r, name, " ".join(cmd[1:])), flush=True)
            p = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, text=True)
            if p.returncode != 0:
                raise SystemExit("ab_bench: bench.py failed (%d) for %s" % (p.returncode, name))
            line = json.loads(p.stdout.strip().splitlines()[-1])
            with open(os.path.join(out, "%s_r%d.json" % (name, r)), "w") as f:
                f.write(json.dumps(line) + "\n")
            runs.append((name, r, dump, line))
    first = next(d for n, _, d, _ in runs if n == "base")
    diffs = {"%s_r%d" % (n, r): same_dumps(first, d) for n, r, d, _ in runs if d != first}
    summary = {"rounds": args.rounds, "bench_args": bench_args, "shapes": {}, "records_identical": all(not v for v in diffs.values()),
               "record_diffs": {k: v for k, v in diffs.items() if v}}
    for s in SHAPES:
        per = {}
        for name, _ in BUILDS:
            ms = [shape_numbers(l)[s][0] for n, _, _, l in runs if n == name and s in shape_numbers(l)]
            gc = [shape_numbers(l)[s][1] for n, _, _, l in runs if n == name and s in shape_numbers(l)]
            if ms:
                med = float(np.median(ms))
                per[name] = {"ms_per_step": ms, "median_ms": med, "spread": (max(ms) - min(ms)) / med, "median_gcups": float(np.median(gc))}
        if len(per) == 2:
            per["change"] = per["new"]["median_ms"] / per["base"]["median_ms"] - 1.0
            summary["shapes"][s] = per
    for key in ("byte_overflows", "mismatches"):
        summary[key] = {"%s_r%d" % (n, r): (l[key] if key in l else None) for n, r, _, l in runs}
    summary["fill_launches_per_step_per_rank"] = {"%s_r%d" % (n, r): l["roofline"]["kernel_launches_per_step_per_rank"] for n, r, _, l in runs}
    summary["clocks"] = {"%s_r%d" % (n, r): l.get("clocks") for n, r, _, l in runs}
    with open(os.path.join(out, "ab_summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    if not args.keep_dumps:
        for _, _, d, _ in runs:
            shutil.rmtree(d, ignore_errors=True)
    print("%-8s %12s %8s %12s %8s %8s" % ("shape", "base ms", "spread", "new ms", "spread", "change"))
    for s, per in summary["shapes"].items():
        print("%-8s %12.1f %7.2f%% %12.1f %7.2f%% %+7.2f%%" % (s, per["base"]["median_ms"], 100 * per["base"]["spread"], per["new"]["median_ms"],
                                                         100 * per["new"]["spread"], 100 * per["change"]))
    print("records identical across all runs:", summary["records_identical"], "" if summary["records_identical"] else summary["record_diffs"])
    print("summary:", os.path.join(out, "ab_summary.json"))
    return 0 if summary["records_identical"] else 1


def main():
    argv = sys.argv[1:]
    bench_args = []
    if "--" in argv:
        k = argv.index("--")
        argv, bench_args = argv[:k], argv[k + 1:]
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="cmd", required=True)
    b = sub.add_parser("build")
    b.add_argument("--base", default="HEAD", help="revision of the base build (default HEAD: the working tree's changes against it)")
    r = sub.add_parser("run")
    r.add_argument("--rounds", type=int, default=3, help="runs of each build")
    r.add_argument("--out", default=None, help="directory of the dumps, bench lines and ab_summary.json")
    r.add_argument("--keep-dumps", action="store_true", help="keep the dumped records (config 4's alone are tens of MB per run)")
    args = ap.parse_args(argv)
    if args.cmd == "build":
        build(args)
        return 0
    return run(args, bench_args)


if __name__ == "__main__":
    sys.exit(main())
