#!/usr/bin/env python
"""Freeze the compiled reference's answers that the tests compare against where the reference is not present.

Needs oracle/_ref/libssw_ref.so (built by `make -C oracle` from the reference tree).  Writes:

  oracle_random_ref.json.gz   the reference's record (scores, ends, begins, flag, CIGAR, mark_mismatch count and
                              marked CIGAR) for each of the 2,500 random cases of
                              test_oracle.py::test_oracle_matches_reference_random (null: ssw_align returned NULL);
  parity_full_ref.npz         for every case of test_gpu_parity_full.py, the positions of a fixed, evenly spread sample
                              of its pairs (<case>_idx) and the reference's records and CIGAR words for them
                              (<case>_rec, <case>_pool; oracle/ssw_harness.c record layout).
"""
import gzip
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import common as C  # noqa: E402
import test_gpu_parity_full as F  # noqa: E402
import test_oracle as O  # noqa: E402


def oracle_random():
    ref = C.load_ref()
    rng = np.random.default_rng(O.RANDOM_SEED)
    out = [ref.align(mark=True, **O.random_case(rng)) for _ in range(O.RANDOM_CASES)]
    with gzip.open(os.path.join(HERE, "oracle_random_ref.json.gz"), "wt") as f:
        json.dump(out, f, separators=(",", ":"))


def parity_full():
    arrays = {}
    for key in F.CASES:
        queries, refs, pq, pr, mat, n, kw = F.case_inputs(key)
        idx = F.golden_sample(len(pq), key)
        rec, pool, _, _, kind = C.cpu_batch(queries, refs, pq[idx], pr[idx], mat, n, 3, 1, impl="reference", **kw)
        assert kind == "reference"
        arrays.update({key + "_idx": idx, key + "_rec": rec, key + "_pool": pool})
        print(key, len(idx), "pairs,", len(pool), "CIGAR words")
    np.savez_compressed(os.path.join(HERE, "parity_full_ref.npz"), **arrays)


if __name__ == "__main__":
    if not C.have_ref():
        raise SystemExit("oracle/_ref/libssw_ref.so not built")
    oracle_random()
    parity_full()
