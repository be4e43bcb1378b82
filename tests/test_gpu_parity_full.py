"""Parity at the sizes SURVEY 8(d) asks for, against the compiled reference:
  config 2: all 1,000 reads x 5 Mbp, flag 0x0f (scores, ends, begins, flag, CIGAR) and flag 0;
  config 3: a fixed 2,000-read subsample of the 100,000-read set;
  config 4: a 200 x 1,000 sub-grid of the protein grid, word scores;
  config 5: 1,000 x 10 kbp long reads, flags 0x0f and 2, every field and every CIGAR word.
Every case is checked against the reference's answers for a fixed sample of its pairs, frozen in
tests/golden/parity_full_ref.npz (tests/golden/make_reference_golden.py).  Where the compiled reference
(oracle/_ref/libssw_ref.so) is present, EVERY pair is also re-computed by it on all usable host cores (~1e12 cells per
case, tens of seconds) and compared; the coverage is printed to stdout."""
import json
import os
import time

import numpy as np
import pytest

import common as C
from test_gpu_parity import FIELDS8, batch_dict, engine  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

THREADS = C.effective_cores()[0]
GOLDEN_NPZ = os.path.join(C.GOLDEN, "parity_full_ref.npz")


_cache = {}


def _workload(ref_len, n_reads, read_len, seed_ref, seed_reads, **kw):
    key = (ref_len, n_reads, read_len, seed_ref, seed_reads, tuple(sorted(kw.items())))
    if key not in _cache:
        _cache[key] = C.make_dna_workload(ref_len, n_reads, read_len, seed_ref=seed_ref, seed_reads=seed_reads, **kw)
    return _cache[key]


CASES = ("config2_flag15", "config2_flag0", "config3", "config4_subgrid", "config4_launch_groups", "config5_flag15", "config5_flag2")


def case_inputs(key):
    """(queries, refs, pair_q, pair_r, mat, n, kw) of one case; gap open 3 / extend 1 throughout, kw = the other
    ssw_align parameters."""
    if key.startswith("config2_flag"):
        ref, reads = _workload(5_000_000, 1000, 150, 1001, 2002)
        kw = dict(flag=int(key[len("config2_flag"):]), filters=0, filterd=32767, mask_len=75, score_size=2)
    elif key == "config3":
        ref, reads = _workload(5_000_000, 2000, 150, 1001, 3003)
        kw = dict(flag=0, filters=0, filterd=0, mask_len=75, score_size=2)
    elif key.startswith("config5_flag"):
        ref, reads = _workload(100_000, 1000, 10_000, 5005, 5006, decoy_frac=0.0, p_sub=0.05, p_ins=0.02, p_del=0.02)
        kw = dict(flag=int(key[len("config5_flag"):]), filters=0, filterd=32767, mask_len=5000, score_size=2)
    else:
        nq, nt = {"config4_subgrid": (200, 1000), "config4_launch_groups": (96, 50_000)}[key]
        W = C.config_workload(4, n_queries=nq, n_targets=nt)
        kw = dict(flag=0, filters=0, filterd=0, mask_len=150, score_size=1)
        return W["queries"], W["refs"], np.repeat(np.arange(nq), nt), np.tile(np.arange(nt), nq), C.BLOSUM50, 24, kw
    n = len(reads)
    return reads, [ref], np.arange(n), np.zeros(n, dtype=np.int64), C.dna_matrix(2, 2), 5, kw


def golden_sample(n_pairs, key):
    """Positions of the pairs whose reference records are frozen: evenly spread over the whole pair list."""
    k = 32 if key.startswith("config5") else 2000 if key.startswith("config4") else 250
    return np.unique(np.linspace(0, n_pairs - 1, min(k, n_pairs)).astype(np.int64))


_expected = {}


def check_all(key, capfd, res, pool, name=None):
    """The frozen sample, then (compiled reference present) EVERY pair re-computed by the reference on all usable host
    cores (pthread harness), compared field by field and CIGAR word by CIGAR word; the coverage goes to stdout."""
    queries, refs, pair_q, pair_r, mat, n, kw = case_inputs(key)
    assert len(res) == len(pair_q)
    with np.load(GOLDEN_NPZ) as g:
        idx, exp, exp_pool = g[key + "_idx"], g[key + "_rec"], g[key + "_pool"]
    assert np.array_equal(idx, golden_sample(len(pair_q), key))
    bad = C.compare_records(res, pool, exp, exp_pool, idx=idx)
    info = {"pairs_total": int(len(pair_q)), "golden_pairs_checked": int(len(idx)), "golden_mismatches": len(bad)}
    assert bad == [], (bad[:3], [(res[idx[i]], exp[i]) for i in bad[:2]])
    if C.have_ref():
        t0 = time.time()
        if _expected.get("key") != key:
            _expected.clear()
            _expected["key"] = key
            _expected["value"] = C.cpu_batch(queries, refs, pair_q, pair_r, mat, n, 3, 1, impl="reference", threads=THREADS, **kw)
        exp, exp_pool, secs, cells, kind = _expected["value"]
        bad = C.compare_records(res, pool, exp, exp_pool)
        info.update({"pairs_checked": int(len(exp)), "mismatches": len(bad), "threads": THREADS,
                     "seconds": round(time.time() - t0, 1), "checker": kind, "checker_gcups": round(cells / secs / 1e9, 1)})
        assert len(exp) == len(pair_q)
        assert bad == [], (bad[:3], [(res[i], exp[i]) for i in bad[:2]])
    with capfd.disabled():
        print("\n[parity %s] %s" % (name or key, json.dumps(info)))


def _align(engine, key):
    queries, refs, _, _, mat, n, kw = case_inputs(key)
    engine.set_sequences(queries, refs)
    return engine.align(mat, n, 3, 1, **kw)


@pytest.mark.parametrize("flag", [0x0f, 0])
def test_config2_all_reads(engine, flag, capfd):
    key = "config2_flag%d" % flag
    res, pool = _align(engine, key)
    check_all(key, capfd, res, pool)


@pytest.mark.parametrize("mode", ["auto", "blocks_3_launches", "columns_3_launches"])
def test_config3_subsample(engine, mode, capfd):
    """the first 2,000 reads of the 100,000-read set of config 3 (seed 3003; the generator is sequential): in one launch
    (automatic: block column maxima), and forced through >= 3 launches by a capped column-maximum budget in both storage
    modes -- the multi-launch path the full 100,000-read batch takes."""
    if mode == "blocks_3_launches":
        engine.set_option("cm_block", 1)
        engine.set_option("cm_budget_mb", 110)           # 1,000 pair-tasks x 312 KB of block maxima = 312 MB
    elif mode == "columns_3_launches":
        engine.set_option("cm_block", 0)
        engine.set_option("cm_budget_mb", 7000)          # 1,000 pair-tasks x 20 MB of column maxima = 20 GB
    try:
        res, pool = _align(engine, "config3")
        launches = engine.timing()["fill_forward_launches"]
    finally:
        engine.set_option("cm_block", -1)
        engine.set_option("cm_budget_mb", 0)
    if mode != "auto":
        assert launches >= 4, launches                   # >= 3 byte-semantics launches + the word re-fill of the overflows
    check_all("config3", capfd, res, pool, name="config3_subsample_" + mode)


def test_config4_subgrid(engine, capfd):
    """200 queries x 1,000 targets of the BLOSUM50 grid (seeds 4004 / 4005), word scores, through the grid path"""
    res, pool = _align(engine, "config4_subgrid")
    check_all("config4_subgrid", capfd, res, pool)


def test_config4_grid_in_launch_groups(engine, capfd):
    """96 queries x 50,000 targets = 4.8 M pairs: large enough for the device-planned grid to run as several launch groups whose
    records are copied back while the next group computes; every pair against the compiled reference."""
    res, pool = _align(engine, "config4_launch_groups")
    assert engine.timing()["fill_forward_launches"] >= 3
    check_all("config4_launch_groups", capfd, res, pool)


@pytest.mark.parametrize("flag", [0x0f, 2])
def test_config5_all_long_reads(engine, flag, capfd):
    key = "config5_flag%d" % flag
    res, pool = _align(engine, key)
    assert int((res["cigar_len"] > 0).sum()) == len(res)
    check_all(key, capfd, res, pool)
