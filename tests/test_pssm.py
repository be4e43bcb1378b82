"""Query profiles (PSSMs): ssw_engine_set_sequences_pssm and the align / search / search_all calls that take params->mat == NULL.

Definition (include/ssw_batch.h): the record of a profile P of L rows over n letters against a reference is what the reference
returns for ssw_init(read = {0, .., L-1}, mat = M, N = max(L, n)) + ssw_align, with M[c * N + i] = P[i][c] and 0 elsewhere.
Read codes are int8, so that construction reaches 128 rows; a profile of any length whose rows take at most 128 distinct values
is the same construction over the distinct rows (read = the index of each row's value), which the checkers take directly.

The checker is the compiled reference where it is present and the oracle port otherwise (C.cpu_batch's choice; the port is
pinned to the reference by test_oracle.py).  Identity cases compare a profile made of a code query's matrix columns with the
code query itself, field for field including every CIGAR word.  Every case runs on the CPU emulator build and, marked gpu, on the
CUDA library."""
import numpy as np
import pytest

import common as C
from test_search import NEVER_GRID, _engine
from test_search_all import reset
from test_search_mixed import FWD_INST

DNA = C.dna_matrix(2, 2)


def col_profile(q, mat, n):
    """P[i][c] = mat[c * n + q[i]]: the profile that scores exactly as the code query q"""
    return np.ascontiguousarray(np.asarray(mat, np.int8).reshape(n, n)[:, np.asarray(q, np.int64)].T)


def same_records(a, pa, b, pb):
    """every field of two record arrays (and every CIGAR word) is equal"""
    assert a.shape == b.shape
    for f in a.dtype.names:
        if f != "cigar_off":
            assert np.array_equal(a[f], b[f]), f
    for x, y in zip(a.reshape(-1), b.reshape(-1)):
        assert list(pa[x["cigar_off"]: x["cigar_off"] + x["cigar_len"]]) == list(pb[y["cigar_off"]: y["cigar_off"] + y["cigar_len"]])


def same_search(a, b):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2])
    same_records(a[1], a[3], b[1], b[3])


def same_all(a, b):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    same_records(a[2], a[3], b[2], b[3])


def distinct_rows(P):
    """(read codes, matrix M, N) of the construction for one profile whose rows take at most 128 values: read = the index of
    each row's value among the distinct rows, N = max(distinct rows, n)"""
    n = P.shape[1]
    uniq, inv = np.unique(P, axis=0, return_inverse=True)
    assert len(uniq) <= 128
    N = max(len(uniq), n)
    M = np.zeros((N, N), np.int8)
    M[:n, : len(uniq)] = uniq.T
    return inv.reshape(-1).astype(np.int8), M.reshape(-1), N


def checker_records(profiles, refs, pq, pr, **kw):
    """the checker's records of pairs (pq[i], pr[i]) through the construction (one matrix per profile)"""
    pq, pr = np.asarray(pq), np.asarray(pr)
    exp = np.zeros(len(pq), dtype=C.HARNESS_DTYPE)
    pools = []
    used = 0
    for q in np.unique(pq):
        sel = np.nonzero(pq == q)[0]
        read, M, N = distinct_rows(profiles[q])
        e, pool, _, _, _ = C.cpu_batch([read], refs, np.zeros(len(sel), np.int32), pr[sel], M, N, threads=4, **kw)
        e["cigar_off"] = np.where(e["cigar_off"] >= 0, e["cigar_off"] + used, e["cigar_off"])
        exp[sel] = e
        pools.append(pool)
        used += len(pool)
    return exp, np.concatenate(pools) if pools else np.zeros(0, np.uint32)


def check_vs_checker(got, gp, exp, ep):
    bad = C.compare_records(got, gp, exp, ep)
    assert bad == [], [(i, got[i], exp[i]) for i in bad[:3]]
    # status 1 exactly where the checker's ssw_align returned NULL
    assert np.array_equal(got["status"], exp["status"])


def dna_reads(lens, ref, seed):
    rng = np.random.default_rng(seed)
    out = []
    for L in lens:
        a = int(rng.integers(0, len(ref) - L - L // 3 - 1))
        out.append(C.mutate_read(rng, ref, a, L, 0.1, 0.01, 0.01))
    return out


def random_profiles(rng, lens, refs, n, lo=-8, hi=8, plant=6, distinct=None):
    """seeded scores in lo .. hi with a planted high-scoring segment (the profile rows along a stretch of a reference score
    `plant` more on its letters); distinct: rows drawn from a pool of that many (longer profiles, for the construction)"""
    out = []
    for L in lens:
        if distinct:
            pool = rng.integers(lo, hi + 1, size=(distinct, n)).astype(np.int16)
            P = pool[rng.integers(0, distinct, size=L)]
        else:
            P = rng.integers(lo, hi + 1, size=(L, n)).astype(np.int16)
        r = refs[int(rng.integers(0, len(refs)))]
        seg = min(L, len(r), int(rng.integers(L // 3, L + 1)))
        i0, j0 = int(rng.integers(0, L - seg + 1)), int(rng.integers(0, len(r) - seg + 1))
        if distinct:                    # n planted rows more: row c scores `plant` on letter c
            planted = np.tile(pool[0], (n, 1))
            planted[np.arange(n), np.arange(n)] += plant
            P[i0: i0 + seg] = planted[r[j0: j0 + seg]]
        else:
            for i in range(seg):
                P[i0 + i, r[j0 + i]] += plant
        out.append(np.clip(P, -128, 127).astype(np.int8))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# cases (each runs on the emulator build and on the GPU)
# ---------------------------------------------------------------------------------------------------------------------

def case_identity_lengths(gpu):
    """column profiles of DNA reads at every row boundary of the forward instances and above 640 rows (strip kernel), score
    sizes 0, 1, 2 (every query holds a letter whose column has the matrix minimum -2, so the byte biases agree), flags 0, 0x08,
    0x0f: the records of the code queries"""
    L, eng = _engine(gpu)
    rng = np.random.default_rng(71)
    ref = rng.integers(0, 4, size=2600).astype(np.int8)
    rows = sorted({G * R for G, R in FWD_INST})
    lens = sorted({x for r in rows for x in (r, r + 1)} | {700, 1000})
    if not gpu:
        lens = [lens[0], 152, 153, 304, 321, 641, 700]
    reads = dna_reads(lens, ref, 72)
    refs = [ref, ref[300:1400]]
    prof = [col_profile(q, DNA, 5) for q in reads]
    for ss in (0, 1, 2):
        for flag in ((0, 0x08, 0x0f) if ss == 2 else (0x0f,)):
            eng.set_sequences(reads, refs)
            a = eng.align(DNA, 5, flag=flag, score_size=ss)
            eng.set_profiles(prof, refs, 5)
            same_records(*eng.align(None, 5, flag=flag, score_size=ss), *a)
    eng.close()


def case_identity_modes(gpu):
    """cm_block 0 / 1 / 2 over chunked references, gapO <= gapE (lane-literal kernel), and the CIGAR of every traceback kernel
    (tb_spec side by side and one after the other, tb_maxbw 0: the global-memory kernel)"""
    L, eng = _engine(gpu)
    rng = np.random.default_rng(73)
    ref = rng.integers(0, 4, size=6000 if gpu else 2400).astype(np.int8)
    reads = dna_reads([150, 151, 300, 96] * (4 if gpu else 1), ref, 74)
    prof = [col_profile(q, DNA, 5) for q in reads]
    runs = [dict(opts={"cm_block": cb, "chunk": 512}, kw={}) for cb in (0, 1, 2)]
    runs += [dict(opts={}, kw=dict(gap_open=1, gap_extend=1)), dict(opts={}, kw=dict(gap_open=2, gap_extend=2, flag=0x0f))]
    runs += [dict(opts={"tb_spec": s, "tb_maxbw": bw}, kw=dict(flag=0x0f)) for s in (0, 1) for bw in (0, -1)]
    for run in runs:
        for name, v in run["opts"].items():
            eng.set_option(name, v)
        for ss in (2, 0):
            eng.set_sequences(reads, [ref])
            a = eng.align(DNA, 5, score_size=ss, **run["kw"])
            eng.set_profiles(prof, [ref], 5)
            same_records(*eng.align(None, 5, score_size=ss, **run["kw"]), *a)
        reset(eng, *run["opts"])
    eng.close()


def case_identity_grid(gpu):
    """grid align, top-k and threshold search over grid tiles, with re-dos (byte overflows at score size 2), a query above 640
    rows and references above grid_max_ref left over: the arrays of the code queries"""
    L, eng = _engine(gpu)
    rng = np.random.default_rng(75)
    refs = [rng.integers(0, 4, size=int(x)).astype(np.int8) for x in rng.integers(120, 400, size=24 if gpu else 9)]
    reads = []
    for i in range(10 if gpu else 5):
        r = refs[i % len(refs)]
        reads.append(C.mutate_read(rng, r, 0, min(len(r) - 10, 150 + 20 * i), 0.05, 0.01, 0.01))
    reads.append(np.concatenate([refs[0], refs[1], refs[2]])[:660])          # above 640 rows: off the grid
    prof = [col_profile(q, DNA, 5) for q in reads]
    eng.set_option("grid_min", 1)
    eng.set_option("grid_max_ref", 350)
    for ss in (2, 0, 1):
        for tile in (0, 4):
            eng.set_option("grid_tile_refs", tile)
            eng.set_sequences(reads, refs)
            a = eng.align(DNA, 5, score_size=ss)
            s = eng.search(DNA, 5, 3, score_size=ss)
            t_seq = eng.timing()
            h = eng.search_all(DNA, 5, 40, score_size=ss)
            eng.set_profiles(prof, refs, 5)
            same_records(*eng.align(None, 5, score_size=ss), *a)
            same_search(eng.search(None, 5, 3, score_size=ss), s)
            t = eng.timing()
            assert t["leftover_pairs"] == t_seq["leftover_pairs"] > 0
            assert t["byte_overflows"] == t_seq["byte_overflows"]
            if ss == 2:
                assert t["byte_overflows"] > 0
            same_all(eng.search_all(None, 5, 40, score_size=ss), h)
    reset(eng, "grid_min", "grid_max_ref", "grid_tile_refs")
    eng.close()


def case_random_vs_checker(gpu):
    """random profiles (up to 128 rows; scores -8 .. 8 with planted segments, one with min >= 0 = bias 0, some that overflow a
    byte) against the checker through the construction, score sizes 0, 1, 2 and flag 0x0f, mask_len L/2 and 15"""
    L, eng = _engine(gpu)
    rng = np.random.default_rng(77)
    n = 20
    refs = [rng.integers(0, n, size=int(x)).astype(np.int8) for x in (300, 500, 180)]
    lens = [int(x) for x in rng.integers(10, 129, size=12 if gpu else 6)]
    prof = random_profiles(rng, lens, refs, n)
    prof.append(random_profiles(rng, [60], refs, n, lo=0, hi=3, plant=2)[0])           # min >= 0: bias 0, every cell scores
    prof.append(random_profiles(rng, [120], refs, n, lo=-8, hi=2, plant=8)[0])         # planted 120 x ~8: overflows a byte
    assert prof[-2].min() >= 0
    eng.set_profiles(prof, refs, n)
    pq, pr = np.repeat(np.arange(len(prof)), len(refs)), np.tile(np.arange(len(refs)), len(prof))
    for ss in (0, 1, 2):
        for mask in (-1, 15):
            got, gp = eng.align(None, n, flag=0x0f, score_size=ss, mask_len=mask, pair_query=pq, pair_ref=pr)
            exp, ep = checker_records(prof, refs, pq, pr, flag=0x0f, score_size=ss, mask_len=mask)
            check_vs_checker(got, gp, exp, ep)
            if ss == 0:
                assert got["status"].sum() > 0                                   # the byte overflows are there
    eng.close()


def case_per_query_bias(gpu):
    """two queries of one pair-task (same reference, same kernel instance) with biases 0 and 8 that both score 250: at score
    sizes 0 and 2 exactly one overflows the byte (limit 255 vs 247); on the general path and on the device-planned grid"""
    L, eng = _engine(gpu)
    rng = np.random.default_rng(79)
    n = 8
    ref = rng.integers(0, n, size=200).astype(np.int8)
    A = np.zeros((50, n), np.int8)
    for i in range(50):
        A[i, ref[40 + i]] = 5
    B = A.copy()
    B[0, (ref[40] + 1) % n] = -8                    # bias 8; the diagonal still scores 50 x 5 = 250
    prof = [A, B]
    eng.set_profiles(prof, [ref], n)
    for grid in (NEVER_GRID, 1):
        eng.set_option("grid_min", grid)
        for ss in (0, 2, 1):
            got, gp = eng.align(None, n, score_size=ss)
            exp, ep = checker_records(prof, [ref], [0, 1], [0, 0], score_size=ss)
            check_vs_checker(got, gp, exp, ep)
            if ss == 0:
                assert list(got["status"]) == [0, 1] and int(got["score1"][0]) == 250
            else:
                assert list(got["score1"]) == [250, 250]
            if ss == 2:
                assert eng.timing()["byte_overflows"] == 1
    reset(eng, "grid_min")
    eng.close()


def case_long_profiles(gpu):
    """profiles of 300 .. 1,500 rows (the strip kernel above 640) whose rows take at most 128 values, against the checker
    through the construction over the distinct rows, flag 0x0f, score sizes 2 and 1"""
    L, eng = _engine(gpu)
    rng = np.random.default_rng(81)
    n = 20
    refs = [rng.integers(0, n, size=x).astype(np.int8) for x in ((1800, 900) if gpu else (900,))]
    lens = (300, 700, 1100, 1500) if gpu else (660, 300)
    prof = random_profiles(rng, lens, refs, n, lo=-4, hi=3, plant=5, distinct=48)
    eng.set_profiles(prof, refs, n)
    pq, pr = np.repeat(np.arange(len(prof)), len(refs)), np.tile(np.arange(len(refs)), len(prof))
    for ss in (2, 1):
        got, gp = eng.align(None, n, flag=0x0f, score_size=ss, pair_query=pq, pair_ref=pr)
        exp, ep = checker_records(prof, refs, pq, pr, flag=0x0f, score_size=ss)
        check_vs_checker(got, gp, exp, ep)
        assert int(got["score1"].max()) > 255
    eng.close()


def case_arguments(gpu):
    """the ABI's rules: a matrix while profiles are resident, NULL while sequences are, another n, mark_mismatch, n outside
    1 .. 64; and sequences set after profiles give today's records on the same engine"""
    L, eng = _engine(gpu)
    rng = np.random.default_rng(83)
    ref = rng.integers(0, 4, size=500).astype(np.int8)
    reads = dna_reads([100, 120], ref, 84)
    prof = [col_profile(q, DNA, 5) for q in reads]
    eng.set_sequences(reads, [ref])
    a = eng.align(DNA, 5, flag=0x0f)
    with pytest.raises(RuntimeError):
        eng.align(None, 5)
    eng.set_profiles(prof, [ref], 5)
    for call in (lambda: eng.align(DNA, 5), lambda: eng.align(None, 4), lambda: eng.search(DNA, 5, 2), lambda: eng.search(None, 6, 2),
                 lambda: eng.search_all(DNA, 5, 1), lambda: eng.search_all(None, 3, 1)):
        with pytest.raises(RuntimeError):
            call()
    b = eng.align(None, 5, flag=0x0f)
    same_records(*b, *a)
    with pytest.raises(RuntimeError):
        eng.mark_mismatch(*b)
    for bad_n in (0, 65):
        with pytest.raises(RuntimeError):
            eng.set_profiles([np.zeros((4, max(bad_n, 1)), np.int8)], [ref], bad_n)
    eng.set_sequences(reads, [ref])
    same_records(*eng.align(DNA, 5, flag=0x0f), *a)
    eng.mark_mismatch(*a)
    eng.set_profiles(prof, [ref], 5)
    same_records(*eng.align(None, 5, flag=0x0f), *a)
    eng.close()


CASES = [case_identity_lengths, case_identity_modes, case_identity_grid, case_random_vs_checker, case_per_query_bias,
         case_long_profiles, case_arguments]


def test_pssm_entry_point_declared_and_exported():
    import os
    with open(os.path.join(C.ROOT, "include", "ssw_batch.h")) as f:
        assert "int ssw_engine_set_sequences_pssm(" in f.read()
    import ctypes as ct
    import subprocess
    from test_search import EMU_DIR
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    assert hasattr(ct.CDLL(os.path.join(EMU_DIR, "libssw_emu.so")), "ssw_engine_set_sequences_pssm")


@pytest.mark.parametrize("case", CASES, ids=lambda f: f.__name__[5:])
def test_pssm_emulated(case, capfd):
    case(False)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda f: f.__name__[5:])
def test_pssm_gpu(case, capfd):
    case(True)


@pytest.mark.gpu
def test_pssm_config4_scale(capfd):
    """the config-4 slice (512 x 50,000, BLOSUM50, score size 1) as column profiles: search (k = 10), search_all and an align
    sample with CIGARs give the arrays of the code queries"""
    w = C.config_workload(4, n_queries=512, n_targets=50_000)
    L, eng = _engine(True)
    eng.set_option("latency_cols", -1)
    kw = dict(gap_open=w["gapO"], gap_extend=w["gapE"], mask_len=w["mask_len"], score_size=w["score_size"])
    rng = np.random.default_rng(85)
    pq = rng.integers(0, 512, size=2000).astype(np.int32)
    pr = rng.integers(0, 50_000, size=2000).astype(np.int32)
    eng.set_sequences(w["queries"], w["refs"])
    s = eng.search(w["mat"], 24, 10, **kw)
    h = eng.search_all(w["mat"], 24, 100, **kw)
    a = eng.align(w["mat"], 24, flag=0x0f, pair_query=pq, pair_ref=pr, **kw)
    eng.set_profiles([col_profile(q, w["mat"], 24) for q in w["queries"]], w["refs"], 24)
    same_search(eng.search(None, 24, 10, **kw), s)
    assert eng.timing()["leftover_pairs"] == 0
    same_all(eng.search_all(None, 24, 100, **kw), h)
    same_records(*eng.align(None, 24, flag=0x0f, pair_query=pq, pair_ref=pr, **kw), *a)
    assert len(h[1]) > 512
    eng.close()
