"""Threshold search (ssw_engine_search_all / ssw_group_search_all): every hit of the full queries x references grid, as a CSR
matrix in pair order.

The expected output is the checker's full grid (C.cpu_batch: the compiled reference where present, the oracle port otherwise)
with the non-hits removed: a hit has status 1 or score1 >= max(min_score, 1).  Row offsets, reference indices, every field and
every CIGAR word are compared.  The grid path (count and compaction on the device) and the general path are forced on the same
inputs and must give identical arrays; launch groups, arming, the rejected pilot group, leftover pairs and device groups are
covered.  What ran where is asserted from the counters of ssw_engine_timing.  The cases run on the CPU emulator build and,
marked gpu, on the CUDA library."""
import ctypes as ct
import os

import numpy as np
import pytest

import common as C
from test_search import NEVER_GRID, EMU_DIR, _engine, _group, dna_grid, grid_records, tie_grid
from test_search_mixed import PROT, small_grid


def hit_mask(exp, min_score):
    return (exp["status"] == 1) | (exp["score1"] >= max(min_score, 1))


def check_all(got, exp, exp_pool, n_q, n_r, min_score):
    """search_all output against the checker grid filtered by the hit rule, in pair order; returns the number of hits"""
    row_off, hit_ref, hits, pool = got
    idx = np.nonzero(hit_mask(exp, min_score))[0]
    per_row = np.bincount(idx // n_r, minlength=n_q)
    assert row_off.dtype == np.int64 and hit_ref.dtype == np.int32
    assert list(row_off) == [0] + list(np.cumsum(per_row)), (list(row_off), list(per_row))
    assert list(hit_ref) == list(idx % n_r)
    assert C.compare_records(hits, pool, exp[idx], exp_pool) == []
    return len(idx)


def same_all(a, b):
    """two search_all outputs are the same arrays (CIGAR words compared through the records)"""
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    for f in C.CMP_FIELDS + ("cigar_len",):
        assert np.array_equal(a[2][f], b[2][f]), f
    for x, y in zip(a[2], b[2]):
        if int(x["cigar_len"]) > 0:
            assert list(a[3][x["cigar_off"]: x["cigar_off"] + x["cigar_len"]]) == list(b[3][y["cigar_off"]: y["cigar_off"] + y["cigar_len"]])


def top_k(got, q, k):
    """the k best of row q of a search_all output under the rank rule of ssw_engine_search (status 1, score1 desc, ref asc)"""
    row_off, hit_ref, hits, _ = got
    a, b = int(row_off[q]), int(row_off[q + 1])
    h, r = hits[a:b], hit_ref[a:b]
    o = np.lexsort((r, -h["score1"].astype(np.int64), -h["status"].astype(np.int64)))[:k]
    return r[o], h[o]


def reset(eng, *opts):
    for o in opts:
        eng.set_option(o, -1)


# ---------------------------------------------------------------------------------------------------------------------
# cases (each runs on the emulator build and on the GPU)
# ---------------------------------------------------------------------------------------------------------------------

def case_dna_thresholds(gpu):
    """score_size 0 / 1 / 2 (status-1 hits, re-done byte overflows) and min_score 0, 1, a middle value and above every score"""
    L, eng = _engine(gpu)
    queries, refs = dna_grid()
    mat = C.dna_matrix(2, 2)
    eng.set_sequences(queries, refs)
    nq, nr = len(queries), len(refs)
    for ss in (2, 1, 0):
        exp, ep = grid_records(queries, refs, mat, 5, 3, 1, score_size=ss)
        if ss == 0:
            assert (exp["status"] == 1).any()
        top = int(exp["score1"].max())
        for ms in (0, 1, 40, top + 1):
            eng.set_option("grid_min", 1)
            dev = eng.search_all(mat, 5, ms, score_size=ss)
            t_dev = eng.timing()
            n = check_all(dev, exp, ep, nq, nr, ms)
            if ms == top + 1:
                assert n == int((exp["status"] == 1).sum())
                if ss != 0:
                    assert n == 0 and not dev[0].any()                  # an empty result: row_off all zero
            else:
                assert n > 0
            eng.align(mat, 5, 3, 1, flag=0, score_size=ss)
            t_al = eng.timing()
            assert t_dev["fill_forward_launches"] == t_al["fill_forward_launches"] > 0    # the grid path ran
            assert t_dev["byte_overflows"] == t_al["byte_overflows"]
            if ss == 2:
                assert t_dev["byte_overflows"] > 0                      # redo pairs merged into their rows
            eng.set_option("grid_min", NEVER_GRID)
            same_all(eng.search_all(mat, 5, ms, score_size=ss), dev)
    reset(eng, "grid_min")
    eng.close()


def case_fallbacks(gpu):
    """the whole-call fallbacks -- the "chunk" option, gapO <= gapE -- give the grid path's arrays and the checker's"""
    L, eng = _engine(gpu)
    queries, refs = dna_grid()
    mat = C.dna_matrix(2, 2)
    eng.set_sequences(queries, refs)
    eng.set_option("grid_min", 1)
    dev = eng.search_all(mat, 5, 20, score_size=2)
    eng.set_option("chunk", 64)
    same_all(eng.search_all(mat, 5, 20, score_size=2), dev)
    eng.set_option("chunk", 0)
    exp, ep = grid_records(queries, refs, mat, 5, 2, 2, score_size=2)
    check_all(eng.search_all(mat, 5, 20, gap_open=2, gap_extend=2, score_size=2), exp, ep, len(queries), len(refs), 20)
    reset(eng, "grid_min")
    eng.close()


def case_launch_groups(gpu):
    """config-4-shaped protein grid over >= 3 launch groups: arming tail 30 (many re-dos merged into their rows), automatic
    arming and no arming; the general path gives the same arrays"""
    L, eng = _engine(gpu)
    W = C.config_workload(4, n_queries=6, n_targets=41)
    eng.set_sequences(W["queries"], W["refs"])
    exp, ep = grid_records(W["queries"], W["refs"], C.BLOSUM50, 24, 3, 1, mask_len=150, score_size=1)
    ms = int(np.percentile(exp["score1"], 80))
    eng.set_option("grid_min", 1)
    eng.set_option("grid_split", 1)
    eng.set_option("grid_group", 1)
    outs = {}
    for arm in (30, -1, 0):
        eng.set_option("grid_arm", arm)
        outs[arm] = eng.search_all(C.BLOSUM50, 24, ms, mask_len=150, score_size=1)
        assert check_all(outs[arm], exp, ep, 6, 41, ms) > 0
        t = eng.timing()
        assert t["fill_forward_launches"] >= 3
        if arm == 30:
            assert t["byte_overflows"] > 20
    same_all(outs[30], outs[0])
    eng.set_option("grid_min", NEVER_GRID)
    same_all(eng.search_all(C.BLOSUM50, 24, ms, mask_len=150, score_size=1), outs[0])
    reset(eng, "grid_min", "grid_split", "grid_group", "grid_arm")
    eng.close()


def case_rejected_pilot(gpu):
    """automatic arming where it cannot pay (short queries inside long targets): the pilot group is rejected and its queries run
    again armed from column 0 -- its hits and its redo list are dropped, no hit is lost or doubled"""
    L, eng = _engine(gpu)
    rng = np.random.default_rng(99)
    tq = [rng.integers(0, 20, size=40).astype(np.int8) for _ in range(6)]
    tt = []
    for k in range(30):
        t = rng.integers(0, 20, size=260).astype(np.int8)
        a = int(rng.integers(0, 200))
        t[a: a + 40] = tq[k % 6]
        tt.append(t)
    exp, ep = grid_records(tq, tt, C.BLOSUM50, 24, 12, 2, mask_len=20, score_size=1)
    eng.set_option("grid_min", 1)
    eng.set_option("grid_split", 1)
    eng.set_option("grid_group", 1)
    for ms in (0, 60):
        eng.set_sequences(tq, tt)                                       # forgets that arming did not pay before
        got = eng.search_all(C.BLOSUM50, 24, ms, gap_open=12, gap_extend=2, mask_len=20, score_size=1)
        t = eng.timing()
        assert t["fill_forward_launches"] == 4 and t["byte_overflows"] == 0, t     # 3 groups, the pilot twice; nothing re-done
        assert check_all(got, exp, ep, 6, 30, ms) > 0
    reset(eng, "grid_min", "grid_split", "grid_group")
    eng.close()


def case_leftovers(gpu):
    """references above grid_max_ref leave the device path: their hits are interleaved at their places within the rows; queries
    above 640 padded rows: their rows come from the general path (leftover_pairs)"""
    L, eng = _engine(gpu)
    queries, refs = small_grid(long_t=(1200, 2500, 1800))
    nq, nr = len(queries), len(refs)
    eng.set_sequences(queries, refs)
    exp, ep = grid_records(queries, refs, C.BLOSUM50, 24, 3, 1, **PROT)
    ms = int(np.percentile(exp["score1"], 70))
    eng.set_option("grid_min", 1)
    eng.set_option("grid_max_ref", 1000)
    n_left = sum(len(r) > 1000 for r in refs)
    got = eng.search_all(C.BLOSUM50, 24, ms, **PROT)
    assert eng.timing()["leftover_pairs"] == n_left * nq and n_left >= 4
    check_all(got, exp, ep, nq, nr, ms)
    long_r = [r for r in range(nr) if len(refs[r]) > 1000]
    assert np.isin(got[1], long_r).any() and not np.isin(got[1], long_r).all()   # both kinds in the rows
    eng.set_option("grid_max_ref", -1)
    queries, refs = small_grid(long_q=(700, 1100))
    nq, nr = len(queries), len(refs)
    eng.set_sequences(queries, refs)
    exp, ep = grid_records(queries, refs, C.BLOSUM50, 24, 3, 1, **PROT)
    eng.set_option("grid_arm", 0)
    got = eng.search_all(C.BLOSUM50, 24, ms, **PROT)
    t = eng.timing()
    assert t["leftover_pairs"] == 2 * nr and t["fill_forward_launches"] > 0
    check_all(got, exp, ep, nq, nr, ms)
    eng.set_option("grid_min", NEVER_GRID)
    same_all(eng.search_all(C.BLOSUM50, 24, ms, **PROT), got)
    reset(eng, "grid_min", "grid_arm")
    eng.close()


def case_flags(gpu):
    """flag 0x0f: begins and CIGARs of the hits only, equal to align of the hit pairs"""
    L, eng = _engine(gpu)
    queries, refs = dna_grid()
    mat = C.dna_matrix(2, 2)
    eng.set_sequences(queries, refs)
    nq, nr = len(queries), len(refs)
    for grid_min in (1, NEVER_GRID):
        eng.set_option("grid_min", grid_min)
        for flag, filters, filterd in ((0x0f, 0, 32767), (0x0f, 250, 60), (2, 120, 0)):
            exp, ep = grid_records(queries, refs, mat, 5, 3, 1, flag=flag, filters=filters, filterd=filterd, score_size=2)
            got = eng.search_all(mat, 5, 30, flag=flag, filters=filters, filterd=filterd, score_size=2)
            check_all(got, exp, ep, nq, nr, 30)
            assert (got[2]["cigar_len"] > 0).any() == (filters < 250)
            hq = np.repeat(np.arange(nq), np.diff(got[0]))
            res, pool = eng.align(mat, 5, 3, 1, flag=flag, filters=filters, filterd=filterd, score_size=2, pair_query=hq, pair_ref=got[1])
            same_all(got, (got[0], got[1], res, pool))
    reset(eng, "grid_min")
    eng.close()


def case_topk_consistency(gpu):
    """the k best of every row of search_all under the rank rule are search(k, min_score): k below, at and above the row
    length, and ties at the cut"""
    L, eng = _engine(gpu)
    mat = C.dna_matrix(2, 2)
    for grid in (dna_grid(), tie_grid()):
        queries, refs = grid
        eng.set_sequences(queries, refs)
        for grid_min in (1, NEVER_GRID):
            eng.set_option("grid_min", grid_min)
            for ms in (0, 30):
                al = eng.search_all(mat, 5, ms, score_size=2)
                lens = np.diff(al[0])
                for k in sorted({1, 4, 6, int(lens.max()), int(lens.max()) + 2} - {0}):
                    hit_ref, hits, n_hits, _ = eng.search(mat, 5, k, min_score=ms, score_size=2)
                    for q in range(len(queries)):
                        r, h = top_k(al, q, k)
                        assert int(n_hits[q]) == len(r) == min(k, int(lens[q]))
                        assert list(hit_ref[q, :len(r)]) == list(r), (q, k)
                        for f in C.CMP_FIELDS:
                            assert np.array_equal(hits[q, :len(r)][f], h[f]), (q, k, f)
    reset(eng, "grid_min")
    eng.close()


def case_max_hits(gpu):
    """a bound one below the hit count fails with -2 and no set; a bound equal to it succeeds"""
    L, eng = _engine(gpu)
    queries, refs = dna_grid()
    mat = C.dna_matrix(2, 2)
    eng.set_sequences(queries, refs)
    f = eng.lib.ssw_engine_search_all
    f.argtypes = [ct.c_void_p, ct.POINTER(L.BatchParams), ct.c_int32, ct.c_int64, ct.POINTER(ct.c_void_p)]
    f.restype = ct.c_int
    P = L.BatchParams(mat.ctypes.data_as(ct.POINTER(ct.c_int8)), 5, 3, 1, 0, 0, 0, -1, 2)
    for grid_min in (1, NEVER_GRID):
        eng.set_option("grid_min", grid_min)
        for ms in (1, 30):
            n = len(eng.search_all(mat, 5, ms)[1])
            assert n > 0
            with pytest.raises(RuntimeError, match="max_hits"):
                eng.search_all(mat, 5, ms, max_hits=n - 1)
            h = ct.c_void_p(12345)
            assert f(eng.h, ct.byref(P), ms, n - 1, ct.byref(h)) == -2 and not h.value
            assert len(eng.search_all(mat, 5, ms, max_hits=n)[1]) == n
    top = int(eng.search_all(mat, 5, 0)[2]["score1"].max())
    got = eng.search_all(mat, 5, top + 1, max_hits=0)                 # no hit: a bound of 0 holds
    assert len(got[1]) == 0 and not got[0].any()
    reset(eng, "grid_min")
    eng.close()


def case_arguments(gpu):
    """NULL engine, params or out, a negative bound and no resident set are refused with -1 and *out NULL"""
    L, eng = _engine(gpu)
    mat = C.dna_matrix(2, 2)

    def f(*args):                                    # untyped params: NULL too (search_all() types the function itself)
        fn = eng.lib.ssw_engine_search_all
        fn.argtypes = [ct.c_void_p, ct.c_void_p, ct.c_int32, ct.c_int64, ct.POINTER(ct.c_void_p)]
        fn.restype = ct.c_int
        return fn(*args)
    P = L.BatchParams(mat.ctypes.data_as(ct.POINTER(ct.c_int8)), 5, 3, 1, 0, 0, 0, -1, 2)
    h = ct.c_void_p(12345)
    assert f(eng.h, ct.addressof(P), 0, 100, ct.byref(h)) == -1 and not h.value        # no resident set
    with pytest.raises(RuntimeError):
        eng.search_all(mat, 5, 0)
    queries, refs = tie_grid()
    eng.set_sequences(queries, refs)
    for args in ((None, ct.addressof(P), 0, 100), (eng.h, None, 0, 100), (eng.h, ct.addressof(P), 0, -1)):
        h = ct.c_void_p(12345)
        assert f(*args, ct.byref(h)) == -1 and not h.value, args
    assert f(eng.h, ct.addressof(P), 0, 100, None) == -1
    h = ct.c_void_p()
    assert f(eng.h, ct.addressof(P), 0, 10 ** 6, ct.byref(h)) == 0 and h.value
    v = L.HitView()
    assert eng.lib.ssw_hit_set_view(h, ct.byref(v)) == 0 and v.n_rows == len(queries)
    assert eng.lib.ssw_hit_set_view(None, ct.byref(v)) == -1
    eng.lib.ssw_hit_set_destroy(h)
    eng.lib.ssw_hit_set_destroy(None)
    grp = _group(L, gpu, 1)
    g = grp.lib.ssw_group_search_all
    g.argtypes = [ct.c_void_p, ct.c_void_p, ct.c_void_p, ct.c_int32, ct.c_int32, ct.c_void_p, ct.c_void_p, ct.c_int32, ct.c_void_p,
                  ct.c_void_p, ct.c_int32, ct.c_int64, ct.POINTER(ct.c_void_p)]
    g.restype = ct.c_int
    h = ct.c_void_p(12345)
    assert g(None, ct.addressof(P), None, 0, 0, None, None, 0, None, None, 0, 100, ct.byref(h)) == -1 and not h.value
    assert g(grp.h, ct.addressof(P), None, 0, 0, None, None, 0, None, None, 0, 100, ct.byref(h)) == -1 and not h.value
    with pytest.raises(RuntimeError, match="max_hits"):
        grp.search_all(queries, refs, mat, 5, 0, max_hits=0)
    grp.close()
    eng.close()


def case_group(gpu):
    """groups of several devices: the arrays of one engine (codes; text with reverse complements) and the checker's"""
    L, eng = _engine(gpu)
    queries, refs = dna_grid()
    mat = C.dna_matrix(2, 2)
    nq, nr = len(queries), len(refs)
    rcq = [(3 - q)[::-1].astype(np.int8) for q in queries]               # codes 0..3 only: complement c -> 3 - c
    exp, ep = grid_records(queries, refs, mat, 5, 3, 1, flag=0x0f, filterd=32767, score_size=2)
    exp2, ep2 = grid_records(queries + rcq, refs, mat, 5, 3, 1, score_size=2)
    eng.set_sequences(queries, refs)
    eng.set_option("grid_min", 1)
    one = eng.search_all(mat, 5, 20, flag=0x0f, filterd=32767, score_size=2)
    eng.close()
    text_q = ["".join("ACGT"[c] for c in q) for q in queries]
    text_r = ["".join("ACGT"[c] for c in r) for r in refs]
    table = np.full(128, 4, dtype=np.int8)
    for i, c in enumerate("ACGT"):
        table[ord(c)] = i
        table[ord(c.lower())] = i
    first = None
    for world in ((1, 2) if gpu else (1, 2, 3, 5)):
        if not gpu:
            os.environ["SSW_EMU_DEVICES"] = str(world)
        try:
            grp = _group(L, gpu, world)
            grp.set_option("grid_min", 1)
            grp.set_option("latency_cols", 0)
            outs = [grp.search_all(queries, refs, mat, 5, 20, flag=0x0f, filterd=32767, score_size=2),
                    grp.search_all(text_q, text_r, mat, 5, 20, table=table, add_reverse_complement=True)]
            grp.close()
        finally:
            os.environ.pop("SSW_EMU_DEVICES", None)
        same_all(outs[0], one)
        check_all(outs[0], exp, ep, nq, nr, 20)
        assert len(outs[1][0]) == 2 * nq + 1
        check_all(outs[1], exp2, ep2, 2 * nq, nr, 20)
        if first is None:
            first = outs
        else:
            for a, b in zip(outs, first):
                same_all(a, b)


def test_search_all_entry_points_declared_and_exported():
    """every new name is declared in include/ssw_batch.h and exported by the libraries that are built"""
    import re
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(C.ROOT, "include", "ssw_batch.h")).read(), flags=re.S)
    for name in ("ssw_engine_search_all", "ssw_group_search_all", "ssw_hit_set_view", "ssw_hit_set_destroy"):
        assert re.search(r"\b(int|void) %s\(" % name, txt), name
        for lib in (C.LIB_OURS, os.path.join(EMU_DIR, "libssw_emu.so")):
            if os.path.exists(lib):
                assert hasattr(ct.CDLL(lib), name), (lib, name)
    assert re.search(r"\}\s*ssw_hit_view;", txt) and "typedef struct ssw_hit_set ssw_hit_set;" in txt


CASES = [case_dna_thresholds, case_fallbacks, case_launch_groups, case_rejected_pilot, case_leftovers, case_flags,
         case_topk_consistency, case_max_hits, case_arguments, case_group]


@pytest.mark.parametrize("case", CASES, ids=[c.__name__[5:] for c in CASES])
def test_search_all_emulated(case, capfd):
    case(False)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.__name__[5:] for c in CASES])
def test_search_all_gpu(case, capfd):
    case(True)


@pytest.mark.gpu
def test_search_all_config4_scale(capfd):
    """256 config-4 queries x all 50,000 targets at a threshold near the 100th best score, on the device path; the rows of a
    sample of queries against the checker's full rows (the compiled reference where present), and every row's 100 best
    against search(100)"""
    L, eng = _engine(True)
    W = C.config_workload(4, n_queries=256)
    eng.set_sequences(W["queries"], W["refs"])
    hit_ref, hits, n_hits, _ = eng.search(C.BLOSUM50, 24, 100, mask_len=150, score_size=1)
    thr = int(np.median(hits[:, 99]["score1"]))
    got = eng.search_all(C.BLOSUM50, 24, thr, mask_len=150, score_size=1)
    t = eng.timing()
    assert t["fill_forward_launches"] > 1 and t["leftover_pairs"] == 0
    lens = np.diff(got[0])
    assert 20 * 256 < lens.sum() < 1000 * 256, lens.sum()
    k_hit_ref, k_hits, k_n, _ = eng.search(C.BLOSUM50, 24, 100, min_score=thr, mask_len=150, score_size=1)
    for q in range(256):
        r, h = top_k(got, q, 100)
        assert int(k_n[q]) == len(r) and list(k_hit_ref[q, :len(r)]) == list(r), q
    n_check = 64 if C.have_ref() and C.effective_cores()[0] >= 16 else 8
    sel = np.linspace(0, 255, n_check).astype(int)
    nr = len(W["refs"])
    exp, ep = grid_records([W["queries"][i] for i in sel], W["refs"], C.BLOSUM50, 24, 3, 1, mask_len=150, score_size=1)
    rows = np.concatenate([np.arange(got[0][q], got[0][q + 1]) for q in sel]).astype(np.int64)
    sub_off = np.concatenate([[0], np.cumsum(lens[sel])]).astype(np.int64)
    check_all((sub_off, got[1][rows], got[2][rows], got[3]), exp, ep, len(sel), nr, thr)
    eng.close()
