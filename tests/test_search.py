"""Top-k search (ssw_engine_search / ssw_group_search): every query's k best hits of the full queries x references grid.

The expected hits come from the full grid of checker records (C.cpu_batch: the compiled reference where present, the
oracle port otherwise), ranked in numpy by the rule of include/ssw_batch.h: a hit has status 1 or score1 >=
max(min_score, 1); status-1 pairs first, then score1 descending, then reference ascending.  Hit lists, hit counts, every
field and every CIGAR word are compared.  The same cases run on the CPU emulator build (tests/cuda_emu, test
infrastructure) and, marked gpu, on the CUDA library; the grid path (device-side selection) and the general path (host
selection) are forced on the same inputs and must agree."""
import ctypes as ct
import importlib.util
import os
import subprocess

import numpy as np
import pytest

import common as C

EMU_DIR = os.path.join(C.ROOT, "tests", "cuda_emu")
NEVER_GRID = 2 ** 31 - 1          # "grid_min" above any grid: the general path


def _pkg():
    spec = importlib.util.spec_from_file_location("ssw_b200_lib", os.path.join(C.PKG, "ssw_lib.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _engine(gpu):
    L = _pkg()
    if gpu:
        assert os.path.exists(C.LIB_OURS), "libssw.so missing: the CUDA extension must be built in-tree"
        eng = L.BatchAligner(device=0)
    else:
        subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
        eng = L.BatchAligner(lib_dir=EMU_DIR, lib_name="libssw_emu.so")
    eng.set_option("latency_cols", 0)          # the layouts of large batches
    return L, eng


def _group(L, gpu, n):
    if gpu:
        return L.GroupAligner(devices=[0] * n)
    return L.GroupAligner(n_devices=n, lib_dir=EMU_DIR, lib_name="libssw_emu.so")


def grid_records(queries, refs, mat, n, gapO, gapE, flag=0, filters=0, filterd=0, mask_len=-1, score_size=2, threads=None):
    """checker records of the full grid, pair p = q * n_r + r"""
    nq, nr = len(queries), len(refs)
    pq, pr = np.repeat(np.arange(nq), nr), np.tile(np.arange(nr), nq)
    exp, pool, _, _, _ = C.cpu_batch(queries, refs, pq, pr, mat, n, gapO, gapE, flag=flag, filters=filters, filterd=filterd,
                                     mask_len=mask_len, score_size=score_size, threads=threads)
    return exp, pool


def ranked(exp, n_q, n_r, k, min_score):
    """per query: the reference indices of its k best hits in rank order"""
    thr = max(min_score, 1)
    out = []
    for q in range(n_q):
        row = exp[q * n_r:(q + 1) * n_r]
        st = row["status"].astype(np.int64)
        sc = np.where(st == 1, 0, row["score1"].astype(np.int64))
        r = np.nonzero((st == 1) | (sc >= thr))[0]
        out.append(r[np.lexsort((r, -sc[r], -st[r]))][:k])
    return out


def check(got, exp, exp_pool, n_q, n_r, k, min_score):
    """search output against the ranked checker grid; returns the number of hits"""
    hit_ref, hits, n_hits, pool = got
    want = ranked(exp, n_q, n_r, k, min_score)
    assert hit_ref.shape == (n_q, k) and hits.shape == (n_q, k) and n_hits.shape == (n_q,)
    for q in range(n_q):
        m = len(want[q])
        assert int(n_hits[q]) == m, (q, int(n_hits[q]), m)
        assert list(hit_ref[q, :m]) == list(want[q]), (q, list(hit_ref[q, :m]), list(want[q]))
        assert (hit_ref[q, m:] == -1).all(), q
        assert C.compare_records(hits[q, :m], pool, exp[q * n_r + want[q]], exp_pool) == [], q
    return int(n_hits.sum())


def same(a, b):
    """two search outputs are the same arrays (CIGAR words compared through the records)"""
    for x, y in zip(a[:3], b[:3]):
        assert x.shape == y.shape
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2])
    ha, hb = a[1].reshape(-1), b[1].reshape(-1)
    for f in C.CMP_FIELDS + ("cigar_len",):
        assert np.array_equal(ha[f], hb[f]), f
    for x, y in zip(ha, hb):
        if int(x["cigar_len"]) > 0:
            assert list(a[3][x["cigar_off"]: x["cigar_off"] + x["cigar_len"]]) == list(b[3][y["cigar_off"]: y["cigar_off"] + y["cigar_len"]])


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------

def dna_grid():
    """ragged DNA grid whose high-identity 150-mers overflow byte scores (status 1 with score_size 0, re-done with 2)"""
    rng = np.random.default_rng(31)
    refs = [rng.integers(0, 4, size=n).astype(np.int8) for n in (260, 97, 400, 33, 180, 300)]
    refs[5] = refs[0].copy()                                             # a duplicate: a tie of every score
    queries = []
    for i, n in enumerate((150, 150, 140, 33, 64, 17, 150, 100, 1)):
        r = refs[(2 * i) % 5]
        if len(r) > n + 10 and i % 4 != 3:
            queries.append(C.mutate_read(rng, r, int(rng.integers(0, len(r) - n - 5)), n, 0.02 if i < 3 else 0.1, 0.005, 0.005))
        else:
            queries.append(rng.integers(0, 4, size=n).astype(np.int8))
    return queries, refs


def tie_grid():
    """duplicated references: the k-th place falls inside a tie"""
    rng = np.random.default_rng(77)
    base = [rng.integers(0, 4, size=n).astype(np.int8) for n in (120, 90, 150)]
    refs = [base[i].copy() for i in (0, 1, 0, 2, 0, 1, 0, 2, 0, 1, 0)]      # reference 0's sequence five times (0, 2, 4, 6, 8, 10 -> six)
    queries = [C.mutate_read(rng, base[0], 10, 60, 0.05, 0.0, 0.0), C.mutate_read(rng, base[1], 5, 50, 0.1, 0.01, 0.01),
               C.mutate_read(rng, base[2], 30, 70, 0.05, 0.0, 0.0), rng.integers(0, 4, size=40).astype(np.int8)]
    return queries, refs


# ---------------------------------------------------------------------------------------------------------------------
# cases (each runs on the emulator build and on the GPU)
# ---------------------------------------------------------------------------------------------------------------------

def case_dna_device_path(gpu):
    L, eng = _engine(gpu)
    queries, refs = dna_grid()
    mat = C.dna_matrix(2, 2)
    eng.set_sequences(queries, refs)
    nq, nr = len(queries), len(refs)
    for ss in (2, 1, 0):
        exp, ep = grid_records(queries, refs, mat, 5, 3, 1, score_size=ss)
        if ss == 0:
            assert (exp["status"] == 1).any()
        for k, ms in ((3, 0), (1, 0), (nr + 2, 0), (4, 40)):
            eng.set_option("grid_min", 1)
            dev = eng.search(mat, 5, k, min_score=ms, score_size=ss)
            t_dev = eng.timing()
            n = check(dev, exp, ep, nq, nr, k, ms)
            assert n > 0
            if ss == 0 and ms == 40:
                assert (dev[1]["status"] == 1).any()                   # status-1 hits whatever min_score is
            # the grid path ran: the same fill launches and re-done pairs as a grid-path align
            eng.align(mat, 5, 3, 1, flag=0, score_size=ss)
            t_al = eng.timing()
            assert t_dev["fill_forward_launches"] == t_al["fill_forward_launches"]
            assert t_dev["byte_overflows"] == t_al["byte_overflows"]
            if ss == 2:
                assert t_dev["byte_overflows"] > 0                      # redo pairs merged into the device's lists
            # the general path on the same inputs: the same arrays
            eng.set_option("grid_min", NEVER_GRID)
            same(eng.search(mat, 5, k, min_score=ms, score_size=ss), dev)
    eng.set_option("grid_min", -1)
    eng.close()


def case_ties(gpu):
    L, eng = _engine(gpu)
    queries, refs = tie_grid()
    mat = C.dna_matrix(2, 2)
    eng.set_sequences(queries, refs)
    nq, nr = len(queries), len(refs)
    exp, ep = grid_records(queries, refs, mat, 5, 3, 1, mask_len=-1, score_size=2)
    s0 = exp["score1"][0: nr]
    assert (s0[[0, 2, 4, 6, 8, 10]] == s0[0]).all() and s0[0] == s0.max()       # query 0: a six-way tie at the top
    thr_few = int(np.sort(exp["score1"])[-3])                                   # leaves fewer than k hits for most queries
    for grid_min in (1, NEVER_GRID):
        eng.set_option("grid_min", grid_min)
        for k, ms in ((1, 0), (4, 0), (6, 0), (7, 0), (nr, 0), (nr + 5, 0), (5, thr_few)):
            check(eng.search(mat, 5, k, min_score=ms), exp, ep, nq, nr, k, ms)
    eng.set_option("grid_min", -1)
    eng.close()


def case_protein(gpu):
    """config-4-shaped grid: several launch groups, many overflow-3 re-dos (arming tail 30) and the automatic arming"""
    L, eng = _engine(gpu)
    W = C.config_workload(4, n_queries=6, n_targets=41)
    eng.set_sequences(W["queries"], W["refs"])
    exp, ep = grid_records(W["queries"], W["refs"], C.BLOSUM50, 24, 3, 1, mask_len=150, score_size=1)
    eng.set_option("grid_min", 1)
    eng.set_option("grid_split", 1)
    eng.set_option("grid_group", 1)
    outs = {}
    for arm in (30, -1, 0):
        eng.set_option("grid_arm", arm)
        outs[arm] = eng.search(C.BLOSUM50, 24, 5, mask_len=150, score_size=1)
        check(outs[arm], exp, ep, 6, 41, 5, 0)
        t = eng.timing()
        assert t["fill_forward_launches"] >= 3
        if arm == 30:
            assert t["byte_overflows"] > 20                            # most maxima lie before the tail: re-done and merged
    same(outs[30], outs[0])
    eng.set_option("grid_min", NEVER_GRID)
    same(eng.search(C.BLOSUM50, 24, 5, mask_len=150, score_size=1), outs[0])
    for opt in ("grid_min", "grid_split", "grid_group", "grid_arm"):
        eng.set_option(opt, -1)
    eng.close()


def case_general_path(gpu):
    """resident sets the grid path does not take: chunked references, a target > 4,096, gapO <= gapE"""
    L, eng = _engine(gpu)
    queries, refs = dna_grid()
    mat = C.dna_matrix(2, 2)
    eng.set_sequences(queries, refs)
    eng.set_option("grid_min", 1)
    dev = eng.search(mat, 5, 4, score_size=2)
    eng.set_option("chunk", 64)
    same(eng.search(mat, 5, 4, score_size=2), dev)
    eng.set_option("chunk", 0)
    rng = np.random.default_rng(5)
    long_ref = rng.integers(0, 4, size=4500).astype(np.int8)
    refs2 = [long_ref, refs[0], long_ref[4300:].copy()]
    qs2 = [long_ref[4200:4290].copy(), C.mutate_read(rng, refs[0], 20, 80, 0.05, 0.01, 0.01), long_ref[100:170].copy()]
    eng.set_sequences(qs2, refs2)
    exp, ep = grid_records(qs2, refs2, mat, 5, 3, 1, mask_len=-1, score_size=2)
    check(eng.search(mat, 5, 2), exp, ep, 3, 3, 2, 0)
    eng.set_sequences(queries[:4], refs[:4])
    exp, ep = grid_records(queries[:4], refs[:4], mat, 5, 2, 2, mask_len=-1, score_size=2)
    check(eng.search(mat, 5, 3, gap_open=2, gap_extend=2), exp, ep, 4, 4, 3, 0)
    eng.set_option("grid_min", -1)
    eng.close()


def case_flags(gpu):
    """begins and CIGARs for the hits only"""
    L, eng = _engine(gpu)
    queries, refs = dna_grid()
    mat = C.dna_matrix(2, 2)
    eng.set_sequences(queries, refs)
    nq, nr = len(queries), len(refs)
    k = 3
    for grid_min in (1, NEVER_GRID):
        eng.set_option("grid_min", grid_min)
        for flag, filters, filterd in ((0x0f, 250, 60), (2, 120, 0), (0x0f, 0, 32767)):
            exp, ep = grid_records(queries, refs, mat, 5, 3, 1, flag=flag, filters=filters, filterd=filterd, score_size=2)
            got = eng.search(mat, 5, k, flag=flag, filters=filters, filterd=filterd, score_size=2)
            t_flag = eng.timing()
            check(got, exp, ep, nq, nr, k, 0)
            assert (got[1]["cigar_len"] > 0).any() == (filters < 250)          # 250 / 60: every CIGAR filtered out (ssw.c:938)
            eng.search(mat, 5, k, score_size=2)
            t0 = eng.timing()
            # the work the flag adds is an align of the hit pairs alone
            hq = np.repeat(np.arange(nq), got[2])
            hr = np.concatenate([got[0][q, :got[2][q]] for q in range(nq)])
            eng.align(mat, 5, 3, 1, flag=flag, filters=filters, filterd=filterd, score_size=2, pair_query=hq, pair_ref=hr)
            t_hits = eng.timing()
            assert t_flag["cells_forward"] - t0["cells_forward"] == t_hits["cells_forward"]
            assert t_flag["fill_reverse_ms"] >= 0 and len(hq) <= nq * k
            eng.align(mat, 5, 3, 1, flag=flag, filters=filters, filterd=filterd, score_size=2)
            assert t_hits["cells_forward"] < eng.timing()["cells_forward"]
    eng.set_option("grid_min", -1)
    eng.close()


def case_group(gpu):
    """groups of 1, 2 and 3 devices: identical arrays (codes and text with reverse complements, with and without CIGARs)"""
    L, _ = _engine(gpu)
    queries, refs = dna_grid()
    mat = C.dna_matrix(2, 2)
    nq, nr = len(queries), len(refs)
    exp, ep = grid_records(queries, refs, mat, 5, 3, 1, flag=0x0f, filterd=32767, score_size=2)
    text_q = ["".join("ACGT"[c] for c in q) for q in queries]
    text_r = ["".join("ACGT"[c] for c in r) for r in refs]
    table = np.full(128, 4, dtype=np.int8)
    for i, c in enumerate("ACGT"):
        table[ord(c)] = i
        table[ord(c.lower())] = i
    first = {}
    for world in (1, 2, 3):
        if not gpu:
            os.environ["SSW_EMU_DEVICES"] = str(world)
        try:
            grp = _group(L, gpu, world)
            grp.set_option("grid_min", 1)
            grp.set_option("latency_cols", 0)
            outs = [grp.search(queries, refs, mat, 5, 3, flag=0x0f, filterd=32767, score_size=2),
                    grp.search(text_q, text_r, mat, 5, 4, min_score=20, table=table, add_reverse_complement=True)]
            grp.close()
        finally:
            os.environ.pop("SSW_EMU_DEVICES", None)
        check(outs[0], exp, ep, nq, nr, 3, 0)
        assert outs[1][0].shape == (2 * nq, 4)
        if world == 1:
            first = outs
        else:
            for a, b in zip(outs, first):
                same(a, b)


def case_rejected(gpu):
    L, eng = _engine(gpu)
    mat = C.dna_matrix(2, 2)
    with pytest.raises(RuntimeError):
        eng.search(mat, 5, 3)                                          # no resident set
    queries, refs = tie_grid()
    eng.set_sequences(queries, refs)
    for k in (0, 1025, -1):
        with pytest.raises(RuntimeError):
            eng.search(mat, 5, k)
    assert eng.search(mat, 5, 1024)[0].shape == (len(queries), 1024)
    f = eng.lib.ssw_engine_search
    P = L.BatchParams(mat.ctypes.data_as(ct.POINTER(ct.c_int8)), 5, 3, 1, 0, 0, 0, -1, 2)
    hr = np.zeros(len(queries) * 2, np.int32)
    hs = np.zeros(len(queries) * 2, L.RESULT_DTYPE)
    nh = np.zeros(len(queries), np.int32)
    ptr = lambda a, t: a.ctypes.data_as(t)
    I32 = ct.POINTER(ct.c_int32)
    assert f(eng.h, ct.byref(P), 2, 0, None, ptr(hs, ct.c_void_p), ptr(nh, I32), None, 0, None) == -1
    assert f(eng.h, ct.byref(P), 2, 0, ptr(hr, I32), None, ptr(nh, I32), None, 0, None) == -1
    assert f(eng.h, ct.byref(P), 2, 0, ptr(hr, I32), ptr(hs, ct.c_void_p), None, None, 0, None) == -1
    assert f(eng.h, ct.byref(P), 2, 0, ptr(hr, I32), ptr(hs, ct.c_void_p), ptr(nh, I32), None, 0, None) == 0
    assert f(None, ct.byref(P), 2, 0, ptr(hr, I32), ptr(hs, ct.c_void_p), ptr(nh, I32), None, 0, None) == -1
    grp = _group(L, gpu, 1)
    with pytest.raises(RuntimeError):
        grp.search(queries, refs, mat, 5, 0)
    with pytest.raises(RuntimeError):
        grp.search(queries, refs, mat, 5, 1025)
    grp.close()
    eng.close()


def test_search_entry_points_declared_and_exported():
    """both entry points are declared in include/ssw_batch.h and exported by the libraries that are built"""
    import re
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(C.ROOT, "include", "ssw_batch.h")).read(), flags=re.S)
    for name in ("ssw_engine_search", "ssw_group_search"):
        assert re.search(r"\bint %s\(" % name, txt), name
        for lib in (C.LIB_OURS, os.path.join(EMU_DIR, "libssw_emu.so")):
            if os.path.exists(lib):
                assert hasattr(ct.CDLL(lib), name), (lib, name)


CASES = [case_dna_device_path, case_ties, case_protein, case_general_path, case_flags, case_group, case_rejected]


@pytest.mark.parametrize("case", CASES, ids=[c.__name__[5:] for c in CASES])
def test_search_emulated(case, capfd):
    case(False)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.__name__[5:] for c in CASES])
def test_search_gpu(case, capfd):
    case(True)


@pytest.mark.gpu
def test_search_config4_scale(capfd):
    """256 config-4 queries x all 50,000 targets, k = 10, on the device path; hit lists of 64 queries against the checker's
    full rows (the compiled reference where present)."""
    L, eng = _engine(True)
    W = C.config_workload(4, n_queries=256)
    eng.set_sequences(W["queries"], W["refs"])
    got = eng.search(C.BLOSUM50, 24, 10, mask_len=150, score_size=1)
    assert eng.timing()["fill_forward_launches"] > 0
    n_check = 64 if C.have_ref() and C.effective_cores()[0] >= 16 else 8
    sel = np.linspace(0, 255, n_check).astype(int)
    nr = len(W["refs"])
    qs = [W["queries"][i] for i in sel]
    exp, ep = grid_records(qs, W["refs"], C.BLOSUM50, 24, 3, 1, mask_len=150, score_size=1)
    sub = (got[0][sel], got[1][sel], got[2][sel], got[3])
    assert check(sub, exp, ep, len(sel), nr, 10, 0) == 10 * len(sel)
    eng.close()
