"""Self-search (ssw_engine_search_self / ssw_group_search_self): every unordered pair of one set that is a hit, computed once.

Pair {i, j} is reported as the record of query = the earlier of the two in canonical order (length, then index) against the
other.  The expected output is the checker's records of those oriented pairs (C.cpu_batch: the compiled reference where
present, the oracle port otherwise) with the non-hits removed, row i holding i's hits in ascending partner index.  The
mirror identity ties it to the threshold search: the self hits and their mirrors are exactly search_all on (S, S) without
the diagonal.  Grid path, general path, launch groups, tiles, off-grid sequences and device groups must give identical
arrays; what ran where is asserted from the counters of ssw_engine_timing.  The cases run on the CPU emulator build and,
marked gpu, on the CUDA library."""
import ctypes as ct
import os

import numpy as np
import pytest

import common as C
from test_search import NEVER_GRID, EMU_DIR, _engine, _group, dna_grid
from test_search_all import hit_mask, reset, same_all
from test_search_mixed import PROT, mixed_workload


def canon(seqs):
    """canonical order (length, then index, ascending) and its inverse"""
    lens = np.array([len(s) for s in seqs], dtype=np.int64)
    order = np.lexsort((np.arange(len(seqs)), lens))
    rank = np.empty(len(seqs), dtype=np.int64)
    rank[order] = np.arange(len(seqs))
    return order, rank


def oriented_pairs(seqs):
    """every unordered pair once, as (earlier in canonical order, later), sorted by (query, partner index); pairs with an empty
    sequence (always the query: it sorts first) align nowhere and are never hits"""
    n = len(seqs)
    _, rank = canon(seqs)
    i, j = np.nonzero(np.ones((n, n), bool))
    lens = np.array([len(s) for s in seqs], dtype=np.int64)
    keep = (rank[i] < rank[j]) & (lens[i] > 0)
    return i[keep].astype(np.int64), j[keep].astype(np.int64)


def expected_self(seqs, mat, n, gapO, gapE, min_score, flag=0, mask_len=-1, score_size=2):
    """(row_off, hit_ref, records, pool) of the checker over the oriented pairs, filtered by the hit rule"""
    pq, pr = oriented_pairs(seqs)
    if len(pq) == 0:
        return np.zeros(len(seqs) + 1, np.int64), pr, None, None
    exp, pool, _, _, _ = C.cpu_batch(seqs, seqs, pq, pr, mat, n, gapO, gapE, flag=flag, mask_len=mask_len, score_size=score_size)
    m = hit_mask(exp, min_score)
    per_row = np.bincount(pq[m], minlength=len(seqs))
    return np.concatenate([[0], np.cumsum(per_row)]).astype(np.int64), pr[m], exp[m], pool


def check_self(got, want):
    row_off, hit_ref, hits, pool = got
    w_off, w_ref, w_rec, w_pool = want
    assert row_off.dtype == np.int64 and hit_ref.dtype == np.int32
    assert list(row_off) == list(w_off), (list(row_off), list(w_off))
    assert list(hit_ref) == list(w_ref)
    if len(w_ref):
        assert C.compare_records(hits, pool, w_rec, w_pool) == []
    return len(w_ref)


def check_mirror(self_out, all_out, seqs):
    """self hits + their mirrors == search_all(S, S) without the diagonal; records of the oriented pairs identical"""
    n = len(seqs)
    _, rank = canon(seqs)
    s_off, s_ref, s_hits, s_pool = self_out
    a_off, a_ref, a_hits, a_pool = all_out
    s_q = np.repeat(np.arange(n), np.diff(s_off))
    a_q = np.repeat(np.arange(n), np.diff(a_off))
    assert (rank[s_q] < rank[s_ref]).all()
    pairs_self = set(zip(s_q.tolist(), s_ref.tolist())) | set(zip(s_ref.tolist(), s_q.tolist()))
    off_diag = a_q != a_ref
    pairs_all = set(zip(a_q[off_diag].tolist(), a_ref[off_diag].tolist()))
    assert pairs_self == pairs_all
    oriented = off_diag & (rank[a_q] < rank[a_ref])
    assert oriented.sum() == len(s_ref)
    assert list(a_q[oriented]) == list(s_q) and list(a_ref[oriented]) == list(s_ref)
    for f in C.CMP_FIELDS + ("cigar_len",):
        assert np.array_equal(a_hits[oriented][f], s_hits[f]), f
    for x, y in zip(a_hits[oriented], s_hits):
        if int(x["cigar_len"]) > 0:
            assert list(a_pool[x["cigar_off"]: x["cigar_off"] + x["cigar_len"]]) == list(s_pool[y["cigar_off"]: y["cigar_off"] + y["cigar_len"]])
    return len(s_ref)


def protein_set(empty=True):
    """proteins of 30 .. 200 aa, every other one carrying a mutated copy of one of two family segments; identical duplicates,
    several sequences of one length and (empty) one of length 0"""
    rng = np.random.default_rng(505)
    fams = [rng.integers(0, 20, size=40).astype(np.int8) for _ in range(2)]
    seqs = []
    for i, n in enumerate((30, 45, 60, 60, 60, 75, 90, 100, 120, 120, 150, 180, 200, 35, 80, 60)):
        s = rng.integers(0, 20, size=n).astype(np.int8)
        if i % 2 == 0:
            seg = fams[(i // 2) % 2][: min(40, n)].copy()
            x = rng.random(len(seg)) < 0.15
            seg[x] = rng.integers(0, 20, size=int(x.sum()))
            b = int(rng.integers(0, n - len(seg) + 1))
            s[b: b + len(seg)] = seg
        seqs.append(s)
    seqs += [seqs[2].copy(), seqs[10].copy()]
    if empty:
        seqs.insert(6, np.zeros(0, np.int8))
    return seqs


def equal_set(n=12, length=120, seed=8):
    """n proteins of one length, every third sharing a segment with the first"""
    rng = np.random.default_rng(seed)
    seqs = [rng.integers(0, 20, size=length).astype(np.int8) for _ in range(n)]
    for i in range(3, n, 3):
        seqs[i][10:70] = seqs[0][20:80]
    return seqs


def _ms(seqs, mat=C.BLOSUM50, n=24, gapO=3, gapE=1, pct=70, **kw):
    pq, pr = oriented_pairs(seqs)
    exp, _, _, _, _ = C.cpu_batch(seqs, seqs, pq, pr, mat, n, gapO, gapE, **kw)
    return int(np.percentile(exp["score1"], pct))


# ---------------------------------------------------------------------------------------------------------------------
# cases (each runs on the emulator build and on the GPU)
# ---------------------------------------------------------------------------------------------------------------------

def case_checker(gpu):
    """protein sets against the checker's oriented records, flags 0 and 0x0f; n = 0, 1, 2, 3"""
    L, eng = _engine(gpu)
    seqs = protein_set()
    ms = _ms(seqs, **PROT)
    eng.set_option("grid_min", 1)
    eng.set_sequences_self(seqs)
    for flag in (0, 0x0f):
        got = eng.search_self(C.BLOSUM50, 24, ms, flag=flag, **PROT)
        assert check_self(got, expected_self(seqs, C.BLOSUM50, 24, 3, 1, ms, flag=flag, **PROT)) > 20
        assert eng.timing()["fill_forward_launches"] > 0
    rng = np.random.default_rng(3)
    base = rng.integers(0, 20, size=90).astype(np.int8)
    for k in (0, 1, 2, 3):
        small = [base.copy() if i != 1 else base[:60].copy() for i in range(k)]
        eng.set_sequences_self(small)
        for flag in (0, 0x0f):
            got = eng.search_self(C.BLOSUM50, 24, 0, flag=flag, **PROT)
            assert len(got[0]) == k + 1
            check_self(got, expected_self(small, C.BLOSUM50, 24, 3, 1, 0, flag=flag, **PROT))
    reset(eng, "grid_min")
    eng.close()


def case_mirror(gpu):
    """on the same engine: search_self and search_all after set_sequences(S, S), grid path and general path, flag 0x0f"""
    L, eng = _engine(gpu)
    seqs = protein_set(empty=False)
    ms = _ms(seqs, **PROT)
    for gm in (1, NEVER_GRID):
        eng.set_option("grid_min", gm)
        for flag in (0, 0x0f):
            eng.set_sequences(seqs, seqs)
            full = eng.search_all(C.BLOSUM50, 24, ms, flag=flag, **PROT)
            eng.set_sequences_self(seqs)
            assert check_mirror(eng.search_self(C.BLOSUM50, 24, ms, flag=flag, **PROT), full, seqs) > 20
    reset(eng, "grid_min")
    eng.close()


def case_dna(gpu):
    """DNA at score sizes 0 / 1 / 2: status-1 hits (byte overflows at score size 0) and re-done byte overflows (2)"""
    L, eng = _engine(gpu)
    queries, refs = dna_grid()
    seqs = refs + queries
    mat = C.dna_matrix(2, 2)
    eng.set_option("grid_min", 1)
    for ss in (0, 1, 2):
        want = expected_self(seqs, mat, 5, 3, 1, 30, score_size=ss)
        eng.set_sequences_self(seqs)
        got = eng.search_self(mat, 5, 30, score_size=ss)
        check_self(got, want)
        t = eng.timing()
        if ss == 0:
            assert (got[2]["status"] == 1).any()
        if ss == 2:
            assert t["byte_overflows"] > 0
        eng.set_sequences(seqs, seqs)
        check_mirror(got, eng.search_all(mat, 5, 30, score_size=ss), seqs)
    reset(eng, "grid_min")
    eng.close()


def case_paths(gpu):
    """grid path, general path (grid_min at its maximum) and the chunk option give identical arrays"""
    L, eng = _engine(gpu)
    seqs = protein_set()
    ms = _ms(seqs, **PROT)
    eng.set_sequences_self(seqs)
    eng.set_option("grid_min", 1)
    dev = eng.search_self(C.BLOSUM50, 24, ms, **PROT)
    assert eng.timing()["fill_forward_launches"] > 0
    eng.set_option("grid_min", NEVER_GRID)
    same_all(eng.search_self(C.BLOSUM50, 24, ms, **PROT), dev)
    eng.set_option("grid_min", 1)
    eng.set_option("chunk", 64)
    same_all(eng.search_self(C.BLOSUM50, 24, ms, **PROT), dev)
    reset(eng, "grid_min", "chunk")
    eng.close()


def case_launch_groups(gpu):
    """>= 3 launch groups with arming forced (tail 30: re-dos), automatic and off; a rejected pilot group"""
    L, eng = _engine(gpu)
    seqs = protein_set()
    ms = _ms(seqs, mask_len=150, score_size=1, pct=80)
    want = expected_self(seqs, C.BLOSUM50, 24, 3, 1, ms, mask_len=150, score_size=1)
    eng.set_option("grid_min", 1)
    eng.set_option("grid_split", 1)
    eng.set_option("grid_group", 1)
    for arm in (30, -1, 0):
        eng.set_option("grid_arm", arm)
        eng.set_sequences_self(seqs)
        check_self(eng.search_self(C.BLOSUM50, 24, ms, mask_len=150, score_size=1), want)
        t = eng.timing()
        assert t["fill_forward_launches"] >= 3
        if arm == 30:
            assert t["byte_overflows"] > 5
    reset(eng, "grid_arm")
    # short sequences inside long ones: automatic arming cannot pay, the pilot is rejected and its queries run again
    rng = np.random.default_rng(99)
    tq = [rng.integers(0, 20, size=40).astype(np.int8) for _ in range(64)]
    tt = []
    for k in range(12):
        t = rng.integers(0, 20, size=260).astype(np.int8)
        a = int(rng.integers(0, 200))
        t[a: a + 40] = tq[k % 6]
        tt.append(t)
    seqs = tq + tt
    want = expected_self(seqs, C.BLOSUM50, 24, 12, 2, 40, mask_len=20, score_size=1)
    launches = {}
    for arm in (0, -1):
        eng.set_option("grid_arm", arm)
        eng.set_sequences_self(seqs)                                    # forgets that arming did not pay before
        got = eng.search_self(C.BLOSUM50, 24, 40, gap_open=12, gap_extend=2, mask_len=20, score_size=1)
        t = eng.timing()
        assert t["byte_overflows"] == 0, t                              # the rejected pilot's re-dos are dropped
        check_self(got, want)
        launches[arm] = t["fill_forward_launches"]
    # the rejected pilot group runs once more, then the groups of arming off follow
    assert launches[-1] == launches[0] + 1 and launches[0] >= 3, launches
    reset(eng, "grid_min", "grid_split", "grid_group", "grid_arm")
    eng.close()


def case_tiles(gpu):
    """grid tiles of 1, 2, 3, 7, n - 1 and n references give identical arrays"""
    L, eng = _engine(gpu)
    seqs = protein_set()
    n = len(seqs)
    ms = _ms(seqs, **PROT)
    eng.set_sequences_self(seqs)
    eng.set_option("grid_min", 1)
    eng.set_option("grid_arm", 0)
    base = eng.search_self(C.BLOSUM50, 24, ms, **PROT)
    cells = eng.timing()["cells_forward"]
    for tile in (1, 2, 3, 7, n - 1, n):
        eng.set_option("grid_tile_refs", tile)
        same_all(eng.search_self(C.BLOSUM50, 24, ms, **PROT), base)
        assert eng.timing()["cells_forward"] == cells, tile
    reset(eng, "grid_min", "grid_arm", "grid_tile_refs")
    eng.close()


def case_leftovers(gpu):
    """queries over 640 rows, references above a lowered grid_max_ref and pairs with both ends off the grid go through the
    general path; leftover_pairs counts the triangle's pairs only"""
    L, eng = _engine(gpu)
    seqs = protein_set() + [np.random.default_rng(4).integers(0, 20, size=n).astype(np.int8) for n in (700, 900, 1100)]
    n = len(seqs)
    lens = np.array([len(s) for s in seqs])
    _, rank = canon(seqs)
    ms = _ms(seqs, **PROT)
    want = expected_self(seqs, C.BLOSUM50, 24, 3, 1, ms, **PROT)
    eng.set_sequences_self(seqs)
    eng.set_option("grid_min", 1)
    for max_ref in (-1, 1000):
        eng.set_option("grid_max_ref", max_ref)
        got = eng.search_self(C.BLOSUM50, 24, ms, **PROT)
        check_self(got, want)
        lim = 65536 if max_ref < 0 else max_ref
        # off the grid: a query over 640 rows against everything after it, an on-grid query against the references above the
        # limit after it; the empty sequence's pairs are not computed
        left = sum(int((rank > rank[i]).sum()) if lens[i] > 640 else int(((rank > rank[i]) & (lens > lim)).sum()) if lens[i] else 0
                   for i in range(n))
        t = eng.timing()
        assert t["leftover_pairs"] == left and left > 0, (t["leftover_pairs"], left)
        assert t["fill_forward_launches"] > 0
    reset(eng, "grid_min", "grid_max_ref")
    eng.close()


def case_max_hits(gpu):
    """the call succeeds exactly at max_hits; one below it returns -2 and no set"""
    L, eng = _engine(gpu)
    seqs = protein_set()
    ms = _ms(seqs, **PROT)
    eng.set_sequences_self(seqs)
    for gm in (1, NEVER_GRID):
        eng.set_option("grid_min", gm)
        got = eng.search_self(C.BLOSUM50, 24, ms, **PROT)
        m = len(got[1])
        assert m > 0
        same_all(eng.search_self(C.BLOSUM50, 24, ms, max_hits=m, **PROT), got)
        with pytest.raises(RuntimeError, match="max_hits"):
            eng.search_self(C.BLOSUM50, 24, ms, max_hits=m - 1, **PROT)
    reset(eng, "grid_min")
    eng.close()


def case_refusals_and_self_mode(gpu):
    """each refusal of the contract; after set_sequences_self, align / search / search_all equal their results after
    set_sequences(S, S)"""
    L, eng = _engine(gpu)
    seqs = protein_set(empty=False)
    eng.set_option("grid_min", 1)
    f = eng.lib.ssw_engine_search_self
    f.argtypes = [ct.c_void_p, ct.c_void_p, ct.c_int32, ct.c_int64, ct.POINTER(ct.c_void_p)]
    f.restype = ct.c_int

    def refused(**kw):
        mat = kw.pop("mat", C.BLOSUM50)
        a, p = (None, None) if mat is None else L._i8(mat)
        P = L.BatchParams(p, 24, kw.get("gap_open", 3), kw.get("gap_extend", 1), 0, 0, 0, -1, 1)
        h = ct.c_void_p(1)
        assert f(eng.h, ct.byref(P), 0, 1 << 20, ct.byref(h)) == -1 and not h.value

    eng.set_sequences(seqs, seqs)
    refused()                                                          # not set by set_sequences_self
    eng.set_sequences_self(seqs)
    refused(gap_open=1, gap_extend=1)
    refused(gap_open=2, gap_extend=3)
    asym = C.BLOSUM50.copy().reshape(24, 24)
    asym[2, 5] += 1
    refused(mat=asym.reshape(-1))
    refused(mat=None)
    ok = C.BLOSUM50.copy().reshape(24, 24)
    ok[23, 23] = 9                                                      # symmetric: the diagonal is free
    eng.search_self(ok.reshape(-1), 24, 50, **PROT)
    prof = [C.BLOSUM50.reshape(24, 24)[s] for s in seqs[:3]]
    eng.set_profiles(prof, seqs[:3], 24)
    refused(mat=None)
    # self mode leaves align / search / search_all as after set_sequences(S, S)
    ms = _ms(seqs, **PROT)
    outs = []
    for setter in (lambda: eng.set_sequences(seqs, seqs), lambda: eng.set_sequences_self(seqs)):
        setter()
        res, pool = eng.align(C.BLOSUM50, 24, 3, 1, flag=0x0f, **PROT)
        outs.append((res, pool, eng.search(C.BLOSUM50, 24, 4, **PROT), eng.search_all(C.BLOSUM50, 24, ms, flag=0x0f, **PROT)))
    (ra, pa, sa, aa), (rb, pb, sb, ab) = outs
    assert C.compare_records(rb, pb, ra, pa) == []
    for x, y in zip(sa[:3], sb[:3]):
        assert np.array_equal(x, y)
    same_all(ab, aa)
    eng.set_sequences_self(seqs)
    eng.set_sequences(seqs[:5], seqs)                                   # ends self mode
    refused()
    reset(eng, "grid_min")
    eng.close()


def case_counters(gpu):
    """an even number of equal-length sequences, grid_arm 0: the self-search fills n^2 / 4 query-pair items, the full search
    n^2 / 2, so cells_forward is exactly half"""
    L, eng = _engine(gpu)
    seqs = equal_set(12)
    eng.set_option("grid_min", 1)
    eng.set_option("grid_arm", 0)
    eng.set_sequences(seqs, seqs)
    full = eng.search_all(C.BLOSUM50, 24, 40, **PROT)
    t_all = eng.timing()
    eng.set_sequences_self(seqs)
    got = eng.search_self(C.BLOSUM50, 24, 40, **PROT)
    t = eng.timing()
    assert t["leftover_pairs"] == 0 and t_all["leftover_pairs"] == 0
    assert 2 * t["cells_forward"] == t_all["cells_forward"] > 0, (t["cells_forward"], t_all["cells_forward"])
    assert 2 * t["grid_cols_useful"] == t_all["grid_cols_useful"]
    check_mirror(got, full, seqs)
    reset(eng, "grid_min", "grid_arm")
    eng.close()


def case_group(gpu):
    """device groups of 1 .. 5 emulated devices (1 .. 3 engines on one GPU) give exactly the one-engine result, flags 0 and 0x0f"""
    L, eng = _engine(gpu)
    seqs = protein_set()
    ms = _ms(seqs, **PROT)
    eng.set_option("grid_min", 1)
    eng.set_sequences_self(seqs)
    one = {flag: eng.search_self(C.BLOSUM50, 24, ms, flag=flag, **PROT) for flag in (0, 0x0f)}
    eng.close()
    for nd in ((1, 2, 3) if gpu else (1, 2, 3, 4, 5)):
        if not gpu:
            os.environ["SSW_EMU_DEVICES"] = str(nd)
        try:
            g = _group(L, gpu, nd)
            g.set_option("grid_min", 1)
            g.set_option("latency_cols", 0)
            for flag in (0, 0x0f):
                same_all(g.search_self(seqs, C.BLOSUM50, 24, ms, flag=flag, **PROT), one[flag])
            g.close()
        finally:
            os.environ.pop("SSW_EMU_DEVICES", None)


def test_search_self_entry_points_declared_and_exported():
    """the new names are declared in include/ssw_batch.h and exported by the libraries that are built; the rank-range entry
    point is not public"""
    import re
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(C.ROOT, "include", "ssw_batch.h")).read(), flags=re.S)
    for name in ("ssw_engine_set_sequences_self", "ssw_engine_search_self", "ssw_group_search_self"):
        assert re.search(r"\bint %s\(" % name, txt), name
        for lib in (C.LIB_OURS, os.path.join(EMU_DIR, "libssw_emu.so")):
            if os.path.exists(lib):
                assert hasattr(ct.CDLL(lib), name), (lib, name)
    assert "search_self_ranks" not in txt


CASES = [case_checker, case_mirror, case_dna, case_paths, case_launch_groups, case_tiles, case_leftovers, case_max_hits,
         case_refusals_and_self_mode, case_counters, case_group]


@pytest.mark.parametrize("case", CASES, ids=[c.__name__[5:] for c in CASES])
def test_search_self_emulated(case, capfd):
    case(False)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.__name__[5:] for c in CASES])
def test_search_self_gpu(case, capfd):
    case(True)


@pytest.mark.gpu
def test_search_self_config4_scale(capfd):
    """about 8,000 config-4-like proteins with planted families on the device path: the mirror identity against the full
    search_all, and the checker on a sample of rows"""
    L, eng = _engine(True)
    W = mixed_workload(100, 7900, seed=77, n_long_t=0, n_long_q=0)
    seqs = W["queries"] + W["refs"]
    n = len(seqs)
    eng.set_sequences(seqs, seqs)
    full = eng.search_all(C.BLOSUM50, 24, 150, **PROT)
    t_all = eng.timing()
    eng.set_sequences_self(seqs)
    got = eng.search_self(C.BLOSUM50, 24, 150, **PROT)
    t = eng.timing()
    _, rank = canon(seqs)
    lens = np.array([len(s) for s in seqs])
    # only pairs of two sequences over 640 aa are left to the general path (the shorter is the query)
    assert t["leftover_pairs"] == sum(int((rank > rank[i]).sum()) for i in np.nonzero(lens > 640)[0])
    assert t["fill_forward_launches"] > 1
    assert t["cells_forward"] < 0.55 * t_all["cells_forward"], (t["cells_forward"], t_all["cells_forward"])
    assert check_mirror(got, full, seqs) > 500
    sel = np.linspace(0, n - 1, 16).astype(int)
    pq = np.concatenate([np.full(int((rank > rank[i]).sum()), i) for i in sel]).astype(np.int64)
    pr = np.concatenate([np.nonzero(rank > rank[i])[0] for i in sel]).astype(np.int64)
    exp, ep, _, _, _ = C.cpu_batch(seqs, seqs, pq, pr, C.BLOSUM50, 24, 3, 1, **PROT)
    m = hit_mask(exp, 150)
    for i in sel:
        a, b = int(got[0][i]), int(got[0][i + 1])
        rows = m & (pq == i)
        assert list(got[1][a:b]) == list(pr[rows]), i
        assert C.compare_records(got[2][a:b], got[3], exp[rows], ep) == [], i
    eng.close()
