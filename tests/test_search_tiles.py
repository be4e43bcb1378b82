"""Grid tiles: the top-k search (ssw_engine_search) and the threshold search (ssw_engine_search_all) over a grid whose references
are cut into contiguous tiles, each run as a grid of its own.  The "grid_tile_refs" option forces small tiles; the automatic
cut only tiles grids of more than 2^31 - 1 pairs (or whose per-query-pair scratch exceeds the launch budget), which the last
case builds on the GPU.

Every tiled result must be the same arrays as the untiled grid, the general path and the checker's grid (C.cpu_batch: the
compiled reference where present, the oracle port otherwise).  Top-k tables of later tiles are merged on the device
(ssw_grid_merge_kernel); ties across a tile boundary go to the smaller reference index.  The cases run on the CPU emulator build
and, marked gpu, on the CUDA library."""
import os
import time

import numpy as np
import pytest

import common as C
from test_search import NEVER_GRID, _engine, _group, check, dna_grid, grid_records, same, tie_grid
from test_search_all import check_all, reset, same_all
from test_search_mixed import PROT, small_grid


def n_tiles(n_r, tile):
    return 1 if tile <= 0 else -(-n_r // tile)


def tile_sizes(n_r):
    return sorted({1, 2, 3, 7, n_r - 1, n_r, 0} - {-1})


def same_counters(t, t0, tiles):
    """what a tiled call reports against the untiled call on the same inputs"""
    assert t["grid_cols_useful"] == t0["grid_cols_useful"] > 0
    assert t["leftover_pairs"] == t0["leftover_pairs"]
    assert t["byte_overflows"] == t0["byte_overflows"]
    assert t["fill_forward_launches"] >= tiles


# ---------------------------------------------------------------------------------------------------------------------
# cases (each runs on the emulator build and on the GPU)
# ---------------------------------------------------------------------------------------------------------------------

def case_topk(gpu):
    """DNA (score sizes 0, 1, 2) and protein grids, k = 1, 3 and more than a row's hits, every tile size: the untiled grid's
    arrays, the general path's and the checker's top-k"""
    L, eng = _engine(gpu)
    mat = C.dna_matrix(2, 2)
    queries, refs = dna_grid()
    nq, nr = len(queries), len(refs)
    eng.set_sequences(queries, refs)
    eng.set_option("grid_min", 1)
    for ss in (2, 1, 0):
        exp, ep = grid_records(queries, refs, mat, 5, 3, 1, score_size=ss)
        for k in (1, 3, nr + 2):
            eng.set_option("grid_tile_refs", 0)
            base = eng.search(mat, 5, k, score_size=ss)
            t0 = eng.timing()
            check(base, exp, ep, nq, nr, k, 0)
            if ss == 2:
                assert t0["byte_overflows"] > 0
            for tile in tile_sizes(nr):
                eng.set_option("grid_tile_refs", tile)
                got = eng.search(mat, 5, k, score_size=ss)
                same_counters(eng.timing(), t0, n_tiles(nr, tile))
                same(got, base)
            eng.set_option("grid_min", NEVER_GRID)
            same(eng.search(mat, 5, k, score_size=ss), base)
            eng.set_option("grid_min", 1)
    queries, refs = small_grid()
    nq, nr = len(queries), len(refs)
    eng.set_sequences(queries, refs)
    exp, ep = grid_records(queries, refs, C.BLOSUM50, 24, 3, 1, **PROT)
    eng.set_option("grid_arm", 0)                         # a rejected pilot counts its columns twice, over its own tile
    for k in (1, 3, nr + 2):
        eng.set_option("grid_tile_refs", 0)
        base = eng.search(C.BLOSUM50, 24, k, **PROT)
        t0 = eng.timing()
        assert t0["leftover_pairs"] == 0
        check(base, exp, ep, nq, nr, k, 0)
        for tile in (1, 7, nr - 1):
            eng.set_option("grid_tile_refs", tile)
            got = eng.search(C.BLOSUM50, 24, k, **PROT)
            same_counters(eng.timing(), t0, n_tiles(nr, tile))
            same(got, base)
    reset(eng, "grid_min", "grid_arm", "grid_tile_refs")
    eng.close()


def case_tile_ties(gpu):
    """tie_grid: query 0 scores the same against references 0, 2, 4, 6, 8 and 10; tiles that split that run with the k-th place
    inside it keep the smaller reference indices"""
    L, eng = _engine(gpu)
    mat = C.dna_matrix(2, 2)
    queries, refs = tie_grid()
    nq, nr = len(queries), len(refs)
    eng.set_sequences(queries, refs)
    exp, ep = grid_records(queries, refs, mat, 5, 3, 1)
    s0 = exp["score1"][:nr]
    assert len({int(s0[r]) for r in (0, 2, 4, 6, 8, 10)}) == 1 and int(s0[0]) == int(s0.max())
    eng.set_option("grid_min", 1)
    for k in (2, 3, 4, 5):
        eng.set_option("grid_tile_refs", 0)
        base = eng.search(mat, 5, k)
        check(base, exp, ep, nq, nr, k, 0)
        assert list(base[0][0]) == [0, 2, 4, 6, 8][:k]
        for tile in (1, 2, 3, 4, 5, 6, 9):
            eng.set_option("grid_tile_refs", tile)
            got = eng.search(mat, 5, k)
            assert eng.timing()["fill_forward_launches"] >= n_tiles(nr, tile)
            same(got, base)
    reset(eng, "grid_min", "grid_tile_refs")
    eng.close()


def case_threshold(gpu):
    """search_all over tiles at min_score 0, 1, a middle value and above every score: the checker's filtered grid and the
    untiled arrays"""
    L, eng = _engine(gpu)
    mat = C.dna_matrix(2, 2)
    queries, refs = dna_grid()
    nq, nr = len(queries), len(refs)
    eng.set_sequences(queries, refs)
    eng.set_option("grid_min", 1)
    for ss in (2, 0):
        exp, ep = grid_records(queries, refs, mat, 5, 3, 1, score_size=ss)
        top = int(exp["score1"].max())
        for ms in (0, 1, 40, top + 1):
            eng.set_option("grid_tile_refs", 0)
            base = eng.search_all(mat, 5, ms, score_size=ss)
            t0 = eng.timing()
            check_all(base, exp, ep, nq, nr, ms)
            for tile in tile_sizes(nr):
                eng.set_option("grid_tile_refs", tile)
                got = eng.search_all(mat, 5, ms, score_size=ss)
                same_counters(eng.timing(), t0, n_tiles(nr, tile))
                same_all(got, base)
    queries, refs = small_grid()
    nq, nr = len(queries), len(refs)
    eng.set_sequences(queries, refs)
    exp, ep = grid_records(queries, refs, C.BLOSUM50, 24, 3, 1, **PROT)
    ms = int(np.percentile(exp["score1"], 70))
    eng.set_option("grid_tile_refs", 0)
    base = eng.search_all(C.BLOSUM50, 24, ms, **PROT)
    check_all(base, exp, ep, nq, nr, ms)
    for tile in (1, 7, nr - 1):
        eng.set_option("grid_tile_refs", tile)
        same_all(eng.search_all(C.BLOSUM50, 24, ms, **PROT), base)
    reset(eng, "grid_min", "grid_tile_refs")
    eng.close()


def case_redo_in_tiles(gpu):
    """re-done pairs inside later tiles: arming tail 30 over launch groups (re-dos in the tiles), a rejected pilot group in the
    first tile; both searches equal the untiled run"""
    L, eng = _engine(gpu)
    W = C.config_workload(4, n_queries=6, n_targets=41)
    eng.set_sequences(W["queries"], W["refs"])
    exp, ep = grid_records(W["queries"], W["refs"], C.BLOSUM50, 24, 3, 1, mask_len=150, score_size=1)
    ms = int(np.percentile(exp["score1"], 80))
    for o, v in (("grid_min", 1), ("grid_split", 1), ("grid_group", 1), ("grid_arm", 30)):
        eng.set_option(o, v)
    eng.set_option("grid_tile_refs", 0)
    base_k = eng.search(C.BLOSUM50, 24, 5, mask_len=150, score_size=1)
    t0 = eng.timing()
    assert t0["byte_overflows"] > 20
    check(base_k, exp, ep, 6, 41, 5, 0)
    base_a = eng.search_all(C.BLOSUM50, 24, ms, mask_len=150, score_size=1)
    check_all(base_a, exp, ep, 6, 41, ms)
    for tile in (5, 10, 40):
        eng.set_option("grid_tile_refs", tile)
        same(eng.search(C.BLOSUM50, 24, 5, mask_len=150, score_size=1), base_k)
        same_counters(eng.timing(), t0, n_tiles(41, tile))
        same_all(eng.search_all(C.BLOSUM50, 24, ms, mask_len=150, score_size=1), base_a)
        assert eng.timing()["byte_overflows"] == t0["byte_overflows"]
    reset(eng, "grid_split", "grid_group", "grid_arm", "grid_tile_refs")

    rng = np.random.default_rng(99)                       # test_search_all.case_rejected_pilot's grid
    tq = [rng.integers(0, 20, size=40).astype(np.int8) for _ in range(6)]
    tt = []
    for k in range(30):
        t = rng.integers(0, 20, size=260).astype(np.int8)
        a = int(rng.integers(0, 200))
        t[a: a + 40] = tq[k % 6]
        tt.append(t)
    exp, ep = grid_records(tq, tt, C.BLOSUM50, 24, 12, 2, mask_len=20, score_size=1)
    eng.set_option("grid_split", 1)
    eng.set_option("grid_group", 1)
    for tile in (0, 10):
        eng.set_option("grid_tile_refs", tile)
        eng.set_sequences(tq, tt)                         # forgets that arming did not pay before
        got = eng.search(C.BLOSUM50, 24, 4, gap_open=12, gap_extend=2, mask_len=20, score_size=1)
        t = eng.timing()
        assert t["fill_forward_launches"] == 3 * n_tiles(30, tile) + 1 and t["byte_overflows"] == 0, t   # the pilot twice
        check(got, exp, ep, 6, 30, 4, 0)
        eng.set_sequences(tq, tt)
        got = eng.search_all(C.BLOSUM50, 24, 60, gap_open=12, gap_extend=2, mask_len=20, score_size=1)
        t = eng.timing()
        assert t["fill_forward_launches"] == 3 * n_tiles(30, tile) + 1 and t["byte_overflows"] == 0, t
        check_all(got, exp, ep, 6, 30, 60)
    reset(eng, "grid_min", "grid_split", "grid_group", "grid_tile_refs")
    eng.close()


def case_leftovers_in_tiles(gpu):
    """references above grid_max_ref between the tiles' references, and queries off the grid: the untiled arrays"""
    L, eng = _engine(gpu)
    eng.set_option("grid_min", 1)
    eng.set_option("grid_arm", 0)
    for long_t, long_q, max_ref in (((1200, 2500, 1800), (), 1000), ((), (700, 1100), -1)):
        queries, refs = small_grid(long_t=long_t, long_q=long_q)
        nq, nr = len(queries), len(refs)
        eng.set_sequences(queries, refs)
        eng.set_option("grid_max_ref", max_ref)
        exp, ep = grid_records(queries, refs, C.BLOSUM50, 24, 3, 1, **PROT)
        ms = int(np.percentile(exp["score1"], 70))
        eng.set_option("grid_tile_refs", 0)
        base_k = eng.search(C.BLOSUM50, 24, 6, **PROT)
        t0 = eng.timing()
        assert t0["leftover_pairs"] > 0
        check(base_k, exp, ep, nq, nr, 6, 0)
        base_a = eng.search_all(C.BLOSUM50, 24, ms, **PROT)
        check_all(base_a, exp, ep, nq, nr, ms)
        for tile in (7,):
            eng.set_option("grid_tile_refs", tile)
            same(eng.search(C.BLOSUM50, 24, 6, **PROT), base_k)
            same_counters(eng.timing(), t0, n_tiles(nr - (3 if long_t else 0), tile))
            same_all(eng.search_all(C.BLOSUM50, 24, ms, **PROT), base_a)
    reset(eng, "grid_min", "grid_arm", "grid_max_ref", "grid_tile_refs")
    eng.close()


def case_flags_tiles(gpu):
    """flag 0x0f over tiles: begins and CIGARs of both searches equal align of the hit pairs"""
    L, eng = _engine(gpu)
    mat = C.dna_matrix(2, 2)
    queries, refs = dna_grid()
    nq = len(queries)
    eng.set_sequences(queries, refs)
    eng.set_option("grid_min", 1)
    eng.set_option("grid_tile_refs", 2)
    kw = dict(flag=0x0f, filterd=32767, score_size=2)
    got = eng.search_all(mat, 5, 30, **kw)
    assert (got[2]["cigar_len"] > 0).any()
    hq = np.repeat(np.arange(nq), np.diff(got[0]))
    res, pool = eng.align(mat, 5, 3, 1, pair_query=hq, pair_ref=got[1], **kw)
    same_all(got, (got[0], got[1], res, pool))
    hit_ref, hits, n_hits, kpool = eng.search(mat, 5, 3, min_score=30, **kw)
    m = np.arange(3)[None, :] < n_hits[:, None]
    res, pool = eng.align(mat, 5, 3, 1, pair_query=np.nonzero(m)[0], pair_ref=hit_ref[m], **kw)
    assert C.compare_records(hits[m], kpool, res, pool) == []
    eng.set_option("grid_tile_refs", 0)
    same(eng.search(mat, 5, 3, min_score=30, **kw), (hit_ref, hits, n_hits, kpool))
    reset(eng, "grid_min", "grid_tile_refs")
    eng.close()


def case_max_hits_tiles(gpu):
    """a max_hits bound first passed in the second tile ends the call with -2 and no set; a bound equal to the count holds"""
    L, eng = _engine(gpu)
    mat = C.dna_matrix(2, 2)
    queries, refs = dna_grid()
    eng.set_sequences(queries, refs)
    eng.set_option("grid_min", 1)
    eng.set_option("grid_tile_refs", 3)
    for ms in (1, 30):
        got = eng.search_all(mat, 5, ms, score_size=1)       # word scores: every hit is final on the grid
        n, n_first = len(got[1]), int((got[1] < 3).sum())
        assert 0 < n_first < n
        with pytest.raises(RuntimeError, match="max_hits"):
            eng.search_all(mat, 5, ms, max_hits=n_first, score_size=1)
        assert eng.timing()["fill_forward_launches"] >= 2        # the bound held through the first tile
        same_all(eng.search_all(mat, 5, ms, max_hits=n, score_size=1), got)
    reset(eng, "grid_min", "grid_tile_refs")
    eng.close()


def case_group_tiles(gpu):
    """groups of several devices with tiles on every engine, codes and text with reverse complements: one untiled engine's
    arrays"""
    L, eng = _engine(gpu)
    queries, refs = dna_grid()
    mat = C.dna_matrix(2, 2)
    rcq = [(3 - q)[::-1].astype(np.int8) for q in queries]
    eng.set_sequences(queries + rcq, refs)
    eng.set_option("grid_min", 1)
    one_k = eng.search(mat, 5, 3, min_score=20, score_size=2)
    one_a = eng.search_all(mat, 5, 20, score_size=2)
    eng.close()
    text_q = ["".join("ACGT"[c] for c in q) for q in queries]
    text_r = ["".join("ACGT"[c] for c in r) for r in refs]
    table = np.full(128, 4, dtype=np.int8)
    for i, c in enumerate("ACGT"):
        table[ord(c)] = i
    for world in ((1, 2) if gpu else (1, 2, 3, 5)):
        if not gpu:
            os.environ["SSW_EMU_DEVICES"] = str(world)
        try:
            grp = _group(L, gpu, world)
            grp.set_option("grid_min", 1)
            grp.set_option("latency_cols", 0)
            grp.set_option("grid_tile_refs", 2)
            got_k = grp.search(text_q, text_r, mat, 5, 3, min_score=20, table=table, add_reverse_complement=True)
            got_a = grp.search_all(text_q, text_r, mat, 5, 20, table=table, add_reverse_complement=True)
            assert all(t["fill_forward_launches"] >= 3 for t in grp.timing() if t["grid_cols_useful"] > 0)
            grp.close()
        finally:
            os.environ.pop("SSW_EMU_DEVICES", None)
        same(got_k, one_k)
        same_all(got_a, one_a)


CASES = [case_topk, case_tile_ties, case_threshold, case_redo_in_tiles, case_leftovers_in_tiles, case_flags_tiles,
         case_max_hits_tiles, case_group_tiles]


@pytest.mark.parametrize("case", CASES, ids=[c.__name__[5:] for c in CASES])
def test_search_tiles_emulated(case, capfd):
    case(False)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.__name__[5:] for c in CASES])
def test_search_tiles_gpu(case, capfd):
    case(True)


@pytest.mark.gpu
def test_search_tiles_above_2g_pairs():
    """a self-search of 46,400 random proteins of 24-40 aa (BLOSUM50, word scores, automatic arming and tiles): 2.153e9 pairs,
    above the 2^31 - 1 that one grid numbers.  Both searches stay on the device path (no leftover pair); the rows of 64 spread
    queries equal an untiled search of those queries against every target, and hits of both searches match the checker."""
    rng = np.random.default_rng(2026)
    n = 46400
    seqs = [rng.integers(0, 20, size=int(m)).astype(np.int8) for m in rng.integers(24, 41, size=n)]
    assert n * n > 2 ** 31 - 1
    kw = dict(gap_open=10, gap_extend=1, mask_len=15, score_size=1)
    L, eng = _engine(True)
    eng.set_sequences(seqs, seqs)
    t_start = time.time()
    hit_ref, hits, n_hits, _ = eng.search(C.BLOSUM50, 24, 4, **kw)
    t_k = eng.timing()
    t_mid = time.time()
    thr = 60                                               # far above a random pair's score, below a self hit's
    got = eng.search_all(C.BLOSUM50, 24, thr, **kw)
    t_a = eng.timing()
    t_end = time.time()
    print("46,400 x 46,400 self-search: search(k = 4) %.1f s, search_all(%d) %.1f s, %d hits"
          % (t_mid - t_start, thr, t_end - t_mid, len(got[1])))
    for t in (t_k, t_a):
        assert t["leftover_pairs"] == 0 and t["fill_forward_launches"] >= 2, t
    assert (n_hits == 4).all()
    assert (np.diff(got[0]) >= 1).all()                   # every sequence finds itself
    sel = np.linspace(0, n - 1, 64).astype(int)
    eng.set_sequences([seqs[i] for i in sel], seqs)
    sub_k = eng.search(C.BLOSUM50, 24, 4, **kw)
    sub_a = eng.search_all(C.BLOSUM50, 24, thr, **kw)
    eng.close()
    assert np.array_equal(hit_ref[sel], sub_k[0]) and np.array_equal(n_hits[sel], sub_k[2])
    for f in C.CMP_FIELDS:
        assert np.array_equal(hits[sel][f], sub_k[1][f]), f
    rows = np.concatenate([np.arange(got[0][q], got[0][q + 1]) for q in sel]).astype(np.int64)
    sub_off = np.concatenate([[0], np.cumsum(np.diff(got[0])[sel])]).astype(np.int64)
    same_all((sub_off, got[1][rows], got[2][rows], got[3]), sub_a)
    # hits against the checker: the 4 best of 16 spread queries and the threshold hits of the same queries
    few = sel[::4]
    pq = np.repeat(few, 4)
    pr = hit_ref[few].reshape(-1)
    exp, ep, _, _, _ = C.cpu_batch(seqs, seqs, pq, pr, C.BLOSUM50, 24, 10, 1, mask_len=15, score_size=1)
    assert C.compare_records(hits[few].reshape(-1), None, exp, ep) == []
    rows = np.concatenate([np.arange(got[0][q], got[0][q + 1]) for q in few]).astype(np.int64)
    pq = np.repeat(few, np.diff(got[0])[few])
    exp, ep, _, _, _ = C.cpu_batch(seqs, seqs, pq, got[1][rows], C.BLOSUM50, 24, 10, 1, mask_len=15, score_size=1)
    assert C.compare_records(got[2][rows], None, exp, ep) == []
