"""The two forms of the fill kernel's cell (ssw_fill.cuh, ssw_cells):

    X form (column mode, re-fills, reverse pass, strips):  X = max(Hd + s, E, 0), H = max(X, F),
                                                            E' = max(E - gapE, X - gapO), F' = max(F - gapE, X - gapO)
    H form (block mode, CM == 2: configs 2 and 3):          H = max(Hd + s, E, F, 0),
                                                            E' = max(E - gapE, H - gapO), F' = max(F - gapE, H - gapO)

With gapO > gapE (the only case the fill kernels run) both give the same H and F in every cell; E differs by the term
F - gapO and never leaves the lane.  So block mode's block maxima must be the maxima of column mode's columns, and every
record must be the same.

1. The recurrences themselves, cell by cell in wrap-around 16-bit arithmetic, on random small matrices with dead rows.
2. Block mode (H form) against the oracle and against column mode (X form) on the emulator build, byte and word semantics,
   gap pairs at the gapO > gapE boundary, reads of 145-151 bp, reads with a deletion next to an insertion (the vertical-
   then-horizontal gap, where the forms' E differ), and chunks of 64 columns (block boundaries inside warm-ups).
3. GPU: the same on a config-2 slice: 1,000 x 150 bp against the 5 Mbp reference, block mode against column mode."""
import subprocess

import numpy as np
import pytest

import common as C
from test_byte_on_word_rows import EMU_DIR, _pkg

GAPS = [(2, 1), (3, 2), (3, 1), (5, 4), (6, 1)]


def _w16(v):
    return ((v + 32768) & 0xFFFF) - 32768


def _columns(score, gap_o, gap_e, from_h):
    """H and F of every cell, column by column, as the kernel computes one lane column (rows = score.shape[1])."""
    n_rows = score.shape[1]
    hd, e = [0] * n_rows, [0] * n_rows
    hs, fs = [], []
    for s in score:
        f, hn, fcol = 0, [0] * n_rows, [0] * n_rows
        for k in range(n_rows):
            t = _w16(hd[k] + int(s[k]))
            if from_h:
                h = max(t, e[k], f, 0)
                hg = _w16(h - gap_o)
                e[k] = max(_w16(e[k] - gap_e), hg)
                f = max(_w16(f - gap_e), hg)
            else:
                x = max(t, e[k], 0)
                xg = _w16(x - gap_o)
                e[k] = max(_w16(e[k] - gap_e), xg)
                h = max(x, f)
                f = max(_w16(f - gap_e), xg)
            hn[k], fcol[k] = h, f
        hd = [0] + hn[:-1]
        hs.append(hn)
        fs.append(fcol)
    return hs, fs


def test_cell_forms_same_h_and_f():
    rng = np.random.default_rng(2024)
    for trial in range(300):
        gap_o, gap_e = GAPS[trial % len(GAPS)]
        rows, cols = int(rng.integers(1, 30)), int(rng.integers(1, 60))
        dead = int(rng.integers(0, 4))
        if trial % 3 == 0:           # DNA-like: match / mismatch
            score = np.where(rng.random((cols, rows)) < 0.4, 2, -2)
        else:                        # protein-like spread
            score = rng.integers(-4, 12, size=(cols, rows))
        if dead:
            score[:, rows - min(dead, rows):] = -32768
        a = _columns(score, gap_o, gap_e, False)
        b = _columns(score, gap_o, gap_e, True)
        assert a == b, (trial, gap_o, gap_e)


def _cases():
    """(ref, reads): 145-151 bp reads copied exactly (byte overflow), with substitutions and indels, and with a deletion
    right next to an insertion; a few shorter reads for the other block-mode instances."""
    rng = np.random.default_rng(777)
    ref = rng.integers(0, 4, size=1500).astype(np.int8)
    reads = []
    for L in range(145, 152):
        start = int(rng.integers(0, len(ref) - L - 40))
        reads.append(ref[start: start + L].copy())
        reads.append(C.mutate_read(rng, ref, int(rng.integers(0, len(ref) - L - 40)), L, 0.08, 0.02, 0.02))
        a = int(rng.integers(0, len(ref) - L - 40))
        cut, d, i = int(rng.integers(30, L - 30)), int(rng.integers(1, 6)), int(rng.integers(1, 6))
        read = np.concatenate([ref[a: a + cut], rng.integers(0, 4, size=i), ref[a + cut + d: a + L + d - i]]).astype(np.int8)
        reads.append(read[:L])
    for L in (40, 64, 100):
        reads.append(C.mutate_read(rng, ref, int(rng.integers(0, len(ref) - L - 10)), L, 0.1, 0.03, 0.03))
    reads.append(np.full(150, 4, dtype=np.int8))                    # all N: score 0
    return ref, reads


def _check_emulated(eng):
    ref, reads = _cases()
    mat = C.dna_matrix(2, 2)
    n = len(reads)
    eng.set_sequences(reads, [ref])
    for gap_o, gap_e in GAPS:
        for score_size in (0, 1, 2):
            exp, exp_pool, _, _, _ = C.cpu_batch(reads, [ref], np.arange(n), np.zeros(n), mat, 5, gap_o, gap_e, flag=0,
                                                mask_len=75, score_size=score_size, threads=4)
            eng.set_option("cm_block", 0)
            col, col_pool = eng.align(mat, 5, gap_o, gap_e, flag=0, mask_len=75, score_size=score_size)
            assert C.compare_records(col, col_pool, exp, exp_pool) == [], (gap_o, gap_e, score_size)
            eng.set_option("cm_block", 1)
            for chunk in (0, 64):
                eng.set_option("chunk", chunk)
                res, pool = eng.align(mat, 5, gap_o, gap_e, flag=0, mask_len=75, score_size=score_size)
                bad = C.compare_records(res, pool, exp, exp_pool)
                assert bad == [], (gap_o, gap_e, score_size, chunk, bad, [(res[i], exp[i]) for i in bad[:2]])
                assert C.compare_records(res, pool, col, col_pool) == []
            eng.set_option("chunk", 0)


def test_emulated_cell_forms():
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    L = _pkg()
    eng = L.BatchAligner(lib_dir=EMU_DIR, lib_name="libssw_emu.so")
    eng.set_option("latency_cols", 0)
    _check_emulated(eng)
    eng.close()


@pytest.mark.gpu
def test_gpu_cell_forms_config2():
    """Config 2's shape (1,000 x 150 bp against 5 Mbp, block mode in one launch) against column mode, which computes
    every cell in the X form; at the config's gaps 3/1 and at 2/1."""
    w = C.config_workload(2)
    L = _pkg()
    eng = L.BatchAligner(device=0)
    eng.set_sequences(w["queries"], w["refs"])
    try:
        for gap_o, gap_e in ((w["gapO"], w["gapE"]), (2, 1)):
            args = dict(flag=w["flag"], mask_len=w["mask_len"], score_size=w["score_size"])
            eng.set_option("cm_block", -1)
            blk, blk_pool = eng.align(w["mat"], w["n"], gap_o, gap_e, **args)
            assert eng.timing()["fill_forward_launches"] >= 1
            eng.set_option("cm_block", 0)
            col, col_pool = eng.align(w["mat"], w["n"], gap_o, gap_e, **args)
            bad = C.compare_records(blk, blk_pool, col, col_pool)
            assert bad == [], (gap_o, gap_e, len(bad), [(blk[i], col[i]) for i in bad[:2]])
    finally:
        eng.close()
