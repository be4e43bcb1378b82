"""Byte semantics filled on the word rows (DESIGN 2): a read whose byte padding adds eight pad rows to a word padding that
already has one (length % 16 in 1..7, e.g. 150 bp: 152 rows instead of 160) is filled on its word rows, and the block-mode
resolve re-fills on the byte rows only the columns [e2, e2 + 8) right of the mask window.

The identity behind it is checked on a numpy restatement of the DESIGN 2 recurrence: with h = H of the last word row,
    C_byte(c) = max(C_word(c), max_{k=1..8} h(c - k))
for the column maxima C over the rows of either padding.  The end-to-end cases are built so that the byte second-best
score lies inside that zone, where a scan of the word column maxima would be wrong; the library (CPU emulator build, and
the real one on the GPU) must still match the reference in every field."""
import importlib.util
import os
import subprocess

import numpy as np
import pytest

import common as C

EMU_DIR = os.path.join(C.ROOT, "tests", "cuda_emu")


def _pkg():
    spec = importlib.util.spec_from_file_location("ssw_b200_lib", os.path.join(C.PKG, "ssw_lib.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def lp_of(length, word):
    g = 8 if word else 16
    return (length + g - 1) // g * g


def fill_rows(read, ref, mat, n, gap_o, gap_e, lp):
    """H of every cell (lp x len(ref)) of the DESIGN 2 recurrence: X = max(0, H(c-1,r-1)+s, E), H = max(X, F),
    E' = max(E-gapE, X-gapO), F(r+1) = max(F(r)-gapE, X(r)-gapO); pad rows (len(read) <= r < lp) score 0."""
    m = np.asarray(mat, dtype=np.int64).reshape(n, n)
    prof = np.zeros((lp, n), dtype=np.int64)
    prof[: len(read)] = m[:, np.asarray(read, dtype=np.int64)].T
    r_idx = np.arange(lp, dtype=np.int64)
    hp = np.zeros(lp, dtype=np.int64)
    e = np.zeros(lp, dtype=np.int64)
    out = np.zeros((lp, len(ref)), dtype=np.int64)
    for c, letter in enumerate(np.asarray(ref, dtype=np.int64)):
        diag = np.concatenate(([0], hp[:-1]))
        x = np.maximum(np.maximum(diag + prof[:, letter], e), 0)
        # F(0) = 0; F(r) = max(-r*gapE, max_{k<r} X(k) - gapO - (r-1-k)*gapE)
        a = np.maximum.accumulate(x - gap_o + r_idx * gap_e)
        f = np.empty(lp, dtype=np.int64)
        f[0] = 0
        f[1:] = np.maximum(-r_idx[1:] * gap_e, a[:-1] - (r_idx[1:] - 1) * gap_e)
        h = np.maximum(x, f)
        e = np.maximum(e - gap_e, x - gap_o)
        out[:, c] = h
        hp = h
    return out


def spill_identity_holds(read, ref, mat, n, gap_o, gap_e, spill_cols=None):
    """spill_cols: how many earlier columns of the last word row spill into a byte column maximum (default: one per extra
    byte pad row, as DESIGN 2 proves; fewer must break the identity)"""
    L = len(read)
    lw, lb = lp_of(L, 1), lp_of(L, 0)
    H = fill_rows(read, ref, mat, n, gap_o, gap_e, lb)
    cw, cb = H[:lw].max(axis=0), H.max(axis=0)
    h = np.concatenate((np.zeros(lb - lw, dtype=np.int64), H[lw - 1]))
    ks = range(1, (lb - lw if spill_cols is None else spill_cols) + 1)
    spill = np.max([h[lb - lw - k: lb - lw - k + len(ref)] for k in ks], axis=0)
    return np.array_equal(cb, np.maximum(cw, spill))


def second_best(colmax, end_ref, mask_len, word):
    """ssw.c:368-381 / :570-583: (largest value, first column) outside the mask window."""
    ref_len = len(colmax)
    e1 = max(end_ref - mask_len, 0)
    e2 = min(end_ref + mask_len, ref_len) + (0 if word else 1)
    v2, i2 = 0, 0
    for c in list(range(0, e1)) + list(range(e2, ref_len)):
        if colmax[c] > v2:
            v2, i2 = int(colmax[c]), c
    return v2, i2


def _adversarial_reads(rng, ref, L):
    start = int(rng.integers(0, len(ref) - L - 20))
    seg = ref[start: start + L].copy()
    yield seg                                                                   # exact copy
    yield np.concatenate([rng.integers(0, 4, size=L // 3), ref[start: start + L - L // 3]]).astype(np.int8)   # partial copy
    ins = seg.copy()
    ins[-3:] = rng.integers(0, 4, size=3)                                       # ends in an insertion / mismatches
    yield ins
    yield np.tile(seg[:5], L // 5 + 1)[:L].astype(np.int8)                       # repeat
    yield C.mutate_read(rng, ref, start, L, 0.1, 0.03, 0.03)


@pytest.mark.parametrize("length", list(range(145, 152)))
def test_byte_pad_rows_only_spill_the_last_word_row(length):
    rng = np.random.default_rng(1000 + length)
    settings = [(2, 2, 3, 1), (1, 3, 5, 2), (3, 6, 8, 1), (2, 1, 2, 1), (1, 1, 6, 2)]
    for match, mismatch, gap_o, gap_e in settings:
        mat = C.dna_matrix(match, mismatch)
        ref = rng.integers(0, 4, size=400).astype(np.int8)
        ref[200:260] = np.tile(ref[100:112], 5)                                  # a repeat region
        reads = list(_adversarial_reads(rng, ref, length)) + [rng.integers(0, 4, size=length).astype(np.int8)]
        for read in reads:
            assert spill_identity_holds(read, ref, mat, 5, gap_o, gap_e), (length, match, mismatch, gap_o, gap_e)


def _zone_cases(rng):
    """Reads whose byte second-best is decided inside [e2, e2 + 8).  The best cell lies in the last read row at column p;
    behind it the pad rows decay by a horizontal gap (1 per column), so column e2 = p + 16 (mask 15) sees about score1 - 16
    on the word rows, but score1 - 8 on the byte rows: their last row gets H(last word row, p + 8) diagonally."""
    ref_len = 2000
    ref = rng.integers(0, 4, size=ref_len).astype(np.int8)
    reads, want_zone = [], []

    def planted(L, end_col, head):
        """read = `head` random bases + the reference up to end_col (inclusive): best cell at (L - 1, end_col)"""
        tail = L - head
        return np.concatenate([rng.integers(0, 4, size=head), ref[end_col - tail + 1: end_col + 1]]).astype(np.int8)

    mask = 15
    for L, e2_target in ((150, 64 * 10), (150, 64 * 12 + 57), (150, 64 * 15 + 63), (149, 64 * 20), (145, 64 * 22 + 57),
                         (150, ref_len - 3), (149, ref_len - 6), (145, ref_len - 9)):
        end_col = e2_target - mask - 1
        reads.append(planted(L, end_col, 60))
        want_zone.append(True)
    reads.append(ref[300:450].copy())                           # overflows the byte limit (score 300): word re-fill
    reads.append(planted(150, 1400, 70))
    reads.append(planted(152, 1500, 60))                        # byte padding = word padding + 8 without a word pad row
    reads.append(planted(160, 1600, 70))                        # byte padding = word padding
    want_zone += [False] * 4
    return ref, reads, mask, want_zone


def _check_zone_cases(eng, cm_chunks, n_expected_zone=8):
    rng = np.random.default_rng(77)
    ref, reads, mask, want_zone = _zone_cases(rng)
    mat = C.dna_matrix(2, 2)
    n = len(reads)
    exp, exp_pool, _, _, _ = C.cpu_batch(reads, [ref], np.arange(n), np.zeros(n), mat, 5, 3, 1, flag=0, mask_len=mask,
                                        score_size=2, threads=4)
    zone_hits = 0
    for i, read in enumerate(reads):
        if not want_zone[i]:
            continue
        L = len(read)
        H = fill_rows(read, ref, mat, 5, 3, 1, lp_of(L, 0))
        cb, cw = H.max(axis=0), H[: lp_of(L, 1)].max(axis=0)
        end_ref = int(exp[i]["ref_end1"])
        assert int(exp[i]["score1"]) == int(cb.max()) and end_ref == int(np.argmax(cb))
        byte2 = second_best(cb, end_ref, mask, False)
        assert byte2 == (int(exp[i]["score2"]), int(exp[i]["ref_end2"])), i
        e2 = min(end_ref + mask, len(ref)) + 1
        assert e2 <= byte2[1] < e2 + 8 and second_best(cw, end_ref, mask, False) != byte2, i
        zone_hits += 1
    assert zone_hits == n_expected_zone
    assert {(int(exp[i]["ref_end1"]) + mask + 1) % 64 for i in range(3)} == {0, 57, 63}
    assert int(exp[n - 4]["score1"]) > 255                                     # the overflowing read: word result
    for chunk in cm_chunks:
        eng.set_option("chunk", chunk)
        res, pool = eng.align(mat, 5, 3, 1, flag=0, mask_len=mask, score_size=2)
        bad = C.compare_records(res, pool, exp, exp_pool)
        assert bad == [], (chunk, bad, [(res[i], exp[i]) for i in bad[:2]])
        assert eng.timing()["byte_overflows"] == 1


def _cells_of_150(eng, rows):
    """A batch of 150 bp reads alone (no overflow, one chunk): cells = pair-tasks x ref_len x rows x 2."""
    rng = np.random.default_rng(5)
    ref = rng.integers(0, 4, size=1800).astype(np.int8)
    reads = [C.mutate_read(rng, ref, int(rng.integers(0, 1600)), 150, 0.25, 0.02, 0.02) for _ in range(6)]
    eng.set_sequences(reads, [ref])
    eng.set_option("chunk", 0)
    mat = C.dna_matrix(2, 2)
    res, pool = eng.align(mat, 5, 3, 1, flag=0, mask_len=75, score_size=2)
    exp, exp_pool, _, _, _ = C.cpu_batch(reads, [ref], np.arange(6), np.zeros(6), mat, 5, 3, 1, flag=0, mask_len=75,
                                        score_size=2, threads=4)
    assert C.compare_records(res, pool, exp, exp_pool) == []
    t = eng.timing()
    assert t["byte_overflows"] == 0
    assert t["cells_forward"] == 3 * len(ref) * rows * 2, t["cells_forward"]


def test_emulated_byte_on_word_rows(capfd):
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    L = _pkg()
    eng = L.BatchAligner(lib_dir=EMU_DIR, lib_name="libssw_emu.so")
    eng.set_option("latency_cols", 0)
    eng.set_option("cm_block", 1)
    rng = np.random.default_rng(77)
    ref, reads, _, _ = _zone_cases(rng)
    eng.set_sequences(reads, [ref])
    _check_zone_cases(eng, (0, 64, 128))
    _cells_of_150(eng, 8 * 19)                   # 150 bp reads on 152 rows (the byte padding would be 160)
    eng.close()


@pytest.mark.gpu
def test_gpu_byte_on_word_rows():
    L = _pkg()
    eng = L.BatchAligner(device=0)
    eng.set_option("latency_cols", 0)
    eng.set_option("cm_block", 1)
    rng = np.random.default_rng(77)
    ref, reads, _, _ = _zone_cases(rng)
    eng.set_sequences(reads, [ref])
    _check_zone_cases(eng, (0, 64, 128))
    _cells_of_150(eng, 8 * 19)
    eng.close()
