"""Byte overflows of reads filled on their word rows are re-resolved, not re-filled (DESIGN 2, 4.2).

A byte alignment of a read with length % 16 in 1..7 is filled on its word rows (145..151 bp: 152 rows, instance (8,19)).
The fill never reads the semantics, so that fill IS the word fill of the read: when the byte score overflows, the word
result is resolved from the same column maxima and item bests, with word semantics (limit, end_ref of a zero score, the
e2 of the second-best scan) and without the byte-row zone item.  The batch below holds only such reads, several of
which overflow, so the whole forward phase is one fill launch.  One overflowing read has its word second-best exactly at
column end_ref + mask_len, which the word scan may take and the byte scan (from end_ref + mask_len + 1) may not."""
import subprocess

import numpy as np
import pytest

import common as C
from test_byte_on_word_rows import EMU_DIR, _pkg, fill_rows, lp_of, second_best

MASK = 15
GAP_O, GAP_E = 3, 1


def _cases(rng):
    """(ref, reads, overflowing, edge): reads of 145..151 bp, `overflowing` the indices of the reads whose byte score
    overflows, `edge` the read whose word second-best lies at end_ref + mask_len."""
    ref_len = 3000
    ref = rng.integers(0, 4, size=ref_len).astype(np.int8)
    reads, overflowing = [], []
    for i, L in enumerate(range(145, 152)):
        start = 100 + 380 * i
        # exact copy: score 2 L >= 290; the best cell is the last read row at column start + L - 1
        reads.append(ref[start: start + L].copy())
        overflowing.append(len(reads) - 1)
        # a mutated copy that stays below the byte limit
        reads.append(C.mutate_read(rng, ref, start + 150, L, 0.2, 0.02, 0.02))
    # near-exact copy with a few substitutions: still overflows, best cell not at the read end
    seg = ref[2800 - 148: 2800].copy()
    seg[[20, 60, 100]] = (seg[[20, 60, 100]] + 1) % 4
    reads.append(seg)
    overflowing.append(len(reads) - 1)
    edge = overflowing[5]                      # 150 bp exact copy
    return ref, reads, overflowing, edge


def _check(eng, chunks):
    rng = np.random.default_rng(4242)
    ref, reads, overflowing, edge = _cases(rng)
    assert {len(r) for r in reads} <= set(range(145, 152)) and len(reads[edge]) == 150
    mat = C.dna_matrix(2, 2)
    n = len(reads)
    eng.set_sequences(reads, [ref])
    exp, exp_pool, _, _, _ = C.cpu_batch(reads, [ref], np.arange(n), np.zeros(n), mat, 5, GAP_O, GAP_E, flag=0,
                                        mask_len=MASK, score_size=2, threads=4)
    limit_byte = 255 - 2                       # 255 - bias; bias = the largest mismatch penalty
    assert sorted(i for i in range(n) if int(exp[i]["score1"]) >= limit_byte) == overflowing

    # the edge read: the word scan takes column end_ref + mask_len, the byte scan cannot
    H = fill_rows(reads[edge], ref, mat, 5, GAP_O, GAP_E, lp_of(150, 1))
    cw = H.max(axis=0)
    end_ref = int(exp[edge]["ref_end1"])
    assert end_ref == int(np.argmax(cw)) and int(exp[edge]["score1"]) == int(cw.max())
    word2 = second_best(cw, end_ref, MASK, True)
    assert word2 == (int(exp[edge]["score2"]), int(exp[edge]["ref_end2"]))
    assert word2[1] == end_ref + MASK and second_best(cw, end_ref, MASK, False) != word2

    for chunk in chunks:
        eng.set_option("chunk", chunk)
        res, pool = eng.align(mat, 5, GAP_O, GAP_E, flag=0, mask_len=MASK, score_size=2)
        bad = C.compare_records(res, pool, exp, exp_pool)
        assert bad == [], (chunk, bad, [(res[i], exp[i]) for i in bad[:2]])
        t = eng.timing()
        assert t["byte_overflows"] == len(overflowing), (chunk, t["byte_overflows"])
        assert t["fill_forward_launches"] == 1, (chunk, t["fill_forward_launches"])    # no word re-fill launch


def test_emulated_byte_overflow_reresolve(capfd):
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    L = _pkg()
    eng = L.BatchAligner(lib_dir=EMU_DIR, lib_name="libssw_emu.so")
    eng.set_option("latency_cols", 0)
    eng.set_option("cm_block", 1)
    _check(eng, (0, 64, 128))
    eng.close()


@pytest.mark.gpu
def test_gpu_byte_overflow_reresolve():
    L = _pkg()
    eng = L.BatchAligner(device=0)
    eng.set_option("latency_cols", 0)
    eng.set_option("cm_block", 1)
    _check(eng, (0, 64, 128))
    eng.close()
