"""Block mode (fill kernel CM == 2) keeps no best cell: the resolve takes the score and the first block holding it from the
block maxima, and re-fills that block with best-cell tracking for the first column and the smallest row (DESIGN 2, 4.2).

The cases put the best cell in the first, a middle and the last block, on both sides of a block boundary, in two blocks
at once (the first must win), at the end of a reference whose length is not a multiple of 8, inside chunk warm-ups
(forced chunks of 64 and 128 columns), and give reads that overflow the byte limit, score 0, or have L mod 16 = 8
(byte rows) and != 8 (word rows), with mask windows of 15 and 75 columns.  Every field must match the checker, and
block mode must give what column mode gives."""
import subprocess

import numpy as np
import pytest

import common as C
from test_byte_on_word_rows import EMU_DIR, _pkg

GAP_O, GAP_E = 3, 1
REF_LEN = 2083                 # 33 blocks, the last one 35 columns, not a multiple of 8


def _cases(n_extra):
    """(ref, reads): reads copied (exactly or with edits) from chosen places of the reference, and n_extra mutated 150 bp
    reads (a pass of many items per CTA on the device)."""
    rng = np.random.default_rng(9090)
    ref = rng.integers(0, 4, size=REF_LEN).astype(np.int8)
    ref[1500:1600] = ref[700:800]                   # the same 100 columns twice: equal maxima in two blocks
    reads = []
    for L in (150, 152, 100):                       # L mod 16 = 6 (word rows), 8 (byte rows), 4
        for end in (L - 1, 639, 640, 1023, 1100, REF_LEN - 1):      # last read column at this reference column
            reads.append(ref[end - L + 1: end + 1].copy())          # exact: byte overflow for L >= 127
            reads.append(C.mutate_read(rng, ref, end - L + 1, L, 0.12, 0.01, 0.01))
    reads.append(ref[705:795].copy())               # lies in both copies: the first one wins
    reads.append(C.mutate_read(rng, ref, 710, 80, 0.1, 0.0, 0.0))
    reads.append(np.full(120, 4, dtype=np.int8))    # all N: score 0
    reads.append(np.tile(np.array([0, 1], dtype=np.int8), 60))     # periodic: equal values down a column
    for _ in range(6):
        reads.append(C.mutate_read(rng, ref, int(rng.integers(0, REF_LEN - 160)), int(rng.integers(90, 153)), 0.15, 0.02, 0.02))
    for _ in range(n_extra):
        reads.append(C.mutate_read(rng, ref, int(rng.integers(0, REF_LEN - 160)), 150, 0.1, 0.0, 0.0))
    return ref, reads


def _check(eng, n_extra):
    ref, reads = _cases(n_extra)
    mat = C.dna_matrix(2, 2)
    n = len(reads)
    eng.set_sequences(reads, [ref])
    for mask in (15, 75):
        exp, exp_pool, _, _, _ = C.cpu_batch(reads, [ref], np.arange(n), np.zeros(n), mat, 5, GAP_O, GAP_E, flag=0,
                                            mask_len=mask, score_size=2, threads=4)
        assert any(int(r["score1"]) >= 253 for r in exp) and any(int(r["score1"]) == 0 for r in exp)
        eng.set_option("cm_block", 0)
        col, col_pool = eng.align(mat, 5, GAP_O, GAP_E, flag=0, mask_len=mask, score_size=2)
        assert C.compare_records(col, col_pool, exp, exp_pool) == []
        eng.set_option("cm_block", 1)
        for chunk in (0, 64, 128):
            eng.set_option("chunk", chunk)
            res, pool = eng.align(mat, 5, GAP_O, GAP_E, flag=0, mask_len=mask, score_size=2)
            bad = C.compare_records(res, pool, exp, exp_pool)
            assert bad == [], (mask, chunk, bad, [(res[i], exp[i]) for i in bad[:2]])
            assert C.compare_records(res, pool, col, col_pool) == []
        eng.set_option("chunk", 0)


def test_emulated_block_best():
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    L = _pkg()
    eng = L.BatchAligner(lib_dir=EMU_DIR, lib_name="libssw_emu.so")
    eng.set_option("latency_cols", 0)
    _check(eng, 0)
    eng.close()


@pytest.mark.gpu
def test_gpu_block_best():
    L = _pkg()
    eng = L.BatchAligner(device=0)
    eng.set_option("latency_cols", 0)
    _check(eng, 80)
    eng.close()
