"""Block mode (fill kernel CM == 2) writes one packed word per 64 reference columns: the maximum of the block's column maxima.
The lanes of a group keep their own block maxima and combine them once per block (DESIGN 4.1), so these words are checked
directly, against the column-mode words (CM == 1, one per column) of the same call folded per 64 columns.

Cases: the instances (8,19), (16,19) and (32,16) (G = 8, 16 and 32 lanes per group), reads of mixed lengths in one launch,
references of 37 (shorter than one block), 64, 200 and 1,163 columns, and one chunk as well as forced chunks of 64 and 320
columns (first and later chunks, each with a warm-up)."""
import ctypes as ct
import subprocess

import numpy as np
import pytest

import common as C
from test_byte_on_word_rows import EMU_DIR, _pkg

GAP_O, GAP_E = 3, 1
# "inst" option value -> read lengths (all within the instance's rows, several padded lengths per launch)
INSTANCES = {15: (129, 137, 150), 14: (200, 251, 300), 8: (300, 390, 480)}
REF_LENS = (37, 64, 200, 1163)
CHUNKS = (0, 64, 320)


def _colmax(eng):
    f = eng.lib.ssw_engine_last_colmax
    f.argtypes = [ct.c_void_p, ct.POINTER(ct.c_uint32), ct.c_int64]
    f.restype = ct.c_int64
    n = f(ct.c_void_p(eng.h), None, 0)
    assert n > 0
    out = np.zeros(n, dtype=np.uint32)
    assert f(ct.c_void_p(eng.h), out.ctypes.data_as(ct.POINTER(ct.c_uint32)), n) == n
    return out


def _halves(w):
    return np.stack([(w & 0xFFFF).astype(np.uint16).view(np.int16), (w >> 16).astype(np.uint16).view(np.int16)], axis=-1)


def _fold(col, ref_len):
    """the column words of one pair-task folded per block of 64 columns: (blocks, 2 halves)"""
    h = _halves(col[:ref_len]).astype(np.int32)
    n_blk = (ref_len + 63) // 64
    pad = np.full((n_blk * 64 - ref_len, 2), -(1 << 20), dtype=np.int32)
    return np.concatenate([h, pad]).reshape(n_blk, 64, 2).max(axis=1)


def _workload(rng, ref_len, lengths, n_reads):
    """a reference cut from a longer sequence, and reads copied with edits from around it (hits on both sides of its ends)"""
    src = rng.integers(0, 4, size=4000).astype(np.int8)
    a = 1500
    ref = src[a: a + ref_len].copy()
    reads = []
    for i in range(n_reads):
        L = lengths[i % len(lengths)]
        start = int(rng.integers(a - L + 16, a + ref_len - 16))
        reads.append(C.mutate_read(rng, src, start, L, 0.08, 0.01, 0.01))
    return ref, reads


def _check(eng, n_reads):
    rng = np.random.default_rng(4242)
    mat = C.dna_matrix(2, 2)
    eng.set_option("latency_cols", 0)
    try:
        for inst, lengths in INSTANCES.items():
            eng.set_option("inst", inst)
            for ref_len in REF_LENS:
                ref, reads = _workload(rng, ref_len, lengths, n_reads)
                eng.set_sequences(reads, [ref])
                for chunk in CHUNKS:
                    # column mode right before every block-mode call: a block word the fill did not write would hold a
                    # column word there, not the block maximum
                    eng.set_option("cm_block", 0)
                    eng.set_option("chunk", 0)
                    eng.align(mat, 5, GAP_O, GAP_E, flag=0, mask_len=15, score_size=1)
                    col = _colmax(eng)
                    eng.set_option("cm_block", 1)
                    eng.set_option("chunk", chunk)
                    eng.align(mat, 5, GAP_O, GAP_E, flag=0, mask_len=15, score_size=1)
                    blk = _colmax(eng)
                    per_col, per_blk = (ref_len + 3) // 4 * 4, (ref_len // 64 + 4) // 4 * 4
                    assert len(col) % per_col == 0 and len(blk) % per_blk == 0
                    n_pt = len(col) // per_col
                    assert n_pt == len(blk) // per_blk and n_pt >= 2
                    for p in range(n_pt):
                        want = _fold(col[p * per_col: (p + 1) * per_col], ref_len)
                        got = _halves(blk[p * per_blk: p * per_blk + len(want)]).astype(np.int32)
                        bad = np.nonzero((got != want).any(axis=1))[0]
                        assert bad.size == 0, (inst, ref_len, chunk, p, bad[:4], got[bad[:4]], want[bad[:4]])
                    assert _fold(col[:per_col], ref_len).max() > 0
    finally:
        for name in ("inst", "cm_block", "chunk", "latency_cols"):
            eng.set_option(name, -1)


def test_emulated_block_words():
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    L = _pkg()
    eng = L.BatchAligner(lib_dir=EMU_DIR, lib_name="libssw_emu.so")
    try:
        _check(eng, 6)
    finally:
        eng.close()


@pytest.mark.gpu
def test_gpu_block_words():
    L = _pkg()
    eng = L.BatchAligner(device=0)
    try:
        _check(eng, 150)
    finally:
        eng.close()
