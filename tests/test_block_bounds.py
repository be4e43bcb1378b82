"""Bounded block words (fill kernel CM == 3, "cm_block" 2 and the automatic mode): the fill stores per 64 columns the largest
row maximum of E sampled once per loop body, w(b), and the resolve re-fills only the blocks whose bracket
w(b) + gapE <= M(b) <= w(b) + gapO + 7 gapE cannot rule them out (DESIGN 2).

- The bracket is checked directly on every stored block against the column-mode words of the same call folded per 64
  columns, for the instances (8,19), (16,19) and (32,16), several reference lengths and chunk lengths.  The lower bound of a
  loop body that straddles two blocks belongs to the later block, so it is checked against max(M(b), M(b + 1)).
- Records of bounded words, exact block maxima ("cm_block" 1) and the checker must be identical on decoy-heavy batches
  (many candidates), references of repeated segments (several blocks tie at score1 and score2), mask windows whose edges
  fall on block boundaries, byte alignments filled on their word rows (the byte-row zone), byte overflows re-resolved from
  the same fill, and alignments with more candidates than the cap of 256 blocks (a read of null letters scores 0
  everywhere, so every block of a 17,000-column reference is a candidate), which go to the exact path."""
import subprocess

import numpy as np
import pytest

import common as C
from test_block_words import INSTANCES, REF_LENS, CHUNKS, _colmax, _fold, _halves, _workload
from test_byte_on_word_rows import EMU_DIR, _pkg

GAP_O, GAP_E = 3, 1


def _check_bounds(eng, n_reads):
    rng = np.random.default_rng(777)
    mat = C.dna_matrix(2, 2)
    eng.set_option("latency_cols", 0)
    try:
        for inst, lengths in INSTANCES.items():
            eng.set_option("inst", inst)
            for ref_len in REF_LENS:
                ref, reads = _workload(rng, ref_len, lengths, n_reads)
                eng.set_sequences(reads, [ref])
                for chunk in CHUNKS:
                    eng.set_option("cm_block", 0)
                    eng.set_option("chunk", 0)
                    eng.align(mat, 5, GAP_O, GAP_E, flag=0, mask_len=15, score_size=1)
                    col = _colmax(eng)
                    eng.set_option("cm_block", 2)
                    eng.set_option("chunk", chunk)
                    eng.align(mat, 5, GAP_O, GAP_E, flag=0, mask_len=15, score_size=1)
                    blk = _colmax(eng)
                    per_col, per_blk = (ref_len + 3) // 4 * 4, (ref_len // 64 + 4) // 4 * 4
                    n_pt = len(col) // per_col
                    assert n_pt == len(blk) // per_blk and n_pt >= 2
                    for p in range(n_pt):
                        m = _fold(col[p * per_col: (p + 1) * per_col], ref_len)
                        w = _halves(blk[p * per_blk: p * per_blk + len(m)]).astype(np.int32)
                        m_next = np.concatenate([m[1:], m[-1:]])
                        upper_bad = np.nonzero((m > w + GAP_O + 7 * GAP_E).any(axis=1))[0]
                        lower_bad = np.nonzero((w + GAP_E > np.maximum(m, m_next)).any(axis=1))[0]
                        assert upper_bad.size == 0 and lower_bad.size == 0, (inst, ref_len, chunk, p, upper_bad[:4], lower_bad[:4])
    finally:
        for name in ("inst", "cm_block", "chunk", "latency_cols"):
            eng.set_option(name, -1)


def _repeat_ref(rng):
    """a reference of a 700-column segment repeated 5 times with a few edits, random in between"""
    seg = rng.integers(0, 4, size=700).astype(np.int8)
    parts = []
    for i in range(5):
        s = seg.copy()
        if i % 2:
            s[rng.integers(0, 700, size=3)] = rng.integers(0, 4, size=3)
        parts += [s, rng.integers(0, 4, size=64 * (i + 1) + 13).astype(np.int8)]
    return np.concatenate(parts), seg


def _cases(rng):
    """(name, ref, reads, mask lengths)"""
    out = []
    # decoys: random reads score about the same everywhere, so many blocks are candidates
    ref = rng.integers(0, 4, size=6000).astype(np.int8)
    reads = [rng.integers(0, 4, size=L).astype(np.int8) for L in (150, 149, 146, 150, 120, 100, 151, 150)]
    reads += [C.mutate_read(rng, ref, int(rng.integers(0, 5800)), 150, 0.15, 0.01, 0.01) for _ in range(4)]
    out.append(("decoys", ref, reads, (15, 75)))
    # repeated segments: several blocks tie at score1 and at score2
    ref, seg = _repeat_ref(rng)
    reads = [seg[a: a + 150].copy() for a in (0, 64, 200, 550)]
    reads += [C.mutate_read(rng, seg, 300, 150, 0.1, 0.01, 0.01), seg[100: 247].copy()]
    out.append(("repeats", ref, reads, (15, 64, 75)))
    # window edges on block boundaries: an exact copy ending at column 64 k - 1 with mask lengths that put e1 / e2 on a block
    # boundary (word and byte semantics differ by one column at e2)
    ref = rng.integers(0, 4, size=4000).astype(np.int8)
    reads = [ref[64 * 20 - 150: 64 * 20].copy(), ref[64 * 40 - 150 + 1: 64 * 40 + 1].copy(),
             C.mutate_read(rng, ref, 64 * 30 - 149, 150, 0.05, 0.0, 0.0)]
    out.append(("edges", ref, reads, (63, 64, 128, 129)))
    # byte overflows (exact copies score 2 L >= 290 with bias 2) next to reads that stay in a byte
    ref = rng.integers(0, 4, size=3000).astype(np.int8)
    reads = []
    for i, L in enumerate(range(145, 152)):
        start = 100 + 380 * i
        reads.append(ref[start: start + L].copy())
        reads.append(C.mutate_read(rng, ref, start + 150, L, 0.2, 0.02, 0.02))
    out.append(("overflows", ref, reads, (15,)))
    # over the cap: 266 candidate blocks for the reads of null letters (code 4 scores 0 against everything)
    ref = rng.integers(0, 4, size=17000).astype(np.int8)
    reads = [np.full(150, 4, dtype=np.int8), C.mutate_read(rng, ref, 9000, 150, 0.15, 0.01, 0.01), np.full(120, 4, dtype=np.int8)]
    out.append(("cap", ref, reads, (15,)))
    return out


def _check_records(eng, chunks):
    rng = np.random.default_rng(31337)
    mat = C.dna_matrix(2, 2)
    eng.set_option("latency_cols", 0)
    try:
        for name, ref, reads, masks in _cases(rng):
            n = len(reads)
            eng.set_sequences(reads, [ref])
            for mask in masks:
                for score_size in (0, 2):
                    exp, exp_pool, _, _, _ = C.cpu_batch(reads, [ref], np.arange(n), np.zeros(n), mat, 5, GAP_O, GAP_E, flag=0,
                                                        mask_len=mask, score_size=score_size, threads=4)
                    for chunk in chunks:
                        eng.set_option("chunk", chunk)
                        for cm_block in (1, 2):
                            eng.set_option("cm_block", cm_block)
                            res, pool = eng.align(mat, 5, GAP_O, GAP_E, flag=0, mask_len=mask, score_size=score_size)
                            bad = C.compare_records(res, pool, exp, exp_pool)
                            assert bad == [], (name, mask, score_size, chunk, cm_block, bad, [(res[i], exp[i]) for i in bad[:2]])
                            t = eng.timing()
                            if cm_block == 1:
                                assert t["block_refills"] == 0 and t["block_exact"] == 0, t
                            elif name == "cap":
                                assert t["block_exact"] == 2, t
                            else:
                                assert t["block_exact"] == 0 and t["block_refills"] >= n // 2, (name, t)
    finally:
        for opt in ("cm_block", "chunk", "latency_cols"):
            eng.set_option(opt, -1)


def _emu():
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    return _pkg().BatchAligner(lib_dir=EMU_DIR, lib_name="libssw_emu.so")


def test_emulated_block_bounds():
    eng = _emu()
    try:
        _check_bounds(eng, 6)
    finally:
        eng.close()


def test_emulated_bounded_records():
    eng = _emu()
    try:
        _check_records(eng, (320,))
    finally:
        eng.close()


@pytest.mark.gpu
def test_gpu_block_bounds():
    eng = _pkg().BatchAligner(device=0)
    try:
        _check_bounds(eng, 150)
    finally:
        eng.close()


@pytest.mark.gpu
def test_gpu_bounded_records():
    eng = _pkg().BatchAligner(device=0)
    try:
        _check_records(eng, (0, 64, 320))
    finally:
        eng.close()
