"""The forward fill's kernel instances, as the public ABI sees them.

The engine keeps one table of (lanes per group G, rows per lane R) instances; the "inst" option indexes it, and
cells_forward / (2 x reference length) of a one-chunk, one-alignment call is the G x R rows of the instance that ran.
These tests pin the table order, the automatic choice (the instance with the fewest rows that covers the padded read),
the launch shape of a CTA-shared-profile launch (8 warps, 16 items per CTA for 300 aa queries), and the option
names of include/ssw_batch.h -- on the CPU emulator build and on the GPU."""
import ctypes as ct
import os
import re
import subprocess

import numpy as np
import pytest

import common as C
from test_byte_on_word_rows import EMU_DIR, _pkg

# G * R of inst 0..15
INST_ROWS = [32, 40, 64, 80, 128, 160, 256, 320, 512, 640, 128, 160, 256, 320, 304, 152]

# read length -> rows of the automatic choice: word / byte semantics in batch layouts, word on the latency path
AUTO_LENGTHS = [20, 33, 40, 64, 70, 128, 150, 160, 250, 300, 320, 500, 640]
AUTO_ROWS = {
    "word": [32, 40, 40, 64, 80, 128, 152, 160, 256, 304, 320, 512, 640],
    "byte": [32, 64, 64, 64, 80, 128, 160, 160, 256, 304, 320, 512, 640],
    "latency": [128, 128, 128, 128, 128, 128, 160, 160, 256, 320, 320, 512, 640],
}


def _rows(eng, ref_len):
    cells = eng.timing()["cells_forward"]
    assert cells % (2 * ref_len) == 0, cells
    return cells // (2 * ref_len)


def _align_checked(eng, reads, refs, mat, n, score_size, mask_len=15):
    nq, nr = len(reads), len(refs)
    res, pool = eng.align(mat, n, 3, 1, flag=0, mask_len=mask_len, score_size=score_size)
    exp, exp_pool, _, _, _ = C.cpu_batch(reads, refs, np.repeat(np.arange(nq), nr), np.tile(np.arange(nr), nq), mat, n,
                                        3, 1, flag=0, mask_len=mask_len, score_size=score_size, threads=4)
    bad = C.compare_records(res, pool, exp, exp_pool)
    assert bad == [], (bad, [(res[i], exp[i]) for i in bad[:2]])


def check_inst_table(eng):
    """"inst" = i runs instance i: every index launches, in the table's order."""
    rng = np.random.default_rng(11)
    ref = rng.integers(0, 4, size=300).astype(np.int8)
    read = np.concatenate([ref[100:112], rng.integers(0, 4, size=8)]).astype(np.int8)
    eng.set_sequences([read], [ref])
    eng.set_option("latency_cols", 0)
    mat = C.dna_matrix(2, 2)
    try:
        for i, rows in enumerate(INST_ROWS):
            eng.set_option("inst", i)
            _align_checked(eng, [read], [ref], mat, 5, 1)
            assert _rows(eng, len(ref)) == rows, (i, _rows(eng, len(ref)))
    finally:
        eng.set_option("inst", -1)


def check_auto_choice(eng):
    """One read per length: the rows the engine picks on its own, and records equal to the checker's."""
    rng = np.random.default_rng(12)
    ref = rng.integers(0, 4, size=800).astype(np.int8)
    mat = C.dna_matrix(2, 2)
    for mode, want in AUTO_ROWS.items():
        eng.set_option("latency_cols", 1 << 20 if mode == "latency" else 0)
        score_size = 0 if mode == "byte" else 1
        got = []
        for L in AUTO_LENGTHS:
            # random read with a planted 40-letter piece of the reference: a real alignment that stays below the byte limit
            read = rng.integers(0, 4, size=L).astype(np.int8)
            at, src = int(rng.integers(0, L - 39)) if L > 40 else 0, int(rng.integers(0, len(ref) - 40))
            k = min(40, L)
            read[at: at + k] = ref[src: src + k]
            eng.set_sequences([read], [ref])
            _align_checked(eng, [read], [ref], mat, 5, score_size)
            got.append(_rows(eng, len(ref)))
        assert got == want, (mode, got)
    eng.set_option("latency_cols", -1)


def check_shared_profile(eng):
    """4 x 300 aa queries against 72 x 400 aa targets: 2 query pairs x 72 = 144 pair-tasks on (16,19), 304 rows.  The launch
    uses 8-warp CTAs with a CTA-shared profile, 16 items per CTA: each query pair's run of 72 items is padded to 80 (11 %,
    so the profile stays shared).  72 is a multiple of 8 but not of 16, so a planner that padded the runs to another CTA
    size (8 items, the 4-warp shape) would put the items of both query pairs into one CTA, which builds one profile for
    both, and the records would be wrong."""
    rng = np.random.default_rng(13)
    targets = [rng.integers(0, 20, size=400).astype(np.int8) for _ in range(72)]
    queries = [C.mutate_read(rng, targets[3 * i], 50, 300, 0.3, 0.02, 0.02, alphabet=20) for i in range(4)]
    assert all(len(q) == 300 for q in queries)
    eng.set_sequences(queries, targets)
    eng.set_option("latency_cols", 0)
    _align_checked(eng, queries, targets, C.BLOSUM50, 24, 1)
    assert eng.timing()["cells_forward"] == 144 * 400 * 304 * 2
    eng.set_option("latency_cols", -1)


def option_names():
    """The option names documented in include/ssw_batch.h (the comment above ssw_engine_set_option)."""
    with open(os.path.join(C.ROOT, "include", "ssw_batch.h")) as f:
        text = f.read()
    block = text[text.index("Tuning knobs"): text.index("int ssw_engine_set_option")]
    return re.findall(r'"(\w+)"', block)


def check_option_names(eng):
    names = option_names()
    assert len(names) == 17 and len(set(names)) == 17, names
    set_opt = eng.lib.ssw_engine_set_option
    for name in names:
        assert set_opt(ct.c_void_p(eng.h), name.encode(), -1) == 0, name
        assert set_opt(None, name.encode(), -1) == 0, name          # -1 restores every option's default
    for handle in (ct.c_void_p(eng.h), None):
        assert set_opt(handle, b"no_such_option", 1) == -1


def _run_all(eng):
    check_inst_table(eng)
    check_auto_choice(eng)
    check_shared_profile(eng)
    check_option_names(eng)


def test_emulated_fill_instances():
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    L = _pkg()
    eng = L.BatchAligner(lib_dir=EMU_DIR, lib_name="libssw_emu.so")
    try:
        _run_all(eng)
    finally:
        eng.close()


@pytest.mark.gpu
def test_gpu_fill_instances():
    L = _pkg()
    eng = L.BatchAligner(device=0)
    try:
        _run_all(eng)
    finally:
        eng.close()
