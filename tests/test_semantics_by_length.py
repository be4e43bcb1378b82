"""Byte semantics on the word rows, and the byte / word hand-over, at every read length class (DESIGN 2, 4.2).

A byte alignment of a read with length % 16 in 1..7 is filled on its word rows in block mode; a fourth re-fill item per
alignment re-does the columns [e2, e2 + 8) right of the mask window on the byte rows, on another kernel instance where
the byte padding needs more rows than the fill instance has (33..39 bp: (8,5) -> (8,8); 145..151 bp: (8,19) -> (8,20)).
When such a byte score overflows, the word result is resolved again from the same fill.  These checks run that machinery
at every kernel instance a byte alignment can land on, next to the controls that must not take it (length % 16 = 8,
equal paddings, the strip kernel), and put the scores exactly on the byte limit on every route that decides between the
two semantics.  Every constructed case asserts its own premise (instance rows, zone hit, exact score, launch count)
from the checker's records or the numpy restatement of the recurrence, so that a construction that drifts fails."""
import subprocess

import numpy as np
import pytest

import common as C
from test_byte_on_word_rows import EMU_DIR, _adversarial_reads, _pkg, fill_rows, lp_of, second_best, spill_identity_holds
from test_fill_instances import INST_ROWS

MASK = 15
GAP_O, GAP_E = 3, 1
NUL = 4                  # the letter N: scores 0 against everything with dna_matrix(n_score=0)
DNA = C.dna_matrix(2, 2)
FORWARD = [i for i in range(len(INST_ROWS)) if not 10 <= i <= 13]     # instances of the automatic forward choice
G32 = [10, 11, 12, 13]                                                  # 32-lane instances (latency path)

# read length (length % 16 in 1..7) -> (rows of the instance its byte alignment is filled on, rows of the zone re-fill)
BYTE_ON_WORD = {
    1: (32, 32), 7: (32, 32), 17: (32, 32), 23: (32, 32),
    33: (40, 64), 37: (40, 64), 39: (40, 64),
    49: (64, 64), 55: (64, 64), 65: (80, 80), 71: (80, 80),
    100: (128, 128), 101: (128, 128),
    129: (152, 152), 135: (152, 152), 145: (152, 160), 151: (152, 160),
    161: (256, 256), 247: (256, 256),
    257: (304, 304), 263: (304, 304), 289: (304, 304), 295: (304, 304),
    305: (320, 320), 311: (320, 320),
    497: (512, 512), 503: (512, 512), 513: (640, 640), 519: (640, 640), 625: (640, 640), 631: (640, 640),
}
# controls -> rows of their byte fill: length % 16 = 8 stays on its byte rows, 0 / 9..15 has equal paddings, 641 runs on
# the strip kernel (3 strips of 32 x 10 rows)
CONTROLS = {8: 32, 24: 32, 40: 64, 152: 160, 632: 640, 144: 152, 633: 640, 640: 640, 641: 960}
# one length per fill instance: the lengths run at chunks 64 and 128, and under every forced instance
PER_INST = [7, 37, 55, 71, 101, 135, 151, 247, 263, 311, 503, 631]


def fewest_rows(lp, insts=FORWARD):
    return min((INST_ROWS[i] for i in insts if INST_ROWS[i] >= lp), default=None)


def _checker(reads, refs, pq, pr, mat, n, score_size):
    return C.cpu_batch(reads, refs, pq, pr, mat, n, GAP_O, GAP_E, flag=0, mask_len=MASK, score_size=score_size, threads=4)[:2]


def _align(eng, mat, n, score_size, exp, exp_pool, pq=None, pr=None, what=""):
    res, pool = eng.align(mat, n, GAP_O, GAP_E, flag=0, mask_len=MASK, score_size=score_size, pair_query=pq, pair_ref=pr)
    bad = C.compare_records(res, pool, exp, exp_pool)
    assert bad == [], (what, bad[:8], [(res[i], exp[i]) for i in bad[:2]])
    return eng.timing()


# ---------------------------------------------------------------------------------------------------------------------
# A. the spill identity on the numpy restatement, at every length class
# ---------------------------------------------------------------------------------------------------------------------

SPILL_SETTINGS = [(C.dna_matrix(m, x), 5, go, ge, 4) for m, x, go, ge in
                  [(2, 2, 3, 1), (1, 3, 5, 2), (3, 6, 8, 1), (2, 1, 2, 1), (1, 1, 6, 2)]] + [(C.BLOSUM50, 24, 3, 1, 20)]


def _spill_inputs(length, seed):
    """(read, ref, mat, n, gapO, gapE): the adversarial reads of test_byte_on_word_rows (copies, partial copies, an
    insertion at the end, a repeat, a mutated copy, a random read) against 400 columns, for every scoring setting.  A read
    longer than fits is a random head followed by such a read of 300 letters (the last rows decide the spill); one shorter
    than 8 letters is the end of such a read of 8."""
    rng = np.random.default_rng(seed)
    for mat, n, go, ge, alpha in SPILL_SETTINGS:
        ref = rng.integers(0, alpha, size=400).astype(np.int8)
        ref[200:260] = np.tile(ref[100:112], 5)
        core = min(max(length, 8), 300)
        reads = list(_adversarial_reads(rng, ref, core)) + [rng.integers(0, alpha, size=core).astype(np.int8)]
        for read in reads:
            read = np.concatenate([rng.integers(0, alpha, size=max(length - core, 0)), read]).astype(np.int8)
            yield read[-length:], ref, mat, n, go, ge


@pytest.mark.parametrize("length", sorted(BYTE_ON_WORD))
def test_spill_identity_by_length(length):
    for read, ref, mat, n, go, ge in _spill_inputs(length, 3000 + length):
        assert len(read) == length
        assert spill_identity_holds(read, ref, mat, n, go, ge), (length, go, ge, n)


def test_spill_identity_needs_all_eight_columns():
    """The comparison can fail: with seven spill columns instead of eight it does on these inputs."""
    fails = 0
    for length in (37, 101, 150):
        for read, ref, mat, n, go, ge in _spill_inputs(length, 3000 + length):
            fails += not spill_identity_holds(read, ref, mat, n, go, ge, spill_cols=7)
    assert fails > 0


# ---------------------------------------------------------------------------------------------------------------------
# the instance table
# ---------------------------------------------------------------------------------------------------------------------

def check_instance_rows(eng):
    """One byte alignment per length, one chunk: cells_forward / (2 x reference length) is the rows of the instance that
    filled it.  Pins BYTE_ON_WORD and CONTROLS, so that the checks below cannot drift onto other instances."""
    for L, (rows, zone) in BYTE_ON_WORD.items():
        assert L % 16 in range(1, 8) and rows == fewest_rows(lp_of(L, 1)), L
        assert zone == (rows if lp_of(L, 0) <= rows else fewest_rows(lp_of(L, 0))), L
    for L, rows in CONTROLS.items():
        assert (L % 16 not in range(1, 8) or L > 640) and rows == (fewest_rows(lp_of(L, 0)) or -(-lp_of(L, 0) // 320) * 320), L
    rng = np.random.default_rng(21)
    ref = rng.integers(0, 4, size=256).astype(np.int8)
    eng.set_option("latency_cols", 0)
    eng.set_option("cm_block", 1)
    for L, rows in list((L, r[0]) for L, r in BYTE_ON_WORD.items()) + list(CONTROLS.items()):
        read = rng.integers(0, 4, size=L).astype(np.int8)
        eng.set_sequences([read], [ref])
        exp, exp_pool = _checker([read], [ref], [0], [0], DNA, 5, 0)
        t = _align(eng, DNA, 5, 0, exp, exp_pool, what=L)
        assert t["fill_forward_launches"] == 1 and t["cells_forward"] == 2 * len(ref) * rows, (L, t["cells_forward"] // 512)


# ---------------------------------------------------------------------------------------------------------------------
# B. zone cases at every length class
# ---------------------------------------------------------------------------------------------------------------------

# e2 = end_ref + MASK + 1 of the planted reads on a 1,024-column reference: on a block boundary, at offsets 57 and 63 of
# a block, and 3 columns before the reference end
ZONE_REF = 1024
ZONE_E2 = (5 * 64, 8 * 64 + 57, 12 * 64 + 63, ZONE_REF - 3)


def _plant(rng, ref, L, e2, alpha=4, tail_max=100, head=NUL):
    """A read of length L whose best cell is its last row at column p = e2 - MASK - 1: a head of `head` letters (random
    ones when head is None) and a random tail of at most tail_max letters copied into ref[.. p].  Behind p the pad rows
    decay by a horizontal gap, one per column, so column e2 sees a higher value on the byte rows (their diagonal reaches
    8 columns further) than on the word rows.  A 1 bp read cannot decay that far: a second copy at p + 1 reaches e2."""
    p = e2 - MASK - 1
    t = min(L, tail_max)
    tail = rng.integers(0, alpha, size=t).astype(np.int8)
    ref[p - t + 1: p + 1] = tail
    if L == 1:
        ref[p + 1] = tail[0]
    h = rng.integers(0, alpha, size=L - t) if head is None else np.full(L - t, head)
    return np.concatenate([h, tail]).astype(np.int8)


def assert_zone(read, ref, rec, mat, n):
    """The checker's record is a byte result whose second best lies in [e2, e2 + 8) and differs from a scan of the
    word-row column maxima (numpy restatement); returns e2."""
    L = len(read)
    H = fill_rows(read, ref, mat, n, GAP_O, GAP_E, lp_of(L, 0))
    cb, cw = H.max(axis=0), H[: lp_of(L, 1)].max(axis=0)
    end_ref = int(rec["ref_end1"])
    assert int(rec["score1"]) == int(cb.max()) < 250 and end_ref == int(np.argmax(cb)), (L, rec)
    byte2 = second_best(cb, end_ref, MASK, False)
    assert byte2 == (int(rec["score2"]), int(rec["ref_end2"])), (L, byte2, rec)
    e2 = min(end_ref + MASK, len(ref)) + 1
    assert e2 <= byte2[1] < e2 + 8 and second_best(cw, end_ref, MASK, False) != byte2, (L, e2, byte2)
    return e2


def _zone_batch(rng):
    """(reads, refs, pair_ref): four zone reads per length of BYTE_ON_WORD, one reference per length (one per read below
    33 bp, whose short tails would find each other), and every control planted the same way."""
    reads, refs, pr, zone = [], [], [], []
    for L in sorted(BYTE_ON_WORD) + sorted(CONTROLS):
        ref = None
        for e2 in ZONE_E2:
            if ref is None or L < 33:
                ref = np.full(ZONE_REF, NUL, dtype=np.int8)
                refs.append(ref)
            reads.append(_plant(rng, ref, L, e2))
            pr.append(len(refs) - 1)
            zone.append(L in BYTE_ON_WORD)
    return reads, refs, np.array(pr), zone


def check_zone_by_length(eng):
    rng = np.random.default_rng(31)
    reads, refs, pr, zone = _zone_batch(rng)
    pq = np.arange(len(reads))
    eng.set_sequences(reads, refs)
    exp, exp_pool = _checker(reads, refs, pq, pr, DNA, 5, 2)
    for i in np.flatnonzero(zone):
        assert assert_zone(reads[i], refs[pr[i]], exp[i], DNA, 5) == ZONE_E2[i % 4]
    assert sum(zone) == 4 * len(BYTE_ON_WORD) and [e2 % 64 for e2 in ZONE_E2[:3]] == [0, 57, 63]
    eng.set_option("latency_cols", 0)
    eng.set_option("cm_block", 1)
    eng.set_option("chunk", 0)
    t = _align(eng, DNA, 5, 2, exp, exp_pool, pq, pr, "chunk 0")
    assert t["byte_overflows"] == 0
    # chunks 64 and 128: one read of one length per fill instance (at 64 up to 320 rows: the warm-up makes it the costly one)
    for chunk, slot, longest in ((64, 1, 320), (128, 2, 640)):
        sub = np.array([i for i in range(len(reads)) if i % 4 == slot and len(reads[i]) in PER_INST
                        and BYTE_ON_WORD[len(reads[i])][0] <= longest])
        eng.set_option("chunk", chunk)
        _align(eng, DNA, 5, 2, exp[sub], exp_pool, pq[sub], pr[sub], "chunk %d" % chunk)
    eng.set_option("chunk", 0)


def check_zone_protein(eng):
    """BLOSUM50 (bias 5, byte limit 250), score_size 2, 100 aa and 290 aa queries (length % 16 = 4 and 2): predicted word
    first, their byte result is filled again on the word rows with a 24-letter profile.  The heads are X (22), which
    scores -1 against every letter: with 3/1 gaps random proteins align with scores that grow with their length."""
    rng = np.random.default_rng(32)
    ref = rng.integers(0, 20, size=2 * ZONE_REF).astype(np.int8)
    reads = [_plant(rng, ref, L, e2 + k * 896, alpha=20, tail_max=16, head=22) for k, L in enumerate((100, 290)) for e2 in ZONE_E2[:3]]
    n = len(reads)
    pq, pr = np.arange(n), np.zeros(n, dtype=np.int64)
    eng.set_sequences(reads, [ref])
    exp, exp_pool = _checker(reads, [ref], pq, pr, C.BLOSUM50, 24, 2)
    for i in range(n):
        assert len(reads[i]) * 15 >= 2 * 250                      # word first
        assert_zone(reads[i], ref, exp[i], C.BLOSUM50, 24)
    eng.set_option("latency_cols", 0)
    eng.set_option("cm_block", 1)
    eng.set_option("chunk", 0)
    _align(eng, C.BLOSUM50, 24, 2, exp, exp_pool, what="protein")


# ---------------------------------------------------------------------------------------------------------------------
# C. pair-tasks with one half of each kind
# ---------------------------------------------------------------------------------------------------------------------

def check_mixed_pairs(eng):
    """129..152 bp (140 bp twice) against one reference.  129..151 run on (8,19): 129..135 and 145..151 with byte_pad 8,
    136..144 without.  The pair-tasks pair neighbours in (fill rows, query) order, so 7 padded + 10 unpadded + 7 padded
    reads give two pair-tasks with one half of each kind; 152 bp needs 160 rows, so every block re-fill of the launch runs
    on (8,20).  33 and 39 bp (both padded, (8,5), zone re-fill on (8,8)) form one pair-task.  Every read is planted so
    that its second best is decided next to the window: a zone hit for the padded ones, a block cut by the window (e2 at
    block offset 57 or 63) or a block boundary for the others."""
    rng = np.random.default_rng(41)
    lengths = [33, 39] + list(range(129, 141)) + list(range(140, 153))
    ref = np.full(192 * (len(lengths) + 1) + 64, NUL, dtype=np.int8)
    reads, e2s = [], []
    for k, L in enumerate(lengths):
        e2 = 192 * (k + 1) + (0, 57, 63)[k % 3]
        reads.append(_plant(rng, ref, L, e2))
        e2s.append(e2)
    n = len(reads)
    pq, pr = np.arange(n), np.zeros(n, dtype=np.int64)
    exp, exp_pool = _checker(reads, [ref], pq, pr, DNA, 5, 2)
    padded = [L % 16 in range(1, 8) for L in lengths]
    for i in range(n):
        if padded[i]:
            assert assert_zone(reads[i], ref, exp[i], DNA, 5) == e2s[i]
        else:
            assert int(exp[i]["ref_end1"]) + MASK + 1 == e2s[i] and int(exp[i]["score2"]) > 0
    # the pairing of the (8,19) launch, restated: queries in (fill rows, id) order, neighbours paired
    inst15 = sorted((i for i in range(n) if 129 <= lengths[i] <= 151), key=lambda i: (lp_of(lengths[i], 1 if padded[i] else 0), i))
    pairs = [(inst15[j], inst15[j + 1]) for j in range(0, len(inst15) - 1, 2)]
    mixed = [(a, b) for a, b in pairs if padded[a] != padded[b]]
    assert len(mixed) == 2 and all(BYTE_ON_WORD.get(lengths[i], (152,))[0] == 152 for i in inst15), mixed
    eng.set_sequences(reads, [ref])
    eng.set_option("latency_cols", 0)
    eng.set_option("cm_block", 1)
    eng.set_option("chunk", 0)
    t = _align(eng, DNA, 5, 2, exp, exp_pool, what="mixed")
    assert t["fill_forward_launches"] == 3 and t["byte_overflows"] == 0     # (8,5), (8,19), (8,20)


# ---------------------------------------------------------------------------------------------------------------------
# D. scores exactly on the byte limit
# ---------------------------------------------------------------------------------------------------------------------

# scoring setting -> (matrix, byte limit, {score: core}) where a core (kind, m) scores exactly `score` against its copy:
# "exact" m matches, "mismatch" m matches around one mismatch, "insert" m matches around one extra read letter (gapO)
THRESHOLDS = {
    "2/2": (C.dna_matrix(2, 2), 253, {252: ("exact", 126), 253: ("insert", 128), 254: ("exact", 127)}),
    "5/4": (C.dna_matrix(5, 4), 251, {250: ("exact", 50), 251: ("mismatch", 51), 252: ("insert", 51)}),
}
# route -> setting -> (length % 16 in 1..7, = 8, equal paddings)
BYTE_FIRST_LENGTHS = {"2/2": (150, 152, 144), "5/4": (100, 88, 96)}
# word first: the longest byte-first length, the prediction length, and longer ones of the other classes
WORD_FIRST_LENGTHS = {"2/2": (252, 253, 257, 264), "5/4": (100, 101, 104, 112)}


def _threshold_batch(rng, setting, L):
    """Three reads of length L (a head of N, which scores 0, then the core) scoring limit - 1, limit and limit + 1, planted
    in one random reference.  Returns (reads, ref, mat, limit)."""
    mat, limit, cores = THRESHOLDS[setting]
    ref = rng.integers(0, 4, size=640).astype(np.int8)
    reads = []
    for k, score in enumerate((limit - 1, limit, limit + 1)):
        kind, m = cores[score]
        end = 180 * (k + 1)
        seg = ref[end - m + 1: end + 1].copy() if kind != "mismatch" else ref[end - m: end + 1].copy()
        half = len(seg) // 2
        if kind == "mismatch":
            seg[half] = (seg[half] + 1) % 4
        elif kind == "insert":
            x = next(b for b in range(4) if b != seg[half - 1] and b != seg[half])
            seg = np.concatenate([seg[:half], [x], seg[half:]])
        assert len(seg) <= L
        reads.append(np.concatenate([np.full(L - len(seg), NUL), seg]).astype(np.int8))
    return reads, ref, mat, limit


def _check_scores(reads, ref, exp, mat, limit, score_size):
    """The checker's scores are exactly limit - 1, limit, limit + 1 (score_size 0: the last two are NULL records).  With
    both profiles the overflowing records carry word semantics, and their word second best lies exactly at
    end_ref + MASK, a column the byte scan may not take."""
    if score_size == 0:
        assert [int(r["status"]) for r in exp] == [0, 1, 1] and int(exp[0]["score1"]) == limit - 1
        return
    assert [int(r["score1"]) for r in exp] == [limit - 1, limit, limit + 1]
    for i in (1, 2):
        L = len(reads[i])
        H = fill_rows(reads[i], ref, mat, 5, GAP_O, GAP_E, lp_of(L, 1))
        cw = H.max(axis=0)
        end_ref = int(exp[i]["ref_end1"])
        assert end_ref == int(np.argmax(cw)) and int(cw.max()) == limit + i - 1
        word2 = second_best(cw, end_ref, MASK, True)
        assert word2 == (int(exp[i]["score2"]), int(exp[i]["ref_end2"])) and word2[1] == end_ref + MASK
        assert second_best(cw, end_ref, MASK, False) != word2


def _threshold_call(eng, reads, ref, mat, limit, score_size, what):
    n = len(reads)
    eng.set_sequences(reads, [ref])
    exp, exp_pool = _checker(reads, [ref], np.arange(n), np.zeros(n, dtype=np.int64), mat, 5, score_size)
    _check_scores(reads, ref, exp, mat, limit, score_size)
    t = _align(eng, mat, 5, score_size, exp, exp_pool, what=what)
    if score_size == 2:
        assert t["byte_overflows"] == sum(int(r["score1"]) >= limit for r in exp) == 2, (what, t)
    return t


def check_thresholds(eng):
    rng = np.random.default_rng(51)
    for setting, lengths in BYTE_FIRST_LENGTHS.items():
        for cls, L in zip(("1..7", "8", "equal"), lengths):
            reads, ref, mat, limit = _threshold_batch(rng, setting, L)
            max_mat = int(mat.max())
            assert L * max_mat < 2 * limit and (L % 16 in range(1, 8)) == (cls == "1..7") and (L % 16 == 8) == (cls == "8")
            rows = fewest_rows(lp_of(L, 0 if cls == "8" else 1))
            # byte first, block mode: an overflow is re-resolved on the same fill except for length % 16 = 8
            eng.set_option("latency_cols", 0)
            eng.set_option("cm_block", 1)
            eng.set_option("grid_min", -1)
            for score_size in (0, 1, 2):
                t = _threshold_call(eng, reads, ref, mat, limit, score_size, ("byte first", setting, L, score_size))
                if score_size == 2:
                    assert t["fill_forward_launches"] == (2 if cls == "8" else 1), (setting, L, t)
                    if cls != "8":
                        assert t["cells_forward"] == 2 * len(ref) * rows * 2, (setting, L, t)
            # the latency path: byte and word semantics of each read in the two halves of its own pair-task, one launch
            eng.set_option("latency_cols", -1)
            eng.set_option("cm_block", -1)
            t = _threshold_call(eng, reads, ref, mat, limit, 2, ("latency", setting, L))
            g32 = fewest_rows(lp_of(L, 0), G32)
            assert t["fill_forward_launches"] == 1 and t["cells_forward"] == len(reads) * len(ref) * g32 * 2, (setting, L, t)
            # the device-planned grid: byte semantics on the byte rows, overflows re-done on the general path
            eng.set_option("latency_cols", 0)
            eng.set_option("cm_block", 1)
            eng.set_option("grid_min", 1)
            for score_size in (0, 2):
                t = _threshold_call(eng, reads, ref, mat, limit, score_size, ("grid", setting, L, score_size))
                assert t["fill_forward_launches"] >= 2, t
                assert t["cells_forward"] >= 2 * len(ref) * fewest_rows(lp_of(L, 0)) * 2, t     # the grid's own launch
            eng.set_option("grid_min", -1)
    # word first: predicted where length x max(mat) >= 2 x limit
    eng.set_option("latency_cols", 0)
    eng.set_option("cm_block", 1)
    for setting, lengths in WORD_FIRST_LENGTHS.items():
        for k, L in enumerate(lengths):
            reads, ref, mat, limit = _threshold_batch(rng, setting, L)
            assert (L * int(mat.max()) >= 2 * limit) == (k > 0)
            for score_size in (0, 2):
                _threshold_call(eng, reads, ref, mat, limit, score_size, ("word first", setting, L, score_size))
    eng.set_option("latency_cols", -1)
    eng.set_option("cm_block", -1)


# ---------------------------------------------------------------------------------------------------------------------
# E. forced instances
# ---------------------------------------------------------------------------------------------------------------------

def check_forced_instances(eng):
    """One length per fill instance under every instance ("inst") whose rows cover its fill rows, 10..13 included: two
    zone reads (half A and half B of one pair-task) and, from 129 bp on, an exact copy whose byte score overflows.  The
    zone re-fill moves to another instance for 37 bp on (8,5) and 151 bp on (8,19)."""
    rng = np.random.default_rng(61)
    eng.set_option("latency_cols", 0)
    eng.set_option("cm_block", 1)
    try:
        for L in PER_INST:
            fill, zone = BYTE_ON_WORD[L]
            ref_len = 384 + max(L, 128) + 64
            refs = [np.full(ref_len, NUL, dtype=np.int8) for _ in range(1 if L >= 33 else 2)]     # short tails find each other
            reads = [_plant(rng, refs[k % len(refs)], L, e2) for k, e2 in enumerate((3 * 64, 5 * 64 + 57))]
            pr = [0, len(refs) - 1]
            if L >= 129:
                refs[0][384: 384 + L] = rng.integers(0, 4, size=L)
                reads.append(refs[0][384: 384 + L].copy())
                pr.append(0)
            n = len(reads)
            pq, pr = np.arange(n), np.array(pr)
            eng.set_sequences(reads, refs)
            exp, exp_pool = _checker(reads, refs, pq, pr, DNA, 5, 2)
            for i in range(2):
                assert_zone(reads[i], refs[pr[i]], exp[i], DNA, 5)
            assert n == 2 or int(exp[2]["score1"]) >= 253
            insts = [i for i, rows in enumerate(INST_ROWS) if rows >= fill]
            assert (L not in (37, 151)) or any(INST_ROWS[i] < zone for i in insts)
            for inst in insts:
                eng.set_option("inst", inst)
                t = _align(eng, DNA, 5, 2, exp, exp_pool, pq, pr, ("inst", inst, L))
                assert t["cells_forward"] % (2 * ref_len * INST_ROWS[inst]) == 0, (inst, L, t)
                assert t["byte_overflows"] == n - 2
    finally:
        eng.set_option("inst", -1)


# ---------------------------------------------------------------------------------------------------------------------
# F. the multi-launch block path (GPU: the budget's unit is 1 MiB)
# ---------------------------------------------------------------------------------------------------------------------

def check_budget_launches(eng):
    """145..151 bp reads against 300 kbp with "cm_budget_mb" 1 (262,144 block words per launch, 55 pair-tasks of 4,692
    words): 240 reads = 120 pair-tasks need 3 launches of (8,19), and their byte overflows the word re-fill after them."""
    rng = np.random.default_rng(71)
    ref_len = 300_000
    ref = rng.integers(0, 4, size=ref_len).astype(np.int8)
    reads = []
    for k in range(240):
        L = 145 + k % 7
        at = 1000 + k * 1200
        if k % 4 == 0:
            reads.append(ref[at: at + L].copy())                                  # overflows
        elif k % 4 == 1:
            e2 = at + 64 * 4 + (0, 57, 63)[k % 3] - at % 64
            reads.append(_plant(rng, ref, L, e2, head=None))                      # zone
        else:
            reads.append(C.mutate_read(rng, ref, at, L, 0.15, 0.02, 0.02))
    n = len(reads)
    eng.set_sequences(reads, [ref])
    exp, exp_pool = _checker(reads, [ref], np.arange(n), np.zeros(n, dtype=np.int64), DNA, 5, 2)
    n_over = sum(int(r["score1"]) >= 253 for r in exp)
    assert n_over >= 60
    words = (ref_len // 64 + 1 + 3) // 4 * 4
    assert (n // 2 + (262144 // words) - 1) // (262144 // words) >= 3
    eng.set_option("latency_cols", 0)
    eng.set_option("cm_block", 1)
    eng.set_option("cm_budget_mb", 1)
    try:
        t = _align(eng, DNA, 5, 2, exp, exp_pool, what="budget")
        assert t["fill_forward_launches"] >= 4 and t["byte_overflows"] == n_over, t
    finally:
        eng.set_option("cm_budget_mb", -1)


def _run_all(eng, gpu=False):
    check_instance_rows(eng)
    check_zone_by_length(eng)
    check_zone_protein(eng)
    check_mixed_pairs(eng)
    check_thresholds(eng)
    check_forced_instances(eng)
    if gpu:
        check_budget_launches(eng)


def test_emulated_semantics_by_length():
    subprocess.run(["make", "-s", "-C", EMU_DIR], check=True)
    L = _pkg()
    eng = L.BatchAligner(lib_dir=EMU_DIR, lib_name="libssw_emu.so")
    try:
        _run_all(eng)
    finally:
        eng.close()


@pytest.mark.gpu
def test_gpu_semantics_by_length():
    L = _pkg()
    eng = L.BatchAligner(device=0)
    try:
        _run_all(eng, gpu=True)
    finally:
        eng.close()
