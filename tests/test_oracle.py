"""CPU tests that PIN the oracle (oracle/ssw_oracle.c):

 * against the golden fixtures frozen from the unmodified reference
   (tests/golden/goldens.json -- includes the reference's shipped regression
   golden demo/old.txt, the README sample and the example.c known answer);
 * against the answers of the unmodified reference (compiled into
   oracle/_ref/libssw_ref.so) to randomised inputs in every parameter regime,
   frozen in tests/golden/oracle_random_ref.json.gz;
 * formulation 2 (Gotoh + ordered bookkeeping, the GPU spec) against
   formulation 1 (literal striped emulation) in the regime gapO > gapE.
"""
import gzip
import json
import os

import numpy as np
import pytest

import common as C


@pytest.fixture(scope="module")
def oracle():
    return C.load_oracle()


@pytest.fixture(scope="module")
def goldens():
    with open(os.path.join(C.GOLDEN, "goldens.json")) as f:
        return json.load(f)


def golden_inputs(case):
    enc = C.encode_dna if case["alphabet"] == "dna" else C.encode_aa
    mat = {"dna_2_2": C.dna_matrix(2, 2), "dna_cpp_2_2": C.dna_matrix_cpp(2, 2), "blosum50": C.BLOSUM50}[case["matrix"]]
    if "refs_npz" in case:
        refs = [np.load(os.path.join(C.GOLDEN, case["refs_npz"]))["ref"]]
    else:
        refs = [enc(r) for r in case["refs"]]
    reads = [enc(q) for q in case["reads"]]
    return mat, refs, reads


def run_golden(lib, case, max_reads=None):
    """Replay one golden case (the CLI's read x reference double loop) and return the mismatches."""
    mat, refs, reads = golden_inputs(case)
    bad = []
    k = 0
    for qi, q in enumerate(reads):
        for r in refs:
            exp = case["expected"][k]
            k += 1
            if max_reads is not None and qi >= max_reads:
                continue
            ml = len(q) // 2 if case["maskLen"] is None else case["maskLen"]
            got = lib.align(q, r, mat, case["n"], case["gapO"], case["gapE"], case["flag"], case["filters"],
                            case["filterd"], ml, case["score_size"], mark="nm" in exp)
            d = C.diff_results(got, exp)
            for extra in ("nm", "cigar_marked"):
                if extra in exp and got.get(extra) != exp[extra]:
                    d.append((extra, got.get(extra), exp[extra]))
            if d:
                bad.append((case["name"], qi, d))
    return bad


def test_oracle_matches_goldens(oracle, goldens, capfd):
    for case in goldens:
        limit = 4 if "refs_npz" in case else None      # 1 Mbp reference: a few reads are enough for the scalar oracle
        assert run_golden(oracle, case, limit) == []


def random_case(rng):
    prot = rng.random() < 0.3
    n = 24 if prot else 5
    mat = C.BLOSUM50.copy() if prot else C.dna_matrix(int(rng.integers(1, 6)), int(rng.integers(1, 6)))
    if rng.random() < 0.2:                               # arbitrary asymmetric matrix
        mat = rng.integers(-6, 7, size=n * n).astype(np.int8)
        for i in range(n):
            mat[i * n + i] = rng.integers(1, 9)
    alpha = 20 if prot else (5 if rng.random() < 0.3 else 4)
    qlen = int(rng.integers(1, 200))
    rlen = int(rng.integers(1, 600))
    ref = rng.integers(0, alpha, size=rlen).astype(np.int8)
    if rng.random() < 0.7 and rlen > qlen + 5:
        read = C.mutate_read(rng, ref, int(rng.integers(0, rlen - qlen)), qlen, 0.1, 0.03, 0.03, alpha)
    else:
        read = rng.integers(0, alpha, size=qlen).astype(np.int8)
    u = rng.random()
    if u < 0.6:
        gapE = int(rng.integers(1, 4)); gapO = gapE + int(rng.integers(1, 8))
    elif u < 0.8:
        gapE = int(rng.integers(0, 5)); gapO = gapE
    else:
        gapO = int(rng.integers(0, 6)); gapE = int(rng.integers(0, 6))
    return dict(read=read, ref=ref, mat=mat, n=n, gapO=gapO, gapE=gapE,
                flag=int(rng.choice([0, 1, 2, 4, 8, 0x0f, 3, 5, 9])),
                filters=int(rng.integers(0, 60)), filterd=int(rng.integers(0, 300)),
                maskLen=int(rng.choice([5, 15, 20, qlen // 2 + 15])), score_size=int(rng.integers(0, 3)))


RANDOM_SEED, RANDOM_CASES = 20260924, 2500


def test_oracle_matches_reference_random(oracle, capfd):
    """The reference's answers to these cases are frozen in golden/oracle_random_ref.json.gz (golden/make_reference_golden.py)."""
    with gzip.open(os.path.join(C.GOLDEN, "oracle_random_ref.json.gz"), "rt") as f:
        expected = json.load(f)
    assert len(expected) == RANDOM_CASES
    rng = np.random.default_rng(RANDOM_SEED)
    bad = []
    for k in range(RANDOM_CASES):
        c = random_case(rng)
        a = oracle.align(mark=True, **c)
        b = expected[k]
        d = C.diff_results(a, b)
        if a and b and (a.get("nm"), a.get("cigar_marked")) != (b.get("nm"), b.get("cigar_marked")):
            d.append(("marked", a.get("cigar_marked"), b.get("cigar_marked")))
        if d:
            bad.append((k, d))
    assert bad == []


def test_gotoh_formulation_equals_striped(oracle, capfd):
    """The GPU-shaped restatement (pass A + pass B, pad rows included) is exact for gapO > gapE."""
    rng = np.random.default_rng(77)
    bad = []
    n_checked = 0
    for k in range(4000):
        c = random_case(rng)
        if c["gapO"] <= c["gapE"]:
            continue
        n_checked += 1
        oracle.lib.oracle_set_formulation(0)
        a = oracle.align(**c)
        oracle.lib.oracle_set_formulation(1)
        b = oracle.align(**c)
        oracle.lib.oracle_set_formulation(0)
        d = C.diff_results(a, b)
        if d:
            bad.append((k, d))
    assert n_checked > 1500 and bad == []
