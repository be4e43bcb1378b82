"""Host-side Python mirror of the reference's ctypes wrapper (src/ssw_lib.py) on top of
the H100-native libssw.so, plus the batched interface of include/ssw_batch.h.

 * ``CSsw`` keeps the reference class's surface (ssw_lib.py:94-197): attributes
   ``ssw_init``, ``init_destroy``, ``ssw_align``, ``align_destroy`` bound with the same
   argument types, and ``CAlignRes`` / ``CProfile`` structures with the same field names,
   so code written against the reference wrapper (e.g. pyssw.py) runs unchanged.
 * ``BatchAligner`` drives ssw_engine_* : many (query, reference) pairs per call.

Nothing here computes alignments; without the CUDA library the import fails loudly.
"""
import ctypes as ct
import os
import os.path as op

import numpy as np

_HERE = op.dirname(op.abspath(__file__))
LIB_NAME = "libssw.so"


class CAlignRes(ct.Structure):
    """s_align (ssw.h:55-66) with the reference wrapper's field names (ssw_lib.py:61-69) plus `nFlag`."""
    _fields_ = [("nScore", ct.c_uint16), ("nScore2", ct.c_uint16),
                ("nRefBeg", ct.c_int32), ("nRefEnd", ct.c_int32),
                ("nQryBeg", ct.c_int32), ("nQryEnd", ct.c_int32),
                ("nRefEnd2", ct.c_int32), ("sCigar", ct.POINTER(ct.c_uint32)),
                ("nCigarLen", ct.c_int32), ("nFlag", ct.c_uint16)]


class CProfile(ct.Structure):
    """Opaque to callers; declared only so that pointer types match the reference wrapper (ssw_lib.py:84-90)."""
    _fields_ = [("pRead", ct.POINTER(ct.c_int8)), ("pMat", ct.POINTER(ct.c_int8)),
                ("nReadLen", ct.c_int32), ("nN", ct.c_int32), ("nScoreSize", ct.c_int8)]


class BatchParams(ct.Structure):
    """ssw_batch_params (include/ssw_batch.h)."""
    _fields_ = [("mat", ct.POINTER(ct.c_int8)), ("n", ct.c_int32),
                ("gap_open", ct.c_uint8), ("gap_extend", ct.c_uint8), ("flag", ct.c_uint8),
                ("filters", ct.c_uint16), ("filterd", ct.c_int32), ("mask_len", ct.c_int32),
                ("score_size", ct.c_int8)]


class EngineTiming(ct.Structure):
    """ssw_engine_timing (include/ssw_batch.h)."""
    _fields_ = [("fill_forward_ms", ct.c_float), ("resolve_ms", ct.c_float), ("fill_reverse_ms", ct.c_float),
                ("traceback_ms", ct.c_float), ("total_ms", ct.c_float),
                ("fill_forward_launches", ct.c_int64), ("other_launches", ct.c_int64),
                ("cells_forward", ct.c_int64), ("byte_overflows", ct.c_int64),
                ("grid_cols_planned", ct.c_int64), ("grid_cols_useful", ct.c_int64), ("leftover_pairs", ct.c_int64),
                ("block_refills", ct.c_int64), ("block_exact", ct.c_int64)]


# numpy view of ssw_batch_result (36 bytes)
RESULT_DTYPE = np.dtype([("score1", "<u2"), ("score2", "<u2"), ("ref_begin1", "<i4"), ("ref_end1", "<i4"),
                         ("read_begin1", "<i4"), ("read_end1", "<i4"), ("ref_end2", "<i4"),
                         ("cigar_off", "<i4"), ("cigar_len", "<i4"), ("flag", "<u2"), ("status", "<u2")])
assert RESULT_DTYPE.itemsize == 36


class HitView(ct.Structure):
    """ssw_hit_view (include/ssw_batch.h)."""
    _fields_ = [("n_rows", ct.c_int32), ("n_hits", ct.c_int64), ("row_off", ct.c_void_p), ("hit_ref", ct.c_void_p),
                ("hits", ct.c_void_p), ("cigar_pool", ct.c_void_p), ("pool_used", ct.c_int64)]


# default bound of search_all: 2^26 hits, 2.7 GB of records and reference indices
SEARCH_ALL_MAX_HITS = 1 << 26


def _copy_out(ptr, n, dtype):
    """n items of dtype at a C pointer, as an owned numpy array (copied as bytes: a copy of the structured record dtype goes
    field by field, several times slower)"""
    dtype = np.dtype(dtype)
    if n <= 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    return np.frombuffer((ct.c_char * (n * dtype.itemsize)).from_address(ptr), dtype=np.uint8).copy().view(dtype)


def _take_hit_set(lib, rv, handle, name, max_hits):
    """(row_off int64, hit_ref int32, hits RESULT_DTYPE, cigar_pool uint32) copied out of an ssw_hit_set, which is destroyed"""
    if rv == -2:
        raise RuntimeError("%s: more than max_hits = %d hits (raise max_hits or min_score)" % (name, max_hits))
    if rv or not handle.value:
        raise RuntimeError("%s failed (%d)" % (name, rv))
    lib.ssw_hit_set_view.argtypes = [ct.c_void_p, ct.POINTER(HitView)]
    lib.ssw_hit_set_view.restype = ct.c_int
    lib.ssw_hit_set_destroy.argtypes = [ct.c_void_p]
    lib.ssw_hit_set_destroy.restype = None
    try:
        v = HitView()
        if lib.ssw_hit_set_view(handle, ct.byref(v)):
            raise RuntimeError("ssw_hit_set_view failed")
        return (_copy_out(v.row_off, v.n_rows + 1, np.int64), _copy_out(v.hit_ref, v.n_hits, np.int32),
                _copy_out(v.hits, v.n_hits, RESULT_DTYPE), _copy_out(v.cigar_pool, v.pool_used, np.uint32))
    finally:
        lib.ssw_hit_set_destroy(handle)


def _load(lib_dir=None, lib_name=LIB_NAME):
    path = op.join(lib_dir or _HERE, lib_name)
    if not op.exists(path):
        raise ImportError("%s not built: run `python __graft_entry__.py` (there is no CPU fallback)" % path)
    return ct.CDLL(path)


class CSsw(object):
    """Same surface as the reference's CSsw (ssw_lib.py:94-197)."""

    def __init__(self, sLibPath=None):
        self.ssw = _load(sLibPath)
        self.ssw_init = self.ssw.ssw_init
        self.ssw_init.argtypes = [ct.POINTER(ct.c_int8), ct.c_int32, ct.POINTER(ct.c_int8), ct.c_int32, ct.c_int8]
        self.ssw_init.restype = ct.POINTER(CProfile)
        self.init_destroy = self.ssw.init_destroy
        self.init_destroy.argtypes = [ct.POINTER(CProfile)]
        self.init_destroy.restype = None
        self.ssw_align = self.ssw.ssw_align
        self.ssw_align.argtypes = [ct.c_void_p, ct.POINTER(ct.c_int8), ct.c_int32, ct.c_uint8, ct.c_uint8,
                                   ct.c_uint8, ct.c_uint16, ct.c_int32, ct.c_int32]
        self.ssw_align.restype = ct.POINTER(CAlignRes)
        self.align_destroy = self.ssw.align_destroy
        self.align_destroy.argtypes = [ct.POINTER(CAlignRes)]
        self.align_destroy.restype = None


def _i8(a):
    a = np.ascontiguousarray(a, dtype=np.int8)
    return a, a.ctypes.data_as(ct.POINTER(ct.c_int8))


def _mat(mat):
    """(array kept alive, pointer) of a scoring matrix; None -> NULL (query profiles resident)."""
    return (None, None) if mat is None else _i8(mat)


def concat(seqs):
    """List of int8 code arrays -> (concatenation, int64 offsets[n+1])."""
    off = np.zeros(len(seqs) + 1, dtype=np.int64)
    if len(seqs):
        off[1:] = np.cumsum([len(s) for s in seqs])
    cat = np.concatenate([np.asarray(s, dtype=np.int8) for s in seqs]) if len(seqs) else np.zeros(0, np.int8)
    return np.ascontiguousarray(cat, dtype=np.int8), off


class BatchAligner(object):
    """ssw_engine_* of include/ssw_batch.h: resident sequences + batched ssw_align."""

    def __init__(self, device=-1, lib_dir=None, lib_name=LIB_NAME):
        self.lib = _load(lib_dir, lib_name)
        L = self.lib
        L.ssw_engine_create.argtypes = [ct.c_int]
        L.ssw_engine_create.restype = ct.c_void_p
        L.ssw_engine_destroy.argtypes = [ct.c_void_p]
        L.ssw_engine_destroy.restype = None
        L.ssw_engine_device_name.argtypes = [ct.c_void_p]
        L.ssw_engine_device_name.restype = ct.c_char_p
        L.ssw_engine_set_sequences.argtypes = [ct.c_void_p, ct.c_int32, ct.POINTER(ct.c_int8), ct.POINTER(ct.c_int64),
                                               ct.c_int32, ct.POINTER(ct.c_int8), ct.POINTER(ct.c_int64)]
        L.ssw_engine_set_sequences.restype = ct.c_int
        L.ssw_engine_align.argtypes = [ct.c_void_p, ct.POINTER(BatchParams), ct.c_int64, ct.POINTER(ct.c_int32),
                                       ct.POINTER(ct.c_int32), ct.c_void_p, ct.POINTER(ct.c_uint32), ct.c_int64,
                                       ct.POINTER(ct.c_int64)]
        L.ssw_engine_align.restype = ct.c_int
        L.ssw_engine_last_timing.argtypes = [ct.c_void_p, ct.POINTER(EngineTiming)]
        L.ssw_engine_last_timing.restype = ct.c_int
        L.ssw_engine_set_option.argtypes = [ct.c_void_p, ct.c_char_p, ct.c_int64]
        L.ssw_engine_set_option.restype = ct.c_int
        self.h = L.ssw_engine_create(device)
        if not self.h:
            raise RuntimeError("ssw_engine_create failed: no usable CUDA device (this library has no CPU path)")
        self.n_q = self.n_r = 0
        self._keep = None
        self._lens = None

    def close(self):
        if self.h:
            self.lib.ssw_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def device_name(self):
        return self.lib.ssw_engine_device_name(self.h).decode()

    def set_option(self, name, value):
        if self.lib.ssw_engine_set_option(self.h, name.encode(), int(value)):
            raise ValueError(name)

    def set_sequences(self, queries, refs):
        """Host -> device copy of the query and reference sets (lists of int8 code arrays)."""
        qc, qo = concat(queries)
        rc, ro = concat(refs)
        rv = self.lib.ssw_engine_set_sequences(self.h, len(queries), qc.ctypes.data_as(ct.POINTER(ct.c_int8)),
                                               qo.ctypes.data_as(ct.POINTER(ct.c_int64)), len(refs),
                                               rc.ctypes.data_as(ct.POINTER(ct.c_int8)),
                                               ro.ctypes.data_as(ct.POINTER(ct.c_int64)))
        if rv:
            raise RuntimeError("ssw_engine_set_sequences failed (%d)" % rv)
        self.n_q, self.n_r = len(queries), len(refs)
        self._lens = (np.diff(qo), np.diff(ro))

    def set_sequences_self(self, seqs):
        """One set (list of int8 code arrays) resident as both the queries and the references (ssw_engine_set_sequences_self):
        align / search / search_all then give what they give after set_sequences(seqs, seqs), and search_self runs."""
        c, o = concat(seqs)
        f = self.lib.ssw_engine_set_sequences_self
        f.argtypes = [ct.c_void_p, ct.c_int32, ct.POINTER(ct.c_int8), ct.POINTER(ct.c_int64)]
        f.restype = ct.c_int
        rv = f(self.h, len(seqs), c.ctypes.data_as(ct.POINTER(ct.c_int8)), o.ctypes.data_as(ct.POINTER(ct.c_int64)))
        if rv:
            raise RuntimeError("ssw_engine_set_sequences_self failed (%d)" % rv)
        self.n_q = self.n_r = len(seqs)
        self._lens = (np.diff(o), np.diff(o))

    def set_profiles(self, profiles, refs, n):
        """Host -> device copy of query profiles (PSSMs) and references (ssw_engine_set_sequences_pssm): `profiles` is a list of
        (L_q, n) int8 arrays, row i = the scores of query position i against the n reference letters; `refs` int8 code arrays.
        Later align / search / search_all calls take mat=None and this n."""
        rows = [np.asarray(p, dtype=np.int8).reshape(-1, n) if n > 0 else np.asarray(p, dtype=np.int8) for p in profiles]
        qo = np.zeros(len(rows) + 1, dtype=np.int64)
        if rows:
            qo[1:] = np.cumsum([len(p) for p in rows])
        qc = np.ascontiguousarray(np.concatenate([p.reshape(-1) for p in rows]) if rows else np.zeros(0, np.int8))
        rc, ro = concat(refs)
        f = self.lib.ssw_engine_set_sequences_pssm
        f.argtypes = [ct.c_void_p, ct.c_int32, ct.POINTER(ct.c_int8), ct.POINTER(ct.c_int64), ct.c_int32,
                      ct.c_int32, ct.POINTER(ct.c_int8), ct.POINTER(ct.c_int64)]
        f.restype = ct.c_int
        rv = f(self.h, len(rows), qc.ctypes.data_as(ct.POINTER(ct.c_int8)), qo.ctypes.data_as(ct.POINTER(ct.c_int64)), int(n),
               len(refs), rc.ctypes.data_as(ct.POINTER(ct.c_int8)), ro.ctypes.data_as(ct.POINTER(ct.c_int64)))
        if rv:
            raise RuntimeError("ssw_engine_set_sequences_pssm failed (%d)" % rv)
        self.n_q, self.n_r = len(rows), len(refs)
        self._lens = (np.diff(qo), np.diff(ro))

    def set_sequences_text(self, queries, refs, table, n, add_reverse_complement=False):
        """Sequences as text (bytes / str): translated to codes with `table` (128 int8 entries) on the device; with
        add_reverse_complement the reverse complement of query k becomes query len(queries) + k."""
        qs = [q.encode() if isinstance(q, str) else bytes(q) for q in queries]
        rs = [r.encode() if isinstance(r, str) else bytes(r) for r in refs]
        qt, rt = b"".join(qs), b"".join(rs)
        qo = np.zeros(len(qs) + 1, dtype=np.int64); qo[1:] = np.cumsum([len(q) for q in qs])
        ro = np.zeros(len(rs) + 1, dtype=np.int64); ro[1:] = np.cumsum([len(r) for r in rs])
        tab = np.ascontiguousarray(table, dtype=np.int8)
        assert tab.size == 128
        f = self.lib.ssw_engine_set_sequences_text
        f.argtypes = [ct.c_void_p, ct.c_int32, ct.c_char_p, ct.POINTER(ct.c_int64), ct.c_int32, ct.c_char_p, ct.POINTER(ct.c_int64),
                      ct.POINTER(ct.c_int8), ct.c_int32, ct.c_int32]
        f.restype = ct.c_int
        rv = f(self.h, len(qs), qt, qo.ctypes.data_as(ct.POINTER(ct.c_int64)), len(rs), rt, ro.ctypes.data_as(ct.POINTER(ct.c_int64)),
               tab.ctypes.data_as(ct.POINTER(ct.c_int8)), int(n), 1 if add_reverse_complement else 0)
        if rv:
            raise RuntimeError("ssw_engine_set_sequences_text failed (%d)" % rv)
        ql = np.diff(qo)
        if add_reverse_complement:
            ql = np.concatenate([ql, ql])
        self.n_q, self.n_r = len(ql), len(rs)
        self._lens = (ql, np.diff(ro))

    def set_sequences_packed(self, queries, refs, bits, n):
        """References delivered as a packed bit stream (bits = 2 or 4 per base, low bits first; unpacked on the device by
        ssw_engine_set_sequences_packed); queries as plain codes.  `n` = alphabet size of the later align() calls."""
        qc, qo = concat(queries)
        rc, ro = concat(refs)
        assert bits in (2, 4) and (rc.size == 0 or int(rc.max()) < (1 << bits))
        per = 8 // bits
        padded = np.zeros((len(rc) + per - 1) // per * per, dtype=np.uint8)
        padded[: len(rc)] = rc.astype(np.uint8)
        packed = np.zeros(len(padded) // per, dtype=np.uint8)
        for k in range(per):
            packed |= (padded[k::per] << (bits * k)).astype(np.uint8)
        f = self.lib.ssw_engine_set_sequences_packed
        f.argtypes = [ct.c_void_p, ct.c_int32, ct.POINTER(ct.c_int8), ct.POINTER(ct.c_int64), ct.c_int32, ct.POINTER(ct.c_uint8),
                      ct.POINTER(ct.c_int64), ct.c_int32, ct.c_int32]
        f.restype = ct.c_int
        rv = f(self.h, len(queries), qc.ctypes.data_as(ct.POINTER(ct.c_int8)), qo.ctypes.data_as(ct.POINTER(ct.c_int64)), len(refs),
               packed.ctypes.data_as(ct.POINTER(ct.c_uint8)), ro.ctypes.data_as(ct.POINTER(ct.c_int64)), int(bits), int(n))
        if rv:
            raise RuntimeError("ssw_engine_set_sequences_packed failed (%d)" % rv)
        self.n_q, self.n_r = len(queries), len(refs)
        self._lens = (np.diff(qo), np.diff(ro))
        return len(packed)

    def align(self, mat, n, gap_open=3, gap_extend=1, flag=0, filters=0, filterd=0, mask_len=-1, score_size=2,
              pair_query=None, pair_ref=None, want_cigar=None, out=None):
        """Align pairs of the resident sequences; returns (results[RESULT_DTYPE], cigar_pool[uint32]).  mat=None with query
        profiles resident (set_profiles).
        out: a results array of a previous call with the same number of pairs to write into (large grids return
        hundreds of MB of records; re-using the buffer avoids mapping and unmapping it on every call)."""
        mat, matp = _mat(mat)
        P = BatchParams(matp, n, gap_open, gap_extend, flag, filters, filterd, mask_len, score_size)
        if pair_query is None:
            n_pairs = self.n_q * self.n_r
            pq = pr = None
        else:
            pq_a = np.ascontiguousarray(pair_query, dtype=np.int32)
            pr_a = np.ascontiguousarray(pair_ref, dtype=np.int32)
            n_pairs = len(pq_a)
            pq = pq_a.ctypes.data_as(ct.POINTER(ct.c_int32))
            pr = pr_a.ctypes.data_as(ct.POINTER(ct.c_int32))
        if out is not None and out.dtype == RESULT_DTYPE and len(out) == n_pairs and out.flags["C_CONTIGUOUS"]:
            res = out
        else:
            res = np.empty(n_pairs, dtype=RESULT_DTYPE)     # every record is written by the library
        if want_cigar is None:
            want_cigar = bool(flag & 7)
        cap = 0
        if want_cigar:
            ql, rl = self._lens
            QL = np.repeat(ql, len(rl)) if pair_query is None else ql[pq_a]
            RL = np.tile(rl, len(ql)) if pair_query is None else rl[pr_a]
            cap = int(np.sum(QL + np.minimum(RL, QL * 128) + 4))
        pool = np.empty(max(cap, 1), dtype=np.uint32)        # worst-case sized, only pool[:used] is meaningful
        used = ct.c_int64(0)
        rv = self.lib.ssw_engine_align(self.h, ct.byref(P), n_pairs, pq, pr, res.ctypes.data_as(ct.c_void_p),
                                       pool.ctypes.data_as(ct.POINTER(ct.c_uint32)), len(pool), ct.byref(used))
        if rv:
            raise RuntimeError("ssw_engine_align failed (%d)" % rv)
        return res, pool[: used.value]

    def search(self, mat, n, k, min_score=0, gap_open=3, gap_extend=1, flag=0, filters=0, filterd=0, mask_len=-1, score_size=2):
        """Top-k search of every resident query against all resident references (ssw_engine_search).  Returns
        (hit_ref[n_q, k] int32, hits[n_q, k] RESULT_DTYPE, n_hits[n_q] int32, cigar_pool[uint32]): row q holds query q's
        n_hits[q] best hits in rank order (status-1 pairs, then score1 descending, then reference ascending); unused slots
        have hit_ref -1.  mat=None with query profiles resident."""
        f = self.lib.ssw_engine_search
        f.argtypes = [ct.c_void_p, ct.POINTER(BatchParams), ct.c_int32, ct.c_int32, ct.POINTER(ct.c_int32), ct.c_void_p,
                      ct.POINTER(ct.c_int32), ct.POINTER(ct.c_uint32), ct.c_int64, ct.POINTER(ct.c_int64)]
        f.restype = ct.c_int
        mat, matp = _mat(mat)
        P = BatchParams(matp, n, gap_open, gap_extend, flag, filters, filterd, mask_len, score_size)
        rows = max(int(k), 0)
        hit_ref = np.empty((self.n_q, rows), dtype=np.int32)
        hits = np.empty((self.n_q, rows), dtype=RESULT_DTYPE)
        n_hits = np.empty(self.n_q, dtype=np.int32)
        cap = 0
        if (flag & 7) and self._lens is not None and len(self._lens[1]):
            ql, rl = self._lens
            cap = int(rows * np.sum(ql + np.minimum(int(rl.max()), ql * 128) + 4))
        pool = np.empty(max(cap, 1), dtype=np.uint32)
        used = ct.c_int64(0)
        rv = f(self.h, ct.byref(P), int(k), int(min_score), hit_ref.ctypes.data_as(ct.POINTER(ct.c_int32)), hits.ctypes.data_as(ct.c_void_p),
               n_hits.ctypes.data_as(ct.POINTER(ct.c_int32)), pool.ctypes.data_as(ct.POINTER(ct.c_uint32)), len(pool), ct.byref(used))
        if rv:
            raise RuntimeError("ssw_engine_search failed (%d)" % rv)
        return hit_ref, hits, n_hits, pool[: used.value]

    def search_all(self, mat, n, min_score, max_hits=SEARCH_ALL_MAX_HITS, gap_open=3, gap_extend=1, flag=0, filters=0, filterd=0,
                   mask_len=-1, score_size=2):
        """Threshold search of every resident query against all resident references (ssw_engine_search_all): every hit
        (status 1 or score1 >= max(min_score, 1)).  Returns (row_off[n_q + 1] int64, hit_ref int32, hits RESULT_DTYPE,
        cigar_pool uint32) in CSR form: row q is [row_off[q], row_off[q + 1]), in ascending reference index.  More hits
        than max_hits raise RuntimeError.  mat=None with query profiles resident."""
        f = self.lib.ssw_engine_search_all
        f.argtypes = [ct.c_void_p, ct.POINTER(BatchParams), ct.c_int32, ct.c_int64, ct.POINTER(ct.c_void_p)]
        f.restype = ct.c_int
        mat, matp = _mat(mat)
        P = BatchParams(matp, n, gap_open, gap_extend, flag, filters, filterd, mask_len, score_size)
        handle = ct.c_void_p()
        rv = f(self.h, ct.byref(P), int(min_score), int(max_hits), ct.byref(handle))
        return _take_hit_set(self.lib, rv, handle, "ssw_engine_search_all", max_hits)

    def search_self(self, mat, n, min_score, max_hits=SEARCH_ALL_MAX_HITS, gap_open=3, gap_extend=1, flag=0, filters=0, filterd=0,
                    mask_len=-1, score_size=2):
        """Self-search of the set made resident by set_sequences_self (ssw_engine_search_self): every unordered pair {i, j},
        i != j, once, as the record of query = the earlier in canonical order (length, then index) against the other, kept by
        the rule of search_all.  Returns (row_off[n + 1], hit_ref, hits, cigar_pool) as search_all: row i holds the hits in
        which i is the query, in ascending partner index.  Needs a symmetric matrix and gap_open > gap_extend."""
        f = self.lib.ssw_engine_search_self
        f.argtypes = [ct.c_void_p, ct.POINTER(BatchParams), ct.c_int32, ct.c_int64, ct.POINTER(ct.c_void_p)]
        f.restype = ct.c_int
        mat, matp = _mat(mat)
        P = BatchParams(matp, n, gap_open, gap_extend, flag, filters, filterd, mask_len, score_size)
        handle = ct.c_void_p()
        rv = f(self.h, ct.byref(P), int(min_score), int(max_hits), ct.byref(handle))
        return _take_hit_set(self.lib, rv, handle, "ssw_engine_search_self", max_hits)

    def mark_mismatch(self, res, pool, pair_query=None, pair_ref=None):
        """mark_mismatch (ssw.c:1019-1074) for every CIGAR of a batch, on the device (ssw_engine_mark_mismatch): `res` / `pool`
        as returned by align() for the same pairs.  Returns (records with cigar_off / cigar_len pointing into the new pool,
        marked pool, nm[int32])."""
        f = self.lib.ssw_engine_mark_mismatch
        f.argtypes = [ct.c_void_p, ct.c_int64, ct.POINTER(ct.c_int32), ct.POINTER(ct.c_int32), ct.c_void_p, ct.POINTER(ct.c_uint32),
                      ct.c_int64, ct.POINTER(ct.c_uint32), ct.c_int64, ct.POINTER(ct.c_int64), ct.POINTER(ct.c_int32)]
        f.restype = ct.c_int
        out = np.array(res, dtype=RESULT_DTYPE, copy=True)
        n_pairs = len(out)
        if pair_query is None:
            pq = pr = None
            q_of = np.repeat(np.arange(self.n_q), self.n_r)
        else:
            pq_a = np.ascontiguousarray(pair_query, dtype=np.int32)
            pr_a = np.ascontiguousarray(pair_ref, dtype=np.int32)
            pq = pq_a.ctypes.data_as(ct.POINTER(ct.c_int32))
            pr = pr_a.ctypes.data_as(ct.POINTER(ct.c_int32))
            q_of = pq_a
        has = out["cigar_len"] > 0
        cap = int(np.sum(self._lens[0][q_of[has]] + out["cigar_len"][has] + 2)) + 8
        pool_in = np.ascontiguousarray(pool, dtype=np.uint32)
        marked = np.empty(cap, dtype=np.uint32)
        nm = np.zeros(n_pairs, dtype=np.int32)
        used = ct.c_int64(0)
        rv = f(self.h, n_pairs, pq, pr, out.ctypes.data_as(ct.c_void_p), pool_in.ctypes.data_as(ct.POINTER(ct.c_uint32)), len(pool_in),
               marked.ctypes.data_as(ct.POINTER(ct.c_uint32)), cap, ct.byref(used), nm.ctypes.data_as(ct.POINTER(ct.c_int32)))
        if rv:
            raise RuntimeError("ssw_engine_mark_mismatch failed (%d)" % rv)
        return out, marked[: used.value], nm

    def timing(self):
        t = EngineTiming()
        self.lib.ssw_engine_last_timing(self.h, ct.byref(t))
        return {k: getattr(t, k) for k, _ in EngineTiming._fields_}


class GroupAligner(object):
    """ssw_group_* of include/ssw_batch.h: one batch over several GPUs of this process (one engine and one host thread per
    device; a full grid is cut by queries, an explicit pair list by DP cells).  Results equal BatchAligner's for the same
    pairs, whatever the number of devices."""

    def __init__(self, n_devices=0, devices=None, lib_dir=None, lib_name=LIB_NAME):
        self.lib = _load(lib_dir, lib_name)
        L = self.lib
        L.ssw_device_count.restype = ct.c_int32
        L.ssw_group_create.argtypes = [ct.c_int32, ct.POINTER(ct.c_int32)]
        L.ssw_group_create.restype = ct.c_void_p
        L.ssw_group_destroy.argtypes = [ct.c_void_p]
        L.ssw_group_destroy.restype = None
        L.ssw_group_size.argtypes = [ct.c_void_p]
        L.ssw_group_size.restype = ct.c_int32
        L.ssw_group_engine.argtypes = [ct.c_void_p, ct.c_int32]
        L.ssw_group_engine.restype = ct.c_void_p
        L.ssw_engine_set_option.argtypes = [ct.c_void_p, ct.c_char_p, ct.c_int64]
        L.ssw_engine_set_option.restype = ct.c_int
        L.ssw_engine_last_timing.argtypes = [ct.c_void_p, ct.POINTER(EngineTiming)]
        L.ssw_engine_last_timing.restype = ct.c_int
        L.ssw_group_align.argtypes = [ct.c_void_p, ct.POINTER(BatchParams), ct.POINTER(ct.c_int8), ct.c_int32,
                                      ct.c_int32, ct.c_void_p, ct.POINTER(ct.c_int64), ct.c_int32, ct.c_void_p, ct.POINTER(ct.c_int64),
                                      ct.c_int64, ct.POINTER(ct.c_int32), ct.POINTER(ct.c_int32), ct.c_void_p, ct.POINTER(ct.c_uint32),
                                      ct.c_int64, ct.POINTER(ct.c_int64), ct.c_int32, ct.POINTER(ct.c_int32)]
        L.ssw_group_align.restype = ct.c_int
        dev = None
        if devices is not None:
            dev_a = np.ascontiguousarray(devices, dtype=np.int32)
            n_devices = len(dev_a)
            dev = dev_a.ctypes.data_as(ct.POINTER(ct.c_int32))
        self.h = L.ssw_group_create(int(n_devices), dev)
        if not self.h:
            raise RuntimeError("ssw_group_create failed: no usable CUDA device (this library has no CPU path)")

    def close(self):
        if self.h:
            self.lib.ssw_group_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def size(self):
        return int(self.lib.ssw_group_size(self.h))

    def set_option(self, name, value):
        """The same option on every engine of the group."""
        for i in range(self.size):
            if self.lib.ssw_engine_set_option(self.lib.ssw_group_engine(self.h, i), name.encode(), int(value)):
                raise ValueError(name)

    def timing(self):
        """Per-device timing records of the last call."""
        out = []
        for i in range(self.size):
            t = EngineTiming()
            self.lib.ssw_engine_last_timing(self.lib.ssw_group_engine(self.h, i), ct.byref(t))
            out.append({k: getattr(t, k) for k, _ in EngineTiming._fields_})
        return out

    def align(self, queries, refs, mat, n, gap_open=3, gap_extend=1, flag=0, filters=0, filterd=0, mask_len=-1, score_size=2,
              pair_query=None, pair_ref=None, table=None, add_reverse_complement=False, marked=False, n_pairs=None):
        """Sequences (lists of int8 code arrays, or of bytes / str with `table`) -> (results[RESULT_DTYPE], cigar_pool[uint32])
        in pair order, plus nm[int32] when marked (CIGARs as mark_mismatch leaves them).  n_pairs: only the first n_pairs
        pairs of the full grid (no pair lists)."""
        mat, matp = _i8(mat)
        P = BatchParams(matp, n, gap_open, gap_extend, flag, filters, filterd, mask_len, score_size)
        if table is None:
            qc, qo = concat(queries)
            rc, ro = concat(refs)
            qptr, rptr, tabp = qc.ctypes.data_as(ct.c_void_p), rc.ctypes.data_as(ct.c_void_p), None
        else:
            qs = [q.encode() if isinstance(q, str) else bytes(q) for q in queries]
            rs = [r.encode() if isinstance(r, str) else bytes(r) for r in refs]
            qc = np.frombuffer(b"".join(qs) + b"\0", dtype=np.uint8)
            rc = np.frombuffer(b"".join(rs) + b"\0", dtype=np.uint8)
            qo = np.zeros(len(qs) + 1, dtype=np.int64); qo[1:] = np.cumsum([len(q) for q in qs])
            ro = np.zeros(len(rs) + 1, dtype=np.int64); ro[1:] = np.cumsum([len(r) for r in rs])
            tab = np.ascontiguousarray(table, dtype=np.int8)
            assert tab.size == 128
            qptr, rptr, tabp = qc.ctypes.data_as(ct.c_void_p), rc.ctypes.data_as(ct.c_void_p), tab.ctypes.data_as(ct.POINTER(ct.c_int8))
        ql, rl = np.diff(qo), np.diff(ro)
        if table is not None and add_reverse_complement:
            ql = np.concatenate([ql, ql])
        if pair_query is None:
            n_pairs = len(ql) * len(rl) if n_pairs is None else int(n_pairs)
            pq = pr = None
            QL, RL = np.repeat(ql, len(rl))[:n_pairs], np.tile(rl, len(ql))[:n_pairs]
        else:
            pq_a = np.ascontiguousarray(pair_query, dtype=np.int32)
            pr_a = np.ascontiguousarray(pair_ref, dtype=np.int32)
            n_pairs = len(pq_a)
            pq = pq_a.ctypes.data_as(ct.POINTER(ct.c_int32))
            pr = pr_a.ctypes.data_as(ct.POINTER(ct.c_int32))
            QL, RL = ql[np.clip(pq_a, 0, len(ql) - 1)], rl[np.clip(pr_a, 0, len(rl) - 1)]      # the library checks the indices
        res = np.empty(n_pairs, dtype=RESULT_DTYPE)
        cap = int(np.sum(QL + np.minimum(RL, QL * 128) + 4)) if (flag & 7) else 0
        pool = np.empty(max(cap, 1), dtype=np.uint32)
        used = ct.c_int64(0)
        nm = np.zeros(n_pairs, dtype=np.int32)
        rv = self.lib.ssw_group_align(self.h, ct.byref(P), tabp, 1 if add_reverse_complement else 0,
                                      len(queries), qptr, qo.ctypes.data_as(ct.POINTER(ct.c_int64)),
                                      len(refs), rptr, ro.ctypes.data_as(ct.POINTER(ct.c_int64)),
                                      n_pairs, pq, pr, res.ctypes.data_as(ct.c_void_p), pool.ctypes.data_as(ct.POINTER(ct.c_uint32)),
                                      len(pool), ct.byref(used), 1 if marked else 0, nm.ctypes.data_as(ct.POINTER(ct.c_int32)))
        if rv:
            raise RuntimeError("ssw_group_align failed (%d)" % rv)
        return (res, pool[: used.value], nm) if marked else (res, pool[: used.value])

    def search(self, queries, refs, mat, n, k, min_score=0, gap_open=3, gap_extend=1, flag=0, filters=0, filterd=0, mask_len=-1,
               score_size=2, table=None, add_reverse_complement=False):
        """BatchAligner.search over the devices of the group (ssw_group_search): sequences as for align().  Returns
        (hit_ref[n_q, k], hits[n_q, k] RESULT_DTYPE, n_hits[n_q], cigar_pool); with add_reverse_complement the rows of the
        reverse complements follow those of the queries."""
        f = self.lib.ssw_group_search
        f.argtypes = [ct.c_void_p, ct.POINTER(BatchParams), ct.POINTER(ct.c_int8), ct.c_int32,
                      ct.c_int32, ct.c_void_p, ct.POINTER(ct.c_int64), ct.c_int32, ct.c_void_p, ct.POINTER(ct.c_int64),
                      ct.c_int32, ct.c_int32, ct.POINTER(ct.c_int32), ct.c_void_p, ct.POINTER(ct.c_int32),
                      ct.POINTER(ct.c_uint32), ct.c_int64, ct.POINTER(ct.c_int64)]
        f.restype = ct.c_int
        mat, matp = _i8(mat)
        P = BatchParams(matp, n, gap_open, gap_extend, flag, filters, filterd, mask_len, score_size)
        if table is None:
            qc, qo = concat(queries)
            rc, ro = concat(refs)
            tabp = None
        else:
            qs = [q.encode() if isinstance(q, str) else bytes(q) for q in queries]
            rs = [r.encode() if isinstance(r, str) else bytes(r) for r in refs]
            qc = np.frombuffer(b"".join(qs) + b"\0", dtype=np.uint8)
            rc = np.frombuffer(b"".join(rs) + b"\0", dtype=np.uint8)
            qo = np.zeros(len(qs) + 1, dtype=np.int64); qo[1:] = np.cumsum([len(q) for q in qs])
            ro = np.zeros(len(rs) + 1, dtype=np.int64); ro[1:] = np.cumsum([len(r) for r in rs])
            tab = np.ascontiguousarray(table, dtype=np.int8)
            assert tab.size == 128
            tabp = tab.ctypes.data_as(ct.POINTER(ct.c_int8))
        ql, rl = np.diff(qo), np.diff(ro)
        if table is not None and add_reverse_complement:
            ql = np.concatenate([ql, ql])
        rows = max(int(k), 0)
        hit_ref = np.empty((len(ql), rows), dtype=np.int32)
        hits = np.empty((len(ql), rows), dtype=RESULT_DTYPE)
        n_hits = np.empty(len(ql), dtype=np.int32)
        cap = int(rows * np.sum(ql + np.minimum(int(rl.max()), ql * 128) + 4)) if (flag & 7) and len(rl) else 0
        pool = np.empty(max(cap, 1), dtype=np.uint32)
        used = ct.c_int64(0)
        rv = f(self.h, ct.byref(P), tabp, 1 if add_reverse_complement else 0, len(queries), qc.ctypes.data_as(ct.c_void_p),
               qo.ctypes.data_as(ct.POINTER(ct.c_int64)), len(refs), rc.ctypes.data_as(ct.c_void_p), ro.ctypes.data_as(ct.POINTER(ct.c_int64)),
               int(k), int(min_score), hit_ref.ctypes.data_as(ct.POINTER(ct.c_int32)), hits.ctypes.data_as(ct.c_void_p),
               n_hits.ctypes.data_as(ct.POINTER(ct.c_int32)), pool.ctypes.data_as(ct.POINTER(ct.c_uint32)), len(pool), ct.byref(used))
        if rv:
            raise RuntimeError("ssw_group_search failed (%d)" % rv)
        return hit_ref, hits, n_hits, pool[: used.value]

    def search_all(self, queries, refs, mat, n, min_score, max_hits=SEARCH_ALL_MAX_HITS, gap_open=3, gap_extend=1, flag=0,
                   filters=0, filterd=0, mask_len=-1, score_size=2, table=None, add_reverse_complement=False):
        """BatchAligner.search_all over the devices of the group (ssw_group_search_all): sequences as for align().  Returns
        (row_off, hit_ref, hits, cigar_pool); with add_reverse_complement the rows of the reverse complements follow those of
        the queries."""
        f = self.lib.ssw_group_search_all
        f.argtypes = [ct.c_void_p, ct.POINTER(BatchParams), ct.POINTER(ct.c_int8), ct.c_int32,
                      ct.c_int32, ct.c_void_p, ct.POINTER(ct.c_int64), ct.c_int32, ct.c_void_p, ct.POINTER(ct.c_int64),
                      ct.c_int32, ct.c_int64, ct.POINTER(ct.c_void_p)]
        f.restype = ct.c_int
        mat, matp = _i8(mat)
        P = BatchParams(matp, n, gap_open, gap_extend, flag, filters, filterd, mask_len, score_size)
        if table is None:
            qc, qo = concat(queries)
            rc, ro = concat(refs)
            tabp = None
        else:
            qs = [q.encode() if isinstance(q, str) else bytes(q) for q in queries]
            rs = [r.encode() if isinstance(r, str) else bytes(r) for r in refs]
            qc = np.frombuffer(b"".join(qs) + b"\0", dtype=np.uint8)
            rc = np.frombuffer(b"".join(rs) + b"\0", dtype=np.uint8)
            qo = np.zeros(len(qs) + 1, dtype=np.int64); qo[1:] = np.cumsum([len(q) for q in qs])
            ro = np.zeros(len(rs) + 1, dtype=np.int64); ro[1:] = np.cumsum([len(r) for r in rs])
            tab = np.ascontiguousarray(table, dtype=np.int8)
            assert tab.size == 128
            tabp = tab.ctypes.data_as(ct.POINTER(ct.c_int8))
        handle = ct.c_void_p()
        rv = f(self.h, ct.byref(P), tabp, 1 if add_reverse_complement else 0, len(queries), qc.ctypes.data_as(ct.c_void_p),
               qo.ctypes.data_as(ct.POINTER(ct.c_int64)), len(refs), rc.ctypes.data_as(ct.c_void_p), ro.ctypes.data_as(ct.POINTER(ct.c_int64)),
               int(min_score), int(max_hits), ct.byref(handle))
        return _take_hit_set(self.lib, rv, handle, "ssw_group_search_all", max_hits)

    def search_self(self, seqs, mat, n, min_score, max_hits=SEARCH_ALL_MAX_HITS, gap_open=3, gap_extend=1, flag=0, filters=0,
                    filterd=0, mask_len=-1, score_size=2):
        """BatchAligner.search_self over the devices of the group (ssw_group_search_self): every device holds the whole set
        (list of int8 code arrays) and takes a range of canonical ranks as queries.  Returns (row_off, hit_ref, hits, cigar_pool)."""
        f = self.lib.ssw_group_search_self
        f.argtypes = [ct.c_void_p, ct.POINTER(BatchParams), ct.c_int32, ct.POINTER(ct.c_int8), ct.POINTER(ct.c_int64),
                      ct.c_int32, ct.c_int64, ct.POINTER(ct.c_void_p)]
        f.restype = ct.c_int
        mat, matp = _mat(mat)
        P = BatchParams(matp, n, gap_open, gap_extend, flag, filters, filterd, mask_len, score_size)
        c, o = concat(seqs)
        handle = ct.c_void_p()
        rv = f(self.h, ct.byref(P), len(seqs), c.ctypes.data_as(ct.POINTER(ct.c_int8)), o.ctypes.data_as(ct.POINTER(ct.c_int64)),
               int(min_score), int(max_hits), ct.byref(handle))
        return _take_hit_set(self.lib, rv, handle, "ssw_group_search_self", max_hits)
