/*
 * ssw_grid.cuh -- device-side planning for large query x reference grids (scores only, flag 0).
 *
 * The reference's CLI aligns every read against every reference in a double loop (src/main.c:462-532); database
 * search workloads (BASELINE config 4: 10 k queries x 50 k targets) make that grid hundreds of millions of pairs.
 * Building one item and two alignment descriptors per pair-task on the host costs more than the kernels, so for a
 * full grid whose references fit one chunk the descriptors are generated on the device from three small tables
 * (queries, query pairs, references), and the resolve output is written straight into the caller-visible
 * ssw_batch_result records.  Pairs whose byte-semantics score overflowed are appended to a list and re-done by the
 * general path.  A top-k search (ssw_engine_search) replaces the emit kernel by a selection kernel that keeps only each
 * query's k best records.
 */
#ifndef SSW_GRID_CUH
#define SSW_GRID_CUH

#include "ssw_common.cuh"
#include "../../include/ssw_batch.h"

struct SswGridQ { int32_t off, len, lp, mask_len; };      /* one query: slice, padded rows of this pass, mask window */

struct SswGridArgs {
	int32_t n_qp;        /* query pairs in this launch */
	int32_t n_r;         /* references */
	int32_t n_r_pad;     /* references rounded up to a whole number of CTAs (dead items in between) */
	int32_t word, limit;
	int32_t arm_tail;    /* > 0: best-cell rows are recorded in the last arm_tail columns of every reference only (SswItem.cend) */
	int64_t cm_words_per_qp;
};

/* thread idx -> item (qp, r): writes the fill item and, for live items, the two alignment descriptors */
__global__ void __launch_bounds__(256)
ssw_grid_plan_kernel(SswGridArgs A, const int2* __restrict__ qp, const SswGridQ* __restrict__ qt,
                     const int64_t* __restrict__ ref_off, const int32_t* __restrict__ ref_len, const int64_t* __restrict__ cm_prefix,
                     SswItem* __restrict__ items, SswAlnDesc* __restrict__ descs)
{
	const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= (int64_t)A.n_qp * A.n_r_pad) return;
	const int pi = (int)(idx / A.n_r_pad), rr = (int)(idx % A.n_r_pad);
	const bool live = rr < A.n_r;
	const int r = live ? rr : A.n_r - 1;
	const int2 pr = qp[pi];
	const SswGridQ qa = qt[pr.x];
	SswItem it;
	it.qa.off = qa.off; it.qa.len = qa.len; it.qa.lp = qa.lp; it.qa.rev = 0;
	it.qb.off = 0; it.qb.len = 0; it.qb.lp = 0; it.qb.rev = 0;
	SswGridQ qb;
	qb.off = 0; qb.len = 0; qb.lp = 0; qb.mask_len = 0;
	if (pr.y >= 0) { qb = qt[pr.y]; it.qb.off = qb.off; it.qb.len = qb.len; it.qb.lp = qb.lp; }
	it.ref_off = ref_off[r]; it.ref_len = ref_len[r];
	it.cend = (A.arm_tail > 0 && live) ? max(0, ref_len[r] - A.arm_tail) : 0;
	it.p0 = 0; it.p1 = live ? ref_len[r] : 0; it.warm = 0; it.term_a = -1;
	it.cm_off = live ? (int64_t)pi * A.cm_words_per_qp + cm_prefix[r] : SSW_CM_NONE;
	items[idx] = it;
	if (live) {
		SswAlnDesc d;
		d.first_item = (int32_t)idx; d.n_items = 1; d.half = 0; d.ref_len = it.ref_len; d.read_len = qa.len;
		d.word = A.word; d.limit = A.limit; d.mask_len = qa.mask_len; d.cm_off = it.cm_off; d.scan_all = 0; d.warm = 0; d.byte_pad = 0;
		const int64_t di = ((int64_t)pi * A.n_r + r) * 2;
		descs[di] = d;
		d.half = 1; d.read_len = qb.len; d.mask_len = qb.mask_len;
		if (pr.y < 0) d.n_items = 0;                                   /* no second query: the resolve kernel skips it */
		descs[di + 1] = d;
	}
}

/* The record of grid pair p = q * n_r + r from its resolve result: the one conversion of the emit and the selection kernels.
 * A result that the general path must re-do (overflow 1 / 2: score limits, 3: best cell before the armed range) leaves the
 * default record and, with kQueue, is appended to the redo list; returns false for it. */
template <bool kQueue>
__device__ __forceinline__ bool ssw_grid_record(const SswFillResult& f, int mask_len, int64_t p, ssw_batch_result& o,
                                                int32_t* __restrict__ redo_list, int32_t* __restrict__ redo_count, int32_t redo_cap)
{
	o.score1 = 0; o.score2 = 0; o.ref_begin1 = -1; o.ref_end1 = 0; o.read_begin1 = -1; o.read_end1 = 0; o.ref_end2 = 0;
	o.cigar_off = -1; o.cigar_len = 0; o.flag = 0; o.status = 0;
	if (f.overflow) {
		if (kQueue) {
			const int slot = atomicAdd(redo_count, 1);
			if (slot < redo_cap) redo_list[slot] = (int32_t)p;
		}
		return false;
	}
	if (f.score > 0) {
		o.score1 = (uint16_t)f.score; o.ref_end1 = f.ref; o.read_end1 = f.read;
		if (mask_len >= 15) { o.score2 = (uint16_t)f.score2; o.ref_end2 = f.ref2; }
		else { o.score2 = 0; o.ref_end2 = -1; }
	}
	return true;
}

/* resolve result -> ssw_batch_result of pair (query, reference); overflowed byte results are queued for a re-run */
__global__ void __launch_bounds__(256)
ssw_grid_emit_kernel(SswGridArgs A, const int2* __restrict__ qp, const SswGridQ* __restrict__ qt,
                     const SswFillResult* __restrict__ res, ssw_batch_result* __restrict__ out,
                     int32_t* __restrict__ redo_list, int32_t* __restrict__ redo_count, int32_t redo_cap)
{
	const int64_t di = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (di >= (int64_t)A.n_qp * A.n_r * 2) return;
	const int h = (int)(di & 1);
	const int64_t pt = di >> 1;
	const int pi = (int)(pt / A.n_r), r = (int)(pt % A.n_r);
	const int2 pr = qp[pi];
	const int q = h ? pr.y : pr.x;
	if (q < 0) return;
	const SswFillResult f = res[di];
	const int64_t p = (int64_t)q * A.n_r + r;
	ssw_batch_result o;
	ssw_grid_record<true>(f, qt[q].mask_len, p, o, redo_list, redo_count, redo_cap);
	out[p] = o;
}

/* ---- top-k selection (ssw_engine_search) ------------------------------------------------------------------------------ */

#define SSW_SELECT_THREADS 256
#define SSW_SEARCH_MAX_K 1024

/* rank key of a hit: ascending order = score descending, then reference index ascending */
__device__ __forceinline__ uint64_t ssw_hit_key(int score, int r) { return ((uint64_t)(0xffff - score) << 32) | (uint32_t)r; }

/* Exclusive block-wide prefix of `pred` over the threads in order (ballot + per-warp counts in `s_warp`); *total receives the
 * block's count.  Every thread of the block must call it. */
__device__ __forceinline__ int ssw_block_prefix(bool pred, int32_t* s_warp, int* total)
{
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const unsigned m = __ballot_sync(0xffffffffu, pred);
	if (lane == 0) s_warp[warp] = __popc(m);
	__syncthreads();
	int before = 0, all = 0;
	for (int w = 0; w < SSW_SELECT_THREADS / 32; ++w) { const int c = s_warp[w]; before += w < warp ? c : 0; all += c; }
	*total = all;
	return before + __popc(m & ((1u << lane) - 1u));
}

/* Histogram scan from the top bucket down: the bucket b in which the `want`-th largest value lies (want >= 1, at most the
 * histogram's total); *above receives the count of the buckets above b.  One thread. */
__device__ __forceinline__ int ssw_hist_cut(const int32_t* hist, int want, int* above)
{
	int acc = 0, b = 255;
	for (; b > 0; --b) {
		if (acc + hist[b] >= want) break;
		acc += hist[b];
	}
	*above = acc;
	return b;
}

/* One CTA per query slot (pi, half) of a launch group: the k best hits of that query among the group's resolve results,
 * written to row q of the n_q x k hit table in rank order (score1 descending, reference ascending).  A hit is a pair whose
 * result is final on the grid (not re-done) with score1 >= min_score (>= 1).  Pairs to re-do are queued as the emit kernel
 * queues them and take no part in the selection; the host merges their records in afterwards.
 *   threshold: two 8-bit histogram passes find the score T of the k-th best hit;
 *   ordered pass: in reference order, every hit above T and the first (k - hits above T) hits at T become candidates;
 *   the <= k candidates are sorted in shared memory and their records written. */
__global__ void __launch_bounds__(SSW_SELECT_THREADS)
ssw_grid_select_kernel(SswGridArgs A, const int2* __restrict__ qp, const SswGridQ* __restrict__ qt,
                       const SswFillResult* __restrict__ res, int32_t k, int32_t min_score,
                       int32_t* __restrict__ hit_ref, ssw_batch_result* __restrict__ hits, int32_t* __restrict__ n_hits,
                       int32_t* __restrict__ redo_list, int32_t* __restrict__ redo_count, int32_t redo_cap)
{
	__shared__ int32_t s_hist[256];
	__shared__ int32_t s_warp[2][SSW_SELECT_THREADS / 32];
	__shared__ int32_t s_cut[3];                       /* threshold score, hits above it, hits in all */
	__shared__ uint64_t s_key[SSW_SEARCH_MAX_K];
	const int h = (int)(blockIdx.x & 1), pi = (int)(blockIdx.x >> 1);
	const int2 pr = qp[pi];
	const int q = h ? pr.y : pr.x;
	if (q < 0) return;                                 /* the whole CTA: no second query in this pair-task */
	const int mask_len = qt[q].mask_len;
	const int n_r = A.n_r, tid = threadIdx.x;
	const SswFillResult* rq = res + (int64_t)pi * n_r * 2 + h;       /* result of reference r: rq[2 * r] */
	const int64_t p0 = (int64_t)q * n_r;

	/* pass 1: histogram of the high score bytes of the hits (and the redo queue) */
	for (int i = tid; i < 256; i += SSW_SELECT_THREADS) s_hist[i] = 0;
	__syncthreads();
	for (int r = tid; r < n_r; r += SSW_SELECT_THREADS) {
		ssw_batch_result o;
		if (ssw_grid_record<true>(rq[2 * (int64_t)r], mask_len, p0 + r, o, redo_list, redo_count, redo_cap) && o.score1 >= min_score)
			atomicAdd(&s_hist[o.score1 >> 8], 1);
	}
	__syncthreads();
	if (tid == 0) {
		int total = 0;
		for (int b = 0; b < 256; ++b) total += s_hist[b];
		s_cut[2] = total;
		s_cut[0] = total <= k ? -1 : ssw_hist_cut(s_hist, k, &s_cut[1]);   /* -1: every hit is kept */
	}
	__syncthreads();
	const int n_all = s_cut[2];
	int thr = s_cut[0], above = 0;
	if (thr >= 0) {
		/* pass 2: low bytes of the hits in the high-byte bucket of the k-th best */
		const int hi = thr, above_hi = s_cut[1];
		for (int i = tid; i < 256; i += SSW_SELECT_THREADS) s_hist[i] = 0;
		__syncthreads();
		for (int r = tid; r < n_r; r += SSW_SELECT_THREADS) {
			ssw_batch_result o;
			if (ssw_grid_record<false>(rq[2 * (int64_t)r], mask_len, p0 + r, o, nullptr, nullptr, 0) && o.score1 >= min_score && (o.score1 >> 8) == hi)
				atomicAdd(&s_hist[o.score1 & 255], 1);
		}
		__syncthreads();
		if (tid == 0) {
			int a = 0;
			const int lo = ssw_hist_cut(s_hist, k - above_hi, &a);
			s_cut[0] = hi << 8 | lo;
			s_cut[1] = above_hi + a;
		}
		__syncthreads();
		thr = s_cut[0];
		above = s_cut[1];
	}
	const int cnt = n_all < k ? n_all : k;
	const int need = thr >= 0 ? k - above : 0;         /* hits at the threshold score that are kept, first in reference order */

	/* pass 3: candidates in reference order (stops once all of them are found) */
	int eq_base = 0, keep_base = 0;
	for (int r0 = 0; r0 < n_r && keep_base < cnt; r0 += SSW_SELECT_THREADS) {
		const int r = r0 + tid;
		bool hit = false;
		int score = 0;
		if (r < n_r) {
			ssw_batch_result o;
			hit = ssw_grid_record<false>(rq[2 * (int64_t)r], mask_len, p0 + r, o, nullptr, nullptr, 0) && o.score1 >= min_score;
			score = o.score1;
		}
		const bool eq = hit && thr >= 0 && score == thr;
		int n_eq = 0, n_keep = 0;
		const int eq_rank = eq_base + ssw_block_prefix(eq, s_warp[0], &n_eq);
		const bool keep = hit && (thr < 0 || score > thr || (eq && eq_rank < need));
		const int slot = keep_base + ssw_block_prefix(keep, s_warp[1], &n_keep);
		if (keep) s_key[slot] = ssw_hit_key(score, r);
		eq_base += n_eq;
		keep_base += n_keep;
	}
	/* bitonic sort of the candidates, padded to a power of two with keys that sort last */
	int size = 1;
	while (size < cnt) size <<= 1;
	for (int i = cnt + tid; i < size; i += SSW_SELECT_THREADS) s_key[i] = ~0ull;
	__syncthreads();
	for (int w = 2; w <= size; w <<= 1)
		for (int j = w >> 1; j > 0; j >>= 1) {
			for (int i = tid; i < size; i += SSW_SELECT_THREADS) {
				const int x = i ^ j;
				if (x > i) {
					const uint64_t a = s_key[i], b = s_key[x];
					if (((i & w) == 0) == (a > b)) { s_key[i] = b; s_key[x] = a; }
				}
			}
			__syncthreads();
		}
	/* the hit records of row q */
	for (int i = tid; i < cnt; i += SSW_SELECT_THREADS) {
		const int r = (int)(uint32_t)s_key[i];
		ssw_batch_result o;
		ssw_grid_record<false>(rq[2 * (int64_t)r], mask_len, p0 + r, o, nullptr, nullptr, 0);
		hits[(int64_t)q * k + i] = o;
		hit_ref[(int64_t)q * k + i] = r;
	}
	if (tid == 0) n_hits[q] = cnt;
}

#endif /* SSW_GRID_CUH */
