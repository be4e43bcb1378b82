/*
 * ssw_grid.cuh -- device-side planning for large query x reference grids (scores only, flag 0).
 *
 * The reference's CLI aligns every read against every reference in a double loop (src/main.c:462-532); database
 * search workloads (BASELINE config 4: 10 k queries x 50 k targets) make that grid hundreds of millions of pairs.
 * Building one item and two alignment descriptors per pair-task on the host costs more than the kernels, so for a
 * full grid whose references fit one chunk the descriptors are generated on the device from three small tables
 * (queries, query pairs, references), and the resolve output is written straight into the caller-visible
 * ssw_batch_result records.  Pairs whose byte-semantics score overflowed are appended to a list and re-done by the
 * general path.
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
	o.score1 = 0; o.score2 = 0; o.ref_begin1 = -1; o.ref_end1 = 0; o.read_begin1 = -1; o.read_end1 = 0; o.ref_end2 = 0;
	o.cigar_off = -1; o.cigar_len = 0; o.flag = 0; o.status = 0;
	if (f.overflow) {
		const int slot = atomicAdd(redo_count, 1);
		if (slot < redo_cap) redo_list[slot] = (int32_t)p;
	} else if (f.score > 0) {
		o.score1 = (uint16_t)f.score; o.ref_end1 = f.ref; o.read_end1 = f.read;
		if (qt[q].mask_len >= 15) { o.score2 = (uint16_t)f.score2; o.ref_end2 = f.ref2; }
		else { o.score2 = 0; o.ref_end2 = -1; }
	}
	out[p] = o;
}

#endif /* SSW_GRID_CUH */
