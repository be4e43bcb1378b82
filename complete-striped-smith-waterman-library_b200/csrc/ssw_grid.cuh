/*
 * ssw_grid.cuh -- device-side planning for large query x reference grids (scores only, flag 0).
 *
 * The reference's CLI aligns every read against every reference in a double loop (src/main.c:462-532); database
 * search workloads (BASELINE config 4: 10 k queries x 50 k targets) make that grid hundreds of millions of pairs.
 * Building one item and two alignment descriptors per pair-task on the host costs more than the kernels, so for a
 * full grid whose references fit one chunk the descriptors are generated on the device from three small tables
 * (queries, query pairs, references; a search passes the sequences that qualify, references in ascending order of their
 * index, and maps the indices back on the host), and the resolve output is written straight into the caller-visible
 * ssw_batch_result records.  Pairs whose byte-semantics score overflowed are appended to a list and re-done by the
 * general path.  A top-k search (ssw_engine_search) replaces the emit kernel by a selection kernel that keeps only each
 * query's k best records; a threshold search (ssw_engine_search_all) by a count and a compaction kernel that keep every hit.
 * Six kernels -- plan, emit, select, merge (top-k over grid tiles), count and compact -- read one query-pair table
 * (SswGridQp), which describes a full grid and a self-search's triangle (ssw_engine_search_self) alike.
 */
#ifndef SSW_GRID_CUH
#define SSW_GRID_CUH

#include "ssw_common.cuh"
#include "../../include/ssw_batch.h"

/* one query: slice, padded rows of this pass, mask window, the score limit of this pass (SswAlnDesc.limit: per query, as query
 * profiles have their own byte bias) */
struct SswGridQ { int32_t off, len, lp, mask_len, limit; };

struct SswGridArgs {
	int32_t n_qp;        /* query pairs in this launch */
	int32_t n_r;         /* references */
	int32_t word;
	int32_t arm_tail;    /* > 0: best-cell rows are recorded in the last arm_tail columns of every reference only (SswItem.cend) */
};

/* One query pair of a launch: queries qa and qb (-1: none) and their first references, lo_a and lo_b (lo_a <= lo_b).  Slot rr of
 * the pair sweeps reference perm[rr]; the host orders the slots so that the references half a needs, [lo_a, n_r), are the slots
 * [0, n_r - lo_a) -- the live slots -- and half b needs [lo_b, n_r).  A full grid has lo_a = lo_b = 0; a self-search, whose
 * references are in canonical order and swept in reverse, the references ranked after each half's query.  The pair's items
 * start at item0 (its live slots padded to whole CTAs), the descriptors of reference r at 2 (desc0 + r - lo_a) and its column
 * maxima at cm0 + cm_prefix[r] - cm_prefix[lo_a].  Entry n_qp of the table holds the launch's totals in item0, desc0 and cm0. */
struct SswGridQp { int32_t qa, qb, lo_a, lo_b; int64_t item0, desc0, cm0; };

/* thread idx -> item (query pair found by binary search over item0, slot rr): writes the fill item and, for live slots, the two
 * alignment descriptors.  Slots are ordered by length where the host can (the groups of a warp, which run as long as their
 * longest item, then end together); descriptors, column maxima and with them the resolve results stay at the reference's own
 * position r, so nothing after the fill knows about the order of the launch.  A dead slot repeats the last live slot's
 * reference with no columns. */
__global__ void __launch_bounds__(256)
ssw_grid_plan_kernel(SswGridArgs A, const SswGridQp* __restrict__ qp, const SswGridQ* __restrict__ qt,
                     const int64_t* __restrict__ ref_off, const int32_t* __restrict__ ref_len, const int64_t* __restrict__ cm_prefix,
                     const int32_t* __restrict__ perm, SswItem* __restrict__ items, SswAlnDesc* __restrict__ descs)
{
	const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= qp[A.n_qp].item0) return;
	int pi = 0;
	for (int hi = A.n_qp - 1; pi < hi;) {
		const int m = (pi + hi + 1) >> 1;
		if (qp[m].item0 <= idx) pi = m; else hi = m - 1;
	}
	const SswGridQp s = qp[pi];
	const int rr = (int)(idx - s.item0), n_live = A.n_r - s.lo_a;
	const bool live = rr < n_live;
	const int r = perm[live ? rr : n_live - 1];
	const SswGridQ qa = qt[s.qa];
	SswItem it;
	it.qa.off = qa.off; it.qa.len = qa.len; it.qa.lp = qa.lp; it.qa.rev = 0;
	it.qb.off = 0; it.qb.len = 0; it.qb.lp = 0; it.qb.rev = 0;
	SswGridQ qb;
	qb.off = 0; qb.len = 0; qb.lp = 0; qb.mask_len = 0; qb.limit = 0;
	if (s.qb >= 0) { qb = qt[s.qb]; it.qb.off = qb.off; it.qb.len = qb.len; it.qb.lp = qb.lp; }
	it.ref_off = ref_off[r]; it.ref_len = ref_len[r];
	it.cend = (A.arm_tail > 0 && live) ? max(0, ref_len[r] - A.arm_tail) : 0;
	it.p0 = 0; it.p1 = live ? ref_len[r] : 0; it.warm = 0; it.term_a = -1;
	it.cm_off = live ? s.cm0 + cm_prefix[r] - cm_prefix[s.lo_a] : SSW_CM_NONE;
	items[idx] = it;
	if (live) {
		SswAlnDesc d;
		d.first_item = (int32_t)idx; d.n_items = 1; d.half = 0; d.ref_len = it.ref_len; d.read_len = qa.len;
		d.word = A.word; d.limit = qa.limit; d.mask_len = qa.mask_len; d.cm_off = it.cm_off; d.scan_all = 0; d.warm = 0; d.byte_pad = 0;
		const int64_t di = (s.desc0 + r - s.lo_a) * 2;
		descs[di] = d;
		d.half = 1; d.read_len = qb.len; d.mask_len = qb.mask_len; d.limit = qb.limit;
		if (s.qb < 0 || r < s.lo_b) d.n_items = 0;                      /* no second query, or a reference it does not need: skipped */
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

/* resolve result -> ssw_batch_result of pair (query, reference); overflowed byte results are queued for a re-run.  An align's
 * grid is full: descriptor di belongs to query pair di / (2 n_r). */
__global__ void __launch_bounds__(256)
ssw_grid_emit_kernel(SswGridArgs A, const SswGridQp* __restrict__ qp, const SswGridQ* __restrict__ qt,
                     const SswFillResult* __restrict__ res, ssw_batch_result* __restrict__ out,
                     int32_t* __restrict__ redo_list, int32_t* __restrict__ redo_count, int32_t redo_cap)
{
	const int64_t di = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (di >= (int64_t)A.n_qp * A.n_r * 2) return;
	const int h = (int)(di & 1);
	const int64_t pt = di >> 1;
	const int pi = (int)(pt / A.n_r), r = (int)(pt % A.n_r);
	const int q = h ? qp[pi].qb : qp[pi].qa;
	if (q < 0) return;
	const SswFillResult f = res[di];
	const int64_t p = (int64_t)q * A.n_r + r;
	ssw_batch_result o;
	ssw_grid_record<true>(f, qt[q].mask_len, p, o, redo_list, redo_count, redo_cap);
	out[p] = o;
}

/* The query slot (pi, half) of CTA blockIdx.x in the selection, count and compaction kernels: its query q (-1: none), the
 * query's mask_len, and the references it needs, [r0, n_r), whose resolve results are rq[2 r] and pair numbers p0 + r. */
struct SswGridSlot { int q, mask_len, r0; const SswFillResult* rq; int64_t p0; };

__device__ __forceinline__ SswGridSlot ssw_grid_slot(int n_r, const SswGridQp* __restrict__ qp, const SswGridQ* __restrict__ qt,
                                                     const SswFillResult* __restrict__ res)
{
	const int h = (int)(blockIdx.x & 1);
	const SswGridQp* s = qp + (blockIdx.x >> 1);
	SswGridSlot o;
	o.q = h ? s->qb : s->qa;
	o.mask_len = o.q >= 0 ? qt[o.q].mask_len : 0;
	o.r0 = h ? s->lo_b : s->lo_a;
	o.rq = res + 2 * (s->desc0 - s->lo_a) + h;
	o.p0 = (int64_t)o.q * n_r;
	return o;
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
 * queues them and take no part in the selection; the host merges their records in afterwards.  A top-k search's grid is full
 * (lo_a = lo_b = 0), so a slot sweeps all n_r references (a start at r0 costs this kernel spills on sm_90a).
 *   threshold: two 8-bit histogram passes find the score T of the k-th best hit;
 *   ordered pass: in reference order, every hit above T and the first (k - hits above T) hits at T become candidates;
 *   the <= k candidates are sorted in shared memory and their records written. */
__global__ void __launch_bounds__(SSW_SELECT_THREADS)
ssw_grid_select_kernel(SswGridArgs A, const SswGridQp* __restrict__ qp, const SswGridQ* __restrict__ qt,
                       const SswFillResult* __restrict__ res, int32_t k, int32_t min_score,
                       int32_t* __restrict__ hit_ref, ssw_batch_result* __restrict__ hits, int32_t* __restrict__ n_hits,
                       int32_t* __restrict__ redo_list, int32_t* __restrict__ redo_count, int32_t redo_cap)
{
	__shared__ int32_t s_hist[256];
	__shared__ int32_t s_warp[2][SSW_SELECT_THREADS / 32];
	__shared__ int32_t s_cut[3];                       /* threshold score, hits above it, hits in all */
	__shared__ uint64_t s_key[SSW_SEARCH_MAX_K];
	const SswGridSlot sl = ssw_grid_slot(A.n_r, qp, qt, res);
	const int q = sl.q;
	if (q < 0) return;                                 /* the whole CTA: no second query in this pair-task */
	const int mask_len = sl.mask_len, n_r = A.n_r, tid = threadIdx.x;
	const SswFillResult* rq = sl.rq;
	const int64_t p0 = sl.p0;

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

/* Top-k search over grid tiles: one CTA per query slot (pi, half) of a launch group of a later tile, run after the selection
 * kernel wrote the slot's row to the tile table (t_*; reference numbers of the tile, offset by r_base here).  Row q of the
 * running table becomes the first min(k, n_a + n_b) of the two rows in rank order -- in place: every thread reads its entries
 * before the barrier and writes them after it.  Every reference of the tile has a larger number than every reference of the
 * running row, so the keys are distinct and the result is the selection over the union (grid hits never have status 1).
 * Output i comes from the merge path: x entries of the running row and i - x of the tile row precede it. */
__global__ void __launch_bounds__(SSW_SELECT_THREADS)
ssw_grid_merge_kernel(const SswGridQp* __restrict__ qp, int32_t k, int32_t r_base,
                      int32_t* __restrict__ hit_ref, ssw_batch_result* __restrict__ hits, int32_t* __restrict__ n_hits,
                      const int32_t* __restrict__ t_ref, const ssw_batch_result* __restrict__ t_hits, const int32_t* __restrict__ t_n)
{
	constexpr int kPer = SSW_SEARCH_MAX_K / SSW_SELECT_THREADS;      /* outputs per thread */
	__shared__ uint64_t s_a[SSW_SEARCH_MAX_K], s_b[SSW_SEARCH_MAX_K];
	const int q = blockIdx.x & 1 ? qp[blockIdx.x >> 1].qb : qp[blockIdx.x >> 1].qa;
	if (q < 0) return;                                 /* the whole CTA: no second query in this pair-task */
	const int tid = threadIdx.x;
	const int64_t row = (int64_t)q * k;
	const int na = n_hits[q], nb = t_n[q];
	for (int i = tid; i < na; i += SSW_SELECT_THREADS) s_a[i] = ssw_hit_key(hits[row + i].score1, hit_ref[row + i]);
	for (int i = tid; i < nb; i += SSW_SELECT_THREADS) s_b[i] = ssw_hit_key(t_hits[row + i].score1, r_base + t_ref[row + i]);
	__syncthreads();
	const int cnt = min(k, na + nb);
	ssw_batch_result o[kPer];
	int32_t ref[kPer];
#pragma unroll
	for (int j = 0; j < kPer; ++j) {
		const int i = tid + j * SSW_SELECT_THREADS;
		if (i < cnt) {
			int lo = max(0, i - nb), hi = min(i, na);
			while (lo < hi) {
				const int m = (lo + hi) >> 1;
				if (s_a[m] < s_b[i - 1 - m]) lo = m + 1; else hi = m;
			}
			const int y = i - lo;
			if (y >= nb || (lo < na && s_a[lo] < s_b[y])) { o[j] = hits[row + lo]; ref[j] = hit_ref[row + lo]; }
			else { o[j] = t_hits[row + y]; ref[j] = r_base + t_ref[row + y]; }
		}
	}
	__syncthreads();
#pragma unroll
	for (int j = 0; j < kPer; ++j) {
		const int i = tid + j * SSW_SELECT_THREADS;
		if (i < cnt) { hits[row + i] = o[j]; hit_ref[row + i] = ref[j]; }
	}
	if (tid == 0) n_hits[q] = cnt;
}

/* ---- threshold search (ssw_engine_search_all): every hit, compacted in reference order ----------------------------------- */

/* One CTA per query slot (pi, half) of a launch group, as the selection kernel: slot_n[slot] receives the number of hits of
 * that query among the group's resolve results (0 for a slot without a query).  The only kernel of the threshold search that
 * queues redo pairs: each pair of the group is visited once, so each is queued once. */
__global__ void __launch_bounds__(SSW_SELECT_THREADS)
ssw_grid_count_kernel(SswGridArgs A, const SswGridQp* __restrict__ qp, const SswGridQ* __restrict__ qt,
                      const SswFillResult* __restrict__ res, int32_t min_score, int32_t* __restrict__ slot_n,
                      int32_t* __restrict__ redo_list, int32_t* __restrict__ redo_count, int32_t redo_cap)
{
	__shared__ int32_t s_n;
	const SswGridSlot sl = ssw_grid_slot(A.n_r, qp, qt, res);
	const int tid = threadIdx.x;
	if (sl.q < 0) {                                    /* the whole CTA: no second query in this pair-task */
		if (tid == 0) slot_n[blockIdx.x] = 0;
		return;
	}
	if (tid == 0) s_n = 0;
	__syncthreads();
	int c = 0;
	for (int r = sl.r0 + tid; r < A.n_r; r += SSW_SELECT_THREADS) {
		ssw_batch_result o;
		if (ssw_grid_record<true>(sl.rq[2 * (int64_t)r], sl.mask_len, sl.p0 + r, o, redo_list, redo_count, redo_cap) && o.score1 >= min_score) ++c;
	}
	if (c) atomicAdd(&s_n, c);
	__syncthreads();
	if (tid == 0) slot_n[blockIdx.x] = s_n;
}

/* Same layout: the hits of a slot in reference order, written contiguously from slot_off[slot] (the host's exclusive prefix of
 * the counts over the group's slots): one ordered ballot pass, as pass 3 of the selection kernel, which stops once the slot's
 * count is reached.  Records and device reference numbers. */
__global__ void __launch_bounds__(SSW_SELECT_THREADS)
ssw_grid_compact_kernel(SswGridArgs A, const SswGridQp* __restrict__ qp, const SswGridQ* __restrict__ qt,
                        const SswFillResult* __restrict__ res, int32_t min_score, const int64_t* __restrict__ slot_off,
                        int32_t* __restrict__ hit_ref, ssw_batch_result* __restrict__ hits)
{
	__shared__ int32_t s_warp[2][SSW_SELECT_THREADS / 32];
	const SswGridSlot sl = ssw_grid_slot(A.n_r, qp, qt, res);
	if (sl.q < 0) return;
	const int n_r = A.n_r, tid = threadIdx.x;
	const int64_t base = slot_off[blockIdx.x], cnt = slot_off[blockIdx.x + 1] - base;
	int64_t done = 0;
	/* two prefix buffers in turn: a step's writes to one cannot race the reads of the step before, which a barrier separates */
	for (int rb = sl.r0, it = 0; rb < n_r && done < cnt; rb += SSW_SELECT_THREADS, ++it) {
		const int r = rb + tid;
		ssw_batch_result o;
		const bool hit = r < n_r && ssw_grid_record<false>(sl.rq[2 * (int64_t)r], sl.mask_len, sl.p0 + r, o, nullptr, nullptr, 0) && o.score1 >= min_score;
		int n = 0;
		const int at = ssw_block_prefix(hit, s_warp[it & 1], &n);
		if (hit) {
			hits[base + done + at] = o;
			hit_ref[base + done + at] = r;
		}
		done += n;
	}
}

#endif /* SSW_GRID_CUH */
