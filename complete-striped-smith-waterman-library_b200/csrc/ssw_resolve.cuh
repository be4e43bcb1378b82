/*
 * ssw_resolve.cuh -- the order-dependent bookkeeping that follows a matrix fill
 * ("pass B" of SURVEY Appendix A.3).  Replaces, per alignment:
 *   - the running strict-'>' maximum / end_ref / overflow logic of the SSE2
 *     loops (src/ssw.c:318-335 byte, :523-537 word),
 *   - the end_read scan (:342-351, :544-553),
 *   - the second-best scan outside the mask window (:368-381, :570-583).
 * One warp per alignment.  Input: the per-item best cells written by the fill
 * kernel and the packed column-maximum row of the pair-task.  Items are in
 * scan order, so the first item holding the maximum also holds its first
 * column.  An item's best cell is at the same time (max, first index) of the
 * column maxima over its range, so the second-best scan reads column maxima
 * only for the few items that straddle the mask window.
 */
#ifndef SSW_RESOLVE_CUH
#define SSW_RESOLVE_CUH

#include "ssw_common.cuh"

#define SSW_RESOLVE_THREADS 128

/* candidate (v, i) beats (bv, bi): larger value, then smaller index; zero never counts */
__device__ static __forceinline__ bool ssw_second_better(int v, int i, int bv, int bi)
{
	return v > bv || (v == bv && v > 0 && i < bi);
}

template <bool SECOND>
__global__ void __launch_bounds__(SSW_RESOLVE_THREADS)
ssw_resolve_kernel(const SswAlnDesc* __restrict__ alns, int n_aln,
                   const SswItemBest* __restrict__ bests, const uint32_t* __restrict__ colmax,
                   SswFillResult* __restrict__ out)
{
	constexpr unsigned FULL = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	const int idx = (int)blockIdx.x * (SSW_RESOLVE_THREADS / 32) + (threadIdx.x >> 5);
	if (idx >= n_aln) return;
	const SswAlnDesc d = alns[idx];
	const int h = d.half;

	/* best cell over the alignment's records: max score, then first scan position, then smallest row */
	int sc = 0, pos = 0x7fffffff, row = 0x7fffffff;
	for (int k = lane; k < d.n_items; k += 32) {
		const SswItemBest b = bests[d.first_item + k];
		const int s = b.score[h], p = b.pos[h], rr = b.row[h];
		if (s > 0 && (s > sc || (s == sc && (p < pos || (p == pos && rr < row))))) { sc = s; pos = p; row = rr; }
	}
#pragma unroll
	for (int off = 16; off >= 1; off >>= 1) {
		const int o_sc = __shfl_xor_sync(FULL, sc, off);
		const int o_pos = __shfl_xor_sync(FULL, pos, off), o_row = __shfl_xor_sync(FULL, row, off);
		if (o_sc > sc || (o_sc == sc && (o_pos < pos || (o_pos == pos && o_row < row)))) { sc = o_sc; pos = o_pos; row = o_row; }
	}
	if (sc == 0) { pos = 0; row = 0; }
	const bool unarmed = sc > 0 && pos < 0;          /* the maximum lies before the armed range of its item: no position, no row */
	if (unarmed) { pos = 0; row = 0; }

	SswFillResult r;
	r.score = sc; r.ref = pos; r.read = row < d.read_len - 1 ? row : d.read_len - 1;
	r.score2 = 0; r.ref2 = 0; r.overflow = 0; r.pad_[0] = r.pad_[1] = 0;
	if (sc == 0) { r.ref = d.word ? 0 : -1; r.read = 0; }
	if (sc >= d.limit) { r.overflow = d.word ? 2 : 1; if (!d.word) r.score = 255; }
	else if (unarmed) r.overflow = 3;                 /* the caller re-does the pair with arm 0 */

	if (SECOND && sc > 0 && !r.overflow && d.cm_off != SSW_CM_NONE) {
		/* allowed columns: [0, e1) and [e2, refLen); smallest index of the largest value, values must be > 0 */
		const int e1 = max(pos - d.mask_len, 0);
		const int e2 = min(pos + d.mask_len, d.ref_len) + (d.word ? 0 : 1);
		const uint32_t* cm = colmax + d.cm_off;
		int v2 = 0, i2 = 0;
		if (d.scan_all) {
			for (int c = lane; c < d.ref_len; c += 32) {
				if (c < e1 || c >= e2) {
					const int v = half_of(cm[c], h);
					if (ssw_second_better(v, c, v2, i2)) { v2 = v; i2 = c; }
				}
			}
		} else
		for (int k0 = 0; k0 < d.n_items; k0 += 32) {
			const int k = k0 + lane;
			bool straddles = false;
			int p0 = 0, p1 = 0;
			if (k < d.n_items) {
				const SswItemBest b = bests[d.first_item + k];
				p0 = b.p0; p1 = b.p1;
				if (p1 <= e1 || p0 >= e2) { if (ssw_second_better(b.score[h], b.pos[h], v2, i2)) { v2 = b.score[h]; i2 = b.pos[h]; } }
				else straddles = true;
			}
			/* items touching the masked window: the warp scans their allowed columns element-wise */
			unsigned todo = __ballot_sync(FULL, straddles);
			while (todo) {
				const int src = __ffs((int)todo) - 1;
				todo &= todo - 1;
				const int q0 = __shfl_sync(FULL, p0, src), q1 = __shfl_sync(FULL, p1, src);
				for (int c = q0 + lane; c < q1; c += 32) {
					if (c < e1 || c >= e2) {
						const int v = half_of(cm[c], h);
						if (ssw_second_better(v, c, v2, i2)) { v2 = v; i2 = c; }
					}
				}
			}
		}
#pragma unroll
		for (int off = 16; off >= 1; off >>= 1) {
			const int o_v = __shfl_xor_sync(FULL, v2, off), o_i = __shfl_xor_sync(FULL, i2, off);
			if (ssw_second_better(o_v, o_i, v2, i2)) { v2 = o_v; i2 = o_i; }
		}
		r.score2 = v2; r.ref2 = i2;
	}
	if (lane == 0) out[idx] = r;
}

/* ---------------------------------------------------------------------------------------------------------- */
/* block-maximum mode (fill kernel CM == 2): one word per SSW_CM_BLOCK columns instead of one per column       */
/* ---------------------------------------------------------------------------------------------------------- */
/*
 * The second-best scan wants (largest value, smallest column) over the columns outside the mask window.  With
 * block maxima that is known exactly for every item that does not touch the window (its best cell is the summary),
 * and per block for the others; single columns are needed only in
 *   - the block cut by the left edge of the window and the block cut by its right edge, and
 *   - the first block holding the largest block maximum among the fully allowed blocks (to find its first column).
 * Stage 1 (ssw_resolve_blocks_kernel) does everything ssw_resolve_kernel does, keeps the best exact candidate in
 * score2/ref2, and emits three re-fill items per alignment (dead ones where nothing is needed): the same pair-task,
 * counted range = one block, warm-up as the chunks of the main launch.  The fill kernel (CM == 1) writes their 64
 * column maxima into a small scratch; stage 2 (ssw_resolve_refill_kernel) folds them in.
 * A byte alignment filled on its word rows (SswAlnDesc.byte_pad > 0) gets a fourth item: columns [e2, e2 + 8) on the
 * byte rows, the only allowed columns whose byte column maxima can exceed the word ones in a way the scan sees (DESIGN 2).
 * Its range starts at e2 rounded down to 4 (the 128-bit column stores of the fill); blocks 0..2 stay on the word rows,
 * they reproduce the columns the main fill summarised.
 */
#define SSW_REFILL_SLOTS 4
#define SSW_REFILL_ZONE 3       /* slot of the byte-row columns right of the mask window */

template <int DUMMY = 0>
__global__ void __launch_bounds__(SSW_RESOLVE_THREADS)
ssw_resolve_blocks_kernel(const SswAlnDesc* __restrict__ alns, int n_aln,
                          const SswItemBest* __restrict__ bests, const uint32_t* __restrict__ blkmax,
                          const SswItem* __restrict__ items, SswFillResult* __restrict__ out,
                          SswItem* __restrict__ refill_items, int32_t* __restrict__ refill_c0)
{
	constexpr unsigned FULL = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	const int idx = (int)blockIdx.x * (SSW_RESOLVE_THREADS / 32) + (threadIdx.x >> 5);
	if (idx >= n_aln) return;
	const SswAlnDesc d = alns[idx];
	const int h = d.half;

	int sc = 0, pos = 0x7fffffff, row = 0x7fffffff;
	for (int k = lane; k < d.n_items; k += 32) {
		const SswItemBest b = bests[d.first_item + k];
		const int s = b.score[h], p = b.pos[h], rr = b.row[h];
		if (s > 0 && (s > sc || (s == sc && (p < pos || (p == pos && rr < row))))) { sc = s; pos = p; row = rr; }
	}
#pragma unroll
	for (int off = 16; off >= 1; off >>= 1) {
		const int o_sc = __shfl_xor_sync(FULL, sc, off);
		const int o_pos = __shfl_xor_sync(FULL, pos, off), o_row = __shfl_xor_sync(FULL, row, off);
		if (o_sc > sc || (o_sc == sc && (o_pos < pos || (o_pos == pos && o_row < row)))) { sc = o_sc; pos = o_pos; row = o_row; }
	}
	if (sc == 0) { pos = 0; row = 0; }
	const bool unarmed = sc > 0 && pos < 0;          /* the maximum lies before the armed range of its item: no position, no row */
	if (unarmed) { pos = 0; row = 0; }

	SswFillResult r;
	r.score = sc; r.ref = pos; r.read = row < d.read_len - 1 ? row : d.read_len - 1;
	r.score2 = 0; r.ref2 = 0; r.overflow = 0; r.pad_[0] = r.pad_[1] = 0;
	if (sc == 0) { r.ref = d.word ? 0 : -1; r.read = 0; }
	if (sc >= d.limit) { r.overflow = d.word ? 2 : 1; if (!d.word) r.score = 255; }
	else if (unarmed) r.overflow = 3;                 /* the caller re-does the pair with arm 0 */

	int slots[SSW_REFILL_SLOTS] = {-1, -1, -1, -1};     /* block ids; the zone slot: its first column */
	int zone_end = 0;
	if (sc > 0 && !r.overflow && d.cm_off != SSW_CM_NONE && d.n_items > 0) {
		const int e1 = max(pos - d.mask_len, 0);
		const int e2 = min(pos + d.mask_len, d.ref_len) + (d.word ? 0 : 1);
		if (d.byte_pad > 0 && e2 < d.ref_len) { slots[SSW_REFILL_ZONE] = e2 & ~3; zone_end = min(e2 + 8, d.ref_len); }
		const uint32_t* bm = blkmax + d.cm_off;
		int vx = 0, ix = 0;                  /* best exact candidate: items that do not touch the window */
		int vb = 0, bb = 0x7fffffff;         /* best fully allowed block of the items that do: (value, smallest block) */
		for (int k0 = 0; k0 < d.n_items; k0 += 32) {
			const int k = k0 + lane;
			bool straddles = false;
			int p0 = 0, p1 = 0;
			if (k < d.n_items) {
				const SswItemBest b = bests[d.first_item + k];
				p0 = b.p0; p1 = b.p1;
				if (p1 <= e1 || p0 >= e2) { if (ssw_second_better(b.score[h], b.pos[h], vx, ix)) { vx = b.score[h]; ix = b.pos[h]; } }
				else straddles = p1 > p0;
			}
			unsigned todo = __ballot_sync(FULL, straddles);
			while (todo) {
				const int src = __ffs((int)todo) - 1;
				todo &= todo - 1;
				const int q0 = __shfl_sync(FULL, p0, src), q1 = __shfl_sync(FULL, p1, src);
				for (int b = q0 / SSW_CM_BLOCK + lane; b * SSW_CM_BLOCK < q1; b += 32) {
					const int bs = b * SSW_CM_BLOCK, be = min(bs + SSW_CM_BLOCK, q1);
					if (be <= e1 || bs >= e2) {
						const int v = half_of(bm[b], h);
						if (v > vb || (v == vb && v > 0 && b < bb)) { vb = v; bb = b; }
					}
				}
			}
		}
#pragma unroll
		for (int off = 16; off >= 1; off >>= 1) {
			const int o_v = __shfl_xor_sync(FULL, vx, off), o_i = __shfl_xor_sync(FULL, ix, off);
			if (ssw_second_better(o_v, o_i, vx, ix)) { vx = o_v; ix = o_i; }
			const int o_vb = __shfl_xor_sync(FULL, vb, off), o_bb = __shfl_xor_sync(FULL, bb, off);
			if (o_vb > vb || (o_vb == vb && o_vb > 0 && o_bb < bb)) { vb = o_vb; bb = o_bb; }
		}
		r.score2 = vx; r.ref2 = ix;
		/* blocks cut by the window edges (e1 > 0 and e2 < ref_len whenever the remainder is non-zero / tested) */
		if (e1 % SSW_CM_BLOCK) slots[0] = e1 / SSW_CM_BLOCK;
		if ((e2 % SSW_CM_BLOCK) && e2 < d.ref_len && e2 / SSW_CM_BLOCK != slots[0]) slots[1] = e2 / SSW_CM_BLOCK;
		if (vb > 0 && vb >= vx) slots[2] = bb;
	}
	if (lane == 0) out[idx] = r;
	if (lane < SSW_REFILL_SLOTS) {
		const int b = slots[lane];
		const int64_t slot = (int64_t)idx * SSW_REFILL_SLOTS + lane;
		SswItem it = items[d.n_items > 0 ? d.first_item : 0];
		it.term_a = -1; it.cend = 0;
		int c0 = -1;
		if (b >= 0) {
			if (lane == SSW_REFILL_ZONE) {
				it.p0 = b; it.p1 = zone_end;
				if (h) it.qb.lp += d.byte_pad; else it.qa.lp += d.byte_pad;
			} else { it.p0 = b * SSW_CM_BLOCK; it.p1 = min(it.p0 + SSW_CM_BLOCK, d.ref_len); }
			it.warm = min(d.warm, it.p0);     /* d.warm is taken from the byte padding */
			it.cm_off = slot * SSW_CM_BLOCK - it.p0;
			c0 = it.p0;
		} else { it.p0 = it.p1 = 0; it.warm = 0; it.cm_off = SSW_CM_NONE; }
		refill_items[slot] = it;
		refill_c0[slot] = c0;
	}
}

/* stage 2: fold the re-filled ranges (single column maxima) into the second-best candidate of stage 1 */
template <int DUMMY = 0>
__global__ void __launch_bounds__(SSW_RESOLVE_THREADS)
ssw_resolve_refill_kernel(const SswAlnDesc* __restrict__ alns, int n_aln, const int32_t* __restrict__ refill_c0,
                          const uint32_t* __restrict__ refill_cm, SswFillResult* __restrict__ out)
{
	constexpr unsigned FULL = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	const int idx = (int)blockIdx.x * (SSW_RESOLVE_THREADS / 32) + (threadIdx.x >> 5);
	if (idx >= n_aln) return;
	const SswAlnDesc d = alns[idx];
	const int h = d.half;
	SswFillResult r = out[idx];
	if (!(r.score > 0 && !r.overflow && d.cm_off != SSW_CM_NONE)) return;
	const int e1 = max(r.ref - d.mask_len, 0);
	const int e2 = min(r.ref + d.mask_len, d.ref_len) + (d.word ? 0 : 1);
	int v2 = r.score2, i2 = r.ref2;
#pragma unroll
	for (int s = 0; s < SSW_REFILL_SLOTS; ++s) {
		const int64_t slot = (int64_t)idx * SSW_REFILL_SLOTS + s;
		const int c0 = refill_c0[slot];
		if (c0 < 0) continue;
		const int c1 = min(s == SSW_REFILL_ZONE ? e2 + 8 : c0 + SSW_CM_BLOCK, d.ref_len);
		for (int j = lane; c0 + j < c1; j += 32) {
			const int c = c0 + j;
			if (c < e1 || c >= e2) {
				const int v = half_of(refill_cm[slot * SSW_CM_BLOCK + j], h);
				if (ssw_second_better(v, c, v2, i2)) { v2 = v; i2 = c; }
			}
		}
	}
#pragma unroll
	for (int off = 16; off >= 1; off >>= 1) {
		const int o_v = __shfl_xor_sync(FULL, v2, off), o_i = __shfl_xor_sync(FULL, i2, off);
		if (ssw_second_better(o_v, o_i, v2, i2)) { v2 = o_v; i2 = o_i; }
	}
	if (lane == 0) { out[idx].score2 = v2; out[idx].ref2 = i2; }
}

#endif /* SSW_RESOLVE_CUH */
