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
 * The block-mode fill keeps no best cell.  Its score is the largest block maximum, and its first column lies in the
 * first block holding that value: stage 0 (ssw_resolve_best_block_kernel) finds that block and emits one re-fill item
 * per alignment for it (the same pair-task, counted range = the block, warm-up as the chunks of the main launch), which
 * the fill kernel (CM == 1) runs with its best-cell tracking: (score, first column, smallest row) of that block is the
 * alignment's best cell.
 * The second-best scan wants (largest value, smallest column) over the columns outside the mask window.  With
 * block maxima that is known per block; single columns are needed only in
 *   - the block cut by the left edge of the window and the block cut by its right edge, and
 *   - the first block holding the largest block maximum among the fully allowed blocks (to find its first column).
 * Stage 1 (ssw_resolve_blocks_kernel) does everything ssw_resolve_kernel does, with the best cell of stage 0, and
 * emits three re-fill items per alignment (dead ones where nothing is needed), built like the one of stage 0.  The fill
 * kernel (CM == 1) writes their 64 column maxima into a small scratch; stage 2 (ssw_resolve_refill_kernel) folds them in.
 * A byte alignment filled on its word rows (SswAlnDesc.byte_pad > 0) gets a fourth item: columns [e2, e2 + 8) on the
 * byte rows, the only allowed columns whose byte column maxima can exceed the word ones in a way the scan sees (DESIGN 2).
 * Its range starts at e2 rounded down to 4 (the 128-bit column stores of the fill); blocks 0..2 stay on the word rows,
 * they reproduce the columns the main fill summarised.
 */
#define SSW_REFILL_SLOTS 4
#define SSW_REFILL_ZONE 3       /* slot of the byte-row columns right of the mask window */

/* re-fill item of columns [p0, p1) of the alignment's pair-task (p1 <= p0: a dead item), warm-up as in the main launch */
__device__ static __forceinline__ SswItem ssw_refill_item(const SswAlnDesc& d, const SswItem* __restrict__ items, int p0, int p1)
{
	SswItem it = items[d.n_items > 0 ? d.first_item : 0];
	it.term_a = -1; it.cend = 0; it.cm_off = SSW_CM_NONE;
	if (p1 > p0) { it.p0 = p0; it.p1 = p1; it.warm = min(d.warm, p0); }     /* d.warm is taken from the byte padding */
	else { it.p0 = it.p1 = 0; it.warm = 0; }
	return it;
}

/* stage 0: the first block holding the largest block maximum of the alignment's half, as a re-fill item (dead when the
 * score is 0).  The byte overflow test needs the score only, but the overflowed result keeps its position and row. */
template <int DUMMY = 0>
__global__ void __launch_bounds__(SSW_RESOLVE_THREADS)
ssw_resolve_best_block_kernel(const SswAlnDesc* __restrict__ alns, int n_aln, const uint32_t* __restrict__ blkmax,
                              const SswItem* __restrict__ items, SswItem* __restrict__ best_items)
{
	constexpr unsigned FULL = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	const int idx = (int)blockIdx.x * (SSW_RESOLVE_THREADS / 32) + (threadIdx.x >> 5);
	if (idx >= n_aln) return;
	const SswAlnDesc d = alns[idx];
	int vb = 0, bb = 0x7fffffff;
	if (d.cm_off != SSW_CM_NONE && d.n_items > 0) {
		const uint32_t* bm = blkmax + d.cm_off;
		const int n_blk = (d.ref_len + SSW_CM_BLOCK - 1) / SSW_CM_BLOCK;
		for (int b = lane; b < n_blk; b += 32) {
			const int v = half_of(bm[b], d.half);
			if (v > vb) { vb = v; bb = b; }
		}
	}
#pragma unroll
	for (int off = 16; off >= 1; off >>= 1) {
		const int o_vb = __shfl_xor_sync(FULL, vb, off), o_bb = __shfl_xor_sync(FULL, bb, off);
		if (o_vb > vb || (o_vb == vb && o_bb < bb)) { vb = o_vb; bb = o_bb; }
	}
	if (lane == 0) best_items[idx] = vb > 0 ? ssw_refill_item(d, items, bb * SSW_CM_BLOCK, min(bb * SSW_CM_BLOCK + SSW_CM_BLOCK, d.ref_len))
	                                        : ssw_refill_item(d, items, 0, 0);
}

/* ---- bounded block words (fill kernel CM == 3) ----
 * The word of block b is w(b), and w(b) + gapE <= M(b) <= U(b) = w(b) + gapO + 7 gapE (DESIGN 2; the lower bound of a loop body
 * that straddles two blocks belongs to the later one, so L(b) = w(b) + gapE <= max(M(b), M(b + 1))).  The exact best cell needs
 * single columns only in the blocks C1 = {b : U(b) >= max(T1, 1)}, T1 = max_b L(b) <= score1, and the second-best scan only in
 * the allowed blocks C2 = {b : U(b) >= max(T2, 1)} (stage 1) besides the window edges and the byte-row zone.  Each stage lists
 * an alignment's candidates in block order in cand[idx * cap ...] and their number in cnt (-1: more than cap; the alignment
 * is then resolved from exact words of its pair-task, ssw_engine.cu).  The host turns the counts into offsets, and
 * ssw_bound_emit_kernel writes one re-fill item per candidate. */
struct SswBound { int gapO, gapE, cap; };
#define SSW_BOUND_CAP 256       /* default cap of the candidates per alignment and stage */

/* blocks b of a row of n_blk words with w(b) >= thr that lie entirely outside [e1, e2), in block order, into out[< cap];
 * returns their number (all of them, also beyond cap) */
__device__ static __forceinline__ int ssw_bound_list(const uint32_t* __restrict__ w, int h, int n_blk, int ref_len, int thr,
                                                     int e1, int e2, int32_t* __restrict__ out, int cap, int lane)
{
	int n = 0;
	for (int b0 = 0; b0 < n_blk; b0 += 32) {
		const int b = b0 + lane;
		bool c = false;
		if (b < n_blk) {
			const int bs = b * SSW_CM_BLOCK, be = min(bs + SSW_CM_BLOCK, ref_len);
			c = (be <= e1 || bs >= e2) && half_of(w[b], h) >= thr;
		}
		const unsigned m = __ballot_sync(0xffffffffu, c);
		const int k = n + __popc(m & ((1u << lane) - 1u));
		if (c && k < cap) out[k] = b;
		n += __popc(m);
	}
	return n;
}

/* stage 0 of the bounded words: the C1 candidates of every alignment */
template <int DUMMY = 0>
__global__ void __launch_bounds__(SSW_RESOLVE_THREADS)
ssw_bound_best_kernel(const SswAlnDesc* __restrict__ alns, int n_aln, const uint32_t* __restrict__ words, SswBound bd,
                      int32_t* __restrict__ cand, int32_t* __restrict__ cnt)
{
	constexpr unsigned FULL = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	const int idx = (int)blockIdx.x * (SSW_RESOLVE_THREADS / 32) + (threadIdx.x >> 5);
	if (idx >= n_aln) return;
	const SswAlnDesc d = alns[idx];
	int n = 0;
	if (d.cm_off != SSW_CM_NONE && d.n_items > 0) {
		const uint32_t* w = words + d.cm_off;
		const int n_blk = (d.ref_len + SSW_CM_BLOCK - 1) / SSW_CM_BLOCK;
		int wm = -32768;
		for (int b = lane; b < n_blk; b += 32) wm = max(wm, half_of(w[b], d.half));
#pragma unroll
		for (int off = 16; off >= 1; off >>= 1) wm = max(wm, __shfl_xor_sync(FULL, wm, off));
		const int t1 = max(wm + bd.gapE, 1);
		n = ssw_bound_list(w, d.half, n_blk, d.ref_len, t1 - bd.gapO - 7 * bd.gapE, 0, 0, cand + (int64_t)idx * bd.cap, bd.cap, lane);
	}
	if (lane == 0) cnt[idx] = n > bd.cap ? -1 : n;
}

/* one re-fill item per listed candidate block at off[idx] + k (cm != 0: with one column word each, at that slot of the scratch) */
template <int DUMMY = 0>
__global__ void __launch_bounds__(SSW_RESOLVE_THREADS)
ssw_bound_emit_kernel(const SswAlnDesc* __restrict__ alns, int n_aln, const SswItem* __restrict__ items, const int32_t* __restrict__ cand,
                      int cap, const int32_t* __restrict__ cnt, const int32_t* __restrict__ off, int cm, SswItem* __restrict__ out)
{
	const int lane = threadIdx.x & 31;
	const int idx = (int)blockIdx.x * (SSW_RESOLVE_THREADS / 32) + (threadIdx.x >> 5);
	if (idx >= n_aln) return;
	const SswAlnDesc d = alns[idx];
	const int n = cnt[idx];
	for (int k = lane; k < n; k += 32) {
		const int c0 = cand[(int64_t)idx * cap + k] * SSW_CM_BLOCK;
		SswItem it = ssw_refill_item(d, items, c0, min(c0 + SSW_CM_BLOCK, d.ref_len));
		const int64_t slot = (int64_t)off[idx] + k;
		if (cm) it.cm_off = slot * SSW_CM_BLOCK - it.p0;
		out[slot] = it;
	}
}

/* Stage 1.  Exact words (BOUND false): `best` holds the re-fill record of stage 0's block, one per alignment.  Bounded words
 * (BOUND true): `best` holds the re-fill records of the alignment's C1 candidates at [off1[idx], off1[idx] + cnt1[idx]), folded
 * here in the same order as the item records of ssw_resolve_kernel (blocks are disjoint, so ties go to the first block); the
 * third slot stays dead, and the C2 candidates of the second-best scan go to cand / cnt2 (ssw_bound_list). */
template <bool BOUND = false>
__global__ void __launch_bounds__(SSW_RESOLVE_THREADS)
ssw_resolve_blocks_kernel(const SswAlnDesc* __restrict__ alns, int n_aln,
                          const SswItemBest* __restrict__ best, const uint32_t* __restrict__ blkmax,
                          const SswItem* __restrict__ items, SswFillResult* __restrict__ out,
                          SswItem* __restrict__ refill_items, int32_t* __restrict__ refill_c0,
                          const int32_t* __restrict__ cnt1 = nullptr, const int32_t* __restrict__ off1 = nullptr,
                          SswBound bd = SswBound{0, 0, 0}, int32_t* __restrict__ cand = nullptr, int32_t* __restrict__ cnt2 = nullptr)
{
	constexpr unsigned FULL = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	const int idx = (int)blockIdx.x * (SSW_RESOLVE_THREADS / 32) + (threadIdx.x >> 5);
	if (idx >= n_aln) return;
	const SswAlnDesc d = alns[idx];
	const int h = d.half;

	int sc = 0, pos = 0, row = 0;
	if (BOUND) {
		pos = 0x7fffffff; row = 0x7fffffff;
		const int n1 = cnt1[idx];
		for (int k = lane; k < n1; k += 32) {
			const SswItemBest b = best[off1[idx] + k];
			const int s = b.score[h], p = b.pos[h], rr = b.row[h];
			if (s > 0 && (s > sc || (s == sc && (p < pos || (p == pos && rr < row))))) { sc = s; pos = p; row = rr; }
		}
#pragma unroll
		for (int off = 16; off >= 1; off >>= 1) {
			const int o_sc = __shfl_xor_sync(FULL, sc, off);
			const int o_pos = __shfl_xor_sync(FULL, pos, off), o_row = __shfl_xor_sync(FULL, row, off);
			if (o_sc > sc || (o_sc == sc && (o_pos < pos || (o_pos == pos && o_row < row)))) { sc = o_sc; pos = o_pos; row = o_row; }
		}
	} else {
		const SswItemBest bc = best[idx];
		sc = bc.score[h]; pos = bc.pos[h]; row = bc.row[h];
	}
	if (sc <= 0) { sc = 0; pos = 0; row = 0; }

	SswFillResult r;
	r.score = sc; r.ref = pos; r.read = row < d.read_len - 1 ? row : d.read_len - 1;
	r.score2 = 0; r.ref2 = 0; r.overflow = 0; r.pad_[0] = r.pad_[1] = 0;
	if (sc == 0) { r.ref = d.word ? 0 : -1; r.read = 0; }
	if (sc >= d.limit) { r.overflow = d.word ? 2 : 1; if (!d.word) r.score = 255; }

	int slots[SSW_REFILL_SLOTS] = {-1, -1, -1, -1};     /* block ids; the zone slot: its first column */
	int zone_end = 0, n2 = 0;
	if (sc > 0 && !r.overflow && d.cm_off != SSW_CM_NONE && d.n_items > 0) {
		const int e1 = max(pos - d.mask_len, 0);
		const int e2 = min(pos + d.mask_len, d.ref_len) + (d.word ? 0 : 1);
		if (d.byte_pad > 0 && e2 < d.ref_len) { slots[SSW_REFILL_ZONE] = e2 & ~3; zone_end = min(e2 + 8, d.ref_len); }
		/* every fully allowed block is a candidate (value, block); chunks start at block boundaries, so the blocks of the
		 * pair-task's row are those of its items */
		const uint32_t* bm = blkmax + d.cm_off;
		const int n_blk = (d.ref_len + SSW_CM_BLOCK - 1) / SSW_CM_BLOCK;
		if (BOUND) {
			/* T2 = max L(b) over the fully allowed blocks b whose successor is fully allowed too (the lower bound of a body that
			 * straddles into b + 1 belongs to b + 1), so T2 <= the largest fully allowed block maximum; only v > 0 can win */
			int t2 = 1;
			for (int b = lane; b + 1 < n_blk; b += 32) {
				const int bs = b * SSW_CM_BLOCK, be = min(bs + 2 * SSW_CM_BLOCK, d.ref_len);
				if (be <= e1 || bs >= e2) t2 = max(t2, half_of(bm[b], h) + bd.gapE);
			}
#pragma unroll
			for (int off = 16; off >= 1; off >>= 1) t2 = max(t2, __shfl_xor_sync(FULL, t2, off));
			n2 = ssw_bound_list(bm, h, n_blk, d.ref_len, t2 - bd.gapO - 7 * bd.gapE, e1, e2, cand + (int64_t)idx * bd.cap, bd.cap, lane);
		}
		int vb = 0, bb = 0x7fffffff;
		if (!BOUND)
		for (int b = lane; b < n_blk; b += 32) {
			const int bs = b * SSW_CM_BLOCK, be = min(bs + SSW_CM_BLOCK, d.ref_len);
			if (be <= e1 || bs >= e2) {
				const int v = half_of(bm[b], h);
				if (v > vb) { vb = v; bb = b; }
			}
		}
#pragma unroll
		for (int off = 16; off >= 1; off >>= 1) {
			const int o_vb = __shfl_xor_sync(FULL, vb, off), o_bb = __shfl_xor_sync(FULL, bb, off);
			if (o_vb > vb || (o_vb == vb && o_vb > 0 && o_bb < bb)) { vb = o_vb; bb = o_bb; }
		}
		/* blocks cut by the window edges (e1 > 0 and e2 < ref_len whenever the remainder is non-zero / tested) */
		if (e1 % SSW_CM_BLOCK) slots[0] = e1 / SSW_CM_BLOCK;
		if ((e2 % SSW_CM_BLOCK) && e2 < d.ref_len && e2 / SSW_CM_BLOCK != slots[0]) slots[1] = e2 / SSW_CM_BLOCK;
		if (vb > 0) slots[2] = bb;
	}
	if (lane == 0) out[idx] = r;
	if (BOUND && lane == 0) cnt2[idx] = n2 > bd.cap ? -1 : n2;
	if (lane < SSW_REFILL_SLOTS) {
		const int b = slots[lane];
		const int64_t slot = (int64_t)idx * SSW_REFILL_SLOTS + lane;
		SswItem it;
		if (b < 0) it = ssw_refill_item(d, items, 0, 0);
		else if (lane == SSW_REFILL_ZONE) {
			it = ssw_refill_item(d, items, b, zone_end);
			if (h) it.qb.lp += d.byte_pad; else it.qa.lp += d.byte_pad;
		} else it = ssw_refill_item(d, items, b * SSW_CM_BLOCK, min(b * SSW_CM_BLOCK + SSW_CM_BLOCK, d.ref_len));
		if (b >= 0) it.cm_off = slot * SSW_CM_BLOCK - it.p0;
		refill_items[slot] = it;
		refill_c0[slot] = b >= 0 ? it.p0 : -1;
	}
}

/* stage 2: fold the re-filled ranges (single column maxima) into the second-best candidate of stage 1 */
/* Bounded words: the C2 candidates (block ids cand[idx * cap + k], k < cnt2[idx]; column words at off2[idx] + k of cm2) as well. */
template <int DUMMY = 0>
__global__ void __launch_bounds__(SSW_RESOLVE_THREADS)
ssw_resolve_refill_kernel(const SswAlnDesc* __restrict__ alns, int n_aln, const int32_t* __restrict__ refill_c0,
                          const uint32_t* __restrict__ refill_cm, SswFillResult* __restrict__ out,
                          const int32_t* __restrict__ cand = nullptr, int cap = 0, const int32_t* __restrict__ cnt2 = nullptr,
                          const int32_t* __restrict__ off2 = nullptr, const uint32_t* __restrict__ cm2 = nullptr)
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
	const int n2 = cnt2 ? cnt2[idx] : 0;
	for (int k = 0; k < n2; ++k) {
		const int c0 = cand[(int64_t)idx * cap + k] * SSW_CM_BLOCK, c1 = min(c0 + SSW_CM_BLOCK, d.ref_len);
		const uint32_t* w = cm2 + (int64_t)(off2[idx] + k) * SSW_CM_BLOCK;
		for (int j = lane; c0 + j < c1; j += 32) {
			const int c = c0 + j;
			if (c < e1 || c >= e2) {
				const int v = half_of(w[j], h);
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
