/*
 * ssw_emul.cuh -- lane-literal evaluation of the reference's striped kernels, for the parameter regimes in which
 * their result depends on the SIMD layout itself:
 *   - gapO <= gapE: the lazy-F loop (src/ssw.c:302-315 byte, :509-520 word) exits after its first segment, so F
 *     from the previous lane stops propagating and H differs from the plain affine recurrence (SURVEY A.6);
 *   - word scores that reach the signed 16-bit saturation of _mm_adds_epi16 (ssw.c:483).
 * One warp per alignment; lane l < 16 (byte) / 8 (word) plays SSE lane l, the segment loop is serial, exactly as in
 * sw_sse2_byte (ssw.c:197-386) / sw_sse2_word (:412-588): same profile values, same saturating operations, same
 * lazy-F early exit, same running maximum, overflow stop, early termination and second-best scan.
 * It is a slow path (no chunking is possible: every column depends on the lazy-F outcome of the previous one);
 * none of the BASELINE configurations uses it.
 */
#ifndef SSW_EMUL_CUH
#define SSW_EMUL_CUH

#include "ssw_common.cuh"

#define SSW_EMUL_WARPS 4
#define SSW_EMUL_THREADS (SSW_EMUL_WARPS * 32)

struct SswEmulTask {
	int32_t q_off, q_len, q_rev;   /* query rows: code[q_off + row], or the reversed prefix code[q_off + q_len-1-row] (query
	                                * profiles: q_off counts rows of n scores) */
	int32_t ref_len;               /* columns scanned: [0, ref_len) forward, ref_len-1 .. 0 when dir == 1 */
	int64_t ref_off;               /* offset of reference column 0 in the padded reference array */
	int32_t dir, word, terminate, bias, mask_len, pad_;
	int64_t state_off;             /* int32 words: 4 arrays of segLen*lanes (pvHStore, pvHLoad, pvE, pvHmax) */
	int64_t cm_off;                /* uint16 elements: maxColumn[ref_len], zero-initialised by the host */
};

__global__ void __launch_bounds__(SSW_EMUL_THREADS)
ssw_emul_kernel(const SswEmulTask* __restrict__ tasks, int n_tasks,
                const int8_t* __restrict__ qcodes, const int8_t* __restrict__ refs,
                const int8_t* __restrict__ mat, int n, int gapO, int gapE,
                int32_t* state, uint16_t* cmax, SswFillResult* __restrict__ out)
{
	constexpr unsigned FULL = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	const int ti = (int)blockIdx.x * SSW_EMUL_WARPS + (threadIdx.x >> 5);
	if (ti >= n_tasks) return;
	const SswEmulTask T = tasks[ti];
	const int L = T.word ? 8 : 16;
	const bool act = lane < L;
	const unsigned amask = (1u << L) - 1u;
	const int segLen = (T.q_len + L - 1) / L;
	const int cells = segLen * L;
	int32_t* Hs = state + T.state_off;
	int32_t* Hl = Hs + cells;
	int32_t* E = Hl + cells;
	int32_t* Hm = E + cells;
	uint16_t* cm = cmax + T.cm_off;
	const int8_t* ref = refs + T.ref_off;
	const int8_t* q = qcodes + (mat ? (int64_t)T.q_off : (int64_t)T.q_off * n);   /* mat == nullptr: n-score profile rows */
	for (int i = lane; i < 4 * cells; i += 32) Hs[i] = 0;
	__syncwarp();

	int vMaxScore = 0, vMaxMark = 0;
	int maxv = 0, end_ref = T.word ? 0 : -1;
	bool overflow = false;

	for (int c = 0; c < T.ref_len; ++c) {
		const int i = T.dir == 1 ? T.ref_len - 1 - c : c;
		const int letter = (int)ref[i];
		__syncwarp();                                                   /* the previous column's stores are visible */
		/* vH = last segment of the previous column shifted up one lane (ssw.c:263-264, :470-471) */
		int vH = (act && lane > 0) ? Hs[(segLen - 1) * L + lane - 1] : 0;
		{ int32_t* t = Hl; Hl = Hs; Hs = t; }
		int vF = 0, vMaxCol = 0;
		if (act) {
			for (int s = 0; s < segLen; ++s) {                       /* inner loop, ssw.c:274-299 / :482-506 */
				const int row = s + lane * segLen;
				int p;
				if (row >= T.q_len) p = T.word ? 0 : T.bias;
				else {
					const int qr = T.q_rev ? T.q_len - 1 - row : row;
					const int m = mat ? (int)mat[letter * n + (int)q[qr]] : (int)q[(int64_t)qr * n + letter];
					p = T.word ? m : ((m + T.bias) & 0xff);
				}
				int h;
				if (T.word) { h = vH + p; h = h > 32767 ? 32767 : (h < -32768 ? -32768 : h); }
				else { h = vH + p; h = h > 255 ? 255 : h; h -= T.bias; h = h < 0 ? 0 : h; }
				int e = E[s * L + lane];
				h = max(h, e);
				h = max(h, vF);
				vMaxCol = max(vMaxCol, h);
				Hs[s * L + lane] = h;
				const int hg = max(h - gapO, 0);
				e = max(max(e - gapE, 0), hg);
				E[s * L + lane] = e;
				vF = max(max(vF - gapE, 0), hg);
				vH = Hl[s * L + lane];
			}
		}
		/* lazy-F (ssw.c:302-315 / :509-520) */
		bool done = false;
		for (int k = 0; k < L && !done; ++k) {
			int up = __shfl_up_sync(FULL, vF, 1);
			vF = lane == 0 ? 0 : up;
			for (int s = 0; s < segLen; ++s) {
				int keep = 0;
				if (act) {
					int h = max(Hs[s * L + lane], vF);
					vMaxCol = max(vMaxCol, h);
					Hs[s * L + lane] = h;
					h = max(h - gapO, 0);
					vF = max(vF - gapE, 0);
					keep = vF > h;
				}
				if ((__ballot_sync(FULL, keep) & amask) == 0) { done = true; break; }
			}
		}
		/* running maximum (ssw.c:318-335 / :523-537) */
		vMaxScore = max(vMaxScore, vMaxCol);
		const bool changed = (__ballot_sync(FULL, act && vMaxScore != vMaxMark) & amask) != 0;
		int colmax = act ? vMaxCol : 0;
#pragma unroll
		for (int off = 8; off >= 1; off >>= 1) colmax = max(colmax, __shfl_xor_sync(FULL, colmax, off, 16));
		if (changed) {
			vMaxMark = vMaxScore;
			int temp = act ? vMaxScore : 0;
#pragma unroll
			for (int off = 8; off >= 1; off >>= 1) temp = max(temp, __shfl_xor_sync(FULL, temp, off, 16));
			temp = __shfl_sync(FULL, temp, 0);
			if (temp > maxv) {
				maxv = temp;
				if (!T.word && maxv + T.bias >= 255) { overflow = true; break; }     /* ssw.c:329 */
				end_ref = i;
				if (act) for (int s = 0; s < segLen; ++s) Hm[s * L + lane] = Hs[s * L + lane];
			}
		}
		colmax = __shfl_sync(FULL, colmax, 0);
		if (lane == 0) cm[i] = (uint16_t)colmax;
		if (colmax == T.terminate) break;                               /* ssw.c:339 / :541 */
	}
	__syncwarp();

	/* end position on the query (ssw.c:342-351 / :544-553) */
	int end_read = T.q_len - 1;
	for (int idx = lane; idx < cells; idx += 32)
		if (Hm[idx] == maxv) {
			const int row = idx / L + (idx % L) * segLen;
			if (row < end_read) end_read = row;
		}
#pragma unroll
	for (int off = 16; off >= 1; off >>= 1) end_read = min(end_read, __shfl_xor_sync(FULL, end_read, off));

	/* second best outside the mask window (ssw.c:368-381 / :570-583) */
	int v2 = 0, i2 = 0;
	{
		const int e1 = (end_ref - T.mask_len) > 0 ? (end_ref - T.mask_len) : 0;
		int e2 = (end_ref + T.mask_len) > T.ref_len ? T.ref_len : (end_ref + T.mask_len);
		if (!T.word) e2 += 1;
		for (int cidx = lane; cidx < T.ref_len; cidx += 32) {
			if (cidx < e1 || cidx >= e2) {
				const int v = (int)cm[cidx];
				if (v > v2) { v2 = v; i2 = cidx; }
			}
		}
#pragma unroll
		for (int off = 16; off >= 1; off >>= 1) {
			const int ov = __shfl_xor_sync(FULL, v2, off), oi = __shfl_xor_sync(FULL, i2, off);
			if (ov > v2 || (ov == v2 && ov > 0 && oi < i2)) { v2 = ov; i2 = oi; }
		}
	}
	if (lane == 0) {
		SswFillResult r;
		r.score = overflow ? 255 : maxv; r.ref = end_ref; r.read = end_read;
		r.score2 = v2; r.ref2 = i2; r.overflow = overflow ? 1 : 0; r.pad_[0] = r.pad_[1] = 0;
		out[ti] = r;
	}
}

#endif /* SSW_EMUL_CUH */
