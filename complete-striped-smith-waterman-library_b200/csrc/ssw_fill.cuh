/*
 * ssw_fill.cuh -- the DP matrix fill (replaces the SSE2 loops of sw_sse2_byte,
 * src/ssw.c:258-340, and sw_sse2_word, :464-542, for both the forward pass and
 * the reverse begin-search pass, :919-926).
 *
 * Formulation (SURVEY Appendix A.1/A.3, validated by oracle_fill_gotoh):
 *     X(c,r) = max(0, H(c-1,r-1) + s(c,r), E(c,r))
 *     H(c,r) = max(X(c,r), F(c,r))
 *     E(c+1,r) = max(E(c,r) - gapE, X(c,r) - gapO)
 *     F(c,r+1) = max(F(c,r) - gapE, X(c,r) - gapO)          (gapO > gapE)
 * (block mode computes the same H and F with the gap openings taken from H, as ssw.c does: ssw_cells)
 * in wrap-free signed 16-bit arithmetic, two alignments per register (s16x2
 * DPX instructions: VIADDMNMX.S16x2[.RELU], VIMNMX[3].S16x2, VIADD.16x2).
 * No lazy-F loop exists here: F is carried exactly down the column.
 *
 * Mapping.  A group of G lanes owns one item; lane t owns query rows
 * [t*R, t*R+R).  The group sweeps the reference as a skewed wavefront: in one
 * step lane t works on scan position s - t, so that the three values that
 * cross a lane boundary (bottom H, outgoing F, partial column maximum) are
 * handed down with one __shfl_up each (block mode: H and F only).  Per-letter query profiles (both
 * alignments packed) live in shared memory; reference letters stream from
 * the padded reference array (null letters outside [0, refLen) keep the state
 * at exactly zero, so pipeline fill and drain need no predication).
 *
 * Two kernels share the same cell code:
 *   ssw_fill_kernel         queries of up to G*R rows: one group per item, items = reference chunks
 *   ssw_fill_strips_kernel  longer queries: the rows are cut into strips of 32*R rows; the strips of one
 *                           pair-task run as a software pipeline over the warps of one CTA, each strip
 *                           consuming the bottom row (H, F, partial column maximum) of the strip above it
 *                           from a boundary buffer a few columns behind its producer.
 *
 * Outputs per item: the lexicographic best cell (score, first scan position,
 * smallest row) per half -- not in block mode (CM == 2, 3) -- and, forward pass,
 * the column maxima over real and pad rows (the reference's maxColumn[],
 * ssw.c:338/:540) as packed s16x2 words.  All order-dependent semantics (strict
 * '>' running maximum, byte overflow, mask window) are applied afterwards by
 * ssw_resolve.cuh.
 */
#ifndef SSW_FILL_CUH
#define SSW_FILL_CUH

#include "ssw_common.cuh"

#define SSW_FILL_WARPS 4
#define SSW_FILL_THREADS (SSW_FILL_WARPS * 32)
#ifndef SSW_STRIP_R
#define SSW_STRIP_R 10                      /* rows per lane of the strip kernel: 320 rows per strip */
#endif
#define SSW_STRIP_MAXW 16                   /* warps per CTA of the strip kernel */
#ifndef SSW_FLOOR_PERIOD
#define SSW_FLOOR_PERIOD 1                   /* loop bodies between refreshes of the group floor of the best-cell bookkeeping */
#endif
#define SSW_STRIP_LAG 48                    /* a strip's last lane ends a super-block this many columns before the strip above */
#define SSW_STRIP_SUPER 4096                /* columns per super-block (granularity of early termination) */
#define SSW_STRIP_BPAD 32                   /* words in front of every boundary array (scan positions down to -32) */

/* rows per lane as the profile STORES them: R, or R + 1 when R = 4a + 3 (three tail words per lane cannot be read with one
 * aligned load; such a lane gets a full fourth segment whose last word is never used: R = 19 is stored like 20 rows and
 * computed as 19 -- 300 aa protein queries pad to 304 rows in word mode, ssw.c:393, and 16 lanes x 19 rows fit them exactly) */
template <int R>
struct SswProfRows { static constexpr int S = (R % 4 == 3) ? R + 1 : R; };

/* word offset of row k of lane `lane` inside one letter's profile block (32*S words):
 * S = 4a + rem; the first 4a rows are a uint4 segments [seg][lane], the tail is [lane][rem]. */
template <int R>
__host__ __device__ static __forceinline__ int ssw_prof_slot(int k, int lane)
{
	constexpr int S = SswProfRows<R>::S, A = S / 4, REM = S % 4;
	return k < 4 * A ? (k / 4) * 128 + lane * 4 + (k % 4) : A * 128 + lane * REM + (k - 4 * A);
}

/* Shared-memory reads of the profile.  On the device they are issued as ld.shared from a 32-bit shared
 * address (no generic-address conversion inside the sweep); the emulator build uses plain loads. */
#ifdef SSW_CPU_EMU
typedef const uint32_t* ssw_saddr;
__device__ static __forceinline__ ssw_saddr ssw_sbase(const uint32_t* p) { return p; }
__device__ static __forceinline__ ssw_saddr ssw_sadd(ssw_saddr a, int words) { return a + words; }
__device__ static __forceinline__ uint4 ssw_lds128(ssw_saddr a) { return *reinterpret_cast<const uint4*>(a); }
__device__ static __forceinline__ uint2 ssw_lds64(ssw_saddr a) { return *reinterpret_cast<const uint2*>(a); }
__device__ static __forceinline__ uint32_t ssw_lds32(ssw_saddr a) { return *a; }
#else
typedef uint32_t ssw_saddr;
__device__ static __forceinline__ ssw_saddr ssw_sbase(const uint32_t* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ static __forceinline__ ssw_saddr ssw_sadd(ssw_saddr a, int words) { return a + 4u * (uint32_t)words; }
__device__ static __forceinline__ uint4 ssw_lds128(ssw_saddr a)
{
	uint4 v;
	asm("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
	return v;
}
__device__ static __forceinline__ uint2 ssw_lds64(ssw_saddr a)
{
	uint2 v;
	asm("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
	return v;
}
__device__ static __forceinline__ uint32_t ssw_lds32(ssw_saddr a)
{
	uint32_t v;
	asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
	return v;
}
#endif

/* shared-memory bytes for an alphabet of n letters */
template <int R>
static inline size_t ssw_fill_smem_bytes(int n, int warps = SSW_FILL_WARPS) { return (size_t)warps * (size_t)(n + 1) * 32 * SswProfRows<R>::S * sizeof(uint32_t); }   /* profiles only; the snapshot area (ssw_snap_smem_bytes) comes on top */

/* ---------------------------------------------------------------------------------------------------------- */
/* shared device code                                                                                          */
/* ---------------------------------------------------------------------------------------------------------- */

/* The profile rows of ssw_build_profile from position-specific query profiles (ssw_engine_set_sequences_pssm): `pssm` holds n
 * scores per row, SswQuery.off counts rows, real row r scores pssm[(off + r) * n + letter]; only rows < len are read.  A row is
 * addressed as a 32-bit offset r * n from its query's first row (the host bounds len * n), as codes are in the matrix. */
template <int R>
__device__ static __forceinline__ void ssw_build_profile_pssm(uint32_t* prof, int lane, int row0, const SswQuery& qa, const SswQuery& qb,
                                                             const int8_t* __restrict__ pssm, int n, int letter0, int letter_step)
{
	const int8_t* pa = pssm + (int64_t)qa.off * n;
	const int8_t* pb = pssm + (int64_t)qb.off * n;
	int ca[R], cb[R];
#pragma unroll
	for (int k = 0; k < R; ++k) {
		const int row = row0 + k;
		ca[k] = row < qa.len ? (qa.rev ? qa.len - 1 - row : row) * n : (row < qa.lp ? -1 : -2);
		cb[k] = row < qb.len ? (qb.rev ? qb.len - 1 - row : row) * n : (row < qb.lp ? -1 : -2);
	}
	for (int letter = letter0; letter <= n; letter += letter_step) {
		uint32_t* pl = prof + letter * (32 * SswProfRows<R>::S);
#pragma unroll
		for (int k = 0; k < R; ++k) {
			int a = SSW_NEG16, b = SSW_NEG16;
			if (letter < n) {
				a = ca[k] >= 0 ? (int)pa[ca[k] + letter] : (ca[k] == -1 ? 0 : SSW_NEG16);
				b = cb[k] >= 0 ? (int)pb[cb[k] + letter] : (cb[k] == -1 ? 0 : SSW_NEG16);
			}
			pl[ssw_prof_slot<R>(k, lane)] = pack2(a, b);
		}
	}
}

/* Build the packed profile rows [row0, row0 + R) of this lane for both queries into `prof`
 * (qP_byte / qP_word analogue, ssw.c:163-188 / :388-410): real rows score mat[letter][code], pad rows 0,
 * rows beyond the query's padded length and the null letter n score -32768 (dead: H stays 0).
 * PSSM: the queries are position-specific profiles (ssw_build_profile_pssm; the host passes mat == nullptr).  A template
 * parameter of the kernels, so that their instances for query codes are compiled from the same code as without profiles. */
template <int R, bool PSSM = false>
__device__ static __forceinline__ void ssw_build_profile(uint32_t* prof, int lane, int row0, const SswQuery& qa, const SswQuery& qb,
                                                        const int8_t* __restrict__ qcodes, const int8_t* __restrict__ mat, int n,
                                                        int letter0 = 0, int letter_step = 1)
{
	if constexpr (PSSM) { ssw_build_profile_pssm<R>(prof, lane, row0, qa, qb, qcodes, n, letter0, letter_step); return; }
	int ca[R], cb[R];
#pragma unroll
	for (int k = 0; k < R; ++k) {
		const int row = row0 + k;
		ca[k] = row < qa.len ? (int)qcodes[qa.off + (qa.rev ? qa.len - 1 - row : row)] : (row < qa.lp ? -1 : -2);
		cb[k] = row < qb.len ? (int)qcodes[qb.off + (qb.rev ? qb.len - 1 - row : row)] : (row < qb.lp ? -1 : -2);
	}
	for (int letter = letter0; letter <= n; letter += letter_step) {
		uint32_t* pl = prof + letter * (32 * SswProfRows<R>::S);
#pragma unroll
		for (int k = 0; k < R; ++k) {
			int a = SSW_NEG16, b = SSW_NEG16;
			if (letter < n) {
				a = ca[k] >= 0 ? (int)mat[letter * n + ca[k]] : (ca[k] == -1 ? 0 : SSW_NEG16);
				b = cb[k] >= 0 ? (int)mat[letter * n + cb[k]] : (cb[k] == -1 ? 0 : SSW_NEG16);
			}
			pl[ssw_prof_slot<R>(k, lane)] = pack2(a, b);
		}
	}
}

/* Profile rows of this lane for one reference letter. */
template <int R>
__device__ static __forceinline__ void ssw_load_scores(uint32_t (&s)[R], ssw_saddr pbase, ssw_saddr ptail, int letter)
{
	constexpr int S = SswProfRows<R>::S, A4 = S / 4, REM = S % 4;
	const ssw_saddr pl = ssw_sadd(pbase, letter * (32 * S));
#pragma unroll
	for (int q = 0; q < A4; ++q) {
		const uint4 v = ssw_lds128(ssw_sadd(pl, q * 128));
		s[4 * q] = v.x; s[4 * q + 1] = v.y; s[4 * q + 2] = v.z;
		if (4 * q + 3 < R) s[4 * q + 3] = v.w;               /* S == R + 1: the last stored word is unused */
	}
	if (REM == 1) s[4 * A4] = ssw_lds32(ssw_sadd(ptail, letter * (32 * S)));
	if (REM == 2) {
		const uint2 v = ssw_lds64(ssw_sadd(ptail, letter * (32 * S)));
		s[4 * A4] = v.x; s[4 * A4 + 1] = v.y;
	}
}

/* The R cells of one lane in one column, + 1/2 ALU instruction per cell pair for the column maximum.
 * In: Hd (H of the previous column, shifted down one row), E, scores, and (inH, inF) from the lane above.
 * Out: Hn (H of this column), updated E and Hd, outH/outF/outC for the lane below (outC = maximum of the column
 * over the rows of this lane and of all lanes above it).
 *
 * Two forms of the cell, selected by FROM_H:
 *   false  X = max(Hd + s, E, 0), H = max(X, F), E' = max(E - gapE, X - gapO), F' = max(F - gapE, X - gapO):
 *          VIADDMNMX.RELU, VIADD.16x2, VIADDMNMX x2, VIMNMX -- 4 ALU-pipe instructions + 1 packed add per cell pair
 *   true   H = max(Hd + s, E, F, 0), E' = max(E - gapE, H - gapO), F' = max(F - gapE, H - gapO) (ssw.c's form):
 *          VIADD.16x2 x2, VIMNMX3.RELU, VIADDMNMX x2 -- 3 ALU-pipe instructions + 2 packed adds, which do not issue
 *          on the ALU pipe (DESIGN 4.1, tools/microbench.cu)
 * Both give the same H and F in every cell (so the same outH, outF, outC and column maxima); only E differs, by the term
 * F - gapO, and E never leaves the lane.  With gapO > gapE: H - gapO = max(X - gapO, F - gapO) and F - gapO < F - gapE,
 * so F' is the same; E of the second form also admits a horizontal gap right after a vertical one (F -> E), and any
 * such path has a companion of no lower score that takes the same moves horizontal first, which the first form admits
 * (E -> F through X), so H is the same.  tests/test_cell_form.py checks both forms against the oracle and each other. */
template <int R, bool FROM_H>
__device__ static __forceinline__ void ssw_cells(uint32_t (&Hd)[R], uint32_t (&E)[R], const uint32_t (&s)[R], uint32_t (&Hn)[R],
                                                uint32_t inH, uint32_t inF, uint32_t inC, uint32_t negO, uint32_t negE,
                                                uint32_t& outH, uint32_t& outF, uint32_t& outC, uint32_t& own)
{
	uint32_t F = inF;
#pragma unroll
	for (int k = 0; k < R; ++k) {
		if constexpr (FROM_H) {
			/* The sum goes in as the LAST operand of the three-way maximum: given as the first, ptxas fuses it into a
			 * VIADDMNMX.RELU with E and adds a VIMNMX.RELU for F, which is the first form's ALU count again. */
			const uint32_t T = __vadd2(Hd[k], s[k]);
			Hn[k] = __vimax3_s16x2_relu(E[k], F, T);
			const uint32_t Hg = __vadd2(Hn[k], negO);
			E[k] = __viaddmax_s16x2(E[k], negE, Hg);
			F = __viaddmax_s16x2(F, negE, Hg);
		} else {
			const uint32_t X = __viaddmax_s16x2_relu(Hd[k], s[k], E[k]);
			const uint32_t Xg = __vadd2(X, negO);
			E[k] = __viaddmax_s16x2(E[k], negE, Xg);
			Hn[k] = __vmaxs2(X, F);
			F = __viaddmax_s16x2(F, negE, Xg);
		}
	}
	/* `own`: maximum of the column over this lane's rows (the best-cell bookkeeping compares it with the lane's running
	 * best); outC: the partial column maximum handed down the lanes, own folded with the value from above */
	uint32_t m;
	if (R >= 3) {
		m = __vimax3_s16x2(Hn[0], Hn[1], Hn[2]);
#pragma unroll
		for (int k = 3; k + 1 < R; k += 2) m = __vimax3_s16x2(m, Hn[k], Hn[k + 1]);
		if (((R - 3) & 1) != 0) { own = __vmaxs2(m, Hn[R - 1]); outC = __vmaxs2(own, inC); }
		else { own = m; outC = __vmaxs2(m, inC); }
	} else {
		m = Hn[0];
		if (R == 2) m = __vmaxs2(m, Hn[1]);
		own = m; outC = __vmaxs2(m, inC);
	}
	Hd[0] = inH;
#pragma unroll
	for (int k = 1; k < R; ++k) Hd[k] = Hn[k - 1];
	outH = Hn[R - 1];
	outF = F;
}

/* Running best of one lane, taken over the partial column maxima it sees (its own rows and all rows above).  On a
 * strict increase of either half the lane records the scan position and parks the column's H values of its rows in
 * a per-thread snapshot (local memory: a handful of vector stores).  The row -- the smallest of ITS rows holding the
 * final best value, or a large sentinel when the value came from a lane above, which then records the same position
 * with the real row -- is looked up in the snapshot once, when the item is finished.  This keeps the event cheap:
 * with lenient gap penalties (BLOSUM50 with 3/1) the running maximum grows along the whole matrix and events are
 * frequent. */
#define SSW_NO_ROW 0x3fffffff
struct SswLaneBest {
	uint32_t best;
	int pos0, pos1, row0, row1;
};
/* The snapshot lives in shared memory, [thread][half][group of four rows] as 128-bit words with one word of padding per
 * thread (2Q+1 words: conflict-free 128-bit stores for every Q in use, addresses = one base register + immediates):
 * an event is (R+3)/4 vector stores per half.  With BLOSUM50 and 3/1 gaps, or along the true diagonal of a long read, the
 * running maximum grows with every column and some lane of a warp has an event on almost every step; a snapshot kept in
 * registers makes every event 2R register moves. */
template <int R, bool SMEM = true>
struct SswSnap {
	uint4* base;        /* this thread's slots: (h, q) is base[h * Q + q] */
	static constexpr int Q = (R + 3) / 4;
};
/* Register variant (the strip-pipelined kernel: 10 rows per lane, one CTA per SM whatever its shared memory, so the
 * snapshot's registers cost no occupancy there). */
template <int R>
struct SswSnap<R, false> {
	uint32_t w[2][R];
};
template <int R>
static inline size_t ssw_snap_smem_bytes(int threads) { return (size_t)(2 * ((R + 3) / 4) + 1) * (size_t)threads * sizeof(uint4); }

template <int R>
__device__ static __forceinline__ void ssw_snap_init(SswSnap<R, true>& sn, uint4* area, int tid)
{
	sn.base = area + (size_t)tid * (2 * SswSnap<R, true>::Q + 1);
#pragma unroll
	for (int i = 0; i < 2 * SswSnap<R, true>::Q; ++i) sn.base[i] = make_uint4(0, 0, 0, 0);
}
template <int R>
__device__ static __forceinline__ void ssw_snap_init(SswSnap<R, false>& sn)
{
#ifndef SSW_CPU_EMU
	asm volatile("" : : "l"(&sn) : "memory");       /* as in round 1: lets the compiler keep the snapshot out of the hot registers */
#endif
#pragma unroll
	for (int k = 0; k < R; ++k) { sn.w[0][k] = 0; sn.w[1][k] = 0; }
}

template <int R>
__device__ static __forceinline__ void ssw_snap_store(const SswSnap<R, true>& sn, int h, const uint32_t (&Hn)[R])
{
	constexpr int Q = SswSnap<R, true>::Q;
#pragma unroll
	for (int q = 0; q < Q; ++q)
		sn.base[h * Q + q] = make_uint4(Hn[4 * q], 4 * q + 1 < R ? Hn[4 * q + 1] : 0u, 4 * q + 2 < R ? Hn[4 * q + 2] : 0u, 4 * q + 3 < R ? Hn[4 * q + 3] : 0u);
}
template <int R>
__device__ static __forceinline__ void ssw_snap_store(SswSnap<R, false>& sn, int h, const uint32_t (&Hn)[R])
{
#pragma unroll
	for (int k = 0; k < R; ++k) sn.w[h][k] = Hn[k];
}

template <int R, bool SMEM>
__device__ static __forceinline__ void ssw_track(SswLaneBest& lb, SswSnap<R, SMEM>& sn, uint32_t nb, const uint32_t (&Hn)[R], int sp, int p0, int p1)
{
#ifndef SSW_CPU_EMU
	asm volatile("" : "+r"(sp));                /* keep the range test inside this path */
#endif
	if (sp >= p0 && sp < p1) {
		if (half_of(nb, 0) > half_of(lb.best, 0)) { lb.pos0 = sp; ssw_snap_store<R>(sn, 0, Hn); }
		if (half_of(nb, 1) > half_of(lb.best, 1)) { lb.pos1 = sp; ssw_snap_store<R>(sn, 1, Hn); }
		lb.best = nb;
	}
}

/* a lane whose best was never recorded by an event (position -1) has no row to offer */
__device__ static __forceinline__ void ssw_track_unrecorded(SswLaneBest& lb)
{
	if (lb.pos0 < 0) lb.row0 = SSW_ROW_UNARMED;
	if (lb.pos1 < 0) lb.row1 = SSW_ROW_UNARMED;
}

/* after the sweep: smallest row of this lane that held the lane's best value when it was recorded */
template <int R>
__device__ static __forceinline__ void ssw_track_rows(SswLaneBest& lb, const SswSnap<R, true>& sn, int row_base)
{
	constexpr int Q = SswSnap<R, true>::Q;
	lb.row0 = SSW_NO_ROW; lb.row1 = SSW_NO_ROW;
#pragma unroll
	for (int q = Q - 1; q >= 0; --q) {
		const uint4 a = sn.base[q], b = sn.base[Q + q];
		const uint32_t wa[4] = {a.x, a.y, a.z, a.w}, wb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
		for (int j = 3; j >= 0; --j) {
			if (4 * q + j >= R) continue;
			if (half_of(wa[j], 0) == half_of(lb.best, 0)) lb.row0 = row_base + 4 * q + j;
			if (half_of(wb[j], 1) == half_of(lb.best, 1)) lb.row1 = row_base + 4 * q + j;
		}
	}
}
template <int R>
__device__ static __forceinline__ void ssw_track_rows(SswLaneBest& lb, const SswSnap<R, false>& sn, int row_base)
{
	lb.row0 = SSW_NO_ROW; lb.row1 = SSW_NO_ROW;
#pragma unroll
	for (int k = R - 1; k >= 0; --k) {
		if (half_of(sn.w[0][k], 0) == half_of(lb.best, 0)) lb.row0 = row_base + k;
		if (half_of(sn.w[1][k], 1) == half_of(lb.best, 1)) lb.row1 = row_base + k;
	}
}

/* maximum of `v` (packed s16x2) over the lanes of a group */
template <int G>
__device__ static __forceinline__ uint32_t ssw_group_max(uint32_t v)
{
#pragma unroll
	for (int off = G / 2; off >= 1; off >>= 1) v = __vmaxs2(v, __shfl_xor_sync(0xffffffffu, v, off, G));
	return v;
}

/* Reduce the lanes of a group to one record per half: max score, then first position, then smallest row. */
template <int G>
__device__ static __forceinline__ void ssw_reduce_best(const SswLaneBest& lb, int& sc0, int& p0, int& r0, int& sc1, int& p1, int& r1)
{
	constexpr unsigned FULL = 0xffffffffu;
	sc0 = half_of(lb.best, 0); sc1 = half_of(lb.best, 1);
	p0 = lb.pos0; p1 = lb.pos1; r0 = lb.row0; r1 = lb.row1;
#pragma unroll
	for (int off = G / 2; off >= 1; off >>= 1) {
		const int o_sc0 = __shfl_down_sync(FULL, sc0, off, G), o_p0 = __shfl_down_sync(FULL, p0, off, G), o_r0 = __shfl_down_sync(FULL, r0, off, G);
		const int o_sc1 = __shfl_down_sync(FULL, sc1, off, G), o_p1 = __shfl_down_sync(FULL, p1, off, G), o_r1 = __shfl_down_sync(FULL, r1, off, G);
		if (o_sc0 > sc0 || (o_sc0 == sc0 && (o_p0 < p0 || (o_p0 == p0 && o_r0 < r0)))) { sc0 = o_sc0; p0 = o_p0; r0 = o_r0; }
		if (o_sc1 > sc1 || (o_sc1 == sc1 && (o_p1 < p1 || (o_p1 == p1 && o_r1 < r1)))) { sc1 = o_sc1; p1 = o_p1; r1 = o_r1; }
	}
}

/* ---------------------------------------------------------------------------------------------------------- */
/* single-strip kernel                                                                                          */
/* ---------------------------------------------------------------------------------------------------------- */

#ifndef SSW_FILL_MINB
#define SSW_FILL_MINB 4                     /* minimum resident CTAs per SM asked of ptxas: 128 registers, 16 warps per SM */
#endif
/* CM: what the forward pass records of the column maxima (the reference's maxColumn[], ssw.c:338/:540)
 *   0  nothing (reverse pass)
 *   1  every column: one packed word per reference column (short references, the re-fill items of mode 2)
 *   2  one packed word per block of SSW_CM_BLOCK columns, and no best cell (`bests` is not written).  The best cell needs
 *      single columns only in the first block holding the largest block maximum, the second-best scan (ssw.c:368-381) only
 *      in the <= 2 blocks cut by the mask window and in the block that holds the winner; ssw_resolve.cuh re-fills those
 *      blocks per alignment with mode 1.  Chunks start at multiples of SSW_CM_BLOCK, and so does every item's sweep
 *      (p0 - warm: the planner rounds the warm-up up to a multiple of SSW_CM_BLOCK).
 *   3  as 2, but the word of a block is w(b), the largest row maximum of E sampled once per loop body over the block, which
 *      brackets the block maximum M(b): w + gapE <= M <= w + gapO + 7 gapE (DESIGN 2; the lower bound of a body that straddles
 *      a block boundary belongs to the later block).  ssw_resolve.cuh re-fills only the blocks the bracket cannot rule out. */
/* WARPS: warps per CTA.  4 by default; 8 where one CTA-shared profile is so large (protein alphabets: 64 KB at 20 rows per
 * lane) that four-warp CTAs would leave the SM with 8 resident warps -- eight warps per profile keep 16. */
/* ARM: items may carry a late arming position (SswItem.cend, device-planned grids); a template parameter so that the kernels
 * that never use it do not pay for the extra predicate per step. */
template <int G, int R, int DIR, int CM, bool TERM, int WARPS = SSW_FILL_WARPS, bool ARM = false, bool PSSM = false>
__global__ void __launch_bounds__(WARPS * 32, WARPS == SSW_FILL_WARPS ? SSW_FILL_MINB : 2)
ssw_fill_kernel(const SswItem* __restrict__ items, int n_items,
                const int8_t* __restrict__ qcodes, const int8_t* __restrict__ refs,
                const int8_t* __restrict__ mat, int n, int gapO, int gapE,
                uint32_t* __restrict__ colmax, SswItemBest* __restrict__ bests, int share)
{
	static_assert(G == 8 || G == 16 || G == 32, "group width");
	static_assert(R >= 1 && R <= 20, "rows per lane");
	static_assert(!TERM || G == 32, "early termination is per warp");
	constexpr int GPW = 32 / G;                 /* groups per warp */
	constexpr int S = SswProfRows<R>::S;        /* rows per lane as stored in the profile */
	constexpr int A4 = S / 4, REM = S % 4;
	constexpr unsigned FULL = 0xffffffffu;

	SSW_DYN_SMEM(uint32_t, smem);
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int g = lane / G, t = lane % G;
	/* share != 0: the host guarantees that all items of this CTA have the same two queries, so one profile serves
	 * every warp (built cooperatively); otherwise each warp keeps the profile(s) of its own groups */
	uint32_t* prof = share ? smem : smem + (size_t)warp * (size_t)(n + 1) * 32 * S;

	const int nwarps = (int)(blockDim.x >> 5);           /* SSW_FILL_WARPS, fewer when per-warp profiles are large */
	const int item_idx = ((int)blockIdx.x * nwarps + warp) * GPW + g;
	const bool live = item_idx < n_items;
	SswItem it;
	if (live) it = items[item_idx];
	else {
		it.qa.off = it.qb.off = 0; it.qa.len = it.qb.len = 0; it.qa.lp = it.qb.lp = 0; it.qa.rev = it.qb.rev = 0;
		it.ref_off = SSW_REF_PAD; it.ref_len = 0; it.cend = 0; it.p0 = it.p1 = 0; it.warm = 0; it.term_a = -1; it.cm_off = SSW_CM_NONE;
	}

	if (share) {
		const SswItem& first = items[(int)blockIdx.x * nwarps * GPW];               /* always a live item */
		ssw_build_profile<R, PSSM>(prof, lane, t * R, first.qa, first.qb, qcodes, mat, n, warp, nwarps);
		__syncthreads();
	} else {
		ssw_build_profile<R, PSSM>(prof, lane, t * R, it.qa, it.qb, qcodes, mat, n);
		__syncwarp();
	}

	/* ---- sweep ---- */
	const uint8_t* rp = reinterpret_cast<const uint8_t*>(refs) + it.ref_off;   /* reference column 0 */
	const uint32_t negO = pack2(-gapO, -gapO), negE = pack2(-gapE, -gapE);
	constexpr bool BLK = CM == 2 || CM == 3;            /* block mode: one word per SSW_CM_BLOCK columns */
	int sL = (it.p0 - it.warm - (G - 1)) & (BLK ? ~7 : ~3);   /* scan position of the group's last lane, multiple of 4 (block mode: of 8) */
	constexpr int U = 8;                                /* scan positions per loop body */
	/* block mode sweeps on to the end of the last block, so that its last lane finishes that block inside the loop (the
	 * columns behind the reference leave the block maximum as it is, see the block fold below) */
	const int p_end = BLK ? (it.p1 + SSW_CM_BLOCK - 1) & ~(SSW_CM_BLOCK - 1) : it.p1;
	int n_body = live && it.p1 > sL ? (p_end - sL + U - 1) / U : 0;
	/* the longest group's count, in a uniform register (REDUX): the loop branch is then uniform, and ptxas issues the
	 * shuffles of the step without the per-step WARPSYNC.COLLECTIVE guards and register copies of a loop it cannot
	 * prove warp-uniform (about 120 instructions per loop body of the (8,19) instance).  The emulator build takes the
	 * same maximum with a shuffle butterfly. */
#ifdef SSW_CPU_EMU
	for (int off = G; off < 32; off <<= 1) n_body = max(n_body, __shfl_xor_sync(FULL, n_body, off));
#else
	n_body = __reduce_max_sync(FULL, n_body);
#endif

	/* column cursor of this lane for step j = 0 of the current body, clamped into the padded array */
	int col = DIR > 0 ? sL + (G - 1 - t) : it.cend - (sL + (G - 1 - t));
	const int col_hi = it.ref_len + SSW_REF_PAD - U, col_lo = -SSW_REF_PAD + U - 1;
	if (DIR > 0) col = min(col, col_hi); else col = max(col, col_lo);
	int sp0 = sL + (G - 1 - t);                         /* this lane's scan position at step j = 0 */

	/* per-lane shared-memory cursors: rows 0..4*A4-1 as uint4 segments, the tail behind them */
	const ssw_saddr pbase = ssw_sadd(ssw_sbase(prof), lane * 4);
	const ssw_saddr ptail = ssw_sadd(ssw_sbase(prof), A4 * 128 + lane * REM);
	/* Lane 0 of a group takes zeros from above (multiplied in: FMA pipe).  The 0/1 is fetched from the lane before with a
	 * shuffle, which ptxas keeps in a register; derived from the thread index, ptxas rebuilds it inside the loop (S2R, LOP3,
	 * ISETP, SEL).  Being opaque to the compiler, it also keeps the masking a multiply. */
	const uint32_t top_keep = __shfl_sync(FULL, t == G - 1 ? 0u : 1u, t + G - 1, G);
	const uint8_t* lptr = rp + col;                     /* letter cursor, advanced together with col */

	uint32_t Hd[R], E[R];
#pragma unroll
	for (int k = 0; k < R; ++k) { Hd[k] = 0; E[k] = 0; }
	uint32_t outH = 0, outF = 0, outC = 0;
	/* Block mode keeps no best cell: the resolve takes the score and the first block holding it from the block maxima and
	 * re-fills that one block with tracking (ssw_resolve.cuh).  So its sweep carries only the recurrence and the maxima. */
	constexpr bool TRACK = !BLK;
	/* Block mode computes the cells in the form with 3 ALU-pipe instructions per cell pair (ssw_cells); the other instances
	 * keep the 4-instruction form, since the 3-instruction form has been timed only in block mode (configs 2 and 3). */
	constexpr bool FROM_H = BLK;
	SswLaneBest lb;
	lb.best = 0; lb.pos0 = lb.pos1 = -1; lb.row0 = lb.row1 = 0;      /* position -1: no recorded event (yet) */
	SswSnap<R> snap;
	if constexpr (TRACK)
		ssw_snap_init<R>(snap, reinterpret_cast<uint4*>(smem + (size_t)(share ? 1 : nwarps) * (size_t)(n + 1) * 32 * S), (int)threadIdx.x);
	/* block mode: this lane's maximum (CM == 3: of its E samples, starting below every sample) of its current block, and of
	 * its last finished one */
	uint32_t blk_acc = CM == 3 ? 0x80008000u : 0u, blk_done = 0;

	for (int body = 0; body < n_body; ++body) {
		uint32_t cmv[U];                                /* per step: outC, or with CM == 2 the maximum over this lane's own rows */
		if (TRACK && (body & (SSW_FLOOR_PERIOD - 1)) == 0) {
			/* lower bound of the group's final maximum: a lane value below it can never be the best cell, so the lane's
			 * running best is raised to (bound - 1) and such values no longer trigger the bookkeeping */
			const uint32_t floor2 = ssw_group_max<G>(lb.best);
			lb.best = __vmaxs2(lb.best, __vadd2(floor2, 0xffffffffu));
		}
		const bool maybe_counted = sp0 + U - 1 >= it.p0 && sp0 < it.p1;   /* this body touches the counted range */
		/* Late arming (DIR > 0, items without warm-up): before scan position `arm` only the VALUE of the running best is kept --
		 * no position, no snapshot, no branch.  If the item's maximum turns out to lie there (its position stays -1) the
		 * resolve step flags the pair and it is re-done with arm 0.  Protein grids: the running maximum grows on every
		 * column, the best cell lies in the last third of the reference for 99.99 % of the pairs (DESIGN 4.1). */
		const bool unarmed = ARM && DIR > 0 && sp0 + U - 1 < it.cend;
#pragma unroll
		for (int j = 0; j < U; ++j) {
			/* values crossing the lane boundary */
			const uint32_t inH = __shfl_up_sync(FULL, outH, 1, G) * top_keep;
			const uint32_t inF = __shfl_up_sync(FULL, outF, 1, G) * top_keep;
			const uint32_t inC = BLK ? 0u : __shfl_up_sync(FULL, outC, 1, G) * top_keep;   /* block mode: outC unused */

			/* reference letter of this lane's scan position and its profile rows */
			int letter = (int)lptr[DIR * j];
			if (DIR < 0) { if (sp0 + j < 0) letter = n; }
			uint32_t s[R], Hn[R];
			ssw_load_scores<R>(s, pbase, ptail, letter);
			uint32_t own;
			ssw_cells<R, FROM_H>(Hd, E, s, Hn, inH, inF, inC, negO, negE, outH, outF, outC, own);
			cmv[j] = CM == 2 ? own : outC;

			/* running best of this lane's rows (strict increase only; rare path) */
			if constexpr (TRACK) {
				const uint32_t nb = __vmaxs2(lb.best, own);
				if (unarmed) lb.best = nb;
				else if (nb != lb.best && maybe_counted) {
					if (ARM && DIR > 0 && sp0 + j < it.cend) lb.best = nb;   /* the body that crosses `arm`: still before it */
					else ssw_track<R>(lb, snap, nb, Hn, sp0 + j, it.p0, it.p1);
				}
			}
		}

		if (CM == 1) {
			if (t == G - 1 && it.cm_off != SSW_CM_NONE) {
#pragma unroll
				for (int q = 0; q < U; q += 4)
					if (sL + q >= it.p0 && sL + q < it.p1)
						*reinterpret_cast<uint4*>(colmax + it.cm_off + sL + q) = make_uint4(cmv[q], cmv[q + 1], cmv[q + 2], cmv[q + 3]);
			}
		}
		if (CM == 2) {
			/* Block maxima per lane.  A block maximum is the maximum over all cells of the block, so every lane keeps its own
			 * over the cells of its rows, and the group combines the lanes once per block: no column maximum travels down the
			 * lanes.  The planner starts every block-mode item at a multiple of SSW_CM_BLOCK (p0 - warm), so sL = p0 - warm - G
			 * at body 0 and lane t is at column 8 * body + j - 1 - t (mod 64) in step j: its next block starts at step
			 * js = t + 1 - 8 * (body mod 8) of a body with body mod 8 < G / 8 (js = 8: right after it), and the last lane
			 * finishes a block at the end of the body with body mod 8 = G / 8 - 1, when every lane of the group has finished
			 * it (a lane is at most G - 1 <= 31 columns ahead, so it holds at most one finished block).  These tests are on
			 * `body`, which is warp-uniform: the bodies between carry no per-step predicate.  The columns behind the reference
			 * are folded in as well: there the null letters leave X = max(0, E) with E(c) <= H(c-1) of the same row, and F
			 * only carries X down, so such a column's maximum never exceeds that of the column before it, and the block
			 * maximum stays the same.  Columns before p0 or of the next chunk end up only in blocks that are not stored. */
			constexpr int BODIES = SSW_CM_BLOCK / U;            /* loop bodies per block */
			const int bm = body % BODIES;
			if (bm < G / U) {
				const int js = t + 1 - U * bm;
				uint32_t lo = blk_acc, hi = 0;
#pragma unroll
				for (int j = 0; j < U; ++j) {
					if (j < js) lo = __vmaxs2(lo, cmv[j]);
					else hi = __vmaxs2(hi, cmv[j]);
				}
				if (js >= 1 && js <= U) { blk_done = lo; blk_acc = hi; }
				else blk_acc = __vmaxs2(lo, hi);
				if (bm == G / U - 1) {
					const uint32_t v = ssw_group_max<G>(blk_done);
					const int c0 = sL + U - SSW_CM_BLOCK;       /* first column of the block just finished */
					if (t == 0 && it.cm_off != SSW_CM_NONE && c0 >= it.p0 && c0 < it.p1) colmax[it.cm_off + c0 / SSW_CM_BLOCK] = v;
				}
			} else {
				blk_acc = __vimax3_s16x2(blk_acc, cmv[0], cmv[1]);
				blk_acc = __vimax3_s16x2(blk_acc, cmv[2], cmv[3]);
				blk_acc = __vimax3_s16x2(blk_acc, cmv[4], cmv[5]);
				blk_acc = __vimax3_s16x2(blk_acc, cmv[6], cmv[7]);
			}
		}
		if (CM == 3) {
			/* Bounded block words (DESIGN 2): no per-step maximum at all.  After step 7 E holds E(r, c + 1) of this lane's last
			 * column c of the body, and in every row H(r, c') <= E(r, c + 1) + gapO + (c - c') gapE for the body's columns c',
			 * while E(r, c + 1) <= H(r, c) - gapE.  So the maximum of E over the lane's rows, once per body, bounds the maxima
			 * of the body's columns from above (+ gapO + 7 gapE) and the maximum of column c from below (+ gapE).  A body
			 * that straddles a block boundary (step js in 1..7) is credited to both blocks: the upper bound holds for both, the
			 * lower one for the later block only, which the resolve accounts for. */
			uint32_t e;
			if (R >= 3) {
				e = __vimax3_s16x2(E[0], E[1], E[2]);
#pragma unroll
				for (int k = 3; k + 1 < R; k += 2) e = __vimax3_s16x2(e, E[k], E[k + 1]);
				if (((R - 3) & 1) != 0) e = __vmaxs2(e, E[R - 1]);
			} else e = R == 2 ? __vmaxs2(E[0], E[1]) : E[0];
			constexpr int BODIES = SSW_CM_BLOCK / U;
			const int bm = body % BODIES;
			if (bm < G / U) {
				const int js = t + 1 - U * bm;
				if (js >= 1 && js <= U) { blk_done = __vmaxs2(blk_acc, e); blk_acc = js < U ? e : 0x80008000u; }
				else blk_acc = __vmaxs2(blk_acc, e);
				if (bm == G / U - 1) {
					const uint32_t v = ssw_group_max<G>(blk_done);
					const int c0 = sL + U - SSW_CM_BLOCK;
					if (t == 0 && it.cm_off != SSW_CM_NONE && c0 >= it.p0 && c0 < it.p1) colmax[it.cm_off + c0 / SSW_CM_BLOCK] = v;
				}
			} else blk_acc = __vmaxs2(blk_acc, e);
		}
		if (TERM) {
			/* reverse pass: stop after the first column whose maximum equals score1 (ssw.c:339/:541) */
			int hit = 0;
			if (t == G - 1 && it.term_a >= 0) {
#pragma unroll
				for (int j = 0; j < U; ++j)
					if (sL + j >= it.p0 && sL + j < it.p1 && half_of(cmv[j], 0) == it.term_a) hit = 1;
			}
			if (__any_sync(FULL, hit)) break;
		}

		sL += U;
		sp0 += U;
		{
			const int ncol = DIR > 0 ? min(col + U, col_hi) : max(col - U, col_lo);
			lptr += ncol - col;
			col = ncol;
		}
	}

	if constexpr (TRACK) {
		ssw_track_rows<R>(lb, snap, t * R);
		ssw_track_unrecorded(lb);
		int sc0, bp0, br0, sc1, bp1, br1;
		ssw_reduce_best<G>(lb, sc0, bp0, br0, sc1, bp1, br1);
		if (live && t == 0) {
			SswItemBest b;
			b.score[0] = sc0; b.pos[0] = bp0; b.row[0] = br0;
			b.score[1] = sc1; b.pos[1] = bp1; b.row[1] = br1;
			b.p0 = it.p0; b.p1 = it.p1;
			bests[item_idx] = b;
		}
	}
}

/* ---------------------------------------------------------------------------------------------------------- */
/* strip-pipelined kernel for queries longer than one strip                                                     */
/* ---------------------------------------------------------------------------------------------------------- */

/*
 * One CTA per pair-task, NW = blockDim.x/32 warps.  Strip s = rows [s*32R, (s+1)*32R) is processed by warp
 * s % NW.  Work is cut into n_super super-blocks of SSW_STRIP_SUPER columns; inside a super-block the strips
 * run as a pipeline: for every column strip s takes the bottom row of strip s-1 (H, F, partial column maximum)
 * from that strip's boundary arrays and publishes its own.  prog[s] (shared memory) is the number of columns
 * strip s has published.  Strip s's last lane ends a super-block SSW_STRIP_LAG*s columns before the block's
 * end, so everything it needs from strip s-1 (40 columns ahead of its last lane) has been published; between
 * super-blocks a strip's lane registers are parked in global memory.  Tasks depend only on lexicographically
 * smaller (super-block, strip) tasks and every warp runs its tasks in that order, so the spin-waits cannot
 * dead-lock.  The reverse pass raises a CTA-wide stop flag when the last strip meets the terminate score;
 * at most about one super-block is computed in vain.  Every (strip, super-block) writes its own
 * SswItemBest record (zeroed by the host beforehand); the resolve kernel reduces them.
 */
struct SswStripTask {
	SswQuery qa, qb;
	int64_t ref_off;
	int32_t ref_len, cend;
	int32_t p1;            /* scan range [0, p1) */
	int32_t term_a;        /* reverse pass: terminate score, else -1 */
	int32_t n_strips, n_super;
	int64_t cm_off;        /* column maxima written by the last strip (forward pass), SSW_CM_NONE: none */
	int64_t bnd_off;       /* boundary arrays: 2 (strip parity) x 3 (H, F, C) x bnd_len words */
	int32_t bnd_len;       /* words per boundary array: multiple of 4, >= p1 + 2*SSW_STRIP_BPAD + 8 */
	int32_t first_best;    /* record of (strip s, super-block b) = first_best + s * n_super + b */
	int64_t park_off;      /* parked lane registers: n_strips x 32 lanes x (2R + 3) words */
	int32_t super;         /* columns per super-block (multiple of 8) */
	int32_t term_b;        /* reverse pass, half B: terminate score, else -1 */
	/* reverse pass: the two alignments of a task are unrelated (own reference window, own end column), so half B has
	 * its own letter stream; p1 above is the larger of the two scan ranges */
	int64_t ref_off_b;
	int32_t cend_b, p1_b;
	int32_t p1_a, pad_;
};

#ifdef SSW_CPU_EMU
template <class T> __device__ static __forceinline__ T ssw_ldcg(const T* p) { return *p; }
#else
template <class T> __device__ static __forceinline__ T ssw_ldcg(const T* p) { return __ldcg(p); }
#endif

/* progress word shared by two CTAs: release store by the producer, acquire load by the consumer (device scope) */
#ifdef SSW_CPU_EMU
__device__ static __forceinline__ int ssw_ld_acquire(const volatile int* p) { return *p; }
__device__ static __forceinline__ void ssw_st_release(volatile int* p, int v) { *p = v; }
#else
__device__ static __forceinline__ int ssw_ld_acquire(const volatile int* p)
{
	int v;
	asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}
__device__ static __forceinline__ void ssw_st_release(volatile int* p, int v)
{
	asm volatile("st.release.gpu.global.s32 [%0], %1;" : : "l"(p), "r"(v) : "memory");
}
#endif

template <int R, int DIR, bool TERM, bool SPLIT, bool PSSM = false>
__global__ void __launch_bounds__(SSW_STRIP_MAXW * 32)
ssw_fill_strips_kernel(const SswStripTask* __restrict__ tasks,
                       const int8_t* __restrict__ qcodes, const int8_t* __restrict__ refs,
                       const int8_t* __restrict__ mat, int n, int gapO, int gapE,
                       uint32_t* __restrict__ colmax, uint32_t* bnd, uint32_t* park,
                       SswItemBest* __restrict__ bests, int parts, int* gsync)
{
	constexpr int A4 = R / 4, REM = R % 4;
	constexpr unsigned FULL = 0xffffffffu;
	constexpr int PARK = 2 * R + 3;
	static_assert(R % 4 != 3, "rows per lane");

	SSW_DYN_SMEM(uint32_t, smem);
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, NW = blockDim.x >> 5;
	/* parts > 1 (forward only): the strips of one task are split into `parts` contiguous blocks, one CTA each; the first
	 * strip of a block follows the last strip of the previous block through a progress word in global memory.  Work is
	 * handed out by a ticket, so the CTA a block waits for has always started (lower ticket): no dead-lock whatever the
	 * order in which the hardware starts CTAs. */
	int unit = (int)blockIdx.x;
	if (SPLIT) {
		__shared__ int s_ticket;
		if (threadIdx.x == 0) s_ticket = atomicAdd(gsync, 1);
		__syncthreads();
		unit = s_ticket;
	}
	const int part = SPLIT ? unit % parts : 0;
	const SswStripTask T = tasks[SPLIT ? unit / parts : unit];
	const int per_part = SPLIT ? (T.n_strips + parts - 1) / parts : T.n_strips;
	const int s_first = part * per_part, s_last = min(T.n_strips, s_first + per_part);      /* this CTA's strips [s_first, s_last) */
	volatile int* gprog_in = gsync + 1 + (SPLIT ? unit - 1 : 0);          /* published by the previous block of the same task */
	volatile int* gprog_out = gsync + 1 + (SPLIT ? unit : 0);
	/* shared memory: NW profiles, then prog[n_strips], the stop flag and the done bits */
	uint32_t* prof = smem + (size_t)warp * (size_t)(n + 1) * 32 * R;
	volatile int* prog = reinterpret_cast<volatile int*>(smem + (size_t)NW * (size_t)(n + 1) * 32 * R);
	volatile int* stop = prog + T.n_strips;                /* 1: every requested half has met its score (reverse pass) */
	volatile int* done = stop + 1;                          /* bit h: half h has met its score */
	const int need_mask = (T.term_a >= 0 ? 1 : 0) | (T.term_b >= 0 ? 2 : 0);
	for (int i = threadIdx.x; i < T.n_strips; i += blockDim.x) prog[i] = -0x40000000;
	if (threadIdx.x == 0) { *stop = 0; *done = 0; }
	__syncthreads();

	const uint8_t* rp = reinterpret_cast<const uint8_t*>(refs) + T.ref_off;
	const uint8_t* rpB = reinterpret_cast<const uint8_t*>(refs) + (DIR < 0 ? T.ref_off_b : T.ref_off);
	const uint32_t negO = pack2(-gapO, -gapO), negE = pack2(-gapE, -gapE);
	const int col_hi = T.ref_len + SSW_REF_PAD - 8, col_lo = -SSW_REF_PAD + 7;
	const ssw_saddr pbase = ssw_sadd(ssw_sbase(prof), lane * 4);
	const ssw_saddr ptail = ssw_sadd(ssw_sbase(prof), A4 * 128 + lane * REM);
	const int start = -32;                               /* first last-lane position: lane 0 starts at -1 */
	const int end = (T.p1 + 7) & ~7;                     /* last-lane positions run over [start, end) */

	for (int sb = 0; sb < T.n_super; ++sb) {
		for (int s = s_first + warp; s < s_last; s += NW) {
			/* last-lane range [lo, hi) of this strip in this super-block */
			const int lag = s * SSW_STRIP_LAG;
			int lo = sb == 0 ? start : max(start, min(end, sb * T.super - lag));
			int hi = sb == T.n_super - 1 ? end : max(start, min(end, (sb + 1) * T.super - lag));
			if (hi <= lo) continue;
			if (TERM) { int st = lane == 0 ? *stop : 0; st = __shfl_sync(FULL, st, 0); if (st) break; }

			ssw_build_profile<R, PSSM>(prof, lane, s * 32 * R + lane * R, T.qa, T.qb, qcodes, mat, n);
			__syncwarp();

			/* lane registers: fresh at the strip's first column, else un-parked */
			uint32_t Hd[R], E[R], outH, outF, outC;
			uint32_t* pk = park + T.park_off + ((size_t)s * 32 + lane) * PARK;
			if (lo == start) {
#pragma unroll
				for (int k = 0; k < R; ++k) { Hd[k] = 0; E[k] = 0; }
				outH = outF = outC = 0;
			} else {
#pragma unroll
				for (int k = 0; k < R; ++k) { Hd[k] = pk[k]; E[k] = pk[R + k]; }
				outH = pk[2 * R]; outF = pk[2 * R + 1]; outC = pk[2 * R + 2];
			}
			SswLaneBest lb;
			lb.best = 0; lb.pos0 = lb.pos1 = -1; lb.row0 = lb.row1 = 0;
			SswSnap<R, false> snap;
			ssw_snap_init<R>(snap);

			const uint32_t* bin = bnd + T.bnd_off + (size_t)((s + 1) & 1) * 3 * T.bnd_len + SSW_STRIP_BPAD;   /* written by strip s-1 */
			uint32_t* bout = bnd + T.bnd_off + (size_t)(s & 1) * 3 * T.bnd_len + SSW_STRIP_BPAD;
			int sL = lo;
			int sp0 = sL + (31 - lane);
			int col = DIR > 0 ? sp0 : T.cend - sp0;
			if (DIR > 0) col = min(col, col_hi); else col = max(col, col_lo);
			const uint8_t* lptr = rp + col;
			int colB = DIR < 0 ? max(T.cend_b - sp0, col_lo) : 0;      /* reverse pass: half B's own letter cursor */
			const uint8_t* lptrB = rpB + colB;
			bool stopped = false;
			int known = -0x40000000, ahead = -0x40000000;       /* progress of the producing CTA as last read (s == s_first only) */
			uint32_t top_keep = lane == 0 ? 0u : 1u;
#ifndef SSW_CPU_EMU
			asm volatile("" : "+r"(top_keep) : : "memory");     /* opaque 0/1 so that the masking stays a multiply */
#endif

			/* lane 0 is at scan position sL+31 .. sL+34 during a body: the last word of the aligned group at
			 * sL+28 (carried from the previous body) and the first three of the group at sL+32 */
			uint32_t cH = 0, cF = 0, cC = 0;
			if (s > 0 && lane == 0 && sL + 28 >= 0) {
				cH = ssw_ldcg(bin + sL + 31); cF = ssw_ldcg(bin + T.bnd_len + sL + 31); cC = ssw_ldcg(bin + 2 * T.bnd_len + sL + 31);
			}

			/* one loop body = 8 scan positions in two halves of 4: the wait for the producer, the stop-flag poll, the
			 * progress word and the cursor updates are paid once per body, the boundary groups (4 words per array) are
			 * loaded and stored per half */
			for (; sL < hi; sL += 8) {
				uint4 gH[2], gF[2], gC[2];
				gH[0] = gH[1] = gF[0] = gF[1] = gC[0] = gC[1] = make_uint4(0, 0, 0, 0);
				int st = 0;                                  /* the stop flag as lane 0 saw it (warp-uniform after the broadcast) */
				if (lane == 0) {
					if (s > 0) {
						const int need = min(sL + 40, end);
						if (SPLIT && s == s_first) {
							/* producer is another CTA: its progress word is read one loop body ahead of the need (the load
							 * of the previous body has landed by now), so the wait loop is only entered when this strip has
							 * really caught up with its producer */
							known = max(known, ahead);
							while (known < need) { SSW_SPIN_PAUSE(); known = ssw_ld_acquire(gprog_in); }
							ahead = known < need + 160 ? ssw_ld_acquire(gprog_in) : known;
						} else {
							while (prog[s - 1] < need && !(st = *stop)) { SSW_SPIN_PAUSE(); }
							__threadfence_block();
						}
#pragma unroll
						for (int h = 0; h < 2; ++h) {
							gH[h] = ssw_ldcg(reinterpret_cast<const uint4*>(bin + sL + 32 + 4 * h));
							gF[h] = ssw_ldcg(reinterpret_cast<const uint4*>(bin + T.bnd_len + sL + 32 + 4 * h));
							gC[h] = ssw_ldcg(reinterpret_cast<const uint4*>(bin + 2 * T.bnd_len + sL + 32 + 4 * h));
						}
					}
					if (TERM) st = *stop;
				}
				st = __shfl_sync(FULL, st, 0);
				if (TERM) { if (st) { stopped = true; break; } }
				const bool maybe_counted = sp0 + 7 >= 0 && sp0 < T.p1;
				int hit = 0;
#pragma unroll
				for (int h = 0; h < 2; ++h) {
					const uint32_t bHv[4] = {cH, gH[h].x, gH[h].y, gH[h].z}, bFv[4] = {cF, gF[h].x, gF[h].y, gF[h].z}, bCv[4] = {cC, gC[h].x, gC[h].y, gC[h].z};
					cH = gH[h].w; cF = gF[h].w; cC = gC[h].w;
					uint32_t cmv[4], hv[4], fv[4];
#pragma unroll
					for (int j = 0; j < 4; ++j) {
						/* lane 0 takes the boundary words (zero in the other lanes) instead of the shuffled ones: a multiply-add
						 * by 0/1 on the FMA pipe rather than a select on the ALU pipe, which is the busy one */
						const uint32_t inH = __shfl_up_sync(FULL, outH, 1) * top_keep + bHv[j];
						const uint32_t inF = __shfl_up_sync(FULL, outF, 1) * top_keep + bFv[j];
						const uint32_t inC = __shfl_up_sync(FULL, outC, 1) * top_keep + bCv[j];
						int letter = (int)lptr[DIR * (4 * h + j)];
						if (DIR < 0) { if (sp0 + 4 * h + j < 0) letter = n; }   /* right of cend; forward scans start inside the null pad */
						uint32_t sc[R], Hn[R];
						ssw_load_scores<R>(sc, pbase, ptail, letter);
						if (DIR < 0) {
							/* half B reads its own reference: its scores come from the profile row of its own letter */
							int letterB = (int)lptrB[-(4 * h + j)];
							if (sp0 + 4 * h + j < 0) letterB = n;
							uint32_t sb[R];
							ssw_load_scores<R>(sb, pbase, ptail, letterB);
#pragma unroll
							for (int k = 0; k < R; ++k) sc[k] = (sc[k] & 0x0000ffffu) | (sb[k] & 0xffff0000u);
						}
						uint32_t own;
						ssw_cells<R, false>(Hd, E, sc, Hn, inH, inF, inC, negO, negE, outH, outF, outC, own);
						cmv[j] = outC; hv[j] = outH; fv[j] = outF;
						const uint32_t nb = __vmaxs2(lb.best, own);
						if (nb != lb.best && maybe_counted) ssw_track<R>(lb, snap, nb, Hn, sp0 + 4 * h + j, 0, T.p1);
					}
					/* the last lane stores the strip's bottom row (the last strip: the column maxima) */
					const int g = sL + 4 * h;
					if (lane == 31 && g >= 0) {
						if (s + 1 < T.n_strips) {
							*reinterpret_cast<uint4*>(bout + g) = make_uint4(hv[0], hv[1], hv[2], hv[3]);
							*reinterpret_cast<uint4*>(bout + T.bnd_len + g) = make_uint4(fv[0], fv[1], fv[2], fv[3]);
							*reinterpret_cast<uint4*>(bout + 2 * T.bnd_len + g) = make_uint4(cmv[0], cmv[1], cmv[2], cmv[3]);
						} else if (T.cm_off != SSW_CM_NONE && g < T.p1) {
							*reinterpret_cast<uint4*>(colmax + T.cm_off + g) = make_uint4(cmv[0], cmv[1], cmv[2], cmv[3]);
						}
					}
					if (TERM && s + 1 == T.n_strips) {
						if (lane == 31) {
#pragma unroll
							for (int j = 0; j < 4; ++j) {
								if (g + j >= 0 && g + j < T.p1_a && half_of(cmv[j], 0) == T.term_a) hit |= 1;
								if (g + j >= 0 && g + j < T.p1_b && half_of(cmv[j], 1) == T.term_b) hit |= 2;
							}
						}
					}
				}
				/* publish: everything up to scan position sL + 8 of this strip's bottom row is in memory */
				if (lane == 31 && sL + 4 >= 0 && s + 1 < T.n_strips) {
					if (SPLIT && s + 1 == s_last) {
						/* consumer in another CTA: device-scope release, amortised over 128 columns (and the final ones) */
						if (((sL + 8) & 127) == 0 || sL + 8 >= hi) ssw_st_release(gprog_out, sL + 8);
					} else {
						__threadfence_block();
						prog[s] = sL + 8;
					}
				}
				if (TERM && s + 1 == T.n_strips) {
					const int hm = (__any_sync(FULL, hit & 1) ? 1 : 0) | (__any_sync(FULL, hit & 2) ? 2 : 0);
					if (hm) {
						int d = 0;
						if (lane == 0) { d = *done | hm; *done = d; if (d == need_mask) *stop = 1; }
						d = __shfl_sync(FULL, d, 0);
						if (d == need_mask) { stopped = true; break; }
					}
				}
				sp0 += 8;
				{
					const int ncol = DIR > 0 ? min(col + 8, col_hi) : max(col - 8, col_lo);
					lptr += ncol - col;
					col = ncol;
					if (DIR < 0) { const int nb_ = max(colB - 8, col_lo); lptrB += nb_ - colB; colB = nb_; }
				}
			}

			/* park the lane registers for the strip's next super-block */
			if (!stopped && hi < end) {
#pragma unroll
				for (int k = 0; k < R; ++k) { pk[k] = Hd[k]; pk[R + k] = E[k]; }
				pk[2 * R] = outH; pk[2 * R + 1] = outF; pk[2 * R + 2] = outC;
			}
			ssw_track_rows<R>(lb, snap, s * 32 * R + lane * R);
			ssw_track_unrecorded(lb);
			int sc0, bp0, br0, sc1, bp1, br1;
			ssw_reduce_best<32>(lb, sc0, bp0, br0, sc1, bp1, br1);
			if (lane == 0) {
				SswItemBest b;
				b.score[0] = sc0; b.pos[0] = bp0; b.row[0] = br0;
				b.score[1] = sc1; b.pos[1] = bp1; b.row[1] = br1;
				b.p0 = 0; b.p1 = T.p1;
				bests[T.first_best + s * T.n_super + sb] = b;
			}
			__syncwarp();
			if (stopped) break;
		}
		if (TERM) { int st = lane == 0 ? *stop : 0; st = __shfl_sync(FULL, st, 0); if (st) break; }
	}
}

#endif /* SSW_FILL_CUH */
