/*
 * ssw_traceback.cuh -- banded affine-gap fill with direction bits, traceback
 * and CIGAR re-scoring: the follow-up kernel that replaces banded_sw
 * (src/ssw.c:590-783) and cigar_alignment_score (:785-811).
 *
 * One warp per alignment (two kernels: rows in shared memory for bands up to
 * SSW_TBP_MAXBW, rows in global memory beyond).  The band of query row i covers reference columns
 * [max(0,i-bw), min(refLen-1,i+bw)] (ssw.c:630-632).  A row is processed 32
 * columns at a time: E and the diagonal term depend only on the previous row;
 * the in-row gap F obeys  F(j+1) = max(Y(j) - gapO, F(j) - min(gapO,gapE))
 * with Y = max(max(E,0), diag + s), which is evaluated exactly with a warp
 * max-plus prefix scan.  The direction codes are pure functions of the cell
 * values, so they come out identical to the reference's scalar loop:
 *     de = 3 if H(i-1,j)-gapO >  E(i-1,j)-gapE else 2          (ssw.c:650-654)
 *     df = 5 if H(i,j-1)-gapO >  F(i,j-1)-gapE else 4          (ssw.c:656-659)
 *     dh = 1 if max(e1,f1) <= diag+s else (e1 > f1 ? de : df)  (ssw.c:661-675)
 * Reference quirks reproduced on purpose (see SURVEY Appendix A.5 and DESIGN.md):
 *   - the cell above the last band column is treated as outside the band for
 *     every row i <= bw+1 (the reference zeroes h_b[edge]/e_b[edge] with `edge`
 *     computed from the current row, ssw.c:633-637), even where the previous
 *     row did reach that column;
 *   - the running maximum and its cell persist across band doublings
 *     (ssw.c:601-602, :667-671), strict '>' in row-major order;
 *   - the traceback loop runs while i >= 0 && j > 0 and the tail rule appends
 *     one more M (ssw.c:690, :745-762);
 *   - a traceback that leaves the band reads the neighbouring row's cell, as
 *     the reference's flat direction array does (set_d, ssw.c:95).
 * Direction storage is 1 byte per band cell: bit0 de==3, bit1 df==5,
 * bits 2-3 source of H (0 diagonal, 1 E, 2 F).
 */
#ifndef SSW_TRACEBACK_CUH
#define SSW_TRACEBACK_CUH

#include <vector>
#include <functional>
#include "ssw_common.cuh"
#include "ssw_host.h"

#ifndef SSW_TB_WARPS
#define SSW_TB_WARPS 4
#endif
#ifndef SSW_TB_PRE
#define SSW_TB_PRE 1                      /* scores of a row's first group are looked up ahead of the row */
#endif
#define SSW_TB_THREADS (SSW_TB_WARPS * 32)
#define SSW_TB_NEGINF (-(1 << 30))       /* INT32_MIN / 2, ssw.c:608 */

enum { SSW_TB_OK = 0, SSW_TB_WIDER = 1, SSW_TB_ERROR = 2, SSW_TB_MISMATCH = 3 };

struct SswTbTask {
	int64_t ref_off;     /* offset of ref[ref_begin1] in the padded reference array */
	int64_t read_off;    /* offset of read[read_begin1] in the query array (query profiles: of its row's first byte) */
	int32_t ref_len, read_len, score;
	int32_t bw;          /* band half-width of this round */
	int32_t max, max_i, max_j;   /* running maximum carried across band doublings */
	int32_t status, cig_len;
	int32_t init_bw;     /* band the current banded_sw call started with (retry rule, ssw.c:952-956) */
	int64_t dir_off;     /* byte offset of this task's direction cells in the scratch */
	int64_t row_off;     /* int32 offset of this task's 4 row buffers */
	int64_t cig_off;     /* word offset of this task's CIGAR buffer */
	int64_t dbg_fill, dbg_walk, dbg_score;   /* clock64 deltas of the last round (diagnostics, SSW_TRACE) */
	int64_t dbg_t0;                          /* %globaltimer (ns) when the task's warp started */
};

__device__ static __forceinline__ int64_t ssw_globaltimer()
{
#ifdef SSW_CPU_EMU
	return 0;
#else
	unsigned long long t;
	asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
	return (int64_t)t;
#endif
}
__device__ static __forceinline__ uint32_t ssw_tb_pack(uint32_t len, uint32_t op) { return (len << 4) | op; }  /* op: M0 I1 D2 */

/* PSSM: the queries are position-specific profiles (ssw_engine_set_sequences_pssm), `read` points at the task's first profile row
 * (n scores per row) and there is no matrix.  rd stands for read row i: its code (smat[letter * n + code]) or, with profiles,
 * its byte offset i * n (read[i * n + letter]). */
template <bool PSSM>
__device__ static __forceinline__ int ssw_tb_rd(const int8_t* read, int n, int i) { return PSSM ? i * n : (int)read[i]; }
template <bool PSSM>
__device__ static __forceinline__ int ssw_tb_score(const int8_t* smat, const int8_t* read, int n, int letter, int rd)
{
	return PSSM ? (int)read[rd + letter] : (int)smat[letter * n + rd];
}

/* Decide whether the band must be doubled (ssw.c:678-679); if not, walk the traceback (ssw.c:683-762) from the
 * maximum cell, run-length encode it and re-score the CIGAR (ssw.c:785-811).  One thread. */
template <bool PSSM>
__device__ static void ssw_tb_finish(SswTbTask& T, SswTbTask* slot, const int8_t* ref, const int8_t* read,
                                     const int8_t* __restrict__ mat, int n, int gapO, int gapE,
                                     const uint8_t* dir, uint32_t* cig_base)
{
	const int rl = T.ref_len, ql = T.read_len, bw = T.bw;
	const int W = 2 * bw + 1;
	const int len = rl > ql ? rl : ql;
	if (T.max < T.score && 2 * bw <= len) { T.status = SSW_TB_WIDER; *slot = T; return; }      /* ssw.c:678-679 */

	uint32_t* cig = cig_base + T.cig_off;
	const size_t dir_cells = (size_t)W * ql;
	int i = T.max_i, j = T.max_j, e = 0, l = 0, state = 2;
	int op = 0, prev = 0;                                         /* 0 M, 1 I, 2 D */
	bool bad = false;
	while (i >= 0 && j > 0) {
		const long long cell = (long long)W * i + (j - max(i - bw, 0));
		if (cell < -1 || cell > (long long)dir_cells) { bad = true; break; }      /* far outside the band: the reference reads unrelated memory */
		const int b = dir[cell];
		int code;
		if (state == 2) { const int hs = (b >> 2) & 3; code = hs == 0 ? 1 : (hs == 1 ? ((b & 1) ? 3 : 2) : (hs == 2 ? ((b & 2) ? 5 : 4) : 0)); }
		else if (state == 0) code = (b & 1) ? 3 : 2;
		else code = (b & 2) ? 5 : 4;
		if (code == 1) { --i; --j; state = 2; op = 0; }
		else if (code == 2) { --i; state = 0; op = 1; }
		else if (code == 3) { --i; state = 2; op = 1; }
		else if (code == 4) { --j; state = 1; op = 2; }
		else if (code == 5) { --j; state = 2; op = 2; }
		else { bad = true; break; }
		if (op == prev) ++e;
		else { cig[l++] = ssw_tb_pack((uint32_t)e, (uint32_t)prev); prev = op; e = 1; }
	}
	if (bad) { T.status = SSW_TB_ERROR; T.cig_len = 0; *slot = T; return; }
	if (op == 0) cig[l++] = ssw_tb_pack((uint32_t)(e + 1), 0);
	else { cig[l++] = ssw_tb_pack((uint32_t)e, (uint32_t)op); cig[l++] = ssw_tb_pack(1, 0); }
	for (int a = 0, b2 = l - 1; a < b2; ++a, --b2) { const uint32_t tmp = cig[a]; cig[a] = cig[b2]; cig[b2] = tmp; }

	int sc = 0, rp = 0, qp = 0;
	for (int k = 0; k < l; ++k) {
		const uint32_t clen = cig[k] >> 4, cop = cig[k] & 15;
		if (cop == 0) {
			for (uint32_t x = 0; x < clen; ++x) { sc += ssw_tb_score<PSSM>(mat, read, n, (int)ref[rp], ssw_tb_rd<PSSM>(read, n, qp)); ++rp; ++qp; }
		} else {
			sc -= gapO + (clen > 1 ? (int)(clen - 1) * gapE : 0);
			if (cop == 1) qp += (int)clen; else rp += (int)clen;
		}
	}
	T.cig_len = l;
	T.status = sc == T.score ? SSW_TB_OK : SSW_TB_MISMATCH;
	*slot = T;
}

/* One 32-column tile of one band row: E and the diagonal term from the previous row, F by a warp max-plus scan
 * with the carries of the tile to the left, H, and the direction byte.  Shared by both banded kernels. */
__device__ static __forceinline__ void ssw_tb_tile(bool act, int i, int j, int beg, int lane, int Hup, int Eup, int Hdg, int s,
                                                  int gapO, int gapE, int g, int& carryF, int& carryH, int& carryFp,
                                                  int& Hv, int& Ev, int& dirb)
{
	constexpr unsigned FULL = 0xffffffffu;
	const int t1 = i == 0 ? -gapO : Hup - gapO;
	const int t2 = i == 0 ? SSW_TB_NEGINF : Eup - gapE;
	Ev = t1 > t2 ? t1 : t2;
	const int de3 = t1 > t2 ? 1 : 0;
	const int e1 = Ev > 0 ? Ev : 0;
	const int T2 = Hdg + s;
	const int Y = e1 > T2 ? e1 : T2;
	/* in-row gap: inclusive max-plus scan of A = Y - gapO with decay g per column */
	int P = act ? Y - gapO : SSW_TB_NEGINF;
#pragma unroll
	for (int d = 1; d < 32; d <<= 1) {
		const int o = __shfl_up_sync(FULL, P, d);
		if (lane >= d) P = max(P, o - d * g);
	}
	const int Pm1 = __shfl_up_sync(FULL, P, 1);
	const int Fv = lane == 0 ? carryF : max(Pm1, carryF - lane * g);
	Hv = Y > Fv ? Y : Fv;
	/* df from the left neighbour's H and F */
	int Hl = __shfl_up_sync(FULL, Hv, 1), Fl = __shfl_up_sync(FULL, Fv, 1);
	if (lane == 0) { Hl = carryH; Fl = carryFp; }
	const int df5 = j == beg ? 1 : ((Hl - gapO > Fl - gapE) ? 1 : 0);       /* j == beg: 0 - gapO > neg_inf - gapE */
	const int f1 = Fv > 0 ? Fv : 0;
	const int T1 = e1 > f1 ? e1 : f1;
	const int hsel = T1 <= T2 ? 0 : (e1 > f1 ? 1 : 2);
	dirb = de3 | (df5 << 1) | (hsel << 2);
	/* carries into the next tile */
	const int P31 = __shfl_sync(FULL, P, 31);
	carryH = __shfl_sync(FULL, Hv, 31);
	carryFp = __shfl_sync(FULL, Fv, 31);
	carryF = max(P31, carryF - 32 * g);
}

/* NT adjacent tiles of one band row at once.  Same arithmetic as ssw_tb_tile, reordered so that the tiles' scans
 * (the long chain of dependent shuffles) are independent instruction streams the scheduler can interleave; only the
 * F carry from tile to tile is serial, and that is one max per tile.  A row of the band then costs about one tile's
 * latency instead of NT. */
template <int NT, bool LAST>
__device__ static __forceinline__ void ssw_tb_tiles(const bool (&act)[NT], int i, const int (&j)[NT], int beg, int lane,
                                                   const int (&Hup)[NT], const int (&Eup)[NT], const int (&Hdg)[NT], const int (&s)[NT],
                                                   int gapO, int gapE, int g, int& carryF, int& carryFp,
                                                   int (&Hv)[NT], int (&Ev)[NT], int (&dirb)[NT], int span)
{
	constexpr unsigned FULL = 0xffffffffu;
	int de3[NT], e1[NT], T2[NT], Y[NT], P[NT];
#pragma unroll
	for (int t = 0; t < NT; ++t) {
		const int t1 = i == 0 ? -gapO : Hup[t] - gapO;
		const int t2 = i == 0 ? SSW_TB_NEGINF : Eup[t] - gapE;
		Ev[t] = t1 > t2 ? t1 : t2;
		de3[t] = t1 > t2 ? 1 : 0;
		e1[t] = Ev[t] > 0 ? Ev[t] : 0;
		T2[t] = Hdg[t] + s[t];
		Y[t] = e1[t] > T2[t] ? e1[t] : T2[t];
		P[t] = act[t] ? Y[t] - gapO : SSW_TB_NEGINF;
	}
	/* `span` active lanes (warp-uniform): distances of span and more cannot contribute, so a narrow band row needs
	 * fewer than five levels of the scan */
#pragma unroll
	for (int d = 1; d < 32; d <<= 1) {
		if (d >= span) break;
#pragma unroll
		for (int t = 0; t < NT; ++t) {
			const int o = __shfl_up_sync(FULL, P[t], d);
			if (lane >= d) P[t] = max(P[t], o - d * g);
		}
	}
	/* Shuffles cost this kernel its time (a warp's shuffles do not overlap, so a radix-4 scan with 7 independent shuffles
	 * instead of 5 dependent ones is slower), so only the ones that are needed are issued:
	 *  - df5 needs F of the left neighbour only: F(j) = max(H(j-1) - gapO, F(j-1) - gapE) is what the scan computes
	 *    (with Y for H and g for gapE: the same value in both gap regimes), hence
	 *    H(j-1) - gapO > F(j-1) - gapE  <=>  F(j) > F(j-1) - gapE, and H of the neighbour is never fetched;
	 *  - the carries out of the last tile of a row (LAST) are never read. */
	int Pm1[NT], P31[NT], cF[NT], Fv[NT];
#pragma unroll
	for (int t = 0; t < NT; ++t) {
		Pm1[t] = __shfl_up_sync(FULL, P[t], 1);
		P31[t] = (LAST && t == NT - 1) ? 0 : __shfl_sync(FULL, P[t], 31);
	}
	cF[0] = carryF;
#pragma unroll
	for (int t = 1; t < NT; ++t) cF[t] = max(P31[t - 1], cF[t - 1] - 32 * g);
	if (!LAST) carryF = max(P31[NT - 1], cF[NT - 1] - 32 * g);
	int F31[NT], Fl[NT];
#pragma unroll
	for (int t = 0; t < NT; ++t) {
		Fv[t] = lane == 0 ? cF[t] : max(Pm1[t], cF[t] - lane * g);
		Hv[t] = Y[t] > Fv[t] ? Y[t] : Fv[t];
		F31[t] = (LAST && t == NT - 1) ? 0 : __shfl_sync(FULL, Fv[t], 31);
		Fl[t] = __shfl_up_sync(FULL, Fv[t], 1);
	}
#pragma unroll
	for (int t = 0; t < NT; ++t) {
		if (lane == 0) Fl[t] = t == 0 ? carryFp : F31[t - 1];
		const int df5 = j[t] == beg ? 1 : ((Fv[t] > Fl[t] - gapE) ? 1 : 0);
		const int f1 = Fv[t] > 0 ? Fv[t] : 0;
		const int T1 = e1[t] > f1 ? e1[t] : f1;
		const int hsel = T1 <= T2[t] ? 0 : (e1[t] > f1 ? 1 : 2);
		dirb[t] = de3[t] | (df5 << 1) | (hsel << 2);
	}
	if (!LAST) carryFp = F31[NT - 1];
}

/* one group of NT tiles of row i starting at column j0: loads from the row ring, ssw_tb_tiles, stores */
template <bool PSSM, int NT, bool LAST, bool PRE = false>
__device__ static __forceinline__ void ssw_tb_row_group(int i, int j0, int beg, int end, int pbeg, bool top_oob, int lane, int rd,
                                                       const int32_t* Hprev, const int32_t* Eprev, int32_t* Hcur, int32_t* Ecur, int mask,
                                                       const int8_t* smat, const int8_t* read, int n, const int8_t* ref, uint8_t* drow,
                                                       int gapO, int gapE, int g, int& carryF, int& carryFp,
                                                       int& bestv, int& besti, int& bestj, const int* spre = nullptr)
{
	bool act[NT];
	int j[NT], Hup[NT], Eup[NT], Hdg[NT], s[NT], Hv[NT], Ev[NT], dirb[NT];
#pragma unroll
	for (int t = 0; t < NT; ++t) {
		j[t] = j0 + 32 * t + lane;
		act[t] = j[t] <= end;
		Hup[t] = 0; Eup[t] = SSW_TB_NEGINF; Hdg[t] = 0; s[t] = 0;
		if (act[t]) {
			if (i > 0) {
				if (!(j[t] == end && top_oob)) { Hup[t] = Hprev[j[t] & mask]; Eup[t] = Eprev[j[t] & mask]; }
				if (j[t] - 1 >= pbeg) Hdg[t] = Hprev[(j[t] - 1) & mask];
			}
			s[t] = PRE ? spre[t] : ssw_tb_score<PSSM>(smat, read, n, (int)ref[j[t]], rd);      /* PRE: looked up ahead of the row (first group) */
		}
	}
	ssw_tb_tiles<NT, LAST>(act, i, j, beg, lane, Hup, Eup, Hdg, s, gapO, gapE, g, carryF, carryFp, Hv, Ev, dirb,
	                 NT == 1 ? min(32, end - j0 + 1) : 32);
#pragma unroll
	for (int t = 0; t < NT; ++t) {
		if (act[t]) {
			Hcur[j[t] & mask] = Hv[t];
			Ecur[j[t] & mask] = Ev[t];
			drow[j[t]] = (uint8_t)dirb[t];
			if (Hv[t] > bestv) { bestv = Hv[t]; besti = i; bestj = j[t]; }
		}
	}
}

/* Row ring width (ints, a power of two) for a band of half-width bw: the live part of a row spans 2*bw + 1 columns, the
 * tiles of a row group may run up to 64 columns beyond it. */
__host__ __device__ static __forceinline__ int ssw_tb_ring_of(int bw)
{
	int r = 128;
	while (r < 2 * bw + 66) r <<= 1;
	return r;
}

/* One banded fill (ssw.c:628-676) by one warp: rows in the warp's shared-memory ring `mine` (4 x ring ints), direction bytes
 * to `dir`, returns the first row-major cell holding the maximum of this band (all lanes). */
template <bool PSSM>
__device__ static __forceinline__ void ssw_tb_band_fill(int lane, int ql, int rl, int bw, const int8_t* ref, const int8_t* read,
                                                       const int8_t* smat, int n, int gapO, int gapE, int g,
                                                       int32_t* mine, int ring, uint8_t* dir, int& bestv, int& besti, int& bestj)
{
	constexpr unsigned FULL = 0xffffffffu;
	const int mask = ring - 1;
	const int W = 2 * bw + 1;
	bestv = 0; besti = 0; bestj = 0;
	int rd_next = ssw_tb_rd<PSSM>(read, n, 0);
	int letn[4];                                         /* reference letters of the next row's first group (clamped into the reference) */
#pragma unroll
	for (int t = 0; t < 4; ++t) letn[t] = (int)ref[min(32 * t + lane, rl - 1)];
	for (int i = 0; i < ql; ++i) {
		/* the rows as offsets from the one shared-memory base: LDS/STS (an array of row pointers indexed by the row parity
		 * lives in local memory and turns every row access into a generic load behind a local load; measured equally fast) */
		const int cur = (i & 1) * ring, prv = ring - cur;
		int32_t* const Hc = mine + cur;
		int32_t* const Ec = mine + 2 * ring + cur;
		const int32_t* const Hp = mine + prv;
		const int32_t* const Ep = mine + 2 * ring + prv;
		const int beg = max(0, i - bw), end = min(rl - 1, i + bw);
		const int pbeg = max(0, i - 1 - bw);
		const bool top_oob = (i <= bw + 1) || (end == i + bw);
		const int rd = rd_next;
		if (i + 1 < ql) rd_next = ssw_tb_rd<PSSM>(read, n, i + 1);
		uint8_t* drow = dir + (size_t)W * i - beg;
		/* scores of the row's first group from the letters fetched during the previous row (the letter fetch and the matrix
		 * look-up behind it would otherwise head the row's dependent chain), then the letters of the next row's first group */
		int spre[4];
#if SSW_TB_PRE
#pragma unroll
		for (int t = 0; t < 4; ++t) spre[t] = ssw_tb_score<PSSM>(smat, read, n, letn[t], rd);
		{
			const int begn = max(0, i + 1 - bw);
#pragma unroll
			for (int t = 0; t < 4; ++t) letn[t] = (int)ref[min(begn + 32 * t + lane, rl - 1)];
		}
#endif
		{
			int carryF = -gapO, carryFp = 0;
			int j0 = beg;
#define SSW_TB_GROUP(NT, LAST, PRE)                                                                                          \
			ssw_tb_row_group<PSSM, NT, LAST, PRE>(i, j0, beg, end, pbeg, top_oob, lane, rd, Hp, Ep, Hc, Ec, mask, smat, read, n, ref, drow, \
			                                gapO, gapE, g, carryF, carryFp, bestv, besti, bestj, spre)
			if (j0 <= end) {                                  /* first group: scores looked up ahead */
				const int tiles = (end - j0) / 32 + 1;
				if (tiles > 4) { SSW_TB_GROUP(4, false, SSW_TB_PRE != 0); j0 += 128; }
				else if (tiles >= 3) { SSW_TB_GROUP(4, true, SSW_TB_PRE != 0); j0 += 128; }
				else if (tiles == 2) { SSW_TB_GROUP(2, true, SSW_TB_PRE != 0); j0 += 64; }
				else { SSW_TB_GROUP(1, true, SSW_TB_PRE != 0); j0 += 32; }
			}
			while (j0 <= end) {
				const int tiles = (end - j0) / 32 + 1;
				if (tiles > 4) { SSW_TB_GROUP(4, false, false); j0 += 128; }
				else if (tiles >= 3) { SSW_TB_GROUP(4, true, false); j0 += 128; }
				else if (tiles == 2) { SSW_TB_GROUP(2, true, false); j0 += 64; }
				else { SSW_TB_GROUP(1, true, false); j0 += 32; }
			}
#undef SSW_TB_GROUP
		}
		__syncwarp();
	}
#pragma unroll
	for (int off = 16; off >= 1; off >>= 1) {
		const int ov = __shfl_xor_sync(FULL, bestv, off), oi = __shfl_xor_sync(FULL, besti, off), oj = __shfl_xor_sync(FULL, bestj, off);
		if (ov > bestv || (ov == bestv && (oi < besti || (oi == besti && oj < bestj)))) { bestv = ov; besti = oi; bestj = oj; }
	}
}

/* Traceback (ssw.c:683-762) of the finished band T.bw by one warp, staged through `stage` (shared memory, stage_bytes): the warp
 * copies blocks of direction bytes with coalesced loads and lane 0 walks inside them (the plain walk pays a DRAM latency per
 * step because every step moves up one band row); then the CIGAR re-scoring (ssw.c:785-811).  Writes the task record. */
template <bool PSSM>
__device__ static __forceinline__ void ssw_tb_walk(SswTbTask& T, SswTbTask* slot, int lane, const uint8_t* dir, uint8_t* stage, int stage_bytes,
                                                  uint32_t* cig, const int8_t* smat, const int8_t* ref, const int8_t* read, int n,
                                                  int gapO, int gapE, long long c1)
{
	constexpr unsigned FULL = 0xffffffffu;
	const int bw = T.bw, W = 2 * bw + 1, ql = T.read_len;
	const long long dir_cells = (long long)W * ql;
	const int rows_per_block = max(1, (stage_bytes - 48) / W);     /* 8 spare bytes + up to 2 x 15 bytes of alignment slack */
	int wi = T.max_i, wj = T.max_j, e = 0, l = 0, state = 2, op = 0, prev = 0;
	int bad = 0, more = (wi >= 0 && wj > 0) ? 1 : 0;
	while (more) {
		const int i_lo = max(0, wi - rows_per_block + 1);
		const long long want = (long long)W * i_lo - 1;               /* first cell the walk may read: x == -1 of the lowest row */
		const long long last = min((long long)W * (wi + 1), dir_cells);   /* last staged cell: x == 2bw+1 of the top row */
		/* 16 bytes per lane and step: the block starts at the 16-byte boundary at or below `want` (never below this task's
		 * own cells: they begin on such a boundary) and ends with the 16-byte word that holds `last` (inside the padded area) */
		const long long base = want - (long long)(reinterpret_cast<uintptr_t>(dir + want) & 15);
		{
			const uint4* src = reinterpret_cast<const uint4*>(dir + base);
			uint4* dst = reinterpret_cast<uint4*>(stage);
			const int n16 = (int)((last - base) / 16) + 1;
			int k = lane;
			for (; k + 96 < n16; k += 128) {
				const uint4 a = src[k], b = src[k + 32], c = src[k + 64], d = src[k + 96];
				dst[k] = a; dst[k + 32] = b; dst[k + 64] = c; dst[k + 96] = d;
			}
			for (; k < n16; k += 32) dst[k] = src[k];
		}
		__syncwarp();
		if (lane == 0) {
			more = 0;
			while (wi >= 0 && wj > 0) {
				if (wi < i_lo) { more = 1; break; }
				const long long cell = (long long)W * wi + (wj - max(wi - bw, 0));
				if (cell < -1 || cell > dir_cells) { bad = 1; break; }    /* far outside the band: the reference reads unrelated memory */
				const int b = (cell >= base && cell <= last) ? (int)stage[cell - base] : (int)dir[cell];
				int code;
				if (state == 2) { const int hs = (b >> 2) & 3; code = hs == 0 ? 1 : (hs == 1 ? ((b & 1) ? 3 : 2) : (hs == 2 ? ((b & 2) ? 5 : 4) : 0)); }
				else if (state == 0) code = (b & 1) ? 3 : 2;
				else code = (b & 2) ? 5 : 4;
				if (code == 1) { --wi; --wj; state = 2; op = 0; }
				else if (code == 2) { --wi; state = 0; op = 1; }
				else if (code == 3) { --wi; state = 2; op = 1; }
				else if (code == 4) { --wj; state = 1; op = 2; }
				else if (code == 5) { --wj; state = 2; op = 2; }
				else { bad = 1; break; }
				if (op == prev) ++e;
				else { cig[l++] = ssw_tb_pack((uint32_t)e, (uint32_t)prev); prev = op; e = 1; }
			}
		}
		more = __shfl_sync(FULL, more, 0);
		wi = __shfl_sync(FULL, wi, 0);
		__syncwarp();
	}
	if (lane != 0) return;
	const long long c2 = clock64();
	T.dbg_walk = c2 - c1;
	if (bad) { T.status = SSW_TB_ERROR; T.cig_len = 0; *slot = T; return; }
	if (op == 0) cig[l++] = ssw_tb_pack((uint32_t)(e + 1), 0);
	else { cig[l++] = ssw_tb_pack((uint32_t)e, (uint32_t)op); cig[l++] = ssw_tb_pack(1, 0); }
	for (int a = 0, b2 = l - 1; a < b2; ++a, --b2) { const uint32_t tmp = cig[a]; cig[a] = cig[b2]; cig[b2] = tmp; }
	/* ---- CIGAR re-scoring (ssw.c:785-811) ---- */
	int sc = 0, rp = 0, qp = 0;
	for (int k = 0; k < l; ++k) {
		const uint32_t clen = cig[k] >> 4, cop = cig[k] & 15;
		if (cop == 0) {
			for (uint32_t x = 0; x < clen; ++x) { sc += ssw_tb_score<PSSM>(smat, read, n, (int)ref[rp], ssw_tb_rd<PSSM>(read, n, qp)); ++rp; ++qp; }
		} else {
			sc -= gapO + (clen > 1 ? (int)(clen - 1) * gapE : 0);
			if (cop == 1) qp += (int)clen; else rp += (int)clen;
		}
	}
	T.cig_len = l;
	T.status = sc == T.score ? SSW_TB_OK : SSW_TB_MISMATCH;
	T.dbg_score = clock64() - c2;
	*slot = T;
}

/*
 * Fast variant for bands up to SSW_TBP_MAXBW: one warp per alignment, four alignments per CTA.  The two live H/E
 * rows sit in shared memory (indexed by reference column modulo the ring width), the scoring matrix too, so a
 * tile's critical path has no global-memory latency.  After the fill the warp stages blocks of direction bytes into
 * its (now free) row memory with coalesced loads and lane 0 walks the traceback inside them.
 */
#define SSW_TBP_MAXBW 990

template <bool PSSM>
__global__ void __launch_bounds__(SSW_TB_THREADS)
ssw_banded_smem_kernel(SswTbTask* __restrict__ tasks, int n_tasks,
                       const int8_t* __restrict__ qcodes, const int8_t* __restrict__ refs,
                       const int8_t* __restrict__ mat, int n, int gapO, int gapE,
                       uint8_t* __restrict__ dir_base, uint32_t* __restrict__ cig_base, int ring)
{
	SSW_DYN_SMEM(int32_t, smem);                                  /* [warp][4][ring] ints, then n*n matrix bytes */
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	int8_t* smat = reinterpret_cast<int8_t*>(smem + (size_t)SSW_TB_WARPS * 4 * ring);
	if (!PSSM) for (int k = threadIdx.x; k < n * n; k += blockDim.x) smat[k] = mat[k];
	__syncthreads();
	const int ti = (int)blockIdx.x * SSW_TB_WARPS + warp;
	if (ti >= n_tasks) return;
	SswTbTask T = tasks[ti];
	T.dbg_t0 = ssw_globaltimer();
	const int8_t* ref = refs + T.ref_off;
	const int8_t* read = qcodes + T.read_off;
	const int rl = T.ref_len, ql = T.read_len;
	const int g = gapO < gapE ? gapO : gapE;
	uint8_t* dir = dir_base + T.dir_off + 1;
	int32_t* mine = smem + (size_t)warp * 4 * ring;
	const int len = rl > ql ? rl : ql;
	const long long c0 = clock64();
	int bw = T.bw;

	/* band-doubling loop of banded_sw (ssw.c:616-680), kept inside the kernel while the doubled band still fits the
	 * row ring: only the last band's directions are needed, and the running maximum is carried in T */
	for (;;) {
		int bestv, besti, bestj;
		ssw_tb_band_fill<PSSM>(lane, ql, rl, bw, ref, read, smat, n, gapO, gapE, g, mine, ring, dir, bestv, besti, bestj);
		if (bestv > T.max) { T.max = bestv; T.max_i = besti; T.max_j = bestj; }     /* strict, carried across doublings */
		if (!(T.max < T.score && 2 * bw <= len)) break;                              /* ssw.c:678-679: done */
		if (2 * (2 * bw) + 66 > ring) {                                              /* the next band needs a wider ring: back to the host */
			T.bw = bw;
			if (lane == 0) { T.status = SSW_TB_WIDER; tasks[ti] = T; }
			return;
		}
		bw *= 2;
		__syncwarp();
	}
	T.bw = bw;
	const long long c1 = clock64();
	T.dbg_fill = c1 - c0; T.dbg_walk = 0; T.dbg_score = 0;
	__threadfence_block();
	__syncwarp();
	ssw_tb_walk<PSSM>(T, tasks + ti, lane, dir, reinterpret_cast<uint8_t*>(mine), 4 * ring * (int)sizeof(int32_t), cig_base + T.cig_off,
	            smat, ref, read, n, gapO, gapE, c1);
}

/*
 * Speculative variant: one CTA per alignment, warp w fills band T.bw << w -- the band-doubling rounds of banded_sw
 * (ssw.c:616-680) side by side instead of one after the other.  A round is a chain of dependent rows (about one tile's
 * scan latency per row whatever the band, up to four tiles), so the rounds of a task cost the time of the widest one instead
 * of their sum; the device is nearly idle during this phase, the extra bands are free.  The reference's sequence is
 * reproduced from the per-round results: the running maximum and its cell persist across rounds with strict '>'
 * (ssw.c:601,667-671), i.e. round k contributes its first row-major maximum only if that exceeds every earlier round's;
 * the first round after which `max >= score || 2*bw > len` is the band the traceback walks (later rounds are discarded).
 * If no speculated round ends the loop the task goes back to the host with the last band tried (status WIDER).
 * Shared memory: the scoring matrix, then the row rings of the rounds (4 x ssw_tb_ring_of(bw_w) ints each).  Direction
 * bytes: round w at dir_off + sum of the earlier rounds' (16-byte aligned) sizes.
 */
#define SSW_TBS_MAXW 8
__host__ __device__ static __forceinline__ size_t ssw_tb_dir_bytes(int bw, int read_len) { return (((size_t)(2 * bw + 1) * (size_t)read_len + 2) + 15) / 16 * 16; }

template <bool PSSM>
__global__ void __launch_bounds__(SSW_TBS_MAXW * 32)
ssw_banded_spec_kernel(SswTbTask* __restrict__ tasks, int n_tasks,
                       const int8_t* __restrict__ qcodes, const int8_t* __restrict__ refs,
                       const int8_t* __restrict__ mat, int n, int gapO, int gapE,
                       uint8_t* __restrict__ dir_base, uint32_t* __restrict__ cig_base, int nw)
{
	SSW_DYN_SMEM(int32_t, smem);
	__shared__ int s_best[SSW_TBS_MAXW][3];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int mat_ints = (n * n + 15) / 16 * 4;
	int8_t* smat = reinterpret_cast<int8_t*>(smem);
	if (!PSSM) for (int k = threadIdx.x; k < n * n; k += blockDim.x) smat[k] = mat[k];
	__syncthreads();
	const int ti = (int)blockIdx.x;
	if (ti >= n_tasks) return;
	SswTbTask T = tasks[ti];
	const int8_t* ref = refs + T.ref_off;
	const int8_t* read = qcodes + T.read_off;
	const int rl = T.ref_len, ql = T.read_len;
	const int g = gapO < gapE ? gapO : gapE;
	const int len = rl > ql ? rl : ql;
	const long long c0 = clock64();
	/* geometry of this warp's round; rounds behind one whose band already exceeds `len` can never run (ssw.c:679) */
	int bw = T.bw, ring_off = mat_ints;
	size_t dir_off = 0;
	bool possible = true;
	for (int w = 0; w < warp; ++w) {
		if (!(2 * bw <= len)) possible = false;
		ring_off += 4 * ssw_tb_ring_of(bw);
		dir_off += ssw_tb_dir_bytes(bw, ql);
		bw *= 2;
	}
	int total_ints = ring_off;
	{
		int b2 = bw;
		for (int w = warp; w < nw; ++w) { total_ints += 4 * ssw_tb_ring_of(b2); b2 *= 2; }
	}
	uint8_t* dir = dir_base + T.dir_off + dir_off + 1;
	if (warp < nw && possible) {
		int bestv, besti, bestj;
		ssw_tb_band_fill<PSSM>(lane, ql, rl, bw, ref, read, smat, n, gapO, gapE, g, smem + ring_off, ssw_tb_ring_of(bw), dir, bestv, besti, bestj);
		if (lane == 0) { s_best[warp][0] = bestv; s_best[warp][1] = besti; s_best[warp][2] = bestj; }
	}
	__threadfence_block();
	__syncthreads();
	if (warp != 0) return;
	/* the reference's sequence over the rounds */
	int kb = T.bw, done = -1, last_bw = T.bw;
	size_t koff = 0, done_off = 0;
	for (int w = 0; w < nw; ++w) {
		if (s_best[w][0] > T.max) { T.max = s_best[w][0]; T.max_i = s_best[w][1]; T.max_j = s_best[w][2]; }
		last_bw = kb;
		if (!(T.max < T.score && 2 * kb <= len)) { done = w; done_off = koff; break; }
		koff += ssw_tb_dir_bytes(kb, ql);
		kb *= 2;
	}
	T.bw = last_bw;
	const long long c1 = clock64();
	T.dbg_fill = c1 - c0; T.dbg_walk = 0; T.dbg_score = 0;
	if (done < 0) {
		if (lane == 0) { T.status = SSW_TB_WIDER; tasks[ti] = T; }
		return;
	}
	ssw_tb_walk<PSSM>(T, tasks + ti, lane, dir_base + T.dir_off + done_off + 1, reinterpret_cast<uint8_t*>(smem + mat_ints),
	            (total_ints - mat_ints) * (int)sizeof(int32_t), cig_base + T.cig_off, smat, ref, read, n, gapO, gapE, c1);
}

/* General variant (any band width): one warp per alignment, H/E rows in global memory. */
template <bool PSSM>
__global__ void __launch_bounds__(SSW_TB_THREADS)
ssw_banded_kernel(SswTbTask* __restrict__ tasks, int n_tasks,
                  const int8_t* __restrict__ qcodes, const int8_t* __restrict__ refs,
                  const int8_t* __restrict__ mat, int n, int gapO, int gapE,
                  uint8_t* __restrict__ dir_base, int32_t* __restrict__ row_base, uint32_t* __restrict__ cig_base)
{
	constexpr unsigned FULL = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	const int ti = (int)blockIdx.x * SSW_TB_WARPS + (threadIdx.x >> 5);
	if (ti >= n_tasks) return;
	SswTbTask T = tasks[ti];
	const int8_t* ref = refs + T.ref_off;
	const int8_t* read = qcodes + T.read_off;
	const int rl = T.ref_len, ql = T.read_len, bw = T.bw;
	const int W = 2 * bw + 1;
	const int g = gapO < gapE ? gapO : gapE;
	uint8_t* dir = dir_base + T.dir_off + 1;                    /* one spare byte in front for x == -1 at row 0 */
	int32_t* Hrow[2] = {row_base + T.row_off + 1, row_base + T.row_off + (rl + 2) + 1};
	int32_t* Erow[2] = {row_base + T.row_off + 2 * (rl + 2) + 1, row_base + T.row_off + 3 * (rl + 2) + 1};

	/* ---------------- banded fill (ssw.c:628-676) ---------------- */
	int bestv = 0, besti = 0, bestj = 0;
	for (int i = 0; i < ql; ++i) {
		const int cur = i & 1, prv = cur ^ 1;
		const int beg = max(0, i - bw), end = min(rl - 1, i + bw);
		const int pbeg = max(0, i - 1 - bw);
		const bool top_oob = (i <= bw + 1) || (end == i + bw);   /* cell above column `end` reads as outside the band */
		const int rd = ssw_tb_rd<PSSM>(read, n, i);
		uint8_t* drow = dir + (size_t)W * i - beg;              /* drow[j] is the cell of column j */
		int carryF = -gapO;                                      /* F of the tile's first column; F(beg) = max(0-gapO, neg_inf-gapE) */
		int carryH = 0, carryFp = 0;                             /* H, F of the column left of the tile */
		for (int j0 = beg; j0 <= end; j0 += 32) {
			const int j = j0 + lane;
			const bool act = j <= end;
			int Hup = 0, Eup = SSW_TB_NEGINF, Hdg = 0, s = 0;
			if (act) {
				if (i > 0) {
					if (!(j == end && top_oob)) { Hup = Hrow[prv][j]; Eup = Erow[prv][j]; }
					if (j - 1 >= pbeg) Hdg = Hrow[prv][j - 1];
				}
				s = ssw_tb_score<PSSM>(mat, read, n, (int)ref[j], rd);
			}
			int Hv, Ev, dirb;
			ssw_tb_tile(act, i, j, beg, lane, Hup, Eup, Hdg, s, gapO, gapE, g, carryF, carryH, carryFp, Hv, Ev, dirb);
			if (act) {
				Hrow[cur][j] = Hv;
				Erow[cur][j] = Ev;
				drow[j] = (uint8_t)dirb;
				if (Hv > bestv) { bestv = Hv; besti = i; bestj = j; }
			}
		}
		__syncwarp();
	}
	/* first row-major cell holding the maximum */
#pragma unroll
	for (int off = 16; off >= 1; off >>= 1) {
		const int ov = __shfl_xor_sync(FULL, bestv, off), oi = __shfl_xor_sync(FULL, besti, off), oj = __shfl_xor_sync(FULL, bestj, off);
		if (ov > bestv || (ov == bestv && (oi < besti || (oi == besti && oj < bestj)))) { bestv = ov; besti = oi; bestj = oj; }
	}
	if (bestv > T.max) { T.max = bestv; T.max_i = besti; T.max_j = bestj; }     /* strict, carried across doublings */
	__threadfence_block();
	__syncwarp();
	if (lane == 0) ssw_tb_finish<PSSM>(T, tasks + ti, ref, read, mat, n, gapO, gapE, dir, cig_base);
}

/*
 * Host driver of P3: band-doubling rounds (ssw.c:616-680) and the full-band retry of ssw_align (:945-957).
 * A round groups the unfinished tasks by kernel shape (row-ring width; 0 = global-memory kernel) and launches the
 * groups concurrently on separate streams: every task is a latency-bound chain (row after row), so a launch lasts
 * as long as its slowest task and overlapping the groups hides most of that.  `emit(i, words, len, failed)` is
 * called once per task with the final CIGAR (failed != 0: banded_sw gave up -> flag 1).
 */
/* finished CIGARs -> one dense array (the per-task buffers are sized for the worst case, ref_len + read_len words):
 * task i's words move from cig[cig_off ...] to dense[row_off ...]; row_off is re-used as the destination offset */
__global__ void __launch_bounds__(128)
ssw_cigar_pack_kernel(const SswTbTask* __restrict__ tasks, int n_tasks, const uint32_t* __restrict__ cig, uint32_t* __restrict__ dense)
{
	const int ti = (int)blockIdx.x;
	if (ti >= n_tasks) return;
	const int len = tasks[ti].status == SSW_TB_OK ? tasks[ti].cig_len : 0;
	const uint32_t* src = cig + tasks[ti].cig_off;
	uint32_t* dst = dense + tasks[ti].row_off;
	for (int k = (int)threadIdx.x; k < len; k += (int)blockDim.x) dst[k] = src[k];
}

static int ssw_traceback_run(cudaStream_t stream, cudaStream_t* side /* 3 side streams of the caller, created on demand */,
                             std::vector<SswTbTask>& tasks,
                             const int8_t* d_q, const int8_t* d_r,
                             const int8_t* d_mat /* nullptr: d_q holds query profiles and read_off counts their bytes */, int n, int gapO, int gapE,
                             SswDevBuf* scratch, float* ms_acc, int64_t* launches,
                             int tb_maxbw /* "tb_maxbw" option: bands above this use the global-memory kernel (tests: 0) */,
                             bool carve /* "carve" option: largest shared-memory carve-out for the traceback kernels */,
                             int tb_spec /* "tb_spec" option: 0 = band-doubling rounds one after the other, 1 = side by side (speculative kernel),
                                            -1 = side by side when the batch is too small to keep the device busy anyway */,
                             const std::function<int(size_t, const uint32_t*, int32_t, int)>& emit)
{
	std::vector<size_t> active(tasks.size());
	for (size_t i = 0; i < tasks.size(); ++i) {
		SswTbTask& t = tasks[i];
		active[i] = i;
		int d = t.ref_len - t.read_len;
		t.bw = t.init_bw = (d < 0 ? -d : d) + 1;                 /* ssw.c:944 */
		t.max = 0; t.max_i = 0; t.max_j = 0; t.status = SSW_TB_WIDER; t.cig_len = 0;
	}
	const size_t free_b = ssw_free_device_bytes();
	const size_t budget = std::max<size_t>((size_t)64 << 20, ssw_budget_share(free_b + scratch->cap));
	/* Rounds of band doubling run side by side by the speculative kernel (1: not used).  Narrow bands (up to four tiles per row)
	 * cost one tile latency per row whatever their width, so all of them go together; of wider ones at most two, so that
	 * a task that needs only the first loses little. */
	/* Config 5 (1,000 reads of 10 kbp): with a thousand tasks in flight the phase is bound by instruction
	 * issue, not by the latency of a row, and the speculative rounds make it slower; a single 10 kbp read
	 * (one ssw_align call) is pure latency and gains.  Automatic: on for a handful of tasks only (slices of 250 tasks were
	 * still slower with it). */
	const bool spec_on = tb_spec > 0 || (tb_spec < 0 && tasks.size() <= 8);
	const int tb_spec_w = tb_spec > 1 ? tb_spec : 129;          /* "tb_spec" values above 1: widest row (columns) of a speculated round */
	auto spec_rounds = [tb_maxbw, spec_on, tb_spec_w](const SswTbTask& t) -> int {
		if (!spec_on) return 1;
		const int len = std::max(t.ref_len, t.read_len);
		int nw = 0, bw = t.bw;
		while (nw < SSW_TBS_MAXW && bw <= tb_maxbw) {
			if (nw >= 1 && 2 * bw + 1 > tb_spec_w) break;      /* only rounds of at most tb_spec_w columns ride along with the first one */
			++nw;
			if (!(2 * bw <= len)) break;
			bw *= 2;
		}
		return nw;
	};
	/* kernel shape of a task: > 0 row-ring width of the one-warp shared-memory kernel, 0 the global-memory kernel,
	 * < 0 minus the number of rounds of the speculative kernel */
	auto ring_of = [tb_maxbw, &spec_rounds](const SswTbTask& t) -> int {
		if (t.bw > tb_maxbw) return 0;
		const int nw = spec_rounds(t);
		if (nw >= 2) return -nw;
		int r = 256;
		while (r < 2 * (4 * t.bw) + 66 && r < 2048) r <<= 1;    /* room for two in-kernel doublings */
		while (r < 2 * t.bw + 66) r <<= 1;
		return r;
	};
	SswTimer tm;
	std::vector<uint32_t> cig_host;
	while (!active.empty()) {
		/* the round: tasks in kernel-shape order, as many as fit the scratch budget */
		std::stable_sort(active.begin(), active.end(), [&](size_t x, size_t y) { return ring_of(tasks[x]) < ring_of(tasks[y]); });
		std::vector<size_t> batch;
		std::vector<int> batch_ring;
		size_t dir_bytes = 0, row_ints = 0, cig_words = 0, k = 0;
		for (; k < active.size(); ++k) {
			SswTbTask& t = tasks[active[k]];
			const int ring = ring_of(t);
			size_t bw_last = (size_t)t.bw;                          /* widest band the kernel may reach by itself */
			if (ring > 0) while (2 * (2 * bw_last) + 66 <= (size_t)ring && 2 * bw_last <= (size_t)std::max(t.ref_len, t.read_len)) bw_last *= 2;
			size_t d = ((2 * bw_last + 1) * (size_t)t.read_len + 2 + 15) / 16 * 16;
			if (ring < 0) {                                         /* speculative kernel: every round has its own direction cells */
				d = 0;
				int b2 = t.bw;
				for (int w = 0; w < -ring; ++w) { d += ssw_tb_dir_bytes(b2, t.read_len); b2 *= 2; }
			}
			const size_t r = ring ? 0 : 4 * ((size_t)t.ref_len + 2);
			const size_t c = (size_t)t.ref_len + (size_t)t.read_len + 4;
			const size_t need = dir_bytes + d + 4 * (row_ints + r) + 4 * (cig_words + c) + sizeof(SswTbTask) * (batch.size() + 1) + 1024;
			if (!batch.empty() && need > budget) break;
			t.dir_off = (int64_t)dir_bytes; t.row_off = (int64_t)row_ints; t.cig_off = (int64_t)cig_words;
			dir_bytes += d; row_ints += r; cig_words += c;
			batch.push_back(active[k]);
			batch_ring.push_back(ring);
		}
		std::vector<size_t> rest(active.begin() + k, active.end());
		const size_t off_rows = (dir_bytes + 255) / 256 * 256;
		const size_t off_cig = off_rows + (row_ints * 4 + 255) / 256 * 256;
		const size_t off_tasks = off_cig + (cig_words * 4 + 255) / 256 * 256;
		const size_t total = off_tasks + sizeof(SswTbTask) * batch.size();
		if (scratch->ensure(total)) return -1;
		std::vector<SswTbTask> bt(batch.size());
		for (size_t i = 0; i < batch.size(); ++i) bt[i] = tasks[batch[i]];
		uint8_t* base = scratch->as<uint8_t>();
		SswTbTask* d_tasks = reinterpret_cast<SswTbTask*>(base + off_tasks);
		uint32_t* d_cig = reinterpret_cast<uint32_t*>(base + off_cig);
		SSW_CUDA_OK(cudaMemcpyAsync(d_tasks, bt.data(), sizeof(SswTbTask) * bt.size(), cudaMemcpyHostToDevice, stream));
		SSW_CUDA_OK(cudaStreamSynchronize(stream));
		tm.start(stream);
		/* one launch per kernel shape, each on its own stream */
		int n_groups = 0;
		for (size_t g0 = 0; g0 < bt.size();) {
			size_t g1 = g0;
			while (g1 < bt.size() && batch_ring[g1] == batch_ring[g0]) ++g1;
			const int ring = batch_ring[g0], cnt = (int)(g1 - g0);
			cudaStream_t st = stream;
			if (n_groups > 0) {
				const int si = (n_groups - 1) % 3;
				if (!side[si]) SSW_CUDA_OK(cudaStreamCreateWithFlags(&side[si], cudaStreamNonBlocking));
				st = side[si];
			}
			const dim3 grid((cnt + SSW_TB_WARPS - 1) / SSW_TB_WARPS);
			if (ring < 0) {
				const int nw = -ring;
				size_t smem = 0;
				for (size_t x = g0; x < g1; ++x) {
					size_t ints = (size_t)(n * n + 15) / 16 * 4;
					int b2 = bt[x].bw;
					for (int w = 0; w < nw; ++w) { ints += 4 * (size_t)ssw_tb_ring_of(b2); b2 *= 2; }
					smem = std::max(smem, ints * sizeof(int32_t));
				}
				auto kern = d_mat ? ssw_banded_spec_kernel<false> : ssw_banded_spec_kernel<true>;
				if (ssw_ensure_dyn_smem(reinterpret_cast<const void*>(kern), smem)) return -1;
				if (carve && ssw_prefer_max_smem(reinterpret_cast<const void*>(kern))) return -1;
				ssw_launch(kern, dim3((unsigned)cnt), dim3(nw * 32), smem, st, d_tasks + g0, cnt, d_q, d_r, d_mat, n, gapO, gapE, base, d_cig, nw);
			} else if (ring) {
				const size_t smem = (size_t)SSW_TB_WARPS * 4 * (size_t)ring * sizeof(int32_t) + (size_t)n * n + 16;
				auto kern = d_mat ? ssw_banded_smem_kernel<false> : ssw_banded_smem_kernel<true>;
				if (ssw_ensure_dyn_smem(reinterpret_cast<const void*>(kern), smem)) return -1;
				if (carve && ssw_prefer_max_smem(reinterpret_cast<const void*>(kern))) return -1;
				ssw_launch(kern, grid, dim3(SSW_TB_THREADS), smem, st, d_tasks + g0, cnt, d_q, d_r, d_mat, n, gapO, gapE, base, d_cig, ring);
			} else {
				ssw_launch(d_mat ? ssw_banded_kernel<false> : ssw_banded_kernel<true>, grid, dim3(SSW_TB_THREADS), 0, st, d_tasks + g0, cnt, d_q, d_r, d_mat, n, gapO, gapE,
				           base, reinterpret_cast<int32_t*>(base + off_rows), d_cig);
			}
			SSW_CUDA_OK(cudaGetLastError());
			*launches += 1;
			++n_groups;
			g0 = g1;
		}
		for (int si = 0; si < 3 && si < n_groups - 1; ++si) SSW_CUDA_OK(cudaStreamSynchronize(side[si]));
		*ms_acc += tm.stop(stream);
		SSW_CUDA_OK(cudaMemcpyAsync(bt.data(), d_tasks, sizeof(SswTbTask) * bt.size(), cudaMemcpyDeviceToHost, stream));
		SSW_CUDA_OK(cudaStreamSynchronize(stream));
		/* bring back only the words the finished paths use: pack them densely into the (now free) direction area */
		std::vector<int64_t> dense_off(bt.size(), 0);
		size_t dense_words = 0;
		{
			std::vector<SswTbTask> pk(bt);
			for (size_t i = 0; i < pk.size(); ++i) {
				dense_off[i] = (int64_t)dense_words;
				pk[i].row_off = (int64_t)dense_words;
				if (pk[i].status == SSW_TB_OK) dense_words += (size_t)pk[i].cig_len;
			}
			if (dense_words * 4 > off_rows) {
				/* (pathological paths with a run per base) no room to pack: copy the worst-case buffers as they are */
				for (size_t i = 0; i < bt.size(); ++i) dense_off[i] = bt[i].cig_off;
				cig_host.resize(cig_words + 1);
				SSW_CUDA_OK(cudaMemcpyAsync(cig_host.data(), base + off_cig, cig_words * 4, cudaMemcpyDeviceToHost, stream));
				SSW_CUDA_OK(cudaStreamSynchronize(stream));
				dense_words = 0;
			} else cig_host.resize(dense_words + 1);
			if (dense_words > 0) {
				SSW_CUDA_OK(cudaMemcpyAsync(d_tasks, pk.data(), sizeof(SswTbTask) * pk.size(), cudaMemcpyHostToDevice, stream));
				ssw_launch(ssw_cigar_pack_kernel, dim3((unsigned)pk.size()), dim3(128), 0, stream, (const SswTbTask*)d_tasks, (int)pk.size(),
				           (const uint32_t*)d_cig, reinterpret_cast<uint32_t*>(base));
				SSW_CUDA_OK(cudaGetLastError());
				*launches += 1;
				SSW_CUDA_OK(cudaMemcpyAsync(cig_host.data(), base, dense_words * 4, cudaMemcpyDeviceToHost, stream));
				SSW_CUDA_OK(cudaStreamSynchronize(stream));
			}
		}
		if (getenv("SSW_TRACE")) {
			double f = 0, w = 0, s = 0; int nf = 0; long long fmax = 0, wmax = 0;
			for (const SswTbTask& x : bt) { f += (double)x.dbg_fill; fmax = std::max<long long>(fmax, x.dbg_fill); if (x.dbg_walk) { w += (double)x.dbg_walk; s += (double)x.dbg_score; wmax = std::max<long long>(wmax, x.dbg_walk); ++nf; } }
			long long t0min = 0x7fffffffffffffffLL, t0max = 0;
			for (const SswTbTask& x : bt) if (x.dbg_t0) { t0min = std::min<long long>(t0min, x.dbg_t0); t0max = std::max<long long>(t0max, x.dbg_t0); }
			fprintf(stderr, "[libssw-b200 trace] traceback round: %zu tasks in %d launches | fill avg %.0f max %lld clk | %d finished: walk avg %.0f max %lld, rescore avg %.0f clk | task starts spread over %.2f ms\n",
			        bt.size(), n_groups, f / bt.size(), fmax, nf, nf ? w / nf : 0.0, wmax, nf ? s / nf : 0.0, t0max > 0 ? (double)(t0max - t0min) * 1e-6 : 0.0);
		}
		std::vector<size_t> next;
		for (size_t i = 0; i < batch.size(); ++i) {
			SswTbTask& t = tasks[batch[i]];
			t = bt[i];
			const int full = t.ref_len > t.read_len ? t.ref_len : t.read_len;
			if (t.status == SSW_TB_WIDER) { t.bw *= 2; next.push_back(batch[i]); }
			else if (t.status == SSW_TB_OK) { if (emit(batch[i], cig_host.data() + dense_off[i], t.cig_len, 0)) return -1; }
			else if (t.status == SSW_TB_ERROR) { if (emit(batch[i], nullptr, 0, 1)) return -1; }
			else {                                                /* score mismatch: one retry at full band (ssw.c:952-956) */
				if (t.init_bw >= full) { if (emit(batch[i], nullptr, 0, 1)) return -1; }
				else { t.bw = t.init_bw = full; t.max = 0; t.max_i = 0; t.max_j = 0; next.push_back(batch[i]); }
			}
		}
		next.insert(next.end(), rest.begin(), rest.end());
		active.swap(next);
	}
	return 0;
}

#endif /* SSW_TRACEBACK_CUH */
