/*
 * ssw_text.cuh -- sequences given as text: letter -> code translation, reverse complement and the padded reference
 * layout are produced on the device (SURVEY 8(f) ranks 2 and 4).
 *
 * The reference's CLI translates every sequence on the host with a 128-entry table before each ssw_init / ssw_align
 * (main.c:476, :504: nt_table / aa_table) and builds the reverse complement of a read as text first (reverse_comple,
 * main.c:95-116: A<->T, C<->G, N->N, lower case folded, anything else becomes byte 4) and translates that.  Here the
 * raw bytes are copied to the device once and one kernel writes
 *   - the query codes, and behind them (optionally) the codes of every query's reverse complement,
 *   - the references in the engine's layout  [64 x null] codes [64 x null]  with null = n.
 */
#ifndef SSW_TEXT_CUH
#define SSW_TEXT_CUH

#include "ssw_common.cuh"

/* complement of one base as the reference's rc_table gives it (main.c:95-104) */
__device__ static __forceinline__ int ssw_rc_letter(int c)
{
	switch (c) {
	case 'A': case 'a': return 'T';
	case 'C': case 'c': return 'G';
	case 'G': case 'g': return 'C';
	case 'T': case 't': case 'U': case 'u': return 'A';
	case 'N': case 'n': return 'N';
	default: return 4;
	}
}

struct SswTextArgs {
	int64_t q_bytes;        /* total query letters */
	int64_t r_bytes;        /* total reference letters */
	int32_t n_q, n_r;
	int32_t add_rc;         /* also write the reverse complements behind the forward queries */
	int32_t pad_;
};

/* table: 128 codes in constant-like global memory; q_off / r_off: n+1 offsets into the texts; r_dst: offset of every
 * reference's first code in the padded array (the pads are filled by a memset before this kernel). */
__global__ void __launch_bounds__(256)
ssw_translate_kernel(SswTextArgs A, const uint8_t* __restrict__ q_text, const int64_t* __restrict__ q_off,
                     const uint8_t* __restrict__ r_text, const int64_t* __restrict__ r_off, const int64_t* __restrict__ r_dst,
                     const int8_t* __restrict__ table, int8_t* __restrict__ q_codes, int8_t* __restrict__ r_codes)
{
	__shared__ int8_t tab[128];
	if (threadIdx.x < 128) tab[threadIdx.x] = table[threadIdx.x];
	__syncthreads();
	const int64_t stride = (int64_t)gridDim.x * blockDim.x;
	const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	for (int64_t i = t0; i < A.q_bytes; i += stride) q_codes[i] = tab[q_text[i] & 127];
	if (A.add_rc) {
		/* letter i of the rc block belongs to query k (binary search over the offsets) at position p; it is the
		 * complement of letter len-1-p of that query */
		for (int64_t i = t0; i < A.q_bytes; i += stride) {
			int lo = 0, hi = A.n_q;
			while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (q_off[mid] <= i) lo = mid; else hi = mid; }
			const int64_t beg = q_off[lo], end = q_off[lo + 1];
			const int c = ssw_rc_letter((int)q_text[end - 1 - (i - beg)]);
			q_codes[A.q_bytes + i] = tab[c & 127];
		}
	}
	for (int64_t i = t0; i < A.r_bytes; i += stride) {
		int lo = 0, hi = A.n_r;
		while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (r_off[mid] <= i) lo = mid; else hi = mid; }
		r_codes[r_dst[lo] + (i - r_off[lo])] = tab[r_text[i] & 127];
	}
}

/* References delivered as packed codes (SURVEY 8(f) rank 4: the CLI's nucleotide codes are 0..4, main.c:84-93, i.e. 4 bits, or 2 bits
 * for N-free sequences): `packed` is the bit stream of the concatenated references, base i at bits [i*bits, i*bits + bits)
 * (low bits first), unpacked here into the engine's padded 1-byte layout.  The resident layout stays one byte per base on
 * purpose: the fill kernel is bound by the ALU pipe and a per-step nibble extract costs ALU slots (tools/microbench.cu:
 * letter fetch); the packing halves / quarters what crosses PCIe and what the caller keeps in host memory. */
__global__ void __launch_bounds__(256)
ssw_unpack_kernel(int64_t r_bases, int32_t n_r, int32_t bits, const uint8_t* __restrict__ packed, const int64_t* __restrict__ r_off,
                  const int64_t* __restrict__ r_dst, int8_t* __restrict__ r_codes)
{
	const int64_t stride = (int64_t)gridDim.x * blockDim.x;
	const unsigned mask = (1u << bits) - 1u;
	for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < r_bases; i += stride) {
		int lo = 0, hi = n_r;
		while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (r_off[mid] <= i) lo = mid; else hi = mid; }
		const int64_t bit = i * bits;
		r_codes[r_dst[lo] + (i - r_off[lo])] = (int8_t)((packed[bit >> 3] >> (bit & 7)) & mask);
	}
}

#endif /* SSW_TEXT_CUH */
