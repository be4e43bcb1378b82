// tools/microbench.cu -- issue-rate probe for the instructions the fill kernel is made of (H100, sm_90a).
// For each op: every warp runs ILP independent chains of the op in a long unrolled loop; cycles are read with
// clock64() around the loop; reported figure = warp-instructions per clock per SM with WARPS resident warps.
// Output: one JSON object on stdout (kept under profiles/ as dpx_peak.json).
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include <cuda_fp16.h>

#define ITERS 2048
#define ILP 8

template <int OP>
__device__ __forceinline__ uint32_t apply(uint32_t a, uint32_t b, uint32_t c, int lane)
{
	if (OP == 0) return __viaddmax_s16x2(a, b, c);
	if (OP == 1) return __viaddmax_s16x2_relu(a, b, c);
	if (OP == 2) return __vmaxs2(a, b);
	if (OP == 3) return __vimax3_s16x2(a, b, c);
	if (OP == 4) return __vadd2(a, b);
	if (OP == 5) return a * b + c;                       // IMAD
	if (OP == 6) return __shfl_up_sync(0xffffffffu, a, 1);
	if (OP == 7) return (a & b) ^ c;                     // LOP3
	if (OP == 8) return a + b + c;                       // IADD3
	if (OP == 9) { uint32_t d; asm("max.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b)); return d; }   // HMNMX2
	return a;
}

template <int OP>
__global__ void probe(uint32_t* out, long long* cyc, uint32_t seed)
{
	uint32_t v[ILP];
	const int lane = threadIdx.x & 31;
#pragma unroll
	for (int i = 0; i < ILP; ++i) v[i] = seed * (i + 1) + threadIdx.x;
	uint32_t b = seed | 1, c = seed >> 3;
	__syncthreads();
	long long t0 = clock64();
#pragma unroll 1
	for (int it = 0; it < ITERS; ++it) {
#pragma unroll
		for (int u = 0; u < 4; ++u)
#pragma unroll
			for (int i = 0; i < ILP; ++i) v[i] = apply<OP>(v[i], OP == 5 ? b : v[(i + 1) % ILP], OP == 5 ? c : v[(i + 3) % ILP], lane);
	}
	long long t1 = clock64();
	uint32_t acc = 0;
#pragma unroll
	for (int i = 0; i < ILP; ++i) acc ^= v[i];
	out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
	if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// mixed: per iteration A DPX ops and B IMADs on independent chains -> does the second pipe add throughput?
template <int NA, int NB>
__global__ void probe_mix(uint32_t* out, long long* cyc, uint32_t seed)
{
	uint32_t va[8], vb[8];
#pragma unroll
	for (int i = 0; i < 8; ++i) { va[i] = seed * (i + 1) + threadIdx.x; vb[i] = seed * (i + 9) + threadIdx.x; }
	uint32_t b = seed | 1, c = seed >> 3;
	__syncthreads();
	long long t0 = clock64();
#pragma unroll 1
	for (int it = 0; it < ITERS; ++it) {
#pragma unroll
		for (int u = 0; u < 4; ++u) {
#pragma unroll
			for (int i = 0; i < NA; ++i) va[i] = __viaddmax_s16x2(va[i], va[(i + 1) % NA], va[(i + 3) % NA]);
#pragma unroll
			for (int i = 0; i < NB; ++i) vb[i] = vb[i] * b + c;
		}
	}
	long long t1 = clock64();
	uint32_t acc = 0;
#pragma unroll
	for (int i = 0; i < 8; ++i) acc ^= va[i] ^ vb[i];
	out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
	if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// mixed: NA DPX ops and NB packed-half maxima (HMNMX2, FMA-side pipe) per iteration on independent chains
template <int NA, int NB>
__global__ void probe_mix_h(uint32_t* out, long long* cyc, uint32_t seed)
{
	uint32_t va[8], vb[8];
#pragma unroll
	for (int i = 0; i < 8; ++i) { va[i] = seed * (i + 1) + threadIdx.x; vb[i] = (seed * (i + 9) + threadIdx.x) & 0x3fff3fffu; }
	__syncthreads();
	long long t0 = clock64();
#pragma unroll 1
	for (int it = 0; it < ITERS; ++it) {
#pragma unroll
		for (int u = 0; u < 4; ++u) {
#pragma unroll
			for (int i = 0; i < NA; ++i) va[i] = __viaddmax_s16x2(va[i], va[(i + 1) % NA], va[(i + 3) % NA]);
#pragma unroll
			for (int i = 0; i < NB; ++i) { uint32_t d; asm volatile("max.f16x2 %0, %1, %2;" : "=r"(d) : "r"(vb[i]), "r"(vb[(i + 1) % NB])); vb[i] = d; }
		}
	}
	long long t1 = clock64();
	uint32_t acc = 0;
#pragma unroll
	for (int i = 0; i < 8; ++i) acc ^= va[i] ^ vb[i];
	out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
	if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}


// ---- second-pipe probes (round 2): can packed-half adds on the FMA pipe run beside DPX maxima on the ALU pipe? ----
// Independent chains only (no cross-chain dependencies), so the figures are issue rates, not latencies.
__device__ __forceinline__ uint32_t hfma2_relu(uint32_t a, uint32_t one, uint32_t c)
{
	uint32_t d; asm volatile("fma.rn.relu.f16x2 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(one), "r"(c)); return d;
}
__device__ __forceinline__ uint32_t hfma2(uint32_t a, uint32_t one, uint32_t c)
{
	uint32_t d; asm volatile("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(one), "r"(c)); return d;
}
__device__ __forceinline__ uint32_t hadd2(uint32_t a, uint32_t c)
{
	uint32_t d; asm volatile("add.rn.f16x2 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(c)); return d;
}

// NA ALU-pipe ops (VIMNMX.S16x2 when AOP == 0, VIADDMNMX.S16x2 when AOP == 1) and NB FMA-pipe ops
// (HFMA2.RELU when FOP == 0, HADD2 when FOP == 1, HFMA2 when FOP == 2, IMAD when FOP == 3) per inner step, every chain independent
template <int NA, int NB, int AOP, int FOP>
__global__ void probe_pipes(uint32_t* out, long long* cyc, uint32_t seed)
{
	uint32_t va[12], vb[12];
#pragma unroll
	for (int i = 0; i < 12; ++i) { va[i] = seed * (i + 1) + threadIdx.x; vb[i] = 0x3c003c00u + ((seed * (i + 9) + threadIdx.x) & 0x00ff00ffu); }
	const uint32_t one = 0x3c003c00u;                    // 1.0 | 1.0
	uint32_t b = (seed & 0x00030003u) | 0x00010001u, c = 0xbc00bc00u;      // c = -1.0 | -1.0
	asm volatile("" : "+r"(b), "+r"(c));
	__syncthreads();
	long long t0 = clock64();
#pragma unroll 1
	for (int it = 0; it < ITERS; ++it) {
#pragma unroll
		for (int u = 0; u < 4; ++u) {
#pragma unroll
			for (int i = 0; i < (NA > NB ? NA : NB); ++i) {
				if (i < NA) va[i] = AOP == 0 ? ((u & 1) ? __vmins2(va[i], c) : __vmaxs2(va[i], b)) : __viaddmax_s16x2(va[i], b, c);
				if (i < NB) vb[i] = FOP == 0 ? hfma2_relu(vb[i], one, c) : FOP == 1 ? hadd2(vb[i], c) : FOP == 2 ? hfma2(vb[i], one, c) : vb[i] * b + c;
			}
		}
		if (AOP == 0) b ^= (uint32_t)it;                 // keep the maxima from being folded
	}
	long long t1 = clock64();
	uint32_t acc = 0;
#pragma unroll
	for (int i = 0; i < 12; ++i) acc ^= va[i] ^ vb[i];
	out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
	if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// The recurrence itself, R rows per lane, no memory traffic: scores rotate through registers.
//   MODE 0: the shipped s16x2 formulation (5 ALU-pipe DPX ops per cell pair)
//   MODE 1: packed-half formulation: 4 HFMA2.RELU (FMA pipe) + 4 VIMNMX.S16x2 (ALU pipe) per cell pair; all values >= 0 so the
//           bit patterns order like integers
//   MODE 2: hybrid: X and H as in MODE 0 (VIADDMNMX.RELU, VIMNMX), the E/F updates with HFMA2.RELU + VIMNMX -- needs values that are
//           valid in both encodings, so it is an issue-rate probe only
template <int R, int MODE>
__global__ void probe_cells(uint32_t* out, long long* cyc, uint32_t seed)
{
	uint32_t Hd[R], E[R], s[R];
#pragma unroll
	for (int k = 0; k < R; ++k) {
		Hd[k] = 0; E[k] = 0;
		const int v = (int)((seed * (k + 3) + threadIdx.x * 7) % 5) - 2;
		if (MODE == 0) s[k] = ((uint32_t)v & 0xffffu) | ((uint32_t)v << 16);
		else { const __half hv = __int2half_rn(v); const uint32_t hb = (uint32_t)__half_as_ushort(hv); s[k] = hb | (hb << 16); }
	}
	const uint32_t one = 0x3c003c00u;
	uint32_t negO = MODE == 0 ? 0xfffdfffdu : 0xc200c200u;            // -3
	uint32_t negE = MODE == 0 ? 0xffffffffu : 0xbc00bc00u;            // -1
	asm volatile("" : "+r"(negO), "+r"(negE));
	uint32_t F = 0, cm = 0, inH = 0;
	__syncthreads();
	long long t0 = clock64();
#pragma unroll 1
	for (int it = 0; it < ITERS; ++it) {
		uint32_t Hn[R];
		F = inH;
#pragma unroll
		for (int k = 0; k < R; ++k) {
			if (MODE == 0) {
				const uint32_t X = __viaddmax_s16x2_relu(Hd[k], s[k], E[k]);
				const uint32_t Xg = __vadd2(X, negO);
				E[k] = __viaddmax_s16x2(E[k], negE, Xg);
				Hn[k] = __vmaxs2(X, F);
				F = __viaddmax_s16x2(F, negE, Xg);
			} else if (MODE == 1) {
				const uint32_t t1 = hfma2_relu(Hd[k], one, s[k]);
				const uint32_t X = __vmaxs2(t1, E[k]);
				const uint32_t Xg = hfma2_relu(X, one, negO);
				E[k] = __vmaxs2(hfma2_relu(E[k], one, negE), Xg);
				Hn[k] = __vmaxs2(X, F);
				F = __vmaxs2(hfma2_relu(F, one, negE), Xg);
			} else {
				const uint32_t X = __viaddmax_s16x2_relu(Hd[k], s[k], E[k]);
				const uint32_t Xg = hfma2_relu(X, one, negO);
				E[k] = __vmaxs2(hfma2_relu(E[k], one, negE), Xg);
				Hn[k] = __vmaxs2(X, F);
				F = __vmaxs2(hfma2_relu(F, one, negE), Xg);
			}
		}
		uint32_t m = __vimax3_s16x2(Hn[0], Hn[1], Hn[2]);
#pragma unroll
		for (int k = 3; k + 1 < R; k += 2) m = __vimax3_s16x2(m, Hn[k], Hn[k + 1]);
		cm = __vmaxs2(cm, m);
		Hd[0] = inH;
#pragma unroll
		for (int k = 1; k < R; ++k) Hd[k] = Hn[k - 1];
		inH = Hn[R - 1] ^ (uint32_t)(it & 1);
		// rotate the scores so that nothing is loop-invariant
		const uint32_t s0 = s[0];
#pragma unroll
		for (int k = 0; k + 1 < R; ++k) s[k] = s[k + 1];
		s[R - 1] = s0;
	}
	long long t1 = clock64();
	uint32_t acc = cm ^ F;
#pragma unroll
	for (int k = 0; k < R; ++k) acc ^= E[k] ^ Hd[k];
	out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
	if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// The loop body of the fill kernel in isolation (R rows per lane, one column per step): profile rows from shared memory
// (LDS.128), three SHFL.UP hand-offs, the cell updates and the lane's column maximum.
//   FORM 0: shipped: 5 ALU-pipe ops per cell pair (VIADDMNMX.RELU, VIADD.16x2, 2 x VIADDMNMX, VIMNMX)
//   FORM 1: biased values (every stored value >= 0, so a packed 16x2 add is an exact 32-bit add): Hd+s and X-gapO as IMAD on the
//           FMA pipe, X = VIMNMX3(t, E, floor), E'/F' = VIADDMNMX, H = VIMNMX: 4 ALU + 2 FMA per cell pair
//   FORM 2: biased values, all four adds as IMAD, four maxima on the ALU pipe: 4 ALU + 4 FMA per cell pair
template <int R, int FORM>
__global__ void probe_body(uint32_t* out, long long* cyc, uint32_t seed)
{
	__shared__ __align__(16) uint32_t prof[4 * 32 * R];
	const int lane = threadIdx.x & 31;
	for (int i = threadIdx.x; i < 4 * 32 * R; i += blockDim.x) {
		const int v = (int)((seed * (i + 3)) % 5) - 2;
		uint32_t w = ((uint32_t)v & 0xffffu) | ((uint32_t)v << 16);
		if (FORM != 0 && v < 0) w -= 0x10000u;           // carry compensation of the packed 32-bit add
		prof[i] = w;
	}
	__syncthreads();
	const uint32_t B = FORM == 0 ? 0u : 0x02000200u;      // bias 512 per half
	uint32_t Hd[R], E[R];
#pragma unroll
	for (int k = 0; k < R; ++k) { Hd[k] = B; E[k] = B; }
	uint32_t negO = FORM == 0 ? 0xfffdfffdu : (uint32_t)(-(int)(3u * 0x10001u));
	uint32_t negE = 0xffffffffu;                          // -1 | -1 (VIADDMNMX operand)
	uint32_t negE32 = (uint32_t)(-(int)(0x10001u));
	uint32_t one = seed - 12344u /* == 1 at run time, unknown to the compiler: keeps the packed adds IMADs */, keep = lane == 0 ? 0u : 1u, floorB = B, top_add = lane == 0 ? B : 0u;
	asm volatile("" : "+r"(negO), "+r"(negE), "+r"(one), "+r"(floorB), "+r"(negE32));
	asm volatile("" : "+r"(keep), "+r"(top_add));
	uint32_t outH = B, outF = B, outC = B, best = 0;
	long long t0 = clock64();
#pragma unroll 1
	for (int it = 0; it < ITERS; it += 4) {
#pragma unroll
		for (int u = 0; u < 4; ++u) {
			const uint32_t inH = __shfl_up_sync(0xffffffffu, outH, 1) * keep + top_add;
			uint32_t F = __shfl_up_sync(0xffffffffu, outF, 1) * keep + top_add;
			const uint32_t inC = __shfl_up_sync(0xffffffffu, outC, 1) * keep + top_add;
			const int letter = (it + u + (int)(best & 1u)) & 3;
			uint32_t s[R], Hn[R];
#pragma unroll
			for (int q = 0; q < R / 4; ++q) {
				const uint4 v = *reinterpret_cast<const uint4*>(&prof[letter * 32 * R + q * 128 + lane * 4]);
				s[4 * q] = v.x; s[4 * q + 1] = v.y; s[4 * q + 2] = v.z; s[4 * q + 3] = v.w;
			}
#pragma unroll
			for (int k = 0; k < R; ++k) {
				if (FORM == 0) {
					const uint32_t X = __viaddmax_s16x2_relu(Hd[k], s[k], E[k]);
					const uint32_t Xg = __vadd2(X, negO);
					E[k] = __viaddmax_s16x2(E[k], negE, Xg);
					Hn[k] = __vmaxs2(X, F);
					F = __viaddmax_s16x2(F, negE, Xg);
				} else if (FORM == 1) {
					const uint32_t t = Hd[k] * one + s[k];
					const uint32_t X = __vimax3_s16x2(t, E[k], floorB);
					const uint32_t Xg = X * one + negO;
					E[k] = __viaddmax_s16x2(E[k], negE, Xg);
					Hn[k] = __vmaxs2(X, F);
					F = __viaddmax_s16x2(F, negE, Xg);
				} else {
					const uint32_t t = Hd[k] * one + s[k];
					const uint32_t X = __vimax3_s16x2(t, E[k], floorB);
					const uint32_t Xg = X * one + negO;
					E[k] = __vmaxs2(E[k] * one + negE32, Xg);
					Hn[k] = __vmaxs2(X, F);
					F = __vmaxs2(F * one + negE32, Xg);
				}
			}
			uint32_t m = __vimax3_s16x2(Hn[0], Hn[1], Hn[2]);
#pragma unroll
			for (int k = 3; k + 1 < R; k += 2) m = __vimax3_s16x2(m, Hn[k], Hn[k + 1]);
			if (((R - 3) & 1) != 0) m = __vmaxs2(m, Hn[R - 1]);
			outC = __vmaxs2(m, inC);
			const uint32_t nb = __vmaxs2(best, m);
			if (nb != best) best = nb;
			Hd[0] = inH;
#pragma unroll
			for (int k = 1; k < R; ++k) Hd[k] = Hn[k - 1];
			outH = Hn[R - 1];
			outF = F;
		}
	}
	long long t1 = clock64();
	uint32_t acc = best ^ outC ^ outF;
#pragma unroll
	for (int k = 0; k < R; ++k) acc ^= E[k] ^ Hd[k];
	out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
	if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// Reference-letter fetch A/B (north_star: "reference bases streamed from HBM with coalesced 128-bit loads"; the shipped kernel
// issues one LDG.U8 per lane and step, served by L1).  The shipped cell formulation with
//   LOADV 0: one byte load per step (as shipped)
//   LOADV 1: one 64-bit load per 8 steps + a byte extract per step (PRMT/SHF on the ALU pipe -- the busy one)
//   LOADV 2: one 128-bit load per 16 steps + byte extracts
template <int R, int LOADV>
__global__ void probe_letters(uint32_t* out, long long* cyc, uint32_t seed, const uint8_t* __restrict__ refbuf)
{
	__shared__ __align__(16) uint32_t prof[5 * 32 * R];
	const int lane = threadIdx.x & 31;
	for (int i = threadIdx.x; i < 5 * 32 * R; i += blockDim.x) {
		const int v = (int)((seed * (i + 3)) % 5) - 2;
		prof[i] = ((uint32_t)v & 0xffffu) | ((uint32_t)v << 16);
	}
	__syncthreads();
	uint32_t Hd[R], E[R];
#pragma unroll
	for (int k = 0; k < R; ++k) { Hd[k] = 0; E[k] = 0; }
	uint32_t negO = 0xfffdfffdu, negE = 0xffffffffu, keep = lane == 0 ? 0u : 1u;
	asm volatile("" : "+r"(negO), "+r"(negE), "+r"(keep));
	uint32_t outH = 0, outF = 0, outC = 0, best = 0;
	const uint8_t* lp = refbuf + (size_t)(blockIdx.x * blockDim.x + threadIdx.x) / 8 * 4096 + 16 * (7 - (lane & 7));   // per-group window, 16-byte aligned
	long long t0 = clock64();
#pragma unroll 1
	for (int it = 0; it < ITERS; it += 16) {
		uint4 w4 = make_uint4(0, 0, 0, 0);
		if (LOADV == 2) w4 = *reinterpret_cast<const uint4*>(lp + (it & 2047));
#pragma unroll
		for (int h = 0; h < 2; ++h) {
			uint2 w2 = make_uint2(0, 0);
			if (LOADV == 1) w2 = *reinterpret_cast<const uint2*>(lp + ((it + 8 * h) & 2047));
			if (LOADV == 2) w2 = h ? make_uint2(w4.z, w4.w) : make_uint2(w4.x, w4.y);
#pragma unroll
			for (int u = 0; u < 8; ++u) {
				const uint32_t inH = __shfl_up_sync(0xffffffffu, outH, 1) * keep;
				uint32_t F = __shfl_up_sync(0xffffffffu, outF, 1) * keep;
				const uint32_t inC = __shfl_up_sync(0xffffffffu, outC, 1) * keep;
				int letter;
				if (LOADV == 0) letter = (int)lp[(it + 8 * h + u) & 2047];
				else letter = (int)(((u < 4 ? w2.x : w2.y) >> (8 * (u & 3))) & 0xffu);
				uint32_t s[R], Hn[R];
#pragma unroll
				for (int q = 0; q < R / 4; ++q) {
					const uint4 v = *reinterpret_cast<const uint4*>(&prof[letter * 32 * R + q * 128 + lane * 4]);
					s[4 * q] = v.x; s[4 * q + 1] = v.y; s[4 * q + 2] = v.z; s[4 * q + 3] = v.w;
				}
#pragma unroll
				for (int k = 0; k < R; ++k) {
					const uint32_t X = __viaddmax_s16x2_relu(Hd[k], s[k], E[k]);
					const uint32_t Xg = __vadd2(X, negO);
					E[k] = __viaddmax_s16x2(E[k], negE, Xg);
					Hn[k] = __vmaxs2(X, F);
					F = __viaddmax_s16x2(F, negE, Xg);
				}
				uint32_t m = __vimax3_s16x2(Hn[0], Hn[1], Hn[2]);
#pragma unroll
				for (int k = 3; k + 1 < R; k += 2) m = __vimax3_s16x2(m, Hn[k], Hn[k + 1]);
				if (((R - 3) & 1) != 0) m = __vmaxs2(m, Hn[R - 1]);
				outC = __vmaxs2(m, inC);
				const uint32_t nb = __vmaxs2(best, m);
				if (nb != best) best = nb;
				Hd[0] = inH;
#pragma unroll
				for (int k = 1; k < R; ++k) Hd[k] = Hn[k - 1];
				outH = Hn[R - 1];
				outF = F;
			}
		}
	}
	long long t1 = clock64();
	uint32_t acc = best ^ outC ^ outF;
#pragma unroll
	for (int k = 0; k < R; ++k) acc ^= E[k] ^ Hd[k];
	out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
	if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <class K>
static double run_letters(K kern, int threads, int sms)
{
	uint32_t* out; long long* cyc; uint8_t* refbuf;
	const size_t ref_bytes = (size_t)sms * threads / 8 * 4096 + 8192;
	cudaMalloc(&out, sizeof(uint32_t) * threads * sms);
	cudaMalloc(&cyc, sizeof(long long) * sms);
	cudaMalloc(&refbuf, ref_bytes);
	uint8_t* h = new uint8_t[ref_bytes];
	uint32_t x = 777;
	for (size_t i = 0; i < ref_bytes; ++i) { x = x * 1664525u + 1013904223u; h[i] = (uint8_t)((x >> 24) & 3); }
	cudaMemcpy(refbuf, h, ref_bytes, cudaMemcpyHostToDevice);
	delete[] h;
	kern<<<sms, threads>>>(out, cyc, 12345u, refbuf);
	kern<<<sms, threads>>>(out, cyc, 12345u, refbuf);
	cudaDeviceSynchronize();
	long long* hc = new long long[sms];
	cudaMemcpy(hc, cyc, sizeof(long long) * sms, cudaMemcpyDeviceToHost);
	double avg = 0;
	for (int i = 0; i < sms; ++i) avg += (double)hc[i];
	avg /= sms;
	delete[] hc;
	cudaFree(out); cudaFree(cyc); cudaFree(refbuf);
	return (double)(threads / 32) * ITERS / avg;          // warp-steps per clock per SM
}

template <class K>
static double run(K kern, int threads, int ops_per_iter, int sms, uint32_t seed = 12345u)
{
	uint32_t* out; long long* cyc;
	cudaMalloc(&out, sizeof(uint32_t) * threads * sms);
	cudaMalloc(&cyc, sizeof(long long) * sms);
	kern<<<sms, threads>>>(out, cyc, seed);
	kern<<<sms, threads>>>(out, cyc, seed);
	cudaDeviceSynchronize();
	long long* h = new long long[sms];
	cudaMemcpy(h, cyc, sizeof(long long) * sms, cudaMemcpyDeviceToHost);
	double avg = 0;
	for (int i = 0; i < sms; ++i) avg += (double)h[i];
	avg /= sms;
	delete[] h;
	cudaFree(out); cudaFree(cyc);
	const double warp_instr = (double)(threads / 32) * ITERS * ops_per_iter;
	return warp_instr / avg;          // warp-instructions per clock per SM
}

int main()
{
	cudaDeviceProp p;
	cudaGetDeviceProperties(&p, 0);
	const int sms = p.multiProcessorCount;
	int clk_khz = 0;
	cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
	printf("{\"device\": \"%s\", \"sms\": %d, \"max_sm_khz\": %d", p.name, sms, clk_khz);
	const char* names[] = {"VIADDMNMX.S16x2", "VIADDMNMX.S16x2.RELU", "VIMNMX.S16x2", "VIMNMX3.S16x2", "VIADD.16x2", "IMAD", "SHFL.UP", "LOP3", "IADD3"};
	for (int threads = 256; threads <= 1024; threads *= 2) {
		double r[9];
		r[0] = run(probe<0>, threads, 4 * ILP, sms);
		r[1] = run(probe<1>, threads, 4 * ILP, sms);
		r[2] = run(probe<2>, threads, 4 * ILP, sms);
		r[3] = run(probe<3>, threads, 4 * ILP, sms);
		r[4] = run(probe<4>, threads, 4 * ILP, sms);
		r[5] = run(probe<5>, threads, 4 * ILP, sms);
		r[6] = run(probe<6>, threads, 4 * ILP, sms);
		r[7] = run(probe<7>, threads, 4 * ILP, sms);
		r[8] = run(probe<8>, threads, 4 * ILP, sms);
		printf(", \"warp_instr_per_clk_per_sm_%dthr\": {", threads);
		for (int i = 0; i < 9; ++i) printf("%s\"%s\": %.3f", i ? ", " : "", names[i], r[i]);
		printf("}");
		if (threads == 1024) {
			const double m44 = run(probe_mix<4, 4>, threads, 4 * 8, sms);
			const double m62 = run(probe_mix<6, 2>, threads, 4 * 8, sms);
			const double m80 = run(probe_mix<8, 0>, threads, 4 * 8, sms);
			const double h80 = run(probe_mix_h<8, 0>, threads, 4 * 8, sms);
			const double h62 = run(probe_mix_h<6, 2>, threads, 4 * 8, sms);
			const double h44 = run(probe_mix_h<4, 4>, threads, 4 * 8, sms);
			const double h08 = run(probe<9>, threads, 4 * ILP, sms);
			printf(", \"mix_dpx_hmnmx2_1024thr\": {\"8+0\": %.3f, \"6+2\": %.3f, \"4+4\": %.3f, \"HMNMX2 alone\": %.3f}", h80, h62, h44, h08);
			printf(", \"mix_dpx_imad_1024thr\": {\"4+4\": %.3f, \"6+2\": %.3f, \"8+0\": %.3f}", m44, m62, m80);
			// fill kernel: 5.5 DPX ops per lane per two cells -> cells/clk/SM = rate * 32 lanes * 2 / 5.5

			// round 2: second-pipe probes
			printf(", \"pipes_1024thr\": {");
			printf("\"HFMA2.RELU alone x8\": %.3f", run(probe_pipes<0, 8, 0, 0>, threads, 4 * 8, sms));
			printf(", \"HADD2 alone x8\": %.3f", run(probe_pipes<0, 8, 0, 1>, threads, 4 * 8, sms));
			printf(", \"HFMA2 alone x8\": %.3f", run(probe_pipes<0, 8, 0, 2>, threads, 4 * 8, sms));
			printf(", \"IMAD alone x8\": %.3f", run(probe_pipes<0, 8, 0, 3>, threads, 4 * 8, sms));
			printf(", \"VIMNMX alone x8\": %.3f", run(probe_pipes<8, 0, 0, 0>, threads, 4 * 8, sms));
			printf(", \"VIADDMNMX alone x8\": %.3f", run(probe_pipes<8, 0, 1, 0>, threads, 4 * 8, sms));
			printf(", \"VIMNMX 8 + HFMA2.RELU 8\": %.3f", run(probe_pipes<8, 8, 0, 0>, threads, 4 * 16, sms));
			printf(", \"VIMNMX 9 + HFMA2.RELU 8\": %.3f", run(probe_pipes<9, 8, 0, 0>, threads, 4 * 17, sms));
			printf(", \"VIMNMX 8 + HFMA2.RELU 4\": %.3f", run(probe_pipes<8, 4, 0, 0>, threads, 4 * 12, sms));
			printf(", \"VIMNMX 8 + HADD2 8\": %.3f", run(probe_pipes<8, 8, 0, 1>, threads, 4 * 16, sms));
			printf(", \"VIADDMNMX 8 + HFMA2.RELU 8\": %.3f", run(probe_pipes<8, 8, 1, 0>, threads, 4 * 16, sms));
			printf(", \"VIADDMNMX 8 + IMAD 8\": %.3f", run(probe_pipes<8, 8, 1, 3>, threads, 4 * 16, sms));
			printf(", \"VIMNMX 8 + IMAD 8\": %.3f", run(probe_pipes<8, 8, 0, 3>, threads, 4 * 16, sms));
			printf("}");
			// the recurrence itself: warp-steps (one column of R rows) per clock per SM -> cell updates per clock per SM = x * 32 * 2 * R
			for (int thr = 256; thr <= 512; thr *= 2) {
				const double c0 = run(probe_cells<20, 0>, thr, 1, sms), c1 = run(probe_cells<20, 1>, thr, 1, sms), c2 = run(probe_cells<20, 2>, thr, 1, sms);
				const double k = 32.0 * 2.0 * 20.0 * sms * (clk_khz * 1e3) / 1e9;
				printf(", \"cells_R20_%dthr_gcups\": {\"s16x2 (shipped)\": %.1f, \"f16x2: 4 HFMA2.RELU + 4 VIMNMX\": %.1f, \"hybrid\": %.1f}", thr, c0 * k, c1 * k, c2 * k);
			}

			for (int thr = 256; thr <= 512; thr *= 2) {
				const double k = 32.0 * 2.0 * 20.0 * sms * (clk_khz * 1e3) / 1e9;
				const double b0 = run(probe_body<20, 0>, thr, 1, sms), b1 = run(probe_body<20, 1>, thr, 1, sms), b2 = run(probe_body<20, 2>, thr, 1, sms);
				printf(", \"fill_body_R20_%dthr_gcups\": {\"shipped: 5 ALU per cell pair\": %.1f, \"biased: 4 ALU + 2 IMAD\": %.1f, \"biased: 4 ALU + 4 IMAD\": %.1f}", thr, b0 * k, b1 * k, b2 * k);
			}
			{
				const double k = 32.0 * 2.0 * 20.0 * sms * (clk_khz * 1e3) / 1e9;
				printf(", \"letter_fetch_R20_512thr_gcups\": {\"LDG.U8 per step (shipped)\": %.1f, \"LDG.64 per 8 steps + byte extract\": %.1f, \"LDG.128 per 16 steps + byte extract\": %.1f}",
				       run_letters(probe_letters<20, 0>, 512, sms) * k, run_letters(probe_letters<20, 1>, 512, sms) * k, run_letters(probe_letters<20, 2>, 512, sms) * k);
			}
			const double cells_per_clk_sm = r[0] * 32.0 * 2.0 / 5.5;
			printf(", \"gcups_peak_5p5_ops_per_cellpair\": %.1f", cells_per_clk_sm * sms * (clk_khz * 1e3) / 1e9);
		}
	}
	printf("}\n");
	return 0;
}
