/*
 * ssw_common.cuh -- shared device/host definitions of the H100 aligner.
 *
 * Terminology (follows the reference, src/ssw.c):
 *   query / read   the profiled sequence (rows of the DP matrix)
 *   reference      the target sequence (columns)
 *   byte / word    the reference's two score semantics (sw_sse2_byte :197-386,
 *                  sw_sse2_word :412-588).  Here both are computed in packed
 *                  s16x2 DPX arithmetic; the semantics only decide the number
 *                  of pad rows (16- vs 8-row granularity), the overflow limit
 *                  and two constants of the second-best scan.
 *   pair-task      two alignments that share a reference and ride in the two
 *                  16-bit halves of every register (A = low half, B = high).
 *   item           one (pair-task, reference chunk) unit of fill work.
 */
#ifndef SSW_COMMON_CUH
#define SSW_COMMON_CUH

#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#ifdef SSW_CPU_EMU
/* tests only: compile the kernels for the CPU fiber emulator (tests/cuda_emu) */
#include "cuda_emu.h"
#else
#include <cuda_runtime.h>
#define SSW_DYN_SMEM(T, name) extern __shared__ __align__(16) unsigned char name##_raw_[]; T* name = reinterpret_cast<T*>(name##_raw_)
#endif

#define SSW_CUDA_OK(expr)                                                                        \
	do {                                                                                         \
		cudaError_t e_ = (expr);                                                                 \
		if (e_ != cudaSuccess) {                                                                 \
			fprintf(stderr, "[libssw-b200] CUDA error %s at %s:%d: %s\n", #expr, __FILE__,       \
			        __LINE__, cudaGetErrorString(e_));                                           \
			return -1;                                                                           \
		}                                                                                        \
	} while (0)

/* Launch helper: a plain function so that template-ids with commas work. */
template <class... KArgs, class... Args>
static inline void ssw_launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args)
{
#ifdef SSW_CPU_EMU
	(void)st;
	cuemu::run_grid(grid, block, smem, [&]() { kern(args...); });
#else
	kern<<<grid, block, smem, st>>>(args...);
#endif
}

/* spin-wait pause: the emulator's fibers are cooperative, so a waiting thread must yield */
#ifdef SSW_CPU_EMU
#define SSW_SPIN_PAUSE() cuemu::yield_now()
#define SSW_SPIN_TIGHT() cuemu::yield_now()
#else
#define SSW_SPIN_PAUSE() __nanosleep(64)     /* waits that are rarely entered (strip pipeline: the producer runs ahead) */
#define SSW_SPIN_TIGHT() ((void)0)           /* hand-offs on the critical path (traceback rows): a sleep would cost ~1 us per row */
#endif

/* ---- geometry constants ---------------------------------------------------- */
#define SSW_REF_PAD 64          /* null letters stored before and after every reference */
#define SSW_NEG16 (-32768)      /* score of dead rows / null letters: keeps H at exactly 0 */
#define SSW_CM_NONE ((int64_t)(-0x7fffffffffffffffLL - 1))   /* cm_off value: no column maxima are recorded */
#define SSW_ROW_UNARMED 0x3ffffffe  /* best-cell row of an item whose maximum lies before its armed range: the pair is re-done with arm 0 */
#define SSW_CM_BLOCK 64         /* columns per block of the block-maximum mode (CM == 2) of the fill kernel */

/* ---- packed s16x2 helpers --------------------------------------------------- */
__host__ __device__ static __forceinline__ uint32_t pack2(int lo, int hi)
{
	return ((uint32_t)lo & 0xffffu) | ((uint32_t)hi << 16);
}
__host__ __device__ static __forceinline__ int half_of(uint32_t v, int h)
{
	return h ? (int)(int16_t)(v >> 16) : (int)(int16_t)(v & 0xffffu);
}

/* ---- device-side descriptors -------------------------------------------------- */

/* One query as the fill kernel sees it: a slice of the concatenated code array,
 * read forwards (P1) or backwards from `off+len-1` (P2: reversed prefix, ssw.c:919). */
struct SswQuery {
	int32_t off;        /* offset of the first code in the concatenated query array */
	int32_t len;        /* number of real rows */
	int32_t lp;         /* rows including pad rows (multiple of 16 or 8) */
	int32_t rev;        /* 1: row j reads code[off + len - 1 - j] */
};

/* One unit of fill work: columns [p0, p1) of a pair-task in scan coordinates.
 * Forward: scan index == reference column.  Reverse: scan index s == column (cend - s). */
struct SswItem {
	SswQuery qa, qb;    /* qb.len == 0: half B is dead */
	int64_t ref_off;    /* offset of reference column 0 inside the padded reference array */
	int32_t ref_len;
	int32_t cend;       /* reverse pass: column of scan index 0 (= ref_end1); forward pass: `arm`, the first scan position whose
	                     * best cell gets its row recorded (0: all of them; see SSW_ROW_UNARMED) */
	int32_t p0, p1;     /* counted scan range */
	int32_t warm;       /* warm-up scan positions before p0 (state build-up, results discarded) */
	int32_t term_a;     /* reverse pass: stop once a column maximum equals this (score1); else -1 */
	int64_t cm_off;     /* offset (in uint32 words) of this pair-task's column-maximum row (block mode: of its row of
	                     * block maxima); SSW_CM_NONE: none.  May be negative for the re-fill items of the block mode. */
};

/* Per item and half: best cell in scan order = (max score, first scan index, smallest row). */
struct SswItemBest {
	int32_t score[2];
	int32_t pos[2];     /* scan index */
	int32_t row[2];
	int32_t p0, p1;     /* the item's counted scan range, copied for the resolve kernel */
};

/* One alignment as the resolve kernel sees it. */
struct SswAlnDesc {
	int32_t first_item; /* items [first_item, first_item + n_items) in scan order */
	int32_t n_items;
	int32_t half;       /* 0: A, 1: B */
	int32_t ref_len;
	int32_t read_len;
	int32_t word;       /* 0: byte semantics, 1: word semantics */
	int32_t limit;      /* byte: 255 - bias (score >= limit overflows); word: 32767 - max(mat) guard */
	int32_t mask_len;
	int64_t cm_off;     /* as in SswItem */
	int32_t scan_all;   /* 1: item records are not column-maximum summaries (strip-pipelined fill): scan every column */
	int32_t warm;       /* block mode: warm-up columns a re-fill of one block of this pair-task needs */
	int32_t byte_pad;   /* block mode, byte semantics filled on the word rows: pad rows of the byte padding that the fill left
	                     * out (the item's lp is the word padding); the resolve re-fills the columns they can change (DESIGN 2) */
};

/* Output of the resolve kernel (the reference's alignment_end[2], ssw.c:104-108, plus status). */
struct SswFillResult {
	int32_t score;      /* best score; 255 when byte semantics overflowed (ssw.c:360) */
	int32_t ref;        /* end_ref   */
	int32_t read;       /* end_read  */
	int32_t score2;
	int32_t ref2;
	int32_t overflow;   /* 1: byte overflow, 2: 16-bit head-room exhausted, 3: best cell before the armed range (row unknown: re-do) */
	int32_t pad_[2];
};

#endif /* SSW_COMMON_CUH */
