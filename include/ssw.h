/*
 * ssw.h -- C ABI of the H100-native Smith-Waterman aligner (drop-in boundary).
 *
 * This header declares the same five entry points, the same result record and
 * the same CIGAR helpers as the SSW library's public header, so that existing
 * consumers (the `ssw_test` CLI, the C++ `Aligner`, the ctypes and JNI
 * wrappers) link against this library without source changes.  Each item
 * names the reference interface it replaces (paths are into the reference
 * tree, `src/`):
 *
 *   s_profile (opaque)   <- ssw.h:37-38   (struct _profile, ssw.c:115-123)
 *   s_align              <- ssw.h:55-66   (LP64 layout: 40 bytes, see below)
 *   ssw_init             <- ssw.h:86      (ssw.c:826-847)
 *   init_destroy         <- ssw.h:91      (ssw.c:849-853)
 *   ssw_align            <- ssw.h:126-134 (ssw.c:855-977)
 *   align_destroy        <- ssw.h:139     (ssw.c:979-982)
 *   mark_mismatch        <- ssw.h:157-164 (ssw.c:1019-1074)
 *   encoded_ops          <- ssw.h:34      (ssw.c:127-160)
 *   to_cigar_int / cigar_int_to_op / cigar_int_to_len <- ssw.h:171-190
 *
 * The implementation behind these symbols is CUDA (sm_90a); there is no CPU
 * compute path.  A call made on a machine without a usable GPU fails loudly
 * (message on stderr, NULL result) instead of falling back.
 *
 * The batched entry points (many pairs per call, which is what a GPU needs)
 * are declared in ssw_batch.h.
 */
#ifndef SSW_H
#define SSW_H

#include <stdio.h>
#include <stdint.h>
#include <string.h>

/* The reference header pulls an SSE header into every consumer translation
 * unit (ssw.h:18-22).  Nothing in this ABI needs it, but some consumers rely
 * on the transitive include, so keep it where it is available. */
#if defined(__ARM_NEON)
/* no vector header needed by this ABI */
#elif defined(__SSE2__) && !defined(__CUDACC__)
#include <emmintrin.h>
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* BAM operation letters by op code, and the BAM length shift. */
#define MAPSTR "MIDNSHP=X"
#ifndef BAM_CIGAR_SHIFT
#define BAM_CIGAR_SHIFT 4u
#endif

/* 128-entry table: ASCII CIGAR letter -> BAM op code (M0 I1 D2 N3 S4 H5 P6 =7 X8). */
extern const uint8_t encoded_ops[];

/* Query profile handle.  Opaque: holds the query, the scoring matrix, the
 * score-width policy and (lazily) the device-side copies. */
struct _profile;
typedef struct _profile s_profile;

/*
 * Alignment result.  All coordinates are 0-based and inclusive.
 *   score1       best local alignment score
 *   score2       best score among reference columns outside the mask window
 *                around ref_end1 (0 when maskLen < 15)
 *   ref_begin1   start of the best alignment on the reference (-1: not computed)
 *   ref_end1     end of the best alignment on the reference
 *   read_begin1  start on the query (-1: not computed)
 *   read_end1    end on the query
 *   ref_end2     reference column of score2 (-1 when maskLen < 15)
 *   cigar        BAM-packed CIGAR words (length << 4 | op), libc heap, or NULL
 *   cigarLen     number of CIGAR words
 *   flag         0 ok; 1 traceback failed (no cigar); 2 begin search fell short
 * Offsets on LP64: 0,2,4,8,12,16,20,24,32,36; sizeof == 40.
 */
typedef struct {
	uint16_t score1;
	uint16_t score2;
	int32_t ref_begin1;
	int32_t ref_end1;
	int32_t	read_begin1;
	int32_t read_end1;
	int32_t ref_end2;
	uint32_t* cigar;
	int32_t cigarLen;
	uint16_t flag;
} s_align;

/*
 * Build a query profile.
 *   read        query as codes in [0, n); borrowed, must outlive the profile
 *   readLen     >= 1
 *   mat         n*n substitution scores, row = reference code, column = query code; borrowed
 *   score_size  0: 8-bit score semantics only (scores < 255 - |min(mat)|),
 *               1: 16-bit semantics only, 2: 8-bit first, 16-bit on overflow
 */
s_profile* ssw_init (const int8_t* read, const int32_t readLen, const int8_t* mat, const int32_t n, const int8_t score_size);

/* Release a profile made by ssw_init. */
void init_destroy (s_profile* p);

/*
 * Align the profiled query against one reference.
 *   ref, refLen   reference codes in [0, n); borrowed for the call
 *   weight_gapO   cost of the first base of a gap (positive)
 *   weight_gapE   cost of every further base of a gap (positive)
 *   flag          0: scores and end positions only.
 *                 bit 0x08: also begin positions.
 *                 bits 0x01/0x02/0x04: also CIGAR; 0x02 only if score1 >= filters;
 *                 0x04 only if both spans <= filterd.  (flag == 2 with
 *                 score1 < filters returns ends only.)
 *   maskLen       half-width of the window masked around ref_end1 for score2;
 *                 values < 15 disable score2 (a notice is printed on stderr)
 * Returns a heap record to be released with align_destroy, or NULL on error
 * (8-bit overflow with score_size 0; no profile; no usable GPU).
 */
s_align* ssw_align (const s_profile* prof,
					const int8_t* ref,
					int32_t refLen,
					const uint8_t weight_gapO,
					const uint8_t weight_gapE,
					const uint8_t flag,
					const uint16_t filters,
					const int32_t filterd,
					const int32_t maskLen);

/* Release a result made by ssw_align (or ssw_align_batch). */
void align_destroy (s_align* a);

/*
 * Rewrite an M/I/D CIGAR as =/X/I/D with soft clips and return the edit
 * distance (mismatches + gap bases).  *cigar is freed and replaced by a new
 * libc-heap array; *cigarLen is updated.
 */
int32_t mark_mismatch (int32_t ref_begin1,
					   int32_t read_begin1,
					   int32_t read_end1,
					   const int8_t* ref,
					   const int8_t* read,
					   int32_t readLen,
					   uint32_t** cigar,
					   int32_t* cigarLen);

/* Pack (length, op letter) into a BAM CIGAR word. */
static inline uint32_t to_cigar_int (uint32_t length, unsigned char op_letter) {
	return (length << BAM_CIGAR_SHIFT) | (encoded_ops[op_letter]);
}

/* Op letter of a BAM CIGAR word (codes above 8 read as 'M'). */
static inline char cigar_int_to_op (uint32_t cigar_int) {
	return (cigar_int & 0xfU) > 8 ? 'M' : MAPSTR[cigar_int & 0xfU];
}

/* Length of a BAM CIGAR word. */
static inline uint32_t cigar_int_to_len (uint32_t cigar_int) {
	return cigar_int >> BAM_CIGAR_SHIFT;
}

#ifdef __cplusplus
}
#endif

#endif /* SSW_H */
