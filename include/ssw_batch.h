/*
 * ssw_batch.h -- batched C ABI of the H100-native aligner.
 *
 * The reference's API aligns one (query, reference) pair per blocking call
 * (ssw.h:126-134); its CLI loops over reads x references around that call
 * (main.c:462-532).  One pair exposes far too little parallelism for a GPU,
 * so the same computation is offered over a whole batch of independent pairs.
 * Every pair's answer is field-for-field what ssw_init(score_size) +
 * ssw_align(...) of ssw.h returns for that pair.
 *
 * All pointers are plain host pointers to caller-owned memory; no type of any
 * framework appears in this interface.  Functions return 0 on success and a
 * negative value on error (message on stderr).  There is no CPU compute path:
 * without a usable CUDA device ssw_engine_create fails.
 */
#ifndef SSW_BATCH_H
#define SSW_BATCH_H

#include <stdint.h>
#include "ssw.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ssw_engine ssw_engine;

/* Scoring and reporting parameters shared by all pairs of a batch; same meaning
 * as the arguments of ssw_init / ssw_align (ssw.h:86, :126-134). */
typedef struct {
	const int8_t* mat;      /* n*n scores, row = reference code, column = query code; NULL with query profiles resident */
	int32_t n;              /* alphabet size (codes are 0..n-1), n <= 64 */
	uint8_t gap_open;       /* weight_gapO */
	uint8_t gap_extend;     /* weight_gapE */
	uint8_t flag;           /* ssw_align flag */
	uint16_t filters;       /* ssw_align filters */
	int32_t filterd;        /* ssw_align filterd */
	int32_t mask_len;       /* ssw_align maskLen; negative: readLen / 2 per query (the CLI's choice, main.c:465) */
	int8_t score_size;      /* ssw_init score_size: 0 byte, 1 word, 2 byte then word */
} ssw_batch_params;

/* Fixed-size per-pair result; same fields as s_align with the CIGAR stored out of line. */
typedef struct {
	uint16_t score1, score2;
	int32_t ref_begin1, ref_end1, read_begin1, read_end1, ref_end2;
	int32_t cigar_off;      /* offset of this pair's words in the batch CIGAR pool, -1 if none */
	int32_t cigar_len;
	uint16_t flag;          /* s_align.flag */
	uint16_t status;        /* 0 ok; 1: ssw_align would have returned NULL (byte overflow with score_size 0) */
} ssw_batch_result;

/* Create an engine bound to CUDA device `device` (-1: current device). NULL on failure. */
ssw_engine* ssw_engine_create(int device);
void ssw_engine_destroy(ssw_engine* e);

/* Name of the device the engine runs on ("" if none). */
const char* ssw_engine_device_name(const ssw_engine* e);

/*
 * Make a set of sequences resident in device memory (host -> device copy).
 *   queries / refs     concatenated codes
 *   query_off/ref_off  n+1 offsets into the concatenations
 * Replaces any previously resident set.
 */
int ssw_engine_set_sequences(ssw_engine* e,
                             int32_t n_queries, const int8_t* queries, const int64_t* query_off,
                             int32_t n_refs, const int8_t* refs, const int64_t* ref_off);

/*
 * The same for sequences given as TEXT: the letters are translated to codes on the device with `table` (128 entries,
 * the reference CLI's nt_table / aa_table, main.c:72-93; bytes are masked to 7 bits), for an alphabet of n codes
 * (the n of the later align calls).  add_reverse_complement != 0 also makes every query's reverse complement resident,
 * as query number n_queries + k (complement on the letters as main.c:95-116 does it: A<->T, C<->G, N->N, other -> 4).
 */
int ssw_engine_set_sequences_text(ssw_engine* e,
                                  int32_t n_queries, const char* queries, const int64_t* query_off,
                                  int32_t n_refs, const char* refs, const int64_t* ref_off,
                                  const int8_t* table, int32_t n, int32_t add_reverse_complement);

/*
 * The same with the references delivered PACKED: `refs_packed` is the bit stream of the concatenated reference codes, base i at
 * bits [i*bits, i*bits + bits) (low bits first), bits = 4 (the CLI's nucleotide codes 0..4, main.c:84-93) or 2 (N-free
 * sequences); ref_off are offsets in BASES.  The stream is unpacked on the device; `n` is the alphabet size of the later
 * align calls.  Queries are plain codes.
 */
int ssw_engine_set_sequences_packed(ssw_engine* e,
                                    int32_t n_queries, const int8_t* queries, const int64_t* query_off,
                                    int32_t n_refs, const uint8_t* refs_packed, const int64_t* ref_off,
                                    int32_t bits, int32_t n);

/*
 * The same with every query given as a position-specific scoring matrix (PSSM, a query profile) instead of codes: row i of
 * query q holds the scores of query position i against the n reference letters, at pssm[(query_off[q] + i) * n + letter].
 *   query_off   n_queries + 1 offsets in ROWS; 1 <= n <= 64; references are codes 0 .. n-1 as for ssw_engine_set_sequences
 *   meaning     the record of query q against reference r is what the reference returns for ssw_init(read = {0, 1, .., L-1},
 *               readLen = L, mat = M, N = max(L, n), score_size) + ssw_align(r, ...) with M[c * N + i] = P[i][c] (c < n, i < L)
 *               and 0 elsewhere: every lookup mat[ref][read[i]] becomes P[i][ref], and the byte bias max(0, -min P) -- with it
 *               the byte-overflow limit 255 - bias -- belongs to each query
 *   calls       while profiles are resident, ssw_engine_align / _search / _search_all take params->mat == NULL and
 *               params->n == n (anything else returns -1); ssw_engine_mark_mismatch returns -1 (no query letters to compare)
 * Replaces any previously resident set; any set_sequences call after it makes query codes resident again.
 */
int ssw_engine_set_sequences_pssm(ssw_engine* e,
                                  int32_t n_queries, const int8_t* pssm, const int64_t* query_off, int32_t n,
                                  int32_t n_refs, const int8_t* refs, const int64_t* ref_off);

/*
 * Align pairs of resident sequences.
 *   pair_query / pair_ref   n_pairs indices; both NULL: the full grid, pair p = query p / n_refs x ref p % n_refs
 *   results                 n_pairs records (host memory)
 *   cigar_pool, pool_cap    optional pool receiving the CIGAR words (may be NULL when flag requests no CIGAR);
 *   pool_used               receives the number of words written
 */
int ssw_engine_align(ssw_engine* e, const ssw_batch_params* params,
                     int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                     ssw_batch_result* results,
                     uint32_t* cigar_pool, int64_t pool_cap, int64_t* pool_used);

/*
 * Top-k search of the resident queries against the resident references (full grid). Hits of query q are at
 * [q*k, q*k + n_hits[q]) of hit_ref / hits, in rank order; unused slots have hit_ref = -1.
 *   hit        a pair with score1 >= max(min_score, 1), or a pair with status 1 (score_size 0, byte overflow: its score is
 *              at least the byte limit; a hit whatever min_score is)
 *   rank       status-1 pairs first, then score1 descending, then reference index ascending (a total order: the result does
 *              not depend on the devices or on the path that ran)
 *   records    field for field what ssw_engine_align returns for that pair with the same params; begins and CIGARs (flag & 7)
 *              are computed for the hits only, into cigar_pool as ssw_engine_align fills it
 *   k          1 .. 1024
 * No record of the n_queries x n_refs grid crosses to the host: the k best of every query are selected on the device where
 * the grid path can run (scores-only planning on the device), on the host per block of queries otherwise.
 *   which pairs run where: the sequences qualify for the device path one by one -- a reference of at most 65,536 letters, a
 *              query whose padded rows one fill instance covers (640) and for which byte semantics are tried first.  Pairs of
 *              a qualifying query and a qualifying reference are computed and selected on the device (if they are at least
 *              "grid_min" pairs); the pairs of every other query, and of every query with every other reference, take the
 *              general path in blocks of at most 4 Mi pairs and are merged into the device's lists per query
 *              (ssw_engine_timing.leftover_pairs counts them).  One long reference costs its own column of the grid, not
 *              the device path.  Conditions on the call -- gap_open <= gap_extend, the "chunk" option -- still send every
 *              pair down the general path.
 *   size       a grid of more than 2^31 - 1 pairs, or one whose references need more scratch per query pair than a launch
 *              may take, is cut into grid tiles (contiguous runs of references), each run on the device; the k best of
 *              every tile are merged into each query's k best on the device, and the hit table still comes back in one copy.
 */
int ssw_engine_search(ssw_engine* e, const ssw_batch_params* params, int32_t k, int32_t min_score,
                      int32_t* hit_ref, ssw_batch_result* hits, int32_t* n_hits,
                      uint32_t* cigar_pool, int64_t pool_cap, int64_t* pool_used);

/*
 * Threshold search of the resident queries against the resident references (full grid): EVERY hit, not the k best.  The
 * size of the answer is known only at the end, so the library allocates it and hands back an opaque set; read it with
 * ssw_hit_set_view and release it with ssw_hit_set_destroy.
 *   hit        the rule of ssw_engine_search: status 1, or score1 >= max(min_score, 1)
 *   output     a sparse matrix in CSR form, one row per resident query (with reverse complements resident, 2 * n_queries
 *              rows, the reverse complements after the queries): row q's hits are [row_off[q], row_off[q + 1]) of hit_ref
 *              (the caller's reference index) and hits; row_off has n_rows + 1 entries
 *   order      within a row, ascending reference index -- so the whole output is in pair order: it is exactly ssw_engine_align
 *              of the full grid with the same params with the non-hits removed (a caller who wants rank order sorts a row)
 *   records    field for field what ssw_engine_align returns for that pair; begins and CIGARs (flag & 7) are computed for the
 *              hits only, into a CIGAR pool the set owns (cigar_off counts words of that pool, at most 2^31 of them)
 *   max_hits   >= 0; a call that finds more hits returns -2 and no set (it may stop as soon as its running count passes the
 *              bound: the guard against a low min_score on a grid of 10^8 pairs)
 * The result does not depend on the path that ran, on how the grid was cut into launch groups or grid tiles (as for
 * ssw_engine_search) or on the number of devices.
 * Where the grid path runs, the hits of every launch group are counted and compacted on the device and copied back while the
 * next group computes: no record of a non-hit crosses to the host, and the device holds one launch group's hits at a time.
 * Which pairs run where is as for ssw_engine_search.  Every failure leaves *out NULL.
 */
typedef struct ssw_hit_set ssw_hit_set;
typedef struct {
	int32_t n_rows;
	int64_t n_hits;
	const int64_t* row_off;            /* n_rows + 1 */
	const int32_t* hit_ref;            /* n_hits */
	const ssw_batch_result* hits;      /* n_hits */
	const uint32_t* cigar_pool;        /* pool_used words (NULL if none) */
	int64_t pool_used;
} ssw_hit_view;

int ssw_engine_search_all(ssw_engine* e, const ssw_batch_params* params, int32_t min_score, int64_t max_hits, ssw_hit_set** out);
/* Pointers into the set, valid until ssw_hit_set_destroy. */
int ssw_hit_set_view(const ssw_hit_set* s, ssw_hit_view* v);
void ssw_hit_set_destroy(ssw_hit_set* s);

/*
 * Self-search: every pair of ONE set that scores at or above a threshold, each unordered pair computed once.
 *   set_sequences_self  makes seqs (n sequences, offsets off[n + 1]) resident as both the queries and the references;
 *              afterwards ssw_engine_align / _search / _search_all give exactly what they give after
 *              ssw_engine_set_sequences(seqs, seqs).  Any other ssw_engine_set_sequences* call ends self mode.
 *   order      canonical order: by (length, index), ascending
 *   pairs      each unordered pair {i, j}, i != j, at most once, as the record of query = the earlier of the two in canonical
 *              order (the shorter; on equal lengths the smaller index) against reference = the other -- field for field what
 *              ssw_engine_align returns for that oriented pair with the same params.  Self-pairs are not reported.
 *   hit        as ssw_engine_search_all: status 1, or score1 >= max(min_score, 1)
 *   output     an ssw_hit_set with n rows: row i holds the hits in which i is the query, in ascending partner index.
 *              max_hits, the -2 return and the flag pass (begins and CIGARs for the hits only, into the set's pool) are
 *              those of ssw_engine_search_all.
 *   refused    (-1, *out NULL) gap_open <= gap_extend, a matrix that is not symmetric on codes < n, mat == NULL, or a resident
 *              set that did not come from ssw_engine_set_sequences_self (profiles included).  With a symmetric matrix and
 *              gap_open > gap_extend a pair scores the same in both orientations, so the hits and their mirrors are exactly
 *              ssw_engine_search_all on (seqs, seqs) with the diagonal removed, at about half the work.
 * On the device path each query pair sweeps only the references ranked after its queries (DESIGN.md section 4.4f).
 */
int ssw_engine_set_sequences_self(ssw_engine* e, int32_t n, const int8_t* seqs, const int64_t* off);
int ssw_engine_search_self(ssw_engine* e, const ssw_batch_params* params, int32_t min_score, int64_t max_hits, ssw_hit_set** out);

/*
 * mark_mismatch (ssw.h:157-164; ssw.c:1019-1074) for the CIGARs of a whole batch, on the device: for every record of
 * `results` that carries a CIGAR (words at cigar_pool[cigar_off ...]) the M runs are split into '=' and 'X' runs, soft
 * clips are added for the unaligned ends of the read, and nm[p] (may be NULL) receives the number of mismatching +
 * inserted + deleted bases.  The pairs must be those of the ssw_engine_align call that produced the records (same
 * resident sequences, same pair lists).  On return cigar_off / cigar_len of those records point into out_pool;
 * out_cap >= sum over the CIGAR-carrying pairs of (query length + 2) words is always enough.
 */
int ssw_engine_mark_mismatch(ssw_engine* e, int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                             ssw_batch_result* results, const uint32_t* cigar_pool, int64_t pool_used,
                             uint32_t* out_pool, int64_t out_cap, int64_t* out_used, int32_t* nm);

/*
 * Convenience: set_sequences + align + conversion to heap s_align records
 * (each to be released with align_destroy; NULL where ssw_align would return NULL).
 * e == NULL draws an engine from the pool that also serves ssw_align (engines are created on demand, up to
 * SSW_B200_ENGINES, default 8; concurrent callers run side by side, each on its own engine and stream).
 */
int ssw_align_batch(ssw_engine* e, const ssw_batch_params* params,
                    int32_t n_queries, const int8_t* queries, const int64_t* query_off,
                    int32_t n_refs, const int8_t* refs, const int64_t* ref_off,
                    int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                    s_align** out);

/* ssw_align_batch followed by ssw_engine_mark_mismatch: the CIGARs of the returned records already carry soft clips and
 * '=' / 'X' runs (what mark_mismatch would make of them), nm[p] (may be NULL) the mismatch counts. */
int ssw_align_batch_marked(ssw_engine* e, const ssw_batch_params* params,
                           int32_t n_queries, const int8_t* queries, const int64_t* query_off,
                           int32_t n_refs, const int8_t* refs, const int64_t* ref_off,
                           int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                           s_align** out, int32_t* nm);

/* ssw_align_batch for text sequences (ssw_engine_set_sequences_text + align + s_align records); with
 * add_reverse_complement the queries n_queries .. 2*n_queries-1 are the reverse complements. */
int ssw_align_batch_text(ssw_engine* e, const ssw_batch_params* params, const int8_t* table, int32_t add_reverse_complement,
                         int32_t n_queries, const char* queries, const int64_t* query_off,
                         int32_t n_refs, const char* refs, const int64_t* ref_off,
                         int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                         s_align** out);

/*
 * Device groups: one batch over several GPUs of one process (main.c:462-532 is a loop over independent pairs; nothing is
 * exchanged while the matrices are filled, so the pair list is simply cut).  A group holds one engine per device and
 * runs every engine from its own host thread.
 *   full grid (pair lists NULL, n_pairs = all queries x all references): the QUERIES are cut into contiguous blocks of
 *       nearly equal total length (equal DP cells, as all of them meet the same references); every device receives its
 *       block of queries and all references and computes its rows of the grid;
 *   explicit pair list: the LIST is cut into contiguous blocks of nearly equal DP cells (query length x reference length:
 *       the split of ssw_dist.shard_bounds); pairs that share a reference stay together; sequences are replicated.
 * Records land in the caller's arrays in pair order exactly as one engine would deliver them; the CIGAR words of the
 * devices are concatenated (cigar_off re-based).  Results do not depend on the number of devices.
 */
typedef struct ssw_group ssw_group;

/* Number of usable CUDA devices (0 if none). */
int32_t ssw_device_count(void);

/* n_devices <= 0: all visible devices; devices == NULL: devices 0 .. n_devices-1.  NULL on failure. */
ssw_group* ssw_group_create(int32_t n_devices, const int32_t* devices);
void ssw_group_destroy(ssw_group* g);
int32_t ssw_group_size(const ssw_group* g);
/* The i-th engine of the group (options, timing of its share of the last call); owned by the group. */
ssw_engine* ssw_group_engine(ssw_group* g, int32_t i);

/*
 * set_sequences + align over the devices of the group.  `table` == NULL: queries / refs are codes (int8_t, as
 * ssw_engine_set_sequences takes them); otherwise they are text translated with `table` on the devices, and
 * add_reverse_complement != 0 adds query n_queries + k = reverse complement of query k (ssw_engine_set_sequences_text).
 * marked != 0 (needs a CIGAR flag): the CIGARs come back as mark_mismatch would leave them and nm[p] (may be NULL)
 * receives the mismatch counts (ssw_engine_mark_mismatch); pool_cap is then counted in marked words.
 */
int ssw_group_align(ssw_group* g, const ssw_batch_params* params, const int8_t* table, int32_t add_reverse_complement,
                    int32_t n_queries, const void* queries, const int64_t* query_off,
                    int32_t n_refs, const void* refs, const int64_t* ref_off,
                    int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                    ssw_batch_result* results, uint32_t* cigar_pool, int64_t pool_cap, int64_t* pool_used,
                    int32_t marked, int32_t* nm);

/* ssw_engine_search over the devices of the group: the queries are cut as for a full grid, every device searches its block
 * against all references, and its hit rows land in the caller's arrays (n_queries x k; with add_reverse_complement
 * 2 * n_queries rows, the reverse complements after the queries).  The CIGAR words of the devices are concatenated
 * (cigar_off re-based).  Results do not depend on the number of devices. */
int ssw_group_search(ssw_group* g, const ssw_batch_params* params, const int8_t* table, int32_t add_reverse_complement,
                     int32_t n_queries, const void* queries, const int64_t* query_off,
                     int32_t n_refs, const void* refs, const int64_t* ref_off,
                     int32_t k, int32_t min_score, int32_t* hit_ref, ssw_batch_result* hits, int32_t* n_hits,
                     uint32_t* cigar_pool, int64_t pool_cap, int64_t* pool_used);

/* ssw_engine_search_all over the devices of the group: the queries are cut as for ssw_group_search, every device returns a
 * set for its block, and the rows are concatenated in query order (with add_reverse_complement the 2 * n_queries rows of
 * ssw_group_search), which keeps pair order; the CIGAR pools are concatenated (cigar_off re-based).  max_hits bounds the
 * total.  Results do not depend on the number of devices. */
int ssw_group_search_all(ssw_group* g, const ssw_batch_params* params, const int8_t* table, int32_t add_reverse_complement,
                         int32_t n_queries, const void* queries, const int64_t* query_off,
                         int32_t n_refs, const void* refs, const int64_t* ref_off,
                         int32_t min_score, int64_t max_hits, ssw_hit_set** out);

/* ssw_engine_search_self over the devices of the group: every device holds the whole set and takes a contiguous range of
 * canonical ranks as queries, cut so that the devices have nearly equal triangle cells; rows of the n sequences are
 * concatenated and the CIGAR pools re-based.  max_hits bounds the total.  Results do not depend on the number of devices. */
int ssw_group_search_self(ssw_group* g, const ssw_batch_params* params, int32_t n, const int8_t* seqs, const int64_t* off,
                          int32_t min_score, int64_t max_hits, ssw_hit_set** out);

/* The same with heap s_align records (ssw_align_batch / _text / _marked over a group); release with align_destroy. */
int ssw_group_align_batch(ssw_group* g, const ssw_batch_params* params, const int8_t* table, int32_t add_reverse_complement,
                          int32_t n_queries, const void* queries, const int64_t* query_off,
                          int32_t n_refs, const void* refs, const int64_t* ref_off,
                          int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                          s_align** out, int32_t marked, int32_t* nm);

/* Device-time breakdown of the last ssw_engine_align / ssw_engine_search / ssw_engine_search_all call (CUDA events on the
 * engine's stream), in ms.  A search counts its selection (count and compaction) kernels in other_launches / resolve_ms. */
typedef struct {
	float fill_forward_ms;   /* matrix fill kernels, forward pass (incl. byte->word reruns) */
	float resolve_ms;        /* bookkeeping kernels */
	float fill_reverse_ms;   /* begin-search fill kernels */
	float traceback_ms;      /* banded traceback kernels */
	float total_ms;          /* first launch to last completion, incl. host planning in between */
	int64_t fill_forward_launches, other_launches;
	int64_t cells_forward;   /* DP cells computed by the forward fill kernels (incl. warm-up and pad rows) */
	int64_t byte_overflows;  /* pairs re-run with word semantics */
	/* counts of the device-planned grid, exact and known before a kernel runs (0 when no grid was planned) */
	int64_t grid_cols_planned;   /* group-columns the fill launches sweep: over the warps, groups per warp x the longest reference of the warp */
	int64_t grid_cols_useful;    /* of these, columns of a group's own reference; useful / planned = the planned sweep efficiency */
	int64_t leftover_pairs;      /* ssw_engine_search(_all): pairs outside the device-planned grid (general path, selection on the host) */
	/* bounded block words of the forward fill ("cm_block" -1 or 2) */
	int64_t block_refills;       /* candidate blocks re-filled to resolve the best cell (C1) and the second best (C2) */
	int64_t block_exact;         /* alignments with more than 256 candidate blocks in a stage, resolved from exact block maxima of their pair-task */
} ssw_engine_timing;
int ssw_engine_last_timing(const ssw_engine* e, ssw_engine_timing* t);
/* Column maxima of the engine's last forward fill launch, for tests: packed s16x2 words (the two alignments of a pair-task),
 * pair-task after pair-task in launch order, (refLen + 3) / 4 * 4 words per pair-task (one per column), or in block mode
 * (refLen / 64 + 4) / 4 * 4 (one per 64 columns; the words after the last block are not written).  Copies up to n_words
 * into out and returns the number of words of that launch, -1 on error. */
int64_t ssw_engine_last_colmax(ssw_engine* e, uint32_t* out, int64_t n_words);

/*
 * Tuning knobs for tests and measurements; none of them changes a result.  Unknown names return -1.  Every engine has
 * its own set; e == NULL addresses the engines behind ssw_align / ssw_align_batch(NULL, ...) (present and future).
 *   "chunk"         reference chunk length in columns of the fill kernel (0 = automatic)
 *   "small_chunk"   the same for launches too small to fill the device (0 = automatic)
 *   "cm_block"      column maxima of the forward fill: -1 automatic (bounded block words for long references), 0 one word per
 *                   column, 1 the exact maximum of every 64 columns (+ re-fill of the blocks whose single columns matter) wherever
 *                   the reference can be chunked, 2 bounded block words (a bracket of every 64 columns' maximum, + re-fill of the
 *                   blocks the bracket cannot rule out: DESIGN 2) wherever the reference can be chunked.  Same results in every mode.
 *   "cm_budget_mb"  cap of the column-maximum scratch per launch in MiB (0 = a share of the free device memory)
 *   "inst"          force forward kernel instance i (rows-per-lane / lanes-per-group table of the engine; -1 = automatic)
 *   "latency_cols"  passes over at most this many reference columns use the 32-lane instances (0 = never)
 *   "parts"         CTAs per task of the strip-pipelined kernel: 0 automatic, 1 never split, 2 / 4 forced
 *   "super"         columns per super-block of the strip-pipelined kernel
 *   "slices"        long-read CIGAR batches cut into slices on helper engines: 0 automatic (three equal slices, from 512
 *                   pairs on six slices each 80 % of the one before it), 1 never, 2 .. 8 forced
 *   "slice_taper"   t in 1 .. 99: every slice holds t % of the pairs of the one before it (0 = equal slices / automatic)
 *   "carve"         1 (default): the kernels of the long-read phases ask for the largest shared-memory carve-out, so that
 *                   their launches can share SMs; 0: the driver's choice per launch (measurements)
 *   "grid_min"      smallest full score-only grid that is planned on the device
 *   "grid_split"    grids of at least this many pairs are cut into launch groups whose records are copied back while the
 *                   next group computes (default 4 Mi pairs); "grid_group": smallest group in query pairs (default 16)
 *   "grid_arm"      device-planned grid: record best-cell rows only in the last k columns of every reference and re-do the pairs
 *                   whose maximum lies earlier (-1 automatic: protein-like alphabets, with a pilot group; 0 off; k > 0 fixed)
 *   "tb_maxbw"      widest band handled by the shared-memory traceback kernel
 *   "tb_spec"       band-doubling rounds of a traceback: 0 one after the other, 1 side by side (one warp per round; rounds of at most
 *                   129 columns ride along with the first), w > 1 the same with rounds of up to w columns,
 *                   -1 (default) side by side for a handful of tasks only (a lone call)
 */
int ssw_engine_set_option(ssw_engine* e, const char* name, int64_t value);
/* Two more names, for the launches of the device-planned grid over references of mixed lengths:
 *   "grid_order"    1 (default): the items of a query pair sweep the references longest first, so that the groups of a warp,
 *                   which run as long as their longest item, end together; 0: in reference order (measurements)
 *   "grid_max_ref"  references longer than this are not planned on the device (default and largest value 65,536; tests)
 *   "grid_tile_refs" ssw_engine_search / ssw_engine_search_all: at most this many qualifying references per grid tile (0,
 *                   the default: automatic -- one tile unless the grid has more than 2^31 - 1 pairs or one query pair's scratch
 *                   over all references exceeds the launch budget; tests, measurements).  Changes no result.
 */

#ifdef __cplusplus
}
#endif

#endif /* SSW_BATCH_H */
