/* ssw_hits.h -- the result of a threshold search (ssw_engine_search_all, ssw_group_search_all): a CSR matrix of hit records
 * that the library allocates and the caller releases with ssw_hit_set_destroy.  Host-only; shared by the engine and the
 * device groups. */
#ifndef SSW_HITS_H
#define SSW_HITS_H

#include <vector>
#include "../../include/ssw_batch.h"

struct ssw_hit_set {
	int32_t n_rows = 0;
	std::vector<int64_t> row_off;             /* n_rows + 1 */
	std::vector<int32_t> hit_ref;
	std::vector<ssw_batch_result> hits;
	std::vector<uint32_t> pool;               /* CIGAR words of the hits (flag & 7) */
};

/* ssw_engine_search_self for the queries of canonical ranks [rank_lo, rank_hi) only (ssw_group_search_self: one range per
 * device); the set still has a row for every resident sequence, those of the other queries empty. */
int ssw_engine_search_self_ranks(ssw_engine* e, const ssw_batch_params* params, int32_t min_score, int64_t max_hits,
                                 int32_t rank_lo, int32_t rank_hi, ssw_hit_set** out);

#endif
