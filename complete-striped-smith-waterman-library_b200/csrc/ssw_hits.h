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

#endif
