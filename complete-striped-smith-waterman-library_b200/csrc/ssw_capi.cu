/*
 * ssw_capi.cu -- the ssw.h entry points (drop-in boundary) on top of the batch engine.
 *
 *   ssw_init / init_destroy      <- src/ssw.c:826-853
 *   ssw_align                    <- src/ssw.c:855-977   (a batch of one pair)
 *   align_destroy                <- src/ssw.c:979-982
 *   mark_mismatch, add_cigar, store_previous_m <- src/ssw.c:984-1074 (host-side CIGAR post-processing)
 *   encoded_ops                  <- src/ssw.c:127-160
 *   ssw_align_batch              new: many pairs per call (include/ssw_batch.h)
 */
#include <condition_variable>
#include <exception>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
#include <vector>
#include <string.h>

#include "ssw_common.cuh"
#include "ssw_host.h"
#include "../../include/ssw.h"
#include "../../include/ssw_batch.h"

/* ASCII CIGAR letter -> BAM op code; letters not in "MIDNSHP=X" map to 0 like the reference table */
extern "C" const uint8_t encoded_ops[128] = {
	0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
	0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, /* '=' */ 7, 0, 0,
	0, 0, 0, 0, /* D */ 2, 0, 0, 0, /* H */ 5, /* I */ 1, 0, 0, 0, /* M */ 0, /* N */ 3, 0,
	/* P */ 6, 0, 0, /* S */ 4, 0, 0, 0, 0, /* X */ 8, 0, 0, 0, 0, 0, 0, 0,
	0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
};

/* The profile of the reference holds striped SSE2 tables (ssw.c:115-123); ours only
 * records what the engine needs.  read and mat are borrowed, as in the reference. */
struct _profile {
	const int8_t* read;
	const int8_t* mat;
	int32_t readLen;
	int32_t n;
	int8_t score_size;
};

s_align* ssw_record_from(const ssw_batch_result& r, const uint32_t* pool);

namespace {
/*
 * The engines behind ssw_align / ssw_align_batch(NULL, ...).  The reference's ssw_align is re-entrant (no locks, no
 * mutable globals: SURVEY 8(b) Threading), so concurrent callers must not be serialised on one engine: calls draw an
 * engine (own stream, own scratch) from a small pool that grows on demand up to SSW_B200_ENGINES (default 8); a caller
 * finding all of them busy waits for one.  A free engine that already holds the caller's reference is preferred
 * (ssw_engine_set_pair skips the upload then).
 */
struct PoolEntry { ssw_engine* e; bool busy; const int8_t* last_ref; int32_t last_len; };
std::mutex g_mu;
std::condition_variable g_cv;
std::vector<PoolEntry> g_pool;
std::vector<std::pair<std::string, int64_t>> g_pool_options;       /* ssw_engine_set_option(NULL, ...) calls, replayed on new engines */

int pool_limit()
{
	static int lim = 0;
	if (!lim) { const char* v = getenv("SSW_B200_ENGINES"); lim = v && atoi(v) > 0 ? atoi(v) : 8; if (lim > 64) lim = 64; }
	return lim;
}

ssw_engine* pool_acquire(const int8_t* ref, int32_t refLen)
{
	std::unique_lock<std::mutex> lock(g_mu);
	for (;;) {
		int pick = -1;
		for (size_t i = 0; i < g_pool.size(); ++i) {
			if (g_pool[i].busy) continue;
			if (ref && g_pool[i].last_ref == ref && g_pool[i].last_len == refLen) { pick = (int)i; break; }
			if (pick < 0) pick = (int)i;
		}
		if (pick >= 0) {
			g_pool[pick].busy = true; g_pool[pick].last_ref = ref; g_pool[pick].last_len = refLen;
			return g_pool[pick].e;
		}
		if ((int)g_pool.size() < pool_limit()) {
			ssw_engine* e = ssw_engine_create(-1);
			if (!e) return nullptr;
			for (const auto& kv : g_pool_options) ssw_engine_set_option(e, kv.first.c_str(), kv.second);
			g_pool.push_back(PoolEntry{e, true, ref, refLen});
			return e;
		}
		g_cv.wait(lock);
	}
}

void pool_release(ssw_engine* e)
{
	{
		std::lock_guard<std::mutex> lock(g_mu);
		for (PoolEntry& p : g_pool) if (p.e == e) p.busy = false;
	}
	g_cv.notify_one();
}

struct PoolGuard {
	ssw_engine* e;
	explicit PoolGuard(ssw_engine* x) : e(x) {}
	~PoolGuard() { if (e) pool_release(e); }
};

inline s_align* record_from(const ssw_batch_result& r, const uint32_t* pool) { return ssw_record_from(r, pool); }
}  // namespace

/* one batch record as a heap s_align (NULL where ssw_align returns NULL); also used by the device groups (ssw_group.cpp) */
s_align* ssw_record_from(const ssw_batch_result& r, const uint32_t* pool)
{
	if (r.status) return nullptr;
	s_align* a = (s_align*)calloc(1, sizeof(s_align));
	if (!a) return nullptr;
	a->score1 = r.score1; a->score2 = r.score2;
	a->ref_begin1 = r.ref_begin1; a->ref_end1 = r.ref_end1;
	a->read_begin1 = r.read_begin1; a->read_end1 = r.read_end1;
	a->ref_end2 = r.ref_end2; a->flag = r.flag;
	if (r.cigar_off >= 0 && r.cigar_len > 0) {
		a->cigar = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)r.cigar_len);   /* libc heap: callers free() it */
		if (!a->cigar) { free(a); return nullptr; }
		memcpy(a->cigar, pool + r.cigar_off, sizeof(uint32_t) * (size_t)r.cigar_len);
		a->cigarLen = r.cigar_len;
	}
	return a;
}

/* ssw_engine_set_option(NULL, name, value): every engine of the pool, present and future */
int ssw_default_engines_option(const char* name, int64_t value)
{
	/* an unknown option must fail now, even while the pool is empty, not at the first ssw_align */
	if (!ssw_engine_has_option(name)) { fprintf(stderr, "[libssw-b200] unknown option '%s'\n", name); return -1; }
	std::lock_guard<std::mutex> lock(g_mu);
	for (PoolEntry& p : g_pool) if (ssw_engine_set_option(p.e, name, value)) return -1;
	for (auto& kv : g_pool_options) if (kv.first == name) { kv.second = value; return 0; }
	g_pool_options.emplace_back(name, value);
	return 0;
}

extern "C" s_profile* ssw_init(const int8_t* read, const int32_t readLen, const int8_t* mat, const int32_t n, const int8_t score_size)
{
	s_profile* p = (s_profile*)calloc(1, sizeof(struct _profile));
	p->read = read; p->mat = mat; p->readLen = readLen; p->n = n; p->score_size = score_size;
	return p;
}

extern "C" void init_destroy(s_profile* p) { free(p); }

extern "C" void align_destroy(s_align* a)
{
	if (!a) return;
	free(a->cigar);
	free(a);
}

extern "C" s_align* ssw_align(const s_profile* prof, const int8_t* ref, int32_t refLen,
                              const uint8_t weight_gapO, const uint8_t weight_gapE, const uint8_t flag,
                              const uint16_t filters, const int32_t filterd, const int32_t maskLen)
{
	if (!prof || !ref || refLen < 0 || prof->readLen < 1 || !prof->read || !prof->mat) return NULL;
	if (maskLen < 15)   /* ssw.c:876-878: printed on every call */
		fprintf(stderr, "When maskLen < 15, the function ssw_align doesn't return 2nd best alignment information.\n");
	try {
		PoolGuard g(pool_acquire(ref, refLen));
		ssw_engine* e = g.e;
		if (!e) return NULL;
		if (ssw_engine_set_pair(e, prof->read, prof->readLen, ref, refLen)) return NULL;
		ssw_batch_params P;
		memset(&P, 0, sizeof(P));
		P.mat = prof->mat; P.n = prof->n; P.gap_open = weight_gapO; P.gap_extend = weight_gapE;
		P.flag = flag; P.filters = filters; P.filterd = filterd; P.mask_len = maskLen < 0 ? 0 : maskLen; P.score_size = prof->score_size;
		ssw_batch_result r;
		/* uninitialised storage: only the words the traceback writes are read */
		const size_t cap = (flag & 7) ? (size_t)prof->readLen + (size_t)refLen + 8 : 8;
		std::unique_ptr<uint32_t[]> pool(new uint32_t[cap]);
		int64_t used = 0;
		const int32_t pq = 0, pr = 0;
		if (ssw_engine_align(e, &P, 1, &pq, &pr, &r, pool.get(), (int64_t)cap, &used)) return NULL;
		return record_from(r, pool.get());
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_align: %s\n", ex.what()); return NULL; }
	catch (...) { return NULL; }
}

namespace {
/* align the resident sequences and turn the records into heap s_align objects */
int collect_batch(ssw_engine* e, const ssw_batch_params* params, int32_t n_queries, const int64_t* query_off,
                  int32_t n_refs, const int64_t* ref_off, int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref, s_align** out,
                  bool marked = false, int32_t* nm = nullptr)
{
	if (n_pairs < 0 || (n_pairs > 0 && (n_queries <= 0 || n_refs <= 0))) return -1;
	std::vector<ssw_batch_result> res((size_t)n_pairs);
	int64_t cap = 0;
	if (params->flag & 7) {
		for (int64_t p = 0; p < n_pairs; ++p) {
			const int32_t q = pair_query ? pair_query[p] : (int32_t)(p / n_refs), r = pair_ref ? pair_ref[p] : (int32_t)(p % n_refs);
			if (q < 0 || q >= n_queries || r < 0 || r >= n_refs) return -1;
			const int64_t ql = query_off[q + 1] - query_off[q], rl = ref_off[r + 1] - ref_off[r];
			/* a path has <= (query span + reference span + 2) words; a positive-scoring path cannot
			 * delete more than (query length * max score / gap_extend) reference bases */
			int64_t span = rl;
			if (params->gap_extend > 0) { const int64_t b = ql + ql * 127 / params->gap_extend; if (b < span) span = b; }
			cap += ql + span + 4;
		}
	}
	/* worst-case sized and mostly untouched: uninitialised storage, not a zero-filled vector */
	std::unique_ptr<uint32_t[]> pool(new uint32_t[(size_t)cap + 8]);
	int64_t used = 0;
	const int rc = ssw_engine_align(e, params, n_pairs, pair_query, pair_ref, res.data(), pool.get(), cap + 8, &used);
	if (rc) return rc;
	if (marked) {
		if (nm) for (int64_t p = 0; p < n_pairs; ++p) nm[p] = 0;
		if (used > 0) {
			/* a marked CIGAR has at most one word per aligned read base plus the deletions and two clips */
			int64_t mcap = 0;
			for (int64_t p = 0; p < n_pairs; ++p) if (res[p].cigar_len > 0) {
				const int32_t q = pair_query ? pair_query[p] : (int32_t)(p / n_refs);
				mcap += (query_off[q + 1] - query_off[q]) + res[p].cigar_len + 2;
			}
			std::unique_ptr<uint32_t[]> mpool(new uint32_t[(size_t)mcap + 8]);
			int64_t mused = 0;
			const int rc2 = ssw_engine_mark_mismatch(e, n_pairs, pair_query, pair_ref, res.data(), pool.get(), used, mpool.get(), mcap + 8, &mused, nm);
			if (rc2) return rc2;
			for (int64_t p = 0; p < n_pairs; ++p) out[p] = record_from(res[p], mpool.get());
			return 0;
		}
	}
	for (int64_t p = 0; p < n_pairs; ++p) out[p] = record_from(res[p], pool.get());
	return 0;
}
}  // namespace

extern "C" int ssw_align_batch(ssw_engine* e, const ssw_batch_params* params,
                               int32_t n_queries, const int8_t* queries, const int64_t* query_off,
                               int32_t n_refs, const int8_t* refs, const int64_t* ref_off,
                               int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                               s_align** out)
{
	if (!params || !out) return -1;
	try {
		PoolGuard g(e ? nullptr : pool_acquire(nullptr, 0));       /* NULL: an engine of the pool that also serves ssw_align */
		if (!e) e = g.e;
		if (!e) return -1;
		if (params->mask_len >= 0 && params->mask_len < 15)
			fprintf(stderr, "When maskLen < 15, the function ssw_align doesn't return 2nd best alignment information.\n");
		const int rc = ssw_engine_set_sequences(e, n_queries, queries, query_off, n_refs, refs, ref_off);
		if (rc) return rc;
		return collect_batch(e, params, n_queries, query_off, n_refs, ref_off, n_pairs, pair_query, pair_ref, out);
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_align_batch: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

extern "C" int ssw_align_batch_marked(ssw_engine* e, const ssw_batch_params* params,
                                      int32_t n_queries, const int8_t* queries, const int64_t* query_off,
                                      int32_t n_refs, const int8_t* refs, const int64_t* ref_off,
                                      int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                                      s_align** out, int32_t* nm)
{
	if (!params || !out) return -1;
	try {
		PoolGuard g(e ? nullptr : pool_acquire(nullptr, 0));
		if (!e) e = g.e;
		if (!e) return -1;
		if (params->mask_len >= 0 && params->mask_len < 15)
			fprintf(stderr, "When maskLen < 15, the function ssw_align doesn't return 2nd best alignment information.\n");
		const int rc = ssw_engine_set_sequences(e, n_queries, queries, query_off, n_refs, refs, ref_off);
		if (rc) return rc;
		return collect_batch(e, params, n_queries, query_off, n_refs, ref_off, n_pairs, pair_query, pair_ref, out, true, nm);
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_align_batch_marked: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

extern "C" int ssw_align_batch_text(ssw_engine* e, const ssw_batch_params* params, const int8_t* table, int32_t add_reverse_complement,
                                    int32_t n_queries, const char* queries, const int64_t* query_off,
                                    int32_t n_refs, const char* refs, const int64_t* ref_off,
                                    int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                                    s_align** out)
{
	if (!params || !out || !table) return -1;
	try {
		PoolGuard g(e ? nullptr : pool_acquire(nullptr, 0));
		if (!e) e = g.e;
		if (!e) return -1;
		if (params->mask_len >= 0 && params->mask_len < 15)
			fprintf(stderr, "When maskLen < 15, the function ssw_align doesn't return 2nd best alignment information.\n");
		const int rc = ssw_engine_set_sequences_text(e, n_queries, queries, query_off, n_refs, refs, ref_off, table, params->n, add_reverse_complement);
		if (rc) return rc;
		if (n_queries <= 0 || !query_off) return n_pairs == 0 ? 0 : -1;
		/* query k + n_queries is the reverse complement of query k */
		const int32_t nq = n_queries * (add_reverse_complement ? 2 : 1);
		std::vector<int64_t> qoff(query_off, query_off + n_queries + 1);
		if (add_reverse_complement) for (int i = 1; i <= n_queries; ++i) qoff.push_back(query_off[n_queries] + query_off[i]);
		return collect_batch(e, params, nq, qoff.data(), n_refs, ref_off, n_pairs, pair_query, pair_ref, out);
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_align_batch_text: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

/* ------------------------------------------------------------------------------------------- */
/* CIGAR post-processing (host, O(alignment length)); exported with the reference's names        */
/* ------------------------------------------------------------------------------------------- */

/* append (length, op) to a growable CIGAR; *p = used, *s = capacity (ssw.c:984-992) */
extern "C" uint32_t* add_cigar(uint32_t* new_cigar, int32_t* p, int32_t* s, uint32_t length, char op)
{
	if (*p >= *s) {
		int32_t cap = *s < 4 ? 4 : *s;
		while (cap <= *p) cap *= 2;
		*s = cap;
		new_cigar = (uint32_t*)realloc(new_cigar, sizeof(uint32_t) * (size_t)cap);
	}
	new_cigar[(*p)++] = to_cigar_int(length, (unsigned char)op);
	return new_cigar;
}

/* flush a pending '=' or 'X' run; choice 0: current op is not M, 1: current base matches, 2: mismatches (ssw.c:994-1009) */
extern "C" uint32_t* store_previous_m(int8_t choice, uint32_t* length_m, uint32_t* length_x, int32_t* p, int32_t* s, uint32_t* new_cigar)
{
	if (*length_m && choice != 1) { new_cigar = add_cigar(new_cigar, p, s, *length_m, '='); *length_m = 0; }
	else if (*length_x && choice != 2) { new_cigar = add_cigar(new_cigar, p, s, *length_x, 'X'); *length_x = 0; }
	return new_cigar;
}

extern "C" int32_t mark_mismatch(int32_t ref_begin1, int32_t read_begin1, int32_t read_end1,
                                 const int8_t* ref, const int8_t* read, int32_t readLen,
                                 uint32_t** cigar, int32_t* cigarLen)
{
	int32_t used = 0, cap = *cigarLen + 2, nm = 0;
	uint32_t* out = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(cap > 0 ? cap : 1));
	uint32_t run_eq = 0, run_x = 0;
	const int8_t* rp = ref + ref_begin1;
	const int8_t* qp = read + read_begin1;
	if (read_begin1 > 0) out = add_cigar(out, &used, &cap, (uint32_t)read_begin1, 'S');
	for (int32_t i = 0; i < *cigarLen; ++i) {
		const char op = cigar_int_to_op((*cigar)[i]);
		const int32_t len = (int32_t)cigar_int_to_len((*cigar)[i]);
		if (op == 'M') {
			for (int32_t k = 0; k < len; ++k, ++rp, ++qp) {
				if (*rp != *qp) { ++nm; out = store_previous_m(2, &run_eq, &run_x, &used, &cap, out); ++run_x; }
				else { out = store_previous_m(1, &run_eq, &run_x, &used, &cap, out); ++run_eq; }
			}
		} else if (op == 'I' || op == 'D') {
			if (op == 'I') qp += len; else rp += len;
			nm += len;
			out = store_previous_m(0, &run_eq, &run_x, &used, &cap, out);
			out = add_cigar(out, &used, &cap, (uint32_t)len, op);
		}
	}
	out = store_previous_m(0, &run_eq, &run_x, &used, &cap, out);
	if (readLen - read_end1 - 1 > 0) out = add_cigar(out, &used, &cap, (uint32_t)(readLen - read_end1 - 1), 'S');
	*cigarLen = used;
	free(*cigar);
	*cigar = out;
	return nm;
}
