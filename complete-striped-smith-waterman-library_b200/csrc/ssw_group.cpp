/*
 * ssw_group.cpp -- one batch over several GPUs of one process (include/ssw_batch.h, "Device groups").
 *
 * The reference's CLI walks reads x references one blocking call at a time (src/main.c:462-532); the pairs are
 * independent, so several devices need no exchange: the pair list (or, for a full grid, the list of queries) is cut
 * into contiguous cell-balanced blocks -- the split of ssw_dist.shard_bounds, which the multi-process path uses --
 * and every device's engine runs its block from its own host thread.  Host-only code over the batch C ABI: no kernel
 * and no CUDA call lives here; what the devices compute is exactly what one engine computes for the same pairs.
 */
#include <algorithm>
#include <exception>
#include <memory>
#include <thread>
#include <vector>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/ssw.h"
#include "../../include/ssw_batch.h"
#include "ssw_hits.h"

s_align* ssw_record_from(const ssw_batch_result& r, const uint32_t* pool);       /* ssw_capi.cu */

struct ssw_group {
	std::vector<ssw_engine*> eng;
};

namespace {

struct Job {
	const ssw_batch_params* P;
	const int8_t* table; int32_t add_rc;
	int32_t n_q; const char* q; const int64_t* qoff;
	int32_t n_r; const char* r; const int64_t* roff;
	int64_t n_pairs; const int32_t* pq; const int32_t* pr;
	bool marked;
};

/* what one device is given and what it hands back */
struct Shard {
	bool grid = false;
	int32_t q0 = 0, q1 = 0;          /* grid: block of the caller's queries */
	int64_t p0 = 0, p1 = 0;          /* list: block of the pair list */
	ssw_batch_result* ext = nullptr;  /* the caller's records where the block is contiguous in pair order (written in place), else res */
	std::vector<ssw_batch_result> res;
	int64_t n = 0;                   /* pairs of this block */
	std::vector<int32_t> nm;
	std::unique_ptr<uint32_t[]> pool;
	int64_t used = 0;
	int rc = 0;
	int64_t pairs() const { return n; }
	ssw_batch_result* records() { return ext ? ext : res.data(); }
	const ssw_batch_result* records() const { return ext ? ext : res.data(); }
};

/* world+1 boundaries of contiguous blocks of nearly equal total weight (ssw_dist.shard_bounds) */
template <class W> std::vector<int64_t> balanced_bounds(int64_t n, int world, W weight)
{
	std::vector<int64_t> b((size_t)world + 1, 0);
	b[world] = n;
	if (n == 0) return b;
	long double total = 0;
	for (int64_t i = 0; i < n; ++i) total += (long double)weight(i);
	long double acc = 0;
	int64_t i = 0;
	for (int r = 1; r < world; ++r) {
		const long double target = total * r / world;
		while (i < n && acc < target) acc += (long double)weight(i++);
		b[r] = i;
	}
	return b;
}

/* worst-case CIGAR words of one pair (the bound ssw_align_batch uses): a path has at most query span + reference span
 * + 2 words, and a positive-scoring path cannot delete more than query length * max score / gap_extend bases */
inline int64_t cigar_bound(int64_t ql, int64_t rl, int gap_extend)
{
	int64_t span = rl;
	if (gap_extend > 0) { const int64_t b = ql + ql * 127 / gap_extend; if (b < span) span = b; }
	return ql + span + 4;
}

void run_shard(ssw_engine* e, const Job& J, Shard& S)
{
	try {
		const ssw_batch_params& P = *J.P;
		const bool want_cigar = (P.flag & 7) != 0;
		int64_t n_pairs = 0, cap = 0;
		std::vector<int64_t> qoff;                  /* offsets of the queries this device holds (rebased; incl. reverse complements) */
		int32_t nq_loc = 0;
		const int32_t* pq = nullptr; const int32_t* pr = nullptr;
		if (S.grid) {
			nq_loc = S.q1 - S.q0;
			if (nq_loc <= 0) return;
			qoff.resize((size_t)nq_loc + 1);
			for (int32_t k = 0; k <= nq_loc; ++k) qoff[k] = J.qoff[S.q0 + k] - J.qoff[S.q0];
			const char* qbase = J.q + J.qoff[S.q0];
			S.rc = J.table ? ssw_engine_set_sequences_text(e, nq_loc, qbase, qoff.data(), J.n_r, J.r, J.roff, J.table, P.n, J.add_rc)
			               : ssw_engine_set_sequences(e, nq_loc, (const int8_t*)qbase, qoff.data(), J.n_r, (const int8_t*)J.r, J.roff);
			if (S.rc) return;
			if (J.add_rc) for (int32_t k = 1; k <= nq_loc; ++k) qoff.push_back(qoff[nq_loc] + qoff[k]);
			const int32_t nq_all = nq_loc * (J.add_rc ? 2 : 1);
			n_pairs = (int64_t)nq_all * J.n_r;
			if (want_cigar) {
				int64_t per_query_refs = 0;
				for (int32_t k = 0; k < nq_all; ++k) {
					const int64_t ql = qoff[k + 1] - qoff[k];
					per_query_refs = 0;
					for (int32_t r = 0; r < J.n_r; ++r) per_query_refs += cigar_bound(ql, J.roff[r + 1] - J.roff[r], P.gap_extend);
					cap += per_query_refs;
				}
			}
		} else {
			n_pairs = S.p1 - S.p0;
			if (n_pairs <= 0) return;
			S.rc = J.table ? ssw_engine_set_sequences_text(e, J.n_q, J.q, J.qoff, J.n_r, J.r, J.roff, J.table, P.n, J.add_rc)
			               : ssw_engine_set_sequences(e, J.n_q, (const int8_t*)J.q, J.qoff, J.n_r, (const int8_t*)J.r, J.roff);
			if (S.rc) return;
			qoff.assign(J.qoff, J.qoff + J.n_q + 1);
			if (J.add_rc) for (int32_t k = 1; k <= J.n_q; ++k) qoff.push_back(J.qoff[J.n_q] + J.qoff[k]);
			pq = J.pq + S.p0; pr = J.pr + S.p0;
			if (want_cigar) for (int64_t p = 0; p < n_pairs; ++p) cap += cigar_bound(qoff[pq[p] + 1] - qoff[pq[p]], J.roff[pr[p] + 1] - J.roff[pr[p]], P.gap_extend);
		}
		if (!S.ext) S.res.resize((size_t)n_pairs);
		S.n = n_pairs;
		ssw_batch_result* const R = S.records();
		S.pool.reset(new uint32_t[(size_t)cap + 8]);         /* worst-case sized and mostly untouched: uninitialised storage */
		S.rc = ssw_engine_align(e, &P, n_pairs, pq, pr, R, S.pool.get(), cap + 8, &S.used);
		if (S.rc) return;
		if (J.marked) {
			S.nm.assign((size_t)n_pairs, 0);
			if (S.used > 0) {
				/* a marked CIGAR has at most one word per aligned read base plus the deletions and two clips */
				int64_t mcap = 0;
				for (int64_t p = 0; p < n_pairs; ++p) if (R[p].cigar_len > 0) {
					const int32_t q = pq ? pq[p] : (int32_t)(p / J.n_r);
					mcap += (qoff[q + 1] - qoff[q]) + R[p].cigar_len + 2;
				}
				std::unique_ptr<uint32_t[]> mpool(new uint32_t[(size_t)mcap + 8]);
				int64_t mused = 0;
				S.rc = ssw_engine_mark_mismatch(e, n_pairs, pq, pr, R, S.pool.get(), S.used, mpool.get(), mcap + 8, &mused, S.nm.data());
				if (S.rc) return;
				S.pool = std::move(mpool);
				S.used = mused;
			}
		}
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] device group: %s\n", ex.what()); S.rc = -1; }
	catch (...) { S.rc = -1; }
}

/* position in the caller's pair order of local pair l of a shard */
inline int64_t global_pair(const Job& J, const Shard& S, int64_t l)
{
	if (!S.grid) return S.p0 + l;
	const int64_t plus = (int64_t)(S.q1 - S.q0) * J.n_r;           /* pairs of the shard's own queries; then their reverse complements */
	return l < plus ? (int64_t)S.q0 * J.n_r + l : ((int64_t)J.n_q + S.q0) * J.n_r + (l - plus);
}

/* work(d) for every device d of the group: one host thread per device, the calling thread taking device 0 */
template <class F> void for_each_device(const ssw_group* g, const F& work)
{
	const int world = (int)g->eng.size();
#ifdef SSW_CPU_EMU
	for (int d = 0; d < world; ++d) work(d);        /* the emulator's fibers are not thread-safe */
#else
	std::vector<std::thread> th;
	th.reserve((size_t)world);
	for (int d = 1; d < world; ++d) {
		try { th.emplace_back([&work, d] { work(d); }); }
		catch (...) { work(d); }                     /* no thread to be had: this block runs here */
	}
	work(0);
	for (std::thread& t : th) t.join();
#endif
}

/* one device's hit set (ssw_engine_search_all, ssw_engine_search_self) and return code */
struct HitPart {
	ssw_hit_set* set = nullptr;
	int rc = 0;
	HitPart() = default;
	HitPart(const HitPart&) = delete;
	HitPart& operator=(const HitPart&) = delete;
	~HitPart() { ssw_hit_set_destroy(set); }
};

/* The hit set of a device group from the sets of its devices: row i is row rows[i].second of device rows[i].first's set, and the
 * CIGAR pools are concatenated in device order with every offset re-based.  Returns -2 (`fn` says so) above max_hits hits. */
int gather_hits(const char* fn, const std::vector<HitPart>& parts, const std::vector<std::pair<int, int32_t>>& rows,
                int64_t max_hits, ssw_hit_set** out)
{
	int64_t n_hits = 0, n_words = 0;
	for (const HitPart& S : parts) if (S.set) { n_hits += (int64_t)S.set->hits.size(); n_words += (int64_t)S.set->pool.size(); }
	if (n_hits > max_hits) { fprintf(stderr, "[libssw-b200] %s: more than max_hits = %lld hits\n", fn, (long long)max_hits); return -2; }
	if (n_words > 0x7fffffff) { fprintf(stderr, "[libssw-b200] more than 2^31 CIGAR words in one batch: split the batch\n"); return -1; }
	std::unique_ptr<ssw_hit_set> s(new ssw_hit_set());
	s->n_rows = (int32_t)rows.size();
	s->row_off.reserve(rows.size() + 1);
	s->row_off.push_back(0);
	s->hit_ref.reserve((size_t)n_hits); s->hits.reserve((size_t)n_hits); s->pool.reserve((size_t)n_words);
	std::vector<int64_t> base(parts.size(), 0);
	for (size_t d = 0; d < parts.size(); ++d) {
		if (!parts[d].set) continue;
		base[d] = (int64_t)s->pool.size();
		s->pool.insert(s->pool.end(), parts[d].set->pool.begin(), parts[d].set->pool.end());
	}
	for (const std::pair<int, int32_t>& row : rows) {
		const ssw_hit_set& S = *parts[row.first].set;
		for (int64_t i = S.row_off[row.second]; i < S.row_off[row.second + 1]; ++i) {
			ssw_batch_result o = S.hits[i];
			if (o.cigar_off >= 0) o.cigar_off += (int32_t)base[row.first];
			s->hits.push_back(o);
			s->hit_ref.push_back(S.hit_ref[i]);
		}
		s->row_off.push_back((int64_t)s->hits.size());
	}
	*out = s.release();
	return 0;
}

int run_job(ssw_group* g, const Job& J, std::vector<Shard>& shards, ssw_batch_result* results)
{
	const ssw_batch_params& P = *J.P;
	if (!P.mat || P.n < 1 || P.n > 64) { fprintf(stderr, "[libssw-b200] device group: bad scoring parameters\n"); return -1; }
	if (J.n_pairs < 0 || (J.pq == nullptr) != (J.pr == nullptr)) return -1;
	if (J.n_q < 0 || J.n_r < 0 || !J.qoff || !J.roff || (J.n_pairs > 0 && (J.n_q == 0 || J.n_r == 0 || !J.q || !J.r))) return -1;
	for (int32_t k = 0; k < J.n_q; ++k) if (J.qoff[k + 1] < J.qoff[k]) { fprintf(stderr, "[libssw-b200] query offsets are not non-decreasing at %d\n", k); return -1; }
	for (int32_t k = 0; k < J.n_r; ++k) if (J.roff[k + 1] < J.roff[k]) { fprintf(stderr, "[libssw-b200] reference offsets are not non-decreasing at %d\n", k); return -1; }
	const int32_t nq_all = J.n_q * (J.add_rc ? 2 : 1);
	const int world = (int)g->eng.size();
	shards.clear(); shards.resize((size_t)world);
	if (J.n_pairs == 0) return 0;
	if (P.mask_len >= 0 && P.mask_len < 15)   /* ssw.c:876-878 prints this on every call; a batch says it once */
		fprintf(stderr, "When maskLen < 15, the function ssw_align doesn't return 2nd best alignment information.\n");
	std::vector<int32_t> gq, gr;              /* a grid prefix that is not the whole grid runs as an explicit list */
	Job JJ = J;
	if (!J.pq && J.n_pairs != (int64_t)nq_all * J.n_r) {
		if (J.n_pairs > (int64_t)nq_all * J.n_r) { fprintf(stderr, "[libssw-b200] device group: more pairs than the grid holds\n"); return -1; }
		gq.resize((size_t)J.n_pairs); gr.resize((size_t)J.n_pairs);
		for (int64_t p = 0; p < J.n_pairs; ++p) { gq[p] = (int32_t)(p / J.n_r); gr[p] = (int32_t)(p % J.n_r); }
		JJ.pq = gq.data(); JJ.pr = gr.data();
	}
	if (!JJ.pq) {
		const std::vector<int64_t> b = balanced_bounds(J.n_q, world, [&](int64_t k) { return J.qoff[k + 1] - J.qoff[k] + 1; });
		for (int d = 0; d < world; ++d) {
			shards[d].grid = true; shards[d].q0 = (int32_t)b[d]; shards[d].q1 = (int32_t)b[d + 1];
			if (results && !J.add_rc) shards[d].ext = results + b[d] * J.n_r;         /* rows q0 .. q1 of the grid are contiguous */
		}
	} else {
		for (int64_t p = 0; p < J.n_pairs; ++p)
			if (JJ.pq[p] < 0 || JJ.pq[p] >= nq_all || JJ.pr[p] < 0 || JJ.pr[p] >= J.n_r) { fprintf(stderr, "[libssw-b200] pair %lld out of range\n", (long long)p); return -1; }
		const std::vector<int64_t> b = balanced_bounds(J.n_pairs, world, [&](int64_t p) {
			const int32_t q = JJ.pq[p] >= J.n_q ? JJ.pq[p] - J.n_q : JJ.pq[p];
			return (J.qoff[q + 1] - J.qoff[q] + 1) * (J.roff[JJ.pr[p] + 1] - J.roff[JJ.pr[p]] + 1);
		});
		for (int d = 0; d < world; ++d) { shards[d].p0 = b[d]; shards[d].p1 = b[d + 1]; if (results) shards[d].ext = results + b[d]; }
	}
	for_each_device(g, [&](int d) { run_shard(g->eng[d], JJ, shards[d]); });
	for (const Shard& S : shards) if (S.rc) return S.rc;
	return 0;
}

Job make_job(const ssw_batch_params* params, const int8_t* table, int32_t add_rc, int32_t n_queries, const void* queries, const int64_t* query_off,
             int32_t n_refs, const void* refs, const int64_t* ref_off, int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref, int32_t marked)
{
	Job J;
	J.P = params; J.table = table; J.add_rc = table && add_rc ? 1 : 0;
	J.n_q = n_queries; J.q = (const char*)queries; J.qoff = query_off;
	J.n_r = n_refs; J.r = (const char*)refs; J.roff = ref_off;
	J.n_pairs = n_pairs; J.pq = pair_query; J.pr = pair_ref; J.marked = marked != 0;
	return J;
}

}  // namespace

extern "C" ssw_group* ssw_group_create(int32_t n_devices, const int32_t* devices)
{
	try {
		const int32_t count = ssw_device_count();
		if (count <= 0) { fprintf(stderr, "[libssw-b200] no usable CUDA device: this library has no CPU compute path\n"); return nullptr; }
		if (n_devices <= 0) { n_devices = count; devices = nullptr; }
		std::unique_ptr<ssw_group> g(new ssw_group());
		for (int32_t i = 0; i < n_devices; ++i) {
			ssw_engine* e = ssw_engine_create(devices ? devices[i] : i);
			if (!e) { for (ssw_engine* x : g->eng) ssw_engine_destroy(x); return nullptr; }
			g->eng.push_back(e);
		}
		return g.release();
	}
	catch (...) { return nullptr; }
}

extern "C" void ssw_group_destroy(ssw_group* g)
{
	if (!g) return;
	for (ssw_engine* e : g->eng) ssw_engine_destroy(e);
	delete g;
}

extern "C" int32_t ssw_group_size(const ssw_group* g) { return g ? (int32_t)g->eng.size() : 0; }

extern "C" ssw_engine* ssw_group_engine(ssw_group* g, int32_t i) { return g && i >= 0 && i < (int32_t)g->eng.size() ? g->eng[i] : nullptr; }

extern "C" int ssw_group_align(ssw_group* g, const ssw_batch_params* params, const int8_t* table, int32_t add_reverse_complement,
                               int32_t n_queries, const void* queries, const int64_t* query_off,
                               int32_t n_refs, const void* refs, const int64_t* ref_off,
                               int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                               ssw_batch_result* results, uint32_t* cigar_pool, int64_t pool_cap, int64_t* pool_used,
                               int32_t marked, int32_t* nm)
{
	if (!g || g->eng.empty() || !params || (n_pairs > 0 && !results)) return -1;
	try {
		if (pool_used) *pool_used = 0;
		const Job J = make_job(params, table, add_reverse_complement, n_queries, queries, query_off, n_refs, refs, ref_off, n_pairs, pair_query, pair_ref, marked);
		std::vector<Shard> shards;
		const int rc = run_job(g, J, shards, results);
		if (rc) return rc;
		int64_t base = 0;
		for (Shard& S : shards) {
			if (S.used > 0) {
				if (!cigar_pool || base + S.used > pool_cap) { fprintf(stderr, "[libssw-b200] CIGAR pool too small\n"); return -1; }
				if (base + S.used > 0x7fffffff) { fprintf(stderr, "[libssw-b200] more than 2^31 CIGAR words in one batch: split the batch\n"); return -1; }
				memcpy(cigar_pool + base, S.pool.get(), sizeof(uint32_t) * (size_t)S.used);
			}
			const bool fix = base > 0 && S.used > 0;
			if (!S.ext || fix || nm)
				for (int64_t l = 0; l < S.pairs(); ++l) {
					const int64_t p = global_pair(J, S, l);
					if (!S.ext) results[p] = S.res[l];
					if (fix && results[p].cigar_off >= 0) results[p].cigar_off += (int32_t)base;
					if (nm) nm[p] = S.nm.empty() ? 0 : S.nm[l];
				}
			base += S.used;
		}
		if (pool_used) *pool_used = base;
		return 0;
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_group_align: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

extern "C" int ssw_group_search(ssw_group* g, const ssw_batch_params* params, const int8_t* table, int32_t add_reverse_complement,
                                int32_t n_queries, const void* queries, const int64_t* query_off,
                                int32_t n_refs, const void* refs, const int64_t* ref_off,
                                int32_t k, int32_t min_score, int32_t* hit_ref, ssw_batch_result* hits, int32_t* n_hits,
                                uint32_t* cigar_pool, int64_t pool_cap, int64_t* pool_used)
{
	if (!g || g->eng.empty() || !params || !params->mat || !hit_ref || !hits || !n_hits) { fprintf(stderr, "[libssw-b200] ssw_group_search: NULL argument\n"); return -1; }
	if (k < 1 || k > 1024) { fprintf(stderr, "[libssw-b200] ssw_group_search: k = %d outside 1 .. 1024\n", k); return -1; }
	if (n_queries <= 0 || n_refs <= 0 || !queries || !refs || !query_off || !ref_off) { fprintf(stderr, "[libssw-b200] ssw_group_search: no sequences\n"); return -1; }
	try {
		if (pool_used) *pool_used = 0;
		const ssw_batch_params& P = *params;
		for (int32_t q = 0; q < n_queries; ++q) if (query_off[q + 1] < query_off[q]) { fprintf(stderr, "[libssw-b200] query offsets are not non-decreasing at %d\n", q); return -1; }
		for (int32_t r = 0; r < n_refs; ++r) if (ref_off[r + 1] < ref_off[r]) { fprintf(stderr, "[libssw-b200] reference offsets are not non-decreasing at %d\n", r); return -1; }
		const bool add_rc = table && add_reverse_complement;
		const bool want_cigar = (P.flag & 7) != 0;
		int64_t max_rl = 0;
		for (int32_t r = 0; r < n_refs; ++r) max_rl = std::max<int64_t>(max_rl, ref_off[r + 1] - ref_off[r]);
		/* the queries cut as for a full grid (ssw_group_align); every device searches its block against all references */
		const int world = (int)g->eng.size();
		const std::vector<int64_t> b = balanced_bounds(n_queries, world, [&](int64_t q) { return query_off[q + 1] - query_off[q] + 1; });
		struct Part {
			int32_t q0 = 0, n = 0;       /* first query; rows searched (queries, then their reverse complements) */
			std::vector<int32_t> ref, nh;
			std::vector<ssw_batch_result> rec;
			std::unique_ptr<uint32_t[]> pool;
			int64_t used = 0;
			int rc = 0;
		};
		std::vector<Part> parts((size_t)world);
		auto work = [&](int d) {
			Part& S = parts[d];
			try {
				S.q0 = (int32_t)b[d];
				const int32_t nq = (int32_t)(b[d + 1] - b[d]);
				if (nq <= 0) return;
				std::vector<int64_t> qoff((size_t)nq + 1);
				for (int32_t j = 0; j <= nq; ++j) qoff[j] = query_off[S.q0 + j] - query_off[S.q0];
				const char* qbase = (const char*)queries + query_off[S.q0];
				ssw_engine* e = g->eng[d];
				S.rc = table ? ssw_engine_set_sequences_text(e, nq, qbase, qoff.data(), n_refs, (const char*)refs, ref_off, table, P.n, add_rc ? 1 : 0)
				             : ssw_engine_set_sequences(e, nq, (const int8_t*)qbase, qoff.data(), n_refs, (const int8_t*)refs, ref_off);
				if (S.rc) return;
				S.n = nq * (add_rc ? 2 : 1);
				int64_t cap = 0;
				if (want_cigar) for (int32_t j = 0; j < nq; ++j) cap += (int64_t)k * cigar_bound(qoff[j + 1] - qoff[j], max_rl, P.gap_extend);
				if (add_rc) cap *= 2;
				S.ref.resize((size_t)S.n * k); S.rec.resize((size_t)S.n * k); S.nh.resize((size_t)S.n);
				S.pool.reset(new uint32_t[(size_t)cap + 8]);
				S.rc = ssw_engine_search(e, &P, k, min_score, S.ref.data(), S.rec.data(), S.nh.data(), S.pool.get(), cap + 8, &S.used);
			}
			catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] device group: %s\n", ex.what()); S.rc = -1; }
			catch (...) { S.rc = -1; }
		};
		for_each_device(g, work);
		for (const Part& S : parts) if (S.rc) return S.rc;
		int64_t base = 0;
		for (const Part& S : parts) {
			if (S.used > 0) {
				if (!cigar_pool || base + S.used > pool_cap) { fprintf(stderr, "[libssw-b200] CIGAR pool too small\n"); return -1; }
				if (base + S.used > 0x7fffffff) { fprintf(stderr, "[libssw-b200] more than 2^31 CIGAR words in one batch: split the batch\n"); return -1; }
				memcpy(cigar_pool + base, S.pool.get(), sizeof(uint32_t) * (size_t)S.used);
			}
			const int32_t nq = add_rc ? S.n / 2 : S.n;
			for (int32_t l = 0; l < S.n; ++l) {
				const int64_t row = l < nq ? (int64_t)S.q0 + l : (int64_t)n_queries + S.q0 + (l - nq);
				n_hits[row] = S.nh[l];
				for (int32_t i = 0; i < k; ++i) {
					ssw_batch_result o = S.rec[(size_t)l * k + i];
					if (o.cigar_off >= 0) o.cigar_off += (int32_t)base;
					hits[row * k + i] = o;
					hit_ref[row * k + i] = S.ref[(size_t)l * k + i];
				}
			}
			base += S.used;
		}
		if (pool_used) *pool_used = base;
		return 0;
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_group_search: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

extern "C" int ssw_group_search_all(ssw_group* g, const ssw_batch_params* params, const int8_t* table, int32_t add_reverse_complement,
                                    int32_t n_queries, const void* queries, const int64_t* query_off,
                                    int32_t n_refs, const void* refs, const int64_t* ref_off,
                                    int32_t min_score, int64_t max_hits, ssw_hit_set** out)
{
	if (!out) { fprintf(stderr, "[libssw-b200] ssw_group_search_all: NULL output\n"); return -1; }
	*out = nullptr;
	if (!g || g->eng.empty() || !params || !params->mat) { fprintf(stderr, "[libssw-b200] ssw_group_search_all: NULL argument\n"); return -1; }
	if (max_hits < 0) { fprintf(stderr, "[libssw-b200] ssw_group_search_all: max_hits = %lld is negative\n", (long long)max_hits); return -1; }
	if (n_queries <= 0 || n_refs <= 0 || !queries || !refs || !query_off || !ref_off) { fprintf(stderr, "[libssw-b200] ssw_group_search_all: no sequences\n"); return -1; }
	try {
		const ssw_batch_params& P = *params;
		for (int32_t q = 0; q < n_queries; ++q) if (query_off[q + 1] < query_off[q]) { fprintf(stderr, "[libssw-b200] query offsets are not non-decreasing at %d\n", q); return -1; }
		for (int32_t r = 0; r < n_refs; ++r) if (ref_off[r + 1] < ref_off[r]) { fprintf(stderr, "[libssw-b200] reference offsets are not non-decreasing at %d\n", r); return -1; }
		const bool add_rc = table && add_reverse_complement;
		/* the queries cut as for ssw_group_search; every device searches its block against all references */
		const int world = (int)g->eng.size();
		const std::vector<int64_t> b = balanced_bounds(n_queries, world, [&](int64_t q) { return query_off[q + 1] - query_off[q] + 1; });
		std::vector<HitPart> parts((size_t)world);
		auto work = [&](int d) {
			HitPart& S = parts[d];
			try {
				const int32_t q0 = (int32_t)b[d], nq = (int32_t)(b[d + 1] - b[d]);
				if (nq <= 0) return;
				std::vector<int64_t> qoff((size_t)nq + 1);
				for (int32_t j = 0; j <= nq; ++j) qoff[j] = query_off[q0 + j] - query_off[q0];
				const char* qbase = (const char*)queries + query_off[q0];
				ssw_engine* e = g->eng[d];
				S.rc = table ? ssw_engine_set_sequences_text(e, nq, qbase, qoff.data(), n_refs, (const char*)refs, ref_off, table, P.n, add_rc ? 1 : 0)
				             : ssw_engine_set_sequences(e, nq, (const int8_t*)qbase, qoff.data(), n_refs, (const int8_t*)refs, ref_off);
				if (S.rc) return;
				S.rc = ssw_engine_search_all(e, &P, min_score, max_hits, &S.set);      /* each block alone is bounded by the total's bound */
			}
			catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] device group: %s\n", ex.what()); S.rc = -1; }
			catch (...) { S.rc = -1; }
		};
		for_each_device(g, work);
		for (const HitPart& S : parts) if (S.rc) return S.rc;
		/* rows in query order -- every block's queries, then (reverse complements) every block's second half -- keep pair order */
		std::vector<std::pair<int, int32_t>> rows;
		rows.reserve((size_t)n_queries * (add_rc ? 2 : 1));
		for (int half = 0; half < (add_rc ? 2 : 1); ++half)
			for (int d = 0; d < world; ++d) {
				const int32_t nq = (int32_t)(b[d + 1] - b[d]);
				for (int32_t l = half * nq; l < (half + 1) * nq; ++l) rows.emplace_back(d, l);
			}
		return gather_hits("ssw_group_search_all", parts, rows, max_hits, out);
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_group_search_all: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

extern "C" int ssw_group_search_self(ssw_group* g, const ssw_batch_params* params, int32_t n, const int8_t* seqs, const int64_t* off,
                                     int32_t min_score, int64_t max_hits, ssw_hit_set** out)
{
	if (!out) { fprintf(stderr, "[libssw-b200] ssw_group_search_self: NULL output\n"); return -1; }
	*out = nullptr;
	if (!g || g->eng.empty() || !params) { fprintf(stderr, "[libssw-b200] ssw_group_search_self: NULL argument\n"); return -1; }
	if (n < 0 || (n > 0 && (!seqs || !off))) { fprintf(stderr, "[libssw-b200] ssw_group_search_self: no sequences\n"); return -1; }
	try {
		for (int32_t i = 0; i < n; ++i) if (off[i + 1] < off[i]) { fprintf(stderr, "[libssw-b200] offsets are not non-decreasing at %d\n", i); return -1; }
		/* canonical order (length, then index) and the triangle cells of each rank: its length times the letters ranked after it */
		std::vector<int32_t> canon((size_t)n), rank((size_t)n);
		for (int32_t i = 0; i < n; ++i) canon[i] = i;
		auto len = [&](int32_t i) { return off[i + 1] - off[i]; };
		std::sort(canon.begin(), canon.end(), [&](int32_t x, int32_t y) { return len(x) != len(y) ? len(x) < len(y) : x < y; });
		for (int32_t t = 0; t < n; ++t) rank[canon[t]] = t;
		std::vector<long double> cells((size_t)n);
		long double later = 0;
		for (int32_t t = n - 1; t >= 0; --t) { cells[t] = (long double)len(canon[t]) * later; later += len(canon[t]); }
		const int world = (int)g->eng.size();
		const std::vector<int64_t> b = balanced_bounds(n, world, [&](int64_t t) { return cells[t]; });
		std::vector<HitPart> parts((size_t)world);
		auto work = [&](int d) {
			HitPart& S = parts[d];
			try {
				ssw_engine* e = g->eng[d];
				S.rc = ssw_engine_set_sequences_self(e, n, seqs, off);
				if (S.rc) return;
				S.rc = ssw_engine_search_self_ranks(e, params, min_score, max_hits, (int32_t)b[d], (int32_t)b[d + 1], &S.set);
			}
			catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] device group: %s\n", ex.what()); S.rc = -1; }
			catch (...) { S.rc = -1; }
		};
		for_each_device(g, work);
		for (const HitPart& S : parts) if (S.rc) return S.rc;
		/* row i comes from the device whose rank range holds rank[i] */
		std::vector<std::pair<int, int32_t>> rows((size_t)n);
		for (int32_t i = 0; i < n; ++i) rows[i] = {(int)(std::upper_bound(b.begin(), b.end(), (int64_t)rank[i]) - b.begin()) - 1, i};
		return gather_hits("ssw_group_search_self", parts, rows, max_hits, out);
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_group_search_self: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}

extern "C" int ssw_group_align_batch(ssw_group* g, const ssw_batch_params* params, const int8_t* table, int32_t add_reverse_complement,
                                     int32_t n_queries, const void* queries, const int64_t* query_off,
                                     int32_t n_refs, const void* refs, const int64_t* ref_off,
                                     int64_t n_pairs, const int32_t* pair_query, const int32_t* pair_ref,
                                     s_align** out, int32_t marked, int32_t* nm)
{
	if (!g || g->eng.empty() || !params || (n_pairs > 0 && !out)) return -1;
	try {
		const Job J = make_job(params, table, add_reverse_complement, n_queries, queries, query_off, n_refs, refs, ref_off, n_pairs, pair_query, pair_ref, marked);
		std::vector<Shard> shards;
		const int rc = run_job(g, J, shards, nullptr);
		if (rc) return rc;
		for (const Shard& S : shards)
			for (int64_t l = 0; l < S.pairs(); ++l) {
				const int64_t p = global_pair(J, S, l);
				out[p] = ssw_record_from(S.records()[l], S.pool.get());
				if (nm) nm[p] = S.nm.empty() ? 0 : S.nm[l];
			}
		return 0;
	}
	catch (const std::exception& ex) { fprintf(stderr, "[libssw-b200] ssw_group_align_batch: %s\n", ex.what()); return -1; }
	catch (...) { return -1; }
}
