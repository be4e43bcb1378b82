/*
 * ssw_cpp.cpp -- StripedSmithWaterman::Aligner over the H100-native libssw.so (include/ssw_cpp.h).
 * Behaviour follows the reference's wrapper (src/ssw_cpp.cpp): default tables :18-50, flag derivation :222-229,
 * the result conversion with soft clips :52-88 and the '='/'X' rewrite with the mismatch count :127-220,
 * AlignImpl :334-369, Clear/ReBuild :371-419.  Host-only code; the alignment itself runs on the GPU.
 */
#include "../../include/ssw_cpp.h"

#include <string.h>

#include <algorithm>
#include <map>
#include <mutex>

#include "../../include/ssw.h"
#include "../../include/ssw_batch.h"

namespace StripedSmithWaterman {
namespace {

uint8_t flag_of(const Filter& f)
{
	uint8_t flag = 0;
	if (f.report_begin_position) flag |= 0x08;
	if (f.report_cigar) flag |= 0x0f;
	return flag;
}

struct CigarWriter {
	std::vector<uint32_t> words;
	std::string text;
	void put(uint32_t len, char op)
	{
		if (!len) return;
		words.push_back(to_cigar_int(len, op));
		text += std::to_string(len);
		text += op;
	}
};

/* s_align -> Alignment: copy the fields, then rewrite the path: soft clips for the unaligned query ends, every M run
 * split into '=' and 'X' runs by comparing the codes, mismatches = X columns + inserted + deleted bases.
 * (The clips are written even when no path was requested, as the reference does, ssw_cpp.cpp:142-146, :206-211.) */
void convert(const s_align& a, const int8_t* ref, const int8_t* query, int32_t query_len, Alignment& out)
{
	out = Alignment();
	out.sw_score = a.score1;
	out.sw_score_next_best = a.score2;
	out.ref_begin = a.ref_begin1;
	out.ref_end = a.ref_end1;
	out.query_begin = a.read_begin1;
	out.query_end = a.read_end1;
	out.ref_end_next_best = a.ref_end2;

	CigarWriter w;
	if (a.read_begin1 > 0) w.put((uint32_t)a.read_begin1, 'S');
	int64_t r = a.ref_begin1, q = a.read_begin1;
	int32_t edits = 0;
	uint32_t run = 0;             /* current '=' or 'X' run; it continues across adjacent M words (ssw_cpp.cpp:153-187) */
	bool run_equal = true;
	for (int32_t i = 0; i < a.cigarLen; ++i) {
		const char op = cigar_int_to_op(a.cigar[i]);
		const uint32_t len = cigar_int_to_len(a.cigar[i]);
		if (op == 'M') {
			for (uint32_t k = 0; k < len; ++k, ++r, ++q) {
				const bool equal = ref[r] == query[q];
				if (run && equal != run_equal) { w.put(run, run_equal ? '=' : 'X'); run = 0; }
				run_equal = equal;
				++run;
				if (!equal) ++edits;
			}
		} else if (op == 'I' || op == 'D') {
			w.put(run, run_equal ? '=' : 'X');
			run = 0;
			w.put(len, op);
			(op == 'I' ? q : r) += len;
			edits += (int32_t)len;
		}
	}
	w.put(run, run_equal ? '=' : 'X');
	const int32_t tail = query_len - a.read_end1 - 1;
	if (tail > 0) w.put((uint32_t)tail, 'S');
	out.cigar.swap(w.words);
	out.cigar_string.swap(w.text);
	out.mismatches = edits;
}

/* the same for a record whose CIGAR was already marked on the device (ssw_align_batch_marked): clips, '=' / 'X' runs and the
 * mismatch count are there, only the text form is made here */
void convert_marked(const s_align& a, int32_t nm, Alignment& out)
{
	out = Alignment();
	out.sw_score = a.score1;
	out.sw_score_next_best = a.score2;
	out.ref_begin = a.ref_begin1;
	out.ref_end = a.ref_end1;
	out.query_begin = a.read_begin1;
	out.query_end = a.read_end1;
	out.ref_end_next_best = a.ref_end2;
	CigarWriter w;
	for (int32_t i = 0; i < a.cigarLen; ++i) w.put(cigar_int_to_len(a.cigar[i]), cigar_int_to_op(a.cigar[i]));
	out.cigar.swap(w.words);
	out.cigar_string.swap(w.text);
	out.mismatches = nm;
}

}  // namespace

void Aligner::DefaultTables()
{
	/* 5 x 5 over A C G T N: match on the diagonal of the four bases, the mismatch penalty everywhere else */
	alphabet_ = 5;
	scores_.assign(25, (int8_t)-mismatch_);
	for (int b = 0; b < 4; ++b) scores_[b * 5 + b] = (int8_t)match_;
	char_code_.assign(128, 4);
	const char* bases = "ACGT";
	for (int b = 0; b < 4; ++b) { char_code_[(int)bases[b]] = (int8_t)b; char_code_[(int)bases[b] + 32] = (int8_t)b; }
}

Aligner::Aligner() { DefaultTables(); }

Aligner::Aligner(uint8_t match_score, uint8_t mismatch_penalty, uint8_t gap_opening_penalty, uint8_t gap_extending_penalty)
    : match_(match_score), mismatch_(mismatch_penalty), gap_open_(gap_opening_penalty), gap_extend_(gap_extending_penalty)
{
	DefaultTables();
}

Aligner::Aligner(const int8_t* score_matrix, int score_matrix_size, const int8_t* translation_matrix, int translation_matrix_size)
    : alphabet_(score_matrix_size),
      scores_(score_matrix, score_matrix + (size_t)score_matrix_size * score_matrix_size),
      char_code_(translation_matrix, translation_matrix + translation_matrix_size)
{
}

void Aligner::Encode(const char* s, size_t n, std::vector<int8_t>& codes) const
{
	codes.resize(n);
	for (size_t i = 0; i < n; ++i) codes[i] = char_code_[(unsigned char)s[i]];
}

size_t Aligner::SetReferenceSequence(const char* ref, size_t ref_len)
{
	ref_codes_.clear();
	if (!char_code_.empty()) Encode(ref, ref_len, ref_codes_);
	return ref_codes_.size();
}

size_t Aligner::SetReferenceSequence(const char* ref) { return SetReferenceSequence(ref, strlen(ref)); }

void Aligner::ClearReferenceSequence() { ref_codes_.clear(); }

void Aligner::SetGapPenalty(uint8_t opening, uint8_t extending)
{
	gap_open_ = opening;
	gap_extend_ = extending;
}

uint16_t Aligner::Run(const char* query, size_t query_len, const std::vector<int8_t>& ref_codes, const Filter& filter,
                      Alignment& alignment, int32_t maskLen) const
{
	if (char_code_.empty()) return 0;
	std::vector<int8_t> q;
	Encode(query, query_len, q);
	s_profile* prof = ssw_init(q.data(), (int32_t)q.size(), scores_.data(), alphabet_, 2);
	s_align* a = ssw_align(prof, ref_codes.data(), (int32_t)ref_codes.size(), gap_open_, gap_extend_, flag_of(filter),
	                       filter.score_filter, filter.distance_filter, std::max(maskLen, 15));
	uint16_t rc = 1;
	if (a) {
		convert(*a, ref_codes.data(), q.data(), (int32_t)q.size(), alignment);
		rc = a->flag;
		align_destroy(a);
	} else {
		alignment = Alignment();   /* no usable device / failed call: the library has already said why on stderr */
	}
	init_destroy(prof);
	return rc;
}

uint16_t Aligner::Align(const char* query, size_t query_len, const Filter& filter, Alignment& alignment, int32_t maskLen) const
{
	if (ref_codes_.empty() || query_len == 0) return 0;
	return Run(query, query_len, ref_codes_, filter, alignment, maskLen);
}

uint16_t Aligner::Align(const char* query, const Filter& filter, Alignment& alignment, int32_t maskLen) const
{
	return Align(query, strlen(query), filter, alignment, maskLen);
}

uint16_t Aligner::Align(const char* query, size_t query_len, const char* ref, size_t ref_len, const Filter& filter,
                        Alignment& alignment, int32_t maskLen) const
{
	if (char_code_.empty() || ref_len == 0 || query_len == 0) return 0;
	std::vector<int8_t> r;
	Encode(ref, ref_len, r);
	return Run(query, query_len, r, filter, alignment, maskLen);
}

uint16_t Aligner::Align(const char* query, const char* ref, const Filter& filter, Alignment& alignment, int32_t maskLen) const
{
	return Align(query, strlen(query), ref, strlen(ref), filter, alignment, maskLen);
}

namespace {
/* device groups of AlignBatch(devices != 1): made on first use, one per device count, shared by all aligners of the
 * process (a group runs one batch at a time) */
std::mutex g_group_mu;
std::map<int32_t, ssw_group*> g_groups;
}

bool Aligner::AlignBatch(const std::vector<std::string>& queries, const Filter& filter, std::vector<Alignment>& alignments,
                         std::vector<uint16_t>* flags, int32_t maskLen, int32_t devices) const
{
	alignments.assign(queries.size(), Alignment());
	if (flags) flags->assign(queries.size(), 0);
	if (char_code_.empty() || ref_codes_.empty() || queries.empty()) return false;
	/* empty queries are skipped like Align() skips them: only the non-empty ones enter the batch */
	std::vector<int8_t> codes;
	std::vector<int64_t> off(1, 0);
	std::vector<size_t> origin;
	for (size_t i = 0; i < queries.size(); ++i) {
		if (queries[i].empty()) continue;
		for (char c : queries[i]) codes.push_back(char_code_[(unsigned char)c]);
		off.push_back((int64_t)codes.size());
		origin.push_back(i);
	}
	if (origin.empty()) return false;
	ssw_batch_params P;
	memset(&P, 0, sizeof P);
	P.mat = scores_.data(); P.n = alphabet_; P.gap_open = gap_open_; P.gap_extend = gap_extend_;
	P.flag = flag_of(filter); P.filters = filter.score_filter; P.filterd = filter.distance_filter;
	P.mask_len = maskLen < 0 ? -1 : std::max(maskLen, 15); P.score_size = 2;
	const int64_t roff[2] = {0, (int64_t)ref_codes_.size()};
	std::vector<s_align*> res(origin.size(), nullptr);
	std::vector<int32_t> nm(origin.size(), 0);
	/* the '=' / 'X' expansion, the soft clips and the mismatch counts of every path come from the device (ssw_mark.cuh) */
	if (devices == 1) {
		if (ssw_align_batch_marked(nullptr, &P, (int32_t)origin.size(), codes.data(), off.data(), 1, ref_codes_.data(), roff,
		                           (int64_t)origin.size(), nullptr, nullptr, res.data(), nm.data()))
			return false;
	} else {
		std::lock_guard<std::mutex> lock(g_group_mu);
		ssw_group*& g = g_groups[devices < 0 ? 0 : devices];
		if (!g) g = ssw_group_create(devices < 0 ? 0 : devices, nullptr);
		if (!g || ssw_group_align_batch(g, &P, nullptr, 0, (int32_t)origin.size(), codes.data(), off.data(), 1, ref_codes_.data(), roff,
		                                (int64_t)origin.size(), nullptr, nullptr, res.data(), 1, nm.data()))
			return false;
	}
	for (size_t k = 0; k < origin.size(); ++k) {
		if (!res[k]) { if (flags) (*flags)[origin[k]] = 1; continue; }
		if (res[k]->cigarLen > 0) convert_marked(*res[k], nm[k], alignments[origin[k]]);
		else convert(*res[k], ref_codes_.data(), codes.data() + off[k], (int32_t)(off[k + 1] - off[k]), alignments[origin[k]]);   /* no path: clips only */
		if (flags) (*flags)[origin[k]] = res[k]->flag;
		align_destroy(res[k]);
	}
	return true;
}

void Aligner::Clear()
{
	scores_.clear();
	char_code_.clear();
	ref_codes_.clear();
}

bool Aligner::ReBuild() { return ReBuild(2, 2, 3, 1); }

bool Aligner::ReBuild(uint8_t match_score, uint8_t mismatch_penalty, uint8_t gap_opening_penalty, uint8_t gap_extending_penalty)
{
	if (!char_code_.empty()) return false;          /* only a cleared aligner can be rebuilt on default tables */
	match_ = match_score; mismatch_ = mismatch_penalty; gap_open_ = gap_opening_penalty; gap_extend_ = gap_extending_penalty;
	ref_codes_.clear();
	DefaultTables();
	return true;
}

bool Aligner::ReBuild(const int8_t* score_matrix, int score_matrix_size, const int8_t* translation_matrix, int translation_matrix_size)
{
	alphabet_ = score_matrix_size;
	scores_.assign(score_matrix, score_matrix + (size_t)score_matrix_size * score_matrix_size);
	char_code_.assign(translation_matrix, translation_matrix + translation_matrix_size);
	return true;
}

}  // namespace StripedSmithWaterman
