/*
 * ssw_cpp.h -- C++ interface of the H100-native aligner: source-compatible with the reference's
 * StripedSmithWaterman::Aligner / Filter / Alignment (reference src/ssw_cpp.h:15-62 Alignment and Filter,
 * :64-233 the public members of Aligner), so programs written against the reference's wrapper (its example.cpp)
 * compile unchanged against this header and link libssw_cpp.a + libssw.so.
 *
 * Own text; the private part differs from the reference's (programs must be recompiled, as with any C++ wrapper),
 * and one member is new: AlignBatch(), which sends many queries to the GPU in one call -- a single Align() exposes
 * one (query, reference) pair, far too little work for an H100.
 */
#ifndef SSW_B200_CPP_H
#define SSW_B200_CPP_H

#include <stddef.h>
#include <stdint.h>

#include <string>
#include <vector>

namespace StripedSmithWaterman {

/* One alignment (reference ssw_cpp.h:15-39).  Positions are 0-based; the begin positions are -1 when not computed.
 * cigar / cigar_string use '=' / 'X' for matches / mismatches and 'S' for the clipped query ends. */
struct Alignment {
  uint16_t sw_score = 0;
  uint16_t sw_score_next_best = 0;
  int32_t ref_begin = 0;
  int32_t ref_end = 0;
  int32_t query_begin = 0;
  int32_t query_end = 0;
  int32_t ref_end_next_best = 0;
  int32_t mismatches = 0;            /* mismatching columns + inserted + deleted bases */
  std::string cigar_string;
  std::vector<uint32_t> cigar;       /* BAM encoding: length << 4 | op */
};

/* What to report (reference ssw_cpp.h:41-62): report_cigar implies the begin positions; the CIGAR is only produced for
 * alignments with score >= score_filter whose reference and query spans are both < distance_filter. */
struct Filter {
  bool report_begin_position = true;
  bool report_cigar = true;
  uint16_t score_filter = 0;
  uint16_t distance_filter = 32767;
};

class Aligner {
public:
  /* {A,C,G,T,N} aligner: match 2, mismatch 2, gap open 3, gap extend 1 */
  Aligner();
  Aligner(uint8_t match_score, uint8_t mismatch_penalty, uint8_t gap_opening_penalty, uint8_t gap_extending_penalty);
  /* any alphabet: score_matrix is size x size, translation_matrix maps a character to its code */
  Aligner(const int8_t* score_matrix, int score_matrix_size, const int8_t* translation_matrix, int translation_matrix_size);

  /* keep a translated reference inside the aligner (replaces the previous one); returns its length */
  size_t SetReferenceSequence(const char* ref, size_t ref_len);
  size_t SetReferenceSequence(const char* ref);
  void ClearReferenceSequence();

  void SetGapPenalty(uint8_t opening, uint8_t extending);

  /* Align against the stored reference / a given reference.  maskLen below 15 is raised to 15.
   * Returns s_align.flag of the result (0 accurate, 1 traceback failed, 2 path may miss a part); 0 on empty input. */
  uint16_t Align(const char* query, size_t query_len, const Filter& filter, Alignment& alignment, int32_t maskLen = 0) const;
  uint16_t Align(const char* query, const Filter& filter, Alignment& alignment, int32_t maskLen = 0) const;
  uint16_t Align(const char* query, size_t query_len, const char* ref, size_t ref_len, const Filter& filter,
                 Alignment& alignment, int32_t maskLen = 0) const;
  uint16_t Align(const char* query, const char* ref, const Filter& filter, Alignment& alignment, int32_t maskLen = 0) const;

  /* NEW: all queries against the stored reference in one GPU batch.  alignments[i] is what
   * Align(queries[i], ...) returns; maskLen < 0 uses length/2 of each query (the CLI's choice, main.c:465).
   * flags (optional) receives the per-query return value of Align.  Returns false if nothing was aligned.
   * devices: GPUs of this process the batch is cut over (ssw_batch.h device groups; 1 = the current device,
   * 0 = all visible devices); the alignments do not depend on it. */
  bool AlignBatch(const std::vector<std::string>& queries, const Filter& filter, std::vector<Alignment>& alignments,
                  std::vector<uint16_t>* flags = nullptr, int32_t maskLen = 0, int32_t devices = 1) const;

  /* drop matrices and reference; ReBuild*() make the aligner usable again (the first two only after Clear()) */
  void Clear();
  bool ReBuild();
  bool ReBuild(uint8_t match_score, uint8_t mismatch_penalty, uint8_t gap_opening_penalty, uint8_t gap_extending_penalty);
  bool ReBuild(const int8_t* score_matrix, int score_matrix_size, const int8_t* translation_matrix, int translation_matrix_size);

private:
  void Encode(const char* s, size_t n, std::vector<int8_t>& codes) const;
  void DefaultTables();
  uint16_t Run(const char* query, size_t query_len, const std::vector<int8_t>& ref_codes, const Filter& filter,
               Alignment& alignment, int32_t maskLen) const;

  uint8_t match_ = 2, mismatch_ = 2, gap_open_ = 3, gap_extend_ = 1;
  int alphabet_ = 5;
  std::vector<int8_t> scores_;      /* alphabet_ x alphabet_ */
  std::vector<int8_t> char_code_;   /* character -> code; empty = aligner cleared */
  std::vector<int8_t> ref_codes_;
};

}  // namespace StripedSmithWaterman

#endif  // SSW_B200_CPP_H
