// ORACLE — TEST INFRASTRUCTURE ONLY (see codec.hpp header).
// CPU restatement of the reference's phrase scorer (SURVEY.md §8f N3), for the kernel that does not exist yet:
//   src/query/phrase_query/phrase_scorer.rs:60-139    intersection_exists / intersection_count / intersection
//   ...:145-218                                        intersection_count_with_slop, intersection_exists_with_slop
//   ...:236-345                                        intersection_count_with_carrying_slop (three and more terms)
//   ...:349-497                                        PhraseScorer::{new_with_offset, phrase_match, compute_phrase_count,
//                                                      compute_phrase_match}
//   ...:500-589                                        advance / seek / score
//   src/postings/segment_postings.rs:232-254           append_positions_with_offset
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

#include "positions.hpp"
#include "query.hpp"

namespace tqo {

inline size_t intersection_count(const std::vector<uint32_t>& left, const std::vector<uint32_t>& right) {
  size_t li = 0, ri = 0, count = 0;
  while (li < left.size() && ri < right.size()) {
    if (left[li] < right[ri]) ++li;
    else if (left[li] == right[ri]) { ++count; ++li; ++ri; }
    else ++ri;
  }
  return count;
}
inline void intersection(std::vector<uint32_t>& left, const std::vector<uint32_t>& right) {
  size_t li = 0, ri = 0, count = 0;
  const size_t ll = left.size();
  while (li < ll && ri < right.size()) {
    if (left[li] < right[ri]) ++li;
    else if (left[li] == right[ri]) { left[count++] = left[li]; ++li; ++ri; }
    else ++ri;
  }
  left.resize(count);
}
inline size_t intersection_count_with_slop(std::vector<uint32_t>& left, const std::vector<uint32_t>& right, uint32_t slop, bool update_left) {
  size_t li = 0, ri = 0, count = 0;
  const size_t ll = left.size(), rl = right.size();
  while (li < ll && ri < rl) {
    const uint32_t lv = left[li], rv = right[ri];
    const uint32_t distance = lv > rv ? lv - rv : rv - lv;
    if (distance <= slop) {
      while (li + 1 < ll) {  // there could be a better match
        if (left[li + 1] > rv) break;
        ++li;
      }
      if (update_left) left[count] = rv;
      ++count; ++li; ++ri;
    } else if (lv < rv) ++li;
    else ++ri;
  }
  if (update_left) left.resize(count);
  return count;
}
inline uint32_t intersection_count_with_carrying_slop(std::vector<uint32_t>& left, std::vector<uint8_t>& left_slops,
                                                      const std::vector<uint32_t>& right, uint32_t max_slop, bool update_left,
                                                      std::vector<uint32_t>& positions_buffer, std::vector<uint8_t>& slops_buffer) {
  size_t li = 0, ri = 0;
  uint32_t count = 0;
  if (left.empty() || right.empty()) {
    if (update_left) { left.clear(); left_slops.clear(); }
    return 0;
  }
  auto add_val = [&](uint8_t slop, uint32_t pos) {
    if (!update_left) return;
    if (!positions_buffer.empty() && positions_buffer.back() == pos) slops_buffer.back() = std::min(slops_buffer.back(), slop);
    else { positions_buffer.push_back(pos); slops_buffer.push_back(slop); }
  };
  auto slop_at = [&](size_t i) -> uint8_t { return i < left_slops.size() ? left_slops[i] : 0; };
  for (;;) {
    const uint32_t lv = left[li], rv = right[ri];
    const uint8_t slop_so_far = slop_at(li);
    const uint32_t distance = (uint32_t)slop_so_far + (lv > rv ? lv - rv : rv - lv);
    if (distance <= max_slop) {
      const bool left_smaller = lv < rv;
      const uint32_t smaller = left_smaller ? lv : rv, larger = left_smaller ? rv : lv;
      size_t sidx = left_smaller ? li : ri;
      const std::vector<uint32_t>& spos = left_smaller ? left : right;
      uint32_t new_slop = distance;
      add_val((uint8_t)new_slop, smaller);
      while (sidx + 1 < spos.size()) {
        const uint32_t next = spos[sidx + 1];
        if (next > larger) break;
        const uint32_t d2 = next > larger ? next - larger : larger - next;
        ++sidx;
        new_slop = (uint32_t)slop_so_far + d2;
        add_val((uint8_t)new_slop, next);
      }
      add_val((uint8_t)new_slop, larger);
      ++count; ++li; ++ri;
    } else if (lv < rv) ++li;
    else ++ri;
    if (li >= left.size() || ri >= right.size()) {
      if (li >= left.size()) {
        const uint32_t lv2 = left.back();
        const uint8_t s2 = left_slops.empty() ? 0 : left_slops.back();
        for (size_t r = ri; r < right.size(); ++r) {
          const uint32_t ns = (lv2 > right[r] ? lv2 - right[r] : right[r] - lv2) + (uint32_t)s2;
          if (ns <= max_slop) add_val((uint8_t)ns, right[r]);
        }
      } else {
        const uint32_t rv2 = right.back();
        for (size_t l = li; l < left.size(); ++l) {
          const uint32_t ns = (left[l] > rv2 ? left[l] - rv2 : rv2 - left[l]) + (uint32_t)slop_at(l);
          if (ns <= max_slop) add_val((uint8_t)ns, left[l]);
        }
      }
      break;
    }
  }
  if (update_left) {
    left.swap(positions_buffer);
    left_slops.swap(slops_buffer);
    positions_buffer.clear();
    slops_buffer.clear();
  }
  return count;
}

// One term of the phrase: its postings + its position stream (PostingsWithOffset over SegmentPostings).
struct PhraseTerm {
  SegmentPostings postings;
  PositionReader reader;
  uint32_t offset = 0;  // max_offset - the term's offset in the phrase
  void positions(std::vector<uint32_t>& out) {  // segment_postings.rs:232-254
    const uint32_t tf = postings.term_freq();
    uint64_t read_offset = postings.block_cursor.skip_reader.position_offset_;
    for (size_t i = 0; i < postings.cur; ++i) read_offset += postings.block_cursor.freq(i);
    out.assign(tf, 0u);
    reader.read(read_offset, out.data(), tf);
    uint32_t cum = offset;
    for (auto& o : out) { cum += o; o = cum; }
  }
};

struct PhraseScorer {
  std::vector<PhraseTerm> terms;  // in the Intersection's order: ascending size_hint (intersection.rs:40-52)
  std::vector<uint32_t> left_positions, right_positions, positions_buffer;
  std::vector<uint8_t> left_slops, slops_buffer;
  uint32_t phrase_count_ = 0;
  uint32_t slop = 0;
  uint32_t doc_ = TERMINATED;
  FieldNormReader fieldnorm_reader;
  Bm25Weight similarity_weight;

  // term_postings: (offset in the phrase, term) in any order; PhraseScorer::new_with_offset.  PhraseQuery first puts its terms
  // in offset order (phrase_query.rs:48-53, stable), so the size_hint sort below breaks ties by offset: which term is `left`
  // of a sloppy two-term count depends on it
  void init(std::vector<std::pair<uint32_t, PhraseTerm>> term_postings) {
    std::stable_sort(term_postings.begin(), term_postings.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    uint32_t max_offset = 0;
    for (auto& tp : term_postings) max_offset = std::max(max_offset, tp.first);
    for (auto& tp : term_postings) { tp.second.offset = max_offset - tp.first; terms.push_back(std::move(tp.second)); }
    std::stable_sort(terms.begin(), terms.end(), [](const PhraseTerm& a, const PhraseTerm& b) { return a.postings.size_hint() < b.postings.size_hint(); });
    doc_ = go_to_first_doc();
    if (doc_ != TERMINATED && !phrase_match()) advance();
  }
  uint32_t doc() const { return doc_; }
  uint32_t phrase_count() const { return phrase_count_; }
  Score score() const { return similarity_weight.score(fieldnorm_reader.fieldnorm_id(doc_), phrase_count_); }

  uint32_t align(uint32_t candidate) {  // leap-frog over all terms (Intersection::advance's inner loop, intersection.rs:122-191)
    for (;;) {
      bool all = true;
      for (auto& t : terms) {
        const uint32_t d = t.postings.seek(candidate);
        if (d > candidate) { candidate = d; all = false; break; }
      }
      if (candidate == TERMINATED) return TERMINATED;
      if (all) return candidate;
    }
  }
  uint32_t go_to_first_doc() {
    uint32_t c = 0;
    for (auto& t : terms) c = std::max(c, t.postings.doc());
    return c == TERMINATED ? TERMINATED : align(c);
  }
  uint32_t advance() {
    for (;;) {
      const uint32_t next = terms[0].postings.advance();
      doc_ = next == TERMINATED ? TERMINATED : align(next);
      if (doc_ == TERMINATED || phrase_match()) return doc_;
    }
  }
  bool phrase_match() {
    phrase_count_ = compute_phrase_count();
    return phrase_count_ > 0;
  }
  uint32_t compute_phrase_count() {
    compute_phrase_match();
    if (slop > 0) {
      if (terms.size() > 2)
        return intersection_count_with_carrying_slop(left_positions, left_slops, right_positions, slop, false, positions_buffer, slops_buffer);
      return (uint32_t)intersection_count_with_slop(left_positions, right_positions, slop, false);
    }
    return (uint32_t)intersection_count(left_positions, right_positions);
  }
  void compute_phrase_match() {
    terms[0].positions(left_positions);
    if (slop > 0) left_slops.clear();
    for (size_t i = 1; i + 1 < terms.size(); ++i) {
      terms[i].positions(right_positions);
      if (slop > 0) {
        if (terms.size() > 2) intersection_count_with_carrying_slop(left_positions, left_slops, right_positions, slop, true, positions_buffer, slops_buffer);
        else intersection_count_with_slop(left_positions, right_positions, slop, true);
      } else {
        intersection(left_positions, right_positions);
      }
      if (left_positions.empty()) { right_positions.clear(); return; }
    }
    terms.back().positions(right_positions);
  }
};

}  // namespace tqo
