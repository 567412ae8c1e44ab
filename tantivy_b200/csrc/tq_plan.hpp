// The batch planner (tq_plan.cpp): what the stages of batch_prepare_impl (tq_engine.cu) hand on to each other.  A batch's
// queries are validated, their clauses resolved to cached tables, and each query is routed to a tile group or to the per-query
// kernels; its (query, segment) pairs are cut into work units and the tile groups staged.  lay_out (tq_engine.cu) turns the
// plan into descriptors on the device.  Host code only.
#pragma once
#include <unordered_map>
#include <vector>

#include "tq_engine_internal.hpp"

namespace tq::host {

constexpr int kTileRounds = 4;  // launches of k_tile per run: the sample launch + three exact ones

// Unit classes of the per-query kernels: the order of tq_batch::n_units / unit_base and of the batch's Unit array.
enum UnitClass : int {
  UC_TERM = TQ_OP_TERM, UC_AND = TQ_OP_AND, UC_OR_WINDOW = TQ_OP_OR,  // k_term, k_and, k_or
  UC_STRIP, UC_STRIP_ROUND1, UC_STRIP_ROUND2, UC_STRIP_ROUND3,        // k_or_strip: main launch (last phase), threshold rounds (phases 0..2)
  UC_PHRASE, UC_CLASSES                                               // k_phrase
};

// One (query, segment) of the plan: its clauses in evaluation order with their block tables resolved.
struct SegPlan {
  uint32_t segment_ord = 0;
  const Segment* seg = nullptr;
  struct Clause { uint32_t first; QList second; uint32_t range_len; };  // doc_freq, clause, bytes of its postings range
  std::vector<Clause> here;
  std::vector<uint32_t> term_idx;  // clause ordinals in arrival order (phrases: before `here` is sorted)
  std::vector<uint16_t> bool_words;  // TQ_OP_BOOL: [n_groups, need_should, n_should, n_not, (len, clauses..) per group, shoulds.., nots..],
                                     // clauses as indices into `here` (tile_admit turns them into slots)
  const uint8_t* fn0 = nullptr;
  const uint8_t* alive = nullptr;      // the docs the query may collect here: the segment's alive bitset, or its filter view's
  const FilterView* view = nullptr;    // TQ_QUERY_FILTER: the view (its non-empty tiles)
  uint32_t no_freq = 0;  // bit a: the a-th clause in arrival order does not read freqs (Basic field or TQ_TERM_IGNORE_FREQ)
  // AND / BOOL: the MUST scorers add up as Intersection::score does, (s0 + s1) + (s2 + s3 + ...), instead of one after another
  // as in block_wand_intersection (oracle/query.hpp, for_each_intersection, says when the reference takes which)
  bool uniform_fn = true, prunable = false, intersection_order = false;
};

// A group of queries that k_tile evaluates together (shared decode, see tq_tile.cuh), while it is being planned.
struct TileGroupBuild {
  struct SegB {
    uint32_t segment_ord = 0, max_doc = 0;
    uint32_t t_lo = 0, t_hi = 0;  // tiles that overlap the segment's doc range (tq_segment_set_doc_range)
    const uint8_t* alive = nullptr;
    const FilterView* view = nullptr;  // the group's filter (one per group): its launches visit only the view's tile runs
    std::vector<TSlot> slots;  // (TSlot::pad chains the slots of one list: several weights / tables of a list are rare)
    std::vector<TQuery> queries;
    std::vector<uint16_t> clauses;
    double dens = 0;  // sum of doc_freq / max_doc over the slots: expected pairs per doc
  };
  std::vector<SegB> segs;
  // (segment_ord, field of the plan's alive words) -> index in segs: fields of one ordinal may differ in doc range, alive copy
  // and filter view, so each field a query's plan takes them from has its own entry
  std::unordered_map<uint64_t, uint32_t> seg_of;
  static uint64_t seg_key(const SegPlan& sp) { return (uint64_t)sp.segment_ord << 32 | sp.seg->field; }
  // list id -> first slot of that list in its home entry slot_home[list id] (kNoSlot: in no entry).  A list lives in one
  // (segment, field), but a query whose clauses span fields brings it into the entry of another field too: there it is looked up
  // among the entry's slots.
  std::vector<uint32_t> slot_head, slot_home;
  uint32_t find_slot(uint32_t si, const QList& ql) const {
    if (ql.list_id >= slot_head.size() || slot_head[ql.list_id] == kNoSlot) return kNoSlot;
    const SegB& sb = segs[si];
    auto same = [&](const TSlot& sl) { return memcmp(&sl.weight, &ql.weight, 4) == 0 && sl.cache_idx == ql.cache_idx; };
    if (slot_home[ql.list_id] != si) {
      for (uint32_t s = 0; s < sb.slots.size(); ++s)
        if (sb.slots[s].list_id == ql.list_id && same(sb.slots[s])) return s;
      return kNoSlot;
    }
    for (uint32_t s = slot_head[ql.list_id]; s != kNoSlot; s = sb.slots[s].pad)
      if (same(sb.slots[s])) return s;
    return kNoSlot;
  }
  uint64_t pairs = 0;                              // elements of the pair arrays (doc_freq rounded up to 128 per slot)
  uint64_t list_bytes = 0;                         // postings-range bytes of the distinct lists
};

// A tile group as the device reads it: slots in their final order, TSegs, TQuerys, clause words, the units of its launches and
// the score chunks of k_score_lists.
struct GroupStage {
  std::vector<TSlot> slots;
  std::vector<TSeg> segs;
  std::vector<TQuery> queries;
  std::vector<uint16_t> clauses;
  std::vector<TUnit> units[kTileRounds];
  std::vector<TUnit> count_units;     // k_count_tiles: every tile of the segments that hold a TQ_QUERY_COUNT_HITS query
  std::vector<uint32_t> count_queries;  // batch ordinals of those queries
  std::vector<SChunk> chunks;
  uint32_t max_slots = 1, p_cap = 1024, max_big = 1, max_queries = 1, max_clause_words = 0, max_clauses = 1;
  size_t tix_words = 0;
  bool union_only = true;  // every TQuery is a term query or a union (k_tile<*, *, true>)
};

// A (query, segment) of the per-query kernels, beside its QSeg: its unit class, the blocks / windows / tiles its units cover, and
// whether it is a strip pair with a threshold sample pass (MaxScore can then skip its dense clauses).
struct SegWork { UnitClass cls; uint32_t total; bool sample; };

// The Count collector's work for a set of queries: the (query, segment) pairs of k_count with their structure words (list ids in
// place of the clause indices), one unit per 8 tiles of 8192 docs.
struct CountPlan {
  std::vector<uint32_t> words;
  std::vector<CountSeg> segs;
  std::vector<uint32_t> segment_ords;  // parallel to segs
  std::vector<Unit> units;
  bool mixed = false;  // some pair has SHOULD or MUST_NOT clauses: k_count<true>
};

// The plan of one batch: what the stages of batch_prepare_impl hand on to each other.
struct BatchPlan {
  const tq_query* queries = nullptr;
  size_t nq = 0;
  int repeat = 0;
  bool terms_on_tile = false;
  std::vector<DQuery> dq;
  std::vector<size_t> q_cands;                          // candidate-region size per query
  std::vector<float> caches;                            // n_caches * 256
  std::unordered_map<uint32_t, uint32_t> cache_by_avg;  // avg bits -> cache idx
  uint32_t last_avg_bits = 0, last_avg_idx = 0xFFFFFFFFu;
  std::vector<const tq_term_seg*> order;  // reused from query to query
  std::vector<SegPlan> plans;             // the current query's, n_plans live entries (reused from query to query)
  size_t n_plans = 0;
  // per-query kernels
  std::vector<QList> qlists;
  std::vector<QSeg> qsegs;
  std::vector<SegWork> work;    // parallel to qsegs
  std::vector<PhraseAux> qaux;  // parallel to qlists once a phrase query shows up
  std::vector<Unit> units[UC_CLASSES];
  uint32_t n_qsegs_op[4] = {0, 0, 0, 0};  // (query, segment) pairs of k_term, k_and + k_phrase, k_or, k_or_strip
  uint32_t strip_cached_max = 0, phrase_ct = 2;
  // tile engine
  std::vector<TileGroupBuild> tgroups;
  std::unordered_map<uint64_t, size_t> open_group;  // filter key (0: none, 1 << 32 | filter_id) -> the group that takes its next queries
  std::vector<GroupStage> gstage;  // parallel to tgroups
  uint64_t tile_pairs_total = 0, pair_cursor = 0, tile_postings = 0, tile_units = 0;
  size_t tix_total_words = 0, tile_bytes = 0;
  // TQ_QUERY_COUNT_HITS (not in a repeat: the hits of the original run stand): the queries on the per-query kernels are counted
  // by k_count (count), the doc_freq shortcuts go to hits_host; the tile groups' queries by k_count_tiles
  bool count_hits = false;
  CountPlan count;
  std::vector<uint64_t> hits_host;
  // totals
  uint64_t built = 0, alg_bytes = 0, postings = 0, op_bytes[3] = {0, 0, 0};
  uint32_t kmax = 1;
  size_t n_cands = 0;
};

// Validates query qi and plans it: into a tile group, or onto the per-query kernels.  ctx->mu held.
int plan_query(tq_ctx* c, BatchPlan& pl, size_t qi);
// Cuts the per-query kernels' (query, segment) pairs into work units, then lays out the candidate regions.
int cut_units(const tq_ctx* c, BatchPlan& pl);
// Tile groups: slot order, pair bases, score chunks, tile ranges of the launches.
int stage_tile_groups(const tq_ctx* c, BatchPlan& pl);
// The Count work of query qi: its (query, segment) pairs go to cp, doc_freq shortcuts to *host_add -- none with all_docs (a sort
// needs every matching doc, not only how many there are).  ctx->mu held.
int plan_count(tq_ctx* c, const tq_query& q, uint32_t qi, std::vector<const tq_term_seg*>& order, CountPlan& cp, uint64_t* host_add,
               bool all_docs = false);

}  // namespace tq::host
