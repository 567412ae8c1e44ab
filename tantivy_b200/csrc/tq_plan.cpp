// The batch planner: validation, clause resolution against the table caches, routing to tile groups or per-query kernels, work
// units and tile-group staging (tq_plan.hpp).  Host code only; built with the engine's host flags (-O3 -ffp-contract=off): the
// tf-norm tables it computes (bm25_tf_cache) must round exactly as before.
#include "tq_plan.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace tq::host {
namespace {

// Calls f(lists, n) per segment on the query's (clause, segment) lists with postings, by (segment, clause); stops at the first error.
// A clause names a segment once, so n <= n_terms.
template <class F>
int for_each_segment(const tq_query& q, std::vector<const tq_term_seg*>& order, F&& f) {
  order.clear();
  for (uint32_t i = 0; i < q.n_term_segs; ++i) {
    if (q.term_segs[i].term_idx >= q.n_terms) return fail(TQ_ERR_INVALID_ARGUMENT, "term_idx out of range");
    if (q.term_segs[i].doc_freq) order.push_back(&q.term_segs[i]);
  }
  std::stable_sort(order.begin(), order.end(), [](const tq_term_seg* a, const tq_term_seg* b) {
    return a->segment_ord != b->segment_ord ? a->segment_ord < b->segment_ord : a->term_idx < b->term_idx;
  });
  for (size_t i = 0, j; i < order.size(); i = j) {
    for (j = i + 1; j < order.size() && order[j]->segment_ord == order[i]->segment_ord; ++j)
      if (order[j]->term_idx == order[j - 1]->term_idx) return fail(TQ_ERR_INVALID_ARGUMENT, "duplicate (term_idx, segment_ord)");
    const int rc = f(order.data() + i, j - i);
    if (rc != TQ_OK) return rc;
  }
  return TQ_OK;
}

// Maps the clause entries of TQ_OP_BOOL structure words (layout: bool_structure) in place; header words and group lengths stay.
template <class W, class Map>
void map_bool_clauses(W* w, size_t n, Map map) {
  size_t x = 4;
  for (uint32_t g = 0; g < w[0]; ++g) {
    const size_t len = w[x++];
    for (size_t e = 0; e < len; ++e, ++x) w[x] = (W)map(w[x]);
  }
  for (; x < n; ++x) w[x] = (W)map(w[x]);
}

// BooleanWeight::complex_scorer for ONE segment (boolean_weight.rs:236-431), term leaves only: `here` = the clauses that have
// postings in the segment (term_idx / doc_freq / weight per entry).  Clauses without postings are EmptyScorers -- removed before
// anything is counted; an empty MUST group empties the query in this segment.  Writes
//   [n_groups, need_should, n_should, n_not, (len, entries..) per MUST group, SHOULD entries.., MUST_NOT entries..]
// (entries = indices into `here`; groups by ascending cost = Intersection's order, entries by descending weight = the union order)
// and returns 1; 0 when nothing can match in this segment; -1 on a bad Occur.  *intersection_order: the groups add up as
// Intersection::score does -- everywhere but in the shape that reaches block_wand_intersection (boolean_weight.rs:312-340):
// >= 2 MUST groups of one TermScorer each that reads freqs (bit a of `no_freq` clear), no SHOULD and no MUST_NOT scorer left.
int bool_structure(const tq_query& q, const uint32_t* term_idx, const uint32_t* dfs, const float* ws, size_t n_here, uint32_t no_freq,
                   std::vector<uint16_t>& words, bool* intersection_order) {
  struct Grp { uint32_t id, first; uint64_t cost; std::vector<uint16_t> cl; };
  std::vector<Grp> groups;
  std::vector<uint16_t> shoulds, nots;
  for (uint32_t t = 0; t < q.n_terms; ++t) {  // declared MUST groups, present or not
    if (q.term_occur[t] > TQ_OCCUR_MUST_NOT) return -1;
    if (q.term_occur[t] != TQ_OCCUR_MUST) continue;
    const uint32_t id = q.term_group ? q.term_group[t] : 256u + t;
    bool known = false;
    for (auto& g : groups) known = known || g.id == id;
    if (!known) groups.push_back(Grp{id, t, 0, {}});
  }
  for (size_t a = 0; a < n_here; ++a) {
    const uint32_t t = term_idx[a];
    if (q.term_occur[t] == TQ_OCCUR_MUST) {
      const uint32_t id = q.term_group ? q.term_group[t] : 256u + t;
      for (auto& g : groups) if (g.id == id) { g.cl.push_back((uint16_t)a); g.cost += dfs[a]; }
    } else (q.term_occur[t] == TQ_OCCUR_SHOULD ? shoulds : nots).push_back((uint16_t)a);
  }
  for (auto& g : groups) if (g.cl.empty()) return 0;
  uint32_t m = q.min_should_match;
  if (m > shoulds.size()) return 0;
  if (m >= 2 && m == shoulds.size()) {  // as many as there are SHOULD clauses: they are MUST clauses (boolean_weight.rs:287-292)
    for (uint16_t a : shoulds) groups.push_back(Grp{512u + a, term_idx[a], dfs[a], {a}});
    shoulds.clear();
    m = 0;
  }
  if (groups.empty() && shoulds.empty()) return 0;
  bool sequential = groups.size() >= 2 && shoulds.empty() && nots.empty();
  for (auto& g : groups) sequential = sequential && g.cl.size() == 1 && !((no_freq >> g.cl[0]) & 1u);
  *intersection_order = !sequential && groups.size() >= 4;  // (with fewer groups both orders give the same sum)
  const uint32_t need = m >= 1 ? m : (groups.empty() ? 1u : 0u);
  auto by_weight = [&](std::vector<uint16_t>& v) { std::stable_sort(v.begin(), v.end(), [&](uint16_t x, uint16_t y) { return ws[x] > ws[y]; }); };
  std::stable_sort(groups.begin(), groups.end(), [](const Grp& x, const Grp& y) { return x.cost < y.cost; });
  words.clear();
  words.push_back((uint16_t)groups.size());
  words.push_back((uint16_t)need);
  words.push_back((uint16_t)shoulds.size());
  words.push_back((uint16_t)nots.size());
  for (auto& g : groups) {
    by_weight(g.cl);
    words.push_back((uint16_t)g.cl.size());
    for (uint16_t a : g.cl) words.push_back(a);
  }
  by_weight(shoulds);
  for (uint16_t a : shoulds) words.push_back(a);
  for (uint16_t a : nots) words.push_back(a);
  return 1;
}

// Would the group still satisfy k_tile's limits with this query added?  exact = false counts every clause as a new list: a cheap
// sufficient test that most queries pass.  exact = true: a clause whose list already has a slot in the group adds nothing.
bool tile_fits(const tq_ctx* c, const TileGroupBuild& g, const SegPlan* plans, size_t n_plans, uint32_t max_queries, bool exact) {
  for (size_t pi = 0; pi < n_plans; ++pi) {
    const SegPlan& sp = plans[pi];
    auto it = g.seg_of.find(TileGroupBuild::seg_key(sp));
    const TileGroupBuild::SegB* sb = it == g.seg_of.end() ? nullptr : &g.segs[it->second];
    if (sb && sb->queries.size() + 1 > max_queries) return false;
    size_t n_slots = sb ? sb->slots.size() : 0;
    double dens = sb ? sb->dens : 0.0;
    for (auto& h : sp.here) {
      if (exact && sb && g.find_slot(it->second, h.second) != kNoSlot) continue;
      ++n_slots;
      dens += (double)h.first / std::max(1u, sp.seg->max_doc);
    }
    if (n_slots > c->tile_max_slots) return false;
    if (dens * kTile * 1.5 + 256.0 > (double)kTileMaxPairs || (c->tile_max_dens_x1000 && dens * 1000.0 > c->tile_max_dens_x1000)) return false;
  }
  return true;
}

// Adds the query to the group (count: k_count_tiles counts its hits); returns the number of new pair elements it brought.
uint64_t tile_admit(TileGroupBuild& g, uint32_t query, int op, bool count, const SegPlan* plans, size_t n_plans) {
  const uint64_t pairs_before = g.pairs;
  for (size_t pi = 0; pi < n_plans; ++pi) {
    const SegPlan& sp = plans[pi];
    auto it = g.seg_of.find(TileGroupBuild::seg_key(sp));
    if (it == g.seg_of.end()) {
      it = g.seg_of.emplace(TileGroupBuild::seg_key(sp), (uint32_t)g.segs.size()).first;
      g.segs.emplace_back();
      g.segs.back().segment_ord = sp.segment_ord;
      g.segs.back().max_doc = sp.seg->max_doc;
      g.segs.back().alive = sp.alive;
      g.segs.back().view = sp.view;
      g.segs.back().t_lo = sp.seg->doc_lo / kTile;
      g.segs.back().t_hi = (uint32_t)(((uint64_t)sp.seg->doc_hi + kTile - 1) / kTile);
    }
    TileGroupBuild::SegB& sb = g.segs[it->second];
    TQuery tq;
    tq.query = query;
    tq.clause_base = (uint32_t)sb.clauses.size();
    tq.n_clauses = (uint16_t)(op == TQ_OP_BOOL ? sp.bool_words.size() : sp.here.size());
    tq.op = (uint8_t)(op == TQ_OP_BOOL ? kTileOpBool : op);
    tq.flags = (sp.prunable ? 1u : 0u) | (sp.intersection_order ? 4u : 0u) | (count ? kTileQueryCount : 0u);
    uint16_t slot_of_here[TQ_MAX_TERMS];
    size_t hi_idx = 0;
    for (auto& h : sp.here) {
      uint32_t slot = g.find_slot(it->second, h.second);
      if (slot == kNoSlot) {
        slot = (uint32_t)sb.slots.size();
        TSlot sl{};
        sl.list_id = h.second.list_id; sl.weight = h.second.weight; sl.cache_idx = h.second.cache_idx; sl.doc_freq = h.first;
        sl.big = kNoSlot;
        sl.pad = kNoSlot;
        if (h.second.list_id >= g.slot_head.size()) {
          g.slot_head.resize((size_t)h.second.list_id + 1024, kNoSlot);
          g.slot_home.resize((size_t)h.second.list_id + 1024, kNoSlot);
        }
        if (g.slot_head[h.second.list_id] == kNoSlot) g.slot_home[h.second.list_id] = it->second;
        if (g.slot_home[h.second.list_id] == it->second) {  // chain (in the home entry)
          sl.pad = g.slot_head[h.second.list_id];
          g.slot_head[h.second.list_id] = slot;
        }
        sb.slots.push_back(sl);
        sb.dens += (double)h.first / std::max(1u, sp.seg->max_doc);
        g.pairs += ((uint64_t)h.first + 127) / 128 * 128;
        g.list_bytes += h.range_len;
      }
      slot_of_here[hi_idx++] = (uint16_t)slot;
      if (op != TQ_OP_BOOL) sb.clauses.push_back((uint16_t)slot);
    }
    if (op == TQ_OP_BOOL) {  // the structure words stay, the clause indices become slots
      const size_t at = sb.clauses.size();
      sb.clauses.insert(sb.clauses.end(), sp.bool_words.begin(), sp.bool_words.end());
      map_bool_clauses(sb.clauses.data() + at, sp.bool_words.size(), [&](uint16_t a) { return slot_of_here[a]; });
    }
    sb.queries.push_back(tq);
  }
  return g.pairs - pairs_before;
}

// The fields of one segment ordinal that a query's clauses name must hold the same docs: a (query, segment) collects from one
// field's alive words (doc range included) and covers one max_doc.
bool same_docs(const Segment& a, const Segment& b) { return a.max_doc == b.max_doc && a.doc_lo == b.doc_lo && a.doc_hi == b.doc_hi; }
int fail_fields() {
  return fail(TQ_ERR_INVALID_ARGUMENT, "the clauses of a query name fields of one segment that differ in max_doc or doc range");
}

// tq_stats' bytes_term / bytes_and / bytes_or class of a query shape: phrases count as AND, mixed boolean queries as OR.
int bytes_class(int op) { return op == TQ_OP_PHRASE ? TQ_OP_AND : (op == TQ_OP_BOOL ? TQ_OP_OR : op); }

// The shape of a query for search (phrase_ok) and for Count, which has no phrase path.
int check_shape(const tq_query& q, bool phrase_ok) {
  if (q.n_terms == 0 || q.n_terms > TQ_MAX_TERMS) return fail(TQ_ERR_INVALID_ARGUMENT, "n_terms must be in 1..TQ_MAX_TERMS");
  if (q.op != TQ_OP_TERM && q.op != TQ_OP_AND && q.op != TQ_OP_OR && q.op != TQ_OP_BOOL && !(phrase_ok && q.op == TQ_OP_PHRASE))
    return fail(TQ_ERR_INVALID_ARGUMENT, "op");
  if (q.op == TQ_OP_TERM && q.n_terms != 1) return fail(TQ_ERR_INVALID_ARGUMENT, "TQ_OP_TERM takes one term");
  return TQ_OK;
}

int validate_query(const tq_ctx* c, const tq_query& q) {
  if (q.k == 0 || q.k > TQ_MAX_K) return fail(TQ_ERR_INVALID_ARGUMENT, "k must be in 1..TQ_MAX_K");
  const int rc = check_shape(q, true);
  if (rc != TQ_OK) return rc;
  if (q.op == TQ_OP_BOOL && (c->tile == 0 || !q.term_occur)) return fail(!q.term_occur ? TQ_ERR_INVALID_ARGUMENT : TQ_ERR_UNSUPPORTED, "TQ_OP_BOOL needs term_occur and the tile engine (TQ_TILE=1)");
  if (!q.weight || (!q.avg_fieldnorm && !q.tf_cache) || (!q.term_segs && q.n_term_segs)) return fail(TQ_ERR_INVALID_ARGUMENT, "query arrays");
  if (q.op == TQ_OP_PHRASE) {
    if (q.n_terms < 2 || q.n_terms > TQ_MAX_PHRASE_TERMS) return fail(TQ_ERR_UNSUPPORTED, "a phrase takes 2..TQ_MAX_PHRASE_TERMS terms on the device path");
    // slop: two terms take intersection_count_with_slop on the device; three and more carry per-position slops through
    // growing buffers (intersection_count_with_carrying_slop, phrase_scorer.rs:236-345) and stay on the reference's CPU path
    if (q.slop != 0 && q.n_terms != 2) return fail(TQ_ERR_UNSUPPORTED, "phrase slop with more than two terms stays on the reference's CPU path");
    if ((!q.term_pos && q.n_term_segs) || !q.term_offset) return fail(TQ_ERR_INVALID_ARGUMENT, "a phrase needs term_pos and term_offset");
  }
  return TQ_OK;
}

// The tf-norm table of every clause: its own rows of tf_cache, or the batch's table of its avg_fieldnorm.
void tf_tables(BatchPlan& pl, const tq_query& q, uint32_t* cache_idx) {
  for (uint32_t t = 0; t < q.n_terms; ++t) {
    if (q.tf_cache) {
      cache_idx[t] = (uint32_t)(pl.caches.size() / 256);
      pl.caches.insert(pl.caches.end(), q.tf_cache + 256 * (size_t)t, q.tf_cache + 256 * (size_t)(t + 1));
      continue;
    }
    uint32_t bits;
    memcpy(&bits, &q.avg_fieldnorm[t], 4);
    if (bits == pl.last_avg_bits && pl.last_avg_idx != 0xFFFFFFFFu) { cache_idx[t] = pl.last_avg_idx; continue; }  // (nearly always the same field)
    auto it = pl.cache_by_avg.find(bits);
    if (it == pl.cache_by_avg.end()) {
      float tab[256];
      bm25_tf_cache(q.avg_fieldnorm[t], tab);
      it = pl.cache_by_avg.emplace(bits, (uint32_t)(pl.caches.size() / 256)).first;
      pl.caches.insert(pl.caches.end(), tab, tab + 256);
    }
    cache_idx[t] = it->second;
    pl.last_avg_bits = bits;
    pl.last_avg_idx = it->second;
  }
}

// The query's SegPlans (pl.plans[0, n_plans)): one per segment that can match, clauses in evaluation order.  ctx->mu held.
int plan_segments(tq_ctx* c, BatchPlan& pl, const tq_query& q, int op, const uint32_t* cache_idx, uint64_t* q_postings) {
  const bool is_phrase = op == TQ_OP_PHRASE;
  pl.n_plans = 0;
  return for_each_segment(q, pl.order, [&](const tq_term_seg* const* ts, size_t n_here) -> int {
    if ((op == TQ_OP_AND || is_phrase) && n_here != q.n_terms) return TQ_OK;  // a clause is absent: empty intersection
    if (pl.n_plans == pl.plans.size()) pl.plans.emplace_back();
    SegPlan& sp = pl.plans[pl.n_plans++];
    sp.here.clear();
    sp.term_idx.clear();
    sp.uniform_fn = true;
    sp.no_freq = 0;
    sp.segment_ord = ts[0]->segment_ord;
    for (size_t a = 0; a < n_here; ++a) {
      const tq_term_seg& t = *ts[a];
      uint32_t id;
      const bool ignore_freq = q.term_flags && (q.term_flags[t.term_idx] & TQ_TERM_IGNORE_FREQ);
      const Segment* prev = sp.seg;
      int rc = get_list(c, t, ignore_freq, &id, &sp.seg);
      if (rc != TQ_OK) return rc;
      if (a > 0 && !same_docs(*prev, *sp.seg)) return fail_fields();
      if (ignore_freq || sp.seg->record_option == TQ_RECORD_BASIC) sp.no_freq |= 1u << a;
      if (a == 0) sp.fn0 = sp.seg->d_fieldnorm; else sp.uniform_fn &= (sp.seg->d_fieldnorm == sp.fn0);
      const uint32_t tw = is_phrase ? 0 : t.term_idx;
      QList ql{id, q.weight[tw], cache_idx[tw], 0};
      if (is_phrase) {  // the clause's position table; QList.pad carries its id to the aux array (append_qsegs)
        if (sp.seg->record_option != TQ_RECORD_FREQS_POSITIONS) return fail(TQ_ERR_INVALID_ARGUMENT, "phrase query on a field without positions");
        rc = get_pos(c, t, q.term_pos[ts[a] - q.term_segs], &ql.pad);
        if (rc != TQ_OK) return rc;
      }
      const uint64_t range = t.postings_end - t.postings_start;
      sp.here.push_back(SegPlan::Clause{t.doc_freq, ql, (uint32_t)range});
      sp.term_idx.push_back(t.term_idx);
      pl.alg_bytes += range + t.doc_freq;
      pl.op_bytes[bytes_class(op)] += range + t.doc_freq;
      pl.postings += t.doc_freq;
      *q_postings += t.doc_freq;
    }
    const int frc = query_alive(c, q, *sp.seg, &sp.alive, &sp.view);
    if (frc != TQ_OK) return frc;
    if (sp.view && sp.view->runs.empty()) { --pl.n_plans; return TQ_OK; }  // the filter keeps no doc of this segment's range
    auto by_doc_freq = [](const SegPlan::Clause& a, const SegPlan::Clause& b) { return a.first < b.first; };
    if (is_phrase) {
      // PhraseScorer keeps its terms by ascending size_hint (intersection.rs:40-52); every clause carries
      // (max_offset - its offset), the shift that lines the terms' positions up (phrase_scorer.rs:349-398).
      // PhraseQuery has put the terms in offset order first (phrase_query.rs:48-53), so equal doc_freqs keep that order:
      // it decides which term is `left` of a sloppy two-term count (phrase_count_slop2)
      uint32_t max_offset = 0;
      for (uint32_t t = 0; t < q.n_terms; ++t) max_offset = std::max(max_offset, q.term_offset[t]);
      for (size_t a = 0; a < sp.here.size(); ++a) sp.here[a].range_len = max_offset - q.term_offset[sp.term_idx[a]];  // (range_len is free here)
      std::stable_sort(sp.here.begin(), sp.here.end(), [](const SegPlan::Clause& a, const SegPlan::Clause& b) { return a.range_len > b.range_len; });
      std::stable_sort(sp.here.begin(), sp.here.end(), by_doc_freq);
    }
    if (op == TQ_OP_AND)  // leader = rarest, then ascending doc_freq; stable (block_wand_intersection.rs:27)
      std::stable_sort(sp.here.begin(), sp.here.end(), by_doc_freq);
    if (op == TQ_OP_OR)
      // Canonical union order = descending Bm25Weight.weight, ties in clause order (the reference's own order is
      // data dependent, block_wand_union.rs:205-208): the f32 sum is taken in this order, and the clauses with the
      // smallest score bounds form a suffix, which is what the MaxScore splits of k_tile / k_or_strip need.
      std::stable_sort(sp.here.begin(), sp.here.end(), [](const SegPlan::Clause& a, const SegPlan::Clause& b) { return a.second.weight > b.second.weight; });
    sp.prunable = true;
    for (auto& h : sp.here) sp.prunable = sp.prunable && std::isfinite(h.second.weight) && h.second.weight >= 0.0f;
    // an AND reaches block_wand_intersection only when every term reads freqs (boolean_weight.rs:318-340); the two orders
    // differ from the fourth scorer on, so fewer keep the kernels' plain loop
    sp.intersection_order = op == TQ_OP_AND && sp.no_freq != 0 && sp.here.size() >= 4;
    if (op == TQ_OP_BOOL) {
      uint32_t dfs[TQ_MAX_TERMS];
      float ws[TQ_MAX_TERMS];
      for (size_t a = 0; a < sp.here.size(); ++a) { dfs[a] = sp.here[a].first; ws[a] = sp.here[a].second.weight; }
      const int st = bool_structure(q, sp.term_idx.data(), dfs, ws, sp.here.size(), sp.no_freq, sp.bool_words, &sp.intersection_order);
      if (st < 0) return fail(TQ_ERR_INVALID_ARGUMENT, "term_occur");
      if (st == 0) --pl.n_plans;
    }
    return TQ_OK;
  });
}

// Puts query qi into a tile group if the tile engine takes it and it fits; false: it runs on the per-query kernels.
bool route_to_tile(const tq_ctx* c, BatchPlan& pl, size_t qi, int op, uint64_t q_postings) {
  const tq_query& q = pl.queries[qi];
  const bool to_tile = pl.repeat ? op == TQ_OP_BOOL
                                 : c->tile != 0 && (((c->tile_ops >> op) & 1u) || op == TQ_OP_BOOL) && (op != TQ_OP_TERM || pl.terms_on_tile);
  if (!to_tile || !pl.n_plans) return false;
  std::vector<TileGroupBuild>& tg = pl.tgroups;
  // a group holds the queries of one filter (or of none): its segments' alive words are that filter's views
  const uint64_t fkey = (q.flags & TQ_QUERY_FILTER) ? (1ull << 32 | q.filter_id) : 0ull;
  auto open = pl.open_group.find(fkey);
  if (open == pl.open_group.end() || (pl.repeat == 2 && !tg[open->second].segs.empty())) {
    tg.emplace_back();
    open = pl.open_group.insert_or_assign(fkey, tg.size() - 1).first;
  }
  // wide unions: every query brings its clause words, work-list entries and (mostly distinct) lists into the CTA's shared
  // memory; smaller groups keep two CTAs per SM (configs[4]: 1.64 s -> 1.05 s per 512 20-term queries on 500M docs)
  const uint32_t max_q = q.n_terms > 8 ? std::min(c->tile_max_queries, c->tile_wide_queries) : c->tile_max_queries;
  const SegPlan* plans = pl.plans.data();
  bool fits = tile_fits(c, tg[open->second], plans, pl.n_plans, max_q, false) || tile_fits(c, tg[open->second], plans, pl.n_plans, max_q, true);
  if (!fits && !tg[open->second].segs.empty() && tile_fits(c, TileGroupBuild{}, plans, pl.n_plans, max_q, false)) {  // the current group is full: open the next one
    tg.emplace_back();
    open->second = tg.size() - 1;
    fits = true;
  }
  const uint64_t tile_pair_budget = (uint64_t)c->tile_scratch_mb * (1u << 20) / 8u;
  if (!fits || pl.tile_pairs_total + q_postings + 128ull * pl.n_plans * q.n_terms > tile_pair_budget) return false;
  pl.tile_pairs_total += tile_admit(tg[open->second], (uint32_t)qi, op, pl.count_hits && (q.flags & TQ_QUERY_COUNT_HITS), plans, pl.n_plans);
  // every doc at or above the running threshold is handed over: the sample launch and the k_theta passes keep that
  // near k; a query that still overflows has the run repeated (flags[1], finalize_run).  A query hands each doc over at
  // most once (every tile once per run, a doc once per (query, tile): by its first posting in the driving clauses), so
  // its postings bound its candidates: the region of a repeat cannot overflow.
  const uint32_t cand_floor = c->tile_cand_floor;  // (test hook: tiny regions overflow)
  pl.q_cands[qi] += pl.repeat ? (size_t)q_postings
                              : (size_t)std::min<uint64_t>(q_postings, std::max<uint64_t>((cand_floor >= 8192 ? 128ull : 1ull) * q.k, cand_floor));
  return true;
}

// The (query, segment) pairs of query qi on the per-query kernels: QSeg, clause lists, unit class.
void append_qsegs(const tq_ctx* c, BatchPlan& pl, size_t qi, int op) {
  const tq_query& q = pl.queries[qi];
  for (size_t pi = 0; pi < pl.n_plans; ++pi) {
    SegPlan& sp = pl.plans[pi];
    auto& here = sp.here;
    QSeg qs;
    memset(&qs, 0, sizeof(qs));
    qs.query = (uint32_t)qi;
    qs.lists_base = (uint32_t)pl.qlists.size();
    qs.segment_ord = sp.segment_ord;
    qs.max_doc = sp.seg->max_doc;
    qs.alive = sp.alive;
    qs.fieldnorm = sp.uniform_fn ? sp.fn0 : nullptr;
    const bool prunable = sp.prunable && op != TQ_OP_TERM;
    qs.flags = (sp.uniform_fn ? 1u : 0u) | (prunable ? 2u : 0u) | (sp.intersection_order ? 4u : 0u);
    UnitClass cls = op == TQ_OP_PHRASE ? UC_PHRASE : (UnitClass)op;
    if (op == TQ_OP_PHRASE) {
      if (pl.qaux.size() < pl.qlists.size()) pl.qaux.resize(pl.qlists.size(), PhraseAux{0, 0, 0});
      for (auto& h : here) { pl.qaux.push_back(PhraseAux{h.second.pad, h.range_len, q.slop}); h.second.pad = 0; }
      pl.phrase_ct = std::max<uint32_t>(pl.phrase_ct, (uint32_t)here.size());
    }
    if (op == TQ_OP_OR && q.k <= kStripMaxK && here.size() <= kStripMaxLists) {
      // strip kernel: clauses with less than one block per kWin-doc window keep their current block decoded in shared memory
      uint32_t n_thin = 0;
      auto is_thin = [&](uint32_t df) { return (uint64_t)df * (kWin / 128u) < (uint64_t)qs.max_doc; };
      for (auto& h : here) if (is_thin(h.first)) ++n_thin;
      if (n_thin <= kMaxCached) {
        uint32_t slot = 0;
        for (auto& h : here) h.second.pad = is_thin(h.first) ? (1u | (slot++ << 1)) : 0u;
        pl.strip_cached_max = std::max(pl.strip_cached_max, n_thin);
        cls = UC_STRIP;
      }
    }
    for (auto& h : here) pl.qlists.push_back(h.second);
    qs.n_lists = (uint32_t)here.size();
    const uint32_t lead_total = here[0].first / 128u + ((here[0].first % 128u) ? 1u : 0u);
    pl.qsegs.push_back(qs);
    bool any_thick = false;
    for (auto& h : here) any_thick = any_thick || (uint64_t)h.first * kStripNeDiv2 >= qs.max_doc;
    const uint32_t total = cls == UC_STRIP ? (qs.max_doc + kWin - 1) / kWin : (op == TQ_OP_OR ? (qs.max_doc + kTileDocs - 1) / kTileDocs : lead_total);
    pl.work.push_back(SegWork{cls, total, cls == UC_STRIP && prunable && any_thick});
    ++pl.n_qsegs_op[cls == UC_PHRASE ? UC_AND : cls];
  }
}

}  // namespace

// The Count work of query qi (Count collector, count_collector.rs; Weight::count, term_weight.rs:179-219): its (query, segment)
// pairs go to cp; a term on a segment without deletes is answered from its doc_freq, added to *host_add (term_weight.rs:179-190).
// ctx->mu held.
int plan_count(tq_ctx* c, const tq_query& q, uint32_t qi, std::vector<const tq_term_seg*>& order, CountPlan& cp, uint64_t* host_add,
               bool all_docs) {
  int rc = check_shape(q, false);
  if (rc != TQ_OK) return rc;
  if (!q.term_segs && q.n_term_segs) return fail(TQ_ERR_INVALID_ARGUMENT, "query arrays");
  if (q.op == TQ_OP_BOOL && (!q.term_occur || !q.weight)) return fail(TQ_ERR_INVALID_ARGUMENT, "TQ_OP_BOOL needs term_occur and weights");
  rc = check_filter(c, q);
  if (rc != TQ_OK) return rc;
  std::vector<uint16_t> words;
  return for_each_segment(q, order, [&](const tq_term_seg* const* ts, size_t n_here) -> int {
    if (q.op == TQ_OP_AND && n_here < q.n_terms) return TQ_OK;  // a clause without postings: empty intersection
    uint32_t ids[TQ_MAX_TERMS];
    const Segment* seg = nullptr;
    for (size_t a = 0; a < n_here; ++a) {
      const Segment* prev = seg;
      const int lrc = get_list(c, *ts[a], false, &ids[a], &seg);
      if (lrc != TQ_OK) return lrc;
      if (a > 0 && !same_docs(*prev, *seg)) return fail_fields();
    }
    // the structure words of this segment, clauses as indices into ts: a term or an OR is one MUST group of its clauses, an AND
    // one group per clause
    if (q.op == TQ_OP_BOOL) {
      uint32_t tix[TQ_MAX_TERMS], dfs[TQ_MAX_TERMS];
      float ws[TQ_MAX_TERMS];
      for (size_t a = 0; a < n_here; ++a) { tix[a] = ts[a]->term_idx; dfs[a] = ts[a]->doc_freq; ws[a] = q.weight[ts[a]->term_idx]; }
      bool io_unused;  // (a count adds no scores)
      const int st = bool_structure(q, tix, dfs, ws, n_here, 0u, words, &io_unused);
      if (st < 0) return fail(TQ_ERR_INVALID_ARGUMENT, "term_occur");
      if (st == 0) return TQ_OK;
    } else if (q.op == TQ_OP_AND) {
      words.assign({(uint16_t)n_here, 0, 0, 0});
      for (size_t a = 0; a < n_here; ++a) words.insert(words.end(), {1, (uint16_t)a});
    } else {
      words.assign({1, 0, 0, 0, (uint16_t)n_here});
      for (size_t a = 0; a < n_here; ++a) words.push_back((uint16_t)a);
    }
    CountSeg cs{};
    const FilterView* view = nullptr;
    const int arc = query_alive(c, q, *seg, &cs.alive, &view);
    if (arc != TQ_OK) return arc;
    if (q.op != TQ_OP_BOOL && n_here == 1 && !cs.alive && !all_docs) {  // TermWeight::count without deletes (nor a filter): the term's doc_freq (term_weight.rs:179-190)
      *host_add += ts[0]->doc_freq;
      return TQ_OK;
    }
    cp.mixed = cp.mixed || words[1] != 0 || words[3] != 0;  // need, n_not
    cs.query = qi; cs.words_base = (uint32_t)cp.words.size(); cs.max_doc = seg->max_doc;
    cp.words.insert(cp.words.end(), words.begin(), words.end());
    map_bool_clauses(cp.words.data() + cs.words_base, words.size(), [&](uint32_t a) { return ids[a]; });
    // units of 8 tiles of 8192 docs over the segment; a filtered query's only over the tiles its filter view leaves non-empty
    const uint32_t seg_idx = (uint32_t)cp.segs.size(), tiles = (cs.max_doc + kTileDocs - 1) / kTileDocs, per = 8;
    if (!view) {
      for (uint32_t t0 = 0; t0 < tiles; t0 += per) cp.units.push_back(Unit{seg_idx, t0, std::min(tiles, t0 + per), 0});
    } else {
      for (const TileRun& r : view->count_runs)
        for (uint32_t t0 = r.t0; t0 < r.t1; t0 += per) cp.units.push_back(Unit{seg_idx, t0, std::min(r.t1, t0 + per), 0});
    }
    cp.segs.push_back(cs);
    cp.segment_ords.push_back(seg->segment_ord);
    return TQ_OK;
  });
}

// Validates query qi and plans it: into a tile group, or onto the per-query kernels.  ctx->mu held.
int plan_query(tq_ctx* c, BatchPlan& pl, size_t qi) {
  const tq_query& q = pl.queries[qi];
  int rc = validate_query(c, q);
  if (rc == TQ_OK) rc = check_filter(c, q);
  if (rc != TQ_OK) return rc;
  const bool count = pl.count_hits && (q.flags & TQ_QUERY_COUNT_HITS);
  if (count && q.op == TQ_OP_PHRASE) return fail(TQ_ERR_INVALID_ARGUMENT, "TQ_QUERY_COUNT_HITS: Count of a phrase query is not on the device path");
  // effective shape: an AND / OR of one clause is that clause (boolean_weight.rs:57-68, block_wand_union.rs:154-157)
  const int op = q.op == TQ_OP_PHRASE ? TQ_OP_PHRASE : (q.op == TQ_OP_BOOL ? TQ_OP_BOOL : (q.n_terms == 1 ? TQ_OP_TERM : q.op));
  pl.kmax = std::max(pl.kmax, q.k);
  pl.alg_bytes += 12ull * q.k;
  pl.op_bytes[bytes_class(op)] += 12ull * q.k;
  uint32_t cache_idx[TQ_MAX_TERMS];
  tf_tables(pl, q, cache_idx);
  pl.dq[qi].k = q.k;
  pl.dq[qi].op = (uint32_t)op;
  uint64_t q_postings = 0;
  rc = plan_segments(c, pl, q, op, cache_idx, &q_postings);
  if (rc != TQ_OK) return rc;
  if (route_to_tile(c, pl, qi, op, q_postings)) return TQ_OK;
  if (op == TQ_OP_BOOL && pl.n_plans) return fail(TQ_ERR_UNSUPPORTED, "TQ_OP_BOOL query does not fit the tile engine's buffers (split the batch / raise TQ_TILE_SCRATCH_MB)");
  append_qsegs(c, pl, qi, op);
  // its hits: k_count, in the same run (the per-query kernels leave no decoded lists behind)
  return count ? plan_count(c, q, (uint32_t)qi, pl.order, pl.count, &pl.hits_host[qi]) : TQ_OK;
}

// Work units. A unit is one CTA's share of a (query, segment). With few (query, segment) pairs in the
// batch every pair is cut into many units (latency); with many, units grow so that a CTA's local
// top-k threshold gets tight and few candidates reach k_final (throughput).  Then the candidate regions follow.
int cut_units(const tq_ctx* c, BatchPlan& pl) {
  const uint32_t target_units = c->target_units;
  for (size_t s = 0; s < pl.qsegs.size(); ++s) {
    const SegWork& w = pl.work[s];
    const uint32_t total = w.total;
    const uint32_t min_per = w.cls == UC_TERM ? c->term_blocks_per_unit
                             : ((w.cls == UC_AND || w.cls == UC_PHRASE) ? c->and_blocks_per_unit : (w.cls == UC_STRIP ? c->strip_windows_per_unit : c->or_tiles_per_unit));
    const uint32_t n_same = pl.n_qsegs_op[w.cls == UC_PHRASE ? UC_AND : w.cls];
    const uint32_t want_units = std::max<uint32_t>(1u, (target_units + n_same - 1) / n_same);
    const uint32_t per = std::max<uint32_t>(min_per, (total + want_units - 1) / want_units);
    const uint32_t query = pl.qsegs[s].query, k = pl.dq[query].k;
    // Threshold sample: the first 1/sample_div of a strip pair's windows run in a launch of their own; the exact k-th
    // best score over all sampled windows of the query (k_theta) then seeds the threshold of the main launch, whose
    // MaxScore split drops the dense clauses from the first window on.  Nothing is scored twice.
    uint32_t first = 0;
    if (w.cls == UC_STRIP && w.sample && total >= 8u * kStripSampleDiv) {
      const uint32_t cut1 = std::max<uint32_t>(kStripWarps, total / kStripSampleDiv);
      const uint32_t cut2 = std::max(cut1, total / kStripSampleDiv2);
      const uint32_t cut3 = std::max(cut2, total / kStripSampleDiv3);
      const uint32_t cuts[4] = {0, cut1, cut2, cut3};
      for (int r = 0; r < 3; ++r)  // round r covers [cuts[r], cuts[r+1]); a k_theta pass follows each round
        for (uint32_t b0 = cuts[r]; b0 < cuts[r + 1]; b0 += per) {
          pl.units[UC_STRIP_ROUND1 + r].push_back(Unit{(uint32_t)s, b0, std::min(cuts[r + 1], b0 + per), 0});
          pl.q_cands[query] += (size_t)kStripWarps * k;
        }
      first = cut3;
    }
    for (uint32_t b0 = first; b0 < total; b0 += per) {
      pl.units[w.cls].push_back(Unit{(uint32_t)s, b0, std::min(total, b0 + per), 0});
      pl.q_cands[query] += w.cls == UC_STRIP ? (size_t)kStripWarps * k : 2u * (size_t)k;  // what one unit may hand over
    }
  }
  for (size_t qi = 0; qi < pl.nq; ++qi) {
    pl.dq[qi].cand_base = (uint32_t)pl.n_cands;
    pl.dq[qi].cand_cap = (uint32_t)pl.q_cands[qi];
    pl.n_cands += pl.q_cands[qi];
    if (pl.n_cands > 0xFFFFFFF0ull) return fail(TQ_ERR_UNSUPPORTED, "batch too large: split it");
  }
  return TQ_OK;
}

namespace {

// The tiles a group's launches visit in one of its segments: its whole doc range, or the runs its filter view leaves non-empty.
std::vector<TileRun> seg_runs(const TileGroupBuild::SegB& sb) {
  if (sb.view) return sb.view->runs;
  if (sb.t_hi > sb.t_lo) return {TileRun{sb.t_lo, sb.t_hi}};
  return {};
}
uint64_t run_tiles(const std::vector<TileRun>& runs) {
  uint64_t n = 0;
  for (const TileRun& r : runs) n += r.t1 - r.t0;
  return n;
}
// Units of at most `per` tiles over the tiles [v0, v1) of `runs` taken one after another; no unit spans two runs.
void push_run_units(std::vector<TUnit>& out, uint32_t si, const std::vector<TileRun>& runs, uint64_t v0, uint64_t v1, uint32_t per) {
  uint64_t base = 0;
  for (const TileRun& r : runs) {
    const uint64_t len = r.t1 - r.t0, lo = std::max(v0, base), hi = std::min(v1, base + len);
    for (uint64_t a = lo; a < hi; a += per) out.push_back(TUnit{si, (uint32_t)(r.t0 + (a - base)), (uint32_t)(r.t0 + (std::min(hi, a + per) - base)), 0});
    base += len;
    if (base >= v1) break;
  }
}
// Tile v of `runs` taken one after another (v < run_tiles(runs)), with the end of its run.
TileRun run_tile(const std::vector<TileRun>& runs, uint64_t v) {
  for (const TileRun& r : runs) {
    if (v < r.t1 - r.t0) return TileRun{(uint32_t)(r.t0 + v), r.t1};
    v -= r.t1 - r.t0;
  }
  return TileRun{runs.back().t1 - 1, runs.back().t1};
}

}  // namespace

// Tile groups: slot order, pair bases, score chunks, tile ranges of the launches.
int stage_tile_groups(const tq_ctx* c, BatchPlan& pl) {
  pl.gstage.resize(pl.tgroups.size());
  const uint32_t big_min = c->tile_big_min;
  for (size_t gi = 0; gi < pl.tgroups.size(); ++gi) {
    TileGroupBuild& tg = pl.tgroups[gi];
    GroupStage& gs = pl.gstage[gi];
    double dens_max = 0;
    uint64_t tiles_total = 0;
    uint32_t kmax_g = 1;
    uint64_t group_tiles = 0;
    // the launches cover only these tiles; tiles_total and the sample spread count them alone, so a sparse filter still gets its samples
    std::vector<std::vector<TileRun>> runs(tg.segs.size());
    for (size_t si = 0; si < tg.segs.size(); ++si) {
      runs[si] = seg_runs(tg.segs[si]);
      group_tiles += run_tiles(runs[si]);
    }
    const uint32_t count_per = (uint32_t)std::max<uint64_t>(c->count_hits_tiles_per_unit, (group_tiles + 1023u) / 1024u);
    for (auto& sb : tg.segs) {
      // dense lists first (they get a tile index and whole warps), then the rest; clause ordinals follow the permutation
      std::vector<uint32_t> perm(sb.slots.size());
      for (uint32_t i = 0; i < perm.size(); ++i) perm[i] = i;
      auto is_big = [&](const TSlot& sl) { return (uint64_t)sl.doc_freq * kTile >= (uint64_t)big_min * std::max(1u, sb.max_doc); };
      // (by descending doc_freq throughout: the threads of a warp that stage sparse slots then see similar lists)
      std::stable_sort(perm.begin(), perm.end(), [&](uint32_t a, uint32_t b2) { return sb.slots[a].doc_freq > sb.slots[b2].doc_freq; });
      std::vector<uint32_t> new_of(perm.size());
      for (uint32_t i = 0; i < perm.size(); ++i) new_of[perm[i]] = i;
      TSeg G{};
      G.slot_base = (uint32_t)gs.slots.size();
      G.n_slots = (uint32_t)sb.slots.size();
      G.query_base = (uint32_t)gs.queries.size();
      G.n_queries = (uint32_t)sb.queries.size();
      G.max_doc = sb.max_doc;
      G.segment_ord = sb.segment_ord;
      G.n_tiles = (sb.max_doc + kTile - 1) / kTile;
      G.alive = sb.alive;
      uint32_t n_big = 0;
      for (uint32_t i = 0; i < perm.size(); ++i) {
        TSlot sl = sb.slots[perm[i]];
        sl.tseg = (uint32_t)gs.segs.size();
        sl.pair_base = (uint32_t)pl.pair_cursor;
        if (is_big(sl) && n_big < kTileMaxBig) sl.big = n_big++;  // (the densest ones: the order above is by descending doc_freq)
        const uint32_t n_total = sl.doc_freq / 128u + ((sl.doc_freq % 128u) ? 1u : 0u);
        for (uint32_t b0 = 0; b0 < n_total; b0 += 64u) gs.chunks.push_back(SChunk{(uint32_t)gs.slots.size(), b0, std::min(n_total, b0 + 64u)});
        pl.pair_cursor += ((uint64_t)sl.doc_freq + 127) / 128 * 128;
        pl.tile_postings += sl.doc_freq;
        gs.slots.push_back(sl);
      }
      G.n_big = n_big;
      G.tix = reinterpret_cast<uint32_t*>(pl.tix_total_words + gs.tix_words);  // offset for now, rebased in lay_out
      gs.tix_words += (size_t)(G.n_tiles + 1) * n_big;
      const uint32_t clause_shift = (uint32_t)gs.clauses.size();
      G.clause_base = clause_shift;
      G.n_clause_words = (uint32_t)sb.clauses.size();
      gs.max_clause_words = std::max(gs.max_clause_words, G.n_clause_words);
      gs.clauses.insert(gs.clauses.end(), sb.clauses.begin(), sb.clauses.end());
      for (auto& tq : sb.queries) {
        TQuery t2 = tq;
        t2.clause_base += clause_shift;
        gs.queries.push_back(t2);
        kmax_g = std::max(kmax_g, pl.dq[tq.query].k);
        gs.max_clauses = std::max<uint32_t>(gs.max_clauses, tq.n_clauses);
        if (tq.op == kTileOpAnd || tq.op == kTileOpBool) gs.union_only = false;
        // clause slots follow the permutation (the structure words of TQ_OP_BOOL queries do not)
        uint16_t* w = gs.clauses.data() + t2.clause_base;
        if (tq.op == kTileOpBool) map_bool_clauses(w, tq.n_clauses, [&](uint16_t s) { return new_of[s]; });
        else for (uint32_t e = 0; e < tq.n_clauses; ++e) w[e] = (uint16_t)new_of[w[e]];
      }
      bool count_seg = false;
      for (auto& tq : sb.queries) {
        if (!(tq.flags & kTileQueryCount)) continue;
        count_seg = true;
        gs.count_queries.push_back(tq.query);
      }
      const std::vector<TileRun>& sruns = runs[gs.segs.size()];  // (G is this group's segment gs.segs.size(), i.e. sb)
      if (count_seg)  // k_count_tiles: every tile the launches visit, about 1024 CTAs per group over all its segments
        push_run_units(gs.count_units, (uint32_t)gs.segs.size(), sruns, 0, run_tiles(sruns), count_per);
      gs.max_slots = std::max(gs.max_slots, G.n_slots);
      gs.max_big = std::max(gs.max_big, G.n_big);
      gs.max_queries = std::max(gs.max_queries, G.n_queries);
      dens_max = std::max(dens_max, sb.dens);
      tiles_total += run_tiles(sruns);
      gs.segs.push_back(G);
    }
    std::sort(gs.count_queries.begin(), gs.count_queries.end());
    gs.count_queries.erase(std::unique(gs.count_queries.begin(), gs.count_queries.end()), gs.count_queries.end());
    pl.tix_total_words += gs.tix_words;
    gs.p_cap =(uint32_t)std::min<double>(kTileMaxPairs, std::max(1024.0, dens_max * kTile * 1.25 + 192.0));
    gs.p_cap = (gs.p_cap + 63u) & ~63u;
    if (c->tile_pcap_hook) gs.p_cap = c->tile_pcap_hook;  // (test hook: overflowing tiles)
    if (pl.repeat) gs.p_cap = kTileMaxPairs;  // the repeat of an overflowed run: the largest tile buffer there is
    // Launches: [0] samples scores on a spread of short tile runs, [1..3] are exact and cover every tile once.
    const uint32_t target = std::max(1u, c->tile_units);
    const uint32_t sample_div = std::max<uint32_t>(2u, c->tile_sample_div);
    // enough sampled tiles for k_max samples to exist: each (query, tile) contributes at most kSamplePerTile
    const uint64_t want_sample_tiles = std::min<uint64_t>(tiles_total / 2, std::max<uint64_t>(tiles_total / sample_div, (uint64_t)kmax_g / 2u + 8u));
    for (uint32_t si = 0; si < gs.segs.size(); ++si) {
      // the segment's tiles taken one after another: its doc range (the whole segment unless one was set), or a filter's runs
      const std::vector<TileRun>& sruns = runs[si];
      const uint32_t nt = (uint32_t)run_tiles(sruns);
      if (nt == 0) continue;
      if (c->tile_sample_div > 1 && nt >= 8 && tiles_total) {
        // short runs of tiles spread over the segment, one CTA each (a sample launch has few tiles: it needs them all in flight)
        const uint32_t seg_sample = (uint32_t)std::max<uint64_t>(1, want_sample_tiles * nt / tiles_total);
        const uint32_t len = std::max<uint32_t>(1u, std::min<uint32_t>(4u, seg_sample / 64u + 1u));
        const uint32_t runs = std::max<uint32_t>(1u, seg_sample / len);
        for (uint32_t r = 0; r < runs; ++r) {
          const uint32_t start = (uint32_t)(((uint64_t)(2 * r + 1) * nt) / (2 * runs));
          const uint32_t t0 = std::min(start, nt - 1), t1 = std::min(nt, t0 + len);
          const TileRun at = run_tile(sruns, t0);  // (a sample run ends with its tile run)
          gs.units[0].push_back(TUnit{si, at.t0, std::min(at.t1, at.t0 + (t1 - t0)), 0});
        }
      }
      const uint32_t cut1 = nt >= 16 ? nt / std::max(2u, c->tile_round_div1) : 0, cut2 = nt >= 16 ? std::max(cut1, nt / std::max(2u, c->tile_round_div2)) : 0;
      const uint32_t cuts[4] = {0, cut1, cut2, nt};
      for (int r = 0; r < 3; ++r) {
        const uint32_t span = cuts[r + 1] - cuts[r];
        if (!span) continue;
        // this launch's share of the target, by its share of all tiles; at least 8 tiles per unit (cursor start-up)
        const uint64_t round_tiles_all = std::max<uint64_t>(1, (uint64_t)tiles_total * span / nt);
        const uint32_t per = (uint32_t)std::max<uint64_t>(tiles_total >= 16ull * target ? 8 : 2, (round_tiles_all + target - 1) / target);
        push_run_units(gs.units[1 + r], si, sruns, cuts[r], cuts[r + 1], per);
      }
    }
    for (int r = 0; r < kTileRounds; ++r) pl.tile_units += gs.units[r].size();
  }
  if (pl.pair_cursor > 0xFFFFFF00ull) return fail(TQ_ERR_UNSUPPORTED, "batch decodes more than 4G postings: split it");
  return TQ_OK;
}

}  // namespace tq::host
