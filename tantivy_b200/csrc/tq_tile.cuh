// The shared-decode query engine: every posting list a batch touches is decoded and scored ONCE per batch, and all
// queries of the batch are evaluated against doc-id tiles of those scored postings held in shared memory.
//
// Why: a (term, doc) BM25 score = Bm25Weight.weight * tf/(tf + norm[fieldnorm_id]) (src/query/bm25.rs:158-175) does not
// depend on the query that asks for it -- the weight belongs to the term.  A 512-query batch of 5-term unions over a
// 100M-doc index asks for 14 G scored postings, but the index only holds 0.3 G: the per-query kernels (k_or_strip ...)
// decode every list ~47 times per step.  Here:
//
//   k_score_lists   K1 + K2 of SURVEY.md §2, once per distinct (list, weight, tf-norm table) of the batch: one warp per
//                   128-doc block, BitPacker4x unpack + strict-delta prefix sum (BlockDecoder::uncompress_block_sorted /
//                   _unsorted, src/postings/compression/mod.rs:105-150), fieldnorm gather (src/fieldnorm/reader.rs:128),
//                   BM25 -> (doc, score) pairs streamed to HBM scratch with 16-byte stores.
//   k_tile          K3/K4/K5/K6 for all queries of the batch at once: a CTA walks a range of 1024-doc tiles; per tile it
//                   stages the pairs of every list into shared memory (sorted by doc inside a list), then evaluates the
//                   queries against them:
//                     * MaxScore with per-tile maxima (the block-max idea of block_wand_union.rs:16-43,171-177 at tile
//                       granularity, with maxima computed from the scores themselves, so they are exact under the
//                       searcher's global statistics -- the stored block-max pair is only exact under the segment's own
//                       average fieldnorm, term_scorer.rs:58-70): clauses are kept in the canonical summation order
//                       (descending weight); the longest suffix whose tile maxima add up to less than the query's
//                       threshold is non-essential and is only LOOKED UP for docs that the essential clauses make
//                       promising;
//                     * the essential postings of all (query, tile) pairs become one work list that the CTA's threads share
//                       evenly: one thread = one posting = one doc, completed by lookups in the query's other clauses (a bit
//                       test + popcount for dense lists, a short binary search for sparse ones), the non-essential suffix
//                       with an early exit as soon as the rest of the bound cannot reach the threshold; pairs with very
//                       many essential postings (and the sample launch) take a warp-private window of f32 score slots
//                       instead (BufferedUnionScorer's shape, union/buffered_union.rs:63-86);
//                     * f32 sums are taken clause by clause in the canonical order, so pruned and exhaustive evaluation
//                       give bit-identical scores;
//                     * survivors (score key >= the query's threshold) go to the query's candidate region, k_final
//                       (TopNHeap / merge_fruits) selects exactly.
//   thresholds      a first launch over 1/32 of the tiles only SAMPLES scores (the complete scores of the docs that hold one of
//                   a union's two heaviest clauses / a conjunction's matches); the k-th best sample is a valid lower bound of
//                   the final k-th score (k_theta_samples).  The exact launches follow,
//                   each ending in k_theta (exact k-th best candidate so far), so most tiles are visited under a
//                   near-final threshold.  Sampled tiles are visited again by the exact launches: nothing is pushed twice.
//
// Everything is bit-exact w.r.t. the oracle's exhaustive mode: same per-posting IEEE operations, same summation order.
#pragma once
#include "tq_kernels.cuh"

namespace tq {

// The tile engine's limits, descriptors (TSlot, TSeg, TQuery, TUnit, SChunk) and TileParams are in tq_layout.h.
constexpr uint32_t kSampleSeg = 6;          // sample launch: postings scored per driving clause and (query, tile)
constexpr uint32_t kSamplePerTile = 4;      // sample launch: the best few partial maxima of a (query, tile)


// ---- K1 + K2, once per batch -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 4) k_score_lists(const BatchParams P, const TileParams TP, uint32_t chunk_base) {
  const SChunk C = TP.chunks[chunk_base + blockIdx.x];
  const TSlot sl = TP.slots[C.slot];
  const ListDesc L = P.lists[sl.list_id];
  const Scorer sc{sl.weight, P.caches + 256u * sl.cache_idx, P.tf_tables + (size_t)(kTfRows * 256u) * sl.cache_idx};
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t* out_docs = TP.p_docs + sl.pair_base;
  float* out_scores = TP.p_scores + sl.pair_base;
  uint32_t* tix = nullptr;
  uint32_t n_big = 0, n_tiles = 0;
  if (sl.big != kNoSlot) {
    const TSeg G = TP.segs[sl.tseg];
    tix = G.tix + sl.big;
    n_big = G.n_big;
    n_tiles = G.n_tiles;
  }
  BlockFetch f;
  uint32_t b = C.b0 + warp;
  if (b < C.b1) fetch_issue(L, b, lane, f);
  for (; b < C.b1; b += kWarps) {
    uint32_t doc[4], tf[4];
    fetch_decode(L, b, f, lane, doc, tf);
    const uint32_t prev_last = b ? __ldg(L.last_doc + b - 1) : 0xFFFFFFFFu;
    if (b + kWarps < C.b1) fetch_issue(L, b + kWarps, lane, f);  // the next block travels while this one is scored
    const uint32_t g0 = b * 128u + lane * 4u;
    uint32_t id[4];
    float s[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const bool valid = g0 + i < L.doc_freq;  // the VInt tail pads with TERMINATED
      id[i] = L.fieldnorm ? (uint32_t)__ldg(L.fieldnorm + (valid ? doc[i] : 0u)) : 1u;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const bool valid = g0 + i < L.doc_freq;
      s[i] = valid ? bm25_score_id(sc, id[i], tf[i]) : 0.0f;
      if (!valid) doc[i] = 0xFFFFFFFFu;
    }
    // the pairs are read back once, by another kernel, after the whole pass: stream them past the L2 lines the gathers re-use
    // (fieldnorm bytes, block tables)
    __stcs(reinterpret_cast<uint4*>(out_docs + g0), make_uint4(doc[0], doc[1], doc[2], doc[3]));
    __stcs(reinterpret_cast<float4*>(out_scores + g0), make_float4(s[0], s[1], s[2], s[3]));
    if (tix) {  // tile index of a dense list: tix[t] = first pair with doc >= t * kTile
      uint32_t pd = __shfl_up_sync(kFull, doc[3], 1);
      if (lane == 0) pd = prev_last;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t g = g0 + i;
        if (g < L.doc_freq) {
          const uint32_t p = i == 0 ? pd : doc[i - 1];
          const uint32_t t_cur = doc[i] / kTile;
          for (uint32_t t = p == 0xFFFFFFFFu ? 0u : p / kTile + 1u; t <= t_cur; ++t) tix[(size_t)t * n_big] = g;
          if (g + 1u == L.doc_freq)
            for (uint32_t t = t_cur + 1u; t <= n_tiles; ++t) tix[(size_t)t * n_big] = L.doc_freq;
        }
      }
    }
  }
}

// ---- tile evaluation -----------------------------------------------------------------------------------------------------
// What a tile keeps in shared memory per slot: info = start | len << 16 (pairs [start, start + len) of off / score, ascending
// docs), the largest score (max), and for DENSE slots (the first n_big of a segment) a 1024-bit presence map (bits) with per-word
// ranks (rank: pairs of the slot before word w), so that "does this list hold doc x, and where" is one bit test + one popcount
// instead of a binary search over hundreds of pairs; for every slot a stripe mask (bit j set = the slot lists a doc of the tile's
// j-th 32-doc stripe; a dense slot's is the ballot of its non-zero presence words).  TileView holds every region of a CTA's dynamic
// shared memory (tile_smem_layout lists them).
struct TileQ; struct TileSeg; struct TileStageA; struct TileTQ;
struct TileView {
  float* score; TileQ* q; TileSeg* seg; TileStageA* a; float* acc;  // (a: in the bytes of seg; acc: in those of q and seg)
  uint32_t *info, *mask, *bits; float* max; TileTQ* tq; uint16_t *rank, *off, *heavy, *cl;
  uint32_t n_big;
};
__device__ __forceinline__ float tile_find(const TileView& V, uint32_t slot, uint32_t off, bool& found) {
  const uint32_t info = V.info[slot];
  if (slot < V.n_big) {
    const uint32_t w = V.bits[slot * 32u + (off >> 5)];
    const uint32_t bit = 1u << (off & 31u);
    found = (w & bit) != 0u;
    if (!found) return 0.0f;
    return V.score[(info & 0xFFFFu) + V.rank[slot * 32u + (off >> 5)] + __popc(w & (bit - 1u))];
  }
  // sparse slot: most lookups miss -- one stripe bit answers them; the rest scans the few pairs of the slot
  found = false;
  if (!((V.mask[slot] >> (off >> 5)) & 1u)) return 0.0f;
  uint32_t lo = info & 0xFFFFu;
  const uint32_t end = lo + (info >> 16);
  if (end - lo > 8u) {
    uint32_t hi = end;
    while (hi - lo > 4u) {
      const uint32_t m = (lo + hi) >> 1;
      if (V.off[m] < off) lo = m + 1u; else hi = m;
    }
  }
  for (; lo < end; ++lo) {
    const uint32_t o = V.off[lo];
    if (o >= off) { found = o == off; break; }
  }
  return found ? V.score[lo] : 0.0f;
}

// A CTA's counters of the current tile: pairs staged (A); heavy pairs (B1) and those a window took (B3); flat pairs (B1); work-list
// segments claimed (B1), taken by a warp (B2) and written (the list filled up from `segvalid` on); whether queries were deferred
// to another round of B1 + B2, and which; the queries whose running threshold is refreshed after the tile (tile_push).
constexpr uint32_t kTileRefreshCap = 16;
struct TileCtl {
  uint32_t total, nheavy, hpos, nflat, nseg, segpos, segvalid, ndefer, defer[kTileMaxQueries / 32u];
  uint32_t nref, ref[kTileRefreshCap];
};

// A candidate of an exact launch: appended to the query's region when its key reaches th_key and the doc is alive, and counted in
// the query's key histogram (TileParams::th_hist).  The k-th push and every max(k / 4, 16)-th after it put the query on the CTA's
// refresh list (a full list drops the entry: the next trigger comes soon enough).
__device__ __forceinline__ void tile_push(const BatchParams& P, const TileParams& TP, TileCtl& C, uint32_t query, float score, uint32_t doc,
                                          uint32_t segment_ord, uint32_t th_key, const uint8_t* __restrict__ alive) {
  const uint32_t key = score_to_key(score);
  if (key < th_key) return;
  if (alive && !is_alive(alive, doc)) return;
  const DQuery Q = P.queries[query];
  const uint32_t idx = atomicAdd(&P.qstate[query].cand_count, 1u);
  if (idx < Q.cand_cap) P.cands[Q.cand_base + idx] = Cand{key, segment_ord, doc, 0u};
  uint32_t* H = TP.th_hist + (size_t)query * kThHistWords;
  const uint32_t b = th_hist_bucket(key, th_hist_base(__ldg(H + kThHistBaseWord)));
  atomicAdd(H + b, 1u);
  atomicAdd(H + kThHistFine + (b >> 5), 1u);
  const uint32_t n = idx + 1u;
  if (n >= Q.k && (n - Q.k) % max(Q.k >> 2, 16u) == 0u) {
    const uint32_t r = atomicAdd(&C.nref, 1u);
    if (r < kTileRefreshCap) C.ref[r] = query;
  }
}

// The running threshold of query `query`, one warp: the highest bucket b whose suffix count (candidates in buckets >= b) reaches
// k, from the coarse counts (two per lane) and then that coarse bucket's 32 fine counts; the threshold rises to edge(b).
// Why this is exact: every candidate counted is a real, alive doc that passes the query's filter, with its complete score; a doc is
// pushed at most once per query and run (the exact launches cover disjoint tile ranges, a (query, tile) pair has one owner per
// doc in B2 and one window in B3, and the sample launch pushes nothing); every count is a lower bound of what its bucket holds,
// however the reads interleave with other CTAs' atomics.  So k docs have keys >= edge(b), and the final k-th key is >= edge(b):
// docs tied at the k-th key still pass `key >= th_key`.  The same holds per rank under the sharded key exchange.  Returns whether
// the threshold rose.
__device__ __forceinline__ bool tile_theta_refresh(const BatchParams& P, const TileParams& TP, uint32_t query, uint32_t lane) {
  const uint32_t* H = TP.th_hist + (size_t)query * kThHistWords;
  const uint32_t k = P.queries[query].k;
  const uint32_t c0 = __ldcg(H + kThHistFine + 2u * lane), c1 = __ldcg(H + kThHistFine + 2u * lane + 1u);
  uint32_t suf = c0 + c1;  // -> the count of coarse buckets >= 2 * lane
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_down_sync(kFull, suf, o);
    if (lane + o < 32u) suf += v;
  }
  const uint32_t hit = __ballot_sync(kFull, suf >= k);
  if (!hit) return false;
  const uint32_t L = 31u - __clz(hit);
  const uint32_t sL = __shfl_sync(kFull, suf, L), c0L = __shfl_sync(kFull, c0, L), c1L = __shfl_sync(kFull, c1, L);
  const bool odd = sL - c0L >= k;
  const uint32_t cb = 2u * L + (odd ? 1u : 0u);
  const uint32_t need = k - (odd ? sL - c0L - c1L : sL - c0L);  // (> 0: the coarse buckets above cb hold fewer than k)
  uint32_t fsuf = __ldcg(H + cb * 32u + lane);
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_down_sync(kFull, fsuf, o);
    if (lane + o < 32u) fsuf += v;
  }
  const uint32_t fhit = __ballot_sync(kFull, fsuf >= need);  // (0 when the fine counts trail the coarse ones: take cb's first)
  const uint32_t b = cb * 32u + (fhit ? 31u - __clz(fhit) : 0u);
  const uint32_t edge = th_hist_edge(b, th_hist_base(__ldg(H + kThHistBaseWord)));
  uint32_t old = 0xFFFFFFFFu;
  if (lane == 0 && edge) old = atomicMax(&P.qstate[query].theta, edge);
  return __shfl_sync(kFull, old, 0) < edge;
}

// One (query, tile) pair that is evaluated posting by posting: what every posting's thread needs to know (16 bytes).
struct TileQ {
  uint16_t qi;           // the query: index into the CTA's copy of the segment's queries (batch ordinal, clause slots)
  uint8_t n_op;          // clauses [0:6) | op << 6
  uint8_t ne_prune;      // essential prefix (unions) / driving clause (conjunctions) [0:6) | prune << 7
  uint32_t th_key;       // the query's threshold when the tile was entered
  float ne;              // bound of the non-essential suffix in this tile (unions); 0 for conjunctions
  uint32_t shared_stripes;  // unions: 32-doc stripes of the tile in which more than one essential clause lists a doc (a posting
                            // outside them is the only essential posting of its doc: no lookup is needed to know its partial sum)
  __device__ __forceinline__ uint32_t n() const { return n_op & 63u; }
  __device__ __forceinline__ uint32_t op() const { return n_op >> 6; }
  __device__ __forceinline__ uint32_t n_e() const { return ne_prune & 63u; }
  __device__ __forceinline__ bool prune() const { return (ne_prune & 128u) != 0; }
};
// the segment's queries as the CTA keeps them on chip (8 bytes)
struct TileTQ {
  uint32_t query;
  uint16_t clause_base;  // local to the segment
  uint8_t n_clauses;
  uint8_t op_flags;      // op [0:2) | Intersection order << 5 | prunable << 7
};
// one essential clause of flat pair q: its postings in the tile are the slot's staged range (info of cl[clause]; the sample
// launch takes at most kSampleSeg of them)
struct TileSeg { uint16_t q, clause; };

// Union: what every clause after essential clause c can add to a doc of this tile -- the tile maxima of the essential clauses
// (c, n_e) plus ne, the bound of the non-essential suffix.
__device__ __forceinline__ float tile_or_tail(const TileView& V, const uint16_t* __restrict__ cl, uint32_t c, uint32_t n_e, float ne) {
  float tail = ne;
  for (uint32_t c2 = c + 1u; c2 < n_e; ++c2) tail += V.max[cl[c2]];
  return tail;
}

// How tile_eval_or leaves a posting (k_tile<*, true, *> counts each: TileParams::counters[16 + exit], tq_stats.tile_b2_exits):
// dropped by the bound taken before the look-ups, complete score but the doc belongs to an earlier essential clause (asked after
// the walk), dropped in the non-essential walk, complete score.  Only the counters instances record it (tile_eval_or<true, *>):
// the other instances keep the two-way exit, whose branch structure the exit codes change (as the function's value they cost
// k_tile 5 % on or5_top100_100M_8seg, H100 80GB HBM3 at 700 W).
enum TileOrExit : uint32_t { kOrBound, kOrOwner, kOrWalk, kOrDone, kOrExits };

// Union: the doc at tile offset `off`, met as posting p of essential clause c (of n_e; n clauses, ne and shared_stripes as in TileQ).
// Exact score in the canonical order, or nothing when the bounds show it cannot reach the threshold.  Returns true when `sum` is a
// complete score; kExit: `ex` says how the posting left.  kTail: `tail` = tile_or_tail(c) is given (else it is summed here, when
// needed).
template <bool kExit, bool kTail>
__device__ __forceinline__ bool tile_eval_or(const TileView& V, const uint16_t* __restrict__ cl, uint32_t n_e, uint32_t n, bool prune,
                                             float ne, float tail, uint32_t shared_stripes, uint32_t c, uint32_t p, uint32_t off,
                                             float theta_f, float& sum, uint32_t& ex) {
  bool f;
  sum = V.score[p];  // (-0.0 + s == s: SumCombiner starts from 0, score_combiner.rs:39-57)
  const bool shared = (shared_stripes >> (off >> 5)) & 1u;
  if (shared) {  // another essential clause lists a doc near this one: look the doc up
    // ... unless the bound says no: if an earlier clause lists the doc, it is dropped anyway; if none does, its score is at
    // most sum + tail (the f32 orders of the two sums differ by less than the margin, as in tile_essential)
    if (prune && (sum + (kTail ? tail : tile_or_tail(V, cl, c, n_e, ne))) * 1.00001f < theta_f) {
      if (kExit) ex = kOrBound;
      return false;
    }
    for (uint32_t c2 = c + 1u; c2 < n_e; ++c2) {
      const float v = tile_find(V, cl[c2], off, f);
      if (f) sum = __fadd_rn(sum, v);
    }
  }
  // the non-essential suffix, densest last; stop as soon as what is left cannot lift the doc over the threshold
  float rem = ne;
  for (uint32_t c2 = n_e; c2 < n; ++c2) {
    if (prune && (sum + rem) * 1.00001f < theta_f) {
      if (kExit) ex = kOrWalk;
      return false;
    }
    const uint32_t slot = cl[c2];
    rem -= V.max[slot];
    const float v = tile_find(V, slot, off, f);
    if (f) sum = __fadd_rn(sum, v);
  }
  // the doc is evaluated by the first essential clause that lists it.  Asked last: whether an earlier clause lists the doc does
  // not change the sum above, and most postings of a shared stripe leave in the walk, so only the few that get here look up the
  // earlier clauses (outside a shared stripe no other essential clause lists the doc)
  if (shared)
    for (uint32_t c1 = 0; c1 < c; ++c1) {
      tile_find(V, cl[c1], off, f);
      if (f) {
        if (kExit) ex = kOrOwner;
        return false;
      }
    }
  if (kExit) ex = kOrDone;
  return true;
}

// Conjunction: the doc (posting p of the driving clause) must be listed by every clause; the score is summed in clause order
// (leader = rarest list first, block_wand_intersection.rs:27,146-158) whichever clause drives the iteration -- one after another,
// or with IO (set for >= 4 clauses only) as Intersection::score adds up (intersection.rs:325-329): (s0 + s1) + (s2 + s3 + ...),
// i.e. the running sum restarts at clause 2 and s0 + s1 is added at the end.  (A template: the plain conjunctions that fill a
// typical batch keep a loop without the restart test.)
template <bool IO>
__device__ __forceinline__ bool tile_eval_and_t(const TileView& V, const uint16_t* __restrict__ cl, uint32_t n, uint32_t drv, uint32_t p,
                                                uint32_t off, float& sum) {
  sum = 0.0f;
  float head = 0.0f;
  for (uint32_t c = 0; c < n; ++c) {
    float v;
    if (c == drv) v = V.score[p];
    else {
      bool f;
      v = tile_find(V, cl[c], off, f);
      if (!f) return false;
    }
    const bool restart = IO && c == 2u;
    if (restart) head = sum;
    sum = (c == 0 || restart) ? v : __fadd_rn(sum, v);
  }
  if (IO) sum = __fadd_rn(head, sum);
  return true;
}
__device__ __forceinline__ bool tile_eval_and(const TileView& V, const uint16_t* __restrict__ cl, uint32_t n, uint32_t drv, uint32_t p, uint32_t off,
                                              bool io, float& sum) {
  return io ? tile_eval_and_t<true>(V, cl, n, drv, p, off, sum) : tile_eval_and_t<false>(V, cl, n, drv, p, off, sum);
}

// Mixed boolean query (BooleanWeight::complex_scorer for term leaves, boolean_weight.rs:236-431): the doc at `off` is met as posting p
// of the clause at word `wi`, one of the driving words [d0, d0 + dn).  It is evaluated once (by the first driving clause that lists
// it): every MUST group needs a clause that lists it (group score = sum of its matching clauses), MUST_NOT clauses must not, at least
// `need` SHOULD clauses must; score = (sum of the group scores, ascending cost) + (sum of the matching SHOULD clauses)
// (Intersection::score, RequiredOptionalScorer::score).  The groups add up like tile_eval_and's clauses: with `io`,
// (g0 + g1) + (g2 + g3 + ...), else one after another.
__device__ __forceinline__ bool tile_eval_bool(const TileView& V, const uint16_t* __restrict__ cl, uint32_t d0, uint32_t wi, uint32_t p, uint32_t off,
                                               bool io, float& sum) {
  bool f;
  for (uint32_t i = d0; i < wi; ++i) {
    tile_find(V, cl[i], off, f);
    if (f) return false;
  }
  const uint32_t ng = cl[0], need = cl[1], ns = cl[2], nn = cl[3];
  uint32_t w = 4;
  float total = 0.0f, head = 0.0f;
  for (uint32_t g = 0; g < ng; ++g) {
    const uint32_t glen = cl[w++];
    float gs = 0.0f;
    bool any = false;
    for (uint32_t e = 0; e < glen; ++e, ++w) {
      float v;
      if (w == wi) { v = V.score[p]; f = true; } else v = tile_find(V, cl[w], off, f);
      if (f) { gs = any ? __fadd_rn(gs, v) : v; any = true; }
    }
    if (!any) return false;
    const bool restart = io && g == 2u;
    if (restart) head = total;
    total = (g == 0 || restart) ? gs : __fadd_rn(total, gs);
  }
  if (io) total = __fadd_rn(head, total);
  float ss = 0.0f;
  uint32_t cnt = 0;
  for (uint32_t e = 0; e < ns; ++e, ++w) {
    float v;
    if (w == wi) { v = V.score[p]; f = true; } else v = tile_find(V, cl[w], off, f);
    if (f) { ss = cnt ? __fadd_rn(ss, v) : v; ++cnt; }
  }
  for (uint32_t e = 0; e < nn; ++e, ++w) {
    tile_find(V, cl[w], off, f);
    if (f) return false;
  }
  if (cnt < need) return false;
  sum = ng ? (cnt ? __fadd_rn(total, ss) : total) : ss;
  return true;
}

// Stage A's scratch (in the then idle work-list segments): the dense slots' ranges of this tile and each warp's prefix over its slots
struct TileStageA {
  uint32_t ba[kTileMaxBig], bn[kTileMaxBig];  // first pair of the slot in this tile, and how many
  uint32_t wpre[kTileWarps][9];
  uint32_t wa[kTileWarps][8];
};

static_assert(sizeof(TileQ) == kTileQBytes && sizeof(TileSeg) == kTileSegBytes && sizeof(TileTQ) == kTileTQBytes &&
                  sizeof(TileStageA) == kTileStageABytes, "tile_smem_layout (tq_layout.h)");

__device__ __forceinline__ TileView tile_view(unsigned char* s_dyn, const TileParams& TP, uint32_t n_big) {
  const TileSmem L = tile_smem_layout(TP.p_cap, TP.max_slots, TP.max_big, TP.max_queries, TP.seg_cap, TP.cl_cap, TP.n_win);
  return TileView{reinterpret_cast<float*>(s_dyn),                reinterpret_cast<TileQ*>(s_dyn + L.list),
                  reinterpret_cast<TileSeg*>(s_dyn + L.seg),       reinterpret_cast<TileStageA*>(s_dyn + L.seg),
                  reinterpret_cast<float*>(s_dyn + L.list),        reinterpret_cast<uint32_t*>(s_dyn + L.info),
                  reinterpret_cast<uint32_t*>(s_dyn + L.mask),     reinterpret_cast<uint32_t*>(s_dyn + L.bits),
                  reinterpret_cast<float*>(s_dyn + L.max),         reinterpret_cast<TileTQ*>(s_dyn + L.tq),
                  reinterpret_cast<uint16_t*>(s_dyn + L.rank),     reinterpret_cast<uint16_t*>(s_dyn + L.off),
                  reinterpret_cast<uint16_t*>(s_dyn + L.heavy),    reinterpret_cast<uint16_t*>(s_dyn + L.cl),
                  n_big};
}

// Per-thread diagnostics of k_tile<*, true, *> (TileParams::counters[0, 7), refreshes and raises: [14, 16), or_exit: [16, 20)); the
// other instances compile them out.  or_exit: the exact launches' B2 union postings by how tile_eval_or left them (TileOrExit; 32
// bits: a thread's share of one launch).
struct TileStats { unsigned long long pairs, skipped, flat, heavy, ess, completed, pushed; uint32_t or_exit[kOrExits], refreshes, raises; };
// Stages of a tile as the cycle counters of k_tile<*, true, *> split a warp's time (TileParams::counters[8 + stage],
// tq_stats.tile_cycles): the cursor prologue, A, B1, B2, B3, and the waits at the barriers between them.
enum TileStage : int { kStPrologue, kStA, kStB1, kStB2, kStB3, kStBarrier, kTileStages };
constexpr int kTileStatWords = 16 + kOrExits;  // TileParams::counters words k_tile<*, true, *> adds to

// ---- the decisions B1 (routing) and B3 (windows) share -------------------------------------------------------------------
// TQ_OP_BOOL: the driving words [d0, d0 + dn) of cl -- the MUST group with the fewest postings in this tile (the first of equals),
// or the SHOULD clauses when there is no MUST group -- and their postings (0: some MUST group has none).  `bound`: the sum of the
// MUST and SHOULD clauses' tile maxima.
__device__ __forceinline__ uint32_t tile_bool_drive(const TileView& V, const uint16_t* __restrict__ cl, uint32_t& d0, uint32_t& dn, float& bound) {
  const uint32_t ng = cl[0], ns = cl[2];
  uint32_t w = 4, best = 0xFFFFFFFFu;
  bound = 0.0f;
  for (uint32_t g = 0; g < ng; ++g) {
    const uint32_t glen = cl[w];
    uint32_t tot = 0;
    for (uint32_t e = 0; e < glen; ++e) { const uint32_t slot = cl[w + 1u + e]; tot += V.info[slot] >> 16; bound += V.max[slot]; }
    if (tot < best) { best = tot; d0 = w + 1u; dn = glen; }
    w += 1u + glen;
  }
  uint32_t s_tot = 0;
  for (uint32_t e = 0; e < ns; ++e) { const uint32_t slot = cl[w + e]; s_tot += V.info[slot] >> 16; bound += V.max[slot]; }
  if (ng == 0u) { best = s_tot; d0 = w; dn = ns; }
  return best;
}

// Conjunction: the driving clause `drv` -- the one with the fewest postings in this tile (the first of equals) -- and its postings.
// `bound`: the sum of the clauses' tile maxima.
__device__ __forceinline__ uint32_t tile_and_drive(const TileView& V, const uint16_t* __restrict__ cl, uint32_t n, uint32_t& drv, float& bound) {
  uint32_t dmin = 0xFFFFFFFFu;
  bound = 0.0f; drv = 0;
  for (uint32_t c = 0; c < n; ++c) {
    const uint32_t len = V.info[cl[c]] >> 16;
    bound += V.max[cl[c]];
    if (len < dmin) { dmin = len; drv = c; }
  }
  return dmin;
}

// Union (MaxScore): the essential prefix of clauses [0, n_e) shrinks while the tile maxima of the suffix it leaves add up to less
// than the threshold; `ne` = the bound of that non-essential suffix.
__device__ __forceinline__ uint32_t tile_essential(const TileView& V, const uint16_t* __restrict__ cl, uint32_t n_e, bool prune, float theta_f, float& ne) {
  ne = 0.0f;
  if (prune) {
    while (n_e > 0) {
      const float b = ne + V.max[cl[n_e - 1u]];
      if (!(b * 1.00001f < theta_f)) break;  // (f32 sums of <= 32 terms differ by < 4e-6 relative between orders)
      ne = b;
      --n_e;
    }
  }
  return n_e;
}

// Sample launch: the warp's best few keys (one per lane in `best`) that reach th_key become samples of the query, largest first.
__device__ __forceinline__ void warp_push_samples(const TileParams& TP, uint32_t query, uint32_t best, uint32_t th_key, uint32_t lane) {
  for (uint32_t r = 0; r < kSamplePerTile; ++r) {
    const uint32_t mk = __reduce_max_sync(kFull, best);
    if (mk == 0u || mk < th_key) break;
    const unsigned who = __ballot_sync(kFull, best == mk);
    if (lane == (uint32_t)__ffs(who) - 1u) {
      const uint32_t idx = atomicAdd(&TP.sample_count[query], 1u);
      if (idx < TP.sample_cap) TP.samples[(size_t)query * TP.sample_cap + idx] = mk;
      best = 0;
    }
  }
}

// ---- the stages of a tile ------------------------------------------------------------------------------------------------
// Prologue: the segment's queries and their clause slots are read for every tile -- keep them on chip (clause_base becomes an index
// into the segment's clause words) -- and every sparse slot's cursor is positioned on its first pair at or after the unit's first
// doc.  Four slots per thread at a time: the binary searches advance in lockstep, so their (dependent) loads overlap -- with
// two-tile units this prologue is a tenth of the CTA's time.
__device__ __forceinline__ void tile_prologue(const TileParams& TP, const TSeg& G, const TSlot* __restrict__ slots, const TileView& V,
                                              bool cl_staged, uint2* cursor, uint32_t t0, uint32_t tid) {
  for (uint32_t i = tid; i < G.n_queries; i += kTileThreads) {
    const TQuery tq = TP.queries[G.query_base + i];
    V.tq[i] = TileTQ{tq.query, (uint16_t)(tq.clause_base - G.clause_base), (uint8_t)tq.n_clauses, (uint8_t)((tq.op & 3u) | ((tq.flags & 4u) << 3) | ((tq.flags & 1u) << 7))};
  }
  if (cl_staged)
    for (uint32_t i = tid; i < G.n_clause_words; i += kTileThreads) V.cl[i] = TP.clauses[G.clause_base + i];
  for (uint32_t s0 = G.n_big + tid; s0 < G.n_slots; s0 += 4u * kTileThreads) {
    const uint32_t lo0 = t0 * kTile;
    const uint32_t* d[4];
    uint32_t a[4], b[4], df[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t s = s0 + (uint32_t)j * kTileThreads;
      const bool in = s < G.n_slots;
      const TSlot sl = slots[in ? s : s0];
      d[j] = TP.p_docs + sl.pair_base;
      df[j] = sl.doc_freq;
      a[j] = 0; b[j] = in ? sl.doc_freq : 0u;
    }
    for (;;) {
      bool any = false;
      uint32_t v[4], m[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        m[j] = (a[j] + b[j]) >> 1;
        if (a[j] < b[j]) { v[j] = __ldg(d[j] + m[j]); any = true; }
      }
      if (!any) break;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (a[j] < b[j]) { if (v[j] < lo0) a[j] = m[j] + 1u; else b[j] = m[j]; }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t s = s0 + (uint32_t)j * kTileThreads;
      if (s < G.n_slots) cursor[s] = make_uint2(a[j], a[j] < df[j] ? __ldg(d[j] + a[j]) : 0xFFFFFFFFu);
    }
  }
}

// Stage A, dense lists: warp w owns slots w, w+8, ... (<= 8 of them).  Their [tix[t], tix[t+1]) ranges (V.a->ba / bn) are laid end
// to end and copied as ONE flat loop, so the loads of all the warp's slots are in flight together (one DRAM round trip per 128
// pairs instead of three dependent ones per slot).
__device__ __forceinline__ void tile_stage_dense(const TileParams& TP, const TSeg& G, const TileView& V, uint32_t& total, uint32_t lo,
                                                 uint32_t warp, uint32_t lane) {
  TileStageA& A = *V.a;
  const uint32_t ne = (G.n_big - warp + kTileWarps - 1u) / kTileWarps;
  uint32_t n_e = 0;
  if (lane < ne) {
    const uint32_t s = warp + lane * kTileWarps;
    n_e = A.bn[s];
    A.wa[warp][lane] = A.ba[s];
  }
  const uint32_t incl = warp_incl_scan(n_e, lane);
  if (lane < 8u) A.wpre[warp][lane + 1u] = incl;
  if (lane == 0) A.wpre[warp][0] = 0u;
  const uint32_t total_w = __shfl_sync(kFull, incl, 7);
  uint32_t base = 0;
  if (lane == 0 && total_w) base = atomicAdd(&total, total_w);
  base = __shfl_sync(kFull, base, 0);
  for (uint32_t e = 0; e < ne; ++e) V.bits[(warp + e * kTileWarps) * 32u + lane] = 0u;
  __syncwarp();
  const bool fits = base + total_w <= TP.p_cap;
  if (fits) {
    for (uint32_t i0 = 0; i0 < total_w; i0 += 128u) {
      uint32_t dd[4], ss[4];
      float vv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t i = i0 + (uint32_t)u * 32u + lane;
        dd[u] = 0xFFFFFFFFu;
        if (i < total_w) {
          uint32_t e = 0;
          while (i >= A.wpre[warp][e + 1u]) ++e;
          ss[u] = warp + e * kTileWarps;
          const size_t g = (size_t)A.wa[warp][e] + (i - A.wpre[warp][e]);
          dd[u] = __ldg(TP.p_docs + g);
          vv[u] = __ldg(TP.p_scores + g);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t i = i0 + (uint32_t)u * 32u + lane;
        if (dd[u] != 0xFFFFFFFFu) {
          const uint32_t off = dd[u] - lo;
          V.off[base + i] = (uint16_t)off;
          V.score[base + i] = vv[u];
          atomicOr(&V.bits[ss[u] * 32u + (off >> 5)], 1u << (off & 31u));
        }
      }
    }
  }
  __syncwarp();
  for (uint32_t e = 0; e < ne; ++e) {
    const uint32_t s = warp + e * kTileWarps;
    const uint32_t b = base + A.wpre[warp][e], n = A.wpre[warp][e + 1u] - A.wpre[warp][e];
    const uint32_t word = V.bits[s * 32u + lane];
    const uint32_t cnt = (uint32_t)__popc(word);
    V.rank[s * 32u + lane] = (uint16_t)(warp_incl_scan(cnt, lane) - cnt);
    const uint32_t mask = __ballot_sync(kFull, word != 0u);  // (presence word j = stripe j)
    float mx = 0.0f;
    if (fits)
      for (uint32_t i = lane; i < n; i += 32) mx = fmaxf(mx, V.score[b + i]);
    mx = __uint_as_float(__reduce_max_sync(kFull, __float_as_uint(mx)));  // mx >= 0
    if (lane == 0) { V.info[s] = (b & 0xFFFFu) | (n << 16); V.max[s] = mx; V.mask[s] = mask; }
  }
}

// Stage A, sparse lists: one thread walks a slot's cursor (and fetches its next slot's cursor while it stages this one).
__device__ __forceinline__ void tile_stage_sparse(const TileParams& TP, const TSeg& G, const TSlot* __restrict__ slots, const TileView& V,
                                                  uint2* cursor, uint32_t& total, uint32_t lo, uint32_t tid) {
  const uint32_t hi = lo + kTile;
  uint2 next_cur = G.n_big + tid < G.n_slots ? cursor[G.n_big + tid] : make_uint2(0u, 0u);
  for (uint32_t s = G.n_big + tid; s < G.n_slots; s += kTileThreads) {
    const uint2 cs = next_cur;
    if (s + kTileThreads < G.n_slots) next_cur = cursor[s + kTileThreads];  // (in flight while this slot is staged)
    uint32_t nd = cs.y;
    if (nd >= hi) {
      V.info[s] = 0u; V.max[s] = 0.0f; V.mask[s] = 0u;
      continue;
    }
    const TSlot sl = slots[s];
    const uint32_t* __restrict__ d = TP.p_docs + sl.pair_base;
    const float* __restrict__ sc = TP.p_scores + sl.pair_base;
    const uint32_t cur = cs.x;
    // the pair at the cursor belongs to this tile (nd < hi); fetch it and the next three, docs and scores, in ONE round trip
    uint32_t d4[4];
    float v4[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const bool in = cur + i < sl.doc_freq;
      d4[i] = in ? __ldg(d + cur + i) : 0xFFFFFFFFu;
      v4[i] = in ? __ldg(sc + cur + i) : 0.0f;
    }
    uint32_t n = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) n += d4[i] < hi ? 1u : 0u;  // ascending: the ones below hi are a prefix
    if (n == 4u) {  // (rare for a sparse list) keep walking
      for (;;) {
        const uint32_t c = cur + n;
        uint32_t e4[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) e4[i] = c + i < sl.doc_freq ? __ldg(d + c + i) : 0xFFFFFFFFu;
        uint32_t k = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) k += e4[i] < hi ? 1u : 0u;
        n += k;
        if (k < 4u) { nd = e4[k]; break; }
      }
    } else {
      nd = d4[n];
    }
    cursor[s] = make_uint2(cur + n, nd);
    if (nd < hi + kTile) {  // the next tile reads this list again: start its pairs on their way to L2 now
      asm volatile("prefetch.global.L2 [%0];" ::"l"(d + cur + n));
      asm volatile("prefetch.global.L2 [%0];" ::"l"(sc + cur + n));
    }
    const uint32_t base = atomicAdd(&total, n);
    float mx = 0.0f;
    uint32_t mask = 0;
    if (base + n <= TP.p_cap) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if ((uint32_t)i < n) {
          const uint32_t off = d4[i] - lo;
          V.off[base + i] = (uint16_t)off;
          V.score[base + i] = v4[i];
          mask |= 1u << (off >> 5);
          mx = fmaxf(mx, v4[i]);
        }
      }
      for (uint32_t i = 4; i < n; ++i) {
        const float v = __ldg(sc + cur + i);
        const uint32_t off = __ldg(d + cur + i) - lo;
        V.off[base + i] = (uint16_t)off;
        V.score[base + i] = v;
        mask |= 1u << (off >> 5);
        mx = fmaxf(mx, v);
      }
    }
    V.info[s] = (base & 0xFFFFu) | (n << 16);
    V.max[s] = mx;
    V.mask[s] = mask;
  }
}

// Stage B1, one thread per query: bounds and routing of query qi in this tile.  Skipped: no doc of the tile can reach the query's
// threshold;  flat: the essential postings become work-list segments that the CTA's threads share evenly (B2);  heavy: a warp
// accumulates the query's window (B3; sample launches, and pairs with many postings).  A work list that fills up defers the
// query to another round of B1 + B2 (the list is sized for the common case).  th_pre0 / th_pre1: the thresholds of queries tid and
// tid + kTileThreads, loaded before stage A.
template <bool kSample, bool kUnionOnly>
__device__ __forceinline__ void tile_route(const BatchParams& P, const TileParams& TP, const TileView& V, TileCtl& C,
                                           const uint16_t* __restrict__ cl0, uint32_t qi, uint32_t th_pre0, uint32_t th_pre1, TileStats& st) {
  const TileTQ tq = V.tq[qi];
  const uint16_t* __restrict__ cl = cl0 + tq.clause_base;
  const uint32_t th_key = qi < kTileThreads ? th_pre0 : qi < 2u * kTileThreads ? th_pre1 : (uint32_t)*(volatile unsigned int*)&P.qstate[tq.query].theta;
  const float theta_f = threshold_score(th_key);
  const bool prune = (tq.op_flags & 128u) && theta_f > 0.0f && !kSample;
  const uint32_t n = tq.n_clauses, op = kUnionOnly ? 0u : tq.op_flags & 3u;
  ++st.pairs;
  TileQ rec;
  rec.qi = (uint16_t)qi; rec.th_key = th_key; rec.n_op = (uint8_t)((op == kTileOpBool ? 0u : n) | (op << 6));
  uint32_t cnt = 0, n_segs = 0, rec_ne = 0;
  uint32_t b_d0 = 0, b_dn = 0;  // kTileOpBool: the driving words
  if (!kUnionOnly && op == kTileOpBool) {
    float bound;
    cnt = tile_bool_drive(V, cl, b_d0, b_dn, bound);
    if (cnt == 0u || (prune && bound * 1.00001f < theta_f)) { ++st.skipped; return; }
    for (uint32_t e = 0; e < b_dn; ++e) n_segs += (V.info[cl[b_d0 + e]] >> 16) ? 1u : 0u;
    rec.ne = __uint_as_float(b_d0 | (b_dn << 16));
    rec.shared_stripes = 0u;
  } else if (!kUnionOnly && op == kTileOpAnd) {
    float bound;
    cnt = tile_and_drive(V, cl, n, rec_ne, bound);
    if (cnt == 0u || (prune && bound * 1.00001f < theta_f)) { ++st.skipped; return; }
    rec.ne = 0.0f; rec.shared_stripes = 0u;
    n_segs = 1;
  } else {
    // sample launch: only the docs of the two heaviest clauses are scored (completely): the best docs of a union nearly
    // always hold its rarest terms, and ANY real score is a valid sample
    uint32_t n_e = n;
    if (kSample) {  // ... extended by further clauses while the tile holds fewer than four of their postings
      uint32_t have = 0;
      n_e = 0;
      while (n_e < n && (n_e < 2u || have < 4u)) { have += V.info[cl[n_e]] >> 16; ++n_e; }
    }
    float ne;
    n_e = tile_essential(V, cl, n_e, prune, theta_f, ne);
    if (n_e == 0) { ++st.skipped; return; }  // no doc of this tile can reach the threshold
    uint32_t seen = 0, shared = 0;
    for (uint32_t c = 0; c < n_e; ++c) {
      const uint32_t slot = cl[c];
      const uint32_t len = V.info[slot] >> 16;
      cnt += len; n_segs += len ? 1u : 0u;
      const uint32_t m = V.mask[slot];
      shared |= seen & m;
      seen |= m;
    }
    if (cnt == 0) { ++st.skipped; return; }  // a doc without an essential posting stays below the threshold
    rec_ne = n_e; rec.ne = ne; rec.shared_stripes = shared;
  }
  rec.ne_prune = (uint8_t)(rec_ne | (prune ? 128u : 0u));
  // sample launch: ANY set of real scores is a valid sample -- at most kSampleSeg postings per driving clause, no window path
  if (kSample && *(volatile unsigned int*)&TP.sample_count[tq.query] >= TP.sample_cap) return;
  bool heavy = !kSample && cnt > TP.light_max && op != kTileOpAnd && op != kTileOpBool && rec_ne >= 2u;
  if (n_segs > TP.seg_cap) heavy = true;  // (test hook sizes only)
  if (!heavy) {
    const uint32_t sb = atomicAdd(&C.nseg, n_segs);
    if (sb + n_segs > TP.seg_cap) {  // the work list is full (entries from here on are not written): next round
      atomicMin(&C.segvalid, sb);
      atomicOr(&C.defer[qi >> 5], 1u << (qi & 31u));
      C.ndefer = 1u;
    } else {
      const uint32_t qslot = atomicAdd(&C.nflat, 1u);
      V.q[qslot] = rec;
      uint32_t w = sb;
      if (!kUnionOnly && op == kTileOpBool) {
        for (uint32_t e = 0; e < b_dn; ++e)
          if (V.info[cl[b_d0 + e]] >> 16) V.seg[w++] = TileSeg{(uint16_t)qslot, (uint16_t)(b_d0 + e)};
      } else if (!kUnionOnly && op == kTileOpAnd) {
        V.seg[w] = TileSeg{(uint16_t)qslot, (uint16_t)rec_ne};
      } else {
        for (uint32_t c = 0; c < rec_ne; ++c)
          if (V.info[cl[c]] >> 16) V.seg[w++] = TileSeg{(uint16_t)qslot, (uint16_t)c};
      }
      ++st.flat;
      st.ess += cnt;
    }
  }
  if (heavy) V.heavy[atomicAdd(&C.nheavy, 1u)] = (uint16_t)qi;
}

// Stage B2: the flat pairs' essential postings, one per thread.  A warp takes 32 work-list segments at a time, one per lane, and
// deals their postings to the lanes 32 at a time (load-balanced expansion).
template <bool kSample, bool kCounters, bool kUnionOnly>
__device__ __forceinline__ void tile_flat(const BatchParams& P, const TileParams& TP, const TSeg& G, const TileView& V, TileCtl& C,
                                          const uint16_t* __restrict__ cl0, uint32_t lo, uint32_t lane, TileStats& st) {
  const uint32_t n_seg = min(C.nseg, C.segvalid);
  for (;;) {
    uint32_t sbase = 0;
    if (lane == 0) sbase = atomicAdd(&C.segpos, 32u);
    sbase = __shfl_sync(kFull, sbase, 0);
    if (sbase >= n_seg) break;
    uint32_t m_len = 0, m_qc = 0, m_start = 0;  // the lane's segment: postings [m_start, m_start + m_len), q | clause << 16
    // kUnionOnly: the segment's query state, read once here and handed to the posting lanes with shuffles (instead of three
    // dependent shared loads per posting): th_key, ne, the clause's tile_or_tail, shared_stripes, clause base | n << 16 |
    // n_e << 22 | prune << 28, query
    uint32_t m_th = 0, m_ne = 0, m_tail = 0, m_ss = 0, m_cb = 0, m_query = 0;
    if (sbase + lane < n_seg) {
      const TileSeg sg = V.seg[sbase + lane];
      uint32_t info;
      if constexpr (kUnionOnly) {
        const TileQ q = V.q[sg.q];
        const TileTQ qq = V.tq[q.qi];
        info = V.info[cl0[qq.clause_base + sg.clause]];
        m_th = q.th_key; m_ne = __float_as_uint(q.ne); m_ss = q.shared_stripes; m_query = qq.query;
        m_tail = __float_as_uint(tile_or_tail(V, cl0 + qq.clause_base, sg.clause, q.n_e(), q.ne));
        m_cb = qq.clause_base | (q.n() << 16) | (q.n_e() << 22) | (q.prune() ? 1u << 28 : 0u);
      } else {
        info = V.info[cl0[V.tq[V.q[sg.q].qi].clause_base + sg.clause]];
      }
      m_qc = sg.q | ((uint32_t)sg.clause << 16);
      m_start = info & 0xFFFFu;
      m_len = kSample ? min(info >> 16, kSampleSeg) : info >> 16;
    }
    const uint32_t incl = warp_incl_scan(m_len, lane);
    const uint32_t total = __shfl_sync(kFull, incl, 31);
    const uint32_t excl = incl - m_len;
    const uint32_t m_pbase = m_start - excl;  // (mod 2^32) the pair index of the chunk item ibase + lane is m_pbase + ibase + lane
    for (uint32_t ibase = 0; ibase < total; ibase += 32u) {
      const uint32_t item = ibase + lane;
      // the segment of item `ibase + lane`: every listed segment holds a posting, so segment numbers grow by one at each
      // start; (segments that start before this chunk) - 1 + (starts at or before the lane's item)
      const uint32_t rel = excl - ibase;  // (wraps for segments that start before the chunk)
      const uint32_t starts = __reduce_or_sync(kFull, (m_len && rel < 32u) ? (1u << rel) : 0u);
      const uint32_t earlier = (uint32_t)__popc(__ballot_sync(kFull, m_len && excl < ibase));
      const uint32_t j = earlier - 1u + (uint32_t)__popc(starts & (0xFFFFFFFFu >> (31u - lane)));
      const uint32_t src = j & 31u;
      const uint32_t p = __shfl_sync(kFull, m_pbase, src) + item;
      const uint32_t qc = __shfl_sync(kFull, m_qc, src);
      uint32_t b_th = 0, b_ne = 0, b_tail = 0, b_ss = 0, b_cb = 0, b_query = 0;
      if constexpr (kUnionOnly) {
        b_th = __shfl_sync(kFull, m_th, src);
        b_ne = __shfl_sync(kFull, m_ne, src);
        b_tail = __shfl_sync(kFull, m_tail, src);
        b_ss = __shfl_sync(kFull, m_ss, src);
        b_cb = __shfl_sync(kFull, m_cb, src);
        b_query = __shfl_sync(kFull, m_query, src);
      }
      uint32_t s_query = 0xFFFFFFFFu - lane, s_key = 0;  // sample launch: this lane's sample (if any), handed over below
      if (item < total) {
        const uint32_t off = V.off[p];
        float sum;
        bool ok;
        uint32_t query, th_key;
        uint32_t ex = kOrExits;  // (a union's posting: how tile_eval_or left it)
        if constexpr (kUnionOnly) {
          query = b_query; th_key = b_th;
          ok = tile_eval_or<kCounters && !kSample, true>(V, cl0 + (b_cb & 0xFFFFu), (b_cb >> 22) & 63u, (b_cb >> 16) & 63u, (b_cb >> 28) != 0u,
                                                         __uint_as_float(b_ne), __uint_as_float(b_tail), b_ss, qc >> 16, p, off, threshold_score(th_key), sum, ex);
        } else {
          const TileSeg sg{(uint16_t)qc, (uint16_t)(qc >> 16)};
          const TileQ q = V.q[sg.q];
          const TileTQ qq = V.tq[q.qi];
          const uint16_t* __restrict__ cl = cl0 + qq.clause_base;
          query = qq.query; th_key = q.th_key;
          const bool io = (qq.op_flags & 32u) != 0;
          if (q.op() == kTileOpBool) ok = tile_eval_bool(V, cl, __float_as_uint(q.ne) & 0xFFFFu, sg.clause, p, off, io, sum);
          else if (q.op() == kTileOpAnd) ok = tile_eval_and(V, cl, q.n(), q.n_e(), p, off, io, sum);
          else ok = tile_eval_or<kCounters && !kSample, false>(V, cl, q.n_e(), q.n(), q.prune(), q.ne, 0.0f, q.shared_stripes, sg.clause, p, off, threshold_score(th_key), sum, ex);
        }
        if (kCounters && !kSample) { st.or_exit[0] += ex == kOrBound; st.or_exit[1] += ex == kOrOwner; st.or_exit[2] += ex == kOrWalk; st.or_exit[3] += ex == kOrDone; }
        if (ok) {
          ++st.completed;
          const uint32_t key = score_to_key(sum);
          if (key >= th_key) ++st.pushed;
          if (!kSample) tile_push(P, TP, C, query, sum, lo + off, G.segment_ord, th_key, G.alive);
          else if (key >= th_key && key != 0u && (!G.alive || is_alive(G.alive, lo + off))) { s_query = query; s_key = key; }  // (a deleted doc bounds nothing)
        }
      }
      if (kSample) {  // one atomic per query and warp step instead of one per sample (the counters are hot)
        const unsigned peers = __match_any_sync(kFull, s_query);
        if (s_key) {
          const uint32_t leader = (uint32_t)__ffs(peers) - 1u;
          uint32_t base = 0;
          if (lane == leader) base = atomicAdd(&TP.sample_count[s_query], (uint32_t)__popc(peers));
          base = __shfl_sync(peers, base, leader);
          const uint32_t idx = base + (uint32_t)__popc(peers & lanemask_lt(lane));
          if (idx < TP.sample_cap) TP.samples[(size_t)s_query * TP.sample_cap + idx] = s_key;
        }
      }
    }
  }
}

// Stage B3 of a conjunction or TQ_OP_BOOL query: the lanes share the postings of the driving words [d0, d0 + dn) of cl, and each
// evaluates its docs with eval(word, posting, doc offset, sum).
template <bool kSample, typename Eval>
__device__ __forceinline__ void tile_heavy_driven(const BatchParams& P, const TileParams& TP, const TSeg& G, const TileView& V, TileCtl& C, const uint16_t* __restrict__ cl,
                                                  uint32_t d0, uint32_t dn, uint32_t query, uint32_t th_key, uint32_t lo, uint32_t lane, TileStats& st, Eval eval) {
  uint32_t best = 0;
  for (uint32_t w = d0; w < d0 + dn; ++w) {
    const uint32_t info = V.info[cl[w]];
    const uint32_t a = info & 0xFFFFu, e = a + (info >> 16);
    for (uint32_t p = a + lane; p < e; p += 32) {
      const uint32_t off = V.off[p];
      float sum;
      if (!eval(w, p, off, sum)) continue;
      if (kSample) { if (!G.alive || is_alive(G.alive, lo + off)) best = max(best, score_to_key(sum)); }  // (a deleted doc bounds nothing)
      else { ++st.completed; tile_push(P, TP, C, query, sum, lo + off, G.segment_ord, th_key, G.alive); }
    }
    if (lane == 0) st.ess += e - a;
  }
  if (kSample) warp_push_samples(TP, query, best, th_key, lane);
}

// Stage B3: heavy pair qi, evaluated by one warp.  A union accumulates its essential clauses into the warp's window `acc` of f32
// score slots, clause by clause (the f32 summation order), then completes each touched doc with the non-essential suffix.
template <bool kSample, bool kUnionOnly>
__device__ __forceinline__ void tile_heavy(const BatchParams& P, const TileParams& TP, const TSeg& G, const TileView& V, TileCtl& C,
                                           const uint16_t* __restrict__ cl0, uint32_t qi, float* acc, uint32_t lo, uint32_t lane, TileStats& st) {
  const TileTQ tq = V.tq[qi];
  const uint16_t* __restrict__ cl = cl0 + tq.clause_base;
  uint32_t th_key = 0;
  if (lane == 0) th_key = *(volatile unsigned int*)&P.qstate[tq.query].theta;
  th_key = __shfl_sync(kFull, th_key, 0);  // one value for the whole warp (the query-wide threshold moves)
  const float theta_f = threshold_score(th_key);
  const bool prune = (tq.op_flags & 128u) && theta_f > 0.0f && !kSample;
  const uint32_t n = tq.n_clauses;
  const bool io = (tq.op_flags & 32u) != 0;
  if (lane == 0) ++st.heavy;
  float bound, ne;  // (the bound B1 needs is not used here)
  if (!kUnionOnly && (tq.op_flags & 3u) == kTileOpBool) {
    uint32_t d0 = 0, dn = 0;
    tile_bool_drive(V, cl, d0, dn, bound);
    return tile_heavy_driven<kSample>(P, TP, G, V, C, cl, d0, dn, tq.query, th_key, lo, lane, st,
                                      [&](uint32_t w, uint32_t p, uint32_t off, float& sum) { return tile_eval_bool(V, cl, d0, w, p, off, io, sum); });
  }
  if (!kUnionOnly && (tq.op_flags & 3u) == kTileOpAnd) {
    uint32_t drv;
    tile_and_drive(V, cl, n, drv, bound);
    return tile_heavy_driven<kSample>(P, TP, G, V, C, cl, drv, 1u, tq.query, th_key, lo, lane, st,
                                      [&](uint32_t w, uint32_t p, uint32_t off, float& sum) { return tile_eval_and(V, cl, n, w, p, off, io, sum); });
  }
  const uint32_t n_e = tile_essential(V, cl, n, prune, theta_f, ne);
  for (uint32_t g = 0; g < kTile / 128u; ++g)  // -0.0 = untouched (-0.0 + s == s)
    *reinterpret_cast<float4*>(acc + g * 128u + lane * 4u) = make_float4(-0.0f, -0.0f, -0.0f, -0.0f);
  __syncwarp();
  float wmax = 0.0f;
  for (uint32_t c = 0; c < n_e; ++c) {  // clause order is the f32 summation order
    const uint32_t info = V.info[cl[c]];
    const uint32_t a = info & 0xFFFFu, e = a + (info >> 16);
    for (uint32_t p = a + lane; p < e; p += 32) {
      const uint32_t o = V.off[p];
      const float v = __fadd_rn(acc[o], V.score[p]);
      acc[o] = v;
      wmax = fmaxf(wmax, v);
    }
    if (lane == 0) st.ess += e - a;
    __syncwarp();
  }
  if (kSample) {
    // the best partial maximum of every lane's slots; the top few of the warp are this (query, tile)'s samples
    uint32_t best = 0;
    for (uint32_t g = 0; g < kTile / 128u; ++g) {
      const uint32_t idx = g * 128u + lane * 4u;
      const float4 v = *reinterpret_cast<const float4*>(acc + idx);
      const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (__float_as_uint(vv[c]) != 0x80000000u && (!G.alive || is_alive(G.alive, lo + idx + c))) best = max(best, score_to_key(vv[c]));  // a deleted doc's score bounds nothing
    }
    warp_push_samples(TP, tq.query, best, th_key, lane);
    return;
  }
  // nothing of this window can reach the threshold when even its largest partial sum plus the bound cannot
  const float mx = __uint_as_float(__reduce_max_sync(kFull, __float_as_uint(wmax)));
  const bool cold = prune && (mx + ne) * 1.00001f < theta_f;
  if (cold && lane == 0) ++st.skipped;
  for (uint32_t g = 0; g < kTile / 128u && !cold; ++g) {
    const uint32_t idx = g * 128u + lane * 4u;
    const float4 v = *reinterpret_cast<const float4*>(acc + idx);
    const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float sum = vv[c];
      if (__float_as_uint(sum) == 0x80000000u) continue;  // untouched
      const uint32_t off = idx + c;
      float rem = ne;
      bool dead = false;
      for (uint32_t c2 = n_e; c2 < n; ++c2) {  // the non-essential suffix, with the same early exit as the flat path
        if (prune && (sum + rem) * 1.00001f < theta_f) { dead = true; break; }
        const uint32_t slot = cl[c2];
        rem -= V.max[slot];
        bool f;
        const float x = tile_find(V, slot, off, f);
        if (f) sum = __fadd_rn(sum, x);
      }
      if (dead) continue;
      ++st.completed;
      if (score_to_key(sum) >= th_key) ++st.pushed;
      tile_push(P, TP, C, tq.query, sum, lo + off, G.segment_ord, th_key, G.alive);
    }
  }
}

// One instantiation per launch kind, so that each compiles only what it runs: kSample = the sample launch (threshold samples
// instead of candidates), kCounters = TQ_TILE_COUNTERS diagnostics, kUnionOnly = every query of the group is a term query or a
// union (no conjunction, no TQ_OP_BOOL: the flat path broadcasts each work-list segment's query state from the lane that reads
// the segment).  The exact launches without counters do ~90 % of the work; they must fit 64 registers so that four CTAs share an SM.
template <bool kSample, bool kCounters, bool kUnionOnly>
__global__ void __launch_bounds__(kTileThreads, kSample || kCounters ? 3 : 4) k_tile(const BatchParams P, const TileParams TP, uint32_t unit_base) {
  // kCounters: each warp's clock64() time by stage (lane 0's view of it); mark(k) books the time since the previous mark to stage k
  long long clk_last = kCounters ? clock64() : 0;
  unsigned long long cyc[kTileStages] = {};
  auto mark = [&](int k) {
    if constexpr (kCounters) {
      const long long now = clock64();
      cyc[k] += (unsigned long long)(now - clk_last);
      clk_last = now;
    }
  };
  extern __shared__ __align__(16) unsigned char s_dyn[];
  __shared__ TileCtl C;
  __shared__ unsigned long long s_stat[kTileStatWords];
  const TUnit U = TP.units[unit_base + blockIdx.x];
  const TSeg G = TP.segs[U.tseg];
  const TSlot* __restrict__ slots = TP.slots + G.slot_base;
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const TileView V = tile_view(s_dyn, TP, G.n_big);
  // sparse slots: (first pair not staged yet, its doc or 0xFFFFFFFF once the list is exhausted), this CTA's share of the
  // launch's cursor scratch; slot s is always walked by the same thread, so no barrier guards it
  uint2* cursor = TP.cursors + (size_t)blockIdx.x * TP.max_slots;
  if (kCounters && tid < kTileStatWords) s_stat[tid] = 0ull;
  if (tid < kTileMaxQueries / 32u) C.defer[tid] = 0u;
  if (tid == 0) C.nref = 0u;
  const bool cl_staged = G.n_clause_words <= TP.cl_cap;
  const uint16_t* __restrict__ cl0 = cl_staged ? V.cl : TP.clauses + G.clause_base;
  tile_prologue(TP, G, slots, V, cl_staged, cursor, U.t0, tid);
  mark(kStPrologue);
  __syncthreads();
  mark(kStBarrier);
  TileStats st{};
  for (uint32_t t = U.t0; t < U.t1; ++t) {
    const uint32_t lo = t * kTile;
    // the thresholds of this thread's B1 queries (qi = tid, tid + kTileThreads): loaded now, they travel while the tile is staged.
    // Thresholds only rise (atomicMax), so a value read before stage A still bounds the query's final k-th score from below
    uint32_t th_pre0 = 0u, th_pre1 = 0u;
    if (tid < G.n_queries) th_pre0 = *(volatile unsigned int*)&P.qstate[V.tq[tid].query].theta;
    if (tid + kTileThreads < G.n_queries) th_pre1 = *(volatile unsigned int*)&P.qstate[V.tq[tid + kTileThreads].query].theta;
    if (tid < G.n_big) {  // three independent loads per dense slot: one round trip for the whole tile
      const uint32_t a = __ldg(G.tix + (size_t)t * G.n_big + tid), b = __ldg(G.tix + (size_t)(t + 1u) * G.n_big + tid);
      V.a->ba[tid] = __ldg(&slots[tid].pair_base) + a;
      V.a->bn[tid] = b - a;
    }
    if (tid == 0) { C.total = 0; C.nheavy = 0; C.hpos = 0; C.nflat = 0; C.nseg = 0; C.segpos = 0; C.segvalid = TP.seg_cap; C.ndefer = 0; }
    mark(kStA);
    __syncthreads();
    mark(kStBarrier);
    if (tid == 0) C.nref = 0u;  // (every warp has read the previous tile's refresh list: nothing is pushed before B2)
    // ---- stage A: this tile's pairs of every slot -> shared memory ----------------------------------------------------------
    if (warp < G.n_big) tile_stage_dense(TP, G, V, C.total, lo, warp, lane);
    tile_stage_sparse(TP, G, slots, V, cursor, C.total, lo, tid);
    mark(kStA);
    __syncthreads();
    mark(kStBarrier);
    if (C.total > TP.p_cap) {  // more pairs than the tile buffer holds: give the batch back to the per-query kernels
      if (tid == 0) atomicExch(TP.flags, 1u);
      __syncthreads();
      mark(kStBarrier);
      continue;
    }
    // ---- stages B1 + B2, in rounds while queries are deferred -----------------------------------------------------------------
    for (uint32_t round = 0;; ++round) {
      for (uint32_t qi = tid; qi < G.n_queries; qi += kTileThreads) {
        if (round) {
          const uint32_t bit = 1u << (qi & 31u);
          if (!(C.defer[qi >> 5] & bit)) continue;
          atomicAnd(&C.defer[qi >> 5], ~bit);
        }
        tile_route<kSample, kUnionOnly>(P, TP, V, C, cl0, qi, th_pre0, th_pre1, st);
      }
      mark(kStB1);
      __syncthreads();
      mark(kStBarrier);
      const bool more_rounds = C.ndefer != 0u;
      tile_flat<kSample, kCounters, kUnionOnly>(P, TP, G, V, C, cl0, lo, lane, st);
      mark(kStB2);
      if (!more_rounds) break;
      __syncthreads();
      if (tid == 0) { C.nflat = 0; C.nseg = 0; C.segpos = 0; C.segvalid = TP.seg_cap; C.ndefer = 0; }
      __syncthreads();
      mark(kStBarrier);
    }
    // ---- stage B3: one warp per heavy pair, a window of f32 score slots ------------------------------------------------------
    const uint32_t n_heavy = C.nheavy;
    if (n_heavy) __syncthreads();  // the windows overlay the work list: every warp must be done with B2
    mark(kStBarrier);
    float* acc = V.acc + warp * kTile;
    for (; warp < TP.n_win;) {  // (the warps without a window go straight to the barrier)
      uint32_t h = 0;
      if (lane == 0) h = atomicAdd(&C.hpos, 1u);
      h = __shfl_sync(kFull, h, 0);
      if (h >= n_heavy) break;
      tile_heavy<kSample, kUnionOnly>(P, TP, G, V, C, cl0, V.heavy[h], acc, lo, lane, st);
      __syncwarp();
    }
    mark(kStB3);
    __syncthreads();
    mark(kStBarrier);
    // ---- the running thresholds of the queries this tile's pushes put on the refresh list (tile_push): a warp per query -------
    if constexpr (!kSample) {
      const uint32_t n_ref = min(C.nref, kTileRefreshCap);
      for (uint32_t i = warp; i < n_ref; i += kTileWarps) {
        const bool raised = tile_theta_refresh(P, TP, C.ref[i], lane);
        if (kCounters && lane == 0) { ++st.refreshes; st.raises += raised ? 1u : 0u; }
      }
      mark(kStB3);
    }
  }
  if constexpr (kCounters) {
    // warp-aggregated diagnostics (s_stat / TileParams::counters: the 7 of TileStats, 8 + the stages, 14 the refreshes, 15 the raises,
    // 16 + the union exits)
    unsigned long long v[9 + kOrExits] = {st.pairs, st.skipped, st.flat, st.heavy, st.ess, st.completed, st.pushed,
                                          st.refreshes, st.raises, st.or_exit[0], st.or_exit[1], st.or_exit[2], st.or_exit[3]};
#pragma unroll
    for (int i = 0; i < 9 + kOrExits; ++i) {
      unsigned long long x = v[i];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(kFull, x, o);
      if (lane == 0 && x) atomicAdd(&s_stat[i < 7 ? i : i < 9 ? 14 + (i - 7) : 16 + (i - 9)], x);
    }
    if (lane == 0)
      for (int k = 0; k < kTileStages; ++k) atomicAdd(&s_stat[8 + k], cyc[k]);
    __syncthreads();
    if (tid < kTileStatWords && tid != 7 && s_stat[tid]) atomicAdd(&TP.counters[tid], s_stat[tid]);
  }
}

// ---- Count next to TopDocs -------------------------------------------------------------------------------------------------
// k_count_tiles: the Count half of (Count, TopDocs) (collector/mod.rs:322-365) for the group's queries that carry
// TQ_QUERY_COUNT_HITS (TQuery::flags & kTileQueryCount), taken from the pairs k_score_lists has already written -- no list is
// decoded again.  A CTA walks a range of tiles of one segment; unlike k_tile it skips nothing, so its units cover every tile of the
// segment's doc range.  Per tile it builds each slot's presence in shared memory: a dense slot (the first n_big) as a 1024-bit map,
// one bit per pair of its tile-index range (what tile_stage_dense stages, without the scores: no pair buffer, no capacity); a
// sparse slot as the doc offsets of its few pairs, walked with a cursor as tile_stage_sparse does (the cursors are this kernel's
// own: k_tile's are in use by the launches next to it).  Then a warp per flagged query evaluates the tile as 32 stripe words, one
// per lane: a term query or a union ORs its clause words, a conjunction ANDs them, TQ_OP_BOOL ANDs its MUST groups (each the OR of
// its clauses), keeps the docs that at least `need` SHOULD words list (a bit-sliced counter per lane: <= 32 clauses fit six words)
// and clears the MUST_NOT words.  And-ed with the alive words (tq_segment_set_doc_range has cleared the docs outside the range in
// them), popcount, a warp sum; one 64-bit add per (query, CTA).  A tile whose sparse offsets exceed kCountSparseCap sets the
// group's overflow word: its flagged queries are then recounted by k_count (tq_batch_fetch_hits).
// (kTileQueryCount, kCountSparseCap, CountTileParams and count_tiles_smem_bytes: tq_layout.h)

// Lane `lane`'s stripe word of `slot` in this tile: bit i = the slot lists doc lo + 32 * lane + i.
__device__ __forceinline__ uint32_t count_word(const uint32_t* bits, const uint32_t* info, const uint16_t* off, uint32_t n_big, uint32_t slot,
                                               uint32_t lane) {
  if (slot < n_big) return bits[slot * 32u + lane];
  const uint32_t in = info[slot];
  uint32_t w = 0;
  for (uint32_t i = in & 0xFFFFu, e = i + (in >> 16); i < e; ++i) {
    const uint32_t o = off[i];
    if ((o >> 5) == lane) w |= 1u << (o & 31u);
  }
  return w;
}

__global__ void __launch_bounds__(kTileThreads) k_count_tiles(const TileParams TP, const CountTileParams CP) {
  extern __shared__ __align__(16) unsigned char s_dyn[];
  __shared__ uint32_t s_total;
  const TUnit U = CP.units[blockIdx.x];
  const TSeg G = TP.segs[U.tseg];
  const TSlot* __restrict__ slots = TP.slots + G.slot_base;
  uint32_t* bits = reinterpret_cast<uint32_t*>(s_dyn);
  uint32_t* info = bits + TP.max_big * 32u;
  uint32_t* cnt = info + TP.max_slots;
  uint16_t* off = reinterpret_cast<uint16_t*>(cnt + TP.max_queries);
  uint2* cursor = CP.cursors + (size_t)blockIdx.x * TP.max_slots;
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  for (uint32_t i = tid; i < G.n_queries; i += kTileThreads) cnt[i] = 0u;
  {  // every sparse slot's cursor on its first pair at or after the unit's first doc
    const uint32_t lo0 = U.t0 * kTile;
    for (uint32_t s = G.n_big + tid; s < G.n_slots; s += kTileThreads) {
      const TSlot sl = slots[s];
      const uint32_t* __restrict__ d = TP.p_docs + sl.pair_base;
      uint32_t a = 0, b = sl.doc_freq;
      while (a < b) {
        const uint32_t m = (a + b) >> 1;
        if (__ldg(d + m) < lo0) a = m + 1u; else b = m;
      }
      cursor[s] = make_uint2(a, a < sl.doc_freq ? __ldg(d + a) : 0xFFFFFFFFu);
    }
  }
  for (uint32_t t = U.t0; t < U.t1; ++t) {
    const uint32_t lo = t * kTile, hi = lo + kTile;
    if (tid == 0) s_total = 0u;
    for (uint32_t i = tid; i < G.n_big * 32u; i += kTileThreads) bits[i] = 0u;
    __syncthreads();
    // dense slots: warp w takes slots w, w + 8, ..., 128 pairs per step
    for (uint32_t s = warp; s < G.n_big; s += kTileWarps) {
      const uint32_t a = __ldg(G.tix + (size_t)t * G.n_big + s), e = __ldg(G.tix + (size_t)(t + 1u) * G.n_big + s);
      const uint32_t* __restrict__ d = TP.p_docs + __ldg(&slots[s].pair_base);
      for (uint32_t i0 = a; i0 < e; i0 += 128u) {
        uint32_t dv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const uint32_t i = i0 + (uint32_t)u * 32u + lane;
          dv[u] = i < e ? __ldg(d + i) : 0xFFFFFFFFu;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (dv[u] != 0xFFFFFFFFu) {
            const uint32_t o = dv[u] - lo;
            atomicOr(&bits[s * 32u + (o >> 5)], 1u << (o & 31u));
          }
      }
    }
    // sparse slots: a thread walks a slot's cursor through the tile
    for (uint32_t s = G.n_big + tid; s < G.n_slots; s += kTileThreads) {
      const uint2 cs = cursor[s];
      if (cs.y >= hi) { info[s] = 0u; continue; }
      const TSlot sl = slots[s];
      const uint32_t* __restrict__ d = TP.p_docs + sl.pair_base;
      uint32_t n = 1, nd;
      for (;;) {
        const uint32_t c = cs.x + n;
        nd = c < sl.doc_freq ? __ldg(d + c) : 0xFFFFFFFFu;
        if (nd >= hi) break;
        ++n;
      }
      cursor[s] = make_uint2(cs.x + n, nd);
      const uint32_t base = atomicAdd(&s_total, n);
      if (base + n <= kCountSparseCap) {
        off[base] = (uint16_t)(cs.y - lo);
        for (uint32_t i = 1; i < n; ++i) off[base + i] = (uint16_t)(__ldg(d + cs.x + i) - lo);
      }
      info[s] = (base & 0xFFFFu) | (n << 16);
    }
    __syncthreads();
    if (s_total > kCountSparseCap) {  // the group's flagged queries are recounted without this kernel: nothing more to do here
      if (tid == 0) atomicOr(CP.overflow, 1u);
      return;
    }
    // lane j's alive word covers docs lo + 32 j .. + 31 (little-endian 64-bit words read as 32-bit halves); no list holds a doc
    // at or beyond max_doc, so those words are never needed
    uint32_t live = 0xFFFFFFFFu;
    if (G.alive) live = lo + lane * 32u < G.max_doc ? __ldg(reinterpret_cast<const uint32_t*>(G.alive) + (lo >> 5) + lane) : 0u;
    for (uint32_t qi = warp; qi < G.n_queries; qi += kTileWarps) {
      const TQuery tq = TP.queries[G.query_base + qi];
      if (!(tq.flags & kTileQueryCount)) continue;
      const uint16_t* __restrict__ cl = TP.clauses + tq.clause_base;
      uint32_t m;
      if (tq.op == kTileOpBool) {
        const uint32_t ng = cl[0], need = cl[1], ns = cl[2], nn = cl[3];
        uint32_t w = 4;
        m = 0xFFFFFFFFu;
        for (uint32_t g = 0; g < ng; ++g) {
          const uint32_t glen = cl[w++];
          uint32_t gm = 0;
          for (uint32_t e = 0; e < glen; ++e, ++w) gm |= count_word(bits, info, off, G.n_big, cl[w], lane);
          m &= gm;
        }
        if (need && __any_sync(kFull, m)) {
          uint32_t sc[6] = {0, 0, 0, 0, 0, 0};  // bit-sliced per-doc count of the SHOULD clauses that list the doc
          for (uint32_t e = 0; e < ns; ++e) {
            uint32_t carry = count_word(bits, info, off, G.n_big, cl[w + e], lane);
#pragma unroll
            for (int b = 0; b < 6; ++b) {
              const uint32_t c2 = sc[b] & carry;
              sc[b] ^= carry;
              carry = c2;
            }
          }
          uint32_t gt = 0, eq = 0xFFFFFFFFu;  // count > need so far / count == need so far, from the top bit down
#pragma unroll
          for (int b = 5; b >= 0; --b) {
            if ((need >> b) & 1u) eq &= sc[b];
            else { gt |= eq & sc[b]; eq &= ~sc[b]; }
          }
          m &= gt | eq;
        }
        w += ns;
        for (uint32_t e = 0; e < nn; ++e) m &= ~count_word(bits, info, off, G.n_big, cl[w + e], lane);
      } else if (tq.op == kTileOpAnd) {
        m = 0xFFFFFFFFu;
        for (uint32_t c = 0; c < tq.n_clauses && __any_sync(kFull, m); ++c) m &= count_word(bits, info, off, G.n_big, cl[c], lane);
      } else {
        m = 0;
        for (uint32_t c = 0; c < tq.n_clauses; ++c) m |= count_word(bits, info, off, G.n_big, cl[c], lane);
      }
      const uint32_t n = __reduce_add_sync(kFull, (uint32_t)__popc(m & live));
      if (lane == 0) cnt[qi] += n;
    }
    __syncthreads();
  }
  for (uint32_t i = tid; i < G.n_queries; i += kTileThreads)
    if (cnt[i]) atomicAdd(CP.hits + TP.queries[G.query_base + i].query, (unsigned long long)cnt[i]);
}

// ---- thresholds from score keys -------------------------------------------------------------------------------------------
// k-th largest of n u32 keys (4-pass radix select), block-wide; returns 0 when n < k.  `need_out`: how many keys equal to the
// result are needed on top of the strictly larger ones to make k.
__device__ __forceinline__ uint32_t block_kth_key(const uint32_t* __restrict__ keys, uint32_t n, uint32_t stride_words, uint32_t k,
                                                  uint32_t* s_hist, uint32_t* s_prefix, uint32_t* s_need) {
  if (n < k) return 0u;
  if (threadIdx.x == 0) { *s_prefix = 0; *s_need = k; }
  uint32_t mask = 0;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    const uint32_t prefix = *s_prefix;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
      const uint32_t key = keys[(size_t)i * stride_words];
      if ((key & mask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t need = *s_need, bsel = 0;
      for (int bin = 255; bin >= 0; --bin) {
        const uint32_t h = s_hist[bin];
        if (h >= need) { bsel = (uint32_t)bin; break; }
        need -= h;
      }
      *s_need = need;
      *s_prefix = prefix | (bsel << shift);
    }
    mask |= 0xFFu << shift;
    __syncthreads();
  }
  return *s_prefix;
}

// After the sample launch: the k-th best sampled score of a query bounds its final k-th score from below.  The threshold it leaves
// is the base of the query's key histogram in the exact launches (th_hist: fixed for the run, before anything is counted).
__global__ void __launch_bounds__(kThreads) k_theta_samples(const BatchParams P, const uint32_t* __restrict__ samples,
                                                            const uint32_t* __restrict__ sample_count, uint32_t sample_cap,
                                                            uint32_t* __restrict__ th_hist) {
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_prefix, s_need;
  const uint32_t q = blockIdx.x;
  const uint32_t n = min(sample_count[q], sample_cap);
  const uint32_t kth = block_kth_key(samples + (size_t)q * sample_cap, n, 1u, P.queries[q].k, s_hist, &s_prefix, &s_need);
  if (threadIdx.x == 0) th_hist[(size_t)q * kThHistWords + kThHistBaseWord] = max(atomicMax(&P.qstate[q].theta, kth), kth) >> 16;
}

// Cross-shard exchange, export side: the k best score keys a query holds so far (samples after the sample launch, else
// candidates), k_stride entries per query, zero padded.  The caller all-gathers these over the shards.
__global__ void __launch_bounds__(kThreads) k_topkeys_export(const BatchParams P, const uint32_t* __restrict__ samples,
                                                             const uint32_t* __restrict__ sample_count, uint32_t sample_cap,
                                                             uint32_t from_samples, uint32_t* __restrict__ out, uint32_t k_stride) {
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_prefix, s_need, s_n;
  const uint32_t q = blockIdx.x;
  const DQuery Q = P.queries[q];
  const uint32_t* keys;
  uint32_t n, stride;
  if (from_samples && samples) { keys = samples + (size_t)q * sample_cap; n = min(sample_count[q], sample_cap); stride = 1u; }
  else { keys = &P.cands[Q.cand_base].score_key; n = min(P.qstate[q].cand_count, Q.cand_cap); stride = sizeof(Cand) / 4u; }
  const uint32_t k = min(Q.k, k_stride);
  uint32_t* o = out + (size_t)q * k_stride;
  for (uint32_t i = threadIdx.x; i < k_stride; i += blockDim.x) o[i] = 0u;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  if (Q.op == 3u) return;  // TQ_OP_PHRASE: its candidates may still be arriving (second stream); no threshold exchange for phrases
  if (n <= k) {
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) o[i] = keys[(size_t)i * stride];
    return;
  }
  const uint32_t kth = block_kth_key(keys, n, stride, k, s_hist, &s_prefix, &s_need);
  const uint32_t above = k - s_need;  // strictly larger keys
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const uint32_t key = keys[(size_t)i * stride];
    if (key > kth) o[atomicAdd(&s_n, 1u)] = key;
  }
  __syncthreads();
  for (uint32_t i = above + threadIdx.x; i < k; i += blockDim.x) o[i] = kth;
}

// ... import side: gathered [n_shards][nq][k_stride] keys -> the exact k-th best of the union becomes the query's threshold.
__global__ void __launch_bounds__(kThreads) k_theta_from_keys(const BatchParams P, const uint32_t* __restrict__ gathered, uint32_t n_shards,
                                                              uint32_t nq, uint32_t k_stride) {
  extern __shared__ uint32_t s_keys[];  // [n_shards * k_stride]
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_prefix, s_need;
  const uint32_t q = blockIdx.x;
  const uint32_t n = n_shards * k_stride;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x)
    s_keys[i] = gathered[((size_t)(i / k_stride) * nq + q) * k_stride + (i % k_stride)];
  __syncthreads();
  const uint32_t kth = block_kth_key(s_keys, n, 1u, P.queries[q].k, s_hist, &s_prefix, &s_need);
  if (threadIdx.x == 0 && kth) atomicMax(&P.qstate[q].theta, kth);
}

}  // namespace tq
