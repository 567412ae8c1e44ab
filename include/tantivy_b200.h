/*
 * tantivy_b200.h — C ABI of the H100-native query-execution path for tantivy segments.
 *
 * The reference (quickwit-oss/tantivy, Rust) has no FFI; its boundary for this path is the
 * trait surface  Searcher::search -> Collector::collect_segment -> Weight::for_each_pruning
 * (src/core/searcher.rs:180-237, src/collector/mod.rs:173-184, src/query/weight.rs:123-132).
 * The entry points below are what a Rust shim implementing `Collector::collect_segment`
 * (or a `gpu_search(&Searcher, &dyn Query, k)` wrapper) would bind; INTEGRATION.md shows
 * that shim.  Every pointer is a plain host pointer unless its name ends in `_dev`.
 * No exceptions cross this boundary: every call returns TQ_OK or a negative error code and
 * `tq_last_error` gives the message.  All entry points are thread-safe per `tq_ctx`
 * (rayon threads call collect_segment concurrently, src/core/executor.rs:60-100).
 *
 * Doc ids are bit-exact w.r.t. the reference CPU path; scores are f32 computed with the
 * reference's operation order (src/query/bm25.rs:158-175).  A zero score comes back as +0.0, also
 * where the reference's is -0.0 (a weight of -0.0, or a negative one whose product underflows):
 * the reference compares scores with partial_cmp, which ties the two zeros and orders them by
 * DocAddress (sort_by_score.rs:99-107), and so do the score keys here.
 */
#ifndef TANTIVY_B200_H
#define TANTIVY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TQ_OK 0
#define TQ_ERR_INVALID_ARGUMENT (-1)
#define TQ_ERR_CUDA (-2)
#define TQ_ERR_NOT_FOUND (-3)
#define TQ_ERR_UNSUPPORTED (-4)
#define TQ_ERR_OOM (-5)
#define TQ_ERR_CORRUPT (-6)
/* A TQ_OP_BOOL query (tile engine only) has a 1024-doc tile of a segment whose postings, summed over its clauses, exceed the
 * largest tile buffer (12288 pairs), so even a repeat of the query alone cannot hold it.  Split the query or the segment. */
#define TQ_ERR_TILE_CAPACITY (-7)

/* schema::IndexRecordOption (src/schema/index_record_option.rs): decides the skip record
 * size 5 / 8 / 12 bytes (src/postings/skip.rs:205-253). */
#define TQ_RECORD_BASIC 0
#define TQ_RECORD_FREQS 1
#define TQ_RECORD_FREQS_POSITIONS 2

/* Query shapes accelerated: the three specialised scorers of the reference
 * (TermWeight::for_each_pruning, term_weight.rs:118; SpecializedScorer::TermIntersection /
 * TermUnion, boolean_weight.rs:17-21,581-600). */
#define TQ_OP_TERM 0
#define TQ_OP_AND 1
#define TQ_OP_OR 2
/* PhraseQuery (PhraseWeight / PhraseScorer, src/query/phrase_query/phrase_scorer.rs:349-589; slop > 0 for two-term phrases only,
 * intersection_count_with_slop :145-186 -- sloppy phrases of more terms return TQ_ERR_UNSUPPORTED): docs that hold
 * every term, at positions that line up with the terms' offsets in the phrase; score = bm25(fieldnorm, phrase_count)
 * under ONE Bm25Weight for the whole phrase (Bm25Weight::for_terms: the idfs add up, bm25.rs:95-129).  Needs a field
 * indexed WithFreqsAndPositions and its `.pos` bytes (tq_segment_register_positions). */
#define TQ_OP_PHRASE 3
/* BooleanQuery of TermQuery leaves with mixed Occurs, and one level of all-SHOULD sub-queries under MUST
 * (`+a +(b OR c)`, `+(c OR b) +(d OR e)`, `a b -c`, minimum_number_should_match): BooleanWeight::complex_scorer
 * (src/query/boolean_query/boolean_weight.rs:236-431) for these shapes.  Per clause term_occur[t] = TQ_OCCUR_*;
 * MUST clauses that share term_group[t] are alternatives of one required group (a MUST clause of its own: a group of
 * one).  A doc matches when every MUST group has a clause that lists it, at least `min_should_match` SHOULD clauses list
 * it (at least one when there is no MUST group: boolean_weight.rs:354-366), and no MUST_NOT clause lists it (Exclude).
 * Score = (sum over the MUST groups, ascending cost, of the sum of their matching clauses) + (sum of the matching SHOULD
 * clauses) -- Intersection::score / RequiredOptionalScorer::score (intersection.rs:325-329, reqopt_scorer.rs:78-94). */
#define TQ_OP_BOOL 4
#define TQ_OCCUR_SHOULD 0
#define TQ_OCCUR_MUST 1
#define TQ_OCCUR_MUST_NOT 2

/* TERMINATED sentinel of src/docset.rs:12 */
#define TQ_TERMINATED 0x7FFFFFFFu
/* Largest k the device path keeps on chip. */
#define TQ_MAX_K 1024u
/* Largest number of clauses in one query on the device path. */
#define TQ_MAX_TERMS 32u
/* Largest number of terms in a phrase on the device path. */
#define TQ_MAX_PHRASE_TERMS 8u

typedef struct tq_ctx tq_ctx;
typedef struct tq_batch tq_batch;

/* One (clause, segment) posting list: postings::TermInfo (src/postings/term_info.rs:9-16) as
 * returned by InvertedIndexReader::get_term_info (src/index/inverted_index_reader.rs:96).
 * postings_start/end are relative to the field's postings body, i.e. AFTER the 8-byte
 * total_num_tokens header (inverted_index_reader.rs:72-73).  A (clause, segment) pair in
 * which the term does not occur is simply not listed. */
typedef struct {
  uint32_t term_idx;    /* clause ordinal inside the query, 0..n_terms */
  uint32_t segment_ord; /* as given to tq_segment_register */
  uint32_t field;
  uint32_t doc_freq;
  uint64_t postings_start;
  uint64_t postings_end;
} tq_term_seg;

/* TermInfo::positions_range of one (clause, segment) (src/postings/term_info.rs:9-16): byte range of the term's position
 * stream inside the field's `.pos` sub-file (layout: src/positions/mod.rs:22-28).  Only read for TQ_OP_PHRASE. */
typedef struct {
  uint64_t positions_start;
  uint64_t positions_end;
} tq_term_pos;

/* One query = one `Weight` (built once for all segments, searcher.rs:226).
 * weight[i]        = Bm25Weight.weight = idf * (1 + K1) * boost        (bm25.rs:141-151)
 * avg_fieldnorm[i] = Bm25Weight.average_fieldnorm of clause i's field; the 256-entry tf
 *                    cache is recomputed from it exactly as bm25.rs:56-69 does.
 * tf_cache         = optional explicit caches [n_terms][256]; overrides avg_fieldnorm.
 * term_flags       = optional [n_terms] bytes (NULL = all 0).  TQ_TERM_IGNORE_FREQ: the clause is a
 *                    TermQuery::new(term, IndexRecordOption::Basic) on a field indexed WITH term
 *                    frequencies: the reference then skips the tf blocks and scores with tf = 1
 *                    (FreqReadingOption::SkipFreq, block_segment_postings.rs:97-140,343-360).
 * flags/threshold  = TQ_QUERY_HAS_THRESHOLD: only docs with score > threshold are collected -- the initial
 *                    `threshold` argument of Weight::for_each_pruning (src/query/weight.rs:123-132); a caller that
 *                    already holds k hits (another shard, an earlier page) passes its k-th score to prune more.
 *                    TQ_QUERY_COUNT_HITS (TERM / AND / OR / BOOL): the batch also counts the query's matching ALIVE docs -- the
 *                    `Count` half of searcher.search(&query, &(Count, TopDocs::with_limit(k)))  (collector/mod.rs:322-365);
 *                    tq_batch_fetch_hits returns it.  The count ignores k and every threshold (they prune the rows only);
 *                    with TQ_OP_PHRASE the flag fails at prepare with TQ_ERR_INVALID_ARGUMENT. */
#define TQ_TERM_IGNORE_FREQ 1u
#define TQ_QUERY_HAS_THRESHOLD 1u
#define TQ_QUERY_COUNT_HITS 2u
/* TQ_QUERY_FILTER: FilterCollector::new(field, predicate, inner) (src/collector/filter_collector_wrapper.rs:160-199) around the
 * query's TopDocs and Count: only docs that are alive, inside this context's doc range AND set in the bitset registered for
 * (filter_id, segment) with tq_filter_register reach the collectors (collector/mod.rs:186-221 drops the deleted docs first).
 * Scores are the unfiltered query's.  Every segment the query names must have a bitset for filter_id, else prepare (and
 * tq_count_batch) fail with TQ_ERR_NOT_FOUND: a missing filter never reads as "all docs" or "no docs".  filter_id is read only
 * with this flag.  TQ_OP_PHRASE takes it for TopDocs. */
#define TQ_QUERY_FILTER 4u
typedef struct {
  int32_t op;
  uint32_t n_terms;
  uint32_t k; /* TopDocs limit+offset, 1..TQ_MAX_K */
  uint32_t n_term_segs;
  const tq_term_seg* term_segs;
  const float* weight;
  const float* avg_fieldnorm;
  const float* tf_cache;
  const uint8_t* term_flags;
  uint32_t flags;
  float threshold;
  /* TQ_OP_PHRASE only (NULL / 0 otherwise): term_pos[i] belongs to term_segs[i]; term_offset[t] = position of clause t
   * inside the phrase (PhraseQuery::new_with_offset, phrase_query.rs).  The clauses may come in any order: like PhraseQuery,
   * the library orders them by offset (stable: clauses with equal offsets keep their order), which decides the phrase
   * count of a sloppy two-term phrase whose terms have equal doc_freq in a segment.  weight[0] / avg_fieldnorm[0] (or the first
   * tf_cache table) describe the phrase's single Bm25Weight, the other entries are ignored; slop (PhraseQuery::set_slop) may be non-zero
   * for two-term phrases. */
  const tq_term_pos* term_pos;
  const uint32_t* term_offset;
  uint32_t slop;
  uint32_t min_should_match; /* TQ_OP_BOOL: BooleanQuery::minimum_number_should_match */
  /* TQ_OP_BOOL only (NULL otherwise): [n_terms] Occur of every clause; [n_terms] group of every MUST clause (NULL: every
   * MUST clause is a group of its own; ignored for the other Occurs). */
  const uint8_t* term_occur;
  const uint8_t* term_group;
  uint32_t filter_id; /* TQ_QUERY_FILTER only: the doc filter of tq_filter_register */
} tq_query;

/* Counters of the last finished batch (per ctx). */
typedef struct {
  uint64_t lists_cached;      /* posting-list block tables resident on the device */
  uint64_t lists_built;       /* block tables built during the last batch */
  uint64_t units;             /* work units launched in the last batch */
  uint64_t kernel_launches;   /* CUDA kernels launched in the last batch */
  uint64_t h2d_bytes;         /* host->device bytes moved by the last batch */
  uint64_t d2h_bytes;         /* device->host bytes moved by the last batch */
  uint64_t algorithmic_bytes; /* SURVEY.md §8(d): sum over (query,segment,term) of postings
                                 range bytes + doc_freq fieldnorm bytes + 12*k output */
  uint64_t postings;          /* sum of doc_freq over all lists touched */
  float kernel_ms;            /* device time of all kernels of the batch (CUDA events on its stream) */
  float total_ms;             /* device time of the whole batch incl. copies */
  float term_ms, and_ms, or_ms, final_ms; /* per-kernel device time (CUDA events on the launching stream) */
  uint64_t units_term, units_and, units_or; /* CTAs launched per kernel */
  uint64_t bytes_term, bytes_and, bytes_or; /* algorithmic bytes per kernel (same formula) */
  /* cumulative since ctx creation.  k_or_strip (default union kernel): [1] windows scored exhaustively (no
   * non-essential clause under the threshold), [2] hot windows (non-essential clauses applied after the essential
   * ones), [3] cold windows (essential clauses only), [5] bytes of packed postings + fieldnorms actually read
   * (SURVEY.md §8d: the roofline figure of a pruned kernel).  Only k_or_strip counts here; the other slots stay 0. */
  uint64_t or_windows[8];
  uint64_t units_or_strip; /* of units_or: CTAs of the barrier-free strip kernel (k_or_strip); the rest ran k_or */
  /* shared-decode tile engine (k_score_lists + k_tile, csrc/tq_tile.cuh) */
  float score_ms, tile_ms, theta_ms;  /* device time of k_score_lists / all k_tile launches / the k_theta passes of the batch */
  float phrase_ms;                    /* device time of k_phrase */
  uint64_t units_tile;          /* CTAs of k_tile over all its launches */
  uint64_t units_phrase;        /* CTAs of k_phrase */
  uint64_t tile_groups;         /* query groups evaluated together (one decode-and-score pass each) */
  uint64_t tile_postings;       /* postings decoded and scored by k_score_lists (every distinct list once) */
  uint64_t tile_list_bytes;     /* bytes of those lists' postings ranges (skip data + packed blocks + VInt tails) */
  uint64_t tile_scratch_bytes;  /* HBM scratch of the pair arrays, tile indexes, samples, key histograms and the sparse-slot cursors */
  uint64_t tile_fallbacks;      /* 1 if the run overflowed a tile engine buffer and was repeated (TQ_OP_BOOL on the tile engine, the rest on the per-query kernels) */
  uint64_t tile_counters[8];    /* cumulative, with TQ_TILE_COUNTERS=1: (query, tile) pairs seen / skipped / light / heavy,
                                   essential postings applied, docs completed, docs at or above the threshold;
                                   [7] (always): dynamic shared memory bytes of a k_tile CTA of the last prepared group */
  uint64_t tile_ctas_per_sm;    /* k_tile CTAs an SM holds at once in the exact launches of the last prepared group (occupancy API) */
  uint64_t tile_cycles[8];      /* cumulative, with TQ_TILE_COUNTERS=1: k_tile warp cycles (clock64) by stage: [0] cursor prologue,
                                   [1] A (staging), [2] B1 (routing), [3] B2 (flat evaluation), [4] B3 (windows and running-threshold
                                   refreshes), [5] barrier waits; not cycles: [6] running-threshold refreshes of the exact launches,
                                   [7] of them those that raised the query's threshold */
  uint64_t tile_groups_union_only; /* of tile_groups: groups whose queries are all term queries and unions, which run the
                                      union-only k_tile instances (k_tile<*, *, true>); the rest run the general instances */
  uint64_t tile_b2_exits[4];    /* cumulative, with TQ_TILE_COUNTERS=1: union postings of the exact k_tile launches' flat evaluation
                                   (stage B2) by how they ended: [0] dropped by the bound taken before the look-ups, [1] not the owner
                                   (completed the walk, but an earlier essential clause lists the doc), [2] dropped in the
                                   non-essential walk, [3] completed */
  float count_hits_ms;          /* device time of the launches that count TQ_QUERY_COUNT_HITS queries (k_count_tiles, k_count) */
  uint64_t units_count_hits;    /* CTAs of those launches */
  /* cumulative since ctx creation: tq_sort_batch.  Device time of k_sort + k_sort_final, their CTAs (one per unit of up to eight
   * 8192-doc tiles, plus one per query), and the 8192-doc tiles the units came to and of those the ones skipped by the bound. */
  float sort_ms;
  uint64_t units_sort;
  uint64_t sort_tiles_seen;
  uint64_t sort_tiles_skipped;
} tq_stats;

/* ---- context ------------------------------------------------------------------------- */
/* One context drives ONE device (one process per GPU; segments shard across processes). */
int tq_ctx_create(int device, tq_ctx** out);
void tq_ctx_destroy(tq_ctx*);
const char* tq_last_error(tq_ctx*);
int tq_get_stats(tq_ctx*, tq_stats* out);
/* Cumulative since ctx creation: tq_histogram_batch.  Device time of k_hist + k_hist_final, their CTAs (one per unit of up to
 * eight 8192-doc tiles, plus one per query), the 8192-doc tiles the units came to and of those the ones counted as one bucket
 * (every value of the tile in one bucket: the tile's matches added without reading a value).  A struct of its own, so that
 * tq_stats keeps its layout. */
typedef struct {
  float hist_ms;
  uint64_t units_hist;
  uint64_t hist_tiles_seen;
  uint64_t hist_tiles_one_bucket;
} tq_histogram_stats;
int tq_get_histogram_stats(tq_ctx*, tq_histogram_stats* out);
/* Cumulative since ctx creation: tq_terms_batch.  Device time of k_terms + k_terms_select over all waves, their CTAs (one per unit
 * of up to eight 8192-doc tiles, plus one per (query, segment)), the 8192-doc tiles the units came to and of those the ones counted
 * as one key (every value of the tile equal: the tile's matches added without reading a value).  A struct of its own, so that
 * tq_stats and tq_histogram_stats keep their layouts. */
typedef struct {
  float terms_ms;
  uint64_t units_terms;
  uint64_t terms_tiles_seen;
  uint64_t terms_tiles_one_key;
} tq_terms_stats;
int tq_get_terms_stats(tq_ctx*, tq_terms_stats* out);
/* Cumulative since ctx creation: tq_metrics_batch.  Device time of k_metrics, its CTAs (one per unit of up to eight 8192-doc
 * tiles), the (tile, column) pairs the units came to and of those the ones added as one value (every value of the tile's column
 * equal: its matches added without reading a value).  A struct of its own, so that the other stats keep their layouts. */
typedef struct {
  float metrics_ms;
  uint64_t units_metrics;
  uint64_t metrics_tiles_seen;
  uint64_t metrics_tiles_one_value;
} tq_metrics_stats;
int tq_get_metrics_stats(tq_ctx*, tq_metrics_stats* out);
/* Cumulative since ctx creation: tq_histogram_metrics_batch.  Device time of k_hist_metrics + k_hist_metrics_final over all waves,
 * their CTAs (one per unit of up to eight 8192-doc tiles, plus one per query), the 8192-doc tiles the units came to and of those
 * the ones in one bucket (every value of the tile in one bucket: its metrics accumulated in registers as tq_metrics_batch does),
 * and the (unit, bucket) accumulators flushed from shared memory at a unit's exit versus the runs of one-bucket tiles flushed
 * straight to global memory (units whose window is too wide for shared memory).  A struct of its own, so that the other stats
 * keep their layouts. */
typedef struct {
  float hist_metrics_ms;
  uint64_t units_hist_metrics;
  uint64_t hist_metrics_tiles_seen;
  uint64_t hist_metrics_tiles_one_bucket;
  uint64_t hist_metrics_flush_shared;
  uint64_t hist_metrics_flush_global;
} tq_hist_metrics_stats;
int tq_get_hist_metrics_stats(tq_ctx*, tq_hist_metrics_stats* out);
/* Cumulative since ctx creation: tq_terms_metrics_batch.  Device time of its kernels over all waves (k_terms, k_terms_order,
 * k_terms_select, k_terms_select_metric, k_terms_mark, k_terms_metrics), their CTAs, the 8192-doc tiles k_terms_metrics came to and
 * of those the ones whose docs with a value all hold one kept key (their metrics reduced per warp without a slot lookup), and the
 * waves.  A struct of its own, so that the other stats keep their layouts. */
typedef struct {
  float terms_metrics_ms;
  uint64_t units_terms_metrics;
  uint64_t terms_metrics_tiles_seen;
  uint64_t terms_metrics_tiles_one_key;
  uint64_t terms_metrics_waves;
} tq_terms_metrics_stats;
int tq_get_terms_metrics_stats(tq_ctx*, tq_terms_metrics_stats* out);
/* Cumulative since ctx creation: tq_range_batch, with and without metrics.  Device time of k_range or k_range_metrics over all
 * waves, their CTAs (one per unit of up to eight 8192-doc tiles), the 8192-doc tiles the units came to and of those the ones in one
 * bucket (the tile's smallest and largest image in one range: its matches added without reading a value).  A struct of its own,
 * so that the other stats keep their layouts. */
typedef struct {
  float range_ms;
  uint64_t units_range;
  uint64_t range_tiles_seen;
  uint64_t range_tiles_one_bucket;
} tq_range_stats;
int tq_get_range_stats(tq_ctx*, tq_range_stats* out);
/* Cumulative since ctx creation: tq_terms_histogram_batch.  Device time of its kernels over all waves (k_terms, k_terms_select,
 * k_terms_mark, k_terms_hist, k_terms_hist_final), their CTAs, the 8192-doc tiles k_terms_hist came to, and of those the ones whose
 * docs with a key all hold one kept key (no key gather), the ones whose histogram values are all in bounds and in one bucket (no
 * value gather), and the ones with both (each warp's matches added to one cell), the waves, and the k_terms_hist units that counted
 * in shared memory (their window of kept slots × buckets fits 8192 cells) and in the wave's grid.  A struct of its own, so that the
 * other stats keep their layouts. */
typedef struct {
  float terms_hist_ms;
  uint64_t units_terms_hist;
  uint64_t terms_hist_tiles_seen;
  uint64_t terms_hist_tiles_one_key;
  uint64_t terms_hist_tiles_one_bucket;
  uint64_t terms_hist_tiles_both;
  uint64_t terms_hist_waves;
  uint64_t terms_hist_units_shared;
  uint64_t terms_hist_units_global;
} tq_terms_hist_stats;
int tq_get_terms_hist_stats(tq_ctx*, tq_terms_hist_stats* out);
/* Cumulative since ctx creation: tq_histogram_terms_batch.  Device time of its kernels over all waves (k_hist_terms,
 * k_hist_terms_final), their CTAs, the 8192-doc tiles k_hist_terms came to, and of those the ones whose values all hold one key (no
 * key gather), the ones whose histogram values are all in bounds and in one bucket (no value gather), and the ones with both (each
 * warp's matches added to one cell), the k_hist_terms units that counted in shared memory (their window of buckets × keys fits 8192
 * cells) and in the wave's grid, the (segment, bucket) rows cut on the device, and the waves.  A struct of its own, so that the
 * other stats keep their layouts. */
typedef struct {
  float hist_terms_ms;
  uint64_t units_hist_terms;
  uint64_t hist_terms_tiles_seen;
  uint64_t hist_terms_tiles_one_key;
  uint64_t hist_terms_tiles_one_bucket;
  uint64_t hist_terms_tiles_both;
  uint64_t hist_terms_units_shared;
  uint64_t hist_terms_units_global;
  uint64_t hist_terms_rows_cut;
  uint64_t hist_terms_waves;
} tq_hist_terms_stats;
int tq_get_hist_terms_stats(tq_ctx*, tq_hist_terms_stats* out);

/* Uploads one field of one segment to HBM (copied; caller keeps ownership of its mmap).
 * idx_body    = the field's sub-file of the `.idx` composite, INCLUDING the 8-byte
 *               total_num_tokens header (serializer.rs:128).
 * fieldnorm   = the field's sub-file of `.fieldnorm` (max_doc bytes); NULL => constant
 *               fieldnorm 1 (term_weight.rs:218).
 * alive_bitset= `.del` payload without its 4-byte max_value header: little-endian 64-bit
 *               words, bit set = alive (common/src/bitset.rs:362-407); NULL => no deletes.
 * Every field of one segment ordinal is registered with the same max_doc and the same `.del` bits, as the fields of one
 * tantivy segment share them; a query may name several fields of an ordinal (a clause each), which are then scored together.
 * A query whose clauses name fields of one ordinal that differ in max_doc or doc range (tq_segment_set_doc_range) is refused
 * with TQ_ERR_INVALID_ARGUMENT. */
int tq_segment_register(tq_ctx*, uint32_t segment_ord, uint32_t field, uint32_t max_doc,
                        int record_option, const uint8_t* idx_body, size_t idx_len,
                        const uint8_t* fieldnorm, size_t fieldnorm_len,
                        const uint8_t* alive_bitset, size_t alive_len);
/* The `.pos` sub-file of a registered (segment, field) with record_option TQ_RECORD_FREQS_POSITIONS (copied to HBM):
 * what SegmentReader::inverted_index hands to PositionReader (src/positions/reader.rs:43-55).  Needed by TQ_OP_PHRASE. */
int tq_segment_register_positions(tq_ctx*, uint32_t segment_ord, uint32_t field, const uint8_t* pos_body, size_t pos_len);
/* Frees a (segment, field) and its cached tables; their ids are reused.  Returns TQ_ERR_INVALID_ARGUMENT while a prepared batch
 * that names the segment has not been destroyed (tq_batch_destroy), since that batch still reads the segment's memory. */
int tq_segment_unregister(tq_ctx*, uint32_t segment_ord, uint32_t field);
/* Restricts what THIS context evaluates of a registered (segment, field) to the docs [doc_lo, doc_hi): the intra-segment split of
 * SURVEY.md §8(e) -- one huge segment registered on several contexts / GPUs, each with its own doc range (the posting lists are
 * block-addressable through the skip list, src/postings/skip.rs:205-302, so a doc range is a unit of work like a segment is in
 * Executor::map, src/core/executor.rs:60-100).  Statistics stay the segment's (the caller counts the segment once); the rows of
 * the ranges merge like the rows of segments (merge_fruits).  Call it before the first search on the segment; a range can only be
 * narrowed.  Docs outside the range behave like deleted docs (Count included); the tile engine skips their tiles altogether. */
int tq_segment_set_doc_range(tq_ctx*, uint32_t segment_ord, uint32_t field, uint32_t doc_lo, uint32_t doc_hi);

/* Per-query doc filters (FilterCollector, src/collector/filter_collector_wrapper.rs:160-199; TQ_QUERY_FILTER).  The caller
 * evaluates its predicate over the segment's fast-field column once -- a doc without a value is rejected, a multi-valued doc is
 * accepted if any value passes (:160-169) -- into `bits` in the `.del` layout (little-endian 64-bit words, bit set = keep) and
 * reuses the filter across queries.  One bitset per (filter_id, segment_ord), copied; it applies to every field registered under
 * that ordinal (a doc filter belongs to the segment, not to a field).  At least one field of the ordinal must be registered
 * (else TQ_ERR_NOT_FOUND) and len * 8 >= max_doc (else TQ_ERR_INVALID_ARGUMENT); bits at or beyond max_doc are ignored.
 * Registering a (filter, segment) again replaces its bitset.  The context keeps alive AND doc range AND filter per (filter,
 * segment, field) on the device, built when a query first uses it, and the 1024-doc tiles it leaves non-empty: the tile engine
 * visits only those.  tq_filter_register of a filter, and tq_filter_unregister, return TQ_ERR_INVALID_ARGUMENT while a prepared
 * batch that names the filter has not been destroyed (tq_batch_destroy).  Unregistering the last field of a segment ordinal
 * drops the ordinal's filter bitsets: a reused ordinal never inherits an old filter. */
int tq_filter_register(tq_ctx*, uint32_t filter_id, uint32_t segment_ord, const uint8_t* bits, size_t len);
/* Frees every bitset of the filter; TQ_ERR_NOT_FOUND if none is registered. */
int tq_filter_unregister(tq_ctx*, uint32_t filter_id);

/* Sort columns (TopDocs::order_by_fast_field / order_by_u64_field: SortByStaticFastValue, src/collector/sort_key/
 * sort_by_static_fast_value.rs).  The caller materialises the segment's `Column::first(doc)` once: values[d] = the u64 image of
 * doc d's first value (common/src/lib.rs: u64 as is; i64 and DateTime v ^ 1 << 63; f64 bits ^ 1 << 63 when the sign bit is clear,
 * !bits when it is set; bool 0 / 1), and `present` in the `.del` layout (bit set = doc d has a value; NULL = every doc has one).
 * Both are copied.  The rules are tq_filter_register's: a column belongs to a segment ordinal, not to a field; at least one field of
 * the ordinal must be registered (else TQ_ERR_NOT_FOUND); n_values must equal max_doc and present_len * 8 >= max_doc (else
 * TQ_ERR_INVALID_ARGUMENT); registering a (column, segment) again replaces it; unregistering the last field of a segment ordinal
 * drops the ordinal's columns.  tq_sort_column_register / _unregister of a column return TQ_ERR_INVALID_ARGUMENT while a
 * tq_sort_batch on another thread reads it. */
int tq_sort_column_register(tq_ctx*, uint32_t column_id, uint32_t segment_ord, const uint64_t* values, size_t n_values,
                            const uint8_t* present, size_t present_len);
/* Frees every segment's column of column_id; TQ_ERR_NOT_FOUND if none is registered. */
int tq_sort_column_unregister(tq_ctx*, uint32_t column_id);

#define TQ_ORDER_DESC 0u /* Order::Desc (ComparatorEnum::Natural): larger values first */
#define TQ_ORDER_ASC 1u  /* Order::Asc (ComparatorEnum::ReverseNoneLower): smaller values first */
typedef struct {
  uint32_t column_id; /* as given to tq_sort_column_register */
  uint32_t order;     /* TQ_ORDER_DESC / TQ_ORDER_ASC */
} tq_sort_spec;

/* Histogram aggregations (AggregationCollector with one `histogram` or `date_histogram` and no sub-aggregation, src/aggregation/
 * bucket/histogram/histogram.rs) read the same registered columns.  Only single-valued columns: the reference counts every value
 * of a multi-valued doc, a sort column holds its first, so a multi-valued field stays on the CPU path. */
#define TQ_FAST_U64 0u  /* how a column's u64 image maps to f64 (f64_from_fastfield_u64, aggregation/mod.rs): u64 as f64 */
#define TQ_FAST_I64 1u  /* i64 as f64 */
#define TQ_FAST_F64 2u  /* the f64 itself */
#define TQ_FAST_BOOL 3u /* 0.0 / 1.0 */
#define TQ_FAST_DATE 4u /* i64 nanoseconds as f64 */
typedef struct {
  uint32_t column_id;        /* a column of tq_sort_column_register */
  uint32_t kind;             /* TQ_FAST_* */
  double interval, offset;   /* in the column's unit (DATE: nanoseconds -- the caller normalises the request's milliseconds) */
  double hard_min, hard_max; /* collect-time bounds; -DBL_MAX / DBL_MAX when the request has none */
} tq_histogram_spec;

/* Terms aggregations (AggregationCollector with one `terms` and no sub-aggregation, src/aggregation/bucket/term_agg/mod.rs) read the
 * same registered columns, single-valued only: the key of a doc is its u64 image (for a str column the term ordinal, registered as
 * ords().first(doc)), so key order is the image order, which is the reference's ordinal and value order. */
#define TQ_TERMS_BY_COUNT 0u      /* order target `_count` */
#define TQ_TERMS_BY_KEY 1u        /* order target `_key` */
#define TQ_TERMS_BY_METRIC 2u     /* order target: a metric sub-aggregation (tq_terms_metrics_batch only; tq_terms_batch returns
                                     TQ_ERR_INVALID_ARGUMENT for it, as for any target outside its defines) */
#define TQ_TERMS_MISSING_NONE 0u  /* docs without a value are not counted */
#define TQ_TERMS_MISSING_IMAGE 1u /* ... count under missing_image (a numeric `missing`, as the column's image of it) */
#define TQ_TERMS_MISSING_AFTER_MAX 2u /* ... count under the segment's largest image + 1 (0 + 1 without a value): a str `missing` */
typedef struct {
  uint32_t column_id;     /* a column of tq_sort_column_register */
  uint32_t target;        /* TQ_TERMS_BY_COUNT / TQ_TERMS_BY_KEY */
  uint32_t order;         /* TQ_ORDER_DESC / TQ_ORDER_ASC */
  uint32_t segment_size;  /* entries kept per segment, >= 1: max(size, segment_size), as TermsAggregationInternal::from_req */
  uint32_t missing_mode;  /* TQ_TERMS_MISSING_* */
  uint32_t pad;
  uint64_t missing_image; /* TQ_TERMS_MISSING_IMAGE: the key of a doc without a value */
} tq_terms_spec;

/* Metric aggregations (avg, sum, min, max, stats, value_count: src/aggregation/metric/stats.rs) over the same registered columns,
 * single-valued only.  One spec per query names up to TQ_METRICS_MAX_COLUMNS columns, all fed by one match pass; each collects the
 * value f64_from_fastfield_u64(image) of every doc the query collects that has one, and, with TQ_METRIC_MISSING, that of
 * missing_image for every such doc without one (fetch_block_with_missing).  The column types a metric reads follow
 * agg_data.rs:529-543: value_count reads str, bool and ip columns too, and those collect 0.0 per value (is_number_or_date_type
 * false, stats.rs:372-375): a TQ_METRIC_COUNT_ONLY column, never read.  Every other metric reads numeric and date columns only;
 * on any other column tantivy reads an empty u64 column (get_ff_reader, accessor_helpers.rs:59-74): a TQ_METRIC_EMPTY column,
 * in which no doc has a value and column_id is not looked up. */
#define TQ_METRICS_MAX_COLUMNS 4
#define TQ_METRIC_MISSING 1u    /* docs without a value collect missing_image (f64_to_fastfield_u64 of `missing`, agg_data.rs:568) */
#define TQ_METRIC_COUNT_ONLY 2u /* every collected value is 0.0: only the count is kept */
#define TQ_METRIC_EMPTY 4u      /* no doc has a value (kind TQ_FAST_U64): only TQ_METRIC_MISSING collects anything */
typedef struct {
  uint32_t column_id;     /* a column of tq_sort_column_register (ignored with TQ_METRIC_EMPTY) */
  uint32_t kind;          /* TQ_FAST_*: how an image maps to f64 */
  uint32_t flags;         /* TQ_METRIC_* */
  uint32_t pad;
  uint64_t missing_image; /* TQ_METRIC_MISSING: the image a doc without a value collects */
} tq_metric_column;
typedef struct {
  uint32_t n_columns;  /* 1 .. TQ_METRICS_MAX_COLUMNS; the same column may appear twice */
  uint32_t pad;
  tq_metric_column columns[TQ_METRICS_MAX_COLUMNS];
} tq_metrics_spec;
/* The intermediate result of one (query, column): IntermediateStats, without the order-dependent Kahan state.
 *   count      values collected, NaN and +-inf included (a count-only column: every value)
 *   n_nan      of them NaN; n_inf of them +-inf
 *   min_image / max_image   the smallest / largest image of the non-NaN values (~0 / 0 when there is none; a count-only column
 *              keeps them so): min and max are the values of these images, f64::MAX / f64::MIN when there is none (the reference's
 *              starting values: NaN never lowers min, and +inf never does either since f64::MAX <= +inf).  -0.0 sorts before +0.0.
 *   sum        the f64 sum of the finite values, added in no particular order; magnitude the f64 sum of their |v|
 *   quantum_exp  Q: the least exponent of the lowest set bit over the finite non-zero values (every one is a multiple of 2^Q);
 *              INT32_MAX when there is none
 * Parts of one query (split segments, several contexts) merge field by field: counts add, min_image takes the min, max_image the
 * max, sum and magnitude add, quantum_exp takes the min.
 * The guard: the merged sum is the reference's Kahan sum, bit for bit, when n_nan == n_inf == 0 and magnitude < 2^(53 + Q), or
 * magnitude is finite when 53 + Q > 1023.  Then every partial sum, in any order, is a multiple of 2^Q below 2^(53 + Q) in magnitude,
 * hence exact: Kahan's compensation stays 0 and every order gives the exact sum (DESIGN §3.8).  Otherwise sum, avg and stats take the
 * CPU path; count, min and max are exact always. */
typedef struct {
  uint64_t count, n_nan, n_inf;
  uint64_t min_image, max_image;
  double sum, magnitude;
  int32_t quantum_exp;
  uint32_t pad;
} tq_metric_part;
#ifdef __cplusplus
static_assert(sizeof(tq_metric_column) == 24 && sizeof(tq_metrics_spec) == 104 && sizeof(tq_metric_part) == 64, "metrics ABI layout");
#endif

/* ---- search -------------------------------------------------------------------------- */
/* The whole hot path for a batch of queries, host buffers in / host buffers out:
 * block decode -> AND/OR/term -> BM25 -> per-segment top-k -> merge_fruits.
 * Replaces Searcher::search_with_executor's segment loop + merge (searcher.rs:220-237).
 * Output row q holds out_count[q] <= k hits sorted by (score desc, segment_ord asc, doc asc)
 * (top_score_collector.rs:591-600); rows are out_stride entries apart. */
int tq_search_batch(tq_ctx*, const tq_query* queries, size_t nq, uint32_t out_stride,
                    float* out_scores, uint32_t* out_segment_ord, uint32_t* out_doc,
                    uint32_t* out_count);

/* The Count collector for term / AND / OR / mixed boolean (TQ_OP_BOOL) queries (src/collector/count_collector.rs;
 * Weight::count, term_weight.rs:179-219): out_counts[q] = number of ALIVE docs matching query q over all its segments.
 * k and thresholds of the queries are ignored (TQ_OP_BOOL reads the weights: they order the clauses).  A term query on a
 * segment without deletes is answered from doc_freq, as the reference does -- unless it carries TQ_QUERY_FILTER (Count inside
 * FilterCollector): then only the docs its filter keeps are counted, over the 8192-doc tiles the filter leaves non-empty. */
int tq_count_batch(tq_ctx*, const tq_query* queries, size_t nq, uint64_t* out_counts);

/* TopDocs::with_limit(k).order_by_fast_field(column, order) for term / AND / OR / mixed boolean (TQ_OP_BOOL) queries, synchronous
 * like tq_count_batch: the docs tq_count_batch counts (alive, inside the doc ranges, kept by the query's filter with
 * TQ_QUERY_FILTER), keyed by sorts[q]'s column.  Row q (out_stride >= k entries apart) holds out_count[q] <= k hits: the docs with
 * a value by value (desc or asc), then the docs without one; ties, None docs included, by (segment_ord asc, doc asc) in both orders
 * (compare_for_top_k, top_score_collector.rs:591-600; order.rs:286-293).  out_values[i] = the u64 image of the hit's value (0 for
 * a doc without one), out_present[i] = 1 if it has one.  `and_offset(o)` is k = limit + o and skipping o rows.  out_hits may be
 * NULL; else out_hits[q] = tq_count_batch's answer for query q, (Count, TopDocs::order_by_fast_field), and every tile of the query
 * is visited.  k must be in 1..TQ_MAX_K.  Weights are read where tq_count_batch reads them (TQ_OP_BOOL); thresholds and
 * TQ_QUERY_COUNT_HITS are ignored.  TQ_OP_PHRASE returns TQ_ERR_UNSUPPORTED; a segment the query names without a column for
 * sorts[q].column_id returns TQ_ERR_NOT_FOUND. */
int tq_sort_batch(tq_ctx*, const tq_query* queries, const tq_sort_spec* sorts, size_t nq, uint32_t out_stride, uint64_t* out_values,
                  uint8_t* out_present, uint32_t* out_segment_ord, uint32_t* out_doc, uint32_t* out_count, uint64_t* out_hits);

/* The segment part of a histogram aggregation for term / AND / OR / mixed boolean (TQ_OP_BOOL) queries, synchronous like
 * tq_count_batch, over the docs tq_count_batch counts.  Per (query, segment) the bounds are [hard_min, hard_max], or every finite
 * value when the segment's column already lies inside them (normalize_histogram_req, histogram.rs:672-699).  A doc with a value
 * val (as f64, by specs[q].kind) inside them falls in bucket pos = floor((val - offset) / interval) as i64 (Rust `as`: saturating,
 * NaN -> 0); docs without a value, NaN and, with the default bounds, +-inf are not counted.  Row q (out_stride entries apart)
 * holds the intermediate result of query q over all its segments: its out_n[q] non-empty buckets in ascending pos, out_pos[i] and
 * out_doc_count[i]; the key of a bucket is pos as f64 * interval + offset, and the final result (gap filling, min_doc_count,
 * extended bounds, keys) is the caller's.  When some out_n[q] > out_stride, every out_n is written and the call returns
 * TQ_ERR_INVALID_ARGUMENT: retry with a larger stride.  out_hits may be NULL; else out_hits[q] = tq_count_batch's answer for query
 * q.  The counters of a query span the bucket range of the column's values in the 8192-doc tiles the query visits, clipped to its
 * bounds: a range of more than 2^20 buckets returns TQ_ERR_UNSUPPORTED (the caller takes the CPU path).  TQ_OP_PHRASE returns
 * TQ_ERR_UNSUPPORTED; a segment without the column TQ_ERR_NOT_FOUND; a kind outside TQ_FAST_* or an interval that is not finite and
 * > 0 TQ_ERR_INVALID_ARGUMENT.  k, thresholds and TQ_QUERY_COUNT_HITS are ignored.  The run holds its columns as tq_sort_batch
 * does. */
int tq_histogram_batch(tq_ctx*, const tq_query* queries, const tq_histogram_spec* specs, size_t nq, uint32_t out_stride,
                       int64_t* out_pos, uint64_t* out_doc_count, uint32_t* out_n, uint64_t* out_hits);

/* The segment part of a terms aggregation for term / AND / OR / mixed boolean (TQ_OP_BOOL) queries, synchronous like
 * tq_count_batch, over the docs tq_count_batch counts.  Per (query, segment): each doc's key is its image (a doc without a value
 * counts under the missing key of specs[q].missing_mode, or not at all); the entries are the keys with a non-zero count, u32 counts
 * as the reference's Bucket::count.  When there are more than segment_size, segment_size are kept by the order (count or key, desc
 * or asc), ties at the cut by key ascending (the reference's select_nth_unstable leaves them unspecified), and the segment reports
 * the count of the entry at position segment_size in that order (term_doc_count_before_cutoff) and the sum of the counts cut
 * (sum_other_doc_count) -- into_intermediate_bucket_result / cut_off_buckets, term_agg/mod.rs:1000-1111, 1328-1353.  Row q
 * (out_stride entries apart) holds query q's kept entries over all its segments, ascending by (segment_ord, key): out_segment_ord[i],
 * out_key[i] (the image) and out_doc_count[i]; out_sum_other[q] and out_error_bound[q] are the sums of the two scalars over its
 * segments.  A segment this context evaluates only part of (tq_segment_set_doc_range narrowed it) is not cut: its entries are all in
 * the row and it adds 0 to both scalars, so that the caller can sum the ranges of the segment and cut once, as the reference cuts
 * each segment once.  Mapping keys to terms or values, the merge and the final result (min_doc_count, order, size) are the caller's.  When
 * some out_n[q] > out_stride, every out_n is written and the call returns TQ_ERR_INVALID_ARGUMENT: retry with a larger stride.
 * out_hits may be NULL; else out_hits[q] = tq_count_batch's answer for query q.  A (query, segment)'s counters span the images of
 * the 8192-doc tiles the query visits there: more than 2^20 keys returns TQ_ERR_UNSUPPORTED naming the query (the caller takes the
 * CPU path).  Queries whose counters exceed the ctx's budget (TQ_TERMS_COUNTER_BUDGET at ctx creation, in counters) run in
 * consecutive waves on one scratch region.  TQ_OP_PHRASE returns TQ_ERR_UNSUPPORTED; a segment without the column
 * TQ_ERR_NOT_FOUND; a target, order or missing mode outside its defines, segment_size 0, or TQ_TERMS_MISSING_AFTER_MAX on a
 * segment whose largest image is 2^64 - 1 TQ_ERR_INVALID_ARGUMENT.  k, thresholds and TQ_QUERY_COUNT_HITS are ignored.  The run
 * holds its columns as tq_sort_batch does. */
int tq_terms_batch(tq_ctx*, const tq_query* queries, const tq_terms_spec* specs, size_t nq, uint32_t out_stride,
                   uint32_t* out_segment_ord, uint64_t* out_key, uint64_t* out_doc_count, uint32_t* out_n, uint64_t* out_sum_other,
                   uint64_t* out_error_bound, uint64_t* out_hits);

/* The intermediate metric results of term / AND / OR / mixed boolean (TQ_OP_BOOL) queries, synchronous like tq_count_batch, over
 * the docs tq_count_batch counts: out[q * TQ_METRICS_MAX_COLUMNS + i] is query q's tq_metric_part of specs[q].columns[i] over all
 * its segments (parts past n_columns are written empty: count 0, images ~0 / 0, sums 0, quantum_exp INT32_MAX).  out_hits may be
 * NULL; else out_hits[q] = tq_count_batch's answer for query q.  Applying the guard, merging parts of other contexts and the final
 * values are the caller's.  TQ_OP_PHRASE returns TQ_ERR_UNSUPPORTED; a segment without a column TQ_ERR_NOT_FOUND; n_columns outside
 * 1 .. TQ_METRICS_MAX_COLUMNS, a kind outside TQ_FAST_* or a flag outside TQ_METRIC_* TQ_ERR_INVALID_ARGUMENT.  k, thresholds and
 * TQ_QUERY_COUNT_HITS are ignored.  The run holds its columns as tq_sort_batch does. */
int tq_metrics_batch(tq_ctx*, const tq_query* queries, const tq_metrics_spec* specs, size_t nq, tq_metric_part* out, uint64_t* out_hits);

/* A histogram with metric sub-aggregations (one `histogram` / `date_histogram` whose `aggs` are avg, sum, min, max, stats and
 * value_count: SegmentHistogramCollector::collect pushing each counted doc to its bucket's sub-aggregation, histogram.rs:490-505),
 * synchronous like tq_count_batch, over the docs tq_count_batch counts.  hspecs[q] is query q's histogram exactly as in
 * tq_histogram_batch, mspecs[q] its metric columns exactly as in tq_metrics_batch; the docs a bucket's metrics collect are the docs
 * the histogram counts in it (a doc without a histogram value, or with one outside the bounds, feeds no metric).  Row q (out_stride
 * buckets apart) holds query q's out_n[q] non-empty buckets over all its segments in ascending pos: out_pos[i] and out_doc_count[i]
 * as tq_histogram_batch writes them, and out_parts[i * TQ_METRICS_MAX_COLUMNS + c] the bucket's tq_metric_part of column c (parts
 * past n_columns are written empty), with tq_metrics_batch's merge rules and guard, applied per (bucket, column) by the caller.
 * When some out_n[q] > out_stride, every out_n is written and the call returns TQ_ERR_INVALID_ARGUMENT: retry with a larger
 * stride.  out_hits may be NULL; else out_hits[q] = tq_count_batch's answer for query q.  A query's accumulators span its bucket
 * range as in tq_histogram_batch, one tq_metric_part per (bucket, column): a range of more than 2^16 buckets returns
 * TQ_ERR_UNSUPPORTED naming the query (the caller takes the CPU path).  Queries whose accumulators exceed the ctx's budget
 * (TQ_HIST_METRICS_BUDGET at ctx creation, in (bucket, column) accumulators) run in consecutive waves on one scratch region.  The
 * errors are those of tq_histogram_batch and tq_metrics_batch: TQ_OP_PHRASE returns TQ_ERR_UNSUPPORTED, a segment without a column
 * TQ_ERR_NOT_FOUND, a bad histogram kind or interval, metric kind, flag or column count TQ_ERR_INVALID_ARGUMENT.  k, thresholds
 * and TQ_QUERY_COUNT_HITS are ignored.  The run holds its columns as tq_sort_batch does. */
int tq_histogram_metrics_batch(tq_ctx*, const tq_query* queries, const tq_histogram_spec* hspecs, const tq_metrics_spec* mspecs, size_t nq,
                               uint32_t out_stride, int64_t* out_pos, uint64_t* out_doc_count, tq_metric_part* out_parts, uint32_t* out_n,
                               uint64_t* out_hits);

/* A terms aggregation with metric sub-aggregations (one `terms` whose `aggs` are avg, sum, min, max, stats and value_count:
 * collect_terms_with_docs pushing every doc the terms count to its term's sub-aggregation, term_agg/mod.rs), synchronous like
 * tq_count_batch, over the docs tq_count_batch counts.  tspecs[q] is query q's terms exactly as in tq_terms_batch, except that its
 * target may also be TQ_TERMS_BY_METRIC; mspecs[q] its metric columns exactly as in tq_metrics_batch.  The docs a term's metrics
 * collect are the docs the terms count under its key, the missing key's included.
 *   Order.  TQ_TERMS_BY_COUNT / TQ_TERMS_BY_KEY cut each segment exactly as tq_terms_batch does.  TQ_TERMS_BY_METRIC reads
 *   orders[q]: the per-segment value of metric orders[q].metric of spec column orders[q].column (compute_metric_value(...)
 *   .unwrap_or(0.0): count as f64; the sum, 0 without values; sum / count, min, max, 0 without values; f64::MAX / f64::MIN for a min
 *   / max of NaN values only), compared as partial_cmp does (-0.0 equals +0.0).  Equal values at the cut keep the lowest keys, and
 *   the two scalars follow that order: term_doc_count_before_cutoff is the doc count of the entry at position segment_size and
 *   sum_other_doc_count the sum of the cut entries' doc counts (the reference's select_nth_unstable_by leaves ties unspecified).
 *   out_order_part[q] is then the ordering column's tq_metric_part over every doc query q's terms collect, cut entries included,
 *   over all its segments: the caller's guard on it decides whether the cut was exact (written empty for the other orders).
 *   Rows.  Row q (out_stride entries apart) holds query q's kept entries over all its segments, ascending by (segment_ord, key), as
 *   tq_terms_batch writes them, and out_parts[i * TQ_METRICS_MAX_COLUMNS + c] the entry's tq_metric_part of column c (parts past
 *   n_columns are written empty); out_sum_other / out_error_bound as in tq_terms_batch.  A segment this context evaluates only part
 *   of is not cut, as in tq_terms_batch.  When some out_n[q] > out_stride, every out_n is written and the call returns
 *   TQ_ERR_INVALID_ARGUMENT: retry with a larger stride.  out_hits may be NULL; else out_hits[q] = tq_count_batch's answer.
 *   Limits.  A (query, segment) whose keys span more than 2^20 returns TQ_ERR_UNSUPPORTED naming the query, as does one whose
 *   kept entries' parts alone exceed the ctx's metrics budget.  Queries run in waves whose counters fit TQ_TERMS_COUNTER_BUDGET and
 *   whose (kept entry, column) parts fit TQ_TERMS_METRICS_BUDGET (at ctx creation).
 *   Errors.  Those of tq_terms_batch and tq_metrics_batch, and TQ_ERR_INVALID_ARGUMENT for TQ_TERMS_BY_METRIC with orders NULL, an
 *   order column >= n_columns or an order metric outside TQ_TERMS_ORDER_*.  k, thresholds and TQ_QUERY_COUNT_HITS are ignored.  The
 *   run holds its columns as tq_sort_batch does. */
#define TQ_TERMS_ORDER_COUNT 0u /* value_count, stats.count */
#define TQ_TERMS_ORDER_SUM 1u   /* sum, stats.sum */
#define TQ_TERMS_ORDER_AVG 2u   /* avg, stats.avg */
#define TQ_TERMS_ORDER_MIN 3u   /* min, stats.min */
#define TQ_TERMS_ORDER_MAX 4u   /* max, stats.max */
typedef struct {
  uint32_t column;  /* index into the query's tq_metrics_spec columns */
  uint32_t metric;  /* TQ_TERMS_ORDER_* */
} tq_terms_metric_order;
#ifdef __cplusplus
static_assert(sizeof(tq_terms_metric_order) == 8, "terms metric order ABI layout");
#endif
int tq_terms_metrics_batch(tq_ctx*, const tq_query* queries, const tq_terms_spec* tspecs, const tq_metrics_spec* mspecs,
                           const tq_terms_metric_order* orders, size_t nq, uint32_t out_stride, uint32_t* out_segment_ord,
                           uint64_t* out_key, uint64_t* out_doc_count, tq_metric_part* out_parts, uint32_t* out_n,
                           uint64_t* out_sum_other, uint64_t* out_error_bound, tq_metric_part* out_order_part, uint64_t* out_hits);

/* A range aggregation (`range`, bucket/range.rs), with or without metric sub-aggregations, synchronous like tq_count_batch, over
 * the docs tq_count_batch counts.  rspecs[q] is query q's buckets in image space, as extend_validate_ranges leaves them: starts
 * strictly ascending from 0, bucket b holding the images in [starts[b], starts[b + 1]) and the last one every image from its start
 * up (get_bucket_pos: the end is never tested).  A doc without a value is not collected.  Row q (out_stride buckets apart) holds
 * every bucket of query q, empty ones included, in start order: out_doc_count[q * out_stride + b] over all its segments and, with
 * mspecs (exactly as in tq_metrics_batch), out_parts[(q * out_stride + b) * TQ_METRICS_MAX_COLUMNS + c] the bucket's tq_metric_part
 * of column c (parts past n_columns are written empty), with tq_metrics_batch's merge rules and guard, applied per (bucket, column)
 * by the caller.  mspecs NULL: doc counts only, and out_parts must be NULL.  out_hits may be NULL; else out_hits[q] =
 * tq_count_batch's answer for query q.  With mspecs, queries whose accumulators exceed the ctx's TQ_HIST_METRICS_BUDGET (in
 * (bucket, column) accumulators) run in consecutive waves.  TQ_OP_PHRASE returns TQ_ERR_UNSUPPORTED, a segment without a column
 * TQ_ERR_NOT_FOUND; out_stride below some n_buckets, n_buckets outside 1 .. TQ_RANGE_MAX_BUCKETS, starts not strictly ascending
 * or starts[0] != 0, out_parts NULL with mspecs (or not NULL without) and the metrics spec errors of tq_metrics_batch
 * TQ_ERR_INVALID_ARGUMENT.  k, thresholds and TQ_QUERY_COUNT_HITS are ignored.  The run holds its columns as tq_sort_batch does. */
#define TQ_RANGE_MAX_BUCKETS 128u
typedef struct {
  uint32_t column_id;                     /* a column of tq_sort_column_register */
  uint32_t n_buckets;                     /* 1 .. TQ_RANGE_MAX_BUCKETS, after extension */
  uint64_t starts[TQ_RANGE_MAX_BUCKETS];  /* strictly ascending images, starts[0] == 0 */
} tq_range_spec;
#ifdef __cplusplus
static_assert(sizeof(tq_range_spec) == 1032, "range ABI layout");
#endif
int tq_range_batch(tq_ctx*, const tq_query* queries, const tq_range_spec* rspecs, const tq_metrics_spec* mspecs, size_t nq,
                   uint32_t out_stride, uint64_t* out_doc_count, tq_metric_part* out_parts, uint64_t* out_hits);

/* A terms aggregation whose only sub-aggregation is a histogram / date_histogram (one `terms` over one `histogram`, the fused
 * collector of term_histogram.rs), synchronous like tq_count_batch, over the docs tq_count_batch counts.  tspecs[q] is query q's
 * terms exactly as in tq_terms_batch (TQ_TERMS_BY_METRIC is TQ_ERR_INVALID_ARGUMENT), hspecs[q] its histogram exactly as in
 * tq_histogram_batch.  Every doc the terms count under a key, the missing key's included, feeds that key's histogram: it counts in
 * bucket pos when it has a histogram value inside the (query, segment)'s bounds, as tq_histogram_batch counts.
 *   Rows.  Row q (out_stride entries apart) holds query q's kept entries over all its segments, ascending by (segment_ord, key), with
 *   the doc counts, out_sum_other and out_error_bound exactly as tq_terms_batch writes them (a segment this context evaluates only
 *   part of is not cut).  The cells of all queries follow one another in one array, query by query and entry by entry in row order:
 *   entry i's non-empty buckets are cells out_cell_first[i] .. + out_cell_n[i] (absolute indices), out_cell_pos (i64) and
 *   out_cell_count in ascending pos, and out_cells[q] counts query q's.  When some out_n[q] > out_stride or the cells of all
 *   queries exceed cell_capacity, every out_n and out_cells is written and the call returns TQ_ERR_INVALID_ARGUMENT: retry with a
 *   larger stride or capacity.  out_hits may be NULL; else out_hits[q] = tq_count_batch's answer.
 *   Limits.  Those of tq_terms_batch and tq_histogram_batch (2^20 keys in a segment, 2^20 buckets in a query), and a (query,
 *   segment) whose grid -- kept entries (every entry of a partial segment) times its bucket span -- exceeds the ctx's cell budget
 *   (TQ_TERMS_HIST_BUDGET at ctx creation, in u32 cells, at most 2^28) returns TQ_ERR_UNSUPPORTED naming the query.  Queries run
 *   in waves whose counters fit TQ_TERMS_COUNTER_BUDGET and whose grids fit TQ_TERMS_HIST_BUDGET.
 *   Errors.  Those of tq_terms_batch and tq_histogram_batch.  k, thresholds and TQ_QUERY_COUNT_HITS are ignored.  The run holds its
 *   columns as tq_sort_batch does. */
int tq_terms_histogram_batch(tq_ctx*, const tq_query* queries, const tq_terms_spec* tspecs, const tq_histogram_spec* hspecs, size_t nq,
                             uint32_t out_stride, uint32_t* out_segment_ord, uint64_t* out_key, uint64_t* out_doc_count, uint32_t* out_n,
                             uint64_t* out_sum_other, uint64_t* out_error_bound, uint64_t cell_capacity, uint64_t* out_cell_first,
                             uint32_t* out_cell_n, int64_t* out_cell_pos, uint64_t* out_cell_count, uint32_t* out_cells, uint64_t* out_hits);

/* A histogram / date_histogram whose only sub-aggregation is a terms (one `histogram` over one `terms`: the sub-aggregation branch
 * of SegmentHistogramCollector::collect, one HashMapTermBuckets per bucket), synchronous like tq_count_batch, over the docs
 * tq_count_batch counts.  hspecs[q] is query q's histogram exactly as in tq_histogram_batch, tspecs[q] its terms exactly as in
 * tq_terms_batch (TQ_TERMS_BY_METRIC is TQ_ERR_INVALID_ARGUMENT).  Every doc the histogram counts in bucket pos -- it has a histogram
 * value inside the (query, segment)'s bounds -- feeds that bucket's terms: under its image, under the missing key, or (without a
 * value and without a missing key) under none.  Each (segment, bucket) is cut to segment_size on its own as tq_terms_batch cuts a
 * segment (a segment this context evaluates only part of is not cut).
 *   Rows.  Row q (out_stride buckets apart) holds query q's non-empty buckets in ascending pos: out_pos (i64) and out_doc_count as
 *   tq_histogram_batch writes them, out_sum_other and out_error_bound summed over the segments, and its kept entries
 *   out_entry_first (an absolute index) .. + out_entry_n.  The entries of all queries follow one another in one array, query by query
 *   and bucket by bucket in row order, each bucket's by (segment_ord, image): out_entry_segment_ord, out_entry_key (the image) and
 *   out_entry_count; out_entries[q] counts query q's.  When some out_n[q] > out_stride or the entries of all queries exceed
 *   entry_capacity, every out_n and out_entries is written and the call returns TQ_ERR_INVALID_ARGUMENT: retry with a larger stride
 *   or capacity.  out_hits may be NULL; else out_hits[q] = tq_count_batch's answer.
 *   Limits.  Those of tq_terms_batch and tq_histogram_batch (2^20 keys in a segment, 2^20 buckets in a query), and a (query,
 *   segment) whose grid -- its bucket span times (its key span + 1) -- exceeds the ctx's cell budget (TQ_HIST_TERMS_BUDGET at ctx
 *   creation, in u32 cells, default 2^24, at most 2^28) returns TQ_ERR_UNSUPPORTED naming the query.  Queries run in waves whose
 *   grids fit that budget.
 *   Errors.  Those of tq_histogram_batch and tq_terms_batch.  k, thresholds and TQ_QUERY_COUNT_HITS are ignored.  The run holds its
 *   columns as tq_sort_batch does. */
int tq_histogram_terms_batch(tq_ctx*, const tq_query* queries, const tq_histogram_spec* hspecs, const tq_terms_spec* tspecs, size_t nq,
                             uint32_t out_stride, int64_t* out_pos, uint64_t* out_doc_count, uint64_t* out_sum_other, uint64_t* out_error_bound,
                             uint64_t* out_entry_first, uint32_t* out_entry_n, uint32_t* out_n, uint64_t entry_capacity,
                             uint32_t* out_entry_segment_ord, uint64_t* out_entry_key, uint64_t* out_entry_count, uint32_t* out_entries,
                             uint64_t* out_hits);

/* The same split in three so that callers can keep inputs/outputs device resident:
 * prepare = host planning + H2D of descriptors + block-table builds (cached per term),
 * run     = scoring kernels + final top-k, results stay in HBM,
 * fetch   = D2H of the result rows. */
int tq_batch_prepare(tq_ctx*, const tq_query* queries, size_t nq, tq_batch** out);
int tq_batch_run(tq_batch*);
/* The run in tq_batch_phases() consecutive phases, for callers that shard an index over several GPUs/processes:
 * phase 0 = everything up to the unions' first threshold round (each query then holds the exact k-th best score over
 * the windows scored so far), the middle phases = the further threshold rounds, the last phase = the rest.  Between
 * two phases tq_batch_thresholds_export_dev writes the nq score keys (order-preserving u32 image of the f32 score,
 * zero-extended to int64; 0 = no bound yet) to a DEVICE array; the caller takes the element-wise MAX over all shards
 * (e.g. ncclAllReduce) and hands it back with tq_batch_thresholds_import_dev.  Every shard then prunes against the best
 * bound any shard found: a valid lower bound of the global k-th score (SURVEY.md §8e "broadcast the running global
 * threshold").  tq_batch_run == all phases in order.
 * A run is in progress from its first phase until its last one has been enqueued.  Meanwhile tq_batch_run finishes it (it
 * starts at the next phase of the run), tq_batch_run_phase with any other phase returns TQ_ERR_INVALID_ARGUMENT and keeps the
 * run where it was, and every result entry point (tq_batch_fetch, tq_batch_fetch_hits, tq_batch_results_dev,
 * tq_batch_results_copy_dev, tq_batch_results_pack_dev, tq_batch_results_pack_dev_async) returns TQ_ERR_INVALID_ARGUMENT and
 * changes nothing: the rows of an earlier run are no longer the batch's answer, and this run's are not there yet. */
int tq_batch_phases(tq_batch*);
int tq_batch_run_phase(tq_batch*, int phase);
int tq_batch_thresholds_export_dev(tq_batch*, int64_t* keys_dev);
int tq_batch_thresholds_import_dev(tq_batch*, const int64_t* keys_dev);
/* The exact form of that exchange (what one GPU holding all segments computes): between two phases every shard exports,
 * per query, the k best score keys it holds so far (u32 order-preserving images of f32 scores, k_stride entries per
 * query, zero padded) -- enqueued on the batch's stream, no host synchronisation; the caller all-gathers the arrays of
 * all shards ON THAT STREAM (tq_batch_stream; e.g. ncclAllGather, or torch.cuda.ExternalStream) into
 * [n_shards][nq][k_stride] and hands them back: the k-th best key of the union becomes every shard's threshold
 * (merge_top_k's bound, sort_key_top_collector.rs:76-95, available before the scoring is over). */
int tq_batch_stream(tq_batch*, void** cuda_stream_out);
int tq_batch_topkeys_export_dev(tq_batch*, uint32_t* keys_dev, uint32_t k_stride);
int tq_batch_thresholds_from_keys_dev(tq_batch*, const uint32_t* gathered_keys_dev, uint32_t n_shards, uint32_t k_stride);
int tq_batch_fetch(tq_batch*, uint32_t out_stride, float* out_scores, uint32_t* out_segment_ord,
                   uint32_t* out_doc, uint32_t* out_count);
/* The Count half of (Count, TopDocs): out_hits[q] (nq entries) = tq_count_batch's answer for query q on this context (alive
 * docs, doc ranges applied) when q carries TQ_QUERY_COUNT_HITS, else 0.  Call it after a finished run (tq_batch_run or the last
 * phase); like tq_batch_fetch it resolves an overflowed run first.  Every run counts from zero.  The tile engine counts from the
 * postings the run has already decoded; queries on the per-query kernels are counted by the Count kernels in the same run. */
int tq_batch_fetch_hits(tq_batch*, uint64_t* out_hits);
/* Device pointers of the result rows of a finished run (none in progress, see tq_batch_phases): row stride = k_max of the batch. */
int tq_batch_results_dev(tq_batch*, const float** scores_dev, const uint32_t** segment_ord_dev,
                         const uint32_t** doc_dev, const uint32_t** count_dev, uint32_t* stride);
/* Copies the result rows of a finished run into caller-owned DEVICE buffers (row stride = k_max of
 * the batch), e.g. torch tensors about to be all-gathered over NCCL. */
int tq_batch_results_copy_dev(tq_batch*, float* scores_dev, uint32_t* segment_ord_dev, uint32_t* doc_dev,
                              uint32_t* count_dev);
/* Allowed at any point, also between two phases of a run: it waits for all work of the batch on both of its streams before its
 * segments, filters, columns and buffers are let go. */
void tq_batch_destroy(tq_batch*);

/* Cross-GPU merge_fruits (sort_key_top_collector.rs:76-95): merges `n_lists` result sets
 * (e.g. the ranks' rows after an NCCL all-gather), all device resident, laid out
 * [list][query][stride], into [query][stride] device rows; same ordering as above. */
int tq_merge_topk_dev(tq_ctx*, uint32_t n_lists, uint32_t nq, uint32_t stride, uint32_t k,
                      const float* scores_dev, const uint32_t* segment_ord_dev,
                      const uint32_t* doc_dev, const uint32_t* count_dev, float* out_scores_dev,
                      uint32_t* out_segment_ord_dev, uint32_t* out_doc_dev,
                      uint32_t* out_count_dev);

/* The same for sharded callers that move ONE buffer per shard: packed = [nq*stride scores | nq*stride segment ords |
 * nq*stride docs | nq counts] as 32-bit words (tq_batch_results_pack_dev writes it with stride = k_max of the batch),
 * n_lists of them pitch_words apart -- what one all-gather of the shards' buffers produces.  The merge is enqueued on
 * cuda_stream (a cudaStream_t, e.g. tq_batch_stream's) and does not synchronise with the host. */
int tq_batch_results_pack_dev(tq_batch*, uint32_t* packed_dev);
/* tq_batch_results_pack_dev without the wait: the copies are enqueued behind the run on the batch's stream, so that pack, all-gather,
 * merge and the NEXT batch's run can all be queued before the host waits for this batch (two batches in flight per GPU).
 * packed_dev holds 3 * nq * k_max + nq + 4 words; the last four are the run's overflow flags -- non-zero on any shard: take
 * tq_batch_results_pack_dev instead (it repeats an overflowed run: TQ_OP_BOOL queries on the tile engine with capacities that hold them, the rest on the per-query kernels). */
int tq_batch_results_pack_dev_async(tq_batch*, uint32_t* packed_dev);
int tq_merge_topk_packed_dev(tq_ctx*, void* cuda_stream, uint32_t n_lists, uint32_t nq, uint32_t stride, uint32_t k,
                             const uint32_t* packed_dev, size_t pitch_words, uint32_t* out_packed_dev);

/* ---- several GPUs behind one handle --------------------------------------------------- */
/* The reference fans a search out over segments inside ONE process (Executor::map, src/core/executor.rs:60-100;
 * Searcher::search_with_executor, src/core/searcher.rs:220-237).  tq_multi is that shape for GPUs: one tq_ctx per
 * device, every (segment, field) lives on one of them (device_index -1 = the least loaded), tq_multi_search_batch runs
 * the devices' shares concurrently (one host thread per device), exchanges the exact k-th best score keys between the
 * phases -- every device prunes like a single device holding all segments -- and merges the rows on the host
 * (merge_fruits, sort_key_top_collector.rs:54-95).  Same arguments and result layout as tq_search_batch.
 * Every field of a segment ordinal lives on the same device(s), so that a query's clauses on the ordinal are scored together:
 * a further field of an ordinal goes where the first one went, whole or split.  Registering it with another device_index, with
 * another max_doc, or whole after split (or split after whole) fails with TQ_ERR_INVALID_ARGUMENT. */
typedef struct tq_multi tq_multi;
int tq_multi_create(const int* devices, int n_devices, tq_multi** out);
void tq_multi_destroy(tq_multi*);
const char* tq_multi_last_error(tq_multi*);
int tq_multi_num_devices(tq_multi*);
int tq_multi_segment_register(tq_multi*, int device_index, uint32_t segment_ord, uint32_t field, uint32_t max_doc,
                              int record_option, const uint8_t* idx_body, size_t idx_len,
                              const uint8_t* fieldnorm, size_t fieldnorm_len,
                              const uint8_t* alive_bitset, size_t alive_len);
/* One (huge) segment over ALL devices of the handle: every device holds the segment's bytes and evaluates its own doc range
 * (tq_segment_set_doc_range; ranges are whole 1024-doc tiles, ceil(max_doc / n_devices) docs each). */
int tq_multi_segment_register_split(tq_multi*, uint32_t segment_ord, uint32_t field, uint32_t max_doc,
                                    int record_option, const uint8_t* idx_body, size_t idx_len,
                                    const uint8_t* fieldnorm, size_t fieldnorm_len,
                                    const uint8_t* alive_bitset, size_t alive_len);
int tq_multi_search_batch(tq_multi*, const tq_query* queries, size_t nq, uint32_t out_stride,
                          float* out_scores, uint32_t* out_segment_ord, uint32_t* out_doc,
                          uint32_t* out_count);
/* tq_filter_register on every device that holds a field of segment_ord (all of them for a split segment: each device's doc range
 * does the rest); TQ_ERR_NOT_FOUND if none does.  Refused on all devices if a prepared batch on any of them names the filter. */
int tq_multi_filter_register(tq_multi*, uint32_t filter_id, uint32_t segment_ord, const uint8_t* bits, size_t len);
/* tq_filter_unregister on every device that has the filter; TQ_ERR_NOT_FOUND if none has it. */
int tq_multi_filter_unregister(tq_multi*, uint32_t filter_id);

/* ---- codec-level access (parity tests and the decode micro-benchmark) ----------------- */
/* Decodes one whole posting list on the device (BlockSegmentPostings::open + advance loop,
 * block_segment_postings.rs:97-140,343-399) into host arrays of doc_freq entries.
 * out_tfs may be NULL. */
int tq_decode_postings(tq_ctx*, const tq_term_seg* list, uint32_t* out_docs, uint32_t* out_tfs);
/* Block-max scores of every full block (SkipReader::block_max_score, skip.rs:175-184) and
 * last_doc_in_block, as the device block table holds them. n = doc_freq / 128 entries. */
int tq_block_table(tq_ctx*, const tq_term_seg* list, float weight, float avg_fieldnorm,
                   uint32_t* out_last_doc, float* out_block_max);

/* ---- BM25 scalars (host; bit-identical to src/query/bm25.rs) -------------------------- */
float tq_bm25_idf(uint64_t doc_freq, uint64_t doc_count);                  /* bm25.rs:52-56 */
float tq_bm25_weight(uint64_t doc_freq, uint64_t doc_count, float boost);  /* bm25.rs:141-151,80-92 */
void tq_bm25_tf_cache(float avg_fieldnorm, float out[256]);               /* bm25.rs:58-69 */
uint32_t tq_id_to_fieldnorm(uint8_t id);                                   /* fieldnorm/code.rs:2-4 */
uint8_t tq_fieldnorm_to_id(uint32_t fieldnorm);                            /* fieldnorm/code.rs:7-11 */

/* ---- segment writer (host; produces tantivy-format bytes for tests and benchmarks) ----- */
/* Restates PostingsSerializer (src/postings/serializer.rs:353-481): appends one term's
 * posting list (docs ascending, tfs >= 1 or NULL) to `body`, returns TermInfo. */
typedef struct tq_field_writer tq_field_writer;
int tq_field_writer_create(int record_option, uint64_t total_num_tokens,
                           const uint8_t* fieldnorm_ids, uint32_t max_doc, tq_field_writer** out);
int tq_field_writer_add_term(tq_field_writer*, const uint32_t* docs, const uint32_t* tfs,
                             uint32_t doc_freq, uint64_t* postings_start, uint64_t* postings_end);
/* Field body = 8-byte LE total_num_tokens followed by every term's postings. */
int tq_field_writer_body(tq_field_writer*, const uint8_t** body, size_t* len);
void tq_field_writer_destroy(tq_field_writer*);

#ifdef __cplusplus
}
#endif
#endif /* TANTIVY_B200_H */
