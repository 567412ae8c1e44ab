// The host-device contract: every struct the host stages for the kernels (descriptors copied with one cudaMemcpyAsync, kernel
// parameters), the capacities the planner sizes them by, and the shared-memory size of each kernel that takes a dynamic amount.
// Host-only translation units include this header without the kernels (plain C++17 plus the CUDA include path); the kernel
// headers include it instead of defining these themselves.  No kernel and no device-only function lives here.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <math.h>
#include <string.h>

#include "../../include/tantivy_b200.h"  // TQ_FAST_*
#include "bm25_host.hpp"  // TQ_HD

namespace tq {

constexpr int kThreads = 256;                 // 8 warps per CTA
constexpr int kWarps = kThreads / 32;
constexpr uint32_t kTileDocs = 8192;          // OR: doc-id tile width held in shared memory
constexpr uint32_t kTfRows = 17;              // term frequencies below this use the precomputed factor table (tf_bits <= 4 => tf <= 16)

// ---- per-query kernels (tq_device.cuh, tq_kernels.cuh) ------------------------------------------------------------------

// One posting list of one (segment, field, term), device resident.  Built once per term by
// k_build_tables from the raw tantivy bytes and cached for the life of the segment (segments
// are immutable, ARCHITECTURE.md "Searcher").
struct ListDesc {
  const uint8_t* blocks;      // the list's bit-packed blocks, copied 16-byte aligned when the table is built
                              // (posting lists start at arbitrary byte offsets inside the .idx body)
  const uint32_t* last_doc;   // [n_total] last doc id of every block; entry n_blocks = last tail doc
  const uint2* blk;           // [n_blocks + 1] .x byte offset from `blocks`, .y packed meta
  const uint4* tab4;          // [n_total] {last_doc, byte offset, meta, last doc of the previous block (0xFFFFFFFF: none)}
                              // one 16-byte record per block so that a 32-wide probe yields position AND record
  const uint32_t* tail_docs;  // [tail_n] the VInt tail, decoded at build time
  const uint32_t* tail_tfs;   // [tail_n]
  const uint8_t* fieldnorm;   // the segment's fieldnorm ids for this field; null => constant id 1
  uint32_t n_blocks;          // full 128-doc blocks
  uint32_t tail_n;            // docs in the VInt tail (0..127)
  uint32_t n_total;           // n_blocks + (tail_n ? 1 : 0)
  uint32_t doc_freq;
  uint32_t has_freq;          // term frequencies are stored (else tf = 1)
  uint32_t build_status;      // 0 ok, else corrupt
};
// meta bits: [0:5) doc_bits, bit 6 strict-delta, [8:14) tf_bits, [16:24) block-max fieldnorm id,
// [24:32) block-max tf code (255 = saturated), see src/postings/skip.rs:16-22,205-253.

struct BuildJob {
  const uint8_t* bytes;  // the term's postings range
  uint32_t len;
  uint32_t doc_freq;
  uint32_t record_option;  // 0/1/2; bit 8: ignore term frequencies (score with tf = 1)
  uint32_t list_id;
};

struct QList {  // one clause of one query in one segment
  uint32_t list_id;
  float weight;        // Bm25Weight.weight
  uint32_t cache_idx;  // which 256-entry tf-norm table
  uint32_t pad;
};
struct QSeg {  // one (query, segment): what Collector::collect_segment sees
  uint32_t query;
  uint32_t lists_base;  // index into qlists; AND: ascending doc_freq (leader first); OR/TERM: clause order
  uint32_t n_lists;
  uint32_t max_doc;
  uint32_t segment_ord;
  uint32_t flags;        // bit 0: every clause reads the same fieldnorm array (`fieldnorm` below); bit 1: prunable (every
                         // weight finite and >= 0); bit 2: AND in Intersection::score order, (s0 + s1) + (s2 + s3 + ...)
  const uint8_t* alive;  // alive bitset bytes or null
  const uint8_t* fieldnorm;  // shared fieldnorm ids (padded to a multiple of kTileDocs) when flags&1
};
struct Unit {  // one CTA's share of a QSeg
  uint32_t qseg;
  uint32_t begin, end;  // TERM/AND: block range of the (leader) list; OR: tile range
  uint32_t pad;
};
struct DQuery {
  uint32_t k;
  uint32_t cand_base;  // first slot of this query's candidate region
  uint32_t cand_cap;
  uint32_t op;
};
struct QState {  // zeroed before every run
  unsigned int theta;       // score key: lower bound of the final k-th best score
  unsigned int cand_count;
};
struct Cand { uint32_t score_key, segment_ord, doc, pad; };

struct BatchParams {
  const ListDesc* lists;
  const float* caches;  // [n_caches][256] tf-norm tables (bm25.rs:58-69)
  const float* tf_tables;  // [n_caches][kTfRows][256]: tf / (tf + norm[id]) for tf < kTfRows
  const QList* qlists;
  const QSeg* qsegs;
  const Unit* units;
  const DQuery* queries;
  QState* qstate;
  Cand* cands;
  float* res_scores;
  uint32_t* res_segs;
  uint32_t* res_docs;
  uint32_t* res_counts;
  uint32_t res_stride;
  uint32_t n_queries;
  unsigned long long* counters;  // [8] k_or_strip windows by route: 1 exhaustive, 2 hot, 3 cold; 5 bytes read
  uint32_t reserved[4];          // unused: keeps the struct at 144 B.  At 128 B nvcc 12.9 loads the kernel parameters another
                                 // way and the code of every kernel changes (k_or_strip measured 0.4% slower on an H100).
  uint32_t* ovf;                 // set by k_final when a query was handed more candidates than its region holds (tile engine only), or null
};

static_assert(sizeof(ListDesc) == 80, "ListDesc layout");
static_assert(sizeof(QList) == 16 && sizeof(QSeg) == 40 && sizeof(Unit) == 16 && sizeof(DQuery) == 16 && sizeof(Cand) == 16,
              "per-query descriptor layout");
static_assert(sizeof(BatchParams) == 144, "BatchParams must stay at 144 B (see `reserved`)");

// k_or_strip (tq_kernels.cuh).  Eligible when k <= kStripMaxK, <= kStripMaxLists clauses and <= kMaxCached thin clauses; otherwise k_or.
constexpr uint32_t kWin = 1024;  // docs per window (multiple of 512)
constexpr uint32_t kMaxCached = 6;
constexpr uint32_t kStripWarps = 4;
constexpr uint32_t kStripThreads = kStripWarps * 32;
constexpr uint32_t kStripMaxLists = 8;
constexpr uint32_t kStripMaxK = 128;
// MaxScore split: a clause with at least one posting per kStripNeDiv docs may turn non-essential; in a union without
// such a clause, the densest one may still go under the looser bound kStripNeDiv2.
constexpr uint32_t kStripNeDiv = 8;
constexpr uint32_t kStripNeDiv2 = 64;
// Threshold sample: the three sample launches of a (query, segment) end at 1/32, 1/8 and 1/2 of its windows.
constexpr uint32_t kStripSampleDiv = 32;
constexpr uint32_t kStripSampleDiv2 = 8;
constexpr uint32_t kStripSampleDiv3 = 2;

// Dynamic shared memory of k_or_strip: per warp a StripWarpFixed and n_cached StripCaches (sizes asserted beside the types).
constexpr size_t kStripWarpFixedBytes = 7424, kStripCacheBytes = 1024;
TQ_HD constexpr size_t strip_smem_bytes(uint32_t n_cached) {
  return kStripWarps * (kStripWarpFixedBytes + (size_t)n_cached * kStripCacheBytes);
}

// words = [n_groups, need, n_should, n_not, (len, list ids..) per group, should list ids.., not list ids..] (32-bit).
struct CountSeg {
  uint32_t query, words_base, max_doc, pad;
  const uint8_t* alive;
};
struct CountParams {
  const ListDesc* lists;
  const uint32_t* words;
  const CountSeg* segs;
  const Unit* units;
  unsigned long long* counts;
};

// ---- sort by a fast field (k_sort, k_sort_final) ------------------------------------------------------------------------
// The key of a doc with a value is v' = value (Desc) or ~value (Asc): larger v' first.  Docs without a value (None) come after
// every doc with one, in (segment, doc) order, in both orders; they travel as a stream of their own.
constexpr uint32_t kSortMaxK = 1024;  // TQ_MAX_K: a k_sort CTA keeps up to this many None docs on chip

// One 8192-doc tile of a registered column: the best v' any doc with a value can have, per order ([0] Desc: the largest value,
// [1] Asc: ~ the smallest), and which kinds of docs it holds.
struct SortTile {
  unsigned long long best[2];
  uint32_t flags;  // kSortTileValues: some doc has a value; kSortTileNone: some doc has none
  uint32_t pad;
};
constexpr uint32_t kSortTileValues = 1, kSortTileNone = 2;
struct SortSeg {  // the column of one (query, segment), parallel to CountParams::segs
  const unsigned long long* values;  // [max_doc] u64 images
  const uint32_t* present;           // bitset in the alive layout (null: every doc has a value)
  const SortTile* tiles;
  uint32_t segment_ord, pad;
};
struct SortQuery {
  uint32_t k;
  uint32_t flags;      // kSortAsc; kSortAllTiles: the query's hits are counted, so no tile is skipped
  uint32_t cand_base;  // first slot of the query's regions in SortParams::cands and ::nones (units of the query x k each)
  uint32_t pad;
};
constexpr uint32_t kSortAsc = 1, kSortAllTiles = 2;
constexpr uint32_t kSortUnitBackward = 1;  // Unit::pad of a k_sort unit: walk its tiles from the last to the first
struct SortQState {  // zeroed before every run
  unsigned long long theta;  // lower bound of the query's k-th v' (a CTA that held k docs with values published its k-th)
  uint32_t full;             // some CTA held k docs with values: no None doc can make the top k
  uint32_t n_cands, n_nones;
  uint32_t pad;
};
struct SortCand { unsigned long long key; uint32_t segment_ord, doc; };  // key: v' (None stream: unused)
struct SortParams {
  CountParams c;  // structure words, (query, segment) pairs, units and hit counters: the Count plan
  const SortSeg* ssegs;
  const SortQuery* queries;
  SortQState* qstate;
  SortCand* cands;  // per query: the docs with values each unit kept (<= k per unit)
  SortCand* nones;  // per query: the first k None docs of each unit in doc order
  unsigned long long* tiles;  // [0] tiles seen, [1] of them skipped
  unsigned long long* res_values;
  uint8_t* res_present;
  uint32_t* res_segs;
  uint32_t* res_docs;
  uint32_t* res_counts;
  uint32_t res_stride;
};
static_assert(sizeof(SortTile) == 24 && sizeof(SortSeg) == 32 && sizeof(SortQuery) == 16 && sizeof(SortQState) == 24 && sizeof(SortCand) == 16,
              "sort descriptor layout");

// ---- histogram of a fast field (k_hist, k_hist_final) -------------------------------------------------------------------
// Doc counts per bucket pos = as_i64(floor((val - offset) / interval)) of the docs Count counts whose value lies in the (query,
// segment)'s bounds.  A query's counters cover its dense range [base, base + n_bins); a unit counts into its own window of them
// (HistUnit): kHistSmemBins or fewer are kept per CTA in shared memory, more go straight to the global u64 counters.  A range above kHistMaxBins is refused (TQ_ERR_UNSUPPORTED).
// The value and the bucket are computed by the same code on the host (the planner's ranges) and on the device (k_hist).
// f64_from_fastfield_u64 (aggregation/mod.rs:374) of a u64 image
TQ_HD inline double hist_value(unsigned long long v, uint32_t kind) {
  constexpr unsigned long long kHigh = 1ull << 63;
  if (kind == TQ_FAST_F64) {
    const unsigned long long bits = (v & kHigh) ? v ^ kHigh : ~v;
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)bits);
#else
    double d;
    memcpy(&d, &bits, 8);
    return d;
#endif
  }
  if (kind == TQ_FAST_I64 || kind == TQ_FAST_DATE) return (double)(long long)(v ^ kHigh);
  return (double)v;  // u64, bool
}
// get_bucket_pos_f64(val, interval, offset) as i64 (histogram.rs:739-741): Rust's `as` saturates and maps NaN to 0
TQ_HD inline long long hist_pos(double val, double offset, double interval) {
#ifdef __CUDA_ARCH__
  const double f = floor(__ddiv_rn(__dsub_rn(val, offset), interval));
#else
  const double f = floor((val - offset) / interval);  // (the host units build with -ffp-contract=off)
#endif
  if (f != f) return 0;
  if (f >= 9223372036854775808.0) return 0x7FFFFFFFFFFFFFFFll;
  if (f < -9223372036854775808.0) return (long long)0x8000000000000000ull;
  return (long long)f;
}
constexpr uint32_t kHistSmemBins = 4096;
constexpr uint32_t kHistMaxBins = 1u << 20;
struct HistSeg {  // the column and bounds of one (query, segment), parallel to CountParams::segs
  const unsigned long long* values;  // [max_doc] u64 images
  const uint32_t* present;           // bitset in the alive layout (null: every doc has a value)
  const SortTile* tiles;             // the column's per-tile bounds (tq_sort_column_register)
  double lo, hi;                     // collect-time bounds after the per-segment collapse: val counts iff lo <= val <= hi
};
struct HistQuery {
  double interval, offset;
  long long base;              // pos of counter 0
  unsigned long long counters; // first counter of the query in HistParams::counts
  uint32_t n_bins;             // 0: no doc of the query can pass its bounds
  uint32_t kind;               // TQ_FAST_*
  uint32_t flags;              // kHistHits: the query's Count is asked for as well
  uint32_t pad;
};
constexpr uint32_t kHistHits = 1;
struct HistUnit {  // the buckets one k_hist unit can count into, parallel to CountParams::units
  uint32_t first;   // its first counter, relative to the query's base
  uint32_t n_bins;  // 0: no value of the unit's tiles passes the bounds
};
struct HistParams {
  CountParams c;  // structure words, (query, segment) pairs, units and hit counters: the Count plan
  const HistSeg* hsegs;
  const HistQuery* queries;
  const HistUnit* hunits;
  unsigned long long* counts;   // every query's counters, zeroed before the run
  unsigned long long* tiles;    // [0] tiles seen, [1] of them counted as one bucket
  long long* res_pos;           // [nq][res_stride]: the non-empty buckets in ascending pos
  unsigned long long* res_count;
  uint32_t* res_n;              // [nq]: how many there are (may exceed res_stride: only res_stride are written)
  uint32_t res_stride;
};
static_assert(sizeof(HistSeg) == 40 && sizeof(HistQuery) == 48 && sizeof(HistUnit) == 8, "histogram descriptor layout");

// ---- terms of a fast field (k_terms, k_terms_select) ----------------------------------------------------------------------
// Doc counts per image of the docs Count counts.  Each (query, segment) has u32 counters over [base, base + n_keys), the images
// of the 8192-doc tiles its units visit (at most kTermsMaxKeys, else TQ_ERR_UNSUPPORTED), and one counter of its matching docs
// without a value; a unit counts into its own window of them (a HistUnit), on chip when it has kHistSmemBins or fewer.  Queries run
// in waves whose counters fit the ctx's budget: a TermsSeg's counters and region are relative to its wave.
constexpr uint32_t kTermsMaxKeys = 1u << 20;
struct TermsSeg {  // one (query, segment), parallel to CountParams::segs
  const unsigned long long* values;  // [max_doc] u64 images
  const uint32_t* present;           // bitset in the alive layout (null: every doc has a value)
  const SortTile* tiles;             // the column's per-tile bounds
  unsigned long long base;           // image of counter 0
  unsigned long long missing;        // the key of a doc without a value (kTermsMissing)
  unsigned long long counters;       // first counter in TermsParams::counts
  unsigned long long region;         // first kept entry in TermsParams::res_key / res_count
  uint32_t n_keys;                   // counters (0: no visited tile holds a value)
  uint32_t segment_size;             // entries kept, >= 1
  uint32_t flags;                    // kTerms*
  uint32_t pad;
};
constexpr uint32_t kTermsHits = 1, kTermsMissing = 2, kTermsByKey = 4, kTermsAsc = 8;
struct TermsParams {
  CountParams c;                // structure words, (query, segment) pairs, units and hit counters: the Count plan of the batch
  const TermsSeg* tsegs;        // parallel to c.segs
  const HistUnit* windows;      // parallel to c.units: each unit's window of its (query, segment)'s counters
  uint32_t* counts;             // the wave's counters, zeroed before it
  uint32_t* missing;            // [wave's (query, segment)s]: their matching docs without a value, zeroed before the wave
  unsigned long long* tiles;    // [0] tiles seen, [1] of them counted as one key
  unsigned long long* res_key;  // the wave's kept entries, each (query, segment) in its region, ascending key
  uint32_t* res_count;
  uint32_t* res_n;              // [wave's (query, segment)s]: kept entries
  unsigned long long* res_other;  // ... sum_other_doc_count
  unsigned long long* res_error;  // ... term_doc_count_before_cutoff
  uint32_t unit_base, seg_base;   // the wave's first unit and first (query, segment)
};
static_assert(sizeof(TermsSeg) == 72, "terms descriptor layout");

// ---- metrics of fast fields (k_metrics) -----------------------------------------------------------------------------------
// One tq_metric_part accumulator per (query, column), fed by every unit of the query: no counters, so no waves and no size limit.
constexpr uint32_t kMetricsMaxColumns = 4;  // TQ_METRICS_MAX_COLUMNS
struct MetricsCol {  // one column of one (query, segment)
  const unsigned long long* values;  // [max_doc] u64 images
  const uint32_t* present;           // bitset in the alive layout (null: every doc has a value)
  const SortTile* tiles;             // the column's per-tile bounds
  unsigned long long missing;        // the image a doc without a value collects (TQ_METRIC_MISSING)
  uint32_t kind;                     // TQ_FAST_*
  uint32_t flags;                    // TQ_METRIC_*
};
struct MetricsSeg {  // one (query, segment), parallel to CountParams::segs
  MetricsCol col[kMetricsMaxColumns];
  uint32_t n_columns;
  uint32_t flags;  // kMetricsHits
  uint32_t pad[2];
};
constexpr uint32_t kMetricsHits = 1;
struct MetricsParams {
  CountParams c;                // structure words, (query, segment) pairs, units and hit counters: the Count plan of the batch
  const MetricsSeg* msegs;      // parallel to c.segs
  tq_metric_part* parts;        // [query][kMetricsMaxColumns], initialised empty by the host
  unsigned long long* tiles;    // [0] (tile, column) pairs seen, [1] of them added as one value
};
static_assert(sizeof(MetricsCol) == 40 && sizeof(MetricsSeg) == 176, "metrics descriptor layout");
// The exponent of the lowest set bit of a finite non-zero |v| (v is a multiple of 2^that); the guard's Q is its minimum.
TQ_HD inline int metric_quantum_exp(unsigned long long abs_bits) {
  const int e = (int)(abs_bits >> 52);
  unsigned long long m = abs_bits & ((1ull << 52) - 1ull);
  if (e) m |= 1ull << 52;
#ifdef __CUDA_ARCH__
  const int tz = __ffsll((long long)m) - 1;
#else
  const int tz = __builtin_ctzll(m);
#endif
  return (e ? e - 1075 : -1074) + tz;
}

// ---- metrics per histogram bucket (k_hist_metrics, k_hist_metrics_final) ------------------------------------------------------
// The histogram's buckets (HistSeg, HistQuery, HistUnit as in k_hist) with one doc counter and kMetricsMaxColumns tq_metric_part
// accumulators per bucket, fed by the columns of the (query, segment)'s MetricsSeg.  A unit whose window has kHistMetricsSmemBins
// or fewer buckets accumulates in shared memory (tq_metric_part layout, flushed per non-empty bucket at exit), a wider one in
// global memory.  A range above kHistMetricsMaxBins is refused (TQ_ERR_UNSUPPORTED); queries run in waves whose accumulators fit
// the ctx's budget, and a HistQuery's counters are relative to its wave.
constexpr uint32_t kHistMetricsSmemBins = 128;
constexpr uint32_t kHistMetricsMaxBins = 1u << 16;
struct HistMetricsParams {
  CountParams c;                // structure words, (query, segment) pairs, units and hit counters: the Count plan of the batch
  const HistSeg* hsegs;         // parallel to c.segs: the histogram column and bounds
  const MetricsSeg* msegs;      // parallel to c.segs: the metric columns
  const HistQuery* queries;     // [nq]: counters relative to the wave
  const HistUnit* hunits;       // parallel to c.units
  unsigned long long* counts;   // the wave's doc counters, zeroed before it
  tq_metric_part* parts;        // [wave's counters][kMetricsMaxColumns], initialised empty before the wave
  unsigned long long* tiles;    // [0] tiles seen, [1] of them in one bucket, [2] buckets flushed from shared, [3] runs flushed to global
  const unsigned long long* rows;  // [nq]: first entry of the query's row in res_*, relative to its wave; the row holds
                                   // min(res_stride, n_bins) entries, so a wave's rows never outnumber its counters
  long long* res_pos;           // the wave's rows: the non-empty buckets in ascending pos
  unsigned long long* res_count;
  tq_metric_part* res_parts;    // [wave's row entries][kMetricsMaxColumns]
  uint32_t* res_n;              // [wave's queries]
  uint32_t res_stride;
  uint32_t unit_base, query_base;  // the wave's first unit and first query
};

// ---- range of a fast field (k_range, k_range_metrics) ---------------------------------------------------------------------
// Doc counts per range bucket b = the last start <= image (get_bucket_pos, range.rs) of the docs Count counts, and with metrics one
// tq_metric_part per (bucket, column) as in k_hist_metrics.  A query's counters are its n_bins buckets, every one of them (the rows
// are dense), and every unit's window is the query's whole bucket list (kRangeMaxBins <= kHistMetricsSmemBins <= kHistSmemBins:
// always on chip).  With metrics, queries run in waves whose accumulators fit the ctx's budget, and counters are relative to the wave.
constexpr uint32_t kRangeMaxBins = 128;  // TQ_RANGE_MAX_BUCKETS
static_assert(kRangeMaxBins <= kHistMetricsSmemBins && kRangeMaxBins <= kHistSmemBins, "a range window always lives in shared memory");
struct RangeSeg {  // the column of one (query, segment), parallel to CountParams::segs
  const unsigned long long* values;  // [max_doc] u64 images
  const uint32_t* present;           // bitset in the alive layout (null: every doc has a value)
  const SortTile* tiles;             // the column's per-tile bounds
};
struct RangeQuery {
  const unsigned long long* starts;  // [n_bins] strictly ascending images, starts[0] == 0 (device)
  unsigned long long counters;       // first counter of the query
  uint32_t n_bins;                   // 1 .. kRangeMaxBins
  uint32_t flags;                    // kRangeHits: the query's Count is asked for as well
};
constexpr uint32_t kRangeHits = 1;
struct RangeParams {
  CountParams c;                // structure words, (query, segment) pairs, units and hit counters: the Count plan
  const RangeSeg* rsegs;        // parallel to c.segs
  const RangeQuery* queries;    // [nq]
  const HistUnit* windows;      // parallel to c.units: {0, n_bins} of the unit's query
  unsigned long long* counts;   // every query's counters, zeroed before the run
  unsigned long long* tiles;    // [0] tiles seen, [1] of them counted as one bucket
};
struct RangeMetricsParams {
  CountParams c;                // structure words, (query, segment) pairs, units and hit counters: the Count plan of the batch
  const RangeSeg* rsegs;        // parallel to c.segs
  const MetricsSeg* msegs;      // parallel to c.segs: the metric columns
  const RangeQuery* queries;    // [nq]: counters relative to the wave
  const HistUnit* windows;      // parallel to c.units
  unsigned long long* counts;   // the wave's doc counters, zeroed before it
  tq_metric_part* parts;        // [wave's counters][kMetricsMaxColumns], zeroed before the wave (complemented as in k_hist_metrics)
  unsigned long long* tiles;    // [0] tiles seen, [1] of them in one bucket, [2] buckets flushed from shared, [3] runs flushed to global
  uint32_t unit_base;           // the wave's first unit
};
static_assert(sizeof(RangeSeg) == 24 && sizeof(RangeQuery) == 24, "range descriptor layout");

// ---- metrics per term (k_terms_order, k_terms_select_metric, k_terms_mark, k_terms_metrics) ---------------------------------
// The terms of k_terms / k_terms_select (TermsSeg, the unit windows, the counters) with the metric columns of the (query, segment)'s
// MetricsSeg.  After the cut, k_terms_mark overwrites the counter of each kept key with kTermsSlot | its index in the (query,
// segment)'s region (a missing key outside the counters gets its slot in `mslot`); k_terms_metrics feeds each counted doc to the
// kMetricsMaxColumns tq_metric_parts of its key's slot (complemented as in k_hist_metrics), in shared memory when the (query,
// segment) keeps kTermsMetricsSmemSlots or fewer entries.  A metric order (kTermsByMetric) first accumulates per key of the
// window the ordering column's value count and its one quantity (the f64 sum, ~min image or max image) in `ocount` / `oq`, and the
// column's part over every collected doc per query; k_terms_select_metric cuts on them.
constexpr uint32_t kTermsByMetric = 16;  // TermsSeg::flags: the order is orders[query]
constexpr uint32_t kTermsSlot = 0x80000000u;
constexpr uint32_t kTermsMetricsSmemSlots = 128;
constexpr uint32_t kTermsOrderSmemKeys = 1024;
struct TermsOrder {  // tq_terms_metric_order of one query
  uint32_t column, metric;
};
struct TermsMetricsParams {
  TermsParams t;                  // the terms of the wave: counters, missing counters, kept entries and scalars
  const MetricsSeg* msegs;        // parallel to t.c.segs
  const TermsOrder* orders;       // [nq]
  uint32_t* ocount;               // parallel to t.counts: the ordering column's values per key (metric orders), zeroed per wave
  unsigned long long* oq;         // ... their sum (f64 bits), ~smallest or largest image
  uint32_t* ocount_missing;       // [wave's (query, segment)s]: the same for a missing key outside the counters
  unsigned long long* oq_missing;
  tq_metric_part* order_parts;    // [nq]: the ordering column over every collected doc, complemented, zeroed once
  uint32_t* mslot;                // [wave's (query, segment)s]: kTermsSlot | slot of a missing key outside the counters, or 0
  tq_metric_part* parts;          // [wave's region][kMetricsMaxColumns], complemented, zeroed per wave
  unsigned long long* tiles;      // [0] tiles k_terms_metrics saw, [1] of them with one kept key
};
static_assert(sizeof(TermsOrder) == 8, "terms order descriptor layout");

// ---- histogram per term (k_terms_hist, k_terms_hist_final) --------------------------------------------------------------------
// The terms of k_terms / k_terms_select / k_terms_mark (TermsSeg, the unit windows, the counters marked with each kept key's slot)
// with the histogram of HistSeg / HistQuery / HistUnit.  Each (query, segment) has a u32 cell grid of (its region's entries) rows ×
// (its bucket span) columns; k_terms_hist counts each doc the terms count under a kept key, and whose histogram value is in bounds,
// in cell (slot, pos - base).  A unit whose window (kept slots × its buckets) has kTermsHistSmemCells or fewer cells counts in
// shared memory and adds its non-zero cells to the grid at exit.  k_terms_hist_final compacts each (query, segment)'s non-empty
// cells, slot by slot in ascending pos, into the wave's cell list.  Queries run in waves whose grids fit the ctx's budget.
constexpr uint32_t kTermsHistSmemCells = 8192;
struct TermsHistSeg {  // the grid of one (query, segment), parallel to CountParams::segs
  unsigned long long grid;  // its first cell in TermsHistParams::grid (relative to the wave)
  long long base;           // pos of column 0
  uint32_t span;            // columns per slot (0: no value of the segment's visited tiles passes its bounds)
  uint32_t pad;
};
struct TermsHistParams {
  TermsParams t;                // the terms of the wave: counters (kept keys marked), missing counters, kept entries and scalars
  const HistSeg* hsegs;         // parallel to t.c.segs: the histogram column and bounds
  const HistQuery* queries;     // [nq]: interval, offset and kind of the query's histogram
  const TermsHistSeg* gsegs;    // parallel to t.c.segs
  const HistUnit* hunits;       // parallel to t.c.units: the unit's buckets, relative to its (query, segment)'s base
  const uint32_t* mslot;        // [wave's (query, segment)s]: kTermsSlot | slot of a missing key outside the counters, or 0
  uint32_t* grid;               // the wave's cells, zeroed before it
  unsigned long long* tiles;    // [0] tiles seen, [1] of them with one kept key, [2] in one bucket, [3] both; units counting [4] in
                                // shared memory, [5] in the grid
  uint32_t* cell_first;         // [wave's region]: first cell of the entry in the wave's cell list (k_terms_hist_final)
  uint32_t* cell_pos;           // the wave's cell list: pos - base of the (query, segment)
  uint32_t* cell_count;
  uint32_t* cell_total;         // [wave's (query, segment)s]: their non-empty cells
  unsigned long long* cursor;   // cells the wave's list holds
};
static_assert(sizeof(TermsHistSeg) == 24, "terms histogram descriptor layout");

// ---- terms per histogram bucket (k_hist_terms, k_hist_terms_final) ----------------------------------------------------------
// The histogram of HistSeg / HistQuery / HistUnit with the terms key windows of TermsSeg (no k_terms counters).  Each (query,
// segment) has a u32 grid of (its bucket span) rows × (n_keys + 1) columns: column k counts the docs of image base + k, column
// n_keys the docs without a value (the missing key when it lies outside the keys, else nothing); a missing key inside the keys
// counts in its own column.  k_hist_terms counts each matching doc whose histogram value is in bounds in cell (pos - base, column):
// a row's cells sum to the histogram's doc count.  A unit whose window (its buckets × its keys + 1) fits kTermsHistSmemCells
// counts in shared memory.  k_hist_terms_final, a warp per row, compacts each row's entries once, cuts each row of a whole segment
// with more than segment_size entries by a warp's radix select over them, and writes the non-empty rows with their kept entries.
struct HistTermsSeg {  // the grid of one (query, segment), parallel to CountParams::segs
  unsigned long long grid;  // its first cell in HistTermsParams::grid (relative to the wave)
  long long base;           // pos of row 0
  uint32_t span;            // rows (0: no value of the segment's visited tiles passes its bounds)
  uint32_t cols;            // n_keys + 1
  uint32_t mcol;            // the column of a doc without a value
  uint32_t n_entries;       // entry columns in key order: n_keys, plus 1 for a missing key outside the keys
  uint32_t mfirst;          // 1: that missing key sorts before the keys (entry 0 is column n_keys)
  uint32_t row;             // its first row in HistTermsParams::rows (relative to the wave)
};
// One non-empty bucket row of a (query, segment) (seg: its index in the wave): its pos - base, doc count, kept entries (first: in
// the wave's entry list) and scalars.
struct HistTermsRow {
  uint32_t pos, doc_count, n, first, seg, pad;
  unsigned long long other, error;
};
// One entry: its index in key order (HistTermsSeg) and doc count.
struct HistTermsEntry { uint32_t key, count; };
struct HistTermsParams {
  CountParams c;                 // structure words, (query, segment) pairs, units and hit counters: the Count plan of the batch
  const TermsSeg* tsegs;         // parallel to c.segs: the terms column, key base and count, missing key, segment_size, flags
  const HistUnit* windows;       // parallel to c.units: the unit's keys, relative to its TermsSeg's base
  const HistSeg* hsegs;          // parallel to c.segs: the histogram column and bounds
  const HistQuery* queries;      // [nq]: interval, offset and kind of the query's histogram
  const HistTermsSeg* gsegs;     // parallel to c.segs
  const HistUnit* hunits;        // parallel to c.units: the unit's buckets, relative to its (query, segment)'s base
  uint32_t* grid;                // the wave's cells, zeroed before it
  HistTermsEntry* ents;          // the entries of the wave's rows that are cut (k_hist_terms_final's scratch)
  HistTermsRow* out_rows;        // the wave's non-empty rows, in any order
  HistTermsEntry* out_ents;      // their kept entries, row by row
  unsigned long long* cursor;    // [0] ents, [1] out_ents, [2] out_rows held
  unsigned long long* tiles;     // [0] tiles seen, [1] of them with one key, [2] in one bucket, [3] both; units counting [4] in
                                 // shared memory, [5] in the grid; [6] rows cut
  uint32_t unit_base, seg_base;  // the wave's first unit and first (query, segment)
  uint32_t n_segs, n_rows;       // the wave's (query, segment)s and rows
};
static_assert(sizeof(HistTermsSeg) == 40 && sizeof(HistTermsRow) == 40 && sizeof(HistTermsEntry) == 8, "histogram terms descriptor layout");

// ---- the tile engine (tq_tile.cuh) --------------------------------------------------------------------------------------

constexpr uint32_t kTile = 1024;            // docs per tile
constexpr uint32_t kTileThreads = 256;
constexpr uint32_t kTileWarps = kTileThreads / 32;
constexpr uint32_t kTileMaxQueries = 1024;  // (query, segment) pairs of one group in one segment
constexpr uint32_t kTileMaxSlots = 4096;    // distinct scored lists of one group in one segment
constexpr uint32_t kTileMaxBig = 64;        // dense lists of one segment that get a tile index and a presence map
constexpr uint32_t kTileMaxPairs = 12288;   // pairs of one tile held in shared memory (start | len are 16-bit fields)
constexpr uint32_t kTileExactWindows = 2;   // warps that take heavy pairs in an exact launch (each owns a window of kTile f32 slots)
constexpr uint32_t kNoSlot = 0xFFFFFFFFu;
constexpr uint32_t kTileOpAnd = 1;  // TQ_OP_AND; term queries and unions share one evaluation (a union of one clause)
constexpr uint32_t kTileOpBool = 3;  // TQ_OP_BOOL: the clause words are [n_groups, need_should, n_should, n_not, (len, slots..) per MUST group,
                                     // SHOULD slots.., MUST_NOT slots..], groups by ascending cost, slots inside by descending weight

struct TSlot {  // one distinct scored list of a group: (posting list, Bm25Weight.weight, tf-norm table)
  uint32_t list_id;
  float weight;
  uint32_t cache_idx;
  uint32_t doc_freq;
  uint32_t pair_base;  // first element of this list's pairs in p_docs / p_scores (multiple of 128)
  uint32_t big;        // column in the segment's tile index, kNoSlot for small lists
  uint32_t tseg;
  uint32_t pad;
};
struct TSeg {  // one segment of a group
  uint32_t slot_base, n_slots, n_big;  // slots [0, n_big) have a tile index and are staged by whole warps
  uint32_t query_base, n_queries;
  uint32_t max_doc, segment_ord, n_tiles;
  uint32_t clause_base, n_clause_words;  // this segment's share of TileParams::clauses (staged in shared memory when it fits)
  uint32_t pad0, pad1;
  const uint8_t* alive;
  uint32_t* tix;  // [(n_tiles + 1)][n_big]: index of the list's first pair with doc >= tile * kTile (written by k_score_lists)
};
struct TQuery {  // one (query, segment): what Collector::collect_segment sees
  uint32_t query;
  uint32_t clause_base;  // into TileParams::clauses: slot ordinals (local to the segment) in canonical summation order
  uint16_t n_clauses;
  uint8_t op;
  uint8_t flags;  // bit 0: prunable (every weight finite and >= 0);
                  // bit 2: AND / BOOL groups in Intersection::score order, (s0 + s1) + (s2 + s3 + ...), not one after another
};
struct TUnit { uint32_t tseg, t0, t1, pad; };
struct SChunk { uint32_t slot, b0, b1; };  // a CTA's share of k_score_lists: blocks [b0, b1) of one slot (global slot ordinal)

static_assert(sizeof(TSlot) == 32 && sizeof(TSeg) == 64 && sizeof(TQuery) == 12 && sizeof(TUnit) == 16 && sizeof(SChunk) == 12,
              "tile descriptor layout");

// Running threshold of the exact k_tile launches: per query of the batch, a count of its pushed candidates' score keys by
// bucket of key >> 16 (1/128 of a binade, 0.8 %) above a per-query base, kThHistFine buckets in kThHistCoarse coarse buckets of 32,
// so that one warp finds the k-th from the top with two reads of one word per lane.  A query's words: fine counts [0, 2048),
// coarse counts [2048, 2112), the base word at kThHistBaseWord (k_theta_samples writes the threshold's key >> 16 there; 0 = no
// threshold yet: kThHistFallbackBase, the key of 2^-4 >> 16, so the window spans 2^-4 .. 2^12).  Zeroed at the start of every run.
constexpr uint32_t kThHistFine = 2048, kThHistCoarse = 64, kThHistBaseWord = kThHistFine + kThHistCoarse;
constexpr uint32_t kThHistWords = kThHistBaseWord + 32u;  // (a multiple of 32 words: every query's region starts on a 128-B line)
constexpr uint32_t kThHistFallbackBase = 0xBD80u;
TQ_HD inline uint32_t th_hist_base(uint32_t base_word) { return base_word ? base_word : kThHistFallbackBase; }
// The bucket of a key: 0 at or below the base, the top bucket above the window.  edge(b) is a key no larger than any key of
// bucket b (0 for bucket 0), and grows with b: edge(bucket(key)) <= key, so k candidates in buckets >= b hold k keys >= edge(b).
TQ_HD inline uint32_t th_hist_bucket(uint32_t key, uint32_t base) {
  const uint32_t hi = key >> 16;
  return hi <= base ? 0u : (hi - base < kThHistFine - 1u ? hi - base : kThHistFine - 1u);
}
TQ_HD inline uint32_t th_hist_edge(uint32_t b, uint32_t base) {
  const uint32_t hi = base + b;
  return b ? (hi < 0xFFFFu ? hi : 0xFFFFu) << 16 : 0u;
}

struct TileParams {
  const TSlot* slots;
  const TSeg* segs;
  const TQuery* queries;
  const uint16_t* clauses;
  const TUnit* units;
  const SChunk* chunks;
  uint32_t* p_docs;
  float* p_scores;
  uint32_t* samples;       // [n_queries of the batch][sample_cap] score keys
  uint32_t* sample_count;  // [n_queries of the batch]
  uint32_t* flags;         // [0]: a tile held more pairs than p_cap (the batch is re-run on the per-query kernels)
  unsigned long long* counters;  // [16] diagnostics: 0 (query, tile) pairs seen, 1 skipped (bound / no essential posting / cold window),
                                 //     2 light pairs, 3 heavy pairs, 4 essential postings applied, 5 docs completed, 6 docs at or above the threshold;
                                 //     [8, 8 + kTileStages) clock64() cycles summed over warps, by stage (TileStage);
                                 //     [16, 16 + kOrExits) B2's union postings by exit (TileOrExit);
                                 //     14 running-threshold refreshes, 15 of them that raised the threshold
                                 //     (null: the launch runs k_tile<*, false, *>)
  uint32_t* th_hist;   // [n_queries of the batch][kThHistWords]: the exact launches' candidate keys by bucket (th_hist_bucket)
  uint2* cursors;      // [CTAs of the largest launch][max_slots] sparse slots' cursors (k_tile)
  uint32_t sample_cap;
  uint32_t p_cap;      // pairs of one tile that fit in shared memory
  uint32_t max_slots;  // largest n_slots of any segment of the group
  uint32_t max_big;    // ... n_big
  uint32_t max_queries;  // ... n_queries
  uint32_t cl_cap;     // clause words staged in shared memory per CTA (0: the segment's clauses are read from global memory)
  uint32_t seg_cap;    // entries of the per-tile work list (essential clauses of the flat pairs)
  uint32_t light_max;  // (query, tile) pairs with at most this many essential postings are evaluated posting by posting (flat path);
                       // above it (and with more than one essential clause) a warp accumulates the query's window
  uint32_t n_win;      // warps of a CTA that own a window (2: heavy pairs are rare; 8 for groups with wide queries)
};

// Sizes of k_tile's on-chip records (TileQ, TileSeg, TileTQ, TileStageA in tq_tile.cuh, asserted there).
constexpr uint32_t kTileQBytes = 16, kTileSegBytes = 4, kTileTQBytes = 8, kTileStageABytes = 1056;

// Shared memory of a k_tile CTA: byte offsets of its regions, in this order (the sparse slots' cursors are not on chip:
// TileParams::cursors).  f32 scores [p_cap] at 0; the work list: TileQ records [max_queries] (`list`) + TileSeg segments [seg_cap]
// (`seg`, which stage A uses for its TileStageA scratch), and in the same bytes the [n_win][kTile] f32 windows of the rare heavy
// pairs (stage B3 starts after the last B2 of the tile); per slot: pair range start | len << 16 (`info`), largest score in the tile
// (`max`, >= 0) and stripe mask [max_slots] each; presence maps [max_big][32]; TileTQ [max_queries]; u16 presence map ranks
// [max_big][32], doc offsets [p_cap], heavy pairs [max_queries] and clause slots [cl_cap].
struct TileSmem { uint32_t list, seg, info, max, mask, bits, tq, rank, off, heavy, cl, end; };
TQ_HD constexpr TileSmem tile_smem_layout(uint32_t p_cap, uint32_t max_slots, uint32_t max_big, uint32_t max_queries,
                                          uint32_t seg_cap, uint32_t cl_cap, uint32_t n_win) {
  const uint32_t seg_bytes = seg_cap * kTileSegBytes > kTileStageABytes ? seg_cap * kTileSegBytes : kTileStageABytes;
  const uint32_t list_bytes = max_queries * kTileQBytes + seg_bytes, win_bytes = n_win * kTile * 4u;
  TileSmem L{};
  L.list = p_cap * 4u;
  L.seg = L.list + max_queries * kTileQBytes;
  L.info = L.list + (((list_bytes > win_bytes ? list_bytes : win_bytes) + 15u) & ~15u);
  L.max = L.info + max_slots * 4u; L.mask = L.max + max_slots * 4u; L.bits = L.mask + max_slots * 4u;
  L.tq = L.bits + max_big * 128u;
  L.rank = L.tq + max_queries * kTileTQBytes;
  L.off = L.rank + max_big * 64u; L.heavy = L.off + p_cap * 2u; L.cl = L.heavy + max_queries * 2u;
  L.end = L.cl + cl_cap * 2u + 64u;
  return L;
}
TQ_HD constexpr size_t tile_smem_bytes(uint32_t p_cap, uint32_t max_slots, uint32_t max_big, uint32_t max_queries, uint32_t seg_cap,
                                       uint32_t cl_cap, uint32_t n_win) {
  return tile_smem_layout(p_cap, max_slots, max_big, max_queries, seg_cap, cl_cap, n_win).end;
}
constexpr uint32_t kTileMaxSmem = 200u * 1024u;  // dynamic shared memory of a k_tile CTA (an H100 allows 227 KB)
constexpr uint32_t kTileMaxWorkList = 4096u;     // TileParams::seg_cap
// A group's clause words are staged in shared memory when its largest segment has at most this many; above it every segment
// reads them from global memory.  The bound keeps the largest layout the planner can produce -- any p_cap up to the repeat's
// kTileMaxPairs -- within kTileMaxSmem, so a group that was admitted is never refused for its shared memory.
constexpr uint32_t kTileMaxStagedClauses = 12288u;
static_assert(tile_smem_bytes(kTileMaxPairs, kTileMaxSlots, kTileMaxBig, kTileMaxQueries, kTileMaxWorkList, kTileMaxStagedClauses,
                              kTileWarps) <= kTileMaxSmem, "the largest k_tile group with staged clause words exceeds its shared memory");

// k_count_tiles
constexpr uint8_t kTileQueryCount = 8;      // TQuery::flags bit 3: count the query's hits (k_tile does not read it)
constexpr uint32_t kCountSparseCap = 8192;  // doc offsets of the sparse slots of one tile held in shared memory

struct CountTileParams {
  const TUnit* units;            // this group's count units
  uint2* cursors;                // [CTAs][max_slots] sparse slots' cursors: (first pair not walked yet, its doc)
  unsigned long long* hits;      // [queries of the batch]
  uint32_t* overflow;            // this group's word: a tile held more sparse offsets than kCountSparseCap
};

// Shared memory of a k_count_tiles CTA: presence maps [max_big][32] | sparse slots' start | len << 16 [max_slots] |
// per-query hit counts [max_queries] | sparse doc offsets (u16) [kCountSparseCap]
TQ_HD constexpr size_t count_tiles_smem_bytes(uint32_t max_slots, uint32_t max_big, uint32_t max_queries) {
  return (size_t)max_big * 128u + (size_t)max_slots * 4u + (size_t)max_queries * 4u + kCountSparseCap * 2u;
}
static_assert(count_tiles_smem_bytes(kTileMaxSlots, kTileMaxBig, kTileMaxQueries) <= 48u * 1024u,
              "k_count_tiles launches without raising its dynamic shared memory limit");

// ---- phrase queries (tq_phrase.cuh) ---------------------------------------------------------------------------------------

constexpr uint32_t kPhraseMaxTerms = 8;
constexpr uint32_t kPhraseWarps = 4;
constexpr uint32_t kPhraseThreads = kPhraseWarps * 32;

struct PosDesc {  // one term's position stream in one segment, built on first use and cached with the segment
  const uint8_t* widths;                 // [n_blocks] bit width of every bit-packed block
  const uint32_t* blk_off;               // [n_blocks + 1] byte offset of block b from `blocks`
  const uint8_t* blocks;                 // the bit-packed blocks (in the `.pos` body, any alignment)
  const uint32_t* tail;                  // [tail_n] the VInt-encoded rest, decoded
  const unsigned long long* post_off;    // [n_posting_blocks + 1] positions that precede posting block b (last entry: the VInt tail block)
  uint32_t n_blocks, tail_n, status, pad;
};
struct PosJob {
  const uint8_t* pos_bytes;   // the term's positions range
  uint32_t pos_len;
  const uint8_t* list_bytes;  // the term's postings range (for the skip records)
  uint32_t list_len;
  uint32_t doc_freq;
  uint32_t pos_id;
  unsigned char* pool;        // the segment's table pool ...
  unsigned long long* pool_cursor;  // ... bump-allocated on the device (the sizes are in the data)
  unsigned long long pool_cap;
};
struct PhraseAux { uint32_t pos_id, offset, slop = 0; };  // per clause of a phrase (parallel to qlists): its position table, max_offset - its offset, the phrase's slop

// dynamic shared memory: per warp [128][ct] PhraseCand (ct = most terms of a phrase in the batch) + [128 docs | 128 tfs | 128 prefixes]
// of a decoded secondary block (reused for the compacted matches)
constexpr size_t kPhraseCandBytes = 12;  // sizeof(PhraseCand), asserted beside it
TQ_HD constexpr size_t phrase_smem_bytes(uint32_t ct) { return kPhraseWarps * (128u * ct * kPhraseCandBytes + 384u * 4u); }

}  // namespace tq
