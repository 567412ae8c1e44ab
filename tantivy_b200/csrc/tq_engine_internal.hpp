// The engine's host-side state, shared by its translation units (tq_engine.cu, tq_plan.cpp): the context (tq_ctx) with its
// segment registry, filter views and device table caches, the staging buffers, and the registry functions the batch planner
// calls.  Host code only: no kernel header is included.
#pragma once
#include <algorithm>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "../../include/tantivy_b200.h"
#include "tq_host.hpp"
#include "tq_layout.h"

namespace tq::host {

struct DevBuf {
  uint8_t* p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    const size_t want = std::max<size_t>(n + n / 4, 1 << 20);
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
struct PinBuf {
  uint8_t* p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    const size_t want = std::max<size_t>(n + n / 4, 1 << 16);
    cudaError_t e = cudaMallocHost(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// Descriptors for the device: arrays placed back to back at 256-byte alignment.  reserve() sizes a pinned buffer and a device
// buffer of that layout (device pointers are valid from then on), copy() fills the pinned one, one H2D copy of `bytes` the other.
struct Staging {
  struct Part { size_t off; const void* src; size_t n; };
  std::vector<Part> parts;
  size_t bytes = 0;
  uint8_t *host = nullptr, *dev = nullptr;  // set by reserve
  size_t add(const void* src, size_t n) {  // src null: space only (device-only data, or filled through on_host)
    parts.push_back(Part{bytes, src, n});
    const size_t off = bytes;
    bytes = align256(bytes + n);
    return off;
  }
  template <class T> size_t add(const std::vector<T>& v) { return add(v.data(), v.size() * sizeof(T)); }
  cudaError_t reserve(PinBuf& pin, DevBuf& d) {
    cudaError_t e = pin.ensure(bytes + 256);
    if (e == cudaSuccess) e = d.ensure(bytes + 256);
    host = pin.p; dev = d.p;
    return e;
  }
  void copy() const { for (const Part& p : parts) if (p.src && p.n) memcpy(host + p.off, p.src, p.n); }
  template <class T> T* on_host(size_t off) const { return reinterpret_cast<T*>(host + off); }
  template <class T> T* on_device(size_t off) const { return reinterpret_cast<T*>(dev + off); }
};

struct ListKey {
  uint32_t segment_ord, field;
  uint64_t postings_start;  // bit 63: the table was built with term frequencies ignored (TQ_TERM_IGNORE_FREQ)
  bool operator==(const ListKey& o) const { return segment_ord == o.segment_ord && field == o.field && postings_start == o.postings_start; }
};
struct ListKeyHash {
  size_t operator()(const ListKey& k) const {
    uint64_t h = k.postings_start * 0x9E3779B97F4A7C15ull ^ ((uint64_t)k.segment_ord << 32 | k.field) * 0xC2B2AE3D27D4EB4Full;
    return (size_t)(h ^ (h >> 29));
  }
};
// A position table is read together with its term's postings (k_phrase), so its key holds both offsets exactly: two terms whose
// (postings_start, positions_start) pairs differ never share a table.
struct PosKey {
  uint32_t segment_ord, field;
  uint64_t postings_start, positions_start;
  bool operator==(const PosKey& o) const {
    return segment_ord == o.segment_ord && field == o.field && postings_start == o.postings_start && positions_start == o.positions_start;
  }
};
struct PosKeyHash {
  size_t operator()(const PosKey& k) const {
    return ListKeyHash{}(ListKey{k.segment_ord, k.field, k.postings_start}) ^ (size_t)(k.positions_start * 0xFF51AFD7ED558CCDull);
  }
};

// Bump allocator over big cudaMalloc chunks for the per-term block tables (immutable, never freed
// individually; dropped with the context).
struct Arena {
  std::vector<uint8_t*> chunks;
  size_t chunk_size = 1u << 20, cap = 0, used = 0;  // chunks double up to 64 MiB: a small segment holds a small arena
  uint8_t* alloc(size_t n, cudaError_t* err) {
    n = (n + 255) & ~(size_t)255;
    if (chunks.empty() || used + n > cap) {
      const size_t sz = std::max(chunk_size, n);
      uint8_t* p = nullptr;
      *err = cudaMalloc(&p, sz);
      if (*err != cudaSuccess) return nullptr;
      chunks.push_back(p);
      cap = sz;
      used = 0;
      chunk_size = std::min<size_t>(chunk_size * 2, 64u << 20);
    }
    uint8_t* r = chunks.back() + used;
    used += n;
    *err = cudaSuccess;
    return r;
  }
  void release() { for (auto* c : chunks) cudaFree(c); chunks.clear(); used = 0; cap = 0; }
};

struct Segment {
  uint32_t segment_ord, field, max_doc;
  int record_option;
  uint8_t* d_idx = nullptr;  // field body incl. the 8-byte header, padded
  size_t idx_len = 0;
  uint8_t* d_fieldnorm = nullptr;
  uint8_t* d_alive = nullptr;
  uint32_t doc_lo = 0, doc_hi = 0;  // the docs this context evaluates (tq_segment_set_doc_range; [0, max_doc) by default)
  Arena arena;  // block tables + aligned block copies of this segment's posting lists; freed with the segment
  uint8_t* d_pos = nullptr;  // the field's `.pos` sub-file (phrase queries), padded
  size_t pos_len = 0;
  uint8_t* d_pos_pool = nullptr;  // position tables of this segment's terms, bump-allocated by k_build_pos_tables
  size_t pos_pool_cap = 0;        // (the first 8 bytes of the pool are the cursor)
};

// A run of tiles [t0, t1) that a filtered query visits.
struct TileRun { uint32_t t0, t1; };

// What a filtered query (TQ_QUERY_FILTER) reads of one (filter, segment, field): alive AND doc range AND filter on the device
// (k_filter_combine, padded like the alive copy: k_count reads whole 32-bit words), and the tiles it leaves
// non-empty, from the host bits and the doc range: runs of 1024-doc tiles of the tile engine (gaps of up to kRunGap empty tiles
// merged, since every unit pays a cursor prologue) and of k_count's 8192-doc tiles.  Built at first use, rebuilt by
// tq_segment_set_doc_range, dropped with the segment or the filter.
struct FilterView {
  uint8_t* d_bits = nullptr;
  std::vector<TileRun> runs, count_runs;
};

// A sort column of one (column_id, segment_ord) (tq_sort_column_register): the u64 images on the device, the present bits (padded
// to whole 8192-doc tiles: k_sort reads a tile's words whole) and the bounds of every 8192-doc tile, on the device for k_sort and
// on the host for the planner, which runs a query's units by descending bound.
// A histogram reads the same column as f64; for TQ_FAST_F64 the planner also needs the bounds of each tile's finite values and
// whether it holds -inf / +inf (finite), since the image bounds of a tile with an infinity or a NaN say nothing of its range.
struct FiniteTile {
  unsigned long long lo, hi;  // smallest and largest image of the tile's finite f64 values (kFiniteAny)
  uint32_t flags;
};
constexpr uint32_t kFiniteAny = 1, kFiniteNegInf = 2, kFinitePosInf = 4;
struct SortColumn {
  unsigned long long* d_values = nullptr;
  uint32_t* d_present = nullptr;  // null: every doc has a value
  SortTile* d_tiles = nullptr;
  std::vector<SortTile> tiles;
  std::vector<FiniteTile> finite;
  unsigned long long min_image = ~0ull, max_image = 0;  // over every doc with a value (none: min_image > max_image)
  void release() { cudaFree(d_values); cudaFree(d_present); cudaFree(d_tiles); d_values = nullptr; d_present = nullptr; d_tiles = nullptr; }
};

// A cache of device tables built at first use (block tables of posting lists, position tables): key -> table id, the ids of
// dropped entries reused first.  An entry the current call schedules takes its id at once (later lookups of the same key share
// it) and stays pending until the call builds the pending tables together (flush_tables, tq_engine.cu) or rolls them back: a
// failed call leaves no entry behind.  ctx->mu held throughout.
template <class Key, class Hash, class Job>
struct TableCache {
  struct Pending { Key key; uint32_t id; Job build; };
  std::unordered_map<Key, uint32_t, Hash> ids;
  std::vector<uint32_t> free_ids;
  std::vector<Pending> pending;
  uint32_t cap = 0, n_ids = 0;

  const uint32_t* find(const Key& key) const {
    auto it = ids.find(key);
    return it == ids.end() ? nullptr : &it->second;
  }
  bool full() const { return free_ids.empty() && n_ids >= cap; }
  // Takes an id for key and schedules its table; the caller fills in what the build kernel reads.
  Job& schedule(const Key& key, uint32_t* id) {
    if (!free_ids.empty()) { *id = free_ids.back(); free_ids.pop_back(); }
    else *id = n_ids++;
    ids.emplace(key, *id);
    pending.push_back(Pending{key, *id, Job{}});
    return pending.back().build;
  }
  // Takes back every scheduled table that was not built: its entry would hand an unbuilt table to the next query on the key.
  void rollback() {
    for (auto& p : pending) {
      auto it = ids.find(p.key);
      if (it != ids.end() && it->second == p.id) ids.erase(it);
      free_ids.push_back(p.id);
    }
    pending.clear();
  }
  // Drops the entries whose key satisfies pred (an unregistered segment's); their ids are reused.
  template <class Pred>
  void drop(Pred pred) {
    for (auto it = ids.begin(); it != ids.end();)
      if (pred(it->first)) { free_ids.push_back(it->second); it = ids.erase(it); } else ++it;
  }
};

// A block table as it is scheduled: the k_build_tables job and the descriptor it starts from.
struct ListBuild { BuildJob job; ListDesc desc; };

}  // namespace tq::host

struct tq_ctx {
  int device = 0;
  std::mutex mu;  // guards segments, list cache, arena, batch pool, stats
  std::map<std::pair<uint32_t, uint32_t>, tq::host::Segment> segments;
  tq::ListDesc* d_lists = nullptr;
  tq::host::TableCache<tq::host::ListKey, tq::host::ListKeyHash, tq::host::ListBuild> list_tables;  // block tables: ListDesc ids
  tq::PosDesc* d_pos_descs = nullptr;  // position tables (phrase queries), same life cycle as the block tables
  tq::host::TableCache<tq::host::PosKey, tq::host::PosKeyHash, tq::PosJob> pos_tables;  // PosDesc ids
  std::map<std::pair<uint32_t, uint32_t>, uint32_t> seg_users;  // (segment, field) -> prepared batches not yet destroyed that name it
  std::map<std::pair<uint32_t, uint32_t>, std::vector<uint8_t>> filters;  // (filter_id, segment_ord) -> the caller's bits, ceil(max_doc / 8) bytes
  std::map<std::tuple<uint32_t, uint32_t, uint32_t>, tq::host::FilterView> filter_views;  // (filter_id, segment_ord, field)
  std::map<uint32_t, uint32_t> filter_users;  // filter_id -> prepared batches not yet destroyed that name it
  std::map<std::pair<uint32_t, uint32_t>, tq::host::SortColumn> sort_columns;  // (column_id, segment_ord)
  std::map<uint32_t, uint32_t> sort_users;  // column_id -> sort runs in progress that read it
  // cumulative tq_stats fields of the sort runs (sort_ms, units_sort, sort_tiles_seen, sort_tiles_skipped)
  double sort_ms = 0;
  uint64_t sort_units = 0, sort_tiles_seen = 0, sort_tiles_skipped = 0;
  // ... and of the histogram runs (hist_ms, units_hist, hist_tiles_seen, hist_tiles_one_bucket)
  double hist_ms = 0;
  uint64_t hist_units = 0, hist_tiles_seen = 0, hist_tiles_one_bucket = 0;
  // ... and of the terms runs (terms_ms, units_terms, terms_tiles_seen, terms_tiles_one_key)
  double terms_ms = 0;
  uint64_t terms_units = 0, terms_tiles_seen = 0, terms_tiles_one_key = 0;
  // ... and of the metrics runs (metrics_ms, units_metrics, metrics_tiles_seen, metrics_tiles_one_value)
  double metrics_ms = 0;
  uint64_t metrics_units = 0, metrics_tiles_seen = 0, metrics_tiles_one_value = 0;
  // ... and of the histogram-with-metrics runs (hist_metrics_ms, units_hist_metrics, tiles seen / in one bucket, flushes)
  double hist_metrics_ms = 0;
  uint64_t hist_metrics_units = 0, hist_metrics_tiles_seen = 0, hist_metrics_tiles_one_bucket = 0, hist_metrics_flush_shared = 0,
           hist_metrics_flush_global = 0;
  // ... and of the terms-with-metrics runs (terms_metrics_ms, units, tiles seen / with one kept key, waves)
  double terms_metrics_ms = 0;
  uint64_t terms_metrics_units = 0, terms_metrics_tiles_seen = 0, terms_metrics_tiles_one_key = 0, terms_metrics_waves = 0;
  // ... and of the range runs, with and without metrics (range_ms, units, tiles seen / in one bucket)
  double range_ms = 0;
  uint64_t range_units = 0, range_tiles_seen = 0, range_tiles_one_bucket = 0;
  // ... and of the terms-with-histogram runs (terms_hist_ms, units, tiles seen / with one kept key / in one bucket / both, waves,
  // k_terms_hist units counting in shared memory / in the grid)
  double terms_hist_ms = 0;
  uint64_t terms_hist_units = 0, terms_hist_tiles_seen = 0, terms_hist_tiles_one_key = 0, terms_hist_tiles_one_bucket = 0,
           terms_hist_tiles_both = 0, terms_hist_waves = 0, terms_hist_units_shared = 0, terms_hist_units_global = 0;
  // ... and of the histogram-with-terms runs (hist_terms_ms, CTAs, tiles seen / with one key / in one bucket / both, k_hist_terms
  // units counting in shared memory / in the grid, rows cut on the device, waves)
  double hist_terms_ms = 0;
  uint64_t hist_terms_units = 0, hist_terms_tiles_seen = 0, hist_terms_tiles_one_key = 0, hist_terms_tiles_one_bucket = 0,
           hist_terms_tiles_both = 0, hist_terms_units_shared = 0, hist_terms_units_global = 0, hist_terms_rows_cut = 0, hist_terms_waves = 0;
  cudaStream_t build_stream = nullptr;
  tq::host::PinBuf build_pin;
  tq::host::DevBuf build_dev;
  std::vector<tq_batch*> pool;
  tq_stats stats{};
  uint32_t term_blocks_per_unit, and_blocks_per_unit, or_tiles_per_unit, strip_windows_per_unit, count_hits_tiles_per_unit;
  uint32_t terms_counter_budget;  // u32 counters one tq_terms_batch wave may hold
  uint32_t hist_metrics_budget;   // (bucket, column) accumulators one tq_histogram_metrics_batch wave may hold
  uint32_t terms_metrics_budget;  // (kept entry, column) parts one tq_terms_metrics_batch wave may hold
  uint32_t terms_hist_budget;     // u32 (kept entry, bucket) cells one tq_terms_histogram_batch wave may hold
  uint32_t hist_terms_budget;     // u32 (bucket, key) cells one tq_histogram_terms_batch wave, and one (query, segment), may hold
  unsigned long long* d_counters = nullptr;  // [0..8) k_or_strip windows by route and bytes read, [8..16) k_tile diagnostics, [16..24) k_tile cycles by stage,
                                             // [24..28) k_tile B2 union postings by exit
  uint32_t tile = 1, tile_scratch_mb = 24576, tile_sample_div = 64, tile_round_div1 = 8, tile_round_div2 = 2, tile_light_max = 384, tile_counters = 0;
  uint32_t tile_ops = 7;  // bit per TQ_OP_*: which query shapes the tile engine takes
  uint32_t tile_seg_cap_hook = 0;
  uint32_t tile_windows = 0;
  uint32_t phrase_side = 1;
  uint32_t tile_terms = 2;
  uint32_t tile_max_slots = tq::kTileMaxSlots, tile_max_queries = tq::kTileMaxQueries, tile_wide_queries = 256;
  uint64_t tile_smem_last = 0, tile_ctas_last = 0;
  uint32_t tile_cand_floor = 32768, tile_max_dens_x1000 = 0, tile_pcap_hook = 0, tile_big_min = 6, tile_units = 0;
  uint32_t target_units = 0;  // CTAs a batch's per-query units aim for (4 x 32 per SM)
};

#define TQ_CUDA(expr)                                                                         \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      tq::host::set_last_error(std::string(#expr) + ": " + cudaGetErrorString(_e));           \
      return TQ_ERR_CUDA;                                                                     \
    }                                                                                         \
  } while (0)

namespace tq::host {

// The block table of a posting list: its id from the cache, or a new id with the build scheduled.  *seg_out: the list's segment.
int get_list(tq_ctx* c, const tq_term_seg& ts, bool ignore_freq, uint32_t* list_id, const Segment** seg_out);
// The position table of one (term, segment), likewise.
int get_pos(tq_ctx* c, const tq_term_seg& ts, const tq_term_pos& tp, uint32_t* pos_id);
// Every segment a filtered query names has a bitset for its filter.
int check_filter(const tq_ctx* c, const tq_query& q);
// The docs query q may collect in segment s: its alive bitset, or for a filtered query the (filter, segment, field) view, built at
// first use.  *view: null for an unfiltered query.
int query_alive(tq_ctx* c, const tq_query& q, const Segment& s, const uint8_t** alive, const FilterView** view);

}  // namespace tq::host
