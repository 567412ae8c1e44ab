// Host engine behind the C ABI of include/tantivy_b200.h, and the only translation unit with kernels: context lifecycle, the
// segment and filter registry, the device table caches and their builds, batch layout and launches, the phases of a run,
// result hand-over, Count, codec access and the device merge.  Batch planning is in tq_plan.cpp, tq_multi in tq_multi.cpp.
//
// Replaces, for TermQuery / all-MUST / all-SHOULD BooleanQuery of TermQuerys collected by
// TopDocs::order_by_score, the reference's per-segment loop
//   Searcher::search_with_executor            src/core/searcher.rs:220-237
//   SortBySimilarityScore::collect_segment_top_k   src/collector/sort_key/sort_by_score.rs:35-66
//   Weight::for_each_pruning                  src/query/weight.rs:123-132
//   TopBySortKeyCollector::merge_fruits       src/collector/sort_key_top_collector.rs:54-60
// There is NO CPU fallback: without a CUDA device every entry point fails with TQ_ERR_CUDA.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "tq_plan.hpp"
#include "tq_tile.cuh"
#include "tq_phrase.cuh"

using namespace tq;
using namespace tq::host;

static constexpr size_t kOrDynSmem = kTileDocs * sizeof(float) + kTileDocs;  // score slots + fieldnorm bytes

namespace tq::host {

namespace {
thread_local std::string g_err;
}  // namespace

void set_last_error(const std::string& msg) { g_err = msg; }
const std::string& last_error() { return g_err; }

bool filter_in_use(tq_ctx* c, uint32_t filter_id) {
  std::lock_guard<std::mutex> g(c->mu);
  return c->filter_users.count(filter_id) != 0;
}

}  // namespace tq::host

static constexpr uint32_t kRunGap = 4;

static uint32_t env_u32(const char* name, uint32_t def) {
  const char* v = getenv(name);
  if (!v || !*v) return def;
  return (uint32_t)strtoul(v, nullptr, 10);
}

constexpr int kCounterWords = 8 + kTileStatWords;  // tq_ctx::d_counters (k_tile adds to those from word 8 on)

// The k_tile instances, indexed sample launch << 2 | counters << 1 | union-only (tile_kernel).
using TileKernel = void (*)(const BatchParams, const TileParams, uint32_t);
static const TileKernel kTileKernels[8] = {k_tile<false, false, false>, k_tile<false, false, true>, k_tile<false, true, false>, k_tile<false, true, true>,
                                           k_tile<true, false, false>,  k_tile<true, false, true>,  k_tile<true, true, false>,  k_tile<true, true, true>};
static TileKernel tile_kernel(bool sample, bool counters, bool union_only) {
  return kTileKernels[(sample ? 4 : 0) + (counters ? 2 : 0) + (union_only ? 1 : 0)];
}

// Appends n elements at src to v and points at the copy (null stays null).  v's capacity must hold them: earlier copies stay put.
template <class T>
static const T* keep(std::vector<T>& v, const T* src, size_t n) {
  if (!src) return nullptr;
  const size_t at = v.size();
  v.insert(v.end(), src, src + n);
  return v.data() + at;
}

// Deep copy of a batch's queries (only kept when the tile engine runs them: an overflowing run is repeated, see finalize_run).
struct OwnedQueries {
  std::vector<tq_query> q;
  std::vector<tq_term_seg> ts;
  std::vector<float> w, avg, cache;
  std::vector<uint8_t> flags;
  std::vector<tq_term_pos> tp;
  std::vector<uint32_t> toff;
  void assign(const tq_query* queries, size_t nq) {
    size_t n_ts = 0, n_t = 0, n_cache = 0;
    for (size_t qi = 0; qi < nq; ++qi) {
      n_ts += queries[qi].n_term_segs;
      n_t += queries[qi].n_terms;
      if (queries[qi].tf_cache) n_cache += 256 * (size_t)queries[qi].n_terms;
    }
    ts.reserve(n_ts); tp.reserve(n_ts);
    w.reserve(n_t); avg.reserve(n_t); flags.reserve(n_t); toff.reserve(n_t);
    cache.reserve(n_cache);
    q.assign(queries, queries + nq);
    for (tq_query& d : q) {
      d.term_segs = keep(ts, d.term_segs, d.n_term_segs);
      d.term_pos = keep(tp, d.term_pos, d.n_term_segs);
      d.weight = keep(w, d.weight, d.n_terms);
      d.avg_fieldnorm = keep(avg, d.avg_fieldnorm, d.n_terms);
      d.tf_cache = keep(cache, d.tf_cache, 256 * (size_t)d.n_terms);
      d.term_flags = keep(flags, d.term_flags, d.n_terms);
      d.term_offset = keep(toff, d.term_offset, d.n_terms);
    }
  }
};

struct tq_batch {
  struct Span { cudaEvent_t a = nullptr, b = nullptr; int kind = 0; };
  struct TileGroup {
    TileParams params{};
    uint32_t n_chunks = 0;
    uint32_t unit_base[kTileRounds] = {0, 0, 0, 0}, n_units[kTileRounds] = {0, 0, 0, 0};
    size_t smem = 0;
    bool union_only = false;  // the group's queries are all term queries and unions: the k_tile<*, *, true> instances run it
    CountTileParams count{};  // k_count_tiles: the group's TQ_QUERY_COUNT_HITS queries
    uint32_t n_count_units = 0;
    size_t count_smem = 0;
    std::vector<uint32_t> count_queries;  // batch ordinals of those queries (recounted by k_count if count.overflow is set)
  };
  tq_ctx* ctx = nullptr;
  cudaStream_t stream = nullptr;
  cudaStream_t side = nullptr;             // k_phrase runs here, next to the tile engine's launches on `stream`
  cudaEvent_t ev_side0 = nullptr, ev_side1 = nullptr;
  bool side_pending = false;               // `stream` has not waited for ev_side1 yet
  cudaEvent_t ev_start = nullptr, ev_k0 = nullptr, ev_k1 = nullptr, ev_end = nullptr;
  std::vector<Span> spans;  // per-kind kernel times of the current run (events are created once and reused)
  size_t n_spans = 0;
  std::vector<TileGroup> groups;
  OwnedQueries owned;
  DevBuf tile_dev;  // pair arrays, tile indexes, samples, flags of the tile engine
  uint32_t* flags_pin = nullptr;  // [0] tile buffer overflow, [1] candidate region overflow (read back after the last phase)
  size_t tile_zero_off = 0, tile_zero_bytes = 0, tile_flags_off = 0;
  bool finalized = false, last_round_sampled = false;
  int repeat = 0;  // 0: a caller's batch; 1, 2: the repeat of an overflowed run (batch_prepare_impl)
  PinBuf pin;      // staged descriptors (H2D source)
  DevBuf dev;      // descriptors on device
  DevBuf scratch;  // qstate + candidates + results
  PinBuf res_pin;  // results (D2H target)
  BatchParams params{};
  size_t desc_bytes = 0;
  uint32_t nq = 0, kmax = 0;
  uint32_t n_units[UC_CLASSES] = {}, unit_base[UC_CLASSES] = {};  // per UnitClass
  uint32_t phrase_ct = 2;                 // most terms of a phrase in the batch (k_phrase's candidate stride)
  const PhraseAux* phrase_aux = nullptr;  // device: per clause of the batch's phrase queries (parallel to qlists)
  uint32_t strip_cached_max = 0;
  size_t qinit_off = 0;
  int next_phase = 0;  // of the current run (0: none started)
  size_t qstate_off = 0, cands_off = 0, res_off = 0, res_bytes = 0, n_cands = 0;
  struct { size_t scores, segs, docs, counts; } res_at{};  // the result columns inside the res_bytes at res_off (and in res_pin)
  tq_stats stats{};
  bool ran = false;
  // TQ_QUERY_COUNT_HITS: per-query hit counters (u64 [nq]) and the groups' overflow words (u32 [groups]) in `scratch` at hits_off,
  // zeroed by phase 0; k_count for the queries on the per-query kernels; hits_host = their doc_freq shortcuts
  bool count_hits = false;
  size_t hits_off = 0, hits_bytes = 0;
  CountParams count_p{};
  uint32_t n_count_units = 0;
  bool count_mixed = false;  // k_count<true>: some pair has SHOULD or MUST_NOT clauses
  std::vector<uint64_t> hits_host;
  PinBuf hits_pin;
  std::vector<std::pair<uint32_t, uint32_t>> held;  // the (segment, field)s its queries name, counted in tq_ctx::seg_users until destroyed
  std::vector<uint32_t> held_filters;               // the filters its queries name, counted in tq_ctx::filter_users until destroyed
  std::vector<uint32_t> held_columns;               // tq_sort_batch: the sort columns it reads, counted in tq_ctx::sort_users
};

// host twin of score_to_key (tq_device.cuh): order-preserving u32 image of a float, -0.0 and +0.0 on one key
static uint32_t host_score_key(float f) {
  uint32_t u;
  f += 0.0f;
  memcpy(&u, &f, 4);
  return u ^ ((u >> 31) ? 0xFFFFFFFFu : 0x80000000u);
}

// ---- per-query doc filters (TQ_QUERY_FILTER) -----------------------------------------------------------------------------------
// Is any bit of docs [a, b) set?
static bool any_bit(const uint8_t* bits, uint64_t a, uint64_t b) {
  for (; a < b && (a & 7u); ++a) if ((bits[a >> 3] >> (a & 7u)) & 1u) return true;
  for (; a + 64 <= b; a += 64) { uint64_t w; memcpy(&w, bits + (a >> 3), 8); if (w) return true; }
  for (; a + 8 <= b; a += 8) if (bits[a >> 3]) return true;
  for (; a < b; ++a) if ((bits[a >> 3] >> (a & 7u)) & 1u) return true;
  return false;
}

// The `tile`-doc tiles of the docs [lo, hi) that hold a set bit, as runs; runs at most `gap` empty tiles apart are merged.
static std::vector<TileRun> tile_runs(const uint8_t* bits, uint32_t lo, uint32_t hi, uint32_t tile, uint32_t gap) {
  std::vector<TileRun> runs;
  if (lo >= hi) return runs;
  const uint32_t t_lo = lo / tile, t_hi = (uint32_t)(((uint64_t)hi + tile - 1) / tile);
  for (uint32_t t = t_lo; t < t_hi; ++t) {
    const uint64_t a = std::max<uint64_t>(lo, (uint64_t)t * tile), b = std::min<uint64_t>(hi, (uint64_t)(t + 1) * tile);
    if (!any_bit(bits, a, b)) continue;
    if (!runs.empty() && t - runs.back().t1 <= gap) runs.back().t1 = t + 1;
    else runs.push_back(TileRun{t, t + 1});
  }
  return runs;
}

// (Re)builds the view of one (filter, segment, field) from the filter's host bits, the segment's alive bitset and its doc range.
// ctx->mu held; nothing on the device reads the view meanwhile (a first build, or tq_segment_set_doc_range after its device sync).
static int build_view(tq_ctx* c, const Segment& s, const std::vector<uint8_t>& bits, FilterView& v) {
  const size_t nbytes = ((size_t)s.max_doc + 7) / 8, padded = ((nbytes + 7) & ~(size_t)7) + 8;
  const uint32_t n_words = (uint32_t)(((uint64_t)s.max_doc + 31) / 32);
  if (!v.d_bits) TQ_CUDA(cudaMalloc(&v.d_bits, padded));
  TQ_CUDA(c->build_dev.ensure(padded));
  TQ_CUDA(cudaMemsetAsync(c->build_dev.p, 0, padded, c->build_stream));
  if (nbytes) TQ_CUDA(cudaMemcpyAsync(c->build_dev.p, bits.data(), std::min(nbytes, bits.size()), cudaMemcpyHostToDevice, c->build_stream));
  TQ_CUDA(cudaMemsetAsync(v.d_bits, 0, padded, c->build_stream));
  if (n_words)
    k_filter_combine<<<(n_words + 255) / 256, 256, 0, c->build_stream>>>(reinterpret_cast<const uint32_t*>(s.d_alive), reinterpret_cast<const uint32_t*>(c->build_dev.p),
                                                                         n_words, s.doc_lo, s.doc_hi, reinterpret_cast<uint32_t*>(v.d_bits));
  TQ_CUDA(cudaGetLastError());
  TQ_CUDA(cudaStreamSynchronize(c->build_stream));
  v.runs = tile_runs(bits.data(), s.doc_lo, s.doc_hi, kTile, kRunGap);
  v.count_runs = tile_runs(bits.data(), s.doc_lo, s.doc_hi, kTileDocs, 0);
  return TQ_OK;
}

namespace tq::host {

int check_filter(const tq_ctx* c, const tq_query& q) {
  if (!(q.flags & TQ_QUERY_FILTER)) return TQ_OK;
  for (uint32_t i = 0; i < q.n_term_segs; ++i)
    if (!c->filters.count({q.filter_id, q.term_segs[i].segment_ord}))
      return fail(TQ_ERR_NOT_FOUND, "a filtered query names a segment without a bitset for its filter (tq_filter_register)");
  return TQ_OK;
}

int query_alive(tq_ctx* c, const tq_query& q, const Segment& s, const uint8_t** alive, const FilterView** view) {
  *view = nullptr;
  *alive = s.d_alive;
  if (!(q.flags & TQ_QUERY_FILTER)) return TQ_OK;
  auto fit = c->filters.find({q.filter_id, s.segment_ord});
  if (fit == c->filters.end()) return fail(TQ_ERR_NOT_FOUND, "a filtered query names a segment without a bitset for its filter (tq_filter_register)");
  const auto key = std::make_tuple(q.filter_id, s.segment_ord, s.field);
  auto it = c->filter_views.find(key);
  if (it == c->filter_views.end()) {
    FilterView v;
    const int rc = build_view(c, s, fit->second, v);
    if (rc != TQ_OK) { cudaFree(v.d_bits); return rc; }
    it = c->filter_views.emplace(key, std::move(v)).first;
  }
  *view = &it->second;
  *alive = it->second.d_bits;
  return TQ_OK;
}

}  // namespace tq::host

// Frees the views whose (filter_id, segment_ord, field) satisfies pred.  ctx->mu held, the device idle.
template <class Pred>
static void drop_views(tq_ctx* c, Pred pred) {
  for (auto it = c->filter_views.begin(); it != c->filter_views.end();)
    if (pred(it->first)) { cudaFree(it->second.d_bits); it = c->filter_views.erase(it); } else ++it;
}

extern "C" {

const char* tq_last_error(tq_ctx*) { return g_err.c_str(); }

int tq_ctx_create(int device, tq_ctx** out) {
  if (!out) return fail(TQ_ERR_INVALID_ARGUMENT, "out is null");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    return fail(TQ_ERR_CUDA, std::string("no CUDA device: the GPU path has no CPU fallback (") + cudaGetErrorString(e) + ")");
  if (device < 0 || device >= n) return fail(TQ_ERR_INVALID_ARGUMENT, "bad device ordinal");
  TQ_CUDA(cudaSetDevice(device));
  int sms = 0;
  TQ_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  size_t free_bytes = 0, total_bytes = 0;
  TQ_CUDA(cudaMemGetInfo(&free_bytes, &total_bytes));
  auto* c = new tq_ctx();
  c->device = device;
  c->list_tables.cap = env_u32("TQ_MAX_LISTS", 1u << 20);
  c->term_blocks_per_unit = env_u32("TQ_TERM_BLOCKS_PER_UNIT", 512);
  c->and_blocks_per_unit = env_u32("TQ_AND_BLOCKS_PER_UNIT", 128);
  c->or_tiles_per_unit = env_u32("TQ_OR_TILES_PER_UNIT", 16);
  // test hook: smallest k_or_strip unit, in kWin-doc windows (1 or 7: warps with no window or one, unit and strip edges in small segments)
  c->strip_windows_per_unit = std::max<uint32_t>(1u, env_u32("TQ_STRIP_WINDOWS_PER_UNIT", kStripWarps * 64u));
  // test hook: smallest k_count_tiles unit, in tiles (1: every tile edge is a unit edge, where the sparse cursors are searched)
  c->count_hits_tiles_per_unit = std::max<uint32_t>(1u, env_u32("TQ_COUNT_HITS_TILES_PER_UNIT", 8));
  // terms counters per wave of tq_terms_batch (256 MB); test hook: a small budget runs a batch in many waves
  c->terms_counter_budget = std::max<uint32_t>(1u, env_u32("TQ_TERMS_COUNTER_BUDGET", 1u << 26));
  c->hist_metrics_budget = std::max<uint32_t>(1u, env_u32("TQ_HIST_METRICS_BUDGET", 1u << 22));
  c->terms_metrics_budget = std::max<uint32_t>(1u, env_u32("TQ_TERMS_METRICS_BUDGET", 1u << 22));
  // histogram cells per wave of tq_terms_histogram_batch (64 MB of grid, 128 MB of cell list); test hook: a small budget runs a
  // batch in many waves and refuses a wide (query, segment)
  c->terms_hist_budget = std::min<uint32_t>(1u << 28, std::max<uint32_t>(1u, env_u32("TQ_TERMS_HIST_BUDGET", 1u << 24)));
  // (bucket, key) cells per wave and per (query, segment) of tq_histogram_terms_batch (64 MB of grid, 128 MB each of entry scratch
  // and entry list); test hook: a small budget runs a batch in many waves and refuses a wide (query, segment)
  c->hist_terms_budget = std::min<uint32_t>(1u << 28, std::max<uint32_t>(1u, env_u32("TQ_HIST_TERMS_BUDGET", 1u << 24)));
  c->tile = env_u32("TQ_TILE", 1);                          // unions take the shared-decode tile engine (tq_tile.cuh); 0 = per-query kernels only
  // (doc, score) pairs one batch may materialise: an eighth of the device memory (10 GB on an 80 GB H100), so that the
  // four batches bench.py keeps prepared fit next to the index; queries past the budget run on the per-query kernels
  c->tile_scratch_mb = env_u32("TQ_TILE_SCRATCH_MB", (uint32_t)(total_bytes / 8 >> 20));
  // share of the tiles in the sample launch (0/1: none).  1/64: the running threshold of the exact launches raises what the
  // samples leave within a few tiles, so a sample launch over twice the tiles costs more than its better seed saves (DESIGN §6)
  c->tile_sample_div = env_u32("TQ_TILE_SAMPLE_DIV", 64);
  c->tile_round_div1 = env_u32("TQ_TILE_ROUND_DIV1", 8);     // the exact launches end at 1/8, 1/2 and all of a segment's tiles
  c->tile_round_div2 = env_u32("TQ_TILE_ROUND_DIV2", 2);
  // essential postings up to which a (query, tile) pair is evaluated posting by posting.  Above it a pair takes one of the
  // CTA's two window warps while its other six wait at the barrier after B3; B2 deals the postings of a pair of a few hundred
  // to all eight warps, so only the largest pairs are worth a window (DESIGN §6)
  c->tile_light_max = env_u32("TQ_TILE_LIGHT_MAX", 384);
  c->tile_counters = env_u32("TQ_TILE_COUNTERS", 0);         // diagnostics (tile_counters of tq_stats)
  c->tile_ops = env_u32("TQ_TILE_OPS", 7);                  // bit 0 term, 1 AND, 2 OR
  c->tile_cand_floor = env_u32("TQ_TILE_CAND_FLOOR", 32768);  // smallest candidate region of a tile query (test hook: tiny regions overflow)
  c->tile_max_dens_x1000 = env_u32("TQ_TILE_MAX_DENS_X1000", 0);  // test hook: cap on a group's pairs per 1000 docs (forces several groups)
  c->tile_pcap_hook = env_u32("TQ_TILE_PCAP", 0);            // test hook: tile buffer size (forces overflowing tiles)
  c->tile_seg_cap_hook = env_u32("TQ_TILE_SEG_CAP", 0);      // test hook: entries of the per-tile work list (forces extra routing rounds)
  c->tile_max_slots = std::min<uint32_t>(kTileMaxSlots, std::max<uint32_t>(64u, env_u32("TQ_TILE_MAX_SLOTS", kTileMaxSlots)));  // distinct lists of one segment per group (shared memory per CTA grows by 12 B per list)
  c->tile_max_queries = std::min<uint32_t>(kTileMaxQueries, std::max<uint32_t>(1u, env_u32("TQ_TILE_MAX_QUERIES", kTileMaxQueries)));  // queries of one segment per group
  c->tile_wide_queries = std::max<uint32_t>(1u, env_u32("TQ_TILE_WIDE_QUERIES", 256));  // ... for queries of more than 8 terms
  c->tile_terms = env_u32("TQ_TILE_TERMS", 2);               // single-term queries on the tile engine: 0 never, 1 always, 2 when the batch has multi-term queries
  c->phrase_side = env_u32("TQ_PHRASE_SIDE_STREAM", 1);      // k_phrase on the batch's second stream, next to the tile engine
  c->tile_windows = env_u32("TQ_TILE_WINDOWS", 0);           // warps with a window for the heavy pairs (0 = kTileExactWindows)
  c->tile_big_min = env_u32("TQ_TILE_BIG_MIN", 6);          // expected pairs per tile from which a list gets a tile index
  c->tile_units = env_u32("TQ_TILE_UNITS", 6u * sms);        // CTAs an exact launch aims for
  c->target_units = env_u32("TQ_TARGET_UNITS", 4u * 32u * sms);
  cudaError_t err = cudaMalloc(&c->d_lists, (size_t)c->list_tables.cap * sizeof(ListDesc));
  if (err == cudaSuccess) err = cudaMemset(c->d_lists, 0, (size_t)c->list_tables.cap * sizeof(ListDesc));
  c->pos_tables.cap = env_u32("TQ_MAX_POS_LISTS", 1u << 18);
  if (err == cudaSuccess) err = cudaMalloc(&c->d_pos_descs, (size_t)c->pos_tables.cap * sizeof(PosDesc));
  if (err == cudaSuccess) err = cudaMemset(c->d_pos_descs, 0, (size_t)c->pos_tables.cap * sizeof(PosDesc));
  if (err == cudaSuccess) err = cudaFuncSetAttribute(k_phrase, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)phrase_smem_bytes(kPhraseMaxTerms));
  if (err == cudaSuccess) err = cudaMalloc(&c->d_counters, kCounterWords * sizeof(unsigned long long));
  if (err == cudaSuccess) err = cudaMemset(c->d_counters, 0, kCounterWords * sizeof(unsigned long long));
  if (err == cudaSuccess) err = cudaStreamCreateWithFlags(&c->build_stream, cudaStreamNonBlocking);
  if (err == cudaSuccess) err = cudaFuncSetAttribute(k_or, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kOrDynSmem);
  if (err == cudaSuccess) err = cudaFuncSetAttribute(k_or_strip, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)strip_smem_bytes(kMaxCached));
  // k_tile's occupancy is bound by shared memory: ask for the largest carveout so that the SM's full 228 KB is there to share
  for (auto kern : kTileKernels) {
    if (err == cudaSuccess) err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTileMaxSmem);
    if (err == cudaSuccess) err = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
  }
  if (err != cudaSuccess) { delete c; return fail(TQ_ERR_CUDA, cudaGetErrorString(err)); }
  *out = c;
  return TQ_OK;
}

void tq_batch_destroy_real(tq_batch* b) {
  if (!b) return;
  cudaSetDevice(b->ctx->device);
  if (b->stream) cudaStreamSynchronize(b->stream);
  if (b->side) { cudaStreamSynchronize(b->side); cudaStreamDestroy(b->side); }
  if (b->ev_side0) cudaEventDestroy(b->ev_side0);
  if (b->ev_side1) cudaEventDestroy(b->ev_side1);
  b->pin.release(); b->dev.release(); b->scratch.release(); b->res_pin.release(); b->tile_dev.release(); b->hits_pin.release();
  if (b->flags_pin) cudaFreeHost(b->flags_pin);
  if (b->ev_start) cudaEventDestroy(b->ev_start);
  if (b->ev_k0) cudaEventDestroy(b->ev_k0);
  if (b->ev_k1) cudaEventDestroy(b->ev_k1);
  if (b->ev_end) cudaEventDestroy(b->ev_end);
  for (auto& sp : b->spans) { if (sp.a) cudaEventDestroy(sp.a); if (sp.b) cudaEventDestroy(sp.b); }
  if (b->stream) cudaStreamDestroy(b->stream);
  delete b;
}

void tq_ctx_destroy(tq_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  for (auto* b : c->pool) tq_batch_destroy_real(b);
  for (auto& kv : c->segments) {
    cudaFree(kv.second.d_idx); cudaFree(kv.second.d_fieldnorm); cudaFree(kv.second.d_alive);
    cudaFree(kv.second.d_pos); cudaFree(kv.second.d_pos_pool);
    kv.second.arena.release();
  }
  for (auto& kv : c->filter_views) cudaFree(kv.second.d_bits);
  for (auto& kv : c->sort_columns) kv.second.release();
  cudaFree(c->d_pos_descs);
  c->build_pin.release(); c->build_dev.release();
  if (c->build_stream) cudaStreamDestroy(c->build_stream);
  cudaFree(c->d_lists);
  cudaFree(c->d_counters);
  delete c;
}

int tq_get_stats(tq_ctx* c, tq_stats* out) {
  if (!c || !out) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(c->mu);
  *out = c->stats;
  out->lists_cached = c->list_tables.ids.size();
  cudaSetDevice(c->device);
  unsigned long long h[kCounterWords];
  if (cudaMemcpy(h, c->d_counters, sizeof(h), cudaMemcpyDeviceToHost) == cudaSuccess) {
    for (int i = 0; i < 8; ++i) { out->or_windows[i] = h[i]; out->tile_counters[i] = h[8 + i]; out->tile_cycles[i] = h[16 + i]; }
    for (int i = 0; i < kOrExits; ++i) out->tile_b2_exits[i] = h[24 + i];
  }
  out->tile_counters[7] = c->tile_smem_last;
  out->tile_ctas_per_sm = c->tile_ctas_last;
  out->sort_ms = (float)c->sort_ms;
  out->units_sort = c->sort_units;
  out->sort_tiles_seen = c->sort_tiles_seen;
  out->sort_tiles_skipped = c->sort_tiles_skipped;
  return TQ_OK;
}

int tq_get_histogram_stats(tq_ctx* c, tq_histogram_stats* out) {
  if (!c || !out) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(c->mu);
  out->hist_ms = (float)c->hist_ms;
  out->units_hist = c->hist_units;
  out->hist_tiles_seen = c->hist_tiles_seen;
  out->hist_tiles_one_bucket = c->hist_tiles_one_bucket;
  return TQ_OK;
}

int tq_get_terms_stats(tq_ctx* c, tq_terms_stats* out) {
  if (!c || !out) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(c->mu);
  out->terms_ms = (float)c->terms_ms;
  out->units_terms = c->terms_units;
  out->terms_tiles_seen = c->terms_tiles_seen;
  out->terms_tiles_one_key = c->terms_tiles_one_key;
  return TQ_OK;
}

int tq_get_metrics_stats(tq_ctx* c, tq_metrics_stats* out) {
  if (!c || !out) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(c->mu);
  out->metrics_ms = (float)c->metrics_ms;
  out->units_metrics = c->metrics_units;
  out->metrics_tiles_seen = c->metrics_tiles_seen;
  out->metrics_tiles_one_value = c->metrics_tiles_one_value;
  return TQ_OK;
}

int tq_get_hist_metrics_stats(tq_ctx* c, tq_hist_metrics_stats* out) {
  if (!c || !out) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(c->mu);
  out->hist_metrics_ms = (float)c->hist_metrics_ms;
  out->units_hist_metrics = c->hist_metrics_units;
  out->hist_metrics_tiles_seen = c->hist_metrics_tiles_seen;
  out->hist_metrics_tiles_one_bucket = c->hist_metrics_tiles_one_bucket;
  out->hist_metrics_flush_shared = c->hist_metrics_flush_shared;
  out->hist_metrics_flush_global = c->hist_metrics_flush_global;
  return TQ_OK;
}

int tq_get_terms_metrics_stats(tq_ctx* c, tq_terms_metrics_stats* out) {
  if (!c || !out) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(c->mu);
  out->terms_metrics_ms = (float)c->terms_metrics_ms;
  out->units_terms_metrics = c->terms_metrics_units;
  out->terms_metrics_tiles_seen = c->terms_metrics_tiles_seen;
  out->terms_metrics_tiles_one_key = c->terms_metrics_tiles_one_key;
  out->terms_metrics_waves = c->terms_metrics_waves;
  return TQ_OK;
}

int tq_get_terms_hist_stats(tq_ctx* c, tq_terms_hist_stats* out) {
  if (!c || !out) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(c->mu);
  out->terms_hist_ms = (float)c->terms_hist_ms;
  out->units_terms_hist = c->terms_hist_units;
  out->terms_hist_tiles_seen = c->terms_hist_tiles_seen;
  out->terms_hist_tiles_one_key = c->terms_hist_tiles_one_key;
  out->terms_hist_tiles_one_bucket = c->terms_hist_tiles_one_bucket;
  out->terms_hist_tiles_both = c->terms_hist_tiles_both;
  out->terms_hist_units_shared = c->terms_hist_units_shared;
  out->terms_hist_units_global = c->terms_hist_units_global;
  out->terms_hist_waves = c->terms_hist_waves;
  return TQ_OK;
}

int tq_get_hist_terms_stats(tq_ctx* c, tq_hist_terms_stats* out) {
  if (!c || !out) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(c->mu);
  out->hist_terms_ms = (float)c->hist_terms_ms;
  out->units_hist_terms = c->hist_terms_units;
  out->hist_terms_tiles_seen = c->hist_terms_tiles_seen;
  out->hist_terms_tiles_one_key = c->hist_terms_tiles_one_key;
  out->hist_terms_tiles_one_bucket = c->hist_terms_tiles_one_bucket;
  out->hist_terms_tiles_both = c->hist_terms_tiles_both;
  out->hist_terms_units_shared = c->hist_terms_units_shared;
  out->hist_terms_units_global = c->hist_terms_units_global;
  out->hist_terms_rows_cut = c->hist_terms_rows_cut;
  out->hist_terms_waves = c->hist_terms_waves;
  return TQ_OK;
}

int tq_get_range_stats(tq_ctx* c, tq_range_stats* out) {
  if (!c || !out) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(c->mu);
  out->range_ms = (float)c->range_ms;
  out->units_range = c->range_units;
  out->range_tiles_seen = c->range_tiles_seen;
  out->range_tiles_one_bucket = c->range_tiles_one_bucket;
  return TQ_OK;
}

int tq_segment_register(tq_ctx* c, uint32_t segment_ord, uint32_t field, uint32_t max_doc, int record_option,
                        const uint8_t* idx_body, size_t idx_len, const uint8_t* fieldnorm, size_t fieldnorm_len,
                        const uint8_t* alive_bitset, size_t alive_len) {
  if (!c || !idx_body || idx_len < 8) return fail(TQ_ERR_INVALID_ARGUMENT, "idx_body must hold the 8-byte header");
  if (record_option < 0 || record_option > 2) return fail(TQ_ERR_INVALID_ARGUMENT, "record_option");
  if (max_doc >= TQ_TERMINATED) return fail(TQ_ERR_INVALID_ARGUMENT, "max_doc");
  if (fieldnorm && fieldnorm_len < max_doc) return fail(TQ_ERR_INVALID_ARGUMENT, "fieldnorm shorter than max_doc");
  if (alive_bitset && alive_len * 8 < max_doc) return fail(TQ_ERR_INVALID_ARGUMENT, "alive bitset shorter than max_doc");
  TQ_CUDA(cudaSetDevice(c->device));
  std::lock_guard<std::mutex> g(c->mu);
  if (c->segments.count({segment_ord, field})) return fail(TQ_ERR_INVALID_ARGUMENT, "segment/field already registered");
  Segment s;
  s.segment_ord = segment_ord; s.field = field; s.max_doc = max_doc; s.record_option = record_option; s.idx_len = idx_len;
  s.doc_lo = 0; s.doc_hi = max_doc;
  const size_t pad = 256;  // decode_block reads one word past a block; the aligned block copy of k_build_tables reads 64 + 8 bytes past the last block
  cudaError_t e = cudaMalloc(&s.d_idx, idx_len + pad);
  if (e == cudaSuccess) e = cudaMemset(s.d_idx + idx_len, 0, pad);
  if (e == cudaSuccess) e = cudaMemcpy(s.d_idx, idx_body, idx_len, cudaMemcpyHostToDevice);
  if (e == cudaSuccess && fieldnorm) {
    const size_t padded = ((size_t)max_doc + kTileDocs - 1) / kTileDocs * kTileDocs + kTileDocs;  // k_or stages whole windows
    e = cudaMalloc(&s.d_fieldnorm, padded);
    if (e == cudaSuccess) e = cudaMemset(s.d_fieldnorm, 0, padded);
    if (e == cudaSuccess) e = cudaMemcpy(s.d_fieldnorm, fieldnorm, max_doc, cudaMemcpyHostToDevice);
  }
  if (e == cudaSuccess && alive_bitset) {
    const size_t alive_padded = ((alive_len + 7) & ~(size_t)7) + 8;  // k_count reads whole 32-bit words
    e = cudaMalloc(&s.d_alive, alive_padded);
    if (e == cudaSuccess) e = cudaMemset(s.d_alive, 0, alive_padded);
    if (e == cudaSuccess) e = cudaMemcpy(s.d_alive, alive_bitset, alive_len, cudaMemcpyHostToDevice);
  }
  if (e != cudaSuccess) {  // nothing of a half-registered segment stays behind
    cudaFree(s.d_idx); cudaFree(s.d_fieldnorm); cudaFree(s.d_alive);
    return fail(TQ_ERR_CUDA, std::string("segment upload: ") + cudaGetErrorString(e));
  }
  c->segments[{segment_ord, field}] = s;
  return TQ_OK;
}

int tq_segment_register_positions(tq_ctx* c, uint32_t segment_ord, uint32_t field, const uint8_t* pos_body, size_t pos_len) {
  if (!c || (!pos_body && pos_len)) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  std::lock_guard<std::mutex> g(c->mu);
  auto it = c->segments.find({segment_ord, field});
  if (it == c->segments.end()) return fail(TQ_ERR_NOT_FOUND, "segment/field not registered");
  Segment& s = it->second;
  if (s.record_option != TQ_RECORD_FREQS_POSITIONS) return fail(TQ_ERR_INVALID_ARGUMENT, "the field was not indexed with positions");
  if (s.d_pos) return fail(TQ_ERR_INVALID_ARGUMENT, "positions already registered");
  // table pool: 4 bytes per position block (<= 1 per 16 bytes of `.pos`), 8 per posting block, 512 + slack per term that is
  // ever queried as part of a phrase
  const size_t pool = pos_len / 4 + s.idx_len / 8 + (4u << 20);
  uint8_t *d_pos = nullptr, *d_pool = nullptr;
  cudaError_t e = cudaMalloc(&d_pos, pos_len + 256);
  if (e == cudaSuccess) e = cudaMemset(d_pos + pos_len, 0, 256);
  if (e == cudaSuccess && pos_len) e = cudaMemcpy(d_pos, pos_body, pos_len, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMalloc(&d_pool, pool);
  if (e == cudaSuccess) e = cudaMemset(d_pool, 0, 64);
  if (e == cudaSuccess) {
    const unsigned long long first = 64;  // the cursor lives in the pool's first word; tables start behind it
    e = cudaMemcpy(d_pool, &first, 8, cudaMemcpyHostToDevice);
  }
  if (e != cudaSuccess) { cudaFree(d_pos); cudaFree(d_pool); return fail(TQ_ERR_CUDA, std::string("positions upload: ") + cudaGetErrorString(e)); }
  s.d_pos = d_pos; s.pos_len = pos_len; s.d_pos_pool = d_pool; s.pos_pool_cap = pool;
  return TQ_OK;
}

// A single huge segment split by doc-id range over several contexts / GPUs (SURVEY.md §8e: every block's first and last doc is known
// from the skip list, so any doc range of a segment is a unit of work of its own; the reference's own parallel axis stops at whole
// segments, src/core/executor.rs:60-100).  Correctness rests on the alive bitset (docs outside the range are "deleted" for this
// context: every kernel already honours it); the speed-up comes from the tile engine, which only visits the tiles of the range.
int tq_segment_set_doc_range(tq_ctx* c, uint32_t segment_ord, uint32_t field, uint32_t doc_lo, uint32_t doc_hi) {
  if (!c) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  std::lock_guard<std::mutex> g(c->mu);
  auto it = c->segments.find({segment_ord, field});
  if (it == c->segments.end()) return fail(TQ_ERR_NOT_FOUND, "segment/field not registered");
  Segment& s = it->second;
  if (doc_lo > doc_hi || doc_hi > s.max_doc) return fail(TQ_ERR_INVALID_ARGUMENT, "doc range must satisfy lo <= hi <= max_doc");
  if (doc_lo < s.doc_lo || doc_hi > s.doc_hi) return fail(TQ_ERR_INVALID_ARGUMENT, "a doc range can only be narrowed");
  TQ_CUDA(cudaDeviceSynchronize());  // batches in flight read the bitset
  const size_t nbytes = ((size_t)s.max_doc + 7) / 8;
  if (!s.d_alive) {
    for (auto& kv : c->list_tables.ids)  // prepared batches keep the segment's (null) alive pointer: set the range before the first search
      if (kv.first.segment_ord == segment_ord && kv.first.field == field) return fail(TQ_ERR_INVALID_ARGUMENT, "set the doc range before the segment is searched");
    const size_t padded = ((nbytes + 7) & ~(size_t)7) + 8;
    uint8_t* d = nullptr;
    TQ_CUDA(cudaMalloc(&d, padded));
    cudaError_t e = cudaMemset(d, 0, padded);
    if (e == cudaSuccess && nbytes) e = cudaMemset(d, 0xFF, nbytes);
    if (e != cudaSuccess) { cudaFree(d); return fail(TQ_ERR_CUDA, cudaGetErrorString(e)); }
    s.d_alive = d;
  }
  auto patch = [&](size_t byte, uint8_t keep) -> cudaError_t {  // alive[byte] &= keep
    uint8_t v = 0;
    cudaError_t e = cudaMemcpy(&v, s.d_alive + byte, 1, cudaMemcpyDeviceToHost);
    v &= keep;
    if (e == cudaSuccess) e = cudaMemcpy(s.d_alive + byte, &v, 1, cudaMemcpyHostToDevice);
    return e;
  };
  auto clear_bits = [&](uint32_t a, uint32_t b) -> cudaError_t {  // docs [a, b) are not alive here (bit d & 7 of byte d >> 3)
    if (a >= b) return cudaSuccess;
    const size_t fb = ((size_t)a + 7) / 8, lb = (size_t)b / 8;  // whole bytes [fb, lb)
    cudaError_t e = cudaSuccess;
    if (fb > lb) return patch(a / 8, (uint8_t)~(((1u << (b - a)) - 1u) << (a & 7u)));  // a and b inside one byte
    if (lb > fb) e = cudaMemset(s.d_alive + fb, 0, lb - fb);
    if (e == cudaSuccess && (a & 7u)) e = patch(a / 8, (uint8_t)((1u << (a & 7u)) - 1u));
    if (e == cudaSuccess && (b & 7u)) e = patch(b / 8, (uint8_t)~((1u << (b & 7u)) - 1u));
    return e;
  };
  cudaError_t e = clear_bits(s.doc_lo, doc_lo);
  if (e == cudaSuccess) e = clear_bits(doc_hi, s.doc_hi);
  if (e != cudaSuccess) return fail(TQ_ERR_CUDA, std::string("doc range: ") + cudaGetErrorString(e));
  s.doc_lo = doc_lo; s.doc_hi = doc_hi;
  for (auto& kv : c->filter_views)  // the segment's filter views follow the new range (in place: prepared batches keep their pointers)
    if (std::get<1>(kv.first) == segment_ord && std::get<2>(kv.first) == field) {
      const int rc = build_view(c, s, c->filters.at({std::get<0>(kv.first), segment_ord}), kv.second);
      if (rc != TQ_OK) return rc;
    }
  return TQ_OK;
}

int tq_segment_unregister(tq_ctx* c, uint32_t segment_ord, uint32_t field) {
  if (!c) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> g(c->mu);
  auto it = c->segments.find({segment_ord, field});
  if (it == c->segments.end()) return fail(TQ_ERR_NOT_FOUND, "segment/field not registered");
  if (c->seg_users.count({segment_ord, field})) return fail(TQ_ERR_INVALID_ARGUMENT, "a prepared batch still uses the segment");
  cudaDeviceSynchronize();
  cudaFree(it->second.d_idx); cudaFree(it->second.d_fieldnorm); cudaFree(it->second.d_alive);
  cudaFree(it->second.d_pos); cudaFree(it->second.d_pos_pool);
  c->pos_tables.drop([&](const PosKey& k) { return k.segment_ord == segment_ord && k.field == field; });
  it->second.arena.release();  // the segment's block tables and aligned block copies go with it ...
  c->segments.erase(it);
  c->list_tables.drop([&](const ListKey& k) { return k.segment_ord == segment_ord && k.field == field; });  // ... and their ids are reused
  drop_views(c, [&](const std::tuple<uint32_t, uint32_t, uint32_t>& k) { return std::get<1>(k) == segment_ord && std::get<2>(k) == field; });
  auto rest = c->segments.lower_bound({segment_ord, 0u});
  if (rest == c->segments.end() || rest->first.first != segment_ord) {  // the ordinal's last field: its filters and sort columns go too
    for (auto fi = c->filters.begin(); fi != c->filters.end();)                // (a reused ordinal starts clean)
      if (fi->first.second == segment_ord) fi = c->filters.erase(fi); else ++fi;
    for (auto ci = c->sort_columns.begin(); ci != c->sort_columns.end();)
      if (ci->first.second == segment_ord) { ci->second.release(); ci = c->sort_columns.erase(ci); } else ++ci;
  }
  return TQ_OK;
}

int tq_filter_register(tq_ctx* c, uint32_t filter_id, uint32_t segment_ord, const uint8_t* bits, size_t len) {
  if (!c || (!bits && len)) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  std::lock_guard<std::mutex> g(c->mu);
  uint32_t max_doc = 0;
  bool any = false;
  for (auto it = c->segments.lower_bound({segment_ord, 0u}); it != c->segments.end() && it->first.first == segment_ord; ++it) {
    any = true;
    max_doc = std::max(max_doc, it->second.max_doc);
  }
  if (!any) return fail(TQ_ERR_NOT_FOUND, "no field of the segment ordinal is registered");
  if (len * 8 < max_doc) return fail(TQ_ERR_INVALID_ARGUMENT, "filter bitset shorter than max_doc");
  if (c->filter_users.count(filter_id)) return fail(TQ_ERR_INVALID_ARGUMENT, "a prepared batch still uses the filter");
  const size_t nbytes = ((size_t)max_doc + 7) / 8;
  std::vector<uint8_t> copy(bits, bits + nbytes);
  if (max_doc & 7u) copy.back() &= (uint8_t)((1u << (max_doc & 7u)) - 1u);  // bits at and beyond max_doc are ignored
  cudaDeviceSynchronize();
  drop_views(c, [&](const std::tuple<uint32_t, uint32_t, uint32_t>& k) { return std::get<0>(k) == filter_id && std::get<1>(k) == segment_ord; });
  c->filters[{filter_id, segment_ord}] = std::move(copy);
  return TQ_OK;
}

int tq_filter_unregister(tq_ctx* c, uint32_t filter_id) {
  if (!c) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  std::lock_guard<std::mutex> g(c->mu);
  if (c->filter_users.count(filter_id)) return fail(TQ_ERR_INVALID_ARGUMENT, "a prepared batch still uses the filter");
  auto first = c->filters.lower_bound({filter_id, 0u});
  if (first == c->filters.end() || first->first.first != filter_id) return fail(TQ_ERR_NOT_FOUND, "filter not registered");
  cudaDeviceSynchronize();
  drop_views(c, [&](const std::tuple<uint32_t, uint32_t, uint32_t>& k) { return std::get<0>(k) == filter_id; });
  while (first != c->filters.end() && first->first.first == filter_id) first = c->filters.erase(first);
  return TQ_OK;
}

// ---- sort columns (tq_sort_batch) ---------------------------------------------------------------------------------------------
int tq_sort_column_register(tq_ctx* c, uint32_t column_id, uint32_t segment_ord, const uint64_t* values, size_t n_values,
                            const uint8_t* present, size_t present_len) {
  if (!c || (!values && n_values) || (!present && present_len)) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  std::lock_guard<std::mutex> g(c->mu);
  uint32_t max_doc = 0;
  bool any = false;
  for (auto it = c->segments.lower_bound({segment_ord, 0u}); it != c->segments.end() && it->first.first == segment_ord; ++it) {
    any = true;
    max_doc = std::max(max_doc, it->second.max_doc);
  }
  if (!any) return fail(TQ_ERR_NOT_FOUND, "no field of the segment ordinal is registered");
  if (n_values != max_doc) return fail(TQ_ERR_INVALID_ARGUMENT, "a sort column holds max_doc values");
  if (present && present_len * 8 < max_doc) return fail(TQ_ERR_INVALID_ARGUMENT, "present bitset shorter than max_doc");
  if (c->sort_users.count(column_id)) return fail(TQ_ERR_INVALID_ARGUMENT, "a sort run still reads the column");
  // the bounds of every 8192-doc tile: the largest and the smallest value of its docs with a value, and which kinds it holds
  const uint32_t n_tiles = (max_doc + kTileDocs - 1) / kTileDocs;
  SortColumn col;
  col.tiles.assign(n_tiles, SortTile{{0ull, 0ull}, 0u, 0u});
  col.finite.assign(n_tiles, FiniteTile{0ull, 0ull, 0u});
  // images of the f64 infinities: finite values lie strictly between them, NaNs beyond them
  constexpr unsigned long long kNegInf = 0x000FFFFFFFFFFFFFull, kPosInf = 0xFFF0000000000000ull;
  for (uint32_t t = 0; t < n_tiles; ++t) {
    unsigned long long hi = 0, lo = ~0ull, fhi = 0, flo = ~0ull;
    uint32_t flags = 0, fflags = 0;
    for (uint32_t d = t * kTileDocs, e = std::min(max_doc, d + kTileDocs); d < e; ++d) {
      if (present && !((present[d >> 3] >> (d & 7u)) & 1u)) { flags |= kSortTileNone; continue; }
      flags |= kSortTileValues;
      const unsigned long long v = values[d];
      hi = std::max<unsigned long long>(hi, v);
      lo = std::min<unsigned long long>(lo, v);
      if (v > kNegInf && v < kPosInf) { fflags |= kFiniteAny; fhi = std::max(fhi, v); flo = std::min(flo, v); }
      else fflags |= v == kNegInf ? kFiniteNegInf : v == kPosInf ? kFinitePosInf : 0u;
    }
    col.tiles[t] = SortTile{{(flags & kSortTileValues) ? hi : 0ull, (flags & kSortTileValues) ? ~lo : 0ull}, flags, 0u};
    col.finite[t] = FiniteTile{flo, fhi, fflags};
    if (flags & kSortTileValues) { col.min_image = std::min<unsigned long long>(col.min_image, lo); col.max_image = std::max<unsigned long long>(col.max_image, hi); }
  }
  const size_t present_bytes = (size_t)n_tiles * (kTileDocs / 8);
  cudaError_t e = cudaMalloc(&col.d_values, std::max<size_t>((size_t)max_doc * 8, 8));
  if (e == cudaSuccess && max_doc) e = cudaMemcpy(col.d_values, values, (size_t)max_doc * 8, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMalloc(&col.d_tiles, std::max<size_t>(n_tiles, 1) * sizeof(SortTile));
  if (e == cudaSuccess && n_tiles) e = cudaMemcpy(col.d_tiles, col.tiles.data(), n_tiles * sizeof(SortTile), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && present && n_tiles) {
    std::vector<uint8_t> bits(present_bytes, 0);
    memcpy(bits.data(), present, ((size_t)max_doc + 7) / 8);
    if (max_doc & 7u) bits[max_doc >> 3] &= (uint8_t)((1u << (max_doc & 7u)) - 1u);  // bits at and beyond max_doc are ignored
    e = cudaMalloc(&col.d_present, present_bytes);
    if (e == cudaSuccess) e = cudaMemcpy(col.d_present, bits.data(), present_bytes, cudaMemcpyHostToDevice);
  }
  if (e != cudaSuccess) { col.release(); return fail(TQ_ERR_CUDA, std::string("sort column upload: ") + cudaGetErrorString(e)); }
  auto it = c->sort_columns.find({column_id, segment_ord});
  if (it != c->sort_columns.end()) { it->second.release(); it->second = std::move(col); }  // (no run reads it: sort_users)
  else c->sort_columns.emplace(std::make_pair(column_id, segment_ord), std::move(col));
  return TQ_OK;
}

int tq_sort_column_unregister(tq_ctx* c, uint32_t column_id) {
  if (!c) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  std::lock_guard<std::mutex> g(c->mu);
  if (c->sort_users.count(column_id)) return fail(TQ_ERR_INVALID_ARGUMENT, "a sort run still reads the column");
  auto first = c->sort_columns.lower_bound({column_id, 0u});
  if (first == c->sort_columns.end() || first->first.first != column_id) return fail(TQ_ERR_NOT_FOUND, "sort column not registered");
  while (first != c->sort_columns.end() && first->first.first == column_id) { first->second.release(); first = c->sort_columns.erase(first); }
  return TQ_OK;
}

}  // extern "C"

// ---- table caches ---------------------------------------------------------------------------------------------------------
namespace tq::host {

int get_list(tq_ctx* c, const tq_term_seg& ts, bool ignore_freq, uint32_t* list_id, const Segment** seg_out) {
  auto sit = c->segments.find({ts.segment_ord, ts.field});
  if (sit == c->segments.end()) return fail(TQ_ERR_NOT_FOUND, "term_seg names a segment/field that is not registered");
  Segment& seg = sit->second;
  *seg_out = &seg;
  if (ts.postings_end < ts.postings_start || ts.postings_end + 8 > seg.idx_len) return fail(TQ_ERR_INVALID_ARGUMENT, "postings range outside the field body");
  if (ts.postings_end - ts.postings_start > 0xFFFFFFFFull) return fail(TQ_ERR_UNSUPPORTED, "posting list larger than 4 GiB");
  ignore_freq = ignore_freq && seg.record_option != 0;
  const ListKey key{ts.segment_ord, ts.field, ts.postings_start | (ignore_freq ? 1ull << 63 : 0ull)};
  if (const uint32_t* id = c->list_tables.find(key)) { *list_id = *id; return TQ_OK; }
  if (c->list_tables.full()) return fail(TQ_ERR_OOM, "posting-list table cache full (TQ_MAX_LISTS)");
  const uint32_t n_blocks = ts.doc_freq / 128u, tail_n = ts.doc_freq % 128u;
  cudaError_t e;
  const size_t n_last = (size_t)n_blocks + 1, n_blk = (size_t)n_blocks + 1;
  const size_t len = (size_t)(ts.postings_end - ts.postings_start);
  const size_t copy_bytes = ((len + 15) & ~(size_t)15) + 128;  // 16-byte aligned copy of the blocks + slack
  uint8_t* mem = seg.arena.alloc(copy_bytes + n_last * 16 + n_last * 4 + 12 + n_blk * 8 + (size_t)tail_n * 8 + 16, &e);
  if (!mem) return fail(TQ_ERR_OOM, std::string("block table alloc: ") + cudaGetErrorString(e));
  ListBuild& lb = c->list_tables.schedule(key, list_id);
  ListDesc& d = lb.desc;
  uint8_t* p = mem;
  d.blocks = p; p += copy_bytes;  // filled by k_build_tables
  d.tab4 = reinterpret_cast<const uint4*>(p); p += n_last * 16;
  d.blk = reinterpret_cast<const uint2*>(p); p += n_blk * 8;
  d.last_doc = reinterpret_cast<const uint32_t*>(p); p += n_last * 4;
  d.tail_docs = reinterpret_cast<const uint32_t*>(p); p += (size_t)tail_n * 4;
  d.tail_tfs = reinterpret_cast<const uint32_t*>(p);
  d.fieldnorm = seg.d_fieldnorm;
  d.n_blocks = n_blocks; d.tail_n = tail_n; d.n_total = n_blocks + (tail_n ? 1u : 0u); d.doc_freq = ts.doc_freq;
  d.build_status = 1;  // until k_build_tables says otherwise
  lb.job.bytes = seg.d_idx + 8 + ts.postings_start;
  lb.job.len = (uint32_t)(ts.postings_end - ts.postings_start);
  lb.job.doc_freq = ts.doc_freq;
  lb.job.record_option = (uint32_t)seg.record_option | (ignore_freq ? 0x100u : 0u);
  lb.job.list_id = *list_id;
  return TQ_OK;
}

int get_pos(tq_ctx* c, const tq_term_seg& ts, const tq_term_pos& tp, uint32_t* pos_id) {
  auto sit = c->segments.find({ts.segment_ord, ts.field});
  if (sit == c->segments.end()) return fail(TQ_ERR_NOT_FOUND, "term_seg names a segment/field that is not registered");
  Segment& seg = sit->second;
  if (!seg.d_pos) return fail(TQ_ERR_INVALID_ARGUMENT, "phrase query on a segment without registered positions (tq_segment_register_positions)");
  if (tp.positions_end < tp.positions_start || tp.positions_end > seg.pos_len) return fail(TQ_ERR_INVALID_ARGUMENT, "positions range outside the `.pos` body");
  if (tp.positions_end - tp.positions_start > 0xFFFFFFFFull) return fail(TQ_ERR_UNSUPPORTED, "position stream larger than 4 GiB");
  const PosKey key{ts.segment_ord, ts.field, ts.postings_start, tp.positions_start};
  if (const uint32_t* id = c->pos_tables.find(key)) { *pos_id = *id; return TQ_OK; }
  if (c->pos_tables.full()) return fail(TQ_ERR_OOM, "position table cache full (TQ_MAX_POS_LISTS)");
  PosJob& job = c->pos_tables.schedule(key, pos_id);
  job.pos_bytes = seg.d_pos + tp.positions_start;
  job.pos_len = (uint32_t)(tp.positions_end - tp.positions_start);
  job.list_bytes = seg.d_idx + 8 + ts.postings_start;
  job.list_len = (uint32_t)(ts.postings_end - ts.postings_start);
  job.doc_freq = ts.doc_freq;
  job.pool = seg.d_pos_pool;
  job.pool_cursor = reinterpret_cast<unsigned long long*>(seg.d_pos_pool);
  job.pool_cap = seg.pos_pool_cap;
  job.pos_id = *pos_id;
  return TQ_OK;
}

}  // namespace tq::host

// Builds the tables a cache has scheduled and waits for them (the first use of a term only): `job_bytes` per table staged by
// fill(host, n) and a status word each, one H2D copy, launch(device, status, n) enqueues the build kernel on the build stream,
// and the status words come back.  A nonzero one fails with status_error(it).  On any failure every scheduled table is rolled
// back (no cache entry survives for a table that was not built); *built += the tables built.  ctx->mu held.
template <class Cache, class Fill, class Launch, class StatusError>
static int flush_tables(tq_ctx* c, Cache& cache, size_t job_bytes, Fill fill, Launch launch, StatusError status_error, uint64_t* built) {
  const size_t n = cache.pending.size();
  if (n == 0) return TQ_OK;
  struct Undo { Cache& cache; ~Undo() { cache.rollback(); } } undo{cache};
  const size_t bytes = n * (job_bytes + 4);
  TQ_CUDA(c->build_pin.ensure(bytes));
  TQ_CUDA(c->build_dev.ensure(bytes));
  uint32_t* hs = reinterpret_cast<uint32_t*>(c->build_pin.p + n * job_bytes);
  uint32_t* ds = reinterpret_cast<uint32_t*>(c->build_dev.p + n * job_bytes);
  fill(c->build_pin.p, n);
  for (size_t i = 0; i < n; ++i) hs[i] = 1;
  TQ_CUDA(cudaMemcpyAsync(c->build_dev.p, c->build_pin.p, bytes, cudaMemcpyHostToDevice, c->build_stream));
  launch(c->build_dev.p, ds, (unsigned)n);
  TQ_CUDA(cudaGetLastError());
  TQ_CUDA(cudaMemcpyAsync(hs, ds, n * 4, cudaMemcpyDeviceToHost, c->build_stream));
  TQ_CUDA(cudaStreamSynchronize(c->build_stream));
  for (size_t i = 0; i < n; ++i)
    if (hs[i] != 0) return status_error(hs[i]);
  *built += n;
  cache.pending.clear();  // (built: nothing to roll back)
  return TQ_OK;
}

// The block tables: [ListDesc][BuildJob] per table.
static int flush_builds(tq_ctx* c, uint64_t* built) {
  const auto& pending = c->list_tables.pending;
  return flush_tables(
      c, c->list_tables, sizeof(ListDesc) + sizeof(BuildJob),
      [&](uint8_t* h, size_t n) {
        for (size_t i = 0; i < n; ++i) {
          reinterpret_cast<ListDesc*>(h)[i] = pending[i].build.desc;
          reinterpret_cast<BuildJob*>(h + n * sizeof(ListDesc))[i] = pending[i].build.job;
        }
      },
      [&](const uint8_t* d, uint32_t* status, unsigned n) {
        k_build_tables<<<n, kThreads, 0, c->build_stream>>>(reinterpret_cast<const BuildJob*>(d + n * sizeof(ListDesc)),
                                                            reinterpret_cast<const ListDesc*>(d), c->d_lists, status);
      },
      [](uint32_t) { return fail(TQ_ERR_CORRUPT, "posting list bytes are not a valid tantivy posting list"); }, built);
}

// The position tables (not counted in lists_built).
static int flush_pos_builds(tq_ctx* c) {
  const auto& pending = c->pos_tables.pending;
  uint64_t built = 0;
  return flush_tables(
      c, c->pos_tables, sizeof(PosJob),
      [&](uint8_t* h, size_t n) { for (size_t i = 0; i < n; ++i) reinterpret_cast<PosJob*>(h)[i] = pending[i].build; },
      [&](const uint8_t* d, uint32_t* status, unsigned n) {
        k_build_pos_tables<<<n, kThreads, 0, c->build_stream>>>(reinterpret_cast<const PosJob*>(d), c->d_pos_descs, status);
      },
      [](uint32_t s) {
        return s == 2 ? fail(TQ_ERR_OOM, "the segment's position-table pool is exhausted")
                      : fail(TQ_ERR_CORRUPT, "position bytes are not a valid tantivy position stream");
      },
      &built);
}

// What the current call scheduled in the table caches and did not build is rolled back when the scope ends (every early error
// return).  ctx->mu held.
struct TableScope {
  tq_ctx* c;
  ~TableScope() { c->list_tables.rollback(); c->pos_tables.rollback(); }
};

// ---- batches ---------------------------------------------------------------------------------------
// Kernel time by kind: CUDA events recorded on the batch's stream around every launch (group of launches) of that kind.
enum SpanKind { SPAN_TERM = 0, SPAN_AND, SPAN_OR, SPAN_FINAL, SPAN_SCORE, SPAN_TILE, SPAN_THETA, SPAN_PHRASE, SPAN_COUNT, SPAN_KINDS };

static int span_begin(tq_batch* b, int kind, cudaStream_t on = nullptr) {
  if (b->n_spans == b->spans.size()) {
    tq_batch::Span s;
    s.kind = kind;
    if (cudaEventCreate(&s.a) != cudaSuccess || cudaEventCreate(&s.b) != cudaSuccess) return -1;
    b->spans.push_back(s);
  }
  tq_batch::Span& s = b->spans[b->n_spans];
  s.kind = kind;
  cudaEventRecord(s.a, on ? on : b->stream);
  return (int)b->n_spans++;
}
static void span_end(tq_batch* b, int idx, cudaStream_t on = nullptr) {
  if (idx >= 0) cudaEventRecord(b->spans[idx].b, on ? on : b->stream);
}

static void collect_times(tq_batch* b) {
  float ms = 0;
  if (cudaEventElapsedTime(&ms, b->ev_k0, b->ev_k1) == cudaSuccess) b->stats.kernel_ms = ms;
  float by_kind[SPAN_KINDS] = {0};
  for (size_t i = 0; i < b->n_spans; ++i)
    if (cudaEventElapsedTime(&ms, b->spans[i].a, b->spans[i].b) == cudaSuccess) by_kind[b->spans[i].kind] += ms;
  b->stats.term_ms = by_kind[SPAN_TERM];
  b->stats.and_ms = by_kind[SPAN_AND];
  b->stats.or_ms = by_kind[SPAN_OR];
  b->stats.final_ms = by_kind[SPAN_FINAL];
  b->stats.score_ms = by_kind[SPAN_SCORE];
  b->stats.tile_ms = by_kind[SPAN_TILE];
  b->stats.theta_ms = by_kind[SPAN_THETA];
  b->stats.phrase_ms = by_kind[SPAN_PHRASE];
  b->stats.count_hits_ms = by_kind[SPAN_COUNT];
}

// The run's kernel times into its stats, and its stats into the context's (tq_get_stats).
static void publish_stats(tq_batch* b) {
  collect_times(b);
  std::lock_guard<std::mutex> g(b->ctx->mu);
  b->ctx->stats = b->stats;
}

// Enqueues a copy of src's result rows (the first min(k_max, stride) of each) and counts into device arrays of row stride `stride`.
static cudaError_t copy_rows(const tq_batch* src, cudaStream_t stream, float* scores, uint32_t* segs, uint32_t* docs, uint32_t* counts, size_t stride) {
  const BatchParams& S = src->params;
  const size_t dp = stride * 4, sp = (size_t)src->kmax * 4, width = std::min(dp, sp);
  auto rows = [&](void* d, const void* s) {  // (one plain copy when both sides have the same stride)
    return dp == sp ? cudaMemcpyAsync(d, s, sp * src->nq, cudaMemcpyDeviceToDevice, stream)
                    : cudaMemcpy2DAsync(d, dp, s, sp, width, src->nq, cudaMemcpyDeviceToDevice, stream);
  };
  cudaError_t e = rows(scores, S.res_scores);
  if (e == cudaSuccess) e = rows(segs, S.res_segs);
  if (e == cudaSuccess) e = rows(docs, S.res_docs);
  if (e == cudaSuccess) e = cudaMemcpyAsync(counts, S.res_counts, (size_t)src->nq * 4, cudaMemcpyDeviceToDevice, stream);
  return e;
}

// k_count over (query, segment) pairs: stages their structure words, the pairs, the units and zeroed per-query counters, runs the
// kernel and adds the counts to out_counts.
static int count_on_device(tq_batch* b, const std::vector<uint32_t>& words, const std::vector<CountSeg>& segs, const std::vector<Unit>& units,
                           bool mixed, size_t nq, uint64_t* out_counts) {
  const std::vector<unsigned long long> zeros(nq, 0);
  Staging st;
  const size_t o_w = st.add(words), o_s = st.add(segs), o_u = st.add(units), o_c = st.add(zeros);
  TQ_CUDA(st.reserve(b->pin, b->dev));
  st.copy();
  const CountParams P{b->ctx->d_lists, st.on_device<const uint32_t>(o_w), st.on_device<const CountSeg>(o_s), st.on_device<const Unit>(o_u),
                      st.on_device<unsigned long long>(o_c)};
  TQ_CUDA(cudaMemcpyAsync(b->dev.p, b->pin.p, st.bytes, cudaMemcpyHostToDevice, b->stream));
  (mixed ? k_count<true> : k_count<false>)<<<(unsigned)units.size(), kThreads, 0, b->stream>>>(P);
  TQ_CUDA(cudaGetLastError());
  TQ_CUDA(cudaMemcpyAsync(b->pin.p + o_c, b->dev.p + o_c, nq * 8, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  const unsigned long long* dc = st.on_host<const unsigned long long>(o_c);
  for (size_t qi = 0; qi < nq; ++qi) out_counts[qi] += dc[qi];
  return TQ_OK;
}

static tq_batch* acquire_batch(tq_ctx* c) {
  {
    std::lock_guard<std::mutex> g(c->mu);
    if (!c->pool.empty()) { tq_batch* b = c->pool.back(); c->pool.pop_back(); return b; }
  }
  auto* b = new tq_batch();
  b->ctx = c;
  if (cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking) != cudaSuccess || cudaStreamCreateWithFlags(&b->side, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&b->ev_side0, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&b->ev_side1, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreate(&b->ev_start) != cudaSuccess ||
      cudaEventCreate(&b->ev_k0) != cudaSuccess || cudaEventCreate(&b->ev_k1) != cudaSuccess || cudaEventCreate(&b->ev_end) != cudaSuccess ||
      cudaMallocHost(&b->flags_pin, 64) != cudaSuccess) {
    tq_batch_destroy_real(b);
    return nullptr;
  }
  return b;
}

// One array of units out of per-class lists; class i starts at base[i] and has n[i] units.
template <class U, size_t N>
static std::vector<U> concat_units(const std::vector<U> (&by_class)[N], uint32_t* base, uint32_t* n) {
  std::vector<U> all;
  for (size_t i = 0; i < N; ++i) {
    base[i] = (uint32_t)all.size();
    n[i] = (uint32_t)by_class[i].size();
    all.insert(all.end(), by_class[i].begin(), by_class[i].end());
  }
  return all;
}

// Stages the descriptors, sizes the tile and run scratch, fills BatchParams / TileParams, starts the upload and tf-table build.
static int lay_out(tq_ctx* c, tq_batch* b, BatchPlan& pl) {
  if (pl.caches.empty()) pl.caches.resize(256, 0.0f);
  if (!pl.qaux.empty() && pl.qaux.size() < pl.qlists.size()) pl.qaux.resize(pl.qlists.size(), PhraseAux{0, 0, 0});
  const size_t nq = pl.nq, nq1 = std::max<size_t>(nq, 1), n_caches = pl.caches.size() / 256;
  const std::vector<Unit> units = concat_units(pl.units, b->unit_base, b->n_units);
  Staging st;
  const size_t o_caches = st.add(pl.caches);
  const size_t o_tftab = st.add(nullptr, n_caches * kTfRows * 256 * 4);  // device only (built by k_build_tf_tables)
  const size_t o_qlists = st.add(pl.qlists), o_qsegs = st.add(pl.qsegs), o_qaux = st.add(pl.qaux), o_units = st.add(units);
  const size_t o_queries = st.add(pl.dq);
  const size_t o_qinit = st.add(nullptr, nq1 * sizeof(QState));  // per-run initial state (threshold keys), filled below
  struct GroupOff { size_t slots, segs, queries, clauses, units, chunks, count_units; };
  std::vector<GroupOff> goff(pl.gstage.size());
  std::vector<std::vector<TUnit>> gunits(pl.gstage.size());
  b->groups.resize(pl.gstage.size());
  for (size_t gi = 0; gi < pl.gstage.size(); ++gi) {
    const GroupStage& gs = pl.gstage[gi];
    gunits[gi] = concat_units(gs.units, b->groups[gi].unit_base, b->groups[gi].n_units);
    goff[gi] = GroupOff{st.add(gs.slots), st.add(gs.segs), st.add(gs.queries), st.add(gs.clauses), st.add(gunits[gi]), st.add(gs.chunks),
                        gs.count_units.empty() ? 0 : st.add(gs.count_units)};
  }
  // k_count for the TQ_QUERY_COUNT_HITS queries on the per-query kernels
  const CountPlan& cp = pl.count;
  size_t o_cnt_words = 0, o_cnt_segs = 0, o_cnt_units = 0;
  if (!cp.units.empty()) { o_cnt_words = st.add(cp.words); o_cnt_segs = st.add(cp.segs); o_cnt_units = st.add(cp.units); }
  b->desc_bytes = st.bytes;
  TQ_CUDA(st.reserve(b->pin, b->dev));

  // ---- tile scratch: pair arrays | tile indexes | samples | sample counts | key histograms | flags + counters ---------------
  uint32_t sample_cap = 0;
  size_t to_docs = 0, to_scores = 0, to_tix = 0, to_samples = 0, to_scount = 0, to_th_hist = 0, to_flags = 0, to_cursors = 0, to_count_cursors = 0;
  if (!pl.gstage.empty()) {
    uint64_t sample_units_tiles = 0;
    for (auto& gs : pl.gstage) for (auto& u : gs.units[0]) sample_units_tiles += u.t1 - u.t0;
    sample_cap = (uint32_t)std::min<uint64_t>(1u << 16, std::max<uint64_t>(256, sample_units_tiles * 8u));
    size_t so2 = 0;
    to_docs = so2; so2 = align256(so2 + (size_t)pl.pair_cursor * 4);
    to_scores = so2; so2 = align256(so2 + (size_t)pl.pair_cursor * 4);
    to_tix = so2; so2 = align256(so2 + pl.tix_total_words * 4);
    to_samples = so2; so2 = align256(so2 + nq1 * sample_cap * 4);
    to_scount = so2; so2 = align256(so2 + nq1 * 4);
    to_th_hist = so2; so2 = align256(so2 + nq1 * kThHistWords * 4);
    to_flags = so2; so2 = align256(so2 + 256);
    size_t cursors = 0;  // k_tile's sparse-slot cursors: max_slots per CTA of the largest launch (launches of a batch run one after another)
    for (auto& gs : pl.gstage)
      for (auto& u : gs.units) cursors = std::max<size_t>(cursors, u.size() * gs.max_slots);
    to_cursors = so2; so2 = align256(so2 + cursors * sizeof(uint2));
    size_t count_cursors = 0;  // k_count_tiles' own cursors (its launches run next to k_tile's, one group after another)
    for (auto& gs : pl.gstage) count_cursors = std::max<size_t>(count_cursors, gs.count_units.size() * gs.max_slots);
    to_count_cursors = so2; so2 = align256(so2 + count_cursors * sizeof(uint2));
    pl.tile_bytes = so2;
    TQ_CUDA(b->tile_dev.ensure(pl.tile_bytes));
  }
  b->tile_zero_off = to_scount;
  b->tile_zero_bytes = pl.gstage.empty() ? 0 : (to_flags + 256 - to_scount);
  b->tile_flags_off = to_flags;
  for (auto& gs : pl.gstage)  // rebase the tile-index offsets to device addresses
    for (auto& G : gs.segs) G.tix = reinterpret_cast<uint32_t*>(b->tile_dev.p + to_tix) + reinterpret_cast<size_t>(G.tix);

  st.copy();
  QState* qi0 = st.on_host<QState>(o_qinit);
  for (size_t qi = 0; qi < nq1; ++qi) {
    qi0[qi].theta = 0; qi0[qi].cand_count = 0;
    if (qi < nq && (pl.queries[qi].flags & TQ_QUERY_HAS_THRESHOLD)) {
      // collect score > threshold: the smallest accepted key is the next representable score (NaN: no filter)
      float th = pl.queries[qi].threshold;
      if (th == 0.0f) th = 0.0f;  // -0.0 and +0.0 are the same threshold
      if (th == th) { const uint32_t key = host_score_key(th); qi0[qi].theta = key == 0xFFFFFFFFu ? key : key + 1u; }
    }
  }
  b->qinit_off = o_qinit;
  b->phrase_aux = st.on_device<const PhraseAux>(o_qaux);
  b->strip_cached_max = pl.strip_cached_max;
  b->phrase_ct = std::min<uint32_t>(pl.phrase_ct, kPhraseMaxTerms);
  for (size_t gi = 0; gi < pl.gstage.size(); ++gi) {
    const GroupStage& gs = pl.gstage[gi];
    tq_batch::TileGroup& run = b->groups[gi];
    run.n_chunks = (uint32_t)gs.chunks.size();
    TileParams& TP = run.params;
    TP.slots = st.on_device<const TSlot>(goff[gi].slots);
    TP.segs = st.on_device<const TSeg>(goff[gi].segs);
    TP.queries = st.on_device<const TQuery>(goff[gi].queries);
    TP.clauses = st.on_device<const uint16_t>(goff[gi].clauses);
    TP.units = st.on_device<const TUnit>(goff[gi].units);
    TP.chunks = st.on_device<const SChunk>(goff[gi].chunks);
    TP.p_docs = reinterpret_cast<uint32_t*>(b->tile_dev.p + to_docs);
    TP.p_scores = reinterpret_cast<float*>(b->tile_dev.p + to_scores);
    TP.samples = reinterpret_cast<uint32_t*>(b->tile_dev.p + to_samples);
    TP.sample_count = reinterpret_cast<uint32_t*>(b->tile_dev.p + to_scount);
    TP.th_hist = reinterpret_cast<uint32_t*>(b->tile_dev.p + to_th_hist);
    TP.flags = reinterpret_cast<uint32_t*>(b->tile_dev.p + to_flags);
    TP.counters = c->tile_counters ? c->d_counters + 8 : nullptr;
    TP.cursors = reinterpret_cast<uint2*>(b->tile_dev.p + to_cursors);
    TP.sample_cap = sample_cap;
    TP.p_cap = gs.p_cap;
    TP.max_slots = gs.max_slots;
    TP.max_big = gs.max_big;
    TP.max_queries = (gs.max_queries + 1u) & ~1u;
    // per-tile work list: about two (query, essential clause) entries per query, more for wide unions; a tile that needs more
    // takes another round of routing + expansion
    TP.seg_cap = std::min<uint32_t>(kTileMaxWorkList, std::max<uint32_t>(256u, std::max<uint32_t>(2u, gs.max_clauses / 4u) * TP.max_queries));
    if (c->tile_seg_cap_hook) TP.seg_cap = c->tile_seg_cap_hook;
    TP.light_max = c->tile_light_max;
    TP.cl_cap = gs.max_clause_words <= kTileMaxStagedClauses ? ((gs.max_clause_words + 3u) & ~3u) : 0u;
    TP.n_win = c->tile_windows ? std::min<uint32_t>(c->tile_windows, kTileWarps) : kTileExactWindows;
    run.smem = tile_smem_bytes(gs.p_cap, gs.max_slots, TP.max_big, TP.max_queries, TP.seg_cap, TP.cl_cap, TP.n_win);
    c->tile_smem_last = run.smem;
    if (run.smem > kTileMaxSmem) return fail(TQ_ERR_UNSUPPORTED, "tile group needs more shared memory than an SM has");
    int ctas = 0;
    run.union_only = gs.union_only;
    // (the exact instance the group runs without TQ_TILE_COUNTERS: the counters instances are built for 3 CTAs per SM)
    TQ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, tile_kernel(false, false, run.union_only), kTileThreads, run.smem));
    c->tile_ctas_last = (uint64_t)ctas;
    run.n_count_units = (uint32_t)gs.count_units.size();
    run.count_queries = gs.count_queries;
    run.count_smem = count_tiles_smem_bytes(TP.max_slots, TP.max_big, TP.max_queries);
  }

  // ---- scratch: qstate | candidates | results | hits + the groups' count overflow words ---------------------------------
  b->kmax = pl.kmax;
  b->n_cands = pl.n_cands;
  size_t so = 0;
  b->qstate_off = so; so = align256(so + nq1 * sizeof(QState));
  b->cands_off = so; so = align256(so + std::max<size_t>(pl.n_cands, 1) * sizeof(Cand));
  b->res_off = so;
  const size_t col = align256(nq1 * pl.kmax * 4);
  b->res_at = {0, col, 2 * col, 3 * col};
  b->res_bytes = b->res_at.counts + align256(nq1 * 4);
  so += b->res_bytes;
  b->count_hits = pl.count_hits;
  b->hits_off = so;
  b->hits_bytes = pl.count_hits ? nq1 * 8 + b->groups.size() * 4 : 0;
  so = align256(so + b->hits_bytes);
  TQ_CUDA(b->scratch.ensure(so));
  if (pl.count_hits) {
    TQ_CUDA(b->hits_pin.ensure(b->hits_bytes));
    b->hits_host = pl.hits_host;
    unsigned long long* hits = reinterpret_cast<unsigned long long*>(b->scratch.p + b->hits_off);
    uint32_t* ovf = reinterpret_cast<uint32_t*>(hits + nq1);
    for (size_t gi = 0; gi < b->groups.size(); ++gi) {
      tq_batch::TileGroup& run = b->groups[gi];
      run.count = CountTileParams{run.n_count_units ? st.on_device<const TUnit>(goff[gi].count_units) : nullptr,
                                  reinterpret_cast<uint2*>(b->tile_dev.p + to_count_cursors), hits, ovf + gi};
    }
    b->n_count_units = (uint32_t)cp.units.size();
    b->count_mixed = cp.mixed;
    if (b->n_count_units)
      b->count_p = CountParams{c->d_lists, st.on_device<const uint32_t>(o_cnt_words), st.on_device<const CountSeg>(o_cnt_segs),
                               st.on_device<const Unit>(o_cnt_units), hits};
  } else {
    b->hits_host.clear();
    b->n_count_units = 0;
  }
  TQ_CUDA(b->res_pin.ensure(b->res_bytes));

  BatchParams& P = b->params;
  P.lists = c->d_lists;
  P.caches = st.on_device<const float>(o_caches);
  P.tf_tables = st.on_device<const float>(o_tftab);
  P.qlists = st.on_device<const QList>(o_qlists);
  P.qsegs = st.on_device<const QSeg>(o_qsegs);
  P.units = st.on_device<const Unit>(o_units);
  P.queries = st.on_device<const DQuery>(o_queries);
  P.qstate = reinterpret_cast<QState*>(b->scratch.p + b->qstate_off);
  P.cands = reinterpret_cast<Cand*>(b->scratch.p + b->cands_off);
  uint8_t* r = b->scratch.p + b->res_off;
  P.res_scores = reinterpret_cast<float*>(r + b->res_at.scores);
  P.res_segs = reinterpret_cast<uint32_t*>(r + b->res_at.segs);
  P.res_docs = reinterpret_cast<uint32_t*>(r + b->res_at.docs);
  P.res_counts = reinterpret_cast<uint32_t*>(r + b->res_at.counts);
  P.res_stride = pl.kmax;
  P.n_queries = (uint32_t)nq;
  P.counters = c->d_counters;
  P.ovf = b->groups.empty() ? nullptr : reinterpret_cast<uint32_t*>(b->tile_dev.p + to_flags) + 1;

  TQ_CUDA(cudaEventRecord(b->ev_start, b->stream));
  TQ_CUDA(cudaMemcpyAsync(b->dev.p, b->pin.p, b->desc_bytes, cudaMemcpyHostToDevice, b->stream));
  const unsigned n = (unsigned)(n_caches * kTfRows * 256);
  k_build_tf_tables<<<(n + 255) / 256, 256, 0, b->stream>>>(P.caches, st.on_device<float>(o_tftab), (uint32_t)n_caches);
  TQ_CUDA(cudaGetLastError());
  return TQ_OK;
}

// ... and the filter views of the filters its queries name: tq_filter_register / tq_filter_unregister refuse those filters until
// the batch is destroyed.  ctx->mu held.
static void hold_filters(tq_ctx* c, tq_batch* b, const tq_query* queries, size_t nq) {
  for (size_t qi = 0; qi < nq; ++qi)
    if (queries[qi].flags & TQ_QUERY_FILTER) b->held_filters.push_back(queries[qi].filter_id);
  std::sort(b->held_filters.begin(), b->held_filters.end());
  b->held_filters.erase(std::unique(b->held_filters.begin(), b->held_filters.end()), b->held_filters.end());
  for (uint32_t f : b->held_filters) ++c->filter_users[f];
}

// A prepared batch holds list ids and alive pointers of the segments its queries name: tq_segment_unregister refuses those
// segments until the batch is destroyed.  ctx->mu held.
static void hold_segments(tq_ctx* c, tq_batch* b, const tq_query* queries, size_t nq) {
  for (size_t qi = 0; qi < nq; ++qi)
    for (uint32_t i = 0; i < queries[qi].n_term_segs; ++i) {
      const std::pair<uint32_t, uint32_t> key{queries[qi].term_segs[i].segment_ord, queries[qi].term_segs[i].field};
      if (b->held.empty() || b->held.back() != key) b->held.push_back(key);
    }
  std::sort(b->held.begin(), b->held.end());
  b->held.erase(std::unique(b->held.begin(), b->held.end()), b->held.end());
  for (const auto& key : b->held) ++c->seg_users[key];
  hold_filters(c, b, queries, nq);
}

// repeat (finalize_run): 0 = a caller's batch.  1 = the repeat of an overflowed run: TERM / AND / OR / phrase queries take the
// per-query kernels; TQ_OP_BOOL queries stay on the tile engine with candidate regions as large as their postings and the largest
// tile buffer.  2 = as 1, but every TQ_OP_BOOL query in a tile group of its own.
static int batch_prepare_impl(tq_ctx* c, const tq_query* queries, size_t nq, int repeat, tq_batch** out) {
  if (!c || !out || (!queries && nq)) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  tq_batch* b = acquire_batch(c);
  if (!b) return fail(TQ_ERR_CUDA, "stream/event creation failed");
  struct Guard { tq_batch* b; bool ok = false; ~Guard() { if (!ok) tq_batch_destroy(b); } } guard{b};
  b->ran = false;
  b->finalized = false;
  b->next_phase = 0;  // a recycled batch may have been abandoned in the middle of a phased run
  b->nq = (uint32_t)nq;
  b->stats = tq_stats{};
  b->n_spans = 0;
  b->groups.clear();
  b->owned = OwnedQueries{};
  b->repeat = repeat;

  BatchPlan pl{queries, nq, repeat};
  pl.dq.resize(nq);
  pl.q_cands.assign(nq, 0);
  for (size_t qi = 0; qi < nq && !repeat && !pl.count_hits; ++qi) pl.count_hits = (queries[qi].flags & TQ_QUERY_COUNT_HITS) != 0;
  if (pl.count_hits) pl.hits_host.assign(nq, 0);
  // Single-term queries ride along on the tile engine when the batch has multi-term queries whose decoded lists they share
  // (mixed workload: 32.6 K q/s against 28.6 K with them on k_term); a batch of nothing but single-term queries has nothing to
  // share and streams its lists through k_term (configs[0]: 1.39 M q/s against 0.49 M).  TQ_TILE_TERMS: 0 never, 1 always, 2 this rule.
  pl.terms_on_tile = c->tile_terms == 1;
  if (c->tile_terms >= 2)
    for (size_t qi = 0; qi < nq && !pl.terms_on_tile; ++qi)
      pl.terms_on_tile = queries[qi].n_terms >= 2 && queries[qi].op != TQ_OP_PHRASE;
  {
    std::lock_guard<std::mutex> g(c->mu);
    TableScope table_scope{c};  // an early error return leaves no half-built table in the caches
    int rc = TQ_OK;
    for (size_t qi = 0; qi < nq && rc == TQ_OK; ++qi) rc = plan_query(c, pl, qi);
    if (rc == TQ_OK) rc = cut_units(c, pl);
    if (rc == TQ_OK) rc = flush_builds(c, &pl.built);
    if (rc == TQ_OK) rc = flush_pos_builds(c);
    if (rc != TQ_OK) return rc;
    hold_segments(c, b, queries, nq);
  }
  int rc = stage_tile_groups(c, pl);
  if (rc == TQ_OK && !pl.tgroups.empty()) b->owned.assign(queries, nq);  // the queries are kept: an overflowing run is repeated (finalize_run)
  if (rc == TQ_OK) rc = lay_out(c, b, pl);
  if (rc != TQ_OK) return rc;

  const uint32_t* nu = b->n_units;
  const uint64_t strip_units = (uint64_t)nu[UC_STRIP] + nu[UC_STRIP_ROUND1] + nu[UC_STRIP_ROUND2] + nu[UC_STRIP_ROUND3];
  b->stats.lists_built = pl.built;
  b->stats.units = nu[UC_TERM] + nu[UC_AND] + nu[UC_OR_WINDOW] + strip_units + nu[UC_PHRASE] + pl.tile_units;
  b->stats.h2d_bytes = b->desc_bytes;
  b->stats.algorithmic_bytes = pl.alg_bytes;
  b->stats.postings = pl.postings;
  b->stats.units_term = nu[UC_TERM]; b->stats.units_and = nu[UC_AND]; b->stats.units_or = nu[UC_OR_WINDOW] + strip_units; b->stats.units_or_strip = strip_units;
  b->stats.bytes_term = pl.op_bytes[0]; b->stats.bytes_and = pl.op_bytes[1]; b->stats.bytes_or = pl.op_bytes[2];
  b->stats.units_tile = pl.tile_units;
  b->stats.units_phrase = nu[UC_PHRASE];
  b->stats.tile_groups = b->groups.size();
  for (auto& g : b->groups) b->stats.tile_groups_union_only += g.union_only ? 1u : 0u;
  b->stats.tile_postings = pl.tile_postings;
  for (auto& tg : pl.tgroups) b->stats.tile_list_bytes += tg.list_bytes;
  b->stats.tile_scratch_bytes = pl.tile_bytes;
  b->stats.units_count_hits = b->n_count_units;
  for (auto& g : b->groups) b->stats.units_count_hits += g.n_count_units;
  guard.ok = true;
  *out = b;
  return TQ_OK;
}

extern "C" {

void tq_batch_destroy(tq_batch* b) {
  if (!b) return;
  cudaSetDevice(b->ctx->device);
  cudaStreamSynchronize(b->stream);
  // a run abandoned after phase 0 may still have k_phrase / the Count kernels on the second stream, reading this batch's
  // descriptors and writing its scratch: the next owner of the pooled buffers must not start before they end
  if (b->side_pending) {
    cudaStreamSynchronize(b->side);
    b->side_pending = false;
  }
  b->next_phase = 0;
  b->ran = false;
  std::lock_guard<std::mutex> g(b->ctx->mu);
  for (const auto& key : b->held) {
    auto it = b->ctx->seg_users.find(key);
    if (--it->second == 0) b->ctx->seg_users.erase(it);
  }
  b->held.clear();
  for (uint32_t f : b->held_filters) {
    auto it = b->ctx->filter_users.find(f);
    if (--it->second == 0) b->ctx->filter_users.erase(it);
  }
  b->held_filters.clear();
  for (uint32_t col : b->held_columns) {
    auto it = b->ctx->sort_users.find(col);
    if (--it->second == 0) b->ctx->sort_users.erase(it);
  }
  b->held_columns.clear();
  b->ctx->pool.push_back(b);  // buffers are recycled by the next batch
}

int tq_batch_prepare(tq_ctx* c, const tq_query* queries, size_t nq, tq_batch** out) {
  return batch_prepare_impl(c, queries, nq, 0, out);
}

}  // extern "C"

// Phases of a run: 0 = term / AND / window-union kernels + the decode-and-score pass and the sample launch of the tile engine
// + the strips' first threshold round, 1 and 2 = the next (exact) tile launches / threshold rounds, 3 = the last tile launch,
// the strips' main launch and k_final.  Every phase but the last ends with the per-query thresholds refreshed (k_theta).
// Sharded callers exchange keys in between.
constexpr int kPhases = 4;

static int launch_tile_round(tq_batch* b, int r, uint64_t* launches) {
  bool any = false;
  for (auto& g : b->groups) any = any || g.n_units[r];
  if (!any) return TQ_OK;
  const int sp = span_begin(b, SPAN_TILE);
  for (auto& g : b->groups) {
    if (!g.n_units[r]) continue;
    auto kern = tile_kernel(r == 0, g.params.counters != nullptr, g.union_only);
    kern<<<g.n_units[r], kTileThreads, g.smem, b->stream>>>(b->params, g.params, g.unit_base[r]);
    ++*launches;
  }
  span_end(b, sp);
  TQ_CUDA(cudaGetLastError());
  return TQ_OK;
}

// Enqueues launch(stream) on the batch's second stream, behind everything enqueued on its main stream so far, when `aside` (the
// last phase waits for it before k_final: side_pending); on the main stream otherwise.
template <class Launch>
static int launch_aside(tq_batch* b, bool aside, Launch launch) {
  if (aside) {
    TQ_CUDA(cudaEventRecord(b->ev_side0, b->stream));
    TQ_CUDA(cudaStreamWaitEvent(b->side, b->ev_side0, 0));
  }
  const int rc = launch(aside ? b->side : b->stream);
  if (rc != TQ_OK) return rc;
  if (aside) {
    TQ_CUDA(cudaEventRecord(b->ev_side1, b->side));
    b->side_pending = true;
  }
  return TQ_OK;
}

static int run_phase(tq_batch* b, int phase) {
  TQ_CUDA(cudaSetDevice(b->ctx->device));
  const BatchParams& P = b->params;
  uint64_t launches = 0;
  if (phase != b->next_phase) return fail(TQ_ERR_INVALID_ARGUMENT, "phases run in order, each once per run");
  const bool tiles = !b->groups.empty();
  auto timed = [&](int kind, auto&& launch) {  // one launch on the batch's stream, its time counted as `kind`
    const int sp = span_begin(b, kind);
    launch();
    ++launches;
    span_end(b, sp);
  };
  if (phase == 0) {
    b->n_spans = 0;
    b->finalized = false;
    if (b->side_pending) { TQ_CUDA(cudaStreamWaitEvent(b->stream, b->ev_side1, 0)); b->side_pending = false; }  // (a run that was abandoned)
    TQ_CUDA(cudaMemcpyAsync(P.qstate, b->dev.p + b->qinit_off, std::max<size_t>(b->nq, 1) * sizeof(QState), cudaMemcpyDeviceToDevice, b->stream));
    if (tiles) TQ_CUDA(cudaMemsetAsync(b->tile_dev.p + b->tile_zero_off, 0, b->tile_zero_bytes, b->stream));
    if (b->count_hits) TQ_CUDA(cudaMemsetAsync(b->scratch.p + b->hits_off, 0, b->hits_bytes, b->stream));  // every run counts from zero
    TQ_CUDA(cudaEventRecord(b->ev_k0, b->stream));
    if (b->n_units[UC_TERM]) timed(SPAN_TERM, [&] { k_term<<<b->n_units[UC_TERM], kThreads, 0, b->stream>>>(P, b->unit_base[UC_TERM]); });
    if (b->n_units[UC_AND]) timed(SPAN_AND, [&] { k_and<<<b->n_units[UC_AND], kThreads, 0, b->stream>>>(P, b->unit_base[UC_AND]); });
    if (b->n_units[UC_PHRASE]) {
      // phrase queries share nothing with the tile engine's launches (their own candidate regions; k_theta and the key export
      // skip them) and k_phrase waits on dependent position loads most of the time: it runs on a second stream next to them
      const int rc = launch_aside(b, tiles && b->ctx->phrase_side, [&](cudaStream_t on) -> int {
        const int sp = span_begin(b, SPAN_PHRASE, on);
        k_phrase<<<b->n_units[UC_PHRASE], kPhraseThreads, phrase_smem_bytes(b->phrase_ct), on>>>(P, b->ctx->d_pos_descs, b->phrase_aux, b->unit_base[UC_PHRASE], b->phrase_ct); ++launches;
        span_end(b, sp, on);
        return TQ_OK;
      });
      if (rc != TQ_OK) return rc;
    }
    if (b->n_units[UC_OR_WINDOW])  // window unions: every union the strip kernel does not take
      timed(SPAN_OR, [&] { k_or<<<b->n_units[UC_OR_WINDOW], kThreads, kOrDynSmem, b->stream>>>(P, b->unit_base[UC_OR_WINDOW]); });
    if (tiles) {  // K1 + K2 once for every distinct list of the batch
      const int sp = span_begin(b, SPAN_SCORE);
      for (auto& g : b->groups)
        if (g.n_chunks) { k_score_lists<<<g.n_chunks, kThreads, 0, b->stream>>>(P, g.params, 0u); ++launches; }
      span_end(b, sp);
      TQ_CUDA(cudaGetLastError());
    }
    if (b->count_hits) {
      // TQ_QUERY_COUNT_HITS: k_count_tiles reads the scored pairs and tile indexes, which nothing writes after k_score_lists, and
      // adds to counters of its own -- it runs on the second stream next to the k_tile launches (as k_phrase does); k_count for
      // the queries on the per-query kernels goes with it
      const int rc = launch_aside(b, tiles, [&](cudaStream_t on) -> int {
        const int sp = span_begin(b, SPAN_COUNT, on);
        for (auto& g : b->groups)
          if (g.n_count_units) { k_count_tiles<<<g.n_count_units, kTileThreads, g.count_smem, on>>>(g.params, g.count); ++launches; }
        if (b->n_count_units) { (b->count_mixed ? k_count<true> : k_count<false>)<<<b->n_count_units, kThreads, 0, on>>>(b->count_p); ++launches; }
        span_end(b, sp, on);
        TQ_CUDA(cudaGetLastError());
        return TQ_OK;
      });
      if (rc != TQ_OK) return rc;
    }
    b->stats.kernel_launches = 0;
  }
  if (phase < kPhases - 1) {
    // tile engine: phase 0 = sample launch, then exact launches; strips: threshold round `phase`
    if (tiles) {
      const int rc = launch_tile_round(b, phase, &launches);
      if (rc != TQ_OK) return rc;
    }
    const int r = UC_STRIP_ROUND1 + phase;
    if (b->n_units[r])
      timed(SPAN_OR, [&] { k_or_strip<<<b->n_units[r], kStripThreads, strip_smem_bytes(b->strip_cached_max), b->stream>>>(P, b->unit_base[r], b->strip_cached_max); });
    bool tile_round = false;
    for (auto& g : b->groups) tile_round = tile_round || g.n_units[phase];
    if ((b->n_units[r] || (tile_round && phase > 0)) && b->nq) timed(SPAN_THETA, [&] { k_theta<<<(unsigned)b->nq, kThreads, 0, b->stream>>>(P); });
    if (tile_round && phase == 0 && b->nq) {
      const TileParams& TP = b->groups[0].params;
      timed(SPAN_THETA, [&] { k_theta_samples<<<(unsigned)b->nq, kThreads, 0, b->stream>>>(P, TP.samples, TP.sample_count, TP.sample_cap, TP.th_hist); });
    }
    TQ_CUDA(cudaGetLastError());
    b->stats.kernel_launches += launches;
    b->next_phase = phase + 1;
    b->last_round_sampled = tile_round && phase == 0;
    return TQ_OK;
  }
  if (tiles) {
    const int rc = launch_tile_round(b, kTileRounds - 1, &launches);
    if (rc != TQ_OK) return rc;
  }
  if (b->n_units[UC_STRIP])
    timed(SPAN_OR, [&] { k_or_strip<<<b->n_units[UC_STRIP], kStripThreads, strip_smem_bytes(b->strip_cached_max), b->stream>>>(P, b->unit_base[UC_STRIP], b->strip_cached_max); });
  TQ_CUDA(cudaGetLastError());
  if (b->side_pending) { TQ_CUDA(cudaStreamWaitEvent(b->stream, b->ev_side1, 0)); b->side_pending = false; }
  if (b->nq) timed(SPAN_FINAL, [&] { k_final<<<b->nq, kThreads, 0, b->stream>>>(P); });
  TQ_CUDA(cudaGetLastError());
  if (tiles) TQ_CUDA(cudaMemcpyAsync(b->flags_pin, b->tile_dev.p + b->tile_flags_off, 16, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaEventRecord(b->ev_k1, b->stream));
  b->stats.kernel_launches += launches;
  b->next_phase = 0;
  b->ran = true;
  return TQ_OK;
}

// After the last phase: wait for the stream.  A run whose tile engine overflowed (a tile with more pairs than its buffer, or a
// query with more candidates than its region) is repeated and the repeat's rows replace ours, query by query.  In the repeat
// TERM / AND / OR / phrase queries take the per-query kernels, which have no such capacities; TQ_OP_BOOL queries, which have no
// per-query kernel, run on the tile engine again with regions that cannot overflow and the largest tile buffer (level 1).  If
// that buffer overflows too, they run once more in tile groups of one query each (level 2); a tile whose postings do not fit
// the buffer even for one query fails with TQ_ERR_TILE_CAPACITY.  Exactness never depends on the fast path's capacity guesses.
static int finalize_run(tq_batch* b) {
  if (!b->ran) return fail(TQ_ERR_INVALID_ARGUMENT, "batch has not run");
  if (b->finalized) return TQ_OK;
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  b->finalized = true;
  if (b->groups.empty()) return TQ_OK;
  const bool pairs_over = b->flags_pin[0] != 0, cands_over = b->flags_pin[1] != 0;
  if (!pairs_over && !cands_over) return TQ_OK;
  if (b->repeat == 2 && pairs_over)
    return fail(TQ_ERR_TILE_CAPACITY, "a TQ_OP_BOOL query has a 1024-doc tile whose postings exceed the tile buffer (12288 pairs) "
                                      "even in a tile group of its own: split the query or the segment");
  if (b->repeat && cands_over) return fail(TQ_ERR_CUDA, "a repeated TQ_OP_BOOL query overflowed a candidate region sized by its postings");
  int level = pairs_over ? 2 : 1;
  tq_batch* fb = nullptr;
  int rc = batch_prepare_impl(b->ctx, b->owned.q.data(), b->owned.q.size(), std::max(level, b->repeat + 1), &fb);
  if (rc == TQ_OK) rc = tq_batch_run(fb);
  if (rc == TQ_OK) rc = finalize_run(fb);  // (a level-1 repeat whose buffer overflowed repeats itself at level 2)
  if (rc == TQ_OK && fb->nq != b->nq) rc = fail(TQ_ERR_CUDA, "repeat batch holds other queries");
  if (rc == TQ_OK && b->nq) {
    const BatchParams& D = b->params;
    cudaError_t e = copy_rows(fb, b->stream, D.res_scores, D.res_segs, D.res_docs, D.res_counts, b->kmax);
    if (e == cudaSuccess) e = cudaStreamSynchronize(b->stream);
    if (e != cudaSuccess) rc = fail(TQ_ERR_CUDA, cudaGetErrorString(e));
  }
  if (fb) tq_batch_destroy(fb);
  b->stats.tile_fallbacks = 1;
  return rc;
}

// The start of every result entry point: the batch has run, no later run is in progress and the outputs are there; then the
// batch's device, and with `finalize` the run waited for and, if it overflowed, repeated (finalize_run).  Between the phases of
// a second run the rows and flags are still the first run's, and finalize_run would mark the run in progress as repaired.
static int results_ready(tq_batch* b, bool have_outputs, bool finalize) {
  if (!b || !b->ran) return fail(TQ_ERR_INVALID_ARGUMENT, "batch has not run");
  if (b->next_phase != 0) return fail(TQ_ERR_INVALID_ARGUMENT, "a run is in progress: finish its phases");
  if (!have_outputs) return fail(TQ_ERR_INVALID_ARGUMENT, "null output");
  TQ_CUDA(cudaSetDevice(b->ctx->device));
  return finalize ? finalize_run(b) : TQ_OK;
}

extern "C" {

int tq_batch_run(tq_batch* b) {
  if (!b) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  for (int p = b->next_phase; p < kPhases; ++p) {
    const int rc = run_phase(b, p);
    if (rc != TQ_OK) { b->next_phase = 0; return rc; }
  }
  return TQ_OK;
}

int tq_batch_phases(tq_batch* b) { return b ? kPhases : 0; }

int tq_batch_run_phase(tq_batch* b, int phase) {
  if (!b || phase < 0 || phase >= kPhases) return fail(TQ_ERR_INVALID_ARGUMENT, "batch / phase");
  const int rc = run_phase(b, phase);
  if (rc != TQ_OK && rc != TQ_ERR_INVALID_ARGUMENT) b->next_phase = 0;  // a failed run starts over
  return rc;
}

int tq_batch_stream(tq_batch* b, void** stream_out) {
  if (!b || !stream_out) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  *stream_out = (void*)b->stream;
  return TQ_OK;
}

int tq_batch_thresholds_export_dev(tq_batch* b, int64_t* keys_dev) {
  if (!b || !keys_dev || b->next_phase == 0) return fail(TQ_ERR_INVALID_ARGUMENT, "export needs a batch between two phases of a run");
  TQ_CUDA(cudaSetDevice(b->ctx->device));
  if (b->nq) k_theta_export<<<(unsigned)((b->nq + 255) / 256), 256, 0, b->stream>>>(b->params.qstate, reinterpret_cast<long long*>(keys_dev), (uint32_t)b->nq);
  TQ_CUDA(cudaGetLastError());
  TQ_CUDA(cudaStreamSynchronize(b->stream));  // the caller's collective runs on its own stream
  return TQ_OK;
}

int tq_batch_thresholds_import_dev(tq_batch* b, const int64_t* keys_dev) {
  if (!b || !keys_dev || b->next_phase == 0) return fail(TQ_ERR_INVALID_ARGUMENT, "import needs a batch between two phases of a run");
  TQ_CUDA(cudaSetDevice(b->ctx->device));
  if (b->nq) k_theta_import<<<(unsigned)((b->nq + 255) / 256), 256, 0, b->stream>>>(b->params.qstate, reinterpret_cast<const long long*>(keys_dev), (uint32_t)b->nq);
  TQ_CUDA(cudaGetLastError());
  return TQ_OK;
}

int tq_batch_topkeys_export_dev(tq_batch* b, uint32_t* keys_dev, uint32_t k_stride) {
  if (!b || !keys_dev || !k_stride || b->next_phase == 0) return fail(TQ_ERR_INVALID_ARGUMENT, "export needs a batch between two phases of a run");
  TQ_CUDA(cudaSetDevice(b->ctx->device));
  if (b->nq) {
    const bool from_samples = b->last_round_sampled && !b->groups.empty();
    const TileParams* TP = b->groups.empty() ? nullptr : &b->groups[0].params;
    k_topkeys_export<<<(unsigned)b->nq, kThreads, 0, b->stream>>>(b->params, TP ? TP->samples : nullptr, TP ? TP->sample_count : nullptr,
                                                                  TP ? TP->sample_cap : 0u, from_samples ? 1u : 0u, keys_dev, k_stride);
  }
  TQ_CUDA(cudaGetLastError());
  return TQ_OK;  // enqueued on the batch's stream (tq_batch_stream): the caller's collective must be ordered behind it
}

int tq_batch_thresholds_from_keys_dev(tq_batch* b, const uint32_t* gathered_dev, uint32_t n_shards, uint32_t k_stride) {
  if (!b || !gathered_dev || !n_shards || !k_stride || b->next_phase == 0) return fail(TQ_ERR_INVALID_ARGUMENT, "import needs a batch between two phases of a run");
  if ((size_t)n_shards * k_stride * 4 > 200u * 1024u) return fail(TQ_ERR_UNSUPPORTED, "n_shards * k_stride too large for one CTA");
  TQ_CUDA(cudaSetDevice(b->ctx->device));
  if (b->nq) {
    const size_t smem = (size_t)n_shards * k_stride * 4;
    if (smem > 48u * 1024u) TQ_CUDA(cudaFuncSetAttribute(k_theta_from_keys, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_theta_from_keys<<<(unsigned)b->nq, kThreads, smem, b->stream>>>(b->params, gathered_dev, n_shards, (uint32_t)b->nq, k_stride);
  }
  TQ_CUDA(cudaGetLastError());
  return TQ_OK;
}

int tq_batch_results_dev(tq_batch* b, const float** scores_dev, const uint32_t** segment_ord_dev, const uint32_t** doc_dev,
                         const uint32_t** count_dev, uint32_t* stride) {
  { const int rc = results_ready(b, true, true); if (rc != TQ_OK) return rc; }
  if (scores_dev) *scores_dev = b->params.res_scores;
  if (segment_ord_dev) *segment_ord_dev = b->params.res_segs;
  if (doc_dev) *doc_dev = b->params.res_docs;
  if (count_dev) *count_dev = b->params.res_counts;
  if (stride) *stride = b->kmax;
  publish_stats(b);
  return TQ_OK;
}

int tq_batch_results_copy_dev(tq_batch* b, float* scores_dev, uint32_t* segment_ord_dev, uint32_t* doc_dev, uint32_t* count_dev) {
  { const int rc = results_ready(b, scores_dev && segment_ord_dev && doc_dev && count_dev, true); if (rc != TQ_OK) return rc; }
  TQ_CUDA(copy_rows(b, b->stream, scores_dev, segment_ord_dev, doc_dev, count_dev, b->kmax));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  publish_stats(b);
  return TQ_OK;
}

int tq_batch_fetch(tq_batch* b, uint32_t out_stride, float* out_scores, uint32_t* out_segment_ord, uint32_t* out_doc, uint32_t* out_count) {
  // (a run without tile groups cannot overflow: it is not finalized, one sync below)
  { const int rc = results_ready(b, out_scores && out_segment_ord && out_doc && out_count, b && !b->groups.empty()); if (rc != TQ_OK) return rc; }
  TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, b->scratch.p + b->res_off, b->res_bytes, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaEventRecord(b->ev_end, b->stream));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  const float* rs = reinterpret_cast<const float*>(b->res_pin.p + b->res_at.scores);
  const uint32_t* rg = reinterpret_cast<const uint32_t*>(b->res_pin.p + b->res_at.segs);
  const uint32_t* rd = reinterpret_cast<const uint32_t*>(b->res_pin.p + b->res_at.docs);
  const uint32_t* rc = reinterpret_cast<const uint32_t*>(b->res_pin.p + b->res_at.counts);
  for (uint32_t q = 0; q < b->nq; ++q) {
    const uint32_t n = std::min(std::min(rc[q], b->kmax), out_stride);
    out_count[q] = rc[q];
    memcpy(out_scores + (size_t)q * out_stride, rs + (size_t)q * b->kmax, n * 4);
    memcpy(out_segment_ord + (size_t)q * out_stride, rg + (size_t)q * b->kmax, n * 4);
    memcpy(out_doc + (size_t)q * out_stride, rd + (size_t)q * b->kmax, n * 4);
  }
  float ms = 0;
  if (cudaEventElapsedTime(&ms, b->ev_start, b->ev_end) == cudaSuccess) b->stats.total_ms = ms;
  b->stats.d2h_bytes = b->res_bytes;
  publish_stats(b);
  return TQ_OK;
}

int tq_batch_fetch_hits(tq_batch* b, uint64_t* out_hits) {
  // (a repeat after a tile overflow does not count: these hits stand)
  { const int rc = results_ready(b, !b || out_hits || !b->nq, true); if (rc != TQ_OK) return rc; }
  for (uint32_t q = 0; q < b->nq; ++q) out_hits[q] = 0;
  if (!b->count_hits) return TQ_OK;
  TQ_CUDA(cudaMemcpyAsync(b->hits_pin.p, b->scratch.p + b->hits_off, b->hits_bytes, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  const uint64_t* hits = reinterpret_cast<const uint64_t*>(b->hits_pin.p);
  const uint32_t* ovf = reinterpret_cast<const uint32_t*>(hits + std::max<uint32_t>(b->nq, 1));
  for (uint32_t q = 0; q < b->nq; ++q) out_hits[q] = hits[q] + b->hits_host[q];
  // a group whose tile held more sparse offsets than k_count_tiles keeps: its queries are counted again by k_count
  for (size_t gi = 0; gi < b->groups.size(); ++gi) {
    const std::vector<uint32_t>& qs = b->groups[gi].count_queries;
    if (!ovf[gi] || qs.empty()) continue;
    std::vector<tq_query> sub(qs.size());
    std::vector<uint64_t> counts(qs.size());
    for (size_t i = 0; i < qs.size(); ++i) sub[i] = b->owned.q[qs[i]];
    const int rc = tq_count_batch(b->ctx, sub.data(), sub.size(), counts.data());
    if (rc != TQ_OK) return rc;
    for (size_t i = 0; i < qs.size(); ++i) out_hits[qs[i]] = counts[i];
  }
  return TQ_OK;
}

int tq_search_batch(tq_ctx* c, const tq_query* queries, size_t nq, uint32_t out_stride, float* out_scores, uint32_t* out_segment_ord,
                    uint32_t* out_doc, uint32_t* out_count) {
  tq_batch* b = nullptr;
  int rc = tq_batch_prepare(c, queries, nq, &b);
  if (rc != TQ_OK) return rc;
  rc = tq_batch_run(b);
  if (rc == TQ_OK) rc = tq_batch_fetch(b, out_stride, out_scores, out_segment_ord, out_doc, out_count);
  tq_batch_destroy(b);
  return rc;
}

int tq_merge_topk_dev(tq_ctx* c, uint32_t n_lists, uint32_t nq, uint32_t stride, uint32_t k, const float* scores_dev,
                      const uint32_t* segment_ord_dev, const uint32_t* doc_dev, const uint32_t* count_dev, float* out_scores_dev,
                      uint32_t* out_segment_ord_dev, uint32_t* out_doc_dev, uint32_t* out_count_dev) {
  if (!c) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  if (k == 0 || k > TQ_MAX_K || stride < 1) return fail(TQ_ERR_INVALID_ARGUMENT, "k / stride");
  TQ_CUDA(cudaSetDevice(c->device));
  if (nq == 0) return TQ_OK;
  k_merge<<<nq, kThreads, 0, 0>>>(n_lists, nq, stride, std::min(k, stride), (size_t)nq * stride, (size_t)nq, scores_dev, segment_ord_dev, doc_dev,
                                  count_dev, out_scores_dev, out_segment_ord_dev, out_doc_dev, out_count_dev);
  TQ_CUDA(cudaGetLastError());
  TQ_CUDA(cudaStreamSynchronize(0));
  return TQ_OK;
}

// Packed form for sharded callers: one buffer per shard = [nq*stride scores | nq*stride segment ords | nq*stride docs | nq counts]
// (32-bit words, what tq_batch_results_pack_dev writes), `n_lists` of them `pitch_words` apart -- the layout ONE all-gather
// produces.  Enqueued on `cuda_stream` (a cudaStream_t; e.g. the batch's, tq_batch_stream) without any host synchronisation.
int tq_merge_topk_packed_dev(tq_ctx* c, void* cuda_stream, uint32_t n_lists, uint32_t nq, uint32_t stride, uint32_t k, const uint32_t* packed_dev,
                             size_t pitch_words, uint32_t* out_packed_dev) {
  if (!c || !packed_dev || !out_packed_dev) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  if (k == 0 || k > TQ_MAX_K || stride < 1 || pitch_words < (size_t)3 * nq * stride + nq) return fail(TQ_ERR_INVALID_ARGUMENT, "k / stride / pitch");
  TQ_CUDA(cudaSetDevice(c->device));
  if (nq == 0) return TQ_OK;
  const size_t rows = (size_t)nq * stride;
  k_merge<<<nq, kThreads, 0, (cudaStream_t)cuda_stream>>>(n_lists, nq, stride, std::min(k, stride), pitch_words, pitch_words,
                                                          reinterpret_cast<const float*>(packed_dev), packed_dev + rows, packed_dev + 2 * rows,
                                                          packed_dev + 3 * rows, reinterpret_cast<float*>(out_packed_dev), out_packed_dev + rows,
                                                          out_packed_dev + 2 * rows, out_packed_dev + 3 * rows);
  TQ_CUDA(cudaGetLastError());
  return TQ_OK;
}

// The result rows of a finished run in the packed layout above (row stride = k_max of the batch), into a caller-owned DEVICE buffer
// of 3 * nq * k_max + nq words.  Waits for the run (a tile-engine overflow is resolved first), then copies on the batch's stream.
int tq_batch_results_pack_dev(tq_batch* b, uint32_t* packed_dev) {
  { const int rc = results_ready(b, packed_dev, true); if (rc != TQ_OK) return rc; }
  const size_t rows = (size_t)b->nq * b->kmax;
  TQ_CUDA(copy_rows(b, b->stream, reinterpret_cast<float*>(packed_dev), packed_dev + rows, packed_dev + 2 * rows, packed_dev + 3 * rows, b->kmax));
  publish_stats(b);
  return TQ_OK;
}

// The same rows WITHOUT waiting for the run: everything is enqueued on the batch's stream right behind the run's last kernel, so a
// sharded caller can queue pack -> all-gather -> merge -> the next batch's run and only then wait for this one (two batches in
// flight).  packed_dev holds 3 * nq * k_max + nq + 4 words; the last four are the run's overflow flags -- all zero: the rows are
// final; anything else: the tile engine overflowed a buffer and the caller must take tq_batch_results_pack_dev (which repeats the
// run, see finalize_run) instead.  The flags travel with the rows, so every shard sees every shard's.
int tq_batch_results_pack_dev_async(tq_batch* b, uint32_t* packed_dev) {
  { const int rc = results_ready(b, packed_dev, false); if (rc != TQ_OK) return rc; }
  const size_t rows = (size_t)b->nq * b->kmax;
  TQ_CUDA(copy_rows(b, b->stream, reinterpret_cast<float*>(packed_dev), packed_dev + rows, packed_dev + 2 * rows, packed_dev + 3 * rows, b->kmax));
  uint32_t* flags = packed_dev + 3 * rows + b->nq;
  if (!b->groups.empty() && !b->finalized)
    TQ_CUDA(cudaMemcpyAsync(flags, b->tile_dev.p + b->tile_flags_off, 16, cudaMemcpyDeviceToDevice, b->stream));
  else
    TQ_CUDA(cudaMemsetAsync(flags, 0, 16, b->stream));  // (per-query kernels cannot overflow; a finalized run has been repaired already)
  return TQ_OK;
}

// ---- Count collector -------------------------------------------------------------------------------------------
int tq_count_batch(tq_ctx* c, const tq_query* queries, size_t nq, uint64_t* out_counts) {
  if (!c || (!queries && nq) || (!out_counts && nq)) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  for (size_t qi = 0; qi < nq; ++qi) out_counts[qi] = 0;
  if (!nq) return TQ_OK;
  tq_batch* b = acquire_batch(c);
  if (!b) return fail(TQ_ERR_CUDA, "stream/event creation failed");
  struct Guard { tq_batch* b; ~Guard() { tq_batch_destroy(b); } } guard{b};
  CountPlan cp;
  {
    std::lock_guard<std::mutex> g(c->mu);
    TableScope table_scope{c};
    uint64_t built = 0;
    std::vector<const tq_term_seg*> order;
    for (size_t qi = 0; qi < nq; ++qi) {
      const int rc = plan_count(c, queries[qi], (uint32_t)qi, order, cp, &out_counts[qi]);
      if (rc != TQ_OK) return rc;
    }
    int rc = flush_builds(c, &built);
    if (rc != TQ_OK) return rc;
    hold_filters(c, b, queries, nq);  // (their views stay until the counts are in: the guard's tq_batch_destroy lets go)
  }
  if (cp.units.empty()) return TQ_OK;
  return count_on_device(b, cp.words, cp.segs, cp.units, cp.mixed, nq, out_counts);
}

// ---- sort by a fast field -------------------------------------------------------------------------------------
int tq_sort_batch(tq_ctx* c, const tq_query* queries, const tq_sort_spec* sorts, size_t nq, uint32_t out_stride, uint64_t* out_values,
                  uint8_t* out_present, uint32_t* out_segment_ord, uint32_t* out_doc, uint32_t* out_count, uint64_t* out_hits) {
  if (!c || (nq && (!queries || !sorts || !out_values || !out_present || !out_segment_ord || !out_doc || !out_count)))
    return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  uint32_t kmax = 1;
  for (size_t qi = 0; qi < nq; ++qi) {
    if (queries[qi].op == TQ_OP_PHRASE) return fail(TQ_ERR_UNSUPPORTED, "sorting phrase queries by a fast field is not on the device path");
    if (queries[qi].k == 0 || queries[qi].k > TQ_MAX_K) return fail(TQ_ERR_INVALID_ARGUMENT, "k must be in 1..TQ_MAX_K");
    if (sorts[qi].order != TQ_ORDER_DESC && sorts[qi].order != TQ_ORDER_ASC) return fail(TQ_ERR_INVALID_ARGUMENT, "order");
    kmax = std::max(kmax, queries[qi].k);
  }
  if (out_stride < kmax) return fail(TQ_ERR_INVALID_ARGUMENT, "out_stride must hold k rows");
  for (size_t qi = 0; qi < nq; ++qi) { out_count[qi] = 0; if (out_hits) out_hits[qi] = 0; }
  if (!nq) return TQ_OK;
  tq_batch* b = acquire_batch(c);
  if (!b) return fail(TQ_ERR_CUDA, "stream/event creation failed");
  struct Guard { tq_batch* b; ~Guard() { tq_batch_destroy(b); } } guard{b};
  CountPlan cp;
  std::vector<SortSeg> ssegs;
  std::vector<SortQuery> sq(nq);
  uint64_t n_cands = 0;
  {
    std::lock_guard<std::mutex> g(c->mu);
    TableScope table_scope{c};
    uint64_t built = 0, unused = 0;
    std::vector<const tq_term_seg*> order;
    std::vector<std::pair<unsigned long long, Unit>> by_bound;
    for (size_t qi = 0; qi < nq; ++qi) {
      const size_t s0 = cp.segs.size(), u0 = cp.units.size();
      int rc = plan_count(c, queries[qi], (uint32_t)qi, order, cp, &unused, true);
      if (rc != TQ_OK) return rc;
      const bool asc = sorts[qi].order == TQ_ORDER_ASC;
      std::vector<const SortColumn*> cols;
      for (size_t si = s0; si < cp.segs.size(); ++si) {
        auto it = c->sort_columns.find({sorts[qi].column_id, cp.segment_ords[si]});
        if (it == c->sort_columns.end()) return fail(TQ_ERR_NOT_FOUND, "a sorted query names a segment without the sort column (tq_sort_column_register)");
        const SortColumn& col = it->second;
        if (col.tiles.size() != (cp.segs[si].max_doc + kTileDocs - 1) / kTileDocs) return fail(TQ_ERR_INVALID_ARGUMENT, "sort column and segment differ in max_doc");
        ssegs.push_back(SortSeg{col.d_values, col.d_present, col.d_tiles, cp.segment_ords[si], 0u});
        cols.push_back(&col);
      }
      // the units with the best possible keys first: they raise the bound that lets the later ones skip their tiles
      by_bound.clear();
      for (size_t ui = u0; ui < cp.units.size(); ++ui) {
        const Unit& u = cp.units[ui];
        const std::vector<SortTile>& tiles = cols[u.qseg - s0]->tiles;
        unsigned long long best = 0;
        bool none = false;
        for (uint32_t t = u.begin; t < u.end; ++t) {
          if (tiles[t].flags & kSortTileValues) best = std::max(best, tiles[t].best[asc ? 1 : 0]);
          none = none || (tiles[t].flags & kSortTileNone);
        }
        // (a unit collects its None docs in doc order, so only a unit without any may walk backwards)
        const bool backward = !none && tiles[u.end - 1].best[asc ? 1 : 0] > tiles[u.begin].best[asc ? 1 : 0];
        by_bound.emplace_back(best, Unit{u.qseg, u.begin, u.end, backward ? kSortUnitBackward : 0u});
      }
      std::stable_sort(by_bound.begin(), by_bound.end(), [](const auto& x, const auto& y) { return x.first > y.first; });
      for (size_t i = 0; i < by_bound.size(); ++i) cp.units[u0 + i] = by_bound[i].second;
      sq[qi] = SortQuery{queries[qi].k, (asc ? kSortAsc : 0u) | (out_hits ? kSortAllTiles : 0u), (uint32_t)n_cands, 0u};
      n_cands += (uint64_t)(cp.units.size() - u0) * queries[qi].k;
    }
    if (n_cands > 0xFFFFFFFFull) return fail(TQ_ERR_INVALID_ARGUMENT, "batch too large: split it");
    int rc = flush_builds(c, &built);
    if (rc != TQ_OK) return rc;
    hold_segments(c, b, queries, nq);  // (the segments, their filter views and the columns stay until the rows are in)
    for (size_t qi = 0; qi < nq; ++qi) b->held_columns.push_back(sorts[qi].column_id);
    std::sort(b->held_columns.begin(), b->held_columns.end());
    b->held_columns.erase(std::unique(b->held_columns.begin(), b->held_columns.end()), b->held_columns.end());
    for (uint32_t col : b->held_columns) ++c->sort_users[col];
  }
  if (cp.units.empty()) return TQ_OK;
  // descriptors: one H2D copy; scratch: results | hits | tile counters (one D2H copy), then the per-query state and candidates
  Staging st;
  const size_t o_w = st.add(cp.words), o_s = st.add(cp.segs), o_u = st.add(cp.units), o_z = st.add(ssegs), o_q = st.add(sq);
  TQ_CUDA(st.reserve(b->pin, b->dev));
  st.copy();
  const size_t rows = nq * (size_t)kmax;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off = align256(off + bytes); return at; };
  const size_t r_values = take(rows * 8), r_hits = take(nq * 8), r_tiles = take(16), r_segs = take(rows * 4), r_docs = take(rows * 4),
               r_counts = take(nq * 4), r_present = take(rows), res_bytes = off;
  const size_t r_qstate = take(nq * sizeof(SortQState)), r_cands = take(n_cands * sizeof(SortCand)), r_nones = take(n_cands * sizeof(SortCand));
  TQ_CUDA(b->scratch.ensure(off));
  TQ_CUDA(b->res_pin.ensure(res_bytes));
  uint8_t* const d = b->scratch.p;
  SortParams P{};
  P.c = CountParams{c->d_lists, st.on_device<const uint32_t>(o_w), st.on_device<const CountSeg>(o_s), st.on_device<const Unit>(o_u),
                    reinterpret_cast<unsigned long long*>(d + r_hits)};
  P.ssegs = st.on_device<const SortSeg>(o_z);
  P.queries = st.on_device<const SortQuery>(o_q);
  P.qstate = reinterpret_cast<SortQState*>(d + r_qstate);
  P.cands = reinterpret_cast<SortCand*>(d + r_cands);
  P.nones = reinterpret_cast<SortCand*>(d + r_nones);
  P.tiles = reinterpret_cast<unsigned long long*>(d + r_tiles);
  P.res_values = reinterpret_cast<unsigned long long*>(d + r_values);
  P.res_present = d + r_present;
  P.res_segs = reinterpret_cast<uint32_t*>(d + r_segs);
  P.res_docs = reinterpret_cast<uint32_t*>(d + r_docs);
  P.res_counts = reinterpret_cast<uint32_t*>(d + r_counts);
  P.res_stride = kmax;
  TQ_CUDA(cudaMemcpyAsync(b->dev.p, b->pin.p, st.bytes, cudaMemcpyHostToDevice, b->stream));
  TQ_CUDA(cudaMemsetAsync(d + r_hits, 0, r_segs - r_hits, b->stream));  // hits, tile counters
  TQ_CUDA(cudaMemsetAsync(d + r_counts, 0, nq * 4, b->stream));
  TQ_CUDA(cudaMemsetAsync(d + r_qstate, 0, nq * sizeof(SortQState), b->stream));
  TQ_CUDA(cudaEventRecord(b->ev_k0, b->stream));
  (cp.mixed ? k_sort<true> : k_sort<false>)<<<(unsigned)cp.units.size(), kThreads, 0, b->stream>>>(P);
  TQ_CUDA(cudaGetLastError());
  k_sort_final<<<(unsigned)nq, kThreads, 0, b->stream>>>(P);
  TQ_CUDA(cudaGetLastError());
  TQ_CUDA(cudaEventRecord(b->ev_k1, b->stream));
  TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d, res_bytes, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  const uint8_t* h = b->res_pin.p;
  const uint32_t* counts = reinterpret_cast<const uint32_t*>(h + r_counts);
  for (size_t qi = 0; qi < nq; ++qi) {
    const size_t src = qi * kmax, dst = qi * (size_t)out_stride, n = counts[qi];
    out_count[qi] = counts[qi];
    memcpy(out_values + dst, h + r_values + src * 8, n * 8);
    memcpy(out_present + dst, h + r_present + src, n);
    memcpy(out_segment_ord + dst, h + r_segs + src * 4, n * 4);
    memcpy(out_doc + dst, h + r_docs + src * 4, n * 4);
    if (out_hits) memcpy(&out_hits[qi], h + r_hits + qi * 8, 8);
  }
  float ms = 0;
  cudaEventElapsedTime(&ms, b->ev_k0, b->ev_k1);
  unsigned long long tiles[2];
  memcpy(tiles, h + r_tiles, 16);
  std::lock_guard<std::mutex> g(c->mu);
  c->sort_ms += ms;
  c->sort_units += cp.units.size() + nq;
  c->sort_tiles_seen += tiles[0];
  c->sort_tiles_skipped += tiles[1];
  return TQ_OK;
}

// ---- histogram of a fast field ---------------------------------------------------------------------------------
// The smallest and largest image of the unit's tiles that hold a value; false: none does.
static bool unit_images(const SortColumn& col, const Unit& u, unsigned long long& lo, unsigned long long& hi) {
  bool any = false;
  lo = ~0ull;
  hi = 0;
  for (uint32_t t = u.begin; t < u.end; ++t) {
    const SortTile& st = col.tiles[t];
    if (!(st.flags & kSortTileValues)) continue;
    lo = std::min<unsigned long long>(lo, ~st.best[1]);
    hi = std::max<unsigned long long>(hi, st.best[0]);
    any = true;
  }
  return any;
}

// The histogram side of one query's plan, after plan_count added its (query, segment)s from s0 and units from u0: per (query,
// segment) its column and bounds after normalize_histogram_req's collapse (hsegs, cols), per unit the first and last pos its tiles'
// values in bounds can take (uwin; first > last: none), and the query's dense range [base, base + len) (compute_dense_range,
// histogram.rs:751-769, over the visited tiles only).  A range above max_bins is TQ_ERR_UNSUPPORTED.
// The registered column column_id of each (query, segment) plan_count added from s0, into cols.  `what` names the query in the
// errors: a segment without the column is TQ_ERR_NOT_FOUND, one whose max_doc differs TQ_ERR_INVALID_ARGUMENT.
static int find_columns(tq_ctx* c, uint32_t column_id, const CountPlan& cp, size_t s0, const char* what, std::vector<const SortColumn*>& cols) {
  cols.clear();
  for (size_t si = s0; si < cp.segs.size(); ++si) {
    auto it = c->sort_columns.find({column_id, cp.segment_ords[si]});
    if (it == c->sort_columns.end()) return fail(TQ_ERR_NOT_FOUND, std::string(what) + " names a segment without the column (tq_sort_column_register)");
    const SortColumn& col = it->second;
    if (col.tiles.size() != (cp.segs[si].max_doc + kTileDocs - 1) / kTileDocs) return fail(TQ_ERR_INVALID_ARGUMENT, "column and segment differ in max_doc");
    cols.push_back(&col);
  }
  return TQ_OK;
}

static int plan_hist_query(tq_ctx* c, const tq_histogram_spec& sp, size_t qi, const CountPlan& cp, size_t s0, size_t u0, uint32_t max_bins,
                           std::vector<HistSeg>& hsegs, std::vector<const SortColumn*>& cols, std::vector<std::pair<long long, long long>>& uwin,
                           long long& base, uint64_t& len) {
  int rc = find_columns(c, sp.column_id, cp, s0, "a histogram query", cols);
  if (rc != TQ_OK) return rc;
  for (const SortColumn* col : cols) {
    // normalize_histogram_req: the hard bounds collapse to every finite value when the segment's column lies inside them
    double lo = sp.hard_min, hi = sp.hard_max;
    if (col->min_image <= col->max_image && hist_value(col->min_image, sp.kind) >= lo && hist_value(col->max_image, sp.kind) <= hi) {
      lo = -DBL_MAX;
      hi = DBL_MAX;
    }
    hsegs.push_back(HistSeg{col->d_values, col->d_present, col->d_tiles, lo, hi});
  }
  // per unit: the buckets of its tiles' values, clipped to its segment's bounds; the query's dense range (compute_dense_range,
  // histogram.rs:751-769, over the visited tiles only) is their union
  uwin.clear();
  long long top = -1;
  base = 0;
  bool any = false;
  for (size_t ui = u0; ui < cp.units.size(); ++ui) {
    const Unit& u = cp.units[ui];
    const size_t k = u.qseg - s0;
    const HistSeg& z = hsegs[u.qseg];
    double umin = INFINITY, umax = -INFINITY;
    if (sp.kind == TQ_FAST_F64) {
      for (uint32_t t = u.begin; t < u.end; ++t) {  // an infinity widens the range only when it is in bounds; a NaN never is
        const FiniteTile& f = cols[k]->finite[t];
        double vmin = INFINITY, vmax = -INFINITY;
        if (f.flags & kFiniteAny) { vmin = hist_value(f.lo, sp.kind); vmax = hist_value(f.hi, sp.kind); }
        if ((f.flags & kFiniteNegInf) && z.lo == -INFINITY) vmin = -INFINITY;
        if ((f.flags & kFinitePosInf) && z.hi == INFINITY) vmax = INFINITY;
        umin = std::min(umin, vmin);
        umax = std::max(umax, vmax);
      }
    } else {
      unsigned long long ilo, ihi;  // (hist_value is monotone in the image for every other kind)
      if (unit_images(*cols[k], u, ilo, ihi)) { umin = hist_value(ilo, sp.kind); umax = hist_value(ihi, sp.kind); }
    }
    const double lo = std::max(umin, z.lo), hi = std::min(umax, z.hi);
    if (!(lo <= hi)) { uwin.emplace_back(1, 0); continue; }  // no value of the unit can pass the bounds
    const long long p0 = hist_pos(lo, sp.offset, sp.interval), p1 = hist_pos(hi, sp.offset, sp.interval);
    uwin.emplace_back(p0, p1);
    base = any ? std::min(base, p0) : p0;
    top = any ? std::max(top, p1) : p1;
    any = true;
  }
  const __int128 n = any ? (__int128)top - base + 1 : 0;
  if (n > max_bins)
    return fail(TQ_ERR_UNSUPPORTED, "query " + std::to_string(qi) + ": its histogram spans more than 2^" + std::to_string(31 - __builtin_clz(max_bins)) +
                                        " buckets (take the CPU path)");
  len = (uint64_t)n;
  return TQ_OK;
}

int tq_histogram_batch(tq_ctx* c, const tq_query* queries, const tq_histogram_spec* specs, size_t nq, uint32_t out_stride,
                       int64_t* out_pos, uint64_t* out_doc_count, uint32_t* out_n, uint64_t* out_hits) {
  if (!c || (nq && (!queries || !specs || !out_n || (out_stride && (!out_pos || !out_doc_count)))))
    return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  for (size_t qi = 0; qi < nq; ++qi) {
    if (queries[qi].op == TQ_OP_PHRASE) return fail(TQ_ERR_UNSUPPORTED, "histograms of phrase queries are not on the device path");
    if (specs[qi].kind > TQ_FAST_DATE) return fail(TQ_ERR_INVALID_ARGUMENT, "histogram kind");
    if (!(specs[qi].interval > 0.0) || !std::isfinite(specs[qi].interval)) return fail(TQ_ERR_INVALID_ARGUMENT, "histogram interval must be finite and > 0");
  }
  for (size_t qi = 0; qi < nq; ++qi) { out_n[qi] = 0; if (out_hits) out_hits[qi] = 0; }
  if (!nq) return TQ_OK;
  tq_batch* b = acquire_batch(c);
  if (!b) return fail(TQ_ERR_CUDA, "stream/event creation failed");
  struct Guard { tq_batch* b; ~Guard() { tq_batch_destroy(b); } } guard{b};
  CountPlan cp;
  std::vector<HistSeg> hsegs;
  std::vector<HistQuery> hq(nq);
  std::vector<HistUnit> hunits;  // parallel to cp.units
  uint64_t n_counters = 0;
  {
    std::lock_guard<std::mutex> g(c->mu);
    TableScope table_scope{c};
    uint64_t built = 0, unused = 0;
    std::vector<const tq_term_seg*> order;
    std::vector<const SortColumn*> cols;
    std::vector<std::pair<long long, long long>> uwin;  // per unit of the query: its first and last pos (first > last: none)
    for (size_t qi = 0; qi < nq; ++qi) {
      const tq_histogram_spec& sp = specs[qi];
      const size_t s0 = cp.segs.size(), u0 = cp.units.size();
      int rc = plan_count(c, queries[qi], (uint32_t)qi, order, cp, &unused, true);
      if (rc != TQ_OK) return rc;
      long long base = 0;
      uint64_t len = 0;
      rc = plan_hist_query(c, sp, qi, cp, s0, u0, kHistMaxBins, hsegs, cols, uwin, base, len);
      if (rc != TQ_OK) return rc;
      for (const auto& w : uwin)
        hunits.push_back(w.first <= w.second ? HistUnit{(uint32_t)(w.first - base), (uint32_t)(w.second - w.first + 1)} : HistUnit{0u, 0u});
      hq[qi] = HistQuery{sp.interval, sp.offset, base, n_counters, (uint32_t)len, sp.kind, out_hits ? kHistHits : 0u, 0u};
      n_counters += (uint64_t)len;
    }
    if (n_counters > (1ull << 27)) return fail(TQ_ERR_INVALID_ARGUMENT, "batch too large: its histograms hold more than 2^27 buckets, split it");
    int rc = flush_builds(c, &built);
    if (rc != TQ_OK) return rc;
    hold_segments(c, b, queries, nq);  // (the segments, their filter views and the columns stay until the rows are in)
    for (size_t qi = 0; qi < nq; ++qi) b->held_columns.push_back(specs[qi].column_id);
    std::sort(b->held_columns.begin(), b->held_columns.end());
    b->held_columns.erase(std::unique(b->held_columns.begin(), b->held_columns.end()), b->held_columns.end());
    for (uint32_t col : b->held_columns) ++c->sort_users[col];
  }
  if (cp.units.empty()) return TQ_OK;
  // descriptors: one H2D copy; scratch: row lengths | hits | tile counters (read back first), the rows (read back as wide as the
  // longest), then the counters
  Staging st;
  const size_t o_w = st.add(cp.words), o_s = st.add(cp.segs), o_u = st.add(cp.units), o_z = st.add(hsegs), o_q = st.add(hq),
               o_h = st.add(hunits);
  TQ_CUDA(st.reserve(b->pin, b->dev));
  st.copy();
  const size_t rows = nq * (size_t)out_stride;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off = align256(off + bytes); return at; };
  const size_t r_n = take(nq * 4), r_hits = take(nq * 8), r_tiles = take(16), head_bytes = off;
  const size_t r_pos = take(rows * 8), r_count = take(rows * 8), r_counters = take(n_counters * 8);
  TQ_CUDA(b->scratch.ensure(off));
  TQ_CUDA(b->res_pin.ensure(r_counters));
  uint8_t* const d = b->scratch.p;
  HistParams P{};
  P.c = CountParams{c->d_lists, st.on_device<const uint32_t>(o_w), st.on_device<const CountSeg>(o_s), st.on_device<const Unit>(o_u),
                    reinterpret_cast<unsigned long long*>(d + r_hits)};
  P.hsegs = st.on_device<const HistSeg>(o_z);
  P.queries = st.on_device<const HistQuery>(o_q);
  P.hunits = st.on_device<const HistUnit>(o_h);
  P.counts = reinterpret_cast<unsigned long long*>(d + r_counters);
  P.tiles = reinterpret_cast<unsigned long long*>(d + r_tiles);
  P.res_pos = reinterpret_cast<long long*>(d + r_pos);
  P.res_count = reinterpret_cast<unsigned long long*>(d + r_count);
  P.res_n = reinterpret_cast<uint32_t*>(d + r_n);
  P.res_stride = out_stride;
  TQ_CUDA(cudaMemcpyAsync(b->dev.p, b->pin.p, st.bytes, cudaMemcpyHostToDevice, b->stream));
  TQ_CUDA(cudaMemsetAsync(d + r_hits, 0, head_bytes - r_hits, b->stream));  // hits, tile counters
  TQ_CUDA(cudaMemsetAsync(d + r_counters, 0, n_counters * 8, b->stream));
  TQ_CUDA(cudaEventRecord(b->ev_k0, b->stream));
  (cp.mixed ? k_hist<true> : k_hist<false>)<<<(unsigned)cp.units.size(), kThreads, 0, b->stream>>>(P);
  TQ_CUDA(cudaGetLastError());
  k_hist_final<<<(unsigned)nq, kThreads, 0, b->stream>>>(P);
  TQ_CUDA(cudaGetLastError());
  TQ_CUDA(cudaEventRecord(b->ev_k1, b->stream));
  TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d, head_bytes, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  const uint8_t* h = b->res_pin.p;
  memcpy(out_n, h + r_n, nq * 4);
  uint32_t widest = 0;
  for (size_t qi = 0; qi < nq; ++qi) widest = std::max(widest, out_n[qi]);
  const bool fits = widest <= out_stride;
  if (fits && widest) {  // the rows, only as wide as the longest
    TQ_CUDA(cudaMemcpy2DAsync(b->res_pin.p + r_pos, (size_t)out_stride * 8, d + r_pos, (size_t)out_stride * 8, (size_t)widest * 8, nq,
                              cudaMemcpyDeviceToHost, b->stream));
    TQ_CUDA(cudaMemcpy2DAsync(b->res_pin.p + r_count, (size_t)out_stride * 8, d + r_count, (size_t)out_stride * 8, (size_t)widest * 8, nq,
                              cudaMemcpyDeviceToHost, b->stream));
    TQ_CUDA(cudaStreamSynchronize(b->stream));
  }
  for (size_t qi = 0; fits && qi < nq; ++qi) {
    const size_t at = qi * (size_t)out_stride;
    memcpy(out_pos + at, h + r_pos + at * 8, (size_t)out_n[qi] * 8);
    memcpy(out_doc_count + at, h + r_count + at * 8, (size_t)out_n[qi] * 8);
    if (out_hits) memcpy(&out_hits[qi], h + r_hits + qi * 8, 8);
  }
  float ms = 0;
  cudaEventElapsedTime(&ms, b->ev_k0, b->ev_k1);
  unsigned long long tiles[2];
  memcpy(tiles, h + r_tiles, 16);
  {
    std::lock_guard<std::mutex> g(c->mu);
    c->hist_ms += ms;
    c->hist_units += cp.units.size() + nq;
    c->hist_tiles_seen += tiles[0];
    c->hist_tiles_one_bucket += tiles[1];
  }
  if (!fits) return fail(TQ_ERR_INVALID_ARGUMENT, "a histogram has more non-empty buckets than out_stride: out_n holds how many");
  return TQ_OK;
}

// ---- terms of a fast field ------------------------------------------------------------------------------------
// The terms of query qi (tq_terms_batch, tq_terms_metrics_batch): one TermsSeg per (query, segment) plan_count added from s0, its
// counters and region relative to the query (counters / region: the query's totals), and one window per unit added from u0.
static int plan_terms_query(tq_ctx* c, const tq_terms_spec& sp, size_t qi, uint32_t flags, const CountPlan& cp, size_t s0, size_t u0,
                            std::vector<TermsSeg>& tsegs, std::vector<HistUnit>& windows, std::vector<const SortColumn*>& cols,
                            std::vector<std::pair<unsigned long long, unsigned long long>>& uwin, uint64_t& counters, uint64_t& region) {
  cols.clear();
  for (size_t si = s0; si < cp.segs.size(); ++si) {
    auto it = c->sort_columns.find({sp.column_id, cp.segment_ords[si]});
    if (it == c->sort_columns.end()) return fail(TQ_ERR_NOT_FOUND, "a terms query names a segment without the column (tq_sort_column_register)");
    const SortColumn& col = it->second;
    if (col.tiles.size() != (cp.segs[si].max_doc + kTileDocs - 1) / kTileDocs) return fail(TQ_ERR_INVALID_ARGUMENT, "column and segment differ in max_doc");
    unsigned long long missing = sp.missing_image;
    if (sp.missing_mode == TQ_TERMS_MISSING_AFTER_MAX) {  // get_missing_val_as_u64_lenient: the column's max_value + 1 (0 without values)
      const unsigned long long top = col.min_image <= col.max_image ? col.max_image : 0ull;
      if (top == ~0ull) return fail(TQ_ERR_INVALID_ARGUMENT, "query " + std::to_string(qi) + ": a str column whose largest image is 2^64 - 1 has no missing key");
      missing = top + 1;
    }
    // a segment this context evaluates only part of (tq_segment_set_doc_range) is not cut here: the reference cuts a segment
    // once, so the caller cuts after summing its ranges; segment_size 0 marks it (every entry is kept, both scalars stay 0)
    bool part = false;
    for (auto s = c->segments.lower_bound({cp.segment_ords[si], 0u}); s != c->segments.end() && s->first.first == cp.segment_ords[si]; ++s)
      part = part || s->second.doc_lo != 0 || s->second.doc_hi != s->second.max_doc;
    tsegs.push_back(TermsSeg{col.d_values, col.d_present, col.d_tiles, 0ull, missing, 0ull, 0ull, 0u, part ? 0u : sp.segment_size, flags, 0u});
    cols.push_back(&col);
  }
  // per unit the images of its tiles; per (query, segment) their union
  uwin.clear();
  for (size_t ui = u0; ui < cp.units.size(); ++ui) {
    const Unit& u = cp.units[ui];
    unsigned long long lo, hi;
    if (!unit_images(*cols[u.qseg - s0], u, lo, hi)) { uwin.emplace_back(1ull, 0ull); continue; }
    uwin.emplace_back(lo, hi);
    TermsSeg& z = tsegs[u.qseg];
    if (!z.n_keys) { z.base = lo; z.n_keys = 1; z.region = hi; }  // (region holds the top until the span is known)
    else { z.base = std::min(z.base, lo); z.region = std::max<unsigned long long>(z.region, hi); }
  }
  for (size_t si = s0; si < cp.segs.size(); ++si) {
    TermsSeg& z = tsegs[si];
    if (z.n_keys) {
      const unsigned long long span_m1 = z.region - z.base;  // (images up to 2^64 - 1: the span is never formed as top + 1)
      if (span_m1 >= kTermsMaxKeys)
        return fail(TQ_ERR_UNSUPPORTED, "query " + std::to_string(qi) + ": its terms span more than 2^20 keys in a segment (take the CPU path)");
      z.n_keys = (uint32_t)span_m1 + 1u;
    }
    if (!z.segment_size) z.segment_size = z.n_keys + 1u;  // more than its entries: no cut
    z.counters = counters;
    z.region = region;
    counters += z.n_keys;
    region += std::min<uint64_t>(z.segment_size, (uint64_t)z.n_keys + ((z.flags & kTermsMissing) ? 1u : 0u));
  }
  for (size_t ui = u0; ui < cp.units.size(); ++ui) {
    const auto& w = uwin[ui - u0];
    windows.push_back(w.first <= w.second ? HistUnit{(uint32_t)(w.first - tsegs[cp.units[ui].qseg].base), (uint32_t)(w.second - w.first + 1)}
                                          : HistUnit{0u, 0u});
  }
  return TQ_OK;
}

int tq_terms_batch(tq_ctx* c, const tq_query* queries, const tq_terms_spec* specs, size_t nq, uint32_t out_stride,
                   uint32_t* out_segment_ord, uint64_t* out_key, uint64_t* out_doc_count, uint32_t* out_n, uint64_t* out_sum_other,
                   uint64_t* out_error_bound, uint64_t* out_hits) {
  if (!c || (nq && (!queries || !specs || !out_n || !out_sum_other || !out_error_bound ||
                    (out_stride && (!out_segment_ord || !out_key || !out_doc_count)))))
    return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  for (size_t qi = 0; qi < nq; ++qi) {
    const tq_terms_spec& sp = specs[qi];
    if (queries[qi].op == TQ_OP_PHRASE) return fail(TQ_ERR_UNSUPPORTED, "terms of phrase queries are not on the device path");
    if (sp.target > TQ_TERMS_BY_KEY || sp.order > TQ_ORDER_ASC || sp.missing_mode > TQ_TERMS_MISSING_AFTER_MAX || !sp.segment_size)
      return fail(TQ_ERR_INVALID_ARGUMENT, "terms spec: target, order, missing mode or segment_size");
  }
  for (size_t qi = 0; qi < nq; ++qi) {
    out_n[qi] = 0;
    out_sum_other[qi] = out_error_bound[qi] = 0;
    if (out_hits) out_hits[qi] = 0;
  }
  if (!nq) return TQ_OK;
  tq_batch* b = acquire_batch(c);
  if (!b) return fail(TQ_ERR_CUDA, "stream/event creation failed");
  struct Guard { tq_batch* b; ~Guard() { tq_batch_destroy(b); } } guard{b};
  CountPlan cp;
  std::vector<TermsSeg> tsegs;    // parallel to cp.segs
  std::vector<HistUnit> windows;  // parallel to cp.units
  std::vector<size_t> q_seg(nq + 1), q_unit(nq + 1);
  std::vector<uint64_t> q_counters(nq, 0), q_region(nq, 0);
  {
    std::lock_guard<std::mutex> g(c->mu);
    TableScope table_scope{c};
    uint64_t built = 0, unused = 0;
    std::vector<const tq_term_seg*> order;
    std::vector<const SortColumn*> cols;
    std::vector<std::pair<unsigned long long, unsigned long long>> uwin;  // per unit of the query: its smallest and largest image
    for (size_t qi = 0; qi < nq; ++qi) {
      const tq_terms_spec& sp = specs[qi];
      const size_t s0 = cp.segs.size(), u0 = cp.units.size();
      q_seg[qi] = s0;
      q_unit[qi] = u0;
      int rc = plan_count(c, queries[qi], (uint32_t)qi, order, cp, &unused, true);
      if (rc != TQ_OK) return rc;
      uint32_t flags = (out_hits ? kTermsHits : 0u) | (sp.missing_mode != TQ_TERMS_MISSING_NONE ? kTermsMissing : 0u) |
                       (sp.target == TQ_TERMS_BY_KEY ? kTermsByKey : 0u) | (sp.order == TQ_ORDER_ASC ? kTermsAsc : 0u);
      rc = plan_terms_query(c, sp, qi, flags, cp, s0, u0, tsegs, windows, cols, uwin, q_counters[qi], q_region[qi]);
      if (rc != TQ_OK) return rc;
    }
    q_seg[nq] = cp.segs.size();
    q_unit[nq] = cp.units.size();
    int rc = flush_builds(c, &built);
    if (rc != TQ_OK) return rc;
    hold_segments(c, b, queries, nq);  // (the segments, their filter views and the columns stay until the rows are in)
    for (size_t qi = 0; qi < nq; ++qi) b->held_columns.push_back(specs[qi].column_id);
    std::sort(b->held_columns.begin(), b->held_columns.end());
    b->held_columns.erase(std::unique(b->held_columns.begin(), b->held_columns.end()), b->held_columns.end());
    for (uint32_t col : b->held_columns) ++c->sort_users[col];
  }
  if (cp.units.empty()) return TQ_OK;
  // waves of consecutive queries whose counters fit the budget (a query above it runs alone); counters and regions relative to it
  struct Wave { size_t q0, q1; uint64_t counters, region; };
  std::vector<Wave> waves;
  uint64_t max_counters = 0, max_region = 0;
  size_t max_segs = 0;
  for (size_t qi = 0; qi < nq; ++qi) {
    if (waves.empty() || (waves.back().counters && waves.back().counters + q_counters[qi] > c->terms_counter_budget))
      waves.push_back(Wave{qi, qi, 0, 0});
    Wave& w = waves.back();
    for (size_t si = q_seg[qi]; si < q_seg[qi + 1]; ++si) { tsegs[si].counters += w.counters; tsegs[si].region += w.region; }
    w.q1 = qi + 1;
    w.counters += q_counters[qi];
    w.region += q_region[qi];
    max_counters = std::max(max_counters, w.counters);
    max_region = std::max(max_region, w.region);
    max_segs = std::max(max_segs, q_seg[w.q1] - q_seg[w.q0]);
  }
  // descriptors: one H2D copy; scratch: hits | tile counters, then one wave's per-(query, segment) results | kept entries |
  // missing counters | counters
  Staging st;
  const size_t o_w = st.add(cp.words), o_s = st.add(cp.segs), o_u = st.add(cp.units), o_z = st.add(tsegs), o_h = st.add(windows);
  TQ_CUDA(st.reserve(b->pin, b->dev));
  st.copy();
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off = align256(off + bytes); return at; };
  const size_t r_hits = take(nq * 8), r_tiles = take(16), head_bytes = off;
  const size_t r_n = take(max_segs * 4), r_other = take(max_segs * 8), r_err = take(max_segs * 8), r_key = take(max_region * 8),
               r_count = take(max_region * 4), wave_bytes = off - head_bytes;
  const size_t r_missing = take(max_segs * 4), r_counters = take(max_counters * 4);
  TQ_CUDA(b->scratch.ensure(off));
  TQ_CUDA(b->res_pin.ensure(std::max(head_bytes, wave_bytes)));
  uint8_t* const d = b->scratch.p;
  TermsParams P{};
  P.c = CountParams{c->d_lists, st.on_device<const uint32_t>(o_w), st.on_device<const CountSeg>(o_s), st.on_device<const Unit>(o_u),
                    reinterpret_cast<unsigned long long*>(d + r_hits)};
  P.tsegs = st.on_device<const TermsSeg>(o_z);
  P.windows = st.on_device<const HistUnit>(o_h);
  P.counts = reinterpret_cast<uint32_t*>(d + r_counters);
  P.missing = reinterpret_cast<uint32_t*>(d + r_missing);
  P.tiles = reinterpret_cast<unsigned long long*>(d + r_tiles);
  P.res_key = reinterpret_cast<unsigned long long*>(d + r_key);
  P.res_count = reinterpret_cast<uint32_t*>(d + r_count);
  P.res_n = reinterpret_cast<uint32_t*>(d + r_n);
  P.res_other = reinterpret_cast<unsigned long long*>(d + r_other);
  P.res_error = reinterpret_cast<unsigned long long*>(d + r_err);
  TQ_CUDA(cudaMemcpyAsync(b->dev.p, b->pin.p, st.bytes, cudaMemcpyHostToDevice, b->stream));
  TQ_CUDA(cudaMemsetAsync(d, 0, head_bytes, b->stream));  // hits, tile counters
  // per (query, segment): its kept entries (ascending key) and scalars, gathered wave by wave
  std::vector<std::vector<std::pair<unsigned long long, uint32_t>>> kept(cp.segs.size());
  std::vector<uint64_t> seg_other(cp.segs.size()), seg_err(cp.segs.size());
  float ms_total = 0;
  const uint8_t* h = b->res_pin.p;
  for (const Wave& w : waves) {
    const size_t sa = q_seg[w.q0], sb = q_seg[w.q1], ua = q_unit[w.q0], ub = q_unit[w.q1];
    if (sa == sb) continue;
    P.unit_base = (uint32_t)ua;
    P.seg_base = (uint32_t)sa;
    TQ_CUDA(cudaMemsetAsync(d + r_missing, 0, (sb - sa) * 4, b->stream));
    TQ_CUDA(cudaMemsetAsync(d + r_counters, 0, w.counters * 4, b->stream));
    TQ_CUDA(cudaEventRecord(b->ev_k0, b->stream));
    if (ub > ua) {
      (cp.mixed ? k_terms<true> : k_terms<false>)<<<(unsigned)(ub - ua), kThreads, 0, b->stream>>>(P);
      TQ_CUDA(cudaGetLastError());
    }
    k_terms_select<<<(unsigned)(sb - sa), kThreads, 0, b->stream>>>(P);
    TQ_CUDA(cudaGetLastError());
    TQ_CUDA(cudaEventRecord(b->ev_k1, b->stream));
    TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d + head_bytes, r_key - head_bytes + w.region * 8, cudaMemcpyDeviceToHost, b->stream));
    TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + (r_count - head_bytes), d + r_count, w.region * 4, cudaMemcpyDeviceToHost, b->stream));
    TQ_CUDA(cudaStreamSynchronize(b->stream));
    float ms = 0;
    cudaEventElapsedTime(&ms, b->ev_k0, b->ev_k1);
    ms_total += ms;
    for (size_t si = sa; si < sb; ++si) {
      const size_t rel = si - sa;
      uint32_t n;
      memcpy(&n, h + (r_n - head_bytes) + rel * 4, 4);
      memcpy(&seg_other[si], h + (r_other - head_bytes) + rel * 8, 8);
      memcpy(&seg_err[si], h + (r_err - head_bytes) + rel * 8, 8);
      kept[si].resize(n);
      for (uint32_t j = 0; j < n; ++j) {
        const size_t e = tsegs[si].region + j;
        unsigned long long key;
        uint32_t count;
        memcpy(&key, h + (r_key - head_bytes) + e * 8, 8);
        memcpy(&count, h + (r_count - head_bytes) + e * 4, 4);
        kept[si][j] = {key, count};
      }
    }
  }
  TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d, head_bytes, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  unsigned long long tiles[2];
  memcpy(tiles, h + r_tiles, 16);
  if (out_hits) memcpy(out_hits, h + r_hits, nq * 8);
  // rows: each query's segments by segment_ord, each in ascending key
  bool fits = true;
  std::vector<size_t> by_ord;
  for (size_t qi = 0; qi < nq; ++qi) {
    by_ord.clear();
    for (size_t si = q_seg[qi]; si < q_seg[qi + 1]; ++si) by_ord.push_back(si);
    std::sort(by_ord.begin(), by_ord.end(), [&](size_t x, size_t y) { return cp.segment_ords[x] < cp.segment_ords[y]; });
    uint32_t n = 0;
    for (size_t si : by_ord) {
      out_sum_other[qi] += seg_other[si];
      out_error_bound[qi] += seg_err[si];
      for (const auto& e : kept[si]) {
        if (n < out_stride) {
          const size_t at = qi * (size_t)out_stride + n;
          out_segment_ord[at] = cp.segment_ords[si];
          out_key[at] = e.first;
          out_doc_count[at] = e.second;
        }
        ++n;
      }
    }
    out_n[qi] = n;
    fits = fits && n <= out_stride;
  }
  {
    std::lock_guard<std::mutex> g(c->mu);
    c->terms_ms += ms_total;
    c->terms_units += cp.units.size() + cp.segs.size();
    c->terms_tiles_seen += tiles[0];
    c->terms_tiles_one_key += tiles[1];
  }
  if (!fits) return fail(TQ_ERR_INVALID_ARGUMENT, "a terms row has more entries than out_stride: out_n holds how many");
  return TQ_OK;
}

// ---- metrics of fast fields ----------------------------------------------------------------------------------
// A metrics spec's column count, kinds and flags (TQ_ERR_INVALID_ARGUMENT).
static int check_metrics_spec(const tq_metrics_spec& sp) {
  if (sp.n_columns < 1 || sp.n_columns > TQ_METRICS_MAX_COLUMNS) return fail(TQ_ERR_INVALID_ARGUMENT, "metrics spec: n_columns must be 1..4");
  for (uint32_t i = 0; i < sp.n_columns; ++i)
    if (sp.columns[i].kind > TQ_FAST_DATE || (sp.columns[i].flags & ~(TQ_METRIC_MISSING | TQ_METRIC_COUNT_ONLY | TQ_METRIC_EMPTY)) ||
        ((sp.columns[i].flags & TQ_METRIC_EMPTY) && ((sp.columns[i].flags & TQ_METRIC_COUNT_ONLY) || sp.columns[i].kind != TQ_FAST_U64)))
      return fail(TQ_ERR_INVALID_ARGUMENT, "metrics spec: column kind or flags");
  return TQ_OK;
}

// One MetricsSeg per (query, segment) plan_count added from s0: the spec's columns in that segment.
static int plan_metrics_segs(tq_ctx* c, const tq_metrics_spec& sp, const CountPlan& cp, size_t s0, bool hits, std::vector<MetricsSeg>& msegs) {
  for (size_t si = s0; si < cp.segs.size(); ++si) {
    MetricsSeg z{};
    z.n_columns = sp.n_columns;
    z.flags = hits ? kMetricsHits : 0u;
    for (uint32_t i = 0; i < sp.n_columns; ++i) {
      const tq_metric_column& mc = sp.columns[i];
      if (mc.flags & TQ_METRIC_EMPTY) {  // (tantivy's empty column: no values, no tiles)
        z.col[i] = MetricsCol{nullptr, nullptr, nullptr, mc.missing_image, mc.kind, mc.flags};
        continue;
      }
      auto it = c->sort_columns.find({mc.column_id, cp.segment_ords[si]});
      if (it == c->sort_columns.end()) return fail(TQ_ERR_NOT_FOUND, "a metrics query names a segment without the column (tq_sort_column_register)");
      const SortColumn& col = it->second;
      if (col.tiles.size() != (cp.segs[si].max_doc + kTileDocs - 1) / kTileDocs) return fail(TQ_ERR_INVALID_ARGUMENT, "column and segment differ in max_doc");
      z.col[i] = MetricsCol{col.d_values, col.d_present, col.d_tiles, mc.missing_image, mc.kind, mc.flags};
    }
    msegs.push_back(z);
  }
  return TQ_OK;
}

// The registered columns a metrics spec reads, for the batch to hold (the caller sorts and dedups b->held_columns).
static void hold_metric_columns(tq_batch* b, const tq_metrics_spec& sp) {
  for (uint32_t i = 0; i < sp.n_columns; ++i)
    if (!(sp.columns[i].flags & TQ_METRIC_EMPTY)) b->held_columns.push_back(sp.columns[i].column_id);
}

int tq_metrics_batch(tq_ctx* c, const tq_query* queries, const tq_metrics_spec* specs, size_t nq, tq_metric_part* out, uint64_t* out_hits) {
  if (!c || (nq && (!queries || !specs || !out))) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  for (size_t qi = 0; qi < nq; ++qi) {
    if (queries[qi].op == TQ_OP_PHRASE) return fail(TQ_ERR_UNSUPPORTED, "metrics of phrase queries are not on the device path");
    int rc = check_metrics_spec(specs[qi]);
    if (rc != TQ_OK) return rc;
  }
  const tq_metric_part empty{0ull, 0ull, 0ull, ~0ull, 0ull, 0.0, 0.0, INT32_MAX, 0u};
  for (size_t qi = 0; qi < nq; ++qi) {
    for (uint32_t i = 0; i < kMetricsMaxColumns; ++i) out[qi * kMetricsMaxColumns + i] = empty;
    if (out_hits) out_hits[qi] = 0;
  }
  if (!nq) return TQ_OK;
  tq_batch* b = acquire_batch(c);
  if (!b) return fail(TQ_ERR_CUDA, "stream/event creation failed");
  struct Guard { tq_batch* b; ~Guard() { tq_batch_destroy(b); } } guard{b};
  CountPlan cp;
  std::vector<MetricsSeg> msegs;  // parallel to cp.segs
  {
    std::lock_guard<std::mutex> g(c->mu);
    TableScope table_scope{c};
    uint64_t built = 0, unused = 0;
    std::vector<const tq_term_seg*> order;
    for (size_t qi = 0; qi < nq; ++qi) {
      const tq_metrics_spec& sp = specs[qi];
      const size_t s0 = cp.segs.size();
      int rc = plan_count(c, queries[qi], (uint32_t)qi, order, cp, &unused, true);
      if (rc != TQ_OK) return rc;
      rc = plan_metrics_segs(c, sp, cp, s0, out_hits != nullptr, msegs);
      if (rc != TQ_OK) return rc;
    }
    int rc = flush_builds(c, &built);
    if (rc != TQ_OK) return rc;
    hold_segments(c, b, queries, nq);  // (the segments, their filter views and the columns stay until the parts are in)
    for (size_t qi = 0; qi < nq; ++qi) hold_metric_columns(b, specs[qi]);
    std::sort(b->held_columns.begin(), b->held_columns.end());
    b->held_columns.erase(std::unique(b->held_columns.begin(), b->held_columns.end()), b->held_columns.end());
    for (uint32_t col : b->held_columns) ++c->sort_users[col];
  }
  if (cp.units.empty()) return TQ_OK;
  // descriptors and the empty accumulators: one H2D copy; scratch: hits | tile counters
  std::vector<tq_metric_part> parts(nq * kMetricsMaxColumns, empty);
  Staging st;
  const size_t o_w = st.add(cp.words), o_s = st.add(cp.segs), o_u = st.add(cp.units), o_z = st.add(msegs), o_p = st.add(parts);
  TQ_CUDA(st.reserve(b->pin, b->dev));
  st.copy();
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off = align256(off + bytes); return at; };
  const size_t r_hits = take(nq * 8), r_tiles = take(16), head_bytes = off;
  TQ_CUDA(b->scratch.ensure(off));
  TQ_CUDA(b->res_pin.ensure(head_bytes + parts.size() * sizeof(tq_metric_part)));
  uint8_t* const d = b->scratch.p;
  MetricsParams P{};
  P.c = CountParams{c->d_lists, st.on_device<const uint32_t>(o_w), st.on_device<const CountSeg>(o_s), st.on_device<const Unit>(o_u),
                    reinterpret_cast<unsigned long long*>(d + r_hits)};
  P.msegs = st.on_device<const MetricsSeg>(o_z);
  P.parts = st.on_device<tq_metric_part>(o_p);
  P.tiles = reinterpret_cast<unsigned long long*>(d + r_tiles);
  TQ_CUDA(cudaMemcpyAsync(b->dev.p, b->pin.p, st.bytes, cudaMemcpyHostToDevice, b->stream));
  TQ_CUDA(cudaMemsetAsync(d, 0, head_bytes, b->stream));  // hits, tile counters
  TQ_CUDA(cudaEventRecord(b->ev_k0, b->stream));
  (cp.mixed ? k_metrics<true> : k_metrics<false>)<<<(unsigned)cp.units.size(), kThreads, 0, b->stream>>>(P);
  TQ_CUDA(cudaGetLastError());
  TQ_CUDA(cudaEventRecord(b->ev_k1, b->stream));
  TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d, head_bytes, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + head_bytes, st.on_device<const uint8_t>(o_p), parts.size() * sizeof(tq_metric_part),
                          cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  const uint8_t* h = b->res_pin.p;
  memcpy(out, h + head_bytes, parts.size() * sizeof(tq_metric_part));
  if (out_hits) memcpy(out_hits, h + r_hits, nq * 8);
  float ms = 0;
  cudaEventElapsedTime(&ms, b->ev_k0, b->ev_k1);
  unsigned long long tiles[2];
  memcpy(tiles, h + r_tiles, 16);
  {
    std::lock_guard<std::mutex> g(c->mu);
    c->metrics_ms += ms;
    c->metrics_units += cp.units.size();
    c->metrics_tiles_seen += tiles[0];
    c->metrics_tiles_one_value += tiles[1];
  }
  return TQ_OK;
}

// ---- metrics per histogram bucket ----------------------------------------------------------------------------
// Waves of consecutive queries whose accumulators (kMetricsMaxColumns per counter) fit the budget (a query above it runs alone),
// query qi holding n_bins[qi] counters: at[qi] is its first counter and row_at[qi] its first row entry in its wave, its row holding
// min(row_cap, n_bins[qi]) entries.
struct Wave { size_t q0, q1; uint64_t counters, rows; };
static std::vector<Wave> plan_waves(const std::vector<uint32_t>& n_bins, uint64_t budget, uint32_t row_cap, std::vector<unsigned long long>& at,
                                    std::vector<unsigned long long>& row_at) {
  std::vector<Wave> waves;
  at.assign(n_bins.size(), 0);
  row_at.assign(n_bins.size(), 0);
  for (size_t qi = 0; qi < n_bins.size(); ++qi) {
    if (waves.empty() || (waves.back().counters && (waves.back().counters + n_bins[qi]) * kMetricsMaxColumns > budget))
      waves.push_back(Wave{qi, qi, 0, 0});
    Wave& w = waves.back();
    at[qi] = w.counters;
    row_at[qi] = w.rows;
    w.q1 = qi + 1;
    w.counters += n_bins[qi];
    w.rows += std::min<uint64_t>(row_cap, n_bins[qi]);
  }
  return waves;
}

int tq_histogram_metrics_batch(tq_ctx* c, const tq_query* queries, const tq_histogram_spec* hspecs, const tq_metrics_spec* mspecs, size_t nq,
                               uint32_t out_stride, int64_t* out_pos, uint64_t* out_doc_count, tq_metric_part* out_parts, uint32_t* out_n,
                               uint64_t* out_hits) {
  if (!c || (nq && (!queries || !hspecs || !mspecs || !out_n || (out_stride && (!out_pos || !out_doc_count || !out_parts)))))
    return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  constexpr uint32_t kC = kMetricsMaxColumns;
  for (size_t qi = 0; qi < nq; ++qi) {
    if (queries[qi].op == TQ_OP_PHRASE) return fail(TQ_ERR_UNSUPPORTED, "histograms of phrase queries are not on the device path");
    if (hspecs[qi].kind > TQ_FAST_DATE) return fail(TQ_ERR_INVALID_ARGUMENT, "histogram kind");
    if (!(hspecs[qi].interval > 0.0) || !std::isfinite(hspecs[qi].interval)) return fail(TQ_ERR_INVALID_ARGUMENT, "histogram interval must be finite and > 0");
    int rc = check_metrics_spec(mspecs[qi]);
    if (rc != TQ_OK) return rc;
  }
  for (size_t qi = 0; qi < nq; ++qi) { out_n[qi] = 0; if (out_hits) out_hits[qi] = 0; }
  if (!nq) return TQ_OK;
  tq_batch* b = acquire_batch(c);
  if (!b) return fail(TQ_ERR_CUDA, "stream/event creation failed");
  struct Guard { tq_batch* b; ~Guard() { tq_batch_destroy(b); } } guard{b};
  CountPlan cp;
  std::vector<HistSeg> hsegs;     // parallel to cp.segs
  std::vector<MetricsSeg> msegs;  // parallel to cp.segs
  std::vector<HistQuery> hq(nq);
  std::vector<HistUnit> hunits;   // parallel to cp.units
  std::vector<size_t> q_unit(nq + 1);
  {
    std::lock_guard<std::mutex> g(c->mu);
    TableScope table_scope{c};
    uint64_t built = 0, unused = 0;
    std::vector<const tq_term_seg*> order;
    std::vector<const SortColumn*> cols;
    std::vector<std::pair<long long, long long>> uwin;  // per unit of the query: its first and last pos (first > last: none)
    for (size_t qi = 0; qi < nq; ++qi) {
      const tq_histogram_spec& sp = hspecs[qi];
      const size_t s0 = cp.segs.size(), u0 = cp.units.size();
      q_unit[qi] = u0;
      int rc = plan_count(c, queries[qi], (uint32_t)qi, order, cp, &unused, true);
      if (rc != TQ_OK) return rc;
      long long base = 0;
      uint64_t len = 0;
      rc = plan_hist_query(c, sp, qi, cp, s0, u0, kHistMetricsMaxBins, hsegs, cols, uwin, base, len);
      if (rc != TQ_OK) return rc;
      rc = plan_metrics_segs(c, mspecs[qi], cp, s0, out_hits != nullptr, msegs);
      if (rc != TQ_OK) return rc;
      for (const auto& w : uwin)
        hunits.push_back(w.first <= w.second ? HistUnit{(uint32_t)(w.first - base), (uint32_t)(w.second - w.first + 1)} : HistUnit{0u, 0u});
      hq[qi] = HistQuery{sp.interval, sp.offset, base, 0ull, (uint32_t)len, sp.kind, out_hits ? kHistHits : 0u, 0u};
    }
    q_unit[nq] = cp.units.size();
    int rc = flush_builds(c, &built);
    if (rc != TQ_OK) return rc;
    hold_segments(c, b, queries, nq);  // (the segments, their filter views and the columns stay until the rows are in)
    for (size_t qi = 0; qi < nq; ++qi) {
      b->held_columns.push_back(hspecs[qi].column_id);
      hold_metric_columns(b, mspecs[qi]);
    }
    std::sort(b->held_columns.begin(), b->held_columns.end());
    b->held_columns.erase(std::unique(b->held_columns.begin(), b->held_columns.end()), b->held_columns.end());
    for (uint32_t col : b->held_columns) ++c->sort_users[col];
  }
  if (cp.units.empty()) return TQ_OK;
  // A query's row holds min(out_stride, n_bins) entries (it has at most n_bins non-empty buckets), so a wave's rows, on the device
  // and in pinned memory, are bounded by its counters and the budget as well.
  std::vector<uint32_t> bins(nq);
  for (size_t qi = 0; qi < nq; ++qi) bins[qi] = hq[qi].n_bins;
  std::vector<unsigned long long> at, row_at;
  const std::vector<Wave> waves = plan_waves(bins, c->hist_metrics_budget, out_stride, at, row_at);
  for (size_t qi = 0; qi < nq; ++qi) hq[qi].counters = at[qi];
  uint64_t max_counters = 0, max_rows = 0;
  size_t max_queries = 0;
  for (const Wave& w : waves) {
    max_counters = std::max(max_counters, w.counters);
    max_rows = std::max(max_rows, w.rows);
    max_queries = std::max(max_queries, w.q1 - w.q0);
  }
  // descriptors: one H2D copy; scratch: hits | tile counters, then one wave's row lengths | rows (pos | doc counts | parts) |
  // doc counters | accumulators
  Staging st;
  const size_t o_w = st.add(cp.words), o_s = st.add(cp.segs), o_u = st.add(cp.units), o_z = st.add(hsegs), o_m = st.add(msegs),
               o_q = st.add(hq), o_h = st.add(hunits), o_r = st.add(row_at);
  TQ_CUDA(st.reserve(b->pin, b->dev));
  st.copy();
  const size_t part_row = (size_t)kC * sizeof(tq_metric_part);
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off = align256(off + bytes); return at; };
  const size_t r_hits = take(nq * 8), r_tiles = take(32), head_bytes = off;
  const size_t r_n = take(max_queries * 4), r_pos = take(max_rows * 8), r_count = take(max_rows * 8), r_parts = take(max_rows * part_row),
               wave_bytes = off - head_bytes;
  const size_t r_counters = take(max_counters * 8), r_acc = take(max_counters * part_row);
  TQ_CUDA(b->scratch.ensure(off));
  TQ_CUDA(b->res_pin.ensure(std::max(head_bytes, wave_bytes)));
  uint8_t* const d = b->scratch.p;
  HistMetricsParams P{};
  P.c = CountParams{c->d_lists, st.on_device<const uint32_t>(o_w), st.on_device<const CountSeg>(o_s), st.on_device<const Unit>(o_u),
                    reinterpret_cast<unsigned long long*>(d + r_hits)};
  P.hsegs = st.on_device<const HistSeg>(o_z);
  P.msegs = st.on_device<const MetricsSeg>(o_m);
  P.queries = st.on_device<const HistQuery>(o_q);
  P.hunits = st.on_device<const HistUnit>(o_h);
  P.rows = st.on_device<const unsigned long long>(o_r);
  P.counts = reinterpret_cast<unsigned long long*>(d + r_counters);
  P.parts = reinterpret_cast<tq_metric_part*>(d + r_acc);
  P.tiles = reinterpret_cast<unsigned long long*>(d + r_tiles);
  P.res_pos = reinterpret_cast<long long*>(d + r_pos);
  P.res_count = reinterpret_cast<unsigned long long*>(d + r_count);
  P.res_parts = reinterpret_cast<tq_metric_part*>(d + r_parts);
  P.res_n = reinterpret_cast<uint32_t*>(d + r_n);
  P.res_stride = out_stride;
  TQ_CUDA(cudaMemcpyAsync(b->dev.p, b->pin.p, st.bytes, cudaMemcpyHostToDevice, b->stream));
  TQ_CUDA(cudaMemsetAsync(d, 0, head_bytes, b->stream));  // hits, tile counters
  const uint8_t* h = b->res_pin.p;
  const size_t p_pos = r_pos - head_bytes, p_count = r_count - head_bytes, p_parts = r_parts - head_bytes;
  float ms_total = 0;
  bool fits = true;
  for (const Wave& w : waves) {
    const size_t ua = q_unit[w.q0], ub = q_unit[w.q1], wq = w.q1 - w.q0;
    P.unit_base = (uint32_t)ua;
    P.query_base = (uint32_t)w.q0;
    TQ_CUDA(cudaMemsetAsync(d + r_counters, 0, w.counters * 8, b->stream));
    TQ_CUDA(cudaMemsetAsync(d + r_acc, 0, w.counters * part_row, b->stream));
    TQ_CUDA(cudaEventRecord(b->ev_k0, b->stream));
    if (ub > ua) {
      (cp.mixed ? k_hist_metrics<true> : k_hist_metrics<false>)<<<(unsigned)(ub - ua), kThreads, 0, b->stream>>>(P);
      TQ_CUDA(cudaGetLastError());
    }
    k_hist_metrics_final<<<(unsigned)wq, kThreads, 0, b->stream>>>(P);
    TQ_CUDA(cudaGetLastError());
    TQ_CUDA(cudaEventRecord(b->ev_k1, b->stream));
    TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d + r_n, wq * 4, cudaMemcpyDeviceToHost, b->stream));
    TQ_CUDA(cudaStreamSynchronize(b->stream));
    float ms = 0;
    cudaEventElapsedTime(&ms, b->ev_k0, b->ev_k1);
    ms_total += ms;
    memcpy(out_n + w.q0, h, wq * 4);
    for (size_t qi = w.q0; qi < w.q1; ++qi) fits = fits && out_n[qi] <= out_stride;
    if (!fits) continue;  // (a row too long: only the lengths of the remaining waves)
    // the rows: the wave's whole region when they fill half of it or more, else each query's row only as long as it is
    uint64_t filled = 0;
    for (size_t qi = w.q0; qi < w.q1; ++qi) filled += out_n[qi];
    auto fetch = [&](size_t at, size_t n) {
      TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + p_pos + at * 8, d + r_pos + at * 8, n * 8, cudaMemcpyDeviceToHost, b->stream));
      TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + p_count + at * 8, d + r_count + at * 8, n * 8, cudaMemcpyDeviceToHost, b->stream));
      TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + p_parts + at * part_row, d + r_parts + at * part_row, n * part_row, cudaMemcpyDeviceToHost,
                              b->stream));
      return TQ_OK;
    };
    if (2 * filled >= w.rows) {
      int rc = fetch(0, w.rows);
      if (rc != TQ_OK) return rc;
    } else {
      for (size_t qi = w.q0; qi < w.q1; ++qi) {
        int rc = out_n[qi] ? fetch(row_at[qi], out_n[qi]) : TQ_OK;
        if (rc != TQ_OK) return rc;
      }
    }
    TQ_CUDA(cudaStreamSynchronize(b->stream));
    for (size_t qi = w.q0; qi < w.q1; ++qi) {
      const size_t at = row_at[qi], dst = qi * (size_t)out_stride, n = out_n[qi];
      memcpy(out_pos + dst, h + p_pos + at * 8, n * 8);
      memcpy(out_doc_count + dst, h + p_count + at * 8, n * 8);
      memcpy(out_parts + dst * kC, h + p_parts + at * part_row, n * part_row);
    }
  }
  TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d, head_bytes, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  if (out_hits) memcpy(out_hits, h + r_hits, nq * 8);
  unsigned long long tiles[4];
  memcpy(tiles, h + r_tiles, 32);
  {
    std::lock_guard<std::mutex> g(c->mu);
    c->hist_metrics_ms += ms_total;
    c->hist_metrics_units += cp.units.size() + nq;
    c->hist_metrics_tiles_seen += tiles[0];
    c->hist_metrics_tiles_one_bucket += tiles[1];
    c->hist_metrics_flush_shared += tiles[2];
    c->hist_metrics_flush_global += tiles[3];
  }
  if (!fits) return fail(TQ_ERR_INVALID_ARGUMENT, "a histogram has more non-empty buckets than out_stride: out_n holds how many");
  return TQ_OK;
}

// ---- metrics per term ----------------------------------------------------------------------------------------
// A tq_metric_part as the accumulators hold it (min_image and quantum_exp complemented) back to the ABI's form.
static tq_metric_part uncomplement(tq_metric_part p) {
  p.min_image = ~p.min_image;
  p.quantum_exp = (int)(0x7FFFFFFFu - (unsigned)p.quantum_exp);
  return p;
}

// Waves of consecutive terms queries whose counters fit counter_budget and whose per-query load q_extra (the metric parts or the
// histogram cells of their kept entries) fits extra_budget; a query above either runs alone (a wave holding neither yet takes any).  Shifts each TermsSeg's counters and
// region to be relative to its wave; a wave's `extra` is where each query's load starts, in at[qi].
struct TermsWave { size_t q0, q1; uint64_t counters, region, extra; };
static std::vector<TermsWave> plan_terms_waves(const std::vector<uint64_t>& q_counters, const std::vector<uint64_t>& q_region,
                                               const std::vector<uint64_t>& q_extra, uint64_t counter_budget, uint64_t extra_budget,
                                               const std::vector<size_t>& q_seg, std::vector<TermsSeg>& tsegs, std::vector<uint64_t>* at = nullptr) {
  std::vector<TermsWave> waves;
  if (at) at->assign(q_counters.size(), 0);
  for (size_t qi = 0; qi < q_counters.size(); ++qi) {
    if (waves.empty() || ((waves.back().counters || waves.back().extra) && (waves.back().counters + q_counters[qi] > counter_budget ||
                                                                            waves.back().extra + q_extra[qi] > extra_budget)))
      waves.push_back(TermsWave{qi, qi, 0, 0, 0});
    TermsWave& w = waves.back();
    for (size_t si = q_seg[qi]; si < q_seg[qi + 1]; ++si) { tsegs[si].counters += w.counters; tsegs[si].region += w.region; }
    if (at) (*at)[qi] = w.extra;
    w.q1 = qi + 1;
    w.counters += q_counters[qi];
    w.region += q_region[qi];
    w.extra += q_extra[qi];
  }
  return waves;
}

int tq_terms_metrics_batch(tq_ctx* c, const tq_query* queries, const tq_terms_spec* tspecs, const tq_metrics_spec* mspecs,
                           const tq_terms_metric_order* orders, size_t nq, uint32_t out_stride, uint32_t* out_segment_ord,
                           uint64_t* out_key, uint64_t* out_doc_count, tq_metric_part* out_parts, uint32_t* out_n,
                           uint64_t* out_sum_other, uint64_t* out_error_bound, tq_metric_part* out_order_part, uint64_t* out_hits) {
  if (!c || (nq && (!queries || !tspecs || !mspecs || !out_n || !out_sum_other || !out_error_bound || !out_order_part ||
                    (out_stride && (!out_segment_ord || !out_key || !out_doc_count || !out_parts)))))
    return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  constexpr uint32_t kC = kMetricsMaxColumns;
  for (size_t qi = 0; qi < nq; ++qi) {
    const tq_terms_spec& sp = tspecs[qi];
    if (queries[qi].op == TQ_OP_PHRASE) return fail(TQ_ERR_UNSUPPORTED, "terms of phrase queries are not on the device path");
    if (sp.target > TQ_TERMS_BY_METRIC || sp.order > TQ_ORDER_ASC || sp.missing_mode > TQ_TERMS_MISSING_AFTER_MAX || !sp.segment_size)
      return fail(TQ_ERR_INVALID_ARGUMENT, "terms spec: target, order, missing mode or segment_size");
    int rc = check_metrics_spec(mspecs[qi]);
    if (rc != TQ_OK) return rc;
    if (sp.target == TQ_TERMS_BY_METRIC &&
        (!orders || orders[qi].column >= mspecs[qi].n_columns || orders[qi].metric > TQ_TERMS_ORDER_MAX))
      return fail(TQ_ERR_INVALID_ARGUMENT, "query " + std::to_string(qi) + ": a metric order needs orders[q] with a column of its spec and a TQ_TERMS_ORDER_* metric");
  }
  const tq_metric_part empty{0ull, 0ull, 0ull, ~0ull, 0ull, 0.0, 0.0, INT32_MAX, 0u};
  for (size_t qi = 0; qi < nq; ++qi) {
    out_n[qi] = 0;
    out_sum_other[qi] = out_error_bound[qi] = 0;
    out_order_part[qi] = empty;
    if (out_hits) out_hits[qi] = 0;
  }
  if (!nq) return TQ_OK;
  tq_batch* b = acquire_batch(c);
  if (!b) return fail(TQ_ERR_CUDA, "stream/event creation failed");
  struct Guard { tq_batch* b; ~Guard() { tq_batch_destroy(b); } } guard{b};
  CountPlan cp;
  std::vector<TermsSeg> tsegs;    // parallel to cp.segs
  std::vector<MetricsSeg> msegs;  // parallel to cp.segs
  std::vector<HistUnit> windows;  // parallel to cp.units
  std::vector<TermsOrder> ord(nq, TermsOrder{0u, 0u});
  std::vector<size_t> q_seg(nq + 1), q_unit(nq + 1);
  std::vector<uint64_t> q_counters(nq, 0), q_region(nq, 0);
  {
    std::lock_guard<std::mutex> g(c->mu);
    TableScope table_scope{c};
    uint64_t built = 0, unused = 0;
    std::vector<const tq_term_seg*> order;
    std::vector<const SortColumn*> cols;
    std::vector<std::pair<unsigned long long, unsigned long long>> uwin;
    for (size_t qi = 0; qi < nq; ++qi) {
      const tq_terms_spec& sp = tspecs[qi];
      const size_t s0 = cp.segs.size(), u0 = cp.units.size();
      q_seg[qi] = s0;
      q_unit[qi] = u0;
      int rc = plan_count(c, queries[qi], (uint32_t)qi, order, cp, &unused, true);
      if (rc != TQ_OK) return rc;
      const uint32_t flags = (out_hits ? kTermsHits : 0u) | (sp.missing_mode != TQ_TERMS_MISSING_NONE ? kTermsMissing : 0u) |
                             (sp.target == TQ_TERMS_BY_KEY ? kTermsByKey : 0u) | (sp.target == TQ_TERMS_BY_METRIC ? kTermsByMetric : 0u) |
                             (sp.order == TQ_ORDER_ASC ? kTermsAsc : 0u);
      rc = plan_terms_query(c, sp, qi, flags, cp, s0, u0, tsegs, windows, cols, uwin, q_counters[qi], q_region[qi]);
      if (rc != TQ_OK) return rc;
      rc = plan_metrics_segs(c, mspecs[qi], cp, s0, false, msegs);
      if (rc != TQ_OK) return rc;
      for (size_t si = s0; si < cp.segs.size(); ++si) {
        const TermsSeg& z = tsegs[si];
        if ((uint64_t)std::min<uint64_t>(z.segment_size, (uint64_t)z.n_keys + ((z.flags & kTermsMissing) ? 1u : 0u)) * kC > c->terms_metrics_budget)
          return fail(TQ_ERR_UNSUPPORTED, "query " + std::to_string(qi) + ": the metric parts of its entries in a segment exceed the device budget (take the CPU path)");
      }
      if (sp.target == TQ_TERMS_BY_METRIC) ord[qi] = TermsOrder{orders[qi].column, orders[qi].metric};
    }
    q_seg[nq] = cp.segs.size();
    q_unit[nq] = cp.units.size();
    int rc = flush_builds(c, &built);
    if (rc != TQ_OK) return rc;
    hold_segments(c, b, queries, nq);  // (the segments, their filter views and the columns stay until the rows are in)
    for (size_t qi = 0; qi < nq; ++qi) {
      b->held_columns.push_back(tspecs[qi].column_id);
      hold_metric_columns(b, mspecs[qi]);
    }
    std::sort(b->held_columns.begin(), b->held_columns.end());
    b->held_columns.erase(std::unique(b->held_columns.begin(), b->held_columns.end()), b->held_columns.end());
    for (uint32_t col : b->held_columns) ++c->sort_users[col];
  }
  if (cp.units.empty()) return TQ_OK;
  // waves of consecutive queries whose counters fit the counter budget and whose kept entries' parts fit the metrics budget (a query
  // above either runs alone); counters and regions relative to the wave
  std::vector<uint64_t> q_parts(nq);
  for (size_t qi = 0; qi < nq; ++qi) q_parts[qi] = q_region[qi] * kC;
  std::vector<TermsWave> waves = plan_terms_waves(q_counters, q_region, q_parts, c->terms_counter_budget, c->terms_metrics_budget, q_seg, tsegs);
  uint64_t max_counters = 0, max_region = 0;
  size_t max_segs = 0;
  std::vector<bool> wave_by_metric(waves.size(), false);
  for (size_t wi = 0; wi < waves.size(); ++wi) {
    const TermsWave& w = waves[wi];
    for (size_t qi = w.q0; qi < w.q1; ++qi) wave_by_metric[wi] = wave_by_metric[wi] || tspecs[qi].target == TQ_TERMS_BY_METRIC;
    max_counters = std::max(max_counters, w.counters);
    max_region = std::max(max_region, w.region);
    max_segs = std::max(max_segs, q_seg[w.q1] - q_seg[w.q0]);
  }
  // descriptors: one H2D copy; scratch: hits | tile counters | order parts, then one wave's per-(query, segment) results | kept
  // entries | their parts, then the wave's accumulators: missing counters and slots | the missing keys' order accumulators |
  // counters | order accumulators
  Staging st;
  const size_t o_w = st.add(cp.words), o_s = st.add(cp.segs), o_u = st.add(cp.units), o_z = st.add(tsegs), o_h = st.add(windows),
               o_m = st.add(msegs), o_o = st.add(ord);
  TQ_CUDA(st.reserve(b->pin, b->dev));
  st.copy();
  const size_t part_row = (size_t)kC * sizeof(tq_metric_part);
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off = align256(off + bytes); return at; };
  const size_t r_hits = take(nq * 8), r_tiles = take(16), r_mtiles = take(16), r_opart = take(nq * sizeof(tq_metric_part)), head_bytes = off;
  const size_t r_n = take(max_segs * 4), r_other = take(max_segs * 8), r_err = take(max_segs * 8), r_key = take(max_region * 8),
               r_count = take(max_region * 4), r_parts = take(max_region * part_row), wave_bytes = off - head_bytes;
  const size_t r_missing = take(max_segs * 4), r_mslot = take(max_segs * 4), r_omc = take(max_segs * 4), r_omq = take(max_segs * 8),
               r_counters = take(max_counters * 4), r_ocount = take(max_counters * 4), r_oq = take(max_counters * 8);
  TQ_CUDA(b->scratch.ensure(off));
  TQ_CUDA(b->res_pin.ensure(std::max(head_bytes, wave_bytes)));
  uint8_t* const d = b->scratch.p;
  TermsMetricsParams P{};
  P.t.c = CountParams{c->d_lists, st.on_device<const uint32_t>(o_w), st.on_device<const CountSeg>(o_s), st.on_device<const Unit>(o_u),
                      reinterpret_cast<unsigned long long*>(d + r_hits)};
  P.t.tsegs = st.on_device<const TermsSeg>(o_z);
  P.t.windows = st.on_device<const HistUnit>(o_h);
  P.t.counts = reinterpret_cast<uint32_t*>(d + r_counters);
  P.t.missing = reinterpret_cast<uint32_t*>(d + r_missing);
  P.t.tiles = reinterpret_cast<unsigned long long*>(d + r_tiles);
  P.t.res_key = reinterpret_cast<unsigned long long*>(d + r_key);
  P.t.res_count = reinterpret_cast<uint32_t*>(d + r_count);
  P.t.res_n = reinterpret_cast<uint32_t*>(d + r_n);
  P.t.res_other = reinterpret_cast<unsigned long long*>(d + r_other);
  P.t.res_error = reinterpret_cast<unsigned long long*>(d + r_err);
  P.msegs = st.on_device<const MetricsSeg>(o_m);
  P.orders = st.on_device<const TermsOrder>(o_o);
  P.ocount = reinterpret_cast<uint32_t*>(d + r_ocount);
  P.oq = reinterpret_cast<unsigned long long*>(d + r_oq);
  P.ocount_missing = reinterpret_cast<uint32_t*>(d + r_omc);
  P.oq_missing = reinterpret_cast<unsigned long long*>(d + r_omq);
  P.order_parts = reinterpret_cast<tq_metric_part*>(d + r_opart);
  P.mslot = reinterpret_cast<uint32_t*>(d + r_mslot);
  P.parts = reinterpret_cast<tq_metric_part*>(d + r_parts);
  P.tiles = reinterpret_cast<unsigned long long*>(d + r_mtiles);
  TQ_CUDA(cudaMemcpyAsync(b->dev.p, b->pin.p, st.bytes, cudaMemcpyHostToDevice, b->stream));
  TQ_CUDA(cudaMemsetAsync(d, 0, head_bytes, b->stream));  // hits, tile counters, order parts (zero: the empty complemented part)
  // per (query, segment): its kept entries (ascending key) with their parts, and its scalars, gathered wave by wave
  struct Entry { unsigned long long key; uint32_t count; tq_metric_part parts[kC]; };
  std::vector<std::vector<Entry>> kept(cp.segs.size());
  std::vector<uint64_t> seg_other(cp.segs.size()), seg_err(cp.segs.size());
  float ms_total = 0;
  uint64_t ctas = 0;
  const uint8_t* h = b->res_pin.p;
  for (size_t wi = 0; wi < waves.size(); ++wi) {
    const TermsWave& w = waves[wi];
    const bool by_metric = wave_by_metric[wi];
    const size_t sa = q_seg[w.q0], sb = q_seg[w.q1], ua = q_unit[w.q0], ub = q_unit[w.q1];
    if (sa == sb) continue;
    P.t.unit_base = (uint32_t)ua;
    P.t.seg_base = (uint32_t)sa;
    TQ_CUDA(cudaMemsetAsync(d + r_missing, 0, r_counters + w.counters * 4 - r_missing, b->stream));  // missing .. counters
    TQ_CUDA(cudaMemsetAsync(d + r_parts, 0, w.region * part_row, b->stream));
    if (by_metric) TQ_CUDA(cudaMemsetAsync(d + r_ocount, 0, r_oq + w.counters * 8 - r_ocount, b->stream));
    TQ_CUDA(cudaEventRecord(b->ev_k0, b->stream));
    const unsigned nu = (unsigned)(ub - ua), ns = (unsigned)(sb - sa);
    if (nu) {
      (cp.mixed ? k_terms<true> : k_terms<false>)<<<nu, kThreads, 0, b->stream>>>(P.t);
      TQ_CUDA(cudaGetLastError());
      if (by_metric) {
        (cp.mixed ? k_terms_order<true> : k_terms_order<false>)<<<nu, kThreads, 0, b->stream>>>(P);
        TQ_CUDA(cudaGetLastError());
      }
    }
    k_terms_select<<<ns, kThreads, 0, b->stream>>>(P.t);
    TQ_CUDA(cudaGetLastError());
    if (by_metric) {
      k_terms_select_metric<<<ns, kThreads, 0, b->stream>>>(P);
      TQ_CUDA(cudaGetLastError());
    }
    k_terms_mark<<<ns, kThreads, 0, b->stream>>>(P);
    TQ_CUDA(cudaGetLastError());
    if (nu) {
      (cp.mixed ? k_terms_metrics<true> : k_terms_metrics<false>)<<<nu, kThreads, 0, b->stream>>>(P);
      TQ_CUDA(cudaGetLastError());
    }
    TQ_CUDA(cudaEventRecord(b->ev_k1, b->stream));
    ctas += (by_metric ? 3u : 2u) * (uint64_t)nu + (by_metric ? 3u : 2u) * (uint64_t)ns;
    TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d + head_bytes, r_key - head_bytes + w.region * 8, cudaMemcpyDeviceToHost, b->stream));
    TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + (r_count - head_bytes), d + r_count, w.region * 4, cudaMemcpyDeviceToHost, b->stream));
    TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + (r_parts - head_bytes), d + r_parts, w.region * part_row, cudaMemcpyDeviceToHost, b->stream));
    TQ_CUDA(cudaStreamSynchronize(b->stream));
    float ms = 0;
    cudaEventElapsedTime(&ms, b->ev_k0, b->ev_k1);
    ms_total += ms;
    for (size_t si = sa; si < sb; ++si) {
      const size_t rel = si - sa;
      uint32_t n;
      memcpy(&n, h + (r_n - head_bytes) + rel * 4, 4);
      memcpy(&seg_other[si], h + (r_other - head_bytes) + rel * 8, 8);
      memcpy(&seg_err[si], h + (r_err - head_bytes) + rel * 8, 8);
      kept[si].resize(n);
      for (uint32_t j = 0; j < n; ++j) {
        const size_t e = tsegs[si].region + j;
        Entry& x = kept[si][j];
        memcpy(&x.key, h + (r_key - head_bytes) + e * 8, 8);
        memcpy(&x.count, h + (r_count - head_bytes) + e * 4, 4);
        for (uint32_t k = 0; k < kC; ++k) {
          tq_metric_part p;
          memcpy(&p, h + (r_parts - head_bytes) + e * part_row + k * sizeof(tq_metric_part), sizeof(p));
          x.parts[k] = uncomplement(p);
        }
      }
    }
  }
  TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d, head_bytes, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  unsigned long long tiles[2];
  memcpy(tiles, h + r_mtiles, 16);
  if (out_hits) memcpy(out_hits, h + r_hits, nq * 8);
  for (size_t qi = 0; qi < nq; ++qi)
    if (tspecs[qi].target == TQ_TERMS_BY_METRIC) {
      tq_metric_part p;
      memcpy(&p, h + r_opart + qi * sizeof(tq_metric_part), sizeof(p));
      out_order_part[qi] = uncomplement(p);
    }
  // rows: each query's segments by segment_ord, each in ascending key
  bool fits = true;
  std::vector<size_t> by_ord;
  for (size_t qi = 0; qi < nq; ++qi) {
    by_ord.clear();
    for (size_t si = q_seg[qi]; si < q_seg[qi + 1]; ++si) by_ord.push_back(si);
    std::sort(by_ord.begin(), by_ord.end(), [&](size_t x, size_t y) { return cp.segment_ords[x] < cp.segment_ords[y]; });
    uint32_t n = 0;
    for (size_t si : by_ord) {
      out_sum_other[qi] += seg_other[si];
      out_error_bound[qi] += seg_err[si];
      for (const Entry& e : kept[si]) {
        if (n < out_stride) {
          const size_t at = qi * (size_t)out_stride + n;
          out_segment_ord[at] = cp.segment_ords[si];
          out_key[at] = e.key;
          out_doc_count[at] = e.count;
          for (uint32_t k = 0; k < kC; ++k) out_parts[at * kC + k] = k < mspecs[qi].n_columns ? e.parts[k] : empty;
        }
        ++n;
      }
    }
    out_n[qi] = n;
    fits = fits && n <= out_stride;
  }
  {
    std::lock_guard<std::mutex> g(c->mu);
    c->terms_metrics_ms += ms_total;
    c->terms_metrics_units += ctas;
    c->terms_metrics_tiles_seen += tiles[0];
    c->terms_metrics_tiles_one_key += tiles[1];
    c->terms_metrics_waves += waves.size();
  }
  if (!fits) return fail(TQ_ERR_INVALID_ARGUMENT, "a terms row has more entries than out_stride: out_n holds how many");
  return TQ_OK;
}

// ---- histogram per term --------------------------------------------------------------------------------------
int tq_terms_histogram_batch(tq_ctx* c, const tq_query* queries, const tq_terms_spec* tspecs, const tq_histogram_spec* hspecs, size_t nq,
                             uint32_t out_stride, uint32_t* out_segment_ord, uint64_t* out_key, uint64_t* out_doc_count, uint32_t* out_n,
                             uint64_t* out_sum_other, uint64_t* out_error_bound, uint64_t cell_capacity, uint64_t* out_cell_first,
                             uint32_t* out_cell_n, int64_t* out_cell_pos, uint64_t* out_cell_count, uint32_t* out_cells, uint64_t* out_hits) {
  if (!c || (nq && (!queries || !tspecs || !hspecs || !out_n || !out_sum_other || !out_error_bound || !out_cells ||
                    (out_stride && (!out_segment_ord || !out_key || !out_doc_count || !out_cell_first || !out_cell_n)) ||
                    (cell_capacity && (!out_cell_pos || !out_cell_count)))))
    return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  for (size_t qi = 0; qi < nq; ++qi) {
    const tq_terms_spec& sp = tspecs[qi];
    const tq_histogram_spec& hs = hspecs[qi];
    if (queries[qi].op == TQ_OP_PHRASE) return fail(TQ_ERR_UNSUPPORTED, "terms of phrase queries are not on the device path");
    if (sp.target > TQ_TERMS_BY_KEY || sp.order > TQ_ORDER_ASC || sp.missing_mode > TQ_TERMS_MISSING_AFTER_MAX || !sp.segment_size)
      return fail(TQ_ERR_INVALID_ARGUMENT, "terms spec: target, order, missing mode or segment_size");
    if (hs.kind > TQ_FAST_DATE) return fail(TQ_ERR_INVALID_ARGUMENT, "histogram kind");
    if (!(hs.interval > 0.0) || !std::isfinite(hs.interval)) return fail(TQ_ERR_INVALID_ARGUMENT, "histogram interval must be finite and > 0");
  }
  for (size_t qi = 0; qi < nq; ++qi) {
    out_n[qi] = out_cells[qi] = 0;
    out_sum_other[qi] = out_error_bound[qi] = 0;
    if (out_hits) out_hits[qi] = 0;
  }
  if (!nq) return TQ_OK;
  tq_batch* b = acquire_batch(c);
  if (!b) return fail(TQ_ERR_CUDA, "stream/event creation failed");
  struct Guard { tq_batch* b; ~Guard() { tq_batch_destroy(b); } } guard{b};
  CountPlan cp;
  std::vector<TermsSeg> tsegs;      // parallel to cp.segs
  std::vector<HistSeg> hsegs;       // parallel to cp.segs
  std::vector<TermsHistSeg> gsegs;  // parallel to cp.segs
  std::vector<HistUnit> windows;    // parallel to cp.units: the unit's keys
  std::vector<HistUnit> hunits;     // parallel to cp.units: the unit's buckets
  std::vector<HistQuery> hq(nq);
  std::vector<size_t> q_seg(nq + 1), q_unit(nq + 1);
  std::vector<uint64_t> q_counters(nq, 0), q_region(nq, 0), q_cells(nq, 0);
  {
    std::lock_guard<std::mutex> g(c->mu);
    TableScope table_scope{c};
    uint64_t built = 0, unused = 0;
    std::vector<const tq_term_seg*> order;
    std::vector<const SortColumn*> cols;
    std::vector<std::pair<unsigned long long, unsigned long long>> uwin;
    std::vector<std::pair<long long, long long>> hwin;  // per unit of the query: its first and last pos (first > last: none)
    for (size_t qi = 0; qi < nq; ++qi) {
      const tq_terms_spec& sp = tspecs[qi];
      const tq_histogram_spec& hs = hspecs[qi];
      const size_t s0 = cp.segs.size(), u0 = cp.units.size();
      q_seg[qi] = s0;
      q_unit[qi] = u0;
      int rc = plan_count(c, queries[qi], (uint32_t)qi, order, cp, &unused, true);
      if (rc != TQ_OK) return rc;
      const uint32_t flags = (out_hits ? kTermsHits : 0u) | (sp.missing_mode != TQ_TERMS_MISSING_NONE ? kTermsMissing : 0u) |
                             (sp.target == TQ_TERMS_BY_KEY ? kTermsByKey : 0u) | (sp.order == TQ_ORDER_ASC ? kTermsAsc : 0u);
      rc = plan_terms_query(c, sp, qi, flags, cp, s0, u0, tsegs, windows, cols, uwin, q_counters[qi], q_region[qi]);
      if (rc != TQ_OK) return rc;
      long long qbase = 0;
      uint64_t qlen = 0;
      rc = plan_hist_query(c, hs, qi, cp, s0, u0, kHistMaxBins, hsegs, cols, hwin, qbase, qlen);
      if (rc != TQ_OK) return rc;
      // per (query, segment): the union of its units' buckets, then each unit's window relative to its first
      std::vector<std::pair<long long, long long>> sspan(cp.segs.size() - s0, {1, 0});
      for (size_t ui = u0; ui < cp.units.size(); ++ui) {
        const auto& w = hwin[ui - u0];
        if (w.first > w.second) continue;
        auto& s = sspan[cp.units[ui].qseg - s0];
        s = s.first > s.second ? w : std::make_pair(std::min(s.first, w.first), std::max(s.second, w.second));
      }
      for (size_t si = s0; si < cp.segs.size(); ++si) {
        const auto& s = sspan[si - s0];
        const TermsSeg& z = tsegs[si];
        const uint32_t span = s.first <= s.second ? (uint32_t)(s.second - s.first + 1) : 0u;
        const uint64_t rows = std::min<uint64_t>(z.segment_size, (uint64_t)z.n_keys + ((z.flags & kTermsMissing) ? 1u : 0u));
        if (rows * span > c->terms_hist_budget)
          return fail(TQ_ERR_UNSUPPORTED, "query " + std::to_string(qi) + ": the histogram cells of its entries in a segment exceed the device budget (take the CPU path)");
        gsegs.push_back(TermsHistSeg{q_cells[qi], span ? s.first : 0ll, span, 0u});
        q_cells[qi] += rows * span;
      }
      if (q_cells[qi] > (1ull << 31))
        return fail(TQ_ERR_UNSUPPORTED, "query " + std::to_string(qi) + ": the histogram cells of its entries exceed 2^31 (take the CPU path)");
      for (size_t ui = u0; ui < cp.units.size(); ++ui) {
        const auto& w = hwin[ui - u0];
        hunits.push_back(w.first <= w.second ? HistUnit{(uint32_t)(w.first - gsegs[cp.units[ui].qseg].base), (uint32_t)(w.second - w.first + 1)}
                                             : HistUnit{0u, 0u});
      }
      hq[qi] = HistQuery{hs.interval, hs.offset, 0ll, 0ull, 0u, hs.kind, 0u, 0u};
    }
    q_seg[nq] = cp.segs.size();
    q_unit[nq] = cp.units.size();
    int rc = flush_builds(c, &built);
    if (rc != TQ_OK) return rc;
    hold_segments(c, b, queries, nq);  // (the segments, their filter views and the columns stay until the rows are in)
    for (size_t qi = 0; qi < nq; ++qi) {
      b->held_columns.push_back(tspecs[qi].column_id);
      b->held_columns.push_back(hspecs[qi].column_id);
    }
    std::sort(b->held_columns.begin(), b->held_columns.end());
    b->held_columns.erase(std::unique(b->held_columns.begin(), b->held_columns.end()), b->held_columns.end());
    for (uint32_t col : b->held_columns) ++c->sort_users[col];
  }
  if (cp.units.empty()) return TQ_OK;
  // waves of consecutive queries whose counters fit the counter budget and whose grids fit the cell budget (a query above either
  // runs alone); counters, regions and grids relative to the wave
  std::vector<uint64_t> at;
  const std::vector<TermsWave> waves = plan_terms_waves(q_counters, q_region, q_cells, c->terms_counter_budget, c->terms_hist_budget, q_seg, tsegs, &at);
  for (size_t qi = 0; qi < nq; ++qi)
    for (size_t si = q_seg[qi]; si < q_seg[qi + 1]; ++si) gsegs[si].grid += at[qi];
  uint64_t max_counters = 0, max_region = 0, max_cells = 0;
  size_t max_segs = 0;
  for (const TermsWave& w : waves) {
    max_counters = std::max(max_counters, w.counters);
    max_region = std::max(max_region, w.region);
    max_cells = std::max(max_cells, w.extra);
    max_segs = std::max(max_segs, q_seg[w.q1] - q_seg[w.q0]);
  }
  // descriptors: one H2D copy; scratch: hits | tile counters, then one wave's per-(query, segment) results | kept entries | their
  // first cells | the cursor | the cell list, then the wave's accumulators: missing counters and slots | counters | the grid
  Staging st;
  const size_t o_w = st.add(cp.words), o_s = st.add(cp.segs), o_u = st.add(cp.units), o_z = st.add(tsegs), o_h = st.add(windows),
               o_hz = st.add(hsegs), o_q = st.add(hq), o_g = st.add(gsegs), o_hu = st.add(hunits);
  TQ_CUDA(st.reserve(b->pin, b->dev));
  st.copy();
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off = align256(off + bytes); return at; };
  const size_t r_hits = take(nq * 8), r_ttiles = take(16), r_tiles = take(48), head_bytes = off;
  const size_t r_n = take(max_segs * 4), r_other = take(max_segs * 8), r_err = take(max_segs * 8), r_key = take(max_region * 8),
               r_count = take(max_region * 4), r_first = take(max_region * 4), r_total = take(max_segs * 4), r_cursor = take(8),
               r_cpos = take(max_cells * 4), r_ccount = take(max_cells * 4), wave_bytes = off - head_bytes;
  const size_t r_missing = take(max_segs * 4), r_mslot = take(max_segs * 4), r_counters = take(max_counters * 4), r_grid = take(max_cells * 4);
  TQ_CUDA(b->scratch.ensure(off));
  TQ_CUDA(b->res_pin.ensure(std::max(head_bytes, wave_bytes)));
  uint8_t* const d = b->scratch.p;
  TermsHistParams P{};
  P.t.c = CountParams{c->d_lists, st.on_device<const uint32_t>(o_w), st.on_device<const CountSeg>(o_s), st.on_device<const Unit>(o_u),
                      reinterpret_cast<unsigned long long*>(d + r_hits)};
  P.t.tsegs = st.on_device<const TermsSeg>(o_z);
  P.t.windows = st.on_device<const HistUnit>(o_h);
  P.t.counts = reinterpret_cast<uint32_t*>(d + r_counters);
  P.t.missing = reinterpret_cast<uint32_t*>(d + r_missing);
  P.t.tiles = reinterpret_cast<unsigned long long*>(d + r_ttiles);
  P.t.res_key = reinterpret_cast<unsigned long long*>(d + r_key);
  P.t.res_count = reinterpret_cast<uint32_t*>(d + r_count);
  P.t.res_n = reinterpret_cast<uint32_t*>(d + r_n);
  P.t.res_other = reinterpret_cast<unsigned long long*>(d + r_other);
  P.t.res_error = reinterpret_cast<unsigned long long*>(d + r_err);
  P.hsegs = st.on_device<const HistSeg>(o_hz);
  P.queries = st.on_device<const HistQuery>(o_q);
  P.gsegs = st.on_device<const TermsHistSeg>(o_g);
  P.hunits = st.on_device<const HistUnit>(o_hu);
  P.mslot = reinterpret_cast<const uint32_t*>(d + r_mslot);
  P.grid = reinterpret_cast<uint32_t*>(d + r_grid);
  P.tiles = reinterpret_cast<unsigned long long*>(d + r_tiles);
  P.cell_first = reinterpret_cast<uint32_t*>(d + r_first);
  P.cell_pos = reinterpret_cast<uint32_t*>(d + r_cpos);
  P.cell_count = reinterpret_cast<uint32_t*>(d + r_ccount);
  P.cell_total = reinterpret_cast<uint32_t*>(d + r_total);
  P.cursor = reinterpret_cast<unsigned long long*>(d + r_cursor);
  TermsMetricsParams M{};  // k_terms_mark's view: the terms and the missing key's slot
  M.mslot = reinterpret_cast<uint32_t*>(d + r_mslot);
  TQ_CUDA(cudaMemcpyAsync(b->dev.p, b->pin.p, st.bytes, cudaMemcpyHostToDevice, b->stream));
  TQ_CUDA(cudaMemsetAsync(d, 0, head_bytes, b->stream));  // hits, tile counters
  // per (query, segment): its kept entries (ascending key) with their non-empty cells, and its scalars, gathered wave by wave
  struct Entry { unsigned long long key; uint32_t count; std::vector<std::pair<long long, uint32_t>> cells; };
  std::vector<std::vector<Entry>> kept(cp.segs.size());
  std::vector<uint64_t> seg_other(cp.segs.size()), seg_err(cp.segs.size());
  float ms_total = 0;
  uint64_t ctas = 0;
  const uint8_t* h = b->res_pin.p;
  auto hp = [&](size_t r) { return h + (r - head_bytes); };
  for (const TermsWave& w : waves) {
    const size_t sa = q_seg[w.q0], sb = q_seg[w.q1], ua = q_unit[w.q0], ub = q_unit[w.q1];
    if (sa == sb) continue;
    P.t.unit_base = (uint32_t)ua;
    P.t.seg_base = (uint32_t)sa;
    M.t = P.t;
    TQ_CUDA(cudaMemsetAsync(d + r_missing, 0, r_counters + w.counters * 4 - r_missing, b->stream));  // missing .. counters
    TQ_CUDA(cudaMemsetAsync(d + r_grid, 0, w.extra * 4, b->stream));
    TQ_CUDA(cudaMemsetAsync(d + r_cursor, 0, 8, b->stream));
    TQ_CUDA(cudaEventRecord(b->ev_k0, b->stream));
    const unsigned nu = (unsigned)(ub - ua), ns = (unsigned)(sb - sa);
    if (nu) {
      (cp.mixed ? k_terms<true> : k_terms<false>)<<<nu, kThreads, 0, b->stream>>>(P.t);
      TQ_CUDA(cudaGetLastError());
    }
    k_terms_select<<<ns, kThreads, 0, b->stream>>>(P.t);
    TQ_CUDA(cudaGetLastError());
    k_terms_mark<<<ns, kThreads, 0, b->stream>>>(M);
    TQ_CUDA(cudaGetLastError());
    if (nu) {
      (cp.mixed ? k_terms_hist<true> : k_terms_hist<false>)<<<nu, kThreads, 0, b->stream>>>(P);
      TQ_CUDA(cudaGetLastError());
    }
    k_terms_hist_final<<<ns, kThreads, 0, b->stream>>>(P);
    TQ_CUDA(cudaGetLastError());
    TQ_CUDA(cudaEventRecord(b->ev_k1, b->stream));
    ctas += 2u * (uint64_t)nu + 3u * (uint64_t)ns;
    TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d + head_bytes, r_key - head_bytes + w.region * 8, cudaMemcpyDeviceToHost, b->stream));
    TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + (r_count - head_bytes), d + r_count, w.region * 4, cudaMemcpyDeviceToHost, b->stream));
    TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + (r_first - head_bytes), d + r_first, r_cpos - r_first, cudaMemcpyDeviceToHost, b->stream));  // first cells .. cursor
    TQ_CUDA(cudaStreamSynchronize(b->stream));
    unsigned long long n_cells;
    memcpy(&n_cells, hp(r_cursor), 8);
    if (n_cells) {  // the cell list, only as long as it is
      TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + (r_cpos - head_bytes), d + r_cpos, n_cells * 4, cudaMemcpyDeviceToHost, b->stream));
      TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + (r_ccount - head_bytes), d + r_ccount, n_cells * 4, cudaMemcpyDeviceToHost, b->stream));
      TQ_CUDA(cudaStreamSynchronize(b->stream));
    }
    float ms = 0;
    cudaEventElapsedTime(&ms, b->ev_k0, b->ev_k1);
    ms_total += ms;
    for (size_t si = sa; si < sb; ++si) {
      const size_t rel = si - sa;
      uint32_t n, total;
      memcpy(&n, hp(r_n) + rel * 4, 4);
      memcpy(&total, hp(r_total) + rel * 4, 4);
      memcpy(&seg_other[si], hp(r_other) + rel * 8, 8);
      memcpy(&seg_err[si], hp(r_err) + rel * 8, 8);
      kept[si].resize(n);
      uint32_t seg_first = 0;
      if (n) memcpy(&seg_first, hp(r_first) + tsegs[si].region * 4, 4);
      for (uint32_t j = 0; j < n; ++j) {
        const size_t e = tsegs[si].region + j;
        Entry& x = kept[si][j];
        memcpy(&x.key, hp(r_key) + e * 8, 8);
        memcpy(&x.count, hp(r_count) + e * 4, 4);
        uint32_t first, end = seg_first + total;
        memcpy(&first, hp(r_first) + e * 4, 4);
        if (j + 1 < n) memcpy(&end, hp(r_first) + (e + 1) * 4, 4);
        x.cells.resize(end - first);
        for (uint32_t k = first; k < end; ++k) {
          uint32_t pos, count;
          memcpy(&pos, hp(r_cpos) + (size_t)k * 4, 4);
          memcpy(&count, hp(r_ccount) + (size_t)k * 4, 4);
          x.cells[k - first] = {gsegs[si].base + (long long)pos, count};
        }
      }
    }
  }
  TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d, head_bytes, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  unsigned long long tiles[6];
  memcpy(tiles, h + r_tiles, 48);
  if (out_hits) memcpy(out_hits, h + r_hits, nq * 8);
  // rows: each query's segments by segment_ord, each in ascending key; cells: each entry's in ascending pos, in row order, the
  // queries' cells one after the other
  bool fits = true;
  std::vector<size_t> by_ord;
  uint64_t nc = 0;
  for (size_t qi = 0; qi < nq; ++qi) {
    by_ord.clear();
    for (size_t si = q_seg[qi]; si < q_seg[qi + 1]; ++si) by_ord.push_back(si);
    std::sort(by_ord.begin(), by_ord.end(), [&](size_t x, size_t y) { return cp.segment_ords[x] < cp.segment_ords[y]; });
    uint32_t n = 0;
    const uint64_t nc0 = nc;
    for (size_t si : by_ord) {
      out_sum_other[qi] += seg_other[si];
      out_error_bound[qi] += seg_err[si];
      for (const Entry& e : kept[si]) {
        if (n < out_stride) {
          const size_t at = qi * (size_t)out_stride + n;
          out_segment_ord[at] = cp.segment_ords[si];
          out_key[at] = e.key;
          out_doc_count[at] = e.count;
          out_cell_first[at] = nc;
          out_cell_n[at] = (uint32_t)e.cells.size();
        }
        for (const auto& cell : e.cells) {
          if (nc < cell_capacity) {
            out_cell_pos[nc] = cell.first;
            out_cell_count[nc] = cell.second;
          }
          ++nc;
        }
        ++n;
      }
    }
    out_n[qi] = n;
    out_cells[qi] = (uint32_t)(nc - nc0);
    fits = fits && n <= out_stride;
  }
  fits = fits && nc <= cell_capacity;
  {
    std::lock_guard<std::mutex> g(c->mu);
    c->terms_hist_ms += ms_total;
    c->terms_hist_units += ctas;
    c->terms_hist_tiles_seen += tiles[0];
    c->terms_hist_tiles_one_key += tiles[1];
    c->terms_hist_tiles_one_bucket += tiles[2];
    c->terms_hist_tiles_both += tiles[3];
    c->terms_hist_units_shared += tiles[4];
    c->terms_hist_units_global += tiles[5];
    c->terms_hist_waves += waves.size();
  }
  if (!fits) return fail(TQ_ERR_INVALID_ARGUMENT, "a terms row has more entries than out_stride, or the cells exceed cell_capacity: out_n and out_cells hold how many");
  return TQ_OK;
}

// ---- terms per histogram bucket ----------------------------------------------------------------------------------
int tq_histogram_terms_batch(tq_ctx* c, const tq_query* queries, const tq_histogram_spec* hspecs, const tq_terms_spec* tspecs, size_t nq,
                             uint32_t out_stride, int64_t* out_pos, uint64_t* out_doc_count, uint64_t* out_sum_other, uint64_t* out_error_bound,
                             uint64_t* out_entry_first, uint32_t* out_entry_n, uint32_t* out_n, uint64_t entry_capacity,
                             uint32_t* out_entry_segment_ord, uint64_t* out_entry_key, uint64_t* out_entry_count, uint32_t* out_entries,
                             uint64_t* out_hits) {
  if (!c || (nq && (!queries || !tspecs || !hspecs || !out_n || !out_entries ||
                    (out_stride && (!out_pos || !out_doc_count || !out_sum_other || !out_error_bound || !out_entry_first || !out_entry_n)) ||
                    (entry_capacity && (!out_entry_segment_ord || !out_entry_key || !out_entry_count)))))
    return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  for (size_t qi = 0; qi < nq; ++qi) {
    const tq_terms_spec& sp = tspecs[qi];
    const tq_histogram_spec& hs = hspecs[qi];
    if (queries[qi].op == TQ_OP_PHRASE) return fail(TQ_ERR_UNSUPPORTED, "histograms of phrase queries are not on the device path");
    if (sp.target > TQ_TERMS_BY_KEY || sp.order > TQ_ORDER_ASC || sp.missing_mode > TQ_TERMS_MISSING_AFTER_MAX || !sp.segment_size)
      return fail(TQ_ERR_INVALID_ARGUMENT, "terms spec: target, order, missing mode or segment_size");
    if (hs.kind > TQ_FAST_DATE) return fail(TQ_ERR_INVALID_ARGUMENT, "histogram kind");
    if (!(hs.interval > 0.0) || !std::isfinite(hs.interval)) return fail(TQ_ERR_INVALID_ARGUMENT, "histogram interval must be finite and > 0");
  }
  for (size_t qi = 0; qi < nq; ++qi) {
    out_n[qi] = out_entries[qi] = 0;
    if (out_hits) out_hits[qi] = 0;
  }
  if (!nq) return TQ_OK;
  tq_batch* b = acquire_batch(c);
  if (!b) return fail(TQ_ERR_CUDA, "stream/event creation failed");
  struct Guard { tq_batch* b; ~Guard() { tq_batch_destroy(b); } } guard{b};
  CountPlan cp;
  std::vector<TermsSeg> tsegs;      // parallel to cp.segs
  std::vector<HistSeg> hsegs;       // parallel to cp.segs
  std::vector<HistTermsSeg> gsegs;  // parallel to cp.segs
  std::vector<HistUnit> windows;    // parallel to cp.units: the unit's keys
  std::vector<HistUnit> hunits;     // parallel to cp.units: the unit's buckets
  std::vector<HistQuery> hq(nq);
  std::vector<size_t> q_seg(nq + 1), q_unit(nq + 1);
  std::vector<uint64_t> q_counters(nq, 0), q_region(nq, 0), q_cells(nq, 0), q_rows(nq, 0);
  {
    std::lock_guard<std::mutex> g(c->mu);
    TableScope table_scope{c};
    uint64_t built = 0, unused = 0;
    std::vector<const tq_term_seg*> order;
    std::vector<const SortColumn*> cols;
    std::vector<std::pair<unsigned long long, unsigned long long>> uwin;
    std::vector<std::pair<long long, long long>> hwin;  // per unit of the query: its first and last pos (first > last: none)
    for (size_t qi = 0; qi < nq; ++qi) {
      const tq_terms_spec& sp = tspecs[qi];
      const tq_histogram_spec& hs = hspecs[qi];
      const size_t s0 = cp.segs.size(), u0 = cp.units.size();
      q_seg[qi] = s0;
      q_unit[qi] = u0;
      int rc = plan_count(c, queries[qi], (uint32_t)qi, order, cp, &unused, true);
      if (rc != TQ_OK) return rc;
      const uint32_t flags = (out_hits ? kTermsHits : 0u) | (sp.missing_mode != TQ_TERMS_MISSING_NONE ? kTermsMissing : 0u) |
                             (sp.target == TQ_TERMS_BY_KEY ? kTermsByKey : 0u) | (sp.order == TQ_ORDER_ASC ? kTermsAsc : 0u);
      uint64_t counters = 0, region = 0;  // (the key windows only: no k_terms counters here)
      rc = plan_terms_query(c, sp, qi, flags, cp, s0, u0, tsegs, windows, cols, uwin, counters, region);
      if (rc != TQ_OK) return rc;
      long long qbase = 0;
      uint64_t qlen = 0;
      rc = plan_hist_query(c, hs, qi, cp, s0, u0, kHistMaxBins, hsegs, cols, hwin, qbase, qlen);
      if (rc != TQ_OK) return rc;
      // per (query, segment): the union of its units' buckets (its rows), then each unit's window relative to its first
      std::vector<std::pair<long long, long long>> sspan(cp.segs.size() - s0, {1, 0});
      for (size_t ui = u0; ui < cp.units.size(); ++ui) {
        const auto& w = hwin[ui - u0];
        if (w.first > w.second) continue;
        auto& s = sspan[cp.units[ui].qseg - s0];
        s = s.first > s.second ? w : std::make_pair(std::min(s.first, w.first), std::max(s.second, w.second));
      }
      for (size_t si = s0; si < cp.segs.size(); ++si) {
        const auto& s = sspan[si - s0];
        const TermsSeg& z = tsegs[si];
        const uint32_t span = s.first <= s.second ? (uint32_t)(s.second - s.first + 1) : 0u, ncol = z.n_keys + 1u;
        if ((uint64_t)span * ncol > c->hist_terms_budget)
          return fail(TQ_ERR_UNSUPPORTED, "query " + std::to_string(qi) + ": the (bucket, key) cells of a segment exceed the device budget (take the CPU path)");
        // the missing key: inside the keys it counts in its own column, outside them in column n_keys, one more entry before or
        // after the keys in key order; without one, column n_keys counts the docs without a value for the doc count alone
        const bool missing = z.flags & kTermsMissing, inside = missing && z.missing - z.base < (unsigned long long)z.n_keys;
        const bool extra = missing && !inside;
        gsegs.push_back(HistTermsSeg{q_cells[qi], span ? s.first : 0ll, span, ncol, inside ? (uint32_t)(z.missing - z.base) : z.n_keys,
                                     z.n_keys + (extra ? 1u : 0u), extra && z.missing < z.base ? 1u : 0u, (uint32_t)q_rows[qi]});
        q_cells[qi] += (uint64_t)span * ncol;
        q_rows[qi] += span;
      }
      if (q_cells[qi] > (1ull << 31))
        return fail(TQ_ERR_UNSUPPORTED, "query " + std::to_string(qi) + ": its (bucket, key) cells exceed 2^31 (take the CPU path)");
      for (size_t ui = u0; ui < cp.units.size(); ++ui) {
        const auto& w = hwin[ui - u0];
        hunits.push_back(w.first <= w.second ? HistUnit{(uint32_t)(w.first - gsegs[cp.units[ui].qseg].base), (uint32_t)(w.second - w.first + 1)}
                                             : HistUnit{0u, 0u});
      }
      hq[qi] = HistQuery{hs.interval, hs.offset, 0ll, 0ull, 0u, hs.kind, 0u, 0u};
    }
    q_seg[nq] = cp.segs.size();
    q_unit[nq] = cp.units.size();
    int rc = flush_builds(c, &built);
    if (rc != TQ_OK) return rc;
    hold_segments(c, b, queries, nq);  // (the segments, their filter views and the columns stay until the rows are in)
    for (size_t qi = 0; qi < nq; ++qi) {
      b->held_columns.push_back(tspecs[qi].column_id);
      b->held_columns.push_back(hspecs[qi].column_id);
    }
    std::sort(b->held_columns.begin(), b->held_columns.end());
    b->held_columns.erase(std::unique(b->held_columns.begin(), b->held_columns.end()), b->held_columns.end());
    for (uint32_t col : b->held_columns) ++c->sort_users[col];
  }
  if (cp.units.empty()) return TQ_OK;
  // waves of consecutive queries whose grids fit the cell budget (a query above it runs alone); grids and rows relative to the wave
  std::vector<uint64_t> at;
  const std::vector<TermsWave> waves = plan_terms_waves(q_counters, q_region, q_cells, 1u, c->hist_terms_budget, q_seg, tsegs, &at);
  uint64_t max_cells = 0, max_rows = 0;
  std::vector<uint64_t> wave_rows(waves.size(), 0);
  for (size_t wi = 0; wi < waves.size(); ++wi) {
    const TermsWave& w = waves[wi];
    uint64_t rows = 0;
    for (size_t qi = w.q0; qi < w.q1; ++qi) {
      for (size_t si = q_seg[qi]; si < q_seg[qi + 1]; ++si) {
        gsegs[si].grid += at[qi];
        gsegs[si].row += (uint32_t)rows;
      }
      rows += q_rows[qi];
    }
    wave_rows[wi] = rows;
    max_cells = std::max(max_cells, w.extra);
    max_rows = std::max(max_rows, rows);
  }
  // descriptors: one H2D copy; scratch: hits | tile counters, then one wave's cursors | rows | entries (read back), then its entry
  // scratch and its grid
  Staging st;
  const size_t o_w = st.add(cp.words), o_s = st.add(cp.segs), o_u = st.add(cp.units), o_z = st.add(tsegs), o_k = st.add(windows),
               o_hz = st.add(hsegs), o_q = st.add(hq), o_g = st.add(gsegs), o_hu = st.add(hunits);
  TQ_CUDA(st.reserve(b->pin, b->dev));
  st.copy();
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off = align256(off + bytes); return at; };
  const size_t r_hits = take(nq * 8), r_tiles = take(56), head_bytes = off;
  const size_t r_cursor = take(24), r_orows = take(max_rows * sizeof(HistTermsRow)), r_oents = take(max_cells * sizeof(HistTermsEntry)),
               wave_bytes = off - head_bytes;
  const size_t r_ents = take(max_cells * sizeof(HistTermsEntry)), r_grid = take(max_cells * 4);
  TQ_CUDA(b->scratch.ensure(off));
  TQ_CUDA(b->res_pin.ensure(std::max(head_bytes, wave_bytes)));
  uint8_t* const d = b->scratch.p;
  HistTermsParams P{};
  P.c = CountParams{c->d_lists, st.on_device<const uint32_t>(o_w), st.on_device<const CountSeg>(o_s), st.on_device<const Unit>(o_u),
                    reinterpret_cast<unsigned long long*>(d + r_hits)};
  P.tsegs = st.on_device<const TermsSeg>(o_z);
  P.windows = st.on_device<const HistUnit>(o_k);
  P.hsegs = st.on_device<const HistSeg>(o_hz);
  P.queries = st.on_device<const HistQuery>(o_q);
  P.gsegs = st.on_device<const HistTermsSeg>(o_g);
  P.hunits = st.on_device<const HistUnit>(o_hu);
  P.grid = reinterpret_cast<uint32_t*>(d + r_grid);
  P.ents = reinterpret_cast<HistTermsEntry*>(d + r_ents);
  P.out_rows = reinterpret_cast<HistTermsRow*>(d + r_orows);
  P.out_ents = reinterpret_cast<HistTermsEntry*>(d + r_oents);
  P.cursor = reinterpret_cast<unsigned long long*>(d + r_cursor);
  P.tiles = reinterpret_cast<unsigned long long*>(d + r_tiles);
  TQ_CUDA(cudaMemcpyAsync(b->dev.p, b->pin.p, st.bytes, cudaMemcpyHostToDevice, b->stream));
  TQ_CUDA(cudaMemsetAsync(d, 0, head_bytes, b->stream));  // hits, tile counters
  // per query: each (segment, non-empty bucket) with its kept entries (image, doc count) in ascending image, gathered wave by wave
  struct SegRow { long long pos; uint32_t segment_ord, doc_count, n; uint64_t other, error; size_t e0; };
  std::vector<std::vector<SegRow>> q_rows_out(nq);
  std::vector<std::pair<unsigned long long, uint32_t>> ents;
  float ms_total = 0;
  uint64_t ctas = 0;
  const uint8_t* h = b->res_pin.p;
  auto hp = [&](size_t r) { return h + (r - head_bytes); };
  int n_sm = 132;
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, c->device);
  for (size_t wi = 0; wi < waves.size(); ++wi) {
    const TermsWave& w = waves[wi];
    const size_t sa = q_seg[w.q0], sb = q_seg[w.q1], ua = q_unit[w.q0], ub = q_unit[w.q1];
    if (sa == sb) continue;
    P.unit_base = (uint32_t)ua;
    P.seg_base = (uint32_t)sa;
    P.n_segs = (uint32_t)(sb - sa);
    P.n_rows = (uint32_t)wave_rows[wi];
    TQ_CUDA(cudaMemsetAsync(d + r_grid, 0, w.extra * 4, b->stream));
    TQ_CUDA(cudaMemsetAsync(d + r_cursor, 0, 24, b->stream));
    TQ_CUDA(cudaEventRecord(b->ev_k0, b->stream));
    const unsigned nu = (unsigned)(ub - ua);
    const unsigned nf = (unsigned)std::min<uint64_t>((wave_rows[wi] + kWarps - 1) / kWarps, (uint64_t)n_sm * 8u);
    if (nu) {
      (cp.mixed ? k_hist_terms<true> : k_hist_terms<false>)<<<nu, kThreads, 0, b->stream>>>(P);
      TQ_CUDA(cudaGetLastError());
    }
    if (nf) {
      k_hist_terms_final<<<nf, kThreads, 0, b->stream>>>(P);
      TQ_CUDA(cudaGetLastError());
    }
    TQ_CUDA(cudaEventRecord(b->ev_k1, b->stream));
    ctas += (uint64_t)nu + nf;
    TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d + head_bytes, 24, cudaMemcpyDeviceToHost, b->stream));  // cursors
    TQ_CUDA(cudaStreamSynchronize(b->stream));
    unsigned long long cur[3];
    memcpy(cur, hp(r_cursor), 24);
    // the output lists, only as long as they are
    if (cur[2]) TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + (r_orows - head_bytes), d + r_orows, cur[2] * sizeof(HistTermsRow), cudaMemcpyDeviceToHost, b->stream));
    if (cur[1]) TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + (r_oents - head_bytes), d + r_oents, cur[1] * sizeof(HistTermsEntry), cudaMemcpyDeviceToHost, b->stream));
    if (cur[1] || cur[2]) TQ_CUDA(cudaStreamSynchronize(b->stream));
    float ms = 0;
    cudaEventElapsedTime(&ms, b->ev_k0, b->ev_k1);
    ms_total += ms;
    const HistTermsRow* rows_h = reinterpret_cast<const HistTermsRow*>(hp(r_orows));
    const HistTermsEntry* ents_h = reinterpret_cast<const HistTermsEntry*>(hp(r_oents));
    for (unsigned long long j = 0; j < cur[2]; ++j) {
      const HistTermsRow& x = rows_h[j];
      const size_t si = sa + x.seg;
      const TermsSeg& z = tsegs[si];
      const HistTermsSeg& g = gsegs[si];
      q_rows_out[cp.segs[si].query].push_back(SegRow{g.base + (long long)x.pos, cp.segment_ords[si], x.doc_count, x.n, x.other, x.error, ents.size()});
      for (uint32_t k = 0; k < x.n; ++k) {
        const HistTermsEntry& e = ents_h[(size_t)x.first + k];
        const uint32_t i = g.mfirst ? (e.key ? e.key - 1u : z.n_keys) : e.key;  // (its column)
        ents.emplace_back(i < z.n_keys ? z.base + i : z.missing, e.count);
      }
    }
  }
  TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d, head_bytes, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  unsigned long long tiles[7];
  memcpy(tiles, h + r_tiles, 56);
  if (out_hits) memcpy(out_hits, h + r_hits, nq * 8);
  // rows: each query's buckets in ascending pos, the segments' parts summed; entries: each bucket's by (segment_ord, image), in
  // row order, the queries' entries one after the other
  bool fits = true;
  uint64_t ne = 0;
  for (size_t qi = 0; qi < nq; ++qi) {
    std::vector<SegRow>& rs = q_rows_out[qi];
    std::sort(rs.begin(), rs.end(), [](const SegRow& x, const SegRow& y) { return x.pos != y.pos ? x.pos < y.pos : x.segment_ord < y.segment_ord; });
    uint32_t n = 0;
    const uint64_t ne0 = ne;
    for (size_t i = 0; i < rs.size();) {
      size_t j = i;
      uint64_t doc = 0, other = 0, error = 0, first = ne;
      for (; j < rs.size() && rs[j].pos == rs[i].pos; ++j) {
        doc += rs[j].doc_count;
        other += rs[j].other;
        error += rs[j].error;
        for (uint32_t k = 0; k < rs[j].n; ++k, ++ne)
          if (ne < entry_capacity) {
            out_entry_segment_ord[ne] = rs[j].segment_ord;
            out_entry_key[ne] = ents[rs[j].e0 + k].first;
            out_entry_count[ne] = ents[rs[j].e0 + k].second;
          }
      }
      if (n < out_stride) {
        const size_t a = qi * (size_t)out_stride + n;
        out_pos[a] = rs[i].pos;
        out_doc_count[a] = doc;
        out_sum_other[a] = other;
        out_error_bound[a] = error;
        out_entry_first[a] = first;
        out_entry_n[a] = (uint32_t)(ne - first);
      }
      ++n;
      i = j;
    }
    out_n[qi] = n;
    out_entries[qi] = (uint32_t)(ne - ne0);
    fits = fits && n <= out_stride;
  }
  fits = fits && ne <= entry_capacity;
  {
    std::lock_guard<std::mutex> g(c->mu);
    c->hist_terms_ms += ms_total;
    c->hist_terms_units += ctas;
    c->hist_terms_tiles_seen += tiles[0];
    c->hist_terms_tiles_one_key += tiles[1];
    c->hist_terms_tiles_one_bucket += tiles[2];
    c->hist_terms_tiles_both += tiles[3];
    c->hist_terms_units_shared += tiles[4];
    c->hist_terms_units_global += tiles[5];
    c->hist_terms_rows_cut += tiles[6];
    c->hist_terms_waves += waves.size();
  }
  if (!fits) return fail(TQ_ERR_INVALID_ARGUMENT, "a histogram row has more buckets than out_stride, or the entries exceed entry_capacity: out_n and out_entries hold how many");
  return TQ_OK;
}

// ---- range of a fast field ------------------------------------------------------------------------------------
// A range spec's bucket count and starts (TQ_ERR_INVALID_ARGUMENT).
static int check_range_spec(const tq_range_spec& r, uint32_t out_stride) {
  if (r.n_buckets < 1 || r.n_buckets > TQ_RANGE_MAX_BUCKETS) return fail(TQ_ERR_INVALID_ARGUMENT, "range spec: n_buckets must be 1..128");
  if (r.starts[0] != 0) return fail(TQ_ERR_INVALID_ARGUMENT, "range spec: starts[0] must be 0");
  for (uint32_t b = 1; b < r.n_buckets; ++b)
    if (r.starts[b] <= r.starts[b - 1]) return fail(TQ_ERR_INVALID_ARGUMENT, "range spec: starts must be strictly ascending");
  if (out_stride < r.n_buckets) return fail(TQ_ERR_INVALID_ARGUMENT, "out_stride must hold every bucket of a range");
  return TQ_OK;
}

int tq_range_batch(tq_ctx* c, const tq_query* queries, const tq_range_spec* rspecs, const tq_metrics_spec* mspecs, size_t nq,
                   uint32_t out_stride, uint64_t* out_doc_count, tq_metric_part* out_parts, uint64_t* out_hits) {
  if (!c || (nq && (!queries || !rspecs || !out_doc_count)) || (mspecs == nullptr) != (out_parts == nullptr))
    return fail(TQ_ERR_INVALID_ARGUMENT, "null (out_parts goes with mspecs)");
  TQ_CUDA(cudaSetDevice(c->device));
  constexpr uint32_t kC = kMetricsMaxColumns;
  for (size_t qi = 0; qi < nq; ++qi) {
    if (queries[qi].op == TQ_OP_PHRASE) return fail(TQ_ERR_UNSUPPORTED, "ranges of phrase queries are not on the device path");
    int rc = check_range_spec(rspecs[qi], out_stride);
    if (rc == TQ_OK && mspecs) rc = check_metrics_spec(mspecs[qi]);
    if (rc != TQ_OK) return rc;
  }
  const tq_metric_part empty{0ull, 0ull, 0ull, ~0ull, 0ull, 0.0, 0.0, INT32_MAX, 0u};
  for (size_t qi = 0; qi < nq; ++qi) {
    for (size_t i = qi * (size_t)out_stride; i < (qi + 1) * (size_t)out_stride; ++i) {
      out_doc_count[i] = 0;
      for (uint32_t k = 0; mspecs && k < kC; ++k) out_parts[i * kC + k] = empty;
    }
    if (out_hits) out_hits[qi] = 0;
  }
  if (!nq) return TQ_OK;
  tq_batch* b = acquire_batch(c);
  if (!b) return fail(TQ_ERR_CUDA, "stream/event creation failed");
  struct Guard { tq_batch* b; ~Guard() { tq_batch_destroy(b); } } guard{b};
  CountPlan cp;
  std::vector<RangeSeg> rsegs;      // parallel to cp.segs
  std::vector<MetricsSeg> msegs;    // parallel to cp.segs, with mspecs
  std::vector<RangeQuery> rq(nq);
  std::vector<HistUnit> windows;    // parallel to cp.units
  std::vector<unsigned long long> starts;  // every query's starts, back to back
  std::vector<size_t> start_at(nq), q_unit(nq + 1);
  {
    std::lock_guard<std::mutex> g(c->mu);
    TableScope table_scope{c};
    uint64_t built = 0, unused = 0;
    std::vector<const tq_term_seg*> order;
    std::vector<const SortColumn*> cols;
    for (size_t qi = 0; qi < nq; ++qi) {
      const tq_range_spec& r = rspecs[qi];
      const size_t s0 = cp.segs.size(), u0 = cp.units.size();
      q_unit[qi] = u0;
      int rc = plan_count(c, queries[qi], (uint32_t)qi, order, cp, &unused, true);
      if (rc != TQ_OK) return rc;
      rc = find_columns(c, r.column_id, cp, s0, "a range query", cols);
      if (rc != TQ_OK) return rc;
      for (const SortColumn* col : cols) rsegs.push_back(RangeSeg{col->d_values, col->d_present, col->d_tiles});
      if (mspecs) {
        rc = plan_metrics_segs(c, mspecs[qi], cp, s0, out_hits != nullptr, msegs);
        if (rc != TQ_OK) return rc;
      }
      windows.insert(windows.end(), cp.units.size() - u0, HistUnit{0u, r.n_buckets});  // (no per-unit window: every bucket)
      start_at[qi] = starts.size();
      starts.insert(starts.end(), r.starts, r.starts + r.n_buckets);
      rq[qi] = RangeQuery{nullptr, 0ull, r.n_buckets, out_hits ? kRangeHits : 0u};
    }
    q_unit[nq] = cp.units.size();
    int rc = flush_builds(c, &built);
    if (rc != TQ_OK) return rc;
    hold_segments(c, b, queries, nq);  // (the segments, their filter views and the columns stay until the rows are in)
    for (size_t qi = 0; qi < nq; ++qi) {
      b->held_columns.push_back(rspecs[qi].column_id);
      if (mspecs) hold_metric_columns(b, mspecs[qi]);
    }
    std::sort(b->held_columns.begin(), b->held_columns.end());
    b->held_columns.erase(std::unique(b->held_columns.begin(), b->held_columns.end()), b->held_columns.end());
    for (uint32_t col : b->held_columns) ++c->sort_users[col];
  }
  if (cp.units.empty()) return TQ_OK;
  // counters: without metrics every query's at once; with metrics in waves of accumulators that fit the budget
  std::vector<Wave> waves;
  if (mspecs) {
    std::vector<uint32_t> bins(nq);
    for (size_t qi = 0; qi < nq; ++qi) bins[qi] = rq[qi].n_bins;
    std::vector<unsigned long long> at, row_at;
    waves = plan_waves(bins, c->hist_metrics_budget, out_stride, at, row_at);
    for (size_t qi = 0; qi < nq; ++qi) rq[qi].counters = at[qi];
  } else {
    waves.push_back(Wave{0, nq, 0, 0});
    for (size_t qi = 0; qi < nq; ++qi) { rq[qi].counters = waves[0].counters; waves[0].counters += rq[qi].n_bins; }
  }
  uint64_t max_counters = 0;
  for (const Wave& w : waves) max_counters = std::max(max_counters, w.counters);
  // descriptors: one H2D copy (the queries point into the starts); scratch: hits | tile counters, then one wave's doc counters |
  // accumulators, read back as they are (the rows are dense)
  Staging st;
  const size_t o_w = st.add(cp.words), o_s = st.add(cp.segs), o_u = st.add(cp.units), o_z = st.add(rsegs), o_m = st.add(msegs),
               o_q = st.add(rq), o_h = st.add(windows), o_st = st.add(starts);
  TQ_CUDA(st.reserve(b->pin, b->dev));
  for (size_t qi = 0; qi < nq; ++qi) rq[qi].starts = st.on_device<const unsigned long long>(o_st) + start_at[qi];
  st.copy();
  const size_t part_row = (size_t)kC * sizeof(tq_metric_part);
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off = align256(off + bytes); return at; };
  const size_t r_hits = take(nq * 8), r_tiles = take(32), head_bytes = off;
  const size_t r_counters = take(max_counters * 8), r_acc = take(mspecs ? max_counters * part_row : 0), wave_bytes = off - head_bytes;
  TQ_CUDA(b->scratch.ensure(off));
  TQ_CUDA(b->res_pin.ensure(std::max(head_bytes, wave_bytes)));
  uint8_t* const d = b->scratch.p;
  const CountParams cparams{c->d_lists, st.on_device<const uint32_t>(o_w), st.on_device<const CountSeg>(o_s), st.on_device<const Unit>(o_u),
                            reinterpret_cast<unsigned long long*>(d + r_hits)};
  TQ_CUDA(cudaMemcpyAsync(b->dev.p, b->pin.p, st.bytes, cudaMemcpyHostToDevice, b->stream));
  TQ_CUDA(cudaMemsetAsync(d, 0, head_bytes, b->stream));  // hits, tile counters
  const uint8_t* h = b->res_pin.p;
  const size_t p_acc = r_acc - head_bytes;
  float ms_total = 0;
  for (const Wave& w : waves) {
    const size_t ua = q_unit[w.q0], ub = q_unit[w.q1];
    TQ_CUDA(cudaMemsetAsync(d + r_counters, 0, w.counters * 8, b->stream));
    if (mspecs) TQ_CUDA(cudaMemsetAsync(d + r_acc, 0, w.counters * part_row, b->stream));
    TQ_CUDA(cudaEventRecord(b->ev_k0, b->stream));
    if (ub > ua && mspecs) {
      RangeMetricsParams P{};
      P.c = cparams;
      P.rsegs = st.on_device<const RangeSeg>(o_z);
      P.msegs = st.on_device<const MetricsSeg>(o_m);
      P.queries = st.on_device<const RangeQuery>(o_q);
      P.windows = st.on_device<const HistUnit>(o_h);
      P.counts = reinterpret_cast<unsigned long long*>(d + r_counters);
      P.parts = reinterpret_cast<tq_metric_part*>(d + r_acc);
      P.tiles = reinterpret_cast<unsigned long long*>(d + r_tiles);
      P.unit_base = (uint32_t)ua;
      (cp.mixed ? k_range_metrics<true> : k_range_metrics<false>)<<<(unsigned)(ub - ua), kThreads, 0, b->stream>>>(P);
      TQ_CUDA(cudaGetLastError());
    } else if (ub > ua) {
      RangeParams P{};
      P.c = cparams;
      P.rsegs = st.on_device<const RangeSeg>(o_z);
      P.queries = st.on_device<const RangeQuery>(o_q);
      P.windows = st.on_device<const HistUnit>(o_h);
      P.counts = reinterpret_cast<unsigned long long*>(d + r_counters);
      P.tiles = reinterpret_cast<unsigned long long*>(d + r_tiles);
      (cp.mixed ? k_range<true> : k_range<false>)<<<(unsigned)(ub - ua), kThreads, 0, b->stream>>>(P);
      TQ_CUDA(cudaGetLastError());
    }
    TQ_CUDA(cudaEventRecord(b->ev_k1, b->stream));
    TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d + r_counters, w.counters * 8, cudaMemcpyDeviceToHost, b->stream));
    if (mspecs) TQ_CUDA(cudaMemcpyAsync(b->res_pin.p + p_acc, d + r_acc, w.counters * part_row, cudaMemcpyDeviceToHost, b->stream));
    TQ_CUDA(cudaStreamSynchronize(b->stream));
    float ms = 0;
    cudaEventElapsedTime(&ms, b->ev_k0, b->ev_k1);
    ms_total += ms;
    const unsigned long long* counts = reinterpret_cast<const unsigned long long*>(h);
    const tq_metric_part* parts = reinterpret_cast<const tq_metric_part*>(h + p_acc);
    for (size_t qi = w.q0; qi < w.q1; ++qi) {
      const size_t dst = qi * (size_t)out_stride;
      memcpy(out_doc_count + dst, counts + rq[qi].counters, (size_t)rq[qi].n_bins * 8);
      for (size_t i = 0; mspecs && i < (size_t)rq[qi].n_bins * kC; ++i) out_parts[dst * kC + i] = uncomplement(parts[rq[qi].counters * kC + i]);
    }
  }
  TQ_CUDA(cudaMemcpyAsync(b->res_pin.p, d, head_bytes, cudaMemcpyDeviceToHost, b->stream));
  TQ_CUDA(cudaStreamSynchronize(b->stream));
  if (out_hits) memcpy(out_hits, h + r_hits, nq * 8);
  unsigned long long tiles[2];
  memcpy(tiles, h + r_tiles, 16);
  {
    std::lock_guard<std::mutex> g(c->mu);
    c->range_ms += ms_total;
    c->range_units += cp.units.size();
    c->range_tiles_seen += tiles[0];
    c->range_tiles_one_bucket += tiles[1];
  }
  return TQ_OK;
}

// ---- codec-level access ---------------------------------------------------------------------------
static int resolve_single(tq_ctx* c, const tq_term_seg* list, uint32_t* id) {
  std::lock_guard<std::mutex> g(c->mu);
  TableScope table_scope{c};
  const Segment* seg;
  uint64_t built = 0;
  int rc = get_list(c, *list, false, id, &seg);
  if (rc != TQ_OK) return rc;
  return flush_builds(c, &built);
}

int tq_decode_postings(tq_ctx* c, const tq_term_seg* list, uint32_t* out_docs, uint32_t* out_tfs) {
  if (!c || !list || !out_docs) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  if (list->doc_freq == 0) return TQ_OK;
  uint32_t id;
  int rc = resolve_single(c, list, &id);
  if (rc != TQ_OK) return rc;
  uint32_t *d_docs = nullptr, *d_tfs = nullptr;
  const size_t bytes = (size_t)list->doc_freq * 4;
  TQ_CUDA(cudaMalloc(&d_docs, bytes));
  TQ_CUDA(cudaMalloc(&d_tfs, bytes));
  const uint32_t n_total = list->doc_freq / 128u + ((list->doc_freq % 128u) ? 1u : 0u);
  k_decode_list<<<(n_total + kWarps - 1) / kWarps, kThreads>>>(c->d_lists, id, d_docs, d_tfs);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpy(out_docs, d_docs, bytes, cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && out_tfs) e = cudaMemcpy(out_tfs, d_tfs, bytes, cudaMemcpyDeviceToHost);
  cudaFree(d_docs); cudaFree(d_tfs);
  if (e != cudaSuccess) return fail(TQ_ERR_CUDA, cudaGetErrorString(e));
  return TQ_OK;
}

int tq_block_table(tq_ctx* c, const tq_term_seg* list, float weight, float avg_fieldnorm, uint32_t* out_last_doc, float* out_block_max) {
  if (!c || !list || !out_last_doc || !out_block_max) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  TQ_CUDA(cudaSetDevice(c->device));
  const uint32_t n = list->doc_freq / 128u;
  if (n == 0) return TQ_OK;
  uint32_t id;
  int rc = resolve_single(c, list, &id);
  if (rc != TQ_OK) return rc;
  float tab[256];
  bm25_tf_cache(avg_fieldnorm, tab);
  float *d_cache = nullptr, *d_bm = nullptr;
  uint32_t* d_last = nullptr;
  TQ_CUDA(cudaMalloc(&d_cache, 1024));
  TQ_CUDA(cudaMalloc(&d_bm, (size_t)n * 4));
  TQ_CUDA(cudaMalloc(&d_last, (size_t)n * 4));
  cudaError_t e = cudaMemcpy(d_cache, tab, 1024, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    k_block_max<<<(n + 255) / 256, 256>>>(c->d_lists, id, weight, d_cache, d_last, d_bm);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(out_last_doc, d_last, (size_t)n * 4, cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemcpy(out_block_max, d_bm, (size_t)n * 4, cudaMemcpyDeviceToHost);
  cudaFree(d_cache); cudaFree(d_bm); cudaFree(d_last);
  if (e != cudaSuccess) return fail(TQ_ERR_CUDA, cudaGetErrorString(e));
  return TQ_OK;
}

}  // extern "C"
