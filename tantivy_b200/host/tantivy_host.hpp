// tantivy_host.hpp — host-side mirror, in C++, of the reference's search API for the accelerated path.
//
// The reference is Rust and no Rust toolchain exists in the build image, so the code that would sit in
// the reference above the C ABI (INTEGRATION.md) is written here with the reference's names, argument
// meaning and error behaviour, so that tests/cpp/host_mirror_tests.cpp reads like the reference's own tests:
//
//   Schema / SchemaBuilder / TEXT / STRING      src/schema/schema.rs, src/schema/text_options.rs:264-285
//   Term::from_field_text                        src/schema/term.rs
//   Index::create_in_ram, IndexWriter            src/index/index.rs, src/indexer/index_writer.rs (add_document,
//                                                delete_term, commit — one segment per commit, single thread)
//   IndexReader::searcher, Searcher              src/core/searcher.rs:133-141,180-237 (search, doc_freq, num_docs)
//   TermQuery, BooleanQuery, BoostQuery, Occur   src/query/term_query/term_query.rs, boolean_query/boolean_query.rs,
//                                                src/query/boost_query.rs
//   TopDocs::with_limit(..).and_offset(..)       src/collector/top_score_collector.rs:61-64,93-96,226-228
//   QueryParser (terms, +must, field:term only)  src/query/query_parser/query_parser.rs
//   CompositeFile / Footer readers (N1)          src/directory/composite_file.rs:111-170, src/directory/footer.rs
//
// Everything the hot path does — block decode, AND/OR, BM25, top-k, merge — happens behind
// tq_search_batch (include/tantivy_b200.h).  There is NO CPU search path in this file: a query shape the
// device path does not cover raises TantivyError (the reference-side shim would delegate those to
// Searcher::search, boolean_weight.rs:595-597), and a machine without a CUDA device raises on first search.
// The indexing side (tokenizer -> postings -> segment bytes) is host code, as in the reference; it exists so
// that tests and examples can build real segments without the Rust crate.
#pragma once
#include <algorithm>
#include <cctype>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <functional>
#include <iterator>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/tantivy_b200.h"
#include "../csrc/bm25_host.hpp"
#include "../csrc/segment_writer.hpp"

namespace tantivy_b200 {

using DocId = uint32_t;
using Score = float;
using SegmentOrdinal = uint32_t;
using Opstamp = uint64_t;

// ---- errors (src/error.rs: TantivyError::{InvalidArgument, SchemaError, SystemError, ...}) --------------------
class TantivyError : public std::runtime_error {
 public:
  enum Kind { InvalidArgument, SchemaError, DataCorruption, SystemError, Unsupported };
  TantivyError(Kind kind, const std::string& msg) : std::runtime_error(msg), kind_(kind) {}
  Kind kind() const { return kind_; }

 private:
  Kind kind_;
};

// ---- schema ------------------------------------------------------------------------------------------------
enum class IndexRecordOption { Basic = 0, WithFreqs = 1, WithFreqsAndPositions = 2 };

struct TextFieldIndexing {
  std::string tokenizer = "default";
  bool fieldnorms = true;
  IndexRecordOption record = IndexRecordOption::Basic;
  TextFieldIndexing set_tokenizer(const std::string& t) const { auto c = *this; c.tokenizer = t; return c; }
  TextFieldIndexing set_fieldnorms(bool f) const { auto c = *this; c.fieldnorms = f; return c; }
  TextFieldIndexing set_index_option(IndexRecordOption r) const { auto c = *this; c.record = r; return c; }
};
struct TextOptions {
  std::optional<TextFieldIndexing> indexing;
  TextOptions set_indexing_options(const TextFieldIndexing& i) const { auto c = *this; c.indexing = i; return c; }
};
// text_options.rs:264-285
inline const TextOptions STRING{TextFieldIndexing{"raw", true, IndexRecordOption::Basic}};
inline const TextOptions TEXT{TextFieldIndexing{"default", true, IndexRecordOption::WithFreqsAndPositions}};

struct Field {
  uint32_t id = 0;
  uint32_t field_id() const { return id; }
  bool operator==(const Field& o) const { return id == o.id; }
  bool operator<(const Field& o) const { return id < o.id; }
};
struct FieldEntry {
  std::string name;
  TextOptions options;
};
class Schema {
 public:
  std::optional<Field> get_field(const std::string& name) const {
    for (uint32_t i = 0; i < entries_.size(); ++i)
      if (entries_[i].name == name) return Field{i};
    return std::nullopt;
  }
  const FieldEntry& get_field_entry(Field f) const {
    if (f.id >= entries_.size()) throw TantivyError(TantivyError::SchemaError, "field does not exist");
    return entries_[f.id];
  }
  size_t num_fields() const { return entries_.size(); }

 private:
  friend class SchemaBuilder;
  std::vector<FieldEntry> entries_;
};
class SchemaBuilder {
 public:
  Field add_text_field(const std::string& name, const TextOptions& options) {
    for (auto& e : schema_.entries_)
      if (e.name == name) throw TantivyError(TantivyError::SchemaError, "field already exists: " + name);
    schema_.entries_.push_back({name, options});
    return Field{(uint32_t)schema_.entries_.size() - 1};
  }
  // a field of another type (date, u64, ...): keeps the field ids of a schema read from meta.json aligned; the search
  // path of this library does not cover it
  Field add_other_field(const std::string& name) { return add_text_field(name, TextOptions{}); }
  Schema build() { return schema_; }

 private:
  Schema schema_;
};

struct Term {
  Field field_;
  std::string text_;
  static Term from_field_text(Field field, const std::string& text) { return Term{field, text}; }
  Field field() const { return field_; }
  const std::string& text() const { return text_; }
};

struct DocAddress {
  SegmentOrdinal segment_ord = 0;
  DocId doc_id = 0;
  DocAddress() = default;
  DocAddress(SegmentOrdinal s, DocId d) : segment_ord(s), doc_id(d) {}
  bool operator==(const DocAddress& o) const { return segment_ord == o.segment_ord && doc_id == o.doc_id; }
  bool operator<(const DocAddress& o) const { return segment_ord != o.segment_ord ? segment_ord < o.segment_ord : doc_id < o.doc_id; }
};

class Document {
 public:
  Document& add_text(Field f, const std::string& text) { values_.push_back({f, text}); return *this; }
  const std::vector<std::pair<Field, std::string>>& field_values() const { return values_; }

 private:
  std::vector<std::pair<Field, std::string>> values_;
};

// ---- tokenizers ("default" = SimpleTokenizer + RemoveLongFilter(40) + LowerCaser, "raw"; tokenizer_manager.rs:53-70)
// ASCII rules: alphanumeric = [0-9A-Za-z] plus every byte >= 0x80 (multi-byte UTF-8 sequences stay inside a token);
// lower-casing touches ASCII only.
inline std::vector<std::string> tokenize(const std::string& tokenizer, const std::string& text) {
  std::vector<std::string> out;
  if (tokenizer == "raw") {
    out.push_back(text);
    return out;
  }
  if (tokenizer != "default") throw TantivyError(TantivyError::SchemaError, "unknown tokenizer: " + tokenizer);
  std::string cur;
  auto flush = [&]() {
    if (!cur.empty() && cur.size() < 40) out.push_back(cur);
    cur.clear();
  };
  for (unsigned char ch : text) {
    const bool alnum = (ch >= '0' && ch <= '9') || (ch >= 'a' && ch <= 'z') || (ch >= 'A' && ch <= 'Z') || ch >= 0x80;
    if (!alnum) { flush(); continue; }
    cur.push_back((ch >= 'A' && ch <= 'Z') ? (char)(ch - 'A' + 'a') : (char)ch);
  }
  flush();
  return out;
}

// ---- segment data --------------------------------------------------------------------------------------------
struct TermInfo {  // src/postings/term_info.rs:9-16
  uint32_t doc_freq = 0;
  uint64_t postings_start = 0, postings_end = 0;
  uint64_t positions_start = 0, positions_end = 0;  // byte range in the `.pos` sub-file (not used by this path yet)
  bool operator==(const TermInfo& o) const {
    return doc_freq == o.doc_freq && postings_start == o.postings_start && postings_end == o.postings_end &&
           positions_start == o.positions_start && positions_end == o.positions_end;
  }
};

struct FieldSegmentData {
  bool indexed = false;
  IndexRecordOption record = IndexRecordOption::Basic;
  bool has_fieldnorms = false;
  std::vector<uint8_t> idx_body;   // the field's `.idx` sub-file: u64 total_num_tokens + posting lists (serializer.rs:128)
  std::vector<uint8_t> fieldnorms; // the field's `.fieldnorm` sub-file: one fieldnorm id per doc
  std::vector<uint8_t> positions;  // the field's `.pos` sub-file (WithFreqsAndPositions fields written by the in-RAM writer)
  std::map<std::string, TermInfo> term_dict;          // term bytes -> TermInfo (filled from the `.term` file by files::open_index, or by the caller)
  std::map<std::string, std::vector<DocId>> term_docs; // kept by the in-RAM writer only, for delete_term
  uint64_t total_num_tokens() const {
    uint64_t v = 0;
    if (idx_body.size() >= 8) std::memcpy(&v, idx_body.data(), 8);
    return v;
  }
};

struct SegmentData {
  uint32_t max_doc = 0;
  std::vector<FieldSegmentData> fields;  // by field id
  std::vector<uint8_t> alive;            // empty = no deletes; else 64-bit LE words, bit set = alive (common/src/bitset.rs:362-407)
  uint32_t num_deleted = 0;
  bool is_alive(DocId d) const { return alive.empty() || ((alive[d >> 3] >> (d & 7u)) & 1u); }
};

class InvertedIndexReader {  // src/index/inverted_index_reader.rs:96 (get_term_info), :120-140 (doc_freq)
 public:
  explicit InvertedIndexReader(const FieldSegmentData* f) : f_(f) {}
  std::optional<TermInfo> get_term_info(const Term& term) const {
    auto it = f_->term_dict.find(term.text());
    if (it == f_->term_dict.end()) return std::nullopt;
    return it->second;
  }
  uint32_t doc_freq(const Term& term) const {
    auto ti = get_term_info(term);
    return ti ? ti->doc_freq : 0u;
  }
  uint64_t total_num_tokens() const { return f_->total_num_tokens(); }

 private:
  const FieldSegmentData* f_;
};

class SegmentReader {
 public:
  SegmentReader(std::shared_ptr<const SegmentData> data, SegmentOrdinal ord) : data_(std::move(data)), ord_(ord) {}
  uint32_t max_doc() const { return data_->max_doc; }
  uint32_t num_docs() const { return data_->max_doc - data_->num_deleted; }
  uint32_t num_deleted_docs() const { return data_->num_deleted; }
  bool is_deleted(DocId d) const { return !data_->is_alive(d); }
  SegmentOrdinal segment_ord() const { return ord_; }
  InvertedIndexReader inverted_index(Field field) const {
    if (field.id >= data_->fields.size() || !data_->fields[field.id].indexed)
      throw TantivyError(TantivyError::SchemaError, "field is not indexed");
    return InvertedIndexReader(&data_->fields[field.id]);
  }
  const SegmentData& data() const { return *data_; }

 private:
  std::shared_ptr<const SegmentData> data_;
  SegmentOrdinal ord_;
};

// ---- queries ---------------------------------------------------------------------------------------------------
enum class Occur { Should, Must, MustNot };

class Query {
 public:
  virtual ~Query() = default;
  virtual std::unique_ptr<Query> box_clone() const = 0;
};
using QueryBox = std::unique_ptr<Query>;

class TermQuery : public Query {
 public:
  TermQuery(Term term, IndexRecordOption option) : term_(std::move(term)), option_(option) {}
  const Term& term() const { return term_; }
  IndexRecordOption index_record_option() const { return option_; }
  QueryBox box_clone() const override { return std::make_unique<TermQuery>(*this); }

 private:
  Term term_;
  IndexRecordOption option_;
};

class BoostQuery : public Query {
 public:
  BoostQuery(QueryBox query, Score boost) : query_(std::move(query)), boost_(boost) {}
  BoostQuery(const BoostQuery& o) : query_(o.query_->box_clone()), boost_(o.boost_) {}
  const Query& inner() const { return *query_; }
  Score boost() const { return boost_; }
  QueryBox box_clone() const override { return std::make_unique<BoostQuery>(*this); }

 private:
  QueryBox query_;
  Score boost_;
};

class BooleanQuery : public Query {
 public:
  BooleanQuery() = default;
  explicit BooleanQuery(std::vector<std::pair<Occur, QueryBox>> clauses) : clauses_(std::move(clauses)) {}
  BooleanQuery(const BooleanQuery& o) {
    for (auto& c : o.clauses_) clauses_.emplace_back(c.first, c.second->box_clone());
  }
  // BooleanQuery::new_multiterms_query (boolean_query.rs): a disjunction of term queries
  static BooleanQuery new_multiterms_query(const std::vector<Term>& terms) {
    BooleanQuery q;
    for (auto& t : terms) q.clauses_.emplace_back(Occur::Should, std::make_unique<TermQuery>(t, IndexRecordOption::WithFreqs));
    return q;
  }
  const std::vector<std::pair<Occur, QueryBox>>& clauses() const { return clauses_; }
  QueryBox box_clone() const override { return std::make_unique<BooleanQuery>(*this); }

 private:
  std::vector<std::pair<Occur, QueryBox>> clauses_;
};

template <class Q>
QueryBox boxed(Q q) { return std::make_unique<Q>(std::move(q)); }

// ---- collector -------------------------------------------------------------------------------------------------
class TopDocs {
 public:
  // top_score_collector.rs:226-228: "Limit must be strictly greater than 0" (the reference panics)
  static TopDocs with_limit(size_t limit) {
    if (limit == 0) throw TantivyError(TantivyError::InvalidArgument, "Limit must be strictly greater than 0.");
    TopDocs t;
    t.limit_ = limit;
    return t;
  }
  TopDocs and_offset(size_t offset) const { TopDocs t = *this; t.offset_ = offset; return t; }
  TopDocs order_by_score() const { return *this; }
  size_t limit() const { return limit_; }
  size_t offset() const { return offset_; }

 private:
  size_t limit_ = 0, offset_ = 0;
};

// Count collector (src/collector/count_collector.rs): searcher.search(query, Count{}) -> number of alive matching docs
struct Count {};

// ---- device context shared by the searchers of one reader snapshot ------------------------------------------
class DeviceIndex {
 public:
  explicit DeviceIndex(int device) : device_(device) {}
  ~DeviceIndex() { if (ctx_) tq_ctx_destroy(ctx_); }
  DeviceIndex(const DeviceIndex&) = delete;
  DeviceIndex& operator=(const DeviceIndex&) = delete;

  // Uploads every indexed field of every segment once (segments are immutable).
  tq_ctx* ensure(const std::vector<SegmentReader>& segments) {
    std::lock_guard<std::mutex> g(mu_);
    if (ctx_) return ctx_;
    tq_ctx* c = nullptr;
    if (tq_ctx_create(device_, &c) != TQ_OK) {
      std::string msg = std::string("no usable CUDA device for the search path: ") + tq_last_error(nullptr);
      throw TantivyError(TantivyError::SystemError, msg);
    }
    for (auto& seg : segments) {
      const SegmentData& d = seg.data();
      for (uint32_t f = 0; f < d.fields.size(); ++f) {
        const FieldSegmentData& fd = d.fields[f];
        if (!fd.indexed) continue;
        const int rc = tq_segment_register(c, seg.segment_ord(), f, d.max_doc, (int)fd.record, fd.idx_body.data(), fd.idx_body.size(),
                                           fd.has_fieldnorms ? fd.fieldnorms.data() : nullptr, fd.has_fieldnorms ? fd.fieldnorms.size() : 0,
                                           d.alive.empty() ? nullptr : d.alive.data(), d.alive.size());
        if (rc != TQ_OK) {
          std::string msg = std::string("tq_segment_register: ") + tq_last_error(c);
          tq_ctx_destroy(c);
          throw TantivyError(TantivyError::SystemError, msg);
        }
      }
    }
    ctx_ = c;
    return ctx_;
  }

 private:
  int device_;
  tq_ctx* ctx_ = nullptr;
  std::mutex mu_;
};

// ---- searcher --------------------------------------------------------------------------------------------------
class Searcher {
 public:
  Searcher(Schema schema, std::vector<SegmentReader> segments, std::shared_ptr<DeviceIndex> device)
      : schema_(std::move(schema)), segments_(std::move(segments)), device_(std::move(device)) {}

  const Schema& schema() const { return schema_; }
  const std::vector<SegmentReader>& segment_readers() const { return segments_; }
  const SegmentReader& segment_reader(SegmentOrdinal ord) const { return segments_.at(ord); }
  // searcher.rs:133-141: alive docs
  uint64_t num_docs() const {
    uint64_t n = 0;
    for (auto& s : segments_) n += s.num_docs();
    return n;
  }
  // Bm25StatisticsProvider for Searcher (src/query/bm25.rs:27-50): N counts deleted docs too
  uint64_t total_num_docs() const {
    uint64_t n = 0;
    for (auto& s : segments_) n += s.max_doc();
    return n;
  }
  uint64_t total_num_tokens(Field field) const {
    uint64_t n = 0;
    for (auto& s : segments_) n += s.inverted_index(field).total_num_tokens();
    return n;
  }
  uint64_t doc_freq(const Term& term) const {
    uint64_t n = 0;
    for (auto& s : segments_) n += s.inverted_index(term.field()).doc_freq(term);
    return n;
  }

  // Searcher::search(query, &TopDocs::with_limit(k).and_offset(o).order_by_score())  (searcher.rs:180-237)
  std::vector<std::pair<Score, DocAddress>> search(const Query& query, const TopDocs& collector) const {
    std::vector<const Query*> one{&query};
    return std::move(search_batch(one, collector)[0]);
  }

  // searcher.search(&query, &Count)
  size_t search(const Query& query, const Count&) const {
    Plan p = plan(query, 1);
    if (p.matches_nothing) return 0;
    tq_query q;
    std::memset(&q, 0, sizeof(q));
    q.op = p.op; q.n_terms = (uint32_t)p.weight.size(); q.k = 1; q.n_term_segs = (uint32_t)p.term_segs.size();
    q.term_segs = p.term_segs.data(); q.weight = p.weight.data(); q.avg_fieldnorm = p.avg.data(); q.term_flags = p.flags.data();
    tq_ctx* ctx = device_->ensure(segments_);
    uint64_t n = 0;
    if (tq_count_batch(ctx, &q, 1, &n) != TQ_OK) throw TantivyError(TantivyError::SystemError, std::string("tq_count_batch: ") + tq_last_error(ctx));
    return (size_t)n;
  }

  // searcher.search(&query, &(Count, TopDocs::with_limit(k)))  (the tuple collector, collector/mod.rs:322-365): both halves from
  // ONE device batch -- the count is taken from the postings the top-k search decodes anyway (TQ_QUERY_COUNT_HITS).
  std::pair<size_t, std::vector<std::pair<Score, DocAddress>>> search(const Query& query, const std::pair<Count, TopDocs>& collectors) const {
    const TopDocs& collector = collectors.second;
    const size_t k = collector.limit() + collector.offset();
    if (k > TQ_MAX_K) throw TantivyError(TantivyError::InvalidArgument, "limit + offset exceeds TQ_MAX_K");
    Plan p = plan(query, (uint32_t)k);
    if (p.matches_nothing) return {0, {}};
    tq_query q;
    std::memset(&q, 0, sizeof(q));
    q.op = p.op; q.n_terms = (uint32_t)p.weight.size(); q.k = (uint32_t)k; q.n_term_segs = (uint32_t)p.term_segs.size();
    q.term_segs = p.term_segs.data(); q.weight = p.weight.data(); q.avg_fieldnorm = p.avg.data(); q.term_flags = p.flags.data();
    q.flags = TQ_QUERY_COUNT_HITS;
    tq_ctx* ctx = device_->ensure(segments_);
    tq_batch* b = nullptr;
    auto check = [&](int rc, const char* what) {
      if (rc == TQ_OK) return;
      const std::string msg = std::string(what) + ": " + tq_last_error(ctx);
      if (b) tq_batch_destroy(b);
      throw TantivyError(TantivyError::SystemError, msg);
    };
    std::vector<float> sc(k);
    std::vector<uint32_t> sg(k), dc(k);
    uint32_t cnt = 0;
    uint64_t n_hits = 0;
    check(tq_batch_prepare(ctx, &q, 1, &b), "tq_batch_prepare");
    check(tq_batch_run(b), "tq_batch_run");
    check(tq_batch_fetch(b, (uint32_t)k, sc.data(), sg.data(), dc.data(), &cnt), "tq_batch_fetch");
    check(tq_batch_fetch_hits(b, &n_hits), "tq_batch_fetch_hits");
    tq_batch_destroy(b);
    std::vector<std::pair<Score, DocAddress>> rows;
    for (size_t r = collector.offset(); r < cnt; ++r) rows.emplace_back(sc[r], DocAddress(sg[r], dc[r]));
    return {(size_t)n_hits, std::move(rows)};
  }

  // Many queries in one device batch (throughput; single queries are launch-latency bound).
  std::vector<std::vector<std::pair<Score, DocAddress>>> search_batch(const std::vector<const Query*>& queries, const TopDocs& collector) const {
    const size_t k = collector.limit() + collector.offset();
    if (k > TQ_MAX_K) throw TantivyError(TantivyError::InvalidArgument, "limit + offset exceeds TQ_MAX_K");
    const size_t nq = queries.size();
    std::vector<Plan> plans(nq);
    std::vector<tq_query> tq(nq);
    std::vector<size_t> live;
    for (size_t i = 0; i < nq; ++i) {
      plans[i] = plan(*queries[i], (uint32_t)k);
      if (plans[i].matches_nothing) continue;
      Plan& p = plans[i];
      tq_query q;
      std::memset(&q, 0, sizeof(q));
      q.op = p.op; q.n_terms = (uint32_t)p.weight.size(); q.k = (uint32_t)k; q.n_term_segs = (uint32_t)p.term_segs.size();
      q.term_segs = p.term_segs.data(); q.weight = p.weight.data(); q.avg_fieldnorm = p.avg.data(); q.term_flags = p.flags.data();
      tq[live.size()] = q;
      live.push_back(i);
    }
    std::vector<std::vector<std::pair<Score, DocAddress>>> out(nq);
    if (live.empty()) return out;
    tq_ctx* ctx = device_->ensure(segments_);
    const size_t n = live.size();
    std::vector<float> sc(n * k);
    std::vector<uint32_t> sg(n * k), dc(n * k), cnt(n);
    if (tq_search_batch(ctx, tq.data(), n, (uint32_t)k, sc.data(), sg.data(), dc.data(), cnt.data()) != TQ_OK)
      throw TantivyError(TantivyError::SystemError, std::string("tq_search_batch: ") + tq_last_error(ctx));
    for (size_t j = 0; j < n; ++j) {
      auto& rows = out[live[j]];
      for (size_t r = collector.offset(); r < cnt[j]; ++r) rows.emplace_back(sc[j * k + r], DocAddress(sg[j * k + r], dc[j * k + r]));
    }
    return out;
  }

 private:
  struct Clause {
    Term term;
    IndexRecordOption option;
    Score boost;
  };
  struct Plan {
    int32_t op = TQ_OP_TERM;
    bool matches_nothing = false;
    std::vector<float> weight, avg;
    std::vector<uint8_t> flags;
    std::vector<tq_term_seg> term_segs;
  };

  // SpecializedScorer classification (boolean_weight.rs:17-21,57-68,318-330): TermQuery -> TERM, BooleanQuery of
  // only-Must TermQuerys -> AND, only-Should -> OR; BoostQuery multiplies the Bm25Weight (bm25.rs:129-131).
  static void flatten(const Query& q, Score boost, std::vector<Clause>& out, int32_t* op) {
    if (auto* t = dynamic_cast<const TermQuery*>(&q)) {
      out.push_back({t->term(), t->index_record_option(), boost});
      *op = TQ_OP_TERM;
      return;
    }
    if (auto* b = dynamic_cast<const BoostQuery*>(&q)) return flatten(b->inner(), boost * b->boost(), out, op);
    if (auto* b = dynamic_cast<const BooleanQuery*>(&q)) {
      std::optional<Occur> occur;
      for (auto& c : b->clauses()) {
        if (c.first == Occur::MustNot || (occur && *occur != c.first))
          throw TantivyError(TantivyError::Unsupported, "only all-Must or all-Should term clauses run on the device path");
        occur = c.first;
        const Query* inner = c.second.get();
        Score cb = boost;
        while (auto* bq = dynamic_cast<const BoostQuery*>(inner)) { cb *= bq->boost(); inner = &bq->inner(); }
        auto* t = dynamic_cast<const TermQuery*>(inner);
        if (!t) throw TantivyError(TantivyError::Unsupported, "nested boolean clauses do not run on the device path");
        out.push_back({t->term(), t->index_record_option(), cb});
      }
      *op = (!occur || out.size() == 1) ? TQ_OP_TERM : (*occur == Occur::Must ? TQ_OP_AND : TQ_OP_OR);
      return;
    }
    throw TantivyError(TantivyError::Unsupported, "query type does not run on the device path");
  }

  Plan plan(const Query& query, uint32_t) const {
    Plan p;
    std::vector<Clause> clauses;
    flatten(query, 1.0f, clauses, &p.op);
    if (clauses.empty()) { p.matches_nothing = true; return p; }
    if (clauses.size() > TQ_MAX_TERMS) throw TantivyError(TantivyError::InvalidArgument, "too many clauses for the device path");
    const uint64_t n_docs = total_num_docs();
    for (uint32_t i = 0; i < clauses.size(); ++i) {
      const Clause& c = clauses[i];
      const FieldEntry& fe = schema_.get_field_entry(c.term.field());
      if (!fe.options.indexing) throw TantivyError(TantivyError::SchemaError, "field " + fe.name + " is not indexed");
      // Bm25Weight::for_terms (bm25.rs:95-118)
      const uint64_t df = doc_freq(c.term);
      p.weight.push_back(tq::bm25_weight(df, n_docs, c.boost));
      p.avg.push_back(n_docs ? (float)total_num_tokens(c.term.field()) / (float)n_docs : 0.0f);
      const bool field_has_freq = fe.options.indexing->record != IndexRecordOption::Basic;
      p.flags.push_back((field_has_freq && c.option == IndexRecordOption::Basic) ? TQ_TERM_IGNORE_FREQ : 0);
      for (auto& s : segments_) {
        auto ti = s.inverted_index(c.term.field()).get_term_info(c.term);
        if (ti && ti->doc_freq)
          p.term_segs.push_back(tq_term_seg{i, s.segment_ord(), c.term.field().id, ti->doc_freq, ti->postings_start, ti->postings_end});
      }
    }
    if (p.term_segs.empty()) p.matches_nothing = true;
    return p;
  }

  Schema schema_;
  std::vector<SegmentReader> segments_;
  std::shared_ptr<DeviceIndex> device_;
};

class IndexReader {
 public:
  IndexReader(Schema schema, std::vector<std::shared_ptr<const SegmentData>> segments, int device) : schema_(std::move(schema)) {
    for (size_t i = 0; i < segments.size(); ++i) readers_.emplace_back(segments[i], (SegmentOrdinal)i);
    device_ = std::make_shared<DeviceIndex>(device);
  }
  Searcher searcher() const { return Searcher(schema_, readers_, device_); }

 private:
  Schema schema_;
  std::vector<SegmentReader> readers_;
  std::shared_ptr<DeviceIndex> device_;
};

// ---- index + writer ----------------------------------------------------------------------------------------------
class Index;
class IndexWriter {
 public:
  explicit IndexWriter(Index* index) : index_(index) {}
  Opstamp add_document(const Document& doc) {
    pending_.push_back({doc, ++opstamp_});
    return opstamp_;
  }
  Opstamp delete_term(const Term& term) {
    deletes_.push_back({term, ++opstamp_});
    return opstamp_;
  }
  Opstamp commit();

 private:
  struct PendingDoc { Document doc; Opstamp opstamp; };
  struct PendingDelete { Term term; Opstamp opstamp; };
  Index* index_;
  std::vector<PendingDoc> pending_;
  std::vector<PendingDelete> deletes_;
  Opstamp opstamp_ = 0;
};

class Index {
 public:
  static Index create_in_ram(const Schema& schema) { return Index(schema); }
  // An index over segments read from files the reference wrote (N1): the caller supplies each segment's data.
  static Index from_segments(const Schema& schema, std::vector<std::shared_ptr<const SegmentData>> segments) {
    Index ix(schema);
    ix.segments_ = std::move(segments);
    return ix;
  }
  const Schema& schema() const { return schema_; }
  IndexWriter writer() { return IndexWriter(this); }
  IndexWriter writer_for_tests() { return IndexWriter(this); }
  IndexReader reader() const { return IndexReader(schema_, segments_, device_); }
  void set_device(int device) { device_ = device; }
  const std::vector<std::shared_ptr<const SegmentData>>& segments() const { return segments_; }

 private:
  friend class IndexWriter;
  explicit Index(const Schema& schema) : schema_(schema) {}
  Schema schema_;
  std::vector<std::shared_ptr<const SegmentData>> segments_;
  int device_ = 0;
};

namespace detail {
inline void set_deleted(SegmentData& seg, DocId d) {
  if (seg.alive.empty()) {
    seg.alive.assign(((size_t)seg.max_doc + 63) / 64 * 8, 0);
    for (DocId i = 0; i < seg.max_doc; ++i) seg.alive[i >> 3] |= (uint8_t)(1u << (i & 7u));
  }
  if (seg.is_alive(d)) {
    seg.alive[d >> 3] &= (uint8_t)~(1u << (d & 7u));
    ++seg.num_deleted;
  }
}
}  // namespace detail

// One segment per commit (the reference's single-threaded writer, index_writer.rs; segment_writer.rs for the
// per-field token counting -> fieldnorm, serializer.rs for the bytes).
inline Opstamp IndexWriter::commit() {
  const Schema& schema = index_->schema_;
  // deletes hit every doc of the committed segments and the pending docs added before the delete (opstamp order)
  for (auto& del : deletes_) {
    for (auto& sp : index_->segments_) {
      const FieldSegmentData& fd = sp->fields.at(del.term.field().id);
      auto it = fd.term_docs.find(del.term.text());
      if (it == fd.term_docs.end()) continue;
      auto copy = std::make_shared<SegmentData>(*sp);
      for (DocId d : it->second) detail::set_deleted(*copy, d);
      sp = copy;
    }
  }
  if (!pending_.empty()) {
    auto seg = std::make_shared<SegmentData>();
    seg->max_doc = (uint32_t)pending_.size();
    const size_t nf = schema.num_fields();
    seg->fields.resize(nf);
    std::vector<std::map<std::string, std::vector<std::pair<DocId, uint32_t>>>> postings(nf);
    std::vector<std::map<std::string, std::vector<uint32_t>>> pos_deltas(nf);  // per term: first position, then gaps, per posting
    std::vector<std::vector<uint32_t>> num_tokens(nf, std::vector<uint32_t>(seg->max_doc, 0));
    for (DocId d = 0; d < seg->max_doc; ++d) {
      std::map<uint32_t, uint32_t> end_position;                        // per field: where the next value's positions start
      std::map<uint32_t, std::map<std::string, uint32_t>> last_pos_of;  // per field: a term's previous position in this doc
      for (auto& fv : pending_[d].doc.field_values()) {
        const FieldEntry& fe = schema.get_field_entry(fv.first);
        if (!fe.options.indexing) continue;
        // several values of one field: the next value starts POSITION_GAP = 1 after the previous one's last token
        // (postings_writer.rs:19,140-163); the fieldnorm counts tokens only
        const uint32_t start_position = end_position[fv.first.id];
        uint32_t value_end = start_position, tok_index = 0;
        std::map<std::string, uint32_t>& last_pos = last_pos_of[fv.first.id];
        for (auto& tok : tokenize(fe.options.indexing->tokenizer, fv.second)) {
          auto& pl = postings[fv.first.id][tok];
          const uint32_t position = start_position + tok_index++;  // token ordinal (positions/mod.rs:1-5)
          value_end = position + 1;
          const bool again = !pl.empty() && pl.back().first == d;
          if (again) ++pl.back().second; else pl.push_back({d, 1u});
          auto lp = last_pos.find(tok);
          pos_deltas[fv.first.id][tok].push_back(again && lp != last_pos.end() ? position - lp->second : position);
          last_pos[tok] = position;
          ++num_tokens[fv.first.id][d];
        }
        end_position[fv.first.id] = value_end + 1;
      }
    }
    for (uint32_t f = 0; f < nf; ++f) {
      const FieldEntry& fe = schema.get_field_entry(Field{f});
      FieldSegmentData& fd = seg->fields[f];
      if (!fe.options.indexing) continue;
      fd.indexed = true;
      fd.record = fe.options.indexing->record;
      fd.has_fieldnorms = fe.options.indexing->fieldnorms;
      uint64_t total = 0;
      for (uint32_t n : num_tokens[f]) total += n;
      if (fd.has_fieldnorms) {
        fd.fieldnorms.resize(seg->max_doc);
        for (DocId d = 0; d < seg->max_doc; ++d) fd.fieldnorms[d] = tq::fieldnorm_to_id(num_tokens[f][d]);
      }
      tq::FieldPostingsWriter w((int)fd.record, total, fd.has_fieldnorms ? fd.fieldnorms.data() : nullptr, seg->max_doc);
      std::vector<uint32_t> docs, tfs;
      for (auto& kv : postings[f]) {  // std::map: terms in byte order, as the term dictionary requires
        docs.clear(); tfs.clear();
        for (auto& p : kv.second) { docs.push_back(p.first); tfs.push_back(p.second); }
        const tq::TermInfoOut ti = w.add_term(docs.data(), fd.record == IndexRecordOption::Basic ? nullptr : tfs.data(), (uint32_t)docs.size());
        TermInfo info{ti.doc_freq, ti.postings_start, ti.postings_end};
        if (fd.record == IndexRecordOption::WithFreqsAndPositions) {  // serializer.rs:436-454: positions_range of the term
          const std::vector<uint32_t>& pd = pos_deltas[f][kv.first];
          info.positions_start = fd.positions.size();
          tq::encode_positions(pd.data(), pd.size(), fd.positions);
          info.positions_end = fd.positions.size();
        }
        fd.term_dict[kv.first] = info;
        fd.term_docs[kv.first] = docs;
      }
      fd.idx_body = w.body();
    }
    for (auto& del : deletes_) {
      auto it = seg->fields.at(del.term.field().id).term_docs.find(del.term.text());
      if (it == seg->fields[del.term.field().id].term_docs.end()) continue;
      for (DocId d : it->second)
        if (pending_[d].opstamp < del.opstamp) detail::set_deleted(*seg, d);
    }
    index_->segments_.push_back(seg);
  }
  pending_.clear();
  deletes_.clear();
  return ++opstamp_;
}

// ---- a small query parser: whitespace separated terms, optional '+' (Must) and 'field:' prefixes ---------------
class QueryParser {
 public:
  static QueryParser for_index(const Index& index, std::vector<Field> default_fields) { return QueryParser(index.schema(), std::move(default_fields)); }
  QueryBox parse_query(const std::string& text) const {
    std::vector<std::pair<Occur, QueryBox>> clauses;
    size_t i = 0;
    while (i < text.size()) {
      while (i < text.size() && text[i] == ' ') ++i;
      size_t j = i;
      while (j < text.size() && text[j] != ' ') ++j;
      if (j == i) break;
      std::string tok = text.substr(i, j - i);
      i = j;
      Occur occur = Occur::Should;
      if (tok[0] == '+') { occur = Occur::Must; tok.erase(0, 1); }
      else if (tok[0] == '-') { occur = Occur::MustNot; tok.erase(0, 1); }
      std::vector<Field> fields = default_fields_;
      const size_t colon = tok.find(':');
      if (colon != std::string::npos) {
        auto f = schema_.get_field(tok.substr(0, colon));
        if (!f) throw TantivyError(TantivyError::InvalidArgument, "Field does not exist: '" + tok.substr(0, colon) + "'");
        fields = {*f};
        tok.erase(0, colon + 1);
      }
      if (fields.size() != 1) throw TantivyError(TantivyError::Unsupported, "exactly one default field (or a field: prefix) is supported");
      const FieldEntry& fe = schema_.get_field_entry(fields[0]);
      if (!fe.options.indexing) throw TantivyError(TantivyError::SchemaError, "field is not indexed");
      auto toks = tokenize(fe.options.indexing->tokenizer, tok);
      if (toks.size() != 1) throw TantivyError(TantivyError::Unsupported, "phrases are not supported by this parser");
      const IndexRecordOption opt = fe.options.indexing->record == IndexRecordOption::Basic ? IndexRecordOption::Basic : IndexRecordOption::WithFreqs;
      clauses.emplace_back(occur, std::make_unique<TermQuery>(Term::from_field_text(fields[0], toks[0]), opt));
    }
    if (clauses.size() == 1 && clauses[0].first != Occur::MustNot) return std::move(clauses[0].second);
    return std::make_unique<BooleanQuery>(std::move(clauses));
  }

 private:
  QueryParser(Schema schema, std::vector<Field> fields) : schema_(std::move(schema)), default_fields_(std::move(fields)) {}
  Schema schema_;
  std::vector<Field> default_fields_;
};

// ---- N1: file framing written by the reference ---------------------------------------------------------------
namespace files {

inline uint32_t crc32(const uint8_t* p, size_t n) {  // IEEE 802.3, as crc32fast (footer.rs)
  static uint32_t table[256];
  static bool init = false;
  if (!init) {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c & 1u) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
      table[i] = c;
    }
    init = true;
  }
  uint32_t c = 0xFFFFFFFFu;
  for (size_t i = 0; i < n; ++i) c = table[(c ^ p[i]) & 0xFFu] ^ (c >> 8);
  return c ^ 0xFFFFFFFFu;
}

struct Footer {
  uint32_t index_format_version = 0;
  uint32_t crc = 0;
  size_t body_len = 0;  // bytes before the footer
};

// file = body ‖ JSON footer ‖ u32 json_len ‖ u32 magic (1337)   (src/directory/footer.rs:18-22,44-51,85-120)
inline Footer read_footer(const uint8_t* file, size_t len, bool verify_crc = true) {
  auto u32_at = [&](size_t off) { uint32_t v; std::memcpy(&v, file + off, 4); return v; };
  if (len < 8) throw TantivyError(TantivyError::DataCorruption, "file too short for a footer");
  if (u32_at(len - 4) != 1337u) throw TantivyError(TantivyError::DataCorruption, "footer magic byte mismatch");
  const uint32_t json_len = u32_at(len - 8);
  if ((size_t)json_len + 8 > len) throw TantivyError(TantivyError::DataCorruption, "footer length out of range");
  const std::string json(reinterpret_cast<const char*>(file + len - 8 - json_len), json_len);
  auto number_after = [&](const std::string& key) -> uint64_t {
    const size_t k = json.find("\"" + key + "\"");
    if (k == std::string::npos) throw TantivyError(TantivyError::DataCorruption, "footer lacks " + key);
    size_t p = json.find(':', k) + 1;
    while (p < json.size() && json[p] == ' ') ++p;
    uint64_t v = 0;
    bool any = false;
    while (p < json.size() && json[p] >= '0' && json[p] <= '9') { v = v * 10 + (uint64_t)(json[p++] - '0'); any = true; }
    if (!any) throw TantivyError(TantivyError::DataCorruption, "footer field " + key + " is not a number");
    return v;
  };
  Footer f;
  f.index_format_version = (uint32_t)number_after("index_format_version");
  f.crc = (uint32_t)number_after("crc");
  f.body_len = len - 8 - json_len;
  if (verify_crc && crc32(file, f.body_len) != f.crc) throw TantivyError(TantivyError::DataCorruption, "crc mismatch");
  return f;
}

inline uint64_t read_vint(const uint8_t* p, size_t len, size_t* pos) {  // common/src/vint.rs: 7 bits per byte, stop bit 0x80
  uint64_t v = 0;
  uint32_t shift = 0;
  while (*pos < len) {
    const uint8_t b = p[(*pos)++];
    v |= (uint64_t)(b & 127u) << shift;
    if (b & 128u) return v;
    shift += 7;
    if (shift > 63) break;
  }
  throw TantivyError(TantivyError::DataCorruption, "truncated vint");
}

struct FileSlice { size_t offset = 0, len = 0; };

// composite = sub-files ‖ VInt(n) ‖ n x (VInt(offset delta), u32 field LE, VInt(idx)) ‖ u32 footer_len
// (src/directory/composite_file.rs:71-85,111-145). Returns (field, idx) -> byte range inside `body`.
inline std::map<std::pair<uint32_t, uint32_t>, FileSlice> open_composite(const uint8_t* body, size_t len) {
  if (len < 4) throw TantivyError(TantivyError::DataCorruption, "composite file too short");
  uint32_t footer_len;
  std::memcpy(&footer_len, body + len - 4, 4);
  if ((size_t)footer_len + 4 > len) throw TantivyError(TantivyError::DataCorruption, "composite footer length out of range");
  const size_t data_len = len - 4 - footer_len;
  const uint8_t* foot = body + data_len;
  size_t pos = 0;
  const uint64_t n = read_vint(foot, footer_len, &pos);
  std::vector<std::pair<std::pair<uint32_t, uint32_t>, size_t>> starts;
  size_t offset = 0;
  for (uint64_t i = 0; i < n; ++i) {
    offset += (size_t)read_vint(foot, footer_len, &pos);
    if (pos + 4 > footer_len) throw TantivyError(TantivyError::DataCorruption, "truncated composite footer");
    uint32_t field;
    std::memcpy(&field, foot + pos, 4);
    pos += 4;
    const uint32_t idx = (uint32_t)read_vint(foot, footer_len, &pos);
    starts.push_back({{field, idx}, offset});
  }
  std::map<std::pair<uint32_t, uint32_t>, FileSlice> out;
  for (size_t i = 0; i < starts.size(); ++i) {
    const size_t end = i + 1 < starts.size() ? starts[i + 1].second : data_len;
    if (starts[i].second > end || end > data_len) throw TantivyError(TantivyError::DataCorruption, "composite offsets out of order");
    out[starts[i].first] = FileSlice{starts[i].second, end - starts[i].second};
  }
  return out;
}

// Fills one field of a SegmentData from the segment's `.idx` and `.fieldnorm` files as written by the reference.
inline void load_field(SegmentData& seg, Field field, IndexRecordOption record, const std::vector<uint8_t>& idx_file,
                       const std::vector<uint8_t>* fieldnorm_file) {
  if (seg.fields.size() <= field.id) seg.fields.resize(field.id + 1);
  FieldSegmentData& fd = seg.fields[field.id];
  const Footer fi = read_footer(idx_file.data(), idx_file.size());
  auto idx_parts = open_composite(idx_file.data(), fi.body_len);
  auto it = idx_parts.find({field.id, 0});
  if (it == idx_parts.end()) throw TantivyError(TantivyError::DataCorruption, "field has no postings sub-file");
  fd.indexed = true;
  fd.record = record;
  fd.idx_body.assign(idx_file.begin() + (long)it->second.offset, idx_file.begin() + (long)(it->second.offset + it->second.len));
  if (fd.idx_body.size() < 8) throw TantivyError(TantivyError::DataCorruption, "postings sub-file lacks total_num_tokens");
  if (fieldnorm_file) {
    const Footer ff = read_footer(fieldnorm_file->data(), fieldnorm_file->size());
    auto fn_parts = open_composite(fieldnorm_file->data(), ff.body_len);
    auto fit = fn_parts.find({field.id, 0});
    if (fit != fn_parts.end()) {
      if (fit->second.len != seg.max_doc) throw TantivyError(TantivyError::DataCorruption, "fieldnorm sub-file length != max_doc");
      fd.has_fieldnorms = true;
      fd.fieldnorms.assign(fieldnorm_file->begin() + (long)fit->second.offset, fieldnorm_file->begin() + (long)(fit->second.offset + fit->second.len));
    }
  }
}

// ---- term dictionary framing (N2, the part the reference tree specifies) ------------------------------------------
// A field's `.term` sub-file = [fst][TermInfoStore][u64 store_len][u32 FST_VERSION = 1][u32 dictionary type = 1]
// (src/termdict/fst_termdict/termdict.rs:78-89,125-143; src/termdict/mod.rs:51-90).  The FST (term bytes -> ordinal) is
// crate tantivy-fst 0.5, not in the reference tree: it is handed back as raw bytes.  The TermInfoStore (ordinal ->
// TermInfo) is in-tree (term_info_store.rs:12-158) and is read here.
inline uint64_t extract_bits(const uint8_t* data, size_t len, size_t addr_bits, uint8_t num_bits) {  // term_info_store.rs:106-124
  const size_t addr_byte = addr_bits / 8;
  uint8_t buf[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (addr_byte < len) std::memcpy(buf, data + addr_byte, std::min<size_t>(8, len - addr_byte));
  uint64_t v;
  std::memcpy(&v, buf, 8);
  v >>= (addr_bits % 8);
  return num_bits >= 64 ? v : v & ((1ull << num_bits) - 1ull);
}

class TermInfoStore {
 public:
  static constexpr size_t kBlockLen = 256, kBlockMetaBytes = 8 + 28 + 3;
  TermInfoStore() = default;
  TermInfoStore(const uint8_t* data, size_t len) {  // TermInfoStore::open
    if (len < 16) throw TantivyError(TantivyError::DataCorruption, "term info store too short");
    uint64_t meta_len;
    std::memcpy(&meta_len, data, 8);
    std::memcpy(&num_terms_, data + 8, 8);
    if (16 + meta_len > len) throw TantivyError(TantivyError::DataCorruption, "term info store: block metas out of range");
    metas_.assign(data + 16, data + 16 + meta_len);
    bits_.assign(data + 16 + meta_len, data + len);
  }
  uint64_t num_terms() const { return num_terms_; }
  TermInfo get(uint64_t term_ord) const {  // TermInfoStore::get + TermInfoBlockMeta::deserialize_term_info
    if (term_ord >= num_terms_) throw TantivyError(TantivyError::InvalidArgument, "term ordinal out of range");
    const size_t block = (size_t)(term_ord / kBlockLen), inner = (size_t)(term_ord % kBlockLen);
    if ((block + 1) * kBlockMetaBytes > metas_.size()) throw TantivyError(TantivyError::DataCorruption, "term info store: missing block meta");
    const uint8_t* m = metas_.data() + block * kBlockMetaBytes;
    uint64_t offset, post_start, pos_start;
    uint32_t doc_freq, post_len, pos_len;
    std::memcpy(&offset, m, 8);
    std::memcpy(&doc_freq, m + 8, 4);
    std::memcpy(&post_start, m + 12, 8);
    std::memcpy(&post_len, m + 20, 4);
    std::memcpy(&pos_start, m + 24, 8);
    std::memcpy(&pos_len, m + 32, 4);
    TermInfo ref;
    ref.doc_freq = doc_freq; ref.postings_start = post_start; ref.postings_end = post_start + post_len;
    ref.positions_start = pos_start; ref.positions_end = pos_start + pos_len;
    if (inner == 0) return ref;
    const uint8_t df_bits = m[36], post_bits = m[37], pos_bits = m[38];
    const size_t nbits = (size_t)df_bits + post_bits + pos_bits;
    if (offset > bits_.size()) throw TantivyError(TantivyError::DataCorruption, "term info store: block offset out of range");
    const uint8_t* d = bits_.data() + offset;
    const size_t dl = bits_.size() - (size_t)offset;
    const size_t a_post = nbits * (inner - 1);  // the end of an entry is the start of the next one
    const size_t a_pos = a_post + post_bits;
    const size_t a_df = a_pos + pos_bits;
    TermInfo ti;
    ti.postings_start = ref.postings_start + extract_bits(d, dl, a_post, post_bits);
    ti.postings_end = ref.postings_start + extract_bits(d, dl, a_post + nbits, post_bits);
    ti.positions_start = ref.positions_start + extract_bits(d, dl, a_pos, pos_bits);
    ti.positions_end = ref.positions_start + extract_bits(d, dl, a_pos + nbits, pos_bits);
    ti.doc_freq = (uint32_t)extract_bits(d, dl, a_df, df_bits);
    return ti;
  }

 private:
  uint64_t num_terms_ = 0;
  std::vector<uint8_t> metas_, bits_;
};

struct TermDictionaryParts {
  std::vector<uint8_t> fst;  // tantivy-fst 0.5 bytes (not decoded here)
  TermInfoStore store;
};
inline TermDictionaryParts open_term_dictionary(const uint8_t* sub, size_t len) {
  if (len < 16) throw TantivyError(TantivyError::DataCorruption, "term dictionary too short");
  uint32_t dict_type, fst_version;
  uint64_t store_len;
  std::memcpy(&dict_type, sub + len - 4, 4);
  std::memcpy(&fst_version, sub + len - 8, 4);
  std::memcpy(&store_len, sub + len - 16, 8);
  if (dict_type != 1u) throw TantivyError(TantivyError::Unsupported, "term dictionary is not the FST kind (sstable dictionaries: quickwit feature)");
  if (fst_version != 1u) throw TantivyError(TantivyError::DataCorruption, "unsupported FST_VERSION");
  if (store_len + 16 > len) throw TantivyError(TantivyError::DataCorruption, "term dictionary: store length out of range");
  TermDictionaryParts parts;
  const size_t fst_len = len - 16 - (size_t)store_len;
  parts.fst.assign(sub, sub + fst_len);
  parts.store = TermInfoStore(sub + fst_len, (size_t)store_len);
  return parts;
}

// ---- term dictionary, FST kind: the term -> ordinal map (N2) --------------------------------------------------------------------
// Third-party format: crate `tantivy-fst` 0.5 (Cargo.toml:28; a fork of BurntSushi's `fst`, same file format), NOT in the reference
// tree.  Its published layout (fst `raw/node.rs`, `raw/mod.rs`, `raw/common_inputs.rs`) is restated here:
//   file   = u64 version (1 or 2) ‖ u64 type ‖ nodes ‖ u64 number of keys ‖ u64 root address; address 0 is the empty final state
//   node   = addressed by its LAST byte (the state byte), fields laid out towards lower addresses:
//     11cccccc  one transition to the node compiled just before (address = end of this node - 1); c = input code (0: the input byte
//               precedes the state byte), output 0
//     10cccccc  one transition: [output (osize)] [address delta (tsize)] [sizes = tsize << 4 | osize] [input] state
//     0Fnnnnnn  any number: F = final; n = transitions (0: the count precedes the state byte, a stored 1 means 256);
//               [final output] [outputs] [address deltas] [inputs] [256-byte index if version >= 2 and more than 32 transitions]
//               [sizes] [count] state; transition i has its input at distance i + 1 below the index, its delta and output i slots below
//               theirs; address = end of the node - delta (delta 0: the empty final state)
//   value of a key = sum of the outputs on its path + the final output of its last node (here: the term ordinal,
//   fst_termdict/termdict.rs:60-66)
//   input codes 1..63 = the 63 most common bytes of the crate's reference corpus (table below).
// PARITY UNPINNED beyond what the reference tree holds: the compat fixtures' one-term FST ("dateformat": nine 11cccccc nodes, one
// 10cccccc node, codes of t e o a r m d f) decodes as restated; multi-transition nodes, outputs and the other 55 table entries are
// pinned by nothing in the tree.  Every dictionary is therefore checked when it is opened (for_each below): the keys must come
// out strictly ascending, as many as the footer says, with the ordinals 0, 1, 2, ... -- a structural misreading throws
// DataCorruption instead of answering wrongly (a wrong table entry that keeps the order would not be caught).
class Fst {
 public:
  Fst() = default;
  Fst(const uint8_t* data, size_t len) : d_(data, data + len) {
    if (len < 32) throw TantivyError(TantivyError::DataCorruption, "fst: too short");
    std::memcpy(&version_, d_.data(), 8);
    if (version_ != 1 && version_ != 2) throw TantivyError(TantivyError::Unsupported, "fst: version " + std::to_string(version_));
    std::memcpy(&len_, d_.data() + len - 16, 8);
    std::memcpy(&root_, d_.data() + len - 8, 8);
    if (root_ >= len - 16) throw TantivyError(TantivyError::DataCorruption, "fst: root address out of range");
  }
  uint64_t len() const { return len_; }
  // Fst::get: the value of `key`, if it is in the set
  std::optional<uint64_t> get(const std::string& key) const {
    Node n = node(root_);
    uint64_t out = 0;
    for (unsigned char b : key) {
      bool found = false;
      for (size_t i = 0; i < n.ntrans && !found; ++i) {
        const Trans t = transition(n, i);
        if (t.input == b) { out += t.output; n = node(t.addr); found = true; }
      }
      if (!found) return std::nullopt;
    }
    if (!n.is_final) return std::nullopt;
    return out + n.final_output;
  }
  // every (key, value) in key order
  void for_each(const std::function<void(const std::string&, uint64_t)>& f) const {
    std::string key;
    size_t budget = 64 * d_.size() + 1024;  // a well-formed FST is walked in far fewer steps; a damaged one must not run away
    walk(node(root_), 0, key, f, 0, budget);
  }

 private:
  struct Node { int kind = 0; size_t start = 0, end = 0, ntrans = 0; bool is_final = false; uint64_t final_output = 0; uint8_t state = 0, tsize = 0, osize = 0; };
  struct Trans { uint8_t input; uint64_t output; size_t addr; };
  static uint8_t common_input(uint8_t code) {  // COMMON_INPUTS_INV[code - 1] (fst raw/common_inputs.rs): the first 63 entries
    static const char kInv[] = "te/oasripcnw.hlm-du012g=:bf3y5&_4v9678k%?xCDASFIBEjPTzRNM+LOqHG";
    return (uint8_t)kInv[code - 1];
  }
  uint8_t at(size_t i) const {
    if (i >= d_.size()) throw TantivyError(TantivyError::DataCorruption, "fst: address out of range");
    return d_[i];
  }
  uint64_t unpack(size_t i, uint8_t n) const {  // little-endian, n bytes
    uint64_t v = 0;
    for (uint8_t k = 0; k < n; ++k) v |= (uint64_t)at(i + k) << (8 * k);
    return v;
  }
  size_t delta_addr(size_t i, uint8_t tsize, size_t node_end) const {
    const uint64_t delta = unpack(i, tsize);
    if (delta == 0) return 0;
    if (delta > node_end) throw TantivyError(TantivyError::DataCorruption, "fst: transition address out of range");
    return node_end - (size_t)delta;
  }
  size_t index_size(const Node& n) const { return version_ >= 2 && n.ntrans > 32 ? 256 : 0; }
  Node node(size_t addr) const {
    Node n;
    if (addr == 0) { n.kind = 0; n.is_final = true; return n; }  // EMPTY_ADDRESS: the final state without transitions
    if (addr < 16) throw TantivyError(TantivyError::DataCorruption, "fst: node address inside the header");
    n.start = addr;
    n.state = at(addr);
    const uint8_t top = n.state >> 6;
    if (top == 3) {  // OneTransNext
      n.kind = 1; n.ntrans = 1;
      const size_t input_len = (n.state & 63u) ? 0 : 1;
      n.end = addr - input_len;
    } else if (top == 2) {  // OneTrans
      n.kind = 2; n.ntrans = 1;
      const size_t input_len = (n.state & 63u) ? 0 : 1;
      const uint8_t sizes = at(addr - input_len - 1);
      n.tsize = sizes >> 4; n.osize = sizes & 15u;
      n.end = addr - input_len - 1 - n.tsize - n.osize;
    } else {  // AnyTrans
      n.kind = 3;
      n.is_final = (n.state & 64u) != 0;
      const size_t ntrans_len = (n.state & 63u) ? 0 : 1;
      if (ntrans_len) { n.ntrans = at(addr - 1); if (n.ntrans == 1) n.ntrans = 256; } else n.ntrans = n.state & 63u;
      const uint8_t sizes = at(addr - ntrans_len - 1);
      n.tsize = sizes >> 4; n.osize = sizes & 15u;
      const size_t total_trans = n.ntrans + n.ntrans * n.tsize + index_size(n);
      const size_t final_osize = n.is_final ? n.osize : 0;
      const size_t body = ntrans_len + 1 + total_trans + n.ntrans * n.osize + final_osize;
      if (body > addr) throw TantivyError(TantivyError::DataCorruption, "fst: node larger than the file");
      n.end = addr - body;
      if (n.is_final && n.osize) n.final_output = unpack(n.end, n.osize);
    }
    if (n.tsize > 8 || n.osize > 8) throw TantivyError(TantivyError::DataCorruption, "fst: pack size above 8");
    return n;
  }
  Trans transition(const Node& n, size_t i) const {
    if (n.kind == 1) {
      const uint8_t code = n.state & 63u;
      return Trans{code ? common_input(code) : at(n.start - 1), 0, n.end - 1};
    }
    if (n.kind == 2) {
      const uint8_t code = n.state & 63u;
      const size_t input_len = code ? 0 : 1;
      const size_t ti = n.start - input_len - 1 - n.tsize;
      return Trans{code ? common_input(code) : at(n.start - 1), n.osize ? unpack(ti - n.osize, n.osize) : 0, delta_addr(ti, n.tsize, n.end)};
    }
    const size_t ntrans_len = (n.state & 63u) ? 0 : 1;
    const size_t below_sizes = n.start - ntrans_len - 1 - index_size(n);  // the inputs end here
    const uint8_t input = at(below_sizes - i - 1);
    const size_t ti = below_sizes - n.ntrans - i * n.tsize - n.tsize;
    const size_t total_trans = n.ntrans + n.ntrans * n.tsize + index_size(n);
    const uint64_t out = n.osize ? unpack(n.start - ntrans_len - 1 - total_trans - i * n.osize - n.osize, n.osize) : 0;
    return Trans{input, out, delta_addr(ti, n.tsize, n.end)};
  }
  void walk(const Node& n, uint64_t out, std::string& key, const std::function<void(const std::string&, uint64_t)>& f, int depth, size_t& budget) const {
    if (depth > 4096) throw TantivyError(TantivyError::Unsupported, "fst: a key of more than 4096 bytes (or a cycle)");
    if (budget < n.ntrans + 1) throw TantivyError(TantivyError::DataCorruption, "fst: more states than the file can hold (damaged)");
    budget -= n.ntrans + 1;
    if (n.is_final) f(key, out + n.final_output);
    // transitions in input order (AnyTrans keeps them sorted; walk them by ascending input whichever way they are stored)
    std::vector<Trans> ts;
    ts.reserve(n.ntrans);
    for (size_t i = 0; i < n.ntrans; ++i) ts.push_back(transition(n, i));
    std::sort(ts.begin(), ts.end(), [](const Trans& a, const Trans& b) { return a.input < b.input; });
    for (const Trans& t : ts) {
      key.push_back((char)t.input);
      walk(node(t.addr), out + t.output, key, f, depth + 1, budget);
      key.pop_back();
    }
  }
  std::vector<uint8_t> d_;
  uint64_t version_ = 0, len_ = 0, root_ = 0;
};

// ---- term dictionary, SSTable kind (N2; the `quickwit` feature: src/termdict/mod.rs:20-30,62-72) -------------------------
// Unlike the FST, this dictionary is specified entirely inside the reference tree (crate `sstable/`, format in sstable/README.md):
//   dictionary = blocks ‖ index ‖ [u64 store_offset (v3)] ‖ u64 index_offset ‖ u64 num_terms ‖ u32 version (2 or 3)
//                                                              (Dictionary::open, sstable/src/dictionary.rs:278-296; index/mod.rs:19-50)
//   block      = u32 block_len (incl. the compress byte; <= 1 ends the stream) ‖ u8 compress (1 = zstd) ‖ values ‖ deltas
//                                                              (BlockReader::read_block, sstable/src/block_reader.rs:47-106)
//   values     = VInt n ‖ VInt postings_start ‖ VInt positions_start ‖ n x (VInt doc_freq, VInt postings_len, VInt positions_len),
//                common::VInt (stop bit 0x80 on the last byte)          (TermInfoValueReader::load, sstable_termdict/mod.rs:56-81)
//   delta      = keep|add byte (add << 4 | keep), or 0x01 ‖ vint keep ‖ vint add (sstable's own vint: 0x80 = continue) ‖ `add`
//                suffix bytes                                           (DeltaReader::read_keep_add, sstable/src/delta.rs:166-196)
// The block index (which of its two forms holds a tantivy-fst map) only accelerates point look-ups: the keys and TermInfos
// of ALL blocks are streamed here, in order, which is what fills FieldSegmentData::term_dict.  Pinned on the byte-level golden of
// sstable/src/lib.rs:417-448 and on sstable_termdict/mod.rs:117-150.
inline uint64_t read_sstable_vint(const uint8_t* p, size_t len, size_t* pos) {  // sstable/src/vint.rs:25-39 (0x80 = more bytes follow)
  uint64_t v = 0;
  uint32_t shift = 0;
  while (*pos < len) {
    const uint8_t b = p[(*pos)++];
    v |= (uint64_t)(b & 127u) << shift;
    if (b < 128u) return v;
    shift += 7;
    if (shift > 63) break;
  }
  throw TantivyError(TantivyError::DataCorruption, "sstable: truncated vint");
}

struct SSTableEntry { std::string key; TermInfo info; };

// `with_term_infos` = false reads a VoidSSTable (no values: the reference's own golden vector)
inline std::vector<SSTableEntry> read_sstable(const uint8_t* dict, size_t len, bool with_term_infos = true) {
  if (len < 20) throw TantivyError(TantivyError::DataCorruption, "sstable: too short for its footer");
  uint64_t index_offset, num_terms;
  uint32_t version;
  std::memcpy(&index_offset, dict + len - 20, 8);
  std::memcpy(&num_terms, dict + len - 12, 8);
  std::memcpy(&version, dict + len - 4, 4);
  if (version != 2u && version != 3u) throw TantivyError(TantivyError::Unsupported, "sstable: version " + std::to_string(version) + " (expected 2 or 3)");
  if (index_offset > len - 20) throw TantivyError(TantivyError::DataCorruption, "sstable: index offset out of range");
  std::vector<SSTableEntry> out;
  out.reserve((size_t)std::min<uint64_t>(num_terms, 1u << 20));
  std::string key;
  size_t at = 0;
  const size_t end = (size_t)index_offset;
  for (;;) {
    if (at == end) break;                                   // (out of data: BlockReader::read_block's `0 =>` arm)
    if (end - at < 4) throw TantivyError(TantivyError::DataCorruption, "sstable: failed to read block_len");
    uint32_t block_len;
    std::memcpy(&block_len, dict + at, 4);
    at += 4;
    if (block_len <= 1) break;                              // the empty block that ends the stream
    const uint8_t compress = dict[at++];
    const size_t body = block_len - 1;
    if (end - at < body) throw TantivyError(TantivyError::DataCorruption, "sstable: failed to read block content");
    if (compress == 1) throw TantivyError(TantivyError::Unsupported, "sstable: zstd-compressed block");
    const uint8_t* b = dict + at;
    at += body;
    size_t pos = 0;
    std::vector<TermInfo> infos;
    if (with_term_infos) {
      const uint64_t n = read_vint(b, body, &pos);
      if (n > body) throw TantivyError(TantivyError::DataCorruption, "sstable: more values than the block has bytes");
      uint64_t postings = read_vint(b, body, &pos), positions = read_vint(b, body, &pos);
      infos.reserve((size_t)n);
      for (uint64_t i = 0; i < n; ++i) {
        TermInfo ti;
        ti.doc_freq = (uint32_t)read_vint(b, body, &pos);
        const uint64_t pl = read_vint(b, body, &pos), ql = read_vint(b, body, &pos);
        ti.postings_start = postings; ti.postings_end = postings + pl;
        ti.positions_start = positions; ti.positions_end = positions + ql;
        postings += pl; positions += ql;
        infos.push_back(ti);
      }
    }
    size_t idx = 0;
    while (pos < body) {
      size_t keep, add;
      const uint8_t ka = b[pos++];
      if (ka == 1u) { keep = (size_t)read_sstable_vint(b, body, &pos); add = (size_t)read_sstable_vint(b, body, &pos); }
      else { keep = ka & 15u; add = ka >> 4; }
      if (keep > key.size() || add > body - pos) throw TantivyError(TantivyError::DataCorruption, "sstable: bad key delta");
      key.resize(keep);
      key.append(reinterpret_cast<const char*>(b + pos), add);
      pos += add;
      SSTableEntry e;
      e.key = key;
      if (with_term_infos) {
        if (idx >= infos.size()) throw TantivyError(TantivyError::DataCorruption, "sstable: more keys than values in a block");
        e.info = infos[idx];
      }
      ++idx;
      if (!out.empty() && !(out.back().key < e.key)) throw TantivyError(TantivyError::DataCorruption, "sstable: keys are not strictly increasing");
      out.push_back(std::move(e));
    }
    if (with_term_infos && idx != infos.size()) throw TantivyError(TantivyError::DataCorruption, "sstable: more values than keys in a block");
  }
  if (out.size() != num_terms) throw TantivyError(TantivyError::DataCorruption, "sstable: " + std::to_string(out.size()) + " keys read, footer says " + std::to_string(num_terms));
  return out;
}

// What the reference writes for one field with the SSTable dictionary (test side and host-mirror files): sstable::Writer with
// TermInfoValueWriter, blocks flushed when they pass `block_len` bytes (sstable/src/lib.rs Writer::insert / finish,
// delta.rs:55-104), a single-block table keeps no index (store_offset 0: "SingleBlockSStable" in the README); tables of
// several blocks would need the block index (an FST map, crate tantivy-fst) and are not written here.
inline std::vector<uint8_t> write_single_block_sstable(const std::vector<SSTableEntry>& entries, bool with_term_infos = true) {
  auto vint = [](std::vector<uint8_t>& o, uint64_t v) {  // common::VInt: stop bit on the last byte
    for (;;) { const uint8_t b = (uint8_t)(v & 127u); v >>= 7; if (v == 0) { o.push_back(b | 128u); return; } o.push_back(b); }
  };
  auto svint = [](std::vector<uint8_t>& o, uint64_t v) {  // sstable vint: continue bit
    for (;;) { const uint8_t b = (uint8_t)(v & 127u); v >>= 7; if (v == 0) { o.push_back(b); return; } o.push_back(b | 128u); }
  };
  std::vector<uint8_t> block;
  if (with_term_infos) {
    vint(block, entries.size());
    if (!entries.empty()) {
      vint(block, entries[0].info.postings_start);
      vint(block, entries[0].info.positions_start);
      for (auto& e : entries) { vint(block, e.info.doc_freq); vint(block, e.info.postings_end - e.info.postings_start); vint(block, e.info.positions_end - e.info.positions_start); }
    }
  }
  std::string prev;
  for (auto& e : entries) {
    size_t keep = 0;
    while (keep < prev.size() && keep < e.key.size() && prev[keep] == e.key[keep]) ++keep;
    const size_t add = e.key.size() - keep;
    if (keep < 16 && add < 16) block.push_back((uint8_t)((add << 4) | keep));
    else { block.push_back(1u); svint(block, keep); svint(block, add); }
    block.insert(block.end(), e.key.begin() + (long)keep, e.key.end());
    prev = e.key;
  }
  std::vector<uint8_t> out;
  auto u32le = [&](uint32_t v) { const uint8_t* p = reinterpret_cast<const uint8_t*>(&v); out.insert(out.end(), p, p + 4); };
  auto u64le = [&](uint64_t v) { const uint8_t* p = reinterpret_cast<const uint8_t*>(&v); out.insert(out.end(), p, p + 8); };
  if (!entries.empty()) {
    u32le((uint32_t)block.size() + 1u);
    out.push_back(0u);  // not compressed
    out.insert(out.end(), block.begin(), block.end());
  }
  u32le(0u);            // no more block
  const uint64_t index_offset = out.size();
  u64le(0u);            // store_offset 0: single block, no index
  u64le(index_offset);
  u64le(entries.size());
  u32le(3u);
  return out;
}

// A field's `.term` sub-file, either kind: the trailing u32 says which (src/termdict/mod.rs:51-90).  SSTable dictionaries are read
// completely (term -> TermInfo); of an FST dictionary only the TermInfoStore is (term ordinal -> TermInfo), see above.
inline uint32_t term_dictionary_type(const uint8_t* sub, size_t len) {
  if (len < 4) throw TantivyError(TantivyError::DataCorruption, "term dictionary too short");
  uint32_t t;
  std::memcpy(&t, sub + len - 4, 4);
  if (t != 1u && t != 2u) throw TantivyError(TantivyError::DataCorruption, "invalid value for DictionaryType");
  return t;
}
inline std::vector<SSTableEntry> open_sstable_term_dictionary(const uint8_t* sub, size_t len) {
  if (term_dictionary_type(sub, len) != 2u) throw TantivyError(TantivyError::Unsupported, "term dictionary is not the SSTable kind");
  return read_sstable(sub, len - 4, true);
}
// An FST dictionary opened completely: every (term, TermInfo) in term order.  The consistency check of the Fst comment above runs
// here: keys strictly ascending, ordinals 0, 1, 2, ..., as many as both the FST's footer and the TermInfoStore say.
inline std::vector<SSTableEntry> open_fst_term_dictionary(const uint8_t* sub, size_t len) {
  const TermDictionaryParts parts = open_term_dictionary(sub, len);
  const Fst fst(parts.fst.data(), parts.fst.size());
  if (fst.len() != parts.store.num_terms()) throw TantivyError(TantivyError::DataCorruption, "term dictionary: the FST and the TermInfoStore disagree on the number of terms");
  std::vector<SSTableEntry> out;
  out.reserve((size_t)std::min<uint64_t>(fst.len(), 1u << 20));
  fst.for_each([&](const std::string& key, uint64_t ord) {
    if (ord != out.size()) throw TantivyError(TantivyError::DataCorruption, "fst: term ordinals are not 0, 1, 2, ... in key order (format misread)");
    if (!out.empty() && !(out.back().key < key)) throw TantivyError(TantivyError::DataCorruption, "fst: keys are not strictly ascending (format misread)");
    out.push_back(SSTableEntry{key, parts.store.get(ord)});
  });
  if (out.size() != fst.len()) throw TantivyError(TantivyError::DataCorruption, "fst: " + std::to_string(out.size()) + " keys found, footer says " + std::to_string(fst.len()));
  return out;
}

// ---- meta.json (src/index/index_meta.rs: IndexMeta { index_settings, segments, schema, opstamp }) ---------------------
// A small JSON reader, enough for the meta file the reference writes.
struct Json {
  enum Type { Null, Bool, Number, String, Array, Object } type = Null;
  bool b = false;
  double num = 0;
  std::string str;
  std::vector<Json> arr;
  std::vector<std::pair<std::string, Json>> obj;
  const Json* get(const std::string& key) const {
    for (auto& kv : obj) if (kv.first == key) return &kv.second;
    return nullptr;
  }
};
namespace detail {
struct JsonParser {
  const std::string& s;
  size_t i = 0;
  [[noreturn]] void bad(const char* what) const { throw TantivyError(TantivyError::DataCorruption, std::string("meta.json: ") + what); }
  void ws() { while (i < s.size() && (s[i] == ' ' || s[i] == '\n' || s[i] == '\t' || s[i] == '\r')) ++i; }
  Json value() {
    ws();
    if (i >= s.size()) bad("unexpected end");
    Json v;
    const char c = s[i];
    if (c == '{') {
      v.type = Json::Object; ++i; ws();
      if (i < s.size() && s[i] == '}') { ++i; return v; }
      for (;;) {
        ws();
        Json k = value();
        if (k.type != Json::String) bad("object key is not a string");
        ws();
        if (i >= s.size() || s[i] != ':') bad("':' expected");
        ++i;
        v.obj.emplace_back(k.str, value());
        ws();
        if (i < s.size() && s[i] == ',') { ++i; continue; }
        if (i < s.size() && s[i] == '}') { ++i; return v; }
        bad("',' or '}' expected");
      }
    }
    if (c == '[') {
      v.type = Json::Array; ++i; ws();
      if (i < s.size() && s[i] == ']') { ++i; return v; }
      for (;;) {
        v.arr.push_back(value());
        ws();
        if (i < s.size() && s[i] == ',') { ++i; continue; }
        if (i < s.size() && s[i] == ']') { ++i; return v; }
        bad("',' or ']' expected");
      }
    }
    if (c == '"') {
      v.type = Json::String; ++i;
      while (i < s.size() && s[i] != '"') {
        if (s[i] == '\\' && i + 1 < s.size()) {
          const char e = s[i + 1];
          if (e == 'n') v.str.push_back('\n'); else if (e == 't') v.str.push_back('\t');
          else if (e == 'u' && i + 5 < s.size()) { v.str.push_back((char)std::stoi(s.substr(i + 2, 4), nullptr, 16)); i += 4; }
          else v.str.push_back(e);
          i += 2;
        } else v.str.push_back(s[i++]);
      }
      if (i >= s.size()) bad("unterminated string");
      ++i;
      return v;
    }
    if (s.compare(i, 4, "true") == 0) { v.type = Json::Bool; v.b = true; i += 4; return v; }
    if (s.compare(i, 5, "false") == 0) { v.type = Json::Bool; i += 5; return v; }
    if (s.compare(i, 4, "null") == 0) { i += 4; return v; }
    size_t j = i;
    while (j < s.size() && (std::isdigit((unsigned char)s[j]) || s[j] == '-' || s[j] == '+' || s[j] == '.' || s[j] == 'e' || s[j] == 'E')) ++j;
    if (j == i) bad("unexpected character");
    v.type = Json::Number;
    v.num = std::stod(s.substr(i, j - i));
    i = j;
    return v;
  }
};
}  // namespace detail
inline Json parse_json(const std::string& text) {
  detail::JsonParser p{text};
  Json v = p.value();
  p.ws();
  if (p.i != text.size()) p.bad("trailing characters");
  return v;
}

// `.del` (SegmentComponent::Delete, named <uuid>.<delete opstamp>.del, index_meta.rs:134-146): BitSet::serialize = u32 max_value LE ‖
// ceil(max_value / 64) little-endian u64 words, bit (d & 63) of word d >> 6 set = doc d alive (common/src/bitset.rs:36-47,217-224;
// ReadOnlyBitSet::open / contains, :362-367,404-409; written by write_alive_bitset, src/fastfield/alive_bitset.rs:12-15, read by
// SegmentReader::open, src/index/segment_reader.rs:177) ‖ the managed-directory footer.  Returns the words as bytes: exactly what
// tq_segment_register takes as alive_bitset.
inline std::vector<uint8_t> read_alive_bitset(const uint8_t* file, size_t len, uint32_t max_doc, uint32_t* num_alive = nullptr) {
  const Footer f = read_footer(file, len);
  if (f.body_len < 4) throw TantivyError(TantivyError::DataCorruption, ".del: too short for the max_value header");
  uint32_t max_value;
  std::memcpy(&max_value, file, 4);
  if (max_value != max_doc) throw TantivyError(TantivyError::DataCorruption, ".del: max_value differs from the segment's max_doc");
  const size_t n_bytes = ((size_t)max_value + 63) / 64 * 8;
  if (f.body_len - 4 != n_bytes) throw TantivyError(TantivyError::DataCorruption, ".del: bitset length does not match max_value");
  std::vector<uint8_t> words(file + 4, file + 4 + n_bytes);
  if (num_alive) {
    uint32_t n = 0;
    for (uint32_t d = 0; d < max_value; ++d) n += (words[d >> 3] >> (d & 7u)) & 1u;  // (ReadOnlyBitSet::iter stops at max_value)
    *num_alive = n;
  }
  return words;
}
// BitSet::serialize + the footer FooterProxy::terminate_ref appends (footer.rs:44-51): what the reference writes for `alive` (test side)
inline std::vector<uint8_t> write_alive_bitset(const std::vector<uint8_t>& alive_words, uint32_t max_doc, uint32_t index_format_version = 7) {
  std::vector<uint8_t> out(4);
  std::memcpy(out.data(), &max_doc, 4);
  const size_t n_bytes = ((size_t)max_doc + 63) / 64 * 8;
  for (size_t i = 0; i < n_bytes; ++i) out.push_back(i < alive_words.size() ? alive_words[i] : 0);
  const std::string json = "{\"version\":{\"major\":0,\"minor\":26,\"patch\":0,\"index_format_version\":" + std::to_string(index_format_version) +
                           "},\"crc\":" + std::to_string(crc32(out.data(), out.size())) + "}";
  const uint32_t json_len = (uint32_t)json.size(), magic = 1337u;
  out.insert(out.end(), json.begin(), json.end());
  const uint8_t* p = reinterpret_cast<const uint8_t*>(&json_len);
  out.insert(out.end(), p, p + 4);
  p = reinterpret_cast<const uint8_t*>(&magic);
  out.insert(out.end(), p, p + 4);
  return out;
}

struct SegmentMeta {  // index_meta.rs: InnerSegmentMeta { segment_id, max_doc, deletes: Option<DeleteMeta{num_deleted_docs, opstamp}> }
  std::string segment_id;  // with dashes, as written
  uint32_t max_doc = 0;
  bool has_deletes = false;
  uint32_t num_deleted_docs = 0;
  uint64_t delete_opstamp = 0;
  std::string file_stem() const {  // SegmentId::uuid_string(): the uuid without dashes (index/segment_id.rs)
    std::string out;
    for (char ch : segment_id) if (ch != '-') out.push_back(ch);
    return out;
  }
};
struct IndexMeta {
  std::vector<SegmentMeta> segments;
  Schema schema;
  uint64_t opstamp = 0;
};

inline IndexMeta read_meta(const std::string& meta_json) {
  const Json root = parse_json(meta_json);
  if (root.type != Json::Object) throw TantivyError(TantivyError::DataCorruption, "meta.json: not an object");
  IndexMeta meta;
  if (const Json* o = root.get("opstamp")) meta.opstamp = (uint64_t)o->num;
  const Json* segs = root.get("segments");
  const Json* schema = root.get("schema");
  if (!segs || segs->type != Json::Array || !schema || schema->type != Json::Array)
    throw TantivyError(TantivyError::DataCorruption, "meta.json: segments / schema missing");
  for (const Json& sj : segs->arr) {
    SegmentMeta sm;
    const Json* id = sj.get("segment_id");
    const Json* md = sj.get("max_doc");
    if (!id || id->type != Json::String || !md || md->type != Json::Number) throw TantivyError(TantivyError::DataCorruption, "meta.json: bad segment entry");
    sm.segment_id = id->str;
    sm.max_doc = (uint32_t)md->num;
    const Json* del = sj.get("deletes");
    if (del && del->type == Json::Object) {
      sm.has_deletes = true;
      if (const Json* n = del->get("num_deleted_docs")) sm.num_deleted_docs = (uint32_t)n->num;
      if (const Json* o = del->get("opstamp")) sm.delete_opstamp = (uint64_t)o->num;
    }
    meta.segments.push_back(sm);
  }
  SchemaBuilder sb;
  for (const Json& fj : schema->arr) {
    const Json* name = fj.get("name");
    const Json* type = fj.get("type");
    if (!name || name->type != Json::String || !type || type->type != Json::String) throw TantivyError(TantivyError::DataCorruption, "meta.json: bad field entry");
    const Json* options = fj.get("options");
    const Json* indexing = (type->str == "text" && options) ? options->get("indexing") : nullptr;
    if (indexing && indexing->type == Json::Object) {  // schema/text_options.rs: TextFieldIndexing { record, fieldnorms, tokenizer }
      TextFieldIndexing ti;
      if (const Json* r = indexing->get("record")) {
        if (r->str == "basic") ti.record = IndexRecordOption::Basic;
        else if (r->str == "freq") ti.record = IndexRecordOption::WithFreqs;
        else if (r->str == "position") ti.record = IndexRecordOption::WithFreqsAndPositions;
        else throw TantivyError(TantivyError::DataCorruption, "meta.json: unknown record option " + r->str);
      }
      if (const Json* f = indexing->get("fieldnorms")) ti.fieldnorms = f->b;
      if (const Json* t = indexing->get("tokenizer")) ti.tokenizer = t->str;
      sb.add_text_field(name->str, TextOptions{ti});
    } else {
      sb.add_other_field(name->str);
    }
  }
  meta.schema = sb.build();
  return meta;
}

// Index::open_in_dir for this path: meta.json + every segment's `.idx` / `.fieldnorm` (read through `read_file(name)`),
// one SegmentData per segment in meta order.  A `.term` file, when there is one, fills FieldSegmentData::term_dict (both kinds of
// dictionary, see above); without it the caller fills it.  A segment with deletes brings its alive bitset from
// `<uuid>.<delete opstamp>.del` (SegmentReader::open, src/index/segment_reader.rs:170-181).
inline Index open_index(const std::string& meta_json, const std::function<std::vector<uint8_t>(const std::string&)>& read_file) {
  const IndexMeta meta = read_meta(meta_json);
  std::vector<std::shared_ptr<const SegmentData>> segments;
  for (const SegmentMeta& sm : meta.segments) {
    auto seg = std::make_shared<SegmentData>();
    seg->max_doc = sm.max_doc;
    if (sm.has_deletes) {
      const std::vector<uint8_t> del = read_file(sm.file_stem() + "." + std::to_string(sm.delete_opstamp) + ".del");
      uint32_t n_alive = 0;
      seg->alive = read_alive_bitset(del.data(), del.size(), sm.max_doc, &n_alive);
      seg->num_deleted = sm.max_doc - n_alive;
      if (sm.max_doc - n_alive != sm.num_deleted_docs)
        throw TantivyError(TantivyError::DataCorruption, "segment " + sm.segment_id + ": .del holds " + std::to_string(sm.max_doc - n_alive) +
                                                             " deleted docs, meta.json says " + std::to_string(sm.num_deleted_docs));
    }
    seg->fields.resize(meta.schema.num_fields());
    const std::vector<uint8_t> idx = read_file(sm.file_stem() + ".idx");
    const std::vector<uint8_t> fn = read_file(sm.file_stem() + ".fieldnorm");
    for (uint32_t f = 0; f < meta.schema.num_fields(); ++f) {
      const FieldEntry& fe = meta.schema.get_field_entry(Field{f});
      if (!fe.options.indexing) continue;
      load_field(*seg, Field{f}, fe.options.indexing->record, idx, fe.options.indexing->fieldnorms ? &fn : nullptr);
    }
    // `.term`: either kind of dictionary is read completely (term -> TermInfo)
    std::vector<uint8_t> term_file;
    try { term_file = read_file(sm.file_stem() + ".term"); } catch (const TantivyError&) { term_file.clear(); }
    if (!term_file.empty()) {
      const Footer tf = read_footer(term_file.data(), term_file.size());
      for (auto& part : open_composite(term_file.data(), tf.body_len)) {
        const uint32_t f = part.first.first;
        if (f >= seg->fields.size() || !seg->fields[f].indexed || part.second.len < 4) continue;
        const uint8_t* sub = term_file.data() + part.second.offset;
        const bool sstable = term_dictionary_type(sub, part.second.len) == 2u;
        for (auto& e : sstable ? open_sstable_term_dictionary(sub, part.second.len) : open_fst_term_dictionary(sub, part.second.len))
          seg->fields[f].term_dict[e.key] = e.info;
      }
    }
    segments.push_back(seg);
  }
  return Index::from_segments(meta.schema, std::move(segments));
}

// Index::open_in_dir (src/index/index.rs): meta.json and the segment files of a directory the reference wrote.
inline Index open_index_in_dir(const std::string& dir) {
  auto read = [&](const std::string& name) {
    std::ifstream f(dir + "/" + name, std::ios::binary);
    if (!f) throw TantivyError(TantivyError::SystemError, "cannot open " + dir + "/" + name);
    return std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  };
  const std::vector<uint8_t> meta = read("meta.json");
  return open_index(std::string(meta.begin(), meta.end()), read);
}

}  // namespace files
}  // namespace tantivy_b200
