// searcher.search(&query, &(Count, TopDocs::with_limit(k))) through the host mirror (tantivy_b200/host/tantivy_host.hpp): the
// tuple collector of collector/mod.rs:322-365 in one device batch.  Each half must equal what its collector alone returns.
#include <cstdio>
#include <functional>
#include <string>

#include "../../tantivy_b200/host/tantivy_host.hpp"

using namespace tantivy_b200;

static int g_failed = 0;
#define CHECK(cond)                                                                  \
  do {                                                                               \
    if (!(cond)) {                                                                   \
      std::printf("    CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #cond);        \
      ++g_failed;                                                                    \
    }                                                                                \
  } while (0)

static Document doc(Field f, const std::string& text) {
  Document d;
  d.add_text(f, text);
  return d;
}

// boolean_query/mod.rs:27-44 (aux_test_helper): docs "a b c", "a c", "b c", "a b c d", "d"
static Index index_boolean_aux() {
  SchemaBuilder sb;
  Field text = sb.add_text_field("text", TEXT);
  Index index = Index::create_in_ram(sb.build());
  IndexWriter w = index.writer_for_tests();
  for (const char* t : {"a b c", "a c", "b c", "a b c d", "d"}) w.add_document(doc(text, t));
  w.commit();
  return index;
}

// three commits (three segments), deletes in the first two, multi-block lists with tf > 1
static Index index_multi_segment() {
  SchemaBuilder sb;
  Field body = sb.add_text_field("body", TEXT);
  Index index = Index::create_in_ram(sb.build());
  IndexWriter w = index.writer_for_tests();
  uint32_t x = 777;
  auto next = [&]() { x = x * 1664525u + 1013904223u; return x >> 8; };
  for (int seg = 0; seg < 3; ++seg) {
    for (int d = 0; d < 900 + 131 * seg; ++d) {
      std::string t = "w" + std::to_string(next() % 7);
      const int len = 1 + (int)(next() % 30);
      for (int i = 0; i < len; ++i) t += " w" + std::to_string(next() % (4 + 13 * (i % 3)));
      if (next() % 5 == 0) t += " rare";
      w.add_document(doc(body, t));
    }
    if (seg == 1) w.delete_term(Term::from_field_text(body, "rare"));
    w.commit();
  }
  return index;
}

static void same_as_the_two_collectors(const Searcher& s, const Query& q, const TopDocs& top) {
  const auto both = s.search(q, std::make_pair(Count{}, top));
  CHECK(both.first == s.search(q, Count{}));
  CHECK(both.second == s.search(q, top));
}

static void test_count_and_top_docs_on_the_aux_index() {
  Index index = index_boolean_aux();
  Field text = *index.schema().get_field("text");
  Searcher searcher = index.reader().searcher();
  QueryParser parser = QueryParser::for_index(index, {text});
  const std::pair<const char*, size_t> cases[] = {{"+a", 3}, {"+a +b", 2}, {"a d", 4}, {"a b c d", 5}, {"+a +d", 1}, {"zzz", 0}, {"d", 2}};
  for (auto& c : cases) {
    QueryBox q = parser.parse_query(c.first);
    const auto both = searcher.search(*q, std::make_pair(Count{}, TopDocs::with_limit(2)));
    CHECK(both.first == c.second);
    CHECK(both.second.size() == std::min<size_t>(2, c.second));
    for (size_t k : {1, 2, 10}) same_as_the_two_collectors(searcher, *q, TopDocs::with_limit(k));
  }
  // a plan that matches nothing: (0, {})
  const auto none = searcher.search(BooleanQuery(), std::make_pair(Count{}, TopDocs::with_limit(5)));
  CHECK(none.first == 0 && none.second.empty());
}

static void test_count_and_top_docs_over_segments_with_deletes() {
  Index index = index_multi_segment();
  Field body = *index.schema().get_field("body");
  Searcher searcher = index.reader().searcher();
  const Term rare = Term::from_field_text(body, "rare");
  {
    TermQuery q(rare, IndexRecordOption::WithFreqs);
    const auto both = searcher.search(q, std::make_pair(Count{}, TopDocs::with_limit(10)));
    CHECK(both.first == searcher.segment_reader(2).inverted_index(body).doc_freq(rare));  // segments 0 and 1 lost theirs
    CHECK(both.first < searcher.doc_freq(rare) && both.second.size() == 10);
    same_as_the_two_collectors(searcher, q, TopDocs::with_limit(1000));
  }
  std::vector<std::pair<Occur, QueryBox>> should, must;
  for (const char* t : {"w0", "w3", "w11", "rare"}) should.emplace_back(Occur::Should, std::make_unique<TermQuery>(Term::from_field_text(body, t), IndexRecordOption::WithFreqs));
  for (const char* t : {"w1", "w2"}) must.emplace_back(Occur::Must, std::make_unique<TermQuery>(Term::from_field_text(body, t), IndexRecordOption::WithFreqs));
  BooleanQuery u(std::move(should)), a(std::move(must));
  for (size_t k : {1, 10, 1000}) {
    same_as_the_two_collectors(searcher, u, TopDocs::with_limit(k));
    same_as_the_two_collectors(searcher, a, TopDocs::with_limit(k));
  }
  same_as_the_two_collectors(searcher, u, TopDocs::with_limit(100).and_offset(200));  // the count ignores the page
  const auto paged = searcher.search(u, std::make_pair(Count{}, TopDocs::with_limit(100).and_offset(200)));
  CHECK(paged.first > 300 && paged.second.size() == 100);
}

int main() {
  const std::pair<const char*, std::function<void()>> tests[] = {
      {"count_and_top_docs_on_the_aux_index", test_count_and_top_docs_on_the_aux_index},
      {"count_and_top_docs_over_segments_with_deletes", test_count_and_top_docs_over_segments_with_deletes}};
  int bad = 0;
  for (auto& t : tests) {
    const int before = g_failed;
    try {
      t.second();
    } catch (const std::exception& e) {
      std::printf("    exception: %s\n", e.what());
      ++g_failed;
    }
    std::printf("%s %s\n", g_failed == before ? "ok  " : "FAIL", t.first);
    bad += g_failed != before;
  }
  std::printf("%d test(s) failed\n", bad);
  return bad ? 1 : 0;
}
