// Host-only entry points of the C ABI: the BM25 scalars (bm25_host.hpp) and the field writer, which serialises posting lists in
// tantivy's format (segment_writer.hpp).  Neither touches the device.
#include <vector>

#include "../../include/tantivy_b200.h"
#include "bm25_host.hpp"
#include "segment_writer.hpp"
#include "tq_host.hpp"

using namespace tq;
using tq::host::fail;

extern "C" {

// ---- BM25 scalars --------------------------------------------------------------------------------------
float tq_bm25_idf(uint64_t doc_freq, uint64_t doc_count) { return bm25_idf(doc_freq, doc_count); }
float tq_bm25_weight(uint64_t doc_freq, uint64_t doc_count, float boost) { return bm25_weight(doc_freq, doc_count, boost); }
void tq_bm25_tf_cache(float avg_fieldnorm, float out[256]) { bm25_tf_cache(avg_fieldnorm, out); }
uint32_t tq_id_to_fieldnorm(uint8_t id) { return id_to_fieldnorm(id); }
uint8_t tq_fieldnorm_to_id(uint32_t fieldnorm) { return fieldnorm_to_id(fieldnorm); }

// ---- segment writer ----------------------------------------------------------------------------------
struct tq_field_writer {
  uint32_t max_doc = 0;
  std::vector<uint8_t> fieldnorm_ids;
  FieldPostingsWriter* w = nullptr;
};

int tq_field_writer_create(int record_option, uint64_t total_num_tokens, const uint8_t* fieldnorm_ids, uint32_t max_doc, tq_field_writer** out) {
  if (!out || record_option < 0 || record_option > 2) return fail(TQ_ERR_INVALID_ARGUMENT, "args");
  auto* fw = new tq_field_writer();
  fw->max_doc = max_doc;
  if (fieldnorm_ids) fw->fieldnorm_ids.assign(fieldnorm_ids, fieldnorm_ids + max_doc);
  fw->w = new FieldPostingsWriter(record_option, total_num_tokens, fieldnorm_ids ? fw->fieldnorm_ids.data() : nullptr, max_doc);
  *out = fw;
  return TQ_OK;
}
int tq_field_writer_add_term(tq_field_writer* fw, const uint32_t* docs, const uint32_t* tfs, uint32_t doc_freq, uint64_t* postings_start,
                             uint64_t* postings_end) {
  if (!fw || (!docs && doc_freq)) return fail(TQ_ERR_INVALID_ARGUMENT, "args");
  for (uint32_t i = 0; i < doc_freq; ++i) {
    if (i && docs[i] <= docs[i - 1]) return fail(TQ_ERR_INVALID_ARGUMENT, "docs must be strictly ascending");
    if (docs[i] >= TQ_TERMINATED || docs[i] >= fw->max_doc) return fail(TQ_ERR_INVALID_ARGUMENT, "doc id out of range (>= max_doc)");
    if (tfs && tfs[i] == 0) return fail(TQ_ERR_INVALID_ARGUMENT, "term frequency 0");
  }
  const TermInfoOut ti = fw->w->add_term(docs, tfs, doc_freq);
  if (postings_start) *postings_start = ti.postings_start;
  if (postings_end) *postings_end = ti.postings_end;
  return TQ_OK;
}
int tq_field_writer_body(tq_field_writer* fw, const uint8_t** body, size_t* len) {
  if (!fw || !body || !len) return fail(TQ_ERR_INVALID_ARGUMENT, "args");
  *body = fw->w->body().data();
  *len = fw->w->body().size();
  return TQ_OK;
}
void tq_field_writer_destroy(tq_field_writer* fw) {
  if (!fw) return;
  delete fw->w;
  delete fw;
}

}  // extern "C"
