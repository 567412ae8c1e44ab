// Several GPUs behind one handle (tq_multi_*), a client of the public C ABI of include/tantivy_b200.h; of the engine it only
// shares the last error and the filter-in-use check (tq_host.hpp).
//
// The reference fans a search out over segments inside one process (Executor::map, src/core/executor.rs:60-100;
// Searcher::search_with_executor, src/core/searcher.rs:220-237).  tq_multi is that shape for GPUs: one tq_ctx per device,
// every segment lives on one of them, a search runs the devices' shares concurrently (one host thread per device), exchanges
// the exact k-th best score keys between the phases (so that every device prunes like a single device holding everything),
// and merges the per-device rows on the host (merge_fruits / merge_top_k, sort_key_top_collector.rs:54-95).
#include <algorithm>
#include <condition_variable>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/tantivy_b200.h"
#include "tq_host.hpp"
#include "tq_layout.h"  // kTile

using namespace tq;
using namespace tq::host;

struct tq_multi {
  std::vector<tq_ctx*> ctxs;
  std::map<std::pair<uint32_t, uint32_t>, std::vector<int>> owner;  // (segment_ord, field) -> indices into ctxs (several: the segment is split by doc range)
  std::vector<uint64_t> load;                           // bytes registered per device
  struct Placement { uint32_t max_doc; bool split; std::vector<int> devices; };
  std::map<uint32_t, Placement> placed;  // segment_ord -> where its fields live: every field of an ordinal on the same devices
  std::mutex mu;
  std::string err;
};

namespace {

// An error of the handle: its own message (tq_multi_last_error) and the thread's (tq_last_error).
int refuse(tq_multi* m, int code, const std::string& msg) {
  m->err = msg;
  return fail(code, msg);
}

struct HostBarrier {
  std::mutex m;
  std::condition_variable cv;
  int n, waiting = 0;
  uint64_t gen = 0;
  explicit HostBarrier(int n_) : n(n_) {}
  template <class F> void arrive(F&& last) {  // `last` runs on exactly one thread while the others wait
    std::unique_lock<std::mutex> lk(m);
    const uint64_t g = gen;
    if (++waiting == n) { last(); waiting = 0; ++gen; cv.notify_all(); }
    else cv.wait(lk, [&] { return gen != g; });
  }
};
}  // namespace

extern "C" {

int tq_multi_create(const int* devices, int n_devices, tq_multi** out) {
  if (!devices || n_devices <= 0 || !out) return fail(TQ_ERR_INVALID_ARGUMENT, "devices");
  auto* m = new tq_multi();
  for (int i = 0; i < n_devices; ++i) {
    tq_ctx* c = nullptr;
    const int rc = tq_ctx_create(devices[i], &c);
    if (rc != TQ_OK) { for (auto* x : m->ctxs) tq_ctx_destroy(x); delete m; return rc; }
    m->ctxs.push_back(c);
  }
  m->load.assign(n_devices, 0);
  *out = m;
  return TQ_OK;
}

void tq_multi_destroy(tq_multi* m) {
  if (!m) return;
  for (auto* c : m->ctxs) tq_ctx_destroy(c);
  delete m;
}

const char* tq_multi_last_error(tq_multi* m) { return m ? m->err.c_str() : last_error().c_str(); }

int tq_multi_num_devices(tq_multi* m) { return m ? (int)m->ctxs.size() : 0; }

int tq_multi_segment_register(tq_multi* m, int device_index, uint32_t segment_ord, uint32_t field, uint32_t max_doc, int record_option,
                              const uint8_t* idx_body, size_t idx_len, const uint8_t* fieldnorm, size_t fieldnorm_len,
                              const uint8_t* alive_bitset, size_t alive_len) {
  if (!m) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(m->mu);
  if (device_index >= (int)m->ctxs.size()) { m->err = "device_index"; return TQ_ERR_INVALID_ARGUMENT; }
  // a query's clauses on one ordinal are scored on one device: a further field of an ordinal goes where its first one went
  auto pit = m->placed.find(segment_ord);
  if (pit != m->placed.end()) {
    const char* why = pit->second.split ? "the ordinal's other fields are split over the devices (tq_multi_segment_register_split)"
                    : pit->second.max_doc != max_doc ? "max_doc differs from the ordinal's other fields"
                    : device_index >= 0 && device_index != pit->second.devices[0] ? "device_index differs from the device of the ordinal's other fields"
                    : nullptr;
    if (why) return refuse(m, TQ_ERR_INVALID_ARGUMENT, why);
    device_index = pit->second.devices[0];
  } else if (device_index < 0) {  // least loaded device: segments shard naturally (SURVEY.md §8e)
    device_index = 0;
    for (size_t i = 1; i < m->load.size(); ++i) if (m->load[i] < m->load[device_index]) device_index = (int)i;
  }
  const int rc = tq_segment_register(m->ctxs[device_index], segment_ord, field, max_doc, record_option, idx_body, idx_len, fieldnorm, fieldnorm_len,
                                     alive_bitset, alive_len);
  if (rc != TQ_OK) { m->err = last_error(); return rc; }
  m->owner[{segment_ord, field}] = std::vector<int>{device_index};
  m->placed.emplace(segment_ord, tq_multi::Placement{max_doc, false, {device_index}});
  m->load[device_index] += idx_len + fieldnorm_len;
  return TQ_OK;
}

// One segment over ALL devices of the handle, device i evaluating the docs [i, i + 1) * ceil(max_doc / n / 1024) * 1024 (whole
// tiles of the tile engine): the intra-segment split of SURVEY.md §8(e) for an index of one (or few) huge segments.
int tq_multi_segment_register_split(tq_multi* m, uint32_t segment_ord, uint32_t field, uint32_t max_doc, int record_option,
                                    const uint8_t* idx_body, size_t idx_len, const uint8_t* fieldnorm, size_t fieldnorm_len,
                                    const uint8_t* alive_bitset, size_t alive_len) {
  if (!m) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(m->mu);
  auto pit = m->placed.find(segment_ord);
  if (pit != m->placed.end() && (!pit->second.split || pit->second.max_doc != max_doc))
    return refuse(m, TQ_ERR_INVALID_ARGUMENT, !pit->second.split ? "the ordinal's other fields are registered whole (tq_multi_segment_register)"
                                                                 : "max_doc differs from the ordinal's other fields");
  const uint32_t nd = (uint32_t)m->ctxs.size();
  const uint32_t per = (uint32_t)((((uint64_t)max_doc + nd - 1) / nd + kTile - 1) / kTile * kTile);
  std::vector<int> owners;
  for (uint32_t d = 0; d < nd; ++d) {
    const uint32_t lo = (uint32_t)std::min<uint64_t>((uint64_t)d * per, max_doc), hi = (uint32_t)std::min<uint64_t>((uint64_t)(d + 1) * per, max_doc);
    int rc = tq_segment_register(m->ctxs[d], segment_ord, field, max_doc, record_option, idx_body, idx_len, fieldnorm, fieldnorm_len, alive_bitset, alive_len);
    if (rc == TQ_OK) rc = tq_segment_set_doc_range(m->ctxs[d], segment_ord, field, lo, hi);
    if (rc != TQ_OK) {
      m->err = last_error();
      tq_segment_unregister(m->ctxs[d], segment_ord, field);
      for (int o : owners) tq_segment_unregister(m->ctxs[o], segment_ord, field);
      set_last_error(m->err);
      return rc;
    }
    owners.push_back((int)d);
    m->load[d] += idx_len + fieldnorm_len;
  }
  m->owner[{segment_ord, field}] = owners;
  m->placed.emplace(segment_ord, tq_multi::Placement{max_doc, true, owners});
  return TQ_OK;
}

int tq_multi_search_batch(tq_multi* m, const tq_query* queries, size_t nq, uint32_t out_stride, float* out_scores, uint32_t* out_segment_ord,
                          uint32_t* out_doc, uint32_t* out_count) {
  if (!m || (!queries && nq) || !out_scores || !out_segment_ord || !out_doc || !out_count) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  const int nd = (int)m->ctxs.size();
  uint32_t kmax = 1;
  for (size_t q = 0; q < nq; ++q) kmax = std::max(kmax, queries[q].k);
  // every device's share of every query: the (clause, segment) lists of the segments it owns
  std::vector<std::vector<tq_query>> dq(nd, std::vector<tq_query>(queries, queries + nq));
  std::vector<std::vector<tq_term_seg>> dts(nd);
  {
    std::lock_guard<std::mutex> g(m->mu);
    std::vector<std::vector<size_t>> first(nd, std::vector<size_t>(nq + 1, 0));
    for (size_t q = 0; q < nq; ++q) {
      for (int d = 0; d < nd; ++d) first[d][q] = dts[d].size();
      for (uint32_t i = 0; i < queries[q].n_term_segs; ++i) {
        const tq_term_seg& ts = queries[q].term_segs[i];
        auto it = m->owner.find({ts.segment_ord, ts.field});
        if (it == m->owner.end()) { m->err = "term_seg names a segment/field that is not registered"; return TQ_ERR_NOT_FOUND; }
        for (int d : it->second) dts[d].push_back(ts);
      }
    }
    for (int d = 0; d < nd; ++d) {
      first[d][nq] = dts[d].size();
      for (size_t q = 0; q < nq; ++q) {
        dq[d][q].term_segs = dts[d].data() + first[d][q];
        dq[d][q].n_term_segs = (uint32_t)(first[d][q + 1] - first[d][q]);
      }
    }
  }
  const size_t rows = std::max<size_t>(nq, 1) * kmax;
  std::vector<std::vector<float>> r_sc(nd, std::vector<float>(rows));
  std::vector<std::vector<uint32_t>> r_sg(nd, std::vector<uint32_t>(rows)), r_dc(nd, std::vector<uint32_t>(rows)), r_ct(nd, std::vector<uint32_t>(std::max<size_t>(nq, 1)));
  std::vector<std::vector<uint32_t>> keys(nd, std::vector<uint32_t>(rows));  // [device][query][kmax] best keys so far
  std::vector<long long> bound(std::max<size_t>(nq, 1), 0);                   // exact k-th best of the union, per query
  std::vector<int> rcs(nd, TQ_OK);
  std::vector<char> aborted(nd, 0);  // the worker stopped only because another device failed
  std::vector<std::string> errs(nd);
  HostBarrier bar(nd);
  bool abort_all = false;
  auto worker = [&](int d) {
    tq_batch* b = nullptr;
    uint32_t* d_keys = nullptr;
    long long* d_bound = nullptr;
    int rc = tq_batch_prepare(m->ctxs[d], dq[d].data(), nq, &b);
    if (rc == TQ_OK && (cudaMalloc(&d_keys, rows * 4) != cudaSuccess || cudaMalloc(&d_bound, std::max<size_t>(nq, 1) * 8) != cudaSuccess)) rc = fail(TQ_ERR_OOM, "exchange buffers");
    cudaStream_t stream = nullptr;
    if (rc == TQ_OK) rc = tq_batch_stream(b, reinterpret_cast<void**>(&stream));
    // Every worker reaches the first key exchange, a failed one with abort_all set, so that no worker waits at the barrier for
    // one that has stopped.  A worker whose prepare failed has no batch to ask for the phase count: it takes one round.
    const int phases = b ? tq_batch_phases(b) : 2;
    for (int p = 0; p < phases; ++p) {
      if (rc == TQ_OK) rc = tq_batch_run_phase(b, p);
      if (p + 1 == phases) break;
      if (rc == TQ_OK) rc = tq_batch_topkeys_export_dev(b, d_keys, kmax);
      if (rc == TQ_OK && (cudaMemcpyAsync(keys[d].data(), d_keys, rows * 4, cudaMemcpyDeviceToHost, stream) != cudaSuccess ||
                          cudaStreamSynchronize(stream) != cudaSuccess)) rc = fail(TQ_ERR_CUDA, "key export");
      if (rc != TQ_OK) { std::lock_guard<std::mutex> g(m->mu); abort_all = true; }
      bar.arrive([&] {  // one thread: the exact k-th best key of the union of all devices' keys
        std::vector<uint32_t> all((size_t)nd * kmax);
        for (size_t q = 0; q < nq; ++q) {
          for (int e = 0; e < nd; ++e) memcpy(all.data() + (size_t)e * kmax, keys[e].data() + q * kmax, (size_t)kmax * 4);
          const uint32_t k = queries[q].k;
          std::nth_element(all.begin(), all.begin() + (k - 1), all.end(), std::greater<uint32_t>());
          bound[q] = (long long)all[k - 1];
        }
      });
      if (abort_all) { if (rc == TQ_OK) { rc = TQ_ERR_CUDA; aborted[d] = 1; } break; }
      if (rc == TQ_OK && cudaMemcpyAsync(d_bound, bound.data(), nq * 8, cudaMemcpyHostToDevice, stream) != cudaSuccess) rc = fail(TQ_ERR_CUDA, "bound import");
      if (rc == TQ_OK && nq) rc = tq_batch_thresholds_import_dev(b, reinterpret_cast<const int64_t*>(d_bound));
    }
    if (rc == TQ_OK) rc = tq_batch_fetch(b, kmax, r_sc[d].data(), r_sg[d].data(), r_dc[d].data(), r_ct[d].data());
    if (rc != TQ_OK) errs[d] = last_error();
    rcs[d] = rc;
    if (b) tq_batch_destroy(b);
    cudaFree(d_keys);
    cudaFree(d_bound);
  };
  std::vector<std::thread> th;
  for (int d = 0; d < nd; ++d) th.emplace_back(worker, d);
  for (auto& t : th) t.join();
  // the error of a device whose own call failed, not of the devices that stopped for it
  for (int d = 0; d < nd; ++d)
    if (rcs[d] != TQ_OK && !aborted[d]) return refuse(m, rcs[d], errs[d]);
  for (int d = 0; d < nd; ++d)
    if (rcs[d] != TQ_OK) return refuse(m, rcs[d], "a device stopped the search without an error of its own");
  // merge_fruits: (score desc, segment_ord asc, doc asc), keep k (top_score_collector.rs:591-600)
  struct Row { float s; uint32_t g, d; };
  std::vector<Row> all;
  for (size_t q = 0; q < nq; ++q) {
    all.clear();
    for (int d = 0; d < nd; ++d) {
      const uint32_t n = std::min(r_ct[d][q], kmax);
      for (uint32_t i = 0; i < n; ++i) all.push_back(Row{r_sc[d][q * kmax + i], r_sg[d][q * kmax + i], r_dc[d][q * kmax + i]});
    }
    std::sort(all.begin(), all.end(), [](const Row& a, const Row& b) {
      if (a.s != b.s) return a.s > b.s;
      if (a.g != b.g) return a.g < b.g;
      return a.d < b.d;
    });
    const uint32_t n = (uint32_t)std::min<size_t>(all.size(), queries[q].k);
    out_count[q] = n;
    for (uint32_t i = 0; i < std::min(n, out_stride); ++i) {
      out_scores[q * out_stride + i] = all[i].s;
      out_segment_ord[q * out_stride + i] = all[i].g;
      out_doc[q * out_stride + i] = all[i].d;
    }
  }
  return TQ_OK;
}

int tq_multi_filter_register(tq_multi* m, uint32_t filter_id, uint32_t segment_ord, const uint8_t* bits, size_t len) {
  if (!m) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(m->mu);
  std::vector<int> devs;  // every device that holds a field of the ordinal
  for (auto it = m->owner.lower_bound({segment_ord, 0u}); it != m->owner.end() && it->first.first == segment_ord; ++it)
    devs.insert(devs.end(), it->second.begin(), it->second.end());
  std::sort(devs.begin(), devs.end());
  devs.erase(std::unique(devs.begin(), devs.end()), devs.end());
  if (devs.empty()) return refuse(m, TQ_ERR_NOT_FOUND, "no field of the segment ordinal is registered");
  for (tq_ctx* c : m->ctxs)  // all or nothing: refused if a prepared batch on any device names the filter
    if (filter_in_use(c, filter_id)) return refuse(m, TQ_ERR_INVALID_ARGUMENT, "a prepared batch still uses the filter");
  for (int d : devs) {
    const int rc = tq_filter_register(m->ctxs[d], filter_id, segment_ord, bits, len);
    if (rc != TQ_OK) { m->err = last_error(); return rc; }
  }
  return TQ_OK;
}

int tq_multi_filter_unregister(tq_multi* m, uint32_t filter_id) {
  if (!m) return fail(TQ_ERR_INVALID_ARGUMENT, "null");
  std::lock_guard<std::mutex> g(m->mu);
  for (tq_ctx* c : m->ctxs)
    if (filter_in_use(c, filter_id)) return refuse(m, TQ_ERR_INVALID_ARGUMENT, "a prepared batch still uses the filter");
  bool any = false;
  for (tq_ctx* c : m->ctxs) {
    const int rc = tq_filter_unregister(c, filter_id);
    if (rc == TQ_ERR_NOT_FOUND) continue;
    if (rc != TQ_OK) { m->err = last_error(); return rc; }
    any = true;
  }
  if (!any) return refuse(m, TQ_ERR_NOT_FOUND, "filter not registered");
  return TQ_OK;
}

}  // extern "C"
