// Test harness for k_tile's running threshold (tests/test_tile_theta_refresh.py): runs tile_push, tile_theta_refresh and
// k_theta_samples (the histogram's base word) from tq_tile.cuh on inputs the test writes, so that each can be compared with a
// plain model of DESIGN §3.1 at the counts, bases and k that an end-to-end run reaches only by chance (fine counts trailing the coarse ones, suffixes equal to k at a bucket edge,
// more than kTileRefreshCap triggers in one tile).  Built as its own library (libtile_theta_harness.so beside the product library);
// the product's C ABI does not change.  Every pointer is a device pointer; each launcher waits for its kernel.
#include <cstddef>

#include "tq_tile.cuh"

using namespace tq;

namespace {

// A CTA's TileCtl between two guard regions, so that a store outside it shows up in the guard words.
constexpr uint32_t kGuardWords = 32;
struct GuardedCtl {
  uint32_t g0[kGuardWords];
  TileCtl C;
  uint32_t g1[kGuardWords];
};
constexpr uint32_t kCtlWords = sizeof(GuardedCtl) / 4u;
static_assert(sizeof(GuardedCtl) % 4u == 0u, "GuardedCtl is copied out word by word");

__host__ __device__ constexpr uint32_t guard_pattern(uint32_t w) { return 0xC7A5E000u ^ (w * 0x9E3779B9u); }

BatchParams harness_params(const DQuery* queries, QState* qstate, Cand* cands) {
  BatchParams P{};
  P.queries = queries;
  P.qstate = qstate;
  P.cands = cands;
  return P;
}

// one warp per query
__global__ void k_refresh_harness(const BatchParams P, const TileParams TP, uint32_t nq, uint32_t* __restrict__ raised) {
  const uint32_t lane = threadIdx.x & 31u, q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (q >= nq) return;
  const bool r = tile_theta_refresh(P, TP, q, lane);
  if (lane == 0) raised[q] = r ? 1u : 0u;
}

// one kTileThreads CTA: pushes[i] = (query, score bits, doc, th_key), thread t takes pushes t, t + kTileThreads, ...  The whole
// GuardedCtl (every word set to guard_pattern first, nref = 0) is copied to ctl_out afterwards.
__global__ void __launch_bounds__(kTileThreads) k_push_harness(const BatchParams P, const TileParams TP, const uint4* __restrict__ pushes,
                                                             uint32_t n, const uint8_t* __restrict__ alive, uint32_t segment_ord,
                                                             uint32_t* __restrict__ ctl_out) {
  __shared__ GuardedCtl S;
  uint32_t* w = reinterpret_cast<uint32_t*>(&S);
  for (uint32_t i = threadIdx.x; i < kCtlWords; i += blockDim.x) w[i] = guard_pattern(i);
  __syncthreads();
  if (threadIdx.x == 0) S.C.nref = 0u;
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const uint4 p = pushes[i];
    tile_push(P, TP, S.C, p.x, __uint_as_float(p.y), p.z, segment_ord, p.w, alive);
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < kCtlWords; i += blockDim.x) ctl_out[i] = w[i];
}

int finish() {
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  return (int)e;
}

}  // namespace

extern "C" {

// [words of the copied-out GuardedCtl, word of nref, word of ref[0], kTileRefreshCap, guard words at each end, its pattern's seed
// check (guard_pattern(0)), kThHistWords]
int tq_theta_harness_layout(uint32_t* out) {
  out[0] = kCtlWords;
  out[1] = (uint32_t)((offsetof(GuardedCtl, C) + offsetof(TileCtl, nref)) / 4u);
  out[2] = (uint32_t)((offsetof(GuardedCtl, C) + offsetof(TileCtl, ref)) / 4u);
  out[3] = kTileRefreshCap;
  out[4] = kGuardWords;
  out[5] = guard_pattern(0);
  out[6] = kThHistWords;
  return 0;
}

// hist: [nq][kThHistWords] (fine counts, coarse counts, base word); queries[q].k; qstate[q].theta = the initial threshold, and
// the refreshed one afterwards; raised[q] = what tile_theta_refresh returned.
int tq_theta_harness_refresh(uint32_t* hist, const DQuery* queries, QState* qstate, uint32_t nq, uint32_t* raised) {
  TileParams TP{};
  TP.th_hist = hist;
  const BatchParams P = harness_params(queries, qstate, nullptr);
  if (nq) k_refresh_harness<<<(nq + kTileWarps - 1u) / kTileWarps, kTileThreads>>>(P, TP, nq, raised);
  return finish();
}

// One CTA's tile_push calls on pushes [n] (uint4: query, f32 score bits, doc, th_key) against the queries' DQuery (k, cand_base,
// cand_cap), QState (cand_count carries over from launch to launch), candidate regions and histograms; alive may be null.
// ctl_out receives the GuardedCtl's words (tq_theta_harness_layout).
int tq_theta_harness_push(const uint4* pushes, uint32_t n, const uint8_t* alive, uint32_t segment_ord, const DQuery* queries,
                          QState* qstate, Cand* cands, uint32_t* hist, uint32_t* ctl_out) {
  TileParams TP{};
  TP.th_hist = hist;
  const BatchParams P = harness_params(queries, qstate, cands);
  k_push_harness<<<1, kTileThreads>>>(P, TP, pushes, n, alive, segment_ord, ctl_out);
  return finish();
}

// k_theta_samples as the sample launch leaves it: samples [nq][sample_cap] score keys, sample_count [nq] (may exceed the cap),
// queries[q].k, qstate[q].theta (the threshold before, raised to the k-th sample); it writes the base word of hist's query regions.
int tq_theta_harness_samples(const uint32_t* samples, const uint32_t* sample_count, uint32_t sample_cap, const DQuery* queries,
                             QState* qstate, uint32_t* hist, uint32_t nq) {
  const BatchParams P = harness_params(queries, qstate, nullptr);
  if (nq) k_theta_samples<<<nq, kThreads>>>(P, samples, sample_count, sample_cap, hist);
  return finish();
}

}  // extern "C"
