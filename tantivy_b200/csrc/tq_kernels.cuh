// The sm_90a kernels of the query path.  One CTA (8 warps) per work unit; one warp per 128-doc
// posting block; exact per-CTA top-k buffers reduced per query by k_final.
//
//   k_build_tables  SkipReader::read_block_info/advance as ONE exclusive scan (src/postings/skip.rs:205-302)
//                   + decode_vint_block for the tail (src/postings/block_segment_postings.rs:56-76)
//   k_term          block_wand_single_scorer's result set (block_wand_union.rs:226-265), exhaustive form
//   k_and           block_wand_intersection's result set (block_wand_intersection.rs:19-179): leader =
//                   rarest list, secondaries probed through their block tables; score summed
//                   leader first, then secondaries by ascending doc_freq (:27,146-158)
//   k_or            BufferedUnionScorer's shape (union/buffered_union.rs:63-151): a doc-id window of
//                   score slots in shared memory, clauses accumulated in clause order
//   k_final         TopBySortKeyCollector::merge_fruits / merge_top_k (sort_key_top_collector.rs:54-95)
#pragma once
#include "tq_device.cuh"

namespace tq {

__device__ __forceinline__ uint32_t load_u32_unaligned(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// One CTA per posting list.  Fills last_doc / blk / tail arrays of its ListDesc.
__global__ void __launch_bounds__(kThreads) k_build_tables(const BuildJob* __restrict__ jobs, const ListDesc* __restrict__ init,
                                                           ListDesc* __restrict__ lists, uint32_t* __restrict__ status_out) {
  const BuildJob J = jobs[blockIdx.x];
  const ListDesc D = init[blockIdx.x];
  ListDesc& L = lists[J.list_id];
  if (threadIdx.x == 0) L = D;  // (list ids are recycled: the slot may hold an unregistered segment's table)
  // Every thread takes the table pointers from `init`, never from the slot thread 0 writes: with `lists` __restrict__ the
  // compiler may load the slot before that store is visible (even across a barrier), and a fresh slot holds null pointers.
  uint32_t* last_doc = const_cast<uint32_t*>(D.last_doc);
  uint2* blk = const_cast<uint2*>(D.blk);
  uint4* tab4 = const_cast<uint4*>(D.tab4);
  uint32_t* tail_docs = const_cast<uint32_t*>(D.tail_docs);
  uint32_t* tail_tfs = const_cast<uint32_t*>(D.tail_tfs);
  const uint32_t n_blocks = J.doc_freq / 128u, tail_n = J.doc_freq % 128u;
  __shared__ uint32_t s_hdr, s_skip_len, s_rec, s_status, s_carry;
  __shared__ uint32_t s_wsum[kWarps];
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  if (tid == 0) {
    const uint32_t ro = J.record_option & 0xFFu;
    uint32_t hdr = 0, skip_len = 0, rec = ro == 0 ? 5u : (ro == 1 ? 8u : 12u), status = 0;
    if (J.doc_freq >= 128u) {  // split_into_skips_and_postings (block_segment_postings.rs:78-88)
      uint64_t v = 0;
      uint32_t shift = 0;
      bool done = false;
      while (hdr < J.len && hdr < 10u) {
        const uint8_t b = J.bytes[hdr++];
        v |= (uint64_t)(b & 127u) << shift;
        shift += 7;
        if (b & 128u) { done = true; break; }
      }
      if (!done || v > (uint64_t)J.len - hdr) status = 1;
      skip_len = (uint32_t)v;
      // a field indexed with freqs can hold terms written without (block_segment_postings.rs:116-123)
      if (rec != 5u && skip_len < 8u * n_blocks) rec = 5u;
      if ((uint64_t)rec * n_blocks > skip_len) status = 1;
    }
    s_hdr = hdr; s_skip_len = skip_len; s_rec = rec; s_status = status; s_carry = 0;
  }
  __syncthreads();
  const uint32_t rec = s_rec;
  const uint8_t* skip = J.bytes + s_hdr;
  const uint8_t* blocks = skip + s_skip_len;
  const uint32_t avail = J.len - s_hdr - s_skip_len;
  if (s_status == 0) {
    for (uint32_t base = 0; base < n_blocks; base += kThreads) {
      const uint32_t i = base + tid;
      uint32_t size = 0, meta = 0, last = 0;
      if (i < n_blocks) {
        const uint8_t* r = skip + (size_t)i * rec;
        last = load_u32_unaligned(r);
        const uint32_t bw = r[4];
        const uint32_t db = bw & 31u, strict = (bw >> 6) & 1u;
        uint32_t tb = 0, bm_fn = 0, bm_tf = 0;
        if (rec == 8u) { tb = r[5]; bm_fn = r[6]; bm_tf = r[7]; }
        else if (rec == 12u) { tb = r[5]; bm_fn = r[10]; bm_tf = r[11]; }
        if (tb > 32u) { tb = 32u; s_status = 1; }
        size = 16u * (db + tb);
        meta = db | (strict << 6) | (tb << 8) | (bm_fn << 16) | (bm_tf << 24);
      }
      const uint32_t incl = warp_incl_scan(size, lane);
      if (lane == 31) s_wsum[warp] = incl;
      __syncthreads();
      uint32_t woff = 0;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) woff += (w < (int)warp) ? s_wsum[w] : 0u;
      const uint32_t excl = s_carry + woff + incl - size;
      if (i < n_blocks) {
        last_doc[i] = last;
        blk[i] = make_uint2(excl, meta);
        const uint32_t prev_last = i ? load_u32_unaligned(skip + (size_t)(i - 1) * rec) : 0xFFFFFFFFu;
        tab4[i] = make_uint4(last, excl, meta, prev_last);
      }
      __syncthreads();
      if (tid == kThreads - 1) s_carry = excl + size;
      __syncthreads();
    }
  }
  if (tid == 0) {
    uint32_t status = s_status;
    const uint32_t total = s_carry;
    blk[n_blocks] = make_uint2(total, 0u);
    if (total > avail) status = 1;
    if (tail_n && status == 0) {
      // decode_vint_block: plain deltas from last_doc_in_previous_block, tfs raw (serializer.rs:456-468)
      const uint8_t* p = blocks + total;
      uint32_t remaining = avail - total, pos = 0;
      uint32_t result = n_blocks ? load_u32_unaligned(skip + (size_t)(n_blocks - 1) * rec) : 0u;
      for (uint32_t i = 0; i < tail_n && status == 0; ++i) {
        uint32_t shift = 0;
        for (;;) {
          if (pos >= remaining) { status = 1; break; }
          const uint8_t b = p[pos++];
          result += (uint32_t)(b & 127u) << shift;
          if (b & 128u) break;
          shift += 7;
        }
        tail_docs[i] = result;
      }
      const bool read_freq = (rec != 5u) && pos < remaining && !(J.record_option & 0x100u);  // block_segment_postings.rs:66-75
      for (uint32_t i = 0; i < tail_n && status == 0; ++i) {
        uint32_t v = 1u;
        if (read_freq) {
          v = 0;
          uint32_t shift = 0;
          for (;;) {
            if (pos >= remaining) { status = 1; break; }
            const uint8_t b = p[pos++];
            v += (uint32_t)(b & 127u) << shift;
            if (b & 128u) break;
            shift += 7;
          }
        }
        tail_tfs[i] = v;
      }
      if (status == 0) {
        last_doc[n_blocks] = tail_docs[tail_n - 1];
        const uint32_t prev_last = n_blocks ? load_u32_unaligned(skip + (size_t)(n_blocks - 1) * rec) : 0xFFFFFFFFu;
        tab4[n_blocks] = make_uint4(tail_docs[tail_n - 1], total, 0xFFFFFFFFu, prev_last);
      }
    }
    L.has_freq = rec != 5u && !(J.record_option & 0x100u);  // SkipFreq: the tf bits stay in the block sizes, nobody reads them
    L.build_status = status;
    status_out[blockIdx.x] = status;
  }
  // 16-byte aligned copy of the bit-packed blocks (L.blocks was pre-set by the host to an arena region of
  // >= len + 64 bytes): posting lists start at arbitrary byte offsets inside the .idx body; the copy lets
  // every lane fetch its vectors with plain LDG.128.
  __syncthreads();
  if (s_status == 0 && s_carry <= avail) {
    const uint32_t total_words = s_carry / 4u + 16u;  // + 64 bytes of slack after the last block
    const uint32_t mis = (uint32_t)((uintptr_t)blocks & 3u);
    const uint32_t* src32 = reinterpret_cast<const uint32_t*>(blocks - mis);
    uint32_t* dst32 = reinterpret_cast<uint32_t*>(const_cast<uint8_t*>(D.blocks));
    const uint32_t sh = mis * 8u;
    for (uint32_t i = tid; i < total_words; i += kThreads) {
      const uint32_t w0 = src32[i], w1 = src32[i + 1];  // the segment body is padded by 256 bytes on the device
      dst32[i] = mis ? __funnelshift_r(w0, w1, sh) : w0;
    }
  }
}

// tf / (tf + norm[id]) for tf < kTfRows, one table per tf-norm cache of the batch; same IEEE operations and
// order as Bm25Weight::tf_factor (bm25.rs:170-175).
__global__ void k_build_tf_tables(const float* __restrict__ caches, float* __restrict__ tables, uint32_t n_caches) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_caches * kTfRows * 256u) return;
  const uint32_t c = i / (kTfRows * 256u), tf = (i >> 8) % kTfRows, id = i & 255u;
  const float t = __uint2float_rn(tf);
  tables[i] = __fdiv_rn(t, __fadd_rn(t, caches[c * 256u + id]));
}

// ---- K1 stand-alone: whole-list decode (parity tests, decode micro-benchmark) ------------------
__global__ void __launch_bounds__(kThreads) k_decode_list(const ListDesc* __restrict__ lists, uint32_t list_id,
                                                          uint32_t* __restrict__ out_docs, uint32_t* __restrict__ out_tfs) {
  const ListDesc L = lists[list_id];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t b = blockIdx.x * kWarps + warp;
  if (b >= L.n_total) return;
  uint32_t doc[4], tf[4];
  decode_block(L, b, lane, doc, tf);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t j = b * 128u + lane * 4u + i;
    if (j < L.doc_freq) { out_docs[j] = doc[i]; if (out_tfs) out_tfs[j] = tf[i]; }
  }
}

// Block-max score of every full block (SkipReader::block_max_score, skip.rs:175-184).
__global__ void k_block_max(const ListDesc* __restrict__ lists, uint32_t list_id, float weight, const float* __restrict__ cache,
                            uint32_t* __restrict__ out_last_doc, float* __restrict__ out_block_max) {
  const ListDesc L = lists[list_id];
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= L.n_blocks) return;
  const uint32_t meta = L.blk[b].y;
  const uint32_t code = meta >> 24;
  const uint32_t tf = code == 255u ? 0xFFFFFFFFu : code;
  out_last_doc[b] = L.last_doc[b];
  const float t = __uint2float_rn(tf);
  out_block_max[b] = __fmul_rn(weight, __fdiv_rn(t, __fadd_rn(t, __ldg(cache + ((meta >> 16) & 255u)))));
}

// ---- shared CTA scaffolding ------------------------------------------------------------------------
struct CtaTopK {
  unsigned long long keys[kCap];
  unsigned int count;
  unsigned long long theta;
  TopKScratch scratch;
};

// ---- single term ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) k_term(const BatchParams P, uint32_t unit_base) {
  __shared__ CtaTopK s_top;
  const Unit U = P.units[unit_base + blockIdx.x];
  const QSeg S = P.qsegs[U.qseg];
  const DQuery Q = P.queries[S.query];
  QState* qs = P.qstate + S.query;
  const QList ql = P.qlists[S.lists_base];
  const ListDesc L = P.lists[ql.list_id];
  const Scorer sc = make_scorer(P, ql);
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { s_top.count = 0; s_top.theta = (unsigned long long)qs->theta << 32; }
  __syncthreads();
  const TopK T{s_top.keys, &s_top.count, &s_top.theta, &s_top.scratch, 0u, (unsigned)kThreads};
  BlockFetch f;
  if (U.begin + warp < U.end) fetch_issue(L, U.begin + warp, lane, f);
  for (uint32_t r = U.begin; r < U.end; r += kWarps) {
    const uint32_t b = r + warp;
    if (b < U.end) {
      uint32_t doc[4], tf[4];
      fetch_decode(L, b, f, lane, doc, tf);
      if (b + kWarps < U.end) fetch_issue(L, b + kWarps, lane, f);  // next round's block travels while this one is scored
      const unsigned long long theta = *T.theta;
      const float theta_f = threshold_score((uint32_t)(theta >> 32));
      bool pass[4];
      float score[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const bool valid = doc[i] < S.max_doc;  // also rejects the kTerminated padding of the tail
        score[i] = valid ? bm25_score(sc, L.fieldnorm, doc[i], tf[i]) : 0.0f;
        pass[i] = valid && score[i] >= theta_f;  // cheap float test first; the exact key test only on survivors
      }
      if (__ballot_sync(kFull, pass[0] | pass[1] | pass[2] | pass[3])) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const unsigned long long key = make_key(score[i], doc[i]);
          bool p = pass[i] && key >= theta;
          if (p && S.alive) p = is_alive(S.alive, doc[i]);
          topk_push(T, p, key, lane);
        }
      }
    }
    topk_round_end(T, Q.k, &qs->theta);
  }
  topk_flush(T, Q, qs, P.cands, S.segment_ord);
}

// ---- intersection ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) k_and(const BatchParams P, uint32_t unit_base) {
  __shared__ uint32_t s_dec[kWarps][256];  // a decoded secondary block: 128 docs, 128 tfs
  __shared__ CtaTopK s_top;
  const Unit U = P.units[unit_base + blockIdx.x];
  const QSeg S = P.qsegs[U.qseg];
  const DQuery Q = P.queries[S.query];
  QState* qs = P.qstate + S.query;
  const QList ql0 = P.qlists[S.lists_base];
  const ListDesc L0 = P.lists[ql0.list_id];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t* dec = s_dec[warp];
  if (threadIdx.x == 0) { s_top.count = 0; s_top.theta = (unsigned long long)qs->theta << 32; }
  __syncthreads();
  const TopK T{s_top.keys, &s_top.count, &s_top.theta, &s_top.scratch, 0u, (unsigned)kThreads};
  // MaxScore for the conjunction (exact): a leader doc whose own score plus the secondaries' bounds (score < weight)
  // cannot reach the threshold is dropped BEFORE its secondary blocks are looked up and decoded -- the lookups are
  // what this kernel spends its time on (block_wand_intersection.rs:60-120 prunes on block maxima for the same reason).
  const bool prunable = (S.flags & 2u) != 0;
  // io: the sum is Intersection::score's (s0 + s1) + (s2 + s3 + ...) (`rest` holds s2 + s3 + ...), else one after another.
  // The bound tests stay upper bounds in either order: prunable weights are >= 0, so every f32 sum of these n <= 32 scores,
  // in any order, is within n * 2^-24 (< 2e-6) relative of the exact sum; the 1.00001 margin covers that.
  const bool io = (S.flags & 4u) != 0;
  const Scorer sc0 = make_scorer(P, ql0);
  float ub_secondaries = 0.0f;
  for (uint32_t s = 1; s < S.n_lists; ++s) ub_secondaries += P.qlists[S.lists_base + s].weight;
  // Without a threshold the first round would look up every leader doc of 8 blocks; one block (one warp) is enough to
  // get a first threshold, the other seven then start pruned.
  bool narrow = prunable && s_top.theta == 0ull;
  for (uint32_t r = U.begin; r < U.end;) {
    const uint32_t width = narrow ? 1u : (uint32_t)kWarps;
    const uint32_t b = r + warp;
    if (warp < width && b < U.end) {
      uint32_t doc[4], tf0[4];
      decode_block(L0, b, lane, doc, tf0);
      uint32_t alive_m = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) alive_m |= (doc[i] < S.max_doc) ? (1u << i) : 0u;  // rejects tail padding
      float total[4] = {0.f, 0.f, 0.f, 0.f}, rest[4] = {0.f, 0.f, 0.f, 0.f};
      float ub = ub_secondaries;
      const float theta_f = prunable ? threshold_score((uint32_t)(*(volatile unsigned long long*)T.theta >> 32)) : 0.0f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if ((alive_m >> i) & 1u) {
          total[i] = bm25_score(sc0, L0.fieldnorm, doc[i], tf0[i]);
          if (theta_f > 0.0f && (total[i] + ub) * 1.00001f < theta_f) alive_m &= ~(1u << i);
        }
      }
      for (uint32_t s = 1; s < S.n_lists; ++s) {
        if (__ballot_sync(kFull, alive_m != 0) == 0) break;
        const QList qls = P.qlists[S.lists_base + s];
        const ListDesc Ls = P.lists[qls.list_id];
        const Scorer sc_s = make_scorer(P, qls);
        uint32_t pending = alive_m;
        uint32_t stf[4] = {1u, 1u, 1u, 1u};
        uint32_t cur = 0;
        for (;;) {
          // smallest unresolved candidate of the warp (candidates ascend with lane*4+i)
          const uint32_t c = (pending & 1u) ? doc[0] : (pending & 2u) ? doc[1] : (pending & 4u) ? doc[2] : (pending & 8u) ? doc[3] : 0xFFFFFFFFu;
          const uint32_t cmin = warp_min(c);
          if (cmin == 0xFFFFFFFFu) break;
          const uint32_t j = first_block_ge(Ls.last_doc, cur, Ls.n_total, cmin, lane);
          if (j >= Ls.n_total) { alive_m &= ~pending; pending = 0; break; }  // past the end of this list
          const uint32_t blk_last = __ldg(Ls.last_doc + j);
          uint32_t sd[4], st[4];
          decode_block(Ls, j, lane, sd, st);
          __syncwarp();
#pragma unroll
          for (int i = 0; i < 4; ++i) { dec[lane * 4 + i] = sd[i]; dec[128 + lane * 4 + i] = st[i]; }
          __syncwarp();
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (((pending >> i) & 1u) && doc[i] <= blk_last) {
              uint32_t lo = 0;
#pragma unroll
              for (uint32_t step = 64; step > 0; step >>= 1)
                if (dec[lo + step - 1] < doc[i]) lo += step;
              if (dec[lo] == doc[i]) stf[i] = dec[128 + lo]; else alive_m &= ~(1u << i);
              pending &= ~(1u << i);
            }
          }
          cur = j + 1;
        }
        ub -= qls.weight;  // what the clauses still to come can add at most
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if ((alive_m >> i) & 1u) {
            const float v = bm25_score(sc_s, Ls.fieldnorm, doc[i], stf[i]);
            const bool to_rest = io && s >= 2u;
            if (!to_rest) total[i] = __fadd_rn(total[i], v);
            else rest[i] = s == 2u ? v : __fadd_rn(rest[i], v);
            const float partial = to_rest ? __fadd_rn(total[i], rest[i]) : total[i];
            if (theta_f > 0.0f && s + 1u < S.n_lists && (partial + ub) * 1.00001f < theta_f) alive_m &= ~(1u << i);
          }
        }
      }
      if (io && S.n_lists > 2u) {
#pragma unroll
        for (int i = 0; i < 4; ++i) total[i] = __fadd_rn(total[i], rest[i]);
      }
      const unsigned long long theta = *T.theta;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const unsigned long long key = make_key(total[i], doc[i]);
        bool pass = ((alive_m >> i) & 1u) && key >= theta;
        if (pass && S.alive) pass = is_alive(S.alive, doc[i]);
        topk_push(T, pass, key, lane);
      }
    }
    topk_round_end(T, Q.k, &qs->theta, !prunable ? kCap - kRoundMargin : (narrow ? Q.k : min(max(4u * Q.k, 128u), kCap - kRoundMargin)));
    r += width;
    narrow = false;
  }
  topk_flush(T, Q, qs, P.cands, S.segment_ord);
}

// ---- union -------------------------------------------------------------------------------------------------
// Shared memory per CTA: kTileDocs f32 score slots (dynamic) + kTileDocs fieldnorm bytes.
// A slot holding -0.0f has not been touched: -0.0 + s == 0.0 + s bit for bit for every s except
// s == -0.0 (SumCombiner starts from 0.0, score_combiner.rs:39-57).
//
// A window of kTileDocs doc ids is skipped when no clause has a block in it, or when even the sum of all clause
// maxima cannot reach the threshold.  Otherwise every clause's blocks are decoded and added in clause order, then
// the window is harvested.
struct OrShared {
  uint32_t blo[2][32], bhi[2][32];  // per clause: block range overlapping the tile (double buffered)
  uint32_t cur[32];                 // per clause: search cursor
  uint32_t any[2];
  uint32_t npass;
  float bound;                      // sum of the clause maxima x 1.00001: no doc can score more
  uint32_t run;                     // the current window is accumulated and harvested
};

// Blocks of a posting list that overlap doc ids [lo, hi), searched from block `from`: returns how many, starting at
// `first`, the first block whose last doc is >= lo (n when there is none; the next window's search starts there).
__device__ __forceinline__ uint32_t window_blocks(const uint32_t* last_doc, uint32_t n, uint32_t from, uint32_t lo, uint32_t hi,
                                                  uint32_t lane, uint32_t& first) {
  first = first_block_ge(last_doc, from, n, lo, lane);
  if (first >= n) return 0;
  // the last block that can hold a doc < hi is the first one whose last doc is >= hi-1
  const uint32_t last = first_block_ge(last_doc, first, n, hi - 1u, lane);
  return (last < n ? last : n - 1u) - first + 1u;
}

__device__ __forceinline__ void or_tile_ranges(const BatchParams& P, const QSeg& S, OrShared& sh, int buf, uint32_t tile,
                                               uint32_t warp, uint32_t lane) {
  const uint32_t lo = tile * kTileDocs;
  const uint32_t hi = min(lo + kTileDocs, S.max_doc);
  for (uint32_t t = warp; t < S.n_lists; t += kWarps) {
    const ListDesc& L = P.lists[P.qlists[S.lists_base + t].list_id];
    uint32_t first;
    const uint32_t cnt = window_blocks(L.last_doc, L.n_total, sh.cur[t], lo, hi, lane, first);
    if (lane == 0) { sh.blo[buf][t] = cnt ? first : 1u; sh.bhi[buf][t] = cnt ? first + cnt - 1u : 0u; sh.cur[t] = first; if (cnt) sh.any[buf] = 1; }
  }
}

// Blocks of clause t are dealt to the warps rotated by the clause ordinal: the single block of a rare
// clause lands on warp (t mod 8), so the rare clauses of a window are fetched by different warps at the same
// time instead of queueing on warp 0.
__device__ __forceinline__ uint32_t or_first_block(const OrShared& sh, int buf, uint32_t t, uint32_t warp) {
  return sh.blo[buf][t] + ((warp + kWarps - (t & (kWarps - 1))) & (kWarps - 1));
}
// next (clause, block) of this warp at or after (t, b) in tile buffer `buf`; t == n_lists when none
__device__ __forceinline__ void or_next_item(const OrShared& sh, int buf, uint32_t n_lists, uint32_t warp, uint32_t& t, uint32_t& b) {
  while (t < n_lists) {
    if (b <= sh.bhi[buf][t] && sh.blo[buf][t] <= sh.bhi[buf][t]) return;
    ++t;
    if (t < n_lists) b = or_first_block(sh, buf, t, warp);
  }
}

// Harvest of the window [lo, lo + kTileDocs) by the threads of T: count what passes, then push in one go when it
// fits; every score slot is reset to -0.0.  A float compare against the threshold score rejects nearly every slot
// (untouched slots hold -0.0, which is below any positive threshold); the exact key test runs only on the survivors.
// *npass is a shared pass count, 0 on entry and on return.
__device__ __forceinline__ void or_harvest(const TopK& T, float* s_acc, const QSeg& S, uint32_t lo, uint32_t k,
                                           unsigned int* theta_global, uint32_t* npass, uint32_t lane) {
  const float neg_zero = __uint_as_float(0x80000000u);
  const unsigned long long theta = *T.theta;
  const float theta_f = threshold_score((uint32_t)(theta >> 32));
  uint32_t passmask = 0;
#pragma unroll 1
  for (int j = 0; j < (int)(kTileDocs / (kThreads * 4)); ++j) {
    const uint32_t idx = (j * kThreads + threadIdx.x) * 4;
    const float4 v = *reinterpret_cast<const float4*>(s_acc + idx);
    if (v.x >= theta_f || v.y >= theta_f || v.z >= theta_f || v.w >= theta_f) {
      const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const uint32_t d = lo + idx + c;
        bool pass = vv[c] >= theta_f && __float_as_uint(vv[c]) != 0x80000000u && make_key(vv[c], d) >= theta;
        if (pass && S.alive) pass = is_alive(S.alive, d);
        passmask |= pass ? (1u << (j * 4 + c)) : 0u;
      }
    }
  }
  const uint32_t wsum = __reduce_add_sync(kFull, (uint32_t)__popc(passmask));
  if (lane == 0 && wsum) atomicAdd(npass, wsum);
  topk_sync(T);
  const bool fits = *T.count + *npass <= kCap;
  topk_sync(T);  // every thread has read the count before anyone starts pushing (the branch must be uniform)
  if (threadIdx.x == 0) *npass = 0;
  if (fits) {
#pragma unroll 1
    for (int j = 0; j < (int)(kTileDocs / (kThreads * 4)); ++j) {
      const uint32_t idx = (j * kThreads + threadIdx.x) * 4;
      const uint32_t sub = (passmask >> (j * 4)) & 15u;
      if (__ballot_sync(kFull, sub != 0)) {
        const float4 v = *reinterpret_cast<const float4*>(s_acc + idx);
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int c = 0; c < 4; ++c) topk_push(T, (sub >> c) & 1u, make_key(vv[c], lo + idx + c), lane);
      }
      *reinterpret_cast<float4*>(s_acc + idx) = make_float4(neg_zero, neg_zero, neg_zero, neg_zero);
    }
    topk_round_end(T, k, theta_global);
  } else {  // cold start: more survivors than the buffer holds; go in rounds with compaction between
    topk_round_end(T, k, theta_global);  // leaves at most kCap - kRoundMargin keys
#pragma unroll 1
    for (int j = 0; j < (int)(kTileDocs / (kThreads * 4)); ++j) {
      const uint32_t idx = (j * kThreads + threadIdx.x) * 4;
      const float4 v = *reinterpret_cast<const float4*>(s_acc + idx);
      const float vv[4] = {v.x, v.y, v.z, v.w};
      const unsigned long long th = *T.theta;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const unsigned long long key = make_key(vv[c], lo + idx + c);
        topk_push(T, ((passmask >> (j * 4 + c)) & 1u) && key >= th, key, lane);
      }
      *reinterpret_cast<float4*>(s_acc + idx) = make_float4(neg_zero, neg_zero, neg_zero, neg_zero);
      topk_round_end(T, k, theta_global);
    }
  }
}

__global__ void __launch_bounds__(kThreads, 3) k_or(const BatchParams P, uint32_t unit_base) {
  extern __shared__ __align__(16) float s_acc[];                  // [kTileDocs]
  uint8_t* s_fn = reinterpret_cast<uint8_t*>(s_acc + kTileDocs);  // [kTileDocs]
  __shared__ CtaTopK s_top;
  __shared__ OrShared sh;
  const Unit U = P.units[unit_base + blockIdx.x];
  const QSeg S = P.qsegs[U.qseg];
  const DQuery Q = P.queries[S.query];
  QState* qs = P.qstate + S.query;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const float neg_zero = __uint_as_float(0x80000000u);
  const bool staged_fn = (S.flags & 1u) && S.fieldnorm != nullptr;
  for (uint32_t i = threadIdx.x; i < kTileDocs; i += kThreads) s_acc[i] = neg_zero;
  if (threadIdx.x < 32) sh.cur[threadIdx.x] = 0;
  if (threadIdx.x == 0) {
    s_top.count = 0; s_top.theta = (unsigned long long)qs->theta << 32;
    sh.any[0] = sh.any[1] = 0; sh.npass = 0;
    // a clause can add at most its weight (tf/(tf+norm) < 1, bm25.rs:170-175); the maxima are added in ascending order
    float mx[32];
    for (uint32_t t = 0; t < S.n_lists; ++t) mx[t] = fmaxf(P.qlists[S.lists_base + t].weight, 0.0f);
    for (uint32_t i = 1; i < S.n_lists; ++i) {
      const float m = mx[i];
      uint32_t j = i;
      while (j > 0 && mx[j - 1] > m) { mx[j] = mx[j - 1]; --j; }
      mx[j] = m;
    }
    float sum = 0.0f;
    for (uint32_t i = 0; i < S.n_lists; ++i) sum += mx[i];
    sh.bound = sum * 1.00001f;  // f32 sums of up to 32 terms differ by < 4e-6 relative
  }
  __syncthreads();
  const TopK T{s_top.keys, &s_top.count, &s_top.theta, &s_top.scratch, 0u, (unsigned)kThreads};
  or_tile_ranges(P, S, sh, 0, U.begin, warp, lane);
  unsigned int theta_g_seen = 0;  // thread 0: query-wide threshold sampled one window ago
  __syncthreads();
  for (uint32_t tile = U.begin; tile < U.end; ++tile) {
    const int buf = (int)((tile - U.begin) & 1u);
    const uint32_t lo = tile * kTileDocs;
    const uint32_t hi = min(lo + kTileDocs, S.max_doc);
    if (threadIdx.x == 0) {
      const unsigned long long g = (unsigned long long)theta_g_seen << 32;
      if (g > s_top.theta) s_top.theta = g;
      theta_g_seen = *(volatile unsigned int*)&qs->theta;  // consumed at the next window
      sh.run = sh.any[buf] && sh.bound >= threshold_score((uint32_t)(s_top.theta >> 32));
    }
    __syncthreads();
    const bool run = sh.run != 0;

    if (run) {
      // ---- accumulate ----------------------------------------------------------------------------------
      // fieldnorm bytes of the window: one coalesced 16-byte row per thread pair instead of a byte gather per posting
      if (staged_fn) {
        const uint4* src = reinterpret_cast<const uint4*>(S.fieldnorm + lo);
        uint4* dst = reinterpret_cast<uint4*>(s_fn);
        for (uint32_t i = threadIdx.x; i < kTileDocs / 16; i += kThreads) dst[i] = __ldg(src + i);
      }
      // first work item of this warp, fetched before the barrier
      uint32_t t = 0, b = or_first_block(sh, buf, 0, warp);
      or_next_item(sh, buf, S.n_lists, warp, t, b);
      BlockFetch f;
      QList ql;
      ListDesc L;
      if (t < S.n_lists) { ql = P.qlists[S.lists_base + t]; L = P.lists[ql.list_id]; fetch_issue(L, b, lane, f); }
      __syncthreads();  // s_fn ready
      for (uint32_t tt = 0; tt < S.n_lists; ++tt) {
        while (t == tt) {
          uint32_t doc[4], tf[4];
          fetch_decode(L, b, f, lane, doc, tf);
          const Scorer scr = make_scorer(P, ql);
          const uint8_t* fn_global = L.fieldnorm;
          // next item (same clause or a later one) starts travelling now
          uint32_t nt = t, nb = b + kWarps;
          or_next_item(sh, buf, S.n_lists, warp, nt, nb);
          if (nt < S.n_lists) {
            if (nt != t) { ql = P.qlists[S.lists_base + nt]; L = P.lists[ql.list_id]; }
            fetch_issue(L, nb, lane, f);
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (doc[i] >= lo && doc[i] < hi) {
              const uint32_t slot = doc[i] - lo;
              const uint32_t id = staged_fn ? (uint32_t)s_fn[slot] : (fn_global ? (uint32_t)__ldg(fn_global + doc[i]) : 1u);
              const float sc = bm25_score_id(scr, id, tf[i]);
              s_acc[slot] = __fadd_rn(s_acc[slot], sc);
            }
          }
          t = nt; b = nb;
        }
        __syncthreads();  // clause order is the f32 summation order
      }
    }

    // ranges of the next window: the searches overlap the harvest below
    if (tile + 1 < U.end) {
      if (threadIdx.x == 0) sh.any[buf ^ 1] = 0;
      __syncthreads();
      or_tile_ranges(P, S, sh, buf ^ 1, tile + 1, warp, lane);
    }

    if (run) or_harvest(T, s_acc, S, lo, Q.k, &qs->theta, &sh.npass, lane);
    else __syncthreads();
  }
  topk_flush(T, Q, qs, P.cands, S.segment_ord);
}

// ---- union, strip form ----------------------------------------------------------------------------------------
// The same result as k_or, organised for latency tolerance: NO block-wide barrier in the loop.  Every warp owns a
// contiguous strip of doc ids and walks it in windows of kWin docs with private score slots, private fieldnorm
// bytes, a private candidate buffer and its own threshold (plus the query-wide one).  Clause order inside a warp
// is program order, so the f32 sum is still taken clause by clause.
//  * thick clauses (>= 1 block per window on average) are decoded window by window: one 32-wide probe of the
//    16-byte block records gives position and record, the packed vectors follow (2 dependent loads);
//  * thinner clauses keep their current block DECODED AND SCORED in shared memory (docs + scores); a window only
//    looks at it when the block's next unread doc falls inside the window, so a block is decoded once per strip.
// Eligible when k <= kStripMaxK, <= kStripMaxLists clauses and <= kMaxCached thin clauses; otherwise k_or.  The limits
// (kWin, kStripWarps, kStripMaxLists, ...) are in tq_layout.h.
constexpr uint32_t kWBuf = 256;
constexpr uint32_t kNoDoc = 0xFFFFFFFFu;

struct StripWarpFixed {  // per warp, dynamic shared memory; followed by n_cached x StripCache
  float acc[kWin + 32];               // + one private dummy slot per lane for postings outside the window
  unsigned long long keys[kWBuf];
  uint8_t fn[kWin];
  uint32_t cur[kStripMaxLists];       // thick: first block that can still matter; thin: block held in the cache
  uint32_t next_doc[kStripMaxLists];  // thin: smallest cached doc not applied yet (kNoDoc: clause exhausted)
  uint32_t pos[kStripMaxLists];       // thin: its index in the cached block (entries are in doc order)
  uint32_t stat[8];                   // lane 0: windows by route (1 exhaustive, 2 hot, 3 cold), [5] 16-byte units read
};
struct StripCache {
  uint32_t doc[128];
  float score[128];
};
static_assert(sizeof(StripWarpFixed) == kStripWarpFixedBytes && sizeof(StripCache) == kStripCacheBytes, "strip_smem_bytes (tq_layout.h)");

__device__ __forceinline__ void fetch_issue_rec(const ListDesc& L, const uint4 rec, uint32_t lane, BlockFetch& f) {
  f.meta = rec.z;
  if (rec.z == 0xFFFFFFFFu) return;  // VInt tail
  f.prev = rec.w == 0xFFFFFFFFu ? 0u : rec.w;
  const uint32_t db = rec.z & 31u, tb = (rec.z >> 8) & 63u;
  const uint4* v = reinterpret_cast<const uint4*>(L.blocks + rec.y);
  const uint32_t wd = (lane * db) >> 5;
  f.dlo = ldg_stream(v + wd);
  f.dhi = ldg_stream(v + wd + 1);
  if (L.has_freq) {
    const uint32_t wt = db + ((lane * tb) >> 5);
    f.tlo = ldg_stream(v + wt);
    f.thi = ldg_stream(v + wt + 1);
  }
}

// warp-level: sort the candidate buffer (descending) and keep the best k
__device__ __noinline__ void strip_compact(unsigned long long* keys, uint32_t& cnt, uint32_t k, unsigned long long& theta,
                                              unsigned int* theta_global, uint32_t lane) {
  for (uint32_t i = cnt + lane; i < kWBuf; i += 32) keys[i] = 0ull;
  __syncwarp();
  for (uint32_t kk = 2; kk <= kWBuf; kk <<= 1) {
    for (uint32_t j = kk >> 1; j > 0; j >>= 1) {
      for (uint32_t p = lane; p < kWBuf / 2; p += 32) {
        const uint32_t i = ((p & ~(j - 1u)) << 1) | (p & (j - 1u));
        const uint32_t ixj = i | j;
        const unsigned long long a = keys[i], b = keys[ixj];
        const bool desc = (i & kk) == 0;
        if (desc ? (a < b) : (a > b)) { keys[i] = b; keys[ixj] = a; }
      }
      __syncwarp();
    }
  }
  if (cnt > k) {
    cnt = k;
    const unsigned long long kth = keys[k - 1];
    if (kth > theta) theta = kth;
    if (lane == 0) atomicMax(theta_global, (unsigned)(kth >> 32));
  }
  __syncwarp();
}

// Decodes block j of a thin clause into the warp's cache, scored (one conflict-free 16-byte store per lane and array).
__device__ __noinline__ uint32_t strip_cache_block(const ListDesc& L, uint32_t j, const Scorer sc, uint32_t max_doc, StripCache& cc, uint32_t lane) {
  uint32_t doc[4], tf[4];
  decode_block(L, j, lane, doc, tf);
  uint32_t cd[4];
  float cs[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const bool valid = doc[i] < max_doc;
    cd[i] = valid ? doc[i] : kNoDoc;
    cs[i] = valid ? bm25_score(sc, L.fieldnorm, doc[i], tf[i]) : 0.0f;
  }
  reinterpret_cast<uint4*>(cc.doc)[lane] = make_uint4(cd[0], cd[1], cd[2], cd[3]);
  reinterpret_cast<float4*>(cc.score)[lane] = make_float4(cs[0], cs[1], cs[2], cs[3]);
  __syncwarp();
  // bytes this touched, in 16-byte units: the packed block (or the decoded tail) + one fieldnorm byte per posting
  return (j < L.n_blocks ? (__ldg(&L.blk[j + 1].x) - __ldg(&L.blk[j].x)) / 16u : L.tail_n / 2u) + 8u;
}

// Positions a thin clause on the first posting >= lo: keeps the cached block when it still reaches lo, else seeks through
// the block table (SkipReader::seek) and caches that block.  cur = block in the cache (n_total: exhausted).
__device__ __noinline__ uint32_t strip_thin_seek(const ListDesc& L, const Scorer sc, uint32_t max_doc, StripCache& cc, bool cache_valid,
                                                    uint32_t lo, uint32_t lane, uint32_t& cur, uint32_t& pos, uint32_t& next_doc) {
  uint32_t j = cur, touched16 = 0;
  if (!(cache_valid && j < L.n_total && __ldg(L.last_doc + j) >= lo)) {
    j = first_block_ge(L.last_doc, cache_valid ? j + 1u : 0u, L.n_total, lo, lane);
    cur = j;
    if (j >= L.n_total) { pos = 128u; next_doc = kNoDoc; return 0; }
    touched16 = strip_cache_block(L, j, sc, max_doc, cc, lane);
  }
  uint32_t below = 0;  // entries are in doc order, padding is kNoDoc: count what lies before lo
#pragma unroll
  for (uint32_t g = 0; g < 4; ++g) below += (uint32_t)__popc(__ballot_sync(kFull, cc.doc[g * 32u + lane] < lo));
  pos = below;
  next_doc = below < 128u ? cc.doc[below] : kNoDoc;
  return touched16;
}

// MaxScore on top of the strips (exact).  The planner orders a union's clauses by descending Bm25Weight.weight — that is
// the order the f32 sum is taken in — so the clauses whose upper bounds (score < weight, since tf/(tf+norm) < 1) add up
// to less than the current threshold are always a SUFFIX of the clause list: the non-essential clauses.  Per window the
// warp applies the essential prefix; if the largest partial sum plus the non-essential bound cannot reach the threshold,
// the window is cold and the non-essential clauses (the dense, expensive ones) are not decoded at all; otherwise they
// are added on top, in order, which continues the very same f32 sum.  A doc without any essential posting scores below
// the threshold by construction.  Non-essential clauses fall behind while windows stay cold and catch up through the
// block table when a window turns hot.
__global__ void __launch_bounds__(kStripThreads) k_or_strip(const BatchParams P, uint32_t unit_base, uint32_t n_cached_max) {
  extern __shared__ __align__(16) unsigned char s_dyn[];
  __shared__ ListDesc s_list[kStripMaxLists];
  __shared__ QList s_ql[kStripMaxLists];
  const Unit U = P.units[unit_base + blockIdx.x];
  const QSeg S = P.qsegs[U.qseg];
  const DQuery Q = P.queries[S.query];
  QState* qs = P.qstate + S.query;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (threadIdx.x < S.n_lists) {
    s_ql[threadIdx.x] = P.qlists[S.lists_base + threadIdx.x];
    s_list[threadIdx.x] = P.lists[s_ql[threadIdx.x].list_id];
  }
  __syncthreads();  // the only block-wide barrier
  const size_t per_warp = sizeof(StripWarpFixed) + (size_t)n_cached_max * sizeof(StripCache);
  StripWarpFixed& W = *reinterpret_cast<StripWarpFixed*>(s_dyn + warp * per_warp);
  StripCache* C = reinterpret_cast<StripCache*>(s_dyn + warp * per_warp + sizeof(StripWarpFixed));
  const float neg_zero = __uint_as_float(0x80000000u);
  // this warp's windows
  const uint32_t n_win = U.end - U.begin;
  const uint32_t w_begin = U.begin + (uint32_t)(((unsigned long long)n_win * warp) / kStripWarps);
  const uint32_t w_end = U.begin + (uint32_t)(((unsigned long long)n_win * (warp + 1)) / kStripWarps);
  for (uint32_t i = lane; i < kWin; i += 32) W.acc[i] = neg_zero;
  const bool staged_fn = (S.flags & 1u) && S.fieldnorm != nullptr;
  const bool prunable = (S.flags & 2u) != 0;  // every weight finite and >= 0
  uint32_t thick_mask = 0;
  uint32_t n_e_min = 0;  // only the thick clauses at the end of the list may turn non-essential: thin ones are cheap to
                         // apply and every clause kept essential tightens the cold-window test
  uint32_t cnt = 0;
  if (lane < 8) W.stat[lane] = 0;  // [5]: postings and fieldnorm bytes actually read, in 16-byte units (SURVEY.md §8d: pruned kernels)
  __syncwarp();
  unsigned long long theta = (unsigned long long)(*(volatile unsigned int*)&qs->theta) << 32;
  if (w_begin < w_end) {
    // ---- strip start: position every clause -------------------------------------------------------------
    const uint32_t lo0 = w_begin * kWin;
    for (uint32_t t = 0; t < S.n_lists; ++t) {
      const ListDesc& L = s_list[t];
      const bool thin = (s_ql[t].pad & 1u) != 0;
      if (!thin) {
        thick_mask |= 1u << t;
        const uint32_t j = first_block_ge(L.last_doc, 0, L.n_total, lo0, lane);
        if (lane == 0) { W.cur[t] = j; W.next_doc[t] = 0; }
      } else {
        uint32_t cur = 0, pos = 0, nd = kNoDoc;
        const uint32_t t16 = strip_thin_seek(L, make_scorer(P, s_ql[t]), S.max_doc, C[s_ql[t].pad >> 1], false, lo0, lane, cur, pos, nd);
        if (lane == 0) { W.cur[t] = cur; W.pos[t] = pos; W.next_doc[t] = nd; W.stat[5] += t16; }
      }
    }
    __syncwarp();
    {  // a clause may turn non-essential when it has at least one posting per kStripNeDiv docs
      n_e_min = S.n_lists;
      while (n_e_min > 0 && (unsigned long long)s_list[n_e_min - 1u].doc_freq * kStripNeDiv >= S.max_doc) --n_e_min;
      // no such clause: the single densest one may still go if it is dense enough to matter (kStripNeDiv2)
      if (n_e_min == S.n_lists && n_e_min > 1 && (unsigned long long)s_list[n_e_min - 1u].doc_freq * kStripNeDiv2 >= S.max_doc) --n_e_min;
    }
    // ---- the windows ---------------------------------------------------------------------------------------
    uint32_t since_refresh = 0;
    for (uint32_t w = w_begin; w < w_end; ++w) {
      const float theta_f = threshold_score((uint32_t)(theta >> 32));
      // essential prefix [0, n_e) / non-essential suffix and its score bound under the current threshold
      uint32_t n_e = S.n_lists;
      float ne_bound = 0.0f;
      if (prunable && theta_f > 0.0f) {
        while (n_e > n_e_min) {
          const float nb = ne_bound + s_ql[n_e - 1u].weight;
          if (!(nb * 1.00001f < theta_f)) break;
          ne_bound = nb;
          --n_e;
        }
        if (n_e == 0) break;  // no doc of this segment can reach the threshold any more
      }
      if (!(thick_mask & ((1u << n_e) - 1u))) {  // only thin essential clauses: jump to the window of their next unread doc
        uint32_t nd = lane < n_e ? W.next_doc[lane] : kNoDoc;
        nd = warp_min(nd);
        if (nd == kNoDoc) break;
        const uint32_t wj = nd / kWin;
        if (wj >= w_end) break;
        if (wj > w) w = wj;
      }
      const uint32_t lo = w * kWin;
      const uint32_t hi = min(lo + kWin, S.max_doc);
      if (++since_refresh == 16u) {  // pick up the query-wide threshold now and then
        since_refresh = 0;
        unsigned int g = lane == 0 ? *(volatile unsigned int*)&qs->theta : 0u;
        g = __shfl_sync(kFull, g, 0);
        const unsigned long long gt = (unsigned long long)g << 32;
        if (gt > theta) theta = gt;
      }
      bool fn_ready = false;  // the window's fieldnorm bytes are staged when the first thick clause needs them
      bool dirty = false;     // the window received at least one score
      bool cold = false;
      float wmax = 0.0f;      // largest partial sum written by this lane (scores are non-negative: it bounds the final sums)
      for (uint32_t t = 0; t < S.n_lists; ++t) {
        if (t >= n_e) {  // can the clauses still to come lift a doc of this window over the threshold?  (asked again
                         // after every non-essential clause: the densest ones come last)
          const float mx = __uint_as_float(__reduce_max_sync(kFull, __float_as_uint(wmax)));
          if ((mx + ne_bound) * 1.00001f < theta_f) { cold = true; break; }
          ne_bound -= s_ql[t].weight;  // (rounding stays far inside the 1e-5 margin of the test)
        }
        const ListDesc& L = s_list[t];
        const bool thin = (s_ql[t].pad & 1u) != 0;
        if (!thin) {
          // ---- thick clause: decode the blocks that overlap [lo, hi) ---------------------------------------
          uint32_t cur = W.cur[t];
          if (cur >= L.n_total) continue;
          uint4 r;
          unsigned m;
          {
            const uint32_t idx = cur + lane;
            r = idx < L.n_total ? __ldg(L.tab4 + idx) : make_uint4(0xFFFFFFFFu, 0, 0, 0);
            m = __ballot_sync(kFull, r.x >= lo);
            if (!m) {  // the clause sat out many windows: seek through the block table
              cur = first_block_ge(L.last_doc, cur + 32u, L.n_total, lo, lane);
              const uint32_t idx2 = cur + lane;
              r = idx2 < L.n_total ? __ldg(L.tab4 + idx2) : make_uint4(0xFFFFFFFFu, 0, 0, 0);
              m = __ballot_sync(kFull, r.x >= lo);
            }
          }
          uint32_t src = (uint32_t)__ffs(m) - 1u;
          uint32_t j = cur + src;
          __syncwarp();  // every lane has read W.cur[t]
          if (lane == 0) W.cur[t] = j;
          if (j >= L.n_total) continue;
          const Scorer sc = make_scorer(P, s_ql[t]);
          uint4 rec;
          rec.x = __shfl_sync(kFull, r.x, src); rec.y = __shfl_sync(kFull, r.y, src);
          rec.z = __shfl_sync(kFull, r.z, src); rec.w = __shfl_sync(kFull, r.w, src);
          if (rec.w != 0xFFFFFFFFu && rec.w + 1u >= hi) continue;  // the block starts at or after the window's end
          BlockFetch f;
          fetch_issue_rec(L, rec, lane, f);
          if (staged_fn && !fn_ready) {
            const uint4* fsrc = reinterpret_cast<const uint4*>(S.fieldnorm + lo);
            uint4* dst = reinterpret_cast<uint4*>(W.fn);
            for (uint32_t i = lane; i < kWin / 16u; i += 32) dst[i] = __ldg(fsrc + i);
            __syncwarp();
            fn_ready = true;
            if (lane == 0) W.stat[5] += kWin / 16u;
          }
          dirty = true;
          uint32_t t16 = 0;  // 16-byte units of packed postings read for this clause and window
          for (;;) {
            uint32_t doc[4], tf[4];
            const bool small_tf = ((f.meta >> 8) & 63u) <= 4u;  // (the VInt tail's marker reads as 63 bits)
            t16 += f.meta == 0xFFFFFFFFu ? L.tail_n / 2u : (f.meta & 31u) + ((f.meta >> 8) & 63u);
            fetch_decode(L, j, f, lane, doc, tf);
            // the next block is needed iff this one ends before the window does
            const bool more = rec.x < hi - 1u && j + 1u < L.n_total;
            if (more) {
              ++j; ++src;
              if (src == 32u) {  // ran off the probe: fetch the next 32 records
                cur = j; src = 0;
                const uint32_t idx = cur + lane;
                r = idx < L.n_total ? __ldg(L.tab4 + idx) : make_uint4(0xFFFFFFFFu, 0, 0, 0);
              }
              rec.x = __shfl_sync(kFull, r.x, src); rec.y = __shfl_sync(kFull, r.y, src);
              rec.z = __shfl_sync(kFull, r.z, src); rec.w = __shfl_sync(kFull, r.w, src);
              fetch_issue_rec(L, rec, lane, f);
            }
            // Branch-free: the four postings of a lane form four independent load chains (fieldnorm byte -> factor
            // table -> score slot) that overlap instead of running one after the other behind divergent branches.
            // Postings outside the window are steered to the lane's dummy slot behind the window (its value is never read back
            // for a result: all four loads precede the four stores).
            bool in[4];
            uint32_t slot[4], id[4];
            float fac[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              in[i] = doc[i] >= lo && doc[i] < hi;
              slot[i] = in[i] ? doc[i] - lo : kWin + lane;
              id[i] = staged_fn ? (uint32_t)W.fn[in[i] ? slot[i] : 0u]
                                : (L.fieldnorm ? (uint32_t)__ldg(L.fieldnorm + (in[i] ? doc[i] : 0u)) : 1u);
            }
            if (small_tf) {  // tf_bits <= 4: every term frequency of the block is inside the factor table
#pragma unroll
              for (int i = 0; i < 4; ++i) fac[i] = __ldg(sc.tf_table + (tf[i] << 8) + id[i]);
            } else {
              bool big = false;
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                fac[i] = __ldg(sc.tf_table + (min(tf[i], kTfRows - 1u) << 8) + id[i]);
                big |= in[i] && tf[i] >= kTfRows;
              }
              if (__ballot_sync(kFull, big)) {  // a term frequency beyond the table: take the divide for those
#pragma unroll
                for (int i = 0; i < 4; ++i)
                  if (in[i] && tf[i] >= kTfRows) fac[i] = bm25_factor_large_tf(sc.cache, id[i], tf[i]);
              }
            }
            float a[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = W.acc[slot[i]];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float nv = __fadd_rn(a[i], bm25_term_score(sc.weight, fac[i]));
              W.acc[slot[i]] = nv;
              wmax = in[i] ? fmaxf(wmax, nv) : wmax;
            }
            if (!more) break;
          }
          if (lane == 0) W.stat[5] += t16;
          __syncwarp();
        } else {
          // ---- thin clause: the decoded block lives in shared memory ---------------------------------------
          StripCache& cc = C[s_ql[t].pad >> 1];
          if (W.next_doc[t] < lo) {  // it sat out some windows as a non-essential clause: skip what lies before this one
            uint32_t cur = W.cur[t], pos = 0, nd = kNoDoc;
            const uint32_t t16 = strip_thin_seek(L, make_scorer(P, s_ql[t]), S.max_doc, cc, cur < L.n_total, lo, lane, cur, pos, nd);
            __syncwarp();
            if (lane == 0) { W.cur[t] = cur; W.pos[t] = pos; W.next_doc[t] = nd; W.stat[5] += t16; }
            __syncwarp();
          }
          for (;;) {
            if (W.next_doc[t] >= hi) break;  // nothing of this clause in the window (also: clause exhausted)
            // entries are in doc order: the window's postings are the next few entries, one per lane
            uint32_t pos = W.pos[t];
            const uint32_t e = pos + lane;
            const uint32_t d = e < 128u ? cc.doc[e] : kNoDoc;
            const bool in = d < hi;  // d >= lo: everything before the cursor is consumed
            const uint32_t napp = (uint32_t)__popc(__ballot_sync(kFull, in));
            if (in) {
              const uint32_t slot = d - lo;
              const float nv = __fadd_rn(W.acc[slot], cc.score[e]);
              W.acc[slot] = nv;
              wmax = fmaxf(wmax, nv);
            }
            dirty = true;
            pos += napp;
            const uint32_t nxt = napp < 32u ? __shfl_sync(kFull, d, napp) : (pos < 128u ? cc.doc[pos] : kNoDoc);
            __syncwarp();
            if (nxt != kNoDoc) {  // the block still holds unread docs (in this window only if all 32 lanes applied)
              if (lane == 0) { W.pos[t] = pos; W.next_doc[t] = nxt; }
              __syncwarp();
              continue;
            }
            // block used up: bring in the next one
            const uint32_t jb = W.cur[t] + 1u;
            __syncwarp();  // every lane has read W.cur[t]
            if (jb >= L.n_total) { if (lane == 0) { W.cur[t] = L.n_total; W.next_doc[t] = kNoDoc; } __syncwarp(); break; }
            const uint32_t t16 = strip_cache_block(L, jb, make_scorer(P, s_ql[t]), S.max_doc, cc, lane);
            const uint32_t first = cc.doc[0];  // a block's first entry is always a real doc
            if (lane == 0) { W.cur[t] = jb; W.next_doc[t] = first; W.pos[t] = 0; W.stat[5] += t16; }
            __syncwarp();
          }
        }
      }
      if (lane == 0) ++W.stat[n_e == S.n_lists ? 1 : (cold ? 3 : 2)];
      // ---- harvest -----------------------------------------------------------------------------------------------
      if (dirty) {
        // the largest partial sum any lane wrote bounds every final score of the window (scores >= 0; a negative
        // one makes the uint compare fail safe): when it is below the threshold the window is only cleared
        const uint32_t mx = __reduce_max_sync(kFull, __float_as_uint(wmax));
        const bool may_pass = !cold && (!(theta_f > 0.0f) || mx >= __float_as_uint(theta_f));
        for (uint32_t g = 0; g < kWin / 128; ++g) {
          const uint32_t idx = g * 128 + lane * 4;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (may_pass) v = *reinterpret_cast<const float4*>(W.acc + idx);
          *reinterpret_cast<float4*>(W.acc + idx) = make_float4(neg_zero, neg_zero, neg_zero, neg_zero);
          // float test first (nearly everything fails it); keys are built for the survivors only
          if (may_pass && __ballot_sync(kFull, v.x >= theta_f || v.y >= theta_f || v.z >= theta_f || v.w >= theta_f)) {
            const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const uint32_t d = lo + idx + c;
              const unsigned long long key = make_key(vv[c], d);
              bool pass = vv[c] >= theta_f && __float_as_uint(vv[c]) != 0x80000000u && key >= theta;
              if (pass && S.alive) pass = is_alive(S.alive, d);
              unsigned mm = __ballot_sync(kFull, pass);
              if (mm) {
                if (cnt + 32u > kWBuf) {  // make room for one key per lane; the threshold may rise
                  strip_compact(W.keys, cnt, Q.k, theta, &qs->theta, lane);
                  pass = pass && key >= theta;
                  mm = __ballot_sync(kFull, pass);
                }
                if (pass) W.keys[cnt + __popc(mm & lanemask_lt(lane))] = key;
                cnt += __popc(mm);
              }
            }
            __syncwarp();
          }
        }
      }
      __syncwarp();  // cursor updates of this window are visible to the next one
    }
  }
  __syncwarp();
  if (P.counters && (lane == 1 || lane == 2 || lane == 3 || lane == 5) && W.stat[lane])
    atomicAdd(&P.counters[lane], (unsigned long long)W.stat[lane] * (lane == 5 ? 16ull : 1ull));
  // ---- hand the survivors over ------------------------------------------------------------------------------
  if (cnt > Q.k) strip_compact(W.keys, cnt, Q.k, theta, &qs->theta, lane);
  unsigned base = 0;
  if (lane == 0 && cnt) base = atomicAdd(&qs->cand_count, cnt);
  base = __shfl_sync(kFull, base, 0);
  for (uint32_t i = lane; i < cnt; i += 32) {
    if (base + i < Q.cand_cap) {
      const unsigned long long key = W.keys[i];
      Cand c;
      c.score_key = (uint32_t)(key >> 32);
      c.segment_ord = S.segment_ord;
      c.doc = 0xFFFFFFFFu - (uint32_t)key;
      c.pad = 0;
      P.cands[Q.cand_base + base + i] = c;
    }
  }
}

// ---- final per-query selection -----------------------------------------------------------------------------
// Keys: a = score_key:32 | (0xFFFFFFFF - segment_ord):32, b = ~doc; descending (a, b) is
// (score desc, segment_ord asc, doc asc) = compare_for_top_k (top_score_collector.rs:591-600).  k_sort_final sorts with a 64-bit b.
template <class B>
__device__ __noinline__ void sort_pairs_desc(unsigned long long* a, B* b, unsigned n) {
  unsigned size = 2;
  while (size < n) size <<= 1;
  for (unsigned i = threadIdx.x; i < size; i += blockDim.x)
    if (i >= n) { a[i] = 0ull; b[i] = 0u; }
  __syncthreads();
  for (unsigned kk = 2; kk <= size; kk <<= 1) {
    for (unsigned j = kk >> 1; j > 0; j >>= 1) {
      for (unsigned i = threadIdx.x; i < size; i += blockDim.x) {
        const unsigned ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a1 = a[i], a2 = a[ixj];
          const B b1 = b[i], b2 = b[ixj];
          const bool first_less = a1 < a2 || (a1 == a2 && b1 < b2);
          const bool first_greater = a1 > a2 || (a1 == a2 && b1 > b2);
          const bool desc = (i & kk) == 0;
          if (desc ? first_less : first_greater) { a[i] = a2; a[ixj] = a1; b[i] = b2; b[ixj] = b1; }
        }
      }
      __syncthreads();
    }
  }
}

// ---- Count collector (N4): how many alive docs match, no scores ----------------------------------------------------
// src/collector/count_collector.rs + Weight::count (term_weight.rs:179-219; BooleanWeight::complex_scorer's scorer,
// boolean_weight.rs:236-431): one CTA walks its share of a (query, segment)'s 8192-doc tiles.  Per tile a result bitmap in
// shared memory = AND over the MUST groups of (OR of the group's clauses), SHOULD clauses counted per doc (byte counters, four
// to a word) against `need`, MUST_NOT clauses cleared, alive bits and-ed in, popcount.  A term query is one MUST group of its
// clause, an OR one group of all its clauses, an AND one group per clause.
// The structure words are CountParams::words (tq_layout.h).

// One 8192-doc tile [lo, hi) of a (query, segment) evaluated as a boolean structure: one pass per MUST group, then one over the
// SHOULD clauses and one over the MUST_NOT clauses.  A pass marks its clauses' postings in s_tmp (SHOULD: counts them in s_cnt) and
// then narrows s_acc; the first MUST group marks s_acc itself.  One posting walk for every pass keeps the caller's registers at
// those of a single inlined decode.  Then on_word(w, bits) for every 32-doc word of the tile: the matching docs, docs at and beyond
// max_doc cleared, alive bits (or the filter view) and-ed in.  Every thread of the CTA calls it; the caller syncs before s_acc is
// written again.  k_count and k_sort share it.
// kMixed: some (query, segment) of the launch has SHOULD or MUST_NOT clauses.  Without them (every term, AND and OR query) every
// pass is a MUST group: that instance has no SHOULD counters and no SHOULD or MUST_NOT pass per tile, which AND queries of
// sparse lists otherwise pay for.
template <bool kMixed, class OnWord>
__device__ __forceinline__ void match_tile(const CountParams& P, const uint8_t* alive, uint32_t wb, uint32_t ng, uint32_t need,
                                           uint32_t lo, uint32_t hi, uint32_t* s_acc, uint32_t* s_tmp, uint32_t* s_cnt, OnWord on_word) {
  constexpr uint32_t kWords = kTileDocs / 32u;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (ng == 0u)
    for (uint32_t w = threadIdx.x; w < kWords; w += blockDim.x) s_acc[w] = 0xFFFFFFFFu;
  uint32_t x = wb + 4u;
  for (uint32_t p = 0; p < (kMixed ? ng + 2u : ng); ++p) {
    const uint32_t kind = p < ng ? 0u : p - ng + 1u;  // 0: MUST group, 1: SHOULD, 2: MUST_NOT
    const uint32_t len = kind == 0u ? P.words[x++] : P.words[wb + kind + 1u];
    const bool should = kMixed && kind == 1u;
    if (should ? need == 0u : len == 0u) { x += len; continue; }  // (a MUST group is never empty)
    uint32_t* const bits = p == 0u ? s_acc : s_tmp;
    if (should)
      for (uint32_t w = threadIdx.x; w < kTileDocs / 4u; w += blockDim.x) s_cnt[w] = 0;
    else
      for (uint32_t w = threadIdx.x; w < kWords; w += blockDim.x) bits[w] = 0;
    __syncthreads();
    for (const uint32_t end = x + len; x < end; ++x) {
      const ListDesc L = P.lists[P.words[x]];
      const uint32_t j0 = first_block_ge(L.last_doc, 0, L.n_total, lo, lane);
      for (uint32_t j = j0 + warp; j < L.n_total; j += kWarps) {
        const uint32_t prev = __ldg(&L.tab4[j].w);
        if (prev != 0xFFFFFFFFu && prev + 1u >= hi) break;  // the block starts at or after the tile's end
        uint32_t doc[4], tf[4];
        decode_block(L, j, lane, doc, tf);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const uint32_t o = doc[i] - lo;
          if (doc[i] >= lo && doc[i] < hi) {
            if (should) atomicAdd(&s_cnt[o >> 2], 1u << ((o & 3u) * 8u));  // <= 32 clauses: no carry
            else atomicOr(&bits[o >> 5], 1u << (o & 31u));
          }
        }
      }
    }
    __syncthreads();
    if (p == 0u && !should) continue;
    for (uint32_t w = threadIdx.x; w < kWords; w += blockDim.x) {
      uint32_t m = s_tmp[w];
      if (should) {
        m = 0;
#pragma unroll
        for (uint32_t b = 0; b < 8; ++b) {
          const uint32_t c4 = s_cnt[w * 8u + b];
#pragma unroll
          for (uint32_t k = 0; k < 4; ++k) m |= (((c4 >> (8u * k)) & 255u) >= need ? 1u : 0u) << (b * 4u + k);
        }
      }
      s_acc[w] &= kind == 2u ? ~m : m;
    }
    __syncthreads();
  }
  for (uint32_t w = threadIdx.x; w < kWords; w += blockDim.x) {
    uint32_t bits = s_acc[w];
    const uint32_t first = lo + w * 32u;
    if (first >= hi) bits = 0;
    else if (hi - first < 32u) bits &= (1u << (hi - first)) - 1u;  // docs beyond max_doc
    if (bits && alive) bits &= __ldg(reinterpret_cast<const uint32_t*>(alive) + ((lo >> 5) + w));
    on_word(w, bits);
  }
}

template <bool kMixed>
__global__ void __launch_bounds__(kThreads) k_count(const CountParams P) {
  __shared__ uint32_t s_acc[kTileDocs / 32u], s_tmp[kTileDocs / 32u];
  __shared__ uint32_t s_cnt[kMixed ? kTileDocs / 4u : 1u];
  __shared__ uint32_t s_part[kWarps];
  const Unit U = P.units[blockIdx.x];
  const CountSeg S = P.segs[U.qseg];
  // (the words are read through P.words, a kernel parameter: no pointer of their own has to live through the posting walk)
  const uint32_t wb = S.words_base, ng = P.words[wb], need = P.words[wb + 1u];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t total = 0;
  for (uint32_t tile = U.begin; tile < U.end; ++tile) {
    const uint32_t lo = tile * kTileDocs, hi = min(lo + kTileDocs, S.max_doc);
    match_tile<kMixed>(P, S.alive, wb, ng, need, lo, hi, s_acc, s_tmp, s_cnt, [&](uint32_t, uint32_t bits) { total += (uint32_t)__popc(bits); });
    __syncthreads();
  }
  total = __reduce_add_sync(kFull, total);
  if (lane == 0) s_part[warp] = total;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long sum = 0;
    for (int w = 0; w < kWarps; ++w) sum += s_part[w];
    if (sum) atomicAdd(&P.counts[P.segs[P.units[blockIdx.x].qseg].query], sum);  // (read here: nothing of it lives through the tiles)
  }
}

// ---- sort by a fast field (TopDocs::order_by_fast_field: SortByStaticFastValue, sort_by_static_fast_value.rs) ----------------
// The docs Count counts, each keyed by its column value, top k.  One CTA per Count unit: per 8192-doc tile it first reads the
// query's threshold and skips the tile when no doc of it can enter the top k -- every doc with a value is below the bound (the
// tile's best v', SortTile) and the query already holds k docs with values or the tile has no None doc -- unless the query's hits
// are counted.  Otherwise match_tile builds the tile's match bitmap, each matching doc with a value is keyed by v' (an 8-byte
// gather) and kept in a shared buffer when v' >= the bound; a full buffer is sorted by (v' desc, doc asc) and cut to k, whose
// k-th v' then bounds the query (atomicMax); so is the buffer at the end of the tile in which it first holds k docs.  A doc is
// dropped only when k docs strictly precede it.  A unit walks its tiles backwards (kSortUnitBackward) when its bounds rise and it
// has no None doc: a column ascending in doc id, sorted Desc, then finds its best docs first.  None docs all tie, so the
// unit keeps its first k in doc order.  At exit each unit hands over at most k docs of each stream: the regions hold that much,
// so nothing is ever dropped for capacity.

// Sorts the buffer by (v' desc, doc asc), keeps its first k and, when it held k, raises the CTA's and the query's bounds.
__device__ __forceinline__ void sort_compact(unsigned long long* s_key, uint32_t* s_doc, uint32_t& s_n, uint32_t k, unsigned long long& s_theta,
                                             uint32_t& s_full, SortQState* qs) {
  const uint32_t n = s_n;
  sort_pairs_desc(s_key, s_doc, n);
  if (threadIdx.x == 0) {
    if (n >= k) {
      const unsigned long long kth = s_key[k - 1];
      if (kth > s_theta) { s_theta = kth; atomicMax(&qs->theta, kth); }
      if (!s_full) { s_full = 1; atomicExch(&qs->full, 1u); }
    }
    s_n = min(n, k);
  }
  __syncthreads();
}

template <bool kMixed>
__global__ void __launch_bounds__(kThreads) k_sort(const SortParams P) {
  static_assert(kTileDocs / 32u == (uint32_t)kThreads, "one 32-doc word of a tile per thread");
  __shared__ uint32_t s_acc[kTileDocs / 32u], s_tmp[kTileDocs / 32u];
  __shared__ uint32_t s_cnt[kMixed ? kTileDocs / 4u : 1u];
  __shared__ unsigned long long s_key[kCap];
  __shared__ uint32_t s_doc[kCap];  // ~doc: descending (key, ~doc) is (v' desc, doc asc)
  __shared__ uint32_t s_none[kSortMaxK];
  __shared__ uint32_t s_part[kWarps];
  __shared__ unsigned long long s_theta;  // max(the k-th v' this CTA held, the query's bound when last read)
  __shared__ uint32_t s_n, s_nn, s_full, s_skip, s_base, s_nbase;
  const Unit U = P.c.units[blockIdx.x];
  const CountSeg S = P.c.segs[U.qseg];
  const SortSeg Z = P.ssegs[U.qseg];
  const SortQuery Q = P.queries[S.query];
  SortQState* const qs = P.qstate + S.query;
  const uint32_t wb = S.words_base, ng = P.c.words[wb], need = P.c.words[wb + 1u];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const bool asc = (Q.flags & kSortAsc) != 0;
  if (threadIdx.x == 0) { s_theta = 0; s_n = 0; s_nn = 0; s_full = 0; }
  uint32_t total = 0, seen = 0, skipped = 0;
  for (uint32_t i = U.begin; i < U.end; ++i) {
    const uint32_t tile = (U.pad & kSortUnitBackward) ? U.end - 1u - (i - U.begin) : i;
    const uint32_t lo = tile * kTileDocs, hi = min(lo + kTileDocs, S.max_doc);
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned long long th = max(s_theta, *reinterpret_cast<volatile unsigned long long*>(&qs->theta));
      const uint32_t full = s_full | *reinterpret_cast<volatile uint32_t*>(&qs->full);
      s_theta = th;
      s_full = full;
      const SortTile T = Z.tiles[tile];
      const bool skip = !(Q.flags & kSortAllTiles) && (!(T.flags & kSortTileValues) || T.best[asc ? 1 : 0] < th) &&
                        (!(T.flags & kSortTileNone) || full);
      s_skip = skip;
      ++seen;
      skipped += skip ? 1u : 0u;
    }
    __syncthreads();
    if (s_skip) continue;
    match_tile<kMixed>(P.c, S.alive, wb, ng, need, lo, hi, s_acc, s_tmp, s_cnt, [&](uint32_t w, uint32_t bits) { s_acc[w] = bits; });
    __syncthreads();
    const uint32_t bits = s_acc[threadIdx.x];
    total += (uint32_t)__popc(bits);
    uint32_t with = bits, none = 0;
    if (Z.present) {
      const uint32_t pw = __ldg(Z.present + (lo >> 5) + threadIdx.x);
      with = bits & pw;
      none = bits & ~pw;
    }
    // None docs: the unit's first k in doc order (a CTA-wide prefix sum over the words), until k docs with values are known
    if (Z.present && !s_full && s_nn < Q.k) {
      const uint32_t c = (uint32_t)__popc(none);
      uint32_t incl = c;
#pragma unroll
      for (uint32_t o = 1; o < 32u; o <<= 1) {
        const uint32_t v = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += v;
      }
      if (lane == 31u) s_part[warp] = incl;
      __syncthreads();
      uint32_t at = s_nn + incl - c;
      for (uint32_t w = 0; w < warp; ++w) at += s_part[w];
      for (uint32_t m = none; m && at < Q.k; m &= m - 1u, ++at) s_none[at] = lo + threadIdx.x * 32u + (uint32_t)(__ffs(m) - 1);
      __syncthreads();
      if (threadIdx.x == 0) {
        uint32_t sum = s_nn;
        for (int w = 0; w < kWarps; ++w) sum += s_part[w];
        s_nn = min(sum, Q.k);
      }
    }
    // docs with values, one per thread and round: a round adds at most kThreads keys, so the buffer is cut before it can overflow
    while (__syncthreads_or(with != 0u)) {
      const unsigned long long th = s_theta;
      if (with) {
        const uint32_t doc = lo + threadIdx.x * 32u + (uint32_t)(__ffs(with) - 1);
        with &= with - 1u;
        const unsigned long long v = __ldg(Z.values + doc);
        const unsigned long long key = asc ? ~v : v;
        if (key >= th) {
          const uint32_t slot = atomicAdd(&s_n, 1u);
          s_key[slot] = key;
          s_doc[slot] = ~doc;
        }
      }
      __syncthreads();
      if (s_n > kCap - (uint32_t)kThreads) sort_compact(s_key, s_doc, s_n, Q.k, s_theta, s_full, qs);
    }
    if (!s_full && s_n >= Q.k) sort_compact(s_key, s_doc, s_n, Q.k, s_theta, s_full, qs);  // the first k: a bound for the next tiles
  }
  __syncthreads();
  if (s_n > Q.k) sort_compact(s_key, s_doc, s_n, Q.k, s_theta, s_full, qs);
  if (Q.flags & kSortAllTiles) {
    total = __reduce_add_sync(kFull, total);
    if (lane == 0) s_part[warp] = total;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (Q.flags & kSortAllTiles) {
      unsigned long long sum = 0;
      for (int w = 0; w < kWarps; ++w) sum += s_part[w];
      if (sum) atomicAdd(&P.c.counts[S.query], sum);
    }
    if (P.tiles && seen) { atomicAdd(&P.tiles[0], (unsigned long long)seen); if (skipped) atomicAdd(&P.tiles[1], (unsigned long long)skipped); }
    s_base = s_n ? atomicAdd(&qs->n_cands, s_n) : 0u;
    if (s_full) s_nn = 0;  // k docs with values are known: no None doc can make the top k
    s_nbase = s_nn ? atomicAdd(&qs->n_nones, s_nn) : 0u;
  }
  __syncthreads();
  SortCand* const cands = P.cands + Q.cand_base + s_base;
  for (uint32_t i = threadIdx.x; i < s_n; i += blockDim.x) cands[i] = SortCand{s_key[i], Z.segment_ord, ~s_doc[i]};
  SortCand* const nones = P.nones + Q.cand_base + s_nbase;
  for (uint32_t i = threadIdx.x; i < s_nn; i += blockDim.x) nones[i] = SortCand{0ull, Z.segment_ord, s_none[i]};
}

// The first min(C, k) of C candidates by (a desc, b desc), (a, b) = key(candidate), sorted into s_a / s_b; returns how many.  A
// 64-bit radix select of the k-th largest a (8 passes, as k_final's 4), then the candidates above it and its ties are sorted --
// the ties slab by slab when they do not fit the buffer, as in k_final.
template <class Key>
__device__ uint32_t select_sorted(const SortCand* __restrict__ cands, uint32_t C, uint32_t k, Key key, unsigned long long* s_a,
                                  unsigned long long* s_b, uint32_t* s_hist, unsigned long long& s_prefix, uint32_t& s_need,
                                  uint32_t& s_ties, uint32_t& s_n) {
  if (C <= kCap) {
    for (uint32_t i = threadIdx.x; i < C; i += blockDim.x) key(cands[i], s_a[i], s_b[i]);
    __syncthreads();
    sort_pairs_desc(s_a, s_b, C);
    return min(C, k);
  }
  if (threadIdx.x == 0) { s_prefix = 0; s_need = k; s_n = 0; }
  unsigned long long mask = 0;
  for (int pass = 0; pass < 8; ++pass) {
    const int shift = 56 - 8 * pass;
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    const unsigned long long prefix = s_prefix;
    for (uint32_t i = threadIdx.x; i < C; i += blockDim.x) {
      unsigned long long a, b;
      key(cands[i], a, b);
      if ((a & mask) == prefix) atomicAdd(&s_hist[(a >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t need = s_need, bsel = 0;
      for (int bin = 255; bin >= 0; --bin) {
        const uint32_t h = s_hist[bin];
        if (h >= need) { bsel = (uint32_t)bin; s_ties = h; break; }
        need -= h;
      }
      s_need = need;
      s_prefix = prefix | ((unsigned long long)bsel << shift);
    }
    mask |= 0xFFull << shift;
    __syncthreads();
  }
  const unsigned long long kth = s_prefix;  // exactly the k-th largest a
  const uint32_t ties = s_ties, above = k - s_need;
  const bool one_sweep = above + ties <= kCap;  // the usual case; else a flood of equal a: the ties slab by slab
  for (uint32_t i = threadIdx.x; i < C; i += blockDim.x) {
    unsigned long long a, b;
    key(cands[i], a, b);
    if (one_sweep ? a >= kth : a > kth) {
      const uint32_t slot = atomicAdd(&s_n, 1u);
      s_a[slot] = a;
      s_b[slot] = b;
    }
  }
  __syncthreads();
  uint32_t have = s_n;
  if (one_sweep) {
    __syncthreads();
    sort_pairs_desc(s_a, s_b, have);
    return min(have, k);
  }
  for (uint32_t next = 0; next < C;) {
    __syncthreads();
    if (threadIdx.x == 0) s_n = have;
    __syncthreads();
    const uint32_t slab_end = min(C, next + (kCap - have));
    for (uint32_t i = next + threadIdx.x; i < slab_end; i += blockDim.x) {
      unsigned long long a, b;
      key(cands[i], a, b);
      if (a == kth) {
        const uint32_t slot = atomicAdd(&s_n, 1u);
        s_a[slot] = a;
        s_b[slot] = b;
      }
    }
    __syncthreads();
    const uint32_t n = s_n;
    __syncthreads();
    sort_pairs_desc(s_a, s_b, n);
    have = min(n, k);
    next = slab_end;
  }
  return have;
}

// The rows of every query: its docs with values by (v' desc, segment asc, doc asc), then, while the row has room, its None docs
// by (segment asc, doc asc) (compare_for_top_k, top_score_collector.rs:591-600; Order::Asc = ReverseNoneLower, order.rs:286-293).
__global__ void __launch_bounds__(kThreads) k_sort_final(const SortParams P) {
  __shared__ unsigned long long s_a[kCap], s_b[kCap];
  __shared__ uint32_t s_hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ uint32_t s_need, s_ties, s_n;
  const uint32_t q = blockIdx.x;
  const SortQuery Q = P.queries[q];
  const uint32_t n_cands = P.qstate[q].n_cands, n_nones = P.qstate[q].n_nones;
  const bool asc = (Q.flags & kSortAsc) != 0;
  const size_t row = (size_t)q * P.res_stride;
  auto address = [](const SortCand& c) { return ~((unsigned long long)c.segment_ord << 32 | c.doc); };  // descending = ascending address
  const uint32_t have = select_sorted(P.cands + Q.cand_base, n_cands, Q.k,
                                      [&](const SortCand& c, unsigned long long& a, unsigned long long& b) { a = c.key; b = address(c); },
                                      s_a, s_b, s_hist, s_prefix, s_need, s_ties, s_n);
  for (uint32_t i = threadIdx.x; i < have; i += blockDim.x) {
    const unsigned long long addr = ~s_b[i];
    P.res_values[row + i] = asc ? ~s_a[i] : s_a[i];
    P.res_present[row + i] = 1;
    P.res_segs[row + i] = (uint32_t)(addr >> 32);
    P.res_docs[row + i] = (uint32_t)addr;
  }
  uint32_t n_none = 0;
  if (have < Q.k && n_nones) {
    __syncthreads();
    n_none = select_sorted(P.nones + Q.cand_base, n_nones, Q.k - have,
                           [&](const SortCand& c, unsigned long long& a, unsigned long long& b) { a = b = address(c); },
                           s_a, s_b, s_hist, s_prefix, s_need, s_ties, s_n);
    for (uint32_t i = threadIdx.x; i < n_none; i += blockDim.x) {
      const unsigned long long addr = ~s_b[i];
      P.res_values[row + have + i] = 0;
      P.res_present[row + have + i] = 0;
      P.res_segs[row + have + i] = (uint32_t)(addr >> 32);
      P.res_docs[row + have + i] = (uint32_t)addr;
    }
  }
  if (threadIdx.x == 0) P.res_counts[q] = have + n_none;
}

// ---- histogram of a fast field (AggregationCollector: histogram / date_histogram, bucket/histogram/histogram.rs) ------------
// The docs Count counts, each with a value in its bounds counted in bucket pos(val).  One CTA per Count unit: per 8192-doc tile
// match_tile builds the match bitmap, and-ed with the present bits.  When the tile's smallest and largest values (SortTile) are
// both in bounds and in one bucket, so is every value between them (pos is monotone in the image): the tile's matches go to that
// bucket without a gather.  Otherwise each thread walks the matches of its own 32-doc word: an 8-byte gather, the conversion, the
// bounds test and pos, one counter increment.  A unit counts into its own window of the query's counters (HistUnit: the buckets of
// its tiles' values in bounds), per CTA in shared memory when the window has kHistSmemBins or fewer (flushed with one 64-bit
// atomicAdd per non-zero bucket at exit), else global.  A timestamp unit of eight tiles spans a few minutes of the column, so even a
// query of many thousand buckets counts on chip.

// The body of k_hist, k_terms and k_range: one CTA per Count unit counts its matching docs by key into its window of counters.  K is the
// key policy, static functions over the (query, segment)'s descriptor Z, the query's Q and the unit's window W (from the origin
// `base`): the one key of a tile with values, if it has one (every value of the tile, matching or not, has it: the tile's matches are added without a gather;
// ~0u: none), whether a value is counted and the index of its counter, and whether matching docs without a value are counted as
// well (K::kMissing: one add per warp at exit).
template <class K, bool kMixed, class Params>
__device__ __forceinline__ void count_unit_keys(const Params& P, const uint32_t unit) {
  static_assert(kTileDocs / 32u == (uint32_t)kThreads, "one 32-doc word of a tile per thread");
  __shared__ uint32_t s_acc[kTileDocs / 32u], s_tmp[kTileDocs / 32u];
  __shared__ uint32_t s_cnt[kMixed ? kTileDocs / 4u : 1u];
  __shared__ uint32_t s_bins[kHistSmemBins];
  __shared__ uint32_t s_part[kWarps];
  __shared__ uint32_t s_one;  // the tile's one key (index into the unit's window), or ~0u
  const Unit U = P.c.units[unit];
  const CountSeg S = P.c.segs[U.qseg];
  const typename K::Seg Z = K::seg(P, U);
  const typename K::Query Q = K::query(P, S, Z);
  const uint32_t wb = S.words_base, ng = P.c.words[wb], need = P.c.words[wb + 1u];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const HistUnit W = K::window(P, unit);
  const typename K::Base base = K::base(Z, Q, W);  // the key of the unit's first counter
  const bool shared = W.n_bins <= kHistSmemBins;
  typename K::Counter* const counts = K::counts(P, Z, Q, W);
  if (shared)
    for (uint32_t i = threadIdx.x; i < W.n_bins; i += blockDim.x) s_bins[i] = 0;
  uint32_t total = 0, one = 0, missing = 0;
  for (uint32_t tile = U.begin; tile < U.end; ++tile) {
    const uint32_t lo = tile * kTileDocs, hi = min(lo + kTileDocs, S.max_doc);
    if (threadIdx.x == 0) {
      const SortTile T = Z.tiles[tile];
      uint32_t idx = 0xFFFFFFFFu;
      if (W.n_bins && (T.flags & kSortTileValues)) K::one(T, Z, Q, W, base, idx);
      s_one = idx;
      one += idx != 0xFFFFFFFFu ? 1u : 0u;
    }
    match_tile<kMixed>(P.c, S.alive, wb, ng, need, lo, hi, s_acc, s_tmp, s_cnt, [&](uint32_t w, uint32_t bits) { s_acc[w] = bits; });
    __syncthreads();
    const uint32_t bits = s_acc[threadIdx.x];
    total += (uint32_t)__popc(bits);
    uint32_t with = Z.present ? bits & __ldg(Z.present + (lo >> 5) + threadIdx.x) : bits;
    if constexpr (K::kMissing) missing += (uint32_t)__popc(bits ^ with);
    if (s_one < W.n_bins) {
      const uint32_t c = __reduce_add_sync(kFull, (uint32_t)__popc(with));
      const uint32_t idx = s_one;
      if (lane == 0 && c) {
        if (shared) atomicAdd(&s_bins[idx], c);
        else atomicAdd(&counts[idx], (typename K::Counter)c);
      }
    } else if (W.n_bins) {
      for (; with; with &= with - 1u) {
        const uint32_t doc = lo + threadIdx.x * 32u + (uint32_t)(__ffs(with) - 1);
        const typename K::Value val = K::value(__ldg(Z.values + doc), Q);
        if (!K::counted(val, Z)) continue;
        const unsigned long long idx = K::index(val, Q, base);
        if (idx < W.n_bins) {  // (always: the window covers every counted value of the unit's tiles)
          if (shared) atomicAdd(&s_bins[idx], 1u);
          else atomicAdd(&counts[idx], (typename K::Counter)1);
        }
      }
    }
    __syncthreads();
  }
  if (shared)
    for (uint32_t i = threadIdx.x; i < W.n_bins; i += blockDim.x)
      if (s_bins[i]) atomicAdd(&counts[i], (typename K::Counter)s_bins[i]);
  if (K::hits(Q)) {
    total = __reduce_add_sync(kFull, total);
    if (lane == 0) s_part[warp] = total;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (K::hits(Q)) {
      unsigned long long sum = 0;
      for (int w = 0; w < kWarps; ++w) sum += s_part[w];
      if (sum) atomicAdd(&P.c.counts[S.query], sum);
    }
    const uint32_t seen = U.end - U.begin;
    if (seen) { atomicAdd(&P.tiles[0], (unsigned long long)seen); if (one) atomicAdd(&P.tiles[1], (unsigned long long)one); }
  }
  if constexpr (K::kMissing) {
    if (Z.flags & kTermsMissing) {
      missing = __reduce_add_sync(kFull, missing);
      if (lane == 0 && missing) atomicAdd(&P.missing[U.qseg - P.seg_base], missing);
    }
  }
}

// The histogram's keys: bucket pos(val) of the values in the (query, segment)'s bounds.
struct HistKeys {
  typedef HistSeg Seg;
  typedef HistQuery Query;
  typedef long long Base;
  typedef double Value;
  typedef unsigned long long Counter;
  static constexpr bool kMissing = false;
  // (Params: HistParams for k_hist, HistMetricsParams for k_hist_metrics)
  template <class Params> static __device__ __forceinline__ HistSeg seg(const Params& P, const Unit& U) { return P.hsegs[U.qseg]; }
  template <class Params> static __device__ __forceinline__ HistQuery query(const Params& P, const CountSeg& S, const HistSeg&) { return P.queries[S.query]; }
  template <class Params> static __device__ __forceinline__ HistUnit window(const Params& P, uint32_t unit) { return P.hunits[unit]; }
  static __device__ __forceinline__ long long base(const HistSeg&, const HistQuery& Q, const HistUnit& W) { return Q.base + (long long)W.first; }
  template <class Params> static __device__ __forceinline__ Counter* counts(const Params& P, const HistSeg&, const HistQuery& Q, const HistUnit& W) { return P.counts + Q.counters + W.first; }
  // the window's first counter in the wave (k_hist_metrics: its parts are kMetricsMaxColumns per counter)
  static __device__ __forceinline__ unsigned long long slot(const HistSeg&, const HistQuery& Q, const HistUnit& W) { return Q.counters + W.first; }
  // one bucket: the tile's smallest and largest values both in bounds and in one bucket (pos is monotone in the image)
  static __device__ __forceinline__ void one(const SortTile T, const HistSeg& Z, const HistQuery& Q, const HistUnit& W, const long long base, uint32_t& idx) {
    const double vmin = hist_value(~T.best[1], Q.kind), vmax = hist_value(T.best[0], Q.kind);
    if (vmin >= Z.lo && vmax <= Z.hi) {
      const long long p = hist_pos(vmin, Q.offset, Q.interval);
      if (p == hist_pos(vmax, Q.offset, Q.interval) && p >= base && p - base < (long long)W.n_bins) idx = (uint32_t)(p - base);
    }
  }
  static __device__ __forceinline__ double value(unsigned long long v, const HistQuery& Q) { return hist_value(v, Q.kind); }
  static __device__ __forceinline__ bool counted(double val, const HistSeg& Z) {
    return val >= Z.lo && val <= Z.hi;  // HistogramBounds::contains (NaN never passes)
  }
  static __device__ __forceinline__ unsigned long long index(double val, const HistQuery& Q, long long base) {
    return (unsigned long long)(hist_pos(val, Q.offset, Q.interval) - base);
  }
  static __device__ __forceinline__ bool hits(const HistQuery& Q) { return Q.flags & kHistHits; }
};

// (3 CTAs per SM: the division's slow path is a call, and at the 64 registers of 4 CTAs the kernel spills around it)
template <bool kMixed>
__global__ void __launch_bounds__(kThreads, 3) k_hist(const HistParams P) {
  count_unit_keys<HistKeys, kMixed>(P, blockIdx.x);
}

// One CTA per query: the non-zero counters of its range, in ascending pos, into its row (a CTA-wide prefix sum per 256 counters).
__global__ void __launch_bounds__(kThreads) k_hist_final(const HistParams P) {
  __shared__ uint32_t s_part[kWarps];
  const uint32_t q = blockIdx.x;
  const HistQuery Q = P.queries[q];
  const unsigned long long* const counts = P.counts + Q.counters;
  const size_t row = (size_t)q * P.res_stride;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t base = 0;  // non-empty buckets before this round of counters (the same on every thread)
  for (uint32_t i0 = 0; i0 < Q.n_bins; i0 += blockDim.x) {
    const uint32_t i = i0 + threadIdx.x;
    const unsigned long long c = i < Q.n_bins ? counts[i] : 0ull;
    const uint32_t mask = __ballot_sync(kFull, c != 0ull);
    if (lane == 0) s_part[warp] = (uint32_t)__popc(mask);
    __syncthreads();
    uint32_t at = base + (uint32_t)__popc(mask & ((1u << lane) - 1u));
    for (uint32_t w = 0; w < warp; ++w) at += s_part[w];
    if (c && at < P.res_stride) {
      P.res_pos[row + at] = Q.base + (long long)i;
      P.res_count[row + at] = c;
    }
    for (int w = 0; w < kWarps; ++w) base += s_part[w];
    __syncthreads();
  }
  if (threadIdx.x == 0) P.res_n[q] = base;
}

// ---- terms of a fast field (AggregationCollector: terms, bucket/term_agg/mod.rs) ---------------------------------------------
// The docs Count counts, each counted under its image, through count_unit_keys: a tile whose smallest and largest image are equal
// adds its matches to that key without a gather, a matching doc without a value goes to the (query, segment)'s missing counter.
struct TermsKeys {
  typedef TermsSeg Seg;
  typedef uint32_t Query;  // the (query, segment)'s flags
  typedef unsigned long long Base;
  typedef unsigned long long Value;
  typedef uint32_t Counter;  // Bucket::count is a u32
  static constexpr bool kMissing = true;
  static __device__ __forceinline__ TermsSeg seg(const TermsParams& P, const Unit& U) { return P.tsegs[U.qseg]; }
  static __device__ __forceinline__ uint32_t query(const TermsParams&, const CountSeg&, const TermsSeg& Z) { return Z.flags; }
  static __device__ __forceinline__ HistUnit window(const TermsParams& P, uint32_t unit) { return P.windows[unit]; }
  static __device__ __forceinline__ unsigned long long base(const TermsSeg& Z, uint32_t, const HistUnit& W) { return Z.base + W.first; }
  static __device__ __forceinline__ Counter* counts(const TermsParams& P, const TermsSeg& Z, uint32_t, const HistUnit& W) { return P.counts + Z.counters + W.first; }
  static __device__ __forceinline__ void one(const SortTile T, const TermsSeg&, uint32_t, const HistUnit& W, const unsigned long long base, uint32_t& idx) {
    if (T.best[0] == ~T.best[1] && T.best[0] - base < W.n_bins) idx = (uint32_t)(T.best[0] - base);
  }
  static __device__ __forceinline__ unsigned long long value(unsigned long long v, uint32_t) { return v; }
  static __device__ __forceinline__ bool counted(unsigned long long, const TermsSeg&) { return true; }
  static __device__ __forceinline__ unsigned long long index(unsigned long long v, uint32_t, unsigned long long base) { return v - base; }
  static __device__ __forceinline__ bool hits(uint32_t flags) { return flags & kTermsHits; }
};

// (4 CTAs per SM: no division here, and the 64 registers hold the loop without spilling)
template <bool kMixed>
__global__ void __launch_bounds__(kThreads, 4) k_terms(const TermsParams P) {
  count_unit_keys<TermsKeys, kMixed>(P, P.unit_base + blockIdx.x);
}

// ---- range of a fast field (AggregationCollector: range, bucket/range.rs) -------------------------------------------------
// The docs Count counts, each with a value counted in range bucket b = the last start <= its image (get_bucket_pos: a binary search
// over the starts, the end never tested), through count_unit_keys.  The image alone decides the bucket: no conversion, no division.
// A tile whose smallest and largest images land in one bucket adds its matches there without a gather; a doc without a value is not
// collected (range has no `missing`).  The window is the query's whole bucket list.
struct RangeKeys {
  typedef RangeSeg Seg;
  typedef RangeQuery Query;
  typedef uint32_t Base;  // (0: the window starts at the query's first bucket)
  typedef unsigned long long Value;
  typedef unsigned long long Counter;
  static constexpr bool kMissing = false;
  // (Params: RangeParams for k_range, RangeMetricsParams for k_range_metrics)
  template <class Params> static __device__ __forceinline__ RangeSeg seg(const Params& P, const Unit& U) { return P.rsegs[U.qseg]; }
  template <class Params> static __device__ __forceinline__ RangeQuery query(const Params& P, const CountSeg& S, const RangeSeg&) { return P.queries[S.query]; }
  template <class Params> static __device__ __forceinline__ HistUnit window(const Params& P, uint32_t unit) { return P.windows[unit]; }
  static __device__ __forceinline__ uint32_t base(const RangeSeg&, const RangeQuery&, const HistUnit&) { return 0u; }
  template <class Params> static __device__ __forceinline__ Counter* counts(const Params& P, const RangeSeg&, const RangeQuery& Q, const HistUnit&) { return P.counts + Q.counters; }
  static __device__ __forceinline__ unsigned long long slot(const RangeSeg&, const RangeQuery& Q, const HistUnit&) { return Q.counters; }
  // upper bound over the starts (through the read-only cache): the last b with starts[b] <= v; starts[0] == 0, so always one.  At
  // most 7 steps for kRangeMaxBins buckets.
  static __device__ __forceinline__ uint32_t bucket(const unsigned long long v, const RangeQuery& Q) {
    uint32_t lo = 0, n = Q.n_bins;
    while (n > 1u) {
      const uint32_t half = n >> 1;
      if (__ldg(Q.starts + lo + half) <= v) lo += half;
      n -= half;
    }
    return lo;
  }
  // one bucket: the tile's smallest and largest images in the same one (the bucket is monotone in the image)
  static __device__ __forceinline__ void one(const SortTile T, const RangeSeg&, const RangeQuery& Q, const HistUnit&, uint32_t, uint32_t& idx) {
    const uint32_t b = bucket(~T.best[1], Q);
    if (b == bucket(T.best[0], Q)) idx = b;
  }
  static __device__ __forceinline__ unsigned long long value(unsigned long long v, const RangeQuery&) { return v; }
  static __device__ __forceinline__ bool counted(unsigned long long, const RangeSeg&) { return true; }
  static __device__ __forceinline__ unsigned long long index(unsigned long long v, const RangeQuery& Q, uint32_t) { return bucket(v, Q); }
  static __device__ __forceinline__ bool hits(const RangeQuery& Q) { return Q.flags & kRangeHits; }
};

// (4 CTAs per SM: the search is a few compares and loads, and the 64 registers hold the loop without spilling)
template <bool kMixed>
__global__ void __launch_bounds__(kThreads, 4) k_range(const RangeParams P) {
  count_unit_keys<RangeKeys, kMixed>(P, blockIdx.x);
}

// Exclusive CTA-wide prefix sum of v (fields packed in v add independently while each total fits its field); *total = the sum.
__device__ __forceinline__ uint32_t cta_scan_excl(const uint32_t v, uint32_t* s_part, uint32_t& total) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (uint32_t d = 1; d < 32u; d <<= 1) {
    const uint32_t y = __shfl_up_sync(kFull, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31u) s_part[warp] = x;
  __syncthreads();
  uint32_t before = 0, sum = 0;
  for (int w = 0; w < kWarps; ++w) {
    const uint32_t p = s_part[w];
    before += w < (int)warp ? p : 0u;
    sum += p;
  }
  __syncthreads();
  total = sum;
  return before + x - v;
}

// One CTA per (query, segment) of a wave: the segment's cut (into_intermediate_bucket_result + cut_off_buckets).  A missing key
// inside the counters' range is folded into its counter; one outside it is one more entry, before or after them in key order.  The
// entries are the non-zero ones.  More than segment_size of them: by count, a radix select (4 passes of 8 bits) finds the count t
// of the segment_size-th entry (t over ~count for asc: the segment_size-th largest t either way) and the entries beyond it are kept
// with the lowest keys at t; by key, the first or last segment_size entries.  The kept entries go to the region in ascending key.
__global__ void __launch_bounds__(kThreads) k_terms_select(const TermsParams P) {
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_part[kWarps];
  __shared__ unsigned long long s_wide[kWarps];
  __shared__ uint32_t s_sel[3];  // the select's prefix, the rank left within it, the entries equal to it
  __shared__ uint32_t s_error;
  const uint32_t rel = blockIdx.x;
  const TermsSeg Z = P.tsegs[P.seg_base + rel];
  uint32_t* const cnt = P.counts + Z.counters;
  const uint32_t n = Z.n_keys, ss = Z.segment_size;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t mc = (Z.flags & kTermsMissing) ? P.missing[rel] : 0u;
  const bool inside = mc && Z.missing - Z.base < (unsigned long long)n;
  const uint32_t extra = mc && !inside ? 1u : 0u, off = extra && Z.missing < Z.base ? 1u : 0u;
  if (inside && threadIdx.x == 0) cnt[Z.missing - Z.base] += mc;
  __syncthreads();
  const uint32_t L = n + extra;  // entries in key order: [missing,] counters[0..n) [, missing]
  auto count_at = [&](uint32_t i) -> uint32_t { i -= off; return i < n ? cnt[i] : mc; };
  auto key_at = [&](uint32_t i) -> unsigned long long { i -= off; return i < n ? Z.base + i : Z.missing; };
  const bool asc = Z.flags & kTermsAsc, by_key = Z.flags & kTermsByKey;
  auto rank_key = [&](uint32_t c) -> uint32_t { return asc ? ~c : c; };  // larger first
  // the entries and their doc count
  uint32_t nz = 0;
  unsigned long long sum = 0;
  for (uint32_t i = threadIdx.x; i < L; i += blockDim.x) {
    const uint32_t c = count_at(i);
    nz += c ? 1u : 0u;
    sum += c;
  }
  nz = __reduce_add_sync(kFull, nz);
  for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(kFull, sum, d);
  if (lane == 0) { s_part[warp] = nz; s_wide[warp] = sum; }
  __syncthreads();
  uint32_t N = 0;
  unsigned long long total = 0;
  for (int w = 0; w < kWarps; ++w) { N += s_part[w]; total += s_wide[w]; }
  __syncthreads();
  const bool cut = N > ss;
  uint32_t t_cut = 0, need = 0;
  if (cut && !by_key) {
    uint32_t prefix = 0, mask = 0, k = ss;
    for (int shift = 24; shift >= 0; shift -= 8) {
      s_hist[threadIdx.x] = 0;
      __syncthreads();
      for (uint32_t i = threadIdx.x; i < L; i += blockDim.x) {
        const uint32_t c = count_at(i);
        const uint32_t t = rank_key(c);
        if (c && (t & mask) == prefix) atomicAdd(&s_hist[(t >> shift) & 255u], 1u);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        uint32_t b = 255, acc = 0;
        for (; acc + s_hist[b] < k; --b) acc += s_hist[b];
        s_sel[0] = prefix | (b << shift);
        s_sel[1] = k - acc;
        s_sel[2] = s_hist[b];
      }
      __syncthreads();
      prefix = s_sel[0];
      k = s_sel[1];
      mask |= 255u << shift;
      __syncthreads();
    }
    t_cut = prefix;
    need = k;  // entries at t_cut to keep, the lowest keys first
    // term_doc_count_before_cutoff: t_cut itself when more entries tie at it, else the largest t below it
    if (threadIdx.x == 0) s_error = s_sel[2] > need ? t_cut : 0u;
    uint32_t below = 0;
    const bool more = s_sel[2] > need;
    __syncthreads();
    if (!more) {
      for (uint32_t i = threadIdx.x; i < L; i += blockDim.x) {
        const uint32_t c = count_at(i);
        const uint32_t t = rank_key(c);
        if (c && t < t_cut) below = max(below, t);
      }
      below = __reduce_max_sync(kFull, below);
      if (lane == 0) atomicMax(&s_error, below);
    }
    __syncthreads();
    if (threadIdx.x == 0) s_error = rank_key(s_error);
  } else if (threadIdx.x == 0) {
    s_error = 0;
  }
  __syncthreads();
  // by key: the entry ranks kept and the rank whose count is reported
  const uint32_t r0 = cut && by_key && !asc ? N - ss : 0u, r_err = cut && by_key ? (asc ? ss : N - ss - 1u) : 0xFFFFFFFFu;
  uint32_t base_nz = 0, base_eq = 0, base_keep = 0;
  unsigned long long kept = 0;
  for (uint32_t i0 = 0; i0 < L; i0 += blockDim.x) {
    const uint32_t i = i0 + threadIdx.x;
    const uint32_t c = i < L ? count_at(i) : 0u;
    const bool eq = c && cut && !by_key && rank_key(c) == t_cut;
    uint32_t tot;
    const uint32_t ex = cta_scan_excl((c ? 1u : 0u) | (eq ? 1u << 16 : 0u), s_part, tot);
    const uint32_t r_nz = base_nz + (ex & 0xFFFFu), r_eq = base_eq + (ex >> 16);
    base_nz += tot & 0xFFFFu;
    base_eq += tot >> 16;
    bool keep = c != 0;
    if (cut) keep = keep && (by_key ? r_nz - r0 < ss : (rank_key(c) > t_cut || (eq && r_eq < need)));
    if (c && r_nz == r_err) s_error = c;
    const uint32_t at = base_keep + cta_scan_excl(keep ? 1u : 0u, s_part, tot);
    base_keep += tot;
    if (keep) {
      P.res_key[Z.region + at] = key_at(i);
      P.res_count[Z.region + at] = c;
      kept += c;
    }
  }
  for (int d = 16; d; d >>= 1) kept += __shfl_xor_sync(kFull, kept, d);
  if (lane == 0) s_wide[warp] = kept;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long k_sum = 0;
    for (int w = 0; w < kWarps; ++w) k_sum += s_wide[w];
    P.res_n[rel] = base_keep;
    P.res_other[rel] = total - k_sum;
    P.res_error[rel] = cut ? s_error : 0u;
  }
}

// ---- metrics of fast fields (AggregationCollector: avg / sum / min / max / stats / value_count, metric/stats.rs) -------------
// The docs Count counts, each collecting its value in every column of the query's spec: one match pass feeds up to four columns.
// One CTA per Count unit: per 8192-doc tile match_tile builds the match bitmap; per column, a tile whose smallest and largest images
// are equal (SortTile: every value of the tile, matching or not, is that one) adds popc(match & present) copies of its value
// without a gather, any other tile has each thread walk the matches of its own 32-doc word with one 8-byte gather per doc.  A
// count-only column is never read, and an empty one (TQ_METRIC_EMPTY) has no value in any doc.  Matching docs without a value are counted per thread and added at exit as copies of the
// missing value.  The accumulators of the four columns live in registers per thread; NaN and +-inf, which only ever decide a
// refusal, are counted in shared memory.  At exit each quantity is reduced per warp, then per CTA, and flushed with one set of
// atomics per (unit, column).  Every add is one f64 operation on exact operands, so under the guard (tantivy_b200.h) every
// partial sum is exact and the order of the adds and atomics cannot change the result.
struct MetricAcc {
  unsigned long long lo, hi;  // smallest / largest image of the non-NaN values
  double sum, mag;            // sum and sum of |v| of the finite values
  uint32_t count, missing;    // values seen; matching docs without a value
  int q;                      // least exponent of the lowest set bit of a finite non-zero value
};

// n copies of the value of `image`
__device__ __forceinline__ void metric_add(MetricAcc& a, const unsigned long long image, const uint32_t kind, const uint32_t n,
                                           uint32_t* s_nan_inf) {
  const double v = hist_value(image, kind);
  if (v != v) { atomicAdd(&s_nan_inf[0], n); return; }
  a.lo = min(a.lo, image);
  a.hi = max(a.hi, image);
  const double av = fabs(v);
  if (av == INFINITY) { atomicAdd(&s_nan_inf[1], n); return; }
  a.sum = __dadd_rn(a.sum, __dmul_rn((double)n, v));
  a.mag = __dadd_rn(a.mag, __dmul_rn((double)n, av));
  if (av != 0.0) a.q = min(a.q, metric_quantum_exp((unsigned long long)__double_as_longlong(av)));
}

template <bool kMixed>
__global__ void __launch_bounds__(kThreads) k_metrics(const MetricsParams P) {
  static_assert(kTileDocs / 32u == (uint32_t)kThreads, "one 32-doc word of a tile per thread");
  static_assert(sizeof(MetricsSeg) % 8u == 0 && sizeof(MetricsSeg) / 8u <= (uint32_t)kThreads, "one word of the descriptor per thread");
  constexpr uint32_t kC = kMetricsMaxColumns;
  __shared__ uint32_t s_acc[kTileDocs / 32u], s_tmp[kTileDocs / 32u];
  __shared__ uint32_t s_cnt[kMixed ? kTileDocs / 4u : 1u];
  __shared__ MetricsSeg s_z;
  __shared__ unsigned long long s_one[kC];  // per column: the tile's one image, when s_has_one
  __shared__ uint32_t s_has_one[kC];
  __shared__ uint32_t s_nan_inf[kC][2];
  __shared__ unsigned long long s_lo[kWarps][kC], s_hi[kWarps][kC];
  __shared__ double s_sum[kWarps][kC], s_mag[kWarps][kC];
  __shared__ uint32_t s_count[kWarps][kC], s_part[kWarps];
  __shared__ int s_q[kWarps][kC];
  const Unit U = P.c.units[blockIdx.x];
  const CountSeg S = P.c.segs[U.qseg];
  if (threadIdx.x < sizeof(MetricsSeg) / 8u)
    reinterpret_cast<unsigned long long*>(&s_z)[threadIdx.x] = reinterpret_cast<const unsigned long long*>(P.msegs + U.qseg)[threadIdx.x];
  if (threadIdx.x < 2u * kC) (&s_nan_inf[0][0])[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t nc = s_z.n_columns;
  const uint32_t wb = S.words_base, ng = P.c.words[wb], need = P.c.words[wb + 1u];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  MetricAcc acc[kC];
#pragma unroll
  for (uint32_t c = 0; c < kC; ++c) acc[c] = MetricAcc{~0ull, 0ull, 0.0, 0.0, 0u, 0u, INT32_MAX};
  uint32_t total = 0, one = 0, seen = 0;
  for (uint32_t tile = U.begin; tile < U.end; ++tile) {
    const uint32_t lo = tile * kTileDocs, hi = min(lo + kTileDocs, S.max_doc);
    if (threadIdx.x < nc) {  // (warp 0)
      const MetricsCol& C = s_z.col[threadIdx.x];
      uint32_t has = 0;
      if (!(C.flags & (TQ_METRIC_COUNT_ONLY | TQ_METRIC_EMPTY))) {
        const SortTile T = C.tiles[tile];
        has = (T.flags & kSortTileValues) && T.best[0] == ~T.best[1] ? 1u : 0u;
        s_one[threadIdx.x] = T.best[0];
        ++seen;
        one += has;
      }
      s_has_one[threadIdx.x] = has;
    }
    match_tile<kMixed>(P.c, S.alive, wb, ng, need, lo, hi, s_acc, s_tmp, s_cnt, [&](uint32_t w, uint32_t bits) { s_acc[w] = bits; });
    __syncthreads();
    const uint32_t bits = s_acc[threadIdx.x];
    total += (uint32_t)__popc(bits);
#pragma unroll
    for (uint32_t c = 0; c < kC; ++c) {
      if (c >= nc) break;
      const MetricsCol& C = s_z.col[c];
      const uint32_t with = (C.flags & TQ_METRIC_EMPTY) ? 0u : C.present ? bits & __ldg(C.present + (lo >> 5) + threadIdx.x) : bits;
      const uint32_t n = (uint32_t)__popc(with);
      acc[c].count += n;
      acc[c].missing += (uint32_t)__popc(bits ^ with);
      if (C.flags & (TQ_METRIC_COUNT_ONLY | TQ_METRIC_EMPTY)) continue;
      if (s_has_one[c]) {
        if (n) metric_add(acc[c], s_one[c], C.kind, n, s_nan_inf[c]);
      } else {
        for (uint32_t m = with; m; m &= m - 1u) {
          const uint32_t doc = lo + threadIdx.x * 32u + (uint32_t)(__ffs(m) - 1);
          metric_add(acc[c], __ldg(C.values + doc), C.kind, 1u, s_nan_inf[c]);
        }
      }
    }
    __syncthreads();
  }
  // missing values, then the warp's figures
#pragma unroll
  for (uint32_t c = 0; c < kC; ++c) {
    if (c >= nc) break;
    const MetricsCol& C = s_z.col[c];
    if ((C.flags & TQ_METRIC_MISSING) && acc[c].missing) {
      acc[c].count += acc[c].missing;
      if (!(C.flags & TQ_METRIC_COUNT_ONLY)) metric_add(acc[c], C.missing, C.kind, acc[c].missing, s_nan_inf[c]);
    }
    uint32_t count = __reduce_add_sync(kFull, acc[c].count);
    int q = __reduce_min_sync(kFull, acc[c].q);
    unsigned long long vlo = acc[c].lo, vhi = acc[c].hi;
    double sum = acc[c].sum, mag = acc[c].mag;
#pragma unroll
    for (int d = 16; d; d >>= 1) {
      vlo = min(vlo, __shfl_xor_sync(kFull, vlo, d));
      vhi = max(vhi, __shfl_xor_sync(kFull, vhi, d));
      sum = __dadd_rn(sum, __shfl_xor_sync(kFull, sum, d));
      mag = __dadd_rn(mag, __shfl_xor_sync(kFull, mag, d));
    }
    if (lane == 0) {
      s_count[warp][c] = count;
      s_q[warp][c] = q;
      s_lo[warp][c] = vlo;
      s_hi[warp][c] = vhi;
      s_sum[warp][c] = sum;
      s_mag[warp][c] = mag;
    }
  }
  if (warp == 0) {
    one = __reduce_add_sync(kFull, one);
    seen = __reduce_add_sync(kFull, seen);
  }
  total = __reduce_add_sync(kFull, total);
  if (lane == 0) s_part[warp] = total;
  __syncthreads();
  if (threadIdx.x < nc) {  // one set of atomics per (unit, column)
    const uint32_t c = threadIdx.x;
    unsigned long long count = 0, vlo = ~0ull, vhi = 0;
    double sum = 0.0, mag = 0.0;
    int q = INT32_MAX;
    for (int w = 0; w < kWarps; ++w) {
      count += s_count[w][c];
      q = min(q, s_q[w][c]);
      vlo = min(vlo, s_lo[w][c]);
      vhi = max(vhi, s_hi[w][c]);
      sum = __dadd_rn(sum, s_sum[w][c]);
      mag = __dadd_rn(mag, s_mag[w][c]);
    }
    tq_metric_part* const out = P.parts + (size_t)S.query * kC + c;
    if (count) {
      atomicAdd(reinterpret_cast<unsigned long long*>(&out->count), count);
      if (s_nan_inf[c][0]) atomicAdd(reinterpret_cast<unsigned long long*>(&out->n_nan), (unsigned long long)s_nan_inf[c][0]);
      if (s_nan_inf[c][1]) atomicAdd(reinterpret_cast<unsigned long long*>(&out->n_inf), (unsigned long long)s_nan_inf[c][1]);
      if (vlo <= vhi) {
        atomicMin(reinterpret_cast<unsigned long long*>(&out->min_image), vlo);
        atomicMax(reinterpret_cast<unsigned long long*>(&out->max_image), vhi);
      }
      atomicAdd(&out->sum, sum);
      atomicAdd(&out->magnitude, mag);
      if (q != INT32_MAX) atomicMin(&out->quantum_exp, q);
    }
  }
  if (threadIdx.x == 0) {
    if (s_z.flags & kMetricsHits) {
      unsigned long long hits = 0;
      for (int w = 0; w < kWarps; ++w) hits += s_part[w];
      if (hits) atomicAdd(&P.c.counts[S.query], hits);
    }
    if (seen) { atomicAdd(&P.tiles[0], (unsigned long long)seen); if (one) atomicAdd(&P.tiles[1], (unsigned long long)one); }
  }
}

// ---- metrics per histogram bucket (histogram / date_histogram with metric sub-aggregations, histogram.rs:490-505) -------------
// The docs k_hist counts, each feeding the metric columns of the (query, segment)'s MetricsSeg in its bucket.  One CTA per Count
// unit on match_tile.  A tile whose values are all in bounds and in one bucket (HistKeys::one) accumulates as k_metrics does, in
// registers, with its one-value tiles and missing copies; the registers carry over consecutive tiles of that bucket (the bucket is
// CTA-uniform there) and are reduced per warp, then per CTA, and flushed with one set of atomics per (run of tiles, column) when
// the bucket changes or the unit ends.  Any other tile has each thread walk the matches of its own 32-doc word: a gather of the
// histogram value, the bounds test and pos (hist_value / hist_pos, as k_hist), then per column a gather and atomics on that
// bucket's accumulators.  A unit's window of kHistMetricsSmemBins or fewer buckets lives in shared memory and is flushed per
// non-empty bucket at exit; a wider one goes to global memory.  The accumulators are tq_metric_parts with min_image and
// quantum_exp stored complemented (~min_image, INT32_MAX - quantum_exp as u32), so that zeroed memory is an empty part and every
// field merges with an add or a max; k_hist_metrics_final undoes the complement.  As in k_metrics every add is one f64 operation
// on exact operands, so under the guard, applied per (bucket, column), the order of the adds cannot change the result.
__device__ __forceinline__ void hm_merge(tq_metric_part* p, const unsigned long long count, const unsigned long long n_nan,
                                         const unsigned long long n_inf, const unsigned long long lo, const unsigned long long hi,
                                         const double sum, const double mag, const int q) {
  if (!count) return;
  atomicAdd(reinterpret_cast<unsigned long long*>(&p->count), count);
  if (n_nan) atomicAdd(reinterpret_cast<unsigned long long*>(&p->n_nan), n_nan);
  if (n_inf) atomicAdd(reinterpret_cast<unsigned long long*>(&p->n_inf), n_inf);
  if (lo <= hi) {
    atomicMax(reinterpret_cast<unsigned long long*>(&p->min_image), ~lo);
    atomicMax(reinterpret_cast<unsigned long long*>(&p->max_image), hi);
  }
  if (mag != 0.0) {  // (finite values all +-0 add nothing to a sum that starts at +0)
    atomicAdd(&p->sum, sum);
    atomicAdd(&p->magnitude, mag);
  }
  if (q != INT32_MAX) atomicMax(reinterpret_cast<unsigned*>(&p->quantum_exp), 0x7FFFFFFFu - (unsigned)q);
}

// one doc of one column into its bucket's accumulator: its value, the missing value, or (count-only) just the count
__device__ __forceinline__ void hm_collect(tq_metric_part* p, const MetricsCol& C, const uint32_t doc, const bool has) {
  if (!has && !(C.flags & TQ_METRIC_MISSING)) return;
  if (C.flags & TQ_METRIC_COUNT_ONLY) {
    atomicAdd(reinterpret_cast<unsigned long long*>(&p->count), 1ull);
    return;
  }
  const unsigned long long image = has ? __ldg(C.values + doc) : C.missing;
  const double v = hist_value(image, C.kind);
  if (v != v) { hm_merge(p, 1ull, 1ull, 0ull, ~0ull, 0ull, 0.0, 0.0, INT32_MAX); return; }
  const double av = fabs(v);
  if (av == INFINITY) { hm_merge(p, 1ull, 0ull, 1ull, image, image, 0.0, 0.0, INT32_MAX); return; }
  hm_merge(p, 1ull, 0ull, 0ull, image, image, v, av, av != 0.0 ? metric_quantum_exp((unsigned long long)__double_as_longlong(av)) : INT32_MAX);
}

// one counted doc of a straddling tile: its bucket's doc counter and every column (cw: the thread's present words per column)
template <class Docs>
__device__ __forceinline__ void hm_doc(Docs* docs, tq_metric_part* parts, const MetricsSeg& z, const uint32_t* cw, const uint32_t doc,
                                       const uint32_t bit) {
  atomicAdd(docs, (Docs)1);
#pragma unroll
  for (uint32_t c = 0; c < kMetricsMaxColumns; ++c) {
    if (c >= z.n_columns) break;
    hm_collect(parts + c, z.col[c], doc, (cw[c] >> bit) & 1u);
  }
}

// The body of k_hist_metrics and k_range_metrics, over the key policy K of count_unit_keys (its seg, query, window, base, counts,
// one, value, counted, index and hits, and slot: the window's first counter, whose parts are kMetricsMaxColumns per counter).
template <class K, bool kMixed, class Params>
__device__ __forceinline__ void metrics_unit_keys(const Params& P) {
  static_assert(kTileDocs / 32u == (uint32_t)kThreads, "one 32-doc word of a tile per thread");
  static_assert(sizeof(MetricsSeg) % 8u == 0 && sizeof(MetricsSeg) / 8u <= (uint32_t)kThreads, "one word of the descriptor per thread");
  constexpr uint32_t kC = kMetricsMaxColumns;
  __shared__ uint32_t s_acc[kTileDocs / 32u], s_tmp[kTileDocs / 32u];
  __shared__ uint32_t s_cnt[kMixed ? kTileDocs / 4u : 1u];
  __shared__ MetricsSeg s_z;
  __shared__ tq_metric_part s_parts[kHistMetricsSmemBins * kC];  // the window's accumulators, when it fits
  __shared__ uint32_t s_docs[kHistMetricsSmemBins];
  __shared__ unsigned long long s_one[kC];  // per column: the tile's one image, when s_has_one
  __shared__ uint32_t s_has_one[kC];
  __shared__ uint32_t s_bucket;             // the tile's one bucket (index into the window), or ~0u
  __shared__ uint32_t s_nan_inf[kC][2];     // the run's NaN and +-inf values per column
  __shared__ unsigned long long s_lo[kWarps][kC], s_hi[kWarps][kC];
  __shared__ double s_sum[kWarps][kC], s_mag[kWarps][kC];
  __shared__ uint32_t s_count[kWarps][kC], s_part[kWarps], s_rdocs[kWarps];
  __shared__ int s_q[kWarps][kC];
  const uint32_t unit = P.unit_base + blockIdx.x;
  const Unit U = P.c.units[unit];
  const CountSeg S = P.c.segs[U.qseg];
  const typename K::Seg Z = K::seg(P, U);
  const typename K::Query Q = K::query(P, S, Z);
  const HistUnit W = K::window(P, unit);
  if (threadIdx.x < sizeof(MetricsSeg) / 8u)
    reinterpret_cast<unsigned long long*>(&s_z)[threadIdx.x] = reinterpret_cast<const unsigned long long*>(P.msegs + U.qseg)[threadIdx.x];
  if (threadIdx.x < 2u * kC) (&s_nan_inf[0][0])[threadIdx.x] = 0;
  const bool shared = W.n_bins <= kHistMetricsSmemBins;
  if (shared) {
    for (uint32_t i = threadIdx.x; i < W.n_bins * (uint32_t)(sizeof(tq_metric_part) / 8u) * kC; i += blockDim.x)
      reinterpret_cast<unsigned long long*>(s_parts)[i] = 0ull;
    for (uint32_t i = threadIdx.x; i < W.n_bins; i += blockDim.x) s_docs[i] = 0;
  }
  __syncthreads();
  const uint32_t nc = s_z.n_columns;
  const uint32_t wb = S.words_base, ng = P.c.words[wb], need = P.c.words[wb + 1u];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const typename K::Base base = K::base(Z, Q, W);  // the key of the window's first bucket
  unsigned long long* const gdocs = K::counts(P, Z, Q, W);
  tq_metric_part* const gparts = P.parts + K::slot(Z, Q, W) * kC;
  MetricAcc acc[kC];
#pragma unroll
  for (uint32_t c = 0; c < kC; ++c) acc[c] = MetricAcc{~0ull, 0ull, 0.0, 0.0, 0u, 0u, INT32_MAX};
  uint32_t rdocs = 0, total = 0, one = 0, flushed_global = 0;
  uint32_t run = 0xFFFFFFFFu;  // the bucket of the register run (CTA-uniform), or none
  // the run into its bucket: missing copies, per warp, per CTA, one merge per column (CTA-uniform: every thread calls it)
  auto flush = [&]() {
#pragma unroll
    for (uint32_t c = 0; c < kC; ++c) {
      if (c >= nc) break;
      const MetricsCol& C = s_z.col[c];
      if ((C.flags & TQ_METRIC_MISSING) && acc[c].missing) {
        acc[c].count += acc[c].missing;
        if (!(C.flags & TQ_METRIC_COUNT_ONLY)) metric_add(acc[c], C.missing, C.kind, acc[c].missing, s_nan_inf[c]);
      }
      uint32_t count = __reduce_add_sync(kFull, acc[c].count);
      int q = __reduce_min_sync(kFull, acc[c].q);
      unsigned long long vlo = acc[c].lo, vhi = acc[c].hi;
      double sum = acc[c].sum, mag = acc[c].mag;
#pragma unroll
      for (int d = 16; d; d >>= 1) {
        vlo = min(vlo, __shfl_xor_sync(kFull, vlo, d));
        vhi = max(vhi, __shfl_xor_sync(kFull, vhi, d));
        sum = __dadd_rn(sum, __shfl_xor_sync(kFull, sum, d));
        mag = __dadd_rn(mag, __shfl_xor_sync(kFull, mag, d));
      }
      if (lane == 0) {
        s_count[warp][c] = count;
        s_q[warp][c] = q;
        s_lo[warp][c] = vlo;
        s_hi[warp][c] = vhi;
        s_sum[warp][c] = sum;
        s_mag[warp][c] = mag;
      }
      acc[c] = MetricAcc{~0ull, 0ull, 0.0, 0.0, 0u, 0u, INT32_MAX};
    }
    rdocs = __reduce_add_sync(kFull, rdocs);
    if (lane == 0) s_rdocs[warp] = rdocs;
    rdocs = 0;
    __syncthreads();
    if (threadIdx.x < nc) {
      const uint32_t c = threadIdx.x;
      unsigned long long count = 0, vlo = ~0ull, vhi = 0;
      double sum = 0.0, mag = 0.0;
      int q = INT32_MAX;
      for (int w = 0; w < kWarps; ++w) {
        count += s_count[w][c];
        q = min(q, s_q[w][c]);
        vlo = min(vlo, s_lo[w][c]);
        vhi = max(vhi, s_hi[w][c]);
        sum = __dadd_rn(sum, s_sum[w][c]);
        mag = __dadd_rn(mag, s_mag[w][c]);
      }
      const unsigned long long n_nan = s_nan_inf[c][0], n_inf = s_nan_inf[c][1];
      s_nan_inf[c][0] = s_nan_inf[c][1] = 0;  // (only this thread reads or resets column c's until the next barrier)
      if (shared) hm_merge(s_parts + run * kC + c, count, n_nan, n_inf, vlo, vhi, sum, mag, q);
      else hm_merge(gparts + (size_t)run * kC + c, count, n_nan, n_inf, vlo, vhi, sum, mag, q);
    } else if (threadIdx.x == 32u) {  // (warp 1: the columns are warp 0's)
      unsigned long long d = 0;
      for (int w = 0; w < kWarps; ++w) d += s_rdocs[w];
      if (d) {
        if (shared) s_docs[run] += (uint32_t)d;
        else atomicAdd(&gdocs[run], d);
      }
    }
    flushed_global += shared ? 0u : 1u;
    __syncthreads();
  };
  for (uint32_t tile = U.begin; tile < U.end; ++tile) {
    const uint32_t lo = tile * kTileDocs, hi = min(lo + kTileDocs, S.max_doc);
    if (threadIdx.x == 0) {
      const SortTile T = Z.tiles[tile];
      uint32_t idx = 0xFFFFFFFFu;
      if (W.n_bins && (T.flags & kSortTileValues)) K::one(T, Z, Q, W, base, idx);
      s_bucket = idx;
      one += idx != 0xFFFFFFFFu ? 1u : 0u;
    }
    if (threadIdx.x < nc) {  // (warp 0)
      const MetricsCol& C = s_z.col[threadIdx.x];
      uint32_t has = 0;
      if (!(C.flags & (TQ_METRIC_COUNT_ONLY | TQ_METRIC_EMPTY))) {
        const SortTile T = C.tiles[tile];
        has = (T.flags & kSortTileValues) && T.best[0] == ~T.best[1] ? 1u : 0u;
        s_one[threadIdx.x] = T.best[0];
      }
      s_has_one[threadIdx.x] = has;
    }
    match_tile<kMixed>(P.c, S.alive, wb, ng, need, lo, hi, s_acc, s_tmp, s_cnt, [&](uint32_t w, uint32_t bits) { s_acc[w] = bits; });
    __syncthreads();
    const uint32_t bits = s_acc[threadIdx.x];
    total += (uint32_t)__popc(bits);
    const uint32_t b = s_bucket;
    if (b < W.n_bins) {  // one bucket: every matching doc with a histogram value is in it
      if (b != run) {
        if (run != 0xFFFFFFFFu) flush();
        run = b;
      }
      const uint32_t hw = Z.present ? bits & __ldg(Z.present + (lo >> 5) + threadIdx.x) : bits;
      rdocs += (uint32_t)__popc(hw);
#pragma unroll
      for (uint32_t c = 0; c < kC; ++c) {
        if (c >= nc) break;
        const MetricsCol& C = s_z.col[c];
        const uint32_t with = (C.flags & TQ_METRIC_EMPTY) ? 0u : C.present ? hw & __ldg(C.present + (lo >> 5) + threadIdx.x) : hw;
        const uint32_t n = (uint32_t)__popc(with);
        acc[c].count += n;
        acc[c].missing += (uint32_t)__popc(hw ^ with);
        if (C.flags & (TQ_METRIC_COUNT_ONLY | TQ_METRIC_EMPTY)) continue;
        if (s_has_one[c]) {
          if (n) metric_add(acc[c], s_one[c], C.kind, n, s_nan_inf[c]);
        } else {
          for (uint32_t m = with; m; m &= m - 1u) {
            const uint32_t doc = lo + threadIdx.x * 32u + (uint32_t)(__ffs(m) - 1);
            metric_add(acc[c], __ldg(C.values + doc), C.kind, 1u, s_nan_inf[c]);
          }
        }
      }
    } else if (W.n_bins) {  // straddling: each doc to its own bucket
      uint32_t hw = Z.present ? bits & __ldg(Z.present + (lo >> 5) + threadIdx.x) : bits;
      if (hw) {
        uint32_t cw[kC];
#pragma unroll
        for (uint32_t c = 0; c < kC; ++c) {
          const MetricsCol& C = s_z.col[c];
          cw[c] = c >= nc || (C.flags & TQ_METRIC_EMPTY) ? 0u : C.present ? __ldg(C.present + (lo >> 5) + threadIdx.x) : 0xFFFFFFFFu;
        }
        for (; hw; hw &= hw - 1u) {
          const uint32_t bit = (uint32_t)(__ffs(hw) - 1), doc = lo + threadIdx.x * 32u + bit;
          const typename K::Value val = K::value(__ldg(Z.values + doc), Q);
          if (!K::counted(val, Z)) continue;
          const unsigned long long idx = K::index(val, Q, base);
          if (idx >= W.n_bins) continue;  // (never: the window covers every counted value of the unit's tiles)
          if (shared) hm_doc(s_docs + idx, s_parts + idx * kC, s_z, cw, doc, bit);
          else hm_doc(gdocs + idx, gparts + idx * kC, s_z, cw, doc, bit);
        }
      }
    }
    __syncthreads();
  }
  if (run != 0xFFFFFFFFu) flush();
  uint32_t flushed_shared = 0;
  if (shared) {  // every non-empty (bucket, column) of the window, and its doc counter, into the global accumulators
    for (uint32_t i = threadIdx.x; i < W.n_bins * kC; i += blockDim.x) {
      const uint32_t bin = i / kC, c = i % kC;
      const tq_metric_part& a = s_parts[i];
      if (c == 0 && s_docs[bin]) {
        atomicAdd(&gdocs[bin], (unsigned long long)s_docs[bin]);
        ++flushed_shared;
      }
      hm_merge(gparts + i, a.count, a.n_nan, a.n_inf, ~a.min_image, a.max_image, a.sum, a.magnitude,
               (int)(0x7FFFFFFFu - (unsigned)a.quantum_exp));
    }
    flushed_shared = __reduce_add_sync(kFull, flushed_shared);
  }
  total = __reduce_add_sync(kFull, total);
  if (lane == 0) { s_part[warp] = total; s_rdocs[warp] = flushed_shared; }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (K::hits(Q)) {
      unsigned long long hits = 0;
      for (int w = 0; w < kWarps; ++w) hits += s_part[w];
      if (hits) atomicAdd(&P.c.counts[S.query], hits);
    }
    unsigned long long fs = 0;
    for (int w = 0; w < kWarps; ++w) fs += s_rdocs[w];
    const uint32_t seen = U.end - U.begin;
    if (seen) { atomicAdd(&P.tiles[0], (unsigned long long)seen); if (one) atomicAdd(&P.tiles[1], (unsigned long long)one); }
    if (fs) atomicAdd(&P.tiles[2], fs);
    if (flushed_global) atomicAdd(&P.tiles[3], (unsigned long long)flushed_global);
  }
}

template <bool kMixed>
__global__ void __launch_bounds__(kThreads, 2) k_hist_metrics(const HistMetricsParams P) {
  metrics_unit_keys<HistKeys, kMixed>(P);
}

// The docs k_range counts, each feeding the metric columns of the (query, segment)'s MetricsSeg in its range bucket: the body of
// k_hist_metrics over RangeKeys.  The window is the query's whole bucket list, so its accumulators always live in shared memory; the
// wave's accumulators are the query's dense rows, which the host reads back and uncomplements (no compaction kernel).
template <bool kMixed>
__global__ void __launch_bounds__(kThreads, 2) k_range_metrics(const RangeMetricsParams P) {
  metrics_unit_keys<RangeKeys, kMixed>(P);
}

// One CTA per query of the wave: its non-empty buckets in ascending pos into its row (the prefix sum of k_hist_final; at most
// res_stride of them, and never more than its n_bins), each with its kMetricsMaxColumns parts, the complement of min_image and
// quantum_exp undone.
__global__ void __launch_bounds__(kThreads) k_hist_metrics_final(const HistMetricsParams P) {
  constexpr uint32_t kC = kMetricsMaxColumns;
  __shared__ uint32_t s_part[kWarps];
  const HistQuery Q = P.queries[P.query_base + blockIdx.x];
  const unsigned long long* const counts = P.counts + Q.counters;
  const tq_metric_part* const parts = P.parts + Q.counters * kC;
  const size_t row = P.rows[P.query_base + blockIdx.x];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t base = 0;  // non-empty buckets before this round of counters (the same on every thread)
  for (uint32_t i0 = 0; i0 < Q.n_bins; i0 += blockDim.x) {
    const uint32_t i = i0 + threadIdx.x;
    const unsigned long long c = i < Q.n_bins ? counts[i] : 0ull;
    const uint32_t mask = __ballot_sync(kFull, c != 0ull);
    if (lane == 0) s_part[warp] = (uint32_t)__popc(mask);
    __syncthreads();
    uint32_t at = base + (uint32_t)__popc(mask & ((1u << lane) - 1u));
    for (uint32_t w = 0; w < warp; ++w) at += s_part[w];
    if (c && at < P.res_stride) {
      P.res_pos[row + at] = Q.base + (long long)i;
      P.res_count[row + at] = c;
      for (uint32_t k = 0; k < kC; ++k) {
        tq_metric_part p = parts[(size_t)i * kC + k];
        p.min_image = ~p.min_image;
        p.quantum_exp = (int)(0x7FFFFFFFu - (unsigned)p.quantum_exp);
        P.res_parts[(row + at) * kC + k] = p;
      }
    }
    for (int w = 0; w < kWarps; ++w) base += s_part[w];
    __syncthreads();
  }
  if (threadIdx.x == 0) P.res_n[blockIdx.x] = base;
}

// ---- metrics per term (terms with metric sub-aggregations: collect_terms_with_docs, term_agg/mod.rs) -------------------------
// The docs k_terms counts under a key feed the metric columns of the (query, segment)'s MetricsSeg in that key's entry.  k_terms
// counts and k_terms_select cuts as for tq_terms_batch; a metric order (kTermsByMetric) adds k_terms_order before the cut, which
// accumulates per key the ordering column's value count and quantity, and k_terms_select_metric, which recuts those (query,
// segment)s by the metric.  k_terms_mark gives each kept key its slot, and k_terms_metrics makes the second match pass that feeds
// the slots' parts.

// The image a collected doc gives column C, or false when the column collects nothing for it (no value and no missing).  The
// image of a count-only column is never read.
__device__ __forceinline__ bool terms_metric_image(const MetricsCol& C, const uint32_t doc, unsigned long long& image) {
  const bool has = !(C.flags & TQ_METRIC_EMPTY) && (!C.present || ((__ldg(C.present + (doc >> 5)) >> (doc & 31u)) & 1u));
  if (!has && !(C.flags & TQ_METRIC_MISSING)) return false;
  image = has && !(C.flags & TQ_METRIC_COUNT_ONLY) ? __ldg(C.values + doc) : C.missing;
  return true;
}

// The ordering quantity of one collected value: its f64 bits for a sum or avg, ~image for a min, the image for a max, 0 for a count,
// a count-only column or a NaN (an order on a column that saw NaN is refused by the caller's check of the total part).  Quantities
// combine with an f64 add (sum, avg) or a max (the rest), and 0 is the empty quantity of either.
__device__ __forceinline__ unsigned long long terms_order_q(const unsigned long long image, const MetricsCol& C, const uint32_t metric) {
  if (metric == TQ_TERMS_ORDER_COUNT || (C.flags & TQ_METRIC_COUNT_ONLY)) return 0ull;
  const double v = hist_value(image, C.kind);
  if (v != v) return 0ull;
  if (metric == TQ_TERMS_ORDER_MIN) return ~image;
  if (metric == TQ_TERMS_ORDER_MAX) return image;
  return (unsigned long long)__double_as_longlong(v);
}
__device__ __forceinline__ unsigned long long terms_order_combine(const unsigned long long a, const unsigned long long b, const bool sum) {
  return sum ? (unsigned long long)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)a), __longlong_as_double((long long)b)))
             : max(a, b);
}
__device__ __forceinline__ void terms_order_atomic(uint32_t* count, unsigned long long* q, const uint32_t n, const unsigned long long v,
                                                   const bool sum) {
  if (!n) return;
  atomicAdd(count, n);
  if (!v) return;
  if (sum) atomicAdd(reinterpret_cast<double*>(q), __longlong_as_double((long long)v));
  else atomicMax(q, v);
}

// compute_metric_value(...).unwrap_or(0.0) of a key's ordering count and quantity (metric/stats.rs:325-356, with the stats' min /
// max starting at f64::MAX / f64::MIN), as the rank k_terms_select_metric selects on: the value's monotone image with -0.0 taken as
// +0.0 (partial_cmp's equality), complemented for an ascending order, so that the larger rank comes first.
__device__ __forceinline__ unsigned long long terms_order_rank(const uint32_t oc, const unsigned long long oq, const MetricsCol& C,
                                                               const uint32_t metric, const bool asc) {
  constexpr double kMax = 1.7976931348623157e308;
  double v = 0.0;
  if (metric == TQ_TERMS_ORDER_COUNT) v = (double)oc;
  else if (oc && !(C.flags & TQ_METRIC_COUNT_ONLY)) {
    if (metric == TQ_TERMS_ORDER_SUM) v = __longlong_as_double((long long)oq);
    else if (metric == TQ_TERMS_ORDER_AVG) v = __ddiv_rn(__longlong_as_double((long long)oq), (double)oc);
    else if (metric == TQ_TERMS_ORDER_MIN) { const double m = hist_value(~oq, C.kind); v = m < kMax ? m : kMax; }
    else { const double m = hist_value(oq, C.kind); v = m > -kMax ? m : -kMax; }
  }
  unsigned long long b = v == 0.0 ? 0ull : (unsigned long long)__double_as_longlong(v);
  b = (b >> 63) ? ~b : b | (1ull << 63);
  return asc ? ~b : b;
}

// One CTA per Count unit of a metric-ordered (query, segment) (the others exit): per counted doc the ordering column's value count
// and quantity into its key's accumulators (the unit's window: in shared memory when it has kTermsOrderSmemKeys keys or fewer), and
// the column's part over every collected doc, reduced per CTA and merged into the query's order part.  A tile whose values are
// all one key, and the docs without a value (the missing key), accumulate in registers and are reduced per warp.
template <bool kMixed>
__global__ void __launch_bounds__(kThreads) k_terms_order(const TermsMetricsParams P) {
  __shared__ uint32_t s_acc[kTileDocs / 32u], s_tmp[kTileDocs / 32u];
  __shared__ uint32_t s_cnt[kMixed ? kTileDocs / 4u : 1u];
  __shared__ uint32_t s_oc[kTermsOrderSmemKeys];
  __shared__ unsigned long long s_oq[kTermsOrderSmemKeys];
  __shared__ uint32_t s_one;  // the tile's one key (index into the unit's window), or ~0u
  __shared__ uint32_t s_nan_inf[2];
  __shared__ unsigned long long s_lo[kWarps], s_hi[kWarps];
  __shared__ double s_sum[kWarps], s_mag[kWarps];
  __shared__ uint32_t s_count[kWarps];
  __shared__ int s_q[kWarps];
  const uint32_t unit = P.t.unit_base + blockIdx.x;
  const Unit U = P.t.c.units[unit];
  const TermsSeg Z = P.t.tsegs[U.qseg];
  if (!(Z.flags & kTermsByMetric)) return;
  const CountSeg S = P.t.c.segs[U.qseg];
  const TermsOrder O = P.orders[S.query];
  const MetricsCol C = P.msegs[U.qseg].col[O.column];
  const HistUnit W = P.t.windows[unit];
  const bool shared = W.n_bins <= kTermsOrderSmemKeys, sum = O.metric == TQ_TERMS_ORDER_SUM || O.metric == TQ_TERMS_ORDER_AVG;
  const bool with_missing = (Z.flags & kTermsMissing) != 0;
  if (shared)
    for (uint32_t i = threadIdx.x; i < W.n_bins; i += blockDim.x) { s_oc[i] = 0; s_oq[i] = 0ull; }
  if (threadIdx.x < 2u) s_nan_inf[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t wb = S.words_base, ng = P.t.c.words[wb], need = P.t.c.words[wb + 1u];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const unsigned long long base = Z.base + W.first;
  uint32_t* const gcnt = P.ocount + Z.counters + W.first;
  unsigned long long* const gq = P.oq + Z.counters + W.first;
  MetricAcc tot{~0ull, 0ull, 0.0, 0.0, 0u, 0u, INT32_MAX};  // the column over every collected doc
  uint32_t m_n = 0;                                        // the missing key's values and quantity
  unsigned long long m_q = 0ull;
  // one collected doc into the total part; true with its quantity when the column collects it
  auto collect = [&](const uint32_t doc, unsigned long long& q) -> bool {
    unsigned long long image;
    if (!terms_metric_image(C, doc, image)) return false;
    ++tot.count;
    if (!(C.flags & TQ_METRIC_COUNT_ONLY)) metric_add(tot, image, C.kind, 1u, s_nan_inf);
    q = terms_order_q(image, C, O.metric);
    return true;
  };
  // a warp's register count and quantity into one key's accumulators
  auto flush_warp = [&](uint32_t n, unsigned long long q, uint32_t* pc, unsigned long long* pq) {
    n = __reduce_add_sync(kFull, n);
#pragma unroll
    for (int d = 16; d; d >>= 1) q = terms_order_combine(q, __shfl_xor_sync(kFull, q, d), sum);
    if (lane == 0) terms_order_atomic(pc, pq, n, q, sum);
  };
  for (uint32_t tile = U.begin; tile < U.end; ++tile) {
    const uint32_t lo = tile * kTileDocs, hi = min(lo + kTileDocs, S.max_doc);
    if (threadIdx.x == 0) {
      const SortTile T = Z.tiles[tile];
      uint32_t idx = 0xFFFFFFFFu;
      if (W.n_bins && (T.flags & kSortTileValues)) TermsKeys::one(T, Z, 0u, W, base, idx);
      s_one = idx;
    }
    match_tile<kMixed>(P.t.c, S.alive, wb, ng, need, lo, hi, s_acc, s_tmp, s_cnt, [&](uint32_t w, uint32_t bits) { s_acc[w] = bits; });
    __syncthreads();
    const uint32_t bits = s_acc[threadIdx.x];
    uint32_t with = Z.present ? bits & __ldg(Z.present + (lo >> 5) + threadIdx.x) : bits;
    if (with_missing)
      for (uint32_t m = bits ^ with; m; m &= m - 1u) {
        unsigned long long q;
        if (collect(lo + threadIdx.x * 32u + (uint32_t)(__ffs(m) - 1), q)) { ++m_n; m_q = terms_order_combine(m_q, q, sum); }
      }
    const uint32_t one = s_one;
    if (one < W.n_bins) {  // one key: registers, one flush per warp
      uint32_t n = 0;
      unsigned long long qs = 0ull;
      for (; with; with &= with - 1u) {
        unsigned long long q;
        if (collect(lo + threadIdx.x * 32u + (uint32_t)(__ffs(with) - 1), q)) { ++n; qs = terms_order_combine(qs, q, sum); }
      }
      flush_warp(n, qs, shared ? &s_oc[one] : &gcnt[one], shared ? &s_oq[one] : &gq[one]);
    } else if (W.n_bins) {
      for (; with; with &= with - 1u) {
        const uint32_t doc = lo + threadIdx.x * 32u + (uint32_t)(__ffs(with) - 1);
        unsigned long long q;
        if (!collect(doc, q)) continue;
        const unsigned long long idx = __ldg(Z.values + doc) - base;
        if (idx < W.n_bins) {  // (always: the window covers every value of the unit's tiles)
          if (shared) terms_order_atomic(&s_oc[idx], &s_oq[idx], 1u, q, sum);
          else terms_order_atomic(&gcnt[idx], &gq[idx], 1u, q, sum);
        }
      }
    }
    __syncthreads();
  }
  if (shared)
    for (uint32_t i = threadIdx.x; i < W.n_bins; i += blockDim.x) terms_order_atomic(&gcnt[i], &gq[i], s_oc[i], s_oq[i], sum);
  if (with_missing) {
    const bool inside = Z.missing - Z.base < (unsigned long long)Z.n_keys;
    const uint32_t rel = U.qseg - P.t.seg_base;
    flush_warp(m_n, m_q, inside ? P.ocount + Z.counters + (Z.missing - Z.base) : P.ocount_missing + rel,
               inside ? P.oq + Z.counters + (Z.missing - Z.base) : P.oq_missing + rel);
  }
  // the total part: per warp, per CTA, one merge
  const uint32_t count = __reduce_add_sync(kFull, tot.count);
  const int q = __reduce_min_sync(kFull, tot.q);
  unsigned long long vlo = tot.lo, vhi = tot.hi;
  double s = tot.sum, mag = tot.mag;
#pragma unroll
  for (int d = 16; d; d >>= 1) {
    vlo = min(vlo, __shfl_xor_sync(kFull, vlo, d));
    vhi = max(vhi, __shfl_xor_sync(kFull, vhi, d));
    s = __dadd_rn(s, __shfl_xor_sync(kFull, s, d));
    mag = __dadd_rn(mag, __shfl_xor_sync(kFull, mag, d));
  }
  if (lane == 0) { s_count[warp] = count; s_q[warp] = q; s_lo[warp] = vlo; s_hi[warp] = vhi; s_sum[warp] = s; s_mag[warp] = mag; }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long n = 0, a = ~0ull, b = 0;
    double x = 0.0, y = 0.0;
    int e = INT32_MAX;
    for (int w = 0; w < kWarps; ++w) {
      n += s_count[w];
      e = min(e, s_q[w]);
      a = min(a, s_lo[w]);
      b = max(b, s_hi[w]);
      x = __dadd_rn(x, s_sum[w]);
      y = __dadd_rn(y, s_mag[w]);
    }
    hm_merge(P.order_parts + S.query, n, s_nan_inf[0], s_nan_inf[1], a, b, x, y, e);
  }
}

// One CTA per (query, segment) of a wave, after k_terms_select: a metric-ordered one with more than segment_size entries is cut
// again by its metric (the others exit, k_terms_select's rows standing).  The entries are those of k_terms_select (the missing
// count already folded into its counter when inside the counters); a radix select (8 passes of 8 bits) over the 64-bit rank of
// terms_order_rank finds the rank t of the segment_size-th entry, and the entries above it are kept with the lowest keys at t.  The
// entry at position segment_size in that order gives term_doc_count_before_cutoff; the doc counts of the entries cut add up to
// sum_other_doc_count.  The kept entries overwrite the (query, segment)'s region in ascending key.
__global__ void __launch_bounds__(kThreads) k_terms_select_metric(const TermsMetricsParams P) {
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_part[kWarps];
  __shared__ unsigned long long s_wide[kWarps];
  __shared__ unsigned long long s_prefix;
  __shared__ uint32_t s_k, s_error;
  const uint32_t rel = blockIdx.x, si = P.t.seg_base + rel;
  const TermsSeg Z = P.t.tsegs[si];
  if (!(Z.flags & kTermsByMetric)) return;
  const TermsOrder O = P.orders[P.t.c.segs[si].query];
  const MetricsCol C = P.msegs[si].col[O.column];
  const uint32_t* const cnt = P.t.counts + Z.counters;
  const uint32_t n = Z.n_keys, ss = Z.segment_size;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t mc = (Z.flags & kTermsMissing) ? P.t.missing[rel] : 0u;
  const bool inside = mc && Z.missing - Z.base < (unsigned long long)n;
  const uint32_t extra = mc && !inside ? 1u : 0u, off = extra && Z.missing < Z.base ? 1u : 0u;
  const uint32_t L = n + extra;  // entries in key order: [missing,] counters[0..n) [, missing]
  const bool asc = Z.flags & kTermsAsc;
  auto count_at = [&](uint32_t i) -> uint32_t { i -= off; return i < n ? cnt[i] : mc; };
  auto key_at = [&](uint32_t i) -> unsigned long long { i -= off; return i < n ? Z.base + i : Z.missing; };
  auto rank_at = [&](uint32_t i) -> unsigned long long {
    i -= off;
    return i < n ? terms_order_rank(P.ocount[Z.counters + i], P.oq[Z.counters + i], C, O.metric, asc)
                 : terms_order_rank(P.ocount_missing[rel], P.oq_missing[rel], C, O.metric, asc);
  };
  uint32_t nz = 0;
  unsigned long long sum = 0;
  for (uint32_t i = threadIdx.x; i < L; i += blockDim.x) {
    const uint32_t c = count_at(i);
    nz += c ? 1u : 0u;
    sum += c;
  }
  nz = __reduce_add_sync(kFull, nz);
  for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(kFull, sum, d);
  if (lane == 0) { s_part[warp] = nz; s_wide[warp] = sum; }
  __syncthreads();
  uint32_t N = 0;
  unsigned long long total = 0;
  for (int w = 0; w < kWarps; ++w) { N += s_part[w]; total += s_wide[w]; }
  if (N <= ss) return;  // (CTA-uniform) no cut: every entry kept, both scalars 0, as k_terms_select wrote them
  __syncthreads();
  unsigned long long prefix = 0, mask = 0;
  uint32_t k = ss + 1u;  // the (segment_size + 1)-th largest rank: the first entry cut, at t_cut or below it
  for (int shift = 56; shift >= 0; shift -= 8) {
    s_hist[threadIdx.x] = 0;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < L; i += blockDim.x) {
      if (!count_at(i)) continue;
      const unsigned long long t = rank_at(i);
      if ((t & mask) == prefix) atomicAdd(&s_hist[(t >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t b = 255, acc = 0;
      for (; acc + s_hist[b] < k; --b) acc += s_hist[b];
      s_prefix = prefix | ((unsigned long long)b << shift);
      s_k = k - acc;
    }
    __syncthreads();
    prefix = s_prefix;
    k = s_k;
    mask |= 255ull << shift;
    __syncthreads();
  }
  // t_cut: the rank of the entry at position segment_size, the k-th (1-based, lowest keys first) of the entries at it; the entries
  // kept are those above t_cut and the k - 1 lowest keys at it
  const unsigned long long t_cut = prefix;
  const uint32_t need = k - 1u;
  uint32_t base_eq = 0, base_keep = 0;
  unsigned long long kept = 0;
  for (uint32_t i0 = 0; i0 < L; i0 += blockDim.x) {
    const uint32_t i = i0 + threadIdx.x;
    const uint32_t c = i < L ? count_at(i) : 0u;
    const unsigned long long t = c ? rank_at(i) : 0ull;
    const bool eq = c && t == t_cut;
    uint32_t tot;
    const uint32_t r_eq = base_eq + cta_scan_excl(eq ? 1u : 0u, s_part, tot);
    base_eq += tot;
    const bool keep = c && (t > t_cut || (eq && r_eq < need));
    if (eq && r_eq == need) s_error = c;
    const uint32_t at = base_keep + cta_scan_excl(keep ? 1u : 0u, s_part, tot);
    base_keep += tot;
    if (keep) {
      P.t.res_key[Z.region + at] = key_at(i);
      P.t.res_count[Z.region + at] = c;
      kept += c;
    }
  }
  for (int d = 16; d; d >>= 1) kept += __shfl_xor_sync(kFull, kept, d);
  if (lane == 0) s_wide[warp] = kept;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long k_sum = 0;
    for (int w = 0; w < kWarps; ++w) k_sum += s_wide[w];
    P.t.res_n[rel] = base_keep;
    P.t.res_other[rel] = total - k_sum;
    P.t.res_error[rel] = s_error;
  }
}

// One CTA per (query, segment) of a wave, after the cut: each kept key's counter becomes kTermsSlot | its index in the region (a
// missing key outside the counters: mslot).  Counts are below 2^31, so a marked counter is told from a count by its top bit.
__global__ void __launch_bounds__(kThreads) k_terms_mark(const TermsMetricsParams P) {
  const uint32_t rel = blockIdx.x;
  const TermsSeg Z = P.t.tsegs[P.t.seg_base + rel];
  uint32_t* const cnt = P.t.counts + Z.counters;
  const uint32_t n = P.t.res_n[rel];
  for (uint32_t j = threadIdx.x; j < n; j += blockDim.x) {
    const unsigned long long key = P.t.res_key[Z.region + j];
    if (key - Z.base < (unsigned long long)Z.n_keys) cnt[key - Z.base] = kTermsSlot | j;
    else P.mslot[rel] = kTermsSlot | j;
  }
}

// The docs of mask m (the thread's 32-doc word at lo) all in one slot: per column as k_metrics adds them (one-value tiles and
// missing copies included), reduced per warp and merged once per (warp, column) into the slot's parts p.  Called by whole warps.
__device__ __forceinline__ void tm_uniform(tq_metric_part* p, const uint32_t m, const uint32_t lo, const MetricsSeg& z,
                                           const unsigned long long* s_one, const uint32_t* s_has_one, uint32_t (*s_ni)[2]) {
  if (!__any_sync(kFull, m)) return;
  const uint32_t lane = threadIdx.x & 31u;
#pragma unroll 1
  for (uint32_t c = 0; c < z.n_columns; ++c) {
    const MetricsCol& C = z.col[c];
    MetricAcc a{~0ull, 0ull, 0.0, 0.0, 0u, 0u, INT32_MAX};
    const uint32_t with = (C.flags & TQ_METRIC_EMPTY) ? 0u : C.present ? m & __ldg(C.present + (lo >> 5) + threadIdx.x) : m;
    const uint32_t n = (uint32_t)__popc(with), miss = (uint32_t)__popc(m ^ with);
    a.count = n;
    if (!(C.flags & (TQ_METRIC_COUNT_ONLY | TQ_METRIC_EMPTY))) {
      if (s_has_one[c]) {
        if (n) metric_add(a, s_one[c], C.kind, n, s_ni[c]);
      } else {
        for (uint32_t w = with; w; w &= w - 1u)
          metric_add(a, __ldg(C.values + lo + threadIdx.x * 32u + (uint32_t)(__ffs(w) - 1)), C.kind, 1u, s_ni[c]);
      }
    }
    if ((C.flags & TQ_METRIC_MISSING) && miss) {
      a.count += miss;
      if (!(C.flags & TQ_METRIC_COUNT_ONLY)) metric_add(a, C.missing, C.kind, miss, s_ni[c]);
    }
    const uint32_t count = __reduce_add_sync(kFull, a.count);
    const int q = __reduce_min_sync(kFull, a.q);
    unsigned long long vlo = a.lo, vhi = a.hi;
    double sum = a.sum, mag = a.mag;
#pragma unroll
    for (int d = 16; d; d >>= 1) {
      vlo = min(vlo, __shfl_xor_sync(kFull, vlo, d));
      vhi = max(vhi, __shfl_xor_sync(kFull, vhi, d));
      sum = __dadd_rn(sum, __shfl_xor_sync(kFull, sum, d));
      mag = __dadd_rn(mag, __shfl_xor_sync(kFull, mag, d));
    }
    __syncwarp();
    if (lane == 0) {
      const uint32_t n_nan = s_ni[c][0], n_inf = s_ni[c][1];
      s_ni[c][0] = s_ni[c][1] = 0;
      hm_merge(p + c, count, n_nan, n_inf, vlo, vhi, sum, mag, q);
    }
    __syncwarp();
  }
}

// One CTA per Count unit: the docs k_terms counted, each into the parts of its key's slot (docs of keys cut feed nothing).  The
// docs without a value go to the missing key's slot, a tile whose values are all one kept key to that key's: both with tm_uniform.
// Any other tile has each thread walk its word's matches: one gather of the key, one lookup of its counter, and per column
// hm_collect.  The parts of a (query, segment) keeping kTermsMetricsSmemSlots entries or fewer accumulate in shared memory and are
// merged into the global ones at exit.
template <bool kMixed>
__global__ void __launch_bounds__(kThreads, 2) k_terms_metrics(const TermsMetricsParams P) {
  static_assert(sizeof(MetricsSeg) % 8u == 0 && sizeof(MetricsSeg) / 8u <= (uint32_t)kThreads, "one word of the descriptor per thread");
  constexpr uint32_t kC = kMetricsMaxColumns;
  constexpr uint32_t kPerDoc = 0xFFFFFFFFu, kSkip = 0xFFFFFFFEu;  // s_slot: walk each doc; no doc with a value feeds a slot
  __shared__ uint32_t s_acc[kTileDocs / 32u], s_tmp[kTileDocs / 32u];
  __shared__ uint32_t s_cnt[kMixed ? kTileDocs / 4u : 1u];
  __shared__ MetricsSeg s_z;
  __shared__ tq_metric_part s_parts[kTermsMetricsSmemSlots * kC];
  __shared__ unsigned long long s_one[kC];
  __shared__ uint32_t s_has_one[kC];
  __shared__ uint32_t s_slot;
  __shared__ uint32_t s_nan_inf[kWarps][kC][2];
  const uint32_t unit = P.t.unit_base + blockIdx.x;
  const Unit U = P.t.c.units[unit];
  const CountSeg S = P.t.c.segs[U.qseg];
  const TermsSeg Z = P.t.tsegs[U.qseg];
  const uint32_t rel = U.qseg - P.t.seg_base, n_kept = P.t.res_n[rel];
  const uint32_t* const cnt = P.t.counts + Z.counters;
  if (threadIdx.x < sizeof(MetricsSeg) / 8u)
    reinterpret_cast<unsigned long long*>(&s_z)[threadIdx.x] = reinterpret_cast<const unsigned long long*>(P.msegs + U.qseg)[threadIdx.x];
  if (threadIdx.x < kWarps * kC * 2u) (&s_nan_inf[0][0][0])[threadIdx.x] = 0;
  const bool shared = n_kept <= kTermsMetricsSmemSlots;
  if (shared)
    for (uint32_t i = threadIdx.x; i < n_kept * (uint32_t)(sizeof(tq_metric_part) / 8u) * kC; i += blockDim.x)
      reinterpret_cast<unsigned long long*>(s_parts)[i] = 0ull;
  uint32_t ms = 0;  // the missing key's slot (CTA-uniform)
  if (Z.flags & kTermsMissing) ms = Z.missing - Z.base < (unsigned long long)Z.n_keys ? cnt[Z.missing - Z.base] : P.mslot[rel];
  __syncthreads();
  const uint32_t nc = s_z.n_columns;
  const uint32_t wb = S.words_base, ng = P.t.c.words[wb], need = P.t.c.words[wb + 1u];
  const uint32_t warp = threadIdx.x >> 5;
  tq_metric_part* const gparts = P.parts + Z.region * kC;
  tq_metric_part* const parts = shared ? s_parts : gparts;
  uint32_t one = 0;
  for (uint32_t tile = U.begin; tile < U.end; ++tile) {
    const uint32_t lo = tile * kTileDocs, hi = min(lo + kTileDocs, S.max_doc);
    if (threadIdx.x == 0) {
      const SortTile T = Z.tiles[tile];
      uint32_t slot = kSkip;
      if ((T.flags & kSortTileValues) && T.best[0] == ~T.best[1]) {
        const unsigned long long i = T.best[0] - Z.base;
        const uint32_t c = i < (unsigned long long)Z.n_keys ? cnt[i] : 0u;
        if (c & kTermsSlot) slot = c & ~kTermsSlot;
      } else if (T.flags & kSortTileValues) {
        slot = kPerDoc;
      }
      s_slot = slot;
      one += slot < kSkip ? 1u : 0u;
    }
    if (threadIdx.x < nc) {  // (warp 0)
      const MetricsCol& C = s_z.col[threadIdx.x];
      uint32_t has = 0;
      if (!(C.flags & (TQ_METRIC_COUNT_ONLY | TQ_METRIC_EMPTY))) {
        const SortTile T = C.tiles[tile];
        has = (T.flags & kSortTileValues) && T.best[0] == ~T.best[1] ? 1u : 0u;
        s_one[threadIdx.x] = T.best[0];
      }
      s_has_one[threadIdx.x] = has;
    }
    match_tile<kMixed>(P.t.c, S.alive, wb, ng, need, lo, hi, s_acc, s_tmp, s_cnt, [&](uint32_t w, uint32_t bits) { s_acc[w] = bits; });
    __syncthreads();
    const uint32_t bits = s_acc[threadIdx.x];
    uint32_t with = Z.present ? bits & __ldg(Z.present + (lo >> 5) + threadIdx.x) : bits;
    if (ms & kTermsSlot) tm_uniform(parts + (ms & ~kTermsSlot) * kC, bits ^ with, lo, s_z, s_one, s_has_one, s_nan_inf[warp]);
    const uint32_t slot = s_slot;
    if (slot < kSkip) {
      tm_uniform(parts + slot * kC, with, lo, s_z, s_one, s_has_one, s_nan_inf[warp]);
    } else if (slot == kPerDoc && with) {
      uint32_t cw[kC];
#pragma unroll
      for (uint32_t c = 0; c < kC; ++c) {
        const MetricsCol& C = s_z.col[c];
        cw[c] = c >= nc || (C.flags & TQ_METRIC_EMPTY) ? 0u : C.present ? __ldg(C.present + (lo >> 5) + threadIdx.x) : 0xFFFFFFFFu;
      }
      for (; with; with &= with - 1u) {
        const uint32_t bit = (uint32_t)(__ffs(with) - 1), doc = lo + threadIdx.x * 32u + bit;
        const uint32_t c = __ldg(cnt + (__ldg(Z.values + doc) - Z.base));  // (the counters cover every value of the visited tiles)
        if (!(c & kTermsSlot)) continue;
        tq_metric_part* const p = parts + (c & ~kTermsSlot) * kC;
#pragma unroll
        for (uint32_t k = 0; k < kC; ++k) {
          if (k >= nc) break;
          hm_collect(p + k, s_z.col[k], doc, (cw[k] >> bit) & 1u);
        }
      }
    }
    __syncthreads();
  }
  if (shared)  // every non-empty (slot, column) into the global parts
    for (uint32_t i = threadIdx.x; i < n_kept * kC; i += blockDim.x) {
      const tq_metric_part& a = s_parts[i];
      hm_merge(gparts + i, a.count, a.n_nan, a.n_inf, ~a.min_image, a.max_image, a.sum, a.magnitude,
               (int)(0x7FFFFFFFu - (unsigned)a.quantum_exp));
    }
  if (threadIdx.x == 0) {
    const uint32_t seen = U.end - U.begin;
    if (seen) { atomicAdd(&P.tiles[0], (unsigned long long)seen); if (one) atomicAdd(&P.tiles[1], (unsigned long long)one); }
  }
}

// ---- histogram per term (terms with one histogram sub-aggregation: collect_terms_with_docs, term_histogram.rs) ---------------
// One CTA per Count unit, after k_terms_mark: the docs k_terms counted, each with a histogram value in its (query, segment)'s
// bounds counted in cell (slot of its key, pos); docs of keys cut count nowhere, docs without a key go to the missing key's slot.
// Per tile, thread 0 reads both columns' SortTile: a tile whose values all hold one kept key skips the key gather, a tile whose
// histogram values are all in bounds and in one bucket (HistKeys::one) skips the value gather, and a tile with both adds each warp's
// count of matching docs with both values to one cell.  A unit whose window (kept slots × its buckets) fits kTermsHistSmemCells
// counts in shared memory (one u32 atomic per doc) and adds its non-zero cells to the grid at exit; a wider one counts in the grid.
template <bool kMixed>
__global__ void __launch_bounds__(kThreads, 3) k_terms_hist(const TermsHistParams P) {
  constexpr uint32_t kPerDoc = 0xFFFFFFFFu, kSkip = 0xFFFFFFFEu;  // s_slot: look each doc's key up; no doc with a key is counted
  __shared__ uint32_t s_acc[kTileDocs / 32u], s_tmp[kTileDocs / 32u];
  __shared__ uint32_t s_cnt[kMixed ? kTileDocs / 4u : 1u];
  __shared__ uint32_t s_cells[kTermsHistSmemCells];
  __shared__ uint32_t s_slot, s_bucket;
  const uint32_t unit = P.t.unit_base + blockIdx.x;
  const Unit U = P.t.c.units[unit];
  const uint32_t rel = U.qseg - P.t.seg_base, n_kept = P.t.res_n[rel];
  const HistUnit W = P.hunits[unit];
  if (!n_kept || !W.n_bins) return;  // (CTA-uniform: nothing of the unit can be counted)
  const CountSeg S = P.t.c.segs[U.qseg];
  const TermsSeg Z = P.t.tsegs[U.qseg];
  const HistSeg H = P.hsegs[U.qseg];
  const HistQuery Q = P.queries[S.query];
  const TermsHistSeg G = P.gsegs[U.qseg];
  const uint32_t* const cnt = P.t.counts + Z.counters;
  const long long base = G.base + (long long)W.first;  // pos of the window's first bucket
  const bool shared = n_kept * W.n_bins <= kTermsHistSmemCells;  // (n_kept * n_bins <= the grid budget < 2^32)
  uint32_t* const gcells = P.grid + G.grid + W.first;
  uint32_t* const cells = shared ? s_cells : gcells;
  const uint32_t row = shared ? W.n_bins : G.span;  // cell (slot, b) of the window: cells[slot * row + b]
  if (shared)
    for (uint32_t i = threadIdx.x; i < n_kept * W.n_bins; i += blockDim.x) s_cells[i] = 0;
  uint32_t ms = kSkip;  // the missing key's slot (CTA-uniform)
  if (Z.flags & kTermsMissing) {
    const uint32_t c = Z.missing - Z.base < (unsigned long long)Z.n_keys ? cnt[Z.missing - Z.base] : P.mslot[rel];
    if (c & kTermsSlot) ms = c & ~kTermsSlot;
  }
  const uint32_t wb = S.words_base, ng = P.t.c.words[wb], need = P.t.c.words[wb + 1u];
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t n_one_key = 0, n_one_bucket = 0, n_both = 0;
  for (uint32_t tile = U.begin; tile < U.end; ++tile) {
    const uint32_t lo = tile * kTileDocs, hi = min(lo + kTileDocs, S.max_doc);
    if (threadIdx.x == 0) {
      const SortTile T = Z.tiles[tile];
      uint32_t slot = kSkip;
      if ((T.flags & kSortTileValues) && T.best[0] == ~T.best[1]) {
        const unsigned long long i = T.best[0] - Z.base;
        const uint32_t c = i < (unsigned long long)Z.n_keys ? cnt[i] : 0u;
        if (c & kTermsSlot) slot = c & ~kTermsSlot;
      } else if (T.flags & kSortTileValues) {
        slot = kPerDoc;
      }
      const SortTile V = H.tiles[tile];
      uint32_t b = 0xFFFFFFFFu;
      if (V.flags & kSortTileValues) HistKeys::one(V, H, Q, W, base, b);
      s_slot = slot;
      s_bucket = b;
      n_one_key += slot < kSkip ? 1u : 0u;
      n_one_bucket += b != 0xFFFFFFFFu ? 1u : 0u;
      n_both += slot < kSkip && b != 0xFFFFFFFFu ? 1u : 0u;
    }
    match_tile<kMixed>(P.t.c, S.alive, wb, ng, need, lo, hi, s_acc, s_tmp, s_cnt, [&](uint32_t w, uint32_t bits) { s_acc[w] = bits; });
    __syncthreads();
    const uint32_t bits = s_acc[threadIdx.x];
    const uint32_t kp = Z.present ? __ldg(Z.present + (lo >> 5) + threadIdx.x) : 0xFFFFFFFFu;
    const uint32_t hp = H.present ? __ldg(H.present + (lo >> 5) + threadIdx.x) : 0xFFFFFFFFu;
    const uint32_t slot = s_slot, b1 = s_bucket;
    const uint32_t kd = slot == kSkip ? 0u : bits & kp & hp;  // matching docs with a key (that may be kept) and a histogram value
    const uint32_t md = ms == kSkip ? 0u : bits & ~kp & hp;   // ... without a key, with a histogram value
    if (b1 != 0xFFFFFFFFu) {  // every histogram value of the tile counts in bucket b1
      const uint32_t nm = __reduce_add_sync(kFull, (uint32_t)__popc(md));
      if (lane == 0 && nm) atomicAdd(&cells[ms * row + b1], nm);
      if (slot < kSkip) {
        const uint32_t nk = __reduce_add_sync(kFull, (uint32_t)__popc(kd));
        if (lane == 0 && nk) atomicAdd(&cells[slot * row + b1], nk);
      } else {
        for (uint32_t w = kd; w; w &= w - 1u) {
          const uint32_t c = __ldg(cnt + (__ldg(Z.values + lo + threadIdx.x * 32u + (uint32_t)(__ffs(w) - 1)) - Z.base));
          if (c & kTermsSlot) atomicAdd(&cells[(c & ~kTermsSlot) * row + b1], 1u);
        }
      }
    } else {
      for (uint32_t w = kd | md; w; w &= w - 1u) {
        const uint32_t bit = (uint32_t)(__ffs(w) - 1), doc = lo + threadIdx.x * 32u + bit;
        uint32_t s = ms;
        if ((kd >> bit) & 1u) {
          s = slot;
          if (slot == kPerDoc) {  // (the counters cover every value of the visited tiles)
            const uint32_t c = __ldg(cnt + (__ldg(Z.values + doc) - Z.base));
            if (!(c & kTermsSlot)) continue;
            s = c & ~kTermsSlot;
          }
        }
        const double val = HistKeys::value(__ldg(H.values + doc), Q);
        if (!HistKeys::counted(val, H)) continue;
        const unsigned long long b = HistKeys::index(val, Q, base);
        if (b < W.n_bins) atomicAdd(&cells[s * row + (uint32_t)b], 1u);  // (always: the window covers every counted value)
      }
    }
    __syncthreads();
  }
  if (shared)
    for (uint32_t i = threadIdx.x; i < n_kept * W.n_bins; i += blockDim.x)
      if (s_cells[i]) atomicAdd(&gcells[(i / W.n_bins) * G.span + i % W.n_bins], s_cells[i]);
  if (threadIdx.x == 0) {
    const uint32_t seen = U.end - U.begin;
    if (seen) atomicAdd(&P.tiles[0], (unsigned long long)seen);
    if (n_one_key) atomicAdd(&P.tiles[1], (unsigned long long)n_one_key);
    if (n_one_bucket) atomicAdd(&P.tiles[2], (unsigned long long)n_one_bucket);
    if (n_both) atomicAdd(&P.tiles[3], (unsigned long long)n_both);
    atomicAdd(&P.tiles[shared ? 4 : 5], 1ull);
  }
}

// One CTA per (query, segment) of a wave: its non-empty cells, slot by slot in ascending pos, into the wave's cell list.  A first
// pass counts them and takes their place in the list (one atomic on the cursor), a second writes them with a CTA-wide prefix sum
// per 256 cells of the flat grid and records each slot's first cell (the cells before its row).
__global__ void __launch_bounds__(kThreads) k_terms_hist_final(const TermsHistParams P) {
  __shared__ uint32_t s_part[kWarps];
  __shared__ unsigned long long s_at;
  const uint32_t rel = blockIdx.x;
  const TermsSeg Z = P.t.tsegs[P.t.seg_base + rel];
  const TermsHistSeg G = P.gsegs[P.t.seg_base + rel];
  const uint32_t n_kept = P.t.res_n[rel];
  const uint32_t n = n_kept * G.span;  // (<= the grid budget)
  const uint32_t* const cells = P.grid + G.grid;
  uint32_t nz = 0;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) nz += cells[i] ? 1u : 0u;
  uint32_t total;
  cta_scan_excl(nz, s_part, total);
  if (threadIdx.x == 0) {
    s_at = total ? atomicAdd(P.cursor, (unsigned long long)total) : 0ull;
    P.cell_total[rel] = total;
  }
  __syncthreads();
  const uint32_t at = (uint32_t)s_at;  // (the wave's list holds at most its grid's cells)
  uint32_t done = 0;
  for (uint32_t i0 = 0; i0 < n; i0 += blockDim.x) {
    const uint32_t i = i0 + threadIdx.x;
    const uint32_t c = i < n ? cells[i] : 0u;
    uint32_t tot;
    const uint32_t ex = done + cta_scan_excl(c ? 1u : 0u, s_part, tot);
    if (i < n && i % G.span == 0u) P.cell_first[Z.region + i / G.span] = at + ex;
    if (c) {
      P.cell_pos[at + ex] = i % G.span;
      P.cell_count[at + ex] = c;
    }
    done += tot;
  }
  if (!G.span)
    for (uint32_t j = threadIdx.x; j < n_kept; j += blockDim.x) P.cell_first[Z.region + j] = at;
}

// ---- terms per histogram bucket (a histogram whose only sub-aggregation is a terms: SegmentHistogramCollector::collect's
// sub-aggregation branch, histogram.rs:490-505, into one HashMapTermBuckets per bucket) -------------------------------------------
// One CTA per Count unit: each matching doc with a histogram value in its (query, segment)'s bounds counted in cell (its bucket, its
// key's column) -- the image's offset from the segment's key base, or the column of a doc without a value.  Per tile, thread 0 reads
// both columns' SortTile: a tile whose values all hold one image skips the key gather, a tile whose histogram values are all in bounds
// and in one bucket (HistKeys::one) skips the value gather, and a tile with both adds each warp's count to one cell.  A unit whose
// window (its buckets × its keys + 1) fits kTermsHistSmemCells counts in shared memory and adds its non-zero cells to the grid at
// exit; a wider one counts in the grid.  With kTermsHits the unit's matches are added to its query's Count.  (Apart from
// k_terms_hist: that kernel looks each key's slot up in the cut's counters, this one takes the key's offset and feeds no cut, and the
// two share only match_tile and HistKeys.)
template <bool kMixed>
__global__ void __launch_bounds__(kThreads, 3) k_hist_terms(const HistTermsParams P) {
  constexpr uint32_t kNone = 0xFFFFFFFFu;
  __shared__ uint32_t s_acc[kTileDocs / 32u], s_tmp[kTileDocs / 32u];
  __shared__ uint32_t s_cnt[kMixed ? kTileDocs / 4u : 1u];
  __shared__ uint32_t s_cells[kTermsHistSmemCells];
  __shared__ uint32_t s_part[kWarps];
  __shared__ uint32_t s_key, s_bucket;
  const uint32_t unit = P.unit_base + blockIdx.x;
  const Unit U = P.c.units[unit];
  const TermsSeg Z = P.tsegs[U.qseg];
  const HistUnit W = P.hunits[unit], K = P.windows[unit];
  const bool hits = Z.flags & kTermsHits;
  if (!W.n_bins && !hits) return;  // (CTA-uniform: no value of the unit is in bounds, and its Count is not asked for)
  const CountSeg S = P.c.segs[U.qseg];
  const HistSeg H = P.hsegs[U.qseg];
  const HistQuery Q = P.queries[S.query];
  const HistTermsSeg G = P.gsegs[U.qseg];
  const long long base = G.base + (long long)W.first;  // pos of the window's first bucket
  const uint32_t kw = K.n_bins + 1u;                  // the window's columns: the unit's keys, then the docs without a value
  const bool shared = W.n_bins * kw <= kTermsHistSmemCells;  // (W.n_bins * kw <= the (query, segment)'s grid <= its budget < 2^32)
  uint32_t* const gcells = P.grid + G.grid + (unsigned long long)W.first * G.cols;
  auto cell = [&](uint32_t b, uint32_t k) -> uint32_t* {  // cell (bucket b, column k) of the window
    return shared ? &s_cells[b * kw + k] : &gcells[(size_t)b * G.cols + (k == K.n_bins ? G.mcol : K.first + k)];
  };
  if (shared)
    for (uint32_t i = threadIdx.x; i < W.n_bins * kw; i += blockDim.x) s_cells[i] = 0;
  const unsigned long long kbase = Z.base + K.first;  // image of the window's column 0
  const uint32_t wb = S.words_base, ng = P.c.words[wb], need = P.c.words[wb + 1u];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t total = 0, n_one_key = 0, n_one_bucket = 0, n_both = 0;
  for (uint32_t tile = U.begin; tile < U.end; ++tile) {
    const uint32_t lo = tile * kTileDocs, hi = min(lo + kTileDocs, S.max_doc);
    if (threadIdx.x == 0) {
      uint32_t k1 = kNone, b1 = kNone;
      const SortTile T = Z.tiles[tile];
      if ((T.flags & kSortTileValues) && T.best[0] == ~T.best[1] && T.best[0] - kbase < K.n_bins) k1 = (uint32_t)(T.best[0] - kbase);
      const SortTile V = H.tiles[tile];
      if (W.n_bins && (V.flags & kSortTileValues)) HistKeys::one(V, H, Q, W, base, b1);
      s_key = k1;
      s_bucket = b1;
      n_one_key += k1 != kNone ? 1u : 0u;
      n_one_bucket += b1 != kNone ? 1u : 0u;
      n_both += k1 != kNone && b1 != kNone ? 1u : 0u;
    }
    match_tile<kMixed>(P.c, S.alive, wb, ng, need, lo, hi, s_acc, s_tmp, s_cnt, [&](uint32_t w, uint32_t bits) { s_acc[w] = bits; });
    __syncthreads();
    const uint32_t bits = s_acc[threadIdx.x];
    total += (uint32_t)__popc(bits);
    const uint32_t kp = Z.present ? __ldg(Z.present + (lo >> 5) + threadIdx.x) : 0xFFFFFFFFu;
    const uint32_t hp = H.present ? __ldg(H.present + (lo >> 5) + threadIdx.x) : 0xFFFFFFFFu;
    const uint32_t k1 = s_key, b1 = s_bucket;
    const uint32_t dd = W.n_bins ? bits & hp : 0u;  // matching docs with a histogram value
    if (b1 != kNone) {  // every histogram value of the tile counts in bucket b1
      const uint32_t nm = __reduce_add_sync(kFull, (uint32_t)__popc(dd & ~kp));
      if (lane == 0 && nm) atomicAdd(cell(b1, K.n_bins), nm);
      if (k1 != kNone) {
        const uint32_t nk = __reduce_add_sync(kFull, (uint32_t)__popc(dd & kp));
        if (lane == 0 && nk) atomicAdd(cell(b1, k1), nk);
      } else {
        for (uint32_t w = dd & kp; w; w &= w - 1u)
          atomicAdd(cell(b1, (uint32_t)(__ldg(Z.values + lo + threadIdx.x * 32u + (uint32_t)(__ffs(w) - 1)) - kbase)), 1u);
      }
    } else {
      for (uint32_t w = dd; w; w &= w - 1u) {
        const uint32_t bit = (uint32_t)(__ffs(w) - 1), doc = lo + threadIdx.x * 32u + bit;
        const double val = HistKeys::value(__ldg(H.values + doc), Q);
        if (!HistKeys::counted(val, H)) continue;
        const unsigned long long b = HistKeys::index(val, Q, base);
        if (b >= W.n_bins) continue;  // (never: the window covers every counted value)
        const uint32_t k = !((kp >> bit) & 1u) ? K.n_bins : k1 != kNone ? k1 : (uint32_t)(__ldg(Z.values + doc) - kbase);
        atomicAdd(cell((uint32_t)b, k), 1u);
      }
    }
    __syncthreads();
  }
  if (shared)
    for (uint32_t i = threadIdx.x; i < W.n_bins * kw; i += blockDim.x)
      if (s_cells[i]) {
        const uint32_t k = i % kw;
        atomicAdd(&gcells[(size_t)(i / kw) * G.cols + (k == K.n_bins ? G.mcol : K.first + k)], s_cells[i]);
      }
  if (hits) {
    total = __reduce_add_sync(kFull, total);
    if (lane == 0) s_part[warp] = total;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (hits) {
      unsigned long long sum = 0;
      for (int w = 0; w < kWarps; ++w) sum += s_part[w];
      if (sum) atomicAdd(&P.c.counts[S.query], sum);
    }
    const uint32_t seen = U.end - U.begin;
    if (seen) atomicAdd(&P.tiles[0], (unsigned long long)seen);
    if (n_one_key) atomicAdd(&P.tiles[1], (unsigned long long)n_one_key);
    if (n_one_bucket) atomicAdd(&P.tiles[2], (unsigned long long)n_one_bucket);
    if (n_both) atomicAdd(&P.tiles[3], (unsigned long long)n_both);
    if (W.n_bins) atomicAdd(&P.tiles[shared ? 4 : 5], 1ull);
  }
}

// One warp per bucket row of a wave, grid-striding over the wave's rows (a row's (query, segment) found by a binary search over their
// first rows); rows leave in any order, each with its (query, segment), and the host orders them by pos.  Per row:
//   A. its doc count (every cell) and entries (the non-zero entry cells); a row without docs writes nothing;
//   B. a row of a whole segment with more than segment_size entries (partial segments have segment_size above their keys): its
//      entries in key order into the wave's scratch (one ballot per 32 columns, its place taken with one atomic), then §3.7's cut
//      over them alone -- by count, a warp's radix select (4 passes of 8 bits, a 256-bin histogram per warp) finds the count t of
//      the segment_size-th entry and keeps the entries above it and the lowest keys at it; by key, the first or last segment_size
//      -- compacted in place, with term_doc_count_before_cutoff and sum_other_doc_count, and copied to the entry list;
//   C. any other row: its entries in key order straight into the entry list, both scalars 0.
// The grid is read twice (A, then B or C) and only kept entries are written to the list the host copies back.
__global__ void __launch_bounds__(kThreads) k_hist_terms_final(const HistTermsParams P) {
  __shared__ uint32_t s_hist[kWarps][256];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, lt = (1u << lane) - 1u;
  uint32_t* const hist = s_hist[warp];
  uint32_t n_cut = 0;
  for (uint32_t g = blockIdx.x * kWarps + warp; g < P.n_rows; g += gridDim.x * kWarps) {
    uint32_t lo = 0, n = P.n_segs;  // the last (query, segment) of the wave whose first row is <= g
    while (n > 1u) {
      const uint32_t half = n >> 1;
      if (P.gsegs[P.seg_base + lo + half].row <= g) lo += half;
      n -= half;
    }
    const TermsSeg Z = P.tsegs[P.seg_base + lo];
    const HistTermsSeg G = P.gsegs[P.seg_base + lo];
    const uint32_t r = g - G.row;  // (< G.span: a (query, segment) without rows has the next one's first row)
    const uint32_t* const row = P.grid + G.grid + (size_t)r * G.cols;
    const uint32_t L = G.n_entries, ss = Z.segment_size, nc = G.cols;
    const bool all_entries = L == nc;  // (else column nc - 1 is not an entry: docs without a value and without a missing key)
    auto col_of = [&](uint32_t i) -> uint32_t { return G.mfirst ? (i ? i - 1u : nc - 1u) : i; };
    // A
    uint32_t doc = 0, N = 0;
    for (uint32_t i = lane; i < nc; i += 32u) {
      const uint32_t v = row[i];
      doc += v;
      N += v && (i + 1u < nc || all_entries) ? 1u : 0u;
    }
    doc = __reduce_add_sync(kFull, doc);
    N = __reduce_add_sync(kFull, N);
    if (!doc) continue;  // (warp-uniform)
    const bool cut = N > ss;
    unsigned long long at = 0;  // the row's entries: in the scratch when it is cut, else in the list
    if (lane == 0 && N) at = atomicAdd(&P.cursor[cut ? 0 : 1], (unsigned long long)N);
    at = __shfl_sync(kFull, at, 0);
    HistTermsEntry* const E = (cut ? P.ents : P.out_ents) + at;
    unsigned long long sum = 0;
    uint32_t k_at = 0;
    for (uint32_t i0 = 0; N && i0 < L; i0 += 32u) {
      const uint32_t i = i0 + lane;
      const uint32_t v = i < L ? row[col_of(i)] : 0u;
      const uint32_t m = __ballot_sync(kFull, v != 0u);
      if (v) E[k_at + (uint32_t)__popc(m & lt)] = HistTermsEntry{i, v};
      k_at += (uint32_t)__popc(m);
      sum += v;
    }
    uint32_t kept = N, first = (uint32_t)at;  // (the wave's lists hold at most its grid's cells)
    unsigned long long other = 0, error = 0;
    if (cut) {
      __syncwarp();
      const bool asc = Z.flags & kTermsAsc, by_key = Z.flags & kTermsByKey;
      auto rank = [&](uint32_t c) -> uint32_t { return asc ? ~c : c; };  // larger first
      uint32_t t_cut = 0, need = 0, err_t = 0;
      if (!by_key) {
        uint32_t prefix = 0, mask = 0, k = ss, n_eq = 0;
        for (int shift = 24; shift >= 0; shift -= 8) {
          for (uint32_t j = lane; j < 256u; j += 32u) hist[j] = 0;
          __syncwarp();
          for (uint32_t j = lane; j < N; j += 32u) {
            const uint32_t t = rank(E[j].count);
            if ((t & mask) == prefix) atomicAdd(&hist[(t >> shift) & 255u], 1u);
          }
          __syncwarp();
          // the bin of the k-th largest: lane l holds bins [8l, 8l + 8); a suffix sum over the lanes finds the one it falls in
          uint32_t s = 0;
#pragma unroll
          for (uint32_t j = 0; j < 8u; ++j) s += hist[lane * 8u + j];
          uint32_t suf = s;
#pragma unroll
          for (uint32_t d = 1; d < 32u; d <<= 1) {
            const uint32_t y = __shfl_down_sync(kFull, suf, d);
            if (lane + d < 32u) suf += y;
          }
          const bool mine = suf >= k && suf - s < k;  // (one lane: the suffix sums rise to the entries matching the prefix >= k)
          const uint32_t who = (uint32_t)(__ffs(__ballot_sync(kFull, mine)) - 1);
          uint32_t b = 0, acc = 0;
          if (mine) {
            acc = suf - s;
            for (b = lane * 8u + 7u; acc + hist[b] < k; --b) acc += hist[b];
          }
          b = __shfl_sync(kFull, b, who);
          acc = __shfl_sync(kFull, acc, who);
          n_eq = hist[b];
          prefix |= b << shift;
          k -= acc;
          mask |= 255u << shift;
          __syncwarp();
        }
        t_cut = prefix;
        need = k;  // entries at t_cut to keep, the lowest keys first
        // term_doc_count_before_cutoff: t_cut itself when more entries tie at it, else the largest t below it
        uint32_t below = 0;
        if (n_eq <= need)
          for (uint32_t j = lane; j < N; j += 32u) {
            const uint32_t t = rank(E[j].count);
            if (t < t_cut) below = max(below, t);
          }
        err_t = rank(n_eq > need ? t_cut : __reduce_max_sync(kFull, below));
      }
      // the kept entries, compacted in place in key order; by key: the entry ranks kept and the rank whose count is reported
      const uint32_t r0 = by_key && !asc ? N - ss : 0u, r_err = by_key ? (asc ? ss : N - ss - 1u) : 0xFFFFFFFFu;
      uint32_t eq_seen = 0, err_c = 0;
      unsigned long long kept_sum = 0;
      kept = 0;
      for (uint32_t j0 = 0; j0 < N; j0 += 32u) {
        const uint32_t j = j0 + lane;
        const HistTermsEntry e = j < N ? E[j] : HistTermsEntry{0u, 0u};
        const uint32_t t = rank(e.count);
        const bool eq = j < N && !by_key && t == t_cut;
        const uint32_t me = __ballot_sync(kFull, eq);
        const bool keep = j < N && (by_key ? j - r0 < ss : (t > t_cut || (eq && eq_seen + (uint32_t)__popc(me & lt) < need)));
        eq_seen += (uint32_t)__popc(me);
        if (j == r_err) err_c = e.count;
        const uint32_t km = __ballot_sync(kFull, keep);
        __syncwarp();  // (every lane has read its entry before any is overwritten)
        if (keep) E[kept + (uint32_t)__popc(km & lt)] = e;
        kept += (uint32_t)__popc(km);
        kept_sum += keep ? e.count : 0u;
      }
      for (int d = 16; d; d >>= 1) {
        sum += __shfl_xor_sync(kFull, sum, d);
        kept_sum += __shfl_xor_sync(kFull, kept_sum, d);
      }
      other = sum - kept_sum;
      error = by_key ? __reduce_max_sync(kFull, err_c) : err_t;
      unsigned long long to = 0;
      if (lane == 0) to = atomicAdd(&P.cursor[1], (unsigned long long)kept);
      to = __shfl_sync(kFull, to, 0);
      __syncwarp();
      for (uint32_t j = lane; j < kept; j += 32u) P.out_ents[to + j] = E[j];
      first = (uint32_t)to;
      ++n_cut;
    }
    if (lane == 0) {
      const unsigned long long o = atomicAdd(&P.cursor[2], 1ull);
      P.out_rows[o] = HistTermsRow{r, doc, kept, first, lo, 0u, other, error};
    }
  }
  if (lane == 0 && n_cut) atomicAdd(&P.tiles[6], (unsigned long long)n_cut);
}

// The docs a filtered query (TQ_QUERY_FILTER) may collect in one (segment, field): alive AND [doc_lo, doc_hi) AND filter, as 32-bit
// words of the alive layout (FilterCollector over the collection loop that skips deleted docs, filter_collector_wrapper.rs:160-199,
// collector/mod.rs:186-221).  alive null: no deletes.  doc_hi <= max_doc, so the bits at and beyond max_doc come out clear.
__global__ void k_filter_combine(const uint32_t* __restrict__ alive, const uint32_t* __restrict__ filter, uint32_t n_words,
                                 uint32_t doc_lo, uint32_t doc_hi, uint32_t* __restrict__ out) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_words) return;
  const uint32_t lo = w * 32u, a = max(doc_lo, lo), b = min(doc_hi, lo + 32u);
  uint32_t m = 0;
  if (a < b) m = (b - lo == 32u ? 0xFFFFFFFFu : (1u << (b - lo)) - 1u) & ~((1u << (a - lo)) - 1u);
  uint32_t v = filter[w] & m;
  if (alive) v &= alive[w];
  out[w] = v;
}

// The exact k-th largest score key among a query's candidates so far (4-pass radix select) becomes a lower bound of
// its threshold: run between the sampled windows and the main launch of k_or_strip.
__global__ void __launch_bounds__(kThreads) k_theta(const BatchParams P) {
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_prefix, s_need;
  const uint32_t q = blockIdx.x;
  const DQuery Q = P.queries[q];
  if (Q.op == 3u) return;  // TQ_OP_PHRASE: one launch, possibly still running on the batch's second stream
  const uint32_t C = min(P.qstate[q].cand_count, Q.cand_cap);
  if (C < Q.k) return;  // fewer than k hits so far: no bound
  const Cand* cands = P.cands + Q.cand_base;
  if (threadIdx.x == 0) { s_prefix = 0; s_need = Q.k; }
  uint32_t mask = 0;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    for (uint32_t i = threadIdx.x; i < C; i += blockDim.x) {
      const uint32_t key = cands[i].score_key;
      if ((key & mask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t need = s_need, bsel = 0;
      for (int bin = 255; bin >= 0; --bin) {
        const uint32_t h = s_hist[bin];
        if (h >= need) { bsel = (uint32_t)bin; break; }
        need -= h;
      }
      s_need = need;
      s_prefix = prefix | (bsel << shift);
    }
    mask |= 0xFFu << shift;
    __syncthreads();
  }
  if (threadIdx.x == 0) atomicMax(&P.qstate[q].theta, s_prefix);
}

__global__ void k_theta_export(const QState* __restrict__ qs, long long* __restrict__ out, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (long long)qs[i].theta;
}
__global__ void k_theta_import(QState* __restrict__ qs, const long long* __restrict__ in, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicMax(&qs[i].theta, (unsigned int)in[i]);
}

// Exact top-k of a query's candidates. Small sets are sorted directly; large ones go through a
// 4-pass radix select on the score key (O(C)), then only the survivors and the boundary ties are sorted.
__global__ void __launch_bounds__(kThreads) k_final(const BatchParams P) {
  __shared__ unsigned long long s_a[kCap];
  __shared__ uint32_t s_b[kCap];
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_prefix, s_need, s_n, s_ties;
  const uint32_t q = blockIdx.x;
  const DQuery Q = P.queries[q];
  const uint32_t C = min(P.qstate[q].cand_count, Q.cand_cap);
  if (threadIdx.x == 0 && P.ovf && P.qstate[q].cand_count > Q.cand_cap) atomicExch(P.ovf, 1u);  // candidates were dropped: the host repeats the run
  const Cand* cands = P.cands + Q.cand_base;
  uint32_t have = 0;
  if (C <= kCap) {
    for (uint32_t i = threadIdx.x; i < C; i += blockDim.x) {
      const Cand c = cands[i];
      s_a[i] = ((unsigned long long)c.score_key << 32) | (unsigned long long)(0xFFFFFFFFu - c.segment_ord);
      s_b[i] = ~c.doc;
    }
    __syncthreads();
    sort_pairs_desc(s_a, s_b, C);
    have = min(C, Q.k);
  } else {
    // k-th largest score key (C > kCap >= k)
    if (threadIdx.x == 0) { s_prefix = 0; s_need = Q.k; s_n = 0; }  // (s_n: set here, behind the loop's barriers -- the four
                                                                    // words share one vector load further down)
    uint32_t mask = 0;
    for (int pass = 0; pass < 4; ++pass) {
      const int shift = 24 - 8 * pass;
      for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
      __syncthreads();
      const uint32_t prefix = s_prefix;
      for (uint32_t i = threadIdx.x; i < C; i += blockDim.x) {
        const uint32_t key = cands[i].score_key;
        if ((key & mask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255u], 1u);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        uint32_t need = s_need, bsel = 0;
        for (int bin = 255; bin >= 0; --bin) {
          const uint32_t h = s_hist[bin];
          if (h >= need) { bsel = (uint32_t)bin; s_ties = h; break; }
          need -= h;
        }
        s_need = need;
        s_prefix = prefix | (bsel << shift);
      }
      mask |= 0xFFu << shift;
      __syncthreads();
    }
    const uint32_t kth = s_prefix;       // exactly the k-th largest score key
    const uint32_t ties_total = s_ties;   // how many candidates carry exactly that key
    const uint32_t above_total = Q.k - s_need;  // strictly better ones (< k)
    if (above_total + ties_total <= kCap) {  // the usual case: one sweep, one sort
      for (uint32_t i = threadIdx.x; i < C; i += blockDim.x) {
        const Cand c = cands[i];
        if (c.score_key >= kth) {
          const uint32_t slot = atomicAdd(&s_n, 1u);
          s_a[slot] = ((unsigned long long)c.score_key << 32) | (unsigned long long)(0xFFFFFFFFu - c.segment_ord);
          s_b[slot] = ~c.doc;
        }
      }
      __syncthreads();
      const uint32_t n = s_n;
      __syncthreads();
      sort_pairs_desc(s_a, s_b, n);
      have = min(n, Q.k);
    } else {  // a flood of equal scores: keep the best (segment, doc) of the ties slab by slab
      for (uint32_t i = threadIdx.x; i < C; i += blockDim.x) {
        const Cand c = cands[i];
        if (c.score_key > kth) {
          const uint32_t slot = atomicAdd(&s_n, 1u);
          s_a[slot] = ((unsigned long long)c.score_key << 32) | (unsigned long long)(0xFFFFFFFFu - c.segment_ord);
          s_b[slot] = ~c.doc;
        }
      }
      __syncthreads();
      have = s_n;
      uint32_t next = 0;
      for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) s_n = have;
        __syncthreads();
        const uint32_t slab_end = min(C, next + (kCap - have));
        for (uint32_t i = next + threadIdx.x; i < slab_end; i += blockDim.x) {
          const Cand c = cands[i];
          if (c.score_key == kth) {
            const uint32_t slot = atomicAdd(&s_n, 1u);
            s_a[slot] = ((unsigned long long)c.score_key << 32) | (unsigned long long)(0xFFFFFFFFu - c.segment_ord);
            s_b[slot] = ~c.doc;
          }
        }
        __syncthreads();
        const uint32_t n = s_n;
        __syncthreads();
        sort_pairs_desc(s_a, s_b, n);
        have = min(n, Q.k);
        next = slab_end;
        if (next >= C) break;
      }
    }
  }
  for (uint32_t i = threadIdx.x; i < have; i += blockDim.x) {
    const size_t o = (size_t)q * P.res_stride + i;
    P.res_scores[o] = key_to_score((uint32_t)(s_a[i] >> 32));
    P.res_segs[o] = 0xFFFFFFFFu - (uint32_t)s_a[i];
    P.res_docs[o] = ~s_b[i];
  }
  if (threadIdx.x == 0) P.res_counts[q] = have;
}

// K7 (device half): merge_fruits across result sets gathered from several GPUs.
// in: n_lists result sets, each [nq][stride] rows sorted like k_final's output (+ [nq] counts), `row_pitch` / `count_pitch`
// elements apart (contiguous [n_lists][nq][stride] arrays: nq * stride / nq; one packed buffer per shard: its size);
// out: [nq][stride].
__global__ void __launch_bounds__(kThreads) k_merge(uint32_t n_lists, uint32_t nq, uint32_t stride, uint32_t k, size_t row_pitch, size_t count_pitch,
                                                    const float* __restrict__ in_scores, const uint32_t* __restrict__ in_segs,
                                                    const uint32_t* __restrict__ in_docs, const uint32_t* __restrict__ in_counts,
                                                    float* __restrict__ out_scores, uint32_t* __restrict__ out_segs,
                                                    uint32_t* __restrict__ out_docs, uint32_t* __restrict__ out_counts) {
  __shared__ unsigned long long s_a[kCap];
  __shared__ uint32_t s_b[kCap];
  const uint32_t q = blockIdx.x;
  uint32_t have = 0;
  for (uint32_t l = 0; l < n_lists; ++l) {
    const uint32_t cnt = min(min(in_counts[(size_t)l * count_pitch + q], stride), k);
    // have <= k <= 1024 and cnt <= 1024, so have + cnt <= kCap
    for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) {
      const size_t o = (size_t)l * row_pitch + (size_t)q * stride + i;
      s_a[have + i] = ((unsigned long long)score_to_key(in_scores[o]) << 32) | (unsigned long long)(0xFFFFFFFFu - in_segs[o]);
      s_b[have + i] = ~in_docs[o];
    }
    const uint32_t n = have + cnt;
    __syncthreads();
    sort_pairs_desc(s_a, s_b, n);
    have = min(n, k);
  }
  for (uint32_t i = threadIdx.x; i < have; i += blockDim.x) {
    const size_t o = (size_t)q * stride + i;
    out_scores[o] = key_to_score((uint32_t)(s_a[i] >> 32));
    out_segs[o] = 0xFFFFFFFFu - (uint32_t)s_a[i];
    out_docs[o] = ~s_b[i];
  }
  if (threadIdx.x == 0) out_counts[q] = have;
}

}  // namespace tq
