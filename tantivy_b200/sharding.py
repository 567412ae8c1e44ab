"""Segment sharding across GPUs: one process per GPU, segments round-robin over ranks, BM25
statistics summed over all shards, per-rank top-k rows all-gathered and merged.

This is the multi-GPU form of the reference's only parallel axis, one task per segment
(src/core/executor.rs:60-100, src/core/searcher.rs:229-235): the per-segment fruits of a rank are
already merged on its GPU (k_final); the cross-rank step is merge_fruits again
(src/collector/sort_key_top_collector.rs:54-60,76-95) over `world` lists of k rows.
The statistics follow Bm25StatisticsProvider for Searcher (src/query/bm25.rs:27-50):
N = sum of max_doc, avg fieldnorm = sum(total_num_tokens) / N, n = sum of doc_freq."""
import os
import numpy as np

from ._abi import QueryBatch
from .lib import bm25_weight


def assign_segments(n_segments, world, rank):
    """Global segment ordinals owned by `rank` (round-robin: segments are equally sized)."""
    return [s for s in range(n_segments) if s % world == rank]


def assign_parts(n_segments, world, rank):
    """Units of work of `rank`: [(global segment ordinal, part, n_parts)].  With at least as many segments as ranks, whole
    segments round-robin (part 0 of 1).  With fewer, every segment is split by doc-id range into world // n_segments parts
    (SURVEY.md §8e: posting lists are block-addressable through the skip list, so a doc range is a unit of work of its own);
    rank r takes part r // n_segments of segment r % n_segments (ranks beyond n_segments * parts stay idle)."""
    if n_segments >= world:
        return [(s, 0, 1) for s in assign_segments(n_segments, world, rank)]
    parts = world // n_segments
    s, part = rank % n_segments, rank // n_segments
    return [(s, part, parts)] if part < parts else []


def doc_range(max_doc, part, n_parts, tile=1024):
    """Docs [lo, hi) of part `part` of `n_parts`: whole 1024-doc tiles of the tile engine, ceil(max_doc / n_parts) docs each
    (the same cut tq_multi_segment_register_split makes)."""
    per = ((max_doc + n_parts - 1) // n_parts + tile - 1) // tile * tile
    return min(part * per, max_doc), min((part + 1) * per, max_doc)


def range_alive_bitset(max_doc, lo, hi):
    """The alive bitset (bit d & 7 of byte d >> 3, common/src/bitset.rs:362-407) of "only docs [lo, hi) exist here": what a
    target without tq_segment_set_doc_range (the CPU oracle in the tests) gets instead."""
    m = np.zeros(max_doc, dtype=bool)
    m[lo:hi] = True
    return np.packbits(m, bitorder="little")


def global_statistics(local_doc_freq, local_tokens, local_docs, dist=None, device=None):
    """Sums per-term doc_freq, token count and doc count over all ranks (all_reduce)."""
    stats = np.concatenate([np.asarray(local_doc_freq, dtype=np.int64), [int(local_tokens), int(local_docs)]]).astype(np.int64)
    if dist is not None and dist.is_initialized() and dist.get_world_size() > 1:
        import torch
        t = torch.from_numpy(stats)
        if device is not None:
            t = t.to(device)
        dist.all_reduce(t)
        stats = t.cpu().numpy()
    nt = len(local_doc_freq)
    df = stats[:nt]
    tokens, docs = int(stats[nt]), int(stats[nt + 1])
    avg = np.float32(np.float32(tokens) / np.float32(docs)) if docs else np.float32(0)
    return df, tokens, docs, avg


def merge_rows_host(scores, segs, docs, counts, k):
    """Host reference of the cross-rank merge: inputs [world, nq, stride] / [world, nq]; returns rows
    ordered (score desc, segment_ord asc, doc asc), like TopDocs (top_score_collector.rs:591-600)."""
    world, nq, stride = scores.shape
    o_sc = np.zeros((nq, k), np.float32)
    o_sg = np.zeros((nq, k), np.uint32)
    o_dc = np.zeros((nq, k), np.uint32)
    o_ct = np.zeros(nq, np.uint32)
    for q in range(nq):
        rows = []
        for r in range(world):
            n = min(int(counts[r, q]), stride)
            rows += [(-float(scores[r, q, i]), int(segs[r, q, i]), int(docs[r, q, i])) for i in range(n)]
        rows.sort()
        rows = rows[:k]
        o_ct[q] = len(rows)
        for i, (ns, g, d) in enumerate(rows):
            o_sc[q, i], o_sg[q, i], o_dc[q, i] = -ns, g, d
    return o_sc, o_sg, o_dc, o_ct


def score_keys(scores):
    """Order-preserving u32 image of f32 scores, as int64 (host twin of score_to_key in csrc/tq_device.cuh):
    the unit in which shards exchange thresholds; 0 = no bound.  -0.0 and +0.0 share one key (partial_cmp ties them)."""
    u = (np.asarray(scores, dtype=np.float32) + np.float32(0)).view(np.uint32).astype(np.int64)
    return np.where(u >> 31, u ^ 0xFFFFFFFF, u ^ 0x80000000)


def key_scores(keys):
    """Inverse of score_keys."""
    k = np.asarray(keys, dtype=np.int64)
    u = np.where(k >> 31, k ^ 0x80000000, k ^ 0xFFFFFFFF).astype(np.uint32)
    return u.view(np.float32)


def exchange_thresholds(dist, keys):
    """Element-wise MAX of every rank's per-query threshold keys (a torch int64 tensor, in place): any rank's k-th best
    score is a lower bound of the global k-th best, so the largest one is the bound every rank may prune against."""
    dist.all_reduce(keys, op=dist.ReduceOp.MAX)
    return keys


class ShardedIndex:
    """This rank's segments of a SynthIndex-like index plus the global statistics.

    `index` must expose n_segments, max_doc[], total_num_tokens[], term_info[s][t], record_option,
    body(s), fieldnorm(s); `global_ords[i]` is the global ordinal of local segment i."""

    def __init__(self, index, global_ords, n_terms, dist=None, device=None, parts=None):
        """parts[i] = (part, n_parts) of local segment i when it is split by doc range over several ranks (default: whole)."""
        self.ix = index
        self.global_ords = list(global_ords)
        self.parts = list(parts) if parts is not None else [(0, 1)] * len(self.global_ords)
        df = np.zeros(n_terms, dtype=np.int64)
        tokens = docs = 0
        if index is not None:
            for s in range(index.n_segments):
                if self.parts[s][0] != 0:
                    continue  # a split segment is counted once, by the rank that holds its first part
                df += np.array([index.term_info[s][t][0] for t in range(n_terms)], dtype=np.int64)
                tokens += index.total_num_tokens[s]
                docs += index.max_doc[s]
        self.df, self.total_tokens, self.total_docs, self.avg = global_statistics(df, tokens, docs, dist, device)
        self.index_bytes = sum(index.body(s).size + index.fieldnorm(s).size + (index.positions(s).size if index.record_option == 2 else 0)
                               for s in range(index.n_segments)) if index is not None else 0

    def register(self, target):
        for i, g in enumerate(self.global_ords):
            part, n_parts = self.parts[i]
            lo, hi = doc_range(self.ix.max_doc[i], part, n_parts)
            ranged = n_parts > 1 and hasattr(target, "segment_set_doc_range")
            alive = range_alive_bitset(self.ix.max_doc[i], lo, hi) if n_parts > 1 and not ranged else None
            target.segment_register(g, 0, self.ix.max_doc[i], self.ix.record_option, self.ix.body(i), self.ix.fieldnorm(i), alive)
            if ranged:
                target.segment_set_doc_range(g, 0, lo, hi)
            if self.ix.record_option == 2:
                target.register_positions(g, 0, self.ix.positions(i))

    def register_filter(self, target, filter_id, bits_per_local_segment):
        """The doc filter `filter_id` on this rank's segments: bits_per_local_segment[i] = the `.del`-layout bitset of local
        segment i over its whole doc space (a split segment's doc range does the rest on the device)."""
        for i, g in enumerate(self.global_ords):
            target.filter_register(filter_id, g, bits_per_local_segment[i])

    def marshal(self, queries):
        """queries: iterable of (op code, [term ordinals], k) -> QueryBatch restricted to this rank's segments.
        op 3 = phrase (terms in phrase order): ONE Bm25Weight::for_terms weight from the GLOBAL statistics."""
        from .lib import bm25_idf
        out = []
        for op, terms, k in queries:
            term_segs, term_pos = [], []
            for clause, t in enumerate(terms):
                for i, g in enumerate(self.global_ords):
                    d, st, en = self.ix.term_info[i][t]
                    if d:
                        term_segs.append((clause, g, 0, d, st, en))
                        if op == 3:
                            term_pos.append(self.ix.term_pos[i][t])
            if op == 3:
                idf_sum = np.float32(0)
                for t in terms:
                    idf_sum = np.float32(idf_sum + np.float32(bm25_idf(int(self.df[t]), self.total_docs)))
                w = np.float32(idf_sum * np.float32(2.2))
                out.append(dict(op=3, k=k, weights=[w] * len(terms), avg_fieldnorm=[self.avg] * len(terms), term_segs=term_segs, term_pos=term_pos,
                                term_offset=list(range(len(terms)))))
            else:
                weights = [bm25_weight(int(self.df[t]), self.total_docs, 1.0) for t in terms]
                out.append(dict(op=op, k=k, weights=weights, avg_fieldnorm=[self.avg] * len(terms), term_segs=term_segs))
        return QueryBatch(out)


def kth_of_gathered_keys(gathered, ks):
    """Host twin of k_theta_from_keys (csrc/tq_tile.cuh): gathered = [n_shards, nq, k_stride] score keys (0 = nothing), ks[q] =
    the query's k.  Returns per query the k-th largest key of the union, or 0 when fewer than k keys exist: the exact k-th best
    score any single process holding all shards would have found over the same docs (merge_top_k's bound,
    sort_key_top_collector.rs:76-95)."""
    g = np.asarray(gathered, dtype=np.int64)
    n_shards, nq, _ = g.shape
    out = np.zeros(nq, dtype=np.int64)
    for q in range(nq):
        keys = np.sort(g[:, q, :].reshape(-1))[::-1]
        k = int(ks[q])
        out[q] = keys[k - 1] if k <= len(keys) else 0
    return out


def local_topkeys(scores, counts, ks, k_stride):
    """Host twin of k_topkeys_export: the k best score keys of every query's rows, zero padded to k_stride."""
    nq = len(ks)
    out = np.zeros((nq, k_stride), dtype=np.int64)
    for q in range(nq):
        n = min(int(counts[q]), int(ks[q]), k_stride)
        out[q, :n] = score_keys(np.sort(np.asarray(scores[q][:int(counts[q])], dtype=np.float32))[::-1][:n])
    return out


class CrossGpuMerger:
    """The cross-shard steps of a sharded search, all enqueued on the batch's own CUDA stream (no host synchronisation
    between the phases of a run):
      * after every phase but the last, every rank exports the k best score keys it holds per query, ONE NCCL all-gather
        moves them, and the exact k-th best of the union becomes every rank's threshold -- the bound a single GPU holding
        all segments would prune with at that point;
      * at the end ONE all-gather moves every rank's packed result rows (scores | segment ords | docs | counts) and
        k_merge (merge_fruits, sort_key_top_collector.rs:76-95) merges them on the device."""

    def __init__(self, ctx, dist, device, nq, k):
        import torch
        self.ctx, self.dist, self.nq, self.k = ctx, dist, nq, k
        self.world = dist.get_world_size()
        self.torch = torch
        i32 = torch.int32
        self.words = 3 * nq * k + nq
        self.pitch = self.words + 4  # + the run's overflow flags (tq_batch_results_pack_dev_async)
        # keys per rank and query in the threshold exchange: the k-th best of the union of every rank's top-kx is a valid lower
        # bound of the global k-th best for any kx (the keys are scores of distinct docs); it is the exact one unless a shard
        # holds more than kx of the global top-k, which 2k/world + 8 makes unlikely for evenly sharded segments
        self.kx = k if self.world <= 2 else min(k, (2 * k + self.world - 1) // self.world + 8)
        if os.environ.get("TANTIVY_B200_EXCHANGE_KEYS"):  # (tests: any value >= 1 is valid)
            self.kx = max(1, min(k, int(os.environ["TANTIVY_B200_EXCHANGE_KEYS"])))
        self.keys_l = torch.zeros((nq, self.kx), dtype=i32, device=device)
        self.keys_g = torch.zeros((self.world, nq, self.kx), dtype=i32, device=device)
        self.rows_l = torch.zeros((self.pitch,), dtype=i32, device=device)
        self.rows_g = torch.zeros((self.world, self.pitch), dtype=i32, device=device)
        self.rows_o = torch.zeros((self.pitch,), dtype=i32, device=device)
        self.rows_h = None  # pinned host copy of the merged rows (fetch_host)
        self.device = device
        self._ks = {}  # id(QueryBatch) -> (the QueryBatch, each query's own k on the device): the merged counts are clamped to it
        self._streams = {}

    def _check(self, batch):
        """The packed rows are read at stride self.k, and tq_batch_results_pack_dev writes them at the batch's largest k: a batch of
        another shape would be misread without any error."""
        qb = batch.qb
        if qb.nq != self.nq or qb.kmax != self.k:
            raise ValueError(f"CrossGpuMerger(nq={self.nq}, k={self.k}) cannot merge a batch of nq={qb.nq}, k_max={qb.kmax}")
        if id(qb) not in self._ks:  # (one copy per QueryBatch, made before any of its work is queued)
            self._ks[id(qb)] = (qb, self.torch.tensor(qb.q["k"][:self.nq].astype(np.int32), device=self.device))

    def _merge(self, batch, h):
        """k_merge of the gathered rows on stream `h` keeps up to self.k rows per query (the batch's largest k); a query with a
        smaller k keeps its own k, as TopDocs over all the segments would."""
        self.ctx.merge_topk_packed_dev(h, self.world, self.nq, self.k, self.k, self.rows_g.data_ptr(), self.pitch, self.rows_o.data_ptr())
        counts = self.rows_o[3 * self.nq * self.k:self.words]
        self.torch.minimum(counts, self._ks[id(batch.qb)][1], out=counts)

    def _stream(self, batch):
        h = batch.stream()
        if h not in self._streams:
            self._streams[h] = self.torch.cuda.ExternalStream(h)
        return self._streams[h], h

    def run(self, batch):
        """All phases of a prepared batch with the exact threshold exchange in between."""
        self._check(batch)
        ext, _ = self._stream(batch)
        n = batch.phases()
        with self.torch.cuda.stream(ext):  # NCCL orders itself behind / in front of the kernels of this stream
            for phase in range(n):
                batch.run_phase(phase)
                if phase + 1 < n:
                    batch.topkeys_export_dev(self.keys_l.data_ptr(), self.kx)
                    self.dist.all_gather_into_tensor(self.keys_g, self.keys_l)
                    batch.thresholds_from_keys_dev(self.keys_g.data_ptr(), self.world, self.kx)

    def __call__(self, batch):
        """batch: a finished tantivy_b200.Batch of this rank.  Returns (scores, segment ords, docs, counts) device tensors of
        the merged rows (every rank holds them); they are complete once the batch's stream is (torch.cuda.synchronize())."""
        self._check(batch)
        ext, h = self._stream(batch)
        batch.results_pack_dev(self.rows_l.data_ptr())  # waits for the run; the copies are on the batch's stream
        with self.torch.cuda.stream(ext):
            self.dist.all_gather_into_tensor(self.rows_g, self.rows_l)
            self._merge(batch, h)
            self.rows_o[self.words:].zero_()
        return self._views()

    def _views(self):
        r = self.nq * self.k
        o = self.rows_o
        return (o[:r].view(self.torch.float32).view(self.nq, self.k), o[r:2 * r].view(self.nq, self.k), o[2 * r:3 * r].view(self.nq, self.k), o[3 * r:self.words])

    def finish_async(self, batch):
        """__call__ without the wait: pack, all-gather and merge are enqueued behind the run on the batch's stream and the host
        returns at once -- the caller may queue the NEXT batch's run (on its own stream, with a merger of its own) before it waits
        for this one in complete().  The run's overflow flags travel with the rows (4 words per rank; their maximum lands behind
        the merged rows), so every rank takes the same decision in complete()."""
        self._check(batch)
        ext, h = self._stream(batch)
        batch.results_pack_dev_async(self.rows_l.data_ptr())
        with self.torch.cuda.stream(ext):
            self.dist.all_gather_into_tensor(self.rows_g, self.rows_l)
            self._merge(batch, h)
            self.torch.amax(self.rows_g[:, self.words:], dim=0, out=self.rows_o[self.words:])

    def complete(self, batch, rows_to_host=True):
        """Waits for a batch queued with run() + finish_async().  Returns the merged rows as numpy (see fetch_host) when
        rows_to_host, else None.  If ANY rank's tile engine overflowed a buffer, every rank repeats the hand-over on the
        waiting path (tq_batch_results_pack_dev repeats an overflowed run): same collectives on all ranks."""
        batch.results_dev()  # waits for the batch's stream; an overflowed run of THIS rank is repaired here
        ext, _ = self._stream(batch)
        with self.torch.cuda.stream(ext):
            host = (self.rows_o if rows_to_host else self.rows_o[self.words:]).cpu()
        flags = host[-4:]
        self.repeats = getattr(self, "repeats", 0)
        if int(flags.max()) != 0:
            self.repeats += 1
            self(batch)
            if rows_to_host:
                return self.fetch_host(batch)
            ext.synchronize()
            return None
        if not rows_to_host:
            return None
        self.rows_h = host
        return self._host_views(host.numpy())

    def fetch_host(self, batch):
        """After __call__(batch): ONE device-to-host copy of the merged rows, issued on the batch's stream (behind the merge kernel)
        and waited for.  Returns numpy (scores f32 [nq, k], segment ords u32, docs u32, counts u32 [nq]); valid until the next
        fetch_host.  (Pageable host memory on purpose: a pinned torch tensor that outlives the CUDA context aborts the interpreter
        at exit.)"""
        import numpy as np
        ext, _ = self._stream(batch)
        with self.torch.cuda.stream(ext):
            self.rows_h = self.rows_o.cpu()  # cudaMemcpyAsync on `ext` + synchronisation of `ext`
        return self._host_views(self.rows_h.numpy())

    def _host_views(self, a):
        import numpy as np
        r = self.nq * self.k
        return (a[:r].view(np.float32).reshape(self.nq, self.k), a[r:2 * r].view(np.uint32).reshape(self.nq, self.k),
                a[2 * r:3 * r].view(np.uint32).reshape(self.nq, self.k), a[3 * r:self.words].view(np.uint32))
