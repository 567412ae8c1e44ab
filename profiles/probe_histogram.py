"""Histogram aggregations on the device (tq_histogram_batch) against Count (tq_count_batch) on the same queries: one 512-query
batch of a bench workload (phrases left out: they are not on the histogram path), on two columns -- a date column ascending in
doc id over the segments in turn (one doc every 7 ms: the log-search case) at a 1 min and a 1 h interval, and uniform random u64
images at 100 buckets.  Per configuration, medians over the steps of: host wall time of tq_histogram_batch and of tq_count_batch
(both synchronous), hist_ms (CUDA events around k_hist + k_hist_final), the 8192-doc tiles seen and the share counted as one
bucket; with and without a contiguous 10 % filter (TQ_QUERY_FILTER).  Prints the card and its power limit, read in the same run.
--check: the same configurations at 10M docs (8 segments of 1.25M), every row compared with a numpy model built from the
decoded posting lists (term: its docs; AND: their intersection; OR: their union; the filter and-ed in), every eighth query.
usage: python profiles/probe_histogram.py [--check] [steps] [workload ...]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import tantivy_b200 as T  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_PHRASE, TQ_QUERY_FILTER  # noqa: E402
from tests import histogram_model as HM  # noqa: E402

args = [a for a in sys.argv[1:] if a != "--check"]
CHECK = "--check" in sys.argv
steps = int(args[0]) if args else 5
names = args[1:] or ["or5_top100_100M_8seg", "mixed_top10_100M_8seg"]
NQ, SEED, FID = 512, 0x7A6E7469, 1
STRIDE = 16384  # wider than any row here: each timed call runs once
card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"gpu": card, "check": CHECK}), flush=True)
# (name, column id, kind, interval, offset)
CONFIGS = [("date_1min", 1, "date", 60e9, 0.0), ("date_1h", 1, "date", 3600e9, 0.0), ("random_100", 2, "u64", float(2**64) / 100, 0.0)]


def med(xs):
    return round(float(np.median(xs)), 3)


def columns(shard):
    rng = np.random.default_rng(SEED)
    out = {1: [], 2: []}
    base = np.int64(1_700_000_000) * 10**9
    for i, g in enumerate(shard.global_ords):
        n = shard.ix.max_doc[i]
        out[1].append(T.fast_value_to_u64(base + np.int64(g) * np.int64(n) * 7_000_000 + np.arange(n, dtype=np.int64) * 7_000_000, "date"))
        out[2].append(rng.integers(0, 2**64 - 1, size=n, dtype=np.uint64, endpoint=True))
    return out


def filter_bits(n):
    m = np.zeros(n, bool)
    m[int(n * 0.45):int(n * 0.55)] = True
    return np.packbits(m, bitorder="little")


class Model:
    """Match sets from the decoded posting lists (the synthetic segments have no deletes)."""

    def __init__(self, ctx, shard):
        self.ctx, self.shard, self.cache, self.matches = ctx, shard, {}, {}

    def docs(self, ts):
        key = (ts[1], ts[4])
        if key not in self.cache:
            self.cache[key] = self.ctx.decode_postings(ts)[0].astype(np.int64)
        return self.cache[key]

    def rows(self, qb, qi, col, kind, interval, offset, filtered):
        if qi not in self.matches:
            self.matches[qi] = self.match(qb, qi)
        parts = []
        for i, d in self.matches[qi]:
            n = self.shard.ix.max_doc[i]
            if filtered:
                d = d[(d >= int(n * 0.45)) & (d < int(n * 0.55))]
            parts.append(HM.collect(col[i][d], None, None, kind, interval, offset))  # (no hard bounds)
        return sorted(HM.merge(parts).items())

    def match(self, qb, qi):
        """[(segment index, matching docs)] of query qi."""
        q = qb.q[qi]
        n_ts = int(q["n_term_segs"])
        start = (int(q["term_segs"]) - qb.term_segs.ctypes.data) // qb.term_segs.itemsize
        ts = qb.term_segs[start:start + n_ts]
        out = []
        for i, g in enumerate(self.shard.global_ords):
            lists = [self.docs(tuple(int(x) for x in t)) for t in ts if int(t["segment_ord"]) == g]
            if not lists or (q["op"] == TQ_OP_AND and len(lists) < int(q["n_terms"])):
                continue
            if q["op"] == TQ_OP_AND:
                d = lists[0]
                for other in lists[1:]:
                    d = np.intersect1d(d, other, assume_unique=True)
            else:  # (a mask, not union1d: the sort behind union1d is the slow part on dense unions)
                m = np.zeros(self.shard.ix.max_doc[i], bool)
                for other in lists:
                    m[other] = True
                d = np.nonzero(m)[0]
            out.append((i, d))
        return out


for name in names:
    wl = dict(bench.WORKLOADS[name])
    if CHECK:
        wl["docs_per_segment"] = 10_000_000 // wl["n_segments"]
    dens, batches = bench.build_query_plan(wl, NQ, 1, SEED)
    shard = bench.make_shard(wl, dens, 0, 1, SEED)
    ctx = T.Context(0)
    shard.register(ctx)
    cols = columns(shard)
    for cid, per_seg in cols.items():
        for i, g in enumerate(shard.global_ords):
            ctx.sort_column_register(cid, g, per_seg[i])
    for i, g in enumerate(shard.global_ords):
        ctx.filter_register(FID, g, filter_bits(shard.ix.max_doc[i]))
    queries = [q for q in batches[0] if bench.OPS[q[0]] != TQ_OP_PHRASE]
    model = Model(ctx, shard) if CHECK else None
    for filtered in (False, True):
        qb = bench.marshal(shard, [(op, terms, 10) for op, terms, _ in queries])
        if filtered:
            qb.q["flags"][:qb.nq] |= TQ_QUERY_FILTER
            qb.q["filter_id"][:qb.nq] = FID
        counts = ctx.count_batch(qb)
        for cname, cid, kind, interval, offset in CONFIGS:
            specs = [(cid, kind, interval, offset)] * qb.nq
            out = ctx.histogram_batch(qb, specs, count_hits=True, stride=STRIDE)  # warm-up (block tables built here)
            assert np.array_equal(out[3], counts), "hits differ from tq_count_batch"
            if CHECK:
                for qi in range(0, qb.nq, 8):  # (every eighth query: the numpy model is the slow part)
                    got = [(int(out[0][qi, j]), int(out[1][qi, j])) for j in range(int(out[2][qi]))]
                    want = model.rows(qb, qi, cols[cid], kind, interval, offset, filtered)
                    assert got == want, f"{name} {cname} filtered={filtered} query {qi}: {got[:3]} vs {want[:3]}"
            wall, hist_ms, seen, one, cwall = [], [], [], [], []
            for _ in range(steps):
                s0 = ctx.stats()
                t0 = time.perf_counter()
                ctx.histogram_batch(qb, specs, stride=STRIDE)
                wall.append(1e3 * (time.perf_counter() - t0))
                s1 = ctx.stats()
                hist_ms.append(s1["hist_ms"] - s0["hist_ms"])
                seen.append(s1["hist_tiles_seen"] - s0["hist_tiles_seen"])
                one.append(s1["hist_tiles_one_bucket"] - s0["hist_tiles_one_bucket"])
                t0 = time.perf_counter()
                ctx.count_batch(qb)
                cwall.append(1e3 * (time.perf_counter() - t0))
            print(json.dumps({"workload": name, "docs": sum(shard.ix.max_doc), "queries": qb.nq, "config": cname, "filter_10pct": filtered,
                              "steps": steps, "checked": CHECK, "hist_wall_ms": med(wall), "hist_ms": med(hist_ms), "count_wall_ms": med(cwall),
                              "tiles_seen": int(med(seen)), "one_bucket_share": round(med(one) / max(med(seen), 1), 3),
                              "max_buckets": int(out[2].max())}), flush=True)
    ctx.close()
    del shard
