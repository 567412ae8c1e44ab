"""Metric aggregations on the device (tq_metrics_batch) against Count (tq_count_batch) on the same queries: one 512-query batch of a
bench workload (phrases left out: they are not on the metrics path), one `stats` per query on one of three columns -- random
integers below 10^6 (byte counts), a value constant over about ten thousand consecutive docs (clustered in doc order: one-value
tiles) and a count-only column (value_count on a str field: the docs with a value are counted, no value is read) -- and on all three
at once (one spec of three columns, one match pass).  Per configuration, medians over the steps of: host wall time of
tq_metrics_batch and of tq_count_batch (both synchronous), metrics_ms (CUDA events around k_metrics), the (tile, column) pairs
seen and the share added as one value, and the share of queries whose sum the guard accepts; with and without a contiguous 10 %
filter (TQ_QUERY_FILTER).  Prints the card and its power limit, read in the same run.  --check: the same configurations at 10M docs
(8 segments of 1.25M), every eighth query's stats compared with tests/metrics_model.py (Kahan in doc order, segments in
segment_ord order) on match sets built from the decoded posting lists.
usage: python profiles/probe_metrics.py [--check] [steps] [workload ...]"""
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
from tantivy_b200 import metrics as Mx  # noqa: E402
from tests import metrics_model as MM  # noqa: E402

args = [a for a in sys.argv[1:] if a != "--check"]
CHECK = "--check" in sys.argv
steps = int(args[0]) if args else 5
names = args[1:] or ["or5_top100_100M_8seg", "mixed_top10_100M_8seg"]
NQ, SEED, FID = 512, 0x7A6E7469, 1
card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"gpu": card, "check": CHECK}), flush=True)
# (name, [(column id, kind, flags)]): the spec of every query
RANDOM, CLUSTERED, COUNT_ONLY = (1, T.TQ_FAST_U64, 0), (2, T.TQ_FAST_U64, 0), (3, T.TQ_FAST_U64, T.TQ_METRIC_COUNT_ONLY)
CONFIGS = [("random_int", [RANDOM]), ("clustered", [CLUSTERED]), ("count_only", [COUNT_ONLY]), ("all_three", [RANDOM, CLUSTERED, COUNT_ONLY])]


def med(xs):
    return round(float(np.median(xs)), 3)


def columns(shard):
    rng = np.random.default_rng(SEED)
    out = {1: [], 2: [], 3: []}
    total = sum(shard.ix.max_doc)
    first = 0
    for i, g in enumerate(shard.global_ords):
        n = shard.ix.max_doc[i]
        out[1].append(rng.integers(0, 10**6, size=n).astype(np.uint64))
        out[2].append(((first + np.arange(n, dtype=np.int64)) * 10_000 // total * 37).astype(np.uint64))
        out[3].append(rng.integers(0, 20, size=n).astype(np.uint64))  # (a str column's ordinals: never read)
        first += n
    return out


def filter_bits(n):
    m = np.zeros(n, bool)
    m[int(n * 0.45):int(n * 0.55)] = True
    return np.packbits(m, bitorder="little")


class Model:
    """Match sets from the decoded posting lists (the synthetic segments have no deletes)."""

    def __init__(self, ctx, shard):
        self.ctx, self.shard, self.cache, self.lists, self.matches = ctx, shard, {}, {}, {}

    def docs(self, ts):
        key = (ts[1], ts[4])
        if key not in self.lists:
            self.lists[key] = self.ctx.decode_postings(ts)[0].astype(np.int64)
        return self.lists[key]

    def stats(self, qb, qi, col, filtered, count_only):
        """metrics_model's merged IntermediateStats of query qi on one column."""
        key = (qi, id(col), filtered, count_only)
        if key in self.cache:
            return self.cache[key]
        if qi not in self.matches:
            self.matches[qi] = self.match(qb, qi)
        segs = []
        for i, d in sorted(self.matches[qi], key=lambda x: self.shard.global_ords[x[0]]):
            n = self.shard.ix.max_doc[i]
            if filtered:
                d = d[(d >= int(n * 0.45)) & (d < int(n * 0.55))]
            vals = np.zeros(len(d)) if count_only else col[i][d].astype(np.float64)
            segs.append(MM.segment_stats(vals.tolist()))
        self.cache[key] = MM.merged(segs)
        return self.cache[key]

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
        for cname, spec in CONFIGS:
            specs = [spec] * qb.nq
            parts, hits = ctx.metrics_batch(qb, specs, count_hits=True)  # warm-up (block tables built here)
            assert np.array_equal(hits, counts), "hits differ from tq_count_batch"
            accepted = [all(Mx.guard(parts[qi, j]) is None for j in range(len(spec))) for qi in range(qb.nq)]
            if CHECK:
                for qi in range(0, qb.nq, 8):  # (every eighth query: the Python model is the slow part)
                    for j, (cid, kind, flags) in enumerate(spec):
                        st = model.stats(qb, qi, cols[cid], filtered, flags & T.TQ_METRIC_COUNT_ONLY)
                        count, s, vmin, vmax = Mx.stats_of(parts[qi, j], kind, flags)
                        assert count == st.count and (count == 0 or (vmin, vmax) == (st.min, st.max)), (name, cname, qi)
                        if Mx.guard(parts[qi, j]) is None:
                            assert s == st.sum, (name, cname, qi, s, st.sum)
            wall, metrics_ms, seen, one, cwall = [], [], [], [], []
            for _ in range(steps):
                s0 = ctx.stats()
                t0 = time.perf_counter()
                ctx.metrics_batch(qb, specs)
                wall.append(1e3 * (time.perf_counter() - t0))
                s1 = ctx.stats()
                metrics_ms.append(s1["metrics_ms"] - s0["metrics_ms"])
                seen.append(s1["metrics_tiles_seen"] - s0["metrics_tiles_seen"])
                one.append(s1["metrics_tiles_one_value"] - s0["metrics_tiles_one_value"])
                t0 = time.perf_counter()
                ctx.count_batch(qb)
                cwall.append(1e3 * (time.perf_counter() - t0))
            print(json.dumps({"workload": name, "docs": sum(shard.ix.max_doc), "queries": qb.nq, "config": cname, "filter_10pct": filtered,
                              "steps": steps, "checked": CHECK, "metrics_wall_ms": med(wall), "metrics_ms": med(metrics_ms), "count_wall_ms": med(cwall),
                              "tiles_seen": int(med(seen)), "one_value_share": round(med(one) / max(med(seen), 1), 3),
                              "guard_accepted": round(sum(accepted) / max(qb.nq, 1), 3)}), flush=True)
    ctx.close()
    del shard
