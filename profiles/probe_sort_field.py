"""TopDocs::order_by_fast_field on the device (tq_sort_batch) against Count (tq_count_batch) on the same queries: one 512-query
batch of a bench workload (phrases left out: they are not on the sort path), k = 10 and 100, Desc and Asc, on two columns -- a
timestamp ascending in doc id over the segments in turn (the log-search case) and uniform random u64 images.  Per configuration,
medians over the steps of: host wall time of tq_sort_batch and of tq_count_batch (both synchronous), sort_ms (CUDA events around
k_sort + k_sort_final) and the 8192-doc tiles seen and skipped; the same with count_hits=True (every tile visited) and with a
contiguous 10 % filter (TQ_QUERY_FILTER).  Prints the card and its power limit, read in the same run.
--check: the same configurations at 10M docs (8 segments of 1.25M), every row compared with a numpy model built from the
decoded posting lists (term: its docs; AND: their intersection; OR: their union; the filter and-ed in), every fourth query.
usage: python profiles/probe_sort_field.py [--check] [steps] [workload ...]"""
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

args = [a for a in sys.argv[1:] if a != "--check"]
CHECK = "--check" in sys.argv
steps = int(args[0]) if args else 5
names = args[1:] or ["or5_top100_100M_8seg", "mixed_top10_100M_8seg"]
NQ, SEED, FID = 512, 0x7A6E7469, 1
COLS = {"timestamp": 1, "random": 2}
card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"gpu": card, "check": CHECK}), flush=True)


def med(xs):
    return round(float(np.median(xs)), 3)


def columns(shard):
    rng = np.random.default_rng(SEED)
    out = {"timestamp": [], "random": []}
    base = np.uint64(1_700_000_000_000_000)
    for i, g in enumerate(shard.global_ords):
        n = shard.ix.max_doc[i]
        out["timestamp"].append(base + np.uint64(g) * np.uint64(10**9) + np.arange(n, dtype=np.uint64) * np.uint64(7))
        out["random"].append(rng.integers(0, 2**64 - 1, size=n, dtype=np.uint64, endpoint=True))
    return out


def filter_bits(n):
    m = np.zeros(n, bool)
    m[int(n * 0.45):int(n * 0.55)] = True
    return np.packbits(m, bitorder="little")


class Model:
    """Match sets from the decoded posting lists (the synthetic segments have no deletes)."""

    def __init__(self, ctx, shard):
        self.ctx, self.shard, self.cache = ctx, shard, {}

    def docs(self, ts):
        key = (ts[1], ts[4])
        if key not in self.cache:
            self.cache[key] = self.ctx.decode_postings(ts)[0].astype(np.int64)
        return self.cache[key]

    def rows(self, qb, qi, cols, order, k, filtered):
        q = qb.q[qi]
        n_ts = int(q["n_term_segs"])
        start = (int(q["term_segs"]) - qb.term_segs.ctypes.data) // qb.term_segs.itemsize
        ts = qb.term_segs[start:start + n_ts]
        vals, sos, docs = [], [], []
        for i, g in enumerate(self.shard.global_ords):
            lists = [self.docs(tuple(int(x) for x in t)) for t in ts if int(t["segment_ord"]) == g]
            if not lists or (q["op"] == TQ_OP_AND and len(lists) < int(q["n_terms"])):
                continue
            d = lists[0]
            for other in lists[1:]:
                d = np.intersect1d(d, other) if q["op"] == TQ_OP_AND else np.union1d(d, other)
            if filtered:
                n = self.shard.ix.max_doc[i]
                d = d[(d >= int(n * 0.45)) & (d < int(n * 0.55))]
            vals.append(cols[i][d])
            sos.append(np.full(len(d), g, np.int64))
            docs.append(d)
        if not vals:
            return []
        v, s, d = np.concatenate(vals), np.concatenate(sos), np.concatenate(docs)
        key = v if order == "desc" else ~v
        idx = np.lexsort((d, s, ~key))[:k]
        return [(int(v[j]), int(s[j]), int(d[j])) for j in idx]


for name in names:
    wl = dict(bench.WORKLOADS[name])
    if CHECK:
        wl["docs_per_segment"] = 10_000_000 // wl["n_segments"]
    dens, batches = bench.build_query_plan(wl, NQ, 1, SEED)
    shard = bench.make_shard(wl, dens, 0, 1, SEED)
    ctx = T.Context(0)
    shard.register(ctx)
    cols = columns(shard)
    for cname, cid in COLS.items():
        for i, g in enumerate(shard.global_ords):
            ctx.sort_column_register(cid, g, cols[cname][i])
    for i, g in enumerate(shard.global_ords):
        ctx.filter_register(FID, g, filter_bits(shard.ix.max_doc[i]))
    queries = [q for q in batches[0] if bench.OPS[q[0]] != TQ_OP_PHRASE]
    model = Model(ctx, shard) if CHECK else None
    for k in (10, 100):
        for filtered in (False, True):
            qb = bench.marshal(shard, [(op, terms, k) for op, terms, _ in queries])
            if filtered:
                qb.q["flags"][:qb.nq] |= TQ_QUERY_FILTER
                qb.q["filter_id"][:qb.nq] = FID
            counts = ctx.count_batch(qb)
            for cname, cid in COLS.items():
                for order in ("desc", "asc"):
                    res, rows = {}, None
                    for hits in (False, True):
                        specs = [(cid, order)] * qb.nq
                        out = ctx.sort_batch(qb, specs, count_hits=hits)  # warm-up (block tables built here)
                        if hits:
                            assert np.array_equal(out[5], counts), "hits differ from tq_count_batch"
                            assert all(np.array_equal(a, b) for a, b in zip(out[:5], rows)), "rows differ with count_hits"
                        rows = out[:5]
                        if CHECK and not hits:
                            for qi in range(0, qb.nq, 4):  # (every fourth query: the numpy model is the slow part)
                                got = [(int(out[0][qi, j]), int(out[2][qi, j]), int(out[3][qi, j])) for j in range(int(out[4][qi]))]
                                want = model.rows(qb, qi, cols[cname], order, k, filtered)
                                assert got == want, f"{name} {cname} {order} k={k} filtered={filtered} query {qi}: {got[:3]} vs {want[:3]}"
                        wall, sort_ms, seen, skipped, cwall = [], [], [], [], []
                        for _ in range(steps):
                            s0 = ctx.stats()
                            t0 = time.perf_counter()
                            ctx.sort_batch(qb, specs, count_hits=hits)
                            wall.append(1e3 * (time.perf_counter() - t0))
                            s1 = ctx.stats()
                            sort_ms.append(s1["sort_ms"] - s0["sort_ms"])
                            seen.append(s1["sort_tiles_seen"] - s0["sort_tiles_seen"])
                            skipped.append(s1["sort_tiles_skipped"] - s0["sort_tiles_skipped"])
                            t0 = time.perf_counter()
                            ctx.count_batch(qb)
                            cwall.append(1e3 * (time.perf_counter() - t0))
                        res["count_hits" if hits else "rows_only"] = {"sort_wall_ms": med(wall), "sort_ms": med(sort_ms), "tiles_seen": int(med(seen)),
                                                                      "tiles_skipped": int(med(skipped)), "count_wall_ms": med(cwall)}
                    print(json.dumps({"workload": name, "docs": sum(shard.ix.max_doc), "queries": qb.nq, "k": k, "column": cname, "order": order,
                                      "filter_10pct": filtered, "steps": steps, "checked": CHECK, **res}), flush=True)
    ctx.close()
    del shard
