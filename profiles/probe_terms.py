"""Terms aggregations on the device (tq_terms_batch) against Count (tq_count_batch) on the same queries: one 512-query batch of a
bench workload (phrases left out: they are not on the terms path), `_count` desc, size 10 (segment_size 100), on four columns --
about 20 values at random (log levels, status codes), 10 K values clustered in doc order (each value over about ten thousand
consecutive docs: a service or host column of a log index written in bursts), 10 K values at random, and 2^20 values at random
(the widest span the device takes).  Per configuration, medians over the steps of: host wall time of tq_terms_batch and of
tq_count_batch (both synchronous), terms_ms (CUDA events around k_terms + k_terms_select), the 8192-doc tiles seen and the share
counted as one key; with and without a contiguous 10 % filter (TQ_QUERY_FILTER).  Prints the card and its power limit, read in
the same run.  --check: the same configurations at 10M docs (8 segments of 1.25M), every eighth query's rows and scalars compared
with tests/terms_model.py on match sets built from the decoded posting lists (term: its docs; AND: their intersection; OR: their
union; the filter and-ed in).
usage: python profiles/probe_terms.py [--check] [steps] [workload ...]"""
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
from tests import terms_model as TM  # noqa: E402

args = [a for a in sys.argv[1:] if a != "--check"]
CHECK = "--check" in sys.argv
steps = int(args[0]) if args else 5
names = args[1:] or ["or5_top100_100M_8seg", "mixed_top10_100M_8seg"]
NQ, SEED, FID = 512, 0x7A6E7469, 1
STRIDE = 1024  # wider than any row here (8 segments x segment_size 100): each timed call runs once
card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"gpu": card, "check": CHECK}), flush=True)
CONFIGS = [("few_20", 1), ("clustered_10k", 2), ("random_10k", 3), ("random_2^20", 4)]  # (name, column id)
SEGMENT_SIZE = 100  # size 10


def med(xs):
    return round(float(np.median(xs)), 3)


def columns(shard):
    rng = np.random.default_rng(SEED)
    out = {1: [], 2: [], 3: [], 4: []}
    total = sum(shard.ix.max_doc)
    first = 0
    for i, g in enumerate(shard.global_ords):
        n = shard.ix.max_doc[i]
        out[1].append(rng.integers(0, 20, size=n).astype(np.uint64))
        out[2].append(((first + np.arange(n, dtype=np.int64)) * 10_000 // total).astype(np.uint64))
        out[3].append(rng.integers(0, 10_000, size=n).astype(np.uint64))
        out[4].append(rng.integers(0, 1 << 20, size=n).astype(np.uint64))
        first += n
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

    def rows(self, qb, qi, col, filtered):
        """(rows [(segment_ord, key, doc_count)], sum_other, error_bound) of query qi, _count desc."""
        if qi not in self.matches:
            self.matches[qi] = self.match(qb, qi)
        rows, other, error = [], 0, 0
        for i, d in sorted(self.matches[qi], key=lambda x: self.shard.global_ords[x[0]]):
            n = self.shard.ix.max_doc[i]
            if filtered:
                d = d[(d >= int(n * 0.45)) & (d < int(n * 0.55))]
            kept, e, o = TM.cut(TM.collect(col[i][d], None, None), SEGMENT_SIZE)
            rows += [(self.shard.global_ords[i], k, c) for k, c in kept]
            other += o
            error += e
        return rows, other, error

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
        for cname, cid in CONFIGS:
            specs = [(cid, T.TQ_TERMS_BY_COUNT, T.TQ_ORDER_DESC, SEGMENT_SIZE)] * qb.nq
            out = ctx.terms_batch(qb, specs, count_hits=True, stride=STRIDE)  # warm-up (block tables built here)
            assert np.array_equal(out[6], counts), "hits differ from tq_count_batch"
            if CHECK:
                for qi in range(0, qb.nq, 8):  # (every eighth query: the numpy model is the slow part)
                    got = ([(int(out[0][qi, j]), int(out[1][qi, j]), int(out[2][qi, j])) for j in range(int(out[3][qi]))],
                           int(out[4][qi]), int(out[5][qi]))
                    want = model.rows(qb, qi, cols[cid], filtered)
                    assert got == want, f"{name} {cname} filtered={filtered} query {qi}: {got[0][:3]} vs {want[0][:3]}"
            wall, terms_ms, seen, one, cwall = [], [], [], [], []
            for _ in range(steps):
                s0 = ctx.stats()
                t0 = time.perf_counter()
                ctx.terms_batch(qb, specs, stride=STRIDE)
                wall.append(1e3 * (time.perf_counter() - t0))
                s1 = ctx.stats()
                terms_ms.append(s1["terms_ms"] - s0["terms_ms"])
                seen.append(s1["terms_tiles_seen"] - s0["terms_tiles_seen"])
                one.append(s1["terms_tiles_one_key"] - s0["terms_tiles_one_key"])
                t0 = time.perf_counter()
                ctx.count_batch(qb)
                cwall.append(1e3 * (time.perf_counter() - t0))
            print(json.dumps({"workload": name, "docs": sum(shard.ix.max_doc), "queries": qb.nq, "config": cname, "filter_10pct": filtered,
                              "steps": steps, "checked": CHECK, "terms_wall_ms": med(wall), "terms_ms": med(terms_ms), "count_wall_ms": med(cwall),
                              "tiles_seen": int(med(seen)), "one_key_share": round(med(one) / max(med(seen), 1), 3),
                              "max_row": int(out[3].max())}), flush=True)
    ctx.close()
    del shard
