"""Terms aggregations with metric sub-aggregations on the device (tq_terms_metrics_batch) against the terms alone and the metrics
alone, on the same queries: one 512-query batch of a bench workload (phrases left out: they are not on these paths).  The terms
columns: about 20 random values, 10 K random values, 2^20 random values and 10 K values clustered in doc order (size 10, segment_size
100).  The metric columns: one `stats` on random integers below 10^6, and three columns (those integers, a value constant over about
ten thousand consecutive docs, a count-only column).  Orders `_count` desc and `avg` desc on the first metric column.  Per
configuration, medians over the steps of: host wall time of the call (synchronous), the device ms of its kernels (CUDA events), and
for tq_terms_metrics_batch the share of tiles whose values are one kept key; with and without a contiguous 10 % filter
(TQ_QUERY_FILTER).  Prints the card and its power limit, read in the same run.  --check: the same configurations at 10M docs (8
segments of 1.25M), every 128th query's rows, scalars and parts (the one-column configurations) compared with tests/terms_metrics_model.py (keys, doc counts, count /
min / max per entry, sums the guard accepts bit for bit) on match sets built from the decoded posting lists.
usage: python profiles/probe_terms_metrics.py [--check] [steps] [workload ...]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import tantivy_b200 as T  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_PHRASE, TQ_QUERY_FILTER, TQ_TERMS_BY_COUNT, TQ_TERMS_BY_METRIC, TQ_TERMS_ORDER_AVG  # noqa: E402
from tantivy_b200 import metrics as Mx  # noqa: E402
from tests import terms_metrics_model as TMM  # noqa: E402

args = [a for a in sys.argv[1:] if a != "--check"]
CHECK = "--check" in sys.argv
steps = int(args[0]) if args else 5
names = args[1:] or ["or5_top100_100M_8seg", "mixed_top10_100M_8seg"]
NQ, SEED, FID, SS = 512, 0x7E3A, 1, 100
card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"gpu": card, "check": CHECK}), flush=True)
R20, R10K, R1M, C10K, RAND, CLUSTERED, COUNT_ONLY = 1, 2, 3, 4, 5, 6, 7
TERMS = {"r20": R20, "r10k": R10K, "r1m": R1M, "c10k": C10K}
STATS = [(RAND, T.TQ_FAST_U64, 0)]
THREE = [(RAND, T.TQ_FAST_U64, 0), (CLUSTERED, T.TQ_FAST_U64, 0), (COUNT_ONLY, T.TQ_FAST_U64, T.TQ_METRIC_COUNT_ONLY)]
ORDERS = {"count": None, "avg": (0, TQ_TERMS_ORDER_AVG)}


def med(xs):
    return round(float(np.median(xs)), 3)


def columns(shard):
    rng = np.random.default_rng(SEED)
    out = {k: [] for k in (R20, R10K, R1M, C10K, RAND, CLUSTERED, COUNT_ONLY)}
    total = sum(shard.ix.max_doc)
    first = 0
    for i, _ in enumerate(shard.global_ords):
        n = shard.ix.max_doc[i]
        at = first + np.arange(n, dtype=np.int64)
        out[R20].append(rng.integers(0, 20, size=n).astype(np.uint64))
        out[R10K].append(rng.integers(0, 10_000, size=n).astype(np.uint64))
        out[R1M].append(rng.integers(0, 1 << 20, size=n).astype(np.uint64))
        out[C10K].append((at * 10_000 // total).astype(np.uint64))
        out[RAND].append(rng.integers(0, 10**6, size=n).astype(np.uint64))
        out[CLUSTERED].append((at * 10_000 // total * 37).astype(np.uint64))
        out[COUNT_ONLY].append(rng.integers(0, 20, size=n).astype(np.uint64))  # (a str column's ordinals: never read)
        first += n
    return out


def filter_bits(n):
    m = np.zeros(n, bool)
    m[int(n * 0.45):int(n * 0.55)] = True
    return np.packbits(m, bitorder="little")


def match(ctx, shard, qb, qi, cache):
    """[(segment index, matching docs)] of query qi, from the decoded posting lists (the synthetic segments have no deletes)."""
    q = qb.q[qi]
    n_ts = int(q["n_term_segs"])
    start = (int(q["term_segs"]) - qb.term_segs.ctypes.data) // qb.term_segs.itemsize
    out = []
    for i, g in enumerate(shard.global_ords):
        lists = []
        for t in qb.term_segs[start:start + n_ts]:
            if int(t["segment_ord"]) != g:
                continue
            key = tuple(int(x) for x in t)
            if key not in cache:
                cache[key] = ctx.decode_postings(key)[0].astype(np.int64)
            lists.append(cache[key])
        if not lists or (q["op"] == TQ_OP_AND and len(lists) < int(q["n_terms"])):
            continue
        m = np.zeros(shard.ix.max_doc[i], bool)
        if q["op"] == TQ_OP_AND:
            m[lists[0]] = True
            for other in lists[1:]:
                mm = np.zeros_like(m)
                mm[other] = True
                m &= mm
        else:
            for other in lists:
                m[other] = True
        out.append((i, np.nonzero(m)[0]))
    return out


class _Values:
    """values[d] of a column as terms_metrics_model.collect reads it: the doc's one value (0.0 on a count-only column)."""

    def __init__(self, images, count_only):
        self.images, self.count_only = images, count_only

    def __getitem__(self, d):
        return [0.0] if self.count_only else [float(self.images[d])]


def check_query(shard, cols, matches, filtered, tcol, spec, order, out, qi):
    """One query's device rows against the model: per segment the docs by key in doc order, Kahan per (key, column), the cut."""
    rows, other, error = [], 0, 0
    for i, d in sorted(matches, key=lambda x: shard.global_ords[x[0]]):
        n = shard.ix.max_doc[i]
        if filtered:
            d = d[(d >= int(n * 0.45)) & (d < int(n * 0.55))]
        sel = np.zeros(n, bool)
        sel[d] = True
        docs = TMM.segment_docs(cols[tcol][i], None, sel)
        vals = [_Values(cols[cid][i], flags & T.TQ_METRIC_COUNT_ONLY) for cid, _, flags in spec]
        entries = {k: (len(ds), {j: TMM.collect(vals[j], ds) for j in range(len(spec))}) for k, ds in docs.items()}
        kept, e, o = TMM.cut(entries, SS, "_count" if order is None else "metric", False, None if order is None else (0, "avg"))
        rows += [(shard.global_ords[i], k, c, st) for k, (c, st) in sorted(kept.items())]
        other, error = other + o, error + e
    n = int(out[4][qi])
    assert [(int(out[0][qi, j]), int(out[1][qi, j]), int(out[2][qi, j])) for j in range(n)] == [r[:3] for r in rows], "rows differ"
    assert (int(out[5][qi]), int(out[6][qi])) == (other, error), "scalars differ"
    for j, (_, _, _, st) in enumerate(rows):
        for c, (_, ckind, flags) in enumerate(spec):
            count, s, vmin, vmax = Mx.stats_of(out[3][qi, j, c], ckind, flags)
            assert count == st[c].count and (count == 0 or (vmin, vmax) == (st[c].min, st[c].max)), ("count/min/max", j, c)
            if Mx.guard(out[3][qi, j, c]) is None:
                assert s == st[c].sum, ("sum", j, c, s, st[c].sum)


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
    postings = {}
    for filtered in (False, True):
        qb = bench.marshal(shard, [(op, terms, 10) for op, terms, _ in queries])
        if filtered:
            qb.q["flags"][:qb.nq] |= TQ_QUERY_FILTER
            qb.q["filter_id"][:qb.nq] = FID
        counts = ctx.count_batch(qb)
        matches = {}
        configs = [("metrics_stats", None, STATS, None), ("metrics_three", None, THREE, None)]
        for tname, tcol in TERMS.items():
            configs.append((f"terms_{tname}", tcol, None, None))
            for sname, spec in (("stats", STATS), ("three", THREE)):
                for oname, order in ORDERS.items():
                    configs.append((f"tm_{tname}_{sname}_{oname}", tcol, spec, order))
        for cname, tcol, spec, order in configs:
            tspec = None if tcol is None else (tcol, TQ_TERMS_BY_COUNT if order is None else TQ_TERMS_BY_METRIC, T.TQ_ORDER_DESC, SS)
            if spec is None:
                run, ms_key, units_key = (lambda: ctx.terms_batch(qb, [tspec] * qb.nq, stride=8 * SS)), "terms_ms", "units_terms"
            elif tcol is None:
                run, ms_key, units_key = (lambda: ctx.metrics_batch(qb, [spec] * qb.nq)), "metrics_ms", "units_metrics"
            else:
                out = ctx.terms_metrics_batch(qb, [tspec] * qb.nq, [spec] * qb.nq, [order] * qb.nq, count_hits=True)  # warm-up; hits checked
                assert np.array_equal(out[8], counts), "hits differ from tq_count_batch"
                run, ms_key, units_key = (lambda: ctx.terms_metrics_batch(qb, [tspec] * qb.nq, [spec] * qb.nq, [order] * qb.nq)), \
                    "terms_metrics_ms", "units_terms_metrics"
                if CHECK and spec is STATS:
                    for qi in range(0, qb.nq, 128):  # (every 128th query, one column: the Python model is the slow part)
                        if qi not in matches:
                            matches[qi] = match(ctx, shard, qb, qi, postings)
                        check_query(shard, cols, matches[qi], filtered, tcol, spec, order, out, qi)
            run()
            wall, dev, seen, one = [], [], [], []
            for _ in range(steps):
                s0 = ctx.stats()
                t0 = time.perf_counter()
                run()
                wall.append(1e3 * (time.perf_counter() - t0))
                s1 = ctx.stats()
                dev.append(s1[ms_key] - s0[ms_key])
                seen.append(s1["terms_metrics_tiles_seen"] - s0["terms_metrics_tiles_seen"])
                one.append(s1["terms_metrics_tiles_one_key"] - s0["terms_metrics_tiles_one_key"])
            rec = {"workload": name, "docs": sum(shard.ix.max_doc), "queries": qb.nq, "config": cname, "filter_10pct": filtered, "steps": steps,
                   "checked": CHECK, "wall_ms": med(wall), "device_ms": med(dev)}
            if ms_key == "terms_metrics_ms":
                rec.update({"tiles_seen": int(med(seen)), "one_key_share": round(med(one) / max(med(seen), 1), 3)})
            print(json.dumps(rec), flush=True)
    ctx.close()
    del shard
