"""Histograms with metric sub-aggregations on the device (tq_histogram_metrics_batch) against Count, the histogram alone and the
metrics alone, on the same queries: one 512-query batch of a bench workload (phrases left out: they are not on these paths).  The
histogram columns: a nanosecond timestamp rising over seven days in doc order (the dashboard case: `date_histogram` at 1 min and
1 h) and random integers below 10^6 at an interval of 10^4 (100 buckets, every tile straddling).  The metric columns: random
integers below 10^6 (byte counts), a value constant over about ten thousand consecutive docs (one-value tiles) and a count-only
column.  Per configuration, medians over the steps of: host wall time of the call (synchronous), the device ms of its kernels
(CUDA events), and for tq_histogram_metrics_batch the share of tiles in one bucket and the (unit, bucket) flushes from shared
memory versus runs flushed to global memory; with and without a contiguous 10 % filter (TQ_QUERY_FILTER).  Prints the card and its
power limit, read in the same run.  --check: the same configurations at 10M docs (8 segments of 1.25M), every 32nd query's buckets
compared with tests/metrics_model.py (doc counts, count / min / max per bucket, sums the guard accepts bit for bit) on match sets
built from the decoded posting lists.
usage: python profiles/probe_hist_metrics.py [--check] [steps] [workload ...]"""
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
TS, RAND, CLUSTERED, COUNT_ONLY = 1, 2, 3, 4
T0 = 1_700_000_000 * 10**9
WEEK = 7 * 86_400 * 10**9
STATS = [(RAND, T.TQ_FAST_U64, 0)]
THREE = [(RAND, T.TQ_FAST_U64, 0), (CLUSTERED, T.TQ_FAST_U64, 0), (COUNT_ONLY, T.TQ_FAST_U64, T.TQ_METRIC_COUNT_ONLY)]
HIST_1M, HIST_1H = (TS, "date", 60e9, 0.0), (TS, "date", 3600e9, 0.0)
HIST_RAND = (RAND, "u64", 1e4, 0.0)
# (name, histogram spec or None, metric columns or None)
CONFIGS = [("count", None, None), ("histogram_1h", HIST_1H, None), ("metrics_stats", None, STATS),
           ("hm_1m_stats", HIST_1M, STATS), ("hm_1m_three", HIST_1M, THREE), ("hm_1h_stats", HIST_1H, STATS), ("hm_1h_three", HIST_1H, THREE),
           ("hm_rand100_stats", HIST_RAND, STATS)]


def med(xs):
    return round(float(np.median(xs)), 3)


def columns(shard):
    rng = np.random.default_rng(SEED)
    out = {TS: [], RAND: [], CLUSTERED: [], COUNT_ONLY: []}
    total = sum(shard.ix.max_doc)
    first = 0
    for i, g in enumerate(shard.global_ords):
        n = shard.ix.max_doc[i]
        at = first + np.arange(n, dtype=np.int64)
        out[TS].append(T.fast_value_to_u64(T0 + at * (WEEK // total) + rng.integers(0, WEEK // total, size=n), "date"))
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


def check_query(shard, cols, matches, filtered, hspec, spec, row):
    """One query's device buckets against the model: Kahan per (segment, bucket) in doc order, merge_fruits in segment_ord order."""
    col, kind, interval, _ = hspec
    per = {}
    for i, d in sorted(matches, key=lambda x: shard.global_ords[x[0]]):
        n = shard.ix.max_doc[i]
        if filtered:
            d = d[(d >= int(n * 0.45)) & (d < int(n * 0.55))]
        img = cols[col][i][d]
        val = (img ^ np.uint64(1 << 63)).view(np.int64).astype(np.float64) if kind == "date" else img.astype(np.float64)
        pos = np.floor(val / interval).astype(np.int64)
        for p in np.unique(pos):
            sel = d[pos == p]
            seg = []
            for cid, _, flags in spec:
                vals = np.zeros(len(sel)) if flags & T.TQ_METRIC_COUNT_ONLY else cols[cid][i][sel].astype(np.float64)
                seg.append(MM.segment_stats(vals.tolist()))
            if p not in per:
                per[int(p)] = [len(sel), seg]
            else:
                per[int(p)][0] += len(sel)
                for a, b in zip(per[int(p)][1], seg):
                    a.merge_fruits(b)
    got = {int(row[0][j]): (int(row[1][j]), row[2][j]) for j in range(int(row[3]))}
    assert sorted(got) == sorted(per), "bucket rows differ"
    for p, (n, stats) in per.items():
        assert got[p][0] == n, ("doc count", p)
        for j, (cid, ckind, flags) in enumerate(spec):
            count, s, vmin, vmax = Mx.stats_of(got[p][1][j], ckind, flags)
            st = stats[j]
            assert count == st.count and (count == 0 or (vmin, vmax) == (st.min, st.max)), ("count/min/max", p, j)
            if Mx.guard(got[p][1][j]) is None:
                assert s == st.sum, ("sum", p, j, s, st.sum)


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
        for cname, hspec, spec in CONFIGS:
            if hspec is None and spec is None:
                run, ms_key = (lambda: ctx.count_batch(qb)), None
            elif spec is None:
                run, ms_key = (lambda: ctx.histogram_batch(qb, [hspec] * qb.nq)), "hist_ms"
            elif hspec is None:
                run, ms_key = (lambda: ctx.metrics_batch(qb, [spec] * qb.nq)), "metrics_ms"
            else:
                out = ctx.hist_metrics_batch(qb, [hspec] * qb.nq, [spec] * qb.nq, count_hits=True)  # warm-up; hits checked
                assert np.array_equal(out[4], counts), "hits differ from tq_count_batch"
                # (the timed calls take the warm-up's widest row as their stride: every step is one run of the kernels)
                width = max(1, int(out[3].max()))
                run, ms_key = (lambda: ctx.hist_metrics_batch(qb, [hspec] * qb.nq, [spec] * qb.nq, stride=width)), "hist_metrics_ms"
                if CHECK:
                    for qi in range(0, qb.nq, 32):  # (every 32nd query: the Python model is the slow part)
                        if qi not in matches:
                            matches[qi] = match(ctx, shard, qb, qi, postings)
                        check_query(shard, cols, matches[qi], filtered, hspec, spec, [x[qi] for x in out[:4]])
            s0 = ctx.stats()
            run()
            units = ctx.stats()["units_hist_metrics"] - s0["units_hist_metrics"]  # (CTAs of one run)
            wall, dev, seen, one, fs, fg = [], [], [], [], [], []
            for _ in range(steps):
                s0 = ctx.stats()
                t0 = time.perf_counter()
                run()
                wall.append(1e3 * (time.perf_counter() - t0))
                s1 = ctx.stats()
                assert s1["units_hist_metrics"] - s0["units_hist_metrics"] == units, "a timed step ran the kernels more than once"
                if ms_key:
                    dev.append(s1[ms_key] - s0[ms_key])
                seen.append(s1["hist_metrics_tiles_seen"] - s0["hist_metrics_tiles_seen"])
                one.append(s1["hist_metrics_tiles_one_bucket"] - s0["hist_metrics_tiles_one_bucket"])
                fs.append(s1["hist_metrics_flush_shared"] - s0["hist_metrics_flush_shared"])
                fg.append(s1["hist_metrics_flush_global"] - s0["hist_metrics_flush_global"])
            rec = {"workload": name, "docs": sum(shard.ix.max_doc), "queries": qb.nq, "config": cname, "filter_10pct": filtered, "steps": steps,
                   "checked": CHECK, "wall_ms": med(wall), "device_ms": med(dev) if dev else None}
            if ms_key == "hist_metrics_ms":
                rec.update({"tiles_seen": int(med(seen)), "one_bucket_share": round(med(one) / max(med(seen), 1), 3),
                            "flush_shared": int(med(fs)), "flush_global": int(med(fg))})
            print(json.dumps(rec), flush=True)
    ctx.close()
    del shard
