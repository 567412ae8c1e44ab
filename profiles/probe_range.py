"""Range aggregations on the device (tq_range_batch) against Count on the same queries: one 512-query batch of a bench workload
(phrases left out: they are not on these paths).  The range columns: a nanosecond timestamp rising over seven days in doc order
(the dashboard case: "last hour / last day / older", 3 ranges, and 24 ranges of seven hours) and random u64 images (5 ranges, and
127 ranges that extend to 128 buckets: every tile straddles).  Each without metrics and with two metric columns (random integers
below 10^6 and a value constant over about ten thousand consecutive docs).  Per configuration, medians over the steps of: host
wall time of the call (synchronous), range_ms (CUDA events around the kernels), and the share of tiles in one bucket; with and
without a contiguous 10 % filter (TQ_QUERY_FILTER).  Prints the card and its power limit, read in the same run.  --check: the
same configurations at 10M docs (8 segments of 1.25M), every 64th query's rows compared with get_bucket_pos (an upper-bound search over the
starts) and tests/metrics_model.py (doc counts, count / min / max per bucket, sums the guard accepts bit for bit) on match sets built from the
decoded posting lists.
usage: python profiles/probe_range.py [--check] [steps] [workload ...]"""
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
from tantivy_b200 import ranges as R  # noqa: E402
from tests import metrics_model as MM  # noqa: E402

args = [a for a in sys.argv[1:] if a != "--check"]
CHECK = "--check" in sys.argv
steps = int(args[0]) if args else 5
names = args[1:] or ["or5_top100_100M_8seg", "mixed_top10_100M_8seg"]
NQ, SEED, FID = 512, 0x7A6E7469, 1
card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"gpu": card, "check": CHECK}), flush=True)
TS, RAND, INTS, CLUSTERED = 1, 2, 3, 4
T0 = 1_700_000_000 * 10**9
HOUR, DAY, WEEK = 3600 * 10**9, 86_400 * 10**9, 7 * 86_400 * 10**9
END = T0 + WEEK
TWO = [(INTS, T.TQ_FAST_U64, 0), (CLUSTERED, T.TQ_FAST_U64, 0)]


def spec(field, kind, bounds):
    """(column, starts) of contiguous ranges between the bounds (None: open), through tantivy_b200.ranges."""
    ranges = [dict(({"from": a} if a is not None else {}), **({"to": b} if b is not None else {})) for a, b in zip(bounds[:-1], bounds[1:])]
    p = R.plan(R.parse_request({"r": {"range": {"field": field, "ranges": ranges}}}), {field: Mx.MetricField(TS if kind == "date" else RAND, kind)})
    return p.rspec


RANGE_TS3 = spec("ts", "date", [None, float(END - DAY), float(END - HOUR), None])
RANGE_TS24 = spec("ts", "date", [float(T0 + i * 7 * HOUR) for i in range(25)])
RANGE_RAND5 = spec("r", "u64", [None, 2.0**62, 2.0**63, 3 * 2.0**62, 2.0**64 - 2**12, None])
RANGE_RAND128 = spec("r", "u64", [float(i * 2**57) for i in range(1, 128)] + [None])
# (name, range spec or None, metric columns or None)
CONFIGS = [("count", None, None)] + [(f"range_{n}{'_two' if m else ''}", s, m) for n, s in
                                     (("ts3", RANGE_TS3), ("ts24", RANGE_TS24), ("rand5", RANGE_RAND5), ("rand128", RANGE_RAND128)) for m in (None, TWO)]


def med(xs):
    return round(float(np.median(xs)), 3)


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


def columns(shard):
    rng = np.random.default_rng(SEED)
    out = {TS: [], RAND: [], INTS: [], CLUSTERED: []}
    total = sum(shard.ix.max_doc)
    first = 0
    for i, g in enumerate(shard.global_ords):
        n = shard.ix.max_doc[i]
        at = first + np.arange(n, dtype=np.int64)
        out[TS].append(T.fast_value_to_u64(T0 + at * (WEEK // total) + rng.integers(0, WEEK // total, size=n), "date"))
        out[RAND].append(rng.integers(0, 2**64 - 1, size=n, dtype=np.uint64, endpoint=True))
        out[INTS].append(rng.integers(0, 10**6, size=n).astype(np.uint64))
        out[CLUSTERED].append((at * 10_000 // total * 37).astype(np.uint64))
        first += n
    return out


def check_query(shard, cols, matches, filtered, rspec, mcols, counts, parts):
    """One query's device row against the model: get_bucket_pos per doc, Kahan per (segment, bucket) in doc order, merge_fruits in
    segment_ord order."""
    col, starts = rspec
    nb = len(starts)
    want_n = np.zeros(nb, np.int64)
    stats = [[MM.segment_stats([]) for _ in (mcols or [])] for _ in range(nb)]
    for i, d in sorted(matches, key=lambda x: shard.global_ords[x[0]]):
        n = shard.ix.max_doc[i]
        if filtered:
            d = d[(d >= int(n * 0.45)) & (d < int(n * 0.55))]
        b = np.searchsorted(np.array(starts, np.uint64), cols[col][i][d], side="right") - 1  # (get_bucket_pos)
        for j in range(nb):
            sel = d[b == j]
            want_n[j] += len(sel)
            for c, (cid, _, _) in enumerate(mcols or []):
                stats[j][c].merge_fruits(MM.segment_stats(cols[cid][i][sel].astype(np.float64).tolist()))
    assert np.array_equal(counts[:nb].astype(np.int64), want_n), "doc counts differ"
    for j in range(nb):
        for c, (cid, ckind, flags) in enumerate(mcols or []):
            count, s, vmin, vmax = Mx.stats_of(parts[j][c], ckind, flags)
            st = stats[j][c]
            assert count == st.count and (count == 0 or (vmin, vmax) == (st.min, st.max)), ("count/min/max", j, c)
            if Mx.guard(parts[j][c]) is None:
                assert s == st.sum, ("sum", j, c, s, st.sum)


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
        for cname, rspec, mcols in CONFIGS:
            if rspec is None:
                run, ms_key = (lambda: ctx.count_batch(qb)), None
            else:
                out = ctx.range_batch(qb, [rspec] * qb.nq, None if mcols is None else [mcols] * qb.nq, count_hits=True)
                assert np.array_equal(out[2], counts), "hits differ from tq_count_batch"
                run, ms_key = (lambda: ctx.range_batch(qb, [rspec] * qb.nq, None if mcols is None else [mcols] * qb.nq)), "range_ms"
                if CHECK:
                    for qi in range(0, qb.nq, 64):  # (every 64th query: the Python model is the slow part)
                        if qi not in matches:
                            matches[qi] = match(ctx, shard, qb, qi, postings)
                        check_query(shard, cols, matches[qi], filtered, rspec, mcols, out[0][qi], None if out[1] is None else out[1][qi])
            run()
            wall, dev, seen, one = [], [], [], []
            for _ in range(steps):
                s0 = ctx.stats()
                t0 = time.perf_counter()
                run()
                wall.append(1e3 * (time.perf_counter() - t0))
                s1 = ctx.stats()
                if ms_key:
                    dev.append(s1[ms_key] - s0[ms_key])
                seen.append(s1["range_tiles_seen"] - s0["range_tiles_seen"])
                one.append(s1["range_tiles_one_bucket"] - s0["range_tiles_one_bucket"])
            rec = {"workload": name, "docs": sum(shard.ix.max_doc), "queries": qb.nq, "config": cname, "filter_10pct": filtered, "steps": steps,
                   "checked": CHECK, "wall_ms": med(wall), "device_ms": med(dev) if dev else None}
            if ms_key:
                rec.update({"buckets": len(rspec[1]), "tiles_seen": int(med(seen)), "one_bucket_share": round(med(one) / max(med(seen), 1), 3)})
            print(json.dumps(rec), flush=True)
    ctx.close()
    del shard
