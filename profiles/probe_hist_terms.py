"""Histograms with a terms sub-aggregation on the device (tq_histogram_terms_batch) against Count, the histogram alone
(tq_histogram_batch) and terms alone (tq_terms_batch) on the same queries: one 512-query batch of a bench workload (phrases left out:
they are not on these paths).  A date_histogram at 1 h and at 1 min of a nanosecond timestamp rising over seven days in doc order, with
a terms on about 20 random values and on 10 K random values (size 10, segment_size 100) under it.  Per configuration, medians over the
steps of: host wall time of the call (synchronous), the call's device ms (CUDA events around its kernels), the shares of tiles with
one key, in one bucket and both, the k_hist_terms units counted in shared memory and in the grid, the rows cut on the device and the
waves; with and without a contiguous 10 % filter (TQ_QUERY_FILTER).  Prints the card and its power limit, read in the same run.
--check: the same configurations at 10M docs (8 segments of 1.25M), every 64th query's buckets, scalars and entries compared with
tests/hist_terms_model.py (its per-bucket cut; its per-doc walk vectorised) on match sets built from the decoded posting lists.
usage: python profiles/probe_hist_terms.py [--check] [steps] [workload ...]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import tantivy_b200 as T  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_PHRASE, TQ_QUERY_FILTER, TQ_TERMS_BY_COUNT, TQ_ORDER_DESC  # noqa: E402
from tests import histogram_model as HM  # noqa: E402
from tests import hist_terms_model as HTM  # noqa: E402
from tests.test_gpu_hist_terms import dev_rows  # noqa: E402

args = [a for a in sys.argv[1:] if a != "--check"]
CHECK = "--check" in sys.argv
steps = int(args[0]) if args else 5
names = args[1:] or ["or5_top100_100M_8seg", "mixed_top10_100M_8seg"]
NQ, SEED, FID = 512, 0x7A6E7469, 1
card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"gpu": card, "check": CHECK}), flush=True)
TS, K20, K10K = 1, 2, 3
T0 = 1_700_000_000 * 10**9
WEEK = 7 * 86_400 * 10**9
HOUR, MINUTE = 3600 * 10**9, 60 * 10**9
F64_MAX = float(np.finfo(np.float64).max)


def tspec(col):
    return (col, TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 100)


def hspec(interval):
    return (TS, "date", float(interval), 0.0, -F64_MAX, F64_MAX)


# (name, terms spec or None, histogram spec or None)
CONFIGS = [("count", None, None), ("terms_k20", tspec(K20), None), ("terms_k10k", tspec(K10K), None), ("hist_1h", None, hspec(HOUR)),
           ("hist_1m", None, hspec(MINUTE))]
CONFIGS += [(f"hist_terms_{h}_{k}", tspec(c), hspec(iv)) for h, iv in (("1h", HOUR), ("1m", MINUTE)) for k, c in (("k20", K20), ("k10k", K10K))]


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
    out = {TS: [], K20: [], K10K: []}
    total = sum(shard.ix.max_doc)
    first = 0
    for i, g in enumerate(shard.global_ords):
        n = shard.ix.max_doc[i]
        at = first + np.arange(n, dtype=np.int64)
        out[TS].append(T.fast_value_to_u64(T0 + at * (WEEK // total) + rng.integers(0, WEEK // total, size=n), "date"))
        out[K20].append(rng.integers(0, 20, size=n).astype(np.uint64))
        out[K10K].append(rng.integers(0, 10_000, size=n).astype(np.uint64))
        first += n
    return out


def segment_buckets(keys, values, docs, interval):
    """tests/hist_terms_model.segment over full columns without bounds, vectorised: {pos: (doc_count, {image: doc_count})}."""
    k = keys[docs].astype(np.uint64)
    pos = HM.as_i64(np.floor((HM.image_to_f64(values[docs], "date") - 0.0) / np.float64(interval)))
    out = {int(p): (int(c), {}) for p, c in zip(*np.unique(pos, return_counts=True))}
    pairs = np.stack([pos, k.view(np.int64)], axis=1) if len(k) else np.zeros((0, 2), np.int64)
    uniq, cnt = np.unique(pairs, axis=0, return_counts=True)
    for (p, a), c in zip(uniq.tolist(), cnt.tolist()):
        out[int(p)][1][int(np.int64(a).view(np.uint64))] = int(c)
    return out


def check_query(shard, cols, matches, filtered, ts, hs, rows):
    """One query's device rows against the model's per-bucket cut (tests/hist_terms_model.cut), summed over the segments."""
    want = {}
    for i, d in sorted(matches, key=lambda x: shard.global_ords[x[0]]):
        n = shard.ix.max_doc[i]
        if filtered:
            d = d[(d >= int(n * 0.45)) & (d < int(n * 0.55))]
        for pos, (c, kept, e, o) in HTM.cut(segment_buckets(cols[ts[0]][i], cols[TS][i], d, hs[2]), ts[3]).items():
            d0, o0, e0, ents = want.get(pos, (0, 0, 0, []))
            want[pos] = (d0 + c, o0 + o, e0 + e, ents + [(shard.global_ords[i], k, m) for k, m in kept])
    assert rows == want, "rows differ from the model"


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
        for cname, ts, hs in CONFIGS:
            stat = None
            if ts is None and hs is None:
                run = lambda: ctx.count_batch(qb)  # noqa: E731
            elif hs is None:
                run, ms_key = (lambda: ctx.terms_batch(qb, [ts] * qb.nq)), "terms_ms"
            elif ts is None:
                run, ms_key = (lambda: ctx.histogram_batch(qb, [hs] * qb.nq)), "hist_ms"
            else:
                try:
                    out = ctx.hist_terms_batch(qb, [hs] * qb.nq, [ts] * qb.nq, count_hits=True)
                except T.TqError as e:  # (a (query, segment) grid over TQ_HIST_TERMS_BUDGET: the batch takes the CPU path)
                    print(json.dumps({"workload": name, "config": cname, "filter_10pct": filtered, "refused": str(e)}), flush=True)
                    continue
                assert np.array_equal(out[11], counts), "hits differ from tq_count_batch"
                ref = ctx.histogram_batch(qb, [hs] * qb.nq)
                assert np.array_equal(out[6], ref[2]) and all(np.array_equal(out[0][q, :n], ref[0][q, :n]) and np.array_equal(out[1][q, :n], ref[1][q, :n])
                                                              for q, n in enumerate(ref[2].tolist())), "buckets differ from the histogram"
                run, ms_key, stat = (lambda: ctx.hist_terms_batch(qb, [hs] * qb.nq, [ts] * qb.nq)), "hist_terms_ms", "hist_terms"
                if CHECK:
                    for qi in range(0, qb.nq, 64):  # (every 64th query: the Python model is the slow part)
                        if qi not in matches:
                            matches[qi] = match(ctx, shard, qb, qi, postings)
                        check_query(shard, cols, matches[qi], filtered, ts, hs, dev_rows(out, qi))
            run()
            wall, dev, tiles, extra = [], [], [], []
            for _ in range(steps):
                s0 = ctx.stats()
                t0 = time.perf_counter()
                run()
                wall.append(1e3 * (time.perf_counter() - t0))
                s1 = ctx.stats()
                if ts is not None or hs is not None:
                    dev.append(s1[ms_key] - s0[ms_key])
                if stat:
                    tiles.append([s1[f"{stat}_tiles_{k}"] - s0[f"{stat}_tiles_{k}"] for k in ("seen", "one_key", "one_bucket", "both")])
                    extra.append([s1[f"{stat}_{k}"] - s0[f"{stat}_{k}"] for k in ("units_shared", "units_global", "rows_cut", "waves")])
            rec = {"workload": name, "docs": sum(shard.ix.max_doc), "queries": qb.nq, "config": cname, "filter_10pct": filtered, "steps": steps,
                   "checked": CHECK, "wall_ms": med(wall), "device_ms": med(dev) if dev else None}
            if tiles:
                t = np.median(np.array(tiles, np.float64), axis=0)
                rec.update({"tiles_seen": int(t[0]), "one_key_share": round(t[1] / max(t[0], 1), 3), "one_bucket_share": round(t[2] / max(t[0], 1), 3),
                            "both_share": round(t[3] / max(t[0], 1), 3)})
                x = np.median(np.array(extra, np.float64), axis=0)
                rec.update({"units_shared": int(x[0]), "units_global": int(x[1]), "rows_cut": int(x[2]), "waves": int(x[3])})
            print(json.dumps(rec), flush=True)
    ctx.close()
    del shard
