"""(Count, TopDocs) in one batch against two batches: one 512-query batch of a bench workload, timed three ways --
  (a) the batch as bench.py runs it (no query flagged);
  (b) (a) followed by tq_count_batch on the same queries (the two-batch way to get both);
  (c) the batch with TQ_QUERY_COUNT_HITS on every query but the phrases (Count of a phrase is not on the device path).
For each: total_ms (CUDA events from prepare's upload to the fetch), tile_ms and count_hits_ms (CUDA events around the launches).
tq_count_batch synchronises inside and publishes no stats: its time in (b) is host wall time around the call, an upper bound of
its device time.  Checks that (c)'s rows are bit-equal to (a)'s and its hits equal (b)'s counts; prints the card and power limit.
usage: python profiles/probe_count_hits.py [steps] [workload ...]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import tantivy_b200 as T  # noqa: E402
from tantivy_b200._abi import TQ_OP_PHRASE, TQ_QUERY_COUNT_HITS  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
names = sys.argv[2:] or ["or5_top100_100M_8seg", "and2_top10_10M_1seg", "mixed_top10_100M_8seg"]
NQ = 512
card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"gpu": card}), flush=True)


def run(ctx, qb, hits=False):
    b = ctx.prepare(qb)
    b.run()
    rows = b.fetch()
    h = b.fetch_hits() if hits else None
    st = ctx.stats()
    b.close()
    return rows, h, st


def summary(xs):
    return round(float(np.median(xs)), 3)


for name in names:
    wl = dict(bench.WORKLOADS[name])
    dens, batches = bench.build_query_plan(wl, NQ, 1, 0x7A6E7469)
    shard = bench.make_shard(wl, dens, 0, 1, 0x7A6E7469)
    ctx = T.Context(0)
    shard.register(ctx)
    qa = bench.marshal(shard, batches[0])
    qc = bench.marshal(shard, batches[0])
    not_phrase = qc.q["op"][:qc.nq] != TQ_OP_PHRASE
    qc.q["flags"][:qc.nq][not_phrase] |= TQ_QUERY_COUNT_HITS
    qn = bench.marshal(shard, [q for q in batches[0] if bench.OPS[q[0]] != TQ_OP_PHRASE])  # (b)'s Count batch: phrases refused there
    a, b_, c = {"total_ms": [], "tile_ms": [], "count_hits_ms": []}, {"total_ms": [], "count_batch_ms": []}, \
        {"total_ms": [], "tile_ms": [], "count_hits_ms": []}
    for i in range(steps + 1):
        ra, _, sa = run(ctx, qa)
        t0 = time.perf_counter()
        counts = np.zeros(qa.nq, np.uint64)
        counts[not_phrase] = ctx.count_batch(qn)
        tc = 1e3 * (time.perf_counter() - t0)
        rc, hc, sc = run(ctx, qc, hits=True)
        if i == 0:  # warm-up: the block tables are built here; check once
            same_rows = all(np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x, y.view(np.uint32) if y.dtype == np.float32 else y)
                            for x, y in zip(ra, rc))
            same_hits = bool((hc == counts).all())
            print(json.dumps({"workload": name, "rows_bit_equal": same_rows, "hits_equal_count_batch": same_hits,
                              "flagged": int(not_phrase.sum()), "tile_groups": sc["tile_groups"], "units_count_hits": sc["units_count_hits"],
                              "launches_a": sa["kernel_launches"], "launches_c": sc["kernel_launches"]}), flush=True)
            assert same_rows and same_hits
            continue
        for k in a:
            a[k].append(sa[k])
            c[k].append(sc[k])
        b_["total_ms"].append(sa["total_ms"] + tc)
        b_["count_batch_ms"].append(tc)
    print(json.dumps({"workload": name, "steps": steps, "a_unflagged": {k: summary(v) for k, v in a.items()},
                      "b_plus_count_batch": {k: summary(v) for k, v in b_.items()},
                      "c_flagged": {k: summary(v) for k, v in c.items()}}), flush=True)
    ctx.close()
    del shard
