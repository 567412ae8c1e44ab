"""Filtered search (TQ_QUERY_FILTER): what a per-query doc filter costs and saves on 512-query batches of a bench workload.
Cases: no filter; one contiguous filter over 1 % / 10 % / 50 % of each segment; one Bernoulli filter of 1 % / 10 % / 50 %; and 1, 8
and 64 distinct filters per batch (contiguous 10 % runs at different offsets, query i takes filter i mod n).  Per case: q/s (host
clock around prepare + run + fetch of a synchronised batch, median of the steps), tile_ms, score_ms, units_tile, and the (query,
tile) pairs k_tile saw (tile_counters[0], one run on a second context with TQ_TILE_COUNTERS=1).  Prints the card and power limit.
--check: 10M docs; every case's rows against a second context whose segments carry alive := filter (the synthetic index has no
deletes), bit for bit.
usage: python profiles/probe_filter.py [--check] [--steps N] [workload ...]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import tantivy_b200 as T  # noqa: E402
from tantivy_b200._abi import TQ_QUERY_FILTER  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--check", action="store_true")
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("workloads", nargs="*", default=["or5_top100_100M_8seg", "mixed_top10_100M_8seg"])
args = ap.parse_args()
NQ = 512
SEED = 0x7A6E7469
card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"gpu": card}), flush=True)


def contiguous(max_doc, frac, offset=0.25):
    m = np.zeros(max_doc, bool)
    lo = int(max_doc * offset) % max_doc
    n = max(1, int(max_doc * frac))
    m[lo:lo + n] = True
    if lo + n > max_doc:
        m[:lo + n - max_doc] = True
    return m


def cases():
    yield "none", None
    for f in (0.01, 0.1, 0.5):
        yield f"contiguous_{f:g}", [lambda md, rng, f=f: contiguous(md, f)]
    for f in (0.01, 0.1, 0.5):
        yield f"bernoulli_{f:g}", [lambda md, rng, f=f: rng.random(md) < f]
    for n in (1, 8, 64):
        yield f"distinct_{n}", [lambda md, rng, i=i, n=n: contiguous(md, 0.1, offset=i / n) for i in range(n)]


def run(ctx, qb):
    t0 = time.perf_counter()
    b = ctx.prepare(qb)
    b.run()
    rows = b.fetch()
    dt = time.perf_counter() - t0
    st = ctx.stats()
    b.close()
    return rows, dt, st


for name in args.workloads:
    wl = dict(bench.WORKLOADS[name])
    if args.check:
        wl["docs_per_segment"] = 10_000_000 // wl["n_segments"]
    dens, batches = bench.build_query_plan(wl, NQ, 1, SEED)
    shard = bench.make_shard(wl, dens, 0, 1, SEED)
    ix = shard.ix
    ctx = T.Context(0)
    shard.register(ctx)
    os.environ["TQ_TILE_COUNTERS"] = "1"
    cctx = T.Context(0)
    os.environ.pop("TQ_TILE_COUNTERS")
    shard.register(cctx)
    for case, makers in cases():
        rng = np.random.default_rng(1)
        qb = bench.marshal(shard, batches[0])
        masks = []
        if makers:
            for fid, mk in enumerate(makers):
                masks.append([mk(ix.max_doc[i], rng) for i in range(ix.n_segments)])
                bits = [np.packbits(m, bitorder="little") for m in masks[-1]]
                for c in (ctx, cctx):
                    shard.register_filter(c, fid, bits)
            q = qb.q[:qb.nq]
            q["flags"] |= TQ_QUERY_FILTER
            q["filter_id"] = np.arange(qb.nq) % len(makers)
        rows, _, _ = run(ctx, qb)  # warm-up: block tables and filter views are built here
        times, tile_ms, score_ms = [], [], []
        for _ in range(args.steps):
            _, dt, st = run(ctx, qb)
            times.append(dt)
            tile_ms.append(st["tile_ms"])
            score_ms.append(st["score_ms"])
        seen0 = cctx.stats()["tile_counters"][0]
        _, _, cst = run(cctx, qb)
        out = {"workload": name, "case": case, "docs": int(sum(ix.max_doc)), "qps": round(qb.nq / float(np.median(times)), 1),
               "tile_ms": round(float(np.median(tile_ms)), 3), "score_ms": round(float(np.median(score_ms)), 3),
               "units_tile": st["units_tile"], "tile_groups": st["tile_groups"], "tile_pairs_seen": cst["tile_counters"][0] - seen0}
        if args.check and makers:
            ok = True
            for fid in range(len(makers)):
                ref = T.Context(0)
                for i, g in enumerate(shard.global_ords):
                    ref.segment_register(g, 0, ix.max_doc[i], ix.record_option, ix.body(i), ix.fieldnorm(i), np.packbits(masks[fid][i], bitorder="little"))
                    if ix.record_option == 2:
                        ref.register_positions(g, 0, ix.positions(i))
                mine = np.nonzero(np.arange(qb.nq) % len(makers) == fid)[0]
                want = ref.search_batch(bench.marshal(shard, [batches[0][j] for j in mine]))
                for a, b in zip(rows, want):
                    ok = ok and np.array_equal(a[mine].view(np.uint32), b.view(np.uint32))
                ref.close()
            out["rows_equal_alive_and_filter"] = ok
            assert ok, case
        if makers:
            for c in (ctx, cctx):
                for fid in range(len(makers)):
                    c.filter_unregister(fid)
        print(json.dumps(out), flush=True)
    ctx.close()
    cctx.close()
    del shard
