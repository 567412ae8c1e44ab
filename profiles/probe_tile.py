"""Probe of the tile engine on a bench workload: per-kind kernel times, tile counters, how B2's union postings ended, k_tile's cycles
by stage, parity of a query sample.
usage: python profiles/probe_tile.py [workload] [nq] [steps] [check]   (env knobs: TQ_TILE*, see tq_ctx_create)"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("TQ_TILE_COUNTERS", "1")
import bench  # noqa: E402
import tantivy_b200 as T  # noqa: E402

wl_name = sys.argv[1] if len(sys.argv) > 1 else "or5_top100_100M_8seg"
nq = int(sys.argv[2]) if len(sys.argv) > 2 else 512
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 5
check = int(sys.argv[4]) if len(sys.argv) > 4 else 16
wl = dict(bench.WORKLOADS[wl_name])
if os.environ.get("PROBE_DOCS"):
    wl["docs_per_segment"] = int(os.environ["PROBE_DOCS"])
dens, batches = bench.build_query_plan(wl, nq, 2, 0x7A6E7469)
t0 = time.time()
shard = bench.make_shard(wl, dens, 0, 1, 0x7A6E7469)
print("index", round(time.time() - t0, 2), "s", shard.index_bytes, "bytes", len(dens), "terms", flush=True)
ctx = T.Context(0)
shard.register(ctx)
qbs = [bench.marshal(shard, b) for b in batches]
keys = keys_ms = ("kernel_ms", "score_ms", "tile_ms", "theta_ms", "final_ms", "or_ms", "and_ms", "term_ms")
STAGES = ("prologue", "A", "B1", "B2", "B3", "barrier")


def stage_shares(cyc):
    """k_tile's warp cycles by stage (tq_stats.tile_cycles, TQ_TILE_COUNTERS=1) as shares of their sum."""
    tot = int(cyc[:len(STAGES)].sum())
    return {s: round(int(c) / tot, 4) for s, c in zip(STAGES, cyc)} if tot else {}


c0 = np.array(ctx.stats()["tile_counters"], dtype=np.int64)
y0 = np.array(ctx.stats()["tile_cycles"], dtype=np.int64)
x0 = np.array(ctx.stats()["tile_b2_exits"], dtype=np.int64)
y_first = None
for i in range(steps + 2):
    t0 = time.perf_counter()
    bt = ctx.prepare(qbs[i % 2])
    t1 = time.perf_counter()
    bt.run()
    bt.results_dev()
    t2 = time.perf_counter()
    st = ctx.stats()
    c1 = np.array(st["tile_counters"], dtype=np.int64)
    y1 = np.array(st["tile_cycles"], dtype=np.int64)
    x1 = np.array(st["tile_b2_exits"], dtype=np.int64)
    if i == 2:
        y_first = y0  # (the first two steps warm up: the summary below covers the rest)
    print(json.dumps({"step": i, "prepare_ms": round(1e3 * (t1 - t0), 2), "run_ms": round(1e3 * (t2 - t1), 2),
                      **{k: round(st[k], 3) for k in keys}, "launches": st["kernel_launches"], "units_tile": st["units_tile"],
                      "tile_postings": st["tile_postings"], "scratch_MB": st["tile_scratch_bytes"] >> 20, "fallback": st["tile_fallbacks"],
                      "groups": st["tile_groups"], "smem": int(c1[7]), "tile_ctas_per_sm": st["tile_ctas_per_sm"],
                      "counters(pairs,skip,light,heavy,ess,compl,pass)": (c1 - c0)[:7].tolist(),
                      "b2_union_exits(bound,not_owner,walk,completed)": (x1 - x0).tolist(),
                      "theta_refresh(refreshes,raises)": (y1 - y0)[6:8].tolist(),
                      "stage_shares": stage_shares(y1 - y0)}), flush=True)
    c0, y0, x0 = c1, y1, x1
    bt.close()
if y_first is not None and (y0 - y_first).any():
    d = y0 - y_first
    print(json.dumps({"k_tile_stage_cycles(steps 2..)": dict(zip(STAGES, d[:len(STAGES)].tolist())), "stage_shares": stage_shares(d),
                      "B1+B2": round(float(d[2] + d[3]) / float(d[:len(STAGES)].sum()), 4)}), flush=True)
if os.environ.get("PROBE_THETA"):
    # how much better would the step be with (nearly) final thresholds from the start?  Run a batch up to its last phase, keep
    # its thresholds, then run the same batch again with those thresholds imported after the sample phase.
    import torch
    keys = torch.zeros(nq, dtype=torch.int64, device="cuda:0")
    bt = ctx.prepare(qbs[0])
    n_ph = bt.phases()
    for ph in range(n_ph - 1):
        bt.run_phase(ph)
    bt.thresholds_export_dev(keys.data_ptr())
    bt.run_phase(n_ph - 1)
    bt.results_dev()
    bt.close()
    c0 = np.array(ctx.stats()["tile_counters"], dtype=np.int64)
    bt = ctx.prepare(qbs[0])
    t1 = time.perf_counter()
    bt.run_phase(0)
    bt.thresholds_import_dev(keys.data_ptr())
    for ph in range(1, n_ph):
        bt.run_phase(ph)
    bt.results_dev()
    t2 = time.perf_counter()
    st = ctx.stats()
    c1 = np.array(st["tile_counters"], dtype=np.int64)
    print(json.dumps({"theta_import": True, "run_ms": round(1e3 * (t2 - t1), 2), **{k: round(st[k], 3) for k in keys_ms},
                      "counters(pairs,skip,light,heavy,ess,compl,pass)": (c1 - c0)[:7].tolist()}), flush=True)
    bt.close()
t0 = time.perf_counter()
out = ctx.search_batch(qbs[0])
print("e2e search_batch ms", round(1e3 * (time.perf_counter() - t0), 2))
if check:
    from oracle import tq_oracle as O
    oi = O.OracleIndex()
    shard.register(oi)
    sub = bench.marshal(shard, batches[0][:check])
    t0 = time.time()
    ref = oi.search_batch(sub, mode=0, n_threads=os.cpu_count())
    bad = 0
    for q in range(check):
        n = int(ref[3][q])
        ok = int(out[3][q]) == n and (out[1][q, :n] == ref[1][q, :n]).all() and (out[2][q, :n] == ref[2][q, :n]).all() and \
            (out[0][q, :n].view(np.uint32) == ref[0][q, :n].view(np.uint32)).all()
        bad += 0 if ok else 1
    print("parity: checked", check, "mismatches", bad, "oracle_s", round(time.time() - t0, 1))
ctx.close()
