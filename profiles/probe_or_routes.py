"""Times the two per-query union kernels (TQ_TILE=0) on the or5 workload's index, three query shapes:
5-term unions at k = 100 take k_or_strip; 5-term unions at k = 256 (past the strip kernel's k) and 12-term unions at
k = 10 (past its clause count) take k_or.
Prints or_ms, units_or and units_or_strip per route and run; TANTIVY_B200_LIB selects the build to time."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["TQ_TILE"] = "0"
import bench as B
import tantivy_b200 as T
wl = dict(B.WORKLOADS["or5_top100_100M_8seg"], n_terms=12)
dens, batches = B.build_query_plan(wl, 256, 2, 0x7A6E7469)  # the 5-term shapes take the first 5 terms of each query
shard = B.make_shard(wl, dens, 0, 1, 0x7A6E7469)
ctx = T.Context(0); shard.register(ctx)
for route, n_terms, k in (("strip", 5, 100), ("k_or_k256", 5, 256), ("k_or", 12, 10)):
    qbs = [B.marshal(shard, [(op, terms[:n_terms], k) for op, terms, _ in b]) for b in batches]
    for it in range(4):
        t0 = time.time(); ctx.search_batch(qbs[it % 2]); dt = time.time() - t0
        st = ctx.stats()
        print(route, "iter", it, "ms", round(dt * 1e3, 1), "or_ms", round(st["or_ms"], 2), "units_or", st["units_or"], "units_or_strip", st["units_or_strip"], flush=True)
