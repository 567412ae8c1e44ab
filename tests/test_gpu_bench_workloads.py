"""bench.py's workloads at the shapes it measures, on the paths it times, against the exhaustive oracle.

The query stream is bench.py's own: WORKLOADS, build_query_plan, make_shard and marshal are imported from it, with its default
seed, queries per step and number of distinct batches (read from its argument parser), so these tests follow the measured stream
if it ever changes.  The truth is oracle/ mode 0 (exhaustive, canonical order) over the whole index, as in bench.py's
parity_check; rows are compared count for count, segment for segment, doc for doc and bit for bit on f32 scores, zeros by value
(helpers.hits).  Every row a step returns is also compared bit for bit with the first rows that batch returned: a prepared batch
that drifts on its second or third run fails even if its first run was right.

  * value leg, one rank: bench.py's pipelined_steps -- the four prepared batches cycled with two in flight, the next batch's run()
    queued before the host waits for the previous one -- for three rounds of the four batches, the rows read after every step;
  * e2e leg, one rank: search_batch alternating between two host output buffers, then e2e_pipelined (prepare step i + 1 while
    step i runs, fetch into host buffers, close);
  * several ranks as threads on one GPU, each with a Context of its own, an in-process process group between them
    (tests/test_gpu_shard_exchange.py) and one CrossGpuMerger at depth 1, with bench.py's make_shard: or5 and mixed at 2 and 8
    ranks and or20 at 8 (whole segments), and2 and term at 2 (doc-range halves of their one segment); rank 0's merged rows
    against the whole index;
  * bench.py itself as a subprocess with --parity-queries 512 and --dump-outputs: its parity block and the dumped rows;
  * the tile engine's counters per step: every batch but term's runs on the tile engine, and no step of or5, or20, and2 or term
    falls back to the per-query kernels.  A group holds up to 1024 queries of each of its segments, so at the defaults only
    or20's twenty-term unions (256 of a segment per group) split a 512-query batch; the value leg runs once more with at most
    128 queries of a segment per group (TQ_TILE_MAX_QUERIES), where every batch of the tile engine takes four groups.

or20_top10_500M_64seg runs 8 of its 64 segments (ordinals 0-7, 62.5M docs at their real size of 7 812 500 docs each) with
bench.py's real query stream; statistics (doc counts, doc frequencies, average fieldnorm) come from those 8 segments.  The full
500M-doc index fits in host memory, but the oracle needs about 1000 s for one batch of it (ORACLE_S), more than this module's
whole budget of about 20 minutes.  bench.py end to end runs the other four workloads.

Sample sizes follow the oracle's cost: ORACLE_S is the measured time of one 512-query batch on the oracle per workload.  The
module took 474 s and 418 s in two runs on an H100 80GB HBM3 (700 W power limit) with 8 host threads, about 300 s of it
building indexes and oracle rows."""
import ast
import os
import subprocess
import sys
import time

import numpy as np
import pytest

from tantivy_b200.sharding import assign_parts, doc_range
from tests.helpers import hits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402  (read only: the measured stream)


def _bench_default(flag):
    """The default of one of bench.py's command-line flags, read from its argument parser's source."""
    tree = ast.parse(open(os.path.join(ROOT, "bench.py")).read())
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and getattr(node.func, "attr", None) == "add_argument" and node.args and \
                isinstance(node.args[0], ast.Constant) and node.args[0].value == flag:
            return next(ast.literal_eval(kw.value) for kw in node.keywords if kw.arg == "default")
    raise KeyError(flag)


SEED = _bench_default("--seed")
NQ = _bench_default("--nq")
N_BATCHES = _bench_default("--batches")
DEPTH = 2             # bench.py's batches in flight on one GPU
CYCLES = 3            # rounds of the N_BATCHES prepared batches in the value leg
TILE_MAX_QUERIES = 1024  # queries of one segment in one tile group (kTileMaxQueries)

TERM, AND2, OR5, OR20, MIXED = ("term_top10_1M_1seg", "and2_top10_10M_1seg", "or5_top100_100M_8seg", "or20_top10_500M_64seg",
                                "mixed_top10_100M_8seg")
OR20_SEGMENTS = 8     # of 64 (module docstring)

# Seconds the oracle (mode 0, 8 host threads of an x86 host) took for batch 0 of each workload, all 512 queries, over the index
# this module builds.  The whole 500M-doc or20 index took 62.7 s for 32 queries (about 1000 s per batch; 25 s to generate, 7 GB of
# host memory): its minimum coverage, 512 + 3 x 64 queries, would cost about 23 minutes of oracle time alone.
ORACLE_S = {TERM: 0.06, AND2: 0.81, OR5: 37.6, MIXED: 7.8, OR20: 114.5}
# Queries of each of batches 1..3 checked against the oracle (batch 0: all of them), from ORACLE_S: all 512 of term and and2
# (3 x 0.8 s); 128 of or5 (3 x 9.4 s); 256 of mixed (3 x 3.9 s); 64 of or20 (3 x 14.3 s).  With batch 0 that is about 5 minutes of
# oracle time for the module, bench.py's own parity checks included.
SAMPLE = {TERM: NQ, AND2: NQ, OR5: 128, MIXED: 256, OR20: 64}
# Ranks of the multi-rank runs: whole segments round-robin where there are at least as many segments, else doc-range parts.
WORLDS = {TERM: (2,), AND2: (2,), OR5: (2, 8), MIXED: (2, 8), OR20: (8,)}
MULTI_RANK = [(name, world) for name, worlds in WORLDS.items() for world in worlds]
# The workloads of the GPU tests, in order.  (pytest groups a module-scoped fixture's parameters by their index: every
# parametrization of `wlx` takes this list or a prefix of it, so each index is one index build.)
ALL = [TERM, AND2, OR5, MIXED, OR20]
# bench.py end to end: its parity check re-runs the oracle over all of batch 0 (ORACLE_S once more).  Not or20: bench.py builds
# the whole 500M-doc index, about 1000 s of oracle time.
BENCH_RUNS = ALL[:4]


def workload(name):
    wl = dict(bench.WORKLOADS[name])
    if name == OR20:
        wl["n_segments"] = OR20_SEGMENTS
    return wl


def plan(name):
    return bench.build_query_plan(bench.WORKLOADS[name], NQ, N_BATCHES, SEED)


def checked_queries(name, batch):
    """The queries of `batch` compared with the oracle: all of batch 0, a seeded sample of the others."""
    if batch == 0 or SAMPLE[name] >= NQ:
        return np.arange(NQ)
    return np.sort(np.random.default_rng([SEED, batch]).choice(NQ, size=SAMPLE[name], replace=False))


# ---- the stream and the splits (no GPU) -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(bench.WORKLOADS))
def test_the_query_stream_is_deterministic(name):
    dens, batches = plan(name)
    dens2, batches2 = plan(name)
    assert dens == dens2 and batches == batches2
    assert len(batches) == N_BATCHES and all(len(b) == NQ for b in batches)
    assert all(k == bench.WORKLOADS[name]["k"] for b in batches for _, _, k in b)


@pytest.mark.parametrize("name", [OR5, MIXED, OR20])
def test_eight_segment_batches_hold_thousands_of_pairs(name):
    """Every term of the stream has hundreds of expected postings in every segment, so each query is a (query, segment) pair of
    every segment: 512 x 8 pairs per batch, more than the 1024 queries of a segment one tile group takes, and at SPLIT_QUERIES
    queries of a segment per group at least four groups."""
    wl = workload(name)
    dens, batches = plan(name)
    assert wl["n_segments"] == 8
    assert min(dens) * wl["docs_per_segment"] > 200
    for b in batches:
        assert len(b) * wl["n_segments"] > TILE_MAX_QUERIES
        assert -(-len(b) // SPLIT_QUERIES) >= 4


def test_mixed_batch0_holds_every_op():
    _, batches = plan(MIXED)
    ops = {op for op, _, _ in batches[0]}
    assert ops == {"term", "and", "or", "phrase"}
    assert {len(t) for op, t, _ in batches[0] if op == "phrase"} == {2, 3}
    assert {len(t) for op, t, _ in batches[0] if op == "or"} == {2, 3, 4}


def test_or20_queries_hold_twenty_distinct_deep_terms():
    dens, batches = plan(OR20)
    rank = {t: round(bench.ZIPF_C / p) for t, p in enumerate(dens)}
    deep = 0
    for b in batches:
        for op, terms, k in b:
            assert op == "or" and len(terms) == 20 and len(set(terms)) == 20 and k == 10
            deep += any(rank[t] > 1000 for t in terms)
    assert deep > NQ  # most queries reach past rank 1000 (ranks go up to 10 000)
    assert max(rank.values()) > 5000


@pytest.mark.parametrize("name,world", MULTI_RANK)
def test_multi_rank_splits_cover_every_doc_once(name, world):
    wl = workload(name)
    n, max_doc = wl["n_segments"], wl["docs_per_segment"]
    held = {s: np.zeros(max_doc, np.int32) for s in range(n)}
    for r in range(world):
        units = assign_parts(n, world, r)
        assert units, (name, world, r)  # no idle rank at these shapes
        for s, part, parts in units:
            lo, hi = doc_range(max_doc, part, parts)
            held[s][lo:hi] += 1
    for s in range(n):
        assert (held[s] == 1).all(), (name, world, s)
    if n < world:
        assert all(len(assign_parts(n, world, r)) == 1 and assign_parts(n, world, r)[0][2] == world // n for r in range(world))


# ---- the GPU legs ---------------------------------------------------------------------------------------------------------------
def _rows(res, q):
    return hits(res, q)


def _bits(res, q):
    """One query's rows as they came, scores by bit pattern."""
    sc, sg, dc, ct = res
    n = int(ct[q])
    return (n, np.asarray(sc[q][:n], np.float32).view(np.uint32).tobytes(), np.asarray(sg[q][:n], np.uint32).tobytes(),
            np.asarray(dc[q][:n], np.uint32).tobytes())


class Bench:
    """One workload: its whole index on the GPU (one Context) and in the oracle, the four marshalled batches, the oracle's rows of
    the checked queries and the first rows each batch returned."""

    def __init__(self, name):
        from oracle import tq_oracle as O
        import tantivy_b200 as T
        self.name, self.wl = name, workload(name)
        self.dens, self.batches = plan(name)
        t0 = time.perf_counter()
        self.shard = bench.make_shard(self.wl, self.dens, 0, 1, SEED)
        self.ctx = T.Context(0)
        self.shard.register(self.ctx)
        self.qbs = [bench.marshal(self.shard, b) for b in self.batches]
        oi = O.OracleIndex()
        self.shard.register(oi)
        self.checked = [checked_queries(name, b) for b in range(N_BATCHES)]
        threads = len(os.sched_getaffinity(0))
        self.want = []
        t1 = time.perf_counter()
        for b in range(N_BATCHES):
            sub = bench.marshal(self.shard, [self.batches[b][q] for q in self.checked[b]])
            ref = oi.search_batch(sub, mode=0, n_threads=threads)
            self.want.append({int(q): _rows(ref, i) for i, q in enumerate(self.checked[b])})
        self.oracle_s = time.perf_counter() - t1
        self.setup_s = time.perf_counter() - t0
        self.first = [None] * N_BATCHES
        self.stats = []
        del oi

    def check(self, b, res, what):
        """Rows of batch b: the first rows it returned, and the oracle's on the checked queries."""
        got = [_bits(res, q) for q in range(NQ)]
        if self.first[b] is None:
            self.first[b] = got
        else:
            bad = [q for q in range(NQ) if got[q] != self.first[b][q]]
            assert not bad, (self.name, what, b, "rows differ from the batch's first rows", bad[:8])
        for q, want in self.want[b].items():
            assert _rows(res, q) == want, (self.name, what, b, q, self.batches[b][q][:2], _rows(res, q)[:3], want[:3])

    def close(self):
        self.ctx.close()


@pytest.fixture(scope="module")
def wlx(request):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    w = Bench(request.param)
    print(f"\n[{w.name}] setup {w.setup_s:.1f} s, oracle {w.oracle_s:.1f} s for {sum(len(c) for c in w.checked)} queries")
    yield w
    w.close()


COUNTERS = ("tile_groups", "tile_groups_union_only", "tile_fallbacks", "tile_scratch_bytes")


def _record(w, ctx, what, b, split=False):
    st = ctx.stats()
    w.stats.append((what, b, split, {k: int(st[k]) for k in COUNTERS}))


def _check_counters(w):
    """Counters of every step so far.  The tile engine runs every batch but term's: in one group or more at the defaults, two or
    more for or20's twenty-term unions (WIDE_QUERIES of a segment per group), four or more with SPLIT_QUERIES.  No step falls back
    to the per-query kernels, except that mixed's fallbacks are only reported."""
    assert w.stats
    per_group = WIDE_QUERIES if w.wl["n_terms"] > 8 else NQ  # (queries of a segment in one group at the defaults)
    for what, b, split, st in w.stats:
        if w.name != TERM:  # (a batch of single-term queries alone takes k_term)
            need = -(-NQ // (SPLIT_QUERIES if split else per_group))
            assert st["tile_groups"] >= need, (w.name, what, b, need, st)
        if w.name != MIXED:
            assert st["tile_fallbacks"] == 0, (w.name, what, b, st)
    print(f"[{w.name}] counters per step: {[(what, b, split, st) for what, b, split, st in w.stats]}")


# The tile groups of the default plan: 1024 queries of a segment fit one group, so at bench.py's defaults a 512-query batch
# needs several groups only where its lists do not fit one tile buffer, or for queries of more than 8 terms (WIDE_QUERIES to a
# segment, TQ_TILE_WIDE_QUERIES).  Measured on an H100: or5, mixed and and2 run in one group, or20 in two, term on k_term.
# TQ_TILE_MAX_QUERIES (the planner's cap on a group's queries of one segment) at SPLIT_QUERIES makes every batch of the tile
# engine run in NQ / SPLIT_QUERIES groups or more, at the same shapes.
WIDE_QUERIES = 256
SPLIT_QUERIES = 128


@pytest.mark.gpu
@pytest.mark.parametrize("grouping", ["default", "split"])
@pytest.mark.parametrize("wlx", ALL, indirect=True)
def test_value_leg_pipelined_steps(wlx, grouping):
    """bench.py's pipelined_steps at depth 2 over the four prepared batches, CYCLES rounds; rows read after every completed step.
    split: on a second context whose tile groups hold at most SPLIT_QUERIES queries of a segment; the rows are the same."""
    from tests.test_gpu_parity import _ctx_with_env
    w = wlx
    split = grouping == "split"
    ctx = w.ctx
    if split:
        ctx = _ctx_with_env(TQ_TILE_MAX_QUERIES=SPLIT_QUERIES)
        w.shard.register(ctx)
    prepared = [ctx.prepare(qb) for qb in w.qbs]
    try:
        done = []

        def complete(j, bt):
            bt.results_dev()  # waits for the step, as bench.py's complete() does
            _record(w, ctx, f"value {grouping}", j % N_BATCHES, split)
            w.check(j % N_BATCHES, bt.fetch(), f"value {grouping} step {j}")
            done.append(j)

        pending = []
        for j in range(CYCLES * N_BATCHES):
            bt = prepared[j % N_BATCHES]
            bt.run()
            pending.append((j, bt))
            if len(pending) >= DEPTH:
                complete(*pending.pop(0))
        while pending:
            complete(*pending.pop(0))
        assert done == list(range(CYCLES * N_BATCHES))
    finally:
        for bt in prepared:
            bt.close()
        if split:
            ctx.close()
    _check_counters(w)


@pytest.mark.gpu
@pytest.mark.parametrize("wlx", ALL, indirect=True)
def test_e2e_leg_serial_and_pipelined(wlx):
    """search_batch into two alternating host buffers, then e2e_pipelined: step i + 1 prepared and queued while step i runs,
    step i fetched into a host buffer and closed."""
    w = wlx
    outs = [w.qbs[i % len(w.qbs)].alloc_out() for i in range(2)]
    for i in range(N_BATCHES + 2):
        b = i % N_BATCHES
        w.ctx.search_batch(w.qbs[b], outs[i % 2])
        _record(w, w.ctx, "e2e serial", b)
        w.check(b, outs[i % 2][1:], f"e2e serial step {i}")
    count = N_BATCHES + 2
    cur = w.ctx.prepare(w.qbs[0])
    cur.run()
    for i in range(count):
        nxt = w.ctx.prepare(w.qbs[(i + 1) % N_BATCHES]) if i + 1 < count else None
        if nxt is not None:
            nxt.run()
        res = cur.fetch(outs[i % 2])[0:4]
        _record(w, w.ctx, "e2e pipelined", i % N_BATCHES)
        w.check(i % N_BATCHES, res, f"e2e pipelined step {i}")
        cur.close()
        cur = nxt
    _check_counters(w)


@pytest.mark.gpu
@pytest.mark.parametrize("wlx", ALL, indirect=True)
def test_multi_rank_merged_rows(wlx):
    """bench.py's multi-rank path with ranks as threads, at each of WORLDS: make_shard per rank (global statistics summed over the
    ranks), a Context and one CrossGpuMerger (depth 1) per rank; every batch once, then batch 0 again; rank 0's merged rows
    against the whole index."""
    for world in WORLDS[wlx.name]:
        _multi_rank(wlx, world)


def _multi_rank(w, world):
    import torch
    import tantivy_b200 as T
    from tantivy_b200.sharding import CrossGpuMerger
    group = ThreadGroup(world)
    shards, ctxs = [None] * world, [None] * world
    got = [[] for _ in range(world)]
    steps = list(range(N_BATCHES)) + [0]

    def rank(r, dist):
        shards[r] = bench.make_shard(w.wl, w.dens, r, world, SEED, dist)
        ctxs[r] = T.Context(0)
        shards[r].register(ctxs[r])
        qbs = [bench.marshal(shards[r], b) for b in w.batches]
        m = CrossGpuMerger(ctxs[r], dist, torch.device("cuda", 0), NQ, w.wl["k"])
        for b in steps:
            bt = ctxs[r].prepare(qbs[b])
            try:
                m.run(bt)
                m.finish_async(bt)
                rows = m.complete(bt, rows_to_host=True)
                got[r].append([_bits(rows, q) for q in range(NQ)] if r else tuple(np.array(x) for x in rows))
            finally:
                bt.close()

    try:
        group.run(rank)
    finally:
        for c in ctxs:
            if c is not None:
                c.close()
    assert shards[0].total_docs == w.shard.total_docs and (shards[0].df == w.shard.df).all() and shards[0].avg == w.shard.avg
    for i, b in enumerate(steps):
        res = got[0][i]
        for q, want in w.want[b].items():
            assert _rows(res, q) == want, (w.name, world, i, b, q, w.batches[b][q][:2], _rows(res, q)[:3], want[:3])
        mine = [_bits(res, q) for q in range(NQ)]
        for r in range(1, world):
            assert got[r][i] == mine, (w.name, world, "rank", r, "merged rows differ from rank 0's", i)


@pytest.mark.gpu
@pytest.mark.parametrize("wlx", BENCH_RUNS, indirect=True)
def test_bench_end_to_end(wlx, tmp_path):
    """bench.py as a subprocess: its parity block over all 512 queries of batch 0, and the rows it dumps after the pipelined
    value leg (fetch of the batch it ran last) against the oracle."""
    import json
    w = wlx
    out = tmp_path / "dump"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--workload", w.name, "--steps", "2", "--warmup", "1",
                        "--parity-queries", str(NQ), "--dump-outputs", str(out), "--no-cpu-baseline"],
                       capture_output=True, text=True, timeout=1800, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1, r.stdout[-2000:]
    d = json.loads(lines[0])
    p = d["parity"]
    assert p["checked"] == NQ and p["mismatches"] == 0 and p["first_mismatch"] is None, p
    assert p["rows"] == sum(len(v) for v in w.want[0].values())
    print(f"[{w.name}] bench.py: parity oracle {p['oracle_s']} s, tile_fallback_steps {d['workload_stats']['tile_fallback_steps']}")
    # what pipelined_steps ran last (bench.py raises --warmup to its minimum; the line reports the value it used)
    last = (d["warmup"] + d["steps"] - 1) % N_BATCHES
    a = {n: np.load(out / f"{n}.npy") for n in ("scores", "segment_ords", "docs", "counts", "query_index")}
    assert (a["query_index"] == np.arange(NQ)).all()
    res = (a["scores"], a["segment_ords"].astype(np.uint32), a["docs"].astype(np.uint32), a["counts"].astype(np.uint32))
    for q, want in w.want[last].items():
        assert _rows(res, q) == want, (w.name, "dumped", last, q, _rows(res, q)[:3], want[:3])
    if w.first[last] is not None:
        assert [_bits(res, q) for q in range(NQ)] == w.first[last]


# ---- ranks as threads -----------------------------------------------------------------------------------------------------------
class ThreadGroup:
    """The in-process process group of tests/test_gpu_shard_exchange.py (all_gather_into_tensor between threads of one process),
    with the all_reduce (sum) that make_shard's global statistics take."""

    def __init__(self, world):
        from tests.test_gpu_shard_exchange import FakeDist
        self.d = FakeDist(world)
        self.world = world

    def view(self, r):
        d, base = self.d, self.d.rank(r)

        class View:
            def get_world_size(self):
                return d.world

            def is_initialized(self):
                return True

            def all_gather_into_tensor(self, out, inp):
                base.all_gather_into_tensor(out, inp)

            def all_reduce(self, t, op=None):
                import torch
                assert op is None  # (a sum)
                out = torch.empty((d.world,) + tuple(t.shape), dtype=t.dtype, device=t.device)
                d.gather(r, out, t)
                t.copy_(out.sum(0))
        return View()

    def run(self, fn):
        """fn(rank, view) on one thread per rank; re-raises the first failure after every thread has ended (a failing rank breaks
        the group's barrier, so no thread waits for it)."""
        import threading
        errors = [None] * self.world

        def body(r):
            try:
                fn(r, self.view(r))
            except BaseException as e:  # noqa: BLE001
                errors[r] = e
                self.d.barrier.abort()

        threads = [threading.Thread(target=body, args=(r,)) for r in range(self.world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout=1200)
        assert not any(t.is_alive() for t in threads)
        first = next((e for e in errors if e is not None and not isinstance(e, threading.BrokenBarrierError)), None) or next(
            (e for e in errors if e is not None), None)
        if first is not None:
            raise first
