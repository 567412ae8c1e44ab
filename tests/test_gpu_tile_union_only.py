"""k_tile's union-only instances: a group whose queries are all term queries and unions runs k_tile<*, *, true> (no conjunction
or TQ_OP_BOOL code, each work-list segment's query state broadcast to its posting lanes); the same queries in a group with a
conjunction run the general instance.  Both must return the oracle's exhaustive rows, bit for bit: on every route through k_tile,
at the scoring edges of tests/test_gpu_scoring_edges.py, on the shapes only unions have (a repeated term, absent clauses, deletes,
initial thresholds, doc-range parts), at every group size up to kTileMaxQueries (1024 queries of a segment) and one past it, and
in the largest group the planner admits.  Every test asserts, through tq_stats.tile_groups_union_only, which instance ran."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from oracle import tq_oracle as O  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM, TQ_RECORD_BASIC, TQ_TERM_IGNORE_FREQ, QueryBatch  # noqa: E402
from tests import score_model as M  # noqa: E402
from tests.helpers import hits, make_query, tile_smem_bytes  # noqa: E402
from tests.test_gpu_parity import (DOC_RANGE_CUTS, TILE_OVERFLOW_HOOKS, TILE_PATH_HOOKS, _ctx_with_env, _tile_queries,  # noqa: E402
                                   assert_same)
from tests.test_gpu_scoring_edges import _segment, _variants, large, small, wide  # noqa: E402,F401  (fixtures)

_DENS = [0.3, 0.15, 0.05, 0.01, 0.002, 0.0001]
_BASE = 9100


def _hook_id(h):
    return ",".join(f"{k}={v}" for k, v in h.items()) or "default"


def assert_instance(st, union_only, groups=None):
    """The batch ran in tile groups (`groups` of them if given), all on the union-only instance or all on the general one;
    nothing overflowed."""
    assert st["tile_groups"] >= 1 if groups is None else st["tile_groups"] == groups, st["tile_groups"]
    assert st["tile_groups_union_only"] == (st["tile_groups"] if union_only else 0), (st["tile_groups_union_only"], st["tile_groups"])
    assert st["tile_fallbacks"] == 0


@pytest.fixture(scope="module")
def synth():
    ix = T.SynthIndex(3, 1_000_000, _DENS, seed=91)
    oi = O.OracleIndex()
    ix.register(oi, segment_base=_BASE)
    return ix, oi


def _unions(ix):
    qs = [ix.query(TQ_OP_OR, terms, k, segment_base=_BASE)
          for k in (1, 10, 100, 1000) for terms in ([0, 5], [0, 4, 5], [1, 0, 5, 3], [5, 4, 3, 2, 1, 0], [2, 3, 4], [0, 1])]
    return qs + [ix.query(TQ_OP_TERM, [t], k, segment_base=_BASE) for t in (0, 3, 5) for k in (10, 100)]


_HOOKS = [dict(), dict(TQ_TILE_SEG_CAP=3), dict(TQ_TILE_LIGHT_MAX=0)]


@pytest.mark.parametrize("hook", _HOOKS, ids=_hook_id)
@pytest.mark.parametrize("counters", [0, 1])
def test_unions_alone_and_beside_a_conjunction(synth, hook, counters):
    ix, oi = synth
    unions = _unions(ix)
    qb_u = QueryBatch(unions)
    qb_m = QueryBatch(unions + [ix.query(TQ_OP_AND, [0, 2], 100, segment_base=_BASE)])  # the group now runs the general instance
    want = oi.search_batch(qb_m, mode=0, n_threads=16)
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, TQ_TILE_COUNTERS=counters, **hook)
    try:
        ix.register(c, segment_base=_BASE)
        g_u = c.search_batch(qb_u)
        st = c.stats()
        assert_instance(st, union_only=True)
        if counters:
            ctr, cyc = st["tile_counters"], st["tile_cycles"]
            assert ctr[2] > 0 and ctr[4] > 0  # light pairs and essential postings went through B2 ...
            if "TQ_TILE_LIGHT_MAX" in hook:
                assert ctr[3] > 0  # ... and heavy pairs through B3
            assert cyc[1] > 0 and cyc[3] > 0  # stage cycles: A and B2 ran
        g_m = c.search_batch(qb_m)
        assert_instance(c.stats(), union_only=False)
    finally:
        c.close()
    assert_same(g_m, want, qb_m.nq)
    assert_same(g_u, want, qb_u.nq)
    for i in range(qb_u.nq):
        assert hits(g_u, i) == hits(g_m, i), f"query {i}: the union-only and the general instance differ"
    assert sum(1 for i in range(qb_u.nq) if hits(g_u, i)) >= qb_u.nq // 2


# ---- every route through k_tile ----------------------------------------------------------------------------------------
_ROUTE_BASE = 9200


@pytest.fixture(scope="module")
def routes():
    """test_tile_paths_agree's index (seed 77: on it no route but the one without a sample launch overflows a candidate region),
    its unions and term queries; the same beside one conjunction; the oracle's rows of the latter."""
    ix = T.SynthIndex(3, 1_000_000, _DENS, seed=77)
    oi = O.OracleIndex()
    ix.register(oi, segment_base=_ROUTE_BASE)
    qs = _tile_queries(ix, _ROUTE_BASE) + [ix.query(TQ_OP_TERM, [t], 10, segment_base=_ROUTE_BASE) for t in range(6)]
    qb_m = QueryBatch(qs + [ix.query(TQ_OP_AND, [0, 1], 10, segment_base=_ROUTE_BASE)])
    return ix, QueryBatch(qs), qb_m, oi.search_batch(qb_m, mode=0, n_threads=16)


def _both_instances(routes, fallbacks, **env):
    ix, qb_u, qb_m, want = routes
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, **env)
    try:
        ix.register(c, segment_base=_ROUTE_BASE)
        g_u = c.search_batch(qb_u)
        st_u = c.stats()
        g_m = c.search_batch(qb_m)
        st_m = c.stats()
    finally:
        c.close()
    for st, union_only in ((st_u, True), (st_m, False)):
        assert st["tile_groups"] == 1 and st["tile_groups_union_only"] == (1 if union_only else 0)
        assert st["tile_fallbacks"] == fallbacks
    assert_same(g_u, want, qb_u.nq)
    assert_same(g_m, want, qb_m.nq)
    for i in range(qb_u.nq):
        assert hits(g_u, i) == hits(g_m, i), f"query {i}: the union-only and the general instance differ"
    return st_u


@pytest.mark.parametrize("hook,counters", [(h, 0) for h in TILE_PATH_HOOKS] + [(dict(TQ_TILE_SEG_CAP=3), 1), (dict(TQ_TILE_LIGHT_MAX=0), 1)],
                         ids=lambda x: _hook_id(x) if isinstance(x, dict) else f"counters={x}")
def test_every_tile_route_union_only(routes, hook, counters):
    """The routes of test_tile_paths_agree on a batch of unions and term queries alone (without TQ_TILE_COUNTERS: the production
    instance, four CTAs per SM) and beside one conjunction: the same rows.  Without a sample launch the k = 1000 unions overflow
    their candidate regions and the run is repeated, as in test_tile_paths_agree."""
    st = _both_instances(routes, 1 if "TQ_TILE_SAMPLE_DIV" in hook else 0, TQ_TILE_COUNTERS=counters, **hook)
    if counters:
        assert st["tile_counters"][4] > 0 and st["tile_cycles"][3] > 0  # essential postings went through B2


@pytest.mark.parametrize("hook", TILE_OVERFLOW_HOOKS, ids=_hook_id)
def test_union_only_overflow_is_repeated(routes, hook):
    _both_instances(routes, 1, **hook)


# ---- the scoring edges of test_gpu_scoring_edges.py, one op per batch ---------------------------------------------------------
@pytest.fixture(scope="module")
def tctx():
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1)
    yield c
    c.close()


def _run_alone(ctx, segs, queries, terms, overflow=()):
    """Term queries and unions in batches of one op each: device == model == oracle (docs, segment ordinals, f32 scores), on the
    union-only instance.  The queries listed in `overflow` go in a batch of their own that overflows and is repeated."""
    osegs, msegs = [o for o, _ in segs], [m for _, m in segs]
    oi = O.OracleIndex()
    for s in osegs:
        s.register(oi)
        s.register(ctx)
    batches = [[i for i, q in enumerate(queries) if q["op"] == op and i not in overflow] for op in (TQ_OP_TERM, TQ_OP_OR)]
    for idx, fallbacks in zip(batches + [list(overflow)], (0, 0, 1)):
        if not idx:
            continue
        qb = QueryBatch([queries[i] for i in idx])
        g = ctx.search_batch(qb)
        st = ctx.stats()
        assert st["tile_groups"] >= 1 and st["tile_groups_union_only"] == st["tile_groups"]
        assert st["tile_fallbacks"] == fallbacks
        c = oi.search_batch(qb, mode=0)
        for j, i in enumerate(idx):
            want = M.search(msegs, queries[i], terms[i])
            assert hits(g, j) == want, f"query {i}: device {hits(g, j)[:4]} != model {want[:4]}"
            assert hits(c, j) == want, f"query {i}: oracle {hits(c, j)[:4]} != model {want[:4]}"


def _flagged(q, flags):
    return dict(q, term_flags=flags)


def test_scoring_edges_small_segment(tctx, small):
    """tf edges and every fieldnorm id; average fieldnorm 1 and 1e6, a tf cache, boosts 0 / -1.5 / 1e4 / 1e-4; a mixed-sign union
    (not prunable) and negative thresholds; clauses read without freqs."""
    lists, lengths = small
    seg = _segment(lists, lengths)
    queries, terms = [], []
    for op, c in [(TQ_OP_TERM, [0]), (TQ_OP_TERM, [1]), (TQ_OP_OR, [0, 1, 2]), (TQ_OP_OR, [4, 3, 2, 1, 0])]:
        for q in _variants(make_query(op, [seg[0]], c, 1024), len(c)):
            queries.append(q)
            terms.append(c)
    q = make_query(TQ_OP_OR, [seg[0]], [0, 1, 4], 1024)
    q["weights"] = [q["weights"][0], -q["weights"][1], q["weights"][2]]
    queries += [q, dict(q, threshold=-0.5), dict(make_query(TQ_OP_OR, [seg[0]], [0, 1], 1024, boost=-1.5), threshold=-1.0)]
    terms += [[0, 1, 4], [0, 1, 4], [0, 1]]
    queries += [_flagged(make_query(TQ_OP_OR, [seg[0]], [0, 1, 2], 1024), [TQ_TERM_IGNORE_FREQ, 0, TQ_TERM_IGNORE_FREQ]),
                _flagged(make_query(TQ_OP_TERM, [seg[0]], [1], 1024), [TQ_TERM_IGNORE_FREQ])]
    terms += [[0, 1, 2], [1]]
    _run_alone(tctx, [seg], queries, terms)


def test_scoring_edges_large_segment(tctx, large):
    """Large-tf docs at the top of every ranking, so that tile-max pruning runs on them."""
    lists, lengths = large
    seg = _segment(lists, lengths)
    queries, terms = [], []
    for op, c in [(TQ_OP_TERM, [0]), (TQ_OP_TERM, [3]), (TQ_OP_OR, [0, 1, 2]), (TQ_OP_OR, [0, 1, 2, 3, 4, 5]), (TQ_OP_OR, [3, 2])]:
        for k in (1, 128, 129, 1024):
            queries.append(make_query(op, [seg[0]], c, k))
            terms.append(c)
    # boost 0 (_variants entry 4): every doc of a dense list scores 0 and ties with the k-th, so all of them are candidates; more
    # than a candidate region holds: that batch is repeated
    tied = []
    for c in ([0, 1, 2], [0], [3]):
        op = TQ_OP_OR if len(c) > 1 else TQ_OP_TERM
        for j, q in enumerate(_variants(make_query(op, [seg[0]], c, 100), len(c))[1:], start=1):
            if j == 4 and c != [3]:
                tied.append(len(queries))
            queries.append(q)
            terms.append(c)
    q = make_query(TQ_OP_OR, [seg[0]], [0, 1, 2, 3], 128)
    q["weights"] = [q["weights"][0], -q["weights"][1], q["weights"][2], -q["weights"][3]]
    queries += [q, dict(q, threshold=-0.25), _flagged(make_query(TQ_OP_OR, [seg[0]], [0, 1, 2, 3, 4, 5], 129), [0, 1, 0, 1, 0, 1])]
    terms += [[0, 1, 2, 3], [0, 1, 2, 3], [0, 1, 2, 3, 4, 5]]
    _run_alone(tctx, [seg], queries, terms, overflow=tied)


def test_scoring_edges_nine_and_thirty_two_clauses(tctx, wide):
    lists, lengths = wide
    seg = _segment(lists, lengths)
    queries, terms = [], []
    for n in (9, 32):
        c = list(range(0, 32, 32 // n))[:n] if n == 9 else list(range(32))
        for k in (1, 128, 129, 1024):
            queries.append(make_query(TQ_OP_OR, [seg[0]], c, k))
            terms.append(c)
        queries.append(_flagged(make_query(TQ_OP_OR, [seg[0]], c, 1024), [0] * (n - 1) + [TQ_TERM_IGNORE_FREQ]))
        terms.append(c)
    _run_alone(tctx, [seg], queries, terms)


def test_scoring_edges_constant_fieldnorm_and_basic_fields(tctx, small):
    lists, lengths = small
    n = len(lengths)
    const = _segment(lists, None, max_doc=n)
    basic = _segment([(d, None) for d, _ in lists], lengths, record_option=TQ_RECORD_BASIC)
    for seg in (const, basic):
        queries, terms = [], []
        for op, c in [(TQ_OP_TERM, [0]), (TQ_OP_OR, [0, 1, 2, 3, 4]), (TQ_OP_OR, [2, 3])]:
            for q in _variants(make_query(op, [seg[0]], c, 1024), len(c)):
                queries.append(q)
                terms.append(c)
        _run_alone(tctx, [seg], queries, terms)


# ---- shapes only unions have ----------------------------------------------------------------------------------------------
def _random_model_segments(rng, n_segments, n_terms, deletes):
    """Explicit segments (device, oracle and model) of 20k-40k docs with lists from dense to rare, optionally with deletes."""
    segs = []
    for _ in range(n_segments):
        max_doc = int(rng.integers(20_000, 40_000))
        lengths = np.clip(np.round(np.exp(rng.normal(np.log(40), 0.7, size=max_doc))), 1, 4096).astype(np.uint32)
        lists = []
        for t in range(n_terms):
            p = (0.4, 0.15, 0.05, 0.01, 0.003, 0.2)[t % 6] * float(rng.uniform(0.7, 1.3))
            docs = np.nonzero(rng.random(max_doc) < p)[0].astype(np.uint32)
            lists.append((docs, np.minimum(rng.geometric(0.5, size=len(docs)), 40).astype(np.uint32)))
        alive = np.packbits(rng.random(max_doc) > 0.25, bitorder="little") if deletes else None
        segs.append(_segment(lists, lengths, alive=alive))
    return segs


def test_repeated_terms_absent_clauses_and_deletes(tctx):
    """`a OR a OR b` (two clauses on one scored list: one doc, two essential postings), the same term under two boosts (two
    lists), a clause absent from one segment and one absent from all but one, over segments with deletes."""
    rng = np.random.default_rng(1201)
    segs = _random_model_segments(rng, 3, 6, deletes=True)
    osegs = [o for o, _ in segs]
    osegs[1].terms[3] = (0, 0, 0)  # term 3 absent from segment 1
    osegs[1].terms[4] = (0, 0, 0)  # term 4 only in segment 0
    osegs[2].terms[4] = (0, 0, 0)
    queries, terms = [], []
    for c, boost in [([0, 0, 1], 1.0), ([1, 0, 1, 4], 1.0), ([0, 0], [1.0, 2.0]), ([2, 5, 2], [0.5, 1.0, 3.0]), ([5, 5, 5, 5], 1.0),
                     ([3, 4], 1.0), ([0, 3, 4], 1.0), ([4, 1, 3, 3], 1.0), ([3, 0], 1.0), ([4, 2, 5, 1, 0, 3], 1.0)]:
        for k in (1, 5, 50, 1000):
            queries.append(make_query(TQ_OP_OR, osegs, c, k, boost=boost))
            terms.append(c)
    for t in (3, 4, 0):
        for k in (5, 1000):
            queries.append(make_query(TQ_OP_TERM, osegs, [t], k))
            terms.append([t])
    _run_alone(tctx, segs, queries, terms)


def test_initial_threshold_like_for_each_pruning(tctx):
    """tq_query.threshold (Weight::for_each_pruning's `threshold`): the middle, last and first score of a finished search, 0, -1."""
    rng = np.random.default_rng(1202)
    segs = _random_model_segments(rng, 3, 6, deletes=False)
    osegs, msegs = [o for o, _ in segs], [m for _, m in segs]
    shapes = [(TQ_OP_TERM, [1]), (TQ_OP_OR, [0, 1, 2, 3, 4]), (TQ_OP_OR, [4, 2]), (TQ_OP_OR, [0, 3, 4]), (TQ_OP_OR, [5, 0, 0]),
              (TQ_OP_OR, [1, 5])]
    base = [make_query(op, osegs, c, 40) for op, c in shapes]
    oi = O.OracleIndex()
    for s in osegs:
        s.register(oi)
        s.register(tctx)
    qb0 = QueryBatch(base)
    g0 = tctx.search_batch(qb0)
    assert_instance(tctx.stats(), union_only=True)
    assert_same(g0, oi.search_batch(qb0, mode=0), qb0.nq)
    queries, terms = [], []
    for i, (op, c) in enumerate(shapes):
        h = hits(g0, i)
        assert len(h) == 40
        for thr in (h[len(h) // 2][0], h[-1][0], h[0][0], 0.0, -1.0):
            queries.append(dict(base[i], threshold=float(thr), k=60))
            terms.append(c)
    qb = QueryBatch(queries)
    g = tctx.search_batch(qb)
    assert_instance(tctx.stats(), union_only=True)
    c = oi.search_batch(qb, mode=0)
    for i, (q, t) in enumerate(zip(queries, terms)):
        want = M.search(msegs, q, t)
        assert hits(g, i) == want, f"query {i}: device {hits(g, i)[:4]} != model {want[:4]}"
        assert hits(c, i) == want
        assert all(s > np.float32(q["threshold"]) for s, _, _ in hits(g, i))


@pytest.mark.parametrize("cuts", DOC_RANGE_CUTS)
def test_doc_range_parts_merge_to_the_whole_segment(cuts):
    """The cuts of test_gpu_parity's doc-range test, with a batch of unions and term queries only."""
    from tantivy_b200.sharding import merge_rows_host
    ix = T.SynthIndex(1, 300_000, [0.3, 0.05, 0.01, 0.002, 0.0004], seed=31)
    for deletes in (False, True):
        alive = np.packbits(np.random.default_rng(5).random(300_000) > 0.3, bitorder="little") if deletes else None
        base = 9300 + int(deletes)
        oi = O.OracleIndex()
        oi.segment_register(base, 0, ix.max_doc[0], ix.record_option, ix.body(0), ix.fieldnorm(0), alive)
        qs = [ix.query(TQ_OP_TERM, [t], 10, segment_base=base) for t in range(5)]
        qs += [ix.query(TQ_OP_OR, ts, k, segment_base=base) for ts in ([0, 1, 2, 3, 4], [3, 4], [1, 4], [2, 3], [0, 1], [4, 0, 4])
               for k in (1, 50, 700)]
        qb = QueryBatch(qs)
        want = oi.search_batch(qb, mode=0, n_threads=8)
        rows = []
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1)
            try:
                c.segment_register(base, 0, ix.max_doc[0], ix.record_option, ix.body(0), ix.fieldnorm(0), alive)
                c.segment_set_doc_range(base, 0, lo, hi)
                r = c.search_batch(qb)
                st = c.stats()
                assert st["tile_groups_union_only"] == st["tile_groups"] and st["tile_fallbacks"] == 0
                if hi > lo:
                    assert st["tile_groups"] >= 1
                for q in range(qb.nq):
                    assert all(lo <= d < hi for _, _, d in hits(r, q))
                rows.append([np.array(x) for x in r])
            finally:
                c.close()
        kmax = max(q["k"] for q in qs)
        m = merge_rows_host(np.stack([r[0] for r in rows]), np.stack([r[1] for r in rows]), np.stack([r[2] for r in rows]),
                            np.stack([r[3] for r in rows]), kmax)
        for q in range(qb.nq):
            n = int(want[3][q])
            assert int(m[3][q]) >= n
            assert (m[1][q, :n] == want[1][q, :n]).all() and (m[2][q, :n] == want[2][q, :n]).all()
            assert (m[0][q, :n].view(np.uint32) == want[0][q, :n].view(np.uint32)).all()


# ---- group size: queries 0..1024 of a segment, both instances --------------------------------------------------------------
# 24 terms from dense to rare on 2 x 200k docs: small enough for the oracle to check every row of every query
_POOL_DENS = [0.3, 0.2, 0.12, 0.08, 0.05, 0.03, 0.02, 0.012, 0.008, 0.005, 0.003, 0.002,
              0.04, 0.01, 0.006, 0.0015, 0.001, 0.0007, 0.0005, 0.0004, 0.0003, 0.0002, 0.025, 0.0025]
_POOL_BASE = 9400
_N_NARROW, _N_WIDE = 1100, 300


@pytest.fixture(scope="module")
def pool():
    """The index, 1100 seeded unions of 2-8 terms, 300 of 9-20 terms (k of 1 / 10 / 100 / 1000 each), a conjunction, and the
    oracle's rows of all of them (one exhaustive batch: a query's rows do not depend on its batch)."""
    ix = T.SynthIndex(2, 200_000, _POOL_DENS, seed=0x5EED)
    assert all(ix.term_info[s][t][0] > 0 for s in range(2) for t in range(len(_POOL_DENS)))
    rng = np.random.default_rng(77)
    nt = len(_POOL_DENS)

    def draw(lo, hi):
        terms = [int(t) for t in rng.choice(nt, size=int(rng.integers(lo, hi + 1)), replace=False)]
        return ix.query(TQ_OP_OR, terms, int(rng.choice([1, 10, 100, 1000])), segment_base=_POOL_BASE)

    narrow = [draw(2, 8) for _ in range(_N_NARROW)]
    wide_ = [draw(9, 20) for _ in range(_N_WIDE)]
    conj = ix.query(TQ_OP_AND, [0, 2], 100, segment_base=_POOL_BASE)
    oi = O.OracleIndex()
    ix.register(oi, segment_base=_POOL_BASE)
    allq = narrow + wide_ + [conj]
    want = oi.search_batch(QueryBatch(allq), mode=0, n_threads=32)
    return ix, narrow, wide_, conj, want


@pytest.fixture(scope="module")
def pool_ctx(pool):
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1)
    pool[0].register(c, segment_base=_POOL_BASE)
    yield c
    c.close()


def _pool_row(pool, q):
    """Index into the pool's oracle rows of query dict q."""
    _, narrow, wide_, conj, _ = pool
    for i, p in enumerate(narrow + wide_ + [conj]):
        if p is q:
            return i
    raise KeyError


def _same_rows(got, gi, want, wi):
    n = int(want[3][wi])
    assert int(got[3][gi]) == n, f"batch row {gi} (pool query {wi}): {int(got[3][gi])} hits, the oracle has {n}"
    assert (got[2][gi, :n] == want[2][wi, :n]).all() and (got[1][gi, :n] == want[1][wi, :n]).all(), f"batch row {gi}: doc ids differ"
    assert (got[0][gi, :n].view(np.uint32) == want[0][wi, :n].view(np.uint32)).all(), f"batch row {gi}: scores differ"


def _run_pool(ctx, pool, queries):
    """Every row of the batch against the oracle; the batch's stats."""
    want = pool[4]
    rows = [_pool_row(pool, q) for q in queries]
    g = ctx.search_batch(QueryBatch(queries))
    st = ctx.stats()
    for gi, wi in enumerate(rows):
        _same_rows(g, gi, want, wi)
    return g, st


def _groups(widths, max_q=1024, wide_q=256):
    """Tile groups the planner opens for queries of these clause counts (in batch order) when only the query limits bind: a
    query of more than 8 clauses joins a group only while it holds fewer than wide_q queries of the segment."""
    groups, size = 1, 0
    for w in widths:
        if size + 1 > (min(max_q, wide_q) if w > 8 else max_q):
            groups, size = groups + 1, 0
        size += 1
    return groups


def _check_groups(st, queries, n_general, **limits):
    groups = _groups([len(q["weights"]) for q in queries], **limits)
    assert st["tile_groups"] == groups and st["tile_groups_union_only"] == groups - n_general, (st["tile_groups"], st["tile_groups_union_only"], groups)
    assert st["tile_fallbacks"] == 0


@pytest.mark.parametrize("n", [255, 257, 511, 513, 1024, 1025])
@pytest.mark.parametrize("conj", [None, "first", "last"])
def test_group_sizes(pool, pool_ctx, n, conj):
    """Batches of n queries per segment: B1 prefetches the thresholds of queries tid and tid + 256 and loads the others in its
    loop; 1025 queries open a second group.  With a conjunction first or last, the group that holds it runs the general instance
    (at 1025: one of the two groups)."""
    _, narrow, _, c, _ = pool
    qs = list(narrow[:n])
    if conj == "first":
        qs[0] = c
    elif conj == "last":
        qs[-1] = c
    _, st = _run_pool(pool_ctx, pool, qs)
    assert st["tile_groups"] == (1 if n <= 1024 else 2)
    _check_groups(st, qs, 1 if conj else 0)


@pytest.mark.parametrize("env,n,n_general", [(dict(TQ_TILE_SEG_CAP=3), 1024, 0), (dict(TQ_TILE_SEG_CAP=3), 1024, 1),
                                              (dict(TQ_TILE_MAX_QUERIES=1), 40, 0), (dict(TQ_TILE_MAX_QUERIES=7), 100, 0),
                                              (dict(TQ_TILE_MAX_QUERIES=7), 100, 1)],
                         ids=lambda x: _hook_id(x) if isinstance(x, dict) else str(x))
def test_group_sizes_under_hooks(pool, env, n, n_general):
    """A three-entry work list defers nearly every pair to further routing rounds (queries above 512 included); one or seven
    queries per group split the batch into many groups.  n_general = 1: a conjunction in the middle of the batch puts its group
    on the general instance."""
    ix, narrow, _, conj, _ = pool
    qs = list(narrow[:n])
    if n_general:
        qs[n // 2 + 3] = conj
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, **env)
    try:
        ix.register(c, segment_base=_POOL_BASE)
        _, st = _run_pool(c, pool, qs)
    finally:
        c.close()
    _check_groups(st, qs, n_general, max_q=env.get("TQ_TILE_MAX_QUERIES", 1024))


@pytest.mark.parametrize("mix", ["alone", "interleaved", "after_narrow"])
def test_wide_union_groups(pool, pool_ctx, mix):
    """300 unions of 9-20 clauses: at most TQ_TILE_WIDE_QUERIES (256) of them per group, alone or among narrow unions."""
    _, narrow, wide_, _, _ = pool
    if mix == "alone":
        qs = list(wide_)
    elif mix == "interleaved":
        qs = [q for pair in zip(wide_, narrow[:_N_WIDE]) for q in pair]
    else:
        qs = narrow[:600] + list(wide_)
    _, st = _run_pool(pool_ctx, pool, qs)
    _check_groups(st, qs, 0)
    assert st["tile_groups"] == {"alone": 2, "interleaved": 3, "after_narrow": 3}[mix]


def test_rows_do_not_depend_on_the_batch(pool, pool_ctx):
    """About 20 queries spread over a 1025-query batch (some above 512): alone in a batch they return the same rows."""
    _, narrow, _, _, want = pool
    big, _ = _run_pool(pool_ctx, pool, narrow[:1025])
    for i in (0, 1, 31, 32, 100, 255, 256, 257, 300, 511, 512, 513, 600, 700, 800, 900, 1000, 1023, 1024):
        one = pool_ctx.search_batch(QueryBatch([narrow[i]]))
        assert_instance(pool_ctx.stats(), union_only=True, groups=1)
        n = int(big[3][i])
        assert int(one[3][0]) == n
        for a, b in zip(one[:3], big[:3]):
            assert (a[0, :n] == b[i, :n]).all(), f"query {i}: alone != in the batch"
        _same_rows(one, 0, want, i)


# ---- the largest group the planner admits ---------------------------------------------------------------------------------
def test_largest_union_group_launches():
    """1024 eight-term unions on one segment over 4096 distinct lists (kTileMaxSlots), 64 of them dense (kTileMaxBig), with the
    lists' densities summing to near the tile pair buffer's limit: one group, on the union-only instance, within the shared
    memory a CTA can have, and the oracle's rows."""
    max_doc, n_terms = 262_144, 4096
    dens = [0.05] * 64 + [0.00109] * (n_terms - 64)
    ix = T.SynthIndex(1, max_doc, dens, seed=0x1A76E)
    base = 9500
    qs = [ix.query(TQ_OP_OR, [(8 * i + j * 17) % n_terms for j in range(8)], (1, 10, 100, 1000)[i % 4], segment_base=base)
          for i in range(1024)]
    # the planner's pair-buffer estimate (stage_tile_groups): slots in the order they join the group (a query's clauses by
    # descending weight), density = doc_freq / max_doc summed
    seen, total = set(), 0.0
    for i in range(1024):
        terms = [(8 * i + j * 17) % n_terms for j in range(8)]
        for _, t in sorted(zip(qs[i]["weights"], terms), key=lambda wt: -wt[0]):
            if t not in seen:
                seen.add(t)
                total += ix.term_info[0][t][0] / max_doc
    assert len(seen) == n_terms
    assert total * 1024 * 1.5 + 256 <= 12288  # tile_fits admits every query ...
    assert total > 7.3  # ... near its limit
    p_cap = (int(min(12288.0, max(1024.0, total * 1024 * 1.25 + 192.0))) + 63) & ~63
    n_big = sum(1 for t in range(n_terms) if ix.term_info[0][t][0] * 1024 >= 6 * max_doc)
    assert n_big >= 64
    want_smem = tile_smem_bytes(p_cap, n_terms, 64, 1024, 2048, 8192, 2)
    oi = O.OracleIndex()
    ix.register(oi, segment_base=base)
    qb = QueryBatch(qs)
    want = oi.search_batch(qb, mode=0, n_threads=32)
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1)
    try:
        ix.register(c, segment_base=base)
        g = c.search_batch(qb)
        st = c.stats()
    finally:
        c.close()
    assert_instance(st, union_only=True, groups=1)
    assert st["tile_counters"][7] == want_smem <= 200 * 1024, (st["tile_counters"][7], want_smem)
    assert st["tile_ctas_per_sm"] >= 1
    assert_same(g, want, qb.nq)
