"""(Count, TopDocs) in one batch: TQ_QUERY_COUNT_HITS and tq_batch_fetch_hits.  Hits are checked against the score model
(tests/score_model.py, M.count) and against tq_count_batch.  Rows are checked bit for bit against the same batch unflagged and
against M.search.  Shapes: TERM, AND of 2-5 clauses, OR of 2-20 and every BOOL_SHAPES entry, with k of 1 / 10 / 1000, with and
without thresholds, over segments with deletes and absent terms, on both engines (BOOL: tile engine only).  Routes: every tile
hook, several tile groups, part of a batch on the per-query kernels, single-term batches on k_term, 1025-query batches,
doc-range parts on several contexts, a phased run with imported thresholds, a prepared batch run twice, sparse offsets that
overflow k_count_tiles' tile buffer, and a segment of 2^31 - 2 docs."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM, QueryBatch  # noqa: E402
from tests import score_model as M  # noqa: E402
from tests.helpers import BOOL_SHAPES, OracleSegment, bool_query, hits, make_query  # noqa: E402
from tests.test_gpu_parity import TILE_OVERFLOW_HOOKS, TILE_PATH_HOOKS, _ctx_with_env, fresh_ord  # noqa: E402
from tests.test_gpu_phrase import PosSegment, phrase_query  # noqa: E402

N_TERMS = 24
DENS = (0.3, 0.1, 0.05, 0.01, 0.002, 0.2)
KS = (1, 10, 1000)
AND_SETS = [[0, 1], [1, 3], [0, 2, 4], [5, 0, 1, 2], [6, 7, 8, 9, 11]]
OR_SETS = [[0, 4], [3, 9], [1, 2, 3], [0, 6, 12, 18, 4], list(range(2, 22, 2)), list(range(20)), [23, 22]]


class Fixture:
    """Three segments: deletes in two of them (the third takes tq_count_batch's doc_freq shortcut for terms), terms absent from
    some segments, doc ranges that hold several thousand tiles in all.  Device segments and their model, same lists."""

    def __init__(self, seed=0xC0):
        rng = np.random.default_rng(seed)
        self.osegs, self.msegs = [], []
        for i in range(3):
            max_doc = int(rng.integers(40_000, 120_000))
            lengths = np.clip(np.round(np.exp(rng.normal(np.log(40), 0.7, size=max_doc))), 1, 4096).astype(np.uint32)
            lists = []
            for t in range(N_TERMS):
                p = DENS[t % len(DENS)] * float(rng.uniform(0.5, 1.5))
                docs = np.nonzero(rng.random(max_doc) < p)[0].astype(np.uint32)
                lists.append((docs, np.minimum(rng.geometric(0.6, size=len(docs)), 10).astype(np.uint32)))
            alive = None if i == 2 else np.packbits(rng.random(max_doc) > 0.15, bitorder="little")
            so = fresh_ord()
            self.osegs.append(OracleSegment(lists, lengths, segment_ord=so, writer_cls=T.FieldWriter, alive=alive))
            self.msegs.append(M.Segment(so, lists, lengths, alive=alive))
        self.osegs[0].terms[6] = (0, 0, 0)  # absent from some segments
        self.osegs[1].terms[3] = (0, 0, 0)
        self.osegs[2].terms[1] = (0, 0, 0)
        self.osegs[2].terms[23] = (0, 0, 0)
        self._counts, self._rows = {}, {}

    def register(self, ctx):
        for s in self.osegs:
            s.register(ctx)
        return ctx

    def query(self, op, terms, k, **extra):
        q = make_query(op, self.osegs, terms, k)
        q.update(extra)
        return q, list(terms)

    @staticmethod
    def _key(q, terms, doc_ranges):
        return repr((q["op"], terms, q["weights"], q.get("term_occur"), q.get("term_group"), q.get("min_should_match"), q["term_segs"],
                     doc_ranges))

    def rows(self, qt, doc_ranges=None):
        """The model's rows, computed once per shape at k = 1000 without a threshold, then cut as the query asks."""
        q, terms = qt
        key = self._key(q, terms, doc_ranges)
        if key not in self._rows:
            self._rows[key] = M.search(self.msegs, dict(q, k=1000, threshold=None), terms, doc_ranges=doc_ranges)
        rows = self._rows[key]
        thr = q.get("threshold")
        if thr is not None:
            rows = [r for r in rows if np.float32(r[0]) > np.float32(thr)]
        return rows[:q["k"]]

    def count(self, qt, doc_ranges=None):
        q, terms = qt
        key = self._key(q, terms, doc_ranges)
        if key not in self._counts:
            self._counts[key] = M.count(self.msegs, q, terms, doc_ranges=doc_ranges)
        return self._counts[key]


@pytest.fixture(scope="module")
def fx():
    return Fixture()


def _plain_queries(fx):
    qs = [fx.query(TQ_OP_TERM, [t], k) for t in (0, 1, 3, 4, 6, 23) for k in KS]
    qs += [fx.query(TQ_OP_AND, c, k) for c in AND_SETS for k in KS]
    qs += [fx.query(TQ_OP_OR, c, k) for c in OR_SETS for k in KS]
    return qs


def _bool_queries(fx):
    out = []
    for terms, occurs, groups, msm in BOOL_SHAPES:
        for k in KS:
            q, _ = fx.query(TQ_OP_OR, terms, k)
            out.append((bool_query(q, occurs, groups, msm), list(terms)))
    return out


def _with_thresholds(fx, qs):
    """Each query again with an initial threshold at its model's k-th score (only the rows above it are collected)."""
    out = []
    for q, terms in qs:
        rows = fx.rows((q, terms))
        if rows:
            out.append((dict(q, threshold=float(rows[min(q["k"], len(rows)) - 1][0])), terms))
    return out


def _flagged(qs, which=None):
    return [dict(q, count_hits=True) if which is None or i in which else q for i, (q, _) in enumerate(qs)]


def _run(ctx, queries, twice=False):
    """prepare -> run -> fetch -> fetch_hits (twice: the prepared batch is run and fetched a second time)."""
    b = ctx.prepare(QueryBatch(queries))
    try:
        out = []
        for _ in range(2 if twice else 1):
            b.run()
            rows = b.fetch()
            out.append((rows, b.fetch_hits(), ctx.stats()))
        return out
    finally:
        b.close()


def _check(ctx, fx, qs, what, which=None, hook_env=None):
    """The batch flagged (all, or the indices in `which`): its rows == the unflagged batch's == the model's; its hits == the model's
    count == tq_count_batch for the flagged queries, 0 for the others."""
    [(rows, got, st)] = _run(ctx, _flagged(qs, which))
    plain = ctx.search_batch(QueryBatch([q for q, _ in qs]))
    counted = ctx.count_batch(QueryBatch([q for q, _ in qs]))
    for i, qt in enumerate(qs):
        assert hits(rows, i) == hits(plain, i) == fx.rows(qt), (what, i, qt[0]["op"], qt[1], qt[0]["k"])
        want = fx.count(qt) if which is None or i in which else 0
        assert int(got[i]) == want, (what, i, qt[0]["op"], qt[1], int(got[i]), want)
        if which is None or i in which:
            assert int(counted[i]) == want, (what, i)
    return st


# ---- every shape on both engines ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["tile", "legacy"])
def test_every_shape_on_both_engines(fx, engine):
    tile = engine == "tile"
    c = fx.register(_ctx_with_env(TQ_TILE=1 if tile else 0, TQ_TILE_TERMS=1))
    try:
        qs = _plain_queries(fx)
        st = _check(c, fx, qs, (engine, "plain"))
        assert (st["tile_groups"] >= 1) == tile and st["units_count_hits"] > 0 and st["count_hits_ms"] > 0, st
        _check(c, fx, _with_thresholds(fx, qs), (engine, "thresholds"))
        if tile:
            bq = _bool_queries(fx)
            _check(c, fx, bq, (engine, "bool"))
            _check(c, fx, _with_thresholds(fx, bq), (engine, "bool thresholds"))
    finally:
        c.close()


def test_flagged_unflagged_and_phrases_in_one_batch(fx):
    rng = np.random.default_rng(3)
    words = np.array(["a", "b", "c", "d"])
    ps = PosSegment([" ".join(rng.choice(words, size=int(rng.integers(1, 12)))) for _ in range(5000)])
    c = fx.register(_ctx_with_env(TQ_TILE=1))
    ps.register(c)
    try:
        qs = _plain_queries(fx)[::2] + _bool_queries(fx)[::3]
        which = set(range(0, len(qs), 3))
        phrase = phrase_query([ps], ["a", "b"], 10)[0]
        mixed = _flagged(qs, which)
        mixed.insert(5, phrase)
        [(rows, got, _)] = _run(c, mixed)
        assert int(got[5]) == 0
        plain = c.search_batch(QueryBatch(mixed))
        for j in range(len(mixed)):
            assert hits(rows, j) == hits(plain, j), j
        got = np.delete(got, 5)
        for i, qt in enumerate(qs):
            assert int(got[i]) == (fx.count(qt) if i in which else 0), (i, qt[1])
            assert hits(rows, i if i < 5 else i + 1) == fx.rows(qt), i
        # a flagged phrase is refused at prepare (Count of a phrase is not on the device path); the context stays usable
        with pytest.raises(T.TqError, match="error -1"):
            c.prepare(QueryBatch([dict(phrase, count_hits=True)]))
        _check(c, fx, qs[:12], "after the refusal")
    finally:
        c.close()


# ---- routes ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hook", TILE_PATH_HOOKS + TILE_OVERFLOW_HOOKS, ids=lambda h: ",".join(f"{k}={v}" for k, v in h.items()))
def test_tile_routes(fx, hook):
    c = fx.register(_ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, **hook))
    try:
        qs = _plain_queries(fx) + _bool_queries(fx)
        st = _check(c, fx, qs, hook)
        assert st["tile_groups"] >= 1 and st["units_count_hits"] > 0, st
        if hook in TILE_OVERFLOW_HOOKS:
            assert st["tile_fallbacks"] == 1, st
    finally:
        c.close()


@pytest.mark.parametrize("env", [dict(TQ_TILE_MAX_DENS_X1000=400), dict(TQ_TILE_SCRATCH_MB=1)], ids=["groups", "scratch"])
def test_several_groups_and_per_query_kernels_in_one_batch(fx, env):
    c = fx.register(_ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, **env))
    try:
        qs = _plain_queries(fx)
        st = _check(c, fx, qs, env)
        if "TQ_TILE_MAX_DENS_X1000" in env:
            assert st["tile_groups"] >= 2, st
        else:  # part of the batch on the tile engine, the rest on the per-query kernels (and counted by k_count)
            assert st["tile_groups"] >= 1 and st["units_or"] + st["units_and"] + st["units_term"] > 0, st
    finally:
        c.close()


def test_single_term_batch_on_k_term(fx):
    c = fx.register(_ctx_with_env(TQ_TILE=1))  # default rule: a batch of single-term queries streams through k_term
    try:
        qs = [fx.query(TQ_OP_TERM, [t], k) for t in range(N_TERMS) for k in KS]
        st = _check(c, fx, qs, "k_term", which=set(range(0, len(qs), 2)))
        assert st["tile_groups"] == 0 and st["units_term"] > 0, st
    finally:
        c.close()


def test_1025_query_batches(fx):
    rng = np.random.default_rng(1025)
    base = _plain_queries(fx) + _bool_queries(fx)
    qs = [base[int(i)] for i in rng.integers(0, len(base), size=1025)]
    c = fx.register(_ctx_with_env(TQ_TILE=1))
    try:
        _check(c, fx, qs, "1025", which=set(int(i) for i in rng.choice(1025, size=700, replace=False)))
    finally:
        c.close()


def test_sparse_offsets_beyond_the_count_tile_buffer():
    """Ten lists that each hold every doc of the first tile, every list sparse (TQ_TILE_BIG_MIN): that tile has 10 240 sparse
    offsets, more than k_count_tiles keeps; the group's queries are recounted by k_count."""
    rng = np.random.default_rng(77)
    max_doc = 300_000
    lengths = np.clip(np.round(np.exp(rng.normal(np.log(40), 0.7, size=max_doc))), 1, 4096).astype(np.uint32)
    lists = []
    for t in range(10):
        docs = np.union1d(np.arange(1024), np.nonzero(rng.random(max_doc) < 0.002)[0]).astype(np.uint32)
        lists.append((docs, np.minimum(rng.geometric(0.6, size=len(docs)), 10).astype(np.uint32)))
    alive = np.packbits(rng.random(max_doc) > 0.1, bitorder="little")
    so = fresh_ord()
    fx = Fixture.__new__(Fixture)
    fx.osegs = [OracleSegment(lists, lengths, segment_ord=so, writer_cls=T.FieldWriter, alive=alive)]
    fx.msegs = [M.Segment(so, lists, lengths, alive=alive)]
    fx._counts, fx._rows = {}, {}
    qs = [fx.query(TQ_OP_OR, list(range(10)), k) for k in KS] + [fx.query(TQ_OP_AND, [0, 1, 2], 10), fx.query(TQ_OP_TERM, [4], 10)]
    for env in (dict(TQ_TILE_BIG_MIN=100000), {}):
        c = fx.register(_ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, **env))
        try:
            _check(c, fx, qs, env)
        finally:
            c.close()


# ---- doc ranges, phases, repeated runs ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("cuts", [[0, 100_001, 10**9], [0, 1, 5000, 77_777, 10**9], [0, 0, 10**9]], ids=["halves", "thirds+", "empty"])
def test_doc_range_parts_add_up(fx, cuts):
    """One context per part of every segment (cuts inside tiles and inside bytes of the alive bitset): each part's hits are the
    model's count over its docs, and they add up to the whole."""
    qs = _plain_queries(fx)[::2] + _bool_queries(fx)[::2]
    total = np.zeros(len(qs), np.uint64)
    for a, b in zip(cuts[:-1], cuts[1:]):
        c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1)
        try:
            ranges = {}
            for s in fx.osegs:
                lo, hi = min(a, s.max_doc), min(b, s.max_doc)
                s.register(c)
                c.segment_set_doc_range(s.segment_ord, 0, lo, hi)
                ranges[s.segment_ord] = (lo, hi)
            [(rows, got, _)] = _run(c, _flagged(qs))
            for i, qt in enumerate(qs):
                assert int(got[i]) == fx.count(qt, doc_ranges=ranges), (cuts, a, i, qt[1])
                assert hits(rows, i) == fx.rows(qt, doc_ranges=ranges), (cuts, a, i)
            total += got
        finally:
            c.close()
    assert [int(x) for x in total] == [fx.count(qt) for qt in qs]


def test_phased_run_with_imported_thresholds(fx):
    torch = pytest.importorskip("torch")
    qs = _plain_queries(fx) + _bool_queries(fx)
    c = fx.register(_ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1))
    try:
        b = c.prepare(QueryBatch(_flagged(qs)))
        keys = torch.zeros(len(qs), dtype=torch.int64, device="cuda:0")
        for p in range(b.phases()):
            b.run_phase(p)
            if p < b.phases() - 1:
                b.thresholds_export_dev(keys.data_ptr())
                b.thresholds_import_dev(keys.data_ptr())
        rows, got = b.fetch(), b.fetch_hits()
        b.close()
        for i, qt in enumerate(qs):
            assert hits(rows, i) == fx.rows(qt), i
            assert int(got[i]) == fx.count(qt), (i, qt[1])
    finally:
        c.close()


def test_prepared_batch_run_twice_counts_from_zero(fx):
    qs = _plain_queries(fx) + _bool_queries(fx)
    c = fx.register(_ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1))
    try:
        (r1, h1, _), (r2, h2, _) = _run(c, _flagged(qs), twice=True)
        assert [int(x) for x in h1] == [int(x) for x in h2] == [fx.count(qt) for qt in qs]
        for i in range(len(qs)):
            assert hits(r1, i) == hits(r2, i), i
    finally:
        c.close()


def test_unflagged_batch_launches_no_count_kernel(fx):
    """A batch without the flag launches what it launched before the flag existed: the flagged batch's launches less its count
    launches (one k_count_tiles per tile group here), and no count CTA."""
    qs = _plain_queries(fx) + _bool_queries(fx)
    c = fx.register(_ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1))
    try:
        [(_, got, st0)] = _run(c, [q for q, _ in qs])
        assert st0["units_count_hits"] == 0 and st0["count_hits_ms"] == 0 and not got.any(), st0
        [(_, _, st1)] = _run(c, _flagged(qs))
        assert st1["kernel_launches"] == st0["kernel_launches"] + st1["tile_groups"], (st0, st1)
        assert {k: v for k, v in st0.items() if k.startswith("units") and k != "units_count_hits"} == \
            {k: v for k, v in st1.items() if k.startswith("units") and k != "units_count_hits"}
    finally:
        c.close()


# ---- a segment of 2^31 - 2 docs --------------------------------------------------------------------------------------------
def test_segment_of_2_to_the_31_docs():
    """H0 of test_gpu_high_doc_ids: 2^31 - 2 docs, no fieldnorms, lists with docs above 2^30 and at max_doc - 1, a dense list of
    2.6M postings, 40 000 consecutive docs (the tile run overflows and is repeated: its hits stand)."""
    from tests.test_gpu_high_doc_ids import BIG, CLUSTER, EDGE, MID, T129, TIES, WIDE, _h0
    h0 = _h0(np.random.default_rng(0x7FFFFFFE))

    def q(op, terms, k):
        return make_query(op, [h0], terms, k), list(terms)

    qs = [q(TQ_OP_TERM, [t], 10) for t in (EDGE, WIDE, BIG, CLUSTER, TIES)]
    qs += [q(TQ_OP_AND, c, 10) for c in ([EDGE, BIG], [BIG, MID], [CLUSTER, BIG], [TIES, MID, BIG])]
    qs += [q(TQ_OP_OR, c, k) for c in ([EDGE, WIDE], [BIG, MID], [CLUSTER, T129, BIG]) for k in (1, 10)]
    want = [M.count_compacted([h0.model], qq, t) for qq, t in qs]
    assert want[2] > 2_500_000 and want[3] == 40_000
    for env in (dict(TQ_TILE=1, TQ_TILE_TERMS=1), dict(TQ_TILE=1, TQ_TILE_TERMS=1, TQ_TILE_BIG_MIN=1), dict(TQ_TILE=0)):
        c = _ctx_with_env(**env)
        try:
            h0.register(c)
            [(rows, got, _)] = _run(c, _flagged(qs))
            assert [int(x) for x in got] == want, env
            assert [int(x) for x in c.count_batch(QueryBatch([qq for qq, _ in qs]))] == want, env
            plain = c.search_batch(QueryBatch([qq for qq, _ in qs]))
            for i in range(len(qs)):
                assert hits(rows, i) == hits(plain, i), (env, i)
        finally:
            c.close()
