"""Queries whose clauses span several fields of one segment (tests/multi_field.py: BODY / TITLE / TAGS / RAW of a 300 000-doc
ordinal, a 70 001-doc ordinal with deletes and terms missing from some fields, an ordinal with TITLE alone) against the score
model, bit for bit (doc ids, segment ordinals, f32 scores) and Count exactly.  A clause reads its own field's postings,
fieldnorms and record option, so a (query, segment) pair reads several fieldnorm arrays: the per-query union kernels take each
posting's fieldnorm from its own list, and one list may appear under two weights or two average fieldnorms in a batch.

Routes: both engines, every tile hook and overflow repeat, the per-query kernels under the smallest and odd unit cuts (k_or and
k_or_strip both run), tq_count_batch and TQ_QUERY_COUNT_HITS, a filter on the ordinals, doc-range parts on every field alike, the
phased threshold exchange and CrossGpuMerger's key exchange, MultiContext with default placement and split registration.  Then
the life cycle of one field of a multi-field ordinal, and the rules for fields that disagree: a tile group keeps one entry per
(ordinal, field) so a field's doc range is its own, a query whose fields differ in doc range is refused, and MultiContext keeps
an ordinal's fields on one device."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_OR, TQ_OP_PHRASE, TQ_OP_TERM, QueryBatch  # noqa: E402
from tantivy_b200.sharding import CrossGpuMerger, doc_range  # noqa: E402
from tests import score_model as M  # noqa: E402
from tests.helpers import OracleSegment, hits  # noqa: E402
from tests.multi_field import BODY, RAW, TAGS, TITLE, Index, battery, expand, with_thresholds  # noqa: E402
from tests.test_gpu_parity import TILE_OVERFLOW_HOOKS, TILE_PATH_HOOKS, _ctx_with_env  # noqa: E402
from tests.test_gpu_query_kernels import HOOKS as UNIT_HOOKS  # noqa: E402
from tests.test_gpu_shard_exchange import merged_rows, run_ranks  # noqa: E402

KMAX = 1024
FID = 7


def _bits(rows):
    return [(int(np.float32(s).view(np.uint32)), g, d) for s, g, d in rows]


class Fixture:
    def __init__(self):
        self.ix = Index(writer_cls=T.FieldWriter)
        self.models = self.ix.models()
        rng = np.random.default_rng(99)
        self.filter = {o.ordinal: np.packbits(rng.random(o.max_doc) < 0.4, bitorder="little") for o in self.ix.ords}
        self.fmodels = [o.model_with(self.filter[o.ordinal] if o.alive is None else np.bitwise_and(o.alive, self.filter[o.ordinal]))
                        for o in self.ix.ords]
        self._rows, self._counts = {}, {}
        base = battery(self.ix)
        self.qts = base + with_thresholds(base, self.rows)

    def _key(self, q, t, filtered, ranges):
        return repr((q["op"], t, q["weights"], q["avg_fieldnorm"], q["term_segs"], q.get("term_flags"), q.get("term_occur"),
                     q.get("term_group"), q.get("min_should_match"), filtered, ranges))

    def rows(self, q, t, filtered=False, ranges=None):
        key = self._key(q, t, filtered, ranges)
        if key not in self._rows:
            self._rows[key] = M.search(self.fmodels if filtered else self.models, dict(q, k=KMAX, threshold=None), t, doc_ranges=ranges)
        rows = self._rows[key]
        thr = q.get("threshold")
        if thr is not None:
            rows = [r for r in rows if np.float32(r[0]) > np.float32(thr)]
        return rows[:q["k"]]

    def count(self, q, t, filtered=False, ranges=None):
        key = self._key(q, t, filtered, ranges)
        if key not in self._counts:
            self._counts[key] = M.count(self.fmodels if filtered else self.models, q, t, doc_ranges=ranges)
        return self._counts[key]


@pytest.fixture(scope="module")
def fx():
    return Fixture()


def _check(fx, ctx, qts, filtered=False, count=True):
    """Rows against the model; the Count half (TQ_QUERY_COUNT_HITS) and tq_count_batch against its counts (phrases: rows only)."""
    extra = dict(filter=FID) if filtered else {}
    qb = QueryBatch([dict(q, count_hits=count and q["op"] != TQ_OP_PHRASE, **extra) for q, _ in qts])
    b = ctx.prepare(qb)
    try:
        b.run()
        g = b.fetch()
        got_hits = b.fetch_hits()
    finally:
        b.close()
    for i, (q, t) in enumerate(qts):
        want = fx.rows(q, t, filtered)
        assert _bits(hits(g, i)) == _bits(want), (i, q["op"], t, q["k"], [ts[2] for ts in q["term_segs"]][:8], hits(g, i)[:3], want[:3])
    if count:
        counted = [(i, qt) for i, qt in enumerate(qts) if qt[0]["op"] != TQ_OP_PHRASE]
        for i, (q, t) in counted:
            assert int(got_hits[i]) == fx.count(q, t, filtered), (i, q["op"], t)
        cnt = ctx.count_batch(QueryBatch([dict(qts[i][0], **extra) for i, _ in counted]))
        for j, (i, (q, t)) in enumerate(counted):
            assert int(cnt[j]) == fx.count(q, t, filtered), (i, q["op"], t)


def _ctx(fx, filters=False, **env):
    c = _ctx_with_env(**env)
    fx.ix.register(c)
    if filters:
        for o in fx.ix.ords:
            c.filter_register(FID, o.ordinal, fx.filter[o.ordinal])
    return c


def _per_query(qts):
    return [qt for qt in qts if qt[0].get("term_occur") is None]  # TQ_OP_BOOL runs on the tile engine only


def test_fixture_reaches_its_edges(fx):
    """Cross-field sums land on one doc, the battery holds 32-clause unions, thin and thick lists of k_or_strip's rule, and body
    lists on both sides of the tile engine's dense threshold."""
    a = fx.ix.ords[0]
    n = a.max_doc
    dfs = [a.osegs[BODY].terms[t][0] for t in range(16)]
    assert any(df * 8 < n for df in dfs) and any(df * 8 >= n for df in dfs)  # k_or_strip: thin and thick
    assert any(df * 1024 >= 6 * n for df in dfs) and any(df * 1024 < 6 * n for df in dfs)  # k_tile: dense and sparse slots
    assert max(len(q["weights"]) for q, _ in fx.qts) == 32
    q, t = next(x for x in fx.qts if x[0]["op"] == TQ_OP_OR and x[0]["k"] == 1024 and x[1] == [0, 0])
    terms_of = {}
    for ts in q["term_segs"]:
        terms_of.setdefault(ts[1], set()).add(ts[2])
    assert len(terms_of[a.ordinal]) == 2
    on_a = [d for _, g, d in fx.rows(q, t) if g == a.ordinal]
    title, body = (np.isin(on_a, a.lists[f][0][0]) for f in (TITLE, BODY))
    assert (title & body).any()


@pytest.mark.parametrize("engine", ["tile", "legacy"])
def test_battery_on_both_engines(fx, engine):
    """Every shape on the tile engine (terms too) and on the per-query kernels, where k_or and k_or_strip both run."""
    if engine == "tile":
        c = _ctx(fx, TQ_TILE=1, TQ_TILE_TERMS=1)
        qts = fx.qts
    else:
        c = _ctx(fx, TQ_TILE=0)
        qts = _per_query(fx.qts)
    try:
        _check(fx, c, qts)
        st = c.stats()
        if engine == "legacy":
            assert st["units_or_strip"] > 0 and st["units_or"] > st["units_or_strip"], st
            assert st["tile_groups"] == 0
        else:
            assert st["tile_groups"] > 0 and st["tile_fallbacks"] == 0
    finally:
        c.close()


@pytest.mark.parametrize("hook", TILE_PATH_HOOKS + TILE_OVERFLOW_HOOKS, ids=lambda h: ",".join(f"{k}={v}" for k, v in h.items()))
def test_every_tile_route(fx, hook):
    c = _ctx(fx, TQ_TILE=1, **hook)
    try:
        _check(fx, c, fx.qts[::2], count=False)
        if "TQ_TILE_PCAP" in hook or "TQ_TILE_CAND_FLOOR" in hook:
            assert c.stats()["tile_fallbacks"] == 1
    finally:
        c.close()


@pytest.mark.parametrize("hook", ["smallest", "odd"])
def test_per_query_unit_cuts(fx, hook):
    """k_term, k_and, k_or_strip and k_or with one unit per block / window / tile, and with odd cuts."""
    c = _ctx(fx, TQ_TILE=0, **UNIT_HOOKS[hook])
    try:
        _check(fx, c, _per_query(fx.qts), count=False)
        st = c.stats()
        assert st["units_or_strip"] > 0 and st["units_or"] > st["units_or_strip"] and st["units_and"] > 0 and st["units_term"] > 0
    finally:
        c.close()


@pytest.mark.parametrize("engine", ["tile", "legacy"])
def test_filter_on_queries_of_different_fields(fx, engine):
    """One filter per ordinal, used by queries that name different fields (and several at once): rows and counts of the model
    over alive AND filter."""
    c = _ctx(fx, filters=True, TQ_TILE=1 if engine == "tile" else 0, TQ_TILE_TERMS=1)
    try:
        qts = fx.qts[::3] if engine == "tile" else _per_query(fx.qts[::3])
        _check(fx, c, [qt for qt in qts if qt[0]["op"] != TQ_OP_PHRASE], filtered=True)
    finally:
        c.close()


def test_doc_range_parts_merge_to_the_whole(fx):
    """Two contexts, each with one doc-range part of every ordinal set on every field alike: counts add up to the whole and the
    merged rows are the whole's."""
    qts = [qt for qt in fx.qts[::2] if qt[0]["op"] != TQ_OP_PHRASE]
    qb = QueryBatch([q for q, _ in qts])
    parts = []
    try:
        for part in range(2):
            c = _ctx_with_env(TQ_TILE=1)
            parts.append(c)
            fx.ix.register(c)
            for o in fx.ix.ords:
                for f in o.fields:
                    c.segment_set_doc_range(o.ordinal, f, *doc_range(o.max_doc, part, 2))
        res = [(c.search_batch(qb), c.count_batch(qb)) for c in parts]
        for i, (q, t) in enumerate(qts):
            assert int(res[0][1][i] + res[1][1][i]) == fx.count(q, t), i
            assert _bits(M.merge_fruits([hits(r[0], i) for r in res], q["k"])) == _bits(fx.rows(q, t)), i
    finally:
        for c in parts:
            c.close()


def _shard_queries(fx, qts, ords):
    return QueryBatch([dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] in ords],
                            **({"term_pos": [p for ts, p in zip(q["term_segs"], q["term_pos"]) if ts[1] in ords]} if "term_pos" in q else {}))
                       for q, _ in qts])


def test_phased_thresholds_and_cross_gpu_merger(fx):
    """Ordinal A on one context, B and C on another: a phased run importing the element-wise max of the thresholds, and
    CrossGpuMerger at world 2 (top-keys exchange + k_merge), give the model's rows."""
    import torch
    qts = [qt for qt in fx.qts if qt[0]["k"] in (10, 129)][::2]
    owners = [{fx.ix.ords[0].ordinal}, {o.ordinal for o in fx.ix.ords[1:]}]
    ctxs, qbs = [], []
    try:
        for r in range(2):
            c = _ctx_with_env(TQ_TILE=1)
            ctxs.append(c)
            for o in fx.ix.ords:
                if o.ordinal in owners[r]:
                    o.register(c)
            qbs.append(_shard_queries(fx, qts, owners[r]))
        bs = [ctxs[r].prepare(qbs[r]) for r in range(2)]
        keys = [torch.zeros(len(qts), dtype=torch.int64, device="cuda:0") for _ in range(2)]
        bests = []
        for p in range(bs[0].phases()):
            for r in range(2):
                bs[r].run_phase(p)
            if p + 1 < bs[0].phases():
                for r in range(2):
                    bs[r].thresholds_export_dev(keys[r].data_ptr())
                bests.append(torch.stack(keys).amax(0).contiguous())
                torch.cuda.synchronize()
                for r in range(2):
                    bs[r].thresholds_import_dev(bests[-1].data_ptr())
        rows = [bs[r].fetch() for r in range(2)]
        torch.cuda.synchronize()
        for b in bs:
            b.close()
        for i, (q, t) in enumerate(qts):
            assert _bits(M.merge_fruits([hits(rows[r], i) for r in range(2)], q["k"])) == _bits(fx.rows(q, t)), i
        got = [None, None]

        def rank(r, dist):
            b = ctxs[r].prepare(qbs[r])
            try:
                m = CrossGpuMerger(ctxs[r], dist, "cuda:0", qbs[r].nq, qbs[r].kmax)
                m.run(b)
                m(b)
                got[r] = merged_rows(m.fetch_host(b), qbs[r].nq)
            finally:
                b.close()

        run_ranks(2, rank)
        for i, (q, t) in enumerate(qts):
            for r in range(2):
                assert _bits(got[r][i]) == _bits(fx.rows(q, t)), (r, i)
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.parametrize("n_ctx", [2, 3])
@pytest.mark.parametrize("split", [False, True])
def test_multi_context(fx, n_ctx, split):
    """MultiContext over n contexts of one GPU, every field registered with the default placement (or split): the fields of an
    ordinal land together, and the merged rows are the model's (no doc twice with a partial score, ANDs across fields intact)."""
    qts = [qt for qt in fx.qts[::2] if qt[0]["op"] != TQ_OP_PHRASE and qt[0].get("term_occur") is None]
    m = T.MultiContext([0] * n_ctx)
    try:
        for o in fx.ix.ords:
            for f in o.fields:
                s = o.osegs[f]
                if split:
                    m.segment_register_split(o.ordinal, f, o.max_doc, s.record_option, s.body, s.fn_ids, o.alive)
                else:
                    m.segment_register(o.ordinal, f, o.max_doc, s.record_option, s.body, s.fn_ids, o.alive)
        g = m.search_batch(QueryBatch([q for q, _ in qts]))
        for i, (q, t) in enumerate(qts):
            assert _bits(hits(g, i)) == _bits(fx.rows(q, t)), (split, i, q["op"], t)
    finally:
        m.close()


def test_multi_context_placement_rules(fx):
    """A second field follows the first one's device; an explicit device_index that disagrees, another max_doc and a whole/split
    mix are refused."""
    a, b = fx.ix.ords[0], fx.ix.ords[1]
    m = T.MultiContext([0, 0])
    try:
        s = a.osegs[BODY]
        m.segment_register(a.ordinal, BODY, a.max_doc, s.record_option, s.body, s.fn_ids, None, device_index=1)
        s = a.osegs[TITLE]
        with pytest.raises(T.TqError, match="error -1: device_index differs"):
            m.segment_register(a.ordinal, TITLE, a.max_doc, s.record_option, s.body, s.fn_ids, None, device_index=0)
        with pytest.raises(T.TqError, match="error -1: max_doc differs"):
            m.segment_register(a.ordinal, TITLE, a.max_doc + 1, s.record_option, s.body, s.fn_ids, None)
        with pytest.raises(T.TqError, match="error -1: the ordinal's other fields are registered whole"):
            m.segment_register_split(a.ordinal, TITLE, a.max_doc, s.record_option, s.body, s.fn_ids, None)
        m.segment_register(a.ordinal, TITLE, a.max_doc, s.record_option, s.body, s.fn_ids, None)  # default: device 1
        s = b.osegs[BODY]
        m.segment_register_split(b.ordinal, BODY, b.max_doc, s.record_option, s.body, s.fn_ids, b.alive)
        s = b.osegs[TITLE]
        with pytest.raises(T.TqError, match="error -1: the ordinal's other fields are split"):
            m.segment_register(b.ordinal, TITLE, b.max_doc, s.record_option, s.body, s.fn_ids, b.alive)
        m.segment_register_split(b.ordinal, TITLE, b.max_doc, s.record_option, s.body, s.fn_ids, b.alive)
        q, t = fx.ix.query(TQ_OP_OR, expand([0, 1, 4], (BODY, TITLE)), 129)
        q2, t2 = fx.ix.query(TQ_OP_AND, [(TITLE, 1), (BODY, 0)], 129)
        ords = {a.ordinal, b.ordinal}
        qts = [(dict(x, term_segs=[ts for ts in x["term_segs"] if ts[1] in ords]), tt) for x, tt in ((q, t), (q2, t2))]
        g = m.search_batch(QueryBatch([x for x, _ in qts]))
        models = [a.model, b.model]
        for i, (x, tt) in enumerate(qts):
            assert _bits(hits(g, i)) == _bits(M.search(models, x, tt)), i
    finally:
        m.close()


def test_tile_group_entries_keep_each_fields_doc_range(fx):
    """Field TITLE of ordinal A evaluates docs [0, 5000) only, BODY the whole segment: a batch with a query on each, on both engines,
    returns each query's own range (the tile engine keeps an entry per (ordinal, field)); counts too.  A query whose clauses name
    both fields of A is refused in search and in Count."""
    a = fx.ix.ords[0]
    qb_body = fx.ix.query(TQ_OP_OR, [(BODY, 0), (BODY, 5)], 1024)
    qb_title = fx.ix.query(TQ_OP_OR, [(TITLE, 1), (TITLE, 5)], 1024)
    qts = [qb_body, qb_title, fx.ix.query(TQ_OP_TERM, [(TITLE, 0)], 129), fx.ix.query(TQ_OP_AND, [(BODY, 1), (BODY, 0)], 10)]
    ranges = [None, {a.ordinal: (0, 5000)}, {a.ordinal: (0, 5000)}, None]
    for engine in ("tile", "legacy"):
        c = _ctx_with_env(TQ_TILE=1 if engine == "tile" else 0, TQ_TILE_TERMS=1)
        try:
            fx.ix.register(c)
            c.segment_set_doc_range(a.ordinal, TITLE, 0, 5000)
            qb = QueryBatch([dict(q, count_hits=True) for q, _ in qts])
            b = c.prepare(qb)
            b.run()
            g, h = b.fetch(), b.fetch_hits()
            b.close()
            cnt = c.count_batch(qb)
            for i, ((q, t), r) in enumerate(zip(qts, ranges)):
                assert _bits(hits(g, i)) == _bits(fx.rows(q, t, ranges=r)), (engine, i)
                assert int(h[i]) == int(cnt[i]) == fx.count(q, t, ranges=r), (engine, i)
            mixed = QueryBatch([fx.ix.query(TQ_OP_OR, expand([0, 1], (BODY, TITLE)), 10)[0]])
            with pytest.raises(T.TqError, match="error -1: the clauses of a query name fields of one segment that differ"):
                c.search_batch(mixed)
            with pytest.raises(T.TqError, match="error -1: the clauses of a query name fields of one segment that differ"):
                c.count_batch(mixed)
            if engine == "tile":
                st = c.stats()
                assert st["tile_groups"] >= 1
        finally:
            c.close()


def test_field_life_cycle(fx):
    """Unregister TITLE of ordinal A and register other content under it: queries on the remaining fields are unaffected,
    lists_cached drops only that field's tables, and the ordinal's filter stays until its last field goes."""
    a = fx.ix.ords[0]
    c = _ctx(fx, filters=True, TQ_TILE=1)
    try:
        rest = [qt for qt in fx.qts if qt[0]["op"] != TQ_OP_PHRASE and all(ts[2] != TITLE for ts in qt[0]["term_segs"])][::3]
        titled = [qt for qt in fx.qts if qt[0]["op"] == TQ_OP_OR and any(ts[2] == TITLE for ts in qt[0]["term_segs"])][::3]
        _check(fx, c, rest + titled, count=False)
        title_lists = {(ts[1], ts[2], ts[4]) for q, _ in titled for ts in q["term_segs"] if ts[1] == a.ordinal and ts[2] == TITLE}
        before = c.stats()["lists_cached"]
        c.segment_unregister(a.ordinal, TITLE)
        assert c.stats()["lists_cached"] == before - len(title_lists)
        _check(fx, c, rest, count=False)
        # other content under (A, TITLE): the lists in reverse term order
        new = OracleSegment(a.lists[TITLE][::-1], a.lengths[TITLE], segment_ord=a.ordinal, field=TITLE, writer_cls=T.FieldWriter,
                            max_doc=a.max_doc)
        c.segment_register(a.ordinal, TITLE, a.max_doc, new.record_option, new.body, new.fn_ids, None)
        nt = len(a.lists[TITLE])
        q = dict(op=TQ_OP_OR, k=129, weights=[1.5, 0.7], avg_fieldnorm=[fx.ix.avg[TITLE]] * 2,
                 term_segs=[new.term_seg(nt - 1 - 1, 0), new.term_seg(nt - 1 - 4, 1)])
        want = M.search([a.model], dict(q, term_segs=[(0, a.ordinal, TITLE) + tuple(q["term_segs"][0][3:]),
                                                      (1, a.ordinal, TITLE) + tuple(q["term_segs"][1][3:])]), [1, 4])
        g = c.search_batch(QueryBatch([q, dict(q, filter=FID)]))
        assert _bits(hits(g, 0)) == _bits(want)
        assert hits(g, 1) and all(np.unpackbits(fx.filter[a.ordinal], bitorder="little")[d] for _, _, d in hits(g, 1))
        _check(fx, c, rest, count=False)
        for f in (BODY, TAGS, RAW):
            c.segment_unregister(a.ordinal, f)
        fq = QueryBatch([dict(q, filter=FID)])
        assert c.search_batch(fq)[3][0] > 0  # TITLE still holds the ordinal: its filter stays
        c.segment_unregister(a.ordinal, TITLE)
        a.osegs[TITLE].register(c)
        with pytest.raises(T.TqError, match="error -3"):
            c.search_batch(QueryBatch([dict(fx.ix.query(TQ_OP_TERM, [(TITLE, 1)], 10)[0], filter=FID)]))
    finally:
        c.close()
