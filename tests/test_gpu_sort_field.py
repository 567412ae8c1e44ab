"""TopDocs::order_by_fast_field on the device (tq_sort_batch: k_sort + k_sort_final) against a numpy model.  The model takes the
docs tests/score_model.py matches (what M.count counts: and-ed with the alive bits, the filter and the doc range), keys each by its
column value and sorts by the reference's order: docs with a value first, by value (Desc: larger first; Asc: smaller first), then
the docs without one; ties by (segment, doc) ascending (compare_for_top_k, top_score_collector.rs:591-600; order.rs:286-293).
Rows are compared exactly: values, present, segment, doc, count and hits.

Fixtures: three segments (deletes in two, the third without), one of 2 * 65536 + 1003 docs (three units of eight 8192-doc tiles,
11 docs in its last 32-doc word), terms absent from some segments, an `edge` term on the first and last doc of every 8192-doc tile
and unit and on max_doc - 1, an `all` term on every doc.  Columns: uniform u64 over the full range (0 and 2^64 - 1 included),
monotone in doc id, all equal, few distinct values, half absent, all absent, i64 with negatives and f64 with +-0.0 through the
mapping."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200._abi import TQ_MAX_K, TQ_OP_AND, TQ_OP_BOOL, TQ_OP_OR, TQ_OP_TERM, QueryBatch  # noqa: E402
from tests import score_model as M  # noqa: E402
from tests.helpers import BOOL_SHAPES, OracleSegment, bool_query, make_query, random_bool_shapes, shape_query  # noqa: E402
from tests.test_gpu_parity import fresh_ord  # noqa: E402

N_TERMS = 12
DENS = (0.3, 0.1, 0.05, 0.01, 0.002, 0.2)
EDGE, ALL = N_TERMS, N_TERMS + 1
SIZES = (2 * 65536 + 1003, 70_001, 45_000)
KS = (1, 10, 1000)
ORDERS = ("desc", "asc")
AND_SETS = [[0, 1], [1, 3], [0, 2, 4], [5, 0, 1, 2], [6, 7, 8, 9, 11]]
OR_SETS = [[0, 4], [3, 9], [1, 2, 3], [0, 6, 10, 4, 8], list(range(N_TERMS)) + [EDGE, ALL] + list(range(6))]
COLUMN_KINDS = ("uniform", "monotone", "equal", "few", "half", "none", "i64", "f64")
COL = {k: 100 + i for i, k in enumerate(COLUMN_KINDS)}
FILTER_KINDS = ("ones", "zeros", "bern1", "bern30", "run", "edges", "deleted")


def packed(mask):
    return np.packbits(np.asarray(mask, bool), bitorder="little")


def unpacked(bits, n):
    return np.unpackbits(np.asarray(bits, np.uint8), bitorder="little", count=n).astype(bool)


def edge_docs(max_doc):
    docs = {0, max_doc - 1}
    for e in range(8192, max_doc, 8192):
        docs.update((e - 1, e))
    return np.array(sorted(docs), np.uint32)


def column(kind, max_doc, seg_i, rng):
    """(u64 images, present mask or None) of one segment's column."""
    present = None
    if kind == "uniform":
        v = rng.integers(0, 2**64 - 1, size=max_doc, dtype=np.uint64, endpoint=True)
        v[:4] = [0, 2**64 - 1, 0, 2**64 - 1]
    elif kind == "monotone":  # a timestamp: docs appended in time order, segments after one another
        v = (np.uint64(1_600_000_000_000) + np.uint64(seg_i) * np.uint64(10**9) + np.arange(max_doc, dtype=np.uint64) * np.uint64(1000))
    elif kind == "equal":
        v = np.full(max_doc, 7, np.uint64)
    elif kind == "few":
        v = rng.integers(0, 4, size=max_doc).astype(np.uint64)
    elif kind == "half":
        v = rng.integers(0, 1000, size=max_doc).astype(np.uint64)
        present = rng.random(max_doc) < 0.5
    elif kind == "none":
        v = np.zeros(max_doc, np.uint64)
        present = np.zeros(max_doc, bool)
    elif kind == "i64":
        v = T.fast_value_to_u64(rng.integers(-50, 50, size=max_doc), "i64")
    else:
        f = rng.choice(np.array([-0.0, 0.0, -1.5, 2.25, np.inf, -np.inf, 3.0]), size=max_doc)
        v = T.fast_value_to_u64(f, "f64")
    return v, present


class Fixture:
    def __init__(self, seed=0x50F7):
        rng = np.random.default_rng(seed)
        self.osegs, self.models, self.alive = [], [], []
        for i, max_doc in enumerate(SIZES):
            lengths = np.clip(np.round(np.exp(rng.normal(np.log(40), 0.7, size=max_doc))), 1, 4096).astype(np.uint32)
            lists = []
            for t in range(N_TERMS):
                docs = np.nonzero(rng.random(max_doc) < DENS[t % len(DENS)])[0].astype(np.uint32)
                lists.append((docs, np.minimum(rng.geometric(0.6, size=len(docs)), 10).astype(np.uint32)))
            e = edge_docs(max_doc)
            lists.append((e, np.ones(len(e), np.uint32)))
            lists.append((np.arange(max_doc, dtype=np.uint32), np.ones(max_doc, np.uint32)))
            alive_mask = rng.random(max_doc) > 0.15
            alive_mask[edge_docs(max_doc)[::2]] = True
            alive = None if i == 2 else packed(alive_mask)
            self.osegs.append(OracleSegment(lists, lengths, segment_ord=fresh_ord(), writer_cls=T.FieldWriter, alive=alive))
            self.alive.append(np.ones(max_doc, bool) if alive is None else alive_mask)
            self.models.append(M.Segment(self.osegs[-1].segment_ord, lists, lengths))
        for s, t in ((0, 6), (1, 3), (2, 1), (2, 11)):  # absent from some segments
            self.osegs[s].terms[t] = (0, 0, 0)
        self.columns = {k: [column(k, s.max_doc, i, rng) for i, s in enumerate(self.osegs)] for k in COLUMN_KINDS}
        self.filters = {}
        for k in FILTER_KINDS:
            masks = []
            for i, s in enumerate(self.osegs):
                m = np.zeros(s.max_doc, bool)
                if k == "ones":
                    m[:] = True
                elif k == "bern1":
                    m = rng.random(s.max_doc) < 0.01
                elif k == "bern30":
                    m = rng.random(s.max_doc) < 0.3
                elif k == "run":
                    m[s.max_doc // 3:s.max_doc // 3 + s.max_doc // 7] = True
                elif k == "edges":
                    m[edge_docs(s.max_doc)] = True
                elif k == "deleted":
                    m = ~self.alive[i]
                masks.append(m)
            self.filters[k] = masks
        self._has = {}

    def register(self, ctx, kinds=COLUMN_KINDS, filters=()):
        for s in self.osegs:
            s.register(ctx)
        for k in kinds:
            self.register_column(ctx, k)
        for j, k in enumerate(filters):
            for i, s in enumerate(self.osegs):
                ctx.filter_register(200 + j, s.segment_ord, packed(self.filters[k][i]))
        return ctx

    def register_column(self, ctx, kind, col_id=None):
        for i, s in enumerate(self.osegs):
            v, p = self.columns[kind][i]
            ctx.sort_column_register(COL[kind] if col_id is None else col_id, s.segment_ord, v, None if p is None else packed(p))

    def query(self, op, terms, k, **extra):
        q = make_query(op, self.osegs, terms, k)
        q.update(extra)
        return q, list(terms)

    def has(self, i, qt):
        q, terms = qt
        key = (i, repr((q["op"], terms, q.get("term_occur"), q.get("term_group"), q.get("min_should_match"), q.get("term_flags"),
                        sorted(ts[0] for ts in q["term_segs"] if ts[1] == self.osegs[i].segment_ord))))
        if key not in self._has:
            d = M._segment_matches(self.models[i], q, terms)
            self._has[key] = np.zeros(self.osegs[i].max_doc, bool) if d is None else d.has.copy()
        return self._has[key]

    def model(self, qt, kind, order, k, masks=None, doc_ranges=None, segs=None):
        """(rows [(value image, present, segment, doc)], count) of the model."""
        vals, pres, sos, docs = [], [], [], []
        for i, s in enumerate(self.osegs):
            if segs is not None and i not in segs:
                continue
            sel = self.has(i, qt) & self.alive[i]
            if masks is not None:
                sel &= masks[i]
            if doc_ranges is not None and i in doc_ranges:
                lo, hi = doc_ranges[i]
                sel[:lo] = False
                sel[hi:] = False
            d = np.nonzero(sel)[0]
            v, p = self.columns[kind][i]
            pr = np.ones(len(d), bool) if p is None else p[d]
            vals.append(np.where(pr, v[d], np.uint64(0)))
            pres.append(pr)
            sos.append(np.full(len(d), s.segment_ord, np.int64))
            docs.append(d.astype(np.int64))
        return sort_rows(np.concatenate(vals), np.concatenate(pres), np.concatenate(sos), np.concatenate(docs), order, k)


def sort_rows(vals, pres, sos, docs, order, k):
    key = vals if order == "desc" else ~vals
    key = np.where(pres, key, np.uint64(0))
    idx = np.lexsort((docs, sos, ~key, ~pres))  # present desc, key desc, segment asc, doc asc
    rows = [(int(vals[i]), bool(pres[i]), int(sos[i]), int(docs[i])) for i in idx[:k]]
    return rows, len(vals)


def device_rows(out, q):
    values, present, segs, docs, counts = out[:5]
    return [(int(values[q, j]) if present[q, j] else 0, bool(present[q, j]), int(segs[q, j]), int(docs[q, j])) for j in range(int(counts[q]))]


@pytest.fixture(scope="module")
def fx():
    return Fixture()


@pytest.fixture(scope="module")
def ctx(fx):
    c = fx.register(T.Context(0), filters=FILTER_KINDS)
    yield c
    c.close()


def shapes(fx):
    rng = np.random.default_rng(7)
    out = [fx.query(TQ_OP_TERM, [t], 10) for t in (0, 3, 4, 6, EDGE, ALL)]
    out += [fx.query(TQ_OP_AND, s, 10) for s in AND_SETS]
    out += [fx.query(TQ_OP_OR, s, 10) for s in OR_SETS]
    for terms, occ, groups, msm in BOOL_SHAPES:
        q, _ = fx.query(TQ_OP_OR, terms, 10)
        out.append((bool_query(q, occ, groups, msm), list(terms)))
    for sh in random_bool_shapes(rng, 8, N_TERMS):
        q, _ = fx.query(TQ_OP_OR, sh["terms"], 10)
        out.append((shape_query(q, sh), list(sh["terms"])))
    return out


def run_and_check(ctx, fx, qts, kind, masks=None, count_hits=True, col=None):
    qb = QueryBatch([qt[0] for qt in qts])
    specs = [(COL[kind] if col is None else col, qt[0]["_order"]) for qt in qts]
    out = ctx.sort_batch(qb, specs, count_hits=count_hits)
    for i, qt in enumerate(qts):
        rows, n = fx.model(qt, kind, qt[0]["_order"], qt[0]["k"], masks=masks(qt) if masks else None)
        got = device_rows(out, i)
        assert got == rows, f"{kind} {qt[0]['_order']} k={qt[0]['k']} query {i} op {qt[0]['op']} {qt[1]}: {got[:5]} vs {rows[:5]}"
        if count_hits:
            assert int(out[5][i]) == n
    return out


def with_order(qts, ks=KS, orders=ORDERS):
    out = []
    for q, terms in qts:
        for k in ks:
            for o in orders:
                out.append((dict(q, k=k, _order=o), terms))
    return out


@pytest.mark.parametrize("kind", COLUMN_KINDS)
def test_shapes_against_model(ctx, fx, kind):
    """Every shape at k 1 / 10 / 1000, Desc and Asc, on one column kind; hits equal tq_count_batch."""
    qts = with_order(shapes(fx))
    out = run_and_check(ctx, fx, qts, kind)
    counts = ctx.count_batch(QueryBatch([qt[0] for qt in qts]))
    assert np.array_equal(out[5], counts)
    # without count_hits the same rows (the tiles may now be skipped)
    out2 = ctx.sort_batch(QueryBatch([qt[0] for qt in qts]), [(COL[kind], qt[0]["_order"]) for qt in qts])
    for i in range(len(qts)):
        assert device_rows(out2, i) == device_rows(out, i)


def test_edges_and_no_match(ctx, fx):
    """Matches on the first and last doc of every 8192-doc tile and unit and on max_doc - 1 (a partial 32-doc word); fewer than
    k docs with values (None rows fill the row); a query with no match."""
    qts = with_order([fx.query(TQ_OP_TERM, [EDGE], 10), fx.query(TQ_OP_AND, [EDGE, 4], 10)], ks=(1, 10, 200))
    for kind in ("half", "none", "monotone", "uniform"):
        run_and_check(ctx, fx, qts, kind)
    q = dict(fx.query(TQ_OP_TERM, [4], 10)[0], term_segs=[])
    out = ctx.sort_batch(QueryBatch([q]), [(COL["uniform"], "desc")], count_hits=True)
    assert out[4][0] == 0 and out[5][0] == 0


def test_skipping_is_exact_and_happens(fx):
    """A column ascending in doc id sorted Desc with k = 10 skips tiles and returns the model's rows; with count_hits the same
    rows, every tile visited, hits equal to tq_count_batch."""
    c = fx.register(T.Context(0), kinds=("monotone",))
    try:
        qts = with_order([fx.query(TQ_OP_TERM, [0], 10), fx.query(TQ_OP_OR, [0, 5], 10), fx.query(TQ_OP_TERM, [ALL], 10)], ks=(10,), orders=("desc",))
        s0 = c.stats()
        out = run_and_check(c, fx, qts, "monotone", count_hits=False)
        s1 = c.stats()
        assert s1["sort_tiles_skipped"] > s0["sort_tiles_skipped"]
        assert s1["sort_tiles_seen"] > s0["sort_tiles_seen"] and s1["units_sort"] > s0["units_sort"] and s1["sort_ms"] > s0["sort_ms"]
        out2 = run_and_check(c, fx, qts, "monotone", count_hits=True)
        s2 = c.stats()
        assert s2["sort_tiles_skipped"] == s1["sort_tiles_skipped"]
        for i in range(len(qts)):
            assert device_rows(out, i) == device_rows(out2, i)
        assert np.array_equal(out2[5], c.count_batch(QueryBatch([qt[0] for qt in qts])))
    finally:
        c.close()


def test_reference_vectors():
    """top_score_collector.rs test_fast_field_ascending_order (beer sizes 12 / 64 / 16 / none) and sort_key/mod.rs
    test_order_by_f64 (altitudes 149 / 27 | 40 | 0 over three segments, AllQuery as a term in every doc)."""
    c = T.Context(0)
    try:
        beer = OracleSegment([(np.arange(4, dtype=np.uint32), np.ones(4, np.uint32))], [3, 3, 3, 2], segment_ord=fresh_ord(), writer_cls=T.FieldWriter)
        beer.register(c)
        c.sort_column_register(1, beer.segment_ord, np.array([12, 64, 16, 0], np.uint64), packed([1, 1, 1, 0]))
        qb = QueryBatch([make_query(TQ_OP_TERM, [beer], [0], 4)] * 2)
        out = c.sort_batch(qb, [(1, "asc"), (1, "desc")])
        so = beer.segment_ord
        assert device_rows(out, 0) == [(12, True, so, 0), (16, True, so, 2), (64, True, so, 1), (0, False, so, 3)]
        assert device_rows(out, 1) == [(64, True, so, 1), (16, True, so, 2), (12, True, so, 0), (0, False, so, 3)]
        segs = []
        for alts in ([149.0, 27.0], [40.0], [0.0]):
            n = len(alts)
            s = OracleSegment([(np.arange(n, dtype=np.uint32), np.ones(n, np.uint32))], [1] * n, segment_ord=fresh_ord(), writer_cls=T.FieldWriter)
            s.register(c)
            c.sort_column_register(2, s.segment_ord, T.fast_value_to_u64(np.array(alts), "f64"))
            segs.append(s)
        qb = QueryBatch([make_query(TQ_OP_TERM, segs, [0], 3)] * 2)
        out = c.sort_batch(qb, [(2, "asc"), (2, "desc")])
        ids = {(segs[0].segment_ord, 0): 0, (segs[0].segment_ord, 1): 1, (segs[1].segment_ord, 0): 2, (segs[2].segment_ord, 0): 3}
        got = [[(float(T.u64_to_fast_value([v], "f64")[0]), ids[(so, d)]) for v, _, so, d in device_rows(out, q)] for q in range(2)]
        assert got[0] == [(0.0, 3), (27.0, 1), (40.0, 2)]
        assert got[1] == [(149.0, 0), (40.0, 2), (27.0, 1)]
    finally:
        c.close()


@pytest.mark.parametrize("limit,offset", [(2, 0), (2, 1), (3, 2), (10, 5), (1, 999)])
def test_offset(ctx, fx, limit, offset):
    """and_offset(o): k = limit + o, then the first o rows skipped (merge_top_k)."""
    qts = with_order([fx.query(TQ_OP_OR, [0, 3], limit + offset)], ks=(limit + offset,))
    out = run_and_check(ctx, fx, qts, "few")
    for i, qt in enumerate(qts):
        rows, _ = fx.model(qt, "few", qt[0]["_order"], limit + offset)
        assert device_rows(out, i)[offset:] == rows[offset:offset + limit]


@pytest.mark.parametrize("fkind", FILTER_KINDS)
def test_filters(ctx, fx, fkind):
    """A filtered sort equals the model over alive AND filter."""
    fid = 200 + FILTER_KINDS.index(fkind)
    base = [fx.query(TQ_OP_TERM, [0], 10), fx.query(TQ_OP_AND, [0, 5], 10), fx.query(TQ_OP_OR, [3, 4, EDGE], 10)]
    q, _ = fx.query(TQ_OP_OR, [0, 1, 4], 10)
    base.append((bool_query(q, [1, 0, 2]), [0, 1, 4]))
    qts = [(dict(q, filter=fid), t) for q, t in with_order(base)]
    for kind in ("uniform", "half", "monotone"):
        run_and_check(ctx, fx, qts, kind, masks=lambda qt: fx.filters[fkind])


def test_doc_ranges_merge(fx):
    """Two contexts, each with half of the big segment's tiles, merged on the host by the sort order, equal one context with the
    whole segment."""
    big = fx.osegs[0]
    half = (big.max_doc // 8192 // 2) * 8192
    parts = []
    for lo, hi in ((0, half), (half, big.max_doc)):
        c = T.Context(0)
        big.register(c)
        c.segment_set_doc_range(big.segment_ord, 0, lo, hi)
        c.sort_column_register(COL["few"], big.segment_ord, fx.columns["few"][0][0])
        parts.append(c)
    try:
        qts = with_order([fx.query(TQ_OP_OR, [0, 4], 10)], ks=(10, 1000))
        qts = [(dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] == big.segment_ord]), t) for q, t in qts]
        qb = QueryBatch([qt[0] for qt in qts])
        specs = [(COL["few"], qt[0]["_order"]) for qt in qts]
        outs = [c.sort_batch(qb, specs, count_hits=True) for c in parts]
        for i, qt in enumerate(qts):
            rows = [r for o in outs for r in device_rows(o, i)]
            vals = np.array([r[0] for r in rows], np.uint64)
            merged, _ = sort_rows(vals, np.array([r[1] for r in rows], bool), np.array([r[2] for r in rows]), np.array([r[3] for r in rows]),
                                  qt[0]["_order"], qt[0]["k"])
            want, n = fx.model(qt, "few", qt[0]["_order"], qt[0]["k"], segs={0})
            assert merged == want
            assert sum(int(o[5][i]) for o in outs) == n
    finally:
        for c in parts:
            c.close()


def test_registry_and_errors(fx):
    c = T.Context(0)
    try:
        s = fx.osegs[2]
        s.register(c)
        q, terms = fx.query(TQ_OP_TERM, [0], 10)
        q = dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] == s.segment_ord])
        qb = QueryBatch([q])

        def code(fn):
            with pytest.raises(T.TqError) as e:
                fn()
            return int(str(e.value).split("error ")[1].split(":")[0])

        assert code(lambda: c.sort_batch(qb, [(5, "desc")])) == -3  # missing column
        assert code(lambda: c.sort_column_register(5, 999_999, np.zeros(3, np.uint64))) == -3  # no field of the ordinal
        assert code(lambda: c.sort_column_register(5, s.segment_ord, np.zeros(s.max_doc - 1, np.uint64))) == -1
        assert code(lambda: c.sort_column_register(5, s.segment_ord, np.zeros(s.max_doc, np.uint64), np.zeros(3, np.uint8))) == -1
        assert code(lambda: c.sort_column_unregister(5)) == -3
        for k in (0, TQ_MAX_K + 1):
            assert code(lambda: c.sort_batch(QueryBatch([dict(q, k=k)]), [(5, "desc")])) == -1
        phrase = dict(q, op=3, term_pos=[(0, 0)] * len(q["term_segs"]), term_offset=[0])
        assert code(lambda: c.sort_batch(QueryBatch([phrase]), [(5, "desc")])) == -4
        # re-register replaces the column
        mask = fx.has(2, (q, terms)) & fx.alive[2]
        c.sort_column_register(5, s.segment_ord, np.arange(s.max_doc, dtype=np.uint64))
        c.sort_column_register(5, s.segment_ord, np.arange(s.max_doc, dtype=np.uint64)[::-1].copy())
        out = c.sort_batch(qb, [(5, "desc")])
        assert int(out[3][0, 0]) == int(np.nonzero(mask)[0][0])
        # unregistering the last field drops the columns; a reused ordinal does not inherit them
        c.segment_unregister(s.segment_ord, 0)
        s.register(c)
        assert code(lambda: c.sort_batch(qb, [(5, "desc")])) == -3
        assert code(lambda: c.sort_column_unregister(5)) == -3
    finally:
        c.close()


def test_unregister_during_run_is_refused(fx):
    """A sort run on another thread holds its column: unregistering or replacing it meanwhile is refused, and the run's rows
    stay the model's."""
    c = fx.register(T.Context(0), kinds=("uniform",))
    try:
        qts = with_order(shapes(fx), ks=(1000,))
        qb = QueryBatch([qt[0] for qt in qts] * 8)
        specs = [(COL["uniform"], qt[0]["_order"]) for qt in qts] * 8
        result, refused, errors = {}, [], []
        started = threading.Event()

        def run():
            started.set()
            try:
                result["out"] = c.sort_batch(qb, specs, count_hits=True)
            except Exception as e:  # noqa: BLE001
                errors.append(e)

        t = threading.Thread(target=run)
        t.start()
        started.wait()
        while t.is_alive():
            try:
                c.sort_column_register(COL["uniform"], fx.osegs[0].segment_ord, fx.columns["uniform"][0][0])
            except T.TqError as e:
                assert "still reads the column" in str(e)
                refused.append(1)
        t.join()
        assert not errors
        assert refused, "the run ended before a registration was tried"
        for i, qt in enumerate(qts):
            rows, n = fx.model(qt, "uniform", qt[0]["_order"], qt[0]["k"])
            assert device_rows(result["out"], i) == rows
        c.sort_column_unregister(COL["uniform"])
    finally:
        c.close()


def test_search_and_count_unchanged_by_sorting(fx):
    """Search and count batches before and after sort batches on one context return what a context that never sorted returns,
    stats included (apart from the sort_* fields)."""
    qts = [fx.query(TQ_OP_OR, [0, 3, 4], 10), fx.query(TQ_OP_AND, [0, 5], 100), fx.query(TQ_OP_TERM, [4], 1000)]
    qb = QueryBatch([q for q, _ in qts])
    a, b = fx.register(T.Context(0)), fx.register(T.Context(0))
    try:
        ra, ca = a.search_batch(qb), a.count_batch(qb)
        sa = a.stats()
        rb0 = b.search_batch(qb)
        b.sort_batch(QueryBatch([q for q, _ in qts]), [(COL["uniform"], "desc")] * 3, count_hits=True)
        rb, cb = b.search_batch(qb), b.count_batch(qb)
        sb = b.stats()
        for x, y, z in zip(ra, rb, rb0):
            assert np.array_equal(x, y) and np.array_equal(x, z)
        assert np.array_equal(ca, cb)
        skip = {"kernel_ms", "total_ms", "term_ms", "and_ms", "or_ms", "final_ms", "score_ms", "tile_ms", "theta_ms", "phrase_ms",
                "count_hits_ms", "lists_cached", "lists_built", "tile_counters", "tile_cycles", "sort_ms", "units_sort", "sort_tiles_seen",
                "sort_tiles_skipped"}
        assert {k: v for k, v in sa.items() if k not in skip} == {k: v for k, v in sb.items() if k not in skip}
        assert sb["units_sort"] > 0 and sa["units_sort"] == 0
    finally:
        a.close()
        b.close()
