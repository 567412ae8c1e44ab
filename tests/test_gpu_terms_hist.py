"""Terms aggregations with a histogram sub-aggregation on the device (tq_terms_histogram_batch: k_terms, k_terms_select, k_terms_mark,
k_terms_hist, k_terms_hist_final) against tests/terms_hist_model.py (per segment each counted doc given its key and pos in doc order,
the cut of terms_model, merge_fruits in segment_ord order, each term's histogram finalised on its own) over the docs
tests/score_model.py matches (and-ed with the alive bits, the filter and the doc range, as Count counts them).  Rows, keys, doc counts,
both scalars and every cell must be exact, the rows and scalars equal to tq_terms_batch's, and for an uncut query without bounds the
cells summed over the entries equal to tq_histogram_batch's buckets.  The fixture is test_gpu_terms_metrics' (three segments with
deletes, terms columns of every kind) with a monotone timestamp column (one-bucket tiles at 1 h, straddling at 1 min) besides its
random columns (NaN and +-inf among them)."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200 import histogram as Hg  # noqa: E402
from tantivy_b200 import metrics as Mx  # noqa: E402
from tantivy_b200 import terms_hist as TH  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_BOOL, TQ_OP_OR, TQ_OP_TERM, QueryBatch  # noqa: E402
from tests import terms_hist_model as THM  # noqa: E402
from tests.test_gpu_hist_metrics import code  # noqa: E402
from tests.test_gpu_sort_field import ALL, FILTER_KINDS, packed, shapes  # noqa: E402
from tests.test_gpu_terms_metrics import TermsMetricsFixture, dictionaries  # noqa: E402
from tests.helpers import OracleSegment, make_query  # noqa: E402
from tests.test_gpu_parity import fresh_ord  # noqa: E402
from tests.test_hist_metrics_host import same_tree  # noqa: E402
from tests.test_terms_hist_host import FIXTURES, check_asserts  # noqa: E402


class TermsHistFixture(TermsMetricsFixture):
    def __init__(self):
        super().__init__()
        for i, s in enumerate(self.osegs):
            doc = np.arange(s.max_doc, dtype=np.int64)
            # a monotone timestamp, 0.1 s per doc: a tile spans under 14 minutes
            self.columns.setdefault("ts", []).append((T.fast_value_to_u64(np.int64(1_700_000_000) * 10**9 + doc * 10**8 + i * 10**12, "date"), None))
            self.kind["ts"] = "date"
        self.mcol = {k: 500 + i for i, k in enumerate(self.columns)}


def fields_of(fx, names):
    return {c: Mx.MetricField(fx.mcol[c], fx.kind[c]) for c in names}


def request(terms, hist, date=False, name="h"):
    return {"t": {"terms": terms, "aggs": {name: {"date_histogram" if date else "histogram": hist}}}}


def model(fx, r, p, qt, masks=None, segs=None):
    """(rows [(segment_ord, image, doc_count, {pos: count})], sum_other, error, final result or AggregationError)."""
    req, hreq = r.req, Hg.device_request(r.hist_req, p.hist_kind)
    lo, hi = hreq.hard_bounds if hreq.hard_bounds is not None else (-Hg.F64_MAX, Hg.F64_MAX)
    rows, other, error, results = [], 0, 0, []
    dicts = dictionaries(fx)
    for i in sorted(range(len(fx.osegs)), key=lambda i: fx.osegs[i].segment_ord):
        if segs is not None and i not in segs:
            continue
        sel = fx.has(i, qt) & fx.alive[i]
        if masks is not None:
            sel = sel & masks[i]
        kv, kp = fx.columns[req.field][i]
        hv, hpr = fx.columns[r.hist_req.field][i]
        mi = fx.missing_image(req.field, i, p.tspec)
        entries = THM.segment(kv, kp, hv, hpr, sel, p.hist_kind, hreq.interval, hreq.offset or 0.0, lo, hi, mi)
        kept, e, o = THM.cut(entries, req.segment_size, req.order_target == "_key", req.order == "asc")
        so = fx.osegs[i].segment_ord
        rows += [(so, k, c, h) for k, (c, h) in sorted(kept.items())]
        other, error = other + o, error + e
        seg = {}
        for k in sorted(kept):
            if p.kind == "str" and req.missing is not None and k == mi:
                seg[T.terms._missing_key(req.missing)] = kept[k]
        for k in sorted(kept):
            if not (p.kind == "str" and req.missing is not None and k == mi):
                seg[T.terms.intermediate_key(k, p.kind, dicts[so])] = kept[k]
        results.append((seg, o, e))
    try:
        res = THM.final(r.name, req, r.hist_name, r.hist_req, p.hist_kind, THM.merge(results))
    except Hg.AggregationError as e:
        res = e
    return rows, other, error, res


def check(ctxs, fx, qts, aggs, masks=None, count_hits=True):
    """Runs qts with one request over every context and compares with the model (and, with one context, the rows with
    tq_terms_batch's)."""
    r = TH.parse_request(aggs)
    fields = fields_of(fx, {r.req.field, r.hist_req.field})
    p = TH.plan(r, fields)
    qb = QueryBatch([qt[0] for qt in qts])
    missing = {s.segment_ord: fx.missing_image(r.req.field, i, p.tspec) for i, s in enumerate(fx.osegs)}
    out = TH.run(ctxs, qb, [r] * len(qts), fields, count_hits=count_hits, dictionaries=dictionaries(fx), missing_images=missing)
    res, hits = out if count_hits else (out, None)
    if count_hits:
        assert np.array_equal(hits, sum(c.count_batch(qb) for c in ctxs))
    wants = [model(fx, r, p, qt, masks) for qt in qts]
    if len(ctxs) == 1:
        dev = ctxs[0].terms_hist_batch(qb, [p.tspec] * len(qts), [p.hspec] * len(qts))
        ref = ctxs[0].terms_batch(qb, [p.tspec] * len(qts))
        for q, w in enumerate(wants):
            rows = TH.rows_of(dev, q)
            assert rows[0] == w[0], (aggs, qts[q][1])
            assert rows[1:] == (w[1], w[2]), (aggs, qts[q][1])
            n = int(ref[3][q])
            assert n == int(dev[3][q]) and all(np.array_equal(a[q, :n], b[q, :n]) for a, b in zip(ref[:3], dev[:3]))
            assert (int(ref[4][q]), int(ref[5][q])) == rows[1:]
    for qt, got, want in zip(qts, res, wants):
        want = want[3]
        if isinstance(want, Hg.AggregationError):
            assert isinstance(got, Hg.AggregationError) and str(got) == str(want), (aggs, qt[1])
        else:
            assert got == want, (aggs, qt[1])
    return res


@pytest.fixture(scope="module")
def fx():
    return TermsHistFixture()


@pytest.fixture(scope="module")
def ctx(fx):
    c = fx.register(T.Context(0), filters=FILTER_KINDS)
    yield c
    c.close()


TERMS = [{"field": "k_str", "missing": "NA", "size": 5, "segment_size": 8},
         {"field": "partial", "size": 4, "segment_size": 12, "order": {"_key": "desc"}},
         {"field": "k_i64", "size": 6, "order": {"_count": "asc"}},
         {"field": "k_f64", "size": 3, "order": {"_key": "asc"}},
         {"field": "k_date", "size": 5, "segment_size": 10},
         {"field": "flag", "missing": 1, "size": 2},
         {"field": "k_ties", "size": 5, "segment_size": 7},
         {"field": "k_r10k", "size": 5, "segment_size": 30}]
HISTS = [({"field": "ts", "fixed_interval": "1h"}, True),
         ({"field": "ts", "fixed_interval": "1m", "min_doc_count": 1}, True),
         ({"field": "ints", "interval": 50.0, "offset": 3.0}, False),
         ({"field": "mixed", "interval": 100000.0, "hard_bounds": {"min": -300000.0, "max": 250000.0}}, False),
         ({"field": "dyadic", "interval": 4096.0, "extended_bounds": {"min": -10000.0, "max": 10000.0}}, False),
         ({"field": "nan_inf", "interval": 1e300, "keyed": True}, False),
         ({"field": "ns", "fixed_interval": "1d", "keyed": True}, True),
         ({"field": "clustered", "interval": 1.0}, False)]


@pytest.mark.parametrize("t", range(len(TERMS)))
def test_columns_against_model(ctx, fx, t):
    """Every terms column kind (str with missing, u64, i64, f64, date, bool) under histograms of u64 / i64 / f64 / date columns,
    monotone (one-bucket tiles) and random (straddling tiles), with NaN and +-inf, bounds, keyed and date keys."""
    for h in range(len(HISTS)):
        if (h + t) % 2:
            continue
        qts = shapes(fx)[(t + h) % 4::4][:6]
        hist, date = HISTS[h]
        check([ctx], fx, qts, request(TERMS[t], hist, date))


@pytest.mark.parametrize("fkind", FILTER_KINDS[::2])
def test_filters(ctx, fx, fkind):
    j = FILTER_KINDS.index(fkind)
    qts = [(dict(q, filter=200 + j), t) for q, t in shapes(fx)[:8]]
    check([ctx], fx, qts, request({"field": "k_str", "size": 4}, {"field": "ts", "fixed_interval": "1m"}, True), masks=fx.filters[fkind])


def placement(c):
    st = c.stats()
    return st["terms_hist_units_shared"], st["terms_hist_units_global"]


def test_shared_and_global_grids_and_tile_shortcuts(fx):
    """A unit window under kTermsHistSmemCells counts on chip, a wider one in the grid (both counted, for term / AND / OR queries and
    for boolean ones, which run k_terms_hist<true>); one-key, one-bucket and both tiles."""
    c = fx.register(T.Context(0))
    try:
        qts = shapes(fx)[:10]
        bools = [qt for qt in shapes(fx) if qt[0]["op"] == TQ_OP_BOOL][:4]
        assert bools
        for batch in (qts, bools):
            s0, g0 = placement(c)
            check([c], fx, batch, request({"field": "k_str", "size": 20, "segment_size": 25}, {"field": "ts", "fixed_interval": "1h"}, True))
            s1, g1 = placement(c)
            assert s1 > s0 and g1 == g0  # (20 kept slots x a unit's few hours: on chip)
            check([c], fx, batch, request({"field": "k_r10k", "size": 20, "segment_size": 400}, {"field": "ints", "interval": 1.0}))
            s2, g2 = placement(c)
            assert g2 > g1  # (400 kept slots x up to 1000 buckets: the grid)
        check([c], fx, qts, request({"field": "clustered", "size": 20}, {"field": "ts", "fixed_interval": "1h"}, True))
        st = c.stats()
        assert 0 < st["terms_hist_tiles_both"] <= min(st["terms_hist_tiles_one_key"], st["terms_hist_tiles_one_bucket"])
        assert st["terms_hist_tiles_one_bucket"] < st["terms_hist_tiles_seen"] and st["terms_hist_ms"] > 0
    finally:
        c.close()


def test_uncut_cells_sum_to_histogram_batch(ctx, fx):
    """segment_size above every entry count and no bounds: the cells summed over the entries are tq_histogram_batch's buckets."""
    qts = shapes(fx)[:10]
    for terms, hist, date in (({"field": "k_str", "segment_size": 100, "missing": "NA"}, {"field": "ts", "fixed_interval": "1m"}, True),
                              ({"field": "k_i64", "segment_size": 100}, {"field": "ints", "interval": 7.0}, False)):
        r = TH.parse_request(request(terms, hist, date))
        p = TH.plan(r, fields_of(fx, {r.req.field, r.hist_req.field}))
        qb = QueryBatch([qt[0] for qt in qts])
        dev = ctx.terms_hist_batch(qb, [p.tspec] * len(qts), [p.hspec] * len(qts))
        ref = ctx.histogram_batch(qb, [p.hspec] * len(qts))
        for q in range(len(qts)):
            tot = {}
            for _, _, _, h in TH.rows_of(dev, q)[0]:
                for pos, n in h.items():
                    tot[pos] = tot.get(pos, 0) + n
            n = int(ref[2][q])
            assert n and tot == {int(a): int(b) for a, b in zip(ref[0][q, :n], ref[1][q, :n])}


def test_split_segments_over_two_contexts(fx):
    """The big segment's halves in two contexts (doc ranges) come back uncut with their cells and are cut once; equal to one context
    over all of it and to the model."""
    big = fx.osegs[0]
    half = (big.max_doc // 8192 // 2) * 8192 + 100
    ctxs = []
    try:
        for lo, hi in ((0, half), (half, big.max_doc), (0, big.max_doc)):
            c = T.Context(0)
            big.register(c)
            c.segment_set_doc_range(big.segment_ord, 0, lo, hi)
            for k in ("k_r10k", "k_ties", "ts", "dyadic"):
                v, p = fx.columns[k][0]
                c.sort_column_register(fx.mcol[k], big.segment_ord, v, None if p is None else packed(p))
            ctxs.append(c)
        for aggs in (request({"field": "k_r10k", "size": 4, "segment_size": 30}, {"field": "ts", "fixed_interval": "1m"}, True),
                     request({"field": "k_ties", "size": 5, "segment_size": 7, "order": {"_count": "asc"}}, {"field": "dyadic", "interval": 1000.0})):
            r = TH.parse_request(aggs)
            fields = fields_of(fx, {r.req.field, r.hist_req.field})
            p = TH.plan(r, fields)
            for q, t in shapes(fx)[:6]:
                q = dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] == big.segment_ord])
                split = TH.run(ctxs[:2], QueryBatch([q]), [r], fields)[0]
                one = TH.run(ctxs[2:], QueryBatch([q]), [r], fields)[0]
                want = model(fx, r, p, (q, t), segs={0})[3]
                assert split == want and one == want, aggs
    finally:
        for c in ctxs:
            c.close()


def same_out(a, b):
    for q in range(len(a[3])):
        assert TH.rows_of(a, q) == TH.rows_of(b, q)
    assert np.array_equal(a[10], b[10])


def device_args(fx, qts, aggs):
    r = TH.parse_request(aggs)
    p = TH.plan(r, fields_of(fx, {r.req.field, r.hist_req.field}))
    return QueryBatch([qt[0] for qt in qts]), [p.tspec] * len(qts), [p.hspec] * len(qts)


def test_waves_budget_stride_and_errors(fx):
    qts = shapes(fx)[:12]
    qt = fx.query(TQ_OP_TERM, [ALL], 10)
    c = fx.register(T.Context(0))
    try:
        for aggs in (request({"field": "k_r10k", "size": 3, "segment_size": 10}, {"field": "ts", "fixed_interval": "1m"}, True),
                     request({"field": "k_str", "size": 3, "missing": "NA"}, {"field": "ints", "interval": 10.0})):
            args = device_args(fx, qts, aggs)
            want = c.terms_hist_batch(*args, count_hits=True)
            same_out(want, c.terms_hist_batch(*args, count_hits=True, stride=1, cell_capacity=1))
            for env, budget in (("TQ_TERMS_COUNTER_BUDGET", "50"), ("TQ_TERMS_HIST_BUDGET", "20000")):
                os.environ[env] = budget  # queries alone or a few to a wave
                try:
                    small = fx.register(T.Context(0))
                finally:
                    del os.environ[env]
                try:
                    got = small.terms_hist_batch(*args, count_hits=True)
                    same_out(want, got)
                    assert np.array_equal(got[11], want[11]) and small.stats()["terms_hist_waves"] > 1
                finally:
                    small.close()
        # a (query, segment) whose grid alone exceeds the budget: TQ_ERR_UNSUPPORTED from the call; through terms_hist.run a
        # TermsHistRefused naming that query, the others of the batch answered
        os.environ["TQ_TERMS_HIST_BUDGET"] = "64"
        try:
            tiny = fx.register(T.Context(0))
        finally:
            del os.environ["TQ_TERMS_HIST_BUDGET"]
        try:
            wide = request({"field": "k_ties", "segment_size": 5}, {"field": "ints", "interval": 1.0})
            args = device_args(fx, [qt], wide)
            assert code(lambda: tiny.terms_hist_batch(*args)) == -4
            narrow = request({"field": "flag", "size": 3}, {"field": "ts", "fixed_interval": "1d"}, True)
            rw, rn = TH.parse_request(wide), TH.parse_request(narrow)
            fields = fields_of(fx, {"k_ties", "ints", "flag", "ts"})
            batch = [qt, qts[1], qt, qts[2]]
            res, hits = TH.run([tiny], QueryBatch([q for q, _ in batch]), [rn, rw, rw, rn], fields, count_hits=True)
            for j in (1, 2):
                assert isinstance(res[j], TH.TermsHistRefused) and "exceed the device budget" in str(res[j]) and int(hits[j]) == 0
            want_hits = tiny.count_batch(QueryBatch([q for q, _ in batch]))
            for j in (0, 3):
                assert res[j] == model(fx, rn, TH.plan(rn, fields), batch[j])[3] and int(hits[j]) == int(want_hits[j])
        finally:
            tiny.close()
        qb, ts, hs = device_args(fx, [qt], request({"field": "k_ties"}, {"field": "ints", "interval": 1.0}))
        assert code(lambda: c.terms_hist_batch(qb, [ts[0][:1] + (2,) + ts[0][2:]], hs)) == -1  # TQ_TERMS_BY_METRIC
        assert code(lambda: c.terms_hist_batch(qb, ts, [hs[0][:2] + (0.0,) + hs[0][3:]])) == -1
        assert code(lambda: c.terms_hist_batch(qb, [(999,) + ts[0][1:]], hs)) == -3
        assert code(lambda: c.terms_hist_batch(qb, ts, [(999,) + hs[0][1:]])) == -3
        phrase = dict(qt[0], op=3, term_pos=[(0, 0)] * len(qt[0]["term_segs"]), term_offset=[0])
        assert code(lambda: c.terms_hist_batch(QueryBatch([phrase]), ts, hs)) == -4
        empty = c.terms_hist_batch(QueryBatch([]), [], [], count_hits=True)
        assert [x.shape[0] for x in empty] == [0] * 12
    finally:
        c.close()


def test_ties_and_key_orders(ctx, fx):
    """Equal counts at the segment cut (lowest keys kept), _key asc / desc, segment_size at and around the 50 keys."""
    qts = [fx.query(TQ_OP_TERM, [ALL], 10), fx.query(TQ_OP_OR, [1, 2, 3], 10), fx.query(TQ_OP_AND, [0, 1], 10)]
    for ss, size, order in ((7, 5, {"_count": "desc"}), (49, 60, {"_key": "asc"}), (50, 5, {"_key": "desc"}), (51, 60, {"_count": "asc"})):
        check([ctx], fx, qts, request({"field": "k_ties", "size": size, "segment_size": ss, "order": order},
                                      {"field": "ts", "fixed_interval": "1h"}, True))


# ---- the reference's tests, and a segment of 2^31 - 2 docs --------------------------------------------------------------------
FIXTURE_CASES = [c for c in FIXTURES if "segments" in c and "refused" not in c]


def fixture_column(kind, docs, field, dictionary=None):
    present = np.array([field in d for d in docs], bool)
    if kind == "str":
        images = np.array([dictionary.index(d[field]) if field in d else 0 for d in docs], np.uint64)
    else:
        vals = np.array([d.get(field, 0) for d in docs], np.float64 if kind == "f64" else np.int64)
        images = T.fast_value_to_u64(vals.astype(np.uint64) if kind == "u64" else vals, kind)
    return images, present


@pytest.mark.parametrize("case", FIXTURE_CASES, ids=[c["name"] for c in FIXTURE_CASES])
def test_reference_fixtures_on_device(case):
    """The reference's vectors end to end: every fixture segment with a matching doc a real segment whose term 0 lists them, every
    field a registered column (a str field as ordinals of the segment's sorted terms), the rows finalised by
    tantivy_b200.terms_hist."""
    fields = {name: Mx.MetricField(i + 1, kind) for i, (name, kind) in enumerate(sorted(case["fields"].items()))}
    r = TH.parse_request(case["aggs"])
    c = T.Context(0)
    try:
        segs, dicts, missing = [], {}, {}
        for docs in case["segments"]:
            n = len(docs)
            hit = np.array([i for i, d in enumerate(docs) if d["hit"]], np.uint32)
            if not len(hit):
                continue  # (a segment without a matching doc adds nothing; a term needs at least one posting)
            s = OracleSegment([(hit, np.ones(len(hit), np.uint32))], [1] * n, segment_ord=fresh_ord(), writer_cls=T.FieldWriter)
            s.register(c)
            for name, f in fields.items():
                kind = case["fields"][name]
                if kind == "str":
                    dicts.setdefault(s.segment_ord, {})[name] = sorted({d[name] for d in docs if name in d})
                images, present = fixture_column(kind, docs, name, dicts.get(s.segment_ord, {}).get(name))
                c.sort_column_register(f.column_id, s.segment_ord, images, None if present.all() else packed(present))
            if fields[r.req.field].kind == "str":
                missing[s.segment_ord] = len(dicts[s.segment_ord][r.req.field])
            segs.append(s)
        q = make_query(TQ_OP_TERM, segs, [0], 10)  # (term 0: the docs the fixture's query matches)
        res, hits = TH.run([c], QueryBatch([q]), [r], fields, count_hits=True,
                           dictionaries={so: d.get(r.req.field) for so, d in dicts.items()}, missing_images=missing)
        assert int(hits[0]) == sum(bool(d["hit"]) for docs in case["segments"] for d in docs)
        if "expected" in case:
            assert same_tree(res[0], case["expected"]), case["name"]
        else:
            check_asserts(case, res[0])
    finally:
        c.close()


def test_segment_of_2_to_the_31_docs():
    """One segment of 2^31 - 2 docs whose three lists, terms column (50 keys and a missing key, 10 % of the docs without one) and
    date column (one doc per second, 10 % without a value) live in its top 300 000 docs and at max_doc - 1.  Term, OR and AND
    queries, cut and uncut, at 1 h (on chip) and 1 min (the grid) and with binding hard bounds: rows, scalars and cells equal the
    model, hits tq_count_batch's.  (The columns' values below the top are zero pages of 16 GiB arrays, never written.)"""
    rng = np.random.default_rng(0x231)
    max_doc = 2**31 - 2
    top = max_doc - 300_000
    lists = []
    for p in (0.2, 0.05, 0.01):
        d = np.union1d(top + np.nonzero(rng.random(max_doc - top) < p)[0], [max_doc - 1]).astype(np.uint32)
        lists.append((d, np.ones(len(d), np.uint32)))
    seg = OracleSegment(lists, None, segment_ord=fresh_ord(), writer_cls=T.FieldWriter, max_doc=max_doc)
    t0 = 1_700_000_000 * 10**9
    top_keys = rng.integers(0, 50, size=max_doc - top).astype(np.uint64)
    top_ts = T.fast_value_to_u64(t0 + np.arange(max_doc - top, dtype=np.int64) * 10**9, "date")
    key_has, ts_has = rng.random(max_doc - top) < 0.9, rng.random(max_doc - top) < 0.9
    key_has[-1] = ts_has[-1] = True

    def present_bits(has):
        bits = np.zeros((max_doc + 7) // 8, np.uint8)
        sel = top + np.nonzero(has)[0]
        np.bitwise_or.at(bits, sel >> 3, (1 << (sel & 7)).astype(np.uint8))
        return bits

    fields = {"k": Mx.MetricField(1, "u64"), "ts": Mx.MetricField(2, "date")}
    c = T.Context(0)
    try:
        seg.register(c)
        for col, top_values, has in ((1, top_keys, key_has), (2, top_ts, ts_has)):
            values = np.zeros(max_doc, np.uint64)
            values[top:] = top_values
            c.sort_column_register(col, seg.segment_ord, values, present_bits(has))
            del values
        qs = [(make_query(TQ_OP_TERM, [seg], [0], 10), lists[0][0]),
              (make_query(TQ_OP_OR, [seg], [0, 1, 2], 10), np.union1d(np.union1d(lists[0][0], lists[1][0]), lists[2][0])),
              (make_query(TQ_OP_AND, [seg], [0, 1], 10), np.intersect1d(lists[0][0], lists[1][0]))]
        qb = QueryBatch([q for q, _ in qs])
        counts = c.count_batch(qb)
        for terms, hist in (({"field": "k", "size": 10, "segment_size": 20, "missing": 7}, {"field": "ts", "fixed_interval": "1h"}),
                            ({"field": "k", "size": 60, "segment_size": 100}, {"field": "ts", "fixed_interval": "1m"}),
                            ({"field": "k", "size": 5, "segment_size": 12, "order": {"_key": "asc"}},
                             {"field": "ts", "fixed_interval": "1m", "hard_bounds": {"min": (t0 + 10**13) // 10**6, "max": (t0 + 2 * 10**14) // 10**6}})):
            r = TH.parse_request(request(terms, hist, True))
            p = TH.plan(r, fields)
            out = c.terms_hist_batch(qb, [p.tspec] * len(qs), [p.hspec] * len(qs), count_hits=True)
            assert np.array_equal(out[11], counts)
            hreq = Hg.device_request(r.hist_req, "date")
            lo, hi = hreq.hard_bounds if hreq.hard_bounds is not None else (-Hg.F64_MAX, Hg.F64_MAX)
            for i, (_, docs) in enumerate(qs):
                sel = np.zeros(max_doc - top, bool)
                sel[docs.astype(np.int64) - top] = True
                mi = p.tspec[5] if r.req.missing is not None else None
                ents = THM.segment(top_keys, key_has, top_ts, ts_has, sel, "date", hreq.interval, 0.0, lo, hi, mi)
                kept, e, o = THM.cut(ents, r.req.segment_size, r.req.order_target == "_key", r.req.order == "asc")
                want = ([(seg.segment_ord, k, n, h) for k, (n, h) in sorted(kept.items())], o, e)
                assert TH.rows_of(out, i) == want and want[0] and any(h for *_, h in want[0]), (terms, hist, i)
        st = c.stats()
        assert st["terms_hist_units_shared"] > 0 and st["terms_hist_units_global"] > 0
    finally:
        c.close()
