"""Histograms with a terms sub-aggregation on the device (tq_histogram_terms_batch: k_hist_terms, k_hist_terms_final) against
tests/hist_terms_model.py (per segment each counted doc given its pos and key in doc order, the cut of terms_model per (segment,
bucket), merge_fruits in segment_ord order, the histogram finalised with each bucket's terms) over the docs tests/score_model.py
matches (and-ed with the alive bits, the filter and the doc range, as Count counts them).  Buckets, doc counts, both scalars and every
entry must be exact; the buckets equal tq_histogram_batch's, a one-bucket histogram's entries and scalars tq_terms_batch's rows, an
uncut query's (pos, key) counts tq_terms_histogram_batch's (key, pos) cells, and the hits tq_count_batch's.  The fixture is
test_gpu_terms_hist's (three segments with deletes, terms columns of every kind, a monotone timestamp, random columns with NaN and
+-inf)."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200 import hist_terms as HT  # noqa: E402
from tantivy_b200 import histogram as Hg  # noqa: E402
from tantivy_b200 import metrics as Mx  # noqa: E402
from tantivy_b200 import terms_hist as TH  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_BOOL, TQ_OP_OR, TQ_OP_TERM, QueryBatch  # noqa: E402
from tests import hist_terms_model as HTM  # noqa: E402
from tests.helpers import OracleSegment, make_query  # noqa: E402
from tests.test_gpu_hist_metrics import code  # noqa: E402
from tests.test_gpu_parity import fresh_ord  # noqa: E402
from tests.test_gpu_sort_field import ALL, FILTER_KINDS, packed, shapes  # noqa: E402
from tests.test_gpu_terms_hist import TermsHistFixture, fixture_column  # noqa: E402
from tests.test_gpu_terms_metrics import dictionaries  # noqa: E402
from tests.test_hist_metrics_host import same_tree  # noqa: E402
from tests.test_hist_terms_host import FIXTURES  # noqa: E402


def fields_of(fx, names):
    return {c: Mx.MetricField(fx.mcol[c], fx.kind[c]) for c in names}


def request(hist, terms, date=False, name="t"):
    return {"h": {"date_histogram" if date else "histogram": hist, "aggs": {name: {"terms": terms}}}}


def dev_rows(out, q):
    """{pos: (doc_count, sum_other, error, [(segment_ord, image, doc_count)])} of query q of Context.hist_terms_batch."""
    r = HT.rows_of(out, q)
    rows = {int(p): (int(d), int(o), int(e), []) for p, d, o, e in zip(r.pos, r.doc_count, r.other, r.error)}
    for b, s, k, c in zip(r.bucket.tolist(), r.seg.tolist(), r.key.tolist(), r.count.tolist()):
        rows[int(r.pos[b])][3].append((s, k, c))
    return rows


def model(fx, r, p, qt, masks=None, segs=None):
    """(rows as dev_rows gives them, final result or AggregationError)."""
    req, hreq = r.req, Hg.device_request(r.hist_req, p.hist_kind)
    lo, hi = hreq.hard_bounds if hreq.hard_bounds is not None else (-Hg.F64_MAX, Hg.F64_MAX)
    rows, results = {}, []
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
        b = HTM.segment(kv, kp, hv, hpr, sel, p.hist_kind, hreq.interval, hreq.offset or 0.0, lo, hi, mi)
        so = fx.osegs[i].segment_ord
        seg = {}
        for pos, (c, kept, e, o) in HTM.cut(b, req.segment_size, req.order_target == "_key", req.order == "asc").items():
            d0, o0, e0, ents = rows.get(pos, (0, 0, 0, []))
            rows[pos] = (d0 + c, o0 + o, e0 + e, ents + [(so, k, n) for k, n in kept])
            keys = {}
            for k, n in kept:
                if p.kind == "str" and req.missing is not None and k == mi:
                    keys[T.terms._missing_key(req.missing)] = n
            for k, n in kept:
                if not (p.kind == "str" and req.missing is not None and k == mi):
                    keys[T.terms.intermediate_key(k, p.kind, dicts[so])] = n
            seg[pos] = (c, keys, o, e)
        results.append(seg)
    rows = {pos: (d, o, e, sorted(ents, key=lambda x: (x[0], x[1]))) for pos, (d, o, e, ents) in rows.items()}
    try:
        res = HTM.final(r.name, r.hist_req, p.hist_kind, r.terms_name, req, HTM.merge(results))
    except Hg.AggregationError as e:
        res = e
    return rows, res


def check(ctxs, fx, qts, aggs, masks=None, count_hits=True):
    """Runs qts with one request over every context and compares with the model (and, with one context, the rows)."""
    r = HT.parse_request(aggs)
    fields = fields_of(fx, {r.req.field, r.hist_req.field})
    p = HT.plan(r, fields)
    qb = QueryBatch([qt[0] for qt in qts])
    missing = {s.segment_ord: fx.missing_image(r.req.field, i, p.tspec) for i, s in enumerate(fx.osegs)}
    out = HT.run(ctxs, qb, [r] * len(qts), fields, count_hits=count_hits, dictionaries=dictionaries(fx), missing_images=missing)
    res, hits = out if count_hits else (out, None)
    if count_hits:
        assert np.array_equal(hits, sum(c.count_batch(qb) for c in ctxs))
    wants = [model(fx, r, p, qt, masks) for qt in qts]
    if len(ctxs) == 1:
        dev = ctxs[0].hist_terms_batch(qb, [p.hspec] * len(qts), [p.tspec] * len(qts))
        for q, w in enumerate(wants):
            assert dev_rows(dev, q) == w[0], (aggs, qts[q][1])
    for qt, got, want in zip(qts, res, wants):
        want = want[1]
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
         ({"field": "nan_inf", "interval": 1e300, "keyed": True}, False)]


@pytest.mark.parametrize("t", range(len(TERMS)))
def test_columns_against_model(ctx, fx, t):
    """Every terms column kind (str with missing, u64, i64, f64, date, bool) under histograms of date / u64 / f64 columns, monotone
    (one-bucket tiles at 1 h) and straddling (1 min, random columns), with NaN and +-inf, bounds, keyed and date keys."""
    for h in range(len(HISTS)):
        if (h + t) % 2:
            continue
        qts = shapes(fx)[(t + h) % 4::4][:6]
        hist, date = HISTS[h]
        check([ctx], fx, qts, request(hist, TERMS[t], date))


def test_missing_equal_to_a_real_value(ctx, fx):
    """A numeric `missing` equal to a key of the column folds into that key's entry; a str `missing` is its own entry."""
    qts = shapes(fx)[:6]
    real = T.terms.intermediate_key(int(fx.columns["k_i64"][0][0][0]), "i64")[1]
    for terms in ({"field": "k_i64", "missing": real, "size": 50, "segment_size": 4}, {"field": "k_str", "missing": "NA", "size": 50}):
        check([ctx], fx, qts, request({"field": "ts", "fixed_interval": "1h"}, terms, True))


@pytest.mark.parametrize("fkind", FILTER_KINDS[::2])
def test_filters(ctx, fx, fkind):
    j = FILTER_KINDS.index(fkind)
    qts = [(dict(q, filter=200 + j), t) for q, t in shapes(fx)[:8]]
    check([ctx], fx, qts, request({"field": "ts", "fixed_interval": "1m"}, {"field": "k_str", "size": 4}, True), masks=fx.filters[fkind])


def test_ties_segment_size_and_key_orders(ctx, fx):
    """Equal counts at the cut (lowest keys kept), _count / _key asc / desc, segment_size below, at and above a bucket's entries."""
    qts = [fx.query(TQ_OP_TERM, [ALL], 10), fx.query(TQ_OP_OR, [1, 2, 3], 10), fx.query(TQ_OP_AND, [0, 1], 10)]
    for ss, size, order in ((7, 5, {"_count": "desc"}), (49, 60, {"_key": "asc"}), (50, 5, {"_key": "desc"}), (51, 60, {"_count": "asc"}),
                            (1, 1, {"_count": "asc"}), (3, 2, {"_key": "desc"})):
        for hist in ({"field": "ts", "fixed_interval": "1h"}, {"field": "ts", "fixed_interval": "1m"}):
            check([ctx], fx, qts, request(hist, {"field": "k_ties", "size": size, "segment_size": ss, "order": order}, True))


def placement(c):
    st = c.stats()
    return st["hist_terms_units_shared"], st["hist_terms_units_global"]


def test_shared_and_global_grids_tile_shortcuts_and_cuts(fx):
    """A unit window under kTermsHistSmemCells counts on chip, a wider one in the grid (for term / AND / OR queries and for boolean
    ones, which run k_hist_terms<true>); one-key, one-bucket and both tiles; rows cut on the device."""
    c = fx.register(T.Context(0))
    try:
        qts = shapes(fx)[:10]
        bools = [qt for qt in shapes(fx) if qt[0]["op"] == TQ_OP_BOOL][:4]
        assert bools
        for batch in (qts, bools):
            s0, g0 = placement(c)
            check([c], fx, batch, request({"field": "ts", "fixed_interval": "1h"}, {"field": "flag", "size": 2}, True))
            s1, g1 = placement(c)
            assert s1 > s0 and g1 == g0  # (3 columns x a unit's few hours: on chip)
            check([c], fx, batch, request({"field": "ints", "interval": 1.0}, {"field": "k_r10k", "size": 3, "segment_size": 4}))
            s2, g2 = placement(c)
            assert g2 > g1  # (10 000 keys x many buckets: the grid)
        check([c], fx, qts, request({"field": "ts", "fixed_interval": "1h"}, {"field": "clustered", "size": 20}, True))
        st = c.stats()
        assert 0 < st["hist_terms_tiles_both"] <= min(st["hist_terms_tiles_one_key"], st["hist_terms_tiles_one_bucket"])
        assert st["hist_terms_tiles_one_bucket"] < st["hist_terms_tiles_seen"] and st["hist_terms_ms"] > 0
        assert st["hist_terms_rows_cut"] > 0
    finally:
        c.close()


def test_cross_checks_with_other_device_paths(ctx, fx):
    """Buckets and doc counts equal tq_histogram_batch's; one bucket over every value gives tq_terms_batch's rows and scalars; an
    uncut query's (pos, key) counts equal tq_terms_histogram_batch's (key, pos) cells."""
    qts = shapes(fx)[:10]
    qb = QueryBatch([qt[0] for qt in qts])
    nq = len(qts)
    for hist, terms, date in (({"field": "ts", "fixed_interval": "1m"}, {"field": "k_str", "missing": "NA", "segment_size": 5}, True),
                              ({"field": "ints", "interval": 7.0, "hard_bounds": {"min": 100.0, "max": 900.0}}, {"field": "k_i64", "segment_size": 3}, False)):
        r = HT.parse_request(request(hist, terms, date))
        p = HT.plan(r, fields_of(fx, {r.req.field, r.hist_req.field}))
        dev = ctx.hist_terms_batch(qb, [p.hspec] * nq, [p.tspec] * nq)
        ref = ctx.histogram_batch(qb, [p.hspec] * nq)
        for q in range(nq):
            n = int(ref[2][q])
            assert int(dev[6][q]) == n and np.array_equal(dev[0][q, :n], ref[0][q, :n]) and np.array_equal(dev[1][q, :n], ref[1][q, :n])
    # one bucket over every value (the monotone timestamp at 1000 days): the entries and scalars are the terms rows of the docs with
    # a timestamp, which is every doc
    for terms in ({"field": "k_str", "missing": "NA", "segment_size": 5}, {"field": "k_ties", "segment_size": 7, "order": {"_key": "desc"}},
                  {"field": "k_f64", "segment_size": 4, "order": {"_count": "asc"}}):
        r = HT.parse_request(request({"field": "ts", "fixed_interval": "1000d"}, terms, True))
        p = HT.plan(r, fields_of(fx, {r.req.field, r.hist_req.field}))
        dev = ctx.hist_terms_batch(qb, [p.hspec] * nq, [p.tspec] * nq)
        ref = ctx.terms_batch(qb, [p.tspec] * nq)
        for q in range(nq):
            rows = dev_rows(dev, q)
            n = int(ref[3][q])
            if not n:
                continue
            (d, o, e, ents), = rows.values()
            assert ents == [(int(a), int(b), int(c)) for a, b, c in zip(ref[0][q, :n], ref[1][q, :n], ref[2][q, :n])]
            assert (o, e) == (int(ref[4][q]), int(ref[5][q]))
    # uncut: (pos, key) counts against tq_terms_histogram_batch's (key, pos) cells
    r = HT.parse_request(request({"field": "ts", "fixed_interval": "1m"}, {"field": "k_str", "missing": "NA", "segment_size": 100000}, True))
    p = HT.plan(r, fields_of(fx, {r.req.field, r.hist_req.field}))
    dev = ctx.hist_terms_batch(qb, [p.hspec] * nq, [p.tspec] * nq)
    th = ctx.terms_hist_batch(qb, [p.tspec] * nq, [p.hspec] * nq)
    for q in range(nq):
        a = {(pos, s, k): c for pos, (_, _, _, ents) in dev_rows(dev, q).items() for s, k, c in ents}
        b = {(pos, s, k): c for s, k, _, h in TH.rows_of(th, q)[0] for pos, c in h.items()}
        assert a == b and a


def test_split_segments_over_two_contexts(fx):
    """The big segment's halves in two contexts (doc ranges) come back uncut and are summed then cut once per bucket; equal to one
    context over all of it and to the model."""
    big = fx.osegs[0]
    half = (big.max_doc // 8192 // 2) * 8192 + 100
    ctxs = []
    try:
        for lo, hi in ((0, half), (half, big.max_doc), (0, big.max_doc)):
            c = T.Context(0)
            big.register(c)
            c.segment_set_doc_range(big.segment_ord, 0, lo, hi)
            for k in ("k_r10k", "k_ties", "ts", "dyadic"):
                v, pr = fx.columns[k][0]
                c.sort_column_register(fx.mcol[k], big.segment_ord, v, None if pr is None else packed(pr))
            ctxs.append(c)
        for aggs in (request({"field": "ts", "fixed_interval": "1h"}, {"field": "k_r10k", "size": 4, "segment_size": 30}, True),
                     request({"field": "dyadic", "interval": 1000.0}, {"field": "k_ties", "size": 5, "segment_size": 7, "order": {"_count": "asc"}})):
            r = HT.parse_request(aggs)
            fields = fields_of(fx, {r.req.field, r.hist_req.field})
            p = HT.plan(r, fields)
            for q, t in shapes(fx)[:6]:
                q = dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] == big.segment_ord])
                split = HT.run(ctxs[:2], QueryBatch([q]), [r], fields)[0]
                one = HT.run(ctxs[2:], QueryBatch([q]), [r], fields)[0]
                want = model(fx, r, p, (q, t), segs={0})[1]
                assert split == want and one == want, aggs
    finally:
        for c in ctxs:
            c.close()


def same_out(a, b):
    for q in range(len(a[6])):
        assert dev_rows(a, q) == dev_rows(b, q)
    assert np.array_equal(a[10], b[10])


def device_args(fx, qts, aggs):
    r = HT.parse_request(aggs)
    p = HT.plan(r, fields_of(fx, {r.req.field, r.hist_req.field}))
    return QueryBatch([qt[0] for qt in qts]), [p.hspec] * len(qts), [p.tspec] * len(qts)


def test_waves_budget_stride_and_errors(fx):
    qts = shapes(fx)[:12]
    qt = fx.query(TQ_OP_TERM, [ALL], 10)
    c = fx.register(T.Context(0))
    try:
        for aggs in (request({"field": "ts", "fixed_interval": "1m"}, {"field": "k_r10k", "size": 3, "segment_size": 10}, True),
                     request({"field": "ints", "interval": 10.0}, {"field": "k_str", "size": 3, "missing": "NA"})):
            args = device_args(fx, qts, aggs)
            want = c.hist_terms_batch(*args, count_hits=True)
            same_out(want, c.hist_terms_batch(*args, count_hits=True, stride=1, entry_capacity=1))
            waves = []
            for budget in (str(1 << b) for b in range(23, 9, -1)):  # fewer queries to a wave, down to a budget that refuses one
                os.environ["TQ_HIST_TERMS_BUDGET"] = budget
                try:
                    small = fx.register(T.Context(0))
                finally:
                    del os.environ["TQ_HIST_TERMS_BUDGET"]
                try:
                    got = small.hist_terms_batch(*args, count_hits=True)
                except T.TqError as e:
                    assert "exceed the device budget" in str(e)
                    break
                finally:
                    waves.append(small.stats()["hist_terms_waves"])
                    small.close()
                same_out(want, got)
                assert np.array_equal(got[11], want[11])
            assert max(waves) > 1, waves
        # a (query, segment) whose grid alone exceeds the budget: TQ_ERR_UNSUPPORTED from the call; through hist_terms.run a
        # HistTermsRefused naming that query, the others of the batch answered
        os.environ["TQ_HIST_TERMS_BUDGET"] = "5000"
        try:
            tiny = fx.register(T.Context(0))
        finally:
            del os.environ["TQ_HIST_TERMS_BUDGET"]
        try:
            wide = request({"field": "ints", "interval": 1.0}, {"field": "k_ties", "segment_size": 5})
            args = device_args(fx, [qt], wide)
            assert code(lambda: tiny.hist_terms_batch(*args)) == -4
            narrow = request({"field": "ts", "fixed_interval": "1d"}, {"field": "flag", "size": 3}, True)
            rw, rn = HT.parse_request(wide), HT.parse_request(narrow)
            fields = fields_of(fx, {"k_ties", "ints", "flag", "ts"})
            batch = [qt, qts[1], qt, qts[2]]
            res, hits = HT.run([tiny], QueryBatch([q for q, _ in batch]), [rn, rw, rw, rn], fields, count_hits=True)
            for j in (1, 2):
                assert isinstance(res[j], HT.HistTermsRefused) and "exceed the device budget" in str(res[j]) and int(hits[j]) == 0
            want_hits = tiny.count_batch(QueryBatch([q for q, _ in batch]))
            for j in (0, 3):
                assert res[j] == model(fx, rn, HT.plan(rn, fields), batch[j])[1] and int(hits[j]) == int(want_hits[j])
        finally:
            tiny.close()
        qb, hs, ts = device_args(fx, [qt], request({"field": "ints", "interval": 1.0}, {"field": "k_ties"}))
        assert code(lambda: c.hist_terms_batch(qb, hs, [ts[0][:1] + (2,) + ts[0][2:]])) == -1  # TQ_TERMS_BY_METRIC
        assert code(lambda: c.hist_terms_batch(qb, hs, [ts[0][:2] + (7,) + ts[0][3:]])) == -1  # order
        assert code(lambda: c.hist_terms_batch(qb, [hs[0][:2] + (0.0,) + hs[0][3:]], ts)) == -1  # interval
        assert code(lambda: c.hist_terms_batch(qb, hs, [(999,) + ts[0][1:]])) == -3
        assert code(lambda: c.hist_terms_batch(qb, [(999,) + hs[0][1:]], ts)) == -3
        phrase = dict(qt[0], op=3, term_pos=[(0, 0)] * len(qt[0]["term_segs"]), term_offset=[0])
        assert code(lambda: c.hist_terms_batch(QueryBatch([phrase]), hs, ts)) == -4
        empty = c.hist_terms_batch(QueryBatch([]), [], [], count_hits=True)
        assert [x.shape[0] for x in empty] == [0] * 12
    finally:
        c.close()


FIXTURE_CASES = [c for c in FIXTURES if "segments" in c and "refused" not in c]


@pytest.mark.parametrize("case", FIXTURE_CASES, ids=[c["name"] for c in FIXTURE_CASES])
def test_reference_fixtures_on_device(case):
    """The reference's vectors end to end: every fixture segment a real segment whose term 0 lists its matching docs, every field a
    registered column (a str field as ordinals of the segment's sorted terms), the rows finalised by tantivy_b200.hist_terms."""
    fields = {name: Mx.MetricField(i + 1, kind) for i, (name, kind) in enumerate(sorted(case["fields"].items()))}
    r = HT.parse_request(case["aggs"])
    c = T.Context(0)
    try:
        segs, dicts, missing = [], {}, {}
        for docs in case["segments"]:
            n = len(docs)
            hit = np.array([i for i, d in enumerate(docs) if d["hit"]], np.uint32)
            if not len(hit):
                continue
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
        q = make_query(TQ_OP_TERM, segs, [0], 10)
        res, hits = HT.run([c], QueryBatch([q]), [r], fields, count_hits=True,
                           dictionaries={so: d.get(r.req.field) for so, d in dicts.items()}, missing_images=missing)
        assert int(hits[0]) == sum(bool(d["hit"]) for docs in case["segments"] for d in docs)
        assert same_tree(res[0], case["expected"]), (case["name"], res[0])
    finally:
        c.close()


def test_segment_of_2_to_the_31_docs():
    """One segment of 2^31 - 2 docs whose three lists, terms column (50 keys, 10 % of the docs without one) and date column (one doc
    per second, 10 % without a value) live in its top 300 000 docs and at max_doc - 1.  Term, OR and AND queries at 1 h and 1 min,
    cut and uncut, with a missing key and with binding hard bounds: rows equal the model, hits tq_count_batch's."""
    rng = np.random.default_rng(0x231)
    max_doc = 2**31 - 2
    top = max_doc - 300_000
    lists = []
    for pr in (0.2, 0.05, 0.01):
        d = np.union1d(top + np.nonzero(rng.random(max_doc - top) < pr)[0], [max_doc - 1]).astype(np.uint32)
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
            r = HT.parse_request(request(hist, terms, True))
            p = HT.plan(r, fields)
            out = c.hist_terms_batch(qb, [p.hspec] * len(qs), [p.tspec] * len(qs), count_hits=True)
            assert np.array_equal(out[11], counts)
            hreq = Hg.device_request(r.hist_req, "date")
            lo, hi = hreq.hard_bounds if hreq.hard_bounds is not None else (-Hg.F64_MAX, Hg.F64_MAX)
            for i, (_, docs) in enumerate(qs):
                sel = np.zeros(max_doc - top, bool)
                sel[docs.astype(np.int64) - top] = True
                mi = p.tspec[5] if r.req.missing is not None else None
                b = HTM.segment(top_keys, key_has, top_ts, ts_has, sel, "date", hreq.interval, 0.0, lo, hi, mi)
                cut = HTM.cut(b, r.req.segment_size, r.req.order_target == "_key", r.req.order == "asc")
                want = {pos: (d, o, e, [(seg.segment_ord, k, n) for k, n in kept]) for pos, (d, kept, e, o) in cut.items()}
                assert dev_rows(out, i) == want and want, (terms, hist, i)
    finally:
        c.close()
