"""Terms aggregations with a histogram sub-aggregation on the CPU side (tantivy_b200.terms_hist): parsing and every refusal, the C
ABI of tq_terms_histogram_batch as mirrored by _abi.py, the merge and single cut of a segment split over contexts, per-term gap filling
with extended_bounds / hard_bounds / min_doc_count / keyed / date keys, the whole-result bucket limit, and the reference's tests
(tests/golden/terms_hist_fixtures.json) through tests/terms_hist_model.py and through the finaliser, with device rows built here from
the docs as the device builds them."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import tantivy_b200 as T
from tantivy_b200 import _abi
from tantivy_b200 import histogram as Hg
from tantivy_b200 import metrics as Mx
from tantivy_b200 import terms_hist as TH
from tantivy_b200.histogram import AggregationError
from tantivy_b200.lib import LIB
from tests import histogram_model as HM
from tests import terms_hist_model as THM
from tests.test_hist_metrics_host import same_tree
from tests.test_histogram_host import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = json.load(open(os.path.join(ROOT, "tests", "golden", "terms_hist_fixtures.json")))["cases"]
FIELDS = {"host": Mx.MetricField(1, "str"), "lat": Mx.MetricField(2, "u64"), "v": Mx.MetricField(3, "f64"), "ok": Mx.MetricField(4, "bool"),
          "tags": Mx.MetricField(5, "u64", multi_valued=True), "json": Mx.MetricField(6, "f64", n_column_types=2), "ip": Mx.MetricField(7, "ip"),
          "ts": Mx.MetricField(8, "date"), "n": Mx.MetricField(10, "u64")}


def request(terms=None, hist=None, date=False, name="t", hname="h", extra=None):
    sub = {hname: {"date_histogram" if date else "histogram": hist or {"field": "lat", "interval": 10.0}}}
    sub.update(extra or {})
    return {name: {"terms": terms or {"field": "host"}, "aggs": sub}}


def test_parse_and_plan():
    r = TH.parse_request(request({"field": "n", "size": 3, "order": {"_key": "asc"}}, {"field": "ts", "fixed_interval": "1h", "offset": "-30m"}, True))
    assert (r.name, r.hist_name, r.is_date_histogram, r.req.size, r.hist_req.interval, r.hist_req.offset) == ("t", "h", True, 3, 3_600_000.0, -1_800_000.0)
    p = TH.plan(r, FIELDS)
    assert (p.kind, p.hist_kind) == ("u64", "date")
    assert p.tspec[:4] == (10, _abi.TQ_TERMS_BY_KEY, _abi.TQ_ORDER_ASC, 30)
    assert p.hspec[:4] == (8, "date", 3.6e12, -1.8e12)
    p = TH.plan(TH.parse_request(request({"field": "host", "missing": "NA"}, {"field": "v", "interval": 0.5, "hard_bounds": [0, 1]})), FIELDS)
    assert p.tspec[4] == _abi.TQ_TERMS_MISSING_AFTER_MAX and p.hspec[4:] == (0.0, 1.0)


@pytest.mark.parametrize("aggs,match", [
    ({"a": {"terms": {"field": "host"}}, "b": {"terms": {"field": "host"}}}, "more than one top-level"),
    ({"t": {"histogram": {"field": "lat", "interval": 1.0}}}, "not a terms aggregation"),
    ({"t": {"terms": {"field": "host"}}}, "without sub-aggregations"),
    (request(extra={"h2": {"histogram": {"field": "v", "interval": 1.0}}}), "more than one sub-aggregation"),
    ({"t": {"terms": {"field": "host"}, "aggs": {"m": {"avg": {"field": "v"}}}}}, "avg under terms is not a histogram"),
    ({"t": {"terms": {"field": "host"}, "aggs": {"r": {"range": {"field": "v", "ranges": [{"to": 1.0}]}}}}}, "range under terms"),
    ({"t": {"terms": {"field": "host"}, "aggs": {"h": {"histogram": {"field": "v", "interval": 1.0}, "aggs": {"m": {"avg": {"field": "v"}}}}}}},
     "nested under the histogram"),
    (request({"field": "host", "order": {"h": "desc"}}), "ordering by the histogram sub-aggregation"),
])
def test_parse_refusals(aggs, match):
    with pytest.raises(TH.TermsHistRefused, match=match):
        TH.parse_request(aggs)


@pytest.mark.parametrize("terms,hist,match", [
    ({"field": "host", "min_doc_count": 0}, None, "min_doc_count 0"),
    ({"field": "host", "include": "a.*"}, None, "include / exclude"),
    ({"field": "tags"}, None, "multi-valued"),
    ({"field": "json"}, None, "several columns"),
    ({"field": "ip"}, None, "ip columns"),
    ({"field": "nope"}, None, "no registered fast column"),
    ({"field": "host"}, {"field": "tags", "interval": 1.0}, "multi-valued"),
    ({"field": "host"}, {"field": "json", "interval": 1.0}, "several column types"),
    ({"field": "host"}, {"field": "host", "interval": 1.0}, "str column"),
    ({"field": "host"}, {"field": "nope", "interval": 1.0}, "no registered fast column"),
])
def test_plan_refusals(terms, hist, match):
    with pytest.raises(TH.TermsHistRefused, match=match):
        TH.plan(TH.parse_request(request(terms, hist)), FIELDS)


def test_malformed_requests():
    with pytest.raises(AggregationError, match="could not find aggregation with name nope"):
        TH.parse_request(request({"field": "host", "order": {"nope": "desc"}}))
    with pytest.raises(AggregationError, match="interval must be a positive value"):
        TH.parse_request(request(hist={"field": "lat", "interval": -1.0}))
    with pytest.raises(AggregationError, match="min_doc_count and extended_bounds"):
        TH.parse_request(request(hist={"field": "lat", "interval": 1.0, "min_doc_count": 1, "extended_bounds": [0, 5]}))
    with pytest.raises(AggregationError):
        TH.parse_request({})


def test_abi_symbols_and_layouts(tmp_path):
    for name in ("tq_terms_histogram_batch", "tq_get_terms_hist_stats"):
        assert hasattr(LIB, name)
    fields = [n for n, _ in _abi.TermsHistStats._fields_]
    assert fields == ["terms_hist_ms", "units_terms_hist", "terms_hist_tiles_seen", "terms_hist_tiles_one_key", "terms_hist_tiles_one_bucket",
                      "terms_hist_tiles_both", "terms_hist_waves", "terms_hist_units_shared", "terms_hist_units_global"]
    assert _layout(tmp_path, "tq_terms_hist_stats", fields) == [getattr(_abi.TermsHistStats, n).offset for n in fields] + [C.sizeof(_abi.TermsHistStats)]
    assert T.TermsHistRefused is TH.TermsHistRefused


# ---- rows as the device builds them --------------------------------------------------------------------------------------------
def out_of(rows_per_query):
    """A Context.terms_hist_batch output from [([(segment_ord, image, doc_count, {pos: count})], sum_other, error)] per query."""
    nq = len(rows_per_query)
    w = max(1, max(len(r[0]) for r in rows_per_query))
    segs, keys, counts = np.zeros((nq, w), np.uint32), np.zeros((nq, w), np.uint64), np.zeros((nq, w), np.uint64)
    first, ncell = np.zeros((nq, w), np.uint64), np.zeros((nq, w), np.uint32)
    pos, cc = [], []
    n, nc, other, error = np.zeros(nq, np.uint32), np.zeros(nq, np.uint32), np.zeros(nq, np.uint64), np.zeros(nq, np.uint64)
    for q, (entries, o, e) in enumerate(rows_per_query):
        for j, (s, k, c, h) in enumerate(entries):
            segs[q, j], keys[q, j], counts[q, j], first[q, j], ncell[q, j] = s, k, c, len(pos), len(h)
            for p in sorted(h):
                pos.append(p)
                cc.append(h[p])
            nc[q] += len(h)
        n[q], other[q], error[q] = len(entries), o, e
    return segs, keys, counts, n, other, error, first, ncell, np.array(pos, np.int64), np.array(cc, np.uint64), nc


def test_rows_of_round_trip():
    rows = [([(0, 3, 5, {-2: 1, 7: 4}), (1, 3, 1, {})], 2, 1), ([], 0, 0)]
    out = out_of(rows)
    assert [TH.rows_of(out, q) for q in range(2)] == rows


def test_split_segment_merged_then_cut_once():
    """A segment split over two contexts comes back uncut from each: counts and cells add by (segment, key), then one cut; a
    whole segment cut on the device is not cut again.  Cut terms take their histograms with them."""
    p = TH.plan(TH.parse_request(request({"field": "n", "size": 2, "segment_size": 2})), FIELDS)
    a = ([(0, 1, 3, {0: 3}), (0, 2, 2, {1: 2}), (0, 3, 1, {2: 1})], 0, 0)
    b = ([(0, 2, 2, {1: 1, 5: 1}), (0, 3, 2, {2: 2}), (1, 9, 4, {0: 4})], 0, 0)
    res = TH.finalize_rows(p, [TH.rows_of(out_of([a]), 0), TH.rows_of(out_of([b]), 0)])["t"]
    # segment 0 summed: 1 -> 3, 2 -> 4, 3 -> 3; cut to two (ties by key): 2 and 1 kept, 3 cut (3 docs, error 3)
    assert [(e["key"], e["doc_count"]) for e in res["buckets"]] == [(2, 4), (9, 4)]
    assert res["sum_other_doc_count"] == 3 + 3 and res["doc_count_error_upper_bound"] == 3
    assert [(x["key"], x["doc_count"]) for x in res["buckets"][0]["h"]["buckets"]] == [(10.0, 3), (20.0, 0), (30.0, 0), (40.0, 0), (50.0, 1)]


def finalize_one(terms, hist, entries, date=False, bucket_limit=Hg.DEFAULT_BUCKET_LIMIT, kind_field="n"):
    p = TH.plan(TH.parse_request(request(dict({"field": kind_field}, **terms), hist, date)), FIELDS)
    return TH.finalize(p, (entries, 0, 0), bucket_limit)["t"]


def test_gap_filling_per_term_and_bounds():
    """Gap filling spans each term's own first and last non-empty bucket; extended_bounds widen it, hard_bounds clip it; a term
    without any histogram value gets no buckets or the extended_bounds fill; min_doc_count drops; keyed maps by key string."""
    ents = {("u64", 1): (5, {1: 1, 2: 1}), ("u64", 2): (3, {4: 3}), ("u64", 3): (2, {})}
    h = {"field": "lat", "interval": 1.0}
    res = finalize_one({"order": {"_key": "asc"}}, h, ents)
    assert [[(b["key"], b["doc_count"]) for b in e["h"]["buckets"]] for e in res["buckets"]] == [[(1.0, 1), (2.0, 1)], [(4.0, 3)], []]
    assert [e["doc_count"] for e in res["buckets"]] == [5, 3, 2]  # (the terms counts, docs without a value included)
    res = finalize_one({"order": {"_key": "asc"}}, dict(h, extended_bounds={"min": 0, "max": 3}), ents)
    assert [[b["key"] for b in e["h"]["buckets"]] for e in res["buckets"]] == [[0.0, 1.0, 2.0, 3.0], [0.0, 1.0, 2.0, 3.0, 4.0], [0.0, 1.0, 2.0, 3.0]]
    res = finalize_one({"order": {"_key": "asc"}}, dict(h, hard_bounds={"min": 2, "max": 3}), {("u64", 1): (5, {2: 1}), ("u64", 2): (3, {})})
    assert [[b["key"] for b in e["h"]["buckets"]] for e in res["buckets"]] == [[2.0], []]
    res = finalize_one({"order": {"_key": "asc"}}, dict(h, min_doc_count=2), ents)
    assert [[b["key"] for b in e["h"]["buckets"]] for e in res["buckets"]] == [[], [4.0], []]
    res = finalize_one({"order": {"_key": "asc"}}, dict(h, keyed=True), ents)
    assert list(res["buckets"][0]["h"]["buckets"]) == ["1", "2"]


def test_date_keys():
    ms = 1_700_000_000_000
    pos = (ms * 10**6) // (3_600_000 * 10**6)
    res = finalize_one({}, {"field": "ts", "fixed_interval": "1h"}, {("u64", 7): (4, {pos: 3, pos + 2: 1})}, date=True)
    b = res["buckets"][0]["h"]["buckets"]
    assert [x["doc_count"] for x in b] == [3, 0, 1]
    assert b[0]["key"] == pos * 3_600_000.0 and b[0]["key_as_string"] == Hg.format_date(pos * 3_600_000 * 10**6)


def test_bucket_limit_over_the_whole_result():
    """Each kept term counts 1 plus its histogram's buckets: exactly the limit is answered, one more is the reference's error."""
    ents = {("u64", k): (10, {0: 1, 9: 1}) for k in range(5)}  # 5 terms x (1 + 10 filled buckets) = 55
    assert len(finalize_one({}, {"field": "lat", "interval": 1.0}, ents, bucket_limit=55)["buckets"]) == 5
    with pytest.raises(AggregationError, match="Limit: 54, Current: 55"):
        finalize_one({}, {"field": "lat", "interval": 1.0}, ents, bucket_limit=54)
    # (a term cut by size does not count)
    assert len(finalize_one({"size": 4}, {"field": "lat", "interval": 1.0}, ents, bucket_limit=44)["buckets"]) == 4
    # each histogram's own gap-fill check applies as well
    with pytest.raises(AggregationError, match="Limit: 5, Current: 10"):
        finalize_one({}, {"field": "lat", "interval": 1.0}, {("u64", 1): (2, {0: 1, 9: 1})}, bucket_limit=5)


def test_model_agrees_with_the_finaliser_on_random_segments():
    rng = np.random.default_rng(5)
    p = TH.plan(TH.parse_request(request({"field": "n", "size": 4, "segment_size": 6}, {"field": "v", "interval": 3.0, "hard_bounds": [-20, 20]})), FIELDS)
    results, rows = [], []
    for s in range(3):
        n = 400
        keys = rng.integers(0, 12, size=n).astype(np.uint64)
        kp = rng.random(n) < 0.9
        vals = np.asarray([T.fast_value_to_u64(x, "f64") for x in rng.normal(0, 15, size=n)], np.uint64)
        vp = rng.random(n) < 0.8
        sel = rng.random(n) < 0.7
        ents = THM.segment(keys, kp, vals, vp, sel, "f64", 3.0, 0.0, -20.0, 20.0)
        kept, e, o = THM.cut(ents, 6)
        rows.append(([(s, k, c, h) for k, (c, h) in sorted(kept.items())], o, e))
        results.append(({("u64", k): v for k, v in kept.items()}, o, e))
    want = THM.final("t", p.request.req, "h", p.request.hist_req, "f64", THM.merge(results))
    assert TH.finalize_rows(p, [rows[0], rows[1], rows[2]]) == want


# ---- the reference's tests ----------------------------------------------------------------------------------------------------
def check_asserts(case, result):
    for path, want in case["asserts"]:
        got = result
        for k in path:
            if got is None or (isinstance(k, int) and k >= len(got)) or (isinstance(k, str) and k not in got):
                got = None
                break
            got = got[k]
        assert same_tree(got, want) or (isinstance(want, int) and got == want and not isinstance(got, bool)), (case["name"], path, got, want)


def image(v, kind):
    return int(v) if kind == "u64" else int(T.fast_value_to_u64(v, kind))


def fixture_run(case):
    """(the finaliser's result over device rows built from the docs, the model's result)."""
    fields = {name: Mx.MetricField(i + 1, kind) for i, (name, kind) in enumerate(sorted(case["fields"].items()))}
    r = TH.parse_request(case["aggs"])
    p = TH.plan(r, fields)
    req, hreq = r.req, Hg.device_request(r.hist_req, p.hist_kind)
    lo, hi = hreq.hard_bounds if hreq.hard_bounds is not None else (-Hg.F64_MAX, Hg.F64_MAX)
    rows, results, dicts, missing = [], [], {}, {}
    for s, seg in enumerate(case["segments"]):
        tf, hf = req.field, r.hist_req.field
        if p.kind == "str":
            dicts[s] = sorted({d[tf] for d in seg if tf in d})
            keys = np.array([dicts[s].index(d[tf]) if tf in d else 0 for d in seg], np.uint64)
            missing[s] = len(dicts[s]) if req.missing is not None else None
        else:
            keys = np.array([image(d.get(tf, 0), p.kind) for d in seg], np.uint64)
            missing[s] = None if req.missing is None else p.tspec[5]
        kp = np.array([tf in d for d in seg])
        vals = np.array([image(d.get(hf, 0), p.hist_kind) for d in seg], np.uint64)
        vp = np.array([hf in d for d in seg])
        sel = np.array([bool(d["hit"]) for d in seg])
        ents = THM.segment(keys, kp, vals, vp, sel, p.hist_kind, hreq.interval, hreq.offset or 0.0, lo, hi, missing[s])
        kept, e, o = THM.cut(ents, req.segment_size, req.order_target == "_key", req.order == "asc")
        rows.append(([(s, k, c, h) for k, (c, h) in sorted(kept.items())], o, e))
        results.append((TH.segment_result(p, kept, dicts.get(s), missing[s]), o, e))
    got = TH.finalize_rows(p, [TH.rows_of(out_of([rw]), 0) for rw in rows], dicts, missing)
    want = THM.final(r.name, req, r.hist_name, r.hist_req, p.hist_kind, THM.merge(results))
    return got, want


SEARCHES = [c for c in FIXTURES if "segments" in c]


@pytest.mark.parametrize("case", SEARCHES, ids=[c["name"] for c in SEARCHES])
def test_reference_fixtures(case):
    if "refused" in case:
        with pytest.raises(TH.TermsHistRefused, match=case["refused"]):
            r = TH.parse_request(case["aggs"])
            TH.plan(r, {name: Mx.MetricField(i + 1, kind) for i, (name, kind) in enumerate(sorted(case["fields"].items()))})
        return
    got, want = fixture_run(case)
    assert got == want
    if "expected" in case:
        assert same_tree(got, case["expected"]), case["name"]
    else:
        check_asserts(case, got)


def test_not_applicable_fixtures_say_why():
    na = [c for c in FIXTURES if "not_applicable" in c]
    assert [c["name"] for c in na] == ["fused_term_histogram_hard_bounds_charges_term_counts"] and "memory limit" in na[0]["not_applicable"]


def test_segment_bounds_collapse_is_the_histogram_models():
    """The model's per-segment bounds are histogram_model's (normalize_histogram_req), so a non-binding hard_bounds keeps every doc."""
    vals = np.asarray([T.fast_value_to_u64(float(v), "f64") for v in range(20)], np.uint64)
    assert HM.segment_bounds(vals, None, "f64", -0.5, 19.5) == (-HM.F64_MAX, HM.F64_MAX)
    assert HM.segment_bounds(vals, None, "f64", 5.0, 14.0) == (5.0, 14.0)
