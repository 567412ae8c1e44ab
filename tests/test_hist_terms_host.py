"""Histograms with a terms sub-aggregation on the CPU side (tantivy_b200.hist_terms): parsing and every refusal, the C ABI of
tq_histogram_terms_batch as mirrored by _abi.py, the rows_of round trip, the sum and single cut of a segment split over contexts,
gap-filled and extended_bounds buckets holding the terms' empty result, date keys and keyed, the whole-result bucket limit, the
show_term_doc_count_error rule, tests/hist_terms_model.py against the finaliser on random segments, and the reference's tests
(tests/golden/hist_terms_fixtures.json) through the model and through the finaliser, with device rows built here from the docs as
the device builds them."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import tantivy_b200 as T
from tantivy_b200 import _abi
from tantivy_b200 import hist_terms as HT
from tantivy_b200 import histogram as Hg
from tantivy_b200 import metrics as Mx
from tantivy_b200 import terms as Tm
from tantivy_b200.histogram import AggregationError
from tantivy_b200.lib import LIB
from tests import hist_terms_model as HTM
from tests.test_hist_metrics_host import same_tree
from tests.test_histogram_host import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = json.load(open(os.path.join(ROOT, "tests", "golden", "hist_terms_fixtures.json")))["cases"]
FIELDS = {"host": Mx.MetricField(1, "str"), "lat": Mx.MetricField(2, "u64"), "v": Mx.MetricField(3, "f64"), "ok": Mx.MetricField(4, "bool"),
          "tags": Mx.MetricField(5, "u64", multi_valued=True), "json": Mx.MetricField(6, "f64", n_column_types=2), "ip": Mx.MetricField(7, "ip"),
          "ts": Mx.MetricField(8, "date"), "n": Mx.MetricField(10, "u64")}


def request(hist=None, terms=None, date=False, name="h", tname="t", extra=None):
    sub = {tname: {"terms": terms or {"field": "host"}}}
    sub.update(extra or {})
    return {name: {"date_histogram" if date else "histogram": hist or {"field": "lat", "interval": 10.0}, "aggs": sub}}


def test_parse_and_plan():
    r = HT.parse_request(request({"field": "ts", "fixed_interval": "1h", "offset": "-30m"}, {"field": "n", "size": 3, "order": {"_key": "asc"}}, True))
    assert (r.name, r.terms_name, r.is_date_histogram, r.req.size, r.hist_req.interval, r.hist_req.offset) == ("h", "t", True, 3, 3_600_000.0, -1_800_000.0)
    p = HT.plan(r, FIELDS)
    assert (p.kind, p.hist_kind) == ("u64", "date")
    assert p.tspec[:4] == (10, _abi.TQ_TERMS_BY_KEY, _abi.TQ_ORDER_ASC, 30)
    assert p.hspec[:4] == (8, "date", 3.6e12, -1.8e12)
    p = HT.plan(HT.parse_request(request({"field": "v", "interval": 0.5, "hard_bounds": [0, 1]}, {"field": "host", "missing": "NA"})), FIELDS)
    assert p.tspec[4] == _abi.TQ_TERMS_MISSING_AFTER_MAX and p.hspec[4:] == (0.0, 1.0)


@pytest.mark.parametrize("aggs,match", [
    ({"a": {"histogram": {"field": "lat", "interval": 1.0}}, "b": {"terms": {"field": "host"}}}, "more than one top-level"),
    ({"h": {"terms": {"field": "host"}, "aggs": {"x": {"histogram": {"field": "lat", "interval": 1.0}}}}}, "top-level terms is not a histogram"),
    ({"h": {"range": {"field": "lat", "ranges": [{"to": 1.0}]}, "aggs": {"t": {"terms": {"field": "host"}}}}}, "under a range"),
    ({"h": {"histogram": {"field": "lat", "interval": 1.0}}}, "without sub-aggregations"),
    (request(extra={"m": {"avg": {"field": "v"}}}), "more than one sub-aggregation under the histogram"),
    ({"h": {"histogram": {"field": "lat", "interval": 1.0}, "aggs": {"m": {"avg": {"field": "v"}}}}}, "metric sub-aggregation.*hist_metrics"),
    ({"h": {"histogram": {"field": "lat", "interval": 1.0}, "aggs": {"x": {"histogram": {"field": "v", "interval": 1.0}}}}},
     "histogram under the histogram is not a terms"),
    ({"h": {"histogram": {"field": "lat", "interval": 1.0}, "aggs": {"t": {"terms": {"field": "host"}, "aggs": {"m": {"avg": {"field": "v"}}}}}}},
     "nested under the terms"),
])
def test_parse_refusals(aggs, match):
    with pytest.raises(HT.HistTermsRefused, match=match):
        HT.parse_request(aggs)


@pytest.mark.parametrize("aggs,match", [
    ({}, "non-empty map"),
    ({"h": {"histogram": {"field": "lat", "interval": 1.0}, "aggs": [1]}}, "not a map"),
    ({"h": {"histogram": {"field": "lat", "interval": 1.0}, "terms": {}}}, "exactly one type"),
    (request(terms={"field": "host", "order": {"m": "desc"}}), "could not find aggregation with name m"),
    (request({"field": "lat", "interval": 0.0}), "interval must be a positive value"),
    (request({"field": "ts", "fixed_interval": "1x"}, date=True), "Unit not recognized"),
    (request(terms={"field": "host", "bogus": 1}), "unknown terms parameter"),
])
def test_malformed_requests(aggs, match):
    with pytest.raises(AggregationError, match=match):
        HT.parse_request(aggs)


@pytest.mark.parametrize("hist,terms,match", [
    (None, {"field": "host", "min_doc_count": 0}, "min_doc_count 0"),
    (None, {"field": "host", "include": "a.*"}, "include / exclude"),
    (None, {"field": "tags"}, "multi-valued"),
    (None, {"field": "json"}, "several columns"),
    (None, {"field": "ip"}, "ip columns"),
    (None, {"field": "nope"}, "no registered fast column"),
    ({"field": "tags", "interval": 1.0}, None, "multi-valued"),
    ({"field": "json", "interval": 1.0}, None, "several column types"),
    ({"field": "host", "interval": 1.0}, None, "str column"),
    ({"field": "nope", "interval": 1.0}, None, "no registered fast column"),
])
def test_plan_refusals(hist, terms, match):
    with pytest.raises(HT.HistTermsRefused, match=match):
        HT.plan(HT.parse_request(request(hist, terms)), FIELDS)


def test_abi_symbol_and_layouts(tmp_path):
    assert hasattr(LIB, "tq_histogram_terms_batch") and hasattr(LIB, "tq_get_hist_terms_stats")
    names = [n for n, _ in _abi.HistTermsStats._fields_]
    got = _layout(tmp_path, "tq_hist_terms_stats", names)
    assert got[:-1] == [getattr(_abi.HistTermsStats, n).offset for n in names] and got[-1] == C.sizeof(_abi.HistTermsStats)


def fake_out(rows_per_query, stride=8):
    """Context.hist_terms_batch's output tuple from [[(pos, doc_count, other, error, [(segment_ord, image, count)])]] per query."""
    nq = len(rows_per_query)
    pos = np.zeros((nq, stride), np.int64)
    docs, other, error, first = (np.zeros((nq, stride), np.uint64) for _ in range(4))
    nent, n, ne = np.zeros((nq, stride), np.uint32), np.zeros(nq, np.uint32), np.zeros(nq, np.uint32)
    eseg, ekey, ecount = [], [], []
    for q, rows in enumerate(rows_per_query):
        n[q] = len(rows)
        for j, (p, d, o, e, ents) in enumerate(rows):
            pos[q, j], docs[q, j], other[q, j], error[q, j], first[q, j], nent[q, j] = p, d, o, e, len(eseg), len(ents)
            for s, k, c in ents:
                eseg.append(s), ekey.append(k), ecount.append(c)
            ne[q] += len(ents)
    return (pos, docs, other, error, first, nent, n, np.array(eseg, np.uint32), np.array(ekey, np.uint64), np.array(ecount, np.uint64), ne)


def test_rows_of_round_trip():
    rows = [[(-3, 5, 1, 2, [(0, 7, 3), (1, 2, 1)]), (4, 2, 0, 0, [])], [], [(0, 1, 0, 0, [(2, 9, 1)])]]
    out = fake_out(rows)
    for q, want in enumerate(rows):
        r = HT.rows_of(out, q)
        got = [(int(p), int(d), int(o), int(e), [(int(s), int(k), int(c)) for b, s, k, c in zip(r.bucket, r.seg, r.key, r.count) if b == j])
               for j, (p, d, o, e) in enumerate(zip(r.pos, r.doc_count, r.other, r.error))]
        assert got == want


def plan_for(hist=None, terms=None, date=False, fields=None):
    return HT.plan(HT.parse_request(request(hist, terms, date)), fields or FIELDS)


def test_split_segment_summed_then_cut_once():
    """A segment evaluated in two parts comes back uncut from each; the finaliser sums its entries per (segment, bucket) and cuts
    once: equal to the cut of the whole segment."""
    p = plan_for(terms={"field": "lat", "size": 2, "segment_size": 2})
    a = HT.rows_of(fake_out([[(0, 6, 0, 0, [(0, 1, 3), (0, 2, 2), (0, 3, 1)])]]), 0)
    b = HT.rows_of(fake_out([[(0, 4, 0, 0, [(0, 2, 2), (0, 3, 2)])]]), 0)
    whole = HT.rows_of(fake_out([[(0, 10, 3, 3, [(0, 2, 4), (0, 1, 3)][::-1])]]), 0)
    got = HT.finalize_rows(p, [a, b])
    assert got == HT.finalize_rows(p, [whole])
    (bucket,) = got["h"]["buckets"]
    assert bucket["doc_count"] == 10 and bucket["t"] == {"buckets": [{"key": 2, "doc_count": 4}, {"key": 1, "doc_count": 3}],
                                                          "sum_other_doc_count": 3, "doc_count_error_upper_bound": 3}


def test_gap_filled_and_extended_buckets_hold_the_empty_terms():
    p = plan_for({"field": "lat", "interval": 10.0, "extended_bounds": {"min": -10.0, "max": 40.0}}, {"field": "lat", "size": 3})
    r = HT.rows_of(fake_out([[(0, 2, 0, 0, [(0, 1, 2)]), (2, 1, 0, 0, [(0, 25, 1)])]]), 0)
    got = HT.finalize_rows(p, [r])["h"]["buckets"]
    empty = {"buckets": [], "sum_other_doc_count": 0, "doc_count_error_upper_bound": 0}
    assert [b["key"] for b in got] == [-10.0, 0.0, 10.0, 20.0, 30.0, 40.0]
    assert [b["t"] for b in got if b["doc_count"] == 0] == [empty] * 4
    assert got[1]["t"]["buckets"] == [{"key": 1, "doc_count": 2}]


def test_date_keys_keyed_and_show_term_doc_count_error():
    p = plan_for({"field": "ts", "fixed_interval": "1h", "keyed": True}, {"field": "host", "order": {"_key": "asc"}}, True)
    r = HT.rows_of(fake_out([[(0, 3, 0, 0, [(0, 0, 2), (0, 1, 1)])]]), 0)
    got = HT.finalize_rows(p, [r], dictionaries={0: ["a", "b"]})["h"]["buckets"]
    (k, b), = got.items()
    assert k == "0" and b["key_as_string"] == "1970-01-01T00:00:00Z" and b["key"] == 0.0
    assert b["t"] == {"buckets": [{"key": "a", "doc_count": 2}, {"key": "b", "doc_count": 1}], "sum_other_doc_count": 0}
    p = plan_for(terms={"field": "host", "show_term_doc_count_error": True, "order": {"_key": "asc"}})
    assert "doc_count_error_upper_bound" in HT.finalize_rows(p, [r], dictionaries={0: ["a", "b"]})["h"]["buckets"][0]["t"]


def test_bucket_limit_over_the_whole_result():
    """Each histogram bucket counts 1 plus its kept terms (get_bucket_count)."""
    p = plan_for(terms={"field": "lat", "size": 10})
    r = HT.rows_of(fake_out([[(0, 3, 0, 0, [(0, 1, 1), (0, 2, 1), (0, 3, 1)]), (1, 1, 0, 0, [(0, 1, 1)])]]), 0)
    assert len(HT.finalize_rows(p, [r], bucket_limit=6)["h"]["buckets"]) == 2
    with pytest.raises(AggregationError, match="Limit: 5, Current: 6"):
        HT.finalize_rows(p, [r], bucket_limit=5)


def device_rows(p, segments, segment_size=None):
    """Rows of one query as the device builds them from [(segment_ord, key images, key present, hist images, hist present,
    selected)]: HTM.segment then the per-(segment, bucket) cut, buckets summed over segments."""
    req, hreq = p.request.req, Hg.device_request(p.request.hist_req, p.hist_kind)
    lo, hi = hreq.hard_bounds if hreq.hard_bounds is not None else (-Hg.F64_MAX, Hg.F64_MAX)
    rows = {}
    for so, kv, kp, hv, hp, sel, mi in segments:
        b = HTM.segment(kv, kp, hv, hp, sel, p.hist_kind, hreq.interval, hreq.offset or 0.0, lo, hi, mi)
        ss = req.segment_size if segment_size is None else segment_size
        for pos, (d, kept, e, o) in HTM.cut(b, ss, req.order_target == "_key", req.order == "asc").items():
            d0, o0, e0, ents = rows.get(pos, (0, 0, 0, []))
            rows[pos] = (d0 + d, o0 + o, e0 + e, ents + [(so, k, n) for k, n in kept])
    return HT.rows_of(fake_out([[(pos,) + rows[pos] for pos in sorted(rows)]], stride=max(1, len(rows))), 0)


@pytest.mark.parametrize("seed", range(6))
def test_model_agrees_with_finaliser_on_random_segments(seed):
    rng = np.random.default_rng(seed)
    terms = [{"field": "lat", "size": 3, "segment_size": 4}, {"field": "n", "size": 5, "order": {"_key": "desc"}, "segment_size": 3, "missing": 2},
             {"field": "n", "size": 2, "order": {"_count": "asc"}, "segment_size": 2}][seed % 3]
    hist = [{"field": "v", "interval": 0.25}, {"field": "lat", "interval": 3.0, "min_doc_count": 2}, {"field": "v", "interval": 0.5, "hard_bounds": [0.2, 0.8]}][seed % 3]
    p = plan_for(hist, terms)
    r = p.request
    segs, results = [], []
    for so in range(3):
        n = int(rng.integers(20, 80))
        kv = rng.integers(0, 8, n).astype(np.uint64)
        kp = rng.random(n) < 0.85
        hk = p.hist_kind
        hv = T.fast_value_to_u64(rng.random(n), "f64") if hk == "f64" else rng.integers(0, 30, n).astype(np.uint64)
        hp = rng.random(n) < 0.9
        sel = rng.random(n) < 0.7
        mi = p.tspec[5] if r.req.missing is not None else None
        segs.append((so, kv, kp, hv, hp, sel, mi))
        hreq = Hg.device_request(r.hist_req, hk)
        lo, hi = hreq.hard_bounds if hreq.hard_bounds is not None else (-Hg.F64_MAX, Hg.F64_MAX)
        b = HTM.segment(kv, kp, hv, hp, sel, hk, hreq.interval, hreq.offset or 0.0, lo, hi, mi)
        seg = {}
        for pos, (d, kept, e, o) in HTM.cut(b, r.req.segment_size, r.req.order_target == "_key", r.req.order == "asc").items():
            seg[pos] = (d, {Tm.intermediate_key(k, p.kind): c for k, c in kept}, o, e)
        results.append(seg)
    want = HTM.final(r.name, r.hist_req, p.hist_kind, r.terms_name, r.req, HTM.merge(results))
    assert HT.finalize_rows(p, [device_rows(p, segs)]) == want
    # the same segments split in two contexts, uncut, summed and cut once by the finaliser
    halves = [device_rows(p, [(so, kv[:len(kv) // 2], kp[:len(kv) // 2], hv[:len(kv) // 2], hp[:len(kv) // 2], sel[:len(kv) // 2], mi)
                                for so, kv, kp, hv, hp, sel, mi in segs], segment_size=10**6),
              device_rows(p, [(so, kv[len(kv) // 2:], kp[len(kv) // 2:], hv[len(kv) // 2:], hp[len(kv) // 2:], sel[len(kv) // 2:], mi)
                                for so, kv, kp, hv, hp, sel, mi in segs], segment_size=10**6)]
    # (a split segment's halves bin against each half's own bounds collapse; without hard bounds that is the same)
    if r.hist_req.hard_bounds is None:
        assert HT.finalize_rows(p, halves) == want


def fixture_rows(case, p):
    """A fixture's device rows, built here from its docs: str keys as ordinals of each segment's sorted terms."""
    segs, dicts = [], {}
    for so, docs in enumerate(case["segments"]):
        f, h = p.request.req.field, p.request.hist_req.field
        kinds = case["fields"]
        dicts[so] = sorted({d[f] for d in docs if f in d}) if kinds[f] == "str" else None
        kv = np.array([dicts[so].index(d[f]) if kinds[f] == "str" and f in d else int(d.get(f, 0)) for d in docs], np.uint64)
        kp = np.array([f in d for d in docs])
        hv = np.array([int(T.fast_value_to_u64(np.array([d.get(h, 0)], np.int64 if kinds[h] != "f64" else np.float64), kinds[h])[0])
                       if kinds[h] != "u64" else int(d.get(h, 0)) for d in docs], np.uint64)
        hp = np.array([h in d for d in docs])
        sel = np.array([bool(d["hit"]) for d in docs])
        segs.append((so, kv, kp, hv, hp, sel, None))
    return device_rows(p, segs), dicts


@pytest.mark.parametrize("case", FIXTURES, ids=[c["name"] for c in FIXTURES])
def test_reference_fixtures(case):
    if "refused" in case:
        with pytest.raises(HT.HistTermsRefused, match=case["refused"]):
            HT.parse_request(case["aggs"])
        return
    fields = {name: Mx.MetricField(i + 1, kind) for i, (name, kind) in enumerate(sorted(case["fields"].items()))}
    p = HT.plan(HT.parse_request(case["aggs"]), fields)
    rows, dicts = fixture_rows(case, p)
    assert same_tree(HT.finalize_rows(p, [rows], dictionaries=dicts), case["expected"]), case["name"]
