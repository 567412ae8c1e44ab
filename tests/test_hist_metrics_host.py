"""Histograms with metric sub-aggregations on the CPU side (tantivy_b200.hist_metrics): parsing and every refusal, the C ABI of
tq_histogram_metrics_batch as mirrored by _abi.py, the merge of contexts by bucket, the exactness guard per (bucket, column) and the
finaliser -- against tests/hist_metrics_model.py and the reference's histogram tests with sub-aggregations, transcribed as data
(tests/golden/hist_metrics_fixtures.json).  Device parts are built here from the docs as the device builds them."""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest

import tantivy_b200 as T
from tantivy_b200 import _abi
from tantivy_b200 import hist_metrics as HMx
from tantivy_b200 import metrics as Mx
from tantivy_b200.histogram import AggregationError
from tantivy_b200.lib import LIB
from tests import hist_metrics_model as HMM
from tests import metrics_model as MM
from tests.test_histogram_host import _layout
from tests.test_metrics_host import same_json

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = json.load(open(os.path.join(ROOT, "tests", "golden", "hist_metrics_fixtures.json")))["cases"]


def request(hist=None, aggs=None, name="h", typ="date_histogram"):
    body = {typ: hist or {"field": "ts", "fixed_interval": "1h"}}
    if aggs is not None:
        body["aggs"] = aggs
    return {name: body}


FIELDS = {"ts": Mx.MetricField(1, "date"), "lat": Mx.MetricField(2, "u64"), "bytes": Mx.MetricField(3, "f64"), "ok": Mx.MetricField(4, "bool"),
          "tags": Mx.MetricField(5, "u64", multi_valued=True), "json": Mx.MetricField(6, "f64", n_column_types=2), "host": Mx.MetricField(7, "str"),
          "a": Mx.MetricField(8, "i64"), "b": Mx.MetricField(9, "i64")}


def test_parse_and_plan():
    r = HMx.parse_request(request(aggs={"avg_lat": {"avg": {"field": "lat"}}, "s": {"stats": {"field": "bytes", "missing": 0}},
                                        "n": {"value_count": {"field": "ok"}}}))
    assert r.name == "h" and r.is_date_histogram and r.req.interval == 3_600_000.0 and [m.name for m in r.metrics] == ["avg_lat", "s", "n"]
    p = HMx.plan(r, FIELDS)
    assert p.hspec == (1, "date", 3_600_000.0 * 1e6, 0.0, -Mx.F64_MAX, Mx.F64_MAX)
    assert len(p.mplan.columns) == 3 and p.mplan.columns[2][2] == T.TQ_METRIC_COUNT_ONLY
    r = HMx.parse_request({"h": {"histogram": {"field": "lat", "interval": 10, "hard_bounds": {"min": 0, "max": 100}},
                                 "aggregations": {"m": {"max": {"field": "lat"}}}}})
    assert not r.is_date_histogram and HMx.plan(r, FIELDS).hspec == (2, "u64", 10.0, 0.0, 0.0, 100.0)


@pytest.mark.parametrize("aggs,match", [
    ({"h": {"terms": {"field": "host"}, "aggs": {"m": {"avg": {"field": "lat"}}}}}, "sub-aggregations under terms"),
    ({"h": {"date_histogram": {"field": "ts", "fixed_interval": "1h"}, "aggs": {"t": {"terms": {"field": "host"}}}}}, "bucket aggregations nested"),
    ({"h": {"date_histogram": {"field": "ts", "fixed_interval": "1h"}, "aggs": {"t": {"histogram": {"field": "lat", "interval": 1}}}}}, "bucket aggregations nested"),
    ({"h": {"date_histogram": {"field": "ts", "fixed_interval": "1h"}, "aggs": {"m": {"avg": {"field": "lat"}}}},
      "x": {"avg": {"field": "lat"}}}, "more than one top-level"),
    (request(aggs={"e": {"extended_stats": {"field": "lat"}}}), "extended_stats"),
    (request(aggs={"e": {"percentiles": {"field": "lat"}}}), "percentiles"),
    (request(aggs={"e": {"cardinality": {"field": "lat"}}}), "cardinality"),
    (request(aggs={"e": {"top_hits": {"size": 1}}}), "top_hits"),
    (request(aggs={"e": {"avg": {"field": "lat"}, "aggs": {"x": {"max": {"field": "lat"}}}}}), "sub-aggregations run on the CPU path"),
    (request(), "without sub-aggregations"),
    ({"m": {"avg": {"field": "lat"}}}, "not a histogram"),
])
def test_parse_refusals(aggs, match):
    with pytest.raises(HMx.HistMetricsRefused, match=match):
        HMx.parse_request(aggs)


@pytest.mark.parametrize("hist,aggs,match", [
    ({"field": "tags", "interval": 1}, {"m": {"avg": {"field": "lat"}}}, "multi-valued"),
    ({"field": "json", "interval": 1}, {"m": {"avg": {"field": "lat"}}}, "several column types"),
    ({"field": "host", "interval": 1}, {"m": {"avg": {"field": "lat"}}}, "str column"),
    ({"field": "nope", "interval": 1}, {"m": {"avg": {"field": "lat"}}}, "no registered fast column"),
    ({"field": "lat", "interval": 1}, {"m": {"avg": {"field": "tags"}}}, "multi-valued columns"),
    ({"field": "lat", "interval": 1}, {"m": {"avg": {"field": "json"}}}, "several column types"),
    ({"field": "lat", "interval": 1}, {k: {"sum": {"field": f}} for k, f in zip("pqrst", ("lat", "bytes", "a", "b", "ts"))}, "more than 4 distinct"),
])
def test_plan_refusals(hist, aggs, match):
    r = HMx.parse_request(request(hist, aggs, typ="histogram"))
    with pytest.raises(HMx.HistMetricsRefused, match=match):
        HMx.plan(r, FIELDS)


def test_malformed_requests():
    for agg in (request({"field": "ts", "calendar_interval": "1d"}, {"m": {"avg": {"field": "lat"}}}),
                request({"field": "lat", "interval": -1}, {"m": {"avg": {"field": "lat"}}}, typ="histogram"),
                request(aggs={"m": {"avg": {}}}), request(aggs={"m": {"median": {"field": "lat"}}}), [], {}):
        with pytest.raises(AggregationError):
            HMx.parse_request(agg)


def test_abi_symbols_and_layouts(tmp_path):
    for name in ("tq_histogram_metrics_batch", "tq_get_hist_metrics_stats"):
        assert hasattr(LIB, name)
    fields = [n for n, _ in _abi.HistMetricsStats._fields_]
    assert fields == ["hist_metrics_ms", "units_hist_metrics", "hist_metrics_tiles_seen", "hist_metrics_tiles_one_bucket",
                      "hist_metrics_flush_shared", "hist_metrics_flush_global"]
    assert _layout(tmp_path, "tq_hist_metrics_stats", fields) == [getattr(_abi.HistMetricsStats, n).offset for n in fields] + [C.sizeof(_abi.HistMetricsStats)]
    assert T.HistMetricsRefused is HMx.HistMetricsRefused


# ---- parts as the device builds them ----------------------------------------------------------------------------------------
def part_of(values):
    """The tq_metric_part of a list of f64 values (none count-only)."""
    p = Mx.empty_parts(1)[0].copy()
    for v in values:
        p["count"] += 1
        if v != v:
            p["n_nan"] += 1
            continue
        img = int(T.fast_value_to_u64(np.array([v]), "f64")[0])
        p["min_image"] = min(int(p["min_image"]), img)
        p["max_image"] = max(int(p["max_image"]), img)
        if abs(v) == float("inf"):
            p["n_inf"] += 1
            continue
        p["sum"] += v
        p["magnitude"] += abs(v)
        if v != 0.0:
            bits = struct.unpack("<Q", struct.pack("<d", abs(v)))[0]
            e, m = bits >> 52, bits & ((1 << 52) - 1)
            q = (e - 1075 if e else -1074) + ((m | (1 << 52 if e else 0)) & -(m | (1 << 52 if e else 0))).bit_length() - 1
            p["quantum_exp"] = min(int(p["quantum_exp"]), q)
    return p


def rows_from(buckets):
    """{pos: (doc_count, parts)} from {pos: [values of column 0]}."""
    out = {}
    for pos, vals in buckets.items():
        parts = Mx.empty_parts()
        parts[0] = part_of(vals)
        out[pos] = (len(vals), parts)
    return out


def f64_plan(aggs, hist=None):
    r = HMx.parse_request(request(hist or {"field": "v", "interval": 1.0}, aggs, typ="histogram"))
    return HMx.plan(r, {"v": Mx.MetricField(1, "f64")})


def test_merge_adds_counts_and_merges_parts():
    a = rows_from({0: [1.0, 2.0], 3: [0.5]})
    b = rows_from({3: [4.0, -1.0], 7: [8.0]})
    m = HMx.merge([a, b])
    assert sorted(m) == [0, 3, 7] and [m[p][0] for p in (0, 3, 7)] == [2, 3, 1]
    part = m[3][1][0]
    assert (int(part["count"]), float(part["sum"]), float(part["magnitude"]), int(part["quantum_exp"])) == (3, 3.5, 5.5, -1)
    assert int(part["min_image"]) == int(T.fast_value_to_u64(np.array([-1.0]), "f64")[0])
    assert (m[3][1][1:]["count"] == 0).all() and (m[3][1][1:]["quantum_exp"] == 2**31 - 1).all()
    assert HMx.merge([a])[0][0] == 2 and HMx.merge([]) == {}


def test_guard_refuses_one_bucket_while_the_others_pass():
    p = f64_plan({"s": {"sum": {"field": "v"}}, "mx": {"max": {"field": "v"}}, "c": {"value_count": {"field": "v"}}})
    rows = rows_from({0: [0.25, 0.5], 1: [1.0, 1.5], 2: [2.1, 2.2, 2.3]})  # bucket 2's decimals fail the guard
    with pytest.raises(HMx.HistMetricsRefused) as e:
        HMx.finalize(p, rows)
    assert set(e.value.refused) == {"s"} and "bucket 2" in e.value.refused["s"]
    b = e.value.answered["h"]["buckets"]
    assert [x["key"] for x in b] == [0.0, 1.0, 2.0] and [x["doc_count"] for x in b] == [2, 2, 3]
    assert all("s" not in x for x in b) and [x["mx"]["value"] for x in b] == [0.5, 1.5, 2.3] and b[2]["c"] == {"value": 3.0}
    ok = HMx.finalize(p, rows_from({0: [0.25, 0.5], 1: [1.0, 1.5]}))
    assert [x["s"]["value"] for x in ok["h"]["buckets"]] == [0.75, 2.5]
    with pytest.raises(HMx.HistMetricsRefused, match="NaN"):
        HMx.finalize(p, rows_from({0: [0.0, float("nan")], 1: [1.0]}))


def test_finalize_shapes():
    aggs = {"st": {"stats": {"field": "v"}}, "s": {"sum": {"field": "v"}}, "sn": {"sum": {"field": "v", "none_if_no_match": True}},
            "a": {"avg": {"field": "v"}}, "mn": {"min": {"field": "v"}}, "mx": {"max": {"field": "v"}}, "c": {"value_count": {"field": "v"}}}
    rows = rows_from({1: [1.0, 1.5], 4: [4.0]})
    # gap filling: buckets 2 and 3 hold the empty sub-aggregation results
    b = HMx.finalize(f64_plan(aggs), rows)["h"]["buckets"]
    assert [x["key"] for x in b] == [1.0, 2.0, 3.0, 4.0] and [x["doc_count"] for x in b] == [2, 0, 0, 1]
    assert b[0]["st"] == {"count": 2, "sum": 2.5, "min": 1.0, "max": 1.5, "avg": 1.25} and b[0]["sn"] == {"value": 2.5}
    for x in b[1:3]:
        assert x["st"] == {"count": 0, "sum": 0.0, "min": None, "max": None, "avg": None}
        assert (x["s"], x["sn"], x["a"], x["mn"], x["mx"], x["c"]) == ({"value": 0.0}, {"value": None}, {"value": None}, {"value": None},
                                                                         {"value": None}, {"value": 0.0})
    assert b[1]["st"] is not b[2]["st"]
    # min_doc_count drops the empty and the small buckets; keyed; extended_bounds
    b = HMx.finalize(f64_plan(aggs, {"field": "v", "interval": 1.0, "min_doc_count": 2}), rows)["h"]["buckets"]
    assert [x["key"] for x in b] == [1.0]
    k = HMx.finalize(f64_plan(aggs, {"field": "v", "interval": 1.0, "keyed": True}), rows)["h"]["buckets"]
    assert list(k) == ["1", "2", "3", "4"] and k["4"]["mx"] == {"value": 4.0}
    b = HMx.finalize(f64_plan(aggs, {"field": "v", "interval": 1.0, "extended_bounds": {"min": -1, "max": 5}}), rows)["h"]["buckets"]
    assert [x["key"] for x in b] == [-1.0, 0.0, 1.0, 2.0, 3.0, 4.0, 5.0] and b[0]["a"] == {"value": None} and b[-1]["c"] == {"value": 0.0}


def test_date_keys_and_metrics_on_the_date_field():
    r = HMx.parse_request({"h": {"date_histogram": {"field": "ts", "fixed_interval": "1h", "offset": "30m"},
                                 "aggs": {"first": {"min": {"field": "ts"}}, "n": {"value_count": {"field": "ts"}}}}})
    p = HMx.plan(r, {"ts": Mx.MetricField(1, "date")})
    h = 3_600 * 10**9
    t0 = 1_700_000_000 * 10**9
    ts = [t0 + 5, t0 + h // 2, t0 + 3 * h]
    imgs = T.fast_value_to_u64(np.array(ts, np.int64), "date")
    pos = {}
    for t, img in zip(ts, imgs):
        pos.setdefault((t - h // 2) // h, []).append(int(img))
    rows = {}
    for q, images in pos.items():
        parts = Mx.empty_parts()
        for c in range(2):
            parts[c]["count"] = len(images)
        parts[0]["min_image"], parts[0]["max_image"] = min(images), max(images)
        rows[q] = (len(images), parts)
    b = HMx.finalize(p, rows)["h"]["buckets"]
    assert [x["doc_count"] for x in b] == [1, 1, 0, 1]  # (t0 is 800 s into its hour)
    assert b[0]["key_as_string"] == "2023-11-14T21:30:00Z" and b[0]["key"] == (t0 // h * h - h // 2) / 1e6
    assert b[0]["first"] == {"value": float(t0 + 5)} and b[2]["first"] == {"value": None} and b[3]["n"] == {"value": 1.0}


# ---- the reference's vectors ------------------------------------------------------------------------------------------------
def fixture_plan(case):
    fields = {name: Mx.MetricField(i + 1, case["fields"][name]) for i, name in enumerate(sorted(case["fields"]))}
    return HMx.plan(HMx.parse_request(case["aggs"]), fields), fields


def same_tree(a, b):
    """Equal JSON trees, floats bit for bit."""
    if isinstance(a, dict) or isinstance(b, dict):
        return isinstance(a, dict) and isinstance(b, dict) and a.keys() == b.keys() and all(same_tree(a[k], b[k]) for k in a)
    if isinstance(a, list) or isinstance(b, list):
        return isinstance(a, list) and isinstance(b, list) and len(a) == len(b) and all(same_tree(x, y) for x, y in zip(a, b))
    if isinstance(a, float) and isinstance(b, float):
        return struct.pack("<d", a) == struct.pack("<d", b)
    return a == b and type(a) is type(b)


def check_asserts(case, result):
    for path, want in case["asserts"]:
        got = result
        for i, k in enumerate(path):
            if isinstance(k, int) and k >= len(got):
                assert want is None and i == len(path) - 1, (case["name"], path)
                got = None
                break
            got = got[k]
        if got is not None or want is not None:
            assert same_json(got, want), (case["name"], path, got, want)


def fixture_rows(case, p):
    """{pos: (doc_count, parts)} per fixture segment, as the device builds them: each hit doc with a histogram value in the
    segment's bounds to its bucket, every metric column collecting its value there."""
    hist_field = p.request.req.field
    _, kind, interval, offset, lo, hi = p.hspec
    out = []
    for seg in case["segments"]:
        buckets = {}
        for doc in seg:
            if not doc["hit"] or hist_field not in doc:
                continue
            v = float(doc[hist_field])
            if lo <= v <= hi:
                buckets.setdefault(int(np.floor((v - offset) / interval)), []).append(doc)
        rows = {}
        for pos, docs in buckets.items():
            parts = Mx.empty_parts()
            for c, (_, ckind, flags, _) in enumerate(p.mplan.columns):
                field = [a.field for a in p.mplan.aggs if p.mplan.slot[a.name] == c][0]
                parts[c] = part_of([float(d[field]) for d in docs if field in d])
            rows[pos] = (len(docs), parts)
        out.append(rows)
    return out


@pytest.mark.parametrize("case", FIXTURES, ids=[c["name"] for c in FIXTURES])
def test_reference_fixtures(case):
    """Each vector through the model and through parts built as the device builds them, merged and finalised by hist_metrics."""
    p, fields = fixture_plan(case)
    got = HMx.finalize(p, HMx.merge(fixture_rows(case, p)))
    check_asserts(case, got)
    # the model: Kahan per (segment, bucket) in doc order, merge_fruits in segment order
    r = p.request
    seg_parts = []
    for seg in case["segments"]:
        hist = [d.get(r.req.field) for d in seg]
        images = T.fast_value_to_u64(np.array([0.0 if v is None else v for v in hist], np.float64), "f64")
        present = np.array([v is not None for v in hist])
        selected = np.array([d["hit"] for d in seg])
        buckets = HMM.segment_buckets(images, present, selected, "f64", r.req.interval, r.req.offset or 0.0)
        values = {a.name: [MM.doc_values(a.type, case["fields"][a.field], d.get(a.field), a.missing) for d in seg] for a in r.metrics}
        seg_parts.append(HMM.segment_part(buckets, values))
    want = HMM.final(r.name, r.req, "f64", HMM.merge(seg_parts), [(a.name, a.type, a.name, a.none_if_no_match) for a in r.metrics])
    assert same_tree(got, want)
    check_asserts(case, want)
