"""The range aggregation's request and result side (tantivy_b200.ranges) without a GPU: parsing and every refusal, the ABI, the
conversions of bounds to images at saturation, extend_validate_ranges in image space with its overlap error, key strings, the merge,
the per-bucket guard, and the reference's range tests (tests/golden/range_fixtures.json) through the finaliser with rows built as
the device builds them, checked against tests/range_model.py as well."""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest

import tantivy_b200 as T
from tantivy_b200 import _abi
from tantivy_b200 import metrics as Mx
from tantivy_b200 import ranges as R
from tantivy_b200.histogram import AggregationError
from tantivy_b200.lib import LIB
from tests import metrics_model as MM
from tests import range_model as RM
from tests.test_hist_metrics_host import same_tree
from tests.test_histogram_host import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = json.load(open(os.path.join(ROOT, "tests", "golden", "range_fixtures.json")))["cases"]
U64_MAX = (1 << 64) - 1
F = Mx.MetricField
FIELDS = {"lat": F(1, "u64"), "t": F(2, "date"), "x": F(3, "f64"), "i": F(4, "i64"), "ok": F(5, "bool"), "host": F(6, "str"),
          "ip": F(7, "ip"), "raw": F(8, "bytes"), "tags": F(9, "u64", multi_valued=True), "json": F(10, "f64", n_column_types=2)}


def request(ranges, field="lat", aggs=None, keyed=None, name="r"):
    body = {"range": {"field": field, "ranges": ranges}}
    if keyed is not None:
        body["range"]["keyed"] = keyed
    if aggs is not None:
        body["aggs"] = aggs
    return {name: body}


def test_parse_and_plan():
    r = R.parse_request(request([{"to": 100}, {"from": 100, "to": 500, "key": "mid"}, {"from": 500}],
                                aggs={"avg_x": {"avg": {"field": "x"}}, "n": {"value_count": {"field": "ok"}}}, keyed=True))
    assert r.name == "r" and r.field == "lat" and r.keyed and [m.name for m in r.metrics] == ["avg_x", "n"]
    assert r.ranges == [(None, None, 100.0), ("mid", 100.0, 500.0), (None, 500.0, None)]
    p = R.plan(r, FIELDS)
    assert p.rspec == (1, [0, 100, 500]) and [b["key"] for b in p.buckets] == ["*-100", "mid", "500-*"]
    assert len(p.mplan.columns) == 2 and p.mplan.columns[1][2] == T.TQ_METRIC_COUNT_ONLY
    assert R.plan(R.parse_request(request([{"from": 10, "to": 20}])), FIELDS).mplan is None
    assert R.parse_request({"r": {"range": {"field": "lat", "ranges": [{}]}, "aggregations": {"m": {"max": {"field": "lat"}}}}}).metrics[0].type == "max"


@pytest.mark.parametrize("aggs, match", [
    ({"a": {"range": {"field": "lat", "ranges": [{}]}}, "b": {"avg": {"field": "lat"}}}, "more than one top-level"),
    ({"r": {"histogram": {"field": "lat", "interval": 1}}}, "not a range aggregation"),
    (request([{}], aggs={"term_agg": {"terms": {"field": "host"}}}), "r.term_agg: bucket aggregations nested under the range"),
    (request([{}], aggs={"h": {"histogram": {"field": "lat", "interval": 1}}}), "r.h: bucket aggregations nested under the range"),
    (request([{}], aggs={"p": {"percentiles": {"field": "lat"}}}), r"r\.p: "),
    (request([{}], aggs={"e": {"extended_stats": {"field": "lat"}}}), r"r\.e: "),
    (request([{}], aggs={"a": {"avg": {"field": "lat"}, "aggs": {"m": {"max": {"field": "lat"}}}}}), "r.a: sub-aggregations run on the CPU path"),
])
def test_parse_refusals(aggs, match):
    with pytest.raises(R.RangeRefused, match=match):
        R.parse_request(aggs)


@pytest.mark.parametrize("field, ranges, match", [
    ("ok", [{"to": 1}], "a range on a bool column"),
    ("host", [{"to": 1}], "a range on a str column"),
    ("ip", [{"to": 1}], "a range on a ip column"),
    ("raw", [{"to": 1}], "a range on a bytes column"),
    ("tags", [{"to": 1}], "multi-valued"),
    ("json", [{"to": 1}], "several column types"),
    ("nope", [{"to": 1}], "no registered fast column"),
    ("x", [{"from": float("nan")}], "a NaN bound"),
    ("lat", [{"from": 10, "to": 5}], "start exceeds its end"),
    ("lat", [{"to": 0}], "an empty range"),
    ("lat", [{"from": 5, "to": 5}], "an empty range"),
    ("lat", [{"from": -3, "to": 0}], "an empty range"),
    ("x", [{"from": -1.7976931348623157e308, "to": 0.0}], "one `from`"),
    ("lat", [{"from": i, "to": i + 1} for i in range(1, 128)], "129 buckets after extension"),
])
def test_plan_refusals(field, ranges, match):
    with pytest.raises(R.RangeRefused, match=match):
        R.plan(R.parse_request(request(ranges, field=field)), FIELDS)


def test_plan_refuses_keyed_duplicate_custom_keys_and_metrics_refusals():
    with pytest.raises(R.RangeRefused, match="sharing a custom key"):
        R.plan(R.parse_request(request([{"key": "a", "to": 1}, {"key": "a", "from": 1}], keyed=True)), FIELDS)
    R.plan(R.parse_request(request([{"key": "a", "to": 1}, {"key": "a", "from": 1}])), FIELDS)  # (a list keeps both)
    with pytest.raises(R.RangeRefused, match="r.m: "):
        R.plan(R.parse_request(request([{}], aggs={"m": {"avg": {"field": "tags"}}})), FIELDS)


def test_malformed_requests():
    with pytest.raises(AggregationError, match="at least one range"):
        R.parse_request(request([]))
    for bad in ({"r": {"range": {"field": "lat"}}}, request([{"from": "x"}]), request([{"from": True}]), request([{"too": 1}]),
                request([{"key": 3}]), {"r": {"range": {"field": "lat", "ranges": [], "extra": 1}}}, {}):
        with pytest.raises(AggregationError):
            R.parse_request(bad)


def test_abi_symbols_and_layouts(tmp_path):
    for name in ("tq_range_batch", "tq_get_range_stats"):
        assert hasattr(LIB, name)
    assert _abi.TQ_RANGE_MAX_BUCKETS == R.TQ_RANGE_MAX_BUCKETS == 128
    fields = [n for n, _ in _abi.RangeSpec._fields_]
    assert fields == ["column_id", "n_buckets", "starts"]
    assert _layout(tmp_path, "tq_range_spec", fields) == [getattr(_abi.RangeSpec, n).offset for n in fields] + [C.sizeof(_abi.RangeSpec)]
    assert [_abi.RANGE_SPEC_DTYPE.fields[n][1] for n in fields] == [getattr(_abi.RangeSpec, n).offset for n in fields]
    fields = [n for n, _ in _abi.RangeStats._fields_]
    assert fields == ["range_ms", "units_range", "range_tiles_seen", "range_tiles_one_bucket"]
    assert _layout(tmp_path, "tq_range_stats", fields) == [getattr(_abi.RangeStats, n).offset for n in fields] + [C.sizeof(_abi.RangeStats)]
    assert T.RangeRefused is R.RangeRefused


def test_conversions_at_saturation():
    cases = {
        "u64": [-1.0, -0.0, 0.0, 0.5, 1.9, 2.0**53 + 2, 2.0**64, 1e30, float("inf"), float("-inf"), float("nan")],
        "i64": [2.0**63, -(2.0**63), 1e30, -1e30, -0.0, 0.0, -1.5, 1.5, float("inf"), float("-inf"), float("nan")],
        "date": [1.7e18, -1.7e18, 2.0**63, float("nan")],
        "f64": [-0.0, 0.0, 5e-324, -5e-324, 2.2250738585072014e-308, float("inf"), float("-inf"), -1.7976931348623157e308],
    }
    for kind, vals in cases.items():
        for v in vals:
            assert R.to_image(v, kind) == RM.to_u64(v, kind), (kind, v)
    assert [R.to_image(v, "u64") for v in (-1.0, 1e30, float("nan"), 1.9)] == [0, U64_MAX, 0, 1]
    assert [R.to_image(v, "i64") for v in (2.0**63, -(2.0**63), float("nan"), -1.5)] == [U64_MAX, 0, 1 << 63, (1 << 63) - 1]
    assert R.to_image(-0.0, "f64") == (1 << 63) - 1 and R.to_image(0.0, "f64") == 1 << 63
    assert R.to_image(5e-324, "f64") == (1 << 63) + 1 and R.to_image(-5e-324, "f64") == (1 << 63) - 2
    assert R.to_image(float("inf"), "f64") == int(T.fast_value_to_u64(np.array([np.inf]), "f64")[0])


def test_overlap_is_decided_in_image_space():
    ranges = [{"from": 0.5, "to": 1.5}, {"from": 1.2, "to": 3}]
    with pytest.raises(AggregationError, match="Overlapping ranges not supported"):
        R.plan(R.parse_request(request(ranges, field="x")), FIELDS)
    with pytest.raises(RM.Overlap):
        RM.extend_validate([(None, 0.5, 1.5), (None, 1.2, 3.0)], "f64")
    p = R.plan(R.parse_request(request(ranges, field="lat")), FIELDS)  # 0..1, 1..3 on a u64 column
    assert p.rspec[1] == [0, 1, 3] and [b["key"] for b in p.buckets] == ["*-1", "1-3", "3-*"]


def test_extension_matches_the_model():
    rng = np.random.default_rng(5)
    for kind in ("u64", "i64", "f64", "date"):
        for _ in range(200):
            pts = sorted(set(rng.integers(-50, 50, size=rng.integers(2, 8)).tolist()))
            ranges = [(None, float(a), float(b)) for a, b in zip(pts[:-1], pts[1:]) if rng.random() < 0.7]
            if not ranges:
                continue
            try:
                want = RM.extend_validate(ranges, kind)
            except RM.Overlap:
                with pytest.raises(AggregationError):
                    R.extend(ranges, kind)
                continue
            assert R.extend(ranges, kind) == want


def test_key_strings():
    assert R.bound_string(0, "u64", True) == "*" and R.bound_string(U64_MAX, "u64", False) == "*"
    assert R.bound_string(0, "u64", False) == "0" and R.bound_string(1 << 63, "u64", True) == "9223372036854776000"  # (Display: shortest digits, padded)
    assert R.bound_string(R.to_image(-0.0, "f64"), "f64", True) == "-0" and R.bound_string(R.to_image(0.1, "f64"), "f64", True) == "0.1"
    assert R.bound_string(R.to_image(1e21, "f64"), "f64", True) == "1000000000000000000000"
    assert R.bound_string(R.to_image(1546300800e9, "date"), "date", True) == "2019-01-01T00:00:00Z"
    assert R.bound_string(R.to_image(-5.0, "i64"), "i64", False) == "-5"
    p = R.plan(R.parse_request(request([{"from": 2.0**63}], field="lat")), FIELDS)
    assert [b["key"] for b in p.buckets] == ["*-9223372036854776000", "9223372036854776000-*"] == \
           [RM.range_string(0, 1 << 63, "u64"), RM.range_string(1 << 63, U64_MAX, "u64")]
    p = R.plan(R.parse_request(request([{"from": 1546300800e9, "to": 1546387200e9}], field="t")), FIELDS)
    e = R.bucket_entry(p.buckets[1], 4, "date")
    assert e == {"key": "2019-01-01T00:00:00Z-2019-01-02T00:00:00Z", "doc_count": 4, "from": 1546300800e9, "to": 1546387200e9,
                 "from_as_string": "2019-01-01T00:00:00Z", "to_as_string": "2019-01-02T00:00:00Z"}


# ---- parts as the device builds them ----------------------------------------------------------------------------------------
def part_of(values, kind):
    """The tq_metric_part of a list of a column's values (its images and f64 values)."""
    p = Mx.empty_parts(1)[0].copy()
    for v in values:
        p["count"] += 1
        img = int(T.fast_value_to_u64(np.array([v], np.float64 if kind == "f64" else np.int64), kind)[0]) if kind != "u64" else int(v)
        f = Mx.value_of_image(img, Mx._VALUE_KINDS[kind])
        if f != f:
            p["n_nan"] += 1
            continue
        p["min_image"] = min(int(p["min_image"]), img)
        p["max_image"] = max(int(p["max_image"]), img)
        if abs(f) == float("inf"):
            p["n_inf"] += 1
            continue
        p["sum"] += f
        p["magnitude"] += abs(f)
        if f != 0.0:
            bits = struct.unpack("<Q", struct.pack("<d", abs(f)))[0]
            e, m = bits >> 52, bits & ((1 << 52) - 1)
            m |= (1 << 52) if e else 0
            p["quantum_exp"] = min(int(p["quantum_exp"]), (e - 1075 if e else -1074) + (m & -m).bit_length() - 1)
    return p


def check_asserts(case, result):
    """The reference's assert_eq!s: [path, value], null for an absent value (an index past the end or a missing key)."""
    for path, want in case["asserts"]:
        got = result
        for k in path:
            if got is None or (isinstance(k, int) and k >= len(got)) or (isinstance(k, str) and k not in got):
                got = None
                break
            got = got[k]
        assert same_tree(got, want) or (isinstance(want, int) and got == want and not isinstance(got, bool)), (case["name"], path, got, want)


def fixture_plan(case):
    fields = {name: F(i + 1, kind) for i, (name, kind) in enumerate(sorted(case["fields"].items()))}
    return R.plan(R.parse_request(case["aggs"]), fields), fields


def collected(case, doc):
    return case.get("all_docs") or doc["hit"]


def device_rows(case, p, fields):
    """(doc_count, parts) per fixture segment, as the device builds them: each collected doc with a value of the range field to
    its bucket, every metric column collecting its value there."""
    field = p.request.field
    starts = p.rspec[1]
    out = []
    for seg in case["segments"]:
        docs = [[] for _ in starts]
        for d in seg:
            if collected(case, d) and field in d:
                img = R.to_image(float(d[field]), p.kind) if p.kind != "u64" else int(d[field])
                docs[RM.bucket_pos(img, starts)].append(d)
        counts = np.array([len(x) for x in docs], np.uint64)
        parts = None
        if p.mplan is not None:
            parts = np.stack([Mx.empty_parts() for _ in starts])
            for c in range(len(p.mplan.columns)):
                f = [a.field for a in p.mplan.aggs if p.mplan.slot[a.name] == c][0]
                for b, ds in enumerate(docs):
                    parts[b][c] = part_of([d[f] for d in ds if f in d], case["fields"][f])
        out.append((counts, parts))
    return out


def model_result(case, p):
    r, kind = p.request, p.kind
    metrics = [(a.name, a.type, a.name, a.none_if_no_match) for a in r.metrics]
    seg_buckets, values = [], []
    starts = [s for _, s, _ in RM.extend_validate(r.ranges, kind)]
    for seg in case["segments"]:
        images = [RM.to_u64(float(d.get(r.field, 0)), kind) if kind != "u64" else int(d.get(r.field, 0)) for d in seg]
        present = np.array([r.field in d for d in seg])
        sel = np.array([bool(collected(case, d)) for d in seg])
        seg_buckets.append(RM.segment_buckets(np.array(images, np.uint64), present, sel, starts))
        values.append({a.name: [MM.doc_values(a.type, case["fields"][a.field], d.get(a.field), a.missing) for d in seg] for a in r.metrics})
    return RM.result(r.name, r.ranges, kind, r.keyed, seg_buckets, values, metrics)


PLANNING = [c for c in FIXTURES if "column_type" in c]
SEARCHES = [c for c in FIXTURES if "segments" in c]


@pytest.mark.parametrize("case", SEARCHES, ids=[c["name"] for c in SEARCHES])
def test_reference_fixtures(case):
    """Each search vector through the finaliser with device-shaped rows (split over two contexts as well), and through the model."""
    if case.get("refused"):
        with pytest.raises(R.RangeRefused, match=case["refused"]):
            R.parse_request(case["aggs"])
        return
    p, fields = fixture_plan(case)
    rows = device_rows(case, p, fields)
    got = R.finalize(p, R.merge(rows))
    halves = [R.merge(rows[:1]), R.merge(rows[1:])] if len(rows) > 1 else [R.merge(rows)]
    assert same_tree(R.finalize(p, R.merge(halves)), got)
    want = model_result(case, p)
    assert same_tree(got, want)
    if "expected" in case:
        assert same_tree(got, case["expected"]), (got, case["expected"])
    else:
        check_asserts(case, got)


@pytest.mark.parametrize("case", PLANNING, ids=[c["name"] for c in PLANNING])
def test_reference_planning_fixtures(case):
    kind = case["column_type"]
    ranges = [(r.get("key"), r.get("from"), r.get("to")) for r in case["ranges"]]
    ext = R.extend(ranges, kind)
    assert ext == RM.extend_validate(ranges, kind)
    if "expected_ranges" in case:
        assert [[s, e] for _, s, e in ext] == case["expected_ranges"]
    if "first_key" in case:
        p = R.plan(R.parse_request(request(case["ranges"], field="f")), {"f": F(1, kind)})
        assert p.buckets[0]["key"] == case["first_key"] and p.buckets[-1]["key"] == case["last_key"]
    for image, pos in case.get("search", []):
        assert RM.bucket_pos(image, [s for _, s, _ in ext]) == pos


def test_merge_and_the_guard_per_bucket():
    """Counts add over contexts, parts merge; a sum failing the guard in one bucket refuses that sum for the whole range, the rest
    answered, the bucket named."""
    aggs = {"s": {"sum": {"field": "x"}}, "m": {"max": {"field": "x"}}}
    p = R.plan(R.parse_request(request([{"to": 10}], aggs=aggs)), FIELDS)
    ok, bad = part_of([1.5, 2.25], "f64"), part_of([0.1] * 3, "f64")
    a = (np.array([2, 0], np.uint64), np.stack([Mx.empty_parts(), Mx.empty_parts()]))
    a[1][0][0] = ok
    b = (np.array([1, 3], np.uint64), np.stack([Mx.empty_parts(), Mx.empty_parts()]))
    b[1][0][0] = part_of([4.0], "f64")
    b[1][1][0] = bad
    counts, parts = R.merge([a, b])
    assert counts.tolist() == [3, 3] and int(parts[0][0]["count"]) == 3 and float(parts[0][0]["sum"]) == 7.75
    with pytest.raises(R.RangeRefused) as e:
        R.finalize(p, (counts, parts))
    assert set(e.value.refused) == {"s"} and "(bucket 10-*)" in e.value.refused["s"]
    buckets = e.value.answered["r"]["buckets"]
    assert [x["key"] for x in buckets] == ["*-10", "10-*"] and buckets[0]["m"] == {"value": 4.0} and "s" not in buckets[0]
    assert buckets[1]["m"] == {"value": 0.1}
    # a zero-doc bucket holds the empty metric results
    res = R.finalize(p, (np.array([0, 0], np.uint64), np.stack([Mx.empty_parts(), Mx.empty_parts()])))
    assert res["r"]["buckets"][0] == {"key": "*-10", "doc_count": 0, "to": 10.0, "s": {"value": 0.0}, "m": {"value": None}}


def test_final_order_follows_from_not_the_request():
    p = R.plan(R.parse_request(request([{"from": 20, "key": "z"}, {"to": 5, "key": "a"}, {"from": 5, "to": 20}], keyed=True)), FIELDS)
    res = R.finalize(p, (np.array([1, 2, 3], np.uint64), None))
    assert list(res["r"]["buckets"]) == ["a", "5-20", "z"]
    assert [b["doc_count"] for b in res["r"]["buckets"].values()] == [1, 2, 3]
