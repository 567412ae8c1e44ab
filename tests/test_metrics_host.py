"""The host side of metric aggregations (tantivy_b200.metrics): parsing, refusals, the ABI layouts, the exactness guard and the
finaliser, against tests/metrics_model.py (a literal restatement of the reference's Kahan collection, merge and finalisation).
The guard is checked on seeded random multisets, doc orders and segment splits: every accepted case must give the model's result
bit for bit.  No GPU: parts are built here the way the device builds them (unordered f64 adds)."""
import ctypes as C
import json
import math
import os
import random
import struct

import numpy as np
import pytest

from tantivy_b200 import metrics as Mx
from tantivy_b200._abi import (METRIC_PART_DTYPE, METRICS_SPEC_DTYPE, TQ_FAST_BOOL, TQ_FAST_DATE, TQ_FAST_F64, TQ_FAST_I64, TQ_FAST_U64,
                               TQ_METRIC_COUNT_ONLY, TQ_METRIC_EMPTY, TQ_METRIC_MISSING, MetricColumn, MetricPart, MetricsSpec, MetricsStats)
from tantivy_b200.histogram import AggregationError
from tantivy_b200.lib import LIB, fast_value_to_u64
from tests import metrics_model as MM
from tests.test_histogram_host import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = json.load(open(os.path.join(ROOT, "tests", "golden", "metrics_fixtures.json")))["cases"]

KIND_NAME = {TQ_FAST_U64: "u64", TQ_FAST_I64: "i64", TQ_FAST_F64: "f64", TQ_FAST_DATE: "date", TQ_FAST_BOOL: "bool"}


def image_of(v, kind):
    return int(fast_value_to_u64(np.array([v], dtype=np.float64 if kind == TQ_FAST_F64 else np.int64), KIND_NAME[kind])[0])


def quantum(v):
    bits = struct.unpack("<Q", struct.pack("<d", abs(v)))[0]
    e, m = bits >> 52, bits & ((1 << 52) - 1)
    if e:
        m |= 1 << 52
    tz = (m & -m).bit_length() - 1
    return (e - 1075 if e else -1074) + tz


def part_of(values, kind=TQ_FAST_F64, rng=None):
    """One tq_metric_part of values, summed in a random order as the device may."""
    p = Mx.empty_parts(1)[0]
    vals = list(values)
    if rng is not None:
        rng.shuffle(vals)
    p["count"] = len(vals)
    s = m = 0.0
    for v in vals:
        if v != v:
            p["n_nan"] += 1
            continue
        img = image_of(v, kind)
        p["min_image"] = min(int(p["min_image"]), img)
        p["max_image"] = max(int(p["max_image"]), img)
        if math.isinf(v):
            p["n_inf"] += 1
            continue
        s += v
        m += abs(v)
        if v != 0.0:
            p["quantum_exp"] = min(int(p["quantum_exp"]), quantum(v))
    p["sum"], p["magnitude"] = s, m
    return p


def as_parts(p):
    out = Mx.empty_parts()
    out[0] = p
    return out


def one_plan(typ, kind="f64", missing=None, none_if_no_match=False):
    body = {"field": "x"}
    if missing is not None:
        body["missing"] = missing
    if none_if_no_match:
        body["none_if_no_match"] = True
    aggs = Mx.parse_request({"a": {typ: body}})
    return Mx.plan(aggs, {"x": Mx.MetricField(7, kind)})


def same(a, b):
    """Equal results, floats bit for bit (-0.0 != +0.0, NaN == NaN)."""
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, float) and isinstance(b, float):
        return struct.pack("<d", a) == struct.pack("<d", b)
    return a == b and type(a) is type(b)


# ---- parsing and refusals --------------------------------------------------------------------------------------------------
def test_parse_defaults_and_missing():
    aggs = Mx.parse_request({"a": {"avg": {"field": "f"}}, "b": {"sum": {"field": "g", "missing": "10.5", "none_if_no_match": True}},
                             "c": {"stats": {"field": "f", "missing": 3}}, "d": {"value_count": {"field": "f"}}})
    assert [(a.name, a.type, a.field, a.missing, a.none_if_no_match) for a in aggs] == [
        ("a", "avg", "f", None, False), ("b", "sum", "g", 10.5, True), ("c", "stats", "f", 3.0, False), ("d", "value_count", "f", None, False)]


@pytest.mark.parametrize("req,msg", [
    ({"a": {"extended_stats": {"field": "f"}}}, "sum of squares|sums squares"),
    ({"a": {"percentiles": {"field": "f"}}}, "percentiles"),
    ({"a": {"cardinality": {"field": "f"}}}, "cardinality"),
    ({"a": {"top_hits": {"size": 1}}}, "top_hits"),
    ({"a": {"avg": {"field": "f"}, "aggs": {"b": {"max": {"field": "f"}}}}}, "sub-aggregations"),
    ({"a": {"avg": {"field": "f"}}, "t": {"terms": {"field": "f"}}}, "bucket aggregation \\(terms\\)"),
])
def test_parse_refusals(req, msg):
    with pytest.raises(Mx.MetricsRefused, match=msg):
        Mx.parse_request(req)


@pytest.mark.parametrize("req", [{}, {"a": {"avg": {}}}, {"a": {"avg": {"field": "f", "interval": 1}}}, {"a": {"max": {"field": "f", "none_if_no_match": True}}},
                                 {"a": {"avg": {"field": "f", "missing": "x"}}}, {"a": {"median": {"field": "f"}}}])
def test_parse_errors(req):
    with pytest.raises(AggregationError):
        Mx.parse_request(req)


def test_plan_shares_columns_and_refuses():
    fields = {"a": Mx.MetricField(1, "u64"), "b": Mx.MetricField(2, "f64"), "c": Mx.MetricField(3, "i64"), "d": Mx.MetricField(4, "date"),
              "e": Mx.MetricField(5, "u64"), "m": Mx.MetricField(6, "u64", multi_valued=True), "j": Mx.MetricField(8, "u64", n_column_types=2),
              "s": Mx.MetricField(9, "str"), "o": Mx.MetricField(10, "bool"), "x": Mx.MetricField(11, "json_obj")}
    p = Mx.plan(Mx.parse_request({"n": {"min": {"field": "a"}}, "x": {"max": {"field": "a"}}, "s": {"stats": {"field": "b"}},
                                  "m": {"sum": {"field": "a", "missing": 5}}}), fields)
    assert p.columns == [(1, TQ_FAST_U64, 0, 0), (2, TQ_FAST_F64, 0, 0), (1, TQ_FAST_U64, TQ_METRIC_MISSING, 5)]
    assert p.slot == {"n": 0, "x": 0, "s": 1, "m": 2}
    # value_count reads str and bool columns (0.0 per value; a str `missing` is None, a bool one `m as u64`); every other metric
    # reads tantivy's empty U64 column there, where `missing` is `m as u64`
    p = Mx.plan(Mx.parse_request({"s": {"value_count": {"field": "s", "missing": 1}}, "o": {"value_count": {"field": "o", "missing": 1}},
                                  "t": {"sum": {"field": "o", "missing": 2.5}}, "u": {"avg": {"field": "s"}}}), fields)
    assert p.columns == [(9, TQ_FAST_U64, TQ_METRIC_COUNT_ONLY, 0), (10, TQ_FAST_BOOL, TQ_METRIC_COUNT_ONLY | TQ_METRIC_MISSING, 1),
                         (0, TQ_FAST_U64, TQ_METRIC_EMPTY | TQ_METRIC_MISSING, 2), (0, TQ_FAST_U64, TQ_METRIC_EMPTY, 0)]
    assert p.slot == {"s": 0, "o": 1, "t": 2, "u": 3}
    for req, msg in (({"q": {"avg": {"field": "m"}}}, "multi-valued"), ({"q": {"avg": {"field": "j"}}}, "several column types"),
                     ({"q": {"avg": {"field": "x"}}}, "json_obj columns"), ({"q": {"avg": {"field": "zz"}}}, "no registered"),
                     ({k: {"avg": {"field": k}} for k in "abcde"}, "more than 4")):
        with pytest.raises(Mx.MetricsRefused, match=msg):
            Mx.plan(Mx.parse_request(req), fields)


def test_spec_part_and_stats_layouts_match_the_compiler(tmp_path):
    for name in ("tq_metrics_batch", "tq_get_metrics_stats"):
        assert hasattr(LIB, name)
    for struct, cls, dtype in (("tq_metric_column", MetricColumn, METRICS_SPEC_DTYPE["columns"].base), ("tq_metrics_spec", MetricsSpec, METRICS_SPEC_DTYPE),
                               ("tq_metric_part", MetricPart, METRIC_PART_DTYPE), ("tq_metrics_stats", MetricsStats, None)):
        fields = [n for n, _ in cls._fields_]
        assert _layout(tmp_path, struct, fields) == [getattr(cls, n).offset for n in fields] + [C.sizeof(cls)], struct
        if dtype is not None:
            assert [dtype.fields[n][1] for n in fields] == [getattr(cls, n).offset for n in fields] and dtype.itemsize == C.sizeof(cls), struct
    assert [n for n, _ in MetricsStats._fields_] == ["metrics_ms", "units_metrics", "metrics_tiles_seen", "metrics_tiles_one_value"]


# ---- the guard --------------------------------------------------------------------------------------------------------------
def model_final(segments, typ):
    return MM.final(MM.merged([MM.segment_stats(s) for s in segments]), typ)


def device_final(segments, typ, rng):
    parts = [as_parts(part_of(s, rng=rng)) for s in segments]
    rng.shuffle(parts)
    return Mx.finalize(one_plan(typ), Mx.merge(parts))["a"]


def random_values(rng):
    n = rng.randrange(0, 60)
    style = rng.randrange(6)
    if style == 0:  # small integers
        return [float(rng.randrange(-1000, 1000)) for _ in range(n)]
    if style == 1:  # dyadic values of a few scales
        return [rng.randrange(-2**20, 2**20) * 2.0 ** rng.randrange(-30, 5) for _ in range(n)]
    if style == 2:  # near the bound: 2^52-ish integers
        return [float(rng.randrange(2**49, 2**50)) * rng.choice((-1, 1)) for _ in range(n)]
    if style == 3:  # decimals
        return [round(rng.uniform(-100, 100), 3) for _ in range(n)]
    if style == 4:  # huge and tiny scales
        e = rng.choice((-1074, -1060, 900, 960, 1000))
        return [rng.randrange(1, 2**10) * 2.0 ** e for _ in range(n)]
    return [rng.choice((0.0, -0.0, 1.0, -1.0, 0.5, 2.0**60)) for _ in range(n)]


def test_guard_property_accepted_cases_are_bit_exact():
    rng = random.Random(0x6A2D)
    accepted = refused = 0
    for _ in range(3000):
        vals = random_values(rng)
        rng.shuffle(vals)
        cuts = sorted(rng.randrange(0, len(vals) + 1) for _ in range(rng.randrange(0, 4)))
        segs = [vals[a:b] for a, b in zip([0] + cuts, cuts + [len(vals)])]
        why = Mx.guard(Mx.merge([as_parts(part_of(s)) for s in segs])[0])
        if why is not None:
            refused += 1
            continue
        accepted += 1
        for typ in ("sum", "avg", "stats", "min", "max", "value_count"):
            assert same(device_final(segs, typ, rng), model_final(segs, typ)), (typ, segs)
        assert same(model_final(segs, "sum")["value"], math.fsum(vals) + 0.0)
    assert accepted > 1200 and refused > 300


def test_guard_boundaries():
    q = -3  # values are multiples of 2^-3
    below = [2.0 ** (52 + q), 2.0 ** (52 + q) - 2.0 ** q]  # sum = 2^(53+q) - 2^q
    at = below + [2.0 ** q]  # sum = 2^(53+q)
    assert int(part_of(below)["quantum_exp"]) == q and Mx.guard(part_of(below)) is None
    assert Mx.guard(part_of(at)) is not None
    assert Mx.guard(part_of([-x for x in at])) is not None
    # subnormal quantum: multiples of 2^-1074
    sub = [5e-324, 3 * 5e-324, 2.0**-1022]
    p = part_of(sub)
    assert int(p["quantum_exp"]) == -1074 and Mx.guard(p) is None
    assert same(model_final([sub], "sum")["value"], math.fsum(sub))
    # 53 + Q > 1023: accepted while the magnitude is finite
    big = [2.0**1000, 2.0**1000 * 3]
    assert int(part_of(big)["quantum_exp"]) == 1000 and Mx.guard(part_of(big)) is None
    assert Mx.guard(part_of([2.0**1023, 2.0**1023])) is not None  # magnitude overflows
    assert Mx.guard(part_of([float("nan"), 1.0])) is not None and Mx.guard(part_of([float("inf")])) is not None
    assert Mx.guard(part_of([])) is None and Mx.guard(part_of([0.0, -0.0])) is None


def test_guard_matters_on_decimals():
    vals = [0.1] * 10 + [1e16, -1e16, 0.3]
    kahan = model_final([vals], "sum")["value"]
    naive = 0.0
    for v in vals:
        naive += v
    assert kahan != naive or kahan != math.fsum(vals)  # the order-dependent sums differ ...
    p = part_of(vals)
    assert Mx.guard(p) is not None  # ... and the guard refuses
    with pytest.raises(Mx.MetricsRefused) as e:
        Mx.finalize(one_plan("sum"), as_parts(p))
    assert "a" in e.value.refused


# ---- the finaliser ------------------------------------------------------------------------------------------------------------
def check_all(values_by_seg, kind="f64"):
    for typ in ("sum", "avg", "stats", "min", "max", "value_count"):
        p = one_plan(typ, kind)
        merged = Mx.merge([as_parts(part_of(s)) for s in values_by_seg])
        try:
            got = Mx.finalize(p, merged)["a"]
        except Mx.MetricsRefused as e:
            assert typ in Mx.SUM_BEARING, (typ, e)
            continue
        assert same(got, model_final(values_by_seg, typ)), (typ, got, model_final(values_by_seg, typ))


@pytest.mark.parametrize("case", [[], [[]], [[float("nan")] * 3], [[float("inf"), float("inf")]], [[float("-inf")]], [[0.0, -0.0], [0.0]],
                                  [[-0.0]], [[0.0]], [[float("nan"), 2.5, float("-inf")], [1.0]], [[3.0, -3.0]]])
def test_finaliser_edges(case):
    check_all(case)


def test_empty_sum_none_if_no_match():
    empty = Mx.empty_parts()
    assert Mx.finalize(one_plan("sum"), empty) == {"a": {"value": 0.0}}
    assert Mx.finalize(one_plan("sum", none_if_no_match=True), empty) == {"a": {"value": None}}
    assert Mx.finalize(one_plan("avg"), empty) == {"a": {"value": None}}
    assert Mx.finalize(one_plan("stats"), empty) == {"a": {"count": 0, "sum": 0.0, "min": None, "max": None, "avg": None}}
    assert Mx.finalize(one_plan("value_count"), empty) == {"a": {"value": 0.0}}


def test_value_count_on_text_and_bool_counts_values():
    p = Mx.empty_parts()
    p[0]["count"] = 5
    for kind in ("str", "bool", "ip"):
        plan = one_plan("value_count", kind)
        assert plan.columns[0][2] == TQ_METRIC_COUNT_ONLY
        assert Mx.finalize(plan, p) == {"a": {"value": 5.0}}


@pytest.mark.parametrize("kind", ["str", "bool", "bytes", "ip"])
def test_other_metrics_on_non_numeric_fields_read_an_empty_column(kind):
    """stats / sum / avg / min / max on a str, bool, bytes or ip field read tantivy's empty U64 column: no value, count 0, and
    with `missing` every collected doc collects `m as u64`."""
    for typ in ("stats", "sum", "avg", "min", "max"):
        plan = one_plan(typ, kind)
        assert plan.columns == [(0, TQ_FAST_U64, TQ_METRIC_EMPTY, 0)]
        assert same(Mx.finalize(plan, Mx.empty_parts())["a"], MM.final(MM.Stats(), typ))
        plan = one_plan(typ, kind, missing=3.7)
        assert plan.columns == [(0, TQ_FAST_U64, TQ_METRIC_EMPTY | TQ_METRIC_MISSING, 3)]
        vals = [v for _ in range(4) for v in MM.doc_values(typ, kind, None, 3.7)]
        assert vals == [3.0] * 4
        assert same(Mx.finalize(plan, as_parts(part_of(vals, TQ_FAST_U64)))["a"], MM.final(MM.segment_stats(vals), typ))
    assert MM.doc_values("value_count", "bytes", None, 2) == [2.0] and MM.doc_values("value_count", "str", None, 2) == []


def test_refusal_keeps_the_other_answers():
    aggs = Mx.parse_request({"s": {"sum": {"field": "x"}}, "n": {"min": {"field": "x"}}, "c": {"value_count": {"field": "x"}}})
    p = Mx.plan(aggs, {"x": Mx.MetricField(7, "f64")})
    with pytest.raises(Mx.MetricsRefused) as e:
        Mx.finalize(p, as_parts(part_of([0.1, 0.2, float("nan")])))
    assert set(e.value.refused) == {"s"} and "NaN" in e.value.refused["s"]
    assert e.value.answered == {"n": {"value": 0.1}, "c": {"value": 3.0}}


def test_integer_kinds_through_images():
    rng = random.Random(5)
    for kind in ("u64", "i64", "date"):
        code = {"u64": TQ_FAST_U64, "i64": TQ_FAST_I64, "date": TQ_FAST_DATE}[kind]
        lo = 0 if kind == "u64" else -10**6
        vals = [float(rng.randrange(lo, 10**6)) for _ in range(200)]
        for typ in ("stats", "min", "max"):
            got = Mx.finalize(one_plan(typ, kind), as_parts(part_of(vals, code)))["a"]
            assert same(got, model_final([vals], typ))


# ---- the reference's vectors ----------------------------------------------------------------------------------------------------
def fixture_plan(case):
    fields = {name: Mx.MetricField(i + 1, case["fields"][name]) for i, name in enumerate(sorted(case["fields"]))}
    return Mx.plan(Mx.parse_request(case["aggs"]), fields), fields


def collected(case, typ, field, missing, seg):
    """The values one fixture segment collects for one aggregation, by the model's column rules."""
    kind = case["fields"][field]
    return [v for doc in seg if doc["hit"] for v in MM.doc_values(typ, kind, doc.get(field), missing)]


def check_fixture(case, expected):
    for name, want in case["expected"].items():
        assert same_json(expected[name], want), (case["name"], name, expected[name], want)


def same_json(got, want):
    if isinstance(want, dict):
        return got.keys() == want.keys() and all(same_json(got[k], want[k]) for k in want)
    if want is None or got is None:
        return got is None and want is None
    return float(got) == float(want)


@pytest.mark.parametrize("case", FIXTURES, ids=[c["name"] for c in FIXTURES])
def test_reference_fixtures(case):
    """Each vector through the model (Kahan per segment, merge_fruits) and through the device's parts, built here per segment as
    the device builds them, merged and finalised by tantivy_b200.metrics."""
    if "refused" in case:
        with pytest.raises(Mx.MetricsRefused, match=case["refused"]):
            fixture_plan(case)
        return
    p, fields = fixture_plan(case)
    model = {}
    for a in p.aggs:
        st = MM.merged([MM.segment_stats(collected(case, a.type, a.field, a.missing, seg)) for seg in case["segments"]])
        model[a.name] = MM.final(st, a.type, a.none_if_no_match)
    check_fixture(case, model)
    # parts: per segment and spec column, the values of the first aggregation that reads the column
    owner = {}
    for a in p.aggs:
        owner.setdefault(p.slot[a.name], a)
    parts = []
    for seg in case["segments"]:
        part = Mx.empty_parts()
        for i, (_, kind, _, _) in enumerate(p.columns):
            a = owner[i]
            part[i] = part_of(collected(case, a.type, a.field, a.missing, seg), kind)
        parts.append(part)
    got = Mx.finalize(p, Mx.merge(parts))
    check_fixture(case, got)
    for name in got:
        assert same(got[name], model[name]), name
