"""The request and result side of the device histogram (tantivy_b200.histogram) on the CPU: date_histogram interval and offset
parsing against the reference's vectors (date_histogram.rs:257-305), the finaliser over the reference's histogram tests transcribed
as data (tests/golden/histogram_fixtures.json) with each segment collected by tests/histogram_model.py, and the C ABI of
tq_histogram_batch as mirrored by _abi.py."""
import ctypes as C
import json
import os
import re
import subprocess

import numpy as np
import pytest

import tantivy_b200 as T
from tantivy_b200 import _abi
from tantivy_b200 import histogram as Hg
from tantivy_b200.lib import LIB
from tests import histogram_model as HM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = json.load(open(os.path.join(ROOT, "tests", "golden", "histogram_fixtures.json")))["cases"]


def test_parse_into_milliseconds():
    assert Hg.parse_into_milliseconds("1m") == 60_000
    assert Hg.parse_into_milliseconds("2m") == 120_000
    assert Hg.parse_into_milliseconds("2minutes") == 120_000
    assert Hg.parse_into_milliseconds("30s") == 30_000
    assert Hg.parse_into_milliseconds("1h") == 3_600_000 and Hg.parse_into_milliseconds("1d") == 86_400_000
    for bad, what in (("2y", "Unit not recognized"), ("2000", "Unit not found"), ("ms", "Number not found"), ("１m", "Number not found"),
                      ("", "Number not found"), ("+1m", "Number not found"), ("99999999999999999999ms", "Number not found"),
                      ("9223372036855ms", "out of bounds"), ("200000d", "out of bounds")):
        with pytest.raises(Hg.AggregationError, match=what):
            Hg.parse_into_milliseconds(bad)
    assert Hg.parse_into_milliseconds("9223372036854ms") == 9223372036854  # the largest whose nanoseconds fit i64


def test_parse_offset_into_milliseconds():
    for text, ms in (("1m", 60_000), ("+1m", 60_000), ("-1m", -60_000), ("2m", 120_000), ("+2m", 120_000), ("-2m", -120_000), ("-2ms", -2)):
        assert Hg.parse_offset_into_milliseconds(text) == ms
    for bad, what in (("2y", "Unit not recognized"), ("2000", "Unit not found"), ("ms", "Number not found"), ("", "offset is invalid"),
                      ("--1m", "Number not found")):
        with pytest.raises(Hg.AggregationError, match=what):
            Hg.parse_offset_into_milliseconds(bad)


def test_as_i64_and_positions():
    assert [Hg.as_i64(x) for x in (np.nan, np.inf, -np.inf, 1e300, -1e300, -0.5, 2.9, -2.9)] == [0, 2**63 - 1, -2**63, 2**63 - 1, -2**63, 0, 2, -2]
    f = np.array([np.nan, np.inf, -np.inf, 9.3e18, -9.3e18, 2.5, -2.5])
    assert list(HM.as_i64(f)) == [Hg.as_i64(x) for x in f]
    assert Hg.bucket_pos(0.3, 0.1, 0.0) == 2  # 0.3 / 0.1 = 2.9999999999999996
    assert Hg.bucket_pos(-0.0, 1.0, 0.0) == 0 and Hg.bucket_pos(-1e-300, 1.0, 0.0) == -1
    assert Hg.bucket_key(3, 0.1, 0.0) == 0.30000000000000004


def test_rust_display_and_dates():
    assert [Hg.rust_f64_display(x) for x in (0.0, 50.0, -0.0, 1.5, 1e20, 0.1, np.inf, np.nan)] == ["0", "50", "-0", "1.5", "100000000000000000000", "0.1", "inf", "NaN"]
    assert Hg.format_date(1420070400000 * 10**6) == "2015-01-01T00:00:00Z"
    assert Hg.format_date(1420070400000 * 10**6 + 500_000_000) == "2015-01-01T00:00:00.5Z"
    assert Hg.format_date(-1) == "1969-12-31T23:59:59.999999999Z"


def test_validation():
    ok = Hg.HistogramAggregation("f", 1.0)
    ok.validate()
    for req, what in ((Hg.HistogramAggregation("f", 0.0), "positive"), (Hg.HistogramAggregation("f", -1.0), "positive"),
                      (Hg.HistogramAggregation("f", 1.0, min_doc_count=1, extended_bounds=(0.0, 1.0)), "min_doc_count and extended_bounds"),
                      (Hg.HistogramAggregation("f", 1.0, hard_bounds=(0.0, 5.0), extended_bounds=(0.0, 6.0)), "inside hard_bounds")):
        with pytest.raises(Hg.AggregationError, match=what):
            req.validate()
    with pytest.raises(Hg.AggregationError, match="sub-aggregations"):
        Hg.parse_request({"histogram": {"field": "f", "interval": 1.0}, "aggs": {"a": {"avg": {"field": "f"}}}})
    req, is_date = Hg.parse_request({"date_histogram": {"field": "d", "fixed_interval": "1h", "offset": "-30m", "hard_bounds": {"min": 0, "max": 10}}})
    assert is_date and (req.interval, req.offset, req.hard_bounds) == (3_600_000.0, -1_800_000.0, (0.0, 10.0))
    spec = Hg.histogram_spec(req, 7, "date")
    assert spec == (7, "date", 3.6e12, -1.8e12, 0.0, 1e7)
    assert Hg.histogram_spec(Hg.HistogramAggregation("f", 2.0), 1, "f64") == (1, "f64", 2.0, 0.0, -Hg.F64_MAX, Hg.F64_MAX)


def test_bucket_limit():
    req = Hg.HistogramAggregation("f", 1.0, extended_bounds=(0.0, 64999.0))
    assert len(Hg.finalize(req, {}, "f64")["buckets"]) == 65000
    with pytest.raises(Hg.AggregationError, match="bucket limit"):
        Hg.finalize(Hg.HistogramAggregation("f", 1.0, extended_bounds=(0.0, 65000.0)), {}, "f64")
    with pytest.raises(Hg.AggregationError, match="bucket limit"):
        Hg.finalize(Hg.HistogramAggregation("f", 1.0, min_doc_count=1), {i: 1 for i in range(65001)}, "f64")


def fixture_images(case):
    """The segments of a fixture as (u64 images, kind)."""
    out = []
    for seg in case["segments"]:
        if case["kind"] == "date":
            ns = np.array([np.datetime64(v.rstrip("Z"), "ns") for v in seg], dtype="datetime64[ns]")
            out.append(T.fast_value_to_u64(ns, "date"))
        else:
            out.append(T.fast_value_to_u64(np.array(seg, dtype=np.float64), "f64"))
    return out


def check_result(case, res):
    buckets = res["buckets"]
    if "expect" in case:
        assert res == case["expect"], case["name"]
    for i, key, count in case.get("checks", []):
        if key is not None:
            assert buckets[i]["key"] == key, (case["name"], i)
        if count is not None:
            assert buckets[i]["doc_count"] == count, (case["name"], i)
    for i, s in enumerate(case.get("key_as_string", [])):
        assert buckets[i]["key_as_string"] == s
    if "n_buckets" in case:
        assert len(buckets) == case["n_buckets"], case["name"]


def run_fixture_host(case):
    req, _ = Hg.parse_request(case["agg"])
    col, kind, interval, offset, lo, hi = Hg.histogram_spec(req, 0, case["kind"])
    parts = [HM.collect(im, None, None, kind, interval, offset, lo, hi) for im in fixture_images(case)]
    return Hg.finalize(req, Hg.merge_intermediate(p.items() for p in parts), kind)


@pytest.mark.parametrize("case", FIXTURES, ids=[c["name"] for c in FIXTURES])
def test_reference_fixtures(case):
    if "error" in case:
        with pytest.raises(Hg.AggregationError) as e:
            run_fixture_host(case)
        assert case["error"] in str(e.value)
        return
    check_result(case, run_fixture_host(case))


def test_collapse_rule():
    """hard_bounds [-inf, inf] over a column holding +inf and no NaN collapse to every finite value: the +inf doc is dropped; with a
    NaN in the column they do not collapse (its max image is the NaN) and the +inf doc counts, at the saturated pos."""
    im = T.fast_value_to_u64(np.array([1.0, np.inf, 2.0]), "f64")
    assert HM.collect(im, None, None, "f64", 1.0, 0.0, -np.inf, np.inf) == {1: 1, 2: 1}
    im = T.fast_value_to_u64(np.array([1.0, np.inf, np.nan]), "f64")
    assert HM.collect(im, None, None, "f64", 1.0, 0.0, -np.inf, np.inf) == {1: 1, 2**63 - 1: 1}
    assert HM.collect(im, None, None, "f64", 1.0, 0.0) == {1: 1}


def test_abi_symbols_and_specs():
    for name in ("tq_histogram_batch", "tq_get_histogram_stats"):
        assert hasattr(LIB, name)
    hdr = open(os.path.join(ROOT, "include", "tantivy_b200.h")).read()
    for i, k in enumerate(("U64", "I64", "F64", "BOOL", "DATE")):
        assert re.search(rf"#define TQ_FAST_{k} {i}u", hdr)
        assert getattr(_abi, f"TQ_FAST_{k}") == i == getattr(T, f"TQ_FAST_{k}")


def _layout(tmp_path, struct, fields):
    src = tmp_path / "off.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "tantivy_b200.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu\\n", offsetof({struct}, {n}));\n' for n in fields)
                   + f'  printf("%zu\\n", sizeof({struct}));\n  return 0;\n}}\n')
    exe = tmp_path / "off"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    return [int(x) for x in subprocess.check_output([str(exe)]).split()]


def test_spec_and_stats_layout_match_the_compiler(tmp_path):
    fields = [n for n, _ in _abi.HistogramSpec._fields_]
    assert fields == ["column_id", "kind", "interval", "offset", "hard_min", "hard_max"]
    assert _layout(tmp_path, "tq_histogram_spec", fields) == [getattr(_abi.HistogramSpec, n).offset for n in fields] + [C.sizeof(_abi.HistogramSpec)]
    assert [_abi.HISTOGRAM_SPEC_DTYPE.fields[n][1] for n in fields] == [getattr(_abi.HistogramSpec, n).offset for n in fields]
    fields = [n for n, _ in _abi.HistogramStats._fields_]
    assert fields == ["hist_ms", "units_hist", "hist_tiles_seen", "hist_tiles_one_bucket"]
    assert _layout(tmp_path, "tq_histogram_stats", fields) == [getattr(_abi.HistogramStats, n).offset for n in fields] + [C.sizeof(_abi.HistogramStats)]
