"""The request and result side of the device terms aggregation (tantivy_b200.terms) on the CPU: parsing, defaults, aliases and
refusals, the finaliser over the reference's terms tests transcribed as data (tests/golden/terms_fixtures.json) with each segment
collected and cut by tests/terms_model.py, and the C ABI of tq_terms_batch as mirrored by _abi.py."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import tantivy_b200 as T
from tantivy_b200 import _abi
from tantivy_b200 import terms as Tm
from tantivy_b200.lib import LIB
from tests import terms_model as TM
from tests.test_histogram_host import _layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = json.load(open(os.path.join(ROOT, "tests", "golden", "terms_fixtures.json")))["cases"]


def test_defaults_and_aliases():
    r = Tm.parse_request({"terms": {"field": "f"}})
    assert (r.size, r.segment_size, r.show_term_doc_count_error, r.min_doc_count, r.order_target, r.order) == (10, 100, True, 1, "_count", "desc")
    assert Tm.parse_request({"terms": {"field": "f", "size": 3}}).segment_size == 30
    assert Tm.parse_request({"terms": {"field": "f", "size": 30, "segment_size": 5}}).segment_size == 30  # max(size, segment_size)
    for alias in ("shard_size", "split_size", "segment_size"):
        assert Tm.parse_request({"terms": {"field": "f", alias: 7, "size": 2}}).segment_size == 7
    for order in ({"_count": "asc"}, {"_key": "desc"}, {"_key": "asc"}):
        assert Tm.parse_request({"terms": {"field": "f", "order": order}}).show_term_doc_count_error is False
    assert Tm.parse_request({"terms": {"field": "f", "order": {"_key": "asc"}, "show_term_doc_count_error": True}}).show_term_doc_count_error


def test_refusals_are_distinct():
    msgs = set()
    cases = [({"terms": {"field": "f"}, "aggs": {"a": {"avg": {"field": "g"}}}}, "str", {}),
             ({"terms": {"field": "f", "order": {"a": "desc"}}}, "str", {}),
             ({"terms": {"field": "f", "include": "a.*"}}, "str", {}),
             ({"terms": {"field": "f", "min_doc_count": 0}}, "str", {}),
             ({"terms": {"field": "f"}}, "str", {"multi_valued": True}),
             ({"terms": {"field": "f"}}, "str", {"n_columns": 2}),
             ({"terms": {"field": "f", "missing": "NA"}}, "u64", {}),
             ({"terms": {"field": "f"}}, "ip", {})]
    for agg, kind, extra in cases:
        with pytest.raises(Tm.TermsRefused) as e:
            Tm.check_device(Tm.parse_request(agg), kind, **extra)
        msgs.add(str(e.value))
    assert len(msgs) == len(cases)


def test_missing_images_and_keys():
    r = Tm.parse_request({"terms": {"field": "f", "missing": 5}})
    assert Tm.terms_spec(r, 3, "u64") == (3, T.TQ_TERMS_BY_COUNT, T.TQ_ORDER_DESC, 100, T.TQ_TERMS_MISSING_IMAGE, 5)
    assert Tm.terms_spec(r, 3, "i64")[5] == int(T.fast_value_to_u64(np.array([5]), "i64")[0])
    assert Tm.terms_spec(r, 3, "f64")[5] == int(T.fast_value_to_u64(np.array([5.0]), "f64")[0])
    assert Tm.terms_spec(r, 3, "str")[4] == T.TQ_TERMS_MISSING_AFTER_MAX
    assert Tm.intermediate_key(int(T.fast_value_to_u64(np.array([2.0]), "f64")[0]), "f64") == ("i64", 2)
    assert Tm.intermediate_key(int(T.fast_value_to_u64(np.array([2.5]), "f64")[0]), "f64") == ("f64", 2.5)
    assert Tm.intermediate_key(1, "bool") == ("bool", True)


def fixture_segments(case):
    """Each fixture segment as (u64 images, present mask, dictionary or None): a str segment's dictionary is its sorted distinct
    terms and its images their ordinals, numbers through fast_value_to_u64, dates from RFC 3339."""
    out = []
    for seg in case["segments"]:
        present = np.array([v is not None for v in seg], bool)
        vals = [v for v in seg if v is not None]
        kind, terms = case["kind"], None
        if kind == "str":
            terms = sorted(set(vals))
            have = np.array([terms.index(v) for v in vals], np.uint64)
        elif kind == "date":
            have = T.fast_value_to_u64(np.array([np.datetime64(v.rstrip("Z"), "ns") for v in vals], dtype="datetime64[ns]"), "date")
        elif kind == "u64":
            have = np.array(vals, np.uint64)
        elif kind == "bool":
            have = T.fast_value_to_u64(np.array(vals, bool), "bool")
        else:
            have = T.fast_value_to_u64(np.array(vals, np.float64 if kind == "f64" else np.int64), kind)
        images = np.zeros(len(seg), np.uint64)
        images[present] = np.asarray(have, np.uint64)
        out.append((images, present, terms))
    return out


def missing_image(spec, images, present):
    """The missing key a segment's docs without a value count under (get_missing_val_as_u64_lenient): the spec's image, or for a
    str column the segment's largest ordinal + 1 -- 0 + 1 without a value (EmptyColumnValues::max_value is 0)."""
    if spec[4] == T.TQ_TERMS_MISSING_NONE:
        return None
    if spec[4] == T.TQ_TERMS_MISSING_IMAGE:
        return spec[5]
    return (int(images[present].max()) if present.any() else 0) + 1


def run_fixture_host(case):
    req = Tm.parse_request(case["agg"])
    spec = Tm.terms_spec(req, 0, case["kind"])
    parts = []
    for images, present, terms in fixture_segments(case):
        mi = missing_image(spec, images, present)
        kept, err, other = TM.cut(TM.collect(images, present, None, mi), req.segment_size, req.order_target == "_key", req.order == "asc")
        parts.append((Tm.segment_result(req, case["kind"], kept, terms, mi), other, err))
    return Tm.finalize(req, Tm.merge(parts))


def check_result(case, res):
    b = res["buckets"]
    for i, key, count in case["checks"]:
        got = b[i]["key"]
        assert (got == key) if isinstance(key, str) else (not isinstance(got, str) and float(got) == float(key)), (case["name"], i, got)
        assert b[i]["doc_count"] == count, (case["name"], i)
    if "n_buckets" in case:
        assert len(b) == case["n_buckets"], case["name"]
    if "sum_other_doc_count" in case:
        assert res["sum_other_doc_count"] == case["sum_other_doc_count"], case["name"]
    if "doc_count_error_upper_bound" in case:
        assert res.get("doc_count_error_upper_bound") == case["doc_count_error_upper_bound"], case["name"]
    for i, st in enumerate(case.get("key_as_string", [])):
        assert b[i]["key_as_string"] == st


@pytest.mark.parametrize("case", FIXTURES, ids=[c["name"] for c in FIXTURES])
def test_reference_fixtures(case):
    if "refused" in case:
        with pytest.raises(Tm.TermsRefused, match=case["refused"]):
            run_fixture_host(case)
        return
    check_result(case, run_fixture_host(case))


def test_missing_key_of_a_segment_without_values():
    """A str segment without any value counts its docs under ordinal 0 + 1, the reference's empty column max + 1 (pinned by
    terms_aggregation_missing_empty); a segment with values under its largest ordinal + 1."""
    spec = Tm.terms_spec(Tm.parse_request({"terms": {"field": "t", "missing": "Empty"}}), 0, "str")
    assert missing_image(spec, np.zeros(3, np.uint64), np.zeros(3, bool)) == 1
    assert missing_image(spec, np.array([0, 4, 2], np.uint64), np.array([1, 1, 0], bool)) == 5


def test_finalize_rows_cuts_a_segment_split_over_contexts():
    """Two contexts each evaluate half of one segment and return it uncut; finalize_rows sums the halves and cuts once, as the
    reference cuts the whole segment."""
    req = Tm.parse_request({"terms": {"field": "t", "size": 1, "segment_size": 1}})
    a = (np.array([7, 7]), np.array([0, 1]), np.array([3, 1]), 2, 0, 0)  # segment 7: key 0 x3, key 1 x1
    b = (np.array([7, 7]), np.array([1, 2]), np.array([3, 2]), 2, 0, 0)  # key 1 x3, key 2 x2
    res = Tm.finalize_rows(req, "u64", [a, b])
    assert res == {"buckets": [{"key": 1, "doc_count": 4}], "sum_other_doc_count": 5, "doc_count_error_upper_bound": 3}


def test_model_tie_rule():
    assert TM.cut({1: 3, 2: 3, 3: 3, 4: 1}, 2) == ([(1, 3), (2, 3)], 3, 4)
    assert TM.cut({1: 3, 2: 3, 3: 1}, 2) == ([(1, 3), (2, 3)], 1, 1)
    assert TM.cut({1: 3, 2: 1, 3: 2}, 1, by_key=True, asc=False) == ([(3, 2)], 1, 4)


def test_spec_and_stats_layout_match_the_compiler(tmp_path):
    for name in ("tq_terms_batch", "tq_get_terms_stats"):
        assert hasattr(LIB, name)
    fields = [n for n, _ in _abi.TermsSpec._fields_]
    assert _layout(tmp_path, "tq_terms_spec", fields) == [getattr(_abi.TermsSpec, n).offset for n in fields] + [C.sizeof(_abi.TermsSpec)]
    assert [_abi.TERMS_SPEC_DTYPE.fields[n][1] for n in fields] == [getattr(_abi.TermsSpec, n).offset for n in fields]
    fields = [n for n, _ in _abi.TermsStats._fields_]
    assert fields == ["terms_ms", "units_terms", "terms_tiles_seen", "terms_tiles_one_key"]
    assert _layout(tmp_path, "tq_terms_stats", fields) == [getattr(_abi.TermsStats, n).offset for n in fields] + [C.sizeof(_abi.TermsStats)]
