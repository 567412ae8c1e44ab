"""Terms aggregations with metric sub-aggregations on the CPU side (tantivy_b200.terms_metrics): parsing and every refusal, the C ABI
of tq_terms_metrics_batch as mirrored by _abi.py, the merge and cut of a segment split over contexts, the metric order's tie rule in
the cut and in the final order, the guards (per bucket and on the order's total part) and the finaliser -- against
tests/terms_metrics_model.py.  Device rows are built here from the docs as the device builds them (part_of: the tq_metric_part of a
list of values)."""
import ctypes as C

import numpy as np
import pytest

import tantivy_b200 as T
from tantivy_b200 import _abi
from tantivy_b200 import metrics as Mx
from tantivy_b200 import terms as Tm
from tantivy_b200 import terms_metrics as TMx
from tantivy_b200.histogram import AggregationError
from tantivy_b200.lib import LIB
from tests import metrics_model as MM
from tests import terms_metrics_model as TMM
from tests.test_hist_metrics_host import part_of, same_tree
from tests.test_histogram_host import _layout

FIELDS = {"host": Mx.MetricField(1, "str"), "lat": Mx.MetricField(2, "u64"), "v": Mx.MetricField(3, "f64"), "ok": Mx.MetricField(4, "bool"),
          "tags": Mx.MetricField(5, "u64", multi_valued=True), "json": Mx.MetricField(6, "f64", n_column_types=2), "ip": Mx.MetricField(7, "ip"),
          "a": Mx.MetricField(8, "i64"), "b": Mx.MetricField(9, "i64"), "n": Mx.MetricField(10, "u64")}


def request(terms=None, aggs=None, name="t"):
    body = {"terms": terms or {"field": "host"}}
    if aggs is not None:
        body["aggs"] = aggs
    return {name: body}


AVG = {"m": {"avg": {"field": "v"}}}


def test_parse_and_plan():
    r = TMx.parse_request(request({"field": "n", "size": 3, "order": {"s.avg": "asc"}},
                                  {"s": {"stats": {"field": "v"}}, "c": {"value_count": {"field": "host"}}, "x": {"max": {"field": "lat"}}}))
    assert r.name == "t" and r.order == ("s", T.terms_metrics.TQ_TERMS_ORDER_AVG) and [m.name for m in r.metrics] == ["s", "c", "x"]
    p = TMx.plan(r, FIELDS)
    assert p.tspec == (10, T.TQ_TERMS_BY_METRIC, T.TQ_ORDER_ASC, 30, T.TQ_TERMS_MISSING_NONE, 0) and p.order == (0, _abi.TQ_TERMS_ORDER_AVG)
    assert len(p.mplan.columns) == 3 and p.mplan.columns[1][2] == T.TQ_METRIC_COUNT_ONLY
    for target, metric in (("x", _abi.TQ_TERMS_ORDER_MAX), ("c", _abi.TQ_TERMS_ORDER_COUNT), ("s.count", _abi.TQ_TERMS_ORDER_COUNT),
                           ("s.sum", _abi.TQ_TERMS_ORDER_SUM), ("s.min", _abi.TQ_TERMS_ORDER_MIN), ("s.max", _abi.TQ_TERMS_ORDER_MAX)):
        r = TMx.parse_request(request({"field": "host", "order": {target: "desc"}}, {"s": {"stats": {"field": "v"}},
                                      "c": {"value_count": {"field": "v"}}, "x": {"max": {"field": "lat"}}}))
        assert r.order[1] == metric and TMx.plan(r, FIELDS).order[1] == metric
    p = TMx.plan(TMx.parse_request(request({"field": "host", "missing": "NA", "order": {"_key": "asc"}}, AVG)), FIELDS)
    assert p.tspec == (1, T.TQ_TERMS_BY_KEY, T.TQ_ORDER_ASC, 100, T.TQ_TERMS_MISSING_AFTER_MAX, 0) and p.order is None
    p = TMx.plan(TMx.parse_request(request({"field": "n", "missing": 7}, {"m": {"sum": {"field": "v", "missing": 1.5}}})), FIELDS)
    assert p.tspec == (10, T.TQ_TERMS_BY_COUNT, T.TQ_ORDER_DESC, 100, T.TQ_TERMS_MISSING_IMAGE, 7) and p.mplan.columns[0][2] == T.TQ_METRIC_MISSING


@pytest.mark.parametrize("aggs,match", [
    (request(aggs={"h": {"histogram": {"field": "lat", "interval": 1}}}), "bucket aggregations nested under terms"),
    (request(aggs={"h": {"terms": {"field": "lat"}}}), "bucket aggregations nested under terms"),
    (request({"field": "host", "order": {"c": "desc"}}, {"c": {"cardinality": {"field": "lat"}}}), "ordering by a cardinality"),
    (request({"field": "host", "order": {"p": "desc"}}, {"p": {"percentiles": {"field": "lat"}}}), "ordering by a percentiles"),
    (request({"field": "host", "order": {"e.avg": "desc"}}, {"e": {"extended_stats": {"field": "lat"}}}), "ordering by a extended_stats"),
    (request({"field": "host", "order": {"h": "desc"}}, {"h": {"top_hits": {"size": 1}}}), "ordering by a top_hits"),
    (request({"field": "host", "order": {"s": "desc"}}, {"s": {"stats": {"field": "lat"}}}), "without a property"),
    (request({"field": "host", "order": {"s.median": "desc"}}, {"s": {"stats": {"field": "lat"}}}), "unknown stats property"),
    (request({"field": "host", "order": {"m.value": "desc"}}, AVG), "property 'm.value' of a single-value metric"),
    (request(aggs={"e": {"cardinality": {"field": "lat"}}}), "cardinality runs on the CPU path"),
    (request(aggs={"e": {"avg": {"field": "lat"}, "aggs": {"x": {"max": {"field": "lat"}}}}}), "sub-aggregations run on the CPU path"),
    (dict(request(aggs=AVG), x={"avg": {"field": "lat"}}), "more than one top-level"),
    (request(), "without sub-aggregations"),
    ({"h": {"histogram": {"field": "lat", "interval": 1}, "aggs": AVG}}, "not a terms aggregation"),
])
def test_parse_refusals(aggs, match):
    with pytest.raises(TMx.TermsMetricsRefused, match=match):
        TMx.parse_request(aggs)


@pytest.mark.parametrize("terms,aggs,match", [
    ({"field": "host", "include": "a.*"}, AVG, "include / exclude"),
    ({"field": "host", "exclude": ["a"]}, AVG, "include / exclude"),
    ({"field": "host", "min_doc_count": 0}, AVG, "min_doc_count 0"),
    ({"field": "tags"}, AVG, "multi-valued"),
    ({"field": "json"}, AVG, "several columns"),
    ({"field": "ip"}, AVG, "ip columns"),
    ({"field": "nope"}, AVG, "no registered fast column"),
    ({"field": "host"}, {"m": {"avg": {"field": "tags"}}}, "multi-valued columns"),
    ({"field": "host"}, {k: {"sum": {"field": f}} for k, f in zip("pqrst", ("lat", "v", "a", "b", "n"))}, "more than 4 distinct"),
    ({"field": "host", "order": {"m": "desc"}}, {k: {"sum": {"field": f}} for k, f in zip("pqrsm", ("lat", "v", "a", "b", "n"))}, "more than 4"),
])
def test_plan_refusals(terms, aggs, match):
    r = TMx.parse_request(request(terms, aggs))
    with pytest.raises(TMx.TermsMetricsRefused, match=match):
        TMx.plan(r, FIELDS)


def test_malformed_requests():
    for agg in (request({"field": "host", "order": {"nope": "desc"}}, AVG), request({"field": "host", "order": {"nope.avg": "asc"}}, AVG),
                request({"field": "host", "order": {"m": "up"}}, AVG), request(aggs={"m": {"avg": {}}}), request({"field": "host", "sise": 3}, AVG),
                [], {}):
        with pytest.raises(AggregationError):
            TMx.parse_request(agg)
    with pytest.raises(AggregationError, match="could not find aggregation with name nope"):
        TMx.parse_request(request({"field": "host", "order": {"nope": "desc"}}, AVG))


def test_abi_symbols_and_layouts(tmp_path):
    for name in ("tq_terms_metrics_batch", "tq_get_terms_metrics_stats"):
        assert hasattr(LIB, name)
    fields = [n for n, _ in _abi.TermsMetricsStats._fields_]
    assert fields == ["terms_metrics_ms", "units_terms_metrics", "terms_metrics_tiles_seen", "terms_metrics_tiles_one_key", "terms_metrics_waves"]
    assert _layout(tmp_path, "tq_terms_metrics_stats", fields) == [getattr(_abi.TermsMetricsStats, n).offset for n in fields] + [C.sizeof(_abi.TermsMetricsStats)]
    assert _layout(tmp_path, "tq_terms_metric_order", ["column", "metric"]) == [0, 4, 8]
    assert (_abi.TQ_TERMS_BY_METRIC, _abi.TQ_TERMS_ORDER_COUNT, _abi.TQ_TERMS_ORDER_SUM, _abi.TQ_TERMS_ORDER_AVG, _abi.TQ_TERMS_ORDER_MIN,
            _abi.TQ_TERMS_ORDER_MAX) == (2, 0, 1, 2, 3, 4)
    assert T.TermsMetricsRefused is TMx.TermsMetricsRefused


# ---- rows as the device builds them ---------------------------------------------------------------------------------------------
def f64_plan(terms, aggs=None):
    return TMx.plan(TMx.parse_request(request(dict({"field": "n"}, **terms), aggs or {"m": {"avg": {"field": "v"}}})), FIELDS)


def parts_of(values):
    parts = Mx.empty_parts()
    parts[0] = part_of(values)
    return parts


def out_of(rows, other=0, error=0, order_values=None):
    """One query of Context.terms_metrics_batch's output from [(segment_ord, image, [column 0 values][, doc_count])] (doc_count:
    the number of values unless given)."""
    n = len(rows)
    segs = np.array([[r[0] for r in rows]], np.uint32).reshape(1, n)
    keys = np.array([[r[1] for r in rows]], np.uint64).reshape(1, n)
    counts = np.array([[r[3] if len(r) > 3 else len(r[2]) for r in rows]], np.uint64).reshape(1, n)
    parts = np.stack([parts_of(r[2]) for r in rows]).reshape(1, n, -1) if n else np.zeros((1, 0, 4), Mx.METRIC_PART_DTYPE)
    opart = part_of(order_values if order_values is not None else [x for r in rows for x in r[2]])
    return (segs, keys, counts, parts, np.array([n], np.uint32), np.array([other], np.uint64), np.array([error], np.uint64),
            np.array([opart]))


def test_cut_tie_rule_minus_zero_and_unwrap_or():
    """The segment cut: -0.0 equals +0.0 and a key with docs but no values is 0.0 (unwrap_or(0.0)), equal values keep the lowest
    keys, the scalars follow that order; the final order: -0.0 before +0.0 (total_cmp) and a key without values at f64::MIN."""
    p = f64_plan({"size": 3, "segment_size": 3, "order": {"m": "desc"}}, {"m": {"min": {"field": "v"}}})
    entries = {0: (5, parts_of([0.0])), 1: (4, parts_of([-0.0])), 2: (3, parts_of([])), 3: (2, parts_of([0.0])), 4: (1, parts_of([-1.0]))}
    kept, e, o = TMx.cut_segment(p, entries)
    assert sorted(kept) == [0, 1, 2] and (e, o) == (2, 3)  # four entries at 0.0, the lowest keys kept; key 3 at position 3
    model = {k: (c, {"m": MM.segment_stats(v)}) for k, (c, v) in
             {0: (5, [0.0]), 1: (4, [-0.0]), 2: (3, []), 3: (2, [0.0]), 4: (1, [-1.0])}.items()}
    mk, me, mo = TMM.cut(model, 3, "metric", False, ("m", "min"))
    assert sorted(mk) == [0, 1, 2] and (me, mo) == (e, o)
    # asc: -1.0 first, then the 0.0 ties by key
    p_asc = f64_plan({"size": 2, "segment_size": 2, "order": {"m": "asc"}}, {"m": {"min": {"field": "v"}}})
    kept, e, o = TMx.cut_segment(p_asc, entries)
    assert sorted(kept) == [0, 4] and (e, o) == (4, 9)
    # the final order: +0.0, -0.0, then f64::MIN for the key without values (desc); ties by key ascending
    p = f64_plan({"size": 10, "order": {"m": "desc"}}, {"m": {"min": {"field": "v"}}})
    res = TMx.finalize(p, ({("u64", k): v for k, v in entries.items()}, 0, 0))
    assert [b["key"] for b in res["t"]["buckets"]] == [0, 3, 1, 4, 2] and res["t"]["buckets"][4]["m"] == {"value": None}
    assert "doc_count_error_upper_bound" not in res["t"]
    merged = ({("u64", k): (c, {"m": MM.segment_stats(v)}) for k, (c, v) in
               {0: (5, [0.0]), 1: (4, [-0.0]), 2: (3, []), 3: (2, [0.0]), 4: (1, [-1.0])}.items()}, 0, 0)
    assert same_tree(res, TMM.final("t", p.request.req, merged, [("m", "min", "m", False)], ("m", "min")))


def test_count_and_key_cuts_are_terms_cuts():
    for terms in ({"segment_size": 2}, {"segment_size": 2, "order": {"_count": "asc"}}, {"segment_size": 3, "order": {"_key": "desc"}}):
        p = f64_plan(terms)
        entries = {k: (c, parts_of([1.0] * c)) for k, c in {5: 3, 1: 3, 9: 1, 2: 7, 4: 3}.items()}
        kept, e, o = TMx.cut_segment(p, entries)
        tk, te, to = Tm.cut_segment({k: c for k, (c, _) in entries.items()}, p.request.req)
        assert sorted(kept) == [k for k, _ in tk] and (e, o) == (te, to)


def test_split_segment_merged_then_cut_once():
    """A segment in two contexts comes back uncut from each: its counts add and parts merge by key before the one cut; a whole
    segment passes through; the scalars of whole segments add."""
    p = f64_plan({"size": 2, "segment_size": 2, "order": {"m": "desc"}})
    a = out_of([(0, 1, [1.0, 3.0]), (0, 2, [10.0]), (0, 3, [2.0])])
    b = out_of([(0, 1, [5.0]), (0, 3, [20.0, 4.0]), (1, 7, [0.5])], other=4, error=1)
    per, other, error, total = TMx.segment_entries(p, [TMx.rows_of(a, 0), TMx.rows_of(b, 0)])
    assert (other, error) == (4, 1) and int(total["count"]) == 8 and float(total["sum"]) == 45.5
    assert {k: c for k, (c, _) in per[0].items()} == {1: 3, 2: 1, 3: 3} and float(per[0][3][1][0]["sum"]) == 26.0
    res = TMx.finalize_rows(p, [TMx.rows_of(a, 0), TMx.rows_of(b, 0)])
    # segment 0 averages: 1 -> 3.0, 2 -> 10.0, 3 -> 26/3; kept 2 and 3, key 1 (3 docs) cut; segment 1 keeps key 7
    assert [(x["key"], x["doc_count"]) for x in res["t"]["buckets"]] == [(2, 1), (3, 3)]
    assert res["t"]["sum_other_doc_count"] == 4 + 3 + 1 and res["t"]["buckets"][1]["m"] == {"value": 26.0 / 3}


def test_guards_per_bucket_and_on_the_order():
    aggs = {"s": {"sum": {"field": "v"}}, "mx": {"max": {"field": "v"}}}
    p = f64_plan({"size": 5}, aggs)
    out = out_of([(0, 1, [0.25, 0.5]), (0, 2, [2.1, 2.2, 2.3]), (0, 3, [1.0])])
    with pytest.raises(TMx.TermsMetricsRefused) as e:
        TMx.finalize_rows(p, [TMx.rows_of(out, 0)])
    assert set(e.value.refused) == {"s"} and "bucket 2" in e.value.refused["s"]
    b = e.value.answered["t"]["buckets"]
    assert [x["key"] for x in b] == [2, 1, 3] and all("s" not in x for x in b) and b[0]["mx"] == {"value": 2.3}
    # the failing bucket cut away by size: answered
    res = TMx.finalize_rows(f64_plan({"size": 1, "order": {"_key": "asc"}}, aggs), [TMx.rows_of(out, 0)])
    assert res["t"]["buckets"][0]["s"] == {"value": 0.75}
    # an order by sum / avg whose total part fails the guard, or any order on a column that saw a NaN: refused as a whole
    for order in ({"s": "desc"}, {"s": "asc"}):
        with pytest.raises(TMx.TermsMetricsRefused, match="the order's sums") as e:
            TMx.finalize_rows(f64_plan({"size": 1, "order": order}, aggs), [TMx.rows_of(out, 0)])
        assert not e.value.answered
    ok = out_of([(0, 1, [0.25]), (0, 3, [1.0])], order_values=[0.25, 1.0, 0.1])  # (a cut entry's decimal, in the total part only)
    with pytest.raises(TMx.TermsMetricsRefused, match="the order's sums"):
        TMx.finalize_rows(f64_plan({"size": 1, "order": {"s": "desc"}}, aggs), [TMx.rows_of(ok, 0)])
    res = TMx.finalize_rows(f64_plan({"size": 1, "order": {"mx": "desc"}}, aggs), [TMx.rows_of(ok, 0)])  # max needs no sum guard
    assert res["t"]["buckets"][0]["key"] == 3
    nan = out_of([(0, 1, [0.25]), (0, 3, [float("nan")])])
    with pytest.raises(TMx.TermsMetricsRefused, match="NaN"):
        TMx.finalize_rows(f64_plan({"size": 1, "order": {"mx": "desc"}}, aggs), [TMx.rows_of(nan, 0)])


def test_finalize_shapes_against_model():
    """Every metric type and order through finalize_rows and through the model, on a str column with `missing` (the missing key
    inserted first, so that a term of the same text replaces it) over two segments."""
    aggs = {"st": {"stats": {"field": "v"}}, "sn": {"sum": {"field": "v", "none_if_no_match": True}}, "a": {"avg": {"field": "v"}},
            "mn": {"min": {"field": "v"}}, "c": {"value_count": {"field": "v"}}}
    dicts = {0: ["x", "y", "NA"], 1: ["y", "z"]}
    # (image 3 / 2: the missing key; image 1 has docs but no value)
    seg_rows = {0: {0: [1.0, 2.0], 1: [], 2: [4.0], 3: [0.5]}, 1: {0: [3.0, 8.0, 1.0], 1: [], 2: [2.0]}}
    doc_count = lambda v: len(v) or 2  # noqa: E731
    for order in ({"_count": "desc"}, {"_key": "asc"}, {"a": "desc"}, {"st.min": "asc"}, {"sn": "asc"}, {"c": "desc"}, {"st.max": "desc"}):
        p = TMx.plan(TMx.parse_request(request({"field": "host", "size": 3, "missing": "NA", "order": order}, aggs)), FIELDS)
        rows = out_of([(s, k, v, doc_count(v)) for s in (0, 1) for k, v in seg_rows[s].items()])
        got = TMx.finalize_rows(p, [TMx.rows_of(rows, 0)], dicts, {0: 3, 1: 2})
        results = []
        for s in (0, 1):
            seg = {}
            for k, v in sorted(seg_rows[s].items()):
                st = MM.segment_stats(v)
                entry = (doc_count(v), {"v": st})
                key = ("str", "NA") if k == {0: 3, 1: 2}[s] else ("str", dicts[s][k])
                if k == {0: 3, 1: 2}[s]:
                    seg = dict([(key, entry)] + list(seg.items()))
                else:
                    seg[key] = entry
            results.append((seg, 0, 0))
        target = next(iter(order))
        name, _, prop = target.partition(".")
        mo = None if target in ("_count", "_key") else (name, prop or {"c": "count", "sn": "sum", "a": "avg", "mn": "min"}[name])
        want = TMM.final("t", p.request.req, TMM.merge(results), [(n, next(iter(a)), "v", n == "sn") for n, a in aggs.items()], mo)
        assert same_tree(got, want), order


def test_empty_and_min_doc_count():
    p = f64_plan({"min_doc_count": 2})
    assert TMx.finalize_rows(p, [TMx.rows_of(out_of([]), 0)]) == {"t": {"buckets": [], "sum_other_doc_count": 0, "doc_count_error_upper_bound": 0}}
    res = TMx.finalize_rows(p, [TMx.rows_of(out_of([(0, 1, [1.0]), (0, 2, [1.0, 2.0])]), 0)])
    assert [b["key"] for b in res["t"]["buckets"]] == [2] and res["t"]["sum_other_doc_count"] == 0
