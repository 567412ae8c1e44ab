"""The request and result side of metric aggregations (src/aggregation/metric/: avg, sum, min, max, stats, value_count), for the
device's intermediate results (Context.metrics_batch).  Pure Python: it parses a request of top-level metric aggregations, refuses
what the device does not run (MetricsRefused: take the CPU path), maps the request's fields to one spec of up to four columns,
merges the parts of any number of contexts, applies the exactness guard and finalises to tantivy's result: {"value": x} per
single-value metric, {"count", "sum", "min", "max", "avg"} per stats.

The device sums in no particular order; the reference sums with Kahan summation in doc order.  The two agree bit for bit when
every partial sum is exact, which the guard proves from the part's magnitude and quantum (tantivy_b200.h, DESIGN §3.8).  A sum,
avg or stats whose figures fail the guard, or that saw a NaN or an infinity, is refused; min, max and value_count never depend on
the order and are always answered."""
import math
from dataclasses import dataclass, field as dc_field
from typing import Optional

import numpy as np

from ._abi import (METRIC_PART_DTYPE, TQ_FAST_BOOL, TQ_FAST_DATE, TQ_FAST_F64, TQ_FAST_I64, TQ_FAST_U64, TQ_METRIC_COUNT_ONLY, TQ_METRIC_EMPTY, TQ_METRIC_MISSING,
                   TQ_METRICS_MAX_COLUMNS)
from .histogram import AggregationError
from .terms import _f64_of_image, _missing_image

METRIC_TYPES = ("avg", "sum", "min", "max", "stats", "value_count")
SUM_BEARING = ("avg", "sum", "stats")
_CPU_METRICS = {
    "extended_stats": "extended_stats sums squares, which needs a guard of its own: the CPU path",
    "percentiles": "percentiles run on the CPU path",
    "cardinality": "cardinality runs on the CPU path",
    "top_hits": "top_hits runs on the CPU path",
}
_BUCKETS = ("terms", "histogram", "date_histogram", "range", "date_range", "filter", "filters", "composite")
# The column types a metric reads (agg_data.rs:529-543): numbers and dates (get_numeric_or_date_column_types); value_count reads
# str, bool and ip too, and those collect 0.0 per value (is_number_or_date_type false, stats.rs:372-375).  A field of no readable
# type is an empty U64 column.
_VALUE_KINDS = {"u64": TQ_FAST_U64, "i64": TQ_FAST_I64, "f64": TQ_FAST_F64, "date": TQ_FAST_DATE}
_OTHER_KINDS = ("bool", "str", "bytes", "ip")
F64_MAX = 1.7976931348623157e308
_U64_MAX = (1 << 64) - 1
_HIGH = 1 << 63
INT32_MAX = 2**31 - 1


class MetricsRefused(ValueError):
    """A metrics request, or some of its aggregations, that the device does not answer exactly; the caller takes the CPU path.
    `refused` maps each refused aggregation's name to the reason; `answered` holds the final results of the others (finalize)."""

    def __init__(self, message, refused=None, answered=None):
        super().__init__(message)
        self.refused = refused or {}
        self.answered = answered or {}


@dataclass
class MetricAggregation:
    """One metric aggregation: its name in the request, its type, and the reference's parameters."""
    name: str
    type: str
    field: str
    missing: Optional[float] = None  # deserialize_option_f64: a number or a numeric string
    none_if_no_match: bool = False   # sum only (sum.rs:30-39)


@dataclass
class MetricField:
    """What the caller knows of a field in the segments it searches: the registered column, its type ("u64", "i64", "f64", "date",
    "bool", "str", "bytes", "ip"), whether it is multi-valued and how many column types it has (a JSON field may have several)."""
    column_id: int
    kind: str
    multi_valued: bool = False
    n_column_types: int = 1


@dataclass
class MetricsPlan:
    """The spec columns of a request and, per aggregation, the index of its column."""
    aggs: list
    columns: list = dc_field(default_factory=list)  # (column_id, TQ_FAST_*, TQ_METRIC_* flags, missing_image) per spec column
    kinds: list = dc_field(default_factory=list)    # the field type of each spec column
    slot: dict = dc_field(default_factory=dict)     # aggregation name -> spec column


def _parse_missing(v):
    if v is None:
        return None
    if isinstance(v, bool):
        raise AggregationError(f"missing {v!r} is not a number")
    if isinstance(v, (int, float)):
        return float(v)
    if isinstance(v, str):
        try:
            return float(v)
        except ValueError:
            raise AggregationError(f"missing {v!r} is not a number") from None
    raise AggregationError(f"missing {v!r} is not a number")


def parse_request(aggs):
    """An Aggregations map {name: {type: {...}}} of top-level metric aggregations -> [MetricAggregation].  Every request the
    device does not run raises MetricsRefused with its own message; a malformed one AggregationError."""
    if not isinstance(aggs, dict) or not aggs:
        raise AggregationError("expected a non-empty map of aggregations")
    out = []
    for name, agg in aggs.items():
        if not isinstance(agg, dict):
            raise AggregationError(f"aggregation {name!r} is not an object")
        if "aggs" in agg or "aggregations" in agg:
            raise MetricsRefused(f"{name}: sub-aggregations run on the CPU path")
        if len(agg) != 1:
            raise AggregationError(f"aggregation {name!r} must have exactly one type")
        (typ, body), = agg.items()
        if typ in _CPU_METRICS:
            raise MetricsRefused(f"{name}: {_CPU_METRICS[typ]}")
        if typ in _BUCKETS:
            raise MetricsRefused(f"{name}: a bucket aggregation ({typ}) mixed in with the metrics runs on the CPU path")
        if typ not in METRIC_TYPES:
            raise AggregationError(f"unknown aggregation type {typ!r}")
        if not isinstance(body, dict) or "field" not in body:
            raise AggregationError(f"{name}: missing field `field`")
        known = {"field", "missing"} | ({"none_if_no_match"} if typ == "sum" else set())
        unknown = set(body) - known
        if unknown:
            raise AggregationError(f"{name}: unknown {typ} parameter(s) {sorted(unknown)}")
        nim = body.get("none_if_no_match")
        out.append(MetricAggregation(name=name, type=typ, field=body["field"], missing=_parse_missing(body.get("missing")),
                                     none_if_no_match=bool(nim) if nim is not None else False))
    return out


def plan(aggs, fields):
    """[MetricAggregation] and {field name: MetricField} -> MetricsPlan: one spec column per distinct (field, missing), up to
    TQ_METRICS_MAX_COLUMNS of them, so that metrics on one field share a column."""
    p = MetricsPlan(aggs=list(aggs))
    index = {}
    for a in p.aggs:
        f = fields.get(a.field)
        if f is None:
            raise MetricsRefused(f"{a.name}: field {a.field!r} has no registered fast column")
        if f.n_column_types != 1:
            raise MetricsRefused(f"{a.name}: a field of several column types (JSON) runs on the CPU path")
        if f.multi_valued:
            raise MetricsRefused(f"{a.name}: multi-valued columns run on the CPU path")
        if f.kind not in _VALUE_KINDS and f.kind not in _OTHER_KINDS:
            raise MetricsRefused(f"{a.name}: {f.kind} columns run on the CPU path")
        column_id, image = f.column_id, 0
        if f.kind in _VALUE_KINDS:
            kind, flags, mtype = _VALUE_KINDS[f.kind], 0, f.kind
        elif a.type == "value_count" and f.kind != "bytes":  # Count reads str, bool and ip columns as 0.0 per value
            kind, flags, mtype = (TQ_FAST_BOOL if f.kind == "bool" else TQ_FAST_U64), TQ_METRIC_COUNT_ONLY, f.kind
        else:  # get_ff_reader finds no column of an allowed type: an empty U64 column (accessor_helpers.rs:59-74)
            column_id, kind, flags, mtype = 0, TQ_FAST_U64, TQ_METRIC_EMPTY, "u64"
        # missing_u64 = f64_to_fastfield_u64(m, type) (agg_data.rs:568, aggregation/mod.rs:394-402): None for str and ip
        if a.missing is not None and mtype not in ("str", "ip"):
            flags |= TQ_METRIC_MISSING
            image = _missing_image(a.missing, "u64" if mtype == "bool" else mtype)
        key = (column_id, kind, flags, image)
        if key not in index:
            if len(p.columns) == TQ_METRICS_MAX_COLUMNS:
                raise MetricsRefused(f"{a.name}: more than {TQ_METRICS_MAX_COLUMNS} distinct fields in one request run on the CPU path")
            index[key] = len(p.columns)
            p.columns.append(key)
            p.kinds.append(f.kind)
        p.slot[a.name] = index[key]
    return p


def empty_parts(n=TQ_METRICS_MAX_COLUMNS):
    parts = np.zeros(n, dtype=METRIC_PART_DTYPE)
    parts["min_image"] = _U64_MAX
    parts["quantum_exp"] = INT32_MAX
    return parts


def merge(parts_list):
    """Merges the parts of one query from any number of contexts (each [TQ_METRICS_MAX_COLUMNS] of METRIC_PART_DTYPE): counts add,
    images take min / max, sums add, quantum_exp takes the min."""
    out = empty_parts()
    for parts in parts_list:
        out["count"] += parts["count"]
        out["n_nan"] += parts["n_nan"]
        out["n_inf"] += parts["n_inf"]
        out["min_image"] = np.minimum(out["min_image"], parts["min_image"])
        out["max_image"] = np.maximum(out["max_image"], parts["max_image"])
        out["sum"] += parts["sum"]
        out["magnitude"] += parts["magnitude"]
        out["quantum_exp"] = np.minimum(out["quantum_exp"], parts["quantum_exp"])
    return out


def guard(part):
    """None when the part's sum is the reference's Kahan sum bit for bit, else the reason it may not be."""
    if int(part["n_nan"]):
        return "a NaN value makes the sum depend on the order"
    if int(part["n_inf"]):
        return "an infinite value makes Kahan's sum depend on where it falls"
    q = int(part["quantum_exp"])
    mag = float(part["magnitude"])
    if q == INT32_MAX:  # no finite non-zero value: every partial sum is zero
        return None
    if 53 + q > 1023:
        return None if math.isfinite(mag) else "the sum of |v| overflows"
    if mag < math.ldexp(1.0, 53 + q):
        return None
    return f"the sum of |v| reaches 2^{53 + q}: a partial sum may round, so the order matters"


def value_of_image(image, kind):
    """f64_from_fastfield_u64 (aggregation/mod.rs:374) of a u64 image of a TQ_FAST_* column."""
    image = int(image)
    if kind == TQ_FAST_F64:
        return _f64_of_image(image)
    if kind in (TQ_FAST_I64, TQ_FAST_DATE):
        return float(image - _HIGH)
    return float(image)


def stats_of(part, kind, flags):
    """(count, sum, min, max) of a part, with the reference's starting values for min / max (f64::MAX / f64::MIN) when no value
    lowers or raises them; min / max None when count is 0."""
    count = int(part["count"])
    if count == 0:
        return 0, 0.0, None, None
    if flags & TQ_METRIC_COUNT_ONLY:
        return count, 0.0, 0.0, 0.0
    lo, hi = int(part["min_image"]), int(part["max_image"])
    if lo > hi:  # every value NaN
        return count, float(part["sum"]), F64_MAX, -F64_MAX
    vmin, vmax = value_of_image(lo, kind), value_of_image(hi, kind)
    return count, float(part["sum"]), min(F64_MAX, vmin), max(-F64_MAX, vmax)


def finalize(p: MetricsPlan, merged):
    """{name: final result} of the plan's aggregations from merge()'s parts (into_final_metric_result,
    intermediate_agg_result.rs:425-462).  Raises MetricsRefused (with `refused` and `answered`) when some sum-bearing aggregation
    fails the guard."""
    answered, refused = {}, {}
    for a in p.aggs:
        i = p.slot[a.name]
        _, kind, flags, _ = p.columns[i]
        part = merged[i]
        count, s, vmin, vmax = stats_of(part, kind, flags)
        if a.type in SUM_BEARING and not flags & TQ_METRIC_COUNT_ONLY:
            why = guard(part)
            if why is not None:
                refused[a.name] = why
                continue
        avg = s / count if count else None
        if a.type == "stats":
            answered[a.name] = {"count": count, "sum": s, "min": vmin, "max": vmax, "avg": avg}
        elif a.type == "sum":
            answered[a.name] = {"value": None if count == 0 and a.none_if_no_match else s}
        elif a.type == "avg":
            answered[a.name] = {"value": avg}
        elif a.type == "min":
            answered[a.name] = {"value": vmin}
        elif a.type == "max":
            answered[a.name] = {"value": vmax}
        else:  # value_count
            answered[a.name] = {"value": float(count)}
    if refused:
        raise MetricsRefused("; ".join(f"{n}: {why}" for n, why in refused.items()), refused=refused, answered=answered)
    return answered


def run(contexts, qb, requests, fields, count_hits=False):
    """Runs one parsed request per query of qb over every Context (each evaluating its own segments or doc ranges) and finalises.
    Returns [{name: result} or MetricsRefused] per query, and the merged hit counts with count_hits."""
    plans = [plan(r, fields) for r in requests]
    specs = [p.columns for p in plans]
    per_ctx, hits = [], np.zeros(qb.nq, dtype=np.uint64)
    for ctx in contexts:
        if count_hits:
            parts, h = ctx.metrics_batch(qb, specs, count_hits=True)
            hits += h
        else:
            parts = ctx.metrics_batch(qb, specs)
        per_ctx.append(parts)
    out = []
    for q, p in enumerate(plans):
        try:
            out.append(finalize(p, merge(parts[q] for parts in per_ctx)))
        except MetricsRefused as e:
            out.append(e)
    return (out, hits) if count_hits else out
