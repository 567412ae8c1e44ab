"""The request and result side of a `range` aggregation (bucket/range.rs), with or without metric sub-aggregations (avg, sum, min,
max, stats, value_count), for the device's intermediate results (Context.range_batch).  Pure Python: it parses a request of one
top-level range, refuses what the device does not run (RangeRefused: take the CPU path), converts and extends the ranges in image
space as extend_validate_ranges does, merges the rows of any number of contexts by bucket, applies the exactness guard per (bucket,
column) and finalises to tantivy's result.

A range reads its field through get_numeric_or_date_column_types(): u64, i64, f64 and date columns.  A doc with a value goes to the
bucket whose start is the last one <= its image (get_bucket_pos; the end is never tested); a doc without one is not collected.  The
intermediate buckets are keyed by range_to_string(start..end), the final key is the custom key when given, and the final buckets are
sorted by `from` (f64::MIN when open) under total_cmp.  A bucket's metrics collect exactly the docs it counts.  When some bucket's
sum, avg or stats fails the guard, that aggregation is refused for the whole range; the others stay answered."""
from dataclasses import dataclass

import numpy as np

from . import metrics as Mx
from ._abi import TQ_FAST_U64, TQ_METRIC_EMPTY
from .histogram import AggregationError, _total_order, format_date, rust_f64_display

TQ_RANGE_MAX_BUCKETS = 128
_RANGE_KINDS = ("u64", "i64", "f64", "date")
_U64_MAX = (1 << 64) - 1
_HIGH = 1 << 63
_F64_MIN = -float(np.finfo(np.float64).max)


class RangeRefused(ValueError):
    """A range request, or some of its sub-aggregations, that the device does not answer exactly; the caller takes the CPU path.
    `refused` maps each refused sub-aggregation's name to the reason; `answered` holds the range's final result with the other
    sub-aggregations ({name: result}), when there is one."""

    def __init__(self, message, refused=None, answered=None):
        super().__init__(message)
        self.refused = refused or {}
        self.answered = answered or {}


@dataclass
class RangeRequest:
    """One top-level range: its name, field, ranges [(key | None, from | None, to | None)], keyed, and its metric
    sub-aggregations (metrics.MetricAggregation; empty: doc counts only)."""
    name: str
    field: str
    ranges: list
    keyed: bool
    metrics: list


@dataclass
class RangePlan:
    """The range's field type, its spec for Context.range_batch ((column_id, starts)), its buckets in start order (key, from, to,
    from_as_string, to_as_string) and the metrics plan of its sub-aggregations (None without)."""
    request: RangeRequest
    kind: str
    rspec: tuple
    buckets: list
    mplan: object


def _bound(v, what):
    if v is None:
        return None
    if isinstance(v, bool):
        raise AggregationError(f"range `{what}` {v!r} is not a number")
    if isinstance(v, (int, float)):
        return float(v)
    if isinstance(v, str):
        try:
            return float(v)
        except ValueError:
            raise AggregationError(f"range `{what}` {v!r} is not a number") from None
    raise AggregationError(f"range `{what}` {v!r} is not a number")


def parse_request(aggs):
    """An Aggregations map {name: {"range": {...}, "aggs"?: {...}}} -> RangeRequest.  Every request the device does not run raises
    RangeRefused with its own message; a malformed one AggregationError."""
    if not isinstance(aggs, dict) or not aggs:
        raise AggregationError("expected a non-empty map of aggregations")
    if len(aggs) != 1:
        raise RangeRefused("more than one top-level aggregation runs on the CPU path")
    (name, agg), = aggs.items()
    if not isinstance(agg, dict):
        raise AggregationError(f"aggregation {name!r} is not an object")
    if "aggs" in agg and "aggregations" in agg:
        raise AggregationError(f"{name}: both `aggs` and `aggregations`")
    sub = agg.get("aggs", agg.get("aggregations"))
    types = [k for k in agg if k not in ("aggs", "aggregations")]
    if len(types) != 1:
        raise AggregationError(f"aggregation {name!r} must have exactly one type")
    if types[0] != "range":
        raise RangeRefused(f"{name}: a top-level {types[0]} is not a range aggregation")
    body = agg["range"]
    if not isinstance(body, dict) or "field" not in body or "ranges" not in body:
        raise AggregationError(f"{name}: a range needs `field` and `ranges`")
    unknown = set(body) - {"field", "ranges", "keyed"}
    if unknown:
        raise AggregationError(f"{name}: unknown range parameter(s) {sorted(unknown)}")
    if not isinstance(body["ranges"], list):
        raise AggregationError(f"{name}: `ranges` is not a list")
    if not body["ranges"]:
        raise AggregationError(f"{name}: a range aggregation needs at least one range")
    ranges = []
    for r in body["ranges"]:
        if not isinstance(r, dict) or set(r) - {"key", "from", "to"}:
            raise AggregationError(f"{name}: a range is an object of `key`, `from` and `to`")
        key = r.get("key")
        if key is not None and not isinstance(key, str):
            raise AggregationError(f"{name}: a range key must be a string")
        ranges.append((key, _bound(r.get("from"), "from"), _bound(r.get("to"), "to")))
    metrics = []
    if sub:
        if not isinstance(sub, dict):
            raise AggregationError(f"{name}: `aggs` is not a map")
        for sname, sagg in sub.items():
            if isinstance(sagg, dict) and any(t in Mx._BUCKETS for t in sagg):
                raise RangeRefused(f"{name}.{sname}: bucket aggregations nested under the range run on the CPU path")
        try:
            metrics = Mx.parse_request(sub)
        except Mx.MetricsRefused as e:
            raise RangeRefused(f"{name}.{e}") from None
    return RangeRequest(name=name, field=body["field"], ranges=ranges, keyed=bool(body.get("keyed", False)), metrics=metrics)


def to_image(v, kind):
    """f64_to_fastfield_u64 (aggregation/mod.rs) of a bound: u64 `v as u64`, i64 / date `(v as i64)` mapped to its image, f64
    v.to_u64(); Rust's `as` truncates toward zero, saturates and maps NaN to 0."""
    if kind == "f64":
        b = int(np.float64(v).view(np.uint64))
        return b ^ _HIGH if not b & _HIGH else b ^ _U64_MAX
    if kind == "u64":
        if v != v or v <= 0:
            return 0
        return _U64_MAX if v >= 18446744073709551616.0 else int(v)
    if v != v:
        i = 0
    elif v >= 9223372036854775808.0:
        i = _HIGH - 1
    elif v < -9223372036854775808.0:
        i = -_HIGH
    else:
        i = int(v)
    return (i + _HIGH) & _U64_MAX


def value_of(image, kind):
    """f64_from_fastfield_u64 of an image of a u64, i64, date or f64 column."""
    return Mx.value_of_image(image, Mx._VALUE_KINDS[kind])


def bound_string(image, kind, is_start):
    """range_to_string's half: `*` for start 0 and end u64::MAX, format_date on a date column, else f64 Display."""
    if (is_start and image == 0) or (not is_start and image == _U64_MAX):
        return "*"
    if kind == "date":
        return format_date(image - _HIGH)
    return rust_f64_display(value_of(image, kind))


def extend(ranges, kind):
    """extend_validate_ranges in image space: [(key, start, end)] sorted stably by start, with 0..first.start before, last.end..
    u64::MAX after and every hole filled.  Raises AggregationError for overlapping ranges (end > next start)."""
    conv = sorted(((k, 0 if f is None else to_image(f, kind), _U64_MAX if t is None else to_image(t, kind)) for k, f, t in ranges),
                  key=lambda b: b[1])
    if conv[0][1] != 0:
        conv.insert(0, (None, 0, conv[0][1]))
    if conv[-1][2] != _U64_MAX:
        conv.append((None, conv[-1][2], _U64_MAX))
    out = [conv[0]]
    for b in conv[1:]:
        prev = out[-1]
        if prev[2] > b[1]:
            raise AggregationError(f"Overlapping ranges not supported range {prev[1]}..{prev[2]}, range+1 {b[1]}..{b[2]}")
        if prev[2] != b[1]:
            out.append((None, prev[2], b[1]))
        out.append(b)
    return out


def plan(r: RangeRequest, fields):
    """RangeRequest and {field name: metrics.MetricField} -> RangePlan: the range's spec and buckets and one metrics spec of up to
    TQ_METRICS_MAX_COLUMNS columns.  Refuses (RangeRefused) what the reference leaves unspecified: NaN bounds, a range whose start
    exceeds its end, equal starts after conversion, and buckets sharing a key string or a sort value."""
    f = fields.get(r.field)
    if f is None:
        raise RangeRefused(f"{r.name}: field {r.field!r} has no registered fast column")
    if f.n_column_types != 1:
        raise RangeRefused(f"{r.name}: a range on a field of several column types (JSON) runs on the CPU path")
    if f.multi_valued:
        raise RangeRefused(f"{r.name}: a range on a multi-valued column runs on the CPU path")
    if f.kind not in _RANGE_KINDS:
        raise RangeRefused(f"{r.name}: a range on a {f.kind} column runs on the CPU path")
    for _, lo, hi in r.ranges:
        if (lo is not None and lo != lo) or (hi is not None and hi != hi):
            raise RangeRefused(f"{r.name}: a NaN bound runs on the CPU path")
    for k, lo, hi in r.ranges:
        s = 0 if lo is None else to_image(lo, f.kind)
        e = _U64_MAX if hi is None else to_image(hi, f.kind)
        if s > e:
            raise RangeRefused(f"{r.name}: a range whose start exceeds its end in the column's image space runs on the CPU path")
    ext = extend(r.ranges, f.kind)
    starts = [s for _, s, _ in ext]
    if len(set(starts)) != len(starts):
        raise RangeRefused(f"{r.name}: an empty range (two buckets with one start) runs on the CPU path")
    if len(ext) > TQ_RANGE_MAX_BUCKETS:
        raise RangeRefused(f"{r.name}: {len(ext)} buckets after extension, more than the device's {TQ_RANGE_MAX_BUCKETS}")
    buckets = []
    for key, s, e in ext:
        name = bound_string(s, f.kind, True) + "-" + bound_string(e, f.kind, False)
        lo = None if s == 0 else value_of(s, f.kind)
        hi = None if e == _U64_MAX else value_of(e, f.kind)
        buckets.append({"name": name, "key": key if key is not None else name, "from": lo, "to": hi})
    if len({b["name"] for b in buckets}) != len(buckets):
        raise RangeRefused(f"{r.name}: two buckets with one key string (images above 2^53) run on the CPU path")
    if len({_total_order(_F64_MIN if b["from"] is None else b["from"]) for b in buckets}) != len(buckets):
        raise RangeRefused(f"{r.name}: two buckets with one `from` (images above 2^53) run on the CPU path")
    if r.keyed and len({b["key"] for b in buckets}) != len(buckets):
        raise RangeRefused(f"{r.name}: keyed buckets sharing a custom key run on the CPU path")
    mplan = None
    if r.metrics:
        try:
            mplan = Mx.plan(r.metrics, fields)
        except Mx.MetricsRefused as e:
            raise RangeRefused(f"{r.name}.{e}") from None
    return RangePlan(request=r, kind=f.kind, rspec=(f.column_id, starts), buckets=buckets, mplan=mplan)


def rows_of(out, q, n_buckets):
    """(doc_count[n_buckets], parts[n_buckets, TQ_METRICS_MAX_COLUMNS] | None) of query q of Context.range_batch's output."""
    counts, parts = out[0], out[1]
    return counts[q, :n_buckets].astype(np.uint64), (parts[q, :n_buckets] if parts is not None else None)


def merge(rows_list):
    """Merges one query's rows of any number of contexts (each evaluating its own segments or doc ranges, all with the query's one
    spec) by bucket: doc counts add, parts merge with metrics.merge's rules."""
    rows_list = list(rows_list)
    counts = sum((c for c, _ in rows_list), np.zeros_like(rows_list[0][0]))
    if rows_list[0][1] is None:
        return counts, None
    n = len(counts)
    parts = np.stack([Mx.merge([p[b] for _, p in rows_list]) for b in range(n)]) if n else None
    return counts, parts


def bucket_entry(b, count, kind):
    """One final bucket {"key", "doc_count"[, "from"][, "to"][, "from_as_string"][, "to_as_string"]}."""
    e = {"key": b["key"], "doc_count": int(count)}
    if b["from"] is not None:
        e["from"] = b["from"]
    if b["to"] is not None:
        e["to"] = b["to"]
    if kind == "date":
        if b["from"] is not None:
            e["from_as_string"] = format_date(int(b["from"]))
        if b["to"] is not None:
            e["to_as_string"] = format_date(int(b["to"]))
    return e


def finalize(p: RangePlan, merged):
    """{name: {"buckets": [...] | {key: ...}}} from merge()'s (doc_count, parts): every bucket in `from` order (total_cmp, an open
    `from` first), each with its metrics' final results.  Raises RangeRefused (with `refused` and `answered`) when some bucket's
    sum-bearing aggregation fails the guard."""
    counts, parts = merged
    refused, entries = {}, []
    for i, b in enumerate(p.buckets):
        sub = {}
        if p.mplan is not None:
            try:
                sub = Mx.finalize(p.mplan, parts[i])
            except Mx.MetricsRefused as e:
                for n, why in e.refused.items():
                    refused.setdefault(n, f"{why} (bucket {b['key']})")
                sub = e.answered
        entries.append((b, counts[i], sub))
    entries.sort(key=lambda x: _total_order(_F64_MIN if x[0]["from"] is None else x[0]["from"]))
    out = []
    for b, count, sub in entries:
        e = bucket_entry(b, count, p.kind)
        e.update({n: v for n, v in sub.items() if n not in refused})
        out.append(e)
    r = p.request
    result = {r.name: {"buckets": {e["key"]: e for e in out}} if r.keyed else {"buckets": out}}
    if refused:
        raise RangeRefused("; ".join(f"{r.name}.{n}: {why}" for n, why in refused.items()), refused=refused, answered=result)
    return result


def run(contexts, qb, requests, fields, count_hits=False):
    """Runs one parsed request per query of qb over every Context (each evaluating its own segments or doc ranges) and finalises.
    Returns [{name: result} or RangeRefused] per query, and the merged hit counts with count_hits."""
    plans = [plan(r, fields) for r in requests]
    rspecs = [p.rspec for p in plans]
    mspecs = None
    if any(p.mplan is not None for p in plans):  # (a range without sub-aggregations in such a batch reads one empty column)
        mspecs = [p.mplan.columns if p.mplan is not None else [(0, TQ_FAST_U64, TQ_METRIC_EMPTY, 0)] for p in plans]
    per_ctx, hits = [], np.zeros(qb.nq, dtype=np.uint64)
    for ctx in contexts:
        out = ctx.range_batch(qb, rspecs, mspecs, count_hits=count_hits)
        if count_hits:
            hits += out[2]
        per_ctx.append(out)
    res = []
    for q, p in enumerate(plans):
        n = len(p.buckets)
        rows = [rows_of(out, q, n) for out in per_ctx] or [(np.zeros(n, np.uint64), np.stack([Mx.empty_parts()] * n) if p.mplan else None)]
        try:
            res.append(finalize(p, merge(rows)))
        except RangeRefused as e:
            res.append(e)
    return (res, hits) if count_hits else res
