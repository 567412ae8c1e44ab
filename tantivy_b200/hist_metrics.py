"""The request and result side of a `histogram` / `date_histogram` whose sub-aggregations are metrics (avg, sum, min, max, stats,
value_count), for the device's intermediate results (Context.hist_metrics_batch).  Pure Python: it parses a request of one top-level
histogram with 1..n metric sub-aggregations, refuses what the device does not run (HistMetricsRefused: take the CPU path), maps the
request to one histogram spec and one metrics spec of up to four columns, merges the rows of any number of contexts by bucket,
applies the exactness guard per (bucket, column) and finalises to tantivy's result: the histogram's buckets (tantivy_b200.histogram)
each holding {name: metric result} (tantivy_b200.metrics).

A bucket's metrics collect the docs the histogram counts in it (SegmentHistogramCollector::collect, histogram.rs:490-505).  A
bucket the gap filling or extended_bounds add holds the empty sub-aggregation results (empty_from_req, histogram.rs:802-826).  When
some bucket's sum, avg or stats fails the guard, that aggregation is refused for the whole histogram; the others stay answered."""
from dataclasses import dataclass

import numpy as np

from . import histogram as Hg
from . import metrics as Mx
from .histogram import AggregationError

_HISTOGRAMS = ("histogram", "date_histogram")
_HIST_KINDS = ("u64", "i64", "f64", "bool", "date")


class HistMetricsRefused(ValueError):
    """A histogram request with metric sub-aggregations, or some of its sub-aggregations, that the device does not answer exactly;
    the caller takes the CPU path.  `refused` maps each refused sub-aggregation's name to the reason; `answered` holds the
    histogram's final result with the other sub-aggregations ({name: result}), when there is one."""

    def __init__(self, message, refused=None, answered=None):
        super().__init__(message)
        self.refused = refused or {}
        self.answered = answered or {}


@dataclass
class HistMetricsRequest:
    """One top-level histogram: its name, the request (HistogramAggregation, a date request in milliseconds), whether it was a
    date_histogram, and its metric sub-aggregations (metrics.MetricAggregation)."""
    name: str
    req: Hg.HistogramAggregation
    is_date_histogram: bool
    metrics: list


@dataclass
class HistMetricsPlan:
    """The histogram's field type, its spec for Context.hist_metrics_batch, and the metrics plan of its sub-aggregations."""
    request: HistMetricsRequest
    kind: str
    hspec: tuple
    mplan: Mx.MetricsPlan


def parse_request(aggs):
    """An Aggregations map {name: {"histogram" | "date_histogram": {...}, "aggs": {...}}} -> HistMetricsRequest.  Every request the
    device does not run raises HistMetricsRefused with its own message; a malformed one AggregationError."""
    if not isinstance(aggs, dict) or not aggs:
        raise AggregationError("expected a non-empty map of aggregations")
    if len(aggs) != 1:
        raise HistMetricsRefused("more than one top-level aggregation runs on the CPU path")
    (name, agg), = aggs.items()
    if not isinstance(agg, dict):
        raise AggregationError(f"aggregation {name!r} is not an object")
    sub = agg.get("aggs", agg.get("aggregations"))
    if "aggs" in agg and "aggregations" in agg:
        raise AggregationError(f"{name}: both `aggs` and `aggregations`")
    types = [k for k in agg if k not in ("aggs", "aggregations")]
    if len(types) != 1:
        raise AggregationError(f"aggregation {name!r} must have exactly one type")
    typ = types[0]
    if typ == "terms":
        raise HistMetricsRefused(f"{name}: sub-aggregations under terms run on the CPU path")
    if typ not in _HISTOGRAMS:
        raise HistMetricsRefused(f"{name}: a top-level {typ} is not a histogram with metric sub-aggregations")
    if not sub:
        raise HistMetricsRefused(f"{name}: a histogram without sub-aggregations runs through tantivy_b200.histogram")
    if not isinstance(sub, dict):
        raise AggregationError(f"{name}: `aggs` is not a map")
    for sname, sagg in sub.items():
        if isinstance(sagg, dict) and any(t in Mx._BUCKETS for t in sagg):
            raise HistMetricsRefused(f"{name}.{sname}: bucket aggregations nested under the histogram run on the CPU path")
    try:
        metrics = Mx.parse_request(sub)
    except Mx.MetricsRefused as e:
        raise HistMetricsRefused(f"{name}.{e}") from None
    if typ == "histogram":
        req, is_date = Hg.HistogramAggregation.from_dict(agg["histogram"]), False
    else:
        req, is_date = Hg.DateHistogramAggregationReq.from_dict(agg["date_histogram"]).to_histogram_req(), True
    req.validate()
    return HistMetricsRequest(name=name, req=req, is_date_histogram=is_date, metrics=metrics)


def plan(r: HistMetricsRequest, fields):
    """HistMetricsRequest and {field name: metrics.MetricField} -> HistMetricsPlan: the histogram's spec and one metrics spec of up
    to TQ_METRICS_MAX_COLUMNS columns."""
    f = fields.get(r.req.field)
    if f is None:
        raise HistMetricsRefused(f"{r.name}: field {r.req.field!r} has no registered fast column")
    if f.n_column_types != 1:
        raise HistMetricsRefused(f"{r.name}: a histogram on a field of several column types (JSON) runs on the CPU path")
    if f.multi_valued:
        raise HistMetricsRefused(f"{r.name}: a histogram on a multi-valued column runs on the CPU path")
    if f.kind not in _HIST_KINDS:
        raise HistMetricsRefused(f"{r.name}: a histogram on a {f.kind} column runs on the CPU path")
    try:
        mplan = Mx.plan(r.metrics, fields)
    except Mx.MetricsRefused as e:
        raise HistMetricsRefused(f"{r.name}.{e}") from None
    return HistMetricsPlan(request=r, kind=f.kind, hspec=Hg.histogram_spec(r.req, f.column_id, f.kind), mplan=mplan)


def rows_of(out, q):
    """{pos: (doc_count, parts)} of query q of Context.hist_metrics_batch's output."""
    pos, counts, parts, n = out[:4]
    return {int(pos[q, j]): (int(counts[q, j]), parts[q, j]) for j in range(int(n[q]))}


def merge(rows_list):
    """Merges one query's rows of any number of contexts by bucket: doc counts add, parts merge with metrics.merge's rules."""
    out = {}
    for rows in rows_list:
        for p, (count, parts) in rows.items():
            if p in out:
                c0, p0 = out[p]
                out[p] = (c0 + count, Mx.merge([p0, parts]))
            else:
                out[p] = (count, Mx.merge([parts]))
    return out


def finalize(p: HistMetricsPlan, merged, bucket_limit=Hg.DEFAULT_BUCKET_LIMIT):
    """{name: the histogram's final result} from merge()'s {pos: (doc_count, parts)}: histogram.finalize's buckets, each with the
    metrics' final results (metrics.finalize per bucket; the empty results in a bucket that only the gap filling or extended_bounds
    add).  Raises HistMetricsRefused (with `refused` and `answered`) when some bucket's sum-bearing aggregation fails the guard."""
    r = p.request
    buckets = Hg.final_buckets(r.req, {pos: c for pos, (c, _) in merged.items()}, p.kind, bucket_limit)
    refused, entries = {}, []
    for key, count, pos in buckets:
        if pos is None:  # (empty_from_req)
            sub = Mx.finalize(p.mplan, Mx.empty_parts())
        else:
            try:
                sub = Mx.finalize(p.mplan, merged[pos][1])
            except Mx.MetricsRefused as e:
                for n, why in e.refused.items():
                    refused.setdefault(n, f"{why} (bucket {Hg.bucket_entry(key, count, p.kind)['key']})")
                sub = e.answered
        entries.append((key, count, sub))
    out = []
    for key, count, sub in entries:
        e = Hg.bucket_entry(key, count, p.kind)
        e.update({n: v for n, v in sub.items() if n not in refused})
        out.append(e)
    result = {r.name: Hg.keyed_or_list(r.req, out)}
    if refused:
        raise HistMetricsRefused("; ".join(f"{r.name}.{n}: {why}" for n, why in refused.items()), refused=refused, answered=result)
    return result


def run(contexts, qb, requests, fields, count_hits=False):
    """Runs one parsed request per query of qb over every Context (each evaluating its own segments or doc ranges) and finalises.
    Returns [{name: result} or HistMetricsRefused] per query, and the merged hit counts with count_hits."""
    plans = [plan(r, fields) for r in requests]
    hspecs = [p.hspec for p in plans]
    mspecs = [p.mplan.columns for p in plans]
    per_ctx, hits = [], np.zeros(qb.nq, dtype=np.uint64)
    for ctx in contexts:
        out = ctx.hist_metrics_batch(qb, hspecs, mspecs, count_hits=count_hits)
        if count_hits:
            hits += out[4]
        per_ctx.append(out)
    res = []
    for q, p in enumerate(plans):
        try:
            res.append(finalize(p, merge(rows_of(out, q) for out in per_ctx)))
        except HistMetricsRefused as e:
            res.append(e)
    return (res, hits) if count_hits else res

