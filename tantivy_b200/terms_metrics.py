"""The request and result side of a `terms` aggregation whose sub-aggregations are metrics (avg, sum, min, max, stats, value_count),
for the device's intermediate results (Context.terms_metrics_batch).  Pure Python: it parses a request of one top-level terms with
1..n metric sub-aggregations, refuses what the device does not run (TermsMetricsRefused: take the CPU path), maps the request to one
terms spec, one metrics spec of up to four columns and an order, merges the rows of any number of contexts by (segment, key) --
cutting once per segment a segment split over contexts -- and then by intermediate key, applies the exactness guard and finalises to
tantivy's result: the terms' buckets (tantivy_b200.terms) each holding {name: metric result} (tantivy_b200.metrics).

A term's metrics collect the docs the terms count under its key (collect_terms_with_docs, term_agg/mod.rs).  The order may be a
metric sub-aggregation: `avg`, `sum`, `min`, `max` or `value_count` by name, a `stats` by `name.count` / `.sum` / `.min` / `.max` /
`.avg`.  Each segment is then cut by compute_metric_value(...).unwrap_or(0.0) under partial_cmp, and the final buckets are ordered
by the merged value, unwrap_or(f64::MIN), under total_cmp; equal values keep the lowest keys in both.  An order by a metric is only
exact when its cut is: the device returns the ordering column's part over every doc the terms collect, and an order on a column that
saw a NaN, or by a sum or avg whose total part fails the guard, is refused.  When some kept bucket's sum, avg or stats fails the guard,
that aggregation is refused for the whole terms; the buckets and the others stay answered."""
import struct
from dataclasses import dataclass, replace
from typing import Optional

import numpy as np

from . import metrics as Mx
from . import terms as Tm
from ._abi import (TQ_METRIC_COUNT_ONLY, TQ_TERMS_BY_METRIC, TQ_TERMS_ORDER_AVG, TQ_TERMS_ORDER_COUNT, TQ_TERMS_ORDER_MAX, TQ_TERMS_ORDER_MIN,
                   TQ_TERMS_ORDER_SUM)
from .histogram import AggregationError

# the metric a sub-aggregation exposes to an order: single-value metrics by name alone, stats by property (stats.rs:325-356)
ORDER_BY_TYPE = {"value_count": TQ_TERMS_ORDER_COUNT, "sum": TQ_TERMS_ORDER_SUM, "avg": TQ_TERMS_ORDER_AVG, "min": TQ_TERMS_ORDER_MIN,
                 "max": TQ_TERMS_ORDER_MAX}
STATS_PROPERTIES = {"count": TQ_TERMS_ORDER_COUNT, "sum": TQ_TERMS_ORDER_SUM, "avg": TQ_TERMS_ORDER_AVG, "min": TQ_TERMS_ORDER_MIN,
                    "max": TQ_TERMS_ORDER_MAX}
F64_MIN = -Mx.F64_MAX


class TermsMetricsRefused(ValueError):
    """A terms request with metric sub-aggregations, or some of its sub-aggregations, that the device does not answer exactly; the
    caller takes the CPU path.  `refused` maps each refused sub-aggregation's name to the reason; `answered` holds the terms' final
    result with the other sub-aggregations ({name: result}), when there is one."""

    def __init__(self, message, refused=None, answered=None):
        super().__init__(message)
        self.refused = refused or {}
        self.answered = answered or {}


@dataclass
class TermsMetricsRequest:
    """One top-level terms: its name, the request (terms.TermsAggregation), its metric sub-aggregations (metrics.MetricAggregation)
    and, for an order by one of them, (its name, TQ_TERMS_ORDER_*)."""
    name: str
    req: Tm.TermsAggregation
    metrics: list
    order: Optional[tuple] = None


@dataclass
class TermsMetricsPlan:
    """The terms' field type, its spec for Context.terms_metrics_batch, the metrics plan and the order ((spec column,
    TQ_TERMS_ORDER_*) or None)."""
    request: TermsMetricsRequest
    kind: str
    tspec: tuple
    mplan: Mx.MetricsPlan
    order: Optional[tuple] = None


def _order_of(name, target, sub):
    """(sub-aggregation name, TQ_TERMS_ORDER_*) of an order target naming a sub-aggregation (get_agg_name_and_property)."""
    agg_name, _, prop = target.partition(".")
    if agg_name not in sub:
        raise AggregationError(f"could not find aggregation with name {agg_name} in metric sub_aggregations")
    sagg = sub[agg_name]
    styp = next((t for t in sagg if t not in ("aggs", "aggregations")), None) if isinstance(sagg, dict) else None
    if styp == "stats":
        if not prop:
            raise TermsMetricsRefused(f"{name}: ordering by the stats {agg_name!r} without a property runs on the CPU path")
        if prop not in STATS_PROPERTIES:
            raise TermsMetricsRefused(f"{name}: ordering by the unknown stats property {target!r} runs on the CPU path")
        return agg_name, STATS_PROPERTIES[prop]
    if styp in ORDER_BY_TYPE:
        if prop:
            raise TermsMetricsRefused(f"{name}: ordering by the property {target!r} of a single-value metric runs on the CPU path")
        return agg_name, ORDER_BY_TYPE[styp]
    raise TermsMetricsRefused(f"{name}: ordering by a {styp} sub-aggregation runs on the CPU path")


def parse_request(aggs):
    """An Aggregations map {name: {"terms": {...}, "aggs": {...}}} -> TermsMetricsRequest.  Every request the device does not run
    raises TermsMetricsRefused with its own message; a malformed one AggregationError."""
    if not isinstance(aggs, dict) or not aggs:
        raise AggregationError("expected a non-empty map of aggregations")
    if len(aggs) != 1:
        raise TermsMetricsRefused("more than one top-level aggregation runs on the CPU path")
    (name, agg), = aggs.items()
    if not isinstance(agg, dict):
        raise AggregationError(f"aggregation {name!r} is not an object")
    if "aggs" in agg and "aggregations" in agg:
        raise AggregationError(f"{name}: both `aggs` and `aggregations`")
    sub = agg.get("aggs", agg.get("aggregations"))
    types = [k for k in agg if k not in ("aggs", "aggregations")]
    if len(types) != 1:
        raise AggregationError(f"aggregation {name!r} must have exactly one type")
    if types[0] != "terms":
        raise TermsMetricsRefused(f"{name}: a top-level {types[0]} is not a terms aggregation with metric sub-aggregations")
    if not sub:
        raise TermsMetricsRefused(f"{name}: a terms aggregation without sub-aggregations runs through tantivy_b200.terms")
    if not isinstance(sub, dict):
        raise AggregationError(f"{name}: `aggs` is not a map")
    req = Tm.TermsAggregation.from_dict(agg["terms"])
    order = None if req.order_target in ("_count", "_key") else _order_of(name, req.order_target, sub)
    for sname, sagg in sub.items():
        if isinstance(sagg, dict) and any(t in Mx._BUCKETS for t in sagg):
            raise TermsMetricsRefused(f"{name}.{sname}: bucket aggregations nested under terms run on the CPU path")
    try:
        metrics = Mx.parse_request(sub)
    except Mx.MetricsRefused as e:
        raise TermsMetricsRefused(f"{name}.{e}") from None
    return TermsMetricsRequest(name=name, req=req, metrics=metrics, order=order)


def plan(r: TermsMetricsRequest, fields):
    """TermsMetricsRequest and {field name: metrics.MetricField} -> TermsMetricsPlan: the terms spec (target TQ_TERMS_BY_METRIC for
    a metric order), one metrics spec of up to TQ_METRICS_MAX_COLUMNS columns and the order's spec column."""
    f = fields.get(r.req.field)
    if f is None:
        raise TermsMetricsRefused(f"{r.name}: field {r.req.field!r} has no registered fast column")
    base = r.req if r.order is None else replace(r.req, order_target="_count")  # (the terms side's own checks)
    try:
        Tm.check_device(base, f.kind, f.multi_valued, f.n_column_types)
        tspec = Tm.terms_spec(base, f.column_id, f.kind)
    except Tm.TermsRefused as e:
        raise TermsMetricsRefused(f"{r.name}: {e}") from None
    try:
        mplan = Mx.plan(r.metrics, fields)
    except Mx.MetricsRefused as e:
        raise TermsMetricsRefused(f"{r.name}.{e}") from None
    order = None
    if r.order is not None:
        tspec = (tspec[0], TQ_TERMS_BY_METRIC) + tuple(tspec[2:])
        order = (mplan.slot[r.order[0]], r.order[1])
    return TermsMetricsPlan(request=r, kind=f.kind, tspec=tspec, mplan=mplan, order=order)


# ---- values of the order ----------------------------------------------------------------------------------------------------
def segment_value(p: TermsMetricsPlan, part):
    """compute_metric_value(...).unwrap_or(0.0) of the ordering column's part of one (segment, key) (stats.rs:325-356)."""
    _, kind, flags, _ = p.mplan.columns[p.order[0]]
    metric = p.order[1]
    count, s, vmin, vmax = Mx.stats_of(part, kind, flags)
    if metric == TQ_TERMS_ORDER_COUNT:
        return float(count)
    if metric == TQ_TERMS_ORDER_SUM:
        return s
    if count == 0:
        return 0.0
    return {TQ_TERMS_ORDER_AVG: s / count, TQ_TERMS_ORDER_MIN: vmin, TQ_TERMS_ORDER_MAX: vmax}[metric]


def final_value(p: TermsMetricsPlan, parts):
    """The final order value of one bucket from its merged parts: get_value_from_aggregation on its final metric result
    (into_final_metric_result), unwrap_or(f64::MIN) -- an avg, min or max without values and a none_if_no_match sum without values
    are null."""
    name, metric = p.request.order
    agg = next(a for a in p.mplan.aggs if a.name == name)
    _, kind, flags, _ = p.mplan.columns[p.order[0]]
    count, s, vmin, vmax = Mx.stats_of(parts[p.order[0]], kind, flags)
    if metric == TQ_TERMS_ORDER_COUNT:
        return float(count)
    if metric == TQ_TERMS_ORDER_SUM:
        return F64_MIN if count == 0 and agg.type == "sum" and agg.none_if_no_match else s
    if count == 0:
        return F64_MIN
    return {TQ_TERMS_ORDER_AVG: s / count, TQ_TERMS_ORDER_MIN: vmin, TQ_TERMS_ORDER_MAX: vmax}[metric]


def total_cmp_key(v):
    """f64::total_cmp as an integer key: -0.0 before +0.0, NaNs at the ends by sign."""
    b = struct.unpack("<q", struct.pack("<d", v))[0]
    return b ^ ((b >> 63) & 0x7FFFFFFFFFFFFFFF)


# ---- rows, merges, guards, final result ---------------------------------------------------------------------------------------
def rows_of(out, q):
    """Query q of Context.terms_metrics_batch's output: ([(segment_ord, image, doc_count, parts)], sum_other, error_bound,
    order_part)."""
    segs, keys, counts, parts, n, other, error, opart = out[:8]
    entries = [(int(segs[q, j]), int(keys[q, j]), int(counts[q, j]), parts[q, j]) for j in range(int(n[q]))]
    return entries, int(other[q]), int(error[q]), opart[q]


def segment_entries(p: TermsMetricsPlan, rows_list):
    """The contexts' rows of one query by segment: ({segment_ord: {image: (doc_count, parts)}}, sum_other, error_bound, the merged
    order part).  A segment split over contexts comes back uncut from each: its counts add and its parts merge here."""
    per, other, error, oparts = {}, 0, 0, []
    for entries, o, e, opart in rows_list:
        for s, image, count, parts in entries:
            seg = per.setdefault(s, {})
            if image in seg:
                c0, p0 = seg[image]
                seg[image] = (c0 + count, Mx.merge([p0, parts]))
            else:
                seg[image] = (count, Mx.merge([parts]))
        other += o
        error += e
        oparts.append(opart)
    return per, other, error, Mx.merge(oparts)[0]  # (each part broadcast over the columns: column 0 holds the merge)


def cut_segment(p: TermsMetricsPlan, entries):
    """One segment's cut of {image: (doc_count, parts)} (terms.cut_segment with the order's segment values): ({image: (doc_count,
    parts)} kept, term_doc_count_before_cutoff, sum_other_doc_count).  A whole segment, cut on the device already, is not cut again."""
    counts = {k: c for k, (c, _) in entries.items()}
    metric = None if p.order is None else {k: segment_value(p, parts[p.order[0]]) for k, (_, parts) in entries.items()}
    kept, e, o = Tm.cut_segment(counts, p.request.req, metric)
    return {k: entries[k] for k, _ in kept}, e, o


def segment_result(p: TermsMetricsPlan, entries, dictionary=None, missing_image=None):
    """One segment's {intermediate key: (doc_count, parts)}, as terms.segment_result maps keys (a str column's missing entry first,
    so that a term of the same text replaces it)."""
    req = p.request.req
    out, rest = {}, []
    for image, v in sorted(entries.items()):
        if p.kind == "str" and req.missing is not None and image == missing_image:
            out[Tm._missing_key(req.missing)] = v
        else:
            rest.append((image, v))
    for image, v in rest:
        out[Tm.intermediate_key(image, p.kind, dictionary)] = v
    return out


def merge(results):
    """merge_fruits over segment results, each ({key: (doc_count, parts)}, sum_other, error_bound): counts add, parts merge."""
    entries, other, error = {}, 0, 0
    for e, o, err in results:
        for k, (c, parts) in e.items():
            if k in entries:
                c0, p0 = entries[k]
                entries[k] = (c0 + c, Mx.merge([p0, parts]))
            else:
                entries[k] = (c, parts)
        other += int(o)
        error += int(err)
    return entries, other, error


def order_guard(p: TermsMetricsPlan, total):
    """None when the metric order's cut is exact over the ordering column's total part, else the reason it may not be."""
    if p.order is None:
        return None
    if int(total["n_nan"]):
        return "the ordering column saw a NaN, which partial_cmp leaves unordered"
    _, _, flags, _ = p.mplan.columns[p.order[0]]
    if p.order[1] in (TQ_TERMS_ORDER_SUM, TQ_TERMS_ORDER_AVG) and not flags & TQ_METRIC_COUNT_ONLY:
        why = Mx.guard(total)
        if why is not None:
            return f"the order's sums may depend on the order of the adds: {why}"
    return None


def finalize(p: TermsMetricsPlan, merged):
    """{name: the terms' final result} from merge()'s ({key: (doc_count, parts)}, sum_other, error_bound): min_doc_count, the order
    (rule of the request, equal values by key ascending), the cut to size, each bucket with its metrics' final results.  Raises
    TermsMetricsRefused (with `refused` and `answered`) when some kept bucket's sum-bearing aggregation fails the guard."""
    r = p.request
    req = r.req
    entries, other, error = merged
    buckets = sorted(((k, c, parts) for k, (c, parts) in entries.items() if c >= req.min_doc_count), key=lambda b: Tm._key_order(b[0]))
    if req.order_target == "_key":
        buckets.sort(key=lambda b: Tm._key_order(b[0]), reverse=req.order == "desc")
    elif r.order is not None:  # (stable, also reversed: equal values stay by key ascending)
        buckets.sort(key=lambda b: total_cmp_key(final_value(p, b[2])), reverse=req.order == "desc")
    else:
        buckets.sort(key=lambda b: b[1], reverse=req.order == "desc")
    cut = sum(c for _, c, _ in buckets[req.size:])
    refused, kept = {}, []
    for k, c, parts in buckets[:req.size]:
        try:
            sub = Mx.finalize(p.mplan, parts)
        except Mx.MetricsRefused as e:
            sub = e.answered
            for n, why in e.refused.items():
                refused.setdefault(n, f"{why} (bucket {Tm._final_key(k)[1]!r})")
        kept.append((k, c, sub))
    out = []
    for k, c, sub in kept:
        e = {"key": Tm._final_key(k)[1], "doc_count": c}
        if k[0] == "bool":
            e["key_as_string"] = "true" if k[1] else "false"
        e.update({n: v for n, v in sub.items() if n not in refused})
        out.append(e)
    res = {"buckets": out, "sum_other_doc_count": other + cut}
    if req.show_term_doc_count_error:
        res["doc_count_error_upper_bound"] = error
    result = {r.name: res}
    if refused:
        raise TermsMetricsRefused("; ".join(f"{r.name}.{n}: {why}" for n, why in refused.items()), refused=refused, answered=result)
    return result


def finalize_rows(p: TermsMetricsPlan, rows_list, dictionaries=None, missing_images=None):
    """The final result of one query from its rows of any number of contexts (rows_of per context): per segment the entries summed
    over the contexts and cut once, the segments merged by intermediate key in segment_ord order, the order's guard on the merged
    total part, then finalize.  dictionaries[segment_ord] = a str segment's terms, missing_images[segment_ord] = its missing image."""
    per, other, error, total = segment_entries(p, rows_list)
    why = order_guard(p, total)
    if why is not None:
        name = p.request.order[0]
        raise TermsMetricsRefused(f"{p.request.name}: ordering by {name}: {why}", refused={p.request.name: why})
    results = []
    for s in sorted(per):
        kept, e, o = cut_segment(p, per[s])
        results.append((segment_result(p, kept, None if dictionaries is None else dictionaries[s],
                                       None if missing_images is None else missing_images.get(s)), o, e))
    entries, o, e = merge(results)
    return finalize(p, (entries, other + o, error + e))


def run(contexts, qb, requests, fields, count_hits=False, dictionaries=None, missing_images=None):
    """Runs one parsed request per query of qb over every Context (each evaluating its own segments or doc ranges) and finalises.
    Returns [{name: result} or TermsMetricsRefused] per query, and the merged hit counts with count_hits."""
    plans = [plan(r, fields) for r in requests]
    per_ctx, hits = [], np.zeros(qb.nq, dtype=np.uint64)
    for ctx in contexts:
        out = ctx.terms_metrics_batch(qb, [p.tspec for p in plans], [p.mplan.columns for p in plans], [p.order for p in plans],
                                      count_hits=count_hits)
        if count_hits:
            hits += out[8]
        per_ctx.append(out)
    res = []
    for q, p in enumerate(plans):
        try:
            res.append(finalize_rows(p, [rows_of(out, q) for out in per_ctx], dictionaries, missing_images))
        except TermsMetricsRefused as e:
            res.append(e)
    return (res, hits) if count_hits else res
