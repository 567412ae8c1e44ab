"""The request and result side of a `terms` aggregation whose only sub-aggregation is a `histogram` / `date_histogram` (the "split
series" chart: the top terms, each with its own time series), for the device's intermediate results (Context.terms_hist_batch).
Pure Python: it parses a request of one top-level terms over exactly one histogram with nothing under it, refuses what the device
does not run (TermsHistRefused: take the CPU path), maps the request to one terms spec and one histogram spec, merges the rows of any
number of contexts by (segment, key) -- cutting once per segment a segment split over contexts -- then by intermediate key and by
bucket pos, and finalises to tantivy's result: the terms' buckets (tantivy_b200.terms) each holding {name: its histogram}
(tantivy_b200.histogram).

A term's histogram collects every doc the terms count under its key, the missing key's included (collect_terms_with_docs;
term_histogram.rs:162-175), each in bucket pos when its value lies in the (query, segment)'s normalised bounds.  A term's doc_count is
the terms count: it includes docs without a histogram value or outside hard_bounds.  Each kept term's histogram is finalised on its
own (histogram.final_buckets: gap filling over its own first and last non-empty bucket, extended_bounds, hard_bounds), and the whole
result is checked against the bucket limit as into_final_result does: each kept term counts 1 plus its histogram's buckets."""
import re
from dataclasses import dataclass

import numpy as np

from . import histogram as Hg
from . import terms as Tm
from ._abi import QueryBatch
from .histogram import AggregationError
from .lib import TqError

_HISTOGRAMS = ("histogram", "date_histogram")
_HIST_KINDS = ("u64", "i64", "f64", "bool", "date")
_SUB = ("aggs", "aggregations")


class TermsHistRefused(ValueError):
    """A terms request with a histogram sub-aggregation that the device does not answer exactly; the caller takes the CPU path."""


@dataclass
class TermsHistRequest:
    """One top-level terms: its name and request (terms.TermsAggregation), and its one histogram: name, request
    (HistogramAggregation, a date request in milliseconds) and whether it was a date_histogram."""
    name: str
    req: Tm.TermsAggregation
    hist_name: str
    hist_req: Hg.HistogramAggregation
    is_date_histogram: bool


@dataclass
class TermsHistPlan:
    """The two fields' kinds and the specs for Context.terms_hist_batch."""
    request: TermsHistRequest
    kind: str
    hist_kind: str
    tspec: tuple
    hspec: tuple


def _one_type(name, agg):
    if not isinstance(agg, dict):
        raise AggregationError(f"aggregation {name!r} is not an object")
    if all(k in agg for k in _SUB):
        raise AggregationError(f"{name}: both `aggs` and `aggregations`")
    types = [k for k in agg if k not in _SUB]
    if len(types) != 1:
        raise AggregationError(f"aggregation {name!r} must have exactly one type")
    return types[0], agg.get("aggs", agg.get("aggregations"))


def parse_request(aggs):
    """An Aggregations map {name: {"terms": {...}, "aggs": {hist_name: {"histogram" | "date_histogram": {...}}}}} ->
    TermsHistRequest.  Every request the device does not run raises TermsHistRefused with its own message; a malformed one
    AggregationError."""
    if not isinstance(aggs, dict) or not aggs:
        raise AggregationError("expected a non-empty map of aggregations")
    if len(aggs) != 1:
        raise TermsHistRefused("more than one top-level aggregation runs on the CPU path")
    (name, agg), = aggs.items()
    typ, sub = _one_type(name, agg)
    if typ != "terms":
        raise TermsHistRefused(f"{name}: a top-level {typ} is not a terms aggregation with a histogram sub-aggregation")
    if not sub:
        raise TermsHistRefused(f"{name}: a terms aggregation without sub-aggregations runs through tantivy_b200.terms")
    if not isinstance(sub, dict):
        raise AggregationError(f"{name}: `aggs` is not a map")
    if len(sub) != 1:
        raise TermsHistRefused(f"{name}: more than one sub-aggregation under terms runs on the CPU path")
    (hname, hagg), = sub.items()
    htyp, hsub = _one_type(f"{name}.{hname}", hagg)
    if htyp not in _HISTOGRAMS:
        raise TermsHistRefused(f"{name}.{hname}: a {htyp} under terms is not a histogram sub-aggregation (the CPU path, or "
                               "tantivy_b200.terms_metrics for metrics)")
    if hsub:
        raise TermsHistRefused(f"{name}.{hname}: aggregations nested under the histogram run on the CPU path")
    req = Tm.TermsAggregation.from_dict(agg["terms"])
    if req.order_target not in ("_count", "_key"):
        agg_name = req.order_target.partition(".")[0]
        if agg_name != hname:
            raise AggregationError(f"could not find aggregation with name {agg_name} in metric sub_aggregations")
        # the reference cuts each segment by compute_metric_value = None (0.0 for every term, ties unspecified) and then fails
        # with an InternalError ("Tried to retrieve value from bucket aggregation") as soon as one term is collected
        raise TermsHistRefused(f"{name}: ordering by the histogram sub-aggregation {hname!r} runs on the CPU path (it is an error there "
                               "once any term is collected)")
    hreq, is_date = Hg.parse_request({htyp: hagg[htyp]})
    hreq.validate()
    return TermsHistRequest(name=name, req=req, hist_name=hname, hist_req=hreq, is_date_histogram=is_date)


def plan(r: TermsHistRequest, fields):
    """TermsHistRequest and {field name: metrics.MetricField} -> TermsHistPlan: the terms spec (terms.terms_spec) and the histogram
    spec (histogram.histogram_spec)."""
    f = fields.get(r.req.field)
    if f is None:
        raise TermsHistRefused(f"{r.name}: field {r.req.field!r} has no registered fast column")
    try:
        Tm.check_device(r.req, f.kind, f.multi_valued, f.n_column_types)
        tspec = Tm.terms_spec(r.req, f.column_id, f.kind)
    except Tm.TermsRefused as e:
        raise TermsHistRefused(f"{r.name}: {e}") from None
    h = fields.get(r.hist_req.field)
    where = f"{r.name}.{r.hist_name}"
    if h is None:
        raise TermsHistRefused(f"{where}: field {r.hist_req.field!r} has no registered fast column")
    if h.n_column_types != 1:
        raise TermsHistRefused(f"{where}: a histogram on a field of several column types (JSON) runs on the CPU path")
    if h.multi_valued:
        raise TermsHistRefused(f"{where}: a histogram on a multi-valued column runs on the CPU path")
    if h.kind not in _HIST_KINDS:
        raise TermsHistRefused(f"{where}: a histogram on a {h.kind} column runs on the CPU path")
    return TermsHistPlan(request=r, kind=f.kind, hist_kind=h.kind, tspec=tspec, hspec=Hg.histogram_spec(r.hist_req, h.column_id, h.kind))


# ---- rows, merges, final result --------------------------------------------------------------------------------------------------
def rows_of(out, q):
    """Query q of Context.terms_hist_batch's output: ([(segment_ord, image, doc_count, {pos: doc_count})], sum_other, error_bound)."""
    segs, keys, counts, n, other, error, first, ncell, pos, ccount = out[:10]
    entries = []
    for j in range(int(n[q])):
        a, b = int(first[q, j]), int(first[q, j]) + int(ncell[q, j])
        entries.append((int(segs[q, j]), int(keys[q, j]), int(counts[q, j]), {int(p): int(c) for p, c in zip(pos[a:b], ccount[a:b])}))
    return entries, int(other[q]), int(error[q])


def _add_hist(into, hist):
    for p, c in hist.items():
        into[p] = into.get(p, 0) + c
    return into


def segment_entries(rows_list):
    """The contexts' rows of one query by segment: ({segment_ord: {image: (doc_count, {pos: doc_count})}}, sum_other, error_bound).
    A segment split over contexts comes back uncut from each: its counts and cells add here."""
    per, other, error = {}, 0, 0
    for entries, o, e in rows_list:
        for s, image, count, hist in entries:
            seg = per.setdefault(s, {})
            c0, h0 = seg.get(image, (0, {}))
            seg[image] = (c0 + count, _add_hist(dict(h0), hist))
        other += o
        error += e
    return per, other, error


def cut_segment(p: TermsHistPlan, entries):
    """One segment's cut of {image: (doc_count, hist)} (terms.cut_segment): ({image: (doc_count, hist)} kept,
    term_doc_count_before_cutoff, sum_other_doc_count); a cut term's histogram is dropped.  A whole segment, cut on the device
    already, is not cut again."""
    kept, e, o = Tm.cut_segment({k: c for k, (c, _) in entries.items()}, p.request.req)
    return {k: entries[k] for k, _ in kept}, e, o


def segment_result(p: TermsHistPlan, entries, dictionary=None, missing_image=None):
    """One segment's {intermediate key: (doc_count, hist)}, as terms.segment_result maps keys (a str column's missing entry first,
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
    """merge_fruits over segment results, each ({key: (doc_count, hist)}, sum_other, error_bound): counts add, histograms add by
    pos."""
    entries, other, error = {}, 0, 0
    for e, o, err in results:
        for k, (c, hist) in e.items():
            c0, h0 = entries.get(k, (0, {}))
            entries[k] = (c0 + c, _add_hist(dict(h0), hist))
        other += int(o)
        error += int(err)
    return entries, other, error


def finalize(p: TermsHistPlan, merged, bucket_limit=Hg.DEFAULT_BUCKET_LIMIT):
    """{name: the terms' final result} from merge()'s ({key: (doc_count, hist)}, sum_other, error_bound): the terms' buckets as
    terms.finalize keeps and orders them (terms.ordered_buckets, terms.bucket_entry), each with its histogram finalised on its own
    (histogram.final_buckets), and the bucket limit over the whole result (AggregationError)."""
    r = p.request
    req = r.req
    entries, other, error = merged
    kept, cut = Tm.ordered_buckets(req, {k: c for k, (c, _) in entries.items()})
    out, total = [], 0
    for k, c in kept:
        hb = Hg.final_buckets(r.hist_req, entries[k][1], p.hist_kind, bucket_limit)
        total += 1 + len(hb)
        e = Tm.bucket_entry(k, c)
        e[r.hist_name] = Hg.keyed_or_list(r.hist_req, [Hg.bucket_entry(key, count, p.hist_kind) for key, count, _ in hb])
        out.append(e)
    if total > bucket_limit:  # (into_final_result: get_bucket_count over the whole result)
        raise AggregationError(f"Aborting aggregation because bucket limit was exceeded. Limit: {bucket_limit}, Current: {total}")
    res = {"buckets": out, "sum_other_doc_count": other + cut}
    if req.show_term_doc_count_error:
        res["doc_count_error_upper_bound"] = error
    return {r.name: res}


def finalize_rows(p: TermsHistPlan, rows_list, dictionaries=None, missing_images=None, bucket_limit=Hg.DEFAULT_BUCKET_LIMIT):
    """The final result of one query from its rows of any number of contexts (rows_of per context): per segment the entries summed
    over the contexts and cut once, the segments merged by intermediate key in segment_ord order, then finalize.
    dictionaries[segment_ord] = a str segment's terms, missing_images[segment_ord] = its missing image."""
    per, other, error = segment_entries(rows_list)
    results = []
    for s in sorted(per):
        kept, e, o = cut_segment(p, per[s])
        results.append((segment_result(p, kept, None if dictionaries is None else dictionaries[s],
                                       None if missing_images is None else missing_images.get(s)), o, e))
    entries, o, e = merge(results)
    return finalize(p, (entries, other + o, error + e), bucket_limit)


_UNSUPPORTED = re.compile(r"^tantivy_b200 error -4: query (\d+): (.*)$")


def _subset(qb, idx):
    """The queries idx of qb as a QueryBatch of their own (its rows point into qb's arrays, which it keeps alive)."""
    sub = object.__new__(QueryBatch)
    sub.__dict__.update(qb.__dict__)
    sub.parent, sub.nq = qb, len(idx)
    sub.q = np.ascontiguousarray(qb.q[np.asarray(idx, dtype=np.int64)]) if idx else np.zeros(1, dtype=qb.q.dtype)
    return sub


def run(contexts, qb, requests, fields, count_hits=False, dictionaries=None, missing_images=None):
    """Runs one parsed request per query of qb over every Context (each evaluating its own segments or doc ranges) and finalises.
    Returns [{name: result}, AggregationError or TermsHistRefused] per query, and the merged hit counts with count_hits.  A query
    the device refuses as too wide (TQ_ERR_UNSUPPORTED naming it: its keys, buckets or grid exceed the device's limits) becomes a
    TermsHistRefused with that reason, and the batch runs again without it; its hit count is then 0 here."""
    plans = [plan(r, fields) for r in requests]
    live, refused = list(range(qb.nq)), {}
    while True:
        sub = qb if len(live) == qb.nq else _subset(qb, live)
        per_ctx, hits = [], np.zeros(qb.nq, dtype=np.uint64)
        try:
            for ctx in contexts:
                out = ctx.terms_hist_batch(sub, [plans[q].tspec for q in live], [plans[q].hspec for q in live], count_hits=count_hits)
                if count_hits:
                    hits[live] += out[11]
                per_ctx.append(out)
            break
        except TqError as e:
            m = _UNSUPPORTED.match(str(e))
            if not m or int(m.group(1)) >= len(live):
                raise
            q = live.pop(int(m.group(1)))
            refused[q] = TermsHistRefused(f"{plans[q].request.name}: {m.group(2)}")
    res, at = [], {q: j for j, q in enumerate(live)}
    for q, p in enumerate(plans):
        if q in refused:
            res.append(refused[q])
            continue
        try:
            res.append(finalize_rows(p, [rows_of(out, at[q]) for out in per_ctx], dictionaries, missing_images))
        except AggregationError as e:
            res.append(e)
    return (res, hits) if count_hits else res
