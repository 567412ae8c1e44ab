"""The request and result side of a `histogram` / `date_histogram` whose only sub-aggregation is a `terms` (the "top values per
interval" chart: the top hosts or status codes in each minute), for the device's intermediate results (Context.hist_terms_batch).
Pure Python: it parses a request of one top-level histogram over exactly one terms with nothing under it, refuses what the device
does not run (HistTermsRefused: take the CPU path), maps the request to one histogram spec and one terms spec, merges the rows of any
number of contexts by bucket pos -- within a bucket per (segment, image), cutting once per segment a segment split over contexts, then
by intermediate key -- and finalises to tantivy's result: the histogram's buckets (tantivy_b200.histogram) each holding {name: its
terms} (tantivy_b200.terms).

A bucket's terms collect every doc the histogram counts in it (the sub-aggregation branch of SegmentHistogramCollector::collect,
histogram.rs:490-505): under its image, under the missing key, or nowhere.  A bucket's doc_count is the histogram count.  Each
(segment, bucket) is cut to segment_size on its own (one HashMapTermBuckets per bucket, cut when the histogram emits it), with its own
term_doc_count_before_cutoff and sum_other_doc_count.  A bucket that only gap filling or extended_bounds adds holds the terms' empty
result, and the whole result is checked against the bucket limit as get_bucket_count counts it: each histogram bucket is 1 plus its
kept terms."""
import re
from dataclasses import dataclass

import numpy as np

from . import histogram as Hg
from . import terms as Tm
from .histogram import AggregationError
from .lib import TqError
from .terms_hist import _one_type, _subset

_HISTOGRAMS = ("histogram", "date_histogram")
_HIST_KINDS = ("u64", "i64", "f64", "bool", "date")
_METRICS = ("avg", "sum", "min", "max", "stats", "value_count")


class HistTermsRefused(ValueError):
    """A histogram request with a terms sub-aggregation that the device does not answer exactly; the caller takes the CPU path."""


@dataclass
class HistTermsRequest:
    """One top-level histogram: its name, request (HistogramAggregation, a date request in milliseconds) and whether it was a
    date_histogram, and its one terms: name and request (terms.TermsAggregation)."""
    name: str
    hist_req: Hg.HistogramAggregation
    is_date_histogram: bool
    terms_name: str
    req: Tm.TermsAggregation


@dataclass
class HistTermsPlan:
    """The two fields' kinds and the specs for Context.hist_terms_batch."""
    request: HistTermsRequest
    hist_kind: str
    kind: str
    hspec: tuple
    tspec: tuple


def parse_request(aggs):
    """An Aggregations map {name: {"histogram" | "date_histogram": {...}, "aggs": {terms_name: {"terms": {...}}}}} ->
    HistTermsRequest.  Every request the device does not run raises HistTermsRefused with its own message; a malformed one
    AggregationError."""
    if not isinstance(aggs, dict) or not aggs:
        raise AggregationError("expected a non-empty map of aggregations")
    if len(aggs) != 1:
        raise HistTermsRefused("more than one top-level aggregation runs on the CPU path")
    (name, agg), = aggs.items()
    typ, sub = _one_type(name, agg)
    if typ == "range":
        raise HistTermsRefused(f"{name}: a terms sub-aggregation under a range runs on the CPU path")
    if typ not in _HISTOGRAMS:
        raise HistTermsRefused(f"{name}: a top-level {typ} is not a histogram with a terms sub-aggregation")
    if not sub:
        raise HistTermsRefused(f"{name}: a histogram without sub-aggregations runs through tantivy_b200.histogram")
    if not isinstance(sub, dict):
        raise AggregationError(f"{name}: `aggs` is not a map")
    if len(sub) != 1:
        raise HistTermsRefused(f"{name}: more than one sub-aggregation under the histogram runs on the CPU path")
    (tname, tagg), = sub.items()
    ttyp, tsub = _one_type(f"{name}.{tname}", tagg)
    if ttyp in _METRICS:
        raise HistTermsRefused(f"{name}.{tname}: a {ttyp} under the histogram is a metric sub-aggregation (tantivy_b200.hist_metrics)")
    if ttyp != "terms":
        raise HistTermsRefused(f"{name}.{tname}: a {ttyp} under the histogram is not a terms sub-aggregation (the CPU path)")
    if tsub:
        raise HistTermsRefused(f"{name}.{tname}: aggregations nested under the terms run on the CPU path")
    req = Tm.TermsAggregation.from_dict(tagg["terms"])
    if req.order_target not in ("_count", "_key"):  # (the terms has no sub-aggregation to order by: term_agg/mod.rs:363-371)
        raise AggregationError(f"could not find aggregation with name {req.order_target.partition('.')[0]} in metric sub_aggregations")
    hreq, is_date = Hg.parse_request({typ: agg[typ]})
    hreq.validate()
    return HistTermsRequest(name=name, hist_req=hreq, is_date_histogram=is_date, terms_name=tname, req=req)


def plan(r: HistTermsRequest, fields):
    """HistTermsRequest and {field name: metrics.MetricField} -> HistTermsPlan: the histogram spec (histogram.histogram_spec) and
    the terms spec (terms.terms_spec)."""
    h = fields.get(r.hist_req.field)
    if h is None:
        raise HistTermsRefused(f"{r.name}: field {r.hist_req.field!r} has no registered fast column")
    if h.n_column_types != 1:
        raise HistTermsRefused(f"{r.name}: a histogram on a field of several column types (JSON) runs on the CPU path")
    if h.multi_valued:
        raise HistTermsRefused(f"{r.name}: a histogram on a multi-valued column runs on the CPU path")
    if h.kind not in _HIST_KINDS:
        raise HistTermsRefused(f"{r.name}: a histogram on a {h.kind} column runs on the CPU path")
    where = f"{r.name}.{r.terms_name}"
    f = fields.get(r.req.field)
    if f is None:
        raise HistTermsRefused(f"{where}: field {r.req.field!r} has no registered fast column")
    try:
        Tm.check_device(r.req, f.kind, f.multi_valued, f.n_column_types)
        tspec = Tm.terms_spec(r.req, f.column_id, f.kind)
    except Tm.TermsRefused as e:
        raise HistTermsRefused(f"{where}: {e}") from None
    return HistTermsPlan(request=r, hist_kind=h.kind, kind=f.kind, hspec=Hg.histogram_spec(r.hist_req, h.column_id, h.kind), tspec=tspec)


# ---- rows, merges, final result --------------------------------------------------------------------------------------------------
@dataclass
class Rows:
    """Query q of Context.hist_terms_batch's output as arrays: per bucket pos, doc_count, sum_other, error; per entry its bucket's
    index, segment_ord, image and doc_count, in row order."""
    pos: np.ndarray
    doc_count: np.ndarray
    other: np.ndarray
    error: np.ndarray
    bucket: np.ndarray
    seg: np.ndarray
    key: np.ndarray
    count: np.ndarray


def rows_of(out, q):
    """Query q of Context.hist_terms_batch's output as Rows (numpy slices and one np.repeat: no per-entry Python)."""
    pos, docs, other, error, first, nent, n, eseg, ekey, ecount = out[:10]
    nb = int(n[q])
    ne = nent[q, :nb].astype(np.int64)
    a = int(first[q, 0]) if nb else 0
    b = a + int(ne.sum())
    return Rows(pos[q, :nb].copy(), docs[q, :nb].copy(), other[q, :nb].copy(), error[q, :nb].copy(), np.repeat(np.arange(nb), ne),
                eseg[a:b].copy(), ekey[a:b].copy(), ecount[a:b].copy())


def _sum_by_pos(rows_list):
    """The buckets of every context summed by pos: (pos, doc_count, sum_other, error) arrays, and the entries (pos, segment_ord,
    image, doc_count) summed per (pos, segment_ord, image), ordered by them.  A segment split over contexts comes back uncut from
    each: its entries add here."""
    pos = np.concatenate([r.pos for r in rows_list]) if rows_list else np.zeros(0, np.int64)
    u, inv = np.unique(pos, return_inverse=True)
    sums = [np.zeros(len(u), dtype=np.uint64) for _ in range(3)]
    for s, name in zip(sums, ("doc_count", "other", "error")):
        np.add.at(s, inv, np.concatenate([getattr(r, name) for r in rows_list]).astype(np.uint64))
    ep = np.concatenate([r.pos[r.bucket] for r in rows_list]) if rows_list else np.zeros(0, np.int64)
    es = np.concatenate([r.seg for r in rows_list]).astype(np.int64) if rows_list else np.zeros(0, np.int64)
    ek = np.concatenate([r.key for r in rows_list]) if rows_list else np.zeros(0, np.uint64)
    ec = np.concatenate([r.count for r in rows_list]).astype(np.uint64) if rows_list else np.zeros(0, np.uint64)
    order = np.lexsort((ek, es, ep))
    ep, es, ek, ec = ep[order], es[order], ek[order], ec[order]
    new = np.ones(len(ep), bool)
    new[1:] = (ep[1:] != ep[:-1]) | (es[1:] != es[:-1]) | (ek[1:] != ek[:-1])
    starts = np.nonzero(new)[0]
    ec = np.add.reduceat(ec, starts) if len(starts) else ec
    return (u, sums[0], sums[1], sums[2]), (ep[starts], es[starts], ek[starts], ec)


def bucket_terms(p: HistTermsPlan, segments, dictionaries=None, missing_images=None):
    """One bucket's terms, merged: segments = [(segment_ord, {image: doc_count})] in segment_ord order, each cut once
    (terms.cut_segment: a whole segment, cut on the device already, is not cut again) and mapped to intermediate keys
    (terms.segment_result).  Returns ({key: doc_count}, sum_other, error_bound) of the cuts made here."""
    req = p.request.req
    results = []
    for s, entries in segments:
        kept, e, o = Tm.cut_segment(entries, req)
        results.append((Tm.segment_result(req, p.kind, kept, None if dictionaries is None else dictionaries[s],
                                          None if missing_images is None else missing_images.get(s)), o, e))
    return Tm.merge(results)


def terms_result(req: Tm.TermsAggregation, merged):
    """The terms' final result of merge()'s ({key: doc_count}, sum_other, error) (terms.finalize), and its kept bucket count."""
    kept, cut = Tm.ordered_buckets(req, merged[0])
    res = {"buckets": [Tm.bucket_entry(k, c) for k, c in kept], "sum_other_doc_count": merged[1] + cut}
    if req.show_term_doc_count_error:
        res["doc_count_error_upper_bound"] = merged[2]
    return res, len(kept)


def finalize(p: HistTermsPlan, merged, bucket_limit=Hg.DEFAULT_BUCKET_LIMIT):
    """{name: the histogram's final result} from {pos: (doc_count, ({key: doc_count}, sum_other, error))}: the histogram's buckets
    as histogram.final_buckets gives them (gap filling, extended_bounds, hard_bounds, min_doc_count), each holding {terms_name: its
    terms' final result} -- the empty result (empty_from_req) for a bucket the histogram adds -- and the bucket limit over the whole
    result (AggregationError)."""
    r = p.request
    out, total = [], 0
    for key, count, pos in Hg.final_buckets(r.hist_req, {q: c for q, (c, _) in merged.items()}, p.hist_kind, bucket_limit):
        res, n = terms_result(r.req, merged[pos][1] if pos is not None else ({}, 0, 0))
        total += 1 + n
        e = Hg.bucket_entry(key, count, p.hist_kind)
        e[r.terms_name] = res
        out.append(e)
    if total > bucket_limit:  # (get_bucket_count over the whole result)
        raise AggregationError(f"Aborting aggregation because bucket limit was exceeded. Limit: {bucket_limit}, Current: {total}")
    return {r.name: Hg.keyed_or_list(r.hist_req, out)}


def finalize_rows(p: HistTermsPlan, rows_list, dictionaries=None, missing_images=None, bucket_limit=Hg.DEFAULT_BUCKET_LIMIT):
    """The final result of one query from its Rows of any number of contexts: per bucket the doc counts and scalars summed, per
    (segment, bucket) the entries summed over the contexts and cut once, merged by intermediate key in segment_ord order, then
    finalize.  dictionaries[segment_ord] = a str segment's terms, missing_images[segment_ord] = its missing image."""
    (pos, docs, other, error), (ep, es, ek, ec) = _sum_by_pos(rows_list)
    merged = {}
    bounds = np.searchsorted(ep, pos, side="left").tolist() + [len(ep)]
    es_l, ek_l, ec_l = es.tolist(), ek.tolist(), ec.tolist()
    for i, q in enumerate(pos.tolist()):
        segments, j, b = [], bounds[i], bounds[i + 1]
        while j < b:
            s, entries = es_l[j], {}
            while j < b and es_l[j] == s:
                entries[ek_l[j]] = int(ec_l[j])
                j += 1
            segments.append((s, entries))
        ent, o, e = bucket_terms(p, segments, dictionaries, missing_images)
        merged[q] = (int(docs[i]), (ent, int(other[i]) + o, int(error[i]) + e))
    return finalize(p, merged, bucket_limit)


_UNSUPPORTED = re.compile(r"^tantivy_b200 error -4: query (\d+): (.*)$")


def run(contexts, qb, requests, fields, count_hits=False, dictionaries=None, missing_images=None):
    """Runs one parsed request per query of qb over every Context (each evaluating its own segments or doc ranges) and finalises.
    Returns [{name: result}, AggregationError or HistTermsRefused] per query, and the merged hit counts with count_hits.  A query
    the device refuses as too wide (TQ_ERR_UNSUPPORTED naming it: its keys, buckets or grid exceed the device's limits) becomes a
    HistTermsRefused with that reason, and the batch runs again without it; its hit count is then 0 here."""
    plans = [plan(r, fields) for r in requests]
    live, refused = list(range(qb.nq)), {}
    while True:
        sub = qb if len(live) == qb.nq else _subset(qb, live)
        per_ctx, hits = [], np.zeros(qb.nq, dtype=np.uint64)
        try:
            for ctx in contexts:
                out = ctx.hist_terms_batch(sub, [plans[q].hspec for q in live], [plans[q].tspec for q in live], count_hits=count_hits)
                if count_hits:
                    hits[live] += out[11]
                per_ctx.append(out)
            break
        except TqError as e:
            m = _UNSUPPORTED.match(str(e))
            if not m or int(m.group(1)) >= len(live):
                raise
            q = live.pop(int(m.group(1)))
            refused[q] = HistTermsRefused(f"{plans[q].request.name}: {m.group(2)}")
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
