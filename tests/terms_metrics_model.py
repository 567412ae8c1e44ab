"""An independent model of a terms aggregation with metric sub-aggregations (bucket/term_agg/mod.rs, intermediate_agg_result.rs:869-1010
and metric/stats.rs:325-356 @ v0.26.0), written without the device's guard.  The rules it pins:

1. Which docs feed a term: every doc the terms count (collect_terms_with_docs) goes to its key's bucket -- the missing key's
   included, which on a numeric column merges with an equal value -- and each column collects what metrics_model.doc_values says.
   A term's doc_count is the terms count, separate from a column's metric count.
2. The segment cut for `_count` / `_key` is terms_model.cut.
3. The segment cut for a metric: each entry's compute_metric_value(...).unwrap_or(0.0) -- count as f64; the Kahan sum (0.0 without
   values); sum / count, min, max when count > 0, else 0.0 -- compared as partial_cmp does (-0.0 equals +0.0), only when there are
   more than segment_size entries.  Equal values keep the lowest keys (the reference's select_nth_unstable_by leaves them
   unspecified), and the scalars follow that order: the doc count at position segment_size is term_doc_count_before_cutoff, the cut
   doc counts add up to sum_other_doc_count.
4. The final order for a metric: the merged value, unwrap_or(f64::MIN) (null for an avg, min or max without values), under
   total_cmp (-0.0 before +0.0), equal values by key ascending; sum_other_doc_count is the segments' plus the final cut's.

Per segment the docs are walked in doc order and collected with Kahan summation (metrics_model.Stats); the segments merge with
merge_fruits in segment_ord order."""
import struct

import numpy as np

from tantivy_b200 import terms as Tm
from tests import metrics_model as MM
from tests import terms_model as TM

F64_MIN = -MM.F64_MAX


def segment_docs(images, present, selected, missing_image=None):
    """{image: [doc, ...]} of one segment: the docs the terms count under each key, in doc order."""
    images = np.asarray(images, dtype=np.uint64)
    sel = np.asarray(selected, bool)
    has = sel if present is None else sel & np.asarray(present, bool)
    out = {}
    for d in np.nonzero(sel)[0].tolist():
        if has[d]:
            out.setdefault(int(images[d]), []).append(d)
        elif missing_image is not None:
            out.setdefault(int(missing_image), []).append(d)
    return {k: sorted(v) for k, v in out.items()}


def collect(values, docs):
    st = MM.Stats()
    for d in docs:
        for v in values[d]:
            st.collect(v)
    return st


def segment_value(st, prop):
    """compute_metric_value(...).unwrap_or(0.0) (rule 3); prop in count, sum, avg, min, max."""
    if prop == "count":
        return float(st.count)
    if prop == "sum":
        return st.sum
    if st.count == 0:
        return 0.0
    return {"avg": st.sum / st.count, "min": st.min, "max": st.max}[prop]


def cut(entries, segment_size, target, asc, order=None):
    """(kept {image: (doc_count, stats)}, error_bound, sum_other) of one segment's {image: (doc_count, {metric key: Stats})}; target
    "_count", "_key" or "metric" with order = (metric key, prop)."""
    if target != "metric":
        kept, e, o = TM.cut({k: c for k, (c, _) in entries.items()}, segment_size, target == "_key", asc)
        return {k: entries[k] for k, _ in kept}, e, o
    items = sorted((k, c, segment_value(st[order[0]], order[1])) for k, (c, st) in entries.items())
    if len(items) <= segment_size:
        return dict((k, entries[k]) for k, _, _ in items), 0, 0
    ranked = sorted(items, key=lambda x: (x[2] if asc else -x[2], x[0]))
    return {k: entries[k] for k, _, _ in ranked[:segment_size]}, ranked[segment_size][1], sum(c for _, c, _ in ranked[segment_size:])


def merge(results):
    """merge_fruits of the segments' ({key: (doc_count, stats)}, sum_other, error) in segment_ord order."""
    out, other, error = {}, 0, 0
    for entries, o, e in results:
        for k, (c, st) in entries.items():
            if k not in out:
                out[k] = (c, {m: _copy(s) for m, s in st.items()})
                continue
            c0, s0 = out[k]
            for m, s in st.items():
                s0[m].merge_fruits(s)
            out[k] = (c0 + c, s0)
        other += o
        error += e
    return out, other, error


def _copy(st):
    c = MM.Stats()
    c.count, c.sum, c.delta, c.min, c.max = st.count, st.sum, st.delta, st.min, st.max
    return c


def _total(v):
    b = struct.unpack("<q", struct.pack("<d", v))[0]
    return b ^ ((b >> 63) & 0x7FFFFFFFFFFFFFFF)


def final(name, req, merged, metrics, order=None):
    """{name: the terms' final result}: metrics = [(agg name, type, metric key, none_if_no_match)], order = (agg name, prop) for a
    metric order."""
    entries, other, error = merged
    buckets = sorted(((k, c, st) for k, (c, st) in entries.items() if c >= req.min_doc_count), key=lambda b: Tm._key_order(b[0]))
    results = {k: {a: MM.final(st[key], typ, nim) for a, typ, key, nim in metrics} for k, _, st in buckets}
    if req.order_target == "_key":
        buckets.sort(key=lambda b: Tm._key_order(b[0]), reverse=req.order == "desc")
    elif order is not None:
        def value(b):
            res = results[b[0]][order[0]]
            v = res["value"] if "value" in res else res[order[1]]
            return F64_MIN if v is None else float(v)
        buckets.sort(key=lambda b: _total(value(b)), reverse=req.order == "desc")
    else:
        buckets.sort(key=lambda b: b[1], reverse=req.order == "desc")
    out = []
    for k, c, _ in buckets[:req.size]:
        e = {"key": Tm._final_key(k)[1], "doc_count": c}
        if k[0] == "bool":
            e["key_as_string"] = "true" if k[1] else "false"
        e.update(results[k])
        out.append(e)
    res = {"buckets": out, "sum_other_doc_count": other + sum(c for _, c, _ in buckets[req.size:])}
    if req.show_term_doc_count_error:
        res["doc_count_error_upper_bound"] = error
    return {name: res}
