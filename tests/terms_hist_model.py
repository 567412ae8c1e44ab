"""An independent model of a terms aggregation whose only sub-aggregation is a histogram (bucket/term_agg/mod.rs,
term_agg/term_histogram.rs and bucket/histogram/histogram.rs @ v0.26.0).  The rules it pins:

1. Which docs feed a term's histogram: every doc the terms count under a key (collect_terms_with_docs), the missing key's included;
   within it a doc counts in bucket pos = as_i64(floor((val - offset) / interval)) when it has a histogram value inside the
   segment's bounds after normalize_histogram_req's collapse (histogram_model.segment_bounds).
2. A term's doc_count is the terms count: docs without a histogram value or outside hard_bounds count in it.
3. The segment cut is terms_model.cut; a cut term's histogram is dropped.
4. Segments merge with merge_fruits in segment_ord order: by key, then by pos.
5. The final terms are ordered and cut to size as terms.finalize does; each kept term's histogram is finalised on its own
   (histogram.final_buckets), and the whole result counts 1 plus its histogram's buckets per kept term against the bucket limit.

Per segment the docs are walked one at a time in doc order, each given its key and its pos."""
import numpy as np

from tantivy_b200 import histogram as Hg
from tantivy_b200 import terms as Tm
from tests import histogram_model as HM
from tests import terms_model as TM


def segment(keys, key_present, values, value_present, selected, kind, interval, offset, hard_min, hard_max, missing_image=None):
    """{image: (doc_count, {pos: doc_count})} of one segment (rules 1, 2): `selected` = the docs the query collects."""
    lo, hi = HM.segment_bounds(values, value_present, kind, hard_min, hard_max)
    vals = HM.image_to_f64(np.asarray(values, dtype=np.uint64), kind)
    out = {}
    for d in np.nonzero(np.asarray(selected, bool))[0].tolist():
        if key_present is None or key_present[d]:
            k = int(keys[d])
        elif missing_image is not None:
            k = int(missing_image)
        else:
            continue
        c, h = out.get(k, (0, {}))
        if value_present is None or value_present[d]:
            v = float(vals[d])
            if lo <= v <= hi:
                p = int(HM.as_i64(np.floor((np.float64(v) - np.float64(offset)) / np.float64(interval))))
                h[p] = h.get(p, 0) + 1
        out[k] = (c + 1, h)
    return out


def cut(entries, segment_size, by_key=False, asc=False):
    """(kept {image: (doc_count, hist)}, error_bound, sum_other) of one segment (rule 3)."""
    kept, e, o = TM.cut({k: c for k, (c, _) in entries.items()}, segment_size, by_key, asc)
    return {k: entries[k] for k, _ in kept}, e, o


def merge(results):
    """Rule 4 over [({key: (doc_count, hist)}, sum_other, error)] in segment_ord order."""
    entries, other, error = {}, 0, 0
    for e, o, err in results:
        for k, (c, h) in e.items():
            c0, h0 = entries.get(k, (0, {}))
            h1 = dict(h0)
            for p, n in h.items():
                h1[p] = h1.get(p, 0) + n
            entries[k] = (c0 + c, h1)
        other += o
        error += err
    return entries, other, error


def final(name, req, hist_name, hist_req, hist_kind, merged, bucket_limit=Hg.DEFAULT_BUCKET_LIMIT):
    """Rule 5: {name: result}, or raises histogram.AggregationError over the bucket limit."""
    entries, other, error = merged
    items = [(k, c, h) for k, (c, h) in entries.items() if c >= req.min_doc_count]
    if req.order_target == "_key":
        items.sort(key=lambda b: Tm._key_order(b[0]), reverse=req.order == "desc")
    else:  # (count, then key ascending)
        items.sort(key=lambda b: (-b[1] if req.order == "desc" else b[1], Tm._key_order(b[0])))
    buckets, total = [], 0
    for k, c, h in items[:req.size]:
        hb = Hg.final_buckets(hist_req, h, hist_kind, bucket_limit)
        total += 1 + len(hb)
        e = {"key": Tm._final_key(k)[1], "doc_count": c}
        if k[0] == "bool":
            e["key_as_string"] = "true" if k[1] else "false"
        e[hist_name] = Hg.keyed_or_list(hist_req, [Hg.bucket_entry(key, n, hist_kind) for key, n, _ in hb])
        buckets.append(e)
    if total > bucket_limit:
        raise Hg.AggregationError(f"Aborting aggregation because bucket limit was exceeded. Limit: {bucket_limit}, Current: {total}")
    res = {"buckets": buckets, "sum_other_doc_count": other + sum(c for _, c, _ in items[req.size:])}
    if req.show_term_doc_count_error:
        res["doc_count_error_upper_bound"] = error
    return {name: res}
