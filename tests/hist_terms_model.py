"""An independent model of a histogram whose only sub-aggregation is a terms (bucket/histogram/histogram.rs and
bucket/term_agg/mod.rs @ v0.26.0).  The rules it pins:

1. Which docs feed a bucket's terms: every doc the histogram counts in bucket pos (SegmentHistogramCollector::collect's
   sub-aggregation branch, histogram.rs:490-505): it has a histogram value inside the segment's bounds after
   normalize_histogram_req's collapse (histogram_model.segment_bounds), pos = as_i64(floor((val - offset) / interval)).  Within the
   bucket a doc counts under its image, under the missing image, or nowhere.
2. A bucket's doc_count is the histogram count: docs without a terms value and without a missing key count in it.
3. Each (segment, bucket) is cut on its own by terms_model.cut (one HashMapTermBuckets per bucket), with its own
   term_doc_count_before_cutoff and sum_other_doc_count.
4. Segments merge with merge_fruits in segment_ord order: by pos, then within a bucket by key.
5. The histogram's buckets are finalised by histogram.final_buckets; each holds its terms ordered and cut to size (count then key
   ascending, or key), and a bucket that only gap filling or extended_bounds adds holds the terms' empty result.  The whole result
   counts 1 plus its kept terms per histogram bucket against the bucket limit.

Per segment the docs are walked one at a time in doc order, each given its pos and its key."""
import numpy as np

from tantivy_b200 import histogram as Hg
from tantivy_b200 import terms as Tm
from tests import histogram_model as HM
from tests import terms_model as TM


def segment(keys, key_present, values, value_present, selected, kind, interval, offset, hard_min, hard_max, missing_image=None):
    """{pos: (doc_count, {image: doc_count})} of one segment (rules 1, 2): `selected` = the docs the query collects."""
    lo, hi = HM.segment_bounds(values, value_present, kind, hard_min, hard_max)
    vals = HM.image_to_f64(np.asarray(values, dtype=np.uint64), kind)
    out = {}
    for d in np.nonzero(np.asarray(selected, bool))[0].tolist():
        if value_present is not None and not value_present[d]:
            continue
        v = float(vals[d])
        if not lo <= v <= hi:
            continue
        p = int(HM.as_i64(np.floor((np.float64(v) - np.float64(offset)) / np.float64(interval))))
        c, t = out.get(p, (0, {}))
        if key_present is None or key_present[d]:
            k = int(keys[d])
            t[k] = t.get(k, 0) + 1
        elif missing_image is not None:
            t[int(missing_image)] = t.get(int(missing_image), 0) + 1
        out[p] = (c + 1, t)
    return out


def cut(buckets, segment_size, by_key=False, asc=False):
    """{pos: (doc_count, kept [(image, doc_count)] ascending, error_bound, sum_other)} of one segment (rule 3)."""
    out = {}
    for p, (c, t) in buckets.items():
        kept, e, o = TM.cut(t, segment_size, by_key, asc)
        out[p] = (c, kept, e, o)
    return out


def merge(results):
    """Rule 4 over [{pos: (doc_count, {key: doc_count}, sum_other, error)}] in segment_ord order: {pos: (doc_count, {key: n},
    sum_other, error)}."""
    out = {}
    for r in results:
        for p, (c, t, o, e) in r.items():
            c0, t0, o0, e0 = out.get(p, (0, {}, 0, 0))
            t1 = dict(t0)
            for k, n in t.items():
                t1[k] = t1.get(k, 0) + n
            out[p] = (c0 + c, t1, o0 + o, e0 + e)
    return out


def final(name, hist_req, hist_kind, terms_name, req, merged, bucket_limit=Hg.DEFAULT_BUCKET_LIMIT):
    """Rule 5: {name: result}, or raises histogram.AggregationError over the bucket limit."""
    out, total = [], 0
    for key, count, pos in Hg.final_buckets(hist_req, {p: v[0] for p, v in merged.items()}, hist_kind, bucket_limit):
        _, t, other, error = merged[pos] if pos is not None else (0, {}, 0, 0)
        items = [(k, c) for k, c in t.items() if c >= req.min_doc_count]
        if req.order_target == "_key":
            items.sort(key=lambda b: Tm._key_order(b[0]), reverse=req.order == "desc")
        else:
            items.sort(key=lambda b: (-b[1] if req.order == "desc" else b[1], Tm._key_order(b[0])))
        buckets = []
        for k, c in items[:req.size]:
            e = {"key": Tm._final_key(k)[1], "doc_count": c}
            if k[0] == "bool":
                e["key_as_string"] = "true" if k[1] else "false"
            buckets.append(e)
        res = {"buckets": buckets, "sum_other_doc_count": other + sum(c for _, c in items[req.size:])}
        if req.show_term_doc_count_error:
            res["doc_count_error_upper_bound"] = error
        total += 1 + len(buckets)
        e = Hg.bucket_entry(key, count, hist_kind)
        e[terms_name] = res
        out.append(e)
    if total > bucket_limit:
        raise Hg.AggregationError(f"Aborting aggregation because bucket limit was exceeded. Limit: {bucket_limit}, Current: {total}")
    return {name: Hg.keyed_or_list(hist_req, out)}
