"""An independent model of a histogram with metric sub-aggregations (SegmentHistogramCollector::collect with a sub-aggregation,
bucket/histogram/histogram.rs:490-505, and metric/stats.rs @ v0.26.0), written without the device's guard: per segment, walk the
docs the query collects in doc order; bucket each by its histogram value as tests/histogram_model.py does (the per-segment bounds,
the bounds test, get_bucket_pos_f64 as i64); feed the doc's values to the bucket's IntermediateStats of every metric with Kahan
summation (tests/metrics_model.py: its value, the missing value, 0.0 on a count-only column); then merge the segments' buckets by
pos in segment_ord order -- a bucket new to the merge is taken as it is, one already there merge_fruits it -- and finalise with
tantivy_b200.histogram's buckets and metrics_model.final."""
import numpy as np

from tantivy_b200 import histogram as Hg
from tests import histogram_model as HM
from tests import metrics_model as MM


def segment_buckets(images, present, selected, kind, interval, offset, hard_min=-HM.F64_MAX, hard_max=HM.F64_MAX):
    """{pos: [doc, ...]} of one segment: the docs the histogram counts in each bucket, in doc order."""
    lo, hi = HM.segment_bounds(images, present, kind, hard_min, hard_max)
    sel = np.asarray(selected, bool).copy()
    if present is not None:
        sel &= np.asarray(present, bool)
    docs = np.nonzero(sel)[0]
    val = HM.image_to_f64(np.asarray(images, dtype=np.uint64)[docs], kind)
    with np.errstate(invalid="ignore"):
        keep = (val >= lo) & (val <= hi)
        pos = HM.as_i64(np.floor((val[keep] - np.float64(offset)) / np.float64(interval)))
    out = {}
    for d, p in zip(docs[keep].tolist(), pos.tolist()):
        out.setdefault(int(p), []).append(d)
    return out


def collect(values, docs):
    """IntermediateStats::collect of values[d] for each doc d in order (values[d]: the list a doc adds, metrics_model.doc_values)."""
    st = MM.Stats()
    for d in docs:
        for v in values[d]:
            st.collect(v)
    return st


def segment_part(buckets, metric_values):
    """{pos: (doc_count, {metric key: Stats})} of one segment: metric_values maps a key to the per-doc value lists."""
    return {p: (len(docs), {k: collect(vals, docs) for k, vals in metric_values.items()}) for p, docs in buckets.items()}


def merge(parts):
    """The segments' parts, given in segment_ord order, merged by pos."""
    out = {}
    for part in parts:
        for p, (n, stats) in part.items():
            if p not in out:
                out[p] = (n, stats)
                continue
            n0, s0 = out[p]
            for k, st in stats.items():
                s0[k].merge_fruits(st)
            out[p] = (n0 + n, s0)
    return out


def final(name, req, kind, merged, metrics):
    """{name: the histogram's final result}: metrics = [(agg name, type, metric key, none_if_no_match)]."""
    buckets = Hg.final_buckets(req, {p: n for p, (n, _) in merged.items()}, kind)
    out = []
    for key, count, pos in buckets:
        e = Hg.bucket_entry(key, count, kind)
        for a, typ, k, nim in metrics:
            e[a] = MM.final(merged[pos][1][k] if pos is not None else MM.Stats(), typ, nim)
        out.append(e)
    return {name: Hg.keyed_or_list(req, out)}
