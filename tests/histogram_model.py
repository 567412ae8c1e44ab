"""An independent model of the segment part of a histogram aggregation (SegmentHistogramCollector, bucket/histogram/histogram.rs
@ v0.26.0): per segment, the bounds after normalize_histogram_req's collapse, each doc's value as f64, the bounds test and
get_bucket_pos_f64 as i64, with Rust's saturating `as` written out (numpy's cast is not saturating).  Returns {pos: doc_count}
per segment; tantivy_b200.histogram.merge_intermediate / finalize take it from there."""
import numpy as np

F64_MAX = float(np.finfo(np.float64).max)
_HIGH = np.uint64(1 << 63)


def image_to_f64(images, kind):
    """f64_from_fastfield_u64 of u64 images (aggregation/mod.rs:374)."""
    u = np.asarray(images, dtype=np.uint64)
    if kind in ("u64", "bool"):
        return u.astype(np.float64)
    if kind in ("i64", "date"):
        return (u ^ _HIGH).view(np.int64).astype(np.float64)
    if kind == "f64":
        return np.where((u & _HIGH) != 0, u ^ _HIGH, ~u).view(np.float64)
    raise ValueError(kind)


def as_i64(f):
    """Rust's `f as i64` on an array: toward zero, saturating at the i64 range, NaN -> 0."""
    f = np.asarray(f, dtype=np.float64)
    out = np.zeros(f.shape, dtype=np.int64)
    ok = np.isfinite(f) & (f < 9223372036854775808.0) & (f >= -9223372036854775808.0)
    out[ok] = f[ok].astype(np.int64)
    out[~np.isnan(f) & (f >= 9223372036854775808.0)] = np.iinfo(np.int64).max
    out[~np.isnan(f) & (f < -9223372036854775808.0)] = np.iinfo(np.int64).min
    return out


def segment_bounds(images, present, kind, hard_min, hard_max):
    """normalize_histogram_req: (lo, hi), collapsed to every finite value when the column's min and max (over the docs with a
    value, in image order) lie inside the hard bounds."""
    u = np.asarray(images, dtype=np.uint64)
    if present is not None:
        u = u[np.asarray(present, bool)]
    if len(u):
        cmin, cmax = image_to_f64(u.min(keepdims=True), kind)[0], image_to_f64(u.max(keepdims=True), kind)[0]
        if cmin >= hard_min and cmax <= hard_max:
            return -F64_MAX, F64_MAX
    return hard_min, hard_max


def collect(images, present, selected, kind, interval, offset, hard_min=-F64_MAX, hard_max=F64_MAX):
    """{pos: doc_count} of one segment: `selected` = the docs the query collects (bool mask, or None for every doc)."""
    lo, hi = segment_bounds(images, present, kind, hard_min, hard_max)
    sel = np.ones(len(images), bool) if selected is None else np.asarray(selected, bool).copy()
    if present is not None:
        sel &= np.asarray(present, bool)
    val = image_to_f64(np.asarray(images, dtype=np.uint64)[sel], kind)
    with np.errstate(invalid="ignore"):
        val = val[(val >= lo) & (val <= hi)]
        pos = as_i64(np.floor((val - np.float64(offset)) / np.float64(interval)))
    keys, counts = np.unique(pos, return_counts=True)
    return {int(k): int(c) for k, c in zip(keys, counts)}


def merge(parts):
    out = {}
    for p in parts:
        for k, c in p.items():
            out[k] = out.get(k, 0) + c
    return out
