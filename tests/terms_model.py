"""An independent model of the segment part of a terms aggregation (SegmentTermCollector::collect and
into_intermediate_bucket_result + cut_off_buckets, bucket/term_agg/mod.rs @ v0.26.0), with the device's rule for equal counts at the
cut: (count, then key ascending).  Per segment: every collected doc counts under its u64 image, a doc without a value under the
missing image (if any); the entries are the non-zero keys; more than segment_size are sorted by the order and cut.  Returns the kept
(image, doc_count) pairs in ascending image with term_doc_count_before_cutoff and sum_other_doc_count."""
import numpy as np


def collect(images, present, selected, missing_image=None):
    """{image: doc_count} of one segment: `selected` = the docs the query collects (bool mask, or None for every doc)."""
    images = np.asarray(images, dtype=np.uint64)
    sel = np.ones(len(images), bool) if selected is None else np.asarray(selected, bool)
    has = sel if present is None else sel & np.asarray(present, bool)
    keys, counts = np.unique(images[has], return_counts=True)
    out = {int(k): int(c) for k, c in zip(keys, counts)}
    n_missing = int(sel.sum() - has.sum())
    if missing_image is not None and n_missing:
        out[int(missing_image)] = out.get(int(missing_image), 0) + n_missing
    return out


def cut(entries, segment_size, by_key=False, asc=False):
    """(kept [(image, doc_count)] ascending, error_bound, sum_other) of one segment's {image: doc_count}."""
    items = sorted((k, c) for k, c in entries.items() if c)
    if by_key:
        order = items[::-1] if not asc else items
    else:  # count desc or asc, ties by key ascending
        order = sorted(items, key=lambda kc: (-kc[1] if not asc else kc[1], kc[0]))
    if len(order) <= segment_size:
        return items, 0, 0
    kept = sorted(order[:segment_size])
    return kept, order[segment_size][1], sum(c for _, c in order[segment_size:])
