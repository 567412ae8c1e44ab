"""An independent model of the range aggregation (bucket/range.rs, agg_data.rs and intermediate_agg_result.rs @ v0.26.0), with or
without metric sub-aggregations, written from the reference's rules rather than from tantivy_b200.ranges:

- f64_to_fastfield_u64 of each bound for the column type (u64 `v as u64`, i64 / date `(v as i64)` to its image, f64 to_u64);
- extend_validate_ranges: sort stably by start, prepend 0..first.start and append last.end..u64::MAX, fill the holes, and the
  overlap error when an end exceeds the next start;
- get_bucket_pos: binary search of the image over the starts, `Err(p) => p - 1`;
- the intermediate key range_to_string(start..end) and the final entries (custom key, from / to, the date strings), sorted by
  from.unwrap_or(f64::MIN) under total_cmp, as a map when keyed;
- per bucket, Kahan collection of every metric in doc order (tests/hist_metrics_model.collect), the segments merged by key in
  segment_ord order."""
import bisect
import struct

import numpy as np

from tantivy_b200.histogram import format_date, rust_f64_display
from tests import hist_metrics_model as HMM
from tests import metrics_model as MM

U64_MAX = (1 << 64) - 1
F64_MIN = -1.7976931348623157e308


class Overlap(ValueError):
    pass


def rust_as_i64(v):
    if v != v:
        return 0
    if v >= 2.0**63:
        return (1 << 63) - 1
    if v < -(2.0**63):
        return -(1 << 63)
    return int(v)


def to_u64(v, kind):
    """f64_to_fastfield_u64."""
    if kind == "u64":
        return 0 if v != v or v <= 0 else (U64_MAX if v >= 2.0**64 else int(v))
    if kind in ("i64", "date"):
        return rust_as_i64(v) + (1 << 63)
    bits = struct.unpack("<Q", struct.pack("<d", v))[0]
    return bits | (1 << 63) if bits >> 63 == 0 else (~bits) & U64_MAX


def from_u64(image, kind):
    """f64_from_fastfield_u64."""
    if kind == "u64":
        return float(image)
    if kind in ("i64", "date"):
        return float(image - (1 << 63))
    bits = image & ~(1 << 63) if image >> 63 else (~image) & U64_MAX
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def extend_validate(ranges, kind):
    """[(key, from, to)] -> [(key, start, end)]."""
    conv = [(k, 0 if f is None else to_u64(f, kind), U64_MAX if t is None else to_u64(t, kind)) for k, f, t in ranges]
    conv.sort(key=lambda b: b[1])
    if conv[0][1] != 0:
        conv.insert(0, (None, 0, conv[0][1]))
    if conv[-1][2] != U64_MAX:
        conv.append((None, conv[-1][2], U64_MAX))
    while True:
        hole = None
        for i in range(len(conv) - 1):
            if conv[i][2] > conv[i + 1][1]:
                raise Overlap(f"Overlapping ranges not supported: {conv[i]} {conv[i + 1]}")
            if conv[i][2] != conv[i + 1][1]:
                hole = i
                break
        if hole is None:
            return conv
        conv.insert(hole + 1, (None, conv[hole][2], conv[hole + 1][1]))


def bucket_pos(image, starts):
    """get_bucket_pos (starts strictly ascending from 0)."""
    return bisect.bisect_right(starts, image) - 1


def range_string(start, end, kind):
    def half(v, is_start):
        if (is_start and v == 0) or (not is_start and v == U64_MAX):
            return "*"
        if kind == "date":
            return format_date(v - (1 << 63))
        return rust_f64_display(from_u64(v, kind))
    return half(start, True) + "-" + half(end, False)


def total_cmp_key(x):
    b = struct.unpack("<q", struct.pack("<d", x))[0]
    return b ^ 0x7FFFFFFFFFFFFFFF if b < 0 else b


def segment_buckets(images, present, selected, starts):
    """[docs of bucket b, in doc order] of one segment: the selected docs with a value."""
    sel = np.asarray(selected, bool).copy()
    if present is not None:
        sel &= np.asarray(present, bool)
    docs = np.nonzero(sel)[0]
    pos = np.searchsorted(np.asarray(starts, dtype=np.uint64), np.asarray(images, dtype=np.uint64)[docs], side="right") - 1
    out = [[] for _ in starts]
    for d, b in zip(docs.tolist(), pos.tolist()):
        out[b].append(d)
    return out


def result(name, ranges, kind, keyed, seg_buckets, metric_values=None, metrics=()):
    """{name: the range's final result} from the segments' bucket doc lists (given in segment_ord order, each [docs per bucket] of
    extend_validate(ranges, kind)), with metrics = [(agg name, type, metric key, none_if_no_match)] over metric_values[segment]
    {metric key: per-doc value lists}."""
    ext = extend_validate(ranges, kind)
    merged = {}
    for si, buckets in enumerate(seg_buckets):
        for (key, s, e), docs in zip(ext, buckets):
            k = range_string(s, e, kind)
            stats = {mk: HMM.collect(vals, docs) for mk, vals in (metric_values[si] if metric_values else {}).items()}
            if k not in merged:
                merged[k] = [len(docs), stats]
            else:
                merged[k][0] += len(docs)
                for mk, st in stats.items():
                    merged[k][1][mk].merge_fruits(st)
    out = []
    for key, s, e in ext:
        k = range_string(s, e, kind)
        n, stats = merged.get(k, (0, {}))
        entry = {"key": key if key is not None else k, "doc_count": n}
        if s != 0:
            entry["from"] = from_u64(s, kind)
        if e != U64_MAX:
            entry["to"] = from_u64(e, kind)
        if kind == "date":
            if "from" in entry:
                entry["from_as_string"] = format_date(int(entry["from"]))
            if "to" in entry:
                entry["to_as_string"] = format_date(int(entry["to"]))
        for a, typ, mk, nim in metrics:
            entry[a] = MM.final(stats.get(mk, MM.Stats()), typ, nim)
        out.append(entry)
    out.sort(key=lambda x: total_cmp_key(x.get("from", F64_MIN)))
    return {name: {"buckets": {x["key"]: x for x in out}} if keyed else {"buckets": out}}
