"""The request and result side of a `terms` aggregation (src/aggregation/bucket/term_agg/mod.rs), for the device's segment part
(Context.terms_batch).  Pure Python: it parses and validates a request (TermsAggregation, with the defaults of
TermsAggregationInternal::from_req), refuses what the device does not run (TermsRefused: take the CPU path), turns a request into the
device's spec, and finalises the per-segment entries of any number of contexts -- keys mapped per segment, summed by key -- into
tantivy's result: {"buckets": [{"key", "doc_count", "key_as_string"?}], "sum_other_doc_count", "doc_count_error_upper_bound"?}.

Only a top-level terms aggregation without sub-aggregations on a single-valued fast field of one column runs on the device."""
from dataclasses import dataclass
from typing import Optional

import numpy as np

from ._abi import TQ_ORDER_ASC, TQ_ORDER_DESC, TQ_TERMS_BY_COUNT, TQ_TERMS_BY_KEY, TQ_TERMS_MISSING_AFTER_MAX, TQ_TERMS_MISSING_IMAGE, TQ_TERMS_MISSING_NONE
from .histogram import AggregationError, as_i64, format_date

KINDS = ("str", "u64", "i64", "f64", "bool", "date")
_HIGH = 1 << 63
_U64_MAX = (1 << 64) - 1


class TermsRefused(ValueError):
    """A terms request the device does not run; the caller takes the CPU path."""


@dataclass
class TermsAggregation:
    """TermsAggregation (term_agg/mod.rs:204-279) after TermsAggregationInternal::from_req's defaults (:317-335)."""
    field: str
    size: int = 10
    segment_size: int = 100
    show_term_doc_count_error: bool = True
    min_doc_count: int = 1
    order_target: str = "_count"  # "_count", "_key" or the name of a sub-aggregation
    order: str = "desc"
    missing: object = None  # str, int or float (Key), or None
    include: object = None
    exclude: object = None

    @classmethod
    def from_dict(cls, d):
        known = {"field", "size", "segment_size", "shard_size", "split_size", "show_term_doc_count_error", "min_doc_count", "order",
                 "missing", "include", "exclude"}
        unknown = set(d) - known
        if unknown:
            raise AggregationError(f"unknown terms parameter(s) {sorted(unknown)}")
        aliases = [k for k in ("segment_size", "shard_size", "split_size") if k in d]
        if len(aliases) > 1:
            raise AggregationError("duplicate field `segment_size`")
        target, order = "_count", "desc"
        if d.get("order") is not None:
            o = d["order"]
            if not isinstance(o, dict) or len(o) != 1:
                raise AggregationError("order expects one {target: \"asc\" | \"desc\"}")
            (target, order), = o.items()
            if order not in ("asc", "desc"):
                raise AggregationError(f"unknown order {order!r}")
        size = d.get("size")
        size = 10 if size is None else int(size)
        seg = d.get(aliases[0]) if aliases else None
        seg = size * 10 if seg is None else int(seg)
        for name, v in (("size", size), ("segment_size", seg)):
            if not 0 <= v < 2**32:
                raise AggregationError(f"{name} must be a u32")
        show = d.get("show_term_doc_count_error")
        mdc = d.get("min_doc_count")
        return cls(field=d["field"], size=size, segment_size=max(seg, size),
                   show_term_doc_count_error=(target == "_count" and order == "desc") if show is None else bool(show),
                   min_doc_count=1 if mdc is None else int(mdc), order_target=target, order=order, missing=d.get("missing"),
                   include=d.get("include"), exclude=d.get("exclude"))


def parse_request(agg):
    """{"terms": {...}} (one entry of an Aggregations map) -> TermsAggregation.  Sub-aggregations are refused (TermsRefused)."""
    if "aggs" in agg or "aggregations" in agg:
        raise TermsRefused("sub-aggregations run on the CPU path")
    if set(agg) != {"terms"}:
        raise AggregationError("expected exactly one `terms`")
    return TermsAggregation.from_dict(agg["terms"])


def check_device(req: TermsAggregation, kind, multi_valued=False, n_columns=1):
    """Refuses (TermsRefused) every request the device does not run on a field of column kind `kind` ("str", "u64", "i64", "f64",
    "bool", "date"; anything else, e.g. "ip", is refused), each with its own message."""
    if req.order_target not in ("_count", "_key"):
        raise TermsRefused("ordering by a sub-aggregation runs on the CPU path")
    if req.include is not None or req.exclude is not None:
        raise TermsRefused("include / exclude run on the CPU path")
    if req.min_doc_count == 0:
        raise TermsRefused("min_doc_count 0 streams the dictionary: the CPU path")
    if kind not in KINDS:
        raise TermsRefused(f"{kind} columns run on the CPU path")
    if multi_valued:
        raise TermsRefused("multi-valued columns run on the CPU path")
    if n_columns != 1:
        raise TermsRefused("a field of several columns (JSON) runs on the CPU path")
    if isinstance(req.missing, str) and kind != "str":
        raise TermsRefused("a text `missing` on a non-text column runs on the CPU path (TermMissingAgg)")
    if isinstance(req.missing, bool) or (req.missing is not None and not isinstance(req.missing, (str, int, float))):
        raise AggregationError(f"missing {req.missing!r} is not a key")
    if kind == "bool" and req.missing is not None and _missing_image(req.missing, kind) > 1:
        raise TermsRefused("a bool `missing` other than 0 or 1 runs on the CPU path")


def _missing_image(missing, kind):
    """get_missing_val_as_u64_lenient on a numeric column: f64_to_fastfield_u64(missing as f64) (aggregation/mod.rs:394-402)."""
    v = float(missing)
    if kind in ("u64", "bool"):
        return 0 if v != v or v <= 0 else (_U64_MAX if v >= 18446744073709551616.0 else int(v))
    if kind in ("i64", "date"):
        return (as_i64(v) + _HIGH) % (1 << 64)
    bits = int(np.float64(v).view(np.uint64))
    return bits ^ _HIGH if bits < _HIGH else bits ^ _U64_MAX  # f64's monotone image


def terms_spec(req: TermsAggregation, column_id, kind):
    """(column_id, target, order, segment_size, missing_mode, missing_image) for Context.terms_batch."""
    check_device(req, kind)
    target = TQ_TERMS_BY_KEY if req.order_target == "_key" else TQ_TERMS_BY_COUNT
    order = TQ_ORDER_ASC if req.order == "asc" else TQ_ORDER_DESC
    if req.segment_size == 0:
        raise TermsRefused("segment_size 0 keeps no entry: the CPU path")
    if req.missing is None:
        return (column_id, target, order, req.segment_size, TQ_TERMS_MISSING_NONE, 0)
    if kind == "str":
        return (column_id, target, order, req.segment_size, TQ_TERMS_MISSING_AFTER_MAX, 0)
    return (column_id, target, order, req.segment_size, TQ_TERMS_MISSING_IMAGE, _missing_image(req.missing, kind))


# ---- keys ------------------------------------------------------------------------------------------------------------------
def _f64_of_image(v):
    v = int(v)
    bits = v ^ _HIGH if v >= _HIGH else v ^ _U64_MAX
    return float(np.uint64(bits).view(np.float64))


def _normalize_f64(x):
    """NumericalValue::normalize of an f64 (columnar/src/value.rs:52-60) as an intermediate key."""
    if x == x and x not in (float("inf"), float("-inf")) and float(x).is_integer():
        if -9223372036854775808.0 <= x <= 9223372036854775807.0:
            return ("i64", as_i64(x))
        if 0.0 <= x <= 18446744073709551615.0:
            return ("u64", int(x))
    return ("f64", x)


def _missing_key(missing):
    """The intermediate key of a str column's missing entry (extract_missing_value, term_agg/mod.rs:939-956)."""
    if isinstance(missing, str):
        return ("str", missing)
    if isinstance(missing, float):
        return ("f64", missing)
    return ("i64", missing) if missing < 2**63 else ("u64", missing)


def intermediate_key(image, kind, terms=None):
    """The IntermediateKey of a column image: a str ordinal through its segment's dictionary (`terms`), numbers as the reference
    converts them (f64 normalised), a date formatted, a bool as such."""
    image = int(image)
    if kind == "str":
        return ("str", terms[image])
    if kind == "u64":
        return ("u64", image)
    if kind == "i64":
        return ("i64", image - _HIGH)
    if kind == "f64":
        return _normalize_f64(_f64_of_image(image))
    if kind == "date":
        return ("str", format_date(image - _HIGH))
    if kind == "bool":
        return ("bool", image > 0)
    raise ValueError(kind)


def segment_result(req: TermsAggregation, kind, entries, dictionary=None, missing_image=None):
    """One segment's intermediate entries {key: doc_count} from its kept (image, doc_count) pairs: on a str column the missing
    entry (image `missing_image`, the column's max + 1) takes the request's missing key and is inserted first, so that a term of
    the same text replaces it, as the reference's per-segment map does."""
    out = {}
    rest = []
    for image, count in entries:
        if kind == "str" and req.missing is not None and int(image) == missing_image:
            out[_missing_key(req.missing)] = int(count)
        else:
            rest.append((image, count))
    for image, count in rest:
        out[intermediate_key(image, kind, dictionary)] = int(count)
    return out


def merge(results):
    """Sums intermediate results -- each (entries {key: doc_count}, sum_other_doc_count, doc_count_error_upper_bound) -- as
    IntermediateBucketResult::merge_fruits does (intermediate_agg_result.rs:745-758)."""
    entries, other, error = {}, 0, 0
    for e, o, err in results:
        for k, c in e.items():
            entries[k] = entries.get(k, 0) + c
        other += int(o)
        error += int(err)
    return entries, other, error


_RANK = {"str": 0, "i64": 1, "u64": 2, "bool": 2, "f64": 3}  # Key's variant order (derived PartialOrd): Str, I64, U64, F64


def _final_key(k):
    return ("u64", int(k[1])) if k[0] == "bool" else k


def _key_order(k):
    k = _final_key(k)
    return (_RANK[k[0]], k[1])


def ordered_buckets(req: TermsAggregation, counts):
    """The final buckets' keys of {key: doc_count}: min_doc_count, the order (`_count` or `_key`; equal counts by key ascending,
    where the reference leaves them unspecified), the cut to size.  Returns ([(key, doc_count)] kept, doc count of the cut)."""
    buckets = [(k, c) for k, c in counts.items() if c >= req.min_doc_count]
    if req.order_target == "_key":
        buckets.sort(key=lambda b: _key_order(b[0]), reverse=req.order == "desc")
    else:
        buckets.sort(key=lambda b: _key_order(b[0]))
        buckets.sort(key=lambda b: b[1], reverse=req.order == "desc")
    return buckets[:req.size], sum(c for _, c in buckets[req.size:])


def bucket_entry(key, count):
    """One final terms bucket {"key", "doc_count"[, "key_as_string"]} of an intermediate key."""
    e = {"key": _final_key(key)[1], "doc_count": count}
    if key[0] == "bool":
        e["key_as_string"] = "true" if key[1] else "false"
    return e


def finalize(req: TermsAggregation, merged):
    """IntermediateTermBucketResult::into_final_result (intermediate_agg_result.rs:869-961) of merge()'s result: ordered_buckets,
    each as bucket_entry."""
    entries, other, error = merged
    kept, cut = ordered_buckets(req, entries)
    res = {"buckets": [bucket_entry(k, c) for k, c in kept], "sum_other_doc_count": other + cut}
    if req.show_term_doc_count_error:
        res["doc_count_error_upper_bound"] = error
    return res


def cut_segment(entries, req: TermsAggregation, metric=None):
    """One segment's cut to segment_size (into_intermediate_bucket_result + cut_off_buckets, term_agg/mod.rs:1000-1111,
    1328-1353) of {image: doc_count}: (kept [(image, doc_count)] ascending, term_doc_count_before_cutoff, sum_other_doc_count).
    Equal counts at the cut keep the lowest images, as the device does.  An order by a sub-aggregation takes metric = {image: the
    segment's compute_metric_value(...).unwrap_or(0.0)}, compared as partial_cmp does (-0.0 equals +0.0), equal values again by
    image ascending."""
    items = sorted((k, c) for k, c in entries.items() if c)
    if len(items) <= req.segment_size:
        return items, 0, 0
    if req.order_target == "_key":
        order = items if req.order == "asc" else items[::-1]
    elif metric is not None:
        order = sorted(items, key=lambda kc: (metric[kc[0]] if req.order == "asc" else -metric[kc[0]], kc[0]))
    else:
        order = sorted(items, key=lambda kc: (kc[1] if req.order == "asc" else -kc[1], kc[0]))
    return sorted(order[:req.segment_size]), order[req.segment_size][1], sum(c for _, c in order[req.segment_size:])


def finalize_rows(req: TermsAggregation, kind, rows, dictionaries=None, missing_images=None):
    """finalize over Context.terms_batch rows of one query from any number of contexts: rows = [(segment_ord, key, doc_count, n,
    sum_other, error_bound) for row q], dictionaries[segment_ord] = that segment's terms (str), missing_images[segment_ord] = its
    missing image (str: the column's max + 1).  A segment split over contexts by doc range (tq_segment_set_doc_range) comes back
    uncut from each: its entries are summed by image over the contexts and cut here, once per segment as the reference cuts; a
    whole segment comes back cut, and cutting it again changes nothing."""
    per, other, error = {}, 0, 0
    for segs, keys, counts, n, o, e in rows:
        for j in range(int(n)):
            seg = per.setdefault(int(segs[j]), {})
            seg[int(keys[j])] = seg.get(int(keys[j]), 0) + int(counts[j])
        other += int(o)
        error += int(e)
    results = []
    for s, entries in per.items():
        kept, e, o = cut_segment(entries, req)
        results.append((segment_result(req, kind, kept, None if dictionaries is None else dictionaries[s],
                                       None if missing_images is None else missing_images.get(s)), o, e))
    ent, o, e = merge(results)
    return finalize(req, (ent, other + o, error + e))
