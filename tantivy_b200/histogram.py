"""The request and result side of a `histogram` / `date_histogram` aggregation (src/aggregation/bucket/histogram/), for the device's
segment part (Context.histogram_batch).  Pure Python: it parses and validates a request (HistogramAggregation,
DateHistogramAggregationReq), turns it into the device's spec (date requests are in milliseconds, a date column in nanoseconds),
and finalises the intermediate rows of any number of shards or contexts -- summed by bucket -- into tantivy's result:
{"buckets": [{"key", "doc_count", "key_as_string"?}]} or, keyed, {"buckets": {key: {...}}}.

Only a top-level histogram without sub-aggregations on a single-valued fast field runs on the device."""
import datetime as _dt
import math
from dataclasses import dataclass
from typing import Optional

import numpy as np

F64_MAX = float(np.finfo(np.float64).max)
DEFAULT_BUCKET_LIMIT = 65000  # aggregation/collector.rs
_I64_MAX, _I64_MIN = 2**63 - 1, -2**63


class AggregationError(ValueError):
    """A request tantivy refuses (TantivyError::InvalidArgument, AggregationError), or a result over the bucket limit."""


def as_i64(f):
    """Rust's `f as i64`: toward zero, saturating, NaN -> 0."""
    f = float(f)
    if f != f:
        return 0
    if f >= 9223372036854775808.0:
        return _I64_MAX
    if f < -9223372036854775808.0:
        return _I64_MIN
    return int(f)


def bucket_pos(val, interval, offset):
    """get_bucket_pos_f64(val, interval, offset) as i64 (histogram.rs:739-741)."""
    return as_i64(np.floor((np.float64(val) - np.float64(offset)) / np.float64(interval)))


def bucket_key(pos, interval, offset):
    """get_bucket_key_from_pos: pos as f64 * interval + offset, two roundings (no fused multiply-add)."""
    return float(np.float64(pos) * np.float64(interval)) + offset


# ---- date_histogram parsing (date_histogram.rs:190-244) -----------------------------------------------------------------------
_UNIT_MS = {"ms": 1, "milliseconds": 1, "s": 1000, "seconds": 1000, "m": 60_000, "minutes": 60_000, "h": 3_600_000, "hours": 3_600_000,
            "d": 86_400_000, "days": 86_400_000}


def parse_into_milliseconds(text):
    """'30s', '1m', '2hours', ... -> milliseconds; only ASCII digits count as digits.  Raises AggregationError for a missing number
    or unit, an unknown unit, and a value whose nanoseconds overflow i64."""
    raw = text.encode("utf-8")
    split = 0
    while split < len(raw) and 0x30 <= raw[split] <= 0x39:
        split += 1
    number, unit = raw[:split], raw[split:]
    if not number:
        raise AggregationError(f"Number not found in passed String {text!r}")
    if not unit:
        raise AggregationError(f"Unit not found in passed String {text!r}")
    n = int(number)
    if n > _I64_MAX:
        raise AggregationError(f"Number not found in passed String {text!r}")
    unit_ms = _UNIT_MS.get(unit.decode("utf-8", errors="replace"))
    if unit_ms is None:
        raise AggregationError(f"Unit not recognized in passed String {unit.decode('utf-8', errors='replace')!r}")
    val = n * unit_ms
    if not (_I64_MIN <= val * 1_000_000 <= _I64_MAX):
        raise AggregationError(f"passed value is out of bounds: {text!r}")
    return val


def parse_offset_into_milliseconds(text):
    """Like parse_into_milliseconds, with an optional leading '+' or '-'."""
    if not text:
        raise AggregationError(f"passed offset is invalid {text!r}")
    if text[0] in "+-":
        val = parse_into_milliseconds(text[1:])
        return -val if text[0] == "-" else val
    return parse_into_milliseconds(text)


# ---- requests ----------------------------------------------------------------------------------------------------------------
def _bounds(b):
    if b is None:
        return None
    lo, hi = (b["min"], b["max"]) if isinstance(b, dict) else b
    return (_date_or_num(lo), _date_or_num(hi))


def _date_or_num(v):
    """deserialize_date_or_num: a number, or an RFC 3339 date string as its milliseconds."""
    if isinstance(v, str):
        d = _dt.datetime.fromisoformat(v.replace("Z", "+00:00"))
        if d.tzinfo is None:
            raise AggregationError("Invalid Rfc3339 formatted date")
        delta = d - _dt.datetime(1970, 1, 1, tzinfo=_dt.timezone.utc)
        return float((delta.days * 86_400_000_000 + delta.seconds * 1_000_000 + delta.microseconds) // 1000)
    return float(v)


@dataclass
class HistogramAggregation:
    """HistogramAggregation (histogram.rs): interval, offset and bounds in the field's unit (ms for a date field)."""
    field: str
    interval: float
    offset: Optional[float] = None
    min_doc_count: Optional[int] = None
    hard_bounds: Optional[tuple] = None
    extended_bounds: Optional[tuple] = None
    keyed: bool = False
    is_normalized_to_ns: bool = False

    @classmethod
    def from_dict(cls, d):
        known = {"field", "interval", "offset", "min_doc_count", "hard_bounds", "extended_bounds", "keyed", "is_normalized_to_ns"}
        unknown = set(d) - known
        if unknown:
            raise AggregationError(f"unknown histogram parameter(s) {sorted(unknown)}")
        return cls(field=d["field"], interval=float(d["interval"]), offset=None if d.get("offset") is None else float(d["offset"]),
                   min_doc_count=d.get("min_doc_count"), hard_bounds=_bounds(d.get("hard_bounds")),
                   extended_bounds=_bounds(d.get("extended_bounds")), keyed=bool(d.get("keyed", False)),
                   is_normalized_to_ns=bool(d.get("is_normalized_to_ns", False)))

    def validate(self):
        if self.interval <= 0.0:
            raise AggregationError("interval must be a positive value")
        if (self.min_doc_count or 0) > 0 and self.extended_bounds is not None:
            raise AggregationError("Cannot set min_doc_count and extended_bounds at the same time")
        if self.hard_bounds is not None and self.extended_bounds is not None:
            (hlo, hhi), (elo, ehi) = self.hard_bounds, self.extended_bounds
            if elo < hlo or ehi > hhi:
                raise AggregationError(f"extended_bounds have to be inside hard_bounds, extended_bounds: [{elo},{ehi}], hard_bounds [{hlo},{hhi}]")

    def normalized(self):
        """normalize_date_time: the request in nanoseconds (interval, offset, both bounds times 1e6)."""
        if self.is_normalized_to_ns:
            return self
        scale = lambda b: None if b is None else (b[0] * 1_000_000.0, b[1] * 1_000_000.0)  # noqa: E731
        return HistogramAggregation(self.field, self.interval * 1_000_000.0, None if self.offset is None else self.offset * 1_000_000.0,
                                    self.min_doc_count, scale(self.hard_bounds), scale(self.extended_bounds), self.keyed, True)


@dataclass
class DateHistogramAggregationReq:
    """DateHistogramAggregationReq (date_histogram.rs): only `fixed_interval`; `interval`, `calendar_interval` and `format` are
    refused."""
    field: str
    fixed_interval: Optional[str] = None
    offset: Optional[str] = None
    min_doc_count: Optional[int] = None
    hard_bounds: Optional[tuple] = None
    extended_bounds: Optional[tuple] = None
    keyed: bool = False
    interval: Optional[str] = None
    calendar_interval: Optional[str] = None
    format: Optional[str] = None

    @classmethod
    def from_dict(cls, d):
        known = {"field", "fixed_interval", "offset", "min_doc_count", "hard_bounds", "extended_bounds", "keyed", "interval",
                 "calendar_interval", "format"}
        unknown = set(d) - known
        if unknown:
            raise AggregationError(f"unknown date_histogram parameter(s) {sorted(unknown)}")
        return cls(field=d["field"], fixed_interval=d.get("fixed_interval"), offset=d.get("offset"), min_doc_count=d.get("min_doc_count"),
                   hard_bounds=_bounds(d.get("hard_bounds")), extended_bounds=_bounds(d.get("extended_bounds")),
                   keyed=bool(d.get("keyed", False)), interval=d.get("interval"), calendar_interval=d.get("calendar_interval"),
                   format=d.get("format"))

    def validate(self):
        if self.interval is not None:
            raise AggregationError(f"`interval` parameter {self.interval!r} in date histogram is unsupported, only `fixed_interval` is supported")
        if self.calendar_interval is not None:
            raise AggregationError(f"`calendar_interval` parameter {self.calendar_interval!r} in date histogram is unsupported, only "
                                   "`fixed_interval` is supported")
        if self.format is not None:
            raise AggregationError("format parameter on date_histogram is unsupported")
        if self.fixed_interval is None:
            raise AggregationError("fixed_interval in date histogram is missing")
        parse_into_milliseconds(self.fixed_interval)

    def to_histogram_req(self):
        self.validate()
        return HistogramAggregation(self.field, float(parse_into_milliseconds(self.fixed_interval)),
                                    None if self.offset is None else float(parse_offset_into_milliseconds(self.offset)),
                                    self.min_doc_count, self.hard_bounds, self.extended_bounds, self.keyed, False)


def parse_request(agg):
    """{"histogram": {...}} or {"date_histogram": {...}} (one entry of an Aggregations map) -> (HistogramAggregation, is_date_histogram).
    A request with sub-aggregations is refused: it is not a device aggregation."""
    if "aggs" in agg or "aggregations" in agg:
        raise AggregationError("sub-aggregations are not supported by the device histogram")
    kinds = [k for k in ("histogram", "date_histogram") if k in agg]
    if len(kinds) != 1 or len(agg) != 1:
        raise AggregationError("expected exactly one `histogram` or `date_histogram`")
    if kinds[0] == "histogram":
        return HistogramAggregation.from_dict(agg["histogram"]), False
    return DateHistogramAggregationReq.from_dict(agg["date_histogram"]).to_histogram_req(), True


def device_request(req: HistogramAggregation, kind):
    """The request as the device collects it (normalize_histogram_req): validated, and in nanoseconds on a date column."""
    req.validate()
    return req.normalized() if kind == "date" else req


def histogram_spec(req: HistogramAggregation, column_id, kind):
    """(column_id, kind, interval, offset, hard_min, hard_max) for Context.histogram_batch."""
    r = device_request(req, kind)
    lo, hi = r.hard_bounds if r.hard_bounds is not None else (-F64_MAX, F64_MAX)
    return (column_id, kind, r.interval, r.offset or 0.0, lo, hi)


# ---- finalisation (histogram.rs:776-931) -----------------------------------------------------------------------------------
def merge_intermediate(rows):
    """Sum intermediate results -- each an iterable of (pos, doc_count), e.g. zip(pos[q, :n[q]], doc_count[q, :n[q]]) -- by bucket:
    the merge of IntermediateBucketResult::Histogram across segments, shards and contexts.  Returns {pos: doc_count}."""
    out = {}
    for row in rows:
        for pos, count in row:
            if count:
                out[int(pos)] = out.get(int(pos), 0) + int(count)
    return out


def format_date(ns):
    """format_date (aggregation/date.rs): RFC 3339 in UTC of i64 nanoseconds, fraction digits only as needed."""
    secs, frac = divmod(int(ns), 1_000_000_000)
    d = _dt.datetime(1970, 1, 1) + _dt.timedelta(seconds=secs)
    if not (0 <= d.year <= 9999):
        raise AggregationError(f"Could not convert {ns} to OffsetDateTime")
    s = d.strftime("%Y-%m-%dT%H:%M:%S")
    if frac:
        s += "." + f"{frac:09d}".rstrip("0")
    return s + "Z"


def rust_f64_display(v):
    """f64's Display in Rust (the key of a keyed bucket): shortest round trip, never an exponent, no trailing '.0'."""
    if v != v:
        return "NaN"
    if math.isinf(v):
        return "inf" if v > 0 else "-inf"
    return np.format_float_positional(v, trim="-")


def final_buckets(req: HistogramAggregation, intermediate, kind, bucket_limit=DEFAULT_BUCKET_LIMIT):
    """The buckets of intermediate_histogram_buckets_to_final_buckets, in key order: (key on the device's grid, doc_count, pos) for
    each bucket of {pos: doc_count} that is kept, and (key, 0, None) for each bucket the gap filling or extended_bounds add."""
    r = device_request(req, kind)
    offset = r.offset or 0.0
    buckets = sorted(((bucket_key(p, r.interval, offset), c, p) for p, c in intermediate.items() if c), key=lambda b: _total_order(b[0]))
    min_doc_count = r.min_doc_count or 0
    if min_doc_count == 0:
        lo, hi = (buckets[0][0], buckets[-1][0]) if buckets else (F64_MAX, -F64_MAX)
        if r.extended_bounds is not None:
            lo, hi = min(lo, r.extended_bounds[0]), max(hi, r.extended_bounds[1])
        if r.hard_bounds is not None:
            lo, hi = max(lo, r.hard_bounds[0]), min(hi, r.hard_bounds[1])
        first, last = bucket_pos(lo, r.interval, offset), bucket_pos(hi, r.interval, offset)
        if last - first + 1 > bucket_limit:
            raise AggregationError(f"Aborting aggregation because bucket limit was exceeded. Limit: {bucket_limit}, Current: {last - first + 1}")
        fill = [bucket_key(p, r.interval, offset) for p in range(first, last + 1)]
        out, i, j = [], 0, 0
        while i < len(buckets) or j < len(fill):  # merge_join_by on the keys (partial_cmp, NaN as equal)
            if j == len(fill) or (i < len(buckets) and buckets[i][0] < fill[j]):
                out.append(buckets[i]); i += 1  # noqa: E702
            elif i == len(buckets) or fill[j] < buckets[i][0]:
                out.append((fill[j], 0, None)); j += 1  # noqa: E702
            else:
                out.append(buckets[i]); i += 1; j += 1  # noqa: E702
        buckets = out
    else:
        buckets = [b for b in buckets if b[1] >= min_doc_count]
    if len(buckets) > bucket_limit:
        raise AggregationError(f"Aborting aggregation because bucket limit was exceeded. Limit: {bucket_limit}, Current: {len(buckets)}")
    return buckets


def bucket_entry(key, count, kind):
    """One final bucket {"key", "doc_count"[, "key_as_string"]}: a date key in milliseconds with its RFC 3339 string."""
    e = {"key": key, "doc_count": count}
    if kind == "date":
        e["key_as_string"] = format_date(as_i64(key))
        e["key"] = key / 1_000_000.0
    return e


def keyed_or_list(req: HistogramAggregation, entries):
    return {"buckets": {rust_f64_display(e["key"]): e for e in entries}} if req.keyed else {"buckets": entries}


def finalize(req: HistogramAggregation, intermediate, kind, bucket_limit=DEFAULT_BUCKET_LIMIT):
    """intermediate_histogram_buckets_to_final_buckets: {pos: doc_count} (merge_intermediate; pos on the device's grid, i.e. of
    device_request(req, kind)) -> tantivy's histogram result.  is_date_agg is kind == "date"."""
    return keyed_or_list(req, [bucket_entry(key, count, kind) for key, count, _ in final_buckets(req, intermediate, kind, bucket_limit)])


def _total_order(x):
    """f64::total_cmp as a sort key."""
    b = int(np.float64(x).view(np.int64))
    return b ^ 0x7FFFFFFFFFFFFFFF if b < 0 else b
