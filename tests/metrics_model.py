"""An independent model of the metric aggregations (metric/stats.rs @ v0.26.0), written without the device's guard: per segment,
IntermediateStats::collect over the collected values in doc order -- each doc's f64_from_fastfield_u64(image), a doc without a
value collecting the missing value when there is one, a count-only column collecting 0.0 -- with Kahan summation; then
merge_fruits over the segments in segment_ord order, and into_final_metric_result.  Python floats are IEEE f64, so every step rounds
as the reference's does.  f64::min / f64::max skip NaN; between -0.0 and +0.0 (unspecified in the reference) min takes -0.0 and
max +0.0, the device's image order."""
import math

F64_MAX = 1.7976931348623157e308


def _is_neg_zero(x):
    return x == 0.0 and math.copysign(1.0, x) < 0


def rust_min(a, b):
    if a != a:
        return b
    if b != b:
        return a
    if a == b:
        return a if _is_neg_zero(a) else b
    return a if a < b else b


def rust_max(a, b):
    if a != a:
        return b
    if b != b:
        return a
    if a == b:
        return b if _is_neg_zero(a) else a
    return a if a > b else b


class Stats:
    """IntermediateStats: count, Kahan sum and delta, min, max (stats.rs:88-175)."""

    def __init__(self):
        self.count, self.sum, self.delta, self.min, self.max = 0, 0.0, 0.0, F64_MAX, -F64_MAX

    def collect(self, value):
        self.count += 1
        y = value - self.delta
        t = self.sum + y
        self.delta = (t - self.sum) - y
        self.sum = t
        self.min = rust_min(self.min, value)
        self.max = rust_max(self.max, value)

    def merge_fruits(self, other):
        self.count += other.count
        y = other.sum - (self.delta + other.delta)
        t = self.sum + y
        self.delta = (t - self.sum) - y
        self.sum = t
        self.min = rust_min(self.min, other.min)
        self.max = rust_max(self.max, other.max)


def segment_stats(values):
    st = Stats()
    for v in values:
        st.collect(float(v))
    return st


def merged(segments):
    """merge_fruits of the segments' Stats, given in segment_ord order."""
    out = Stats()
    for st in segments:
        out.merge_fruits(st)
    return out


def final(st, typ, none_if_no_match=False):
    """into_final_metric_result (intermediate_agg_result.rs:425-462) of one aggregation of type typ."""
    n = st.count
    avg = st.sum / n if n else None
    if typ == "stats":
        return {"count": n, "sum": st.sum, "min": st.min if n else None, "max": st.max if n else None, "avg": avg}
    if typ == "sum":
        return {"value": None if n == 0 and none_if_no_match else st.sum}
    if typ == "avg":
        return {"value": avg}
    if typ == "min":
        return {"value": st.min if n else None}
    if typ == "max":
        return {"value": st.max if n else None}
    return {"value": float(n)}  # value_count


# ---- what a doc collects (agg_data.rs:529-573, accessor_helpers.rs:49-74, aggregation/mod.rs:374-402) ----------------------------
NUMERIC = ("u64", "i64", "f64", "date")
COUNT_TYPES = NUMERIC + ("str", "bool", "ip")  # value_count's allowed column types
_I64_MIN, _I64_MAX, _U64_MAX = -2**63, 2**63 - 1, 2**64 - 1


def column_type(typ, kind):
    """The column a metric of type typ reads on a field of type kind: the field's own when its type is allowed, else tantivy's
    empty U64 column ("empty")."""
    return kind if kind in (COUNT_TYPES if typ == "value_count" else NUMERIC) else "empty"


def _saturate(m, lo, hi):
    """Rust's `m as i64` / `m as u64`: NaN to 0, saturating."""
    if m != m:
        return 0
    if m <= lo:
        return lo
    if m >= hi:
        return hi
    return int(m)


def missing_value(m, ctype):
    """f64_from_fastfield_u64(f64_to_fastfield_u64(m, type)): the f64 a doc without a value collects, or None (str, ip)."""
    if ctype in ("u64", "bool"):
        return float(_saturate(m, 0, _U64_MAX))
    if ctype in ("i64", "date"):
        return float(_saturate(m, _I64_MIN, _I64_MAX))
    if ctype == "f64":
        return float(m)
    return None


def doc_values(typ, kind, value, missing=None):
    """The values one collected doc adds: its own (0.0 on a str, bool or ip column), the missing value, or none."""
    ctype = column_type(typ, kind)
    if ctype == "empty":
        ctype, value = "u64", None
    if value is None:
        if missing is None:
            return []
        v = missing_value(float(missing), ctype)
        if v is None:
            return []
    else:
        v = float(value) if ctype in NUMERIC else 0.0
    return [v if ctype in NUMERIC else 0.0]
