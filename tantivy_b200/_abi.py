"""ctypes mirror of include/tantivy_b200.h (structs and constants only; no library is loaded here).

Shared by the product binding (tantivy_b200/lib.py) and by the test-only oracle binding
(oracle/tq_oracle.py) so that one marshalled query batch can be handed to either side.
"""
import ctypes as C

import numpy as np

TQ_OK = 0
TQ_RECORD_BASIC, TQ_RECORD_FREQS, TQ_RECORD_FREQS_POSITIONS = 0, 1, 2
TQ_OP_TERM, TQ_OP_AND, TQ_OP_OR, TQ_OP_PHRASE, TQ_OP_BOOL = 0, 1, 2, 3, 4
TQ_OCCUR_SHOULD, TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT = 0, 1, 2
TERMINATED = 0x7FFFFFFF
TQ_MAX_K = 1024
TQ_MAX_TERMS = 32
TQ_TERM_IGNORE_FREQ = 1
TQ_QUERY_HAS_THRESHOLD = 1
TQ_QUERY_COUNT_HITS = 2
TQ_QUERY_FILTER = 4
TQ_ORDER_DESC, TQ_ORDER_ASC = 0, 1
TQ_FAST_U64, TQ_FAST_I64, TQ_FAST_F64, TQ_FAST_BOOL, TQ_FAST_DATE = 0, 1, 2, 3, 4
TQ_TERMS_BY_COUNT, TQ_TERMS_BY_KEY, TQ_TERMS_BY_METRIC = 0, 1, 2
TQ_TERMS_ORDER_COUNT, TQ_TERMS_ORDER_SUM, TQ_TERMS_ORDER_AVG, TQ_TERMS_ORDER_MIN, TQ_TERMS_ORDER_MAX = 0, 1, 2, 3, 4
TQ_TERMS_MISSING_NONE, TQ_TERMS_MISSING_IMAGE, TQ_TERMS_MISSING_AFTER_MAX = 0, 1, 2
TQ_METRICS_MAX_COLUMNS = 4
TQ_METRIC_MISSING, TQ_METRIC_COUNT_ONLY, TQ_METRIC_EMPTY = 1, 2, 4

u8p = C.POINTER(C.c_uint8)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)
f32p = C.POINTER(C.c_float)


class TermSeg(C.Structure):
    """tq_term_seg — postings::TermInfo of one (clause, segment) (src/postings/term_info.rs:9-16)."""
    _fields_ = [
        ("term_idx", C.c_uint32),
        ("segment_ord", C.c_uint32),
        ("field", C.c_uint32),
        ("doc_freq", C.c_uint32),
        ("postings_start", C.c_uint64),
        ("postings_end", C.c_uint64),
    ]


TERM_SEG_DTYPE = np.dtype(
    [("term_idx", "<u4"), ("segment_ord", "<u4"), ("field", "<u4"), ("doc_freq", "<u4"),
     ("postings_start", "<u8"), ("postings_end", "<u8")]
)
assert TERM_SEG_DTYPE.itemsize == C.sizeof(TermSeg) == 32


class TermPos(C.Structure):
    """tq_term_pos — TermInfo::positions_range of one (clause, segment)."""
    _fields_ = [("positions_start", C.c_uint64), ("positions_end", C.c_uint64)]


TERM_POS_DTYPE = np.dtype([("positions_start", "<u8"), ("positions_end", "<u8")])


class Query(C.Structure):
    """tq_query — one Weight for all segments (src/core/searcher.rs:226)."""
    _fields_ = [
        ("op", C.c_int32),
        ("n_terms", C.c_uint32),
        ("k", C.c_uint32),
        ("n_term_segs", C.c_uint32),
        ("term_segs", C.POINTER(TermSeg)),
        ("weight", f32p),
        ("avg_fieldnorm", f32p),
        ("tf_cache", f32p),
        ("term_flags", u8p),
        ("flags", C.c_uint32),
        ("threshold", C.c_float),
        ("term_pos", C.POINTER(TermPos)),
        ("term_offset", u32p),
        ("slop", C.c_uint32),
        ("min_should_match", C.c_uint32),
        ("term_occur", u8p),
        ("term_group", u8p),
        ("filter_id", C.c_uint32),
    ]


_QUERY_FIELDS = np.dtype(
    [("op", "<i4"), ("n_terms", "<u4"), ("k", "<u4"), ("n_term_segs", "<u4"),
     ("term_segs", "<u8"), ("weight", "<u8"), ("avg_fieldnorm", "<u8"), ("tf_cache", "<u8"), ("term_flags", "<u8"),
     ("flags", "<u4"), ("threshold", "<f4"), ("term_pos", "<u8"), ("term_offset", "<u8"), ("slop", "<u4"), ("min_should_match", "<u4"),
     ("term_occur", "<u8"), ("term_group", "<u8"), ("filter_id", "<u4")]
)
# (the C struct ends in 4 bytes of padding: it is 8-byte aligned)
QUERY_DTYPE = np.dtype({"names": list(_QUERY_FIELDS.names), "formats": [_QUERY_FIELDS.fields[n][0] for n in _QUERY_FIELDS.names],
                        "offsets": [_QUERY_FIELDS.fields[n][1] for n in _QUERY_FIELDS.names], "itemsize": C.sizeof(Query)})
assert QUERY_DTYPE.itemsize == C.sizeof(Query) == 112


class Stats(C.Structure):
    """tq_stats."""
    _fields_ = [
        ("lists_cached", C.c_uint64),
        ("lists_built", C.c_uint64),
        ("units", C.c_uint64),
        ("kernel_launches", C.c_uint64),
        ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64),
        ("algorithmic_bytes", C.c_uint64),
        ("postings", C.c_uint64),
        ("kernel_ms", C.c_float),
        ("total_ms", C.c_float),
        ("term_ms", C.c_float),
        ("and_ms", C.c_float),
        ("or_ms", C.c_float),
        ("final_ms", C.c_float),
        ("units_term", C.c_uint64),
        ("units_and", C.c_uint64),
        ("units_or", C.c_uint64),
        ("bytes_term", C.c_uint64),
        ("bytes_and", C.c_uint64),
        ("bytes_or", C.c_uint64),
        ("or_windows", C.c_uint64 * 8),
        ("units_or_strip", C.c_uint64),
        ("score_ms", C.c_float),
        ("tile_ms", C.c_float),
        ("theta_ms", C.c_float),
        ("phrase_ms", C.c_float),
        ("units_tile", C.c_uint64),
        ("units_phrase", C.c_uint64),
        ("tile_groups", C.c_uint64),
        ("tile_postings", C.c_uint64),
        ("tile_list_bytes", C.c_uint64),
        ("tile_scratch_bytes", C.c_uint64),
        ("tile_fallbacks", C.c_uint64),
        ("tile_counters", C.c_uint64 * 8),
        ("tile_ctas_per_sm", C.c_uint64),
        ("tile_cycles", C.c_uint64 * 8),
        ("tile_groups_union_only", C.c_uint64),
        ("tile_b2_exits", C.c_uint64 * 4),
        ("count_hits_ms", C.c_float),
        ("units_count_hits", C.c_uint64),
        ("sort_ms", C.c_float),
        ("units_sort", C.c_uint64),
        ("sort_tiles_seen", C.c_uint64),
        ("sort_tiles_skipped", C.c_uint64),
    ]


class HistogramStats(C.Structure):
    """tq_histogram_stats — the cumulative counters of tq_histogram_batch (tq_get_histogram_stats)."""
    _fields_ = [("hist_ms", C.c_float), ("units_hist", C.c_uint64), ("hist_tiles_seen", C.c_uint64), ("hist_tiles_one_bucket", C.c_uint64)]


class TermsStats(C.Structure):
    """tq_terms_stats — the cumulative counters of tq_terms_batch (tq_get_terms_stats)."""
    _fields_ = [("terms_ms", C.c_float), ("units_terms", C.c_uint64), ("terms_tiles_seen", C.c_uint64), ("terms_tiles_one_key", C.c_uint64)]


class SortSpec(C.Structure):
    """tq_sort_spec — the column and Order of TopDocs::order_by_fast_field for one query."""
    _fields_ = [("column_id", C.c_uint32), ("order", C.c_uint32)]


SORT_SPEC_DTYPE = np.dtype([("column_id", "<u4"), ("order", "<u4")])
assert SORT_SPEC_DTYPE.itemsize == C.sizeof(SortSpec) == 8


class HistogramSpec(C.Structure):
    """tq_histogram_spec — the column, its kind (TQ_FAST_*), the grid and the collect-time bounds of one query's histogram."""
    _fields_ = [("column_id", C.c_uint32), ("kind", C.c_uint32), ("interval", C.c_double), ("offset", C.c_double),
                ("hard_min", C.c_double), ("hard_max", C.c_double)]


HISTOGRAM_SPEC_DTYPE = np.dtype([("column_id", "<u4"), ("kind", "<u4"), ("interval", "<f8"), ("offset", "<f8"), ("hard_min", "<f8"),
                                 ("hard_max", "<f8")])
assert HISTOGRAM_SPEC_DTYPE.itemsize == C.sizeof(HistogramSpec) == 40


class TermsSpec(C.Structure):
    """tq_terms_spec — the column, order target and direction, segment_size and missing key of one query's terms aggregation."""
    _fields_ = [("column_id", C.c_uint32), ("target", C.c_uint32), ("order", C.c_uint32), ("segment_size", C.c_uint32),
                ("missing_mode", C.c_uint32), ("pad", C.c_uint32), ("missing_image", C.c_uint64)]


TERMS_SPEC_DTYPE = np.dtype([("column_id", "<u4"), ("target", "<u4"), ("order", "<u4"), ("segment_size", "<u4"), ("missing_mode", "<u4"),
                             ("pad", "<u4"), ("missing_image", "<u8")])
assert TERMS_SPEC_DTYPE.itemsize == C.sizeof(TermsSpec) == 32


class MetricsStats(C.Structure):
    """tq_metrics_stats — the cumulative counters of tq_metrics_batch (tq_get_metrics_stats)."""
    _fields_ = [("metrics_ms", C.c_float), ("units_metrics", C.c_uint64), ("metrics_tiles_seen", C.c_uint64), ("metrics_tiles_one_value", C.c_uint64)]


class HistMetricsStats(C.Structure):
    """tq_hist_metrics_stats — the cumulative counters of tq_histogram_metrics_batch (tq_get_hist_metrics_stats)."""
    _fields_ = [("hist_metrics_ms", C.c_float), ("units_hist_metrics", C.c_uint64), ("hist_metrics_tiles_seen", C.c_uint64),
                ("hist_metrics_tiles_one_bucket", C.c_uint64), ("hist_metrics_flush_shared", C.c_uint64), ("hist_metrics_flush_global", C.c_uint64)]


class MetricColumn(C.Structure):
    """tq_metric_column — one column of a metrics spec: its kind, TQ_METRIC_* flags and missing image."""
    _fields_ = [("column_id", C.c_uint32), ("kind", C.c_uint32), ("flags", C.c_uint32), ("pad", C.c_uint32), ("missing_image", C.c_uint64)]


class MetricsSpec(C.Structure):
    """tq_metrics_spec — the 1..TQ_METRICS_MAX_COLUMNS columns one query's metrics read."""
    _fields_ = [("n_columns", C.c_uint32), ("pad", C.c_uint32), ("columns", MetricColumn * TQ_METRICS_MAX_COLUMNS)]


class MetricPart(C.Structure):
    """tq_metric_part — the intermediate result of one (query, column)."""
    _fields_ = [("count", C.c_uint64), ("n_nan", C.c_uint64), ("n_inf", C.c_uint64), ("min_image", C.c_uint64), ("max_image", C.c_uint64),
                ("sum", C.c_double), ("magnitude", C.c_double), ("quantum_exp", C.c_int32), ("pad", C.c_uint32)]


METRIC_COLUMN_DTYPE = np.dtype([("column_id", "<u4"), ("kind", "<u4"), ("flags", "<u4"), ("pad", "<u4"), ("missing_image", "<u8")])
METRICS_SPEC_DTYPE = np.dtype([("n_columns", "<u4"), ("pad", "<u4"), ("columns", METRIC_COLUMN_DTYPE, (TQ_METRICS_MAX_COLUMNS,))])
METRIC_PART_DTYPE = np.dtype([("count", "<u8"), ("n_nan", "<u8"), ("n_inf", "<u8"), ("min_image", "<u8"), ("max_image", "<u8"), ("sum", "<f8"),
                              ("magnitude", "<f8"), ("quantum_exp", "<i4"), ("pad", "<u4")])
assert METRIC_COLUMN_DTYPE.itemsize == C.sizeof(MetricColumn) == 24
assert METRICS_SPEC_DTYPE.itemsize == C.sizeof(MetricsSpec) == 104
assert METRIC_PART_DTYPE.itemsize == C.sizeof(MetricPart) == 64


class TermsMetricsStats(C.Structure):
    """tq_terms_metrics_stats — the cumulative counters of tq_terms_metrics_batch (tq_get_terms_metrics_stats)."""
    _fields_ = [("terms_metrics_ms", C.c_float), ("units_terms_metrics", C.c_uint64), ("terms_metrics_tiles_seen", C.c_uint64),
                ("terms_metrics_tiles_one_key", C.c_uint64), ("terms_metrics_waves", C.c_uint64)]


class TermsMetricOrder(C.Structure):
    """tq_terms_metric_order — the spec column and TQ_TERMS_ORDER_* metric a TQ_TERMS_BY_METRIC query is ordered by."""
    _fields_ = [("column", C.c_uint32), ("metric", C.c_uint32)]


TERMS_METRIC_ORDER_DTYPE = np.dtype([("column", "<u4"), ("metric", "<u4")])
assert TERMS_METRIC_ORDER_DTYPE.itemsize == C.sizeof(TermsMetricOrder) == 8


TQ_RANGE_MAX_BUCKETS = 128


class RangeSpec(C.Structure):
    """tq_range_spec — the column and the strictly ascending bucket starts (images, starts[0] == 0) of one query's range."""
    _fields_ = [("column_id", C.c_uint32), ("n_buckets", C.c_uint32), ("starts", C.c_uint64 * TQ_RANGE_MAX_BUCKETS)]


RANGE_SPEC_DTYPE = np.dtype([("column_id", "<u4"), ("n_buckets", "<u4"), ("starts", "<u8", (TQ_RANGE_MAX_BUCKETS,))])
assert RANGE_SPEC_DTYPE.itemsize == C.sizeof(RangeSpec) == 1032


class RangeStats(C.Structure):
    """tq_range_stats — the cumulative counters of tq_range_batch (tq_get_range_stats)."""
    _fields_ = [("range_ms", C.c_float), ("units_range", C.c_uint64), ("range_tiles_seen", C.c_uint64), ("range_tiles_one_bucket", C.c_uint64)]


class TermsHistStats(C.Structure):
    """tq_terms_hist_stats — the cumulative counters of tq_terms_histogram_batch (tq_get_terms_hist_stats)."""
    _fields_ = [("terms_hist_ms", C.c_float), ("units_terms_hist", C.c_uint64), ("terms_hist_tiles_seen", C.c_uint64),
                ("terms_hist_tiles_one_key", C.c_uint64), ("terms_hist_tiles_one_bucket", C.c_uint64), ("terms_hist_tiles_both", C.c_uint64),
                ("terms_hist_waves", C.c_uint64), ("terms_hist_units_shared", C.c_uint64), ("terms_hist_units_global", C.c_uint64)]


class HistTermsStats(C.Structure):
    """tq_hist_terms_stats — the cumulative counters of tq_histogram_terms_batch (tq_get_hist_terms_stats)."""
    _fields_ = [("hist_terms_ms", C.c_float), ("units_hist_terms", C.c_uint64), ("hist_terms_tiles_seen", C.c_uint64),
                ("hist_terms_tiles_one_key", C.c_uint64), ("hist_terms_tiles_one_bucket", C.c_uint64), ("hist_terms_tiles_both", C.c_uint64),
                ("hist_terms_units_shared", C.c_uint64), ("hist_terms_units_global", C.c_uint64), ("hist_terms_rows_cut", C.c_uint64),
                ("hist_terms_waves", C.c_uint64)]


def ptr(arr, typ):
    """numpy array -> ctypes pointer (array must stay alive while the pointer is used)."""
    if arr is None:
        return typ()
    return arr.ctypes.data_as(typ)


class QueryBatch:
    """A marshalled array of tq_query with everything it points to kept alive.

    `queries` is an iterable of dicts / objects with fields
      op, k, weights[n_terms], avg_fieldnorm[n_terms], term_segs: list of
      (term_idx, segment_ord, field, doc_freq, postings_start, postings_end),
      tf_cache (optional [n_terms,256]), term_flags (optional [n_terms] bytes, TQ_TERM_IGNORE_FREQ),
      threshold (optional float: only docs scoring above it are collected),
      count_hits (optional bool: the batch also counts the query's matching alive docs, Batch.fetch_hits),
      phrase queries (op TQ_OP_PHRASE): term_pos = list of (positions_start, positions_end) parallel to term_segs,
      term_offset = [n_terms] offsets in the phrase, slop (optional, must be 0 on the device path);
      boolean queries (op TQ_OP_BOOL): term_occur = [n_terms] TQ_OCCUR_*, term_group = optional [n_terms] group ids of the MUST
      clauses, min_should_match (optional);
      filter (optional int id of a doc filter registered with Context.filter_register: FilterCollector around the query's
      TopDocs and Count; sets TQ_QUERY_FILTER).
    Built with numpy so that a batch of thousands of queries marshals in milliseconds.
    """

    def __init__(self, queries):
        queries = list(queries)
        self.nq = len(queries)
        n_ts = sum(len(q["term_segs"]) for q in queries)
        n_terms = sum(len(q["weights"]) for q in queries)
        self.term_segs = np.zeros(max(n_ts, 1), dtype=TERM_SEG_DTYPE)
        self.weights = np.zeros(max(n_terms, 1), dtype=np.float32)
        self.avgs = np.zeros(max(n_terms, 1), dtype=np.float32)
        self.caches = []
        self.q = np.zeros(max(self.nq, 1), dtype=QUERY_DTYPE)
        ts_base = self.term_segs.ctypes.data
        w_base = self.weights.ctypes.data
        a_base = self.avgs.ctypes.data
        its, iw = 0, 0
        self.kmax = 1
        for i, q in enumerate(queries):
            nt = len(q["weights"])
            ts = q["term_segs"]
            if len(ts):
                block = np.asarray(ts, dtype=np.uint64).reshape(-1, 6)
                v = self.term_segs[its:its + len(ts)]
                v["term_idx"] = block[:, 0]
                v["segment_ord"] = block[:, 1]
                v["field"] = block[:, 2]
                v["doc_freq"] = block[:, 3]
                v["postings_start"] = block[:, 4]
                v["postings_end"] = block[:, 5]
            self.weights[iw:iw + nt] = q["weights"]
            self.avgs[iw:iw + nt] = q["avg_fieldnorm"]
            row = self.q[i]
            row["op"] = q["op"]
            row["n_terms"] = nt
            row["k"] = q["k"]
            row["n_term_segs"] = len(ts)
            row["term_segs"] = ts_base + its * TERM_SEG_DTYPE.itemsize
            row["weight"] = w_base + iw * 4
            row["avg_fieldnorm"] = a_base + iw * 4
            cache = q.get("tf_cache")
            if cache is not None:
                cache = np.ascontiguousarray(cache, dtype=np.float32).reshape(nt, 256)
                self.caches.append(cache)
                row["tf_cache"] = cache.ctypes.data
            if q.get("threshold") is not None:
                row["flags"] = TQ_QUERY_HAS_THRESHOLD
                row["threshold"] = q["threshold"]
            if q.get("count_hits"):
                row["flags"] |= TQ_QUERY_COUNT_HITS
            filt = q.get("filter")
            if filt is not None:
                if isinstance(filt, (bool, np.bool_)) or not isinstance(filt, (int, np.integer)) or not 0 <= int(filt) < 1 << 32:
                    raise ValueError(f"query {i}: filter must be a filter id in 0 .. 2**32 - 1, got {filt!r}")
                row["flags"] |= TQ_QUERY_FILTER
                row["filter_id"] = int(filt)
            tpos = q.get("term_pos")
            if tpos is not None:
                tp = np.zeros(max(len(tpos), 1), dtype=TERM_POS_DTYPE)
                if len(tpos):
                    blockp = np.asarray(tpos, dtype=np.uint64).reshape(-1, 2)
                    tp["positions_start"][:len(tpos)] = blockp[:, 0]
                    tp["positions_end"][:len(tpos)] = blockp[:, 1]
                toff = np.ascontiguousarray(q["term_offset"], dtype=np.uint32).reshape(nt)
                self.caches += [tp, toff]
                row["term_pos"] = tp.ctypes.data
                row["term_offset"] = toff.ctypes.data
                row["slop"] = int(q.get("slop", 0))
            occ = q.get("term_occur")
            if occ is not None:
                occ = np.ascontiguousarray(occ, dtype=np.uint8).reshape(nt)
                self.caches.append(occ)
                row["term_occur"] = occ.ctypes.data
                grp = q.get("term_group")
                if grp is not None:
                    grp = np.ascontiguousarray(grp, dtype=np.uint8).reshape(nt)
                    self.caches.append(grp)
                    row["term_group"] = grp.ctypes.data
                row["min_should_match"] = int(q.get("min_should_match", 0))
            flags = q.get("term_flags")
            if flags is not None:
                flags = np.ascontiguousarray(flags, dtype=np.uint8).reshape(nt)
                self.caches.append(flags)
                row["term_flags"] = flags.ctypes.data
            self.kmax = max(self.kmax, int(q["k"]))
            its += len(ts)
            iw += nt

    @property
    def ptr(self):
        return C.cast(self.q.ctypes.data, C.POINTER(Query))

    def alloc_out(self, stride=None):
        stride = stride or self.kmax
        n = max(self.nq, 1)
        return (
            stride,
            np.zeros((n, stride), dtype=np.float32),
            np.zeros((n, stride), dtype=np.uint32),
            np.zeros((n, stride), dtype=np.uint32),
            np.zeros(n, dtype=np.uint32),
        )
