"""ctypes binding of the product library tantivy_b200/_lib/libtantivy_b200.so (the C ABI of
include/tantivy_b200.h).  The library is CUDA-only: if it is missing, importing fails loudly;
if no GPU is present, tq_ctx_create fails loudly.  Nothing here falls back to a CPU path."""
import ctypes as C
import os

import numpy as np

from ._abi import (HISTOGRAM_SPEC_DTYPE, METRIC_PART_DTYPE, METRICS_SPEC_DTYPE, SORT_SPEC_DTYPE, TERMS_SPEC_DTYPE, TQ_METRICS_MAX_COLUMNS, MetricPart,
                   MetricsSpec, MetricsStats, HistMetricsStats, TermsMetricsStats, TermsMetricOrder, TERMS_METRIC_ORDER_DTYPE, TQ_FAST_BOOL, TQ_FAST_DATE, TQ_FAST_F64, TQ_FAST_I64, TQ_FAST_U64,
                   TQ_ORDER_ASC, TQ_ORDER_DESC, HistogramSpec, HistogramStats, Query, QueryBatch, SortSpec, Stats, TermSeg, TermsSpec, TermsStats,
                   RANGE_SPEC_DTYPE, RangeSpec, RangeStats, TermsHistStats, HistTermsStats, TQ_RANGE_MAX_BUCKETS, f32p, ptr, u8p, u32p, u64p)

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("TANTIVY_B200_LIB") or os.path.join(_HERE, "_lib", "libtantivy_b200.so")  # (override: A/B builds)


class TqError(RuntimeError):
    pass


def _load():
    if not os.path.exists(SO_PATH):
        raise ImportError(
            f"{SO_PATH} is missing: build it with `make -C tantivy_b200/csrc` (or __graft_entry__.build()). "
            "There is no CPU fallback for the query path.")
    lib = C.CDLL(SO_PATH)
    vp, sz = C.c_void_p, C.c_size_t
    lib.tq_last_error.restype = C.c_char_p
    lib.tq_last_error.argtypes = [vp]
    lib.tq_ctx_create.argtypes = [C.c_int, C.POINTER(vp)]
    lib.tq_ctx_destroy.argtypes = [vp]
    lib.tq_get_stats.argtypes = [vp, C.POINTER(Stats)]
    lib.tq_get_histogram_stats.argtypes = [vp, C.POINTER(HistogramStats)]
    lib.tq_get_terms_stats.argtypes = [vp, C.POINTER(TermsStats)]
    lib.tq_get_metrics_stats.argtypes = [vp, C.POINTER(MetricsStats)]
    lib.tq_get_hist_metrics_stats.argtypes = [vp, C.POINTER(HistMetricsStats)]
    lib.tq_get_terms_metrics_stats.argtypes = [vp, C.POINTER(TermsMetricsStats)]
    lib.tq_get_range_stats.argtypes = [vp, C.POINTER(RangeStats)]
    lib.tq_get_terms_hist_stats.argtypes = [vp, C.POINTER(TermsHistStats)]
    lib.tq_get_hist_terms_stats.argtypes = [vp, C.POINTER(HistTermsStats)]
    lib.tq_segment_register.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, u8p, sz, u8p, sz, u8p, sz]
    lib.tq_segment_register_positions.argtypes = [vp, C.c_uint32, C.c_uint32, u8p, sz]
    lib.tq_segment_unregister.argtypes = [vp, C.c_uint32, C.c_uint32]
    lib.tq_segment_set_doc_range.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    lib.tq_filter_register.argtypes = [vp, C.c_uint32, C.c_uint32, u8p, sz]
    lib.tq_filter_unregister.argtypes = [vp, C.c_uint32]
    lib.tq_multi_filter_register.argtypes = [vp, C.c_uint32, C.c_uint32, u8p, sz]
    lib.tq_multi_filter_unregister.argtypes = [vp, C.c_uint32]
    lib.tq_search_batch.argtypes = [vp, C.POINTER(Query), sz, C.c_uint32, f32p, u32p, u32p, u32p]
    lib.tq_batch_prepare.argtypes = [vp, C.POINTER(Query), sz, C.POINTER(vp)]
    lib.tq_count_batch.argtypes = [vp, C.POINTER(Query), sz, u64p]
    lib.tq_sort_column_register.argtypes = [vp, C.c_uint32, C.c_uint32, u64p, sz, u8p, sz]
    lib.tq_sort_column_unregister.argtypes = [vp, C.c_uint32]
    lib.tq_sort_batch.argtypes = [vp, C.POINTER(Query), C.POINTER(SortSpec), sz, C.c_uint32, u64p, u8p, u32p, u32p, u32p, u64p]
    lib.tq_histogram_batch.argtypes = [vp, C.POINTER(Query), C.POINTER(HistogramSpec), sz, C.c_uint32, C.POINTER(C.c_int64), u64p, u32p, u64p]
    lib.tq_terms_batch.argtypes = [vp, C.POINTER(Query), C.POINTER(TermsSpec), sz, C.c_uint32, u32p, u64p, u64p, u32p, u64p, u64p, u64p]
    lib.tq_metrics_batch.argtypes = [vp, C.POINTER(Query), C.POINTER(MetricsSpec), sz, C.POINTER(MetricPart), u64p]
    lib.tq_histogram_metrics_batch.argtypes = [vp, C.POINTER(Query), C.POINTER(HistogramSpec), C.POINTER(MetricsSpec), sz, C.c_uint32,
                                               C.POINTER(C.c_int64), u64p, C.POINTER(MetricPart), u32p, u64p]
    lib.tq_terms_metrics_batch.argtypes = [vp, C.POINTER(Query), C.POINTER(TermsSpec), C.POINTER(MetricsSpec), C.POINTER(TermsMetricOrder), sz,
                                           C.c_uint32, u32p, u64p, u64p, C.POINTER(MetricPart), u32p, u64p, u64p, C.POINTER(MetricPart), u64p]
    lib.tq_range_batch.argtypes = [vp, C.POINTER(Query), C.POINTER(RangeSpec), C.POINTER(MetricsSpec), sz, C.c_uint32, u64p, C.POINTER(MetricPart),
                                   u64p]
    lib.tq_terms_histogram_batch.argtypes = [vp, C.POINTER(Query), C.POINTER(TermsSpec), C.POINTER(HistogramSpec), sz, C.c_uint32, u32p, u64p,
                                             u64p, u32p, u64p, u64p, C.c_uint64, u64p, u32p, C.POINTER(C.c_int64), u64p, u32p, u64p]
    lib.tq_histogram_terms_batch.argtypes = [vp, C.POINTER(Query), C.POINTER(HistogramSpec), C.POINTER(TermsSpec), sz, C.c_uint32,
                                             C.POINTER(C.c_int64), u64p, u64p, u64p, u64p, u32p, u32p, C.c_uint64, u32p, u64p, u64p, u32p, u64p]
    lib.tq_batch_run.argtypes = [vp]
    lib.tq_batch_run_phase.argtypes = [vp, C.c_int]
    lib.tq_batch_phases.argtypes = [vp]
    lib.tq_batch_thresholds_export_dev.argtypes = [vp, vp]
    lib.tq_batch_thresholds_import_dev.argtypes = [vp, vp]
    lib.tq_batch_stream.argtypes = [vp, C.POINTER(vp)]
    lib.tq_batch_topkeys_export_dev.argtypes = [vp, vp, C.c_uint32]
    lib.tq_batch_thresholds_from_keys_dev.argtypes = [vp, vp, C.c_uint32, C.c_uint32]
    lib.tq_batch_fetch.argtypes = [vp, C.c_uint32, f32p, u32p, u32p, u32p]
    lib.tq_batch_fetch_hits.argtypes = [vp, u64p]
    lib.tq_batch_results_dev.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(C.c_uint32)]
    lib.tq_batch_results_copy_dev.argtypes = [vp, vp, vp, vp, vp]
    lib.tq_batch_destroy.argtypes = [vp]
    lib.tq_merge_topk_dev.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.tq_batch_results_pack_dev.argtypes = [vp, vp]
    lib.tq_batch_results_pack_dev_async.argtypes = [vp, vp]
    lib.tq_merge_topk_packed_dev.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp, sz, vp]
    lib.tq_multi_create.argtypes = [C.POINTER(C.c_int), C.c_int, C.POINTER(vp)]
    lib.tq_multi_destroy.argtypes = [vp]
    lib.tq_multi_last_error.restype = C.c_char_p
    lib.tq_multi_last_error.argtypes = [vp]
    lib.tq_multi_num_devices.argtypes = [vp]
    lib.tq_multi_segment_register.argtypes = [vp, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, u8p, sz, u8p, sz, u8p, sz]
    lib.tq_multi_segment_register_split.argtypes = [vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, u8p, sz, u8p, sz, u8p, sz]
    lib.tq_multi_search_batch.argtypes = [vp, C.POINTER(Query), sz, C.c_uint32, f32p, u32p, u32p, u32p]
    lib.tq_decode_postings.argtypes = [vp, C.POINTER(TermSeg), u32p, u32p]
    lib.tq_block_table.argtypes = [vp, C.POINTER(TermSeg), C.c_float, C.c_float, u32p, f32p]
    lib.tq_bm25_idf.restype = C.c_float
    lib.tq_bm25_idf.argtypes = [C.c_uint64, C.c_uint64]
    lib.tq_bm25_weight.restype = C.c_float
    lib.tq_bm25_weight.argtypes = [C.c_uint64, C.c_uint64, C.c_float]
    lib.tq_bm25_tf_cache.argtypes = [C.c_float, f32p]
    lib.tq_id_to_fieldnorm.restype = C.c_uint32
    lib.tq_id_to_fieldnorm.argtypes = [C.c_uint8]
    lib.tq_fieldnorm_to_id.restype = C.c_uint8
    lib.tq_fieldnorm_to_id.argtypes = [C.c_uint32]
    lib.tq_field_writer_create.argtypes = [C.c_int, C.c_uint64, u8p, C.c_uint32, C.POINTER(vp)]
    lib.tq_field_writer_add_term.argtypes = [vp, u32p, u32p, C.c_uint32, u64p, u64p]
    lib.tq_field_writer_body.argtypes = [vp, C.POINTER(u8p), C.POINTER(sz)]
    lib.tq_field_writer_destroy.argtypes = [vp]
    # synthetic segment generator (csrc/synth.cpp)
    lib.tqs_generate.restype = vp
    lib.tqs_generate.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(C.c_double), C.c_uint32, C.c_uint64, C.c_int, C.c_int, C.c_uint32, C.c_uint32]
    lib.tqs_destroy.argtypes = [vp]
    lib.tqs_num_segments.restype = C.c_uint32
    lib.tqs_num_segments.argtypes = [vp]
    lib.tqs_max_doc.restype = C.c_uint32
    lib.tqs_max_doc.argtypes = [vp, C.c_uint32]
    lib.tqs_total_num_tokens.restype = C.c_uint64
    lib.tqs_total_num_tokens.argtypes = [vp, C.c_uint32]
    lib.tqs_body.argtypes = [vp, C.c_uint32, C.POINTER(u8p), C.POINTER(sz)]
    lib.tqs_fieldnorm.argtypes = [vp, C.c_uint32, C.POINTER(u8p), C.POINTER(sz)]
    lib.tqs_term_info.argtypes = [vp, C.c_uint32, C.c_uint32, u32p, u64p, u64p]
    lib.tqs_positions.argtypes = [vp, C.c_uint32, C.POINTER(u8p), C.POINTER(sz)]
    lib.tqs_term_pos.argtypes = [vp, C.c_uint32, C.c_uint32, u64p, u64p]
    return lib


LIB = _load()


def _check(rc, ctx=None):
    if rc != 0:
        raise TqError(f"tantivy_b200 error {rc}: {LIB.tq_last_error(ctx).decode(errors='replace')}")


_HIGHEST_BIT = np.uint64(1 << 63)
FAST_VALUE_KINDS = ("u64", "i64", "f64", "bool", "date")
_FAST_KIND = {"u64": TQ_FAST_U64, "i64": TQ_FAST_I64, "f64": TQ_FAST_F64, "bool": TQ_FAST_BOOL, "date": TQ_FAST_DATE}


def _histogram_specs(specs, nq):
    """HISTOGRAM_SPEC_DTYPE rows of (column_id, kind, interval, offset[, hard_min, hard_max]) tuples."""
    spec = np.zeros(max(nq, 1), dtype=HISTOGRAM_SPEC_DTYPE)
    for i, sp in enumerate(specs):
        col, kind, interval, offset = sp[:4]
        hard_min, hard_max = sp[4:6] if len(sp) > 4 else (-np.finfo(np.float64).max, np.finfo(np.float64).max)
        spec[i] = (col, _FAST_KIND.get(kind, kind), interval, offset, hard_min, hard_max)
    return spec


def _terms_specs(specs, nq):
    """TERMS_SPEC_DTYPE rows of (column_id, target, order, segment_size[, missing_mode, missing_image]) tuples."""
    spec = np.zeros(max(nq, 1), dtype=TERMS_SPEC_DTYPE)
    for i, sp in enumerate(specs):
        col, target, order, segment_size = sp[:4]
        mode, image = sp[4:6] if len(sp) > 4 else (0, 0)
        spec[i] = (col, target, order, segment_size, mode, 0, image)
    return spec


def _metrics_specs(specs, nq):
    """METRICS_SPEC_DTYPE rows of lists of (column_id, kind[, flags, missing_image]) columns."""
    spec = np.zeros(max(nq, 1), dtype=METRICS_SPEC_DTYPE)
    for i, cols in enumerate(specs):
        cols = list(cols)
        spec[i]["n_columns"] = len(cols)
        for j, col in enumerate(cols[:TQ_METRICS_MAX_COLUMNS]):
            flags, image = (tuple(col[2:4]) + (0, 0))[:2]
            spec[i]["columns"][j] = (col[0], col[1], flags, 0, image)
    return spec

def _range_specs(specs, nq):
    """RANGE_SPEC_DTYPE rows of (column_id, starts) tuples: starts the bucket starts in image space, ascending from 0."""
    spec = np.zeros(max(nq, 1), dtype=RANGE_SPEC_DTYPE)
    for i, (col, starts) in enumerate(specs):
        starts = [int(x) for x in starts]
        if len(starts) > TQ_RANGE_MAX_BUCKETS:
            raise ValueError(f"query {i}: a range has at most {TQ_RANGE_MAX_BUCKETS} buckets, got {len(starts)}")
        spec[i]["column_id"] = col
        spec[i]["n_buckets"] = len(starts)
        spec[i]["starts"][:len(starts)] = np.array(starts, dtype=np.uint64)
    return spec


def fast_value_to_u64(values, kind):
    """The u64 image of fast-field values (MonotonicallyMappableToU64, common/src/lib.rs), what tq_sort_column_register takes:
    u64 as is; i64 v ^ 2^63; f64 bits ^ 2^63 when the sign bit is clear (+0.0 included), !bits when it is set (-0.0 included);
    bool 0 / 1; date (numpy datetime64, or int64 nanoseconds since the epoch) as its i64 nanoseconds.  Order-preserving."""
    if kind == "u64":
        return np.asarray(values, dtype=np.uint64).copy()
    if kind == "i64":
        return np.asarray(values, dtype=np.int64).view(np.uint64) ^ _HIGHEST_BIT
    if kind == "date":
        v = np.asarray(values)
        if np.issubdtype(v.dtype, np.datetime64):
            v = v.astype("datetime64[ns]").view(np.int64)
        return np.asarray(v, dtype=np.int64).view(np.uint64) ^ _HIGHEST_BIT
    if kind == "f64":
        bits = np.asarray(values, dtype=np.float64).view(np.uint64)
        neg = (bits & _HIGHEST_BIT) != 0
        return np.where(neg, ~bits, bits ^ _HIGHEST_BIT)
    if kind == "bool":
        return np.asarray(values, dtype=bool).astype(np.uint64)
    raise ValueError(f"kind must be one of {FAST_VALUE_KINDS}, got {kind!r}")


def u64_to_fast_value(images, kind):
    """The reverse of fast_value_to_u64 (MonotonicallyMappableToU64::from_u64): date gives datetime64[ns]."""
    u = np.asarray(images, dtype=np.uint64)
    if kind == "u64":
        return u.copy()
    if kind in ("i64", "date"):
        v = (u ^ _HIGHEST_BIT).view(np.int64)
        return v.view("datetime64[ns]") if kind == "date" else v
    if kind == "f64":
        return np.where((u & _HIGHEST_BIT) != 0, u ^ _HIGHEST_BIT, ~u).view(np.float64)
    if kind == "bool":
        return u > 0
    raise ValueError(f"kind must be one of {FAST_VALUE_KINDS}, got {kind!r}")


def bm25_idf(doc_freq, doc_count):
    return LIB.tq_bm25_idf(doc_freq, doc_count)


def bm25_weight(doc_freq, doc_count, boost=1.0):
    return LIB.tq_bm25_weight(doc_freq, doc_count, boost)


def bm25_tf_cache(avg):
    out = np.zeros(256, dtype=np.float32)
    LIB.tq_bm25_tf_cache(avg, ptr(out, f32p))
    return out


def id_to_fieldnorm(i):
    return LIB.tq_id_to_fieldnorm(i)


def fieldnorm_to_id(f):
    return LIB.tq_fieldnorm_to_id(f)


class FieldWriter:
    """Host-side PostingsSerializer equivalent (src/postings/serializer.rs:353-481)."""

    def __init__(self, record_option, total_num_tokens, fieldnorm_ids, max_doc):
        self._fn = None if fieldnorm_ids is None else np.ascontiguousarray(fieldnorm_ids, dtype=np.uint8)
        h = C.c_void_p()
        _check(LIB.tq_field_writer_create(record_option, int(total_num_tokens), ptr(self._fn, u8p), max_doc, C.byref(h)))
        self.h = h

    def add_term(self, docs, tfs=None):
        docs = np.ascontiguousarray(docs, dtype=np.uint32)
        tfs = None if tfs is None else np.ascontiguousarray(tfs, dtype=np.uint32)
        s, e = C.c_uint64(), C.c_uint64()
        _check(LIB.tq_field_writer_add_term(self.h, ptr(docs, u32p), ptr(tfs, u32p), len(docs), C.byref(s), C.byref(e)))
        return int(s.value), int(e.value)

    def body(self):
        p, n = u8p(), C.c_size_t()
        _check(LIB.tq_field_writer_body(self.h, C.byref(p), C.byref(n)))
        return np.ctypeslib.as_array(p, shape=(n.value,)).copy()

    def __del__(self):
        if getattr(self, "h", None):
            LIB.tq_field_writer_destroy(self.h)
            self.h = None


class SynthIndex:
    """Deterministic synthetic segments in tantivy format (csrc/synth.cpp, SURVEY.md §8d)."""

    def __init__(self, n_segments, docs_per_segment, densities, seed=0x7A6E7469, record_option=1, n_threads=0, segment_base=0,
                 segment_stride=1):
        dens = np.ascontiguousarray(densities, dtype=np.float64)
        self.densities = dens
        self.n_threads = n_threads or (os.cpu_count() or 1)
        self.h = LIB.tqs_generate(n_segments, docs_per_segment, dens.ctypes.data_as(C.POINTER(C.c_double)), len(dens), seed,
                                  record_option, self.n_threads, segment_base, segment_stride)
        self.n_segments = n_segments
        self.record_option = record_option
        self.max_doc = [LIB.tqs_max_doc(self.h, s) for s in range(n_segments)]
        self.total_num_tokens = [LIB.tqs_total_num_tokens(self.h, s) for s in range(n_segments)]
        # term_info[s][t] = (doc_freq, start, end); term_pos[s][t] = (positions_start, positions_end) with record_option 2
        self.term_info, self.term_pos = [], []
        df, st, en = C.c_uint32(), C.c_uint64(), C.c_uint64()
        for s in range(n_segments):
            row, prow = [], []
            for t in range(len(dens)):
                LIB.tqs_term_info(self.h, s, t, C.byref(df), C.byref(st), C.byref(en))
                row.append((df.value, st.value, en.value))
                if record_option == 2:
                    LIB.tqs_term_pos(self.h, s, t, C.byref(st), C.byref(en))
                    prow.append((st.value, en.value))
            self.term_info.append(row)
            self.term_pos.append(prow)

    def body(self, s):
        p, n = u8p(), C.c_size_t()
        LIB.tqs_body(self.h, s, C.byref(p), C.byref(n))
        return np.ctypeslib.as_array(p, shape=(n.value,))

    def fieldnorm(self, s):
        p, n = u8p(), C.c_size_t()
        LIB.tqs_fieldnorm(self.h, s, C.byref(p), C.byref(n))
        return np.ctypeslib.as_array(p, shape=(n.value,))

    def positions(self, s):
        """The segment's `.pos` body (record_option 2)."""
        p, n = u8p(), C.c_size_t()
        LIB.tqs_positions(self.h, s, C.byref(p), C.byref(n))
        return np.ctypeslib.as_array(p, shape=(max(n.value, 1),))[:n.value]

    def num_docs(self):
        return sum(self.max_doc)

    def avg_fieldnorm(self):
        return np.float32(np.float32(sum(self.total_num_tokens)) / np.float32(self.num_docs()))

    def doc_freq(self, t):
        return sum(self.term_info[s][t][0] for s in range(self.n_segments))

    def register(self, target, field=0, segment_base=0):
        """target: Context (GPU) or an oracle index with the same segment_register signature."""
        for s in range(self.n_segments):
            target.segment_register(segment_base + s, field, self.max_doc[s], self.record_option, self.body(s), self.fieldnorm(s), None)
            if self.record_option == 2:
                target.register_positions(segment_base + s, field, self.positions(s))

    def phrase_query(self, terms, k, field=0, segment_base=0, segments=None):
        """PhraseQuery over `terms` (in phrase order): ONE Bm25Weight::for_terms weight (the idfs add up, bm25.rs:95-129)."""
        n_docs = self.num_docs()
        avg = self.avg_fieldnorm()
        idf_sum = np.float32(0)
        for t in terms:
            idf_sum = np.float32(idf_sum + np.float32(bm25_idf(self.doc_freq(t), n_docs)))
        weight = np.float32(idf_sum * np.float32(2.2))
        term_segs, term_pos = [], []
        for clause, t in enumerate(terms):
            for s in (range(self.n_segments) if segments is None else segments):
                df, st, en = self.term_info[s][t]
                if df:
                    term_segs.append((clause, segment_base + s, field, df, st, en))
                    term_pos.append(self.term_pos[s][t])
        return dict(op=3, k=k, weights=[weight] * len(terms), avg_fieldnorm=[avg] * len(terms), term_segs=term_segs, term_pos=term_pos,
                    term_offset=list(range(len(terms))))

    def query(self, op, terms, k, field=0, segment_base=0, boost=1.0, segments=None):
        n_docs = self.num_docs()
        avg = self.avg_fieldnorm()
        weights, term_segs = [], []
        for clause, t in enumerate(terms):
            weights.append(bm25_weight(self.doc_freq(t), n_docs, boost))
            for s in (range(self.n_segments) if segments is None else segments):
                df, st, en = self.term_info[s][t]
                if df:
                    term_segs.append((clause, segment_base + s, field, df, st, en))
        return dict(op=op, k=k, weights=weights, avg_fieldnorm=[avg] * len(terms), term_segs=term_segs)

    def __del__(self):
        if getattr(self, "h", None):
            LIB.tqs_destroy(self.h)
            self.h = None


class Context:
    """tq_ctx: one CUDA device holding registered segments and the per-term block-table cache."""

    def __init__(self, device=0):
        h = C.c_void_p()
        _check(LIB.tq_ctx_create(device, C.byref(h)))
        self.h = h
        self.device = device
        self._hist_metrics_stride = 0  # the widest row hist_metrics_batch has returned (its next first try)
        self._terms_metrics_stride = 0  # the widest row terms_metrics_batch has returned (its next first try)
        self._terms_hist_sizes = (0, 0)  # the widest row and the most cells terms_hist_batch has returned (its next first try)
        self._hist_terms_sizes = (0, 0)  # the widest row and the most entries hist_terms_batch has returned (its next first try)

    def segment_register(self, segment_ord, field, max_doc, record_option, idx_body, fieldnorm=None, alive=None):
        idx_body = np.ascontiguousarray(idx_body, dtype=np.uint8)
        fn = None if fieldnorm is None else np.ascontiguousarray(fieldnorm, dtype=np.uint8)
        al = None if alive is None else np.ascontiguousarray(alive, dtype=np.uint8)
        _check(LIB.tq_segment_register(self.h, segment_ord, field, max_doc, record_option, ptr(idx_body, u8p), idx_body.size,
                                       ptr(fn, u8p), 0 if fn is None else fn.size, ptr(al, u8p), 0 if al is None else al.size), self.h)

    def register_positions(self, segment_ord, field, pos_bytes):
        """The field's `.pos` sub-file of a registered segment (phrase queries)."""
        p = np.ascontiguousarray(pos_bytes, dtype=np.uint8)
        _check(LIB.tq_segment_register_positions(self.h, segment_ord, field, ptr(p, u8p), p.size), self.h)

    def segment_unregister(self, segment_ord, field):
        _check(LIB.tq_segment_unregister(self.h, segment_ord, field), self.h)

    def segment_set_doc_range(self, segment_ord, field, doc_lo, doc_hi):
        """This context evaluates only the docs [doc_lo, doc_hi) of the segment (intra-segment split over GPUs)."""
        _check(LIB.tq_segment_set_doc_range(self.h, segment_ord, field, doc_lo, doc_hi), self.h)

    def filter_register(self, filter_id, segment_ord, bits):
        """The doc filter `filter_id` of one segment (every field registered under the ordinal): `bits` in the `.del` layout,
        bit d & 7 of byte d >> 3 set = keep doc d (np.packbits(mask, bitorder="little")).  Queries with filter=filter_id collect
        only the alive docs it keeps (FilterCollector)."""
        b = np.ascontiguousarray(bits, dtype=np.uint8)
        _check(LIB.tq_filter_register(self.h, filter_id, segment_ord, ptr(b, u8p), b.size), self.h)

    def filter_unregister(self, filter_id):
        _check(LIB.tq_filter_unregister(self.h, filter_id), self.h)

    def sort_column_register(self, column_id, segment_ord, values, present=None):
        """The sort column `column_id` of one segment (every field registered under the ordinal): `values` = the u64 images of
        each doc's first value (max_doc of them, fast_value_to_u64), `present` = bits in the `.del` layout, set = the doc has a
        value (np.packbits(mask, bitorder="little"); None: every doc has one)."""
        v = np.ascontiguousarray(values, dtype=np.uint64)
        p = None if present is None else np.ascontiguousarray(present, dtype=np.uint8)
        _check(LIB.tq_sort_column_register(self.h, column_id, segment_ord, ptr(v, u64p), v.size, ptr(p, u8p), 0 if p is None else p.size), self.h)

    def sort_column_unregister(self, column_id):
        _check(LIB.tq_sort_column_unregister(self.h, column_id), self.h)

    def sort_batch(self, qb: QueryBatch, specs, count_hits=False):
        """TopDocs::with_limit(k).order_by_fast_field(column, order) per query (tq_sort_batch); specs = one (column_id, order) per
        query, order TQ_ORDER_DESC / TQ_ORDER_ASC or "desc" / "asc".  Returns (values, present, segs, docs, counts) -- rows of the
        batch's largest k, values as u64 images (u64_to_fast_value maps them back), present as bool -- and with count_hits=True the
        Count of every query as well."""
        specs = list(specs)
        if len(specs) != qb.nq:
            raise ValueError(f"one sort spec per query: {len(specs)} for {qb.nq} queries")
        spec = np.zeros(max(qb.nq, 1), dtype=SORT_SPEC_DTYPE)
        for i, (col, order) in enumerate(specs):
            spec[i]["column_id"] = col
            spec[i]["order"] = {"desc": TQ_ORDER_DESC, "asc": TQ_ORDER_ASC}.get(order, order)
        n, stride = max(qb.nq, 1), qb.kmax
        values = np.zeros((n, stride), dtype=np.uint64)
        present = np.zeros((n, stride), dtype=np.uint8)
        segs = np.zeros((n, stride), dtype=np.uint32)
        docs = np.zeros((n, stride), dtype=np.uint32)
        counts = np.zeros(n, dtype=np.uint32)
        hits = np.zeros(n, dtype=np.uint64) if count_hits else None
        _check(LIB.tq_sort_batch(self.h, qb.ptr, spec.ctypes.data_as(C.POINTER(SortSpec)), qb.nq, stride, ptr(values, u64p), ptr(present, u8p),
                                 ptr(segs, u32p), ptr(docs, u32p), ptr(counts, u32p), ptr(hits, u64p)), self.h)
        out = (values, present.astype(bool), segs, docs, counts)
        return out + (hits[:qb.nq],) if count_hits else out

    def histogram_batch(self, qb: QueryBatch, specs, count_hits=False, stride=4096):
        """The segment part of a histogram aggregation per query (tq_histogram_batch) over sort columns; specs = one
        (column_id, kind, interval, offset[, hard_min, hard_max]) per query, kind "u64" / "i64" / "f64" / "bool" / "date" or a
        TQ_FAST_* value, interval, offset and bounds in the column's unit (date: nanoseconds; tantivy_b200.histogram turns requests
        into specs).  Returns (pos, doc_count, n): row q holds the n[q] non-empty buckets of query q in ascending pos, over all its
        segments -- and with count_hits=True the Count of every query as well.  Raises TqError with code -4 (TQ_ERR_UNSUPPORTED)
        when a query's bucket range is too wide for the device.  `stride` is the row width tried first: a longer row runs the
        batch again at its width."""
        specs = list(specs)
        if len(specs) != qb.nq:
            raise ValueError(f"one histogram spec per query: {len(specs)} for {qb.nq} queries")
        spec = _histogram_specs(specs, qb.nq)
        n = max(qb.nq, 1)
        while True:
            pos = np.empty((n, stride), dtype=np.int64)  # (only the first n[q] entries of row q are written)
            counts = np.empty((n, stride), dtype=np.uint64)
            nb = np.zeros(n, dtype=np.uint32)
            hits = np.zeros(n, dtype=np.uint64) if count_hits else None
            rc = LIB.tq_histogram_batch(self.h, qb.ptr, spec.ctypes.data_as(C.POINTER(HistogramSpec)), qb.nq, stride,
                                        pos.ctypes.data_as(C.POINTER(C.c_int64)), ptr(counts, u64p), ptr(nb, u32p), ptr(hits, u64p))
            if rc == -1 and int(nb.max()) > stride:  # TQ_ERR_INVALID_ARGUMENT with the row lengths: a wider row
                stride = int(nb.max())
                continue
            _check(rc, self.h)
            out = (pos, counts, nb)
            return out + (hits[:qb.nq],) if count_hits else out

    def terms_batch(self, qb: QueryBatch, specs, count_hits=False, stride=1024):
        """The segment part of a terms aggregation per query (tq_terms_batch) over sort columns; specs = one
        (column_id, target, order, segment_size[, missing_mode, missing_image]) per query, target TQ_TERMS_BY_*, order TQ_ORDER_*,
        missing_mode TQ_TERMS_MISSING_* (tantivy_b200.terms turns requests into specs).  Returns (segment_ord, key, doc_count, n,
        sum_other, error_bound): row q holds the n[q] kept entries of query q, ascending by (segment_ord, key image), over all its
        segments, and sum_other[q] / error_bound[q] the sums of sum_other_doc_count / term_doc_count_before_cutoff over them -- and
        with count_hits=True the Count of every query as well.  Raises TqError with code -4 (TQ_ERR_UNSUPPORTED) when a
        (query, segment)'s keys span too wide a range for the device.  `stride` is the row width tried first: a longer row runs the
        batch again at its width."""
        specs = list(specs)
        if len(specs) != qb.nq:
            raise ValueError(f"one terms spec per query: {len(specs)} for {qb.nq} queries")
        spec = _terms_specs(specs, qb.nq)
        n = max(qb.nq, 1)
        while True:
            segs = np.empty((n, stride), dtype=np.uint32)  # (only the first n[q] entries of row q are written)
            keys = np.empty((n, stride), dtype=np.uint64)
            counts = np.empty((n, stride), dtype=np.uint64)
            nb = np.zeros(n, dtype=np.uint32)
            other = np.zeros(n, dtype=np.uint64)
            error = np.zeros(n, dtype=np.uint64)
            hits = np.zeros(n, dtype=np.uint64) if count_hits else None
            rc = LIB.tq_terms_batch(self.h, qb.ptr, spec.ctypes.data_as(C.POINTER(TermsSpec)), qb.nq, stride, ptr(segs, u32p), ptr(keys, u64p),
                                    ptr(counts, u64p), ptr(nb, u32p), ptr(other, u64p), ptr(error, u64p), ptr(hits, u64p))
            if rc == -1 and int(nb.max()) > stride:  # TQ_ERR_INVALID_ARGUMENT with the row lengths: a wider row
                stride = int(nb.max())
                continue
            _check(rc, self.h)
            out = (segs, keys, counts, nb, other[:qb.nq], error[:qb.nq])
            return out + (hits[:qb.nq],) if count_hits else out

    def metrics_batch(self, qb: QueryBatch, specs, count_hits=False):
        """The intermediate metric results per query (tq_metrics_batch) over sort columns; specs = one list per query of 1..4
        (column_id, kind[, flags, missing_image]) columns, kind TQ_FAST_*, flags TQ_METRIC_* (tantivy_b200.metrics turns requests into
        specs).  Returns a structured array [nq, TQ_METRICS_MAX_COLUMNS] of METRIC_PART_DTYPE (count, n_nan, n_inf, min_image,
        max_image, sum, magnitude, quantum_exp), columns past a query's spec empty -- and with count_hits=True the Count of every query
        as well."""
        specs = list(specs)
        if len(specs) != qb.nq:
            raise ValueError(f"one metrics spec per query: {len(specs)} for {qb.nq} queries")
        spec = _metrics_specs(specs, qb.nq)
        parts = np.zeros((max(qb.nq, 1), TQ_METRICS_MAX_COLUMNS), dtype=METRIC_PART_DTYPE)
        hits = np.zeros(max(qb.nq, 1), dtype=np.uint64) if count_hits else None
        _check(LIB.tq_metrics_batch(self.h, qb.ptr, spec.ctypes.data_as(C.POINTER(MetricsSpec)), qb.nq, parts.ctypes.data_as(C.POINTER(MetricPart)),
                                    ptr(hits, u64p)), self.h)
        return (parts[:qb.nq], hits[:qb.nq]) if count_hits else parts[:qb.nq]

    def hist_metrics_batch(self, qb: QueryBatch, hspecs, mspecs, count_hits=False, stride=None):
        """A histogram with metric sub-aggregations per query (tq_histogram_metrics_batch) over sort columns; hspecs = one histogram
        spec per query as histogram_batch takes them, mspecs = one list of 1..4 metric columns per query as metrics_batch takes them
        (tantivy_b200.hist_metrics turns requests into both).  Returns (pos, doc_count, parts, n): row q holds the n[q] non-empty
        buckets of query q in ascending pos over all its segments, parts[q, j] the [TQ_METRICS_MAX_COLUMNS] METRIC_PART_DTYPE parts
        of bucket j (columns past the query's spec empty) -- and with count_hits=True the Count of every query as well.  Raises
        TqError with code -4 (TQ_ERR_UNSUPPORTED) when a query's bucket range is too wide for the device.  `stride` is the row width
        tried first (default: the widest row this context has returned, at least 256): a longer row runs the batch again at its
        width, so a context serving the same dashboard shapes runs each batch once."""
        hspecs, mspecs = list(hspecs), list(mspecs)
        if stride is None:
            stride = max(256, self._hist_metrics_stride)
        if len(hspecs) != qb.nq or len(mspecs) != qb.nq:
            raise ValueError(f"one histogram and one metrics spec per query: {len(hspecs)} and {len(mspecs)} for {qb.nq} queries")
        hspec, mspec = _histogram_specs(hspecs, qb.nq), _metrics_specs(mspecs, qb.nq)
        n = max(qb.nq, 1)
        while True:
            pos = np.empty((n, stride), dtype=np.int64)  # (only the first n[q] entries of row q are written)
            counts = np.empty((n, stride), dtype=np.uint64)
            parts = np.empty((n, stride, TQ_METRICS_MAX_COLUMNS), dtype=METRIC_PART_DTYPE)
            nb = np.zeros(n, dtype=np.uint32)
            hits = np.zeros(n, dtype=np.uint64) if count_hits else None
            rc = LIB.tq_histogram_metrics_batch(self.h, qb.ptr, hspec.ctypes.data_as(C.POINTER(HistogramSpec)),
                                                mspec.ctypes.data_as(C.POINTER(MetricsSpec)), qb.nq, stride,
                                                pos.ctypes.data_as(C.POINTER(C.c_int64)), ptr(counts, u64p),
                                                parts.ctypes.data_as(C.POINTER(MetricPart)), ptr(nb, u32p), ptr(hits, u64p))
            if rc == -1 and int(nb.max()) > stride:  # TQ_ERR_INVALID_ARGUMENT with the row lengths: a wider row
                stride = int(nb.max())
                continue
            _check(rc, self.h)
            self._hist_metrics_stride = max(self._hist_metrics_stride, int(nb[:qb.nq].max(initial=0)))
            out = (pos[:qb.nq], counts[:qb.nq], parts[:qb.nq], nb[:qb.nq])
            return out + (hits[:qb.nq],) if count_hits else out

    def range_batch(self, qb: QueryBatch, rspecs, mspecs=None, count_hits=False):
        """A range aggregation per query (tq_range_batch) over sort columns, with or without metric sub-aggregations; rspecs = one
        (column_id, starts) per query, starts the query's 1..TQ_RANGE_MAX_BUCKETS bucket starts in image space, strictly ascending
        from 0 (tantivy_b200.ranges turns requests into them); mspecs = None, or one list of 1..4 metric columns per query as
        metrics_batch takes them.  Returns (doc_count, parts) -- and with count_hits=True the Count of every query as well: row q
        holds every bucket of query q in start order, doc_count[q, b] over all its segments and parts[q, b] its
        [TQ_METRICS_MAX_COLUMNS] METRIC_PART_DTYPE parts (None without mspecs).  Rows are max(n_buckets) wide; entries past a
        query's own buckets are zero."""
        rspecs = list(rspecs)
        if len(rspecs) != qb.nq or (mspecs is not None and len(list(mspecs)) != qb.nq):
            raise ValueError(f"one range spec (and metrics spec, if any) per query for {qb.nq} queries")
        rspec = _range_specs(rspecs, qb.nq)
        mspec = _metrics_specs(list(mspecs), qb.nq) if mspecs is not None else None
        stride = int(rspec["n_buckets"][:qb.nq].max(initial=1))
        n = max(qb.nq, 1)
        counts = np.zeros((n, stride), dtype=np.uint64)
        parts = np.zeros((n, stride, TQ_METRICS_MAX_COLUMNS), dtype=METRIC_PART_DTYPE) if mspec is not None else None
        hits = np.zeros(n, dtype=np.uint64) if count_hits else None
        _check(LIB.tq_range_batch(self.h, qb.ptr, rspec.ctypes.data_as(C.POINTER(RangeSpec)),
                                  mspec.ctypes.data_as(C.POINTER(MetricsSpec)) if mspec is not None else None, qb.nq, stride,
                                  ptr(counts, u64p), parts.ctypes.data_as(C.POINTER(MetricPart)) if parts is not None else None,
                                  ptr(hits, u64p)), self.h)
        out = (counts[:qb.nq], parts[:qb.nq] if parts is not None else None)
        return out + (hits[:qb.nq],) if count_hits else out

    def terms_metrics_batch(self, qb: QueryBatch, tspecs, mspecs, orders=None, count_hits=False, stride=None):
        """A terms aggregation with metric sub-aggregations per query (tq_terms_metrics_batch) over sort columns; tspecs = one terms
        spec per query as terms_batch takes them (target also TQ_TERMS_BY_METRIC), mspecs = one list of 1..4 metric columns per query
        as metrics_batch takes them, orders = one (spec column, TQ_TERMS_ORDER_*) or None per query, read for TQ_TERMS_BY_METRIC
        (tantivy_b200.terms_metrics turns requests into all three).  Returns (segment_ord, key, doc_count, parts, n, sum_other,
        error_bound, order_part): row q holds the n[q] kept entries of query q ascending by (segment_ord, key image) as terms_batch
        returns them, parts[q, j] the [TQ_METRICS_MAX_COLUMNS] METRIC_PART_DTYPE parts of entry j, and order_part[q] the ordering
        column's part over every doc the query's terms collect (empty for the _count / _key orders) -- and with count_hits=True the
        Count of every query as well.  Raises TqError with code -4 (TQ_ERR_UNSUPPORTED) when a (query, segment) is too wide for the
        device.  `stride` is the row width tried first (default: the widest row this context has returned, at least 1024): a longer
        row runs the batch again at its width, so a context serving the same table shapes runs each batch once."""
        tspecs, mspecs = list(tspecs), list(mspecs)
        orders = [None] * qb.nq if orders is None else list(orders)
        if stride is None:
            stride = max(1024, self._terms_metrics_stride)
        if len(tspecs) != qb.nq or len(mspecs) != qb.nq or len(orders) != qb.nq:
            raise ValueError(f"one terms spec, metrics spec and order per query: {len(tspecs)}, {len(mspecs)} and {len(orders)} for {qb.nq} queries")
        tspec, mspec = _terms_specs(tspecs, qb.nq), _metrics_specs(mspecs, qb.nq)
        order = np.zeros(max(qb.nq, 1), dtype=TERMS_METRIC_ORDER_DTYPE)
        for i, o in enumerate(orders):
            if o is not None:
                order[i] = tuple(o)
        order_ptr = order.ctypes.data_as(C.POINTER(TermsMetricOrder)) if any(o is not None for o in orders) else None  # (NULL: no order)
        n = max(qb.nq, 1)
        while True:
            segs = np.empty((n, stride), dtype=np.uint32)  # (only the first n[q] entries of row q are written)
            keys = np.empty((n, stride), dtype=np.uint64)
            counts = np.empty((n, stride), dtype=np.uint64)
            parts = np.empty((n, stride, TQ_METRICS_MAX_COLUMNS), dtype=METRIC_PART_DTYPE)
            nb = np.zeros(n, dtype=np.uint32)
            other = np.zeros(n, dtype=np.uint64)
            error = np.zeros(n, dtype=np.uint64)
            opart = np.zeros(n, dtype=METRIC_PART_DTYPE)
            hits = np.zeros(n, dtype=np.uint64) if count_hits else None
            rc = LIB.tq_terms_metrics_batch(self.h, qb.ptr, tspec.ctypes.data_as(C.POINTER(TermsSpec)), mspec.ctypes.data_as(C.POINTER(MetricsSpec)),
                                            order_ptr, qb.nq, stride, ptr(segs, u32p), ptr(keys, u64p),
                                            ptr(counts, u64p), parts.ctypes.data_as(C.POINTER(MetricPart)), ptr(nb, u32p), ptr(other, u64p),
                                            ptr(error, u64p), opart.ctypes.data_as(C.POINTER(MetricPart)), ptr(hits, u64p))
            if rc == -1 and int(nb.max()) > stride:  # TQ_ERR_INVALID_ARGUMENT with the row lengths: a wider row
                stride = int(nb.max())
                continue
            _check(rc, self.h)
            self._terms_metrics_stride = max(self._terms_metrics_stride, int(nb[:qb.nq].max(initial=0)))
            out = (segs[:qb.nq], keys[:qb.nq], counts[:qb.nq], parts[:qb.nq], nb[:qb.nq], other[:qb.nq], error[:qb.nq], opart[:qb.nq])
            return out + (hits[:qb.nq],) if count_hits else out

    def terms_hist_batch(self, qb: QueryBatch, tspecs, hspecs, count_hits=False, stride=None, cell_capacity=None):
        """A terms aggregation whose only sub-aggregation is a histogram, per query (tq_terms_histogram_batch) over sort columns;
        tspecs = one terms spec per query as terms_batch takes them, hspecs = one histogram spec per query as histogram_batch takes
        them (tantivy_b200.terms_hist turns requests into both).  Returns (segment_ord, key, doc_count, n, sum_other, error_bound,
        cell_first, cell_n, cell_pos, cell_count, n_cells): row q holds the n[q] kept entries of query q as terms_batch returns them,
        and entry j's non-empty buckets are cells cell_first[q, j] .. + cell_n[q, j] of the one cell array (pos, doc_count),
        ascending pos; n_cells[q] counts query q's cells -- and with count_hits=True the Count of every query as well.  Raises TqError
        with code -4 (TQ_ERR_UNSUPPORTED) when a (query, segment) is too wide for the device.  `stride` / `cell_capacity` are the
        sizes tried first (default: the widest row and the most cells this context has returned, at least 1024 / 65536): larger
        results run the batch again at their sizes."""
        tspecs, hspecs = list(tspecs), list(hspecs)
        if len(tspecs) != qb.nq or len(hspecs) != qb.nq:
            raise ValueError(f"one terms and one histogram spec per query: {len(tspecs)} and {len(hspecs)} for {qb.nq} queries")
        if stride is None:
            stride = max(1024, self._terms_hist_sizes[0])
        if cell_capacity is None:
            cell_capacity = max(65536, self._terms_hist_sizes[1])
        tspec, hspec = _terms_specs(tspecs, qb.nq), _histogram_specs(hspecs, qb.nq)
        n = max(qb.nq, 1)
        while True:
            segs = np.empty((n, stride), dtype=np.uint32)  # (only the first n[q] entries of row q, and sum(n_cells) cells, are written)
            keys = np.empty((n, stride), dtype=np.uint64)
            counts = np.empty((n, stride), dtype=np.uint64)
            first = np.empty((n, stride), dtype=np.uint64)
            ncell = np.empty((n, stride), dtype=np.uint32)
            pos = np.empty(cell_capacity, dtype=np.int64)
            ccount = np.empty(cell_capacity, dtype=np.uint64)
            nb = np.zeros(n, dtype=np.uint32)
            nc = np.zeros(n, dtype=np.uint32)
            other = np.zeros(n, dtype=np.uint64)
            error = np.zeros(n, dtype=np.uint64)
            hits = np.zeros(n, dtype=np.uint64) if count_hits else None
            rc = LIB.tq_terms_histogram_batch(self.h, qb.ptr, tspec.ctypes.data_as(C.POINTER(TermsSpec)), hspec.ctypes.data_as(C.POINTER(HistogramSpec)),
                                              qb.nq, stride, ptr(segs, u32p), ptr(keys, u64p), ptr(counts, u64p), ptr(nb, u32p), ptr(other, u64p),
                                              ptr(error, u64p), cell_capacity, ptr(first, u64p), ptr(ncell, u32p),
                                              pos.ctypes.data_as(C.POINTER(C.c_int64)), ptr(ccount, u64p), ptr(nc, u32p), ptr(hits, u64p))
            total = int(nc.sum(dtype=np.uint64))
            if rc == -1 and (int(nb.max()) > stride or total > cell_capacity):  # TQ_ERR_INVALID_ARGUMENT with the lengths: larger sizes
                stride, cell_capacity = max(stride, int(nb.max())), max(cell_capacity, total)
                continue
            _check(rc, self.h)
            self._terms_hist_sizes = (max(self._terms_hist_sizes[0], int(nb[:qb.nq].max(initial=0))), max(self._terms_hist_sizes[1], total))
            out = (segs[:qb.nq], keys[:qb.nq], counts[:qb.nq], nb[:qb.nq], other[:qb.nq], error[:qb.nq], first[:qb.nq], ncell[:qb.nq],
                   pos[:total], ccount[:total], nc[:qb.nq])
            return out + (hits[:qb.nq],) if count_hits else out

    def hist_terms_batch(self, qb: QueryBatch, hspecs, tspecs, count_hits=False, stride=None, entry_capacity=None):
        """A histogram whose only sub-aggregation is a terms, per query (tq_histogram_terms_batch) over sort columns; hspecs = one
        histogram spec per query as histogram_batch takes them, tspecs = one terms spec per query as terms_batch takes them
        (tantivy_b200.hist_terms turns requests into both).  Returns (pos, doc_count, sum_other, error_bound, entry_first, entry_n,
        n, entry_segment_ord, entry_key, entry_count, n_entries): row q holds the n[q] non-empty buckets of query q in ascending pos,
        and bucket j's kept entries are entries entry_first[q, j] .. + entry_n[q, j] of the one entry array (segment_ord, image,
        doc_count), by (segment_ord, image); n_entries[q] counts query q's entries -- and with count_hits=True the Count of every
        query as well.  Raises TqError with code -4 (TQ_ERR_UNSUPPORTED) when a (query, segment) is too wide for the device.
        `stride` / `entry_capacity` are the sizes tried first (default: the widest row and the most entries this context has
        returned, at least 1024 / 65536): larger results run the batch again at their sizes."""
        hspecs, tspecs = list(hspecs), list(tspecs)
        if len(tspecs) != qb.nq or len(hspecs) != qb.nq:
            raise ValueError(f"one histogram and one terms spec per query: {len(hspecs)} and {len(tspecs)} for {qb.nq} queries")
        if stride is None:
            stride = max(1024, self._hist_terms_sizes[0])
        if entry_capacity is None:
            entry_capacity = max(65536, self._hist_terms_sizes[1])
        hspec, tspec = _histogram_specs(hspecs, qb.nq), _terms_specs(tspecs, qb.nq)
        n = max(qb.nq, 1)
        while True:
            pos = np.empty((n, stride), dtype=np.int64)  # (only the first n[q] buckets of row q, and sum(n_entries) entries, are written)
            docs = np.empty((n, stride), dtype=np.uint64)
            other = np.empty((n, stride), dtype=np.uint64)
            error = np.empty((n, stride), dtype=np.uint64)
            first = np.empty((n, stride), dtype=np.uint64)
            nent = np.empty((n, stride), dtype=np.uint32)
            eseg = np.empty(entry_capacity, dtype=np.uint32)
            ekey = np.empty(entry_capacity, dtype=np.uint64)
            ecount = np.empty(entry_capacity, dtype=np.uint64)
            nb = np.zeros(n, dtype=np.uint32)
            ne = np.zeros(n, dtype=np.uint32)
            hits = np.zeros(n, dtype=np.uint64) if count_hits else None
            rc = LIB.tq_histogram_terms_batch(self.h, qb.ptr, hspec.ctypes.data_as(C.POINTER(HistogramSpec)), tspec.ctypes.data_as(C.POINTER(TermsSpec)),
                                              qb.nq, stride, pos.ctypes.data_as(C.POINTER(C.c_int64)), ptr(docs, u64p), ptr(other, u64p),
                                              ptr(error, u64p), ptr(first, u64p), ptr(nent, u32p), ptr(nb, u32p), entry_capacity, ptr(eseg, u32p),
                                              ptr(ekey, u64p), ptr(ecount, u64p), ptr(ne, u32p), ptr(hits, u64p))
            total = int(ne.sum(dtype=np.uint64))
            if rc == -1 and (int(nb.max()) > stride or total > entry_capacity):  # TQ_ERR_INVALID_ARGUMENT with the lengths: larger sizes
                stride, entry_capacity = max(stride, int(nb.max())), max(entry_capacity, total)
                continue
            _check(rc, self.h)
            self._hist_terms_sizes = (max(self._hist_terms_sizes[0], int(nb[:qb.nq].max(initial=0))), max(self._hist_terms_sizes[1], total))
            out = (pos[:qb.nq], docs[:qb.nq], other[:qb.nq], error[:qb.nq], first[:qb.nq], nent[:qb.nq], nb[:qb.nq], eseg[:total],
                   ekey[:total], ecount[:total], ne[:qb.nq])
            return out + (hits[:qb.nq],) if count_hits else out

    def search_batch(self, batch: QueryBatch, out=None):
        stride, scores, segs, docs, counts = out or batch.alloc_out()
        _check(LIB.tq_search_batch(self.h, batch.ptr, batch.nq, stride, ptr(scores, f32p), ptr(segs, u32p), ptr(docs, u32p),
                                   ptr(counts, u32p)), self.h)
        return scores, segs, docs, counts

    def count_batch(self, qb: QueryBatch):
        """Count collector: alive docs matching each query (tq_count_batch)."""
        out = np.zeros(max(qb.nq, 1), dtype=np.uint64)
        _check(LIB.tq_count_batch(self.h, qb.ptr, qb.nq, ptr(out, u64p)), self.h)
        return out[:qb.nq]

    def prepare(self, batch: QueryBatch):
        return Batch(self, batch)

    def decode_postings(self, term_seg):
        ts = TermSeg(*[int(x) for x in term_seg])
        docs = np.zeros(max(ts.doc_freq, 1), dtype=np.uint32)
        tfs = np.zeros(max(ts.doc_freq, 1), dtype=np.uint32)
        _check(LIB.tq_decode_postings(self.h, C.byref(ts), ptr(docs, u32p), ptr(tfs, u32p)), self.h)
        return docs[:ts.doc_freq], tfs[:ts.doc_freq]

    def block_table(self, term_seg, weight, avg_fieldnorm):
        ts = TermSeg(*[int(x) for x in term_seg])
        n = ts.doc_freq // 128
        last = np.zeros(max(n, 1), dtype=np.uint32)
        bm = np.zeros(max(n, 1), dtype=np.float32)
        _check(LIB.tq_block_table(self.h, C.byref(ts), weight, avg_fieldnorm, ptr(last, u32p), ptr(bm, f32p)), self.h)
        return last[:n], bm[:n]

    def stats(self):
        s = Stats()
        _check(LIB.tq_get_stats(self.h, C.byref(s)), self.h)
        hs = HistogramStats()
        _check(LIB.tq_get_histogram_stats(self.h, C.byref(hs)), self.h)
        out = {name: (list(getattr(s, name)) if name in ("or_windows", "tile_counters", "tile_cycles", "tile_b2_exits") else getattr(s, name)) for name, _ in Stats._fields_}
        out.update({name: getattr(hs, name) for name, _ in HistogramStats._fields_})
        ts = TermsStats()
        _check(LIB.tq_get_terms_stats(self.h, C.byref(ts)), self.h)
        out.update({name: getattr(ts, name) for name, _ in TermsStats._fields_})
        ms = MetricsStats()
        _check(LIB.tq_get_metrics_stats(self.h, C.byref(ms)), self.h)
        out.update({name: getattr(ms, name) for name, _ in MetricsStats._fields_})
        hm = HistMetricsStats()
        _check(LIB.tq_get_hist_metrics_stats(self.h, C.byref(hm)), self.h)
        out.update({name: getattr(hm, name) for name, _ in HistMetricsStats._fields_})
        tm = TermsMetricsStats()
        _check(LIB.tq_get_terms_metrics_stats(self.h, C.byref(tm)), self.h)
        out.update({name: getattr(tm, name) for name, _ in TermsMetricsStats._fields_})
        rs = RangeStats()
        _check(LIB.tq_get_range_stats(self.h, C.byref(rs)), self.h)
        out.update({name: getattr(rs, name) for name, _ in RangeStats._fields_})
        th = TermsHistStats()
        _check(LIB.tq_get_terms_hist_stats(self.h, C.byref(th)), self.h)
        out.update({name: getattr(th, name) for name, _ in TermsHistStats._fields_})
        ht = HistTermsStats()
        _check(LIB.tq_get_hist_terms_stats(self.h, C.byref(ht)), self.h)
        out.update({name: getattr(ht, name) for name, _ in HistTermsStats._fields_})
        return out

    def merge_topk_dev(self, n_lists, nq, stride, k, scores, segs, docs, counts, out_scores, out_segs, out_docs, out_counts):
        """All arguments are raw device addresses (int), e.g. torch tensors' data_ptr()."""
        _check(LIB.tq_merge_topk_dev(self.h, n_lists, nq, stride, k, scores, segs, docs, counts, out_scores, out_segs, out_docs,
                                     out_counts), self.h)

    def merge_topk_packed_dev(self, stream, n_lists, nq, stride, k, packed, pitch_words, out_packed):
        """packed / out_packed: raw device addresses; stream: cudaStream_t as int (0 = the default stream).  No host sync."""
        _check(LIB.tq_merge_topk_packed_dev(self.h, stream, n_lists, nq, stride, k, packed, pitch_words, out_packed), self.h)

    def close(self):
        if getattr(self, "h", None):
            LIB.tq_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()


class MultiContext:
    """tq_multi: several devices behind one handle (segments sharded over them, in-process fan-out and merge)."""

    def __init__(self, devices):
        arr = (C.c_int * len(devices))(*devices)
        h = C.c_void_p()
        _check(LIB.tq_multi_create(arr, len(devices), C.byref(h)))
        self.h = h

    def segment_register(self, segment_ord, field, max_doc, record_option, idx_body, fieldnorm=None, alive=None, device_index=-1):
        idx_body = np.ascontiguousarray(idx_body, dtype=np.uint8)
        fn = None if fieldnorm is None else np.ascontiguousarray(fieldnorm, dtype=np.uint8)
        al = None if alive is None else np.ascontiguousarray(alive, dtype=np.uint8)
        rc = LIB.tq_multi_segment_register(self.h, device_index, segment_ord, field, max_doc, record_option, ptr(idx_body, u8p), idx_body.size,
                                           ptr(fn, u8p), 0 if fn is None else fn.size, ptr(al, u8p), 0 if al is None else al.size)
        if rc != 0:
            raise TqError(f"tantivy_b200 error {rc}: {LIB.tq_multi_last_error(self.h).decode(errors='replace')}")

    def segment_register_split(self, segment_ord, field, max_doc, record_option, idx_body, fieldnorm=None, alive=None):
        """One segment on every device of the handle, each evaluating its own doc range."""
        idx_body = np.ascontiguousarray(idx_body, dtype=np.uint8)
        fn = None if fieldnorm is None else np.ascontiguousarray(fieldnorm, dtype=np.uint8)
        al = None if alive is None else np.ascontiguousarray(alive, dtype=np.uint8)
        rc = LIB.tq_multi_segment_register_split(self.h, segment_ord, field, max_doc, record_option, ptr(idx_body, u8p), idx_body.size,
                                                 ptr(fn, u8p), 0 if fn is None else fn.size, ptr(al, u8p), 0 if al is None else al.size)
        if rc != 0:
            raise TqError(f"tantivy_b200 error {rc}: {LIB.tq_multi_last_error(self.h).decode(errors='replace')}")

    def filter_register(self, filter_id, segment_ord, bits):
        """Context.filter_register on every device that holds the segment (all of them for a split segment)."""
        b = np.ascontiguousarray(bits, dtype=np.uint8)
        rc = LIB.tq_multi_filter_register(self.h, filter_id, segment_ord, ptr(b, u8p), b.size)
        if rc != 0:
            raise TqError(f"tantivy_b200 error {rc}: {LIB.tq_multi_last_error(self.h).decode(errors='replace')}")

    def filter_unregister(self, filter_id):
        rc = LIB.tq_multi_filter_unregister(self.h, filter_id)
        if rc != 0:
            raise TqError(f"tantivy_b200 error {rc}: {LIB.tq_multi_last_error(self.h).decode(errors='replace')}")

    def search_batch(self, batch: QueryBatch, out=None):
        stride, scores, segs, docs, counts = out or batch.alloc_out()
        rc = LIB.tq_multi_search_batch(self.h, batch.ptr, batch.nq, stride, ptr(scores, f32p), ptr(segs, u32p), ptr(docs, u32p), ptr(counts, u32p))
        if rc != 0:
            raise TqError(f"tantivy_b200 error {rc}: {LIB.tq_multi_last_error(self.h).decode(errors='replace')}")
        return scores, segs, docs, counts

    def close(self):
        if getattr(self, "h", None):
            LIB.tq_multi_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()


class Batch:
    """tq_batch: prepare once, run (device only), fetch (D2H)."""

    def __init__(self, ctx: Context, qb: QueryBatch):
        self.ctx, self.qb = ctx, qb
        h = C.c_void_p()
        _check(LIB.tq_batch_prepare(ctx.h, qb.ptr, qb.nq, C.byref(h)), ctx.h)
        self.h = h

    def run(self):
        _check(LIB.tq_batch_run(self.h), self.ctx.h)

    def phases(self):
        return LIB.tq_batch_phases(self.h)

    def run_phase(self, phase):
        """Phases 0 .. phases()-1 in order; thresholds may be exchanged between two of them (tq_batch_run_phase)."""
        _check(LIB.tq_batch_run_phase(self.h, phase), self.ctx.h)

    def thresholds_export_dev(self, keys_dev):
        """keys_dev: device address of nq int64 (e.g. a torch tensor's data_ptr()); waits for the batch's stream."""
        _check(LIB.tq_batch_thresholds_export_dev(self.h, keys_dev), self.ctx.h)

    def thresholds_import_dev(self, keys_dev):
        _check(LIB.tq_batch_thresholds_import_dev(self.h, keys_dev), self.ctx.h)

    def stream(self):
        """The CUDA stream (cudaStream_t as int) every launch of this batch is enqueued on."""
        s = C.c_void_p()
        _check(LIB.tq_batch_stream(self.h, C.byref(s)), self.ctx.h)
        return s.value or 0

    def topkeys_export_dev(self, keys_dev, k_stride):
        """keys_dev: device address of nq * k_stride uint32; enqueued on the batch's stream, no host sync."""
        _check(LIB.tq_batch_topkeys_export_dev(self.h, keys_dev, k_stride), self.ctx.h)

    def thresholds_from_keys_dev(self, gathered_dev, n_shards, k_stride):
        _check(LIB.tq_batch_thresholds_from_keys_dev(self.h, gathered_dev, n_shards, k_stride), self.ctx.h)

    def fetch(self, out=None):
        stride, scores, segs, docs, counts = out or self.qb.alloc_out()
        _check(LIB.tq_batch_fetch(self.h, stride, ptr(scores, f32p), ptr(segs, u32p), ptr(docs, u32p), ptr(counts, u32p)), self.ctx.h)
        return scores, segs, docs, counts

    def fetch_hits(self):
        """The Count half of (Count, TopDocs): uint64 [nq], the matching alive docs of every query run with count_hits=True
        (0 for the others).  After a finished run, like fetch."""
        out = np.zeros(max(self.qb.nq, 1), dtype=np.uint64)
        _check(LIB.tq_batch_fetch_hits(self.h, ptr(out, u64p)), self.ctx.h)
        return out[:self.qb.nq]

    def results_dev(self):
        s, g, d, c = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        stride = C.c_uint32()
        _check(LIB.tq_batch_results_dev(self.h, C.byref(s), C.byref(g), C.byref(d), C.byref(c), C.byref(stride)), self.ctx.h)
        return s.value, g.value, d.value, c.value, stride.value

    def results_copy_dev(self, scores, segs, docs, counts):
        """raw device addresses (e.g. torch tensor .data_ptr()) of [nq, kmax] / [nq] buffers"""
        _check(LIB.tq_batch_results_copy_dev(self.h, scores, segs, docs, counts), self.ctx.h)

    def results_pack_dev(self, packed):
        """packed: raw device address of 3 * nq * kmax + nq 32-bit words (scores | segment ords | docs | counts)."""
        _check(LIB.tq_batch_results_pack_dev(self.h, packed), self.ctx.h)

    def results_pack_dev_async(self, packed):
        """As results_pack_dev, enqueued behind the run WITHOUT waiting for it; packed holds 4 more words (the run's overflow
        flags: non-zero on any shard = take results_pack_dev)."""
        _check(LIB.tq_batch_results_pack_dev_async(self.h, packed), self.ctx.h)

    def close(self):
        if getattr(self, "h", None):
            LIB.tq_batch_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()
