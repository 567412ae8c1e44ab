"""Histograms with metric sub-aggregations on the device (tq_histogram_metrics_batch: k_hist_metrics + k_hist_metrics_final) against
tests/hist_metrics_model.py (per segment the matching docs in doc order, bucketed as the reference buckets them, Kahan collection
per (bucket, metric), merge_fruits by bucket in segment_ord order) over the docs tests/score_model.py matches (and-ed with the alive
bits, the filter and the doc range, as Count counts them).  Rows, keys and doc counts must be exact, and equal to
tq_histogram_batch's; count, min and max exact always; every accepted sum and average bit-equal to the model's; every column built to
fail the guard refused wherever a bucket collects enough of its values.  The fixture is test_gpu_metrics' (test_gpu_sort_field's three
segments with deletes, the `edge` term on every tile and unit edge, the metric columns) with histogram columns: nanosecond
timestamps whose tiles lie inside one bucket, straddle buckets, or jump far apart (one-bucket runs in units whose window is too wide
for shared memory), the random u64 column and f64 columns with NaN and +-inf."""
import os
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200 import hist_metrics as HMx  # noqa: E402
from tantivy_b200 import metrics as Mx  # noqa: E402
from tantivy_b200._abi import TQ_FAST_I64, TQ_FAST_U64, TQ_METRIC_COUNT_ONLY, TQ_OP_TERM, QueryBatch  # noqa: E402
from tests import hist_metrics_model as HMM  # noqa: E402
from tests import metrics_model as MM  # noqa: E402
from tests.helpers import OracleSegment, make_query  # noqa: E402
from tests.test_gpu_metrics import MetricsFixture, same, to_f64  # noqa: E402
from tests.test_gpu_parity import fresh_ord  # noqa: E402
from tests.test_gpu_sort_field import ALL, FILTER_KINDS, packed, shapes  # noqa: E402
from tests.test_hist_metrics_host import FIXTURES, check_asserts, fixture_plan  # noqa: E402

TYPES = ("stats", "sum", "avg", "min", "max", "value_count")
MUST_REFUSE = {"decimal": 50, "ns": 20}  # columns whose bucket sums the guard must refuse from this many values on
HOUR = 3600 * 10**9


class HistMetricsFixture(MetricsFixture):
    def __init__(self):
        super().__init__()
        rng = np.random.default_rng(0x4D7)
        t0 = np.int64(1_700_000_000) * 10**9 - np.int64(1_700_000_000 % 3600) * 10**9  # an hour boundary
        starts = (t0, t0 + 40 * HOUR, t0 + 500 * HOUR)
        for i, s in enumerate(self.osegs):
            n = s.max_doc
            doc = np.arange(n, dtype=np.int64)
            if i == 0:  # about a second apart: tiles straddle minutes, lie inside days
                ts = starts[0] + np.cumsum(rng.integers(0, 2 * 10**9, size=n))
            elif i == 1:  # tiles 30 h apart, 100 ms steps inside: one bucket per tile at 1 h, units of several hundred buckets
                ts = starts[1] + (doc // 8192) * 30 * HOUR + (doc % 8192) * 10**8
            else:  # a millisecond apart: one-bucket runs at 1 min
                ts = starts[2] + doc * 10**6
            self.columns.setdefault("ts", []).append((T.fast_value_to_u64(ts, "date"), (rng.random(n) < 0.97) if i != 2 else None))
        self.kind["ts"] = "date"
        self.mcol["ts"] = 500 + len(self.mcol)


def sub_aggs(cols, missing=None):
    """One aggregation of every type on each column (field = the column's name)."""
    out = {}
    for c in cols:
        body = {"field": c} if missing is None else {"field": c, "missing": missing}
        for typ in TYPES:
            out[f"{c}.{typ}"] = {typ: body}
    return out


def fields_of(fx, names):
    return {c: Mx.MetricField(fx.mcol[c], fx.kind[c]) for c in names}


def metric_values(fx, i, c, typ, missing):
    """Per doc of segment i the list of values a metric of type typ on column c collects: metrics_model.doc_values, computed for
    the whole column at once (cached on the fixture)."""
    cache = fx.__dict__.setdefault("_metric_values", {})
    key = (i, c, MM.column_type(typ, fx.kind[c]), missing)
    if key not in cache:
        v, p = fx.columns[c][i]
        ctype = key[2]
        pres = np.ones(len(v), bool) if p is None else np.asarray(p, bool)
        if ctype == "empty":
            ctype, pres = "u64", np.zeros(len(v), bool)
        numeric = ctype in MM.NUMERIC
        f = to_f64(v, fx.kind[c]) if numeric else np.zeros(len(v))
        mv = None if missing is None else MM.missing_value(float(missing), ctype)
        vals = np.where(pres, f, (mv if numeric else 0.0) if mv is not None else 0.0)
        has = pres | (mv is not None)
        f_all, p_all = to_f64(v, fx.kind[c]), (np.ones(len(v), bool) if p is None else p)
        for d in range(0, len(v), 997):  # (spot check against the model's per-doc rule)
            want = MM.doc_values(typ, fx.kind[c], float(f_all[d]) if p_all[d] else None, missing)
            assert len(want) == int(has[d]) and (not want or struct.pack("<d", want[0]) == struct.pack("<d", vals[d])), (c, typ, d)
        cache[key] = [[x] if h else [] for x, h in zip(vals.tolist(), has.tolist())]
    return cache[key]


class Model:
    """The model's result of one request over the fixture, per query (values computed once per segment and metric key)."""

    def __init__(self, fx, r):
        self.fx, self.r = fx, r
        self.keys = {}  # agg name -> (column, column type, missing)
        for a in r.metrics:
            self.keys[a.name] = (a.field, MM.column_type(a.type, fx.kind[a.field]), a.missing, a.type)
        self.values = {}

    def vals(self, i, key):
        if (i, key[:3]) not in self.values:
            self.values[(i, key[:3])] = metric_values(self.fx, i, key[0], key[3], key[2])
        return self.values[(i, key[:3])]

    def __call__(self, qt, masks=None, segs=None):
        fx, r = self.fx, self.r
        req = r.req
        spec = HMx.Hg.histogram_spec(req, 0, fx.kind[req.field])
        lo, hi = (spec[4], spec[5])
        parts = []
        for i, s in sorted(enumerate(fx.osegs), key=lambda x: x[1].segment_ord):
            if segs is not None and i not in segs:
                continue
            sel = fx.has(i, qt) & fx.alive[i]
            if masks is not None:
                sel = sel & masks[i]
            v, p = fx.columns[req.field][i]
            buckets = HMM.segment_buckets(v, p, sel, fx.kind[req.field], spec[2], spec[3], lo, hi)
            parts.append(HMM.segment_part(buckets, {k[:3]: self.vals(i, k) for k in self.keys.values()}))
        merged = HMM.merge(parts)
        metrics = [(a.name, a.type, self.keys[a.name][:3], a.none_if_no_match) for a in r.metrics]
        return HMM.final(r.name, req, fx.kind[req.field], merged, metrics), merged


def buckets_of(res, name="h"):
    b = res[name]["buckets"]
    return list(b.values()) if isinstance(b, dict) else b


def check(ctxs, fx, qts, hist, cols, missing=None, masks=None, count_hits=True, extra=None):
    """Runs qts with one request over every context and compares with the model; returns (accepted, refused) sum-bearing results."""
    aggs = {"h": dict(hist, aggs=dict(sub_aggs(cols, missing), **(extra or {})))}
    r = HMx.parse_request(aggs)
    hfield = r.req.field
    fields = fields_of(fx, set(cols) | {hfield} | {v[next(iter(v))]["field"] for v in (extra or {}).values()})
    qb = QueryBatch([qt[0] for qt in qts])
    out = HMx.run(ctxs, qb, [r] * len(qts), fields, count_hits=count_hits)
    res, hits = out if count_hits else (out, None)
    if count_hits:
        assert np.array_equal(hits, sum(c.count_batch(qb) for c in ctxs))
    if len(ctxs) == 1:  # rows and doc counts: tq_histogram_batch's
        p = HMx.plan(r, fields)
        dev = ctxs[0].hist_metrics_batch(qb, [p.hspec] * len(qts), [p.mplan.columns] * len(qts))
        ref = ctxs[0].histogram_batch(qb, [p.hspec] * len(qts))
        for q in range(len(qts)):
            n = int(ref[2][q])
            assert int(dev[3][q]) == n and np.array_equal(dev[0][q, :n], ref[0][q, :n]) and np.array_equal(dev[1][q, :n], ref[1][q, :n])
    model = Model(fx, r)
    tally = [0, 0]
    for qt, got in zip(qts, res):
        want, merged = model(qt, masks)
        answered, refused = (got.answered, got.refused) if isinstance(got, HMx.HistMetricsRefused) else (got, {})
        gb, wb = buckets_of(answered), buckets_of(want)
        assert [(b["key"], b["doc_count"]) for b in gb] == [(b["key"], b["doc_count"]) for b in wb], (hist, qt[1])
        for name in refused:
            assert name.split(".")[1] in Mx.SUM_BEARING, name
            tally[1] += 1
        for a in r.metrics:
            if a.name in refused:
                continue
            tally[0] += a.type in Mx.SUM_BEARING
            for g, w in zip(gb, wb):
                assert same(g[a.name], w[a.name]), (a.name, qt[1], g["key"], g[a.name], w[a.name])
            col = a.field
            if col in MUST_REFUSE and a.type in Mx.SUM_BEARING:
                k = model.keys[a.name][:3]
                worst = max((st[k].count for _, st in merged.values()), default=0)
                assert worst < MUST_REFUSE[col], f"{a.name} on {worst} values in one bucket should have been refused"
    return tally


@pytest.fixture(scope="module")
def fx():
    return HistMetricsFixture()


@pytest.fixture(scope="module")
def ctx(fx):
    c = fx.register(T.Context(0), filters=FILTER_KINDS)
    yield c
    c.close()


HISTS = {
    "ts_1m": {"date_histogram": {"field": "ts", "fixed_interval": "1m", "min_doc_count": 1}},
    "ts_2h": {"date_histogram": {"field": "ts", "fixed_interval": "2h", "offset": "-30m"}},
    "ts_1h": {"date_histogram": {"field": "ts", "fixed_interval": "1h"}},
    "ts_1d": {"date_histogram": {"field": "ts", "fixed_interval": "1d", "min_doc_count": 1}},
    "rand_128": {"histogram": {"field": "uniform", "interval": 2.0**57}},
    "rand_256": {"histogram": {"field": "uniform", "interval": 2.0**56}},
    "nan_inf": {"histogram": {"field": "nan_inf", "interval": 0.5}},
    "nan_inf_hard": {"histogram": {"field": "nan_inf", "interval": 0.5, "hard_bounds": {"min": -1.0, "max": 1.0}}},
    "f64_hard": {"histogram": {"field": "f64", "interval": 1.0, "hard_bounds": {"min": -1.5, "max": 2.5}}},
}
GROUPS = [("ints",), ("ints", "big"), ("dyadic", "decimal", "flag"), ("partial", "ns", "const", "clustered"), ("nan_inf", "i64", "us_half")]


@pytest.mark.parametrize("hist", list(HISTS))
def test_histograms_against_model(ctx, fx, hist):
    """Every histogram column and interval with 1-4 metric columns; every query shape for the first group."""
    qts = shapes(fx) if hist in ("ts_1h", "rand_128") else shapes(fx)[::2]
    acc = ref = 0
    for j, cols in enumerate(GROUPS):
        a, r = check([ctx], fx, qts if j == 0 else qts[:: 3 + j], HISTS[hist], cols)
        acc, ref = acc + a, ref + r
    assert acc > 0


def test_guard_refuses_decimals_and_nanoseconds_per_bucket(ctx, fx):
    acc, ref = check([ctx], fx, shapes(fx)[:8], HISTS["ts_1d"], ("ints", "decimal", "ns"))
    assert acc > 0 and ref > 0


@pytest.mark.parametrize("fkind", FILTER_KINDS)
def test_filters(ctx, fx, fkind):
    j = FILTER_KINDS.index(fkind)
    qts = [(dict(q, filter=200 + j), t) for q, t in shapes(fx)[:8]]
    check([ctx], fx, qts, HISTS["ts_1h"], ("ints", "dyadic", "flag"), masks=fx.filters[fkind])
    check([ctx], fx, qts[:4], HISTS["rand_128"], ("partial",), masks=fx.filters[fkind], count_hits=False)


@pytest.mark.parametrize("missing", [7, -3.5])
def test_missing_and_the_same_column_twice(ctx, fx, missing):
    extra = {"ints_m.sum": {"sum": {"field": "ints", "missing": missing}}, "flag_n.value_count": {"value_count": {"field": "flag", "missing": missing}}}
    check([ctx], fx, shapes(fx)[:10], HISTS["ts_2h"], ("partial", "half"), missing=missing, extra=extra)
    check([ctx], fx, shapes(fx)[:6], HISTS["ts_1m"], ("us_half",), missing=missing)


def test_shared_and_global_windows_and_one_bucket_runs(fx):
    c = fx.register(T.Context(0))
    try:
        check([c], fx, shapes(fx)[:6], HISTS["rand_128"], ("ints",))
        st = c.stats()
        assert st["hist_metrics_flush_shared"] > 0 and st["hist_metrics_flush_global"] == 0
        check([c], fx, shapes(fx)[:6], HISTS["ts_1h"], ("ints", "const"))  # segment 1: one-bucket tiles, windows of ~200 buckets
        st2 = c.stats()
        assert st2["hist_metrics_flush_global"] > 0 and st2["hist_metrics_tiles_one_bucket"] > st["hist_metrics_tiles_one_bucket"]
        assert st2["hist_metrics_tiles_seen"] >= st2["hist_metrics_tiles_one_bucket"] and st2["hist_metrics_ms"] > 0 and st2["units_hist_metrics"] > 0
    finally:
        c.close()


def test_split_segments_over_two_contexts(fx):
    """The big segment's halves in two contexts (doc ranges), merged by hist_metrics.run, against one context over all of it."""
    big = fx.osegs[0]
    half = (big.max_doc // 8192 // 2) * 8192 + 100
    cols = ("ints", "dyadic", "partial")
    ctxs = []
    try:
        for lo, hi in ((0, half), (half, big.max_doc), (0, big.max_doc)):
            c = T.Context(0)
            big.register(c)
            c.segment_set_doc_range(big.segment_ord, 0, lo, hi)
            for k in cols + ("ts",):
                v, p = fx.columns[k][0]
                c.sort_column_register(fx.mcol[k], big.segment_ord, v, None if p is None else packed(p))
            ctxs.append(c)
        aggs = {"h": dict(HISTS["ts_1m"], aggs=sub_aggs(cols))}
        r = HMx.parse_request(aggs)
        fields = fields_of(fx, cols + ("ts",))
        model = Model(fx, r)
        for hits in (False, True):
            for q, t in shapes(fx)[:8]:
                q = dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] == big.segment_ord])
                qb = QueryBatch([q])
                split = HMx.run(ctxs[:2], qb, [r], fields, count_hits=hits)
                one = HMx.run(ctxs[2:], qb, [r], fields, count_hits=hits)
                if hits:
                    (split, hs), (one, ho) = split, one
                    assert np.array_equal(hs, ho)
                split, one = split[0], one[0]
                if isinstance(one, HMx.HistMetricsRefused):
                    assert isinstance(split, HMx.HistMetricsRefused) and split.refused.keys() == one.refused.keys()
                    split, one = split.answered, one.answered
                assert same(split, one)
                want, _ = model((q, t), segs={0})
                for g, w in zip(buckets_of(one), buckets_of(want)):
                    assert g["key"] == w["key"] and g["doc_count"] == w["doc_count"]
                    for name in g:
                        if name not in ("key", "doc_count", "key_as_string"):
                            assert same(g[name], w[name]), name
    finally:
        for c in ctxs:
            c.close()


def ramp_context(n, values):
    lists = [(np.arange(n, dtype=np.uint32), np.ones(n, np.uint32))]
    seg = OracleSegment(lists, None, segment_ord=fresh_ord(), writer_cls=T.FieldWriter, max_doc=n)
    c = T.Context(0)
    seg.register(c)
    c.sort_column_register(1, seg.segment_ord, T.fast_value_to_u64(values, "i64"))
    return c, make_query(TQ_OP_TERM, [seg], [0], 10)


def code(fn):
    with pytest.raises(T.TqError) as e:
        fn()
    return int(str(e.value).split("error ")[1].split(":")[0])


def test_range_limit_waves_and_stride():
    """A range of exactly 2^16 buckets runs, one more is TQ_ERR_UNSUPPORTED; a tiny budget runs one query per wave and a
    one-bucket stride retries, both with the same rows and parts."""
    n = 1 << 16
    c, q = ramp_context(n + 1, np.minimum(np.arange(n + 1), n - 1))
    try:
        qb = QueryBatch([q])
        spec = (1, TQ_FAST_I64, 1.0, 0.0)
        cols = [(1, TQ_FAST_I64), (1, TQ_FAST_I64, TQ_METRIC_COUNT_ONLY)]
        pos, counts, parts, nb = c.hist_metrics_batch(qb, [spec], [cols])
        assert int(nb[0]) == n and np.array_equal(pos[0, :n], np.arange(n)) and counts[0, :n].sum() == n + 1 and counts[0, n - 1] == 2
        assert np.array_equal(parts[0, :n, 0]["sum"], np.arange(n) * counts[0, :n]) and (parts[0, :n, 1]["count"] == counts[0, :n]).all()
        assert (parts[0, :n, 2:]["count"] == 0).all()
    finally:
        c.close()
    c, q = ramp_context(n + 1, np.arange(n + 1))
    try:
        assert code(lambda: c.hist_metrics_batch(QueryBatch([q]), [spec], [cols])) == -4
    finally:
        c.close()


def test_waves_and_stride_retry(fx):
    qts = shapes(fx)[:12]
    qb = QueryBatch([qt[0] for qt in qts])
    r = HMx.parse_request({"h": dict(HISTS["ts_2h"], aggs=sub_aggs(("ints", "partial")))})
    p = HMx.plan(r, fields_of(fx, ("ints", "partial", "ts")))
    args = (qb, [p.hspec] * len(qts), [p.mplan.columns] * len(qts))
    base = fx.register(T.Context(0))
    os.environ["TQ_HIST_METRICS_BUDGET"] = "8"  # every query alone in its wave
    try:
        small = fx.register(T.Context(0))
    finally:
        del os.environ["TQ_HIST_METRICS_BUDGET"]
    try:
        want = base.hist_metrics_batch(*args, count_hits=True)
        for got in (small.hist_metrics_batch(*args, count_hits=True), base.hist_metrics_batch(*args, count_hits=True, stride=1)):
            for q in range(len(qts)):
                n = int(want[3][q])
                assert int(got[3][q]) == n
                assert np.array_equal(got[0][q, :n], want[0][q, :n]) and np.array_equal(got[1][q, :n], want[1][q, :n])
                for f in ("count", "n_nan", "n_inf", "min_image", "max_image", "quantum_exp", "sum", "magnitude"):
                    assert np.array_equal(got[2][q, :n][f], want[2][q, :n][f]), f
            assert np.array_equal(got[4], want[4])
        assert max(int(x) for x in want[3]) > 1
    finally:
        base.close()
        small.close()


def test_one_run_per_call_once_the_width_is_known(fx):
    """A row wider than the first stride costs one more run of the kernels; the context then starts at the widest row it has
    returned, so the same batch runs once.  An empty batch returns empty arrays."""
    qts = shapes(fx)[:8]
    qb = QueryBatch([qt[0] for qt in qts])
    r = HMx.parse_request({"h": dict(HISTS["ts_1m"], aggs=sub_aggs(("ints",)))})
    p = HMx.plan(r, fields_of(fx, ("ints", "ts")))
    args = (qb, [p.hspec] * len(qts), [p.mplan.columns] * len(qts))
    c = fx.register(T.Context(0))
    try:
        runs = lambda: c.stats()["units_hist_metrics"]  # noqa: E731
        u0 = runs()
        first = c.hist_metrics_batch(*args)
        u1 = runs()
        second = c.hist_metrics_batch(*args)
        u2 = runs()
        assert int(first[3].max()) > 256 and u1 - u0 == 2 * (u2 - u1) > 0
        assert np.array_equal(first[3], second[3])
        for q, n in enumerate(first[3].tolist()):  # (entries past n[q] are not written)
            for a, b in zip(first[:2] + (first[2]["count"],), second[:2] + (second[2]["count"],)):
                assert np.array_equal(a[q, :n], b[q, :n])
        empty = c.hist_metrics_batch(QueryBatch([]), [], [], count_hits=True)
        assert [x.shape[0] for x in empty] == [0] * 5
    finally:
        c.close()


def test_rows_of_a_wave_with_one_wide_query(fx):
    """Narrow queries around one whose range is wide: each query's row holds at most its range, so the wave's rows stay within
    its accumulators; every row equals the query's row run alone."""
    qts = shapes(fx)[:6]
    hs = [HMx.plan(HMx.parse_request({"h": dict(HISTS[k], aggs=sub_aggs(("ints",)))}), fields_of(fx, ("ints", "ts", "uniform")))
          for k in ("ts_1d", "ts_1m", "rand_128")]
    specs = [hs[i % 3] for i in range(len(qts))]
    qb = QueryBatch([qt[0] for qt in qts])
    c = fx.register(T.Context(0))
    try:
        out = c.hist_metrics_batch(qb, [p.hspec for p in specs], [p.mplan.columns for p in specs], stride=1 << 16)
        for q, (qt, p) in enumerate(zip(qts, specs)):
            one = c.hist_metrics_batch(QueryBatch([qt[0]]), [p.hspec], [p.mplan.columns])
            n = int(one[3][0])
            assert int(out[3][q]) == n and np.array_equal(out[0][q, :n], one[0][0, :n]) and np.array_equal(out[1][q, :n], one[1][0, :n])
            for f in ("count", "min_image", "max_image", "sum", "quantum_exp"):
                assert np.array_equal(out[2][q, :n][f], one[2][0, :n][f]), f
    finally:
        c.close()


def test_error_codes(fx):
    c = fx.register(T.Context(0))
    try:
        qt = fx.query(TQ_OP_TERM, [ALL], 10)
        qb = QueryBatch([qt[0]])
        h = (fx.mcol["ts"], "date", 60e9, 0.0)
        good = [(fx.mcol["ints"], TQ_FAST_U64)]
        assert code(lambda: c.hist_metrics_batch(qb, [(999, "date", 60e9, 0.0)], [good])) == -3
        assert code(lambda: c.hist_metrics_batch(qb, [h], [[(999, TQ_FAST_U64)]])) == -3
        for hs, ms in (((fx.mcol["ts"], 7, 60e9, 0.0), good), ((fx.mcol["ts"], "date", 0.0, 0.0), good), ((fx.mcol["ts"], "date", np.inf, 0.0), good),
                       (h, []), (h, good * 5), (h, [(fx.mcol["ints"], 9)]), (h, [(fx.mcol["ints"], TQ_FAST_U64, 16, 0)])):
            assert code(lambda: c.hist_metrics_batch(qb, [hs], [ms])) == -1
        phrase = dict(qt[0], op=3, term_pos=[(0, 0)] * len(qt[0]["term_segs"]), term_offset=[0])
        assert code(lambda: c.hist_metrics_batch(QueryBatch([phrase]), [h], [good])) == -4
    finally:
        c.close()


def fixture_column(kind, docs, field):
    present = np.array([field in d for d in docs], bool)
    vals = np.array([d.get(field, 0) for d in docs], np.float64 if kind == "f64" else np.int64)
    return T.fast_value_to_u64(vals, kind), present


@pytest.mark.parametrize("case", FIXTURES, ids=[c["name"] for c in FIXTURES])
def test_reference_fixtures_on_device(case):
    """The reference's vectors end to end: every segment a real segment whose term 0 lists the collected docs, every field a
    registered column, the rows finalised by tantivy_b200.hist_metrics."""
    p, fields = fixture_plan(case)
    c = T.Context(0)
    try:
        segs = []
        for docs in case["segments"]:
            n = len(docs)
            hit = np.array([i for i, d in enumerate(docs) if d["hit"]] or [0], np.uint32)
            s = OracleSegment([(hit, np.ones(len(hit), np.uint32))], [1] * n, segment_ord=fresh_ord(), writer_cls=T.FieldWriter)
            s.register(c)
            for name, f in fields.items():
                images, present = fixture_column(case["fields"][name], docs, name)
                c.sort_column_register(f.column_id, s.segment_ord, images, None if present.all() else packed(present))
            segs.append(s)
        q = make_query(TQ_OP_TERM, segs, [0], 10) if segs else dict(op=TQ_OP_TERM, k=10, weights=[1.0], avg_fieldnorm=[1.0], term_segs=[])
        res, hits = HMx.run([c], QueryBatch([q]), [p.request], fields, count_hits=True)
        assert int(hits[0]) == sum(d["hit"] for docs in case["segments"] for d in docs)
        check_asserts(case, res[0])
    finally:
        c.close()
