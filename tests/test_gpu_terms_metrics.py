"""Terms aggregations with metric sub-aggregations on the device (tq_terms_metrics_batch: k_terms, k_terms_order, k_terms_select,
k_terms_select_metric, k_terms_mark, k_terms_metrics) against tests/terms_metrics_model.py (per segment the counted docs by key in doc
order with Kahan collection, the cut of rule 3, merge_fruits in segment_ord order, the final order of rule 4) over the docs
tests/score_model.py matches (and-ed with the alive bits, the filter and the doc range, as Count counts them).  Rows, keys, doc counts,
both scalars, metric counts, min and max must be exact, and for `_count` / `_key` equal to tq_terms_batch's; every accepted sum and
average bit-equal to the model's; a column built to fail the guard refused.  The fixture is test_gpu_metrics' (three segments with
deletes, the `edge` term on every tile and unit edge, its metric columns) with terms columns of every kind and columns built for the
metric order: values equal across keys at the cut, -0.0 against +0.0, keys with docs but no metric value."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200 import metrics as Mx  # noqa: E402
from tantivy_b200 import terms as Tm  # noqa: E402
from tantivy_b200 import terms_metrics as TMx  # noqa: E402
from tantivy_b200._abi import (TQ_FAST_U64, TQ_OP_OR, TQ_OP_TERM, TQ_TERMS_BY_COUNT, TQ_TERMS_BY_METRIC, TQ_TERMS_MISSING_AFTER_MAX,  # noqa: E402
                               TQ_TERMS_MISSING_NONE, TQ_TERMS_ORDER_AVG, QueryBatch)
from tests import terms_metrics_model as TMM  # noqa: E402
from tests import metrics_model as MM  # noqa: E402
from tests.test_gpu_hist_metrics import code, metric_values  # noqa: E402
from tests.test_gpu_metrics import MetricsFixture, same  # noqa: E402
from tests.test_gpu_sort_field import ALL, FILTER_KINDS, packed, shapes  # noqa: E402

TYPES = ("stats", "sum", "avg", "min", "max", "value_count")
MUST_REFUSE = {"decimal": 50, "ns": 20}  # columns whose bucket sums the guard must refuse from this many values on
N_STR = 20


class TermsMetricsFixture(MetricsFixture):
    def __init__(self):
        super().__init__()
        rng = np.random.default_rng(0x7E6)
        for i, s in enumerate(self.osegs):
            n = s.max_doc
            doc = np.arange(n)
            span = rng.integers(0, 1 << 20, size=n).astype(np.uint64)
            span[[0, n - 1]] = [0, (1 << 20) - 1]
            span1 = span.copy()
            span1[n - 1] = 1 << 20
            ties = doc % 50
            extra = {
                "k_str": ("str", rng.integers(0, N_STR, size=n).astype(np.uint64), rng.random(n) < 0.9),
                "k_i64": ("i64", T.fast_value_to_u64(rng.integers(-20, 20, size=n), "i64"), None),
                "k_f64": ("f64", T.fast_value_to_u64(1.0 + rng.integers(0, 4, size=n) * 2.0**-52, "f64"), None),
                "k_date": ("date", T.fast_value_to_u64(np.int64(1_600_000_000) * 10**9 + rng.integers(0, 40, size=n) * 1000, "date"), None),
                "k_r10k": ("u64", rng.integers(0, 10_000, size=n).astype(np.uint64), None),
                "k_ties": ("u64", ties.astype(np.uint64), None),
                "span20": ("u64", span, None),
                "span20p1": ("u64", span1, None),
                # a metric of k_ties' key alone: every order value ties across ten keys
                "tv": ("f64", T.fast_value_to_u64((ties % 5).astype(np.float64), "f64"), None),
                # -0.0 on the even keys of k_ties, +0.0 on the odd ones: equal under partial_cmp, ordered under total_cmp
                "zeros": ("f64", T.fast_value_to_u64(np.where(ties % 2 == 0, -0.0, 0.0), "f64"), None),
                # no value on the keys of k_ties that are multiples of 7: keys with docs but no metric value
                "sparse": ("u64", rng.integers(0, 100, size=n).astype(np.uint64), ties % 7 != 0),
            }
            for k, (kind, v, p) in extra.items():
                self.columns.setdefault(k, []).append((v, p))
                self.kind[k] = kind
        self.mcol = {k: 500 + i for i, k in enumerate(self.columns)}

    def missing_image(self, col, i, tspec):
        mode, image = tspec[4], tspec[5]
        if mode == TQ_TERMS_MISSING_NONE:
            return None
        if mode != TQ_TERMS_MISSING_AFTER_MAX:
            return image
        v, p = self.columns[col][i]
        have = v if p is None else v[p]
        return (int(have.max()) if len(have) else 0) + 1


def sub_aggs(cols, missing=None):
    out = {}
    for c in cols:
        body = {"field": c} if missing is None else {"field": c, "missing": missing}
        for typ in TYPES:
            out[f"{c}_{typ}"] = {typ: body}
    return out


def fields_of(fx, names):
    return {c: Mx.MetricField(fx.mcol[c], fx.kind[c]) for c in names}


def dictionaries(fx):
    """A str column's terms per segment: its ordinals' texts."""
    return {s.segment_ord: [f"term{j:02d}" for j in range(N_STR)] for s in fx.osegs}


class Model:
    """The model's result of one request over the fixture."""

    def __init__(self, fx, r, p):
        self.fx, self.r, self.p = fx, r, p
        self.keys = {a.name: (a.field, MM.column_type(a.type, fx.kind[a.field]), a.missing, a.type) for a in r.metrics}
        self.values = {}

    def vals(self, i, key):
        if (i, key[:3]) not in self.values:
            self.values[(i, key[:3])] = metric_values(self.fx, i, key[0], key[3], key[2])
        return self.values[(i, key[:3])]

    def __call__(self, qt, masks=None, segs=None):
        """(rows [(segment_ord, image, doc_count)], sum_other, error, final result, per-segment kept entries)."""
        fx, r, p = self.fx, self.r, self.p
        req, col = r.req, r.req.field
        target = "metric" if r.order else req.order_target
        order = None
        if r.order:
            typ = next(a.type for a in r.metrics if a.name == r.order[0])
            prop = req.order_target.partition(".")[2] or {"value_count": "count"}.get(typ, typ)
            order = (self.keys[r.order[0]][:3], prop)
        rows, other, error, results = [], 0, 0, []
        dicts = dictionaries(fx)
        for i in sorted(range(len(fx.osegs)), key=lambda i: fx.osegs[i].segment_ord):
            if segs is not None and i not in segs:
                continue
            sel = fx.has(i, qt) & fx.alive[i]
            if masks is not None:
                sel = sel & masks[i]
            v, pr = fx.columns[col][i]
            mi = fx.missing_image(col, i, p.tspec)
            docs = TMM.segment_docs(v, pr, sel, mi)
            entries = {k: (len(d), {key[:3]: TMM.collect(self.vals(i, key), d) for key in self.keys.values()}) for k, d in docs.items()}
            kept, e, o = TMM.cut(entries, req.segment_size, target, req.order == "asc", order)
            so = fx.osegs[i].segment_ord
            rows += [(so, k, c) for k, (c, _) in sorted(kept.items())]
            other, error = other + o, error + e
            seg = {}
            for k in sorted(kept):  # (terms.segment_result's key mapping: a str column's missing entry first)
                if p.kind == "str" and req.missing is not None and k == mi:
                    seg[Tm._missing_key(req.missing)] = kept[k]
            for k in sorted(kept):
                if not (p.kind == "str" and req.missing is not None and k == mi):
                    seg[Tm.intermediate_key(k, p.kind, dicts[so])] = kept[k]
            results.append((seg, o, e))
        merged = TMM.merge(results)
        metrics = [(a.name, a.type, self.keys[a.name][:3], a.none_if_no_match) for a in r.metrics]
        return rows, other, error, TMM.final(r.name, req, merged, metrics, None if order is None else (r.order[0], order[1]))


def check(ctxs, fx, qts, terms, cols, missing=None, masks=None, count_hits=True, extra=None):
    """Runs qts with one request over every context and compares with the model; returns (accepted sum-bearing results, refusals)."""
    aggs = {"t": {"terms": terms, "aggs": dict(sub_aggs(cols, missing), **(extra or {}))}}
    r = TMx.parse_request(aggs)
    fields = fields_of(fx, set(cols) | {r.req.field} | {v[next(iter(v))]["field"] for v in (extra or {}).values()})
    p = TMx.plan(r, fields)
    qb = QueryBatch([qt[0] for qt in qts])
    missing = {s.segment_ord: fx.missing_image(r.req.field, i, p.tspec) for i, s in enumerate(fx.osegs)}
    out = TMx.run(ctxs, qb, [r] * len(qts), fields, count_hits=count_hits, dictionaries=dictionaries(fx), missing_images=missing)
    res, hits = out if count_hits else (out, None)
    if count_hits:
        assert np.array_equal(hits, sum(c.count_batch(qb) for c in ctxs))
    model = Model(fx, r, p)
    wants = [model(qt, masks) for qt in qts]
    if len(ctxs) == 1:  # the rows and scalars; for _count / _key tq_terms_batch's
        dev = ctxs[0].terms_metrics_batch(qb, [p.tspec] * len(qts), [p.mplan.columns] * len(qts), [p.order] * len(qts))
        ref = ctxs[0].terms_batch(qb, [p.tspec] * len(qts)) if p.order is None else None
        for q, w in enumerate(wants):
            n = int(dev[4][q])
            got = [(int(dev[0][q, j]), int(dev[1][q, j]), int(dev[2][q, j])) for j in range(n)]
            assert got == w[0], (terms, qts[q][1])
            assert (int(dev[5][q]), int(dev[6][q])) == (w[1], w[2]), (terms, qts[q][1])
            if ref is not None:
                assert n == int(ref[3][q]) and (int(ref[4][q]), int(ref[5][q])) == (w[1], w[2])
    tally = [0, 0]
    for qt, got, want in zip(qts, res, wants):
        want = want[3]
        if isinstance(got, TMx.TermsMetricsRefused) and not got.answered:  # the order refused
            col = next(a.field for a in r.metrics if p.mplan.slot[a.name] == p.order[0])
            assert col in MUST_REFUSE or col == "nan_inf", (col, str(got))
            tally[1] += 1
            continue
        answered, refused = (got.answered, got.refused) if isinstance(got, TMx.TermsMetricsRefused) else (got, {})
        gb, wb = answered["t"]["buckets"], want["t"]["buckets"]
        assert [(b["key"], b["doc_count"]) for b in gb] == [(b["key"], b["doc_count"]) for b in wb], (terms, qt[1])
        for k in ("sum_other_doc_count", "doc_count_error_upper_bound"):
            assert answered["t"].get(k) == want["t"].get(k), (k, terms, qt[1])
        for name in refused:
            assert next(a.type for a in r.metrics if a.name == name) in Mx.SUM_BEARING, name
            tally[1] += 1
        for a in r.metrics:
            if a.name in refused:
                continue
            tally[0] += a.type in Mx.SUM_BEARING
            for g, w in zip(gb, wb):
                assert same(g[a.name], w[a.name]), (a.name, terms, qt[1], g["key"], g[a.name], w[a.name])
    return tally


@pytest.fixture(scope="module")
def fx():
    return TermsMetricsFixture()


@pytest.fixture(scope="module")
def ctx(fx):
    c = fx.register(T.Context(0), filters=FILTER_KINDS)
    yield c
    c.close()


ORDERS = [{"_count": "desc"}, {"_count": "asc"}, {"_key": "desc"}, {"_key": "asc"}, {"ints_avg": "desc"}, {"ints_stats.min": "asc"},
          {"sparse_value_count": "desc"}, {"ints_stats.sum": "asc"}, {"sparse_max": "desc"}, {"sparse_avg": "asc"}, {"ints_sum": "desc"},
          {"sparse_stats.avg": "desc"}, {"ints_min": "desc"}, {"ints_stats.count": "asc"}, {"sparse_stats.max": "asc"}]
TERMS_COLS = ["k_str", "k_i64", "k_f64", "k_date", "flag", "partial", "clustered", "k_r10k", "k_ties"]


@pytest.mark.parametrize("col", TERMS_COLS)
def test_columns_and_orders_against_model(ctx, fx, col):
    """Every terms column kind, every order, segment_size below and above the entry count, 1-4 metric columns (k_str's are a
    count-only and an empty column)."""
    acc = 0
    c = TERMS_COLS.index(col)
    for j, order in enumerate(ORDERS[c % 2::2][:5] + ORDERS[4 + c::len(TERMS_COLS)][:1]):
        qts = shapes(fx)[(c + j) % 5::5]
        for ss in (3, 1000):
            a, _ = check([ctx], fx, qts, {"field": col, "size": 4, "segment_size": ss, "order": order}, ("ints", "sparse", "k_str"))
            acc += a
    assert acc > 0


@pytest.mark.parametrize("order", [{"tv_avg": "desc"}, {"tv_avg": "asc"}, {"zeros_min": "asc"}, {"zeros_stats.max": "desc"},
                                   {"tv_stats.count": "desc"}, {"sparse_avg": "desc"}, {"sparse_stats.min": "asc"}])
def test_ties_zeros_and_keys_without_values(ctx, fx, order):
    """Order values equal across keys at the cut (lowest keys kept, the scalars in that order), -0.0 against +0.0 (equal in the cut,
    ordered in the final result), keys with docs but no value (0.0 in the cut, f64::MIN in the final order); segment_size below, at
    and above the 50 keys."""
    qts = [fx.query(TQ_OP_TERM, [ALL], 10), fx.query(TQ_OP_OR, [1, 2, 3], 10)]
    for ss, size in ((7, 5), (13, 60), (49, 5), (50, 5), (51, 60)):
        check([ctx], fx, qts, {"field": "k_ties", "size": size, "segment_size": ss, "order": order}, ("tv", "zeros", "sparse"))


def test_guard_refusals(ctx, fx):
    """A decimal column's sums are refused per bucket, answered elsewhere; an order by its avg, or by any metric of a column that
    saw a NaN, is refused as a whole."""
    qts = shapes(fx)[:8]
    acc, ref = check([ctx], fx, qts, {"field": "k_str", "size": 5}, ("ints", "decimal", "ns"))
    assert acc > 0 and ref > 0
    for order in ({"decimal_avg": "desc"}, {"nan_inf_max": "desc"}, {"nan_inf_stats.count": "asc"}):
        _, ref = check([ctx], fx, qts[:4], {"field": "k_i64", "size": 5, "segment_size": 5, "order": order}, ("ints", "decimal", "nan_inf"))
        assert ref > 0, order


@pytest.mark.parametrize("fkind", FILTER_KINDS)
def test_filters(ctx, fx, fkind):
    j = FILTER_KINDS.index(fkind)
    qts = [(dict(q, filter=200 + j), t) for q, t in shapes(fx)[:8]]
    check([ctx], fx, qts, {"field": "k_r10k", "size": 5, "segment_size": 20, "order": {"ints_avg": "desc"}}, ("ints", "dyadic"),
          masks=fx.filters[fkind])
    check([ctx], fx, qts[:4], {"field": "k_str", "size": 3, "missing": "NA"}, ("flag",), masks=fx.filters[fkind], count_hits=False)


@pytest.mark.parametrize("missing", [7, -3.5])
def test_missing_on_both_sides(ctx, fx, missing):
    """`missing` on the terms (str: the segment's largest image + 1; numeric: merged with an equal value or one more entry) and
    on the metrics."""
    for terms in ({"field": "partial", "missing": 5, "segment_size": 4}, {"field": "partial", "missing": 1 << 40, "order": {"ints_sum": "desc"}},
                  {"field": "k_str", "missing": "NA", "segment_size": 3, "order": {"partial_avg": "asc"}},
                  {"field": "clustered", "missing": 0, "order": {"_key": "asc"}}):
        check([ctx], fx, shapes(fx)[:10], terms, ("partial", "ints", "us_half"), missing=missing)


def test_split_segments_over_two_contexts(fx):
    """The big segment's halves in two contexts (doc ranges) come back uncut and are cut once by terms_metrics; equal to one
    context over all of it and to the model."""
    big = fx.osegs[0]
    half = (big.max_doc // 8192 // 2) * 8192 + 100
    cols = ("ints", "dyadic", "sparse")
    ctxs = []
    try:
        for lo, hi in ((0, half), (half, big.max_doc), (0, big.max_doc)):
            c = T.Context(0)
            big.register(c)
            c.segment_set_doc_range(big.segment_ord, 0, lo, hi)
            for k in cols + ("k_r10k", "k_ties"):
                v, p = fx.columns[k][0]
                c.sort_column_register(fx.mcol[k], big.segment_ord, v, None if p is None else packed(p))
            ctxs.append(c)
        for terms in ({"field": "k_r10k", "size": 4, "segment_size": 30, "order": {"ints_avg": "desc"}},
                      {"field": "k_ties", "size": 5, "segment_size": 7, "order": {"_count": "asc"}},
                      {"field": "k_ties", "size": 5, "segment_size": 9, "order": {"sparse_stats.min": "asc"}}):
            for q, t in shapes(fx)[:6]:
                q = dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] == big.segment_ord])
                r = TMx.parse_request({"t": {"terms": terms, "aggs": sub_aggs(cols)}})
                fields = fields_of(fx, cols + (terms["field"],))
                split = TMx.run(ctxs[:2], QueryBatch([q]), [r], fields)[0]
                one = TMx.run(ctxs[2:], QueryBatch([q]), [r], fields)[0]
                want = Model(fx, r, TMx.plan(r, fields))((q, t), segs={0})[3]
                for got in (split, one):
                    refused = got.refused if isinstance(got, TMx.TermsMetricsRefused) else {}
                    got = got.answered if isinstance(got, TMx.TermsMetricsRefused) else got
                    gb, wb = got["t"]["buckets"], want["t"]["buckets"]
                    assert [(b["key"], b["doc_count"]) for b in gb] == [(b["key"], b["doc_count"]) for b in wb], terms
                    assert got["t"]["sum_other_doc_count"] == want["t"]["sum_other_doc_count"], terms
                    for g, w in zip(gb, wb):
                        assert all(same(g[n], w[n]) for n in g if n not in refused), terms
    finally:
        for c in ctxs:
            c.close()


def device_args(fx, qts, terms, cols, order=None):
    r = TMx.parse_request({"t": {"terms": terms, "aggs": sub_aggs(cols)}})
    p = TMx.plan(r, fields_of(fx, tuple(cols) + (terms["field"],)))
    return (QueryBatch([qt[0] for qt in qts]), [p.tspec] * len(qts), [p.mplan.columns] * len(qts), [p.order] * len(qts))


def same_out(a, b):
    for q in range(len(a[4])):
        n = int(a[4][q])
        assert int(b[4][q]) == n
        for x, y in zip(a[:3], b[:3]):
            assert np.array_equal(x[q, :n], y[q, :n])
        for f in ("count", "n_nan", "n_inf", "min_image", "max_image", "quantum_exp", "sum", "magnitude"):
            assert np.array_equal(a[3][q, :n][f], b[3][q, :n][f]), f
    for x, y in zip(a[5:7], b[5:7]):
        assert np.array_equal(x, y)
    assert a[7].tobytes() == b[7].tobytes()


def test_span_budget_waves_stride_and_errors(fx):
    qt = fx.query(TQ_OP_TERM, [ALL], 10)
    qts = shapes(fx)[:12]
    c = fx.register(T.Context(0))
    try:
        check([c], fx, [qt], {"field": "span20", "size": 3, "order": {"ints_avg": "desc"}}, ("ints",))  # 2^20 keys: accepted
        qb, ts, ms, os_ = device_args(fx, [qt], {"field": "span20p1", "order": {"ints_avg": "desc"}}, ("ints",))
        assert code(lambda: c.terms_metrics_batch(qb, ts, ms, os_)) == -4
        # waves and the stride retry give the same rows, parts, scalars and order parts
        for terms in ({"field": "k_r10k", "size": 3, "segment_size": 10, "order": {"ints_avg": "desc"}},
                      {"field": "k_str", "size": 3, "missing": "NA", "order": {"_count": "desc"}}):
            args = device_args(fx, qts, terms, ("ints", "sparse"))
            want = c.terms_metrics_batch(*args, count_hits=True)
            same_out(want, c.terms_metrics_batch(*args, count_hits=True, stride=1))
            for env, budget in (("TQ_TERMS_COUNTER_BUDGET", "50"), ("TQ_TERMS_METRICS_BUDGET", "200")):
                os.environ[env] = budget  # every query alone in its wave
                try:
                    small = fx.register(T.Context(0))
                finally:
                    del os.environ[env]
                try:
                    got = small.terms_metrics_batch(*args, count_hits=True)
                    same_out(want, got)
                    assert np.array_equal(got[8], want[8]) and small.stats()["terms_metrics_waves"] > 1
                finally:
                    small.close()
        # a (query, segment) whose parts alone exceed the budget
        os.environ["TQ_TERMS_METRICS_BUDGET"] = "16"
        try:
            tiny = fx.register(T.Context(0))
        finally:
            del os.environ["TQ_TERMS_METRICS_BUDGET"]
        try:
            qb, ts, ms, os_ = device_args(fx, [qt], {"field": "k_ties", "segment_size": 5}, ("ints",))
            assert code(lambda: tiny.terms_metrics_batch(qb, ts, ms, os_)) == -4
        finally:
            tiny.close()
        # errors
        qb, ts, ms, os_ = device_args(fx, [qt], {"field": "k_ties", "order": {"ints_avg": "desc"}}, ("ints",))
        assert code(lambda: c.terms_metrics_batch(qb, ts, ms, None)) == -1
        assert code(lambda: c.terms_metrics_batch(qb, ts, ms, [(4, TQ_TERMS_ORDER_AVG)])) == -1
        assert code(lambda: c.terms_metrics_batch(qb, ts, ms, [(0, 5)])) == -1
        assert code(lambda: c.terms_metrics_batch(qb, [ts[0][:1] + (3,) + ts[0][2:]], ms, os_)) == -1
        assert code(lambda: c.terms_metrics_batch(qb, ts, [[(fx.mcol["ints"], 9)]], os_)) == -1
        assert code(lambda: c.terms_metrics_batch(qb, [(999,) + ts[0][1:]], ms, os_)) == -3
        assert code(lambda: c.terms_metrics_batch(qb, ts, [[(999, TQ_FAST_U64)]], os_)) == -3
        assert code(lambda: c.terms_batch(qb, [ts[0]])) == -1  # TQ_TERMS_BY_METRIC is not a target of tq_terms_batch
        phrase = dict(qt[0], op=3, term_pos=[(0, 0)] * len(qt[0]["term_segs"]), term_offset=[0])
        assert code(lambda: c.terms_metrics_batch(QueryBatch([phrase]), ts, ms, os_)) == -4
        empty = c.terms_metrics_batch(QueryBatch([]), [], [], count_hits=True)
        assert [x.shape[0] for x in empty] == [0] * 9
    finally:
        c.close()


def test_one_run_per_call_once_the_width_is_known_and_stats(fx):
    qts = shapes(fx)[:8]
    args = device_args(fx, qts, {"field": "k_r10k", "segment_size": 3000, "order": {"_key": "asc"}}, ("ints",))
    c = fx.register(T.Context(0))
    try:
        runs = lambda: c.stats()["units_terms_metrics"]  # noqa: E731
        u0 = runs()
        first = c.terms_metrics_batch(*args)
        u1 = runs()
        second = c.terms_metrics_batch(*args)
        u2 = runs()
        assert int(first[4].max()) > 1024 and u1 - u0 == 2 * (u2 - u1) > 0
        same_out(first, second)
        check([c], fx, qts[:4], {"field": "clustered", "size": 3}, ("ints", "const"))
        st = c.stats()
        assert 0 < st["terms_metrics_tiles_one_key"] <= st["terms_metrics_tiles_seen"] and st["terms_metrics_ms"] > 0
    finally:
        c.close()


def test_by_metric_rows_keep_terms_batch_entries_when_uncut(ctx, fx):
    """segment_size above every segment's entry count: a metric order keeps every entry, exactly tq_terms_batch's rows."""
    qts = shapes(fx)[:10]
    qb, ts, ms, os_ = device_args(fx, qts, {"field": "k_str", "segment_size": 100, "order": {"ints_avg": "asc"}}, ("ints",))
    got = ctx.terms_metrics_batch(qb, ts, ms, os_)
    ref = ctx.terms_batch(qb, [(t[0], TQ_TERMS_BY_COUNT) + tuple(t[2:]) for t in ts])
    for q in range(len(qts)):
        n = int(ref[3][q])
        assert int(got[4][q]) == n and all(np.array_equal(a[q, :n], b[q, :n]) for a, b in zip(got[:3], ref[:3]))
        assert (int(got[5][q]), int(got[6][q])) == (0, 0) and ts[q][1] == TQ_TERMS_BY_METRIC
