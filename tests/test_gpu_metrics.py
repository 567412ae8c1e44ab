"""Metric aggregations on the device (tq_metrics_batch: k_metrics) against tests/metrics_model.py (the reference's Kahan collection in
doc order, merge_fruits in segment_ord order, into_final_metric_result) over the docs tests/score_model.py matches (and-ed with the
alive bits, the filter and the doc range, as Count counts them).  Every accepted sum and average must be bit-equal to the model's;
count, min and max must be exact always; every column built to fail the guard must be refused.  The fixture is
test_gpu_sort_field's (three segments, deletes in two, an `edge` term on every 8192-doc tile and unit edge, an `all` term) with
metric columns: small integers, u64 multiples of 2^40 near 2^63, i64 of mixed sign, bool, dyadic and decimal f64, f64 with NaN and
+-inf (one segment all NaN), a constant and a clustered column (one-value tiles), columns present in some segments only and
nanosecond dates."""
import math
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200 import metrics as Mx  # noqa: E402
from tantivy_b200._abi import (TQ_FAST_BOOL, TQ_FAST_DATE, TQ_FAST_F64, TQ_FAST_I64, TQ_FAST_U64, TQ_METRIC_COUNT_ONLY, TQ_METRIC_EMPTY, TQ_METRIC_MISSING,  # noqa: E402
                               TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM, QueryBatch)
from tests import metrics_model as MM  # noqa: E402
from tests.helpers import OracleSegment, make_query  # noqa: E402
from tests.test_gpu_parity import fresh_ord  # noqa: E402
from tests.test_gpu_sort_field import ALL, FILTER_KINDS, Fixture, packed, shapes  # noqa: E402
from tests.test_metrics_host import FIXTURES, check_fixture, fixture_plan  # noqa: E402

TYPES = ("stats", "sum", "avg", "min", "max", "value_count")
# columns whose sums the guard must refuse whenever a query collects enough of them
MUST_REFUSE = {"decimal": 50, "ns": 20}


class MetricsFixture(Fixture):
    def __init__(self):
        super().__init__()
        rng = np.random.default_rng(0x3E7)
        self.kind = {"uniform": "u64", "monotone": "u64", "equal": "u64", "few": "u64", "half": "u64", "none": "u64", "i64": "i64", "f64": "f64"}
        for i, s in enumerate(self.osegs):
            n = s.max_doc
            doc = np.arange(n)
            nan_inf = rng.choice(np.array([np.nan, np.inf, -np.inf, 1.0, -2.0, 0.5]), size=n) if i != 1 else np.full(n, np.nan)
            extra = {
                "ints": ("u64", rng.integers(0, 1000, size=n).astype(np.uint64), None),
                "big": ("u64", ((np.uint64(1 << 23) - rng.integers(0, 1 << 10, size=n).astype(np.uint64)) << np.uint64(40)), None),
                "mixed": ("i64", T.fast_value_to_u64(rng.integers(-10**6, 10**6, size=n), "i64"), None),
                "flag": ("bool", T.fast_value_to_u64(rng.random(n) < 0.3, "bool"), rng.random(n) < 0.9),
                "dyadic": ("f64", T.fast_value_to_u64(rng.integers(-2**20, 2**20, size=n) * 2.0**-8, "f64"), rng.random(n) < 0.8),
                "decimal": ("f64", T.fast_value_to_u64(np.round(rng.uniform(-100, 100, size=n), 3), "f64"), None),
                "nan_inf": ("f64", T.fast_value_to_u64(nan_inf, "f64"), None),
                "const": ("i64", T.fast_value_to_u64(np.full(n, -42), "i64"), None),
                "clustered": ("u64", (doc // 9000).astype(np.uint64), rng.random(n) < 0.97),
                "partial": ("u64", (doc % 30).astype(np.uint64), (rng.random(n) < 0.7) if i != 1 else np.zeros(n, bool)),
                "ns": ("date", T.fast_value_to_u64(np.int64(1_700_000_000) * 10**9 + rng.integers(0, 10**12, size=n), "date"), rng.random(n) < 0.95),
                "us_half": ("date", T.fast_value_to_u64(np.int64(1_700_000_000) * 10**6 + rng.integers(0, 10**6, size=n) * 1000, "date"),
                            rng.random(n) < 0.5),
            }
            for k, (kind, v, p) in extra.items():
                self.columns.setdefault(k, []).append((v, p))
                self.kind[k] = kind
        self.mcol = {k: 500 + i for i, k in enumerate(self.columns)}

    def register(self, ctx, filters=()):
        super().register(ctx, kinds=(), filters=filters)
        for k in self.columns:
            for i, s in enumerate(self.osegs):
                v, p = self.columns[k][i]
                ctx.sort_column_register(self.mcol[k], s.segment_ord, v, None if p is None else packed(p))
        return ctx

    def values(self, qt, col, i, missing=None, masks=None, typ="stats"):
        """The values segment i collects for a metric of type typ on the column, in doc order, by the model's column rules
        (metrics_model.doc_values): 0.0 per value on a bool column under value_count, none on tantivy's empty column otherwise."""
        sel = self.has(i, qt) & self.alive[i]
        if masks is not None:
            sel = sel & masks[i]
        v, p = self.columns[col][i]
        kind = self.kind[col]
        ctype = MM.column_type(typ, kind)
        pres = np.ones(len(v), bool) if p is None else p
        if ctype == "empty":
            ctype, pres = "u64", np.zeros(len(v), bool)
        f = to_f64(v, kind) if ctype in MM.NUMERIC else np.zeros(len(v))
        mv = None if missing is None else MM.missing_value(float(missing), ctype)
        if mv is not None:
            f = np.where(pres, f, mv if ctype in MM.NUMERIC else 0.0)
            return f[sel].tolist()
        return f[sel & pres].tolist()

    def stats(self, qt, col, missing=None, masks=None, typ="stats"):
        order = sorted(range(len(self.osegs)), key=lambda i: self.osegs[i].segment_ord)
        return MM.merged([MM.segment_stats(self.values(qt, col, i, missing, masks, typ)) for i in order])

    def model(self, qt, col, typ, missing=None, masks=None):
        return MM.final(self.stats(qt, col, missing, masks, typ), typ)


def to_f64(images, kind):
    images = np.asarray(images, np.uint64)
    if kind == "f64":
        high = np.uint64(1 << 63)
        bits = np.where(images >= high, images ^ high, ~images)
        return bits.view(np.float64)
    if kind in ("i64", "date"):
        return (images ^ np.uint64(1 << 63)).view(np.int64).astype(np.float64)
    return images.astype(np.float64)


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, float) and isinstance(b, float):
        return struct.pack("<d", a) == struct.pack("<d", b)
    return a == b


def request(fx, cols, missing=None):
    """One aggregation of every type on each column (field = the column's name), and the MetricField map."""
    aggs, fields = {}, {}
    for c in cols:
        body = {"field": c} if missing is None else {"field": c, "missing": missing}
        for typ in TYPES:
            aggs[f"{c}.{typ}"] = {typ: body}
        fields[c] = Mx.MetricField(fx.mcol[c], fx.kind[c])
    return Mx.parse_request(aggs), fields


def check(ctx, fx, qts, cols, missing=None, masks=None, count_hits=True):
    """Runs qts with one request over cols and compares every aggregation with the model; returns (accepted, refused) sums."""
    aggs, fields = request(fx, cols, missing)
    qb = QueryBatch([qt[0] for qt in qts])
    res, hits = Mx.run([ctx], qb, [aggs] * len(qts), fields, count_hits=True)
    assert np.array_equal(hits, ctx.count_batch(qb))
    tally = [0, 0]
    for qt, r in zip(qts, res):
        answered, refused = (r.answered, r.refused) if isinstance(r, Mx.MetricsRefused) else (r, {})
        st = {}
        for a in aggs:
            c, typ = a.name.split(".")
            key = (c, MM.column_type(typ, fx.kind[c]))
            if key not in st:
                st[key] = fx.stats(qt, c, missing, masks, typ)
            want = MM.final(st[key], typ)
            if a.name in refused:
                assert typ in Mx.SUM_BEARING
                tally[1] += 1
                continue
            tally[0] += typ in Mx.SUM_BEARING
            assert same(answered[a.name], want), (a.name, qt[1], answered[a.name], want)
            if c in MUST_REFUSE and typ in Mx.SUM_BEARING:
                n = sum(len(fx.values(qt, c, i, missing, masks, typ)) for i in range(len(fx.osegs)))
                assert n < MUST_REFUSE[c], f"{a.name} on {n} values should have been refused"
    return tally


@pytest.fixture(scope="module")
def fx():
    return MetricsFixture()


@pytest.fixture(scope="module")
def ctx(fx):
    c = fx.register(T.Context(0), filters=FILTER_KINDS)
    yield c
    c.close()


# (a bool field takes two spec columns: count-only for value_count, tantivy's empty column for the other metrics)
GROUPS = [("ints", "big", "flag"), ("dyadic", "decimal", "nan_inf", "const"), ("clustered", "partial", "ns", "us_half"),
          ("uniform", "f64", "i64", "half"), ("none", "equal", "mixed")]


@pytest.mark.parametrize("cols", GROUPS, ids=["+".join(g) for g in GROUPS])
def test_shapes_against_model(ctx, fx, cols):
    """Every query shape of the sort fixture (term, AND, OR, mixed boolean: both kernel instances), four columns per spec."""
    acc, ref = check(ctx, fx, shapes(fx), cols)
    assert acc + ref > 0


def test_guard_accepts_integers_and_refuses_decimals(ctx, fx):
    acc, ref = check(ctx, fx, shapes(fx)[:12], ("ints", "big", "decimal", "ns"))
    assert acc > 0 and ref > 0


@pytest.mark.parametrize("fkind", FILTER_KINDS)
def test_filters(ctx, fx, fkind):
    j = FILTER_KINDS.index(fkind)
    qts = [(dict(q, filter=200 + j), t) for q, t in shapes(fx)[:10]]
    check(ctx, fx, qts, ("ints", "dyadic", "flag"), masks=fx.filters[fkind])


@pytest.mark.parametrize("missing", [7, -3.5, 1e300])
def test_missing_on_each_kind(ctx, fx, missing):
    """`missing` on u64 (values in two segments of three), i64, f64, bool and date columns."""
    check(ctx, fx, shapes(fx)[:14], ("partial", "mixed", "flag"), missing=missing)
    check(ctx, fx, shapes(fx)[:14], ("us_half", "half", "dyadic"), missing=missing)


def test_same_column_twice_and_one_to_four_columns(ctx, fx):
    qts = shapes(fx)[:6]
    qb = QueryBatch([q for q, _ in qts])
    cols = [(fx.mcol["ints"], TQ_FAST_U64), (fx.mcol["ints"], TQ_FAST_U64, TQ_METRIC_MISSING, 5), (fx.mcol["ints"], TQ_FAST_U64),
            (fx.mcol["flag"], TQ_FAST_BOOL, TQ_METRIC_COUNT_ONLY)]
    full = ctx.metrics_batch(qb, [cols] * len(qts))
    assert np.array_equal(full[:, 0], full[:, 2]) and np.array_equal(full[:, 0], full[:, 1])  # (ints has a value everywhere)
    for n in (1, 2, 3):
        parts, hits = ctx.metrics_batch(qb, [cols[:n]] * len(qts), count_hits=True)
        assert np.array_equal(parts[:, :n], full[:, :n]) and np.array_equal(hits, ctx.count_batch(qb))
        assert (parts[:, n:]["count"] == 0).all() and (parts[:, n:]["quantum_exp"] == 2**31 - 1).all()


def test_one_value_tiles_are_counted(fx):
    c = fx.register(T.Context(0))
    try:
        check(c, fx, shapes(fx)[:8], ("const", "clustered"))
        st = c.stats()
        assert st["metrics_tiles_one_value"] > 0 and st["metrics_tiles_seen"] >= st["metrics_tiles_one_value"]
        assert st["units_metrics"] > 0 and st["metrics_ms"] > 0
    finally:
        c.close()


def test_split_segment_over_two_contexts(fx):
    """The big segment's halves in two contexts (doc ranges): merged parts equal one context's over the whole segment."""
    big = fx.osegs[0]
    half = (big.max_doc // 8192 // 2) * 8192 + 100
    ctxs = []
    cols = ("ints", "dyadic", "partial", "nan_inf")
    try:
        for lo, hi in ((0, half), (half, big.max_doc), (0, big.max_doc)):
            c = T.Context(0)
            big.register(c)
            c.segment_set_doc_range(big.segment_ord, 0, lo, hi)
            for k in cols:
                v, p = fx.columns[k][0]
                c.sort_column_register(fx.mcol[k], big.segment_ord, v, None if p is None else packed(p))
            ctxs.append(c)
        aggs, fields = request(fx, cols)
        for q, t in shapes(fx)[:10]:
            q = dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] == big.segment_ord])
            qb = QueryBatch([q])
            spec = [Mx.plan(aggs, fields).columns]
            a, b, whole = (c.metrics_batch(qb, spec)[0] for c in ctxs)
            m = Mx.merge([a, b])
            for f in ("count", "n_nan", "n_inf", "min_image", "max_image", "quantum_exp"):
                assert np.array_equal(m[f], whole[f]), f
            split = Mx.run(ctxs[:2], qb, [aggs], fields)[0]
            one = Mx.run(ctxs[2:], qb, [aggs], fields)[0]
            if isinstance(one, Mx.MetricsRefused):
                assert isinstance(split, Mx.MetricsRefused) and split.refused.keys() == one.refused.keys()
                split, one = split.answered, one.answered
            assert same(split, one)
            for name, r in one.items():
                col, typ = name.split(".")
                vals = fx.values((q, t), col, 0, typ=typ)
                assert same(r, MM.final(MM.segment_stats(vals), typ)), name
    finally:
        for c in ctxs:
            c.close()


def test_guard_at_the_bound():
    """One query's |v| sum is exactly 2^53 with Q = 0 (refused), another's one quantum below it (accepted and exact)."""
    n = 10_000
    a = np.array([0, 1, 2], np.uint32)  # 2^52 + (2^52 - 1) + 1 = 2^53
    b = np.array([0, 1], np.uint32)     # 2^53 - 1
    alld = np.arange(n, dtype=np.uint32)
    lists = [(a, np.ones(3, np.uint32)), (b, np.ones(2, np.uint32)), (alld, np.ones(n, np.uint32))]
    seg = OracleSegment(lists, None, segment_ord=fresh_ord(), writer_cls=T.FieldWriter, max_doc=n)
    vals = np.zeros(n, np.uint64)
    vals[:3] = [2**52, 2**52 - 1, 1]
    c = T.Context(0)
    try:
        seg.register(c)
        c.sort_column_register(1, seg.segment_ord, vals)
        aggs = Mx.parse_request({"s": {"sum": {"field": "v"}}, "x": {"max": {"field": "v"}}})
        fields = {"v": Mx.MetricField(1, "u64")}
        qb = QueryBatch([make_query(TQ_OP_TERM, [seg], [0], 10), make_query(TQ_OP_TERM, [seg], [1], 10)])
        at, below = Mx.run([c], qb, [aggs, aggs], fields)
        assert isinstance(at, Mx.MetricsRefused) and set(at.refused) == {"s"} and at.answered == {"x": {"value": float(2**52)}}
        assert below == {"s": {"value": float(2**53 - 1)}, "x": {"value": float(2**52)}}
        assert below["s"]["value"] == MM.segment_stats([2.0**52, 2.0**52 - 1]).sum
    finally:
        c.close()


def test_error_codes(fx):
    def code(fn):
        with pytest.raises(T.TqError) as e:
            fn()
        return int(str(e.value).split("error ")[1].split(":")[0])

    c = fx.register(T.Context(0))
    try:
        qt = fx.query(TQ_OP_TERM, [ALL], 10)
        qb = QueryBatch([qt[0]])
        good = (fx.mcol["ints"], TQ_FAST_U64)
        assert code(lambda: c.metrics_batch(qb, [[(999, TQ_FAST_U64)]])) == -3
        for bad in ([], [good] * 5, [(fx.mcol["ints"], 5)], [(fx.mcol["ints"], TQ_FAST_U64, 8, 0)],
                    [(0, TQ_FAST_U64, TQ_METRIC_EMPTY | TQ_METRIC_COUNT_ONLY, 0)], [(0, TQ_FAST_F64, TQ_METRIC_EMPTY, 0)]):
            assert code(lambda: c.metrics_batch(qb, [bad])) == -1
        # an empty column names no registered column: with `missing` every collected doc collects it
        parts = c.metrics_batch(qb, [[(999, TQ_FAST_U64, TQ_METRIC_EMPTY), (999, TQ_FAST_U64, TQ_METRIC_EMPTY | TQ_METRIC_MISSING, 7)]])
        n = int(c.count_batch(qb)[0])
        assert int(parts[0, 0]["count"]) == 0 and int(parts[0, 0]["quantum_exp"]) == 2**31 - 1
        assert (int(parts[0, 1]["count"]), int(parts[0, 1]["min_image"]), int(parts[0, 1]["max_image"]), float(parts[0, 1]["sum"])) == (n, 7, 7, 7.0 * n)
        phrase = dict(qt[0], op=3, term_pos=[(0, 0)] * len(qt[0]["term_segs"]), term_offset=[0])
        assert code(lambda: c.metrics_batch(QueryBatch([phrase]), [[good]])) == -4
    finally:
        c.close()


def test_segment_of_2_to_the_31_docs():
    """One segment of 2^31 - 2 docs; values in its top 300 000 docs and at max_doc - 1 (10 % without one, `missing` on them)."""
    rng = np.random.default_rng(0x31)
    max_doc = 2**31 - 2
    top = max_doc - 300_000
    lists = []
    for p in (0.2, 0.05):
        d = np.union1d(top + np.nonzero(rng.random(max_doc - top) < p)[0], [max_doc - 1]).astype(np.uint32)
        lists.append((d, np.ones(len(d), np.uint32)))
    seg = OracleSegment(lists, None, segment_ord=fresh_ord(), writer_cls=T.FieldWriter, max_doc=max_doc)
    top_values = rng.integers(0, 10**6, size=max_doc - top).astype(np.uint64)
    values = np.zeros(max_doc, np.uint64)
    values[top:] = top_values
    has = rng.random(max_doc - top) < 0.9
    has[-1] = True
    present = np.zeros((max_doc + 7) // 8, np.uint8)
    sel = top + np.nonzero(has)[0]
    np.bitwise_or.at(present, sel >> 3, (1 << (sel & 7)).astype(np.uint8))
    c = T.Context(0)
    try:
        seg.register(c)
        c.sort_column_register(9, seg.segment_ord, values, present)
        del values
        qs = [(make_query(TQ_OP_TERM, [seg], [0], 10), lists[0][0]), (make_query(TQ_OP_OR, [seg], [0, 1], 10), np.union1d(lists[0][0], lists[1][0])),
              (make_query(TQ_OP_AND, [seg], [0, 1], 10), np.intersect1d(lists[0][0], lists[1][0]))]
        aggs = Mx.parse_request({"s": {"stats": {"field": "v", "missing": 3}}, "c": {"value_count": {"field": "v"}}})
        qb = QueryBatch([q for q, _ in qs])
        res, hits = Mx.run([c], qb, [aggs] * 3, {"v": Mx.MetricField(9, "u64")}, count_hits=True)
        assert np.array_equal(hits, c.count_batch(qb))
        for r, (_, docs) in zip(res, qs):
            i = docs.astype(np.int64) - top
            with_missing = np.where(has[i], top_values[i], 3).astype(np.float64)
            assert same(r["s"], MM.final(MM.segment_stats(with_missing.tolist()), "stats"))
            assert r["c"] == {"value": float(has[i].sum())}
    finally:
        c.close()


def test_counts_min_max_exact_when_refused(ctx, fx):
    """A refused sum still leaves count, min and max exact (NaN and +-inf columns, one segment all NaN)."""
    qts = shapes(fx)[:10]
    aggs = Mx.parse_request({"n": {"min": {"field": "nan_inf"}}, "x": {"max": {"field": "nan_inf"}}, "c": {"value_count": {"field": "nan_inf"}},
                             "s": {"stats": {"field": "nan_inf"}}})
    fields = {"nan_inf": Mx.MetricField(fx.mcol["nan_inf"], "f64")}
    res = Mx.run([ctx], QueryBatch([q for q, _ in qts]), [aggs] * len(qts), fields)
    for qt, r in zip(qts, res):
        vals = sum((fx.values(qt, "nan_inf", i) for i in range(3)), [])
        answered = r.answered if isinstance(r, Mx.MetricsRefused) else r
        if any(math.isnan(v) or math.isinf(v) for v in vals):
            assert isinstance(r, Mx.MetricsRefused) and "s" in r.refused
        for name in ("n", "x", "c"):
            assert same(answered[name], fx.model(qt, "nan_inf", {"n": "min", "x": "max", "c": "value_count"}[name])), name


def fixture_column(kind, docs, field):
    """(u64 images, present mask) of one fixture segment's column (a str column's images: ordinals of its sorted terms)."""
    present = np.array([field in d for d in docs], bool)
    vals = [d[field] for d in docs if field in d]
    if kind == "str":
        terms = sorted(set(vals))
        have = np.array([terms.index(v) for v in vals], np.uint64)
    elif kind in ("u64", "bool"):
        have = np.array(vals, np.uint64)
    else:
        have = T.fast_value_to_u64(np.array(vals, np.float64 if kind == "f64" else np.int64), kind)
    images = np.zeros(len(docs), np.uint64)
    images[present] = np.asarray(have, np.uint64)
    return images, present


@pytest.mark.parametrize("case", [c for c in FIXTURES if "refused" not in c], ids=[c["name"] for c in FIXTURES if "refused" not in c])
def test_reference_fixtures_on_device(case):
    """The reference's metric vectors end to end: every segment a real segment whose term 0 lists the collected docs, every field a
    registered column (present bits for the docs without a value), the parts finalised by tantivy_b200.metrics."""
    p, fields = fixture_plan(case)
    c = T.Context(0)
    try:
        segs = []
        for docs in case["segments"]:
            n = len(docs)
            hit = np.array([i for i, d in enumerate(docs) if d["hit"]] or [0], np.uint32)
            s = OracleSegment([(hit, np.ones(len(hit), np.uint32)), (np.arange(n, dtype=np.uint32), np.ones(n, np.uint32))], [1] * n,
                              segment_ord=fresh_ord(), writer_cls=T.FieldWriter)
            if not any(d["hit"] for d in docs):
                s.terms[0] = (0, 0, 0)
            s.register(c)
            for name, f in fields.items():
                images, present = fixture_column(case["fields"][name], docs, name)
                c.sort_column_register(f.column_id, s.segment_ord, images, None if present.all() else packed(present))
            segs.append(s)
        q = make_query(TQ_OP_TERM, segs, [0], 10) if segs else dict(op=TQ_OP_TERM, k=10, weights=[1.0], avg_fieldnorm=[1.0], term_segs=[])
        res, hits = Mx.run([c], QueryBatch([q]), [p.aggs], fields, count_hits=True)
        assert int(hits[0]) == sum(d["hit"] for docs in case["segments"] for d in docs)
        check_fixture(case, res[0])
    finally:
        c.close()
