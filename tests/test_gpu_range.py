"""Range aggregations on the device (tq_range_batch: k_range, k_range_metrics) against tests/range_model.py (per segment the matching
docs in doc order, bucketed by the binary search over the extended starts, Kahan collection per (bucket, metric), merged by key
string in segment_ord order) over the docs tests/score_model.py matches (and-ed with the alive bits, the filter and the doc range, as
Count counts them).  Keys, from / to, doc counts, count, min and max must be exact; every accepted sum and average bit-equal to the
model's.  The fixture is test_gpu_hist_metrics' (three segments with deletes, the `edge` term on every tile and unit edge, the
metric columns, the nanosecond timestamps) with the sort columns' u64 (images 0 and u64::MAX included), i64 and f64 (-0.0, +0.0,
+-inf) columns and the NaN / +-inf f64 column."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200 import metrics as Mx  # noqa: E402
from tantivy_b200 import ranges as R  # noqa: E402
from tantivy_b200._abi import TQ_FAST_U64, TQ_METRIC_COUNT_ONLY, TQ_OP_PHRASE, TQ_OP_TERM, QueryBatch  # noqa: E402
from tests import metrics_model as MM  # noqa: E402
from tests import range_model as RM  # noqa: E402
from tests.test_gpu_hist_metrics import HOUR, HistMetricsFixture, fields_of, metric_values, sub_aggs  # noqa: E402
from tests.test_gpu_metrics import same  # noqa: E402
from tests.test_gpu_sort_field import FILTER_KINDS, packed, shapes  # noqa: E402
from tests.helpers import OracleSegment, make_query  # noqa: E402
from tests.test_gpu_parity import fresh_ord  # noqa: E402
from tests.test_hist_metrics_host import same_tree  # noqa: E402
from tests.test_range_host import SEARCHES, check_asserts, collected, fixture_plan  # noqa: E402

T0 = (1_700_000_000 - 1_700_000_000 % 3600) * 10**9  # the fixture's first timestamp hour
B57 = float(2**57)


def ranges_of(bounds, keys=None):
    """Contiguous ranges between consecutive bounds (None: open)."""
    return [dict(({"from": a} if a is not None else {}), **({"to": b} if b is not None else {}), **({"key": keys[i]} if keys else {}))
            for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:]))]


RANGES = {
    "ts_3": {"field": "ts", "ranges": ranges_of([None, T0 + 10 * HOUR, T0 + 100 * HOUR, None])},
    "ts_24": {"field": "ts", "ranges": ranges_of([T0 + 40 * HOUR + i * 30 * HOUR for i in range(25)])},
    "monotone_5": {"field": "monotone", "ranges": ranges_of([1.6e12 + i * 3e7 for i in range(6)], keys=list("abcde"))},
    "u64_1": {"field": "uniform", "ranges": [{}]},
    "u64_2": {"field": "uniform", "ranges": [{"to": 2.0**63}], "keyed": True},
    "u64_5": {"field": "uniform", "ranges": ranges_of([None, 2.0**61, 2.0**62, 2.0**63, 3 * 2.0**62, None])},
    "u64_127": {"field": "uniform", "ranges": ranges_of([None] + [i * B57 for i in range(1, 127)] + [None])},
    "u64_128": {"field": "uniform", "ranges": ranges_of([i * B57 for i in range(1, 128)] + [None])},
    "partial_edges": {"field": "partial", "ranges": ranges_of([0, 10, 20, 29])},
    "i64": {"field": "i64", "ranges": ranges_of([-50, -10, 0, 10, 49])},
    "f64_zeros": {"field": "f64", "ranges": [{"to": -0.0}, {"from": -0.0, "to": 0.0}, {"from": 0.0, "to": 2.25}, {"from": 3.0}]},
    "nan_inf": {"field": "nan_inf", "ranges": ranges_of([-1.0, 0.75, 1.0, None])},
}
GROUPS = [(), ("ints",), ("ints", "big"), ("dyadic", "decimal", "flag"), ("partial", "ns", "const", "clustered")]


@pytest.fixture(scope="module")
def fx():
    return HistMetricsFixture()


@pytest.fixture(scope="module")
def ctx(fx):
    c = fx.register(T.Context(0), filters=FILTER_KINDS)
    yield c
    c.close()


def request(rng, cols, missing=None, extra=None):
    agg = {"range": rng}
    if cols or extra:
        agg["aggs"] = dict(sub_aggs(cols, missing), **(extra or {}))
    return {"r": agg}


def model(fx, aggs, r, qt, masks=None, segs=None):
    """The model's result of the parsed request r (of the raw request aggs) for one query."""
    body = aggs["r"]["range"]
    field, kind = body["field"], fx.kind[body["field"]]
    ranges = [(x.get("key"), None if x.get("from") is None else float(x["from"]), None if x.get("to") is None else float(x["to"]))
              for x in body["ranges"]]
    starts = [s for _, s, _ in RM.extend_validate(ranges, kind)]
    seg_buckets, values = [], []
    metrics = [(a.name, a.type, (a.field, MM.column_type(a.type, fx.kind[a.field]), a.missing, a.type), a.none_if_no_match) for a in r.metrics]
    for i, _ in sorted(enumerate(fx.osegs), key=lambda x: x[1].segment_ord):
        if segs is not None and i not in segs:
            continue
        sel = fx.has(i, qt) & fx.alive[i]
        if masks is not None:
            sel = sel & masks[i]
        images, present = fx.columns[field][i]
        seg_buckets.append(RM.segment_buckets(images, present, sel, starts))
        values.append({k: metric_values(fx, i, k[0], k[3], k[2]) for _, _, k, _ in metrics})
    return RM.result("r", ranges, kind, bool(body.get("keyed")), seg_buckets, values, metrics)


def buckets_of(res):
    b = res["r"]["buckets"]
    return list(b.values()) if isinstance(b, dict) else b


def compare(got, want, r):
    """got (a result or RangeRefused) against the model; returns the refused names."""
    answered, refused = (got.answered, got.refused) if isinstance(got, R.RangeRefused) else (got, {})
    assert isinstance(answered["r"]["buckets"], dict) == isinstance(want["r"]["buckets"], dict)
    gb, wb = buckets_of(answered), buckets_of(want)
    assert [{k: v for k, v in b.items() if k not in {a.name for a in r.metrics}} for b in gb] == \
           [{k: v for k, v in b.items() if k not in {a.name for a in r.metrics}} for b in wb]
    for name in refused:
        assert name.split(".")[1] in Mx.SUM_BEARING, name
    for a in r.metrics:
        if a.name not in refused:
            for g, w in zip(gb, wb):
                assert same(g[a.name], w[a.name]), (a.name, g["key"], g[a.name], w[a.name])
    return refused


def check(ctxs, fx, qts, rng, cols, missing=None, masks=None, count_hits=True, extra=None):
    aggs = request(rng, cols, missing, extra)
    r = R.parse_request(aggs)
    names = set(cols) | {rng["field"]} | {v[next(iter(v))]["field"] for v in (extra or {}).values()}
    qb = QueryBatch([qt[0] for qt in qts])
    out = R.run(ctxs, qb, [r] * len(qts), fields_of(fx, names), count_hits=count_hits)
    res, hits = out if count_hits else (out, None)
    if count_hits:
        assert np.array_equal(hits, sum(c.count_batch(qb) for c in ctxs))
    tally = [0, 0]
    for qt, got in zip(qts, res):
        refused = compare(got, model(fx, aggs, r, qt, masks), r)
        tally[0] += sum(a.type in Mx.SUM_BEARING and a.name not in refused for a in r.metrics)
        tally[1] += len(refused)
    return tally


@pytest.mark.parametrize("rng", list(RANGES))
def test_ranges_against_model(ctx, fx, rng):
    """Every column kind and bucket count with 0-4 metric columns; every query shape without metrics and for the first group."""
    qts = shapes(fx)
    for j, cols in enumerate(GROUPS):
        check([ctx], fx, qts if j < 2 else qts[:: 2 + j], RANGES[rng], cols)


def test_doc_counts_alone_match_the_metrics_rows(ctx, fx):
    """k_range's counts equal k_range_metrics' for every shape; the rows hold every bucket, empty ones included."""
    qts = shapes(fx)
    qb = QueryBatch([qt[0] for qt in qts])
    p = R.plan(R.parse_request(request(RANGES["u64_128"], ("ints",))), fields_of(fx, ("uniform", "ints")))
    counts, parts = ctx.range_batch(qb, [p.rspec] * len(qts))
    assert parts is None and counts.shape == (len(qts), 128)
    counts2, parts2 = ctx.range_batch(qb, [p.rspec] * len(qts), [p.mplan.columns] * len(qts))
    assert np.array_equal(counts, counts2) and parts2.shape == (len(qts), 128, 4)
    assert np.array_equal(parts2[:, :, 0]["count"], counts)  # ints has a value in every doc


def test_tile_shortcut_counters(fx):
    """A sorted timestamp column puts most tiles in one bucket, a random one straddles."""
    c = fx.register(T.Context(0))
    try:
        check([c], fx, shapes(fx)[:6], RANGES["ts_3"], ())
        st = c.stats()
        assert 0 < st["range_tiles_one_bucket"] < st["range_tiles_seen"] and st["range_ms"] > 0 and st["units_range"] > 0
        one = st["range_tiles_one_bucket"]
        check([c], fx, shapes(fx)[:6], RANGES["u64_128"], ())
        st2 = c.stats()
        assert st2["range_tiles_one_bucket"] - one < (st2["range_tiles_seen"] - st["range_tiles_seen"]) // 4
    finally:
        c.close()


@pytest.mark.parametrize("fkind", FILTER_KINDS)
def test_filters(ctx, fx, fkind):
    j = FILTER_KINDS.index(fkind)
    qts = [(dict(q, filter=200 + j), t) for q, t in shapes(fx)[:8]]
    check([ctx], fx, qts, RANGES["ts_24"], ("ints", "dyadic", "flag"), masks=fx.filters[fkind])
    check([ctx], fx, qts[:4], RANGES["u64_5"], (), masks=fx.filters[fkind], count_hits=False)


@pytest.mark.parametrize("missing", [7, -3.5])
def test_missing_the_same_column_twice_and_count_only(ctx, fx, missing):
    extra = {"ints_m.sum": {"sum": {"field": "ints", "missing": missing}}, "flag_n.value_count": {"value_count": {"field": "flag", "missing": missing}}}
    check([ctx], fx, shapes(fx)[:10], RANGES["partial_edges"], ("half", "partial"), missing=missing, extra=extra)
    check([ctx], fx, shapes(fx)[:6], RANGES["ts_3"], ("us_half",), missing=missing)


def test_guard_refusal_in_one_bucket(ctx, fx):
    """The decimal sums fail the guard in some bucket: they are refused for the whole range, naming the first failing bucket, and
    the rest stays answered.  The narrow first bucket mostly holds no decimal value, so the refusal usually comes from the wide one."""
    rng = {"field": "uniform", "ranges": [{"to": 2.0**40}]}
    qts = shapes(fx)[:8]
    aggs = request(rng, ("decimal", "ints"))
    r = R.parse_request(aggs)
    fields = fields_of(fx, ("uniform", "decimal", "ints"))
    qb = QueryBatch([qt[0] for qt in qts])
    res = R.run([ctx], qb, [r] * len(qts), fields)
    p = R.plan(r, fields)
    _, parts = ctx.range_batch(qb, [p.rspec] * len(qts), [p.mplan.columns] * len(qts))
    col = p.mplan.slot["decimal.sum"]
    only_wide = 0
    for q, (qt, got) in enumerate(zip(qts, res)):
        refused = compare(got, model(fx, aggs, r, qt), r)
        failing = [b for b in range(2) if Mx.guard(parts[q, b, col]) is not None]
        assert set(refused) == ({"decimal.stats", "decimal.sum", "decimal.avg"} if failing else set())
        if failing:
            key = p.buckets[failing[0]]["key"]
            assert all(why.endswith(f"(bucket {key})") for why in refused.values())
            only_wide += failing == [1]
    assert only_wide > 0


def test_split_segment_over_two_contexts(fx):
    """The big segment's halves in two contexts (doc ranges), merged by ranges.run, against the model on the whole segment."""
    big = fx.osegs[0]
    half = (big.max_doc // 8192 // 2) * 8192 + 100
    cols = ("ints", "dyadic", "partial")
    ctxs = []
    try:
        for lo, hi in ((0, half), (half, big.max_doc)):
            c = T.Context(0)
            big.register(c)
            c.segment_set_doc_range(big.segment_ord, 0, lo, hi)
            for k in cols + ("ts", "uniform"):
                v, p = fx.columns[k][0]
                c.sort_column_register(fx.mcol[k], big.segment_ord, v, None if p is None else packed(p))
            ctxs.append(c)
        for rng in ("ts_24", "u64_5"):
            for cs in ((), cols):
                aggs = request(RANGES[rng], cs)
                r = R.parse_request(aggs)
                fields = fields_of(fx, cs + (RANGES[rng]["field"],))
                for q, t in shapes(fx)[:8]:
                    q = dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] == big.segment_ord])
                    (got,), hits = R.run(ctxs, QueryBatch([q]), [r], fields, count_hits=True)
                    assert int(hits[0]) == sum(int(c.count_batch(QueryBatch([q]))[0]) for c in ctxs)
                    compare(got, model(fx, aggs, r, (q, t), segs={0}), r)
    finally:
        for c in ctxs:
            c.close()


def test_waves_match_one_wave(fx):
    """A budget of 8 accumulators runs every query in a wave of its own, with the same rows."""
    qts = shapes(fx)[:12]
    qb = QueryBatch([qt[0] for qt in qts])
    p = R.plan(R.parse_request(request(RANGES["ts_24"], ("ints", "partial"))), fields_of(fx, ("ints", "partial", "ts")))
    base = fx.register(T.Context(0))
    os.environ["TQ_HIST_METRICS_BUDGET"] = "8"
    try:
        small = fx.register(T.Context(0))
    finally:
        del os.environ["TQ_HIST_METRICS_BUDGET"]
    try:
        a = base.range_batch(qb, [p.rspec] * len(qts), [p.mplan.columns] * len(qts), count_hits=True)
        b = small.range_batch(qb, [p.rspec] * len(qts), [p.mplan.columns] * len(qts), count_hits=True)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2])
        assert a[1].tobytes() == b[1].tobytes()
        assert a[0].sum() > 0
    finally:
        base.close()
        small.close()


def code(fn):
    with pytest.raises(T.TqError) as e:
        fn()
    return int(str(e.value).split("error ")[1].split(":")[0])


def test_error_codes_and_empty_batch(ctx, fx):
    qb = QueryBatch([shapes(fx)[0][0]])
    col = fx.mcol["uniform"]
    ints = [(fx.mcol["ints"], TQ_FAST_U64)]
    counts, parts = ctx.range_batch(QueryBatch([]), [])
    assert counts.shape[0] == 0 and parts is None
    assert code(lambda: ctx.range_batch(qb, [(col, [0, 5, 5])])) == -1       # starts not strictly ascending
    assert code(lambda: ctx.range_batch(qb, [(col, [1, 5])])) == -1          # starts[0] != 0
    assert code(lambda: ctx.range_batch(qb, [(col, [])])) == -1              # no bucket
    assert code(lambda: ctx.range_batch(qb, [(col, [0])], [[]])) == -1       # a metrics spec without columns
    assert code(lambda: ctx.range_batch(qb, [(col, [0])], [[(fx.mcol["ints"], 9)]])) == -1  # a metric kind outside TQ_FAST_*
    assert code(lambda: ctx.range_batch(qb, [(999, [0])])) == -3             # no such column
    assert code(lambda: ctx.range_batch(qb, [(col, [0])], [ints + [(999, TQ_FAST_U64, TQ_METRIC_COUNT_ONLY)]])) == -3
    phrase = dict(shapes(fx)[0][0], op=TQ_OP_PHRASE)
    assert code(lambda: ctx.range_batch(QueryBatch([phrase]), [(col, [0])])) == -4
    with pytest.raises(ValueError):
        ctx.range_batch(qb, [(col, list(range(129)))])


def fixture_column(kind, docs, field):
    present = np.array([field in d for d in docs], bool)
    vals = np.array([d.get(field, 0) for d in docs], np.float64 if kind == "f64" else np.int64)
    images = T.fast_value_to_u64(vals.astype(np.uint64) if kind == "u64" else vals, kind)
    return images, present


RUNNABLE = [c for c in SEARCHES if not c.get("refused")]


@pytest.mark.parametrize("case", RUNNABLE, ids=[c["name"] for c in RUNNABLE])
def test_reference_fixtures_on_device(case):
    """The reference's vectors end to end: every segment a real segment whose term 0 lists the collected docs, every numeric field
    a registered column, the rows finalised by tantivy_b200.ranges."""
    p, fields = fixture_plan(case)
    c = T.Context(0)
    try:
        segs = []
        for docs in case["segments"]:
            n = len(docs)
            if not any(collected(case, d) for d in docs):
                continue  # (a segment without a collected doc adds nothing; a term needs at least one posting)
            hit = np.array([i for i, d in enumerate(docs) if collected(case, d)], np.uint32)
            s = OracleSegment([(hit, np.ones(len(hit), np.uint32))], [1] * n, segment_ord=fresh_ord(), writer_cls=T.FieldWriter)
            s.register(c)
            for name, f in fields.items():
                if case["fields"][name] in ("u64", "i64", "f64", "date"):
                    images, present = fixture_column(case["fields"][name], docs, name)
                    c.sort_column_register(f.column_id, s.segment_ord, images, None if present.all() else packed(present))
            segs.append(s)
        q = make_query(TQ_OP_TERM, segs, [0], 10)
        res, hits = R.run([c], QueryBatch([q]), [p.request], fields, count_hits=True)
        assert int(hits[0]) == sum(bool(collected(case, d)) for docs in case["segments"] for d in docs)
        if "expected" in case:
            assert same_tree(res[0], case["expected"])
        else:
            check_asserts(case, res[0])
    finally:
        c.close()
