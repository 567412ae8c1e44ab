"""Terms aggregations on the device (tq_terms_batch: k_terms + k_terms_select) against tests/terms_model.py over the docs
tests/score_model.py matches (and-ed with the alive bits and the filter, as Count counts them).  Rows -- the kept entries of every
segment ascending by (segment_ord, key) --, both scalars and hits are compared exactly.  The fixture is test_gpu_sort_field's (three
segments, deletes in two, an `edge` term on every 8192-doc tile and unit edge, an `all` term) with more columns: low-cardinality and
clustered ordinals, ramps on both sides of the shared-memory counter threshold, bool, date, images at 2^64 - 1 and spans of 2^20
and 2^20 + 1 keys."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200 import terms as Tm  # noqa: E402
from tantivy_b200._abi import (TQ_OP_OR, TQ_OP_TERM, TQ_ORDER_ASC, TQ_ORDER_DESC, TQ_TERMS_BY_COUNT, TQ_TERMS_BY_KEY, TQ_TERMS_MISSING_AFTER_MAX,  # noqa: E402
                               TQ_TERMS_MISSING_IMAGE, TQ_TERMS_MISSING_NONE, QueryBatch)
from tests import terms_model as TM  # noqa: E402
from tests.helpers import OracleSegment, make_query  # noqa: E402
from tests.test_gpu_parity import fresh_ord  # noqa: E402
from tests.test_terms_host import FIXTURES, check_result, fixture_segments, missing_image  # noqa: E402
from tests.test_gpu_sort_field import ALL, EDGE, FILTER_KINDS, Fixture, packed, shapes  # noqa: E402

ORDERS = [(TQ_TERMS_BY_COUNT, TQ_ORDER_DESC), (TQ_TERMS_BY_COUNT, TQ_ORDER_ASC), (TQ_TERMS_BY_KEY, TQ_ORDER_DESC), (TQ_TERMS_BY_KEY, TQ_ORDER_ASC)]
MAX = 2**64 - 1


class TermsFixture(Fixture):
    def __init__(self):
        super().__init__()
        rng = np.random.default_rng(0x7E5)
        for i, s in enumerate(self.osegs):
            n = s.max_doc
            doc = np.arange(n)
            span = rng.integers(0, 1 << 20, size=n).astype(np.uint64)
            span[[0, n - 1]] = [0, (1 << 20) - 1]
            span1 = span.copy()
            span1[n - 1] = 1 << 20
            extra = {
                "str20": (rng.integers(0, 20, size=n).astype(np.uint64), None),
                "clustered": ((doc // 9000).astype(np.uint64), rng.random(n) < 0.95),
                "random10k": (rng.integers(0, 10_000, size=n).astype(np.uint64), None),
                "ramp4096": ((doc % 4096).astype(np.uint64), None),
                "ramp4097": ((doc % 4097).astype(np.uint64), None),
                "bool": (T.fast_value_to_u64(rng.random(n) < 0.3, "bool"), rng.random(n) < 0.9),
                "date": (T.fast_value_to_u64(np.int64(1_600_000_000) * 10**9 + rng.integers(0, 40, size=n) * 1000, "date"), None),  # 1 µs steps: a span the device takes
                "top": ((MAX - rng.integers(0, 5, size=n).astype(np.uint64)).astype(np.uint64), rng.random(n) < 0.8),
                "span20": (span, None),
                "span20p1": (span1, None),
                "ties": ((doc % 50).astype(np.uint64), None),
                # values in the first and last segment, none in the middle one: the missing key is max + 1 in one, 1 in the other
                "partial": ((doc % 30).astype(np.uint64), (rng.random(n) < 0.7) if i != 1 else np.zeros(n, bool)),
                # f64 images are dense only within a few ulps: four neighbours of 1.0 (values of mixed sign are refused below)
                "fewf": (T.fast_value_to_u64(1.0 + rng.integers(0, 4, size=n) * 2.0**-52, "f64"), None),
            }
            for k, v in extra.items():
                self.columns.setdefault(k, []).append(v)
        self.tcol = {k: 400 + i for i, k in enumerate(self.columns)}

    def register(self, ctx, filters=()):
        super().register(ctx, kinds=(), filters=filters)
        for k in self.columns:
            for i, s in enumerate(self.osegs):
                v, p = self.columns[k][i]
                ctx.sort_column_register(self.tcol[k], s.segment_ord, v, None if p is None else packed(p))
        return ctx

    def missing_image(self, col, i, mode, image):
        if mode == TQ_TERMS_MISSING_NONE:
            return None
        if mode == TQ_TERMS_MISSING_IMAGE:
            return image
        v, p = self.columns[col][i]
        have = v if p is None else v[p]
        return (int(have.max()) if len(have) else 0) + 1

    def tmodel(self, qt, col, target, order, ss, mode=TQ_TERMS_MISSING_NONE, image=0, masks=None):
        rows, other, error = [], 0, 0
        for i in sorted(range(len(self.osegs)), key=lambda i: self.osegs[i].segment_ord):
            sel = self.has(i, qt) & self.alive[i]
            if masks is not None:
                sel &= masks[i]
            v, p = self.columns[col][i]
            kept, e, o = TM.cut(TM.collect(v, p, sel, self.missing_image(col, i, mode, image)), ss, target == TQ_TERMS_BY_KEY,
                                order == TQ_ORDER_ASC)
            rows += [(self.osegs[i].segment_ord, k, c) for k, c in kept]
            other += o
            error += e
        return rows, other, error


def rows(out, q):
    segs, keys, counts, n = out[:4]
    return [(int(segs[q, j]), int(keys[q, j]), int(counts[q, j])) for j in range(int(n[q]))]


def code(fn):
    with pytest.raises(T.TqError) as e:
        fn()
    return int(str(e.value).split("error ")[1].split(":")[0])


@pytest.fixture(scope="module")
def fx():
    return TermsFixture()


@pytest.fixture(scope="module")
def ctx(fx):
    c = fx.register(T.Context(0), filters=FILTER_KINDS)
    yield c
    c.close()


def run_check(ctx, fx, qts, col, target, order, ss, mode=TQ_TERMS_MISSING_NONE, image=0, masks=None):
    qb = QueryBatch([q for q, _ in qts])
    out = ctx.terms_batch(qb, [(fx.tcol[col], target, order, ss, mode, image)] * len(qts), count_hits=True)
    for i, qt in enumerate(qts):
        want, other, error = fx.tmodel(qt, col, target, order, ss, mode, image, masks)
        assert rows(out, i) == want, f"{col} {target}/{order} ss {ss} query {i} op {qt[0]['op']} {qt[1]}"
        assert (int(out[4][i]), int(out[5][i])) == (other, error), f"{col} {target}/{order} ss {ss} query {i}"
    if masks is None:
        assert np.array_equal(out[6], ctx.count_batch(qb))


@pytest.mark.parametrize("col", ["str20", "clustered", "random10k", "ramp4096", "ramp4097", "few", "half", "none", "i64", "bool", "date",
                                 "top", "ties", "fewf", "equal"])
def test_shapes_orders_against_model(ctx, fx, col):
    for target, order in ORDERS:
        for ss in (1, 10, 5000):
            run_check(ctx, fx, shapes(fx), col, target, order, ss)


def test_segment_size_edges(ctx, fx):
    qt = fx.query(TQ_OP_TERM, [ALL], 10)
    for col in ("str20", "ties", "ramp4097"):
        per_seg = [len(TM.collect(*fx.columns[col][i], fx.has(i, qt) & fx.alive[i])) for i in range(len(fx.osegs))]
        for n in sorted(set(per_seg)):
            for ss in (n - 1, n, n + 1):
                if ss >= 1:
                    for target, order in ORDERS:
                        run_check(ctx, fx, [qt], col, target, order, ss)


def test_missing_modes(ctx, fx):
    qts = shapes(fx)
    for target, order in ORDERS:
        run_check(ctx, fx, qts, "half", target, order, 7, TQ_TERMS_MISSING_AFTER_MAX)
        run_check(ctx, fx, qts, "half", target, order, 7, TQ_TERMS_MISSING_IMAGE, 5)  # equal to an existing value: the counts merge
        run_check(ctx, fx, qts, "half", target, order, 7, TQ_TERMS_MISSING_IMAGE, 1 << 40)  # outside the range: one more entry
        run_check(ctx, fx, qts, "half", target, order, 7, TQ_TERMS_MISSING_IMAGE, 0)
        run_check(ctx, fx, qts, "none", target, order, 3, TQ_TERMS_MISSING_AFTER_MAX)  # no value in any segment: the key is 0 + 1
        run_check(ctx, fx, qts, "partial", target, order, 4, TQ_TERMS_MISSING_AFTER_MAX)
        run_check(ctx, fx, qts, "clustered", target, order, 2, TQ_TERMS_MISSING_AFTER_MAX)
        run_check(ctx, fx, qts, "bool", target, order, 1, TQ_TERMS_MISSING_IMAGE, 0)
        run_check(ctx, fx, qts, "top", target, order, 3, TQ_TERMS_MISSING_IMAGE, 7)


def test_filters(ctx, fx):
    qts = shapes(fx)[:8]
    for j, fkind in enumerate(FILTER_KINDS):
        fq = [(dict(q, filter=200 + j), t) for q, t in qts]
        run_check(ctx, fx, fq, "str20", TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 5, masks=fx.filters[fkind])
        run_check(ctx, fx, fq, "half", TQ_TERMS_BY_KEY, TQ_ORDER_ASC, 5, TQ_TERMS_MISSING_AFTER_MAX, masks=fx.filters[fkind])


def test_span_limit_waves_stride_and_errors(fx):
    qt = fx.query(TQ_OP_TERM, [ALL], 10)
    qb = QueryBatch([qt[0]])
    c = fx.register(T.Context(0))
    try:
        run_check(c, fx, [qt], "span20", TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 10)  # 2^20 keys: accepted
        assert code(lambda: c.terms_batch(qb, [(fx.tcol["span20p1"], 0, 0, 10)])) == -4
        assert code(lambda: c.terms_batch(qb, [(fx.tcol["monotone"], 0, 0, 10)])) == -4
        assert code(lambda: c.terms_batch(qb, [(fx.tcol["f64"], 0, 0, 10)])) == -4  # +-0, -1.5, 2.25, +-inf: images far apart
        assert code(lambda: c.terms_batch(qb, [(999, 0, 0, 10)])) == -3
        for bad in ((fx.tcol["few"], 2, 0, 10), (fx.tcol["few"], 0, 2, 10), (fx.tcol["few"], 0, 0, 0), (fx.tcol["few"], 0, 0, 10, 3, 0)):
            assert code(lambda: c.terms_batch(qb, [bad])) == -1
        phrase = dict(qt[0], op=3, term_pos=[(0, 0)] * len(qt[0]["term_segs"]), term_offset=[0])
        assert code(lambda: c.terms_batch(QueryBatch([phrase]), [(fx.tcol["few"], 0, 0, 10)])) == -4
        # a row wider than the first stride: the call retries at its width
        out = c.terms_batch(qb, [(fx.tcol["ramp4097"], TQ_TERMS_BY_KEY, TQ_ORDER_ASC, 5000)], stride=16)
        assert int(out[3][0]) == sum(min(5000, 4097) for _ in fx.osegs) and rows(out, 0) == fx.tmodel(qt, "ramp4097", 1, 1, 5000)[0]
    finally:
        c.close()
    import os
    os.environ["TQ_TERMS_COUNTER_BUDGET"] = "5000"  # every query alone in its wave, several waves per batch
    try:
        c = fx.register(T.Context(0))
    finally:
        del os.environ["TQ_TERMS_COUNTER_BUDGET"]
    try:
        for target, order in ORDERS:
            run_check(c, fx, shapes(fx), "random10k", target, order, 10)
            run_check(c, fx, shapes(fx), "str20", target, order, 3, TQ_TERMS_MISSING_AFTER_MAX)
        st = c.stats()
        assert st["units_terms"] > 0 and st["terms_tiles_seen"] > 0 and st["terms_ms"] > 0
    finally:
        c.close()


def test_one_key_tiles_are_counted(fx):
    c = fx.register(T.Context(0))
    try:
        qt = fx.query(TQ_OP_TERM, [ALL], 10)
        run_check(c, fx, [qt], "clustered", TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 10)
        st = c.stats()
        assert 0 < st["terms_tiles_one_key"] <= st["terms_tiles_seen"]
    finally:
        c.close()


def test_request_through_device(ctx, fx):
    """The request layer end to end on a str column: spec, device rows, per-segment dictionaries, finaliser."""
    qt = fx.query(TQ_OP_TERM, [EDGE], 10)
    dicts = {s.segment_ord: [f"term{j:02d}" for j in range(20)] for s in fx.osegs}
    for body in ({"field": "f"}, {"field": "f", "size": 3, "order": {"_key": "desc"}}, {"field": "f", "size": 2, "segment_size": 2},
                 {"field": "f", "missing": "NA", "order": {"_count": "asc"}}):
        req = Tm.parse_request({"terms": body})
        spec = Tm.terms_spec(req, fx.tcol["str20"], "str")
        out = ctx.terms_batch(QueryBatch([qt[0]]), [spec])
        got = Tm.finalize_rows(req, "str", [tuple(x[0] for x in out[:6])], dicts, {s: 20 for s in dicts})
        parts = []
        for i, s in enumerate(fx.osegs):
            v, p = fx.columns["str20"][i]
            kept, e, o = TM.cut(TM.collect(v, p, fx.has(i, qt) & fx.alive[i]), req.segment_size, req.order_target == "_key", req.order == "asc")
            parts.append((Tm.segment_result(req, "str", kept, dicts[s.segment_ord], 20), o, e))
        assert got == Tm.finalize(req, Tm.merge(parts)), body


def test_doc_ranges_are_cut_once_per_segment(fx):
    """Two contexts, each with half of the big segment's tiles, return it uncut; finalize_rows sums the halves and cuts once, and
    equals the model over the whole segment (a small segment_size, so the cut matters)."""
    big = fx.osegs[0]
    half = (big.max_doc // 8192 // 2) * 8192
    parts = []
    for lo, hi in ((0, half), (half, big.max_doc)):
        c = T.Context(0)
        big.register(c)
        c.segment_set_doc_range(big.segment_ord, 0, lo, hi)
        c.sort_column_register(fx.tcol["random10k"], big.segment_ord, fx.columns["random10k"][0][0])
        parts.append(c)
    try:
        q, t = fx.query(TQ_OP_OR, [0, 4], 10)
        q = dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] == big.segment_ord])
        for body in ({"field": "f", "size": 3, "segment_size": 5}, {"field": "f", "size": 2, "order": {"_key": "desc"}, "segment_size": 4}):
            req = Tm.parse_request({"terms": body})
            spec = Tm.terms_spec(req, fx.tcol["random10k"], "u64")
            outs = [c.terms_batch(QueryBatch([q]), [spec]) for c in parts]
            for o in outs:  # uncut: every entry of its half, both scalars 0
                assert (int(o[4][0]), int(o[5][0])) == (0, 0) and int(o[3][0]) > req.segment_size
            got = Tm.finalize_rows(req, "u64", [tuple(x[0] for x in o[:6]) for o in outs])
            sel = fx.has(0, (q, t)) & fx.alive[0]
            kept, e, o = TM.cut(TM.collect(fx.columns["random10k"][0][0], None, sel), req.segment_size, req.order_target == "_key", req.order == "asc")
            assert got == Tm.finalize(req, Tm.merge([(Tm.segment_result(req, "u64", kept), o, e)])), body
    finally:
        for c in parts:
            c.close()


@pytest.mark.parametrize("case", [c for c in FIXTURES if "refused" not in c], ids=[c["name"] for c in FIXTURES if "refused" not in c])
def test_reference_fixtures_on_device(case):
    """The reference's terms vectors end to end: every segment a real segment with an `all` term standing in for AllQuery, its
    values a registered column (present bits for the docs without one), the rows finalised by tantivy_b200.terms."""
    c = T.Context(0)
    try:
        req = Tm.parse_request(case["agg"])
        spec = Tm.terms_spec(req, 1, case["kind"])
        segs, dicts, missing = [], {}, {}
        for images, present, terms in fixture_segments(case):
            n = len(images)
            s = OracleSegment([(np.arange(n, dtype=np.uint32), np.ones(n, np.uint32))], [1] * n, segment_ord=fresh_ord(), writer_cls=T.FieldWriter)
            s.register(c)
            c.sort_column_register(1, s.segment_ord, images, None if present.all() else packed(present))
            segs.append(s)
            dicts[s.segment_ord] = terms
            missing[s.segment_ord] = missing_image(spec, images, present)
        qb = QueryBatch([make_query(TQ_OP_TERM, segs, [0], 10)])
        spans = [int(im[p].max()) - int(im[p].min()) for im, p, _ in fixture_segments(case) if p.any()]
        if any(sp >= 1 << 20 for sp in spans):  # (u64 ids, ns dates, f64 integers: images far apart) the CPU path's
            assert code(lambda: c.terms_batch(qb, [spec])) == -4
            return
        out = c.terms_batch(qb, [spec], count_hits=True)
        assert int(out[6][0]) == sum(len(s) for s in case["segments"])
        check_result(case, Tm.finalize_rows(req, case["kind"], [tuple(x[0] for x in out[:6])], dicts, missing))
    finally:
        c.close()
