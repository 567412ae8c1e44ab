"""Histogram aggregations on the device (tq_histogram_batch: k_hist + k_hist_final) against tests/histogram_model.py over the docs
tests/score_model.py matches (and-ed with the alive bits, the filter and the doc range, as Count counts them).  Rows -- the
non-empty buckets in ascending pos and their doc counts -- and hits are compared exactly.  The fixture is test_gpu_sort_field's
(three segments, deletes in two, an `edge` term on every 8192-doc tile and unit edge, an `all` term) with more columns: date,
bool, f64 with +-0, +-inf, NaN and subnormals, tenths (values that land on bucket edges after the f64 division) and ramps on
both sides of the shared-memory counter threshold."""
import ctypes as C
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200 import histogram as Hg  # noqa: E402
from tantivy_b200._abi import HISTOGRAM_SPEC_DTYPE, TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM, HistogramSpec, QueryBatch, ptr, u32p, u64p  # noqa: E402
from tantivy_b200.lib import LIB  # noqa: E402
from tests import histogram_model as HM  # noqa: E402
from tests.helpers import OracleSegment, make_query  # noqa: E402
from tests.test_gpu_parity import fresh_ord  # noqa: E402
from tests.test_gpu_sort_field import ALL, EDGE, FILTER_KINDS, Fixture, packed, shapes  # noqa: E402
from tests.test_histogram_host import FIXTURES, check_result, fixture_images  # noqa: E402

INF = float("inf")
FMAX = Hg.F64_MAX
# column -> (fast kind, [(interval, offset), ...]) -- every pair runs every shape
COLUMNS = {
    "uniform": ("u64", [(2.0**50, 0.0), (2.0**54, 12345.0), (2.0**45, 0.0)]),  # 16385, 1025 and 2^19 + 1 buckets
    "monotone": ("u64", [(3000.0, 0.0), (1e8, -0.5), (1e15, 0.0)]),  # many, few (one-bucket tiles) and one bucket
    "equal": ("u64", [(1.0, 0.0), (0.1, 0.0)]),
    "few": ("u64", [(1.0, 0.0), (7.0, -3.5)]),
    "half": ("u64", [(7.0, 0.5), (0.1, 0.0)]),
    "none": ("u64", [(1.0, 0.0)]),
    "i64": ("i64", [(7.0, -2.25), (1.0, 0.0)]),
    "f64s": ("f64", [(0.1, 0.0), (1.0, 0.0), (2.5, -0.75)]),
    "f64i": ("f64", [(0.5, 0.0)]),
    "bool": ("bool", [(1.0, 0.0), (0.5, 0.0)]),
    "date": ("date", [(60e9, 0.0), (3600e9, -1800e9)]),  # 1 min, 1 h with a half-hour offset
    "tenths": ("f64", [(0.1, 0.0), (0.3, 0.1)]),
    "ramp4096": ("i64", [(1.0, 0.0)]),  # exactly kHistSmemBins counters
    "ramp4097": ("i64", [(1.0, 0.0)]),  # one above: global counters
}
HCOL = {k: 300 + i for i, k in enumerate(COLUMNS)}
F64S = np.array([-0.0, 0.0, -1.5, 2.25, INF, -INF, 3.0, np.nan, 5e-324, -5e-324, 2.2250738585072014e-308, 0.3, 0.7, -np.nan])


class HistFixture(Fixture):
    def __init__(self):
        super().__init__()
        rng = np.random.default_rng(0x4157)
        for i, s in enumerate(self.osegs):
            n = s.max_doc
            doc = np.arange(n)
            extra = {
                "f64s": (T.fast_value_to_u64(rng.choice(F64S, size=n), "f64"), None),
                "f64i": (T.fast_value_to_u64(rng.choice(np.array([-1.5, 2.25, INF, -INF, 3.0]), size=n), "f64"), None),
                "bool": (T.fast_value_to_u64(rng.random(n) < 0.3, "bool"), rng.random(n) < 0.9),
                "date": (T.fast_value_to_u64(np.int64(1_600_000_000) * 10**9 + np.int64(i) * 10**12 + doc.astype(np.int64) * 10**9, "date"), None),
                "tenths": (T.fast_value_to_u64((doc % 1000) * 0.1, "f64"), None),
                "ramp4096": (T.fast_value_to_u64(doc % 4096, "i64"), None),
                "ramp4097": (T.fast_value_to_u64(doc % 4097, "i64"), None),
            }
            for k, v in extra.items():
                self.columns.setdefault(k, []).append(v)

    def register(self, ctx, filters=()):
        super().register(ctx, kinds=(), filters=filters)
        for k in COLUMNS:
            self.register_hcol(ctx, k)
        return ctx

    def register_hcol(self, ctx, col):
        for i, s in enumerate(self.osegs):
            v, p = self.columns[col][i]
            ctx.sort_column_register(HCOL[col], s.segment_ord, v, None if p is None else packed(p))

    def hmodel(self, qt, col, interval, offset, lo=-FMAX, hi=FMAX, masks=None):
        kind = COLUMNS[col][0]
        parts = []
        for i in range(len(self.osegs)):
            sel = self.has(i, qt) & self.alive[i]
            if masks is not None:
                sel &= masks[i]
            v, p = self.columns[col][i]
            parts.append(HM.collect(v, p, sel, kind, interval, offset, lo, hi))
        return sorted(HM.merge(parts).items())


def rows(out, q):
    pos, counts, n = out[:3]
    return [(int(pos[q, j]), int(counts[q, j])) for j in range(int(n[q]))]


def code(fn):
    with pytest.raises(T.TqError) as e:
        fn()
    return int(str(e.value).split("error ")[1].split(":")[0])


@pytest.fixture(scope="module")
def fx():
    return HistFixture()


@pytest.fixture(scope="module")
def ctx(fx):
    c = fx.register(T.Context(0), filters=FILTER_KINDS)
    yield c
    c.close()


def run_check(ctx, fx, qts, col, interval, offset, lo=-FMAX, hi=FMAX, masks=None):
    kind = COLUMNS[col][0]
    qb = QueryBatch([q for q, _ in qts])
    out = ctx.histogram_batch(qb, [(HCOL[col], kind, interval, offset, lo, hi)] * len(qts), count_hits=True)
    for i, qt in enumerate(qts):
        want = fx.hmodel(qt, col, interval, offset, lo, hi, masks=masks)
        assert rows(out, i) == want, f"{col} interval {interval} offset {offset} query {i} op {qt[0]['op']} {qt[1]}"
    assert np.array_equal(out[3], ctx.count_batch(qb)) if masks is None else True
    return out


@pytest.mark.parametrize("col", list(COLUMNS))
def test_shapes_against_model(ctx, fx, col):
    """Every query shape (term, AND, OR, BOOL_SHAPES, random boolean shapes) on one column at each of its intervals."""
    for interval, offset in COLUMNS[col][1]:
        run_check(ctx, fx, shapes(fx), col, interval, offset)


def test_bounds(ctx, fx):
    """Binding, non-binding (collapsed) and half-open hard bounds; +-inf in bounds and out of them."""
    qts = [fx.query(TQ_OP_TERM, [ALL], 10), fx.query(TQ_OP_OR, [0, 4], 10), fx.query(TQ_OP_AND, [0, 1], 10)]
    run_check(ctx, fx, qts, "half", 7.0, 0.5, 100.0, 600.0)
    run_check(ctx, fx, qts, "half", 7.0, 0.5, -1.0, 2000.0)  # wider than the column: collapsed
    run_check(ctx, fx, qts, "half", 1.0, 0.0, 999.0, 5000.0)
    run_check(ctx, fx, qts, "f64s", 0.25, -0.125, -2.0, 2.5)
    run_check(ctx, fx, qts, "f64i", 0.5, 0.0, -INF, INF)  # collapses: the column has no NaN, so its +-inf docs are dropped
    run_check(ctx, fx, qts, "i64", 2.0, 0.0, -10.5, 10.5)
    run_check(ctx, fx, qts, "date", 60e9, 0.0, 1.6e18 + 5e11, 1.6e18 + 1.5e12)
    # in bounds, an infinity falls in a saturated bucket: that range is the CPU path's
    for lo, hi, col in ((-1e9, INF, "f64i"), (-INF, INF, "f64s")):
        assert code(lambda: ctx.histogram_batch(QueryBatch([qts[0][0]]), [(HCOL[col], "f64", 0.5, 0.0, lo, hi)])) == -4


def test_edges_and_no_match(ctx, fx):
    qts = [fx.query(TQ_OP_TERM, [EDGE], 10), fx.query(TQ_OP_AND, [EDGE, 4], 10), fx.query(TQ_OP_OR, [EDGE, 3], 10)]
    for col in ("monotone", "tenths", "ramp4097", "half"):
        for interval, offset in COLUMNS[col][1]:
            run_check(ctx, fx, qts, col, interval, offset)
    q = dict(fx.query(TQ_OP_TERM, [4], 10)[0], term_segs=[])
    out = ctx.histogram_batch(QueryBatch([q]), [(HCOL["few"], "u64", 1.0, 0.0)], count_hits=True)
    assert out[2][0] == 0 and out[3][0] == 0


@pytest.mark.parametrize("fkind", FILTER_KINDS)
def test_filters(ctx, fx, fkind):
    fid = 200 + FILTER_KINDS.index(fkind)
    base = [fx.query(TQ_OP_TERM, [0], 10), fx.query(TQ_OP_AND, [0, 5], 10), fx.query(TQ_OP_OR, [3, 4, EDGE], 10), fx.query(TQ_OP_TERM, [ALL], 10)]
    qts = [(dict(q, filter=fid), t) for q, t in base]
    for col in ("monotone", "date", "uniform"):
        interval, offset = COLUMNS[col][1][0]
        out = run_check(ctx, fx, qts, col, interval, offset, masks=fx.filters[fkind])
        assert np.array_equal(out[3], ctx.count_batch(QueryBatch([q for q, _ in qts])))


def test_one_bucket_tiles(fx):
    """A timestamp of one doc per second at a one-day interval counts most 8192-doc tiles as one bucket; u64 noise none.  Rows equal
    the model."""
    c = fx.register(T.Context(0))
    try:
        qts = [fx.query(TQ_OP_TERM, [ALL], 10), fx.query(TQ_OP_OR, [0, 5], 10)]
        s0 = c.stats()
        run_check(c, fx, qts, "date", 86400e9, 0.0)
        s1 = c.stats()
        assert s1["hist_tiles_one_bucket"] - s0["hist_tiles_one_bucket"] > (s1["hist_tiles_seen"] - s0["hist_tiles_seen"]) // 2
        assert s1["units_hist"] > s0["units_hist"] and s1["hist_ms"] > s0["hist_ms"]
        run_check(c, fx, qts, "uniform", 2.0**50, 0.0)
        s2 = c.stats()
        assert s2["hist_tiles_one_bucket"] == s1["hist_tiles_one_bucket"] and s2["hist_tiles_seen"] > s1["hist_tiles_seen"]
    finally:
        c.close()


def test_doc_ranges_merge(fx):
    """Two contexts, each with half of the big segment's tiles: their rows summed equal the model over the whole segment."""
    big = fx.osegs[0]
    half = (big.max_doc // 8192 // 2) * 8192
    parts = []
    for lo, hi in ((0, half), (half, big.max_doc)):
        c = T.Context(0)
        big.register(c)
        c.segment_set_doc_range(big.segment_ord, 0, lo, hi)
        c.sort_column_register(HCOL["tenths"], big.segment_ord, fx.columns["tenths"][0][0])
        parts.append(c)
    try:
        q, t = fx.query(TQ_OP_OR, [0, 4], 10)
        q = dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] == big.segment_ord])
        outs = [c.histogram_batch(QueryBatch([q]), [(HCOL["tenths"], "f64", 0.3, 0.1)], count_hits=True) for c in parts]
        got = sorted(Hg.merge_intermediate(rows(o, 0) for o in outs).items())
        sel = fx.has(0, (q, t)) & fx.alive[0]
        assert got == sorted(HM.collect(fx.columns["tenths"][0][0], None, sel, "f64", 0.3, 0.1).items())
        assert sum(int(o[3][0]) for o in outs) == int(sel.sum())
    finally:
        for c in parts:
            c.close()


def test_errors_and_stride_retry(ctx, fx):
    q, _ = fx.query(TQ_OP_TERM, [ALL], 10)
    qb = QueryBatch([q])
    assert code(lambda: ctx.histogram_batch(qb, [(999, "u64", 1.0, 0.0)])) == -3  # no such column
    assert code(lambda: ctx.histogram_batch(qb, [(HCOL["uniform"], "u64", 1.0, 0.0)])) == -4  # over 2^20 buckets
    for interval in (0.0, -1.0, INF, float("nan")):
        assert code(lambda: ctx.histogram_batch(qb, [(HCOL["few"], "u64", interval, 0.0)])) == -1
    assert code(lambda: ctx.histogram_batch(qb, [(HCOL["few"], 7, 1.0, 0.0)])) == -1
    phrase = dict(q, op=3, term_pos=[(0, 0)] * len(q["term_segs"]), term_offset=[0])
    assert code(lambda: ctx.histogram_batch(QueryBatch([phrase]), [(HCOL["few"], "u64", 1.0, 0.0)])) == -4
    # a row wider than out_stride: every row length is written and the call fails; Context.histogram_batch retries wider
    spec = np.zeros(2, HISTOGRAM_SPEC_DTYPE)
    spec[0] = (HCOL["ramp4097"], 1, 1.0, 0.0, -FMAX, FMAX)
    spec[1] = (HCOL["few"], 0, 1.0, 0.0, -FMAX, FMAX)
    qb2 = QueryBatch([q, q])
    pos, cnt, n = np.zeros((2, 8), np.int64), np.zeros((2, 8), np.uint64), np.zeros(2, np.uint32)
    rc = LIB.tq_histogram_batch(ctx.h, qb2.ptr, spec.ctypes.data_as(C.POINTER(HistogramSpec)), 2, 8, pos.ctypes.data_as(C.POINTER(C.c_int64)),
                                ptr(cnt, u64p), ptr(n, u32p), None)
    assert rc == -1 and list(n) == [4097, 4]
    out = ctx.histogram_batch(qb2, [(HCOL["ramp4097"], "i64", 1.0, 0.0), (HCOL["few"], "u64", 1.0, 0.0)])
    assert rows(out, 0) == fx.hmodel((q, [ALL]), "ramp4097", 1.0, 0.0) and len(rows(out, 0)) == 4097
    assert rows(out, 1) == fx.hmodel((q, [ALL]), "few", 1.0, 0.0)


def test_unregister_during_run_is_refused(fx):
    """A histogram run on another thread holds its column: re-registering it meanwhile is refused, and the run's rows stay the
    model's.  The batch is large (every shape 32 times, each doc through the gather path) so that the run outlasts several
    registration attempts; a run that still ends first is repeated, at most three times."""
    c = fx.register(T.Context(0))
    try:
        qts = shapes(fx)
        qb = QueryBatch([q for q, _ in qts] * 32)
        specs = [(HCOL["tenths"], "f64", 0.1, 0.0)] * qb.nq
        refused, errors = [], []
        for _ in range(3):
            result = {}
            started = threading.Event()

            def run():
                started.set()
                try:
                    result["out"] = c.histogram_batch(qb, specs, count_hits=True)
                except Exception as e:  # noqa: BLE001
                    errors.append(e)

            t = threading.Thread(target=run)
            t.start()
            started.wait()
            while t.is_alive():
                try:
                    c.sort_column_register(HCOL["tenths"], fx.osegs[0].segment_ord, fx.columns["tenths"][0][0])
                except T.TqError as e:
                    assert "still reads the column" in str(e)
                    refused.append(1)
            t.join()
            assert not errors
            for i, qt in enumerate(qts):
                assert rows(result["out"], i) == fx.hmodel(qt, "tenths", 0.1, 0.0)
            if refused:
                break
        assert refused, "no registration was tried while a run held the column"
        c.sort_column_unregister(HCOL["tenths"])
        assert code(lambda: c.histogram_batch(QueryBatch([qts[0][0]]), [(HCOL["tenths"], "f64", 0.1, 0.0)])) == -3
    finally:
        c.close()


def test_segment_of_2_to_the_31_docs():
    """One segment of 2^31 - 2 docs: three lists and a date column (one doc per second, 10 % of the docs without a value) in its
    top 300 000 docs and at max_doc - 1.  Term, OR and AND queries at 1 s (unit windows above the shared-memory threshold), 1 min
    and 1 h, and with binding hard bounds, equal the model; hits equal tq_count_batch.  (The column's values below the top are
    zero pages of a 16 GiB array, never written.)"""
    rng = np.random.default_rng(0x31)
    max_doc = 2**31 - 2
    top = max_doc - 300_000
    lists = []
    for p in (0.2, 0.05, 0.01):
        d = np.union1d(top + np.nonzero(rng.random(max_doc - top) < p)[0], [max_doc - 1]).astype(np.uint32)
        lists.append((d, np.ones(len(d), np.uint32)))
    seg = OracleSegment(lists, None, segment_ord=fresh_ord(), writer_cls=T.FieldWriter, max_doc=max_doc)
    values = np.zeros(max_doc, np.uint64)
    values[top:] = T.fast_value_to_u64(np.int64(1_700_000_000) * 10**9 + np.arange(max_doc - top, dtype=np.int64) * 10**9, "date")
    has = np.zeros(max_doc - top, bool)
    has[rng.random(max_doc - top) < 0.9] = True
    has[-1] = True
    present = np.zeros((max_doc + 7) // 8, np.uint8)
    sel = top + np.nonzero(has)[0]
    np.bitwise_or.at(present, sel >> 3, (1 << (sel & 7)).astype(np.uint8))
    c = T.Context(0)
    try:
        seg.register(c)
        c.sort_column_register(9, seg.segment_ord, values, present)
        del values
        top_values = T.fast_value_to_u64(np.int64(1_700_000_000) * 10**9 + np.arange(max_doc - top, dtype=np.int64) * 10**9, "date")
        qs = [(make_query(TQ_OP_TERM, [seg], [0], 10), lambda: lists[0][0]),
              (make_query(TQ_OP_OR, [seg], [0, 1, 2], 10), lambda: np.union1d(np.union1d(lists[0][0], lists[1][0]), lists[2][0])),
              (make_query(TQ_OP_AND, [seg], [0, 1], 10), lambda: np.intersect1d(lists[0][0], lists[1][0]))]
        qb = QueryBatch([q for q, _ in qs])
        counts = c.count_batch(qb)
        t0 = 1_700_000_000 * 10**9
        for interval, offset, lo, hi in ((1e9, 0.0, -FMAX, FMAX), (60e9, 0.0, -FMAX, FMAX), (3600e9, -1800e9, -FMAX, FMAX),
                                         (60e9, 0.0, t0 + 1e13, t0 + 2e14)):
            out = c.histogram_batch(qb, [(9, "date", interval, offset, lo, hi)] * len(qs), count_hits=True)
            assert np.array_equal(out[3], counts)
            for i, (_, docs) in enumerate(qs):
                m = np.zeros(max_doc - top, bool)
                m[docs().astype(np.int64) - top] = True
                want = sorted(HM.collect(top_values, has, m, "date", interval, offset, lo, hi).items())
                assert rows(out, i) == want and want, (interval, i)
    finally:
        c.close()


@pytest.mark.parametrize("case", [c for c in FIXTURES if "error" not in c], ids=[c["name"] for c in FIXTURES if "error" not in c])
def test_reference_fixtures_on_device(case):
    """The reference's histogram vectors end to end: every segment a real segment with an `all` term standing in for AllQuery,
    its values a registered column, the rows finalised by tantivy_b200.histogram."""
    c = T.Context(0)
    try:
        req, _ = Hg.parse_request(case["agg"])
        spec = Hg.histogram_spec(req, 1, case["kind"])
        segs = []
        for im in fixture_images(case):
            n = len(im)
            if n == 0:
                continue
            s = OracleSegment([(np.arange(n, dtype=np.uint32), np.ones(n, np.uint32))], [1] * n, segment_ord=fresh_ord(), writer_cls=T.FieldWriter)
            s.register(c)
            c.sort_column_register(1, s.segment_ord, im)
            segs.append(s)
        inter = {}
        if segs:
            out = c.histogram_batch(QueryBatch([make_query(TQ_OP_TERM, segs, [0], 10)]), [spec], count_hits=True)
            inter = Hg.merge_intermediate([rows(out, 0)])
            assert int(out[3][0]) == sum(len(s) for s in case["segments"])
        check_result(case, Hg.finalize(req, inter, case["kind"]))
    finally:
        c.close()
