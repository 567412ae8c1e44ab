"""tq_sort_batch (k_sort + k_sort_final) and tq_histogram_batch (k_hist + k_hist_final) at the edges the small fixture of
test_gpu_sort_field / test_gpu_histogram does not reach, against the same models: Fixture.model / sort_rows, tests/histogram_model.py
and the match sets of tests/score_model.py.  Rows are compared exactly (value images, present, segment, doc; every (pos,
doc_count)); every run with count_hits checks its hits against tq_count_batch.

Fixture A: four segments of 0.57M-1.1M docs (71-135 tiles, 9-17 units of eight 8192-doc tiles each), each size leaving a partial
last 32-doc word, deletes in three, ordinals 5000, 1200, 0 and 2^31 + 7 registered and listed in term_segs in that order (plan
order is ordinal order, so the two differ).  Columns: timestamps ascending and descending in doc id, a `sparse` column with values on
0.05 % of the docs (ascending in doc id: every unit's bounds rise, so only its None docs keep it walking forwards), three-valued
`ties`, uniform u64, i64 extremes, f64 specials, a `window` column whose unit windows are 4096 buckets wide on some units and 9000
on others, and `tiebound`, whose k-th value's lowest-address ties sit in units the planner orders after the bound is set.  Filter
NOVALUE keeps the docs without a value in `sparse`: rows of None docs only.

The tests without the gpu mark check, with numpy and the planner's tile arithmetic only, that Fixture A reaches those edges, and
cross-check histogram_model.collect against a scalar restatement on the histogram edge values."""
import ctypes as C
import math
import struct
import threading
import types

import numpy as np
import pytest

import tantivy_b200 as T
from tantivy_b200 import histogram as Hg
from tantivy_b200._abi import (HISTOGRAM_SPEC_DTYPE, TQ_MAX_K, TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM, HistogramSpec, QueryBatch, ptr,
                               u32p, u64p)
from tantivy_b200.lib import LIB
from tests import histogram_model as HM
from tests import multi_field as MF
from tests import score_model as M
from tests.helpers import OracleSegment, make_query
from tests.test_gpu_sort_field import (ALL, DENS, EDGE, FILTER_KINDS, N_TERMS, Fixture, device_rows, edge_docs, packed, shapes,
                                       sort_rows, unpacked)

gpu = pytest.mark.gpu

TILE, UNIT_TILES = 8192, 8
K_CAP = 2048  # k_sort_final's on-chip candidate buffer
SMEM_BINS, MAX_BINS, MAX_COUNTERS = 4096, 1 << 20, 1 << 27
FMAX = Hg.F64_MAX
I64_MIN, I64_MAX = -2**63, 2**63 - 1
SIZES_A = (1_105_007, 573_451, 820_013, 655_369)
ORDS_A = (5000, 1200, 0, 2**31 + 7)
DELETES_A = (True, True, False, True)
KS_A = (1, 2, 255, 256, 257, 1000, 1023, 1024)
ORDERS = ("desc", "asc")
KINDS_A = ("uniform", "ts_asc", "ts_desc", "sparse", "ties", "i64ext", "f64ext", "window", "tiebound")
COL_A = {k: 400 + i for i, k in enumerate(KINDS_A)}
HKIND = {"uniform": "u64", "ts_asc": "u64", "ts_desc": "u64", "sparse": "u64", "ties": "u64", "i64ext": "i64", "f64ext": "f64",
         "window": "i64", "tiebound": "u64"}
F64_SPECIAL = np.array([-0.0, 0.0, np.inf, -np.inf, np.nan, -np.nan, 1e308, -1e308, 5e-324, 1.5, -2.5, 3.0])
TIE_LOW, TIE_K, TIE_TOP = 50, 100, 200  # tiebound's values
NOVALUE = 250  # filter id: the docs without a value in `sparse`


def tiles_of(max_doc):
    return (max_doc + TILE - 1) // TILE


def unit_ranges(max_doc):
    """The Count plan's units of an unfiltered query: [first tile, end tile) of eight tiles each."""
    n = tiles_of(max_doc)
    return [(t, min(n, t + UNIT_TILES)) for t in range(0, n, UNIT_TILES)]


def columns_a(rng, i, n):
    """{kind: (u64 images, present or None)} of segment i (n docs)."""
    doc = np.arange(n, dtype=np.int64)
    unit = doc // (TILE * UNIT_TILES)
    out = {}
    u = rng.integers(0, 2**64 - 1, size=n, dtype=np.uint64, endpoint=True)
    u[:4] = [0, 2**64 - 1, 2**64 - 1, 0]
    out["uniform"] = (u, None)
    out["ts_asc"] = (np.uint64(1_600_000_000_000) + np.uint64(i * 10**9) + doc.astype(np.uint64) * np.uint64(1000), None)
    out["ts_desc"] = (np.uint64(1_700_000_000_000) - np.uint64(i * 10**9) - doc.astype(np.uint64) * np.uint64(1000), None)
    sp = rng.random(n) < 0.0005
    sp[TILE - 1::TILE] = True  # (a value in every tile: each unit's bounds rise from its first tile to its last)
    sp[-1] = True
    out["sparse"] = (doc.astype(np.uint64) // np.uint64(7), sp)
    out["ties"] = (rng.choice(np.array([5, 6, 7], np.uint64), size=n, p=[0.2, 0.3, 0.5]), None)
    out["i64ext"] = (T.fast_value_to_u64(rng.choice(np.array([I64_MIN, I64_MAX, -1, 0, 17], np.int64), size=n), "i64"), None)
    out["f64ext"] = (T.fast_value_to_u64(rng.choice(F64_SPECIAL, size=n), "f64"), None)
    wide = (unit % 2 == 0) & (i in (1, 3))  # segments 0 and 2 (ordinals 5000 and 0): every unit 4096 buckets wide
    out["window"] = (T.fast_value_to_u64(np.where(wide, doc % 9000, doc % 4096), "i64"), None)
    t = np.full(n, TIE_LOW, np.uint64)
    if ORDS_A[i] == 0:  # sparse ties in every tile; the first unit walks backwards from its last tile, which alone holds k ties
        t[rng.random(n) < 0.001] = TIE_K
        t[7 * TILE:8 * TILE:4] = TIE_K
        t[7 * TILE:8 * TILE:64] = TIE_TOP
    else:
        t[rng.random(n) < 0.3] = TIE_K
        t[doc % 5000 == 0] = TIE_TOP
    out["tiebound"] = (t, None)
    return out


class FixtureA(Fixture):
    """Fixture's terms (N_TERMS random lists, `edge`, `all`) and methods over the four big segments.  build=False: the alive bits
    and columns only (numpy)."""

    def __init__(self, build=True, seed=0xA11):
        rng = np.random.default_rng(seed)
        self.sizes = SIZES_A
        self.alive, self.columns = [], {k: [] for k in KINDS_A}
        for i, n in enumerate(SIZES_A):
            a = rng.random(n) > 0.12
            a[edge_docs(n)[::2]] = True
            self.alive.append(a if DELETES_A[i] else np.ones(n, bool))
            for k, v in columns_a(rng, i, n).items():
                self.columns[k].append(v)
        self.filters = {}
        for k in FILTER_KINDS:
            masks = []
            for i, n in enumerate(SIZES_A):
                m = np.zeros(n, bool)
                if k == "ones":
                    m[:] = True
                elif k == "bern1":
                    m = rng.random(n) < 0.01
                elif k == "bern30":
                    m = rng.random(n) < 0.3
                elif k == "run":
                    m[n // 3 + 5:n // 3 + n // 7] = True  # (cuts inside a 32-doc word at both ends)
                elif k == "edges":
                    m[edge_docs(n)] = True
                elif k == "deleted":
                    m = ~self.alive[i]
                masks.append(m)
            self.filters[k] = masks
        self.novalue = [~p for _, p in self.columns["sparse"]]
        self._has = {}
        self.osegs, self.models = [], []
        if not build:
            return
        for i, n in enumerate(SIZES_A):
            lengths = np.clip(np.round(np.exp(rng.normal(np.log(40), 0.7, size=n))), 1, 4096).astype(np.uint32)
            lists = []
            for t in range(N_TERMS):
                docs = np.nonzero(rng.random(n) < DENS[t % len(DENS)])[0].astype(np.uint32)
                lists.append((docs, np.minimum(rng.geometric(0.6, size=len(docs)), 10).astype(np.uint32)))
            e = edge_docs(n)
            lists.append((e, np.ones(len(e), np.uint32)))
            lists.append((np.arange(n, dtype=np.uint32), np.ones(n, np.uint32)))
            alive = packed(self.alive[i]) if DELETES_A[i] else None
            self.osegs.append(OracleSegment(lists, lengths, segment_ord=ORDS_A[i], writer_cls=T.FieldWriter, alive=alive))
            self.models.append(M.Segment(ORDS_A[i], lists, lengths))
        for s, t in ((0, 6), (1, 3), (2, 11)):  # absent from some segments
            self.osegs[s].terms[t] = (0, 0, 0)

    def register(self, ctx, kinds=KINDS_A, filters=FILTER_KINDS):
        for s in self.osegs:
            s.register(ctx)
        for k in kinds:
            self.register_column(ctx, k)
        for j, k in enumerate(filters):
            for i, s in enumerate(self.osegs):
                ctx.filter_register(200 + FILTER_KINDS.index(k), s.segment_ord, packed(self.filters[k][i]))
        for i, s in enumerate(self.osegs):
            ctx.filter_register(NOVALUE, s.segment_ord, packed(self.novalue[i]))
        return ctx

    def register_column(self, ctx, kind, col_id=None, segs=None):
        for i, s in enumerate(self.osegs):
            if segs is None or i in segs:
                v, p = self.columns[kind][i]
                ctx.sort_column_register(COL_A[kind] if col_id is None else col_id, s.segment_ord, v, None if p is None else packed(p))


def model(fx, qt, kind, order, k, masks=None, doc_ranges=None, segs=None):
    """Fixture.model's (rows, count), each segment's docs first cut to the ones that can make its own top k (its k best docs with a
    value, ties at the k-th by doc, and its first k None docs); sort_rows orders the rest."""
    vals, pres, sos, docs, n = [], [], [], [], 0
    for i, s in enumerate(fx.osegs):
        if segs is not None and i not in segs:
            continue
        sel = fx.has(i, qt) & fx.alive[i]
        if masks is not None:
            sel &= masks[i]
        if doc_ranges is not None and i in doc_ranges:
            lo, hi = doc_ranges[i]
            sel[:lo] = False
            sel[hi:] = False
        d = np.nonzero(sel)[0]
        n += len(d)
        v, p = fx.columns[kind][i]
        pr = np.ones(len(d), bool) if p is None else p[d]
        dv, dn = d[pr], d[~pr][:k]
        if len(dv) > k:
            key = v[dv] if order == "desc" else ~v[dv]
            kth = np.partition(key, len(key) - k)[len(key) - k]
            above = np.nonzero(key > kth)[0]
            ties = np.nonzero(key == kth)[0][:k - len(above)]
            dv = dv[np.union1d(above, ties)]
        dd = np.concatenate([dv, dn])
        pp = np.concatenate([np.ones(len(dv), bool), np.zeros(len(dn), bool)])
        vals.append(np.where(pp, v[dd], np.uint64(0)))
        pres.append(pp)
        sos.append(np.full(len(dd), s.segment_ord, np.int64))
        docs.append(dd.astype(np.int64))
    rows, _ = sort_rows(np.concatenate(vals), np.concatenate(pres), np.concatenate(sos), np.concatenate(docs), order, k)
    return rows, n


def hmodel(fx, qt, kind, interval, offset, lo=-FMAX, hi=FMAX, masks=None, doc_ranges=None, segs=None):
    parts = []
    for i in range(len(fx.osegs)):
        if segs is not None and i not in segs:
            continue
        sel = fx.has(i, qt) & fx.alive[i]
        if masks is not None:
            sel &= masks[i]
        if doc_ranges is not None and i in doc_ranges:
            a, b = doc_ranges[i]
            sel[:a] = False
            sel[b:] = False
        v, p = fx.columns[kind][i]
        parts.append(HM.collect(v, p, sel, HKIND[kind], interval, offset, lo, hi))
    return sorted(HM.merge(parts).items())


def hrows(out, q):
    pos, counts, n = out[:3]
    return [(int(pos[q, j]), int(counts[q, j])) for j in range(int(n[q]))]


def code(fn):
    with pytest.raises(T.TqError) as e:
        fn()
    return int(str(e.value).split("error ")[1].split(":")[0])


def run_sorted(ctx, fx, base, kind, ks=KS_A, orders=ORDERS, count_hits=True, masks=None, extra=None):
    """Every base query at every k and order in ONE batch; rows against the model (computed once per query and order at the
    largest k: the rows at a smaller k are its prefix), hits against tq_count_batch."""
    qts = [(dict(q, k=k, **(extra or {})), t, b, o) for b, (q, t) in enumerate(base) for k in ks for o in orders]
    qb = QueryBatch([q for q, _, _, _ in qts])
    out = ctx.sort_batch(qb, [(COL_A[kind], o) for _, _, _, o in qts], count_hits=count_hits)
    cache = {}
    for i, (q, t, b, o) in enumerate(qts):
        if (b, o) not in cache:
            cache[(b, o)] = model(fx, (q, t), kind, o, max(ks), masks=masks)
        rows, n = cache[(b, o)]
        got = device_rows(out, i)
        assert got == rows[:q["k"]], f"{kind} {o} k={q['k']} query {b} op {q['op']} {t}: {got[:4]} vs {rows[:4]}"
    if count_hits:
        assert np.array_equal(out[5], ctx.count_batch(qb))
        for i, (q, t, b, o) in enumerate(qts):
            assert int(out[5][i]) == cache[(b, o)][1]
    return out, qts


def run_hist(ctx, fx, qts, kind, interval, offset, lo=-FMAX, hi=FMAX, masks=None):
    qb = QueryBatch([q for q, _ in qts])
    out = ctx.histogram_batch(qb, [(COL_A[kind], HKIND[kind], interval, offset, lo, hi)] * len(qts), count_hits=True)
    for i, qt in enumerate(qts):
        want = hmodel(fx, qt, kind, interval, offset, lo, hi, masks=masks)
        assert hrows(out, i) == want, f"{kind} interval {interval} offset {offset} [{lo}, {hi}] query {i} op {qt[0]['op']} {qt[1]}"
    assert np.array_equal(out[3], ctx.count_batch(qb))
    return out


# ---- reach checks (numpy and the planner's tile arithmetic; no GPU) ----------------------------------------------------------
@pytest.fixture(scope="module")
def data_a():
    return FixtureA(build=False)


def test_fixture_a_sizes_and_ordinals():
    """9-17 units a segment, a partial last 32-doc word everywhere, a unit of one tile, ordinals out of registration order and
    one above 2^31."""
    units = [len(unit_ranges(n)) for n in SIZES_A]
    assert min(units) >= 9 and max(units) == 17
    assert all(n % 32 for n in SIZES_A)
    assert any(e - b == 1 for n in SIZES_A for b, e in unit_ranges(n))
    assert list(ORDS_A) != sorted(ORDS_A) and max(ORDS_A) >= 2**31 and 0 in ORDS_A


def test_fixture_a_none_stream_exceeds_the_final_buffer(data_a):
    """`sparse` at k = 1024 over the alive docs of filter NOVALUE (the docs without a value): no doc with a value matches, so the
    whole row is None docs; each unit hands over min(k, its None docs), more than k_sort_final holds on chip, so the None rows go
    through its radix select; and the row is exactly the first k None docs of one unit (the lowest ordinal's first), so every one of
    the k that unit hands over is needed."""
    handed, first = 0, None
    for i in sorted(range(4), key=lambda i: ORDS_A[i]):
        p = data_a.columns["sparse"][i][1]
        sel = data_a.alive[i] & data_a.novalue[i]
        assert not (sel & p).any()
        for b, e in unit_ranges(SIZES_A[i]):
            c = int(sel[b * TILE:e * TILE].sum())
            first = c if first is None else first
            handed += min(TQ_MAX_K, c)
    assert handed > K_CAP and first >= TQ_MAX_K
    # and every unit's bounds rise: only its None docs keep it walking forwards
    for i, n in enumerate(SIZES_A):
        v, p = data_a.columns["sparse"][i]
        best = [int(v[t * TILE:(t + 1) * TILE][p[t * TILE:(t + 1) * TILE]].max(initial=0)) for t in range(tiles_of(n))]
        assert all(best[e - 1] > best[b] for b, e in unit_ranges(n) if e - b > 1)


def test_fixture_a_windows_on_both_sides_of_the_shared_memory_threshold(data_a):
    """`window` at interval 1: one query's units count into windows of 4096 buckets (shared memory) and of 9000 (global)."""
    widths = set()
    for i, n in enumerate(SIZES_A):
        w = HM.image_to_f64(data_a.columns["window"][i][0], "i64")
        for b, e in unit_ranges(n):
            seg = w[b * TILE:min(n, e * TILE)]
            widths.add(int(seg.max() - seg.min()) + 1)
    assert {SMEM_BINS, 9000} <= widths


def test_fixture_a_ties_land_behind_the_bound(data_a):
    """`tiebound` Desc at k = 1024 over every alive doc: fewer than k docs hold the top value, so the k-th value is the tie value,
    and its ties with the lowest addresses (ordinal 0) sit in units the planner orders after units that alone hold k docs at or
    above it -- and in the early tiles of a unit that walks backwards."""
    k = TQ_MAX_K
    top = sum(int(((data_a.columns["tiebound"][i][0] == TIE_TOP) & data_a.alive[i]).sum()) for i in range(4))
    assert top < k
    units = []  # (best, ordinal, unit, backward, docs >= TIE_K), in plan order
    plan = sorted(range(4), key=lambda i: ORDS_A[i])  # the plan walks segments by ordinal
    for i in plan:
        v = data_a.columns["tiebound"][i][0]
        for u, (b, e) in enumerate(unit_ranges(SIZES_A[i])):
            best = [int(v[t * TILE:(t + 1) * TILE].max()) for t in range(b, e)]
            units.append((max(best), ORDS_A[i], u, best[-1] > best[0], int((v[b * TILE:e * TILE] >= TIE_K).sum())))
    order = sorted(range(len(units)), key=lambda j: -units[j][0])  # stable: the planner's std::stable_sort by best
    first_full = next(p for p, j in enumerate(order) if units[j][4] >= k)
    late = [p for p, j in enumerate(order) if units[j][1] == 0 and units[j][2] > 0]
    assert late and min(late) > first_full
    u0 = next(j for j in range(len(units)) if units[j][1] == 0 and units[j][2] == 0)
    assert units[u0][3] and units[u0][0] == TIE_TOP  # backwards; its tiles 0-6 hold the ties
    # that unit's last tile, which it reads first, alone holds k docs at or above the tie value: the CTA's own bound is the tie
    # value before it reads tiles 6 .. 0, whatever the other CTAs do; and the rows need ties from those tiles
    i0 = ORDS_A.index(0)
    v = data_a.columns["tiebound"][i0][0]
    assert int((v[7 * TILE:8 * TILE] >= TIE_K).sum()) >= k
    vals, sos, docs = [], [], []
    for i in range(4):
        d = np.nonzero(data_a.alive[i] & (data_a.columns["tiebound"][i][0] >= TIE_K))[0]
        vals.append(data_a.columns["tiebound"][i][0][d])
        sos.append(np.full(len(d), ORDS_A[i], np.int64))
        docs.append(d)
    vals = np.concatenate(vals)
    rows, _ = sort_rows(vals, np.ones(len(vals), bool), np.concatenate(sos), np.concatenate(docs), "desc", k)
    assert rows[-1][0] == TIE_K and any(r[2] == 0 and r[0] == TIE_K and r[3] < 7 * TILE for r in rows)


# ---- the histogram model against a scalar restatement (no GPU) ---------------------------------------------------------------
def scalar_value(image, kind):
    image = int(image)
    if kind in ("u64", "bool"):
        return float(image)
    if kind in ("i64", "date"):
        return float(image - 2**63)
    bits = image ^ 2**63 if image >= 2**63 else image ^ (2**64 - 1)
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def scalar_pos(v, offset, interval):
    """get_bucket_pos_f64: ((v - offset) / interval).floor() as i64 (Rust's `as`: NaN 0, saturating)."""
    q = (v - offset) / interval
    if q != q:
        return 0
    if q == math.inf:
        return I64_MAX
    if q == -math.inf:
        return I64_MIN
    return max(I64_MIN, min(I64_MAX, math.floor(q)))


def scalar_collect(images, present, kind, interval, offset, hard_min=-FMAX, hard_max=FMAX):
    have = [int(x) for j, x in enumerate(images) if present is None or present[j]]
    lo, hi = hard_min, hard_max
    if have and scalar_value(min(have), kind) >= hard_min and scalar_value(max(have), kind) <= hard_max:
        lo, hi = -FMAX, FMAX
    out = {}
    for x in have:
        v = scalar_value(x, kind)
        if v >= lo and v <= hi:
            p = scalar_pos(v, offset, interval)
            out[p] = out.get(p, 0) + 1
    return out


def edge_cases():
    """(name, u64 images, present or None, kind, interval, offset, hard_min, hard_max): the histogram edges of the GPU tests."""
    d = lambda x: T.fast_value_to_u64(np.asarray(x, np.int64), "date")  # noqa: E731
    i64 = lambda x: T.fast_value_to_u64(np.asarray(x, np.int64), "i64")  # noqa: E731
    day = 86_400 * 10**9
    neg_dates = d(np.arange(-5 * day, 3 * day, 3_600 * 10**9 + 7))
    ext = i64([I64_MIN, I64_MIN + 2048, I64_MIN + 4096, -1, 0, I64_MAX - 4096, I64_MAX - 1024, I64_MAX])
    big = np.uint64(2**60) + np.arange(0, 600, 3, dtype=np.uint64)
    together = np.uint64(2**60) + np.arange(128, dtype=np.uint64)  # (f64 spacing 256 there: every one rounds to 2^60)
    specials = T.fast_value_to_u64(F64_SPECIAL, "f64")
    return [
        ("negative dates by the hour", neg_dates, None, "date", 3_600e9, 0.0, -FMAX, FMAX),
        ("negative dates by the day, offset -1.5 days", neg_dates, None, "date", float(day), -1.5 * day, -FMAX, FMAX),
        ("offset larger than the interval", i64(np.arange(-300, 300)), None, "i64", 7.0, 123.5, -FMAX, FMAX),
        ("offset far below the interval", i64(np.arange(-300, 300)), None, "i64", 7.0, -1e6 - 0.25, -FMAX, FMAX),
        ("pos saturates at i64::MAX", ext[5:], None, "i64", 1.0, 0.0, 0.0, FMAX),
        ("pos saturates at i64::MIN", ext[:3], None, "i64", 1.0, 4096.0, -FMAX, 0.0),
        ("i64 extremes by 2^60", ext, None, "i64", 2.0**60, 0.0, -FMAX, FMAX),
        ("u64 above 2^53 rounding together", together, None, "u64", 1.0, 0.0, -FMAX, FMAX),
        ("u64 above 2^53 at 256", big, None, "u64", 256.0, 0.0, -FMAX, FMAX),
        ("f64 specials in bounds", specials, None, "f64", 0.5, 0.0, -10.0, 10.0),
        ("f64 specials, half present", specials, np.arange(len(specials)) % 2 == 0, "f64", 1e307, 0.0, -FMAX, FMAX),
        ("one bucket out of bounds", np.array([5, 15, 25, 15, 5], np.uint64), None, "u64", 100.0, 0.0, 10.0, 20.0),
    ]


@pytest.mark.parametrize("case", edge_cases(), ids=lambda c: c[0])
def test_histogram_model_against_scalar_restatement(case):
    _, images, present, kind, interval, offset, lo, hi = case
    want = scalar_collect(images, present, kind, interval, offset, lo, hi)
    assert HM.collect(images, present, None, kind, interval, offset, lo, hi) == want
    assert want  # (every case keeps some value)


def test_saturating_cases_span_few_buckets():
    """The saturating ranges stay within 2^20 buckets (the device takes them); i64 extremes at interval 1 do not."""
    for name, images, present, kind, interval, offset, lo, hi in edge_cases():
        pos = list(scalar_collect(images, present, kind, interval, offset, lo, hi))
        if "saturates" in name:
            assert max(pos) - min(pos) + 1 <= SMEM_BINS + 1 and (I64_MAX in pos or I64_MIN in pos)
    ext = edge_cases()[6][1]
    pos = list(scalar_collect(ext, None, "i64", 1.0, 0.0))
    assert max(pos) - min(pos) + 1 > MAX_BINS


def test_cut_model_equals_fixture_model():
    """model() (each segment cut to its own top k first) equals Fixture.model on test_gpu_sort_field's fixture."""
    fx = Fixture()
    qts = [fx.query(TQ_OP_TERM, [0], 10), fx.query(TQ_OP_OR, [0, 4], 10), fx.query(TQ_OP_TERM, [ALL], 10)]
    for kind in ("few", "half", "equal", "uniform"):
        for qt in qts:
            for o in ORDERS:
                for k in (1, 7, 1000):
                    assert model(fx, qt, kind, o, k) == fx.model(qt, kind, o, k)
                    assert model(fx, qt, kind, o, k, masks=fx.filters["bern30"]) == fx.model(qt, kind, o, k, masks=fx.filters["bern30"])


# ---- Fixture A on the device -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fxa():
    return FixtureA()


@pytest.fixture(scope="module")
def ctx_a(fxa):
    c = fxa.register(T.Context(0))
    yield c
    c.close()


SORT_ALL_SHAPES = ("uniform", "ts_asc", "sparse", "ties", "tiebound")


@gpu
@pytest.mark.parametrize("kind", KINDS_A)
def test_many_units_every_shape(ctx_a, fxa, kind):
    """Every shape (on five columns; the first twelve on the others) at k 1, 2, 255, 256, 257, 1000, 1023 and 1024 in one batch,
    Desc and Asc, with count_hits; the same rows without it."""
    base = shapes(fxa) if kind in SORT_ALL_SHAPES else shapes(fxa)[:12]
    out, qts = run_sorted(ctx_a, fxa, base, kind)
    out2 = ctx_a.sort_batch(QueryBatch([q for q, _, _, _ in qts]), [(COL_A[kind], o) for _, _, _, o in qts])
    for i in range(len(qts)):
        assert device_rows(out2, i) == device_rows(out, i)


@gpu
@pytest.mark.parametrize("kind,order", [("ts_asc", "desc"), ("ts_desc", "asc")])
def test_many_units_skipping(ctx_a, fxa, kind, order):
    """A timestamp sorted against its doc order skips tiles over many units; the rows stay the model's."""
    base = [fxa.query(TQ_OP_TERM, [ALL], 10), fxa.query(TQ_OP_OR, [0, 5], 10), fxa.query(TQ_OP_AND, [0, 1], 10)]
    s0 = ctx_a.stats()
    run_sorted(ctx_a, fxa, base, kind, orders=(order,), count_hits=False)
    s1 = ctx_a.stats()
    assert s1["sort_tiles_skipped"] > s0["sort_tiles_skipped"]


@gpu
@pytest.mark.parametrize("fkind", FILTER_KINDS)
def test_many_units_filters(ctx_a, fxa, fkind):
    """Every filter kind on a subset of the shapes: sort (three columns) and histogram rows over alive AND filter."""
    fid = 200 + FILTER_KINDS.index(fkind)
    base = shapes(fxa)[::4]
    masks = fxa.filters[fkind]
    for kind in ("sparse", "ties", "ts_asc"):
        run_sorted(ctx_a, fxa, base, kind, ks=(1, 256, 1024), masks=masks, extra=dict(filter=fid))
    qts = [(dict(q, filter=fid), t) for q, t in base]
    run_hist(ctx_a, fxa, qts, "window", 1.0, 0.0, masks=masks)


@gpu
def test_ties_behind_the_bound(ctx_a, fxa):
    """`tiebound` Desc: the rows hold exactly the lowest-address ties of the k-th value, which sit in units ordered after the bound
    is set and in the first tiles of a backward unit.  For the `all` query that unit sets its own bound to the tie value from its
    last tile, the first it reads, so its tiles 0-6 are read at that bound whatever the other CTAs do."""
    base = [fxa.query(TQ_OP_TERM, [ALL], 10), fxa.query(TQ_OP_OR, [0, 1], 10), fxa.query(TQ_OP_TERM, [0], 10)]
    out, qts = run_sorted(ctx_a, fxa, base, "tiebound", ks=(1000, 1024), orders=("desc",), count_hits=False)
    rows = device_rows(out, 1)
    assert rows[-1][0] == TIE_K and any(r[2] == 0 and r[0] == TIE_K and r[3] < 7 * TILE for r in rows)


@gpu
def test_rows_of_none_docs_only(ctx_a, fxa):
    """`sparse` through filter NOVALUE: no matching doc has a value, so every row is a None doc, and at k = 1024 the row is the
    first k None docs of the lowest ordinal's first unit -- all k of the ones it hands over -- picked from more None candidates
    than k_sort_final holds on chip."""
    base = [fxa.query(TQ_OP_TERM, [ALL], 10), fxa.query(TQ_OP_OR, [0, 4], 10), fxa.query(TQ_OP_TERM, [0], 10),
            fxa.query(TQ_OP_AND, [0, ALL], 10), fxa.query(TQ_OP_TERM, [EDGE], 10)]
    out, qts = run_sorted(ctx_a, fxa, base, "sparse", masks=fxa.novalue, extra=dict(filter=NOVALUE))
    rows = device_rows(out, [i for i, (q, _, b, o) in enumerate(qts) if b == 0 and q["k"] == TQ_MAX_K][0])
    assert len(rows) == TQ_MAX_K and not any(r[1] for r in rows) and {r[2] for r in rows} == {0}


HIST_A = [("window", 1.0, 0.0, -FMAX, FMAX), ("window", 1.0, 0.0, 0.0, 5000.0), ("ts_asc", 1e6, 0.0, -FMAX, FMAX),
          ("ts_desc", 3e6, -1.5e6, -FMAX, FMAX), ("i64ext", 2.0**60, 0.0, -FMAX, FMAX), ("f64ext", 1.0, 0.0, -100.0, 100.0),
          ("sparse", 100.0, 0.0, -FMAX, FMAX), ("tiebound", 1000.0, 0.0, 60.0, 150.0)]


@gpu
@pytest.mark.parametrize("spec", HIST_A, ids=lambda s: f"{s[0]}-{s[1]}-{s[3]}")
def test_many_units_histogram(ctx_a, fxa, spec):
    """Every shape (the first twelve for the columns without window edges) per spec.  `window`: units of 4096 buckets (shared
    memory) and of 9000 (global counters) count into one query's counters; with hard bounds [0, 5000] the segments of ordinals 5000
    and 0 collapse their bounds and the others do not.  `tiebound` in [60, 150]: tiles of one value out of bounds."""
    kind, interval, offset, lo, hi = spec
    qts = shapes(fxa) if kind in ("window", "ts_asc") else shapes(fxa)[:12]
    run_hist(ctx_a, fxa, qts, kind, interval, offset, lo, hi)


@gpu
def test_unaligned_doc_ranges(fxa):
    """Segment of ordinal 5000 split at 8191 and 3 * 8192 + 17, one context each (unfiltered and through a filter view): merged
    sort rows equal the whole segment's, summed histogram rows equal the model and the hits add up."""
    seg = fxa.osegs[0]
    cuts = (0, 8191, 3 * 8192 + 17, seg.max_doc)
    parts = []
    try:
        for lo, hi in zip(cuts, cuts[1:]):
            c = T.Context(0)
            parts.append(c)
            seg.register(c)
            c.segment_set_doc_range(seg.segment_ord, 0, lo, hi)
            c.filter_register(7, seg.segment_ord, packed(fxa.filters["bern30"][0]))
            for kind in ("sparse", "ties", "window"):
                fxa.register_column(c, kind, segs={0})
        for filt in (False, True):
            masks = fxa.filters["bern30"] if filt else None
            extra = dict(filter=7) if filt else {}
            base = [fxa.query(TQ_OP_OR, [0, 4, EDGE], 10), fxa.query(TQ_OP_TERM, [ALL], 10), fxa.query(TQ_OP_AND, [EDGE, ALL], 10)]
            base = [(dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] == seg.segment_ord], **extra), t) for q, t in base]
            for kind in ("sparse", "ties"):
                qts = [(dict(q, k=k), t, o) for q, t in base for k in (1, 257, 1024) for o in ORDERS]
                qb = QueryBatch([q for q, _, _ in qts])
                outs = [c.sort_batch(qb, [(COL_A[kind], o) for _, _, o in qts], count_hits=True) for c in parts]
                for i, (q, t, o) in enumerate(qts):
                    rows = [r for out in outs for r in device_rows(out, i)]
                    merged, _ = sort_rows(np.array([r[0] for r in rows], np.uint64), np.array([r[1] for r in rows], bool),
                                          np.array([r[2] for r in rows]), np.array([r[3] for r in rows]), o, q["k"])
                    want, n = model(fxa, (q, t), kind, o, q["k"], masks=masks, segs={0})
                    assert merged == want, (kind, o, q["k"], t, filt)
                    assert sum(int(out[5][i]) for out in outs) == n
            qb = QueryBatch([q for q, _ in base])
            outs = [c.histogram_batch(qb, [(COL_A["window"], "i64", 1.0, 0.0)] * len(base), count_hits=True) for c in parts]
            for i, qt in enumerate(base):
                got = sorted(Hg.merge_intermediate(hrows(o, i) for o in outs).items())
                assert got == hmodel(fxa, qt, "window", 1.0, 0.0, masks=masks, segs={0})
                assert sum(int(o[3][i]) for o in outs) == sum(int(c.count_batch(QueryBatch([qt[0]]))[0]) for c in parts)
    finally:
        for c in parts:
            c.close()


# ---- histogram caps and semantics on small segments ----------------------------------------------------------------------------
def all_segment(c, max_doc, ordinal=1):
    s = OracleSegment([(np.arange(max_doc, dtype=np.uint32), np.ones(max_doc, np.uint32))], [1] * max_doc, segment_ord=ordinal,
                      writer_cls=T.FieldWriter)
    s.register(c)
    return s


@gpu
def test_histogram_bucket_and_counter_caps():
    """A query of exactly 2^20 buckets is taken and equals the model; 2^20 + 1 is refused (-4).  128 such queries -- 2^27
    counters, 1 GiB of device scratch, and 2 GiB of rows -- are taken; one counter more is refused (-1)."""
    c = T.Context(0)
    try:
        s = all_segment(c, MAX_BINS)
        v = T.fast_value_to_u64(np.arange(MAX_BINS, dtype=np.int64), "i64")
        c.sort_column_register(1, s.segment_ord, v)
        w = v.copy()
        w[-1] = T.fast_value_to_u64(np.array([MAX_BINS], np.int64), "i64")[0]
        c.sort_column_register(2, s.segment_ord, w)
        q = make_query(TQ_OP_TERM, [s], [0], 10)
        out = c.histogram_batch(QueryBatch([q]), [(1, "i64", 1.0, 0.0)], count_hits=True, stride=MAX_BINS)
        assert hrows(out, 0) == sorted(HM.collect(v, None, None, "i64", 1.0, 0.0).items()) and int(out[3][0]) == MAX_BINS
        assert code(lambda: c.histogram_batch(QueryBatch([q]), [(2, "i64", 1.0, 0.0)])) == -4
        n = MAX_COUNTERS // MAX_BINS
        pos, cnt, nb = c.histogram_batch(QueryBatch([q] * n), [(1, "i64", 1.0, 0.0)] * n, stride=MAX_BINS)
        assert (nb == MAX_BINS).all()
        assert np.array_equal(pos[0], np.arange(MAX_BINS)) and (cnt == 1).all() and (pos == pos[0]).all()
        del pos, cnt
        specs = [(1, "i64", 1.0, 0.0)] * n + [(1, "i64", 1.0, 0.0, 0.0, 0.0)]
        assert code(lambda: c.histogram_batch(QueryBatch([q] * (n + 1)), specs, stride=1)) == -1
        one = c.histogram_batch(QueryBatch([q]), [specs[-1]])
        assert hrows(one, 0) == [(0, 1)]
    finally:
        c.close()


@pytest.fixture(scope="module")
def edge_ctx():
    """Two segments of 3 tiles + 5 docs: every edge case's values cycled over the first, the second all in one tile (one bucket
    per tile wherever the values allow)."""
    cases = edge_cases()
    c = T.Context(0)
    segs = [all_segment(c, 3 * TILE + 5, ordinal=o) for o in (11, 3)]
    data = []
    for j, (name, images, present, kind, interval, offset, lo, hi) in enumerate(cases):
        cols = []
        for si, s in enumerate(segs):
            idx = np.arange(s.max_doc) % len(images) if si == 0 else np.minimum(np.arange(s.max_doc) // TILE, len(images) - 1)
            p = None if present is None else np.asarray(present, bool)[idx]
            cols.append((np.asarray(images, np.uint64)[idx].copy(), p))
            c.sort_column_register(50 + j, s.segment_ord, cols[-1][0], None if p is None else packed(p))
        data.append(cols)
    yield c, segs, cases, data
    c.close()


@gpu
def test_histogram_edge_values(edge_ctx):
    """Negative dates, |offset| > interval, pos saturating at either end within an accepted range, i64 extremes, u64 above 2^53
    that round to one f64 (a tile of distinct images in one bucket), f64 specials, tiles of one bucket out of bounds: the device
    equals the model over both segments, each on its own and together."""
    c, segs, cases, data = edge_ctx
    for j, (name, images, present, kind, interval, offset, lo, hi) in enumerate(cases):
        for use in ((0,), (1,), (0, 1)):
            q = make_query(TQ_OP_TERM, [segs[i] for i in use], [0], 10)
            s0 = c.stats()
            out = c.histogram_batch(QueryBatch([q]), [(50 + j, kind, interval, offset, lo, hi)], count_hits=True)
            s1 = c.stats()
            want = sorted(HM.merge([HM.collect(*data[j][i], None, kind, interval, offset, lo, hi) for i in use]).items())
            assert hrows(out, 0) == want, (name, use)
            assert int(out[3][0]) == sum(segs[i].max_doc for i in use)
            if name == "u64 above 2^53 rounding together" and use == (0,):  # 128 distinct images a tile, one bucket: no gather
                assert len(np.unique(data[j][0][0][:TILE])) == 128 and want == [(2**60, segs[0].max_doc)]
                assert s1["hist_tiles_one_bucket"] - s0["hist_tiles_one_bucket"] == tiles_of(segs[0].max_doc)


@gpu
def test_bound_collapse_differs_per_segment(edge_ctx):
    """One query, two segments: one column inside the hard bounds (collapsed), the other not -- in both plan orders."""
    c, segs, _, _ = edge_ctx
    inside = T.fast_value_to_u64(np.arange(segs[0].max_doc) % 50 + 10, "i64")
    outside = T.fast_value_to_u64(np.arange(segs[0].max_doc) % 90 - 20, "i64")
    for col, (a, b) in ((90, (inside, outside)), (91, (outside, inside))):
        c.sort_column_register(col, segs[0].segment_ord, a)
        c.sort_column_register(col, segs[1].segment_ord, b)
        q = make_query(TQ_OP_TERM, segs, [0], 10)
        for interval, offset in ((1.0, 0.0), (7.0, 0.5)):
            out = c.histogram_batch(QueryBatch([q]), [(col, "i64", interval, offset, 0.0, 60.0)])
            want = sorted(HM.merge([HM.collect(x, None, None, "i64", interval, offset, 0.0, 60.0) for x in (a, b)]).items())
            assert hrows(out, 0) == want


# ---- doc ids up to 2^31 - 2 ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def big():
    """One segment of 2^31 - 2 docs (about 17 GiB of device memory; the column's host array is 16 GiB of never-written zero pages
    below its top): four lists and a date column in its top 300 000 docs and at max_doc - 1, 10 % of them without a value, the
    values in runs of 2048 equal ones (the top docs tie, both ways).  The fourth list holds the docs without a value and every
    1000th doc of the top: fewer than k of its docs have a value, so its rows end in None docs."""
    rng = np.random.default_rng(0x7FFF)
    max_doc = 2**31 - 2
    top = max_doc - 300_000
    has = rng.random(max_doc - top) < 0.9
    has[-1] = True
    lists = []
    for p in (0.2, 0.05, 0.01):
        d = np.union1d(top + np.nonzero(rng.random(max_doc - top) < p)[0], [max_doc - 1]).astype(np.uint32)
        lists.append((d, np.ones(len(d), np.uint32)))
    d = (top + np.union1d(np.nonzero(~has)[0], np.arange(0, max_doc - top, 1000))).astype(np.uint32)
    lists.append((d, np.ones(len(d), np.uint32)))
    seg = OracleSegment(lists, None, segment_ord=2**31 + 1, writer_cls=T.FieldWriter, max_doc=max_doc)
    t0 = 1_700_000_000 * 10**9
    top_values = T.fast_value_to_u64(t0 + (np.arange(max_doc - top, dtype=np.int64) // 2048) * 10**9, "date")
    present = np.zeros((max_doc + 7) // 8, np.uint8)
    sel = top + np.nonzero(has)[0]
    np.bitwise_or.at(present, sel >> 3, (1 << (sel & 7)).astype(np.uint8))
    c = T.Context(0)
    seg.register(c)
    values = np.zeros(max_doc, np.uint64)
    values[top:] = top_values
    c.sort_column_register(9, seg.segment_ord, values, present)
    del values
    qs = [(make_query(TQ_OP_TERM, [seg], [0], 10), lists[0][0]),
          (make_query(TQ_OP_OR, [seg], [0, 1, 2], 10), np.union1d(np.union1d(lists[0][0], lists[1][0]), lists[2][0])),
          (make_query(TQ_OP_AND, [seg], [0, 1], 10), np.intersect1d(lists[0][0], lists[1][0])),
          (make_query(TQ_OP_TERM, [seg], [3], 10), lists[3][0])]
    yield types.SimpleNamespace(ctx=c, seg=seg, top=top, top_values=top_values, has=has, qs=qs, max_doc=max_doc, t0=t0)
    c.close()


@gpu
def test_big_segment_sort(big):
    """Sort on the 2^31 - 2 doc segment, Desc and Asc, k 10 and 1024: packed addresses, None docs and value gathers near 2^31.
    The fourth query's rows at k = 1024 end in None docs."""
    qts = [(dict(q, k=k), docs, o) for q, docs in big.qs for k in (10, TQ_MAX_K) for o in ORDERS]
    qb = QueryBatch([q for q, _, _ in qts])
    out = big.ctx.sort_batch(qb, [(9, o) for _, _, o in qts], count_hits=True)
    assert np.array_equal(out[5], big.ctx.count_batch(qb))
    for i, (q, docs, o) in enumerate(qts):
        d = docs.astype(np.int64)
        pr = big.has[d - big.top]
        vals = np.where(pr, big.top_values[d - big.top], np.uint64(0))
        want, n = sort_rows(vals, pr, np.full(len(d), big.seg.segment_ord, np.int64), d, o, q["k"])
        assert device_rows(out, i) == want, (i, o, q["k"])
        assert int(out[5][i]) == n
    for i, (q, docs, o) in enumerate(qts):
        if docs is big.qs[3][1] and q["k"] == TQ_MAX_K:
            rows = device_rows(out, i)
            assert len(rows) == TQ_MAX_K and 0 < sum(not r[1] for r in rows) < TQ_MAX_K and min(r[3] for r in rows) >= big.top


@gpu
def test_big_segment_histogram(big):
    qb = QueryBatch([q for q, _ in big.qs])
    for interval, offset, lo, hi in ((1e9, 0.0, -FMAX, FMAX), (3600e9, -1800e9, -FMAX, FMAX), (60e9, 0.0, big.t0 + 2e10, big.t0 + 1e11)):
        out = big.ctx.histogram_batch(qb, [(9, "date", interval, offset, lo, hi)] * len(big.qs), count_hits=True)
        for i, (_, docs) in enumerate(big.qs):
            m = np.zeros(big.max_doc - big.top, bool)
            m[docs.astype(np.int64) - big.top] = True
            want = sorted(HM.collect(big.top_values, big.has, m, "date", interval, offset, lo, hi).items())
            assert hrows(out, i) == want and want, (interval, i)
            assert int(out[3][i]) == len(docs)


# ---- clauses across fields ---------------------------------------------------------------------------------------------------
class MultiFieldFixture(Fixture):
    """Fixture's has() / model() over the ordinals of tests/multi_field.py, one column per ordinal."""

    def __init__(self):
        self.ix = MF.Index(writer_cls=T.FieldWriter)
        rng = np.random.default_rng(0x3F)
        self.osegs = [types.SimpleNamespace(segment_ord=o.ordinal, max_doc=o.max_doc) for o in self.ix.ords]
        self.models = self.ix.models()
        self.alive = [np.ones(o.max_doc, bool) if o.alive is None else unpacked(o.alive, o.max_doc) for o in self.ix.ords]
        self.columns = {"mf": [(rng.integers(0, 40, size=o.max_doc).astype(np.uint64), rng.random(o.max_doc) < 0.9) for o in self.ix.ords]}
        self._has = {}


@gpu
def test_clauses_across_fields():
    """The multi-field battery's queries whose clauses name several fields: sort (Desc and Asc) and histogram rows equal the model
    over M._segment_matches, hits equal tq_count_batch."""
    fx = MultiFieldFixture()
    qts = [qt for qt in MF.battery(fx.ix, phrase=False) if len({ts[2] for ts in qt[0]["term_segs"]}) > 1]
    assert len(qts) > 20
    c = fx.ix.register(T.Context(0))
    try:
        for i, o in enumerate(fx.ix.ords):
            v, p = fx.columns["mf"][i]
            c.sort_column_register(77, o.ordinal, v, packed(p))
        qb = QueryBatch([q for q, _ in qts] * 2)
        orders = ["desc"] * len(qts) + ["asc"] * len(qts)
        out = c.sort_batch(qb, [(77, o) for o in orders], count_hits=True)
        counts = c.count_batch(qb)
        assert np.array_equal(out[5], counts)
        for i, o in enumerate(orders):
            qt = qts[i % len(qts)]
            want, n = fx.model(qt, "mf", o, qt[0]["k"])
            assert device_rows(out, i) == want, (i, o, qt[1])
            assert int(out[5][i]) == n
        hq = QueryBatch([q for q, _ in qts])
        out = c.histogram_batch(hq, [(77, "u64", 3.0, 1.0)] * len(qts), count_hits=True)
        assert np.array_equal(out[3], counts[:len(qts)])
        for i, qt in enumerate(qts):
            parts = [HM.collect(*fx.columns["mf"][j], fx.has(j, qt) & fx.alive[j], "u64", 3.0, 1.0) for j in range(len(fx.osegs))]
            assert hrows(out, i) == sorted(HM.merge(parts).items()), (i, qt[1])
    finally:
        c.close()


# ---- holds and concurrency ---------------------------------------------------------------------------------------------------
@gpu
def test_concurrent_runs_on_one_context(ctx_a, fxa):
    """Six threads on one context, each looping sort, histogram, count and search batches over a column of its own and the shared
    ones: every result equals the single-threaded run.  Afterwards every column re-registers and unregisters."""
    base = [fxa.query(TQ_OP_OR, [0, 3], 10), fxa.query(TQ_OP_AND, [0, EDGE], 10), fxa.query(TQ_OP_TERM, [ALL], 10)]
    qb = QueryBatch([dict(q, k=k) for q, _ in base for k in (10, 1024)])
    own = ("ts_asc", "ts_desc", "sparse", "i64ext", "f64ext", "tiebound")

    def flat(res):
        sort, hist, count, search = res
        return ([device_rows(sort, i) for i in range(qb.nq)], sort[5].tolist(), [hrows(hist, i) for i in range(qb.nq)], hist[3].tolist(),
                count.tolist(), [x.tolist() for x in search])

    def work(t):
        kinds = (own[t], "uniform", "ties")
        res = [ctx_a.sort_batch(qb, [(COL_A[kinds[j % 3]], ORDERS[(j + t) % 2]) for j in range(qb.nq)], count_hits=True)]
        res.append(ctx_a.histogram_batch(qb, [(COL_A[k], HKIND[k], 1.0, 0.0) for k in ("window", "window", "ties") * 2], count_hits=True))
        res.append(ctx_a.count_batch(qb))
        res.append(ctx_a.search_batch(qb))
        return res

    want = [flat(work(t)) for t in range(6)]
    errors, got = [], {}

    def loop(t):
        try:
            for it in range(3):
                got[(t, it)] = flat(work(t))
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=loop, args=(t,)) for t in range(6)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert len(got) == 18 and all(res == want[t] for (t, _), res in got.items())
    for t in range(6):  # the reference run itself: the sort rows of the thread's own column against the model
        assert want[t][0][0] == model(fxa, base[0], own[t], ORDERS[t % 2], 10)[0]
    for k in KINDS_A:
        fxa.register_column(ctx_a, k, segs={2})
        fxa.register_column(ctx_a, k, col_id=COL_A[k] + 1000, segs={2})
        ctx_a.sort_column_unregister(COL_A[k] + 1000)


@gpu
def test_holds_released_after_failures(ctx_a, fxa):
    """A missing column at query 1, a phrase at query 1, k = 0, a refused 2^20 range and the out_stride failure after the run: each
    leaves no hold, so the columns it named re-register."""
    q, _ = fxa.query(TQ_OP_TERM, [ALL], 10)
    ok = (COL_A["ties"], "desc")
    phrase = dict(q, op=3, term_pos=[(0, 0)] * len(q["term_segs"]), term_offset=[0])
    hs = (COL_A["window"], "i64", 1.0, 0.0)
    fails = [(lambda: ctx_a.sort_batch(QueryBatch([q, q]), [ok, (999, "desc")]), -3),
             (lambda: ctx_a.sort_batch(QueryBatch([q, phrase]), [ok, ok]), -4),
             (lambda: ctx_a.sort_batch(QueryBatch([q, dict(q, k=0)]), [ok, ok]), -1),
             (lambda: ctx_a.histogram_batch(QueryBatch([q, q]), [hs, (999, "i64", 1.0, 0.0)]), -3),
             (lambda: ctx_a.histogram_batch(QueryBatch([q, phrase]), [hs, hs]), -4),
             (lambda: ctx_a.histogram_batch(QueryBatch([q, q]), [hs, (COL_A["uniform"], "u64", 1.0, 0.0)]), -4)]
    for fn, rc in fails:
        assert code(fn) == rc
        for k in ("ties", "window", "uniform"):
            fxa.register_column(ctx_a, k, segs={1})
    spec = np.zeros(1, HISTOGRAM_SPEC_DTYPE)
    spec[0] = (COL_A["window"], 1, 1.0, 0.0, -FMAX, FMAX)
    pos, cnt, n = np.zeros((1, 4), np.int64), np.zeros((1, 4), np.uint64), np.zeros(1, np.uint32)
    rc = LIB.tq_histogram_batch(ctx_a.h, QueryBatch([q]).ptr, spec.ctypes.data_as(C.POINTER(HistogramSpec)), 1, 4,
                                pos.ctypes.data_as(C.POINTER(C.c_int64)), ptr(cnt, u64p), ptr(n, u32p), None)
    assert rc == -1 and int(n[0]) == 9000
    fxa.register_column(ctx_a, "window", segs={1})


@gpu
def test_lengths_only_call(ctx_a, fxa):
    """out_stride = 0: -1 with every row length written; a second call at the widest length returns the model's rows."""
    base = [fxa.query(TQ_OP_TERM, [ALL], 10), fxa.query(TQ_OP_AND, [0, EDGE], 10), fxa.query(TQ_OP_OR, [2, 4], 10)]
    qb = QueryBatch([q for q, _ in base])
    spec = np.zeros(3, HISTOGRAM_SPEC_DTYPE)
    for i in range(3):
        spec[i] = (COL_A["window"], 1, 1.0, 0.0, -FMAX, FMAX)
    n = np.full(3, 0xFFFFFFFF, np.uint32)
    rc = LIB.tq_histogram_batch(ctx_a.h, qb.ptr, spec.ctypes.data_as(C.POINTER(HistogramSpec)), 3, 0, None, None, ptr(n, u32p), None)
    want = [hmodel(fxa, qt, "window", 1.0, 0.0) for qt in base]
    assert rc == -1 and [int(x) for x in n] == [len(w) for w in want]
    w = int(n.max())
    pos, cnt, n2 = np.zeros((3, w), np.int64), np.zeros((3, w), np.uint64), np.zeros(3, np.uint32)
    rc = LIB.tq_histogram_batch(ctx_a.h, qb.ptr, spec.ctypes.data_as(C.POINTER(HistogramSpec)), 3, w,
                                pos.ctypes.data_as(C.POINTER(C.c_int64)), ptr(cnt, u64p), ptr(n2, u32p), None)
    assert rc == 0
    for i in range(3):
        assert hrows((pos, cnt, n2), i) == want[i]


@gpu
def test_collectors_keep_to_their_own_stats(ctx_a, fxa):
    """A histogram run changes no non-timing tq_stats field and grows units_hist by its units + nq; a sort run leaves the
    histogram stats unchanged."""
    q, _ = fxa.query(TQ_OP_TERM, [ALL], 10)
    qb = QueryBatch([q, q])
    units = sum(len(unit_ranges(n)) for n in SIZES_A)
    hist = {"hist_ms", "units_hist", "hist_tiles_seen", "hist_tiles_one_bucket"}
    spec = [(COL_A["window"], "i64", 1.0, 0.0)] * 2
    ctx_a.histogram_batch(qb, spec, stride=9000)  # (lists built once; rows of 9000 buckets: one run, no retry)
    ctx_a.sort_batch(qb, [(COL_A["ties"], "desc")] * 2)
    s0 = ctx_a.stats()
    ctx_a.histogram_batch(qb, spec, count_hits=True, stride=9000)
    s1 = ctx_a.stats()
    assert {k: v for k, v in s0.items() if k not in hist and not k.endswith("_ms")} == {k: v for k, v in s1.items() if k not in hist and not k.endswith("_ms")}
    assert s1["units_hist"] - s0["units_hist"] == 2 * units + 2
    assert s1["hist_tiles_seen"] - s0["hist_tiles_seen"] == 2 * sum(tiles_of(n) for n in SIZES_A)
    ctx_a.sort_batch(qb, [(COL_A["ties"], "desc")] * 2, count_hits=True)
    s2 = ctx_a.stats()
    assert {k: s2[k] for k in hist} == {k: s1[k] for k in hist}
    assert s2["units_sort"] - s1["units_sort"] == 2 * units + 2
