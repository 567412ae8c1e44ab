"""The fast-field aggregations (tq_terms_batch, tq_metrics_batch, tq_histogram_metrics_batch, tq_terms_metrics_batch,
tq_range_batch, tq_terms_histogram_batch, tq_histogram_terms_batch) at the edges the small fixture of the per-feature tests does not
reach, against the same models (tests/terms_model.py, metrics_model.py, hist_metrics_model.py, terms_metrics_model.py,
range_model.py, terms_hist_model.py, hist_terms_model.py) over the match sets of tests/score_model.py.

Fixture AG is test_gpu_fast_field_edges' Fixture A (four segments of 0.57M-1.1M docs, 9-17 units of eight 8192-doc tiles each,
deletes in three, ordinals 5000, 1200, 0 and 2^31 + 7 registered in that order) with aggregation columns built so that one query
(the `all` term) has units on both sides of every per-unit threshold: terms key windows of 4096 / 4097 keys (k_terms counters) and
1024 / 1025 (k_terms_order), histogram-with-metrics windows of 128 / 129 buckets with one-bucket runs that cross unit ends, change
bucket mid-unit and end a unit whose window is in global memory, terms-histogram cells of 8192 / 8193 for k_terms_hist and
k_hist_terms; and guard columns whose Σ|v| per (bucket, column) of that query is exactly 2^(53+Q) - 2^Q on one bucket and exactly
2^(53+Q) on another, for Q = 0 (u64), Q = -30 (dyadic f64), Q = -1074 (subnormals only) and Q = 971 (the `53 + Q > 1023` branch:
one total is f64::MAX, the other overflows), through one-value tiles and missing-value copies.

The guard (tantivy_b200.h, metrics.guard) accepts a part exactly when it holds no NaN or +-inf and the exact Σ|v| is below
2^min(53+Q, 1024): the tests without the gpu mark check that claim on seeded value sets summed as the device sums them, and the
device tests take that exact rule, computed from the values, as the expected decision for every (query, bucket, column).  Where the
rule accepts, the sum is exact, so the model's Kahan sum is the exact sum: the device parts are checked against it with numpy, which
lets every shape and filter run through every entry point; the doc-by-doc Python models run on sparse queries whose units have the
same windows as the `all` query.  Under the guard no merged result depends on the order in which a module's run() merges segments
(accepted sums are exact, min and max follow the image order): what the ordinal tests observe is the device rows' u32 order.

Also: a segment of 2^31 - 2 docs (test_gpu_fast_field_edges' `big`) through terms, range with metrics, histogram metrics and terms
metrics, with keys and values in its top tiles and at max_doc - 1."""
import os
import random
import struct
import threading
import types
import zlib
from fractions import Fraction

import numpy as np
import pytest

import tantivy_b200 as T
from tantivy_b200 import hist_terms as HT
from tantivy_b200 import metrics as Mx
from tantivy_b200 import terms_hist as TH
from tantivy_b200._abi import (METRIC_PART_DTYPE, TQ_FAST_DATE, TQ_FAST_F64, TQ_FAST_I64, TQ_FAST_U64, TQ_METRIC_MISSING, TQ_OP_AND, TQ_OP_OR,
                               TQ_OP_TERM, TQ_ORDER_ASC, TQ_ORDER_DESC, TQ_TERMS_BY_COUNT, TQ_TERMS_BY_KEY, TQ_TERMS_BY_METRIC,
                               TQ_TERMS_MISSING_AFTER_MAX, TQ_TERMS_MISSING_IMAGE, TQ_TERMS_MISSING_NONE, TQ_TERMS_ORDER_AVG,
                               TQ_TERMS_ORDER_MAX, TQ_TERMS_ORDER_MIN, TQ_TERMS_ORDER_SUM, QueryBatch)
from tests import metrics_model as MM
from tests import terms_metrics_model as TMM
from tests import terms_model as TM
from tests.test_gpu_fast_field_edges import (NOVALUE, ORDS_A, SIZES_A, TILE, UNIT_TILES, FixtureA, big, code, tiles_of,  # noqa: F401
                                             unit_ranges)
from tests.test_gpu_sort_field import ALL, EDGE, FILTER_KINDS, packed, shapes

gpu = pytest.mark.gpu

TERMS_SMEM, ORDER_SMEM, TM_SMEM_SLOTS, HM_SMEM_BINS, TH_SMEM_CELLS = 4096, 1024, 128, 128, 8192
TERMS_MAX_KEYS, HM_MAX_BINS = 1 << 20, 1 << 16
UNIT_DOCS = TILE * UNIT_TILES
INT32_MAX = 2**31 - 1
# guard classes: (column kind, Q); B = 2^53 units of 2^Q is the bound 2^(53+Q)
CLASSES = {"q0": ("u64", 0), "qn": ("f64", -30), "qs": ("f64", -1074), "qb": ("f64", 971)}
B = 1 << 53
BUCKET_TARGETS = (B - 1, B, B // 4 + 1, B + 3)  # per gk value: at the bound less one quantum, at the bound, below, above
GK_BUCKETS = 4


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def quantum_exp(x):
    """metric_quantum_exp (tq_layout.h) of a finite non-zero |x|: the exponent of its lowest set bit."""
    bits = _bits(abs(x))
    e, m = bits >> 52, bits & ((1 << 52) - 1)
    if e:
        m |= 1 << 52
    return (e - 1075 if e else -1074) + ((m & -m).bit_length() - 1)


def exact_rule(values):
    """(accept, exact signed sum as a Fraction or None) of the guard's exact rule over f64 values: no NaN or +-inf, and the
    exact Σ|v| below 2^min(53 + Q, 1024), Q the least quantum_exp of the non-zero values."""
    v = np.asarray(values, np.float64)
    if not np.isfinite(v).all():
        return False, None
    u, c = np.unique(v, return_counts=True)
    nz = [(float(x), int(n)) for x, n in zip(u, c) if x != 0.0]
    if not nz:
        return True, Fraction(0)
    q = min(quantum_exp(x) for x, _ in nz)
    mag = sum(Fraction(abs(x)) * n for x, n in nz)
    return mag < Fraction(2) ** min(53 + q, 1024), sum(Fraction(x) * n for x, n in nz)


def f64_of(images, kind):
    images = np.asarray(images, np.uint64)
    if kind == "f64":
        high = np.uint64(1 << 63)
        return np.where(images >= high, images ^ high, ~images).view(np.float64)
    if kind in ("i64", "date"):
        return (images ^ np.uint64(1 << 63)).view(np.int64).astype(np.float64)
    return images.astype(np.float64)


# ---- the guard columns ---------------------------------------------------------------------------------------------------------
def guard_units(rng, groups, collected, present, targets, tile_of, one_tiles, missing_k=None):
    """Per segment the integer multiples k of 2^Q (and signs) of a guard column: every doc of group g gets a filler that is an even
    multiple (so it does not set Q), the docs of the tiles in one_tiles one shared value per tile, and a few collected docs of each
    group an adjustment that brings the group's exact Σ|v| over the collected docs (missing copies of missing_k included) to
    targets[g] exactly; the last adjustment is odd, so Q is the class's own.  Every k stays below 2^51 (subnormal for Q = -1074)."""
    ks = [np.zeros(len(g), np.int64) for g in groups]
    sizes = [int(sum(((g == gi) & c).sum() for g, c in zip(groups, collected))) for gi in range(len(targets))]
    for gi, target in enumerate(targets):
        f = 2
        while 8 * f * sizes[gi] < target:  # fillers of mean 3.5 f, so they add up to 0.22 - 0.44 of the target
            f *= 2
        f //= 4
        rest = 0
        spots = []
        for si, g in enumerate(groups):
            sel = g == gi
            k = f * rng.integers(0, 8, size=len(g))
            tiles = tile_of[si]
            one = sel & np.isin(tiles, one_tiles[si])
            k = np.where(one, f * 4, k)
            ks[si] = np.where(sel, k, ks[si])
            has = sel & collected[si] & (present[si] if present is not None else True)
            rest += int(ks[si][has].sum())
            if missing_k is not None and present is not None:
                rest += missing_k * int((sel & collected[si] & ~present[si]).sum())
            cand = np.nonzero(has & ~one)[0]
            spots += [(si, int(d)) for d in rng.choice(cand, size=min(3, len(cand)), replace=False)]
        assert len(spots) >= 5 and rest < target, (gi, rest, target)
        for si, d in spots:
            rest -= int(ks[si][d])
            ks[si][d] = 0
        r = target - rest
        a = (r // len(spots)) & ~1
        parts = [a] * (len(spots) - 1)
        last = r - sum(parts)
        if last % 2 == 0:  # an even target: one more odd pair keeps the quantum at 2^Q
            parts[0] += 1
            last -= 1
        for (si, d), k in zip(spots, parts + [last]):
            ks[si][d] = k
        assert all(0 <= k < 1 << 51 for k in parts + [last]), (gi, parts, last)
    return ks


def guard_images(ks, kind, q, rng, signed, tile_of):
    """The column's images; f64 values take a random sign per doc, one sign per tile on the tiles of one value."""
    out = []
    for k, t in zip(ks, tile_of):
        if kind == "u64":
            out.append(k.astype(np.uint64))
            continue
        v = np.ldexp(k.astype(np.float64), q)
        if signed:
            flip = np.where(t % 3 == 0, (rng.random(int(t[-1]) + 1) < 0.4)[t], rng.random(len(k)) < 0.4)
            v = np.where(flip, -v, v)
        out.append(T.fast_value_to_u64(v, "f64"))
    return out


class FixtureAG(FixtureA):
    """Fixture A with the aggregation columns: self.kind / self.mcol as the per-feature fixtures have them, so their check()
    helpers run on it.  build=False: the alive bits and columns only (numpy)."""

    def __init__(self, build=True, seed=0xA6):
        super().__init__(build=build)
        rng = np.random.default_rng(seed)
        self.kind, self.missing_k = {}, {}
        cols = {}
        tile_of, groups, one_tiles = [], [], []
        for i, n in enumerate(SIZES_A):
            doc = np.arange(n, dtype=np.int64)
            t, u = doc // TILE, doc // UNIT_DOCS
            j = t % UNIT_TILES
            w4 = np.where(u % 2 == 0, 4096, 4097)
            w1 = np.where(u % 2 == 0, 1024, 1025)
            add = lambda name, kind, v, p=None: cols.setdefault(name, (kind, []))[1].append((v, p))  # noqa: E731
            add("tk", "u64", (1000 * (u % 3) + doc % w4).astype(np.uint64), doc % 97 != 5)
            add("tk1", "u64", (500 * (u % 2) + doc % w1).astype(np.uint64))
            add("tk128", "u64", (doc % (TM_SMEM_SLOTS if i in (0, 2) else 200)).astype(np.uint64))
            # histogram with metrics: per unit type u % 4 -- 0: 128 buckets (shared); 1: 129 (global), ending in a run of two
            # one-bucket tiles; 2: one bucket on tiles 0-4, another on 5-7; 3: that bucket again on tiles 0-1 (the run goes on across
            # the unit end), 100 buckets on 2-4, a far bucket on 5-7 (a global window that ends in a run)
            hm = np.select([u % 4 == 0, u % 4 == 1, u % 4 == 2, u % 4 == 3],
                           [doc % 128,
                            np.where(j < 6, 1000 + doc % 129, 1007),
                            np.where(j < 5, 2000 + u, 2001 + u),
                            np.select([j < 2, j < 5], [2001 + u - 1, 3000 + doc % 100], 3150 + u)])
            add("hmk", "i64", T.fast_value_to_u64(hm, "i64"))
            # terms with histogram: unit windows of 8192 / 8193 / 4096 / 2731 buckets, one key a unit but two on type 3
            thv = np.select([u % 4 == 0, u % 4 == 1, u % 4 == 2], [doc % 8192, doc % 8193, doc % 4096], doc % 2731)
            thk = np.where(u % 4 == 3, 20 + (doc & 1), 10 + u % 3)
            add("thv", "i64", T.fast_value_to_u64(thv, "i64"))
            add("thk", "u64", thk.astype(np.uint64))
            gk = np.where(t % 5 == 4, doc % GK_BUCKETS, (t // 2) % GK_BUCKETS)
            add("gk", "u64", gk.astype(np.uint64))
            add("sz", "f64", T.fast_value_to_u64(np.where(u % 2 == 0, -0.0, 0.0), "f64"))
            add("ints", "u64", rng.integers(0, 1000, size=n).astype(np.uint64), rng.random(n) < 0.9)
            tile_of.append(t)
            groups.append(gk)
            tl = np.arange(tiles_of(n))
            one_tiles.append(tl[(tl % 3 == 0) & (tl % 5 != 4)])  # (the gk value of a tile of t % 5 != 4 is one)
        collected = self.alive
        whole = [np.zeros(n, np.int64) for n in SIZES_A]
        for c, (kind, q) in CLASSES.items():
            signed = kind == "f64"
            ks = guard_units(rng, groups, collected, None, BUCKET_TARGETS, tile_of, one_tiles)
            cols[f"g_{c}"] = (kind, [(v, None) for v in guard_images(ks, kind, q, rng, signed, tile_of)])
            pres = [rng.random(n) > 0.05 for n in SIZES_A]
            mk = 2
            ks = guard_units(rng, groups, collected, pres, BUCKET_TARGETS, tile_of, one_tiles, missing_k=mk)
            cols[f"gm_{c}"] = (kind, [(v, p) for v, p in zip(guard_images(ks, kind, q, rng, signed, tile_of), pres)])
            self.missing_k[f"gm_{c}"] = float(np.ldexp(float(mk), q))
            for name, target in (("w", B - 1), ("x", B)):
                ks = guard_units(rng, whole, collected, None, (target,), tile_of, one_tiles)
                cols[f"{name}_{c}"] = (kind, [(v, None) for v in guard_images(ks, kind, q, rng, signed, tile_of)])
        for name, (kind, per_seg) in cols.items():
            self.columns[name] = per_seg
            self.kind[name] = kind
        self.mcol = {k: 600 + i for i, k in enumerate(cols)}

    def register(self, ctx, filters=FILTER_KINDS, names=None):
        super().register(ctx, kinds=(), filters=filters)
        for k in self.mcol if names is None else names:
            self.register_agg_column(ctx, k)
        return ctx

    def register_agg_column(self, ctx, k, col_id=None, segs=None):
        for i, s in enumerate(self.osegs):
            if segs is None or i in segs:
                v, p = self.columns[k][i]
                ctx.sort_column_register(self.mcol[k] if col_id is None else col_id, s.segment_ord, v, None if p is None else packed(p))

    def missing_image(self, col, i, tspec):
        mode, image = tspec[4], tspec[5]
        if mode == TQ_TERMS_MISSING_NONE:
            return None
        if mode != TQ_TERMS_MISSING_AFTER_MAX:
            return image
        v, p = self.columns[col][i]
        have = v if p is None else v[p]
        return (int(have.max()) if len(have) else 0) + 1

    def selected(self, i, qt, masks=None):
        sel = self.has(i, qt) & self.alive[i]
        return sel if masks is None else sel & masks[i]

    def values(self, name, i, sel, missing=None):
        """The f64 values segment i collects on column `name` over the docs sel, in doc order (and the docs they came from)."""
        v, p = self.columns[name][i]
        f = f64_of(v, self.kind[name])
        if p is None:
            return f[sel], np.nonzero(sel)[0]
        if missing is None:
            return f[sel & p], np.nonzero(sel & p)[0]
        f = np.where(p, f, missing)
        return f[sel], np.nonzero(sel)[0]


def mspec(fx, name, missing=False):
    kind = {"u64": TQ_FAST_U64, "i64": TQ_FAST_I64, "f64": TQ_FAST_F64}[fx.kind[name]]
    if not missing:
        return (fx.mcol[name], kind, 0, 0)
    m = fx.missing_k[name]
    image = int(np.uint64(m)) if fx.kind[name] == "u64" else int(T.fast_value_to_u64(np.array([m]), "f64")[0])
    return (fx.mcol[name], kind, TQ_METRIC_MISSING, image)


def guard_specs(fx, c):
    """The four guard columns of class c as one metrics spec: (name, with missing) per spec column."""
    return [(f"g_{c}", False), (f"gm_{c}", True), (f"w_{c}", False), (f"x_{c}", False)]


def unit_widths(values, present, n, lo_tile=0):
    """[(unit, window width)] of one segment's column over the Count units of an unfiltered query (images are the values)."""
    out = []
    for u, (b, e) in enumerate(unit_ranges(n)):
        v = values[b * TILE:min(n, e * TILE)]
        if present is not None:
            v = v[present[b * TILE:min(n, e * TILE)]]
        out.append((u, int(v.max()) - int(v.min()) + 1 if len(v) else 0))
    return out


# ---- reach checks (numpy and the planner's unit arithmetic; no GPU) ----------------------------------------------------------
@pytest.fixture(scope="module")
def data_ag():
    return FixtureAG(build=False)


def test_fixture_ag_terms_windows_on_both_sides(data_ag):
    """The `all` query's units count `tk` in windows of exactly 4096 keys (shared) and 4097 (global), and `tk1` in windows of 1024
    and 1025 keys (k_terms_order's shared and global accumulators); every segment's span stays under 2^20 keys."""
    for name, pair in (("tk", (TERMS_SMEM, TERMS_SMEM + 1)), ("tk1", (ORDER_SMEM, ORDER_SMEM + 1))):
        widths = set()
        for i, n in enumerate(SIZES_A):
            v, p = data_ag.columns[name][i]
            widths |= {w for _, w in unit_widths(v, p, n)}
            have = v if p is None else v[p]
            assert int(have.max()) - int(have.min()) < TERMS_MAX_KEYS
        assert set(pair) <= widths, (name, sorted(widths))
        assert all(w <= pair[1] for w in widths)


def test_fixture_ag_hist_metrics_windows_and_runs(data_ag):
    """`hmk` at interval 1: windows of 128 (shared) and 129 buckets (global) in one query; one-bucket tiles whose bucket carries
    over a unit end; a bucket change between two one-bucket tiles inside a unit; and a unit with a global window whose last tiles
    are a one-bucket run (its final flush goes to global memory)."""
    widths, across, mid, global_tail = set(), False, False, False
    for i, n in enumerate(SIZES_A):
        v = f64_of(data_ag.columns["hmk"][i][0], "i64")
        one = [v[t * TILE] if (v[t * TILE:(t + 1) * TILE] == v[t * TILE]).all() else None for t in range(tiles_of(n))]
        for u, (b, e) in enumerate(unit_ranges(n)):
            w = v[b * TILE:min(n, e * TILE)]
            width = int(w.max() - w.min()) + 1
            widths.add(width)
            if b > 0 and one[b] is not None and one[b - 1] == one[b]:
                across = True
            mid = mid or any(one[t] is not None and one[t + 1] is not None and one[t] != one[t + 1] for t in range(b, e - 1))
            global_tail = global_tail or (width > HM_SMEM_BINS and e - b >= 2 and one[e - 1] is not None and one[e - 1] == one[e - 2])
    assert {HM_SMEM_BINS, HM_SMEM_BINS + 1} <= widths and across and mid and global_tail


def test_fixture_ag_terms_hist_cells(data_ag):
    """`thk` / `thv` at interval 1: with one kept key per segment (segment_size 1) k_terms_hist's unit windows hold exactly 8192
    and 8193 cells; k_hist_terms' windows (buckets x (keys + 1)) exactly 8192 and 8193."""
    th, ht = set(), set()
    for i, n in enumerate(SIZES_A):
        k = data_ag.columns["thk"][i][0]
        h = f64_of(data_ag.columns["thv"][i][0], "i64")
        for b, e in unit_ranges(n):
            hb, kb = h[b * TILE:min(n, e * TILE)], k[b * TILE:min(n, e * TILE)]
            nb = int(hb.max() - hb.min()) + 1
            th.add(nb)
            ht.add(nb * (int(kb.max()) - int(kb.min()) + 2))
    assert {TH_SMEM_CELLS, TH_SMEM_CELLS + 1} <= th and {TH_SMEM_CELLS, TH_SMEM_CELLS + 1} <= ht


def test_fixture_ag_guard_totals_at_the_bound(data_ag):
    """For the `all` query (every alive doc), per guard class and gk bucket, the exact Σ|v| is 2^(53+Q) - 2^Q, 2^(53+Q), below and
    above it, with Q the class's own; the whole-query columns are at 2^(53+Q) - 2^Q and 2^(53+Q).  Every bucket holds one-value
    tiles of the `all` query (8192 equal values), the gm columns missing copies, and for Q = -1074 every value is subnormal."""
    for c, (kind, q) in CLASSES.items():
        for name, missing in guard_specs(data_ag, c):
            vals, buckets = [], []
            for i in range(4):
                sel = data_ag.alive[i]
                f, docs = data_ag.values(name, i, sel, data_ag.missing_k.get(name) if missing else None)
                vals.append(f)
                buckets.append(data_ag.columns["gk"][i][0][docs].astype(np.int64))
            vals, buckets = np.concatenate(vals), np.concatenate(buckets)
            targets = BUCKET_TARGETS if name[0] == "g" else ((B - 1,) if name[0] == "w" else (B,))
            for b, target in enumerate(targets):
                v = vals if name[0] != "g" else vals[buckets == b]
                nz = v[v != 0]
                assert min(quantum_exp(float(x)) for x in np.unique(np.abs(nz))) == q, (name, b)
                assert sum(Fraction(float(x)) * int(n) for x, n in zip(*np.unique(np.abs(v), return_counts=True))) == Fraction(target) * Fraction(2) ** q
                assert exact_rule(v)[0] == (target < B), (name, b)
                if q == -1074:
                    assert (np.abs(nz) < 2.0**-1022).all()
            if missing:
                assert sum(int((~data_ag.columns[name][i][1] & data_ag.alive[i]).sum()) for i in range(4)) > 1000
        v = data_ag.columns[f"g_{c}"][0][0]
        gk = data_ag.columns["gk"][0][0]
        ones = [t for t in range(tiles_of(SIZES_A[0])) if (v[t * TILE:(t + 1) * TILE] == v[t * TILE]).all() and v[t * TILE] != 0]
        assert {int(gk[t * TILE]) for t in ones} == set(range(GK_BUCKETS))


def test_fixture_ag_signed_zeros_across_units(data_ag):
    """`sz`: -0.0 on the even units and +0.0 on the odd ones, so every gk bucket of the `all` query holds both, from different units."""
    for i, n in enumerate(SIZES_A):
        f = f64_of(data_ag.columns["sz"][i][0], "f64")
        gk = data_ag.columns["gk"][i][0]
        for b in range(GK_BUCKETS):
            neg = np.signbit(f) & (gk == b)
            assert neg.any() and (~np.signbit(f) & (gk == b)).any()
        assert len({bool(np.signbit(f[b * TILE])) for b, _ in unit_ranges(n)}) == 2


def test_fixture_ag_ordinals_and_units(data_ag):
    units = [len(unit_ranges(n)) for n in SIZES_A]
    assert min(units) >= 9 and max(units) == 17 and max(ORDS_A) >= 2**31 and list(ORDS_A) != sorted(ORDS_A)


# ---- the guard's claim (no GPU) ------------------------------------------------------------------------------------------------
def device_part(values, rng, one_runs=True):
    """A tq_metric_part of `values` summed as the device sums them, in a random order: the values split into random tiles, a tile
    of equal values added as one n x v product (k_metrics' one-value tile, and the missing copies), the others value by value,
    each tile's partial added to a random warp, the warps' partials added in a random order, then an atomic add per CTA."""
    part = Mx.empty_parts(1)[0]
    vals = list(values)
    rng.shuffle(vals)
    ctas = []
    while vals:
        take = rng.randint(1, max(1, len(vals)))
        ctas.append(vals[:take])
        vals = vals[take:]
    order = list(range(len(ctas)))
    rng.shuffle(order)
    total_sum, total_mag = 0.0, 0.0
    q = INT32_MAX
    for ci in order:
        warps = [[0.0, 0.0] for _ in range(rng.randint(1, 4))]
        groups = {}
        for x in ctas[ci]:
            groups.setdefault(_bits(x), []).append(x)
        chunks = []
        for xs in groups.values():
            if one_runs and len(xs) > 1 and rng.random() < 0.5:
                chunks.append(("n", xs[0], len(xs)))
            else:
                chunks += [("n", x, 1) for x in xs]
        rng.shuffle(chunks)
        for _, x, n in chunks:
            if x != x:
                part["n_nan"] += n
                continue
            if abs(x) == float("inf"):
                part["n_inf"] += n
                continue
            w = rng.choice(warps)
            w[0] += float(n) * x
            w[1] += float(n) * abs(x)
            if x != 0.0:
                q = min(q, quantum_exp(x))
        s = m = 0.0
        for w in warps:
            s += w[0]
            m += w[1]
        total_sum += s
        total_mag += m
    part["count"] = len(values)
    part["sum"] = total_sum
    part["magnitude"] = total_mag
    part["quantum_exp"] = q
    return part


def kahan(values):
    return MM.segment_stats(values).sum


def constructed_sets():
    """(name, values, refused sets on which some order must differ) -- the constructions of the fixture's guard columns, small."""
    out = []
    for c, (kind, q) in CLASSES.items():
        e = lambda k: float(np.ldexp(float(k), q))  # noqa: E731
        for label, target in (("bound-1", B - 1), ("bound", B), ("bound+1", B + 1), ("bound+3", B + 3)):
            quarter = (target // 4) & ~1
            pin = 0 if target % 2 else 1  # (an even target: a value of 2^Q keeps the quantum)
            vals = [e(quarter), -e(quarter) if kind == "f64" else e(quarter), e(target - 2 * quarter - pin)] + [e(1)] * pin
            out.append((f"{c} {label}", vals, False))
        # a sum past the bound whose partials round, one order against another
        out.append((f"{c} rounding", [e(1 << 52), e(1 << 52), e(1), e(1)], True))
        # an n x v product that rounds: 3 copies of an odd mantissa near 2^52
        out.append((f"{c} product", [e((1 << 52) + 1)] * 3 + [e(1)] * 2, True))
        # through missing copies: many copies of a small value reaching the bound less one quantum, and at it
        out.append((f"{c} copies bound-1", [e(2)] * 1000 + [e((B - 1) - 2000)], False))
        out.append((f"{c} copies bound", [e(2)] * 1000 + [e(B - 2001), e(1)], False))
    qs = lambda k: float(np.ldexp(float(k), -1074))  # noqa: E731
    out.append(("subnormal mix", [qs(3), qs(5), qs(7), -qs(11)] * 50, False))
    out.append(("nan", [1.0, float("nan")], False))
    out.append(("inf", [1.0, float("inf"), -2.0], False))
    out.append(("zeros", [0.0, -0.0, -0.0], False))
    out.append(("overflow", [1.7976931348623157e308, 1.7976931348623157e308], False))
    return out


def seeded_sets(seed):
    r = np.random.default_rng(seed)
    out = []
    for _ in range(40):
        q = int(r.choice([0, -8, -30, -52, -1074, 900, 971, 975]))
        n = int(r.integers(2, 60))
        scale = int(r.integers(1, 55))
        ks = r.integers(1, 2**min(scale, 52), size=n)
        vals = [float(np.ldexp(float(k), q)) * (1 if r.random() < 0.7 else -1) for k in ks]
        vals = [x for x in vals if np.isfinite(x)]
        if r.random() < 0.3:
            vals += [vals[0]] * int(r.integers(1, 5000))
        out.append((f"seeded {seed} q={q} n={len(vals)}", vals, False))
    return out


@pytest.mark.parametrize("case", constructed_sets() + seeded_sets(1) + seeded_sets(2), ids=lambda c: c[0])
def test_guard_rule_is_exact(case):
    """Over shuffled device-like orders (one-value tiles as n x v, warps, CTAs): metrics.guard accepts exactly when the exact rule
    does; then every order's sum is the model's Kahan sum bit for bit; on the constructed refusals some order differs."""
    name, values, must_differ = case
    rng = random.Random(zlib.crc32(name.encode()))
    accept, exact = exact_rule(values)
    want = kahan(values)
    sums = set()
    for _ in range(24):
        part = device_part(values, rng)
        assert (Mx.guard(part) is None) == accept, (name, part)
        if accept:
            assert _bits(float(part["sum"])) == _bits(want), (name, float(part["sum"]), want)
            assert float(part["sum"]) == float(exact)
        sums.add(_bits(float(part["sum"])))
    if accept:
        assert _bits(want) == _bits(float(exact))
    if must_differ:
        assert not accept and (len(sums) > 1 or _bits(want) not in sums), name


def test_guard_at_the_bound_cannot_round():
    """At Σ|v| = 2^(53+Q) exactly no order rounds (the rule refuses it all the same): every partial sum below the bound is exact,
    and only the whole sum of one sign reaches it."""
    for c, (kind, q) in CLASSES.items():
        vals = [float(np.ldexp(float(k), q)) for k in ((1 << 51), (1 << 51), (1 << 52) - 1, 1)]
        rng = random.Random(7)
        assert not exact_rule(vals)[0]
        got = {_bits(float(device_part(vals, rng)["sum"])) for _ in range(20)}
        assert got == {_bits(kahan(vals))} or q == 971  # (2^1024 overflows: every order gives inf)


# ---- Fixture AG on the device ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fxg():
    return FixtureAG()


@pytest.fixture(scope="module")
def ctx_g(fxg):
    c = fxg.register(T.Context(0))
    yield c
    c.close()


def few_shapes(fx):
    """The `all` term, an OR and an AND."""
    return [fx.query(TQ_OP_TERM, [ALL], 10), fx.query(TQ_OP_OR, [0, 4], 10), fx.query(TQ_OP_AND, [0, ALL], 10)]


def model_shapes(fx):
    """Sparse queries (about 1 % and 0.2 % of the docs) that still match in every tile, so their units have the windows of the
    `all` query: the shapes the doc-by-doc Python models walk."""
    return [fx.query(TQ_OP_OR, [3, 4], 10), fx.query(TQ_OP_TERM, [4], 10)]


def seg_order(fx):
    return sorted(range(len(fx.osegs)), key=lambda i: fx.osegs[i].segment_ord)


def terms_rows(out, q):
    """[(segment_ord, key, doc_count)] of query q of terms_batch's output (terms_metrics_batch's: its n is out[4])."""
    segs, keys, counts, n = out[:3] + (out[4] if out[3].dtype == METRIC_PART_DTYPE else out[3],)
    return [(int(segs[q, j]), int(keys[q, j]), int(counts[q, j])) for j in range(int(n[q]))]


def terms_want(fx, qt, col, target, order, ss, mode=TQ_TERMS_MISSING_NONE, image=0, masks=None, segs=None):
    rows, other, error = [], 0, 0
    for i in seg_order(fx):
        if segs is not None and i not in segs:
            continue
        v, p = fx.columns[col][i]
        mi = fx.missing_image(col, i, (0, 0, 0, 0, mode, image))
        kept, e, o = TM.cut(TM.collect(v, p, fx.selected(i, qt, masks), mi), ss, target == TQ_TERMS_BY_KEY, order == TQ_ORDER_ASC)
        rows += [(fx.osegs[i].segment_ord, k, c) for k, c in kept]
        other, error = other + o, error + e
    return rows, other, error


def run_terms(ctx, fx, qts, specs, masks=None):
    qb = QueryBatch([q for q, _ in qts])
    out = ctx.terms_batch(qb, specs, count_hits=True)
    assert np.array_equal(out[6], ctx.count_batch(qb))
    for qi, (qt, sp) in enumerate(zip(qts, specs)):
        col = next(k for k, v in fx.mcol.items() if v == sp[0])
        want = terms_want(fx, qt, col, sp[1], sp[2], sp[3], *(sp[4:] or ()), masks=masks)
        assert (terms_rows(out, qi), int(out[4][qi]), int(out[5][qi])) == want, (col, sp, qt[1])
    return out


TERMS_SPECS = [(TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 10), (TQ_TERMS_BY_COUNT, TQ_ORDER_ASC, 4097), (TQ_TERMS_BY_KEY, TQ_ORDER_DESC, 1000),
               (TQ_TERMS_BY_KEY, TQ_ORDER_ASC, 1 << 16)]


@gpu
@pytest.mark.parametrize("col", ["tk", "tk1", "thk", "gk"])
def test_terms_many_units_every_shape(ctx_g, fxg, col):
    """Every shape, four orders and segment sizes cut and uncut, in one batch: rows in u32 segment_ord order (2^31 + 7 last), both
    scalars and the hits; on `tk` a missing key inside the key span and one outside it."""
    base = shapes(fxg)
    specs, qts = [], []
    for qt in base:
        for target, order, ss in TERMS_SPECS:
            qts.append(qt)
            specs.append((fxg.mcol[col], target, order, ss))
    if col == "tk":
        for qt in base[::3]:
            for image in (5, 10**6):
                qts.append(qt)
                specs.append((fxg.mcol[col], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 50, TQ_TERMS_MISSING_IMAGE, image))
            qts.append(qt)
            specs.append((fxg.mcol[col], TQ_TERMS_BY_KEY, TQ_ORDER_ASC, 20, TQ_TERMS_MISSING_AFTER_MAX, 0))
    out = run_terms(ctx_g, fxg, qts, specs)
    segs = [s for q in range(len(qts)) for s in dict.fromkeys(int(x) for x in out[0][q, :int(out[3][q])])]
    assert 2**31 + 7 in segs
    for q in range(len(qts)):
        so = [int(x) for x in out[0][q, :int(out[3][q])]]
        assert so == sorted(so)


TQ_KIND = {"u64": TQ_FAST_U64, "i64": TQ_FAST_I64, "f64": TQ_FAST_F64, "date": TQ_FAST_DATE}


def part_of(parts_list):
    return Mx.merge(parts_list)


def check_part(part, vals, what):
    """A device part (merged) against the values it collected: count, min / max images, the guard's decision against the exact rule
    and, when accepted, the sum bit-equal to the exact sum (the model's Kahan sum whenever the rule accepts)."""
    v = np.asarray(vals, np.float64)
    assert int(part["count"]) == len(v), what
    accept, exact = exact_rule(v)
    assert (Mx.guard(part) is None) == accept, (what, int(part["quantum_exp"]), float(part["magnitude"]), accept)
    if accept:
        assert _bits(float(part["sum"])) == _bits(float(exact)), (what, float(part["sum"]), float(exact))
    nn = v[~np.isnan(v)]
    if len(nn):
        lo, hi = float(nn.min()), float(nn.max())
        if lo == 0.0 and np.signbit(nn[nn == 0.0]).any():
            lo = -0.0
        if hi == 0.0 and not np.signbit(nn[nn == 0.0]).all():
            hi = 0.0
        kind = TQ_KIND[what[1]]  # (the u64 and i64 columns here hold values below 2^53: their f64 values are their images)
        assert _bits(Mx.value_of_image(int(part["min_image"]), kind)) == _bits(lo), (what, "min")
        assert _bits(Mx.value_of_image(int(part["max_image"]), kind)) == _bits(hi), (what, "max")
    return accept


def bucket_values(fx, qt, name, missing, key_col, key_of, masks=None):
    """{bucket: f64 values} of column `name` over the docs the query collects, by key_of(images of key_col) per doc."""
    out = {}
    for i in seg_order(fx):
        sel = fx.selected(i, qt, masks)
        f, docs = fx.values(name, i, sel, fx.missing_k.get(name) if missing else None)
        keys = key_of(fx.columns[key_col][i][0][docs])
        for b in np.unique(keys):
            out.setdefault(int(b), []).append(f[keys == b])
    return {b: np.concatenate(v) for b, v in out.items()}


def guard_queries(fx):
    return few_shapes(fx)[:2] + [(dict(fx.query(TQ_OP_TERM, [ALL], 10)[0], filter=200 + FILTER_KINDS.index("bern30")), [ALL])]


def masks_of(fx, qt):
    f = qt[0].get("filter")
    return None if f is None else fx.filters[FILTER_KINDS[f - 200]]


@gpu
@pytest.mark.parametrize("c", list(CLASSES))
def test_guard_at_scale_metrics(ctx_g, fxg, c):
    """tq_metrics_batch: the four guard columns of one class in one spec, many CTAs adding atomically: per (query, column) the
    device accepts exactly where the exact rule does (both totals at the bound for the `all` query), accepted sums bit-exact."""
    cols = guard_specs(fxg, c)
    qts = guard_queries(fxg)
    qb = QueryBatch([q for q, _ in qts])
    parts, hits = ctx_g.metrics_batch(qb, [[mspec(fxg, n, m) for n, m in cols]] * len(qts), count_hits=True)
    assert np.array_equal(hits, ctx_g.count_batch(qb))
    decided = []
    for qi, qt in enumerate(qts):
        for ci, (name, missing) in enumerate(cols):
            vals = np.concatenate([fxg.values(name, i, fxg.selected(i, qt, masks_of(fxg, qt)), fxg.missing_k.get(name) if missing else None)[0]
                                   for i in seg_order(fxg)])
            decided.append(check_part(parts[qi, ci], vals, (name, fxg.kind[name], qi)))
    assert decided[2] and not decided[3]  # the `all` query: w_ at 2^(53+Q) - 2^Q accepted, x_ at 2^(53+Q) refused


HM_GUARD_GRIDS = ((1.0, 0.0), (0.01, 0.0))  # windows of 4 buckets (shared) and of 301 (global) over the same gk buckets


@gpu
@pytest.mark.parametrize("c", list(CLASSES))
def test_guard_at_scale_hist_metrics_and_range(ctx_g, fxg, c):
    """Per (query, bucket, column) of tq_histogram_metrics_batch on gk (shared and global windows, one-bucket runs and straddling
    tiles) and of tq_range_batch on gk: the guard's decision is the exact rule's, accepted sums bit-exact; the range's doc counts
    alone equal its counts with metrics, and the histogram's doc counts equal tq_histogram_batch's."""
    cols = guard_specs(fxg, c)
    ms = [mspec(fxg, n, m) for n, m in cols]
    qts = guard_queries(fxg)
    qb = QueryBatch([q for q, _ in qts])
    seen = set()
    for interval, offset in HM_GUARD_GRIDS:
        hs = (fxg.mcol["gk"], "u64", interval, offset)
        pos, counts, parts, nb, hits = ctx_g.hist_metrics_batch(qb, [hs] * len(qts), [ms] * len(qts), count_hits=True)
        ref = ctx_g.histogram_batch(qb, [hs] * len(qts))
        assert np.array_equal(hits, ctx_g.count_batch(qb))
        for qi, qt in enumerate(qts):
            n = int(nb[qi])
            assert n == int(ref[2][qi]) and np.array_equal(pos[qi, :n], ref[0][qi, :n]) and np.array_equal(counts[qi, :n], ref[1][qi, :n])
            key_of = lambda im: np.floor(im.astype(np.float64) / interval).astype(np.int64)  # noqa: E731
            for ci, (name, missing) in enumerate(cols):
                want = bucket_values(fxg, qt, name, missing, "gk", key_of, masks_of(fxg, qt))
                assert [int(p) for p in pos[qi, :n]] == sorted(want)
                for j in range(n):
                    b = int(pos[qi, j])
                    seen.add((qi, name, int(round(b * interval)), check_part(parts[qi, j, ci], want[b], (name, fxg.kind[name], qi, b))))
    counts_m, parts_r, hits = ctx_g.range_batch(qb, [(fxg.mcol["gk"], [0, 1, 2, 3])] * len(qts), [ms] * len(qts), count_hits=True)
    counts_a, none = ctx_g.range_batch(qb, [(fxg.mcol["gk"], [0, 1, 2, 3])] * len(qts))
    assert none is None and np.array_equal(counts_a, counts_m)
    for qi, qt in enumerate(qts):
        for ci, (name, missing) in enumerate(cols):
            want = bucket_values(fxg, qt, name, missing, "gk", lambda im: im.astype(np.int64), masks_of(fxg, qt))
            for b in range(GK_BUCKETS):
                check_part(parts_r[qi, b, ci], want.get(b, np.zeros(0)), (name, fxg.kind[name], qi, "range", b))
    # the `all` query's g_ columns: bucket 0 (2^(53+Q) - 2^Q) accepted and bucket 1 (2^(53+Q)) refused, on both grids
    for name in (f"g_{c}", f"gm_{c}"):
        assert (0, name, 0, True) in seen and (0, name, 1, False) in seen


@gpu
@pytest.mark.parametrize("c", list(CLASSES))
def test_guard_at_scale_terms_metrics(ctx_g, fxg, c):
    """tq_terms_metrics_batch with gk as the key: per (query, term, column) merged over the segments, the decision is the exact
    rule's and accepted sums are bit-exact; the `_count` rows equal tq_terms_batch's."""
    cols = guard_specs(fxg, c)
    ms = [mspec(fxg, n, m) for n, m in cols]
    qts = guard_queries(fxg)
    qb = QueryBatch([q for q, _ in qts])
    ts = (fxg.mcol["gk"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 10)
    out = ctx_g.terms_metrics_batch(qb, [ts] * len(qts), [ms] * len(qts), count_hits=True)
    ref = ctx_g.terms_batch(qb, [ts] * len(qts))
    for qi, qt in enumerate(qts):
        n = int(out[4][qi])
        assert terms_rows(out, qi) == terms_rows(ref, qi) and (int(out[5][qi]), int(out[6][qi])) == (int(ref[4][qi]), int(ref[5][qi]))
        for ci, (name, missing) in enumerate(cols):
            want = bucket_values(fxg, qt, name, missing, "gk", lambda im: im.astype(np.int64), masks_of(fxg, qt))
            by_key = {}
            for j in range(n):
                by_key.setdefault(int(out[1][qi, j]), []).append(out[3][qi, j, ci])
            assert sorted(by_key) == sorted(want)
            for k, ps in by_key.items():
                check_part(part_of([np.array([p]) for p in ps])[0], want[k], (name, fxg.kind[name], qi, k))


TM_ORDERS = ((TQ_TERMS_ORDER_SUM, "sum"), (TQ_TERMS_ORDER_AVG, "avg"), (TQ_TERMS_ORDER_MIN, "min"), (TQ_TERMS_ORDER_MAX, "max"))


@gpu
@pytest.mark.parametrize("c", list(CLASSES))
def test_guard_decides_the_metric_order(ctx_g, fxg, c):
    """Terms on gk ordered by a guard column's sum / avg (min / max beside them), cut to 2 of 4 keys per segment: the order is
    refused exactly where the exact rule refuses the ordering column over every collected doc (w_ at 2^(53+Q) - 2^Q: accepted; x_
    at 2^(53+Q): refused), and an accepted order cuts as the model does."""
    q_all = fxg.query(TQ_OP_TERM, [ALL], 10)
    for name in (f"w_{c}", f"x_{c}", f"g_{c}"):
        specs = []
        for metric, prop in TM_ORDERS:
            for direction in (TQ_ORDER_DESC, TQ_ORDER_ASC):
                specs.append(((fxg.mcol["gk"], TQ_TERMS_BY_METRIC, direction, 2), (0, metric), prop))
        qb = QueryBatch([q_all[0]] * len(specs))
        out = ctx_g.terms_metrics_batch(qb, [s[0] for s in specs], [[mspec(fxg, name)]] * len(specs), [s[1] for s in specs])
        allv = np.concatenate([fxg.values(name, i, fxg.selected(i, q_all))[0] for i in seg_order(fxg)])
        accept, _ = exact_rule(allv)
        assert accept == (name[0] == "w")
        for qi, (ts, (_, metric), prop) in enumerate(specs):
            opart = out[7][qi]
            if metric in (TQ_TERMS_ORDER_SUM, TQ_TERMS_ORDER_AVG):
                assert (Mx.guard(opart) is None) == accept, (name, prop)
                if not accept:
                    continue
            rows = []
            for i in seg_order(fxg):
                f, docs = fxg.values(name, i, fxg.selected(i, q_all))
                keys = fxg.columns["gk"][i][0][docs].astype(np.int64)
                entries = {}
                for k in range(GK_BUCKETS):
                    st = MM.Stats()
                    v = f[keys == k]
                    ok, exact = exact_rule(v)
                    st.count, st.sum = len(v), float(exact) if ok else MM.segment_stats(v).sum
                    st.min, st.max = (float(v.min()), float(v.max())) if len(v) else (MM.F64_MAX, -MM.F64_MAX)
                    entries[k] = (len(v), {"m": st})
                kept, e, o = TMM.cut(entries, 2, "metric", ts[2] == TQ_ORDER_ASC, ("m", prop))
                rows += [(fxg.osegs[i].segment_ord, k, cnt) for k, (cnt, _) in sorted(kept.items())]
            assert terms_rows(out, qi) == rows, (name, prop, ts[2])


# ---- the per-feature models over Fixture AG ------------------------------------------------------------------------------------
from tests import test_gpu_hist_metrics as GHM  # noqa: E402
from tests import test_gpu_hist_terms as GHT  # noqa: E402
from tests import test_gpu_range as GR  # noqa: E402
from tests import test_gpu_terms_hist as GTH  # noqa: E402
from tests import test_gpu_terms_metrics as GTM  # noqa: E402


@gpu
def test_hist_metrics_windows_and_runs_against_model(ctx_g, fxg):
    """`hmk` at interval 1 with `ints` and `sz`: units of 128 buckets (shared), 129 (global), one-bucket runs across unit ends,
    bucket changes mid-unit and a global window ending in a run -- the final result equals hist_metrics_model's and the doc counts
    equal tq_histogram_batch's; over the `all` query -0.0 / +0.0 from different units in one bucket give min -0.0 and max +0.0."""
    GHM.check([ctx_g], fxg, model_shapes(fxg), {"histogram": {"field": "hmk", "interval": 1}}, ["ints", "sz"])
    res = GHM.HMx.run([ctx_g], QueryBatch([few_shapes(fxg)[0][0]]), [GHM.HMx.parse_request(
        {"h": {"histogram": {"field": "gk", "interval": 1}, "aggs": {"lo": {"min": {"field": "sz"}}, "hi": {"max": {"field": "sz"}}}}})],
        GHM.fields_of(fxg, {"gk", "sz"}))[0]
    for b in GHM.buckets_of(res):
        assert _bits(b["lo"]["value"]) == _bits(-0.0) and _bits(b["hi"]["value"]) == _bits(0.0)


def test_fixture_ag_terms_metrics_slots_on_both_sides(data_ag):
    """`tk128` at segment_size 129: the segments of ordinals 5000 and 0 keep exactly 128 entries (k_terms_metrics' parts in shared
    memory), the others 129 (global), in one query."""
    kept = [min(129, len(np.unique(data_ag.columns["tk128"][i][0]))) for i in range(4)]
    assert sorted(set(kept)) == [TM_SMEM_SLOTS, TM_SMEM_SLOTS + 1]


@gpu
def test_terms_metrics_slots_and_order_windows_against_model(ctx_g, fxg):
    """`tk128` at segment_size 129: one query keeps 128 entries in two segments and 129 in the others (k_terms_metrics' parts in
    shared and in global memory); `tk1` (unit windows of 1024 and 1025 keys: k_terms_order in shared and in global memory) ordered
    by an `ints` metric.  The final results equal terms_metrics_model's, the `_count` rows tq_terms_batch's."""
    qts = model_shapes(fxg)
    GTM.check([ctx_g], fxg, qts, {"field": "tk128", "size": 20, "segment_size": 129}, ["ints", "sz"])
    out = ctx_g.terms_metrics_batch(QueryBatch([qts[0][0]]), [(fxg.mcol["tk128"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 129)],
                                    [[mspec(fxg, "ints")]])
    per = {}
    for s, _, _ in terms_rows(out, 0):
        per[s] = per.get(s, 0) + 1
    assert sorted(set(per.values())) == [TM_SMEM_SLOTS, TM_SMEM_SLOTS + 1]
    for order in ({"ints_avg": "asc"}, {"ints_stats.max": "desc"}):
        GTM.check([ctx_g], fxg, qts[:1], {"field": "tk1", "size": 20, "segment_size": 129, "order": order}, ["ints"])


@gpu
@pytest.mark.parametrize("ss", [1, 3])
def test_terms_hist_cells_against_model(ctx_g, fxg, ss):
    """`thk` with a histogram of `thv` at interval 1: one kept key per segment (windows of exactly 8192 cells in shared memory and
    8193 in the grid), and three; the result equals terms_hist_model's, rows and scalars tq_terms_batch's."""
    GTH.check([ctx_g], fxg, model_shapes(fxg), GTH.request({"field": "thk", "size": 3, "segment_size": ss}, {"field": "thv", "interval": 1}))


@gpu
def test_hist_terms_cells_against_model_and_terms_hist(ctx_g, fxg):
    """`thv` buckets with terms of `thk`: unit windows of 4096 x 2 = 8192 cells (shared) and 2731 x 3 = 8193 (global); the result
    equals hist_terms_model's.  Uncut, its (pos, key) counts equal the (key, pos) cells of tq_terms_histogram_batch, and those
    cells summed over the keys equal tq_histogram_batch's doc counts."""
    GHT.check([ctx_g], fxg, model_shapes(fxg), GHT.request({"field": "thv", "interval": 1}, {"field": "thk", "size": 10, "segment_size": 100}))
    qts = few_shapes(fxg)[:2]
    qb = QueryBatch([q for q, _ in qts])
    hs = (fxg.mcol["thv"], "i64", 1.0, 0.0)
    ts = (fxg.mcol["thk"], TQ_TERMS_BY_KEY, TQ_ORDER_ASC, 1000)
    ht = ctx_g.hist_terms_batch(qb, [hs] * 2, [ts] * 2)
    th = ctx_g.terms_hist_batch(qb, [ts] * 2, [hs] * 2)
    hist = ctx_g.histogram_batch(qb, [hs] * 2, stride=16384)
    for q in range(2):
        a = {(s, k, p): c for p, (_, _, _, ents) in GHT.dev_rows(ht, q).items() for s, k, c in ents}
        b = {(s, k, p): c for s, k, _, cells in TH.rows_of(th, q)[0] for p, c in cells.items()}
        assert a == b and a
        by_pos = {}
        for (_, _, p), c in b.items():
            by_pos[p] = by_pos.get(p, 0) + c
        assert sorted(by_pos.items()) == [(int(hist[0][q, j]), int(hist[1][q, j])) for j in range(int(hist[2][q]))]


@gpu
def test_range_with_guard_columns_against_model(ctx_g, fxg):
    """Range buckets on gk with metrics on a guard column and `sz` over the `all` query: the final result equals range_model's
    wherever the device answers, and the buckets at 2^(53+Q) and above are refused."""
    rng = {"field": "gk", "ranges": [{"to": 1}, {"from": 1, "to": 2}, {"from": 2, "to": 3}, {"from": 3}]}
    tally = GR.check([ctx_g], fxg, few_shapes(fxg)[:1], rng, ["g_q0", "sz"])
    assert tally[0] and tally[1]


def th_want(fx, qt, kcol, hcol, ss, masks=None):
    """terms_hist_model's rules 1-3 restated with numpy for integer columns at interval 1 without bounds: per segment the terms
    count and terms_model.cut, then the kept keys' (key, pos) cells.  ([(segment_ord, key, doc_count, {pos: n})], sum_other, error)."""
    rows, other, error = [], 0, 0
    for i in seg_order(fx):
        sel = fx.selected(i, qt, masks)
        kv, kp = fx.columns[kcol][i]
        hv = f64_of(fx.columns[hcol][i][0], fx.kind[hcol]).astype(np.int64)
        kept, e, o = TM.cut(TM.collect(kv, kp, sel), ss)
        other, error = other + o, error + e
        has = sel if kp is None else sel & kp
        for k, c in kept:
            d = has & (kv == np.uint64(k))
            p, n = np.unique(hv[d], return_counts=True)
            rows.append((fx.osegs[i].segment_ord, k, c, {int(a): int(b) for a, b in zip(p, n)}))
    return rows, other, error


def ht_want(fx, qt, hcol, kcol, ss, masks=None):
    """hist_terms_model's rules 1-4 restated with numpy for integer columns at interval 1 without bounds: per segment and bucket the
    doc count and terms_model.cut of the bucket's keys.  {pos: (doc_count, sum_other, error, [(segment_ord, key, n)])}."""
    out = {}
    for i in seg_order(fx):
        sel = fx.selected(i, qt, masks)
        kv, kp = fx.columns[kcol][i]
        hv = f64_of(fx.columns[hcol][i][0], fx.kind[hcol]).astype(np.int64)
        for p in np.unique(hv[sel]):
            d = sel & (hv == p)
            kept, e, o = TM.cut(TM.collect(kv, kp, d), ss)
            dc, so, er, ents = out.get(int(p), (0, 0, 0, []))
            out[int(p)] = (dc + int(d.sum()), so + o, er + e, ents + [(fx.osegs[i].segment_ord, k, c) for k, c in kept])
    return out


def terms_metrics_against_rule(ctx, fx, qts, masks, key="gk", ss=3, cols=("g_qn", "ints")):
    """tq_terms_metrics_batch: rows and scalars equal tq_terms_batch's; each kept (segment, key)'s parts against the values that
    segment's docs of that key collect (count, min, max, the guard's decision, accepted sums)."""
    qb = QueryBatch([q for q, _ in qts])
    ts = (fx.mcol[key], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, ss)
    out = ctx.terms_metrics_batch(qb, [ts] * len(qts), [[mspec(fx, n) for n in cols]] * len(qts), stride=4096)
    ref = ctx.terms_batch(qb, [ts] * len(qts), stride=4096)
    ords = {s.segment_ord: i for i, s in enumerate(fx.osegs)}
    for qi, qt in enumerate(qts):
        rows = terms_rows(out, qi)
        assert rows == terms_rows(ref, qi) and (int(out[5][qi]), int(out[6][qi])) == (int(ref[4][qi]), int(ref[5][qi]))
        assert rows == terms_want(fx, qt, key, TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, ss, masks=masks)[0]
        for j, (so, k, _) in enumerate(rows):
            i = ords[so]
            for ci, name in enumerate(cols):
                sel = fx.selected(i, qt, masks) & (fx.columns[key][i][0] == np.uint64(k))
                check_part(out[3][qi, j, ci], fx.values(name, i, sel)[0], (name, fx.kind[name], qi, so, k))


def grids_against_models(ctx, fx, qts, masks):
    """tq_terms_histogram_batch (thk by gk buckets, cut to 2 keys a segment) and tq_histogram_terms_batch (gk buckets with thk
    terms, cut to 1 key a bucket) against th_want / ht_want; the terms rows also against tq_terms_batch's."""
    qb = QueryBatch([q for q, _ in qts])
    ts = (fx.mcol["thk"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 2)
    hs = (fx.mcol["gk"], "u64", 1.0, 0.0)
    th = ctx.terms_hist_batch(qb, [ts] * len(qts), [hs] * len(qts))
    ref = ctx.terms_batch(qb, [ts] * len(qts))
    ht = ctx.hist_terms_batch(qb, [hs] * len(qts), [ts[:3] + (1,)] * len(qts))
    for qi, qt in enumerate(qts):
        got = TH.rows_of(th, qi)
        assert got == th_want(fx, qt, "thk", "gk", 2, masks), qi
        assert [r[:3] for r in got[0]] == terms_rows(ref, qi)
        assert GHT.dev_rows(ht, qi) == ht_want(fx, qt, "gk", "thk", 1, masks), qi


def _parts_against_rule(ctx, fx, qts, masks, cols=("g_qn", "ints", "sz")):
    """tq_metrics_batch, tq_histogram_metrics_batch (on `hmk`) and tq_range_batch (on gk) parts against the exact rule."""
    qb = QueryBatch([q for q, _ in qts])
    ms = [mspec(fx, n) for n in cols]
    parts = ctx.metrics_batch(qb, [ms] * len(qts))
    pos, counts, hparts, nb = ctx.hist_metrics_batch(qb, [(fx.mcol["hmk"], "i64", 1.0, 0.0)] * len(qts), [ms] * len(qts))
    rc, rparts = ctx.range_batch(qb, [(fx.mcol["gk"], [0, 1, 2, 3])] * len(qts), [ms] * len(qts))
    for qi, qt in enumerate(qts):
        for ci, name in enumerate(cols):
            vals = np.concatenate([fx.values(name, i, fx.selected(i, qt, masks))[0] for i in seg_order(fx)])
            check_part(parts[qi, ci], vals, (name, fx.kind[name], qi))
            hv = bucket_values(fx, qt, name, False, "hmk", lambda im: f64_of(im, "i64").astype(np.int64), masks)
            assert [int(p) for p in pos[qi, :int(nb[qi])]] == sorted(b for b, v in hv.items() if len(v)) or name == "ints"
            for j in range(int(nb[qi])):
                b = int(pos[qi, j])
                check_part(hparts[qi, j, ci], hv.get(b, np.zeros(0)), (name, fx.kind[name], qi, b))
            rv = bucket_values(fx, qt, name, False, "gk", lambda im: im.astype(np.int64), masks)
            for b in range(GK_BUCKETS):
                check_part(rparts[qi, b, ci], rv.get(b, np.zeros(0)), (name, fx.kind[name], qi, "range", b))


def every_entry_point_against_models(ctx, fx, qts, masks=None):
    run_terms(ctx, fx, qts, [(fx.mcol["tk"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 100)] * len(qts), masks=masks)
    _parts_against_rule(ctx, fx, qts, masks)
    terms_metrics_against_rule(ctx, fx, qts, masks)
    grids_against_models(ctx, fx, qts, masks)


@gpu
def test_every_shape_every_entry_point(ctx_g, fxg):
    """Every shape of shapes() in one batch per entry point, unfiltered: terms against terms_model; metrics, histogram metrics,
    range and terms metrics parts against the exact rule; terms histogram and histogram terms against numpy restatements of their
    models' rules over terms_model.cut."""
    every_entry_point_against_models(ctx_g, fxg, shapes(fxg))


@gpu
@pytest.mark.parametrize("fkind", FILTER_KINDS)
def test_filters_every_entry_point(ctx_g, fxg, fkind):
    """A filter kind on a subset of the shapes through all seven entry points, as test_every_shape_every_entry_point checks them,
    over the alive docs the filter keeps."""
    fid = 200 + FILTER_KINDS.index(fkind)
    qts = [(dict(q, filter=fid), t) for q, t in shapes(fxg)[::6]]
    every_entry_point_against_models(ctx_g, fxg, qts, fxg.filters[fkind])


@gpu
def test_filter_novalue(ctx_g, fxg):
    """Filter NOVALUE (Fixture A's docs without a `sparse` value) through all seven entry points."""
    qts = [(dict(q, filter=NOVALUE), t) for q, t in few_shapes(fxg)]
    every_entry_point_against_models(ctx_g, fxg, qts, fxg.novalue)


# ---- ordinals, split segments, waves -----------------------------------------------------------------------------------------
@gpu
def test_rows_in_ordinal_order_and_python_runs(ctx_g, fxg):
    """A query whose plan order (by ordinal: 0, 1200, 5000, 2^31 + 7) differs from its registration and term_segs order: the terms
    rows hold segments in u32 order, and each module's run() over them equals its model (which merges in segment_ord order)."""
    qt = model_shapes(fxg)[0]
    assert [ts[1] for ts in qt[0]["term_segs"]] != sorted(ts[1] for ts in qt[0]["term_segs"])
    out = run_terms(ctx_g, fxg, [qt], [(fxg.mcol["tk"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 3)])
    assert [int(x) for x in dict.fromkeys(out[0][0, :int(out[3][0])])] == sorted(ORDS_A)
    GTM.check([ctx_g], fxg, [qt], {"field": "gk", "size": 4, "order": {"_key": "asc"}}, ["w_qn"])
    GHM.check([ctx_g], fxg, [qt], {"histogram": {"field": "gk", "interval": 1}}, ["w_q0"])
    GR.check([ctx_g], fxg, [qt], {"field": "gk", "ranges": [{"to": 2}, {"from": 2}]}, ["w_qn"])
    GTH.check([ctx_g], fxg, [qt], GTH.request({"field": "gk", "size": 4}, {"field": "gk", "interval": 1}))
    GHT.check([ctx_g], fxg, [qt], GHT.request({"field": "gk", "interval": 1}, {"field": "thk", "size": 5}))


class SegmentView(FixtureAG):
    """Fixture AG restricted to its segment 0 (ordinal 5000), for contexts that each hold a doc range of it."""

    def __init__(self, fx):  # noqa: super-init-not-called
        self.osegs, self.models, self.alive = fx.osegs[:1], fx.models[:1], fx.alive[:1]
        self.columns = {k: v[:1] for k, v in fx.columns.items()}
        self.filters = {k: v[:1] for k, v in fx.filters.items()}
        self.kind, self.mcol, self.missing_k, self._has = fx.kind, fx.mcol, fx.missing_k, {}

    def narrow(self, qt):
        q, t = qt
        return dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] == self.osegs[0].segment_ord]), t


@gpu
def test_unaligned_doc_ranges(fxg):
    """Segment of ordinal 5000 split at 8191 and 3 * 8192 + 17, one context per piece, unfiltered and through a filter view: each
    module's multi-context run equals the whole segment's model.  The terms pieces come back uncut (both scalars 0), and cut once
    after summing they equal the whole segment's cut."""
    view = SegmentView(fxg)
    seg = fxg.osegs[0]
    cuts = (0, 8191, 3 * 8192 + 17, seg.max_doc)
    parts = []
    try:
        for lo, hi in zip(cuts, cuts[1:]):
            c = T.Context(0)
            parts.append(c)
            seg.register(c)
            c.segment_set_doc_range(seg.segment_ord, 0, lo, hi)
            c.filter_register(7, seg.segment_ord, packed(fxg.filters["bern30"][0]))
            for k in ("tk", "gk", "hmk", "thk", "thv", "ints", "g_qn", "w_q0"):
                fxg.register_agg_column(c, k, segs={0})
        for filt in (False, True):
            masks = view.filters["bern30"] if filt else None
            extra = dict(filter=7) if filt else {}
            qts = [(dict(q, **extra), t) for q, t in (view.narrow(qt) for qt in model_shapes(fxg))]
            qb = QueryBatch([q for q, _ in qts])
            for target, order, ss in ((TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 30), (TQ_TERMS_BY_KEY, TQ_ORDER_ASC, 50)):
                outs = [c.terms_batch(qb, [(fxg.mcol["tk"], target, order, ss)] * len(qts)) for c in parts]
                for qi, qt in enumerate(qts):
                    summed = {}
                    for o in outs:
                        assert (int(o[4][qi]), int(o[5][qi])) == (0, 0)
                        for _, k, n in terms_rows(o, qi):
                            summed[k] = summed.get(k, 0) + n
                    whole = TM.collect(*view.columns["tk"][0], view.selected(0, qt, masks))
                    assert summed == whole
                    assert TM.cut(summed, ss, target == TQ_TERMS_BY_KEY, order == TQ_ORDER_ASC) == \
                        TM.cut(whole, ss, target == TQ_TERMS_BY_KEY, order == TQ_ORDER_ASC)
            GTM.check(parts, view, qts, {"field": "tk", "size": 10, "segment_size": 30}, ["ints"], masks=masks)
            GHM.check(parts, view, qts, {"histogram": {"field": "hmk", "interval": 1}}, ["g_qn"], masks=masks)
            GR.check(parts, view, qts, {"field": "gk", "ranges": [{"to": 1}, {"from": 1, "to": 3}, {"from": 3}]}, ["w_q0"], masks=masks)
            GTH.check(parts, view, qts, GTH.request({"field": "thk", "size": 2, "segment_size": 2}, {"field": "thv", "interval": 64}), masks=masks)
            GHT.check(parts, view, qts, GHT.request({"field": "gk", "interval": 1}, {"field": "tk", "size": 3, "segment_size": 5}), masks=masks)
            mx, _ = Mx.run(parts, qb, [Mx.parse_request({"s": {"stats": {"field": "w_q0"}}})] * len(qts),
                           {"w_q0": Mx.MetricField(fxg.mcol["w_q0"], "u64")}, count_hits=True)
            for qt, r in zip(qts, mx):
                vals = view.values("w_q0", 0, view.selected(0, qt, masks))[0]
                assert isinstance(r, dict) and r["s"] == MM.final(MM.segment_stats(vals), "stats")  # (below the bound: answered)
    finally:
        for c in parts:
            c.close()


def norm_part(p):
    """A part's order-free fields, and its sum and magnitude where the guard accepts it (elsewhere they depend on the order)."""
    ok = Mx.guard(p) is None
    return (int(p["count"]), int(p["n_nan"]), int(p["n_inf"]), int(p["min_image"]), int(p["max_image"]), int(p["quantum_exp"]),
            _bits(float(p["sum"])) if ok else None, _bits(float(p["magnitude"])) if ok else None)


def norm(kind, out, nq):
    """The written part of an entry point's output, per query (the arrays past a row's length are never written)."""
    if kind == "terms":
        return [(terms_rows(out, q), int(out[4][q]), int(out[5][q])) + ((int(out[6][q]),) if len(out) > 6 else ()) for q in range(nq)]
    if kind == "metrics":
        return [[norm_part(p) for p in out[q]] for q in range(nq)]
    if kind == "hist_metrics":
        pos, counts, parts, nb = out[:4]
        return [[(int(pos[q, j]), int(counts[q, j]), [norm_part(x) for x in parts[q, j]]) for j in range(int(nb[q]))] for q in range(nq)]
    if kind == "terms_metrics":
        return [(terms_rows(out, q), [[norm_part(x) for x in out[3][q, j]] for j in range(int(out[4][q]))], int(out[5][q]), int(out[6][q]),
                 norm_part(out[7][q])) for q in range(nq)]
    if kind == "range":
        counts, parts = out[:2]
        return [(counts[q].tolist(), None if parts is None else [[norm_part(x) for x in parts[q, b]] for b in range(parts.shape[1])])
                for q in range(nq)]
    if kind == "terms_hist":
        return [TH.rows_of(out, q) for q in range(nq)]
    return [GHT.dev_rows(out, q) for q in range(nq)]


def every_entry_point(ctx, fx, qb, nq):
    """One call of each aggregation entry point over the fixture's threshold columns, normalised."""
    ms = [mspec(fx, "g_qn"), mspec(fx, "ints"), mspec(fx, "gm_q0", True)]
    return [
        norm("terms", ctx.terms_batch(qb, [(fx.mcol["tk"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 100)] * nq, count_hits=True), nq),
        norm("metrics", ctx.metrics_batch(qb, [ms] * nq), nq),
        norm("hist_metrics", ctx.hist_metrics_batch(qb, [(fx.mcol["hmk"], "i64", 1.0, 0.0)] * nq, [ms] * nq, stride=4096), nq),
        norm("terms_metrics", ctx.terms_metrics_batch(qb, [(fx.mcol["tk1"], TQ_TERMS_BY_METRIC, TQ_ORDER_DESC, 129)] * nq, [ms] * nq,
                                                      [(1, TQ_TERMS_ORDER_SUM)] * nq, stride=4096), nq),
        norm("range", ctx.range_batch(qb, [(fx.mcol["gk"], [0, 2, 3])] * nq, [ms] * nq), nq),
        norm("terms_hist", ctx.terms_hist_batch(qb, [(fx.mcol["thk"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 1)] * nq,
                                                [(fx.mcol["thv"], "i64", 1.0, 0.0)] * nq), nq),
        norm("hist_terms", ctx.hist_terms_batch(qb, [(fx.mcol["thv"], "i64", 1.0, 0.0)] * nq,
                                                [(fx.mcol["thk"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 2)] * nq), nq),
    ]


# each at least one (query, segment)'s need, and below one query's
BUDGETS = {"TQ_TERMS_COUNTER_BUDGET": "7000", "TQ_HIST_METRICS_BUDGET": "300", "TQ_TERMS_METRICS_BUDGET": "2100",
           "TQ_TERMS_HIST_BUDGET": "20000", "TQ_HIST_TERMS_BUDGET": "150000"}


# the wave counters each hook must raise; tq_histogram_metrics_batch keeps none (see the test)
WAVE_STATS = {"TQ_TERMS_COUNTER_BUDGET": ("terms_metrics_waves", "terms_hist_waves"), "TQ_HIST_METRICS_BUDGET": (),
              "TQ_TERMS_METRICS_BUDGET": ("terms_metrics_waves",), "TQ_TERMS_HIST_BUDGET": ("terms_hist_waves",),
              "TQ_HIST_TERMS_BUDGET": ("hist_terms_waves",)}


@gpu
@pytest.mark.parametrize("var", list(BUDGETS))
def test_small_budget_waves_equal_one_wave(ctx_g, fxg, var):
    """A fresh context with a small budget for one hook runs the batch in more waves than the default context (its wave counters
    grow more; for the histogram-metrics hook, which has no wave counter, every query alone needs more buckets than the budget and
    the terms counter hook is checked the same way); every entry point's result equals the default context's."""
    qts = few_shapes(fxg)
    qb = QueryBatch([q for q, _ in qts])
    d0 = ctx_g.stats()
    want = every_entry_point(ctx_g, fxg, qb, len(qts))
    d1 = ctx_g.stats()
    if var == "TQ_HIST_METRICS_BUDGET":  # the `hmk` buckets of each query (every one visits every tile): more than the budget
        span = max(int(f64_of(v, "i64").max()) for v, _ in fxg.columns["hmk"]) - min(int(f64_of(v, "i64").min()) for v, _ in fxg.columns["hmk"]) + 1
        assert span > int(BUDGETS[var])
    if var == "TQ_TERMS_COUNTER_BUDGET":  # the `tk` counters of each query: one segment's fit the budget, the query's do not
        spans = [int(v[p].max()) - int(v[p].min()) + 1 for v, p in fxg.columns["tk"]]
        assert max(spans) <= int(BUDGETS[var]) < sum(spans)
    os.environ[var] = BUDGETS[var]
    try:
        c = T.Context(0)
    finally:
        del os.environ[var]
    try:
        fxg.register(c, filters=(), names=("tk", "tk1", "hmk", "gk", "thk", "thv", "g_qn", "ints", "gm_q0"))
        s0 = c.stats()
        got = every_entry_point(c, fxg, qb, len(qts))
        s1 = c.stats()
        for name, g, w in zip(("terms", "metrics", "hist_metrics", "terms_metrics", "range", "terms_hist", "hist_terms"), got, want):
            assert g == w, (var, name)
        for k in WAVE_STATS[var]:
            assert s1[k] - s0[k] > d1[k] - d0[k] >= 1, (var, k, s1[k] - s0[k], d1[k] - d0[k])
    finally:
        c.close()


# ---- concurrency, holds, stats ---------------------------------------------------------------------------------------------------
@gpu
def test_concurrent_entry_points_on_one_context(ctx_g, fxg):
    """Six threads on one context, each looping a different aggregation entry point over shared columns and a private one: every
    result equals the single-threaded run; afterwards every column re-registers and unregisters."""
    qts = few_shapes(fxg)
    qb = QueryBatch([q for q, _ in qts])
    nq = len(qts)
    private = {t: 900 + t for t in range(6)}
    for t in range(6):
        fxg.register_agg_column(ctx_g, "ints", col_id=private[t])
    own = lambda t: (private[t], TQ_FAST_U64, 0, 0)  # noqa: E731
    ms = lambda t: [mspec(fxg, "g_qn"), own(t)]  # noqa: E731
    works = [
        lambda t: norm("terms", ctx_g.terms_batch(qb, [(fxg.mcol["tk"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 50)] * nq, count_hits=True), nq),
        lambda t: norm("metrics", ctx_g.metrics_batch(qb, [ms(t)] * nq), nq),
        lambda t: norm("hist_metrics", ctx_g.hist_metrics_batch(qb, [(fxg.mcol["hmk"], "i64", 1.0, 0.0)] * nq, [ms(t)] * nq, stride=4096), nq),
        lambda t: norm("terms_metrics", ctx_g.terms_metrics_batch(qb, [(fxg.mcol["tk1"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 129)] * nq, [ms(t)] * nq,
                                                                  stride=4096), nq),
        lambda t: norm("range", ctx_g.range_batch(qb, [(fxg.mcol["gk"], [0, 1, 3])] * nq, [ms(t)] * nq), nq),
        lambda t: norm("terms_hist", ctx_g.terms_hist_batch(qb, [(private[t], TQ_TERMS_BY_KEY, TQ_ORDER_ASC, 5)] * nq,
                                                            [(fxg.mcol["thv"], "i64", 1.0, 0.0)] * nq), nq),
    ]
    want = [works[t](t) for t in range(6)]
    errors, got = [], {}

    def loop(t):
        try:
            for it in range(3):
                got[(t, it)] = works[t](t)
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=loop, args=(t,)) for t in range(6)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert len(got) == 18 and all(res == want[t] for (t, _), res in got.items())
    for t in range(6):
        fxg.register_agg_column(ctx_g, "ints", col_id=private[t], segs={2})
        ctx_g.sort_column_unregister(private[t])
    for k in ("tk", "tk1", "hmk", "gk", "thk", "thv", "g_qn"):
        fxg.register_agg_column(ctx_g, k, segs={2})


@gpu
def test_holds_released_after_failures(ctx_g, fxg):
    """Each entry point with a missing column at query 1, a phrase at query 1, a refused span (2^20 + 1 terms keys, 2^16 + 1
    histogram-with-metrics buckets), and each strided one with a too-small out_stride (metrics and range rows are dense: they take
    no stride): each fails with its code and leaves no hold, so the columns it named re-register."""
    q, _ = fxg.query(TQ_OP_TERM, [ALL], 10)
    phrase = dict(q, op=3, term_pos=[(0, 0)] * len(q["term_segs"]), term_offset=[0])
    wide = 990  # a column of 2^20 + 1 keys in one segment
    wide_v = np.zeros(SIZES_A[2], np.uint64)
    wide_v[-1] = TERMS_MAX_KEYS
    ctx_g.sort_column_register(wide, fxg.osegs[2].segment_ord, wide_v)
    for i in (0, 1, 3):
        ctx_g.sort_column_register(wide, fxg.osegs[i].segment_ord, np.zeros(SIZES_A[i], np.uint64))
    hm_wide = 991  # 2^16 + 1 buckets at interval 1
    hv = T.fast_value_to_u64(np.where(np.arange(SIZES_A[2]) == 0, HM_MAX_BINS, 0), "i64")
    for i in range(4):
        ctx_g.sort_column_register(hm_wide, fxg.osegs[i].segment_ord, hv if i == 2 else T.fast_value_to_u64(np.zeros(SIZES_A[i], np.int64), "i64"))
    ms = [mspec(fxg, "g_qn")]
    ts = (fxg.mcol["tk"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 10)
    hs = (fxg.mcol["hmk"], "i64", 1.0, 0.0)
    gs = (fxg.mcol["gk"], "u64", 1.0, 0.0)
    bad_ts, bad_hs = (999, TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 10), (999, "i64", 1.0, 0.0)
    qq, qp = QueryBatch([q, q]), QueryBatch([q, phrase])
    fails = [
        (lambda: ctx_g.terms_batch(qq, [ts, bad_ts]), -3), (lambda: ctx_g.terms_batch(qp, [ts, ts]), -4),
        (lambda: ctx_g.terms_batch(qq, [ts, (wide,) + ts[1:]]), -4),
        (lambda: ctx_g.metrics_batch(qq, [ms, [(999, TQ_FAST_U64, 0, 0)]]), -3), (lambda: ctx_g.metrics_batch(qp, [ms, ms]), -4),
        (lambda: ctx_g.hist_metrics_batch(qq, [hs, bad_hs], [ms, ms]), -3), (lambda: ctx_g.hist_metrics_batch(qp, [hs, hs], [ms, ms]), -4),
        (lambda: ctx_g.hist_metrics_batch(qq, [hs, (hm_wide, "i64", 1.0, 0.0)], [ms, ms]), -4),
        (lambda: ctx_g.terms_metrics_batch(qq, [ts, bad_ts], [ms, ms]), -3), (lambda: ctx_g.terms_metrics_batch(qp, [ts, ts], [ms, ms]), -4),
        (lambda: ctx_g.terms_metrics_batch(qq, [ts, (wide,) + ts[1:]], [ms, ms]), -4),
        (lambda: ctx_g.range_batch(qq, [(fxg.mcol["gk"], [0, 1]), (999, [0, 1])], [ms, ms]), -3),
        (lambda: ctx_g.range_batch(qp, [(fxg.mcol["gk"], [0, 1])] * 2, [ms, ms]), -4),
        (lambda: ctx_g.terms_hist_batch(qq, [ts, bad_ts], [gs, gs]), -3), (lambda: ctx_g.terms_hist_batch(qp, [ts, ts], [gs, gs]), -4),
        (lambda: ctx_g.hist_terms_batch(qq, [gs, bad_hs], [ts, ts]), -3), (lambda: ctx_g.hist_terms_batch(qp, [gs, gs], [ts, ts]), -4),
    ]
    for i, (fn, rc) in enumerate(fails):
        assert code(fn) == rc, i
        for k in ("tk", "hmk", "gk", "g_qn"):
            fxg.register_agg_column(ctx_g, k, segs={1})
        ctx_g.sort_column_register(wide, fxg.osegs[2].segment_ord, wide_v)
        ctx_g.sort_column_register(hm_wide, fxg.osegs[2].segment_ord, hv)
    # too small a stride: -1 with the lengths, then the same columns re-register
    from tantivy_b200.lib import LIB
    import ctypes as C
    from tantivy_b200._abi import TERMS_SPEC_DTYPE, TermsSpec, ptr, u32p, u64p
    spec = np.zeros(1, TERMS_SPEC_DTYPE)
    spec[0]["column_id"], spec[0]["target"], spec[0]["order"], spec[0]["segment_size"] = fxg.mcol["tk"], TQ_TERMS_BY_KEY, TQ_ORDER_ASC, 100
    segs, keys, cnt = np.zeros((1, 4), np.uint32), np.zeros((1, 4), np.uint64), np.zeros((1, 4), np.uint64)
    n, other, err = np.zeros(1, np.uint32), np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    rc = LIB.tq_terms_batch(ctx_g.h, QueryBatch([q]).ptr, spec.ctypes.data_as(C.POINTER(TermsSpec)), 1, 4, ptr(segs, u32p), ptr(keys, u64p),
                            ptr(cnt, u64p), ptr(n, u32p), ptr(other, u64p), ptr(err, u64p), None)
    assert rc == -1 and int(n[0]) == 400
    fxg.register_agg_column(ctx_g, "tk", segs={1})
    # the other strided entry points: a first try at row width 1 (one cell, one entry) fails with -1 and the lengths after its run
    # (its units are counted), the wrapper runs again at the lengths, and the result equals a call at a wide enough width
    qb1 = QueryBatch([q])
    strided = [("hist_metrics", "units_hist_metrics", lambda st: ctx_g.hist_metrics_batch(qb1, [hs], [ms], stride=st)),
               ("terms_metrics", "units_terms_metrics", lambda st: ctx_g.terms_metrics_batch(qb1, [ts], [ms], stride=st)),
               ("terms_hist", "units_terms_hist", lambda st: ctx_g.terms_hist_batch(qb1, [ts], [gs], stride=st, cell_capacity=st)),
               ("hist_terms", "units_hist_terms", lambda st: ctx_g.hist_terms_batch(qb1, [gs], [ts], stride=st, entry_capacity=st))]
    for name, units, fn in strided:
        s0 = ctx_g.stats()
        wide_out = norm(name, fn(1 << 16), 1)
        s1 = ctx_g.stats()
        small_out = norm(name, fn(1), 1)
        s2 = ctx_g.stats()
        assert small_out == wide_out and s2[units] - s1[units] > s1[units] - s0[units] > 0, name
        for k in ("tk", "hmk", "gk", "g_qn"):
            fxg.register_agg_column(ctx_g, k, segs={1})
    ctx_g.sort_column_unregister(wide)
    ctx_g.sort_column_unregister(hm_wide)


STAT_GROUPS = {"terms": "terms_", "metrics": "metrics_", "hist_metrics": "hist_metrics_", "terms_metrics": "terms_metrics_",
               "range": "range_", "terms_hist": "terms_hist_", "hist_terms": "hist_terms_"}


@gpu
def test_runs_keep_to_their_own_stats(ctx_g, fxg):
    """Each entry point's run changes only its own tq_get_*_stats counters (timings aside)."""
    from tantivy_b200._abi import (HistMetricsStats, HistTermsStats, MetricsStats, RangeStats, TermsHistStats, TermsMetricsStats,
                                   TermsStats)
    groups = {"terms": TermsStats, "metrics": MetricsStats, "hist_metrics": HistMetricsStats, "terms_metrics": TermsMetricsStats,
              "range": RangeStats, "terms_hist": TermsHistStats, "hist_terms": HistTermsStats}
    fields = {g: {n for n, _ in s._fields_} for g, s in groups.items()}
    qts = few_shapes(fxg)[:1]
    qb = QueryBatch([q for q, _ in qts])
    ms = [mspec(fxg, "g_qn")]
    runs = {
        "terms": lambda: ctx_g.terms_batch(qb, [(fxg.mcol["tk"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 10)]),
        "metrics": lambda: ctx_g.metrics_batch(qb, [ms]),
        "hist_metrics": lambda: ctx_g.hist_metrics_batch(qb, [(fxg.mcol["hmk"], "i64", 1.0, 0.0)], [ms], stride=4096),
        "terms_metrics": lambda: ctx_g.terms_metrics_batch(qb, [(fxg.mcol["tk1"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 10)], [ms]),
        "range": lambda: ctx_g.range_batch(qb, [(fxg.mcol["gk"], [0, 1])], [ms]),
        "terms_hist": lambda: ctx_g.terms_hist_batch(qb, [(fxg.mcol["thk"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 1)], [(fxg.mcol["thv"], "i64", 1.0, 0.0)]),
        "hist_terms": lambda: ctx_g.hist_terms_batch(qb, [(fxg.mcol["thv"], "i64", 1.0, 0.0)], [(fxg.mcol["thk"], TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 2)]),
    }
    for g, fn in runs.items():
        fn()  # (sizes known: one run per call)
        s0 = ctx_g.stats()
        fn()
        s1 = ctx_g.stats()
        others = set().union(*(fields[h] for h in fields if h != g)) - fields[g]
        changed = {k for k in s1 if s1[k] != s0[k] and not k.endswith("_ms")}
        assert changed and changed <= fields[g], (g, changed - fields[g])
        assert not changed & others


# ---- a segment of 2^31 - 2 docs ------------------------------------------------------------------------------------------------
BIG_KEY_COL = 21


@pytest.fixture(scope="module")
def big_keys(big):
    """test_gpu_fast_field_edges' segment of 2^31 - 2 docs (its lists and date column 9 in the top 300 000 docs and at
    max_doc - 1) with a key column beside the dates: (doc - top) % 1000 on the docs with a date, and key 1000 only at max_doc - 1."""
    n = big.max_doc - big.top
    keys = (np.arange(n, dtype=np.uint64) % np.uint64(1000))
    keys[-1] = 1000
    present = np.zeros((big.max_doc + 7) // 8, np.uint8)
    sel = big.top + np.nonzero(big.has)[0]
    np.bitwise_or.at(present, sel >> 3, (1 << (sel & 7)).astype(np.uint8))
    values = np.zeros(big.max_doc, np.uint64)
    values[big.top:] = keys
    big.ctx.sort_column_register(BIG_KEY_COL, big.seg.segment_ord, values, present)
    del values
    return types.SimpleNamespace(keys=keys, dates=f64_of(big.top_values, "date"))


def big_selected(big, docs):
    m = np.zeros(big.max_doc - big.top, bool)
    m[docs.astype(np.int64) - big.top] = True
    return m & big.has


@gpu
def test_big_segment_terms_range_hist_metrics_terms_metrics(big, big_keys):
    """The 2^31 - 2 doc segment through tq_terms_batch, tq_range_batch with metrics, tq_histogram_metrics_batch and
    tq_terms_metrics_batch: values and keys in the top tiles and at max_doc - 1.  Terms rows against terms_model (cut and uncut:
    the key of max_doc - 1 alone among them); every part against the values it collects (count, min and max images, the guard's
    decision, accepted sums); hits against tq_count_batch."""
    qb = QueryBatch([q for q, _ in big.qs])
    nq = len(big.qs)
    so = big.seg.segment_ord
    ctx = big.ctx
    ms = [(BIG_KEY_COL, TQ_FAST_U64, 0, 0), (9, TQ_FAST_DATE, 0, 0)]
    cols = (("key", big_keys.keys.astype(np.float64), "u64"), ("date", big_keys.dates, "date"))
    sels = [big_selected(big, docs) for _, docs in big.qs]
    for target, order, ss in ((TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 100), (TQ_TERMS_BY_KEY, TQ_ORDER_ASC, 2000)):
        out = ctx.terms_batch(qb, [(BIG_KEY_COL, target, order, ss)] * nq, count_hits=True)
        assert np.array_equal(out[6], ctx.count_batch(qb))
        for qi, sel in enumerate(sels):
            kept, e, o = TM.cut(TM.collect(big_keys.keys, None, sel), ss, target == TQ_TERMS_BY_KEY, order == TQ_ORDER_ASC)
            assert (terms_rows(out, qi), int(out[4][qi]), int(out[5][qi])) == ([(so, k, c) for k, c in kept], o, e), (qi, ss)
            if qi < 3 and ss == 2000:
                assert (so, 1000, 1) in terms_rows(out, qi)
    # range on the keys with metrics on the keys and the dates
    starts = [0, 250, 500, 1000]
    counts, parts, hits = ctx.range_batch(qb, [(BIG_KEY_COL, starts)] * nq, [ms] * nq, count_hits=True)
    counts_a, _ = ctx.range_batch(qb, [(BIG_KEY_COL, starts)] * nq)
    assert np.array_equal(counts, counts_a) and np.array_equal(hits, ctx.count_batch(qb))
    for qi, sel in enumerate(sels):
        b = np.searchsorted(np.array(starts), big_keys.keys, side="right") - 1
        for bi in range(len(starts)):
            d = sel & (b == bi)
            assert int(counts[qi, bi]) == int(d.sum())
            for ci, (name, vals, kind) in enumerate(cols):
                check_part(parts[qi, bi, ci], vals[d], (name, kind, qi, "range", bi))
    # a histogram of the keys by 100 with the same metrics
    pos, hcounts, hparts, nb = ctx.hist_metrics_batch(qb, [(BIG_KEY_COL, "u64", 100.0, 0.0)] * nq, [ms] * nq)
    for qi, sel in enumerate(sels):
        p = (big_keys.keys // np.uint64(100)).astype(np.int64)
        want = sorted((int(x), int(c)) for x, c in zip(*np.unique(p[sel], return_counts=True)))
        assert [(int(pos[qi, j]), int(hcounts[qi, j])) for j in range(int(nb[qi]))] == want
        for j in range(int(nb[qi])):
            d = sel & (p == int(pos[qi, j]))
            for ci, (name, vals, kind) in enumerate(cols):
                check_part(hparts[qi, j, ci], vals[d], (name, kind, qi, "hist", int(pos[qi, j])))
    # terms of the keys with the same metrics, cut to 100 keys
    ts = (BIG_KEY_COL, TQ_TERMS_BY_COUNT, TQ_ORDER_DESC, 100)
    tm = ctx.terms_metrics_batch(qb, [ts] * nq, [ms] * nq)
    ref = ctx.terms_batch(qb, [ts] * nq)
    for qi, sel in enumerate(sels):
        rows = terms_rows(tm, qi)
        assert rows == terms_rows(ref, qi) and (int(tm[5][qi]), int(tm[6][qi])) == (int(ref[4][qi]), int(ref[5][qi]))
        for j, (_, k, c) in enumerate(rows):
            d = sel & (big_keys.keys == np.uint64(k))
            assert int(d.sum()) == c
            for ci, (name, vals, kind) in enumerate(cols):
                check_part(tm[3][qi, j, ci], vals[d], (name, kind, qi, "terms", k))
