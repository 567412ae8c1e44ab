"""The Count kernels (k_count, k_count_tiles, k_filter_combine) against the score model at every tile, word and unit
edge.  Every count is checked exactly against tests/score_model.py (the docs its scorers match, and-ed with the alive bits, the
filter and the doc range, as M.count does); every batch that counts hits returns the same rows as the batch without the flag.

Fixtures: a 279 531-doc ladder segment of 32 lists where docs listed by exactly c lists, for every c in 0..32, sit on the first and
last doc of every 1024-doc tile, 8192-doc tile and default k_count_tiles unit, on offsets 0 and 31 of 32-doc words, on both halves
of 64-bit alive words, on docs 0..7 and on max_doc - 1 (listed by all 32); lists on both sides of the dense threshold, some ending
a 128-doc block on the doc before an 8192-doc tile and some on its first doc.  The ladder comes three times: few deletes, deletes
on half the planted docs (max_doc - 1 too), and no alive bitset.  Small segments of 1, 33, 1025, 8192 and 8193 docs, with lists
absent from some of them.  A segment whose tile holds exactly 8192 and 8193 sparse offsets, and a segment of 2^31 - 2 docs."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200._abi import (TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT, TQ_OCCUR_SHOULD, TQ_OP_AND, TQ_OP_BOOL, TQ_OP_OR,  # noqa: E402
                               TQ_OP_TERM, TQ_TERM_IGNORE_FREQ, QueryBatch)
from tests import score_model as M  # noqa: E402
from tests.helpers import OracleSegment, bool_query, hits, make_query, random_bool_shapes  # noqa: E402
from tests.test_gpu_parity import _ctx_with_env, fresh_ord  # noqa: E402

S, R, X = TQ_OCCUR_SHOULD, TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT
NL = 32
KS = (1, 10, 1000)
TILE, CTILE = 1024, 8192  # k_count_tiles' tile (and 8 of them: its default unit), k_count's tile
LADDER_DOCS = 34 * CTILE + 1003  # 273 tiles of 1024 docs, 35 of 8192 (the last ones partial), 11 docs in the last 32-doc word
DENSE_MIN = 6  # TQ_TILE_BIG_MIN's default: a list with >= 6 postings per 1024-doc tile gets a presence map


def _ceil(a, b):
    return -(-a // b)


def packed(mask):
    return np.packbits(np.asarray(mask, bool), bitorder="little")


def _planted(max_doc, rng, top=NL):
    """{doc: level} on the edge docs.  Each kind of place cycles through the levels 0..top from its own offset, so every level
    sits on every kind of place that has top + 1 docs or more; a doc on several kinds takes the first kind's level."""
    level = {}

    def put(docs, off):
        i = 0
        for d in docs:
            d = int(d)
            if 0 <= d < max_doc and d not in level:
                level[d] = (i + off) % (top + 1)
                i += 1

    put([max_doc - 1], top)                                         # the last doc, in the last partial word: every list
    put(range(0, max_doc, CTILE), 1)                                # first / last doc of 8192-doc tiles = default units
    put(range(CTILE - 1, max_doc, CTILE), 7)
    put(range(0, max_doc, TILE), 3)                                 # first / last doc of 1024-doc tiles
    put(range(TILE - 1, max_doc, TILE), 11)
    n_w = min(200, max_doc // 32)
    w = rng.choice(max_doc // 32, size=n_w, replace=False) * 32 if n_w else np.zeros(0, int)
    put(w, 5)                                                       # offsets 0 and 31 of 32-doc words
    put(w + 31, 13)
    n_h = min(200, max_doc // 64)
    h = rng.choice(max_doc // 64, size=n_h, replace=False) * 64 if n_h else np.zeros(0, int)
    put(h + 31, 17)                                                 # both halves of 64-bit alive words
    put(h + 32, 19)
    put(range(8), 23)                                               # docs 0..7 (a doc range narrowed twice inside byte 0)
    return level


def _align_blocks(docs, planted, edges, rng, max_doc):
    """Adds unplanted docs below each edge e so that the list's doc before e (its doc e - 1 or e) ends a 128-doc block."""
    docs = set(int(d) for d in docs)
    for e, last in edges:
        before = sum(1 for d in docs if d < last)
        need = (127 - before) % 128
        free = [d for d in range(max(0, e - 4096), last) if d not in docs and d not in planted]
        docs.update(int(d) for d in rng.choice(free, size=need, replace=False))
    return np.array(sorted(docs), np.uint32)


def ladder_lists(max_doc, rng, align=False):
    """32 lists: background postings at densities from 0.03 % to 30 % (both sides of TQ_TILE_BIG_MIN) plus the planted docs.
    Below one tile the levels stop at 7 (at 3 below one word): a TQ_OP_BOOL query whose clauses list more than about 7.8 docs
    per doc does not fit k_tile's pair buffer (kTileMaxPairs) and is refused."""
    level = _planted(max_doc, rng, NL if max_doc >= TILE else (7 if max_doc >= 32 else 3))
    planted = np.array(sorted(level), np.int64)
    members = [[] for _ in range(NL)]
    for d in planted:
        for t in rng.choice(NL, size=level[int(d)], replace=False):
            members[int(t)].append(int(d))
    dens = rng.permutation(np.geomspace(0.0003, 0.3, NL))
    lists = []
    for t in range(NL):
        bg = rng.random(max_doc) < dens[t]
        bg[planted] = False
        lists.append(np.union1d(np.nonzero(bg)[0], members[t]).astype(np.uint32))
    if align:  # per 8192-doc tile edge e: one list that holds e ends a block on e, another that holds e - 1 ends one on e - 1
        per_list = [[] for _ in range(NL)]
        for e in range(CTILE, max_doc, CTILE):
            on = [t for t in range(NL) if e in members[t]]
            before = [t for t in range(NL) if e - 1 in members[t]]
            if on:
                t_on = int(rng.choice(on))
                per_list[t_on].append((e, e))
                before = [t for t in before if t != t_on]
            if before:
                per_list[int(rng.choice(before))].append((e, e - 1))
        pset = set(level)
        for t in range(NL):
            if per_list[t]:
                lists[t] = _align_blocks(lists[t], pset, per_list[t], rng, max_doc)
    return [(d, rng.integers(1, 11, size=len(d)).astype(np.uint32)) for d in lists], level


class Seg:
    """One registered segment: its OracleSegment, its model (alive None: the docs the scorers match before deletes), the mask of
    its alive docs, and a content key (copies of the same lists share the model's matches)."""

    def __init__(self, lists, lengths, alive, absent=(), content=None, max_doc=None):
        so = fresh_ord()
        absent = set(absent) | {t for t, (d, _) in enumerate(lists) if len(d) == 0}
        write = [(d, tf) if t not in absent else (np.array([0], np.uint32), np.array([1], np.uint32)) for t, (d, tf) in enumerate(lists)]
        self.o = OracleSegment(write, lengths, segment_ord=so, writer_cls=T.FieldWriter, alive=alive, max_doc=max_doc)
        for t in absent:
            self.o.terms[t] = (0, 0, 0)
        self.ord, self.max_doc, self.absent = so, self.o.max_doc, absent
        model_lists = [(d, tf) if t not in absent else (np.zeros(0, np.uint32), np.zeros(0, np.uint32)) for t, (d, tf) in enumerate(lists)]
        self.m = M.Segment(so, model_lists, lengths)
        self.alive = np.ones(self.max_doc, bool) if alive is None else \
            np.unpackbits(alive, bitorder="little", count=self.max_doc).astype(bool)
        self.content = content if content is not None else so

    def register(self, ctx):
        self.o.register(ctx)


def _lengths(rng, n):
    return np.clip(np.round(np.exp(rng.normal(np.log(40), 0.7, size=n))), 1, 4096).astype(np.uint32)


class Fixture:
    def __init__(self, seed=0xC0C0):
        rng = np.random.default_rng(seed)
        lists, self.level = ladder_lists(LADDER_DOCS, rng, align=True)
        self.lists = lists
        lengths = _lengths(rng, LADDER_DOCS)
        planted = np.array(sorted(self.level))
        few = rng.random(LADDER_DOCS) > 0.05
        few[planted] = True
        half = rng.random(LADDER_DOCS) > 0.1
        half[planted] = rng.random(len(planted)) > 0.5
        half[LADDER_DOCS - 1] = False
        self.ladder = Seg(lists, lengths, packed(few), content="ladder")
        self.ladder_del = Seg(lists, lengths, packed(half), content="ladder")
        self.ladder_none = Seg(lists, lengths, None, content="ladder")
        self.small = []
        for max_doc, has_alive, absent in ((1, False, ()), (33, True, range(20, 32)), (1025, True, range(28, 32)), (8192, False, ()),
                                           (8193, True, (5,))):
            sl, _ = ladder_lists(max_doc, rng)
            alive = packed(rng.random(max_doc) > 0.2) if has_alive else None
            self.small.append(Seg(sl, _lengths(rng, max_doc), alive, absent=absent))
        self.segs = [self.ladder, self.ladder_del, self.ladder_none] + self.small
        self._has = {}
        n_dense = sum(len(d) * TILE >= DENSE_MIN * LADDER_DOCS for d, _ in lists)
        assert 8 <= n_dense <= NL - 8, n_dense  # a 32-clause query mixes dense and sparse slots

    def register(self, ctx, segs=None):
        for s in segs or self.segs:
            s.register(ctx)
        return ctx

    def query(self, shape, k, segs=None):
        """shape = (op, terms, occurs, groups, msm, flags); its query over the segments (all of the fixture's by default)."""
        op, terms, occ, groups, msm, flags = shape
        q = make_query(op if op != TQ_OP_BOOL else TQ_OP_OR, [s.o for s in segs or self.segs], terms, k)
        if op == TQ_OP_BOOL:
            q = bool_query(q, occ, groups, msm)
        if flags is not None:
            q["term_flags"] = list(flags)
        return q, list(terms)

    def has(self, seg, qt):
        """The docs the model's scorers match in seg, before deletes (M.count's d.has); shared by copies of the same lists."""
        q, terms = qt
        key = (seg.content, repr((q["op"], terms, q.get("term_occur"), q.get("term_group"), q.get("min_should_match"),
                                  q.get("term_flags"), sorted(ts[0] for ts in q["term_segs"] if ts[1] == seg.ord))))
        if key not in self._has:
            d = M._segment_matches(seg.m, q, terms)
            self._has[key] = np.zeros(seg.max_doc, bool) if d is None else d.has.copy()
        return self._has[key]

    def count(self, qt, masks=None, segs=None):
        """The model's count over the segments: matched AND alive (AND masks[seg], the filter and doc range, where given)."""
        n = 0
        for s in segs or self.segs:
            sel = self.has(s, qt) & s.alive
            if masks is not None and s in masks:
                sel &= masks[s]
            n += int(sel.sum())
        return n


@pytest.fixture(scope="module")
def fx():
    return Fixture()


def _shapes(rng):
    """The structured shapes (op, terms, occurs, groups, msm, flags) over the 32 lists, then about 100 random BOOL shapes with
    their own k."""
    a32 = list(range(NL))
    out = [(TQ_OP_BOOL, a32, [S] * NL, None, m, None) for m in range(NL + 2)]
    for m in (0, 1, 2, 16, 30, 31, 32):
        out.append((TQ_OP_BOOL, a32, [S] * 31 + [R], None, m, None))
        out.append((TQ_OP_BOOL, a32, [S] * 30 + [R, X], None, m, None))
    out.append((TQ_OP_BOOL, a32, [R] * NL, [1] * NL, 0, None))                           # one MUST group of 32 alternatives
    out.append((TQ_OP_BOOL, a32, [R] * NL, [1 + t // 8 for t in a32], 0, None))          # 4 groups of 8
    out.append((TQ_OP_BOOL, a32, [R] * NL, [1 + t // 2 for t in a32], 0, None))          # 16 groups of 2
    out.append((TQ_OP_BOOL, a32, [X] * 31 + [R], None, 0, None))
    out.append((TQ_OP_BOOL, a32, [S] + [X] * 31, None, 0, None))
    # repeated terms: the repeat decides the count
    out.append((TQ_OP_BOOL, [3, 3, 20], [S, S, S], None, 2, None))
    out.append((TQ_OP_BOOL, [3, 3, 3, 20, 9], [S] * 5, None, 3, None))
    out.append((TQ_OP_BOOL, [17, 17, 17, 4], [S] * 4, None, 3, None))
    out.append((TQ_OP_BOOL, [5, 8, 5], [S, S, X], None, 0, None))                        # SHOULD and MUST_NOT of one list
    out.append((TQ_OP_BOOL, [6, 6, 12], [S, S, S], None, 2, [TQ_TERM_IGNORE_FREQ, 0, 0]))  # two slots, the same docs
    out.append((TQ_OP_BOOL, [6, 6], [R, R], [1, 2], 0, [0, TQ_TERM_IGNORE_FREQ]))
    # lists absent from small segments: msm 12 of lists 16..31 is above the SHOULD clauses present in the 33-doc segment (4) and
    # equal to them in the 1025-doc one (12); a MUST group of lists 28..31 is empty in both
    out.append((TQ_OP_BOOL, list(range(16, 32)), [S] * 16, None, 12, None))
    out.append((TQ_OP_BOOL, [28, 29, 30, 31, 0, 1, 2, 3], [R] * 4 + [S] * 4, [1] * 4 + [0] * 4, 1, None))
    out.append((TQ_OP_AND, a32, None, None, 0, None))
    out.append((TQ_OP_OR, a32, None, None, 0, None))
    out += [(TQ_OP_TERM, [t], None, None, 0, None) for t in a32]
    rnd = [(TQ_OP_BOOL, sh["terms"], sh["occurs"], sh["groups"], sh["msm"], sh["flags"], sh["k"])
           for sh in random_bool_shapes(rng, 100, NL, n_wide=8)]
    return out, rnd


def _queries(fx, segs=None, ks=KS, n_random=100):
    structured, rnd = _shapes(np.random.default_rng(0x32))
    qts = [fx.query(sh, k, segs) for sh in structured for k in ks]
    qts += [fx.query(sh[:6], sh[6], segs) for sh in rnd[:n_random]]
    return qts


def _run(ctx, queries):
    b = ctx.prepare(QueryBatch(queries))
    try:
        b.run()
        return b.fetch(), b.fetch_hits(), ctx.stats()
    finally:
        b.close()


def _check(ctx, fx, qts, what, masks=None, filt=None, segs=None, bool_rows=True):
    """The flagged batch's hits and tq_count_batch == the model; its rows == the unflagged batch's.  filt: the queries' filter id
    (None: unfiltered); bool_rows=False on the per-query kernels (no TQ_OP_BOOL rows there: those queries are only counted)."""
    want = [fx.count(qt, masks, segs) for qt in qts]
    extra = {} if filt is None else dict(filter=filt)
    counted = ctx.count_batch(QueryBatch([dict(q, **extra) for q, _ in qts]))
    assert [int(x) for x in counted] == want, (what, "count_batch", [(i, int(c), w) for i, (c, w) in enumerate(zip(counted, want)) if c != w][:6])
    idx = [i for i, (q, _) in enumerate(qts) if bool_rows or q["op"] != TQ_OP_BOOL]
    rows, got, st = _run(ctx, [dict(qts[i][0], count_hits=True, **extra) for i in idx])
    plain = ctx.search_batch(QueryBatch([dict(qts[i][0], **extra) for i in idx]))
    bad = [(i, qts[i][1][:4], int(got[j]), want[i]) for j, i in enumerate(idx) if int(got[j]) != want[i]]
    assert not bad, (what, "hits", bad[:6])
    for j, i in enumerate(idx):
        assert hits(rows, j) == hits(plain, j), (what, "rows", i)
    return st


# ---- every route ---------------------------------------------------------------------------------------------------------------
# several groups: by queries per group (a 32-clause query here brings all of a segment's lists, so a density cap that splits the
# batch would refuse it)
ROUTES = {"default": {}, "all_dense": dict(TQ_TILE_BIG_MIN=1), "all_sparse": dict(TQ_TILE_BIG_MIN=100000),
          "groups": dict(TQ_TILE_MAX_QUERIES=40, TQ_TILE_WIDE_QUERIES=16), "unit1": dict(TQ_COUNT_HITS_TILES_PER_UNIT=1),
          "unit3": dict(TQ_COUNT_HITS_TILES_PER_UNIT=3)}


@pytest.mark.parametrize("route", list(ROUTES) + ["per_query"])
def test_every_shape_on_every_route(fx, route):
    tile = route != "per_query"
    c = fx.register(_ctx_with_env(TQ_TILE=1 if tile else 0, TQ_TILE_TERMS=1, **ROUTES.get(route, {})))
    try:
        st = _check(c, fx, _queries(fx), route, bool_rows=tile)
        assert st["units_count_hits"] > 0, st
        if route == "groups":
            assert st["tile_groups"] >= 2, st
        if not tile:
            assert st["tile_groups"] == 0, st
    finally:
        c.close()


@pytest.mark.parametrize("per", [1, 3, 8])
def test_count_units_follow_the_unit_rule(fx, per):
    """One unfiltered tile group: k_count_tiles' units are max(per, ceil(group tiles / 1024)) tiles of each segment's tiles."""
    c = fx.register(_ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, TQ_COUNT_HITS_TILES_PER_UNIT=per))
    try:
        st = _check(c, fx, _queries(fx, ks=(10,), n_random=0), per)
        assert st["tile_groups"] == 1, st
        tiles = [_ceil(s.max_doc, TILE) for s in fx.segs]
        count_per = max(per, _ceil(sum(tiles), 1024))
        assert st["units_count_hits"] == sum(_ceil(t, count_per) for t in tiles), (st["units_count_hits"], tiles, count_per)
    finally:
        c.close()


# ---- filters and doc ranges on the ladder segments -------------------------------------------------------------------------------
def _filters(fx):
    n = LADDER_DOCS
    edges = np.zeros(n, bool)
    edges[np.array(sorted(fx.level))] = True
    run = np.zeros(n, bool)
    run[32 * 1000 + 5:32 * 7000 + 27] = True  # both ends inside 32-doc words
    last = np.zeros(n, bool)
    last[(n // TILE) * TILE:] = np.random.default_rng(5).random(n - (n // TILE) * TILE) < 0.5  # only the last, partial tile
    return {1: edges, 2: np.ones(n, bool), 3: run, 4: last}


def _ladder_queries(fx):
    segs = [fx.ladder, fx.ladder_del, fx.ladder_none]
    structured, rnd = _shapes(np.random.default_rng(0x32))
    pick = structured[::3] + [sh for sh in structured if sh[0] == TQ_OP_TERM][::5]
    return segs, [fx.query(sh, 10, segs) for sh in pick] + [fx.query(sh[:6], sh[6], segs) for sh in rnd[:24]]


def _check_filtered(c, fx, segs, qts, ranges, what, fids=(1, 2, 3, 4)):
    """Unfiltered and under every filter, with the doc ranges {seg: (lo, hi)} of the context."""
    rmask = {}
    for s in segs:
        lo, hi = ranges.get(s, (0, s.max_doc))
        m = np.zeros(s.max_doc, bool)
        m[lo:hi] = True
        rmask[s] = m
    _check(c, fx, qts, (what, None), masks=rmask, segs=segs)
    for fid, fm in _filters(fx).items():
        if fid not in fids:
            continue
        _check(c, fx, qts, (what, fid), masks={s: rmask[s] & fm for s in segs}, filt=fid, segs=segs)


# doc ranges: lo / hi at word offsets 1 and 31 next to planted docs (offset 0: an 8192-doc tile's first doc; offset 31: a 1024-doc
# tile's last doc), at 1024- and 8192-doc tile edges +- 1
RANGES = [(5 * CTILE + 1, 30 * CTILE + 1), (7 * TILE - 1, 200 * TILE - 1), (3 * CTILE - 1, 20 * CTILE + 1), (TILE + 1, LADDER_DOCS - 31 * 32 - 1)]


@pytest.mark.parametrize("rng_i", range(len(RANGES)))
@pytest.mark.parametrize("engine", ["tile", "per_query"])
def test_filters_and_doc_ranges(fx, rng_i, engine):
    """Filters registered before and after the range is set; count hits and tq_count_batch."""
    segs, qts = _ladder_queries(fx)
    if engine == "per_query":
        qts = [qt for qt in qts if qt[0]["op"] != TQ_OP_BOOL]
    lo, hi = RANGES[rng_i]
    filters = _filters(fx)
    c = _ctx_with_env(TQ_TILE=1 if engine == "tile" else 0, TQ_TILE_TERMS=1)
    try:
        fx.register(c, segs)
        for fid in (1, 2):
            for s in segs:
                c.filter_register(fid, s.ord, packed(filters[fid]))
        for s in segs:
            c.segment_set_doc_range(s.ord, 0, lo, hi)
        for fid in (3, 4):
            for s in segs:
                c.filter_register(fid, s.ord, packed(filters[fid]))
        _check_filtered(c, fx, segs, qts, {s: (lo, hi) for s in segs}, (engine, lo, hi))
    finally:
        c.close()


def test_doc_range_narrowed_twice_inside_one_byte(fx):
    """[0, n) -> [3, n - 2) -> [5, n - 5): the second narrowing clears docs 3 and 4 inside byte 0 of the alive bitset.  Filters 1, 2
    before the first narrowing, 3 after it, 4 after the second; the segment without deletes gets its bitset at the first one."""
    segs, qts = _ladder_queries(fx)
    filters = _filters(fx)
    n = LADDER_DOCS
    assert fx.level[4] > 0 and fx.level[3] > 0
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1)
    try:
        fx.register(c, segs)

        def reg(fid):
            for s in segs:
                c.filter_register(fid, s.ord, packed(filters[fid]))

        reg(1)
        reg(2)
        for s in segs:
            c.segment_set_doc_range(s.ord, 0, 3, n - 2)
        reg(3)
        _check_filtered(c, fx, segs, qts[::2], {s: (3, n - 2) for s in segs}, "first", fids=(1, 2, 3))
        for s in segs:
            c.segment_set_doc_range(s.ord, 0, 5, n - 5)
        reg(4)
        _check_filtered(c, fx, segs, qts, {s: (5, n - 5) for s in segs}, "second")
    finally:
        c.close()


# ---- k_count_tiles' sparse-offset buffer ---------------------------------------------------------------------------------------
def test_sparse_offsets_at_and_past_the_tile_buffer():
    """Every list sparse (TQ_TILE_BIG_MIN=100000).  Lists 0..7 hold every doc of tile 5: exactly kCountSparseCap (8192) offsets;
    with list 8's one posting there, 8193: the group is recounted through tq_count_batch, which must apply the filter and the
    doc range again.  Tiles 0..4 of the same unit hold other offsets of lists 0..7 (about 95 % of their docs)."""
    rng = np.random.default_rng(0xCA9)
    max_doc = 20_000
    t5 = np.arange(5 * TILE, 6 * TILE)
    lists = []
    for t in range(11):
        m = rng.random(max_doc) < (0.95 if t < 8 else 0.02)
        m[6 * TILE:] = rng.random(max_doc - 6 * TILE) < 0.01
        m[t5] = t < 8
        if t == 8:
            m[5 * TILE + 517] = True
        d = np.nonzero(m)[0].astype(np.uint32)
        lists.append((d, rng.integers(1, 11, size=len(d)).astype(np.uint32)))
    alive = packed(rng.random(max_doc) > 0.1)
    seg = Seg(lists, _lengths(rng, max_doc), alive)
    fx = Fixture.__new__(Fixture)
    fx.segs, fx._has = [seg], {}

    def shapes(with8):
        out = [(TQ_OP_TERM, [t], None, None, 0, None) for t in range(8)] + [
            (TQ_OP_AND, [0, 1], None, None, 0, None), (TQ_OP_AND, list(range(8)), None, None, 0, None),
            (TQ_OP_OR, [0, 9], None, None, 0, None), (TQ_OP_BOOL, list(range(8)), [S] * 8, None, 7, None),
            (TQ_OP_BOOL, list(range(8)), [S] * 8, None, 8, None), (TQ_OP_BOOL, [0, 9, 10], [R, X, S], None, 0, None)]
        if with8:
            out += [(TQ_OP_TERM, [8], None, None, 0, None), (TQ_OP_OR, [8, 9], None, None, 0, None), (TQ_OP_OR, list(range(9)), None, None, 0, None)]
        return [fx.query(sh, 10) for sh in out]

    filt = rng.random(max_doc) < 0.5
    lo, hi = 37, max_doc - 11
    rmask = np.zeros(max_doc, bool)
    rmask[lo:hi] = True
    for with8 in (False, True):
        c = fx.register(_ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, TQ_TILE_BIG_MIN=100000))
        try:
            qts = shapes(with8)
            st = _check(c, fx, qts, ("whole", with8))
            assert st["tile_groups"] == 1, st
            c.filter_register(7, seg.ord, packed(filt))
            c.segment_set_doc_range(seg.ord, 0, lo, hi)
            _check(c, fx, qts, ("range", with8), masks={seg: rmask})
            _check(c, fx, qts, ("filter + range", with8), masks={seg: rmask & filt}, filt=7)
        finally:
            c.close()


# ---- a segment of 2^31 - 2 docs ------------------------------------------------------------------------------------------------
def test_segment_of_2_to_the_31_docs():
    """No fieldnorms; 32 lists in the top 300 000 docs and at max_doc - 1; random BOOL shapes and 32 SHOULD clauses, as count hits
    on the tile engine (default, every list dense) and through tq_count_batch; the model on the compacted doc space."""
    rng = np.random.default_rng(0x7FFF)
    max_doc = 2**31 - 2
    top = max_doc - 300_000
    lists = []
    for p in rng.permutation(np.geomspace(0.0005, 0.2, NL)):
        d = np.union1d(top + np.nonzero(rng.random(max_doc - top) < p)[0], [max_doc - 1]).astype(np.uint32)
        lists.append((d, rng.integers(1, 9, size=len(d)).astype(np.uint32)))
    so = fresh_ord()
    seg = OracleSegment(lists, None, segment_ord=so, writer_cls=T.FieldWriter, max_doc=max_doc)
    cm = M.Compacted(so, lists, max_doc)
    shapes = [dict(terms=list(range(NL)), occurs=[S] * NL, groups=[0] * NL, msm=3, flags=[0] * NL, k=10)]
    shapes += random_bool_shapes(rng, 20, NL, n_wide=3)
    qs = []
    for sh in shapes:
        q = bool_query(make_query(TQ_OP_OR, [seg], sh["terms"], sh["k"]), sh["occurs"], sh["groups"], sh["msm"])
        q["term_flags"] = list(sh["flags"])
        qs.append((q, sh["terms"]))
    want = [M.count_compacted([cm], q, t) for q, t in qs]
    assert want[0] > 0
    for env in (dict(), dict(TQ_TILE_BIG_MIN=1)):
        c = _ctx_with_env(TQ_TILE=1, **env)
        try:
            seg.register(c)
            rows, got, _ = _run(c, [dict(q, count_hits=True) for q, _ in qs])
            assert [int(x) for x in got] == want, env
            plain = c.search_batch(QueryBatch([q for q, _ in qs]))
            for i in range(len(qs)):
                assert hits(rows, i) == hits(plain, i), (env, i)
            if not env:
                assert [int(x) for x in c.count_batch(QueryBatch([q for q, _ in qs]))] == want
        finally:
            c.close()
