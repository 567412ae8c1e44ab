"""Every query path at doc ids from 2^24 up to 2^31 - 2 against the score model (tests/score_model.py), bit for bit (zero scores
by value: the device returns +0.0 for -0.0).  Tantivy allows a segment of TERMINATED - 1 = 2^31 - 2 docs; every other test queries
segments of at most 12.5M docs, so a doc id rounded through f32 (exact only below 2^24), kept in a narrow field or multiplied past
32 bits would pass them all.

The model cannot hold a 2^31-doc segment (about 25 bytes per doc and query), so it runs on a compacted doc space
(score_model.Compacted, proved against the plain model in test_score_model_compacted.py).  The segments are written directly from
uint8 fieldnorm-id arrays:
  H0  max_doc 2^31 - 2, no fieldnorms, no deletes: docs at 0, 2^24 - 1, 2^24, 2^24 + 1, 2^30 +- 1 and max_doc - 1; one 128-doc
      block with a gap of 2^30 (doc width 31); lists of 1 / 127 / 128 / 129 / 257 docs ending at max_doc - 1; a list of 2.6M
      postings (a dense slot under TQ_TILE_BIG_MIN=1, with a tile index over 2M tiles); 40 000 consecutive docs below max_doc,
      which the planner's density estimate misses (the tiles there overflow and the batch is repeated); 30 000 docs above 2^30
      with tf 1, which all tie (more than a CTA buffer of candidates reaches k_final);
  H1  max_doc 2^31 - 2 with fieldnorm ids (each of 0..255 at a listed doc, the last doc included) and deletes around 2^24, 2^30
      and in the last, partial byte of the alive bitset;
  H2  a phrase segment of 2^26 + 5 docs, positions at docs above 2^24 and at max_doc - 1, deletes;
  S   an ordinary segment of 50 000 docs: merged rows mix small and large doc ids over segment ordinals.
Paths: both engines, the tile-engine routes and overflow hooks, the per-query kernels' unit cuts, the phrase routes, Count,
doc-range parts, tq_multi's split registration and CrossGpuMerger's packed rows and k_merge."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM, TQ_RECORD_FREQS, TQ_TERM_IGNORE_FREQ, QueryBatch  # noqa: E402
from tantivy_b200.sharding import CrossGpuMerger, doc_range, merge_rows_host  # noqa: E402
from tests import score_model as M  # noqa: E402
from tests.helpers import _FN_TABLE, hits, make_query, random_bool_shapes, shape_query  # noqa: E402
from tests.test_gpu_parity import TILE_OVERFLOW_HOOKS, TILE_PATH_HOOKS, _ctx_with_env  # noqa: E402
from tests.test_gpu_phrase import PosSegment, phrase_query  # noqa: E402
from tests.test_gpu_phrase_edges import ROUTES  # noqa: E402
from tests.test_gpu_query_kernels import HOOKS  # noqa: E402
from tests.test_gpu_shard_exchange import merged_rows, run_ranks  # noqa: E402

MAXD = 0x7FFFFFFE          # TERMINATED - 1: the largest max_doc there is
B24, B30 = 1 << 24, 1 << 30
H2D = (1 << 26) + 5
KMAX = 1024
KS = (1, 10, 128, 129, 1024)
EDGE, WIDE, T1, T127, T128, T129, T257, BIG, CLUSTER, TIES, MID = range(11)
N_TERMS = 11
TAILS = {T1: 1, T127: 127, T128: 128, T129: 129, T257: 257}
EDGE_DOCS = np.array([0, B24 - 1, B24, B24 + 1, B30 - 1, B30 + 1, MAXD - 1], np.uint32)


def _rows(rows):
    return [(float(s), int(g), int(d)) for s, g, d in rows]


class Seg:
    """One segment written by the product's writer from a fieldnorm-id array (None: no fieldnorms), and its compacted model.
    lists = {term: (docs, tfs)}; terms without a list have no postings here."""

    def __init__(self, so, lists, max_doc, fn_ids=None, alive=None, tokens=None):
        self.segment_ord, self.max_doc, self.fn_ids, self.alive = so, max_doc, fn_ids, alive
        self.record_option = TQ_RECORD_FREQS
        self.total_num_tokens = max_doc if fn_ids is None else tokens
        full = [lists.get(t, (np.zeros(0, np.uint32), np.zeros(0, np.uint32))) for t in range(N_TERMS)]
        w = T.FieldWriter(TQ_RECORD_FREQS, self.total_num_tokens, fn_ids, max_doc)
        self.terms = []
        for d, tf in full:
            self.terms.append((len(d), *w.add_term(d, tf)) if len(d) else (0, 0, 0))
        self.body = w.body()
        del w
        self.model = M.Compacted(so, full, max_doc, fn_ids=fn_ids, alive=alive)

    def term_seg(self, t, clause=0):
        df, s, e = self.terms[t]
        return (clause, self.segment_ord, 0, df, s, e)

    def register(self, target, doc_range_=None):
        target.segment_register(self.segment_ord, 0, self.max_doc, self.record_option, self.body, self.fn_ids, self.alive)
        if doc_range_ is not None:
            target.segment_set_doc_range(self.segment_ord, 0, *doc_range_)


def _tfs(rng, n, hi=16):
    return rng.integers(1, hi + 1, size=n).astype(np.uint32)


def _with(docs, extra):
    return np.union1d(np.asarray(docs, np.uint32), np.asarray(extra, np.uint32)).astype(np.uint32)


def _common_lists(rng, big_n, mid_n, ties_n):
    """The lists H0 and H1 share in shape (each segment draws its own): every list holds max_doc - 1."""
    last = [MAXD - 1]
    b = MAXD - 64
    wide = np.concatenate([np.arange(b - B30 - 63, b - B30 + 1), np.arange(b, MAXD)]).astype(np.uint32)  # one gap of 2^30
    lists = {EDGE: (EDGE_DOCS, np.array([3, 9, 12, 7, 5, 15, 11], np.uint32)), WIDE: (wide, _tfs(rng, 128, 20))}
    for t, n in TAILS.items():
        d = (MAXD - 1 - 3 * np.arange(n)[::-1]).astype(np.uint32)
        lists[t] = (d, _tfs(rng, n, 30))
    big = _with(rng.integers(0, MAXD, size=big_n, dtype=np.int64), list(EDGE_DOCS))
    lists[BIG] = (big, _tfs(rng, len(big), 1 << 16))  # (tf <= 16 without fieldnorms: 160 000 docs would tie at the top score)
    lists[CLUSTER] = (np.arange(MAXD - 40_000, MAXD, dtype=np.uint32), _tfs(rng, 40_000, 4))
    # two tied docs just below 2^30, whose low 24 bits (0xFFFFF9, 0xFFFFFF) sort after those of the ties above it: a merge of the
    # halves [0, 2^30) and [2^30, max_doc) that broke ties on a cut doc id would put them last
    ties = _with(B30 + 5 + 3 * np.arange(ties_n), last + [B30 - 7, B30 - 1])
    lists[TIES] = (ties, np.ones(len(ties), np.uint32))
    mid = _with(rng.integers(0, MAXD, size=mid_n, dtype=np.int64), [B24, B30 + 1, MAXD - 1])
    lists[MID] = (mid, _tfs(rng, len(mid)))
    return lists


def _h0(rng):
    return Seg(0, _common_lists(rng, 2_600_000, 200_000, 30_000), MAXD)


def _h1(rng):
    lists = _common_lists(rng, 300_000, 100_000, 20_000)
    del lists[TIES]  # (the ties are H0's alone)
    ids_at = _with(B24 - 300 + 7 * np.arange(100), B30 + 11 * np.arange(155))  # 255 docs around 2^24 and above 2^30
    ids_at = ids_at[ids_at != MAXD - 1][:255]
    assert len(ids_at) == 255
    lists[EDGE] = (_with(EDGE_DOCS, ids_at), None)
    lists[EDGE] = (lists[EDGE][0], _tfs(rng, len(lists[EDGE][0]), 40))
    base = 20
    fn = np.full(MAXD, base, np.uint8)  # 2 GiB
    listed = np.unique(np.concatenate([d for d, _ in lists.values()]))
    fn[listed] = rng.integers(0, 256, size=len(listed)).astype(np.uint8)
    fn[ids_at] = np.arange(255, dtype=np.uint8)
    fn[MAXD - 1] = 255
    tab = _FN_TABLE.astype(np.int64)
    tokens = int(MAXD * tab[base] + (tab[fn[listed]] - tab[base]).sum())
    alive = np.full((MAXD + 7) // 8, 0xFF, np.uint8)  # 256 MiB
    alive[-1] = (1 << (MAXD % 8)) - 1  # the last byte holds 6 docs
    dead = [B24 - 1, B24 + 1, B30 - 1, B30 + 3, MAXD - 2, MAXD - 5]
    dead += [int(d) for d in rng.choice(listed, size=len(listed) // 5, replace=False) if d not in (B24, B30 + 1, MAXD - 1)]
    dead = np.asarray(dead, np.int64)
    np.bitwise_and.at(alive, dead >> 3, ~(np.left_shift(1, dead & 7)).astype(np.uint8))
    return Seg(1, lists, MAXD, fn_ids=fn, alive=alive, tokens=tokens), ids_at


def _s(rng):
    n = 50_000
    lengths = np.clip(np.round(np.exp(rng.normal(np.log(30), 0.8, size=n))), 1, 3000).astype(np.uint32)
    fn = (np.searchsorted(_FN_TABLE, lengths, side="right") - 1).astype(np.uint8)
    lists = {}
    for t, p in zip([EDGE, WIDE, T127, T257, BIG, CLUSTER, MID], (0.02, 0.05, 0.01, 0.02, 0.2, 0.1, 0.1)):
        d = np.nonzero(rng.random(n) < p)[0].astype(np.uint32)
        lists[t] = (d, _tfs(rng, len(d)))
    return Seg(2, lists, n, fn_ids=fn, tokens=int(_FN_TABLE[fn].sum()))


# ---- queries and the model's rows ----------------------------------------------------------------------------------------
def _q(segs, op, terms, k, **extra):
    q = make_query(op, segs, terms, k)
    q.update(extra)
    return q, list(terms)


AND_SMALL = [[EDGE, BIG], [BIG, MID], [TIES, BIG, MID], [WIDE, T257], [T129, BIG, EDGE]]
AND_WIDE = [[EDGE, BIG, MID, TIES], [BIG, T129, TIES, MID, WIDE], [EDGE, WIDE, T1, BIG, TIES, MID, T257, T128]]
OR_SETS = [[EDGE, WIDE], [BIG, MID], [TIES, MID], [EDGE, T1, T127, T128, T129, T257, WIDE],
           [BIG, MID, TIES, EDGE, WIDE, T1, T127, T129, T257]]
OR_32 = [t for t in range(40) if t % N_TERMS != CLUSTER][:32]


def _main_queries(segs):
    """TERM, AND of 2-3 and of 4-8 MUST clauses (both summation orders), OR of 2-9 and of 32 clauses, initial thresholds: none over
    the cluster (no tile overflows)."""
    qs = [_q(segs, TQ_OP_TERM, [t], k) for t in range(N_TERMS) if t != CLUSTER for k in KS]
    for c in AND_SMALL:
        qs += [_q(segs, TQ_OP_AND, c, k) for k in (1, 10, 1024)]
    for c in AND_WIDE:  # one clause without freqs: Intersection::score's order instead of one after another
        qs += [_q(segs, TQ_OP_AND, c, k) for k in (10, 1024)]
        qs += [_q(segs, TQ_OP_AND, c, k, term_flags=[0] * (len(c) - 1) + [TQ_TERM_IGNORE_FREQ]) for k in (10, 1024)]
    for c in OR_SETS:
        qs += [_q(segs, TQ_OP_OR, c, k) for k in KS]
    qs += [_q(segs, TQ_OP_OR, [t % N_TERMS for t in OR_32], k) for k in (10, 1024)]
    return qs


def _cluster_queries(segs):
    """Unions and intersections over the 40 000 consecutive docs below max_doc."""
    qs = [_q(segs, TQ_OP_TERM, [CLUSTER], k) for k in (10, 1024)]
    qs += [_q(segs, TQ_OP_OR, [CLUSTER, T257, T129, BIG], k) for k in (1, 129, 1024)]
    qs += [_q(segs, TQ_OP_AND, [CLUSTER, BIG], k) for k in (10, 1024)]
    qs += [_q(segs, TQ_OP_AND, [CLUSTER, T127, T257, WIDE], 10)]
    return qs


def _bool_queries(segs, rng):
    out = []
    for sh in random_bool_shapes(rng, 12, N_TERMS, n_wide=1):
        sh["terms"] = [BIG if t == CLUSTER else t for t in sh["terms"]]
        q = make_query(TQ_OP_OR, segs, sh["terms"], sh["k"], boost=list(sh["boosts"]))
        out.append((shape_query(q, sh), sh["terms"]))
    return out


def _with_thresholds(segs, rows_of):
    """Initial thresholds just below, at and just above the k-th score."""
    out = []
    for c, op in (([BIG], TQ_OP_TERM), ([BIG, MID], TQ_OP_OR), ([EDGE, BIG], TQ_OP_AND)):
        for k in (10, 128):
            base = _q(segs, op, c, k)
            rows = rows_of(base)
            s = np.float32(rows[min(k, len(rows)) - 1][0])
            for thr in (np.nextafter(s, np.float32(-np.inf)), s, np.nextafter(s, np.float32(np.inf))):
                out.append((dict(base[0], threshold=float(thr)), c))
    return out


class Model:
    """The compacted model's rows and counts of queries over a set of segments, computed once per query shape."""

    def __init__(self, segs):
        self.csegs = [s.model for s in segs]
        self._rows, self._counts = {}, {}

    @staticmethod
    def _key(q, terms):
        return repr((q["op"], list(terms), q["weights"], q["term_segs"], q.get("term_flags"), q.get("term_occur"), q.get("term_group"),
                     q.get("min_should_match")))

    def rows(self, qt, doc_ranges=None):
        q, terms = qt
        key = (self._key(q, terms), repr(doc_ranges))
        if key not in self._rows:
            self._rows[key] = _rows(M.search_compacted(self.csegs, dict(q, k=KMAX, threshold=None), terms, doc_ranges=doc_ranges))
        rows = self._rows[key]
        thr = q.get("threshold")
        if thr is not None:
            rows = [r for r in rows if np.float32(r[0]) > np.float32(thr)]
        return rows[:q["k"]]

    def count(self, qt, doc_ranges=None):
        q, terms = qt
        key = (self._key(q, terms), repr(doc_ranges))
        if key not in self._counts:
            self._counts[key] = M.count_compacted(self.csegs, q, terms, doc_ranges=doc_ranges)
        return self._counts[key]


class Battery:
    def __init__(self, model, queries):
        self.queries = queries
        self.qb = QueryBatch([q for q, _ in queries])
        self.want = [model.rows(qt) for qt in queries]
        self.counts = [model.count(qt) for qt in queries]

    def check(self, result, what):
        for i, w in enumerate(self.want):
            got = hits(result, i)
            q, t = self.queries[i]
            assert got == w, (what, i, q["op"], t, q["k"], got[:4], w[:4])


class Fixture:
    def __init__(self):
        rng = np.random.default_rng(0x7FFFFFFE)
        self.h0 = _h0(rng)
        self.h1, self.h1_ids = _h1(rng)
        self.s = _s(rng)
        self.segs = [self.h0, self.h1, self.s]
        self.model = Model(self.segs)
        main = _main_queries(self.segs)
        main += _with_thresholds(self.segs, self.model.rows)
        # a term of 2.6M postings spread over 2M tiles: from k = 10 on, more docs clear the sampled threshold than a candidate
        # region holds, and the batch is repeated (exact, asserted); the rest of the battery stays on the tile engine
        big = [qt for qt in main if qt[1] == [BIG] and qt[0]["k"] >= 10]
        self.big_term = Battery(self.model, big)
        self.main = Battery(self.model, [qt for qt in main if qt not in big])
        self.cluster = Battery(self.model, _cluster_queries(self.segs))
        self.bools = Battery(self.model, _bool_queries(self.segs, rng))
        self.unions = Battery(self.model, [qt for qt in main if qt[0]["op"] == TQ_OP_OR])

    def register(self, ctx):
        for s in self.segs:
            s.register(ctx)
        return ctx


def _reach(fx):
    """The batteries return what they are about."""
    rows = [r for b in (fx.main, fx.cluster, fx.big_term, fx.bools) for w in b.want for r in w]
    h0 = {d for _, g, d in rows if g == 0}
    h1 = {d for _, g, d in rows if g == 1}
    for docs in (h0, h1):
        assert MAXD - 1 in docs and any(d >= B24 for d in docs) and any(d >= (1 << 31) - 130 for d in docs)
        assert any(B30 <= d < MAXD - 40_000 for d in docs)
    assert {B24, B24 + 1, B30 + 1, 0} <= h0
    assert B24 in h1 and B24 + 1 not in h1 and B24 - 1 not in h1 and MAXD - 2 not in h1  # deleted docs stay out
    assert {g for _, g, _ in rows} == {0, 1, 2}
    ties = next(w for (q, t), w in zip(fx.main.queries, fx.main.want) if t == [TIES] and q["k"] == KMAX and "threshold" not in q)
    h0_ties = fx.h0.model.docs[fx.h0.model.seg.lists[TIES][0]]
    assert len(h0_ties) > 10 * 2048 and [(g, d) for _, g, d in ties] == [(0, int(d)) for d in h0_ties[:KMAX]]
    assert len({s for s, _, _ in ties}) == 1  # one tied score
    assert sum(len(w) for w in fx.main.want) > 5000
    assert len(np.unique(fx.h1.fn_ids[fx.h1.model.docs])) == 256 and fx.h1.fn_ids[MAXD - 1] == 255
    assert len(np.unique(fx.h1.fn_ids[np.asarray(sorted(h1), np.int64)])) > 100


@pytest.fixture(scope="module")
def fx():
    f = Fixture()
    _reach(f)
    return f


def _check_counts(c, battery, what):
    got = c.count_batch(battery.qb)
    assert list(got) == battery.counts, (what, [(i, int(a), b) for i, (a, b) in enumerate(zip(got, battery.counts)) if a != b][:4])


# ---- every shape on both engines ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["tile", "legacy"])
def test_every_shape_on_both_engines(fx, engine):
    tile = engine == "tile"
    c = fx.register(_ctx_with_env(TQ_TILE=1 if tile else 0, TQ_TILE_TERMS=1))
    try:
        fx.main.check(c.search_batch(fx.main.qb), (engine, "main"))
        st = c.stats()
        assert st["tile_fallbacks"] == 0 and (st["tile_groups"] >= 1) == tile, st
        for b, name in ((fx.cluster, "cluster"), (fx.big_term, "big term")):  # (the cluster's tiles overflow the estimated buffer)
            b.check(c.search_batch(b.qb), (engine, name))
            assert c.stats()["tile_fallbacks"] == (1 if tile else 0), (name, c.stats())
        if tile:
            fx.bools.check(c.search_batch(fx.bools.qb), (engine, "bool"))
        for b, name in ((fx.main, "main"), (fx.cluster, "cluster"), (fx.big_term, "big term"), (fx.bools, "bool")):
            _check_counts(c, b, (engine, name))
    finally:
        c.close()


# ---- routes ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hook", TILE_PATH_HOOKS + TILE_OVERFLOW_HOOKS, ids=lambda h: ",".join(f"{k}={v}" for k, v in h.items()))
def test_tile_routes(fx, hook):
    overflow = hook in TILE_OVERFLOW_HOOKS
    c = fx.register(_ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, **hook))
    try:
        fx.main.check(c.search_batch(fx.main.qb), hook)
        st = c.stats()
        assert st["tile_groups"] >= 1
        # without a sample launch the first exact launch hands over every match of its tiles: the k = 1024 unions overflow
        # their candidate regions and the batch is repeated on the per-query kernels
        assert st["tile_fallbacks"] == (1 if overflow or "TQ_TILE_SAMPLE_DIV" in hook else 0), st
        fx.unions.check(c.search_batch(fx.unions.qb), (hook, "unions"))
        st = c.stats()
        assert st["tile_groups"] >= 1 and st["tile_groups_union_only"] == st["tile_groups"], st
        fx.bools.check(c.search_batch(fx.bools.qb), (hook, "bool"))
    finally:
        c.close()


def _per_query_batteries(fx, hook):
    """Under unit cuts of one or a few tiles / windows a union over 2^31 docs hands over 2k candidates per unit (2M strip units and
    262 144 k_or units per segment): there the unions over all three segments run with k = 1, and the unions over H0 and S alone
    with k = 10; everything else at every k."""
    if hook not in ("smallest", "odd"):
        return [fx.main]
    if not hasattr(fx, "small_k"):
        fx.small_k = Battery(fx.model, [qt for qt in fx.main.queries if qt[0]["op"] != TQ_OP_OR or qt[0]["k"] == 1])
        h0s = [fx.h0, fx.s]
        fx.small_k_h0s = Battery(Model(h0s), [_q(h0s, TQ_OP_OR, c, 10) for c in OR_SETS])
    return [fx.small_k, fx.small_k_h0s]


@pytest.mark.parametrize("hook", [h for h in HOOKS if h != "default"])
def test_per_query_kernel_unit_cuts(fx, hook):
    c = fx.register(_ctx_with_env(TQ_TILE=0, **HOOKS[hook]))
    try:
        for b in _per_query_batteries(fx, hook):
            b.check(c.search_batch(b.qb), hook)
            st = c.stats()
            assert st["tile_groups"] == 0 and st["units_or"] > 0, st
            if b is not getattr(fx, "small_k_h0s", None):
                assert st["units_term"] > 0 and st["units_and"] > 0, st
    finally:
        c.close()


# ---- phrases on a 2^26 + 5 doc segment --------------------------------------------------------------------------------------
def _h2():
    rng = np.random.default_rng(226)
    docs = _with(rng.integers(B24, H2D, size=3000, dtype=np.int64), [H2D - 1, B24, B24 + 1])
    docs = _with(docs, rng.integers(0, B24, size=300, dtype=np.int64))
    p = {"p0": {}, "p1": {}, "p2": {}}
    for d in docs.tolist():
        a = sorted(set(rng.integers(0, 40, size=int(rng.integers(1, 4))).tolist()))
        p["p0"][d] = a
        if rng.random() < 0.7 or d == H2D - 1:
            p["p1"][d] = sorted({x + 1 for x in a} | ({int(rng.integers(0, 40))} if rng.random() < 0.3 else set()))
        if rng.random() < 0.5:
            p["p2"][d] = sorted({x + 2 for x in a})
    p["c0"] = {d: [0] for d in range(H2D - 20_000, H2D, 2)}  # every other doc: the union's tiles overflow under TQ_TILE_PCAP
    lengths = np.full(H2D, 12, np.uint32)
    lengths[docs] = rng.integers(3, 200, size=len(docs))
    alive_b = np.ones(H2D, bool)
    alive_b[rng.choice(docs, size=len(docs) // 5, replace=False)] = False
    alive_b[[H2D - 1, B24]] = True
    alive_b[B24 + 1] = False
    alive = np.packbits(alive_b, bitorder="little")
    ps = PosSegment.from_positions(p, lengths, alive=alive)
    lists = [(np.array(sorted(p[t]), np.uint32), np.array([len(p[t][d]) for d in sorted(p[t])], np.uint32)) for t in ps.vocab]
    model = M.Compacted(ps.ord, lists, H2D, fn_ids=ps.seg.fn_ids, alive=alive, positions=[p[t] for t in ps.vocab])
    qs = []
    for ph, off, slop in ((["p0", "p1"], None, 0), (["p0", "p1", "p2"], None, 0), (["p1", "p0"], [1, 0], 0), (["p0", "p2"], [0, 2], 0),
                          (["p0", "p1"], None, 1), (["p1", "p0"], [1, 0], 2)):
        for k in (1, 10, 128, 1024):
            q = phrase_query([ps], ph, k, offsets=off)[0]
            if slop:
                q["slop"] = slop
            qs.append((q, [ps.vocab.index(t) for t in ph]))
    n_docs, avg = ps.n_docs, np.float32(np.float32(ps.tokens) / np.float32(ps.n_docs))
    for k in (10, 1024):  # a union next to the phrases: a tile group
        ts = [ps.vocab.index("c0"), ps.vocab.index("p0")]
        weights = [T.bm25_weight(ps.term(t)[0], n_docs) for t in ("c0", "p0")]
        term_segs = [(c, ps.ord, 0, *ps.term(t)[:3]) for c, t in enumerate(("c0", "p0"))]
        qs.append((dict(op=TQ_OP_OR, k=k, weights=weights, avg_fieldnorm=[avg] * 2, term_segs=term_segs), ts))
    want = [_rows(M.search_compacted([model], q, t)) for q, t in qs]
    got = {d for w in want for _, _, d in w}
    assert H2D - 1 in got and any(B24 < d < H2D - 20_000 for d in got) and B24 + 1 not in got
    assert all(len(w) > 0 for w in want)
    return ps, qs, want


@pytest.fixture(scope="module")
def h2():
    return _h2()


@pytest.mark.parametrize("route", list(ROUTES))
def test_phrases_above_2_to_the_24_on_every_route(h2, route):
    ps, qs, want = h2
    c = _ctx_with_env(**ROUTES[route])
    try:
        ps.register(c)
        g = c.search_batch(QueryBatch([q for q, _ in qs]))
        for i, w in enumerate(want):
            assert hits(g, i) == w, (route, i, hits(g, i)[:4], w[:4])
        st = c.stats()
        assert st["units_phrase"] > 0
        if route in ("side_stream", "one_stream"):
            assert st["tile_groups"] >= 1 and st["tile_fallbacks"] == 0
        if route in ("no_tile", "small_units"):
            assert st["tile_groups"] == 0
        if route == "repeated":
            assert st["tile_fallbacks"] == 1
    finally:
        c.close()


# ---- doc-range parts, tq_multi's split and the sharded hand-over ---------------------------------------------------------
CUTS = [0, B24, B24 + 1, B30 + 3, MAXD - 1, MAXD]


@pytest.fixture(scope="module")
def halves(fx):
    """A battery over H0 and H1 alone (the segments that are split)."""
    segs = [fx.h0, fx.h1]
    model = Model(segs)
    qs = [_q(segs, TQ_OP_TERM, [t], k) for t in (EDGE, WIDE, T257, BIG, TIES, MID) for k in (10, 1024)]
    qs += [_q(segs, TQ_OP_AND, c, k) for c in AND_SMALL[:3] + AND_WIDE[:2] for k in (10, 1024)]
    qs += [_q(segs, TQ_OP_OR, c, k) for c in OR_SETS for k in (10, 1024)]
    qs += _bool_queries(segs, np.random.default_rng(31))[:6]
    return segs, model, Battery(model, qs)


def test_doc_range_parts_merge_to_the_whole_segment(halves):
    """Parts [0, 2^24), [2^24, 2^24 + 1), [2^24 + 1, 2^30 + 3), an empty one, [2^30 + 3, max_doc - 1), [max_doc - 1, max_doc) of H0
    and H1, each on a context of its own: every part returns docs of its range only; merged like segment fruits the parts' rows are
    the whole segments' rows, and their Counts add up to the whole Count."""
    segs, model, b = halves
    parts = list(zip(CUTS[:-1], CUTS[1:]))
    parts.insert(3, (B30 + 3, B30 + 3))
    rows, counts = [], np.zeros(b.qb.nq, np.uint64)
    for lo, hi in parts:
        c = T.Context(0)
        try:
            for s in segs:
                s.register(c, (lo, hi))
            r = c.search_batch(b.qb)
            for i in range(b.qb.nq):
                assert all(lo <= d < hi for _, _, d in hits(r, i)), ((lo, hi), i)
            rows.append([np.array(x) for x in r])
            counts += c.count_batch(b.qb)
        finally:
            c.close()
    assert list(counts) == b.counts
    m = merge_rows_host(*[np.stack([r[j] for r in rows]) for j in range(4)], b.qb.kmax)
    for i, (w, (q, _)) in enumerate(zip(b.want, b.queries)):
        n = min(int(m[3][i]), q["k"])
        assert [(float(m[0][i, j]), int(m[1][i, j]), int(m[2][i, j])) for j in range(n)] == w, i
    top = {d for w in b.want for _, _, d in w}
    assert {B24, MAXD - 1} <= top and any(B30 + 3 <= d < MAXD - 1 for d in top) and any(B24 + 1 <= d < B30 + 3 for d in top)


@pytest.mark.parametrize("n_ctx", [2, 3])
def test_multi_handle_split_of_a_2_to_the_31_doc_segment(halves, n_ctx):
    """tq_multi_segment_register_split of H0 and H1 over two contexts (cut at 2^30) and three (cut at a multiple of 1024 that is
    not a power of two): the rows of the whole segments."""
    segs, model, b = halves
    cut = doc_range(MAXD, 0, n_ctx)[1]
    assert cut == (B30 if n_ctx == 2 else 715_828_224) and cut % 1024 == 0
    m = T.MultiContext([0] * n_ctx)
    try:
        for s in segs:
            m.segment_register_split(s.segment_ord, 0, s.max_doc, s.record_option, s.body, s.fn_ids, s.alive)
        g = m.search_batch(b.qb)
    finally:
        m.close()
    for i, w in enumerate(b.want):
        assert hits(g, i) == w, (n_ctx, i, hits(g, i)[:4], w[:4])
    docs = {d for i in range(b.qb.nq) for _, _, d in hits(g, i)}
    assert any(d < cut for d in docs) and any(d >= cut for d in docs)


def test_sharded_handover_of_doc_ids_above_2_to_the_30(halves):
    """CrossGpuMerger at world 2, each rank holding one half of H0 and H1 (cut at 2^30): the packed rows and k_merge carry the doc
    ids unchanged, and the merged rows are the whole segments'."""
    pytest.importorskip("torch")
    segs, model, b = halves
    ctxs = [T.Context(0) for _ in range(2)]
    got = [None, None]
    try:
        for r in range(2):
            for s in segs:
                s.register(ctxs[r], doc_range(MAXD, r, 2))

        def rank(r, dist):
            bt = ctxs[r].prepare(b.qb)
            try:
                m = CrossGpuMerger(ctxs[r], dist, "cuda:0", b.qb.nq, b.qb.kmax)
                m.run(bt)
                m(bt)
                got[r] = merged_rows(m.fetch_host(bt), b.qb.nq)
            finally:
                bt.close()
        run_ranks(2, rank)
    finally:
        for c in ctxs:
            c.close()
    ties = next(w for (q, t), w in zip(b.queries, b.want) if t == [TIES] and q["k"] == 10)
    assert [d for _, _, d in ties[:3]] == [B30 - 7, B30 - 1, B30 + 5]  # tied rows from both ranks, in doc order across the cut
    for r in range(2):
        for i, w in enumerate(b.want):
            assert got[r][i] == w, (r, i, got[r][i][:4], w[:4])
    assert any(d >= B30 for w in got[0] for _, _, d in w) and any(d < B30 for w in got[0] for _, _, d in w)
