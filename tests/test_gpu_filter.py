"""Filtered search (TQ_QUERY_FILTER, FilterCollector around TopDocs and Count): a filtered query on a context returns what the same
unfiltered query returns on segments registered with alive := alive AND filter.  Rows are checked bit for bit and counts exactly
against the score model (tests/score_model.py) over those segments, and against device contexts and the oracle that hold them.
Filter kinds: all ones (rows equal the unfiltered query's), all zeros, Bernoulli 1 % and 30 %, one contiguous run, single bits on
both sides of the 1024- and 8192-doc tile edges, bits only on deleted docs; a segment without deletes (the Count shortcut is
bypassed).  Shapes: TERM, AND of 2-5, OR of 2-20, every BOOL_SHAPES entry (tile engine), phrases of 2-8 terms and sloppy two-term
phrases; k of 1 / 10 / 1000, with and without thresholds, on both engines.  Routes: every tile hook, several groups, batches split
by the scratch budget, single-term batches on k_term, one batch mixing unfiltered queries and three filters.  Skipping, doc-range
parts, MultiContext, CrossGpuMerger, a phased run with imported thresholds, a segment of 2^31 - 2 docs, and the lifetime and error
rules of the filter registry."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from oracle import tq_oracle as O  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM, QueryBatch  # noqa: E402
from tantivy_b200.sharding import CrossGpuMerger, doc_range  # noqa: E402
from tests import score_model as M  # noqa: E402
from tests.helpers import BOOL_SHAPES, OracleSegment, bool_query, hits, make_query  # noqa: E402
from tests.test_gpu_parity import TILE_OVERFLOW_HOOKS, TILE_PATH_HOOKS, _ctx_with_env, fresh_ord  # noqa: E402
from tests.test_gpu_shard_exchange import merged_rows, run_ranks  # noqa: E402

N_TERMS = 24
DENS = (0.3, 0.1, 0.05, 0.01, 0.002, 0.2)
KS = (1, 10, 1000)
AND_SETS = [[0, 1], [1, 3], [0, 2, 4], [5, 0, 1, 2], [6, 7, 8, 9, 11]]
OR_SETS = [[0, 4], [3, 9], [1, 2, 3], [0, 6, 12, 18, 4], list(range(2, 22, 2)), list(range(20)), [23, 22]]
KINDS = ("ones", "zeros", "bern1", "bern30", "run", "edges", "deleted")
FID = {k: 10 + i for i, k in enumerate(KINDS)}


def packed(mask):
    return np.packbits(np.asarray(mask, bool), bitorder="little")


def unpacked(bits, n):
    return np.unpackbits(np.asarray(bits, np.uint8), bitorder="little", count=n).astype(bool)


def filter_mask(kind, max_doc, alive_mask, rng):
    m = np.zeros(max_doc, bool)
    if kind == "ones":
        m[:] = True
    elif kind == "bern1":
        m = rng.random(max_doc) < 0.01
    elif kind == "bern30":
        m = rng.random(max_doc) < 0.3
    elif kind == "run":
        m[max_doc // 3:max_doc // 3 + max_doc // 7] = True
    elif kind == "edges":
        for e in range(1024, max_doc, 1024):
            if e % 8192 == 0 or e % 5120 == 0:
                m[e - 1] = m[e] = True
    elif kind == "deleted":
        m = ~alive_mask
    return m


class Fixture:
    """Three segments (deletes in two; the third has none), terms absent from some segments, and every filter kind on each."""

    def __init__(self, seed=0xF17):
        rng = np.random.default_rng(seed)
        self.osegs, self.lists, self.lengths, self.alive = [], [], [], []
        for i in range(3):
            max_doc = int(rng.integers(40_000, 120_000))
            lengths = np.clip(np.round(np.exp(rng.normal(np.log(40), 0.7, size=max_doc))), 1, 4096).astype(np.uint32)
            lists = []
            for t in range(N_TERMS):
                p = DENS[t % len(DENS)] * float(rng.uniform(0.5, 1.5))
                docs = np.nonzero(rng.random(max_doc) < p)[0].astype(np.uint32)
                lists.append((docs, np.minimum(rng.geometric(0.6, size=len(docs)), 10).astype(np.uint32)))
            alive = None if i == 2 else packed(rng.random(max_doc) > 0.15)
            self.osegs.append(OracleSegment(lists, lengths, segment_ord=fresh_ord(), writer_cls=T.FieldWriter, alive=alive))
            self.lists.append(lists)
            self.lengths.append(lengths)
            self.alive.append(alive)
        for s, t in ((0, 6), (1, 3), (2, 1), (2, 23)):  # absent from some segments (the model follows the queries' term_segs)
            self.osegs[s].terms[t] = (0, 0, 0)
        self.bits = {k: [] for k in KINDS}
        for k in KINDS:
            for s in self.osegs:
                am = np.ones(s.max_doc, bool) if s.alive is None else unpacked(s.alive, s.max_doc)
                self.bits[k].append(packed(filter_mask(k, s.max_doc, am, rng)))
        self._models, self._rows, self._counts = {}, {}, {}

    def combined(self, kind, i):
        """alive AND filter of segment i: the segment the filtered query must behave like."""
        f = self.bits[kind][i]
        return f.copy() if self.alive[i] is None else np.bitwise_and(self.alive[i], f)

    def model(self, kind):
        """The model's segments with alive AND filter (kind None: the plain alive bits)."""
        if kind not in self._models:
            self._models[kind] = [M.Segment(s.segment_ord, self.lists[i], self.lengths[i],
                                            alive=self.alive[i] if kind is None else self.combined(kind, i))
                                  for i, s in enumerate(self.osegs)]
        return self._models[kind]

    def register(self, ctx, kinds=KINDS):
        for s in self.osegs:
            s.register(ctx)
        for k in kinds:
            for i, s in enumerate(self.osegs):
                ctx.filter_register(FID[k], s.segment_ord, self.bits[k][i])
        return ctx

    def register_combined(self, target, kind):
        """The same segments with alive := alive AND filter (unfiltered queries on them are the reference)."""
        for i, s in enumerate(self.osegs):
            target.segment_register(s.segment_ord, 0, s.max_doc, s.record_option, s.body, s.fn_ids, self.combined(kind, i))
        return target

    def query(self, op, terms, k, **extra):
        q = make_query(op, self.osegs, terms, k)
        q.update(extra)
        return q, list(terms)

    def _key(self, kind, q, terms, doc_ranges):
        return repr((kind, q["op"], terms, q.get("term_occur"), q.get("term_group"), q.get("min_should_match"), q["term_segs"], doc_ranges))

    def rows(self, kind, qt, doc_ranges=None):
        q, terms = qt
        key = self._key(kind, q, terms, doc_ranges)
        if key not in self._rows:
            self._rows[key] = M.search(self.model(kind), dict(q, k=1000, threshold=None), terms, doc_ranges=doc_ranges)
        rows = self._rows[key]
        thr = q.get("threshold")
        if thr is not None:
            rows = [r for r in rows if np.float32(r[0]) > np.float32(thr)]
        return rows[:q["k"]]

    def count(self, kind, qt, doc_ranges=None):
        q, terms = qt
        key = self._key(kind, q, terms, doc_ranges)
        if key not in self._counts:
            self._counts[key] = M.count(self.model(kind), q, terms, doc_ranges=doc_ranges)
        return self._counts[key]


@pytest.fixture(scope="module")
def fx():
    return Fixture()


@pytest.fixture(scope="module", params=["tile", "legacy"])
def ctx(request, fx):
    c = _ctx_with_env(TQ_TILE=1 if request.param == "tile" else 0, TQ_TILE_TERMS=1)
    c.engine = request.param
    fx.register(c)
    yield c
    c.close()


def _plain(fx):
    qs = [fx.query(TQ_OP_TERM, [t], k) for t in (0, 1, 3, 4, 23) for k in KS]
    qs += [fx.query(TQ_OP_AND, c, k) for c in AND_SETS for k in KS]
    qs += [fx.query(TQ_OP_OR, c, k) for c in OR_SETS for k in KS]
    return qs


def _bools(fx):
    out = []
    for terms, occurs, groups, msm in BOOL_SHAPES:
        for k in KS:
            q, _ = fx.query(TQ_OP_OR, terms, k)
            out.append((bool_query(q, occurs, groups, msm), list(terms)))
    return out


def _thresholds(fx, kind, qs):
    out = []
    for q, terms in qs:
        rows = fx.rows(kind, (q, terms))
        if rows:
            out.append((dict(q, threshold=float(rows[min(q["k"], len(rows)) - 1][0])), terms))
    return out


def _check(fx, ctx, qts, kinds, count=True):
    """qts[i] runs under filter kinds[i] (None: unfiltered): rows against the model, the Count half and tq_count_batch."""
    qb = QueryBatch([dict(q, filter=None if k is None else FID[k], count_hits=count and q["op"] != 3) for (q, _), k in zip(qts, kinds)])
    b = ctx.prepare(qb)
    try:
        b.run()
        g = b.fetch()
        got_hits = b.fetch_hits()
    finally:
        b.close()
    for i, (qt, k) in enumerate(zip(qts, kinds)):
        want = fx.rows(k, qt)
        assert hits(g, i) == want, (i, k, qt[0]["op"], qt[1], qt[0]["k"], hits(g, i)[:4], want[:4])
        if count:
            assert int(got_hits[i]) == fx.count(k, qt), (i, k, qt[1])
    if count:
        cnt = ctx.count_batch(qb)
        for i, (qt, k) in enumerate(zip(qts, kinds)):
            assert int(cnt[i]) == fx.count(k, qt), (i, k, qt[1])
    return g


@pytest.mark.parametrize("kind", KINDS)
def test_filter_kinds_on_every_shape(fx, ctx, kind):
    """TERM / AND / OR (+ BOOL on the tile engine), k of 1 / 10 / 1000, with and without thresholds: rows, hits and counts equal the
    model over alive AND filter."""
    qs = _plain(fx) + (_bools(fx) if ctx.engine == "tile" else [])
    qs = qs + _thresholds(fx, kind, qs)
    g = _check(fx, ctx, qs, [kind] * len(qs))
    if kind == "ones":  # all ones: bit-equal to the unfiltered query
        u = ctx.search_batch(QueryBatch([q for q, _ in qs]))
        for a, b in zip(g, u):
            assert np.array_equal(a, b)


@pytest.mark.parametrize("hook", TILE_PATH_HOOKS + TILE_OVERFLOW_HOOKS, ids=lambda h: ",".join(f"{k}={v}" for k, v in h.items()))
def test_every_tile_route_keeps_the_filter(fx, hook):
    """Every k_tile route and overflow repeat, a batch mixing unfiltered queries and three filters (the repeat keeps them)."""
    c = _ctx_with_env(TQ_TILE=1, **hook)
    try:
        fx.register(c, kinds=("bern30", "run", "edges"))
        base = [fx.query(TQ_OP_OR, s, k) for s in OR_SETS[2:6] for k in (10, 1000)]
        base += [fx.query(TQ_OP_AND, s, 10) for s in AND_SETS[:3]] + _bools(fx)[::4]
        qs, kinds = [], []
        for i, qt in enumerate(base):
            for k in (None, "bern30", "run", "edges")[i % 2:i % 2 + 3]:
                qs.append(qt)
                kinds.append(k)
        _check(fx, c, qs, kinds)
        if "TQ_TILE_PCAP" in hook or "TQ_TILE_CAND_FLOOR" in hook:
            assert c.stats()["tile_fallbacks"] == 1
    finally:
        c.close()


def test_mixed_batch_equals_contexts_with_combined_alive(fx):
    """Unfiltered queries, three filters and the same query under different filters in one batch, over several tile groups, and
    part of the batch on the per-query kernels (scratch budget): each row equals the unfiltered query's on a context whose segments
    carry alive AND filter, and the oracle's."""
    kinds3 = ("bern1", "run", "deleted")
    qts = [fx.query(TQ_OP_OR, s, k) for s in OR_SETS for k in (10, 1000)] + [fx.query(TQ_OP_AND, s, 10) for s in AND_SETS]
    qs, kinds = [], []
    for i, qt in enumerate(qts):
        for k in (None,) + kinds3:
            if (i + len(qs)) % 3:
                qs.append(qt)
                kinds.append(k)
    refs = {k: fx.register_combined(T.Context(0), k) for k in kinds3}
    oracles = {k: fx.register_combined(O.OracleIndex(), k) for k in kinds3}
    for env in (dict(), dict(TQ_TILE_MAX_DENS_X1000=300), dict(TQ_TILE_SCRATCH_MB=1)):
        c = _ctx_with_env(TQ_TILE=1, **env)
        try:
            fx.register(c, kinds=kinds3)
            g = _check(fx, c, qs, kinds)
            if "TQ_TILE_MAX_DENS_X1000" in env:
                assert c.stats()["tile_groups"] >= 5
            for k in kinds3:
                idx = [i for i, x in enumerate(kinds) if x == k]
                plain = QueryBatch([qs[i][0] for i in idx])
                r, o = refs[k].search_batch(plain), oracles[k].search_batch(plain, mode=0)
                for j, i in enumerate(idx):
                    assert hits(g, i) == hits(r, j) == hits(o, j), (k, i)
        finally:
            c.close()
    for r in refs.values():
        r.close()


def test_single_term_batch_on_k_term(fx):
    """A batch of single-term queries only streams through k_term (default TQ_TILE_TERMS rule), with filters."""
    c = _ctx_with_env(TQ_TILE=1)
    try:
        fx.register(c, kinds=("bern30", "edges", "zeros"))
        qs = [fx.query(TQ_OP_TERM, [t], k) for t in (0, 1, 4, 5) for k in KS]
        kinds = [("bern30", "edges", "zeros", None)[i % 4] for i in range(len(qs))]
        _check(fx, c, qs, kinds)
        assert c.stats()["units_term"] > 0 and c.stats()["units_tile"] == 0
    finally:
        c.close()


def test_phrases_under_filters():
    """Phrases of 2..8 terms and sloppy two-term phrases, filtered: equal to the oracle and a device context on alive AND filter."""
    ix = T.SynthIndex(3, 60_000, [0.3, 0.2, 0.1, 0.25, 0.15, 0.3, 0.2, 0.1], seed=0x5A, record_option=2)
    rng = np.random.default_rng(7)
    base = 9000
    masks = [rng.random(ix.max_doc[s]) < 0.3 for s in range(3)]
    alive = [packed(rng.random(ix.max_doc[s]) > 0.1) for s in range(3)]
    comb = [np.bitwise_and(alive[s], packed(masks[s])) for s in range(3)]
    c, r, oi = T.Context(0), T.Context(0), O.OracleIndex()
    try:
        for tgt, al in ((c, alive), (r, comb), (oi, comb)):
            for s in range(3):
                tgt.segment_register(base + s, 0, ix.max_doc[s], 2, ix.body(s), ix.fieldnorm(s), al[s])
                tgt.register_positions(base + s, 0, ix.positions(s))
        for s in range(3):
            c.filter_register(3, base + s, packed(masks[s]))
        qs = []
        for n in range(2, 9):
            for k in KS:
                qs.append(ix.phrase_query(list(range(n)), k, segment_base=base))
        for slop in (1, 3):
            qs.append(dict(ix.phrase_query([0, 3], 100, segment_base=base), slop=slop))
        qs.append(ix.query(TQ_OP_OR, [0, 1, 2], 50, segment_base=base))
        g = c.search_batch(QueryBatch([dict(q, filter=3) for q in qs]))
        want = r.search_batch(QueryBatch(qs))
        o = oi.search_batch(QueryBatch(qs), mode=0)
        for i in range(len(qs)):
            assert hits(g, i) == hits(want, i) == hits(o, i), i
    finally:
        c.close()
        r.close()


def test_skipping_visits_only_non_empty_tiles():
    """With a contiguous filter over about 2 % of the tiles, k_tile sees at most (non-empty tiles) x queries (query, tile) pairs per
    launch, far fewer than unfiltered, and the rows stay exact."""
    ix = T.SynthIndex(2, 1_000_000, [0.05, 0.02, 0.01, 0.004], seed=0x51)
    base = 9100
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_COUNTERS=1)
    r = T.Context(0)
    try:
        ix.register(c, segment_base=base)
        masks = []
        for s in range(2):
            m = np.zeros(ix.max_doc[s], bool)
            m[300_000:320_000] = True  # 20 of 977 tiles (2 %)
            masks.append(m)
            c.filter_register(5, base + s, packed(m))
            r.segment_register(base + s, 0, ix.max_doc[s], ix.record_option, ix.body(s), ix.fieldnorm(s), packed(m))
        qs = [ix.query(TQ_OP_OR, [0, 1, 2, 3], 10, segment_base=base), ix.query(TQ_OP_OR, [1, 2], 100, segment_base=base),
              ix.query(TQ_OP_AND, [0, 1], 10, segment_base=base)]
        seen0 = c.stats()["tile_counters"][0]
        u = c.search_batch(QueryBatch(qs))
        seen_u = c.stats()["tile_counters"][0] - seen0
        g = c.search_batch(QueryBatch([dict(q, filter=5) for q in qs]))
        seen_f = c.stats()["tile_counters"][0] - seen0 - seen_u
        non_empty = 2 * 21  # tiles 292 .. 312 of each segment
        assert 0 < seen_f <= 2 * non_empty * len(qs)  # (the sample launch and the exact launches: each visits a tile at most once)
        assert seen_f * 10 < seen_u
        want = r.search_batch(QueryBatch(qs))
        for i in range(len(qs)):
            assert hits(g, i) == hits(want, i)
        assert u[3].sum() > 0
    finally:
        c.close()
        r.close()


def test_doc_range_parts_add_up(fx):
    """Doc-range parts of every segment on two contexts, the filters registered before set_doc_range on one and after it on the
    other: counts add up to the whole and the merged rows are the whole's.  A view built before the range is narrowed follows it."""
    kind = "bern30"
    qts = [fx.query(TQ_OP_OR, s, 1000) for s in OR_SETS[:4]] + [fx.query(TQ_OP_AND, s, 1000) for s in AND_SETS[:3]]
    qb = QueryBatch([dict(q, filter=FID[kind]) for q, _ in qts])
    parts = []
    for part in range(2):
        c = T.Context(0)
        for i, s in enumerate(fx.osegs):
            s.register(c)
            if part == 0:
                c.filter_register(FID[kind], s.segment_ord, fx.bits[kind][i])
        for s in fx.osegs:
            c.segment_set_doc_range(s.segment_ord, 0, *doc_range(s.max_doc, part, 2))
        if part == 1:
            for i, s in enumerate(fx.osegs):
                c.filter_register(FID[kind], s.segment_ord, fx.bits[kind][i])
        parts.append((c, c.search_batch(qb), c.count_batch(qb)))
    for i, qt in enumerate(qts):
        assert int(parts[0][2][i] + parts[1][2][i]) == fx.count(kind, qt)
        merged = M.merge_fruits([hits(p[1], i) for p in parts], qt[0]["k"])
        assert merged == fx.rows(kind, qt)
    for c, _, _ in parts:
        c.close()
    # narrowing after a filtered search: the view is rebuilt (segments 0 and 1 have deletes, so their range may move later)
    c = T.Context(0)
    try:
        fx.register(c, kinds=(kind,))
        c.search_batch(qb)
        ranges = {}
        for s in fx.osegs[:2]:
            lo, hi = s.max_doc // 4, s.max_doc // 2
            c.segment_set_doc_range(s.segment_ord, 0, lo, hi)
            ranges[s.segment_ord] = (lo, hi)
        g, cnt = c.search_batch(qb), c.count_batch(qb)
        for i, qt in enumerate(qts):
            assert hits(g, i) == fx.rows(kind, qt, doc_ranges=ranges)
            assert int(cnt[i]) == fx.count(kind, qt, doc_ranges=ranges)
    finally:
        c.close()


@pytest.mark.parametrize("n_ctx", [2, 3])
def test_multi_context_and_split_segments(fx, n_ctx):
    """MultiContext over n contexts of one GPU (whole segments, and split segments whose filter goes to every device) equals one."""
    kind = "run"
    qts = [fx.query(TQ_OP_OR, s, k) for s in OR_SETS[:5] for k in KS] + [fx.query(TQ_OP_AND, s, 10) for s in AND_SETS[:3]]
    qb = QueryBatch([dict(q, filter=FID[kind]) for q, _ in qts])
    for split in (False, True):
        m = T.MultiContext([0] * n_ctx)
        try:
            for i, s in enumerate(fx.osegs):
                if split:
                    m.segment_register_split(s.segment_ord, 0, s.max_doc, s.record_option, s.body, s.fn_ids, s.alive)
                else:
                    m.segment_register(s.segment_ord, 0, s.max_doc, s.record_option, s.body, s.fn_ids, s.alive, device_index=i % n_ctx)
                m.filter_register(FID[kind], s.segment_ord, fx.bits[kind][i])
            g = m.search_batch(qb)
            for i, qt in enumerate(qts):
                assert hits(g, i) == fx.rows(kind, qt), (split, i)
            m.filter_unregister(FID[kind])
            with pytest.raises(T.TqError, match="error -3"):
                m.search_batch(qb)
        finally:
            m.close()


@pytest.mark.parametrize("world", [2, 4])
def test_cross_gpu_merger_and_phased_thresholds(fx, world):
    """Segments spread over `world` contexts of one GPU, each with its filters: CrossGpuMerger (key exchange + k_merge) gives the
    model's rows; a phased run that imports another rank's thresholds too."""
    import torch
    kind = "bern30"
    qts = [fx.query(TQ_OP_OR, s, 100) for s in OR_SETS[:5]] + [fx.query(TQ_OP_AND, s, 100) for s in AND_SETS[:2]]
    ctxs, qbs = [], []
    for r in range(world):
        c = T.Context(0)
        mine = [i for i in range(3) if i % world == r]
        for i in mine:
            fx.osegs[i].register(c)
            c.filter_register(FID[kind], fx.osegs[i].segment_ord, fx.bits[kind][i])
        ctxs.append(c)
        ords = {fx.osegs[i].segment_ord for i in mine}
        qbs.append(QueryBatch([dict(q, filter=FID[kind], term_segs=[ts for ts in q["term_segs"] if ts[1] in ords]) for q, _ in qts]))
    got = [None] * world

    def rank(r, dist):
        b = ctxs[r].prepare(qbs[r])
        try:
            m = CrossGpuMerger(ctxs[r], dist, "cuda:0", qbs[r].nq, qbs[r].kmax)
            m.run(b)
            m(b)
            got[r] = merged_rows(m.fetch_host(b), qbs[r].nq)
        finally:
            b.close()

    try:
        run_ranks(world, rank)
        for i, qt in enumerate(qts):
            for r in range(world):
                assert got[r][i] == fx.rows(kind, qt)
        # phased: rank 0 imports the element-wise max of every rank's thresholds between the phases
        bs = [ctxs[r].prepare(qbs[r]) for r in range(world)]
        keys = [torch.zeros(len(qts), dtype=torch.int64, device="cuda:0") for _ in range(world)]
        bests = []  # (kept until the imports have run)
        for p in range(bs[0].phases()):
            for r in range(world):
                bs[r].run_phase(p)
            if p + 1 < bs[0].phases():
                for r in range(world):
                    bs[r].thresholds_export_dev(keys[r].data_ptr())
                bests.append(torch.stack(keys).amax(0).contiguous())
                torch.cuda.synchronize()
                for r in range(world):
                    bs[r].thresholds_import_dev(bests[-1].data_ptr())
        rows = [bs[r].fetch() for r in range(world)]
        torch.cuda.synchronize()
        for i, qt in enumerate(qts):
            assert M.merge_fruits([hits(rows[r], i) for r in range(world)], qt[0]["k"]) == fx.rows(kind, qt)
        for b in bs:
            b.close()
    finally:
        for c in ctxs:
            c.close()


def test_high_doc_ids():
    """One segment of 2^31 - 2 docs, postings and filter bits only near its top: equal to a context whose alive bitset is the filter."""
    max_doc = 2**31 - 2
    rng = np.random.default_rng(31)
    top = max_doc - 300_000
    lists = []
    for p in (0.2, 0.05, 0.01):
        docs = (top + np.nonzero(rng.random(max_doc - top) < p)[0]).astype(np.uint32)
        lists.append((docs, np.minimum(rng.geometric(0.5, size=len(docs)), 8).astype(np.uint32)))
    seg = OracleSegment(lists, None, segment_ord=fresh_ord(), writer_cls=T.FieldWriter, max_doc=max_doc)
    mask_bits = np.zeros((max_doc + 7) // 8, np.uint8)
    sel = top + np.nonzero(rng.random(max_doc - top) < 0.4)[0]
    np.bitwise_or.at(mask_bits, sel >> 3, (1 << (sel & 7)).astype(np.uint8))
    c, r = _ctx_with_env(TQ_TILE=1), T.Context(0)
    try:
        seg.register(c)
        c.filter_register(1, seg.segment_ord, mask_bits)
        r.segment_register(seg.segment_ord, 0, max_doc, seg.record_option, seg.body, None, mask_bits)
        qs = [make_query(TQ_OP_TERM, [seg], [1], 100), make_query(TQ_OP_OR, [seg], [0, 1, 2], 1000), make_query(TQ_OP_AND, [seg], [0, 1], 10)]
        qb = QueryBatch([dict(q, filter=1, count_hits=True) for q in qs])
        g = c.search_batch(qb)
        want = r.search_batch(QueryBatch(qs))
        for i in range(len(qs)):
            assert hits(g, i) == hits(want, i) and int(g[3][i]) > 0
        assert list(c.count_batch(qb)) == list(r.count_batch(QueryBatch(qs)))
    finally:
        c.close()
        r.close()


def test_lifetime_and_errors(fx):
    """Missing filter: -3 at prepare (search and count); short bitset: -1; unknown ordinal: -3; unregister and re-register refused
    while a batch is prepared, fine after it is destroyed; a reused ordinal never inherits a filter; a failed batch leaves the
    context usable."""
    c = T.Context(0)
    try:
        fx.register(c, kinds=("run",))
        s0 = fx.osegs[0]
        qt = fx.query(TQ_OP_OR, [0, 1, 2], 10)
        ok = QueryBatch([dict(qt[0], filter=FID["run"])])
        missing = QueryBatch([dict(qt[0], filter=99)])
        with pytest.raises(T.TqError, match="error -3"):
            c.search_batch(missing)
        with pytest.raises(T.TqError, match="error -3"):
            c.count_batch(missing)
        with pytest.raises(T.TqError, match="error -1"):
            c.filter_register(7, s0.segment_ord, np.zeros(s0.max_doc // 8 - 1, np.uint8))
        with pytest.raises(T.TqError, match="error -3"):
            c.filter_register(7, 987_654, np.zeros(16, np.uint8))
        with pytest.raises(T.TqError, match="error -3"):
            c.filter_unregister(7)
        assert hits(c.search_batch(ok)) == fx.rows("run", qt)  # usable after the failures
        b = c.prepare(ok)
        with pytest.raises(T.TqError, match="error -1"):
            c.filter_unregister(FID["run"])
        with pytest.raises(T.TqError, match="error -1"):
            c.filter_register(FID["run"], s0.segment_ord, fx.bits["run"][0])
        c.filter_register(FID["ones"], s0.segment_ord, fx.bits["ones"][0])  # another filter is free
        b.run()
        assert hits(b.fetch()) == fx.rows("run", qt)
        b.close()
        c.filter_unregister(FID["run"])
        with pytest.raises(T.TqError, match="error -3"):
            c.search_batch(ok)
        # segment churn: the ordinal's last field goes, and its filters with it
        so = fresh_ord()
        seg = OracleSegment(fx.lists[0], fx.lengths[0], segment_ord=so, writer_cls=T.FieldWriter)
        seg.register(c)
        c.filter_register(42, so, fx.bits["bern1"][0])
        q1 = QueryBatch([dict(make_query(TQ_OP_OR, [seg], [0, 1], 10), filter=42)])
        assert int(c.search_batch(q1)[3][0]) > 0
        c.segment_unregister(so, 0)
        seg.register(c)
        with pytest.raises(T.TqError, match="error -3"):
            c.search_batch(q1)
        c.filter_register(42, so, fx.bits["zeros"][0])  # a new bitset for the reused ordinal
        assert int(c.search_batch(q1)[3][0]) == 0
        assert int(c.count_batch(q1)[0]) == 0
    finally:
        c.close()
