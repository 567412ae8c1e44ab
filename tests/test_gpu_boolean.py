"""TQ_OP_BOOL on the device: seeded random mixed boolean shapes (tests/helpers.py:random_bool_shapes) against the oracle on every
route of the tile engine, with thresholds, the two-phase key exchange, several contexts and doc-range parts, and batches whose
tile run overflows (the repeat must keep BOOL queries exact: they have no per-query kernel).  On a context limited to the
per-query kernels a BOOL batch is refused and Count still answers."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from oracle import tq_oracle as O  # noqa: E402
from tantivy_b200._abi import (TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT, TQ_OCCUR_SHOULD, TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM,  # noqa: E402
                               TQ_RECORD_BASIC, TQ_RECORD_FREQS, QueryBatch)
from tests import score_model as M  # noqa: E402
from tests.helpers import (BOOL_BRANCHES, GOLDEN, OracleSegment, bool_branches, bool_query, bool_shape_query, hits, make_query,  # noqa: E402
                           random_bool_shapes, shape_query)
from tests.test_gpu_parity import _ctx_with_env, assert_same, both, fresh_ord  # noqa: E402

_REFUSED = "TQ_OP_BOOL needs term_occur and the tile engine"


@pytest.fixture(scope="module", params=["tile", "legacy"])
def ctx(request):
    c = _ctx_with_env(TQ_TILE=1 if request.param == "tile" else 0, TQ_TILE_TERMS=1)
    c.engine = request.param
    yield c
    c.close()


def _refused_but_counted(ctx, qb, oi):
    """The per-query kernels have no TQ_OP_BOOL: the batch is refused (no silent fallback); Count (k_count) answers."""
    with pytest.raises(T.TqError, match=_REFUSED):
        ctx.search_batch(qb)
    assert (ctx.count_batch(qb) == oi.count_batch(qb)).all()


# ---- the 3 x 1M-doc synthetic index -------------------------------------------------------------------------------------
_DENS = [0.3, 0.15, 0.05, 0.01, 0.002, 0.0001]


@pytest.fixture(scope="module")
def synth():
    ix = T.SynthIndex(3, 1_000_000, _DENS, seed=77)
    base = 7000
    oi = O.OracleIndex()
    ix.register(oi, segment_base=base)
    return ix, oi, base, {}


def _synth_bool(ix, base, shape, k=None):
    q = ix.query(TQ_OP_OR, shape["terms"], shape["k"] if k is None else k, segment_base=base)
    q["weights"] = [O.bm25_weight(ix.doc_freq(t), ix.num_docs(), b) for t, b in zip(shape["terms"], shape["boosts"])]
    return shape_query(q, shape)


def _synth_bool_queries(ix, base, n, seed):
    return [_synth_bool(ix, base, sh) for sh in random_bool_shapes(np.random.default_rng(seed), n, len(_DENS))]


def _oracle_rows(synth, key, qb):
    """The oracle's rows of a synth batch, computed once per module."""
    ix, oi, base, cache = synth
    if key not in cache:
        cache[key] = oi.search_batch(qb, mode=0, n_threads=16)
    return cache[key]


def _registered(synth, c):
    ix, oi, base, _ = synth
    ix.register(c, segment_base=base)
    return c


@pytest.fixture(scope="module")
def synth_ctx(ctx, synth):
    return _registered(synth, ctx)


def test_random_shapes_on_the_synthetic_index(synth_ctx, synth):
    ix, oi, base, _ = synth
    qs = _synth_bool_queries(ix, base, 48, 11)
    qb = QueryBatch(qs)
    seen = set()
    for q in qs:
        for s in range(3):
            seen |= bool_branches(q, base + s)
    assert seen >= {"optional_with_must", "optional_without_must", "required_union", "required_disjunction", "exclude_1",
                    "exclude_many", "msm_gt_n", "groups4_intersection"}
    if synth_ctx.engine != "tile":
        _refused_but_counted(synth_ctx, qb, oi)
        return
    g = synth_ctx.search_batch(qb)
    assert_same(g, _oracle_rows(synth, "random48", qb), qb.nq)
    assert sum(1 for i in range(qb.nq) if hits(g, i)) >= 10  # (many shapes over six terms match nothing: msm > n, -a, ...)


# ---- small explicit segments: device == model == oracle ---------------------------------------------------------------
def _small_segments(rng):
    osegs, msegs = [], []
    for i in range(3):
        max_doc = int(rng.integers(300, 40_000))
        lengths = np.clip(np.round(np.exp(rng.normal(np.log(40), 0.7, size=max_doc))), 1, 4096).astype(np.uint32)
        lists = []
        for t in range(8):
            # (a 32-clause query brings up to 32 distinct (list, weight) slots: their densities must fit one tile buffer)
            p = (0.3, 0.1, 0.05, 0.01, 0.002)[t % 5] * float(rng.uniform(0.5, 1.5))
            docs = np.nonzero(rng.random(max_doc) < p)[0].astype(np.uint32)
            lists.append((docs, np.minimum(rng.geometric(0.6, size=len(docs)), 10).astype(np.uint32)))
        alive = np.packbits(rng.random(max_doc) > 0.2, bitorder="little")
        so = fresh_ord()
        osegs.append(OracleSegment(lists, lengths, segment_ord=so, writer_cls=T.FieldWriter, alive=alive))
        msegs.append(M.Segment(so, lists, lengths, alive=alive))
    osegs[0].terms[6] = (0, 0, 0)  # absent from some segments: EmptyScorers there
    osegs[1].terms[3] = (0, 0, 0)
    osegs[2].terms[1] = (0, 0, 0)
    return osegs, msegs


def test_random_shapes_on_small_segments_with_deletes(ctx):
    rng = np.random.default_rng(12)
    osegs, msegs = _small_segments(rng)
    shapes = random_bool_shapes(rng, 160, 8)
    qs = [bool_shape_query(osegs, sh) for sh in shapes]
    seen = set()
    for q in qs:
        for s in osegs:
            seen |= bool_branches(q, s.segment_ord)
    assert BOOL_BRANCHES <= seen, BOOL_BRANCHES - seen
    oi = both(ctx, osegs)
    qb = QueryBatch(qs)
    if ctx.engine != "tile":
        _refused_but_counted(ctx, qb, oi)
        return
    g, c = ctx.search_batch(qb), oi.search_batch(qb, mode=0)
    assert_same(g, c, qb.nq)
    for i, (q, sh) in enumerate(zip(qs, shapes)):
        assert hits(g, i) == M.search(msegs, q, sh["terms"]), f"query {i}"


# ---- every route of k_tile, and overflowing runs, with BOOL queries in the batch ------------------------------------------
_ROUTES = [dict(TQ_TILE_SEG_CAP=8), dict(TQ_TILE_SEG_CAP=3), dict(TQ_TILE_LIGHT_MAX=0), dict(TQ_TILE_LIGHT_MAX=0, TQ_TILE_WINDOWS=8),
           dict(TQ_TILE_LIGHT_MAX=100000), dict(TQ_TILE_SAMPLE_DIV=0), dict(TQ_TILE_BIG_MIN=1), dict(TQ_TILE_BIG_MIN=100000),
           dict(TQ_TILE_UNITS=1), dict(TQ_TILE_ROUND_DIV1=2, TQ_TILE_ROUND_DIV2=2)]
_OVERFLOWS = [dict(TQ_TILE_PCAP=64), dict(TQ_TILE_CAND_FLOOR=4), dict(TQ_TILE_SAMPLE_DIV=0, TQ_TILE_CAND_FLOOR=64)]


def _mixed_batch(ix, base):
    qs = []
    for k in (1, 10, 100, 1000):
        for terms in ([0, 5], [0, 4, 5], [1, 0, 5, 3], [5, 4, 3, 2, 1, 0], [2, 3, 4]):
            qs.append(ix.query(TQ_OP_OR, terms, k, segment_base=base))
    qs += [ix.query(TQ_OP_AND, terms, k, segment_base=base) for k in (10, 200) for terms in ([0, 1], [1, 4], [2, 3, 4])]
    qs += [ix.query(TQ_OP_TERM, [t], 10, segment_base=base) for t in (0, 3, 5)]
    # (boost 0 on every clause of a query ties all the docs it matches: the tie tests cover that; here a run should overflow only
    # where a hook makes it)
    shapes = random_bool_shapes(np.random.default_rng(21), 24, len(_DENS))
    for sh in shapes:
        sh["boosts"] = [b if b != 0.0 else 1.0 for b in sh["boosts"]]
    return qs + [_synth_bool(ix, base, sh) for sh in shapes]


@pytest.mark.parametrize("hook", _ROUTES + _OVERFLOWS, ids=lambda h: ",".join(f"{k}={v}" for k, v in h.items()))
def test_bool_queries_on_every_tile_route(synth, hook):
    """The hooks of test_tile_paths_agree and of test_tile_overflow_is_repeated_on_the_per_query_kernels with BOOL queries in the
    batch.  Where the run overflows, the repeat returns the oracle's rows for every query (BOOL queries on the tile engine again)
    and the device-resident / packed results (the sharded hand-over) take the same route."""
    ix, oi, base, _ = synth
    c = _registered(synth, _ctx_with_env(TQ_TILE=1, TQ_TILE_COUNTERS=1, **hook))
    try:
        qb = QueryBatch(_mixed_batch(ix, base))
        want = _oracle_rows(synth, "mixed", qb)
        g = c.search_batch(qb)
        assert_same(g, want, qb.nq)
        st = c.stats()
        assert st["tile_groups"] >= 1
        # without a sample launch the first exact launch hands over every match of its tiles: k = 1000 overflows its region
        overflow = hook in _OVERFLOWS or "TQ_TILE_SAMPLE_DIV" in hook
        assert st["tile_fallbacks"] == (1 if overflow else 0)
        if hook == dict(TQ_TILE_SEG_CAP=3):
            assert st["tile_counters"][3] > 0  # heavy pairs: BOOL pairs take the window path (B3)
        if overflow:
            import torch
            bt = c.prepare(qb)
            try:
                bt.run()
                words = 3 * qb.nq * qb.kmax + qb.nq
                packed = torch.zeros(words + 4, dtype=torch.int32, device="cuda:0")
                bt.results_pack_dev_async(packed.data_ptr())
                torch.cuda.synchronize()
                assert int(packed[words:].abs().max()) != 0  # the flags tell a sharded caller to take the waiting path
                bt.results_pack_dev(packed.data_ptr())
                torch.cuda.synchronize()
                p = packed.cpu().numpy()
                r = qb.nq * qb.kmax
                rows = (p[:r].view(np.float32).reshape(qb.nq, qb.kmax), p[r:2 * r].view(np.uint32).reshape(qb.nq, qb.kmax),
                        p[2 * r:3 * r].view(np.uint32).reshape(qb.nq, qb.kmax), p[3 * r:words].view(np.uint32))
                assert_same(rows, want, qb.nq)
                assert_same(bt.fetch(), want, qb.nq)
            finally:
                bt.close()
    finally:
        c.close()


# ---- ties: more tied docs than a candidate region holds, at default settings ----------------------------------------------
def _tie_segments(kind):
    """Two segments of 100k docs in which every doc of term 0 scores the same: term 0 on every other doc, term 1 (the excluded
    one) on every 7th, term 2 = term 0 (for OR / AND)."""
    max_doc = 100_000  # (x 2 segments: about 86k tied docs for +a -b, 100k for +a +c)
    a = np.arange(0, max_doc, 2, dtype=np.uint32)
    b = np.arange(0, max_doc, 7, dtype=np.uint32)
    segs = []
    for _ in range(2):
        if kind == "basic":  # IndexRecordOption::Basic: tf = 1 everywhere, one fieldnorm for all docs
            lists = [(a, None), (b, None), (a, None)]
            segs.append(OracleSegment(lists, np.full(max_doc, 12), record_option=TQ_RECORD_BASIC, segment_ord=fresh_ord(), writer_cls=T.FieldWriter))
        elif kind == "no_fieldnorms":  # constant fieldnorm 1; equal tfs
            lists = [(a, np.full(len(a), 3, np.uint32)), (b, np.ones(len(b), np.uint32)), (a, np.full(len(a), 3, np.uint32))]
            segs.append(OracleSegment(lists, None, segment_ord=fresh_ord(), writer_cls=T.FieldWriter, max_doc=max_doc))
        else:  # tf = 1 and every length of one fieldnorm bucket
            lo, hi = GOLDEN["field_norms_table"][60:62]
            lengths = lo + np.arange(max_doc) % (hi - lo)
            lists = [(a, np.ones(len(a), np.uint32)), (b, np.ones(len(b), np.uint32)), (a, np.ones(len(a), np.uint32))]
            segs.append(OracleSegment(lists, lengths, segment_ord=fresh_ord(), writer_cls=T.FieldWriter))
    return segs, a, b


@pytest.mark.parametrize("kind", ["basic", "no_fieldnorms", "shared_fieldnorm_id"])
def test_tie_heavy_queries_overflow_and_stay_exact(ctx, kind):
    """+a -b, a -b, +a +c and 'both of a c' with ~43k tied docs per segment: every tied doc is a candidate, more than a region
    of max(128 k, 32768) holds.  The rows are the lowest (segment, doc) pairs; OR / AND of the same lists pin the repeat on the
    per-query kernels."""
    segs, a, b = _tie_segments(kind)
    oi = both(ctx, segs)
    if kind == "shared_fieldnorm_id":
        assert len(set(segs[0].fieldnorms.tolist())) > 1 and len(set(segs[0].fn_ids.tolist())) == 1
    bools = []
    for k in (10, 200):
        bools.append(bool_query(make_query(TQ_OP_OR, segs, [0, 1], k), [TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT]))
        bools.append(bool_query(make_query(TQ_OP_OR, segs, [0, 1], k), [TQ_OCCUR_SHOULD, TQ_OCCUR_MUST_NOT]))
        bools.append(bool_query(make_query(TQ_OP_OR, segs, [0, 2], k), [TQ_OCCUR_MUST, TQ_OCCUR_MUST]))
        bools.append(bool_query(make_query(TQ_OP_OR, segs, [0, 2], k), [TQ_OCCUR_SHOULD, TQ_OCCUR_SHOULD], msm=2))
    plain = [make_query(op, segs, [0, 2], k) for op in (TQ_OP_OR, TQ_OP_AND) for k in (10, 200)]
    qb_plain = QueryBatch(plain)
    g = ctx.search_batch(qb_plain)
    assert_same(g, oi.search_batch(qb_plain, mode=0), qb_plain.nq)
    for i, q in enumerate(plain):
        assert [(s, d) for _, s, d in hits(g, i)] == [(segs[0].segment_ord, int(d)) for d in a[:q["k"]]]
    if ctx.engine == "tile":
        assert ctx.stats()["tile_fallbacks"] == 1
    qb = QueryBatch(bools + plain)
    if ctx.engine != "tile":
        _refused_but_counted(ctx, qb, oi)
        return
    g = ctx.search_batch(qb)
    assert ctx.stats()["tile_fallbacks"] == 1
    assert_same(g, oi.search_batch(qb, mode=0), qb.nq)
    not_b = a[a % 7 != 0]
    for i, q in enumerate(bools):
        docs = not_b if q["term_occur"][1] == TQ_OCCUR_MUST_NOT else a
        assert [(s, d) for _, s, d in hits(g, i)] == [(segs[0].segment_ord, int(d)) for d in docs[:q["k"]]], f"query {i}"
        assert len({s for s, _, _ in hits(g, i)}) == 1  # all tied
    for s in segs:
        ctx.segment_unregister(s.segment_ord, 0)


def test_lone_bool_query_beyond_the_largest_tile_buffer(ctx):
    """A BOOL query whose clauses hold more postings in one 1024-doc tile than the largest tile buffer (12288 pairs) cannot be
    repeated on the tile engine either: TQ_ERR_TILE_CAPACITY, and the context stays usable.  Twelve such lists still fit."""
    max_doc = 200_000
    rng = np.random.default_rng(3)
    lists = []
    for t in range(13):  # every doc of the first tile, and a sparse rest
        rest = np.nonzero(rng.random(max_doc - 1024) < 0.002)[0].astype(np.uint32) + 1024
        docs = np.concatenate([np.arange(1024, dtype=np.uint32), rest])
        lists.append((docs, rng.integers(1, 5, size=len(docs)).astype(np.uint32)))
    lengths = rng.integers(5, 60, size=max_doc)
    seg = OracleSegment(lists, lengths, segment_ord=fresh_ord(), writer_cls=T.FieldWriter)
    oi = both(ctx, [seg])
    wide = bool_query(make_query(TQ_OP_OR, [seg], list(range(13)), 10), [TQ_OCCUR_SHOULD] * 13)
    fits = bool_query(make_query(TQ_OP_OR, [seg], list(range(12)), 10), [TQ_OCCUR_SHOULD] * 11 + [TQ_OCCUR_MUST_NOT])
    if ctx.engine != "tile":
        _refused_but_counted(ctx, QueryBatch([wide, fits]), oi)
        return
    with pytest.raises(T.TqError, match=r"error -7: .*exceed the tile buffer"):
        ctx.search_batch(QueryBatch([wide]))
    qb = QueryBatch([fits, make_query(TQ_OP_OR, [seg], list(range(13)), 10)])  # the OR repeats on the per-query kernels
    g = ctx.search_batch(qb)
    assert ctx.stats()["tile_fallbacks"] == 1
    assert_same(g, oi.search_batch(qb, mode=0), qb.nq)
    ctx.segment_unregister(seg.segment_ord, 0)


# ---- thresholds, the key exchange, several contexts, doc-range parts ---------------------------------------------------
def test_bool_with_initial_thresholds(synth_ctx, synth):
    ix, oi, base, _ = synth
    base_qs = _synth_bool_queries(ix, base, 16, 31)
    for q in base_qs:
        q["k"] = 20
    qb0 = QueryBatch(base_qs)
    if synth_ctx.engine != "tile":
        _refused_but_counted(synth_ctx, qb0, oi)
        return
    g0 = synth_ctx.search_batch(qb0)
    assert_same(g0, oi.search_batch(qb0, mode=0, n_threads=16), qb0.nq)
    queries = []
    for i, q in enumerate(base_qs):
        h = hits(g0, i)
        for thr in ([h[-1][0], h[len(h) // 2][0]] if h else []) + [0.0, -1.0, 1e9]:
            q2 = dict(q)
            q2["threshold"] = float(thr)
            q2["k"] = 50
            queries.append(q2)
    qb = QueryBatch(queries)
    g = synth_ctx.search_batch(qb)
    assert_same(g, oi.search_batch(qb, mode=0, n_threads=16), qb.nq)
    for i, q in enumerate(queries):
        assert all(s > np.float32(q["threshold"]) for s, _, _ in hits(g, i))


def test_bool_two_phase_topkeys_exchange_and_two_contexts(synth_ctx, synth):
    import torch
    ix, oi, base, _ = synth
    qs = _synth_bool_queries(ix, base, 16, 41) + [ix.query(TQ_OP_OR, [0, 4, 5], 100, segment_base=base)]
    qb = QueryBatch(qs)
    if synth_ctx.engine != "tile":
        _refused_but_counted(synth_ctx, qb, oi)
        return
    plain = synth_ctx.search_batch(qb)
    assert_same(plain, oi.search_batch(qb, mode=0, n_threads=16), qb.nq)
    kmax = qb.kmax
    for shards in (1, 2):
        keys = torch.zeros((shards, qb.nq, kmax), dtype=torch.int32, device="cuda:0")
        b = synth_ctx.prepare(qb)
        for phase in range(b.phases()):
            b.run_phase(phase)
            if phase + 1 < b.phases():
                b.topkeys_export_dev(keys[0].data_ptr(), kmax)
                b.thresholds_from_keys_dev(keys.data_ptr(), shards, kmax)
        out = b.fetch()
        b.close()
        for x, y in zip(plain, out):
            assert (x == y).all()
    m = T.MultiContext([0, 0])
    try:
        for s in range(ix.n_segments):
            m.segment_register(base + s, 0, ix.max_doc[s], ix.record_option, ix.body(s), ix.fieldnorm(s), None)
        assert_same(m.search_batch(qb), plain, qb.nq)
    finally:
        m.close()


@pytest.mark.parametrize("cuts", [[0, 101_376, 202_752, 300_000], [0, 1, 77_777, 77_780, 262_144, 299_999, 300_000], [0, 0, 300_000]])
def test_bool_doc_range_parts_merge_to_the_whole_segment(ctx, cuts):
    """tq_segment_set_doc_range with BOOL queries: the parts' merged rows and summed Counts are the whole segment's."""
    from tantivy_b200.sharding import merge_rows_host
    ix = T.SynthIndex(1, 300_000, [0.3, 0.05, 0.01, 0.002, 0.0004], seed=31)
    alive = np.packbits(np.random.default_rng(5).random(300_000) > 0.3, bitorder="little")
    base = fresh_ord()
    oi = O.OracleIndex()
    oi.segment_register(base, 0, ix.max_doc[0], ix.record_option, ix.body(0), ix.fieldnorm(0), alive)
    shapes = random_bool_shapes(np.random.default_rng(51), 20, 5, n_wide=1)
    qs = []
    for sh in shapes:
        q = ix.query(TQ_OP_OR, sh["terms"], sh["k"], segment_base=base)
        q["weights"] = [O.bm25_weight(ix.doc_freq(t), ix.num_docs(), bo) for t, bo in zip(sh["terms"], sh["boosts"])]
        qs.append(shape_query(q, sh))
    qb = QueryBatch(qs)
    want_counts = oi.count_batch(qb)
    tile = ctx.engine == "tile"
    want = oi.search_batch(qb, mode=0, n_threads=8) if tile else None
    rows, counts = [], np.zeros(qb.nq, dtype=np.uint64)
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        c = _ctx_with_env(TQ_TILE=1 if tile else 0, TQ_TILE_TERMS=1)
        try:
            c.segment_register(base, 0, ix.max_doc[0], ix.record_option, ix.body(0), ix.fieldnorm(0), alive)
            c.segment_set_doc_range(base, 0, lo, hi)
            counts += c.count_batch(qb)
            if tile:
                r = c.search_batch(qb)
                for q in range(qb.nq):
                    assert all(lo <= d < hi for _, _, d in hits(r, q))
                rows.append([np.array(x) for x in r])
            else:
                with pytest.raises(T.TqError, match=_REFUSED):
                    c.search_batch(qb)
        finally:
            c.close()
    assert (counts == want_counts).all(), (counts, want_counts)
    if not tile:
        return
    kmax = max(q["k"] for q in qs)
    m = merge_rows_host(np.stack([r[0] for r in rows]), np.stack([r[1] for r in rows]), np.stack([r[2] for r in rows]), np.stack([r[3] for r in rows]), kmax)
    for q in range(qb.nq):
        n = int(want[3][q])
        assert int(m[3][q]) >= n
        assert (m[1][q, :n] == want[1][q, :n]).all() and (m[2][q, :n] == want[2][q, :n]).all()
        assert (m[0][q, :n].view(np.uint32) == want[0][q, :n].view(np.uint32)).all()

