"""k_tile's running threshold at its edges, end to end.  Rows are compared bit for bit with the oracle's exhaustive mode, or with
tests/score_model.py where the segments are built here, and every threshold a phase leaves must stay at or below the query's
final k-th key and never fall (the phase invariant).

- Imported final thresholds, a direct overshoot detector: a batch runs once, then again with every query's final k-th key
  imported after phase 0 (the sample launch).  No sound refresh can raise a threshold past that, so with TQ_TILE_COUNTERS the
  refreshes (tq_stats.tile_cycles[6]) must be > 0 and the raises ([7]) exactly 0, on every route with a sample launch, over
  unions, ANDs, terms and TQ_OP_BOOL shapes, with a filter and with doc-range parts.  The second run starts from the first's
  histograms unless they are zeroed.
- Dead top docs: segments whose best docs for every query (1024+ decoys holding every term with a high tf and a short field, in
  the first 1/8 of each segment and in every tile) are deleted, filtered out or outside the segment's doc range.
- The refresh list overflowing: 1024 queries in one group at k = 1 and 16; several groups (seven queries a group, or a density
  cap) next to phrase queries and queries on k_term, k_and and the union kernels.
- Every route, other launch cuts, the multi-field fixture, repeated terms; MultiContext of two contexts on one GPU (rows only).
- Keys at the ends of the space: sums that overflow to +inf, every clause boosted by -1.5, a mixed-sign union whose k-th score is
  near 0, with and without the sample launch."""
import contextlib
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from oracle import tq_oracle as O  # noqa: E402
from tantivy_b200._abi import (TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT, TQ_OCCUR_SHOULD, TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM,  # noqa: E402
                               QueryBatch)
from tantivy_b200.lib import bm25_weight  # noqa: E402
from tests import score_model as M  # noqa: E402
from tests.helpers import OracleSegment, bool_query, hits, make_query, random_bool_shapes, shape_query  # noqa: E402
from tests.test_gpu_parity import TILE_PATH_HOOKS, _ctx_with_env, assert_same  # noqa: E402

_DENS = [0.3, 0.15, 0.05, 0.01, 0.002, 0.0001]
_BASE = 9500
_KS = (1, 10, 100, 1024)
S_, M_, N_ = TQ_OCCUR_SHOULD, TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT
SAMPLED_HOOKS = [h for h in TILE_PATH_HOOKS if "TQ_TILE_SAMPLE_DIV" not in h] + [dict()]
# candidate regions that hold every posting of their query (min(postings, max(128 k, floor))): nothing overflows, nothing is repeated
_ALL_CANDIDATES = dict(TQ_TILE_CAND_FLOOR=1 << 22)
CUT_HOOKS = [dict(TQ_TILE_ROUND_DIV1=4), dict(TQ_TILE_ROUND_DIV1=16, TQ_TILE_ROUND_DIV2=4)]


def _hook_id(h):
    return "-".join(f"{k[8:].lower()}{v}" for k, v in h.items()) or "default"


def _key(score):
    u = int(np.float32(score).view(np.uint32))
    if u == 0x80000000:  # -0.0 shares +0.0's key
        u = 0
    return u ^ (0xFFFFFFFF if u >> 31 else 0x80000000)


def _final_keys(rows, ks):
    """The score key of each query's final k-th row; 0 when it holds fewer than k rows (no threshold may be set then)."""
    out = np.zeros(len(ks), dtype=np.int64)
    for i, k in enumerate(ks):
        if rows[3][i] == k:
            out[i] = _key(rows[0][i, k - 1])
    return out


def _final_keys_of_rows(rows_list, ks):
    return np.array([_key(r[k - 1][0]) if len(r) >= k else 0 for r, k in zip(rows_list, ks)], dtype=np.int64)


def _phased(c, qb, final, runs=1, import_final=False, seen=None):
    """Runs the batch phase by phase `runs` times on one prepared batch; after every phase but the last the thresholds must be at
    least the previous phase's and at most the final k-th keys.  import_final: the final keys are imported after phase 0 of the
    last run.  seen: receives the refresh and raise counters as the last run starts.  Returns the rows of each run."""
    import torch
    keys = torch.zeros(qb.nq, dtype=torch.int64, device="cuda:0")
    fin = torch.from_numpy(final).to("cuda:0")
    b = c.prepare(qb)
    out = []
    try:
        for run in range(runs):
            last = run + 1 == runs
            if last and seen is not None:
                torch.cuda.synchronize()
                seen["before"] = _counters(c)
            n_ph = b.phases()
            prev = np.zeros(qb.nq, dtype=np.int64)
            for ph in range(n_ph):
                b.run_phase(ph)
                if ph + 1 < n_ph:
                    if import_final and ph == 0 and last:
                        b.thresholds_import_dev(fin.data_ptr())
                    b.thresholds_export_dev(keys.data_ptr())
                    now = keys.cpu().numpy().copy()
                    assert (now >= prev).all(), ("a threshold fell", run, ph, np.nonzero(now < prev))
                    assert (now <= final).all(), ("a threshold passed the final k-th key", run, ph, np.nonzero(now > final))
                    prev = now
            out.append(b.fetch())
    finally:
        b.close()
    return out


@contextlib.contextmanager
def _env(**env):
    """The tuning knobs that contexts read from the environment when they are created, for the duration of the block."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _counters(c):
    cy = c.stats()["tile_cycles"]
    return int(cy[6]), int(cy[7])


# ---- the synthetic index -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def synth():
    ix = T.SynthIndex(3, 600_000, _DENS, seed=97)
    return ix


def _weights(ix, terms, boosts):
    return [bm25_weight(ix.doc_freq(t), ix.num_docs(), b) for t, b in zip(terms, boosts)]


def _mixed_queries(ix, base, ks=_KS, n_bool=12, seed=98):
    qs = [ix.query(TQ_OP_OR, terms, k, segment_base=base) for k in ks for terms in ([0, 5], [0, 1, 2, 3, 4], [1, 3, 4], [0, 0, 1])]
    qs += [ix.query(TQ_OP_AND, terms, k, segment_base=base) for k in ks for terms in ([0, 1], [0, 2, 3])]
    qs += [ix.query(TQ_OP_TERM, [t], k, segment_base=base) for k in ks for t in (0, 2)]
    # repeated terms in TQ_OP_BOOL: twice as SHOULD, in one MUST group, as SHOULD and MUST_NOT
    for k in (10, 1024):
        qs.append(bool_query(ix.query(TQ_OP_OR, [0, 1, 0], k, segment_base=base), [S_, M_, S_]))
        qs.append(bool_query(ix.query(TQ_OP_OR, [1, 1, 2, 0], k, segment_base=base), [M_, M_, S_, S_], groups=[3, 3, 0, 0]))
        qs.append(bool_query(ix.query(TQ_OP_OR, [2, 0, 2], k, segment_base=base), [S_, S_, N_]))
    rng = np.random.default_rng(seed)
    for sh in random_bool_shapes(rng, n_bool, len(_DENS), n_wide=1):
        q = ix.query(TQ_OP_OR, sh["terms"], sh["k"], segment_base=base)
        q["weights"] = _weights(ix, sh["terms"], sh["boosts"])
        qs.append(shape_query(q, sh))
    return qs


class _Views:
    """The synthetic index as a context sees it (plain, under filter 7, or as doc-range parts) and the oracle's rows for it."""

    def __init__(self, ix):
        self.ix = ix
        rng = np.random.default_rng(99)
        self.filt = [np.packbits(rng.random(ix.max_doc[s]) < 0.55, bitorder="little") for s in range(ix.n_segments)]
        # parts that start and end inside 32-doc words and 1024-doc tiles
        self.ranges = [(8192 * 3 + 17 + s * 1000, ix.max_doc[s] - 4093 - s) for s in range(ix.n_segments)]
        self.qs = _mixed_queries(ix, _BASE)
        self.rows = {}

    def _alive(self, view, s):
        if view == "filter":
            return self.filt[s]
        if view == "range":
            lo, hi = self.ranges[s]
            m = np.zeros(self.ix.max_doc[s], bool)
            m[lo:hi] = True
            return np.packbits(m, bitorder="little")
        return None

    def batch(self, view):
        return QueryBatch([dict(q, filter=7) for q in self.qs] if view == "filter" else self.qs)

    def want(self, view):
        if view not in self.rows:
            oi = O.OracleIndex()
            for s in range(self.ix.n_segments):
                oi.segment_register(_BASE + s, 0, self.ix.max_doc[s], 1, self.ix.body(s), self.ix.fieldnorm(s), self._alive(view, s))
            self.rows[view] = oi.search_batch(QueryBatch(self.qs), mode=0, n_threads=16)
        return self.rows[view]

    def context(self, view, **env):
        c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, **env)
        self.ix.register(c, segment_base=_BASE)
        for s in range(self.ix.n_segments):
            if view == "filter":
                c.filter_register(7, _BASE + s, self.filt[s])
            elif view == "range":
                c.segment_set_doc_range(_BASE + s, 0, *self.ranges[s])
        return c


@pytest.fixture(scope="module")
def views(synth):
    return _Views(synth)


@pytest.mark.parametrize("view", ["plain", "filter", "range"])
@pytest.mark.parametrize("hook", SAMPLED_HOOKS, ids=_hook_id)
def test_imported_final_thresholds_are_never_raised(views, hook, view):
    """Run 1: phase by phase, the phase invariant.  Run 2 (same prepared batch): the final k-th keys imported after the sample
    launch; the refreshes still run, and none may raise."""
    want = views.want(view)
    qb = views.batch(view)
    final = _final_keys(want, [q["k"] for q in views.qs])
    assert (final > 0).sum() > qb.nq // 2
    c = views.context(view, TQ_TILE_COUNTERS=1, **hook)
    try:
        first = _phased(c, qb, final)[0]
        assert_same(first, want, qb.nq)
        r0, x0 = _counters(c)
        second = _phased(c, qb, final, runs=1, import_final=True)[0]
        assert_same(second, want, qb.nq)
        r1, x1 = _counters(c)
        assert r1 - r0 > 0, "no refresh ran"
        assert x1 - x0 == 0, f"{x1 - x0} refreshes raised a threshold past the final k-th key"
        # the same again on one prepared batch run twice: the repeat must start from zeroed histograms
        seen = {}
        third = _phased(c, qb, final, runs=2, import_final=True, seen=seen)[1]
        assert_same(third, want, qb.nq)
        assert _counters(c)[1] == seen["before"][1], "a repeated run raised a threshold past the final k-th key"
    finally:
        c.close()


@pytest.mark.parametrize("hook", [h for h in TILE_PATH_HOOKS if "TQ_TILE_SAMPLE_DIV" in h] + CUT_HOOKS, ids=_hook_id)
def test_phase_invariant_on_other_routes(views, hook):
    """Without a sample launch the first wave of CTAs pushes under threshold 0 and would overflow the default candidate regions,
    so the batch would be repeated on the per-query kernels: there the regions hold every posting (_ALL_CANDIDATES).  No run may
    be repeated, so the rows compared are k_tile's."""
    want = views.want("plain")
    qb = views.batch("plain")
    final = _final_keys(want, [q["k"] for q in views.qs])
    c = views.context("plain", **hook, **(_ALL_CANDIDATES if "TQ_TILE_SAMPLE_DIV" in hook else {}))
    try:
        for rows in _phased(c, qb, final, runs=2):
            assert_same(rows, want, qb.nq)
        assert c.stats()["tile_fallbacks"] == 0
    finally:
        c.close()


# ---- dead top docs -----------------------------------------------------------------------------------------------------------
_N_TERMS = 5
_DEAD_DOCS = 160_000


def _decoy_segments(rng, ords, decoy_of):
    """Segments whose decoys (decoy_of(max_doc) -> bool mask) hold every term with tf 30 in a one-token field: the best doc of
    every query.  The other docs hold each term by its density, tf 1..3, 10..80 tokens."""
    out = []
    for so in ords:
        n = _DEAD_DOCS
        decoy = decoy_of(n)
        lengths = rng.integers(10, 81, size=n).astype(np.uint32)
        lengths[decoy] = 1
        lists = []
        for dens in (0.3, 0.1, 0.05, 0.02, 0.01)[:_N_TERMS]:
            has = (rng.random(n) < dens) | decoy
            docs = np.nonzero(has)[0].astype(np.uint32)
            tfs = rng.integers(1, 4, size=len(docs)).astype(np.uint32)
            tfs[decoy[docs]] = 30
            lists.append((docs, tfs))
        out.append((so, lists, lengths, decoy))
    return out


def _first_eighth_and_every_tile(n):
    d = np.zeros(n, bool)
    d[:n // 8:16] = True  # 1250 docs in the tiles of the first exact launch
    d[700::1024] = True   # and one in every tile, the sample launch's among them
    return d


_RANGE = (20_517, _DEAD_DOCS - 2_900)


def _outside_the_range(n):
    lo, hi = _RANGE
    d = np.zeros(n, bool)
    d[:lo:12] = True
    d[lo - 200:lo] = True  # the tiles the part shares with the docs before it
    d[hi:hi + 200] = True
    d[hi::8] = True
    return d


def _dead_queries(osegs, ks):
    qs = []
    for k in ks:
        for terms in ([0, 1], [0, 1, 2, 3, 4], [2, 3, 4], [1]):
            qs.append((make_query(TQ_OP_OR if len(terms) > 1 else TQ_OP_TERM, osegs, terms, k), terms))
        for terms in ([0, 1], [1, 2, 3]):
            qs.append((make_query(TQ_OP_AND, osegs, terms, k), terms))
        qs.append((bool_query(make_query(TQ_OP_OR, osegs, [1, 0, 2], k), [M_, S_, S_]), [1, 0, 2]))
        qs.append((bool_query(make_query(TQ_OP_OR, osegs, [0, 1, 2, 3], k), [S_] * 4, msm=2), [0, 1, 2, 3]))
    return qs


@pytest.mark.parametrize("how", ["deleted", "filtered", "out_of_range"])
def test_dead_top_docs(how):
    rng = np.random.default_rng(0xDEAD)
    ords = (_BASE + 40, _BASE + 41)
    segs = _decoy_segments(rng, ords, _outside_the_range if how == "out_of_range" else _first_eighth_and_every_tile)
    osegs, models, doc_ranges = [], [], None
    for so, lists, lengths, decoy in segs:
        assert decoy[:_DEAD_DOCS // 8].sum() >= 1024
        dead = np.packbits(~decoy, bitorder="little")
        osegs.append(OracleSegment(lists, lengths, segment_ord=so, writer_cls=T.FieldWriter, alive=dead if how == "deleted" else None))
        models.append(M.Segment(so, lists, lengths, alive=dead if how != "out_of_range" else None))
    if how == "out_of_range":
        doc_ranges = {so: _RANGE for so in ords}
    qts = _dead_queries(osegs, _KS)
    want = [M.search(models, q, t, doc_ranges=doc_ranges) for q, t in qts]
    qb = QueryBatch([dict(q, filter=3) if how == "filtered" else q for q, _ in qts])
    final = _final_keys_of_rows(want, [q["k"] for q, _ in qts])
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, TQ_TILE_COUNTERS=1)
    try:
        for s in osegs:
            s.register(c)
            if how == "filtered":
                c.filter_register(3, s.segment_ord, np.packbits(~segs[osegs.index(s)][3], bitorder="little"))
            elif how == "out_of_range":
                c.segment_set_doc_range(s.segment_ord, 0, *_RANGE)
        for rows in _phased(c, qb, final, runs=2):
            for i, (q, _) in enumerate(qts):
                assert hits(rows, i) == want[i], (i, q["k"], hits(rows, i)[:3], want[i][:3])
        assert _counters(c)[1] > 0
        # without the dead docs' exclusion every query's best rows would be decoys: the fixture does what it claims
        live = [M.Segment(so, lists, lengths) for so, lists, lengths, _ in segs]
        top = M.search(live, qts[1][0], qts[1][1])
        assert all(segs[ords.index(so)][3][d] for _, so, d in top[:10])
    finally:
        c.close()


# ---- large groups and several groups -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small():
    ix = T.SynthIndex(2, 300_000, _DENS, seed=101, record_option=2)  # with positions: phrase queries
    oi = O.OracleIndex()
    ix.register(oi, segment_base=_BASE + 20)
    return ix, oi


@pytest.mark.parametrize("k", [1, 16])
def test_1024_queries_in_one_group(small, k):
    """Every query pushes its first candidates in the same tiles: far more than 16 refreshes trigger in a tile of a CTA."""
    ix, oi = small
    base = _BASE + 20
    rng = np.random.default_rng(102 + k)
    qs = []
    while len(qs) < 1024:
        n = int(rng.integers(1, 5))
        terms = [int(t) for t in rng.choice(5, size=n, replace=False)]
        op = TQ_OP_TERM if n == 1 else (TQ_OP_AND if rng.random() < 0.3 else TQ_OP_OR)
        qs.append(ix.query(op, terms, k, segment_base=base))
    qb = QueryBatch(qs)
    want = oi.search_batch(qb, mode=0, n_threads=16)
    final = _final_keys(want, [k] * qb.nq)
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, TQ_TILE_COUNTERS=1)
    try:
        ix.register(c, segment_base=base)
        for rows in _phased(c, qb, final, runs=2):
            assert_same(rows, want, qb.nq)
        st = c.stats()
        assert st["tile_groups"] == 1 and st["tile_fallbacks"] == 0
        assert st["tile_cycles"][6] > 16 * 64  # refreshes
    finally:
        c.close()


def _group_queries(ix, base, route):
    """max_queries: the mixed queries, several groups of seven.  dens: a cap of 55 pairs per 1000 docs; lists 2 (0.05) and 5
    (0.0001) fill one group, 3 and 4 (0.01, 0.002) another, and every query on list 0 or 1 fits no group."""
    if route == "max_queries":
        return _mixed_queries(ix, base, ks=_KS, n_bool=6, seed=103)
    qs = []
    for k in _KS:
        qs += [ix.query(TQ_OP_OR, t, k, segment_base=base) for t in ([2, 5], [3, 4], [4, 3, 5], [0, 2], [1, 3, 4])]
        qs += [ix.query(TQ_OP_AND, t, k, segment_base=base) for t in ([2, 5], [3, 4], [0, 1], [1, 3])]
        qs += [ix.query(TQ_OP_TERM, [t], k, segment_base=base) for t in (0, 2, 3)]
        qs.append(bool_query(ix.query(TQ_OP_OR, [3, 4, 3], k, segment_base=base), [M_, S_, S_]))
        qs.append(bool_query(ix.query(TQ_OP_OR, [2, 5, 4], k, segment_base=base), [S_, S_, N_]))
    return qs


# TQ_TILE_TERMS=0 puts term queries on k_term and TQ_TILE_OPS=5 (terms, unions) AND queries on k_and, next to the tile groups;
# with the density cap the queries on the dense lists fit no group and take k_term / k_and / the union kernels
_GROUP_ROUTES = {"max_queries": dict(TQ_TILE_MAX_QUERIES=7, TQ_TILE_TERMS=0, TQ_TILE_OPS=5),
                 "dens": dict(TQ_TILE_MAX_DENS_X1000=55, TQ_TILE_TERMS=1)}


@pytest.mark.parametrize("route", list(_GROUP_ROUTES))
def test_several_groups_next_to_the_per_query_kernels(small, route):
    """Several tile groups in one batch with phrase queries (k_phrase) and queries on the per-query kernels, which share the
    batch's thresholds and candidate regions: rows, and the phase invariant for every query."""
    ix, oi = small
    base = _BASE + 20
    qs = _group_queries(ix, base, route)
    qs += [ix.phrase_query([0, 1], k, segment_base=base) for k in (10, 100)]
    qb = QueryBatch(qs)
    want = oi.search_batch(qb, mode=0, n_threads=16)
    final = _final_keys(want, [q["k"] for q in qs])
    c = _ctx_with_env(TQ_TILE=1, **_GROUP_ROUTES[route])
    try:
        ix.register(c, segment_base=base)
        for rows in _phased(c, qb, final, runs=2):
            assert_same(rows, want, qb.nq)
        st = c.stats()
        assert st["tile_groups"] > 1 and st["tile_fallbacks"] == 0
        assert st["units_term"] > 0 and st["units_and"] > 0, {k: st[k] for k in ("units_term", "units_and", "units_or")}
    finally:
        c.close()


# ---- multi-field, MultiContext -----------------------------------------------------------------------------------------------
def test_multi_field_fixture():
    from tests.multi_field import Index, battery
    ix = Index(writer_cls=T.FieldWriter)
    qts = battery(ix, phrase=False)
    want = [M.search(ix.models(), q, t) for q, t in qts]
    qb = QueryBatch([q for q, _ in qts])
    final = _final_keys_of_rows(want, [q["k"] for q, _ in qts])
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1)
    try:
        ix.register(c)
        for rows in _phased(c, qb, final, runs=2):
            for i in range(qb.nq):
                assert hits(rows, i) == want[i], i
    finally:
        c.close()


def test_multi_context_of_two(views):
    """Rows only: MultiContext runs the phases and the threshold exchange between its contexts inside search_batch, where the
    thresholds cannot be read."""
    want = views.want("plain")
    qb = views.batch("plain")
    with _env(TQ_TILE=1, TQ_TILE_TERMS=1):
        m = T.MultiContext([0, 0])
    try:
        views.ix.register(m, segment_base=_BASE)
        assert_same(m.search_batch(qb), want, qb.nq)
    finally:
        m.close()


# ---- keys at the ends of the space ---------------------------------------------------------------------------------------------
def _extreme_queries(ix, base, ks):
    qs = []
    for k in ks:
        for terms in ([0, 1, 2], [0, 1, 2, 3, 4]):
            q = ix.query(TQ_OP_OR, terms, k, segment_base=base)
            qs.append(dict(q, weights=_weights(ix, terms, [2e37] * len(terms))))  # sums overflow to +inf
            qs.append(dict(q, weights=_weights(ix, terms, [1e38] * len(terms))))  # (and some weights too)
            qs.append(dict(q, weights=_weights(ix, terms, [-1.5] * len(terms))))  # every score negative: the base below 0x8000
            qs.append(dict(q, weights=_weights(ix, terms, [1.0 if i % 2 == 0 else -1.0 for i in range(len(terms))])))
        # a rare positive clause next to clauses of weight +-0 and negative ones: the k-th score is 0 or just below it
        for terms, boosts in (([5, 3], [1.0, -0.0]), ([5, 3], [1.0, 0.0]), ([5, 3, 0], [1.0, -1.0, 0.0]), ([5, 4, 3], [1.0, 1e-30, -1e-30])):
            q = ix.query(TQ_OP_OR, terms, k, segment_base=base)
            qs.append(dict(q, weights=_weights(ix, terms, boosts)))
        q = ix.query(TQ_OP_AND, [0, 1], k, segment_base=base)
        qs.append(dict(q, weights=_weights(ix, [0, 1], [1.0, -1.0])))
    return qs


@pytest.mark.parametrize("env", [dict(), dict(TQ_TILE_SAMPLE_DIV=0)], ids=["samples", "no_samples"])
def test_extreme_keys(synth, env):
    """The unprunable queries push every doc at or above a threshold that the sample launch (if any) and the refreshes set: the
    candidate regions hold every posting (_ALL_CANDIDATES), so that no run is repeated on the per-query kernels and the rows
    compared are k_tile's."""
    ix = synth
    oi = O.OracleIndex()
    ix.register(oi, segment_base=_BASE)
    qs = _extreme_queries(ix, _BASE, _KS)
    qb = QueryBatch(qs)
    want = oi.search_batch(qb, mode=0, n_threads=16)
    final = _final_keys(want, [q["k"] for q in qs])
    assert (final == 0xFF800000).any() and ((final > 0) & (final < 0x80000000)).any() and (final == 0x80000000).any()
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_COUNTERS=1, **_ALL_CANDIDATES, **env)
    try:
        ix.register(c, segment_base=_BASE)
        for rows in _phased(c, qb, final, runs=2):
            assert_same(rows, want, qb.nq)
        assert c.stats()["tile_fallbacks"] == 0
        if not env:
            r0, x0 = _counters(c)
            assert_same(_phased(c, qb, final, import_final=True)[0], want, qb.nq)
            assert _counters(c)[1] == x0 and _counters(c)[0] > r0
    finally:
        c.close()
