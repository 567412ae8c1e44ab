"""k_tile's shared stripes and B2's exits from a union posting, against the oracle's exhaustive rows, bit for bit.

Stage B1 marks the 32-doc stripes of a tile in which more than one essential clause of a union lists a doc (a dense slot, one
with a presence map per tile, gets an exact mask from its presence words); a posting outside them is the only essential
posting of its doc and skips the look-ups.  Inside a shared stripe B2 first drops a posting whose score plus the tile maxima of
the clauses after it cannot reach the threshold (with a 1.00001 margin for the f32 summation order), then one whose doc an
earlier essential clause lists; the non-essential walk drops the rest that cannot reach it.
These tests put two dense essential clauses in no common stripe, in one, and in every stripe, docs at the stripe edges 31 / 32
and the tile edges 1023 / 1024, deletes, a negative boost (no pruning), TQ_TILE_COUNTERS=1 (tq_stats.tile_b2_exits), and docs
whose score ties the threshold where the f32 bound and the score differ in the last bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from oracle import tq_oracle as O  # noqa: E402
from tantivy_b200._abi import TQ_OP_OR, TQ_OP_TERM, QueryBatch  # noqa: E402
from tests import score_model as M  # noqa: E402
from tests.helpers import hits, make_query  # noqa: E402
from tests.test_gpu_parity import _ctx_with_env, assert_same  # noqa: E402
from tests.test_gpu_scoring_edges import _segment  # noqa: E402

_MAX_DOC = 64 * 1024  # 64 tiles


def _per_tile(offsets, rng=None, keep=1.0):
    """Docs at these offsets of every tile (a random share `keep` of them)."""
    docs = (np.arange(_MAX_DOC // 1024)[:, None] * 1024 + np.asarray(sorted(offsets))[None, :]).ravel()
    if rng is not None and keep < 1.0:
        docs = docs[rng.random(len(docs)) < keep]
    return docs.astype(np.uint32)


def _stripes(stripes, within):
    return [32 * s + w for s in stripes for w in within]


_EVEN, _ODD = range(0, 32, 2), range(1, 32, 2)


def _lists(rng):
    """0: even stripes; 1: odd stripes (no stripe in common with 0); 2: odd stripes and one doc of stripe 2 (one stripe in
    common with 0); 3: every stripe (all in common with 0); 4: the stripe and tile edges 0, 31, 32, 1023 (1024 is the next
    tile's 0); 5: rare.  Lists 0-3 hold >= 6 pairs per tile: dense slots with a presence map."""
    offs = [_stripes(_EVEN, (0, 5, 31)), _stripes(_ODD, (0, 13, 31)), _stripes(_ODD, (2, 31)) + [64 + 7],
            _stripes(range(32), (3, 31)), [0, 31, 32, 1023]]
    docs = [_per_tile(o, rng, 0.9) for o in offs] + [np.sort(rng.choice(_MAX_DOC, 300, replace=False)).astype(np.uint32)]
    return [(d, rng.integers(1, 24, size=len(d)).astype(np.uint32)) for d in docs]


_SHAPES = [[0, 1], [0, 2], [0, 3], [1, 3], [0, 1, 4], [0, 3, 4, 5], [1, 2, 3], [3, 0, 4], [0, 1, 2, 3, 4, 5], [4, 0, 3]]


def _queries(seg, boost=1.0):
    qs, terms = [], []
    for c in _SHAPES:
        for k in (1, 10, 100, 1000):
            qs.append(make_query(TQ_OP_OR, [seg], c, k, boost=boost))
            terms.append(c)
    return qs, terms


def _check(segs, queries, terms, **env):
    """device == oracle (exhaustive) == model, on the union-only k_tile instance, nothing repeated."""
    osegs, msegs = [o for o, _ in segs], [m for _, m in segs]
    oi = O.OracleIndex()
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, **env)
    try:
        for s in osegs:
            s.register(oi)
            s.register(c)
        qb = QueryBatch(queries)
        g = c.search_batch(qb)
        st = c.stats()
    finally:
        c.close()
    assert st["tile_groups"] >= 1 and st["tile_groups_union_only"] == st["tile_groups"] and st["tile_fallbacks"] == 0
    assert_same(g, oi.search_batch(qb, mode=0), qb.nq)
    for i, (q, t) in enumerate(zip(queries, terms)):
        assert hits(g, i) == M.search(msegs, q, t), f"query {i}"
    return g, st


@pytest.mark.parametrize("counters", [0, 1])
@pytest.mark.parametrize("deletes", [False, True])
def test_dense_clauses_sharing_no_one_and_every_stripe(counters, deletes):
    rng = np.random.default_rng(4401)
    lengths = np.clip(np.round(np.exp(rng.normal(np.log(30), 0.6, size=_MAX_DOC))), 1, 2000).astype(np.uint32)
    alive = np.packbits(rng.random(_MAX_DOC) > 0.2, bitorder="little") if deletes else None
    seg = _segment(_lists(rng), lengths, alive=alive)
    queries, terms = _queries(seg[0])
    _, st = _check([seg], queries, terms, TQ_TILE_COUNTERS=counters)
    if counters:
        ex = st["tile_b2_exits"]
        assert ex[1] > 0 and ex[3] > 0  # postings that were not the owner of their doc, and completed ones
        assert ex[0] + ex[2] > 0  # and some the bounds dropped


def test_negative_boost_turns_pruning_off():
    """Not prunable (a negative weight): no bound is taken, every essential posting that owns its doc is completed."""
    rng = np.random.default_rng(4402)
    lengths = np.clip(np.round(np.exp(rng.normal(np.log(30), 0.6, size=_MAX_DOC))), 1, 2000).astype(np.uint32)
    seg = _segment(_lists(rng), lengths)
    queries, terms = [], []
    for c in _SHAPES:
        for k in (1, 100):
            q = make_query(TQ_OP_OR, [seg[0]], c, k, boost=[-1.5 if j == 1 else 1.0 for j in range(len(c))])
            queries.append(q)
            terms.append(c)
    _, st = _check([seg], queries, terms, TQ_TILE_COUNTERS=1)
    ex = st["tile_b2_exits"]
    assert ex[0] == 0 and ex[2] == 0 and ex[3] > 0


# ---- a tie at the threshold --------------------------------------------------------------------------------------------
# Every doc listed by b, c and d (not by a) scores fl(fl(s_b + s_c) + s_d) (canonical order: descending weight), and there are
# many more of them than k, so that score becomes the threshold.  c and d are non-essential (their bound is fl(s_d + s_c)),
# b is the last essential clause, and a lists a doc in every stripe of those docs, so b's postings take the bound before the
# look-ups: fl(s_b + fl(s_d + s_c)).  The boosts are chosen so that this bound is one ulp BELOW the tied score: only the
# 1.00001 margin keeps those docs.
_TIE_OFFS = [0, 31, 32, 63, 64, 500, 1023]
_TIE_NEXT = {0: 1, 31: 30, 32: 33, 63: 62, 64: 65, 500: 501, 1023: 1022}  # a's doc in the same stripe


def _term_score(seg, t, boost):
    q = make_query(TQ_OP_TERM, [seg[0]], [t], 1, boost=boost)
    return np.float32(M.search([seg[1]], q, [t])[0][0])


def _tie_fixture():
    y = _per_tile(_TIE_OFFS)
    a = _per_tile([_TIE_NEXT[o] for o in _TIE_OFFS])
    ones = [np.ones(len(d), np.uint32) for d in (a, y)]
    seg = _segment([(a, ones[0]), (y, ones[1]), (y, ones[1]), (y, ones[1])], None, max_doc=_MAX_DOC)
    f = np.float32
    for bc in np.arange(0.60, 0.95, 0.01):
        for bd in np.arange(0.20, 0.55, 0.005):
            sb, sc, sd = _term_score(seg, 1, 1.0), _term_score(seg, 2, float(bc)), _term_score(seg, 3, float(bd))
            tie = f(f(sb + sc) + sd)
            bound = f(sb + f(sd + sc))
            if not (sb > sc > sd and bound < tie):
                continue
            ba = 1.0 + 0.5 * float(bc + bd)  # s_b < s_a < the tied score: a's own docs stay below it
            sa = _term_score(seg, 0, ba)
            if sb < sa < tie:
                return seg, [ba, 1.0, float(bc), float(bd)]
    raise AssertionError("no boosts with a bound one ulp below the tied score")


@pytest.mark.parametrize("counters", [0, 1])
def test_tie_at_the_threshold_keeps_every_tied_doc(counters):
    seg, boosts = _tie_fixture()
    queries = [make_query(TQ_OP_OR, [seg[0]], [0, 1, 2, 3], k, boost=boosts) for k in (4, 10, 50, 200)]
    g, st = _check([seg], queries, [[0, 1, 2, 3]] * len(queries), TQ_TILE_COUNTERS=counters)
    for i, q in enumerate(queries):
        assert len(hits(g, i)) == q["k"]
        assert len({s for s, _, _ in hits(g, i)}) == 1  # all tied
