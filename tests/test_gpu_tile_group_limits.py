"""k_tile's general instance (AND and TQ_OP_BOOL groups) at the limits of one tile group: 1024 (query, segment) pairs, 4096
distinct lists and 64 tile-indexed dense lists per segment, and the clause words of a segment staged in shared memory or read
from global memory.  The fixture's segment A (262 144 docs) holds 4096 lists, 96 of them dense, whose densities sum to just
under what tile_fits admits in one group; segment B (30 011 docs, deletes) lacks a quarter of A's lists and has 10 dense ones,
so a group's two segments differ in n_slots, n_big and clause words while the layout is sized by the group's maxima.

Every device test checks the rows against the oracle's exhaustive rows (a seeded sample also against tests/score_model.py),
Count through TQ_QUERY_COUNT_HITS and tq_count_batch against the oracle's Count, and asserts from tq_stats how many groups ran,
on which instance, whether the run was repeated, and the shared memory of the last group (tile_counters[7]) against a
restatement of the planner's sizing (`_layout`)."""
import os
import re

import numpy as np
import pytest

import tantivy_b200 as T
from oracle import tq_oracle as O
from tantivy_b200._abi import TQ_OCCUR_MUST, TQ_OCCUR_SHOULD, TQ_OP_AND, TQ_OP_BOOL, TQ_OP_OR, TQ_OP_TERM, QueryBatch
from tests import score_model as M
from tests.helpers import OracleSegment, bool_query, hits, make_query, tile_smem_bytes

# k_tile's limits (csrc/tq_layout.h; test_layout_constants_match_the_header reads them from there)
MAX_QUERIES, MAX_SLOTS, MAX_BIG, MAX_PAIRS = 1024, 4096, 64, 12288
MAX_SMEM, MAX_WORK_LIST, MAX_STAGED_CLAUSES = 200 * 1024, 4096, 12288
BIG_MIN = 6  # TQ_TILE_BIG_MIN's default: a list with at least this many postings per 1024-doc tile gets a tile index

_A_DOCS, _B_DOCS = 262_144, 30_011
_A_ORD, _B_ORD = 9700, 9701
_N_LISTS = 4096
_HEAVY = [0.5, 0.45, 0.4, 0.38, 0.35, 0.32, 0.3, 0.28]  # lists 0..7: every MUST group holds one, so BOOL queries have hits
_N_DENSE_A = 96  # lists 0..95 are dense in A; 63 and 64 (the 64th and 65th densest) share one doc_freq
_B_DENSE = list(range(10))  # dense in B: the heavy lists and lists 8, 9
_KS = (1, 10, 129, 1000)


def _in_b(t):
    return t < 8 or t % 4 != 3


def _doc_freqs():
    """Each segment's doc_freq per list (0: absent)."""
    rng = np.random.default_rng(0x6C1A)
    a = np.zeros(_N_LISTS, np.int64)
    a[:8] = np.round(np.array(_HEAVY) * _A_DOCS)
    a[8:_N_DENSE_A] = np.round(np.linspace(0.06, 0.03, _N_DENSE_A - 8) * _A_DOCS)
    a[64] = a[63]
    a[_N_DENSE_A:] = rng.integers(20, 61, size=_N_LISTS - _N_DENSE_A)
    b = np.zeros(_N_LISTS, np.int64)
    b[:8] = np.round(np.array(_HEAVY) * _B_DOCS)
    b[8:10] = round(0.03 * _B_DOCS)
    b[10:_N_DENSE_A] = round(0.004 * _B_DOCS)
    b[_N_DENSE_A:] = rng.integers(15, 46, size=_N_LISTS - _N_DENSE_A)
    b[[t for t in range(_N_LISTS) if not _in_b(t)]] = 0
    return a, b


DF = dict(zip((_A_ORD, _B_ORD), _doc_freqs()))
MAX_DOC = {_A_ORD: _A_DOCS, _B_ORD: _B_DOCS}


# ---- the queries --------------------------------------------------------------------------------------------------------
class Q:
    """A query as the fixture builds it: op, terms (list ordinals), occurs and MUST group ids (TQ_OP_BOOL), k."""

    def __init__(self, op, terms, k, occurs=None, groups=None):
        self.op, self.terms, self.k, self.occurs, self.groups = op, list(terms), k, occurs, groups


def _others(start=8):
    """The lists other than the heavy ones, round and round."""
    t = start
    while True:
        yield t
        t = 8 + (t - 7) % (_N_LISTS - 8)


def _must(groups, k, should=()):
    """+(g0..) +(g1..) .. should..: one MUST group per entry of `groups`, then SHOULD clauses."""
    terms = [t for g in groups for t in g] + list(should)
    ids = [i + 1 for i, g in enumerate(groups) for _ in g]
    return Q(TQ_OP_BOOL, terms, k, [TQ_OCCUR_MUST] * len(ids) + [TQ_OCCUR_SHOULD] * len(should), ids + [0] * len(should))


def w12(i, o):
    """+(h a b) +(h' c d): 12 clause words where every clause is present."""
    return _must([[i % 8, next(o), next(o)], [(i + 3) % 8, next(o), next(o)]], _KS[i % 4])


def w13(i, o):
    q = w12(i, o)
    return _must([q.terms[:3], q.terms[3:]], q.k, should=[next(o)])


def w16(i, o):
    """+(h0 a) +(h1 b) +(h2 c) +(h3 d): MUST groups of two, 16 words."""
    return _must([[(i + j) % 8, next(o)] for j in range(4)], _KS[i % 4])


def w20(i, o):
    """Eight single-clause MUST groups, 20 words: seven heavy lists and one other (every fourth query: the eighth heavy one)."""
    heavy = [(i + j) % 8 for j in range(7)]
    return _must([[t] for t in heavy + [(i + 7) % 8 if i % 4 == 0 else next(o)]], _KS[i % 4])


def w68(i, o):
    """32 single-clause MUST groups, 68 words (a wide query): the eight heavy lists and 24 others, so no doc matches.  (A list
    named four times would count four times in tile_fits' estimate of a new group and exceed its pair budget.)"""
    return _must([[(i + j) % 8] for j in range(8)] + [[next(o)] for _ in range(24)], _KS[i % 4])


def and8(i, o):
    return Q(TQ_OP_AND, [(i + j) % 8 for j in range(7)] + [next(o) if i % 2 else (i + 7) % 8], _KS[i % 4])


def _words(q, seg):
    """Clause words of q's (query, segment) pair as the planner writes them (TQuery::n_clauses; bool_structure for TQ_OP_BOOL,
    min_should_match 0), None when q has no plan in the segment."""
    present = [DF[seg][t] > 0 for t in q.terms]
    if q.op in (TQ_OP_TERM, TQ_OP_OR):
        return sum(present) or None
    if q.op == TQ_OP_AND:
        return len(q.terms) if all(present) else None
    groups = {}
    should = nots = 0
    for c, (occ, g) in enumerate(zip(q.occurs, q.groups)):
        if occ == TQ_OCCUR_MUST:
            groups[g] = groups.get(g, 0) + present[c]
        elif present[c]:
            should, nots = should + (occ == TQ_OCCUR_SHOULD), nots + (occ != TQ_OCCUR_SHOULD)
    if any(n == 0 for n in groups.values()) or (not groups and not should):
        return None
    return 4 + sum(1 + n for n in groups.values()) + should + nots


def _layout(queries, big_min=BIG_MIN, repeat=False):
    """One tile group of `queries`, sized as stage_tile_groups and lay_out size it (TQ_TILE_WINDOWS unset: two windows)."""
    per = {}
    max_clauses = 0
    for seg in (_A_ORD, _B_ORD):
        slots, words, n_q = set(), [], 0
        for q in queries:
            w = _words(q, seg)
            if w is None:
                continue
            n_q += 1
            words.append(w)
            max_clauses = max(max_clauses, w)
            slots |= {t for t in q.terms if DF[seg][t] > 0}
        dens = sum(DF[seg][t] / MAX_DOC[seg] for t in slots)
        big = sum(1 for t in slots if DF[seg][t] * 1024 >= big_min * MAX_DOC[seg])
        per[seg] = dict(n_slots=len(slots), n_big=min(big, MAX_BIG), qualifying=big, n_queries=n_q, words=sum(words), dens=dens,
                        clause_bases=np.cumsum([0] + words[:-1]))
    dens = max(p["dens"] for p in per.values())
    p_cap = MAX_PAIRS if repeat else (int(min(MAX_PAIRS, max(1024.0, dens * 1024 * 1.25 + 192.0))) + 63) & ~63
    max_q = (max(p["n_queries"] for p in per.values()) + 1) & ~1
    seg_cap = min(MAX_WORK_LIST, max(256, max(2, max_clauses // 4) * max_q))
    max_words = max(p["words"] for p in per.values())
    cl_cap = (max_words + 3) & ~3 if max_words <= MAX_STAGED_CLAUSES else 0
    args = (p_cap, max(p["n_slots"] for p in per.values()), max(p["n_big"] for p in per.values()), max_q, seg_cap, cl_cap, 2)
    return dict(per=per, p_cap=p_cap, cl_cap=cl_cap, seg_cap=seg_cap, args=args, smem=int(tile_smem_bytes(*args)))


def _fits_one_group(queries):
    """tile_fits' limits for the whole batch as one group: queries per segment (256 while a query has more than 8 terms),
    slots and expected pairs per tile."""
    for seg in (_A_ORD, _B_ORD):
        n = 0
        for q in queries:
            if _words(q, seg) is not None:
                n += 1
                assert n <= (256 if len(q.terms) > 8 else MAX_QUERIES)
        lay = _layout(queries)["per"][seg]
        assert lay["n_slots"] <= MAX_SLOTS and lay["dens"] * 1024 * 1.5 + 256 <= MAX_PAIRS


# the batches of the clause-word tests: 1024 queries each, clause words in A at the staging bound, one past it, the bound
# before this fix (16384: the largest general layout), 20192, and 256 wide queries followed by 768 of 20 words
def _batch(kind):
    o = _others()
    if kind == "staged_at_bound":  # 960 x 12 + 32 x 8 (AND) + 32 x 16 = 12288
        return [w12(i, o) for i in range(960)] + [and8(i, o) for i in range(32)] + [w16(i, o) for i in range(32)]
    if kind == "global_past_bound":  # one 12-word query made 13
        qs = _batch("staged_at_bound")
        return qs[:500] + [w13(500, _others(3000))] + qs[501:]
    if kind == "w16":  # 1024 x 16 = 16384 words over all 4096 lists
        return [w16(i, o) for i in range(1024)]
    if kind == "w20":  # 1000 x 20 + 24 x 8 = 20192
        return [w20(i, o) for i in range(1000)] + [and8(i, o) for i in range(24)]
    if kind == "wide_then_narrow":  # 256 x 68 + 768 x 20 = 32768: the last query's words start at 32748
        return [w68(i, o) for i in range(256)] + [w20(i, o) for i in range(768)]
    raise KeyError(kind)


_KINDS = ["staged_at_bound", "global_past_bound", "w16", "w20", "wide_then_narrow"]
_WORDS_A = {"staged_at_bound": 12288, "global_past_bound": 12289, "w16": 16384, "w20": 20192, "wide_then_narrow": 32768}


def _dense_batch(general):
    """Unions and term queries over the 96 dense lists of A (both sides of the 64th and 65th densest, which tie), the heavy lists
    and sparse ones; with `general` also an AND and TQ_OP_BOOL queries, so that the group runs the general instance."""
    o = _others(96)
    qs = [Q(TQ_OP_OR, [j, j + 1, j + 2, next(o)], _KS[j % 4]) for j in range(0, 96, 3)]
    cut = ([63, 64], [64, 63, 65], [62, 63, 64, 65, 66], [0, 63], [1, 64, 100], list(range(60, 68)))
    qs += [Q(TQ_OP_OR, ts, k) for ts in cut for k in _KS]
    qs += [Q(TQ_OP_TERM, [t], k) for t in (63, 64, 65, 40, 90) for k in (10, 1000)]
    qs += [Q(TQ_OP_OR, [next(o) for _ in range(6)], _KS[i % 4]) for i in range(64)]
    if general:
        qs += [Q(TQ_OP_AND, [0, 1, 63], 10), Q(TQ_OP_AND, [2, 64], 129)]
        qs += [_must([[0, 63], [1, 64]], k) for k in _KS] + [_must([[2, 65, next(o)], [3]], 1000, should=[64, 70])]
    return qs


# ---- CPU: the fixture and the layouts ---------------------------------------------------------------------------------------
def _header_constant(text, name):
    m = re.search(r"constexpr uint32_t[^;]*\b" + name + r"\s*=\s*([0-9u* ]+?)[;,]", text)
    assert m, name
    return eval(m.group(1).replace("u", ""))


def test_layout_constants_match_the_header():
    src = open(os.path.join(os.path.dirname(__file__), "..", "tantivy_b200", "csrc", "tq_layout.h")).read()
    for name, want in [("kTileMaxQueries", MAX_QUERIES), ("kTileMaxSlots", MAX_SLOTS), ("kTileMaxBig", MAX_BIG),
                       ("kTileMaxPairs", MAX_PAIRS), ("kTileMaxSmem", MAX_SMEM), ("kTileMaxWorkList", MAX_WORK_LIST),
                       ("kTileMaxStagedClauses", MAX_STAGED_CLAUSES)]:
        assert _header_constant(src, name) == want, name


def test_the_fixture_reaches_every_edge():
    a, b = DF[_A_ORD], DF[_B_ORD]
    # A: 96 dense lists, a doc_freq tie at the 64th / 65th densest, the rest sparse; every list fits one group, just
    dense_a = np.nonzero(a * 1024 >= BIG_MIN * _A_DOCS)[0]
    assert list(dense_a) == list(range(_N_DENSE_A))
    order = np.argsort(-a, kind="stable")
    assert a[order[MAX_BIG - 1]] == a[order[MAX_BIG]] and a[order[MAX_BIG]] > a[order[MAX_BIG + 1]]
    assert {int(order[MAX_BIG - 1]), int(order[MAX_BIG])} == {63, 64}
    dens_a = a.sum() / _A_DOCS
    assert 7.3 < dens_a and dens_a * 1024 * 1.5 + 256 <= MAX_PAIRS
    # B: a quarter of A's lists missing, 10 dense, deletes (in the device fixture)
    assert (b > 0).sum() < _N_LISTS * 0.8 and (b > 0).sum() > _N_LISTS * 0.7
    assert list(np.nonzero(b * 1024 >= BIG_MIN * _B_DOCS)[0]) == _B_DENSE
    for kind in _KINDS:
        qs = _batch(kind)
        assert len(qs) == MAX_QUERIES
        _fits_one_group(qs)
        lay = _layout(qs)
        pa, pb = lay["per"][_A_ORD], lay["per"][_B_ORD]
        assert pa["words"] == _WORDS_A[kind] and pa["n_queries"] == MAX_QUERIES, kind
        assert (lay["cl_cap"] > 0) == (kind == "staged_at_bound"), kind
        assert pb["words"] < pa["words"] and pb["n_slots"] < pa["n_slots"] and pb["n_big"] < pa["n_big"] == MAX_BIG, kind
        assert lay["smem"] <= MAX_SMEM and _layout(qs, repeat=True)["smem"] <= MAX_SMEM, kind
        assert any(q.op == TQ_OP_AND for q in qs) or kind in ("w16", "wide_then_narrow")
    assert _layout(_batch("w16"))["per"][_A_ORD]["n_slots"] == MAX_SLOTS
    assert _layout(_batch("staged_at_bound"))["cl_cap"] == MAX_STAGED_CLAUSES
    wide = _layout(_batch("wide_then_narrow"))["per"][_A_ORD]
    assert wide["clause_bases"][-1] == 32748 < 2 ** 16  # TileTQ keeps a segment-local clause base in a u16
    for general in (False, True):
        lay = _layout(_dense_batch(general))["per"][_A_ORD]
        assert lay["qualifying"] == _N_DENSE_A and lay["n_big"] == MAX_BIG and lay["qualifying"] - MAX_BIG >= 32
        assert {63, 64, 65} <= {t for q in _dense_batch(general) for t in q.terms}


def test_the_largest_layouts_fit():
    """Every layout the planner can produce: p_cap up to the repeat's kTileMaxPairs, up to kTileMaxQueries (even), slots, dense
    lists and work-list entries, every staged clause-word cap, two or eight windows.  The layout grows with each argument, so the
    other arguments at their maxima bound it."""
    p_caps = np.arange(1024, MAX_PAIRS + 1, 64)[:, None]
    cl_caps = np.arange(0, MAX_STAGED_CLAUSES + 1, 4)[None, :]
    for n_win in (2, 8):
        smem = tile_smem_bytes(p_caps, MAX_SLOTS, MAX_BIG, MAX_QUERIES, MAX_WORK_LIST, cl_caps, n_win)
        assert smem.max() <= MAX_SMEM, smem.max()
        top = [MAX_PAIRS, MAX_SLOTS, MAX_BIG, MAX_QUERIES, MAX_WORK_LIST, MAX_STAGED_CLAUSES, n_win]
        for arg in range(7):  # monotone in every argument
            lo = list(top)
            lo[arg] = 0 if arg != 6 else 2
            assert tile_smem_bytes(*lo) <= tile_smem_bytes(*top)
    q = np.arange(2, MAX_QUERIES + 1, 2)[:, None]
    seg = np.arange(256, MAX_WORK_LIST + 1, 4)[None, :]
    assert tile_smem_bytes(MAX_PAIRS, MAX_SLOTS, MAX_BIG, q, seg, MAX_STAGED_CLAUSES, 8).max() <= MAX_SMEM
    # the first run's pair buffer: tile_fits caps the expected pairs per tile at (12288 - 256) / 1.5
    first = (int(min(MAX_PAIRS, (MAX_PAIRS - 256) / 1.5 * 1.25 + 192)) + 63) & ~63
    assert first == 10240
    # the staging bound of the parent commit, 16384 words: the repeat of the w16 batch needed 211 008 B
    w16 = _layout(_batch("w16"), repeat=True)
    args = list(w16["args"])
    args[5] = 16384
    assert tile_smem_bytes(*args) == 211_008 > MAX_SMEM
    assert w16["smem"] <= MAX_SMEM


# ---- the device fixture -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fx():
    rng = np.random.default_rng(0x71E5)
    segs = []
    for seg in (_A_ORD, _B_ORD):
        n = MAX_DOC[seg]
        lengths = np.clip(np.round(np.exp(rng.normal(np.log(40), 0.7, size=n))), 1, 4096).astype(np.uint32)
        lists = []
        for t in range(_N_LISTS):
            df = int(DF[seg][t])
            docs = np.sort(rng.choice(n, size=df, replace=False)).astype(np.uint32) if df else np.zeros(0, np.uint32)
            lists.append((docs, np.minimum(rng.geometric(0.5, size=df), 40).astype(np.uint32)))
        alive = np.packbits(rng.random(n) > 0.25, bitorder="little") if seg == _B_ORD else None
        o = OracleSegment(lists, lengths, segment_ord=seg, writer_cls=T.FieldWriter, alive=alive)
        segs.append((o, M.Segment(seg, lists, lengths, alive=alive)))
    oi = O.OracleIndex()
    for o, _ in segs:
        o.register(oi)
    return segs, oi


def _query(fx, q):
    osegs = [o for o, _ in fx[0]]
    d = make_query(TQ_OP_OR if q.op == TQ_OP_BOOL else q.op, osegs, q.terms, q.k)
    return bool_query(d, q.occurs, q.groups) if q.op == TQ_OP_BOOL else d


def _ctx_with_env(**env):
    """tq_ctx_create reads its tuning knobs from the environment."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return T.Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _run(fx, queries, **env):
    """The batch with every query counting its hits, on a context with these knobs: (rows, hits, tq_count_batch, stats)."""
    qs = [_query(fx, q) for q in queries]
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, **env)
    try:
        for o, _ in fx[0]:
            o.register(c)
        b = c.prepare(QueryBatch([dict(q, count_hits=True) for q in qs]))
        try:
            b.run()
            rows = b.fetch()
            got = b.fetch_hits()
            st = c.stats()
        finally:
            b.close()
        counts = c.count_batch(QueryBatch(qs))
    finally:
        c.close()
    return rows, got, counts, st


_EXPECTED = {}


def _check(fx, queries, out, n_model=12):
    """Rows == the oracle's, bit for bit; both Counts == the oracle's; a seeded sample of queries also == score_model."""
    rows, got, counts, _ = out
    segs, oi = fx
    qb = QueryBatch([_query(fx, q) for q in queries])
    key = tuple((q.op, tuple(q.terms), q.k, tuple(q.occurs or ()), tuple(q.groups or ())) for q in queries)
    if key not in _EXPECTED:  # (several tests run one batch under different knobs)
        _EXPECTED[key] = oi.search_batch(qb, mode=0, n_threads=32), oi.count_batch(qb)
    want, want_n = _EXPECTED[key]
    for i in range(qb.nq):
        assert hits(rows, i) == hits(want, i), f"query {i}: device {hits(rows, i)[:4]} != oracle {hits(want, i)[:4]}"
    assert (got == want_n).all(), f"count hits differ at {np.nonzero(got != want_n)[0][:8]}"
    assert (counts == want_n).all(), f"tq_count_batch differs at {np.nonzero(counts != want_n)[0][:8]}"
    msegs = [m for _, m in segs]
    for i in np.random.default_rng(len(queries)).choice(len(queries), size=min(n_model, len(queries)), replace=False):
        q = _query(fx, queries[i])
        assert hits(want, i) == M.search(msegs, q, queries[i].terms), f"query {i}: oracle != model"
        assert int(want_n[i]) == M.count(msegs, q, queries[i].terms)
    assert sum(1 for i in range(qb.nq) if hits(want, i)) >= qb.nq // 8  # (the rows compared are not all empty)


def _assert_groups(st, groups, union_only=False, fallbacks=0, smem=None):
    assert st["tile_groups"] == groups, st["tile_groups"]
    assert st["tile_groups_union_only"] == (groups if union_only else 0), st["tile_groups_union_only"]
    assert st["tile_fallbacks"] == fallbacks, st["tile_fallbacks"]
    if smem is not None:
        assert st["tile_counters"][7] == smem, (st["tile_counters"][7], smem)
    assert st["tile_counters"][7] <= MAX_SMEM


# ---- GPU: clause words staged or read from global memory ----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", _KINDS)
def test_clause_words_staged_or_global(fx, kind):
    """1024 queries of one group: clause words at the staging bound (staged), one past it, at 16 384 and 20 192 (global), and
    256 wide queries before 768 narrow ones, whose segment-local clause bases reach 32 748.  AND queries and MUST groups of two
    ride along; B holds fewer words, slots and dense lists than A."""
    qs = _batch(kind)
    out = _run(fx, qs)
    _assert_groups(out[3], 1, smem=_layout(qs)["smem"])
    _check(fx, qs, out)


# ---- GPU: the largest general layout and its repeats -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("env,fallbacks", [(dict(), 0), (dict(TQ_TILE_CAND_FLOOR=4), 1), (dict(TQ_TILE_PCAP=64), 1)],
                         ids=["first_run", "repeat_level1", "repeat_level2"])
def test_largest_general_layout_and_its_repeats(fx, env, fallbacks):
    """1024 queries +(h0 a) +(h1 b) +(h2 c) +(h3 d) over all 4096 lists of A, 64 of them tile-indexed, 16 384 clause words.
    TQ_TILE_CAND_FLOOR=4 overflows candidate regions only: the run is repeated at level 1 in the same group with the largest tile
    buffer (12 288 pairs), whose layout must still fit (with clause words staged at 16 384 it needed 211 008 B and prepare failed
    with TQ_ERR_UNSUPPORTED).  TQ_TILE_PCAP=64 overflows the tile buffer: level 2, one group per query.  Counts come from the
    first run either way."""
    qs = _batch("w16")
    rows, got, counts, st = out = _run(fx, qs, **env)
    first = _layout(qs)
    assert first["per"][_A_ORD]["n_slots"] == MAX_SLOTS and first["args"][2] == MAX_BIG
    if fallbacks == 0:
        _assert_groups(st, 1, smem=first["smem"])
    elif "TQ_TILE_CAND_FLOOR" in env:
        _assert_groups(st, 1, fallbacks=1, smem=_layout(qs, repeat=True)["smem"])  # (the repeat's group is the last laid out)
    else:
        _assert_groups(st, 1, fallbacks=1, smem=_layout(qs[-1:], repeat=True)["smem"])  # (... its last group: the last query)
    _check(fx, qs, out)


# ---- GPU: more than 64 dense lists in one segment ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("big_min", [None, 1], ids=["big_min_default", "big_min_1"])
@pytest.mark.parametrize("general", [False, True], ids=["union_only", "general"])
def test_more_dense_lists_than_tile_indexes(fx, general, big_min):
    """96 lists of A meet the density rule; the 64 densest get a tile index and a presence map, the rest (the 65th densest,
    which ties with the 64th, among them) are sparse slots, staged one thread per slot by k_tile and through the sparse offsets
    by k_count_tiles."""
    qs = _dense_batch(general)
    env = {} if big_min is None else dict(TQ_TILE_BIG_MIN=big_min)
    lay = _layout(qs, big_min=big_min or BIG_MIN)
    pa = lay["per"][_A_ORD]
    assert pa["n_big"] == MAX_BIG and pa["qualifying"] - MAX_BIG >= 32
    out = _run(fx, qs, **env)
    _assert_groups(out[3], 1, union_only=not general, smem=lay["smem"])
    _check(fx, qs, out)


# ---- GPU: the slot limit ------------------------------------------------------------------------------------------------------
def _slot_batch():
    """q0..q7 bring 64 distinct lists of A (8 each); q8..q15 name only those lists, regrouped (they join the group through
    tile_fits' exact pass: counted as new, 64 + 8 lists would not fit); q16 brings one new list and opens a second group; q17
    names lists of the first group only and joins the second.  A conjunction and a BOOL query run the general instance."""
    base = [0, 1] + list(range(200, 262))
    qs = [Q(TQ_OP_OR, base[8 * i:8 * i + 8], _KS[i % 4]) for i in range(8)]
    qs += [Q(TQ_OP_OR, [base[(8 * j + 9 * i) % 64] for j in range(8)], _KS[i % 4]) for i in range(8)]
    qs[9] = _must([[0, base[1]], [1, base[10]]], 1000, should=[base[20], base[30]])
    qs += [Q(TQ_OP_OR, base[:7] + [300], 129), Q(TQ_OP_AND, [0, base[5]], 10)]
    return qs


def _slot_groups(queries, max_slots):
    """The planner's groups when only the slot limit binds (tile_fits, both passes): lists of A per group."""
    groups = [set()]
    for q in queries:
        new = {t for t in q.terms if DF[_A_ORD][t] > 0}
        if len(groups[-1]) + len(new) > max_slots and len(groups[-1] | new) > max_slots:
            groups.append(set())
        groups[-1] |= new
    return groups


def test_slot_batch_reaches_the_slot_limit():
    qs = _slot_batch()
    g = _slot_groups(qs, 64)
    assert len(g) == 2 and len(g[0]) == 64
    assert len(_slot_groups(qs[:16], 64)) == 1
    assert len(_slot_groups(qs, MAX_SLOTS)) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("max_slots,groups", [(64, 2), (1, 2), (None, 1)], ids=["64", "1_clamps_to_64", "default"])
def test_slot_limit(fx, max_slots, groups):
    qs = _slot_batch()
    env = {} if max_slots is None else dict(TQ_TILE_MAX_SLOTS=max_slots)
    assert len(_slot_groups(qs, max(64, max_slots or MAX_SLOTS))) == groups
    out = _run(fx, qs, **env)
    _assert_groups(out[3], groups)
    _check(fx, qs, out, n_model=len(qs))
