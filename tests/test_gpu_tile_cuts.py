"""k_tile at its default cuts: the light / heavy routing of stage B1, the sample plan of phase 0 and the tile cuts of the three
exact launches, end to end.  Rows are compared with tests/score_model.py bit for bit (docs, segment ordinals, f32 scores; a
zero score by value); every threshold a phase leaves must stay at or below the query's final k-th key; and the routing counters
(TQ_TILE_COUNTERS=1, tq_stats.tile_counters) must equal a count taken from the fixture's doc sets.

The counters, as tile_route (tq_tile.cuh) adds them: [0] pairs = every (group query, tile) that B1 routes, one per tile of a
launch's units and per query of the group's segment, pairs without a posting of the query included (a query that a full work
list defers is routed again in the same tile and counts again); [1] skipped = pairs no doc of which can reach the threshold (no
posting at all, no essential posting, a conjunction clause without postings); [2] light = pairs whose essential postings went
to the shared work list (stage B2); [3] heavy = pairs a window warp evaluated (stage B3).  tq_get_stats reads the cumulative
device counters, so their difference across one run_phase (the device idle) is that phase's launch: phase 0 the sample launch,
phases 1-3 the exact launches.  Exact launches route a pair to B3 when it is a union of >= 2 essential clauses with more than
TQ_TILE_LIGHT_MAX (default 384) essential postings in the tile, or when it has more work-list segments (essential clauses with
postings; 1 for a conjunction; the driving clauses with postings for TQ_OP_BOOL) than the work list holds (TQ_TILE_SEG_CAP);
sample launches never take the first rule.  Tiles are 1024 docs, so one clause holds at most 1024 postings of a tile.

- The light / heavy cut: a ladder segment of 256 tiles whose queries (one per rung, their own terms) hold L - 1, L and L + 1
  essential postings in a tile for L = 1, 96, 383, 384, 385, spread over 2-8 clauses or all in one clause (up to 1000
  postings), as unions, single terms, conjunctions and TQ_OP_BOOL shapes, with tiles where one query is heavy and another
  light, and queries heavy in one tile and light in their other.  Every query matches fewer than k = 1024 docs, so no threshold
  leaves 0 and nothing is pruned: a pair's essential postings are all its postings in the tile.  Run at the built-in defaults
  (the prediction is L = 384's exactly), at TQ_TILE_LIGHT_MAX = 1, 96, 383, 384, 385, without the sample launch, and with the
  work list sized at the largest light pair's segment count and one below it.
- Mixed routing under pruning at the defaults: Zipf unions of 5 and 20 terms, k = 1, 10, 100 and 1000, over segments whose
  densest unions hold more and fewer than 384 postings a tile, with count_hits, a filter and doc-range parts: the exact launches
  route pairs both ways in one run.
- The sample plan and the round cuts: segments of 7, 8, 9, 15, 16, 17, 63, 64, 65 and 1000 tiles (some with a partial last tile),
  batched so that each bound of the sample-tile count (tiles / 64, k_max / 2 + 8, tiles / 2) decides somewhere, sample runs of
  1-4 tiles, filters whose tile runs are one tile long, doc ranges that start inside a tile.  The exact launches together must
  route each (group query, tile of the segment's doc range or filter runs) pair exactly once, and no segment under 8 tiles may
  hold a sample unit.
The fixture checks at the end run without a GPU."""
import functools

import numpy as np
import pytest
import torch

import tantivy_b200 as T
from tantivy_b200._abi import (TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT, TQ_OCCUR_SHOULD, TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM, QueryBatch)
from tests import score_model as M
from tests.helpers import OracleSegment, bool_query, hits, make_query

_TILE = 1024
_K = 1024  # TQ_MAX_K
_DEFAULT_LIGHT_MAX = 384
_SAMPLE_DIV = 64  # TQ_TILE_SAMPLE_DIV's default
_RUN_GAP = 4  # a filter view merges tile runs at most this many empty tiles apart
S_, M_, N_ = TQ_OCCUR_SHOULD, TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT
_PAIRS, _SKIPPED, _LIGHT, _HEAVY = range(4)
# the device tests: gpu-marked, and skipped where there is no CUDA device (the fixture checks run everywhere)
_DEVICE = pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")


def _hook_id(h):
    return "-".join(f"{k[8:].lower()}{v}" for k, v in h.items()) or "default"


def _lengths(rng, n):
    return rng.integers(1, 200, size=n).astype(np.uint32)


def _tfs(rng, n):
    return rng.integers(1, 11, size=n).astype(np.uint32)


# ---- the ladder: per-tile posting counts on both sides of every light_max tried ---------------------------------------------------
_LADDER_TILES = 256
_LADDER_ORD = 7300
_CUTS = (1, 96, 383, 384, 385)
_RUNG_COUNTS = sorted({c + d for c in _CUTS for d in (-1, 0, 1)} - {0})  # 1, 2, 95 .. 97, 382 .. 386
_SECOND = (386, 383, 97, 9)  # a union rung's count in its second tile (>= 8: every clause has postings in the segment)


def _split(total, m):
    """total postings over m clauses, as evenly as possible (the first clauses take the remainder)."""
    return [total // m + (1 if i < total % m else 0) for i in range(m)]


class _Q:
    """One ladder query: op, its clause terms (ladder list indices), TQ_OP_BOOL structure, and per tile the postings of each clause."""

    def __init__(self, name, op, n, occurs=None, groups=None, exclusive=True):
        self.name, self.op, self.n = name, op, n
        self.occurs, self.groups = occurs, groups
        self.exclusive = exclusive  # no other query has postings in its tiles
        self.tiles = {}  # tile -> [postings per clause]
        self.terms = None


@functools.lru_cache(maxsize=None)
def _ladder_plan():
    """The ladder's queries with their tiles and per-clause counts (the doc sets are drawn from this in _ladder_lists)."""
    qs = []
    for c in _RUNG_COUNTS:
        for m in (2, 3, 5, 8):
            q = _Q(f"or{m}_{c}", TQ_OP_OR, m)
            q.tiles = {None: _split(c, m), "second": _split(_SECOND[len(qs) % 4], m)}
            qs.append(q)
    for c in (383, 385, 1000):  # single terms: one essential clause, light however many postings
        q = _Q(f"term_{c}", TQ_OP_TERM, 1)
        q.tiles = {None: [c]}
        qs.append(q)
    for c, m in ((385, 2), (1000, 2), (700, 4)):  # every posting of the tile in one clause of a union: heavy above L
        q = _Q(f"one_of{m}_{c}", TQ_OP_OR, m)
        q.tiles = {None: [c] + [0] * (m - 1), "second": [0] + [5] * (m - 1)}
        qs.append(q)
    # conjunctions: the driving clause holds c; a second tile without the first clause (a tile holds at most 1024 pairs in all)
    for m, cs in ((2, (1, 96, 97, 384, 385, 480)), (3, (1, 96, 97, 300))):
        for c in cs:
            q = _Q(f"and{m}_{c}", TQ_OP_AND, m)
            q.tiles = {None: [c] + [c + 7 * (i + 1) for i in range(m - 1)], "second": [0] + [50] * (m - 1)}
            qs.append(q)
    for c in (384, 385, 480):  # TQ_OP_BOOL: +a +b c (drives with a), SHOULD-only over 8 clauses, +(a b) c -d (a group of two)
        q = _Q(f"bool_mm_{c}", None, 3, occurs=[M_, M_, S_], groups=[1, 2, 0])
        q.tiles = {None: [c, c + 5, 10]}
        qs.append(q)
        q = _Q(f"bool_should8_{c}", None, 8, occurs=[S_] * 8, groups=[0] * 8)
        q.tiles = {None: _split(c, 8)}
        qs.append(q)
        q = _Q(f"bool_grp_{c}", None, 4, occurs=[M_, M_, S_, N_], groups=[1, 1, 0, 0])
        q.tiles = {None: _split(c, 2) + [20, 3]}
        qs.append(q)
    for j, (h, l) in enumerate(((385, 383), (386, 384), (1000, 4))):  # one tile, one query heavy and another light
        a, b = _Q(f"shared_heavy_{j}", TQ_OP_OR, 3, exclusive=False), _Q(f"shared_light_{j}", TQ_OP_OR, 4, exclusive=False)
        a.tiles = {("shared", j): _split(h, 3)}
        b.tiles = {("shared", j): _split(l, 4)}
        qs += [a, b]
    # tiles: every query's own, spread over the segment; the shared tiles last
    rng = np.random.default_rng(7301)
    keys = [(i, t) for i, q in enumerate(qs) for t in q.tiles if not (isinstance(t, tuple) and t[0] == "shared")]
    shared = sorted({t for q in qs for t in q.tiles if isinstance(t, tuple) and t[0] == "shared"})
    slots = rng.permutation(_LADDER_TILES)[:len(keys) + len(shared)]
    where = {k: int(s) for k, s in zip(keys, slots)}
    where.update({t: int(s) for t, s in zip(shared, slots[len(keys):])})
    term = 0
    for i, q in enumerate(qs):
        q.tiles = {where.get((i, t), where.get(t)): cnt for t, cnt in q.tiles.items()}
        q.terms = list(range(term, term + q.n))
        term += q.n
    return qs


@functools.lru_cache(maxsize=None)
def _ladder_lists():
    """(lists, lengths): one list per clause of every ladder query, its docs drawn at random inside the query's tiles."""
    rng = np.random.default_rng(7302)
    qs = _ladder_plan()
    lists = []
    for q in qs:
        for c in range(q.n):
            docs = []
            for t, cnt in q.tiles.items():
                if cnt[c]:
                    docs.append(t * _TILE + np.sort(rng.choice(_TILE, cnt[c], replace=False)))
            d = np.sort(np.concatenate(docs)).astype(np.uint32)
            lists.append((d, _tfs(rng, len(d))))
    return lists, _lengths(rng, _LADDER_TILES * _TILE)


def _per_tile(docs, n_tiles):
    return np.bincount(np.asarray(docs, np.int64) // _TILE, minlength=n_tiles)


@functools.lru_cache(maxsize=None)
def _ladder_counts():
    """counts[i][c] = the per-tile postings of clause c of query i, counted from the doc sets."""
    lists, _ = _ladder_lists()
    return [np.stack([_per_tile(lists[t][0], _LADDER_TILES) for t in q.terms]) for q in _ladder_plan()]


def _bool_words(q):
    """(MUST groups as clause lists, SHOULD clauses) of a ladder TQ_OP_BOOL query."""
    groups = {}
    for c in range(q.n):
        if q.occurs[c] == M_:
            groups.setdefault(q.groups[c], []).append(c)
    return list(groups.values()), [c for c in range(q.n) if q.occurs[c] == S_]


def _drive(q, cnt):
    """(the postings that decide the route, work-list segments, is a union) of ladder query q in a tile whose clause postings are
    cnt, nothing pruned (the threshold is 0): every clause of a union is essential."""
    if q.op == TQ_OP_AND:
        return int(cnt.min()), 1, False
    if q.op is None:  # TQ_OP_BOOL: the MUST group with the fewest postings (the first of equals), else the SHOULD clauses
        groups, should = _bool_words(q)
        g = groups[int(np.argmin([int(cnt[g].sum()) for g in groups]))] if groups else should
        return int(cnt[g].sum()), int((cnt[g] > 0).sum()), False
    return int(cnt.sum()), int((cnt > 0).sum()), True


def _route(q, cnt, light_max, seg_cap=1 << 30):
    """How an exact launch routes ladder query q in a tile whose clause postings are cnt: "skipped", "light" or "heavy"."""
    drive, n_segs, union = _drive(q, cnt)
    if drive == 0:
        return "skipped"
    if (union and q.n >= 2 and drive > light_max) or n_segs > seg_cap:
        return "heavy"
    return "light"


def _ladder_predict(idx, light_max, seg_cap=1 << 30):
    """(pairs, skipped, light, heavy) of the exact launches over the ladder queries idx."""
    qs, counts = _ladder_plan(), _ladder_counts()
    out = {"skipped": 0, "light": 0, "heavy": 0}
    for i in idx:
        for t in range(_LADDER_TILES):
            out[_route(qs[i], counts[i][:, t], light_max, seg_cap)] += 1
    return np.array([len(idx) * _LADDER_TILES, out["skipped"], out["light"], out["heavy"]], dtype=np.int64)


def _ladder_exclusive():
    return [i for i, q in enumerate(_ladder_plan()) if q.exclusive]


def _ladder_seg_cap():
    """The most work-list segments of a light pair among the queries with tiles of their own, at the default light_max."""
    qs, counts = _ladder_plan(), _ladder_counts()
    return max(_drive(qs[i], counts[i][:, t])[1] for i in _ladder_exclusive() for t in range(_LADDER_TILES)
               if _route(qs[i], counts[i][:, t], _DEFAULT_LIGHT_MAX) == "light")


# ---- the sample plan and the round cuts ----------------------------------------------------------------------------------------
_SMALL_TILES = (7, 8, 9, 15, 16, 17, 63, 64, 65)
_BIG_TILES = 1000
_PARTIAL = {8: 1000, 9: 333, 17: 700, 65: 1, _BIG_TILES: 100}  # docs missing from the last tile
_CUT_ORD = 7400
_CUT_DENS = (0.3, 0.08, 0.01)


def _cut_max_doc(nt):
    return nt * _TILE - _PARTIAL.get(nt, 0)


def _cut_ord(nt):
    return _CUT_ORD + nt


def _cut_filter(nt):
    """The filter of a segment: random docs of every sixth tile (runs of one tile, five empty tiles apart: never merged)."""
    n = _cut_max_doc(nt)
    rng = np.random.default_rng(7400 + nt)
    keep = (np.arange(n) // _TILE % 6 == 0) & (rng.random(n) < 0.5)
    return keep


def _cut_range(nt):
    """A doc range that starts inside a tile (and ends inside one)."""
    n = _cut_max_doc(nt)
    return (700, n - 300) if nt < 15 else (3 * _TILE + 517, n - 1500)


def _view_tiles(nt, view):
    """The tiles the exact launches must visit, from the doc range or the filter bits alone: [(t0, t1)] runs."""
    n = _cut_max_doc(nt)
    if view == "range":
        lo, hi = _cut_range(nt)
        return [(lo // _TILE, -(-hi // _TILE))]
    if view == "filter":
        has = np.nonzero(_per_tile(np.nonzero(_cut_filter(nt))[0], -(-n // _TILE)))[0]
        runs = []
        for t in has:
            if runs and t - runs[-1][1] <= _RUN_GAP:
                runs[-1][1] = int(t) + 1
            else:
                runs.append([int(t), int(t) + 1])
        return [tuple(r) for r in runs]
    return [(0, -(-n // _TILE))]


def _run_tile(runs, v):
    for t0, t1 in runs:
        if v < t1 - t0:
            return t0 + v, t1
        v -= t1 - t0
    return runs[-1][1] - 1, runs[-1][1]


def _sample_plan(seg_runs, kmax, div=_SAMPLE_DIV):
    """The sample launch's units [(segment index, t0, t1)] of one tile group, its sample-tile count and which bound set it:
    max(tiles / div, k_max / 2 + 8), at most tiles / 2, spread over the segments of >= 8 tiles as runs of 1-4 tiles starting at
    (2r + 1) * nt / (2 * runs) and clipped to the end of their tile run."""
    total = sum(t1 - t0 for runs in seg_runs for t0, t1 in runs)
    by_div, by_k, half = total // div, kmax // 2 + 8, total // 2
    want = min(half, max(by_div, by_k))
    bound = "half" if want == half and half < max(by_div, by_k) else ("div" if by_div > by_k else "kmax")
    units = []
    for si, runs in enumerate(seg_runs):
        nt = sum(t1 - t0 for t0, t1 in runs)
        if nt < 8:
            continue
        seg_sample = max(1, want * nt // total)
        ln = max(1, min(4, seg_sample // 64 + 1))
        n_runs = max(1, seg_sample // ln)
        for r in range(n_runs):
            t0 = min((2 * r + 1) * nt // (2 * n_runs), nt - 1)
            t1 = min(nt, t0 + ln)
            a0, a1 = _run_tile(runs, t0)
            units.append((si, a0, min(a1, a0 + (t1 - t0))))
    return units, want, bound


def _round_split(nt):
    """The tiles of each exact launch in a segment of nt run tiles: one launch below 16 tiles, else cuts at nt / 8 and nt / 2."""
    if nt < 16:
        return (0, 0, nt)
    c1, c2 = nt // 8, nt // 2
    return (c1, c2 - c1, nt - c2)


# (segments by tile count, k) of each batch; every batch is one tile group
_CUT_BATCHES = {
    "small_k1": (_SMALL_TILES, 1),               # sample tiles: k_max / 2 + 8 = 8
    "small_kmax": (_SMALL_TILES, _K),            # tiles / 2 = 132
    "big_k1": (_SMALL_TILES + (_BIG_TILES,), 1),  # tiles / 64 = 19
    "big_kmax": (_SMALL_TILES + (_BIG_TILES,), _K),  # k_max / 2 + 8 = 520: runs of 4 tiles in the big segment
    "big_k200": ((_BIG_TILES,), 200),            # 108: runs of 2 tiles
    "big_k300": ((_BIG_TILES,), 300),            # 158: runs of 3 tiles
    "seg7": ((7,), _K),                          # below 8 tiles: no sample unit
    "seg8": ((8,), 1),                           # 8 tiles: 4 sample tiles
    "seg16": ((16,), _K),
}
_CUT_QUERIES = (("or", [0, 1, 2]), ("or", [1, 2]), ("and", [0, 1]), ("term", [2]), ("bool", [0, 1, 2]))


def _cut_seg_runs(batch, view):
    tiles, k = _CUT_BATCHES[batch]
    return [_view_tiles(nt, view) for nt in tiles], k


# ---- the mixed routing fixture -------------------------------------------------------------------------------------------------
_MIX_TILES = 600
_MIX_ORD = 7500
_MIX_RANKS = 60
_MIX_SCALE = (0.3, 0.1)  # density of rank r in segment s: scale / r


@functools.lru_cache(maxsize=None)
def _mix_lists(s):
    rng = np.random.default_rng(7500 + s)
    n = _MIX_TILES * _TILE - 77 * s
    lists = []
    for r in range(1, _MIX_RANKS + 1):
        d = np.nonzero(rng.random(n) < _MIX_SCALE[s] / r)[0].astype(np.uint32)
        lists.append((d, _tfs(rng, len(d))))
    return lists, _lengths(rng, n)


def _zipf_terms(rng, n, n_terms):
    ranks = np.arange(1, _MIX_RANKS + 1)
    p = (1.0 / ranks) / (1.0 / ranks).sum()
    return [sorted(int(r) - 1 for r in rng.choice(ranks, size=n_terms, replace=False, p=p)) for _ in range(n)]


@functools.lru_cache(maxsize=None)
def _mix_shapes():
    rng = np.random.default_rng(7503)
    return [(t, k) for n_terms in (5, 20) for k in (1, 10, 100, 1000) for t in _zipf_terms(rng, 3, n_terms)]


def _mix_filter(s):
    n = len(_mix_lists(s)[1])
    rng = np.random.default_rng(7510 + s)
    return rng.random(n) < 0.6


def _mix_range(s):
    n = len(_mix_lists(s)[1])
    return (40 * _TILE + 333 + 1000 * s, n - 5 * _TILE - 17)


# ---- GPU side ------------------------------------------------------------------------------------------------------------------
def _key(score):
    u = int(np.float32(score).view(np.uint32))
    if u == 0x80000000:  # -0.0 shares +0.0's key
        u = 0
    return u ^ (0xFFFFFFFF if u >> 31 else 0x80000000)


def _final_keys(want, ks):
    """The score key of each query's final k-th row; 0 when it holds fewer than k rows."""
    return np.array([_key(r[k - 1][0]) if len(r) >= k else 0 for r, k in zip(want, ks)], dtype=np.int64)


def _counters(c):
    return np.array(c.stats()["tile_counters"][:4], dtype=np.int64)


def _run_phases(c, qb, final, count=False):
    """One run, phase by phase; after every phase but the last the thresholds must not fall and must stay at or below the final
    k-th keys.  Returns (rows, per-phase routing counters [4 x 4], hits or None)."""
    keys = torch.zeros(qb.nq, dtype=torch.int64, device="cuda:0")
    b = c.prepare(qb)
    per = []
    try:
        torch.cuda.synchronize()
        prev_c = _counters(c)
        prev = np.zeros(qb.nq, dtype=np.int64)
        n_ph = b.phases()
        assert n_ph == 4
        for ph in range(n_ph):
            b.run_phase(ph)
            if ph + 1 < n_ph:
                b.thresholds_export_dev(keys.data_ptr())
                now = keys.cpu().numpy().copy()
                assert (now >= prev).all(), ("a threshold fell", ph, np.nonzero(now < prev))
                assert (now <= final).all(), ("a threshold passed the final k-th key", ph, np.nonzero(now > final))
                prev = now
            torch.cuda.synchronize()
            cur = _counters(c)
            per.append(cur - prev_c)
            prev_c = cur
        rows = b.fetch()
        got_hits = b.fetch_hits() if count else None
    finally:
        b.close()
    st = c.stats()
    assert st["tile_fallbacks"] == 0, "the run was repeated: the counters would hold the repeat's launches too"
    assert st["tile_groups"] >= 1
    return rows, np.stack(per), got_hits


def _assert_rows(rows, want):
    for i, w in enumerate(want):
        assert hits(rows, i) == w, (i, hits(rows, i)[:4], w[:4])


def _ctx(**env):
    from tests.test_gpu_parity import _ctx_with_env
    return _ctx_with_env(TQ_TILE_COUNTERS=1, **env)


class _Built:
    """Device segments (the product's writer) and model segments of one fixture."""

    def __init__(self, segs):
        self.osegs = [OracleSegment(lists, lengths, segment_ord=so, writer_cls=T.FieldWriter) for so, lists, lengths in segs]
        self.models = {so: M.Segment(so, lists, lengths) for so, lists, lengths in segs}
        self.raw = {so: (lists, lengths) for so, lists, lengths in segs}

    def oseg(self, so):
        return next(s for s in self.osegs if s.segment_ord == so)


@functools.lru_cache(maxsize=None)
def _ladder_built():
    lists, lengths = _ladder_lists()
    return _Built([(_LADDER_ORD, lists, lengths)])


def _ladder_queries(idx):
    b = _ladder_built()
    seg = [b.oseg(_LADDER_ORD)]
    qs, terms = [], []
    for i in idx:
        q = _ladder_plan()[i]
        if q.op is None:
            mq = bool_query(make_query(TQ_OP_OR, seg, q.terms, _K), q.occurs, q.groups)
        else:
            mq = make_query(q.op, seg, q.terms, _K)
        qs.append(mq)
        terms.append(q.terms)
    return qs, terms


def _ladder_run(idx, env):
    b = _ladder_built()
    qs, terms = _ladder_queries(idx)
    want = [M.search([b.models[_LADDER_ORD]], q, t) for q, t in zip(qs, terms)]
    assert all(len(w) < _K for w in want)  # no threshold can leave 0
    qb = QueryBatch(qs)
    c = _ctx(**env)
    try:
        b.oseg(_LADDER_ORD).register(c)
        rows, per, _ = _run_phases(c, qb, np.zeros(len(qs), dtype=np.int64))
        groups = c.stats()["tile_groups"]
    finally:
        c.close()
    _assert_rows(rows, want)
    assert groups == 1
    return per


_LIGHT_HOOKS = [dict()] + [dict(TQ_TILE_LIGHT_MAX=L) for L in _CUTS] + [dict(TQ_TILE_SAMPLE_DIV=0)]


@pytest.mark.gpu
@_DEVICE
@pytest.mark.parametrize("hook", _LIGHT_HOOKS, ids=_hook_id)
def test_light_heavy_cut_on_the_ladder(hook):
    """The exact launches route every (query, tile) of the ladder as the doc sets predict at this light_max; the built-in
    default routes exactly as 384.  The sample launch routes no pair to B3."""
    idx = list(range(len(_ladder_plan())))
    per = _ladder_run(idx, hook)
    light_max = hook.get("TQ_TILE_LIGHT_MAX", _DEFAULT_LIGHT_MAX)
    want = _ladder_predict(idx, light_max)
    exact = per[1:].sum(axis=0)
    print(f"ladder {_hook_id(hook)}: exact pairs/skipped/light/heavy {exact.tolist()}, sample {per[0].tolist()}")
    assert exact.tolist() == want.tolist(), (exact.tolist(), want.tolist())
    if hook.get("TQ_TILE_SAMPLE_DIV") == 0:
        assert per[0].tolist() == [0, 0, 0, 0]
    else:
        assert per[0][_HEAVY] == 0 and per[0][_PAIRS] > 0
        units, _, _ = _sample_plan([[(0, _LADDER_TILES)]], _K)
        assert per[0][_PAIRS] == len(idx) * sum(t1 - t0 for _, t0, t1 in units)


@pytest.mark.gpu
@_DEVICE
@pytest.mark.parametrize("below", [0, 1], ids=["cap", "cap_minus_1"])
def test_seg_cap_cut_on_the_ladder(below):
    """A pair with more work-list segments than the list holds goes to B3, whatever its op: the work list sized at the largest
    light pair's segment count keeps every pair where the default puts it; one entry less sends exactly those pairs to B3.  The
    queries here have their tiles to themselves, so no tile's light pairs together overfill the list (no pair is deferred)."""
    idx = _ladder_exclusive()
    cap = _ladder_seg_cap() - below
    per = _ladder_run(idx, dict(TQ_TILE_SEG_CAP=cap))
    exact = per[1:].sum(axis=0)
    want = _ladder_predict(idx, _DEFAULT_LIGHT_MAX, cap)
    print(f"ladder seg_cap {cap}: exact {exact.tolist()}")
    assert exact.tolist() == want.tolist(), (exact.tolist(), want.tolist())


# ---- mixed routing -------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _mix_built():
    return _Built([(_MIX_ORD + s, *_mix_lists(s)) for s in range(2)])


@pytest.mark.gpu
@_DEVICE
@pytest.mark.parametrize("view", ["count", "filter", "range"])
def test_mixed_routing_under_pruning_at_the_defaults(view):
    """Zipf unions at the built-in knobs: exact rows, thresholds never past the final k-th key, and the exact launches route
    pairs to B2 and to B3 in one run (one CTA evaluates both kinds)."""
    b = _mix_built()
    ords = [_MIX_ORD, _MIX_ORD + 1]
    osegs = [b.oseg(so) for so in ords]
    models, doc_ranges = [b.models[so] for so in ords], None
    if view == "filter":
        models = [M.Segment(so, *b.raw[so], alive=np.packbits(_mix_filter(s), bitorder="little")) for s, so in enumerate(ords)]
    elif view == "range":
        doc_ranges = {so: _mix_range(s) for s, so in enumerate(ords)}
    qs, terms = [], []
    for t, k in _mix_shapes():
        q = make_query(TQ_OP_OR, osegs, t, k)
        if view == "count":
            q["count_hits"] = True
        if view == "filter":
            q["filter"] = 5
        qs.append(q)
        terms.append(t)
    want = [M.search(models, q, t, doc_ranges=doc_ranges) for q, t in zip(qs, terms)]
    final = _final_keys(want, [q["k"] for q in qs])
    qb = QueryBatch(qs)
    c = _ctx()
    try:
        for s, so in enumerate(ords):
            b.oseg(so).register(c)
            if view == "filter":
                c.filter_register(5, so, np.packbits(_mix_filter(s), bitorder="little"))
            elif view == "range":
                c.segment_set_doc_range(so, 0, *_mix_range(s))
        rows, per, got = _run_phases(c, qb, final, count=view == "count")
    finally:
        c.close()
    _assert_rows(rows, want)
    if view == "count":
        assert got.tolist() == [M.count(models, q, t) for q, t in zip(qs, terms)]
    exact = per[1:].sum(axis=0)
    print(f"mixed {view}: exact pairs/skipped/light/heavy {exact.tolist()}, sample {per[0].tolist()}")
    assert exact[_LIGHT] > 0 and exact[_HEAVY] > 0, exact.tolist()
    assert per[0][_HEAVY] == 0


# ---- the sample plan and the round cuts ------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _cut_built():
    segs = []
    for nt in _SMALL_TILES + (_BIG_TILES,):
        rng = np.random.default_rng(7420 + nt)
        n = _cut_max_doc(nt)
        lists = []
        for d in _CUT_DENS:
            docs = np.nonzero(rng.random(n) < d)[0].astype(np.uint32)
            lists.append((docs, _tfs(rng, len(docs))))
        segs.append((_cut_ord(nt), lists, _lengths(rng, n)))
    return _Built(segs)


def _cut_queries(osegs, k, view):
    qs, terms = [], []
    for op, t in _CUT_QUERIES:
        if op == "bool":
            q = bool_query(make_query(TQ_OP_OR, osegs, t, k), [M_, S_, S_])
        else:
            q = make_query({"or": TQ_OP_OR, "and": TQ_OP_AND, "term": TQ_OP_TERM}[op], osegs, t, k)
        if view == "filter":
            q["filter"] = 9
        qs.append(q)
        terms.append(t)
    return qs, terms


@pytest.mark.gpu
@_DEVICE
@pytest.mark.parametrize("view", ["plain", "filter", "range"])
@pytest.mark.parametrize("batch", list(_CUT_BATCHES))
def test_sample_plan_and_round_cuts(batch, view):
    """Every (group query, tile of the segment's doc range or filter runs) pair is routed exactly once by the exact launches, in
    the launch the round cuts give its tile; the sample launch routes the pairs of its planned units (none in a segment under 8
    tiles); rows exact; the thresholds after the sample launch at or below the final k-th keys."""
    tiles, k = _CUT_BATCHES[batch]
    b = _cut_built()
    ords = [_cut_ord(nt) for nt in tiles]
    osegs = [b.oseg(so) for so in ords]
    models, doc_ranges = [b.models[so] for so in ords], None
    if view == "filter":
        models = [M.Segment(so, *b.raw[so], alive=np.packbits(_cut_filter(nt), bitorder="little")) for nt, so in zip(tiles, ords)]
    elif view == "range":
        doc_ranges = {so: _cut_range(nt) for nt, so in zip(tiles, ords)}
    qs, terms = _cut_queries(osegs, k, view)
    want = [M.search(models, q, t, doc_ranges=doc_ranges) for q, t in zip(qs, terms)]
    final = _final_keys(want, [q["k"] for q in qs])
    qb = QueryBatch(qs)
    c = _ctx()
    try:
        for nt, so in zip(tiles, ords):
            b.oseg(so).register(c)
            if view == "filter":
                c.filter_register(9, so, np.packbits(_cut_filter(nt), bitorder="little"))
            elif view == "range":
                c.segment_set_doc_range(so, 0, *_cut_range(nt))
        rows, per, _ = _run_phases(c, qb, final)
        groups = c.stats()["tile_groups"]
    finally:
        c.close()
    _assert_rows(rows, want)
    assert groups == 1
    nq = len(qs)
    seg_runs = [_view_tiles(nt, view) for nt in tiles]
    # exactly once: the tiles of every segment's doc range or filter runs, times the group's queries
    visit = sum(t1 - t0 for runs in seg_runs for t0, t1 in runs)
    assert per[1:, _PAIRS].sum() == nq * visit, (per[1:, _PAIRS].tolist(), nq * visit)
    split = np.array([_round_split(sum(t1 - t0 for t0, t1 in runs)) for runs in seg_runs]).sum(axis=0)
    assert per[1:, _PAIRS].tolist() == (nq * split).tolist()
    assert (per[1:, _PAIRS] == per[1:, _SKIPPED] + per[1:, _LIGHT] + per[1:, _HEAVY]).all()
    units, _, _ = _sample_plan(seg_runs, k)
    assert per[0][_PAIRS] == nq * sum(t1 - t0 for _, t0, t1 in units), (per[0].tolist(), units[:8])
    assert per[0][_HEAVY] == 0
    if all(sum(t1 - t0 for t0, t1 in runs) < 8 for runs in seg_runs):
        assert per[0].tolist() == [0, 0, 0, 0]


# ---- the fixtures themselves (no GPU) --------------------------------------------------------------------------------------------
def test_fixture_ladder_has_the_intended_per_tile_counts():
    qs, counts = _ladder_plan(), _ladder_counts()
    used = set()
    for q, cnt in zip(qs, counts):
        tiles = np.nonzero(cnt.sum(axis=0))[0]
        assert 1 <= len(tiles) <= 2, q.name
        for t, want in q.tiles.items():
            assert cnt[:, t].tolist() == list(want), (q.name, t)
        assert (cnt.sum(axis=1) > 0).all(), q.name  # every clause has postings in the segment
        used.update(int(t) for t in tiles)
    # every posting lies in the query's own tiles, and a tile holds at most 1024 postings over all queries
    total = sum(cnt.sum(axis=0) for cnt in counts)
    assert total.max() <= _TILE and total[[t for t in range(_LADDER_TILES) if t not in used]].sum() == 0
    # unions of 2-8 clauses at L - 1, L and L + 1 essential postings for every cut tried
    union_totals = {int(c.sum(axis=0)[t]) for q, c in zip(qs, counts) if q.op == TQ_OP_OR and q.n >= 2 for t in q.tiles}
    for L in _CUTS:
        assert {L - 1, L, L + 1} - {0} <= union_totals, L
    # k = 1024 is never reached: no threshold leaves 0, nothing is pruned
    b_lists, _ = _ladder_lists()
    for q in qs:
        docs = np.unique(np.concatenate([b_lists[t][0] for t in q.terms]))
        assert len(docs) < _K, q.name


def test_fixture_ladder_predictions_pin_every_cut():
    """Each cut tried routes the ladder differently from its neighbours, so the default (384) is told apart from 383 and 385;
    every branch of the rule decides some pair at the default."""
    idx = list(range(len(_ladder_plan())))
    preds = {L: _ladder_predict(idx, L) for L in _CUTS}
    for a, b in zip(_CUTS, _CUTS[1:]):
        assert preds[a].tolist() != preds[b].tolist(), (a, b)
    d = preds[_DEFAULT_LIGHT_MAX]
    assert d[_LIGHT] > 0 and d[_HEAVY] > 0 and d[_SKIPPED] > 0
    qs, counts = _ladder_plan(), _ladder_counts()
    routed = {}
    for i, q in enumerate(qs):
        for t in q.tiles:
            routed.setdefault(q.name.split("_")[0], set()).add(_route(q, counts[i][:, t], _DEFAULT_LIGHT_MAX, 1 << 30))
    assert routed["term"] == {"light"} and "light" in routed["and2"] and routed["bool"] == {"light"}
    assert "heavy" in routed["one"] and {"light", "heavy"} <= routed["or5"]
    # a query heavy in one tile and light in its other; tiles with a heavy and a light query
    assert any(len({_route(q, counts[i][:, t], 384, 1 << 30) for t in q.tiles}) == 2 for i, q in enumerate(qs))
    shared = {t for q in qs if not q.exclusive for t in q.tiles}
    for t in shared:
        kinds = [_route(q, counts[i][:, t], 384, 1 << 30) for i, q in enumerate(qs) if t in q.tiles]
        assert sorted(kinds) == ["heavy", "light"], t
    # the work-list cut: one entry less than the largest light pair's segments moves pairs, of more than one op, to B3
    ex = _ladder_exclusive()
    cap = _ladder_seg_cap()
    assert cap >= 2
    a, b = _ladder_predict(ex, 384, cap), _ladder_predict(ex, 384, cap - 1)
    assert a.tolist() == _ladder_predict(ex, 384).tolist() and b[_HEAVY] > a[_HEAVY]


def test_fixture_segment_sizes_on_both_sides_of_8_16_64():
    for nt in _SMALL_TILES + (_BIG_TILES,):
        n = _cut_max_doc(nt)
        assert -(-n // _TILE) == nt and (n % _TILE != 0) == (nt in _PARTIAL)
    assert {7, 8, 9} <= set(_SMALL_TILES) and {15, 16, 17} <= set(_SMALL_TILES) and {63, 64, 65} <= set(_SMALL_TILES)
    assert any(n < 8 for n in _SMALL_TILES) and any(n < 16 for n in _SMALL_TILES if n >= 8)
    # the round split covers every tile once, with one launch below 16 tiles
    for nt in range(1, 200):
        s = _round_split(nt)
        assert sum(s) == nt and (s[0] == s[1] == 0) == (nt < 16)
    # every bound of the sample-tile count decides in some batch; sample runs of 1, 2, 3 and 4 tiles
    bounds, lens = set(), set()
    for batch in _CUT_BATCHES:
        for view in ("plain", "filter", "range"):
            seg_runs, k = _cut_seg_runs(batch, view)
            units, want, bound = _sample_plan(seg_runs, k)
            if view == "plain":
                bounds.add(bound)
                lens.update(t1 - t0 for _, t0, t1 in units)
            nts = [sum(t1 - t0 for t0, t1 in r) for r in seg_runs]
            assert all(nts[si] >= 8 for si, _, _ in units)
            if view == "plain" and batch == "seg7":
                assert not units
            if view == "plain" and batch == "seg8":
                assert len(units) == 4
    assert bounds == {"div", "kmax", "half"}, bounds
    assert lens == {1, 2, 3, 4}, lens
    # filters whose runs are shorter than a sample run clip it; ranges start inside a tile
    big_f = _view_tiles(_BIG_TILES, "filter")
    assert all(t1 - t0 == 1 for t0, t1 in big_f)
    seg_runs, k = _cut_seg_runs("big_kmax", "filter")
    _, want, _ = _sample_plan(seg_runs, k)
    nt_big = len(big_f)
    assert want * nt_big // sum(t1 - t0 for r in seg_runs for t0, t1 in r) >= 64  # runs of >= 2 tiles over 1-tile filter runs
    for nt in _SMALL_TILES + (_BIG_TILES,):
        lo, hi = _cut_range(nt)
        assert lo % _TILE and hi % _TILE and 0 < lo < hi < _cut_max_doc(nt)


def test_fixture_mixed_unions_straddle_384():
    """Unprunable, the union of a query's clauses holds more than 384 postings in the tiles of one segment and fewer in another."""
    above = below = 0
    for t, _ in _mix_shapes():
        for s in range(2):
            lists, lengths = _mix_lists(s)
            n_tiles = -(-len(lengths) // _TILE)
            per = sum(_per_tile(lists[i][0], n_tiles) for i in t)
            above += int((per > 384).sum())
            below += int(((per > 0) & (per <= 384)).sum())
    assert above > 0 and below > 0
