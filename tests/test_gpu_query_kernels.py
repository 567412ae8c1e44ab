"""The per-query kernels -- k_term, k_and, k_or_strip and k_or -- against the numpy model of tests/score_model.py and the oracle,
bit for bit (doc ids, segment ordinals, f32 scores), with the tile engine off and under forced unit cuts: the default cut; one
unit per 128-doc block, 8192-doc tile and 1024-doc window; cuts of 3 / 5 / 3 / 7 (not powers of two, and strips of 7 windows
split 1/2/2/2 over the four warps); one unit per (query, segment) pair, the unit size of a full batch, where the CTA top-k
compactions of tq_device.cuh run.

Segment A (299 993 docs) takes k_or_strip's three threshold rounds, and its last window, tile and unit are partial.  The best
docs of a rare list sit on both sides of the windows where rounds and units start, of every third tile and of every block edge
of that list, so a boundary that is skipped or evaluated twice changes the rows.  Segment B has deletes and no rounds; segment C
has no fieldnorms and tens of thousands of tied keys.  Every batch holds one kernel class: its unit counts are checked against
cut_units' rule, and the strip batch's window routes are seen to run.  A mixed batch that overflows the tile engine is repeated
on these kernels, at the default unit size and at one unit per pair."""
from collections import Counter

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import tq_oracle as O  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM, TQ_TERM_IGNORE_FREQ, QueryBatch  # noqa: E402
from tests import score_model as M  # noqa: E402
from tests.helpers import hits, make_query  # noqa: E402
from tests.test_gpu_parity import _ctx_with_env  # noqa: E402
from tests.test_gpu_scoring_edges import _every_id_lengths, _segment, _tfs  # noqa: E402

BLOCK, WIN, TILE = 128, 1024, 8192  # a posting block, a k_or_strip window, a k_or tile
N_A, N_B, N_C = 299_993, 70_001, 40_000
T0, T1, CL, M0, M1 = 0, 1, 2, 3, 4  # thick 0.45 / 0.15, clustered, thin 0.05 / 0.03 (may turn non-essential)
R = list(range(5, 12))              # r0..r6: thin and rare (<= 0.01)
C0, C1, C2 = 0, 1, 2                # segment C: 0.9 (tf 1), 0.5 (tf 1 or 2), 0.05 (tf 1)
KMAX = 1024

HOOKS = {
    "default": {},
    "smallest": dict(TQ_TERM_BLOCKS_PER_UNIT=1, TQ_AND_BLOCKS_PER_UNIT=1, TQ_OR_TILES_PER_UNIT=1, TQ_STRIP_WINDOWS_PER_UNIT=1,
                     TQ_TARGET_UNITS=1 << 24),
    "odd": dict(TQ_TERM_BLOCKS_PER_UNIT=3, TQ_AND_BLOCKS_PER_UNIT=5, TQ_OR_TILES_PER_UNIT=3, TQ_STRIP_WINDOWS_PER_UNIT=7,
                TQ_TARGET_UNITS=1 << 24),
    "one_unit": dict(TQ_TARGET_UNITS=1),
}
MIN_PER = {"term": ("TQ_TERM_BLOCKS_PER_UNIT", 512), "and": ("TQ_AND_BLOCKS_PER_UNIT", 128), "or": ("TQ_OR_TILES_PER_UNIT", 16),
           "strip": ("TQ_STRIP_WINDOWS_PER_UNIT", 256)}


def _ceil(a, b):
    return -(-a // b)


def _strip_cuts(total):
    """cut_units: a sampled strip pair's threshold rounds cover windows [0, cut1), [cut1, cut2), [cut2, cut3)."""
    cut1 = max(4, total // 32)
    cut2 = max(cut1, total // 8)
    return cut1, cut2, max(cut2, total // 2)


def _planted_a():
    """doc -> tf of r0's planted best docs in segment A (doc length 1): the first and last doc of the windows where the strip
    rounds start (the largest tfs), both sides of every window edge where a unit of 1, 7, 256 or all windows starts inside a
    round or the main launch, both sides of every third tile edge (k_or units of 3 tiles) and the segment's last doc."""
    total = _ceil(N_A, WIN)
    cuts = _strip_cuts(total)
    out = {}
    for w in cuts:
        for d in (w * WIN - 1, w * WIN, w * WIN + WIN - 1):
            out[d] = 5000 + len(out)
    bounds = [0, *cuts, total]
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        for w in range(lo, hi, 7):
            for d in (w * WIN - 1, w * WIN):
                if d >= 0:
                    out.setdefault(d, 1000 + len(out))
    for t in range(3, _ceil(N_A, TILE), 3):
        for d in (t * TILE - 1, t * TILE):
            out.setdefault(d, 500 + len(out))
    out.setdefault(N_A - 1, 2000)
    return out


def _lengths(rng, n):
    lengths = np.clip(np.round(np.exp(rng.normal(np.log(40), 0.7, size=n))), 1, 4096).astype(np.uint32)
    every = _every_id_lengths()
    lengths[rng.choice(n, size=2 * len(every), replace=False)] = np.tile(every, 2)  # every fieldnorm id occurs
    return lengths


def _list(rng, n, p, always=(), ranges=None, tf_edges=True):
    """Docs with probability p (only inside `ranges` if given) plus `always`; tf <= 16 except one block and the VInt tail of
    tf edges >= 16 (tf_edges)."""
    keep = rng.random(n) < p
    if ranges is not None:
        inside = np.zeros(n, bool)
        for lo, hi in ranges:
            inside[lo:hi] = True
        keep &= inside
    keep[np.asarray(sorted(always), np.int64)] = True
    docs = np.nonzero(keep)[0].astype(np.uint32)
    nb = len(docs) // BLOCK
    return docs, _tfs(rng, len(docs), [int(rng.integers(0, nb)), -1] if tf_edges and nb else [])


def _lists(rng, n, plants=None):
    """t0, t1, cl, m0, m1, r0..r6 over n docs; the window and tile edges, doc 0 and doc n - 1 in the thick and thin lists."""
    edge = [0, n - 1, WIN - 1, WIN, TILE - 1, TILE]
    best = list(plants) if plants else []
    clusters = [(n * 2 // 30, n * 5 // 30), (n * 14 // 30, n * 17 // 30), (n * 25 // 30, n * 28 // 30)]
    lists = [_list(rng, n, 0.45, edge + best), _list(rng, n, 0.15, edge + best),
             _list(rng, n, 0.6, [0, n - 1], ranges=clusters),  # thick by doc_freq, absent between three doc ranges
             _list(rng, n, 0.05, edge + best), _list(rng, n, 0.03, edge)]
    r0 = _list(rng, n, 0.009, best, tf_edges=False)
    lists.append(r0)
    lists += [_list(rng, n, p, edge if p == 0.008 else ()) for p in (0.008, 0.006, 0.005, 0.004, 0.003, 0.002)]
    return lists


def _fixture_segments():
    rng = np.random.default_rng(4321)
    # A: r0's best docs planted, and both sides of each of r0's block edges (units of k_term and k_and start at blocks)
    plants = _planted_a()
    lengths = _lengths(rng, N_A)
    lists_a = _lists(rng, N_A, plants)
    docs, tfs = lists_a[R[0]]
    at = np.searchsorted(docs, np.array(sorted(plants), np.uint32))
    tfs[at] = [plants[d] for d in sorted(plants)]
    for b in range(1, _ceil(len(docs), BLOCK)):
        for i in (b * BLOCK - 1, b * BLOCK):
            tfs[i] = max(int(tfs[i]), 100 + b)
    for i in (0, len(docs) - 1):
        tfs[i] = max(int(tfs[i]), 99)
    lengths[docs[tfs >= 99]] = 1
    a = _segment(lists_a, lengths)
    # B: no strip threshold rounds (69 windows), a fifth of the docs deleted
    alive = np.packbits(rng.random(N_B) > 0.2, bitorder="little")
    b = _segment(_lists(rng, N_B), _lengths(rng, N_B), alive=alive)
    # C: no fieldnorms, tf = 1 (and 1 or 2): tied keys by the ten thousand
    lists_c = []
    for p, tf2 in ((0.9, False), (0.5, True), (0.05, False)):
        d = np.nonzero(rng.random(N_C) < p)[0].astype(np.uint32)
        lists_c.append((d, (1 + (rng.random(len(d)) < 0.5) * tf2).astype(np.uint32)))
    c = _segment(lists_c, None, max_doc=N_C)
    return a, b, c


def _bits(rows):
    return [(int(np.float32(s).view(np.uint32)), g, d) for s, g, d in rows]


class Fixture:
    """Segments A, B and C for the device, the model and the oracle; the model's rows of every query shape."""

    def __init__(self):
        self.a, self.b, self.c = _fixture_segments()
        self.ab = [self.a[0], self.b[0]]
        self.cc = [self.c[0]]
        self.msegs = [self.a[1], self.b[1], self.c[1]]
        self.oracle = O.OracleIndex()
        for o, _ in (self.a, self.b, self.c):
            o.register(self.oracle)
        self._rows = {}

    def register(self, ctx):
        for o, _ in (self.a, self.b, self.c):
            o.register(ctx)
        return ctx

    def rows(self, q, terms):
        """The model's rows of q: its top KMAX rows without a threshold (once per query shape), then cut by q's threshold and k."""
        key = repr((q["op"], list(terms), q["weights"], q["avg_fieldnorm"], q["term_segs"], q.get("term_flags")))
        if key not in self._rows:
            self._rows[key] = M.search(self.msegs, dict(q, k=KMAX, threshold=None), terms)
        rows = self._rows[key]
        thr = q.get("threshold")
        if thr is not None:
            rows = [r for r in rows if np.float32(r[0]) > np.float32(thr)]
        return rows[:q["k"]]


class Battery:
    """Queries of one kernel class and their expected rows (the model's, checked against the oracle once)."""

    def __init__(self, fx, queries):
        self.queries = [q for q, _ in queries]
        self.terms = [t for _, t in queries]
        self.qb = QueryBatch(self.queries)
        self.want = [fx.rows(q, t) for q, t in queries]
        ref = fx.oracle.search_batch(self.qb, mode=0, n_threads=8)
        for i, w in enumerate(self.want):
            assert _bits(hits(ref, i)) == _bits(w), ("oracle", i, hits(ref, i)[:4], w[:4])

    def check(self, result, what):
        for i, w in enumerate(self.want):
            got = hits(result, i)
            assert _bits(got) == _bits(w), (what, i, self.queries[i]["op"], self.terms[i], self.queries[i]["k"], got[:4], w[:4])


def _q(op, segs, terms, k, boost=1.0, **extra):
    q = make_query(op, segs, terms, k, boost=boost)
    q.update(extra)
    return q, list(terms)


def _term_queries(fx):
    qs = [_q(TQ_OP_TERM, fx.ab, [t], k) for t in range(12) for k in (1, 10, 128, 129, 1000, 1024)]
    qs += [_q(TQ_OP_TERM, fx.cc, [t], k) for t in (C0, C1, C2) for k in (1, 10, 128, 129, 1000, 1024)]
    for segs, t in ((fx.ab, T0), (fx.ab, R[0]), (fx.cc, C1)):  # initial thresholds just below, at and just above the k-th score
        for k in (10, 128):
            base = _q(TQ_OP_TERM, segs, [t], k)
            s = np.float32(fx.rows(*base)[k - 1][0])
            for thr in (np.nextafter(s, np.float32(-np.inf)), s, np.nextafter(s, np.float32(np.inf))):
                qs.append((dict(base[0], threshold=float(thr)), [t]))
    qs += [_q(TQ_OP_TERM, fx.ab, [T1], 128, boost=0.0), _q(TQ_OP_TERM, fx.cc, [C0], 1024, boost=0.0)]
    return qs


AND_SETS = [[R[0], T0], [T0, T1], [R[0], T1, T0], [T1, M0, T0], [T0, T1, M0, CL], [CL, T0], [T1, CL], [T0, T1, M0, M1, R[0]]]


def _and_queries(fx):
    qs = []
    for c in AND_SETS:
        qs += [_q(TQ_OP_AND, fx.ab, c, k) for k in (1, 10, 1000)]
        # one clause without freqs: from four clauses on, Intersection::score's order instead of one after another
        qs += [_q(TQ_OP_AND, fx.ab, c, k, term_flags=[0] * (len(c) - 1) + [TQ_TERM_IGNORE_FREQ]) for k in (10, 1000)]
        qs.append(_q(TQ_OP_AND, fx.ab, c, 10, boost=[1.0] * (len(c) - 1) + [-1.5]))  # not prunable
    qs += [_q(TQ_OP_AND, fx.cc, [C0, C1], k) for k in (10, 1000)]
    return qs


# thick + thick, thick + thin, thin only (with and without a clause that may turn non-essential, six thin), 7 and 8 clauses,
# clustered + dense
UNION_SETS = [[T0, T1], [T0, R[0]], [T1, M0], [R[0], R[1]], [M0, R[0], R[2]], R[:6], [T0, T1, M0, M1, R[0], R[1], R[2]],
              [T0, T1, CL, M0, M1, R[0], R[1], R[2]], [CL, T0], [CL, R[0]]]
BOOSTS = (0.0, -1.5, 1e4)  # on the rare clause of t0 t1 r0: the last one reorders the canonical sum


def _strip_queries(fx):
    qs = [_q(TQ_OP_OR, fx.ab, c, k) for c in UNION_SETS for k in (1, 10, 128)]
    qs += [_q(TQ_OP_OR, fx.ab, [T0, T1, R[0]], k, boost=[1.0, 1.0, b]) for b in BOOSTS for k in (1, 10, 128)]
    qs += [_q(TQ_OP_OR, fx.cc, [C0, C1], k) for k in (10, 128)]
    return qs


def _window_queries(fx):
    qs = [_q(TQ_OP_OR, fx.ab, c, k) for c in UNION_SETS for k in (129, 1000)]
    qs += [_q(TQ_OP_OR, fx.ab, [T0, T1, CL, M0, M1] + R[:4], k) for k in (10, 1000)]
    qs += [_q(TQ_OP_OR, fx.ab, list(range(12)), k) for k in (128, 1000)]
    qs += [_q(TQ_OP_OR, fx.ab, [T0, R[0], T0, R[0], T1, M0, M1, R[1], R[2], CL], k) for k in (10, 1000)]  # repeated terms
    qs += [_q(TQ_OP_OR, fx.ab, R, k) for k in (1, 10, 128)]  # seven thin clauses: too many for the strip kernel's cache
    qs += [_q(TQ_OP_OR, fx.ab, [T0, T1, R[0]], 1000, boost=[1.0, 1.0, b]) for b in BOOSTS]
    qs.append(_q(TQ_OP_OR, fx.cc, [C0, C1, C2], 1000))
    return qs


@pytest.fixture(scope="module")
def fx():
    f = Fixture()
    f.batteries = {"term": Battery(f, _term_queries(f)), "and": Battery(f, _and_queries(f)), "strip": Battery(f, _strip_queries(f)),
                   "or": Battery(f, _window_queries(f))}
    return f


def _pairs(fx, queries):
    """(unit class, work total, sampled, k) of every (query, segment) pair of a batch, by append_qsegs' rules."""
    out = []
    for q in queries:
        n = len(q["weights"])
        for seg in fx.ab + fx.cc:
            dfs = [ts[3] for ts in sorted(q["term_segs"]) if ts[1] == seg.segment_ord]
            if not dfs or (q["op"] == TQ_OP_AND and len(dfs) < n):
                continue
            if q["op"] == TQ_OP_TERM:
                out.append(("term", _ceil(dfs[0], BLOCK), False, q["k"]))
            elif q["op"] == TQ_OP_AND:
                out.append(("and", _ceil(min(dfs), BLOCK), False, q["k"]))
            elif q["k"] <= 128 and len(dfs) <= 8 and sum(df * (WIN // BLOCK) < seg.max_doc for df in dfs) <= 6:
                prunable = all(np.isfinite(w) and w >= 0 for w in q["weights"])
                out.append(("strip", _ceil(seg.max_doc, WIN), prunable and any(df * 64 >= seg.max_doc for df in dfs), q["k"]))
            else:
                out.append(("or", _ceil(seg.max_doc, TILE), False, q["k"]))
    return out


def _expected_units(fx, queries, env):
    """cut_units' unit counts per class, and the bytes of the candidate regions (16-byte candidates)."""
    target = env["TQ_TARGET_UNITS"]
    pairs = _pairs(fx, queries)
    n_same = Counter(p[0] for p in pairs)
    units, cand_bytes = Counter(), 0
    for cls, total, sampled, k in pairs:
        name, default = MIN_PER[cls]
        per = max(env.get(name, default), _ceil(total, max(1, _ceil(target, n_same[cls]))))
        bounds = [0, total]
        if cls == "strip" and sampled and total >= 8 * 32:
            bounds = [0, *_strip_cuts(total), total]
        n = sum(_ceil(hi - lo, per) for lo, hi in zip(bounds[:-1], bounds[1:]))
        units[cls] += n
        cand_bytes += n * (4 if cls == "strip" else 2) * k * 16
    return units, cand_bytes


def _check_routes(fx, name, st, w0, env):
    own = {"term": "units_term", "and": "units_and", "strip": "units_or", "or": "units_or"}[name]
    for key in ("units_term", "units_and", "units_or", "units_tile", "units_phrase"):
        assert (st[key] > 0) == (key == own), (name, key, st[key])
    dw = [a - b for a, b in zip(st["or_windows"], w0)]
    if name == "strip":
        assert st["units_or_strip"] == st["units_or"]
        assert dw[1] > 0 and dw[2] > 0 and dw[3] > 0, dw  # exhaustive, hot and cold windows
    else:
        assert st["units_or_strip"] == 0 and dw == [0] * 8, dw
    if "TQ_TARGET_UNITS" in env:
        units, cand_bytes = _expected_units(fx, fx.batteries[name].queries, env)
        assert (st["units_term"], st["units_and"], st["units_or"], st["units_or_strip"]) == \
            (units["term"], units["and"], units["or"] + units["strip"], units["strip"]), (name, dict(units))
        assert cand_bytes < 1 << 30, cand_bytes


@pytest.mark.parametrize("hook", list(HOOKS))
def test_per_query_kernels_under_unit_cuts(fx, hook):
    env = dict(TQ_TILE=0, **HOOKS[hook])
    c = fx.register(_ctx_with_env(**env))
    try:
        for name, b in fx.batteries.items():
            w0 = c.stats()["or_windows"]
            b.check(c.search_batch(b.qb), (hook, name))
            _check_routes(fx, name, c.stats(), w0, env)
    finally:
        c.close()


def test_unit_rule_reaches_the_edges(fx):
    """The battery reaches what it is about: strip pairs with threshold rounds and without, the planted docs in the rows, and
    under one unit per pair three extra units per sampled strip pair."""
    pairs = _pairs(fx, fx.batteries["strip"].queries)
    rounds = [s and t >= 8 * 32 for _, t, s, _ in pairs]
    assert any(rounds) and not all(rounds)
    assert any(s and t < 8 * 32 for _, t, s, _ in pairs)  # segment B: sampled, but too short for the rounds
    units, _ = _expected_units(fx, fx.batteries["strip"].queries, HOOKS["one_unit"])
    assert units["strip"] == len(pairs) + 3 * sum(rounds)
    a = fx.a[0].segment_ord
    got = {d for w in fx.batteries["strip"].want for _, g, d in w if g == a}
    for w in _strip_cuts(_ceil(N_A, WIN)):
        assert {w * WIN - 1, w * WIN, w * WIN + WIN - 1} <= got, w
    tied = fx.batteries["term"].want[next(i for i, q in enumerate(fx.batteries["term"].queries)
                                          if q["term_segs"][0][1] == fx.c[0].segment_ord and q["k"] == KMAX)]
    assert len({s for s, _, _ in tied}) == 1  # c0's top 1024 rows are one tied score


@pytest.mark.parametrize("full_units", [False, True])
def test_mixed_overflow_repeated_on_per_query_kernels(fx, full_units):
    """Term, AND, strip-union and window-union queries on the tile engine with a tile buffer of 64 pairs: the run overflows and
    is repeated on the per-query kernels, with the default units or one unit per (query, segment) pair."""
    queries, want = [], []
    for b in fx.batteries.values():
        queries += b.queries[::6]
        want += b.want[::6]
    env = dict(TQ_TILE=1, TQ_TILE_PCAP=64)
    if full_units:
        env["TQ_TARGET_UNITS"] = 1
    c = fx.register(_ctx_with_env(**env))
    try:
        g = c.search_batch(QueryBatch(queries))
        for i, w in enumerate(want):
            assert _bits(hits(g, i)) == _bits(w), (i, hits(g, i)[:4], w[:4])
        assert c.stats()["tile_fallbacks"] == 1
    finally:
        c.close()
