"""A long-lived context against the numpy model of tests/score_model.py: what it keeps between batches.

A context caches block tables (list_cache) and position tables (pos_cache) across batches, recycles their ids when a segment is
unregistered, rolls back the builds of a batch that fails, and reuses pooled batch buffers.  The tests here drive one context through
all of that and compare every answer with the model (docs, segment ordinals and f32 scores, zero by value), and the cache counters of
tq_stats with a test-side model of the cache:

  * position-cache collisions: terms whose (postings_start, positions_start) pairs a key folded into one word would confuse;
  * a seeded session per engine: segments registered (deletes, positions, Basic, no fieldnorms, odd max_doc), unregistered and
    replaced by other content under the same ordinal, doc ranges, searches and Counts of every query shape, the two cache entries of
    a list read with and without freqs, failing batches, prepared batches run out of order and pooled buffers that grow and shrink;
  * capacity limits (TQ_MAX_LISTS, TQ_MAX_POS_LISTS) and recycled ids;
  * tq_segment_unregister refused while a prepared batch names the segment.
"""
import copy
from collections import Counter, defaultdict

import numpy as np
import pytest

import tantivy_b200 as T
from oracle import tq_oracle as O
from tantivy_b200._abi import (TQ_OP_AND, TQ_OP_BOOL, TQ_OP_OR, TQ_OP_PHRASE, TQ_OP_TERM, TQ_RECORD_BASIC, TQ_RECORD_FREQS,
                               TQ_TERM_IGNORE_FREQ, QueryBatch)
from tests import score_model as M
from tests.helpers import OracleSegment, bool_shape_query, hits, make_query, random_bool_shapes
from tests.test_gpu_parity import _ctx_with_env
from tests.test_gpu_phrase import PosSegment, phrase_query


# ---- position-cache keys ----------------------------------------------------------------------------------------------------
def _folded_pos_key(postings_start, positions_start):
    """The position-cache key the library once used: both offsets folded into one word.  Two terms collide when
    pA ^ 2 sA == pB ^ 2 sB."""
    return positions_start ^ (postings_start << 1) ^ (1 << 62)


class Collisions:
    """A Zipf-text phrase segment (oracle writer) and the pairs of its terms (vocabulary indices a < b) whose folded keys are equal."""

    def __init__(self):
        rng = np.random.default_rng(0xC011)
        n_words = 6000
        p = 1.0 / np.arange(1, n_words + 1) ** 1.05
        words = np.array([f"w{i:04d}" for i in range(n_words)])
        self.texts = [" ".join(rng.choice(words, size=int(rng.integers(5, 60)), p=p / p.sum())) for _ in range(2500)]
        self.seg = PosSegment(self.texts, writer_cls=O.FieldWriter)
        self.index = {t: i for i, t in enumerate(self.seg.vocab)}
        by_key = defaultdict(list)
        for i, t in enumerate(self.seg.vocab):
            _, s, _, ps, _ = self.seg.term(t)
            by_key[_folded_pos_key(s, ps)].append(i)
        self.pairs = [(a, b) for v in by_key.values() for x, a in enumerate(v) for b in v[x + 1:]]

    def phrases(self, i):
        """Phrases around the first occurrence of term i that has two words after it and one before: "t next", "t . after"~1,
        "before t next"."""
        t = self.seg.vocab[i]
        for d in sorted(self.seg.positions[t]):
            toks = self.texts[d].split()
            for j in self.seg.positions[t][d]:
                if 1 <= j and j + 2 < len(toks):
                    return [([t, toks[j + 1]], 0), ([t, toks[j + 2]], 1), ([toks[j - 1], t, toks[j + 1]], 0)]
        return None


@pytest.fixture(scope="module")
def coll():
    return Collisions()


def test_folded_position_key_collides_on_the_fixture(coll):
    """The fixture holds the case the GPU test below is about: at least 20 pairs of distinct terms whose folded keys are equal,
    some adjacent in the term dictionary, some far apart."""
    assert len(coll.pairs) >= 20, len(coll.pairs)
    assert sum(b - a == 1 for a, b in coll.pairs) >= 5
    assert sum(b - a > 100 for a, b in coll.pairs) >= 5
    for a, b in coll.pairs:
        ta, tb = coll.seg.term(coll.seg.vocab[a]), coll.seg.term(coll.seg.vocab[b])
        assert (ta[1], ta[3]) != (tb[1], tb[3])
        assert _folded_pos_key(ta[1], ta[3]) == _folded_pos_key(tb[1], tb[3])


def _with_ord(ps, ordinal):
    """The same segment bytes under another ordinal."""
    c = copy.copy(ps)
    c.seg = copy.copy(ps.seg)
    c.ord = c.seg.segment_ord = ordinal
    return c


def _phrase_battery(segs, model, index, phrases):
    queries, terms = [], []
    for words, slop in phrases:
        q = phrase_query(segs, words, 1000)[0]
        q["slop"] = slop
        queries.append(q)
        terms.append([index[w] for w in words])
    return queries, [M.search(model, q, t) for q, t in zip(queries, terms)]


@pytest.mark.gpu
def test_phrases_on_terms_whose_folded_position_keys_collide(coll):
    """On one context: phrases of every term A of the colliding pairs, then a separate batch of every B (B's position table must not
    be A's), then both mixed; then the three again on a second ordinal that holds the same bytes.  Two-term phrases, with slop, and
    three-term phrases, k = 1000: every match is compared with the model and the oracle."""
    usable = [(a, b) for a, b in coll.pairs if coll.phrases(a) and coll.phrases(b)]
    adjacent = [p for p in usable if p[1] - p[0] == 1][:16]
    far = [p for p in usable if p[1] - p[0] > 100][:16]
    chosen = adjacent + far
    assert len(adjacent) >= 5 and len(far) >= 5
    ctx = T.Context(0)
    try:
        for seg in (coll.seg, _with_ord(coll.seg, coll.seg.ord + 5000)):
            seg.register(ctx)
            oi = O.OracleIndex()
            seg.register(oi)
            model = [seg.model(seg.vocab)]
            side_a = [ph for a, _ in chosen for ph in coll.phrases(a)]
            side_b = [ph for _, b in chosen for ph in coll.phrases(b)]
            mixed = [ph for a, b in chosen for ph in coll.phrases(b)[:2] + coll.phrases(a)[1:]]
            for name, phrases in (("A", side_a), ("B", side_b), ("mixed", mixed)):
                queries, want = _phrase_battery([seg], model, coll.index, phrases)
                qb = QueryBatch(queries)
                g = ctx.search_batch(qb)
                c = oi.search_batch(qb, mode=0)
                for i, w in enumerate(want):
                    assert hits(g, i) == w, (seg.ord, name, phrases[i], hits(g, i)[:4], w[:4])
                    assert hits(c, i) == w, ("oracle", seg.ord, name, phrases[i])
                assert sum(len(w) > 0 for w in want) >= len(want) // 2  # the phrases do match
    finally:
        ctx.close()


# ---- segments of the session ------------------------------------------------------------------------------------------------
N_TERMS = 6
NAMES = [f"t{i}" for i in range(N_TERMS)]  # (sorted: a PosSegment's list i is term i)
DENS = (0.4, 0.15, 0.06, 0.02, 0.008, 0.003)
KS = (1, 10, 129, 1000)
KINDS = ("basic", "no_fieldnorms", "positions_deletes", "freqs", "deletes", "positions")  # (register steps take them in turn)


class Seg:
    """One segment's content under an ordinal: the bytes (OracleSegment, and a PosSegment for the kinds with positions) and the
    model's view of it."""

    def __init__(self, rng, ordinal, kind):
        self.ord, self.kind = ordinal, kind
        self.basic = kind == "basic"
        self.ps = None
        with_pos = kind.startswith("positions")
        max_doc = 2 * int(rng.integers(1000, 3000 if with_pos else 10000)) + 1  # odd: never a multiple of 32 or 8192
        alive = np.packbits(rng.random(max_doc) > 0.25, bitorder="little") if kind.endswith("deletes") else None
        if with_pos:
            lengths = rng.integers(2, 24, size=max_doc)
            words = rng.choice(N_TERMS, size=int(lengths.sum()), p=np.array(DENS) / sum(DENS))
            positions = {t: {} for t in NAMES}
            at = 0
            for d, n in enumerate(lengths.tolist()):
                for j, w in enumerate(words[at:at + n].tolist()):
                    positions[NAMES[w]].setdefault(d, []).append(j)
                at += n
            assert all(positions.values())
            self.ps = PosSegment.from_positions(positions, lengths, alive=alive)
            self.ps.ord = self.ps.seg.segment_ord = ordinal
            self.o = self.ps.seg
            self.m = self.ps.model(NAMES)
        else:
            lists = []
            for p in DENS:
                docs = np.nonzero(rng.random(max_doc) < p)[0].astype(np.uint32)
                if len(docs) == 0:
                    docs = np.array([max_doc - 1], np.uint32)
                lists.append((docs, None if self.basic else rng.integers(1, 9, size=len(docs)).astype(np.uint32)))
            lengths = None if kind == "no_fieldnorms" else rng.integers(1, 60, size=max_doc)
            self.o = OracleSegment(lists, lengths, record_option=TQ_RECORD_BASIC if self.basic else TQ_RECORD_FREQS, segment_ord=ordinal,
                                   writer_cls=T.FieldWriter, alive=alive, max_doc=max_doc)
            self.m = M.Segment(ordinal, lists, lengths, alive=alive, basic=self.basic, max_doc=max_doc)
        self.max_doc = max_doc

    def register(self, ctx):
        if self.ps is not None:
            self.ps.register(ctx)
        else:
            self.o.register(ctx)

    def restrict(self, lo, hi):
        """The model of tq_segment_set_doc_range(lo, hi): docs outside [lo, hi) count as deleted."""
        keep = np.zeros(self.max_doc, bool)
        keep[lo:hi] = True
        self.m.alive = keep if self.m.alive is None else self.m.alive & keep


def _q(op, segs, terms, k, **extra):
    q = make_query(op, [s.o for s in segs], list(terms), k)
    q.update(extra)
    return q, list(terms)


def _phrase(segs, terms, k, slop=0):
    q = phrase_query([s.ps for s in segs], [NAMES[t] for t in terms], k)[0]
    q["slop"] = slop
    return q, list(terms)


class Session:
    """One context, the segments registered on it, and a model of its list cache: the (segment, postings_start, ignore_freq) keys
    that were built by a batch that succeeded, on segments still registered."""

    def __init__(self, ctx, engine, seed):
        self.ctx, self.tile = ctx, engine == "tile"
        self.rng = np.random.default_rng(seed)
        self.segs = {}
        self.freed = []
        self.cache = set()
        self.built = 0
        self.max_nq = self.max_k = 0
        self.next_ord = 100
        self.shapes = random_bool_shapes(np.random.default_rng(seed + 1), 24, N_TERMS, n_wide=0)
        self.n_shapes = 0
        self.done = Counter()
        self.kind_i = 0

    # -- the cache model --
    def keys(self, q, search):
        """get_list's keys for one query: the clauses of each segment where the query can match (an AND or a phrase needs every
        clause there); a Count reads every list with its freqs."""
        n = len(q["weights"])
        flags = q.get("term_flags") if search else None
        per = defaultdict(list)
        for ts in q["term_segs"]:
            if ts[3] > 0:
                per[ts[1]].append(ts)
        out = set()
        for so, tss in per.items():
            if q["op"] in (TQ_OP_AND, TQ_OP_PHRASE) and len(tss) != n:
                continue
            for ts in tss:
                ignore = flags is not None and bool(flags[ts[0]] & TQ_TERM_IGNORE_FREQ) and not self.segs[so].basic
                out.add((so, ts[4], ignore))
        return out

    def absorb(self, qs, search=True):
        new = set().union(*[self.keys(q, search) for q, _ in qs]) - self.cache
        self.cache |= new
        return len(new)

    def check_cache(self, what):
        st = self.ctx.stats()
        assert st["lists_cached"] == len(self.cache), (what, st["lists_cached"], len(self.cache))
        assert st["lists_built"] == self.built, (what, st["lists_built"], self.built)

    # -- segments --
    def live(self):
        return [self.segs[o] for o in sorted(self.segs)]

    def register(self, kind=None, ordinal=None):
        if kind is None:
            kind = KINDS[self.kind_i % len(KINDS)]
            self.kind_i += 1
        if ordinal is None:
            ordinal = self.next_ord
            self.next_ord += 1
        s = Seg(self.rng, ordinal, kind)
        s.register(self.ctx)
        self.segs[ordinal] = s
        self.done["register_" + kind] += 1
        return s

    def unregister(self, ordinal=None):
        if ordinal is None:
            ordinal = int(self.rng.choice(sorted(self.segs)))
        self.ctx.segment_unregister(ordinal, 0)
        del self.segs[ordinal]
        self.cache = {k for k in self.cache if k[0] != ordinal}
        self.freed.append(ordinal)
        self.done["unregister"] += 1

    # -- queries --
    def _k(self):
        return int(self.rng.choice(KS))

    def _terms(self, lo, hi):
        return sorted(int(t) for t in self.rng.choice(N_TERMS, size=int(self.rng.integers(lo, hi + 1)), replace=False))

    def queries(self, segs=None, count=False):
        """Term, AND, OR and (tile engine or Count) BOOL queries over the segments, phrases over those with positions (not in a
        Count); one query with an initial threshold taken from its own model rows."""
        segs = segs or self.live()
        r = self.rng
        qs = [_q(TQ_OP_TERM, segs, [int(r.integers(N_TERMS))], self._k()) for _ in range(2)]
        qs += [_q(TQ_OP_AND, segs, self._terms(2, 3), self._k()), _q(TQ_OP_OR, segs, self._terms(2, 4), self._k())]
        if self.tile or count:
            for _ in range(2):
                shape = self.shapes[self.n_shapes % len(self.shapes)]
                self.n_shapes += 1
                qs.append((bool_shape_query([s.o for s in segs], shape), list(shape["terms"])))
        pos = [s for s in segs if s.ps is not None]
        if pos and not count:
            a, b, c = (int(t) for t in r.choice(N_TERMS, size=3, replace=False))
            qs += [_phrase(pos, [a, b], self._k(), slop=int(r.integers(0, 3))), _phrase(pos, [b, a, c], self._k()), _phrase(pos, [a, a], 10)]
        if not count:
            i = int(r.integers(len(qs)))
            q, t = qs[i]
            rows = self.model_rows(dict(q, threshold=None), t)
            if rows:
                qs[i] = (dict(q, threshold=rows[len(rows) // 2][0]), t)
                self.done["threshold"] += 1
        return qs

    def model_rows(self, q, terms):
        return M.search([s.m for s in self.live()], q, terms)

    def check_rows(self, result, qs, what):
        for i, (q, t) in enumerate(qs):
            want = self.model_rows(q, t)
            got = hits(result, i)
            assert got == want, (what, i, q["op"], t, q["k"], q.get("threshold"), got[:4], want[:4])

    # -- steps --
    def search(self, qs=None, what="search"):
        qs = qs if qs is not None else self.queries()
        g = self.ctx.search_batch(QueryBatch([q for q, _ in qs]))
        self.check_rows(g, qs, what)
        self.built = self.absorb(qs)
        self.max_nq = max(self.max_nq, len(qs))
        self.max_k = max([self.max_k] + [q["k"] for q, _ in qs])
        self.done["search"] += 1
        self.done.update(op_name(q) for q, _ in qs)
        return g

    def count(self, qs=None):
        qs = qs if qs is not None else self.queries(count=True)
        got = self.ctx.count_batch(QueryBatch([q for q, _ in qs]))
        msegs = [s.m for s in self.live()]
        assert [int(x) for x in got] == [M.count(msegs, q, t) for q, t in qs], ("count", [q["op"] for q, _ in qs])
        self.absorb(qs, search=False)  # (a Count publishes no batch statistics: lists_built stays the last search's)
        self.done["count"] += 1

    def ignore_freq(self):
        """One list read with its freqs and without them: two cache entries, two scorings."""
        segs = [s for s in self.live() if not s.basic and s.kind != "no_fieldnorms"] or [self.register("freqs")]
        s = segs[int(self.rng.integers(len(segs)))]
        t = int(self.rng.integers(3))
        with_f = _q(TQ_OP_TERM, [s], [t], 1000)
        without = _q(TQ_OP_TERM, [s], [t], 1000, term_flags=[TQ_TERM_IGNORE_FREQ])
        self.search([with_f], "freqs")
        self.search([without], "ignore_freq")
        g = self.search([with_f, without], "both")
        assert [x[0] for x in hits(g, 0)] != [x[0] for x in hits(g, 1)]
        assert (s.ord, s.o.terms[t][1], False) in self.cache and (s.ord, s.o.terms[t][1], True) in self.cache
        self.done["ignore_freq"] += 1

    def doc_range(self):
        """A freshly registered segment restricted to [lo, hi) before its first search (the alive bitset is created then): lo and
        hi inside bytes of the bitset."""
        s = self.register(("freqs", "deletes", "positions")[self.done["doc_range"] % 3])
        lo = 8 * int(self.rng.integers(1, s.max_doc // 40)) + 3
        hi = s.max_doc - 8 * int(self.rng.integers(1, s.max_doc // 40)) - 5
        self.ctx.segment_set_doc_range(s.ord, 0, lo, hi)
        s.restrict(lo, hi)
        solo = [_q(TQ_OP_TERM, [s], [t], 1000) for t in range(3)]
        self.count(solo + self.queries(count=True))
        self.search(solo + self.queries())
        self.done["doc_range"] += 1

    def fresh_lists(self, n):
        """(segment, term, flags) of lists not in the cache, for queries that schedule new builds."""
        out = []
        for s in self.live():
            for t in range(N_TERMS):
                for flags in ([0], [TQ_TERM_IGNORE_FREQ]):
                    key = (s.ord, s.o.terms[t][1], bool(flags[0]) and not s.basic)
                    if key not in self.cache and key not in {(x.ord, x.o.terms[u][1], bool(f[0]) and not x.basic) for x, u, f in out}:
                        out.append((s, t, flags))
        idx = self.rng.permutation(len(out))[:n]
        return [out[i] for i in idx]

    def fail(self, kind):
        """A batch of valid queries on lists not yet built, then one that fails: nothing of it stays in the cache, the next batch
        answers, and the lists the failed batch had scheduled are built and searched."""
        if kind == "positions_range" and not any(s.ps is not None for s in self.live()):
            self.register("positions")
        fresh = self.fresh_lists(N_TERMS * 2 * len(self.segs))
        if not any(f == [0] for _, _, f in fresh) or len(fresh) < 3:
            self.register("freqs")
            fresh = self.fresh_lists(N_TERMS * 2 * len(self.segs))
        target = next(x for x in fresh if x[2] == [0])  # (its list is not cached as read with freqs)
        cs, ct, _ = target
        valid = [_q(TQ_OP_TERM, [s], [t], 10, term_flags=f) for s, t, f in [x for x in fresh if x is not target][:2]]
        if kind == "unknown_segment":
            bad = _q(TQ_OP_TERM, [cs], [ct], 10)[0]
            bad["term_segs"] = [(0, max(self.next_ord, 100) + 1000, 0, 10, 0, 10)]
            code = -3
        elif kind == "postings_range":
            bad = _q(TQ_OP_TERM, [cs], [ct], 10)[0]
            df, start, _ = cs.o.terms[ct]
            bad["term_segs"] = [(0, cs.ord, 0, df, start, len(cs.o.body))]
            code = -1
        elif kind == "positions_range":
            ps = [s for s in self.live() if s.ps is not None][0]
            bad = _phrase([ps], [0, 1], 10)[0]
            start = bad["term_pos"][0][0]
            bad["term_pos"] = [(start, len(ps.ps.pos_bytes) + 16)] + list(bad["term_pos"][1:])
            code = -1
        else:  # corrupt: doc_freq 1000 in two bytes, at the start of a real list that is not cached (its key is the list's)
            bad = _q(TQ_OP_TERM, [cs], [ct], 10)[0]
            df, start, _ = cs.o.terms[ct]
            bad["term_segs"] = [(0, cs.ord, 0, 1000, start, start + 2)]
            code = -6
        with pytest.raises(T.TqError, match=rf"error {code}:"):
            self.ctx.search_batch(QueryBatch([q for q, _ in valid] + [bad]))
        self.check_cache("failed " + kind)
        # the real list under the rolled-back key of the corrupt one is built afresh
        self.search(valid + [_q(TQ_OP_TERM, [cs], [ct], 1000)] + self.queries(), "after failed " + kind)
        self.done["fail_" + kind] += 1

    def prepared(self):
        """Three prepared batches run out of order, one of them twice, fetched in another order; a segment they name cannot be
        unregistered meanwhile."""
        sets = [self.queries() for _ in range(3)]
        batches, built = [], []
        try:
            for qs in sets:
                batches.append(self.ctx.prepare(QueryBatch([q for q, _ in qs])))
                built.append(self.absorb(qs))
            named = sets[0][0][0]["term_segs"][0][1]
            with pytest.raises(T.TqError, match="a prepared batch still uses the segment"):
                self.ctx.segment_unregister(named, 0)
            for i in (1, 0, 2, 0):
                batches[i].run()
            for i in (2, 0, 1):
                self.check_rows(batches[i].fetch(), sets[i], f"prepared {i}")
                self.built = built[i]  # (the fetched batch's builds, counted when it was prepared)
                self.check_cache(f"prepared {i}")
        finally:
            for b in batches:
                b.close()
        self.max_nq = max([self.max_nq] + [len(qs) for qs in sets])
        self.done["prepared"] += 1

    def grow_and_shrink(self):
        """A prepared batch larger in nq than any before on this context and with k = TQ_MAX_K (its pooled buffers must grow), then a
        smaller one."""
        big = []
        while len(big) <= self.max_nq:
            big += self.queries()
        big += [_q(TQ_OP_OR, self.live(), [0, 1, 2], 1024), _q(TQ_OP_TERM, self.live(), [0], 1024)]
        assert len(big) > self.max_nq and (self.max_k < 1024 or self.done["grow_and_shrink"])
        small = self.queries()[:2]
        for qs in (big, small):
            b = self.ctx.prepare(QueryBatch([q for q, _ in qs]))
            try:
                self.built = self.absorb(qs)
                b.run()
                self.check_rows(b.fetch(), qs, f"pooled {len(qs)}")
            finally:
                b.close()
            self.check_cache(f"pooled {len(qs)}")
        self.max_nq, self.max_k = len(big), 1024
        self.done["grow_and_shrink"] += 1

    def reregister(self):
        """Different content under an ordinal that was unregistered: a stale table or descriptor would show up as wrong rows."""
        if not self.freed:
            self.unregister()
        ordinal = self.freed.pop(int(self.rng.integers(len(self.freed))))
        self.register(KINDS[int(self.rng.integers(len(KINDS)))], ordinal)
        self.done["reregister"] += 1
        self.search(self.queries(), "re-registered")


def op_name(q):
    return {TQ_OP_TERM: "term", TQ_OP_AND: "and", TQ_OP_OR: "or", TQ_OP_BOOL: "bool", TQ_OP_PHRASE: "phrase"}[q["op"]]


STEPS = (["search"] * 6 + ["count"] * 4 + ["register"] * 4 + ["unregister"] * 3 + ["reregister"] * 3 + ["ignore_freq"] * 2 + ["doc_range"] * 2
         + ["fail_unknown_segment", "fail_postings_range", "fail_positions_range", "fail_corrupt"] + ["prepared"] * 2 + ["grow_and_shrink"] * 2)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["tile", "legacy"])
def test_seeded_long_lived_session(engine):
    """About forty seeded steps on one context (TQ_TILE=1 / 0; BOOL only on the tile engine), each answer against the model, the
    cache counters against the cache model after every step."""
    ctx = _ctx_with_env(TQ_TILE=1 if engine == "tile" else 0)
    s = Session(ctx, engine, 0x5E55 + (engine == "tile"))
    try:
        for kind in ("freqs", "positions", "positions_deletes", "deletes"):
            s.register(kind)
        s.check_cache("start")
        order = [STEPS[i] for i in s.rng.permutation(len(STEPS))]
        for n, step in enumerate(order):
            if step.startswith("fail_"):
                s.fail(step[5:])
            elif step == "register":
                if len(s.segs) >= 7:
                    s.unregister()
                s.register()
            elif step == "unregister":
                if len(s.segs) <= 2:
                    s.register()
                s.unregister()
            else:
                getattr(s, step)()
            s.check_cache(f"step {n}: {step}")
        for kind in KINDS:
            assert s.done["register_" + kind] >= 1, kind
        need = ["unregister", "reregister", "search", "count", "threshold", "ignore_freq", "doc_range", "prepared", "grow_and_shrink",
                "term", "and", "or", "phrase", "fail_unknown_segment", "fail_postings_range", "fail_positions_range", "fail_corrupt"]
        for what in need + (["bool"] if engine == "tile" else []):
            assert s.done[what] >= 1, (what, s.done)
    finally:
        ctx.close()


# ---- capacity limits ----------------------------------------------------------------------------------------------------------
def _search_model(ctx, segs, qs):
    g = ctx.search_batch(QueryBatch([q for q, _ in qs]))
    for i, (q, t) in enumerate(qs):
        assert hits(g, i) == M.search([s.m for s in segs], q, t), i


@pytest.mark.gpu
def test_list_cache_capacity():
    """TQ_MAX_LISTS=8: a batch that needs more block tables than are left fails with TQ_ERR_OOM and leaves the cache as it was; a
    batch that fits answers; once a segment is unregistered the batch that failed runs on the recycled ids."""
    rng = np.random.default_rng(81)
    a, b = Seg(rng, 1, "freqs"), Seg(rng, 2, "deletes")
    ctx = _ctx_with_env(TQ_MAX_LISTS=8)
    try:
        for s in (a, b):
            s.register(ctx)
        _search_model(ctx, [a, b], [_q(TQ_OP_OR, [a], [0, 1, 2, 3, 4], 100)])
        assert ctx.stats()["lists_cached"] == 5
        big = [_q(TQ_OP_OR, [b], list(range(N_TERMS)), 100), _q(TQ_OP_AND, [b], [0, 5], 10)]
        with pytest.raises(T.TqError, match=r"error -5: .*TQ_MAX_LISTS"):
            ctx.search_batch(QueryBatch([q for q, _ in big]))
        assert ctx.stats()["lists_cached"] == 5
        _search_model(ctx, [a, b], [_q(TQ_OP_AND, [b], [0, 1], 10), _q(TQ_OP_TERM, [a, b], [0], 1000)])
        assert ctx.stats()["lists_cached"] == 7
        with pytest.raises(T.TqError, match=r"error -5: .*TQ_MAX_LISTS"):
            ctx.search_batch(QueryBatch([q for q, _ in big]))
        assert ctx.stats()["lists_cached"] == 7
        ctx.segment_unregister(a.ord, 0)
        assert ctx.stats()["lists_cached"] == 2
        _search_model(ctx, [b], big)
        st = ctx.stats()
        assert st["lists_cached"] == 6 and st["lists_built"] == 4
    finally:
        ctx.close()


@pytest.mark.gpu
def test_position_cache_capacity():
    """TQ_MAX_POS_LISTS=3: a phrase batch that needs more position tables than are left fails with TQ_ERR_OOM (its block tables are
    rolled back too); phrases that fit answer; after the other segment is unregistered the batch runs on recycled position ids."""
    rng = np.random.default_rng(82)
    p, q = Seg(rng, 1, "positions"), Seg(rng, 2, "positions_deletes")
    ctx = _ctx_with_env(TQ_MAX_POS_LISTS=3)
    try:
        for s in (p, q):
            s.register(ctx)
        _search_model(ctx, [p, q], [_phrase([p], [0, 1], 1000), _phrase([p], [1, 0], 1000, slop=1)])
        assert ctx.stats()["lists_cached"] == 2
        three = [_phrase([q], [0, 1, 2], 1000), _phrase([q], [2, 0], 10)]
        with pytest.raises(T.TqError, match=r"error -5: .*TQ_MAX_POS_LISTS"):
            ctx.search_batch(QueryBatch([x for x, _ in three]))
        assert ctx.stats()["lists_cached"] == 2
        _search_model(ctx, [p, q], [_phrase([p], [2, 0], 1000), _phrase([p], [0, 1, 2], 1000)])  # the third table
        assert ctx.stats()["lists_cached"] == 3
        with pytest.raises(T.TqError, match=r"error -5: .*TQ_MAX_POS_LISTS"):
            ctx.search_batch(QueryBatch([x for x, _ in three]))
        ctx.segment_unregister(p.ord, 0)
        _search_model(ctx, [q], three)
        assert ctx.stats()["lists_cached"] == 3
    finally:
        ctx.close()


# ---- unregister under a prepared batch --------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_unregister_refused_while_a_prepared_batch_names_the_segment():
    """A prepared batch holds its segments' list ids and alive pointers: unregistering one of them is refused until the batch is
    closed; a segment the batch does not name can go.  Afterwards the context answers, also for new content under the ordinal."""
    rng = np.random.default_rng(83)
    a, b, c = Seg(rng, 1, "freqs"), Seg(rng, 2, "deletes"), Seg(rng, 3, "basic")
    ctx = T.Context(0)
    try:
        for s in (a, b, c):
            s.register(ctx)
        qs = [_q(TQ_OP_TERM, [a], [0], 10), _q(TQ_OP_OR, [a, b], [0, 1, 3], 100)]
        bt = ctx.prepare(QueryBatch([q for q, _ in qs]))
        try:
            bt.run()
            for o in (a.ord, b.ord):
                with pytest.raises(T.TqError, match=r"error -1: a prepared batch still uses the segment"):
                    ctx.segment_unregister(o, 0)
            ctx.segment_unregister(c.ord, 0)
            out = bt.fetch()
            for i, (q, t) in enumerate(qs):
                assert hits(out, i) == M.search([a.m, b.m], q, t)
        finally:
            bt.close()
        ctx.segment_unregister(a.ord, 0)
        assert ctx.stats()["lists_cached"] == 3  # b's lists 0, 1, 3
        _search_model(ctx, [b], [_q(TQ_OP_OR, [b], [0, 1, 3], 100)])
        a2 = Seg(rng, a.ord, "no_fieldnorms")
        a2.register(ctx)
        _search_model(ctx, [a2, b], [_q(TQ_OP_TERM, [a2], [0], 10), _q(TQ_OP_OR, [a2, b], [0, 1, 3], 100)])
    finally:
        ctx.close()
