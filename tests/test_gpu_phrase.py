"""GPU parity of phrase queries (SURVEY.md §8f N3): k_phrase through the C ABI against the oracle's PhraseScorer restatement
(oracle/phrase.hpp, pinned on the reference's own phrase tests in tests/test_phrase_goldens.py / test_oracle_golden.py).
Segments are written in tantivy's format with positions (`.idx` WithFreqsAndPositions + `.pos`)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from oracle import tq_oracle as O  # noqa: E402
from tantivy_b200._abi import TQ_OP_PHRASE, TQ_RECORD_FREQS_POSITIONS, QueryBatch  # noqa: E402
from tests import score_model as M  # noqa: E402
from tests.helpers import OracleSegment, f32, hits  # noqa: E402
from tests.test_phrase_goldens import build  # noqa: E402


@pytest.fixture(scope="module")
def ctx():
    c = T.Context(0)
    yield c
    c.close()


_next = [7000]


class PosSegment:
    """One segment: posting lists with term frequencies, the matching `.pos` bytes, per-term ranges.  Built from `texts`, or
    with PosSegment.from_positions from explicit positions."""

    def __init__(self, texts, writer_cls=T.FieldWriter):
        postings, lengths = build(texts)
        self._build({t: {d: ps for d, ps in pl} for t, pl in postings.items()}, np.maximum(np.array(lengths), 1), None, writer_cls)

    @classmethod
    def from_positions(cls, positions, lengths, alive=None, writer_cls=T.FieldWriter):
        """positions = {term: {doc: ascending positions}}, lengths = every doc's token count (its fieldnorm), alive = the
        segment's alive bitset (np.packbits, little-endian) or None."""
        s = cls.__new__(cls)
        s._build(positions, np.asarray(lengths), alive, writer_cls)
        return s

    def _build(self, positions, lengths, alive, writer_cls):
        _next[0] += 1
        self.ord = _next[0]
        self.vocab = sorted(positions)
        self.positions = positions
        self.alive = alive
        lists, pos, self.pos_range = [], [], {}
        cursor = 0
        for t in self.vocab:
            docs = sorted(positions[t])
            lists.append((np.array(docs, dtype=np.uint32), np.array([len(positions[t][d]) for d in docs], dtype=np.uint32)))
            deltas = []
            for d in docs:
                ps = positions[t][d]
                deltas += [ps[0]] + [b - a for a, b in zip(ps, ps[1:])]
            data = bytes(O.positions_serialize(deltas))
            self.pos_range[t] = (cursor, cursor + len(data))
            cursor += len(data)
            pos.append(data)
        self.pos_bytes = np.frombuffer(b"".join(pos), dtype=np.uint8)
        self.lengths = lengths
        self.seg = OracleSegment(lists, lengths, record_option=TQ_RECORD_FREQS_POSITIONS, segment_ord=self.ord, writer_cls=writer_cls, alive=alive)
        self.n_docs = len(lengths)
        self.tokens = self.seg.total_num_tokens

    def model(self, vocab):
        """The same segment for tests/score_model.py, one posting list per term of `vocab` (empty where it is absent)."""
        lists, pos = [], []
        for t in vocab:
            p = self.positions.get(t, {})
            docs = sorted(p)
            lists.append((np.array(docs, dtype=np.uint32), np.array([len(p[d]) for d in docs], dtype=np.uint32)))
            pos.append(p)
        return M.Segment(self.ord, lists, self.lengths, alive=self.alive, positions=pos)

    def register(self, target):
        self.seg.register(target)
        target.register_positions(self.ord, 0, self.pos_bytes)

    def term(self, t):
        if t not in self.vocab:
            return None
        df, s, e = self.seg.terms[self.vocab.index(t)]
        ps, pe = self.pos_range[t]
        return df, s, e, ps, pe


def phrase_query(segs, phrase, k, offsets=None):
    offsets = list(range(len(phrase))) if offsets is None else offsets
    n_docs = sum(s.n_docs for s in segs)
    avg = f32(f32(sum(s.tokens for s in segs)) / f32(n_docs))
    idf_sum = f32(0)
    for t in phrase:
        df = sum((s.term(t) or (0,))[0] for s in segs)
        idf_sum = f32(idf_sum + O.bm25_idf(df, n_docs))
    weight = f32(idf_sum * f32(2.2))
    term_segs, term_pos, oracle_terms = [], [], []
    for clause, t in enumerate(phrase):
        for s in segs:
            ti = s.term(t)
            if ti is None:
                continue
            df, a, e, ps, pe = ti
            term_segs.append((clause, s.ord, 0, df, a, e))
            term_pos.append((ps, pe))
            oracle_terms.append((offsets[clause], s.ord, 0, df, a, e, ps, pe))
    q = dict(op=TQ_OP_PHRASE, k=k, weights=[weight] * len(phrase), avg_fieldnorm=[avg] * len(phrase), term_segs=term_segs, term_pos=term_pos,
             term_offset=offsets)
    return q, oracle_terms, weight, avg


def expected_rows(oi, segs, oracle_terms, n_phrase_terms, weight, avg, k, slop=0):
    """PhraseScorer per segment (only segments that hold every term), then TopDocs order."""
    rows = []
    for s in segs:
        mine = [t for t in oracle_terms if t[1] == s.ord]
        if len({t[0] for t in mine}) < n_phrase_terms:
            continue
        rows += oi.phrase_search(mine, weight, avg, slop=slop, cap=1 << 16)
    rows = sorted(((np.float32(sc), sg, d) for sg, d, sc, _ in rows), key=lambda r: (-r[0], r[1], r[2]))
    return [(float(sc), sg, d) for sc, sg, d in rows[:k]]


def check(ctx, segs, phrases, ks=(1, 10, 200)):
    oi = O.OracleIndex()
    for s in segs:
        s.register(oi)
        s.register(ctx)
    queries, want = [], []
    for phrase in phrases:
        for k in ks:
            q, ot, w, avg = phrase_query(segs, phrase, k)
            queries.append(q)
            want.append(expected_rows(oi, segs, ot, len(set(range(len(phrase)))), w, avg, k))
    qb = QueryBatch(queries)
    g = ctx.search_batch(qb)
    for i, w in enumerate(want):
        got = hits(g, i)
        assert [(s, d) for _, s, d in got] == [(s, d) for _, s, d in w], (phrases[i // len(ks)], got[:5], w[:5])
        assert [np.float32(x[0]) for x in got] == [np.float32(x[0]) for x in w]
    return g


def test_reference_phrase_fixtures(ctx):
    """src/query/phrase_query/mod.rs:41-91,163-169: doc sets and scores of the reference's own tests."""
    seg = PosSegment(["b b b d c g c", "a b b d c g c", "a b a b c", "c a b a d ga a", "a b c"])
    g = check(ctx, [seg], [["a", "b"], ["a", "b", "c"], ["b", "b"], ["g", "a"], ["c", "g", "c"]], ks=(10,))
    assert [d for _, _, d in hits(g, 0)] and sorted(d for _, _, d in hits(g, 0)) == [1, 2, 3, 4]
    assert sorted(d for _, _, d in hits(g, 1)) == [2, 4]
    assert sorted(d for _, _, d in hits(g, 2)) == [0, 1]
    assert hits(g, 3) == []
    seg2 = PosSegment(["a b c", "a b c a b"])
    g = check(ctx, [seg2], [["a", "b"]], ks=(10,))
    by_doc = {d: s for s, _, d in hits(g, 0)}
    assert abs(by_doc[0] - 0.40618482) <= 1e-6 and abs(by_doc[1] - 0.46844664) <= 1e-6


def _random_texts(rng, n_docs, vocab, lo, hi, p=None):
    words = np.array(vocab)
    out = []
    for _ in range(n_docs):
        n = int(rng.integers(lo, hi))
        out.append(" ".join(rng.choice(words, size=n, p=p)))
    return out


def test_phrases_over_many_blocks_and_segments(ctx):
    """Lists of several posting blocks, position streams of many bit-packed blocks + a VInt rest, three segments, phrases of
    2..5 terms, repeated terms, an absent term, k from 1 to 1000."""
    rng = np.random.default_rng(31)
    vocab = [f"w{i}" for i in range(12)]
    p = np.array([0.3, 0.2, 0.12, 0.1, 0.08, 0.06, 0.05, 0.04, 0.02, 0.015, 0.01, 0.005])
    p = p / p.sum()
    segs = [PosSegment(_random_texts(rng, n, vocab, 3, 60, p)) for n in (1500, 700, 2300)]
    phrases = [["w0", "w1"], ["w1", "w0"], ["w0", "w0"], ["w2", "w0", "w1"], ["w5", "w3"], ["w0", "w1", "w0", "w2"], ["w9", "w0"],
               ["w3", "w2", "w1", "w0", "w0"], ["w11", "w10"], ["w0", "zzz"]]
    check(ctx, segs, phrases, ks=(1, 10, 1000))


def test_long_documents_cross_position_blocks(ctx):
    """Docs with hundreds of occurrences of a term: one doc's positions span several 128-delta blocks."""
    rng = np.random.default_rng(32)
    vocab = ["x", "y", "z", "q"]
    segs = [PosSegment(_random_texts(rng, 300, vocab, 200, 900, [0.5, 0.3, 0.15, 0.05]))]
    check(ctx, segs, [["x", "y"], ["y", "x", "x"], ["q", "z"], ["x", "x", "x", "x"]], ks=(5, 300))


def check_slop(ctx, segs, phrases, slops, ks=(1, 10, 400), offsets=None):
    oi = O.OracleIndex()
    for s in segs:
        s.register(oi)
        s.register(ctx)
    queries, want, names = [], [], []
    for phrase in phrases:
        for slop in slops:
            for k in ks:
                q, ot, w, avg = phrase_query(segs, phrase, k, offsets=offsets)
                q["slop"] = slop
                queries.append(q)
                want.append(expected_rows(oi, segs, ot, len(phrase), w, avg, k, slop=slop))
                names.append((phrase, slop, k))
    qb = QueryBatch(queries)
    g = ctx.search_batch(qb)
    c = oi.search_batch(qb, mode=0)  # the oracle's batch path takes the query's slop too
    for i, w in enumerate(want):
        got = hits(g, i)
        assert [(s, d) for _, s, d in got] == [(s, d) for _, s, d in w], (names[i], got[:5], w[:5])
        assert [np.float32(x[0]) for x in got] == [np.float32(x[0]) for x in w], names[i]
        assert hits(c, i) == got, names[i]
    return g


def test_two_term_phrases_with_slop(ctx):
    """PhraseQuery::set_slop for two terms = intersection_count_with_slop (phrase_scorer.rs:145-186; the reference's cases
    phrase_query/mod.rs:117-160,292-330 are pinned on the oracle in tests/test_phrase_goldens.py): the doc sets and phrase counts of
    the oracle's PhraseScorer, for both term orders (which term is `left` follows the per-segment doc_freq), repeated terms,
    long docs whose positions cross 128-delta blocks, several segments."""
    seg = PosSegment(["a b c d", "a c b", "b a", "a x x b", "a x x x b", "b x a x b a", "a a a b b b", "c c", "b"])
    g = check_slop(ctx, [seg], [["a", "b"], ["b", "a"], ["a", "a"], ["c", "a"]], slops=(1, 2, 3), ks=(10,))
    by = lambda i: sorted(d for _, _, d in hits(g, i))
    assert by(0) == [0, 1, 5, 6]           # "a b"~1: adjacent or one word in between (a swap costs 2)
    assert by(1) == [0, 1, 2, 3, 5, 6]     # "a b"~2
    assert 4 in by(2) and 3 in by(2)       # "a b"~3
    rng = np.random.default_rng(77)
    vocab = [f"w{i}" for i in range(8)]
    p = np.array([0.35, 0.25, 0.15, 0.1, 0.07, 0.05, 0.02, 0.01])
    segs = [PosSegment(_random_texts(rng, n, vocab, 2, 50, p)) for n in (900, 1700)]
    check_slop(ctx, segs, [["w0", "w1"], ["w1", "w0"], ["w4", "w0"], ["w0", "w5"], ["w2", "w2"], ["w6", "w7"], ["w0", "zzz"]], slops=(1, 2, 5))
    long_seg = PosSegment(_random_texts(rng, 250, ["x", "y", "z", "q"], 200, 700, [0.5, 0.3, 0.15, 0.05]))
    check_slop(ctx, [long_seg], [["x", "y"], ["q", "z"], ["z", "q"], ["x", "x"]], slops=(1, 4), ks=(5, 300))
    # offsets other than 0, 1 (PhraseQuery::new_with_offset): "w0 * w1" with slop
    segs2 = [PosSegment(_random_texts(rng, n, vocab, 2, 50, p)) for n in (600, 800)]
    check_slop(ctx, segs2, [["w0", "w1"], ["w3", "w0"]], slops=(1, 3), offsets=[0, 2], ks=(10,))


def test_phrase_needs_positions_and_rejects_slop(ctx):
    seg = PosSegment(["a b c", "a b"])
    seg.seg.register(ctx)  # postings only, no positions yet
    q, _, _, _ = phrase_query([seg], ["a", "b"], 10)
    with pytest.raises(T.TqError):
        ctx.search_batch(QueryBatch([q]))
    ctx.register_positions(seg.ord, 0, seg.pos_bytes)
    assert len(hits(ctx.search_batch(QueryBatch([q])), 0)) == 2
    q2 = dict(q)
    q2["slop"] = 1
    assert len(hits(ctx.search_batch(QueryBatch([q2])), 0)) == 2  # two terms: slop runs on the device
    q3, _, _, _ = phrase_query([seg], ["a", "b", "c"], 10)
    q3["slop"] = 1
    with pytest.raises(T.TqError):  # three and more terms with slop (carrying slops) stay on the reference's CPU path
        ctx.search_batch(QueryBatch([q3]))


def test_synthetic_index_with_positions_mixed_batch(ctx):
    """The benchmark's generator with positions (csrc/synth.cpp, record_option 2): phrase queries in one batch with term / AND /
    OR queries (BASELINE.json configs[3]'s mix), several segments, against the oracle's search_batch (PhraseScorer restatement)."""
    from tantivy_b200._abi import TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM
    dens = [0.3, 0.15, 0.05, 0.01, 0.002]
    ix = T.SynthIndex(3, 400_000, dens, seed=11, record_option=TQ_RECORD_FREQS_POSITIONS)
    base = 8800
    ix.register(ctx, segment_base=base)
    oi = O.OracleIndex()
    ix.register(oi, segment_base=base)
    qs = []
    for k in (1, 10, 100):
        for terms in ([0, 1], [1, 0], [0, 0], [0, 1, 2], [2, 0], [3, 0], [0, 1, 0], [4, 3]):
            qs.append(ix.phrase_query(terms, k, segment_base=base))
        qs += [ix.query(TQ_OP_OR, [0, 2, 4], k, segment_base=base), ix.query(TQ_OP_AND, [1, 2], k, segment_base=base), ix.query(TQ_OP_TERM, [3], k, segment_base=base)]
    qb = QueryBatch(qs)
    g = ctx.search_batch(qb)
    c = oi.search_batch(qb, mode=0, n_threads=8)
    for i in range(qb.nq):
        assert hits(g, i) == hits(c, i), (i, hits(g, i)[:3], hits(c, i)[:3])
    assert any(len(hits(g, i)) > 0 for i in range(8))  # the phrases do match
    assert ctx.stats()["units_phrase"] > 0
