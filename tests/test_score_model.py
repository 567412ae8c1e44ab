"""The numpy model of the reference's scorers (tests/score_model.py) against the reference's pinned scores and against the oracle,
bit for bit.  The oracle is our own restatement of the reference; the model is a second, independent one, so a decision the oracle
and the kernels share (they are compared with each other everywhere else) is checked here.  Runs on CPU."""
import numpy as np
import pytest

from oracle import tq_oracle as O
from tantivy_b200._abi import (TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT, TQ_OCCUR_SHOULD, TQ_OP_AND, TQ_OP_BOOL, TQ_OP_OR, TQ_OP_TERM,
                               TQ_RECORD_BASIC, TQ_RECORD_FREQS, TQ_RECORD_FREQS_POSITIONS, QueryBatch)
from tests import score_model as M
from tests.helpers import (BOOL_BOOSTS, BOOL_BRANCHES, BOOL_KS, BOOL_SHAPES, OracleSegment, bool_branches, bool_query, bool_shape_query,
                          hits, make_query, random_bool_shapes)


def _pair(lists, lengths, segment_ord=0, alive=None, record_option=TQ_RECORD_FREQS, max_doc=None):
    """The same segment for the oracle and for the model."""
    o = OracleSegment(lists, lengths, record_option=record_option, segment_ord=segment_ord, alive=alive, max_doc=max_doc)
    m = M.Segment(segment_ord, lists, lengths, alive=alive, basic=record_option == TQ_RECORD_BASIC, max_doc=max_doc)
    return o, m


def _oracle(osegs, queries, mode=0):
    ix = O.OracleIndex()
    for s in osegs:
        s.register(ix)
    return ix.search_batch(QueryBatch(queries), mode=mode)


def _assert_model_is_oracle(osegs, msegs, queries, terms, modes=(0,)):
    for mode in modes:
        res = _oracle(osegs, [q for q in queries], mode)
        for i, (q, t) in enumerate(zip(queries, terms)):
            want = M.search(msegs, q, t)
            got = hits(res, i)
            assert got == want, f"query {i} (mode {mode}): oracle {got[:4]} != model {want[:4]}"
    return res


# ---- the reference's pinned scores -------------------------------------------------------------------------------------
def _near(a, b, rel=1e-6):
    return abs(a - b) <= rel * max(abs(a), abs(b))


def test_pinned_union_and_boost():
    # src/query/boolean_query/mod.rs:221-259: docs "a b c", "a c", "b c"; a OR b; doc 0 scores 0.84163445, 1.6832689 with boost 2
    o, m = _pair([([0, 1], [1, 1]), ([0, 2], [1, 1])], [3, 2, 2], record_option=TQ_RECORD_FREQS_POSITIONS)
    for boost, want in ((1.0, 0.84163445), (2.0, 1.6832689)):
        rows = M.search([m], make_query(TQ_OP_OR, [o], [0, 1], 3, boost=boost), [0, 1])
        assert _near({d: s for s, _, d in rows}[0], want)


def test_pinned_intersection():
    # src/query/boolean_query/mod.rs:262-291: +a +b over "a b c", "a c", "b c", "a b c d", "d" -> 0.977973, 0.84699446
    o, m = _pair([([0, 1, 3], [1, 1, 1]), ([0, 2, 3], [1, 1, 1])], [3, 2, 2, 4, 1], record_option=TQ_RECORD_FREQS_POSITIONS)
    rows = M.search([m], make_query(TQ_OP_AND, [o], [0, 1], 10), [0, 1])
    assert [d for _, _, d in rows] == [0, 3]
    assert _near(rows[0][0], 0.977973) and _near(rows[1][0], 0.84699446)


def test_pinned_term_scores():
    # src/collector/top_score_collector.rs:838-857 ("droopy tax") and src/query/term_query/mod.rs:21-44 (Basic field) / :82-129
    o, m = _pair([([1, 2], [1, 1]), ([0, 1], [1, 1])], [4, 6, 3], record_option=TQ_RECORD_FREQS_POSITIONS)
    rows = M.search([m], make_query(TQ_OP_OR, [o], [0, 1], 4), [0, 1])
    assert [d for _, _, d in rows] == [1, 2, 0]
    assert all(_near(s, w) for (s, _, _), w in zip(rows, [0.81221175, 0.5376842, 0.48527452]))
    o, m = _pair([([0], None)], [1], record_option=TQ_RECORD_BASIC)
    assert _near(M.search([m], make_query(TQ_OP_TERM, [o], [0], 1), [0])[0][0], 0.28768212)
    o, m = _pair([([0], [2]), ([0, 1], [1, 1])], [18, 2], record_option=TQ_RECORD_FREQS_POSITIONS)
    assert _near(M.search([m], make_query(TQ_OP_TERM, [o], [0], 2), [0])[0][0], 0.77802235)


# ---- model == oracle where both must agree ---------------------------------------------------------------------------
def _random_pairs(rng, n_segments, n_terms, deletes=False, max_doc_range=(300, 20_000), dens=(0.5, 0.2, 0.05, 0.01, 0.002)):
    out = []
    for i in range(n_segments):
        max_doc = int(rng.integers(*max_doc_range))
        lengths = np.clip(np.round(np.exp(rng.normal(np.log(40), 0.7, size=max_doc))), 1, 4096).astype(np.uint32)
        lists = []
        for t in range(n_terms):
            docs = np.nonzero(rng.random(max_doc) < dens[t % len(dens)] * float(rng.uniform(0.5, 1.5)))[0].astype(np.uint32)
            lists.append((docs, np.minimum(rng.geometric(0.6, size=len(docs)), 10).astype(np.uint32)))
        alive = np.packbits(rng.random(max_doc) > 0.2, bitorder="little") if deletes else None
        out.append(_pair(lists, lengths, segment_ord=10 + i, alive=alive))
    return [o for o, _ in out], [m for _, m in out]


@pytest.mark.parametrize("n_segments", [1, 3])
def test_term_and_or_match_the_oracle(n_segments):
    rng = np.random.default_rng(20 + n_segments)
    osegs, msegs = _random_pairs(rng, n_segments, 6, deletes=n_segments == 3)
    shapes = [(TQ_OP_TERM, [t]) for t in range(5)] + [(TQ_OP_AND, c) for c in ([0, 1], [4, 3], [0, 1, 2], [0, 1, 2, 3, 4])]
    shapes += [(TQ_OP_OR, c) for c in ([0, 1], [4, 3], [0, 1, 2], [0, 1, 2, 3, 4, 5])]
    queries, terms = [], []
    for op, c in shapes:
        for k in (1, 10, 1000):
            queries.append(make_query(op, osegs, c, k))
            terms.append(c)
    _assert_model_is_oracle(osegs, msegs, queries, terms)
    # the oracle's restated Block-WAND paths too, where the reference's order is not data dependent (unions: block_wand_union.rs:205-208)
    not_or = [i for i, q in enumerate(queries) if q["op"] != TQ_OP_OR]
    _assert_model_is_oracle(osegs, msegs, [queries[i] for i in not_or], [terms[i] for i in not_or], modes=(1,))


def test_mixed_boolean_shapes_match_the_oracle():
    rng = np.random.default_rng(31)
    osegs, msegs = _random_pairs(rng, 3, 6, deletes=True)
    osegs[1].terms[3] = (0, 0, 0)  # absent from one segment: an EmptyScorer there
    osegs[2].terms[1] = (0, 0, 0)
    queries, terms = [], []
    for c, occ, grp, msm in BOOL_SHAPES:
        for k in (5, 1000):
            queries.append(bool_query(make_query(TQ_OP_OR, osegs, c, k), occ, grp, msm))
            terms.append(c)
    _assert_model_is_oracle(osegs, msegs, queries, terms)
    ix = O.OracleIndex()
    for s in osegs:
        s.register(ix)
    counts = ix.count_batch(QueryBatch(queries))
    assert [M.count(msegs, q, t) for q, t in zip(queries, terms)] == list(counts)


def test_thresholds_absent_terms_and_deletes_match_the_oracle():
    rng = np.random.default_rng(41)
    osegs, msegs = _random_pairs(rng, 3, 4, deletes=True)
    osegs[1].terms[3] = (0, 0, 0)
    osegs[2].terms[2] = (0, 0, 0)
    queries, terms = [], []
    for op, c in [(TQ_OP_TERM, [3]), (TQ_OP_AND, [0, 3]), (TQ_OP_AND, [2, 1]), (TQ_OP_OR, [0, 2, 3])]:
        for thr in (None, 0.0, -1.0, 1.5, 1e9):
            q = make_query(op, osegs, c, 50)
            if thr is not None:
                q["threshold"] = thr
            queries.append(q)
            terms.append(c)
    _assert_model_is_oracle(osegs, msegs, queries, terms)


# ---- four and more MUST scorers: the two summation orders of an intersection ---------------------------------------------
@pytest.fixture(scope="module")
def dense():
    """One 20k-doc segment of nine dense terms (term 4 sparse): four-scorer intersections have many matches."""
    rng = np.random.default_rng(1)
    max_doc = 20_000
    lengths = np.clip(np.round(np.exp(rng.normal(np.log(40), 0.7, size=max_doc))), 1, 4096).astype(np.uint32)
    lists = []
    for p in (0.9, 0.8, 0.7, 0.6, 0.05, 0.5, 0.45, 0.4, 0.35):
        docs = np.nonzero(rng.random(max_doc) < p)[0].astype(np.uint32)
        lists.append((docs, np.minimum(rng.geometric(0.5, size=len(docs)), 40).astype(np.uint32)))
    return lists, lengths


def _order_case(segs, q, terms):
    """model == oracle bit for bit, and the other summation order changes a returned score (the case is not vacuous)."""
    osegs, msegs = segs
    got = hits(_oracle(osegs, [q]))
    want = M.search(msegs, q, terms)
    assert got == want, f"oracle {got[:4]} != model {want[:4]}"
    if q["op"] == TQ_OP_AND:  # the oracle's reference-faithful path: block_wand_intersection or the Intersection
        assert hits(_oracle(osegs, [q], mode=1)) == want
    io = M.search(msegs, q, terms, intersection_order=True)
    seq = M.search(msegs, q, terms, intersection_order=False)
    assert [s for s, _, _ in io] != [s for s, _, _ in seq], "both summation orders give the same rows"
    return want


def _one(dense, record_option=TQ_RECORD_FREQS):
    lists, lengths = dense
    if record_option == TQ_RECORD_BASIC:
        lists = [(d, None) for d, _ in lists]
    o, m = _pair(lists, lengths, record_option=record_option)
    return [o], [m]


@pytest.mark.parametrize("n", [4, 5, 8])
def test_and_of_terms_reading_freqs_sums_one_after_another(dense, n):
    segs = _one(dense)
    terms = [0, 1, 2, 3, 5, 6, 7, 8][:n]
    q = make_query(TQ_OP_AND, segs[0], terms, 1000)
    assert _order_case(segs, q, terms) == M.search(segs[1], q, terms, intersection_order=False)


@pytest.mark.parametrize("n", [4, 5, 8])
def test_and_with_a_term_ignoring_freqs_sums_like_intersection(dense, n):
    segs = _one(dense)
    terms = [0, 1, 2, 3, 5, 6, 7, 8][:n]
    q = make_query(TQ_OP_AND, segs[0], terms, 1000)
    q["term_flags"] = [0] * (n - 1) + [1]
    assert _order_case(segs, q, terms) == M.search(segs[1], q, terms, intersection_order=True)


@pytest.mark.parametrize("n", [4, 5])
def test_and_on_a_basic_field_sums_like_intersection(dense, n):
    rng = np.random.default_rng(5)
    lists, lengths = dense
    # tf = 1 everywhere: vary the weights so that the scores are not all alike
    segs = _one(dense, TQ_RECORD_BASIC)
    terms = [0, 1, 2, 3, 5][:n]
    q = make_query(TQ_OP_AND, segs[0], terms, 1000)
    q["weights"] = [float(np.float32(w * rng.uniform(0.3, 3.0))) for w in q["weights"]]
    assert _order_case(segs, q, terms) == M.search(segs[1], q, terms, intersection_order=True)


_ORDER_BOOL = [  # (terms, occurs, groups, msm, Intersection order?)
    ([0, 1, 2, 3, 4], [1, 1, 1, 1, 2], None, 0, True),                          # +a +b +c +d -e
    ([0, 1, 2, 3, 5], [1, 1, 1, 1, 0], None, 0, True),                          # +a +b +c +d f (RequiredOptionalScorer)
    ([0, 5, 1, 6, 2, 7, 3, 8], [1] * 8, [0, 0, 1, 1, 2, 2, 3, 3], 0, True),     # +(a|f) +(b|g) +(c|h) +(d|i)
    ([0, 1, 2, 3, 5], [1, 1, 1, 0, 0], None, 2, False),                         # +a +b +c, both of d f: five MUST TermScorers
    ([0, 1, 2, 3, 5, 4], [1, 1, 1, 0, 0, 2], None, 2, True),                    # ... and -e
    ([0, 1, 2, 3, 5], [1, 1, 1, 1, 1], None, 0, False),                         # five MUST terms: block_wand_intersection
]


@pytest.mark.parametrize("case", range(len(_ORDER_BOOL)))
def test_boolean_with_four_or_more_must_scorers(dense, case):
    terms, occ, grp, msm, io = _ORDER_BOOL[case]
    segs = _one(dense)
    q = bool_query(make_query(TQ_OP_OR, segs[0], terms, 1000), occ, grp, msm)
    assert _order_case(segs, q, terms) == M.search(segs[1], q, terms, intersection_order=io)


def test_must_not_without_postings_in_one_segment(dense):
    """+a +b +c +d -e over three segments; e has no postings in the middle one.  There the Exclude is dropped and the four
    TermScorers reach block_wand_intersection (sequential); the other two segments sum as Intersection::score does."""
    lists, lengths = dense
    pairs = [_pair(lists, lengths, segment_ord=so) for so in (3, 4, 5)]
    osegs, msegs = [o for o, _ in pairs], [m for _, m in pairs]
    osegs[1].terms[4] = (0, 0, 0)
    terms = [0, 1, 2, 3, 4]
    q = bool_query(make_query(TQ_OP_OR, osegs, terms, 1024), [1, 1, 1, 1, 2])
    rows = _order_case((osegs, msegs), q, terms)
    # neither order alone gives these rows: the segments follow different rules
    assert rows != M.search(msegs, q, terms, intersection_order=True)
    assert rows != M.search(msegs, q, terms, intersection_order=False)


# ---- random mixed boolean shapes: every branch of complex_scorer ---------------------------------------------------------
def _random_bool_case(seed, n_queries):
    rng = np.random.default_rng(seed)
    osegs, msegs = _random_pairs(rng, 3, 8, deletes=True)
    osegs[0].terms[6] = (0, 0, 0)  # terms without postings in some segments: EmptyScorers there
    osegs[1].terms[3] = (0, 0, 0)
    osegs[1].terms[7] = (0, 0, 0)
    osegs[2].terms[1] = (0, 0, 0)
    shapes = random_bool_shapes(rng, n_queries, 8)
    return osegs, msegs, shapes, [bool_shape_query(osegs, sh) for sh in shapes]


def test_random_boolean_shapes_match_the_oracle():
    """Several hundred seeded random TQ_OP_BOOL shapes (repeated terms, msm 0..n+1, boosts 0 / -1.5 / 1e4, TQ_TERM_IGNORE_FREQ,
    32 clauses) over three segments with deletes and absent terms: model == oracle for the rows and for Count, and together
    the shapes take every branch of complex_scorer."""
    osegs, msegs, shapes, queries = _random_bool_case(4242, 360)
    seen = set()
    for q in queries:
        for s in osegs:
            seen |= bool_branches(q, s.segment_ord)
    assert BOOL_BRANCHES <= seen, BOOL_BRANCHES - seen
    _assert_model_is_oracle(osegs, msegs, queries, [sh["terms"] for sh in shapes])
    ix = O.OracleIndex()
    for s in osegs:
        s.register(ix)
    counts = ix.count_batch(QueryBatch(queries))
    assert [M.count(msegs, q, sh["terms"]) for q, sh in zip(queries, shapes)] == list(counts)
    assert sum(1 for c in counts if c) > len(queries) // 3  # (not a vacuous comparison)


def test_random_boolean_shapes_cover_the_generator():
    """The generator makes what its callers rely on: 1-12 and 32 clauses, MUST groups of 1-4, msm up to n_should + 1, each
    repeated-term pattern, every boost and k."""
    shapes = random_bool_shapes(np.random.default_rng(4242), 360, 8)
    assert {len(s["terms"]) for s in shapes} == set(range(1, 13)) | {32}
    sizes = set()
    pats = set()
    for s in shapes:
        groups = {}
        for c, (o, g) in enumerate(zip(s["occurs"], s["groups"])):
            if o == TQ_OCCUR_MUST:
                groups.setdefault(g, []).append(s["terms"][c])
        sizes |= {len(m) for m in groups.values()}
        if any(len(set(m)) < len(m) for m in groups.values()):
            pats.add("twice in one group")
        firsts = [set(m) for m in groups.values()]
        if any(a & b for i, a in enumerate(firsts) for b in firsts[i + 1:]):
            pats.add("in two groups")
        should = {t for t, o in zip(s["terms"], s["occurs"]) if o == TQ_OCCUR_SHOULD}
        if should & {t for t, o in zip(s["terms"], s["occurs"]) if o == TQ_OCCUR_MUST_NOT}:
            pats.add("should and must_not")
    assert sizes == {1, 2, 3, 4}
    assert pats == {"twice in one group", "in two groups", "should and must_not"}
    assert any(s["msm"] == s["occurs"].count(TQ_OCCUR_SHOULD) + 1 for s in shapes)
    assert {b for s in shapes for b in s["boosts"]} == set(BOOL_BOOSTS)
    assert {s["k"] for s in shapes} == set(BOOL_KS)
    assert any(f for s in shapes for f in s["flags"])


# ---- phrase queries ------------------------------------------------------------------------------------------------------
def _phrase_segs(*texts_per_seg):
    from tests.test_gpu_phrase import PosSegment
    return [PosSegment(t, writer_cls=O.FieldWriter) for t in texts_per_seg]


def _phrase_rows(segs, phrase, k=10, offsets=None, **extra):
    """(model rows, oracle rows) of one phrase query over `segs`; offsets[c] = the phrase offset of clause c."""
    from tests.test_gpu_phrase import phrase_query
    q, _, _, _ = phrase_query(segs, phrase, k, offsets=offsets)
    q.update(extra)
    vocab = sorted({t for s in segs for t in s.vocab} | set(phrase))
    want = M.search([s.model(vocab) for s in segs], q, [vocab.index(t) for t in phrase])
    ix = O.OracleIndex()
    for s in segs:
        s.register(ix)
    return want, hits(ix.search_batch(QueryBatch([q]), mode=0))


def test_phrase_model_reproduces_the_reference_phrase_tests():
    """phrase_query/mod.rs:41-91,163-169 (as tests/test_phrase_goldens.py states them): doc sets and the two pinned scores."""
    texts = ["b b b d c g c", "a b b d c g c", "a b a b c", "c a b a d ga a", "a b c"]
    segs = _phrase_segs(texts)
    for phrase, docs in ((["a", "b"], [1, 2, 3, 4]), (["a", "b", "c"], [2, 4]), (["b", "b"], [0, 1]), (["g", "a"], [])):
        want, got = _phrase_rows(segs, phrase)
        assert sorted(d for _, _, d in want) == docs and got == want, phrase
    want, got = _phrase_rows(_phrase_segs(["a b b d c g c", "a b a b c"]), ["a", "b"])
    assert sorted(d for _, _, d in want) == [0, 1] and got == want
    want, got = _phrase_rows(_phrase_segs(["a b c", "a b c a b"]), ["a", "b"])
    by_doc = {d: s for s, _, d in want}
    assert _near(by_doc[0], 0.40618482) and _near(by_doc[1], 0.46844664) and got == want


def test_phrase_model_slop_doc_sets():
    """The doc sets test_two_term_phrases_with_slop asserts on the device."""
    segs = _phrase_segs(["a b c d", "a c b", "b a", "a x x b", "a x x x b", "b x a x b a", "a a a b b b", "c c", "b"])
    docs = {}
    for slop in (1, 2, 3):
        want, got = _phrase_rows(segs, ["a", "b"], slop=slop)
        assert got == want, slop
        docs[slop] = sorted(d for _, _, d in want)
    assert docs[1] == [0, 1, 5, 6] and docs[2] == [0, 1, 2, 3, 5, 6] and {3, 4} <= set(docs[3])


@pytest.mark.parametrize("left,right,slop,expected", [
    # phrase_scorer.rs test_slop: the matched right positions
    ([1], [2], 1, [2]), ([1], [3], 1, []), ([1], [3], 2, [3]), ([], [2], 100000, []), ([5, 7, 11], [1, 5, 10, 12], 1, [5, 10]),
    ([1, 5, 6, 9, 10, 12], [6, 8, 9, 12], 1, [6, 8, 9, 12]), ([1, 5, 6, 9, 10, 12], [6, 8, 9, 12], 10, [6, 8, 9, 12]),
    ([1, 3, 5], [2, 4, 6], 1, [2, 4, 6]),
    # test_merge_slop
    ([1, 2], [1], 1, [1]), ([3], [4], 2, [4]), ([1, 5, 6, 9, 10, 12], [6, 8, 9, 12], 10, [6, 8, 9, 12]),
])
def test_phrase_model_slop_matches_the_reference_cases(left, right, slop, expected):
    assert M.slop_matches(left, right, slop) == expected


def test_phrase_clauses_are_taken_in_offset_order():
    """One doc "a a b b", the phrase a@0 b@1 with slop 1, clauses passed as (b, offset 1), (a, offset 0).  Both terms have doc_freq
    1, so the offset order decides `left`: shifted a = [1, 2], b = [2, 3]; left = a counts 1 (left = b would count 2).  The oracle
    agrees with the model in both clause orders."""
    segs = _phrase_segs(["a a b b"])
    one, got = _phrase_rows(segs, ["a", "b"], offsets=[0, 1], slop=1)
    assert got == one
    swapped, got = _phrase_rows(segs, ["b", "a"], offsets=[1, 0], slop=1)
    assert swapped == one and got == one
    assert len(one) == 1 and one == _phrase_rows(segs, ["a", "b"])[0]  # the score of phrase count 1: "a b" without slop


def test_random_phrases_match_the_oracle():
    """Random texts in three segments (one with deletes): phrases of 2 to 8 terms, gaps / repeated / out-of-order offsets, slop,
    thresholds: model == oracle, and the model is not vacuous."""
    rng = np.random.default_rng(808)
    vocab = ["w0", "w1", "w2", "w3", "w4"]
    p = [0.4, 0.25, 0.15, 0.12, 0.08]
    texts = [[" ".join(rng.choice(vocab, size=int(rng.integers(2, 40)), p=p)) for _ in range(n)] for n in (300, 500, 200)]
    segs = _phrase_segs(*texts)
    alive = np.packbits(rng.random(segs[1].n_docs) > 0.3, bitorder="little")
    from tests.test_gpu_phrase import PosSegment
    segs[1] = PosSegment.from_positions(segs[1].positions, segs[1].lengths, alive=alive, writer_cls=O.FieldWriter)
    n_hits = 0
    cases = [(["w0", "w1"], None, 0), (["w1", "w0"], [1, 0], 2), (["w0", "w2", "w1"], [0, 2, 5], 0), (["w0", "w1", "w0"], [3, 4, 5], 0),
             (["w0", "w1", "w1"], [0, 1, 1], 0), (["w0", "w1", "w2"], [2, 0, 1], 0), (["w0", "w0"], [0, 0], 1), (["w0"] * 8, None, 0),
             (["w0", "w1", "w0", "w0", "w2", "w0"], None, 0), (["w3", "w4"], [1, 0], 1), (["w3", "w4"], [1, 0], 3)]
    for phrase, offsets, slop in cases:
        for extra in ({}, {"threshold": 1.0}):
            want, got = _phrase_rows(segs, phrase, k=50, offsets=offsets, slop=slop, **extra)
            assert got == want, (phrase, offsets, slop, extra)
            n_hits += len(want)
    assert n_hits > 200


# ---- merge_fruits: the cross-segment and cross-shard merge ----------------------------------------------------------------
def test_merge_fruits_of_segments_and_doc_range_parts_is_the_whole_search():
    """The rows of each segment alone, and of doc-range parts of the segments (docs outside a part count as deleted), merged by
    merge_fruits are the rows of one search over every segment: for terms, AND, OR and boolean shapes, k from 1 to 1000."""
    rng = np.random.default_rng(77)
    osegs, msegs = _random_pairs(rng, 3, 6, deletes=True, max_doc_range=(2000, 6000))
    queries, terms = [], []
    for op, c in [(TQ_OP_TERM, [1]), (TQ_OP_AND, [0, 2]), (TQ_OP_OR, [0, 1, 2, 3, 4, 5]), (TQ_OP_OR, [3, 4])]:
        for k in (1, 10, 1000):
            queries.append(make_query(op, osegs, c, k))
            terms.append(c)
    for c, occ, grp, msm in BOOL_SHAPES[:6]:
        queries.append(bool_query(make_query(TQ_OP_OR, osegs, c, 100), occ, grp, msm))
        terms.append(c)
    n_rows = 0
    for q, t in zip(queries, terms):
        want = M.search(msegs, q, t)
        n_rows += len(want)
        assert M.merge_fruits([M.search([s], q, t) for s in msegs], q["k"]) == want
        parts = []
        for s in msegs:
            cuts = [0, 1, s.max_doc // 3, s.max_doc // 3, s.max_doc - 7, s.max_doc]
            parts += [M.search([s], q, t, doc_ranges={s.segment_ord: (lo, hi)}) for lo, hi in zip(cuts[:-1], cuts[1:])]
        assert M.merge_fruits(parts, q["k"]) == want
        assert M.merge_fruits(parts[::-1], q["k"]) == want  # (the order of the lists does not matter)
    assert n_rows > 2000


def test_signed_zero_scores_tie_and_are_ordered_by_doc():
    """An OR of a +0.0-weight clause and a -0.0-weight clause: every score is +-0.0, and -0.0 == +0.0 as under partial_cmp, so the
    rows come in (segment, doc) order whichever zero a doc has -- the -0.0 clause's lower docs first.  merge_fruits agrees."""
    lists = [(np.arange(10, 20), np.ones(10)), (np.arange(0, 10), np.ones(10))]
    o0, m0 = _pair(lists, np.full(20, 5), segment_ord=0)
    o1, m1 = _pair(lists, np.full(20, 5), segment_ord=1)
    q = make_query(TQ_OP_OR, [o0, o1], [0, 1], 100)
    q["weights"] = [0.0, -0.0]
    rows = M.search([m0, m1], q, [0, 1])
    assert [(so, d) for _, so, d in rows] == [(so, d) for so in (0, 1) for d in range(20)]
    signs = {d: np.signbit(s) for s, so, d in rows if so == 0}
    assert all(signs[d] for d in range(10)) and not any(signs[d] for d in range(10, 20))  # (both zeros are there)
    assert M.merge_fruits([M.search([m1], q, [0, 1]), M.search([m0], q, [0, 1])], 100) == rows
    assert M.merge_fruits([[(0.0, 3, 5)], [(-0.0, 3, 4)], [(-0.0, 2, 9)], [(1e-45, 9, 9)]], 3) == [(1e-45, 9, 9), (-0.0, 2, 9), (-0.0, 3, 4)]


# ---- multi-field segments ----------------------------------------------------------------------------------------------
def test_one_field_multi_field_segment_is_the_single_field_model():
    """A segment written as a one-field multi-field segment gives the rows and counts of the plain Segment, bit for bit."""
    rng = np.random.default_rng(77)
    osegs, msegs = _random_pairs(rng, 3, 6, deletes=True)
    wrapped = [M.Segment.multi_field(m.segment_ord, {0: dict(lists=m.lists, lengths=l, basic=m.basic)}, m.max_doc, alive=o.alive)
               for o, m, l in zip(osegs, msegs, [o.fieldnorms for o in osegs])]
    queries, terms = [], []
    for op, c in [(TQ_OP_TERM, [1]), (TQ_OP_AND, [0, 1, 2, 3, 4]), (TQ_OP_OR, [0, 1, 2, 3, 4, 5])]:
        for k in (1, 10, 1000):
            queries.append(make_query(op, osegs, c, k))
            terms.append(c)
    for c, occ, grp, msm in BOOL_SHAPES:
        queries.append(bool_query(make_query(TQ_OP_OR, osegs, c, 1000), occ, grp, msm))
        terms.append(c)
    for q, t in zip(queries, terms):
        a, b = M.search(msegs, q, t), M.search(wrapped, q, t)
        assert [(np.float32(s).view(np.uint32), g, d) for s, g, d in a] == [(np.float32(s).view(np.uint32), g, d) for s, g, d in b]
        assert M.count(msegs, q, t) == M.count(wrapped, q, t)


@pytest.fixture(scope="module")
def multi_field_index():
    from tests.multi_field import Index
    return Index(sizes=(30_000, 7_001, 5_000))


def test_multi_field_model_is_the_oracle(multi_field_index):
    """Clauses over several fields of one segment ordinal (each field its own lists, fieldnorms and record option, one alive
    bitset): the model's rows and counts equal the oracle's, which looks up every clause's (segment, field)."""
    from tests.multi_field import battery
    ix = multi_field_index
    oi = ix.register(O.OracleIndex())
    qts = battery(ix, phrase=False)
    assert max(len(q["weights"]) for q, _ in qts) == 32
    res = oi.search_batch(QueryBatch([q for q, _ in qts]), mode=0)
    for i, (q, t) in enumerate(qts):
        assert hits(res, i) == M.search(ix.models(), q, t), (i, q["op"], t)
    counts = oi.count_batch(QueryBatch([q for q, _ in qts]))
    assert list(counts) == [M.count(ix.models(), q, t) for q, t in qts]
    # the fields do sum on one doc: some OR row holds clauses of two fields
    q, t = next(x for x in qts if x[0]["op"] == TQ_OP_OR and x[0]["k"] == 1024)
    assert len({ts[2] for ts in q["term_segs"]}) >= 2
