"""The score model on a compacted doc space (tests/score_model.py Compacted) against the model on the whole segment, and the BM25
scalars at index sizes of 2^32 docs and more.  The compacted model is what the GPU tests of segments with up to 2^31 - 2 docs
compare against (tests/test_gpu_high_doc_ids.py), so it has to equal the plain model on every shape it knows.  Runs on CPU."""
import numpy as np
import pytest

import tantivy_b200 as T
from oracle import tq_oracle as O
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_OR, TQ_OP_PHRASE, TQ_OP_TERM, TQ_TERM_IGNORE_FREQ
from tests import score_model as M
from tests.helpers import _FN_TABLE, fieldnorm_ids, random_bool_shapes, shape_query

N_TERMS = 6
DENS = (0.4, 0.2, 0.1, 0.05, 0.3, 0.01)


def _segment(rng, so, n, norms, deletes):
    """Lists over the first 80% of n docs (the rest is listed nowhere), positions for every posting (tf = their number); the
    plain model's Segment and the Compacted one of the same content."""
    lengths = rng.integers(1, 3000, size=n).astype(np.uint32) if norms else None
    lists, positions = [], []
    for t in range(N_TERMS):
        keep = rng.random(n) < DENS[t]
        keep[int(n * 0.8):] = False
        docs = np.nonzero(keep)[0].astype(np.uint32)
        pos = {int(d): sorted(set(rng.integers(0, 12, size=int(rng.integers(1, 5))).tolist())) for d in docs}
        lists.append((docs, np.array([len(pos[int(d)]) for d in docs], np.uint32)))
        positions.append(pos)
    alive = np.packbits(rng.random(n) > 0.25, bitorder="little") if deletes else None
    full = M.Segment(so, lists, lengths, alive=alive, max_doc=n, positions=positions)
    fn = None if lengths is None else fieldnorm_ids(lengths)
    comp = M.Compacted(so, lists, n, fn_ids=fn, alive=alive, positions=positions)
    return full, comp


def _query(op, segs, terms, k, **extra):
    n_docs = sum(s.max_doc for s in segs)
    weights, term_segs = [], []
    for c, t in enumerate(terms):
        df = sum(len(s.lists[t][0]) for s in segs)
        weights.append(O.bm25_weight(df, n_docs))
        term_segs += [(c, s.segment_ord, 0, len(s.lists[t][0]), 0, 0) for s in segs if len(s.lists[t][0])]
    q = dict(op=op, k=k, weights=weights, avg_fieldnorm=[np.float32(41.5)] * len(terms), term_segs=term_segs)
    q.update(extra)
    return q, list(terms)


def _queries(rng, segs):
    qs = [_query(TQ_OP_TERM, segs, [t], k) for t in range(N_TERMS) for k in (1, 10, 1000)]
    for terms in ([0, 1], [1, 0, 2], [0, 1, 4, 2], [0, 4, 1, 2, 3]):
        qs += [_query(TQ_OP_AND, segs, terms, k) for k in (3, 1000)]
        qs.append(_query(TQ_OP_AND, segs, terms, 1000, term_flags=[0] * (len(terms) - 1) + [TQ_TERM_IGNORE_FREQ]))
    qs += [_query(TQ_OP_OR, segs, terms, k) for terms in ([0, 1], [2, 3, 5], list(range(N_TERMS))) for k in (5, 1000)]
    for sh in random_bool_shapes(rng, 16, N_TERMS, n_wide=1):
        q, _ = _query(TQ_OP_OR, segs, sh["terms"], sh["k"])
        qs.append((shape_query(q, sh), sh["terms"]))
    for terms, offsets, slop in (([0, 1], [0, 1], 0), ([2, 0, 1], [2, 0, 1], 0), ([0, 4], [0, 2], 0), ([1, 0], [1, 0], 1),
                                 ([0, 1], [0, 1], 2)):
        q, _ = _query(TQ_OP_PHRASE, segs, terms, 1000, term_offset=offsets, slop=slop)
        q["weights"] = [q["weights"][0]] * len(terms)
        qs.append((q, terms))
    return qs


def _thresholded(q, rows):
    """q with its initial threshold at the score of the middle row (ties at the cut included)."""
    return dict(q, threshold=float(rows[len(rows) // 2][0])) if rows else q


def _cuts(comp, rng):
    """Doc ranges of one segment: cuts on listed docs, between listed docs (on unlisted ones) and in the unlisted tail."""
    docs = comp.docs
    listed = [int(docs[i]) for i in rng.choice(len(docs), size=4, replace=False)]
    unlisted = np.setdiff1d(np.arange(comp.max_doc, dtype=np.uint32), docs)
    free = [int(unlisted[i]) for i in rng.choice(len(unlisted), size=4, replace=False)]
    pts = sorted(set(listed + free))
    out = [(0, comp.max_doc), (pts[0], pts[-1]), (pts[1], pts[1]), (pts[2], comp.max_doc), (0, pts[3])]
    out += [(a, b) for a, b in zip(pts[:-1], pts[1:])]
    return out, listed, free


def test_compacted_model_equals_the_model_on_the_whole_segment():
    rng = np.random.default_rng(0xC0DE)
    pairs = [_segment(rng, 0, 3000, True, True), _segment(rng, 1, 2000, False, False), _segment(rng, 2, 1500, True, False)]
    full = [f for f, _ in pairs]
    comp = [c for _, c in pairs]
    for f, c in pairs:  # not vacuous: docs outside every list, a real renumbering
        assert 0 < len(c.docs) < f.max_doc and int(c.docs[-1]) < f.max_doc * 0.8
    queries = _queries(rng, full)
    ranges = {}
    for c in comp:
        ranges[c.seg.segment_ord], listed, free = _cuts(c, rng)
        assert any(lo in listed or hi in listed for lo, hi in ranges[c.seg.segment_ord])
        assert any(lo in free or hi in free for lo, hi in ranges[c.seg.segment_ord])
    n_rows = 0
    for q, terms in queries:
        want = M.search(full, q, terms)
        assert M.search_compacted(comp, q, terms) == want, (q["op"], terms, q["k"])
        assert M.count_compacted(comp, q, terms) == M.count(full, q, terms), (q["op"], terms)
        qt = _thresholded(q, want)
        assert M.search_compacted(comp, qt, terms) == M.search(full, qt, terms), (q["op"], terms, "threshold")
        if q["op"] == TQ_OP_AND:
            for io in (False, True):
                assert M.search_compacted(comp, q, terms, intersection_order=io) == M.search(full, q, terms, intersection_order=io)
        for i in range(len(ranges[0])):
            dr = {so: r[i % len(r)] for so, r in ranges.items()}
            assert M.search_compacted(comp, q, terms, doc_ranges=dr) == M.search(full, q, terms, doc_ranges=dr), (q["op"], terms, dr)
            assert M.count_compacted(comp, q, terms, doc_ranges=dr) == M.count(full, q, terms, doc_ranges=dr), (q["op"], terms, dr)
        n_rows += len(want)
    ops = {q["op"] for q, _ in queries}
    assert n_rows > 5000 and len(ops) == 5
    assert any(q["op"] == TQ_OP_PHRASE and M.search(full, q, t) for q, t in queries)


# ---- BM25 scalars at doc_count >= 2^32 ---------------------------------------------------------------------------------
def _idf_f32(doc_freq, doc_count):
    """bm25.rs idf in f32: ln(1 + (doc_count - doc_freq + 0.5) / (doc_freq + 0.5)), each u64 cast to f32 once; the logarithm
    correctly rounded (the library's logf may be one ulp off it)."""
    f32 = np.float32
    x = (f32(doc_count - doc_freq) + f32(0.5)) / (f32(doc_freq) + f32(0.5))
    return f32(np.log(np.float64(f32(1) + x)))


@pytest.mark.parametrize("doc_count", [2 ** 32, 2 ** 32 + 1, 2 * (2 ** 31 - 2) + 50_000, 3 * (2 ** 31 - 2), 2 ** 40 + 7])
def test_idf_and_weight_beyond_two_to_the_32_docs(doc_count):
    for doc_freq in (1, 2, 40_000, 2_500_000, 2 ** 31 - 2, doc_count // 2, doc_count - 1):
        want = _idf_f32(doc_freq, doc_count)
        exact = np.log1p((doc_count - doc_freq + 0.5) / (doc_freq + 0.5))
        for name, idf in (("library", T.bm25_idf(doc_freq, doc_count)), ("oracle", O.bm25_idf(doc_freq, doc_count))):
            idf = np.float32(idf)
            ulps = abs(int(idf.view(np.int32)) - int(want.view(np.int32)))
            assert ulps <= 1, (name, doc_freq, doc_count, idf, want)
            assert abs(float(idf) - exact) <= 4 * M.EPS * (1 + exact), (name, doc_freq, doc_count, idf, exact)
            for boost in (1.0, 2.5):
                w = np.float32(idf * np.float32(2.2))
                if boost != 1.0:
                    w = np.float32(w * np.float32(boost))
                got = np.float32(T.bm25_weight(doc_freq, doc_count, boost) if name == "library" else O.bm25_weight(doc_freq, doc_count, boost))
                assert got == w, (name, doc_freq, doc_count, boost, got, w)
    # the u64 doc count is not cut to 32 bits: 2^32 + n docs is not n docs
    assert np.float32(T.bm25_idf(1, 2 ** 32 + 10)) > np.float32(T.bm25_idf(1, 10)) + 10
