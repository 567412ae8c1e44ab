"""Shared helpers of the test-suite (oracle-side segment construction, like the reference's
test-only constructors SegmentPostings::create_from_docs_and_tfs / TermScorer::create_for_test,
src/postings/segment_postings.rs:94, src/query/term_query/term_scorer.rs:33)."""
import json
import os

import numpy as np

from oracle import tq_oracle as O
from tantivy_b200._abi import (TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT, TQ_OCCUR_SHOULD, TQ_OP_AND, TQ_OP_BOOL, TQ_OP_OR, TQ_OP_TERM,
                               TQ_RECORD_FREQS, TQ_TERM_IGNORE_FREQ, QueryBatch)

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_fixtures.json")))


def f32(x):
    return np.float32(x)


_FN_TABLE = np.array(GOLDEN["field_norms_table"], dtype=np.uint64)


def fieldnorm_ids(fieldnorms):
    """fieldnorm_to_id for an array: index of the last table entry <= fieldnorm (code.rs:7-11)."""
    f = np.asarray(fieldnorms, dtype=np.uint64)
    return (np.searchsorted(_FN_TABLE, f, side="right") - 1).astype(np.uint8)


class OracleSegment:
    """One segment, one field, built from explicit posting lists (docs, tfs) and doc lengths."""

    def __init__(self, posting_lists, fieldnorms, record_option=TQ_RECORD_FREQS, segment_ord=0, field=0,
                 writer_cls=None, alive=None, max_doc=None):
        if fieldnorms is None:  # field without fieldnorms: constant fieldnorm 1 (term_weight.rs:218)
            self.fieldnorms, self.fn_ids = None, None
            self.max_doc = max_doc
            self.total_num_tokens = max_doc
        else:
            self.fieldnorms = np.asarray(fieldnorms, dtype=np.uint32)
            self.max_doc = len(self.fieldnorms)
            self.fn_ids = fieldnorm_ids(self.fieldnorms)
            self.total_num_tokens = int(self.fieldnorms.astype(np.uint64).sum())
        self.record_option = record_option
        self.segment_ord, self.field = segment_ord, field
        writer_cls = writer_cls or O.FieldWriter
        w = writer_cls(record_option, self.total_num_tokens, self.fn_ids, self.max_doc)
        self.terms = []
        for docs, tfs in posting_lists:
            s, e = w.add_term(docs, tfs)
            self.terms.append((len(docs), s, e))
        self.body = w.body()
        self.alive = alive

    def term_seg(self, term, clause=0):
        df, s, e = self.terms[term]
        return (clause, self.segment_ord, self.field, df, s, e)

    def register(self, index):
        index.segment_register(self.segment_ord, self.field, self.max_doc, self.record_option, self.body, self.fn_ids, self.alive)


def searcher_stats(segments):
    """Bm25StatisticsProvider for Searcher (src/query/bm25.rs:27-50): N = sum max_doc,
    avg = total_num_tokens / N as f32."""
    n_docs = sum(s.max_doc for s in segments)
    tokens = sum(s.total_num_tokens for s in segments)
    return n_docs, f32(f32(tokens) / f32(n_docs))


def make_query(op, segments, terms, k, boost=1.0):
    """terms = list of term ordinals (same ordinal in every segment); boost = one value, or one per clause."""
    n_docs, avg = searcher_stats(segments)
    weights, term_segs = [], []
    for clause, t in enumerate(terms):
        df = sum(s.terms[t][0] for s in segments)
        weights.append(O.bm25_weight(df, n_docs, boost[clause] if isinstance(boost, (list, tuple)) else boost))
        for s in segments:
            if s.terms[t][0] > 0:
                term_segs.append(s.term_seg(t, clause))
    return dict(op=op, k=k, weights=weights, avg_fieldnorm=[avg] * len(terms), term_segs=term_segs)


BOOL_SHAPES = [  # (terms, occurs, groups, msm): the shapes of benches/and_or_queries.rs:142-155 and of boolean_query/mod.rs
    ([2, 1, 3], [1, 1, 1], [0, 1, 1], 0),            # +c +(b OR d)
    ([0, 2, 5], [1, 1, 1], [0, 1, 1], 0),            # +e +(c OR a)
    ([2, 1, 3, 0], [1, 1, 1, 1], [0, 0, 1, 1], 0),   # +(c OR b) +(d OR e)
    ([0, 1, 4], [1, 0, 0], None, 0),                 # +a b e   (RequiredOptionalScorer)
    ([1, 2, 0], [0, 0, 2], None, 0),                 # b c -a
    ([3, 0, 1], [1, 2, 2], None, 0),                 # +d -a -b (Exclude with two scorers)
    ([1, 2, 3, 4], [1, 1, 0, 2], [7, 7, 9, 9], 0),   # +(b OR c) d -e
    ([0, 1, 2, 3], [1, 0, 0, 0], None, 2),           # +a and at least two of b c d
    ([1, 2, 3, 4], [0, 0, 0, 0], None, 2),           # at least two of b c d e (Disjunction with minimum match)
    ([1, 2], [0, 0], None, 2),                       # as many as there are: they act as MUST clauses
    ([0, 1], [1, 1], None, 0),                       # plain conjunction
    ([3, 4, 5], [0, 0, 0], None, 0),                 # plain union
    ([2], [1], None, 0),                             # +c
    ([2], [2], None, 0),                             # -c alone: nothing
]


def bool_query(q, occurs, groups=None, msm=0):
    """A TQ_OP_BOOL copy of a make_query dict: an Occur per clause, optional MUST group ids, minimum_should_match."""
    q = dict(q)
    q["op"] = TQ_OP_BOOL
    q["term_occur"] = occurs
    if groups is not None:
        q["term_group"] = groups
    q["min_should_match"] = msm
    return q


BOOL_BOOSTS = (1.0, 0.0, -1.5, 1e4)
BOOL_KS = (1, 10, 128, 129, 1000)


def random_bool_shapes(rng, n, n_terms, n_wide=3):
    """n seeded random TQ_OP_BOOL shapes over the term ordinals 0..n_terms-1, each a dict of terms, occurs, groups, msm, flags,
    boosts and k.  1-12 clauses (the first n_wide shapes: 32); MUST clauses in groups of 1-4 (group ids in random order over the
    clauses); minimum_should_match 0..n_should+1; TQ_TERM_IGNORE_FREQ on about a fifth of the clauses; per clause a boost of
    BOOL_BOOSTS; k of BOOL_KS.  Every eighth shape is a conjunction of single-clause MUST groups.  Shape i repeats a term by i % 4: not at all / in two MUST groups / twice in one MUST group /
    as a SHOULD and a MUST_NOT clause."""
    shapes = []
    for i in range(n):
        n_cl = 32 if i < n_wide else int(rng.integers(1, 13))
        occ = [int(o) for o in rng.choice([TQ_OCCUR_SHOULD, TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT], size=n_cl, p=[0.45, 0.35, 0.2])]
        terms = [int(t) for t in rng.integers(0, n_terms, size=n_cl)]
        repeat = i % 4
        pure = i % 8 == 4  # every clause a MUST group of its own, all reading freqs: block_wand_intersection from four on
        if pure:
            occ = [TQ_OCCUR_MUST] * n_cl
        if repeat == 3 and n_cl >= 2:  # the same term as SHOULD and as MUST_NOT
            a, b = (int(x) for x in rng.choice(n_cl, size=2, replace=False))
            occ[a], occ[b], terms[b] = TQ_OCCUR_SHOULD, TQ_OCCUR_MUST_NOT, terms[a]
        if repeat in (1, 2) and occ.count(TQ_OCCUR_MUST) < 2 and n_cl >= 2:
            for c in rng.choice(n_cl, size=2, replace=False):
                occ[int(c)] = TQ_OCCUR_MUST
        must = [c for c in range(n_cl) if occ[c] == TQ_OCCUR_MUST]
        sizes = []
        while sum(sizes) < len(must):
            sizes.append(min(int(rng.integers(1, 5)), len(must) - sum(sizes)))
        if pure:
            sizes = [1] * len(must)
        if repeat == 1 and len(sizes) == 1 and sizes[0] >= 2:  # two groups are needed
            sizes = [1, sizes[0] - 1]
        if repeat == 2 and len(sizes) >= 2 and max(sizes) < 2:  # a group of two is needed
            sizes = [2] + sizes[2:]
        ids = rng.permutation(len(sizes)) + 1
        order = rng.permutation(must)
        groups = [0] * n_cl
        pos = 0
        for g, sz in zip(ids, sizes):
            for c in order[pos:pos + sz]:
                groups[int(c)] = int(g)
            pos += sz
        members = {}
        for c in must:
            members.setdefault(groups[c], []).append(c)
        ms = list(members.values())
        if repeat == 1 and len(ms) >= 2:  # one term in two MUST groups
            terms[ms[1][0]] = terms[ms[0][0]]
        if repeat == 2:  # one term twice in one MUST group
            big = [m for m in ms if len(m) >= 2]
            if big:
                terms[big[0][1]] = terms[big[0][0]]
        n_should = occ.count(TQ_OCCUR_SHOULD)
        shapes.append(dict(terms=terms, occurs=occ, groups=groups, msm=int(rng.integers(0, n_should + 2)),
                           flags=[TQ_TERM_IGNORE_FREQ if rng.random() < 0.2 and not pure else 0 for _ in range(n_cl)],
                           boosts=[float(b) for b in rng.choice(BOOL_BOOSTS, size=n_cl, p=[0.7, 0.1, 0.1, 0.1])],
                           k=int(rng.choice(BOOL_KS))))
    return shapes


def shape_query(q, shape):
    """The TQ_OP_BOOL query of a shape, from a make_query / SynthIndex.query dict of its terms (weights already boosted)."""
    q = bool_query(q, shape["occurs"], shape["groups"], shape["msm"])
    q["term_flags"] = list(shape["flags"])
    return q


def bool_shape_query(segments, shape):
    return shape_query(make_query(TQ_OP_OR, segments, shape["terms"], shape["k"], boost=list(shape["boosts"])), shape)


def bool_branches(q, segment_ord, basic=False):
    """Which way BooleanWeight::complex_scorer (boolean_weight.rs:236-431) goes for TQ_OP_BOOL query q on one segment, restated
    from the reference's code: a set of labels.  Clauses without postings in the segment are EmptyScorers and drop out;
    basic = the segment's field is indexed without freqs."""
    occ, grp = q["term_occur"], q.get("term_group")
    n = len(occ)
    flags = q.get("term_flags") or [0] * n
    present = {ts[0] for ts in q["term_segs"] if ts[1] == segment_ord and ts[3] > 0}
    groups = {}
    for c in range(n):
        if occ[c] == TQ_OCCUR_MUST:
            g = groups.setdefault(grp[c] if grp is not None else 256 + c, [])
            if c in present:
                g.append(c)
    if any(not g for g in groups.values()):
        return {"empty_must"}
    groups = list(groups.values())
    should = [c for c in range(n) if occ[c] == TQ_OCCUR_SHOULD and c in present]
    must_not = [c for c in range(n) if occ[c] == TQ_OCCUR_MUST_NOT and c in present]
    m = int(q.get("min_should_match", 0))
    if m > len(should):
        return {"msm_gt_n"}
    out = set()
    if m >= 2 and m == len(should):  # the SHOULD clauses become MUST clauses
        out.add("msm_eq_n")
        groups += [[c] for c in should]
        should, m = [], 0
    if not should:
        if not groups:
            return {"nothing"}
        out.add("must_only")
    elif m == 0:
        out.add("optional_with_must" if groups else "optional_without_must")
    else:
        out.add("required_union" if m == 1 else "required_disjunction")
    if must_not:
        out.add("exclude_1" if len(must_not) == 1 else "exclude_many")
    if len(groups) >= 4:  # block_wand_intersection: MUST TermScorers reading freqs and nothing else (:312-340)
        seq = not should and not must_not and all(len(g) == 1 and not basic and not (flags[g[0]] & TQ_TERM_IGNORE_FREQ) for g in groups)
        out.add("groups4_sequential" if seq else "groups4_intersection")
    return out


BOOL_BRANCHES = {"empty_must", "msm_gt_n", "msm_eq_n", "optional_with_must", "optional_without_must", "required_union",
                 "required_disjunction", "exclude_1", "exclude_many", "groups4_sequential", "groups4_intersection"}


def tile_smem_bytes(p_cap, max_slots, max_big, max_queries, seg_cap, cl_cap, n_win):
    """tile_smem_bytes (csrc/tq_layout.h) restated: TileQ 16 B, TileSeg 4 B, TileTQ 8 B, kTile = 1024, stage-A scratch 264 words.
    Takes numpy arrays as well as ints."""
    union = np.maximum(max_queries * 16 + np.maximum(seg_cap * 4, (2 * 64 + 8 * 17) * 4), n_win * 1024 * 4)
    union = (union + 15) & ~15
    return (p_cap * 4 + union + max_slots * 12 + max_big * 128 + max_queries * 8 + max_big * 64 + p_cap * 2 + max_queries * 2 +
            cl_cap * 2 + 64)


def hits(result, i=0):
    scores, segs, docs, counts = result
    n = int(counts[i])
    return [(float(scores[i, j]), int(segs[i, j]), int(docs[i, j])) for j in range(n)]
