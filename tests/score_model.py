"""A plain numpy model of the reference's BM25 scorers and collectors, independent of `oracle/` and of the product library.

Inputs are the raw posting lists, doc lengths, alive bits, the terms' positions (phrase queries) and the query dict of
`tantivy_b200._abi.QueryBatch`.  The query's
Bm25Weight.weight and average fieldnorm (or explicit tf cache) are taken as given; everything else is computed in np.float32 with
the reference's operation order (paths relative to the reference tree, quickwit-oss/tantivy @ 70f0b03).  numpy's f32 + - * / round
to nearest like the reference's f32 code, so the model is bit-exact where the order is.  Every score is computed again in float64
and checked against a rounding bound: a formula slip that the oracle and the model shared would show there.
"""
import numpy as np

from tantivy_b200._abi import (TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT, TQ_OCCUR_SHOULD, TQ_OP_AND, TQ_OP_BOOL, TQ_OP_OR, TQ_OP_PHRASE,
                               TQ_OP_TERM, TQ_TERM_IGNORE_FREQ)
from tests.helpers import _FN_TABLE, fieldnorm_ids

f32, f64 = np.float32, np.float64
K1, B = f32(1.2), f32(0.75)  # bm25.rs:8-9
EPS = 2.0 ** -23


class Segment:
    """One segment of one field: posting lists [(docs, tfs or None)], per-doc token counts (None: a field without
    fieldnorms, constant fieldnorm 1, term_weight.rs:218), alive bits (np.packbits little-endian, None: no deletes),
    basic=True for a field indexed without freqs (IndexRecordOption::Basic), positions (phrase queries) = for every list index
    {doc: ascending positions of the term in the doc}."""

    def __init__(self, segment_ord, lists, lengths, alive=None, basic=False, max_doc=None, positions=None):
        self.segment_ord = segment_ord
        self.lists = [(np.asarray(d, np.uint32), None if t is None else np.asarray(t, np.uint32)) for d, t in lists]
        self.max_doc = len(lengths) if lengths is not None else max_doc
        self.fn_ids = fieldnorm_ids(lengths) if lengths is not None else np.ones(self.max_doc, np.uint8)
        self.alive = None if alive is None else np.unpackbits(np.asarray(alive, np.uint8), bitorder="little")[:self.max_doc].astype(bool)
        self.basic = basic
        self.positions = positions
        self.fields = None  # (multi_field: field id -> that field's Segment)

    @classmethod
    def multi_field(cls, segment_ord, fields, max_doc, alive=None):
        """One segment ordinal with several fields: fields = {field id: dict(lists=, lengths= (None: no fieldnorms), basic=,
        positions=)}.  Every field shares max_doc and the alive bits, as the fields of one tantivy segment do; a clause reads the
        field its term_segs entry names (lists, fieldnorm ids and record option of that field)."""
        per = {f: cls(segment_ord, d["lists"], d.get("lengths"), alive=alive, basic=d.get("basic", False), max_doc=max_doc,
                      positions=d.get("positions")) for f, d in fields.items()}
        assert all(s.max_doc == max_doc for s in per.values())
        seg = per[min(per)]
        out = cls.__new__(cls)
        out.__dict__.update(seg.__dict__)
        out.fields = per
        return out

    def field(self, f):
        """The Segment of field f (a single-field segment is every field's: its callers name field 0 or none)."""
        return self if self.fields is None else self.fields[f]


def tf_cache(avg, dtype=f32):
    """cached_tf_component for the 256 fieldnorm ids: K1 * (1 - B + B * fieldnorm / avg) (bm25.rs:58-68)."""
    fn = _FN_TABLE.astype(f32).astype(dtype)  # (`fieldnorm as Score`: f32 first)
    k1, b, avg = dtype(K1), dtype(B), dtype(f32(avg))
    return k1 * ((dtype(1) - b) + (b * fn) / avg)


class _Term:
    """TermScorer of one clause in one segment: docs, and their scores in f32 (weight * tf / (tf + norm), bm25.rs:179-193)
    and in f64 from the same inputs."""

    def __init__(self, seg, q, clause, list_idx):
        docs, tfs = seg.lists[list_idx]
        flags = q.get("term_flags")
        self.reads_freqs = not seg.basic and not (flags is not None and flags[clause] & TQ_TERM_IGNORE_FREQ)
        tf = tfs if self.reads_freqs and tfs is not None else np.ones(len(docs), np.uint32)  # NoFreq / SkipFreq: tf = 1
        self.docs, self.df, self.clause = docs, len(docs), clause
        self.weight = f32(q["weights"][clause])
        ids = seg.fn_ids[docs]
        cache = q.get("tf_cache")
        if cache is not None:
            c32 = np.asarray(cache, f32).reshape(-1, 256)[clause]
            c64 = c32.astype(f64)
        else:
            c32, c64 = tf_cache(q["avg_fieldnorm"][clause]), tf_cache(q["avg_fieldnorm"][clause], f64)
        t32 = tf.astype(f32)  # (`term_freq as Score`)
        self.s32 = self.weight * (t32 / (t32 + c32[ids]))
        t64 = tf.astype(f64)
        self.s64 = f64(self.weight) * (t64 / (t64 + c64[ids]))


class _Dense:
    """Per-doc partial sums over a segment: which docs match, their f32 sum, f64 sum and sum of |term scores|."""

    def __init__(self, max_doc):
        self.has = np.zeros(max_doc, bool)
        self.s32 = np.zeros(max_doc, f32)
        self.s64 = np.zeros(max_doc, f64)
        self.mag = np.zeros(max_doc, f64)
        self.n = np.zeros(max_doc, np.int32)  # term scores in the sum

    def add_term(self, t):
        """SumCombiner: the first matching score, then += (score_combiner.rs:39-57)."""
        d = t.docs
        self.s32[d] = np.where(self.has[d], self.s32[d] + t.s32, t.s32)
        self.s64[d] += t.s64
        self.mag[d] += np.abs(t.s64)
        self.n[d] += 1
        self.has[d] = True

    def add(self, other, mask):
        """self += other on `mask` (other's docs), f32 in that order; a doc without a sum yet takes other's."""
        self.s32 = np.where(mask, np.where(self.has, self.s32 + other.s32, other.s32), self.s32)
        self.s64 = np.where(mask, self.s64 + other.s64, self.s64)
        self.mag = np.where(mask, self.mag + other.mag, self.mag)
        self.n = np.where(mask, self.n + other.n, self.n)
        self.has = self.has | mask


def _union(terms, max_doc):
    """A union's sum in the project's canonical order: descending Bm25Weight.weight, ties in clause order (DESIGN.md §5; the
    reference's own order is data dependent, buffered_union.rs:69-85, block_wand_union.rs:205-208)."""
    u = _Dense(max_doc)
    for t in sorted(terms, key=lambda t: -t.weight):
        u.add_term(t)
    return u


def _intersect(parts, max_doc, intersection_order):
    """Scorers s0, s1, s2, ... (ascending cost, stable) of an intersection: the docs all of them match, summed
    ((s0 + s1) + s2) + s3 ... as block_wand_intersection does (block_wand_intersection.rs:146-158), or
    (s0 + s1) + (s2 + s3 + ...) as Intersection::score does (intersection.rs:325-329)."""
    out = _Dense(max_doc)
    out.has[:] = True
    for p in parts:
        out.has &= p.has
    m = out.has
    head = _Dense(max_doc)
    rest = _Dense(max_doc)
    for i, p in enumerate(parts):
        (rest if intersection_order and i >= 2 else head).add(p, m)
    if intersection_order and len(parts) > 2:
        head.add(rest, m)
    head.has = m.copy()
    return head


def _segment_matches(seg, q, terms, intersection_order=None):
    """complex_scorer / the specialised scorers for one segment: a _Dense of the matching docs (before deletes), or None."""
    op = q["op"]
    field_of = {ts[0]: ts[2] for ts in q["term_segs"] if ts[1] == seg.segment_ord and ts[3] > 0}  # present clause -> its field
    if op == TQ_OP_PHRASE:
        return _phrase_matches(seg.field(field_of[0]) if 0 in field_of else seg, q, terms)
    n = len(q["weights"])
    scorer = {c: _Term(seg.field(field_of[c]), q, c, terms[c]) for c in range(n) if c in field_of}  # (in clause order)
    if op == TQ_OP_TERM or (op in (TQ_OP_AND, TQ_OP_OR) and n == 1):
        return _union(list(scorer.values()), seg.max_doc) if scorer else None
    if op == TQ_OP_OR:
        return _union(list(scorer.values()), seg.max_doc) if scorer else None
    if op == TQ_OP_AND:
        if len(scorer) < n:  # an EmptyScorer MUST empties the intersection (boolean_weight.rs:248-252)
            return None
        ts = sorted(scorer.values(), key=lambda t: t.df)  # stable: ties in clause order (intersection.rs:31)
        # block_wand_intersection only when every TermScorer reads freqs (boolean_weight.rs:318-330)
        io = not all(t.reads_freqs for t in ts) if intersection_order is None else intersection_order
        return _intersect([_union([t], seg.max_doc) for t in ts], seg.max_doc, io)
    assert op == TQ_OP_BOOL
    occ = q["term_occur"]
    grp = q.get("term_group")
    groups = {}  # MUST groups in declaration order: group id -> present clauses
    for c in range(n):
        if occ[c] == TQ_OCCUR_MUST:
            groups.setdefault(grp[c] if grp is not None else 256 + c, [])
            if c in scorer:
                groups[grp[c] if grp is not None else 256 + c].append(scorer[c])
    if any(not g for g in groups.values()):  # boolean_weight.rs:248-252
        return None
    groups = list(groups.values())
    should = [scorer[c] for c in range(n) if occ[c] == TQ_OCCUR_SHOULD and c in scorer]
    must_not = [scorer[c] for c in range(n) if occ[c] == TQ_OCCUR_MUST_NOT and c in scorer]
    m = int(q.get("min_should_match", 0))
    if m > len(should):  # boolean_weight.rs:275-279
        return None
    if m >= 2 and m == len(should):  # :292-297: as many as there are, they are MUST clauses
        groups += [[t] for t in should]
        should, m = [], 0
    if not groups and not should:
        return None
    need = m if m >= 1 else (0 if groups else 1)
    groups.sort(key=lambda g: sum(t.df for t in g))  # a union's cost = the sum of its scorers' (buffered_union.rs:326-328)
    # block_wand_intersection: >= 2 MUST scorers, each a TermScorer reading freqs, nothing else left (boolean_weight.rs:312-340)
    sequential = len(groups) >= 2 and not should and not must_not and all(len(g) == 1 and g[0].reads_freqs for g in groups)
    io = not sequential if intersection_order is None else intersection_order
    opt = _union(should, seg.max_doc)
    ok = opt.n >= need
    if groups:
        out = _intersect([_union(g, seg.max_doc) for g in groups], seg.max_doc, io)
        ok &= out.has
        out.add(opt, ok & opt.has)  # RequiredOptionalScorer: req + opt (reqopt_scorer.rs:78-94)
    else:
        out = opt
        ok &= opt.has
    for t in must_not:  # Exclude (exclude.rs)
        ok[t.docs] = False
    out.has = ok
    return out


def slop_matches(left, right, slop):
    """intersection_count_with_slop as documented (phrase_scorer.rs:138-186): walking both ascending lists, a left position within
    `slop` of the right one is a match -- unless a later left position is still not beyond the right one, which is the better
    match -- and then both sides move on; otherwise the side with the smaller position moves on.  Not symmetric: a right
    position may precede its left one by up to `slop`.  Returns the matched right positions (their count is the phrase count)."""
    out, i, j = [], 0, 0
    while i < len(left) and j < len(right):
        if abs(int(left[i]) - int(right[j])) <= slop:
            while i + 1 < len(left) and left[i + 1] <= right[j]:
                i += 1
            out.append(right[j])
            i, j = i + 1, j + 1
        elif left[i] < right[j]:
            i += 1
        else:
            j += 1
    return out


def _phrase_matches(seg, q, terms):
    """PhraseWeight::scorer over one segment (phrase_query.rs:48-53, phrase_weight.rs, phrase_scorer.rs:349-589): the clauses in
    offset order (stable), each clause's positions shifted by max_offset - its offset; docs that hold every clause; phrase count =
    size of the intersection of the shifted sets, or with slop (two terms) slop_matches(left, right) where left is the first clause
    after a stable sort by this segment's doc_freq (the Intersection's order, intersection.rs:89).  Score = weight[0] *
    tf_factor(fieldnorm_id, count) with row 0 of tf_cache (or avg_fieldnorm[0]): ONE Bm25Weight for the whole phrase."""
    n = len(q["weights"])
    present = {ts[0] for ts in q["term_segs"] if ts[1] == seg.segment_ord and ts[3] > 0}
    if len(present) < n:  # a clause without postings here: no match
        return None
    offsets = [int(o) for o in q["term_offset"]]
    order = sorted(range(n), key=lambda c: offsets[c])
    max_off = max(offsets)
    slop = int(q.get("slop", 0))
    if slop:
        assert n == 2, "sloppy phrases of three and more terms are not modelled"
        order = sorted(order, key=lambda c: len(seg.lists[terms[c]][0]))
    docs = seg.lists[terms[order[0]]][0]
    for c in order[1:]:
        docs = np.intersect1d(docs, seg.lists[terms[c]][0])
    cnt = np.zeros(seg.max_doc, np.int64)
    for d in docs.tolist():
        shifted = [[p + max_off - offsets[c] for p in seg.positions[terms[c]][d]] for c in order]
        if slop:
            cnt[d] = len(slop_matches(shifted[0], shifted[1], slop))
        else:
            cnt[d] = len(set.intersection(*[set(s) for s in shifted]))
    out = _Dense(seg.max_doc)
    out.has = cnt > 0
    cache = q.get("tf_cache")
    if cache is not None:
        c32 = np.asarray(cache, f32).reshape(-1, 256)[0]
        c64 = c32.astype(f64)
    else:
        c32, c64 = tf_cache(q["avg_fieldnorm"][0]), tf_cache(q["avg_fieldnorm"][0], f64)
    w = f32(q["weights"][0])
    t32, t64 = cnt.astype(f32), cnt.astype(f64)
    with np.errstate(invalid="ignore", divide="ignore"):
        out.s32 = np.where(out.has, w * (t32 / (t32 + c32[seg.fn_ids])), f32(0))
        out.s64 = np.where(out.has, f64(w) * (t64 / (t64 + c64[seg.fn_ids])), 0.0)
    out.mag = np.abs(out.s64)
    out.n = out.has.astype(np.int32)
    return out


def _check_rounding(d, sel):
    """|f32 - f64| <= (n + 2) * 2^-23 * sum |term scores|: the model's f32 formula agrees with its f64 restatement."""
    err = np.abs(d.s32[sel].astype(f64) - d.s64[sel])
    bound = (d.n[sel] + 2) * EPS * d.mag[sel]
    bad = np.nonzero(err > bound)[0]
    assert len(bad) == 0, f"f32 score off its f64 value beyond rounding: {d.s32[sel][bad[:4]]} vs {d.s64[sel][bad[:4]]}"


def merge_fruits(lists, k):
    """merge_fruits (sort_key_top_collector.rs:76-95): the rows [(score, segment_ord, doc)] of several lists in one, by score desc
    (partial_cmp: -0.0 and +0.0 are equal, sort_by_score.rs:99-107), then segment asc, doc asc; the first k."""
    rows = sorted((r for rows in lists for r in rows), key=lambda r: (-r[0], r[1], r[2]))
    return [(float(s), int(so), int(doc)) for s, so, doc in rows[:k]]


def search(segments, q, terms, intersection_order=None, doc_ranges=None):
    """TopDocs over the segments: rows [(score, segment_ord, doc)] sorted by score desc, segment asc, doc asc (merge_fruits,
    top_score_collector.rs:591-600), deleted docs skipped, with a threshold only scores strictly above it (weight.rs:47-60).
    terms[c] = the posting list (index into Segment.lists) of clause c; q["term_segs"] says in which segments it has postings.
    intersection_order forces one summation order for every intersection (None: the reference's rule).
    doc_ranges = {segment_ord: (lo, hi)}: only docs [lo, hi) of that segment exist (the others count as deleted), e.g. the part of
    a segment one shard holds; `segments` itself may be any subset of the index's (a shard's), with the weights of the whole index."""
    rows = []
    thr = q.get("threshold")
    has_thr = thr is not None and thr == thr  # (a NaN threshold is no threshold)
    for seg in sorted(segments, key=lambda s: s.segment_ord):
        d = _segment_matches(seg, q, terms, intersection_order)
        if d is None:
            continue
        sel = d.has.copy()
        if seg.alive is not None:
            sel &= seg.alive
        if doc_ranges is not None and seg.segment_ord in doc_ranges:
            lo, hi = doc_ranges[seg.segment_ord]
            sel[:lo] = False
            sel[hi:] = False
        _check_rounding(d, sel)
        if has_thr:
            sel &= d.s32 > f32(thr)
        docs = np.nonzero(sel)[0]
        rows += [(f32(s), seg.segment_ord, int(doc)) for s, doc in zip(d.s32[docs], docs)]
    return merge_fruits([rows], q["k"])


def count(segments, q, terms, doc_ranges=None):
    """Count collector: alive docs that match (count_collector.rs); doc_ranges as in search."""
    total = 0
    for seg in segments:
        d = _segment_matches(seg, q, terms)
        if d is None:
            continue
        sel = d.has & seg.alive if seg.alive is not None else d.has.copy()
        if doc_ranges is not None and seg.segment_ord in doc_ranges:
            lo, hi = doc_ranges[seg.segment_ord]
            sel[:lo] = False
            sel[hi:] = False
        total += int(sel.sum())
    return total


class Compacted:
    """A segment of any max_doc (up to 2^31 - 2) on a compacted doc space, for search and count.  A score depends only on a doc's
    postings, fieldnorm id and alive bit, and the order of rows only on the order of doc ids, so the model is exact over the sorted
    union of the docs that occur in the segment's lists (and positions), mapped onto 0..n-1: `docs[i]` is the real id of doc i.
    fn_ids = the segment's fieldnorm id per doc (uint8, None: no fieldnorms), alive = its packed alive bitset (None: no deletes);
    neither is expanded to max_doc.  Weights and average fieldnorms stay those of the real index: queries carry them."""

    def __init__(self, segment_ord, lists, max_doc, fn_ids=None, alive=None, basic=False, positions=None):
        parts = [np.asarray(d, np.uint32) for d, _ in lists]
        if positions is not None:
            parts += [np.fromiter(p, np.uint32, len(p)) for p in positions]
        self.docs = np.unique(np.concatenate(parts)) if parts else np.zeros(0, np.uint32)
        assert len(self.docs) == 0 or int(self.docs[-1]) < max_doc
        self.max_doc = max_doc
        mapped = [(np.searchsorted(self.docs, np.asarray(d, np.uint32)), t) for d, t in lists]
        lengths = None if fn_ids is None else _FN_TABLE[np.asarray(fn_ids)[self.docs]]
        bits = None
        if alive is not None:
            a = np.asarray(alive, np.uint8)
            bits = np.packbits((a[self.docs >> 3] >> (self.docs & 7)) & 1, bitorder="little")
        pos = None
        if positions is not None:
            pos = [{int(np.searchsorted(self.docs, d)): ps for d, ps in p.items()} for p in positions]
        self.seg = Segment(segment_ord, mapped, lengths, alive=bits, basic=basic, max_doc=len(self.docs), positions=pos)

    def doc_range(self, lo, hi):
        """[lo, hi) of real doc ids on the compacted space."""
        return int(np.searchsorted(self.docs, lo)), int(np.searchsorted(self.docs, hi))


def _compacted_ranges(csegs, doc_ranges):
    if doc_ranges is None:
        return None
    by = {c.seg.segment_ord: c for c in csegs}
    return {so: by[so].doc_range(lo, hi) for so, (lo, hi) in doc_ranges.items() if so in by}


def search_compacted(csegs, q, terms, intersection_order=None, doc_ranges=None):
    """search over Compacted segments: rows with real doc ids; doc_ranges in real doc ids."""
    rows = search([c.seg for c in csegs], q, terms, intersection_order, _compacted_ranges(csegs, doc_ranges))
    docs = {c.seg.segment_ord: c.docs for c in csegs}
    return [(s, g, int(docs[g][d])) for s, g, d in rows]


def count_compacted(csegs, q, terms, doc_ranges=None):
    return count([c.seg for c in csegs], q, terms, _compacted_ranges(csegs, doc_ranges))
