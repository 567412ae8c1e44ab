"""A multi-field index for the score model, the oracle and the device: segment ordinals whose fields each have their own posting
lists, fieldnorms and record option, and queries whose clauses name different fields (a title + body search, the expansion of
QueryParser over several default fields).

Fields: BODY (WithFreqsAndPositions, about 40 tokens a doc, positions for the phrase terms), TITLE (WithFreqs, about 3 tokens, a
different fieldnorm distribution), TAGS (Basic: no freqs) and RAW (no fieldnorms).  A term's lists in different fields are drawn
around one base doc set, so the fields overlap and cross-field sums land on one doc.  Ordinals: A (every field), B (deletes; some
fields lack some terms), C (only TITLE, so its queries read one fieldnorm array that is not field 0's).  Weights and average
fieldnorms are the Searcher's per field: N = the sum of max_doc over every ordinal, tokens = the field's own total."""
import numpy as np

from oracle import tq_oracle as O
from tantivy_b200._abi import (TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT, TQ_OCCUR_SHOULD, TQ_OP_AND, TQ_OP_BOOL, TQ_OP_OR, TQ_OP_PHRASE,
                               TQ_OP_TERM, TQ_RECORD_BASIC, TQ_RECORD_FREQS, TQ_RECORD_FREQS_POSITIONS, TQ_TERM_IGNORE_FREQ)
from tests import score_model as M
from tests.helpers import OracleSegment, f32

BODY, TAGS, RAW, TITLE = 0, 1, 2, 3
FIELDS = (BODY, TAGS, RAW, TITLE)
RECORD = {BODY: TQ_RECORD_FREQS_POSITIONS, TITLE: TQ_RECORD_FREQS, TAGS: TQ_RECORD_BASIC, RAW: TQ_RECORD_FREQS}
# term densities of the base doc sets: thick (k_or_strip's thick lists, the tile engine's dense slots), middling, rare
DENS = (0.3, 0.15, 0.06, 0.02, 0.008, 0.004, 0.002, 0.001, 0.25, 0.1, 0.03, 0.012, 0.005, 0.003, 0.01, 0.01)
V = len(DENS)
P0, P1 = 14, 15  # the phrase terms of BODY (positions registered)
SHARE = {BODY: 1.0, TITLE: 0.25, TAGS: 0.5, RAW: 0.4}  # the part of a term's base docs each field holds
# (ordinal index, field, term): absent there (ordinal B lacks some terms in some fields)
ABSENT = {(1, TITLE, 0), (1, TITLE, 3), (1, TAGS, 2), (1, RAW, 1), (1, BODY, 7), (1, TAGS, 9)}


def _field_lists(rng, n, field, bases):
    lists = []
    for t, base in enumerate(bases):
        keep = base[rng.random(len(base)) < SHARE[field]]
        extra = np.nonzero(rng.random(n) < DENS[t] * (0.3 if field == BODY else 0.05))[0]
        docs = np.union1d(keep, extra).astype(np.uint32)
        if field == TAGS:
            lists.append((docs, None))
        elif field == TITLE:
            lists.append((docs, np.minimum(rng.geometric(0.8, size=len(docs)), 3).astype(np.uint32)))
        else:
            lists.append((docs, np.minimum(rng.geometric(0.5, size=len(docs)), 24).astype(np.uint32)))
    return lists


def _positions(rng, docs, tfs, lengths):
    """{doc: ascending positions} with tf positions below the doc's length (the length is raised where it is too short)."""
    out = {}
    for d, tf in zip(docs.tolist(), tfs.tolist()):
        lengths[d] = max(int(lengths[d]), tf + 2)
        out[d] = sorted(rng.choice(int(lengths[d]), size=tf, replace=False).tolist())
    return out


def _phrase_plant(rng, pos, lengths):
    """In about half the docs that hold both phrase terms, P1 right behind one of P0's positions."""
    for d in sorted(set(pos[P0]) & set(pos[P1])):
        if rng.random() < 0.5:
            p = pos[P0][d][0] + 1
            if p < lengths[d] and p not in pos[P0][d]:
                pos[P1][d] = sorted(set(pos[P1][d][1:]) | {p}) if len(pos[P1][d]) > 1 else [p]


class Ordinal:
    """One segment ordinal: per field the OracleSegment (writer output for oracle and device) and the model's multi-field Segment."""

    def __init__(self, rng, idx, ordinal, max_doc, fields, deletes, writer_cls):
        self.idx, self.ordinal, self.max_doc, self.fields = idx, ordinal, max_doc, fields
        bases = [np.nonzero(rng.random(max_doc) < p)[0] for p in DENS]
        self.alive = np.packbits(rng.random(max_doc) > 0.2, bitorder="little") if deletes else None
        self.lists, self.lengths, self.pos, self.pos_bytes, self.pos_range = {}, {}, {}, None, {}
        for f in fields:
            self.lists[f] = _field_lists(rng, max_doc, f, bases)
            if f == BODY:
                self.lengths[f] = np.clip(np.round(np.exp(rng.normal(np.log(36), 0.6, size=max_doc))), 1, 2000).astype(np.uint32)
            elif f in (TITLE, TAGS):
                self.lengths[f] = (1 + rng.poisson(2.0 if f == TITLE else 4.0, size=max_doc)).astype(np.uint32)
            else:
                self.lengths[f] = None
        if BODY in fields:
            lengths = self.lengths[BODY]
            self.pos = {t: _positions(rng, *self.lists[BODY][t], lengths) for t in (P0, P1)}
            _phrase_plant(rng, self.pos, lengths)
            for t in (P0, P1):  # tf = the number of positions
                docs = self.lists[BODY][t][0]
                self.lists[BODY][t] = (docs, np.array([len(self.pos[t][d]) for d in docs.tolist()], np.uint32))
            chunks, cursor = [], 0
            for t in (P0, P1):
                deltas = []
                for d in self.lists[BODY][t][0].tolist():
                    ps = self.pos[t][d]
                    deltas += [ps[0]] + [b - a for a, b in zip(ps, ps[1:])]
                data = bytes(O.positions_serialize(deltas))
                self.pos_range[t] = (cursor, cursor + len(data))
                cursor += len(data)
                chunks.append(data)
            self.pos_bytes = np.frombuffer(b"".join(chunks), dtype=np.uint8)
        self.osegs = {f: OracleSegment(self.lists[f], self.lengths[f], record_option=RECORD[f], segment_ord=ordinal, field=f,
                                       writer_cls=writer_cls, alive=self.alive, max_doc=max_doc) for f in fields}
        for i, f, t in ABSENT:  # (the queries name no list there; the model follows their term_segs)
            if i == idx:
                self.osegs[f].terms[t] = (0, 0, 0)
        self.model = self.model_with(self.alive)

    def model_with(self, alive):
        """The model's multi-field Segment of this ordinal with the alive bits `alive` on every field."""
        mf = {f: dict(lists=self.lists[f], lengths=self.lengths[f], basic=RECORD[f] == TQ_RECORD_BASIC) for f in self.fields}
        if BODY in self.fields:
            mf[BODY]["positions"] = [self.pos.get(t, {}) for t in range(V)]
        return M.Segment.multi_field(self.ordinal, mf, self.max_doc, alive=alive)

    def register(self, target, fields=None, alive=None):
        for f in (self.fields if fields is None else fields):
            s = self.osegs[f]
            target.segment_register(self.ordinal, f, self.max_doc, s.record_option, s.body, s.fn_ids, self.alive if alive is None else alive)
            if f == BODY:
                target.register_positions(self.ordinal, f, self.pos_bytes)


class Index:
    """Ordinals A (every field), B (deletes, terms missing from some fields) and C (TITLE only)."""

    def __init__(self, sizes=(300_000, 70_001, 50_000), seed=0xF1E1D, writer_cls=None, ordinals=(40, 41, 42)):
        rng = np.random.default_rng(seed)
        shapes = [(FIELDS, False), (FIELDS, True), ((TITLE,), False)]
        self.ords = [Ordinal(rng, i, o, n, fs, dl, writer_cls) for i, (o, n, (fs, dl)) in enumerate(zip(ordinals, sizes, shapes))]
        self.n_docs = sum(o.max_doc for o in self.ords)
        self.avg = {}
        for f in FIELDS:
            tokens = sum(o.osegs[f].total_num_tokens for o in self.ords if f in o.fields)
            self.avg[f] = f32(f32(tokens) / f32(self.n_docs))

    def register(self, target):
        for o in self.ords:
            o.register(target)
        return target

    def models(self):
        return [o.model for o in self.ords]

    def doc_freq(self, f, t):
        return sum(o.osegs[f].terms[t][0] for o in self.ords if f in o.fields)

    def query(self, op, clauses, k, boost=1.0, avg=None, **extra):
        """clauses = [(field, term)]; boost = one value or one per clause; avg = {clause: field whose average it takes} (a list
        under another field's average).  Returns (query dict, the model's terms)."""
        weights, avgs, term_segs = [], [], []
        for c, (f, t) in enumerate(clauses):
            b = boost[c] if isinstance(boost, (list, tuple)) else boost
            weights.append(O.bm25_weight(self.doc_freq(f, t), self.n_docs, b))
            avgs.append(self.avg[(avg or {}).get(c, f)])
            for o in self.ords:
                if f in o.fields and o.osegs[f].terms[t][0] > 0:
                    term_segs.append(o.osegs[f].term_seg(t, c))
        q = dict(op=op, k=k, weights=weights, avg_fieldnorm=avgs, term_segs=term_segs)
        q.update(extra)
        return q, [t for _, t in clauses]

    def phrase(self, k):
        """body:"p0 p1": one Bm25Weight for the two terms (idfs add up), BODY's average."""
        idf = f32(0)
        for t in (P0, P1):
            idf = f32(idf + f32(O.bm25_idf(self.doc_freq(BODY, t), self.n_docs)))
        w = f32(idf * f32(2.2))
        term_segs, term_pos = [], []
        for c, t in enumerate((P0, P1)):
            for o in self.ords:
                if BODY in o.fields and o.osegs[BODY].terms[t][0] > 0:
                    term_segs.append(o.osegs[BODY].term_seg(t, c))
                    term_pos.append(o.pos_range[t])
        q = dict(op=TQ_OP_PHRASE, k=k, weights=[w, w], avg_fieldnorm=[self.avg[BODY]] * 2, term_segs=term_segs, term_pos=term_pos,
                 term_offset=[0, 1])
        return q, [P0, P1]


def expand(terms, fields):
    """QueryParser's expansion over several default fields: every term in every field, term-major."""
    return [(f, t) for t in terms for f in fields]


KS = (1, 10, 129, 1024)


def battery(ix, bool_ok=True, phrase=True):
    """The shapes of the multi-field suite, as (query, terms): TERM on each field; ORs over 2-4 fields of 1-8 terms (up to 32
    clauses); ANDs across fields (4-8 MUST scorers with a Basic or TQ_TERM_IGNORE_FREQ clause too); BOOL (+(title:a body:a)
    +(title:b body:b), SHOULD with MUST_NOT on another field, minimum_should_match across fields); boosts of 0 and -1.5; one
    list under one weight with two averages; a phrase on BODY.  Fields alternate from query to query."""
    qs = []
    for f in FIELDS:
        for t in (0, 4, 9, 13):
            qs += [ix.query(TQ_OP_TERM, [(f, t)], k) for k in (1, 129)]
    ors = [expand([0], (TITLE, BODY)), expand([4, 9], (BODY, TITLE)), expand([1, 5, 6], (TITLE, BODY, TAGS)),
           expand([3, 6, 7, 12], (RAW, BODY, TITLE, TAGS)), expand([0, 8], (TITLE, BODY)), expand([5, 6, 7], (TITLE, TAGS)),
           expand(list(range(2, 10)), (BODY, TITLE, TAGS, RAW)), expand([10, 11, 12, 13, 2], (TITLE, RAW)),
           expand([6, 7, 13], (TITLE, BODY)), expand([1, 2], (TAGS, RAW))]
    for cl in ors:
        qs += [ix.query(TQ_OP_OR, cl, k) for k in KS]
    ands = [[(TITLE, 1), (BODY, 0)], [(BODY, 2), (TITLE, 2)], [(TITLE, 9), (BODY, 1), (RAW, 8)],
            [(BODY, 0), (TITLE, 8), (BODY, 9), (RAW, 1)], [(BODY, 0), (TAGS, 8), (BODY, 1), (TITLE, 0), (RAW, 9)],
            [(BODY, 8), (BODY, 0), (TITLE, 9), (RAW, 0), (BODY, 9), (TITLE, 8), (TAGS, 0), (BODY, 2)]]
    for cl in ands:
        qs += [ix.query(TQ_OP_AND, cl, k) for k in (1, 10, 1024)]
        if len(cl) >= 4:  # one clause without freqs: Intersection::score's order
            qs.append(ix.query(TQ_OP_AND, cl, 10, term_flags=[0] * (len(cl) - 1) + [TQ_TERM_IGNORE_FREQ]))
    # boosts 0 and negative: not prunable
    qs += [ix.query(TQ_OP_OR, expand([0, 4], (BODY, TITLE)), 10, boost=[1.0, 0.0, 1.0, -1.5]),
           ix.query(TQ_OP_AND, [(BODY, 0), (TITLE, 8)], 129, boost=[-1.5, 1.0])]
    # one list under one weight and two averages (its own field's and TITLE's), in the same batch and inside one query
    qs += [ix.query(TQ_OP_OR, [(BODY, 1), (BODY, 4)], 129), ix.query(TQ_OP_OR, [(BODY, 1), (BODY, 4)], 129, avg={0: TITLE}),
           ix.query(TQ_OP_OR, [(BODY, 1), (TITLE, 4), (BODY, 5)], 10, avg={2: TITLE}),
           ix.query(TQ_OP_TERM, [(BODY, 4)], 10, avg={0: TITLE})]
    if bool_ok:
        M_, S_, N_ = TQ_OCCUR_MUST, TQ_OCCUR_SHOULD, TQ_OCCUR_MUST_NOT
        bools = [([(TITLE, 1), (BODY, 1), (TITLE, 2), (BODY, 2)], [M_] * 4, [1, 1, 2, 2], 0),        # +(title:a body:a) +(title:b body:b)
                 ([(TITLE, 0), (BODY, 0), (TITLE, 9), (BODY, 9)], [M_] * 4, [1, 1, 2, 2], 0),
                 ([(BODY, 0), (TITLE, 0), (TITLE, 3)], [S_, S_, N_], None, 0),                     # SHOULD, MUST_NOT on another field
                 ([(BODY, 1), (TITLE, 1), (TAGS, 1), (RAW, 5)], [S_, S_, S_, N_], None, 2),       # minimum_should_match across fields
                 ([(TITLE, 8), (BODY, 8), (TAGS, 9), (RAW, 9), (BODY, 3)], [M_, S_, S_, S_, N_], [1, 0, 0, 0, 0], 2),
                 ([(BODY, 0), (TITLE, 1), (TAGS, 8), (RAW, 0), (BODY, 9)], [M_] * 5, None, 0)]     # five MUST groups, a Basic one
        for cl, occ, grp, msm in bools:
            for k in (10, 1024):
                q, t = ix.query(TQ_OP_OR, cl, k)
                q.update(op=TQ_OP_BOOL, term_occur=occ, min_should_match=msm)
                if grp is not None:
                    q["term_group"] = grp
                qs.append((q, t))
    if phrase:
        qs += [ix.phrase(k) for k in (10, 129)]
    return qs


def with_thresholds(qs, rows_of):
    """Copies of some queries with an initial threshold at their k-th score (rows_of(q, terms) = the model's rows)."""
    out = []
    for i, (q, t) in enumerate(qs):
        if i % 5 or q["k"] < 10:
            continue
        rows = rows_of(q, t)
        if rows:
            out.append((dict(q, threshold=float(rows[min(q["k"], len(rows)) - 1][0])), t))
    return out
