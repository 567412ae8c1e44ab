"""Phrase queries (k_phrase) at their edges, on every route: the device, the numpy model of tests/score_model.py and the oracle
(oracle/phrase.hpp) must agree bit for bit -- doc ids, segment ordinals and f32 scores.

Position streams: bit-width-0 blocks, a 32-bit delta inside a bit-packed block, streams without a VInt rest, a doc with thousands
of occurrences.  Posting lists of 1, 127, 128, 129, 256 and 257 docs as leader and as secondary.  Phrases of 2 to 8 terms in one
batch, offsets with gaps, repeats and in any clause order, slop.  Zero / negative / huge weights, explicit tf caches, deletes,
initial thresholds, thousands of ties.  Routes: the side stream next to the tile engine, one stream, no tile engine, an
overflowing run that is repeated; prepare / run / fetch, phased runs with threshold and top-keys exchanges, doc-range parts and
segments spread over several contexts."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from oracle import tq_oracle as O  # noqa: E402
from tantivy_b200._abi import TQ_OP_OR, QueryBatch  # noqa: E402
from tantivy_b200.sharding import merge_rows_host, score_keys  # noqa: E402
from tests import score_model as M  # noqa: E402
from tests.helpers import hits  # noqa: E402
from tests.test_gpu_parity import DOC_RANGE_CUTS, _ctx_with_env  # noqa: E402
from tests.test_gpu_phrase import PosSegment, phrase_query  # noqa: E402

B31 = 1 << 31
DF_SIZES = (1, 127, 128, 129, 256, 257)
DF_POS = {1: 3, 127: 0, 128: 5, 129: 1, 256: 4, 257: 2}  # the fixed position of term d<n> in every doc that holds it


def _streams_segment(rng):
    """Position-stream edges.  z0 / z1: 300 docs with z0 at 0 (every delta 0: bit width 0) and z1 at 1.  b0 / b1: doc 0 holds b0 at
    0 and 2^31 + 3, b1 at 2^31 + 4 (32-bit deltas inside the first bit-packed block), docs 1..200 the pair at 5, 6.  m0 / m1 / m2:
    256, 256 and 128 deltas (no VInt rest).  r0 / r1: doc 350 holds "r0 r1" 3000 times."""
    n = 400
    lengths = rng.integers(5, 60, size=n)
    lengths[350] = 6500
    p = {"z0": {d: [0] for d in range(300)}, "z1": {d: [1] for d in range(300)}}
    p["b0"] = {0: [0, B31 + 3], **{d: [5] for d in range(1, 201)}}
    p["b1"] = {0: [B31 + 4], **{d: [6] for d in range(1, 201)}}
    p["m0"] = {d: [3, 9] for d in range(128)}
    p["m1"] = {d: [4, 12] for d in range(128)}
    p["m2"] = {d: [7, 8] for d in range(64)}
    p["r0"] = {350: [100 + 2 * i for i in range(3000)], **{d: [0] for d in range(351, 361)}}
    p["r1"] = {350: [101 + 2 * i for i in range(3000)], **{d: [1] for d in range(351, 400, 3)}}
    return PosSegment.from_positions(p, lengths)


def _df_segment(rng):
    """d<n> on docs 0, 3, 6, ... (n docs) at DF_POS[n], and once more 20 later in every 15th doc; e300 on docs 0..299 at 6: a
    secondary that ends before the leader d129 / d256 / d257 does."""
    n = 800
    p = {}
    for size in DF_SIZES:
        p[f"d{size}"] = {3 * i: [DF_POS[size]] + ([DF_POS[size] + 20] if (3 * i) % 15 == 0 else []) for i in range(size)}
    p["e300"] = {d: [6] + ([26] if d % 15 == 0 else []) for d in range(300)}
    return PosSegment.from_positions(p, rng.integers(8, 40, size=n))


def _plant_texts(rng, n):
    """Random texts over w0..w7 with "w0 w1 ... w7" or eight w0 planted in some docs."""
    vocab = np.array([f"w{i}" for i in range(8)])
    p = np.array([0.3, 0.2, 0.15, 0.1, 0.09, 0.07, 0.05, 0.04])
    out = []
    for _ in range(n):
        words = list(rng.choice(vocab, size=int(rng.integers(2, 40)), p=p / p.sum()))
        r = rng.random()
        at = int(rng.integers(0, len(words) + 1))
        if r < 0.3:
            words[at:at] = [f"w{i}" for i in range(8)]
        elif r < 0.4:
            words[at:at] = ["w0"] * 8
        out.append(" ".join(words))
    return out


def _uv_segments(rng):
    """u and v with equal doc_freq in the first segment (doc 0 = "a a b b" of the offset-order example: u = a, v = b) and unequal
    doc_freq in the second."""
    n = 200
    pu, pv = {0: [0, 1]}, {0: [2, 3]}
    for d in range(1, n):
        pu[d] = sorted(set(rng.integers(0, 20, size=int(rng.integers(1, 6))).tolist()))
        pv[d] = sorted(set(rng.integers(0, 20, size=int(rng.integers(1, 6))).tolist()))
    eq = PosSegment.from_positions({"u": pu, "v": pv}, rng.integers(4, 30, size=n))
    pu, pv = {}, {}
    for d in range(300):
        if rng.random() < 0.6:
            pu[d] = sorted(set(rng.integers(0, 20, size=int(rng.integers(1, 6))).tolist()))
        if rng.random() < 0.4:
            pv[d] = sorted(set(rng.integers(0, 20, size=int(rng.integers(1, 6))).tolist()))
    ne = PosSegment.from_positions({"u": pu, "v": pv}, rng.integers(4, 30, size=300))
    return [eq, ne]


def _tie_segments():
    """Three segments of 3000 docs in which "t0 t1" occurs once in every doc, all docs of one length: every doc ties."""
    return [PosSegment.from_positions({"t0": {d: [0] for d in range(3000)}, "t1": {d: [1] for d in range(3000)}}, np.full(3000, 10))
            for _ in range(3)]


def _deleted_copy(seg, phrase, rng):
    """seg with its 10 best docs for `phrase` deleted (and a fifth of the rest)."""
    best = [d for _, _, d in M.search([seg.model(phrase)], phrase_query([seg], phrase, 10)[0], list(range(len(phrase))))]
    alive = rng.random(seg.n_docs) > 0.2
    alive[best] = False
    return PosSegment.from_positions(seg.positions, seg.lengths, alive=np.packbits(alive, bitorder="little"))


class Battery:
    """Segments, the queries over them, and each query's rows from the model (checked against the oracle once)."""

    def __init__(self, segs, queries):
        self.segs = segs
        self.vocab = sorted({t for s in segs for t in s.vocab})
        msegs = [s.model(self.vocab) for s in segs]
        self.queries = [q for q, _ in queries]
        self.qb = QueryBatch(self.queries)
        self.want = [M.search(msegs, q, [self.vocab.index(t) for t in terms]) for q, terms in queries]
        oi = O.OracleIndex()
        for s in segs:
            s.register(oi)
        ref = oi.search_batch(self.qb, mode=0, n_threads=8)
        for i, w in enumerate(self.want):
            assert _bits(hits(ref, i)) == _bits(w), (i, hits(ref, i)[:4], w[:4])

    def register(self, ctx):
        for s in self.segs:
            s.register(ctx)
        return ctx

    def check(self, result, what=""):
        for i, w in enumerate(self.want):
            got = hits(result, i)
            assert _bits(got) == _bits(w), (what, i, got[:4], w[:4])


def _bits(rows):
    return [(int(np.float32(s).view(np.uint32)), g, d) for s, g, d in rows]


def _pq(segs, phrase, k, offsets=None, **extra):
    q = phrase_query(segs, phrase, k, offsets=offsets)[0]
    q.update(extra)
    return q, phrase


def _or(segs, terms, k):
    """A union over the same segments (an OR query: the batch then has a tile group next to the phrases)."""
    n_docs = sum(s.n_docs for s in segs)
    avg = np.float32(np.float32(sum(s.tokens for s in segs)) / np.float32(n_docs))
    term_segs, weights = [], []
    for c, t in enumerate(terms):
        df = sum((s.term(t) or (0,))[0] for s in segs)
        weights.append(O.bm25_weight(df, n_docs))
        for s in segs:
            ti = s.term(t)
            if ti:
                term_segs.append((c, s.ord, 0, ti[0], ti[1], ti[2]))
    return dict(op=TQ_OP_OR, k=k, weights=weights, avg_fieldnorm=[avg] * len(terms), term_segs=term_segs), terms


def _scored(q, **kw):
    q = dict(q[0]), q[1]
    q[0].update(kw)
    return q


def _battery_queries(segs, base_rows):
    """Every edge above over `segs`; base_rows(q) = the model's rows of q (for the thresholds)."""
    qs = []
    # position streams
    qs += [_pq(segs, ph, k) for ph in (["z0", "z1"], ["b0", "b1"], ["m0", "m1"], ["m2", "m0"], ["r0", "r1"], ["z1", "z0"]) for k in (5, 300)]
    qs.append(_pq(segs, ["m0", "m1"], 200, offsets=[0, 1], slop=3))
    qs.append(_pq(segs, ["r1", "r0"], 20, offsets=[1, 0], slop=2))
    # posting lists of 1 .. 257 docs as leader and secondary, the rarest clause neither first nor at offset 0
    for a in DF_SIZES:
        for b in DF_SIZES:
            if a != b:
                qs.append(_pq(segs, [f"d{a}", f"d{b}"], 300, offsets=[DF_POS[a], DF_POS[b]]))
    qs.append(_pq(segs, ["d257", "d1", "d127"], 10, offsets=[2, 3, 0]))
    qs.append(_pq(segs, ["d256", "d128", "d129", "d257"], 300, offsets=[4, 5, 1, 2]))
    qs += [_pq(segs, [f"d{a}", "e300"], 300, offsets=[DF_POS[a], 6]) for a in (129, 256, 257, 1)]
    # shapes: 2..8 terms in one batch, eight copies of one term, gaps, offsets not from 0, repeated and out-of-order offsets
    for n in range(2, 9):
        qs += [_pq(segs, [f"w{i}" for i in range(n)], k) for k in (1, 50)]
    qs += [_pq(segs, ["w0"] * 8, k) for k in (10, 400)]
    qs.append(_pq(segs, ["w0", "w2", "w5"], 100, offsets=[0, 2, 5]))
    qs.append(_pq(segs, ["w3", "w4", "w5"], 100, offsets=[3, 4, 5]))
    qs.append(_pq(segs, ["w0", "w1", "w1"], 100, offsets=[0, 1, 1]))
    qs.append(_pq(segs, ["w2", "w0", "w1"], 100, offsets=[2, 0, 1]))
    qs.append(_pq(segs, ["w7", "w5", "w6", "w4"], 100, offsets=[7, 5, 6, 4]))
    for slop in (0, 1, 2, 3):
        qs.append(_pq(segs, ["w1", "w0"], 100, offsets=[1, 0], slop=slop))
        qs.append(_pq(segs, ["v", "u"], 300, offsets=[1, 0], slop=slop))
        qs.append(_pq(segs, ["u", "v"], 300, offsets=[0, 1], slop=slop))
    qs.append(_pq(segs, ["w0", "w1"], 100, offsets=[0, 0], slop=1))
    qs.append(_pq(segs, ["w2", "w5"], 100, offsets=[0, 3], slop=2))
    # scoring: weight 0 (every doc ties), -1.5 and 1e4; a tf cache whose other rows and weights are NaN; average fieldnorms 1 and 1e6
    for ph in (["w0", "w1"], ["d257", "d128"], ["b0", "b1"]):
        base = _pq(segs, ph, 200, offsets=None if ph[0] != "d257" else [2, 5])
        nan = float("nan")
        qs += [_scored(base, weights=[w] + base[0]["weights"][1:]) for w in (0.0, -1.5, 1e4)]
        cache = np.full((len(ph), 256), nan, np.float32)
        cache[0] = M.tf_cache(np.float32(base[0]["avg_fieldnorm"][0]) * np.float32(1.7))
        qs.append(_scored(base, tf_cache=cache, weights=[base[0]["weights"][0]] + [nan] * (len(ph) - 1)))
        qs += [_scored(base, avg_fieldnorm=[a] * len(ph)) for a in (1.0, 1e6)]
    # ties: k of 1, 127, 128, 129 and 1024 over three segments of 3000 tied docs
    qs += [_pq(segs, ["t0", "t1"], k) for k in (1, 127, 128, 129, 1024)]
    # initial thresholds: a tied score, between two scores, -0.0, NaN and 1e9
    for ph in (["w0", "w1"], ["d257", "d128"], ["z0", "z1"]):
        base = _pq(segs, ph, 100, offsets=None if ph[0] != "d257" else [2, 5])
        scores = [np.float32(s) for s, _, _ in base_rows(base)]
        tied = next(s for i, s in enumerate(scores) if s < scores[0] and s in scores[i + 1:])
        lo = next(s for s in scores if s < scores[0])
        between = np.float32((np.float64(scores[0]) + np.float64(lo)) / 2)
        assert lo < between < scores[0]
        qs += [_scored(base, threshold=float(t)) for t in (tied, between, -0.0, float("nan"), 1e9)]
    # unions in the same batch
    qs += [_or(segs, ts, k) for ts in (["w0", "w1", "w2"], ["z0", "d257", "u"]) for k in (10, 100)]
    return qs


@pytest.fixture(scope="module")
def battery():
    rng = np.random.default_rng(2024)
    shapes = [PosSegment(_plant_texts(rng, n)) for n in (700, 450)]
    segs = [_streams_segment(rng), _df_segment(rng)] + shapes + [_deleted_copy(shapes[0], ["w0", "w1"], rng)]
    segs += _uv_segments(rng) + _tie_segments()

    def base_rows(q):
        vocab = sorted({t for s in segs for t in s.vocab})
        return M.search([s.model(vocab) for s in segs], q[0], [vocab.index(t) for t in q[1]])
    b = Battery(segs, _battery_queries(segs, base_rows))
    _battery_is_not_vacuous(b)
    return b


def _battery_is_not_vacuous(b):
    """The edges the battery is about are in its expected rows."""
    streams = b.segs[0]
    assert any((streams.ord, 0) == (g, d) for w in b.want for _, g, d in w)       # the doc with the 32-bit deltas matches
    assert any((streams.ord, 350) == (g, d) for w in b.want for _, g, d in w)     # the doc with 3000 occurrences matches
    ties = [s.ord for s in b.segs[-3:]]
    for k in (1, 127, 128, 129, 1024):
        i = next(i for i, q in enumerate(b.queries) if q.get("term_offset") is not None and q["k"] == k
                 and q["term_segs"][0][1] in ties and "threshold" not in q)
        assert [(g, d) for _, g, d in b.want[i]] == [(min(ties), d) for d in range(k)]  # the lowest (segment, doc) pairs
    for i, q in enumerate(b.queries):
        if q.get("threshold") is not None and q["threshold"] == q["threshold"]:  # (a NaN threshold is no threshold)
            assert all(s > np.float32(q["threshold"]) for s, _, _ in b.want[i])
    assert sum(len(w) for w in b.want) > 5000


ROUTES = {"side_stream": {}, "one_stream": dict(TQ_PHRASE_SIDE_STREAM=0), "no_tile": dict(TQ_TILE=0), "repeated": dict(TQ_TILE_PCAP=64)}


@pytest.mark.parametrize("route", list(ROUTES))
def test_phrase_battery_on_every_route(battery, route):
    c = battery.register(_ctx_with_env(**ROUTES[route]))
    try:
        g = c.search_batch(battery.qb)
        battery.check(g, route)
        st = c.stats()
        assert st["units_phrase"] > 0
        if route in ("side_stream", "one_stream"):
            assert st["tile_groups"] >= 1 and st["tile_fallbacks"] == 0
        if route == "no_tile":
            assert st["tile_groups"] == 0
        if route == "repeated":
            assert st["tile_fallbacks"] == 1
    finally:
        c.close()


@pytest.fixture(scope="module")
def ctx(battery):
    c = battery.register(T.Context(0))
    yield c
    c.close()


def test_phrase_battery_prepared_and_packed(battery, ctx):
    """prepare / run / fetch, and the packed device-resident rows of results_pack_dev_async."""
    import torch
    qb = battery.qb
    bt = ctx.prepare(qb)
    try:
        bt.run()
        rows = bt.fetch()
        battery.check(rows, "fetch")
        words = 3 * qb.nq * qb.kmax + qb.nq
        packed = torch.zeros(words + 4, dtype=torch.int32, device="cuda:0")
        bt.results_pack_dev_async(packed.data_ptr())
        torch.cuda.synchronize()
        p = packed.cpu().numpy()
        assert int(np.abs(p[words:]).max()) == 0  # the run did not overflow: the packed rows are final
        r = qb.nq * qb.kmax
        got = (p[:r].view(np.float32).reshape(qb.nq, qb.kmax), p[r:2 * r].view(np.uint32).reshape(qb.nq, qb.kmax),
               p[2 * r:3 * r].view(np.uint32).reshape(qb.nq, qb.kmax), p[3 * r:words].view(np.uint32))
        for a, b in zip(got, rows):
            assert (np.asarray(a)[:qb.nq] == np.asarray(b)[:qb.nq]).all()
    finally:
        bt.close()


def test_phrase_battery_phased_with_threshold_exchange(battery, ctx):
    """run_phase with the all-reduce-MAX threshold exchange between phases, then with the final k-th keys imported after phase 0
    (a valid foreign bound: phrase queries are not skipped by the import, so it prunes them too)."""
    import torch
    qb = battery.qb
    keys = torch.zeros(qb.nq, dtype=torch.int64, device="cuda:0")
    b = ctx.prepare(qb)
    try:
        n = b.phases()
        for phase in range(n):
            b.run_phase(phase)
            if phase + 1 < n:
                b.thresholds_export_dev(keys.data_ptr())
                b.thresholds_import_dev(keys.data_ptr())
        battery.check(b.fetch(), "phased")
        final = np.zeros(qb.nq, np.int64)
        for i, (q, w) in enumerate(zip(battery.queries, battery.want)):
            if len(w) == q["k"]:
                final[i] = score_keys([w[-1][0]])[0]
        b.run_phase(0)
        k2 = torch.from_numpy(final).to("cuda:0")
        b.thresholds_import_dev(k2.data_ptr())
        for phase in range(1, n):
            b.run_phase(phase)
        battery.check(b.fetch(), "final k-th keys imported")
    finally:
        b.close()


@pytest.mark.parametrize("shards", [1, 2])
def test_phrase_battery_topkeys_exchange(battery, ctx, shards):
    import torch
    qb = battery.qb
    kmax = qb.kmax
    keys = torch.zeros((shards, qb.nq, kmax), dtype=torch.int32, device="cuda:0")
    b = ctx.prepare(qb)
    try:
        for phase in range(b.phases()):
            b.run_phase(phase)
            if phase + 1 < b.phases():
                b.topkeys_export_dev(keys[0].data_ptr(), kmax)
                b.thresholds_from_keys_dev(keys.data_ptr(), shards, kmax)
        battery.check(b.fetch(), f"topkeys x{shards}")
    finally:
        b.close()


def test_phrase_clause_order_decides_left_of_a_sloppy_phrase(ctx):
    """One doc "a a b b", the phrase a@0 b@1 with slop 1 (equal doc_freq): passed as (a, 0), (b, 1) or as (b, 1), (a, 0) it is
    the same PhraseQuery, with phrase count 1 (left = a: shifted a = [1, 2], b = [2, 3]) -- the score of "a b" without slop."""
    seg = PosSegment.from_positions({"a": {0: [0, 1]}, "b": {0: [2, 3]}}, [4])
    seg.register(ctx)
    oi = O.OracleIndex()
    seg.register(oi)
    qs = [_pq([seg], ["a", "b"], 10, offsets=[0, 1], slop=1), _pq([seg], ["b", "a"], 10, offsets=[1, 0], slop=1), _pq([seg], ["a", "b"], 10)]
    qb = QueryBatch([q for q, _ in qs])
    g, c = ctx.search_batch(qb), oi.search_batch(qb, mode=0)
    want = M.search([seg.model(["a", "b"])], qs[2][0], [0, 1])
    assert len(want) == 1
    for i, (q, terms) in enumerate(qs):
        assert M.search([seg.model(["a", "b"])], q, [["a", "b"].index(t) for t in terms]) == want
        assert _bits(hits(g, i)) == _bits(want), ("device", i, hits(g, i))
        assert _bits(hits(c, i)) == _bits(want), ("oracle", i, hits(c, i))


def test_phrase_refusals(battery, ctx):
    """Nine terms: TQ_ERR_UNSUPPORTED.  Count of a phrase: TQ_ERR_INVALID_ARGUMENT, no count.  The context stays usable."""
    segs = battery.segs
    q9, _ = _pq(segs, [f"w{i}" for i in range(8)] + ["w0"], 10)
    with pytest.raises(T.TqError, match=r"error -4\b"):
        ctx.search_batch(QueryBatch([q9]))
    with pytest.raises(T.TqError, match=r"error -1\b"):
        ctx.count_batch(QueryBatch([battery.queries[0]]))
    g = ctx.search_batch(QueryBatch(battery.queries[:4]))
    for i in range(4):
        assert _bits(hits(g, i)) == _bits(battery.want[i])


def _merged(parts, nq, k):
    return merge_rows_host(*[np.stack([np.asarray(p[j])[:nq] for p in parts]) for j in range(4)], k)


def _assert_rows(m, want, queries):
    """Merged rows (kept up to the batch's largest k) against the expected rows of each query."""
    for i, (w, q) in enumerate(zip(want, queries)):
        n = min(int(m[3][i]), q["k"])
        got = [(float(m[0][i, j]), int(m[1][i, j]), int(m[2][i, j])) for j in range(n)]
        assert _bits(got) == _bits(w), (i, got[:4], w[:4])


def test_phrase_segments_over_two_contexts_with_topkeys_exchange(battery):
    """Two contexts holding different segments, run phase by phase with the top-keys exchange between them (each exports its k
    best keys, both take the thresholds of the gathered keys): their rows merged like segment fruits are the whole battery's."""
    import torch
    segs = battery.segs
    halves = [segs[0::2], segs[1::2]]
    ctxs, batches, qbs = [], [], []
    try:
        for half in halves:
            c = T.Context(0)
            ctxs.append(c)
            for s in half:
                s.register(c)
            mine = {s.ord for s in half}
            qs = []
            for q in battery.queries:
                keep = [i for i, ts in enumerate(q["term_segs"]) if ts[1] in mine]
                q2 = dict(q, term_segs=[q["term_segs"][i] for i in keep])
                if "term_pos" in q:
                    q2["term_pos"] = [q["term_pos"][i] for i in keep]
                qs.append(q2)
            qbs.append(QueryBatch(qs))
            batches.append(c.prepare(qbs[-1]))
        nq, kmax = battery.qb.nq, battery.qb.kmax
        keys = torch.zeros((2, nq, kmax), dtype=torch.int32, device="cuda:0")
        n = max(b.phases() for b in batches)
        for phase in range(n):
            for b in batches:
                if phase < b.phases():
                    b.run_phase(phase)
            if phase + 1 < n:
                for r, b in enumerate(batches):
                    b.topkeys_export_dev(keys[r].data_ptr(), kmax)
                torch.cuda.synchronize()
                for b in batches:
                    b.thresholds_from_keys_dev(keys.data_ptr(), 2, kmax)
                torch.cuda.synchronize()
        parts = [b.fetch() for b in batches]
        _assert_rows(_merged(parts, nq, kmax), battery.want, battery.queries)
    finally:
        for b in batches:
            b.close()
        for c in ctxs:
            c.close()


def _big_segment(alive):
    """300k docs: g0 / g1 / g2 at base + 0 / 1 / 2 in a fifth / a tenth / a twentieth of the docs, some twice."""
    rng = np.random.default_rng(99)
    n = 300_000
    base = rng.integers(0, 30, size=n)
    p = {}
    for t, dens in enumerate((0.2, 0.1, 0.05)):
        docs = np.nonzero(rng.random(n) < dens)[0].tolist()
        twice = (rng.random(len(docs)) < 0.3).tolist()
        p[f"g{t}"] = {d: [int(base[d]) + t] + ([int(base[d]) + t + 40] if tw else []) for d, tw in zip(docs, twice)}
    return PosSegment.from_positions(p, rng.integers(5, 80, size=n), alive=alive)


@pytest.mark.parametrize("deletes", [False, True])
def test_phrase_doc_range_parts_merge_to_the_whole_segment(deletes):
    """tq_segment_set_doc_range with positions registered: each part (one context each) returns the rows of its docs; merged they
    are the rows of one context holding the whole segment, which are the model's."""
    alive = np.packbits(np.random.default_rng(5).random(300_000) > 0.3, bitorder="little") if deletes else None
    seg = _big_segment(alive)
    segs = [seg]
    qs = [_pq(segs, ph, k, offsets=off, slop=slop) for ph, off, slop in
          ((["g0", "g1"], None, 0), (["g1", "g2"], None, 0), (["g0", "g1", "g2"], None, 0), (["g2", "g0"], [2, 0], 0),
           (["g1", "g0"], [1, 0], 2), (["g0", "g2"], [0, 2], 1)) for k in (10, 100)]
    qs += [_or(segs, ["g0", "g2"], 50)]
    vocab = seg.vocab
    want = [M.search([seg.model(vocab)], q, [vocab.index(t) for t in terms]) for q, terms in qs]
    qb = QueryBatch([q for q, _ in qs])
    c = T.Context(0)
    try:
        seg.register(c)
        g = c.search_batch(qb)
        for i, w in enumerate(want):
            assert _bits(hits(g, i)) == _bits(w), i
    finally:
        c.close()
    for cuts in DOC_RANGE_CUTS:
        parts = []
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            c = T.Context(0)
            try:
                seg.register(c)
                c.segment_set_doc_range(seg.ord, 0, lo, hi)
                r = c.search_batch(qb)
                for i in range(qb.nq):
                    assert all(lo <= d < hi for _, _, d in hits(r, i))
                parts.append([np.array(x) for x in r])
            finally:
                c.close()
        _assert_rows(_merged(parts, qb.nq, qb.kmax), want, [q for q, _ in qs])
