"""The sharded search path against the independent score model (tests/score_model.py), on one GPU: every rank is a thread with a
Context of its own, and an in-process process group moves the tensors between them.

  * CrossGpuMerger (tantivy_b200/sharding.py) at 2, 3, 4 and 8 ranks, with the default number of exchanged keys per query and with
    one: the merged rows equal the rows of one search over the whole index, and every exchanged key is a key of a doc the rank holds;
  * two batches in flight (run / finish_async / complete), with one rank overflowing its tile buffers, one rank with several tile
    groups, and with the per-query kernels only;
  * k_merge (tq_merge_topk_dev, tq_merge_topk_packed_dev) on synthetic rows, and k_theta_from_keys on synthetic keys;
  * tq_multi over three and four contexts on the same index.
Scores are compared bit for bit, except that a zero score is compared by value: the device returns +0.0 for -0.0 (partial_cmp ties
them, sort_by_score.rs:99-107)."""
import collections
import os
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import tantivy_b200 as T  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM, QueryBatch  # noqa: E402
from tantivy_b200.sharding import CrossGpuMerger, assign_parts, doc_range  # noqa: E402
from tests import score_model as M  # noqa: E402
from tests.helpers import OracleSegment, bool_shape_query, make_query, random_bool_shapes  # noqa: E402

DEV = "cuda:0"
N_TERMS = 8
HOT = (0, 1)     # terms whose best docs all sit in the first 2048 docs of segment 0
ZERO = (4, 5)    # the signed-zero clauses: term 5 holds the lower docs of every segment, term 4 the upper ones
ONE_SEG = 7      # postings in segment 1 only
NOWHERE = 6      # postings in no segment


def key(score):
    """Order-preserving u32 key of an f32 score, -0.0 and +0.0 on one key; 0 is below every score's key."""
    u = int((np.float32(score) + np.float32(0)).view(np.uint32))
    return u ^ 0xFFFFFFFF if u >> 31 else u | 0x80000000


def _ctx_with_env(**env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return T.Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _rows(q_rows):
    """Model rows -> comparable tuples (zero scores by value)."""
    return [(float(s), int(g), int(d)) for s, g, d in q_rows]


# ---- the index ---------------------------------------------------------------------------------------------------------------
class Index:
    """Four segments (ordinals 0..3) for the GPU (OracleSegment bodies) and for the model:
      0 "hot": 6000 docs; the first 2048 are one-token docs with tf 8-12 of the HOT terms, so one shard holds the whole global
        top-k of the queries over them (more than the keys it exchanges);
      1 with deletes (a fifth of the docs), the only one with postings of ONE_SEG;
      2 without fieldnorms and tf 1-2: thousands of exactly tied scores, inside the segment and across its doc-range parts;
      3 small: 300 docs."""

    def __init__(self):
        rng = np.random.default_rng(0x5A4D)
        specs = [(6000, True, False), (5000, True, True), (4000, False, False), (300, True, False)]
        self.osegs, self.msegs = [], []
        for so, (n, norms, deletes) in enumerate(specs):
            lengths = np.clip(np.round(np.exp(rng.normal(np.log(30), 0.8, size=n))), 1, 2000).astype(np.uint32) if norms else None
            lists = []
            for t in range(N_TERMS):
                if t in ZERO:
                    docs = np.arange(n // 2, n) if t == ZERO[0] else np.arange(0, n // 2)
                    docs = docs[rng.random(len(docs)) < 0.3]
                else:
                    p = np.full(n, (0.25, 0.12, 0.3, 0.05, 0, 0, 0.1, 0.2)[t])
                    if so == 0 and t in HOT:
                        p[:2048] = 0.6
                    docs = np.nonzero(rng.random(n) < p)[0]
                tfs = rng.geometric(0.6, size=len(docs)).clip(1, 2 if not norms else 20)
                if so == 0 and t in HOT:
                    hot = docs < 2048
                    tfs[hot] = rng.integers(8, 13, size=int(hot.sum()))
                    tfs[~hot] = 1
                lists.append((docs.astype(np.uint32), tfs.astype(np.uint32)))
            if so == 0:
                lengths[:2048] = 1
                lengths[2048:] = np.maximum(lengths[2048:], 20)
            alive = np.packbits(rng.random(n) > 0.2, bitorder="little") if deletes else None
            o = OracleSegment(lists, lengths, segment_ord=so, alive=alive, max_doc=None if norms else n)
            for t in range(N_TERMS):
                if t == NOWHERE or (t == ONE_SEG and so != 1):
                    o.terms[t] = (0, 0, 0)
            self.osegs.append(o)
            self.msegs.append(M.Segment(so, lists, lengths, alive=alive, max_doc=None if norms else n))
        self.queries, self.terms = self._queries(rng)

    def _queries(self, rng):
        qs = []

        def add(q, terms):
            qs.append((q, list(terms)))

        o = self.osegs
        for t, k in ((0, 10), (1, 1000), (3, 129), (ONE_SEG, 100), (NOWHERE, 10), (2, 1024)):
            add(make_query(TQ_OP_TERM, o, [t], k), [t])
        for ts, k in (([0, 1], 100), ([1, 2, 3], 1024), ([0, 2], 1), ([0, 1], 128), ([2, 3, ONE_SEG], 10)):
            add(make_query(TQ_OP_AND, o, ts, k), ts)
        wide = [0, 1, 2, 3, 4, 5, ONE_SEG, 0, 3, 1]  # > 8 clauses
        for ts, k in (([0, 1, 2], 128), ([2, 3, ONE_SEG], 1000), ([0, 1], 129), (wide, 100), (wide, 1024), ([3, NOWHERE], 10),
                      ([0, 1, 3, 2], 1)):
            add(make_query(TQ_OP_OR, o, ts, k), ts)
        # signed zeros: +0.0 OR -0.0 (the -0.0 clause holds the lower docs); -0.0 alone; -0.0 beside a +0.0 term of one segment
        for k in (1, 129, 1000):
            q = make_query(TQ_OP_OR, o, list(ZERO), k)
            q["weights"] = [0.0, -0.0]
            add(q, ZERO)
        q = make_query(TQ_OP_TERM, o, [ZERO[1]], 100)
        q["weights"] = [-0.0]
        add(q, [ZERO[1]])
        q = make_query(TQ_OP_OR, o, [ZERO[1], ONE_SEG], 1024)
        q["weights"] = [-0.0, 0.0]
        add(q, [ZERO[1], ONE_SEG])
        self.n_plain = len(qs)
        for sh in random_bool_shapes(rng, 8, 4, n_wide=1):  # (terms 0-3: postings in every segment)
            add(bool_shape_query(o, sh), sh["terms"])
        return [q for q, _ in qs], [t for _, t in qs]

    def want(self, queries=None, terms=None):
        queries, terms = queries or self.queries, terms or self.terms
        return [_rows(M.search(self.msegs, q, t)) for q, t in zip(queries, terms)]


@pytest.fixture(scope="module")
def index():
    ix = Index()
    want = ix.want()
    # (not vacuous: the hot queries fill k from segment 0's first docs, the zero queries hold both zeros, ties abound)
    assert len(want[1]) == 1000 and all(g == 0 and d < 2048 for _, g, d in want[1])
    assert sum(len(w) for w in want) > 5000 and want[4] == [] and {g for _, g, _ in want[3]} == {1}
    return ix, want


# ---- shards ------------------------------------------------------------------------------------------------------------------
def rank_units(ix, world, rank):
    """[(segment ordinal, doc range [lo, hi) or None: the whole segment)] of a rank: segments round-robin (world 3: two, one and one),
    or with more ranks than segments every segment split by doc range (world 8: halves)."""
    return [(s, None if n == 1 else doc_range(ix.msegs[s].max_doc, p, n)) for s, p, n in assign_parts(4, world, rank)]


def rank_queries(queries, units):
    mine = {s for s, _ in units}
    return [dict(q, term_segs=[ts for ts in q["term_segs"] if ts[1] in mine]) for q in queries]


def register(ix, ctx, units):
    for s, r in units:
        ix.osegs[s].register(ctx)
        if r is not None:
            ctx.segment_set_doc_range(s, 0, r[0], r[1])


def rank_model(ix, units, q, terms, k=None):
    segs = [ix.msegs[s] for s, _ in units]
    ranges = {s: r for s, r in units if r is not None}
    return M.search(segs, dict(q, k=k or q["k"]), terms, doc_ranges=ranges)


class FakeDist:
    """all_gather_into_tensor between threads of one process: each rank synchronises its current stream, publishes a copy of its
    input in a new slot per collective, waits for every rank at a barrier and copies every slot into its output on its current
    stream.  A rank that fails breaks the barrier, so no thread waits for it.  Every gathered key tensor is recorded."""

    def __init__(self, world):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=120)
        self.lock = threading.Lock()
        self.slots = collections.defaultdict(lambda: [None] * world)
        self.calls = [0] * world
        self.keys = {}  # collective index -> [world, nq, kx] numpy (uint32)

    def rank(self, r):
        d = self

        class View:
            def get_world_size(self):
                return d.world

            def all_gather_into_tensor(self, out, inp):
                d.gather(r, out, inp)
        return View()

    def gather(self, r, out, inp):
        s = torch.cuda.current_stream()
        s.synchronize()
        i = self.calls[r]
        self.calls[r] += 1
        mine = inp.clone()
        s.synchronize()
        with self.lock:
            self.slots[i][r] = mine
        self.barrier.wait()
        slot = self.slots[i]
        for j in range(self.world):
            out[j].copy_(slot[j].view(out[j].shape))
        if inp.dim() == 2:  # the threshold exchange's [nq, kx] keys (result rows are 1-D)
            s.synchronize()
            with self.lock:
                self.keys.setdefault(i, torch.stack(slot).cpu().numpy().view(np.uint32))
        self.barrier.wait()  # (every rank has read slot i)


def run_ranks(world, fn):
    """fn(rank, dist view) on one thread per rank; re-raises the first failure after every thread has ended."""
    d = FakeDist(world)
    errors = [None] * world

    def body(r):
        try:
            fn(r, d.rank(r))
        except BaseException as e:  # noqa: BLE001
            errors[r] = e
            d.barrier.abort()

    threads = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in threads)
    first = next((e for e in errors if e is not None and not isinstance(e, threading.BrokenBarrierError)), None) or next(
        (e for e in errors if e is not None), None)
    if first is not None:
        raise first
    return d


def merged_rows(m, nq):
    sc, sg, dc, ct = m
    return [[(float(sc[q, j]), int(sg[q, j]), int(dc[q, j])) for j in range(int(ct[q]))] for q in range(nq)]


def assert_rows(got, want, queries, what):
    for q, (g, w) in enumerate(zip(got, want)):
        assert len(g) <= queries[q]["k"], (what, q, len(g), queries[q]["k"])
        assert g == w, (what, q, queries[q]["op"], queries[q]["k"], g[:4], w[:4])


@pytest.fixture(scope="module")
def theta_ctx(index):
    """One context holding the whole index."""
    c = T.Context(0)
    for o in index[0].osegs:
        o.register(c)
    yield c
    c.close()


# ---- a. CrossGpuMerger against the model ---------------------------------------------------------------------------------------
def _check_exchanges(d, world, all_keys, queries, want, kx):
    """Every exchange: per rank at most min(k, kx) keys, a sub-multiset of the keys of the rank's alive matching docs (all_keys[rank,
    query], descending; so, sorted, each key is below the same place of the rank's own top list), and the union's k-th key <= the
    global k-th key.  Returns how many bounds were below the global k-th key."""
    inexact = 0
    assert d.keys, "no threshold exchange ran"
    for g in d.keys.values():
        assert g.shape == (world, len(queries), kx)
        for q, qq in enumerate(queries):
            k = qq["k"]
            union = []
            for r in range(world):
                nz = sorted((int(x) for x in g[r, q] if x), reverse=True)
                assert len(nz) <= min(k, kx), (world, r, q, len(nz))
                have = collections.Counter(all_keys[r, q])
                have.subtract(collections.Counter(nz))
                assert min(have.values(), default=0) >= 0, (world, r, q, "a key of no doc of the rank", nz[:4])
                assert all(a <= b for a, b in zip(nz, all_keys[r, q])), (world, r, q)
                union += nz
            union.sort(reverse=True)
            bound = union[k - 1] if len(union) >= k else 0
            exact = key(want[q][k - 1][0]) if len(want[q]) >= k else 0
            assert bound <= exact, (world, q, bound, exact)
            inexact += bound < exact
    return inexact


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_merger_matches_the_model(index, world, monkeypatch):
    """Segments (world 8: doc-range halves of segments) spread over `world` ranks; run + __call__ + fetch_host on every rank gives
    the model's rows over the whole index, with each query's own k, for the default number of exchanged keys and for one."""
    ix, want = index
    units_of = [rank_units(ix, world, r) for r in range(world)]
    assert sorted(s for u in units_of for s, _ in u) == sorted(s for s in range(4) for _ in range(1 if world <= 4 else 2))
    rank_keys = {(r, q): sorted((key(s) for s, _, _ in rank_model(ix, units_of[r], qq, t, k=10 ** 7)), reverse=True)
                 for r in range(world) for q, (qq, t) in enumerate(zip(ix.queries, ix.terms))}
    ctxs = [T.Context(0) for _ in range(world)]
    try:
        for r in range(world):
            register(ix, ctxs[r], units_of[r])
        qbs = [QueryBatch(rank_queries(ix.queries, units_of[r])) for r in range(world)]
        for keys_env in (None, "1"):
            if keys_env is None:
                monkeypatch.delenv("TANTIVY_B200_EXCHANGE_KEYS", raising=False)
            else:
                monkeypatch.setenv("TANTIVY_B200_EXCHANGE_KEYS", keys_env)
            got, kxs = [None] * world, [None] * world

            def rank(r, dist):
                b = ctxs[r].prepare(qbs[r])
                try:
                    m = CrossGpuMerger(ctxs[r], dist, DEV, qbs[r].nq, qbs[r].kmax)
                    kxs[r] = m.kx
                    m.run(b)
                    m(b)
                    got[r] = merged_rows(m.fetch_host(b), qbs[r].nq)
                finally:
                    b.close()
            d = run_ranks(world, rank)
            for r in range(world):
                assert_rows(got[r], want, ix.queries, f"world {world} rank {r} keys {keys_env}")
            kx = kxs[0]
            assert kx == (1 if keys_env else (1024 if world <= 2 else min(1024, (2048 + world - 1) // world + 8)))
            inexact = _check_exchanges(d, world, rank_keys, ix.queries, want, kx)
            assert inexact > 0  # the bound is below the global k-th for some query (a shard held more than kx of the top-k)
    finally:
        for c in ctxs:
            c.close()


def test_merger_refuses_a_batch_of_another_shape(index):
    """The merger reads the packed rows at stride k: a batch whose largest k or query count differs is refused."""
    ix, _ = index
    c = T.Context(0)
    try:
        for o in ix.osegs:
            o.register(c)
        qb = QueryBatch(ix.queries[:ix.n_plain])
        b = c.prepare(qb)
        d = FakeDist(1).rank(0)
        for nq, k in ((qb.nq, qb.kmax - 1), (qb.nq + 1, qb.kmax), (qb.nq - 1, qb.kmax)):
            m = CrossGpuMerger(c, d, DEV, nq, k)
            with pytest.raises(ValueError, match="cannot merge"):
                m.run(b)
            with pytest.raises(ValueError, match="cannot merge"):
                m.finish_async(b)
            b.run()
            with pytest.raises(ValueError, match="cannot merge"):
                m(b)
        b.close()
    finally:
        c.close()


# ---- b. two batches in flight ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["default", "one_rank_overflows", "one_rank_many_groups", "per_query_kernels"])
def test_two_batches_in_flight(index, variant):
    """Per rank two mergers A and B: run(A), finish_async(A), run(B), finish_async(B), complete(A), complete(B) -- both row sets
    exact.  One rank with a tiny tile buffer (TQ_TILE_PCAP=64) overflows: every rank repeats once.  One rank's planner opens
    several tile groups (at most three queries of a segment per group; the key export reads group 0's samples after phase 0).  TQ_TILE=0: the per-query kernels."""
    ix, want = index
    world = 3
    units_of = [rank_units(ix, world, r) for r in range(world)]
    env = [dict() for _ in range(world)]
    if variant == "one_rank_overflows":
        env[1] = dict(TQ_TILE=1, TQ_TILE_PCAP=64)
    elif variant == "one_rank_many_groups":
        env[0] = dict(TQ_TILE=1, TQ_TILE_MAX_QUERIES=3)
    elif variant == "per_query_kernels":
        env = [dict(TQ_TILE=0) for _ in range(world)]
    n = ix.n_plain if variant == "per_query_kernels" else len(ix.queries)  # (TQ_OP_BOOL needs the tile engine)
    qa = ix.queries[:n]
    qb_ = [dict(q, k=max(1, q["k"] // 2 + 1)) for q in qa]  # B: other k, other rows
    want_b = [_rows(M.search(ix.msegs, q, t)) for q, t in zip(qb_, ix.terms[:n])]
    ctxs = [_ctx_with_env(**e) for e in env]
    got, repeats, stats = [None] * world, [None] * world, [None] * world
    try:
        for r in range(world):
            register(ix, ctxs[r], units_of[r])
        batches = [(QueryBatch(rank_queries(qa, units_of[r])), QueryBatch(rank_queries(qb_, units_of[r]))) for r in range(world)]

        def rank(r, dist):
            a, b = (ctxs[r].prepare(x) for x in batches[r])
            try:
                ma = CrossGpuMerger(ctxs[r], dist, DEV, n, batches[r][0].kmax)
                mb = CrossGpuMerger(ctxs[r], dist, DEV, n, batches[r][1].kmax)
                ma.run(a)
                ma.finish_async(a)
                mb.run(b)
                mb.finish_async(b)
                ra = ma.complete(a)
                rb = mb.complete(b)
                got[r] = (merged_rows(ra, n), merged_rows(rb, n))
                repeats[r] = (ma.repeats, mb.repeats)
                stats[r] = ctxs[r].stats()
            finally:
                a.close()
                b.close()
        run_ranks(world, rank)
    finally:
        for c in ctxs:
            c.close()
    for r in range(world):
        assert_rows(got[r][0], want[:n], qa, f"{variant} rank {r} A")
        assert_rows(got[r][1], want_b, qb_, f"{variant} rank {r} B")
    assert len(set(repeats)) == 1, repeats  # every rank takes the same decision (ties at k = 1024 may overflow a candidate region)
    if variant == "one_rank_overflows":
        assert repeats[0][0] == 1, repeats
    if variant == "per_query_kernels":  # (they cannot overflow)
        assert repeats[0] == (0, 0), repeats
    if variant == "one_rank_many_groups":
        assert stats[0]["tile_groups"] > 1
    if variant == "per_query_kernels":
        assert all(st["tile_groups"] == 0 for st in stats)


# ---- d. k_merge on synthetic rows ----------------------------------------------------------------------------------------------
_POOL = np.array([7.5, 3.25, 1.0, 1e-30, 1e-40, 1.4e-45, 0.0, -0.0, -1.4e-45, -2.0, -1e30, np.inf, -np.inf, 3.25, 1.0], np.float32)


def _synthetic_lists(rng, n_lists, nq, stride, k):
    """Per list and query: rows sorted like k_final's output (scores from _POOL: negative, subnormal, +-inf, +-0.0, exact ties
    across lists; segment ords 0-2, the same ord in several lists as from doc-range parts; docs unique per ord) and a count of
    0, < k, = stride or > stride."""
    sc = np.zeros((n_lists, nq, stride), np.float32)
    sg = np.zeros((n_lists, nq, stride), np.uint32)
    dc = np.zeros((n_lists, nq, stride), np.uint32)
    ct = np.zeros((n_lists, nq), np.uint32)
    lists = [[None] * nq for _ in range(n_lists)]
    for q in range(nq):
        docs = rng.permutation(3 * n_lists * stride)  # (unique (ord, doc) over the lists)
        for l in range(n_lists):
            c = [0, max(0, k - 1 - l % 3), stride, stride + 5, int(rng.integers(0, stride + 1))][(l + q) % 5]
            n = min(c, stride)
            rows = [(float(_POOL[rng.integers(len(_POOL))]), int(rng.integers(3)), int(docs[l * stride + i])) for i in range(n)]
            rows = M.merge_fruits([rows], n)
            sc[l, q, :n] = [r[0] for r in rows]
            sg[l, q, :n] = [r[1] for r in rows]
            dc[l, q, :n] = [r[2] for r in rows]
            ct[l, q] = c
            lists[l][q] = rows
    want = [M.merge_fruits([lists[l][q] for l in range(n_lists)], k) for q in range(nq)]
    return (sc, sg, dc, ct), want


@pytest.mark.parametrize("k", [1, 2, 129, 1024])
@pytest.mark.parametrize("n_lists", [1, 2, 3, 8, 16])
def test_k_merge_synthetic_rows(n_lists, k):
    rng = np.random.default_rng(1000 * n_lists + k)
    nq, stride = 5, k + 3
    (sc, sg, dc, ct), want = _synthetic_lists(rng, n_lists, nq, stride, k)
    assert any(len(w) == k for w in want) or n_lists == 1
    c = T.Context(0)
    try:
        t = [torch.from_numpy(x.view(np.int32).copy()).to(DEV) for x in (sc, sg, dc, ct)]
        out = [torch.full((nq, stride), -1, dtype=torch.int32, device=DEV) for _ in range(3)] + [torch.zeros(nq, dtype=torch.int32, device=DEV)]
        torch.cuda.synchronize()
        c.merge_topk_dev(n_lists, nq, stride, k, *[x.data_ptr() for x in t], *[x.data_ptr() for x in out])
        o = [x.cpu().numpy() for x in out]
        plain = merged_rows((o[0].view(np.float32), o[1].view(np.uint32), o[2].view(np.uint32), o[3].view(np.uint32)), nq)
        # packed: one buffer per list, pitch_words larger than the packed size
        words = 3 * nq * stride + nq
        pitch = words + 37
        packed = np.full((n_lists, pitch), 0x7F7F7F7F, np.uint32)
        for l in range(n_lists):
            packed[l, :words] = np.concatenate([sc[l].reshape(-1).view(np.uint32), sg[l].reshape(-1), dc[l].reshape(-1), ct[l]])
        p = torch.from_numpy(packed.view(np.int32)).to(DEV)
        po = torch.zeros(words, dtype=torch.int32, device=DEV)
        torch.cuda.synchronize()
        c.merge_topk_packed_dev(0, n_lists, nq, stride, k, p.data_ptr(), pitch, po.data_ptr())
        torch.cuda.synchronize()
        a = po.cpu().numpy().view(np.uint32)
        r = nq * stride
        packed_rows = merged_rows((a[:r].view(np.float32).reshape(nq, stride), a[r:2 * r].reshape(nq, stride), a[2 * r:3 * r].reshape(nq, stride), a[3 * r:]), nq)
    finally:
        c.close()
    for q in range(nq):
        assert plain[q] == want[q], (q, plain[q][:6], want[q][:6])
        assert packed_rows[q] == want[q], (q, packed_rows[q][:6], want[q][:6])
        assert all(not np.signbit(s) for s, _, _ in plain[q] if s == 0)  # a zero comes back as +0.0


# ---- e. k_theta_from_keys on synthetic keys -------------------------------------------------------------------------------------
_THETA_KS = [1, 10, 129, 1000, 1024]


def _key_pattern(rng, pattern, n, k):
    if pattern == "equal":
        v = np.full(n, 0xE1234567, np.uint32)
    elif pattern == "low_byte":
        v = (0xF0ABCD00 + rng.integers(0, 256, size=n)).astype(np.uint32)
    elif pattern == "top_byte":
        v = ((rng.integers(0xC8, 0xF1, size=n) << 24) | 0x00123456).astype(np.uint32)
    elif pattern == "k_minus_1":
        v = rng.integers(0xC8000000, 0xF0000000, size=n).astype(np.uint32)
        if n >= k:
            v[rng.permutation(n)[:n - (k - 1)]] = 0
    else:  # "inf": the key of +inf among others
        v = rng.integers(0xC8000000, 0xF0000000, size=n).astype(np.uint32)
        v[rng.permutation(n)[:max(1, n // 3)]] = key(np.inf)
    return v


@pytest.mark.parametrize("shards,k_stride", [(1, 1), (1, 1024), (2, 129), (3, 100), (7, 10), (50, 1), (16, 700), (50, 1024)])
def test_theta_from_synthetic_keys(index, theta_ctx, shards, k_stride):
    """Between phases 0 and 1: import a synthetic [shards, nq, k_stride] key array; the threshold becomes max(before, the k-th
    largest key of the union), or stays when the union has fewer than k non-zero keys.  50 x 1024 keys are exactly the limit."""
    ix, _ = index
    c = theta_ctx
    qs = [make_query(TQ_OP_OR, ix.osegs, [0, 1, 2], k) for k in _THETA_KS]
    rng = np.random.default_rng(shards * 7919 + k_stride)
    moved = 0
    for pattern in ("equal", "low_byte", "top_byte", "k_minus_1", "inf"):
        g = np.zeros((shards, len(qs), k_stride), np.uint32)
        kth = []
        for q, k in enumerate(_THETA_KS):
            v = _key_pattern(rng, pattern, shards * k_stride, k)
            g[:, q, :] = v.reshape(shards, k_stride)
            s = np.sort(v)[::-1]
            kth.append(int(s[k - 1]) if len(s) >= k else 0)
        b = c.prepare(QueryBatch(qs))
        try:
            b.run_phase(0)
            before = torch.zeros(len(qs), dtype=torch.int64, device=DEV)
            after = torch.zeros(len(qs), dtype=torch.int64, device=DEV)
            b.thresholds_export_dev(before.data_ptr())
            gd = torch.from_numpy(g.view(np.int32)).to(DEV)
            torch.cuda.synchronize()
            b.thresholds_from_keys_dev(gd.data_ptr(), shards, k_stride)
            b.thresholds_export_dev(after.data_ptr())
            bf, af = before.cpu().numpy(), after.cpu().numpy()
        finally:
            b.close()
        for q in range(len(qs)):
            assert int(af[q]) == max(int(bf[q]), kth[q]), (pattern, q, hex(int(bf[q])), hex(int(af[q])), hex(kth[q]))
            moved += int(af[q]) != int(bf[q])
    assert moved > 0


def test_theta_from_keys_refuses_more_than_one_cta_holds(index, theta_ctx):
    """More than 200 KB of keys per query (one CTA's shared memory) is refused, not cut."""
    ix, _ = index
    b = theta_ctx.prepare(QueryBatch([make_query(TQ_OP_OR, ix.osegs, [0, 1], 10)]))
    try:
        b.run_phase(0)
        g = torch.zeros(51 * 1024, dtype=torch.int32, device=DEV)
        for shards, k_stride in ((51, 1024), (50, 1025), (1, 51201)):
            with pytest.raises(T.TqError, match="too large for one CTA"):
                b.thresholds_from_keys_dev(g.data_ptr(), shards, k_stride)
    finally:
        b.close()


# ---- f. tq_multi on the same index ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_ctx", [3, 4])
def test_multi_handle_matches_the_model_and_the_merger(index, n_ctx):
    """tq_multi over n_ctx contexts of device 0 (segments round-robin, its own key exchange and host merge): the model's rows, so
    the same rows CrossGpuMerger gives at that world."""
    ix, want = index
    m = T.MultiContext([0] * n_ctx)
    try:
        for o in ix.osegs:
            m.segment_register(o.segment_ord, 0, o.max_doc, o.record_option, o.body, o.fn_ids, o.alive, device_index=o.segment_ord % n_ctx)
        qb = QueryBatch(ix.queries)
        got = merged_rows(m.search_batch(qb), qb.nq)
    finally:
        m.close()
    assert_rows(got, want, ix.queries, f"tq_multi x{n_ctx}")
