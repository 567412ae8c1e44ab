"""k_tile's union-only instances: a group whose queries are all term queries and unions runs k_tile<*, *, true> (no conjunction
or TQ_OP_BOOL code, each work-list segment's query state broadcast to its posting lanes); the same queries in a group with a
conjunction run the general instance.  Both must return the oracle's exhaustive rows, bit for bit, on the default route, with the
work list deferring pairs to further routing rounds, and with every union pair on the window path (B3)."""
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from oracle import tq_oracle as O  # noqa: E402
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM, QueryBatch  # noqa: E402
from tests.helpers import hits  # noqa: E402
from tests.test_gpu_parity import _ctx_with_env, assert_same  # noqa: E402

_DENS = [0.3, 0.15, 0.05, 0.01, 0.002, 0.0001]
_BASE = 9100


@pytest.fixture(scope="module")
def synth():
    ix = T.SynthIndex(3, 1_000_000, _DENS, seed=91)
    oi = O.OracleIndex()
    ix.register(oi, segment_base=_BASE)
    return ix, oi


def _unions(ix):
    qs = [ix.query(TQ_OP_OR, terms, k, segment_base=_BASE)
          for k in (1, 10, 100, 1000) for terms in ([0, 5], [0, 4, 5], [1, 0, 5, 3], [5, 4, 3, 2, 1, 0], [2, 3, 4], [0, 1])]
    return qs + [ix.query(TQ_OP_TERM, [t], k, segment_base=_BASE) for t in (0, 3, 5) for k in (10, 100)]


_HOOKS = [dict(), dict(TQ_TILE_SEG_CAP=3), dict(TQ_TILE_LIGHT_MAX=0)]


@pytest.mark.parametrize("hook", _HOOKS, ids=lambda h: ",".join(f"{k}={v}" for k, v in h.items()) or "default")
@pytest.mark.parametrize("counters", [0, 1])
def test_unions_alone_and_beside_a_conjunction(synth, hook, counters):
    ix, oi = synth
    unions = _unions(ix)
    qb_u = QueryBatch(unions)
    qb_m = QueryBatch(unions + [ix.query(TQ_OP_AND, [0, 2], 100, segment_base=_BASE)])  # the group now runs the general instance
    want = oi.search_batch(qb_m, mode=0, n_threads=16)
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, TQ_TILE_COUNTERS=counters, **hook)
    try:
        ix.register(c, segment_base=_BASE)
        g_u = c.search_batch(qb_u)
        st = c.stats()
        assert st["tile_groups"] >= 1 and st["tile_fallbacks"] == 0
        if counters:
            ctr, cyc = st["tile_counters"], st["tile_cycles"]
            assert ctr[2] > 0 and ctr[4] > 0  # light pairs and essential postings went through B2 ...
            if "TQ_TILE_LIGHT_MAX" in hook:
                assert ctr[3] > 0  # ... and heavy pairs through B3
            assert cyc[1] > 0 and cyc[3] > 0  # stage cycles: A and B2 ran
        g_m = c.search_batch(qb_m)
        assert c.stats()["tile_fallbacks"] == 0
    finally:
        c.close()
    assert_same(g_m, want, qb_m.nq)
    assert_same(g_u, want, qb_u.nq)
    for i in range(qb_u.nq):
        assert hits(g_u, i) == hits(g_m, i), f"query {i}: the union-only and the general instance differ"
    assert sum(1 for i in range(qb_u.nq) if hits(g_u, i)) >= qb_u.nq // 2
