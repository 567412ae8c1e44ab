"""k_tile's running threshold: inside the exact launches each query's threshold rises to the k-th of its pushed candidates' keys,
read from a histogram of those keys (tile_push counts, tile_theta_refresh reads it after the tile).  Rows must stay the oracle's
exhaustive rows, bit for bit, and every threshold a phase leaves must stay at or below the final k-th key: at k = 1 .. 1024, with
many docs tied at the k-th score (Basic fields, ignore-freq), with no sample launch (the histogram's fallback window) and keys
above and below it (boosts), on repeated runs of one batch and candidate-region overflows, for TQ_OP_BOOL, filters, count_hits and
the cross-shard key exchange.  With TQ_TILE_COUNTERS the refreshes and raises are counted (tq_stats.tile_cycles[6], [7])."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import tantivy_b200 as T  # noqa: E402
from oracle import tq_oracle as O  # noqa: E402
from tantivy_b200._abi import (TQ_OCCUR_MUST, TQ_OCCUR_MUST_NOT, TQ_OCCUR_SHOULD, TQ_OP_AND, TQ_OP_OR, TQ_OP_TERM,  # noqa: E402
                               TQ_TERM_IGNORE_FREQ, QueryBatch)
from tests.helpers import bool_query  # noqa: E402
from tests.test_gpu_parity import TILE_OVERFLOW_HOOKS, _ctx_with_env, assert_same  # noqa: E402

_DENS = [0.3, 0.15, 0.05, 0.01, 0.002, 0.0001]
_BASE = 9300
_KS = (1, 10, 100, 1024)


@pytest.fixture(scope="module")
def synth():
    ix = T.SynthIndex(3, 1_000_000, _DENS, seed=93)
    oi = O.OracleIndex()
    ix.register(oi, segment_base=_BASE)
    return ix, oi


@pytest.fixture(scope="module")
def basic():
    """Basic record option: every tf is 1, so a term's docs score by fieldnorm alone and thousands tie at every score."""
    ix = T.SynthIndex(2, 700_000, [0.4, 0.2, 0.05, 0.01], seed=94, record_option=0)
    oi = O.OracleIndex()
    ix.register(oi, segment_base=_BASE + 10)
    return ix, oi


def _queries(ix, base, ks=_KS, boost=1.0):
    qs = [ix.query(TQ_OP_OR, terms, k, segment_base=base, boost=boost)
          for k in ks for terms in ([0, 5], [0, 1, 2, 3, 4], [1, 3, 4], [5, 4, 3, 2, 1, 0])]
    qs += [ix.query(TQ_OP_AND, terms, k, segment_base=base, boost=boost) for k in ks for terms in ([0, 1], [0, 2, 3])]
    qs += [ix.query(TQ_OP_TERM, [t], k, segment_base=base, boost=boost) for k in ks for t in (0, 2)]
    return qs


def _run(env, ix, base, qb):
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, **env)
    try:
        ix.register(c, segment_base=base)
        g = c.search_batch(qb)
        return g, c.stats()
    finally:
        c.close()


def _final_keys(rows, ks):
    """The score key of each query's final k-th row; 0 when it holds fewer than k rows (no threshold may be set then)."""
    out = np.zeros(len(ks), dtype=np.int64)
    for i, k in enumerate(ks):
        if rows[3][i] == k:
            u = int(np.float32(rows[0][i, k - 1]).view(np.uint32))
            out[i] = u ^ (0xFFFFFFFF if u >> 31 else 0x80000000)
    return out


@pytest.mark.parametrize("counters", [0, 1])
def test_rows_at_every_k(synth, counters):
    ix, oi = synth
    qb = QueryBatch(_queries(ix, _BASE))
    g, st = _run(dict(TQ_TILE_COUNTERS=counters), ix, _BASE, qb)
    assert_same(g, oi.search_batch(qb, mode=0, n_threads=16), qb.nq)
    assert st["tile_groups"] == 1 and st["tile_fallbacks"] == 0
    if counters:
        refreshes, raises = st["tile_cycles"][6], st["tile_cycles"][7]
        assert refreshes > 0 and 0 < raises <= refreshes, (refreshes, raises)


@pytest.mark.parametrize("hook", [dict(), dict(TQ_TILE_SAMPLE_DIV=0), dict(TQ_TILE_LIGHT_MAX=0)], ids=["default", "no_samples", "windows"])
def test_every_phase_leaves_a_lower_bound(synth, hook):
    """Run phase by phase and export the thresholds after each: never above the final k-th key, never falling."""
    import torch
    ix, oi = synth
    qs = _queries(ix, _BASE)
    qb = QueryBatch(qs)
    want = oi.search_batch(qb, mode=0, n_threads=16)
    final = _final_keys(want, [q["k"] for q in qs])
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, **hook)
    try:
        ix.register(c, segment_base=_BASE)
        keys = torch.zeros(qb.nq, dtype=torch.int64, device="cuda:0")
        for _ in range(2):  # the second run of the same batch starts from zeroed histograms again
            b = c.prepare(qb)
            n_ph = b.phases()
            prev = np.zeros(qb.nq, dtype=np.int64)
            for ph in range(n_ph):
                b.run_phase(ph)
                if ph + 1 < n_ph:
                    b.thresholds_export_dev(keys.data_ptr())
                    now = keys.cpu().numpy().copy()
                    assert (now >= prev).all() and (now <= final).all(), np.nonzero(now > final)
                    prev = now
            out = b.fetch()
            b.close()
            assert_same(out, want, qb.nq)
        assert (prev[final > 0] > 0).any()  # the running thresholds did rise
    finally:
        c.close()


def test_ties_at_the_kth_score(basic):
    """Thousands of docs share each score: the refresh stops at the tied key's bucket edge, and every tied doc is still handed
    over.  Regions that overflow are repeated."""
    ix, oi = basic
    base = _BASE + 10
    qs = [ix.query(TQ_OP_TERM, [t], k, segment_base=base) for t in (0, 1, 2) for k in _KS]
    qs += [ix.query(TQ_OP_OR, terms, k, segment_base=base) for terms in ([0, 3], [1, 2, 3], [0, 1]) for k in _KS]
    qs += [dict(ix.query(TQ_OP_OR, [0, 2, 3], k, segment_base=base), term_flags=[TQ_TERM_IGNORE_FREQ] * 3) for k in (10, 1024)]
    qb = QueryBatch(qs)
    g, st = _run(dict(TQ_TILE_COUNTERS=1), ix, base, qb)
    assert_same(g, oi.search_batch(qb, mode=0, n_threads=16), qb.nq)
    assert st["tile_cycles"][6] > 0


@pytest.mark.parametrize("boost", [1.0, 1e4, 1e-4])
def test_no_samples_and_keys_outside_the_window(synth, boost):
    """Without a sample launch the histogram's base is 0 and its window is the fallback 2^-4 .. 2^12: boost 1e4 puts every key
    above it (the top bucket), 1e-4 below it (bucket 0: no raise)."""
    ix, oi = synth
    qb = QueryBatch(_queries(ix, _BASE, ks=(1, 10, 100), boost=boost))
    g, st = _run(dict(TQ_TILE_SAMPLE_DIV=0, TQ_TILE_COUNTERS=1), ix, _BASE, qb)
    assert_same(g, oi.search_batch(qb, mode=0, n_threads=16), qb.nq)
    if boost == 1e-4:
        assert st["tile_cycles"][7] == 0  # every key is in bucket 0
    else:
        assert st["tile_cycles"][7] > 0


@pytest.mark.parametrize("hook", TILE_OVERFLOW_HOOKS)
def test_overflow_repeats_start_from_zeroed_histograms(synth, hook):
    ix, oi = synth
    qb = QueryBatch(_queries(ix, _BASE))
    want = oi.search_batch(qb, mode=0, n_threads=16)
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1, **hook)
    try:
        ix.register(c, segment_base=_BASE)
        for _ in range(2):
            assert_same(c.search_batch(qb), want, qb.nq)
        assert c.stats()["tile_fallbacks"] == 1
    finally:
        c.close()


def test_bool_filters_and_count_hits(synth):
    """TQ_OP_BOOL queries (general k_tile instance) next to unions, under a doc filter, with count_hits on half of them."""
    ix, _ = synth
    rng = np.random.default_rng(95)
    masks = [rng.random(ix.max_doc[s]) < 0.6 for s in range(ix.n_segments)]
    packed = [np.packbits(m, bitorder="little") for m in masks]
    qs = []
    for k in _KS:
        qs.append(bool_query(ix.query(TQ_OP_OR, [0, 1, 2], k, segment_base=_BASE), [TQ_OCCUR_MUST, TQ_OCCUR_SHOULD, TQ_OCCUR_SHOULD]))
        qs.append(bool_query(ix.query(TQ_OP_OR, [0, 2, 3, 1], k, segment_base=_BASE),
                             [TQ_OCCUR_SHOULD, TQ_OCCUR_SHOULD, TQ_OCCUR_SHOULD, TQ_OCCUR_MUST_NOT]))
        qs.append(ix.query(TQ_OP_OR, [0, 1, 3, 4], k, segment_base=_BASE))
    c, oi = _ctx_with_env(TQ_TILE=1, TQ_TILE_COUNTERS=1), O.OracleIndex()
    try:
        ix.register(c, segment_base=_BASE)
        for s in range(ix.n_segments):
            c.filter_register(7, _BASE + s, packed[s])
            oi.segment_register(_BASE + s, 0, ix.max_doc[s], 1, ix.body(s), ix.fieldnorm(s), packed[s])
        for filt in (None, 7):
            qb = QueryBatch([dict(q, filter=filt, count_hits=i % 2 == 0) for i, q in enumerate(qs)])
            want_qb = QueryBatch(qs)
            g = c.search_batch(qb)
            if filt is None:
                o = O.OracleIndex()
                ix.register(o, segment_base=_BASE)
                want = o.search_batch(want_qb, mode=0, n_threads=16)
            else:
                want = oi.search_batch(want_qb, mode=0, n_threads=16)
            assert_same(g, want, qb.nq)
        assert c.stats()["tile_cycles"][7] > 0
    finally:
        c.close()


@pytest.mark.parametrize("shards", [1, 2])
def test_key_exchange(synth, shards):
    """The cross-shard key exchange between phases (as CrossGpuMerger runs it) on top of the running thresholds: same rows."""
    import torch
    ix, oi = synth
    qb = QueryBatch(_queries(ix, _BASE, ks=(1, 10, 100)))
    want = oi.search_batch(qb, mode=0, n_threads=16)
    c = _ctx_with_env(TQ_TILE=1, TQ_TILE_TERMS=1)
    try:
        ix.register(c, segment_base=_BASE)
        kmax = qb.kmax
        keys = torch.zeros((shards, qb.nq, kmax), dtype=torch.int32, device="cuda:0")
        b = c.prepare(qb)
        n_ph = b.phases()
        for ph in range(n_ph):
            b.run_phase(ph)
            if ph + 1 < n_ph:
                b.topkeys_export_dev(keys[0].data_ptr(), kmax)
                b.thresholds_from_keys_dev(keys.data_ptr(), shards, kmax)  # shard 1 (if any) reports nothing: zeros
        out = b.fetch()
        b.close()
        assert_same(out, want, qb.nq)
    finally:
        c.close()
