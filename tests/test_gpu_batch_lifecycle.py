"""The tq_batch life cycle against the score model: prepare, whole and phased runs, the five ways to read rows and fetch_hits, destroy,
and the per-context pool every entry point takes its batch from.

  * a seeded walk over one context: up to four prepared batches alive at once, each driven through whole runs, phases in and out of
    order, threshold exchanges between phases, reads before, during and after a run, and destroy at any point (also right after
    phase 0, while k_phrase and the Count kernels still run on the batch's second stream); between them tq_count_batch, tq_sort_batch
    and the terms / metrics / histogram entry points take pooled batches that may just have been abandoned.  A state machine in
    Python predicts every return code; every answer is checked against tests/score_model.py or the fast-field models.  The walk
    runs on the tile engine's defaults, on TQ_TILE=0, on TQ_PHRASE_SIDE_STREAM=0, and with the tile buffers and candidate regions
    cut so small that every run overflows and is repaired (TQ_TILE_PCAP=64, TQ_TILE_CAND_FLOOR=4);
  * results asked for between the phases of a second run are refused, and the repair of that run's overflow still happens;
  * three batches in flight, the middle one abandoned after phase 0, its pooled buffers reused;
  * tq_multi with one device failing: its error code and message come back, and the handle answers the next batch.
Rows are compared doc for doc, segment for segment and bit for bit on f32 scores, zeros by value (helpers.hits)."""
import os

import numpy as np
import pytest

import tantivy_b200 as T
from tantivy_b200._abi import TQ_OP_AND, TQ_OP_BOOL, TQ_OP_OR, TQ_OP_TERM, TQ_RECORD_BASIC, QueryBatch
from tests import score_model as M
from tests.helpers import OracleSegment, bool_shape_query, hits, make_query, random_bool_shapes
from tests.test_gpu_histogram import COLUMNS as HIST_COLUMNS
from tests.test_gpu_histogram import FMAX, HistFixture
from tests.test_gpu_histogram import rows as hist_rows
from tests.test_gpu_metrics import MetricsFixture
from tests.test_gpu_metrics import check as metrics_check
from tests.test_gpu_parity import _ctx_with_env
from tests.test_gpu_phrase import PosSegment, phrase_query
from tests.test_gpu_sort_field import Fixture as SortFixture
from tests.test_gpu_sort_field import device_rows, packed, with_order
from tests.test_gpu_sort_field import shapes as ff_shapes
from tests.test_gpu_terms import ORDERS as TERMS_ORDERS
from tests.test_gpu_terms import TermsFixture
from tests.test_gpu_terms import run_check as terms_check

N_TERMS = 8
NAMES = [f"t{i}" for i in range(N_TERMS)]  # (sorted: the positions segment's list i is term i)
DENS = (0.4, 0.15, 0.06, 0.02, 0.008, 0.003, 0.1, 0.3)
KS = (1, 10, 129, 1024)
FILTER = 7
ORD_A, ORD_B, ORD_SPARE = 9001, 9002, 9004

# ---- the state machine ------------------------------------------------------------------------------------------------------
# A batch is fresh (prepared, never run), mid1 (phase 0 done), mid (phase 1 or 2 done), done (a run finished, not read since) or
# read (a finalising read has waited for the run and repaired an overflow).
STATES = ("fresh", "mid1", "mid", "done", "read")
READS = ("fetch", "results_dev", "copy_dev", "pack_dev", "pack_async", "fetch_hits")
CALLS = ("run", "phase", "phase_wrong", "exchange") + READS + ("close",)
EXCHANGES = ("theta", "keys1", "keys2", "kth")
FAST_FIELDS = ("count", "sort", "terms", "metrics", "histogram")
MAX_LIVE = 4
WALK_STEPS = 220
SEEDS = (0x11FE, 0x2C7C)


def predict(state, next_phase, call, arg=None):
    """(return code, next state, next phase) of a batch call in a state."""
    mid = state in ("mid1", "mid")
    if call == "run":
        return 0, "done", 0
    if call == "phase":
        if next_phase == 3:
            return 0, "done", 0
        return 0, "mid1" if next_phase == 0 else "mid", next_phase + 1
    if call == "phase_wrong":
        return -1, state, next_phase
    if call == "exchange":
        return (0 if mid else -1), state, next_phase
    if call in READS:
        if state not in ("done", "read"):
            return -1, state, next_phase
        return 0, ("read" if call != "pack_async" else state), next_phase
    assert call == "close"
    return 0, None, 0


# The kind of every query a walk draws its batches from: only the kinds matter to the plan; Index builds the queries.
POOL_KINDS = (["term"] * 4 + ["and"] * 4 + ["or"] * 5 + ["bool"] * 6 + ["phrase"] * 4 + ["hits"] * 4 + ["filter"] * 3 + ["threshold"] * 3
              + ["spare"] * 2)


def plan_walk(seed, bool_ok, n_steps=WALK_STEPS):
    """The walk of one seed as a list of steps, with the return code the state machine predicts for each, and the set of
    (state, call) pairs it visits.  bool_ok = the context runs TQ_OP_BOOL queries (the tile engine): otherwise a batch holding one
    is refused at prepare with TQ_ERR_UNSUPPORTED.  Calls on batches prefer pairs the walk has not visited yet."""
    rng = np.random.default_rng(seed)
    kinds = POOL_KINDS
    live = {}  # slot -> [state, next_phase, holds_spare]
    steps, seen = [], set()
    next_slot = 0
    for _ in range(n_steps):
        r = rng.random()
        if not live or (len(live) < MAX_LIVE and r < 0.12):
            nq = int(rng.integers(2, len(kinds) + 1)) if rng.random() < 0.5 else int(rng.integers(2, 9))
            qi = sorted(int(i) for i in rng.choice(len(kinds), size=nq, replace=False))
            if rng.random() < 0.7:  # phrases and count_hits next to the tile engine: work on the second stream
                qi = sorted(set(qi) | {kinds.index("phrase") + int(rng.integers(4)), kinds.index("hits") + int(rng.integers(4))})
            if not bool_ok and rng.random() < 0.75:  # (the per-query kernels: most batches leave TQ_OP_BOOL out)
                qi = [i for i in qi if kinds[i] != "bool"] or [0]
            refused = not bool_ok and any(kinds[i] == "bool" for i in qi)
            steps.append(("prepare", next_slot, qi, -4 if refused else 0))
            seen.add(("ctx", "prepare_refused" if refused else "prepare"))
            if not refused:
                live[next_slot] = ["fresh", 0, any(kinds[i] == "spare" for i in qi)]
            next_slot += 1
            continue
        if r < 0.2:
            what = FAST_FIELDS[int(rng.integers(len(FAST_FIELDS)))]
            steps.append(("fast", what, int(rng.integers(1 << 30)), 0))
            seen.add(("ctx", what))
            continue
        if r < 0.24:
            held = any(v[2] for v in live.values())
            steps.append(("unregister", None, None, -1 if held else 0))
            seen.add(("ctx", "unregister_held" if held else "unregister"))
            continue
        options = [(s, c) for s in sorted(live) for c in CALLS]
        fresh = [o for o in options if (live[o[0]][0], o[1]) not in seen]
        # (phase 1 leads to the state visited least)
        to_mid = [(sl, "phase") for sl in sorted(live) if live[sl][0] == "mid1" and any(("mid", c) not in seen for c in CALLS)]
        src = to_mid if to_mid and rng.random() < 0.5 else fresh if fresh and rng.random() < 0.8 else options
        slot, call = src[int(rng.integers(len(src)))]
        state, nxt, _ = live[slot]
        arg = None
        if call == "phase_wrong":
            arg = int(rng.choice([p for p in (0, 1, 2, 3, 4) if p != nxt]))
        elif call == "exchange":
            arg = EXCHANGES[int(rng.integers(len(EXCHANGES)))]
        rc, new_state, new_next = predict(state, nxt, call, arg)
        seen.add((state, call))
        steps.append(("batch", slot, (call, arg, state, nxt), rc))
        if new_state is None:
            del live[slot]
        else:
            live[slot][0], live[slot][1] = new_state, new_next
    for slot in sorted(live):
        steps.append(("batch", slot, ("close", None, live[slot][0], live[slot][1]), 0))
    return steps, seen


@pytest.mark.parametrize("bool_ok", [True, False], ids=["tile", "no_tile"])
def test_walk_visits_every_state_and_call(bool_ok):
    """Each seed's walk calls every batch entry point in every state of the state machine, prepares, uses every fast-field entry
    point, and unregisters the spare segment both while a batch holds it and when none does."""
    for seed in SEEDS:
        steps, seen = plan_walk(seed, bool_ok)
        missing = [(s, c) for s in STATES for c in CALLS if (s, c) not in seen]
        assert not missing, (seed, missing)
        for what in ("prepare", "unregister_held", "unregister") + FAST_FIELDS:
            assert ("ctx", what) in seen, (seed, what)
        if not bool_ok:
            assert ("ctx", "prepare_refused") in seen, seed
        # the walk ends with nothing alive, and closes a batch right after phase 0
        assert sum(1 for s in steps if s[0] == "batch" and s[2][0] == "close" and s[2][2] == "mid1") >= 1, seed


# ---- the index --------------------------------------------------------------------------------------------------------------
DEV = "cuda:0"


def _lists(rng, max_doc, basic):
    out = []
    for p in DENS:
        docs = np.nonzero(rng.random(max_doc) < p)[0].astype(np.uint32)
        out.append((docs, None if basic else rng.integers(1, 9, size=len(docs)).astype(np.uint32)))
    return out


def _filtered(m, mask):
    """The model's segment with alive := alive AND the filter (FilterCollector)."""
    c = M.Segment.__new__(M.Segment)
    c.__dict__.update(m.__dict__)
    c.alive = mask.copy() if m.alive is None else m.alive & mask
    return c


class Index:
    """Segment A (250k docs, freqs, deletes), segment B (212k docs, Basic), a positions segment P (30k docs, deletes) and a small
    spare segment the walk unregisters and registers again; one filter on A, B and P; the query pool of POOL_KINDS with every
    query's model rows, and its model Count."""

    def __init__(self):
        rng = np.random.default_rng(0xB47C)
        n_a, n_b, n_p, n_s = 250_003, 212_345, 30_001, 5_003
        la, lb, ls = _lists(rng, n_a, False), _lists(rng, n_b, True), _lists(rng, n_s, False)
        len_a, len_b, len_s = rng.integers(1, 60, size=n_a), rng.integers(1, 60, size=n_b), rng.integers(1, 60, size=n_s)
        alive_a = packed(rng.random(n_a) > 0.2)
        self.a = OracleSegment(la, len_a, segment_ord=ORD_A, writer_cls=T.FieldWriter, alive=alive_a)
        self.b = OracleSegment(lb, len_b, record_option=TQ_RECORD_BASIC, segment_ord=ORD_B, writer_cls=T.FieldWriter)
        self.s = OracleSegment(ls, len_s, segment_ord=ORD_SPARE, writer_cls=T.FieldWriter)
        self.ma, self.mb = M.Segment(ORD_A, la, len_a, alive=alive_a), M.Segment(ORD_B, lb, len_b, basic=True)
        self.ms = M.Segment(ORD_SPARE, ls, len_s)
        lengths = rng.integers(2, 24, size=n_p)
        words = rng.choice(N_TERMS, size=int(lengths.sum()), p=np.array(DENS) / sum(DENS))
        positions = {t: {} for t in NAMES}
        at = 0
        for d, n in enumerate(lengths.tolist()):
            for j, w in enumerate(words[at:at + n].tolist()):
                positions[NAMES[w]].setdefault(d, []).append(j)
            at += n
        self.p = PosSegment.from_positions(positions, lengths, alive=packed(rng.random(n_p) > 0.1))
        self.mp = self.p.model(NAMES)
        self.masks = {s.segment_ord: rng.random(s.max_doc) < 0.5 for s in (self.a, self.b, self.p.seg)}
        self.pool = self._pool(np.random.default_rng(0x9001))
        assert [k for k, _, _ in self.pool] == POOL_KINDS

    def register(self, ctx):
        for s in (self.a, self.b, self.s):
            s.register(ctx)
        self.p.register(ctx)
        for o, m in self.masks.items():
            ctx.filter_register(FILTER, o, packed(m))

    def _pool(self, rng):
        segs, msegs = [self.a, self.b, self.p.seg], [self.ma, self.mb, self.mp]
        fsegs = [_filtered(m, self.masks[m.segment_ord]) for m in msegs]
        out = []

        def add(kind, q, terms, model_segs=msegs):
            rows = M.search(model_segs, q, terms)
            out.append((kind, (q, terms), (rows, M.count(model_segs, q, terms) if q["op"] != 3 else None)))

        def mk(op, terms, k, on=segs, **extra):
            q = make_query(op, on, terms, k)
            q.update(extra)
            return q

        for t, k in ((0, 1024), (3, 10), (5, 129), (7, 1)):
            add("term", mk(TQ_OP_TERM, [t], k), [t])
        for terms, k in (([0, 1], 10), ([1, 6, 7], 129), ([0, 7], 1024), ([2, 3], 1)):
            add("and", mk(TQ_OP_AND, terms, k), terms)
        for terms, k in (([0, 1, 6], 1024), ([2, 4], 10), ([3, 5, 7], 129), ([0, 2, 4, 6], 1), ([1, 7], 10)):
            add("or", mk(TQ_OP_OR, terms, k), terms)
        # (up to six clauses: a wider shape over these dense lists needs more than the tile engine's scratch)
        for sh in [sh for sh in random_bool_shapes(rng, 40, N_TERMS, n_wide=0) if len(sh["terms"]) <= 6][:6]:
            add("bool", bool_shape_query(segs, sh), list(sh["terms"]))
        for terms, k, slop in (([0, 7], 10, 0), ([7, 0, 1], 129, 0), ([1, 0], 1024, 1), ([6, 6], 10, 0)):
            q = phrase_query([self.p], [NAMES[t] for t in terms], k)[0]
            q["slop"] = slop
            add("phrase", q, terms)
        for op, terms, k in ((TQ_OP_TERM, [1], 10), (TQ_OP_OR, [0, 6, 7], 10), (TQ_OP_AND, [0, 7], 129), (TQ_OP_OR, [2, 3, 4], 1024)):
            add("hits", mk(op, terms, k, count_hits=True), terms)
        for op, terms, k in ((TQ_OP_OR, [0, 1], 10), (TQ_OP_TERM, [6], 129), (TQ_OP_AND, [0, 6], 1024)):
            add("filter", mk(op, terms, k, filter=FILTER), terms, fsegs)
        for op, terms, k in ((TQ_OP_OR, [0, 6], 10), (TQ_OP_AND, [0, 1], 1024), (TQ_OP_TERM, [7], 129)):
            rows = M.search(msegs, mk(op, terms, k), terms)
            add("threshold", mk(op, terms, k, threshold=rows[len(rows) // 2][0]), terms)
        for op, terms, k in ((TQ_OP_TERM, [0], 10), (TQ_OP_OR, [0, 1, 2], 129)):
            add("spare", mk(op, terms, k, on=[self.s]), terms, [self.ms])
        return out


class FastFields(MetricsFixture):
    """The metric fixture's segments and columns (the sort fixture's columns among them), with the terms and histogram models."""
    tmodel = TermsFixture.tmodel
    missing_image = TermsFixture.missing_image
    hmodel = HistFixture.hmodel

    def __init__(self):
        super().__init__()
        self.tcol = self.mcol


@pytest.fixture(scope="module")
def ix():
    return Index()


@pytest.fixture(scope="module")
def ff():
    return FastFields()


def rc_of(fn):
    """(0, None) or the (code, message) of the TqError fn raises."""
    try:
        fn()
        return 0, None
    except T.TqError as e:
        return int(str(e).split("error ")[1].split(":")[0]), str(e)


def key(score):
    """Order-preserving u32 key of an f32 score (the device's), -0.0 and +0.0 on one key."""
    u = int((np.float32(score) + np.float32(0)).view(np.uint32))
    return u ^ 0xFFFFFFFF if u >> 31 else u | 0x80000000


class _DevView:
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


def _from_packed(p, nq, kmax):
    r = nq * kmax
    return (p[:r].view(np.float32).reshape(nq, kmax), p[r:2 * r].view(np.uint32).reshape(nq, kmax),
            p[2 * r:3 * r].view(np.uint32).reshape(nq, kmax), p[3 * r:3 * r + nq].view(np.uint32))


SENTINEL = 0x5A5A5A5A


class Walker:
    """Runs a plan_walk on a context and checks every return code and every answer."""

    def __init__(self, ctx, ix, ff, bool_ok):
        import torch
        self.torch = torch
        self.ctx, self.ix, self.ff, self.bool_ok = ctx, ix, ff, bool_ok
        self.live = {}
        self.nonzero_flags = 0
        self.ff_qts = [qt for qt in ff_shapes(ff) if bool_ok or qt[0]["op"] != TQ_OP_BOOL]

    # -- answers --
    def check_rows(self, s, result, what):
        for i, pi in enumerate(s["qi"]):
            kind, (q, terms), (rows, _) = self.ix.pool[pi]
            got = hits(result, i)
            assert got == rows, (what, i, kind, q["op"], terms, q["k"], got[:3], rows[:3])

    def check_hits(self, s, got):
        want = [self.ix.pool[pi][2][1] if self.ix.pool[pi][1][0].get("count_hits") else 0 for pi in s["qi"]]
        assert [int(x) for x in got] == want, ("fetch_hits", got, want)

    # -- calls --
    def read(self, s, call, expect):
        torch, bt, nq, kmax = self.torch, s["b"], s["nq"], s["kmax"]
        words = 3 * nq * kmax + nq
        if call == "fetch":
            out = s["qb"].alloc_out()
            for a in out[1:]:
                a.view(np.uint32)[...] = SENTINEL
            rc, msg = rc_of(lambda: bt.fetch(out))
            result, untouched = out[1:], all((a.view(np.uint32) == SENTINEL).all() for a in out[1:])
        elif call == "results_dev":
            got = []
            rc, msg = rc_of(lambda: got.append(bt.results_dev()))
            untouched = True
            if rc == 0:
                sp, gp, dp, cp, stride = got[0]
                assert stride == kmax

                def host(ptr, n, t):
                    return torch.as_tensor(_DevView(ptr, n, t), device=DEV).cpu().numpy()
                result = (host(sp, nq * kmax, "<f4").reshape(nq, kmax), host(gp, nq * kmax, "<u4").reshape(nq, kmax),
                          host(dp, nq * kmax, "<u4").reshape(nq, kmax), host(cp, nq, "<u4"))
        elif call == "copy_dev":
            bufs = [torch.full((nq * kmax,), SENTINEL, dtype=torch.int32, device=DEV) for _ in range(3)]
            bufs.append(torch.full((nq,), SENTINEL, dtype=torch.int32, device=DEV))
            torch.cuda.synchronize()
            rc, msg = rc_of(lambda: bt.results_copy_dev(*[x.data_ptr() for x in bufs]))
            p = np.concatenate([x.cpu().numpy() for x in bufs])
            result, untouched = _from_packed(p, nq, kmax), (p.view(np.uint32) == SENTINEL).all()
        else:  # pack_dev / pack_async
            buf = torch.full((words + 4,), SENTINEL, dtype=torch.int32, device=DEV)
            torch.cuda.synchronize()
            fn = bt.results_pack_dev if call == "pack_dev" else bt.results_pack_dev_async
            rc, msg = rc_of(lambda: fn(buf.data_ptr()))
            torch.cuda.synchronize()
            p = buf.cpu().numpy()
            result, untouched = _from_packed(p, nq, kmax), (p.view(np.uint32) == SENTINEL).all()
            if rc == 0 and call == "pack_async":
                flags = p[words:].view(np.uint32)
                if s["state"] == "read":
                    assert not flags.any(), ("a repaired run's flags", flags)
                if flags.any():
                    self.nonzero_flags += 1
                    return rc, msg  # (rows not final: the caller takes results_pack_dev)
        if rc == 0 and expect == 0:
            self.check_rows(s, result, call)
        if rc != 0:
            assert untouched, (call, "a refused read wrote its outputs")
        return rc, msg

    def exchange(self, s, kind):
        torch, bt, nq, kmax = self.torch, s["b"], s["nq"], s["kmax"]
        if kind == "theta":
            keys = torch.zeros(nq, dtype=torch.int64, device=DEV)
            torch.cuda.synchronize()
            rc, msg = rc_of(lambda: bt.thresholds_export_dev(keys.data_ptr()))
            if rc == 0:
                bt.thresholds_import_dev(keys.data_ptr())
        elif kind in ("keys1", "keys2"):
            n = 1 if kind == "keys1" else 2  # (two shards: this one and one that holds nothing)
            buf = torch.zeros(n * nq * kmax, dtype=torch.int32, device=DEV)
            torch.cuda.synchronize()
            rc, msg = rc_of(lambda: bt.topkeys_export_dev(buf.data_ptr(), kmax))
            if rc == 0:
                bt.thresholds_from_keys_dev(buf.data_ptr(), n, kmax)
        else:  # the final k-th keys of an earlier run (none for phrases: they take no threshold exchange)
            kth = []
            for pi in s["qi"]:
                kind_, (q, _), (rows, _) = self.ix.pool[pi]
                kth.append(key(rows[q["k"] - 1][0]) if len(rows) >= q["k"] and q["op"] != 3 else 0)
            keys = torch.tensor(kth, dtype=torch.int64, device=DEV)
            torch.cuda.synchronize()
            rc, msg = rc_of(lambda: bt.thresholds_import_dev(keys.data_ptr()))
        torch.cuda.synchronize()
        return rc, msg

    def fast(self, what, seed):
        r = np.random.default_rng(seed)
        ctx, ix, ff = self.ctx, self.ix, self.ff
        if what == "count":
            qi = [int(i) for i in r.choice(len(ix.pool), size=10, replace=False) if ix.pool[int(i)][1][0]["op"] != 3]
            got = ctx.count_batch(QueryBatch([ix.pool[i][1][0] for i in qi]))
            assert [int(x) for x in got] == [ix.pool[i][2][1] for i in qi], "count"
            return
        qts = [self.ff_qts[int(i)] for i in r.choice(len(self.ff_qts), size=3, replace=False)]
        if what == "sort":
            kind = str(r.choice(["uniform", "half", "i64"]))
            qts = with_order(qts, ks=(int(r.choice(KS)),))
            out = ctx.sort_batch(QueryBatch([q for q, _ in qts]), [(ff.mcol[kind], q["_order"]) for q, _ in qts], count_hits=True)
            for i, qt in enumerate(qts):
                rows, n = SortFixture.model(ff, qt, kind, qt[0]["_order"], qt[0]["k"])
                assert (device_rows(out, i), int(out[5][i])) == (rows, n), ("sort", kind, i)
        elif what == "terms":
            target, order = TERMS_ORDERS[int(r.integers(len(TERMS_ORDERS)))]
            terms_check(ctx, ff, qts, str(r.choice(["few", "half", "i64"])), target, order, int(r.choice([1, 10, 5000])))
        elif what == "metrics":
            metrics_check(ctx, ff, qts, [("ints", "big", "flag"), ("dyadic", "const", "partial")][int(r.integers(2))])
        else:
            col = str(r.choice(["uniform", "few", "i64"]))
            kind = HIST_COLUMNS[col][0]
            interval, offset = HIST_COLUMNS[col][1][0]
            out = ctx.histogram_batch(QueryBatch([q for q, _ in qts]), [(ff.mcol[col], kind, interval, offset, -FMAX, FMAX)] * len(qts),
                                      count_hits=True)
            for i, qt in enumerate(qts):
                assert hist_rows(out, i) == ff.hmodel(qt, col, interval, offset), ("histogram", col, i)

    def step(self, n, st):
        what, a, b, expect = st
        ctx, ix = self.ctx, self.ix
        if what == "prepare":
            qb = QueryBatch([ix.pool[i][1][0] for i in b])
            got = []
            rc, msg = rc_of(lambda: got.append(ctx.prepare(qb)))
            assert rc == expect, (n, st, msg)
            if rc == 0:
                self.live[a] = dict(b=got[0], qb=qb, qi=b, nq=qb.nq, kmax=qb.kmax, state="fresh", next=0, ran=False)
            return
        if what == "fast":
            self.fast(a, b)
            return
        if what == "unregister":
            rc, msg = rc_of(lambda: ctx.segment_unregister(ORD_SPARE, 0))
            assert rc == expect, (n, st, msg)
            if rc == 0:
                ix.s.register(ctx)
            else:
                assert "a prepared batch still uses the segment" in msg, msg
            return
        call, arg, state, nxt = b
        s = self.live[a]
        assert (s["state"], s["next"]) == (state, nxt), (n, st, s["state"], s["next"])
        bt = s["b"]
        if call == "run":
            rc, msg = rc_of(bt.run)
        elif call == "phase":
            rc, msg = rc_of(lambda: bt.run_phase(nxt))
        elif call == "phase_wrong":
            rc, msg = rc_of(lambda: bt.run_phase(arg))
        elif call == "exchange":
            rc, msg = self.exchange(s, arg)
        elif call == "fetch_hits":
            got = []
            rc, msg = rc_of(lambda: got.append(bt.fetch_hits()))
            if rc == 0:
                self.check_hits(s, got[0])
        elif call == "close":
            bt.close()
            del self.live[a]
            return
        else:
            rc, msg = self.read(s, call, expect)
        assert rc == expect, (n, st, msg)
        if rc != 0 and call in READS and s["ran"] and state in ("mid1", "mid"):
            assert "a run is in progress" in msg, msg
        _, s["state"], s["next"] = predict(state, nxt, call, arg)
        if s["state"] == "done" and call in ("run", "phase"):
            s["ran"] = True

    def run(self, steps):
        try:
            for n, st in enumerate(steps):
                self.step(n, st)
        finally:
            for s in self.live.values():
                s["b"].close()
        assert not self.live


CONFIGS = {"defaults": {}, "no_tile": dict(TQ_TILE=0), "phrase_main_stream": dict(TQ_PHRASE_SIDE_STREAM=0),
           "pcap64": dict(TQ_TILE_PCAP=64), "cand_floor4": dict(TQ_TILE_CAND_FLOOR=4)}


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS, ids=["seed0", "seed1"])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_seeded_walk(ix, ff, config, seed):
    """One seeded walk over one context (plan_walk: every (state, call) pair), every return code as the state machine predicts and
    every answer as the models give it.  pcap64 / cand_floor4: every tile run overflows its buffers or regions, and a finalising
    read repairs it."""
    env = CONFIGS[config]
    bool_ok = env.get("TQ_TILE", 1) != 0
    ctx = _ctx_with_env(**env)
    try:
        ix.register(ctx)
        ff.register(ctx)
        Walker(ctx, ix, ff, bool_ok).run(plan_walk(seed, bool_ok)[0])
    finally:
        ctx.close()


def _pick(ix, kinds_terms):
    """Pool indices of the queries of the given (kind, terms, k)."""
    out = []
    for kind, terms, k in kinds_terms:
        out.append(next(i for i, (kd, (q, t), _) in enumerate(ix.pool) if kd == kind and t == terms and q["k"] == k))
    return out


OVERFLOWING = [("or", [0, 1, 6], 1024), ("and", [0, 7], 1024), ("term", [0], 1024), ("hits", [2, 3, 4], 1024), ("phrase", [1, 0], 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("read", ["fetch", "pack_async"])
def test_results_refused_during_a_second_run_and_its_overflow_repaired(ix, read):
    """TQ_TILE_PCAP=64 (every tile run overflows): run -> fetch -> phase 0 -> the read is refused -> phases 1-3 -> the rows equal the
    model; with results_pack_dev_async the flags at the end say the rows are not final, and the fetch after it repairs them."""
    import torch
    ctx = _ctx_with_env(TQ_TILE_PCAP=64)
    try:
        ix.register(ctx)
        qi = _pick(ix, OVERFLOWING) + [next(i for i, p in enumerate(ix.pool) if p[0] == "bool" and p[2][0])]
        w = Walker.__new__(Walker)
        w.ix, w.torch = ix, torch
        qb = QueryBatch([ix.pool[i][1][0] for i in qi])
        bt = ctx.prepare(qb)
        s = dict(b=bt, qb=qb, qi=qi, nq=qb.nq, kmax=qb.kmax, state="done")
        try:
            bt.run()
            w.check_rows(s, bt.fetch(), "first run")
            bt.run_phase(0)
            rc, msg = (rc_of(bt.fetch) if read == "fetch" else w.read(s, "pack_async", -1))
            assert rc == -1 and "a run is in progress" in msg, msg
            for p in (1, 2, 3):
                bt.run_phase(p)
            if read == "pack_async":
                words = 3 * qb.nq * qb.kmax + qb.nq
                buf = torch.zeros(words + 4, dtype=torch.int32, device=DEV)
                bt.results_pack_dev_async(buf.data_ptr())
                torch.cuda.synchronize()
                assert buf[words:].cpu().numpy().any(), "the overflowed run's flags"
            w.check_rows(s, bt.fetch(), "second run")
            assert ctx.stats()["tile_fallbacks"] == 1
            w.check_hits(s, bt.fetch_hits())
        finally:
            bt.close()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_three_batches_in_flight_one_abandoned(ix):
    """Three prepared batches submitted back to back as bench.py's pipelined steps do; the middle one is closed after its phase 0
    (phrases and count_hits still on its second stream).  The first one is read and run again, the third read; then tq_count_batch
    takes the pooled batches.  Every answer equals the model."""
    ctx = T.Context(0)
    try:
        ix.register(ctx)
        w = Walker.__new__(Walker)
        w.ix = ix
        n = len(ix.pool)
        sets = [list(range(0, n, 2)), list(range(n)), list(range(1, n, 2))]
        sets = [[i for i in qi if ix.pool[i][0] != "spare"] for qi in sets]
        qbs = [QueryBatch([ix.pool[i][1][0] for i in qi]) for qi in sets]
        bts = [ctx.prepare(qb) for qb in qbs]
        ss = [dict(b=b, qb=qb, qi=qi) for b, qb, qi in zip(bts, qbs, sets)]
        try:
            bts[0].run()
            bts[1].run_phase(0)
            bts[2].run()
            bts[1].close()
            w.check_rows(ss[0], bts[0].fetch(), "first")
            bts[0].run()
            w.check_rows(ss[0], bts[0].fetch(), "first again")
            w.check_hits(ss[0], bts[0].fetch_hits())
            w.check_rows(ss[2], bts[2].fetch(), "third")
            w.check_hits(ss[2], bts[2].fetch_hits())
            bts[2].close()
            counted = [i for i in range(n) if ix.pool[i][1][0]["op"] != 3]
            for _ in range(2):  # (the third batch's buffers, then the abandoned one's)
                got = ctx.count_batch(QueryBatch([ix.pool[i][1][0] for i in counted]))
                assert [int(x) for x in got] == [ix.pool[i][2][1] for i in counted]
            again = ctx.prepare(qbs[1])
            try:
                again.run()
                w.check_rows(ss[1], again.fetch(), "the abandoned batch's queries")
            finally:
                again.close()
        finally:
            for b in bts:
                b.close()
    finally:
        ctx.close()


def _multi_with_env(devices, **env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return T.MultiContext(devices)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.mark.gpu
def test_multi_reports_the_failing_device_and_answers_next(ix):
    """tq_multi over two contexts with TQ_MAX_LISTS=6: A on device 0, B on device 1.  A batch whose share on device 1 needs more
    block tables than that fails there at prepare; device 0 has run phase 0 of its share (unions on the tile engine with
    count_hits: k_count_tiles on the batch's second stream) and gives up.  The call reports device 1's TQ_ERR_OOM and its message.
    The next batch on the same handle reuses device 0's abandoned batch and returns the model's rows.  (tq_multi registers no
    positions, so the work on the second stream is the Count kernels', not k_phrase's.)"""
    m = _multi_with_env([0, 0], TQ_MAX_LISTS=6)
    try:
        for dev, s in ((0, ix.a), (1, ix.b)):
            m.segment_register(s.segment_ord, 0, s.max_doc, s.record_option, s.body, s.fn_ids, s.alive, device_index=dev)
        ab, a, b = [ix.a, ix.b], [ix.a], [ix.b]
        failing = [dict(make_query(TQ_OP_OR, ab, [0, 1, 6], 10), count_hits=True), dict(make_query(TQ_OP_AND, a, [0, 1], 129), count_hits=True),
                   make_query(TQ_OP_OR, b, list(range(N_TERMS)), 10)]
        with pytest.raises(T.TqError, match=r"error -5: .*TQ_MAX_LISTS"):
            m.search_batch(QueryBatch(failing))
        qts = [(dict(make_query(TQ_OP_OR, ab, [0, 1, 6], 10), count_hits=True), [0, 1, 6]),
               (dict(make_query(TQ_OP_AND, a, [0, 1], 129), count_hits=True), [0, 1]), (make_query(TQ_OP_TERM, ab, [7], 1024), [7]),
               (make_query(TQ_OP_OR, ab, [0, 6], 1024), [0, 6])]
        for _ in range(2):
            g = m.search_batch(QueryBatch([q for q, _ in qts]))
            for i, (q, t) in enumerate(qts):
                assert hits(g, i) == M.search([ix.ma, ix.mb], q, t), i
    finally:
        m.close()
