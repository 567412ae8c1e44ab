"""k_tile's running threshold, piece by piece: tile_push and tile_theta_refresh (tq_tile.cuh) run on inputs written here
(tests/cuda/tile_theta_harness.cu, built beside the product library) and are compared with a plain model written from DESIGN §3.1.

The model's refresh rule: take the highest coarse bucket cb whose suffix count reaches k; need = k minus the coarse suffix above
cb; take the highest fine bucket of cb whose suffix inside cb reaches need, else cb's first bucket; the threshold becomes
max(old, edge), and stays untouched when the edge is 0.  Independently of that rule, a soundness check: the counts as read must
vouch for at least k keys at or above the edge the threshold rose to.  The cases reach what an end-to-end run reaches only by
chance: a suffix equal to k exactly at a coarse and at a fine edge in every lane and coarse bucket, k reached only in bucket 0,
everything in the top bucket, fewer than k counts, fine counts trailing and leading the coarse ones (a refresh reads the coarse
counts first while other SMs keep adding), every base word that matters (0 = the fallback window, 1, 0x8000, 0xBD80, the key of
+inf, 0xFFFF) and old thresholds below, at and above the edge.

The push harness runs one kTileThreads CTA of tile_push calls, three launches in a row, so candidate indexes continue as they do
across a launch: counts, candidates, refresh triggers (the k-th push and every max(k / 4, 16)-th after it) and the CTA's 16-entry
refresh list, overflowing, between guard words.

The sample harness runs k_theta_samples, which raises each query's threshold to its k-th best sample and writes the threshold's
key >> 16 as the histogram's base word: 0 (the fallback window) when there are fewer than k samples and no threshold before."""
import collections
import ctypes as C
import os

import numpy as np
import pytest

FINE, COARSE = 2048, 64
BASE_WORD = FINE + COARSE
WORDS = BASE_WORD + 32
FALLBACK_BASE = 0xBD80  # the key of 2^-4, >> 16
REFRESH_CAP = 16
BASE_WORDS = (0, 1, 0x8000, 0xBD80, 0xFF80, 0xFFFF)  # 0xFF80: the key of +inf >> 16
KS = (1, 2, 15, 16, 17, 63, 64, 255, 256, 1023, 1024)


# ---- the model ----------------------------------------------------------------------------------------------------------------
def score_key(score):
    """Order-preserving u32 image of an f32 score; -0.0 and +0.0 share one key."""
    s = np.asarray(score, dtype=np.float32) + np.float32(0.0)
    u = s.view(np.uint32).astype(np.uint64)
    return np.where(u >> 31, u ^ 0xFFFFFFFF, u ^ 0x80000000).astype(np.uint32)


def th_hist_base(base_word):
    return int(base_word) if base_word else FALLBACK_BASE


def th_hist_bucket(key, base):
    """key >> 16 above the base: 0 at or below it, the top bucket above the window."""
    hi = int(key) >> 16
    return 0 if hi <= base else min(hi - base, FINE - 1)


def th_hist_edge(b, base):
    """The lowest key bucket b can hold (0 for bucket 0), clamped to the top of the key space."""
    return 0 if b == 0 else min(base + b, 0xFFFF) << 16


def refresh(fine, coarse, base_word, k, theta):
    """(new theta, raised, bucket or None) of one refresh, by the rule of DESIGN §3.1."""
    above = 0
    for cb in range(COARSE - 1, -1, -1):
        if above + int(coarse[cb]) >= k:
            break
        above += int(coarse[cb])
    else:
        return theta, False, None
    need = k - above
    lane, inside = 0, 0
    for ln in range(31, -1, -1):
        inside += int(fine[cb * 32 + ln])
        if inside >= need:
            lane = ln
            break
    b = cb * 32 + lane
    edge = th_hist_edge(b, th_hist_base(base_word))
    if edge == 0:
        return theta, False, b
    return max(theta, edge), theta < edge, b


def vouched(fine, coarse, b):
    """How many keys >= edge(b) the counts vouch for: a coarse bucket above b's by the larger of its coarse count and its fine sum
    (each is a lower bound of what it holds), b's own coarse bucket by its fine counts from b on, or by its coarse count as well
    when b is its first bucket."""
    cb = b // 32
    fine_sums = fine.reshape(COARSE, 32).sum(axis=1, dtype=np.int64)
    n = int(np.maximum(coarse[cb + 1:].astype(np.int64), fine_sums[cb + 1:]).sum())
    own = int(fine[b:(cb + 1) * 32].sum(dtype=np.int64))
    if b % 32 == 0:
        own = max(own, int(coarse[cb]))
    return n + own


def check_sound(fine, coarse, base_word, k, theta0, theta1, raised):
    """A refresh may only raise the threshold, says so exactly when it did, and only to an edge that k counted keys reach."""
    assert theta1 >= theta0
    assert bool(raised) == (theta1 > theta0)
    if theta1 > theta0:
        base = th_hist_base(base_word)
        b = next(b for b in range(1, FINE) if th_hist_edge(b, base) == theta1)  # (edges never fall: the lowest vouches most)
        assert vouched(fine, coarse, b) >= k, (b, k)


# ---- the cases --------------------------------------------------------------------------------------------------------------
def _coarse_of(fine):
    return fine.reshape(COARSE, 32).sum(axis=1).astype(np.uint32)


def _case(fine, base_word, k, theta=0, coarse=None, name=""):
    fine = np.asarray(fine, dtype=np.uint32)
    return dict(fine=fine, coarse=_coarse_of(fine) if coarse is None else np.asarray(coarse, dtype=np.uint32),
                base_word=base_word, k=k, theta=theta, name=name)


def _exact_at(b, k, rng):
    """k counts whose suffix reaches k exactly at bucket b: one in b, k - 1 spread over the buckets above it (or, at the top,
    all of them in b)."""
    fine = np.zeros(FINE, np.uint32)
    if b == FINE - 1:
        fine[b] = k
        return fine
    fine[b] = 1
    if k > 1:
        np.add.at(fine, rng.integers(b + 1, FINE, size=k - 1), 1)
    return fine


def hand_cases():
    rng = np.random.default_rng(0x7E7A)
    cases = []
    for cb in range(COARSE):  # suffix == k at a coarse edge (lane cb // 2, both parities), and at a fine edge of each lane L
        for k in (1, 17, 256):
            cases.append(_case(_exact_at(cb * 32, k, rng), 0xBD80, k, name=f"coarse_edge_{cb}_{k}"))
        ln = 1 + cb % 31
        cases.append(_case(_exact_at(cb * 32 + ln, 16, rng), 0x8000, 16, name=f"fine_edge_{cb}_{ln}"))
    for k in KS:
        base_word = BASE_WORDS[k % len(BASE_WORDS)]
        f = np.zeros(FINE, np.uint32)
        f[0] = k + 5
        cases.append(_case(f, base_word, k, name=f"bucket0_{k}"))  # edge 0: no raise
        f = np.zeros(FINE, np.uint32)
        f[0], f[7] = k, k - 1
        cases.append(_case(f, base_word, k, name=f"bucket0_with_k_minus_1_above_{k}"))
        f = np.zeros(FINE, np.uint32)
        f[FINE - 1] = k
        cases.append(_case(f, base_word, k, name=f"top_{k}"))
        f = np.zeros(FINE, np.uint32)
        np.add.at(f, rng.integers(0, FINE, size=k - 1), 1)
        cases.append(_case(f, base_word, k, name=f"fewer_than_k_{k}"))
        # fine counts trailing the coarse ones: cb's coarse count already holds k, its fine counts hold less than need
        for cb in (5, 32, 63):
            f = np.zeros(FINE, np.uint32)
            f[cb * 32 + 20] = k // 2
            co = _coarse_of(f)
            co[cb] = k
            cases.append(_case(f, base_word, k, coarse=co, name=f"fine_trailing_{cb}_{k}"))
            # ... and some of the coarse buckets above cb trail their fine counts' coarse sums
            f2 = f.copy()
            f2[(cb - 1) * 32 + 3] = k  # fine counts leading: the coarse bucket below has not seen them yet
            co2 = _coarse_of(f2)
            co2[cb - 1] = 0
            co2[cb] = k
            cases.append(_case(f2, base_word, k, coarse=co2, name=f"fine_leading_below_{cb}_{k}"))
            f3 = f.copy()
            f3[cb * 32 + 31] = k  # fine counts of cb leading its coarse count
            co3 = _coarse_of(f3)
            co3[cb] = k - (k > 1)
            co3[cb - 1] = 2
            cases.append(_case(f3, base_word, k, coarse=co3, name=f"fine_leading_{cb}_{k}"))
    for base_word in BASE_WORDS:  # every base word with a spread of counts
        for k in KS:
            f = np.zeros(FINE, np.uint32)
            np.add.at(f, rng.integers(0, FINE, size=k + int(rng.integers(0, 3 * k + 2))), 1)
            cases.append(_case(f, base_word, k, name=f"spread_{base_word:x}_{k}"))
    return cases


def sweep_cases(n, seed=0x5EED):
    """Seeded: counts bunched around a random bucket, k of KS, a random base word, then fine or coarse counts held back by a
    random amount (as a refresh reads them while other pushes are between their two atomics)."""
    rng = np.random.default_rng(seed)
    cases = []
    for i in range(n):
        k = int(rng.choice(KS))
        total = int(rng.integers(max(1, k - 3), 4 * k + 40))
        centre, spread = rng.integers(0, FINE), rng.choice([1, 4, 40, 400])
        b = np.clip(np.rint(rng.normal(centre, spread, size=total)), 0, FINE - 1).astype(np.int64)
        fine = np.bincount(b, minlength=FINE).astype(np.uint32)
        coarse = _coarse_of(fine)
        kind = i % 3
        if kind == 1:  # fine counts trailing
            held = rng.integers(0, 3, size=FINE).astype(np.uint32)
            fine = fine - np.minimum(fine, held)
        elif kind == 2:  # coarse counts trailing
            held = rng.integers(0, 3, size=COARSE).astype(np.uint32)
            coarse = coarse - np.minimum(coarse, held)
        cases.append(_case(fine, int(rng.choice(BASE_WORDS)), k, coarse=coarse, name=f"sweep_{i}"))
    return cases


def with_thetas(cases):
    """Each case with an old threshold of 0, and below, at and above the edge the model picks."""
    out = []
    for c in cases:
        _, _, b = refresh(c["fine"], c["coarse"], c["base_word"], c["k"], 0)
        edge = 0 if b is None else th_hist_edge(b, th_hist_base(c["base_word"]))
        for theta in sorted({0, max(edge - 1, 0), edge, min(edge + 1, 0xFFFFFFFF), 0xFFFFFFFF if edge else 0x3F800000}):
            out.append(dict(c, theta=theta))
    return out


# ---- CPU: the model against its own soundness check ------------------------------------------------------------------------
def test_refresh_model_is_sound():
    cases = with_thetas(hand_cases() + sweep_cases(600))
    kinds = collections.Counter()
    for c in cases:
        theta1, raised, b = refresh(c["fine"], c["coarse"], c["base_word"], c["k"], c["theta"])
        check_sound(c["fine"], c["coarse"], c["base_word"], c["k"], c["theta"], theta1, raised)
        name = c["name"]
        base = th_hist_base(c["base_word"])
        if name.startswith("coarse_edge_"):
            cb = int(name.split("_")[2])
            assert b == cb * 32
            kinds["coarse_edge"] += 1
        elif name.startswith("fine_edge_"):
            _, _, cb, ln = name.split("_")
            assert b == int(cb) * 32 + int(ln)
        elif name.startswith("bucket0"):
            assert b == 0 and theta1 == c["theta"] and not raised
        elif name.startswith("top_"):
            assert b == FINE - 1 and theta1 == max(c["theta"], th_hist_edge(FINE - 1, base))
        elif name.startswith("fewer_than_k"):
            assert b is None and theta1 == c["theta"] and not raised
        elif name.startswith("fine_trailing"):
            assert b % 32 == 0  # the fine counts of cb hold less than need: cb's first bucket
            kinds["trailing"] += 1
        elif name.startswith("fine_leading_below"):
            assert b == int(name.split("_")[3]) * 32 + 20 or b == int(name.split("_")[3]) * 32
        if raised:
            kinds["raised"] += 1
        if b is not None and th_hist_edge(b, base) == c["theta"]:
            kinds["theta_at_edge"] += 1
    assert kinds["coarse_edge"] >= 64 * 3 * 2 and kinds["trailing"] > 0 and kinds["raised"] > 1000 and kinds["theta_at_edge"] > 100
    # the edges the base words give: the fallback window, the clamp at the top of the key space
    assert th_hist_edge(1, th_hist_base(0)) == (FALLBACK_BASE + 1) << 16
    assert th_hist_edge(FINE - 1, 0xFF80) == 0xFFFF0000 and th_hist_edge(1, 0xFFFF) == 0xFFFF0000
    assert th_hist_bucket(score_key(np.inf), 0xFF80) == 0 and th_hist_bucket(score_key(np.inf), 0xFF7F) == 1


def test_soundness_check_rejects_an_overshoot():
    """The check is not vacuous: one bucket above the model's choice, or the trailing case's fine choice, is refused."""
    f = np.zeros(FINE, np.uint32)
    f[100], f[140] = 1, 9
    co = _coarse_of(f)
    theta, raised, b = refresh(f, co, 0x8000, 10, 0)
    assert b == 100 and raised
    with pytest.raises(AssertionError):
        check_sound(f, co, 0x8000, 10, 0, th_hist_edge(101, 0x8000), True)
    f = np.zeros(FINE, np.uint32)
    f[5 * 32 + 20] = 3
    co = _coarse_of(f)
    co[5] = 8
    theta, raised, b = refresh(f, co, 0x8000, 8, 0)
    assert b == 5 * 32
    with pytest.raises(AssertionError):
        check_sound(f, co, 0x8000, 8, 0, th_hist_edge(5 * 32 + 20, 0x8000), True)


def test_push_trigger_rule():
    """The pushes n (1-based, per query) that put a query on the refresh list: n >= k and (n - k) % max(k // 4, 16) == 0."""
    assert [n for n in range(1, 60) if _triggers(n, 1)] == [1, 17, 33, 49]
    assert [n for n in range(1, 2000) if _triggers(n, 1024)] == [1024, 1280, 1536, 1792]
    assert [n for n in range(1, 60) if _triggers(n, 17)] == [17, 33, 49]


def _triggers(n, k):
    return n >= k and (n - k) % max(k // 4, 16) == 0


# ---- the device harness ---------------------------------------------------------------------------------------------------
def _harness():
    from tantivy_b200 import lib
    path = os.path.join(os.path.dirname(lib.SO_PATH), "libtile_theta_harness.so")
    h = C.CDLL(path)
    vp = C.c_void_p
    h.tq_theta_harness_layout.argtypes = [vp]
    h.tq_theta_harness_refresh.argtypes = [vp, vp, vp, C.c_uint32, vp]
    h.tq_theta_harness_push.argtypes = [vp, C.c_uint32, vp, C.c_uint32, vp, vp, vp, vp, vp]
    h.tq_theta_harness_samples.argtypes = [vp, vp, C.c_uint32, vp, vp, vp, C.c_uint32]
    lay = np.zeros(8, np.uint32)
    assert h.tq_theta_harness_layout(lay.ctypes.data) == 0
    assert lay[6] == WORDS and lay[3] == REFRESH_CAP
    return h, lay


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).to("cuda:0")


def _host(t, dtype=np.uint32):
    return t.cpu().numpy().view(dtype)


@pytest.mark.gpu
def test_refresh_against_the_model():
    h, _ = _harness()
    cases = with_thetas(hand_cases() + sweep_cases(3000))
    nq = len(cases)
    hist = np.zeros((nq, WORDS), np.uint32)
    queries = np.zeros((nq, 4), np.uint32)
    qstate = np.zeros((nq, 2), np.uint32)
    for i, c in enumerate(cases):
        hist[i, :FINE] = c["fine"]
        hist[i, FINE:BASE_WORD] = c["coarse"]
        hist[i, BASE_WORD] = c["base_word"]
        hist[i, BASE_WORD + 1:] = 0xFFFFFFFF  # (the rest of the region is never read)
        queries[i, 0] = c["k"]
        qstate[i, 0] = c["theta"]
    d_hist, d_q, d_st, d_raised = _dev(hist), _dev(queries), _dev(qstate), _dev(np.full(nq, 7, np.uint32))
    assert h.tq_theta_harness_refresh(d_hist.data_ptr(), d_q.data_ptr(), d_st.data_ptr(), nq, d_raised.data_ptr()) == 0
    theta, raised = _host(d_st).reshape(nq, 2)[:, 0], _host(d_raised)
    assert (_host(d_hist).reshape(nq, WORDS) == hist).all()  # read-only
    bad = []
    for i, c in enumerate(cases):
        t1, r1, _ = refresh(c["fine"], c["coarse"], c["base_word"], c["k"], c["theta"])
        if (int(theta[i]), bool(raised[i])) != (t1, r1):
            bad.append((c["name"], c["k"], hex(c["base_word"]), hex(c["theta"]), hex(int(theta[i])), hex(t1), int(raised[i]), r1))
            continue
        check_sound(c["fine"], c["coarse"], c["base_word"], c["k"], c["theta"], int(theta[i]), int(raised[i]))
    assert not bad, f"{len(bad)} of {nq} refreshes differ from the model: {bad[:6]}"


def _push_scenario(rng, alive_kind):
    """Queries with every k of KS (cap below, at and above what they are pushed), pushes over three launches."""
    nq = 64
    ks = np.array([KS[i % len(KS)] for i in range(nq)], np.uint32)
    ks[-28:] = 1 + (np.arange(28) % 3)  # many queries at k 1..3 trigger in the same launch: the refresh list overflows
    base_words = np.array([BASE_WORDS[i % len(BASE_WORDS)] for i in range(nq)], np.uint32)
    n_push = rng.integers(0, 3 * ks.astype(np.int64) + 40)
    caps = np.where(np.arange(nq) % 4 == 0, np.maximum(n_push // 2, 1), n_push + 8).astype(np.uint32)
    caps[5] = 0
    max_doc = 5000
    alive = None
    if alive_kind == "bits":
        alive = np.packbits(rng.random(max_doc) < 0.7, bitorder="little")
    pushes = []
    for q in range(nq):
        for _ in range(int(n_push[q])):
            mode = rng.integers(0, 8)
            if mode == 0:
                score = rng.choice([0.0, -0.0, np.inf, -1.5, 1e-30, 3e38])
            else:
                score = float(np.exp2(rng.uniform(-8, 14)))
            key = int(score_key(np.float32(score)))
            th = int(rng.choice([0, key, key + 1 if key < 0xFFFFFFFF else key, max(key - 1, 0),
                                 int(score_key(np.float32(np.exp2(rng.uniform(-8, 14)))))]))
            pushes.append((q, int(np.float32(score).view(np.uint32)), int(rng.integers(0, max_doc)), th))
    pushes = np.array(pushes, np.uint32)
    pushes = pushes[rng.permutation(len(pushes))]
    cut = np.sort(rng.integers(0, len(pushes), size=2))
    return ks, base_words, caps, alive, max_doc, np.split(pushes, cut)


@pytest.mark.gpu
@pytest.mark.parametrize("alive_kind", ["bits", "none"])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_push_against_the_model(alive_kind, seed):
    h, lay = _harness()
    n_ctl, w_nref, w_ref, cap_ref, n_guard = (int(x) for x in lay[:5])
    rng = np.random.default_rng(0x9057 + seed)
    ks, base_words, caps, alive, max_doc, launches = _push_scenario(rng, alive_kind)
    nq = len(ks)
    gap = 8  # sentinel candidates after every region
    bases = np.concatenate([[0], np.cumsum(caps.astype(np.int64) + gap)[:-1]]).astype(np.uint32)
    n_cand = int(bases[-1]) + int(caps[-1]) + gap
    queries = np.stack([ks, bases, caps, np.zeros(nq, np.uint32)], axis=1)
    hist = np.zeros((nq, WORDS), np.uint32)
    hist[:, BASE_WORD] = base_words
    sentinel = np.uint32(0xDEADBEEF)
    d_q, d_st = _dev(queries), _dev(np.zeros((nq, 2), np.uint32))
    d_c, d_h = _dev(np.full((n_cand, 4), sentinel, np.uint32)), _dev(hist)
    d_alive = _dev(np.concatenate([alive, np.zeros(-len(alive) % 4, np.uint8)]).view(np.uint32)) if alive is not None else None
    want_fine = np.zeros((nq, FINE), np.int64)
    count = np.zeros(nq, np.int64)
    launch_cands, nrefs = [], []
    for li, pushes in enumerate(launches):
        seg = 100 + li
        d_p = _dev(pushes.reshape(-1, 4) if len(pushes) else np.zeros((1, 4), np.uint32))
        d_ctl = _dev(np.zeros(n_ctl, np.uint32))
        rc = h.tq_theta_harness_push(d_p.data_ptr(), len(pushes), d_alive.data_ptr() if d_alive is not None else None, seg,
                                     d_q.data_ptr(), d_st.data_ptr(), d_c.data_ptr(), d_h.data_ptr(), d_ctl.data_ptr())
        assert rc == 0
        before = count.copy()
        passing = collections.defaultdict(list)
        for q, sbits, doc, th in pushes:
            key = int(score_key(np.uint32(sbits).view(np.float32)))
            if key < th or (alive is not None and not (alive[doc >> 3] >> (doc & 7)) & 1):
                continue
            passing[int(q)].append((key, seg, int(doc), 0))
            count[q] += 1
            want_fine[q, th_hist_bucket(key, th_hist_base(base_words[q]))] += 1
        triggers = collections.Counter()
        for q in range(nq):
            for n in range(int(before[q]) + 1, int(count[q]) + 1):
                if _triggers(n, int(ks[q])):
                    triggers[q] += 1
        ctl = _host(d_ctl)
        nref = int(ctl[w_nref])
        assert nref == sum(triggers.values()), (li, nref, triggers)
        stored = collections.Counter(int(x) for x in ctl[w_ref:w_ref + min(nref, cap_ref)])
        assert sum(stored.values()) == min(nref, cap_ref) and not stored - triggers, (stored, triggers)
        untouched = np.ones(n_ctl, bool)
        untouched[w_nref] = False
        untouched[w_ref:w_ref + min(nref, cap_ref)] = False
        pattern = (np.uint32(0xC7A5E000) ^ (np.arange(n_ctl, dtype=np.uint64) * 0x9E3779B9 & 0xFFFFFFFF).astype(np.uint32))
        assert int(pattern[0]) == int(lay[5])
        assert (ctl[untouched] == pattern[untouched]).all(), np.nonzero(ctl != pattern)  # guards and the rest of TileCtl
        assert n_guard == 32
        launch_cands.append((before, passing))
        nrefs.append(nref)
    st = _host(d_st).reshape(nq, 2)
    assert (st[:, 0] == 0).all() and (st[:, 1] == count).all()
    got_hist = _host(d_h).reshape(nq, WORDS)
    assert (got_hist[:, :FINE] == want_fine).all()
    assert (got_hist[:, FINE:BASE_WORD] == want_fine.reshape(nq, COARSE, 32).sum(axis=2)).all()
    assert (got_hist[:, BASE_WORD] == base_words).all() and (got_hist[:, BASE_WORD + 1:] == 0).all()
    cands = _host(d_c).reshape(n_cand, 4)
    for q in range(nq):
        b0, cap = int(bases[q]), int(caps[q])
        assert (cands[b0 + min(int(count[q]), cap):b0 + cap + gap] == sentinel).all(), q  # nothing at or past the cap
        for before, passing in launch_cands:
            lo = int(before[q])
            hi = min(lo + len(passing[q]), cap)
            if lo >= hi:
                continue
            got = collections.Counter(tuple(int(x) for x in r) for r in cands[b0 + lo:b0 + hi])
            want = collections.Counter(passing[q])
            assert sum(got.values()) == hi - lo and not got - want, (q, got - want)
            if lo + len(passing[q]) <= cap:
                assert got == want, q
    assert max(nrefs) > cap_ref  # the refresh list overflowed
    assert (count > caps).any() and (count[ks == 1] >= 17).any()


def sample_base(samples, k, theta):
    """(threshold, base word) after k_theta_samples: the k-th largest sample key (0 when there are fewer than k), raised into the
    threshold before; the base word is that threshold's key >> 16."""
    s = np.sort(np.asarray(samples, dtype=np.uint64))[::-1]
    kth = int(s[k - 1]) if len(s) >= k else 0
    t = max(int(theta), kth)
    return t, t >> 16


def _sample_cases(rng, cap):
    """(samples held, count written, k, threshold before): fewer than k samples with and without a threshold before, exactly k,
    more, counts past the cap, ties at the k-th key, keys at the top and bottom of the key space, a threshold above the k-th."""
    cases = []
    for k in KS:
        for n in sorted({0, max(k - 1, 0), k, k + 1, min(3 * k, cap), cap}):
            for kind in range(4):
                if kind == 0:
                    keys = score_key(np.exp2(rng.uniform(-6, 14, size=n)).astype(np.float32))
                elif kind == 1:  # ties: few distinct keys
                    keys = rng.choice(score_key(np.float32([0.5, 1.0, 7.25, 7.25])), size=n)
                elif kind == 2:  # the ends: +inf, negative scores, +-0.0
                    keys = rng.choice(score_key(np.float32([np.inf, -1.5, -3e38, 0.0, -0.0, 1e-30])), size=n)
                else:  # low halves that the base word drops
                    keys = (rng.integers(0x8000, 0x10000, size=n) << 16 | rng.integers(0, 0x10000, size=n)).astype(np.uint32)
                for theta in (0, int(score_key(np.float32(3.0))), 0xFFFF1234):
                    count = n if n < cap or kind != 3 else n + 17  # (more written than the region holds: only cap are read)
                    cases.append((keys.astype(np.uint32), count, k, theta))
    return cases


@pytest.mark.gpu
def test_sample_base_word_against_the_model():
    """k_theta_samples: the threshold after the sample launch and the base word it writes for the exact launches' histograms."""
    h, _ = _harness()
    rng = np.random.default_rng(0xBA5E)
    cap = 2048
    cases = _sample_cases(rng, cap)
    nq = len(cases)
    samples = np.zeros((nq, cap), np.uint32)
    counts = np.zeros(nq, np.uint32)
    queries = np.zeros((nq, 4), np.uint32)
    qstate = np.zeros((nq, 2), np.uint32)
    hist = np.full((nq, WORDS), 0xA5A5A5A5, np.uint32)
    for i, (keys, count, k, theta) in enumerate(cases):
        samples[i, :len(keys)] = keys
        counts[i] = count
        queries[i, 0] = k
        qstate[i, 0] = theta
    d_s, d_n, d_q, d_st, d_h = _dev(samples), _dev(counts), _dev(queries), _dev(qstate), _dev(hist)
    assert h.tq_theta_harness_samples(d_s.data_ptr(), d_n.data_ptr(), cap, d_q.data_ptr(), d_st.data_ptr(), d_h.data_ptr(), nq) == 0
    theta = _host(d_st).reshape(nq, 2)[:, 0]
    got = _host(d_h).reshape(nq, WORDS)
    bad = []
    for i, (keys, count, k, th0) in enumerate(cases):
        held = keys[:min(count, cap)]
        t, base = sample_base(held, k, th0)
        if (int(theta[i]), int(got[i, BASE_WORD])) != (t, base):
            bad.append((i, k, len(held), hex(th0), hex(int(theta[i])), hex(t), hex(int(got[i, BASE_WORD])), hex(base)))
    assert not bad, f"{len(bad)} of {nq} differ from the model: {bad[:6]}"
    others = np.ones(WORDS, bool)
    others[BASE_WORD] = False
    assert (got[:, others] == 0xA5A5A5A5).all()  # only the base word is written
    # the fallback case is reached: fewer than k samples and no threshold before leave base word 0
    assert any(len(c[0]) < c[2] and c[3] == 0 for c in cases)
