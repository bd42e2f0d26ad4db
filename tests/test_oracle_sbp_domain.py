"""The scenes of sbp_domain_scenes.py on the CPU: each scene holds the candidate lists it is designed for and produces its
facts on the sequential model (chain depths, the queries the kernel's warp receives after 48 rounds, the rule-0 pass
count, the MODE-2 re-assignments, the histogram counts); each named wrong variant of the loop changes the outcome of the
scenes that name it, and every variant is named by one; the oracle's guided search, SearchForInitialization and every
routine-level matcher the GPU file realises the scenes through (WindowSearch, SearchByProjection(F1, F2), the local-map
search, SearchByProjection(Frame, Frame) and SearchByProjection(Frame, KeyFrame)) equal the model index for index; where
the reference build is present, its own ORBmatcher equals the oracle on the same realisations.  SearchByProjection(Frame,
KeyFrame) is the exception: the reference reaches it only through a scripted map (tests/ref_scenarios.py, where
test_oracle_vs_ref.py pins the oracle's routine to it), not through frames built from arrays."""
import functools

import numpy as np
import pytest

import oracle as O
import sbp_domain_scenes as S


def _scenes():
    return ([S.chains_scene(1), S.chains_scene(2), S.tails_scene(1), S.tails_scene(2), S.tie_tails_scene(), S.star_scene(64),
             S.ladder_scene(), S.init_scene()] + S.hist_scenes())


SCENES = _scenes()
IDS = [s.name for s in SCENES]


def _frame(sc):
    return O.OracleFrame(sc.kps, sc.desc, S.W, S.H)


def _oracle(sc):
    f = _frame(sc)
    if sc.rule == 3:
        f1 = O.OracleFrame(S.f1_keypoints(sc), sc.qdesc, S.W, S.H)
        prev = np.stack([sc.qu, sc.qv], 1)
        n, m12, _ = O.search_for_initialization(f1, f, prev, int(S.R), nnratio=sc.nnratio, check_orientation=bool(sc.hist))
        return n, m12
    return O.guided_search(f, sc.qu, sc.qv, sc.qr, sc.qlo, sc.qhi, sc.qdesc, sc.qangle, sc.rule, sc.nnratio, sc.th_dist,
                           sc.hist, slot_owner=sc.slot_owner())


@pytest.mark.parametrize("sc", SCENES, ids=IDS)
def test_lists_and_distances_are_as_designed(sc):
    S.check_distances(sc)
    assert S.lists_of(sc, _frame(sc)) == sc.lists


@pytest.mark.parametrize("sc", SCENES, ids=IDS)
def test_oracle_equals_sequential_model(sc):
    n, so = _oracle(sc)
    n_m, so_m = S.sequential(sc)
    assert n == n_m and np.array_equal(so, so_m)


@pytest.mark.parametrize("sc", SCENES, ids=IDS)
def test_named_variants_change_the_outcome(sc):
    base = S.outcome(sc)
    for v in sc.changes:
        n, so = S.outcome(sc, v)
        assert n != base[0] or not np.array_equal(so, base[1]), v


def test_every_variant_is_named_by_a_scene():
    named = set(v for sc in SCENES for v in sc.changes)
    assert named == set(S.VARIANTS)


@pytest.mark.parametrize("rule", [1, 2])
def test_chain_schedule(rule):
    """Chain depth d: query i decides in round i + 1, so depths up to 48 finish inside the rounds and depth 49 is the first
    to hand its last query to the warp; the warp then sees the round-1/2 queries of the re-run and pick-only pairs
    (higher indices) as decided.  Free chains reject everything; blocked chains shift by one; the schedule's result is the
    sequential loop's."""
    sc = next(s for s in SCENES if s.name == "chains-rule%d" % rule)
    n, so, rnd, warp = S.rounds(sc)
    n_m, so_m = S.sequential(sc)
    assert n == n_m and np.array_equal(so, so_m)
    expect_warp = []
    for kind in ("free", "blocked"):
        for d, qs in sc.facts[kind].items():
            assert [rnd.get(q) for q in qs] == [i + 1 if i < 48 else None for i in range(d)], (kind, d)
            expect_warp += qs[48:]
            for i, q in enumerate(qs):
                taken = [s for s in range(sc.n) if so[s] == q]
                assert taken == ([sc.lists[q][1]] if kind == "blocked" else []), (kind, d, i)
    assert sorted(warp) == sorted(expect_warp) and len(warp) == 2 * (1 + 2 + 152)
    r, x = sc.facts["rerun"]
    assert (rnd[r], rnd[x]) == (1, 2) and so[sc.lists[r][0]] == -1 and so[sc.lists[x][0]] == x and r > warp[0]
    p0, p1 = sc.facts["pick_only"]
    assert (rnd[p0], rnd[p1]) == (1, 2) and so[sc.lists[p1][1]] == p1
    e = sc.facts["edges"]
    got = [int(any(so == q)) for q in e]
    assert got == ([1, 0, 1, 0] if rule == 1 else [1, 0, 1, 1, 0])


@pytest.mark.parametrize("name", ["tails-rule1", "tails-rule2", "ties-rule1"])
def test_tail_schedule(name):
    """The tail query of each 49-deep chain is the only query the warp receives, and it accepts: the single entry without a
    second (1), the best in the list's last chunk (31-65), ties at 31 / 32 broken by position (rule 2: best and second
    on two octaves; rule 1 with nnratio 1.0: best == second)."""
    sc = next(s for s in SCENES if s.name == name)
    rule = sc.rule
    tie = name != "tails-rule1"
    n, so, rnd, warp = S.rounds(sc)
    assert sorted(warp) == sorted(sc.facts["tails"].values())
    for L, q in sc.facts["tails"].items():
        assert len(sc.lists[q]) == L
        pos = sc.lists[q].index(int(np.flatnonzero(so == q)[0]))
        assert pos == (0 if L == 1 else 31 if (tie and L > 32) else L - 1), (L, pos)
    assert n == len(sc.facts["tails"]) and np.array_equal(so, S.sequential(sc)[1])


def test_star_and_ladder_passes():
    """Star of K queries on K slots: query q ends on slot q after K + 1 synchronous passes (the last changes nothing).
    Ladders: each query displaces the next, depth d takes d + 1 passes; a slot occupied inside the cascade leaves the
    query before it unmatched and the rest shifts on; th_dist is kept and th_dist + 1 dropped."""
    star = next(s for s in SCENES if s.name.startswith("star"))
    n, so, npass = S.passes(star)
    K = star.facts["K"]
    assert n == K and list(so) == list(range(K)) and npass == K + 1
    assert np.array_equal(so, S.sequential(star)[1])
    lad = next(s for s in SCENES if s.name == "ladders")
    n, so, npass = S.passes(lad)
    assert np.array_equal(so, S.sequential(lad)[1]) and npass == 200 + 1
    for d, qs in lad.facts["ladders"].items():
        assert [int(np.flatnonzero(so == q)[0]) for q in qs] == [lad.lists[q][1] for q in qs]
    holed = lad.facts["holed"]
    matched = [int(any(so == q)) for q in holed]
    assert matched == [0 if i in (19, 39) else 1 for i in range(60)]
    kept, dropped = lad.facts["th"]
    assert any(so == kept) and not any(so == dropped)


def test_star_1000_sequential():
    """The K = 1000 star of the GPU file: query q ends on slot q."""
    star = S.star_scene(1000)
    n, so = S.sequential(star)
    assert n == 1000 and list(so) == list(range(1000))
    n_o, so_o = _oracle(star)
    assert n_o == n and np.array_equal(so_o, so)


def test_init_reassignment_and_histogram():
    """MODE 2: q takes s at 20 and q + 1 falls back to t; the three-query re-assignment chain ends on its last query, the
    displaced ones keep their histogram entries (bin 5 holds 3 entries against 27 in bin 0, enough to keep p matched);
    lists of 32 and 40 entries accept their best; TH_LOW 50 kept and 51 dropped; 9 vs 12 dropped and 8 vs 12 kept."""
    sc = next(s for s in SCENES if s.name == "init")
    n, m12 = S.sequential(sc)
    q, s, t = sc.facts["prefetch"]
    assert m12[q] == s and m12[q + 1] == t
    chain, s2, p = sc.facts["reassign"]
    assert list(m12[chain]) == [-1, -1, s2] and m12[p] >= 0
    counts = S.hist_counts(sc)
    assert counts[5] == 3 and counts[0] == 27 and sum(counts) == 30
    assert [m12[x] >= 0 for x in sc.facts["long"]] == [True, True]
    assert [sc.lists[x].index(m12[x]) for x in sc.facts["long"]] == [31, 35]
    assert [m12[x] >= 0 for x in sc.facts["th"]] == [True, False]
    assert [m12[x] >= 0 for x in sc.facts["ratio"]] == [False, True]


def test_histogram_facts():
    """Bin counts and kept bins of the histogram scenes, float32 throughout: 0.1f * 10 == 1 and 0.1f * 20 == 2 (kept at
    equality), one below dropped; the first three of four tied maxima kept; +0 and -0.0 in bin 0, just below 0 in bin 12,
    the half-bin boundary between bins 0 and 1."""
    sc = {s.name: s for s in SCENES}
    lo, hi = S.half_bin_below()
    assert S.rot_bin(lo, 0.0) == 0 and S.rot_bin(hi, 0.0) == 1 and S.rot_bin(-0.0, 0.0) == 0 and S.rot_bin(0.0, 0.0) == 0
    tiny = float(np.nextafter(np.float32(0), np.float32(1)))
    assert S.rot_bin(-tiny, 0.0) == 12 and S.rot_bin(0.0, 0.0, "rot_le_zero_wrap") == 12
    expect = {"max2-at": (0, 3, -1), "max3-at": (0, 3, 6), "max2-below": (0, -1, -1), "max3-below": (0, 3, -1),
              "max-ties": (0, 4, 7), "angles": (0, 1, 12)}
    for name, keep in expect.items():
        assert S.three_maxima(S.hist_counts(sc[name])) == keep, name
    n_all = sum(len(v) for v in sc["angles"].facts["groups"].values())
    n, _ = S.sequential(sc["angles"])
    assert n_all - n == 3    # bins 7 (2) and 11 (1) dropped


def test_split_chain_geometry():
    """The split scene straddles the host entry's launch boundary: the first query of the second launch is inside the chain."""
    sc = S.split_chain_scene()
    qcap, chain = sc.facts["qcap"], sc.facts["chain"]
    assert chain[0] < qcap < chain[-1]
    n, so = S.sequential(sc)
    assert n == len(chain) and all(so[sc.lists[q][1]] == q for q in chain)
    n_o, so_o = _oracle(sc)
    assert n_o == n and np.array_equal(so_o, so)


# ---- the routine-level matchers the GPU file realises the scenes through: oracle == sequential loop ----

@functools.lru_cache(maxsize=None)
def scene(name):
    return S.star_scene(1000) if name == "star-1000" else next(s for s in SCENES if s.name == name)


RULE0 = ["ladders", "star-64", "star-1000", "max2-at", "max3-at", "max2-below", "max3-below", "max-ties", "angles"]
RULE1 = ["chains-rule1", "tails-rule1", "ties-rule1"]
RULE2 = ["chains-rule2", "tails-rule2"]
WIN = int(S.R)


def oracle_ff(sc, ori):
    """SearchByProjection(Frame, Frame, th = 6): the Last frame is S.f1_keypoints with the map points S.world_points."""
    has, outl = np.ones(sc.nq, np.uint8), np.zeros(sc.nq, np.uint8)
    return O.search_by_projection_ff(_frame(sc), O.OracleFrame(S.f1_keypoints(sc), sc.qdesc, S.W, S.H), has, outl,
                                     S.world_points(sc), S.T_ID, 1.0, 1.0, 0.0, 0.0, float(WIN), check_orientation=ori,
                                     cur_mp=sc.slot_owner())


def oracle_kf(sc, ori):
    """SearchByProjection(Frame, KeyFrame, th = 6, ORBdist = TH_HIGH): min_dist 1e9 predicts level 0 (octaves -1..1)."""
    return O.search_by_projection_kf(_frame(sc), np.ones(sc.nq, np.uint8), S.world_points(sc), np.full(sc.nq, 1e9, np.float32),
                                     sc.qdesc, sc.qangle, S.T_ID, 1.0, 1.0, 0.0, 0.0, float(WIN), S.TH_HIGH,
                                     check_orientation=ori, cur_mp=sc.slot_owner())


def oracle_window(sc):
    has, _ = S.window_search_view(sc)
    return O.window_search(O.OracleFrame(S.f1_keypoints(sc), sc.qdesc, S.W, S.H), _frame(sc), has, WIN, nnratio=sc.nnratio,
                           check_orientation=True)


def oracle_f1f2(sc):
    return O.search_by_projection_f1f2(O.OracleFrame(S.f1_keypoints(sc), sc.qdesc, S.W, S.H), _frame(sc), np.ones(sc.nq, np.uint8),
                                       S.world_points(sc), S.T_ID, 1.0, 1.0, 0.0, 0.0, WIN, nnratio=sc.nnratio,
                                       f2_mp=sc.slot_owner())


def local_points_args(sc):
    """SearchByProjection(Frame, vector<MapPoint*>, th = 1.25): predicted level 1 and view cosine 0 make the window
    4 * 1.25 * 1.2 px over octaves 0..1."""
    n = sc.nq
    return (np.ones(n, np.uint8), np.stack([sc.qu, sc.qv], 1).astype(np.float32), np.ones(n, np.int32), np.zeros(n, np.float32),
            sc.qdesc, 1.25)


def oracle_local_points(sc):
    return O.search_local_points(_frame(sc), *local_points_args(sc), nnratio=sc.nnratio, f_mp=sc.slot_owner())


def _same(got, want):
    assert got[0] == want[0] and np.array_equal(got[1], want[1])


@pytest.mark.parametrize("ori", [False, True])
@pytest.mark.parametrize("name", RULE0)
def test_projection_routines_equal_the_loop(name, ori):
    """Rule 0 through SearchByProjection(Frame, Frame) and (Frame, KeyFrame): the star and ladder cascades, the th_dist
    edges and the histogram scenes, with and without the histogram."""
    sc = scene(name)
    want = S.sequential(S.with_hist(sc, int(ori)))
    _same(oracle_ff(sc, ori), want)
    _same(oracle_kf(sc, ori), want)


@pytest.mark.parametrize("name", RULE1)
def test_window_search_and_f1f2_equal_the_loop(name):
    """Rule 1 through WindowSearch (no occupied slots: the queries whose list holds one are left out; its histogram holds
    one bin, all angles being 0) and through SearchByProjection(F1, F2) (occupied slots as F2's map points)."""
    sc = scene(name)
    _, view = S.window_search_view(sc)
    n, m21 = oracle_window(sc)
    assert n > 0
    _same((n, m21), S.sequential(S.with_hist(view, 1)))
    _same(oracle_f1f2(sc), S.sequential(sc))


@pytest.mark.parametrize("name", RULE2)
def test_local_points_equal_the_loop(name):
    sc = scene(name)
    _same(oracle_local_points(sc), S.sequential(sc))


# ---- the reference's own ORBmatcher on the same realisations ----

from oracle import ref as REF  # noqa: E402

needs_ref = pytest.mark.skipif(not REF.available(), reason="reference build (oracle/_ref) absent")


def _ref_frame(k, d):
    return REF.RefFrame.from_arrays(k, d, S.W, S.H, fx=1.0, fy=1.0, cx=0.0, cy=0.0)


@needs_ref
@pytest.mark.parametrize("name", RULE1)
def test_reference_window_search_and_f1f2(name):
    sc = scene(name)
    has, _ = S.window_search_view(sc)
    r1, r2 = _ref_frame(S.f1_keypoints(sc), sc.qdesc), _ref_frame(sc.kps, sc.desc)
    _same(REF.window_search(r1, r2, has, WIN, nnratio=sc.nnratio, check_orientation=True), oracle_window(sc))
    _same(REF.search_by_projection_f1f2(r1, r2, np.ones(sc.nq, np.uint8), S.world_points(sc), S.T_ID, WIN, nnratio=sc.nnratio,
                                        f2_mp=sc.slot_owner()), oracle_f1f2(sc))


@needs_ref
@pytest.mark.parametrize("ori", [False, True])
@pytest.mark.parametrize("name", RULE0)
def test_reference_search_by_projection_ff(name, ori):
    sc = scene(name)
    r_cur, r_last = _ref_frame(sc.kps, sc.desc), _ref_frame(S.f1_keypoints(sc), sc.qdesc)
    got = REF.search_by_projection_ff(r_cur, r_last, np.ones(sc.nq, np.uint8), np.zeros(sc.nq, np.uint8), S.world_points(sc),
                                      S.T_ID, float(WIN), check_orientation=ori, cur_mp=sc.slot_owner())
    _same(got, oracle_ff(sc, ori))


@needs_ref
@pytest.mark.parametrize("name", RULE2)
def test_reference_search_local_points(name):
    sc = scene(name)
    got = REF.search_local_points(_ref_frame(sc.kps, sc.desc), *local_points_args(sc), nnratio=sc.nnratio, f_mp=sc.slot_owner())
    _same(got, oracle_local_points(sc))


@needs_ref
def test_reference_search_for_initialization():
    sc = scene("init")
    f1k = S.f1_keypoints(sc)
    prev = np.stack([sc.qu, sc.qv], 1).astype(np.float32)
    n_o, m_o, p_o = O.search_for_initialization(O.OracleFrame(f1k, sc.qdesc, S.W, S.H), _frame(sc), prev, WIN, nnratio=sc.nnratio,
                                                check_orientation=True)
    n_r, m_r, p_r = REF.search_for_initialization(_ref_frame(f1k, sc.qdesc), _ref_frame(sc.kps, sc.desc), prev, WIN,
                                                  nnratio=sc.nnratio, check_orientation=True)
    assert n_o == n_r and np.array_equal(m_o, m_r) and np.array_equal(p_o, p_r)
    assert n_o == S.sequential(sc)[0]
