"""The scenes of tests/bow_domain_scenes.py on the CPU: each one contains the boundary events it is built for (counted on the
oracle's output), and on them the oracle equals the reference's own DBoW2 / ORBmatcher.cc / MapPoint.cc (oracle/_ref)."""
import os

import numpy as np
import pytest

import bow_domain_scenes as S
import oracle as O
from oracle import ref as R

HAVE_REF = R.available() or os.path.isdir(os.path.join(R.REFERENCE_ROOT, "src"))
needs_ref = pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref is built from /root/reference, which is absent, and no prebuilt "
                                                    "library travels with this checkout")


def test_kp_dtype_matches_the_oracle():
    assert S.KP_DTYPE == O.KP_DTYPE


# ---- scenes do what they are built for --------------------------------------------------------------------------------------
def test_distance_set_and_knn2_scenes():
    q, t, d = S.distance_set()
    assert np.array_equal(S.hamming(q, t), d) and set(d.tolist()) == set(range(257))
    assert all(O.hamming(q[i], t[i]) == d[i] for i in range(0, len(d), 37))
    for g in (1, 127, 128, 129, 255, 256, 1000):
        qq, db, planted = S.knn2_scene(g, 257)
        bd, bi, sd = O.knn2(qq, db[:g])
        D = S.hamming(qq[:, None, :], db[None, :g, :])
        assert np.array_equal(bd, D.min(1)) and np.array_equal(bi, D.argmin(1))
        for qi, grp, pos in planted:
            assert bd[qi] == 10 and bi[qi] == pos[0] and sd[qi] == 10, (g, qi, pos)   # a tie: first index, second == best
        if g == 1:
            assert np.all(sd == 2 ** 31 - 1)


@pytest.mark.parametrize("k", [1, 2, 31, 32, 33, 64, 100])
def test_tie_vocabulary_queries_tie_where_built(k):
    L = 6 if k <= 33 else 3
    voc = S.tie_vocabulary(k, L, seed=k)
    q, labels = S.tie_queries(voc, seed=k)
    c = voc["node_desc"][1:1 + k]
    D = S.hamming(q[:, None, :], c[None, :, :])
    for i, lab in enumerate(labels):
        if lab.startswith("tie"):
            a, b = map(int, lab.split()[1].split("/"))
            assert D[i, a] == D[i, b] and np.sum(D[i] == D[i].min()) == 2 and D[i, a] == D[i].min(), lab
        elif lab.startswith("all"):
            assert np.all(D[i] == D[i, 0])
        elif lab == "distance 0":
            assert D[i].min() == 0
    if k == 1:
        assert D[labels.index("complement"), 0] == 256
    # the descent takes the first minimum on every level: root child a, then child 0 of every deeper node
    leaf, _ = O.bow_descend(voc, q, 0)
    start = voc["level_start"]
    for i, lab in enumerate(labels):
        p = int(np.argmin(D[i]))
        node = 1 + p
        for l in range(2, L + 1):
            node = int(voc["children"][voc["child_ptr"][node]])
        assert leaf[i] == node, (k, lab)
    assert leaf.min() >= start[L]


def test_orbvoc_shape_ids_pass_2_16_and_2_20():
    voc = S.orbvoc_shape_vocabulary()
    assert len(voc["node_desc"]) == 1111111
    q, ids = S.orbvoc_queries(voc, 16)
    leaf, node = O.bow_descend(voc, q, 1)
    assert (leaf >= 1 << 20).sum() >= 4 and (node >= 1 << 16).sum() >= 8


def _run_bow(variant, f1, f2, nnratio, ori):
    return O.search_by_bow(variant, f1.desc, f1.flag, f1.kps["angle"], f1.fv(), f2.desc, f2.flag, f2.kps["angle"], f2.fv(),
                           nnratio=nnratio, check_orientation=ori)


def test_bow_boundary_pair_events():
    f1, f2, E = S.bow_boundary_pair()
    seen = set()
    for v in (0, 1):
        for r in S.BOW_RATIOS:
            n, out = _run_bow(v, f1, f2, r, False)
            for lab, i1, i2 in E.applicable(variant=v, nnratio=r):
                assert S.match_of(v, out, i1) == i2, (v, r, lab)
                seen.add(lab.split(" at ")[0])
    for must in ("TH_LOW 50 v0", "TH_LOW 50 v1", "ratio 30/40", "ratio 30/50", "tie 31/32", "tie 5/37", "contention 3",
                 "contention fallback rejected 2", "lone valid v1", "invalid best v0", "length 300 best 150 second 151"):
        assert must in seen, must
    assert F32_ratio_facts()


def F32_ratio_facts():
    f = np.float32
    return f(0.75) * f(40) == f(30) and f(0.6) * f(50) > f(30) and 0.6 * 50 <= 30.0000000001


def _kept(variant, out, pairs):
    return [S.match_of(variant, out, i1) == i2 for i1, i2 in pairs]


def test_rotation_scenes():
    sweep = S.rotation_sweep()
    assert any(S.rot_bin(*m) != S.rot_bin_div(*m) for m in sweep)   # round(rot*(1.0f/30)) and round(rot/30) part somewhere
    assert {S.rot_bin(*m) for m in sweep} >= set(range(13))
    jobs = S.rotation_jobs()
    assert sum(not all(k) for _, _, k in jobs) > 20 and sum(all(k) for _, _, k in jobs) > 20
    for j, (name, matches, kept) in enumerate(jobs):
        f1, f2, pairs = S.rotation_pair(matches, j)
        for v in (0, 1):
            _, out = _run_bow(v, f1, f2, 0.75, True)
            assert _kept(v, out, pairs) == kept, (name, v)
            _, out = _run_bow(v, f1, f2, 0.75, False)
            assert all(_kept(v, out, pairs)), (name, v)
        f1, f2, pairs = S.rotation_pair(matches, j, kind="tri")
        _, m12 = _run_tri(f1, f2, S.F12_LINE_Y, S.sigma2(8), True)
        assert [m12[i1] == i2 for i1, i2 in pairs] == kept, name


def _run_tri(f1, f2, F12, sig2, ori):
    return O.search_for_triangulation(f1.kps, f1.desc, f1.flag, f1.fv(), f2.kps, f2.desc, f2.flag, f2.fv(), F12, sig2,
                                      check_orientation=ori)


@pytest.mark.parametrize("nlevels", [8, 32])
def test_triangulation_boundary_pair_events(nlevels):
    f1, f2, E, sig2 = S.tri_boundary_pair(nlevels=nlevels)
    _, m12 = _run_tri(f1, f2, S.F12_LINE_Y, sig2, False)
    for lab, i1, i2 in E.applicable():
        assert m12[i1] == i2, lab
    # a y2 the reference's double comparison accepts and a float comparison would reject
    edges = S.epipolar_edges(sig2)
    assert any(ok and not (np.float32(y * y) < np.float32(3.84 * float(sig2[l]))) for l, y, ok in edges)
    assert any(abs(float(y) - 1.9595917) < 1e-6 for l, y, ok in edges if l == 0 and ok)
    _, m12 = _run_tri(f1, f2, np.zeros(9, np.float32), sig2, False)
    assert np.all(m12 == -1)


@pytest.mark.parametrize("kind", ["bow", "tri"])
def test_big_pairs(kind):
    f1, f2, E = S.big_pair(kind)
    if kind == "bow":
        for v in (0, 1):
            _, out = _run_bow(v, f1, f2, 0.75, True)
            for lab, i1, i2 in E.applicable():
                assert S.match_of(v, out, i1) == i2, (v, lab)
    else:
        _, m12 = _run_tri(f1, f2, S.F12_LINE_Y, S.sigma2(8), True)
        for lab, i1, i2 in E.applicable():
            assert m12[i1] == i2, lab


def test_distinctive_groups():
    groups = S.distinctive_groups()
    ptr = np.concatenate([[0], np.cumsum([len(g) for _, g in groups])]).astype(np.int32)
    best = O.distinctive_descriptors(np.concatenate([g for _, g in groups]), ptr)
    edges = 0
    for (lab, g), b in zip(groups, best):
        med = S.medians(g)
        assert b == int(np.argmin(med)), lab
        if lab.startswith("lane edge"):
            assert b == 1 and med[1] == int(lab.split()[-1]) and med[2] == med[1], lab
            edges += 1
        if lab.startswith("row-0 lane edge"):
            assert b == 1 and med[0] == int(lab.split()[-1]) and med[1] == med[2] == 1, lab
            edges += 1
        if lab.startswith("complement 3"):
            assert med[0] == 256
    assert edges == 37 + 56
    # no group reaches a least median above 170 (see distinctive_groups): the largest one is on the 170/171 edge
    assert max(S.medians(g).min() for _, g in groups) == 170


def test_fv_numpy_is_dbow2s_feature_vector():
    """The numpy restatement the GPU FeatureVector sweep is checked against equals the oracle's DBoW2 transform (which
    test_tie_vocabularies_against_dbow2 pins to the reference) on leaf / node ids from a real descent, stopped word included."""
    voc = S.tie_vocabulary(40, 4, seed=9)
    live = voc["weight"] > 0
    q, _ = S.tie_queries(voc, seed=9)
    rng = np.random.default_rng(3)
    desc = np.concatenate([q[rng.integers(0, len(q), 3000)], rng.integers(0, 256, (1000, 32), dtype=np.uint8)])
    stopped = 0
    for levelsup in (0, 2, 4):
        leaf, node = O.bow_descend(voc, desc, levelsup)
        stopped += int((~live[leaf]).sum())
        got = S.fv_numpy(leaf, node, len(desc), len(desc), live)
        want = O.bow_transform(voc, desc, levelsup)[1]
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), levelsup
    assert stopped > 0


def test_fv_frames_events():
    live = np.ones(64, bool)
    live[[5, 9]] = False
    leaf, node, counts = S.fv_frames(2049, 64, live)
    ids, ptr, items = S.fv_numpy(leaf[9], node[9], counts[9], 2049, live)
    assert list(ptr[1:3]) == [1024, 2048]
    ids, ptr, items = S.fv_numpy(leaf[3], node[3], counts[3], 2049, live)
    assert ptr[-1] < 2049 and len(ids) > 100   # stopped and out-of-range leaves dropped
    assert {0, 2 ** 31 - 1} <= set(S.fv_numpy(leaf[10], node[10], counts[10], 2049, live)[0].tolist())


# ---- the oracle equals the reference's own code on these scenes --------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("k,L", [(1, 6), (2, 6), (31, 4), (32, 4), (33, 4), (64, 3), (100, 3)])
def test_tie_vocabularies_against_dbow2(tmp_path, k, L):
    voc = S.tie_vocabulary(k, L, seed=k)
    q, _ = S.tie_queries(voc, seed=k)
    path = str(tmp_path / "voc.txt")
    R.write_vocabulary_text(voc, path)
    V = R.RefVocabulary(path)
    for levelsup in (0, 1, 4, L - 1, L, L + 1, 1000):
        ref = V.transform(q, levelsup)
        orc = O.bow_transform(voc, q, levelsup=levelsup, weighting=0, norm=1)
        for a, b in zip(ref[0] + ref[1], orc[0] + orc[1]):
            assert np.array_equal(a, b), (k, L, levelsup)


def _ref_keyframe(Sc, fr, nlevels=8):
    f = Sc.frame(fr.kps, fr.desc, 640, 480, 500.0, 500.0, 320.0, 240.0, 1.2, nlevels)
    kf = Sc.keyframe(f, np.eye(4, dtype=np.float32)[:3])
    Sc.set_feature_vector(kf, fr.fv())
    ids = np.full(len(fr.desc), -1, np.int64)
    for i in np.flatnonzero(fr.flag):
        ids[i] = Sc.map_point(np.array([0, 0, 4], np.float32), fr.desc[i], None, 1.0, 30.0, kf)
        Sc.observe(kf, ids[i], i)
    return f, kf, {int(m): i for i, m in enumerate(ids) if m >= 0}


def _ref_bow(Sc, variant, f1, f2, nnratio, ori):
    fa, kf1, to1 = _ref_keyframe(Sc, f1)
    fb, kf2, to2 = _ref_keyframe(Sc, f2)
    if variant == 0:
        Sc.set_feature_vector(fb, f2.fv())
        n, mp = Sc.search_by_bow_kf_frame(kf1, fb, nnratio, ori)
        out = np.array([to1.get(int(m), -1) for m in mp], np.int32)
    else:
        n, mp = Sc.search_by_bow_kf_kf(kf1, kf2, nnratio, ori)
        out = np.array([to2.get(int(m), -1) for m in mp], np.int32)
    fa.close(); fb.close()
    return n, out


@needs_ref
def test_bow_scenes_against_orbmatcher():
    Sc = R.Scene("ref")
    f1, f2, _ = S.bow_boundary_pair()
    for v in (0, 1):
        for r in S.BOW_RATIOS:
            assert [np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b
                    for a, b in zip(_ref_bow(Sc, v, f1, f2, r, False), _run_bow(v, f1, f2, r, False))] == [True, True], (v, r)
    jobs = S.rotation_jobs()
    for j, (name, matches, _) in enumerate(jobs[:6] + jobs[6::5]):
        f1, f2, _ = S.rotation_pair(matches, j)
        for v in (0, 1):
            n_r, o_r = _ref_bow(Sc, v, f1, f2, 0.75, True)
            n_o, o_o = _run_bow(v, f1, f2, 0.75, True)
            assert n_r == n_o and np.array_equal(o_r, o_o), (name, v)


def _ref_tri(Sc, f1, f2, F12, ori, nlevels=8):
    fa, kf1, _ = _ref_keyframe(Sc, f1, nlevels)
    fb, kf2, _ = _ref_keyframe(Sc, f2, nlevels)
    n, pairs = Sc.search_for_triangulation(kf1, kf2, F12, 0.6, ori)
    fa.close(); fb.close()
    return n, pairs


@needs_ref
@pytest.mark.parametrize("nlevels", [8, 32])
def test_triangulation_scenes_against_orbmatcher(nlevels):
    Sc = R.Scene("ref")
    f1, f2, _, sig2 = S.tri_boundary_pair(nlevels=nlevels)
    for F12 in (S.F12_LINE_Y, np.zeros(9, np.float32)):
        n_r, pairs = _ref_tri(Sc, f1, f2, F12, False, nlevels)
        n_o, m12 = _run_tri(f1, f2, F12, sig2, False)
        want = np.array([(i, m12[i]) for i in range(len(m12)) if m12[i] >= 0], np.int32).reshape(-1, 2)
        assert n_r == n_o and np.array_equal(pairs, want)
    jobs = S.rotation_jobs()
    for j, (name, matches, _) in enumerate(jobs[:6] + jobs[6::7]):
        f1, f2, _ = S.rotation_pair(matches, j, kind="tri")
        n_r, pairs = _ref_tri(Sc, f1, f2, S.F12_LINE_Y, True)
        n_o, m12 = _run_tri(f1, f2, S.F12_LINE_Y, S.sigma2(8), True)
        want = np.array([(i, m12[i]) for i in range(len(m12)) if m12[i] >= 0], np.int32).reshape(-1, 2)
        assert n_r == n_o and np.array_equal(pairs, want), name


@needs_ref
def test_distinctive_groups_against_mappoint():
    import ctypes as C
    Sc = R.Scene("ref")
    L = Sc.L
    L.ref_mp_observation_order.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    small = [(lab, g) for lab, g in S.distinctive_groups() if len(g) <= 40]
    nk = max(len(g) for _, g in small)
    kps = np.zeros(1, O.KP_DTYPE)
    kps["x"], kps["y"] = 100.0, 100.0
    checked = 0
    for lab, g in small:
        kfs = []
        for d in g:
            f = Sc.frame(kps, d[None, :], 640, 480, 500.0, 500.0, 320.0, 240.0)
            kfs.append(Sc.keyframe(f, np.eye(4, dtype=np.float32)[:3]))
            f.close()
        mp = Sc.map_point(np.array([0, 0, 4], np.float32), g[0], None, 1.0, 30.0, kfs[0])
        for kf in kfs:
            Sc.observe(kf, mp, 0)
        got = Sc.compute_distinctive(mp)
        ok_, oi_ = np.zeros(nk, np.int32), np.zeros(nk, np.int32)
        n = L.ref_mp_observation_order(mp, ok_.ctypes.data, oi_.ctypes.data, nk)
        order = np.stack([g[kfs.index(int(ok_[j]))] for j in range(n)])
        best = O.distinctive_descriptors(order, np.array([0, n], np.int32))
        assert np.array_equal(got, order[best[0]]), lab
        checked += 1
    assert checked > 40
