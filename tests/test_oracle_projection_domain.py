"""The projecting matchers at their rounding edges, on the CPU: on every scene of projection_domain_scenes.py (general poses,
TUM-like intrinsics, points on the image bounds, keypoints on the window edges, ratios on the scale factors, cosines on 0.998,
side-2 keypoints on the epipolar threshold) the restatement equals the oracle's SearchByProjection(Frame, Frame),
SearchByProjection(Frame, KeyFrame), SearchByProjection(F1, F2), the local-map search and SearchForTriangulation match for
match; each scene holds its facts; each named variant changes exactly the scenes that name it; and the reference's own
ORBmatcher equals the oracle on every scene."""
import numpy as np
import pytest

import oracle as O
import projection_domain_scenes as S
from oracle import ref as R

SCENES = S.scenes()
IDS = [s.name for s in SCENES]
ORB_W, ORB_H = S.W, S.H


def needs_ref():
    if not R.available():
        pytest.skip("oracle/_ref/libref_orbslam.so not built (needs the reference sources)")


def one_node(n):
    """a FeatureVector with every feature in node 0"""
    return np.array([0], np.int32), np.array([0, n], np.int32), np.arange(n, dtype=np.int32)


def frame(kps, desc, s):
    return O.OracleFrame(kps, desc, ORB_W, ORB_H, s.scale, s.nlevels)


def run_oracle(s, ori=True):
    """the oracle's routine on scene s: (nmatches, rows in the restatement's layout)"""
    if s.routine == "ff":
        n = len(s.world)
        return O.search_by_projection_ff(frame(s.cur_kps, s.cur_desc, s), frame(s.last_kps, s.last_desc, s), np.ones(n, np.uint8),
                                         np.zeros(n, np.uint8), s.world, s.T, S.FX, S.FY, S.CX, S.CY, s.th, check_orientation=ori)
    if s.routine == "kf":
        n = len(s.world)
        return O.search_by_projection_kf(frame(s.cur_kps, s.cur_desc, s), np.ones(n, np.uint8), s.world, s.min_dist, s.desc,
                                         np.zeros(n, np.float32), s.T, S.FX, S.FY, S.CX, S.CY, s.th, s.orb_dist, check_orientation=ori)
    if s.routine == "f1f2":
        return O.search_by_projection_f1f2(frame(s.f1_kps, s.f1_desc, s), frame(s.f2_kps, s.f2_desc, s), np.ones(len(s.world), np.uint8),
                                           s.world, s.T, S.FX, S.FY, S.CX, S.CY, s.window, nnratio=s.nnratio)
    if s.routine == "local":
        return O.search_local_points(frame(s.kps, s.desc, s), np.ones(len(s.proj), np.uint8), s.proj, s.level, s.view_cos, s.mp_desc,
                                     s.th, nnratio=s.nnratio)
    n1, n2 = len(s.k1), len(s.k2)
    return O.search_for_triangulation(s.k1, s.d1, np.zeros(n1, np.uint8), one_node(n1), s.k2, s.d2, np.zeros(n2, np.uint8),
                                      one_node(n2), s.F12, s.sig2, check_orientation=ori)


@pytest.mark.parametrize("s", SCENES, ids=IDS)
def test_restatement_equals_oracle(s):
    n, rows = s.run()
    for ori in (True, False):
        n_o, rows_o = run_oracle(s, ori)
        assert n_o == n and np.array_equal(rows_o, rows), ori


def _matched(s, rows, q):
    return rows[q] >= 0 if s.routine == "tri" else q in rows


def window_radius(s, q):
    """the search radius of query q as the routine computes it"""
    sf = S.scale_table(s.scale, s.nlevels)
    if s.routine == "f1f2":
        return np.float32(s.window)
    if s.routine == "ff":
        return np.float32(s.th) * sf[s.last_kps["octave"][q]]
    if s.routine == "kf":
        lv = S.predicted_level(np.float32(S.dist3d(s.T, s.world[q])[0] / s.min_dist[q]), sf)
        return np.float32(s.th) * sf[lv]
    return np.float32(S.view_radius(s.view_cos[q]) * np.float32(s.th)) * sf[s.level[q]]


@pytest.mark.parametrize("s", SCENES, ids=IDS)
def test_facts(s):
    """every query matches as its decision says, and sits where it claims"""
    n, rows = s.run()
    assert len(s.facts) >= 8
    assert {q for q, _, _ in s.facts} == set(range(len(s.facts)))
    assert n == sum(m for _, _, m in s.facts)
    for q, label, matched in s.facts:
        assert _matched(s, rows, q) == matched, label
    if s.routine in ("ff", "kf", "f1f2"):
        u, v = S.project(s.T, s.world)
    if "bounds" in s.name:
        for q, label, matched in s.facts:
            side = next(sd for sd in S.SIDES if label.endswith(sd[0]))
            val = (u, v)[side[1]][q]
            assert (val == side[2]) == matched and (val - side[2]) * side[3] >= 0, label
            if not matched and side[2] != 0:
                assert val == S.steps(side[2], side[3]), label
    if "window" in s.name or s.routine == "local":
        k = s.f2_kps if s.routine == "f1f2" else s.kps if s.routine == "local" else s.cur_kps
        uu, vv = (s.proj[:, 0], s.proj[:, 1]) if s.routine == "local" else (u, v)
        for q, label, matched in s.facts:
            if label.startswith("at r") or label.startswith("beyond r"):
                d = abs(np.float32(k["x"][q] - uu[q])) if " dx " in label else abs(np.float32(k["y"][q] - vv[q]))
                r = window_radius(s, q)
                assert (d == r) == label.startswith("at r") and d >= r, label
                assert 20 <= uu[q] < 32 and 20 <= vv[q] < 32
    if s.routine == "kf" and "level" in s.name:
        d3 = S.dist3d(s.T, s.world)
        sf = S.scale_table(s.scale, s.nlevels)
        for q, label, matched in s.facts:
            ratio = np.float32(d3[q] / s.min_dist[q])
            if label.startswith("ratio =="):
                assert ratio == sf[int(label.split("[")[1][:-1])], label
            elif "below sf" in label:
                assert ratio == S.next_down(sf[int(label.split("[")[1][:-1])]), label
            elif "above sf[" in label and "n-1" not in label:
                assert ratio == S.next_up(sf[int(label.split("[")[1][:-1])]), label
    if s.routine == "local":
        assert [np.float32(c) for c in s.view_cos[-4:]] == [np.float32(0.998), S.next_down(np.float32(0.998)), 1, 0.5]
    if s.routine == "tri":
        for q, label, matched in s.facts:
            ok, dsqr = S.epipolar(s.k1["x"][q], s.k1["y"][q], s.k2["x"][q], s.k2["y"][q], s.F12, s.sig2[s.k2["octave"][q]])
            thr = 3.84 * np.float64(s.sig2[s.k2["octave"][q]])
            assert ok == matched and (np.float64(dsqr) < thr) == matched, label
            assert (np.float64(S.next_up(dsqr)) >= thr) if matched else (np.float64(S.next_down(dsqr)) < thr), label
        assert len({int(o) for o in s.k2["octave"]}) >= 8   # levels where the walk found both edge floats


@pytest.mark.parametrize("s", SCENES, ids=IDS)
def test_variants_change_exactly_the_named_scenes(s):
    for v in S.ALL_VARIANTS:
        assert S.changes(s, v) == (v in s.variants), v
    assert s.variants <= set(S.VARIANTS_BY_ROUTINE[s.routine])


def test_every_variant_changes_every_routine_it_applies_to():
    for routine, variants in S.VARIANTS_BY_ROUTINE.items():
        for v in variants:
            if v == "radius_pow":   # powf equals the product chain for 1.5 (every power up to 1.5^11 is exact)
                assert np.array_equal(S.scale_table(1.5, 12), S.scale_table(1.5, 12, v))
            assert any(v in s.variants for s in SCENES if s.routine == routine), (routine, v)


def test_scene_geometry_is_general():
    """rotations that are no multiple of 90 degrees, fx != fy, non-integer principal point, depths 0.5-50"""
    for T in S.POSES.values():
        R_ = T[:, :3].astype(np.float64)
        assert np.allclose(R_ @ R_.T, np.eye(3), atol=1e-6)
        assert (np.abs(R_) > 0.05).sum() >= 7
    assert S.FX != S.FY and S.CX != np.round(S.CX) and S.CY != np.round(S.CY)
    depths = np.concatenate([S.camera_point(s.T, s.world)[2] for s in SCENES if s.routine in ("ff", "kf", "f1f2")])
    assert depths.min() >= 0.4 and depths.max() <= 51 and depths.max() > 20 and depths.min() < 5


# ---- the reference's own ORBmatcher ------------------------------------------------------------------------------------------
def _ref_frame(kps, desc, s, which="ref"):
    return R.RefFrame.from_arrays(kps, desc, ORB_W, ORB_H, float(S.FX), float(S.FY), float(S.CX), float(S.CY), s.scale, s.nlevels, which=which)


def run_reference(s, ori):
    if s.routine == "ff":
        n = len(s.world)
        fc, fl = _ref_frame(s.cur_kps, s.cur_desc, s), _ref_frame(s.last_kps, s.last_desc, s)
        out = R.search_by_projection_ff(fc, fl, np.ones(n, np.uint8), np.zeros(n, np.uint8), s.world, s.T, s.th, check_orientation=ori)
        fc.close(); fl.close()
        return out
    if s.routine == "f1f2":
        f1, f2 = _ref_frame(s.f1_kps, s.f1_desc, s), _ref_frame(s.f2_kps, s.f2_desc, s)
        out = R.search_by_projection_f1f2(f1, f2, np.ones(len(s.world), np.uint8), s.world, s.T, s.window, nnratio=s.nnratio)
        f1.close(); f2.close()
        return out
    if s.routine == "local":
        f = _ref_frame(s.kps, s.desc, s)
        out = R.search_local_points(f, np.ones(len(s.proj), np.uint8), s.proj, s.level, s.view_cos, s.mp_desc, s.th, nnratio=s.nnratio)
        f.close()
        return out
    Sc = R.Scene("ref")
    if s.routine == "kf":
        n = len(s.world)
        fcur = Sc.frame(s.cur_kps, s.cur_desc, ORB_W, ORB_H, float(S.FX), float(S.FY), float(S.CX), float(S.CY), s.scale, s.nlevels)
        fkf = Sc.frame(S.keypoints(np.full((n, 2), 320.0), 0), s.desc, ORB_W, ORB_H, float(S.FX), float(S.FY), float(S.CX), float(S.CY),
                       s.scale, s.nlevels)
        kf = Sc.keyframe(fkf, s.T)
        ids = {}
        for i in range(n):
            mp = Sc.map_point(s.world[i], s.desc[i], None, min_dist=float(s.min_dist[i]), max_dist=1e6, ref_kf=kf)
            Sc.observe(kf, mp, i)
            ids[int(mp)] = i
        Sc.set_pose(fcur, s.T)
        nm, mp = Sc.search_by_projection_frame_kf(fcur, kf, [], s.th, s.orb_dist, 0.9, ori)
        fcur.close(); fkf.close()
        return nm, np.array([ids.get(int(m), -1) for m in mp], np.int32)
    n1, n2 = len(s.k1), len(s.k2)
    f1 = Sc.frame(s.k1, s.d1, ORB_W, ORB_H, float(S.FX), float(S.FY), float(S.CX), float(S.CY), s.scale, s.nlevels)
    f2 = Sc.frame(s.k2, s.d2, ORB_W, ORB_H, float(S.FX), float(S.FY), float(S.CX), float(S.CY), s.scale, s.nlevels)
    kf1, kf2 = Sc.keyframe(f1, S.POSES["a"]), Sc.keyframe(f2, S.POSES["b"])
    Sc.set_feature_vector(kf1, one_node(n1))
    Sc.set_feature_vector(kf2, one_node(n2))
    nm, pairs = Sc.search_for_triangulation(kf1, kf2, s.F12, 0.6, ori)
    f1.close(); f2.close()
    m12 = np.full(n1, -1, np.int32)
    for i1, i2 in pairs:
        m12[i1] = i2
    return nm, m12


@pytest.mark.parametrize("s", SCENES, ids=IDS)
def test_reference_orbmatcher_equals_oracle(s):
    needs_ref()
    for ori in ((True, False) if s.routine in ("ff", "kf", "tri") else (True,)):
        n_r, rows_r = run_reference(s, ori)
        n_o, rows_o = run_oracle(s, ori)
        assert n_r == n_o and np.array_equal(rows_r, rows_o), ori
