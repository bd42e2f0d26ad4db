"""CPU pins of the MapPoint::UpdateNormalAndDepth rule (DESIGN.md §2): the oracle (oracle/orb_oracle_normal_depth.c) against
the reference's own MapPoint.cc on scripted maps, and against the numpy restatement of tests/normal_depth_scenes.py; each
scene changes under the wrong variants it names; the shim's `x + y*beta` against python-cv2's cv2.scaleAdd golden vectors."""
import os

import numpy as np
import pytest

from oracle import normal_depth as N

import normal_depth_scenes as S

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "opencv_scaleadd.npz")
SCENES = S.all_scenes()
IDS = [s["name"] for s in SCENES]

needs_ref = pytest.mark.skipif(not N.ref_available(), reason="oracle/_ref/libref_drivers.so not built (reference sources absent)")


def _oracle(scene):
    w, rc, ro, gp, oc, _ = S.host_arrays(scene)
    return N.normal_depth(w, rc, ro, gp, oc, scene["scale_factor"], S.scale_table(scene["scale_factor"], scene["nlevels"]))


def _restate(scene, variant=None):
    w, rc, ro, gp, oc, ob = S.host_arrays(scene)
    return S.restate(w, rc, ro, gp, oc, ob, scene["scale_factor"], S.scale_table(scene["scale_factor"], scene["nlevels"]), variant)


def run_reference(scene):
    """The scene through the reference's own KeyFrame / MapPoint: returns (normal, min_dist, max_dist) from the getters,
    after checking that every GetCameraCenter(), the scale table and every observation order are what the scene says."""
    sfac, nl = scene["scale_factor"], scene["nlevels"]
    M = N.RefMap()
    try:
        for k in scene["kfs"]:
            T = np.hstack([np.eye(3, dtype=np.float32), -k["center"].reshape(3, 1)])
            M.add_keyframe(T, k["octaves"], sfac, nl, bad=k["bad"])
        for i, k in enumerate(scene["kfs"]):
            c, s, t = M.keyframe(i, nl)
            assert S.same(c, k["center"]), i
            assert S.same(s, np.float32(sfac)) and S.same(t, S.scale_table(sfac, nl))
        ids = []
        for p in scene["points"]:
            mp = M.add_point(p["pos"], p["ref"])
            for k, j in p["obs"]:
                M.add_observation(mp, k, j)
            assert M.observations(mp) == p["obs"]
            if p["bad"]:
                M.set_point_bad(mp)
            ids.append(mp)
        if any(p["pos2"] is not None for p in scene["points"]):
            for mp in ids:                 # the state before the bundle adjustment
                M.update(mp)
            for mp, p in zip(ids, scene["points"]):
                M.set_world_pos(mp, p["pos2"])
        out = [M.update(mp) for mp in ids]
        return (np.array([o[0] for o in out], np.float32), np.array([o[1] for o in out], np.float32),
                np.array([o[2] for o in out], np.float32))
    finally:
        M.close()


@needs_ref
@pytest.mark.parametrize("scene", SCENES, ids=IDS)
def test_oracle_equals_reference(scene):
    ref = run_reference(scene)
    ora = _oracle(scene)
    for a, b, what in zip(ref, ora, ("normal", "min_dist", "max_dist")):
        assert S.same(a, b), (scene["name"], what)


@pytest.mark.parametrize("scene", SCENES, ids=IDS)
def test_restatement_equals_oracle(scene):
    for a, b in zip(_restate(scene), _oracle(scene)):
        assert S.same(a, b), scene["name"]


@pytest.mark.parametrize("scene", SCENES, ids=IDS)
def test_scene_changes_under_its_variants(scene):
    good = _oracle(scene)
    for v in scene["variants"]:
        assert v in S.VARIANTS
        bad = _restate(scene, v)
        assert not all(S.same(a, b) for a, b in zip(good, bad)), (scene["name"], v)


def test_every_variant_is_named_by_a_scene():
    assert set(S.VARIANTS) == {v for s in SCENES for v in s["variants"]}


def test_scene_facts():
    """Each scene holds what it is built for."""
    by = {s["name"]: s for s in SCENES}
    counts = sorted({len(p["obs"]) for p in by["counts"]["points"]})
    assert counts == [1, 31, 32, 33, 64, 65, 1000]
    assert any(by["bad_keyframes"]["kfs"][k]["bad"] for p in by["bad_keyframes"]["points"] for k, _ in p["obs"])
    for nl in (1, 8, 32):
        sc = by["octaves_L%d" % nl]
        _, _, ro, _, _, _ = S.host_arrays(sc)
        assert set(ro.tolist()) == ({0} if nl == 1 else {0, nl - 1})
    n, a, b = _oracle(by["degenerate"])
    assert a[0] == 0 and b[0] == 0 and np.isfinite(n[0]).all()       # on the reference centre, the reference KF not observing
    assert np.isnan(n[1]).all() and np.isfinite(a[1])                 # on an observer's centre
    assert not n[2].any() and a[2] == 0 and b[2] == 0                 # bad point: untouched
    assert all(p["pos2"] is not None for p in by["local_ba"]["points"])


@needs_ref
def test_rotated_keyframes_through_the_reference():
    """Keyframes with general rotations: the centres are whatever the reference's GetCameraCenter() returns (its
    -Rcw.t()*tcw), and the oracle fed with those bits equals the reference."""
    rng = np.random.default_rng(11)
    M = N.RefMap()
    try:
        kfs, centers, octaves = 50, [], []
        for i in range(kfs):
            q = rng.standard_normal(4)
            q /= np.linalg.norm(q)
            w, x, y, z = q
            R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                          [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                          [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], np.float32)
            t = (rng.standard_normal(3) * 3).astype(np.float32)
            octaves.append(rng.integers(0, 8, 8).astype(np.int32))
            M.add_keyframe(np.hstack([R, t.reshape(3, 1)]), octaves[-1], 1.2, 8)
            centers.append(M.keyframe(i, 8)[0])
        centers = np.array(centers, np.float32)
        world, refc, refo, gp, oc, got = [], [], [], [0], [], []
        for i in range(100):
            ks = np.sort(rng.choice(kfs, int(rng.integers(1, 40)), replace=False))
            r = int(ks[rng.integers(0, len(ks))])
            pos = (centers[r] + rng.standard_normal(3) * 10).astype(np.float32)
            mp = M.add_point(pos, r)
            for k in ks:
                M.add_observation(mp, int(k), int(k) % 8)
            got.append(M.update(mp))
            world.append(pos)
            refc.append(centers[r])
            refo.append(octaves[r][r % 8])
            gp.append(gp[-1] + len(ks))
            oc.extend(centers[ks])
        assert len({tuple(c) for c in centers.tolist()}) == kfs
        ora = N.normal_depth(np.array(world), np.array(refc), refo, gp, np.array(oc), 1.2, S.scale_table(1.2, 8))
        assert S.same(np.array([g[0] for g in got]), ora[0])
        assert S.same(np.array([g[1] for g in got]), ora[1]) and S.same(np.array([g[2] for g in got]), ora[2])
    finally:
        M.close()


def _golden():
    d = np.load(GOLD)
    a, b, al, out = d["src1"], d["src2"], d["alpha"], d["out"]
    sep = (a * al[:, None]).astype(np.float32) + b                                     # product rounded, then the add
    fused = (a.astype(np.float64) * al[:, None].astype(np.float64) + b).astype(np.float32)
    return a, b, al, out, sep, fused


def test_golden_cases_discriminate_fusion():
    a, b, al, out, sep, fused = _golden()
    assert len(a) == 500 and (sep != fused).any(axis=1).all()


@needs_ref
def test_shim_scale_add_against_cv2_golden():
    """The shim evaluates `normal + normali/cv::norm(normali)` as OpenCV 2.4's scaleAdd_32f does: the product rounded to
    float, then the add.  python-cv2 4.13's cv2.scaleAdd returns the FUSED value on every component where the two differ
    (its scalar tail is compiled with FMA contraction), so it cannot arbitrate this rule: the shim equals cv2 wherever the
    roundings agree and equals the separately rounded value everywhere.  Pinned as found, so that a cv2 that changes
    either way shows up here."""
    a, b, al, out, sep, fused = _golden()
    got = np.array([N.shim_scale_add(b[i], a[i], float(al[i])) for i in range(len(a))])
    diff = sep != fused
    assert S.same(got, sep)
    assert S.same(got[~diff], out[~diff])
    assert S.same(out[diff], fused[diff])
