"""CPU test of the GetObservations oracle (oracle/orb_oracle_observations.c): after every step of every scene of
tests/observation_scenes.py and tests/covis_scenes.py (the large map included), the oracle's list of every point, built
from the live keyframes' rows alone, equals the reference's own MapPoint::GetObservations() (oracle/_ref/libref_observations.so),
and its ref_obs equals observations[GetReferenceKeyFrame()] with absent read as 0.  The one scene that overwrites a row
cell without a reference path differs from the reference exactly as DESIGN.md §2 records."""
import numpy as np
import pytest

import covis_scenes as S
import observation_scenes as OS
from oracle import observations as OO

needs_ref = pytest.mark.skipif(not OO.ref_available(), reason="oracle/_ref/libref_observations.so not built (needs the reference sources)")


def oracle_inputs(model, slot_of, K):
    """kf_mp / counts in slot rows (Model.inputs), live and keys per slot (key = creation index), ref slot per point"""
    kf_mp, counts, gp, obs = model.inputs(slot_of, K)
    n = len(model.nfeat)
    live, keys = np.zeros(K, np.uint8), np.zeros(K, np.uint64)
    live[slot_of[:n]] = model.live() if isinstance(model, OS.ObsModel) else ~np.array(model.kf_bad, bool)
    keys[slot_of[:n]] = np.arange(n, dtype=np.uint64)
    ref = getattr(model, "ref", None)
    ref_slot = np.array([slot_of[r] if r >= 0 else 0 for r in ref], np.int32) if ref is not None else None
    return kf_mp, counts, gp, obs, live, keys, ref_slot


def ref_step(ref, model, step):
    """the step on the reference's own map"""
    op = step[0]
    if op in ("kf", "kfq"):
        ref.add_keyframe(step[1])
    elif op == "pts":
        ref.add_points(step[1])
        ref.observe_many(step[2], step[3], step[4])
    elif op == "update":
        for kf in step[1]:
            ref.update(kf)
    elif op == "erase_kf":
        ref.set_bad_keyframe(step[1])
    elif op == "bad_pt":
        ref.set_bad_point(step[1])
    elif op == "erase_match":
        ref.erase_match(step[1], step[2])
    elif op == "row":
        ref.add_map_point(step[1], step[2], step[3])
    elif op == "process":   # ProcessNewKeyFrame, mnId > 1: every match that is not bad, ascending i
        for i, m in enumerate(ref.matches(step[1])):
            if m >= 0:
                ref.add_observation(m, step[1], i)
    elif op == "observe":
        ref.observe(step[1], step[2], step[3])
    elif op == "replace":
        ref.replace(step[1], step[2])
    elif op == "ba_erase":
        ref.ba_erase(step[1], step[2])


def compare(ref, model, scene, slot_of, points, where):
    K, cap = scene.nkf, scene.cap
    kf_mp, counts, gp, obs, live, keys, ref_slot = oracle_inputs(model, slot_of, K)
    rc, ptr, got, nobs, ref_obs = OO.observations(points, len(model.obs), kf_mp, counts, cap, live, keys, ref_slot)
    assert rc == 0, where
    div = getattr(model, "divergent", set())
    for j, m in enumerate(points):
        ks, ix = ref.observations(m)
        want = [int(slot_of[k]) * cap + i for k, i in zip(ks, ix)]
        lst = got[ptr[j]:ptr[j + 1]].tolist()
        if m in div:   # a row overwrite: pinned by test_overwritten_cell_is_recorded
            continue
        assert lst == want, (where, "observations", m)
        if ref_obs is not None and not ref.point_bad(m):
            r = ref.reference(m)
            assert r == model.ref[m], (where, "mpRefKF", m)
            o = dict(zip(ks, ix))
            assert ref_obs[j] == int(slot_of[r]) * cap + o.get(r, 0), (where, "ref_obs", m)
    return ptr, got


def run(scene, model_cls=OS.ObsModel, every=True):
    ref, model, slot_of = OO.RefObservations(), model_cls(scene), scene.slots()
    try:
        for t, step in enumerate(scene.steps):
            model.apply(step)
            ref_step(ref, model, step)
            if every or step[0] != "update":
                compare(ref, model, scene, slot_of, list(range(len(model.obs))), (scene.name, t, step[0]))
        return model
    finally:
        ref.close()


@needs_ref
@pytest.mark.parametrize("scene", OS.small_scenes(), ids=lambda s: s.name)
def test_oracle_equals_reference_observations(scene):
    run(scene)


@needs_ref
@pytest.mark.parametrize("scene", S.small_scenes(), ids=lambda s: s.name)
def test_oracle_equals_reference_on_covis_scenes(scene):
    run(scene)


@needs_ref
def test_oracle_equals_reference_large_map():
    """2000 keyframes x 2000 features, ~8 observations per point"""
    run(S.scene_large(), every=False)


@needs_ref
def test_overwritten_cell_is_recorded():
    """the row overwrite: the oracle's inverse lists b for the new point and drops it from the old one, while the
    reference's old point keeps b"""
    scene = OS.scene_overwritten_cell()
    ref, model, slot_of = OO.RefObservations(), OS.ObsModel(scene), scene.slots()
    try:
        for step in scene.steps:
            model.apply(step)
            ref_step(ref, model, step)
        a, b, c = 0, 1, 2
        old, new = 1, 4
        assert model.divergent == {old, new}
        assert [k for k in ref.observations(old)[0]] == [a, b, c]
        assert ref.observations(new)[0] == [a, c]
        kf_mp, counts, _, _, live, keys, _ = oracle_inputs(model, slot_of, scene.nkf)
        rc, ptr, got, _, _ = OO.observations([old, new], len(model.obs), kf_mp, counts, scene.cap, live, keys)
        assert rc == 0
        assert got[ptr[0]:ptr[1]].tolist() == [int(slot_of[a]) * scene.cap + 1, int(slot_of[c]) * scene.cap + 1]
        assert got[ptr[1]:ptr[2]].tolist() == [int(slot_of[k]) * scene.cap + i for k, i in ((a, 10), (b, 1), (c, 10))]
    finally:
        ref.close()


def test_oracle_lists_are_the_model_host_lists():
    """on every scene up to its first row overwrite or lone erase_match, the all-points lists are Model.inputs' group_ptr / obs (the host lists the
    three existing device entries take)"""
    for scene in OS.small_scenes() + S.small_scenes():
        model, slot_of = OS.ObsModel(scene), scene.slots()
        for step in scene.steps:
            model.apply(step)
            if model.divergent:
                break
            kf_mp, counts, gp, obs, live, keys, _ = oracle_inputs(model, slot_of, scene.nkf)
            rc, ptr, got, nobs, _ = OO.observations(np.arange(len(model.obs)), len(model.obs), kf_mp, counts, scene.cap, live, keys)
            assert rc == 0 and ptr.tolist() == gp.tolist() and got.tolist() == obs.tolist(), (scene.name, step[0])


def test_oracle_statuses():
    """bad input: only ptr; overflow: ptr and the size needed"""
    cap, K = 4, 3
    kf_mp = np.array([0, 1, 0, -1, 1, 2, -1, -1, 2, 0, 1, -1], np.int32)
    counts = np.array([4, 4, 4], np.int32)
    live, keys = np.ones(K, np.uint8), np.array([30, 10, 20], np.uint64)
    rc, ptr, obs, nobs, _ = OO.observations([0, 1, 2], 3, kf_mp, counts, cap, live, keys)
    assert rc == 0 and ptr.tolist() == [0, 2, 5, 7] and nobs == 7
    # key order is slot 1, 2, 0; slot 0 names point 0 at features 0 and 2: the last one
    assert obs.tolist() == [2 * cap + 1, 0 * cap + 2, 1 * cap + 0, 2 * cap + 2, 0 * cap + 1, 1 * cap + 1, 2 * cap + 0]
    assert OO.observations([0, 1, 2], 3, kf_mp, counts, cap, live, keys, obs_cap=ptr[-1] - 1)[:2][0] == -3
    assert OO.observations([0, 1, 2], 3, kf_mp, counts, cap, live, keys, obs_cap=ptr[-1] - 1)[3] == ptr[-1]
    assert OO.observations([0, 0], 3, kf_mp, counts, cap, live, keys)[0] == -1
    assert OO.observations([3], 3, kf_mp, counts, cap, live, keys)[0] == -1
    assert OO.observations([0], 2, kf_mp, counts, cap, live, keys)[0] == -1          # a row value >= npoints
    assert OO.observations([0], 3, kf_mp, np.array([5, 4, 4], np.int32), cap, live, keys)[0] == -1
    assert OO.observations([0], 3, kf_mp, np.array([5, 4, 4], np.int32), cap, np.array([0, 1, 1], np.uint8), keys)[0] == 0   # not live
    assert OO.observations([0], 3, kf_mp, counts, cap, live, keys, ref_slot=[3])[0] == -1
