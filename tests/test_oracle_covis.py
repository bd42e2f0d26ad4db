"""CPU test of the covisibility-graph oracle (oracle/orb_oracle_covis.c) against the reference's own KeyFrame.cc /
MapPoint.cc (oracle/_ref/libref_covis.so): after every step of every scene of tests/covis_scenes.py the ordered lists,
ordered weights, weight maps in key order and parents agree, and the scene model's inputs are what the reference's map
holds."""
import numpy as np
import pytest

import covis_scenes as S
from oracle import covis as OC

pytestmark = pytest.mark.skipif(not OC.ref_available(), reason="oracle/_ref/libref_covis.so not built (needs the reference sources)")


def _compare(ref, orc, slot_of, kfs, where):
    to_slot = lambda ids: [int(slot_of[i]) for i in ids]
    for kf in kfs:
        s = int(slot_of[kf])
        rk, rw = ref.ordered(kf)
        assert (to_slot(rk), rw) == orc.ordered(s), (where, "ordered", kf)
        rk, rw = ref.weights(kf)
        assert (to_slot(rk), rw) == orc.weights(s), (where, "weights", kf)
        rp = ref.parent(kf)
        assert (int(slot_of[rp]) if rp >= 0 else -1) == orc.parent(s), (where, "parent", kf)


def _check_inputs(ref, model, scene, nkf):
    for kf in range(nkf):
        m = ref.matches(kf)
        row = model.kf_mp[kf, :len(m)].copy()
        if len(model.bad):
            row[(row >= 0) & model.bad[np.maximum(row, 0)]] = -1
        assert m == row.tolist(), ("mvpMapPoints", kf)
    for mp in range(len(model.obs)):
        ks, ix = ref.observations(mp)
        o = model.obs[mp]
        assert ks == sorted(o) and ix == [o[k] for k in sorted(o)], ("observations", mp)
        assert ref.point_bad(mp) == bool(model.bad[mp])


def run(scene, full=True):
    """Replays the scene on the reference, the model and the oracle; compares after every step (every keyframe when
    `full`, else the keyframes the step can change)."""
    ref, model, slot_of = OC.RefCovis(), S.Model(scene), scene.slots()
    K = max(scene.nkf, 1)
    orc = OC.CovisOracle(K)
    nkf = 0
    try:
        for t, step in enumerate(scene.steps):
            op = step[0]
            model.apply(step)
            touched = []
            if op == "kf":
                k = ref.add_keyframe(step[1])
                assert k == nkf and ref.mnid(k) == k
                orc.add(slot_of[k], k, k)
                nkf += 1
            elif op == "pts":
                ref.add_points(step[1])
                ref.observe_many(step[2], step[3], step[4])
            elif op == "update":
                kf_mp, counts, gp, obs = model.inputs(slot_of, K)
                for kf in step[1]:
                    before = ref.parent(kf)
                    ref.update(kf)
                    got = orc.update(slot_of[kf], kf_mp, counts, scene.cap, gp, obs if len(obs) else np.zeros(1, np.int32))
                    after = ref.parent(kf)
                    assert got == (int(slot_of[after]) if after >= 0 and before < 0 else -1), (scene.name, t, kf)
                    touched += [kf] + ref.weights(kf)[0]
            elif op == "erase_kf":
                touched = [step[1]] + ref.weights(step[1])[0]
                ref.set_bad_keyframe(step[1])
                orc.erase(slot_of[step[1]])
            elif op == "bad_pt":
                ref.set_bad_point(step[1])
            elif op == "erase_match":
                ref.erase_match(step[1], step[2])
            _compare(ref, orc, slot_of, range(nkf) if full else sorted(set(touched)), (scene.name, t, op))
            if full:
                _check_inputs(ref, model, scene, nkf)
        _compare(ref, orc, slot_of, range(nkf), (scene.name, "end"))
        return ref, orc, slot_of
    finally:
        ref.close()
        orc.close()


@pytest.mark.parametrize("scene", S.small_scenes(), ids=lambda s: s.name)
def test_oracle_equals_reference_keyframe(scene):
    run(scene)


def test_oracle_equals_reference_capacity_scene():
    scene, hub, hub2 = S.scene_capacity()
    scene.update([hub])
    scene.update([hub2])
    run(scene)


def test_scenes_exercise_their_quirks():
    """the scenes reach the cases they are named for (the oracle is checked against the reference above)"""
    sc = S.scene_changed_unchanged()
    ref, model, slot_of = OC.RefCovis(), S.Model(sc), sc.slots()
    try:
        lists = []
        for step in sc.steps:
            model.apply(step)
            if step[0] == "kf":
                ref.add_keyframe(step[1])
            elif step[0] == "pts":
                ref.add_points(step[1])
                ref.observe_many(step[2], step[3], step[4])
            elif step[0] == "update":
                for kf in step[1]:
                    ref.update(kf)
                lists.append(ref.ordered(0))
        assert lists[0] == ([2, 1], [18, 16])          # filtered: D's 5 left out
        assert lists[1] == ([2, 1], [18, 16])          # B's unchanged AddConnection: still filtered
        assert lists[2] == ([2, 1, 3], [20, 16, 5])    # C's changed AddConnection: the full sort
    finally:
        ref.close()
    sc = S.scene_culling()
    ref, orc, slot_of = run(sc)


def test_oracle_equals_reference_large_map():
    """2000 keyframes x 2000 features, ~8 observations per point, updated as batches of 64"""
    run(S.scene_large(), full=False)
