"""CPU test of the KeyFrameCulling oracle (oracle/orb_oracle_kf_culling.c): after every step of every scene of
tests/kf_culling_scenes.py (the 2000 x 2000 map included), the reference's own LocalMapping::KeyFrameCulling
(oracle/_ref/libref_kf_culling.so) and the oracle, run on the same map, agree on the verdict list, and the map the scene's
model reaches by erasing the reference's ERASED keyframes in list order equals the reference's in every keyframe's row,
every point's isBad(), mpRefKF and observation list, and the oracle's rows, point flags, reference slots and made-bad
points.  Also: the device's integer comparison equals the reference's double one for every nMPs up to 65535, and the
oracle's statuses."""
import numpy as np
import pytest

import covis_key_scenes as KM
import covis_scenes as S
import kf_culling_scenes as KS
from oracle import kf_culling as KC
from test_oracle_observations import ref_step as obs_ref_step

needs_ref = pytest.mark.skipif(not KC.ref_available(), reason="oracle/_ref/libref_kf_culling.so not built (needs the reference sources)")


def cull_inputs(model, slot_of, K, not_erase=(), keys=None):
    """the oracle's (and the device's) per-slot arrays from the model: rows (bad points -1), counts, live, mnId == 0, keys
    (keys[k] for keyframe k; the creation index when None), mbNotErase, octaves, point flags and reference slots"""
    cap, n = model.cap, len(model.nfeat)
    kf_mp, counts, _, _ = model.inputs(slot_of, K)
    live, id0, ne = np.zeros(K, np.uint8), np.zeros(K, np.uint8), np.zeros(K, np.uint8)
    key_slot = np.zeros(K, np.uint64)
    live[slot_of[:n]] = model.live()
    id0[slot_of[:n]] = [m == 0 for m in model.mnid]
    key_slot[slot_of[:n]] = KM.key_list(keys, n)
    ne[[int(slot_of[k]) for k in not_erase]] = 1
    octave = np.zeros((K, cap), np.int32)
    octave[slot_of[:n]] = model.oct
    ref_slot = np.array([slot_of[r] if r >= 0 else 0 for r in model.ref], np.int32)
    return dict(kf_mp=kf_mp, counts=counts, live=live, id0=id0, keys=key_slot, not_erase=ne, octave=octave.ravel(),
                point_bad=model.bad.astype(np.uint8), ref_slot=ref_slot)


def oracle_cull(model, slot_of, K, cand_slots, not_erase=(), obs_cap=None, keys=None):
    a = cull_inputs(model, slot_of, K, not_erase, keys)
    return KC.cull(cand_slots, a["live"], a["id0"], a["keys"], a["not_erase"], a["kf_mp"], a["counts"], a["octave"], model.cap,
                   a["point_bad"], a["ref_slot"], obs_cap=obs_cap), a


def normalized(rows, bad):
    r = np.array(rows, np.int32)
    m = r >= 0
    if len(bad):
        r[m & bad[np.where(m, r, 0)]] = -1
    return r


def compare_map(ref, model, where, points=None):
    """the model's map equals the reference's: rows, isBad(), observations, mpRefKF"""
    for k in range(len(model.nfeat)):
        want = normalized(model.kf_mp[k, :model.nfeat[k]], model.bad).tolist()
        assert ref.matches(k) == want, (where, "row", k)
    for m in (range(len(model.obs)) if points is None else points):
        assert ref.point_bad(m) == bool(model.bad[m]), (where, "isBad", m)
        ks, ix = ref.observations(m)
        assert list(zip(ks, ix)) == sorted(model.obs[m].items(), key=lambda e: model.key(e[0])), (where, "observations", m)
        if not model.bad[m]:
            assert ref.reference(m) == model.ref[m], (where, "mpRefKF", m)


def run(scene, check_every=True, keys=None, trace=None):
    """keys[k] is keyframe k's order key (the creation index when None); with `trace`, every cull's oracle result is
    appended to it"""
    ref, model, slot_of = KC.RefKfCulling(), KS.CullModel(scene, keys), scene.slots()
    K = scene.nkf
    try:
        if keys is not None:
            ref.set_kf_order(KM.rank(keys[:scene.nkf]))
        for t, step in enumerate(scene.steps):
            where = (scene.name, t, step[0])
            op = step[0]
            if op == "octave":
                model.apply(step)
                ref.set_octaves(step[1], model.oct[step[1]])
                continue
            if op != "cull":
                model.apply(step)
                obs_ref_step(ref, model, step)
                if check_every:
                    compare_map(ref, model, where)
                continue
            cur, ne = step[1], step[2]
            for k in ne:
                ref.set_not_erase(k)
            ids = ref.ordered(cur)[0]
            out, _ = oracle_cull(model, slot_of, K, slot_of[ids], ne, keys=keys)
            assert out["status"] == 0, where
            if trace is not None:
                trace.append({k: (v.tolist() if hasattr(v, "tolist") else v) for k, v in out.items()})
            rids, verdicts, _ = ref.cull(cur)
            assert rids == ids, where
            assert out["verdict_slot"].tolist() == slot_of[ids].tolist(), where
            assert out["verdict"].tolist() == verdicts, (where, list(zip(ids, verdicts)), out["verdict"].tolist())
            was_bad = model.bad.copy()
            model.apply(step, erased=[k for k, v in zip(ids, verdicts) if v == KC.ERASED])
            compare_map(ref, model, where)
            assert (out["point_bad"].astype(bool) == model.bad).all(), where
            assert out["bad_points"].tolist() == np.flatnonzero(model.bad & ~was_bad).tolist(), where
            assert (normalized(out["kf_mp"], model.bad) == model.inputs(slot_of, K)[0]).all(), where
            defined = np.array([r >= 0 for r in model.ref], bool)
            assert (out["ref_slot"][defined] == slot_of[np.array(model.ref)[defined]]).all(), where
        return model
    finally:
        ref.close()


@needs_ref
@pytest.mark.parametrize("scene", KS.small_scenes(), ids=lambda s: s.name)
def test_oracle_equals_reference_kf_culling(scene):
    run(scene)


@needs_ref
def test_scenes_reach_their_verdicts():
    """each scene produces the verdicts its docstring names (so it fails under the wrong variant it is built against)"""
    E, Kp, R, N, Z = KC.ERASED, KC.KEPT, KC.RETIRED, KC.NOT_ERASE, KC.SKIP_ID0
    want = {   # creation index -> verdict, for the keyframes each scene is about
        "nothing_redundant": {4: Kp, 5: Kp}, "ratio_boundary": {4: Kp, 5: E, 6: Kp}, "observations_3_4": {4: Kp, 5: E},
        "octave_gate": {4: E, 5: Kp}, "duplicate_cells": {4: Kp}, "order": {4: Kp, 5: E, 6: E, 7: E},
        "id0_not_erase": {0: Z, 4: N}, "stale": {5: Kp, 6: R}, "ref_and_cascade": {5: E},
    }
    for scene in KS.small_scenes():
        ref, model = KC.RefKfCulling(), KS.CullModel(scene)
        try:
            for step in scene.steps:
                if step[0] == "octave":
                    model.apply(step)
                    ref.set_octaves(step[1], model.oct[step[1]])
                elif step[0] == "cull":
                    for k in step[2]:
                        ref.set_not_erase(k)
                    ids, verdicts, _ = ref.cull(step[1])
                    got = dict(zip(ids, verdicts))
                    for k, v in want[scene.name].items():
                        assert got.get(k) == v, (scene.name, k, got)
                else:
                    model.apply(step)
                    obs_ref_step(ref, model, step)
        finally:
            ref.close()


@needs_ref
def test_oracle_equals_reference_large_map():
    """2000 keyframes x 2000 features, ~8 observations per point, two culls"""
    run(KS.large_culls(S.scene_large()), check_every=False)


def test_integer_comparison_equals_the_double_one():
    """10*r > 9*n (the device) == (double)r > 0.9*(double)n (LocalMapping.cc:573) for every n in 0..65535 and r in 0..n: both
    hold exactly from a threshold on r up, and the thresholds are equal"""
    n = np.arange(65536, dtype=np.int64)
    t_int = (9 * n) // 10 + 1                    # the least r with 10*r > 9*n
    nd = 0.9 * n.astype(np.float64)
    assert (t_int.astype(np.float64) > nd).all()
    assert not ((t_int - 1).astype(np.float64) > nd).any()


def test_oracle_statuses():
    """bad input: -1 with nothing written; overflow: -3 with the size needed"""
    cap, K = 4, 3
    kf_mp = np.array([0, 1, 2, -1, 0, 1, 2, -1, 0, 1, -1, -1], np.int32)
    counts = np.array([4, 4, 4], np.int32)
    live, id0, keys, ne = np.ones(K, np.uint8), np.array([1, 0, 0], np.uint8), np.arange(K, dtype=np.uint64), np.zeros(K, np.uint8)
    octave = np.zeros(K * cap, np.int32)
    pb, rs = np.zeros(3, np.uint8), np.zeros(3, np.int32)

    def call(**kw):
        a = dict(cand=[1, 2], live=live, id0=id0, keys=keys, not_erase=ne, kf_mp=kf_mp, counts=counts, octave=octave, cap=cap,
                 point_bad=pb, ref_slot=rs)
        a.update(kw)
        return KC.cull(**a)

    ok = call()
    assert ok["status"] == 0 and ok["nobs"] == 8 and ok["verdict"].tolist() == [KC.KEPT, KC.KEPT]
    assert call(obs_cap=7)["status"] == -3 and call(obs_cap=7)["nobs"] == 8
    assert call(counts=np.array([4, 5, 4], np.int32))["status"] == -1
    assert call(kf_mp=np.where(kf_mp == 2, 3, kf_mp))["status"] == -1
    bad_oct = octave.copy()
    bad_oct[0] = 32                                                  # an observer of point 0 at octave 32
    assert call(octave=bad_oct)["status"] == -1
    assert call(octave=bad_oct, point_bad=np.array([1, 0, 0], np.uint8))["status"] == 0   # ... of a bad point: not read
    assert call(ref_slot=np.array([0, 3, 0], np.int32))["status"] == -1
    assert call(cand=[1, 3])["status"] == -1                          # a listed slot >= nframes
